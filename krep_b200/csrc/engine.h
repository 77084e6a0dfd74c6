// engine.h — per-device engine contexts and internal entry points shared by engine.cu / host_api.cu.
//
// One process can drive several CUDA devices (krep.c:2851-2905 hands chunks to pool threads; here the chunks of one
// search call go to the visible H100s): every device the library touches gets a DevCtx — two streams, its occurrence
// list, its staging ring — created on first use.  Plans are compiled once on the host and uploaded to a device the
// first time it runs them (plan_on_device).
#pragma once
#include <mutex>
#include <vector>
#include "common.h"

namespace kb {

// Occurrence lists of up to PACK_KEYS keys are sorted by one CTA (k_finish) and come back to the host together with
// the count in the scan's single stream synchronisation; longer lists take the CUB radix sort + a second read-back.
static constexpr uint32_t PACK_KEYS = 16384;
static constexpr int SCAN_SLOTS = 2; // scans in flight per device (krep_b200_scan_shard_begin / _end)

struct StageSlot
{
    uint8_t *buf = nullptr; // pinned
    cudaEvent_t ev = nullptr;
    bool in_flight = false;
};

struct PendingScan
{
    bool active = false;
    const Plan *plan = nullptr;
    krep_b200_shard_t shard;
    int want_positions = 0;
    cudaStream_t stream = nullptr;
};

struct RegexPackBufs;
struct LongBufs;

struct DevCtx
{
    bool ready = false;
    int device = 0, sm_count = 0;
    cudaStream_t scan_stream = nullptr, copy_stream = nullptr;
    cudaStream_t fin_stream = nullptr; // spare stream (k_finish ran here in an experiment; it now follows its scan in-stream)
    // every scan slot has its own occurrence list and counter: scan i+1 may append while k_finish still sorts list i
    unsigned long long *d_counter = nullptr;                // per slot, 64 bytes apart: [0] occurrences, [1] finished k_finish CTAs
    bool counter_clean[SCAN_SLOTS] = {false, false};        // k_finish leaves the counter at zero: no memset before the next scan
    uint64_t *d_list[SCAN_SLOTS] = {nullptr, nullptr};      // key_cap keys each
    uint64_t *d_alt = nullptr;                              // radix sort's alternate buffer (lists beyond PACK_KEYS)
    uint64_t key_cap = 0;
    void *d_sort_tmp = nullptr;
    size_t sort_tmp_bytes = 0;
    uint64_t *d_bounds = nullptr; // -c: line bounds, 2 per key
    uint64_t bounds_cap = 0;
    uint64_t *h_bounds = nullptr; // pinned
    uint64_t h_bounds_cap = 0;
    // scan results: [0] = occurrence count, [1 .. 1+min(count, PACK_KEYS)] = sorted keys; h_pack is mapped pinned memory
    // the finish kernel writes through, d_pack the device copy that krep_b200_export_packed hands to a collective
    uint64_t *d_pack[SCAN_SLOTS] = {nullptr, nullptr}, *h_pack[SCAN_SLOTS] = {nullptr, nullptr};
    cudaEvent_t ev_a[SCAN_SLOTS] = {nullptr, nullptr}, ev_b[SCAN_SLOTS] = {nullptr, nullptr};
    cudaEvent_t ev_done[SCAN_SLOTS] = {nullptr, nullptr}; // recorded after k_finish: what scan_end waits for
    cudaEvent_t ev_scanned[SCAN_SLOTS] = {nullptr, nullptr}; // recorded on the scan's stream when its kernels are enqueued
    cudaEvent_t ev_ca = nullptr, ev_cb = nullptr;          // timing of krep_b200_count_lines_shard
    PendingScan pend[SCAN_SLOTS];
    int next_slot = 0;
    uint64_t serial = 0;
    cudaStream_t result_stream = nullptr; // stream the most recent result's device lists were produced on
    // fused -c (scan_count.cu): one record per partition
    void *d_line_recs = nullptr;
    uint64_t line_recs_cap = 0;
    uint64_t *d_line_out = nullptr, *h_line_out = nullptr; // shard records (lines, flags), 2 words each; h_ is mapped pinned
    uint64_t line_out_cap = 0;
    unsigned long long *d_set_acc = nullptr; // pattern-set -c (scan_set_count.cu): k_set_lines' two accumulators
    // host-text entry points: device ring the caller's buffer streams through + pinned staging ring + key read-back
    uint8_t *d_ring = nullptr;
    size_t ring_slot_bytes = 0;
    int ring_slots = 0;
    std::vector<cudaEvent_t> ring_landed, ring_scanned;
    std::vector<StageSlot> stage;
    size_t stage_bytes = 0;
    std::vector<cudaEvent_t> ev_pool;
    uint64_t *h_keys = nullptr; // pinned
    uint64_t h_keys_cap = 0;
    uint8_t *h_batch = nullptr; // pinned: texts of one krep_b200_search_batch call, packed
    uint64_t h_batch_cap = 0;
    uint8_t *d_rx_batch = nullptr; // the text table of a krep_b200_regex_search_batch call (RegexBatchDev)
    size_t rx_batch_cap = 0;
    // resident batches (krep_b200_search_batch_resident, DESIGN §12.9): the packed texts, grown on demand and kept, and
    // the gather table (source offset, packed offset, length per text) with one last byte per text after it
    uint8_t *d_gather = nullptr;
    uint64_t gather_cap = 0;
    uint64_t *d_gather_tab = nullptr;
    uint64_t gather_tab_cap = 0; // bytes
    RegexPackBufs *rx_pack = nullptr; // -E rows of resident shards (scan_regex_pack.cu)
    LongBufs *rx_long = nullptr;      // scratch of the -E long-line pass (scan_regex_long.cu)
};

// scan_regex_pack.cu — the -E row of a resident shard (layout: RegexRowHeader, csrc/common.h)
struct RegexPackStats
{
    float scan_ms = 0.f, pack_ms = 0.f; // device time: the k_regex_lines scan with its sort, and the pack kernels
    uint64_t packed_bytes = 0;          // row bytes
};
// One k_regex_lines scan of the shard in `mode` with its keys sorted on the device (engine.cu); long_lines: followed by
// the long-line pass (nullptr: not).  batch: the shard is a packed -E batch with this text table, scanned in the
// kernel's batch mode; the count mode then leaves one line count per text in device_lines[0 .. batch->n_texts).
int regex_scan_keys(DevCtx &E, const Plan *plan, const krep_b200_shard_t *shard, RegexMode mode, const char *who, uint64_t *cnt,
                    const uint64_t **d_sorted, uint64_t *device_lines, const LongLineOpts *long_lines = nullptr,
                    const RegexBatchDev *batch = nullptr);
// Packs the row of the shard whose sorted keys (nkeys, in `mode`'s layout) are at d_keys into engine-owned device memory
// on the device's scan stream, and synchronises: *d_row, *row_bytes.  The row stays valid until the next pack on the device.
int regex_pack_row(DevCtx &E, const krep_b200_shard_t *sh, int mode, const uint64_t *d_keys, uint64_t nkeys,
                   uint64_t device_lines, const void **d_row, uint64_t *row_bytes, float *pack_ms);
uint8_t *regex_pack_host_buffer(DevCtx &E, uint64_t bytes); // pinned host room for a row read-back (grown as needed)
void regex_pack_free(DevCtx &E);
// scan_batch_gather.cu: k_batch_gather on stream st.  d_tab: nt source offsets (bytes from d_base), nt packed offsets
// (ascending, 16-byte aligned), nt lengths; writes total bytes (a multiple of 16) to d_out, fill between the texts, and
// each non-empty text's last byte to d_last[t] when d_last is set.
int batch_gather(const void *d_base, const uint64_t *d_tab, uint32_t nt, uint64_t total, uint8_t fill, uint8_t *d_out,
                 uint8_t *d_last, cudaStream_t st);
void long_lines_free(DevCtx &E);

struct ErrState
{
    int code = 0;
    char msg[512] = "";
};
void get_error(ErrState *e);         // the calling thread's error state
void adopt_error(const ErrState &e); // make another thread's error this thread's (no second print)

std::recursive_mutex &engine_mutex();
int primary_device();            // device bound by krep_b200_init, else the calling thread's current device; -1 = no GPU
int visible_devices();           // cudaGetDeviceCount (0 when CUDA is unusable)
DevCtx *ctx_get(int device);     // creates the context on first use; nullptr after set_error
DevCtx *ctx_primary();           // ctx_get(primary_device())
DevCtx *ctx_of_pointer(const void *d_ptr); // the context of the device that owns d_ptr, else ctx_primary()
void engine_shutdown();
void prewarm_host_path(DevCtx &C); // host_api.cu: rings + occurrence list for the pageable-text path
void keep_devices_visible(); // the host manages devices itself: do not narrow CUDA_VISIBLE_DEVICES
void warm_join();    // waits for the krep_b200_warmup thread, if one is running
bool warm_running();

struct DeviceGuard // restores the calling thread's current device
{
    int saved = -1;
    DeviceGuard() { if (cudaGetDevice(&saved) != cudaSuccess) { saved = -1; cudaGetLastError(); } }
    ~DeviceGuard() { if (saved >= 0) cudaSetDevice(saved); }
};

Plan *plan_build(const search_params_t *P, int algo, bool only_matching);
// nullptr = refused (no error raised); max_states below REGEX_MAX_STATES only for test plans (krep_b200_regex_plan_split)
Plan *regex_plan_build(const search_params_t *P, std::string *why, uint32_t max_states = REGEX_MAX_STATES);
void plan_free(Plan *p);
const PlanDev *plan_on_device(const Plan *p, DevCtx &C); // uploads on first use; nullptr on CUDA errors
int resolve_algo(const search_params_t *P, int algo); // host_api.cu: precondition fallbacks of the simd_* entries

unsigned long long *slot_counter(DevCtx &C, int slot);
int scan_begin(DevCtx &C, const Plan *plan, const krep_b200_shard_t *sh, int want_positions, cudaStream_t stream, int *slot);
int scan_end(DevCtx &C, int slot, ScanOut *out);
int scan_shard(DevCtx &C, const Plan *plan, const krep_b200_shard_t *sh, int want_positions, cudaStream_t stream, ScanOut *out);
// k_finish: count + small-list sort + counter reset; keys_to_host = false brings back the count only
int finish_scan(DevCtx &C, int slot, int want_sort, cudaStream_t stream, bool keys_to_host = true);
int ensure_keys(DevCtx &C, uint64_t cap);
int reset_counter(DevCtx &C, int slot, cudaStream_t stream);
int sort_keys(DevCtx &C, int slot, uint64_t n, int end_bit, cudaStream_t stream, const uint64_t **sorted);
int key_end_bit(const Plan *plan, uint64_t max_offset, RegexMode mode = RX_FILTER); // mode: of a regex plan's keys
int fetch_keys(DevCtx &C, const ScanOut &so, const uint64_t **h); // sorted keys on the host (no copy when they came back packed)
void add_kernel_ms(float ms);
void reset_kernel_ms();
float get_kernel_ms();
void set_kernel_ms(float ms);
void trace(const char *fmt, ...); // KREP_B200_TRACE=1: "[krep_b200 +12.3 ms] ..." on stderr

// scan_count.cu — fused -c (count of matching lines computed in the scan)
bool count_lines_eligible(const Plan *plan, const search_params_t *P, int algo);
int ensure_line_out(DevCtx &C, uint64_t n);
int launch_count_lines(DevCtx &C, const Plan *plan, const krep_b200_shard_t *sh, cudaStream_t stream, uint64_t index);
uint64_t combine_line_records(const uint64_t *recs, size_t n); // records in text order -> number of matching lines

// scan_set_count.cu — fused -c for pattern sets (count_lines_eligible AC plans).  set_count_begin enqueues the shard's
// scan into the occurrence list of `slot` with k_finish (count only to the host); set_count_end waits for that count and
// enqueues the record into E.h_line_out / E.d_line_out at `index` (synchronous when the list overflowed).  Work on one
// slot must be ended before the slot is begun again; the other slot may be begun in between.
int set_count_slot(const DevCtx &C); // a slot that no krep_b200_scan_shard_begin holds
int set_count_begin(DevCtx &C, const Plan *plan, const krep_b200_shard_t *sh, cudaStream_t stream, int slot);
int set_count_end(DevCtx &C, const Plan *plan, const krep_b200_shard_t *sh, cudaStream_t stream, int slot, uint64_t index);

// Merges ascending key lists into dst (room for the sum of counts); lists of literal keys from rank-ordered shards are
// already globally ordered, lists of pattern-set keys (ordered by END offset but owned by START offset) are not.
uint64_t merge_key_lists(const uint64_t *const *lists, const uint64_t *counts, uint32_t n_lists, uint64_t *dst);

} // namespace kb
