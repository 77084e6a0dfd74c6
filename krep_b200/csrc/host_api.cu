// host_api.cu — the search_func_t-typed entry points (host text in, match_result_t out) and the rest of
// the host-facing C ABI: option globals, dispatch (select_search_algorithm), AC trie handles,
// match_result helpers.
//
// Data path of one call (north_star): the caller's buffer (krep's mmap, krep.c:2680) is staged into
// HBM in chunks — straight from the caller's memory when it is already page-locked, otherwise through
// a ring of pinned staging buffers filled by host threads — with cudaMemcpyAsync on a copy stream,
// while the scan stream runs the filter kernel on every chunk whose bytes have landed.  All chunk
// kernels append to one device occurrence list, which is sorted on the device, read back, and replayed
// under the emulated kernel's policy (semantics.cpp).  There is no CPU scan anywhere on this path.
#include <algorithm>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <omp.h>
#include <sys/mman.h>
#include <thread>
#include "common.h"
#include "engine.h"

namespace kb {

// ---- krep.c:117-120 mirrored option globals ---------------------------------------------------
static bool g_only_matching = false;
static bool g_force_no_simd = false;
static std::string g_algo_override; // "", "auto", "bm", "kmp"

// The reference binary this library stands in for is the AVX2 build (Makefile:31-35, krep.c:47-59):
// KREP_USE_AVX2 = KREP_USE_SSE42 = 1, SIMD_MAX_PATTERN_LEN = 32 (krep.c:104-106).
static constexpr size_t SIMD_MAX_PATTERN_LEN = 32;

// Precondition fallbacks of the simd_* entry points (krep.c:4708-4712, 4883-4895, 5115-5126).
int resolve_algo(const search_params_t *P, int algo)
{
    const size_t m = P->pattern_len;
    if (algo == KREP_B200_ALGO_AVX512)
    {
        if (m == 0 || m > 64 || !P->case_sensitive) return KREP_B200_ALGO_BMH;
        if (m <= 32) algo = KREP_B200_ALGO_AVX2;
    }
    if (algo == KREP_B200_ALGO_AVX2)
    {
        if (m == 0 || m > 32 || !P->case_sensitive) return KREP_B200_ALGO_BMH;
        if (m <= 16) algo = KREP_B200_ALGO_SSE42;
    }
    if (algo == KREP_B200_ALGO_SSE42)
    {
        if (m == 0 || m > 16 || !P->case_sensitive) return KREP_B200_ALGO_BMH;
    }
    if (algo == KREP_B200_ALGO_NEON && (m == 0 || !P->case_sensitive)) return KREP_B200_ALGO_BMH; // krep.c:4511
    return algo;
}

// ---- plan cache ---------------------------------------------------------------------------------
static std::vector<Plan *> g_plan_cache; // most recent last; plans are device-independent (uploaded per device on use)

static bool plan_matches(const Plan *pl, const search_params_t *P, int algo, bool only_matching)
{
    if (pl->is_regex || algo == KREP_B200_ALGO_REGEX) return false; // regex plans: cached_regex_plan
    if (pl->algo != algo || pl->case_sensitive != P->case_sensitive || pl->count_lines != P->count_lines_mode) return false;
    if (pl->is_ac)
    {
        if ((pl->whole_word != 0) != P->whole_word) return false;
        if (pl->patterns.size() != P->num_patterns) return false;
        for (size_t k = 0; k < P->num_patterns; k++)
        {
            if (pl->pat_lens[k] != P->pattern_lens[k]) return false;
            if (P->pattern_lens[k] && memcmp(pl->patterns[k].data(), P->patterns[k], P->pattern_lens[k]) != 0) return false;
        }
        return true;
    }
    size_t m = algo == KREP_B200_ALGO_MEMCHR ? (P->pattern_len ? 1 : 0) : P->pattern_len;
    if (pl->m != m || memcmp(pl->pattern.data(), P->pattern, m) != 0) return false;
    if ((pl->whole_word != 0) != P->whole_word) return false;
    return pl->built_only_matching == only_matching;
}

static void cache_insert(Plan *pl)
{
    if (g_plan_cache.size() >= 16)
    {
        plan_free(g_plan_cache.front());
        g_plan_cache.erase(g_plan_cache.begin());
    }
    g_plan_cache.push_back(pl);
}

static Plan *cached_plan(const search_params_t *P, int algo, bool only_matching)
{
    for (size_t i = 0; i < g_plan_cache.size(); i++)
        if (plan_matches(g_plan_cache[i], P, algo, only_matching))
        {
            Plan *pl = g_plan_cache[i];
            g_plan_cache.erase(g_plan_cache.begin() + i);
            g_plan_cache.push_back(pl); // most recent last
            return pl;
        }
    Plan *pl = plan_build(P, algo, only_matching);
    if (pl) cache_insert(pl);
    return pl;
}

// Regexes the compiler refused (regex string, case flag, reason), most recent last.  Trying to split a large set can
// take seconds before it is refused, and krep asks once per file (search_file): the refusal is remembered.
struct RegexRefusal
{
    std::string regex;
    bool case_sensitive;
    std::string why;
};
static std::vector<RegexRefusal> g_regex_refusals;

// The regex plan of params (keyed by the regex string krep compiles and the case flag); nullptr and *why when the
// compiler refuses the pattern.  Host only: no device is touched until the plan runs.
static Plan *cached_regex_plan(const search_params_t *P, std::string *why)
{
    std::string re;
    if (!regex_source(P, &re))
    {
        *why = "no pattern";
        return nullptr;
    }
    for (const RegexRefusal &r : g_regex_refusals)
        if (r.case_sensitive == P->case_sensitive && r.regex == re)
        {
            *why = r.why;
            return nullptr;
        }
    for (size_t i = 0; i < g_plan_cache.size(); i++)
    {
        Plan *pl = g_plan_cache[i];
        if (pl->is_regex && pl->regex == re && pl->case_sensitive == P->case_sensitive)
        {
            g_plan_cache.erase(g_plan_cache.begin() + i);
            g_plan_cache.push_back(pl);
            return pl;
        }
    }
    Plan *pl = regex_plan_build(P, why);
    if (pl) cache_insert(pl);
    else if (MB_CUR_MAX == 1) // a refusal for the process locale may not hold after a setlocale
    {
        if (g_regex_refusals.size() >= 16) g_regex_refusals.erase(g_regex_refusals.begin());
        g_regex_refusals.push_back(RegexRefusal{re, P->case_sensitive, *why});
    }
    return pl;
}

// cached_regex_plan without the reason; nullptr for null params too
static Plan *regex_plan_of(const search_params_t *P)
{
    std::string why;
    return P ? cached_regex_plan(P, &why) : nullptr;
}

// The plan a -E call runs, or nullptr with the error set when the compiler refused the pattern.
static Plan *regex_plan_or_refuse(const search_params_t *P)
{
    std::string why;
    Plan *plan = cached_regex_plan(P, &why);
    if (!plan)
        set_error(-3, "this regex is not run on the GPU (%s); krep_b200_select_search_algorithm returns NULL for it", why.c_str());
    return plan;
}

void plan_cache_clear()
{
    g_regex_refusals.clear();
    for (Plan *p : g_plan_cache) plan_free(p);
    g_plan_cache.clear();
}

// AC-trie handles given to the host (krep_b200_ac_trie_build) own their plan: they are not part of the cache and live
// until krep_b200_ac_trie_free.  The magic word sits first so that a foreign pointer (the reference's own ac_trie_t,
// whose first word is a node pointer) can be told apart by reading 8 bytes.
struct TrieHandle
{
    uint64_t magic;
    Plan *plan;
};
static constexpr uint64_t TRIE_MAGIC = 0x6b7265705f747269ull; // "krep_tri"

// ---- staging: host text -> HBM, overlapped with the scan ----------------------------------------
#define CKH(call)                                                                                  \
    do                                                                                             \
    {                                                                                              \
        cudaError_t e_ = (call);                                                                   \
        if (e_ != cudaSuccess)                                                                     \
        {                                                                                          \
            set_error(-2, "CUDA error %s at %s:%d (%s)", cudaGetErrorName(e_), __FILE__, __LINE__, \
                      cudaGetErrorString(e_));                                                     \
            return -2;                                                                             \
        }                                                                                          \
    } while (0)

static size_t env_mb(const char *name, size_t dflt_mb)
{
    const char *v = getenv(name);
    if (!v || !*v) return dflt_mb << 20;
    long x = atol(v);
    return x > 0 ? (size_t)x << 20 : dflt_mb << 20;
}

// The caller's text streams through a small ring of device buffers (3 slots of one chunk + halo each) instead of
// being made resident as a whole: HBM use is bounded whatever the file size, nothing proportional to the text is
// allocated, and a slot is refilled as soon as the scan of its previous occupant has finished.
static int ensure_ring(DevCtx &E, size_t slot_bytes, int slots)
{
    slot_bytes = (slot_bytes + 255) & ~(size_t)255;
    if (E.ring_slot_bytes >= slot_bytes && E.ring_slots >= slots) return 0;
    CKH(cudaDeviceSynchronize());
    cudaFree(E.d_ring);
    E.d_ring = nullptr;
    E.ring_slot_bytes = 0;
    E.ring_slots = 0;
    cudaError_t e = cudaMalloc(&E.d_ring, slot_bytes * slots);
    if (e != cudaSuccess)
    {
        set_error(-2, "cannot allocate %zu bytes of HBM for the staging ring (%s)", slot_bytes * slots, cudaGetErrorString(e));
        return -2;
    }
    E.ring_slot_bytes = slot_bytes;
    E.ring_slots = slots;
    while ((int)E.ring_landed.size() < slots)
    {
        cudaEvent_t a, b;
        CKH(cudaEventCreateWithFlags(&a, cudaEventDisableTiming));
        CKH(cudaEventCreateWithFlags(&b, cudaEventDisableTiming));
        E.ring_landed.push_back(a);
        E.ring_scanned.push_back(b);
    }
    return 0;
}

static int ensure_stage(DevCtx &E, size_t bytes, int slots)
{
    if (E.stage_bytes >= bytes && (int)E.stage.size() >= slots) return 0;
    for (auto &s : E.stage)
    {
        cudaFreeHost(s.buf);
        if (s.ev) cudaEventDestroy(s.ev);
    }
    E.stage.clear();
    E.stage.resize(slots);
    for (auto &s : E.stage)
    {
        CKH(cudaMallocHost(&s.buf, bytes));
        CKH(cudaEventCreateWithFlags(&s.ev, cudaEventDisableTiming));
        s.in_flight = false;
    }
    E.stage_bytes = bytes;
    return 0;
}

static cudaEvent_t pool_event(DevCtx &E, size_t idx)
{
    while (E.ev_pool.size() <= idx)
    {
        cudaEvent_t ev;
        cudaEventCreate(&ev);
        E.ev_pool.push_back(ev);
    }
    return E.ev_pool[idx];
}

static int copy_threads()
{
    static int nt = 0;
    if (!nt)
    {
        const char *v = getenv("KREP_B200_COPY_THREADS");
        nt = v ? atoi(v) : 8; // host threads per device (8 saturate one PCIe link; many more oversubscribe it) that move the caller's (pageable) text into the pinned staging ring
        nt = std::max(1, std::min(nt, std::max(1, omp_get_num_procs())));
    }
    return nt;
}

// Pageable source (krep's file mapping, not pre-populated): populate the page tables of a piece in one batched call
// before copying it, instead of taking one minor fault per 4 KiB page inside memcpy.  MADV_POPULATE_READ (Linux 5.14);
// a kernel without it returns EINVAL and the copy simply faults its way through.
static inline void populate_piece(const uint8_t *src, size_t n)
{
#ifndef MADV_POPULATE_READ
#define MADV_POPULATE_READ 22
#endif
    static const bool on = !getenv("KREP_B200_NO_POPULATE_READ");
    if (!on) return;
    const uintptr_t a = (uintptr_t)src & ~(uintptr_t)4095, e = ((uintptr_t)src + n + 4095) & ~(uintptr_t)4095;
    (void)madvise((void *)a, e - a, MADV_POPULATE_READ);
}

static void parallel_copy(uint8_t *dst, const uint8_t *src, size_t n)
{
    const int nt = copy_threads();
    if (n < (8u << 20) || nt == 1)
    {
        populate_piece(src, n);
        memcpy(dst, src, n);
        return;
    }
    const size_t piece = (n / nt + 4095) & ~(size_t)4095;
#pragma omp parallel for num_threads(nt) schedule(static)
    for (int i = 0; i < nt; i++)
    {
        const size_t off = (size_t)i * piece;
        if (off < n)
        {
            populate_piece(src + off, std::min(piece, n - off));
            memcpy(dst + off, src + off, std::min(piece, n - off));
        }
    }
}

static bool is_pinned(const void *p)
{
    cudaPointerAttributes a;
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess)
    {
        cudaGetLastError();
        return false;
    }
    return a.type == cudaMemoryTypeHost;
}

// Called by the warm-up thread once the context exists: the buffers a search on pageable host text (krep's mmap) will
// ask for — device ring, pinned staging ring, occurrence list — are allocated while the host is still opening its file.
void prewarm_host_path(DevCtx &E)
{
    const size_t slot = env_mb("KREP_B200_STAGE_MB", 32) + 4096; // chunk + the longest possible halo (1025) + slack
    if (ensure_ring(E, slot, 3) != 0 || ensure_stage(E, slot, 3) != 0 || ensure_keys(E, 1) != 0) clear_error();
}

// One device's share of a search call: global bytes [begin, end) of the caller's text (end - begin a multiple of the
// chunk size except for the last device), streamed chunk by chunk — host (pinned directly, pageable through the pinned
// staging ring filled by host threads) -> copy stream -> ring slot -> scan stream — every chunk owning the starts in
// its own bytes and reading `halo` bytes of the next chunk (copied with it: the source is host memory, so overlapping
// reads cost nothing) and taking its -w context bytes straight from the host text.  All chunk scans of the device
// append to one occurrence list; k_finish / the radix sort order it.  If the list overflows, it is grown and the
// range is staged again.
// The text table of a packed -E batch (DESIGN §12.5), global offsets: text i is [start[i], end[i]), and seg[g] is the
// first text i with end[i] > g * REGEX_SEG (n_texts when there is none).
struct RegexBatch
{
    std::vector<uint64_t> start, end;
    std::vector<uint32_t> seg;
    const LongLineOpts *long_lines = nullptr; // the long-line pass after each chunk's scan (nullptr: none)
};

// Copies the table to the device (on its scan stream, behind the scans before it).
static int upload_regex_batch(DevCtx &E, const RegexBatch &B, RegexBatchDev *out)
{
    const size_t nt = B.end.size(), bytes = nt * 16 + B.seg.size() * 4;
    if (bytes > E.rx_batch_cap)
    {
        cudaFree(E.d_rx_batch);
        E.d_rx_batch = nullptr;
        E.rx_batch_cap = 0;
        CKH(cudaMalloc(&E.d_rx_batch, bytes + bytes / 4));
        E.rx_batch_cap = bytes + bytes / 4;
    }
    uint64_t *d = (uint64_t *)E.d_rx_batch;
    CKH(cudaMemcpyAsync(d, B.start.data(), nt * 8, cudaMemcpyHostToDevice, E.scan_stream));
    CKH(cudaMemcpyAsync(d + nt, B.end.data(), nt * 8, cudaMemcpyHostToDevice, E.scan_stream));
    CKH(cudaMemcpyAsync(d + 2 * nt, B.seg.data(), B.seg.size() * 4, cudaMemcpyHostToDevice, E.scan_stream));
    *out = RegexBatchDev{d, d + nt, (const uint32_t *)(d + 2 * nt), (uint32_t)nt};
    return 0;
}

struct RangeJob
{
    DevCtx *C = nullptr;
    const Plan *plan = nullptr;
    const char *text = nullptr;
    size_t n = 0, begin = 0, end = 0, chunk = 0;
    int want_positions = 0;
    bool pinned = false;
    bool count_lines = false; // fused -c of a literal or pattern-set plan: every chunk leaves one line record instead of keys
    std::vector<uint64_t> line_recs; // (lines, flags) per chunk, text order
    // -E: the scan's mode.  RX_COUNT: every chunk adds its device-decided matching lines and leaves its uncertain keys
    RegexMode regex_mode = RX_FILTER;
    uint64_t regex_lines = 0; // lines of the range decided MATCHED on the device
    const RegexBatch *batch = nullptr; // -E batch: the text is packed texts; RX_COUNT then counts per text
    const LongLineOpts *long_lines = nullptr; // -E: the long-line pass after each chunk's scan (DESIGN §12.8)
    std::vector<uint64_t> text_lines;  // batch, fused -c: lines of each text decided MATCHED in this range
    // results
    int rc = 0;
    ScanOut so;
    const uint64_t *h_keys = nullptr;
    std::vector<uint64_t> own_keys; // copy of the keys when the device's buffers are reused before the merge
    float kernel_ms = 0.f;
    ErrState err;
};

static int stream_range(RangeJob &J)
{
    DevCtx &E = *J.C;
    CKH(cudaSetDevice(E.device));
    const Plan *plan = J.plan;
    if (!plan_on_device(plan, E)) return -2;
    // occurrence + the byte after it (-w); regex: how far a line may run past its thread's segment (scan_regex.cu)
    const uint32_t halo = plan->is_regex ? REGEX_HALO : (plan->is_ac ? plan->max_len : plan->m) + 1;
    const size_t chunk = J.chunk, n = J.n;
    const size_t span = J.end - J.begin;
    const size_t nchunks = (span + chunk - 1) / chunk;
    const int nslots = nchunks >= 3 ? 3 : (int)std::max<size_t>(nchunks, 1);
    if (ensure_ring(E, std::min(chunk, span) + halo + 64, nslots) != 0) return -2;
    if (!J.pinned && ensure_stage(E, std::min(chunk, span) + halo + 64, nslots) != 0) return -2;
    if (J.want_positions && ensure_keys(E, 1) != 0) return -2;
    if (J.count_lines && ensure_line_out(E, nchunks) != 0) return -2;
    // the range's line counter: d_line_out[0] (a batch: one per text, d_line_out[0 .. n_texts))
    const size_t n_lines = J.batch ? J.batch->end.size() : 1;
    const bool regex_count = J.regex_mode == RX_COUNT;
    if (regex_count && ensure_line_out(E, (n_lines + 1) / 2) != 0) return -2;
    unsigned long long *d_regex_lines = regex_count ? (unsigned long long *)E.d_line_out : nullptr;
    RegexBatchDev batch_dev{};
    if (J.batch && upload_regex_batch(E, *J.batch, &batch_dev) != 0) return -2;
    reset_kernel_ms();
    const int slot = 0;
    // pattern-set -c: chunk c's scan is begun in list slot c % 2 before chunk c - 1 is ended (its record computed), so
    // the host's wait for c - 1's count overlaps chunk c's copy; a chunk's ring slot is free again once it is ended
    const bool set_count = J.count_lines && plan->is_ac;
    krep_b200_shard_t set_part[SCAN_SLOTS];
    auto set_end = [&](size_t c) -> int {
        const int s = (int)(c % SCAN_SLOTS);
        const int rc = set_count_end(E, plan, &set_part[s], E.scan_stream, s, c);
        if (rc != 0) return rc;
        CKH(cudaEventRecord(E.ring_scanned[c % E.ring_slots], E.scan_stream));
        return 0;
    };
    for (int attempt = 0; attempt < 3; attempt++)
    {
        CKH(cudaStreamWaitEvent(E.scan_stream, E.ev_done[slot], 0));
        if (!set_count && reset_counter(E, slot, E.scan_stream) != 0) return -2;
        if (d_regex_lines) CKH(cudaMemsetAsync(d_regex_lines, 0, n_lines * sizeof(unsigned long long), E.scan_stream)); // also on a re-stage
        for (size_t c = 0; c < nchunks; c++)
        {
            const size_t off = J.begin + c * chunk, len = std::min(chunk, J.end - off);
            const size_t src_len = std::min(len + halo, n - off);
            const int rs = (int)(c % E.ring_slots);
            uint8_t *d_slot = E.d_ring + (size_t)rs * E.ring_slot_bytes;
            if (c >= (size_t)E.ring_slots) CKH(cudaStreamWaitEvent(E.copy_stream, E.ring_scanned[rs], 0));
            if (J.pinned)
                CKH(cudaMemcpyAsync(d_slot, J.text + off, src_len, cudaMemcpyHostToDevice, E.copy_stream));
            else
            {
                StageSlot &s = E.stage[c % E.stage.size()];
                if (s.in_flight) CKH(cudaEventSynchronize(s.ev));
                parallel_copy(s.buf, (const uint8_t *)J.text + off, src_len);
                CKH(cudaMemcpyAsync(d_slot, s.buf, src_len, cudaMemcpyHostToDevice, E.copy_stream));
                CKH(cudaEventRecord(s.ev, E.copy_stream));
                s.in_flight = true;
            }
            CKH(cudaEventRecord(E.ring_landed[rs], E.copy_stream));
            CKH(cudaStreamWaitEvent(E.scan_stream, E.ring_landed[rs], 0));
            krep_b200_shard_t part;
            part.d_text = d_slot;
            part.avail_len = src_len;
            part.own_begin = 0;
            part.own_end = len;
            part.global_offset = off;
            part.prev_byte = off > 0 ? (int32_t)(uint8_t)J.text[off - 1] : -1;
            part.next_byte = off + src_len < n ? (int32_t)(uint8_t)J.text[off + src_len] : -1;
            cudaEvent_t a = pool_event(E, 2 * c), b = pool_event(E, 2 * c + 1);
            CKH(cudaEventRecord(a, E.scan_stream));
            int rc;
            if (set_count)
            {
                set_part[c % SCAN_SLOTS] = part;
                rc = set_count_begin(E, plan, &part, E.scan_stream, (int)(c % SCAN_SLOTS));
            }
            else
                rc = J.count_lines ? launch_count_lines(E, plan, &part, E.scan_stream, c)
                                   : launch_scan(E, plan, &part, J.want_positions, E.scan_stream, slot, d_regex_lines,
                                                 J.regex_mode == RX_OFFSETS, J.batch ? &batch_dev : nullptr, J.long_lines);
            if (rc != 0) return rc;
            CKH(cudaEventRecord(b, E.scan_stream));
            if (!set_count) CKH(cudaEventRecord(E.ring_scanned[rs], E.scan_stream));
            else if (c > 0 && (rc = set_end(c - 1)) != 0) return rc;
        }
        if (set_count)
        {
            const int rc = set_end(nchunks - 1);
            if (rc != 0) return rc;
        }
        CKH(cudaGetLastError());
        if (!J.count_lines && finish_scan(E, slot, J.want_positions, E.scan_stream) != 0) return -2;
        if (d_regex_lines)
            CKH(cudaMemcpyAsync(E.h_line_out, d_regex_lines, n_lines * sizeof(uint64_t), cudaMemcpyDeviceToHost, E.scan_stream));
        CKH(cudaStreamSynchronize(E.scan_stream));
        if (!J.count_lines) CKH(cudaEventSynchronize(E.ev_done[slot])); // k_finish runs on the finish stream
        for (auto &s : E.stage) s.in_flight = false;
        for (size_t c = 0; c < nchunks; c++)
        {
            float ms = 0.f;
            if (cudaEventElapsedTime(&ms, E.ev_pool[2 * c], E.ev_pool[2 * c + 1]) == cudaSuccess) add_kernel_ms(ms);
            else cudaGetLastError();
        }
        if (J.count_lines)
        {
            J.line_recs.assign(E.h_line_out, E.h_line_out + 2 * nchunks);
            J.so = ScanOut();
            return 0;
        }
        if (regex_count && J.batch) J.text_lines.assign(E.h_line_out, E.h_line_out + n_lines);
        else if (regex_count) J.regex_lines = E.h_line_out[0];
        const uint64_t cnt = E.h_pack[slot][0];
        J.so = ScanOut();
        J.so.count = cnt;
        J.so.device = E.device;
        J.so.serial = ++E.serial;
        E.result_stream = E.scan_stream;
        if (!J.want_positions) return 0;
        if (cnt <= E.key_cap)
        {
            J.so.stored = cnt;
            if (cnt <= PACK_KEYS)
            {
                J.so.d_keys = E.d_pack[slot] + 1;
                J.so.h_sorted = E.h_pack[slot] + 1;
                return 0;
            }
            return sort_keys(E, slot, cnt, key_end_bit(plan, n, J.regex_mode), E.scan_stream, &J.so.d_keys);
        }
        // list overflowed: grow it and stage the range again (the ring holds only the last chunks)
        J.so.overflow = 1;
        if (ensure_keys(E, cnt + cnt / 8 + 1024) != 0) return -2;
        reset_kernel_ms();
    }
    set_error(-4, "occurrence list kept overflowing");
    return -4;
}

// ---- which devices a host-text call uses --------------------------------------------------------
static std::vector<int> g_devices; // krep_b200_set_devices; empty = automatic

static std::vector<int> host_devices(size_t n)
{
    std::vector<int> out;
    const int vis = visible_devices();
    if (vis == 0) return out;
    if (!g_devices.empty())
    {
        for (int d : g_devices)
            if (d >= 0 && d < vis && std::find(out.begin(), out.end(), d) == out.end()) out.push_back(d);
        if (!out.empty()) return out;
    }
    const int prim = primary_device();
    if (prim < 0) return out;
    // default: ONE device.  From a pageable file mapping a second GPU adds little — the host side (page faults + staging
    // copies of one process) is the limit — and every further context costs start-up time.  KREP_B200_DEVICES=<k> (or
    // krep_b200_set_devices) spreads the call over k devices, which pays for pinned host text.
    int want = 1;
    const char *v = getenv("KREP_B200_DEVICES");
    if (v && *v && atoi(v) > 0) want = atoi(v);
    want = std::max(1, std::min(want, vis));
    out.push_back(prim);
    for (int d = 0; d < vis && (int)out.size() < want; d++)
        if (d != prim) out.push_back(d);
    return out;
}

// Result of one host-text search over all devices: total count, and (if wanted) the merged sorted key list on the host.
struct HostScan
{
    uint64_t count = 0;
    const uint64_t *keys = nullptr;
    uint64_t nkeys = 0;
    std::vector<uint64_t> merged; // backing store when several devices contributed
    uint64_t regex_lines = 0;     // fused -E -c: lines decided MATCHED on the devices (the keys are the uncertain lines)
    std::vector<uint64_t> text_lines; // the same per text of a batch
};

// count_lines: the fused -c of a literal or pattern-set plan, a line record per chunk.  regex_mode: the k_regex_lines
// mode of a regex plan (want_positions set): RX_COUNT leaves a device line count per range next to the keys of the
// uncertain lines, RX_OFFSETS match keys and uncertain-line keys.  batch: the text is a packed -E batch with this text
// table (DESIGN §12.5).
static int stage_and_scan(const Plan *plan, const char *text, size_t n, int want_positions, HostScan *hs, bool count_lines = false,
                          RegexMode regex_mode = RX_FILTER, const RegexBatch *batch = nullptr)
{
    const bool pinned = is_pinned(text);
    const size_t chunk = pinned ? env_mb("KREP_B200_CHUNK_MB", 256) : env_mb("KREP_B200_STAGE_MB", 32);
    std::vector<int> devs = host_devices(n);
    if (devs.empty())
    {
        set_error(-1, "no CUDA device available; this engine has no CPU fallback");
        return -1;
    }
    const size_t nchunks = std::max<size_t>((n + chunk - 1) / chunk, 1);
    if (devs.size() > nchunks) devs.resize(nchunks);
    const size_t D = devs.size();
    // one contiguous range of chunks per device; KREP_B200_RANGES=<k> cuts the text into more ranges than devices
    // (a device then takes its ranges one after the other) — used by the tests to drive the cross-range merge on one GPU
    size_t R = D;
    if (const char *v = getenv("KREP_B200_RANGES"))
        if (atoi(v) > 0) R = std::min<size_t>(std::max<size_t>((size_t)atoi(v), D), nchunks);
    std::vector<RangeJob> jobs(R);
    const size_t per = (nchunks + R - 1) / R; // chunks per range
    for (size_t i = 0; i < R; i++)
    {
        RangeJob &J = jobs[i];
        J.plan = plan;
        J.text = text;
        J.n = n;
        J.chunk = chunk;
        J.begin = std::min(i * per * chunk, n);
        J.end = std::min((i + 1) * per * chunk, n);
        J.want_positions = want_positions;
        J.pinned = pinned;
        J.count_lines = count_lines;
        J.regex_mode = regex_mode;
        J.batch = batch;
        J.long_lines = !plan->is_regex ? nullptr : batch ? batch->long_lines : long_lines_default();
    }
    trace("search: %zu bytes (%s host memory), %zu device(s), %zu range(s), chunk %zu MiB", n, pinned ? "pinned" : "pageable", D, R,
          chunk >> 20);
    // the ranges run on one host thread per device (on the calling thread when there is only one device); every thread
    // brings up its own device's context if it does not exist yet, so several contexts are created side by side
    auto run_device = [&jobs, &devs, D, R](size_t d) {
        for (size_t i = d; i < R; i += D)
        {
            RangeJob &J = jobs[i];
            J.C = ctx_get(devs[d]);
            if (!J.C)
            {
                J.rc = -1;
                break;
            }
            J.rc = J.begin < J.end ? stream_range(J) : 0;
            J.kernel_ms = get_kernel_ms();
            if (J.rc != 0) break;
            if (R > D && J.so.stored) // the device's buffers are reused by its next range: keep this range's keys
            {
                const uint64_t *k = nullptr;
                if ((J.rc = fetch_keys(*J.C, J.so, &k)) != 0) break;
                J.own_keys.assign(k, k + J.so.stored);
                J.h_keys = J.own_keys.data();
            }
        }
    };
    if (D == 1)
    {
        run_device(0);
        float ksum = 0.f;
        for (auto &J : jobs)
        {
            if (J.rc != 0) return J.rc;
            ksum += J.kernel_ms;
        }
        set_kernel_ms(ksum);
    }
    else
    {
        std::vector<std::thread> th;
        for (size_t d = 0; d < D; d++)
            th.emplace_back([&jobs, &run_device, d, D, R] {
                clear_error();
                run_device(d);
                for (size_t i = d; i < R; i += D) get_error(&jobs[i].err);
            });
        for (auto &t : th) t.join();
        std::vector<float> kdev(D, 0.f);
        for (size_t i = 0; i < R; i++)
        {
            if (jobs[i].rc != 0)
            {
                adopt_error(jobs[i].err);
                return jobs[i].rc;
            }
            kdev[i % D] += jobs[i].kernel_ms;
        }
        set_kernel_ms(*std::max_element(kdev.begin(), kdev.end())); // devices scan concurrently: the slowest one's time
    }
    trace("search: all ranges scanned (slowest device: %.2f ms of scan kernels)", get_kernel_ms());
    hs->count = 0;
    hs->keys = nullptr;
    hs->nkeys = 0;
    hs->regex_lines = 0;
    hs->text_lines.clear();
    if (batch && regex_mode == RX_COUNT)
    {
        // every line is decided by one range: the per-text counts add up
        hs->text_lines.assign(batch->end.size(), 0);
        for (auto &J : jobs)
            for (size_t i = 0; i < J.text_lines.size(); i++) hs->text_lines[i] += J.text_lines[i];
    }
    if (count_lines)
    {
        // chunk records of all ranges, in text order -> matching lines (a line cut by a chunk / range / device edge is
        // counted on both sides and subtracted once)
        std::vector<uint64_t> all;
        for (auto &J : jobs) all.insert(all.end(), J.line_recs.begin(), J.line_recs.end());
        hs->count = combine_line_records(all.data(), all.size() / 2);
        return 0;
    }
    for (auto &J : jobs)
    {
        hs->count += J.so.count;
        hs->regex_lines += J.regex_lines; // every line is decided by one range: the counts add up
    }
    if (!want_positions) return 0;
    for (auto &J : jobs)
    {
        if (J.so.stored == 0 || J.h_keys || !J.C) continue;
        cudaSetDevice(J.C->device);
        if (fetch_keys(*J.C, J.so, &J.h_keys) != 0) return -2;
    }
    if (R == 1)
    {
        hs->keys = jobs[0].h_keys;
        hs->nkeys = jobs[0].so.stored;
        return 0;
    }
    // ranges are in text order: literal and regex keys concatenate in order, pattern-set keys (ordered by end, owned by start) need
    // the merge around each cut
    std::vector<const uint64_t *> lists;
    std::vector<uint64_t> counts;
    uint64_t total = 0;
    for (auto &J : jobs)
    {
        lists.push_back(J.h_keys);
        counts.push_back(J.so.stored);
        total += J.so.stored;
    }
    hs->merged.resize(total);
    hs->nkeys = merge_key_lists(lists.data(), counts.data(), (uint32_t)lists.size(), hs->merged.data());
    hs->keys = hs->merged.data();
    trace("search: merged %llu keys from %zu ranges", (unsigned long long)hs->nkeys, R);
    return 0;
}

// Does the emulated kernel keep every (whole-word-valid) occurrence?  If so a bare count is enough.
static bool keeps_all(int algo, bool only_matching, const search_params_t *P, const Plan *pl)
{
    if (pl->is_ac) return true;
    if (pl->emit_len != pl->m) return false;
    // window kernels: tail sub-search, AVX-512's skipped windows and the -m re-basing all need the list
    if (algo == KREP_B200_ALGO_AVX2 || algo == KREP_B200_ALGO_AVX512 || algo == KREP_B200_ALGO_NEON) return false;
    if (pl->border_free) return true; // occurrences cannot overlap: every overlap policy keeps all
    switch (algo)
    {
    case KREP_B200_ALGO_BMH: return !(only_matching && !P->count_lines_mode);
    case KREP_B200_ALGO_MEMCHR: return true;
    case KREP_B200_ALGO_MEMCHR_SHORT: return !only_matching;
    case KREP_B200_ALGO_SSE42: return only_matching;
    default: return false;
    }
}

// Return value of the emulated kernel when all `total` occurrences are kept and only the -m limit acts.
static uint64_t limited_count(int algo, const search_params_t *P, uint64_t total)
{
    const uint64_t maxc = P->max_count;
    switch (algo)
    {
    case KREP_B200_ALGO_BMH:
    case KREP_B200_ALGO_MEMCHR_SHORT:
        // count first, test afterwards (krep.c:1355-1367): with -m 0 in a pure count mode one match still counts
        if (total == 0) return 0;
        return maxc == 0 ? 1 : std::min<uint64_t>(total, maxc);
    default:
        return std::min<uint64_t>(total, maxc);
    }
}

// The early returns every reference kernel takes before it looks at the text.  Returns true when the call is already
// answered (*ret); otherwise *algo is the kernel whose policy applies (precondition fallbacks resolved).
static bool early_answer(int entry_algo, const search_params_t *P, const char *text, size_t n, match_result_t *res, int *algo_out,
                         uint64_t *ret)
{
    *ret = 0;
    int algo = entry_algo;
    size_t m = 0;
    if (algo == KREP_B200_ALGO_AC)
    {
        if (!P->ac_trie || !text) return true;  // aho_corasick.c:306
        if (P->max_count == 0) return true;     // aho_corasick.c:316
        if (n == 0)                             // aho_corasick.c:442-463
        {
            for (size_t k = 0; k < P->num_patterns; k++)
                if (P->pattern_lens[k] == 0)
                {
                    if (P->track_positions && res) result_push(res, 0, 0);
                    *ret = 1;
                    return true;
                }
            return true;
        }
    }
    else
    {
        algo = resolve_algo(P, algo);
        m = P->pattern_len;
        switch (algo)
        {
        case KREP_B200_ALGO_KMP:
            if (P->max_count == 0) return true;
            if (m == 0 || n < m) return true;
            break;
        case KREP_B200_ALGO_MEMCHR:
            if (P->max_count == 0 || n == 0) return true;
            m = 1;
            break;
        case KREP_B200_ALGO_MEMCHR_SHORT:
            if (P->max_count == 0 && (P->count_lines_mode || P->track_positions)) return true;
            if (m < 2 || m > 3 || n < m) return true;
            break;
        default: // BMH, SSE42, the long simd entries, NEON
            if (P->max_count == 0 && (P->count_lines_mode || P->track_positions)) return true;
            if (m == 0 || n < m) return true;
            break;
        }
        if (!P->pattern) return true;
        if (m > 1024)
        {
            set_error(-3, "pattern longer than 1024 bytes (MAX_PATTERN_LENGTH, krep.c:77)");
            return true;
        }
    }
    *algo_out = algo;
    return false;
}

// The plan a call runs: the host's own trie handle when it was built by krep_b200_ac_trie_build for these very
// patterns, else the cache.
static Plan *plan_for(const search_params_t *P, int algo, bool only_matching)
{
    if (algo == KREP_B200_ALGO_AC && P->ac_trie)
    {
        const TrieHandle *h = reinterpret_cast<const TrieHandle *>(P->ac_trie);
        if (h->magic == TRIE_MAGIC && h->plan && plan_matches(h->plan, P, algo, only_matching)) return h->plan;
    }
    return cached_plan(P, algo, only_matching);
}

static uint64_t run_search(int entry_algo, const search_params_t *P, const char *text, size_t n, match_result_t *res)
{
    std::lock_guard<std::recursive_mutex> lk(engine_mutex());
    clear_error();
    if (!P) return 0;
    const bool only_matching = g_only_matching;
    int algo = entry_algo;
    uint64_t early = 0;
    if (early_answer(entry_algo, P, text, n, res, &algo, &early)) return early;
    if (warm_running())
    {
        // the context is still being created on the warm-up thread: meanwhile fault the caller's pages in (a file the
        // host mapped without MAP_POPULATE) with the staging threads, so that the copy loop later runs at link speed
        // (opt-in: faulting pages in the same process while cuInit / context creation run slows both down — they
        // fight over the address-space lock)
        if (n >= (64u << 20) && getenv("KREP_B200_PREFAULT"))
        {
            trace("search: pre-faulting %zu bytes while the context comes up", n);
            const long pages = (long)((n + 4095) / 4096);
            unsigned long sink = 0;
#pragma omp parallel for num_threads(copy_threads()) schedule(static) reduction(+ : sink)
            for (long pg = 0; pg < pages; pg++) sink += (unsigned char)text[(size_t)pg * 4096];
            if (sink == 0x5EED5EED5EEDull) trace("(unlikely checksum)");
        }
        warm_join();
        trace("search: context ready");
    }
    if (visible_devices() == 0)
    {
        set_error(-1, "no CUDA device available; this engine has no CPU fallback");
        return 0;
    }
    DeviceGuard guard;
    Plan *plan = plan_for(P, algo, only_matching);
    if (!plan) return 0;
    const bool want_result = P->track_positions && res;
    const bool need_list = P->count_lines_mode || want_result || !keeps_all(algo, only_matching, P, plan) ||
                           plan->whole_word == 2;
    HostScan hs;
    if (count_lines_eligible(plan, P, algo) && !getenv("KREP_B200_NO_FUSED_COUNT"))
    {
        // -c: the scan counts matching lines itself; the -m limit caps the count (every kernel stops at max_count lines,
        // max_count == 0 was answered above)
        if (stage_and_scan(plan, text, n, 0, &hs, true) != 0) return 0;
        return std::min<uint64_t>(hs.count, P->max_count);
    }
    if (stage_and_scan(plan, text, n, need_list ? 1 : 0, &hs) != 0) return 0;
    if (!need_list) return limited_count(algo, P, hs.count);
    Replay r{hs.keys, (size_t)hs.nkeys, text, n, 0};
    const uint64_t ret = plan->is_ac ? replay_ac(P, r, res) : replay_literal(algo, P, only_matching, plan->m, r, res);
    trace("search: replay done (%llu)", (unsigned long long)ret);
    return ret;
}

// Can a -E call with these params count its lines on the device?  -c without -w (count_lines_mode, not -co) on a plan
// whose per-line answer is glibc's.  KREP_B200_NO_FUSED_COUNT is not looked at here.
static bool regex_count_exact(const search_params_t *P, const Plan *plan)
{
    return P->count_lines_mode && !P->whole_word && plan->rx->count_exact;
}

static bool regex_count_fused(const search_params_t *P, const Plan *plan)
{
    return regex_count_exact(P, plan) && !getenv("KREP_B200_NO_FUSED_COUNT");
}

// Can a -E call with these params compute its match offsets on the device?  Positions or -co (track_positions without
// count_lines_mode), no -w, on a plan whose match automaton is exact and fits (offsets_exact).
// KREP_B200_NO_DEVICE_MATCHES is not looked at here.
static bool regex_matches_exact(const search_params_t *P, const Plan *plan)
{
    return P->track_positions && !P->count_lines_mode && !P->whole_word && plan->rx->offsets_exact;
}

static bool regex_matches_device(const search_params_t *P, const Plan *plan)
{
    return regex_matches_exact(P, plan) && !getenv("KREP_B200_NO_DEVICE_MATCHES");
}

// The k_regex_lines mode a -E call with these params takes.
static RegexMode regex_call_mode(const search_params_t *P, const Plan *plan)
{
    return regex_count_fused(P, plan) ? RX_COUNT : regex_matches_device(P, plan) ? RX_OFFSETS : RX_FILTER;
}

// -E (regex_search, krep.c:1389): the device flags the lines the regex can match in (k_regex_lines), glibc's regexec
// on the caller's regex_t confirms them and computes every offset (replay_regex).  A -c call on a count_exact plan
// counts the lines the device can decide there and leaves glibc only the uncertain ones.  A positions or -co call on an
// offsets_exact plan takes the offsets of the lines the device decides from the device and leaves glibc only the
// uncertain ones (DESIGN §12.2).  regex_answer turns each mode's keys into the answer.  The empty text is answered on
// the host, as the reference does, without a launch.
static uint64_t run_regex(const search_params_t *P, const char *text, size_t n, match_result_t *res)
{
    std::lock_guard<std::recursive_mutex> lk(engine_mutex());
    clear_error();
    if (!P || regex_returns_early(P)) return 0;
    if (n == 0) return regex_empty_text(P, res);
    if (!text) return 0;
    warm_join();
    if (visible_devices() == 0)
    {
        set_error(-1, "no CUDA device available; this engine has no CPU fallback");
        return 0;
    }
    DeviceGuard guard;
    Plan *plan = regex_plan_or_refuse(P);
    if (!plan) return 0;
    const RegexMode mode = regex_call_mode(P, plan);
    HostScan hs;
    if (stage_and_scan(plan, text, n, 1, &hs, false, mode) != 0) return 0;
    const uint64_t ret = regex_answer(P, mode, hs.regex_lines, Replay{hs.keys, (size_t)hs.nkeys, text, n, 0}, res);
    trace("search: regex mode %d: %llu keys to regexec or offsets, %llu lines counted on the device (%llu)", mode,
          (unsigned long long)hs.nkeys, (unsigned long long)hs.regex_lines, (unsigned long long)ret);
    return ret;
}

// ---- -E on resident shards (DESIGN §12.4): a row per shard, resolved on the host ----
static thread_local RegexPackStats t_rx_stats; // of the most recent krep_b200_search_shards / _regex_export_shard call

// Scan + pack of one shard: the row is left in the engine's memory of the shard's device.
static int regex_export(const Plan *plan, const search_params_t *P, const krep_b200_shard_t *sh, const char *who, DevCtx **ctx,
                        const void **d_row, uint64_t *row_bytes)
{
    if (!plan->is_regex)
    {
        set_error(-3, "%s: not a regex plan", who);
        return -3;
    }
    DevCtx *C = ctx_of_pointer(sh->d_text);
    if (!C) return -1;
    cudaSetDevice(C->device);
    const RegexMode mode = regex_call_mode(P, plan);
    uint64_t cnt = 0, lines = 0;
    const uint64_t *d_sorted = nullptr;
    CKH(cudaEventRecord(C->ev_ca, C->scan_stream));
    int rc = regex_scan_keys(*C, plan, sh, mode, who, &cnt, &d_sorted, &lines, long_lines_default());
    if (rc != 0) return rc;
    CKH(cudaEventRecord(C->ev_cb, C->scan_stream));
    float pack_ms = 0.f, scan_ms = 0.f;
    rc = regex_pack_row(*C, sh, mode, d_sorted, cnt, lines, d_row, row_bytes, &pack_ms);
    if (rc != 0) return rc;
    cudaEventElapsedTime(&scan_ms, C->ev_ca, C->ev_cb);
    t_rx_stats.scan_ms += scan_ms;
    t_rx_stats.pack_ms += pack_ms;
    t_rx_stats.packed_bytes += *row_bytes;
    trace("regex row: mode %d, %llu keys, %llu bytes (scan %.3f ms, pack %.3f ms)", mode, (unsigned long long)cnt,
          (unsigned long long)*row_bytes, scan_ms, pack_ms);
    *ctx = C;
    return 0;
}

// The shards of a -E search must tile one whole text: owned ranges that abut from offset 0 to the text's end.
static bool regex_tiling_ok(const krep_b200_shard_t *s, uint32_t n)
{
    if (n == 0 || !s) return false;
    if (s[0].global_offset + s[0].own_begin != 0 || s[0].prev_byte != -1) return false;
    for (uint32_t i = 0; i < n; i++)
    {
        if (s[i].own_begin > s[i].own_end || s[i].own_end > s[i].avail_len) return false;
        if (i && s[i - 1].global_offset + s[i - 1].own_end != s[i].global_offset + s[i].own_begin) return false;
    }
    return s[n - 1].next_byte == -1 && s[n - 1].own_end == s[n - 1].avail_len;
}

// krep_b200_search_shards for a regex plan: krep_b200_regex_search's answer on the text the shards tile, from one row per
// shard (scanned and packed on the shard's device, read back in one copy) resolved by regex_resolve_rows.
static uint64_t search_shards_regex(const Plan *plan, const search_params_t *P, const krep_b200_shard_t *shards, uint32_t n_shards,
                                    match_result_t *res)
{
    t_rx_stats = RegexPackStats();
    if (!regex_tiling_ok(shards, n_shards))
    {
        set_error(-3, "krep_b200_search_shards: the shards of a regex search must tile one text: the first owns from global "
                      "offset 0 with prev_byte -1, owned ranges abut, the last has next_byte -1 and own_end == avail_len");
        return 0;
    }
    if (regex_returns_early(P)) return 0;
    const krep_b200_shard_t &last = shards[n_shards - 1];
    if (last.global_offset + last.avail_len == 0) return regex_empty_text(P, res);
    DeviceGuard guard;
    std::vector<std::vector<uint8_t>> copies(n_shards > 1 ? n_shards : 0);
    std::vector<const void *> rows(n_shards);
    for (uint32_t i = 0; i < n_shards; i++)
    {
        DevCtx *C = nullptr;
        const void *d_row = nullptr;
        uint64_t bytes = 0;
        if (regex_export(plan, P, &shards[i], "krep_b200_search_shards", &C, &d_row, &bytes) != 0) return 0;
        uint8_t *h = regex_pack_host_buffer(*C, bytes);
        if (!h) return 0;
        if (cudaMemcpyAsync(h, d_row, bytes, cudaMemcpyDeviceToHost, C->scan_stream) != cudaSuccess ||
            cudaStreamSynchronize(C->scan_stream) != cudaSuccess)
        {
            set_error(-2, "reading a regex row back failed (%s)", cudaGetErrorString(cudaGetLastError()));
            return 0;
        }
        if (n_shards == 1) rows[i] = h; // the pinned buffer is the next row's too: keep a copy when there is one
        else
        {
            copies[i].assign(h, h + bytes);
            rows[i] = copies[i].data();
        }
    }
    int err = 0;
    const uint64_t ret = regex_resolve_rows(P, rows.data(), n_shards, res, &err);
    trace("search_shards: regex over %u shards, %llu row bytes (%llu)", n_shards, (unsigned long long)t_rx_stats.packed_bytes,
          (unsigned long long)ret);
    return err ? 0 : ret;
}

// The packed layout of a batch: text f (f in `live`, in that order) at the 16-byte aligned (*off)[f], followed by at
// least `gap` bytes up to the next text's offset or the returned total.  The host pack (pack_texts) and the device
// gather of resident batches (k_batch_gather) both place the texts by it.
static uint64_t pack_layout(const size_t *lens, const std::vector<size_t> &live, size_t gap, std::vector<uint64_t> *off)
{
    uint64_t t = 0;
    for (size_t f : live)
    {
        (*off)[f] = t;
        t = (t + lens[f] + gap + 15) & ~15ull;
    }
    return t;
}

// Packs texts[f] for f in `live` (ascending) into the device's pinned batch buffer with the staging threads, placed by
// pack_layout, with `fill` in the gaps.
static int pack_texts(DevCtx &E, const char *const *texts, const size_t *lens, const std::vector<size_t> &live, size_t gap,
                      uint8_t fill, std::vector<uint64_t> *off, uint64_t *total)
{
    const uint64_t t = pack_layout(lens, live, gap, off);
    *total = t;
    if (t > E.h_batch_cap)
    {
        cudaFreeHost(E.h_batch);
        E.h_batch = nullptr;
        E.h_batch_cap = 0;
        CKH(cudaMallocHost(&E.h_batch, t + t / 4 + 4096));
        E.h_batch_cap = t + t / 4 + 4096;
    }
    // only the gaps are filled
    const long nl = (long)live.size();
    uint8_t *const hb = E.h_batch;
    const uint64_t *o = off->data();
#pragma omp parallel for num_threads(copy_threads()) schedule(dynamic, 16)
    for (long i = 0; i < nl; i++)
    {
        const size_t f = live[(size_t)i];
        const uint64_t end = o[f] + lens[f], next = i + 1 < nl ? o[live[(size_t)i + 1]] : t;
        memcpy(hb + o[f], texts[f], lens[f]);
        memset(hb + end, fill, next - end);
    }
    return 0;
}

// The early returns of a literal / pattern-set batch, text by text: counts[f] gets each early answer, algo_of[f] the
// kernel of every other text.  text_of(f) stands for text f (only whether it is null is read).  Returns that kernel (the
// resolved kernel depends on params only, except for the n < m early return), or -1 when every text was answered.
template <class TextOf>
static int batch_early_answers(int entry_algo, const search_params_t *P, size_t nt, const size_t *lens, TextOf text_of,
                               uint64_t *counts, match_result_t *const *results, std::vector<int> *algo_of)
{
    algo_of->assign(nt, -1);
    int algo = -1;
    for (size_t f = 0; f < nt; f++)
    {
        int a = entry_algo;
        uint64_t early = 0;
        counts[f] = 0;
        if (early_answer(entry_algo, P, text_of(f), lens[f], results ? results[f] : nullptr, &a, &early)) counts[f] = early;
        else (*algo_of)[f] = algo = a;
    }
    return algo;
}

// Cuts the sorted key list of a packed literal / pattern-set batch per text — an occurrence belongs to a text only if
// it lies wholly inside it — and replays each cut exactly as a separate call would have been (same early returns, own -m
// limit, own line context), with Replay::base = the text's packed offset off[f].  texts: the host texts; nullptr
// replays from the keys alone, as resident shards do, with -c taking `bounds` (two line bounds per key, in key order).
static void replay_batch_cuts(const Plan *plan, int algo, const search_params_t *P, bool only_matching, const uint64_t *keys,
                              uint64_t nkeys, const uint64_t *bounds, size_t gap, const std::vector<int> &algo_of,
                              const std::vector<uint64_t> &off, const char *const *texts, const size_t *lens, uint64_t *counts,
                              match_result_t *const *results)
{
    // texts are in ascending offset order; keys ascend by start, or by end for pattern sets
    std::vector<uint64_t> mine, mine_bounds;
    size_t j = 0;
    for (size_t f = 0; f < algo_of.size(); f++)
    {
        if (algo_of[f] < 0) continue;
        const uint64_t lo = off[f], hi = off[f] + lens[f];
        mine.clear();
        mine_bounds.clear();
        while (j < nkeys)
        {
            uint64_t s, e;
            if (plan->is_ac)
            {
                e = keys[j] >> AC_END_SHIFT;
                s = e - (1024 - ((keys[j] >> AC_LEN_SHIFT) & 1023));
            }
            else
            {
                s = keys[j] >> LIT_TAG_BITS;
                e = s + ((keys[j] >> 2) & 1 ? plan->m : plan->emit_len);
            }
            const uint64_t ord = plan->is_ac ? e : s; // the coordinate the list is sorted by
            if (ord >= hi + (plan->is_ac ? gap : 0)) break; // belongs to a later text
            if (s >= lo && e <= hi)
            {
                mine.push_back(keys[j]);
                if (bounds)
                {
                    mine_bounds.push_back(bounds[2 * j]);
                    mine_bounds.push_back(bounds[2 * j + 1]);
                }
            }
            j++;
        }
        Replay r{mine.data(), mine.size(), texts ? texts[f] : nullptr, lens[f], lo, bounds ? mine_bounds.data() : nullptr};
        match_result_t *res = results ? results[f] : nullptr;
        counts[f] = plan->is_ac ? replay_ac(P, r, res) : replay_literal(algo, P, only_matching, plan->m, r, res);
    }
}

// Many texts, one launch (SURVEY §8 f4: small files lose to launch and copy latency one by one).  The texts are packed
// into one pinned buffer at 16-byte aligned offsets, separated by zero gaps longer than the longest pattern, copied and
// scanned as ONE shard; the sorted occurrence list is then cut per text and replayed (replay_batch_cuts).  A gap byte is
// 0, i.e. not a word character: -w sees a text boundary there, as it should.
static int run_batch(int entry_algo, const search_params_t *P, const char *const *texts, const size_t *lens, size_t nt,
                     uint64_t *counts, match_result_t *const *results)
{
    warm_join();
    std::lock_guard<std::recursive_mutex> lk(engine_mutex());
    clear_error();
    if (!P || !texts || !lens || !counts)
    {
        set_error(-3, "krep_b200_search_batch: null argument");
        return -3;
    }
    const bool only_matching = g_only_matching;
    std::vector<int> algo_of;
    const int algo = batch_early_answers(entry_algo, P, nt, lens, [&](size_t f) { return texts[f]; }, counts, results, &algo_of);
    if (krep_b200_last_error() != 0) return -3;
    if (algo < 0) return 0; // every text was answered by an early return
    DeviceGuard guard;
    DevCtx *Cp = ctx_primary();
    if (!Cp) return -1;
    Plan *plan = plan_for(P, algo, only_matching);
    if (!plan) return -2;
    const size_t gap = (size_t)(plan->is_ac ? plan->max_len : plan->m) + 16;
    std::vector<size_t> live;
    for (size_t f = 0; f < nt; f++)
        if (algo_of[f] >= 0) live.push_back(f);
    std::vector<uint64_t> off(nt, 0);
    uint64_t total = 0;
    DevCtx &E = *Cp;
    if (pack_texts(E, texts, lens, live, gap, 0, &off, &total) != 0) return -2;
    HostScan hs;
    if (stage_and_scan(plan, (const char *)E.h_batch, total, 1, &hs) != 0) return -2;
    replay_batch_cuts(plan, algo, P, only_matching, hs.keys, hs.nkeys, nullptr, gap, algo_of, off, texts, lens, counts, results);
    return 0;
}

// ---- -E over many texts (DESIGN §12.5) ----
struct RegexBatchTimes
{
    double pack_ms = 0, resolve_ms = 0; // host clock: packing (with the text table), and the per-text replays
};
static thread_local RegexBatchTimes t_rx_batch; // of the most recent krep_b200_regex_search_batch call

static double ms_since(std::chrono::steady_clock::time_point t0)
{
    return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
}

// The text table of the texts f in `live` (ascending, lens[f] > 0) packed at off[f] into `total` bytes; seg[g]: the first
// text that ends after g * REGEX_SEG.
static void regex_batch_table(const size_t *lens, const std::vector<size_t> &live, const std::vector<uint64_t> &off, uint64_t total,
                              RegexBatch *B)
{
    const size_t nl = live.size();
    B->start.resize(nl);
    B->end.resize(nl);
    for (size_t i = 0; i < nl; i++)
    {
        B->start[i] = off[live[i]];
        B->end[i] = B->start[i] + lens[live[i]];
    }
    B->seg.resize((total + REGEX_SEG - 1) / REGEX_SEG);
    for (size_t g = 0, i = 0; g < B->seg.size(); g++)
    {
        while (i < nl && B->end[i] <= (uint64_t)g * REGEX_SEG) i++;
        B->seg[g] = (uint32_t)i;
    }
}

// One k_regex_lines scan in `mode` of the texts f in `live` (ascending, lens[f] > 0): packed with '\n' gaps (at least
// one '\n' after each text, up to the next 16-byte boundary), so that no line and no automaton walk crosses from one
// text into the next, and scanned by stage_and_scan as one text in the kernel's batch mode.  *off (indexed by f):
// packed offsets; *hs: the sorted keys in packed coordinates and, in RX_COUNT, the device line count of each live text
// (indexed like `live`).  long_lines: the long-line pass after each chunk's scan, in the batch
// rules (DESIGN §12.8); nullptr leaves every line past the kernel's reach uncertain.
static int regex_batch_scan(const Plan *plan, const char *const *texts, const size_t *lens, const std::vector<size_t> &live,
                            RegexMode mode, const LongLineOpts *long_lines, const char *who, std::vector<uint64_t> *off, HostScan *hs)
{
    if (live.size() >= UINT32_MAX)
    {
        set_error(-3, "%s: too many texts in one call", who);
        return -3;
    }
    DevCtx *Cp = ctx_primary();
    if (!Cp) return -1;
    const auto t0 = std::chrono::steady_clock::now();
    uint64_t total = 0;
    if (pack_texts(*Cp, texts, lens, live, 1, '\n', off, &total) != 0) return -2;
    RegexBatch B;
    B.long_lines = long_lines;
    regex_batch_table(lens, live, *off, total, &B);
    t_rx_batch.pack_ms += ms_since(t0);
    trace("regex batch: %zu texts packed into %llu bytes", live.size(), (unsigned long long)total);
    return stage_and_scan(plan, (const char *)Cp->h_batch, total, 1, hs, false, mode, &B);
}

// krep_b200_regex_search_batch: text i gets krep_b200_regex_search(P, texts[i], lens[i], results[i])'s answer.  The
// early returns are answered on the host; the other texts take one batch scan in the mode regex_call_mode picks for P,
// and each text is then replayed on its own bytes with its own keys (Replay::base = its packed offset): its own -m
// budget, its own last line and end-of-text quirks (the kernel leaves each text's last line uncertain).
static int run_regex_batch(const search_params_t *P, const char *const *texts, const size_t *lens, size_t nt, uint64_t *counts,
                           match_result_t *const *results)
{
    warm_join();
    std::lock_guard<std::recursive_mutex> lk(engine_mutex());
    clear_error();
    t_rx_batch = RegexBatchTimes();
    if (!P || (nt && (!texts || !lens || !counts)))
    {
        set_error(-3, "krep_b200_regex_search_batch: null argument");
        return -3;
    }
    for (size_t f = 0; f < nt; f++) counts[f] = 0;
    if (regex_returns_early(P)) return 0;
    std::vector<size_t> live;
    for (size_t f = 0; f < nt; f++)
        if (lens[f] > 0 && texts[f]) live.push_back(f);
    DeviceGuard guard;
    if (!live.empty())
    {
        if (visible_devices() == 0)
        {
            set_error(-1, "no CUDA device available; this engine has no CPU fallback");
            return -1;
        }
        Plan *plan = regex_plan_or_refuse(P);
        if (!plan) return -3;
        const RegexMode mode = regex_call_mode(P, plan);
        std::vector<uint64_t> off(nt, 0);
        HostScan hs;
        const int rc = regex_batch_scan(plan, texts, lens, live, mode, long_lines_default(), "krep_b200_regex_search_batch", &off, &hs);
        if (rc != 0) return rc;
        const auto t0 = std::chrono::steady_clock::now();
        // keys ascend in packed coordinates: one pass cuts them per text (nothing outside a text is kept)
        const int shift = regex_key_shift(mode);
        size_t j = 0;
        for (size_t i = 0; i < live.size(); i++)
        {
            const size_t f = live[i];
            const uint64_t lo = off[f], hi = off[f] + lens[f];
            while (j < hs.nkeys && (hs.keys[j] >> shift) < lo) j++;
            size_t k = j;
            while (k < hs.nkeys && (hs.keys[k] >> shift) < hi) k++;
            const Replay r{hs.keys + j, k - j, texts[f], lens[f], lo};
            counts[f] = regex_answer(P, mode, mode == RX_COUNT ? hs.text_lines[i] : 0, r, results ? results[f] : nullptr);
            j = k;
        }
        t_rx_batch.resolve_ms = ms_since(t0);
        trace("regex batch: mode %d, %zu texts, %llu keys (resolved in %.3f ms)", mode, live.size(), (unsigned long long)hs.nkeys,
              t_rx_batch.resolve_ms);
    }
    for (size_t f = 0; f < nt; f++)
        if (lens[f] == 0) counts[f] = regex_empty_text(P, results ? results[f] : nullptr);
    return 0;
}

// ---- many HBM-resident texts in one call (DESIGN §12.9) ----
struct ResidentTimes
{
    float gather_ms = 0.f, scan_ms = 0.f; // device time: k_batch_gather; the scan with its sort (and, -E, the row pack)
    double resolve_ms = 0;                // host clock: the per-text replays
};
static thread_local ResidentTimes t_resident; // of the most recent resident batch call

// The engine of the device that holds d_base, or nullptr with the error set: -3 when d_base is not device memory or
// the bytes from the lowest text start to the highest text end are not all mapped device memory.  The check walks
// the driver's cuMemGetAddressRange from the lowest start: a cudaMalloc allocation answers in one step, memory mapped
// in several chunks (virtual memory management, such as torch's expandable segments) in one step per chunk, and an
// unmapped hole refuses the call.  Without the driver entry point only d_base itself is checked.
static DevCtx *resident_ctx(const char *who, const void *d_base, const uint64_t *offsets, const size_t *lens, size_t nt)
{
    cudaPointerAttributes a;
    if (!d_base || cudaPointerGetAttributes(&a, d_base) != cudaSuccess || a.type != cudaMemoryTypeDevice)
    {
        cudaGetLastError();
        set_error(-3, "%s: d_base is not device memory", who);
        return nullptr;
    }
    uint64_t lo = UINT64_MAX, hi = 0;
    for (size_t f = 0; f < nt; f++)
        if (lens[f])
        {
            if (offsets[f] > UINT64_MAX - lens[f] || offsets[f] + lens[f] > UINT64_MAX - (uintptr_t)d_base)
            {
                set_error(-3, "%s: text %zu ends past the address space", who, f);
                return nullptr;
            }
            lo = std::min<uint64_t>(lo, offsets[f]);
            hi = std::max<uint64_t>(hi, offsets[f] + lens[f]);
        }
    if (hi > lo)
    {
        typedef int (*AddressRange)(unsigned long long *base, size_t *size, unsigned long long ptr);
        static AddressRange range = [] {
            void *fn = nullptr;
            cudaDriverEntryPointQueryResult q;
            if (cudaGetDriverEntryPoint("cuMemGetAddressRange", &fn, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess)
            {
                cudaGetLastError();
                fn = nullptr;
            }
            return (AddressRange)fn;
        }();
        const unsigned long long end = (unsigned long long)(uintptr_t)d_base + hi;
        unsigned long long p = (unsigned long long)(uintptr_t)d_base + lo;
        while (range && p < end)
        {
            unsigned long long ab = 0;
            size_t as = 0;
            cudaPointerAttributes pa;
            const bool mapped = range(&ab, &as, p) == 0 && as > 0 && ab + as > p &&
                                cudaPointerGetAttributes(&pa, (const void *)(uintptr_t)p) == cudaSuccess &&
                                pa.type == cudaMemoryTypeDevice && pa.device == a.device;
            if (!mapped)
            {
                cudaGetLastError();
                set_error(-3, "%s: the texts are not all in device memory of device %d (byte %llu from d_base is not)", who,
                          a.device, (unsigned long long)(p - (uintptr_t)d_base));
                return nullptr;
            }
            p = ab + as;
        }
    }
    DevCtx *C = ctx_get(a.device);
    if (C) cudaSetDevice(C->device);
    return C;
}

// Packs the texts f in `live` (in that order) from d_base into E.d_gather on the device, placed by pack_layout with
// `fill` in the gaps, as pack_texts packs host texts.  last: each text's last byte, indexed like live.
static int gather_resident(DevCtx &E, const char *who, const void *d_base, const uint64_t *offsets, const size_t *lens,
                           const std::vector<size_t> &live, size_t gap, uint8_t fill, std::vector<uint64_t> *off, uint64_t *total,
                           std::vector<uint8_t> *last)
{
    *total = pack_layout(lens, live, gap, off);
    const size_t nl = live.size();
    if (*total > E.gather_cap)
    {
        CKH(cudaStreamSynchronize(E.scan_stream));
        cudaFree(E.d_gather);
        E.d_gather = nullptr;
        E.gather_cap = 0;
        const uint64_t want = *total + *total / 8 + 4096;
        cudaError_t e = cudaMalloc(&E.d_gather, want);
        if (e != cudaSuccess && (e = cudaMalloc(&E.d_gather, *total)) == cudaSuccess) E.gather_cap = *total;
        else if (e == cudaSuccess) E.gather_cap = want;
        if (e != cudaSuccess)
        {
            cudaGetLastError();
            E.d_gather = nullptr;
            set_error(-2, "%s: the packed batch needs %llu bytes of HBM on device %d, which cannot be allocated (%s); search the "
                          "texts in smaller batches", who, (unsigned long long)*total, E.device, cudaGetErrorString(e));
            return -2;
        }
    }
    std::vector<uint64_t> tab(3 * nl);
    for (size_t i = 0; i < nl; i++)
    {
        tab[i] = offsets[live[i]];
        tab[nl + i] = (*off)[live[i]];
        tab[2 * nl + i] = lens[live[i]];
    }
    const uint64_t tab_bytes = 24 * (uint64_t)nl + nl + 8;
    if (tab_bytes > E.gather_tab_cap)
    {
        CKH(cudaStreamSynchronize(E.scan_stream));
        cudaFree(E.d_gather_tab);
        E.d_gather_tab = nullptr;
        E.gather_tab_cap = 0;
        CKH(cudaMalloc(&E.d_gather_tab, tab_bytes + tab_bytes / 4));
        E.gather_tab_cap = tab_bytes + tab_bytes / 4;
    }
    cudaStream_t st = E.scan_stream;
    uint8_t *d_last = last ? (uint8_t *)(E.d_gather_tab + 3 * nl) : nullptr;
    if (nl) CKH(cudaMemcpyAsync(E.d_gather_tab, tab.data(), tab.size() * 8, cudaMemcpyHostToDevice, st));
    cudaEvent_t a = pool_event(E, 0), b = pool_event(E, 1);
    CKH(cudaEventRecord(a, st));
    if (batch_gather(d_base, E.d_gather_tab, (uint32_t)nl, *total, fill, E.d_gather, d_last, st) != 0) return -2;
    CKH(cudaEventRecord(b, st));
    if (last)
    {
        last->resize(nl);
        if (nl) CKH(cudaMemcpyAsync(last->data(), d_last, nl, cudaMemcpyDeviceToHost, st));
    }
    CKH(cudaStreamSynchronize(st));
    float ms = 0.f;
    CKH(cudaEventElapsedTime(&ms, a, b));
    t_resident.gather_ms += ms;
    trace("%s: %zu texts gathered into %llu bytes (%.3f ms)", who, nl, (unsigned long long)*total, ms);
    return 0;
}

// The packed buffer as one shard: it owns all its bytes and has no neighbours.
static krep_b200_shard_t packed_shard(const DevCtx &E, uint64_t total)
{
    krep_b200_shard_t sh;
    memset(&sh, 0, sizeof sh);
    sh.d_text = E.d_gather;
    sh.avail_len = total;
    sh.own_begin = 0;
    sh.own_end = total;
    sh.global_offset = 0;
    sh.prev_byte = -1;
    sh.next_byte = -1;
    return sh;
}

// krep_b200_search_batch_resident: krep_b200_search_batch's answers for texts that live in HBM.  The texts are gathered on
// their device into one buffer laid out as run_batch packs host texts (gaps longer than the longest pattern), scanned as
// one shard, and cut and replayed per text by replay_batch_cuts.  No host copy of a text exists, so each cut replays from
// its keys alone, as resident shards do: -w from the tag bits the scan computed (a gap byte is not a word character, so a
// text's edges read as text boundaries), and -c from the line bounds the scan of a count_lines plan found.  The gaps are
// zero bytes, as on the host, except under -c, where they are '\n': the device's search for a line bound then stops at
// the text's own edges, so it reads no byte of another text and finds the text's own find_line_start / find_line_end
// (DESIGN §12.9).  No occurrence changes with the fill, since a key counts only when it lies wholly inside its text.
static int run_batch_resident(int entry_algo, const search_params_t *P, const void *d_base, const uint64_t *offsets,
                              const size_t *lens, size_t nt, uint64_t *counts, match_result_t *const *results)
{
    static const char *who = "krep_b200_search_batch_resident";
    warm_join();
    std::lock_guard<std::recursive_mutex> lk(engine_mutex());
    clear_error();
    t_resident = ResidentTimes();
    if (!P || (nt && (!offsets || !lens || !counts)))
    {
        set_error(-3, "%s: null argument", who);
        return -3;
    }
    if (nt == 0) return 0;
    for (size_t f = 0; f < nt; f++) counts[f] = 0;
    if (visible_devices() == 0)
    {
        set_error(-1, "no CUDA device available; this engine has no CPU fallback");
        return -1;
    }
    DeviceGuard guard;
    DevCtx *Cp = resident_ctx(who, d_base, offsets, lens, nt);
    if (!Cp) return krep_b200_last_error() ? krep_b200_last_error() : -1;
    DevCtx &E = *Cp;
    const bool only_matching = g_only_matching;
    std::vector<int> algo_of;
    const int algo = batch_early_answers(entry_algo, P, nt, lens, [&](size_t f) { return (const char *)d_base + offsets[f]; },
                                         counts, results, &algo_of);
    if (krep_b200_last_error() != 0) return -3;
    if (algo < 0) return 0;
    Plan *plan = plan_for(P, algo, only_matching);
    if (!plan) return -2;
    const size_t gap = (size_t)(plan->is_ac ? plan->max_len : plan->m) + 16;
    std::vector<size_t> live;
    for (size_t f = 0; f < nt; f++)
        if (algo_of[f] >= 0) live.push_back(f);
    if (live.size() >= UINT32_MAX)
    {
        set_error(-3, "%s: too many texts in one call", who);
        return -3;
    }
    std::vector<uint64_t> off(nt, 0);
    uint64_t total = 0;
    const uint8_t fill = P->count_lines_mode ? '\n' : 0;
    int rc = gather_resident(E, who, d_base, offsets, lens, live, gap, fill, &off, &total, nullptr);
    if (rc != 0) return rc;
    const krep_b200_shard_t sh = packed_shard(E, total);
    ScanOut so;
    if ((rc = scan_shard(E, plan, &sh, 1, E.scan_stream, &so)) != 0) return rc;
    t_resident.scan_ms = get_kernel_ms();
    const uint64_t *keys = nullptr;
    if (fetch_keys(E, so, &keys) != 0) return -2;
    // -c: the line bounds of every key, the "same line as my neighbour" markers resolved over the whole list (a '\n' gap
    // lies between any two texts, so a marker never reaches into another text)
    std::vector<uint64_t> bounds;
    const bool lines = P->count_lines_mode && so.stored;
    if (lines)
    {
        if (!so.d_bounds)
        {
            set_error(-2, "%s: the -c scan left no line bounds", who);
            return -2;
        }
        bounds.resize(2 * so.stored);
        CKH(cudaMemcpyAsync(bounds.data(), so.d_bounds, bounds.size() * 8, cudaMemcpyDeviceToHost, E.result_stream));
        CKH(cudaStreamSynchronize(E.result_stream));
        for (uint64_t i = 0; i < so.stored; i++)
            if (bounds[2 * i] == LB_SAME_AS_PREV) bounds[2 * i] = i ? bounds[2 * (i - 1)] : 0;
        for (uint64_t i = so.stored; i-- > 0;)
            if (bounds[2 * i + 1] == LB_SAME_AS_NEXT) bounds[2 * i + 1] = i + 1 < so.stored ? bounds[2 * (i + 1) + 1] : total;
    }
    const auto t0 = std::chrono::steady_clock::now();
    replay_batch_cuts(plan, algo, P, only_matching, keys, so.stored, lines ? bounds.data() : nullptr, gap, algo_of, off, nullptr,
                      lens, counts, results);
    t_resident.resolve_ms = ms_since(t0);
    trace("%s: %zu texts, %llu keys (resolved in %.3f ms)", who, live.size(), (unsigned long long)so.stored, t_resident.resolve_ms);
    return 0;
}

// krep_b200_regex_search_batch_resident: krep_b200_regex_search_batch's answers for texts that live in HBM.  The texts
// are gathered on their device with '\n' gaps as regex_batch_scan packs host texts, scanned once in the kernel's batch
// mode (with the long-line pass), and the bytes of the lines glibc must see come back in one row (scan_regex_pack.cu);
// each text is then resolved from its part of the row (regex_resolve_batch) with its own length, last byte and -m
// budget.  Empty texts keep the host answer.
static int run_regex_batch_resident(const search_params_t *P, const void *d_base, const uint64_t *offsets, const size_t *lens,
                                    size_t nt, uint64_t *counts, match_result_t *const *results)
{
    static const char *who = "krep_b200_regex_search_batch_resident";
    warm_join();
    std::lock_guard<std::recursive_mutex> lk(engine_mutex());
    clear_error();
    t_resident = ResidentTimes();
    if (!P || (nt && (!offsets || !lens || !counts)))
    {
        set_error(-3, "%s: null argument", who);
        return -3;
    }
    if (nt == 0) return 0;
    for (size_t f = 0; f < nt; f++) counts[f] = 0;
    if (visible_devices() == 0)
    {
        set_error(-1, "no CUDA device available; this engine has no CPU fallback");
        return -1;
    }
    DeviceGuard guard;
    DevCtx *Cp = resident_ctx(who, d_base, offsets, lens, nt);
    if (!Cp) return krep_b200_last_error() ? krep_b200_last_error() : -1;
    DevCtx &E = *Cp;
    if (regex_returns_early(P)) return 0;
    std::vector<size_t> live;
    for (size_t f = 0; f < nt; f++)
        if (lens[f] > 0) live.push_back(f);
    if (!live.empty())
    {
        Plan *plan = regex_plan_or_refuse(P);
        if (!plan) return -3;
        if (live.size() >= UINT32_MAX)
        {
            set_error(-3, "%s: too many texts in one call", who);
            return -3;
        }
        const RegexMode mode = regex_call_mode(P, plan);
        const size_t nl = live.size();
        std::vector<uint64_t> off(nt, 0);
        std::vector<uint8_t> last;
        uint64_t total = 0;
        int rc = gather_resident(E, who, d_base, offsets, lens, live, 1, '\n', &off, &total, &last);
        if (rc != 0) return rc;
        RegexBatch B;
        regex_batch_table(lens, live, off, total, &B);
        RegexBatchDev bd;
        if (upload_regex_batch(E, B, &bd) != 0) return -2;
        const krep_b200_shard_t sh = packed_shard(E, total);
        uint64_t cnt = 0, row_bytes = 0;
        const uint64_t *d_sorted = nullptr;
        const void *d_row = nullptr;
        std::vector<uint64_t> text_lines(nl, 0);
        cudaEvent_t a = pool_event(E, 0), b = pool_event(E, 1);
        CKH(cudaEventRecord(a, E.scan_stream));
        if ((rc = regex_scan_keys(E, plan, &sh, mode, who, &cnt, &d_sorted, text_lines.data(), long_lines_default(), &bd)) != 0)
            return rc;
        CKH(cudaEventRecord(b, E.scan_stream));
        float pack_ms = 0.f, scan_ms = 0.f;
        if ((rc = regex_pack_row(E, &sh, mode, d_sorted, cnt, 0, &d_row, &row_bytes, &pack_ms)) != 0) return rc;
        CKH(cudaEventElapsedTime(&scan_ms, a, b));
        t_resident.scan_ms = scan_ms + pack_ms;
        uint8_t *h = regex_pack_host_buffer(E, row_bytes);
        if (!h) return -2;
        CKH(cudaMemcpyAsync(h, d_row, row_bytes, cudaMemcpyDeviceToHost, E.scan_stream));
        CKH(cudaStreamSynchronize(E.scan_stream));
        const auto t0 = std::chrono::steady_clock::now();
        std::vector<uint64_t> lo(nl), cnts(nl, 0);
        std::vector<size_t> len(nl);
        std::vector<match_result_t *> res(nl, nullptr);
        for (size_t i = 0; i < nl; i++)
        {
            lo[i] = off[live[i]];
            len[i] = lens[live[i]];
            if (results) res[i] = results[live[i]];
        }
        if ((rc = regex_resolve_batch(P, h, nl, lo.data(), len.data(), last.data(), text_lines.data(), cnts.data(), res.data())) != 0)
            return rc;
        for (size_t i = 0; i < nl; i++) counts[live[i]] = cnts[i];
        t_resident.resolve_ms = ms_since(t0);
        trace("%s: mode %d, %zu texts, %llu keys, %llu row bytes (resolved in %.3f ms)", who, mode, nl, (unsigned long long)cnt,
              (unsigned long long)row_bytes, t_resident.resolve_ms);
    }
    for (size_t f = 0; f < nt; f++)
        if (lens[f] == 0) counts[f] = regex_empty_text(P, results ? results[f] : nullptr);
    return 0;
}

} // namespace kb

using namespace kb;

extern "C" {

void krep_b200_set_only_matching(bool on) { g_only_matching = on; }
bool krep_b200_get_only_matching(void) { return g_only_matching; }
void krep_b200_set_force_no_simd(bool on) { g_force_no_simd = on; }
void krep_b200_set_algo_override(const char *name) { g_algo_override = name ? name : ""; }

uint64_t krep_b200_boyer_moore_search(const search_params_t *p, const char *t, size_t n, match_result_t *r)
{
    return run_search(KREP_B200_ALGO_BMH, p, t, n, r);
}
uint64_t krep_b200_kmp_search(const search_params_t *p, const char *t, size_t n, match_result_t *r)
{
    return run_search(KREP_B200_ALGO_KMP, p, t, n, r);
}
uint64_t krep_b200_memchr_search(const search_params_t *p, const char *t, size_t n, match_result_t *r)
{
    return run_search(KREP_B200_ALGO_MEMCHR, p, t, n, r);
}
uint64_t krep_b200_memchr_short_search(const search_params_t *p, const char *t, size_t n, match_result_t *r)
{
    return run_search(KREP_B200_ALGO_MEMCHR_SHORT, p, t, n, r);
}
uint64_t krep_b200_simd_sse42_search(const search_params_t *p, const char *t, size_t n, match_result_t *r)
{
    return run_search(KREP_B200_ALGO_SSE42, p, t, n, r);
}
uint64_t krep_b200_simd_avx2_search(const search_params_t *p, const char *t, size_t n, match_result_t *r)
{
    return run_search(KREP_B200_ALGO_AVX2, p, t, n, r);
}
uint64_t krep_b200_simd_avx512_search(const search_params_t *p, const char *t, size_t n, match_result_t *r)
{
    return run_search(KREP_B200_ALGO_AVX512, p, t, n, r);
}
uint64_t krep_b200_aho_corasick_search(const search_params_t *p, const char *t, size_t n, match_result_t *r)
{
    return run_search(KREP_B200_ALGO_AC, p, t, n, r);
}
uint64_t krep_b200_neon_search(const search_params_t *p, const char *t, size_t n, match_result_t *r)
{
    return run_search(KREP_B200_ALGO_NEON, p, t, n, r);
}
uint64_t krep_b200_regex_search(const search_params_t *p, const char *t, size_t n, match_result_t *r)
{
    return run_regex(p, t, n, r);
}


int krep_b200_regex_search_batch(const search_params_t *params, const char *const *texts, const size_t *lens, size_t n_texts,
                                 uint64_t *counts, match_result_t *const *results)
{
    return run_regex_batch(params, texts, lens, n_texts, counts, results);
}

// The kernel a batch entry point emulates, or -1 with the error set (regex_batch: the call that batches regex searches).
static int batch_entry_algo(search_func_t entry, const char *who, const char *regex_batch)
{
    int algo = -1;
    if (entry == krep_b200_boyer_moore_search) algo = KREP_B200_ALGO_BMH;
    else if (entry == krep_b200_kmp_search) algo = KREP_B200_ALGO_KMP;
    else if (entry == krep_b200_memchr_search) algo = KREP_B200_ALGO_MEMCHR;
    else if (entry == krep_b200_memchr_short_search) algo = KREP_B200_ALGO_MEMCHR_SHORT;
    else if (entry == krep_b200_simd_sse42_search) algo = KREP_B200_ALGO_SSE42;
    else if (entry == krep_b200_simd_avx2_search) algo = KREP_B200_ALGO_AVX2;
    else if (entry == krep_b200_simd_avx512_search) algo = KREP_B200_ALGO_AVX512;
    else if (entry == krep_b200_aho_corasick_search) algo = KREP_B200_ALGO_AC;
    else if (entry == krep_b200_neon_search) algo = KREP_B200_ALGO_NEON;
    if (entry == krep_b200_regex_search) set_error(-3, "%s: regex searches are batched by %s", who, regex_batch);
    else if (algo < 0) set_error(-3, "%s: entry must be one of this library's search_func_t entry points", who);
    return algo;
}

int krep_b200_search_batch(search_func_t entry, const search_params_t *params, const char *const *texts, const size_t *lens,
                           size_t n_texts, uint64_t *counts, match_result_t *const *results)
{
    const int algo = batch_entry_algo(entry, "krep_b200_search_batch", "krep_b200_regex_search_batch");
    if (algo < 0) return -3;
    return run_batch(algo, params, texts, lens, n_texts, counts, results);
}

int krep_b200_search_batch_resident(search_func_t entry, const search_params_t *params, const void *d_base, const uint64_t *offsets,
                                    const size_t *lens, size_t n_texts, uint64_t *counts, match_result_t *const *results)
{
    clear_error();
    for (size_t f = 0; counts && f < n_texts; f++) counts[f] = 0;
    const int algo = batch_entry_algo(entry, "krep_b200_search_batch_resident", "krep_b200_regex_search_batch_resident");
    if (algo < 0) return -3;
    return run_batch_resident(algo, params, d_base, offsets, lens, n_texts, counts, results);
}

int krep_b200_regex_search_batch_resident(const search_params_t *params, const void *d_base, const uint64_t *offsets,
                                          const size_t *lens, size_t n_texts, uint64_t *counts, match_result_t *const *results)
{
    return run_regex_batch_resident(params, d_base, offsets, lens, n_texts, counts, results);
}

void krep_b200_batch_resident_stats(float *gather_ms, float *scan_ms, double *resolve_ms)
{
    if (gather_ms) *gather_ms = t_resident.gather_ms;
    if (scan_ms) *scan_ms = t_resident.scan_ms;
    if (resolve_ms) *resolve_ms = t_resident.resolve_ms;
}

int64_t krep_b200_batch_gather_raw(const void *base, const uint64_t *offsets, const size_t *lens, size_t n, int gap_kind,
                                   size_t max_gap, void *dst_host, uint64_t cap)
{
    static const char *who = "krep_b200_batch_gather_raw";
    warm_join();
    std::lock_guard<std::recursive_mutex> lk(engine_mutex());
    clear_error();
    if (!base || (n && (!offsets || !lens)) || (cap && !dst_host) || gap_kind < 0 || gap_kind > 1)
    {
        set_error(-3, "%s: bad argument", who);
        return -3;
    }
    const size_t gap = gap_kind == 0 ? max_gap + 16 : 1;
    const uint8_t fill = gap_kind == 0 ? 0 : '\n';
    std::vector<size_t> live(n);
    for (size_t f = 0; f < n; f++) live[f] = f;
    std::vector<uint64_t> off(n, 0);
    uint64_t total = 0;
    DeviceGuard guard;
    cudaPointerAttributes a;
    const bool on_device = cudaPointerGetAttributes(&a, base) == cudaSuccess && a.type == cudaMemoryTypeDevice;
    cudaGetLastError();
    if (!on_device)
    {
        // host texts: the host batch's own pack, for comparison
        DevCtx *Cp = ctx_primary();
        if (!Cp) return -1;
        std::vector<const char *> texts(n);
        for (size_t f = 0; f < n; f++) texts[f] = (const char *)base + offsets[f];
        if (pack_texts(*Cp, texts.data(), lens, live, gap, fill, &off, &total) != 0) return -2;
        if (cap) memcpy(dst_host, Cp->h_batch, std::min<uint64_t>(total, cap));
        return (int64_t)total;
    }
    DevCtx *Cp = resident_ctx(who, base, offsets, lens, n);
    if (!Cp) return krep_b200_last_error() ? krep_b200_last_error() : -1;
    const int rc = gather_resident(*Cp, who, base, offsets, lens, live, gap, fill, &off, &total, nullptr);
    if (rc != 0) return rc;
    if (cap && total)
    {
        CKH(cudaMemcpy(dst_host, Cp->d_gather, std::min<uint64_t>(total, cap), cudaMemcpyDeviceToHost));
    }
    return (int64_t)total;
}

void krep_b200_regex_batch_stats(double *pack_ms, double *resolve_ms)
{
    if (pack_ms) *pack_ms = t_rx_batch.pack_ms;
    if (resolve_ms) *resolve_ms = t_rx_batch.resolve_ms;
}

// One batch scan in the given mode, its keys sorted and read back (DESIGN §12.5), with or without the long-line pass.
static int64_t regex_batch_raw(const char *who, const search_params_t *P, const char *const *texts, const size_t *lens,
                               size_t n_texts, int mode, const LongLineOpts *long_lines, uint64_t *offsets, uint64_t *keys,
                               uint64_t cap, uint64_t *text_lines)
{
    warm_join();
    std::lock_guard<std::recursive_mutex> lk(engine_mutex());
    clear_error();
    if (!P || (n_texts && (!texts || !lens)) || (cap && !keys))
    {
        set_error(-3, "%s: null argument", who);
        return -3;
    }
    Plan *plan = regex_plan_of(P);
    if (!plan || !regex_mode_available(*plan->rx, mode))
    {
        set_error(-3, "%s: mode %d is not available for this pattern", who, mode);
        return -3;
    }
    std::vector<size_t> live;
    for (size_t f = 0; f < n_texts; f++)
    {
        if (lens[f] > 0 && texts[f]) live.push_back(f);
        if (offsets) offsets[f] = UINT64_MAX;
        if (text_lines) text_lines[f] = 0;
    }
    if (live.empty()) return 0;
    DeviceGuard guard;
    std::vector<uint64_t> off(n_texts, 0);
    HostScan hs;
    const int rc = regex_batch_scan(plan, texts, lens, live, (RegexMode)mode, long_lines, who, &off, &hs);
    if (rc != 0) return rc;
    for (size_t i = 0; i < live.size(); i++)
    {
        if (offsets) offsets[live[i]] = off[live[i]];
        if (text_lines && mode == RX_COUNT) text_lines[live[i]] = hs.text_lines[i];
    }
    if (hs.nkeys && cap) memcpy(keys, hs.keys, std::min<uint64_t>(hs.nkeys, cap) * sizeof(uint64_t));
    return (int64_t)hs.nkeys;
}

int64_t krep_b200_regex_search_batch_raw(const search_params_t *P, const char *const *texts, const size_t *lens, size_t n_texts,
                                         int mode, uint64_t *offsets, uint64_t *keys, uint64_t cap, uint64_t *text_lines)
{
    return regex_batch_raw("krep_b200_regex_search_batch_raw", P, texts, lens, n_texts, mode, nullptr, offsets, keys, cap,
                           text_lines);
}

int64_t krep_b200_regex_search_batch_long_raw(const search_params_t *P, const char *const *texts, const size_t *lens,
                                              size_t n_texts, int mode, uint32_t slice_bytes, uint32_t ckpt_bytes,
                                              uint64_t *offsets, uint64_t *keys, uint64_t cap, uint64_t *text_lines)
{
    const char *who = "krep_b200_regex_search_batch_long_raw";
    LongLineOpts o;
    if (long_lines_opts(who, slice_bytes, ckpt_bytes, &o) != 0) return -3;
    return regex_batch_raw(who, P, texts, lens, n_texts, mode, long_lines_default() ? &o : nullptr, offsets, keys, cap,
                           text_lines);
}

// krep.c:1873-1914
static bool is_repetitive_pattern(const char *pattern, size_t len)
{
    if (len < 3) return false;
    size_t run = 0;
    char prev = pattern[0];
    for (size_t i = 1; i < len; i++)
    {
        if (pattern[i] == prev)
        {
            if (++run >= len / 2) return true;
        }
        else
        {
            run = 0;
            prev = pattern[i];
        }
    }
    for (size_t period = 2; period <= len / 2; period++)
    {
        bool periodic = true;
        for (size_t i = period; i < len && periodic; i++) periodic = pattern[i] == pattern[i % period];
        if (periodic) return true;
    }
    return false;
}

// krep.c:1771-1870, for the AVX2 build of the reference (SIMD_MAX_PATTERN_LEN 32).
search_func_t krep_b200_select_search_algorithm(const search_params_t *P)
{
    if (!P) return NULL;
    if (P->use_regex)
    {
        // the regex goes to the GPU line filter when its compiler accepts the pattern; a refused one stays with the
        // host's regex_search
        std::lock_guard<std::recursive_mutex> lk(engine_mutex());
        return regex_plan_of(P) ? krep_b200_regex_search : NULL;
    }
    if (P->num_patterns > 1) return krep_b200_aho_corasick_search;
    if (!g_algo_override.empty() && g_algo_override != "auto")
    {
        if (g_algo_override == "bm") return krep_b200_boyer_moore_search;
        if (g_algo_override == "kmp") return krep_b200_kmp_search;
    }
    const size_t m = P->pattern_len;
    const bool can_simd = !g_force_no_simd && m <= SIMD_MAX_PATTERN_LEN;
    if (m == 1) return krep_b200_memchr_search;
    if (m < 4) return (can_simd && P->case_sensitive) ? krep_b200_simd_avx2_search : krep_b200_memchr_short_search;
    if (can_simd && m <= 32) return krep_b200_simd_avx2_search;
    if (m < 8 && is_repetitive_pattern(P->pattern, m)) return krep_b200_kmp_search;
    return krep_b200_boyer_moore_search;
}

const char *krep_b200_get_algorithm_name(search_func_t f)
{
    if (f == krep_b200_boyer_moore_search) return "Boyer-Moore-Horspool";
    if (f == krep_b200_kmp_search) return "Knuth-Morris-Pratt";
    if (f == krep_b200_aho_corasick_search) return "Aho-Corasick";
    if (f == krep_b200_memchr_search) return "memchr";
    if (f == krep_b200_memchr_short_search) return "memchr-short";
    if (f == krep_b200_simd_sse42_search) return "SSE4.2";
    if (f == krep_b200_simd_avx2_search) return "AVX2";
    if (f == krep_b200_simd_avx512_search) return "AVX-512";
    if (f == krep_b200_neon_search) return "NEON";
    if (f == krep_b200_regex_search) return "Regex (GPU line filter + regexec)";
    return "Unknown";
}

// ---- AC trie handles (aho_corasick.c:111 / 274 / 287) ----
ac_trie_t *krep_b200_ac_trie_build(const search_params_t *params)
{
    warm_join();
    std::lock_guard<std::recursive_mutex> lk(engine_mutex());
    clear_error();
    if (!params || params->num_patterns == 0) return NULL; // aho_corasick.c:113
    if (visible_devices() == 0)
    {
        set_error(-1, "no CUDA device available; this engine has no CPU fallback");
        return NULL;
    }
    Plan *pl = plan_build(params, KREP_B200_ALGO_AC, false); // owned by the handle, not by the plan cache
    if (!pl) return NULL;
    TrieHandle *h = new TrieHandle{TRIE_MAGIC, pl};
    return reinterpret_cast<ac_trie_t *>(h);
}
void krep_b200_ac_trie_free(ac_trie_t *trie)
{
    TrieHandle *h = reinterpret_cast<TrieHandle *>(trie);
    if (!h || h->magic != TRIE_MAGIC) return;
    std::lock_guard<std::recursive_mutex> lk(engine_mutex());
    plan_free(h->plan);
    h->magic = 0;
    delete h;
}
bool krep_b200_ac_trie_root_has_outputs(const ac_trie_t *trie)
{
    const TrieHandle *h = reinterpret_cast<const TrieHandle *>(trie);
    if (!h || h->magic != TRIE_MAGIC || !h->plan) return false;
    for (uint32_t len : h->plan->pat_lens)
        if (len == 0) return true; // an empty pattern's index sits on the root (aho_corasick.c:145)
    return false;
}

void krep_b200_set_devices(const int *devices, int n)
{
    std::lock_guard<std::recursive_mutex> lk(engine_mutex());
    if (devices && n > 0) keep_devices_visible();
    g_devices.clear();
    for (int i = 0; devices && i < n; i++) g_devices.push_back(devices[i]);
}

// ---- match_result helpers (krep.c:139 / 175 / 244 / 256) ----
match_result_t *krep_b200_match_result_init(uint64_t initial_capacity)
{
    match_result_t *r = (match_result_t *)malloc(sizeof *r);
    if (!r) return NULL;
    if (initial_capacity == 0) initial_capacity = 16;
    if (initial_capacity > SIZE_MAX / sizeof(match_position_t))
    {
        free(r);
        return NULL;
    }
    r->positions = (match_position_t *)malloc(initial_capacity * sizeof(match_position_t));
    if (!r->positions)
    {
        free(r);
        return NULL;
    }
    r->count = 0;
    r->capacity = initial_capacity;
    return r;
}
bool krep_b200_match_result_add(match_result_t *r, size_t s, size_t e) { return result_push(r, s, e); }
void krep_b200_match_result_free(match_result_t *r)
{
    if (!r) return;
    free(r->positions);
    free(r);
}
bool krep_b200_match_result_merge(match_result_t *dest, const match_result_t *src, size_t chunk_offset)
{
    if (!dest || !src || src->count == 0) return true;
    for (uint64_t i = 0; i < src->count; i++)
        if (!result_push(dest, src->positions[i].start_offset + chunk_offset, src->positions[i].end_offset + chunk_offset))
            return false;
    return true;
}

uint64_t krep_b200_replay(int algo, const search_params_t *P, bool only_matching, const uint64_t *keys, uint64_t nkeys,
                          const char *text, size_t text_len, match_result_t *result)
{
    if (!P) return 0;
    if (P->count_lines_mode && !text && nkeys)
    {
        set_error(-3, "krep_b200_replay: -c line counting needs the host text");
        return 0;
    }
    if (algo == KREP_B200_ALGO_REGEX)
    {
        clear_error();
        if (!text && text_len)
        {
            set_error(-3, "krep_b200_replay: regex keys are confirmed by regexec on the host text");
            return 0;
        }
        return replay_regex(P, Replay{keys, (size_t)nkeys, text, text_len, 0}, result);
    }
    Replay r{keys, (size_t)nkeys, text, text_len ? text_len : (SIZE_MAX >> 1), 0};
    if (algo == KREP_B200_ALGO_AC) return replay_ac(P, r, result);
    algo = resolve_algo(P, algo);
    const uint32_t m = algo == KREP_B200_ALGO_MEMCHR ? 1u : (uint32_t)P->pattern_len;
    return replay_literal(algo, P, only_matching, m, r, result);
}

uint64_t krep_b200_replay_lines(int algo, const search_params_t *P, bool only_matching, const uint64_t *keys, uint64_t nkeys,
                                const uint64_t *bounds, size_t text_len, match_result_t *result)
{
    if (!P) return 0;
    if (algo == KREP_B200_ALGO_REGEX)
    {
        set_error(-3, "krep_b200_replay_lines: regex keys need the host text (krep_b200_replay)");
        return 0;
    }
    if (P->count_lines_mode && !bounds && nkeys)
    {
        set_error(-3, "krep_b200_replay_lines: -c needs the line bounds");
        return 0;
    }
    Replay r{keys, (size_t)nkeys, nullptr, text_len ? text_len : (SIZE_MAX >> 1), 0, bounds};
    if (algo == KREP_B200_ALGO_AC) return replay_ac(P, r, result);
    algo = resolve_algo(P, algo);
    const uint32_t m = algo == KREP_B200_ALGO_MEMCHR ? 1u : (uint32_t)P->pattern_len;
    return replay_literal(algo, P, only_matching, m, r, result);
}

// ---- fused -c on resident shards ----
int krep_b200_count_lines_shard(const krep_b200_plan_t *plan_, const search_params_t *P, const krep_b200_shard_t *shard, void *stream,
                                krep_b200_line_count_t *out)
{
    std::lock_guard<std::recursive_mutex> lk(engine_mutex());
    clear_error();
    const Plan *plan = reinterpret_cast<const Plan *>(plan_);
    if (!plan || !P || !shard || !out)
    {
        set_error(-3, "krep_b200_count_lines_shard: null argument");
        return -3;
    }
    if (!count_lines_eligible(plan, P, plan->algo))
    {
        set_error(-3, "krep_b200_count_lines_shard: this plan's -c result needs the occurrence list (window kernel, newline in "
                      "a pattern or tag-mode -w): use krep_b200_scan_shard + krep_b200_collect");
        return -3;
    }
    DeviceGuard guard;
    DevCtx *C = ctx_of_pointer(shard->d_text);
    if (!C) return -1;
    cudaStream_t st = stream ? (cudaStream_t)stream : C->scan_stream;
    reset_kernel_ms();
    if (cudaEventRecord(C->ev_ca, st) != cudaSuccess) return -2;
    int rc = launch_count_lines(*C, plan, shard, st, 0);
    if (rc != 0) return rc;
    if (cudaEventRecord(C->ev_cb, st) != cudaSuccess || cudaStreamSynchronize(st) != cudaSuccess)
    {
        set_error(-2, "CUDA error in the fused line count (%s)", cudaGetErrorString(cudaGetLastError()));
        return -2;
    }
    float ms = 0.f;
    cudaEventElapsedTime(&ms, C->ev_ca, C->ev_cb);
    add_kernel_ms(ms);
    out->lines = C->h_line_out[0];
    out->flags = (uint32_t)C->h_line_out[1];
    out->reserved = 0;
    return 0;
}

uint64_t krep_b200_combine_line_counts(const krep_b200_line_count_t *recs, size_t n, size_t max_count)
{
    if (!recs) return 0;
    std::vector<uint64_t> flat(2 * n);
    for (size_t i = 0; i < n; i++)
    {
        flat[2 * i] = recs[i].lines;
        flat[2 * i + 1] = recs[i].flags;
    }
    return std::min<uint64_t>(combine_line_records(flat.data(), n), max_count);
}

// ---- several resident shards, one answer: search_file's chunk loop + merge (krep.c:2851-3004) for text that already
// lives in HBM, possibly on several GPUs of this process.  Scans run concurrently on distinct devices; per-shard lists are
// merged by key; the emulated kernel's policy is replayed once over the whole list (so -m, overlap rules and the
// emission order are global, not per shard).
uint64_t krep_b200_search_shards(const krep_b200_plan_t *plan_, const search_params_t *P, const krep_b200_shard_t *shards,
                                 uint32_t n_shards, match_result_t *result)
{
    std::lock_guard<std::recursive_mutex> lk(engine_mutex());
    clear_error();
    const Plan *plan = reinterpret_cast<const Plan *>(plan_);
    if (!plan || !P || (!shards && n_shards))
    {
        set_error(-3, "krep_b200_search_shards: null argument");
        return 0;
    }
    if (plan->is_regex) return search_shards_regex(plan, P, shards, n_shards, result);
    DeviceGuard guard;
    std::vector<DevCtx *> ctx(n_shards, nullptr);
    uint64_t text_len = 0;
    for (uint32_t i = 0; i < n_shards; i++)
    {
        ctx[i] = ctx_of_pointer(shards[i].d_text);
        if (!ctx[i]) return 0;
        text_len = std::max<uint64_t>(text_len, shards[i].global_offset + shards[i].avail_len);
    }
    reset_kernel_ms();
    if (P->count_lines_mode)
    {
        if (!count_lines_eligible(plan, P, plan->algo))
        {
            set_error(-3, "krep_b200_search_shards: -c over several shards is only available where the scan counts lines itself "
                          "(single literals and pattern sets; see krep_b200_count_lines_shard)");
            return 0;
        }
        if (P->max_count == 0) return 0;
        std::vector<uint64_t> recs(2 * (size_t)n_shards);
        for (uint32_t i = 0; i < n_shards; i++) // size every device's record array first: growing it later would move it
        {
            cudaSetDevice(ctx[i]->device);
            if (ensure_line_out(*ctx[i], n_shards) != 0) return 0;
        }
        // a pattern set's record needs its scan's count on the host first: each device ends its previous shard before it
        // begins the next one, so shards on distinct devices are scanned concurrently
        std::vector<int> pending(MAX_DEV, -1);
        auto set_end = [&](int i) {
            DevCtx &C = *ctx[i];
            cudaSetDevice(C.device);
            return set_count_end(C, plan, &shards[i], C.scan_stream, set_count_slot(C), (uint64_t)i);
        };
        for (uint32_t i = 0; i < n_shards; i++)
        {
            DevCtx &C = *ctx[i];
            if (plan->is_ac && pending[C.device] >= 0 && set_end(pending[C.device]) != 0) return 0;
            cudaSetDevice(C.device);
            if (plan->is_ac)
            {
                if (set_count_begin(C, plan, &shards[i], C.scan_stream, set_count_slot(C)) != 0) return 0;
                pending[C.device] = (int)i;
            }
            else if (launch_count_lines(C, plan, &shards[i], C.scan_stream, i) != 0)
                return 0;
        }
        for (int d = 0; d < MAX_DEV; d++)
            if (pending[d] >= 0 && set_end(pending[d]) != 0) return 0;
        for (uint32_t i = 0; i < n_shards; i++)
        {
            cudaSetDevice(ctx[i]->device);
            if (cudaStreamSynchronize(ctx[i]->scan_stream) != cudaSuccess)
            {
                set_error(-2, "CUDA error in the fused line count (%s)", cudaGetErrorString(cudaGetLastError()));
                return 0;
            }
            recs[2 * i] = ctx[i]->h_line_out[2 * i];
            recs[2 * i + 1] = ctx[i]->h_line_out[2 * i + 1];
        }
        return std::min<uint64_t>(combine_line_records(recs.data(), n_shards), P->max_count);
    }
    const bool need_list = (P->track_positions && result) || !keeps_all(plan->algo, plan->built_only_matching, P, plan) || plan->whole_word == 2;
    std::vector<std::vector<uint64_t>> keys(n_shards);
    std::vector<int> pending(MAX_DEV, -1); // shard whose scan is in flight on each device
    std::vector<int> slot_of(n_shards, 0);
    uint64_t total_count = 0;
    float kmax = 0.f;
    auto finish = [&](int i) -> int {
        DevCtx &C = *ctx[i];
        cudaSetDevice(C.device);
        ScanOut so;
        int rc = scan_end(C, slot_of[i], &so);
        kmax = std::max(kmax, get_kernel_ms());
        if (rc != 0) return rc;
        total_count += so.count;
        if (need_list && so.stored)
        {
            const uint64_t *k = nullptr;
            if ((rc = fetch_keys(C, so, &k)) != 0) return rc;
            keys[i].assign(k, k + so.stored);
        }
        return 0;
    };
    for (uint32_t i = 0; i < n_shards; i++)
    {
        DevCtx &C = *ctx[i];
        if (pending[C.device] >= 0)
        {
            if (finish(pending[C.device]) != 0) return 0;
            pending[C.device] = -1;
        }
        cudaSetDevice(C.device);
        if (scan_begin(C, plan, &shards[i], need_list ? 1 : 0, nullptr, &slot_of[i]) != 0) return 0;
        pending[C.device] = (int)i;
    }
    for (int d = 0; d < MAX_DEV; d++)
        if (pending[d] >= 0 && finish(pending[d]) != 0) return 0;
    set_kernel_ms(kmax);
    if (!need_list) return limited_count(plan->algo, P, total_count);
    std::vector<const uint64_t *> lists;
    std::vector<uint64_t> counts;
    uint64_t total = 0;
    for (auto &k : keys)
    {
        lists.push_back(k.data());
        counts.push_back(k.size());
        total += k.size();
    }
    std::vector<uint64_t> merged(total ? total : 1);
    const uint64_t nk = merge_key_lists(lists.data(), counts.data(), (uint32_t)lists.size(), merged.data());
    Replay r{merged.data(), (size_t)nk, nullptr, text_len ? (size_t)text_len : (SIZE_MAX >> 1), 0};
    if (plan->is_ac) return replay_ac(P, r, result);
    return replay_literal(plan->algo, P, plan->built_only_matching, plan->m, r, result);
}

// ---- shard result -> match_result_t under the emulated kernel's policy ----
uint64_t krep_b200_collect(const krep_b200_plan_t *plan_, const search_params_t *P, const krep_b200_device_result_t *dev,
                           match_result_t *result)
{
    std::lock_guard<std::recursive_mutex> lk(engine_mutex());
    clear_error();
    const Plan *plan = reinterpret_cast<const Plan *>(plan_);
    if (!plan || !P || !dev) return 0;
    if (plan->is_regex)
    {
        set_error(-3, "krep_b200_collect: a device result does not carry its shard's text, which a regex plan needs: call "
                      "krep_b200_search_shards (or krep_b200_regex_export_shard + krep_b200_regex_resolve)");
        return 0;
    }
    if (P->count_lines_mode && dev->stored && !dev->d_line_bounds)
    {
        set_error(-3, "krep_b200_collect: -c needs a plan created with count_lines_mode (line bounds are computed by the scan)");
        return 0;
    }
    if (!dev->stored) return limited_count(plan->algo, P, plan->is_ac || keeps_all(plan->algo, g_only_matching, P, plan) ? dev->count : 0);
    DeviceGuard guard;
    DevCtx *Cp = ctx_get(dev->device);
    if (!Cp) return 0;
    DevCtx &E = *Cp;
    ScanOut so;
    so.count = dev->count;
    so.stored = dev->stored;
    so.d_keys = dev->d_keys;
    // the keys came back with the count if the list was short and no later scan has reused the slot
    if (dev->serial == E.serial && dev->stored <= PACK_KEYS && dev->slot >= 0 && dev->slot < SCAN_SLOTS)
        so.h_sorted = E.h_pack[dev->slot] + 1;
    const uint64_t *keys = nullptr;
    if (fetch_keys(E, so, &keys) != 0) return 0;
    Replay r{keys, (size_t)so.stored, nullptr, dev->text_len ? (size_t)dev->text_len : (SIZE_MAX >> 1), 0};
    if (P->count_lines_mode)
    {
        // read the device-computed line bounds back and resolve the "same line as my neighbour" markers
        const uint64_t nb = 2 * so.stored;
        if (nb > E.h_bounds_cap)
        {
            cudaFreeHost(E.h_bounds);
            E.h_bounds = nullptr;
            E.h_bounds_cap = 0;
            if (cudaMallocHost(&E.h_bounds, (nb + nb / 4 + 1024) * sizeof(uint64_t)) != cudaSuccess)
            {
                set_error(-2, "cannot allocate pinned memory for line bounds");
                return 0;
            }
            E.h_bounds_cap = nb + nb / 4 + 1024;
        }
        cudaStream_t st = E.result_stream ? E.result_stream : E.scan_stream; // ordered after the sort and k_line_bounds
        if (cudaMemcpyAsync(E.h_bounds, dev->d_line_bounds, nb * sizeof(uint64_t), cudaMemcpyDeviceToHost, st) != cudaSuccess ||
            cudaStreamSynchronize(st) != cudaSuccess)
        {
            set_error(-2, "reading line bounds back failed");
            return 0;
        }
        uint64_t *b = E.h_bounds;
        for (uint64_t i = 0; i < so.stored; i++)
            if (b[2 * i] == LB_SAME_AS_PREV) b[2 * i] = i ? b[2 * (i - 1)] : LB_OUTSIDE_SHARD;
        for (uint64_t i = so.stored; i-- > 0;)
            if (b[2 * i + 1] == LB_SAME_AS_NEXT) b[2 * i + 1] = i + 1 < so.stored ? b[2 * (i + 1) + 1] : LB_OUTSIDE_SHARD;
        for (uint64_t i = 0; i < nb; i++)
            if (b[i] == LB_OUTSIDE_SHARD)
            {
                set_error(-3, "krep_b200_collect: a matching line continues into a neighbouring shard; -c needs newline-aligned shards");
                return 0;
            }
        r.bounds = b;
    }
    if (plan->is_ac) return replay_ac(P, r, result);
    return replay_literal(plan->algo, P, plan->built_only_matching, plan->m, r, result);
}

// ---- -E rows of resident shards ----
int krep_b200_regex_export_shard(const krep_b200_plan_t *plan_, const search_params_t *P, const krep_b200_shard_t *shard, void *stream,
                                 void *dst, uint64_t dst_cap, uint64_t *row_bytes, const void **d_row)
{
    std::lock_guard<std::recursive_mutex> lk(engine_mutex());
    clear_error();
    const Plan *plan = reinterpret_cast<const Plan *>(plan_);
    if (!plan || !P || !shard || !row_bytes)
    {
        set_error(-3, "krep_b200_regex_export_shard: null argument");
        return -3;
    }
    DeviceGuard guard;
    if (stream && cudaStreamSynchronize((cudaStream_t)stream) != cudaSuccess)
    {
        set_error(-2, "krep_b200_regex_export_shard: the caller's stream failed (%s)", cudaGetErrorString(cudaGetLastError()));
        return -2;
    }
    t_rx_stats = RegexPackStats();
    DevCtx *C = nullptr;
    const void *row = nullptr;
    int rc = regex_export(plan, P, shard, "krep_b200_regex_export_shard", &C, &row, row_bytes);
    if (rc != 0) return rc;
    if (d_row) *d_row = row;
    if (!dst) return 0;
    if (dst_cap < *row_bytes)
    {
        set_error(-5, "krep_b200_regex_export_shard: the row needs %llu bytes, dst has %llu", (unsigned long long)*row_bytes,
                  (unsigned long long)dst_cap);
        return -5;
    }
    CKH(cudaMemcpyAsync(dst, row, *row_bytes, cudaMemcpyDefault, C->scan_stream));
    CKH(cudaStreamSynchronize(C->scan_stream));
    return 0;
}

uint64_t krep_b200_regex_resolve(const search_params_t *P, const void *const *rows, uint32_t n_rows, match_result_t *result)
{
    clear_error();
    if (!P || regex_returns_early(P)) return 0;
    int err = 0;
    const uint64_t ret = regex_resolve_rows(P, rows, n_rows, result, &err);
    return err ? 0 : ret;
}

void krep_b200_regex_export_stats(float *scan_ms, float *pack_ms, uint64_t *packed_bytes)
{
    if (scan_ms) *scan_ms = t_rx_stats.scan_ms;
    if (pack_ms) *pack_ms = t_rx_stats.pack_ms;
    if (packed_bytes) *packed_bytes = t_rx_stats.packed_bytes;
}

// ---- test hook: the line filter of a regex plan, run on the host ----
int64_t krep_b200_regex_filter_host(const search_params_t *P, const char *text, size_t n, uint64_t *line_starts, uint64_t cap,
                                    int *widened)
{
    std::lock_guard<std::recursive_mutex> lk(engine_mutex());
    Plan *pl = regex_plan_of(P);
    if (!pl) return -1;
    std::vector<uint64_t> v;
    regex_lines_host(*pl->rx, text, text ? n : 0, &v);
    for (size_t i = 0; i < v.size() && i < cap; i++) line_starts[i] = v[i];
    if (widened) *widened = pl->rx->widened ? 1 : 0;
    return (int64_t)v.size();
}

// ---- test hooks: the fused -E -c, decided and run on the host ----
int krep_b200_regex_count_mode(const search_params_t *P)
{
    std::lock_guard<std::recursive_mutex> lk(engine_mutex());
    Plan *pl = regex_plan_of(P);
    if (!pl) return -1;
    return regex_count_fused(P, pl) ? 1 : 0;
}

int64_t krep_b200_regex_count_host(const search_params_t *P, const char *text, size_t n, uint64_t reach)
{
    std::lock_guard<std::recursive_mutex> lk(engine_mutex());
    Plan *pl = regex_plan_of(P);
    if (!pl || !regex_count_exact(P, pl)) return -1;
    if (regex_returns_early(P)) return 0;
    if (n == 0) return (int64_t)regex_empty_text(P, nullptr);
    if (!text) return 0;
    std::vector<uint64_t> keys;
    const uint64_t device_lines = regex_count_lines_host(*pl->rx, text, n, reach, &keys);
    for (uint64_t &k : keys) k <<= LIT_TAG_BITS;
    return (int64_t)regex_answer(P, RX_COUNT, device_lines, Replay{keys.data(), keys.size(), text, n, 0}, nullptr);
}

// ---- test hooks: split plans (DESIGN §12.7) ----
int krep_b200_regex_automata(const search_params_t *P)
{
    std::lock_guard<std::recursive_mutex> lk(engine_mutex());
    Plan *pl = regex_plan_of(P);
    if (!pl) return -1;
    return pl->rx->groups.empty() ? 1 : (int)pl->rx->groups.size();
}

krep_b200_plan_t *krep_b200_regex_plan_split(const search_params_t *P, uint32_t max_states)
{
    std::lock_guard<std::recursive_mutex> lk(engine_mutex());
    clear_error();
    if (!P || max_states < 3 || max_states > REGEX_MAX_STATES)
    {
        set_error(-3, "krep_b200_regex_plan_split: null params, or a state cap outside [3, %u]", REGEX_MAX_STATES);
        return nullptr;
    }
    std::string why;
    Plan *pl = regex_plan_build(P, &why, max_states); // not in the plan cache: only krep_b200_plan_destroy frees it
    if (!pl) set_error(-3, "this regex has no plan under a cap of %u states (%s)", max_states, why.c_str());
    return reinterpret_cast<krep_b200_plan_t *>(pl);
}

int64_t krep_b200_regex_plan_host(const krep_b200_plan_t *plan_, int mode, const char *text, size_t n, uint64_t reach,
                                  uint64_t *keys, uint64_t cap, uint64_t *device_lines)
{
    std::lock_guard<std::recursive_mutex> lk(engine_mutex());
    clear_error();
    const Plan *plan = reinterpret_cast<const Plan *>(plan_);
    if (!plan || !plan->is_regex || (!text && n) || (cap && !keys) || !regex_mode_available(*plan->rx, mode))
    {
        set_error(-3, "krep_b200_regex_plan_host: bad argument, or mode %d is not available for this plan", mode);
        return -3;
    }
    std::vector<uint64_t> v;
    uint64_t lines = 0;
    switch (mode)
    {
    case RX_FILTER: regex_lines_host(*plan->rx, text, n, &v); break;
    case RX_COUNT: lines = regex_count_lines_host(*plan->rx, text, n, reach, &v); break;
    default: regex_matches_host(*plan->rx, text, n, reach, &v);
    }
    if (mode != RX_OFFSETS)
        for (uint64_t &k : v) k <<= LIT_TAG_BITS;
    for (size_t i = 0; i < v.size() && i < cap; i++) keys[i] = v[i];
    if (device_lines) *device_lines = lines;
    return (int64_t)v.size();
}

// ---- test hooks: -E offsets, decided and run on the host ----
int krep_b200_regex_match_mode(const search_params_t *P)
{
    std::lock_guard<std::recursive_mutex> lk(engine_mutex());
    Plan *pl = regex_plan_of(P);
    if (!pl) return -1;
    return regex_matches_device(P, pl) ? 1 : 0;
}

int64_t krep_b200_regex_matches_host(const search_params_t *P, const char *text, size_t n, uint64_t reach, match_result_t *res)
{
    std::lock_guard<std::recursive_mutex> lk(engine_mutex());
    Plan *pl = regex_plan_of(P);
    if (!pl || !regex_matches_exact(P, pl)) return -1;
    if (regex_returns_early(P)) return 0;
    if (n == 0) return (int64_t)regex_empty_text(P, res);
    if (!text) return 0;
    std::vector<uint64_t> keys;
    regex_matches_host(*pl->rx, text, n, reach, &keys);
    return (int64_t)regex_answer(P, RX_OFFSETS, 0, Replay{keys.data(), keys.size(), text, n, 0}, res);
}

} // extern "C"
