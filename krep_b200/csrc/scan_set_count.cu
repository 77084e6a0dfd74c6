// scan_set_count.cu — fused `-c` for pattern sets (-f, several -e): the line record of a shard (scan_count.cu's LineRec)
// computed from its sorted occurrence keys on the device, so that neither the keys nor their line bounds leave the GPU.
//
// aho_corasick_search (aho_corasick.c:390-403) walks occurrences in the order of their end and counts one when the line
// of its start differs from the last line it counted; -w is applied before that test and -m caps the count.  When no
// pattern holds a '\n', an occurrence's start and its last byte lie on one line, and those lines never decrease in end
// order, so the count is min(lines that hold an occurrence, max_count): the quantity the literal fused count computes.
// The same record monoid therefore folds it across staging chunks, ranges, devices, shards and ranks, cut at any byte.
//
//   * the shard is scanned by the pattern-set kernels into a slot's occurrence list like any other scan; k_finish
//     publishes the count (and rank-sorts a short list on the device), CUB sorts a longer one;
//   * k_set_lines walks the sorted keys, ordered by end: key i opens a new line exactly when a '\n' lies between the
//     last byte of key i-1 and the start of key i.  A lane looks at the first 64 bytes of that gap itself; a gap that is
//     longer and holds no newline there is searched by the whole warp, which stops at its first newline.  No byte lies
//     in two gaps, so the work is bounded by the text whatever the density or the line lengths;
//   * the flags come from the first and the last key and the owned range: FIRST_OPEN when no newline lies between
//     own_begin and the first key's start, LAST_PENDING when none lies between the last key's last byte and own_end (an
//     occurrence that straddles own_end leaves its line pending); a range without keys only needs HAS_NL;
//   * a shard whose occurrences do not fit the list is not given a longer list: its owned range is cut into pieces whose
//     lists fit, and their records are folded in order.
#include <algorithm>
#include "engine.h"
#include "line_rec.cuh"

namespace kb {

#define CKS(call)                                                                                  \
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

struct SetLinesDev
{
    const uint64_t *keys; // sorted (AC layout, csrc/common.h)
    uint64_t n;
    const uint8_t *text;  // the shard's buffer, 16-byte aligned
    uint64_t avail_len, global_offset, own_begin, own_end;
    unsigned long long *acc; // [0] keys after the first that open a new line, [1] flags
};

static constexpr uint32_t SET_THREADS = 256;
static constexpr uint32_t SET_ROUNDS = 4;      // keys per lane: a warp takes 32 * SET_ROUNDS consecutive keys
static constexpr uint32_t SET_LANE_UNITS = 4;  // 16-byte units of a gap a lane searches on its own

__device__ __forceinline__ uint64_t key_last(const SetLinesDev &D, uint64_t key)
{
    return (key >> AC_END_SHIFT) - D.global_offset - 1;
}
__device__ __forceinline__ uint64_t key_first(const SetLinesDev &D, uint64_t key)
{
    return (key >> AC_END_SHIFT) - (1024 - ((key >> AC_LEN_SHIFT) & 1023)) - D.global_offset;
}

// newline bits of the 16 bytes at `unit` (a multiple of 16) that lie inside [lo, hi)
__device__ __forceinline__ uint32_t nl_unit(const SetLinesDev &D, uint64_t unit, uint64_t lo, uint64_t hi)
{
    uint32_t nm = 0;
    if (unit + 16 <= D.avail_len) nm = nl_mask16(__ldg(reinterpret_cast<const uint4 *>(D.text + unit)));
    else
        for (uint64_t q = unit; q < D.avail_len; q++) nm |= (D.text[q] == '\n' ? 1u : 0u) << (uint32_t)(q - unit);
    return nm & range_mask16(unit, lo, hi);
}

// Is there a newline in [lo, hi)?  The whole warp (lo, hi warp-uniform), 2 KiB per step, stops at the first one.
__device__ __noinline__ bool warp_has_nl(const SetLinesDev &D, uint64_t lo, uint64_t hi)
{
    const uint32_t lane = threadIdx.x & 31;
    for (uint64_t base = lo & ~15ull; base < hi; base += 2048)
    {
        uint32_t nm = 0;
#pragma unroll
        for (uint32_t u = 0; u < 4; u++)
        {
            const uint64_t unit = base + 512ull * u + 16ull * lane;
            if (unit < hi) nm |= nl_unit(D, unit, lo, hi);
        }
        if (__any_sync(0xffffffffu, nm != 0)) return true;
    }
    return false;
}

// One lane's look at the gap [lo, hi): 1 = it holds a newline, 0 = it does not, 2 = undecided (*lo is then moved past
// the bytes looked at).
__device__ __forceinline__ uint32_t lane_gap(const SetLinesDev &D, uint64_t &lo, uint64_t hi)
{
    const uint64_t a = lo & ~15ull;
#pragma unroll
    for (uint32_t u = 0; u < SET_LANE_UNITS; u++)
    {
        const uint64_t unit = a + 16ull * u;
        if (unit >= hi) return 0;
        if (nl_unit(D, unit, lo, hi)) return 1;
    }
    lo = a + 16ull * SET_LANE_UNITS;
    return lo >= hi ? 0u : 2u;
}

__global__ void __launch_bounds__(SET_THREADS) k_set_lines(const __grid_constant__ SetLinesDev D)
{
    const uint32_t lane = threadIdx.x & 31;
    const uint64_t warp = ((uint64_t)blockIdx.x * SET_THREADS + threadIdx.x) >> 5;
    if (warp == 0)
    {
        uint32_t flags;
        if (D.n == 0) flags = warp_has_nl(D, D.own_begin, D.own_end) ? LR_HAS_NL : 0u;
        else
        {
            flags = LR_HAS_HIT | LR_HAS_NL;
            if (!warp_has_nl(D, D.own_begin, key_first(D, D.keys[0]))) flags |= LR_FIRST_OPEN;
            const uint64_t last = key_last(D, D.keys[D.n - 1]);
            if (last + 1 >= D.own_end || !warp_has_nl(D, last + 1, D.own_end)) flags |= LR_LAST_PENDING;
        }
        if (lane == 0) D.acc[1] = flags;
    }
    const uint64_t base = warp * (32ull * SET_ROUNDS);
    if (base >= D.n) return;
    uint32_t opened = 0;
#pragma unroll 1
    for (uint32_t r = 0; r < SET_ROUNDS; r++)
    {
        const uint64_t i = base + 32ull * r + lane;
        const bool live = i < D.n;
        const uint64_t k = live ? D.keys[i] : 0;
        uint64_t kp = __shfl_up_sync(0xffffffffu, k, 1);
        if (lane == 0 && live && i > 0) kp = D.keys[i - 1];
        uint64_t lo = 0, hi = 0;
        uint32_t v = 0;
        if (live && i > 0)
        {
            lo = key_last(D, kp) + 1;
            hi = key_first(D, k);
            if (lo < hi) v = lane_gap(D, lo, hi);
        }
        // the gaps no lane could settle: one warp-wide search each
        for (uint32_t u = __ballot_sync(0xffffffffu, v == 2); u; u &= u - 1)
        {
            const uint32_t src = (uint32_t)__ffs(u) - 1;
            const bool f = warp_has_nl(D, __shfl_sync(0xffffffffu, lo, src), __shfl_sync(0xffffffffu, hi, src));
            if (lane == src) v = f ? 1u : 0u;
        }
        opened += v;
    }
    opened = __reduce_add_sync(0xffffffffu, opened);
    if (lane == 0 && opened) atomicAdd(D.acc, (unsigned long long)opened);
}

// The record of n keys from the accumulators, written where launch_count_lines' records go; leaves them at zero.
__global__ void k_set_record(unsigned long long *acc, uint64_t n, uint64_t *d_out, uint64_t *h_out)
{
    const uint64_t lines = n ? acc[0] + 1 : 0, flags = acc[1];
    d_out[0] = lines;
    d_out[1] = flags;
    h_out[0] = lines;
    h_out[1] = flags;
    acc[0] = 0;
    acc[1] = 0;
}

int set_count_slot(const DevCtx &E) { return E.pend[0].active ? 1 : 0; }

int set_count_begin(DevCtx &E, const Plan *plan, const krep_b200_shard_t *sh, cudaStream_t st, int slot)
{
    if (E.pend[slot].active)
    {
        set_error(-3, "pattern-set -c: %d scans begun with krep_b200_scan_shard_begin are still in flight on device %d; end "
                      "them first", SCAN_SLOTS, E.device);
        return -3;
    }
    if (ensure_keys(E, 1) != 0) return -2;
    CKS(cudaStreamWaitEvent(st, E.ev_done[slot], 0));
    if (reset_counter(E, slot, st) != 0) return -2;
    const int rc = launch_scan(E, plan, sh, 1, st, slot);
    if (rc != 0) return rc;
    return finish_scan(E, slot, 1, st, false) != 0 ? -2 : 0;
}

// Enqueues k_set_lines over the cnt keys of the scan in `slot` (sorted by k_finish or by CUB) and the record at `index`.
static int set_lines(DevCtx &E, const Plan *plan, const krep_b200_shard_t *sh, cudaStream_t st, int slot, uint64_t cnt,
                     uint64_t index)
{
    const uint64_t *keys = E.d_pack[slot] + 1;
    if (cnt > PACK_KEYS && sort_keys(E, slot, cnt, key_end_bit(plan, sh->global_offset + sh->avail_len), st, &keys) != 0)
        return -2;
    if (!E.d_set_acc)
    {
        CKS(cudaMalloc(&E.d_set_acc, 2 * sizeof(unsigned long long)));
        CKS(cudaMemset(E.d_set_acc, 0, 2 * sizeof(unsigned long long)));
    }
    SetLinesDev D;
    D.keys = keys;
    D.n = cnt;
    D.text = (const uint8_t *)sh->d_text;
    D.avail_len = sh->avail_len;
    D.global_offset = sh->global_offset;
    D.own_begin = sh->own_begin;
    D.own_end = std::min(sh->own_end, sh->avail_len);
    D.acc = E.d_set_acc;
    const uint64_t per_block = SET_THREADS * SET_ROUNDS;
    const unsigned grid = (unsigned)std::max<uint64_t>((cnt + per_block - 1) / per_block, 1);
    k_set_lines<<<grid, SET_THREADS, 0, st>>>(D);
    CKS(cudaGetLastError());
    k_set_record<<<1, 1, 0, st>>>(E.d_set_acc, cnt, E.d_line_out + 2 * index, E.h_line_out + 2 * index);
    CKS(cudaGetLastError());
    count_launch(2);
    return 0;
}

// The record of owned range [b, e) of the shard, whose cnt occurrences overflow the list, folded into (lines, flags):
// the range is cut into pieces of equal length that would each fill half the list at the range's mean density; each is
// scanned and counted on its own (one that still overflows is cut again), in text order.  Synchronous.
static int set_count_pieces(DevCtx &E, const Plan *plan, const krep_b200_shard_t &sh, cudaStream_t st, int slot, uint64_t index,
                            uint64_t b, uint64_t e, uint64_t cnt, uint64_t *lines, uint32_t *flags)
{
    const uint64_t pieces = std::max<uint64_t>(2, (2 * cnt + E.key_cap - 1) / E.key_cap);
    const uint64_t step = (e - b + pieces - 1) / pieces;
    for (uint64_t pb = b; pb < e; pb += step)
    {
        krep_b200_shard_t part = sh;
        part.own_begin = pb;
        part.own_end = std::min(pb + step, e);
        int rc = set_count_begin(E, plan, &part, st, slot);
        if (rc != 0) return rc;
        CKS(cudaEventSynchronize(E.ev_done[slot]));
        const uint64_t c = E.h_pack[slot][0];
        // a single byte starts at most AC_MAX_PATTERNS occurrences, fewer than the list holds: the cuts end
        if (c > E.key_cap) rc = set_count_pieces(E, plan, part, st, slot, index, part.own_begin, part.own_end, c, lines, flags);
        else if ((rc = set_lines(E, plan, &part, st, slot, c, index)) == 0)
        {
            CKS(cudaStreamSynchronize(st));
            append_rec(*lines, *flags, E.h_line_out[2 * index], (uint32_t)E.h_line_out[2 * index + 1]);
        }
        if (rc != 0) return rc;
    }
    return 0;
}

int set_count_end(DevCtx &E, const Plan *plan, const krep_b200_shard_t *sh, cudaStream_t st, int slot, uint64_t index)
{
    CKS(cudaEventSynchronize(E.ev_done[slot]));
    const uint64_t cnt = E.h_pack[slot][0];
    if (cnt <= E.key_cap) return set_lines(E, plan, sh, st, slot, cnt, index);
    trace("set count: %llu occurrences overflow the %llu-key list: counted in pieces", (unsigned long long)cnt,
          (unsigned long long)E.key_cap);
    uint64_t lines = 0;
    uint32_t flags = 0;
    const int rc = set_count_pieces(E, plan, *sh, st, slot, index, sh->own_begin, std::min(sh->own_end, sh->avail_len), cnt,
                                    &lines, &flags);
    if (rc != 0) return rc;
    E.h_line_out[2 * index] = lines;
    E.h_line_out[2 * index + 1] = flags;
    CKS(cudaMemcpyAsync(E.d_line_out + 2 * index, E.h_line_out + 2 * index, 2 * sizeof(uint64_t), cudaMemcpyHostToDevice, st));
    return 0;
}

} // namespace kb
