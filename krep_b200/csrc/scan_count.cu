// scan_count.cu — fused `-c` for single literals: the number of distinct lines that hold at least one occurrence,
// computed in the scan itself so that only a count (plus four edge flags per shard) leaves the GPU.
//
// Replaces the count_lines_mode branches of the reference kernels (boyer_moore_search krep.c:1331-1351, kmp_search
// krep.c:1690-1712, memchr_search krep.c:3950-3974, memchr_short_search krep.c:4436-4460, simd_sse42_search
// krep.c:4778-4798): every one of them counts a line the first time it sees an occurrence whose find_line_start
// (krep.c:363) differs from the last counted one, i.e. — for a pattern without a newline in it and any policy that
// eventually looks at every whole-word-valid occurrence — the number of lines containing an occurrence.  The list path
// (k_lit_* + sort + k_line_bounds + host replay) computes the same number at 24 bytes per occurrence; at one
// occurrence per 64 bytes that is more traffic than the text.  Here:
//
//   * the text is cut into PARTITIONS (64 KiB by default); a warp owns a partition and walks it front to back in
//     2 KiB tiles (4 coalesced 16-byte vectors per lane), so "the previous occurrence" is warp-local state;
//   * a 512-byte vector without filter candidates (the streaming loop: same filters as scan_literal.cu) costs
//     nothing extra — newlines are NOT tracked there;
//   * a vector with candidates takes the slow path: candidates verified exactly (per-byte case masks, -w against the
//     global text, ownership by start offset), 16-bit hit and newline masks per lane, and one round of ballots that
//     counts the newline-delimited segments of the vector that hold a hit.  Whether the line that was open when the
//     previous hit was seen has ended in the skipped, candidate-free bytes is settled lazily by scanning just those
//     bytes for a newline (one 512-byte step in ordinary text; bounded by the distance to the previous hit, so O(text)
//     in total whatever the line lengths);
//   * each partition leaves (lines, has_hit, first_open, last_pending, has_nl); these form a monoid under "append",
//     k_count_finish folds them in order into ONE record per shard, and the host folds shard records (staging chunks,
//     devices, ranks) the same way: a line that straddles a cut is counted by both sides, and subtracted once when the
//     left side's last line is still open and the right side's first hit lies before its first newline.
//
// A hit is accounted at its PROXY position (aligned-word filter: the first aligned word inside the occurrence, at most
// 3 bytes after the start); the pattern contains no newline, so proxy and start are on the same line.
#include <algorithm>
#include "engine.h"
#include "line_rec.cuh"
#include "lit_filters.cuh"

namespace kb {

struct CountDev
{
    LitDevParams p;
    uint64_t own_end; // min(shard own_end, avail_len)
    uint32_t part_groups, n_parts;
    uint32_t exact;   // the window filter decides by itself (<= 4 pattern bytes under an exact mask, no -w): no verify loads
    uint32_t tail;    // the vector groups stop short of the owned range (end of the buffer): the last partition's warp
                      // also walks the bytes behind them
    LineRec *recs;
};

struct PartState
{
    uint32_t lines = 0;
    bool has_hit = false, first_open = false, pending = false, seen_nl = false;
    uint64_t covered_to = 0; // newline knowledge is complete for bytes below this
};

__device__ __noinline__ unsigned verify_exact_call(const LitDevParams &p, long long cand) { return verify_exact(p, cand); }

// Is there a newline in bytes [lo, hi)?  Warp-cooperative, 512 bytes per step, stops at the first one.
__device__ __noinline__ bool scan_for_newline(const LitDevParams &p, uint64_t lo, uint64_t hi)
{
    const uint32_t lane = threadIdx.x & 31;
    if (hi > p.avail_len) hi = p.avail_len;
    for (uint64_t base = lo & ~15ull; base < hi; base += 512)
    {
        const uint64_t unit = base + 16ull * lane;
        uint32_t nm = 0;
        if (unit < hi && unit + 16 > lo)
        {
            if (unit + 16 <= p.avail_len) nm = nl_mask16(__ldg(reinterpret_cast<const uint4 *>(p.text + unit)));
            else
                for (uint64_t q = unit; q < p.avail_len; q++) nm |= (p.text[q] == '\n' ? 1u : 0u) << (uint32_t)(q - unit);
            nm &= range_mask16(unit, lo, hi);
        }
        if (__any_sync(0xffffffffu, nm != 0)) return true;
    }
    return false;
}

// Before a span that starts at `upto` is accounted: has the line that was open at covered_to ended in the skipped bytes?
__device__ __forceinline__ void settle(const LitDevParams &p, PartState &S, uint64_t upto)
{
    if (S.covered_to < upto && (S.pending || (!S.has_hit && !S.seen_nl)))
        if (scan_for_newline(p, S.covered_to, upto))
        {
            S.pending = false;
            S.seen_nl = true;
        }
}

// Accounts one span of 32 consecutive units (16 bits each: hm = hits by position, nm = newlines by position, lane order
// = text order; a hit and a newline never share a position).  All of this is warp-uniform.
__device__ __forceinline__ void account(PartState &S, uint32_t hm, uint32_t nm)
{
    const uint32_t lane = threadIdx.x & 31;
    const bool has_nl = nm != 0;
    const uint32_t fnl = has_nl ? (uint32_t)__ffs(nm) - 1 : 0, lnl = has_nl ? 31u - (uint32_t)__clz(nm) : 0;
    const bool f = has_nl && (hm & ((1u << fnl) - 1u)) != 0;  // hits before the unit's first newline
    const bool l = has_nl && ((hm >> lnl) >> 1) != 0;         // hits after its last newline
    uint32_t inner = 0;                                        // segments strictly inside the unit that hold a hit
    if (__popc(nm) >= 2)
    {
        uint32_t prev = fnl, rest = nm & (nm - 1);
        while (rest)
        {
            const uint32_t nx = (uint32_t)__ffs(rest) - 1;
            if (hm & (((1u << nx) - 1u) & ~((2u << prev) - 1u))) inner++;
            prev = nx;
            rest &= rest - 1;
        }
    }
    const uint32_t A = __ballot_sync(0xffffffffu, has_nl), T = __ballot_sync(0xffffffffu, !has_nl && hm != 0);
    const uint32_t F = __ballot_sync(0xffffffffu, f), Lm = __ballot_sync(0xffffffffu, l);
    uint32_t innersum = 0;
    if (__ballot_sync(0xffffffffu, inner != 0)) innersum = __reduce_add_sync(0xffffffffu, inner);
    if (A == 0)
    {
        if (T)
        {
            if (!S.pending)
            {
                S.lines++;
                if (!S.has_hit && !S.seen_nl) S.first_open = true;
            }
            S.pending = true;
            S.has_hit = true;
        }
        return;
    }
    const uint32_t j1 = (uint32_t)__ffs(A) - 1, jr = 31u - (uint32_t)__clz(A);
    if ((T & ((1u << j1) - 1u)) || ((F >> j1) & 1u)) // the segment that was open on entry
    {
        if (!S.pending)
        {
            S.lines++;
            if (!S.has_hit && !S.seen_nl) S.first_open = true;
        }
        S.has_hit = true;
    }
    S.pending = false;
    S.seen_nl = true;
    bool gap = false; // the segment between the previous newline unit's last newline and this unit's first one
    if (has_nl && lane != j1)
    {
        const uint32_t below = A & ((1u << lane) - 1u);
        const uint32_t pj = 31u - (uint32_t)__clz(below);
        const uint32_t between = ((1u << lane) - 1u) & ~((2u << pj) - 1u);
        gap = ((Lm >> pj) & 1u) || (T & between) || f;
    }
    const uint32_t G = __ballot_sync(0xffffffffu, gap);
    S.lines += (uint32_t)__popc(G) + innersum;
    if (G || innersum) S.has_hit = true;
    if (((Lm >> jr) & 1u) || ((T >> jr) >> 1)) // the segment still open on exit
    {
        S.lines++;
        S.has_hit = true;
        S.pending = true;
    }
}

// The accounting state that account() touches, as one scalar, so that the out-of-line copy below passes it in registers.
__device__ __forceinline__ uint64_t pack_state(const PartState &S)
{
    return (uint64_t)S.lines | ((uint64_t)((S.has_hit ? 1u : 0u) | (S.first_open ? 2u : 0u) | (S.pending ? 4u : 0u) | (S.seen_nl ? 8u : 0u)) << 32);
}
__device__ __forceinline__ void unpack_state(uint64_t k, PartState &S)
{
    S.lines = (uint32_t)k;
    const uint32_t f = (uint32_t)(k >> 32);
    S.has_hit = f & 1u;
    S.first_open = f & 2u;
    S.pending = f & 4u;
    S.seen_nl = f & 8u;
}
// One copy of the accounting code for the whole kernel.  Inlined four times per tile (plus the hit-mask code) the kernel
// grew to 5 400 instructions and stalled mostly on instruction fetch; the state and both masks fit into three
// registers, so the call is cheap.
__device__ __noinline__ uint64_t account_call(uint64_t packed, uint32_t hm, uint32_t nm)
{
    PartState S;
    unpack_state(packed, S);
    account(S, hm, nm);
    return pack_state(S);
}

// Exact hit mask of this lane's 16 bytes (bit = position of the hit's proxy byte inside the unit).
template <bool WINDOW>
__device__ __noinline__ uint32_t hit_mask16(const CountDev &D, uint64_t unit, const uint4 &v, uint32_t nx)
{
    const LitDevParams &p = D.p;
    const uint32_t w[5] = {v.x, v.y, v.z, v.w, nx};
    uint32_t hm = 0;
    if (WINDOW)
    {
        const uint32_t mask = p.fold & p.win_mask, k0 = p.K[0];
#pragma unroll
        for (int k = 0; k < 4; k++)
#pragma unroll
            for (int r = 0; r < 4; r++)
            {
                const uint32_t win = r == 0 ? w[k] : __funnelshift_r(w[k], w[k + 1], 8 * r);
                if ((win & mask) == k0)
                {
                    const uint64_t st = unit + 4 * k + r;
                    const bool ok = D.exact ? (st >= p.own_begin && st < p.own_end && st + p.m <= p.avail_len)
                                            : verify_exact_call(p, (long long)st) != 0;
                    if (ok) hm |= 1u << (4 * k + r);
                }
            }
    }
    else
    {
#pragma unroll
        for (int k = 0; k < 4; k++)
#pragma unroll
            for (int d = 0; d < 4; d++)
                if ((w[k] & p.fold) == p.K[d] && verify_exact_call(p, (long long)(unit + 4 * k) - d)) hm |= 1u << (4 * k);
    }
    return hm;
}

// Bytes behind the last full vector of the shard: one byte per lane.
// (state by value in, by value out: a reference would pin the caller's state to local memory for the whole kernel)
__device__ __noinline__ PartState count_tail(const CountDev &D, PartState S, uint64_t cov, uint64_t nl_lo, uint64_t nl_hi, bool window)
{
    const LitDevParams &p = D.p;
    const uint32_t lane = threadIdx.x & 31;
    if (p.avail_len < p.emit_len && cov >= nl_hi) return S;
    const uint64_t last_start = p.avail_len >= p.emit_len ? p.avail_len - p.emit_len : 0;
    uint64_t end = nl_hi > last_start + 1 ? nl_hi : last_start + 1;
    if (!window && end < cov + 1) end = cov + 1; // starts in [cov - 3, cov) are picked up by the lane at cov
    for (uint64_t base = cov; base < end; base += 32)
    {
        settle(p, S, base > nl_lo ? base : nl_lo);
        const uint64_t q = base + lane;
        uint32_t hm = 0, nm = 0;
        if (q < end)
        {
            if (p.avail_len >= p.emit_len && q >= p.tail_start && q <= last_start && verify_exact(p, (long long)q)) hm = 1;
            // aligned-word filter: starts up to 3 bytes before the first uncovered byte have their aligned word here
            if (!window && q == cov && p.avail_len >= p.emit_len)
                for (uint64_t s = p.tail_start; s < cov && s <= last_start; s++)
                    if (verify_exact(p, (long long)s)) hm = 1;
            if (q >= nl_lo && q < nl_hi && q < p.avail_len && p.text[q] == '\n') nm = 1;
            if (nm) hm = 0; // (cannot happen: a pattern byte is not a newline)
        }
        account(S, hm, nm);
        S.covered_to = base + 32;
    }
    return S;
}

#ifndef KREP_B200_COUNT_MINB
#define KREP_B200_COUNT_MINB 3 // resident CTAs per SM the kernel is compiled for (3: 80 registers; 2: 128, no spills)
#endif
template <bool WINDOW, bool FOLD, bool MASKED>
__global__ void __launch_bounds__(256, KREP_B200_COUNT_MINB) k_count_lines(const __grid_constant__ CountDev D)
{
    const LitDevParams &p = D.p;
    const uint4 *__restrict__ t4 = reinterpret_cast<const uint4 *>(p.text);
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t warp_global = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, total_warps = (gridDim.x * blockDim.x) >> 5;
    const uint32_t k0 = p.K[0], k1 = p.K[1], k2 = p.K[2], k3 = p.K[3], fold = p.fold, mask = p.win_mask;
    const uint32_t c1 = p.mulc[0], c2 = p.mulc[1], c3 = p.mulc[2];
    for (uint32_t pi = warp_global; pi < D.n_parts; pi += total_warps)
    {
        const uint64_t ga = p.group_begin + (uint64_t)pi * D.part_groups;
        uint64_t gb = ga + D.part_groups;
        if (gb > p.group_end) gb = p.group_end;
        const bool last_part = pi + 1 == D.n_parts;
        // newlines of [nl_lo, nl_hi) belong to this partition (the partitions' ranges tile the owned range)
        const uint64_t nl_lo = ga * 16 > p.own_begin ? ga * 16 : p.own_begin;
        const uint64_t nl_hi = (last_part || gb * 16 > D.own_end) ? D.own_end : gb * 16;
        PartState S;
        S.covered_to = nl_lo;
        for (uint64_t g = ga; g < gb; g += 128)
        {
            uint4 v[4];
            uint32_t nx[4];
            bool ok[4];
#pragma unroll
            for (int u = 0; u < 4; u++)
            {
                const uint64_t gi = g + 32 * u + lane;
                ok[u] = gi < gb;
                v[u] = ok[u] ? ld_stream(t4 + gi) : make_uint4(0u, 0u, 0u, 0u);
                nx[u] = 0;
                if (WINDOW && ok[u] && (lane == 31 || gi + 1 >= gb)) nx[u] = __ldg(reinterpret_cast<const uint32_t *>(t4 + gi + 1));
            }
            uint32_t cand = 0;
#pragma unroll
            for (int u = 0; u < 4; u++)
            {
                bool h;
                if (WINDOW)
                {
                    const uint32_t nb = __shfl_down_sync(0xffffffffu, v[u].x, 1);
                    if (!(lane == 31 || g + 32 * u + lane + 1 >= gb)) nx[u] = nb;
                    h = hit_vec_w<FOLD, MASKED>(v[u], nx[u], fold, mask, k0, c1, c2, c3);
                }
                else
                    h = hit_vec<FOLD>(v[u], fold, k0, k1, k2, k3);
                cand |= (h && ok[u]) ? (1u << u) : 0u;
            }
            const uint32_t any = __reduce_or_sync(0xffffffffu, cand);
            if (any)
            {
                // A tile with a candidate is accounted as a whole, in place: hit masks for the vectors that have candidates,
                // newline masks for all four (from the registers), one round of ballots per vector.  Only the gap between the
                // previous accounted tile and this one may need memory (settle), and only while a line is open.
                const uint64_t tile_lo = g * 16;
                settle(p, S, tile_lo > nl_lo ? tile_lo : nl_lo);
                const bool inside = tile_lo >= nl_lo && tile_lo + 2048 <= nl_hi;
                uint64_t st = pack_state(S);
#pragma unroll
                for (int u = 0; u < 4; u++)
                {
                    const uint64_t unit = tile_lo + 512ull * u + 16ull * lane;
                    uint32_t hm = 0, nm = 0;
                    if (ok[u])
                    {
                        if ((cand >> u) & 1u) hm = hit_mask16<WINDOW>(D, unit, v[u], nx[u]);
                        nm = nl_mask16(v[u]);
                        if (!inside) nm &= range_mask16(unit, nl_lo, nl_hi);
                    }
                    st = account_call(st, hm, nm);
                }
                unpack_state(st, S);
                S.covered_to = tile_lo + 2048;
            }
        }
        if (last_part && D.tail) S = count_tail(D, S, gb * 16, nl_lo, nl_hi, WINDOW);
        // close the partition
        uint32_t flags = 0;
        if (S.has_hit)
        {
            if (S.pending && S.covered_to < nl_hi && scan_for_newline(p, S.covered_to, nl_hi)) S.pending = false;
            flags = LR_HAS_HIT | (S.first_open ? LR_FIRST_OPEN : 0u) | (S.pending ? LR_LAST_PENDING : 0u) | LR_HAS_NL;
        }
        else
        {
            const bool nl = S.seen_nl || (S.covered_to < nl_hi && scan_for_newline(p, S.covered_to, nl_hi));
            flags = nl ? LR_HAS_NL : 0u;
        }
        if (lane == 0) D.recs[pi] = LineRec{S.lines, flags};
    }
}

// Folds the partition records, in order, into one shard record: each thread folds a contiguous slice, thread 0 folds the
// 1024 partial results.
__global__ void __launch_bounds__(1024) k_count_finish(const LineRec *recs, uint32_t n, uint64_t *d_out, uint64_t *h_out)
{
    __shared__ uint64_t s_lines[1024];
    __shared__ uint32_t s_flags[1024];
    const uint32_t per = (n + blockDim.x - 1) / blockDim.x;
    const uint32_t a = threadIdx.x * per, b = a + per < n ? a + per : n;
    uint64_t lines = 0;
    uint32_t flags = 0;
    for (uint32_t i = a; i < b; i++) append_rec(lines, flags, recs[i].lines, recs[i].flags);
    s_lines[threadIdx.x] = lines;
    s_flags[threadIdx.x] = flags;
    __syncthreads();
    if (threadIdx.x == 0)
    {
        lines = 0;
        flags = 0;
        for (uint32_t t = 0; t < blockDim.x; t++) append_rec(lines, flags, s_lines[t], s_flags[t]);
        d_out[0] = lines;
        d_out[1] = flags;
        h_out[0] = lines;
        h_out[1] = flags;
    }
}

// ---------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------
#define CKC(call)                                                                                  \
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

// Does the fused count give exactly what the emulated kernel's -c replay gives?  (See the header comment; the window
// kernels' tail sub-search recounts a straddling line, tag-mode -w plans need the cursor walk, prefix plans are -o.
// Pattern sets: scan_set_count.cu, as long as no pattern holds a newline.)
bool count_lines_eligible(const Plan *plan, const search_params_t *P, int algo)
{
    if (!P->count_lines_mode || plan->is_regex || plan->whole_word == 2) return false;
    if (plan->is_ac)
    {
        for (const std::string &s : plan->patterns)
            if (s.find('\n') != std::string::npos) return false;
        return true;
    }
    if (plan->emit_len != plan->m) return false;
    if (plan->pattern.find('\n') != std::string::npos) return false;
    return algo == KREP_B200_ALGO_BMH || algo == KREP_B200_ALGO_KMP || algo == KREP_B200_ALGO_MEMCHR ||
           algo == KREP_B200_ALGO_MEMCHR_SHORT || algo == KREP_B200_ALGO_SSE42;
}

int ensure_line_out(DevCtx &E, uint64_t n)
{
    if (n <= E.line_out_cap) return 0;
    CKC(cudaDeviceSynchronize());
    cudaFree(E.d_line_out);
    cudaFreeHost(E.h_line_out);
    E.d_line_out = nullptr;
    E.h_line_out = nullptr;
    E.line_out_cap = 0;
    uint64_t cap = 64;
    while (cap < n) cap *= 2;
    CKC(cudaMalloc(&E.d_line_out, cap * 2 * sizeof(uint64_t)));
    CKC(cudaHostAlloc(&E.h_line_out, cap * 2 * sizeof(uint64_t), cudaHostAllocMapped | cudaHostAllocPortable));
    E.line_out_cap = cap;
    return 0;
}

// Enqueues the fused count of one shard on `stream`; its record lands in E.h_line_out[2*index .. 2*index+1] (mapped pinned
// memory: readable after the stream is synchronised) and E.d_line_out likewise.  A pattern set's count waits for its
// scan's occurrence count on the host before it enqueues the rest (scan_set_count.cu).
int launch_count_lines(DevCtx &E, const Plan *plan, const krep_b200_shard_t *sh, cudaStream_t stream, uint64_t index)
{
    if (((uintptr_t)sh->d_text & 15) != 0)
    {
        set_error(-3, "shard text pointer must be 16-byte aligned");
        return -3;
    }
    const PlanDev *pd = plan_on_device(plan, E);
    if (!pd) return -2;
    if (ensure_line_out(E, index + 1) != 0) return -2;
    if (plan->is_ac)
    {
        const int slot = set_count_slot(E);
        const int rc = set_count_begin(E, plan, sh, stream, slot);
        return rc != 0 ? rc : set_count_end(E, plan, sh, stream, slot, index);
    }
    CountDev D;
    memset(&D, 0, sizeof D);
    LitDevParams &p = D.p;
    const uint64_t own_end = sh->own_end < sh->avail_len ? sh->own_end : sh->avail_len;
    p.text = (const uint8_t *)sh->d_text;
    p.avail_len = sh->avail_len;
    p.own_begin = sh->own_begin;
    p.own_end = own_end;
    p.global_offset = sh->global_offset;
    p.prev_byte = sh->prev_byte;
    p.next_byte = sh->next_byte;
    uint64_t total_groups;
    const bool window = plan->filter == FILTER_WINDOW4;
    if (!window)
    {
        total_groups = sh->avail_len / 16;
        p.tail_start = total_groups ? total_groups * 16 - 3 : 0;
    }
    else
    {
        total_groups = sh->avail_len >= 20 ? (sh->avail_len - 20) / 16 + 1 : 0;
        p.tail_start = total_groups * 16;
    }
    p.group_begin = sh->own_begin / 16;
    p.group_end = (own_end + 2) / 16 + 1;
    D.tail = p.group_end > total_groups ? 1u : 0u;
    if (p.group_end > total_groups) p.group_end = total_groups;
    if (p.group_begin > p.group_end) p.group_begin = p.group_end;
    p.m = plan->m;
    p.emit_len = plan->emit_len;
    for (int d = 0; d < 4; d++) p.K[d] = plan->K[d];
    p.fold = plan->fold;
    p.win_mask = plan->win_mask;
    p.mulc[0] = 1u << 24;
    p.mulc[1] = 1u << 16;
    p.mulc[2] = 1u << 8;
    p.pat_val = pd->d_pat_val;
    p.pat_mask = pd->d_pat_mask;
    p.whole_word = plan->whole_word;
    D.own_end = own_end;
    {
        bool letters = true;
        for (unsigned char ch : plan->pattern) letters &= is_alpha_c(ch);
        D.exact = (window && plan->m <= 4 && plan->whole_word == 0 && (plan->case_sensitive || letters)) ? 1u : 0u;
    }
    const uint64_t groups = p.group_end - p.group_begin;
    // read on every launch (getenv is nothing next to a launch), so that a process can change the partition size
    const char *v = getenv("KREP_B200_COUNT_PART_KB");
    const uint32_t kb_ = v && atoi(v) > 0 ? (uint32_t)atoi(v) : 64;
    uint64_t part = std::max<uint32_t>(128, kb_ * 64 / 128 * 128); // groups, a multiple of the 128-group tile
    const uint64_t max_parts = 1u << 18;
    if ((groups + part - 1) / part > max_parts) part = ((groups + max_parts - 1) / max_parts + 127) / 128 * 128;
    D.part_groups = (uint32_t)part;
    D.n_parts = (uint32_t)std::max<uint64_t>((groups + part - 1) / part, 1);
    if (D.n_parts > E.line_recs_cap)
    {
        CKC(cudaStreamSynchronize(stream));
        cudaFree(E.d_line_recs);
        E.d_line_recs = nullptr;
        E.line_recs_cap = 0;
        const uint64_t cap = std::max<uint64_t>(D.n_parts, 1u << 16);
        CKC(cudaMalloc(&E.d_line_recs, cap * sizeof(LineRec)));
        E.line_recs_cap = cap;
    }
    D.recs = (LineRec *)E.d_line_recs;
    const bool folded = plan->fold != 0xFFFFFFFFu, masked = plan->win_mask != 0xFFFFFFFFu;
    const uint64_t want_blocks = ((uint64_t)D.n_parts + 7) / 8;
    const unsigned grid = (unsigned)std::min<uint64_t>(want_blocks, (uint64_t)E.sm_count * KREP_B200_COUNT_MINB);
    if (!window)
    {
        if (folded) k_count_lines<false, true, false><<<grid, 256, 0, stream>>>(D);
        else k_count_lines<false, false, false><<<grid, 256, 0, stream>>>(D);
    }
    else if (folded)
    {
        if (masked) k_count_lines<true, true, true><<<grid, 256, 0, stream>>>(D);
        else k_count_lines<true, true, false><<<grid, 256, 0, stream>>>(D);
    }
    else
    {
        if (masked) k_count_lines<true, false, true><<<grid, 256, 0, stream>>>(D);
        else k_count_lines<true, false, false><<<grid, 256, 0, stream>>>(D);
    }
    CKC(cudaGetLastError());
    k_count_finish<<<1, 1024, 0, stream>>>(D.recs, D.n_parts, E.d_line_out + 2 * index, E.h_line_out + 2 * index);
    CKC(cudaGetLastError());
    count_launch(2);
    return 0;
}

// Folds shard records (text order) into the number of matching lines.
uint64_t combine_line_records(const uint64_t *recs, size_t n)
{
    uint64_t lines = 0;
    uint32_t flags = 0;
    for (size_t i = 0; i < n; i++) append_rec(lines, flags, recs[2 * i], (uint32_t)recs[2 * i + 1]);
    return lines;
}

} // namespace kb
