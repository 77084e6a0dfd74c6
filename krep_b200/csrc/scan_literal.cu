// scan_literal.cu — single-literal scan kernels for sm_90a.
//
// Replaces the inner loops of boyer_moore_search (krep.c:1294-1382), kmp_search (krep.c:1663-1763),
// memchr_search / memchr_short_search (krep.c:3918-4023, 4396-4500) and the simd_* searches
// (krep.c:4737-4866, 4914-5056, 5145-5255).  All of those enumerate the occurrences of one literal;
// they differ only in which occurrences they keep afterwards (overlap policy, -w, -c, -m), which
// semantics.cpp replays over the sorted occurrence list.  So the device work is one thing:
// emit every position where the literal occurs, exactly once, at HBM speed.
//
// Design (HBM-bound byte scan, no tensor cores — nothing here is a contraction):
//   * every thread streams 16-byte vectors (LDG.128, coalesced: a warp reads 512 contiguous bytes),
//     UNROLL vectors in flight per thread; the grid is sized to the SM count x resident CTAs and walks
//     the shard with a grid stride, so neighbouring CTAs read neighbouring DRAM pages;
//   * the hot loop only FILTERS, with ~1 integer op per corpus byte:
//       ALIGNED4 (pattern_len >= 7): an occurrence at p fully contains the aligned word j = ceil(p/4),
//         which then equals P[d..d+4) with d = 4j-p in 0..3.  Each aligned text word is compared with
//         those four constants — no halo, no shuffles, no shared memory; case-insensitive search ANDs
//         the word with 0xDFDFDFDF first (a superset filter: folds letters exactly, aliases a few
//         punctuation bytes, verified exactly afterwards);
//       WINDOW4 (pattern_len < 7): the 4-byte window at every byte offset, built with funnel shifts from
//         the thread's own words plus the first word of the next vector, is compared with P[0..4) under a
//         length mask;
//   * a thread whose vector contains a candidate (rare) calls the out-of-line verifier, which compares
//     all pattern bytes under the exact per-byte case mask, evaluates the whole-word boundary against the
//     global text (shard context bytes at the edges, so results equal the reference's single-chunk run,
//     SURVEY §8 a12), checks shard ownership by start offset and appends one 64-bit key.
//
// Algorithmic traffic: 1 byte read per corpus byte (+ 8 B written per occurrence).
#include <mutex>
#include "common.h"
#include "lit_filters.cuh"

#ifndef KREP_B200_WARP_EMIT
#define KREP_B200_WARP_EMIT 1 // 1: warp-cooperative emission (one atomicAdd per warp and vector); 0: one per occurrence
#endif

namespace kb {

// Exact check of one candidate start + emission. Out of line on purpose: keeps the streaming loop's
// register footprint small; executed for a vanishing fraction of positions on low-hit-rate corpora.
// Returns 1 when the occurrence was only counted (count-only launch), else 0.
__device__ __noinline__ unsigned verify_emit(const LitDevParams &p, long long cand)
{
    const unsigned tag = verify_exact(p, cand);
    if (!tag) return 0;
    if (p.want_positions)
    {
        const unsigned long long slot = atomicAdd(p.counter, 1ULL);
        if (slot < p.cap) p.out[slot] = ((p.global_offset + (uint64_t)cand) << LIT_TAG_BITS) | (tag & 7u);
        return 0;
    }
    return 1;
}

__device__ __noinline__ unsigned slow_aligned4(const LitDevParams &p, uint64_t group, uint4 v)
{
    unsigned n = 0;
    const uint32_t w[4] = {v.x & p.fold, v.y & p.fold, v.z & p.fold, v.w & p.fold};
#pragma unroll
    for (int k = 0; k < 4; k++)
#pragma unroll
        for (int d = 0; d < 4; d++)
            if (w[k] == p.K[d]) n += verify_emit(p, (long long)(group * 16 + 4 * k) - d);
    return n;
}

// Warp-cooperative emission for one 16-byte vector per lane (all 32 lanes call; `mine` = this lane's vector holds a filter
// candidate).  Each lane verifies its own candidates exactly; then the warp reserves ONE contiguous run of the occurrence
// list — one atomicAdd per warp and vector instead of one per occurrence: the ballot / prefix-sum compaction of match
// offsets — and every lane writes its keys at its prefix offset.  On low-hit-rate corpora this costs what the old
// per-lane path did (the warp diverged for the one lane anyway); at one occurrence per 64 bytes it issues 8x fewer
// atomics on the one counter.  Returns the lane's occurrence count when the launch only counts.
template <bool WINDOW>
__device__ __noinline__ unsigned emit_warp(const LitDevParams &p, uint64_t group, uint4 v, uint32_t nx, bool mine)
{
    const uint32_t lane = threadIdx.x & 31;
    uint32_t valid = 0; // bit i: candidate i is an occurrence (WINDOW: start = 16g + i; else i = 4k + d: start = 16g + 4k - d)
    uint64_t tags = 0;  // 3 tag bits per candidate (full, ws_ok, we_ok)
    if (mine)
    {
        const uint32_t w[5] = {v.x, v.y, v.z, v.w, nx};
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
                        const unsigned t = verify_exact(p, (long long)(group * 16 + 4 * k + r));
                        if (t)
                        {
                            valid |= 1u << (4 * k + r);
                            tags |= (uint64_t)(t & 7u) << (3 * (4 * k + r));
                        }
                    }
                }
        }
        else
        {
#pragma unroll
            for (int k = 0; k < 4; k++)
#pragma unroll
                for (int d = 0; d < 4; d++)
                    if ((w[k] & p.fold) == p.K[d])
                    {
                        const unsigned t = verify_exact(p, (long long)(group * 16 + 4 * k) - d);
                        if (t)
                        {
                            valid |= 1u << (4 * k + d);
                            tags |= (uint64_t)(t & 7u) << (3 * (4 * k + d));
                        }
                    }
        }
    }
    const uint32_t n = (uint32_t)__popc(valid);
    if (!p.want_positions) return n;
    uint32_t incl = n;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1)
    {
        const uint32_t t = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= (uint32_t)o) incl += t;
    }
    const uint32_t total = __shfl_sync(0xffffffffu, incl, 31);
    if (total == 0) return 0;
    unsigned long long base = 0;
    if (lane == 31) base = atomicAdd(p.counter, (unsigned long long)total);
    base = __shfl_sync(0xffffffffu, base, 31);
    unsigned long long slot = base + (incl - n);
    while (valid)
    {
        const uint32_t i = (uint32_t)__ffs(valid) - 1;
        valid &= valid - 1;
        const long long start = WINDOW ? (long long)(group * 16 + i) : (long long)(group * 16 + (i & ~3u)) - (long long)(i & 3u);
        if (slot < p.cap) p.out[slot] = ((p.global_offset + (uint64_t)start) << LIT_TAG_BITS) | ((tags >> (3 * i)) & 7u);
        slot++;
    }
    return 0;
}

__device__ __forceinline__ void tail_and_count(const LitDevParams &p, unsigned long long local_cnt)
{
    if (blockIdx.x == 0 && threadIdx.x < 32 && p.avail_len >= p.emit_len)
    {
        const uint64_t last = p.avail_len - p.emit_len;
        for (uint64_t s = p.tail_start + threadIdx.x; s <= last; s += 32) local_cnt += verify_emit(p, (long long)s);
    }
    if (!p.want_positions)
    {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) local_cnt += __shfl_xor_sync(0xffffffffu, local_cnt, o);
        if ((threadIdx.x & 31) == 0 && local_cnt) atomicAdd(p.counter, local_cnt);
    }
}

template <bool FOLD, int UNROLL>
__global__ void __launch_bounds__(256, 4) k_lit_aligned4(const __grid_constant__ LitDevParams p)
{
    const uint4 *__restrict__ t4 = reinterpret_cast<const uint4 *>(p.text);
    const uint32_t k0 = p.K[0], k1 = p.K[1], k2 = p.K[2], k3 = p.K[3], fold = p.fold;
    unsigned long long local_cnt = 0;
    const uint64_t tile = (uint64_t)blockDim.x * UNROLL;
    const uint64_t stride = (uint64_t)gridDim.x * tile;
    uint64_t g0 = p.group_begin + (uint64_t)blockIdx.x * tile;
    for (; g0 + tile <= p.group_end; g0 += stride)
    {
        uint4 v[UNROLL];
#pragma unroll
        for (int u = 0; u < UNROLL; u++) v[u] = ld_stream(t4 + g0 + (uint64_t)u * blockDim.x + threadIdx.x);
        bool hit = false;
#pragma unroll
        for (int u = 0; u < UNROLL; u++) hit |= hit_vec<FOLD>(v[u], fold, k0, k1, k2, k3);
#if KREP_B200_WARP_EMIT
        if (__any_sync(0xffffffffu, hit)) // rare; the whole warp goes (full tiles: all 32 lanes are here)
        {
#pragma unroll
            for (int u = 0; u < UNROLL; u++)
            {
                const bool mine = hit_vec<FOLD>(v[u], fold, k0, k1, k2, k3);
                if (__any_sync(0xffffffffu, mine))
                    local_cnt += emit_warp<false>(p, g0 + (uint64_t)u * blockDim.x + threadIdx.x, v[u], 0u, mine);
            }
        }
#else
        if (hit)
        {
#pragma unroll
            for (int u = 0; u < UNROLL; u++)
                if (hit_vec<FOLD>(v[u], fold, k0, k1, k2, k3))
                    local_cnt += slow_aligned4(p, g0 + (uint64_t)u * blockDim.x + threadIdx.x, v[u]);
        }
#endif
    }
    if (g0 < p.group_end) // the one ragged tile
    {
        for (int u = 0; u < UNROLL; u++)
        {
            const uint64_t g = g0 + (uint64_t)u * blockDim.x + threadIdx.x;
            if (g < p.group_end)
            {
                const uint4 v = ld_stream(t4 + g);
                if (hit_vec<FOLD>(v, fold, k0, k1, k2, k3)) local_cnt += slow_aligned4(p, g, v);
            }
        }
    }
    tail_and_count(p, local_cnt);
}

__device__ __noinline__ unsigned slow_window4(const LitDevParams &p, uint64_t group, uint4 v, uint32_t nx)
{
    unsigned n = 0;
    const uint32_t w[5] = {v.x, v.y, v.z, v.w, nx};
    const uint32_t mask = p.fold & p.win_mask, k0 = p.K[0];
#pragma unroll
    for (int k = 0; k < 4; k++)
#pragma unroll
        for (int r = 0; r < 4; r++)
        {
            const uint32_t win = r == 0 ? w[k] : __funnelshift_r(w[k], w[k + 1], 8 * r);
            if ((win & mask) == k0) n += verify_emit(p, (long long)(group * 16 + 4 * k + r));
        }
    return n;
}

// Main loads of the window kernel: the sector that holds a warp's "next word" is touched twice (once as lane 31's
// next-word load, once as the following warp's vector), so these loads keep the default L2 policy instead of
// evict-first; KREP_B200_W4_CS=1 at build time restores the streaming hint for comparison.
// On the H100 a second load per lane is what limits the window kernel: with every lane loading its own next word (0) a
// -i 4-byte scan of 40 GiB runs at 0.69 TB/s, with lane 31 loading + shuffle (2) at 2.63 TB/s (H100 80GB HBM3, 700 W,
// same counts); how the windows are extracted (IMAD.HI, PRMT or funnel shift) makes no measurable difference once the
// load is gone.  Warp-cooperative emission lengthens the streaming loop.  Defaults: 2 / 0.
#ifndef KREP_B200_W4_NX
#define KREP_B200_W4_NX 2 // how the window kernel gets the word behind a vector: 0 = every lane loads it, 1 / 2 = shuffle
#endif
#ifndef KREP_B200_W4_WARP_EMIT
#define KREP_B200_W4_WARP_EMIT 0
#endif
#ifdef KREP_B200_W4_CS
#define WLOAD(q) ld_stream(q)
#else
#define WLOAD(q) __ldg(q)
#endif
template <bool FOLD, bool MASKED, int UNROLL>
__global__ void __launch_bounds__(256, 4) k_lit_window4(const __grid_constant__ LitDevParams p)
{
    const uint4 *__restrict__ t4 = reinterpret_cast<const uint4 *>(p.text);
    const uint32_t fold = p.fold, mask = p.win_mask, k0 = p.K[0];
    const uint32_t c1 = p.mulc[0], c2 = p.mulc[1], c3 = p.mulc[2]; // 2^24, 2^16, 2^8
    const bool lane31 = (threadIdx.x & 31) == 31;
    unsigned long long local_cnt = 0;
    const uint64_t tile = (uint64_t)blockDim.x * UNROLL;
    const uint64_t stride = (uint64_t)gridDim.x * tile;
    uint64_t g0 = p.group_begin + (uint64_t)blockIdx.x * tile;
    for (; g0 + tile <= p.group_end; g0 += stride)
    {
        uint4 v[UNROLL];
        uint32_t nx[UNROLL];
#pragma unroll
        for (int u = 0; u < UNROLL; u++)
        {
            const uint4 *q = t4 + g0 + (uint64_t)u * blockDim.x + threadIdx.x;
            v[u] = WLOAD(q);
#if KREP_B200_W4_NX == 0
            nx[u] = __ldg(reinterpret_cast<const uint32_t *>(q + 1)); // every lane loads its own next word (L1/L2 hit)
#elif KREP_B200_W4_NX == 2
            // the word after the vector is the next lane's v.x: only lane 31 has to load it — as ONE predicated
            // instruction (a branch around the load would make the warp reconverge before every shuffle below)
            nx[u] = 0u;
            asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.u32 p, %2, 0;\n\t@p ld.global.nc.u32 %0, [%1];\n\t}"
                         : "+r"(nx[u])
                         : "l"(reinterpret_cast<const uint32_t *>(q + 1)), "r"((uint32_t)lane31));
#else
            nx[u] = lane31 ? __ldg(reinterpret_cast<const uint32_t *>(q + 1)) : 0u;
#endif
        }
#if KREP_B200_W4_NX != 0
#pragma unroll
        for (int u = 0; u < UNROLL; u++)
        {
            const uint32_t nb = __shfl_down_sync(0xffffffffu, v[u].x, 1);
#if KREP_B200_W4_NX == 2
            nx[u] = lane31 ? nx[u] : nb; // a select, not a branch
#else
            if (!lane31) nx[u] = nb;
#endif
        }
#endif
        uint32_t hm = 0; // bit u: vector u holds a candidate
#pragma unroll
        for (int u = 0; u < UNROLL; u++)
            hm |= hit_vec_w<FOLD, MASKED>(v[u], nx[u], fold, mask, k0, c1, c2, c3) ? (1u << u) : 0u;
        // Needles of 1..3 bytes (MASKED) occur often — `the` once per 7 KiB of English-like text, once per 64 B in the density
        // sweep — so their kernels emit warp-cooperatively (one atomicAdd per warp and vector); the 4..6-byte kernels
        // keep the per-occurrence path, whose streaming loop is shorter.
        if constexpr (MASKED || KREP_B200_W4_WARP_EMIT)
        {
            const uint32_t anyhm = __reduce_or_sync(0xffffffffu, hm);
            if (anyhm)
            {
#pragma unroll
                for (int u = 0; u < UNROLL; u++)
                    if ((anyhm >> u) & 1u)
                        local_cnt += emit_warp<true>(p, g0 + (uint64_t)u * blockDim.x + threadIdx.x, v[u], nx[u], (hm >> u) & 1u);
            }
        }
        else if (hm)
        {
#pragma unroll
            for (int u = 0; u < UNROLL; u++)
                if ((hm >> u) & 1u) local_cnt += slow_window4(p, g0 + (uint64_t)u * blockDim.x + threadIdx.x, v[u], nx[u]);
        }
    }
    if (g0 < p.group_end)
    {
        for (int u = 0; u < UNROLL; u++)
        {
            const uint64_t g = g0 + (uint64_t)u * blockDim.x + threadIdx.x;
            if (g < p.group_end)
            {
                const uint4 v = ld_stream(t4 + g);
                const uint32_t nx = __ldg(reinterpret_cast<const uint32_t *>(t4 + g + 1));
                if (hit_vec_w<FOLD, MASKED>(v, nx, fold, mask, k0, c1, c2, c3)) local_cnt += slow_window4(p, g, v, nx);
            }
        }
    }
    tail_and_count(p, local_cnt);
}

// ------------------------------------------------------------------------------------ launch
static int g_occ[6] = {0, 0, 0, 0, 0, 0}; // identical on every device of the box (all sm_90)

template <typename K>
static int occupancy(K kernel)
{
    int nb = 0;
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, kernel, 256, 0);
    return nb > 0 ? nb : 1;
}

void launch_literal(const Plan *plan, const LitDevParams &p, int sm_count, cudaStream_t s)
{
    constexpr int UNROLL = 4;
    static std::once_flag once;
    std::call_once(once, [] {
        g_occ[0] = occupancy(k_lit_aligned4<false, UNROLL>);
        g_occ[1] = occupancy(k_lit_aligned4<true, UNROLL>);
        g_occ[2] = occupancy(k_lit_window4<false, false, UNROLL>);
        g_occ[3] = occupancy(k_lit_window4<true, false, UNROLL>);
        g_occ[4] = occupancy(k_lit_window4<false, true, UNROLL>);
        g_occ[5] = occupancy(k_lit_window4<true, true, UNROLL>);
    });
    const uint64_t groups = p.group_end > p.group_begin ? p.group_end - p.group_begin : 0;
    const uint64_t tile = 256ull * UNROLL;
    uint64_t tiles = (groups + tile - 1) / tile;
    if (tiles == 0) tiles = 1; // still need the tail warp
    const bool folded = plan->fold != 0xFFFFFFFFu, masked = plan->win_mask != 0xFFFFFFFFu;
    const int which = plan->filter == FILTER_WINDOW4 ? 2 + (folded ? 1 : 0) + (masked ? 2 : 0) : (folded ? 1 : 0);
    uint64_t resident = (uint64_t)sm_count * g_occ[which];
    const unsigned grid = (unsigned)(tiles < resident ? tiles : resident);
    if (which == 2)
        k_lit_window4<false, false, UNROLL><<<grid, 256, 0, s>>>(p);
    else if (which == 3)
        k_lit_window4<true, false, UNROLL><<<grid, 256, 0, s>>>(p);
    else if (which == 4)
        k_lit_window4<false, true, UNROLL><<<grid, 256, 0, s>>>(p);
    else if (which == 5)
        k_lit_window4<true, true, UNROLL><<<grid, 256, 0, s>>>(p);
    else if (which == 1)
        k_lit_aligned4<true, UNROLL><<<grid, 256, 0, s>>>(p);
    else
        k_lit_aligned4<false, UNROLL><<<grid, 256, 0, s>>>(p);
    count_launch();
}

} // namespace kb
