// scan_multi.cu — multi-pattern scan for sm_90a; replaces aho_corasick_search's per-byte goto/fail
// walk (aho_corasick.c:328-437) and ac_trie_build (aho_corasick.c:111-271).
//
// The reference chases pointers through 2 KB trie nodes, one dependent load per text byte.  A GPU at
// HBM speed cannot afford a serial automaton, so the same result set — every occurrence of every
// pattern, nested and overlapping ones included, duplicates in the pattern list emitted once per
// index (aho_corasick.c:361) — is produced by filter + verify instead:
//
//   * SAMPLED WINDOW FILTER.  With Lmin the shortest pattern, pick a window width w and a sampling
//     stride s in {1,2,4} with w + s - 1 <= Lmin.  Every occurrence starting at p then contains the
//     w-byte window at a = ceil(p/s)*s, which equals bytes [d, d+w) of its pattern with d = a-p < s.
//     All s*K such pattern windows are hashed into a table that lives in SHARED MEMORY (up to 192 KB of
//     the SM's 227 KB); the hot loop hashes the text window at every multiple of s and tests one bit.
//     Text is streamed exactly once with coalesced 16-byte loads.
//       Lmin >= 6 : k_ac_tri4 — stride 4, the window is ONE aligned text word (see the TRI4 section):
//                   4 lookups per 16 bytes, candidates queued per warp and verified in batches;
//       Lmin  = 5 : k_ac_scan<2> — stride 2, paired lookups sharing one shared-memory load;
//       Lmin <= 4 : k_ac_scan<1> — stride 1.
//   * EXACT TABLE (L2-resident, open addressing): a window (k_ac_scan) or 6-byte prefix (k_ac_tri4) that
//     passed the filter is looked up exactly — this kills filter false positives in ~one L2 load;
//   * VERIFY compares the whole pattern at p = a - d under the exact per-byte case mask, applies the
//     whole-word test against the global text, shard ownership by start offset, and emits one key
//     (end << 24 | (1023 - (len-1)) << 14 | pattern_index) whose ascending order is
//     aho_corasick_search's emission order (end ascending, longest first, list order).
//
// Case-insensitive search hashes (text & 0xDF..DF) against equally folded pattern windows (a superset
// filter); the verify step is exact, equal to lower_table on both sides (aho_corasick.c:161, 333).
#include <algorithm>
#include <cstring>
#include <unordered_map>
#include "common.h"

namespace kb {

struct AcSlot
{
    uint64_t key; // folded window value (low w bytes)
    uint32_t first, count;
};

struct AcDevTables
{
    uint32_t *d_bitmap = nullptr; // 2^B bits
    uint8_t *d_bitmap2 = nullptr; // tri4: 2^23-bit second-level filter over the 6-byte prefixes (L2 resident)
    AcSlot *d_slots = nullptr;    // nslots (power of two)
    uint32_t *d_list = nullptr;   // (pattern << 2) | d
    uint8_t *d_pool_val = nullptr, *d_pool_mask = nullptr;
    uint32_t *d_pat_off = nullptr, *d_pat_len = nullptr;
    uint32_t bitmap_bytes = 0, nslots = 0, w = 0, s = 0, npat = 0;
    uint64_t wmask = 0; // low w bytes
    uint32_t fold = 0xFFFFFFFFu;
    uint32_t mul_lo = 0, mul_hi = 0, mul_b = 0, bit_shift = 0;
    bool tri4 = false; // aligned-word stride-4 filter (Lmin >= 6), see k_ac_tri4
    uint32_t cls_mask = 0, cls_val = 0;
};

// What ac_build_tables compiles on the host; ac_upload_tables copies it to each device that runs the plan.
struct AcHostTables
{
    std::vector<uint32_t> bitmap;
    std::vector<uint8_t> bitmap2;
    std::vector<AcSlot> slots;
    std::vector<uint32_t> list;
    std::vector<uint8_t> pool_val, pool_mask;
    std::vector<uint32_t> pat_off, pat_len;
    AcDevTables proto; // the scalar fields (device pointers null)
};

struct AcDev
{
    const uint32_t *bitmap;
    const uint8_t *bitmap2;
    const AcSlot *slots;
    const uint32_t *list;
    const uint8_t *pool_val, *pool_mask;
    const uint32_t *pat_off, *pat_len;
    uint32_t nslots, w, npat, bitmap_bytes;
    uint32_t wmask_lo, wmask_hi, fold;
    uint32_t mul_lo, mul_hi, mul_b, bit_shift; // hash multipliers (low zero bytes mask the window), bit-index shift for w < 4
    // launch
    const uint8_t *text;
    uint64_t avail_len, own_begin, own_end, global_offset;
    int32_t prev_byte, next_byte;
    uint64_t group_begin, group_end, tail_a; // occurrences whose sampled window position is >= tail_a go to the tail warp
    uint64_t *out;
    uint64_t cap;
    unsigned long long *counter;
    uint32_t whole_word, want_positions;
    uint32_t zero; // always 0; opaque to the compiler (see the software pipeline in k_ac_scan)
    uint32_t cls_mask, cls_val; // tri4: bits on which ALL pattern trigrams agree — a text word that differs there skips its lookup
    uint32_t pf_dist; // tri4: L2 prefetch distance in tiles (0 = off)
};

static constexpr uint32_t HC1 = 0x9E3779B1u, HC2 = 0x85EBCA77u;

__host__ __device__ __forceinline__ uint32_t slot_hash(uint32_t lo, uint32_t hi)
{
    uint32_t h = lo * 0x9E3779B1u + hi * 0x85EBCA77u; // murmur3-style finaliser: the table index uses the low bits
    h ^= h >> 16;
    h *= 0x85EBCA6Bu;
    h ^= h >> 13;
    h *= 0xC2B2AE35u;
    return h ^ (h >> 16);
}

__device__ __forceinline__ bool dev_is_word2(int c)
{
    return (c >= '0' && c <= '9') || (c >= 'A' && c <= 'Z') || (c >= 'a' && c <= 'z') || c == '_';
}

// exact check of pattern k at start p (p may be negative / out of range) + emission
__device__ __noinline__ unsigned ac_verify_emit(const AcDev &A, uint32_t k, long long cand)
{
    if (cand < (long long)A.own_begin || cand >= (long long)A.own_end) return 0;
    const uint64_t p = (uint64_t)cand;
    const uint32_t len = A.pat_len[k];
    if (len == 0 || p + len > A.avail_len) return 0;
    const uint8_t *t = A.text + p;
    const uint8_t *val = A.pool_val + A.pat_off[k], *msk = A.pool_mask + A.pat_off[k];
    for (uint32_t i = 0; i < len; i++)
        if ((t[i] & msk[i]) != val[i]) return 0;
    if (A.whole_word)
    {
        const uint64_t e = p + len;
        const int pb = p > 0 ? (int)t[-1] : A.prev_byte;
        const int nb = e < A.avail_len ? (int)A.text[e] : A.next_byte;
        if (dev_is_word2(pb) || dev_is_word2(nb)) return 0;
    }
    if (A.want_positions)
    {
        const unsigned long long slot = atomicAdd(A.counter, 1ULL);
        if (slot < A.cap)
            A.out[slot] = ((A.global_offset + p + len) << AC_END_SHIFT) | ((uint64_t)(1023u - (len - 1)) << AC_LEN_SHIFT) | k;
        return 0;
    }
    return 1;
}

// window value (lo,hi canonical: folded + masked to w bytes) at sampled position a passed the bitmap
__device__ __forceinline__ unsigned ac_probe(const AcDev &A, uint64_t a, uint32_t lo, uint32_t hi)
{
    const uint64_t key = ((uint64_t)hi << 32) | lo;
    uint32_t h = slot_hash(lo, hi) & (A.nslots - 1);
    unsigned n = 0;
    for (;;)
    {
        const AcSlot sl = A.slots[h];
        if (sl.count == 0) return n;
        if (sl.key == key)
        {
            for (uint32_t i = 0; i < sl.count; i++)
            {
                const uint32_t e = A.list[sl.first + i];
                n += ac_verify_emit(A, e >> 2, (long long)a - (long long)(e & 3));
            }
            return n;
        }
        h = (h + 1) & (A.nslots - 1);
    }
}

// Ordered streaming loads for the software pipeline.  The hardware tracks outstanding loads with a handful of
// counting scoreboards, so waiting for batch i also waits for every load issued before the wait.  The loop
// therefore (1) touches batch i (forcing its wait), THEN (2) issues batch i+1, then (3) filters batch i;
// volatile asm keeps that order.
__device__ __forceinline__ uint4 ld_stream_ordered(const uint4 *p)
{
    uint4 v;
    asm volatile("ld.global.cs.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
    return v;
}
__device__ __forceinline__ uint4 ld_vec_ordered(const uint4 *p) // default L2 policy: candidate groups are re-read from L2
{
    uint4 v;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
    return v;
}
__device__ __forceinline__ uint32_t ld_u32_ordered(const uint32_t *p)
{
    uint32_t v;
    asm volatile("ld.global.nc.u32 %0, [%1];" : "=r"(v) : "l"(p));
    return v;
}
__device__ __forceinline__ uint32_t ld_u8_ordered(const uint8_t *p)
{
    uint32_t v;
    asm volatile("ld.global.nc.u8 %0, [%1];" : "=r"(v) : "l"(p));
    return v;
}
__device__ __forceinline__ uint2 ld_u64_ordered(const uint2 *p)
{
    uint2 v;
    asm volatile("ld.global.nc.v2.u32 {%0,%1}, [%2];" : "=r"(v.x), "=r"(v.y) : "l"(p));
    return v;
}
__device__ __forceinline__ void touch(const uint4 &v, const uint2 &n)
{
    asm volatile("" ::"r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w), "r"(n.x), "r"(n.y));
}

__device__ __forceinline__ uint32_t lds_u8(uint32_t saddr)
{
    uint32_t v;
    asm volatile("ld.shared.u8 %0, [%1];" : "=r"(v) : "r"(saddr));
    return v;
}

// The filter for one 16-byte group: 16/S bitmap lookups.  Per lookup:
//   window extraction   free for word-aligned windows, two funnel shifts otherwise            (ALU)
//   hash = lo*M1 + hi*M2   the multipliers' low zero bytes mask the window to w bytes for free  (FMA pipe)
//   byte address = mulhi(hash, bitmap_bytes) + smem base   (well-mixed high hash bits)         (FMA pipe)
//   one LDS.U8; the byte is replicated x4 (v * 0x01010101) so that a wrapping shift by the low   (LSU, FMA)
//   hash bits selects bit (hash & 7) without masking; results are OR-ed                          (ALU x2)
// DETAIL=false returns only "some lookup hit" in bit 0; DETAIL=true returns one bit per lookup
// (first lookup = highest bit) and is used by the rare path only.
template <int S, bool FOLD, bool DETAIL>
__device__ __forceinline__ uint32_t ac_group_filter(const uint8_t *s_mem, uint4 v, uint2 nx, uint32_t fold, uint32_t m1,
                                                    uint32_t m2, uint32_t nbytes, uint32_t bit_shift)
{
    uint32_t w[6] = {v.x, v.y, v.z, v.w, nx.x, nx.y};
    if (FOLD)
    {
#pragma unroll
        for (int i = 0; i < 6; i++) w[i] &= fold;
    }
    uint32_t acc = 0;
#pragma unroll
    for (int k = 0; k < 4; k++)
#pragma unroll
        for (int r = 0; r < 4; r += S)
        {
            const uint32_t lo = r == 0 ? w[k] : __funnelshift_r(w[k], w[k + 1], 8 * r);
            const uint32_t hi = r == 0 ? w[k + 1] : __funnelshift_r(w[k + 1], w[k + 2], 8 * r);
            const uint32_t h = lo * m1 + hi * m2;
            const uint32_t byte = s_mem[__umulhi(h, nbytes)];
            const uint32_t sel = S == 1 ? (h >> bit_shift) : h;
            const uint32_t t = __funnelshift_r(byte * 0x01010101u, 0u, sel);
            if (DETAIL) acc = acc * 2 + (t & 1u);
            else acc |= t;
        }
    return DETAIL ? acc : (acc & 1u);
}

__device__ __forceinline__ uint32_t lds_u32(uint32_t saddr)
{
    uint32_t v;
    asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(saddr));
    return v;
}

// S == 2 (w = 4 or 5): PAIRED lookups.  The shared-memory gather is the scarce resource (a random warp-wide
// LDS costs ~3.5 bank-conflict wavefronts on the one-wavefront-per-cycle L1 data pipe), so the windows at a
// and a+2 share ONE load: they overlap in T = bytes [a+2, a+w), which picks the 32-bit bitmap word; the two
// bytes only window A has pick one of the word's low 16 bits, the two bytes only window B has pick one of its
// high 16 bits.  Every pattern window is therefore entered twice at build time (A view: word by its last w-2
// bytes, bit by its first 2; B view: word by its first w-2 bytes, bit by its last 2).  All hashing runs on the
// FMA pipe (multipliers with low zero bytes mask for free; mulhi by 16 extracts the top 4 hash bits).
template <bool FOLD, bool DETAIL>
__device__ __forceinline__ uint32_t ac_pair_filter(const uint8_t *s_mem, uint4 v, uint32_t nx0, uint32_t fold, uint32_t mT,
                                                   uint32_t mA, uint32_t mB, uint32_t nbytes)
{
    uint32_t w[5] = {v.x, v.y, v.z, v.w, nx0};
    if (FOLD)
    {
#pragma unroll
        for (int i = 0; i < 5; i++) w[i] &= fold;
    }
    uint32_t acc = 0;
#pragma unroll
    for (int k = 0; k < 4; k++)
    {
        const uint32_t x = __funnelshift_r(w[k], w[k + 1], 16);              // bytes a+2 .. a+5
        const uint32_t word = *reinterpret_cast<const uint32_t *>(s_mem + (__umulhi(x * mT, nbytes) & ~3u));
        const uint32_t tA = __funnelshift_r(word, 0u, __umulhi(w[k] * mA, 16u));          // bit 0..15
        const uint32_t tB = __funnelshift_r(word, 0u, __umulhi(w[k + 1] * mB, 16u) + 16u); // bit 16..31
        if (DETAIL) acc = acc * 4 + (tA & 1u) * 2 + (tB & 1u);
        else acc |= tA | tB;
    }
    return DETAIL ? acc : (acc & 1u);
}

// ---------------------------------------------------------------------------------------------
// Rare path.  Candidate groups parked by the streaming loop are verified 32 at a time, one group per
// lane, in warp-synchronous loops (every lane pops one hit, then all lanes step their hash-table probe
// together), so the slow path keeps the whole warp busy instead of trailing single lanes.
// ---------------------------------------------------------------------------------------------
template <int S, bool FOLD>
__device__ __noinline__ unsigned ac_verify_groups(const AcDev &A, const uint8_t *s_mem, uint64_t g, bool valid)
{
    const uint4 *t4 = reinterpret_cast<const uint4 *>(A.text);
    uint32_t hits = 0;
    uint32_t w[6] = {0, 0, 0, 0, 0, 0};
    if (valid)
    {
        const uint4 v = __ldg(t4 + g);
        const uint2 nx = __ldg(reinterpret_cast<const uint2 *>(t4 + g + 1));
        w[0] = v.x; w[1] = v.y; w[2] = v.z; w[3] = v.w; w[4] = nx.x; w[5] = nx.y;
        if constexpr (S == 2)
            hits = ac_pair_filter<FOLD, true>(s_mem, v, nx.x, A.fold, A.mul_lo, A.mul_hi, A.mul_b, A.bitmap_bytes);
        else
            hits = ac_group_filter<S, FOLD, true>(s_mem, v, nx, A.fold, A.mul_lo, A.mul_hi, A.bitmap_bytes, A.bit_shift);
    }
    constexpr int NLOOK = 16 / S;
    unsigned n = 0;
    while (__any_sync(0xffffffffu, hits != 0))
    {
        bool active = hits != 0;
        uint64_t key = 0, a = 0;
        uint32_t h = 0;
        if (active)
        {
            const int bit = 31 - __clz(hits);
            hits &= ~(1u << bit);
            const int o = (NLOOK - 1 - bit) * S; // byte offset of the window inside the group
            const int k = o >> 2, r = o & 3;
            uint32_t lo = w[0], hi = w[1], h2 = w[2];
#pragma unroll
            for (int j = 1; j < 4; j++)
                if (k == j) { lo = w[j]; hi = w[j + 1]; h2 = w[j + 2 < 6 ? j + 2 : 5]; }
            if (r)
            {
                lo = __funnelshift_r(lo, hi, 8 * r);
                hi = __funnelshift_r(hi, h2, 8 * r);
            }
            lo &= A.fold & A.wmask_lo;
            hi &= A.fold & A.wmask_hi;
            key = ((uint64_t)hi << 32) | lo;
            h = slot_hash(lo, hi) & (A.nslots - 1);
            a = g * 16 + o;
        }
        while (__any_sync(0xffffffffu, active))
        {
            if (active)
            {
                const AcSlot sl = A.slots[h];
                if (sl.count == 0) active = false;
                else if (sl.key == key)
                {
                    for (uint32_t i = 0; i < sl.count; i++)
                    {
                        const uint32_t e = A.list[sl.first + i];
                        n += ac_verify_emit(A, e >> 2, (long long)a - (long long)(e & 3));
                    }
                    active = false;
                }
                else h = (h + 1) & (A.nslots - 1);
            }
        }
    }
    return n;
}

template <int UNROLL>
struct AcQueue
{
    static constexpr int CAP = 32 * UNROLL + 32; // a remainder of < 32 plus one full iteration of new candidates
};

template <int S, bool FOLD, int THREADS, int UNROLL>
__global__ void __launch_bounds__(THREADS, 1) k_ac_scan(const __grid_constant__ AcDev A)
{
    extern __shared__ __align__(16) uint8_t s_mem[];
    constexpr int QCAP = AcQueue<UNROLL>::CAP;
    const uint32_t nbytes = A.bitmap_bytes;
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    uint32_t *s_cnt = reinterpret_cast<uint32_t *>(s_mem + nbytes) + warp; // this warp's queue length
    uint64_t *s_q = reinterpret_cast<uint64_t *>(s_mem + nbytes + 128) + warp * QCAP;
    {
        const uint4 *src = reinterpret_cast<const uint4 *>(A.bitmap);
        uint4 *dst = reinterpret_cast<uint4 *>(s_mem);
        for (uint32_t i = threadIdx.x; i < nbytes / 16; i += THREADS) dst[i] = src[i];
        if (lane == 0) *s_cnt = 0;
    }
    __syncthreads();
    const uint4 *__restrict__ t4 = reinterpret_cast<const uint4 *>(A.text);
    const uint32_t fold = A.fold, m1 = A.mul_lo, m2 = A.mul_hi, m3 = A.mul_b, bit_shift = A.bit_shift;
    unsigned long long local_cnt = 0;
    constexpr uint64_t tile = (uint64_t)THREADS * UNROLL;
    const uint64_t stride = (uint64_t)gridDim.x * tile;

    // The 8 bytes that follow a group's vector: for S == 2 only one word is needed and it comes from the next
    // lane's registers (shuffle), so only lane 31 loads it; other strides load it per lane.  Either way the load
    // is issued together with the vector (prefetched), never in front of its use.
    auto load_next = [&](const uint4 *q) -> uint2 {
        if constexpr (S == 2)
            return lane == 31 ? make_uint2(ld_u32_ordered(reinterpret_cast<const uint32_t *>(q + 1)), 0u) : make_uint2(0u, 0u);
        else
            return ld_u64_ordered(reinterpret_cast<const uint2 *>(q + 1)); // in bounds by group_end
    };
    auto filter = [&](const uint4 &v, const uint2 &nx) -> uint32_t {
        if constexpr (S == 2)
        {
            uint32_t nx0 = __shfl_down_sync(0xffffffffu, v.x, 1);
            if (lane == 31) nx0 = nx.x;
            return ac_pair_filter<FOLD, false>(s_mem, v, nx0, fold, m1, m2, m3, nbytes);
        }
        else
            return ac_group_filter<S, FOLD, false>(s_mem, v, nx, fold, m1, m2, nbytes, bit_shift);
    };
    // Candidate groups are parked in this warp's shared-memory queue and verified 32 at a time.
    auto park = [&](uint32_t hit, uint64_t g) {
        if (hit) s_q[atomicAdd(s_cnt, 1u)] = g;
    };
    auto drain = [&](bool all) {
        __syncwarp();
        uint32_t c = *reinterpret_cast<volatile uint32_t *>(s_cnt);
        if (c >= 32 || (all && c))
        {
            while (c >= 32)
            {
                c -= 32;
                local_cnt += ac_verify_groups<S, FOLD>(A, s_mem, s_q[c + lane], true);
            }
            if (all && c)
            {
                local_cnt += ac_verify_groups<S, FOLD>(A, s_mem, lane < c ? s_q[lane] : 0, lane < c);
                c = 0;
            }
            __syncwarp();
            if (lane == 0) *s_cnt = c;
            __syncwarp();
        }
    };

    // Register double buffering: the vectors of the next tile are requested before the current tile is
    // filtered, so HBM latency overlaps this warp's own ~260 filter instructions (plus the other warps).
    // Software pipeline over register double buffers.  The hardware tracks outstanding loads with a handful
    // of counting scoreboards, so a wait for batch i also waits for anything issued before the wait; the loop
    // therefore first moves batch i out of the landing registers (that is where the wait happens, on every
    // path), only then issues batch i+1, and then filters batch i out of the copies.
    uint64_t g0 = A.group_begin + (uint64_t)blockIdx.x * tile;
    uint4 vn[UNROLL];
    uint2 nxn[UNROLL];
#pragma unroll
    for (int u = 0; u < UNROLL; u++)
    {
        vn[u] = make_uint4(0u, 0u, 0u, 0u);
        nxn[u] = make_uint2(0u, 0u);
    }
    if (g0 + tile <= A.group_end)
    {
#pragma unroll
        for (int u = 0; u < UNROLL; u++)
        {
            const uint4 *q = t4 + g0 + (uint64_t)u * THREADS + threadIdx.x;
            vn[u] = ld_stream_ordered(q);
            nxn[u] = load_next(q);
        }
    }
    for (; g0 + tile <= A.group_end; g0 += stride)
    {
        uint4 v[UNROLL];
        uint2 nx[UNROLL];
#pragma unroll
        for (int u = 0; u < UNROLL; u++)
        {
            v[u] = vn[u];
            nx[u] = nxn[u];
            touch(v[u], nx[u]);
        }
        const uint64_t gn = g0 + stride;
        // HBM latency comes off the registers: every warp bulk-prefetches its 1/(THREADS/32) share of the CTA tile that
        // is PF iterations ahead of the register double buffer into L2 (one instruction per warp and tile)
        if (A.pf_dist != 0 && lane == 0)
        {
            const uint64_t gp = gn + (uint64_t)A.pf_dist * stride;
            if (gp + tile <= A.group_end)
                asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(t4 + gp + (uint64_t)warp * (tile / (THREADS / 32))),
                             "r"((uint32_t)(tile / (THREADS / 32) * 16)) : "memory");
        }
        if (gn + tile <= A.group_end)
        {
#pragma unroll
            for (int u = 0; u < UNROLL; u++)
            {
                const uint4 *q = t4 + gn + (uint64_t)u * THREADS + threadIdx.x;
                vn[u] = ld_stream_ordered(q);
                nxn[u] = load_next(q);
            }
        }
        uint32_t hit[UNROLL], anyhit = 0;
#pragma unroll
        for (int u = 0; u < UNROLL; u++) anyhit |= hit[u] = filter(v[u], nx[u]);
        if (anyhit) // one branch for the whole batch: the common case parks nothing
        {
#pragma unroll
            for (int u = 0; u < UNROLL; u++) park(hit[u], g0 + (uint64_t)u * THREADS + threadIdx.x);
        }
        drain(false);
    }
    if (g0 < A.group_end) // ragged tile: whole warps stay converged (lanes past the end re-read the last group, report no hit)
    {
        for (int u = 0; u < UNROLL; u++)
        {
            const uint64_t g = g0 + (uint64_t)u * THREADS + threadIdx.x;
            const uint64_t gc = g < A.group_end ? g : A.group_end - 1;
            const uint4 vv = __ldcs(t4 + gc);
            uint32_t hit = filter(vv, load_next(t4 + gc));
            if (S == 2 && g + 1 == A.group_end && lane != 31) // the neighbour lane holds a clamped group: use the true next word
                hit = ac_pair_filter<FOLD, false>(s_mem, vv, __ldg(reinterpret_cast<const uint32_t *>(t4 + gc + 1)), fold, m1, m2, m3, nbytes);
            park(g < A.group_end ? hit : 0u, g);
        }
    }
    drain(true);
    // tail: occurrences whose sampled window lies beyond the vector loop — brute force, lanes over patterns
    if (blockIdx.x == 0 && threadIdx.x < 32)
    {
        const uint64_t first = A.tail_a >= (uint64_t)(S - 1) ? A.tail_a - (S - 1) : 0;
        for (uint64_t p = first; p < A.avail_len; p++)
        {
            const uint64_t a = (p + S - 1) / S * S;
            if (a < A.tail_a) continue;
            for (uint32_t k = threadIdx.x; k < A.npat; k += 32) local_cnt += ac_verify_emit(A, k, (long long)p);
        }
    }
    if (!A.want_positions)
    {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) local_cnt += __shfl_xor_sync(0xffffffffu, local_cnt, o);
        if (lane == 0 && local_cnt) atomicAdd(A.counter, local_cnt);
    }
}

// =============================================================================================
// TRI4 — the stride-4 filter for pattern sets whose shortest pattern has exactly 6 bytes.
//
// With Lmin = 6 a sampling stride of 4 leaves only a 3-byte window (w + s - 1 <= Lmin), and 4*K trigrams of
// lowercase-ish patterns are far too dense for a plain bitmap.  But an occurrence at p = a - d (a aligned, d in 0..3)
// of a pattern of length L also fixes byte a+3 whenever L - d >= 4 — i.e. for every (pattern, d) except (L = 6, d = 3).
// So one aligned text word w = bytes [a, a+4) is the whole lookup key, with NO shifting and NO neighbour bytes:
//     word index = hash(low three bytes of w)          IMAD (multiplier with a zero low byte drops byte 3) + IMAD.HI
//     bit index  = low five bits of byte 3 of w         IMAD.HI by 2^8 (w >> 24 on the FMA pipe); SHF.W wraps at 32
// and the (L = 6, d = 3) entries, which do not know byte a+3, set all 32 bits of their word.  Per 16 bytes that is
// 4 lookups of ~7 instructions split evenly between the FMA and ALU pipes, and 4 shared-memory loads — half the
// instructions of the stride-2 paired filter above.  A lookup passes for ~1 % of the positions of English-like text
// against 1000 patterns; those groups are queued per warp and verified 32 at a time:
//
// Exact table (L2 resident, AcSlot open addressing): key = the folded first 6 bytes of a pattern, value = list of the
// pattern indices that start with them.  A passed lookup at aligned position a means "some pattern may contain this
// word at offset d", so each of the four starts p = a - d is tested by probing its 6 bytes [p, p+6) — four independent
// L2 loads issued together, almost always an empty slot — and only a prefix hit goes on to the full compare.
// =============================================================================================
// cm / cv: the bits on which all pattern trigrams agree (e.g. 0x00E0E0E0 / 0x00606060 for lowercase-only sets).  A text
// word that differs there cannot pass, so its lane sits the shared-memory load out: the load is a random gather whose
// cost is its bank conflicts (~3.6 wavefronts with 32 lanes active), and the shared-memory pipe is what bounds this
// kernel — with a third of the lanes active the same instruction takes ~1.9 wavefronts.
template <bool FOLD>
__device__ __forceinline__ uint32_t tri4_filter(uint32_t s_base, const uint4 &v, uint32_t fold, uint32_t m1, uint32_t nbytes,
                                                uint32_t c8, uint32_t cm, uint32_t cv)
{
    uint32_t w[4] = {v.x, v.y, v.z, v.w};
    uint32_t acc = 0;
#pragma unroll
    for (int k = 0; k < 4; k++)
    {
        if (FOLD) w[k] &= fold;
        // branch-free: the lane's load is predicated off (word = 0) when the class test fails
        const uint32_t addr = s_base + (__umulhi(w[k] * m1, nbytes) & ~3u);
        uint32_t word;
        // one LOP3 computes (w & cm) ^ cv and sets the predicate "differs" (lop3 with a predicate output)
        asm volatile("{\n\t.reg .pred p, f;\n\t.reg .b32 t;\n\tsetp.ne.u32 f, 0, 0;\n\tlop3.or.b32 t|p, %2, %3, %4, 0x6A, f;\n\t"
                     "mov.u32 %0, 0;\n\t@!p ld.shared.u32 %0, [%1];\n\t}"
                     : "=r"(word)
                     : "r"(addr), "r"(w[k]), "r"(cm), "r"(cv));
        acc |= __funnelshift_r(word, 0u, __umulhi(w[k], c8));
    }
    return acc & 1u;
}

__device__ __forceinline__ uint32_t prefix_hash(uint32_t lo, uint32_t hi) { return lo * HC1 + hi * HC2; }

// Queue entry (32 bytes of shared memory, one candidate group):
//     [0,8)   meta = rel << 6 | next_partial << 5 | 0 << 4 | mask       rel  = group index relative to group_begin
//                                                                         mask = lookups still to verify (0 = unknown)
//     [8,12)  the 4 bytes before the group     [12,16) the 4 bytes after it      [16,32) the group itself
// The group comes from the pushing lane's registers; the two neighbour words are fetched by cp.async straight into the
// entry (no register, no stall at push time), so verification never goes back to global memory for text.
// One entry per lane.  Every lane verifies ONE passed lookup per call; a group with more than one puts the rest back
// into the queue, so a batch costs one L2 round trip (the four prefix probes).
// Inlined into the scan kernel at its drain sites: a call would force the prefetched vectors of the streaming loop
// through the ABI's few callee-saved registers, i.e. into local memory on every iteration.
static constexpr uint32_t TRI4_ENTRY = 32, TRI4_QCAP = 64;

template <bool FOLD>
__device__ __forceinline__ unsigned tri4_verify_batch(const AcDev &A, uint32_t s_base, uint32_t q_base, uint32_t slot, bool valid,
                                                       uint32_t &qn, uint32_t lt_mask)
{
    unsigned n = 0;
    uint32_t X[6] = {0, 0, 0, 0, 0, 0}; // bytes [16g-4, 16g+20): previous word, the group, next word
    uint32_t meta_lo = 0, meta_hi = 0;
    if (valid)
    {
        const uint32_t e = q_base + slot * TRI4_ENTRY;
        asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(meta_lo), "=r"(meta_hi), "=r"(X[0]), "=r"(X[5]) : "r"(e));
        asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(X[1]), "=r"(X[2]), "=r"(X[3]), "=r"(X[4]) : "r"(e + 16));
    }
    uint32_t km = meta_lo & 15u;
    const uint64_t g = A.group_begin + ((((uint64_t)meta_hi << 32) | meta_lo) >> 6);
    if (valid)
    {
        if (meta_lo & 32u) // the 4 bytes after the group are not all readable (last full group of the text): byte loads
        {
            const uint64_t nb = (g + 1) * 16;
            X[5] = 0;
            for (uint64_t i = nb; i < A.avail_len; i++) X[5] |= (uint32_t)A.text[i] << (8 * (i - nb));
        }
        if (FOLD)
        {
#pragma unroll
            for (int i = 0; i < 6; i++) X[i] &= A.fold;
        }
        if (km == 0)
        {
#pragma unroll
            for (int k = 0; k < 4; k++)
            {
                const uint32_t w = X[k + 1];
                const uint32_t word = lds_u32(s_base + (__umulhi(w * A.mul_lo, A.bitmap_bytes) & ~3u));
                km |= ((word >> (__umulhi(w, A.mul_hi) & 31u)) & 1u) << k;
            }
        }
    }
    const int k = km ? __ffs(km) - 1 : 0;
    const bool work = km != 0;
    km &= km - 1;
    {
        // lookups beyond the first go back into the queue (room is guaranteed: this batch just left it); the entry is
        // re-written from the registers it was read into (FOLD was applied: folding is idempotent)
        const uint32_t b = __ballot_sync(0xffffffffu, km != 0);
        if (b)
        {
            __syncwarp(); // the slots written below may be the ones other lanes have just read their entries from
            if (km)
            {
                const uint32_t e = q_base + (qn + __popc(b & lt_mask)) * TRI4_ENTRY;
                asm volatile("st.shared.v4.u32 [%0], {%1,%2,%3,%4};" ::"r"(e), "r"((meta_lo & ~15u) | km), "r"(meta_hi), "r"(X[0]), "r"(X[5]));
                asm volatile("st.shared.v4.u32 [%0], {%1,%2,%3,%4};" ::"r"(e + 16), "r"(X[1]), "r"(X[2]), "r"(X[3]), "r"(X[4]));
            }
            qn += __popc(b);
        }
    }
    if (!work) return 0;
    // words X[k], X[k+1], X[k+2] without dynamic register indexing
    uint32_t y0 = X[0], y1 = X[1], y2 = X[2];
    if (k == 1) { y0 = X[1]; y1 = X[2]; y2 = X[3]; }
    if (k == 2) { y0 = X[2]; y1 = X[3]; y2 = X[4]; }
    if (k == 3) { y0 = X[3]; y1 = X[4]; y2 = X[5]; }
    const long long a = (long long)(g * 16 + 4 * k);
    // start p = a - d: 6 bytes at byte offset 4 - d of (y0 y1 y2)
    uint32_t lo[4], hi[4], h[4];
    lo[0] = y1; hi[0] = y2 & 0xFFFFu;
#pragma unroll
    for (int d = 1; d < 4; d++)
    {
        lo[d] = __funnelshift_r(y0, y1, 8 * (4 - d));
        hi[d] = __funnelshift_r(y1, y2, 8 * (4 - d)) & 0xFFFFu;
    }
    const uint32_t nmask = A.nslots - 1;
    const AcSlot *slots = A.slots;
    // second-level filter: one bit per 23-bit prefix hash in a 1 MB L2-resident bitmap; four byte loads issued together
    uint32_t pass = 0;
    {
        uint32_t by[4];
#pragma unroll
        for (int d = 0; d < 4; d++)
        {
            h[d] = prefix_hash(lo[d], hi[d]);
            by[d] = ld_u8_ordered(A.bitmap2 + (h[d] >> 12));
        }
#pragma unroll
        for (int d = 0; d < 4; d++) pass |= ((by[d] >> ((h[d] >> 9) & 7u)) & 1u) << d;
    }
    if (pass == 0) return 0; // the common case: nothing starts with any of the four
#pragma unroll 1
    for (int d = 0; d < 4; d++)
    {
        if (!((pass >> d) & 1u)) continue;
        const uint32_t lod = d == 0 ? lo[0] : (d == 1 ? lo[1] : (d == 2 ? lo[2] : lo[3]));
        const uint32_t hid = d == 0 ? hi[0] : (d == 1 ? hi[1] : (d == 2 ? hi[2] : hi[3]));
        uint32_t hh = (d == 0 ? h[0] : (d == 1 ? h[1] : (d == 2 ? h[2] : h[3]))) & nmask;
        for (;;)
        {
            const AcSlot q = slots[hh];
            if (q.count == 0) break;
            if (q.key == (((uint64_t)hid << 32) | lod))
            {
#pragma unroll 1
                for (uint32_t i = 0; i < q.count; i++) n += ac_verify_emit(A, A.list[q.first + i], a - d);
                break;
            }
            hh = (hh + 1) & nmask;
        }
    }
    return n;
}

template <bool FOLD, int THREADS>
__global__ void __launch_bounds__(THREADS, 1) k_ac_tri4(const __grid_constant__ AcDev A)
{
    extern __shared__ __align__(16) uint8_t s_mem[];
    constexpr uint32_t TILE = (uint32_t)THREADS * 4; // groups per CTA iteration; each warp owns 128 consecutive groups of it
    const uint32_t nbytes = A.bitmap_bytes;
    const uint32_t tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    {
        const uint4 *src = reinterpret_cast<const uint4 *>(A.bitmap);
        uint4 *dst = reinterpret_cast<uint4 *>(s_mem);
        for (uint32_t i = tid; i < nbytes / 16; i += THREADS) dst[i] = src[i];
    }
    __syncthreads();
    const uint32_t s_base = (uint32_t)__cvta_generic_to_shared(s_mem);
    const uint32_t q_base = s_base + nbytes + warp * (TRI4_QCAP * TRI4_ENTRY); // this warp's candidate queue
    const uint32_t fold = A.fold, m1 = A.mul_lo, c8 = A.mul_hi; // c8 = 2^8: umulhi(w, 2^8) = w >> 24 on the FMA pipe
    const uint32_t lt_mask = (1u << lane) - 1u;
    unsigned long long local_cnt = 0;
    uint32_t qn = 0; // entries in this warp's queue (warp-uniform, lives in a register)
    const uint8_t *const text0 = A.text + A.group_begin * 16; // byte address of relative group 0
    const uint4 *const t4rel = reinterpret_cast<const uint4 *>(text0);
    // relative group that has no byte before it (group 0 of the buffer), and first relative group whose following
    // 4 bytes are not all readable (16 (g + 1) + 4 > avail_len)
    const uint32_t no_prev_rel = A.group_begin == 0 ? 0u : 0xFFFFFFFFu;
    const uint64_t g_lim = A.avail_len >= 20 ? (A.avail_len - 20) / 16 + 1 : 0; // groups g < g_lim have a readable next word
    const uint32_t next_ok_rel = g_lim <= A.group_begin ? 0u : (g_lim - A.group_begin > 0xFFFFFFFFull ? 0xFFFFFFFFu : (uint32_t)(g_lim - A.group_begin));

    // verify queued candidates 32 at a time while at least `threshold` are waiting (32 in the loop, 1 at the end)
    auto drain = [&](uint32_t threshold) {
        while (qn >= threshold)
        {
            asm volatile("cp.async.wait_all;" ::: "memory"); // this lane's copies into its entries have landed ...
            __syncwarp();                                     // ... and so have everybody else's
            const uint32_t take = qn < 32 ? qn : 32;
            qn -= take;
            local_cnt += tri4_verify_batch<FOLD>(A, s_base, q_base, qn + lane, lane < take, qn, lt_mask);
            __syncwarp();
        }
    };
    // Queue the groups named by hm (bit u: group rel0 + 32u).  One warp-aggregated push per round — every lane with a
    // passed lookup queues the lowest of its (up to 4) groups; almost always a single round.  The entry's 24 text bytes
    // are copied by cp.async from L2 (the group was streamed through it a moment ago), so this needs no registers of the
    // streaming loop and runs while the next vectors are in flight.
    auto push_hits = [&](uint32_t hm, uint32_t rel0) {
        for (;;)
        {
            const uint32_t b = __ballot_sync(0xffffffffu, hm != 0);
            if (b == 0) break;
            if (hm)
            {
                const uint32_t u = __ffs(hm) - 1;
                hm &= hm - 1;
                const uint32_t rel = rel0 + u * 32;
                const uint32_t e = q_base + (qn + __popc(b & lt_mask)) * TRI4_ENTRY;
                const uint8_t *gp = text0 + (size_t)rel * 16;
                const bool has_prev = rel != no_prev_rel, next_ok = rel < next_ok_rel;
                asm volatile("st.shared.v2.u32 [%0], {%1,%2};" ::"r"(e), "r"((rel << 6) | (next_ok ? 0u : 32u)), "r"(rel >> 26));
                asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(e + 16), "l"(gp) : "memory");
                if (has_prev) asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(e + 8), "l"(gp - 4) : "memory");
                else asm volatile("st.shared.u32 [%0], %1;" ::"r"(e + 8), "r"(0u));
                if (next_ok) asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(e + 12), "l"(gp + 16) : "memory");
            }
            qn += __popc(b);
            drain(32);
        }
    };
    const uint32_t cm = A.cls_mask, cv = A.cls_val;
    auto filter4 = [&](const uint4 &v0, const uint4 &v1, const uint4 &v2, const uint4 &v3) -> uint32_t {
        uint32_t hm = tri4_filter<FOLD>(s_base, v0, fold, m1, nbytes, c8, cm, cv);
        hm |= tri4_filter<FOLD>(s_base, v1, fold, m1, nbytes, c8, cm, cv) << 1;
        hm |= tri4_filter<FOLD>(s_base, v2, fold, m1, nbytes, c8, cm, cv) << 2;
        hm |= tri4_filter<FOLD>(s_base, v3, fold, m1, nbytes, c8, cm, cv) << 3;
        return hm;
    };

    // This CTA owns the full tiles blockIdx.x, blockIdx.x + gridDim.x, ... ; n_groups < 2^32 per launch (host splits).
    // Inside a tile warp w owns groups [128w, 128w+128): vector u of lane l is group 128w + 32u + l, so every vector
    // load of a warp covers 512 contiguous bytes and a warp's share of a tile is one contiguous 2 KB piece.
    const uint32_t n_groups = (uint32_t)(A.group_end - A.group_begin);
    const uint32_t full_tiles = n_groups / TILE;
    const uint32_t n_it = full_tiles > blockIdx.x ? (full_tiles - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;
    const uint32_t rel_step = gridDim.x * TILE;
    uint32_t rel = blockIdx.x * TILE + warp * 128 + lane; // the only loop-carried position: pointers are rebuilt from it

    // HBM latency is taken off the registers by a bulk L2 prefetch (one instruction per warp and tile, PF tiles ahead);
    // the remaining L2-hit latency of the vector loads is covered by queueing the PREVIOUS tile's passed lookups
    // between issuing the loads and using them.
    const uint32_t PF = A.pf_dist;
    {
        // prime the prefetch pipeline
        const uint4 *q = t4rel + (blockIdx.x * TILE + warp * 128);
#pragma unroll 1
        for (uint32_t i = 0; i < PF && i < n_it; i++)
            if (lane == 0) asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(q + (size_t)i * rel_step), "r"(2048u) : "memory");
    }
    uint32_t hm_prev = 0, rel_prev = 0;
    for (uint32_t it = 0; it < n_it; it++)
    {
        const uint4 *ptr = t4rel + rel;
        if (PF != 0 && it + PF < n_it && lane == 0)
            asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(ptr + (size_t)PF * rel_step), "r"(2048u) : "memory");
        const uint4 a0 = ld_vec_ordered(ptr), a1 = ld_vec_ordered(ptr + 32), a2 = ld_vec_ordered(ptr + 64), a3 = ld_vec_ordered(ptr + 96);
        push_hits(hm_prev, rel_prev);
        hm_prev = filter4(a0, a1, a2, a3);
        rel_prev = rel;
        rel += rel_step;
    }
    push_hits(hm_prev, rel_prev);
    // ragged remainder (< one tile), handled by the CTA whose turn it would be; lanes past the end re-read the last
    // group and are masked out
    if (full_tiles % gridDim.x == blockIdx.x && full_tiles * TILE < n_groups)
    {
        const uint32_t r0 = full_tiles * TILE + warp * 128 + lane;
        uint4 rv[4];
        uint32_t vm = 0;
#pragma unroll
        for (int u = 0; u < 4; u++)
        {
            const uint32_t r = r0 + (uint32_t)u * 32;
            rv[u] = __ldg(t4rel + (r < n_groups ? r : n_groups - 1));
            vm |= (r < n_groups ? 1u : 0u) << u;
        }
        push_hits(filter4(rv[0], rv[1], rv[2], rv[3]) & vm, r0);
    }
    drain(1);
    // tail: occurrences whose aligned window position lies beyond the last full group — brute force, lanes over patterns
    if (A.zero == 0 && blockIdx.x == 0 && tid < 32)
    {
        const uint64_t first = A.tail_a >= 3 ? A.tail_a - 3 : 0;
        for (uint64_t p = first; p < A.avail_len; p++)
        {
            const uint64_t a = (p + 3) / 4 * 4;
            if (a < A.tail_a) continue;
            for (uint32_t k = tid; k < A.npat; k += 32) local_cnt += ac_verify_emit(A, k, (long long)p);
        }
    }
    if (!A.want_positions)
    {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) local_cnt += __shfl_xor_sync(0xffffffffu, local_cnt, o);
        if (lane == 0 && local_cnt) atomicAdd(A.counter, local_cnt);
    }
}

// ------------------------------------------------------------------------------------- build
static uint64_t pat_window(const uint8_t *p, uint32_t w, uint32_t fold)
{
    uint32_t lo = 0, hi = 0;
    for (uint32_t i = 0; i < w; i++)
    {
        if (i < 4) lo |= (uint32_t)p[i] << (8 * i);
        else hi |= (uint32_t)p[i] << (8 * (i - 4));
    }
    return ((uint64_t)(hi & fold) << 32) | (lo & fold);
}

int ac_build_tables(Plan *plan)
{
    AcHostTables *H = new AcHostTables();
    plan->ach = H;
    AcDevTables *T = &H->proto;
    const uint32_t K = (uint32_t)plan->patterns.size();
    T->npat = K;
    uint32_t lmin = 0xFFFFFFFFu, lmax = 0;
    for (uint32_t k = 0; k < K; k++)
    {
        const uint32_t len = plan->pat_lens[k];
        if (len == 0) continue; // empty patterns never match during the scan (aho_corasick.c:374)
        lmin = std::min(lmin, len);
        lmax = std::max(lmax, len);
    }
    if (lmax == 0) lmin = 0;
    plan->min_len = lmin;
    plan->max_len = lmax;
    uint32_t w, s;
    // Lmin >= 6: the aligned-word filter (k_ac_tri4).  Lmin == 6 keys it by the word's low three bytes and selects the
    // bit with its top byte ("tri"); from Lmin = 7 on every (pattern, d) knows the whole aligned word, so the word index
    // is a hash of all four bytes and the bit index a second hash of them ("quad") — same kernel, other constants.
    const bool tri4 = lmin >= 6, quad = lmin >= 7;
    T->tri4 = tri4;
    if (tri4) { w = quad ? 4 : 3; s = 4; }
    else if (lmin >= 5) { w = lmin - 1; s = 2; }
    else { w = lmin ? lmin : 1; s = 1; }
    T->w = w;
    T->s = s;
    T->wmask = w >= 8 ? ~0ull : ((1ull << (8 * w)) - 1);
    T->fold = plan->case_sensitive ? 0xFFFFFFFFu : 0xDFDFDFDFu;
    // hash = lo*mul_lo + hi*mul_hi; a multiplier with k low zero bytes ignores the top k bytes of its operand
    T->mul_lo = w >= 4 ? HC1 : (HC1 << (8 * (4 - w)));
    T->mul_hi = w > 4 ? (w >= 8 ? HC2 : (HC2 << (8 * (8 - w)))) : 0u;
    T->bit_shift = w >= 4 ? 0u : 8 * (4 - w);
    if (tri4) // k_ac_tri4: word index = umulhi(w * mul_lo, bytes), bit index = umulhi(w, mul_hi) & 31
    {
        T->mul_lo = quad ? HC1 : (HC1 << 8);  // tri: the zero low byte drops byte 3 of the word
        T->mul_hi = quad ? HC2 : (1u << 8);   // tri: w >> 24 (on the FMA pipe)
        T->mul_b = 0;
    }
    if (s == 2) // paired scheme (ac_pair_filter): mT masks T to w-2 bytes, mA to 2 bytes, mB to w-2 bytes
    {
        T->mul_lo = HC1 << (8 * (4 - (w - 2)));
        T->mul_hi = HC2 << 16;
        T->mul_b = 0xC2B2AE35u << (8 * (4 - (w - 2)));
    }

    // pattern pool (exact compare data) + window entries
    std::vector<uint32_t> off(K), len(K);
    std::vector<uint8_t> pv, pm;
    struct Ent { uint64_t key; uint32_t e; };
    std::vector<Ent> ents;
    std::vector<std::pair<uint32_t, uint32_t>> tri_bits; // tri4: (trigram, bits to set in its word)
    for (uint32_t k = 0; k < K; k++)
    {
        off[k] = (uint32_t)pv.size();
        len[k] = plan->pat_lens[k];
        const uint8_t *pb = (const uint8_t *)plan->patterns[k].data();
        for (uint32_t i = 0; i < len[k]; i++)
        {
            const uint8_t m = (!plan->case_sensitive && is_alpha_c(pb[i])) ? 0xDF : 0xFF;
            pm.push_back(m);
            pv.push_back(pb[i] & m);
        }
        if (len[k] == 0) continue;
        if (tri4)
        {
            // exact table of k_ac_tri4: keyed by the (folded) first 6 bytes of the pattern, value = pattern index
            ents.push_back({pat_window(pb, 6, T->fold) & 0xFFFFFFFFFFFFull, k});
            for (uint32_t d = 0; d < 4; d++)
            {
                if (quad)
                {
                    const uint32_t word = (uint32_t)pat_window(pb + d, 4, T->fold);
                    tri_bits.push_back({word, 1u << ((uint32_t)(((uint64_t)word * T->mul_hi) >> 32) & 31u)});
                    continue;
                }
                const uint32_t tri = (uint32_t)pat_window(pb + d, 3, T->fold) & 0xFFFFFFu;
                // (len, d) = (6, 3) does not know byte a+3: all 32 bits
                tri_bits.push_back({tri, len[k] - d >= 4 ? (1u << ((pb[d + 3] & T->fold) & 31u)) : 0xFFFFFFFFu});
            }
            continue;
        }
        for (uint32_t d = 0; d < s; d++) ents.push_back({pat_window(pb + d, w, T->fold) & T->wmask, (k << 2) | d});
    }
    std::stable_sort(ents.begin(), ents.end(), [](const Ent &a, const Ent &b) { return a.key < b.key; });
    size_t distinct = 0;
    for (size_t i = 0; i < ents.size(); i++)
        if (i == 0 || ents[i].key != ents[i - 1].key) distinct++;
    // bitmap size (bytes, any multiple of 16 — addresses come from mulhi, not masking): keep the false-positive
    // rate of one lookup around 0.2 % or better, 16 KB .. 192 KB of the SM's 227 KB shared memory
    uint32_t nby = 16u << 10;
    if (tri4)
    {
        // one 32-bit word per trigram: keep word occupancy around 7 % or less
        std::vector<uint32_t> tris;
        for (auto &tb : tri_bits) tris.push_back(tb.first);
        std::sort(tris.begin(), tris.end());
        const double ntri = (double)(std::unique(tris.begin(), tris.end()) - tris.begin());
        while (nby < (128u << 10) && ntri * 56.0 > (double)nby) nby *= 2;
        if (nby == (128u << 10) && ntri * 56.0 > (double)nby) nby = 176u << 10; // + 40-48 KB of candidate queues <= 227 KB
    }
    else
    {
        while (nby < (128u << 10) && (double)distinct / (double)(nby * 8.0) > 0.002) nby *= 2;
        if (nby == (128u << 10) && (double)distinct / (double)(nby * 8.0) > 0.0015) nby = 192u << 10;
    }
    T->bitmap_bytes = nby;
    std::vector<uint32_t> bitmap(nby / 4, 0);
    uint32_t nslots = 16;
    while (nslots < 8 * distinct + 1) nslots *= 2; // load factor <= 1/8: a miss (the common case) ends after ~1.1 probes
    T->nslots = nslots;
    std::vector<AcSlot> slots(nslots, AcSlot{0, 0, 0});
    std::vector<uint32_t> list(ents.size());
    for (size_t i = 0; i < ents.size();)
    {
        size_t j = i;
        while (j < ents.size() && ents[j].key == ents[i].key) { list[j] = ents[j].e; j++; }
        const uint32_t lo = (uint32_t)ents[i].key, hi = (uint32_t)(ents[i].key >> 32);
        if (tri4)
        {
        }
        else if (s == 2)
        {
            // window bytes c0..c(w-1) as a 64-bit little-endian value
            const uint64_t c = ents[i].key;
            const uint32_t tl = w - 2, tmask = tl >= 4 ? 0xFFFFFFFFu : ((1u << (8 * tl)) - 1);
            auto word_of = [&](uint32_t t) { return (uint32_t)(((uint64_t)(t * T->mul_lo) * nby) >> 32) >> 2; };
            auto top4 = [](uint32_t x) { return (uint32_t)(((uint64_t)x * 16u) >> 32); };
            const uint32_t first2 = (uint32_t)(c & 0xFFFF), lastT = (uint32_t)(c >> 16) & tmask;
            const uint32_t firstT = (uint32_t)c & tmask;
            bitmap[word_of(lastT)] |= 1u << top4(first2 * T->mul_hi);               // A view
            bitmap[word_of(firstT)] |= 1u << (16 + top4(lastT * T->mul_b));          // B view (bytes 2..w-1)
        }
        else
        {
            const uint32_t hsh = lo * T->mul_lo + hi * T->mul_hi;
            const uint32_t baddr = (uint32_t)(((uint64_t)hsh * nby) >> 32); // byte address in the bitmap
            const uint32_t bit = (s == 1 ? (hsh >> T->bit_shift) : hsh) & 7;
            bitmap[baddr >> 2] |= 1u << (8 * (baddr & 3) + bit);
        }
        uint32_t h = (tri4 ? lo * HC1 + hi * HC2 : slot_hash(lo, hi)) & (nslots - 1);
        while (slots[h].count) h = (h + 1) & (nslots - 1);
        slots[h] = AcSlot{ents[i].key, (uint32_t)i, (uint32_t)(j - i)};
        i = j;
    }
    for (auto &tb : tri_bits) bitmap[(uint32_t)(((uint64_t)(tb.first * T->mul_lo) * nby) >> 32) >> 2] |= tb.second;
    if (tri4 && !tri_bits.empty())
    {
        const uint32_t span = quad ? 0xFFFFFFFFu : 0x00FFFFFFu; // bytes of the word every entry knows
        uint32_t agree = span;
        for (auto &tb : tri_bits) agree &= ~(tb.first ^ tri_bits[0].first);
        T->cls_mask = agree & span;
        T->cls_val = tri_bits[0].first & T->cls_mask;
    }
    if (tri4)
    {
        std::vector<uint8_t> b2(1u << 20, 0); // bit index = top 23 bits of prefix_hash
        for (auto &e : ents)
        {
            const uint32_t hsh = (uint32_t)e.key * HC1 + (uint32_t)(e.key >> 32) * HC2;
            b2[hsh >> 12] |= (uint8_t)(1u << ((hsh >> 9) & 7u));
        }
        H->bitmap2.swap(b2);
    }
    if (pv.empty()) { pv.push_back(0); pm.push_back(0); }
    if (list.empty()) list.push_back(0);
    if (off.empty()) { off.push_back(0); len.push_back(0); }
    H->bitmap.swap(bitmap);
    H->slots.swap(slots);
    H->list.swap(list);
    H->pool_val.swap(pv);
    H->pool_mask.swap(pm);
    H->pat_off.swap(off);
    H->pat_len.swap(len);
    char name[96];
    snprintf(name, sizeof name, "window%u/stride%u%s bitmap %uKB%s", w, s, tri4 ? (quad ? " aligned-word hash" : " tri4+byte-select") : (s == 2 ? " paired" : ""), nby >> 10,
             plan->case_sensitive ? "" : " fold");
    plan->filter_name = name;
    return 0;
}

void ac_free_tables(Plan *plan)
{
    delete plan->ach;
    plan->ach = nullptr;
}

template <typename T>
static bool upload(T **dst, const std::vector<T> &src)
{
    if (src.empty()) return true;
    return cudaMalloc(dst, src.size() * sizeof(T)) == cudaSuccess &&
           cudaMemcpy(*dst, src.data(), src.size() * sizeof(T), cudaMemcpyHostToDevice) == cudaSuccess;
}

AcDevTables *ac_upload_tables(const Plan *plan)
{
    const AcHostTables *H = plan->ach;
    AcDevTables *T = new AcDevTables(H->proto);
    if (upload(&T->d_bitmap, H->bitmap) && upload(&T->d_bitmap2, H->bitmap2) && upload(&T->d_slots, H->slots) &&
        upload(&T->d_list, H->list) && upload(&T->d_pool_val, H->pool_val) && upload(&T->d_pool_mask, H->pool_mask) &&
        upload(&T->d_pat_off, H->pat_off) && upload(&T->d_pat_len, H->pat_len))
        return T;
    set_error(-2, "CUDA allocation/copy failed uploading the pattern-set tables");
    ac_free_device(T);
    return nullptr;
}

void ac_free_device(AcDevTables *T)
{
    if (!T) return;
    cudaFree(T->d_bitmap);
    cudaFree(T->d_bitmap2);
    cudaFree(T->d_slots);
    cudaFree(T->d_list);
    cudaFree(T->d_pool_val);
    cudaFree(T->d_pool_mask);
    cudaFree(T->d_pat_off);
    cudaFree(T->d_pat_len);
    delete T;
}

void launch_ac(const Plan *plan, const AcDevTables *T, const AcLaunch &a, int sm_count, cudaStream_t st)
{
    (void)plan;
    AcDev A;
    memset(&A, 0, sizeof A);
    A.bitmap = T->d_bitmap;
    A.bitmap2 = T->d_bitmap2;
    A.slots = T->d_slots;
    A.list = T->d_list;
    A.pool_val = T->d_pool_val;
    A.pool_mask = T->d_pool_mask;
    A.pat_off = T->d_pat_off;
    A.pat_len = T->d_pat_len;
    A.bitmap_bytes = T->bitmap_bytes;
    A.nslots = T->nslots;
    A.w = T->w;
    A.npat = T->npat;
    A.wmask_lo = (uint32_t)T->wmask;
    A.wmask_hi = (uint32_t)(T->wmask >> 32);
    A.fold = T->fold;
    A.mul_lo = T->mul_lo;
    A.mul_hi = T->mul_hi;
    A.bit_shift = T->bit_shift;
    A.mul_b = T->mul_b;
    A.cls_mask = T->cls_mask;
    A.cls_val = T->cls_val;
    A.text = a.text;
    A.avail_len = a.avail_len;
    A.own_begin = a.own_begin;
    A.own_end = a.own_end;
    A.global_offset = a.global_offset;
    A.prev_byte = a.prev_byte;
    A.next_byte = a.next_byte;
    A.out = a.out;
    A.cap = a.cap;
    A.counter = a.counter;
    A.whole_word = a.whole_word;
    A.want_positions = a.want_positions;
    // vector groups need the 16-byte vector plus 8 following bytes in bounds
    const uint64_t total_groups = a.avail_len >= 24 ? (a.avail_len - 24) / 16 + 1 : 0;
    A.tail_a = total_groups * 16;
    A.group_begin = a.own_begin / 16;
    A.group_end = (a.own_end + 3) / 16 + 1; // sampled window of an owned start lies < own_end + s
    if (A.group_end > total_groups) A.group_end = total_groups;
    if (A.group_begin > A.group_end) A.group_begin = A.group_end;

    if (T->tri4)
    {
        constexpr int UNROLL = 4;
        // CTA size: KREP_B200_AC_THREADS = 640 (default: 96 registers, no spills) | 768; L2 prefetch distance: KREP_B200_AC_PF (tiles, 0 = off)
        static int threads = 0, pf_dist = 4;
        if (!threads)
        {
            if (const char *v = getenv("KREP_B200_AC_PF")) pf_dist = atoi(v);
            const char *e = getenv("KREP_B200_AC_THREADS");
            threads = e && atoi(e) == 768 ? 768 : 640;
        }
        A.pf_dist = (uint32_t)pf_dist;
        const uint64_t full_groups = a.avail_len / 16; // a lookup only needs its own aligned word
        A.tail_a = full_groups * 16;
        A.group_begin = a.own_begin / 16;
        A.group_end = (a.own_end + 3) / 16 + 1; // aligned window position of an owned start lies < own_end + 4
        if (A.group_end > full_groups) A.group_end = full_groups;
        if (A.group_begin > A.group_end) A.group_begin = A.group_end;
        const size_t smem = (size_t)T->bitmap_bytes + (size_t)(threads / 32) * TRI4_QCAP * TRI4_ENTRY;
        const bool f = T->fold != 0xFFFFFFFFu;
        void (*kernel)(AcDev) = nullptr;
        if (threads == 768) kernel = f ? k_ac_tri4<true, 768> : k_ac_tri4<false, 768>;
        else kernel = f ? k_ac_tri4<true, 640> : k_ac_tri4<false, 640>;
        cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        // queue entries hold 32-bit relative group indices: at most 2^31 groups (32 GiB) per launch
        const uint64_t gb = A.group_begin, ge = A.group_end, max_groups = 1ull << 31;
        const uint64_t tile = (uint64_t)threads * UNROLL;
        uint64_t b0 = gb;
        do
        {
            const uint64_t e0 = ge - b0 > max_groups ? b0 + max_groups : ge;
            A.group_begin = b0;
            A.group_end = e0;
            A.zero = b0 == gb ? 0u : 1u; // the first launch also scans the tail bytes
            uint64_t blocks = (e0 - b0 + tile - 1) / tile;
            if (blocks == 0) blocks = 1;
            if (blocks > (uint64_t)sm_count) blocks = sm_count;
            kernel<<<(unsigned)blocks, threads, smem, st>>>(A);
            count_launch();
            b0 = e0;
        } while (b0 < ge);
        return;
    }
    constexpr int THREADS = 640, UNROLL = 4;
    {
        static int pf = -1;
        if (pf < 0)
        {
            const char *v = getenv("KREP_B200_AC_PF");
            pf = v ? atoi(v) : 4;
        }
        A.pf_dist = (uint32_t)pf;
    }
    const size_t smem = (size_t)T->bitmap_bytes + 128 + (size_t)(THREADS / 32) * AcQueue<UNROLL>::CAP * sizeof(uint64_t);
    auto kernel = [&]() -> void (*)(AcDev) {
        const bool f = T->fold != 0xFFFFFFFFu;
        if (T->s == 1) return f ? k_ac_scan<1, true, THREADS, UNROLL> : k_ac_scan<1, false, THREADS, UNROLL>;
        if (T->s == 2) return f ? k_ac_scan<2, true, THREADS, UNROLL> : k_ac_scan<2, false, THREADS, UNROLL>;
        return f ? k_ac_scan<4, true, THREADS, UNROLL> : k_ac_scan<4, false, THREADS, UNROLL>;
    }();
    cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    const uint64_t groups = A.group_end - A.group_begin;
    const uint64_t tile = (uint64_t)THREADS * UNROLL;
    uint64_t blocks = (groups + tile - 1) / tile;
    if (blocks == 0) blocks = 1;
    if (blocks > (uint64_t)sm_count) blocks = sm_count; // one resident CTA per SM (shared-memory bitmap)
    kernel<<<(unsigned)blocks, THREADS, smem, st>>>(A);
    count_launch();
}

} // namespace kb
