// lit_filters.cuh — device helpers shared by the single-literal kernels (scan_literal.cu: occurrence lists;
// scan_count.cu: fused -c line counting): the two streaming filters and the exact verifier.
#pragma once
#include "common.h"

namespace kb {

__device__ __forceinline__ bool dev_is_word(int c)
{
    return (c >= '0' && c <= '9') || (c >= 'A' && c <= 'Z') || (c >= 'a' && c <= 'z') || c == '_';
}

// Exact check of one candidate start: ownership by start offset, all pattern bytes under the per-byte case mask, the
// whole-word boundary against the global text (shard context bytes at the edges).  Returns 0 when `cand` is not an
// occurrence this shard owns (or fails -w in drop mode), else 0x8 | full << 2 | ws_ok << 1 | we_ok (the key's tag bits).
__device__ __forceinline__ unsigned verify_exact(const LitDevParams &p, long long cand)
{
    if (cand < (long long)p.own_begin || cand >= (long long)p.own_end) return 0;
    const uint64_t c = (uint64_t)cand;
    if (c + p.emit_len > p.avail_len) return 0;
    const uint8_t *t = p.text + c;
    const uint8_t *val = p.pat_val, *msk = p.pat_mask;
    for (uint32_t k = 0; k < p.emit_len; k++)
        if ((t[k] & msk[k]) != val[k]) return 0;
    unsigned full = 1;
    if (p.m > p.emit_len)
    {
        if (c + p.m > p.avail_len) full = 0;
        else
            for (uint32_t k = p.emit_len; k < p.m; k++)
                if ((t[k] & msk[k]) != val[k]) { full = 0; break; }
    }
    unsigned ww_tag = 3; // ws_ok << 1 | we_ok
    if (p.whole_word)
    {
        const uint64_t e = c + p.m;
        const int pb = c > 0 ? (int)t[-1] : p.prev_byte;
        const int nb = e < p.avail_len ? (int)p.text[e] : p.next_byte;
        ww_tag = (dev_is_word(pb) ? 0u : 2u) | (dev_is_word(nb) ? 0u : 1u);
        if (p.whole_word == 1 && ww_tag != 3) return 0;
    }
    return 8u | (full << 2) | ww_tag;
}

__device__ __forceinline__ uint4 ld_stream(const uint4 *ptr)
{
    return __ldcs(ptr); // ld.global.cs: streamed once, evict-first
}

// ------------------------------------------------------------------------------------ ALIGNED4
template <bool FOLD>
__device__ __forceinline__ bool hit_word(uint32_t w, uint32_t fold, uint32_t k0, uint32_t k1, uint32_t k2, uint32_t k3)
{
    if (FOLD) w &= fold;
    return (w == k0) | (w == k1) | (w == k2) | (w == k3);
}
template <bool FOLD>
__device__ __forceinline__ bool hit_vec(const uint4 &v, uint32_t fold, uint32_t k0, uint32_t k1, uint32_t k2, uint32_t k3)
{
    return hit_word<FOLD>(v.x, fold, k0, k1, k2, k3) | hit_word<FOLD>(v.y, fold, k0, k1, k2, k3) |
           hit_word<FOLD>(v.z, fold, k0, k1, k2, k3) | hit_word<FOLD>(v.w, fold, k0, k1, k2, k3);
}

// ------------------------------------------------------------------------------------ WINDOW4
// The 4-byte window at byte offset 4k+r is (lo >> 8r) | (hi << (32-8r)).  A funnel shift would put it on the ALU
// pipe next to the compares (SHF/LOP3/ISETP all issue there at half rate).  The
// same value is umulhi(lo, 2^(32-8r)) + hi * 2^(32-8r) — an IMAD.HI and an IMAD on the FMA pipe —
// so per text word the ALU pipe only sees the case fold (one LOP3, -i only) and the four compares.  The
// multipliers come from kernel parameters so that the compiler cannot strength-reduce them back into shifts.
template <bool MASKED>
__device__ __forceinline__ bool hit_pair(uint32_t lo, uint32_t hi, uint32_t mask, uint32_t k0, uint32_t c1, uint32_t c2,
                                         uint32_t c3)
{
    uint32_t x0 = lo, x1 = hi * c1 + __umulhi(lo, c1), x2 = hi * c2 + __umulhi(lo, c2), x3 = hi * c3 + __umulhi(lo, c3);
    if (MASKED)
    {
        x0 &= mask; x1 &= mask; x2 &= mask; x3 &= mask;
    }
    return (x0 == k0) | (x1 == k0) | (x2 == k0) | (x3 == k0);
}
template <bool FOLD, bool MASKED>
__device__ __forceinline__ bool hit_vec_w(const uint4 &v, uint32_t nx, uint32_t fold, uint32_t mask, uint32_t k0,
                                          uint32_t c1, uint32_t c2, uint32_t c3)
{
    uint32_t w0 = v.x, w1 = v.y, w2 = v.z, w3 = v.w, w4 = nx;
    if (FOLD)
    {
        w0 &= fold; w1 &= fold; w2 &= fold; w3 &= fold; w4 &= fold;
    }
    return hit_pair<MASKED>(w0, w1, mask, k0, c1, c2, c3) | hit_pair<MASKED>(w1, w2, mask, k0, c1, c2, c3) |
           hit_pair<MASKED>(w2, w3, mask, k0, c1, c2, c3) | hit_pair<MASKED>(w3, w4, mask, k0, c1, c2, c3);
}


} // namespace kb
