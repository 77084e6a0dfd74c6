// line_rec.cuh — the fused -c line record (krep_b200_line_count_t on the device) and its fold, plus the newline masks the
// kernels that compute it share (scan_count.cu: single literals, scan_set_count.cu: pattern sets).
#pragma once
#include <stdint.h>

namespace kb {

enum : uint32_t
{
    LR_HAS_HIT = 1,      // at least one owned occurrence
    LR_FIRST_OPEN = 2,   // the first occurrence lies before the first newline of the range (its line began earlier)
    LR_LAST_PENDING = 4, // no newline between the last occurrence and the end of the range (its line goes on)
    LR_HAS_NL = 8        // the range holds a newline (only meaningful, and only computed, for ranges without a hit)
};

struct LineRec
{
    uint32_t lines, flags;
};

// (lines, flags) of range A followed by range B
__host__ __device__ __forceinline__ void append_rec(uint64_t &lines, uint32_t &flags, uint64_t blines, uint32_t bflags)
{
    const bool ah = flags & LR_HAS_HIT, bh = bflags & LR_HAS_HIT;
    if (!bh)
    {
        if (ah && (bflags & LR_HAS_NL)) flags &= ~(uint32_t)LR_LAST_PENDING;
        flags |= bflags & LR_HAS_NL;
        return;
    }
    if (!ah)
    {
        const bool had_nl = flags & LR_HAS_NL;
        lines = blines;
        flags = bflags | LR_HAS_NL * had_nl;
        if (had_nl) flags &= ~(uint32_t)LR_FIRST_OPEN;
        return;
    }
    lines += blines;
    if ((flags & LR_LAST_PENDING) && (bflags & LR_FIRST_OPEN)) lines--; // one line, counted on both sides of the cut
    flags = LR_HAS_HIT | LR_HAS_NL | (flags & LR_FIRST_OPEN) | (bflags & LR_LAST_PENDING);
}

#ifdef __CUDACC__
// 4-bit mask of the bytes of w that equal '\n' (exact per byte)
__device__ __forceinline__ uint32_t nl_nibble(uint32_t w)
{
    const uint32_t x = w ^ 0x0A0A0A0Au;
    const uint32_t y = ~(((x & 0x7F7F7F7Fu) + 0x7F7F7F7Fu) | x | 0x7F7F7F7Fu); // 0x80 in every zero byte of x
    return ((y >> 7) * 0x10204080u) >> 28;
}
__device__ __forceinline__ uint32_t nl_mask16(const uint4 &v)
{
    return nl_nibble(v.x) | (nl_nibble(v.y) << 4) | (nl_nibble(v.z) << 8) | (nl_nibble(v.w) << 12);
}
// bits of a 16-byte unit at byte position `unit` that lie inside [lo, hi)
__device__ __forceinline__ uint32_t range_mask16(uint64_t unit, uint64_t lo, uint64_t hi)
{
    uint32_t m = 0xFFFFu;
    if (unit < lo) m = lo - unit >= 16 ? 0u : (m & ~((1u << (uint32_t)(lo - unit)) - 1u));
    if (unit + 16 > hi) m = hi <= unit ? 0u : (m & ((1u << (uint32_t)(hi - unit)) - 1u));
    return m;
}
#endif

} // namespace kb
