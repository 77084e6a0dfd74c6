// scan_regex.cuh — device helpers of the -E line walks shared by k_regex_lines (scan_regex.cu) and the long-line pass
// (scan_regex_long.cu).
#pragma once
#include "common.h"

namespace kb {

// The aligned 16 bytes around the last position read, in registers.
struct Window
{
    const uint8_t *text;
    uint64_t avail;
    uint64_t base;
    uint4 v;

    __device__ __forceinline__ void load(uint64_t b)
    {
        base = b;
        if (b + 16 <= avail)
        {
            v = __ldg(reinterpret_cast<const uint4 *>(text + b));
            return;
        }
        uint32_t w[4] = {0, 0, 0, 0};
#pragma unroll
        for (int k = 0; k < 16; k++)
            if (b + k < avail) w[k >> 2] |= (uint32_t)text[b + k] << ((k & 3) * 8);
        v = make_uint4(w[0], w[1], w[2], w[3]);
    }
    __device__ __forceinline__ uint32_t at(uint64_t q)
    {
        const uint64_t b = q & ~15ull;
        if (b != base) load(b);
        const uint32_t i = (uint32_t)q & 15u;
        const uint32_t w = (i & 8) ? ((i & 4) ? v.w : v.z) : ((i & 4) ? v.y : v.x);
        return (w >> ((i & 3) * 8)) & 0xFFu;
    }
};

__device__ __forceinline__ bool has_newline(uint4 v)
{
    auto z = [](uint32_t x) {
        x ^= 0x0A0A0A0Au;
        return (x - 0x01010101u) & ~x & 0x80808080u;
    };
    return (z(v.x) | z(v.y) | z(v.z) | z(v.w)) != 0;
}

// The rows of the G automata of a split plan in one line walk, and the line's state from them in the row convention of
// one automaton whose DEAD row is 1: 0 = MATCHED (one automaton matched), 1 = DEAD (all are dead), 2 = live.
template <int G>
struct SetRows
{
    uint32_t r[G];

    __device__ __forceinline__ uint32_t state(const RegexLaunch &a) const
    {
        bool matched = false, live = false;
#pragma unroll
        for (int g = 0; g < G; g++)
        {
            matched |= r[g] == 0;
            live |= r[g] > a.grp[g].nclasses;
        }
        return matched ? 0u : live ? 2u : 1u;
    }
    __device__ __forceinline__ void begin(const RegexLaunch &a)
    {
#pragma unroll
        for (int g = 0; g < G; g++) r[g] = a.grp[g].start;
    }
    // G independent lookups: a DEAD automaton steps to DEAD
    __device__ __forceinline__ void step(const RegexLaunch &a, const uint16_t *img, uint32_t b)
    {
        const uint8_t *bytes = reinterpret_cast<const uint8_t *>(img);
#pragma unroll
        for (int g = 0; g < G; g++) r[g] = img[a.grp[g].trans + r[g] + bytes[a.grp[g].cls * 2 + b]];
    }
    // the '\n' column: 0 where the automaton accepts at the end of the line, DEAD elsewhere (and for a DEAD one)
    __device__ __forceinline__ void end_of_line(const RegexLaunch &a, const uint16_t *img)
    {
#pragma unroll
        for (int g = 0; g < G; g++) r[g] = img[a.grp[g].trans + r[g] + a.grp[g].nl_class];
    }
};

} // namespace kb
