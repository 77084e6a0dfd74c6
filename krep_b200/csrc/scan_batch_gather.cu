// scan_batch_gather.cu — packs HBM-resident texts into one batch buffer on sm_90a (DESIGN §12.9).
//
// krep_b200_search_batch_resident / krep_b200_regex_search_batch_resident take texts that already live in device memory
// (d_base[src[t] .. src[t] + len[t]), any alignment, any order, overlapping or repeated).  The batch paths scan one packed
// buffer: text t at the 16-byte aligned dst[t] (pack_layout, host_api.cu), followed by fill bytes up to dst[t + 1] (or
// the total).  k_batch_gather writes that buffer byte for byte as the host's pack_texts would:
//   - a thread per 16 output bytes, one aligned 16-byte store; a long text is spread over as many threads and CTAs as it
//     has vectors, and a vector of gap bytes is written by the same threads;
//   - the source is read as two aligned 16-byte loads and a funnel shift, so any alignment of d_base works.  The first
//     load of a text may read up to 15 bytes before its start: they lie in the same 16-byte granule, so in the same
//     allocation (device allocations start at least 256-byte aligned).  A load that would pass the text's end reads
//     byte by byte instead, since a text may end where its allocation ends;
//   - each CTA finds the texts its 4 KiB of output covers with one binary search over dst[], and each thread searches
//     only that range;
//   - the thread that writes a text's last byte also stores it in last[t] (when last is given): the windowed -E replay
//     needs it for the empty string after a final '\n'.
#include "common.h"

namespace kb {

namespace {

constexpr int BG_THREADS = 256;

// The last t in [lo, hi] with dst[t] <= o (dst[lo] <= o holds).
__device__ __forceinline__ uint32_t text_at(const uint64_t *__restrict__ dst, uint32_t lo, uint32_t hi, uint64_t o)
{
    while (lo < hi)
    {
        const uint32_t mid = (lo + hi + 1) >> 1;
        if (__ldg(dst + mid) <= o) lo = mid;
        else hi = mid - 1;
    }
    return lo;
}

__device__ __forceinline__ uint4 load_src(const uint8_t *p, const uint8_t *end) // p 16-byte aligned; bytes at or past end read as 0
{
    if (p + 16 <= end) return __ldg(reinterpret_cast<const uint4 *>(p));
    uint32_t w[4] = {0, 0, 0, 0};
#pragma unroll
    for (int k = 0; k < 16; k++)
        if (p + k < end) w[k >> 2] |= (uint32_t)p[k] << ((k & 3) * 8);
    return make_uint4(w[0], w[1], w[2], w[3]);
}

__device__ __forceinline__ uint32_t pick(const uint32_t (&w)[8], uint32_t i)
{
    uint32_t r = w[0];
#pragma unroll
    for (uint32_t k = 1; k < 8; k++) r = i == k ? w[k] : r;
    return r;
}

__global__ void __launch_bounds__(BG_THREADS) k_batch_gather(const uint8_t *__restrict__ base, const uint64_t *__restrict__ src,
                                                             const uint64_t *__restrict__ dst, const uint64_t *__restrict__ len,
                                                             uint32_t nt, uint64_t nvec, uint32_t fill, uint4 *__restrict__ out,
                                                             uint8_t *__restrict__ last)
{
    __shared__ uint32_t s_range[2];
    const uint64_t v0 = (uint64_t)blockIdx.x * BG_THREADS;
    if (threadIdx.x < 2)
    {
        const uint64_t o = threadIdx.x == 0 ? v0 * 16 : ((v0 + BG_THREADS < nvec ? v0 + BG_THREADS : nvec) - 1) * 16;
        s_range[threadIdx.x] = text_at(dst, 0, nt - 1, o);
    }
    __syncthreads();
    const uint64_t v = v0 + threadIdx.x;
    if (v >= nvec) return;
    const uint64_t o = v * 16;
    const uint32_t t = text_at(dst, s_range[0], s_range[1], o);
    const uint64_t in = o - __ldg(dst + t), n = __ldg(len + t);
    const uint32_t fw = fill * 0x01010101u;
    uint32_t r[4] = {fw, fw, fw, fw};
    if (in < n)
    {
        const uint32_t valid = n - in < 16 ? (uint32_t)(n - in) : 16u;
        const uint8_t *s = base + __ldg(src + t) + in, *end = base + __ldg(src + t) + n;
        const uint8_t *a = reinterpret_cast<const uint8_t *>((uintptr_t)s & ~(uintptr_t)15);
        const uint32_t sh = (uint32_t)((uintptr_t)s & 15);
        const uint4 x0 = load_src(a, end);
        const uint4 x1 = sh + valid > 16 ? load_src(a + 16, end) : make_uint4(0, 0, 0, 0);
        const uint32_t w[8] = {x0.x, x0.y, x0.z, x0.w, x1.x, x1.y, x1.z, x1.w};
        const uint32_t ws = sh >> 2, bs = (sh & 3) * 8;
#pragma unroll
        for (uint32_t k = 0; k < 4; k++)
        {
            const uint32_t b = __funnelshift_r(pick(w, k + ws), pick(w, k + ws + 1), bs);
            const int keep = (int)valid - 4 * (int)k; // bytes of this word that belong to the text; the rest are fill
            if (keep >= 4) r[k] = b;
            else if (keep > 0)
            {
                const uint32_t m = (1u << (8 * keep)) - 1u;
                r[k] = (b & m) | (fw & ~m);
            }
        }
        if (last && in + 16 >= n) last[t] = end[-1];
    }
    out[v] = make_uint4(r[0], r[1], r[2], r[3]);
}

} // namespace

int batch_gather(const void *d_base, const uint64_t *d_tab, uint32_t nt, uint64_t total, uint8_t fill, uint8_t *d_out,
                 uint8_t *d_last, cudaStream_t st)
{
    if (nt == 0 || total == 0) return 0;
    const uint64_t nvec = total / 16;
    const uint64_t grid = (nvec + BG_THREADS - 1) / BG_THREADS;
    k_batch_gather<<<(unsigned)grid, BG_THREADS, 0, st>>>((const uint8_t *)d_base, d_tab, d_tab + nt, d_tab + 2 * (uint64_t)nt, nt, nvec,
                                                          fill, reinterpret_cast<uint4 *>(d_out), d_last);
    count_launch();
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess)
    {
        set_error(-2, "CUDA error %s in the batch gather (%s)", cudaGetErrorName(e), cudaGetErrorString(e));
        return -2;
    }
    return 0;
}

} // namespace kb
