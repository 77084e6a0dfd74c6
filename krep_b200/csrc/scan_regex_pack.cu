// scan_regex_pack.cu — the -E row of a resident shard on sm_90a (DESIGN §12.4; layout: RegexRowHeader, csrc/common.h).
//
// After a k_regex_lines scan, glibc still has to see some lines: every flagged line (filter mode), or the uncertain ones
// (count and match mode).  A resident shard has no host copy of its text, so the bytes of exactly those lines are packed
// here into one row that comes back in one copy:
//   1. k_pack_lines    — a warp per listed line finds its '\n' (up to avail_len) with 16-byte loads and one ballot per
//                        512 bytes; O(length) per line, lines of any length, no warp waits for another.  One more warp
//                        finds the head (own_begin up to its first '\n') when the shard starts mid-line;
//   2. k_seg_marks + an exclusive scan (CUB) — lines that abut (end + 1 == next start) merge into segments;
//   3. k_seg_bounds, k_seg_sizes + an exclusive scan — each segment's bytes and its 16-byte aligned place in the row;
//   4. k_pack_copy     — a thread per 16 output bytes: two aligned 16-byte loads of the text, a funnel shift, one aligned
//                        16-byte store; a long segment is spread over as many threads (and CTAs) as it has vectors;
//   5. k_row_fill      — the header and the segment table; the keys are one device-to-device copy.
#include <cub/device/device_scan.cuh>
#include <cub/device/device_select.cuh>
#include <algorithm>
#include <cstring>
#include "common.h"
#include "engine.h"

namespace kb {

struct RegexPackBufs
{
    uint64_t cap = 0;                       // entries of the per-line arrays
    uint64_t *sel = nullptr, *le = nullptr; // listed line keys, their ends (exclusive, relative to d_text)
    uint32_t *flag = nullptr, *segid = nullptr;
    uint64_t *seg_start = nullptr, *seg_end = nullptr, *plen = nullptr, *seg_off = nullptr;
    uint64_t *meta = nullptr;   // device: PM_* words
    uint64_t *h_meta = nullptr; // pinned
    void *tmp = nullptr;
    size_t tmp_bytes = 0;
    uint8_t *row = nullptr;
    uint64_t row_cap = 0;
    uint8_t *h_row = nullptr; // pinned
    uint64_t h_row_cap = 0;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
};

namespace {

enum { PM_NSEL = 0, PM_NSEG = 1, PM_SEG_BYTES = 2, PM_HEAD_LEN = 3, PM_FLAGS = 4, PM_WORDS = 8 };
constexpr int PK_THREADS = 256;

struct PackGeo
{
    const uint8_t *text;
    uint64_t avail, own_begin, own_end, G;
    int32_t prev_byte, next_byte;
    int shift; // key >> shift = global line start
};

__device__ __forceinline__ uint4 load_vec(const uint8_t *text, uint64_t avail, uint64_t q) // aligned q; zero past avail
{
    if (q + 16 <= avail) return __ldg(reinterpret_cast<const uint4 *>(text + q));
    uint32_t w[4] = {0, 0, 0, 0};
#pragma unroll
    for (int k = 0; k < 16; k++)
        if (q + k < avail) w[k >> 2] |= (uint32_t)text[q + k] << ((k & 3) * 8);
    return make_uint4(w[0], w[1], w[2], w[3]);
}

__device__ __forceinline__ uint32_t nl_bits(uint32_t x) // bit k: byte k of x is '\n'
{
    const uint32_t e = __vcmpeq4(x, 0x0A0A0A0Au);
    return ((e >> 7) & 1u) | ((e >> 14) & 2u) | ((e >> 21) & 4u) | ((e >> 28) & 8u);
}

// Position of the first '\n' in [p, lim), or lim.  Called by a whole warp with the same p and lim.
__device__ uint64_t warp_find_nl(const uint8_t *text, uint64_t avail, uint64_t p, uint64_t lim, uint32_t lane)
{
    for (uint64_t base = p & ~15ull; base < lim; base += 512)
    {
        const uint64_t q = base + (uint64_t)lane * 16;
        uint32_t m = 0;
        if (q < lim)
        {
            const uint4 v = load_vec(text, avail, q);
            m = nl_bits(v.x) | (nl_bits(v.y) << 4) | (nl_bits(v.z) << 8) | (nl_bits(v.w) << 12);
            if (q < p) m &= 0xFFFFu << (uint32_t)(p - q);
            if (lim - q < 16) m &= (1u << (uint32_t)(lim - q)) - 1u;
        }
        const uint32_t b = __ballot_sync(0xFFFFFFFFu, m != 0);
        if (b)
        {
            const int l = __ffs(b) - 1;
            const uint32_t ml = __shfl_sync(0xFFFFFFFFu, m, l);
            return base + (uint64_t)l * 16 + (uint64_t)(__ffs(ml) - 1);
        }
    }
    return lim;
}

// 1. Line ends of the listed lines (warp w < nsel), and the head and the row flags (warp nsel).
__global__ void __launch_bounds__(PK_THREADS) k_pack_lines(const PackGeo g, const uint64_t *__restrict__ sel, uint64_t *__restrict__ le,
                                                           uint64_t *__restrict__ meta)
{
    const uint32_t lane = threadIdx.x & 31;
    const uint64_t nwarps = ((uint64_t)gridDim.x * blockDim.x) >> 5;
    const uint64_t nsel = meta[PM_NSEL];
    for (uint64_t w = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; w <= nsel; w += nwarps)
    {
        if (w == nsel)
        {
            const int before = g.own_begin == 0 ? g.prev_byte : (int)g.text[g.own_begin - 1];
            uint64_t head = 0, flags = 0;
            if (before >= 0 && before != '\n')
            {
                const uint64_t e = warp_find_nl(g.text, g.avail, g.own_begin, g.own_end, lane);
                head = (e < g.own_end ? e + 1 : g.own_end) - g.own_begin;
                flags |= ROW_HEAD;
            }
            if (g.next_byte < 0 && g.own_end >= g.avail)
            {
                flags |= ROW_LAST;
                if (g.avail) flags |= (uint64_t)g.text[g.avail - 1] << ROW_LAST_BYTE_SHIFT;
            }
            if (lane == 0)
            {
                meta[PM_HEAD_LEN] = head;
                meta[PM_FLAGS] = flags;
            }
            continue;
        }
        const uint64_t p = (sel[w] >> g.shift) - g.G;
        const uint64_t e = warp_find_nl(g.text, g.avail, p, g.avail, lane);
        if (lane == 0) le[w] = e < g.avail ? e + 1 : g.avail;
    }
}

// 2. A segment starts at every listed line that does not begin where the previous one ended.
__global__ void k_seg_marks(const PackGeo g, const uint64_t *__restrict__ sel, const uint64_t *__restrict__ le, uint64_t n,
                            const uint64_t *__restrict__ meta, uint32_t *__restrict__ flag)
{
    const uint64_t nsel = meta[PM_NSEL];
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x)
        flag[i] = i < nsel && (i == 0 || le[i - 1] != (sel[i] >> g.shift) - g.G) ? 1u : 0u;
}

// 3a. Each segment's first byte (from its first line) and end (from its last line); the number of segments.
__global__ void k_seg_bounds(const PackGeo g, const uint64_t *__restrict__ sel, const uint64_t *__restrict__ le,
                             const uint32_t *__restrict__ flag, const uint32_t *__restrict__ segid, uint64_t *__restrict__ seg_start,
                             uint64_t *__restrict__ seg_end, uint64_t *__restrict__ meta)
{
    const uint64_t nsel = meta[PM_NSEL];
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nsel; i += (uint64_t)gridDim.x * blockDim.x)
    {
        const uint32_t s = segid[i] + flag[i] - 1; // segid: segment starts before line i (exclusive), so i's segment
        if (flag[i]) seg_start[s] = (sel[i] >> g.shift) - g.G;
        if (i + 1 == nsel || flag[i + 1]) seg_end[s] = le[i];
        if (i + 1 == nsel) meta[PM_NSEG] = (uint64_t)s + 1;
    }
}

// 3b. Padded byte counts (0 past the last segment, so that one scan over all n entries gives the offsets).
__global__ void k_seg_sizes(const uint64_t *__restrict__ seg_start, const uint64_t *__restrict__ seg_end, uint64_t n,
                            const uint64_t *__restrict__ meta, uint64_t *__restrict__ plen)
{
    const uint64_t nseg = meta[PM_NSEG];
    for (uint64_t s = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; s < n; s += (uint64_t)gridDim.x * blockDim.x)
        plen[s] = s < nseg ? round16(seg_end[s] - seg_start[s]) : 0;
}

__global__ void k_seg_total(const uint64_t *__restrict__ plen, const uint64_t *__restrict__ seg_off, uint64_t *__restrict__ meta)
{
    const uint64_t nseg = meta[PM_NSEG];
    meta[PM_SEG_BYTES] = nseg ? seg_off[nseg - 1] + plen[nseg - 1] : 0;
}

__device__ __forceinline__ uint32_t pick(const uint32_t (&w)[8], uint32_t i)
{
    uint32_t r = w[0];
#pragma unroll
    for (uint32_t k = 1; k < 8; k++) r = i == k ? w[k] : r;
    return r;
}

// 4. Output vector v of the packed bytes: the head's vectors first, then each segment's.
__global__ void __launch_bounds__(PK_THREADS) k_pack_copy(const PackGeo g, const uint64_t *__restrict__ seg_start,
                                                          const uint64_t *__restrict__ seg_end, const uint64_t *__restrict__ seg_off,
                                                          const uint64_t *__restrict__ meta, uint4 *__restrict__ out, uint64_t nvec)
{
    const uint64_t head_len = meta[PM_HEAD_LEN], hv = round16(head_len) / 16, nseg = meta[PM_NSEG];
    for (uint64_t v = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; v < nvec; v += (uint64_t)gridDim.x * blockDim.x)
    {
        uint64_t src, valid;
        if (v < hv)
        {
            src = g.own_begin + v * 16;
            valid = head_len - v * 16;
        }
        else
        {
            const uint64_t o = (v - hv) * 16;
            uint64_t lo = 0, hi = nseg - 1; // the last segment whose offset is <= o
            while (lo < hi)
            {
                const uint64_t mid = (lo + hi + 1) >> 1;
                if (seg_off[mid] <= o) lo = mid;
                else hi = mid - 1;
            }
            const uint64_t in = o - seg_off[lo];
            src = seg_start[lo] + in;
            valid = seg_end[lo] - seg_start[lo] - in;
        }
        if (valid > 16) valid = 16;
        // 16 unaligned source bytes from two aligned vectors: byte k of the output is byte sh + k of w[]
        const uint64_t a = src & ~15ull;
        const uint32_t sh = (uint32_t)(src & 15);
        const uint4 v0 = load_vec(g.text, g.avail, a);
        const uint4 v1 = sh + valid > 16 ? load_vec(g.text, g.avail, a + 16) : make_uint4(0, 0, 0, 0);
        const uint32_t w[8] = {v0.x, v0.y, v0.z, v0.w, v1.x, v1.y, v1.z, v1.w};
        const uint32_t ws = sh >> 2, bs = (sh & 3) * 8;
        uint32_t o[4];
#pragma unroll
        for (uint32_t k = 0; k < 4; k++)
        {
            o[k] = __funnelshift_r(pick(w, k + ws), pick(w, k + ws + 1), bs);
            const int keep = (int)valid - 4 * (int)k; // bytes of this word that belong to the line
            if (keep <= 0) o[k] = 0;
            else if (keep < 4) o[k] &= (1u << (8 * keep)) - 1u;
        }
        out[v] = make_uint4(o[0], o[1], o[2], o[3]);
    }
}

// 5. Header and segment table.
__global__ void k_row_fill(const PackGeo g, const RegexRowHeader h, const uint64_t *__restrict__ seg_start,
                           const uint64_t *__restrict__ seg_end, uint8_t *__restrict__ row)
{
    const uint64_t i0 = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    RegexRowSeg *tab = reinterpret_cast<RegexRowSeg *>(row + sizeof(RegexRowHeader) + h.nkeys * 8);
    if (i0 == 0)
    {
        *reinterpret_cast<RegexRowHeader *>(row) = h;
        if (h.nkeys & 1) *reinterpret_cast<uint64_t *>(tab + h.nseg) = 0; // the table's pad to 16 bytes: rows are deterministic
    }
    // a segment that reaches avail_len without its '\n' goes on in the next shard, unless this one ends the text
    const bool open_end = g.next_byte >= 0 && g.avail && g.text[g.avail - 1] != '\n';
    for (uint64_t s = i0; s < h.nseg; s += (uint64_t)gridDim.x * blockDim.x)
    {
        const uint64_t b = seg_start[s], e = seg_end[s];
        tab[s].start = g.G + b;
        tab[s].len_cont = ((e - b) << 1) | ((open_end && e == g.avail) ? 1u : 0u);
    }
}

struct IsLine // filter / count mode: every key is a line; match mode: keys with low bit 0
{
    int match;
    __host__ __device__ bool operator()(const uint64_t &k) const { return !match || !(k & 1); }
};

} // namespace

#define CKP(call)                                                                                                       \
    do                                                                                                                  \
    {                                                                                                                   \
        cudaError_t e_ = (call);                                                                                        \
        if (e_ != cudaSuccess)                                                                                          \
        {                                                                                                               \
            set_error(-2, "CUDA error %s in the regex row pack (%s:%d)", cudaGetErrorName(e_), __FILE__, __LINE__);     \
            return -2;                                                                                                  \
        }                                                                                                               \
    } while (0)

static int pack_reserve(RegexPackBufs &B, uint64_t n)
{
    if (n <= B.cap && B.meta) return 0;
    const uint64_t c = std::max<uint64_t>(n + n / 4, 4096);
    cudaFree(B.sel); cudaFree(B.le); cudaFree(B.flag); cudaFree(B.segid);
    cudaFree(B.seg_start); cudaFree(B.seg_end); cudaFree(B.plen); cudaFree(B.seg_off);
    B.sel = B.le = B.seg_start = B.seg_end = B.plen = B.seg_off = nullptr;
    B.flag = B.segid = nullptr;
    B.cap = 0;
    CKP(cudaMalloc(&B.sel, c * 8));
    CKP(cudaMalloc(&B.le, c * 8));
    CKP(cudaMalloc(&B.flag, c * 4));
    CKP(cudaMalloc(&B.segid, c * 4));
    CKP(cudaMalloc(&B.seg_start, c * 8));
    CKP(cudaMalloc(&B.seg_end, c * 8));
    CKP(cudaMalloc(&B.plen, c * 8));
    CKP(cudaMalloc(&B.seg_off, c * 8));
    if (!B.meta) CKP(cudaMalloc(&B.meta, PM_WORDS * 8));
    if (!B.h_meta) CKP(cudaMallocHost(&B.h_meta, PM_WORDS * 8));
    if (!B.ev0) CKP(cudaEventCreate(&B.ev0));
    if (!B.ev1) CKP(cudaEventCreate(&B.ev1));
    B.cap = c;
    return 0;
}

static int pack_tmp(RegexPackBufs &B, size_t need, cudaStream_t st)
{
    if (need <= B.tmp_bytes) return 0;
    CKP(cudaStreamSynchronize(st));
    cudaFree(B.tmp);
    B.tmp = nullptr;
    B.tmp_bytes = 0;
    CKP(cudaMalloc(&B.tmp, need));
    B.tmp_bytes = need;
    return 0;
}

int regex_pack_row(DevCtx &E, const krep_b200_shard_t *sh, int mode, const uint64_t *d_keys, uint64_t nkeys, uint64_t device_lines,
                   const void **d_row, uint64_t *row_bytes, float *pack_ms)
{
    if (!E.rx_pack) E.rx_pack = new RegexPackBufs();
    RegexPackBufs &B = *E.rx_pack;
    cudaStream_t st = E.scan_stream;
    const uint64_t n = nkeys ? nkeys : 1;
    if (pack_reserve(B, n) != 0) return -2;
    PackGeo g;
    g.text = (const uint8_t *)sh->d_text;
    g.avail = sh->avail_len;
    g.own_begin = sh->own_begin;
    g.own_end = sh->own_end < sh->avail_len ? sh->own_end : sh->avail_len;
    g.G = sh->global_offset;
    g.prev_byte = sh->prev_byte;
    g.next_byte = sh->next_byte;
    g.shift = regex_key_shift((RegexMode)mode);
    const unsigned grid_n = (unsigned)std::min<uint64_t>((n + PK_THREADS - 1) / PK_THREADS, (uint64_t)E.sm_count * 16);
    CKP(cudaEventRecord(B.ev0, st));
    CKP(cudaMemsetAsync(B.meta, 0, PM_WORDS * 8, st));
    // the lines glibc must see, in key order (NumSelected lands in meta[PM_NSEL])
    const IsLine pred{mode == RX_OFFSETS};
    size_t need = 0, need2 = 0, need3 = 0;
    CKP(cub::DeviceSelect::If(nullptr, need, d_keys, B.sel, B.meta + PM_NSEL, (int64_t)nkeys, pred, st));
    CKP(cub::DeviceScan::ExclusiveSum(nullptr, need2, B.flag, B.segid, (int64_t)n, st));
    CKP(cub::DeviceScan::ExclusiveSum(nullptr, need3, B.plen, B.seg_off, (int64_t)n, st));
    if (pack_tmp(B, std::max(need, std::max(need2, need3)), st) != 0) return -2;
    if (nkeys) CKP(cub::DeviceSelect::If(B.tmp, need, d_keys, B.sel, B.meta + PM_NSEL, (int64_t)nkeys, pred, st));
    // a warp per line, plus the head's warp
    const uint64_t warps = n + 1;
    const unsigned grid_w = (unsigned)std::min<uint64_t>((warps * 32 + PK_THREADS - 1) / PK_THREADS, (uint64_t)E.sm_count * 32);
    k_pack_lines<<<grid_w, PK_THREADS, 0, st>>>(g, B.sel, B.le, B.meta);
    k_seg_marks<<<grid_n, PK_THREADS, 0, st>>>(g, B.sel, B.le, n, B.meta, B.flag);
    need2 = B.tmp_bytes;
    CKP(cub::DeviceScan::ExclusiveSum(B.tmp, need2, B.flag, B.segid, (int64_t)n, st));
    k_seg_bounds<<<grid_n, PK_THREADS, 0, st>>>(g, B.sel, B.le, B.flag, B.segid, B.seg_start, B.seg_end, B.meta);
    k_seg_sizes<<<grid_n, PK_THREADS, 0, st>>>(B.seg_start, B.seg_end, n, B.meta, B.plen);
    need3 = B.tmp_bytes;
    CKP(cub::DeviceScan::ExclusiveSum(B.tmp, need3, B.plen, B.seg_off, (int64_t)n, st));
    k_seg_total<<<1, 1, 0, st>>>(B.plen, B.seg_off, B.meta);
    count_launch(6);
    CKP(cudaGetLastError());
    CKP(cudaMemcpyAsync(B.h_meta, B.meta, PM_WORDS * 8, cudaMemcpyDeviceToHost, st));
    CKP(cudaStreamSynchronize(st));
    const uint64_t nseg = B.h_meta[PM_NSEG], head_len = B.h_meta[PM_HEAD_LEN], seg_bytes = B.h_meta[PM_SEG_BYTES];
    const uint64_t fixed = regex_row_fixed_bytes(nkeys, nseg), data = round16(head_len) + seg_bytes, total = fixed + data;
    trace("regex pack: %llu keys, %llu lines, %llu segments, head %llu, %llu segment bytes", (unsigned long long)nkeys,
          (unsigned long long)B.h_meta[PM_NSEL], (unsigned long long)nseg, (unsigned long long)head_len, (unsigned long long)seg_bytes);
    // the packed lines are disjoint ranges of the shard's readable bytes: anything larger is a fault of the pack
    if (nseg > B.h_meta[PM_NSEL] || seg_bytes > round16(g.avail) + 16 * nseg || head_len > g.own_end - g.own_begin)
    {
        set_error(-2, "regex row pack: inconsistent sizes (%llu lines, %llu segments, %llu bytes)",
                  (unsigned long long)B.h_meta[PM_NSEL], (unsigned long long)nseg, (unsigned long long)seg_bytes);
        return -2;
    }
    if (total > B.row_cap)
    {
        cudaFree(B.row);
        B.row = nullptr;
        B.row_cap = 0;
        const uint64_t c = total + total / 4 + 4096;
        CKP(cudaMalloc(&B.row, c));
        B.row_cap = c;
    }
    RegexRowHeader h;
    memset(&h, 0, sizeof h);
    h.magic = REGEX_ROW_MAGIC;
    h.mode = (uint64_t)mode;
    h.row_bytes = total;
    h.device_lines = device_lines;
    h.nkeys = nkeys;
    h.nseg = nseg;
    h.head_len = head_len;
    h.flags = B.h_meta[PM_FLAGS];
    h.own_begin = g.G + g.own_begin;
    h.own_end = g.G + g.own_end;
    h.avail_end = g.G + g.avail;
    const unsigned grid_s = (unsigned)std::max<uint64_t>(1, std::min<uint64_t>((nseg + PK_THREADS - 1) / PK_THREADS, (uint64_t)E.sm_count * 16));
    k_row_fill<<<grid_s, PK_THREADS, 0, st>>>(g, h, B.seg_start, B.seg_end, B.row);
    if (nkeys) CKP(cudaMemcpyAsync(B.row + sizeof(RegexRowHeader), d_keys, nkeys * 8, cudaMemcpyDeviceToDevice, st));
    const uint64_t nvec = data / 16;
    if (nvec)
    {
        const unsigned grid_c = (unsigned)std::min<uint64_t>((nvec + PK_THREADS - 1) / PK_THREADS, (uint64_t)E.sm_count * 32);
        k_pack_copy<<<grid_c, PK_THREADS, 0, st>>>(g, B.seg_start, B.seg_end, B.seg_off, B.meta, reinterpret_cast<uint4 *>(B.row + fixed),
                                                   nvec);
        count_launch();
    }
    count_launch();
    CKP(cudaGetLastError());
    CKP(cudaEventRecord(B.ev1, st));
    CKP(cudaStreamSynchronize(st));
    if (pack_ms)
    {
        float ms = 0.f;
        cudaEventElapsedTime(&ms, B.ev0, B.ev1);
        *pack_ms = ms;
    }
    *d_row = B.row;
    *row_bytes = total;
    return 0;
}

uint8_t *regex_pack_host_buffer(DevCtx &E, uint64_t bytes)
{
    if (!E.rx_pack) E.rx_pack = new RegexPackBufs();
    RegexPackBufs &B = *E.rx_pack;
    if (bytes > B.h_row_cap)
    {
        cudaFreeHost(B.h_row);
        B.h_row = nullptr;
        B.h_row_cap = 0;
        const uint64_t c = bytes + bytes / 4 + 4096;
        if (cudaMallocHost(&B.h_row, c) != cudaSuccess)
        {
            cudaGetLastError();
            set_error(-2, "cannot allocate pinned memory for a regex row");
            return nullptr;
        }
        B.h_row_cap = c;
    }
    return B.h_row;
}

void regex_pack_free(DevCtx &E)
{
    RegexPackBufs *B = E.rx_pack;
    if (!B) return;
    cudaFree(B->sel); cudaFree(B->le); cudaFree(B->flag); cudaFree(B->segid);
    cudaFree(B->seg_start); cudaFree(B->seg_end); cudaFree(B->plen); cudaFree(B->seg_off);
    cudaFree(B->meta); cudaFreeHost(B->h_meta); cudaFree(B->tmp); cudaFree(B->row); cudaFreeHost(B->h_row);
    if (B->ev0) cudaEventDestroy(B->ev0);
    if (B->ev1) cudaEventDestroy(B->ev1);
    delete B;
    E.rx_pack = nullptr;
}

} // namespace kb
