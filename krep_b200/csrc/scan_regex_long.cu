// scan_regex_long.cu — -E lines longer than the reach of k_regex_lines, decided on the device (DESIGN §12.8).
//
// k_regex_lines walks a line at most REGEX_HALO bytes past its thread's segment; a line whose '\n' lies further away
// leaves as an uncertain key.  This pass runs after it, on the same stream, the same bytes and in the same mode, and
// takes the uncertain keys of lines that went out of reach but whose '\n' lies within avail_len (not the text's last
// line, shorter than REGEX_LONG_MAX_LINE).  For each it does what k_regex_lines would have done with unbounded reach:
//
//   pick    one warp per key this scan appended: is there a '\n' in [p, limit)?  If not, the line goes to the work list;
//   ends    one CTA per picked line: its '\n' from limit on; the line is cut into slices of S bytes (slice numbers
//           handed out by one atomic per line, owner[] maps a slice back to its line);
//   slices  one thread per slice walks it from a guess (slice 0: the start rows; slice k: the start rows walked over the
//           C bytes before the slice) and records its rows at every C bytes (checkpoint 0 = entry, last = exit);
//   chain   one thread per line goes through its slices in order with the true rows: where they equal a slice's
//           recorded entry, or the recorded rows at a checkpoint the thread reaches by re-walking, the record is the
//           truth from there on.  A MATCHED or DEAD state is absorbing, so the rows recorded after convergence carry
//           the verdict; a live line at its end takes the '\n' column.  No give-up rule: the worst case is one
//           sequential walk of the line;
//   compact the keys the verdicts remove are overwritten with ~0 by the chain, and the list is closed up behind them;
//   match   (match mode) one warp per line decided MATCHED enumerates its matches as k_regex_lines does, 32 starts at
//           a time, within the same step budget; a line over budget or with a match of REGEX_LONG_MAX_MATCH bytes or
//           more keeps its uncertain key.
//
// Batches (krep_b200_regex_search_batch): pick, ends and chain take BATCH instantiations that find a picked line's
// text, leave its own text's last line alone and count on its text's counter, as k_regex_lines<MODE, true, G> does.
//
// Slices are processed in rounds of at most round_slices so that the records stay within REC_BYTES.  Every kernel
// returns at once when there is nothing to do, so a scan without long lines pays a few empty launches.
#include <atomic>
#include <cstdlib>
#include "common.h"
#include "engine.h"
#include "scan_regex.cuh"

#define CKL(call)                                                                                  \
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

namespace kb {

namespace {

constexpr int LL_THREADS = 256;
constexpr int LL_SET_THREADS = 512; // split plans: one CTA per SM (an image of up to REGEX_SET_SMEM_BYTES)
constexpr uint64_t REC_BYTES = 64ull << 20; // slice records of one round
constexpr uint64_t REMOVED = ~0ull;         // a list entry whose key the pass removed
constexpr int WALK_CHUNK = 8;               // k_long_match: steps between two checks for a lane that finished with a match

enum : uint32_t
{
    PK_PENDING = 0, // slices to chain
    PK_SKIP = 1,    // not taken (no '\n' within avail_len, the text's last line, too long): the key stays
    PK_KEEP = 2,    // decided, the key stays (filter mode: MATCHED)
    PK_REMOVED = 3, // decided, the key was overwritten with REMOVED
};

struct LongPick
{
    uint64_t p, nl, key_idx, base; // line start and '\n' (local offsets), index of its key in the list, first slice
    uint32_t nslices, state;
    uint16_t rows[REGEX_MAX_GROUPS]; // chain: the true rows at the start of the next slice to chain
};

struct LongCtl
{
    unsigned long long snap, end; // the list's length before k_regex_lines, and after it
    unsigned long long npicks, nslices, nremoved, nmatch;
};

struct LongArgs
{
    LongCtl *ctl;
    LongPick *picks;
    uint64_t pick_cap;
    uint32_t *owner; // slice -> its line's pick index
    uint64_t owner_cap;
    uint16_t *rec; // round_slices records of nck * G rows
    uint64_t round_slices;
    uint64_t *tmp;   // compaction: the keys moved into holes
    uint32_t *mlist; // match mode: picks decided MATCHED
    uint32_t slice, ckpt, nck, mode;
};

} // namespace

struct LongBufs
{
    LongCtl *ctl = nullptr;
    LongPick *picks = nullptr;
    uint64_t pick_cap = 0;
    uint32_t *owner = nullptr;
    uint64_t owner_cap = 0;
    uint16_t *rec = nullptr;
    uint64_t rec_words = 0;
    uint64_t *tmp = nullptr;
    uint32_t *mlist = nullptr;
    uint32_t *pick_text = nullptr; // batches: the text of each picked line
};

namespace {

__device__ __forceinline__ uint64_t reach_limit(const RegexLaunch &a, uint64_t p)
{
    const uint64_t sb = a.own_begin + (p - a.own_begin) / REGEX_SEG * REGEX_SEG;
    const uint64_t se = sb + REGEX_SEG < a.own_end ? sb + REGEX_SEG : a.own_end;
    return se + REGEX_HALO < a.avail_len ? se + REGEX_HALO : a.avail_len;
}

// bit k set where byte k of v is '\n'
__device__ __forceinline__ uint32_t newline_mask(uint4 v)
{
    uint32_t m = 0;
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int k = 0; k < 16; k++) m |= (((w[k >> 2] >> ((k & 3) * 8)) & 0xFFu) == '\n' ? 1u : 0u) << k;
    return m;
}

__device__ __forceinline__ uint4 load16(const RegexLaunch &a, uint64_t q)
{
    Window W{a.text, a.avail_len, ~0ull, make_uint4(0, 0, 0, 0)};
    W.load(q);
    return W.v;
}

// copies `words` 16-bit words of the image to shared memory
__device__ __forceinline__ void load_image(const RegexLaunch &a, uint32_t words)
{
    extern __shared__ uint4 s_raw[];
    const uint4 *src = reinterpret_cast<const uint4 *>(a.trans);
    for (uint32_t i = threadIdx.x; i < words / 8; i += blockDim.x) s_raw[i] = src[i];
    __syncthreads();
}

__global__ void k_long_begin(const unsigned long long *counter, LongCtl *ctl)
{
    ctl->snap = counter[0];
    ctl->end = 0;
    ctl->npicks = ctl->nslices = ctl->nremoved = ctl->nmatch = 0;
}

// One warp per key appended by this scan: the line goes to the work list when no '\n' lies in [p, limit) and limit is
// below avail_len.  Nothing is picked when the list overflowed (the scan is redone with a longer list).  BATCH: the
// picked line's text goes to pick_text[idx], found as k_regex_lines finds it (its keys are never lines in a gap).
// pick_text stays outside LongPick so that the single-text kernels keep their layout.
template <bool BATCH>
__global__ void __launch_bounds__(LL_THREADS) k_long_pick(const __grid_constant__ RegexLaunch a, const LongArgs L,
                                                          uint32_t *pick_text)
{
    const uint64_t snap = L.ctl->snap, end = a.counter[0];
    if (blockIdx.x == 0 && threadIdx.x == 0) L.ctl->end = end;
    if (end > a.cap) return;
    const int shift = a.matches ? REGEX_MATCH_SHIFT : LIT_TAG_BITS;
    const uint32_t lane = threadIdx.x & 31;
    const uint64_t nwarps = (uint64_t)gridDim.x * blockDim.x / 32;
    for (uint64_t i = snap + ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) / 32; i < end; i += nwarps)
    {
        const uint64_t k = a.out[i];
        if (a.matches && (k & 1)) continue; // a match key
        const uint64_t p = (k >> shift) - a.global_offset;
        const uint64_t limit = reach_limit(a, p);
        if (limit >= a.avail_len) continue; // the '\n' cannot lie within avail_len
        bool found = false;
        for (uint64_t b = p & ~15ull; b < limit && !found; b += 32 * 16)
        {
            const uint64_t q = b + lane * 16;
            uint32_t m = 0;
            if (q < limit)
            {
                m = newline_mask(load16(a, q));
                if (q < p) m &= ~0u << (p - q);
                if (q + 16 > limit) m &= (1u << (limit - q)) - 1;
            }
            found = __any_sync(0xFFFFFFFFu, m != 0);
        }
        if (found || lane != 0) continue;
        const unsigned long long idx = atomicAdd(&L.ctl->npicks, 1ull);
        if (idx >= L.pick_cap) continue; // cannot happen with the sizing of long_lines_begin: the key stays
        LongPick &P = L.picks[idx];
        P.p = p;
        P.nl = ~0ull;
        P.key_idx = i;
        P.nslices = 0;
        P.state = PK_SKIP;
        if constexpr (BATCH)
        {
            const uint64_t gp = a.global_offset + p;
            uint32_t t = a.seg_text[gp / REGEX_SEG];
            while (t + 1 < a.n_texts && a.text_end[t] <= gp) t++;
            pick_text[idx] = t;
        }
    }
}

// One CTA per picked line: its '\n' at or after limit (below p + REGEX_LONG_MAX_LINE and avail_len), its slices.  The
// line of the text's last byte is not taken: a single text's ('\n' at avail_len - 1, nothing after the shard), or in a
// batch its own text's (the '\n' is the text's final byte or the gap's first: batch rule 2 of k_regex_lines).
template <bool BATCH>
__global__ void __launch_bounds__(LL_THREADS) k_long_ends(const __grid_constant__ RegexLaunch a, const LongArgs L,
                                                          const uint32_t *pick_text)
{
    __shared__ unsigned long long s_nl, s_base;
    __shared__ uint32_t s_ns;
    const uint64_t n = L.ctl->npicks < L.pick_cap ? L.ctl->npicks : L.pick_cap;
    for (uint64_t i = blockIdx.x; i < n; i += gridDim.x)
    {
        LongPick &P = L.picks[i];
        const uint64_t p = P.p, limit = reach_limit(a, p);
        const uint64_t stop = p + REGEX_LONG_MAX_LINE < a.avail_len ? p + REGEX_LONG_MAX_LINE : a.avail_len;
        if (threadIdx.x == 0) s_nl = ~0ull;
        __syncthreads();
        constexpr int V = 4; // vectors in flight per thread
        for (uint64_t b = limit & ~15ull; b < stop; b += (uint64_t)LL_THREADS * 16 * V)
        {
            uint64_t best = ~0ull;
#pragma unroll
            for (int v = 0; v < V; v++)
            {
                const uint64_t q = b + ((uint64_t)v * LL_THREADS + threadIdx.x) * 16;
                if (q >= stop) continue;
                uint32_t m = newline_mask(load16(a, q));
                if (q < limit) m &= ~0u << (limit - q);
                if (q + 16 > stop) m &= (1u << (stop - q)) - 1;
                if (m && q + __ffs(m) - 1 < best) best = q + __ffs(m) - 1;
            }
            if (best != ~0ull) atomicMin(&s_nl, (unsigned long long)best);
            if (__syncthreads_or(best != ~0ull)) break;
        }
        if (threadIdx.x == 0)
        {
            const uint64_t nl = s_nl;
            uint32_t ns = 0;
            s_base = 0;
            if (nl != ~0ull && !(BATCH ? a.global_offset + nl + 1 >= a.text_end[pick_text[i]]
                                       : nl + 1 == a.avail_len && a.next_byte < 0))
            {
                ns = (uint32_t)((nl - p + L.slice - 1) / L.slice);
                const unsigned long long base = atomicAdd(&L.ctl->nslices, (unsigned long long)ns);
                if (base + ns > L.owner_cap) ns = 0; // cannot happen with the sizing of long_lines_begin
                s_base = base;
            }
            s_ns = ns;
            P.nl = nl;
            P.base = s_base;
            P.nslices = ns;
            P.state = ns ? PK_PENDING : PK_SKIP;
            for (uint32_t g = 0; g < REGEX_MAX_GROUPS; g++) P.rows[g] = (uint16_t)a.grp[g].start;
        }
        __syncthreads();
        for (uint32_t j = threadIdx.x; j < s_ns; j += blockDim.x) L.owner[s_base + j] = (uint32_t)i;
        __syncthreads();
    }
}

template <int G>
__device__ __forceinline__ bool rows_equal(const SetRows<G> &R, const uint16_t *rec)
{
    bool eq = true;
#pragma unroll
    for (int g = 0; g < G; g++) eq &= R.r[g] == rec[g];
    return eq;
}

template <int G>
__device__ __forceinline__ void rows_load(SetRows<G> &R, const uint16_t *rec)
{
#pragma unroll
    for (int g = 0; g < G; g++) R.r[g] = rec[g];
}

// walks [x, end) while the rows are live (2); returns the state
template <int G>
__device__ __forceinline__ uint32_t walk(const RegexLaunch &a, const uint16_t *img, Window &W, SetRows<G> &R, uint64_t x,
                                         uint64_t end)
{
    uint32_t st = R.state(a);
    for (; x < end && st == 2; x++)
    {
        R.step(a, img, W.at(x));
        st = R.state(a);
    }
    return st;
}

// Slices [r0, r1) of this round, one thread each: the speculative walk and its records.
template <int G>
__global__ void __launch_bounds__(G == 1 ? LL_THREADS : LL_SET_THREADS, G == 1 ? 0 : 1)
    k_long_slices(const __grid_constant__ RegexLaunch a, const LongArgs L, uint64_t r0)
{
    extern __shared__ uint4 s_raw[];
    const uint16_t *img = reinterpret_cast<const uint16_t *>(s_raw);
    const uint64_t total = L.ctl->nslices < L.owner_cap ? L.ctl->nslices : L.owner_cap;
    const uint64_t r1 = r0 + L.round_slices < total ? r0 + L.round_slices : total;
    const uint64_t first = r0 + (uint64_t)blockIdx.x * blockDim.x;
    if (first >= r1) return;
    load_image(a, a.line_words);
    Window W{a.text, a.avail_len, ~0ull, make_uint4(0, 0, 0, 0)};
    for (uint64_t s = first + threadIdx.x; s < r1; s += (uint64_t)gridDim.x * blockDim.x)
    {
        const LongPick &P = L.picks[L.owner[s]];
        const uint64_t x0 = P.p + (s - P.base) * L.slice;
        const uint64_t x1 = x0 + L.slice < P.nl ? x0 + L.slice : P.nl;
        SetRows<G> R;
        R.begin(a);
        if (x0 > P.p) walk<G>(a, img, W, R, x0 - L.ckpt > P.p ? x0 - L.ckpt : P.p, x0); // the guess
        uint16_t *rec = L.rec + (s - r0) * L.nck * G;
        uint64_t x = x0;
        for (uint32_t j = 0; j < L.nck; j++)
        {
            const uint64_t to = x0 + (uint64_t)j * L.ckpt < x1 ? x0 + (uint64_t)j * L.ckpt : x1;
            walk<G>(a, img, W, R, x, to);
            x = to;
#pragma unroll
            for (int g = 0; g < G; g++) rec[j * G + g] = (uint16_t)R.r[g];
        }
    }
}

// The verdict of a line: the key goes (count, match), or goes unless MATCHED (filter); count mode counts it (BATCH: on
// its text's counter), match mode queues it for k_long_match.
template <bool BATCH>
__device__ __forceinline__ void decide(const RegexLaunch &a, const LongArgs &L, LongPick &P, uint32_t i, bool matched,
                                       const uint32_t *pick_text)
{
    if (L.mode == 0 && matched)
    {
        P.state = PK_KEEP;
        return;
    }
    a.out[P.key_idx] = REMOVED;
    P.state = PK_REMOVED;
    atomicAdd(&L.ctl->nremoved, 1ull);
    if (!matched) return;
    if (L.mode == 1) atomicAdd(BATCH ? a.text_lines + pick_text[i] : a.line_count, 1ull);
    else if (L.mode == 2) L.mlist[atomicAdd(&L.ctl->nmatch, 1ull)] = i;
}

// One thread per line with slices in this round: chains them in order (see the head of the file).
template <int G, bool BATCH>
__global__ void __launch_bounds__(G == 1 ? LL_THREADS : LL_SET_THREADS, G == 1 ? 0 : 1)
    k_long_chain(const __grid_constant__ RegexLaunch a, const LongArgs L, uint64_t r0, const uint32_t *pick_text)
{
    extern __shared__ uint4 s_raw[];
    const uint16_t *img = reinterpret_cast<const uint16_t *>(s_raw);
    const uint64_t n = L.ctl->npicks < L.pick_cap ? L.ctl->npicks : L.pick_cap;
    if ((uint64_t)blockIdx.x * blockDim.x >= n) return;
    load_image(a, a.line_words);
    const uint64_t r1 = r0 + L.round_slices;
    Window W{a.text, a.avail_len, ~0ull, make_uint4(0, 0, 0, 0)};
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x)
    {
        LongPick &P = L.picks[i];
        if (P.state != PK_PENDING) continue;
        const uint64_t lo = P.base > r0 ? P.base : r0, end = P.base + P.nslices, hi = end < r1 ? end : r1;
        if (lo >= hi) continue;
        SetRows<G> T;
#pragma unroll
        for (int g = 0; g < G; g++) T.r[g] = P.rows[g];
        uint32_t st = T.state(a);
        for (uint64_t s = lo; s < hi && st == 2; s++)
        {
            const uint16_t *rec = L.rec + (s - r0) * L.nck * G;
            if (rows_equal<G>(T, rec))
            {
                rows_load<G>(T, rec + (L.nck - 1) * G);
                st = T.state(a);
                continue;
            }
            // re-walk from the true rows until they meet the record at a checkpoint
            const uint64_t x0 = P.p + (s - P.base) * L.slice;
            const uint64_t x1 = x0 + L.slice < P.nl ? x0 + L.slice : P.nl;
            uint64_t x = x0;
            for (uint32_t j = 1; j < L.nck; j++)
            {
                const uint64_t to = x0 + (uint64_t)j * L.ckpt < x1 ? x0 + (uint64_t)j * L.ckpt : x1;
                st = walk<G>(a, img, W, T, x, to);
                x = to;
                if (st != 2) break;
                if (rows_equal<G>(T, rec + j * G))
                {
                    rows_load<G>(T, rec + (L.nck - 1) * G);
                    st = T.state(a);
                    break;
                }
            }
        }
        if (st == 2 && hi < end)
        {
#pragma unroll
            for (int g = 0; g < G; g++) P.rows[g] = (uint16_t)T.r[g];
            continue; // the next round goes on
        }
        if (st == 2)
        {
            T.end_of_line(a, img); // the '\n' column
            st = T.state(a);
        }
        decide<BATCH>(a, L, P, (uint32_t)i, st == 0, pick_text);
    }
}

// One CTA: closes up the list behind the removed keys (the list is unordered; k_finish or the radix sort order it).
__global__ void __launch_bounds__(1024) k_long_compact(const __grid_constant__ RegexLaunch a, const LongArgs L)
{
    __shared__ unsigned long long s_a, s_b;
    const uint64_t removed = L.ctl->nremoved;
    if (removed == 0) return;
    const uint64_t end = L.ctl->end, new_end = end - removed;
    const uint64_t n = L.ctl->npicks < L.pick_cap ? L.ctl->npicks : L.pick_cap;
    if (threadIdx.x == 0) s_a = s_b = 0;
    __syncthreads();
    for (uint64_t i = new_end + threadIdx.x; i < end; i += blockDim.x)
    {
        const uint64_t k = a.out[i];
        if (k != REMOVED) L.tmp[atomicAdd(&s_a, 1ull)] = k;
    }
    __syncthreads();
    for (uint64_t j = threadIdx.x; j < n; j += blockDim.x)
    {
        const LongPick &P = L.picks[j];
        if (P.state == PK_REMOVED && P.key_idx < new_end) a.out[P.key_idx] = L.tmp[atomicAdd(&s_b, 1ull)];
    }
    __syncthreads();
    if (threadIdx.x == 0) a.counter[0] = new_end;
}

// Keys of one warp, appended with one reservation per 32.
struct KeyBuf
{
    uint64_t key = 0;
    uint32_t n = 0;

    __device__ __forceinline__ void flush(const RegexLaunch &a, uint32_t lane)
    {
        if (n == 0) return;
        unsigned long long base = 0;
        if (lane == 0) base = atomicAdd(a.counter, (unsigned long long)n);
        base = __shfl_sync(0xFFFFFFFFu, base, 0) + lane;
        if (lane < n && base < a.cap) a.out[base] = key;
        n = 0;
    }
    __device__ __forceinline__ void push(const RegexLaunch &a, uint32_t lane, uint64_t k)
    {
        if (lane == n) key = k;
        if (++n == 32) flush(a, lane);
    }
};

// Match mode: one warp per line decided MATCHED.  The reference's loop inside the line [p, nl] as in k_regex_lines (from
// cur, the leftmost start s with a match and its longest end e; then cur = e, or s + 1 after an empty match; '^' at p
// only, '$' at nl only), the starts tried 32 at a time: lane l walks start s0 + l, and the steps of the sequential loop
// are the lanes' steps summed in start order, so the enumeration stops at the start where the sequential loop would; a
// start whose own walk goes past the budget is not emitted (the line keeps its key, so glibc decides it either way).
// Work: a round of 32 starts lasts at most its counted steps plus WALK_CHUNK, and every round counts at least one step,
// so one line costs at most (WALK_CHUNK + 1) x (budget + 1) steps of its warp (DESIGN §12.8).
template <int G>
__global__ void __launch_bounds__(G == 1 ? LL_THREADS : LL_SET_THREADS, G == 1 ? 0 : 1)
    k_long_match(const __grid_constant__ RegexLaunch a, const LongArgs L)
{
    extern __shared__ uint4 s_raw[];
    const uint16_t *img = reinterpret_cast<const uint16_t *>(s_raw);
    const uint8_t *bytes = reinterpret_cast<const uint8_t *>(img);
    const uint64_t nm = L.ctl->nmatch;
    const uint64_t w0 = ((uint64_t)blockIdx.x * blockDim.x) / 32;
    if (w0 >= nm) return;
    load_image(a, a.image_words);
    const uint32_t lane = threadIdx.x & 31;
    for (uint64_t w = w0 + threadIdx.x / 32; w < nm; w += (uint64_t)gridDim.x * blockDim.x / 32)
    {
        const LongPick &P = L.picks[L.mlist[w]];
        const uint64_t p = P.p, len = P.nl - P.p;
        const uint64_t budget = (uint64_t)a.ngroups * (REGEX_MATCH_STEPS_PER_BYTE * len + REGEX_MATCH_STEPS_BASE);
        uint64_t steps = 0, cur = 0;
        bool flag = false;
        KeyBuf kb;
        while (cur <= len && steps <= budget)
        {
            bool found = false;
            uint64_t ms = 0, me = 0;
            for (uint64_t s0 = cur;; s0 += 32)
            {
                const uint64_t s = s0 + lane;
                // Lane l walks start s.  A walk may run to the end of a line of up to 2^30 bytes, so the work is bounded
                // twice: a walk stops after `rem` steps (past that the line is over budget whatever it finds), and every
                // WALK_CHUNK steps the lanes above the lowest lane that finished with a match stop (their starts lie
                // inside that match or after it, and the sequential loop never tries them).
                const uint64_t rem = budget - steps + 1;
                uint64_t st = 0, e = 0, x = s;
                bool f = false, over = false, active = s <= len;
                int g = -1;
                const uint16_t *M = img;
                const uint8_t *cls = bytes;
                uint32_t gnl = 0, r = 0;
                while (__any_sync(0xFFFFFFFFu, active))
                {
                    for (int k = 0; k < WALK_CHUNK && active; k++)
                    {
                        if (g >= 0 && x < len && r != 0)
                        {
                            r = M[r + cls[__ldg(a.text + p + x++)]];
                            if (M[r + gnl] & (x == len ? RX_ACC_EOL : RX_ACC)) f = true, e = e > x ? e : x;
                        }
                        else if (++g < (int)a.ngroups && g < G)
                        {
                            // the next automaton of the plan, from start s
                            M = img + a.grp[g].match;
                            cls = bytes + a.grp[g].cls * 2;
                            gnl = a.grp[g].nl_class;
                            r = s == 0 ? a.grp[g].match_bol : a.grp[g].match_mid;
                            x = s;
                            if (M[r + gnl] & (s == len ? RX_ACC_EOL : RX_ACC)) f = true, e = e > s ? e : s;
                        }
                        else
                        {
                            active = false;
                            break;
                        }
                        if (++st > rem) over = true, active = false;
                    }
                    const uint32_t fin = __ballot_sync(0xFFFFFFFFu, !active && f && !over && s <= len);
                    if (fin && lane > (uint32_t)(__ffs(fin) - 1)) active = false;
                }
                // steps before this lane's start: the sequential loop tries it while s <= len and steps <= budget
                uint64_t incl = st;
#pragma unroll
                for (int o = 1; o < 32; o <<= 1)
                {
                    const uint64_t v = __shfl_up_sync(0xFFFFFFFFu, incl, o);
                    if (lane >= (uint32_t)o) incl += v;
                }
                const uint64_t before = steps + incl - st;
                const bool valid = s <= len && before <= budget;
                const uint32_t invalid = __ballot_sync(0xFFFFFFFFu, !valid);
                const uint32_t stop = __ballot_sync(0xFFFFFFFFu, valid && (f || over));
                const uint32_t overs = __ballot_sync(0xFFFFFFFFu, over);
                const int fi = invalid ? __ffs(invalid) - 1 : 32, fs = stop ? __ffs(stop) - 1 : 32;
                if (fs < fi)
                {
                    if ((overs >> fs) & 1)
                    {
                        steps = budget + 1; // this start's walk alone goes past the budget: its match is not emitted
                        break;
                    }
                    found = true;
                    steps = __shfl_sync(0xFFFFFFFFu, before + st, fs);
                    ms = s0 + fs;
                    me = __shfl_sync(0xFFFFFFFFu, e, fs);
                    break;
                }
                if (fi < 32)
                {
                    steps = __shfl_sync(0xFFFFFFFFu, before, fi);
                    break;
                }
                steps = __shfl_sync(0xFFFFFFFFu, before + st, 31);
            }
            if (!found) break;
            if (me - ms >= REGEX_LONG_MAX_MATCH)
            {
                flag = true;
                break;
            }
            kb.push(a, lane, ((a.global_offset + p + ms) << REGEX_MATCH_SHIFT) | ((me - ms) << LIT_TAG_BITS) | 1);
            cur = me == ms ? ms + 1 : me;
        }
        if (steps > budget) flag = true;
        if (flag) kb.push(a, lane, (a.global_offset + p) << REGEX_MATCH_SHIFT); // the whole line goes to regexec
        kb.flush(a, lane);
    }
}

struct Sizes
{
    uint32_t slice, ckpt, nck;
    uint64_t pick_cap, owner_cap, round_slices, rounds;
};

Sizes sizes_of(const RegexLaunch &a, const LongLineOpts &o)
{
    Sizes z;
    z.slice = o.slice_bytes ? o.slice_bytes : REGEX_LONG_SLICE;
    z.ckpt = o.ckpt_bytes ? o.ckpt_bytes : REGEX_LONG_CKPT;
    z.nck = (z.slice + z.ckpt - 1) / z.ckpt + 1;
    const uint64_t own = a.own_end > a.own_begin ? a.own_end - a.own_begin : 0;
    // picked lines are disjoint and each runs more than REGEX_HALO bytes past its start; every line adds at most one
    // partial slice.  Both hold for a chunk of a packed batch as well: its lines, gaps included, are still disjoint and
    // within avail_len, whichever texts they belong to.
    z.pick_cap = own / (REGEX_HALO + 1) + 2;
    z.owner_cap = (a.avail_len + z.slice - 1) / z.slice + z.pick_cap;
    const uint64_t g = a.ngroups > 1 ? (a.ngroups <= 2 ? 2 : a.ngroups <= 4 ? 4 : 8) : 1;
    const uint64_t per_round = REC_BYTES / (z.nck * g * 2);
    z.round_slices = z.owner_cap < per_round ? z.owner_cap : per_round;
    z.rounds = (z.owner_cap + z.round_slices - 1) / z.round_slices;
    return z;
}

int grow(void **p, uint64_t *cap, uint64_t need, size_t elem)
{
    if (need <= *cap) return 0;
    CKL(cudaDeviceSynchronize());
    cudaFree(*p);
    *p = nullptr;
    *cap = 0;
    CKL(cudaMalloc(p, need * elem));
    *cap = need;
    return 0;
}

LongArgs args_of(const LongBufs &B, const Sizes &z, const RegexLaunch &a)
{
    LongArgs L;
    L.ctl = B.ctl;
    L.picks = B.picks;
    L.pick_cap = z.pick_cap;
    L.owner = B.owner;
    L.owner_cap = z.owner_cap;
    L.rec = B.rec;
    L.round_slices = z.round_slices;
    L.tmp = B.tmp;
    L.mlist = B.mlist;
    L.slice = z.slice;
    L.ckpt = z.ckpt;
    L.nck = z.nck;
    // the mode k_regex_lines ran in (launch_regex): a batch counts on text_lines, a single text on line_count
    L.mode = a.line_count || a.text_lines ? 1u : a.matches ? 2u : 0u;
    return L;
}

// grid of a kernel: enough CTAs for `work` items of `per_cta`, at most what fits on the device at once
template <typename K>
unsigned grid_for(K kernel, int threads, size_t smem, int sm_count, uint64_t work, uint64_t per_cta)
{
    int per_sm = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, threads, smem) != cudaSuccess || per_sm < 1)
    {
        cudaGetLastError();
        per_sm = 1;
    }
    const uint64_t need = (work + per_cta - 1) / per_cta, resident = (uint64_t)sm_count * per_sm;
    return (unsigned)(need == 0 ? 1 : need < resident ? need : resident);
}

// Above the default 48 KiB a kernel must opt in, once per device (the attribute belongs to the current device); `done`
// is the calling instantiation's flags.
template <typename K>
int opt_in(K kernel, size_t smem, std::atomic<bool> *done)
{
    if (smem <= 48 * 1024) return 0;
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= MAX_DEV)
    {
        set_error(-2, "long-line pass: no current CUDA device (%s)", cudaGetErrorString(cudaGetLastError()));
        return -2;
    }
    if (done[dev].load()) return 0;
    if (cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)REGEX_SET_SMEM_BYTES) != cudaSuccess)
    {
        set_error(-2, "long-line pass: the device refused %u bytes of dynamic shared memory (%s)", REGEX_SET_SMEM_BYTES,
                  cudaGetErrorString(cudaGetLastError()));
        return -2;
    }
    done[dev].store(true);
    return 0;
}

template <int G, bool BATCH>
int launch_walks(const RegexLaunch &a, const LongArgs &L, const Sizes &z, int sm_count, cudaStream_t s, const uint32_t *pick_text)
{
    const int threads = G == 1 ? LL_THREADS : LL_SET_THREADS;
    const size_t line_smem = (size_t)a.line_words * 2;
    static std::atomic<bool> done_slices[MAX_DEV], done_chain[MAX_DEV];
    if (opt_in(k_long_slices<G>, line_smem, done_slices) || opt_in(k_long_chain<G, BATCH>, line_smem, done_chain)) return -2;
    const unsigned gs = grid_for(k_long_slices<G>, threads, line_smem, sm_count, z.round_slices, threads);
    const unsigned gc = grid_for(k_long_chain<G, BATCH>, threads, line_smem, sm_count, z.pick_cap, threads);
    for (uint64_t r = 0; r < z.rounds; r++)
    {
        k_long_slices<G><<<gs, threads, line_smem, s>>>(a, L, r * z.round_slices);
        k_long_chain<G, BATCH><<<gc, threads, line_smem, s>>>(a, L, r * z.round_slices, pick_text);
        count_launch(2);
    }
    return 0;
}

template <bool BATCH>
int launch_walks_g(const RegexLaunch &a, const LongArgs &L, const Sizes &z, int sm_count, cudaStream_t s, const uint32_t *pick_text)
{
    const uint32_t G = a.ngroups <= 1 ? 1 : a.ngroups <= 2 ? 2 : a.ngroups <= 4 ? 4 : 8;
    return G == 1 ? launch_walks<1, BATCH>(a, L, z, sm_count, s, pick_text)
           : G == 2 ? launch_walks<2, BATCH>(a, L, z, sm_count, s, pick_text)
           : G == 4 ? launch_walks<4, BATCH>(a, L, z, sm_count, s, pick_text)
                    : launch_walks<8, BATCH>(a, L, z, sm_count, s, pick_text);
}

// the work list of one scan: picks and their ends (BATCH: with each line's text)
template <bool BATCH>
void launch_picks(const RegexLaunch &a, const LongArgs &L, const Sizes &z, int sm_count, cudaStream_t s, uint32_t *pick_text)
{
    k_long_pick<BATCH><<<grid_for(k_long_pick<BATCH>, LL_THREADS, 0, sm_count, 1ull << 20, LL_THREADS / 32), LL_THREADS, 0, s>>>(
        a, L, pick_text);
    k_long_ends<BATCH><<<grid_for(k_long_ends<BATCH>, LL_THREADS, 0, sm_count, z.pick_cap, 1), LL_THREADS, 0, s>>>(a, L, pick_text);
    count_launch(2);
}

template <int G>
int launch_match(const RegexLaunch &a, const LongArgs &L, const Sizes &z, int sm_count, cudaStream_t s)
{
    const int threads = G == 1 ? LL_THREADS : LL_SET_THREADS;
    const size_t smem = (size_t)a.image_words * 2;
    static std::atomic<bool> done[MAX_DEV];
    if (opt_in(k_long_match<G>, smem, done)) return -2;
    const unsigned gm = grid_for(k_long_match<G>, threads, smem, sm_count, z.pick_cap, threads / 32);
    k_long_match<G><<<gm, threads, smem, s>>>(a, L);
    count_launch();
    return 0;
}

} // namespace

const LongLineOpts *long_lines_default()
{
    static const LongLineOpts prod;
    return getenv("KREP_B200_NO_LONG_LINES") ? nullptr : &prod;
}

int long_lines_opts(const char *who, uint32_t slice_bytes, uint32_t ckpt_bytes, LongLineOpts *o)
{
    o->slice_bytes = slice_bytes ? slice_bytes : REGEX_LONG_SLICE;
    o->ckpt_bytes = ckpt_bytes ? ckpt_bytes : REGEX_LONG_CKPT;
    if (o->slice_bytes > (1u << 20) || o->ckpt_bytes > o->slice_bytes || (o->slice_bytes + o->ckpt_bytes - 1) / o->ckpt_bytes > 1024)
    {
        clear_error();
        set_error(-3, "%s: slices of 1 .. 2^20 bytes with checkpoints every 1 .. slice bytes, at most 1024 per slice (got %u / %u)",
                  who, slice_bytes, ckpt_bytes);
        return -3;
    }
    return 0;
}

int long_lines_begin(DevCtx &E, const RegexLaunch &a, const LongLineOpts &o, cudaStream_t s)
{
    if (!E.rx_long) E.rx_long = new LongBufs();
    LongBufs &B = *E.rx_long;
    const Sizes z = sizes_of(a, o);
    if (!B.ctl) CKL(cudaMalloc(&B.ctl, sizeof(LongCtl)));
    if (z.pick_cap > B.pick_cap)
    {
        // the work list, the compaction's keys, the match list and the lines' texts have one entry per picked line
        CKL(cudaDeviceSynchronize());
        cudaFree(B.picks);
        cudaFree(B.tmp);
        cudaFree(B.mlist);
        cudaFree(B.pick_text);
        B.picks = nullptr;
        B.tmp = nullptr;
        B.mlist = nullptr;
        B.pick_text = nullptr;
        B.pick_cap = 0;
        CKL(cudaMalloc(&B.picks, z.pick_cap * sizeof(LongPick)));
        CKL(cudaMalloc(&B.tmp, z.pick_cap * sizeof(uint64_t)));
        CKL(cudaMalloc(&B.mlist, z.pick_cap * sizeof(uint32_t)));
        CKL(cudaMalloc(&B.pick_text, z.pick_cap * sizeof(uint32_t)));
        B.pick_cap = z.pick_cap;
    }
    if (grow((void **)&B.owner, &B.owner_cap, z.owner_cap, sizeof(uint32_t))) return -2;
    const uint64_t g = a.ngroups > 1 ? (a.ngroups <= 2 ? 2 : a.ngroups <= 4 ? 4 : 8) : 1;
    if (grow((void **)&B.rec, &B.rec_words, z.round_slices * z.nck * g, sizeof(uint16_t))) return -2;
    k_long_begin<<<1, 1, 0, s>>>(a.counter, B.ctl);
    CKL(cudaGetLastError());
    count_launch();
    return 0;
}

int launch_long_lines(DevCtx &E, const RegexLaunch &a, const LongLineOpts &o, cudaStream_t s)
{
    const LongBufs &B = *E.rx_long;
    const Sizes z = sizes_of(a, o);
    const LongArgs L = args_of(B, z, a);
    // a batch (DESIGN §12.5): each picked line's text decides its last-line rule and takes its count
    const bool batch = a.text_end != nullptr;
    if (batch) launch_picks<true>(a, L, z, E.sm_count, s, B.pick_text);
    else launch_picks<false>(a, L, z, E.sm_count, s, nullptr);
    int rc = batch ? launch_walks_g<true>(a, L, z, E.sm_count, s, B.pick_text)
                   : launch_walks_g<false>(a, L, z, E.sm_count, s, nullptr);
    if (rc != 0) return rc;
    const uint32_t G = a.ngroups <= 1 ? 1 : a.ngroups <= 2 ? 2 : a.ngroups <= 4 ? 4 : 8;
    k_long_compact<<<1, 1024, 0, s>>>(a, L);
    count_launch();
    if (L.mode == 2)
    {
        rc = G == 1 ? launch_match<1>(a, L, z, E.sm_count, s)
             : G == 2 ? launch_match<2>(a, L, z, E.sm_count, s)
             : G == 4 ? launch_match<4>(a, L, z, E.sm_count, s)
                      : launch_match<8>(a, L, z, E.sm_count, s);
        if (rc != 0) return rc;
    }
    CKL(cudaGetLastError());
    trace("long lines%s: mode %u, slices of %u bytes, checkpoints every %u, %llu round(s)", batch ? " (batch)" : "", L.mode,
          z.slice, z.ckpt, (unsigned long long)z.rounds);
    return 0;
}

void long_lines_free(DevCtx &E)
{
    LongBufs *B = E.rx_long;
    if (!B) return;
    cudaFree(B->ctl);
    cudaFree(B->picks);
    cudaFree(B->owner);
    cudaFree(B->rec);
    cudaFree(B->tmp);
    cudaFree(B->mlist);
    cudaFree(B->pick_text);
    delete B;
    E.rx_long = nullptr;
}

} // namespace kb
