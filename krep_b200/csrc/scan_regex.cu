// scan_regex.cu — the line filter of -E searches on sm_90a.
//
// One question per line: can the regex match somewhere in it?  The line automaton (regex_dfa.cpp) answers it; the
// flagged lines go back as keys (global line start << LIT_TAG_BITS) through the engine's occurrence list, and glibc's
// regexec confirms them on the host (replay_regex, semantics.cpp).  Nothing here computes a match offset.
//
//   * the transition table (row-offset entries, <= 32 KiB) and the 256-byte class map live in shared memory;
//   * a thread owns a segment of RX_SEG bytes of the shard's owned range, and in it every line whose first byte lies
//     in the segment (a segment starts a line only when the byte before it is '\n' — at a shard edge that byte is the
//     shard's prev_byte, and there is none at the start of the text);
//   * the owner runs the automaton from the line's first byte, across its segment's end if needed, up to the line's
//     newline.  Once the line is MATCHED (flagged) or DEAD (cannot match any more) it skips to the newline 16 bytes
//     at a time;
//   * a line that runs more than REGEX_HALO bytes past its segment, or past the shard's readable bytes, is flagged
//     unverified: always safe, glibc then looks at it on the host;
//   * the text is read as aligned 16-byte vectors held in registers (one LDG.128 per 16 bytes of a thread's walk);
//   * in count mode (fused -E -c) the same walk counts the lines it decides MATCHED (one atomic per warp) and emits
//     keys for the uncertain lines only;
//   * in match mode (offsets on the device) the same walk decides the lines, and each line decided MATCHED is walked
//     again with the anchored match automaton to emit one key per match, in the reference's order (DESIGN §12.2);
//   * in batch mode (krep_b200_regex_search_batch) the text is many texts packed with '\n' gaps, and each line belongs
//     to its own text: gap lines are skipped, each text's last line is uncertain, -c counts per text (DESIGN §12.5);
//   * a split plan (DESIGN §12.7) runs the instantiations G = 2, 4, 8: the same walk over G automata at once, each byte
//     read once and fed to all of them; the line is MATCHED when one of them is, DEAD when all are.
//
// Work per byte: one class lookup and one transition lookup in shared memory per automaton.
#include <atomic>
#include <cooperative_groups.h>
#include "common.h"
#include "engine.h"
#include "scan_regex.cuh"

namespace cg = cooperative_groups;

namespace kb {

namespace {

constexpr int RX_THREADS = 256;
// split plans: an image of up to REGEX_SET_SMEM_BYTES leaves one CTA per SM, so the CTA is large; 512 threads keep
// the 8-automaton instantiations within 128 registers without spills (ptxas, DESIGN §12.7)
constexpr int RX_SET_THREADS = 512;
constexpr uint32_t RX_SEG = REGEX_SEG; // bytes of owned range per thread

// Position of the first '\n' in [q, end), or end.
__device__ __forceinline__ uint64_t next_newline(Window &W, uint64_t q, uint64_t end)
{
    while (q < end)
    {
        if ((q & 15) == 0 && q + 16 <= end)
        {
            if (W.base != q) W.load(q);
            if (!has_newline(W.v))
            {
                q += 16;
                continue;
            }
        }
        if (W.at(q) == '\n') return q;
        q++;
    }
    return end;
}

// Match mode: reserve one slot of the occurrence list per calling thread, one atomic per coalesced group, and store the
// key there.
__device__ __forceinline__ void emit_key(const RegexLaunch &a, uint64_t key)
{
    cg::coalesced_group g = cg::coalesced_threads();
    unsigned long long base = 0;
    if (g.thread_rank() == 0) base = atomicAdd(a.counter, (unsigned long long)g.size());
    base = g.shfl(base, 0) + g.thread_rank();
    if (base < a.cap) a.out[base] = key;
}

// Batch count mode: adds the thread's lines of text t to that text's counter.
template <int MODE>
__device__ __forceinline__ void add_text_lines(const RegexLaunch &a, uint32_t t, uint32_t &counted)
{
    if constexpr (MODE == RX_COUNT)
        if (counted)
        {
            atomicAdd(a.text_lines + t, (unsigned long long)counted);
            counted = 0;
        }
}

// RX_FILTER: the filter (one key per flagged line).  RX_COUNT: the fused -c of plans whose per-line answer is exact
// (RegexDfa::count_exact).  A line the walk decides (MATCHED or DEAD, or its '\n' read through the '\n' column) is
// settled on the device, and a MATCHED one is counted; only the uncertain lines leave as keys: a line whose '\n' lies
// beyond the walk's limit, and the line that holds the text's last byte (decided or not, so that both end-of-text
// quirks of the reference stay with glibc: DESIGN §12.1).  RX_OFFSETS (RegexDfa::offsets_exact): the same uncertain
// lines leave keys (REGEX_MATCH_SHIFT layout); a line decided MATCHED is enumerated with the anchored match automaton
// (DESIGN §12.2) within a step budget, and a line over its budget leaves an uncertain key as well.
// BATCH (krep_b200_regex_search_batch, DESIGN §12.5): the text is many texts packed with '\n' gaps.  Three rules differ:
// a line that starts in a gap belongs to no text (the walk jumps to the next text's first byte, and processes that line
// only if it still lies in the segment); in count and match mode the uncertain line is the one holding its own text's
// last byte (its '\n' is the text's final byte or the gap's first); and count mode adds its lines to one counter per
// text, once when the thread leaves a text and once at the end.
// G == 1: the plan's one automaton.  G = 2, 4, 8: a split plan (DESIGN §12.7), its a.ngroups automata in the
// first slots of G, the spare ones started DEAD; the walk runs on SetRows, and in match mode every automaton is tried at
// each start: the match starts at the first start where one accepts and ends at the longest of their ends, within
// a.ngroups times the step budget of one automaton.  Launch bounds: the split instantiations ask for one CTA per SM,
// which lets ptxas give them up to 128 registers (without it, it holds them near 40 and spills); 0 leaves G == 1 as it was.
template <int MODE, bool BATCH, int G>
__global__ void __launch_bounds__(G == 1 ? RX_THREADS : RX_SET_THREADS, G == 1 ? 0 : 1) k_regex_lines(const __grid_constant__ RegexLaunch a)
{
    extern __shared__ uint4 s_raw[];
    uint16_t *s_tab = reinterpret_cast<uint16_t *>(s_raw);
    const uint32_t tab_words = (a.ntrans + 7) & ~7u; // the class map follows the table, 16-byte aligned
    // match mode: the match table follows the class map (split plans: the match tables follow all line tables)
    const uint32_t nvec = G > 1 ? (MODE == RX_OFFSETS ? a.image_words : a.line_words) / 8
                                : (tab_words * 2 + 256 + (MODE == RX_OFFSETS ? regex_tab_words(a.nmtrans) * 2 : 0u)) / 16;
    const uint4 *src = reinterpret_cast<const uint4 *>(a.trans);
    for (uint32_t i = threadIdx.x; i < nvec; i += blockDim.x) s_raw[i] = src[i];
    __syncthreads();
    const uint8_t *s_cls = reinterpret_cast<const uint8_t *>(s_tab + tab_words);
    const uint16_t *s_mtab = s_tab + tab_words + 128;
    const uint32_t dead = G > 1 ? 1u : a.nclasses, nl = a.nl_class;

    const uint64_t own = a.own_end > a.own_begin ? a.own_end - a.own_begin : 0;
    const uint64_t nseg = (own + RX_SEG - 1) / RX_SEG;
    Window W{a.text, a.avail_len, ~0ull, make_uint4(0, 0, 0, 0)};
    uint32_t counted = 0; // RX_COUNT: lines of this thread decided MATCHED (BATCH: of text t, not yet added)
    // BATCH: the text of the current line start and its global end
    uint32_t t = 0;
    uint64_t t_end = 0;
    for (uint64_t sg = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; sg < nseg; sg += (uint64_t)gridDim.x * blockDim.x)
    {
        const uint64_t sb = a.own_begin + sg * RX_SEG;
        const uint64_t se = sb + RX_SEG < a.own_end ? sb + RX_SEG : a.own_end;
        const uint64_t limit = se + REGEX_HALO < a.avail_len ? se + REGEX_HALO : a.avail_len;
        uint64_t p = sb;
        const int before = sb == 0 ? a.prev_byte : (int)W.at(sb - 1);
        if (before >= 0 && before != '\n')
        {
            p = next_newline(W, sb, se) + 1; // the line in progress belongs to an earlier segment
            if (p > se) continue;
        }
        if constexpr (BATCH)
        {
            const uint32_t t0 = a.seg_text[(a.global_offset + sb) / RX_SEG];
            if (t0 != t) add_text_lines<MODE>(a, t, counted);
            t = t0;
            t_end = 0; // reloaded at the first line
        }
        while (p < se)
        {
            if constexpr (BATCH)
            {
                // the text this line starts in: texts ending at or before it are behind the thread for good
                const uint64_t gp = a.global_offset + p;
                if (gp >= t_end)
                {
                    while (t < a.n_texts && (t_end = a.text_end[t]) <= gp)
                    {
                        add_text_lines<MODE>(a, t, counted);
                        t++;
                    }
                    if (t >= a.n_texts) break; // only the gap after the last text is left
                    const uint64_t t_start = a.text_start[t];
                    if (gp < t_start)
                    {
                        // a line in the gap: on to the text's first byte (the byte before it is a gap '\n')
                        p = t_start - a.global_offset;
                        if (p >= se) break;
                    }
                }
            }
            uint32_t row;
            uint64_t q = p;
            SetRows<G> R;
            if constexpr (G == 1)
            {
                row = a.start;
                while (row > dead && q < limit)
                {
                    const uint32_t b = W.at(q);
                    if (b == '\n') break;
                    row = s_tab[row + s_cls[b]];
                    q++;
                }
            }
            else
            {
                R.begin(a);
                row = R.state(a);
                while (row > dead && q < limit)
                {
                    const uint32_t b = W.at(q);
                    if (b == '\n') break;
                    R.step(a, s_tab, b);
                    row = R.state(a);
                    q++;
                }
            }
            bool flag;
            if constexpr (MODE != RX_FILTER)
            {
                if constexpr (G == 1)
                {
                    if (row > dead && q < limit) row = s_tab[row + nl]; // the walk stopped at the line's '\n'
                }
                else if (row > dead && q < limit)
                {
                    R.end_of_line(a, s_tab);
                    row = R.state(a);
                }
                if (row <= dead) q = next_newline(W, q, limit);
                if constexpr (BATCH) flag = q >= limit || a.global_offset + q + 1 >= t_end; // out of reach, or its text's last byte
                else flag = q >= limit || (q + 1 == a.avail_len && a.next_byte < 0); // '\n' out of reach, or the text's last byte
                if constexpr (MODE == RX_COUNT) counted += (!flag && row == 0) ? 1u : 0u;
            }
            else
            {
                if (row <= dead) flag = row == 0;                                           // MATCHED / DEAD
                else if (q < limit || (q == a.avail_len && a.next_byte < 0)) // end of the line
                {
                    if constexpr (G == 1) flag = s_tab[row + nl] == 0;
                    else
                    {
                        R.end_of_line(a, s_tab);
                        flag = R.state(a) == 0;
                    }
                }
                else flag = true;                                                        // line not seen to its end: unverified
            }
            if constexpr (MODE == RX_OFFSETS && G > 1)
            {
                if (!flag && row == 0)
                {
                    const uint32_t len = (uint32_t)(q - p);
                    const uint32_t budget = a.ngroups * (REGEX_MATCH_STEPS_PER_BYTE * len + REGEX_MATCH_STEPS_BASE);
                    const uint8_t *bytes = reinterpret_cast<const uint8_t *>(s_tab);
                    uint32_t steps = 0, cur = 0;
                    while (cur <= len && steps <= budget)
                    {
                        uint32_t s = cur, e = 0;
                        bool found = false;
                        for (; s <= len && steps <= budget; s++)
                        {
#pragma unroll
                            for (int g = 0; g < G; g++)
                            {
                                if (g >= (int)a.ngroups) break;
                                const uint16_t *M = s_tab + a.grp[g].match;
                                const uint8_t *cls = bytes + a.grp[g].cls * 2;
                                const uint32_t gnl = a.grp[g].nl_class;
                                uint32_t r = s == 0 ? a.grp[g].match_bol : a.grp[g].match_mid;
                                steps++;
                                if (M[r + gnl] & (s == len ? RX_ACC_EOL : RX_ACC)) found = true, e = max(e, s);
                                for (uint32_t x = s; x < len && r != 0;)
                                {
                                    r = M[r + cls[W.at(p + x++)]];
                                    steps++;
                                    if (M[r + gnl] & (x == len ? RX_ACC_EOL : RX_ACC)) found = true, e = max(e, x);
                                }
                            }
                            if (found) break;
                        }
                        if (!found) break;
                        emit_key(a, ((a.global_offset + p + s) << REGEX_MATCH_SHIFT) | ((uint64_t)(e - s) << LIT_TAG_BITS) | 1);
                        cur = e == s ? s + 1 : e;
                    }
                    flag = steps > budget; // over budget: the whole line goes to regexec
                }
            }
            else if constexpr (MODE == RX_OFFSETS)
            {
                if (!flag && row == 0)
                {
                    // the reference's loop inside the line [p, q]: from cur, the leftmost start s with a match and its
                    // longest end e; then cur = e, or s + 1 after an empty match.  '^' holds at p only, '$' at q only.
                    // offsets are relative to p: a decided line is at most RX_SEG + REGEX_HALO bytes long
                    const uint32_t len = (uint32_t)(q - p);
                    const uint32_t budget = REGEX_MATCH_STEPS_PER_BYTE * len + REGEX_MATCH_STEPS_BASE;
                    uint32_t steps = 0, cur = 0;
                    while (cur <= len && steps <= budget)
                    {
                        uint32_t s = cur, e = 0;
                        bool found = false;
                        for (; s <= len && steps <= budget; s++)
                        {
                            uint32_t r = s == 0 ? a.match_bol : a.match_mid;
                            steps++;
                            if (s_mtab[r + nl] & (s == len ? RX_ACC_EOL : RX_ACC)) found = true, e = s;
                            for (uint32_t x = s; x < len && r != 0;)
                            {
                                r = s_mtab[r + s_cls[W.at(p + x++)]];
                                steps++;
                                if (s_mtab[r + nl] & (x == len ? RX_ACC_EOL : RX_ACC)) found = true, e = x;
                            }
                            if (found) break;
                        }
                        if (!found) break;
                        emit_key(a, ((a.global_offset + p + s) << REGEX_MATCH_SHIFT) | ((uint64_t)(e - s) << LIT_TAG_BITS) | 1);
                        cur = e == s ? s + 1 : e;
                    }
                    flag = steps > budget; // over budget: the whole line goes to regexec
                }
            }
            if (flag)
            {
                cg::coalesced_group g = cg::coalesced_threads();
                unsigned long long base = 0;
                if (g.thread_rank() == 0) base = atomicAdd(a.counter, (unsigned long long)g.size());
                base = g.shfl(base, 0) + g.thread_rank();
                if (base < a.cap) a.out[base] = (a.global_offset + p) << (MODE == RX_OFFSETS ? REGEX_MATCH_SHIFT : LIT_TAG_BITS);
            }
            if constexpr (MODE == RX_FILTER)
                if (row <= dead) q = next_newline(W, q, limit);
            if (q >= limit) break; // the next line starts beyond this thread's reach, hence beyond its segment
            p = q + 1;
        }
    }
    if constexpr (BATCH)
        add_text_lines<MODE>(a, t, counted);
    else if constexpr (MODE == RX_COUNT)
    {
        // every thread of the block gets here: one atomic per warp
        const uint32_t w = __reduce_add_sync(0xFFFFFFFFu, counted);
        if ((threadIdx.x & 31) == 0 && w) atomicAdd(a.line_count, (unsigned long long)w);
    }
}

} // namespace

template <int MODE, bool BATCH>
static void launch_regex_t(const RegexLaunch &a, int sm_count, cudaStream_t s)
{
    const size_t smem = (size_t)((a.ntrans + 7) & ~7u) * 2 + 256 + (MODE == RX_OFFSETS ? (size_t)regex_tab_words(a.nmtrans) * 2 : 0);
    int per_sm = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_regex_lines<MODE, BATCH, 1>, RX_THREADS, smem) != cudaSuccess || per_sm < 1)
    {
        cudaGetLastError();
        per_sm = 1;
    }
    const uint64_t own = a.own_end > a.own_begin ? a.own_end - a.own_begin : 0;
    const uint64_t blocks_needed = (own + (uint64_t)RX_SEG * RX_THREADS - 1) / ((uint64_t)RX_SEG * RX_THREADS);
    const uint64_t resident = (uint64_t)sm_count * per_sm;
    const unsigned grid = (unsigned)(blocks_needed == 0 ? 1 : blocks_needed < resident ? blocks_needed : resident);
    trace("regex%s%s: %u CTAs x %d threads (%d per SM), %zu bytes of shared memory", BATCH ? " batch" : "",
          MODE == RX_COUNT ? " count" : MODE == RX_OFFSETS ? " match" : "", grid, RX_THREADS, per_sm, smem);
    k_regex_lines<MODE, BATCH, 1><<<grid, RX_THREADS, smem, s>>>(a);
    count_launch();
}

template <int MODE, bool BATCH, int G>
static int launch_regex_sets_t(const RegexLaunch &a, int sm_count, cudaStream_t s)
{
    const size_t smem = (size_t)(MODE == RX_OFFSETS ? a.image_words : a.line_words) * 2;
    // above the default 48 KiB a kernel must opt in, once per device (the attribute belongs to the current device)
    static std::atomic<bool> opted_in[MAX_DEV];
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= MAX_DEV)
    {
        set_error(-2, "regex scan: no current CUDA device (%s)", cudaGetErrorString(cudaGetLastError()));
        return -2;
    }
    if (!opted_in[dev].load())
    {
        if (cudaFuncSetAttribute(k_regex_lines<MODE, BATCH, G>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 (int)REGEX_SET_SMEM_BYTES) != cudaSuccess)
        {
            set_error(-2, "regex scan of %d automata: device %d refused %u bytes of dynamic shared memory (%s)", G, dev,
                      REGEX_SET_SMEM_BYTES, cudaGetErrorString(cudaGetLastError()));
            return -2;
        }
        opted_in[dev].store(true);
    }
    int per_sm = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_regex_lines<MODE, BATCH, G>, RX_SET_THREADS, smem) != cudaSuccess ||
        per_sm < 1)
    {
        cudaGetLastError();
        per_sm = 1;
    }
    const uint64_t own = a.own_end > a.own_begin ? a.own_end - a.own_begin : 0;
    const uint64_t blocks_needed = (own + (uint64_t)RX_SEG * RX_SET_THREADS - 1) / ((uint64_t)RX_SEG * RX_SET_THREADS);
    const uint64_t resident = (uint64_t)sm_count * per_sm;
    const unsigned grid = (unsigned)(blocks_needed == 0 ? 1 : blocks_needed < resident ? blocks_needed : resident);
    trace("regex sets%s%s: %u automata, %u CTAs x %d threads (%d per SM), %zu bytes of shared memory", BATCH ? " batch" : "",
          MODE == RX_COUNT ? " count" : MODE == RX_OFFSETS ? " match" : "", a.ngroups, grid, RX_SET_THREADS, per_sm, smem);
    k_regex_lines<MODE, BATCH, G><<<grid, RX_SET_THREADS, smem, s>>>(a);
    count_launch();
    return 0;
}

template <int MODE, bool BATCH>
static int launch_regex_sets(const RegexLaunch &a, int sm_count, cudaStream_t s)
{
    if (a.ngroups <= 2) return launch_regex_sets_t<MODE, BATCH, 2>(a, sm_count, s);
    if (a.ngroups <= 4) return launch_regex_sets_t<MODE, BATCH, 4>(a, sm_count, s);
    return launch_regex_sets_t<MODE, BATCH, 8>(a, sm_count, s);
}

int launch_regex(const RegexLaunch &a, int sm_count, cudaStream_t s)
{
    if (a.ngroups > 1)
    {
        if (a.text_end)
        {
            if (a.text_lines) return launch_regex_sets<RX_COUNT, true>(a, sm_count, s);
            if (a.matches) return launch_regex_sets<RX_OFFSETS, true>(a, sm_count, s);
            return launch_regex_sets<RX_FILTER, true>(a, sm_count, s);
        }
        if (a.line_count) return launch_regex_sets<RX_COUNT, false>(a, sm_count, s);
        if (a.matches) return launch_regex_sets<RX_OFFSETS, false>(a, sm_count, s);
        return launch_regex_sets<RX_FILTER, false>(a, sm_count, s);
    }
    if (a.text_end)
    {
        if (a.text_lines) launch_regex_t<RX_COUNT, true>(a, sm_count, s);
        else if (a.matches) launch_regex_t<RX_OFFSETS, true>(a, sm_count, s);
        else launch_regex_t<RX_FILTER, true>(a, sm_count, s);
    }
    else if (a.line_count) launch_regex_t<RX_COUNT, false>(a, sm_count, s);
    else if (a.matches) launch_regex_t<RX_OFFSETS, false>(a, sm_count, s);
    else launch_regex_t<RX_FILTER, false>(a, sm_count, s);
    return 0;
}

} // namespace kb
