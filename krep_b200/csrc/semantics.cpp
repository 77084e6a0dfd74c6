// semantics.cpp — replays each reference kernel's control flow over the sorted occurrence list that the
// device produced.  The device enumerates WHERE the literal(s) occur (the byte-scanning work, ~100 % of
// the reference's run time); which occurrences a given reference kernel counts/reports — its overlap
// policy, what its cursor does after a -w reject, -c line skipping, the -m limit and its per-kernel
// quirks — is a walk over that list, O(occurrences), never over the text.  Line boundaries for -c are
// looked up in the caller's host buffer around occurrences only (memrchr/memchr, as the reference
// does in find_line_start/find_line_end, krep.c:363-408).
#define _GNU_SOURCE
#include <algorithm>
#include <cassert>
#include <cstdlib>
#include <cstring>
#include <cstdio>
#include <omp.h>
#include <regex.h>
#include <vector>
#include "common.h"

namespace kb {

// krep.c:175-241 (growth policy: 16, then doubling; memory stays free()-able)
bool result_push(match_result_t *r, size_t s, size_t e)
{
    if (!r) return false;
    if (r->count >= r->capacity)
    {
        uint64_t nc = r->capacity ? r->capacity * 2 : 16;
        match_position_t *np = r->capacity ? (match_position_t *)realloc(r->positions, nc * sizeof *np)
                                           : (match_position_t *)malloc(nc * sizeof *np);
        if (!np)
        {
            perror("Error reallocating match positions array");
            return false;
        }
        r->positions = np;
        r->capacity = nc;
    }
    r->positions[r->count].start_offset = s;
    r->positions[r->count].end_offset = e;
    r->count++;
    return true;
}

static inline size_t line_start(const char *t, size_t n, size_t pos) // krep.c:363
{
    if (pos > n) pos = n;
    if (pos == 0) return 0;
    const void *nl = memrchr(t, '\n', pos);
    return nl ? (size_t)((const char *)nl - t) + 1 : 0;
}
static inline size_t line_end(const char *t, size_t n, size_t pos) // krep.c:401
{
    if (pos >= n) return n;
    const void *nl = memchr(t + pos, '\n', n - pos);
    return nl ? (size_t)((const char *)nl - t) : n;
}

namespace {
struct Cursor
{
    const uint64_t *k;
    size_t n, i = 0;
    uint64_t base;
    const uint64_t *bounds = nullptr; // device-computed line bounds (global offsets), 2 per key; used when no host text
    bool tail = false; // sub-buffer replay: an occurrence at position 0 has no byte before it (krep.h:314)
    size_t pos(size_t j) const { return (size_t)((k[j] >> LIT_TAG_BITS) - base); }
    bool full(size_t j) const { return (k[j] >> 2) & 1; }
    bool ww(size_t j) const { return (tail && pos(j) == 0) ? (k[j] & 1) : ((k[j] & 3) == 3); }
    void skip_below_base()
    {
        while (i < n && (k[i] >> LIT_TAG_BITS) < base) i++;
    }
    // find_line_start / find_line_end (krep.c:363-408) for the occurrence with key index j at position s, relative to
    // this cursor's (sub-)buffer: from the host text when there is one, else from the device-computed bounds (a line
    // start before the sub-buffer is clipped to it, exactly what memrchr over the sub-buffer returns).
    size_t lstart(size_t j, const char *t, size_t len, size_t s) const
    {
        if (t || !bounds) return line_start(t, len, s);
        return bounds[2 * j] > base ? (size_t)(bounds[2 * j] - base) : 0;
    }
    size_t lend(size_t j, const char *t, size_t len, size_t ls) const
    {
        if (t || !bounds) return line_end(t, len, ls);
        const size_t e = (size_t)(bounds[2 * j + 1] - base);
        return e < len ? e : len;
    }
    // index of the first full occurrence starting at or after `from`, or n
    size_t next_full(size_t from)
    {
        while (i < n && (pos(i) < from || !full(i))) i++;
        return i;
    }
    // index of the first key (full or prefix-only) at or after `from`, or n
    size_t next_any(size_t from)
    {
        while (i < n && pos(i) < from) i++;
        return i;
    }
};
} // namespace

// boyer_moore_search, krep.c:1260-1385
static uint64_t replay_bmh(const search_params_t *P, bool only_matching, size_t m, Cursor c, const char *t, size_t n,
                           match_result_t *res)
{
    if (P->max_count == 0 && (P->count_lines_mode || P->track_positions)) return 0;
    uint64_t cnt = 0;
    size_t last_line = SIZE_MAX, from = 0;
    for (;;)
    {
        const size_t j = c.next_full(from);
        if (j == c.n) break;
        const size_t s = c.pos(j);
        if (P->whole_word && !c.ww(j)) { from = s + 1; continue; }
        bool bumped = false;
        if (P->count_lines_mode)
        {
            const size_t ls = c.lstart(j, t, n, s);
            if (ls != last_line)
            {
                cnt++; last_line = ls; bumped = true;
                if (cnt >= P->max_count) break;
                const size_t le = c.lend(j, t, n, ls);
                const size_t nx = le < n ? le + 1 : n;
                if (nx > s) { from = nx; continue; }
            }
        }
        else
        {
            cnt++; bumped = true;
            if (P->track_positions && res && cnt <= P->max_count) result_push(res, s, s + m);
        }
        if (bumped && cnt >= P->max_count) break;
        from = (only_matching && !P->count_lines_mode) ? s + m : s + 1;
    }
    return cnt;
}

// kmp_search, krep.c:1628-1767
static uint64_t replay_kmp(const search_params_t *P, size_t m, Cursor c, const char *t, size_t n, match_result_t *res)
{
    if (P->max_count == 0) return 0;
    uint64_t cnt = 0;
    size_t last_line = SIZE_MAX, from = 0;
    for (;;)
    {
        const size_t j = c.next_full(from);
        if (j == c.n) break;
        const size_t s = c.pos(j);
        from = s + m;
        if (P->whole_word && !c.ww(j)) continue;
        if (P->count_lines_mode)
        {
            const size_t ls = c.lstart(j, t, n, s);
            if (ls != last_line)
            {
                if (P->max_count != SIZE_MAX && cnt >= P->max_count) break;
                cnt++; last_line = ls;
                const size_t le = c.lend(j, t, n, ls);
                from = le < n ? le + 1 : n;
            }
        }
        else
        {
            if (P->max_count != SIZE_MAX && cnt >= P->max_count)
            {
                if (P->track_positions && res) result_push(res, s, s + m); // krep.c:1719: one past the limit
                break;
            }
            cnt++;
            if (P->track_positions && res) result_push(res, s, s + m);
        }
    }
    return cnt;
}

// memchr_search, krep.c:3891-4041 (incl. the 4096-entry staging buffer and its clipped final flush)
static uint64_t replay_memchr(const search_params_t *P, Cursor c, const char *t, size_t n, match_result_t *res)
{
    if (P->max_count == 0) return 0;
    enum { BUF = 4096 };
    match_position_t *buf = (match_position_t *)malloc(BUF * sizeof *buf);
    size_t nb = 0;
    uint64_t cnt = 0;
    size_t last_line = SIZE_MAX, from = 0;
    const bool tracking = P->track_positions && res;
    while (from < n)
    {
        const size_t j = c.next_full(from);
        if (j == c.n) break;
        const size_t s = c.pos(j);
        if (P->whole_word && !c.ww(j)) { from = s + 1; continue; }
        if (P->count_lines_mode)
        {
            const size_t ls = c.lstart(j, t, n, s);
            if (ls != last_line)
            {
                if (P->max_count != SIZE_MAX && cnt >= P->max_count) break;
                cnt++; last_line = ls;
                const size_t le = c.lend(j, t, n, ls);
                from = le < n ? le + 1 : n;
            }
            else from = s + 1;
        }
        else
        {
            if (P->max_count != SIZE_MAX && cnt >= P->max_count)
            {
                if (tracking)
                {
                    if (nb < BUF) { buf[nb].start_offset = s; buf[nb].end_offset = s + 1; nb++; }
                    else result_push(res, s, s + 1);
                }
                break;
            }
            cnt++;
            if (tracking)
            {
                if (nb >= BUF)
                {
                    for (size_t q = 0; q < nb; q++) result_push(res, buf[q].start_offset, buf[q].end_offset);
                    nb = 0;
                }
                buf[nb].start_offset = s; buf[nb].end_offset = s + 1; nb++;
            }
            from = s + 1;
        }
    }
    if (tracking && nb > 0)
    {
        const uint64_t have = res->count;
        const uint64_t room = (P->max_count == SIZE_MAX) ? nb : (have >= P->max_count ? 0 : P->max_count - have);
        const size_t lim = nb < room ? nb : (size_t)room;
        for (size_t q = 0; q < lim; q++) result_push(res, buf[q].start_offset, buf[q].end_offset);
    }
    free(buf);
    return cnt;
}

// memchr_short_search, krep.c:4371-4503.  With -o the list holds every first-byte hit (full bit set on
// real occurrences) because the reference's cursor jumps pattern_len past ANY first-byte hit.
static uint64_t replay_memchr_short(const search_params_t *P, bool only_matching, size_t m, Cursor c, const char *t,
                                    size_t n, match_result_t *res)
{
    if (P->max_count == 0 && (P->count_lines_mode || P->track_positions)) return 0;
    if (m < 2 || m > 3 || n < m) return 0;
    uint64_t cnt = 0;
    size_t last_line = SIZE_MAX, cur = 0;
    while (n - cur >= m)
    {
        const size_t j = only_matching ? c.next_any(cur) : c.next_full(cur);
        if (j == c.n) break;
        const size_t h = c.pos(j);
        if (h > n - m) break; // memchr range is remaining_len - pattern_len + 1 (krep.c:4401)
        if (c.full(j))
        {
            if (P->whole_word && !c.ww(j)) { cur = h + 1; continue; }
            bool bumped = false;
            if (P->count_lines_mode)
            {
                const size_t ls = c.lstart(j, t, n, h);
                if (ls != last_line)
                {
                    cnt++; last_line = ls; bumped = true;
                    if (cnt >= P->max_count) break;
                    const size_t le = c.lend(j, t, n, ls);
                    const size_t nx = le < n ? le + 1 : n;
                    if (nx > cur) { cur = nx; continue; }
                }
            }
            else
            {
                cnt++; bumped = true;
                if (P->track_positions && res && cnt <= P->max_count) result_push(res, h, h + m);
            }
            if (bumped && cnt >= P->max_count) break;
        }
        const size_t adv = (h - cur) + (only_matching ? m : 1);
        if (adv > n - cur) break;
        cur += adv;
    }
    return cnt;
}

// simd_sse42_search, krep.c:4702-4869 (preconditions already resolved by the caller).  The scan slides a window of
// min(16, remaining) bytes by chunk-m+1 until it holds a full match, so it always reports the first occurrence at or
// after the cursor; the window start itself only shows in -c mode, where the jump to the next line is computed from
// the match offset but added to the window start (krep.c:4791-4795) — it lands `index` bytes before the next line.
static uint64_t replay_sse42(const search_params_t *P, bool only_matching, size_t m, Cursor c, const char *t, size_t n,
                             match_result_t *res)
{
    if (P->max_count == 0 && (P->count_lines_mode || P->track_positions)) return 0;
    uint64_t cnt = 0;
    size_t last_line = SIZE_MAX, cur = 0;
    const size_t step = 17 - m; // window advance on a miss while 16 bytes remain (krep.c:4858); m <= 16
    while (n - cur >= m)
    {
        const size_t j = c.next_full(cur);
        if (j == c.n) break;
        const size_t s = c.pos(j);
        size_t wcur = cur; // start of the window in which s is found
        for (;;)
        {
            const size_t rem = n - wcur, chunk = rem < 16 ? rem : 16;
            if (s - wcur <= chunk - m) break; // always true once fewer than 16 bytes remain (s + m <= n)
            const size_t k1 = (s - wcur - (16 - m) + step - 1) / step; // windows until the occurrence fits
            const size_t k2 = (n - 16 - wcur) / step + 1;              // windows until fewer than 16 bytes remain
            wcur += (k1 < k2 ? k1 : k2) * step;
        }
        if (!P->whole_word || c.ww(j))
        {
            bool bumped = false;
            if (P->count_lines_mode)
            {
                const size_t ls = c.lstart(j, t, n, s);
                if (ls != last_line)
                {
                    if (cnt >= P->max_count) break;
                    cnt++; last_line = ls; bumped = true;
                    const size_t le = c.lend(j, t, n, ls);
                    if (le < n) { cur = wcur + ((le + 1) - s); continue; }
                }
            }
            else
            {
                if (cnt >= P->max_count) break;
                cnt++; bumped = true;
                if (P->track_positions && res && cnt <= P->max_count) result_push(res, s, s + m);
            }
            if (bumped && cnt >= P->max_count) break;
        }
        cur = only_matching ? s + 1 : s + m;
        if (cur > n) cur = n;
    }
    return cnt;
}

// simd_avx2_search for 17..32-byte needles (W = 32, krep.c:4897-5098) and simd_avx512_search for 33..64-byte
// needles (W = 64, krep.c:5128-5285): W-byte windows from a cursor, every occurrence inside a window kept in
// ascending order (overlaps included, whatever -o says); -c re-aims the cursor at the next line; the < W tail is a
// boyer_moore_search on the SUB-buffer (its own -w / -c context, -o advance, re-based -m) whose positions are then
// re-based by index arithmetic on the result vector; AVX-512 skips a window when < (m-1)+64 bytes remain (krep.c:5171).
// neon_search (W = 16, krep.c:4506-4694, any needle length) walks the same way with three differences: the -m limit is
// also tested before counting, the -c jump needs the line to end in a newline, and the tail's positions are re-based
// over the last tail_count entries of the result vector.
static uint64_t replay_window(const search_params_t *P, bool only_matching, size_t m, size_t W, Cursor c, const char *t,
                              size_t n, match_result_t *res)
{
    if (P->max_count == 0 && (P->count_lines_mode || P->track_positions)) return 0;
    const bool neon = W == 16;
    const size_t maxc = P->max_count;
    uint64_t cnt = 0;
    size_t last_line = SIZE_MAX, cur = 0;
    bool exhausted = false;
    while (n - cur >= W)
    {
        size_t j = c.next_full(cur);
        if (j == c.n) { exhausted = true; break; }
        const size_t s0 = c.pos(j);
        if (s0 - cur >= W)
        {
            // empty windows: step as the reference would, but never past the last full window
            const size_t k0 = (s0 - cur) / W, kmax = (n - cur) / W;
            cur += W * (k0 < kmax ? k0 : kmax);
            continue;
        }
        if (W == 64 && n - cur < (m - 1) + 64) { cur += 64; continue; }
        bool line_skipped = false;
        for (; j < c.n && c.pos(j) < cur + W; j++)
        {
            if (!c.full(j)) continue;
            const size_t s = c.pos(j);
            if (P->whole_word && !c.ww(j)) continue;
            bool bumped = false;
            if (P->count_lines_mode)
            {
                const size_t ls = c.lstart(j, t, n, s);
                if (ls != last_line)
                {
                    if (neon && cnt >= maxc) return cnt; // krep.c:4571
                    cnt++; last_line = ls; bumped = true;
                    if (!neon && cnt >= maxc) return cnt;
                    const size_t le = c.lend(j, t, n, ls);
                    const size_t nx = le < n ? le + 1 : n;
                    if (nx > cur && !(neon && le >= n)) // krep.c:4578: NEON only jumps when the line has a newline
                    {
                        cur = nx; // advance is clipped to the remaining length, i.e. cur <= n (nx <= n already)
                        line_skipped = true;
                        break;
                    }
                }
            }
            else
            {
                if (neon && cnt >= maxc) return cnt; // krep.c:4601
                cnt++; bumped = true;
                if (P->track_positions && res && cnt <= maxc) result_push(res, s, s + m);
            }
            if (bumped && cnt >= maxc) return cnt;
        }
        if (line_skipped) continue;
        cur += W;
    }
    const size_t rem = n - cur;
    if (!exhausted && rem >= m)
    {
        search_params_t tail = *P;
        if (maxc != SIZE_MAX) tail.max_count = cnt >= maxc ? 0 : maxc - cnt;
        Cursor tc = c;
        tc.base = c.base + cur;
        tc.tail = true;
        tc.skip_below_base();
        const uint64_t tcnt = replay_bmh(&tail, only_matching, m, tc, t ? t + cur : nullptr, rem, res);
        if (res && P->track_positions && tcnt > 0)
        {
            if (neon)
            {
                if (res->count >= tcnt) // krep.c:4673-4680
                    for (uint64_t k = 0; k < tcnt; k++)
                    {
                        res->positions[res->count - tcnt + k].start_offset += cur;
                        res->positions[res->count - tcnt + k].end_offset += cur;
                    }
            }
            else if (W == 32)
            {
                const uint64_t b0 = cnt > res->count ? res->count : cnt; // krep.c:5077-5079
                for (uint64_t k = b0; k < res->count; k++)
                {
                    res->positions[k].start_offset += cur;
                    res->positions[k].end_offset += cur;
                }
            }
            else
            {
                const uint64_t b0 = res->count >= tcnt ? res->count - tcnt : 0; // krep.c:5275
                for (uint64_t k = 0; k < tcnt && b0 + k < res->count; k++)
                {
                    res->positions[b0 + k].start_offset += cur;
                    res->positions[b0 + k].end_offset += cur;
                }
            }
        }
        cnt += tcnt;
        if (W == 32 && maxc != SIZE_MAX && cnt > maxc) cnt = maxc; // krep.c:5092
    }
    return cnt;
}

// The common case needs no cursor logic at all: when no two occurrences in the list overlap, no -m limit is set and
// lines are not being counted, boyer_moore_search, kmp_search, memchr_search and simd_sse42_search all keep exactly the
// occurrences that pass -w, in order (their cursors only differ in how far they step INSIDE an occurrence).  One pass
// validates that, a second one fills the result vector in bulk (grown by the reference's doubling rule, krep.c:175).
static bool replay_keep_all(int algo, const search_params_t *P, uint32_t m, const Replay &r, match_result_t *res, uint64_t *out)
{
    if (P->count_lines_mode || P->max_count != SIZE_MAX) return false;
    if (algo != KREP_B200_ALGO_BMH && algo != KREP_B200_ALGO_KMP && algo != KREP_B200_ALGO_SSE42 && algo != KREP_B200_ALGO_MEMCHR)
        return false;
    // long lists (the density sweep: 10^7..10^8 occurrences) are validated and copied by several host threads, each on
    // a contiguous slice of the list; short ones stay on the calling thread
    const int nt = r.n >= (1u << 20) ? std::min(8, std::max(1, omp_get_max_threads())) : 1;
    std::vector<uint64_t> kept_of((size_t)nt + 1, 0);
    bool bad = false;
#pragma omp parallel for num_threads(nt) schedule(static, 1) reduction(|| : bad)
    for (int t = 0; t < nt; t++)
    {
        const size_t a = r.n * (size_t)t / (size_t)nt, b = r.n * (size_t)(t + 1) / (size_t)nt;
        uint64_t prev = a ? (r.keys[a - 1] >> LIT_TAG_BITS) : 0, kept = 0;
        for (size_t j = a; j < b; j++)
        {
            const uint64_t k = r.keys[j], s = k >> LIT_TAG_BITS;
            if (!(k & 4) || (j && s < prev + m)) // a prefix-only key, or an overlap: full replay
            {
                bad = true;
                break;
            }
            prev = s;
            kept += !P->whole_word || (k & 3) == 3;
        }
        kept_of[(size_t)t + 1] = kept;
    }
    if (bad) return false;
    for (int t = 0; t < nt; t++) kept_of[(size_t)t + 1] += kept_of[(size_t)t];
    const uint64_t kept = kept_of[(size_t)nt];
    *out = kept;
    if (!(P->track_positions && res) || kept == 0) return true;
    uint64_t cap = res->capacity ? res->capacity : 16;
    while (cap < res->count + kept) cap *= 2;
    if (cap != res->capacity || !res->positions)
    {
        match_position_t *np = (match_position_t *)realloc(res->capacity ? res->positions : nullptr, cap * sizeof *np);
        if (!np) return false; // let the ordinary path report the allocation failure
        res->positions = np;
        res->capacity = cap;
    }
    match_position_t *const o0 = res->positions + res->count;
#pragma omp parallel for num_threads(nt) schedule(static, 1)
    for (int t = 0; t < nt; t++)
    {
        const size_t a = r.n * (size_t)t / (size_t)nt, b = r.n * (size_t)(t + 1) / (size_t)nt;
        match_position_t *o = o0 + kept_of[(size_t)t];
        for (size_t j = a; j < b; j++)
        {
            const uint64_t k = r.keys[j];
            if (P->whole_word && (k & 3) != 3) continue;
            const size_t s = (size_t)((k >> LIT_TAG_BITS) - r.base);
            o->start_offset = s;
            o->end_offset = s + m;
            o++;
        }
    }
    res->count += kept;
    return true;
}

uint64_t replay_literal(int algo, const search_params_t *P, bool only_matching, uint32_t m, const Replay &r,
                        match_result_t *res)
{
    uint64_t quick = 0;
    if (replay_keep_all(algo, P, m, r, res, &quick)) return quick;
    Cursor c{r.keys, r.n, 0, r.base, r.text ? nullptr : r.bounds};
    switch (algo)
    {
    case KREP_B200_ALGO_AVX2: return replay_window(P, only_matching, m, 32, c, r.text, r.text_len, res);   // resolved: 17..32 B
    case KREP_B200_ALGO_AVX512: return replay_window(P, only_matching, m, 64, c, r.text, r.text_len, res); // resolved: 33..64 B
    case KREP_B200_ALGO_NEON: return replay_window(P, only_matching, m, 16, c, r.text, r.text_len, res);
    case KREP_B200_ALGO_KMP: return replay_kmp(P, m, c, r.text, r.text_len, res);
    case KREP_B200_ALGO_MEMCHR: return replay_memchr(P, c, r.text, r.text_len, res);
    case KREP_B200_ALGO_MEMCHR_SHORT: return replay_memchr_short(P, only_matching, m, c, r.text, r.text_len, res);
    case KREP_B200_ALGO_SSE42: return replay_sse42(P, only_matching, m, c, r.text, r.text_len, res);
    default: return replay_bmh(P, only_matching, m, c, r.text, r.text_len, res);
    }
}

// aho_corasick_search, aho_corasick.c:299-466; keys arrive in emission order, -w rejects already dropped
uint64_t replay_ac(const search_params_t *P, const Replay &r, match_result_t *res)
{
    if (P->max_count == 0) return 0;
    const size_t maxc = P->max_count;
    uint64_t found = 0;
    size_t last_line = SIZE_MAX;
    for (size_t j = 0; j < r.n; j++)
    {
        if (found >= maxc) return found;
        const uint64_t key = r.keys[j];
        const size_t e = (size_t)((key >> AC_END_SHIFT) - r.base);
        const size_t len = 1024 - (size_t)((key >> AC_LEN_SHIFT) & 1023);
        const size_t s = e - len;
        if (P->count_lines_mode)
        {
            const size_t ls = (r.text || !r.bounds) ? line_start(r.text, r.text_len, s)
                                                    : (r.bounds[2 * j] > r.base ? (size_t)(r.bounds[2 * j] - r.base) : 0);
            if (ls != last_line)
            {
                found++; last_line = ls;
                if (found >= maxc) return found;
            }
        }
        else
        {
            found++;
            if (P->track_positions && res) result_push(res, s, e);
            if (found >= maxc) return found;
        }
    }
    return found;
}

// ---- regex_search (krep.c:1389-1579) over the lines the device flagged ----------------------------------------------
bool regex_returns_early(const search_params_t *P)
{
    return (P->max_count == 0 && (P->count_lines_mode || P->track_positions)) || !P->compiled_regex;
}

uint64_t regex_empty_text(const search_params_t *P, match_result_t *res)
{
    regmatch_t m;
    if (regexec((const regex_t *)P->compiled_regex, "", 1, &m, 0) != 0) return 0;
    if (!P->count_lines_mode && P->track_positions && res) result_push(res, 0, 0);
    return 1;
}

// Under REG_NEWLINE no match contains a '\n' (regex_dfa.cpp refuses character sets that hold one), so the reference loop
// is unchanged if (1) the cursor skips every line the filter did not flag — glibc finds no match starting there, from
// the line start or from any position inside it — and (2) each regexec call is clipped to the run of consecutive
// flagged lines the cursor is in: [cur, E) with E the byte after the run's last newline, and REG_NOTEOL when E is not
// the end of the text, so that '$' cannot match at a false end of string.  Every match, and every -w / -c / -m
// decision, is glibc's own on the caller's regex_t.  r.keys are the flagged line starts (ascending, global offsets).
//
// Windowed (r.window_len set, resident shards): r.text holds only [origin, origin + window_len), and every run the keys
// form lies inside it.  The replay never reads outside the window (WINDOW_ASSERT in debug builds) because:
//   * REG_NOTEOL depends on the run ending before the TRUE end of the text (n), not before the end of the window;
//   * the byte before a run is the '\n' that ends the previous line (or there is none), so at_line_start and -w's
//     is_word_c(t[start - 1]) read the window for every start above its origin and know the answer at the origin; -w's
//     t[end] lies inside too: a match never contains '\n', so it ends at or before the '\n' that ends its line;
//   * the empty string at n is decided from r.last_byte when the window does not hold the text's last byte.
#ifdef KREP_B200_DEBUG
#define WINDOW_ASSERT(c) assert(c)
#else
#define WINDOW_ASSERT(c) ((void)0)
#endif
uint64_t replay_regex(const search_params_t *P, const Replay &r, match_result_t *res)
{
    if (regex_returns_early(P)) return 0;
    const regex_t *regex = (const regex_t *)P->compiled_regex;
    const char *t = r.text;
    const size_t n = r.text_len;
    if (n == 0) return regex_empty_text(P, res);
    // krep.c:1422 passes compilation flags as execution flags: REG_NEWLINE has the value of REG_STARTEND and REG_ICASE
    // the value of REG_NOTEOL.  Passed on exactly as the reference does.
    const int base_eflags = REG_STARTEND | REG_NEWLINE | (P->case_sensitive ? 0 : REG_ICASE);
    const size_t max_count = P->max_count;
    const size_t RUN_MAX = (size_t)1 << 30; // regoff_t is an int: a run is cut (at a line start) before it gets near 2^31
    const size_t org = r.origin, wend = r.window_len == SIZE_MAX ? n : org + r.window_len; // t[x - org] is byte x
    auto at = [&](size_t x) {
        WINDOW_ASSERT(x >= org && x < wend);
        return (unsigned char)t[x - org];
    };
    auto key_pos = [&](size_t j) { return (size_t)((r.keys[j] >> LIT_TAG_BITS) - r.base); };
    auto after_line = [&](size_t s) {
        if (s >= n) return n;
        WINDOW_ASSERT(s >= org && s <= wend);
        const void *nl = s < wend ? memchr(t + (s - org), '\n', wend - s) : nullptr;
        WINDOW_ASSERT(nl || wend == n); // a window holds whole lines
        return nl ? (size_t)((const char *)nl - t) + org + 1 : n;
    };
    auto first_of_line = [&](size_t s) { // line_start(): a window starts at a line start
        WINDOW_ASSERT(s >= org && s <= wend);
        const void *nl = s > org ? memrchr(t, '\n', s - org) : nullptr;
        return nl ? (size_t)((const char *)nl - t) + org + 1 : org;
    };
    size_t ki = 0, run_end = 0, cur = 0, last_line = SIZE_MAX;
    uint64_t count = 0;
    while (cur < n)
    {
        if (cur >= run_end)
        {
            // the next run: the first flagged line that ends after the cursor, and the flagged lines right behind it
            size_t s = 0, e = 0;
            bool found = false;
            while (ki < r.n && !found)
            {
                s = key_pos(ki++);
                if (s >= n) break;
                e = after_line(s);
                found = e > cur;
            }
            if (!found)
            {
                // no flagged line left.  A text that ends with '\n' still has an empty string after it, where the
                // reference's search from the cursor can end with an empty match (^ or $ at the end of the text) —
                // unless that end belongs to another decider
                if (r.stop < n || (r.last_byte >= 0 ? r.last_byte : at(n - 1)) != '\n') break;
                s = e = n;
            }
            const size_t run_start = s;
            while (ki < r.n && e < n && key_pos(ki) == e && e - run_start < RUN_MAX) e = after_line(key_pos(ki++));
            run_end = e;
            if (cur < run_start) cur = run_start;
        }
        regmatch_t pmatch[1];
        pmatch[0].rm_so = 0;
        pmatch[0].rm_eo = (regoff_t)(run_end - cur);
        const bool at_line_start = cur == org || at(cur - 1) == '\n'; // the byte before a window is a '\n' (or none)
        const int eflags = base_eflags | (at_line_start ? 0 : REG_NOTBOL) | (run_end < n ? REG_NOTEOL : 0);
        WINDOW_ASSERT(cur >= org && run_end <= wend);
        const int rc = regexec(regex, t + (cur - org), 1, pmatch, eflags);
        if (rc != 0)
        {
            if (rc == REG_NOMATCH)
            {
                cur = run_end; // nothing more in this run: on to the next one
                continue;
            }
            char ebuf[256];
            regerror(rc, regex, ebuf, sizeof(ebuf));
            fprintf(stderr, "krep: Regex execution error: %s\n", ebuf);
            return count;
        }
        if (pmatch[0].rm_so == -1 || pmatch[0].rm_eo == -1)
        {
            fprintf(stderr, "krep: Warning: regexec returned success but invalid offsets.\n");
            break;
        }
        const size_t so = (size_t)pmatch[0].rm_so, eo = (size_t)pmatch[0].rm_eo;
        if (eo < so)
        {
            fprintf(stderr, "krep: Warning: regexec returned eo < so.\n");
            cur = std::min(cur + so + 1, n);
            continue;
        }
        const size_t start = cur + so, end = cur + eo;
        if (r.stop < n && start >= run_end && run_end < n)
        {
            // an empty match at the clipped end: '^' after the run's last '\n'.  It lies in the next line, whose matches
            // are not this replay's to report (the reference finds it there, from that line's start)
            cur = run_end;
            continue;
        }
        if (P->whole_word && ((start > org && is_word_c(at(start - 1))) || (end < n && is_word_c(at(end)))))
        {
            cur = std::min(cur + so + 1, n); // krep.c:1487-1501
            continue;
        }
        if (P->count_lines_mode)
        {
            const size_t ls = first_of_line(start);
            if (ls != last_line)
            {
                count++;
                last_line = ls;
                if (count >= max_count) break;
                cur = after_line(ls); // krep.c:1515-1519: on to the next line
                continue;
            }
        }
        else
        {
            count++;
            if (P->track_positions && res) result_push(res, start, end);
        }
        if (count >= max_count) break;
        const size_t next = cur + (so == eo ? so + 1 : eo);
        cur = next > n ? n : next;
    }
    return count;
}

// -E offsets on the device (DESIGN §12.2).  r.keys: ascending match-mode keys — a match key per match of a line the
// device decided, an uncertain-line key per line it left to regexec (sorted before any match key inside that line,
// which the replay skips: the device ran over its step budget there).  Walked in order with the -m limit applied in that
// order: match keys become positions; each stretch of consecutive uncertain lines goes through replay_regex, stopped
// at the next line the device decided (Replay::stop), its positions appended in order.  Exact because no match crosses
// a line and, for plans without word assertions, what regexec finds in a line does not depend on where the cursor
// entered it (at or before the line's start).
uint64_t replay_regex_matches(const search_params_t *P, const Replay &r, match_result_t *res)
{
    const char *t = r.text;
    const size_t n = r.text_len;
    const uint64_t max_count = P->max_count;
    auto after_line = [&](size_t s) {
        const size_t e = line_end(t, n, s);
        return e < n ? e + 1 : n;
    };
    std::vector<uint64_t> lines; // uncertain line starts, shifted as replay_regex reads them
    uint64_t count = 0;
    size_t i = 0;
    while (i < r.n && count < max_count)
    {
        const uint64_t k = r.keys[i];
        const size_t pos = (size_t)((k >> REGEX_MATCH_SHIFT) - r.base);
        if (k & 1)
        {
            const size_t len = (size_t)((k >> LIT_TAG_BITS) & ((1u << (REGEX_MATCH_SHIFT - LIT_TAG_BITS)) - 1));
            count++;
            if (res) result_push(res, pos, pos + len);
            i++;
            continue;
        }
        // a stretch of uncertain lines: up to the next match key outside them
        lines.clear();
        size_t end = 0;
        while (i < r.n)
        {
            const uint64_t u = r.keys[i];
            const size_t s = (size_t)((u >> REGEX_MATCH_SHIFT) - r.base);
            if (u & 1)
            {
                if (s < end) // a match key inside an uncertain line
                {
                    i++;
                    continue;
                }
                break;
            }
            lines.push_back((uint64_t)s << LIT_TAG_BITS);
            end = after_line(s);
            i++;
        }
        search_params_t sub = *P;
        sub.max_count = (size_t)(max_count - count);
        Replay g{lines.data(), lines.size(), t, n, 0};
        g.stop = end < n ? end : SIZE_MAX;
        count += replay_regex(&sub, g, res);
    }
    return count;
}

// Windowed replays (resident shards, DESIGN §12.4).  Running replay_regex window by window gives what one call over the
// whole text gives: a window starts at a line start, and a run cut there behaves as the RUN_MAX cut does — every call
// but the one whose window ends at n has stop set, so an empty match at its clipped end ('^' after its last '\n') is left
// to the next window, where the whole-text replay also finds it (from that line's start, the next run's start).  The
// cursor, the -m budget and (for -c) the last counted line carry over: a line lies in one window only.
uint64_t replay_regex_windows(const search_params_t *P, const uint64_t *keys, size_t nkeys, const RegexWindow *w, size_t nw,
                              size_t n, int last_byte, bool at_end, match_result_t *res)
{
    if (regex_returns_early(P)) return 0;
    const size_t max_count = P->max_count;
    uint64_t count = 0;
    size_t j = 0, covered = 0; // covered: end of the last window replayed
    for (size_t i = 0; i < nw && j < nkeys && count < max_count; i++)
    {
        const size_t wb = w[i].origin, we = wb + w[i].len;
        while (j < nkeys && (size_t)(keys[j] >> LIT_TAG_BITS) < wb) j++; // a key outside every window: not a line glibc sees
        const size_t j0 = j;
        while (j < nkeys && (size_t)(keys[j] >> LIT_TAG_BITS) < we) j++;
        if (j == j0) continue;
        search_params_t sub = *P;
        sub.max_count = max_count - count;
        Replay g{keys + j0, j - j0, w[i].bytes, n, 0};
        g.origin = wb;
        g.window_len = w[i].len;
        g.stop = we < n ? we : SIZE_MAX;
        g.last_byte = last_byte;
        count += replay_regex(&sub, g, res);
        covered = we;
    }
    // The empty string at n: the whole-text replay tries it once its keys run out before n, if the text ends in '\n'
    // and the budget allows.  A last window that ends at n has decided it already; otherwise one call with no keys and
    // an empty window at n does, from the last byte of the text.
    if (at_end && count < max_count && covered < n && n > 0)
    {
        search_params_t sub = *P;
        sub.max_count = max_count - count;
        Replay g{nullptr, 0, "", n, 0};
        g.origin = n;
        g.window_len = 0;
        g.last_byte = last_byte;
        count += replay_regex(&sub, g, res);
    }
    return count;
}

// replay_regex_matches over windows: the same walk; a stretch of uncertain lines goes through replay_regex_windows, whose
// windows (runs of uncertain lines) end where the stretch ends, so the stop rule is the one the whole-text walk applies.
uint64_t replay_regex_matches_windows(const search_params_t *P, const uint64_t *keys, size_t nkeys, const RegexWindow *w,
                                      size_t nw, size_t n, int last_byte, match_result_t *res)
{
    const uint64_t max_count = P->max_count;
    std::vector<uint64_t> lines;
    uint64_t count = 0;
    size_t i = 0, wi = 0;
    while (i < nkeys && count < max_count)
    {
        const uint64_t k = keys[i];
        const size_t pos = (size_t)(k >> REGEX_MATCH_SHIFT);
        if (k & 1)
        {
            const size_t len = (size_t)((k >> LIT_TAG_BITS) & ((1u << (REGEX_MATCH_SHIFT - LIT_TAG_BITS)) - 1));
            count++;
            if (res) result_push(res, pos, pos + len);
            i++;
            continue;
        }
        lines.clear();
        size_t end = 0;
        while (wi < nw && w[wi].origin + w[wi].len <= pos) wi++;
        size_t wj = wi;
        while (i < nkeys)
        {
            const uint64_t u = keys[i];
            const size_t s = (size_t)(u >> REGEX_MATCH_SHIFT);
            if (u & 1)
            {
                if (s < end)
                {
                    i++;
                    continue;
                }
                break;
            }
            lines.push_back((uint64_t)s << LIT_TAG_BITS);
            // the end of the line at s, from the window that holds it
            while (wj < nw && w[wj].origin + w[wj].len <= s) wj++;
            end = n;
            if (wj < nw && w[wj].origin <= s)
            {
                const size_t off = s - w[wj].origin;
                const void *nl = memchr(w[wj].bytes + off, '\n', w[wj].len - off);
                if (nl) end = w[wj].origin + (size_t)((const char *)nl - w[wj].bytes) + 1;
            }
            i++;
        }
        search_params_t sub = *P;
        sub.max_count = (size_t)(max_count - count);
        count += replay_regex_windows(&sub, lines.data(), lines.size(), w + wi, nw - wi, n, last_byte, false, res);
    }
    return count;
}

// The filter's keys are the flagged lines replay_regex confirms; the offsets mode's are match and uncertain-line keys
// (replay_regex_matches, DESIGN §12.2).  The fused -c answers  min(lines the device decided MATCHED + replay_regex over
// the uncertain lines, max_count).  Why this is the reference's count: without -w and -o the loop of krep.c:1389-1579
// calls regexec only at line starts (after a counted line the cursor jumps to the next line start; with no match left
// the loop ends) and never with REG_NOTBOL, and under REG_NEWLINE no match contains a '\n'.  So a line is counted
// exactly when glibc finds a match in it from its start, each line independently of the others — which the automaton of
// a count_exact plan decides — and the -m limit only caps the total.  Two answers depend on the end of the text rather
// than on one line: '$' cannot match at the end of the text under -i (REG_ICASE passed as an execution flag is
// REG_NOTEOL), and a text that ends in '\n' holds an empty string at n that is counted when the last line was not and
// the regex matches there.  The line holding the text's last byte is always among the uncertain keys, so both are
// decided inside glibc's last run, as in the reference; skipping the lines counted on the device changes nothing for the
// runs in between, since each run starts at a line start.
uint64_t regex_answer(const search_params_t *P, RegexMode mode, uint64_t device_lines, const Replay &r, match_result_t *res)
{
    switch (mode)
    {
    case RX_COUNT: return std::min<uint64_t>(device_lines + replay_regex(P, r, nullptr), P->max_count);
    case RX_OFFSETS: return replay_regex_matches(P, r, res);
    default: return replay_regex(P, r, res);
    }
}

uint64_t regex_answer_windows(const search_params_t *P, RegexMode mode, uint64_t device_lines, const std::vector<uint64_t> &keys,
                              const std::vector<RegexWindow> &w, size_t n, int last_byte, bool at_end, match_result_t *res)
{
    switch (mode)
    {
    case RX_COUNT:
        return std::min<uint64_t>(
            device_lines + replay_regex_windows(P, keys.data(), keys.size(), w.data(), w.size(), n, last_byte, at_end, nullptr),
            P->max_count);
    case RX_OFFSETS: return replay_regex_matches_windows(P, keys.data(), keys.size(), w.data(), w.size(), n, last_byte, res);
    default: return replay_regex_windows(P, keys.data(), keys.size(), w.data(), w.size(), n, last_byte, at_end, res);
    }
}

} // namespace kb
