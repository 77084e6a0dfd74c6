// regex_rows.cpp — a -E search's answer from the rows of the resident shards that tile the text (DESIGN §12.4, §12.6).
//
// A row (layout: RegexRowHeader, csrc/common.h) holds what glibc needs of one shard: its keys, and the bytes of the
// lines glibc must see, packed into segments.  The resolver stitches the segments cut at a shard's readable end with the
// heads of the shards that follow, and replays the rows' keys over the segments as windows (replay_regex_windows), so
// the answer is krep_b200_regex_search's on the same text without that text.
//
// One resolver answers for a part of the rows: the lines owned by consecutive shards, with only the heads of the shards
// after them.  The whole text is the part that owns every row and decides the end of the text; a rank of a
// one-process-per-GPU job resolves its own shard as a part, and the parts' answers concatenate (DESIGN §12.6).
#include <algorithm>
#include <cstring>
#include <deque>
#include <string>
#include <vector>
#include "common.h"

namespace kb {

static_assert(KREP_B200_REGEX_ROW_HEADER == sizeof(RegexRowHeader), "the header size the C ABI names");

namespace {
struct RowView
{
    const RegexRowHeader *h;
    const uint64_t *keys;
    const RegexRowSeg *segs;
    const char *head;
    const char *bytes; // the first segment's bytes
};

bool view_row(const void *row, uint64_t mode, RowView *v)
{
    const RegexRowHeader *h = (const RegexRowHeader *)row;
    if (!h || h->magic != REGEX_ROW_MAGIC || h->mode > RX_OFFSETS || h->mode != mode) return false;
    const uint8_t *b = (const uint8_t *)h;
    v->h = h;
    v->keys = (const uint64_t *)(b + sizeof(RegexRowHeader));
    v->segs = (const RegexRowSeg *)(v->keys + h->nkeys);
    v->head = (const char *)b + regex_row_fixed_bytes(h->nkeys, h->nseg);
    v->bytes = v->head + round16(h->head_len);
    return true;
}

// The shard owns a line start: a line starts at its own_begin (no head) or right after its head, inside its range.
bool holds_line_start(const RegexRowHeader &h)
{
    return h.own_begin < h.own_end && (!(h.flags & ROW_HEAD) || h.own_begin + h.head_len < h.own_end);
}

// The answer of the lines owned by v[0, n_own), capped at P->max_count.  v[n_own, n_rows) are the shards that follow,
// in order; only their heads are read.  Why a part's answer is exact (DESIGN §12.6):
//  - a line belongs to the shard that holds its first byte; a part replays only its own lines' windows, and a line cut
//    at its readable end is stitched from the heads that follow.  Every window starts at a line start and the replay
//    stops at each window's end (Replay::stop), so nothing but the -m budget crosses from one part into the next;
//  - the empty string at n is tried by exactly one part: at_end (the owner of the last line start).  Only that part can
//    have a window that ends at n; the others must not try it from an empty window at n either, or a text ending in
//    '\n' would count '^$' or 'x*' there once per part;
//  - each part resolves with the whole max_count, so its answer is the first max_count items of its unbounded answer:
//    the parts' answers concatenated in text order and cut to max_count are the whole answer.
uint64_t resolve_views(const search_params_t *P, const std::vector<RowView> &v, uint32_t n_own, size_t n, int last_byte,
                       bool at_end, match_result_t *res, int *err)
{
    const uint32_t n_rows = (uint32_t)v.size();
    if (n == 0)
    {
        *err = 0;
        return at_end ? regex_empty_text(P, res) : 0;
    }

    // windows: the segments in text order, a segment cut at its shard's readable end completed from the heads after it
    std::vector<RegexWindow> win;
    std::deque<std::string> stitched; // owns the bytes of completed segments (deque: stable addresses)
    std::vector<uint64_t> keys;
    uint64_t device_lines = 0;
    for (uint32_t i = 0; i < n_own; i++)
    {
        const RowView &r = v[i];
        keys.insert(keys.end(), r.keys, r.keys + r.h->nkeys);
        device_lines += r.h->device_lines;
        const char *p = r.bytes;
        for (uint64_t s = 0; s < r.h->nseg; s++)
        {
            const uint64_t start = r.segs[s].start, len = r.segs[s].len_cont >> 1;
            const bool cont = r.segs[s].len_cont & 1;
            if ((!win.empty() && start < win.back().origin + win.back().len) || start + len > n)
            {
                set_error(-3, "krep_b200_regex_resolve: row %u: segments overlap, are out of order or end past the text", i);
                return 0;
            }
            if (!cont)
            {
                win.push_back(RegexWindow{(size_t)start, p, (size_t)len});
                p += round16(len);
                continue;
            }
            // the line goes on past this shard's readable bytes: into the heads of the shards that follow
            std::string line(p, (size_t)len);
            p += round16(len);
            uint64_t have = start + len;
            bool done = false;
            for (uint32_t j = i + 1; j < n_rows && !done; j++)
            {
                const RegexRowHeader &hj = *v[j].h;
                if (!(hj.flags & ROW_HEAD) || hj.own_begin > have)
                {
                    set_error(-3, "krep_b200_regex_resolve: the line at %llu runs past row %u's readable bytes but row %u "
                                  "does not continue it", (unsigned long long)start, i, j);
                    return 0;
                }
                const uint64_t he = hj.own_begin + hj.head_len;
                if (he > have) line.append(v[j].head + (have - hj.own_begin), (size_t)(he - have));
                have = std::max(have, he);
                done = hj.head_len && v[j].head[hj.head_len - 1] == '\n';
            }
            if (!done && have != n)
            {
                set_error(-3, "krep_b200_regex_resolve: the line at %llu ends nowhere", (unsigned long long)start);
                return 0;
            }
            stitched.push_back(std::move(line));
            win.push_back(RegexWindow{(size_t)start, stitched.back().data(), stitched.back().size()});
        }
    }
    *err = 0;
    return regex_answer_windows(P, (RegexMode)v[0].h->mode, device_lines, keys, win, n, last_byte, at_end, res);
}
} // namespace

uint64_t regex_resolve_rows(const search_params_t *P, const void *const *rows, uint32_t n_rows, match_result_t *res, int *err)
{
    *err = -3;
    if (!rows || n_rows == 0)
    {
        set_error(-3, "krep_b200_regex_resolve: no rows");
        return 0;
    }
    std::vector<RowView> v(n_rows);
    for (uint32_t i = 0; i < n_rows; i++)
    {
        if (!rows[i] || !view_row(rows[i], ((const RegexRowHeader *)rows[0])->mode, &v[i]))
        {
            set_error(-3, "krep_b200_regex_resolve: row %u is not a regex row of the same mode as row 0", i);
            return 0;
        }
        const RegexRowHeader *h = v[i].h;
        // the shards must tile one whole text: owned ranges that abut from 0, the last one ending the text
        const bool first_ok = i > 0 || h->own_begin == 0;
        const bool abut = i == 0 || v[i - 1].h->own_end == h->own_begin;
        const bool last_ok = (i + 1 == n_rows) == ((h->flags & ROW_LAST) != 0);
        if (!first_ok || !abut || !last_ok || h->own_end > h->avail_end || h->own_begin > h->own_end)
        {
            set_error(-3, "krep_b200_regex_resolve: the rows do not tile one text (row %u owns [%llu, %llu))", i,
                      (unsigned long long)h->own_begin, (unsigned long long)h->own_end);
            return 0;
        }
    }
    const RegexRowHeader &last = *v[n_rows - 1].h;
    const size_t n = (size_t)last.avail_end;
    const int last_byte = n ? (int)((last.flags >> ROW_LAST_BYTE_SHIFT) & 0xFF) : -1;
    return resolve_views(P, v, n_rows, n, last_byte, true, res, err); // the part that owns every row
}

// Each text of a packed batch is resolved alone, as resolve_views resolves a one-shard text: its keys and the parts of the
// row's segments that lie in it, moved to its own coordinates, replayed over its own length, last byte and -m budget.
// A segment can run past a text's end (its last line ends at the gap's '\n') or into the next text (lines of two texts
// that abut across a one-byte gap merge into one segment): only the bytes inside the text are its window.  Every window
// still starts at a line start, the text's own or its first byte.
int regex_resolve_batch(const search_params_t *P, const void *row, size_t n_texts, const uint64_t *lo, const size_t *len,
                        const uint8_t *last, const uint64_t *text_lines, uint64_t *counts, match_result_t *const *res)
{
    RowView v;
    if (!row || !view_row(row, ((const RegexRowHeader *)row)->mode, &v))
    {
        set_error(-3, "regex batch: not a regex row");
        return -3;
    }
    const RegexMode mode = (RegexMode)v.h->mode;
    const uint64_t nkeys = v.h->nkeys, nseg = v.h->nseg;
    const int shift = regex_key_shift(mode);
    std::vector<const char *> bytes(nseg);
    const char *p = v.bytes;
    for (uint64_t s = 0; s < nseg; s++)
    {
        if (v.segs[s].len_cont & 1)
        {
            set_error(-3, "regex batch: a segment runs past the packed buffer");
            return -3;
        }
        bytes[s] = p;
        p += round16(v.segs[s].len_cont >> 1);
    }
    std::vector<uint64_t> keys;
    std::vector<RegexWindow> win;
    uint64_t j = 0, s0 = 0;
    for (size_t i = 0; i < n_texts; i++)
    {
        const uint64_t b = lo[i], e = lo[i] + len[i];
        keys.clear();
        while (j < nkeys && (v.keys[j] >> shift) < b) j++;
        for (; j < nkeys && (v.keys[j] >> shift) < e; j++) keys.push_back(v.keys[j] - (b << shift));
        win.clear();
        while (s0 < nseg && v.segs[s0].start + (v.segs[s0].len_cont >> 1) <= b) s0++;
        for (uint64_t s = s0; s < nseg && v.segs[s].start < e; s++)
        {
            const uint64_t sb = std::max<uint64_t>(v.segs[s].start, b), se = std::min<uint64_t>(v.segs[s].start + (v.segs[s].len_cont >> 1), e);
            if (se > sb) win.push_back(RegexWindow{(size_t)(sb - b), bytes[s] + (sb - v.segs[s].start), (size_t)(se - sb)});
        }
        counts[i] = regex_answer_windows(P, mode, mode == RX_COUNT ? text_lines[i] : 0, keys, win, len[i], last[i], true,
                                         res ? res[i] : nullptr);
    }
    return 0;
}

} // namespace kb

using namespace kb;

uint64_t krep_b200_regex_resolve_part(const search_params_t *P, const void *const *rows, uint32_t n_rows, uint32_t n_own,
                                      uint64_t text_len, int last_byte, int decides_end, match_result_t *result)
{
    clear_error();
    if (!P) return 0;
    if (regex_returns_early(P)) return 0;
    if (!rows || n_own == 0 || n_own > n_rows || (text_len && (last_byte < 0 || last_byte > 255)))
    {
        set_error(-3, "krep_b200_regex_resolve_part: needs 1 <= n_own <= n_rows rows, and the last byte of a non-empty text");
        return 0;
    }
    std::vector<RowView> v(n_rows);
    for (uint32_t i = 0; i < n_rows; i++)
    {
        if (!rows[i] || !view_row(rows[i], ((const RegexRowHeader *)rows[0])->mode, &v[i]))
        {
            set_error(-3, "krep_b200_regex_resolve_part: row %u is not a regex row of the same mode as row 0", i);
            return 0;
        }
        // consecutive shards of one tiling of text_len bytes; a non-empty shard that ends the text carries its last byte
        const RegexRowHeader *h = v[i].h;
        const bool abut = i == 0 || v[i - 1].h->own_end == h->own_begin;
        const bool last_ok = !(h->flags & ROW_LAST) ||
                             (h->avail_end == text_len &&
                              (h->own_begin == h->own_end || (int)((h->flags >> ROW_LAST_BYTE_SHIFT) & 0xFF) == last_byte));
        if (!abut || !last_ok || h->own_begin > h->own_end || h->own_end > h->avail_end || h->avail_end > text_len)
        {
            set_error(-3, "krep_b200_regex_resolve_part: the rows are not consecutive shards of one text of %llu bytes (row %u "
                          "owns [%llu, %llu))", (unsigned long long)text_len, i, (unsigned long long)h->own_begin,
                      (unsigned long long)h->own_end);
            return 0;
        }
    }
    int err = 0;
    const uint64_t ret = resolve_views(P, v, n_own, (size_t)text_len, last_byte, decides_end != 0, result, &err);
    return err ? 0 : ret;
}

uint64_t krep_b200_regex_row_head(const void *row, void *dst, uint64_t cap)
{
    clear_error();
    RowView v;
    if (!row || !view_row(row, ((const RegexRowHeader *)row)->mode, &v))
    {
        set_error(-3, "krep_b200_regex_row_head: not a regex row");
        return 0;
    }
    const uint64_t bytes = regex_row_fixed_bytes(0, 0) + round16(v.h->head_len);
    if (!dst || cap < bytes) return bytes;
    RegexRowHeader h = *v.h;
    h.row_bytes = bytes;
    h.device_lines = 0;
    h.nkeys = h.nseg = 0;
    memcpy(dst, &h, sizeof h);
    memset((char *)dst + sizeof h, 0, bytes - sizeof h);
    memcpy((char *)dst + regex_row_fixed_bytes(0, 0), v.head, v.h->head_len);
    return bytes;
}

int krep_b200_regex_tiling(const void *headers, uint32_t n, krep_b200_regex_tiling_t *out, int32_t *head_to,
                           uint64_t *head_bytes)
{
    clear_error();
    if (!headers || n == 0 || !out)
    {
        set_error(-3, "krep_b200_regex_tiling: no rows");
        return -3;
    }
    auto hdr = [&](uint32_t i) { return (const RegexRowHeader *)((const char *)headers + (size_t)i * sizeof(RegexRowHeader)); };
    const uint64_t text_len = hdr(n - 1)->avail_end;
    int32_t last_byte = -1;
    for (uint32_t i = 0; i < n; i++)
    {
        const RegexRowHeader &h = *hdr(i);
        const bool row_ok = h.magic == REGEX_ROW_MAGIC && h.mode <= RX_OFFSETS && h.mode == hdr(0)->mode;
        const bool first_ok = i > 0 || (h.own_begin == 0 && !(h.flags & ROW_HEAD)); // the text starts at a line start
        const bool abut = i == 0 || hdr(i - 1)->own_end == h.own_begin;
        // a shard ends the text when it owns up to its end; only empty shards may follow it (shard_bounds gives trailing
        // shards an empty range when the text is short), and the last shard ends it
        const bool last_ok = (h.flags & ROW_LAST) ? h.own_end == text_len && h.avail_end == text_len
                                                  : i + 1 < n && h.own_end < text_len;
        if (!row_ok || !first_ok || !abut || !last_ok || h.own_begin > h.own_end || h.own_end > h.avail_end ||
            h.avail_end > text_len)
        {
            set_error(-3, "krep_b200_regex_tiling: the rows do not tile one text (row %u owns [%llu, %llu) of %llu bytes)", i,
                      (unsigned long long)h.own_begin, (unsigned long long)h.own_end, (unsigned long long)text_len);
            return -3;
        }
        // the first shard that ends the text holds its last byte (an empty one after it may not)
        if (text_len && last_byte < 0 && (h.flags & ROW_LAST)) last_byte = (int32_t)((h.flags >> ROW_LAST_BYTE_SHIFT) & 0xFF);
    }
    out->text_len = text_len;
    out->last_byte = last_byte;
    out->decider = 0;
    int32_t holder = -1; // the last shard so far that holds a line start
    for (uint32_t i = 0; i < n; i++)
    {
        const RegexRowHeader &h = *hdr(i);
        const bool sends = (h.flags & ROW_HEAD) && holder >= 0;
        if (head_to) head_to[i] = sends ? holder : -1;
        if (head_bytes) head_bytes[i] = sends ? regex_row_fixed_bytes(0, 0) + round16(h.head_len) : 0;
        if (holds_line_start(h))
        {
            holder = (int32_t)i;
            out->decider = i;
        }
    }
    return 0;
}
