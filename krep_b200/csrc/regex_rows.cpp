// regex_rows.cpp — a -E search's answer from the rows of the resident shards that tile the text (DESIGN §12.4).
//
// A row (layout: RegexRowHeader, csrc/common.h) holds what glibc needs of one shard: its keys, and the bytes of the
// lines glibc must see, packed into segments.  The resolver stitches the segments cut at a shard's readable end with the
// heads of the shards that follow, and replays the rows' keys over the segments as windows (replay_regex_windows), so
// the answer is krep_b200_regex_search's on the same text without that text.
#include <algorithm>
#include <cstring>
#include <deque>
#include <string>
#include <vector>
#include "common.h"

namespace kb {

namespace {
struct RowView
{
    const RegexRowHeader *h;
    const uint64_t *keys;
    const RegexRowSeg *segs;
    const char *head;
    const char *bytes; // the first segment's bytes
};
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
        const RegexRowHeader *h = (const RegexRowHeader *)rows[i];
        if (!h || h->magic != REGEX_ROW_MAGIC || h->mode > 2 || h->mode != ((const RegexRowHeader *)rows[0])->mode)
        {
            set_error(-3, "krep_b200_regex_resolve: row %u is not a regex row of the same mode as row 0", i);
            return 0;
        }
        const uint8_t *b = (const uint8_t *)h;
        const uint64_t fixed = regex_row_fixed_bytes(h->nkeys, h->nseg);
        v[i].h = h;
        v[i].keys = (const uint64_t *)(b + sizeof(RegexRowHeader));
        v[i].segs = (const RegexRowSeg *)(v[i].keys + h->nkeys);
        v[i].head = (const char *)b + fixed;
        v[i].bytes = v[i].head + round16(h->head_len);
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
    const uint64_t mode = v[0].h->mode;
    if (n == 0)
    {
        *err = 0;
        return replay_regex(P, Replay{nullptr, 0, nullptr, 0, 0}, res); // krep.c:1403-1416
    }

    // windows: the segments in text order, a segment cut at its shard's readable end completed from the heads after it
    std::vector<RegexWindow> win;
    std::deque<std::string> stitched; // owns the bytes of completed segments (deque: stable addresses)
    std::vector<uint64_t> keys;
    uint64_t device_lines = 0;
    for (uint32_t i = 0; i < n_rows; i++)
    {
        const RowView &r = v[i];
        keys.insert(keys.end(), r.keys, r.keys + r.h->nkeys);
        device_lines += r.h->device_lines;
        const char *p = r.bytes;
        for (uint64_t s = 0; s < r.h->nseg; s++)
        {
            const uint64_t start = r.segs[s].start, len = r.segs[s].len_cont >> 1;
            const bool cont = r.segs[s].len_cont & 1;
            if (!win.empty() && start < win.back().origin + win.back().len)
            {
                set_error(-3, "krep_b200_regex_resolve: row %u: segments overlap or are out of order", i);
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
    uint64_t ret;
    if (mode == 2) ret = replay_regex_matches_windows(P, keys.data(), keys.size(), win.data(), win.size(), n, last_byte, res);
    else if (mode == 1)
        ret = std::min<uint64_t>(device_lines + replay_regex_windows(P, keys.data(), keys.size(), win.data(), win.size(), n,
                                                                     last_byte, true, nullptr),
                                 P->max_count);
    else ret = replay_regex_windows(P, keys.data(), keys.size(), win.data(), win.size(), n, last_byte, true, res);
    return ret;
}

} // namespace kb
