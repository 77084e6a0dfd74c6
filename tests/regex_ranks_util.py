"""Shared by the rank-sharded -E tests: texts cut into shards at every kind of place a cut can fall, and the answer of
a tiling assembled from per-part answers (krep_b200_regex_resolve_part) the way krep_b200/sharding.py assembles it."""
import random

import regex_kernel_model as km
import regex_rows_util as rr
from krep_b200 import lib

PATTERNS = [("^$", dict()), ("x*", dict()), ("x$", dict(case_sensitive=False)), ("the[a-z]*", dict(whole_word=True)),
            ("\\bthe", dict()), ("the[a-z]*", dict())]
MODES = [dict(), dict(count=True), dict(count=True, only_matching=True), dict(only_matching=True), dict(max_count=1),
         dict(max_count=2), dict(max_count=3), dict(max_count=7), dict(count=True, max_count=2),
         dict(count=True, only_matching=True, max_count=3)]
HALOS = [0, 17, km.REGEX_HALO]


def params(pat, **kw):
    from krep_b200.abi import Params
    return Params([pat.encode() if isinstance(pat, str) else pat], regex=True, **kw)


def _body(seed):
    rng = random.Random(seed)
    words = [b"the", b"thex", b"x", b"X", b"ab", b"other", b"", b"the_", b"xx"]
    lines = []
    for _ in range(40):
        lines.append(b" ".join(rng.choice(words) for _ in range(rng.randint(0, 6))))
    return b"\n".join(lines)


def cut_texts(world):
    """-> [(name, text, cuts)] with len(cuts) == world - 1: cuts at a line start, mid-line, on a '\\n', inside a last
    line that spans three shards (two when world == 2), a shard that holds no line start, trailing empty shards (as
    shard_bounds gives a short text), each text with and without a final '\\n'."""
    out = []
    for tail in (b"\n", b""):
        body = _body(len(tail))
        n0 = len(body)
        long_last = b"the " + b"x" * 300 + b" the thex"
        for name, text, want in [
            ("line_start", body + tail, lambda t: [t.index(b"\n", 50 * i + 10) + 1 for i in range(1, world)]),
            ("mid_line", body + tail, lambda t: [t.index(b"\n", 50 * i + 10) - 2 for i in range(1, world)]),
            ("on_newline", body + tail, lambda t: [t.index(b"\n", 50 * i + 10) for i in range(1, world)]),
            # the last two cuts fall inside the last line: it spans three shards (with world 2: two)
            ("last_line_spans", body + b"\n" + long_last + tail,
             lambda t: ([40 * i for i in range(1, world - 2)] + [n0 + 101, n0 + 201])[-(world - 1):]),
            # shards inside one long line hold no line start (with 2 shards: the second, inside the last line)
            ("no_line_start", b"ab\nthe " + b"y" * 500 + b" x\nthe x" + tail,
             lambda t: [100, 300, 400, 505, 508, 512][:world - 1]),
            ("trailing_empty", b"the x\nab" + tail, lambda t: [len(t)] * (world - 1)),
        ]:
            cuts = sorted(want(text))
            assert len(cuts) == world - 1 or world == 1, (name, cuts)
            out.append((name + ("_nl" if tail else "_no_nl"), text, cuts[:world - 1] if world > 1 else []))
    return out


def tiling_rows(P, text, cuts, halo):
    return [rr.twin_row(P, sh) for sh in rr.tile(text, cuts, halo)]


def part_rows(rows, tiling_info, first, end):
    """The rows part [first, end) resolves: its own rows, then the head-only rows of the shards whose heads it reads."""
    _t, head_to, _nb = tiling_info
    heads = [lib.regex_row_head(rows[j]) for j in range(end, len(rows)) if first <= head_to[j] < end]
    return rows[first:end] + heads


def parts_answer(P, rows, groups):
    """The answer assembled from parts: groups = [(first, end)] consecutive ranges of rows, each resolved with
    krep_b200_regex_resolve_part; answers concatenated in order and cut to max_count."""
    info = lib.regex_tiling(b"".join(bytes(r[:lib.REGEX_ROW_HEADER]) for r in rows), len(rows))
    t = info[0]
    count, pos = 0, []
    for first, end in groups:
        c, p = lib.regex_resolve_part(P, part_rows(rows, info, first, end), end - first, t.text_len, t.last_byte,
                                      first <= t.decider < end)
        count += c
        pos += p
    mc = P.struct.max_count
    return min(count, mc), pos[:mc]
