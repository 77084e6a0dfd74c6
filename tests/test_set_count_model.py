"""CPU: the fused -c of pattern sets (csrc/scan_set_count.cu) is exact — line records of a pattern set's occurrences,
cut anywhere and folded in the library's order, give the reference's aho_corasick_search -c.

Each tile of a random tiling is modelled as the device sees it (tests/scan_model.py): its own buffer with a halo and
context bytes, the pattern-set keys it owns, and scan_model.line_record of their starts.  The records are folded by
krep_b200_combine_line_counts and compared with the compiled reference (the oracle port when it is not built).  One set
with a '\\n' pattern shows why such sets keep the occurrence list."""
import ctypes as C
import random

import numpy as np
import pytest

import oracle_util as ou
import scan_model as sm
from krep_b200 import lib
from krep_b200.abi import Params, SIZE_MAX


class LineCount(C.Structure):
    _fields_ = [("lines", C.c_uint64), ("flags", C.c_uint32), ("reserved", C.c_uint32)]


def combine(recs, max_count=SIZE_MAX):
    L = lib.load()
    L.krep_b200_combine_line_counts.argtypes = [C.POINTER(LineCount), C.c_size_t, C.c_size_t]
    L.krep_b200_combine_line_counts.restype = C.c_uint64
    arr = (LineCount * max(len(recs), 1))(*[LineCount(a, b, 0) for a, b in recs])
    return int(L.krep_b200_combine_line_counts(arr, len(recs), max_count))


def checker():
    return ou.reference() or ou.port()


def reference_count(pats, text, cs, ww, max_count):
    p = Params(pats, case_sensitive=cs, whole_word=ww, count=True, max_count=max_count)
    return checker().run("aho_corasick", p, text, with_result=False)[0]


def tile_record(pats, cs, ww, text, b, e, halo):
    """The record of owned range [b, e) scanned from a buffer of its own (halo bytes past e, context bytes)."""
    n = len(text)
    avail = min(e + halo, n)
    buf = text[b:avail]
    prev, nxt = (text[b - 1] if b else -1), (text[avail] if avail < n else -1)
    keys = sm.ac_keys(buf, avail - b, 0, e - b, 0, prev, nxt, pats, cs, ww)
    return sm.line_record(buf, 0, e - b, sm.key_starts(keys, True).astype(np.int64))


def fold_tiles(pats, cs, ww, text, cuts, halo, max_count=SIZE_MAX):
    recs = [tile_record(pats, cs, ww, text, b, e, halo) for b, e in zip(cuts, cuts[1:])]
    return combine(recs, max_count), recs


ALPHABETS = [
    b"ab\n",
    b"abAB \n",
    b"ab\x00\r\n",
    bytes(range(256)),
    b"\xe9\xc9\x80\xffa\n",
    b"a_1 Z\xe9\n",       # word bytes next to spaces and high bytes (-w)
    b"abc\n\n\n",          # empty lines
    b"abcAB\x00\r ",       # no newline at all
]


def derived_set(rng, alpha):
    """A set with overlapping members, prefixes and suffixes of each other, duplicates, case twins and 1-byte ones."""
    body = bytes(c for c in alpha if c != 10) or b"a"
    pats = [bytes(rng.choice(body) for _ in range(rng.randint(1, 5))) for _ in range(rng.randint(1, 4))]
    base = rng.choice(pats)
    extra = [base[:max(1, len(base) - 1)], base[1:] or base, base, base.swapcase(), bytes([rng.choice(body)]),
             base + bytes([rng.choice(body)])]
    pats += rng.sample(extra, rng.randint(0, len(extra)))
    rng.shuffle(pats)
    return pats


def random_text(rng, alpha, pats):
    n = rng.choice([1, 2, 7, 16, 33, 64, 100, 257, 600])
    out = bytearray()
    while len(out) < n:
        if rng.random() < 0.3:
            p = rng.choice(pats)
            out += p if rng.random() < 0.6 else p.swapcase()
        else:
            out += bytes(rng.choice(alpha) for _ in range(rng.randint(1, 6)))
    text = bytes(out[:n])
    if rng.random() < 0.3 and 10 in alpha:
        text += b"\n"
    return text


def random_cuts(rng, text, pats):
    """0, n, and cuts at random bytes, on a hit's first byte, inside a hit, on a newline and just after one."""
    n = len(text)
    cuts = {0, n}
    for _ in range(rng.choice([0, 1, 2, 5, 9])):
        cuts.add(rng.randint(0, n))
    starts = sm.key_starts(sm.ac_keys(text, n, 0, n, 0, -1, -1, pats, True, False), True).astype(np.int64)
    nls = [i for i, c in enumerate(text) if c == 10]
    for arr, deltas in ((starts.tolist(), (0, 1)), (nls, (0, 1))):
        for q in rng.sample(arr, min(2, len(arr))):
            cuts.add(min(q + rng.choice(deltas), n))
    return sorted(cuts)


@pytest.mark.parametrize("seed", range(6))
def test_folded_set_records_equal_the_reference_count(seed):
    rng = random.Random(9090 + seed)
    checked = 0
    for _ in range(400):
        alpha = rng.choice(ALPHABETS)
        pats = derived_set(rng, alpha)
        text = random_text(rng, alpha, pats)
        cs, ww = rng.random() < 0.5, rng.random() < 0.3
        mc = rng.choice([SIZE_MAX, SIZE_MAX, 1, 2, 7])
        halo = max(len(p) for p in pats) - 1 + rng.choice([0, 0, 1, 7])
        cuts = random_cuts(rng, text, pats)
        got, recs = fold_tiles(pats, cs, ww, text, cuts, halo, mc)
        want = reference_count(pats, text, cs, ww, mc)
        assert got == want, (pats, text, cs, ww, mc, cuts, halo, recs, want)
        checked += 1
    assert checked == 400


def test_fixed_sets_by_hand():
    """Overlaps, a prefix and a suffix of one line counted once; -m caps; a line cut inside a hit is counted once."""
    text = b"abcd\nxbcy\n\nabab\r\nno"
    pats = [b"abc", b"bc", b"c", b"ab", b"abc"]
    want = reference_count(pats, text, True, False, SIZE_MAX)
    assert want == 3
    n = len(text)
    for cuts in ([0, n], [0, 1, 2, 3, n], [0, 5, 6, 7, n], [0, 13, n], list(range(n + 1))):
        assert fold_tiles(pats, True, False, text, cuts, 2)[0] == want, cuts
    assert fold_tiles(pats, True, False, text, [0, 7, n], 2, 2)[0] == 2
    # -i with case twins, -w with a word byte after the hit
    twins, t2 = [b"AB", b"ab"], b"Ab\naB\nx"
    assert fold_tiles(twins, False, False, t2, [0, 4, 7], 1)[0] == reference_count(twins, t2, False, False, SIZE_MAX) == 2
    t3 = b"ab_\nab"
    assert fold_tiles([b"ab"], True, True, t3, [0, 2, 6], 1)[0] == reference_count([b"ab"], t3, True, True, SIZE_MAX) == 1


def test_a_newline_in_a_pattern_breaks_the_record():
    """With '\\n' in a pattern an occurrence spans two lines, and start lines are no longer ordered like ends: in "x\\nab"
    the reference meets "a" (line 2), then "x\\nab" (line 1), then "b" (line 2 again) and counts three lines, while the
    record counts the two lines that hold a start.  Such sets keep the occurrence list (count_lines_eligible)."""
    pats, text = [b"a", b"x\nab", b"b"], b"x\nab"
    want = reference_count(pats, text, True, False, SIZE_MAX)
    got = fold_tiles(pats, True, False, text, [0, len(text)], 2)[0]
    assert got != want, (got, want)
