"""CPU check of tests/regex_long_model.py, the reference the GPU tests hold the -E long-line pass to: over random regexes,
texts with many lines longer than the kernel's reach and random tilings into shards, the model's decided answers plus
the reference loop over the lines it leaves uncertain reproduce the reference's -c count, -co count and positions, with
-i and -m; lines the filter drops have no match; and where no line is out of reach the model is regex_kernel_model's."""
import ctypes as C
import random

import pytest

from krep_b200 import lib
from krep_b200.abi import Params
import regex_kernel_model as km
import regex_long_model as lm
import regex_util as ru


def _params(pats, icase, **kw):
    try:
        return Params([p.encode() for p in pats], regex=True, case_sensitive=not icase, **kw)
    except ValueError:
        return None


def _flagged(params, buf):
    L = lib.load()
    b = C.create_string_buffer(bytes(buf), len(buf) + 1)
    cap = bytes(buf).count(b"\n") + 2
    out = (C.c_uint64 * cap)()
    k = L.krep_b200_regex_filter_host(params.ref(), b, len(buf), out, cap, None)
    assert 0 <= k <= cap, k
    return set(out[:k])


def test_taken_lines_follow_the_contract():
    R = km.REGEX_SEG + km.REGEX_HALO
    # out of reach with its '\n' within avail_len: taken; the '\n' at limit - 1: the kernel's own line
    sh = km.Shard(b"a" * R + b"\nb\n", 0, km.REGEX_SEG)
    assert lm.taken_lines(sh) == [(0, R)]
    sh = km.Shard(b"a" * (R - 1) + b"\nb\n", 0, km.REGEX_SEG)
    assert lm.taken_lines(sh) == []
    # the text's last line stays uncertain; with a byte after the shard it is taken
    assert lm.taken_lines(km.Shard(b"a" * R + b"\n", 0, km.REGEX_SEG)) == []
    assert lm.taken_lines(km.Shard(b"a" * R + b"\n", 0, km.REGEX_SEG, next_byte=ord("b"))) == [(0, R)]
    # the '\n' beyond avail_len
    assert lm.taken_lines(km.Shard(b"a" * (R + 10), 0, km.REGEX_SEG, next_byte=ord("\n"))) == []
    # a line starting mid-shard, owned from own_begin > 0
    buf = b"xy\n" + b"c" * 9000 + b"\nz\n"
    assert lm.taken_lines(km.Shard(buf, 2, 300, prev_byte=ord("q"))) == [(3, 9003)]


@pytest.mark.parametrize("icase", [False, True])
def test_model_plus_reference_is_the_reference(icase):
    rng = random.Random(11 + icase)
    checked = 0
    for it in range(40):
        pats = [rng.choice(["a[^x]*b", "(ab)*c", "^x.*y$", "a{3}b", ".*QQ|,", "b+ ", "x$", "^a", "c a"]) if rng.random() < 0.5
                else ru.random_regex(rng) for _ in range(rng.choice([1, 1, 2]))]
        Pc = _params(pats, icase, count=True)
        Pp = _params(pats, icase)
        if Pc is None or Pp is None:
            continue
        m = rng.choice([1, 3, 1 << 62])
        Pcm = _params(pats, icase, count=True, max_count=m)
        Pco = _params(pats, icase, count=True, only_matching=True)
        Ppm = _params(pats, icase, max_count=m)
        text = lm.long_lines_text(rng, rng.randint(1, 40000))
        n = len(text)
        cuts = [rng.randint(0, n) for _ in range(rng.choice([0, 1, 2, 4]))]
        count_keys, match_keys, lines = [], [], 0
        for d, sh in km.tiling(text, cuts, rng):
            g = km.GlibcLines(Pp, sh.buf)
            e1 = lm.expect(sh, 1, g)
            e2 = lm.expect(sh, 2, g, budget_free=True)
            count_keys += e1.keys
            lines += e1.device_lines
            # a line that keeps its key in match mode goes to the reference loop whole
            match_keys += e2.keys + sorted(e2.must_flag)
            flagged = _flagged(Pp, sh.buf)
            for p, nl in lm.taken_lines(sh):
                if p not in flagged:
                    assert not g.verdict(p, nl), (pats, icase, d + p)
        total = km.resolve(Pc, text, 0, count_keys=count_keys, device_lines=lines)
        assert total == ru.ref_regex_search(Pc, text)[0], (pats, icase, n, sorted(cuts))
        assert min(total, m) == ru.ref_regex_search(Pcm, text)[0], (pats, icase, n, m)
        pos = km.resolve(Pp, text, 0, match_keys=sorted(match_keys))
        assert pos == ru.ref_regex_search(Pp, text)[1], (pats, icase, n, sorted(cuts))
        assert len(pos) == ru.ref_regex_search(Pco, text)[0], (pats, icase, n)
        assert pos[:m] == ru.ref_regex_search(Ppm, text)[1], (pats, icase, n, m)
        checked += 1
    assert checked > 25


def test_long_match_keeps_the_key():
    # a match of 8192 bytes or more does not fit the key: the line keeps its key with the matches before it
    P = _params(["b|a+"], False)
    line = b"b" + b"a" * 9000 + b"b"
    sh = km.Shard(line + b"\nx\n")
    e = lm.expect(sh, 2, km.GlibcLines(P, sh.buf))
    lk = 0
    assert e.must_flag == {lk}
    assert e.prefix_lines[lk] == [(0 << 16) | (1 << 3) | 1]


def test_equals_kernel_model_within_reach():
    rng = random.Random(5)
    for it in range(40):
        P = _params([ru.random_regex(rng)], rng.random() < 0.3)
        if P is None:
            continue
        text = b"".join(ru.random_text(rng, rng.randint(1, 300)) for _ in range(rng.randint(1, 40)))
        for d, sh in km.tiling(text, [rng.randint(0, len(text))], rng):
            g = km.GlibcLines(P, sh.buf)
            flagged = _flagged(P, sh.buf)
            assert lm.taken_lines(sh) == []
            for mode, oracle in ((0, flagged), (1, g), (2, g)):
                a, b = lm.expect(sh, mode, oracle), km.expect(sh, mode, oracle)
                assert (a.keys, a.device_lines, a.optional, a.prefix_lines) == \
                    (b.keys, b.device_lines, b.optional, b.prefix_lines), (it, mode)
