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


def test_sizes_follow_the_design():
    # DESIGN §12.8: one round for a 256 MiB chunk and its halo, 3 for a 10 GiB shard at G = 1, 22 at G = 8
    chunk = 256 << 20
    assert lm.sizes(chunk + km.REGEX_HALO, chunk, 1).rounds == 1
    assert lm.sizes(10 << 30, 10 << 30, 1).rounds == 3
    z = lm.sizes(10 << 30, 10 << 30, 8)
    assert z.rounds == 22 and z.nck == 17 and z.round_slices == (64 << 20) // 272
    assert [lm.sizes(10 << 30, 10 << 30, n).rounds for n in (2, 3, 5, 7)] == [6, 11, 22, 22]
    # the per-round slice counts the GPU tests size their texts from: slice 1 / checkpoint 1, and 1024 / 1
    big = 1 << 30
    assert [lm.sizes(big, big, g, 1, 1).round_slices for g in (1, 2, 4, 8)] == [16777216, 8388608, 4194304, 2097152]
    assert [lm.sizes(big, big, g, 1024, 1).round_slices for g in (1, 8)] == [32736, 4092]
    # a checkpoint that does not divide the slice adds a short last one; the round never exceeds the slice map
    assert lm.sizes(100, 100, 1, 7, 3).nck == 4 and lm.sizes(100, 100, 1, 7, 3).round_slices == 17
    assert lm.sizes(0, 0, 1).rounds == 1 and lm.sizes(0, 0, 1).pick_cap == 2
    assert lm.sizes(1 << 20, 1 << 20, 1).pick_cap == (1 << 20) // 4097 + 2


def test_slices_needed():
    R = km.REGEX_SEG + km.REGEX_HALO
    # lines of k*S - 1, k*S and k*S + 1 bytes: k, k and k + 1 slices; a line the pass does not take adds none
    for n, want in ((2 * R - 1, 2), (2 * R, 2), (2 * R + 1, 3)):
        sh = km.Shard(b"a" * n + b"\nb\n", 0, km.REGEX_SEG)
        assert lm.slices_needed(sh, R) == want, n
    sh = km.Shard(b"a" * (R - 1) + b"\n" + b"b" * 5000 + b"\n" + b"c" * 6000 + b"\n", 0, km.REGEX_SEG + R)
    assert lm.taken_lines(sh) == [(R, R + 5000)]
    assert lm.slices_needed(sh, 1) == 5000 and lm.slices_needed(sh) == 2


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


def test_host_twin_leaves_long_matches_to_regexec():
    # krep_b200_regex_matches_host with unbounded reach (the GPU tests' oracle for long texts): a match of 8192 bytes or
    # more does not fit the key's 13-bit length field, so the line goes to regexec whole, as in the long-line pass
    for pats, body in ((["b|a+"], lambda n: b"b" + b"a" * n + b"b"), (["^[^x]*kqk"], lambda n: b"kqk" + b"c" * n + b"kqk")):
        P = _params(pats, False)
        for n in (8185, 8186, 8191, 8192, 16663, 30919):
            text = b"x\n" + body(n) + b"\nz" * 3 + b"\n"
            assert km.HookLines(P, text, P).pos == ru.ref_regex_search(P, text)[1], (pats, n)


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
