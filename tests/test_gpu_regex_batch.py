"""-E over many texts in one call: krep_b200_regex_search_batch must give every text exactly what
krep_b200_regex_search gives it alone (and what the reference loop gives), on all three paths; and the batch mode of
k_regex_lines, seen through krep_b200_regex_search_batch_raw, must emit exactly what tests/regex_batch_model.py says."""
import ctypes as C
import random

import numpy as np
import pytest

from krep_b200 import lib
from krep_b200.abi import Params
import regex_batch_model as bm
import regex_kernel_model as km
import regex_util as ru

pytestmark = pytest.mark.gpu
SPEC = (0x5EED0001, 0x5EED0002, 1 << 16, b"qzXv9Kpw")
NO_POS = (1 << 64) - 1
KNOBS = [{}, {"KREP_B200_NO_FUSED_COUNT": "1"}, {"KREP_B200_NO_DEVICE_MATCHES": "1"},
         {"KREP_B200_NO_FUSED_COUNT": "1", "KREP_B200_NO_DEVICE_MATCHES": "1"}]


@pytest.fixture(scope="module", autouse=True)
def _init():
    L = lib.load()
    assert L.krep_b200_init(0) == 0, L.krep_b200_last_error_string()


@pytest.fixture(autouse=True)
def _knobs_off(monkeypatch):
    monkeypatch.delenv("KREP_B200_NO_FUSED_COUNT", raising=False)
    monkeypatch.delenv("KREP_B200_NO_DEVICE_MATCHES", raising=False)


def _params(pat, **kw):
    return Params([pat.encode()], regex=True, **kw)


def answer_texts(rng):
    """Every size of the contract, with and without a final '\\n', and the odd texts."""
    out = [b""]
    for n in (1, 15, 16, 17, 255, 256, 257, 4095, 4096, 4097, 9000, 70000):
        body = ru.random_text(rng, n) if n < 9000 else km.random_lines_text(rng, n + 10)[:n]
        out.append(body[:-1] + b"\n")
        out.append(body[:-1] + b"a")
    out += [b"\n", b"\n" * 300, b"\x00" * 40, b"ab\x00ab\n\x00x", b"ab " * 3000, b"ab " * 3000 + b"\n",
            b"x" * (km.REGEX_HALO + 700) + b"\nab\n", b"abc\n\nab", b""]
    rng.shuffle(out)
    return out


PATTERNS = ["^$", "x*", "^", "$", "a|ab|abc", "the[a-z]*", "\\bab\\b", "x$", "a+b"]
OPTIONS = [dict(), dict(case_sensitive=False), dict(whole_word=True), dict(count=True), dict(count=True, only_matching=True),
           dict(max_count=1), dict(max_count=2), dict(max_count=3), dict(count=True, max_count=2)]


def test_answers(monkeypatch):
    rng = random.Random(7)
    texts = answer_texts(rng)
    for pat in PATTERNS:
        for opt in OPTIONS:
            P = _params(pat, **opt)
            want = [ru.ref_regex_search(P, t) for t in texts]
            for knobs in KNOBS:
                for k in ("KREP_B200_NO_FUSED_COUNT", "KREP_B200_NO_DEVICE_MATCHES"):
                    if k in knobs:
                        monkeypatch.setenv(k, knobs[k])
                    else:
                        monkeypatch.delenv(k, raising=False)
                got = lib.regex_search_batch(P, texts)
                for i, t in enumerate(texts):
                    assert got[i] == want[i], (pat, opt, knobs, i, len(t), got[i][0], want[i][0], got[i][1][:4], want[i][1][:4])
                if knobs in ({}, KNOBS[3]):
                    single = [lib.search("regex", P, t) for t in texts]
                    assert got == single, (pat, opt, knobs)
                counts = lib.regex_search_batch(P, texts, with_result=False)
                assert [c for c, _ in counts] == [c for c, _ in want], (pat, opt, knobs)


def raw_batch(P, texts, mode, cap=1 << 16):
    """The hook. -> (sorted keys, packed offsets, per-text device lines); retried with room for every key."""
    L = lib.load()
    n = len(texts)
    _keep, tarr, larr = lib.text_array(texts)
    offs = (C.c_uint64 * max(n, 1))()
    tl = (C.c_uint64 * max(n, 1))()
    first = None
    while True:
        keys = np.zeros(max(cap, 1), dtype=np.uint64)
        k = L.krep_b200_regex_search_batch_raw(P.ref(), tarr, larr, n, mode, offs, keys.ctypes.data_as(C.POINTER(C.c_uint64)),
                                               cap, tl)
        assert k >= 0, (k, L.krep_b200_last_error_string())
        assert first is None or first == k
        if k <= cap:
            return keys[:k].tolist(), list(offs[:n]), list(tl[:n])
        first, cap = k, k


def modes_of(pat, **kw):
    L = lib.load()
    modes = [0]
    if L.krep_b200_regex_count_mode(_params(pat, count=True, **kw).ref()) == 1:
        modes.append(1)
    if L.krep_b200_regex_match_mode(_params(pat, **kw).ref()) == 1:
        modes.append(2)
    return modes


def check_raw(pat, texts, chunk=None, big=False, **kw):
    """Hook vs model in every mode the pattern admits. -> the Batch model"""
    P = _params(pat, **kw)
    b = bm.Batch(texts, chunk)
    flagged = km.HookLines(P, b.buf).flagged
    modes = modes_of(pat, **kw)
    oracle = km.HookLines(P, b.buf, P if 2 in modes else None) if big else km.GlibcLines(P, b.buf)
    for mode in modes:
        keys, offs, tl = raw_batch(P, texts, mode)
        assert offs == [NO_POS if o is None else o for o in b.offs], (pat, mode)
        if mode == 0:
            req, opt = b.expect(0, flagged)
            got = set(keys)
            assert len(got) == len(keys) and set(req) <= got and got <= set(req) | opt, (pat, sorted(set(req) - got)[:4],
                                                                                      sorted(got - set(req) - opt)[:4])
            assert tl == [0] * len(texts)
            continue
        want, per = b.expect(mode, oracle, budget_free=big or pat in BUDGET_FREE)
        assert keys == want, (pat, mode, len(keys), len(want), sorted(set(keys) ^ set(want))[:4])
        assert tl == [per.get(i, 0) for i in range(len(texts))], (pat, mode)
    return b


BUDGET_FREE = {"b$", "^a", "x*", "ab"}


def short_line_texts(rng, k):
    """Texts of lines of at most 30 bytes (no line can reach the match mode's step budget), some without a final '\\n'."""
    out = []
    for _ in range(k):
        lines = [bytes(rng.choice(b"aabbcx ") for _ in range(rng.randint(0, 30))) for _ in range(rng.randint(1, 60))]
        t = b"\n".join(lines) + (b"\n" if rng.random() < 0.5 else b"")
        out.append(t if rng.random() > 0.05 else b"")
    return out


def test_raw_against_model():
    rng = random.Random(21)
    texts = short_line_texts(rng, 200)
    for pat in ["b$", "^a", "x*", "ab", "a+b", "(ab|ba)c?", "^$", "a|ab|abc", "\\bab\\b"]:
        b = check_raw(pat, texts)
        # count mode on short lines: the only uncertain line of a text is its last one
        unc = {p for i, p, _, u in b.lines if u}
        assert unc == {b.offs[i] + ru.line_starts(texts[i])[-1] for i in b.live}, pat
    long_texts = answer_texts(rng)
    for pat in ["b$", "^a", "x*", "ab"]:
        check_raw(pat, long_texts)
    check_raw("a+b", texts, case_sensitive=False)


def _corpus_texts(rng, k, lo, hi):
    n = k * hi
    corpus = lib.corpus_host(lib.make_spec(*SPEC), 0, n)
    out, p = [], 0
    for _ in range(k):
        m = rng.randint(lo, hi)
        t = corpus[p:p + m]
        p += m
        if rng.random() < 0.5:
            t = t.rstrip(b"\n") + b"\n"
        out.append(t)
    return out


@pytest.mark.parametrize("ranges", [None, "3"])
def test_chunks_and_ranges(monkeypatch, ranges):
    # 1 MiB chunks: many texts straddle a chunk edge; three ranges on one GPU merge their keys and sum their counters
    monkeypatch.setenv("KREP_B200_CHUNK_MB", "1")
    if ranges:
        monkeypatch.setenv("KREP_B200_RANGES", ranges)
    rng = random.Random(33)
    texts = _corpus_texts(rng, 120, 1, 70000)
    assert sum(map(len, texts)) > 3 << 20
    for pat in ["the[a-z]*", "qzXv[0-9]Kpw", "^the"]:
        check_raw(pat, texts, chunk=1 << 20, big=True)
        for opt in (dict(count=True), dict(), dict(max_count=2)):
            P = _params(pat, **opt)
            assert lib.regex_search_batch(P, texts) == [lib.search("regex", P, t) for t in texts], (pat, opt)


def test_overflow_restage_zeroes_counters():
    # a count-mode key list longer than the initial 2^20 keys (one uncertain last line per text): the scan is staged
    # again on a grown list, and the per-text counters must come back zeroed, not doubled
    L = lib.load()
    L.krep_b200_shutdown()
    assert L.krep_b200_init(0) == 0, L.krep_b200_last_error_string()
    texts = [b"a\nb"] * ((1 << 20) + 5000)
    P = _params("a", count=True)
    keys, offs, tl = raw_batch(P, texts, 1, cap=2 << 20)
    assert len(keys) == len(texts)
    assert keys == [(o + 2) << km.LIT_TAG_BITS for o in offs]
    assert set(tl) == {1}
    got = lib.regex_search_batch(P, texts[:3000] + [b"a\na", b"b\nb"])
    assert got[-2:] == [(2, []), (0, [])] and all(g == (1, []) for g in got[:3000])


def test_twenty_thousand_texts():
    rng = random.Random(44)
    texts = _corpus_texts(rng, 20000, 0, 600)
    for opt in (dict(count=True), dict(), dict(count=True, only_matching=True)):
        P = _params("the[a-z]*", **opt)
        got = lib.regex_search_batch(P, texts)
        assert got == [lib.search("regex", P, t) for t in texts], opt
    P = _params("the[a-z]*", count=True)
    keys, offs, tl = raw_batch(P, texts, 1, cap=1 << 20)
    b = bm.Batch(texts)
    want, per = b.expect(1, km.HookLines(P, b.buf))
    assert keys == want
    assert tl == [per.get(i, 0) for i in range(len(texts))]


def test_refused_pattern():
    L = lib.load()
    P = _params("ab\\sab")
    texts = [b"ab ab\n", b"", b"xx"]
    _keep, tarr, larr = lib.text_array(texts)
    counts = (C.c_uint64 * 3)(7, 7, 7)
    assert L.krep_b200_regex_search_batch(P.ref(), tarr, larr, 3, counts, None) == -3
    assert L.krep_b200_last_error() == -3
    assert list(counts) == [0, 0, 0]


def test_early_returns_launch_nothing():
    L = lib.load()
    texts = [b"", b"", b""]
    P = _params("^$", count=True)
    before = L.krep_b200_launch_count()
    assert lib.regex_search_batch(P, texts) == [(1, [])] * 3
    P = _params("^$")
    assert lib.regex_search_batch(P, texts) == [(1, [(0, 0)])] * 3
    P = _params("a", count=True, max_count=0)
    assert lib.regex_search_batch(P, [b"a\n", b"ba"]) == [(0, [])] * 2
    P = _params("a")
    P.struct.compiled_regex = None
    assert lib.regex_search_batch(P, [b"a\n", b"ba"]) == [(0, [])] * 2
    assert L.krep_b200_launch_count() == before
    # empty texts among others are still answered on the host
    P = _params("^$", count=True)
    assert lib.regex_search_batch(P, [b"", b"a\n\nb", b""]) == [(1, []), (1, []), (1, [])]
