"""The -E long-line pass on batches (scan_regex_long.cu in batch mode, DESIGN §12.5 and §12.8):
krep_b200_regex_search_batch_long_raw against tests/regex_batch_long_model.py exactly, keys and per-text counts, in
every mode the pattern admits and at several slice and checkpoint sizes; and krep_b200_regex_search_batch against
krep_b200_regex_search and the reference loop on long-line texts, on all three paths, with and without
KREP_B200_NO_LONG_LINES."""
import ctypes as C
import random

import numpy as np
import pytest

from krep_b200 import lib
from krep_b200.abi import Params
import regex_batch_long_model as blm
import regex_kernel_model as km
import regex_util as ru
from test_gpu_regex_sets import err_patterns, set_text

pytestmark = pytest.mark.gpu
NO_POS = (1 << 64) - 1
SIZES = [(4096, 256), (64, 16), (16, 4)]
R = km.REGEX_SEG + km.REGEX_HALO
LENS = (4096, 4097, 4352, 4353, 8191, 8192, 8193, 12287, 12288, 12289)
ALPHABET = b"abcxy ,Q"
# patterns whose enumeration provably stays within the step budget on these texts (as in test_gpu_regex_long.py)
BUDGET_FREE = {"the[a-z]*", "b|a+", "c a"}
KNOBS = [{}, {"KREP_B200_NO_FUSED_COUNT": "1"}, {"KREP_B200_NO_DEVICE_MATCHES": "1"},
         {"KREP_B200_NO_FUSED_COUNT": "1", "KREP_B200_NO_DEVICE_MATCHES": "1"}]


@pytest.fixture(scope="module", autouse=True)
def _init():
    L = lib.load()
    assert L.krep_b200_init(0) == 0, L.krep_b200_last_error_string()


@pytest.fixture(autouse=True)
def _device_paths_on(monkeypatch):
    for k in ("KREP_B200_NO_FUSED_COUNT", "KREP_B200_NO_DEVICE_MATCHES", "KREP_B200_NO_LONG_LINES"):
        monkeypatch.delenv(k, raising=False)


def _params(pats, **kw):
    pats = [pats] if isinstance(pats, str) else pats
    return Params([p.encode() for p in pats], regex=True, **kw)


def modes_of(P, Pc):
    L = lib.load()
    return [0] + ([1] if L.krep_b200_regex_count_mode(Pc.ref()) == 1 else []) + \
        ([2] if L.krep_b200_regex_match_mode(P.ref()) == 1 else [])


def raw(P, texts, mode, sizes=(0, 0), long=True, cap=1 << 16):
    """One batch scan through the long hook (or the pass-free hook with long=False).
    -> (sorted keys, packed offsets, per-text device lines); retried with room for every key."""
    L = lib.load()
    n = len(texts)
    _keep, tarr, larr = lib.text_array(texts)
    offs = (C.c_uint64 * max(n, 1))()
    tl = (C.c_uint64 * max(n, 1))()
    while True:
        keys = np.zeros(max(cap, 1), dtype=np.uint64)
        kp = keys.ctypes.data_as(C.POINTER(C.c_uint64))
        if long:
            k = L.krep_b200_regex_search_batch_long_raw(P.ref(), tarr, larr, n, mode, sizes[0], sizes[1], offs, kp, cap, tl)
        else:
            k = L.krep_b200_regex_search_batch_raw(P.ref(), tarr, larr, n, mode, offs, kp, cap, tl)
        assert k >= 0, (k, L.krep_b200_last_error_string())
        if k <= cap:
            return keys[:k].tolist(), list(offs[:n]), list(tl[:n])
        cap = k


def check_model(pats, texts, chunk=None, sizes_list=SIZES, big=False, budget_free=False, **kw):
    """Long hook vs model in every mode the pattern admits. -> the LongBatch model"""
    P, Pc = _params(pats, **kw), _params(pats, count=True, **kw)
    b = blm.LongBatch(texts, chunk)
    modes = modes_of(P, Pc)
    flagged = km.HookLines(P, b.buf).flagged
    oracle = km.HookLines(P, b.buf, P if 2 in modes else None) if big else km.GlibcLines(P, b.buf)
    for mode in modes:
        exp = b.expect(mode, flagged if mode == 0 else oracle, budget_free)
        for sizes in sizes_list:
            keys, offs, tl = raw(P, texts, mode, sizes)
            assert offs == [NO_POS if o is None else o for o in b.offs], (pats, mode)
            blm.check(b, exp, keys, tl, (pats, mode, sizes, chunk))
    return b


def _line(rng, n):
    b = bytes(rng.choice(ALPHABET) for _ in range(n))
    if rng.random() < 0.3 and n >= 2:
        b = b"x" + b[1:-1] + b"y"
    return b


def edge_texts(rng):
    """Long lines of the edge lengths between short ones, and the texts whose ends the pass must leave alone."""
    out = []
    for _ in range(6):
        parts = []
        for _ in range(rng.randint(2, 5)):
            parts.append(_line(rng, rng.choice(LENS)) + b"\n")
            parts.append(ru.random_text(rng, rng.randint(1, 200)))
        out.append(b"".join(parts))
    L = rng.choice(LENS)
    out += [
        _line(rng, 5000) + b"\n" + _line(rng, L),               # a long last line without its '\n'
        _line(rng, 5000) + b"\n" + _line(rng, L) + b"\n",       # ... with it
        _line(rng, 9000) + b"\nab c\n",                          # a long line, then a short last line
        b"q\n" + _line(rng, 4400) + b"\n",                      # a long line whose '\n' is the text's last byte
        b"", b"a", b"\n", b"",                                   # one-byte and empty texts between long ones
        _line(rng, 8192) + b"\nx",
        b"z",
        _line(rng, R) + b"\n" + _line(rng, R + 1) + b"\n" + _line(rng, R - 1) + b"\nb",
    ]
    rng.shuffle(out)
    return out


PATTERNS = ["a[^x]*b", "(ab)*c", "^x.*y$", ".*QQ|,", "the[a-z]*", "b|a+", "c a", "x$"]


@pytest.mark.parametrize("pat", PATTERNS)
def test_hook_against_model(pat):
    rng = random.Random(sum(pat.encode()))
    b = check_model(pat, edge_texts(rng), budget_free=pat in BUDGET_FREE)
    assert b.taken, pat
    # the last line of every text stays uncertain
    lasts = {b.offs[i] + ru.line_starts(b.texts[i])[-1] for i in b.live}
    assert not lasts & {p for _, p, _ in b.taken}


def test_icase_and_many_texts_share_one_work_list():
    # 300 texts in one chunk, each with long lines and a short last line: the counts go to the right text
    rng = random.Random(5)
    texts = []
    for i in range(300):
        t = b"".join(_line(rng, rng.choice(LENS)) + b"\n" + ru.random_text(rng, rng.randint(0, 40)).replace(b"\n", b" ") + b"\n"
                     for _ in range(rng.randint(1, 3)))
        texts.append(t + b"ab" if i % 3 else t)
    b = check_model("a[^x]*B", texts, sizes_list=[(0, 0)], case_sensitive=False)
    # a line of 4352 bytes or more is out of reach wherever it starts; it is taken unless it is its text's last line
    def far(t):
        lines = t.split(b"\n")[:-1] if t.endswith(b"\n") else t.split(b"\n")
        return any(len(x) >= R for x in lines[:-1])
    with_long = {i for i, t in enumerate(texts) if far(t)}
    assert len(with_long) > 250 and with_long <= {i for i, _, _ in b.taken}
    check_model("c a", texts, sizes_list=[(64, 16)], budget_free=True)


@pytest.mark.parametrize("ranges", [None, "3"])
def test_chunks_and_ranges(monkeypatch, ranges):
    # 1 MiB chunks: texts and long lines across chunk edges (cut lines stay uncertain); three ranges on one GPU
    monkeypatch.setenv("KREP_B200_CHUNK_MB", "1")
    if ranges:
        monkeypatch.setenv("KREP_B200_RANGES", ranges)
    rng = random.Random(33)
    texts = []
    while sum(map(len, texts)) < (3 << 20) + 500000:
        parts = [_line(rng, rng.choice(LENS + (30000, 70000))) + b"\n" + ru.random_text(rng, rng.randint(1, 300))
                 for _ in range(rng.randint(1, 8))]
        texts.append(b"".join(parts))
    for pat in ("the[a-z]*", "a[^x]*b"):
        b = check_model(pat, texts, chunk=1 << 20, sizes_list=[(0, 0)], big=True)
        cut = [p for _, p, nl, _ in b.lines if nl is None and b.buf.find(b"\n", p) >= (p >> 20 << 20) + (1 << 20) + km.REGEX_HALO]
        assert cut and b.taken and not set(cut) & {p for _, p, _ in b.taken}
        for opt in (dict(count=True), dict(), dict(max_count=2)):
            P = _params(pat, **opt)
            assert lib.regex_search_batch(P, texts) == [lib.search("regex", P, t) for t in texts], (pat, opt)


def test_split_plan_of_three_automata():
    rng = random.Random(0x5E7)
    pats = err_patterns(rng, 90)
    P = _params(pats)
    assert lib.load().krep_b200_regex_automata(P.ref()) == 3
    words = [b"ERR" + p[3:6].encode() + b"qwer77 code=ab" for p in pats]
    texts = []
    for _ in range(12):
        parts = [set_text(rng, words, rng.choice(LENS)).replace(b"\n", b" ") + b"\n" + set_text(rng, words, rng.randint(1, 300))
                 for _ in range(rng.randint(1, 3))]
        texts.append(b"".join(parts))
    b = check_model(pats, texts, sizes_list=[(0, 0), (16, 4)], budget_free=True)
    assert b.taken
    for kw in (dict(), dict(count=True), dict(max_count=2)):
        P = _params(pats, **kw)
        assert lib.regex_search_batch(P, texts) == [lib.search("regex", P, t) for t in texts], kw


def test_count_overflow_restage_does_not_double(monkeypatch):
    # more uncertain keys than a fresh list holds: the first staging overflows in a later chunk and is redone on a grown
    # list; the lines the pass counted in the first chunks are counted once
    monkeypatch.setenv("KREP_B200_CHUNK_MB", "1")
    L = lib.load()
    L.krep_b200_shutdown()
    assert L.krep_b200_init(0) == 0, L.krep_b200_last_error_string()
    long = b"ab " * 1500
    texts = [long + b"\na\nb"] * 300 + [b"a\nb"] * ((1 << 20) + 100)
    P = _params("a", count=True)
    keys, offs, tl = raw(P, texts, 1, cap=2 << 20)
    assert len(keys) == len(texts)
    assert tl == [2] * 300 + [1] * ((1 << 20) + 100)
    got = lib.regex_search_batch(P, texts[:300] + texts[-3:])
    assert all(c == 2 for c, _ in got[:300]) and all(c == 1 for c, _ in got[300:])


def test_refused_sizes():
    L = lib.load()
    P = _params("a")
    _keep, tarr, larr = lib.text_array([b"a\n"])
    for s, c in ((1 << 21, 1), (16, 32), (4096, 1)):
        assert L.krep_b200_regex_search_batch_long_raw(P.ref(), tarr, larr, 1, 0, s, c, None, None, 0, None) == -3
        assert L.krep_b200_last_error() == -3


def test_knob_equals_pass_free_hook(monkeypatch):
    rng = random.Random(9)
    texts = edge_texts(rng)
    P, Pc = _params("a[^x]*b"), _params("a[^x]*b", count=True)
    on = {m: raw(P, texts, m) for m in modes_of(P, Pc)}
    monkeypatch.setenv("KREP_B200_NO_LONG_LINES", "1")
    for m in on:
        assert raw(P, texts, m) == raw(P, texts, m, long=False), m
    monkeypatch.delenv("KREP_B200_NO_LONG_LINES")
    assert all(raw(P, texts, m) == on[m] for m in on)
    assert any(len(on[m][0]) < len(raw(P, texts, m, long=False)[0]) for m in on)


OPTIONS = [dict(), dict(case_sensitive=False), dict(whole_word=True), dict(count=True), dict(count=True, only_matching=True),
           dict(max_count=1), dict(max_count=2), dict(max_count=3)]


@pytest.mark.parametrize("no_long", [False, True])
def test_answers(monkeypatch, no_long):
    rng = random.Random(17)
    texts = edge_texts(rng)
    if no_long:
        monkeypatch.setenv("KREP_B200_NO_LONG_LINES", "1")
    for pat in ("the[a-z]*", "a[^x]*b", "c a|x$"):
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
                assert got == want, (pat, opt, knobs, [i for i in range(len(texts)) if got[i] != want[i]][:4])
                if knobs in ({}, KNOBS[3]):
                    assert got == [lib.search("regex", P, t) for t in texts], (pat, opt, knobs)
