"""-E on the host side: the line automaton against glibc, the refusals, and the clipped regexec loop of
krep_b200_replay(KREP_B200_ALGO_REGEX) against the reference's regex_search loop.  No GPU needed."""
import ctypes as C
import random

import pytest

from krep_b200 import lib
from krep_b200.abi import ALGO_REGEX, REG_NOTBOL, Params
import oracle_util as ou
import regex_util as ru


def _params(pats, **kw):
    if isinstance(pats, str):
        pats = [pats]
    return Params([p.encode() for p in pats], regex=True, **kw)


def _glibc_lines(params, text, any_start):
    """Line starts where glibc finds a match inside the line (from its start; with any_start also from every later
    position with REG_NOTBOL)."""
    rx = params.regex
    buf = C.create_string_buffer(text, len(text) + 1)
    out = []
    for s in ru.line_starts(text):
        e = text.find(b"\n", s)
        e = len(text) if e < 0 else e
        hit = rx.search(buf, s, e, 0) is not None
        k = s + 1
        while any_start and not hit and k <= e:
            hit = rx.search(buf, k, e, REG_NOTBOL) is not None
            k += 1
        if hit:
            out.append(s)
    return out


def _compiles(pat, **kw):
    try:
        return _params(pat, **kw)
    except ValueError:  # glibc refuses it too
        return None


def test_filter_is_sound_and_exact_where_not_widened():
    rng = random.Random(0x5EED)
    checked = exact = 0
    for it in range(2500):
        pats = [ru.random_regex(rng) for _ in range(rng.choice([1, 1, 1, 2]))]
        kw = dict(case_sensitive=rng.random() < 0.7, whole_word=rng.random() < 0.25)
        P = _compiles(pats, **kw)
        if P is None:
            continue
        text = ru.random_text(rng, rng.randint(0, 90))
        got = ru.filter_host(P, text)
        assert got is not None, (pats, kw)
        flagged, widened = got
        want = _glibc_lines(P, text, any_start=True)
        assert set(want) <= set(flagged), (pats, kw, text, want, flagged)
        checked += 1
        if not widened:
            assert flagged == _glibc_lines(P, text, any_start=False), (pats, kw, text, flagged)
            exact += 1
    assert checked > 2000 and exact > 800, (checked, exact)


@pytest.mark.parametrize("pat,kw,widened", [
    ("ab+c", {}, False), ("^a.c$", {}, False), ("(foo|bar)[0-9]{2,3}", {}, False), ("x*", {}, False),
    ("^$", {}, False), ("[a-c]+_[[:digit:]]", {"case_sensitive": False}, True), ("[[:alpha:]]+_[0-9]", {"case_sensitive": False}, False), ("abc", {"case_sensitive": False}, False),
    ("abc", {"whole_word": True}, True), ("\\<a", {}, True),
])
def test_filter_marks_widening(pat, kw, widened):
    P = _params(pat, **kw)
    got = ru.filter_host(P, b"abbc\nfoo123\n\nA_1\n")
    assert got is not None and got[1] == widened


@pytest.mark.parametrize("pat", ["(a)\\1", "a\\`", "b\\'", "\\s", "a\\Wb", "[[:space:]]x", "[[:cntrl:]]", "\\q",
                                 "[ab]*a[ab]{14}", "[[.a.]]", "a\\Sb"])
def test_refused_patterns_stay_on_the_host(pat):
    L = lib.load()
    P = _params(pat)
    assert ru.filter_host(P, b"abc\n") is None
    assert L.krep_b200_select_search_algorithm(P.ref()) is None


def test_selector_takes_accepted_regexes():
    L = lib.load()
    P = _params("qzXv[0-9]+Kpw")
    f = L.krep_b200_select_search_algorithm(P.ref())
    assert f == C.cast(L.krep_b200_regex_search, C.c_void_p).value
    assert b"Regex" in L.krep_b200_get_algorithm_name(f)
    assert ALGO_REGEX == 9


CLIP_PATTERNS = ["^", "$", "^$", "x*", "(a|)b", "\\bab\\b", "\\<a", "\\Bb", "[ab]{2,3}", "a|b$", "^a|b", "b*$", "ab|ba",
                 "(^|x)a", "a($|c)", ".", "a.?b", "\\>", "\\b", "[^a]*"]


def _texts(rng):
    yield b""
    yield b"ab"
    yield b"\n\nab\n\n"
    yield b"cab ab\nab"
    for _ in range(6):
        yield ru.random_text(rng, rng.randint(1, 60))


def test_clipped_loop_equals_reference_loop():
    """Skipping unflagged lines and clipping regexec to runs of flagged lines is the reference loop unchanged."""
    rng = random.Random(42)
    n = 0
    for pat in CLIP_PATTERNS + [ru.random_regex(rng) for _ in range(60)]:
        for kw in ru.CASES:
            P = _compiles(pat, **kw)
            if P is None:
                continue
            for text in _texts(rng):
                want = ru.ref_regex_search(P, text)
                got = ru.filter_host(P, text)
                if got is None:
                    continue
                keys = [s << 3 for s in got[0]]
                assert ru.replay(P, keys, text) == want, (pat, kw, text)
                # every line flagged (the filter may always answer wider) must not change the answer either
                assert ru.replay(P, [s << 3 for s in ru.line_starts(text)], text) == want, (pat, kw, text)
                n += 1
    assert n > 3000, n


def test_max_count_zero_and_missing_regex():
    P = _params("a", max_count=0)
    assert ru.replay(P, [0], b"a\n") == (0, []) == ru.ref_regex_search(P, b"a\n")
    P = _params("a", max_count=0, count=True, only_matching=True)  # -co -m 0: the reference does not return early
    assert ru.replay(P, [0], b"a\n") == ru.ref_regex_search(P, b"a\n")
    P = _params("a")
    P.struct.compiled_regex = None
    assert ru.replay(P, [0], b"a\n") == (0, [])


def test_restatement_matches_compiled_reference():
    chk = ou.reference()
    if chk is None:
        pytest.skip("compiled reference not available")
    f = chk.lib.regex_search
    f.argtypes = ou._SIG
    f.restype = C.c_uint64
    rng = random.Random(7)
    for pat in CLIP_PATTERNS + [ru.random_regex(rng) for _ in range(40)]:
        for kw in ru.CASES:
            P = _compiles(pat, **kw)
            if P is None:
                continue
            for text in _texts(rng):
                res = chk._new(16)
                try:
                    cnt = f(P.ref(), C.create_string_buffer(text, len(text) + 1).raw, len(text), res)
                    r = res.contents
                    got = (int(cnt), [(r.positions[i].start_offset, r.positions[i].end_offset) for i in range(r.count)])
                finally:
                    chk._free(res)
                if not P.struct.track_positions:
                    got = (got[0], [])
                assert got == ru.ref_regex_search(P, text), (pat, kw, text)
