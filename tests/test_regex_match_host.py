"""-E offsets on the host: krep_b200_regex_matches_host (the line automaton decides the lines it can within a walk bound,
the match automaton enumerates the matches of each line decided MATCHED within the scan's step budget, regexec takes the
rest) against the reference's regex_search loop, the end-of-text quirks, and which calls krep_b200_regex_match_mode
sends to the device.  No GPU needed."""
import ctypes as C
import random

import pytest

from krep_b200 import lib
from krep_b200.abi import Params
import oracle_util as ou
import regex_util as ru

UNBOUNDED = (1 << 64) - 1
REACHES = [1, 3, 16, UNBOUNDED]
# positions, -co, -i, and -m limits
OPTS = [dict(), dict(count=True, only_matching=True), dict(case_sensitive=False), dict(max_count=1), dict(max_count=2),
        dict(max_count=3), dict(max_count=7), dict(count=True, only_matching=True, max_count=2)]

# the longest alternative matters, empty loops, anchors in alternations, and a pattern that runs over the step budget
EXTRA_PATTERNS = ["a|ab|abc", "(a|ab)(c|bcd)", "abc|ab|a", "(a|ab)(bc|c)?", "(a*)*", "(|a)+", "a{,2}", "x{0}", "x{0}y",
                  "(a*)+b", "(a|b*)*c", "((a|)*)*", "(a{0,2}){2}", "a*", "x*", "$", "^", "^$", "b|$", "^|a", "a$|b",
                  "(^a|b)", "(a|^)b", "a($|c)", "[^a]*$", "^.*$", ".", "[a-c]*d", "the[a-z]*", "[tT]h[a-z]*", "a.c"]


def _params(pats, **kw):
    if isinstance(pats, str):
        pats = [pats]
    return Params([p.encode() for p in pats], regex=True, **kw)


def _compiles(pats, **kw):
    try:
        return _params(pats, **kw)
    except ValueError:  # glibc refuses it too
        return None


def match_mode(P):
    return lib.load().krep_b200_regex_match_mode(P.ref())


def matches_host(P, text, reach=UNBOUNDED):
    L = lib.load()
    buf = C.create_string_buffer(text, len(text) + 1)
    res = L.krep_b200_match_result_init(16)
    try:
        cnt = L.krep_b200_regex_matches_host(P.ref(), buf, len(text), reach, res)
        r = res.contents
        return cnt, [(r.positions[i].start_offset, r.positions[i].end_offset) for i in range(r.count)]
    finally:
        L.krep_b200_match_result_free(res)


WIDE = bytes(range(0x80, 0x100, 7)) + b"\x00\t\r\n\n\n aAbBcCxX09_.,;:!?-()[]{}\\/'\"$^*+|thTHe"


def wide_text(rng, n):
    return bytes(rng.choice(WIDE) for _ in range(n))


def _texts(rng):
    yield b"\n"
    yield b"x\n\n"
    for _ in range(2):
        yield wide_text(rng, rng.randint(1, 70))
    t = ru.random_text(rng, rng.randint(1, 70))
    yield t
    yield t + b"\n"


def test_matches_host_equals_reference_loop():
    rng = random.Random(0x0FF5)
    pats = EXTRA_PATTERNS + [ru.random_regex(rng) for _ in range(220)]
    checked = 0
    modes = {0: 0, 1: 0, -1: 0}
    for i, pat in enumerate(pats):
        for kw in OPTS:
            P = _compiles(pat, **kw)
            if P is None:
                continue
            mode = match_mode(P)
            modes[mode] += 1
            if mode != 1:
                continue
            for text in _texts(rng):
                want = ru.ref_regex_search(P, text)
                for reach in REACHES:
                    assert matches_host(P, text, reach) == want, (pat, kw, reach, text)
                    checked += 1
    print(f"eligible cases checked: {checked} (calls by mode: {modes})")
    assert checked > 25000 and modes[1] > 1000, (checked, modes)


def test_empty_match_after_a_match():
    P = _params("a*")
    for text, want in [(b"aab", [(0, 2), (2, 2)]), (b"aab\n", [(0, 2), (2, 2), (3, 3)]),
                       (b"aab\nb\n", [(0, 2), (2, 2), (3, 3), (4, 4), (5, 5)])]:
        assert ru.ref_regex_search(P, text) == (len(want), want)
        for reach in REACHES:
            assert matches_host(P, text, reach) == (len(want), want), (text, reach)


@pytest.mark.parametrize("pat", ["$", "x*", "^", "^$", "a|ab|abc", "(a|ab)(c|bcd)"])
@pytest.mark.parametrize("text", [b"ab\nabcd\n", b"ab\nabcd\n\n", b"ab\n\nabcd", b"\n", b"\n\n", b"x"])
def test_end_of_text(pat, text):
    for kw in (dict(), dict(case_sensitive=False), dict(max_count=2)):
        P = _params(pat, **kw)
        assert match_mode(P) == 1
        want = ru.ref_regex_search(P, text)
        for reach in REACHES:
            assert matches_host(P, text, reach) == want, (kw, reach)


def test_icase_end_of_text():
    # -i passes REG_ICASE as an execution flag: its value is REG_NOTEOL, so '$' does not match at the end of the text
    P = _params("x$", case_sensitive=False)
    assert match_mode(P) == 1
    for text, want in [(b"ax\nbx", [(1, 2)]), (b"ax\nbx\n", [(1, 2), (4, 5)])]:
        assert ru.ref_regex_search(P, text) == (len(want), want)
        for reach in REACHES:
            assert matches_host(P, text, reach) == (len(want), want), (text, reach)


def test_step_budget():
    # [a-c]*d on long a-c runs: the enumeration is quadratic, so the lines run over their budget and go to regexec
    rng = random.Random(3)
    run = bytes(rng.choice(b"abc") for _ in range(3000))
    text = b"xd abd\n" + run + b"\n" + run + b"d\n" + b"cd\n" + run[:500] + b"\nz"
    for kw in (dict(), dict(max_count=3), dict(count=True, only_matching=True)):
        P = _params("[a-c]*d", **kw)
        assert match_mode(P) == 1
        want = ru.ref_regex_search(P, text)
        for reach in REACHES:
            assert matches_host(P, text, reach) == want, (kw, reach)


def test_early_returns():
    P = _params("a*")
    assert matches_host(P, b"") == ru.ref_regex_search(P, b"") == (1, [(0, 0)])
    P = _params("a", max_count=0)
    assert matches_host(P, b"a\n") == (0, [])
    P = _params("a")
    P.struct.compiled_regex = None
    assert matches_host(P, b"a\n") == (0, [])


@pytest.mark.parametrize("kw", [dict(), dict(only_matching=True), dict(count=True, only_matching=True),
                                dict(case_sensitive=False), dict(max_count=3)])
def test_match_mode_device(kw):
    for pat in ("the(x|y)*", "a|ab|abc", "x*", "^$"):
        assert match_mode(_params(pat, **kw)) == 1


@pytest.mark.parametrize("pat,kw", [
    ("abc", dict(whole_word=True)),                                # -w
    ("\\bab", dict()),                                             # a word assertion widens the automaton
    ("[a-c]+_[0-9]", dict(case_sensitive=False)),                  # an -i bracket widened by case folding
    ("(^a)*", dict()),                                             # an anchor inside a repeated group
    ("abc", dict(count=True)),                                     # -c is counted, not enumerated
])
def test_match_mode_regexec(pat, kw):
    P = _params(pat, **kw)
    assert match_mode(P) == 0
    assert matches_host(P, b"abc\n")[0] == -1


def test_match_mode_refused():
    P = _params("\\s")
    assert match_mode(P) == -1
    assert matches_host(P, b"a b\n")[0] == -1


def test_no_device_matches_knob(monkeypatch):
    P = _params("the[a-z]*")
    monkeypatch.setenv("KREP_B200_NO_DEVICE_MATCHES", "1")
    assert match_mode(P) == 0
    # the host procedure itself does not depend on the knob
    assert matches_host(P, b"the\nxthey\n") == (2, [(0, 3), (5, 9)])


def test_matches_host_equals_compiled_reference():
    chk = ou.reference()
    if chk is None:
        pytest.skip("compiled reference not available")
    f = chk.lib.regex_search
    f.argtypes = ou._SIG
    f.restype = C.c_uint64
    rng = random.Random(17)
    n = 0
    for i, pat in enumerate(EXTRA_PATTERNS + [ru.random_regex(rng) for _ in range(60)]):
        for kw in (dict(max_count=2), dict(case_sensitive=i % 2 == 0), dict(count=True, only_matching=True)):
            P = _compiles(pat, **kw)
            if P is None or match_mode(P) != 1:
                continue
            for text in _texts(rng):
                res = chk._new(16)
                try:
                    cnt = f(P.ref(), C.create_string_buffer(text, len(text) + 1).raw, len(text), res)
                    r = res.contents
                    want = (int(cnt), [(r.positions[i].start_offset, r.positions[i].end_offset) for i in range(r.count)])
                finally:
                    chk._free(res)
                for reach in (3, UNBOUNDED):
                    assert matches_host(P, text, reach) == want, (pat, kw, reach, text)
                n += 1
    assert n > 400, n
