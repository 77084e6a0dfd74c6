"""The fused -E -c on the host: krep_b200_regex_count_host (the line automaton decides the lines it can within a walk
bound, regexec the rest) against the reference's regex_search loop, the two end-of-text quirks, and which calls
krep_b200_regex_count_mode sends to the device.  No GPU needed."""
import ctypes as C
import random

import pytest

from krep_b200 import lib
from krep_b200.abi import SIZE_MAX, Params
import oracle_util as ou
import regex_util as ru

UNBOUNDED = (1 << 64) - 1
REACHES = [1, 3, 16, UNBOUNDED]
MAX_COUNTS = [1, 2, 7, SIZE_MAX]

# nested and empty repeats, and anchors inside alternations
EXTRA_PATTERNS = ["(a*)*", "(|a)+", "x{0}", "a{,2}", "(a*)+b", "(a|b*)*c", "(^a|b)", "(a|^)b", "a|^b", "a$|b", "(a$|b)c",
                  "(^|x)a", "a($|c)", "^(a|b$)", "(^$|a)", "b|$", "^|a", "((a|)*)*", "(a{0,2}){2}", "x{0}y", "x{0}$",
                  "[^a]*$", "^.*$", "^[[:upper:]]+$", "\\.+$", "[a-z]*x", "^$", "x*", "the[a-z]*", "^a.c$"]


def _params(pats, **kw):
    if isinstance(pats, str):
        pats = [pats]
    return Params([p.encode() for p in pats], regex=True, **kw)


def _compiles(pats, **kw):
    try:
        return _params(pats, **kw)
    except ValueError:  # glibc refuses it too
        return None


def count_mode(P):
    return lib.load().krep_b200_regex_count_mode(P.ref())


def count_host(P, text, reach=UNBOUNDED):
    buf = C.create_string_buffer(text, len(text) + 1)
    return lib.load().krep_b200_regex_count_host(P.ref(), buf, len(text), reach)


WIDE = bytes(range(0x80, 0x100, 7)) + b"\x00\t\r\n\n\n aAbBcCxX09_.,;:!?-()[]{}\\/'\"$^*+|thTHe"


def wide_text(rng, n):
    return bytes(rng.choice(WIDE) for _ in range(n))


def _texts(rng):
    yield b"\n"
    yield b"x\n\n"
    for _ in range(3):
        yield wide_text(rng, rng.randint(1, 70))
    t = ru.random_text(rng, rng.randint(1, 70))
    yield t
    yield t + b"\n"


def test_count_host_equals_reference_loop():
    rng = random.Random(0xC0DE)
    pats = EXTRA_PATTERNS + [ru.random_regex(rng) for _ in range(260)]
    checked = 0
    modes = {0: 0, 1: 0, -1: 0}
    for i, pat in enumerate(pats):
        icase = i % 3 == 1
        base = _compiles(pat, count=True, case_sensitive=not icase)
        if base is None:
            continue
        mode = count_mode(base)
        modes[mode] += 1
        if mode != 1:
            continue
        for text in _texts(rng):
            for mc in MAX_COUNTS:
                P = _params(pat, count=True, case_sensitive=not icase, max_count=mc)
                want = ru.ref_regex_search(P, text)[0]
                for reach in REACHES:
                    assert count_host(P, text, reach) == want, (pat, icase, mc, reach, text)
                    checked += 1
    assert checked > 15000 and modes[1] > 150, (checked, modes)


def test_end_of_text_quirks():
    # -i passes REG_ICASE as an execution flag: its value is REG_NOTEOL, so '$' does not match at the end of the text
    P = _params("x$", count=True, case_sensitive=False)
    assert count_mode(P) == 1
    for text, want in [(b"ax\nbx", 1), (b"ax\nbx\n", 2)]:
        assert ru.ref_regex_search(P, text)[0] == want
        for reach in REACHES:
            assert count_host(P, text, reach) == want, (text, reach)
    # the empty string after a final '\n' counts when the last line was not counted
    P = _params("^$", count=True)
    assert count_mode(P) == 1
    for text, want in [(b"b\n", 1), (b"b\n\n", 1), (b"\n", 1), (b"\n\n", 2), (b"b", 0)]:
        assert ru.ref_regex_search(P, text)[0] == want
        for reach in REACHES:
            assert count_host(P, text, reach) == want, (text, reach)


def test_early_returns():
    P = _params("a*", count=True)
    assert count_host(P, b"") == ru.ref_regex_search(P, b"")[0] == 1
    P = _params("a", count=True, max_count=0)
    assert count_host(P, b"a\n") == 0
    P = _params("a", count=True)
    P.struct.compiled_regex = None
    assert count_host(P, b"a\n") == 0


@pytest.mark.parametrize("pat", ["the[a-z]*", "^a.c$", "x*", "^$"])
def test_count_mode_device(pat):
    assert count_mode(_params(pat, count=True)) == 1


@pytest.mark.parametrize("pat,kw", [
    ("abc", dict(count=True, whole_word=True)),                    # -w
    ("\\bab", dict(count=True)),                                   # a word assertion widens the automaton
    ("[a-c]+_[0-9]", dict(count=True, case_sensitive=False)),      # an -i bracket widened by case folding
    ("abc", dict(count=True, only_matching=True)),                 # -co counts matches, not lines
    ("abc", dict()),                                               # positions
])
def test_count_mode_regexec(pat, kw):
    P = _params(pat, **kw)
    assert count_mode(P) == 0
    assert count_host(P, b"abc\n") == -1


def test_count_mode_refused():
    P = _params("\\s", count=True)
    assert count_mode(P) == -1
    assert count_host(P, b"a b\n") == -1


def test_no_fused_count_knob(monkeypatch):
    P = _params("the[a-z]*", count=True)
    monkeypatch.setenv("KREP_B200_NO_FUSED_COUNT", "1")
    assert count_mode(P) == 0
    assert count_host(P, b"the\nxthey\n") == 2  # the host procedure itself does not depend on the knob


def test_count_host_equals_compiled_reference():
    chk = ou.reference()
    if chk is None:
        pytest.skip("compiled reference not available")
    f = chk.lib.regex_search
    f.argtypes = ou._SIG
    f.restype = C.c_uint64
    rng = random.Random(11)
    n = 0
    for i, pat in enumerate(EXTRA_PATTERNS + [ru.random_regex(rng) for _ in range(60)]):
        for mc in (2, SIZE_MAX):
            P = _compiles(pat, count=True, case_sensitive=i % 2 == 0, max_count=mc)
            if P is None or count_mode(P) != 1:
                continue
            for text in _texts(rng):
                res = chk._new(16)
                try:
                    want = int(f(P.ref(), C.create_string_buffer(text, len(text) + 1).raw, len(text), res))
                finally:
                    chk._free(res)
                for reach in (3, UNBOUNDED):
                    assert count_host(P, text, reach) == want, (pat, mc, text)
                n += 1
    assert n > 400, n
