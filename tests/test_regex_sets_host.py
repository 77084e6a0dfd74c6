"""Split -E plans on the host (DESIGN §12.7): which alternations become split plans, which stay single automata or
refused, and the host twins of the split scan (krep_b200_regex_filter_host / _count_host / _matches_host for
production plans, krep_b200_regex_plan_host for plans split by a lowered state cap) against the reference's
regex_search loop over glibc.  No GPU needed."""
import ctypes as C
import random
import string

import pytest

from krep_b200 import lib
from krep_b200.abi import Params
import oracle_util as ou
import regex_kernel_model as km
import regex_util as ru

UNBOUNDED = (1 << 64) - 1
REACHES = [1, 3, 16, UNBOUNDED]


def _params(pats, **kw):
    if isinstance(pats, str):
        pats = [pats]
    return Params([p.encode() for p in pats], regex=True, **kw)


def automata(P):
    return lib.load().krep_b200_regex_automata(P.ref())


def lower_words(rng, k, lo=8, hi=12):
    return ["".join(rng.choice(string.ascii_lowercase) for _ in range(rng.randint(lo, hi))) for _ in range(k)]


def alnum_words(rng, k):
    return ["".join(rng.choice(string.ascii_letters + string.digits) for _ in range(rng.randint(6, 10))) for _ in range(k)]


def err_patterns(rng, k):
    return ["ERR%s[a-z]{4}[0-9]+ code=[a-z]+" % "".join(rng.choice(string.ascii_lowercase) for _ in range(3))
            for _ in range(k)]


def xk(k):
    """k x's then y, written as x{255} blocks and a remainder: one automaton of about k states."""
    return "x{255}" * (k // 255) + ("x{%d}" % (k % 255) if k % 255 else "") + "y"


# ---- which plans split ----------------------------------------------------------------------------------------------

@pytest.mark.parametrize("name,make", [
    ("80 lowercase literals", lambda rng: lower_words(rng, 80)),
    ("60 ERR patterns", lambda rng: err_patterns(rng, 60)),
    ("40 alphanumeric literals", lambda rng: alnum_words(rng, 40)),
    ("200 lowercase literals", lambda rng: lower_words(rng, 200)),
    ("200 alphanumeric literals", lambda rng: alnum_words(rng, 200)),
])
def test_refused_sets_now_split(name, make):
    pats = make(random.Random(name))
    L = lib.load()
    P = _params(pats)
    g = automata(P)
    assert 2 <= g <= 8, (name, g)
    assert L.krep_b200_select_search_algorithm(P.ref()) == C.cast(L.krep_b200_regex_search, C.c_void_p).value
    assert L.krep_b200_regex_count_mode(_params(pats, count=True).ref()) == 1
    # one pattern with a top-level alternation splits the same way
    assert automata(_params("|".join("(%s)" % p for p in pats))) == g


def test_image_budget_decides_offsets():
    rng = random.Random(7)
    low = lower_words(rng, 200)
    assert automata(_params(low + ["the[a-z]*"])) >= 2
    assert lib.load().krep_b200_regex_match_mode(_params(low + ["the[a-z]*"]).ref()) == 1  # match tables fit
    aln = alnum_words(rng, 200)
    assert lib.load().krep_b200_regex_match_mode(_params(aln).ref()) == 0  # only the line tables fit
    assert lib.load().krep_b200_regex_count_mode(_params(aln, count=True).ref()) == 1


@pytest.mark.parametrize("pats,match_mode,name", [
    (["the[a-z]*"], 1, "regex-lines"), (["a|ab|abc"], 1, "regex-lines"), (["ab", "x[0-9]", "^c"], 1, "regex-lines"),
    ([xk(3000)], 1, "regex-lines"), (["\\bab", "cd"], 0, "regex-lines-widened"),
    # the largest sets one automaton holds: their match tables do not fit next to the line table
    (lower_words(random.Random(1), 60), 0, "regex-lines"), (alnum_words(random.Random(2), 30), 0, "regex-lines"),
])
def test_plans_that_compile_stay_single(pats, match_mode, name):
    L = lib.load()
    P = _params(pats)
    assert automata(P) == 1
    # the filter name and the modes these plans had before split plans existed
    assert L.krep_b200_regex_count_mode(_params(pats, count=True).ref()) == (0 if name.endswith("widened") else 1)
    assert L.krep_b200_regex_match_mode(P.ref()) == match_mode
    sp = SplitPlan(P, 4096)  # the production compile, uncached (its name needs no device)
    try:
        assert sp.name == name
    finally:
        sp.close()


@pytest.mark.parametrize("name,pats", [
    ("a \\s branch", lower_words(random.Random(3), 80) + ["a\\sb"]),
    ("a \\S branch", lower_words(random.Random(3), 80) + ["a\\Sb"]),
    ("one branch over the limit", lower_words(random.Random(4), 10) + [xk(8000)]),
    ("one pattern over the limit", [xk(8000)]),
    ("[ab]*a[ab]{14}", ["[ab]*a[ab]{14}"]),
    ("500 lowercase literals", lower_words(random.Random(5), 500)),
])
def test_still_refused(name, pats):
    L = lib.load()
    P = _params(pats)
    assert automata(P) == -1, name
    assert ru.filter_host(P, b"abc\n") is None
    assert L.krep_b200_select_search_algorithm(P.ref()) is None


# ---- texts ------------------------------------------------------------------------------------------------------------

WIDE = bytes(range(0x80, 0x100, 7)) + b"\x00\t\r\n\n\n aAbBcCxX09_.,;:!?-()[]{}\\/'\"$^*+|"


def set_text(rng, pats, n, words=()):
    """Lines mixing whole words of the set, their prefixes and case variants, and bytes NUL, '\\r', 0x80-0xFF."""
    out = bytearray()
    while len(out) < n:
        r = rng.random()
        if words and r < 0.3:
            w = rng.choice(words)
            out += w[: rng.randint(1, len(w))] if rng.random() < 0.3 else w
            if rng.random() < 0.2:
                out += bytes(rng.choice(WIDE) for _ in range(rng.randint(0, 3)))
        elif words and r < 0.4:
            out += rng.choice(words).upper()
        elif r < 0.6:
            out += bytes(rng.choice(WIDE) for _ in range(rng.randint(1, 6)))
        else:
            out += ru.random_text(rng, rng.randint(1, 12))
        out += rng.choice([b" ", b"", b"\n", b"\r\n", b"\n\n"])
    return bytes(out[:n])


def _count_host(P, text, reach):
    buf = C.create_string_buffer(text, len(text) + 1)
    return lib.load().krep_b200_regex_count_host(P.ref(), buf, len(text), reach)


def _matches_host(P, text, reach):
    L = lib.load()
    buf = C.create_string_buffer(text, len(text) + 1)
    res = L.krep_b200_match_result_init(16)
    try:
        cnt = L.krep_b200_regex_matches_host(P.ref(), buf, len(text), reach, res)
        r = res.contents
        return cnt, [(r.positions[i].start_offset, r.positions[i].end_offset) for i in range(r.count)]
    finally:
        L.krep_b200_match_result_free(res)


def _lines_glibc(P, text):
    """The line starts of the lines glibc matches in (the last one ends at the end of the text)."""
    buf = C.create_string_buffer(text, len(text) + 1)
    out = []
    for p in ru.line_starts(text):
        nl = text.find(b"\n", p)
        end = len(text) if nl < 0 else nl + 1
        if P.regex.search(buf, p, end, km._eflags(P)) is not None:
            out.append(p)
    return out


# positions, -c, -co, -i, -w and -m limits
OPTS = [dict(), dict(count=True), dict(count=True, only_matching=True), dict(case_sensitive=False),
        dict(case_sensitive=False, count=True), dict(whole_word=True), dict(whole_word=True, count=True),
        dict(max_count=1), dict(max_count=2), dict(max_count=3), dict(max_count=7), dict(count=True, max_count=2)]


def _check_production(pats, text, kw, paths):
    P = _params(pats, **kw)
    want = ru.ref_regex_search(P, text)
    got = _lines_glibc(P, text)
    flt = ru.filter_host(P, text)
    assert flt is not None
    flagged, widened = flt
    assert set(got) <= set(flagged), (kw, sorted(set(got) - set(flagged))[:5])
    if not widened:
        assert flagged == got, kw
    if _count_host(P, text, UNBOUNDED) >= 0:
        paths["count"] += 1
        for reach in REACHES:
            assert _count_host(P, text, reach) == want[0], (kw, reach)
    if _matches_host(P, text, UNBOUNDED)[0] >= 0:
        paths["match"] += 1
        for reach in REACHES:
            assert _matches_host(P, text, reach) == want, (kw, reach)


def _production_sets():
    rng = random.Random(0x5E75)
    low = lower_words(rng, 90)
    errs = err_patterns(rng, 60)
    edge = ["^ab", "yz$", "(ka|kab)(c|bcd)", "qk|qkj|qkjv", "A_"]
    return [
        ("lowercase", low + ["the[a-z]*"], [w.encode() for w in low] + [b"the", b"thee", b"theX"]),
        ("ERR", errs, [b"ERR" + p[3:6].encode() + b"abcd12 code=zz" for p in errs]),
        ("edge branches", low[:40] + edge + low[40:], [w.encode() for w in low] + [b"abcd", b"kabcd", b"qkjv", b"yz", b"A_"]),
    ]


@pytest.mark.parametrize("name,pats,words", _production_sets())
def test_production_split_sets_equal_reference(name, pats, words):
    assert automata(_params(pats)) >= 2, name
    rng = random.Random(name)
    paths = {"count": 0, "match": 0}
    for n in (1, 40, 900, 3000):
        text = set_text(rng, pats, n, words)
        for t in (text, text.rstrip(b"\n") + b"\n"):
            for kw in OPTS:
                _check_production(pats, t, kw, paths)
    assert paths["count"] and paths["match"], paths


def test_production_split_equals_compiled_reference():
    chk = ou.reference()
    if chk is None:
        pytest.skip("compiled reference not available")
    f = chk.lib.regex_search
    f.argtypes = ou._SIG
    f.restype = C.c_uint64
    n = 0
    for name, pats, words in _production_sets():
        rng = random.Random(name + "ref")
        for kw in (dict(), dict(count=True), dict(max_count=3), dict(case_sensitive=False), dict(count=True, only_matching=True)):
            P = _params(pats, **kw)
            for size in (50, 2000):
                text = set_text(rng, pats, size, words)
                res = chk._new(16)
                try:
                    cnt = f(P.ref(), C.create_string_buffer(text, len(text) + 1).raw, len(text), res)
                    r = res.contents
                    want = (int(cnt), [(r.positions[i].start_offset, r.positions[i].end_offset) for i in range(r.count)])
                finally:
                    chk._free(res)
                assert ru.ref_regex_search(P, text) == want
                if _count_host(P, text, 3) >= 0:
                    assert _count_host(P, text, 3) == want[0]
                    n += 1
                if _matches_host(P, text, 3)[0] >= 0:
                    assert _matches_host(P, text, 3) == want
                    n += 1
    assert n > 10, n


# ---- plans split by a lowered state cap -------------------------------------------------------------------------------

class SplitPlan:
    """krep_b200_regex_plan_split of params under a state cap; None when refused under it."""

    def __init__(self, P, cap):
        L = lib.load()
        self.P = P
        self.h = L.krep_b200_regex_plan_split(P.ref(), cap)
        L.krep_b200_last_error()
        self.name = L.krep_b200_plan_filter_name(self.h).decode() if self.h else None

    def close(self):
        if self.h:
            lib.load().krep_b200_plan_destroy(self.h)

    def host(self, mode, text, reach=UNBOUNDED):
        """-> (keys, device_lines), or None when the plan does not admit the mode."""
        L = lib.load()
        buf = C.create_string_buffer(text, len(text) + 1)
        cap = len(text) * 2 + 8
        keys = (C.c_uint64 * cap)()
        dl = C.c_uint64(0)
        k = L.krep_b200_regex_plan_host(self.h, mode, buf, len(text), reach, keys, cap, C.byref(dl))
        if k < 0:
            L.krep_b200_last_error()
            return None
        assert k <= cap
        return list(keys[:k]), dl.value


def forced_splits(rng, n_sets, caps=(4, 6, 8, 12, 20)):
    """(branches, case flag, SplitPlan) for random sets of ru.random_regex branches that split under some cap."""
    out = []
    while len(out) < n_sets:
        branches = [ru.random_regex(rng) for _ in range(rng.randint(2, 10))]
        icase = rng.random() < 0.25
        try:
            P = _params(branches, case_sensitive=not icase)
        except ValueError:
            continue
        for cap in rng.sample(caps, len(caps)):
            sp = SplitPlan(P, cap)
            if sp.name and "split" in sp.name:
                out.append((branches, icase, sp))
                break
            sp.close()
    return out


def short_lines_text(rng, n):
    """Lines of at most km.BUDGET_FREE_LEN bytes, so that no line of the match mode reaches its step budget."""
    out = bytearray()
    while len(out) < n:
        line = ru.random_text(rng, rng.randint(0, 12)).replace(b"\n", b"") if rng.random() < 0.7 else \
            bytes(rng.choice(WIDE.replace(b"\n", b"")) for _ in range(rng.randint(0, 12)))
        out += line[: km.BUDGET_FREE_LEN] + b"\n"
    text = bytes(out[:n])
    return text if rng.random() < 0.5 else text.rstrip(b"\n")


def test_forced_splits_equal_reference():
    rng = random.Random(0xF0CE)
    checked = {0: 0, 1: 0, 2: 0}
    names = set()
    for branches, icase, sp in forced_splits(rng, 120):
        names.add(sp.name)
        try:
            Pc = _params(branches, case_sensitive=not icase, count=True)
            for _ in range(3):
                text = short_lines_text(rng, rng.randint(1, 300))
                flagged = [k >> 3 for k in sp.host(0, text)[0]]
                got = _lines_glibc(sp.P, text)
                assert set(got) <= set(flagged), (branches, text)
                if not sp.name.endswith("widened"):
                    assert flagged == got, (branches, text)
                checked[0] += 1
                want_c = ru.ref_regex_search(Pc, text)[0]
                want_p = ru.ref_regex_search(sp.P, text)[1]
                for reach in REACHES:
                    r = sp.host(1, text, reach)
                    if r is not None:
                        assert km.resolve(Pc, text, 0, count_keys=r[0], device_lines=r[1]) == want_c, (branches, reach)
                        checked[1] += 1
                    r = sp.host(2, text, reach)
                    if r is not None:
                        assert km.resolve(sp.P, text, 0, match_keys=r[0]) == want_p, (branches, reach, text)
                        checked[2] += 1
        finally:
            sp.close()
    print(f"forced splits: {checked} ({sorted(names)})")
    assert checked[1] > 300 and checked[2] > 200, checked
    assert {"regex-lines-split", "regex-lines-split-widened"} <= names


# One automaton holds at most about 70 literals of 8-12 lowercase letters (80 are refused, see above): branches with
# 100 such literals between them cannot share a group, whatever the packing.
PAD = lower_words(random.Random(0xA11), 300)


def _spread(*branches):
    """branches with 100 padding literals between each two: every branch in a group of its own."""
    out = [branches[0]]
    for k, b in enumerate(branches[1:]):
        out += PAD[100 * k: 100 * (k + 1)] + [b]
    return out


@pytest.mark.parametrize("branches,texts", [
    (_spread("xa", "xab", "xabc"), [b"xabc\nxab\nxa\nzxabcxab\n", b"xabcxabxa"]),     # the longest end in the last group
    (_spread("xabc", "xab", "xa"), [b"xabc\nxab\nxa\nzxabcxab\n", b"xabcxabxa"]),     # ... and in the first
    (_spread("ab?", "(ab)+c", "b+"), [b"ababc\nbbb\na\nabbabc\n", b"cababcb"]),
    (_spread("^ab", "b$", "abc$"), [b"ab\nba\nabc\nabcab\nxabc", b"\n\nab"]),        # anchors
    (_spread("q", "^q*$", "qq"), [b"\nq\nqq\nqqq\n\nxqq\n", b"qqq"]),                 # a branch matching empty lines
])
def test_longest_end_over_groups(branches, texts):
    # the union's match at a start ends at the longest end of any automaton, whichever group holds that branch
    P = _params(branches)
    assert automata(P) >= len(branches) // 100 + 1, automata(P)
    assert lib.load().krep_b200_regex_match_mode(P.ref()) == 1  # offsets on the device's path
    for kw in (dict(), dict(count=True, only_matching=True), dict(max_count=2)):
        P = _params(branches, **kw)
        for text in texts:
            want = ru.ref_regex_search(P, text)
            assert want[0] > 0
            for reach in REACHES:
                assert _matches_host(P, text, reach) == want, (kw, text, reach)


def test_large_match_table_in_a_group():
    # q[gh]*g[gh]{13}: a line table that fits, a match automaton of more than 65536 entries.  Entries are 16-bit row
    # offsets, so such a table cannot be used: the offsets go to regexec.  With {12} the table fits and they stay.
    big = "(" + "|".join(["zzzzzzzz"] * 500) + ")"  # 4000 NFA states each: the whole alternation is too large
    rng = random.Random(13)
    texts = [b"qgghghghhhggghhgghhhghhggghg x\nq\n"] + [bytes(rng.choice(b"qgh x\n") for _ in range(rng.randint(1, 90)))
                                                      for _ in range(150)]
    for rep, device in ((13, 0), (12, 1)):
        pats = [big, big, "q", "q[gh]*g[gh]{%d}" % rep]
        P = _params(pats)
        assert automata(P) == 2
        assert lib.load().krep_b200_regex_match_mode(P.ref()) == device, rep
        Pc = _params(pats, count=True)
        for text in texts:
            want = ru.ref_regex_search(P, text)
            for reach in (3, UNBOUNDED):
                if device:
                    assert _matches_host(P, text, reach) == want, (rep, text)
                assert _count_host(Pc, text, reach) == ru.ref_regex_search(Pc, text)[0], (rep, text)
        # a plan split under a lower cap keeps the same rule for its match tables
        sp = SplitPlan(P, 4096)
        try:
            r = sp.host(2, texts[0])
            assert (r is not None) == bool(device)
            if r is not None:
                assert km.resolve(P, texts[0], 0, match_keys=r[0]) == ru.ref_regex_search(P, texts[0])[1]
        finally:
            sp.close()


def test_split_plan_hook_arguments():
    L = lib.load()
    P = _params(["ab", "cd"])
    assert not L.krep_b200_regex_plan_split(P.ref(), 2)
    assert L.krep_b200_last_error() == -3
    assert not L.krep_b200_regex_plan_split(P.ref(), 5000)
    L.krep_b200_last_error()
    sp = SplitPlan(_params(["ab\\b", "cd"]), 4096)  # one automaton, widened by the word assertion
    try:
        assert sp.name == "regex-lines-widened"
        assert sp.host(1, b"ab\n") is None and sp.host(2, b"ab\n") is None
        assert sp.host(0, b"ab\nx\ncd\n") == ([0 << 3, 5 << 3], 0)
    finally:
        sp.close()


@pytest.mark.parametrize("pats,cap,admits", [
    (["the[a-z]*"], 4096, {0, 1, 2}),
    (["\\bab", "cd"], 4096, {0}),                                            # widened: the filter only
    (lower_words(random.Random(1), 60), 4096, {0, 1}),                       # no room for the match table
    (lower_words(random.Random(7), 200) + ["the[a-z]*"], 4096, {0, 1, 2}),  # split
    (alnum_words(random.Random(7), 200), 4096, {0, 1}),                      # split, line tables only
    (lower_words(random.Random(3), 80) + ["\\bab"], 4096, {0}),              # split, widened
    (["abc", "xyz", "q[0-9]+"], 6, {0, 1, 2}),                               # split by the lowered cap
    (["ab\\b", "cd", "efg"], 6, {0}),
])
def test_plan_host_refuses_modes_the_plan_lacks(pats, cap, admits):
    # modes outside 0..2, and the count / match modes of plans not exact for them, are refused as a bad argument
    L = lib.load()
    sp = SplitPlan(_params(pats), cap)
    try:
        assert sp.h, pats
        keys = (C.c_uint64 * 8)()
        dl = C.c_uint64(0)
        for mode in (-1, 0, 1, 2, 3):
            k = L.krep_b200_regex_plan_host(sp.h, mode, b"abc the\nxyz q1\n", 15, UNBOUNDED, keys, 8, C.byref(dl))
            err = L.krep_b200_last_error()
            if mode in admits:
                assert k >= 0 and err == 0, (mode, k, err)
            else:
                assert k == -3 and err == -3, (mode, k, err)
    finally:
        sp.close()
