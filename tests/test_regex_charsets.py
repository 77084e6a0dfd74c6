"""-E character sets byte by byte: the set the line automaton reads for each bracket expression, class, literal and
escape, case-sensitive and -i, against glibc's regexec asked about every byte but '\\n'; the fused -c and the device
match walk run on the host on the same atoms; and a grammar fuzz of these atoms with empty groups, zero and stacked
intervals, anchors and word assertions over full-byte text.  No GPU needed."""
import ctypes as C
import random
import string

import pytest

from krep_b200 import lib
from krep_b200.abi import SIZE_MAX, Params
import regex_util as ru
import test_regex_dfa as td

UNBOUNDED = (1 << 64) - 1
PRINTABLE = [chr(c) for c in range(0x20, 0x7F)]
# one line per byte, NUL, control bytes, punctuation and 0x80-0xFF included; every line ends in '\n'
BYTE_LINES = b"".join(bytes([b]) + b"\n" for b in range(256) if b != 10)
BYTE_STARTS = ru.line_starts(BYTE_LINES)
CLASSES = ["alpha", "digit", "alnum", "upper", "lower", "blank", "punct", "print", "graph", "xdigit"]
EDGE_BRACKETS = ["[]a]", "[^]a]", "[a-]", "[-a]", "[]-a]", "[!--]", "[^-]", "[--/]", "[]-]", "[a[]", "[\\]", "[.]",
                 "[*+?{]", "[|()$^]", "[^^]", "[x[:digit:]]", "[[:upper:]_]", "[[:alpha:][:digit:]]", "[a-cx-zA-C0-3]",
                 "[Z-a]", "[0-9A-Fa-f]", "[@-Z_]", "[`-{]", "[+--]", "[ -/:-@[-`{-~]"]
SPECIAL = set(".[\\()*+?{|^$")


def _compiles(pats, **kw):
    if isinstance(pats, str):
        pats = [pats]
    try:
        return Params([p.encode() for p in pats], regex=True, **kw)
    except ValueError:  # glibc refuses it too
        return None


def bracket_ranges():
    """Every range [x-y] and [^x-y] over printable ASCII with x <= y, but y = ']' ([x-]] is the set {x, '-'} and then a
    literal ']') and the matching lists of x = '^' ([^-y] is negated)."""
    pairs = [(x, y) for x in PRINTABLE for y in PRINTABLE if x <= y != "]"]
    return ["[%s-%s]" % (x, y) for x, y in pairs if x != "^"] + ["[^%s-%s]" % (x, y) for x, y in pairs]


def other_atoms():
    out = ["[[:%s:]]" % c for c in CLASSES] + ["[^[:%s:]]" % c for c in CLASSES]
    out += EDGE_BRACKETS + ["[^" + b[1:] for b in EDGE_BRACKETS if not b.startswith("[^")]
    out += [c for c in PRINTABLE if c not in SPECIAL] + ["\\" + c for c in string.punctuation] + [".", "\\w"]
    return out


def byte_set(starts):
    return {BYTE_LINES[s] for s in starts}


def glibc_set(P):
    """The bytes b for which glibc matches the regex P on the one-byte string b."""
    buf = C.create_string_buffer(BYTE_LINES, len(BYTE_LINES) + 1)
    return {BYTE_LINES[s] for s in BYTE_STARTS if P.regex.search(buf, s, s + 1, 0) is not None}


def count_host(P, text, reach=UNBOUNDED):
    buf = C.create_string_buffer(text, len(text) + 1)
    return lib.load().krep_b200_regex_count_host(P.ref(), buf, len(text), reach)


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


class AtomCheck:
    """Runs check() on many atoms and keeps every disagreement, by kind, so that one failure shows them all."""

    def __init__(self, icase):
        self.icase = icase
        self.n = dict(checked=0, exact=0, refused=0, device_paths=0)
        self.bad = dict(unsound=[], inexact=[], icase_bracket=[], device_paths=[])

    def check(self, atom):
        """^atom$ on every byte: glibc's set within the automaton's, equal to it unless the plan is widened; then the
        device paths the bare atom's plan admits, on the same lines, against the reference loop."""
        P = _compiles("^%s$" % atom, case_sensitive=not self.icase)
        if P is None:
            return
        got = ru.filter_host(P, BYTE_LINES)
        if got is None:
            self.n["refused"] += 1
            return
        flagged, widened = got
        want, have = glibc_set(P), byte_set(flagged)
        self.n["checked"] += 1
        if not want <= have:
            self.bad["unsound"].append((atom, bytes(sorted(want - have))))
        if not widened:
            self.n["exact"] += 1
            if have != want:
                self.bad["inexact"].append((atom, bytes(sorted(have ^ want))))
        elif self.icase and atom.startswith("[") and have != want:
            # an -i bracket expression reads glibc's own bytes; its plan is still marked widened when the parsed set is
            # not closed under case
            self.bad["icase_bracket"].append((atom, bytes(sorted(have ^ want))))
        L = lib.load()
        for kw in (dict(count=True), dict(), dict(max_count=3)):
            Pk = _compiles(atom, case_sensitive=not self.icase, **kw)
            if kw.get("count"):
                if L.krep_b200_regex_count_mode(Pk.ref()) != 1:
                    continue
                ok = count_host(Pk, BYTE_LINES) == ru.ref_regex_search(Pk, BYTE_LINES)[0]
            else:
                if L.krep_b200_regex_match_mode(Pk.ref()) != 1:
                    continue
                ok = matches_host(Pk, BYTE_LINES) == ru.ref_regex_search(Pk, BYTE_LINES)
            self.n["device_paths"] += 1
            if not ok:
                self.bad["device_paths"].append((atom, kw))

    def assert_clean(self):
        bad = {k: (len(v), v[:4]) for k, v in self.bad.items() if v}
        assert not bad, (self.icase, bad)


@pytest.mark.parametrize("icase", [False, True], ids=["case", "icase"])
def test_every_range_byte_by_byte(icase):
    a = AtomCheck(icase)
    for atom in bracket_ranges():
        a.check(atom)
    a.assert_clean()
    assert a.n["checked"] > 7800 and a.n["exact"] > (8700 if not icase else 1400), a.n
    assert a.n["device_paths"] > (26000 if not icase else 4400), a.n


@pytest.mark.parametrize("icase", [False, True], ids=["case", "icase"])
def test_classes_edges_literals_and_escapes(icase):
    a = AtomCheck(icase)
    for atom in other_atoms():
        a.check(atom)
    a.assert_clean()
    assert a.n["checked"] > 170 and a.n["exact"] > 150 and a.n["device_paths"] > 450, a.n


@pytest.mark.parametrize("pat,text,want", [
    # glibc folds the text's bytes under -i, not the range: [A-z] holds letters only, [a-|] and [z-{] hold [\]^_`
    ("[A-z]", b"_\n[\nab\n`\na_b\n\\\n", 2),
    ("a[A-z]b", b"a_b\na`b\naZb\n", 1),
    ("[a-|]", b"_\n`\n{\n}\n", 3),
    ("[z-{]", b"Z\n[\n^\nY\ny\n", 3),
    ("[#-Z]", b"_\nq\n#\n", 2),
])
def test_icase_ranges_follow_glibc(pat, text, want):
    P = _compiles(pat, case_sensitive=False, count=True)
    assert ru.ref_regex_search(P, text)[0] == want
    flagged, _ = ru.filter_host(P, text)
    assert set(td._glibc_lines(P, text, any_start=True)) <= set(flagged)
    if lib.load().krep_b200_regex_count_mode(P.ref()) == 1:
        assert count_host(P, text) == want


def test_icase_range_glibc_refuses():
    # [Z-a] is a range without -i; under -i glibc folds it to [Z-A] and refuses it
    assert _compiles("[Z-a]") is not None
    assert _compiles("[Z-a]", case_sensitive=False) is None


# ---- grammar fuzz ----------------------------------------------------------------------------------------------------

FUZZ_RANGES = ["[A-z]", "[a-|]", "[z-{]", "[#-Z]", "[2-z]", "[c-~]", "[Z-a]", "[^A-z]", "[^a-|]", "[_-a]", "[[-`]",
               "[a-c]", "[A-C]", "[0-9]", "[!-/]", "[ -~]"]
SUFFIXES = ["", "", "", "", "*", "+", "?", "{0}", "{0,0}", "{,2}", "{2}{2}", "*+", "+?", "{1,2}", "{2,}"]
# a group inside a group repeats at most once: glibc's regexec takes seconds on nested repeats of groups that match empty
NESTED_GROUP_SUFFIXES = ["", "", "?", "{0}", "{0,0}"]
ASSERTIONS = ["^", "$", "\\b", "\\B", "\\<", "\\>"]
FUZZ_BYTES = bytes([0, 13, 0x80, 0xC1, 0xDF, 0xE9, 0xFF]) + b"[\\]^_`{|}~" + b"aAbBcCzZ09#-./!"


def fuzz_atom(rng, atoms):
    return rng.choice(FUZZ_RANGES) if rng.random() < 0.4 else rng.choice(atoms)


def fuzz_regex(rng, atoms, depth=0):
    parts = []
    for _ in range(rng.randint(1, 3)):
        r = rng.random()
        if r < 0.1:
            parts.append(rng.choice(ASSERTIONS))
            continue
        if r < 0.22 and depth < 2:
            alts = [fuzz_regex(rng, atoms, depth + 1) for _ in range(rng.randint(1, 3))]
            if rng.random() < 0.2:
                alts.append("")
            group = "(" + "|".join(alts) + ")"
        elif r < 0.27:
            group = rng.choice(["()", "(|a)"])
        else:
            parts.append(fuzz_atom(rng, atoms) + rng.choice(SUFFIXES))
            continue
        parts.append(group + rng.choice(SUFFIXES if depth == 0 else NESTED_GROUP_SUFFIXES))
    return "".join(parts)


def fuzz_text(rng, n):
    """Bytes around the set edges, any byte now and then, and newlines."""
    out = bytearray()
    for _ in range(n):
        r = rng.random()
        out.append(10 if r < 0.12 else rng.randrange(256) if r < 0.25 else rng.choice(FUZZ_BYTES))
    return bytes(out)


def test_grammar_fuzz():
    rng = random.Random(0xC5E7)
    atoms = other_atoms()
    n = dict(filter=0, exact=0, count=0, matches=0)
    L = lib.load()
    for _ in range(3000):
        pats = [fuzz_regex(rng, atoms) for _ in range(rng.choice([1, 1, 1, 2]))]
        icase = rng.random() < 0.5
        P = _compiles(pats, case_sensitive=not icase)
        if P is None:
            continue
        text = fuzz_text(rng, rng.randint(0, 120))
        got = ru.filter_host(P, text)
        if got is None:
            continue
        flagged, widened = got
        assert set(td._glibc_lines(P, text, any_start=True)) <= set(flagged), (pats, icase, text)
        n["filter"] += 1
        if not widened:
            assert flagged == td._glibc_lines(P, text, any_start=False), (pats, icase, text)
            n["exact"] += 1
        mc = rng.choice([SIZE_MAX, SIZE_MAX, 1, 2, 5])
        Pc = _compiles(pats, case_sensitive=not icase, count=True, max_count=mc)
        if L.krep_b200_regex_count_mode(Pc.ref()) == 1:
            want = ru.ref_regex_search(Pc, text)[0]
            for reach in (3, UNBOUNDED):
                assert count_host(Pc, text, reach) == want, (pats, icase, mc, reach, text)
            n["count"] += 1
        Pm = _compiles(pats, case_sensitive=not icase, max_count=mc)
        if L.krep_b200_regex_match_mode(Pm.ref()) == 1:
            want = ru.ref_regex_search(Pm, text)
            for reach in (3, UNBOUNDED):
                assert matches_host(Pm, text, reach) == want, (pats, icase, mc, reach, text)
            n["matches"] += 1
    assert n["filter"] > 2500 and n["exact"] > 1500 and n["count"] > 1500 and n["matches"] > 1400, n
