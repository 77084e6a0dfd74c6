"""krep_b200_regex_resolve on rows built on the host (tests/regex_rows_util.py, the twin of krep_b200_regex_export_shard)
must give krep_b200_regex_search's answer — the reference loop over glibc, and the library's host procedures for the
fused -c and the device offsets — for any tiling of the text and any halo."""
import random

import pytest

from krep_b200 import lib
from krep_b200.abi import SIZE_MAX, Params
import regex_kernel_model as km
import regex_rows_util as rr
import regex_util as ru


def _params(pat, **kw):
    return Params([pat.encode() if isinstance(pat, str) else pat], regex=True, **kw)


def _host_procedure(P, text):
    """krep_b200_regex_search's own host procedure where the library has one (fused -c, device offsets), else None."""
    L = lib.load()
    import ctypes as C
    buf = C.create_string_buffer(text, len(text) + 1)
    if L.krep_b200_regex_count_mode(P.ref()) == 1:
        return L.krep_b200_regex_count_host(P.ref(), buf, len(text), SIZE_MAX), None
    if L.krep_b200_regex_match_mode(P.ref()) == 1:
        res = L.krep_b200_match_result_init(16)
        try:
            n = L.krep_b200_regex_matches_host(P.ref(), buf, len(text), SIZE_MAX, res)
            r = res.contents
            return n, [(r.positions[i].start_offset, r.positions[i].end_offset) for i in range(r.count)]
        finally:
            L.krep_b200_match_result_free(res)
    return None


def resolve(P, text, cuts, halo):
    rows = [rr.twin_row(P, sh) for sh in rr.tile(text, cuts, halo)]
    return lib.regex_resolve(P, rows)


def check(P, text, cuts, halo, what=""):
    if ru.filter_host(P, text) is None:
        return
    got = resolve(P, text, cuts, halo)
    want = ru.ref_regex_search(P, text)
    if not P.struct.track_positions:
        want = (want[0], [])
    assert got == want, (what, P.patterns, cuts, halo, got[0], want[0], got[1][:5], want[1][:5])
    hp = _host_procedure(P, text)
    if hp is not None:
        assert got[0] == hp[0], (what, got[0], hp[0])
        if hp[1] is not None:
            assert got[1] == hp[1], what


HALOS = [0, 17, km.REGEX_HALO]


def _cuts(rng, text, k):
    n = len(text)
    if n < 2 or k <= 1:
        return []
    return sorted(rng.sample(range(1, n), min(k - 1, n - 1)))


def test_random_regexes_tilings():
    rng = random.Random(7)
    done = 0
    while done < 60:
        pat = ru.random_regex(rng)
        case = rng.choice(ru.CASES)
        try:
            P = _params(pat, **case)
        except ValueError:
            continue
        if ru.filter_host(P, b"") is None:
            continue
        text = ru.random_text(rng, rng.randint(0, 700))
        if rng.random() < 0.5:
            text = text.rstrip(b"\n") + b"\n"
        k = rng.choice([1, 2, 3, 7])
        check(P, text, _cuts(rng, text, k), rng.choice(HALOS), what=(pat, case))
        done += 1


@pytest.mark.parametrize("pat", ["the[a-z]*", "b$", "^a", "x*", "a+b", "^$", "(ab|ba)c?"])
@pytest.mark.parametrize("case", [dict(), dict(count=True), dict(count=True, only_matching=True), dict(only_matching=True),
                                  dict(whole_word=True), dict(case_sensitive=False), dict(max_count=1), dict(max_count=2),
                                  dict(max_count=3), dict(max_count=7), dict(count=True, max_count=3)])
def test_patterns_modes(pat, case):
    rng = random.Random(hash((pat, tuple(sorted(case.items())))) & 0xFFFF)
    text = km.random_lines_text(rng, 12000)
    P = _params(pat, **case)
    for k in (1, 2, 3, 7):
        for halo in HALOS:
            check(P, text, _cuts(rng, text, k), halo, what=(k, halo))


def test_cut_kinds():
    """Cuts at a line start, mid-line, on a '\\n', and three inside one long line (it spans four shards)."""
    line = b"ab " * 2000 + b"the end\n"
    text = b"the a\nxx the\n" + line + b"b\n\nthe\nab"
    ls = text.index(line)
    cuts = [6, 9, 12, ls + 100, ls + 2500, ls + 4000, len(text) - 3]
    for pat in ["the[a-z]*", "end$", "^ab", "b$", "^$", "a"]:
        for case in [dict(), dict(count=True), dict(whole_word=True), dict(case_sensitive=False), dict(max_count=2)]:
            for halo in HALOS:
                check(_params(pat, **case), text, cuts, halo, what=(pat, case, halo))


@pytest.mark.parametrize("tail", [b"", b"\n", b"\n\n", b"x", b"X\n"])
def test_end_of_text(tail):
    """The empty string at n and '$' under -i (REG_NOTEOL) at the text's end, whatever the last shard holds."""
    rng = random.Random(len(tail))
    text = b"ab\nxx\n\nthe x\n" * 50 + tail
    for pat, case in [("^$", dict()), ("^$", dict(count=True)), ("x$", dict(case_sensitive=False)),
                      ("x$", dict(case_sensitive=False, count=True)), ("$", dict()), ("^", dict(count=True)), ("x*", dict())]:
        P = _params(pat, **case)
        for k in (1, 2, 3, 7):
            for halo in HALOS:
                check(P, text, _cuts(rng, text, k), halo, what=(pat, case, k, halo))


def test_empty_text():
    for pat in ["^$", "a", "x*"]:
        for case in [dict(), dict(count=True)]:
            P = _params(pat, **case)
            got = lib.regex_resolve(P, [rr.twin_row(P, km.Shard(b""))])
            want = ru.ref_regex_search(P, b"")
            assert got[0] == want[0], (pat, case)


def test_bad_tilings_refused():
    L = lib.load()
    text = b"the a\nthe b\nthe c\n"
    P = _params("the")
    rows = [rr.twin_row(P, sh) for sh in rr.tile(text, [6, 12], 4)]
    assert lib.regex_resolve(P, rows) == ru.ref_regex_search(P, text)
    for bad in (rows[1:], [rows[0], rows[2]], rows[:2], [rows[1], rows[0], rows[2]]):
        with pytest.raises(RuntimeError):
            lib.regex_resolve(P, bad)
    L.krep_b200_last_error()
