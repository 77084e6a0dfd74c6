"""-E on resident shards: krep_b200_search_shards on regex plans must return what krep_b200_regex_search returns on the
same bytes (and the reference loop over glibc), for any tiling and halo, in all three paths; and the rows the pack
kernels build must equal host slicing of the shard byte for byte."""
import ctypes as C
import random

import pytest

from krep_b200 import lib
from krep_b200.abi import ALGO_REGEX, Params, Shard
import regex_kernel_model as km
import regex_rows_util as rr
import regex_util as ru

pytestmark = pytest.mark.gpu
HALOS = [0, 17, km.REGEX_HALO]


@pytest.fixture(scope="module", autouse=True)
def _init():
    L = lib.load()
    assert L.krep_b200_init(0) == 0, L.krep_b200_last_error_string()


@pytest.fixture(autouse=True)
def _device_paths_on(monkeypatch):
    monkeypatch.delenv("KREP_B200_NO_FUSED_COUNT", raising=False)
    monkeypatch.delenv("KREP_B200_NO_DEVICE_MATCHES", raising=False)


def _params(pat, **kw):
    return Params([pat.encode() if isinstance(pat, str) else pat], regex=True, **kw)


class Resident:
    """Shards (regex_kernel_model.Shard) copied to the device, and their krep_b200_shard_t."""

    def __init__(self, shards, device=0):
        import torch
        import gpu_util as gu
        with torch.cuda.device(device):
            self.bufs = [gu.to_device(sh.buf) for sh in shards]
        self.model = shards
        self.structs = [Shard(b.data_ptr(), sh.avail, sh.own_begin, sh.own_end, sh.global_offset, sh.prev_byte, sh.next_byte)
                        for b, sh in zip(self.bufs, shards)]


def _plan(P):
    L = lib.load()
    h = L.krep_b200_plan_create(P.ref(), ALGO_REGEX)
    lib.check(L)
    assert h
    return h


def shards_answer(P, res):
    L = lib.load()
    h = _plan(P)
    try:
        lib.load().krep_b200_set_only_matching(bool(P.only_matching))
        return lib.search_shards(h, P, res.structs)
    finally:
        L.krep_b200_set_only_matching(False)
        L.krep_b200_plan_destroy(h)


def check(P, text, cuts, halo, ref=True, what=""):
    if ru.filter_host(P, text) is None:
        return
    got = shards_answer(P, Resident(rr.tile(text, cuts, halo)))
    want = lib.search("regex", P, text)
    assert got == want, (what, P.patterns, len(cuts), halo, got[0], want[0], got[1][:4], want[1][:4])
    if ref:
        r = ru.ref_regex_search(P, text)
        assert got == (r[0], r[1] if P.struct.track_positions else []), what


def _cuts(rng, n, k):
    return sorted(rng.sample(range(1, n), k - 1)) if n > k else []


def test_random_regexes():
    rng = random.Random(11)
    done = 0
    while done < 40:
        pat = ru.random_regex(rng)
        case = rng.choice(ru.CASES)
        try:
            P = _params(pat, **case)
        except ValueError:
            continue
        text = km.random_lines_text(rng, rng.randint(1, 20000))
        check(P, text, _cuts(rng, len(text), rng.choice([1, 2, 3, 7])), rng.choice(HALOS), what=(pat, case))
        done += 1


@pytest.mark.parametrize("pat", ["the[a-z]*", "^a", "b$", "x*", "^$", "\\bthe"])
@pytest.mark.parametrize("case", [dict(), dict(count=True), dict(count=True, only_matching=True), dict(only_matching=True),
                                  dict(whole_word=True), dict(case_sensitive=False), dict(max_count=1), dict(max_count=3),
                                  dict(max_count=7), dict(count=True, max_count=2)])
def test_patterns_modes(pat, case):
    rng = random.Random(5)
    text = km.random_lines_text(rng, 30000).replace(b"x", b"the", 200)
    P = _params(pat, **case)
    for k in (1, 3, 7):
        check(P, text, _cuts(rng, len(text), k), rng.choice(HALOS), what=k)


@pytest.mark.parametrize("knob", ["KREP_B200_NO_FUSED_COUNT", "KREP_B200_NO_DEVICE_MATCHES"])
def test_knobs_force_filter(monkeypatch, knob):
    monkeypatch.setenv(knob, "1")
    rng = random.Random(3)
    text = km.random_lines_text(rng, 20000)
    for pat in ["the[a-z]*", "a+b", "^$"]:
        for case in [dict(), dict(count=True), dict(max_count=2)]:
            check(_params(pat, **case), text, _cuts(rng, len(text), 3), 17, what=(knob, pat, case))


def test_corpus_slice():
    spec = lib.make_spec(0x5EED0001, 0x5EED0002, 1 << 16, b"qzXv9Kpw")
    text = lib.corpus_host(spec, 0, 2 << 20)
    rng = random.Random(1)
    for pat, case in [("the[a-z]*", dict(count=True)), ("the[a-z]*", dict()), ("the[a-z]*", dict(whole_word=True)),
                      ("\\bthe", dict(count=True)), ("qz[A-Z]v", dict())]:
        for k, halo in [(1, 0), (4, km.REGEX_HALO), (7, 17)]:
            check(_params(pat, **case), text, _cuts(rng, len(text), k), halo, ref=False, what=(pat, case, k, halo))


def test_long_lines_across_cuts():
    """1 MiB lines cut by several shards, halos shorter than the lines."""
    rng = random.Random(2)
    big = bytes(rng.choice(b"abcx ") for _ in range(1 << 20))
    text = b"the a\n" + big + b" the\n" + b"xx\n" + big + b"the"
    cuts = [3, 1000, 300000, 700000, (1 << 20) + 20, (1 << 20) + 500000]
    for pat, case in [("the", dict()), ("the$", dict()), ("x*", dict(count=True)), ("a[bc]", dict(max_count=3)),
                      ("the", dict(whole_word=True))]:
        for halo in HALOS:
            check(_params(pat, **case), text, cuts, halo, ref=False, what=(pat, case, halo))


def test_key_lists_above_one_cta_finish():
    """More listed lines than the one-CTA finish sorts (16 384): the radix-sorted list feeds the pack."""
    text = b"".join(b"the %d\nab\n" % i for i in range(30000))
    for case in [dict(), dict(count=True), dict(whole_word=True)]:
        for k in (1, 3):
            check(_params("the [0-9]*", **case), text, _cuts(random.Random(k), len(text), k), 17, ref=False, what=case)


def test_two_devices():
    L = lib.load()
    if L.krep_b200_device_count() < 2:
        pytest.skip("needs two GPUs")
    rng = random.Random(9)
    text = km.random_lines_text(rng, 40000)
    shards = rr.tile(text, _cuts(rng, len(text), 4), 100)
    res = [Resident([sh], device=i % 2) for i, sh in enumerate(shards)]
    merged = Resident.__new__(Resident)
    merged.structs = [r.structs[0] for r in res]
    for pat, case in [("the[a-z]*", dict()), ("a+b", dict(count=True)), ("b$", dict(whole_word=True))]:
        P = _params(pat, **case)
        assert shards_answer(P, merged) == lib.search("regex", P, text)


def test_geometry_errors():
    L = lib.load()
    text = b"the a\nthe b\nthe c\n" * 10
    P = _params("the")
    h = _plan(P)
    try:
        good = Resident(rr.tile(text, [40, 100], 8))
        assert lib.search_shards(h, P, good.structs) == lib.search("regex", P, text)
        s = good.structs

        def bad(structs):
            arr = (Shard * len(structs))(*structs)
            cnt = L.krep_b200_search_shards(h, P.ref(), arr, len(structs), None)
            assert cnt == 0 and L.krep_b200_last_error() == -3

        bad(s[1:])                 # does not start at 0
        bad([s[0], s[2]])          # a gap
        bad(s[:2])                 # does not end the text
        s0 = Shard.from_buffer_copy(s[0])
        s0.prev_byte = 10
        bad([s0, s[1], s[2]])      # the first shard claims a byte before it
        s2 = Shard.from_buffer_copy(s[2])
        s2.own_end = s2.avail_len - 1
        bad([s[0], s[1], s2])      # the last shard does not own its last byte
        bad([])
    finally:
        L.krep_b200_plan_destroy(h)


def export(h, P, st):
    L = lib.load()
    nb = C.c_uint64(0)
    drow = C.c_void_p()
    assert L.krep_b200_regex_export_shard(h, P.ref(), C.byref(st), None, None, 0, C.byref(nb), C.byref(drow)) == 0
    buf = C.create_string_buffer(nb.value)
    assert L.krep_b200_regex_export_shard(h, P.ref(), C.byref(st), None, buf, nb.value, C.byref(nb), None) == 0
    small = C.create_string_buffer(16)
    assert L.krep_b200_regex_export_shard(h, P.ref(), C.byref(st), None, small, 16, C.byref(nb), None) == -5
    L.krep_b200_last_error()
    return buf.raw


def pack_text(rng):
    """Empty lines, lines of 1..16 bytes, lines over 64 KiB, in random order."""
    parts = []
    for _ in range(400):
        r = rng.random()
        if r < 0.2:
            parts.append(b"\n")
        elif r < 0.97:
            parts.append(bytes(rng.choice(b"abxt ") for _ in range(rng.randint(1, 16))) + b"\n")
        else:
            parts.append(bytes(rng.choice(b"abxt ") for _ in range(rng.randint(65537, 70000))) + b"\n")
    return b"".join(parts)


@pytest.mark.parametrize("seed", range(6))
def test_pack_rows_equal_host_slicing(seed):
    """The device row (keys from the device's own scan) equals the host twin built from the same keys: header, segment
    table, head and packed bytes, for lines of every kind, unaligned starts, and segments that end at avail_len."""
    rng = random.Random(seed)
    text = pack_text(rng)
    if seed % 2:
        text = text.rstrip(b"\n")
    pats = [("a", dict()), ("a|x", dict(count=True)), ("^$", dict()), ("t", dict(whole_word=True)), ("b*", dict()),
            ("^a|b$", dict(count=True))]
    pat, case = pats[seed]
    P = _params(pat, **case)
    h = _plan(P)
    try:
        cuts = sorted(rng.sample(range(1, len(text)), 3))
        halo = [0, 17, 200, km.REGEX_HALO][seed % 4]
        shards = rr.tile(text, cuts, halo)
        res = Resident(shards)
        rows = []
        for sh, st in zip(shards, res.structs):
            row = export(h, P, st)
            d = rr.parse_row(row)
            assert d["magic"] == rr.MAGIC and d["mode"] == rr.call_mode(P) and d["row_bytes"] == len(row)
            want = rr.build_row(sh, d["mode"], d["keys"], d["device_lines"])
            if row != want:
                w = rr.parse_row(want)
                for f in ("nseg", "head_len", "flags", "own_begin", "own_end", "avail_end"):
                    assert d[f] == w[f], (f, d[f], w[f])
                for a, b in zip(d["segs"], w["segs"]):
                    assert a[:3] == b[:3], (a[:3], b[:3])
                    assert a[3] == b[3], a[:3]
                assert d["head"] == w["head"]
                assert row == want
            rows.append(row)
        want = lib.search("regex", P, text)
        assert lib.regex_resolve(P, rows) == want
    finally:
        lib.load().krep_b200_plan_destroy(h)
