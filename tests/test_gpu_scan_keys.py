"""-m gpu: what the literal and pattern-set scans write, not only what the replay makes of it.

Every case runs krep_b200_scan_shard and reads the exact count and the sorted keys back with krep_b200_export_packed
(and, for -c plans, the line bounds of k_line_bounds), or the record of krep_b200_count_lines_shard, and compares them
with tests/scan_model.py — key by key, word by word.  Each case first asserts the plan's filter name, so the report
shows which kernel it ran: k_lit_aligned4, k_lit_window4 (plain, -i, masked for 1-3 bytes), k_ac_scan at stride 1 and 2,
k_ac_tri4 in its tri and quad forms, k_count_lines, k_line_bounds, and k_finish's rank sort next to CUB's."""
import ctypes as C
import os
import random
import subprocess
import sys
import zlib

import numpy as np
import pytest
import torch

import gpu_util as gu
import scan_model as sm
from krep_b200 import lib
from krep_b200.abi import ALGO_AC, DeviceResult, Params, Shard
from test_replay import ALGO
from test_scan_model import FOLD_ALIASES, FULL_BYTE_ALPHABETS, LineCount

pytestmark = pytest.mark.gpu

PARTNER = {}
for _a, _b in FOLD_ALIASES:
    PARTNER[_a], PARTNER[_b] = _b, _a
# pattern bytes: letters, the word-fold aliases, NUL, high bytes, a high byte whose low bits are '\n'
PAT_BYTES = b"aBz_@`[{\\|^~\x7f\x00 1\x11\xc1\xe1\xe9\xc9\x8a\xff"
CONTEXT = [-1, ord("\n"), ord("a"), ord("_"), 0x00, 0xE9]


@pytest.fixture(scope="module", autouse=True)
def _init():
    L = lib.load()
    assert L.krep_b200_init(0) == 0, L.krep_b200_last_error_string()
    L.krep_b200_count_lines_shard.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(Shard), C.c_void_p, C.POINTER(LineCount)]
    L.krep_b200_count_lines_shard.restype = C.c_int


def rpat(rng, m):
    return bytes(rng.choice(PAT_BYTES) for _ in range(m))


def is_letter(c):
    return c < 128 and chr(c).isalpha()


def partner(rng, c):
    """The byte the 0xDF word fold confuses with c (a letter's other case), else its bit-7 partner."""
    if is_letter(c):
        return c ^ 0x20
    return PARTNER.get(c, c ^ 0x80) if rng.random() < 0.8 else c ^ 0x80


def cased(rng, p, cs):
    """An occurrence of p: p itself, or under -i p with some letters case-flipped."""
    return p if cs else bytes(c ^ 0x20 if is_letter(c) and rng.random() < 0.5 else c for c in p)


def variant(rng, p, cs):
    """An occurrence (cased), or a near miss: one byte swapped for its fold alias or bit-7 partner."""
    if rng.random() < 0.5:
        return cased(rng, p, cs)
    b = bytearray(p)
    i = rng.randrange(len(b))
    b[i] = partner(rng, b[i])
    return bytes(b)


def near_text(rng, pats, cs, n, alphabet):
    out = bytearray()
    live = [p for p in pats if p] or [b"x"]
    while len(out) < n:
        r = rng.random()
        if r < 0.55:
            out += variant(rng, rng.choice(live), cs)
        else:
            out += bytes(rng.choice(alphabet) for _ in range(rng.randint(1, 5)))
    return bytes(out[:n])


class Plan:
    """A plan, the shape the model expects of it, and the check that the library built that kernel."""

    def __init__(self, func, pats, cs=True, ww=False, o=False, count=False):
        L = lib.load()
        self.func, self.pats, self.cs, self.ww, self.o = func, pats, cs, ww, o
        self.P = Params(pats, case_sensitive=cs, whole_word=ww, only_matching=o, count=count)
        self.shape = sm.plan_shape(func, pats, cs, ww, o)
        L.krep_b200_set_only_matching(o)
        try:
            self.h = L.krep_b200_plan_create(self.P.ref(), ALGO[func])
        finally:
            L.krep_b200_set_only_matching(False)
        lib.check(L)
        assert self.h
        self.name = L.krep_b200_plan_filter_name(self.h).decode()
        assert sm.filter_matches(self.name, self.shape, cs), (func, pats, self.name, self.shape)
        self.is_ac = func == "aho_corasick"
        self.bounds = bool(self.P.struct.count_lines_mode)

    def close(self):
        lib.load().krep_b200_plan_destroy(self.h)

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def model(self, buf, avail, ob, oe, go=0, prev=-1, nxt=-1):
        return sm.shard_keys(self.shape, self.pats, self.cs, buf, avail, ob, oe, go, prev, nxt, self.ww)


class _DevWords:
    """A torch view of engine-owned device memory (uint64 words read as int64)."""

    def __init__(self, ptr, n):
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": "<i8", "data": (ptr, False), "version": 2, "strides": None}


def scan(plan, dev, avail, ob, oe, go=0, prev=-1, nxt=-1):
    """-> (count, sorted keys, bounds or None, overflow) of one krep_b200_scan_shard."""
    L = lib.load()
    sh = Shard(dev.data_ptr(), avail, ob, oe, go, prev, nxt)
    out = DeviceResult()
    rc = L.krep_b200_scan_shard(plan.h, C.byref(sh), 1, None, C.byref(out))
    lib.check(L)
    assert rc == 0
    assert out.stored == out.count
    row = torch.empty(out.stored + 1, dtype=torch.int64, device="cuda")
    assert L.krep_b200_export_packed(C.byref(out), row.data_ptr(), out.stored, None) == 0
    row = row.cpu().numpy().view(np.uint64)
    bounds = None
    if out.d_line_bounds and out.stored:
        bounds = torch.as_tensor(_DevWords(out.d_line_bounds, 2 * out.stored), device="cuda").cpu().numpy().view(np.uint64)
    assert plan.bounds == (bounds is not None) or out.stored == 0
    return int(row[0]), row[1:], bounds, out.overflow


def check_scan(plan, dev, buf, avail, ob, oe, go=0, prev=-1, nxt=-1, what=""):
    want = plan.model(buf, avail, ob, oe, go, prev, nxt)
    cnt, keys, bounds, _ = scan(plan, dev, avail, ob, oe, go, prev, nxt)
    ctx = (what, plan.func, plan.pats, plan.cs, plan.ww, plan.o, avail, ob, oe, go, prev, nxt)
    assert cnt == want.size, ctx + (cnt, want.size)
    if not np.array_equal(keys, want):
        k = min(keys.size, want.size)
        diff = np.flatnonzero(keys[:k] != want[:k])
        bad = int(diff[0]) if diff.size else k
        raise AssertionError(ctx + ("first difference at", bad, keys[bad:bad + 4].tolist(), want[bad:bad + 4].tolist()))
    if plan.bounds and want.size:
        wb = sm.line_bounds(want, buf, avail, go, prev, nxt, plan.is_ac)
        assert np.array_equal(bounds, wb), ctx + ("bounds", bounds.tolist()[:16], wb.tolist()[:16])
    return cnt


# (id, func, pattern maker, case_sensitive, whole_word, -o) — the filter each one must reach is plan_shape's
KINDS = [
    ("aligned4", "boyer_moore", lambda r: [rpat(r, 8)], True, False, False),
    ("aligned4-fold", "boyer_moore", lambda r: [rpat(r, 9)], False, False, False),
    ("aligned4-fold-w", "boyer_moore", lambda r: [rpat(r, 11)], False, True, False),
    ("window4-m4", "boyer_moore", lambda r: [rpat(r, 4)], True, False, False),
    ("window4-m5-fold", "boyer_moore", lambda r: [rpat(r, 5)], False, False, False),
    ("window4-m6-w", "boyer_moore", lambda r: [rpat(r, 6)], True, True, False),
    ("masked-m1", "memchr", lambda r: [rpat(r, 1)], True, False, False),
    ("masked-m1-fold", "memchr", lambda r: [b"a"], False, False, False),
    ("masked-m2-fold", "boyer_moore", lambda r: [rpat(r, 2)], False, False, False),
    ("masked-m3-w", "boyer_moore", lambda r: [rpat(r, 3)], True, True, False),
    ("masked-m3-fold", "boyer_moore", lambda r: [b"a" + rpat(r, 2)], False, False, False),
    ("prefix", "memchr_short", lambda r: [rpat(r, 3)], True, False, True),
    ("prefix-fold-w", "memchr_short", lambda r: [rpat(r, 2)], False, True, True),
    ("tag-kmp", "kmp", lambda r: [b"\xe9a\x00\xe9a"], False, True, False),
    ("tag-sse42", "sse42", lambda r: [b"1\x80_1\x80"], True, True, False),
    ("tag-avx2", "avx2", lambda r: [rpat(r, 20)], True, True, False),
    ("ac-stride1", "aho_corasick", lambda r: [rpat(r, 3), rpat(r, 4), rpat(r, 9), b"", rpat(r, 1)], True, False, False),
    ("ac-stride1-fold-w", "aho_corasick", lambda r: [rpat(r, 4), rpat(r, 2), rpat(r, 7)], False, True, False),
    ("ac-stride2", "aho_corasick", lambda r: [rpat(r, 5), rpat(r, 5), rpat(r, 12)], True, False, False),
    ("ac-stride2-fold", "aho_corasick", lambda r: [rpat(r, 5), rpat(r, 8), rpat(r, 30)], False, False, False),
    ("ac-tri4", "aho_corasick", lambda r: [rpat(r, 6), rpat(r, 6), rpat(r, 7), rpat(r, 40)], True, False, False),
    ("ac-tri4-fold-w", "aho_corasick", lambda r: [rpat(r, 6), rpat(r, 10)], False, True, False),
    ("ac-quad", "aho_corasick", lambda r: [rpat(r, 7), rpat(r, 8), rpat(r, 33)], True, False, False),
    ("ac-quad-fold", "aho_corasick", lambda r: [rpat(r, 7), rpat(r, 26), rpat(r, 64)], False, False, False),
]
KIND_IDS = [k[0] for k in KINDS]


def make_plan(kind, seed, count=False):
    _, func, mk, cs, ww, o = kind
    rng = random.Random(seed)
    pats = mk(rng)
    if func == "aho_corasick" and rng.random() < 0.5:
        pats = pats + [pats[0]]  # a duplicate emits its own keys
    return Plan(func, pats if func == "aho_corasick" else pats[:1], cs, ww, o, count), rng


@pytest.mark.parametrize("kind", KINDS, ids=KIND_IDS)
def test_keys_and_bounds_over_every_small_geometry(kind):
    """Every avail_len 0..80; every residue mod 16 of own_begin and own_end with halos of 0, m + 1 and longer, around
    the window kernels' 20-byte rule, the aligned kernel's tail_start = 16 * groups - 3 and the pattern sets' 24-byte
    rule; context bytes from none to word, NUL and high bytes; nonzero global offsets."""
    plan, rng = make_plan(kind, zlib.crc32(kind[0].encode()), count=True)
    with plan:
        m = max(len(p) for p in plan.pats) if plan.is_ac else plan.shape.m
        n = 200 + m
        i = 0
        for ai, alpha in enumerate(FULL_BYTE_ALPHABETS):
            buf = near_text(rng, plan.pats, plan.cs, n, alpha)
            dev = gu.to_device(buf)
            if ai < 3:
                for a in range(0, 81):
                    check_scan(plan, dev, buf, a, 0, a, what="avail")
            # every residue of own_begin with four of own_end per alphabet (a different four each time)
            for rb in range(16):
                for j in range(4):
                    re_ = (5 * rb + 3 * ai + 4 * j) % 16
                    ob, oe = 32 + rb, 64 + re_ + 16 * (ai % 3)
                    halo = (0, m + 1, m + 1 + 7 * ((rb + j) % 5))[(rb + j + ai) % 3]
                    avail = min(oe + halo, n)
                    go = 0 if i % 4 == 0 else (1 << 36) + 16 * i
                    check_scan(plan, dev, buf, avail, ob, oe, go, CONTEXT[i % 6], CONTEXT[(i // 6) % 6], what="residues")
                    i += 1


def test_pattern_set_offset_limit():
    """A pattern-set key holds 40 bits of end offset: a shard ending just below 2^40 scans, one ending at it is
    refused with -3 before any launch."""
    L = lib.load()
    plan, rng = make_plan(KINDS[KIND_IDS.index("ac-tri4")], 5)
    with plan:
        buf = near_text(rng, plan.pats, plan.cs, 300, FULL_BYTE_ALPHABETS[1])
        dev = gu.to_device(buf)
        go = (1 << 40) - 300 - 1
        assert check_scan(plan, dev, buf, 300, 0, 300, go) > 0
        out = DeviceResult()
        sh = Shard(dev.data_ptr(), 300, 0, 300, go + 1, -1, -1)
        assert L.krep_b200_scan_shard(plan.h, C.byref(sh), 1, None, C.byref(out)) == -3
        assert L.krep_b200_last_error() == -3
        assert check_scan(plan, dev, buf, 300, 0, 300, 123) > 0  # the engine scans on after the refusal


def plant_text(rng, plan, n, seed):
    """n bytes of uniform noise with an occurrence (or an alias near miss) planted at -m .. +1 of every 2 KiB
    boundary, and densely in the last 96 bytes (the ragged tile).  The 2 KiB boundaries are the fused count's tiles and
    hold every CTA tile boundary (16 KiB for the literal kernels, 40 KiB for the pattern-set kernels) and so every grid
    stride."""
    t = np.random.default_rng(seed).integers(0, 256, n, dtype=np.uint8)
    live = [p for p in plan.pats if p]
    m = max(len(p) for p in live)
    for j, b in enumerate(range(2048, n - 200, 2048)):
        p = rng.choice(live)
        pos = b + (j % (m + 2)) - m
        v = variant(rng, p, plan.cs) if j % 4 == 3 else cased(rng, p, plan.cs)
        t[pos:pos + len(v)] = np.frombuffer(v, np.uint8)
    pos = n - 96
    while pos + m <= n:
        p = rng.choice(live)
        t[pos:pos + len(p)] = np.frombuffer(p, np.uint8)
        pos += len(p) + rng.randint(0, 2)
    p = live[0]
    t[n - len(p):] = np.frombuffer(p, np.uint8)  # one ends on the last byte
    return t.tobytes()


SCALE = ["aligned4", "aligned4-fold", "window4-m5-fold", "masked-m2-fold", "masked-m1", "prefix", "tag-avx2",
         "ac-stride1", "ac-stride2-fold", "ac-tri4", "ac-quad-fold"]


@pytest.mark.parametrize("kid", SCALE)
def test_keys_at_scale_across_tiles_and_grid_strides(kid):
    """About 24 MiB (more than two grid strides of every kernel) as one shard, then as a shard with an owned range that
    starts and ends off the 16-byte grid."""
    plan, rng = make_plan(KINDS[KIND_IDS.index(kid)], 99)
    with plan:
        n = 24 * (1 << 20) + 777
        buf = plant_text(rng, plan, n, 1234)
        dev = gu.to_device(buf)
        cnt = check_scan(plan, dev, buf, n, 0, n, what="whole")
        assert cnt > 9000, cnt
        check_scan(plan, dev, buf, n - 5, 13, n - 29, 1 << 30, ord("a"), 0xE9, what="inner")
        del dev
        torch.cuda.empty_cache()


@pytest.mark.parametrize("k", [sm.PACK_KEYS - 1, sm.PACK_KEYS, sm.PACK_KEYS + 1])
def test_list_sizes_around_the_rank_sort_limit(k):
    """k_finish rank-sorts up to 16 384 keys, CUB sorts longer lists; both must give the same sorted list (and line
    bounds behind it)."""
    rng = np.random.default_rng(k)
    n = 1 << 20
    t = rng.integers(0, 256, n, dtype=np.uint8)
    t[t == ord("q")] = ord("p")
    t[np.sort(rng.choice(n, k, replace=False))] = ord("q")
    buf = t.tobytes()
    with Plan("memchr", [b"q"], count=True) as plan:
        dev = gu.to_device(buf)
        assert check_scan(plan, dev, buf, n, 0, n) == k
    with Plan("aho_corasick", [b"q"], count=True) as plan:
        assert check_scan(plan, dev, buf, n, 0, n) == k


def _overflow_case():
    """More than the initial 2^20-key list: the scan overflows, grows the list and scans again."""
    L = lib.load()
    assert L.krep_b200_init(0) == 0
    n = 3 * (1 << 20) + 200000
    t = np.full(n, ord("."), dtype=np.uint8)
    t[::3] = ord("q")
    t[1::97] = ord("\n")
    buf = t.tobytes()
    dev = gu.to_device(buf)
    # ~1.10 M keys overflow the initial list (which grows to 2^21), ~2.2 M overflow the grown one; the rescan leaves a
    # complete list (overflow 0: nothing left to call again for)
    for func, pats in (("memchr", [b"q"]), ("aho_corasick", [b"q", b".q"])):
        with Plan(func, pats, count=True) as plan:
            want = plan.model(buf, n, 0, n)
            cnt, keys, bounds, overflow = scan(plan, dev, n, 0, n)
            assert want.size > (1 << 20) and cnt == want.size and overflow == 0, (func, want.size, cnt, overflow)
            assert np.array_equal(keys, want)
            assert np.array_equal(bounds, sm.line_bounds(want, buf, n, 0, -1, -1, plan.is_ac))
    print("overflow ok")


def test_list_overflow_in_a_fresh_process():
    """The grown list stays for the rest of a process, so the overflow is provoked in a process of its own."""
    here = os.path.dirname(os.path.abspath(__file__))
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([here, os.path.dirname(here), os.environ.get("PYTHONPATH", "")]))
    r = subprocess.run([sys.executable, "-c", "import test_gpu_scan_keys as t; t._overflow_case()"], cwd=here, env=env,
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "overflow ok" in r.stdout, r.stdout[-2000:] + r.stderr[-4000:]


def test_pattern_set_edges():
    """16 384 patterns (the index field full) and 16 385 (refused); a 1024-byte pattern; patterns longer than the 24
    text bytes a tri4 queue entry carries that differ only after them; duplicates, empty patterns, and patterns that
    differ only in a fold alias or in bit 7."""
    L = lib.load()
    rng = random.Random(17)
    big = [bytes(rng.choice(PAT_BYTES) for _ in range(8)) for _ in range(sm.AC_MAX_PATTERNS)]
    with Plan("aho_corasick", big) as plan:
        pieces = []
        for k in list(range(0, len(big), 37)) + [len(big) - 1, len(big) - 2]:
            pieces += [big[k], variant(rng, big[k], True), b"\n"]
        buf = b"".join(pieces)
        dev = gu.to_device(buf)
        check_scan(plan, dev, buf, len(buf), 0, len(buf))
        keys = plan.model(buf, len(buf), 0, len(buf))
        assert sm.AC_MAX_PATTERNS - 1 in (keys & np.uint64(0x3FFF)).tolist()  # the last index emits
    p = Params(big + [b"x"])
    assert not L.krep_b200_plan_create(p.ref(), ALGO_AC)
    assert L.krep_b200_last_error() == -3
    long = bytes(rng.choice(PAT_BYTES) for _ in range(1024))
    head = bytes(rng.choice(PAT_BYTES) for _ in range(24))
    sets = [
        ([long, long[:6], long[500:510]], True),
        ([head + b"tail-one", head + b"tail-two", head + b"tail-on\xe5", head[:6]], True),     # differ after byte 24
        ([head + b"Tail-One", head + b"tail-one"], False),
        ([b"ab\x00cd@f", b"AB\x20CD`F", b"ab\x00cd@f", b"", b"ab\x80cd@f"], False),             # fold aliases, bit 7
        ([b"ab[cd", b"ab{cd", b"", b"ab[cd", b"AB[CD\xc1"], False),
        ([b"\xc1\xc9\xde\xc0\xc1\xc9", b"\xe1\xe9\xfe\xe0\xe1\xe9", b"\x11\x12\x13\x14\x15\x16\x17"], False),
    ]
    for pats, cs in sets:
        with Plan("aho_corasick", pats, cs, count=True) as plan:
            pieces = []
            for _ in range(60):
                p = rng.choice([q for q in pats if q])
                pieces += [variant(rng, p, cs), rng.choice([b"", b" ", b"\n", b"_", b"\xe9"])]
            buf = b"".join(pieces)
            dev = gu.to_device(buf)
            for ob, oe, avail in ((0, len(buf), len(buf)), (5, len(buf) - 7, len(buf) - 3), (16, len(buf) // 2, len(buf))):
                check_scan(plan, dev, buf, avail, ob, oe, 64, CONTEXT[ob % 6], CONTEXT[oe % 6])


# ----------------------------------------------------------------------------------------------------- fused -c
FUSED_KINDS = [
    ("aligned4", "boyer_moore", b"\xe9ab_\x00@1x", True, False),
    ("aligned4-fold-w", "boyer_moore", b"@aB[\xc1z`1", False, True),
    ("window4-m5", "sse42", b"aB\x00@z", True, False),
    ("window4-m6-fold", "kmp", b"aB_@\xe9z", False, False),
    ("masked-m2-fold", "boyer_moore", b"a@", False, False),
    ("masked-m2-exact-fold", "boyer_moore", b"aB", False, False),
    ("masked-m3-exact", "memchr_short", b"\x8a\x00a", True, False),
    ("masked-m1", "memchr", b"\xe9", True, False),
    ("masked-m3-w", "boyer_moore", b"a_1", True, True),
]


def count_record(plan, ptr, avail, ob, oe, go=0, prev=-1, nxt=-1):
    L = lib.load()
    sh = Shard(ptr, avail, ob, oe, go, prev, nxt)
    rec = LineCount()
    rc = L.krep_b200_count_lines_shard(plan.h, plan.P.ref(), C.byref(sh), None, C.byref(rec))
    lib.check(L)
    assert rc == 0
    return int(rec.lines), int(rec.flags)


def fused_texts(rng, pat, cs):
    nl_free = near_text(rng, [pat], cs, 30000, b"ab_\xe9\x8a\x0b ")
    long_lines = bytearray(near_text(rng, [pat], cs, 60000, bytes(range(11, 256))))
    for q in range(0, len(long_lines), 10240):
        long_lines[q] = 10                              # 10 KiB lines: longer than a 2 KiB partition
    dense = near_text(rng, [pat], cs, 200000, b"\n\n" + bytes(range(256)))
    return {
        "full-byte": near_text(rng, [pat], cs, 300000, FULL_BYTE_ALPHABETS[0] + b"\n" * 8),
        "alias": near_text(rng, [pat], cs, 100000, FULL_BYTE_ALPHABETS[1]),
        "no-newline": nl_free.replace(b"\n", b" "),
        "no-hit": bytes(rng.choice(b"\n.\x00\xff") for _ in range(40000)),
        "long-lines": bytes(long_lines),
        "dense": dense,
        "edges": pat + b"\n" + dense[:5000] + b"\n" + pat,
        "nl-edges": b"\n" + pat + dense[:3000] + pat + b"\n",
    }


@pytest.mark.parametrize("part_kb", ["2", "8", None])
@pytest.mark.parametrize("fk", FUSED_KINDS, ids=[k[0] for k in FUSED_KINDS])
def test_fused_count_records_on_random_cuts(fk, part_kb, monkeypatch):
    """krep_b200_count_lines_shard's record (lines AND flags) against the model on cuts anywhere, cuts on a hit's first
    byte, just after a hit, on a newline and just after one; 2 KiB, 8 KiB and the default 64 KiB partitions."""
    if part_kb is None:
        monkeypatch.delenv("KREP_B200_COUNT_PART_KB", raising=False)
    else:
        monkeypatch.setenv("KREP_B200_COUNT_PART_KB", part_kb)
    kid, func, pat, cs, ww = fk
    rng = random.Random(kid + str(part_kb))
    with Plan(func, [pat], cs, ww, count=True) as plan:
        assert plan.shape.ww_mode != 2
        for tname, text in fused_texts(rng, pat, cs).items():
            n = len(text)
            dev = gu.to_device(text)
            hits = (sm.key_starts(plan.model(text, n, 0, n), False)).astype(np.int64)
            nls = np.flatnonzero(np.frombuffer(text, np.uint8) == 10)
            marks = [0, n]
            for arr in (hits, nls):
                if arr.size:
                    for q in rng.sample(list(arr), min(6, arr.size)):
                        marks += [int(q), int(q) + 1]
            marks += [rng.randint(0, n) for _ in range(8)]
            marks = sorted({min(max(q, 0), n) for q in marks})
            for b, e in zip(marks, marks[1:]):
                halo = rng.choice([plan.shape.m - 1, plan.shape.m + 1, 64])
                avail = min(e + halo, n)
                got = count_record(plan, dev.data_ptr(), avail, b, e)
                starts = sm.key_starts(plan.model(text, avail, b, e), False).astype(np.int64)
                want = sm.line_record(text, b, e, starts)
                assert got == want, (kid, part_kb, tname, n, b, e, avail, got, want)
            # the same shard in a buffer of its own, with context bytes
            b, e = marks[len(marks) // 3], marks[2 * len(marks) // 3]
            avail = min(e + plan.shape.m + 1, n)
            own = gu.to_device(text[b:avail])
            prev, nxt = (text[b - 1] if b else -1), (text[avail] if avail < n else -1)
            got = count_record(plan, own.data_ptr(), avail - b, 0, e - b, b, prev, nxt)
            starts = sm.key_starts(plan.model(text[b:avail], avail - b, 0, e - b, 0, prev, nxt), False).astype(np.int64)
            assert got == sm.line_record(text[b:avail], 0, e - b, starts), (kid, part_kb, tname, b, e, got)
