"""-m gpu: fused -c for pattern sets (csrc/scan_set_count.cu) — the record of a shard computed from its sorted keys on
the device.  Raw records of krep_b200_count_lines_shard against tests/scan_model.py, flags included, in every
pattern-set kernel regime; folds of shards cut anywhere (krep_b200_combine_line_counts and one krep_b200_search_shards
call) against the reference; a shard whose occurrences overflow the list; and host text, pinned and pageable, against
the reference and the occurrence-list path (KREP_B200_NO_FUSED_COUNT=1)."""
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
import oracle_util as ou
import scan_model as sm
from krep_b200 import lib
from krep_b200.abi import ALGO_AC, Params, Shard, SIZE_MAX

pytestmark = pytest.mark.gpu


class LineCount(C.Structure):
    _fields_ = [("lines", C.c_uint64), ("flags", C.c_uint32), ("reserved", C.c_uint32)]


@pytest.fixture(scope="module", autouse=True)
def _init():
    L = lib.load()
    assert L.krep_b200_init(0) == 0, L.krep_b200_last_error_string()
    L.krep_b200_count_lines_shard.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(Shard), C.c_void_p, C.POINTER(LineCount)]
    L.krep_b200_count_lines_shard.restype = C.c_int
    L.krep_b200_combine_line_counts.argtypes = [C.POINTER(LineCount), C.c_size_t, C.c_size_t]
    L.krep_b200_combine_line_counts.restype = C.c_uint64


def checker():
    return ou.reference() or ou.port()


class SetPlan:
    def __init__(self, pats, cs=True, ww=False, max_count=SIZE_MAX):
        L = lib.load()
        self.pats, self.cs, self.ww = pats, cs, ww
        self.P = Params(pats, case_sensitive=cs, whole_word=ww, count=True, max_count=max_count)
        self.h = L.krep_b200_plan_create(self.P.ref(), ALGO_AC)
        lib.check(L)
        assert self.h
        self.name = L.krep_b200_plan_filter_name(self.h).decode()
        shape = sm.plan_shape("aho_corasick", pats, cs, ww)
        assert sm.filter_matches(self.name, shape, cs), (pats, self.name, shape)

    def __enter__(self):
        return self

    def __exit__(self, *a):
        lib.load().krep_b200_plan_destroy(self.h)

    def record(self, ptr, avail, ob, oe, go=0, prev=-1, nxt=-1):
        L = lib.load()
        sh = Shard(ptr, avail, ob, oe, go, prev, nxt)
        rec = LineCount()
        rc = L.krep_b200_count_lines_shard(self.h, self.P.ref(), C.byref(sh), None, C.byref(rec))
        lib.check(L)
        assert rc == 0
        return int(rec.lines), int(rec.flags)

    def model(self, buf, avail, ob, oe, go=0, prev=-1, nxt=-1):
        keys = sm.ac_keys(buf, avail, ob, oe, go, prev, nxt, self.pats, self.cs, self.ww)
        return sm.line_record(buf, ob, oe, (sm.key_starts(keys, True).astype(np.int64) - go))


def rpat(rng, m, alpha=b"abcdeXYZ_\xe9\x00"):
    return bytes(rng.choice(alpha) for _ in range(m))


# (id, pattern-set maker, case_sensitive, whole_word): shortest pattern 1-4 (k_ac_scan stride 1), 5 (stride 2), 6
# (k_ac_tri4), 7 and longer (the quad form)
REGIMES = [
    ("min1", lambda r: [rpat(r, 1), rpat(r, 3), rpat(r, 9)], True, False),
    ("min2-fold", lambda r: [rpat(r, 2), rpat(r, 4), rpat(r, 2)], False, False),
    ("min3-w", lambda r: [rpat(r, 3), rpat(r, 5)], True, True),
    ("min5", lambda r: [rpat(r, 5), rpat(r, 8), rpat(r, 12)], True, False),
    ("min5-fold-w", lambda r: [rpat(r, 5), rpat(r, 6)], False, True),
    ("min6", lambda r: [rpat(r, 6), rpat(r, 6), rpat(r, 10)], True, False),
    ("min6-fold", lambda r: [rpat(r, 6), rpat(r, 9)], False, False),
    ("min7", lambda r: [rpat(r, 7), rpat(r, 11), rpat(r, 30)], True, False),
    ("min8-fold-w", lambda r: [rpat(r, 8), rpat(r, 9)], False, True),
]


def make_set(regime, seed):
    rng = random.Random(seed)
    pats = regime[1](rng)
    pats.append(pats[0].swapcase() if rng.random() < 0.5 else pats[0])  # a case twin or a duplicate
    return pats, rng


def set_text(rng, pats, cs, n, alpha, nl_every=None):
    """Filler from the alphabet with an occurrence (case-flipped under -i) or a near miss planted every ~40 bytes;
    newlines from the alphabet, or every nl_every bytes."""
    g = np.random.default_rng(rng.randrange(1 << 30))
    t = np.frombuffer(alpha, np.uint8)[g.integers(0, len(alpha), n)].copy()
    for j, q in enumerate(np.sort(g.integers(0, max(n - 64, 1), n // 40)).tolist()):
        p = pats[j % len(pats)]
        if j % 3 == 2:
            b = bytearray(p)
            b[j % len(b)] ^= 0x20
            p = bytes(b)
        elif not cs and j % 2:
            p = p.swapcase()
        t[q:q + len(p)] = np.frombuffer(p, np.uint8)[:n - q]
    if nl_every:
        t[::nl_every] = 10
    return t.tobytes()


def geometries(rng, text, plan):
    """(ob, oe, avail): the whole text, random cuts, cuts on a hit's first byte / inside a hit / on a newline / just
    after one, an occurrence straddling own_end."""
    n = len(text)
    keys = sm.ac_keys(text, n, 0, n, 0, -1, -1, plan.pats, plan.cs, plan.ww)
    starts = sm.key_starts(keys, True).astype(np.int64).tolist()
    nls = np.flatnonzero(np.frombuffer(text, np.uint8) == 10).tolist()
    marks = {0, n}
    for arr, d in ((starts, (0, 1, 2)), (nls, (0, 1))):
        for q in rng.sample(arr, min(5, len(arr))):
            marks.add(min(q + rng.choice(d), n))
    marks |= {rng.randint(0, n) for _ in range(5)}
    marks = sorted(marks)
    maxlen = max(len(p) for p in plan.pats)
    out = [(b, e, min(e + rng.choice([maxlen - 1, maxlen + 1, 100]), n)) for b, e in zip(marks, marks[1:])]
    out.append((0, n, n))
    if starts:
        s = rng.choice(starts)
        out.append((max(0, s - 37), s + 1, n))  # the owned range ends inside an occurrence
    return out


@pytest.mark.parametrize("regime", REGIMES, ids=[r[0] for r in REGIMES])
def test_raw_records_equal_the_model(regime):
    """Lines AND flags of krep_b200_count_lines_shard on views into one buffer and on buffers of their own with
    context bytes, over texts with short lines, no newline, no occurrence, and lines longer than 1 MiB."""
    pats, rng = make_set(regime, zlib.crc32(regime[0].encode()))
    _, _, cs, ww = regime
    with SetPlan(pats, cs, ww) as plan:
        texts = {
            "short-lines": set_text(rng, pats, cs, 50_000, b"ab _\n\x00\xe9"),
            "full-byte": set_text(rng, pats, cs, 40_000, bytes(range(256))),
            "no-newline": set_text(rng, pats, cs, 30_000, b"ab _\x00\xe9"),
            "no-hit": bytes(rng.choice(b"\n\r.,;") for _ in range(30_000)),
            "long-lines": set_text(rng, pats, cs, 3 * (1 << 20) + 99, b"ab _\x00", nl_every=(1 << 20) + 4099),
            "sparse-long": b"." * (1 << 20) + pats[0] + b"." * ((1 << 20) + 7) + pats[-1] + b"\n" + b"." * 5000 + pats[0],
        }
        for tname, text in texts.items():
            n = len(text)
            dev = gu.to_device(text)
            for ob, oe, avail in geometries(rng, text, plan):
                got = plan.record(dev.data_ptr(), avail, ob, oe)
                want = plan.model(text, avail, ob, oe)
                assert got == want, (regime[0], tname, n, ob, oe, avail, got, want)
            # a shard in a buffer of its own at a global offset, with context bytes present and absent
            for b, e in ((n // 3, 2 * n // 3), (1, n - 1)):
                avail = min(e + max(map(len, pats)) + 1, n)
                own = gu.to_device(text[b:avail])
                for prev, nxt in ((text[b - 1], text[avail] if avail < n else -1), (-1, -1)):
                    got = plan.record(own.data_ptr(), avail - b, 0, e - b, b, prev, nxt)
                    want = plan.model(text[b:avail], avail - b, 0, e - b, 0, prev, nxt)
                    assert got == want, (regime[0], tname, b, e, prev, nxt, got, want)
            del dev
        torch.cuda.empty_cache()


def _cuts(rng, text, pats, nsh):
    """nsh shards: cuts on a hit's first byte, inside a hit, on a newline and just after one, or anywhere."""
    n = len(text)
    keys = sm.ac_keys(text, n, 0, n, 0, -1, -1, pats, True, False)
    starts = sm.key_starts(keys, True).astype(np.int64).tolist()
    nls = np.flatnonzero(np.frombuffer(text, np.uint8) == 10).tolist()
    cuts = set()
    while len(cuts) < nsh - 1:
        kind = len(cuts) % 4
        if kind == 0 and starts:
            q = rng.choice(starts)
        elif kind == 1 and starts:
            q = rng.choice(starts) + 1
        elif kind == 2 and nls:
            q = rng.choice(nls) + rng.choice([0, 1])
        else:
            q = rng.randint(1, n - 1)
        if 0 < q < n:
            cuts.add(q)
    return [0] + sorted(cuts) + [n]


def _devices():
    return list(range(torch.cuda.device_count()))


@pytest.mark.parametrize("multi_gpu", [False, True])
def test_shards_cut_anywhere_fold_to_the_reference(multi_gpu):
    """1 / 2 / 5 / 8 shards, folded from krep_b200_count_lines_shard records and answered by one krep_b200_search_shards
    -c call, equal the reference with -m unlimited, 1 and 3; with several GPUs the shards go round the devices."""
    devs = _devices()
    if multi_gpu and len(devs) < 2:
        pytest.skip("one GPU: the several-device fold needs two")
    L = lib.load()
    rng = random.Random(77 + multi_gpu)
    for regime in (REGIMES[0], REGIMES[3], REGIMES[5], REGIMES[8]):
        pats, _ = make_set(regime, rng.randrange(1 << 16))
        _, _, cs, ww = regime
        for n, alpha in ((400_000, b"ab _\n\n\x00"), (200_000, b"ab _\x00")):
            text = set_text(rng, pats, cs, n, alpha)
            halo = max(map(len, pats)) + 1
            for nsh in (1, 2, 5, 8):
                cuts = _cuts(rng, text, pats, nsh)
                keep, shards = [], []
                for g, (b, e) in enumerate(zip(cuts, cuts[1:])):
                    avail = min(e + halo, n)
                    dev = f"cuda:{devs[g % len(devs)]}" if multi_gpu else "cuda:0"
                    with torch.cuda.device(dev):
                        buf = gu.to_device(text[b:avail])
                    keep.append(buf)
                    shards.append(Shard(buf.data_ptr(), avail - b, 0, e - b, b, text[b - 1] if b else -1,
                                        text[avail] if avail < n else -1))
                for mc in (SIZE_MAX, 1, 3):
                    want = checker().run("aho_corasick", Params(pats, case_sensitive=cs, whole_word=ww, count=True, max_count=mc),
                                         text, with_result=False)[0]
                    with SetPlan(pats, cs, ww, mc) as plan:
                        recs = (LineCount * nsh)()
                        for g, sh in enumerate(shards):
                            rc = L.krep_b200_count_lines_shard(plan.h, plan.P.ref(), C.byref(sh), None, C.byref(recs[g]))
                            lib.check(L)
                            assert rc == 0
                        got = int(L.krep_b200_combine_line_counts(recs, nsh, mc))
                        assert got == want, (regime[0], n, nsh, cuts, mc, got, want)
                        got = lib.search_shards(plan.h, plan.P, shards, with_result=False)[0]
                        assert got == want, (regime[0], n, nsh, cuts, mc, "search_shards", got, want)


def _overflow_case():
    """A shard with a 1-byte pattern on every byte: more occurrences than the engine's initial 2^20-key list holds
    (ensure_keys), counted in pieces without growing the list."""
    L = lib.load()
    assert L.krep_b200_init(0) == 0
    L.krep_b200_count_lines_shard.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(Shard), C.c_void_p, C.POINTER(LineCount)]
    L.krep_b200_count_lines_shard.restype = C.c_int
    cap = 1 << 20
    n = 3 * cap + 12345
    t = np.full(n, ord("q"), dtype=np.uint8)
    t[5::1000] = ord("\n")
    t[2 * cap:2 * cap + 300000] = ord(".")        # a quiet stretch: the density the cut assumed is not the piece's
    text = t.tobytes()
    dev = gu.to_device(text)
    for pats, ob, oe in (([b"q"], 0, n), ([b"q", b"qq"], 7, n - 3), ([b"Q", b"."], 1, n)):
        with SetPlan(pats, cs=pats[0] != b"Q") as plan:
            keys = sm.ac_keys(text, n, ob, oe, 0, -1, -1, pats, plan.cs, False)
            assert keys.size > cap, keys.size
            got = plan.record(dev.data_ptr(), n, ob, oe)
            want = sm.line_record(text, ob, oe, sm.key_starts(keys, True).astype(np.int64))
            assert got == want, (pats, got, want)
            # the whole text as the answer of a search: the reference's -c
            p = Params(pats, case_sensitive=plan.cs, count=True)
            assert lib.search("aho_corasick", p, text)[0] == checker().run("aho_corasick", p, text, with_result=False)[0]
    print("set overflow ok")


def test_dense_shard_past_the_list_capacity_in_a_fresh_process():
    """The list a process grows stays grown, so the engine's initial capacity is only certain in a process of its own."""
    here = os.path.dirname(os.path.abspath(__file__))
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([here, os.path.dirname(here), os.environ.get("PYTHONPATH", "")]))
    r = subprocess.run([sys.executable, "-c", "import test_gpu_set_count as t; t._overflow_case()"], cwd=here, env=env,
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and "set overflow ok" in r.stdout, r.stdout[-2000:] + r.stderr[-4000:]


@pytest.mark.parametrize("pinned", [False, True])
@pytest.mark.parametrize("ranges", ["1", "3"])
def test_host_text_counts_from_chunk_records(pinned, ranges, monkeypatch):
    """aho_corasick -c on host text in 1 MiB chunks: the records of many chunks (and ranges) folded equal the reference
    and the occurrence-list path."""
    monkeypatch.setenv("KREP_B200_STAGE_MB", "1")
    monkeypatch.setenv("KREP_B200_CHUNK_MB", "1")
    monkeypatch.setenv("KREP_B200_RANGES", ranges)
    monkeypatch.delenv("KREP_B200_NO_FUSED_COUNT", raising=False)
    rng = random.Random(int(ranges) * 2 + pinned)
    chk = checker()
    for regime in REGIMES:
        pats, _ = make_set(regime, rng.randrange(1 << 16))
        _, _, cs, ww = regime
        for n, alpha, nl_every in ((3 * (1 << 20) + 333, b"ab _\n\x00\xe9", None), (2 * (1 << 20) + 17, b"ab _", 700_001),
                                   (4000, b"ab\n", None)):
            text = set_text(rng, pats, cs, n, alpha, nl_every)
            if pinned:
                host = torch.empty(n, dtype=torch.uint8, pin_memory=True)
                host.numpy()[:] = np.frombuffer(text, np.uint8)
                kw = dict(text_ptr=host.data_ptr(), text_len=n)
            else:
                kw = {}
            for mc in (SIZE_MAX, 2):
                opts = dict(case_sensitive=cs, whole_word=ww, count=True, max_count=mc)
                want = chk.run("aho_corasick", Params(pats, **opts), text, with_result=False)
                got = lib.search("aho_corasick", Params(pats, **opts), text, with_result=False, **kw)
                assert got == want, (regime[0], n, pinned, ranges, mc, got[0], want[0])
                monkeypatch.setenv("KREP_B200_NO_FUSED_COUNT", "1")
                assert lib.search("aho_corasick", Params(pats, **opts), text, with_result=False, **kw) == want
                monkeypatch.delenv("KREP_B200_NO_FUSED_COUNT")
