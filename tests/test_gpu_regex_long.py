"""The -E long-line pass (scan_regex_long.cu, DESIGN §12.8): krep_b200_regex_scan_shard_long_raw against
tests/regex_long_model.py exactly, for single and split plans, in every mode the plan admits and at several slice and
checkpoint sizes; the search entry points against the reference on texts whose lines run past the kernel's reach; the
overflow re-scan; rows of resident shards; the 2^30 rule and the KREP_B200_NO_LONG_LINES knob."""
import ctypes as C
import random
import time

import numpy as np
import pytest

from krep_b200 import lib
from krep_b200.abi import ALGO_REGEX, Params, Shard
import regex_kernel_model as km
import regex_long_model as lm
import regex_rows_util as rr
import regex_util as ru
from test_gpu_regex import _want
import test_gpu_regex_shards as gs

pytestmark = pytest.mark.gpu
SIZES = [(0, 0), (64, 16), (16, 4)]
PATTERNS = ["a[^x]*b", "(ab)*c", "^x.*y$", "x{255}y", ".*QQ|,", "the[a-z]*", "b|a+", "c a"]
# patterns whose enumeration provably stays within the step budget on these texts (a start walks at most a few bytes, or
# a run that the match from its first byte consumes): their match keys must be exact, not a prefix
BUDGET_FREE = {"the[a-z]*", "b|a+", "c a"}


@pytest.fixture(scope="module", autouse=True)
def _init():
    L = lib.load()
    assert L.krep_b200_init(0) == 0, L.krep_b200_last_error_string()


@pytest.fixture(autouse=True)
def _device_paths_on(monkeypatch):
    for k in ("KREP_B200_NO_FUSED_COUNT", "KREP_B200_NO_DEVICE_MATCHES", "KREP_B200_NO_LONG_LINES"):
        monkeypatch.delenv(k, raising=False)


class Plan:
    """A regex plan (split when max_states is given) and the modes the hook admits for it."""

    def __init__(self, pats, max_states=None, case_sensitive=True):
        L = lib.load()
        pats = [pats] if isinstance(pats, str) else pats
        self.P = Params([p.encode() for p in pats], regex=True, case_sensitive=case_sensitive)
        self.h = (L.krep_b200_plan_create(self.P.ref(), ALGO_REGEX) if max_states is None
                  else L.krep_b200_regex_plan_split(self.P.ref(), max_states))
        L.krep_b200_last_error()
        self.modes = []
        if self.h:
            buf = gs.Resident([km.Shard(b"a\n")])
            for m in (0, 1, 2):
                if L.krep_b200_regex_scan_shard_long_raw(self.h, C.byref(buf.structs[0]), m, 0, 0, None, 0, None) >= 0:
                    self.modes.append(m)
                L.krep_b200_last_error()

    def close(self):
        if self.h:
            lib.load().krep_b200_plan_destroy(self.h)


def hook(plan, st, mode, sizes=(0, 0), long=True, cap=1 << 16):
    """Sorted keys and device_lines of one scan (the long-line hook, or the raw hook with long=False)."""
    L = lib.load()
    while True:
        keys = np.zeros(cap, dtype=np.uint64)
        dl = C.c_uint64(12345)
        kp = keys.ctypes.data_as(C.POINTER(C.c_uint64))
        if long:
            k = L.krep_b200_regex_scan_shard_long_raw(plan.h, C.byref(st), mode, sizes[0], sizes[1], kp, cap, C.byref(dl))
        else:
            k = L.krep_b200_regex_scan_shard_raw(plan.h, C.byref(st), mode, kp, cap, C.byref(dl))
        assert k >= 0, (k, L.krep_b200_last_error_string())
        if k <= cap:
            return keys[:k].tolist(), dl.value
        cap = k


def _line(rng, n, alphabet):
    b = bytes(rng.choice(alphabet) for _ in range(n))
    if rng.random() < 0.3 and n >= 2:
        b = b"x" + b[1:-1] + b"y"
    return b


def long_text(rng, alphabet=b"abcxy ,Q", lens=(4095, 4096, 4097, 4351, 4352, 4353, 8191, 8192, 8193, 12288, 20000)):
    parts = []
    for _ in range(rng.randint(4, 9)):
        parts.append(_line(rng, rng.choice(lens), alphabet) + b"\n")
        parts.append(ru.random_text(rng, rng.randint(1, 200)))
    if rng.random() < 0.5:
        parts.append(_line(rng, rng.choice(lens), alphabet) + b"\n")  # a long last line
    return b"".join(parts)


def shards_of(rng, text):
    """Whole-text shards (no byte after it, and one after it) and a random tiling, as regex_kernel_model.Shard."""
    out = [km.Shard(text), km.Shard(text, next_byte=ord("z"))]
    cuts = sorted(rng.sample(range(1, len(text)), 3))
    out += [sh for _, sh in km.tiling(text, cuts, rng)]
    # owned from own_begin > 0 after a cut mid-line, with a readable byte before and after
    a = rng.randint(1, len(text) // 2)
    out.append(km.Shard(text[a - (a % 16):], a % 16, len(text) - a + a % 16, a - (a % 16), text[a - (a % 16) - 1], ord("q")))
    return out


def run_model(plan, shards, sizes_list=SIZES, what="", budget_free=False):
    for sh in shards:
        res = gs.Resident([sh])
        st = res.structs[0]
        g = km.GlibcLines(plan.P, sh.buf)
        flagged = km.HookLines(plan.P, sh.buf).flagged
        for mode in plan.modes:
            exp = lm.expect(sh, mode, flagged if mode == 0 else g, budget_free)
            for sizes in sizes_list:
                keys, dl = hook(plan, st, mode, sizes)
                lm.check(exp, keys, dl, (what, plan.P.patterns, mode, sizes, sh.own_begin, sh.own_end, sh.avail,
                                         sh.prev_byte, sh.next_byte))


@pytest.mark.parametrize("pat", PATTERNS)
def test_hook_against_model(pat):
    rng = random.Random(hash(pat) & 0xFFFF)
    plan = Plan(pat)
    if not plan.h:
        pytest.skip(f"{pat} is refused")
    try:
        for it in range(2):
            run_model(plan, shards_of(rng, long_text(rng)), what=it, budget_free=pat in BUDGET_FREE)
    finally:
        plan.close()


@pytest.mark.parametrize("icase", [False, True])
def test_split_plans(icase):
    rng = random.Random(7 + icase)
    plan = Plan(["the[a-z]*|a[^x]*b|(ab)*c|b,c|^x.*y$"], max_states=8, case_sensitive=not icase)
    assert plan.h
    try:
        assert "split" in lib.load().krep_b200_plan_filter_name(plan.h).decode()
        run_model(plan, shards_of(rng, long_text(rng, alphabet=b"abcxyAB ,the")))
    finally:
        plan.close()


def test_over_budget_and_long_match():
    plan = Plan(".*QQ|,")
    try:
        rng = random.Random(3)
        line = bytes(rng.choice(b"ab ,") for _ in range(30000))
        sh = km.Shard(b"x\n" + line + b"\nz\n")
        run_model(plan, [sh], sizes_list=[(0, 0)])
        # every start walks `.*QQ` to the line's end: over budget after a few starts, the line keeps its key
        keys, _ = hook(plan, gs.Resident([sh]).structs[0], 2)
        assert 2 << 16 in keys
    finally:
        plan.close()
    plan = Plan("b|a+")
    try:
        sh = km.Shard(b"b" + b"a" * 9000 + b"b\n" + b"a" * 5000 + b"\nq\n")
        run_model(plan, [sh])
        keys, _ = hook(plan, gs.Resident([sh]).structs[0], 2)
        assert 0 in keys  # the line with a 9000-byte match keeps its key
    finally:
        plan.close()


def test_enumeration_work_is_bounded():
    # `ab|b.*c` on `abab...` without a `c`: every start on a `b` walks `b.*c` to the end of the line, but the winning
    # start (the `a` before it) matches `ab` in a few steps.  The lanes past the winner must stop, or a round of 32
    # starts costs a walk of the whole line.
    plan = Plan("ab|b.*c")
    try:
        assert 2 in plan.modes
        n = 1 << 20
        sh = km.Shard(b"ab" * n + b"\nz\n")
        st = gs.Resident([sh]).structs[0]
        t0 = time.perf_counter()
        keys, _ = hook(plan, st, 2, cap=n + 8)
        took = time.perf_counter() - t0
        want = (np.arange(0, 2 * n, 2, dtype=np.uint64) << np.uint64(16)) | np.uint64((2 << 3) | 1)
        assert len(keys) == n + 1 and keys[-1] == (2 * n + 1) << 16
        assert np.array_equal(np.array(keys[:n], dtype=np.uint64), want)
        assert took < 60, took
    finally:
        plan.close()


def test_overflow_rescan():
    # one long line with more matches than a fresh key list holds
    plan = Plan("a")
    try:
        n = 3 << 20
        sh = km.Shard(b"a" * n + b"\nb\n")
        keys, _ = hook(plan, gs.Resident([sh]).structs[0], 2, cap=n + 8)
        want = (np.arange(n, dtype=np.uint64) << np.uint64(16)) | np.uint64((1 << 3) | 1)
        assert len(keys) == n + 1 and keys[-1] == (n + 1) << 16
        assert np.array_equal(np.array(keys[:n], dtype=np.uint64), want)
    finally:
        plan.close()


def _big_text(seed):
    rng = random.Random(seed)
    parts = []
    for L in (300000, 5000, 1300000, 9000, 700000, 4200):
        parts.append(_line(rng, L, b"abcthe ,xy") + b"\n")
        parts.append(ru.random_text(rng, rng.randint(1, 2000)))
    return b"".join(parts)


CASES = [("the[a-z]*", dict(count=True)), ("the[a-z]*", dict(count=True, only_matching=True)), ("the[a-z]*", dict()),
         ("TH[a-z]*", dict(case_sensitive=False)), ("the", dict(whole_word=True)), ("a[^x]*b", dict(max_count=1)),
         ("c,|a b", dict(max_count=3)), ("the[a-z]*|a[^x]*b|(ab)*c|b,c", dict(count=True))]


@pytest.mark.parametrize("pinned", [False, True])
def test_search_against_reference(monkeypatch, pinned):
    import torch
    monkeypatch.setenv("KREP_B200_STAGE_MB", "1")
    monkeypatch.setenv("KREP_B200_CHUNK_MB", "1")
    text = _big_text(5)
    buf = None
    if pinned:
        buf = torch.empty(len(text), dtype=torch.uint8).pin_memory()
        buf.numpy()[:] = np.frombuffer(text, dtype=np.uint8)
    for pat, kw in CASES:
        P = Params([pat.encode()], regex=True, **kw)
        lib.load().krep_b200_set_only_matching(bool(kw.get("only_matching")))
        try:
            if pinned:
                got = lib.search("regex", P, None, text_ptr=buf.data_ptr(), text_len=len(text))
            else:
                got = lib.search("regex", P, text)
        finally:
            lib.load().krep_b200_set_only_matching(False)
        want = _want(P, text)
        assert got[0] == want[0] and (not P.struct.track_positions or got[1] == want[1]), (pat, kw, got[0], want[0])


@pytest.mark.parametrize("seed", range(3))
def test_resident_shards(seed):
    rng = random.Random(seed)
    text = _big_text(seed)
    n = len(text)
    for pat, kw in CASES[:4] + CASES[5:7]:
        P = Params([pat.encode()], regex=True, **kw)
        gs.check(P, text, sorted(rng.sample(range(1, n), 2)), rng.choice([0, 17, km.REGEX_HALO]), ref=False, what=seed)
    # the rows of the shards are the host's slicing of their own keys
    P = Params([b"the[a-z]*"], regex=True, count=bool(seed % 2))
    h = gs._plan(P)
    try:
        shards = rr.tile(text, sorted(rng.sample(range(1, n), 3)), km.REGEX_HALO)
        res = gs.Resident(shards)
        rows = []
        for sh, st in zip(shards, res.structs):
            row = gs.export(h, P, st)
            d = rr.parse_row(row)
            assert row == rr.build_row(sh, d["mode"], d["keys"], d["device_lines"])
            rows.append(row)
        assert lib.regex_resolve(P, rows) == lib.search("regex", P, text)
    finally:
        lib.load().krep_b200_plan_destroy(h)


def test_line_of_2_30_bytes_stays_uncertain():
    text = b"ab\n" + b"a" * (1 << 30) + b"\nab\n"
    sh = km.Shard(text)
    plan = Plan("b")
    try:
        res = gs.Resident([sh])
        keys, dl = hook(plan, res.structs[0], 1)
        assert keys == [3 << 3, (len(text) - 3) << 3] and dl == 1
        P = Params([b"b"], regex=True, count=True)
        assert lib.search_shards(plan.h, P, res.structs)[0] == 2
    finally:
        plan.close()


def test_knob(monkeypatch):
    rng = random.Random(9)
    text = long_text(rng)
    sh = km.Shard(text)
    for pat in ("a[^x]*b", "the[a-z]*"):
        plan = Plan(pat)
        try:
            st = gs.Resident([sh]).structs[0]
            on = {m: hook(plan, st, m) for m in plan.modes}
            monkeypatch.setenv("KREP_B200_NO_LONG_LINES", "1")
            for m in plan.modes:
                assert hook(plan, st, m) == hook(plan, st, m, long=False)
            off = [lib.search("regex", Params([pat.encode()], regex=True, **kw), text) for kw in (dict(), dict(count=True))]
            monkeypatch.delenv("KREP_B200_NO_LONG_LINES")
            assert off == [lib.search("regex", Params([pat.encode()], regex=True, **kw), text) for kw in (dict(), dict(count=True))]
            assert all(hook(plan, st, m) == on[m] for m in plan.modes)
        finally:
            plan.close()
