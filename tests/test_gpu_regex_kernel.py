"""What k_regex_lines decides, not only what glibc answers afterwards: krep_b200_regex_scan_shard_raw hands back the raw
keys (and the count mode's line counter) of one scan, and every case here compares them exactly with
tests/regex_kernel_model.py, in every mode the plan admits (0 = line filter, 1 = fused -c, 2 = match offsets).

The end-to-end tests of test_gpu_regex*.py cannot see a kernel that decides too little: glibc recomputes every line
the kernel hands back, so flagging every line as uncertain gives the right answer, only about 17x slower.  These tests
fail on that."""
import ctypes as C
import random

import numpy as np
import pytest

from krep_b200 import lib
from krep_b200.abi import ALGO_REGEX, Params, Shard
import regex_kernel_model as km
import regex_util as ru
from test_gpu_regex import _want

pytestmark = pytest.mark.gpu
SPEC = (0x5EED0001, 0x5EED0002, 1 << 16, b"qzXv9Kpw")


@pytest.fixture(scope="module", autouse=True)
def _init():
    L = lib.load()
    assert L.krep_b200_init(0) == 0, L.krep_b200_last_error_string()


@pytest.fixture(autouse=True)
def _device_paths_on(monkeypatch):
    # Plan.modes asks the library which path a call takes; the knobs that turn the device paths off would make it
    # report modes the plan (and the hook) still admit
    monkeypatch.delenv("KREP_B200_NO_FUSED_COUNT", raising=False)
    monkeypatch.delenv("KREP_B200_NO_DEVICE_MATCHES", raising=False)


def _params(pats, **kw):
    if isinstance(pats, str):
        pats = [pats]
    return Params([p.encode() for p in pats], regex=True, **kw)


class Plan:
    """A regex plan and the modes it admits (by the library's own eligibility answers for -c and positions calls)."""

    def __init__(self, pats, case_sensitive=True, whole_word=False):
        L = lib.load()
        self.P = _params(pats, case_sensitive=case_sensitive, whole_word=whole_word)
        self.Pc = _params(pats, case_sensitive=case_sensitive, whole_word=whole_word, count=True)
        self.h = L.krep_b200_plan_create(self.P.ref(), ALGO_REGEX)
        lib.check(L)
        assert self.h, pats
        self.modes = [0]
        if L.krep_b200_regex_count_mode(self.Pc.ref()) == 1:
            self.modes.append(1)
        if L.krep_b200_regex_match_mode(self.P.ref()) == 1:
            self.modes.append(2)

    def close(self):
        lib.load().krep_b200_plan_destroy(self.h)

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()


def raw(plan, ptr, sh, mode, cap=1 << 16):
    """The hook on the device bytes at ptr (sh.buf there). -> (sorted keys, device_lines)
    When the keys do not fit in cap the scan runs again with room for all of them; it must give the same count."""
    L = lib.load()
    shard = Shard(ptr, sh.avail, sh.own_begin, sh.own_end, sh.global_offset, sh.prev_byte, sh.next_byte)
    first = None
    while True:
        keys = np.zeros(max(cap, 1), dtype=np.uint64)
        dl = C.c_uint64(12345)
        k = L.krep_b200_regex_scan_shard_raw(plan.h, C.byref(shard), mode, keys.ctypes.data_as(C.POINTER(C.c_uint64)), cap,
                                             C.byref(dl))
        assert k >= 0, (k, L.krep_b200_last_error_string())
        assert first is None or (k, dl.value) == first, (mode, first, k, dl.value)
        if k <= cap:
            return keys[:k].tolist(), dl.value
        first, cap = (k, dl.value), k


def to_device(data):
    import gpu_util as gu
    return gu.to_device(data)


def run_shard(plan, ptr, sh, oracle=None, budget_free=False, what=""):
    """Hook vs model in every mode the plan admits; the refused modes must be refused. -> {mode: (keys, device_lines)}"""
    L = lib.load()
    flagged = km.HookLines(plan.P, sh.buf).flagged
    oracle = oracle or km.GlibcLines(plan.P, sh.buf)
    out = {}
    for mode in (0, 1, 2):
        if mode not in plan.modes:
            shard = Shard(ptr, sh.avail, sh.own_begin, sh.own_end, sh.global_offset, sh.prev_byte, sh.next_byte)
            assert L.krep_b200_regex_scan_shard_raw(plan.h, C.byref(shard), mode, None, 0, None) < 0
            L.krep_b200_last_error()
            continue
        keys, dl = raw(plan, ptr, sh, mode)
        exp = km.expect(sh, mode, flagged if mode == 0 else oracle, budget_free)
        km.check(exp, keys, dl, (what, mode, plan.P.patterns, sh.own_begin, sh.own_end, sh.avail, sh.prev_byte, sh.next_byte))
        out[mode] = (keys, dl)
    return out


# patterns whose match mode cannot reach the step budget on these texts (every start walks a bounded number of bytes,
# or a run of x's once): their long lines are compared exactly, not in the prefix form
BUDGET_FREE = {"b$", "^a", "x*", "ab"}
GEO_PATS = ["b$", "^a", "x*", "ab", "a+b", "(ab|ba)c?", "^$", "a|ab|abc"]


def geometry_text(rng, n):
    """Lines of every length 1..64 (so line starts cover every residue mod 16), some empty, in random order."""
    parts = []
    while sum(map(len, parts)) < n:
        L = rng.randint(0, 64)
        parts.append(bytes(rng.choice(b"aabbcx ") for _ in range(L)) + b"\n")
    return b"".join(parts)


def test_geometry_sweep():
    rng = random.Random(31)
    text = geometry_text(rng, 14000)
    cases = []
    for ob in (0, 1, 15, 16, 17, 255, 256, 257):
        for own in (0, 1, 255, 1000):
            cases.append((ob, own, rng.choice([0, 1, 4095, 4096, 4097, 8192]), rng.choice([-1, 10, 97]), rng.choice([-1, 10, 97])))
    for tail in (0, 1, 4095, 4096, 4097, 8192):
        for prev in (-1, 10, 97):
            for nxt in (-1, 10, 97):
                cases.append((rng.choice([0, 1, 15, 16, 17, 255, 256, 257]), rng.randint(0, 1300), tail, prev, nxt))
    for i, (ob, own, tail, prev, nxt) in enumerate(cases):
        cut = text[: max(ob + own + tail, 1)]
        pat = GEO_PATS[i % len(GEO_PATS)]
        with Plan(pat) as plan:
            for buf in (cut[:-1] + b"\n", cut[:-1] + b"a"):  # shard text with and without a final '\n'
                sh = km.Shard(buf, ob, ob + own, 1000, prev, nxt)
                run_shard(plan, to_device(buf).data_ptr(), sh, budget_free=pat in BUDGET_FREE, what=i)


def test_newline_at_the_reach_limit():
    # a line starting at a segment's first, second and last byte whose '\n' falls at limit-1, limit and limit+1
    rng = random.Random(32)
    for ob in (0, 17):
        for j, off in ((1, 0), (1, 1), (1, 255), (0, 0), (2, 255)):
            p = ob + 256 * j + off
            se = ob + 256 * (j + 1)
            limit = se + km.REGEX_HALO
            for nl in (limit - 1, limit, limit + 1):
                head = bytes(rng.choice(b"ab ") for _ in range(p - 1)) + b"\n" if p else b""
                body = b"a" + bytes(rng.choice(b"ab ") for _ in range(nl - p - 2)) + b"b"
                buf = head + body + b"\nab\n" + b"ba\n" * 40
                assert buf[nl] == 10 and (p == 0 or buf[p - 1] == 10)
                t = to_device(buf)
                for own_end in (se, se + 1000):
                    sh = km.Shard(buf, ob, own_end, 0, -1, rng.choice([-1, 10]))
                    lines = {ln.p: ln for ln in km.owned_lines(sh)}
                    if p >= ob:
                        assert (lines[p].nl is None) == (nl >= limit)
                    for pat in ("b$", "^a", "ab"):
                        with Plan(pat) as plan:
                            run_shard(plan, t.data_ptr(), sh, budget_free=True, what=(ob, j, off, nl))


def test_newlines_on_segment_edges():
    # '\n' at sb-1, sb, se-1 and se of every segment, empty lines across the edges
    rng = random.Random(33)
    for ob in (0, 5, 16):
        buf = bytearray(geometry_text(rng, 6000))
        for sb in range(ob + 256, len(buf) - 300, 256):
            k = rng.randint(0, 3)
            if k == 0:
                buf[sb - 1] = 10
            elif k == 1:
                buf[sb] = 10
            elif k == 2:
                buf[sb - 1] = buf[sb] = 10
            else:
                buf[sb - 2] = buf[sb - 1] = buf[sb] = buf[sb + 1] = 10
        buf = bytes(buf)
        t = to_device(buf)
        for own_end in (len(buf), len(buf) - 4097, ob + 256 * 7):
            for pat in GEO_PATS:
                with Plan(pat) as plan:
                    sh = km.Shard(buf, ob, own_end, 0, 10, -1)
                    run_shard(plan, t.data_ptr(), sh, budget_free=pat in BUDGET_FREE, what=(ob, own_end))


@pytest.mark.parametrize("nshards", [2, 3, 7])
def test_tilings(nshards):
    rng = random.Random(40 + nshards)
    for it in range(6):
        text = km.random_lines_text(rng, rng.randint(20000, 40000))
        n = len(text)
        t = to_device(text)
        cuts = [rng.randint(0, n) for _ in range(nshards - 1)]
        shards = km.tiling(text, cuts, rng)
        for pat in ("a+b", "b$", "x*", "^a|c ", "(ab|ba)c?"):
            with Plan(pat) as plan:
                count_keys, match_keys, lines = [], [], 0
                for d, sh in shards:
                    out = run_shard(plan, t.data_ptr() + d, sh, budget_free=pat in BUDGET_FREE, what=(it, pat, d))
                    if 1 in out:
                        count_keys += out[1][0]
                        lines += out[1][1]
                    if 2 in out:
                        match_keys += out[2][0]
                assert 1 in plan.modes and 2 in plan.modes, pat
                assert count_keys == sorted(count_keys) and match_keys == sorted(match_keys)
                assert km.resolve(plan.Pc, text, 0, count_keys=count_keys, device_lines=lines) == _want(plan.Pc, text)[0]
                assert km.resolve(plan.P, text, 0, match_keys=match_keys) == _want(plan.P, text)[1]


OPTS = [dict(), dict(count=True), dict(count=True, only_matching=True), dict(case_sensitive=False), dict(whole_word=True),
        dict(max_count=1), dict(max_count=7)]


def test_random_regexes():
    rng = random.Random(50)
    done = 0
    while done < 200:
        pats = [ru.random_regex(rng) for _ in range(rng.choice([1, 1, 2]))]
        icase = rng.random() < 0.3
        try:
            _params(pats, case_sensitive=not icase)
        except ValueError:
            continue
        if ru.filter_host(_params(pats), b"") is None:
            continue  # refused by the device compiler
        text = km.random_lines_text(rng, rng.randint(1, 6000))
        t = to_device(text)
        with Plan(pats, case_sensitive=not icase) as plan:
            out = run_shard(plan, t.data_ptr(), km.Shard(text), what=pats)
            assert ru.replay(plan.P, out[0][0], text) == _want(plan.P, text), (pats, icase)  # the filter keys, confirmed
        for kw in OPTS:
            P = _params(pats, **{"case_sensitive": not icase, **kw})
            assert lib.search("regex", P, text) == _want(P, text), (pats, icase, kw)
        done += 1


def ac_d_walk(line):
    """The match mode's enumeration of [a-c]*d over one line (without its '\\n'), restated with that regex's automaton
    written out by hand (S: a-c -> S, d -> ACC; ACC: anything -> DEAD), steps counted as the kernel counts them.
    -> (matches, over budget)"""
    S, ACC, DEAD = 1, 2, 0
    n = len(line)
    budget = km.STEPS_PER_BYTE * n + km.STEPS_BASE
    steps, cur, out = 0, 0, []
    while cur <= n and steps <= budget:
        s, e, found = cur, 0, False
        while s <= n and steps <= budget:
            r, x = S, s
            steps += 1
            while x < n and r != DEAD:
                c = line[x]
                r = (S if c in b"abc" else ACC if c == ord("d") else DEAD) if r == S else DEAD
                x += 1
                steps += 1
                if r == ACC:
                    found, e = True, x
            if found:
                break
            s += 1
        if not found:
            break
        out.append((s, e))
        cur = e if e != s else s + 1
    return out, steps > budget


def test_step_budget_boundary():
    # lines whose enumeration takes exactly the budget, and one step more: the first are enumerated on the device,
    # the second leave an uncertain key after the matches emitted so far
    lines = []
    for head in (b"", b"cd ", b"d"):
        over = [ac_d_walk(head + b"a" * r + b" cd")[1] for r in range(200)]
        r = over.index(True)
        assert r > 20 and not any(over[:r]) and all(over[r:])
        lines += [head + b"a" * (r - 1) + b" cd", head + b"a" * r + b" cd", head + b"ab" * (r // 2 + 1) + b" cd"]
    text = b"\n".join(lines) + b"\nzz\n"
    t = to_device(text)
    g = km.GlibcLines(_params("[a-c]*d"), text)
    want, p = [], 0
    for line in lines:
        ms, over = ac_d_walk(line)
        if not over:
            assert [(p + s, p + e) for s, e in ms] == g.matches(p, p + len(line))  # the restatement is the reference's
        want += [p << 16] if over else []
        want += [((p + s) << 16) | ((e - s) << 3) | 1 for s, e in ms]
        p += len(line) + 1
    with Plan("[a-c]*d") as plan:
        assert 2 in plan.modes
        keys, _ = raw(plan, t.data_ptr(), km.Shard(text), 2)
    assert keys == sorted(want + [p << 16])  # the last line ("zz") holds the text's last byte


def xk(k):
    """k x's then y, written as x{255} blocks and a remainder (counts above 255 are refused)."""
    s = "x{255}" * (k // 255) + ("x{%d}" % (k % 255) if k % 255 else "")
    return s + "y"


def _largest(ok, lo, hi):
    """Largest k in [lo, hi) with ok(k), given ok(lo) and not ok(hi)."""
    assert ok(lo) and not ok(hi)
    while hi - lo > 1:
        mid = (lo + hi) // 2
        lo, hi = (mid, hi) if ok(mid) else (lo, mid)
    return lo


def test_automata_at_the_table_limits():
    L = lib.load()
    has_plan = lambda k: ru.filter_host(_params(xk(k)), b"") is not None  # noqa: E731
    matches = lambda k: L.krep_b200_regex_match_mode(_params(xk(k)).ref()) == 1  # noqa: E731
    k_plan = _largest(has_plan, 1, 8000)   # line table at the 4096-state / 32 KiB limit
    k_match = _largest(matches, 1, k_plan)  # match table just fits in what is left of 48 KiB
    assert 3000 < k_plan < 4096 and 2000 < k_match < k_plan, (k_plan, k_match)
    rng = random.Random(60)
    for k, want_modes in ((k_plan, [0, 1]), (k_match, [0, 1, 2]), (k_match + 1, [0, 1])):
        lines = []
        for r in (k - 1, k, k + 1, k, k - 1):
            lines += [b"x" * r + b"y", b"x" * r, b"ax" * 3 + b"x" * r + b"yy", b"y"]
        rng.shuffle(lines)
        text = b"\n".join(lines) + b"\n"
        t = to_device(text)
        with Plan(xk(k)) as plan:
            assert plan.modes == want_modes, (k, plan.modes)
            out = run_shard(plan, t.data_ptr(), km.Shard(text), budget_free=True, what=k)
            assert out[1][1] >= 4  # the deepest states were reached and accepted
    # many byte classes: a literal of 76 distinct bytes gives each its own column of the table
    lit = "0123456789ABCDEFGHIJKLMNOPQRSTUVWXYZabcdefghijklmnopqrstuvwxyz_-~!@#%&=:;,<>"
    assert len(set(lit)) == 76
    body = []
    for _ in range(3000):
        r = rng.random()
        if r < 0.1:
            body.append(lit)
        elif r < 0.5:
            body.append(lit[: rng.randint(1, 75)])
        else:
            body.append("".join(rng.choice(lit) for _ in range(rng.randint(0, 40))))
        body.append(rng.choice([" ", "\n", ""]))
    text = "".join(body).encode()
    t = to_device(text)
    with Plan(lit) as plan:
        assert plan.modes == [0, 1, 2]
        run_shard(plan, t.data_ptr(), km.Shard(text), budget_free=True, what="classes")
    with Plan(lit[:40] + "[a-f]*" + lit[40:], case_sensitive=False) as plan:
        run_shard(plan, t.data_ptr(), km.Shard(text), what="classes -i")


def _fresh_context():
    """Drops the engine's contexts, so the next scan starts with the initial occurrence list (2^20 keys)."""
    L = lib.load()
    L.krep_b200_shutdown()
    assert L.krep_b200_init(0) == 0, L.krep_b200_last_error_string()


@pytest.mark.parametrize("size", ["rank", "radix", "overflow"])
def test_list_sizes(size):
    # up to 16 384 keys the finish kernel's rank sort orders them, beyond that the radix sort; beyond the initial list
    # of 2^20 keys the scan overflows and runs again in the same mode on a grown list.  The hook gets room for every key
    # on its first call, so the keys compared with the model are those of that call: after a fresh context, of the
    # overflow's re-scan.  The count mode cannot overflow here (it leaves a key per uncertain line only, and more than
    # 2^20 of those would take gigabytes of lines longer than 4 KiB): its counter is checked on the grown list.
    corpus = lib.corpus_host(lib.make_spec(*SPEC), 0, 2 << 20)
    n = {"rank": 9000, "radix": 200000, "overflow": 2 << 20}[size]
    cases = [(corpus[:n], "x*", 2)]  # an (empty or x-run) match at every byte
    if size != "rank":
        cases.append((b"a\n" * (3 * n // 4) + b"a", "a", 0))  # a flagged line every 2 bytes
    for text, pat, mode in cases:
        if size == "overflow":
            _fresh_context()
        t = to_device(text)
        with Plan(pat) as plan:
            sh = km.Shard(text)
            keys, dl = raw(plan, t.data_ptr(), sh, mode, cap=4 << 20)
            oracle = km.HookLines(plan.P, text, plan.P if mode == 2 else None)
            km.check(km.expect(sh, mode, oracle.flagged if mode == 0 else oracle, budget_free=True), keys, dl, (size, mode))
            lo, hi = {"rank": (0, 16384), "radix": (16384, 1 << 20), "overflow": (1 << 20, 1 << 30)}[size]
            assert lo < len(keys) <= hi, (size, mode, len(keys))
            k1, dl1 = raw(plan, t.data_ptr(), sh, 1)  # the count mode's line counter, after the list grew
            km.check(km.expect(sh, 1, oracle), k1, dl1, (size, 1))


def test_global_offsets():
    rng = random.Random(70)
    text = geometry_text(rng, 3000)
    t = to_device(text)
    for G in (0, (1 << 32) - 8, (1 << 40) + 16, (1 << 48) - 1 - len(text)):
        for pat in ("a+b", "x*"):
            with Plan(pat) as plan:
                run_shard(plan, t.data_ptr(), km.Shard(text, 0, len(text), G), budget_free=pat in BUDGET_FREE, what=G)
    L = lib.load()
    with Plan("a+b") as plan:
        for G, ok in (((1 << 48) - 1 - len(text), True), ((1 << 48) - len(text), False)):
            shard = Shard(t.data_ptr(), len(text), 0, len(text), G, -1, -1)
            keys = (C.c_uint64 * 4096)()
            rc = L.krep_b200_regex_scan_shard_raw(plan.h, C.byref(shard), 2, keys, 4096, None)
            assert (rc > 0) == ok, (G, rc)
            if ok:
                assert all(((keys[i] >> 16) >> 47) == 1 for i in range(min(rc, 4096)))
            L.krep_b200_last_error()
            # the other modes have no such limit
            assert L.krep_b200_regex_scan_shard_raw(plan.h, C.byref(shard), 1, keys, 4096, None) >= 0


def test_grid_stride_wrap():
    # 96 MiB of short lines: more segments than one pass of the grid covers (SMs x 8 CTAs x 256 threads x 256 bytes)
    import gpu_util as gu
    spec = lib.make_spec(*SPEC)
    n = 96 << 20
    text = lib.corpus_host(spec, 0, n)
    t = gu.device_corpus(spec, 0, n)
    last = text.rfind(b"\n", 0, n - 1) + 1
    for pat in ("the[a-z]*", "[tT]h[a-z]*"):
        with Plan(pat) as plan:
            assert plan.modes == [0, 1, 2]
            oracle = km.HookLines(plan.P, text, plan.P)
            sh = km.Shard(text)
            keys, dl = raw(plan, t.data_ptr(), sh, 1)
            assert keys == [last << 3]  # every line shorter than 4 KiB is decided on the device, but the last one
            assert dl == len(oracle.flagged - {last}) and dl > 1000
            keys, dl = raw(plan, t.data_ptr(), sh, 2)
            want = sorted([last << 16] + [(s << 16) | ((e - s) << 3) | 1 for s, e in oracle.pos if s < last])
            assert keys == want
