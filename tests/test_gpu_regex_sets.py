"""Split -E plans on the GPU (DESIGN §12.7): the raw keys of k_regex_lines' split instantiations against
tests/regex_kernel_model.py in every mode a plan admits, and krep_b200_regex_search, krep_b200_search_shards and
krep_b200_regex_search_batch on split plans against the reference's regex_search loop; the relinked CLI against the
stock CLI with -f pattern files."""
import ctypes as C
import os
import random
import string
import subprocess
import sys

import numpy as np
import pytest

from krep_b200 import lib
from krep_b200.abi import ALGO_REGEX, Params, Shard
import gpu_util as gu
import oracle_util as ou
import regex_kernel_model as km
import regex_util as ru

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu
UNBOUNDED = (1 << 64) - 1


@pytest.fixture(scope="module", autouse=True)
def _init():
    L = lib.load()
    assert L.krep_b200_init(0) == 0, L.krep_b200_last_error_string()


@pytest.fixture(autouse=True)
def _device_paths_on(monkeypatch):
    monkeypatch.delenv("KREP_B200_NO_FUSED_COUNT", raising=False)
    monkeypatch.delenv("KREP_B200_NO_DEVICE_MATCHES", raising=False)


def _params(pats, **kw):
    if isinstance(pats, str):
        pats = [pats]
    return Params([p.encode() for p in pats], regex=True, **kw)


def lower_words(rng, k):
    return ["".join(rng.choice(string.ascii_lowercase) for _ in range(rng.randint(8, 12))) for _ in range(k)]


def alnum_words(rng, k):
    return ["".join(rng.choice(string.ascii_letters + string.digits) for _ in range(rng.randint(6, 10))) for _ in range(k)]


def err_patterns(rng, k):
    return ["ERR%s[a-z]{4}[0-9]+ code=[a-z]+" % "".join(rng.choice(string.ascii_lowercase) for _ in range(3))
            for _ in range(k)]


def set_text(rng, words, n):
    """Lines of random bytes and words of the set (whole, cut, upper-cased), with NUL, '\\r' and 0x80-0xFF."""
    wide = bytes(range(0x80, 0x100, 7)) + b"\x00\t\r aAbBx09_.,;"
    out = bytearray()
    while len(out) < n:
        r = rng.random()
        if r < 0.3:
            w = rng.choice(words)
            out += w[: rng.randint(1, len(w))] if rng.random() < 0.3 else w
        elif r < 0.38:
            out += rng.choice(words).upper()
        elif r < 0.55:
            out += bytes(rng.choice(wide) for _ in range(rng.randint(1, 6)))
        else:
            out += ru.random_text(rng, rng.randint(1, 30)).replace(b"\n", b" ")
        out += rng.choice([b" ", b"", b"\n", b"\r\n", b"\n\n", b"the "])
    return bytes(out[:n])


def _sets():
    rng = random.Random(0x5E7)
    low = lower_words(rng, 120)
    errs = err_patterns(rng, 60)
    return {
        "lowercase": (low + ["the[a-z]*"], [w.encode() for w in low] + [b"the", b"thexx"]),
        "ERR": (errs, [b"ERR" + p[3:6].encode() + b"qwer77 code=ab" for p in errs]),
    }


SETS = _sets()


class RawPlan:
    """A regex plan handle (production, or split under a state cap) and the modes it admits."""

    def __init__(self, P, cap=None):
        L = lib.load()
        self.P = P
        self.h = L.krep_b200_plan_create(P.ref(), ALGO_REGEX) if cap is None else L.krep_b200_regex_plan_split(P.ref(), cap)
        L.krep_b200_last_error()
        self.name = L.krep_b200_plan_filter_name(self.h).decode() if self.h else None
        self.modes = [m for m in (0, 1, 2) if self.h and self._host(m, b"a\n") is not None]

    def _host(self, mode, text):
        L = lib.load()
        buf = C.create_string_buffer(text, len(text) + 1)
        cap = text.count(b"\n") * 64 + len(text) + 8
        keys = (C.c_uint64 * cap)()
        dl = C.c_uint64(0)
        k = L.krep_b200_regex_plan_host(self.h, mode, buf, len(text), UNBOUNDED, keys, cap, C.byref(dl))
        if k < 0:
            L.krep_b200_last_error()
            return None
        return list(keys[:k]), dl.value

    def flagged(self, text):
        return set(k >> km.LIT_TAG_BITS for k in self._host(0, text)[0])

    def close(self):
        if self.h:
            lib.load().krep_b200_plan_destroy(self.h)


def raw(plan, ptr, sh, mode):
    L = lib.load()
    shard = Shard(ptr, sh.avail, sh.own_begin, sh.own_end, sh.global_offset, sh.prev_byte, sh.next_byte)
    cap = 1 << 16
    while True:
        keys = np.zeros(cap, dtype=np.uint64)
        dl = C.c_uint64(12345)
        k = L.krep_b200_regex_scan_shard_raw(plan.h, C.byref(shard), mode, keys.ctypes.data_as(C.POINTER(C.c_uint64)), cap,
                                             C.byref(dl))
        assert k >= 0, (k, L.krep_b200_last_error_string())
        if k <= cap:
            return keys[:k].tolist(), dl.value
        cap = k


def run_shard(plan, ptr, sh, budget_free=False, what=""):
    """Hook vs model in every mode the plan admits (verdicts and matches from glibc on the shard's own bytes)."""
    oracle = km.GlibcLines(plan.P, sh.buf)
    for mode in plan.modes:
        keys, dl = raw(plan, ptr, sh, mode)
        exp = km.expect(sh, mode, plan.flagged(sh.buf) if mode == 0 else oracle, budget_free)
        km.check(exp, keys, dl, (what, mode, plan.name, sh.own_begin, sh.own_end, sh.avail, sh.global_offset))


def short_lines_text(rng, n):
    out = bytearray()
    while len(out) < n:
        out += ru.random_text(rng, rng.randint(0, km.BUDGET_FREE_LEN)).replace(b"\n", b"") + b"\n"
    return bytes(out[:n])


def test_forced_splits_raw_keys():
    """Random alternations split into 2..8 automata by a low state cap, over tilings of one text."""
    rng = random.Random(0x5917)
    text = short_lines_text(rng, 20000)
    t = gu.to_device(text)
    done, names = 0, set()
    while done < 40:
        branches = [ru.random_regex(rng) for _ in range(rng.randint(2, 10))]
        try:
            P = _params(branches, case_sensitive=rng.random() < 0.8)
        except ValueError:
            continue
        for cap in (4, 6, 8, 12, 20):
            plan = RawPlan(P, cap)
            if plan.name and "split" in plan.name:
                break
            plan.close()
        else:
            continue
        try:
            names.add(plan.name)
            run_shard(plan, t.data_ptr(), km.Shard(text), budget_free=True, what=branches)
            cuts = sorted(rng.sample(range(1, len(text)), rng.randint(1, 5)))
            for d, sh in km.tiling(text, cuts, rng):
                run_shard(plan, t.data_ptr() + d, sh, budget_free=True, what=(branches, d))
            done += 1
        finally:
            plan.close()
    assert {"regex-lines-split", "regex-lines-split-widened"} <= names, names


def test_geometry_sweep():
    """Every line start residue and length, long lines past the walk's reach, and shards cut anywhere."""
    rng = random.Random(77)
    text = km.random_lines_text(rng, 60000)
    t = gu.to_device(text)
    for branches, cap in ((["ab", "b$", "^c", "a[0-9]", "ba+c"], 6), (["(ab|ba)c?", "c{2}", "b$", "^$"], 6)):
        plan = RawPlan(_params(branches), cap)
        try:
            assert plan.name and "split" in plan.name, (branches, plan.name)
            run_shard(plan, t.data_ptr(), km.Shard(text), what=branches)
            for k in range(4):
                cuts = sorted(rng.sample(range(1, len(text)), 3))
                for d, sh in km.tiling(text, cuts, rng):
                    run_shard(plan, t.data_ptr() + d, sh, what=(branches, k, d))
        finally:
            plan.close()


@pytest.mark.parametrize("name,make,modes", [
    ("200 lowercase + the[a-z]*", lambda rng: lower_words(rng, 200) + ["the[a-z]*"], [0, 1, 2]),
    ("200 alphanumeric", lambda rng: alnum_words(rng, 200), [0, 1]),
])
def test_sets_at_the_image_budget(name, make, modes):
    rng = random.Random(name)
    pats = make(rng)
    P = _params(pats)
    plan = RawPlan(P)
    try:
        assert plan.name == "regex-lines-split" and plan.modes == modes, (plan.name, plan.modes)
        text = set_text(rng, [p.encode() for p in pats if "[" not in p], 200000)
        t = gu.to_device(text)
        run_shard(plan, t.data_ptr(), km.Shard(text), what=name)
        for d, sh in km.tiling(text, sorted(rng.sample(range(1, len(text)), 3)), rng):
            run_shard(plan, t.data_ptr() + d, sh, what=(name, d))
    finally:
        plan.close()


def test_global_offsets_up_to_the_key_limit():
    pats, words = SETS["lowercase"]
    rng = random.Random(48)
    text = set_text(rng, words, 30000)
    t = gu.to_device(text)
    plan = RawPlan(_params(pats))
    try:
        assert plan.modes == [0, 1, 2]
        for go in (1 << 40, (1 << 48) - len(text) - 16 * 9):
            go &= ~15
            run_shard(plan, t.data_ptr(), km.Shard(text, global_offset=go, prev_byte=10), what=go)
    finally:
        plan.close()


OPTS = [dict(), dict(count=True), dict(count=True, only_matching=True), dict(only_matching=True),
        dict(case_sensitive=False), dict(case_sensitive=False, count=True), dict(whole_word=True),
        dict(whole_word=True, count=True), dict(max_count=1), dict(max_count=2), dict(max_count=3), dict(max_count=7)]


def _want(P, text):
    chk = ou.reference()
    if chk is None:
        return ru.ref_regex_search(P, text)
    f = chk.lib.regex_search
    f.argtypes = ou._SIG
    f.restype = C.c_uint64
    res = chk._new(16)
    try:
        cnt = f(P.ref(), C.create_string_buffer(text, len(text) + 1).raw, len(text), res)
        r = res.contents
        return int(cnt), [(r.positions[i].start_offset, r.positions[i].end_offset) for i in range(r.count)]
    finally:
        chk._free(res)


@pytest.mark.parametrize("set_name", list(SETS))
def test_search_on_host_text_larger_than_a_chunk(set_name, monkeypatch):
    monkeypatch.setenv("KREP_B200_CHUNK_MB", "1")
    monkeypatch.setenv("KREP_B200_STAGE_MB", "1")
    pats, words = SETS[set_name]
    L = lib.load()
    assert L.krep_b200_regex_automata(_params(pats).ref()) >= 2
    assert L.krep_b200_regex_count_mode(_params(pats, count=True).ref()) == 1
    assert L.krep_b200_regex_match_mode(_params(pats).ref()) == 1
    rng = random.Random(set_name)
    text = set_text(rng, words, (2 << 20) + 777)
    for kw in OPTS:
        P = _params(pats, **kw)
        want = _want(P, text)
        got = lib.search("regex", P, text)
        assert got[0] == want[0] and got[1] == (want[1] if P.struct.track_positions else []), (set_name, kw, got[0], want[0])


@pytest.mark.parametrize("n_shards", [1, 4])
def test_search_shards(n_shards):
    pats, words = SETS["lowercase"]
    rng = random.Random(n_shards)
    text = set_text(rng, words, 300000)
    cuts = sorted(rng.sample(range(1, len(text)), n_shards - 1))
    for kw in (dict(), dict(count=True), dict(case_sensitive=False), dict(max_count=3), dict(whole_word=True)):
        P = _params(pats, **kw)
        shards = [sh for _, sh in km.tiling(text, cuts, rng)]
        bufs = [gu.to_device(sh.buf) for sh in shards]
        structs = [Shard(b.data_ptr(), sh.avail, sh.own_begin, sh.own_end, sh.global_offset, sh.prev_byte, sh.next_byte)
                   for b, sh in zip(bufs, shards)]
        L = lib.load()
        h = L.krep_b200_plan_create(P.ref(), ALGO_REGEX)
        lib.check(L)
        try:
            got = lib.search_shards(h, P, structs)
        finally:
            L.krep_b200_plan_destroy(h)
        want = ru.ref_regex_search(P, text)
        assert got == (want[0], want[1] if P.struct.track_positions else []), (n_shards, kw, got[0], want[0])


def test_regex_search_batch():
    pats, words = SETS["ERR"]
    rng = random.Random(99)
    texts = [set_text(rng, words, rng.choice([0, 1, 50, 3000, 40000])) for _ in range(60)]
    for kw in (dict(), dict(count=True), dict(count=True, only_matching=True), dict(max_count=2), dict(case_sensitive=False)):
        P = _params(pats, **kw)
        got = lib.regex_search_batch(P, texts)
        for i, t in enumerate(texts):
            want = ru.ref_regex_search(P, t)
            assert got[i] == (want[0], want[1] if P.struct.track_positions else []), (kw, i)


CLI_FLAGS = [["-c"], ["-o"], ["-c", "-i"], ["-w"], ["-c", "-w"], [], ["-c", "-m", "3"]]


def test_cli_pattern_file(tmp_path):
    sys.path.insert(0, os.path.join(ROOT, "krep_b200", "shim"))
    sys.path.insert(0, os.path.join(ROOT, "oracle"))
    import build_krep_gpu
    import build_oracle
    stock = build_oracle.build_ref()[1]
    gpu = build_krep_gpu.build()
    if not stock or not gpu:
        pytest.skip("stock or GPU-backed krep binary not available (built only where the reference sources are)")
    env = {k: v for k, v in os.environ.items() if k != "KREP_B200_KEEP_VISIBLE"}
    for set_name, (pats, words) in SETS.items():
        assert lib.load().krep_b200_regex_automata(_params(pats).ref()) >= 2
        pf = tmp_path / (set_name + ".txt")
        pf.write_text("\n".join(pats) + "\n")
        rng = random.Random(set_name + "cli")
        body = set_text(rng, words, 400000).replace(b"\x00", b" ")
        data = tmp_path / (set_name + ".data")
        data.write_bytes(body.rstrip(b"\n") + b"\n")
        for flags in CLI_FLAGS:
            a = subprocess.run([stock, "-t", "1", "--color=never", *flags, "-E", "-f", str(pf), str(data)], capture_output=True)
            b = subprocess.run([gpu, "--color=never", *flags, "-E", "-f", str(pf), str(data)], capture_output=True, env=env)
            assert (b.returncode, b.stdout) == (a.returncode, a.stdout), (set_name, flags, a.stdout[:200], b.stdout[:200],
                                                                          b.stderr[:300])


def _spread(pad, *branches):
    """branches with 100 padding literals between each two: more than one automaton holds, so every branch sits in a
    group of its own."""
    out = [branches[0]]
    for k, b in enumerate(branches[1:]):
        out += pad[100 * k: 100 * (k + 1)] + [b]
    return out


def test_longest_end_over_groups_and_large_match_tables():
    """The union's match ends at the longest end of any automaton, whichever group holds that branch; and a group whose
    match automaton has 2^13 x 6 entries, close to the 16-bit limit of its row offsets."""
    rng = random.Random(0x10E)
    pad = lower_words(random.Random(0xA11), 300)
    big = "(" + "|".join(["zzzzzzzz"] * 500) + ")"
    cases = [(_spread(pad, "xa", "xab", "xabc"), b"xabc xab xa zxabcxab"), (_spread(pad, "xabc", "xab", "xa"), b"xabcxabxa"),
             (_spread(pad, "^ab", "b$", "abc$"), b"abc abcab xabc"), (_spread(pad, "q", "^q*$", "qq"), b"q qq qqq xqq"),
             ([big, big, "q", "q[gh]*g[gh]{12}"], b"qgghghghhhggghhgghhhghhggghg x q qgh")]
    for branches, alphabet in cases:
        P = _params(branches)
        L = lib.load()
        assert L.krep_b200_regex_automata(P.ref()) >= 2
        plan = RawPlan(P)
        try:
            assert plan.modes == [0, 1, 2], (branches[0], plan.modes)
            lines = [bytes(rng.choice(alphabet) for _ in range(rng.randint(0, 25))) for _ in range(3000)]
            text = b"\n".join(lines) + b"\n"
            t = gu.to_device(text)
            run_shard(plan, t.data_ptr(), km.Shard(text), budget_free=True, what=branches[0])
            for kw in (dict(), dict(max_count=5), dict(count=True)):
                Pk = _params(branches, **kw)
                want = ru.ref_regex_search(Pk, text)
                assert want[0] > 0
                assert lib.search("regex", Pk, text) == (want[0], want[1] if Pk.struct.track_positions else []), kw
        finally:
            plan.close()
