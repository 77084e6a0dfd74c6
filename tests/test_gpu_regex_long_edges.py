"""The -E long-line pass (scan_regex_long.cu, DESIGN §12.8) where its bookkeeping turns over: krep_b200_regex_scan_shard_
long_raw against tests/regex_long_model.py exactly, in every mode the plan admits, with

  * slice records in several rounds at every split width (G = 1, 2, 4, 8), and in production at G = 8 on 2.35 GiB;
  * random regexes and forced splits at slice / checkpoint sizes from 1 / 1 to 2^20 / 1024, with lines of k*S - 1,
    k*S and k*S + 1 bytes; the refused sizes;
  * a work list as dense as the geometry allows, and compactions that remove thousands of keys;
  * split images above 48 KiB (the shared-memory opt-in) and automata at the line table's limits (deep uint16 rows).

The cases whose regime only the engine's trace shows (automata per plan, rounds per scan) run in a child process with
KREP_B200_TRACE=1, which the trace reads once per process; the parent asserts on the child's trace."""
import ctypes as C
import os
import random
import re
import subprocess
import sys
import types

import numpy as np
import pytest

from krep_b200 import lib
from krep_b200.abi import Params, Shard
import regex_kernel_model as km
import regex_long_model as lm
import regex_util as ru
import test_gpu_regex_shards as gs
from test_gpu_regex_kernel import _largest, xk
from test_gpu_regex_long import Plan, hook
from test_gpu_regex_sets import lower_words, set_text

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
UNBOUNDED = (1 << 64) - 1
KNOBS = ("KREP_B200_NO_FUSED_COUNT", "KREP_B200_NO_DEVICE_MATCHES", "KREP_B200_NO_LONG_LINES")
# anchored branches: every line can die, some stay live to their '\n', and `^x[a-z ]*y$` makes the slices' guesses
# disagree with the truth along the whole line.  Under a cap of 7 states no two neighbours share an automaton (the nine
# need more automata than a split plan holds), so the first k branches split into exactly k automata.
BRANCHES = ["^[^x]*kqk", "^x[a-z ]*y$", "^[b-e ]*a$", "^[^x]*jqj", "^c[b-e ]*,,$", "^[^x]*zqz", "^d[^,]*jj$", "^[^x]*wqw",
            "^e[a-z ]*,b$"]
SPLIT_CAP = 7
# (label, G, automata, branches, state cap): one plan per width of the pass
BUCKETS = [("G1", 1, 1, 3, None), ("G2", 2, 2, 2, SPLIT_CAP), ("G4", 4, 4, 4, SPLIT_CAP), ("G8", 8, 7, 7, SPLIT_CAP)]
ROUND_SIZES = [(1, 1), (1024, 1)]
RANDOM_SIZES = [(1, 1), (2, 1), (5, 5), (7, 3), (100, 7), (1024, 1), (4096, 4096), (1 << 20, 1024), (0, 0)]
BODY = np.frombuffer(b"bcde ", dtype=np.uint8)
GO = 1 << 44  # a large global offset (mode 2 keys hold offsets below 2^48)


@pytest.fixture(scope="module", autouse=True)
def _init():
    L = lib.load()
    assert L.krep_b200_init(0) == 0, L.krep_b200_last_error_string()


@pytest.fixture(autouse=True)
def _device_paths_on(monkeypatch):
    for k in KNOBS:
        monkeypatch.delenv(k, raising=False)


def _mark(label):
    """Tags the trace lines that follow (the child's stderr) with label."""
    sys.stderr.write("@@ %s\n" % label)
    sys.stderr.flush()


def _flagged(plan, buf, split):
    """Filter-mode oracle: starts of the lines the plan's automata flag, with unbounded reach (split plans: the host twin
    of the split plan itself)."""
    if not split:
        return km.HookLines(plan.P, buf).flagged
    L = lib.load()
    b = C.create_string_buffer(bytes(buf), len(buf) + 1)
    cap = bytes(buf).count(b"\n") + 2
    keys = (C.c_uint64 * cap)()
    k = L.krep_b200_regex_plan_host(plan.h, 0, b, len(buf), UNBOUNDED, keys, cap, None)
    assert 0 <= k <= cap, (k, L.krep_b200_last_error_string())
    return set(v >> km.LIT_TAG_BITS for v in keys[:k])


def compare(plan, shards, sizes_list, split=False, big=False, budget_free=False, what=""):
    """The hook against the model for every shard, admitted mode and size.  big: verdicts and matches from the host
    twins (tens of MB), else from glibc line by line.  -> the last shard's models by mode."""
    exps = {}
    for sh in shards:
        res = gs.Resident([sh])
        st = res.structs[0]
        if big:
            oracle = km.HookLines(plan.P, sh.buf, plan.P if 2 in plan.modes else None)
        else:
            oracle = km.GlibcLines(plan.P, sh.buf)
        for mode in plan.modes:
            exp = lm.expect(sh, mode, _flagged(plan, sh.buf, split) if mode == 0 else oracle, budget_free)
            exps[mode] = exp
            for sizes in sizes_list:
                keys, dl = hook(plan, st, mode, sizes, cap=len(exp.keys) + 1024)
                lm.check(exp, keys, dl, (what, plan.P.patterns[:2], mode, sizes, sh.own_begin, sh.own_end, sh.avail,
                                         sh.global_offset, sh.prev_byte, sh.next_byte))
        del res
    return exps


def tiled(text, d, ob, go=GO):
    """The shard that owns text from d + ob on (d a multiple of 16), at global offset go + d, with the byte before."""
    return km.Shard(text[d:], ob, len(text) - d, go + d, text[d - 1] if d else -1, -1)


def _body(g, n):
    return BODY[g.integers(0, len(BODY), n)].tobytes() if n > 0 else b""


def mixed_line(g, n):
    """A line of n >= 8 content bytes that the BRANCHES decide at its start, in its last bytes, midway, or only at its
    '\\n', or whose slices' guesses never agree with the truth."""
    k = int(g.integers(0, 8))
    if k == 0:
        return b"kqk" + _body(g, n - 3)                                  # matched at once
    if k == 1:
        return b"b" + _body(g, n - 4) + b"kqk"                           # matched in its last bytes only
    if k == 2:
        return b"x," + _body(g, n - 2)                                   # DEAD at once
    if k == 3:
        h = int(g.integers(1, n - 1))
        return b"b" + _body(g, h - 1) + b"x" + _body(g, n - h - 1)       # DEAD midway
    if k == 4:
        return b"x" + _body(g, n - 2) + b"y"                             # live to its '\n', then matched; guesses disagree
    if k == 5:
        return b"x" + _body(g, n - 2) + b"z"                             # live to its '\n', no match
    if k == 6:
        return b"b" + _body(g, n - 2) + b"a"                             # `a$`
    return _body(g, n)


def rounds_text(g, G):
    """Long mixed lines (and a few short ones) with enough bytes in lines past the reach that the slices of ROUND_SIZES
    fill more than two rounds of records at width G."""
    need = 0
    for S, Ck in ROUND_SIZES:
        per_round = lm.REC_BYTES // (((S + Ck - 1) // Ck + 1) * G * 2)
        need = max(need, (2 * per_round + 1) * S)
    parts, long_bytes = [], 0
    while long_bytes < need * 1.06:
        if g.random() < 0.15:
            parts.append(_body(g, int(g.integers(0, 200))) + b"\n")
        else:
            n = int(g.integers(km.REGEX_SEG + km.REGEX_HALO + 1, 40000))
            parts.append(mixed_line(g, n) + b"\n")
            long_bytes += n
    return b"".join(parts) + b"kqk\n"


def _child_init():
    L = lib.load()
    assert L.krep_b200_init(0) == 0, L.krep_b200_last_error_string()
    for k in KNOBS:
        os.environ.pop(k, None)


def _case_rounds():
    """Case run in a child: several record rounds at every width."""
    _child_init()
    g = np.random.default_rng(0x20D5)
    for label, G, na, nb, cap in BUCKETS:
        _mark(label)
        plan = Plan(["|".join(BRANCHES[:nb])], max_states=cap)
        try:
            assert plan.h and plan.modes == [0, 1, 2], (label, plan.modes)
            text = rounds_text(g, G)
            shards = [km.Shard(text, next_byte=ord("z")), tiled(text, 4800, 5)]
            for sh in shards:
                for S, Ck in ROUND_SIZES:
                    z = lm.sizes(sh.avail, sh.own_end - sh.own_begin, na, S, Ck)
                    used = lm.slices_needed(sh, S)
                    assert used > 2 * z.round_slices and z.rounds >= 3, (label, S, Ck, used, z)
            compare(plan, shards, ROUND_SIZES, split=cap is not None, big=True, budget_free=True, what=label)
        finally:
            plan.close()
        print(label, len(text), "bytes")
    print("case ok")


def production_text(L, n, mean, seed):
    """n bytes of the synthetic corpus on the device, its newlines respaced to lines of mean/2 .. 3*mean/2 bytes."""
    import torch
    spec = lib.make_spec(0x5EED0001, 0x5EED0002, 1 << 10, b"the")
    t = torch.empty(n + 64, dtype=torch.uint8, device="cuda")
    assert L.krep_b200_corpus_generate(C.byref(spec), t.data_ptr(), 0, n, None) == 0, L.krep_b200_last_error_string()
    v = t[:n]
    v[v == 10] = 32
    gen = torch.Generator(device="cuda").manual_seed(seed)
    gaps = torch.randint(mean // 2, mean + mean // 2 + 1, (n // mean + 2,), device="cuda", generator=gen)
    pos = torch.cumsum(gaps, 0)
    v[pos[pos < n]] = 10
    torch.cuda.synchronize()
    return t


def _case_production():
    """Case run in a child: a resident shard of long lines at production sizes and G = 8, in at least 3 rounds."""
    _child_init()
    L = lib.load()
    pats = lower_words(random.Random(300), 300) + ["the[a-z]*"]
    Pc = Params([p.encode() for p in pats], regex=True, count=True)
    assert L.krep_b200_regex_automata(Pc.ref()) == 5 and L.krep_b200_regex_count_mode(Pc.ref()) == 1
    per_round = lm.sizes(1 << 40, 1 << 40, 5).round_slices
    n = (5 * per_round // 2) * lm.SLICE
    t = production_text(L, n, 64 << 10, 77)
    t[n:] = 0
    host = t.cpu().numpy()
    sh = types.SimpleNamespace(buf=host[:n], avail=n, own_begin=0, own_end=n, global_offset=0, prev_byte=-1, next_byte=-1)
    z = lm.sizes(n, n, 5)
    used = lm.slices_needed(sh)
    assert used > 2 * z.round_slices and z.rounds >= 3, (n, used, z)
    plan = Plan(pats)
    try:
        shard = Shard(t.data_ptr(), n, 0, n, 0, -1, -1)
        want = L.krep_b200_regex_count_host(Pc.ref(), host.ctypes.data, n, UNBOUNDED)
        assert want > 0
        cap = int(np.count_nonzero(host[:n] == 10)) + 2
        flagged = np.zeros(cap, dtype=np.uint64)
        k = L.krep_b200_regex_filter_host(plan.P.ref(), host.ctypes.data, n, flagged.ctypes.data_as(C.POINTER(C.c_uint64)),
                                          cap, None)
        assert 0 <= k <= cap, k
        exp = lm.expect(sh, 0, set(flagged[:k].tolist()))
        _mark("production")
        got = lib.search_shards(plan.h, Pc, [shard], with_result=False)[0]
        assert got == want, (got, want)
        keys, dl = hook(plan, shard, 0, cap=len(exp.keys) + 1024)
        lm.check(exp, keys, dl, "production filter")
        print("production", n, "bytes,", len(lm.taken_lines(sh)), "long lines,", used, "slices,", want, "lines counted")
    finally:
        plan.close()
    print("case ok")


def _case_images():
    """Case run in a child: a split image above 48 KiB (the opt-in of slices, chain and match) over long lines."""
    _child_init()
    rng = random.Random(0x1A6E)
    pats = lower_words(random.Random(200), 200) + ["the[a-z]*"]
    words = [p.encode() for p in pats[:-1]]
    parts = []
    for _ in range(160):
        parts.append(set_text(rng, words, rng.choice([4353, 4400, 5000, 8192, 9000, 20000])).replace(b"\n", b" ") + b"\n")
        parts.append(set_text(rng, words, rng.randint(1, 300)))
    text = b"".join(parts)
    _mark("images")
    plan = Plan(pats)
    try:
        assert plan.modes == [0, 1, 2], plan.modes
        sh = km.Shard(text, next_byte=ord("z"))
        assert len(lm.taken_lines(sh)) > 100
        compare(plan, [sh, tiled(text, 160, 3)], [(0, 0), (64, 16)], big=True, what="images")
    finally:
        plan.close()
    print("case ok")


def run_child(case):
    """Runs case in a fresh process with the trace on. -> {label: [trace lines]}"""
    env = dict(os.environ, KREP_B200_TRACE="1",
               PYTHONPATH=os.pathsep.join([HERE, os.path.dirname(HERE), os.environ.get("PYTHONPATH", "")]))
    for k in KNOBS:
        env.pop(k, None)
    r = subprocess.run([sys.executable, "-c", "import test_gpu_regex_long_edges as t; t.%s()" % case], cwd=HERE, env=env,
                       capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0 and "case ok" in r.stdout, r.stdout[-2000:] + r.stderr[-4000:]
    out, cur = {}, None
    for line in r.stderr.splitlines():
        if line.startswith("@@ "):
            cur = line[3:].strip()
            out[cur] = []
        elif cur is not None and line.startswith("[krep_b200 "):
            out[cur].append(line)
    return out


AUTOMATA = re.compile(r"\] regex sets[a-z ]*: (\d+) automata, .* (\d+) bytes of shared memory")
SINGLE = re.compile(r"\] regex[a-z ]*: \d+ CTAs")
ROUNDS = re.compile(r"\] long lines: mode (\d), slices of (\d+) bytes, checkpoints every (\d+), (\d+) round")


def _automata(lines):
    return [(int(m.group(1)), int(m.group(2))) for m in map(AUTOMATA.search, lines) if m]


def _rounds(lines):
    return [tuple(int(x) for x in m.groups()) for m in map(ROUNDS.search, lines) if m]


def test_rounds_at_every_width():
    tr = run_child("_case_rounds")
    for label, G, na, nb, cap in BUCKETS:
        lines = tr[label]
        if G == 1:
            assert not _automata(lines) and any(SINGLE.search(s) for s in lines), lines[:4]
        else:
            assert {a for a, _ in _automata(lines)} == {na}, (label, lines[:4])
            assert lm.width(na) == G
        rounds = [r for r in _rounds(lines) if (r[1], r[2]) in ROUND_SIZES]
        # every mode at both sizes on both shards (a hook call whose keys overflow its buffer scans again), in at least
        # 3 rounds
        assert {(m, s) for m, s, _, _ in rounds} == {(m, s) for m in (0, 1, 2) for s, _ in ROUND_SIZES}, (label, rounds)
        assert len(rounds) >= 12 and min(r[3] for r in rounds) >= 3, (label, rounds)


def test_production_rounds_at_g8():
    tr = run_child("_case_production")
    lines = tr["production"]
    assert {a for a, _ in _automata(lines)} == {5}, lines[:4]
    rounds = _rounds(lines)
    assert {m for m, *_ in rounds} == {0, 1} and all(r[1:3] == (lm.SLICE, lm.CKPT) for r in rounds), rounds
    assert min(r[3] for r in rounds) >= 3, rounds


def test_split_images_above_48_kib():
    lines = run_child("_case_images")["images"]
    got = _automata(lines)
    assert {a for a, _ in got} == {3}, lines[:4]
    assert all(b > 48 * 1024 for _, b in got), got
    assert {m for m, *_ in _rounds(lines)} == {0, 1, 2}


def edge_text(rng, S):
    """lm.long_lines_text with lines of k*S - 1, k*S and k*S + 1 bytes just past the reach (the last slice one byte, or
    one byte short of a full slice)."""
    S = S or lm.SLICE
    k = max(1, -(-(km.REGEX_SEG + km.REGEX_HALO + 2) // S))
    text = lm.long_lines_text(rng, rng.randint(1000, 30000))
    lines = [bytes(rng.choice(b"abcx ,") for _ in range(min(n, 300))) * (n // 300 + 1) for n in (k * S - 1, k * S, k * S + 1)]
    lines = [ln[:n] for ln, n in zip(lines, (k * S - 1, k * S, k * S + 1))]
    rng.shuffle(lines)
    cut = text.find(b"\n", len(text) // 2) + 1
    return text[:cut] + b"\n".join(lines) + b"\n" + text[cut:]


def edge_shards(rng, text):
    """The whole text (with and without a byte after it), and two shards of a random cut, the second at a large global
    offset."""
    cut = rng.randint(1, len(text) - 1)
    d = cut & ~15
    first = km.Shard(text[: min(len(text), cut + km.REGEX_HALO)], 0, cut, 0, -1,
                     text[cut + km.REGEX_HALO] if cut + km.REGEX_HALO < len(text) else -1)
    return [km.Shard(text), km.Shard(text, next_byte=ord("z")), first, tiled(text, d, cut - d)]


def test_random_regexes():
    rng = random.Random(0x7A11)
    done = splits = 0
    while done < 150:
        pats = [ru.random_regex(rng) for _ in range(rng.choice([1, 1, 2]))]
        icase = rng.random() < 0.3
        try:
            plan = Plan(pats, case_sensitive=not icase)
        except ValueError:
            continue
        try:
            if not plan.h:
                continue
            S, Ck = rng.choice(RANDOM_SIZES)
            text = edge_text(rng, S)
            big = S == 1 << 20  # lines of 1 MiB: verdicts and matches from the host twins
            compare(plan, edge_shards(rng, text), [(S, Ck)], big=big, what=(done, icase))
            done += 1
        finally:
            plan.close()
    while splits < 40:
        branches = [ru.random_regex(rng) for _ in range(rng.randint(2, 6))]
        icase = rng.random() < 0.3
        plan = None
        for cap in (4, 6, 8, 12, 20):
            try:
                plan = Plan(["|".join(branches)], max_states=cap, case_sensitive=not icase)
            except ValueError:
                break
            if plan.h and "split" in lib.load().krep_b200_plan_filter_name(plan.h).decode():
                break
            plan.close()
            plan = None
        if plan is None:
            continue
        try:
            S, Ck = rng.choice(RANDOM_SIZES[:-2] + RANDOM_SIZES[-1:])
            text = edge_text(rng, S)
            compare(plan, edge_shards(rng, text), [(S, Ck), (0, 0)], split=True, what=("split", splits, branches))
            splits += 1
        finally:
            plan.close()


def test_refused_sizes():
    L = lib.load()
    plan = Plan("a[^x]*b")
    try:
        rng = random.Random(4)
        text = edge_text(rng, 1024)
        sh = km.Shard(text)
        res = gs.Resident([sh])
        keys = np.zeros(16, dtype=np.uint64)
        for S, Ck in (((1 << 20) + 1, 1), ((1 << 20) + 1, 1 << 20), (16, 17), (1025, 1), (2048, 1)):
            n0 = L.krep_b200_launch_count()
            k = L.krep_b200_regex_scan_shard_long_raw(plan.h, C.byref(res.structs[0]), 1, S, Ck,
                                                      keys.ctypes.data_as(C.POINTER(C.c_uint64)), 16, None)
            assert k == -3 and L.krep_b200_launch_count() == n0, (S, Ck, k)
            L.krep_b200_last_error()
        # the engine scans on after a refusal, at the largest admitted sizes among others
        compare(plan, [sh], [(1 << 20, 1024), (1024, 1), (1, 1)], what="after refusals")
    finally:
        plan.close()


def dense_text(g, ob, own_bytes, short=0.0):
    """Lines that each end one byte past the reach from their own start (4352 - o content bytes for a start at offset o
    of its 256-byte segment, counted from own_begin = ob), half of them with a match; with probability `short` a short
    matched line in between.  -> text, whose owned range starts at ob."""
    parts, p = [b"q" * (ob - 1) + b"\n"], ob
    while p - ob < own_bytes:
        if g.random() < short:
            parts.append(b"kqk\n")
            p += 4
            continue
        n = km.REGEX_SEG + km.REGEX_HALO - (p - ob) % km.REGEX_SEG
        ln = _body(g, n)
        if g.random() < 0.5:
            i = int(g.integers(0, n - 3))
            ln = ln[:i] + b"kqk" + ln[i + 3:]
        parts.append(ln + b"\n")
        p += n + 1
    parts.append(b"end\n")
    return b"".join(parts)


@pytest.mark.parametrize("short", [0.0, 0.3])
def test_dense_work_list_and_compaction(short):
    g = np.random.default_rng(0xDE45 + int(short * 10))
    ob = 37
    text = dense_text(g, ob, 64 << 20, short)
    sh = km.Shard(text, ob, len(text), GO, ord("\n"), -1)
    plan = Plan("kqk|^x[a-z ]*y$")
    try:
        assert plan.modes == [0, 1, 2]
        z = lm.sizes(sh.avail, sh.own_end - sh.own_begin, 1)
        taken = lm.taken_lines(sh)
        if short == 0.0:
            assert len(taken) >= 0.9 * z.pick_cap, (len(taken), z.pick_cap)
        exps = compare(plan, [sh], [(0, 0), (7, 3)], big=True, budget_free=True, what=("dense", short))
        # count mode removes every taken key in one compaction, filter mode the unmatched ones, between kept keys
        starts = {p for p, _ in taken}
        kept = [k for k in exps[0].keys if (k >> km.LIT_TAG_BITS) - GO in starts]
        assert len(taken) > 1024 and len(taken) - len(kept) > 1024 and len(kept) > 1024, (len(taken), len(kept))
        assert exps[1].device_lines > 1024
    finally:
        plan.close()


def test_deep_rows_at_the_table_limits():
    has_plan = lambda k: ru.filter_host(Params([xk(k).encode()], regex=True), b"") is not None  # noqa: E731
    matches = lambda k: lib.load().krep_b200_regex_match_mode(Params([xk(k).encode()], regex=True).ref()) == 1  # noqa: E731
    k_plan = _largest(has_plan, 1, 8000)
    k_match = _largest(matches, 1, k_plan)
    rng = random.Random(61)
    for k, want_modes in ((k_plan, [0, 1]), (k_match, [0, 1, 2])):
        lines = []
        for r in (k - 1, k, k + 1):
            lines += [b"a" * 5000 + b"x" * r + b"y", b"a" * 5000 + b"x" * r, b"a" * 4999 + b"x" * r + b"yx" * 3, b"y"]
        rng.shuffle(lines)
        text = b"\n".join(lines) + b"\nz\n"
        plan = Plan(xk(k))
        try:
            assert plan.modes == want_modes, (k, plan.modes)
            sh = km.Shard(text)
            assert len(lm.taken_lines(sh)) == 9
            exps = compare(plan, [sh, tiled(text, 5008, 9)], [(0, 0), (16, 4), (4096, 4096)], what=k)
            assert exps[1].device_lines >= 2  # the deepest states were reached and accepted
        finally:
            plan.close()
