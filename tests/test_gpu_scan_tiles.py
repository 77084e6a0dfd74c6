"""-m gpu: the literal and pattern-set scans inside their streaming loops, key by key against tests/scan_model.py.

test_gpu_scan_keys.py holds every kernel to the model on buffers too small to enter a main loop, and at scale on noise
with one occurrence per 2 KiB.  The texts here (tests/scan_tiles.py) reach what those leave out: an occurrence at every
(lane, byte residue) pair of a warp vector, so every lane-to-lane window of k_lit_window4 and k_ac_scan<2> crosses its
shuffled word; near misses at every pattern byte; dense runs of self-overlapping needles on every CTA-tile and
grid-stride edge, at group 0 and in the last 24 bytes, where emit_warp's prefix sum carries up to 512 keys per warp
vector and k_ac_tri4's queue fills and takes re-pushed lookups; a whole k_ac_scan tile in which every group parks, so
a warp's queue takes a remainder plus a full iteration (AcQueue::CAP).  A mismatch names the kernel and the lane, residue,
warp, vector row, CTA tile and grid stride of the first differing key."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

import gpu_util as gu
import scan_model as sm
import scan_tiles as st
from test_gpu_scan_keys import FUSED_KINDS, KIND_IDS, KINDS, Plan, count_record, scan
from test_gpu_scan_keys import _init  # noqa: F401  (module fixture: init + count_lines_shard signature)

pytestmark = pytest.mark.gpu

# inner shard: own_begin off the 16-byte grid but in group 0, so every kernel's tiles (measured from group_begin) keep
# their edges where the dense runs straddle them; own_end = n - 29, avail_len = n - 5
INNER = (13, 29, 5)
INNER_GO = (1 << 30) + 7
INNER_CTX = (ord("a"), 0xE9)


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def where(plan, start, ob):
    tri4_tile = st.TRI4_768_TILE if os.environ.get("KREP_B200_AC_THREADS") == "768" else st.AC_TILE
    return st.where(plan.name, start, ob // 16, sms(), tri4_tile)


def _first_diff(got, want):
    """(key, 'missing' | 'extra') of the smallest key in one sorted list and not the other."""
    missing = np.setdiff1d(want, got, assume_unique=False)
    extra = np.setdiff1d(got, want, assume_unique=False)
    if missing.size and (not extra.size or missing[0] <= extra[0]):
        return int(missing[0]), "missing"
    if extra.size:
        return int(extra[0]), "extra"
    return None, "same keys, other multiplicity or order"


def check_tiles(plan, dev, buf, avail, ob, oe, go=0, prev=-1, nxt=-1, what=""):
    """check_scan with a failure message that says where in the streaming loop the first differing key lies."""
    want = plan.model(buf, avail, ob, oe, go, prev, nxt)
    cnt, keys, bounds, overflow = scan(plan, dev, avail, ob, oe, go, prev, nxt)
    assert overflow == 0 and want.size < (1 << 20), (what, plan.name, want.size, overflow)
    ctx = (what, plan.name, plan.func, plan.pats[:4], plan.cs, plan.ww, plan.o, avail, ob, oe, go, prev, nxt)
    if cnt != want.size or not np.array_equal(keys, want):
        key, how = _first_diff(keys, want)
        at = "" if key is None else where(plan, int(sm.key_starts([key], plan.is_ac)[0]) - go, ob)
        raise AssertionError(f"{what}: {plan.name}: count {cnt} vs model {want.size}; first differing key {key} ({how}): "
                             f"{at}\n{ctx}")
    if plan.bounds and want.size:
        wb = sm.line_bounds(want, buf, avail, go, prev, nxt, plan.is_ac)
        if not np.array_equal(bounds, wb):
            i = int(np.flatnonzero(bounds != wb)[0]) // 2
            s = int(sm.key_starts(want[i:i + 1], plan.is_ac)[0]) - go
            raise AssertionError(f"{what}: k_line_bounds behind {plan.name}: key {i}: {bounds[2 * i:2 * i + 2].tolist()} "
                                 f"vs model {wb[2 * i:2 * i + 2].tolist()}: {where(plan, s, ob)}\n{ctx}")
    return want


def count_only(plan, dev, avail, ob, oe, go=0, prev=-1, nxt=-1):
    return int(gu.scan(plan.h, dev, avail, ob, oe, go, prev, nxt, want_positions=False).count)


def case_of(kind, builder):
    return st.kind_case(kind, 11) if builder == "sweep" else st.dense_case(kind)


def run_case(case, builder, seed, what=""):
    """Whole shard and inner shard, keys + bounds and count-only; -> the plan's filter name."""
    func, pats, cs, ww, o = case
    n = st.TEXT_LEN
    buf = st.text_for(builder, pats, cs, n, sms(), seed, func == "aho_corasick")
    with Plan(func, pats, cs, ww, o, count=True) as plan:
        dev = gu.to_device(buf)
        want = check_tiles(plan, dev, buf, n, 0, n, what=f"{what}{builder} whole")
        assert want.size > sm.PACK_KEYS, want.size  # CUB sorts these lists
        assert count_only(plan, dev, n, 0, n) == want.size, (what, plan.name, "count-only whole")
        ob, oe, av = INNER[0], n - INNER[1], n - INNER[2]
        want = check_tiles(plan, dev, buf, av, ob, oe, INNER_GO, *INNER_CTX, what=f"{what}{builder} inner")
        assert count_only(plan, dev, av, ob, oe, INNER_GO, *INNER_CTX) == want.size, (what, plan.name, "count-only inner")
        del dev
        torch.cuda.empty_cache()
        return plan.name


@pytest.mark.parametrize("builder", ["sweep", "dense"])
@pytest.mark.parametrize("kind", KINDS, ids=KIND_IDS)
def test_keys_on_every_lane_and_tile_edge(kind, builder):
    """Every key and line bound of a 19 MiB shard and of an inner shard (owned range off the 16-byte grid, a global
    offset, context bytes), and the count of a count-only launch (tail_and_count's warp reduction under dense hits)."""
    run_case(case_of(kind, builder), builder, 1 + KINDS.index(kind))


@pytest.mark.parametrize("case", [c for _, c in st.DENSE_EXTRA], ids=[i for i, _ in st.DENSE_EXTRA])
def test_long_periodic_needles_in_dense_runs(case):
    """64- and 1024-byte periodic needles: k_lit_aligned4 verifies a long compare at every other offset of a run."""
    assert run_case(case, "dense", 77).startswith("aligned4")


@pytest.mark.parametrize("part_kb", ["2", None])
@pytest.mark.parametrize("builder", ["sweep", "dense"])
@pytest.mark.parametrize("fk", FUSED_KINDS, ids=[k[0] for k in FUSED_KINDS])
def test_fused_count_on_every_lane_and_tile_edge(fk, builder, part_kb, monkeypatch):
    """krep_b200_count_lines_shard's record on the same texts equals the model's line record, whole and inner shard,
    at the default partition and at 2 KiB."""
    if part_kb is None:
        monkeypatch.delenv("KREP_B200_COUNT_PART_KB", raising=False)
    else:
        monkeypatch.setenv("KREP_B200_COUNT_PART_KB", part_kb)
    kid, func, pat, cs, ww = fk
    if builder == "dense":
        pat = st.periodic(len(pat), ww, 1 + FUSED_KINDS.index(fk) % 2)
    n = st.TEXT_LEN
    buf = st.text_for(builder, [pat], cs, n, sms(), 3 + FUSED_KINDS.index(fk))
    with Plan(func, [pat], cs, ww, count=True) as plan:
        assert plan.shape.ww_mode != 2
        dev = gu.to_device(buf)
        ob, oe, av = INNER[0], n - INNER[1], n - INNER[2]
        for b, e, a in ((0, n, n), (ob, oe, av)):
            starts = sm.key_starts(plan.model(buf, a, b, e), False).astype(np.int64)
            want = sm.line_record(buf, b, e, starts)
            got = count_record(plan, dev.data_ptr(), a, b, e)
            assert got == want, (kid, builder, part_kb, plan.name, b, e, a, got, want)


# ------------------------------------------------------------------------------------------- AC knobs, fresh processes
KNOB_KINDS = ["ac-stride1", "ac-stride2", "ac-tri4", "ac-quad"]


def _tri4_kernels_launched():
    """Names of the k_ac_tri4 kernels one tri4 scan launches, as the CUDA profiler records them: the CTA size is a
    template argument (k_ac_tri4<FOLD, THREADS>), so this shows which KREP_B200_AC_THREADS the library took."""
    from torch.profiler import ProfilerActivity, profile
    case = st.kind_case(KINDS[KIND_IDS.index("ac-tri4")], 11)
    buf = st.text_for("sweep", case[1], case[2], 1 << 20, sms(), 5)
    with Plan(*case) as plan:
        dev = gu.to_device(buf)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            scan(plan, dev, len(buf), 0, len(buf))
            torch.cuda.synchronize()
    return sorted({e.name for e in prof.events() if "k_ac_tri4" in e.name})


def _knob_case():
    """The tri, quad, stride-1 and stride-2 cases under whatever KREP_B200_AC_THREADS / KREP_B200_AC_PF this process
    started with (both are read once per process)."""
    from krep_b200 import lib
    L = lib.load()
    assert L.krep_b200_init(0) == 0
    names = _tri4_kernels_launched()
    threads = "768" if os.environ.get("KREP_B200_AC_THREADS") == "768" else "640"
    got = {m.group(1) for m in (re.search(r"k_ac_tri4<\w+,\s*(\d+)>", n) for n in names) if m}
    assert got == {threads}, (threads, names)
    for kid in KNOB_KINDS:
        kind = KINDS[KIND_IDS.index(kid)]
        for builder in ("sweep", "dense"):
            run_case(case_of(kind, builder), builder, 1 + KINDS.index(kind), what=f"{kid} ")
    print("knobs ok")


@pytest.mark.parametrize("env", [{"KREP_B200_AC_THREADS": "768"}, {"KREP_B200_AC_PF": "0"}, {"KREP_B200_AC_PF": "64"}],
                         ids=["threads768", "pf0", "pf64"])
def test_pattern_set_knobs_in_a_fresh_process(env):
    """k_ac_tri4 at 768 threads (48 KiB tiles, 24 warp queues; the profiled kernel name shows the library took the
    setting), and the L2 prefetch off and further ahead than a CTA has tiles: the same keys as the model.  On these
    19 MiB texts a CTA has about 4 tiles, so KREP_B200_AC_PF=64 issues no prefetch at all: it checks that a distance
    past the end is harmless, and takes the same k_ac_tri4 path as KREP_B200_AC_PF=0; the prefetch distance itself
    has no observable other than time."""
    here = os.path.dirname(os.path.abspath(__file__))
    penv = dict(os.environ, PYTHONPATH=os.pathsep.join([here, os.path.dirname(here), os.environ.get("PYTHONPATH", "")]))
    penv.pop("KREP_B200_AC_THREADS", None)
    penv.pop("KREP_B200_AC_PF", None)
    penv.update(env)
    r = subprocess.run([sys.executable, "-c", "import test_gpu_scan_tiles as t; t._knob_case()"], cwd=here, env=penv,
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and "knobs ok" in r.stdout, r.stdout[-2000:] + r.stderr[-4000:]
