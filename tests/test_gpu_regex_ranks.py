"""-E over rank-resident shards (krep_b200/sharding.py, RegexRanks): every rank exports its own shard's row on the GPU and
resolves its own lines; rank 0's count and positions must equal krep_b200_regex_search on the whole host text.  World
sizes 2 and 3 over gloo with every process on the same GPU (each with its own resident shard), and world 1 over NCCL;
all three paths (fused -c, offsets on the device, line filter + regexec), both knobs, the cut kinds of
tests/regex_ranks_util.py, and a bad tiling that must fail on every rank without a hang."""
import os
import random

import pytest

import regex_kernel_model as km
import regex_ranks_util as rk
import regex_rows_util as rr
from test_regex_ranks_host import run_spawned

pytestmark = pytest.mark.gpu
KNOBS = ["KREP_B200_NO_FUSED_COUNT", "KREP_B200_NO_DEVICE_MATCHES"]


def cases(world):
    rng = random.Random(100 + world)
    out = []
    for name, text, cuts in rk.cut_texts(world):
        for pat, opts in rk.PATTERNS:
            for mode in rng.sample(rk.MODES, 3):
                out.append((name, pat, dict(opts, **mode), text, cuts, rng.choice(rk.HALOS), None))
    text = km.random_lines_text(rng, 40000).replace(b"x", b"the", 300)
    for pat, opts in rk.PATTERNS:
        for mode in rk.MODES:
            cuts = sorted(rng.sample(range(1, len(text)), world - 1))
            out.append(("random", pat, dict(opts, **mode), text, cuts, rng.choice(rk.HALOS), None))
    for knob in KNOBS:
        for pat, opts in [("the[a-z]*", dict(count=True)), ("the[a-z]*", dict()), ("^$", dict(max_count=3)),
                          ("x*", dict(count=True, only_matching=True))]:
            cuts = sorted(rng.sample(range(1, len(text)), world - 1))
            out.append(("knob", pat, opts, text, cuts, 17, knob))
    return out


def worker(rank, world, port, q):
    import torch
    import torch.distributed as dist
    import gpu_util as gu
    from krep_b200 import lib, sharding
    from krep_b200.abi import ALGO_REGEX, Shard
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    for k in KNOBS:
        os.environ.pop(k, None)
    torch.cuda.set_device(0)
    backend = "nccl" if world == 1 else "gloo"
    dist.init_process_group(backend, rank=rank, world_size=world)
    device = "cuda:0" if backend == "nccl" else "cpu"
    L = lib.load()
    bad, modes = [], set()
    try:
        assert L.krep_b200_init(0) == 0, L.krep_b200_last_error_string()
        ranks = sharding.RegexRanks(rank, world, device, capacity=256)  # small: the grow-and-export-again path runs
        for name, pat, opts, text, cuts, halo, knob in cases(world):
            P = rk.params(pat, **opts)
            if knob:
                os.environ[knob] = "1"
            sh = rr.tile(text, cuts, halo)[rank]
            buf = gu.to_device(sh.buf)
            st = Shard(buf.data_ptr(), sh.avail, sh.own_begin, sh.own_end, sh.global_offset, sh.prev_byte, sh.next_byte)
            plan = L.krep_b200_plan_create(P.ref(), ALGO_REGEX)
            lib.check(L)
            L.krep_b200_set_only_matching(bool(P.only_matching))
            try:
                got = ranks.search(plan, P, st)
                if rank == 0:
                    modes.add(rr.call_mode(P))
                    want = lib.search("regex", P, text)
                    got = (got[0], [tuple(x) for x in got[1].tolist()])
                    if got != want:
                        bad.append((name, pat, opts, halo, knob, got[0], want[0], got[1][:3], want[1][:3]))
                elif got is not None:
                    bad.append(("rank answered", rank))
            finally:
                L.krep_b200_set_only_matching(False)
                L.krep_b200_plan_destroy(plan)
                if knob:
                    os.environ.pop(knob, None)
        if rank == 0 and modes != {0, 1, 2}:
            bad.append(("paths not all taken", sorted(modes)))
        # a bad tiling fails on every rank, and none waits: the last rank's shard claims one byte less
        P = rk.params("the")
        text = b"the a\nthe b\nthe c\n" * 5
        sh = rr.tile(text, [16 * i for i in range(1, world)], 4)[rank]
        buf = gu.to_device(sh.buf)
        own_begin = sh.own_begin + (1 if rank == world - 1 else 0)
        st = Shard(buf.data_ptr(), sh.avail, own_begin, sh.own_end, sh.global_offset, sh.prev_byte, sh.next_byte)
        plan = L.krep_b200_plan_create(P.ref(), ALGO_REGEX)
        try:
            ranks.search(plan, P, st)
            bad.append(("bad tiling accepted", rank))
        except RuntimeError as e:
            if "tile" not in str(e):
                bad.append(("unexpected error", rank, str(e)))
        finally:
            L.krep_b200_plan_destroy(plan)
        dist.barrier()
    finally:
        dist.destroy_process_group()
    q.put((rank, bad))


@pytest.mark.parametrize("world", [1, 2, 3])
def test_ranks_equal_regex_search(world):
    out = run_spawned(worker, world, timeout=900)
    assert all(v == [] for v in out.values()), out
