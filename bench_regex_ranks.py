"""-E on a corpus sharded across ranks, one process per shard (krep_b200/sharding.py, RegexRanks): each rank generates
its own shard in HBM (krep_b200_corpus_generate, one `the` per KiB as in bench_regex_resident.py), exports its row,
resolves its own lines, and rank 0 gathers counts and positions.  The five calls of bench_regex_resident.py, best of
--steps after --warmup (a barrier before each call).  Reports per rank the export (scan + pack + row read-back, with the
scan and pack device times), the exchange and the resolve time, and rank 0's whole-call GB/s.  At one rank the count
and a digest of the positions are checked against krep_b200_search_shards on the same bytes.  Prints one JSON line
(rank 0).

  torchrun --nproc_per_node N bench_regex_ranks.py [--gib 10] [--steps 3] [--warmup 1] [--backend gloo]

The exchange moves host data (row headers, heads, answers), so the default transport is a gloo group on CPU tensors;
--backend nccl stages the same messages through each rank's GPU.  Ranks share the GPUs round-robin: on a box with one
GPU, N ranks are N processes on that GPU — what that measures is whether the host (glibc) time divides by N.

Writes nothing into the tree."""
import argparse
import ctypes as C
import hashlib
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (workload seeds)
from bench_regex import provenance  # noqa: E402
from bench_regex_resident import CASES, CORPUS  # noqa: E402
from krep_b200 import lib, sharding  # noqa: E402
from krep_b200.abi import ALGO_REGEX, Params, Shard  # noqa: E402

HALO = 4096


def digest(pos):
    """sha256 of the positions as little-endian (start, end) uint64 pairs — bench_regex_resident.digest's bytes."""
    return hashlib.sha256(pos.contiguous().numpy().astype("<u8").tobytes()).hexdigest()[:16]


def shards_answer(L, plan, P, shard, want_pos):
    arr = (Shard * 1)(shard)
    res = L.krep_b200_match_result_init(16) if want_pos else None
    try:
        cnt = L.krep_b200_search_shards(plan, P.ref(), arr, 1, res)
        lib.check(L)
        import torch
        return int(cnt), (sharding._result_positions(res) if res else torch.zeros((0, 2), dtype=torch.int64))
    finally:
        if res:
            L.krep_b200_match_result_free(res)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gib", type=float, default=10.0)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--backend", default="gloo", choices=["gloo", "nccl"])
    ap.add_argument("--cases", default=",".join(CASES))
    a = ap.parse_args()
    import torch
    import torch.distributed as dist
    rank, world = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
    local = int(os.environ.get("LOCAL_RANK", 0))
    ngpu = torch.cuda.device_count()
    dev = local % ngpu
    torch.cuda.set_device(dev)
    dist.init_process_group(a.backend, rank=rank, world_size=world)
    L = lib.load()
    assert L.krep_b200_init(0) == 0, L.krep_b200_last_error_string()
    os.environ.pop("KREP_B200_NO_FUSED_COUNT", None)
    os.environ.pop("KREP_B200_NO_DEVICE_MATCHES", None)
    name, power = provenance()
    n = int(a.gib * bench.GIB) & ~15
    needle, flags, period = CORPUS
    spec = lib.make_spec(bench.SEED, bench.PLANT_SEED, period, needle, flags)
    begin, own, avail = sharding.shard_bounds(n, world, rank, HALO)
    t = torch.empty(avail + 64, dtype=torch.uint8, device="cuda")
    assert L.krep_b200_corpus_generate(C.byref(spec), t.data_ptr(), begin, avail, None) == 0
    torch.cuda.synchronize()
    prev_b = lib.corpus_host(spec, begin - 1, 1)[0] if begin else -1
    next_b = lib.corpus_host(spec, begin + avail, 1)[0] if begin + avail < n else -1
    shard = Shard(t.data_ptr(), avail, 0, own, begin, prev_b, next_b)
    device = f"cuda:{dev}" if a.backend == "nccl" else "cpu"
    ranks = sharding.RegexRanks(rank, world, device)
    out = dict(metric="regex_ranks", gpu=name, power_limit_w=power, ranks=world, gpus=ngpu,
               layout=(f"{world} processes on one GPU" if ngpu == 1 and world > 1 else f"{world} ranks on {min(world, ngpu)} GPUs"),
               backend=a.backend, bytes=n, steps=a.steps, warmup=a.warmup, cases={})
    for cname in a.cases.split(","):
        c = CASES[cname]
        P = Params(c["regex"], regex=True, **c["opts"])
        plan = L.krep_b200_plan_create(P.ref(), ALGO_REGEX)
        lib.check(L)
        best, counts, digests = None, set(), set()
        for i in range(a.warmup + a.steps):
            dist.barrier()
            t0 = time.perf_counter()
            got = ranks.search(plan, P, shard)
            wall = time.perf_counter() - t0
            scan, pack, nb = C.c_float(), C.c_float(), C.c_uint64()
            L.krep_b200_regex_export_stats(C.byref(scan), C.byref(pack), C.byref(nb))
            mine = dict(ranks.times, scan_ms=scan.value, pack_ms=pack.value, row_bytes=nb.value)
            per = [None] * world
            dist.all_gather_object(per, mine)
            if rank == 0:
                counts.add(got[0])
                digests.add(digest(got[1]))
                if i >= a.warmup and (best is None or wall < best[0]):
                    best = (wall, per, got)
        if rank == 0:
            assert len(counts) == 1 and len(digests) == 1, (cname, counts, digests)
            wall, per, got = best
            r = dict(regex=c["regex"].decode(), opts=c["opts"], count=got[0], digest=digest(got[1]), gbs=n / wall / 1e9,
                     wall_ms=wall * 1e3,
                     per_rank=[{k: (round(v, 2) if isinstance(v, float) else v) for k, v in p.items()} for p in per])
            if world == 1:
                cnt, pos = shards_answer(L, plan, P, shard, bool(P.struct.track_positions))
                assert cnt == got[0] and digest(pos) == r["digest"], (cname, cnt, got[0])
                r["check"] = dict(search_shards_count=cnt, search_shards_digest=digest(pos), equal=True)
            out["cases"][cname] = r
        L.krep_b200_plan_destroy(plan)
    dist.barrier()
    dist.destroy_process_group()
    if rank == 0:
        print(json.dumps(out))


if __name__ == "__main__":
    main()
