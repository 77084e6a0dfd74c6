"""Fused -c over pattern sets (-f): the line record computed on the GPU from the set's sorted keys (csrc/scan_set_count.cu)
against the occurrence-list path it replaces (KREP_B200_NO_FUSED_COUNT=1: keys, line bounds and a host replay).

Arms, per workload:
  * the whole krep_b200_aho_corasick_search -c call on pinned host text (--e2e-gib), both paths alternated;
  * a resident corpus (--resident-gib on GPU 0): krep_b200_count_lines_shard on one shard, and one
    krep_b200_search_shards -c call over 4 shards that cut lines;
  * the stock CLI `krep -t 1 -c -f` on the first --cpu-mib of the corpus, and the fused count of the same bytes.
The counts of the arms on the same bytes must agree.  Prints one JSON line with the GPU's name and power limit, read in
the same run.

  python bench_sets_count.py [--e2e-gib 1] [--resident-gib 10] [--cpu-mib 256] [--steps 5] [--warmup 1]

Writes nothing into the tree (the CLI's pattern and sample files go to a temporary directory)."""
import argparse
import ctypes as C
import json
import os
import random
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (corpus seeds and the -f pattern list)
from bench_regex import provenance  # noqa: E402
from krep_b200 import lib  # noqa: E402
from krep_b200.abi import ALGO_AC, Params, Shard, SIZE_MAX  # noqa: E402

KNOB = "KREP_B200_NO_FUSED_COUNT"


def short_set():
    rng = random.Random(0x5EED0004)
    pats = {b"the"}
    while len(pats) < 50:
        pats.add(bytes(rng.choice(b"bcdfgjkmpqvwxyz") for _ in range(rng.randint(2, 3))))
    return sorted(pats)


# name: the set, corpus (needle, flags, plant period)
WORKLOADS = {
    # bench.py's multi1000 (BASELINE config 4's set): rare hits
    "rare1000": dict(pats=lambda: bench.multi_patterns(1000, b"kqzvxjwpy"), corpus=(b"kqzvxjwpy", 0, 1 << 22)),
    # the same set with one member planted every 80 bytes (the corpus generator's densest plant for a 9-byte needle)
    "dense1000_80": dict(pats=lambda: bench.multi_patterns(1000, b"kqzvxjwpy"), corpus=(b"kqzvxjwpy", 0, 80)),
    # shortest pattern 2 bytes (k_ac_scan at stride 1)
    "short50": dict(pats=short_set, corpus=(b"the", 0, 1 << 10)),
}


def spec_of(wl):
    needle, flags, period = wl["corpus"]
    return lib.make_spec(bench.SEED, bench.PLANT_SEED, period, needle, flags)


class LineCount(C.Structure):
    _fields_ = [("lines", C.c_uint64), ("flags", C.c_uint32), ("reserved", C.c_uint32)]


def host_call(P, h, nbytes, fused):
    if fused:
        os.environ.pop(KNOB, None)
    else:
        os.environ[KNOB] = "1"
    try:
        t0 = time.perf_counter()
        cnt, _ = lib.search("aho_corasick", P, None, with_result=False, text_ptr=h.data_ptr(), text_len=nbytes)
        return cnt, time.perf_counter() - t0
    finally:
        os.environ.pop(KNOB, None)


def whole_call(L, pats, h, nbytes, steps, warmup):
    """Both paths of the whole call on pinned text, alternated: best wall time of each."""
    P = Params(pats, count=True)
    best, counts = {True: None, False: None}, {True: set(), False: set()}
    for i in range(warmup + steps):
        for fused in ((True, False) if i % 2 == 0 else (False, True)):
            cnt, wall = host_call(P, h, nbytes, fused)
            counts[fused].add(cnt)
            if i >= warmup and (best[fused] is None or wall < best[fused]):
                best[fused] = wall
    assert len(counts[True]) == 1 and counts[True] == counts[False], counts
    return dict(count=counts[True].pop(), record_gbs=nbytes / best[True] / 1e9, record_s=best[True],
                list_gbs=nbytes / best[False] / 1e9, list_s=best[False], speedup=best[False] / best[True])


def resident(L, wl, pats, nbytes, steps, warmup):
    """count_lines_shard on the whole corpus as one shard; search_shards -c on 4 shards (views of the same buffer)."""
    import torch
    t = torch.empty(nbytes + 64, dtype=torch.uint8, device="cuda")
    assert L.krep_b200_corpus_generate(C.byref(spec_of(wl)), t.data_ptr(), 0, nbytes, None) == 0
    torch.cuda.synchronize()
    halo = max(map(len, pats)) + 1
    P = Params(pats, count=True)
    P.struct.ac_trie = 1
    plan = L.krep_b200_plan_create(P.ref(), ALGO_AC)
    lib.check(L)
    one = Shard(t.data_ptr(), nbytes, 0, nbytes, 0, -1, -1)
    # 4 shards cut at 16-byte aligned offsets (anywhere in a line); context bytes from the buffer itself
    cuts = [nbytes * k // 4 // 16 * 16 for k in range(4)] + [nbytes]
    host = lambda q: int(t[q].item()) if 0 <= q < nbytes else -1  # noqa: E731
    four = [Shard(t.data_ptr() + b, min(e + halo, nbytes) - b, 0, e - b, b, host(b - 1), host(min(e + halo, nbytes)))
            for b, e in zip(cuts, cuts[1:])]
    rec = LineCount()

    def one_shard():
        assert L.krep_b200_count_lines_shard(plan, P.ref(), C.byref(one), None, C.byref(rec)) == 0, \
            L.krep_b200_last_error_string()
        return int(L.krep_b200_combine_line_counts(C.byref(rec), 1, SIZE_MAX))

    def four_shards():
        return lib.search_shards(plan, P, four, with_result=False)[0]

    out = {}
    try:
        L.krep_b200_count_lines_shard.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(Shard), C.c_void_p, C.POINTER(LineCount)]
        L.krep_b200_count_lines_shard.restype = C.c_int
        L.krep_b200_combine_line_counts.argtypes = [C.POINTER(LineCount), C.c_size_t, C.c_size_t]
        L.krep_b200_combine_line_counts.restype = C.c_uint64
        for name, fn in (("shard1", one_shard), ("shards4", four_shards)):
            counts, times = set(), []
            for i in range(warmup + steps):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                counts.add(fn())
                torch.cuda.synchronize()
                if i >= warmup:
                    times.append(time.perf_counter() - t0)
            assert len(counts) == 1, counts
            out[name] = dict(count=counts.pop(), s=min(times), gbs=nbytes / min(times) / 1e9)
        assert out["shard1"]["count"] == out["shards4"]["count"], out
    finally:
        L.krep_b200_plan_destroy(plan)
        del t
        torch.cuda.empty_cache()
    return out


def cpu_baseline(pats, h, nbytes):
    """Stock `krep -t 1 -c -f` on the first nbytes of the corpus, and the fused count of the same bytes."""
    cli = os.path.join(ROOT, "oracle", "_ref", "krep")
    fused, _ = host_call(Params(pats, count=True), h, nbytes, True)
    if not os.path.exists(cli):
        return dict(cpu_gbs=None, cpu_note="stock CLI not built", slice_fused_count=fused)
    with tempfile.TemporaryDirectory() as d:
        path, pat_file = os.path.join(d, "sample.txt"), os.path.join(d, "patterns.txt")
        with open(path, "wb") as f:
            f.write(h.numpy()[:nbytes].tobytes())
        with open(pat_file, "wb") as f:
            f.write(b"\n".join(pats) + b"\n")
        cmd = [cli, "-t", "1", "-c", "-f", pat_file, path]
        subprocess.run(cmd, capture_output=True)  # page cache warm
        t0 = time.perf_counter()
        r = subprocess.run(cmd, capture_output=True, text=True)
        s = time.perf_counter() - t0
    stock = int(r.stdout.strip().rsplit(":", 1)[-1]) if r.returncode in (0, 1) and r.stdout.strip() else None  # "path:count"
    assert stock == fused, (stock, fused, r.stdout[:200], r.stderr[:200])
    return dict(cpu_gbs=nbytes / s / 1e9, cpu_s=s, cpu_count=stock, slice_fused_count=fused)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--e2e-gib", type=float, default=1.0)
    ap.add_argument("--resident-gib", type=float, default=10.0)
    ap.add_argument("--cpu-mib", type=int, default=256)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--workloads", default=",".join(WORKLOADS))
    a = ap.parse_args()
    import torch
    torch.cuda.set_device(0)
    L = lib.load()
    assert L.krep_b200_init(0) == 0, L.krep_b200_last_error_string()
    name, power = provenance()
    nbytes, rbytes = int(a.e2e_gib * bench.GIB), int(a.resident_gib * bench.GIB)
    cpu_bytes = min(a.cpu_mib << 20, nbytes)
    out = dict(metric="sets_count", gpu=name, power_limit_w=power, e2e_bytes=nbytes, resident_bytes=rbytes,
               cpu_bytes=cpu_bytes, workloads={})
    for wname in a.workloads.split(","):
        wl = WORKLOADS[wname]
        pats = wl["pats"]()
        h = torch.empty(nbytes, dtype=torch.uint8).pin_memory()
        assert L.krep_b200_corpus_generate_host(C.byref(spec_of(wl)), h.data_ptr(), 0, nbytes) == 0
        r = dict(patterns=len(pats), shortest=min(map(len, pats)))
        r["whole_call"] = whole_call(L, pats, h, nbytes, a.steps, a.warmup)
        r["resident"] = resident(L, wl, pats, rbytes, a.steps, a.warmup)
        r.update(cpu_baseline(pats, h, cpu_bytes))
        out["workloads"][wname] = r
        del h
    print(json.dumps(out))


if __name__ == "__main__":
    main()
