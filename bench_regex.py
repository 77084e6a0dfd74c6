"""-E throughput: the device line filter (k_regex_lines) on an HBM-resident synthetic corpus, the whole
krep_b200_regex_search call on pinned host text (H2D + filter + glibc regexec on the flagged lines), and the stock CLI
`krep -t 1 -E` on a slice of the same corpus.  Prints one JSON line.

  python bench_regex.py [--gib 10] [--e2e-gib 1] [--cpu-mib 256] [--steps 3] [--warmup 1]

Writes nothing into the tree (the CPU baseline's sample file goes to a temporary directory)."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (workload seeds, data-sheet peak)
from krep_b200 import lib  # noqa: E402
from krep_b200.abi import ALGO_REGEX, Params, Shard, DeviceResult  # noqa: E402

# name: regex, Params options, corpus (needle, flags, plant period), CLI flags
WORKLOADS = {
    "rare_literal": dict(regex=b"qzXv[0-9]Kpw", opts={}, corpus=(b"qzXv9Kpw", 0, 1 << 20), cli=["-c"]),
    "rare_class_led": dict(regex=b"[A-Z]zXv[0-9]Kp", opts={}, corpus=(b"qzXv9Kpw", 0, 1 << 20), cli=["-c"]),
    "icase_alternation": dict(regex=b"qzxv9kpw|zebra|quartz", opts=dict(case_sensitive=False), corpus=(b"QzXv9Kpw", 1, 1 << 20),
                              cli=["-c", "-i"]),
    "dense_the_c": dict(regex=b"the[a-z]*", opts=dict(count=True), corpus=(b"the", 0, 1 << 10), cli=["-c"]),
}


def provenance():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        power = float(out.splitlines()[0]) if out else None
    except (OSError, ValueError, subprocess.TimeoutExpired):
        power = None
    return name, power


def kernel_rate(L, wl, nbytes, steps, warmup):
    """GB/s of the scan kernel alone (CUDA events around k_regex_lines) on one HBM-resident shard."""
    import torch
    needle, flags, period = wl["corpus"]
    spec = lib.make_spec(bench.SEED, bench.PLANT_SEED, period, needle, flags)
    t = torch.empty(nbytes + 64, dtype=torch.uint8, device="cuda")
    assert L.krep_b200_corpus_generate(C.byref(spec), t.data_ptr(), 0, nbytes, None) == 0
    torch.cuda.synchronize()
    P = Params(wl["regex"], regex=True, **wl["opts"])
    plan = L.krep_b200_plan_create(P.ref(), ALGO_REGEX)
    lib.check(L)
    try:
        sh = Shard(t.data_ptr(), nbytes, 0, nbytes, 0, -1, -1)
        ms, lines = [], 0
        for i in range(warmup + steps):
            out = DeviceResult()
            assert L.krep_b200_scan_shard(plan, C.byref(sh), 1, None, C.byref(out)) == 0
            lib.check(L)
            if i >= warmup:
                ms.append(L.krep_b200_last_kernel_ms())
                lines = int(out.count)
        best = min(ms)
        return dict(kernel_gbs=nbytes / best / 1e6, kernel_ms=best, flagged_lines=lines, filter=L.krep_b200_plan_filter_name(plan).decode())
    finally:
        L.krep_b200_plan_destroy(plan)
        del t
        torch.cuda.empty_cache()


def end_to_end(L, wl, nbytes, steps, warmup):
    """Whole krep_b200_regex_search call on pinned host text: copy, filter, regexec on the flagged lines."""
    import torch
    needle, flags, period = wl["corpus"]
    spec = lib.make_spec(bench.SEED, bench.PLANT_SEED, period, needle, flags)
    h = torch.empty(nbytes, dtype=torch.uint8).pin_memory()
    assert L.krep_b200_corpus_generate_host(C.byref(spec), h.data_ptr(), 0, nbytes) == 0
    P = Params(wl["regex"], regex=True, **wl["opts"])
    walls, kms, cnt = [], [], 0
    for i in range(warmup + steps):
        t0 = time.perf_counter()
        cnt, _ = lib.search("regex", P, None, with_result=P.struct.track_positions, text_ptr=h.data_ptr(), text_len=nbytes)
        wall = time.perf_counter() - t0
        if i >= warmup:
            walls.append(wall)
            kms.append(L.krep_b200_last_kernel_ms())
    best = min(walls)
    return dict(e2e_gbs=nbytes / best / 1e9, e2e_s=best, e2e_kernel_ms=kms[walls.index(best)], e2e_count=int(cnt))


def cpu_baseline(wl, nbytes):
    cli = os.path.join(ROOT, "oracle", "_ref", "krep")
    if not os.path.exists(cli):
        return dict(cpu_gbs=None, cpu_note="stock CLI not built")
    L = lib.load()
    needle, flags, period = wl["corpus"]
    spec = lib.make_spec(bench.SEED, bench.PLANT_SEED, period, needle, flags)
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "sample.txt")
        buf = C.create_string_buffer(nbytes)
        assert L.krep_b200_corpus_generate_host(C.byref(spec), buf, 0, nbytes) == 0
        with open(path, "wb") as f:
            f.write(buf.raw)
        del buf
        cmd = [cli, "-t", "1", *wl["cli"], "-E", wl["regex"].decode(), path]
        subprocess.run(cmd, capture_output=True)  # page cache warm
        t0 = time.perf_counter()
        r = subprocess.run(cmd, capture_output=True, text=True)
        s = time.perf_counter() - t0
    return dict(cpu_gbs=nbytes / s / 1e9, cpu_s=s, cpu_out=r.stdout.strip()[:40])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gib", type=float, default=10.0)
    ap.add_argument("--e2e-gib", type=float, default=1.0)
    ap.add_argument("--cpu-mib", type=int, default=256)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--workloads", default=",".join(WORKLOADS))
    a = ap.parse_args()
    import torch
    torch.cuda.set_device(0)
    L = lib.load()
    assert L.krep_b200_init(0) == 0, L.krep_b200_last_error_string()
    peak, peak_src = bench.peaks()
    name, power = provenance()
    out = dict(metric="regex_filter", gpu=name, power_limit_w=power, hbm_peak_gbs=peak, hbm_peak_source=peak_src,
               kernel_bytes=int(a.gib * bench.GIB), e2e_bytes=int(a.e2e_gib * bench.GIB), cpu_bytes=a.cpu_mib << 20,
               workloads={})
    for wname in a.workloads.split(","):
        wl = WORKLOADS[wname]
        r = dict(regex=wl["regex"].decode(), opts=wl["opts"])
        r.update(kernel_rate(L, wl, int(a.gib * bench.GIB), a.steps, a.warmup))
        r["kernel_fraction_of_peak"] = r["kernel_gbs"] / peak
        r.update(end_to_end(L, wl, int(a.e2e_gib * bench.GIB), a.steps, a.warmup))
        r.update(cpu_baseline(wl, a.cpu_mib << 20))
        out["workloads"][wname] = r
    print(json.dumps(out))


if __name__ == "__main__":
    main()
