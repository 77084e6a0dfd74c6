"""-E pattern sets too large for one automaton (split plans, DESIGN §12.7): for each set, the plan (automata, path,
host build time), the filter kernel on an HBM-resident synthetic corpus, the whole krep_b200_regex_search call for -c
and for positions on pinned host text, and the stock CLI `krep -c -E -f set.txt` (with -t 1 and with its default
threads) on a slice of the same corpus: what such a set gets without the GPU.  The library's count must equal the
-t 1 CLI's; the default-thread CLI's is reported beside it (krep's regex chunks do not overlap, so it can lose a match
that straddles a chunk edge).  Prints one JSON line.

  python bench_regex_sets.py [--gib 10] [--e2e-gib 1] [--cpu-mib 256] [--steps 3] [--warmup 1]

Writes nothing into the tree (the CLI's pattern and sample files go to a temporary directory)."""
import argparse
import ctypes as C
import json
import os
import random
import string
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (workload seeds)
from bench_regex import provenance  # noqa: E402
from krep_b200 import lib  # noqa: E402
from krep_b200.abi import ALGO_REGEX, DeviceResult, Params, Shard  # noqa: E402

THE_CORPUS = (b"the", 0, 1 << 10)  # one planted "the" per KiB, as the other -E benchmarks


def _lower(rng, k):
    return ["".join(rng.choice(string.ascii_lowercase) for _ in range(rng.randint(8, 12))) for _ in range(k)]


def _err(rng, k):
    return ["ERR%s[a-z]{4}[0-9]+ code=[a-z]+" % "".join(rng.choice(string.ascii_lowercase) for _ in range(3))
            for _ in range(k)]


def workloads():
    low = _lower(random.Random(200), 200)
    return {
        "lower200_the": dict(patterns=low + ["the[a-z]*"], corpus=THE_CORPUS),  # dense: a match per KiB
        "lower200": dict(patterns=low, corpus=THE_CORPUS),                      # rare
        "err100": dict(patterns=_err(random.Random(100), 100), corpus=THE_CORPUS),
    }


def _params(pats, **kw):
    return Params([p.encode() for p in pats], regex=True, **kw)


def plan_info(L, pats):
    t0 = time.perf_counter()
    g = L.krep_b200_regex_automata(_params(pats).ref())  # builds (and caches) the plan
    build_ms = (time.perf_counter() - t0) * 1e3
    assert g >= 2, g
    return dict(automata=g, plan_build_ms=build_ms, count_mode=L.krep_b200_regex_count_mode(_params(pats, count=True).ref()),
                match_mode=L.krep_b200_regex_match_mode(_params(pats).ref()))


def kernel_rate(L, wl, nbytes, steps, warmup):
    """GB/s of the filter scan alone (CUDA events around k_regex_lines) on one HBM-resident shard."""
    import torch
    needle, flags, period = wl["corpus"]
    spec = lib.make_spec(bench.SEED, bench.PLANT_SEED, period, needle, flags)
    t = torch.empty(nbytes + 64, dtype=torch.uint8, device="cuda")
    assert L.krep_b200_corpus_generate(C.byref(spec), t.data_ptr(), 0, nbytes, None) == 0
    torch.cuda.synchronize()
    P = _params(wl["patterns"])
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
        return dict(filter=L.krep_b200_plan_filter_name(plan).decode(), kernel_gbs=nbytes / best / 1e6, kernel_ms=best,
                    flagged_lines=lines)
    finally:
        L.krep_b200_plan_destroy(plan)
        del t
        torch.cuda.empty_cache()


def host_corpus(L, wl, nbytes):
    import torch
    needle, flags, period = wl["corpus"]
    spec = lib.make_spec(bench.SEED, bench.PLANT_SEED, period, needle, flags)
    h = torch.empty(nbytes, dtype=torch.uint8).pin_memory()
    assert L.krep_b200_corpus_generate_host(C.byref(spec), h.data_ptr(), 0, nbytes) == 0
    return h


def whole_call(L, P, h, nbytes, steps, warmup):
    """Best wall time of krep_b200_regex_search on the pinned text (positions into a match_result_t), and that call's
    scan-kernel time."""
    best, cnt = None, set()
    for i in range(warmup + steps):
        res = L.krep_b200_match_result_init(16) if P.struct.track_positions else None
        try:
            t0 = time.perf_counter()
            c = L.krep_b200_regex_search(P.ref(), C.c_void_p(h.data_ptr()), nbytes, res)
            wall = time.perf_counter() - t0
            lib.check(L)
        finally:
            if res:
                L.krep_b200_match_result_free(res)
        cnt.add(int(c))
        if i >= warmup and (best is None or wall < best[0]):
            best = (wall, L.krep_b200_last_kernel_ms())
    assert len(cnt) == 1, cnt
    return dict(count=cnt.pop(), gbs=nbytes / best[0] / 1e9, s=best[0], scan_ms=best[1])


def cli_baseline(L, wl, h, nbytes):
    """Stock `krep -c -E -f set.txt` with -t 1 and with its default threads on the first nbytes, and the library's count
    of the same bytes."""
    cli = os.path.join(ROOT, "oracle", "_ref", "krep")
    lib_count = lib.search("regex", _params(wl["patterns"], count=True), None, with_result=False, text_ptr=h.data_ptr(),
                           text_len=nbytes)[0]
    if not os.path.exists(cli):
        return dict(cpu_note="stock CLI not built", slice_lib_count=lib_count)
    out = dict(slice_lib_count=lib_count)
    with tempfile.TemporaryDirectory() as d:
        pf, path = os.path.join(d, "set.txt"), os.path.join(d, "sample.txt")
        with open(pf, "w") as f:
            f.write("\n".join(wl["patterns"]) + "\n")
        with open(path, "wb") as f:
            f.write(h.numpy()[:nbytes].tobytes())
        for key, threads in (("cpu_t1", ["-t", "1"]), ("cpu_default", [])):
            cmd = [cli, *threads, "-c", "-E", "-f", pf, path]
            subprocess.run(cmd, capture_output=True)  # page cache warm
            t0 = time.perf_counter()
            r = subprocess.run(cmd, capture_output=True, text=True)
            s = time.perf_counter() - t0
            cnt = int(r.stdout.strip().rsplit(":", 1)[-1]) if r.returncode in (0, 1) and r.stdout.strip() else None
            out.update({key + "_gbs": nbytes / s / 1e9, key + "_s": s, key + "_count": cnt})
    assert out["cpu_t1_count"] == lib_count, (out, lib_count)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gib", type=float, default=10.0)
    ap.add_argument("--e2e-gib", type=float, default=1.0)
    ap.add_argument("--cpu-mib", type=int, default=256)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--workloads", default="lower200_the,lower200,err100")
    a = ap.parse_args()
    import torch
    torch.cuda.set_device(0)
    L = lib.load()
    assert L.krep_b200_init(0) == 0, L.krep_b200_last_error_string()
    name, power = provenance()
    kb, eb = int(a.gib * bench.GIB), int(a.e2e_gib * bench.GIB)
    cb = min(a.cpu_mib << 20, eb)
    out = dict(metric="regex_sets", gpu=name, power_limit_w=power, kernel_bytes=kb, e2e_bytes=eb, cpu_bytes=cb, workloads={})
    wls = workloads()
    for wname in a.workloads.split(","):
        wl = wls[wname]
        r = dict(patterns=len(wl["patterns"]))
        r.update(plan_info(L, wl["patterns"]))
        r.update(kernel_rate(L, wl, kb, a.steps, a.warmup))
        h = host_corpus(L, wl, eb)
        for key, kw in (("c", dict(count=True)), ("positions", dict())):
            r.update({key + "_" + k: v for k, v in whole_call(L, _params(wl["patterns"], **kw), h, eb, a.steps, a.warmup).items()})
        r.update(cli_baseline(L, wl, h, cb))
        del h
        out["workloads"][wname] = r
    print(json.dumps(out))


if __name__ == "__main__":
    main()
