"""Fused -E -c: the whole krep_b200_regex_search -c call on pinned host text with the count computed on the GPU (only
the uncertain lines go to glibc's regexec) against the same call with KREP_B200_NO_FUSED_COUNT=1 (regexec confirms
every flagged line), alternated in one process, and the stock CLI `krep -t 1 -c -E` on a slice of the same corpus.
The counts of the three must agree.  Prints one JSON line.

  python bench_regex_count.py [--e2e-gib 1] [--cpu-mib 256] [--steps 5] [--warmup 1]

Writes nothing into the tree (the CLI's sample file goes to a temporary directory)."""
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

import bench  # noqa: E402  (workload seeds)
from bench_regex import provenance  # noqa: E402
from krep_b200 import lib  # noqa: E402
from krep_b200.abi import Params  # noqa: E402

KNOB = "KREP_B200_NO_FUSED_COUNT"

# name: regex, Params options, corpus (needle, flags, plant period), CLI flags
WORKLOADS = {
    "dense_the_c": dict(regex=b"the[a-z]*", opts={}, corpus=(b"the", 0, 1 << 10), cli=[]),
    "dense_class_led_c": dict(regex=b"[tT]h[a-z]*", opts={}, corpus=(b"the", 0, 1 << 10), cli=[]),
    "two_words_line_c": dict(regex=b"^[a-z]+ [a-z]+$", opts={}, corpus=(b"the", 0, 1 << 10), cli=[]),
    "rare_literal_c": dict(regex=b"qzXv[0-9]Kpw", opts={}, corpus=(b"qzXv9Kpw", 0, 1 << 20), cli=[]),
}


def host_corpus(L, wl, nbytes):
    import torch
    needle, flags, period = wl["corpus"]
    spec = lib.make_spec(bench.SEED, bench.PLANT_SEED, period, needle, flags)
    h = torch.empty(nbytes, dtype=torch.uint8).pin_memory()
    assert L.krep_b200_corpus_generate_host(C.byref(spec), h.data_ptr(), 0, nbytes) == 0
    return h


def count_call(L, P, h, nbytes, fused):
    if fused:
        os.environ.pop(KNOB, None)
    else:
        os.environ[KNOB] = "1"
    try:
        assert L.krep_b200_regex_count_mode(P.ref()) == (1 if fused else 0)
        t0 = time.perf_counter()
        cnt, _ = lib.search("regex", P, None, with_result=False, text_ptr=h.data_ptr(), text_len=nbytes)
        return cnt, time.perf_counter() - t0, L.krep_b200_last_kernel_ms()
    finally:
        os.environ.pop(KNOB, None)


def end_to_end(L, wl, h, nbytes, steps, warmup):
    """Both arms of the whole call, alternated: best wall time of each, and the fused arm's scan-kernel time."""
    P = Params(wl["regex"], regex=True, count=True, **wl["opts"])
    best = {True: None, False: None}
    counts = {True: set(), False: set()}
    for i in range(warmup + steps):
        for fused in ((True, False) if i % 2 == 0 else (False, True)):
            cnt, wall, kms = count_call(L, P, h, nbytes, fused)
            counts[fused].add(cnt)
            if i >= warmup and (best[fused] is None or wall < best[fused][0]):
                best[fused] = (wall, kms)
    assert len(counts[True]) == 1 and counts[True] == counts[False], counts
    (fw, fk), (uw, uk) = best[True], best[False]
    return dict(count=counts[True].pop(), fused_gbs=nbytes / fw / 1e9, fused_s=fw, fused_kernel_ms=fk,
                regexec_gbs=nbytes / uw / 1e9, regexec_s=uw, regexec_kernel_ms=uk, speedup=uw / fw)


def cpu_baseline(L, wl, h, nbytes):
    """Stock `krep -t 1 -c -E` on the first nbytes of the corpus, and the fused count of the same bytes."""
    cli = os.path.join(ROOT, "oracle", "_ref", "krep")
    P = Params(wl["regex"], regex=True, count=True, **wl["opts"])
    fused, _, _ = count_call(L, P, h, nbytes, True)
    if not os.path.exists(cli):
        return dict(cpu_gbs=None, cpu_note="stock CLI not built", slice_fused_count=fused)
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "sample.txt")
        with open(path, "wb") as f:
            f.write(h.numpy()[:nbytes].tobytes())
        cmd = [cli, "-t", "1", "-c", *wl["cli"], "-E", wl["regex"].decode(), path]
        subprocess.run(cmd, capture_output=True)  # page cache warm
        t0 = time.perf_counter()
        r = subprocess.run(cmd, capture_output=True, text=True)
        s = time.perf_counter() - t0
    stock = int(r.stdout.strip().rsplit(":", 1)[-1]) if r.returncode in (0, 1) and r.stdout.strip() else None  # "path:count"
    assert stock == fused, (wl["regex"], stock, fused, r.stdout[:200], r.stderr[:200])
    return dict(cpu_gbs=nbytes / s / 1e9, cpu_s=s, cpu_count=stock, slice_fused_count=fused)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--e2e-gib", type=float, default=1.0)
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
    nbytes = int(a.e2e_gib * bench.GIB)
    cpu_bytes = min(a.cpu_mib << 20, nbytes)
    out = dict(metric="regex_count", gpu=name, power_limit_w=power, e2e_bytes=nbytes, cpu_bytes=cpu_bytes, workloads={})
    for wname in a.workloads.split(","):
        wl = WORKLOADS[wname]
        h = host_corpus(L, wl, nbytes)
        r = dict(regex=wl["regex"].decode(), opts=wl["opts"])
        r.update(end_to_end(L, wl, h, nbytes, a.steps, a.warmup))
        r.update(cpu_baseline(L, wl, h, cpu_bytes))
        out["workloads"][wname] = r
        del h
    print(json.dumps(out))


if __name__ == "__main__":
    main()
