"""-E offsets on the GPU: the whole krep_b200_regex_search positions (or -co) call on pinned host text with the match
offsets computed on the GPU (only the uncertain lines go to glibc's regexec) against the same call with
KREP_B200_NO_DEVICE_MATCHES=1 (regexec computes every offset on the flagged lines), alternated in one process, and the
stock CLI `krep -t 1 -co -E` on a slice of the same corpus.  The two arms must give the same count and the same digest
of positions, and the stock count must agree.  Prints one JSON line.

  python bench_regex_match.py [--e2e-gib 1] [--cpu-mib 256] [--steps 5] [--warmup 1]

Writes nothing into the tree (the CLI's sample file goes to a temporary directory)."""
import argparse
import ctypes as C
import hashlib
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (workload seeds)
from bench_regex import provenance  # noqa: E402
from krep_b200 import lib  # noqa: E402
from krep_b200.abi import Params  # noqa: E402

KNOB = "KREP_B200_NO_DEVICE_MATCHES"

# name: regex, Params options, corpus (needle, flags, plant period), optional cap on the text size
WORKLOADS = {
    "dense_the": dict(regex=b"the[a-z]*", opts={}, corpus=(b"the", 0, 1 << 10)),
    "dense_the_co": dict(regex=b"the[a-z]*", opts=dict(count=True, only_matching=True), corpus=(b"the", 0, 1 << 10)),
    "dense_class_led": dict(regex=b"[tT]h[a-z]*", opts={}, corpus=(b"the", 0, 1 << 10)),
    "rare_literal": dict(regex=b"qzXv[0-9]Kpw", opts={}, corpus=(b"qzXv9Kpw", 0, 1 << 20)),
    # every start before a line's first comma walks to the line's end: lines with a comma run over the step budget and
    # go to regexec, which is quadratic on them too (about 4 MB/s), hence the smaller text
    "budget_heavy": dict(regex=b".*QQ|,", opts={}, corpus=(b"the", 0, 1 << 10), max_bytes=16 << 20),
}


def host_corpus(L, wl, nbytes):
    import torch
    needle, flags, period = wl["corpus"]
    spec = lib.make_spec(bench.SEED, bench.PLANT_SEED, period, needle, flags)
    h = torch.empty(nbytes, dtype=torch.uint8).pin_memory()
    assert L.krep_b200_corpus_generate_host(C.byref(spec), h.data_ptr(), 0, nbytes) == 0
    return h


def match_call(L, P, h, nbytes, device):
    """One whole call; -> (count, sha256 of the (start, end) pairs, wall seconds, scan-kernel ms)."""
    if device:
        os.environ.pop(KNOB, None)
    else:
        os.environ[KNOB] = "1"
    res = L.krep_b200_match_result_init(1 << 20)
    try:
        assert L.krep_b200_regex_match_mode(P.ref()) == (1 if device else 0)
        L.krep_b200_set_only_matching(bool(P.only_matching))
        t0 = time.perf_counter()
        cnt = L.krep_b200_regex_search(P.ref(), C.c_void_p(h.data_ptr()), nbytes, res)
        wall = time.perf_counter() - t0
        lib.check(L)
        kms = L.krep_b200_last_kernel_ms()
        r = res.contents
        pos = np.ctypeslib.as_array(C.cast(r.positions, C.POINTER(C.c_uint64)), shape=(2 * r.count,)) if r.count else np.zeros(0, np.uint64)
        return int(cnt), hashlib.sha256(pos.tobytes()).hexdigest()[:16], int(r.count), wall, kms
    finally:
        L.krep_b200_set_only_matching(False)
        L.krep_b200_match_result_free(res)
        os.environ.pop(KNOB, None)


def end_to_end(L, wl, h, nbytes, steps, warmup):
    """Both arms of the whole call, alternated: best wall time of each, and its scan-kernel time."""
    P = Params(wl["regex"], regex=True, **wl["opts"])
    best = {True: None, False: None}
    outs = {True: set(), False: set()}
    for i in range(warmup + steps):
        for device in ((True, False) if i % 2 == 0 else (False, True)):
            cnt, digest, npos, wall, kms = match_call(L, P, h, nbytes, device)
            outs[device].add((cnt, digest, npos))
            if i >= warmup and (best[device] is None or wall < best[device][0]):
                best[device] = (wall, kms)
    assert len(outs[True]) == 1 and outs[True] == outs[False], outs
    (dw, dk), (rw, rk) = best[True], best[False]
    cnt, digest, npos = outs[True].pop()
    return dict(count=cnt, positions=npos, digest=digest, device_gbs=nbytes / dw / 1e9, device_s=dw, device_kernel_ms=dk,
                regexec_gbs=nbytes / rw / 1e9, regexec_s=rw, regexec_kernel_ms=rk, speedup=rw / dw)


def cpu_baseline(L, wl, h, nbytes):
    """Stock `krep -t 1 -co -E` on the first nbytes of the corpus, and the device count of the same bytes (-co)."""
    cli = os.path.join(ROOT, "oracle", "_ref", "krep")
    P = Params(wl["regex"], regex=True, count=True, only_matching=True, **{k: v for k, v in wl["opts"].items()
                                                                          if k not in ("count", "only_matching")})
    dev = match_call(L, P, h, nbytes, True)[0]
    if not os.path.exists(cli):
        return dict(cpu_gbs=None, cpu_note="stock CLI not built", slice_device_count=dev)
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "sample.txt")
        with open(path, "wb") as f:
            f.write(h.numpy()[:nbytes].tobytes())
        cmd = [cli, "-t", "1", "-co", "-E", wl["regex"].decode(), path]
        subprocess.run(cmd, capture_output=True)  # page cache warm
        t0 = time.perf_counter()
        r = subprocess.run(cmd, capture_output=True, text=True)
        s = time.perf_counter() - t0
    stock = int(r.stdout.strip().rsplit(":", 1)[-1]) if r.returncode in (0, 1) and r.stdout.strip() else None  # "path:count"
    assert stock == dev, (wl["regex"], stock, dev, r.stdout[:200], r.stderr[:200])
    return dict(cpu_gbs=nbytes / s / 1e9, cpu_s=s, cpu_count=stock, slice_device_count=dev)


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
    out = dict(metric="regex_match", gpu=name, power_limit_w=power, e2e_bytes=nbytes, cpu_bytes=cpu_bytes, workloads={})
    for wname in a.workloads.split(","):
        wl = WORKLOADS[wname]
        wbytes = min(nbytes, wl.get("max_bytes", nbytes))
        h = host_corpus(L, wl, wbytes)
        r = dict(regex=wl["regex"].decode(), opts=wl["opts"], bytes=wbytes)
        r.update(end_to_end(L, wl, h, wbytes, a.steps, a.warmup))
        r.update(cpu_baseline(L, wl, h, min(cpu_bytes, wbytes)))
        out["workloads"][wname] = r
        del h
    print(json.dumps(out))


if __name__ == "__main__":
    main()
