"""-E over many small texts: krep_b200_regex_search_batch against a loop of krep_b200_regex_search over the same texts
(arms alternated in one process, best of --steps after --warmup) and against the stock `krep -t 1 -r -E` over the same
texts written as files to a temporary directory.  Two workloads cut from bench.py's synthetic corpus (about 20 000 texts
of about 4 KiB, about 2 000 of about 64 KiB; half of them end in '\\n'), three calls: the rare regex (-c), dense
-c 'the[a-z]*' (fused count) and positions of 'the[a-z]*' (offsets on the device).  All arms must agree on the counts
(the stock CLI's: the sum of its per-file -c counts, or its -o lines), the two library arms on a digest of every
text's positions.  Reports each arm's call time and GB/s, and the batch's scan time (krep_b200_last_kernel_ms), packing
time and host resolution time (the per-text replays, with at least one regexec per text on the -c and offsets paths).
Prints one JSON line.

  python bench_regex_batch.py [--steps 3] [--warmup 1] [--workloads small,large] [--no-stock]

Writes nothing into the tree."""
import argparse
import ctypes as C
import hashlib
import json
import os
import random
import shutil
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (workload seeds)
from bench_regex import provenance  # noqa: E402
from bench_regex_resident import CORPUS, sm_clock  # noqa: E402
from krep_b200 import lib  # noqa: E402
from krep_b200.abi import MatchResult, Params  # noqa: E402

WORKLOADS = {"small": (20000, 2048, 6144), "large": (2000, 32768, 98304)}  # texts, min and max bytes
CASES = {
    "rare_c": dict(regex=b"qzXv[0-9]Kpw", opts=dict(count=True), stock=["-c"]),
    "the_c": dict(regex=b"the[a-z]*", opts=dict(count=True), stock=["-c"]),
    "the_positions": dict(regex=b"the[a-z]*", opts={}, stock=["-o"]),
}
STOCK = os.path.join(ROOT, "oracle", "_ref", "krep")


def cut_texts(k, lo, hi, seed):
    """k texts cut one after the other from the corpus; half of them are extended to their line's '\\n'."""
    rng = random.Random(seed)
    n = k * (hi + 4096)
    needle, flags, period = CORPUS
    spec = lib.make_spec(bench.SEED, bench.PLANT_SEED, period, needle, flags)
    corpus = lib.corpus_host(spec, 0, n)
    texts, p = [], 0
    for _ in range(k):
        m = rng.randint(lo, hi)
        e = p + m
        if rng.random() < 0.5:
            nl = corpus.find(b"\n", e - 1)
            e = nl + 1 if 0 <= nl < p + hi + 4096 else e
        texts.append(corpus[p:e])
        p = e
    return texts


class Texts:
    """The texts in one host buffer, with the pointer and length arrays both library arms use."""

    def __init__(self, texts):
        self.n = len(texts)
        self.buf = C.create_string_buffer(b"".join(texts), max(sum(map(len, texts)), 1))
        base = C.addressof(self.buf)
        offs, o = [], 0
        for t in texts:
            offs.append(o)
            o += len(t)
        self.bytes = o
        self.ptrs = (C.c_void_p * self.n)(*[base + x for x in offs])
        self.lens = (C.c_size_t * self.n)(*[len(t) for t in texts])


def digest(results):
    h = hashlib.sha256()
    for i, res in enumerate(results):
        r = res.contents
        for k in range(r.count):
            h.update(i.to_bytes(4, "little") + r.positions[k].start_offset.to_bytes(8, "little") +
                     r.positions[k].end_offset.to_bytes(8, "little"))
    return h.hexdigest()[:16]


def batch_arm(L, P, T, results):
    for r in results:
        r.contents.count = 0
    counts = (C.c_uint64 * T.n)()
    rarr = (C.POINTER(MatchResult) * T.n)(*results) if results else None
    t0 = time.perf_counter()
    rc = L.krep_b200_regex_search_batch(P.ref(), C.cast(T.ptrs, C.POINTER(C.c_char_p)), T.lens, T.n, counts, rarr)
    wall = time.perf_counter() - t0
    lib.check(L)
    assert rc == 0, rc
    pack, resolve = C.c_double(), C.c_double()
    L.krep_b200_regex_batch_stats(C.byref(pack), C.byref(resolve))
    return list(counts), wall, L.krep_b200_last_kernel_ms(), pack.value, resolve.value


def loop_arm(L, P, T, results):
    for r in results:
        r.contents.count = 0
    f = L.krep_b200_regex_search
    ref = P.ref()
    counts = [0] * T.n
    t0 = time.perf_counter()
    for i in range(T.n):
        counts[i] = f(ref, T.ptrs[i], T.lens[i], results[i] if results else None)
    wall = time.perf_counter() - t0
    lib.check(L)
    return counts, wall


def stock_arm(case, d):
    t0 = time.perf_counter()
    r = subprocess.run([STOCK, "-t", "1", "-r", *case["stock"], "-E", case["regex"].decode(), d], capture_output=True)
    wall = time.perf_counter() - t0
    assert r.returncode in (0, 1), r.stderr[-500:]
    lines = r.stdout.splitlines()
    if "-c" in case["stock"]:
        return sum(int(x.rsplit(b":", 1)[1]) for x in lines), wall
    return len(lines), wall


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--workloads", default=",".join(WORKLOADS))
    ap.add_argument("--cases", default=",".join(CASES))
    ap.add_argument("--no-stock", action="store_true")
    a = ap.parse_args()
    import torch
    torch.cuda.set_device(0)
    L = lib.load()
    assert L.krep_b200_init(0) == 0, L.krep_b200_last_error_string()
    os.environ.pop("KREP_B200_NO_FUSED_COUNT", None)
    os.environ.pop("KREP_B200_NO_DEVICE_MATCHES", None)
    name, power = provenance()
    clock0 = sm_clock()
    stock = os.path.exists(STOCK) and not a.no_stock
    out = dict(metric="regex_batch", gpu=name, power_limit_w=power, sm_clock_mhz=clock0[0], sm_clock_max_mhz=clock0[1],
               steps=a.steps, warmup=a.warmup, stock=stock, workloads={})
    for wname in a.workloads.split(","):
        k, lo, hi = WORKLOADS[wname]
        texts = cut_texts(k, lo, hi, seed={"small": 1, "large": 2}.get(wname, 0))
        T = Texts(texts)
        w = dict(texts=T.n, bytes=T.bytes, ending_in_newline=sum(t.endswith(b"\n") for t in texts), cases={})
        tmp = None
        if stock:
            tmp = tempfile.mkdtemp(prefix="krep_batch_")
            for i, t in enumerate(texts):
                with open(os.path.join(tmp, f"t{i:05d}.txt"), "wb") as fh:
                    fh.write(t)
        try:
            for cname in a.cases.split(","):
                c = CASES[cname]
                P = Params([c["regex"]], regex=True, **c["opts"])
                want_pos = bool(P.struct.track_positions)
                res_b = [L.krep_b200_match_result_init(16) for _ in range(T.n)] if want_pos else []
                res_l = [L.krep_b200_match_result_init(16) for _ in range(T.n)] if want_pos else []
                best = {}
                for i in range(a.warmup + a.steps):
                    for arm in (("batch", "loop") if i % 2 == 0 else ("loop", "batch")):
                        if arm == "batch":
                            cb, wall, scan, pack, resolve = batch_arm(L, P, T, res_b)
                            if i >= a.warmup and ("batch" not in best or wall < best["batch"][0]):
                                best["batch"] = (wall, scan, pack, resolve)
                        else:
                            cl, wall = loop_arm(L, P, T, res_l)
                            if i >= a.warmup and ("loop" not in best or wall < best["loop"][0]):
                                best["loop"] = (wall,)
                assert cb == cl, (wname, cname, [i for i in range(T.n) if cb[i] != cl[i]][:5])
                r = dict(regex=c["regex"].decode(), opts=c["opts"], count=sum(cb))
                if want_pos:
                    r["digest_batch"], r["digest_loop"] = digest(res_b), digest(res_l)
                    assert r["digest_batch"] == r["digest_loop"], (wname, cname)
                for x in res_b + res_l:
                    L.krep_b200_match_result_free(x)
                wall, scan, pack, resolve = best["batch"]
                r["batch"] = dict(call_ms=wall * 1e3, gbs=T.bytes / wall / 1e9, scan_ms=scan, pack_ms=pack, resolve_ms=resolve)
                r["loop"] = dict(call_ms=best["loop"][0] * 1e3, gbs=T.bytes / best["loop"][0] / 1e9)
                if stock:
                    sw = None
                    for _ in range(min(a.steps, 2)):
                        sc, t = stock_arm(c, tmp)
                        assert sc == sum(cb), (wname, cname, sc, sum(cb))
                        sw = t if sw is None else min(sw, t)
                    r["stock"] = dict(call_ms=sw * 1e3, gbs=T.bytes / sw / 1e9, count=sc)
                r["speedup_vs_loop"] = best["loop"][0] / wall
                w["cases"][cname] = r
        finally:
            if tmp:
                shutil.rmtree(tmp, ignore_errors=True)
        out["workloads"][wname] = w
    out["sm_clock_mhz_end"] = sm_clock()[0]
    print(json.dumps(out))


if __name__ == "__main__":
    main()
