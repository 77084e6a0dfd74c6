"""-E over batches of texts with long lines: krep_b200_regex_search_batch with the long-line pass (DESIGN §12.8) against
the same call under KREP_B200_NO_LONG_LINES=1 (every long line to glibc), a loop of krep_b200_regex_search over the same
texts, and the stock `krep -t 1 -r -E` over the texts written as files to a temporary directory.  The library arms are
alternated in one process, best of --steps after --warmup; the stock CLI runs once after a warm-up run.

Workloads: bench.py's corpus with its newlines respaced as in bench_regex_long.py (lines uniform in [L/2, 3L/2]), then
cut into texts as bench_regex_batch.py cuts (half of them extended to their line's '\\n'): about 1 000 texts of about
1 MiB with 64 KiB lines, and about 100 texts of about 8 MiB with 1 MiB lines.  Cases: the rare regex (-c), -c
'the[a-z]*' (fused count), positions of 'the[a-z]*' (offsets on the device) and -w 'the[a-z]*' positions (the line
filter).  All arms must agree on the counts (the stock CLI's: the sum of its per-file -c counts, or its -o lines), the
library arms on a digest of every text's positions.  Reports each arm's call time and GB/s, and for the batch arms the
scan time (krep_b200_last_kernel_ms, the pass included), packing time and host resolution time, with the card's name,
power limit and SM clock.  Prints one JSON line.

  python bench_regex_batch_long.py [--steps 2] [--warmup 1] [--workloads 64k,1m] [--cases ...] [--no-stock]

Writes nothing into the tree."""
import argparse
import ctypes as C
import json
import os
import random
import shutil
import sys
import tempfile

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (corpus seeds)
from bench_regex import provenance  # noqa: E402
from bench_regex_batch import STOCK, Texts, batch_arm, digest, loop_arm, stock_arm  # noqa: E402
from bench_regex_long import respaced  # noqa: E402
from bench_regex_resident import sm_clock  # noqa: E402
from krep_b200 import lib  # noqa: E402
from krep_b200.abi import Params  # noqa: E402

# texts, min and max bytes, mean line length
WORKLOADS = {"64k": (1000, 512 << 10, 1536 << 10, 64 << 10), "1m": (100, 4 << 20, 12 << 20, 1 << 20)}
CASES = {
    "rare_c": dict(regex=b"qzXv[0-9]Kpw", opts=dict(count=True), stock=["-c"]),
    "the_c": dict(regex=b"the[a-z]*", opts=dict(count=True), stock=["-c"]),
    "the_positions": dict(regex=b"the[a-z]*", opts={}, stock=["-o"]),
    "the_w_positions": dict(regex=b"the[a-z]*", opts=dict(whole_word=True), stock=["-w", "-o"]),
}


def long_line_texts(k, lo, hi, mean, seed):
    """k texts cut one after the other from the corpus respaced to lines of about `mean` bytes; half of them are
    extended to their line's '\\n'."""
    import torch
    n = (k * (hi + mean * 2) + 15) & ~15
    spec = lib.make_spec(bench.SEED, bench.PLANT_SEED, 1 << 10, b"the", 0)
    t = torch.empty(n + 64, dtype=torch.uint8, device="cuda")
    assert lib.load().krep_b200_corpus_generate(C.byref(spec), t.data_ptr(), 0, n, None) == 0
    respaced(t, n, mean, 0, seed)
    corpus = t[:n].cpu().numpy().tobytes()
    del t
    rng = random.Random(seed)
    texts, p = [], 0
    for _ in range(k):
        e = p + rng.randint(lo, hi)
        if rng.random() < 0.5:
            nl = corpus.find(b"\n", e - 1)
            e = nl + 1 if 0 <= nl < p + hi + 2 * mean else e
        texts.append(corpus[p:e])
        p = e
    return texts


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=2)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--workloads", default=",".join(WORKLOADS))
    ap.add_argument("--cases", default=",".join(CASES))
    ap.add_argument("--no-stock", action="store_true")
    a = ap.parse_args()
    import torch
    torch.cuda.set_device(0)
    L = lib.load()
    assert L.krep_b200_init(0) == 0, L.krep_b200_last_error_string()
    for k in ("KREP_B200_NO_FUSED_COUNT", "KREP_B200_NO_DEVICE_MATCHES", "KREP_B200_NO_LONG_LINES"):
        os.environ.pop(k, None)
    name, power = provenance()
    clock0 = sm_clock()
    stock = os.path.exists(STOCK) and not a.no_stock
    out = dict(metric="regex_batch_long", gpu=name, power_limit_w=power, sm_clock_mhz=clock0[0], sm_clock_max_mhz=clock0[1],
               steps=a.steps, warmup=a.warmup, stock=stock, workloads={})
    for wi, wname in enumerate(a.workloads.split(",")):
        k, lo, hi, mean = WORKLOADS[wname]
        texts = long_line_texts(k, lo, hi, mean, 4321 + wi)
        T = Texts(texts)
        w = dict(texts=T.n, bytes=T.bytes, mean_line=mean, lines=sum(t.count(b"\n") + (not t.endswith(b"\n")) for t in texts),
                 cases={})
        tmp = None
        if stock:
            tmp = tempfile.mkdtemp(prefix="krep_batch_long_")
            for i, t in enumerate(texts):
                with open(os.path.join(tmp, f"t{i:05d}.txt"), "wb") as fh:
                    fh.write(t)
        try:
            for cname in a.cases.split(","):
                c = CASES[cname]
                P = Params([c["regex"]], regex=True, **c["opts"])
                want_pos = bool(P.struct.track_positions)
                arms = ("batch", "batch_no_long", "loop")
                res = {arm: [L.krep_b200_match_result_init(16) for _ in range(T.n)] if want_pos else [] for arm in arms}
                best, counts, digests = {}, {}, {}
                for i in range(a.warmup + a.steps):
                    for arm in (arms if i % 2 == 0 else arms[::-1]):
                        if arm == "loop":
                            cnt, wall = loop_arm(L, P, T, res[arm])
                            split = {}
                        else:
                            if arm == "batch_no_long":
                                os.environ["KREP_B200_NO_LONG_LINES"] = "1"
                            try:
                                cnt, wall, scan, pack, resolve = batch_arm(L, P, T, res[arm])
                            finally:
                                os.environ.pop("KREP_B200_NO_LONG_LINES", None)
                            split = dict(scan_ms=scan, pack_ms=pack, resolve_ms=resolve)
                        counts.setdefault(arm, set()).add(tuple(cnt))
                        if want_pos:
                            digests.setdefault(arm, set()).add(digest(res[arm]))
                        if i >= a.warmup and (arm not in best or wall < best[arm]["call_ms"] / 1e3):
                            best[arm] = dict(call_ms=wall * 1e3, gbs=T.bytes / wall / 1e9, **split)
                assert all(len(v) == 1 for v in counts.values()) and len(set.union(*counts.values())) == 1, (wname, cname)
                total = sum(next(iter(counts["batch"])))
                r = dict(regex=c["regex"].decode(), opts=c["opts"], count=total, **best)
                if want_pos:
                    assert all(len(v) == 1 for v in digests.values()) and len(set.union(*digests.values())) == 1, (wname, cname)
                    r["digest"] = next(iter(digests["batch"]))
                for x in sum(res.values(), []):
                    L.krep_b200_match_result_free(x)
                if stock:
                    stock_arm(c, tmp)  # warm-up: page cache
                    sc, sw = stock_arm(c, tmp)
                    r["stock"] = dict(call_ms=sw * 1e3, gbs=T.bytes / sw / 1e9, count=sc)
                r["speedup_vs_no_long"] = best["batch_no_long"]["call_ms"] / best["batch"]["call_ms"]
                r["speedup_vs_loop"] = best["loop"]["call_ms"] / best["batch"]["call_ms"]
                w["cases"][cname] = r
        finally:
            if tmp:
                shutil.rmtree(tmp, ignore_errors=True)
        out["workloads"][wname] = w
    out["sm_clock_mhz_end"] = sm_clock()[0]
    print(json.dumps(out))
    bad = [(wn, cn) for wn, w in out["workloads"].items() for cn, r in w["cases"].items()
           if "stock" in r and r["stock"]["count"] != r["count"]]
    assert not bad, f"the stock CLI's counts differ: {bad}"


if __name__ == "__main__":
    main()
