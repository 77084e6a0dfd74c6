"""-E on lines longer than the kernel's reach: the long-line pass (DESIGN §12.8) against KREP_B200_NO_LONG_LINES=1 (every
long line to glibc), alternated in one process, best of --steps after --warmup.

Corpora: bench.py's corpus as it is (short lines: the pass finds nothing), with its newlines respaced so that lines
average 8 KiB, 64 KiB, 1 MiB, 4 MiB or 16 MiB (uniform in [L/2, 3L/2]), and the 1 MiB corpus with one 64 MiB line at
its start.  Each is searched resident (krep_b200_search_shards,
one shard: whole call, and the scan and pack device time of each arm — the scan includes the pass, so the difference of
the arms' scan times is the pass's) and as pinned host text (krep_b200_regex_search, whole call).  Workloads: -c
'the[a-z]*', positions of 'the[a-z]*', -c 'qzXv[0-9]Kpw' and -w -E 'the[a-z]*' positions.  Both arms must give equal
counts and position digests.  Stock `krep -t 1` runs on the first --cpu-mib MiB of each corpus written to a temporary
file (skipped when oracle/_ref/krep was not built).  Prints one JSON line with the card's name and power limit.

  python bench_regex_long.py [--gib 10] [--host-gib 1] [--steps 3] [--warmup 1] [--cpu-mib 256] [--corpora short,8k,...]

Writes nothing into the tree."""
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

import bench  # noqa: E402  (corpus seeds)
from bench_regex import provenance  # noqa: E402
from bench_regex_resident import digest, resident_call  # noqa: E402
from krep_b200 import lib  # noqa: E402
from krep_b200.abi import ALGO_REGEX, Params, Shard  # noqa: E402

CASES = {
    "the_c": dict(regex=b"the[a-z]*", opts=dict(count=True), cli=["-c"]),
    "the_positions": dict(regex=b"the[a-z]*", opts={}, cli=["-o"]),
    "rare_c": dict(regex=b"qzXv[0-9]Kpw", opts=dict(count=True), cli=["-c"]),
    "the_w_positions": dict(regex=b"the[a-z]*", opts=dict(whole_word=True), cli=["-w", "-o"]),
}
# mean line length, length of a first line (0: none); "short" keeps the corpus's own lines (the pass finds nothing: the
# two arms differ by its empty launches only)
CORPORA = {"short": (0, 0), "8k": (8 << 10, 0), "64k": (64 << 10, 0), "1m": (1 << 20, 0), "4m": (4 << 20, 0),
           "16m": (16 << 20, 0), "64m": (1 << 20, 64 << 20)}


def respaced(t, n, mean, first, seed):
    """t[:n] with every '\\n' replaced by ' ' and new ones every L bytes, L uniform in [mean/2, 3*mean/2]; `first` > 0:
    the first line has `first` bytes."""
    import torch
    if mean == 0:
        return
    g = torch.Generator(device="cuda").manual_seed(seed)
    v = t[:n]
    v[v == 10] = 32
    k = n // mean + 2
    gaps = torch.randint(mean // 2, mean + mean // 2 + 1, (k,), device="cuda", generator=g)
    if first:
        gaps[0] = first
    pos = torch.cumsum(gaps, 0)
    pos = pos[pos < n]
    v[pos] = 10
    torch.cuda.synchronize()


def timed(fn, knob_off):
    if knob_off:
        os.environ["KREP_B200_NO_LONG_LINES"] = "1"
    else:
        os.environ.pop("KREP_B200_NO_LONG_LINES", None)
    try:
        return fn()
    finally:
        os.environ.pop("KREP_B200_NO_LONG_LINES", None)


def host_call(P, ptr, n, want_pos):
    t0 = time.perf_counter()
    cnt, pos = lib.search("regex", P, None, with_result=want_pos, text_ptr=ptr, text_len=n)
    return cnt, pos, time.perf_counter() - t0


def stock_cli(t, nbytes, case):
    """Stock `krep -t 1` over the first nbytes of the corpus as a file (page cache warm), or None when not built."""
    cli = os.path.join(ROOT, "oracle", "_ref", "krep")
    if not os.path.exists(cli):
        return None
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "sample.txt")
        t[:nbytes].cpu().numpy().tofile(path)
        cmd = [cli, "-t", "1", *case["cli"], "-E", case["regex"].decode(), path]
        subprocess.run(cmd, capture_output=True)
        t0 = time.perf_counter()
        subprocess.run(cmd, capture_output=True)
        s = time.perf_counter() - t0
    return dict(cli_gbs=nbytes / s / 1e9, cli_s=s)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gib", type=float, default=10.0)
    ap.add_argument("--host-gib", type=float, default=1.0)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--corpora", default=",".join(CORPORA))
    ap.add_argument("--cases", default=",".join(CASES))
    ap.add_argument("--cpu-mib", type=int, default=256)
    a = ap.parse_args()
    import torch
    torch.cuda.set_device(0)
    L = lib.load()
    assert L.krep_b200_init(0) == 0, L.krep_b200_last_error_string()
    for k in ("KREP_B200_NO_FUSED_COUNT", "KREP_B200_NO_DEVICE_MATCHES", "KREP_B200_NO_LONG_LINES"):
        os.environ.pop(k, None)
    name, power = provenance()
    n = int(a.gib * bench.GIB) & ~15
    nh = min(int(a.host_gib * bench.GIB) & ~15, n)
    spec = lib.make_spec(bench.SEED, bench.PLANT_SEED, 1 << 10, b"the", 0)
    t = torch.empty(n + 64, dtype=torch.uint8, device="cuda")
    out = dict(metric="regex_long", gpu=name, power_limit_w=power, bytes=n, host_bytes=nh, steps=a.steps, warmup=a.warmup,
               corpora={})
    for ci, cname in enumerate(a.corpora.split(",")):
        mean, first = CORPORA[cname]
        assert L.krep_b200_corpus_generate(C.byref(spec), t.data_ptr(), 0, n, None) == 0
        respaced(t, n, mean, first, 1234 + ci)
        hc = torch.empty(nh, dtype=torch.uint8).pin_memory()
        hc.copy_(t[:nh])
        shards = [Shard(t.data_ptr(), n, 0, n, 0, -1, -1)]
        res_c = {}
        for cname2 in a.cases.split(","):
            c = CASES[cname2]
            P = Params(c["regex"], regex=True, **c["opts"])
            plan = L.krep_b200_plan_create(P.ref(), ALGO_REGEX)
            lib.check(L)
            want_pos = bool(P.struct.track_positions)
            best, seen = {}, {}
            for i in range(a.warmup + a.steps):
                for off in ((False, True) if i % 2 == 0 else (True, False)):
                    cnt, pos, wall, scan, pack, _ = timed(lambda: resident_call(L, plan, P, shards, want_pos), off)
                    hcnt, hpos, hwall = timed(lambda: host_call(P, hc.data_ptr(), nh, want_pos), off)
                    seen.setdefault(off, set()).add((cnt, digest(pos), hcnt, digest(hpos)))
                    if i >= a.warmup:
                        b = best.setdefault(off, dict(wall=1e30, scan=0.0, pack=0.0, hwall=1e30))
                        if wall < b["wall"]:
                            b.update(wall=wall, scan=scan, pack=pack)
                        b["hwall"] = min(b["hwall"], hwall)
            assert len(seen[False]) == 1 and seen[False] == seen[True], (cname, cname2, seen)
            cnt, _, hcnt, _ = next(iter(seen[False]))
            r = dict(regex=c["regex"].decode(), opts=c["opts"], count=cnt, host_count=hcnt)
            for off, b in best.items():
                r["knob_off" if off else "pass"] = dict(
                    resident_gbs=n / b["wall"] / 1e9, resident_ms=b["wall"] * 1e3, scan_ms=b["scan"], pack_ms=b["pack"],
                    host_text_gbs=nh / b["hwall"] / 1e9, host_text_ms=b["hwall"] * 1e3)
            r["pass_ms"] = r["pass"]["scan_ms"] - r["knob_off"]["scan_ms"]
            r["stock_krep_t1"] = stock_cli(t, min(a.cpu_mib << 20, n), c)
            res_c[cname2] = r
            L.krep_b200_plan_destroy(plan)
        out["corpora"][cname] = res_c
        del hc
    print(json.dumps(out))


if __name__ == "__main__":
    main()
