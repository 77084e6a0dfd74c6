"""-E on an HBM-resident corpus: krep_b200_search_shards on regex plans, the corpus tiled into one shard and into 4, for
five calls — the rare regex, -c 'the[a-z]*' (fused count), positions of 'the[a-z]*' (offsets on the device),
-w -E 'the[a-z]*' positions (line filter + pack + regexec) and -c -E '\\bthe' (a widened plan: filter + regexec).  Arms
alternated, best of --steps after --warmup.  Reports the scan and pack device time, the packed row bytes, the host time
(the rest of the call: row read-back and glibc) and the whole call's GB/s.  Before timing, the same five calls on a
prefix of the corpus are checked against krep_b200_regex_search on a pinned host copy of it: equal counts and an equal
digest of the positions.  Prints one JSON line.

  python bench_regex_resident.py [--gib 10] [--check-gib 1] [--steps 5] [--warmup 1]

Writes nothing into the tree."""
import argparse
import ctypes as C
import hashlib
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (workload seeds)
from bench_regex import provenance  # noqa: E402
from krep_b200 import lib  # noqa: E402
from krep_b200.abi import ALGO_REGEX, Params, Shard  # noqa: E402

# one `the` per KiB planted in the corpus; the rare regex matches the planted needle of bench.py's corpus only
CORPUS = (b"the", 0, 1 << 10)
CASES = {
    "rare": dict(regex=b"qzXv[0-9]Kpw", opts=dict(count=True)),
    "the_c": dict(regex=b"the[a-z]*", opts=dict(count=True)),
    "the_positions": dict(regex=b"the[a-z]*", opts={}),
    "the_w_positions": dict(regex=b"the[a-z]*", opts=dict(whole_word=True)),
    "bthe_c": dict(regex=b"\\bthe", opts=dict(count=True)),
}


def sm_clock():
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=clocks.sm,clocks.max.sm", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        cur, mx = (float(x) for x in out.splitlines()[0].split(","))
        return cur, mx
    except (OSError, ValueError, IndexError, subprocess.TimeoutExpired):
        return None, None


def tiles(ptr, n, k):
    """k shards over [0, n) at ptr, cut at 16-byte aligned offsets, each reading REGEX_HALO bytes past its owned range."""
    halo = 4096
    cuts = [0] + [(n * i // k) & ~15 for i in range(1, k)] + [n]
    out = []
    for b, e in zip(cuts, cuts[1:]):
        end = min(n, e + halo)
        out.append(Shard(ptr + b, end - b, 0, e - b, b, -1 if b == 0 else 0, -1 if end == n else 0))
    return out


def fix_bytes(shards, host_byte):
    """prev_byte / next_byte of each shard from the text (host_byte(i) reads byte i)."""
    for s in shards:
        if s.global_offset:
            s.prev_byte = host_byte(s.global_offset - 1)
        end = s.global_offset + s.avail_len
        s.next_byte = -1 if s.next_byte == -1 else host_byte(end)
    return shards


def digest(pos):
    h = hashlib.sha256()
    for s, e in pos:
        h.update(s.to_bytes(8, "little") + e.to_bytes(8, "little"))
    return h.hexdigest()[:16]


def resident_call(L, plan, P, shards, with_result):
    arr = (Shard * len(shards))(*shards)
    res = L.krep_b200_match_result_init(16) if with_result else None
    try:
        t0 = time.perf_counter()
        cnt = L.krep_b200_search_shards(plan, P.ref(), arr, len(shards), res)
        wall = time.perf_counter() - t0
        lib.check(L)
        scan, pack, nb = C.c_float(), C.c_float(), C.c_uint64()
        L.krep_b200_regex_export_stats(C.byref(scan), C.byref(pack), C.byref(nb))
        pos = []
        if res:
            r = res.contents
            pos = [(r.positions[i].start_offset, r.positions[i].end_offset) for i in range(r.count)]
        return int(cnt), pos, wall, scan.value, pack.value, nb.value
    finally:
        if res:
            L.krep_b200_match_result_free(res)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gib", type=float, default=10.0)
    ap.add_argument("--check-gib", type=float, default=1.0)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--cases", default=",".join(CASES))
    a = ap.parse_args()
    import torch
    torch.cuda.set_device(0)
    L = lib.load()
    assert L.krep_b200_init(0) == 0, L.krep_b200_last_error_string()
    os.environ.pop("KREP_B200_NO_FUSED_COUNT", None)
    os.environ.pop("KREP_B200_NO_DEVICE_MATCHES", None)
    name, power = provenance()
    n = int(a.gib * bench.GIB) & ~15
    nc = min(int(a.check_gib * bench.GIB) & ~15, n)
    needle, flags, period = CORPUS
    spec = lib.make_spec(bench.SEED, bench.PLANT_SEED, period, needle, flags)
    t = torch.empty(n + 64, dtype=torch.uint8, device="cuda")
    assert L.krep_b200_corpus_generate(C.byref(spec), t.data_ptr(), 0, n, None) == 0
    torch.cuda.synchronize()
    hc = torch.empty(nc, dtype=torch.uint8).pin_memory()
    hc.copy_(t[:nc])
    host_byte = lambda i: int(t[i].item())  # noqa: E731
    clock0 = sm_clock()
    out = dict(metric="regex_resident", gpu=name, power_limit_w=power, sm_clock_mhz=clock0[0], sm_clock_max_mhz=clock0[1],
               bytes=n, check_bytes=nc, steps=a.steps, warmup=a.warmup, cases={})
    for cname in a.cases.split(","):
        c = CASES[cname]
        P = Params(c["regex"], regex=True, **c["opts"])
        plan = L.krep_b200_plan_create(P.ref(), ALGO_REGEX)
        lib.check(L)
        want_pos = bool(P.struct.track_positions)
        # agreement on the prefix: resident (1 and 4 shards) against the host-text entry point
        hcnt, hpos = lib.search("regex", P, None, with_result=want_pos, text_ptr=hc.data_ptr(), text_len=nc)
        check = dict(host_count=hcnt, host_digest=digest(hpos))
        for k in (1, 4):
            cnt, pos, _, _, _, _ = resident_call(L, plan, P, fix_bytes(tiles(t.data_ptr(), nc, k), host_byte), want_pos)
            assert cnt == hcnt and digest(pos) == check["host_digest"], (cname, k, cnt, hcnt)
            check[f"resident_{k}_count"] = cnt
        r = dict(regex=c["regex"].decode(), opts=c["opts"], check=check)
        arms = {k: fix_bytes(tiles(t.data_ptr(), n, k), host_byte) for k in (1, 4)}
        best, counts = {}, {1: set(), 4: set()}
        for i in range(a.warmup + a.steps):
            for k in ((1, 4) if i % 2 == 0 else (4, 1)):
                cnt, _, wall, scan, pack, nb = resident_call(L, plan, P, arms[k], want_pos)
                counts[k].add(cnt)
                if i >= a.warmup and (k not in best or wall < best[k][0]):
                    best[k] = (wall, scan, pack, nb)
        assert len(counts[1]) == 1 and counts[1] == counts[4], counts
        r["count"] = counts[1].pop()
        for k, (wall, scan, pack, nb) in best.items():
            r[f"shards_{k}"] = dict(gbs=n / wall / 1e9, wall_ms=wall * 1e3, scan_ms=scan, pack_ms=pack, packed_bytes=nb,
                                    host_ms=wall * 1e3 - scan - pack)
        out["cases"][cname] = r
        L.krep_b200_plan_destroy(plan)
    out["sm_clock_mhz_end"] = sm_clock()[0]
    print(json.dumps(out))


if __name__ == "__main__":
    main()
