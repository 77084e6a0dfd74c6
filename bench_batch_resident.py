"""Many HBM-resident texts in one call: krep_b200_search_batch_resident / krep_b200_regex_search_batch_resident against
the host batches (krep_b200_search_batch / krep_b200_regex_search_batch) on pinned host copies of the same texts, and,
for the 2 000-text workload, a loop of krep_b200_search_shards with one call per text (each text copied to a 16-byte
aligned place of its own first, outside the timing).  The arms alternate in one process, best of --steps after
--warmup.

Workloads: texts cut one after the other from bench.py's corpus as bench_regex_batch.py cuts them (half of them
extended to their line's '\\n'), held back to back in one uint8 CUDA tensor: 20 000 x ~4 KiB, 2 000 x ~64 KiB and
1 000 000 x ~1 KiB, and the 4 KiB texts again with every '\\n' made a space (one line per text, as documents often
are; a text's line bounds then reach its edges).  Cases: an 8-byte literal (positions and -c), a 1000-pattern set of 6-12 bytes (-c), -E -c
'qzXv[0-9]Kpw', -E -c 'the[a-z]*' and -E 'the[a-z]*' positions.  Every arm must give the same per-text digest (counts
and positions).  Reports each arm's call time and GB/s of text, and for the resident arm the gather, scan and resolve
times and the gather's copy rate (bytes read plus bytes written over the gather time), with the card's name, power
limit and SM clock.  Prints one JSON line.

  python bench_batch_resident.py [--steps 2] [--warmup 1] [--workloads 4k,64k,1k,4k_nonl] [--cases ...]

Writes nothing into the tree."""
import argparse
import ctypes as C
import hashlib
import json
import os
import random
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (corpus seeds)
from bench_regex import provenance  # noqa: E402
from bench_regex_batch import CORPUS  # noqa: E402
from bench_regex_resident import sm_clock  # noqa: E402
from krep_b200 import lib  # noqa: E402
from krep_b200.abi import ALGO_AC, ALGO_BMH, ALGO_REGEX, MatchResult, Params, Shard  # noqa: E402

# texts, min and max bytes
WORKLOADS = {"4k": (20000, 2 << 10, 6 << 10), "64k": (2000, 32 << 10, 96 << 10), "1k": (1000000, 512, 1536),
             "4k_nonl": (20000, 2 << 10, 6 << 10)}  # the 4 KiB texts with every '\n' made a space: one line per text


def set_patterns():
    rng = random.Random(1000)
    return [bytes(rng.choice(b"abcdefghijklmnopqrstuvwxyz") for _ in range(rng.randint(6, 12))) for _ in range(1000)]


CASES = {
    "lit_positions": dict(func="boyer_moore", pats=[b"tion and"], opts={}),
    "lit_c": dict(func="boyer_moore", pats=[b"tion and"], opts=dict(count=True)),
    "set_c": dict(func="aho_corasick", pats=None, opts=dict(count=True)),
    "rx_rare_c": dict(func="regex", pats=[b"qzXv[0-9]Kpw"], opts=dict(count=True)),
    "rx_the_c": dict(func="regex", pats=[b"the[a-z]*"], opts=dict(count=True)),
    "rx_the_positions": dict(func="regex", pats=[b"the[a-z]*"], opts={}),
}


def cut_texts(k, lo, hi, seed):
    rng = random.Random(seed)
    n = k * (hi + 4096)
    needle, flags, period = CORPUS
    spec = lib.make_spec(bench.SEED, bench.PLANT_SEED, period, needle, flags)
    corpus = lib.corpus_host(spec, 0, n)
    offs, lens, p = [], [], 0
    for _ in range(k):
        e = p + rng.randint(lo, hi)
        if rng.random() < 0.5:
            nl = corpus.find(b"\n", e - 1)
            e = nl + 1 if 0 <= nl < p + hi + 4096 else e
        offs.append(p)
        lens.append(e - p)
        p = e
    return corpus[:p], offs, lens


class Arrays:
    """ctypes arrays of one call: offsets, lens, host pointers into the pinned copy, counts, results."""

    def __init__(self, L, pinned, offs, lens, with_result):
        n = len(lens)
        self.n = n
        self.offs = (C.c_uint64 * n)(*offs)
        self.lens = (C.c_size_t * n)(*lens)
        base = pinned.data_ptr()
        self.texts = (C.c_char_p * n)(*[C.cast(C.c_void_p(base + o), C.c_char_p) for o in offs])
        self.counts = (C.c_uint64 * n)()
        self.res = [L.krep_b200_match_result_init(16) for _ in range(n)] if with_result else []
        self.rarr = (C.POINTER(MatchResult) * n)(*self.res) if with_result else None

    def reset(self):
        for r in self.res:
            r.contents.count = 0

    def digest(self):
        h = hashlib.sha256()
        h.update(bytes(self.counts))
        for i, r in enumerate(self.res):
            c = r.contents
            if c.count:
                h.update(i.to_bytes(4, "little") + C.string_at(c.positions, c.count * C.sizeof(c.positions[0])))
        return h.hexdigest()[:16]

    def free(self, L):
        for r in self.res:
            L.krep_b200_match_result_free(r)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=2)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--workloads", default=",".join(WORKLOADS))
    ap.add_argument("--cases", default=",".join(CASES))
    args = ap.parse_args()
    import torch
    L = lib.load()
    assert L.krep_b200_init(0) == 0
    name, power = provenance()
    clk, clk_max = sm_clock()
    out = {"gpu": name, "power_limit_w": power, "sm_clock_mhz": clk, "sm_clock_max_mhz": clk_max, "results": []}
    pats_set = set_patterns()
    for wname in args.workloads.split(","):
        k, lo, hi = WORKLOADS[wname]
        buf, offs, lens = cut_texts(k, lo, hi, seed=k)
        if wname.endswith("_nonl"):
            buf = buf.replace(b"\n", b" ")
        nbytes = sum(lens)
        host = torch.frombuffer(bytearray(buf), dtype=torch.uint8)
        pinned = host.pin_memory()
        dev = host.cuda()
        # the loop arm's texts, each at a 16-byte aligned place
        loop_dev, loop_offs = None, []
        if wname == "64k":
            p = 0
            for n in lens:
                loop_offs.append(p)
                p = (p + n + 15) & ~15
            loop_dev = torch.zeros(p + 64, dtype=torch.uint8, device="cuda")
            for o, lo_, n in zip(loop_offs, offs, lens):
                loop_dev[o:o + n] = dev[lo_:lo_ + n]
        torch.cuda.synchronize()
        del host
        for cname in args.cases.split(","):
            case = CASES[cname]
            pats = case["pats"] or pats_set
            regex = case["func"] == "regex"
            P = Params(pats, regex=regex, **case["opts"])
            if case["func"] == "aho_corasick":
                P.struct.ac_trie = L.krep_b200_ac_trie_build(P.ref())
            with_result = bool(P.struct.track_positions)
            entry = None if regex else C.cast(getattr(L, lib.SEARCH_ENTRIES[case["func"]]), C.c_void_p)
            arms = {}

            def resident(A):
                if regex:
                    return L.krep_b200_regex_search_batch_resident(P.ref(), dev.data_ptr(), A.offs, A.lens, A.n, A.counts, A.rarr)
                return L.krep_b200_search_batch_resident(entry, P.ref(), dev.data_ptr(), A.offs, A.lens, A.n, A.counts, A.rarr)

            def host_batch(A):
                if regex:
                    return L.krep_b200_regex_search_batch(P.ref(), A.texts, A.lens, A.n, A.counts, A.rarr)
                return L.krep_b200_search_batch(entry, P.ref(), A.texts, A.lens, A.n, A.counts, A.rarr)

            arms["resident"] = (resident, Arrays(L, pinned, offs, lens, with_result))
            arms["host_batch"] = (host_batch, Arrays(L, pinned, offs, lens, with_result))
            plan = None
            if loop_dev is not None:
                plan = L.krep_b200_plan_create(P.ref(), ALGO_REGEX if regex else ALGO_AC if case["func"] == "aho_corasick" else ALGO_BMH)
                shards = [Shard(loop_dev.data_ptr() + o, n, 0, n, 0, -1, -1) for o, n in zip(loop_offs, lens)]

                def loop(A):
                    for i, sh in enumerate(shards):
                        A.counts[i] = L.krep_b200_search_shards(plan, P.ref(), C.byref(sh), 1, A.res[i] if A.res else None)
                        if L.krep_b200_last_error() != 0:
                            return L.krep_b200_last_error()
                    return 0

                arms["shards_loop"] = (loop, Arrays(L, pinned, offs, lens, with_result))
            best = {a: float("inf") for a in arms}
            stats = None
            for step in range(args.warmup + args.steps):
                for a, (fn, A) in arms.items():
                    A.reset()
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    rc = fn(A)
                    dt = time.perf_counter() - t0
                    assert rc == 0, (wname, cname, a, rc, L.krep_b200_last_error_string())
                    if step >= args.warmup and dt < best[a]:
                        best[a] = dt
                        if a == "resident":
                            stats = lib.batch_resident_stats()
            digests = {a: A.digest() for a, (_, A) in arms.items()}
            g_ms, s_ms, r_ms = stats
            # bytes the gather writes: the packed size (pack_layout), gaps of the longest pattern + 16 (-E: 1) included
            gap = 1 if regex else max(len(p) for p in pats) + 16
            packed = 0
            for n in lens:
                packed = (packed + n + gap + 15) & ~15
            row = {"workload": wname, "texts": k, "bytes": nbytes, "case": cname,
                   "digests_equal": len(set(digests.values())) == 1, "digest": digests["resident"],
                   "gather_ms": round(g_ms, 3), "scan_ms": round(s_ms, 3), "resolve_ms": round(r_ms, 3),
                   "gather_gb_s": round((nbytes + packed) / (g_ms * 1e6), 1) if g_ms > 0 else None}
            for a in arms:
                row[a + "_ms"] = round(best[a] * 1e3, 2)
                row[a + "_gb_s"] = round(nbytes / best[a] / 1e9, 2)
            out["results"].append(row)
            print(json.dumps(row), file=sys.stderr, flush=True)
            for _, A in arms.values():
                A.free(L)
            if plan:
                L.krep_b200_plan_destroy(plan)
            if P.struct.ac_trie:
                L.krep_b200_ac_trie_free(P.struct.ac_trie)
                P.struct.ac_trie = None
        del dev, pinned, loop_dev
        torch.cuda.empty_cache()
    out["all_digests_equal"] = all(r["digests_equal"] for r in out["results"])
    print(json.dumps(out))


if __name__ == "__main__":
    main()
