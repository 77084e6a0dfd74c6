#!/usr/bin/env python
"""bench.py — BASELINE.json's metric: GB/s scanned over an HBM-resident synthetic corpus.

    python bench.py [--gpus N] [--steps K] [--warmup W] [--impl ours|reference] [--gib G] [--workload NAME] [--no-side]
                    [--dump-outputs DIR]

Headline (value / roofline / e2e) = BASELINE configs[1]: 8-byte literal over 10 GiB of HBM-resident synthetic ASCII per
GPU, count + all offsets.  For N>1 (launched by torchrun, one rank per GPU) each rank holds its own 10 GiB shard
(+halo) of an N x 10 GiB corpus (weak scaling), scans it, and one NCCL gather brings counts and offsets to rank 0
(SURVEY §8e), which merges them by key and replays them into krep's match_result_t.

The same JSON line carries a `workloads` object with BASELINE configs[2], [3] and [4] at their stated TOTAL sizes,
sharded over the N GPUs the run was launched with (strong scaling): -i 4-byte literal on 50 GiB, 1000 patterns on
20 GiB (20 / 10 / 5 / 2.5 GiB per GPU at N = 1 / 2 / 4 / 8) and -w 16-byte literal on 40 GiB (every total fits one
80 GB H100 at N = 1).

A step = one pass of the hot path over the resident shard: filter+verify kernel, the one-CTA finish kernel (count +
sorted list, one synchronisation), policy replay into krep's match_result_t (N>1: + export, gather, key merge; rank 0
does its host work for step i while step i+1 scans).  Inputs are >= 2.5 GiB >> 50 MB L2, so nothing survives in L2
between steps.  One JSON line on stdout (rank 0).

--dump-outputs DIR writes what the caller of the timed path received in the last timed step of the headline workload
(rank 0): DIR/matches.npy (the count) and DIR/positions.npy (the match_result_t (start, end) offsets), float64.  Inputs
depend only on the arguments, so two builds can be compared output for output.
"""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import tempfile
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

GIB = 1 << 30
WORKLOADS = {
    # name: (needle, params kwargs, corpus flags, plant period, description)
    "literal8": dict(needle=b"qzXv9Kpw", opts={}, flags=0, period=1 << 20,
                     desc="8-byte literal, case-sensitive, count + all offsets (BASELINE configs[1])"),
    "icase4": dict(needle=b"QzXv", opts=dict(case_sensitive=False), flags=1, period=1 << 20,
                   desc="-i 4-byte literal (BASELINE configs[2])"),
    "word16": dict(needle=b"needleneedle0016", opts=dict(whole_word=True), flags=2, period=1 << 26,
                   desc="-w 16-byte literal, low hit rate (BASELINE configs[4])"),
    "multi1000": dict(needle=b"kqzvxjwpy", opts={}, flags=0, period=1 << 22, multi=1000,
                      desc="1000 patterns of 6-12 bytes (-f), Aho-Corasick result set (BASELINE configs[3])"),
    "multi1000_5to12": dict(needle=b"kqzvxjwpy", opts={}, flags=0, period=1 << 22, multi=1000, lens=(5, 12),
                            desc="1000 patterns of 5-12 bytes (-f): shortest pattern 5, stride-2 paired filter (k_ac_scan)"),
    # hit-density workloads (not BASELINE configs): config 1's pattern `the`, planted once per 1 KiB / 64 B
    "the_1k": dict(needle=b"the", opts={}, flags=0, period=1 << 10,
                   desc="3-byte literal `the`, one planted per 1 KiB (plus accidental hits), count + all offsets"),
    "the_64": dict(needle=b"the", opts={}, flags=0, period=1 << 6,
                   desc="3-byte literal `the`, one planted per 64 B (plus accidental hits), count + all offsets"),
    "the_1k_c": dict(needle=b"the", opts=dict(count=True), flags=0, period=1 << 10,
                     desc="`-c the` (count matching lines), one planted per 1 KiB"),
    "the_64_c": dict(needle=b"the", opts=dict(count=True), flags=0, period=1 << 6,
                     desc="`-c the` (count matching lines), one planted per 64 B"),
    # side workloads (not BASELINE configs): other regimes of the multi-pattern filter
    "multi1000_8to14": dict(needle=b"kqzvxjwpy", opts={}, flags=0, period=1 << 22, multi=1000, lens=(8, 14),
                            desc="1000 patterns of 8-14 bytes (-f): shortest pattern >= 7, full-word hash filter"),
    "multi1000_i": dict(needle=b"kqzvxjwpy", opts=dict(case_sensitive=False), flags=1, period=1 << 22, multi=1000,
                        desc="1000 patterns of 6-12 bytes, -i"),
}
SEED, PLANT_SEED = 0x5EED0001, 0x5EED0002
# BASELINE configs[2..4]: (workload, TOTAL GiB over all GPUs) — strong scaling over the N the run is launched with
SIDE_WORKLOADS = [("icase4", 50.0), ("multi1000", 20.0), ("word16", 40.0)]
# at N = 1 only: hit-density sweep on 10 GiB
DENSITY_WORKLOADS = [("the_1k", 10.0), ("the_64", 10.0), ("the_1k_c", 10.0), ("the_64_c", 10.0), ("multi1000_5to12", 10.0)]


def peaks():
    path = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(path):
        with open(path) as f:
            return float(json.load(f)["hbm_gbs"]), "measured (MEASURED_PEAKS.json hbm_gbs, copy read+write)"
    return 3350.0, "data sheet (H100 SXM, HBM3 3.35 TB/s; not measured)"


def multi_patterns(n, needle, lens=(6, 12)):
    import random
    rng = random.Random(0x5EED0003)
    alpha = "abcdefghijklmnopqrstuvwxyz"
    pats = {needle}
    while len(pats) < n:
        pats.add("".join(rng.choice(alpha) for _ in range(rng.randint(*lens))).encode())
    return [needle] + sorted(pats - {needle})


class ClockSampler:
    """nvidia-smi clocks / throttle reasons.  The sampler runs from before the warm-up
    (nvidia-smi takes ~100 ms to produce its first line) and only samples whose timestamp falls inside the
    timed region are reported; if the region was too short to contain one, the nearest samples are used."""

    def __init__(self, index):
        self.index = index
        self.proc = None
        self.path = None
        self.t0 = self.t1 = None

    def start(self):
        try:
            fd, self.path = tempfile.mkstemp(suffix=".csv")
            os.close(fd)
            q = ("timestamp,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,"
                 "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,"
                 "clocks_event_reasons.sw_power_cap")
            self.proc = subprocess.Popen(["nvidia-smi", f"--id={self.index}", f"--query-gpu={q}",
                                          "--format=csv,noheader,nounits", "-lms", "20"],
                                         stdout=open(self.path, "w"), stderr=subprocess.DEVNULL)
        except Exception:
            self.proc = None

    def wait_first_sample(self, timeout=3.0):
        """nvidia-smi needs ~100 ms before its first line: do not let a short timed region start (and end) before it."""
        t_end = time.time() + timeout
        while self.proc and time.time() < t_end:
            try:
                if os.path.getsize(self.path) > 0:
                    return
            except OSError:
                return
            time.sleep(0.01)

    def mark_begin(self):
        self.t0 = time.time()

    def mark_end(self):
        self.t1 = time.time()

    def stop(self):
        import datetime
        out = {"sm_mhz": None, "sm_max_mhz": None, "reasons": [], "samples": 0}
        if not self.proc:
            return out
        time.sleep(0.05)
        self.proc.terminate()
        try:
            self.proc.wait(timeout=5)
        except Exception:
            self.proc.kill()
        rows = []
        try:
            for line in open(self.path):
                f = [x.strip() for x in line.split(",")]
                if len(f) < 8:
                    continue
                try:
                    ts = datetime.datetime.strptime(f[0], "%Y/%m/%d %H:%M:%S.%f").timestamp()
                    rows.append((ts, float(f[1]), float(f[2]), float(f[3]), f[4:8]))
                except ValueError:
                    continue
            os.unlink(self.path)
        except Exception:
            pass
        if not rows:
            return out
        inside = [r for r in rows if self.t0 is not None and self.t0 <= r[0] <= self.t1]
        used = inside
        if not used:  # region shorter than the sampling period: take the samples closest to it
            mid = 0.5 * ((self.t0 or rows[-1][0]) + (self.t1 or rows[-1][0]))
            used = sorted(rows, key=lambda r: abs(r[0] - mid))[:3]
        reasons = set()
        for r in used:
            for name, v in zip(("hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"), r[4]):
                if v.lower().startswith("active"):
                    reasons.add(name)
        return {"sm_mhz": statistics.median(r[1] for r in used), "sm_max_mhz": max(r[2] for r in used),
                "power_w_max": max(r[3] for r in used), "reasons": sorted(reasons), "samples": len(used),
                "samples_inside_timed_region": len(inside)}


# ------------------------------------------------------------------------------------------------
# reference arm / cpu baseline: the stock krep CLI built from /root/reference (oracle/_ref/krep), all host threads,
# plus an in-process call of the reference's own kernel function (oracle/_ref/libkrep_ref.so) on one thread.
# This leg never maps libkrep_b200.so: the corpus sample is written by a child process.
# ------------------------------------------------------------------------------------------------
_SAMPLE_WRITER = r"""
import ctypes as C, sys
sys.path.insert(0, sys.argv[1])
from krep_b200 import lib
seed, plant_seed, period, flags, nbytes = (int(x) for x in sys.argv[4:9])
needle, path = bytes.fromhex(sys.argv[2]), sys.argv[3]
spec = lib.make_spec(seed, plant_seed, period, needle, flags)
done = False
try:
    import torch
    if torch.cuda.is_available():
        L = lib.load()
        t = torch.empty(nbytes + 64, dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        assert L.krep_b200_corpus_generate(C.byref(spec), t.data_ptr(), 0, nbytes, None) == 0
        t[:nbytes].cpu().numpy().tofile(path)
        done = True
except Exception as e:
    print(f"[bench] GPU corpus generation unavailable ({e}); using the host twin", file=sys.stderr)
if not done:
    with open(path, "wb") as f:
        step = 64 << 20
        for off in range(0, nbytes, step):
            f.write(lib.corpus_host(spec, off, min(step, nbytes - off)))
"""


def write_sample(wl, nbytes, path):
    """Writes corpus bytes [0, nbytes) of the workload to `path` in a CHILD process (GPU generator when available, else
    the host twin), so that the process timing the reference never loads the product library."""
    r = subprocess.run([sys.executable, "-c", _SAMPLE_WRITER, ROOT, wl["needle"].hex(), path, str(SEED), str(PLANT_SEED),
                        str(wl["period"]), str(wl["flags"]), str(nbytes)], stdout=sys.stderr, stderr=sys.stderr)
    if r.returncode != 0 or not os.path.exists(path) or os.path.getsize(path) != nbytes:
        raise RuntimeError("writing the corpus sample failed")


def krep_cli_cmd(cli, wl, sample_path, pat_file):
    if wl["opts"].get("count"):
        cmd = [cli, "-c"]                        # -c: count matching lines
    else:
        cmd = [cli, "-c", "-o"]                  # -co: count matches (scan + count, no output formatting)
    if not wl["opts"].get("case_sensitive", True):
        cmd.append("-i")
    if wl["opts"].get("whole_word"):
        cmd.append("-w")
    if wl.get("multi"):
        cmd += ["-f", pat_file, sample_path]
    else:
        cmd += [wl["needle"].decode(), sample_path]
    return cmd


def in_process_reference(wl, pats, sample_path, nbytes):
    """The reference's own kernel function called in-process on the in-memory slice (one call on the whole buffer = the
    -t 1 result; excludes process start and mmap population).  -> dict or None."""
    try:
        sys.path.insert(0, os.path.join(ROOT, "tests"))
        import oracle_util as ou
        from krep_b200.abi import Params          # ctypes struct mirrors only: does not load any library
        ref = ou.reference()
        if ref is None:
            return None
        with open(sample_path, "rb") as f:
            data = f.read(nbytes)
        opts = dict(wl["opts"])
        if pats:
            func = "aho_corasick"
        elif not opts.get("case_sensitive", True) or len(wl["needle"]) > 16:
            func = "boyer_moore"                  # what simd_avx2_search falls back to (krep.c:4883)
        elif len(wl["needle"]) < 4:
            func = "avx2" if opts.get("case_sensitive", True) else "memchr_short"
        else:
            func = "sse42"
        best, cnt = None, 0
        for _ in range(2):
            p = Params(pats if pats else wl["needle"], only_matching=not opts.get("count"), **{**opts, "count": True})
            t0 = time.perf_counter()
            cnt, _ = ref.run(func, p, data, with_result=False)
            dt = time.perf_counter() - t0
            best = dt if best is None else min(best, dt)
        return {"value": len(data) / best / 1e9, "unit": "GB/s", "threads": 1, "function": ou.FUNCS[func][1],
                "sample": f"{len(data) >> 20} MiB in memory, best of 2 calls of the reference's own function "
                          f"(oracle/_ref/libkrep_ref.so)", "count": cnt}
    except Exception as e:  # noqa: BLE001
        return {"error": str(e)}


def run_cpu_reference(wl_name, wl, sample_bytes, steps, warmup, in_process=True):
    """Times the unmodified reference on a bounded sample of the workload. -> dict(value GB/s, cores, kind, sample, count, ms)"""
    sys.path.insert(0, os.path.join(ROOT, "oracle"))
    import build_oracle
    _, cli = build_oracle.build_ref()
    shm = "/dev/shm" if os.path.isdir("/dev/shm") else tempfile.gettempdir()
    sample_path = os.path.join(shm, f"krep_b200_sample_{os.getpid()}.txt")
    pat_file = sample_path + ".pats"
    pats = multi_patterns(wl["multi"], wl["needle"], wl.get("lens", (6, 12))) if wl.get("multi") else None
    write_sample(wl, sample_bytes, sample_path)
    if pats:
        with open(pat_file, "wb") as f:
            f.write(b"\n".join(pats) + b"\n")
    cores = os.cpu_count() or 1
    times, count, single, inproc = [], None, None, None
    try:
        if cli:
            cmd = krep_cli_cmd(cli, wl, sample_path, pat_file)
            for it in range(warmup + steps):
                t0 = time.perf_counter()
                r = subprocess.run(cmd, capture_output=True, text=True)
                dt = time.perf_counter() - t0
                if it == 0 and dt * (warmup + steps - 1) > 150.0 and sample_bytes > (64 << 20):
                    # keep the whole reference arm within a few minutes whatever the host: shrink the slice
                    shrink = max(64 << 20, int(sample_bytes * 150.0 / (dt * (warmup + steps - 1))) & ~0xFFFFF)
                    with open(sample_path, "r+b") as f:
                        f.truncate(shrink)
                    sample_bytes = shrink
                    continue  # this run timed the larger slice: not recorded
                if it >= warmup:
                    times.append(dt)
                last = r.stdout.strip().splitlines()[-1] if r.stdout.strip() else "0"
                count = int(last.rsplit(":", 1)[-1])
            kind = "reference"
            how = f"stock krep CLI (oracle/_ref/krep, -msse4.2 -mavx2 build) `{' '.join(cmd[1:-1])} FILE`, default threads"
            # SURVEY §8d also asks for the -t 1 figure: one run on the first 256 MiB of the same file
            try:
                small = min(sample_bytes, 256 << 20)
                small_path = sample_path + ".t1"
                with open(sample_path, "rb") as fi, open(small_path, "wb") as fo:
                    fo.write(fi.read(small))
                cmd1 = cmd[:1] + ["-t", "1"] + cmd[1:-1] + [small_path]
                subprocess.run(cmd1, capture_output=True)
                t0 = time.perf_counter()
                subprocess.run(cmd1, capture_output=True)
                single = {"value": small / (time.perf_counter() - t0) / 1e9, "unit": "GB/s", "sample": f"{small >> 20} MiB, -t 1, one run after one warm-up"}
                os.unlink(small_path)
            except Exception:  # noqa: BLE001
                single = None
            if in_process:
                inproc = in_process_reference(wl, pats, sample_path, min(sample_bytes, 256 << 20))
        else:
            # compiled reference absent: time the scalar oracle port on one core
            sys.path.insert(0, os.path.join(ROOT, "tests"))
            import oracle_util as ou
            from krep_b200.abi import Params
            data = open(sample_path, "rb").read()
            func = "aho_corasick" if pats else "sse42"
            for it in range(warmup + steps):
                p = Params(pats if pats else wl["needle"], count=True, only_matching=True, **wl["opts"])
                t0 = time.perf_counter()
                count, _ = ou.port().run(func, p, data, with_result=False)
                dt = time.perf_counter() - t0
                if it >= warmup:
                    times.append(dt)
            kind, cores = "port", 1
            how = "oracle/krep_oracle.c scalar port, 1 thread"
        if not times:  # every recorded slot was consumed by the shrink step (steps == 1, warmup == 0)
            t0 = time.perf_counter()
            subprocess.run(cmd, capture_output=True, text=True)
            times.append(time.perf_counter() - t0)
    finally:
        for pth in (sample_path, pat_file):
            if os.path.exists(pth):
                os.unlink(pth)
    mean = sum(times) / len(times)
    extra = {}
    if cli and single:
        extra["single_thread"] = single
    if inproc:
        extra["in_process"] = inproc
    try:
        with open("/proc/cpuinfo") as f:
            extra["cpu_model"] = next((ln.split(":", 1)[1].strip() for ln in f if ln.startswith("model name")), None)
    except OSError:
        pass
    return dict(extra, value=sample_bytes / mean / 1e9, best=sample_bytes / min(times) / 1e9, unit="GB/s", cores=cores, kind=kind,
                sample_bytes=sample_bytes,
                sample=f"{sample_bytes / GIB:.2f} GiB slice [0, n) of the same corpus in {shm}; whole-process wall, "
                       f"mean of {len(times)} runs after {warmup} warm-up; {how}",
                count=count, ms=mean * 1e3)


CPU_KEYS = ("value", "unit", "cores", "kind", "sample", "sample_bytes", "single_thread", "in_process", "cpu_model")


# ------------------------------------------------------------------------------------------------
def main():
    # The contract is ONE JSON line on stdout: keep the real stdout aside and point fd 1 at stderr, so that nothing a
    # native library prints (e.g. NCCL's version banner) can land in front of it.
    sys.stdout.flush()
    real_stdout = os.fdopen(os.dup(1), "w")
    os.dup2(2, 1)
    try:
        _main(real_stdout)
    finally:
        real_stdout.flush()


def workload_config(wl, gib_per_gpu, world, total_gib=None):
    size = (f"{total_gib:g} GiB synthetic ASCII in total, {gib_per_gpu:g} GiB per GPU" if total_gib is not None
            else f"{gib_per_gpu:g} GiB synthetic ASCII per GPU")
    return {"workload": f"{wl['desc']}; {size}, seed {SEED:#x}, 1 planted needle per "
                        f"{wl['period'] >> 10 if wl['period'] >= 1024 else wl['period'] / 1024:g} KiB",
            "needle": wl["needle"].decode(), "bytes_per_gpu": int(gib_per_gpu * GIB), "l2": "inputs >> L2 (no flush needed)"}


class Runner:
    """Everything one rank needs to run workloads on its resident shard."""

    def __init__(self, args):
        import torch
        import torch.distributed as dist
        from krep_b200 import lib, sharding
        self.torch, self.dist, self.lib, self.sharding = torch, dist, lib, sharding
        self.args = args
        self.rank = int(os.environ.get("RANK", "0"))
        self.world = int(os.environ.get("WORLD_SIZE", "1"))
        self.local_rank = int(os.environ.get("LOCAL_RANK", "0"))
        torch.cuda.set_device(self.local_rank)
        self.cpu_group = None
        if self.world > 1:
            dist.init_process_group("nccl", device_id=torch.device("cuda", self.local_rank))
            self.cpu_group = dist.new_group(backend="gloo")   # host-side barrier: no kernel spinning on an idle GPU
        self.L = lib.load()
        assert self.L.krep_b200_init(self.local_rank) == 0, self.L.krep_b200_last_error_string()
        self.stream = torch.cuda.current_stream()
        self.sptr = C.c_void_p(self.stream.cuda_stream)
        self.text = None
        self.gatherer = sharding.KeyGatherer(self.world, self.rank, "cuda") if self.world > 1 else None

    def barrier(self):
        if self.world > 1:
            self.dist.barrier()
        self.torch.cuda.synchronize()

    def ensure_text(self, nbytes):
        if self.text is None or self.text.numel() < nbytes:
            self.text = None
            self.torch.cuda.empty_cache()
            self.text = self.torch.empty(nbytes, dtype=self.torch.uint8, device="cuda")

    def max_over_ranks(self, x):
        if self.world == 1:
            return float(x), [float(x)]
        t = self.torch.tensor([float(x)], dtype=self.torch.float64, device="cuda")
        allv = [self.torch.zeros_like(t) for _ in range(self.world)]
        self.dist.all_gather(allv, t)
        vals = [float(v.item()) for v in allv]
        return max(vals), vals

    # -------------------------------------------------------------------------------------------
    def run(self, name, total_bytes, steps, warmup, sampler=None):
        """One workload on a corpus of total_bytes sharded over all ranks. -> dict (rank 0) / None."""
        torch, dist, lib, L = self.torch, self.dist, self.lib, self.L
        from krep_b200.abi import ALGO_AC, ALGO_AVX2, DeviceResult, Params, Shard
        wl = WORKLOADS[name]
        world, rank = self.world, self.rank
        pats = multi_patterns(wl["multi"], wl["needle"], wl.get("lens", (6, 12))) if wl.get("multi") else None
        maxlen = max(map(len, pats)) if pats else len(wl["needle"])
        halo = maxlen + 1
        g0, own, avail = self.sharding.shard_bounds(total_bytes, world, rank, halo)
        spec = lib.make_spec(SEED, PLANT_SEED, wl["period"], wl["needle"], wl["flags"])
        self.ensure_text(avail + 64)
        assert L.krep_b200_corpus_generate(C.byref(spec), self.text.data_ptr(), g0, avail, self.sptr) == 0
        prev_byte = lib.corpus_host(spec, g0 - 1, 1)[0] if g0 > 0 else -1
        next_byte = lib.corpus_host(spec, g0 + avail, 1)[0] if g0 + avail < total_bytes else -1
        torch.cuda.synchronize()
        # default mode (positions tracked) unless the workload is a -c count; what select_search_algorithm picks
        # (krep.c:1771): AVX2 entry -> SSE4.2 kernel for <= 16 bytes, BMH for -i
        params = Params(pats if pats else wl["needle"], **wl["opts"])
        if pats:
            params.struct.ac_trie = 1
        algo = ALGO_AC if pats else ALGO_AVX2
        plan = L.krep_b200_plan_create(params.ref(), algo)
        lib.check(L)
        shard = Shard(self.text.data_ptr(), avail, 0, own, g0, prev_byte, next_byte)
        dev = DeviceResult()
        res = L.krep_b200_match_result_init(1 << 16)
        count_only = bool(wl["opts"].get("count"))
        g = self.gatherer
        state = {"total": 0, "host_ms": 0.0}

        def finish_single():
            res.contents.count = 0
            return L.krep_b200_collect(plan, params.ref(), C.byref(dev), res)

        if count_only:
            # -c: the fused line count (csrc/scan_count.cu) — only a (lines, flags) record leaves the GPU
            assert world == 1, "the -c side workloads run at N = 1"
            from krep_b200.abi import SIZE_MAX

            class LineCount(C.Structure):
                _fields_ = [("lines", C.c_uint64), ("flags", C.c_uint32), ("reserved", C.c_uint32)]

            L.krep_b200_count_lines_shard.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(Shard), C.c_void_p, C.POINTER(LineCount)]
            L.krep_b200_count_lines_shard.restype = C.c_int
            L.krep_b200_combine_line_counts.argtypes = [C.POINTER(LineCount), C.c_size_t, C.c_size_t]
            L.krep_b200_combine_line_counts.restype = C.c_uint64
            rec = LineCount()

            def count_step():
                rc = L.krep_b200_count_lines_shard(plan, params.ref(), C.byref(shard), self.sptr, C.byref(rec))
                assert rc == 0, L.krep_b200_last_error_string()
                state["total"] = L.krep_b200_combine_line_counts(C.byref(rec), 1, SIZE_MAX)
                return L.krep_b200_last_kernel_ms()

            for _ in range(max(warmup, 3)):
                count_step()
            L.krep_b200_reset_launch_count()
            self.barrier()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(self.stream)
            kernel_ms = [count_step() for _ in range(steps)]
            e1.record(self.stream)
            self.barrier()
            step_ms = e0.elapsed_time(e1) / max(steps, 1)
            k = sum(kernel_ms) / max(len(kernel_ms), 1)
            peak, peak_src = peaks()
            achieved = total_bytes / (k * 1e-3) / 1e9
            self._last = dict(plan=plan, params=params, res=res, pats=pats, algo=algo, total=int(state["total"]),
                              own=own, avail=avail, g0=g0, spec=spec, halo=halo)
            return {"value": total_bytes / (step_ms * 1e-3) / 1e9, "unit": "GB/s", "ms_per_step": step_ms, "steps": steps,
                    "total_bytes": total_bytes, "bytes_per_gpu": total_bytes, "matches": int(state["total"]), "first_matches": [],
                    "filter": L.krep_b200_plan_filter_name(plan).decode() + " + fused line count", "halo": halo,
                    "kernel_ms": k, "kernel_ms_per_rank": [k], "ms_per_step_per_rank": [step_ms], "exchange_ms": 0.0,
                    "exchange_ms_per_rank": [0.0], "rank0_host_ms_per_step": 0.0,
                    "roofline": {"bound": "hbm", "achieved": achieved, "peak": peak, "unit": "GB/s", "frac": achieved / peak,
                                 "kernel_ms": k, "algorithmic_bytes_per_launch": total_bytes, "peak_source": peak_src},
                    "gpu_launches": int(L.krep_b200_launch_count())}

        def process(slot):
            """rank 0, N>1: merge the gathered rows by key and replay them into match_result_t."""
            t0 = time.perf_counter()
            keys, counts = g.fetch(slot)
            res.contents.count = 0
            arr = C.cast(keys.data_ptr(), C.POINTER(C.c_uint64))
            state["total"] = L.krep_b200_replay(algo, params.ref(), False, arr, keys.numel(), None, total_bytes, res)
            state["host_ms"] += (time.perf_counter() - t0) * 1e3

        def scan(ticket_box):
            rc = L.krep_b200_scan_shard_begin(plan, C.byref(shard), 1, self.sptr, C.byref(ticket_box))
            assert rc == 0, L.krep_b200_last_error_string()

        def end(ticket_box):
            rc = L.krep_b200_scan_shard_end(ticket_box.value, C.byref(dev))
            assert rc == 0, L.krep_b200_last_error_string()
            return L.krep_b200_last_kernel_ms()

        tickets = [C.c_int(0), C.c_int(0)]
        # warm-up (N>1: also sizes the exchange buffers on all ranks, collectively)
        for _ in range(max(warmup, 3)):
            scan(tickets[0])
            end(tickets[0])
            if world == 1:
                state["total"] = finish_single()
            else:
                while not g.negotiate(int(dev.stored)):
                    pass
                L.krep_b200_export_packed(C.byref(dev), g.row_ptr(), g.cap, self.sptr)
                g.post(0)
                if rank == 0:
                    process(0)
        # Lists that come back packed with the count (<= 16384 occurrences on every rank) let the steps overlap: scan
        # i+1 (and, N>1, its export + gather) is enqueued before the host waits for scan i, so the GPU runs back to
        # back and all host work of step i (replay; on rank 0 the key merge too) happens while step i+1 scans.
        fits = 1 if int(dev.stored) <= min(16384, g.cap if g else 16384) else 0
        if world > 1:
            ft = torch.tensor([fits], dtype=torch.int64, device="cuda")
            dist.all_reduce(ft, op=dist.ReduceOp.MIN)
            fits = int(ft.item())
        overlapped = bool(fits)
        L.krep_b200_reset_launch_count()
        state["host_ms"] = 0.0
        if sampler is not None and rank == 0:
            sampler.wait_first_sample()
        self.barrier()
        if sampler is not None:
            sampler.mark_begin()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        xa = [torch.cuda.Event(enable_timing=True) for _ in range(steps)]
        xb = [torch.cuda.Event(enable_timing=True) for _ in range(steps)]
        kernel_ms = []

        def exchange(i):
            """N>1: row of step i -> rank 0 (enqueued behind whatever is already on the stream)."""
            xa[i].record(self.stream)
            rc = L.krep_b200_export_packed_async(tickets[i & 1].value, g.row_ptr(), min(g.cap, 16384))
            assert rc == 0, L.krep_b200_last_error_string()
            g.post(i & 1)
            xb[i].record(self.stream)

        self._tickets = tickets
        e0.record(self.stream)
        if overlapped:
            # software pipeline, two scans in flight: the stream always holds the next scan behind the current one; the
            # finish kernel of scan i runs on the library's finish stream while scan i+1 scans; all host work of step i
            # (N=1: replay; rank 0: key merge + replay) happens while scan i+2 is already queued
            for i in range(min(2, steps)):
                scan(tickets[i & 1])
            for i in range(steps):
                if world > 1:
                    exchange(i)
                kernel_ms.append(end(tickets[i & 1]))      # waits for scan i's finish kernel only
                if i + 2 < steps:
                    scan(tickets[i & 1])                   # step i+2 into the slot that has just been ended
                if world == 1:
                    state["total"] = finish_single()
                elif rank == 0:
                    process(i & 1)
        else:
            for i in range(steps):
                scan(tickets[0])
                if world > 1 and rank == 0 and i > 0:
                    process((i - 1) & 1)                   # host work of step i-1 while scan i runs
                kernel_ms.append(end(tickets[0]))
                if world == 1:
                    state["total"] = finish_single()
                else:
                    xa[i].record(self.stream)
                    L.krep_b200_export_packed(C.byref(dev), g.row_ptr(), g.cap, self.sptr)
                    g.post(i & 1)
                    xb[i].record(self.stream)
            if world > 1 and rank == 0 and steps:
                process((steps - 1) & 1)
        e1.record(self.stream)
        self.barrier()
        if sampler is not None:
            sampler.mark_end()
        elapsed_ms = e0.elapsed_time(e1)
        launches = int(L.krep_b200_launch_count())
        exch = sum(a.elapsed_time(b) for a, b in zip(xa, xb)) / max(steps, 1) if world > 1 else 0.0
        step_max, step_all = self.max_over_ranks(elapsed_ms / max(steps, 1))
        k_max, k_all = self.max_over_ranks(sum(kernel_ms) / max(len(kernel_ms), 1))
        x_max, x_all = self.max_over_ranks(exch)
        if world > 1:
            flag = torch.tensor([1 if (rank == 0 and g.overflowed) else 0], dtype=torch.int64, device="cuda")
            dist.all_reduce(flag)
            assert int(flag.item()) == 0, "key exchange overflowed its buffers in the timed loop"
        out = None
        if rank == 0:
            peak, peak_src = peaks()
            per_gpu = total_bytes / world
            achieved = per_gpu / (k_max * 1e-3) / 1e9
            first = [(res.contents.positions[i].start_offset, res.contents.positions[i].end_offset)
                     for i in range(min(3, res.contents.count))]
            out = {
                "value": total_bytes / (step_max * 1e-3) / 1e9, "unit": "GB/s", "ms_per_step": step_max, "steps": steps,
                "total_bytes": total_bytes, "bytes_per_gpu": int(per_gpu), "matches": int(state["total"]), "first_matches": first,
                "filter": L.krep_b200_plan_filter_name(plan).decode(), "halo": halo,
                "kernel_ms": k_max, "kernel_ms_per_rank": k_all, "ms_per_step_per_rank": step_all,
                "exchange_ms": x_max, "exchange_ms_per_rank": x_all, "rank0_host_ms_per_step": state["host_ms"] / max(steps, 1),
                "steps_overlapped": overlapped,
                "roofline": {"bound": "hbm", "achieved": achieved, "peak": peak, "unit": "GB/s", "frac": achieved / peak,
                             "kernel_ms": k_max, "algorithmic_bytes_per_launch": int(per_gpu), "peak_source": peak_src},
                "gpu_launches": launches,
            }
        self._last = dict(plan=plan, params=params, res=res, pats=pats, algo=algo, total=int(state["total"]),
                          own=own, avail=avail, g0=g0, spec=spec, halo=halo)
        return out

    def drain(self):
        """After an exception inside a workload: end whatever scans are still in flight so the next workload starts clean."""
        from krep_b200.abi import DeviceResult
        junk = DeviceResult()
        for t in getattr(self, "_tickets", []):
            self.L.krep_b200_scan_shard_end(t.value, C.byref(junk))
        self.torch.cuda.synchronize()

    def release_last(self):
        last = getattr(self, "_last", None)
        if last:
            last["params"].struct.ac_trie = None
            self.L.krep_b200_plan_destroy(last["plan"])
            self.L.krep_b200_match_result_free(last["res"])
            self._last = None

    # -------------------------------------------------------------------------------------------
    def e2e(self, name, total_bytes, steps):
        """The same metric through the search_func_t entry point on PINNED HOST text, copies inside the timed region.
        N = 1: this process, its GPU.  N > 1: ONE call in ONE process (rank 0) that spreads the text over all N GPUs
        (krep_b200_set_devices) — what a krep host calling the drop-in gets; the other ranks wait on a host barrier."""
        torch, lib, L = self.torch, self.lib, self.L
        last = self._last
        wl = WORKLOADS[name]
        world, rank = self.world, self.rank
        out = None
        if rank == 0:
            # the whole text in pinned host memory; if the box cannot pin that much, a prefix of it (stated in the output)
            want_bytes = total_bytes
            try:
                with open("/proc/meminfo") as f:
                    avail_kb = next(int(ln.split()[1]) for ln in f if ln.startswith("MemAvailable"))
                while total_bytes > (16 << 30) and total_bytes > avail_kb * 1024 // 2:
                    total_bytes //= 2
            except Exception:  # noqa: BLE001
                pass
            host = None
            t_alloc = time.perf_counter()
            while host is None:
                try:
                    host = torch.empty(total_bytes, dtype=torch.uint8, pin_memory=True)
                except RuntimeError:
                    if total_bytes <= (1 << 30):
                        raise
                    total_bytes //= 2
            total_bytes -= total_bytes % 16
            t_alloc = time.perf_counter() - t_alloc
            piece = min(self.text.numel() - 64, total_bytes) // 16 * 16
            for off in range(0, total_bytes, piece):     # materialise the whole corpus in host memory through GPU 0
                ln = min(piece, total_bytes - off)
                assert L.krep_b200_corpus_generate(C.byref(last["spec"]), self.text.data_ptr(), off, ln, self.sptr) == 0
                host[off:off + ln].copy_(self.text[:ln])
            torch.cuda.synchronize()
            entry = "aho_corasick" if last["pats"] else "avx2"
            fn = getattr(L, lib.SEARCH_ENTRIES[entry])
            params, res = last["params"], last["res"]
            L.krep_b200_set_only_matching(False)
            devs = (C.c_int * world)(*range(world))
            L.krep_b200_set_devices(devs, world)

            def e2e_step():
                res.contents.count = 0
                c = fn(params.ref(), C.c_void_p(host.data_ptr()), total_bytes, res)
                lib.check(L)
                return int(c)

            e2e_step()                                     # warm-up: contexts on every device, rings, plan uploads
            t0 = time.perf_counter()
            got = 0
            for _ in range(steps):
                got = e2e_step()
            dt = (time.perf_counter() - t0) / steps
            L.krep_b200_set_devices(None, 0)
            out = {"value": total_bytes / dt / 1e9, "unit": "GB/s", "h2d_bytes_per_step": total_bytes,
                   "d2h_bytes_per_step": 8 * world + 8 * got, "ms_per_step": dt * 1e3, "steps": steps,
                   "api": lib.SEARCH_ENTRIES[entry] + "(params, pinned host text, len, match_result_t*) — one call, one process, "
                          f"{world} device(s) (krep_b200_set_devices)",
                   "bytes": total_bytes, "full_corpus": total_bytes == want_bytes, "matches": got,
                   "agrees_with_device_path": (got == last["total"]) if total_bytes == want_bytes else None,
                   "scan_kernel_ms_slowest_device": float(L.krep_b200_last_kernel_ms()), "pinned_alloc_s": t_alloc}
            del host
        if world > 1:
            self.dist.barrier(group=self.cpu_group)
        return out


DUMP_BYTES = 64 << 20


def dump_outputs(out_dir, last):
    """The headline's last timed step as its caller received it: the count krep reports and the match_result_t
    offsets as (start, end) rows, float64 (exact below 2^53).  A list too long for DUMP_BYTES is reduced to a fixed,
    seeded sample of rows; their row numbers go to positions_rows.npy."""
    import numpy as np
    os.makedirs(out_dir, exist_ok=True)
    res = last["res"].contents
    n = int(res.count)
    np.save(os.path.join(out_dir, "matches.npy"), np.array([last["total"]], dtype=np.float64))
    pos = np.zeros((0, 2), dtype=np.float64)
    if n:
        raw = np.ctypeslib.as_array(C.cast(res.positions, C.POINTER(C.c_uint64)), shape=(n, 2))
        cap = (DUMP_BYTES - (1 << 20)) // 24            # 16 B per row + 8 B for its row number
        if n > cap:
            rows = np.unique(np.random.default_rng(0x5EED0004).integers(0, n, size=cap))
            np.save(os.path.join(out_dir, "positions_rows.npy"), rows.astype(np.float64))
            raw = raw[rows]
        pos = raw.astype(np.float64)
    np.save(os.path.join(out_dir, "positions.npy"), pos)


def _main(out_stream):
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--gib", type=float, default=10.0, help="headline corpus GiB per GPU")
    ap.add_argument("--workload", default="literal8", choices=list(WORKLOADS))
    ap.add_argument("--cpu-sample-gib", type=float, default=2.0)
    ap.add_argument("--e2e-steps", type=int, default=3)
    ap.add_argument("--side-steps", type=int, default=10)
    ap.add_argument("--no-e2e", action="store_true")
    ap.add_argument("--no-cpu", action="store_true")
    ap.add_argument("--no-side", action="store_true", help="skip the BASELINE configs[2..4] side workloads")
    ap.add_argument("--dump-outputs", metavar="DIR", help="write the headline's last-step outputs as .npy files to DIR")
    args = ap.parse_args()
    args.warmup = max(args.warmup, 0)
    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    wl = WORKLOADS[args.workload]
    metric = "GB/s scanned (HBM-resident corpus)"
    config = workload_config(wl, args.gib, world)

    if args.impl == "reference":
        if rank != 0:
            return
        sample = int(min(args.cpu_sample_gib, args.gib) * GIB)
        r = run_cpu_reference(args.workload, wl, sample, max(args.steps, 1), args.warmup)
        config["cpu_slice_bytes"] = r["sample_bytes"]
        print(json.dumps({
            "impl": "reference", "metric": metric, "value": r["value"], "unit": "GB/s", "n_gpus": args.gpus,
            "steps": args.steps, "warmup": args.warmup, "ms_per_step": r["ms"], "higher_is_better": True,
            "scaling": "weak", "vs_baseline": None, "dtype": "u8", "data": "synthetic", "config": config,
            "cpu_baseline": {k: r[k] for k in CPU_KEYS if k in r},
            "e2e": {"value": r["value"], "unit": "GB/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
            "matches_in_sample": r["count"],
        }), file=out_stream)
        return

    R = Runner(args)
    torch, dist = R.torch, R.dist
    n = int(args.gib * GIB)
    n -= n % 16
    sampler = ClockSampler(R.local_rank)
    if rank == 0:
        sampler.start()
    try:
        head = R.run(args.workload, world * n, args.steps, args.warmup, sampler)  # weak scaling: n owned bytes per GPU
    finally:
        clocks = sampler.stop() if rank == 0 else None                            # never leave nvidia-smi running
    if args.dump_outputs and rank == 0:
        dump_outputs(args.dump_outputs, R._last)
    e2e = None
    if not args.no_e2e:
        e2e = R.e2e(args.workload, world * n, args.e2e_steps)
    R.release_last()

    side = {}
    if not args.no_side and args.workload == "literal8":
        todo = list(SIDE_WORKLOADS) + (list(DENSITY_WORKLOADS) if world == 1 else [])
        for name, total_gib in todo:
            total = int(total_gib * GIB) // (16 * world) * (16 * world)
            try:
                r = R.run(name, total, args.side_steps if (name, total_gib) in SIDE_WORKLOADS else 3, 3)
            except Exception as e:  # noqa: BLE001  (all ranks fail alike: sizes and code are identical)
                R.drain()
                r = {"error": str(e)} if rank == 0 else None
            R.release_last()
            if rank == 0 and r is not None:
                r["config"] = workload_config(WORKLOADS[name], total_gib / world, world, total_gib)
                r["scaling"] = "strong" if (name, total_gib) in SIDE_WORKLOADS else "n/a (N = 1 only)"
                side[name] = r

    if rank != 0:
        if world > 1:
            dist.destroy_process_group()
        return
    R.text = None
    torch.cuda.empty_cache()

    out = {
        "metric": metric, "value": head["value"], "unit": "GB/s", "n_gpus": world, "steps": args.steps, "warmup": max(args.warmup, 3),
        "ms_per_step": head["ms_per_step"], "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "u8",
        "data": "synthetic", "config": dict(config, filter=head["filter"],
                                            parallelism=f"{world} shard(s), owned by match start, halo {head['halo']} B"),
        "matches": head["matches"], "first_matches": head["first_matches"],
        "roofline": dict(head["roofline"], note="achieved = corpus bytes of one shard / mean scan-kernel duration (CUDA events on the "
                                               "launching stream, inside the timed region; max over ranks)"),
        "kernel_ms_per_rank": head["kernel_ms_per_rank"], "ms_per_step_per_rank": head["ms_per_step_per_rank"],
        "exchange_ms": head["exchange_ms"], "exchange_ms_per_rank": head["exchange_ms_per_rank"],
        "rank0_host_ms_per_step": head["rank0_host_ms_per_step"], "steps_overlapped": head.get("steps_overlapped"),
        "gpu_launches": head["gpu_launches"], "clocks": clocks,
    }
    if e2e:
        out["e2e"] = e2e
    if not args.no_cpu and world == 1:
        try:
            r = run_cpu_reference(args.workload, wl, int(min(args.cpu_sample_gib, args.gib) * GIB), 3, 1)
            out["cpu_baseline"] = {k: r[k] for k in CPU_KEYS if k in r}
            out["cpu_baseline"]["matches_in_sample"] = r["count"]
            out["config"]["cpu_slice_bytes"] = r["sample_bytes"]
        except Exception as e:  # noqa: BLE001
            out["cpu_baseline"] = {"error": str(e)}
        for name, r in side.items():
            if "error" in r:
                continue
            try:
                c = run_cpu_reference(name, WORKLOADS[name], 1 << 30, 2, 1)
                r["cpu_baseline"] = {k: c[k] for k in CPU_KEYS if k in c}
                r["cpu_baseline"]["matches_in_sample"] = c["count"]
            except Exception as e:  # noqa: BLE001
                r["cpu_baseline"] = {"error": str(e)}
    if side:
        out["workloads"] = side
    print(json.dumps(out), file=out_stream)
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
