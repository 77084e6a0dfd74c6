"""Build recipe for libkrep_b200.so (the product: CUDA kernels + C ABI), in-tree, sm_90a only."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, "libkrep_b200.so")
SOURCES = ["engine.cu", "scan_literal.cu", "scan_multi.cu", "scan_count.cu", "scan_set_count.cu", "scan_regex.cu", "scan_regex_long.cu", "scan_regex_pack.cu", "scan_batch_gather.cu",
           "host_api.cu",
           "semantics.cpp", "regex_dfa.cpp", "regex_rows.cpp"]
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
         "-Xcompiler", "-fPIC,-fopenmp,-Wall,-Wno-unused-function", "-Xptxas", "-v"]


def _stale(target, deps):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(HERE, "..", "include", "krep_b200.h")]
    objdir = os.path.join(HERE, "build")
    os.makedirs(objdir, exist_ok=True)
    objs = []
    procs = []
    for src in SOURCES:
        obj = os.path.join(objdir, src.rsplit(".", 1)[0] + ".o")
        objs.append(obj)
        if force or _stale(obj, deps):
            cmd = [NVCC, *FLAGS, "-c", os.path.join(CSRC, src), "-o", obj]
            procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    failed = False
    for src, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            sys.stderr.write(f"--- nvcc {src} failed ---\n{out}\n")
            failed = True
        elif verbose:
            print(f"--- {src} ---\n{out}")
    if failed:
        raise RuntimeError("krep_b200 build failed")
    if procs or force or _stale(OUT, objs):
        cmd = [NVCC, "-shared", "-o", OUT, *objs, "-Xcompiler", "-fopenmp", "-lgomp"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            sys.stderr.write(r.stdout + r.stderr)
            raise RuntimeError("krep_b200 link failed")
    return OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
