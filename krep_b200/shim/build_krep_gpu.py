"""Builds the drop-in demonstration: the reference's own krep CLI with its search kernels replaced by
libkrep_b200.so.

Nothing from the reference is committed: krep.c is read where it lies (KREP_REF_DIR, default
/root/reference), three textual edits are applied in memory (each anchor must occur exactly once), the
result is compiled with gcc against include/krep_b200.h into oracle/_ref/ (git-ignored, beside the other
binaries built from the reference sources).

  1. #include "krep_b200.h" after krep.c's own includes (krep.h is included first, so the header's
     type restatement is skipped and krep's own search_params_t / match_result_t are used);
  2. the stock select_search_algorithm (krep.c:1771) is renamed select_search_algorithm_cpu and
     krep_b200_dispatch.inc is appended: the new select_search_algorithm mirrors the -o / --no-simd /
     --algo globals into the library and returns the krep_b200_* function;
  3. search_file hands the whole file to ONE search call (krep.c:2765: the single-chunk branch) — the GPU
     does its own tiling, and the result is the reference's -t 1 result rather than its multi-thread
     chunk-edge artefacts (SURVEY §8 a12).  -E searches too, when the library takes the pattern (krep's
     regex chunks do not overlap, so a match across a chunk edge would be lost); a refused pattern keeps
     krep's own threading;
  4. main calls krep_b200_warmup() right before it starts searching (krep.c:3818; for -E only when the library
     takes the pattern), and the file is mapped
     without MAP_POPULATE for literal searches (krep.c:2679): CUDA start-up overlaps the file handling.

The output binary is oracle/_ref/krep_gpu: same CLI, same output code, GPU scan.
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF_DIR = os.environ.get("KREP_REF_DIR", "/root/reference")
OUT_DIR = os.path.join(ROOT, "oracle", "_ref")
LIB_DIR = os.path.join(ROOT, "krep_b200")


def _replace_once(src, old, new, what):
    if src.count(old) != 1:
        raise RuntimeError(f"build_krep_gpu: anchor for {what} found {src.count(old)} times (expected 1)")
    return src.replace(old, new)


def patched_source():
    with open(os.path.join(REF_DIR, "krep.c")) as f:
        src = f.read()
    src = _replace_once(src, '#include "aho_corasick.h"', '#include "aho_corasick.h"\n#include "krep_b200.h"',
                        "the include")
    src = _replace_once(src, "search_func_t select_search_algorithm(const search_params_t *params)\n{",
                        "static search_func_t select_search_algorithm_cpu(const search_params_t *params)\n{",
                        "select_search_algorithm")
    src = _replace_once(src, "    run_single_thread_inline = (actual_thread_count == 1);",
                        "    if (!current_params.use_regex || krep_b200_select_search_algorithm(&current_params))\n"
                        "        actual_thread_count = 1; /* krep_b200: one call per file */\n"
                        "    run_single_thread_inline = (actual_thread_count == 1);", "the chunk count")
    # 4. start-up: the GPU context comes up on a background thread while search_file opens and maps the file, and the
    #    mapping is not pre-populated by one kernel thread (the library's staging threads fault it in, in parallel)
    src = _replace_once(src, "    // --- Execute Search ---\n    int exit_code = 1;",
                        "    if (!params.use_regex || krep_b200_select_search_algorithm(&params))\n"
                        "        krep_b200_warmup(); /* krep_b200: context creation overlaps the file handling */\n"
                        "    // --- Execute Search ---\n    int exit_code = 1;", "the warm-up call")
    src = _replace_once(src, "int mmap_flags_populate = mmap_base_flags | MAP_POPULATE;",
                        "int mmap_flags_populate = mmap_base_flags | ((current_params.use_regex || getenv(\"KREP_B200_MAP_POPULATE\")) ? MAP_POPULATE : 0); /* krep_b200 */",
                        "MAP_POPULATE")
    with open(os.path.join(HERE, "krep_b200_dispatch.inc")) as f:
        src += "\n" + f.read()
    return src


def available():
    return os.path.isfile(os.path.join(REF_DIR, "krep.c"))


def build(force=False):
    """-> path of the GPU-backed krep CLI, or None when neither the reference sources nor a prebuilt binary exist."""
    out = os.path.join(OUT_DIR, "krep_gpu")
    if not available():
        return out if os.path.exists(out) else None
    os.makedirs(OUT_DIR, exist_ok=True)
    csrc = os.path.join(OUT_DIR, "krep_b200_patched.c")
    deps = [os.path.join(REF_DIR, "krep.c"), os.path.join(REF_DIR, "aho_corasick.c"),
            os.path.join(HERE, "krep_b200_dispatch.inc"), os.path.join(ROOT, "include", "krep_b200.h"), __file__]
    if not force and os.path.exists(out) and all(os.path.getmtime(d) <= os.path.getmtime(out) for d in deps):
        return out
    with open(csrc, "w") as f:
        f.write(patched_source())
    cmd = ["gcc", "-O3", "-std=c11", "-pthread", "-D_GNU_SOURCE", "-D_DEFAULT_SOURCE", "-msse4.2", "-mavx2", "-w",
           "-I", REF_DIR, "-I", os.path.join(ROOT, "include"), "-o", out, csrc, os.path.join(REF_DIR, "aho_corasick.c"),
           "-L", LIB_DIR, "-lkrep_b200", "-Wl,-rpath,$ORIGIN/../../krep_b200"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    os.unlink(csrc)  # the patched copy of the reference source is never kept
    if r.returncode != 0:
        sys.stderr.write(" ".join(cmd) + "\n" + r.stdout + r.stderr)
        raise RuntimeError("krep_gpu build failed")
    return out


if __name__ == "__main__":
    print(build(force="--force" in sys.argv))
