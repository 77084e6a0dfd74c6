"""The drop-in demonstration (SURVEY §8b, INTEGRATION.md): the reference's own krep CLI, relinked so that
select_search_algorithm returns the krep_b200_* entry points, must print exactly what the stock CLI prints
with -t 1 — same lines, same counts, same exit status — for every flag that reaches the hot path."""
import os
import random
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "krep_b200", "shim"))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import build_krep_gpu  # noqa: E402
import build_oracle  # noqa: E402


def test_patch_anchors_apply_to_the_reference_source():
    if not build_krep_gpu.available():
        pytest.skip("reference sources not present")
    src = build_krep_gpu.patched_source()
    assert "select_search_algorithm_cpu" in src and "krep_b200_select_search_algorithm(params)" in src


def _visible_gpus():
    try:
        out = subprocess.run(["nvidia-smi", "-L"], capture_output=True, text=True).stdout
        n = sum(1 for ln in out.splitlines() if ln.startswith("GPU "))
    except OSError:
        return 0
    cvd = os.environ.get("CUDA_VISIBLE_DEVICES")
    return min(n, len([x for x in cvd.split(",") if x])) if cvd else n


def _text(rng, n):
    words = [b"the", b"quick", b"Brown", b"fox_1", b"needle", b"NEEDLE", b"Needle", b"ab", b"abab", b"aaa", b"x",
             b"haystack", b"needleneedle", b"aba"]
    out = bytearray()
    while len(out) < n:
        out += rng.choice(words)
        out += rng.choice([b" ", b" ", b" ", b"\n", b"", b",", b"_", b". "])
    return bytes(out[:n])


CASES = [
    ["needle"], ["-c", "needle"], ["-o", "needle"], ["-c", "-o", "needle"], ["-i", "needle"], ["-w", "needle"],
    ["-i", "-w", "-c", "needle"], ["-m", "7", "needle"], ["-c", "-m", "3", "the"], ["-o", "-m", "5", "aba"],
    ["--algo=bm", "-c", "the"], ["--algo=kmp", "-o", "abab"], ["--no-simd", "-o", "aba"], ["-o", "aaa"], ["-o", "x"],
    ["-o", "ab"], ["-i", "-o", "ab"], ["-c", "zzzz-not-there"], ["-e", "needle", "-e", "fox_1", "-e", "quick Br"],
    ["-o", "-e", "ab", "-e", "abab", "-e", "aba"], ["-i", "-c", "-e", "NEEDLE", "-e", "the"],
    ["-w", "-o", "-e", "needle", "-e", "aaa"], ["the quick Brown fox_1 needle"], ["-F", "-c", "fox_1"],
]


@pytest.mark.gpu
@pytest.mark.parametrize("size", [900, 70_000, 9_000_000])
def test_gpu_krep_prints_what_stock_krep_prints(tmp_path, size):
    stock = build_oracle.build_ref()[1]
    gpu = build_krep_gpu.build()
    if not stock or not gpu:
        pytest.skip("stock or GPU-backed krep binary not available (built only where the reference sources are)")
    # the CLI is a one-shot process: let the library hide the GPUs it does not use (conftest keeps them visible for the
    # in-process tests), or every invocation pays cuInit for the whole box
    env_gpu = {k: v for k, v in os.environ.items() if k != "KREP_B200_KEEP_VISIBLE"}
    rng = random.Random(size)
    path = tmp_path / "corpus.txt"
    path.write_bytes(_text(rng, size))
    pats = tmp_path / "pats.txt"
    pats.write_bytes(b"needle\nquick\nfox_1 ne\nabab\n")
    # every GPU-backed process pays a CUDA context creation (seconds), so the full flag matrix runs on one size only
    if size == 70_000:
        cases = CASES + [["-f", str(pats)], ["-c", "-f", str(pats)]]
    elif size < 70_000:
        cases = [["needle"], ["-c", "-w", "needle"], ["-o", "aba"], ["-i", "-o", "-e", "NEEDLE", "-e", "the"],
                 ["-o", "-m", "2", "ab"], ["-c", "zzzz-not-there"]]
    else:
        cases = [["-c", "needle"], ["-c", "-o", "-i", "needle"], ["-c", "-w", "-e", "needle", "-e", "fox_1", "-e", "quick Br"],
                 ["-c", "-m", "1000", "the quick Brown fox_1 needle"]]
    for flags in cases:
        a = subprocess.run([stock, "-t", "1", "--color=never", *flags, str(path)], capture_output=True)
        b = subprocess.run([gpu, "--color=never", *flags, str(path)], capture_output=True, env=env_gpu)
        assert (b.returncode, b.stdout) == (a.returncode, a.stdout), (flags, a.stdout[:300], b.stdout[:300], b.stderr[:300])
    # the same file spread over every GPU of the box inside the one search call (1 MiB chunks so that every device gets a
    # range): the output must not change
    ndev = _visible_gpus()
    if size == 9_000_000 and ndev >= 2:
        env = dict(env_gpu, KREP_B200_DEVICES=str(ndev), KREP_B200_STAGE_MB="1", KREP_B200_CHUNK_MB="1")
        for flags in cases + [["-o", "-e", "needle", "-e", "fox_1 ne", "-e", "ab"]]:
            a = subprocess.run([stock, "-t", "1", "--color=never", *flags, str(path)], capture_output=True)
            b = subprocess.run([gpu, "--color=never", *flags, str(path)], capture_output=True, env=env)
            assert (b.returncode, b.stdout) == (a.returncode, a.stdout), (ndev, flags, a.stdout[:300], b.stdout[:300], b.stderr[:300])
    if size != 900:
        return
    # -s STRING and stdin go through search_string (krep.c:1999): no sort, bare count
    for flags in (["-c", "-s", "aba", "abababa"], ["-i", "-o", "-s", "NEEDLE", "a needle in a Needle stack"]):
        a = subprocess.run([stock, "--color=never", *flags], capture_output=True)
        b = subprocess.run([gpu, "--color=never", *flags], capture_output=True, env=env_gpu)
        assert (b.returncode, b.stdout) == (a.returncode, a.stdout), (flags, a.stdout, b.stdout, b.stderr)
    for flags in (["-o", "-e", "he", "-e", "she", "-e", "hers"], ["-c", "she"]):
        a = subprocess.run([stock, "--color=never", *flags], input=b"ushers and hers\nshe sells\n", capture_output=True)
        b = subprocess.run([gpu, "--color=never", *flags], input=b"ushers and hers\nshe sells\n", capture_output=True, env=env_gpu)
        assert (b.returncode, b.stdout) == (a.returncode, a.stdout), (flags, a.stdout, b.stdout, b.stderr)
