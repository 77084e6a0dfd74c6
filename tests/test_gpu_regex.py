"""-E on the GPU: krep_b200_regex_search (device line filter + regexec on the flagged lines) must return exactly what
the reference's regex_search returns — count, every (start, end), their order — and the relinked CLI must print what
the stock CLI prints with -t 1."""
import ctypes as C
import os
import random
import subprocess
import sys

import pytest

from krep_b200 import lib
from krep_b200.abi import ALGO_REGEX, Params
import oracle_util as ou
import regex_util as ru

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu


def _params(pats, **kw):
    if isinstance(pats, str):
        pats = [pats]
    return Params([p.encode() for p in pats], regex=True, **kw)


def _want(P, text):
    chk = ou.reference()
    if chk is None:
        return ru.ref_regex_search(P, text)
    f = chk.lib.regex_search
    f.argtypes = ou._SIG
    f.restype = C.c_uint64
    res = chk._new(16)
    try:
        cnt = f(P.ref(), C.create_string_buffer(text, len(text) + 1).raw, len(text), res)
        r = res.contents
        return int(cnt), [(r.positions[i].start_offset, r.positions[i].end_offset) for i in range(r.count)]
    finally:
        chk._free(res)


def _check(pats, text, **kw):
    P = _params(pats, **kw)
    got = lib.search("regex", P, text)
    want = _want(P, text)
    assert got == want, (pats, kw, len(text), got[0], want[0], got[1][:5], want[1][:5])
    return got


@pytest.fixture(scope="module", autouse=True)
def _init():
    L = lib.load()
    assert L.krep_b200_init(0) == 0, L.krep_b200_last_error_string()


OPTS = [dict(), dict(count=True), dict(count=True, only_matching=True), dict(case_sensitive=False), dict(whole_word=True),
        dict(max_count=1), dict(max_count=7)]


def test_random_texts_all_options():
    rng = random.Random(11)
    pats = ["a+b", "^a", "b$", "(ab|ba)c?", "[0-9]x", "\\<a.b", "x*", "^", "$", "^$", ".", "[^ab]{2}", "A_", "\\bab\\b"]
    for pat in pats:
        for kw in OPTS:
            for n in (0, 1, 37, 1000, 20000):
                _check(pat, ru.random_text(rng, n), **kw)
    for kw in OPTS:
        _check(["ab", "x[0A]", "^c"], ru.random_text(rng, 5000), **kw)  # several -e patterns


def test_edge_texts():
    for text in (b"", b"\n", b"\n\n\n", b"abc", b"abc\n", b"a\n\nb\n\n", b"ab\nab"):
        for pat in ("x*", "^", "$", "^$", "b", "a|$"):
            for kw in OPTS:
                _check(pat, text, **kw)


SPEC = (0x5EED0001, 0x5EED0002, 1 << 16, b"qzXv9Kpw")


@pytest.mark.parametrize("pat,kw", [
    ("qzXv[0-9]Kpw", {}), ("[A-Z][a-z]+[0-9]x", {}), ("(qzxv|the ) ?e", {"case_sensitive": False}), ("the[a-z]*", {"count": True}),
    ("the[a-z]*", {"count": True, "only_matching": True}), ("^[a-z]+ [a-z]+$", {}), ("[0-9]{4}", {}), ("etao", {"whole_word": True}),
    ("th(e|a)", {"max_count": 7}),
])
def test_corpus_slices(pat, kw):
    text = lib.corpus_host(lib.make_spec(*SPEC), 0, 6 << 20)
    _check(pat, text, **kw)


def test_line_longer_than_the_kernel_bound():
    rng = random.Random(5)
    long_line = bytes(rng.choice(b"abcdef ") for _ in range(1 << 20))
    text = b"x1\n" + long_line + b"qq9\n" + b"ab\n" + long_line[:300000] + b"\nqq7"
    for pat in ("qq[0-9]", "^x", "f a", "q$", "^ab$"):
        for kw in (dict(), dict(count=True)):
            _check(pat, text, **kw)


def test_lines_cut_by_staging_chunks(monkeypatch):
    monkeypatch.setenv("KREP_B200_STAGE_MB", "1")
    monkeypatch.setenv("KREP_B200_CHUNK_MB", "1")
    monkeypatch.setenv("KREP_B200_RANGES", "3")
    text = lib.corpus_host(lib.make_spec(*SPEC), 0, (5 << 20) + 12345)
    for pat, kw in (("qzXv[0-9]Kpw", {}), ("the[a-z]*", {"count": True}), ("^[a-z]+$", {}), ("e t", {"max_count": 100000})):
        _check(pat, text, **kw)


def test_lines_cut_across_devices(monkeypatch):
    if lib.load().krep_b200_device_count() < 2:
        pytest.skip("needs two or more GPUs")
    monkeypatch.setenv("KREP_B200_DEVICES", str(lib.load().krep_b200_device_count()))
    monkeypatch.setenv("KREP_B200_STAGE_MB", "1")
    monkeypatch.setenv("KREP_B200_CHUNK_MB", "1")
    text = lib.corpus_host(lib.make_spec(*SPEC), 0, (6 << 20) + 777)
    for pat, kw in (("qzXv[0-9]Kpw", {}), ("the[a-z]*", {"count": True}), ("^[a-z]+ ", {})):
        _check(pat, text, **kw)


@pytest.mark.parametrize("nshards", [2, 3])
def test_resident_shards_replay(nshards):
    import torch
    import gpu_util as gu
    L = lib.load()
    text = lib.corpus_host(lib.make_spec(*SPEC), 0, (3 << 20) + 101)
    n = len(text)
    for pat, kw in (("qzXv[0-9]Kpw", {}), ("the[a-z]*", {"count": True}), ("^[a-z]+ [a-z]+$", {"max_count": 50})):
        P = _params(pat, **kw)
        plan = L.krep_b200_plan_create(P.ref(), ALGO_REGEX)
        lib.check(L)
        assert plan
        try:
            t = gu.to_device(text)
            keys = []
            cut = [(n * i // nshards) & ~15 for i in range(nshards)] + [n]
            for i in range(nshards):
                b, e = cut[i], cut[i + 1]
                halo_end = min(e + 8192, n)
                shard = t[b:]
                dev = gu.scan(plan, shard, halo_end - b, 0, e - b, b, text[b - 1] if b else -1, text[halo_end] if halo_end < n else -1)
                out = torch.empty(max(dev.stored, 1), dtype=torch.int64, device="cuda")
                assert L.krep_b200_export_keys(C.byref(dev), out.data_ptr(), dev.stored, None) == 0
                torch.cuda.synchronize()
                keys += [int(k) for k in out[: dev.stored].cpu().tolist()]
            assert keys == sorted(keys)
            arr = (C.c_uint64 * max(len(keys), 1))(*keys)
            res = L.krep_b200_match_result_init(16)
            try:
                cnt = L.krep_b200_replay(ALGO_REGEX, P.ref(), False, arr, len(keys), text, n, res)
                lib.check(L)
                r = res.contents
                got = (int(cnt), [(r.positions[i].start_offset, r.positions[i].end_offset) for i in range(r.count)])
            finally:
                L.krep_b200_match_result_free(res)
            assert got == lib.search("regex", P, text) == _want(P, text), (pat, kw)
        finally:
            L.krep_b200_plan_destroy(plan)


def test_batch_refuses_regex():
    L = lib.load()
    with pytest.raises(RuntimeError):
        lib.search_batch("regex", _params("ab"), [b"ab\n", b"cab"])
    L.krep_b200_last_error()


CLI_CASES = [["-E", "qz[A-Z]v"], ["-c", "-E", "the[a-z]*"], ["-o", "-E", "[0-9]{2}"], ["-i", "-E", "NEEDLE|fox"],
             ["-w", "-E", "ab(ab)?"], ["-m", "3", "-E", "the"], ["-c", "-o", "-E", "a+"], ["-E", "-e", "^the", "-e", "x$"],
             ["-c", "-E", "^$"], ["-c", "-E", "ab\\sab"]]  # the last one is refused (\s): CPU regex_search through the fallback


def test_cli_dropin_regex(tmp_path):
    sys.path.insert(0, os.path.join(ROOT, "krep_b200", "shim"))
    sys.path.insert(0, os.path.join(ROOT, "oracle"))
    import build_krep_gpu
    import build_oracle
    stock = build_oracle.build_ref()[1]
    gpu = build_krep_gpu.build()
    if not stock or not gpu:
        pytest.skip("stock or GPU-backed krep binary not available (built only where the reference sources are)")
    env = {k: v for k, v in os.environ.items() if k != "KREP_B200_KEEP_VISIBLE"}
    rng = random.Random(3)
    words = [b"the", b"quick", b"fox", b"NEEDLE", b"needle", b"ab", b"abab", b"12", b"7", b"x", b"qzXv", b"aa"]
    body = bytearray()
    while len(body) < 300_000:
        body += rng.choice(words) + rng.choice([b" ", b" ", b"\n", b"", b"\n\n"])
    path = tmp_path / "corpus.txt"
    path.write_bytes(bytes(body))
    for flags in CLI_CASES:
        a = subprocess.run([stock, "-t", "1", "--color=never", *flags, str(path)], capture_output=True)
        b = subprocess.run([gpu, "--color=never", *flags, str(path)], capture_output=True, env=env)
        assert (b.returncode, b.stdout) == (a.returncode, a.stdout), (flags, a.stdout[:300], b.stdout[:300], b.stderr[:300])
    for flags in (["-c", "-E", "-s", "a+b", "aab ab\nb"], ["-o", "-E", "-s", "[0-9]+", "a12 b3"]):
        a = subprocess.run([stock, "--color=never", *flags], capture_output=True)
        b = subprocess.run([gpu, "--color=never", *flags], capture_output=True, env=env)
        assert (b.returncode, b.stdout) == (a.returncode, a.stdout), (flags, a.stdout, b.stdout, b.stderr)
    a = subprocess.run([stock, "--color=never", "-E", "s?he"], input=b"ushers and hers\nshe sells\n", capture_output=True)
    b = subprocess.run([gpu, "--color=never", "-E", "s?he"], input=b"ushers and hers\nshe sells\n", capture_output=True, env=env)
    assert (b.returncode, b.stdout) == (a.returncode, a.stdout), (a.stdout, b.stdout, b.stderr)
