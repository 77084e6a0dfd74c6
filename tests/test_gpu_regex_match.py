"""-E offsets on the GPU: a positions or -co call whose offsets the device computes (krep_b200_regex_match_mode == 1)
must return what the reference's regex_search returns, what the regexec path (KREP_B200_NO_DEVICE_MATCHES=1) returns,
and what the same decision procedure run on the host (krep_b200_regex_matches_host) returns — count, every position and
their order; the relinked CLI must print what the stock CLI prints with -t 1."""
import ctypes as C
import os
import random
import subprocess
import sys

import numpy as np
import pytest

from krep_b200 import lib
from krep_b200.abi import Params
import oracle_util as ou
import regex_util as ru

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu
UNBOUNDED = (1 << 64) - 1
KNOB = "KREP_B200_NO_DEVICE_MATCHES"


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


def _host(P, text):
    L = lib.load()
    buf = C.create_string_buffer(text, len(text) + 1)
    res = L.krep_b200_match_result_init(16)
    try:
        cnt = L.krep_b200_regex_matches_host(P.ref(), buf, len(text), UNBOUNDED, res)
        r = res.contents
        return int(cnt), [(r.positions[i].start_offset, r.positions[i].end_offset) for i in range(r.count)]
    finally:
        L.krep_b200_match_result_free(res)


def _check(pat, text, monkeypatch, want=None, **kw):
    P = _params(pat, **kw)
    L = lib.load()
    assert L.krep_b200_regex_match_mode(P.ref()) == 1, (pat, kw)
    dev = lib.search("regex", P, text)
    with monkeypatch.context() as m:
        m.setenv(KNOB, "1")
        assert L.krep_b200_regex_match_mode(P.ref()) == 0
        knob = lib.search("regex", P, text)
    host = _host(P, text)
    want = _want(P, text) if want is None else want
    assert dev[0] == knob[0] == host[0] == want[0], (pat, kw, len(text), dev[0], knob[0], host[0], want[0])
    assert dev == knob == host == want, (pat, kw, len(text))
    return dev


@pytest.fixture(scope="module", autouse=True)
def _init():
    L = lib.load()
    assert L.krep_b200_init(0) == 0, L.krep_b200_last_error_string()


OPTS = [dict(), dict(only_matching=True), dict(count=True, only_matching=True), dict(case_sensitive=False),
        dict(max_count=1), dict(max_count=7), dict(max_count=100000)]


def test_random_texts(monkeypatch):
    rng = random.Random(21)
    pats = ["a+b", "^a", "b$", "(ab|ba)c?", "[0-9]x", "x*", "a*", "^", "$", "^$", ".", "[^0-9 ]{2}", "A_", "^a.c$",
            "(a*)*", "(|a)+", "a{,2}", "x{0}", "a|^b", "a|ab|abc", "(a|ab)(c|bcd)"]
    for pat in pats:
        for kw in OPTS:
            for n in (1, 37, 1000, 20000):
                _check(pat, ru.random_text(rng, n), monkeypatch, **kw)
    for kw in OPTS:
        _check(["ab", "x[0-9]", "^c"], ru.random_text(rng, 5000), monkeypatch, **kw)  # several -e patterns


def test_edge_texts(monkeypatch):
    wide = bytes(range(0x80, 0x100)) + b"\x00\t\r aab\n"
    for text in (b"\n", b"\n\n\n", b"abc", b"abc\n", b"a\n\nb\n\n", b"ab\nab", b"aab", b"aab\n", b"ax\nbx", b"ax\nbx\n",
                 wide * 3, wide * 3 + b"\n"):
        for pat in ("x*", "a*", "^", "$", "^$", "b", "a|$", "x$", ".", "a|ab|abc"):
            for kw in OPTS:
                _check(pat, text, monkeypatch, **kw)


SPEC = (0x5EED0001, 0x5EED0002, 1 << 16, b"qzXv9Kpw")


@pytest.mark.parametrize("pat,kw", [
    ("the[a-z]*", {}), ("the[a-z]*", {"count": True, "only_matching": True}), ("[tT]h[a-z]*", {}),
    ("^[a-z]+ [a-z]+$", {}), ("qzXv[0-9]Kpw", {}), ("(qzxv|the ) ?e", {"case_sensitive": False}),
    ("th(e|a)", {"max_count": 7}), ("e t", {"max_count": 1}), ("(a|an|and) ", {}),
])
def test_corpus_slices(pat, kw, monkeypatch):
    text = lib.corpus_host(lib.make_spec(*SPEC), 0, 6 << 20)
    _check(pat, text, monkeypatch, **kw)


def test_lines_longer_than_the_kernel_bound(monkeypatch):
    rng = random.Random(5)
    long_line = bytes(rng.choice(b"abcdef ") for _ in range(1 << 20))
    text = b"x1\n" + long_line + b"qq9\n" + b"ab\n" + long_line[:300000] + b"\nqq7"
    for pat in ("qq[0-9]", "^x", "f a", "q$", "^ab$"):
        for kw in (dict(), dict(max_count=2), dict(count=True, only_matching=True)):
            _check(pat, text, monkeypatch, **kw)
            _check(pat, text + b"\n", monkeypatch, **kw)


def test_lines_over_the_step_budget(monkeypatch):
    # [a-c]*d on lines of a-c runs that fit the walk: quadratic enumeration, the lines go to regexec
    rng = random.Random(8)
    lines = []
    for k in range(3000):
        run = bytes(rng.choice(b"abc") for _ in range(rng.randint(1, 1500)))
        lines.append(run + (b"d" if k % 3 == 0 else b"") + b" cd")
    text = b"\n".join(lines) + b"\n"
    for kw in (dict(), dict(max_count=2500), dict(count=True, only_matching=True)):
        _check("[a-c]*d", text, monkeypatch, **kw)


def test_lines_cut_by_staging_chunks(monkeypatch):
    monkeypatch.setenv("KREP_B200_STAGE_MB", "1")
    monkeypatch.setenv("KREP_B200_CHUNK_MB", "1")
    monkeypatch.setenv("KREP_B200_RANGES", "3")
    text = lib.corpus_host(lib.make_spec(*SPEC), 0, (5 << 20) + 12345)
    cut = bytearray(text)
    for k in range(1, 6):
        cut[(k << 20) + 5] = 10  # a newline a few bytes after each MiB boundary
    for t in (text, bytes(cut)):
        for pat, kw in (("the[a-z]*", {}), ("^[a-z]+$", {}), ("e t", {"max_count": 100000}), ("qzXv", {"max_count": 7}),
                        ("[a-z]*", {"count": True, "only_matching": True})):
            _check(pat, t, monkeypatch, **kw)


def test_pinned_text_chunks(monkeypatch):
    import torch
    monkeypatch.setenv("KREP_B200_CHUNK_MB", "1")
    text = lib.corpus_host(lib.make_spec(*SPEC), 0, (3 << 20) + 99)
    pinned = torch.empty(len(text), dtype=torch.uint8).pin_memory()
    pinned.numpy()[:] = np.frombuffer(text, dtype=np.uint8)
    for pat, kw in (("the[a-z]*", {}), ("[tT]h[a-z]*", {"max_count": 5000})):
        P = _params(pat, **kw)
        assert lib.load().krep_b200_regex_match_mode(P.ref()) == 1
        got = lib.search("regex", P, None, text_ptr=pinned.data_ptr(), text_len=len(text))
        assert got == _want(P, text)


def test_lines_cut_across_devices(monkeypatch):
    if lib.load().krep_b200_device_count() < 2:
        pytest.skip("needs two or more GPUs")
    monkeypatch.setenv("KREP_B200_DEVICES", str(lib.load().krep_b200_device_count()))
    monkeypatch.setenv("KREP_B200_STAGE_MB", "1")
    monkeypatch.setenv("KREP_B200_CHUNK_MB", "1")
    text = lib.corpus_host(lib.make_spec(*SPEC), 0, (6 << 20) + 777)
    for pat, kw in (("the[a-z]*", {}), ("^[a-z]+ ", {}), ("th(e|a)", {"max_count": 100000})):
        _check(pat, text, monkeypatch, **kw)


def test_every_line_uncertain(monkeypatch):
    # each line runs further past its thread's segment than the walk may read: every line goes to regexec
    rng = random.Random(9)
    line = bytes(rng.choice(b"abc ") for _ in range(5000))
    text = (line + b"\n") * 1500 + b"zz"
    _check("a b", text, monkeypatch)
    _check("^zz$", text, monkeypatch)
    _check("c*", text, monkeypatch, max_count=20000)


def test_overflow_restage(monkeypatch):
    # x* holds an empty match at every byte: one key per byte, more than the first occurrence list holds
    text = lib.corpus_host(lib.make_spec(*SPEC), 0, 3 << 20)
    _check("x*", text, monkeypatch)
    _check(".", text, monkeypatch, count=True, only_matching=True)


def test_max_count_at_device_glibc_boundaries(monkeypatch):
    # device lines and uncertain (long) lines alternate: -m limits that end inside a device line, inside an uncertain
    # line, and right at the boundaries between them
    rng = random.Random(13)
    long_line = bytes(rng.choice(b"ab ") for _ in range(9000))
    parts = []
    for _ in range(6):
        parts += [b"ab ab ab", long_line, b"b a"]
    text = b"\n".join(parts) + b"\nab"
    P = _params("ab?")
    full = _want(P, text)
    assert full[0] > 100
    bounds = sorted({1, 2, 3, 4, 5, full[0] // 2, full[0] - 1, full[0], full[0] + 1})
    first_long = text.index(long_line)
    k = sum(1 for s, _ in full[1] if s < first_long)
    bounds += [k - 1, k, k + 1]
    for mc in bounds:
        _check("ab?", text, monkeypatch, max_count=mc)
        _check("ab?", text, monkeypatch, max_count=mc, count=True, only_matching=True)


CLI_CASES = [["-E", "the[a-z]*"], ["-o", "-E", "the[a-z]*"], ["-co", "-E", "the[a-z]*"], ["-i", "-E", "NEEDLE|fox"],
             ["-o", "-i", "-E", "needle|x"], ["-m", "3", "-E", "the"], ["-o", "-m", "5", "-E", "[a-z]+"],
             ["-E", "-e", "^the", "-e", "x$"], ["-o", "-E", "-e", "ab", "-e", "1[0-9]"], ["-co", "-E", "x*"],
             ["-co", "-E", "^$"], ["-o", "-i", "-E", "x$"]]


def test_cli_dropin_regex_match(tmp_path):
    sys.path.insert(0, os.path.join(ROOT, "krep_b200", "shim"))
    sys.path.insert(0, os.path.join(ROOT, "oracle"))
    import build_krep_gpu
    import build_oracle
    stock = build_oracle.build_ref()[1]
    gpu = build_krep_gpu.build()
    if not stock or not gpu:
        pytest.skip("stock or GPU-backed krep binary not available (built only where the reference sources are)")
    env = {k: v for k, v in os.environ.items() if k != "KREP_B200_KEEP_VISIBLE"}
    rng = random.Random(4)
    words = [b"the", b"quick", b"fox", b"NEEDLE", b"needle", b"ab", b"x", b"12", b"aX"]
    body = bytearray()
    while len(body) < 300_000:
        body += rng.choice(words) + rng.choice([b" ", b" ", b"\n", b"", b"\n\n"])
    files = {"nl.txt": bytes(body).rstrip(b"\n") + b"\n", "no_nl.txt": bytes(body).rstrip(b"\n") + b" ax",
             "nl2.txt": bytes(body).rstrip(b"\n") + b"\n\n"}
    for name, data in files.items():
        path = tmp_path / name
        path.write_bytes(data)
        for flags in CLI_CASES:
            a = subprocess.run([stock, "-t", "1", "--color=never", *flags, str(path)], capture_output=True)
            b = subprocess.run([gpu, "--color=never", *flags, str(path)], capture_output=True, env=env)
            assert (b.returncode, b.stdout) == (a.returncode, a.stdout), (name, flags, a.stdout[:300], b.stdout[:300], b.stderr[:300])
