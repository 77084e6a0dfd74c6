"""Many HBM-resident texts in one call: krep_b200_search_batch_resident and krep_b200_regex_search_batch_resident must
give every text exactly what the host batches give for host copies of the same texts (and, for -E, what the reference
loop gives), and k_batch_gather must build the host batch's packed buffer byte for byte."""
import ctypes as C
import os
import random
import subprocess
import sys
import time

import numpy as np
import pytest
import torch

from krep_b200 import lib
from krep_b200.abi import Params
import regex_kernel_model as km
import regex_util as ru

pytestmark = pytest.mark.gpu
KNOBS = ["KREP_B200_NO_FUSED_COUNT", "KREP_B200_NO_DEVICE_MATCHES", "KREP_B200_NO_LONG_LINES"]


@pytest.fixture(scope="module", autouse=True)
def _init():
    L = lib.load()
    assert L.krep_b200_init(0) == 0, L.krep_b200_last_error_string()


@pytest.fixture(autouse=True)
def _knobs_off(monkeypatch):
    for k in KNOBS:
        monkeypatch.delenv(k, raising=False)


class Corpus:
    """The texts laid end to end in one CUDA tensor at a storage offset (so d_base has any alignment), listed out of
    order, with one text repeated and one that overlaps two neighbours."""

    def __init__(self, rng, texts, shift=None):
        order = list(range(len(texts)))
        rng.shuffle(order)
        buf, pos = bytearray(), [0] * len(texts)
        for i in order:
            pos[i] = len(buf)
            buf += texts[i]
        shift = rng.randrange(16) if shift is None else shift
        store = torch.zeros(len(buf) + shift + 64, dtype=torch.uint8, device="cuda")
        if buf:
            store[shift:shift + len(buf)] = torch.frombuffer(bytearray(buf), dtype=torch.uint8).cuda()
        torch.cuda.synchronize()
        self.tensor = store[shift:]  # a view with a storage offset
        self.buf = bytes(buf)
        self.offsets = list(pos)
        self.lens = [len(t) for t in texts]
        if texts:
            j = rng.randrange(len(texts))  # the same text twice
            self.offsets.append(pos[j])
            self.lens.append(len(texts[j]))
            if len(buf) > 40:  # a text across the seam of two others
                o = rng.randrange(len(buf) - 40)
                self.offsets.append(o)
                self.lens.append(rng.randrange(1, min(9000, len(buf) - o)))
        self.texts = [self.buf[o:o + n] for o, n in zip(self.offsets, self.lens)]


def host_pack(texts, gap_kind, max_gap):
    """The host batch's packed buffer (krep_b200_batch_gather_raw on host texts runs pack_texts)."""
    L = lib.load()
    n = len(texts)
    buf = b"".join(texts)
    offs, p = [], 0
    for t in texts:
        offs.append(p)
        p += len(t)
    hb = C.create_string_buffer(buf, max(len(buf), 1))
    oarr = (C.c_uint64 * max(n, 1))(*offs)
    larr = (C.c_size_t * max(n, 1))(*[len(t) for t in texts])
    total = L.krep_b200_batch_gather_raw(hb, oarr, larr, n, gap_kind, max_gap, None, 0)
    assert total >= 0, L.krep_b200_last_error_string()
    out = C.create_string_buffer(max(total, 1))
    assert L.krep_b200_batch_gather_raw(hb, oarr, larr, n, gap_kind, max_gap, out, total) == total
    return out.raw[:total]


def device_pack(corpus, gap_kind, max_gap):
    L = lib.load()
    n = len(corpus.lens)
    oarr = (C.c_uint64 * max(n, 1))(*corpus.offsets)
    larr = (C.c_size_t * max(n, 1))(*corpus.lens)
    total = L.krep_b200_batch_gather_raw(corpus.tensor.data_ptr(), oarr, larr, n, gap_kind, max_gap, None, 0)
    assert total >= 0, L.krep_b200_last_error_string()
    out = C.create_string_buffer(max(total, 1))
    assert L.krep_b200_batch_gather_raw(corpus.tensor.data_ptr(), oarr, larr, n, gap_kind, max_gap, out, total) == total
    return out.raw[:total]


def test_gather_equals_the_host_pack():
    rng = random.Random(11)
    lens = [0, 1, 2, 15, 16, 17, 31, 33, 255, 256, 257, 4095, 4096, 4097, 65535, 65536, 70000]
    texts = [bytes(rng.randrange(1, 256) for _ in range(n)) if n < 5000 else np.random.default_rng(n).integers(
        0, 256, n, dtype=np.uint8).tobytes() for n in lens]
    for shift in range(16):
        corpus = Corpus(rng, texts, shift=shift)
        for gap_kind, max_gap in ((0, 0), (0, 7), (0, 64), (1, 0)):
            want = host_pack(corpus.texts, gap_kind, max_gap)
            got = device_pack(corpus, gap_kind, max_gap)
            assert got == want, (shift, gap_kind, max_gap, len(got), len(want))


def mixed_text(rng, n):
    words = [b"needle", b"the", b"ab", b"quick", b"fox_1", b"x", b"NeEdLe"]
    out = bytearray()
    while len(out) < n:
        r = rng.random()
        out += rng.choice(words) if r < 0.35 else b"\n" if r < 0.45 else bytes([rng.choice(b" .,-_aAzZ09")])
    return bytes(out[:n])


def literal_texts(rng):
    texts = []
    for _ in range(150):
        n = rng.choice([0, 1, 3, 5, 6, 17, 64, 300, 2000, 9000])
        t = bytearray(mixed_text(rng, n))
        if n >= 12 and rng.random() < 0.5:
            t[:6] = b"needle"
        if n >= 12 and rng.random() < 0.5:
            t[-6:] = b"needle"
        if rng.random() < 0.3:  # one line, no '\n': its line runs into both neighbours without the clip
            t = t.replace(b"\n", b" ")
        texts.append(bytes(t))
    # patterns split across the seam of two texts in the source buffer
    texts += [b"xx nee", b"dle yy", b"ab\nnee", b"dle\nab", b"thequick", b"fox_1 ne", b"edle"]
    return texts


LITERALS = [
    ("boyer_moore", [b"needle"]), ("kmp", [b"abab"]), ("kmp", [b"needle"]), ("memchr", [b"x"]), ("memchr_short", [b"ab"]),
    ("sse42", [b"needle"]), ("avx2", [b"the quick Brown fox_1"]), ("avx2", [b"needle needle needle"]),
    ("avx512", [b"needle " * 6]), ("neon", [b"quick"]), ("aho_corasick", [b"needle", b"quick", b"ab", b"fox_1 needle"]),
    ("boyer_moore", [b"\x00\x00"]),
]
LIT_OPTIONS = [dict(), dict(case_sensitive=False), dict(whole_word=True), dict(count=True), dict(only_matching=True),
               dict(count=True, only_matching=True), dict(max_count=1), dict(max_count=2), dict(max_count=3),
               dict(count=True, max_count=2), dict(count=True, case_sensitive=False, whole_word=True)]


@pytest.mark.parametrize("func,pats", LITERALS)
def test_literal_entries_equal_the_host_batch(func, pats):
    rng = random.Random(len(func) * 31 + len(pats[0]))
    corpus = Corpus(rng, literal_texts(rng))
    for opt in LIT_OPTIONS:
        P = Params(pats, **opt)
        want = lib.search_batch(func, Params(pats, **opt), corpus.texts)
        got = lib.search_batch_resident(func, P, corpus.tensor, corpus.offsets, corpus.lens)
        for i in range(len(want)):
            assert got[i] == want[i], (func, pats, opt, i, corpus.lens[i], got[i][0], want[i][0], got[i][1][:4], want[i][1][:4])
        counts = lib.search_batch_resident(func, P, corpus.tensor, torch.tensor(corpus.offsets), torch.tensor(corpus.lens),
                                           with_result=False)
        assert [c for c, _ in counts] == [c for c, _ in want], (func, pats, opt)


def regex_texts(rng):
    out = [b""]
    for n in (1, 15, 16, 17, 255, 256, 257, 4095, 4096, 4097, 9000, 70000):
        body = ru.random_text(rng, n) if n < 9000 else km.random_lines_text(rng, n + 10)[:n]
        out.append(body[:-1] + b"\n")
        out.append(body[:-1] + b"a")
    out += [b"\n", b"\n" * 300, b"\x00" * 40, b"ab\x00ab\n\x00x", b"ab " * 3000, b"ab " * 3000 + b"\n",
            b"x" * (km.REGEX_HALO + 700) + b"\nab\n", b"x" * 20000 + b"ab\n" + b"the" * 3000, b"abc\n\nab", b"",
            b"xx\n", b"x", b"the\n\n"]
    return out


PATTERNS = ["^$", "x*", "^", "$", "x$", "a|ab|abc", "the[a-z]*", "a+b"]
RX_OPTIONS = [dict(), dict(case_sensitive=False), dict(whole_word=True), dict(count=True), dict(count=True, only_matching=True),
              dict(max_count=1), dict(max_count=2), dict(max_count=3), dict(count=True, max_count=2)]
RX_KNOBS = [{}, {"KREP_B200_NO_FUSED_COUNT": "1"}, {"KREP_B200_NO_DEVICE_MATCHES": "1"}, {"KREP_B200_NO_LONG_LINES": "1"}]


def set_knobs(monkeypatch, knobs):
    for k in KNOBS:
        if k in knobs:
            monkeypatch.setenv(k, knobs[k])
        else:
            monkeypatch.delenv(k, raising=False)


@pytest.mark.parametrize("pat", PATTERNS)
def test_regex_equals_the_host_batch_and_the_reference(pat, monkeypatch):
    rng = random.Random(pat)
    corpus = Corpus(rng, regex_texts(rng))
    for opt in RX_OPTIONS:
        P = Params([pat.encode()], regex=True, **opt)
        want = [ru.ref_regex_search(P, t) for t in corpus.texts]
        for knobs in RX_KNOBS:
            set_knobs(monkeypatch, knobs)
            got = lib.regex_search_batch_resident(P, corpus.tensor, corpus.offsets, corpus.lens)
            for i in range(len(want)):
                assert got[i] == want[i], (pat, opt, knobs, i, corpus.lens[i], got[i][0], want[i][0], got[i][1][:4], want[i][1][:4])
            if knobs in ({}, RX_KNOBS[3]):
                assert got == lib.regex_search_batch(P, corpus.texts), (pat, opt, knobs)


def test_regex_i_dollar_and_a_split_set(monkeypatch):
    rng = random.Random(5)
    words = ["".join(rng.choice("abcdefghijklmnopqrstuvwxyz") for _ in range(rng.randint(8, 12))) for _ in range(120)]
    pats = [w.encode() for w in words] + [b"the[a-z]*"]
    assert lib.load().krep_b200_regex_automata(Params(pats, regex=True).ref()) >= 2
    texts = []
    for _ in range(80):
        n = rng.choice([0, 1, 50, 3000, 40000])
        lines = []
        while sum(len(x) + 1 for x in lines) < n:
            lines.append(" ".join(rng.choice(words + ["the", "thexx", "zz"]) for _ in range(rng.randint(0, 12))))
        texts.append(("\n".join(lines)[:n]).encode())
    corpus = Corpus(rng, texts)
    for P in (Params([b"x$"], regex=True, case_sensitive=False), Params([b"x$"], regex=True, case_sensitive=False, count=True)):
        assert lib.regex_search_batch_resident(P, corpus.tensor, corpus.offsets, corpus.lens) == \
            [ru.ref_regex_search(P, t) for t in corpus.texts]
    for kw in (dict(), dict(count=True), dict(count=True, only_matching=True), dict(max_count=2), dict(case_sensitive=False)):
        P = Params(pats, regex=True, **kw)
        got = lib.regex_search_batch_resident(P, corpus.tensor, corpus.offsets, corpus.lens)
        assert got == lib.regex_search_batch(P, corpus.texts), kw
        for i, t in enumerate(corpus.texts):
            want = ru.ref_regex_search(P, t)
            assert got[i] == (want[0], want[1] if P.struct.track_positions else []), (kw, i)


def test_twenty_thousand_texts_in_one_call():
    rng = random.Random(20000)
    texts = [mixed_text(rng, rng.choice([0, 1, 40, 200, 1000])) for _ in range(20000)]
    corpus = Corpus(rng, texts)
    for P in (Params([b"the[a-z]*"], regex=True), Params([b"the[a-z]*"], regex=True, count=True)):
        assert lib.regex_search_batch_resident(P, corpus.tensor, corpus.offsets, corpus.lens) == \
            lib.regex_search_batch(P, corpus.texts)
    for opt in (dict(), dict(count=True)):
        assert lib.search_batch_resident("boyer_moore", Params([b"needle"], **opt), corpus.tensor, corpus.offsets, corpus.lens) == \
            lib.search_batch("boyer_moore", Params([b"needle"], **opt), corpus.texts)


def _raw_call(L, regex, P, base, offs, lens):
    n = len(lens)
    oarr = (C.c_uint64 * max(n, 1))(*offs)
    larr = (C.c_size_t * max(n, 1))(*lens)
    counts = (C.c_uint64 * max(n, 1))(*([7] * max(n, 1)))
    if regex:
        rc = L.krep_b200_regex_search_batch_resident(P.ref(), base, oarr, larr, n, counts, None)
    else:
        entry = C.cast(L.krep_b200_boyer_moore_search, C.c_void_p)
        rc = L.krep_b200_search_batch_resident(entry, P.ref(), base, oarr, larr, n, counts, None)
    return rc, list(counts[:n])


def test_edge_cases():
    L = lib.load()
    rng = random.Random(3)
    corpus = Corpus(rng, [b"needle\n", b"", b"x needle", b""])
    base = corpus.tensor.data_ptr()
    assert _raw_call(L, False, Params([b"needle"]), base, [], []) == (0, [])
    assert _raw_call(L, True, Params([b"needle"], regex=True), base, [], []) == (0, [])
    assert lib.search_batch_resident("boyer_moore", Params([b"needle"]), corpus.tensor, [0, 3], [0, 0]) == [(0, [])] * 2
    assert lib.regex_search_batch_resident(Params([b"^$"], regex=True), corpus.tensor, [0, 3], [0, 0]) == \
        [ru.ref_regex_search(Params([b"^$"], regex=True), b"")] * 2
    P0 = Params([b"needle"], max_count=0)
    assert lib.search_batch_resident("boyer_moore", P0, corpus.tensor, corpus.offsets, corpus.lens) == \
        lib.search_batch("boyer_moore", Params([b"needle"], max_count=0), corpus.texts)
    R0 = Params([b"needle"], regex=True, max_count=0)
    assert lib.regex_search_batch_resident(R0, corpus.tensor, corpus.offsets, corpus.lens) == \
        lib.regex_search_batch(R0, corpus.texts)
    RN = Params([b"needle"], regex=True)
    RN.struct.compiled_regex = None
    assert lib.regex_search_batch_resident(RN, corpus.tensor, corpus.offsets, corpus.lens) == [(0, [])] * len(corpus.lens)
    # a refused regex: -3, every count 0
    refused = Params([b"ab\\sab"], regex=True)
    assert _raw_call(L, True, refused, base, corpus.offsets, corpus.lens) == (-3, [0] * len(corpus.lens))
    # host memory as d_base: -3
    host = C.create_string_buffer(corpus.buf, len(corpus.buf) + 1)
    for regex in (False, True):
        P = Params([b"needle"], regex=regex)
        rc, counts = _raw_call(L, regex, P, C.cast(host, C.c_void_p), corpus.offsets, corpus.lens)
        assert rc == -3 and counts == [0] * len(corpus.lens)
        # a text past the end of the allocation: -3
        rc, _ = _raw_call(L, regex, P, base, [0, 1 << 40], [4, 4])
        assert rc == -3
    # the regex search entry is refused by the literal batch
    oarr, larr, cnt = (C.c_uint64 * 1)(0), (C.c_size_t * 1)(4), (C.c_uint64 * 1)()
    assert L.krep_b200_search_batch_resident(C.cast(L.krep_b200_regex_search, C.c_void_p), Params([b"needle"]).ref(), base,
                                             oarr, larr, 1, cnt, None) == -3
    # the same call twice (the kept buffers are reused), then a larger batch, then the first again
    P = Params([b"needle"])
    first = lib.search_batch_resident("boyer_moore", P, corpus.tensor, corpus.offsets, corpus.lens)
    assert first == lib.search_batch_resident("boyer_moore", P, corpus.tensor, corpus.offsets, corpus.lens)
    big = Corpus(rng, [mixed_text(rng, 5000) for _ in range(300)])
    assert lib.search_batch_resident("boyer_moore", P, big.tensor, big.offsets, big.lens) == \
        lib.search_batch("boyer_moore", Params([b"needle"]), big.texts)
    assert first == lib.search_batch_resident("boyer_moore", P, corpus.tensor, corpus.offsets, corpus.lens)
    g, s, r = lib.batch_resident_stats()
    assert g >= 0 and s >= 0 and r >= 0


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_texts_on_a_second_device():
    rng = random.Random(1)
    texts = [mixed_text(rng, rng.choice([10, 500, 3000])) for _ in range(50)]
    corpus = Corpus(rng, texts)
    t1 = corpus.tensor.to("cuda:1")
    torch.cuda.synchronize(1)
    for opt in (dict(), dict(count=True)):
        assert lib.search_batch_resident("boyer_moore", Params([b"needle"], **opt), t1, corpus.offsets, corpus.lens) == \
            lib.search_batch("boyer_moore", Params([b"needle"], **opt), corpus.texts)
    P = Params([b"the[a-z]*"], regex=True)
    assert lib.regex_search_batch_resident(P, t1, corpus.offsets, corpus.lens) == lib.regex_search_batch(P, corpus.texts)


def one_line_texts(rng, words, k, lo, hi):
    """k texts cut from words and filler with no '\\n' at all: each text is one line, as documents often are."""
    pool = b" ".join(rng.choice(words) if rng.random() < 0.3 else b"zq" for _ in range(1 << 20))
    out = []
    for _ in range(k):
        n = rng.randint(lo, hi)
        o = rng.randrange(len(pool) - n)
        out.append(pool[o:o + n])
    return out


def test_count_on_one_line_texts_stays_inside_each_text():
    """-c over texts without any '\\n': a text's line bounds reach its own edges.  The device's search for them must
    stop there rather than walk the neighbouring texts, so dense keys over 100 000 texts cost about what the host
    batch's own line search costs, not keys x buffer; answers equal the host batch's."""
    rng = random.Random(404)
    words = [bytes(rng.choice(b"abcdefghijklmnopqrstuvwxyz") for _ in range(rng.randint(6, 12))) for _ in range(200)]
    texts = one_line_texts(rng, words, 100000, 1024, 3072)
    corpus = Corpus(rng, texts)
    cases = [("aho_corasick", words, dict(count=True)), ("aho_corasick", words, dict(count=True, max_count=1)),
             ("boyer_moore", [words[0]], dict(count=True)), ("boyer_moore", [b"zq"], dict(count=True))]
    for func, pats, opt in cases:
        want = lib.search_batch(func, Params(pats, **opt), corpus.texts, with_result=False)
        t0 = time.perf_counter()
        got = lib.search_batch_resident(func, Params(pats, **opt), corpus.tensor, corpus.offsets, corpus.lens, with_result=False)
        dt = time.perf_counter() - t0
        assert got == want, (func, len(pats), opt)
        assert dt < 20, (func, len(pats), opt, dt)  # about 0.1 s; a line search across texts would take minutes
    small = Corpus(rng, one_line_texts(rng, words, 300, 0, 300) + [b"", words[1], b" " + words[2] + b" "])
    for func, pats, opt in cases + [("aho_corasick", words, dict(count=True, whole_word=True))]:
        assert lib.search_batch_resident(func, Params(pats, **opt), small.tensor, small.offsets, small.lens) == \
            lib.search_batch(func, Params(pats, **opt), small.texts), (func, len(pats), opt)


EXPANDABLE_CHILD = r"""
import random, sys
import torch
sys.path.insert(0, sys.argv[1])
from krep_b200 import lib
from krep_b200.abi import Params
import test_gpu_batch_resident as t
assert lib.load().krep_b200_init(0) == 0
rng = random.Random(8)
# grown in several steps, so that the tensor's memory is mapped in more than one chunk
keep = [torch.empty(n << 20, dtype=torch.uint8, device="cuda") for n in (3, 50, 7)]
del keep
big = torch.randint(32, 127, (300 << 20,), dtype=torch.uint8, device="cuda")
big[::97] = 10
torch.cuda.synchronize()
offs = [0, 1, (100 << 20) + 3, (150 << 20) - 5, (300 << 20) - 4096, 12345, (200 << 20) + 7]
lens = [4096, 70000, 9000, 1 << 20, 4096, (299 << 20), 100]
host = big.cpu().numpy().tobytes()
texts = [host[o:o + n] for o, n in zip(offs, lens)]
for opt in (dict(), dict(count=True)):
    P = Params([b"ab"], **opt)
    assert lib.search_batch_resident("boyer_moore", P, big, offs, lens) == lib.search_batch("boyer_moore", Params([b"ab"], **opt), texts)
P = Params([b"a[bc]d"], regex=True, count=True)
assert lib.regex_search_batch_resident(P, big, offs, lens) == lib.regex_search_batch(P, texts)
print("case ok")
"""


def test_texts_in_expandable_segments():
    """A tensor from torch's expandable segments is mapped in chunks; texts that span them are one allocation to the
    caller and must be searched, not refused."""
    here = os.path.dirname(os.path.abspath(__file__))
    env = dict(os.environ, PYTORCH_CUDA_ALLOC_CONF="expandable_segments:True",
               PYTHONPATH=os.pathsep.join([here, os.path.dirname(here), os.environ.get("PYTHONPATH", "")]))
    for k in KNOBS:
        env.pop(k, None)
    r = subprocess.run([sys.executable, "-c", EXPANDABLE_CHILD, here], cwd=here, env=env, capture_output=True, text=True,
                       timeout=900)
    assert r.returncode == 0 and "case ok" in r.stdout, r.stdout[-2000:] + r.stderr[-4000:]
