"""-m gpu: parity of the CUDA path, called through the C ABI, against the oracle.
Bit-exact bar: count, every (start,end) and their order."""
import ctypes as C
import json
import os
import random

import pytest

import oracle_util as ou
from krep_b200 import lib
from krep_b200.abi import (ALGO_AC, ALGO_BMH, ALGO_SSE42, CORPUS_EMBED_HALF, CORPUS_RANDOM_CASE, Params, SIZE_MAX)
from test_oracle import _vectors, params_from, random_case, text_from

pytestmark = pytest.mark.gpu


def checker():
    return ou.reference() or ou.port()


@pytest.mark.parametrize("v", _vectors(), ids=lambda v: f'{v["func"]}:{v["pat"][0][:8] or "(empty)"}:{v["src"].split()[0]}')
def test_reference_test_vectors_through_c_abi(v):
    cnt, pos = lib.search(v["func"], params_from(v), text_from(v), with_result=v.get("res", False))
    assert cnt == v["expect"], v["src"]
    if "npos" in v:
        assert len(pos) == v["npos"], v["src"]


def test_committed_reference_fixtures_through_c_abi():
    with open(os.path.join(os.path.dirname(__file__), "golden", "ref_fixtures.json")) as f:
        fx = json.load(f)["cases"]
    for c in fx:
        p = Params([bytes.fromhex(x) for x in c["pat"]], case_sensitive=c["cs"], count=c["count"],
                   only_matching=c["o"], whole_word=c["w"], max_count=c["m"] if c["m"] >= 0 else SIZE_MAX)
        cnt, pos = lib.search(c["func"], p, bytes.fromhex(c["text"]), with_result=c["res"])
        assert cnt == c["count_out"] and [list(x) for x in pos] == c["pos_out"], c


@pytest.mark.parametrize("func", list(ou.FUNCS) + ["avx512", "neon"])
def test_random_differential_vs_oracle(func):
    rng = random.Random(4242 + len(func))
    chk = {"avx512": ou.reference512() or ou.port(), "neon": ou.reference_neon() or ou.port()}.get(func) or checker()
    for _ in range(700):
        pats, text, opts, with_res = random_case(rng, func)
        got = lib.search(func, Params(pats, **opts), text, with_result=with_res)
        want = chk.run(func, Params(pats, **opts), text, with_result=with_res)
        assert got == want, (func, pats, text, opts, with_res, got, want)


def _mixed_text(rng, n):
    words = [b"the", b"quick", b"Brown", b"fox_1", b"needle", b"NEEDLE", b"ab", b"abab", b"aaa", b"x"]
    out = bytearray()
    while len(out) < n:
        out += rng.choice(words)
        out += rng.choice([b" ", b" ", b"\n", b"", b",", b"_"])
    return bytes(out[:n])


@pytest.mark.parametrize("func,pat", [
    ("sse42", b"needle"), ("sse42", b"the quick"), ("sse42", b"abab"), ("boyer_moore", b"aaa"),
    ("boyer_moore", b"needle Brown"), ("kmp", b"abab"), ("memchr", b"x"), ("memchr_short", b"ab"),
    ("boyer_moore", b"the quick Brown fox_1 needle NEEDLE"), ("sse42", b"fox_1 needle NEE"),
    ("avx2", b"needle Brown fox_1 ne"), ("avx2", b"ab abab aaa x ab abab"), ("avx2", b"the quick Brown fox_1 needle NEE"),
])
@pytest.mark.parametrize("opts", [
    dict(), dict(case_sensitive=False), dict(whole_word=True), dict(count=True), dict(only_matching=True),
    dict(count=True, only_matching=True), dict(max_count=5), dict(whole_word=True, only_matching=True, case_sensitive=False),
    dict(count=True, whole_word=True, max_count=3),
])
def test_medium_text_all_modes(func, pat, opts):
    rng = random.Random(9)
    text = _mixed_text(rng, 300_000)
    got = lib.search(func, Params(pat, **opts), text)
    want = checker().run(func, Params(pat, **opts), text)
    assert got == want


def test_chunked_staging_path_matches_single_copy(monkeypatch):
    """Host text larger than the staging chunk: occurrences straddling chunk edges, -w context across edges."""
    rng = random.Random(5)
    text = bytearray(_mixed_text(rng, 5 * (1 << 20) + 12345))
    pat = b"straddle_me"
    mb = 1 << 20
    for c in range(1, 5):
        for delta in (-len(pat), -5, -1, 0, 1):
            s = c * mb + delta
            text[s:s + len(pat)] = pat
    text[2 * mb - 6 - 1] = ord("Z")          # word char right before an occurrence that ends at the edge region
    text = bytes(text)
    monkeypatch.setenv("KREP_B200_STAGE_MB", "1")
    monkeypatch.setenv("KREP_B200_CHUNK_MB", "1")
    for func, opts in [("sse42", {}), ("boyer_moore", dict(whole_word=True)), ("boyer_moore", dict(count=True)),
                       ("kmp", dict(case_sensitive=False)), ("sse42", dict(count=True, only_matching=True))]:
        got = lib.search(func, Params(pat, **opts), text)
        want = checker().run(func, Params(pat, **opts), text)
        assert got == want, (func, opts)
    pats = [b"straddle_me", b"addle", b"fox_1 ne", b"quick"]
    got = lib.search("aho_corasick", Params(pats), text)
    want = checker().run("aho_corasick", Params(pats), text)
    assert got == want


def test_aho_corasick_many_patterns():
    rng = random.Random(11)
    text = _mixed_text(rng, 400_000)
    alpha = b"abcdefghijklmnopqrstuvwxyz"
    pats = [bytes(rng.choice(alpha) for _ in range(rng.randint(6, 12))) for _ in range(990)]
    pats += [b"needle", b"quick Brow", b"fox_1 needle", b"NEEDLE", b"the quick", b"abababab", b"aaaaaa", b"needle",
             b"ox_1 nee", b"Brown fox_1"]
    for opts in [dict(), dict(case_sensitive=False), dict(whole_word=True), dict(count=True), dict(max_count=17)]:
        got = lib.search("aho_corasick", Params(pats, **opts), text)
        want = checker().run("aho_corasick", Params(pats, **opts), text)
        assert got == want, opts
        assert got[0] > 0


def test_aho_corasick_short_and_mixed_lengths():
    rng = random.Random(12)
    text = _mixed_text(rng, 100_000)
    for pats in ([b"a", b"ab", b"the quick"], [b"x", b"ee"], [b"ab", b"abab", b"ababab"], [b"needle", b"ne", b"e"],
                 [b"quick", b"uick ", b"fox_1"], [b"", b"the"]):
        for opts in [dict(), dict(case_sensitive=False), dict(whole_word=True)]:
            got = lib.search("aho_corasick", Params(pats, **opts), text)
            want = checker().run("aho_corasick", Params(pats, **opts), text)
            assert got == want, (pats, opts)


def test_aho_corasick_shortest_pattern_6_bytes_or_more_aligned_word_filter():
    """Pattern sets whose shortest pattern has >= 6 bytes take the aligned-word stride-4 filter (k_ac_tri4): keyed by
    three bytes + a selector byte when the shortest pattern has 6 bytes, by a hash of the whole word from 7 on.  Every
    start alignment, the (len 6, d 3) entries that do not know the selector byte, tails shorter than a group, heavy
    overlap, -i and -w."""
    rng = random.Random(66)
    chk = checker()
    for trial in range(90):
        alpha = rng.choice([b"ab", b"abc", b"abcdefgh \n", b"aAbB_ 1\n"])
        lmin = rng.choice([6, 6, 7, 8, 11])
        n = rng.choice([6, 7, 15, 16, 17, 31, 32, 33, 47, 64, 100, 1000, 5000, 70_000])
        text = bytes(rng.choice(alpha) for _ in range(n))
        pats = []
        for _ in range(rng.randint(1, 12)):
            m = rng.randint(lmin, lmin + 4)
            if n >= m and rng.random() < 0.8:
                s = rng.randrange(0, n - m + 1)
                pats.append(text[s:s + m])
            else:
                pats.append(bytes(rng.choice(alpha) for _ in range(m)))
        if rng.random() < 0.3:
            pats.append(pats[0])
        pats[rng.randrange(len(pats))] = (pats[0] * 2)[:lmin]  # at least one pattern of the minimum length
        opts = dict(case_sensitive=rng.random() < 0.6, whole_word=rng.random() < 0.3,
                    count=rng.random() < 0.2, max_count=rng.choice([SIZE_MAX, SIZE_MAX, 1, 5]))
        got = lib.search("aho_corasick", Params(pats, **opts), text)
        want = chk.run("aho_corasick", Params(pats, **opts), text)
        assert got == want, (pats, text[:200], opts, got[0], want[0])
    # all four alignments of a minimum-length pattern and of a longer one around group and buffer edges
    for base in (b"x" * 64, b"q" * 61):
        for pat, other in ((b"needle", b"zzzzzz"), (b"needle_7", b"zzzzzz"), (b"needle_7", b"zzzzzzzz"), (b"needle_7_9", b"yyyyyyyy")):
            for off in range(0, len(base) - len(pat) + 1):
                text = base[:off] + pat + base[off + len(pat):]
                got = lib.search("aho_corasick", Params([pat, other]), text)
                assert got == (1, [(off, off + len(pat))]), (pat, off, got)


@pytest.mark.parametrize("func,pats,opts", [
    ("sse42", [b"needle"], dict()),
    ("boyer_moore", [b"ab"], dict(whole_word=True)),
    ("boyer_moore", [b"the"], dict(count=True)),
    ("boyer_moore", [b"NeEdLe"], dict(case_sensitive=False, max_count=2)),
    ("kmp", [b"abab"], dict()),
    ("memchr", [b"x"], dict()),
    ("memchr_short", [b"ab"], dict(only_matching=True)),
    ("avx2", [b"the quick Brown fox_1"], dict()),
    ("neon", [b"quick"], dict(count=True)),
    ("aho_corasick", [b"needle", b"quick", b"ab", b"fox_1 needle"], dict()),
    ("aho_corasick", [b"needle", b"haystack"], dict(whole_word=True, max_count=3)),
    ("boyer_moore", [b"\x00\x00"], dict()),                  # matches the zero gaps between packed texts: must not leak
])
def test_batch_of_small_texts_equals_one_call_each(func, pats, opts):
    """krep_b200_search_batch packs many texts into one launch; every text must get exactly what a call of its own
    gives — including empty texts, texts shorter than the pattern, matches at the very start / end of a text, -w at
    the text boundaries, per-text -m and -c."""
    rng = random.Random(len(func) * 7 + len(pats))
    texts = []
    for i in range(160):
        n = rng.choice([0, 1, 3, 5, 6, 17, 64, 300, 2000, 9000])
        t = bytearray(_mixed_text(rng, n)) if n else bytearray()
        if n >= 12 and rng.random() < 0.5:
            t[:6] = b"needle"
        if n >= 12 and rng.random() < 0.5:
            t[-6:] = b"needle"
        if n >= 4 and rng.random() < 0.2:
            t[n // 2:n // 2 + 2] = b"\x00\x00"
        texts.append(bytes(t))
    chk = {"neon": ou.reference_neon() or ou.port()}.get(func) or checker()
    got = lib.search_batch(func, Params(pats, **opts), texts)
    for i, t in enumerate(texts):
        want = chk.run(func, Params(pats, **opts), t)
        assert got[i] == want, (func, pats, opts, i, len(t), got[i][0], want[0])


def test_long_needles_65_to_1024_bytes():
    """Needles beyond every SIMD kernel's range (krep.c:77 MAX_PATTERN_LENGTH 1024): boyer_moore_search semantics."""
    rng = random.Random(77)
    base = _mixed_text(rng, 600_000)
    for m in (65, 100, 255, 256, 257, 1000, 1024):
        s0 = rng.randrange(0, len(base) - m)
        pat = base[s0:s0 + m]
        text = bytearray(base)
        for at in (0, 12345, 300_001, len(base) - m):
            text[at:at + m] = pat
        text = bytes(text)
        for opts in (dict(), dict(case_sensitive=False), dict(count=True), dict(whole_word=True)):
            got = lib.search("boyer_moore", Params(pat, **opts), text)
            want = checker().run("boyer_moore", Params(pat, **opts), text)
            assert got == want and (opts.get("whole_word") or got[0] >= 4), (m, opts, got[0], want[0])


def test_ac_trie_handles_own_their_plan():
    """krep_b200_ac_trie_build hands out an owned handle: building many tries must not invalidate earlier ones
    (round-1 finding: handles pointed into a 16-entry LRU cache)."""
    L = lib.load()
    text = _mixed_text(random.Random(3), 50_000)
    handles = []
    for i in range(40):
        p = Params([b"needle", b"quick", b"pat%04d" % i] + ([b""] if i == 0 else []))
        h = L.krep_b200_ac_trie_build(p.ref())
        assert h
        handles.append((h, p))
    assert L.krep_b200_ac_trie_root_has_outputs(handles[0][0]) is True
    assert L.krep_b200_ac_trie_root_has_outputs(handles[1][0]) is False
    h, p = handles[3]
    p.struct.ac_trie = h
    res = L.krep_b200_match_result_init(16)
    cnt = L.krep_b200_aho_corasick_search(p.ref(), C.cast(C.c_char_p(text), C.c_void_p), len(text), res)
    lib.check(L)
    L.krep_b200_match_result_free(res)
    p.struct.ac_trie = None
    assert cnt == checker().run("aho_corasick", Params([b"needle", b"quick", b"pat0003"]), text)[0] > 0
    for h, _ in handles:
        L.krep_b200_ac_trie_free(h)
