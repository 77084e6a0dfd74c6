"""Pins the parity oracle (oracle/krep_oracle.c) — CPU only.

1. against the known-answer vectors of the reference's own tests (tests/golden/reference_vectors.json);
2. against committed fixtures produced by the compiled, unmodified reference
   (tests/golden/ref_fixtures.json, written by tests/golden/make_fixtures.py in the build container);
3. differentially on seeded random inputs over every option combination, against digests of what the compiled,
   unmodified reference answered on the same inputs (tests/golden/ref_differential.npz, also written by
   tests/golden/make_fixtures.py).
"""
import hashlib
import json
import os
import random

import numpy as np
import pytest

import oracle_util as ou
from krep_b200.abi import Params, SIZE_MAX

GOLD = os.path.join(os.path.dirname(__file__), "golden")


def params_from(v):
    count = v.get("count", False)
    o = v.get("o", False)
    p = Params([x.encode("latin1") for x in v["pat"]], case_sensitive=v.get("cs", True), count=count,
               only_matching=o, whole_word=v.get("w", False), max_count=v.get("m", SIZE_MAX))
    if v.get("otrack"):  # create_literal_params(..., only_match=true) without the -o global
        p.struct.track_positions = True
        p.struct.count_matches_mode = bool(count)
        p.struct.count_lines_mode = False
    if "track" in v:
        p.struct.track_positions = v["track"]
    return p


def text_from(v):
    t = bytes.fromhex(v["text_hex"]) if "text_hex" in v else v["text"].encode("latin1")
    return t[: v["len"]] if "len" in v else t


def _vectors():
    with open(os.path.join(GOLD, "reference_vectors.json")) as f:
        return json.load(f)["vectors"]


@pytest.mark.parametrize("v", _vectors(), ids=lambda v: f'{v["func"]}:{v["pat"][0][:8] or "(empty)"}:{v["src"].split()[0]}')
def test_port_matches_reference_test_vectors(v):
    cnt, pos = ou.port().run(v["func"], params_from(v), text_from(v), with_result=v.get("res", False))
    assert cnt == v["expect"], v["src"]
    if "npos" in v:
        assert len(pos) == v["npos"], v["src"]


def test_reference_build_agrees_with_its_own_vectors():
    ref = ou.reference()
    if ref is None:
        pytest.skip("compiled reference not available")
    for v in _vectors():
        chk = ou.reference_neon() if v["func"] == "neon" else ref   # neon_search only exists in the NEON build
        if chk is None:
            continue
        cnt, pos = chk.run(v["func"], params_from(v), text_from(v), with_result=v.get("res", False))
        assert cnt == v["expect"], v["src"]


def test_port_10mb_two_planted_needles():
    # test/test_krep.c:609-655: a..z cycling text, "performancetest" planted at size/4 and 3*size/4 -> 2
    size = 10 * 1024 * 1024
    text = bytearray((b"abcdefghijklmnopqrstuvwxyz" * (size // 26 + 1))[:size])
    pat = b"performancetest"
    for p in (size // 4, 3 * size // 4):
        text[p:p + len(pat)] = pat
    text = bytes(text)
    for f in ("sse42", "boyer_moore", "kmp"):
        cnt, pos = ou.port().run(f, Params(pat), text)
        assert cnt == 2 and [s for s, _ in pos] == [size // 4, 3 * size // 4]


def test_port_matches_committed_reference_fixtures():
    path = os.path.join(GOLD, "ref_fixtures.json")
    with open(path) as f:
        fx = json.load(f)
    assert fx["cases"], "empty fixture file"
    for c in fx["cases"]:
        p = Params([bytes.fromhex(x) for x in c["pat"]], case_sensitive=c["cs"], count=c["count"],
                   only_matching=c["o"], whole_word=c["w"], max_count=c["m"] if c["m"] >= 0 else SIZE_MAX)
        cnt, pos = ou.port().run(c["func"], p, bytes.fromhex(c["text"]), with_result=c["res"])
        assert cnt == c["count_out"], c
        assert [list(x) for x in pos] == c["pos_out"], c


# ---------------------------------------------------------------------------------------------
# differential test against the compiled reference's stored answers
# ---------------------------------------------------------------------------------------------
ALPHABETS = [b"ab", b"abc \n", b"aAbB_ 1\n", b"abcdefghij klmnop\nQRS"]


def random_case(rng, func, alphabets=ALPHABETS):
    alpha = rng.choice(alphabets)
    n = rng.choice([0, 1, 2, 3, 5, 8, 15, 16, 17, 31, 33, 64, 100, 257, 1000])
    text = bytes(rng.choice(alpha) for _ in range(n))
    if func == "aho_corasick":
        k = rng.randint(1, 6)
        pats = []
        for _ in range(k):
            m = rng.randint(1, 5)
            if text and rng.random() < 0.6 and len(text) >= m:
                s = rng.randrange(0, len(text) - m + 1)
                pats.append(text[s:s + m])
            else:
                pats.append(bytes(rng.choice(alpha) for _ in range(m)))
        if rng.random() < 0.2:
            pats.append(pats[0])  # duplicate pattern -> duplicate emissions (aho_corasick.c:361)
    else:
        lo, hi = {"memchr": (1, 1), "memchr_short": (2, 3), "sse42": (1, 18), "avx2": (14, 36),
                  "avx512": (28, 70), "neon": (1, 24)}.get(func, (1, 20))
        m = rng.randint(lo, hi)
        if (func in ("avx2", "avx512", "neon") and rng.random() < 0.5) or rng.random() < 0.25:
            # periodic needle + periodic text: many overlapping occurrences, window / tail edges everywhere
            unit = bytes(rng.choice(alpha) for _ in range(rng.randint(1, 3)))
            m = min(m, rng.choice([m, m, 2, 3, 4, 6]))
            n = rng.choice([31, 32, 33, 47, 63, 64, 65, 90, 96, 127, 128, 129, 200, 257])
            text = bytearray((unit * (n // len(unit) + 1))[:n])
            for _ in range(rng.randint(0, 4)):
                text[rng.randrange(n)] = rng.choice(b" \n_xZ")
            text = bytes(text)
        if text and rng.random() < 0.7 and len(text) >= m:
            s = rng.randrange(0, len(text) - m + 1)
            pat = text[s:s + m]
        else:
            pat = bytes(rng.choice(alpha) for _ in range(m))
        if rng.random() < 0.3:
            pat = pat.swapcase()
        pats = [pat]
    opts = dict(
        case_sensitive=rng.random() < (0.9 if func in ("avx2", "avx512", "neon") else 0.5),
        count=rng.random() < 0.35,
        only_matching=rng.random() < 0.4,
        whole_word=rng.random() < 0.35,
        max_count=rng.choice([SIZE_MAX, SIZE_MAX, SIZE_MAX, 0, 1, 2, 3, 7]),
    )
    return pats, text, opts, rng.random() < 0.85


# func -> (seed, number of random cases); avx512 / neon answers come from the reference's AVX-512 and NEON builds
DIFFERENTIAL_CASES = {"boyer_moore": (1, 3000), "kmp": (2, 3000), "memchr": (3, 3000), "memchr_short": (4, 3000),
                      "sse42": (5, 3000), "aho_corasick": (6, 3000), "avx2": (7, 3000), "avx512": (8, 3000),
                      "neon": (9, 4000)}


def answer_digest(answer):
    """4-byte digest of a checker's (count, [(start, end), ...]) answer."""
    return int.from_bytes(hashlib.blake2b(repr(answer).encode(), digest_size=4).digest(), "little")


def differential_cases(func):
    seed, n = DIFFERENTIAL_CASES[func]
    rng = random.Random(seed)
    return [random_case(rng, func) for _ in range(n)]


def _port_vs_stored_reference_answers(func):
    want = np.load(os.path.join(GOLD, "ref_differential.npz"))[func]
    cases = differential_cases(func)
    assert len(want) == len(cases)
    for it, (pats, text, opts, with_res) in enumerate(cases):
        a = ou.port().run(func, Params(pats, **opts), text, with_result=with_res)
        assert answer_digest(a) == want[it], (func, it, pats, text, opts, with_res, a)


@pytest.mark.parametrize("func", list(ou.FUNCS))
def test_port_vs_compiled_reference_differential(func):
    _port_vs_stored_reference_answers(func)


def test_port_vs_avx512_build_of_the_reference():
    """simd_avx512_search only exists in the reference's AVX-512 build; pin oracle_avx512_search against it."""
    _port_vs_stored_reference_answers("avx512")


def test_port_vs_neon_build_of_the_reference():
    """neon_search only exists in the reference's ARM build; its source was compiled against a scalar arm_neon.h
    (five intrinsics) to produce the stored answers that pin oracle_neon_search."""
    _port_vs_stored_reference_answers("neon")
