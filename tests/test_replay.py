"""CPU: the host-side policy replay (csrc/semantics.cpp, exported as krep_b200_replay) reproduces every
reference kernel's count/offsets/order when fed the raw occurrence list — checked against the oracle
port (and the compiled reference when present) over all option combinations.  The occurrence list is
built here in Python exactly as the device emits it (sorted keys with tag bits)."""
import ctypes as C
import random

import pytest

import oracle_util as ou
from krep_b200 import lib
from krep_b200.abi import (ALGO_AC, ALGO_AVX2, ALGO_AVX512, ALGO_BMH, ALGO_KMP, ALGO_MEMCHR, ALGO_MEMCHR_SHORT, ALGO_NEON,
                           ALGO_SSE42, MatchResult, Params, SIZE_MAX)
from scan_model import device_like_keys
from test_oracle import random_case

ALGO = {"boyer_moore": ALGO_BMH, "kmp": ALGO_KMP, "memchr": ALGO_MEMCHR, "memchr_short": ALGO_MEMCHR_SHORT,
        "sse42": ALGO_SSE42, "aho_corasick": ALGO_AC, "avx2": ALGO_AVX2, "avx512": ALGO_AVX512, "neon": ALGO_NEON}


def replay(func, params, keys, text, with_result):
    L = lib.load()
    arr = (C.c_uint64 * max(len(keys), 1))(*keys)
    res = L.krep_b200_match_result_init(16) if with_result else None
    if func == "aho_corasick":
        params.struct.ac_trie = 1  # only tested for NULL by the real entry point; replay ignores it
    try:
        cnt = L.krep_b200_replay(ALGO[func], params.ref(), bool(params.only_matching), arr, len(keys), text, len(text), res)
        pos = []
        if res:
            r = res.contents
            pos = [(r.positions[i].start_offset, r.positions[i].end_offset) for i in range(r.count)]
        return int(cnt), pos
    finally:
        params.struct.ac_trie = None
        if res:
            L.krep_b200_match_result_free(res)


def early_out(func, params, text):
    """The pre-device early-outs of run_search (host_api.cu), needed because replay starts after them."""
    s = params.struct
    m = s.pattern_len
    n = len(text)
    if func == "aho_corasick":
        return s.max_count == 0 or n == 0
    if func == "kmp":
        return s.max_count == 0 or m == 0 or n < m
    if func == "memchr":
        return s.max_count == 0 or n == 0
    if func == "memchr_short":
        return (s.max_count == 0 and (s.count_lines_mode or s.track_positions)) or m < 2 or m > 3 or n < m
    return (s.max_count == 0 and (s.count_lines_mode or s.track_positions)) or m == 0 or n < m


@pytest.mark.parametrize("func", list(ALGO))
def test_replay_matches_oracle(func):
    rng = random.Random(77 + ALGO[func])
    if func == "avx512":
        checkers = [ou.port()] + ([ou.reference512()] if ou.reference512() else [])
    elif func == "neon":
        checkers = [ou.port()] + ([ou.reference_neon()] if ou.reference_neon() else [])
    else:
        checkers = [ou.port()] + ([ou.reference()] if ou.reference() else [])
    n_checked = 0
    for _ in range(2500):
        pats, text, opts, with_res = random_case(rng, func)
        if func == "sse42" and (len(pats[0]) > 16 or not opts["case_sensitive"]):
            continue  # falls back to boyer_moore_search: covered by that parametrisation
        p = Params(pats, **opts)
        if early_out(func, p, text):
            continue
        keys = device_like_keys(func, pats, text, opts["case_sensitive"], opts["whole_word"], opts["only_matching"])
        got = replay(func, p, keys, text, with_res)
        for chk in checkers:
            want = chk.run(func, Params(pats, **opts), text, with_result=with_res)
            assert got == want, (chk.kind, func, pats, text, opts, with_res, got, want)
        n_checked += 1
    assert n_checked > 500


def _bounds_for(func, keys, text):
    """Line bounds as k_line_bounds delivers them (after marker resolution): per key the first byte of the line that
    holds the occurrence's start and the position of that line's newline (or the text length)."""
    out = []
    for k in keys:
        if func == "aho_corasick":
            e = k >> 24
            s = e - (1024 - ((k >> 14) & 1023))
        else:
            s = k >> 3
        ls = text.rfind(b"\n", 0, s) + 1
        le = text.find(b"\n", s)
        out += [ls, len(text) if le < 0 else le]
    return out


@pytest.mark.parametrize("func", list(ALGO))
def test_count_lines_replay_from_line_bounds_only(func):
    """-c without any host text: the replay reads line starts / ends from the per-occurrence bounds."""
    rng = random.Random(991 + ALGO[func])
    L = lib.load()
    chk = ou.port()
    n_checked = 0
    for _ in range(4000):
        pats, text, opts, _ = random_case(rng, func)
        opts = dict(opts, count=True, only_matching=False)
        if func == "sse42" and (len(pats[0]) > 16 or not opts["case_sensitive"]):
            continue
        p = Params(pats, **opts)
        if early_out(func, p, text):
            continue
        keys = device_like_keys(func, pats, text, opts["case_sensitive"], opts["whole_word"], False)
        bounds = _bounds_for(func, keys, text)
        arr = (C.c_uint64 * max(len(keys), 1))(*keys)
        barr = (C.c_uint64 * max(len(bounds), 1))(*bounds)
        if func == "aho_corasick":
            p.struct.ac_trie = 1
        cnt = L.krep_b200_replay_lines(ALGO[func], p.ref(), False, arr, len(keys), barr, len(text), None)
        p.struct.ac_trie = None
        want = chk.run(func, Params(pats, **opts), text, with_result=False)
        assert int(cnt) == want[0], (func, pats, text, opts, int(cnt), want[0])
        n_checked += 1
    assert n_checked > 300


def test_bulk_replay_of_a_long_list_is_the_same_on_several_threads():
    """Lists of 2^20 keys and more take the multi-threaded bulk path of the replay (csrc/semantics.cpp replay_keep_all):
    slices validated and copied by several host threads.  Must equal the straightforward answer, with and without -w
    rejects, and fall back to the cursor replay when an overlap sits exactly on a slice boundary."""
    import numpy as np
    L = lib.load()
    n, m = (1 << 20) + 12345, 3
    rng = np.random.default_rng(5)
    starts = np.arange(n, dtype=np.uint64) * 5 + 2
    for whole_word in (False, True):
        tags = rng.choice(np.array([7, 7, 7, 6, 5, 4], dtype=np.uint64), size=n) if whole_word else np.full(n, 7, dtype=np.uint64)
        keys = np.ascontiguousarray((starts << np.uint64(3)) | tags)
        p = Params(b"abc", whole_word=whole_word)
        res = L.krep_b200_match_result_init(16)
        cnt = L.krep_b200_replay(ALGO_BMH, p.ref(), False, keys.ctypes.data_as(C.POINTER(C.c_uint64)), n, None, int(starts[-1]) + 10, res)
        keep = (tags & np.uint64(3)) == 3
        assert cnt == int(keep.sum()) == res.contents.count
        got = np.ctypeslib.as_array(C.cast(res.contents.positions, C.POINTER(C.c_uint64)), shape=(int(cnt), 2))
        assert np.array_equal(got[:, 0], starts[keep]) and np.array_equal(got[:, 1], starts[keep] + np.uint64(m))
        L.krep_b200_match_result_free(res)
    # an overlapping pair right at a slice boundary (n * t / 8): the bulk path must refuse, the cursor walk decides
    keys2 = (starts << np.uint64(3)) | np.uint64(7)
    b = n * 3 // 8
    keys2[b] = ((starts[b - 1] + np.uint64(1)) << np.uint64(3)) | np.uint64(7)
    keys2 = np.ascontiguousarray(keys2)
    for algo, expect in ((ALGO_BMH, n), (ALGO_KMP, n - 1)):        # BMH keeps overlapping occurrences, KMP does not
        res = L.krep_b200_match_result_init(16)
        cnt = L.krep_b200_replay(algo, Params(b"aaa").ref(), False, keys2.ctypes.data_as(C.POINTER(C.c_uint64)), n, None, int(starts[-1]) + 10, res)
        assert cnt == expect == res.contents.count
        L.krep_b200_match_result_free(res)
