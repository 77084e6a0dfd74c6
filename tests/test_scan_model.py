"""CPU: pins tests/scan_model.py, the byte-exact model of what the literal and pattern-set scans write, to the compiled
reference (the oracle port when the reference is not built), on inputs over every byte value.

The model's keys, fed to the host replay (krep_b200_replay), must give the reference's answer; its line bounds, resolved
and fed to krep_b200_replay_lines, the reference's -c; and its fused -c records, folded over random cuts by
krep_b200_combine_line_counts, the reference's -c again.  The GPU side (test_gpu_scan_keys.py) then only has to equal
the model."""
import ctypes as C
import random

import numpy as np
import pytest

import oracle_util as ou
import scan_model as sm
from krep_b200 import lib
from krep_b200.abi import Params, SIZE_MAX
from test_oracle import random_case
from test_replay import ALGO, early_out, replay

# The byte pairs the -i word compare (text & 0xDFDFDFDF) cannot tell apart although only letters fold: NUL / space,
# @ / `, [ / {, \ / |, ] / }, ^ / ~, _ / DEL, digits / 0x10-0x19, 0xC0-0xDE / 0xE0-0xFE.
FOLD_ALIASES = [(0x00, 0x20), (0x40, 0x60), (0x5B, 0x7B), (0x5C, 0x7C), (0x5D, 0x7D), (0x5E, 0x7E), (0x5F, 0x7F)] + \
               [(0x30 + d, 0x10 + d) for d in range(10)] + [(0xC0 + d, 0xE0 + d) for d in range(31)]


def _alias(pairs):
    return bytes(sorted({b for p in pairs for b in p})) + b"aA\n"


FULL_BYTE_ALPHABETS = [
    bytes(range(256)),                                                  # uniform
    _alias(FOLD_ALIASES),                                               # every alias pair
    _alias(FOLD_ALIASES[:3]), _alias(FOLD_ALIASES[3:7]) + b"bB",        # a few pairs: dense aliases of pattern bytes
    _alias([(0x31, 0x11), (0x39, 0x19), (0xC1, 0xE1), (0xDE, 0xFE), (0xC9, 0xE9)]),
    b"\x00\x00\x00\xff\xff\xff a\n",                                    # runs of NUL and 0xFF
    b"\n\x8a\x0b\n\x8a\x0b a",                                          # newline next to 0x8A and 0x0B
    b"a_1Z\xe9\xc1\x80\xff\x00 \n",                                     # word bytes next to high bytes (-w)
]


def full_byte_case(rng, func):
    return random_case(rng, func, FULL_BYTE_ALPHABETS)


def checkers(func):
    if func == "avx512":
        return [ou.reference512() or ou.port()]
    if func == "neon":
        return [ou.reference_neon() or ou.port()]
    return [ou.reference() or ou.port()]


def _skip(func, opts, pats):
    # the sse42 entry hands these to boyer_moore_search: covered by that parametrisation
    return func == "sse42" and (len(pats[0]) > 16 or not opts["case_sensitive"])


def model_keys(func, pats, text, opts):
    shape = sm.plan_shape(func, pats, opts["case_sensitive"], opts["whole_word"], opts["only_matching"])
    return shape, sm.shard_keys(shape, pats, opts["case_sensitive"], text, len(text), 0, len(text),
                                ww=opts["whole_word"]).tolist()


@pytest.mark.parametrize("func", list(ALGO))
def test_model_keys_replay_to_the_reference_answer(func):
    rng = random.Random(4242 + ALGO[func])
    chks = checkers(func)
    n_checked = 0
    for _ in range(1500):
        pats, text, opts, with_res = full_byte_case(rng, func)
        if _skip(func, opts, pats):
            continue
        p = Params(pats, **opts)
        if early_out(func, p, text):
            continue
        _, keys = model_keys(func, pats, text, opts)
        got = replay(func, p, keys, text, with_res)
        for chk in chks:
            want = chk.run(func, Params(pats, **opts), text, with_result=with_res)
            assert got == want, (chk.kind, func, pats, text, opts, with_res, got, want)
        n_checked += 1
    assert n_checked > 400


@pytest.mark.parametrize("func", list(ALGO))
def test_model_line_bounds_replay_to_the_reference_count(func):
    L = lib.load()
    rng = random.Random(5151 + ALGO[func])
    chk = checkers(func)[0]
    n_checked = 0
    for _ in range(1500):
        pats, text, opts, _ = full_byte_case(rng, func)
        opts = dict(opts, count=True, only_matching=False)
        if _skip(func, opts, pats):
            continue
        p = Params(pats, **opts)
        if early_out(func, p, text):
            continue
        shape, keys = model_keys(func, pats, text, opts)
        bounds = sm.line_bounds(keys, text, len(text), 0, -1, -1, func == "aho_corasick")
        rb = sm.resolve_bounds(bounds)
        assert sm.LB_OUTSIDE_SHARD not in rb          # a whole text: every line ends inside it
        arr = (C.c_uint64 * max(len(keys), 1))(*keys)
        barr = (C.c_uint64 * max(len(rb), 1))(*rb)
        if func == "aho_corasick":
            p.struct.ac_trie = 1
        cnt = L.krep_b200_replay_lines(ALGO[func], p.ref(), False, arr, len(keys), barr, len(text), None)
        p.struct.ac_trie = None
        want = chk.run(func, Params(pats, **opts), text, with_result=False)[0]
        assert int(cnt) == want, (func, pats, text, opts, int(cnt), want)
        n_checked += 1
    assert n_checked > 400


class LineCount(C.Structure):
    _fields_ = [("lines", C.c_uint64), ("flags", C.c_uint32), ("reserved", C.c_uint32)]


def combine(recs, max_count=SIZE_MAX):
    L = lib.load()
    L.krep_b200_combine_line_counts.argtypes = [C.POINTER(LineCount), C.c_size_t, C.c_size_t]
    L.krep_b200_combine_line_counts.restype = C.c_uint64
    arr = (LineCount * max(len(recs), 1))(*[LineCount(a, b, 0) for a, b in recs])
    return int(L.krep_b200_combine_line_counts(arr, len(recs), max_count))


def random_cuts(rng, n):
    k = rng.choice([0, 1, 2, 5])
    return sorted({0, n, *(rng.randint(0, n) for _ in range(k))})


def shard_record(shape, pat, cs, text, b, e, halo):
    """The fused -c record of owned range [b, e) scanned from a buffer of its own: halo bytes past e, context bytes."""
    n = len(text)
    avail = min(e + halo, n)
    buf = text[b:avail]
    keys = sm.literal_keys(buf, avail - b, 0, e - b, b, text[b - 1] if b else -1, text[avail] if avail < n else -1,
                           pat, cs, shape.emit_len, shape.ww_mode)
    starts = (sm.key_starts(keys, False).astype(np.int64) - b)
    return sm.line_record(buf, 0, e - b, starts)


FUSED = ["boyer_moore", "kmp", "memchr", "memchr_short", "sse42"]


@pytest.mark.parametrize("func", FUSED)
def test_line_records_fold_to_the_reference_count(func):
    """Records of random cuts (halo m - 1 and longer), folded, give -c; -m caps the fold."""
    rng = random.Random(6161 + ALGO[func])
    chk = checkers(func)[0]
    n_checked = 0
    for _ in range(1500):
        pats, text, opts, _ = full_byte_case(rng, func)
        opts = dict(opts, count=True, only_matching=False)
        if _skip(func, opts, pats):
            continue
        p = Params(pats, **opts)
        if early_out(func, p, text):
            continue
        shape = sm.plan_shape(func, pats, opts["case_sensitive"], opts["whole_word"], False)
        pat = bytes(pats[0])[:shape.m]
        if shape.ww_mode == 2 or b"\n" in pat:
            continue  # not counted by the fused kernel (count_lines_eligible)
        want = chk.run(func, Params(pats, **opts), text, with_result=False)[0]
        cuts = random_cuts(rng, len(text))
        halo = shape.m - 1 + rng.choice([0, 0, 1, 7])
        recs = [shard_record(shape, pat, opts["case_sensitive"], text, b, e, halo) for b, e in zip(cuts, cuts[1:])]
        assert combine(recs, opts["max_count"]) == want, (func, pats, text, opts, cuts, recs, want)
        n_checked += 1
    assert n_checked > 200


def test_line_record_and_bounds_by_hand():
    """Fixed cases of the record flags and of the bound markers, spelled out."""
    t = b"ab\nxab ab\nab"
    #     0123 456789 01
    assert sm.line_record(t, 0, len(t), [0, 4, 7, 10]) == (3, 1 | 2 | 4 | 8)
    assert sm.line_record(t, 3, 10, [4, 7]) == (1, 1 | 2 | 8)          # newline at 9 closes the line: not pending
    assert sm.line_record(t, 3, 9, [4, 7]) == (1, 1 | 2 | 4 | 8)       # ... unless it lies outside the owned range
    assert sm.line_record(t, 0, 2, []) == (0, 0)
    assert sm.line_record(t, 0, 3, []) == (0, 8)
    keys = sm.literal_keys(t, len(t), 0, len(t), 100, -1, -1, b"ab", True, 2, 0)
    assert (keys >> np.uint64(3)).tolist() == [100, 104, 107, 110]
    b = sm.line_bounds(keys, t, len(t), 100, -1, -1, False).tolist()
    P, N = sm.LB_SAME_AS_PREV, sm.LB_SAME_AS_NEXT
    assert b == [100, 102, 103, N, P, 109, 110, 112]
    assert sm.resolve_bounds(b) == [100, 102, 103, 109, 103, 109, 110, 112]
    # a shard that cuts lines on both sides: the first line starts and the last one ends outside it
    b = sm.line_bounds(keys, t, len(t), 100, ord("x"), ord("y"), False).tolist()
    assert b[0] == sm.LB_OUTSIDE_SHARD and b[-1] == sm.LB_OUTSIDE_SHARD
    b = sm.line_bounds(keys, t, len(t), 100, ord("\n"), ord("\n"), False).tolist()
    assert b[0] == 100 and b[-1] == 112
    # pattern sets: no neighbour markers, both directions search the whole buffer
    ak = sm.ac_keys(t, len(t), 0, len(t), 0, -1, -1, [b"ab", b"b", b"", b"ab"], True, False)
    # end ascending, then the longer pattern, then list order; the duplicate "ab" emits its own keys, "" none
    assert [(int(k) >> 24, int(k) & 0x3FFF) for k in ak] == [(e, k) for e in (2, 6, 9, 12) for k in (0, 3, 1)]
    assert sm.line_bounds(ak, t, len(t), 0, -1, -1, True).tolist()[:4] == [0, 2, 0, 2]


def test_model_fold_is_the_c_locale_fold():
    """Under -i only ASCII letters fold: every alias pair of the word fold is told apart, every letter pair is not."""
    for a, b in FOLD_ALIASES:
        for pat, txt in ((bytes([a]) * 2, bytes([b]) * 2), (bytes([b]) * 2, bytes([a]) * 2)):
            assert sm.literal_keys(txt, 2, 0, 2, 0, -1, -1, pat, False, 2, 0).size == 0, (hex(a), hex(b))
            assert sm.ac_keys(txt, 2, 0, 2, 0, -1, -1, [pat], False, False).size == 0, (hex(a), hex(b))
    for c in range(ord("a"), ord("z") + 1):
        assert sm.literal_keys(bytes([c - 32]), 1, 0, 1, 0, -1, -1, bytes([c]), False, 1, 0).size == 1


@pytest.mark.parametrize("func", list(ou.FUNCS) + ["avx512", "neon"])
def test_port_matches_reference_on_full_byte_inputs(func):
    """The port is pinned to the reference on the ASCII alphabets (tests/golden/ref_differential.npz); these are the
    same option mixes over every byte value."""
    ref = {"avx512": ou.reference512, "neon": ou.reference_neon}.get(func, ou.reference)()
    if ref is None:
        pytest.skip(f"compiled reference for {func} not available (oracle/_ref is built from the reference sources)")
    rng = random.Random(7373 + ALGO[func])
    for _ in range(1500):
        pats, text, opts, with_res = full_byte_case(rng, func)
        a = ou.port().run(func, Params(pats, **opts), text, with_result=with_res)
        b = ref.run(func, Params(pats, **opts), text, with_result=with_res)
        assert a == b, (func, pats, text, opts, with_res, a, b)
