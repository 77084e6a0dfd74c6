"""-i bracket ranges on the GPU, where glibc's set is not the case closure of the range ([A-z] holds letters only;
[a-|] and [z-{] hold [\\]^_`): the raw keys of k_regex_lines against tests/regex_kernel_model.py in every mode a plan
admits, for one-automaton and split plans; and krep_b200_regex_search, krep_b200_search_shards and
krep_b200_regex_search_batch with -i against the reference's regex_search loop on full-byte text."""
import random

import pytest

from krep_b200 import lib
from krep_b200.abi import ALGO_REGEX, Params, Shard
import gpu_util as gu
import regex_kernel_model as km
import regex_util as ru
from test_gpu_regex_sets import RawPlan, lower_words, run_shard
import test_regex_dfa as td

pytestmark = pytest.mark.gpu
ICASE = dict(case_sensitive=False)
ATOMS = ["[A-z]", "a[A-z]b", "[^A-z]", "[2-z]_", "[a-|]+", "[z-{]", "[#-Z]x"]
# (patterns, filter name, modes): [A-z] next to 200 words folds into one automaton (a line with a letter matches), in
# context it splits; [a-|] widens the plan (its parsed range is not closed under case), so only the filter runs
WORDS = lower_words(random.Random("charset words"), 200)
SETS = {
    "200 words + [A-z]": (WORDS[:100] + ["[A-z]"] + WORDS[100:], "regex-lines", [0, 1]),
    "200 words + x[A-z]y": (WORDS[:100] + ["x[A-z]y", "[^A-z]_[^A-z]"] + WORDS[100:], "regex-lines-split", [0, 1, 2]),
    "200 words + _[a-|]_": (WORDS[:100] + ["_[a-|]_"] + WORDS[100:], "regex-lines-split-widened", [0]),
}
EDGE = b"[\\]^_`{|}~@AZaz xy" + bytes([0, 13, 0x80, 0xC1, 0xFF])


@pytest.fixture(scope="module", autouse=True)
def _init():
    L = lib.load()
    assert L.krep_b200_init(0) == 0, L.krep_b200_last_error_string()


@pytest.fixture(autouse=True)
def _device_paths_on(monkeypatch):
    monkeypatch.delenv("KREP_B200_NO_FUSED_COUNT", raising=False)
    monkeypatch.delenv("KREP_B200_NO_DEVICE_MATCHES", raising=False)


def _params(pats, **kw):
    if isinstance(pats, str):
        pats = [pats]
    return Params([p.encode() for p in pats], regex=True, **kw)


def charset_text(rng, n, words=(), long_lines=True):
    """Short lines of the bytes around Z..a and z..{, NUL, '\\r' and 0x80-0xFF, with fragments like a_b and aZb, words
    of the set (some upper-cased), any byte now and then, and with long_lines a line longer than the kernel's reach."""
    out = bytearray()
    while len(out) < n:
        if long_lines and rng.random() < 0.01:
            out += bytes(rng.choice(EDGE) for _ in range(rng.randint(4200, 5000))) + b"\n"
            continue
        for _ in range(rng.randint(0, 4)):
            r = rng.random()
            if r < 0.3 and words:
                w = rng.choice(words).encode()
                out += w.upper() if rng.random() < 0.3 else w
            elif r < 0.5:
                out += b"a" + bytes([rng.choice(EDGE)]) + b"b"
            elif r < 0.6:
                out.append(rng.randrange(256))
            else:
                out += bytes(rng.choice(EDGE) for _ in range(rng.randint(1, 6)))
        out += b"\n"
    text = bytes(out[:n])
    return text if rng.random() < 0.5 else text.rstrip(b"\n") + b"\n"


def check_plan(P, text, name, modes, rng, what):
    """The plan's filter is sound against glibc on text; its raw keys equal the model's on the whole text and on a
    tiling of it, in every mode it admits."""
    plan = RawPlan(P)
    try:
        assert plan.name == name and plan.modes == modes, (what, plan.name, plan.modes)
        assert set(td._glibc_lines(P, text, any_start=False)) <= plan.flagged(text), what
        t = gu.to_device(text)
        run_shard(plan, t.data_ptr(), km.Shard(text), what=what)
        for d, sh in km.tiling(text, sorted(rng.sample(range(1, len(text)), 3)), rng):
            run_shard(plan, t.data_ptr() + d, sh, what=(what, d))
    finally:
        plan.close()


@pytest.mark.parametrize("atom", ATOMS)
def test_atom_raw_keys(atom):
    rng = random.Random(atom)
    P = _params(atom, **ICASE)
    exact = lib.load().krep_b200_regex_count_mode(_params(atom, count=True, **ICASE).ref()) == 1
    check_plan(P, charset_text(rng, 120000), "regex-lines" if exact else "regex-lines-widened", [0, 1, 2] if exact else [0],
               rng, atom)


@pytest.mark.parametrize("set_name", list(SETS))
def test_set_raw_keys(set_name):
    pats, name, modes = SETS[set_name]
    rng = random.Random(set_name)
    check_plan(_params(pats, **ICASE), charset_text(rng, 200000, WORDS), name, modes, rng, set_name)


OPTS = [dict(count=True), dict(), dict(max_count=3), dict(count=True, max_count=5), dict(count=True, only_matching=True)]
CASES = {**{a: [a] for a in ATOMS}, **{k: pats for k, (pats, _, _) in SETS.items()}}


def _want(P, text):
    r = ru.ref_regex_search(P, text)
    return r[0], r[1] if P.struct.track_positions else []


@pytest.mark.parametrize("case", list(CASES))
def test_search_entry_points(case):
    """krep_b200_regex_search on one text, krep_b200_search_shards on 1 and 4 shards of it, and
    krep_b200_regex_search_batch on texts of 0..20000 bytes, with -i, against the reference loop."""
    pats = CASES[case]
    rng = random.Random(case)
    words = WORDS if len(pats) > 1 else ()
    text = charset_text(rng, 300000, words)
    batch = [charset_text(rng, rng.choice([1, 50, 3000, 20000]), words, long_lines=False) for _ in range(30)] + [b""]
    L = lib.load()
    for kw in OPTS:
        P = _params(pats, **ICASE, **kw)
        want = _want(P, text)
        assert lib.search("regex", P, text) == want, (pats, kw)
        h = L.krep_b200_plan_create(P.ref(), ALGO_REGEX)
        lib.check(L)
        try:
            L.krep_b200_set_only_matching(bool(P.only_matching))
            for k in (1, 4):
                cuts = sorted(rng.sample(range(1, len(text)), k - 1))
                shards = [sh for _, sh in km.tiling(text, cuts, rng)]
                bufs = [gu.to_device(sh.buf) for sh in shards]
                structs = [Shard(b.data_ptr(), sh.avail, sh.own_begin, sh.own_end, sh.global_offset, sh.prev_byte,
                                 sh.next_byte) for b, sh in zip(bufs, shards)]
                assert lib.search_shards(h, P, structs) == want, (pats, kw, k)
        finally:
            L.krep_b200_set_only_matching(False)
            L.krep_b200_plan_destroy(h)
        got = lib.regex_search_batch(P, batch)
        for i, t in enumerate(batch):
            assert got[i] == _want(P, t), (pats, kw, i)
