"""CPU check of tests/regex_kernel_model.py, the reference the GPU tests hold k_regex_lines to: over random regexes,
random texts and random tilings of each text into shards, every line is owned by exactly one shard, and the model's
decided answers plus the reference loop over its uncertain lines reproduce the reference's -c count and positions."""
import random

import pytest

from krep_b200.abi import Params
import regex_kernel_model as km
from regex_kernel_model import random_lines_text, tiling
import regex_util as ru


def test_every_line_owned_once():
    rng = random.Random(1)
    for it in range(200):
        text = random_lines_text(rng, rng.randint(0, 12000))
        n = len(text)
        cuts = [rng.randint(0, n) for _ in range(rng.choice([0, 1, 2, 6, 20]))]
        owners = []
        for d, sh in tiling(text, cuts, rng):
            owners += [d + ln.p for ln in km.owned_lines(sh)]
        assert owners == ru.line_starts(text), (it, n, sorted(cuts))


def test_uncertain_lines_follow_the_reach():
    # '\n' at limit-1 is within reach, at limit it is not; the line holding the text's last byte is uncertain only at
    # the end of the text
    for extra in (km.REGEX_HALO - 1, km.REGEX_HALO):
        text = b"a" * (km.REGEX_SEG + extra) + b"\nb\n"
        sh = km.Shard(text, 0, km.REGEX_SEG)
        (ln,) = km.owned_lines(sh)
        assert (ln.nl is None) == (extra == km.REGEX_HALO)
    sh = km.Shard(b"ab\ncd\n", next_byte=-1)
    assert [ln.uncertain for ln in km.owned_lines(sh)] == [False, True]
    sh = km.Shard(b"ab\ncd\n", next_byte=ord("x"))
    assert [ln.uncertain for ln in km.owned_lines(sh)] == [False, False]
    assert [ln.p for ln in km.owned_lines(km.Shard(b"ab\ncd", prev_byte=ord("a")))] == [3]
    assert [ln.p for ln in km.owned_lines(km.Shard(b"ab\ncd", prev_byte=10))] == [0, 3]


@pytest.mark.parametrize("icase", [False, True])
def test_model_plus_reference_is_the_reference(icase):
    rng = random.Random(2 + icase)
    checked = 0
    for it in range(120):
        pats = [ru.random_regex(rng) for _ in range(rng.choice([1, 1, 2]))]
        try:
            Pc = Params([p.encode() for p in pats], regex=True, count=True, case_sensitive=not icase)
            Pp = Params([p.encode() for p in pats], regex=True, case_sensitive=not icase)
        except ValueError:
            continue
        text = random_lines_text(rng, rng.randint(1, 9000))
        n = len(text)
        cuts = [rng.randint(0, n) for _ in range(rng.choice([0, 1, 2, 6]))]
        count_keys, match_keys, lines = [], [], 0
        for d, sh in tiling(text, cuts, rng):
            g = km.GlibcLines(Pp, sh.buf)
            e1 = km.expect(sh, 1, g)
            e2 = km.expect(sh, 2, g, budget_free=True)
            count_keys += e1.keys
            lines += e1.device_lines
            match_keys += e2.keys
        assert km.resolve(Pc, text, 0, count_keys=count_keys, device_lines=lines) == ru.ref_regex_search(Pc, text)[0], \
            (pats, icase, n, sorted(cuts))
        assert km.resolve(Pp, text, 0, match_keys=match_keys) == ru.ref_regex_search(Pp, text)[1], (pats, icase, n, sorted(cuts))
        checked += 1
    assert checked > 80
