"""CPU check of tests/regex_batch_long_model.py, the reference the GPU tests hold the long-line pass of
krep_b200_regex_search_batch to: over random regexes, batches of texts with many lines longer than the kernel's reach and
several chunkings of the packed buffer, the model's decided answers plus the reference loop over each text's uncertain
lines give each text's reference -c count, -co count and positions, with -i, -w and -m; lines the filter drops have no
match; each text's last line is never taken; and on texts without long lines the model is Batch.expect."""
import ctypes as C
import random

import pytest

from krep_b200 import lib
from krep_b200.abi import Params
import regex_batch_long_model as blm
import regex_kernel_model as km
import regex_long_model as lm
import regex_util as ru


def _params(pats, icase, **kw):
    try:
        return Params([p.encode() for p in pats], regex=True, case_sensitive=not icase, **kw)
    except ValueError:
        return None


def _flagged(params, buf):
    L = lib.load()
    b = C.create_string_buffer(bytes(buf), len(buf) + 1)
    cap = bytes(buf).count(b"\n") + 2
    out = (C.c_uint64 * cap)()
    k = L.krep_b200_regex_filter_host(params.ref(), b, len(buf), out, cap, None)
    assert 0 <= k <= cap, k
    return set(out[:k])


def long_texts(rng, k):
    """Texts of long and short lines, some a single long line, some ending in a long line with or without its '\\n', and
    empty and one-byte texts between them."""
    out = []
    for _ in range(k):
        r = rng.random()
        if r < 0.1:
            out.append(rng.choice([b"", b"a", b"\n"]))
        elif r < 0.2:
            out.append(bytes(rng.choice(b"abc x") for _ in range(rng.choice([4097, 4352, 9000]))))
        else:
            out.append(lm.long_lines_text(rng, rng.randint(1, 30000)))
            if rng.random() < 0.3:
                out[-1] += bytes(rng.choice(b"abc ,") for _ in range(rng.randint(4090, 9000)))  # a long last line
    return out


def test_taken_lines_follow_the_batch_rules():
    R = km.REGEX_SEG + km.REGEX_HALO
    long = b"a" * R
    texts = [long + b"\nb\n", long + b"\n", long, b"", b"q", long + b"\n" + long + b"\nz", b"x\n" + b"c" * 9000 + b"\nz\n"]
    b = blm.LongBatch(texts)
    got = [(i, p - b.offs[i], nl - b.offs[i]) for i, p, nl in b.taken]
    # text 0: taken; 1: its '\n' is the text's last byte; 2: its '\n' is the gap's first; 5: the first line only
    assert got == [(0, 0, R), (5, 0, R), (5, R + 1, 2 * R + 1), (6, 2, 9002)]
    # a chunk edge: the '\n' beyond the chunk and its halo leaves the line uncertain
    b = blm.LongBatch([b"a" * (3 * R) + b"\nb\n"], chunk=4096)
    assert b.taken == []
    b = blm.LongBatch([b"a" * (R + 10) + b"\nb\n"], chunk=4096)
    assert [(p, nl) for _, p, nl in b.taken] == [(0, R + 10)]


def test_sizes_hold_for_a_packed_batch():
    # the work list and the slice map of every chunk hold what the pass takes there, at S = 1 and the production size
    rng = random.Random(4)
    for it in range(20):
        texts = long_texts(rng, rng.randint(1, 12))
        for chunk in (4096, 1 << 16, 1 << 20):
            b = blm.LongBatch(texts, chunk)
            n = len(b.buf)
            for c in range(0, max(n, 1), chunk):
                own, avail = min(chunk, n - c), min(n, c + chunk + km.REGEX_HALO) - c
                mine = [(p, nl) for _, p, nl in b.taken if c <= p < c + chunk]
                for S in (1, lm.SLICE):
                    z = lm.sizes(avail, own, 1, S, 1)
                    assert len(mine) <= z.pick_cap
                    assert sum(-(-(nl - p) // S) for p, nl in mine) <= z.owner_cap, (it, chunk, c, S)


def test_every_text_last_line_stays_uncertain():
    rng = random.Random(6)
    for it in range(40):
        texts = long_texts(rng, rng.randint(1, 10))
        b = blm.LongBatch(texts, rng.choice([4096, 1 << 20]))
        taken = {p for _, p, _ in b.taken}
        for i in b.live:
            assert b.offs[i] + ru.line_starts(texts[i])[-1] not in taken, (it, i)


@pytest.mark.parametrize("icase", [False, True])
def test_model_plus_reference_is_the_reference(icase):
    rng = random.Random(21 + icase)
    checked = 0
    for it in range(40):
        pats = [rng.choice(["a[^x]*b", "(ab)*c", "^x.*y$", "a{3}b", ".*QQ|,", "b+ ", "x$", "^a", "c a", "^$", "x*"])
                if rng.random() < 0.5 else ru.random_regex(rng) for _ in range(rng.choice([1, 1, 2]))]
        Pp = _params(pats, icase)
        if Pp is None:
            continue
        m = rng.choice([1, 2, 3])
        Pc = _params(pats, icase, count=True)
        Pcm = _params(pats, icase, count=True, max_count=m)
        Pco = _params(pats, icase, count=True, only_matching=True)
        Ppm = _params(pats, icase, max_count=m)
        Pw = _params(pats, icase, whole_word=True)
        texts = long_texts(rng, rng.randint(1, 8))
        b = blm.LongBatch(texts, rng.choice([4096, 1 << 16, 1 << 20]))
        g = km.GlibcLines(Pp, b.buf)
        flagged = _flagged(Pp, b.buf)
        e0 = b.expect(0, flagged)
        e1 = b.expect(1, g)
        e2 = b.expect(2, g, budget_free=True)
        # a line the filter drops has no match, so no -w match either
        for i, p, nl in b.taken:
            if p not in flagged:
                assert not g.verdict(p, nl), (pats, icase, it, i)
        kept = {k >> km.LIT_TAG_BITS for k in e0.keys} | {k >> km.LIT_TAG_BITS for k in e0.optional}
        for i in b.live:
            G = b.offs[i]
            t = texts[i]
            ck = b.text_keys(e1.keys, i, km.LIT_TAG_BITS)
            mk = b.text_keys(sorted(e2.keys + sorted(e2.must_flag)), i, km.REGEX_MATCH_SHIFT)
            total = km.resolve(Pc, t, G, count_keys=ck, device_lines=e1.per[i])
            assert total == ru.ref_regex_search(Pc, t)[0], (pats, icase, it, i)
            assert min(total, m) == ru.ref_regex_search(Pcm, t)[0], (pats, icase, it, i, m)
            pos = km.resolve(Pp, t, G, match_keys=mk)
            assert pos == ru.ref_regex_search(Pp, t)[1], (pats, icase, it, i)
            assert len(pos) == ru.ref_regex_search(Pco, t)[0], (pats, icase, it, i)
            assert pos[:m] == ru.ref_regex_search(Ppm, t)[1], (pats, icase, it, i, m)
            # -w: every match lies on a line the filter keeps or leaves uncertain
            starts = ru.line_starts(t)
            for s, _ in ru.ref_regex_search(Pw, t)[1]:
                ls = starts[sum(1 for x in starts if x <= s) - 1]
                assert G + ls in kept, (pats, icase, it, i, s)
        checked += 1
    assert checked > 25


def test_equals_batch_model_without_long_lines():
    rng = random.Random(8)
    for it in range(30):
        P = _params([ru.random_regex(rng)], rng.random() < 0.3)
        if P is None:
            continue
        texts = [ru.random_text(rng, rng.randint(0, 3000)) for _ in range(rng.randint(1, 10))]
        b = blm.LongBatch(texts, rng.choice([256, 4096, 1 << 20]))
        assert b.taken == []
        g = km.GlibcLines(P, b.buf)
        flagged = _flagged(P, b.buf)
        for mode, oracle in ((0, flagged), (1, g), (2, g)):
            e = b.expect(mode, oracle, budget_free=True)
            keys, x = blm.bm.Batch.expect(b, mode, oracle, budget_free=True)
            if mode == 0:
                assert (sorted(e.keys), e.optional) == (sorted(keys), x), (it, mode)
            elif mode == 1:
                assert (e.keys, e.per) == (keys, x), (it, mode)
            else:
                assert (e.keys, e.prefix_lines, e.must_flag) == (keys, {}, set()), (it, mode)
