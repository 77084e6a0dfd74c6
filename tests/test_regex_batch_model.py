"""CPU check of tests/regex_batch_model.py, the reference the GPU tests hold the batch mode of k_regex_lines to: over
random regexes, random texts and chunkings of the packed buffer, every line of every text is processed exactly once and
no line of a gap is, and the model's decided answers plus the reference loop over each text's uncertain lines give each
text's reference answer."""
import random

import pytest

from krep_b200.abi import Params
import regex_batch_model as bm
import regex_kernel_model as km
import regex_util as ru


def random_texts(rng, k):
    out = []
    for _ in range(k):
        r = rng.random()
        if r < 0.1:
            out.append(b"")
        elif r < 0.15:
            out.append(b"\n" * rng.randint(1, 40))
        elif r < 0.2:
            out.append(bytes(rng.choice(b"ab\x00") for _ in range(rng.randint(1, 50))))
        else:
            out.append(km.random_lines_text(rng, rng.choice([1, 15, 16, 17, rng.randint(1, 700), rng.randint(1, 6000)])))
        if out[-1] and rng.random() < 0.5:
            out[-1] = out[-1].rstrip(b"\n") or b"x"
    return out


def test_pack_layout():
    buf, offs = bm.pack([b"abc", b"", b"x" * 15, b"y" * 16, b"z\n"])
    assert offs == [0, None, 16, 32, 64]
    assert buf == b"abc" + b"\n" * 13 + b"x" * 15 + b"\n" + b"y" * 16 + b"\n" * 16 + b"z\n" + b"\n" * 14


def test_every_text_line_processed_once():
    rng = random.Random(5)
    for it in range(120):
        texts = random_texts(rng, rng.randint(1, 30))
        for chunk in (256, 4096, 1 << 20):
            b = bm.Batch(texts, chunk)
            got = [(i, p) for i, p, _, _ in b.lines]
            want = [(i, b.offs[i] + p) for i in b.live for p in ru.line_starts(texts[i])]
            assert got == want, (it, chunk)
            # the line holding each text's last byte is uncertain, and the only one when every line is short
            for i in b.live:
                last = b.offs[i] + ru.line_starts(texts[i])[-1]
                unc = [p for j, p, _, u in b.lines if j == i and u]
                assert last in unc, (it, chunk, i)
                if max(map(len, texts[i].split(b"\n"))) < km.REGEX_SEG:
                    assert unc == [last], (it, chunk, i)


@pytest.mark.parametrize("icase", [False, True])
def test_model_plus_reference_is_the_reference(icase):
    rng = random.Random(11 + icase)
    checked = 0
    fixed = ["^$", "x*", "^", "$", "a|ab|abc", "b$", "\\bab\\b", "x$"]
    for it in range(80):
        pats = [fixed[it] if it < len(fixed) else ru.random_regex(rng)]
        try:
            Pc = Params([p.encode() for p in pats], regex=True, count=True, case_sensitive=not icase)
            Pp = Params([p.encode() for p in pats], regex=True, case_sensitive=not icase)
        except ValueError:
            continue
        texts = random_texts(rng, rng.randint(1, 12))
        b = bm.Batch(texts, rng.choice([256, 512, 4096, 1 << 20]))
        g = km.GlibcLines(Pp, b.buf)
        ck, per = b.expect(1, g)
        mk, _ = b.expect(2, g, budget_free=True)
        for i in b.live:
            G = b.offs[i]
            keys_c = b.text_keys(ck, i, km.LIT_TAG_BITS)
            keys_m = b.text_keys(mk, i, km.REGEX_MATCH_SHIFT)
            assert km.resolve(Pc, texts[i], G, count_keys=keys_c, device_lines=per[i]) == ru.ref_regex_search(Pc, texts[i])[0], \
                (pats, icase, it, i)
            assert km.resolve(Pp, texts[i], G, match_keys=keys_m) == ru.ref_regex_search(Pp, texts[i])[1], (pats, icase, it, i)
        checked += 1
    assert checked > 50
