"""What one batch scan of krep_b200_regex_search_batch hands back with the -E long-line pass after each chunk's scan
(krep_b200_regex_search_batch_long_raw, DESIGN §12.5 and §12.8), for tests.  Built on regex_batch_model.Batch (the
packed buffer cut into chunks, each chunk a shard) and on the rules of regex_long_model.taken_lines / expect.

The pass takes a line of a text that k_regex_lines leaves out of reach (its '\\n' at or beyond the owner's limit) when

  * its '\\n' lies within the chunk's readable bytes (the chunk and REGEX_HALO bytes after it),
  * it is not its own text's last line (batch rule 2: its '\\n' is not the text's final byte or the gap's first),
  * it is shorter than 2^30 bytes,

and decides it as regex_long_model.expect does; count mode counts it on its own text.  Every other line is as in
Batch.expect.
"""
import numpy as np

import regex_batch_model as bm
import regex_kernel_model as km
import regex_long_model as lm


class LongBatch(bm.Batch):
    """Batch with the lines the pass takes: taken = [(text index, global p, global '\\n')], in order."""

    def __init__(self, texts, chunk=None):
        super().__init__(texts, chunk)
        nls = np.flatnonzero(np.frombuffer(self.buf, dtype=np.uint8) == 10)
        n = len(self.buf)
        self.taken = []
        for i, p, nl, _ in self.lines:
            if nl is not None:
                continue  # within reach: k_regex_lines' own line
            k = int(np.searchsorted(nls, p))
            if k == len(nls):
                continue
            q = int(nls[k])
            if q >= min(n, p // self.chunk * self.chunk + self.chunk + km.REGEX_HALO):
                continue  # the '\n' lies beyond the chunk's readable bytes
            if q + 1 >= self.offs[i] + len(self.texts[i]):
                continue  # the text's last line
            if q - p >= lm.MAX_LINE:
                continue
            self.taken.append((i, p, q))

    def expect(self, mode, oracle, budget_free=False):
        """-> regex_kernel_model.Expected of the whole batch (global keys) with .per = {text index: device lines} and
        .must_flag (match-mode line keys that must stay).  oracle: as regex_long_model.expect, over self.buf."""
        taken = {p: nl for _, p, nl in self.taken}
        per = {i: 0 for i in self.live}
        if mode == 0:
            keys, optional = [], set()
            for _, p, nl, _ in self.lines:
                k = p << km.LIT_TAG_BITS
                if nl is None and p not in taken:
                    optional.add(k)
                elif p in oracle:
                    keys.append(k)
            exp = km.Expected(0, keys, 0, self.lines, optional)
        elif mode == 1:
            keys = []
            for i, p, nl, unc in self.lines:
                if p in taken:
                    per[i] += oracle.verdict(p, taken[p])
                elif unc:
                    keys.append(p << km.LIT_TAG_BITS)
                elif oracle.verdict(p, nl):
                    per[i] += 1
            exp = km.Expected(1, keys, sum(per.values()), self.lines)
        else:
            keys, prefix, must = [], {}, set()
            for _, p, nl, unc in self.lines:
                lk = p << km.REGEX_MATCH_SHIFT
                if unc and p not in taken:
                    keys.append(lk)
                    continue
                nl = taken.get(p, nl)
                ms = oracle.matches(p, nl)
                long_at = next((j for j, (s, e) in enumerate(ms) if e - s >= lm.MAX_MATCH), None) if p in taken else None
                mk = [(s << km.REGEX_MATCH_SHIFT) | ((e - s) << km.LIT_TAG_BITS) | 1 for s, e in ms[:long_at]]
                if long_at is not None:
                    must.add(lk)
                    prefix[lk] = mk
                elif budget_free or (p not in taken and nl - p <= km.BUDGET_FREE_LEN) or not mk:
                    keys += mk
                else:
                    prefix[lk] = mk
            exp = km.Expected(2, sorted(keys), 0, self.lines, prefix_lines=prefix)
            exp.must_flag = must
        exp.per = per
        if mode != 2:
            exp.must_flag = set()
        return exp


def check(b, exp, keys, text_lines, what=""):
    """Hook output (sorted keys, per-text device lines indexed like b.texts) against the model."""
    lm.check(exp, keys, sum(text_lines) if exp.mode == 1 else 0, what)
    want = [exp.per.get(i, 0) if exp.mode == 1 else 0 for i in range(len(b.texts))]
    assert list(text_lines) == want, (what, [(i, g, w) for i, (g, w) in enumerate(zip(text_lines, want)) if g != w][:5])
