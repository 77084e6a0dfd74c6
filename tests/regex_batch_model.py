"""What one batch scan of krep_b200_regex_search_batch must hand back (k_regex_lines in batch mode, DESIGN §12.5), for
tests.  Built on tests/regex_kernel_model.py: the packed buffer is scanned as one text cut into chunks, each chunk a
shard of that text, and three rules differ from the single-text kernel:

  1. a line that starts in a gap (the '\\n' bytes after a text) belongs to no text: it is not processed;
  2. in count and match mode a line is uncertain when its '\\n' is out of reach (as before) or when it holds its own
     text's last byte (nl + 1 >= the text's end: its '\\n' is the text's final byte or the gap's first);
  3. count mode counts the decided lines with a match per text.

Filter mode needs no end-of-text rule: the gap's first '\\n' ends a text's last line, where the single-text kernel
reads the '\\n' column at the end of the text.
"""
import bisect

import regex_kernel_model as km


def pack(texts):
    """The library's packing: each non-empty text at a 16-byte aligned offset, followed by at least one '\\n' up to the
    next 16-byte boundary.  -> (buf, offsets: packed offset per text or None when the text is not packed)"""
    parts, offs, t = [], [], 0
    for x in texts:
        if not x:
            offs.append(None)
            continue
        offs.append(t)
        nxt = (t + len(x) + 1 + 15) & ~15
        parts.append(x + b"\n" * (nxt - t - len(x)))
        t = nxt
    return b"".join(parts), offs


def chunks(buf, chunk):
    """The shards stage_and_scan cuts the packed text into: own [c, c + chunk), readable up to REGEX_HALO bytes further."""
    n, out = len(buf), []
    for c in range(0, n, chunk):
        end = min(n, c + chunk + km.REGEX_HALO)
        out.append(km.Shard(buf[c:end], 0, min(chunk, n - c), c, buf[c - 1] if c else -1, buf[end] if end < n else -1))
    return out


class Batch:
    """The packed buffer of `texts` with its text table and the lines each chunk owns, after rule 1."""

    def __init__(self, texts, chunk=None):
        self.texts = list(texts)
        self.buf, self.offs = pack(self.texts)
        self.live = [i for i, o in enumerate(self.offs) if o is not None]
        self.start = [self.offs[i] for i in self.live]
        self.end = [self.offs[i] + len(self.texts[i]) for i in self.live]
        self.chunk = chunk or max(len(self.buf), 1)
        self.lines = []  # (text index, global line start, global '\n' or None, uncertain)
        for sh in chunks(self.buf, self.chunk):
            G = sh.global_offset
            for ln in km.owned_lines(sh):
                p = G + ln.p
                k = bisect.bisect_right(self.start, p) - 1
                if k < 0 or p >= self.end[k]:
                    continue  # rule 1: a line in a gap
                nl = None if ln.nl is None else G + ln.nl
                self.lines.append((self.live[k], p, nl, nl is None or nl + 1 >= self.end[k]))

    def expect(self, mode, oracle, budget_free=False):
        """-> (sorted keys, {text index: device lines}) of a mode-0/1/2 scan; filter mode: (required keys, optional keys).
        oracle: as regex_kernel_model.expect, over self.buf (filter mode: the set of flagged line starts)."""
        if mode == 0:
            keys, optional = [], set()
            for _, p, nl, _ in self.lines:
                if nl is None:
                    optional.add(p << km.LIT_TAG_BITS)
                elif p in oracle:
                    keys.append(p << km.LIT_TAG_BITS)
            return keys, optional
        if mode == 1:
            keys = [p << km.LIT_TAG_BITS for _, p, _, unc in self.lines if unc]
            per = {i: 0 for i in self.live}
            for i, p, nl, unc in self.lines:
                if not unc and oracle.verdict(p, nl):
                    per[i] += 1
            return keys, per
        keys = []
        for _, p, nl, unc in self.lines:
            if unc:
                keys.append(p << km.REGEX_MATCH_SHIFT)
                continue
            assert budget_free or nl - p <= km.BUDGET_FREE_LEN, "long decided line: the model needs budget_free texts"
            keys += [(s << km.REGEX_MATCH_SHIFT) | ((e - s) << km.LIT_TAG_BITS) | 1 for s, e in oracle.matches(p, nl)]
        return sorted(keys), {}

    def text_keys(self, keys, i, shift):
        """The keys of text i (packed coordinates)."""
        lo, hi = self.offs[i], self.offs[i] + len(self.texts[i])
        return [k for k in keys if lo <= k >> shift < hi]
