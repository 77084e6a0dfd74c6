"""A plain restatement of what one k_regex_lines scan of a shard must hand back (scan_regex.cu, DESIGN §12), for tests.

A shard is the bytes at d_text (`buf`, avail_len of them) plus the numbers of krep_b200_shard_t.  The model says which
lines the shard owns, which of them the kernel cannot decide (uncertain), and, for the decided ones, the verdict and the
matches glibc's regexec gives on the line, through the regex_t that Params(..., regex=True) compiles and with the flags
regex_util.ref_regex_search uses.  The kernel's output in each mode follows from that:

  filter : on owned lines whose '\\n' lies within reach, key (G+p) << 3 exactly for the lines the line automaton flags
           (krep_b200_regex_filter_host); on the other owned lines a key is allowed but not required;
  count  : keys (G+p) << 3 of the uncertain lines, and the number of decided lines with a match;
  match  : keys (G+p) << 16 of the uncertain lines, and (s << 16) | ((e-s) << 3) | 1 for every match of every decided
           line with a match.  A line over the kernel's step budget carries its uncertain key and a prefix of its matches.
"""
import bisect
import ctypes as C

import numpy as np

from krep_b200 import lib
from krep_b200.abi import REG_ICASE, REG_NEWLINE, REG_NOTBOL, REG_STARTEND
import regex_util as ru

# restated from krep_b200/csrc/common.h
REGEX_SEG = 256
REGEX_HALO = 4096
LIT_TAG_BITS = 3
REGEX_MATCH_SHIFT = 16
STEPS_PER_BYTE, STEPS_BASE = 8, 256
# a line of at most this many bytes (before its '\n') cannot reach the match mode's step budget:
# (L+1) + L(L+1)/2 <= 8L + 256 for L <= 30
BUDGET_FREE_LEN = 30


class Shard:
    """krep_b200_shard_t over buf (= the bytes at d_text, avail_len == len(buf))."""

    def __init__(self, buf, own_begin=0, own_end=None, global_offset=0, prev_byte=-1, next_byte=-1):
        self.buf = bytes(buf)
        self.avail = len(self.buf)
        self.own_begin = own_begin
        self.own_end = self.avail if own_end is None else own_end
        self.global_offset = global_offset
        self.prev_byte = prev_byte
        self.next_byte = next_byte


class Line:
    __slots__ = ("p", "nl", "uncertain")

    def __init__(self, p, nl, uncertain):
        self.p, self.nl, self.uncertain = p, nl, uncertain


def owned_lines(sh):
    """[Line] for every line start p the shard owns, in order; nl is None when its '\\n' lies out of reach."""
    a = np.frombuffer(sh.buf, dtype=np.uint8)
    nls = np.flatnonzero(a == 10)
    own_end = min(sh.own_end, sh.avail)
    if sh.own_begin >= own_end:
        return []
    starts = nls + 1
    starts = starts[(starts >= max(sh.own_begin, 1)) & (starts < own_end)].tolist()
    if sh.own_begin == 0 and sh.prev_byte in (-1, 10):
        starts.insert(0, 0)
    out = []
    for p in starts:
        se = min(sh.own_begin + REGEX_SEG * ((p - sh.own_begin) // REGEX_SEG + 1), own_end)
        limit = min(se + REGEX_HALO, sh.avail)
        k = int(np.searchsorted(nls, p))
        nl = int(nls[k]) if k < len(nls) and nls[k] < limit else None
        unc = nl is None or (nl + 1 == sh.avail and sh.next_byte == -1)
        out.append(Line(p, nl, unc))
    return out


def _eflags(params):
    return REG_STARTEND | REG_NEWLINE | (0 if params.struct.case_sensitive else REG_ICASE)


class GlibcLines:
    """Verdicts and matches of single lines of buf, from glibc (the reference loop restricted to the line)."""

    def __init__(self, params, buf):
        self.params, self.rx = params, params.regex
        self.buf = C.create_string_buffer(bytes(buf), len(buf) + 1)
        self.base = _eflags(params)

    def matches(self, p, nl):
        """From cur = p, the leftmost match starting at or before nl (REG_NOTBOL once cur != p); then cur = e, or s+1
        after an empty match; while cur <= nl.  -> [(s, e)] relative to buf."""
        out, cur = [], p
        while cur <= nl:
            r = self.rx.search(self.buf, cur, nl + 1, self.base | (0 if cur == p else REG_NOTBOL))
            if r is None or cur + r[0] > nl:
                break
            s, e = cur + r[0], cur + r[1]
            out.append((s, e))
            cur = s + 1 if s == e else e
        return out

    def verdict(self, p, nl):
        r = self.rx.search(self.buf, p, nl + 1, self.base)
        return r is not None and r[0] <= nl - p


class HookLines:
    """The same answers for texts too large for per-line calls: verdicts from krep_b200_regex_filter_host (exact for
    count_exact plans), matches from krep_b200_regex_matches_host with unbounded reach (offsets_exact plans).  Both are
    fuzzed against glibc by the CPU suite."""

    def __init__(self, params, buf, positions_params=None):
        L = lib.load()
        b = C.create_string_buffer(bytes(buf), len(buf) + 1)
        cap = bytes(buf).count(b"\n") + 2
        out = (C.c_uint64 * cap)()
        k = L.krep_b200_regex_filter_host(params.ref(), b, len(buf), out, cap, None)
        assert 0 <= k <= cap, k
        self.flagged = set(np.ctypeslib.as_array(out)[:k].tolist())
        self.starts = []
        self.pos = []
        if positions_params is not None:
            res = L.krep_b200_match_result_init(16)
            try:
                n = L.krep_b200_regex_matches_host(positions_params.ref(), b, len(buf), (1 << 64) - 1, res)
                assert n >= 0, n
                r = res.contents
                self.pos = [(r.positions[i].start_offset, r.positions[i].end_offset) for i in range(r.count)]
                self.starts = [s for s, _ in self.pos]
            finally:
                L.krep_b200_match_result_free(res)

    def verdict(self, p, nl):
        return p in self.flagged

    def matches(self, p, nl):
        i, j = bisect.bisect_left(self.starts, p), bisect.bisect_right(self.starts, nl)
        return self.pos[i:j]


class Expected:
    """The model's answer for one shard in one mode."""

    def __init__(self, mode, keys, device_lines, lines, optional=(), prefix_lines=None):
        self.mode = mode
        self.keys = keys                  # sorted: keys the kernel must emit
        self.device_lines = device_lines  # count mode: decided lines with a match
        self.lines = lines
        self.optional = set(optional)     # filter mode: keys allowed but not required
        self.prefix_lines = prefix_lines or {}  # match mode: line key -> match keys, for lines that may go over budget


def expect(sh, mode, oracle, budget_free=False):
    """Model of a mode-0/1/2 scan of sh.  oracle: GlibcLines / HookLines over sh.buf (filter mode: a set of flagged line
    starts, krep_b200_regex_filter_host over sh.buf).  budget_free: every decided line is known to stay within the step
    budget (else lines longer than BUDGET_FREE_LEN may take the prefix form)."""
    G = sh.global_offset
    lines = owned_lines(sh)
    if mode == 0:
        keys, optional = [], []
        for ln in lines:
            k = (G + ln.p) << LIT_TAG_BITS
            if ln.nl is None:
                optional.append(k)
            elif ln.p in oracle:
                keys.append(k)
        return Expected(0, keys, 0, lines, optional)
    if mode == 1:
        keys = [(G + ln.p) << LIT_TAG_BITS for ln in lines if ln.uncertain]
        dl = sum(1 for ln in lines if not ln.uncertain and oracle.verdict(ln.p, ln.nl))
        return Expected(1, keys, dl, lines)
    keys, prefix = [], {}
    for ln in lines:
        lk = (G + ln.p) << REGEX_MATCH_SHIFT
        if ln.uncertain:
            keys.append(lk)
            continue
        ms = [((G + s) << REGEX_MATCH_SHIFT) | ((e - s) << LIT_TAG_BITS) | 1 for s, e in oracle.matches(ln.p, ln.nl)]
        if not budget_free and ln.nl - ln.p > BUDGET_FREE_LEN and ms:
            prefix[lk] = ms
        else:
            keys += ms
    return Expected(2, sorted(keys), 0, lines, prefix_lines=prefix)


def check(exp, keys, device_lines, what=""):
    """Asserts that a hook result (sorted keys, device_lines) is what the model allows."""
    assert keys == sorted(keys), what
    if exp.mode == 1:
        assert device_lines == exp.device_lines, (what, device_lines, exp.device_lines)
    else:
        assert device_lines == 0, what
    if exp.mode == 0:
        got = set(keys)
        missing = set(exp.keys) - got
        extra = got - set(exp.keys) - exp.optional
        assert not missing and not extra, (what, sorted(missing)[:5], sorted(extra)[:5])
        assert len(got) == len(keys), what
        return
    if exp.mode == 1 or not exp.prefix_lines:
        if keys != exp.keys:
            a, b = set(keys), set(exp.keys)
            raise AssertionError((what, len(keys), len(exp.keys), sorted(a - b)[:5], sorted(b - a)[:5]))
        return
    # match mode with lines that may go over budget: split the output by line and compare line by line
    fixed = set(exp.keys)
    rest = [k for k in keys if k not in fixed]
    assert len(keys) - len(rest) == len(fixed), (what, sorted(fixed - set(keys))[:5])
    starts = sorted(exp.prefix_lines)
    by_line = {}
    for k in rest:
        i = bisect.bisect_right(starts, k) - 1
        assert i >= 0, (what, hex(k))
        by_line.setdefault(starts[i], []).append(k)
    for lk, ms in exp.prefix_lines.items():
        got = by_line.get(lk, [])
        if got == ms:
            continue
        assert got and got[0] == lk and got[1:] == ms[: len(got) - 1], (what, hex(lk), [hex(k) for k in got[:4]],
                                                                      [hex(k) for k in ms[:4]])


def tiling(text, cuts, rng):
    """Shards over text cut at `cuts`: d_text at each cut rounded down to 16, own_begin the remainder, a readable halo
    of random length past the owned range. -> [(offset of d_text in text, Shard)]"""
    n = len(text)
    bounds = [0] + sorted(cuts) + [n]
    out = []
    for b, e in zip(bounds, bounds[1:]):
        d = b & ~15
        end = min(n, e + rng.choice([0, 1, 100, REGEX_HALO, REGEX_HALO + REGEX_SEG, 1 << 20]))
        out.append((d, Shard(text[d:end], b - d, e - d, d, text[d - 1] if d else -1, text[end] if end < n else -1)))
    return out


def random_lines_text(rng, n):
    """regex_util.random_text with an occasional line longer than the kernel's reach."""
    parts = []
    while sum(map(len, parts)) < n:
        if rng.random() < 0.1:
            parts.append(bytes(rng.choice(b"abcx ") for _ in range(rng.randint(4000, 5000))) + b"\n")
        else:
            parts.append(ru.random_text(rng, rng.randint(1, 400)))
    text = b"".join(parts)[:n]
    return text if rng.random() < 0.5 else text.rstrip(b"\n") + b"\n"


def resolve(params, text, G, count_keys=None, device_lines=0, match_keys=None):
    """Whole-text answers from concatenated hook outputs over a tiling of `text` (shard global offsets relative to G):
    the device's decided lines plus the reference loop over its uncertain lines.  The line that holds the text's last
    byte runs to the end of the text (it may also hold the empty string at n).  -> count, or [(s, e)]."""
    g = GlibcLines(params, text)
    n = len(text)

    def tail(p):
        nl = text.find(b"\n", p)
        return nl if 0 <= nl < n - 1 else None

    if count_keys is not None:
        total = device_lines
        for k in count_keys:
            p = (k >> LIT_TAG_BITS) - G
            nl = tail(p)
            if nl is None:
                total += ru.ref_regex_search(params, text[p:])[0]
            else:
                total += g.verdict(p, nl)
        return total
    pos = []
    for k in match_keys:
        p = (k >> REGEX_MATCH_SHIFT) - G
        if k & 1:
            pos.append((p, p + ((k >> LIT_TAG_BITS) & 0x1FFF)))
            continue
        nl = tail(p)
        if nl is None:
            pos += [(p + s, p + e) for s, e in ru.ref_regex_search(params, text[p:])[1]]
        else:
            pos += g.matches(p, nl)
    return pos
