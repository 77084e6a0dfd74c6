"""Byte-exact model of what the literal and pattern-set scans write to device memory — pure Python + numpy, no GPU.

The kernels behind it (k_lit_aligned4 / k_lit_window4 in csrc/scan_literal.cu, k_ac_tri4 / k_ac_scan in
csrc/scan_multi.cu, k_count_lines in csrc/scan_count.cu, k_line_bounds and k_finish in csrc/engine.cu) filter and then
verify; whatever filter a plan uses, the list it leaves must be exactly the one defined here from the text alone:

* literal keys (csrc/common.h:15-21, verify_exact in csrc/lit_filters.cuh): one key per start s with
  own_begin <= s < min(own_end, avail_len) and s + emit_len <= avail_len whose first emit_len bytes equal the pattern's
  under the plan's fold; key = (global_offset + s) << 3 | full << 2 | ws_ok << 1 | we_ok.  full = all m bytes match
  (and fit); ws_ok / we_ok = no word byte before s / at s + m, taken from prev_byte / next_byte at the buffer's edges.
  -w mode 1 drops a key whose tag is not 3, mode 2 keeps it tagged, mode 0 tags 3.
* the fold under -i is the C locale's: a text byte and a pattern byte are equal when their ASCII lower cases are
  (engine.cu:559 masks with 0xDF on ASCII letters only — the same relation); no other byte folds.
* pattern-set keys (ac_verify_emit, csrc/scan_multi.cu): one key per (pattern index, owned start) of a non-empty pattern
  that fits below avail_len and matches; key = (global_offset + s + len) << 24 | (1023 - (len - 1)) << 14 | index.
  Duplicate patterns give one key each; -w drops failures.
* line bounds (k_line_bounds, engine.cu:839-896): two words per sorted key, markers LB_* included.
* fused -c records (k_count_lines + k_count_finish, csrc/scan_count.cu:35-41, include/krep_b200.h:338-344).
"""
from collections import namedtuple

import numpy as np

LIT_TAG_BITS, AC_END_SHIFT, AC_LEN_SHIFT, AC_MAX_PATTERNS = 3, 24, 14, 1 << 14
AC_MAX_OFFSET = 1 << 40  # pattern-set shards must end below this global offset (launch_scan refuses with -3)
LB_SAME_AS_PREV, LB_SAME_AS_NEXT, LB_OUTSIDE_SHARD = (1 << 64) - 1, (1 << 64) - 2, (1 << 64) - 3
LINES_HAS_HIT, LINES_FIRST_OPEN, LINES_LAST_PENDING, LINES_HAS_NL = 1, 2, 4, 8
PACK_KEYS = 16384  # lists up to this long are rank-sorted by k_finish, longer ones by CUB (engine.cu:989)

_LOWER = np.arange(256, dtype=np.uint8)
_LOWER[ord("A"):ord("Z") + 1] += 32
_WORD = np.zeros(257, dtype=bool)  # index 256 stands for "no byte" (-1)
for _c in b"0123456789ABCDEFGHIJKLMNOPQRSTUVWXYZabcdefghijklmnopqrstuvwxyz_":
    _WORD[_c] = True

Shape = namedtuple("Shape", "algo m emit_len ww_mode filter")


def resolve_algo(func, m, cs):
    """The precondition fallbacks of the simd entries (host_api.cu resolve_algo)."""
    if func == "avx512":
        if m == 0 or m > 64 or not cs:
            return "boyer_moore"
        if m <= 32:
            func = "avx2"
    if func == "avx2":
        if m == 0 or m > 32 or not cs:
            return "boyer_moore"
        if m <= 16:
            func = "sse42"
    if func == "sse42" and (m == 0 or m > 16 or not cs):
        return "boyer_moore"
    if func == "neon" and (m == 0 or not cs):
        return "boyer_moore"
    return func


def border_free(pattern, cs):
    """No proper prefix of the (folded) pattern is also a suffix: its occurrences cannot overlap (engine.cu:437)."""
    s = bytes(pattern) if cs else bytes(_LOWER[np.frombuffer(bytes(pattern), np.uint8)])
    pi = [0] * len(s)
    for i in range(1, len(s)):
        k = pi[i - 1]
        while k and s[i] != s[k]:
            k = pi[k - 1]
        pi[i] = k + (s[i] == s[k])
    return not s or pi[-1] == 0


def plan_shape(func, pats, cs=True, ww=False, only_matching=False):
    """(algo, m, emit_len, whole_word mode 0/1/2, filter) of the plan krep_b200_plan_create builds (engine.cu:529-577;
    pattern sets: csrc/scan_multi.cu:872-879).  `filter` is the beginning of krep_b200_plan_filter_name; a pattern set's
    name goes on with its bitmap size and ends in " fold" under -i."""
    if func == "aho_corasick":
        lens = [len(p) for p in pats if p]
        lmin = min(lens) if lens else 0
        if lmin >= 7:
            name = "window4/stride4 aligned-word hash"
        elif lmin == 6:
            name = "window3/stride4 tri4+byte-select"
        elif lmin == 5:
            name = "window4/stride2 paired"
        else:
            name = f"window{lmin or 1}/stride1 bitmap"
        return Shape(func, lmin, None, 1 if ww else 0, name)
    pat = bytes(pats[0] if isinstance(pats, (list, tuple)) else pats)
    algo = resolve_algo(func, len(pat), cs)
    if algo == "memchr":
        pat = pat[:1]
    m = len(pat)
    emit_len = 1 if algo == "memchr_short" and only_matching else m
    mode = 0
    if ww:
        tag = emit_len != m or algo in ("avx2", "avx512", "neon")
        if not tag and not border_free(pat, cs):
            tag = algo == "kmp" or (algo == "sse42" and not only_matching)
        mode = 2 if tag else 1
    name = ("aligned4" if emit_len >= 7 else "window4") + ("" if cs else "-fold")
    return Shape(algo, m, emit_len, mode, name)


def filter_matches(name, shape, cs):
    """Does the library's filter name say the plan runs the kernel `shape` expects?"""
    if shape.algo == "aho_corasick":
        return name.startswith(shape.filter) and name.endswith(" fold") == (not cs)
    return name == shape.filter


def _u8(text):
    return np.frombuffer(bytes(text), dtype=np.uint8) if not isinstance(text, np.ndarray) else text


def _fold(a, cs):
    return a if cs else _LOWER[a]


def _candidates(t, lo, hi, first_bytes):
    """Starts in [lo, hi) whose byte is one of first_bytes."""
    lut = np.zeros(256, dtype=bool)
    lut[np.frombuffer(bytes(first_bytes), np.uint8)] = True
    return np.flatnonzero(lut[t[lo:hi]]).astype(np.int64) + lo


def _windows(t, s, w):
    """Little-endian value of the w <= 8 bytes at each start s (all of them inside t)."""
    v = np.zeros(s.size, dtype=np.uint64)
    for j in range(w):
        v |= t[s + j].astype(np.uint64) << np.uint64(8 * j)
    return v


def _le(b):
    return int.from_bytes(bytes(b), "little")


def _verify_rest(t, starts, pats_rows, lo_byte, chunk=1 << 16):
    """Keep the (start, row) pairs whose bytes [lo_byte, L) equal the pattern row's (t holds every byte read)."""
    L = pats_rows.shape[1]
    if L <= lo_byte or starts.size == 0:
        return np.ones(starts.size, dtype=bool)
    ok = np.empty(starts.size, dtype=bool)
    cols = np.arange(lo_byte, L)
    for a in range(0, starts.size, chunk):
        s = starts[a:a + chunk]
        ok[a:a + chunk] = (t[s[:, None] + cols[None, :]] == pats_rows[a:a + chunk, lo_byte:]).all(axis=1)
    return ok


def match_starts(t, lo, hi, pat):
    """Starts s in [lo, hi) with t[s:s+len(pat)] == pat (the caller keeps s + len(pat) <= len(t))."""
    L = len(pat)
    if hi <= lo or L == 0:
        return np.zeros(0, dtype=np.int64)
    w = min(L, 8)
    s = _candidates(t, lo, hi, pat[:1])
    s = s[_windows(t, s, w) == np.uint64(_le(pat[:w]))]
    if L > w:
        rows = np.broadcast_to(np.frombuffer(bytes(pat), np.uint8), (s.size, L))
        s = s[_verify_rest(t, s, rows, w)]
    return s


def _is_word_at(t, idx, context_byte):
    """Is the byte at each index a word byte?  Indexes outside t read `context_byte` (-1: no byte, not a word byte)."""
    b = np.full(idx.shape, context_byte, dtype=np.int64)
    inside = (idx >= 0) & (idx < t.size)
    b[inside] = t[idx[inside]]
    return _WORD[np.where(b < 0, 256, b)]


def _word_before(t, s, prev_byte):
    return _is_word_at(t, s - 1, prev_byte)


def _word_at(t, e, avail_len, next_byte):
    return _is_word_at(t[:avail_len], e, next_byte)


def literal_keys(text, avail_len, own_begin, own_end, global_offset, prev_byte, next_byte, pattern, cs, emit_len, ww_mode):
    """Sorted uint64 keys one literal scan of the shard leaves (see the module doc)."""
    t = _fold(_u8(text)[:avail_len], cs)
    pat = _fold(np.frombuffer(bytes(pattern), np.uint8), cs).tobytes()
    m = len(pat)
    own_end = min(own_end, avail_len)
    s = match_starts(t, own_begin, min(own_end, avail_len - emit_len + 1), pat[:emit_len])
    full = np.ones(s.size, dtype=np.uint64)
    if m > emit_len:
        fits = s + m <= avail_len
        f = np.zeros(s.size, dtype=bool)
        sf = s[fits]
        f[fits] = _verify_rest(t, sf, np.broadcast_to(np.frombuffer(pat, np.uint8), (sf.size, m)), emit_len)
        full = f.astype(np.uint64)
    tag = np.full(s.size, 3, dtype=np.uint64)
    if ww_mode:
        raw = _u8(text)[:avail_len]
        ws = ~_word_before(raw, s, prev_byte)
        we = ~_word_at(raw, s + m, avail_len, next_byte)
        tag = (ws.astype(np.uint64) << np.uint64(1)) | we.astype(np.uint64)
        if ww_mode == 1:
            keep = tag == 3
            s, full, tag = s[keep], full[keep], tag[keep]
    return ((s.astype(np.uint64) + np.uint64(global_offset)) << np.uint64(LIT_TAG_BITS)) | (full << np.uint64(2)) | tag


def ac_keys(text, avail_len, own_begin, own_end, global_offset, prev_byte, next_byte, patterns, cs, whole_word):
    """Sorted uint64 keys one pattern-set scan of the shard leaves (see the module doc)."""
    raw = _u8(text)[:avail_len]
    t = _fold(raw, cs)
    own_end = min(own_end, avail_len)
    by_len = {}
    for k, p in enumerate(patterns):
        if p:
            by_len.setdefault(len(p), []).append(k)
    out = []
    for L, ks in by_len.items():
        hi = min(own_end, avail_len - L + 1)
        if hi <= own_begin:
            continue
        rows = _fold(np.frombuffer(b"".join(bytes(patterns[k]) for k in ks), np.uint8).reshape(len(ks), L), cs)
        w = min(L, 8)
        pv = np.array([_le(r[:w]) for r in rows], dtype=np.uint64)
        order = np.argsort(pv, kind="stable")
        pv_sorted, ks_sorted, rows_sorted = pv[order], np.array(ks, dtype=np.int64)[order], rows[order]
        c = _candidates(t, own_begin, hi, rows[:, 0].tobytes())
        tv = _windows(t, c, w)
        a = np.searchsorted(pv_sorted, tv, "left")
        b = np.searchsorted(pv_sorted, tv, "right")
        n = b - a
        cand = np.flatnonzero(n)
        if cand.size == 0:
            continue
        reps = n[cand]
        s = np.repeat(c[cand], reps)
        first = np.repeat(a[cand], reps)
        within = np.arange(reps.sum()) - np.repeat(np.cumsum(reps) - reps, reps)
        j = first + within
        if L > w:
            ok = _verify_rest(t, s, rows_sorted[j], w)
            s, j = s[ok], j[ok]
        if whole_word:
            ok = ~_word_before(raw, s, prev_byte) & ~_word_at(raw, s + L, avail_len, next_byte)
            s, j = s[ok], j[ok]
        out.append(((s.astype(np.uint64) + np.uint64(global_offset + L)) << np.uint64(AC_END_SHIFT))
                   | np.uint64((1023 - (L - 1)) << AC_LEN_SHIFT) | ks_sorted[j].astype(np.uint64))
    return np.sort(np.concatenate(out)) if out else np.zeros(0, dtype=np.uint64)


def key_starts(keys, is_ac):
    keys = np.asarray(keys, dtype=np.uint64)
    if not is_ac:
        return keys >> np.uint64(LIT_TAG_BITS)
    return (keys >> np.uint64(AC_END_SHIFT)) - (np.uint64(1024) - ((keys >> np.uint64(AC_LEN_SHIFT)) & np.uint64(1023)))


def line_bounds(keys, text, avail_len, global_offset, prev_byte, next_byte, is_ac):
    """The 2 * len(keys) words k_line_bounds writes for the sorted keys (engine.cu:839-916), markers included.

    Literal plans search backwards only down to the previous key's start and forwards only up to the next key's start
    (LB_SAME_AS_PREV / LB_SAME_AS_NEXT when no newline lies there); pattern sets search the whole buffer.  At the
    buffer's edges the line goes on into a neighbour (LB_OUTSIDE_SHARD) unless the context byte is absent or a newline."""
    n = len(keys)
    out = np.zeros(2 * n, dtype=np.uint64)
    if n == 0:
        return out
    s = key_starts(keys, is_ac).astype(np.int64) - global_offset
    nl = np.flatnonzero(_u8(text)[:avail_len] == 10)
    has_prev = prev_byte >= 0 and prev_byte != 10
    has_next = next_byte >= 0 and next_byte != 10
    i = np.arange(n)
    lb = np.zeros(n, dtype=np.int64)
    ub = np.full(n, avail_len, dtype=np.int64)
    if not is_ac:
        lb[1:] = s[:-1]
        ub[:-1] = s[1:]
    j = np.searchsorted(nl, s, "left")          # nl[j-1] < s <= nl[j]
    padded = np.concatenate(([-1], nl, [avail_len]))
    last, nxt = padded[j], padded[j + 1]        # last newline before s, first one at or after it
    found_b = last >= lb
    found_f = nxt < ub
    go = np.uint64(global_offset)
    default_b = np.uint64(LB_OUTSIDE_SHARD if has_prev else global_offset)
    default_f = np.uint64(LB_OUTSIDE_SHARD if has_next else global_offset + avail_len)
    ls = np.where(found_b, last.astype(np.uint64) + go + np.uint64(1), default_b)
    le = np.where(found_f, nxt.astype(np.uint64) + go, default_f)
    if not is_ac:
        ls = np.where(~found_b & (i > 0), np.uint64(LB_SAME_AS_PREV), ls)
        le = np.where(~found_f & (i + 1 < n), np.uint64(LB_SAME_AS_NEXT), le)
    out[0::2], out[1::2] = ls, le
    return out


def resolve_bounds(bounds):
    """The markers resolved as krep_b200_collect resolves them (host_api.cu): SAME_AS_PREV takes the previous key's line
    start, SAME_AS_NEXT the next key's line end; a marker with no neighbour becomes LB_OUTSIDE_SHARD."""
    b = [int(x) for x in bounds]
    n = len(b) // 2
    for i in range(n):
        if b[2 * i] == LB_SAME_AS_PREV:
            b[2 * i] = b[2 * (i - 1)] if i else LB_OUTSIDE_SHARD
    for i in range(n - 1, -1, -1):
        if b[2 * i + 1] == LB_SAME_AS_NEXT:
            b[2 * i + 1] = b[2 * (i + 1) + 1] if i + 1 < n else LB_OUTSIDE_SHARD
    return b


def line_record(text, own_begin, own_end, starts):
    """(lines, flags) of krep_b200_count_lines_shard for a shard whose owned occurrences start at `starts` (buffer
    offsets, any order).  Only the owned range's newlines count: the shard cuts a line there, and the fold of the records
    (krep_b200_combine_line_counts) joins the two halves.  lines = newline-delimited segments of the owned range that
    hold an occurrence start; FIRST_OPEN = no newline before the first one, LAST_PENDING = none after the last one.
    A record with a hit always has HAS_NL set (scan_count.cu:367); without one, HAS_NL says whether the range holds a
    newline."""
    t = _u8(text)
    nl = np.flatnonzero(t[own_begin:own_end] == 10) + own_begin
    h = np.unique(np.asarray(starts, dtype=np.int64))
    if h.size == 0:
        return 0, (LINES_HAS_NL if nl.size else 0)
    seg = np.searchsorted(nl, h, "left")
    flags = LINES_HAS_HIT | LINES_HAS_NL
    if seg[0] == 0:
        flags |= LINES_FIRST_OPEN
    if seg[-1] == nl.size:
        flags |= LINES_LAST_PENDING
    return int(np.unique(seg).size), flags


def shard_keys(shape, pats, cs, buf, avail_len, own_begin, own_end, global_offset=0, prev_byte=-1, next_byte=-1, ww=False):
    """literal_keys / ac_keys for the plan `shape` describes."""
    if shape.algo == "aho_corasick":
        return ac_keys(buf, avail_len, own_begin, own_end, global_offset, prev_byte, next_byte, pats, cs, ww)
    pat = bytes(pats[0] if isinstance(pats, (list, tuple)) else pats)[:shape.m]
    return literal_keys(buf, avail_len, own_begin, own_end, global_offset, prev_byte, next_byte, pat, cs, shape.emit_len,
                        shape.ww_mode)


def device_like_keys(func, pats, text, cs, whole_word, only_matching):
    """The list of a scan of the whole text as one shard, every key tagged under -w (as a tag-mode plan leaves it; the
    replay drops the failures of a drop-mode plan itself).  A plain list of ints."""
    n = len(text)
    if func == "aho_corasick":
        return ac_keys(text, n, 0, n, 0, -1, -1, pats, cs, whole_word).tolist()
    shape = plan_shape(func, pats, cs, whole_word, only_matching)
    if shape.m == 0:
        return []
    return literal_keys(text, n, 0, n, 0, -1, -1, bytes(pats[0])[:shape.m], cs, shape.emit_len, 2 if whole_word else 0).tolist()
