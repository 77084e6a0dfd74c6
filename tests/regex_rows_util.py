"""A host twin of krep_b200_regex_export_shard for tests: the row (csrc/common.h, RegexRowHeader) of a shard built in
Python from host text, from the keys tests/regex_kernel_model.py says the scan emits.  Also the reader of a row, so
that a device row can be compared field by field with host slicing."""
import struct

import regex_kernel_model as km
from krep_b200 import lib

MAGIC = 0x31776F725F78726B
ROW_HEAD, ROW_LAST = 1, 2
HEADER = 128


def r16(v):
    return (v + 15) & ~15


def pad16(b):
    return b + b"\0" * (r16(len(b)) - len(b))


def call_mode(params):
    """The k_regex_lines mode a -E call with params takes (as krep_b200_regex_search decides it)."""
    L = lib.load()
    if L.krep_b200_regex_count_mode(params.ref()) == 1:
        return 1
    if L.krep_b200_regex_match_mode(params.ref()) == 1:
        return 2
    return 0


def twin_keys(params, sh, mode):
    """Keys (and the count mode's device lines) a scan of sh may emit, from the model: filter mode flags every line it
    cannot see to its end; match mode leaves every line that could reach the step budget to glibc whole."""
    if mode == 0:
        exp = km.expect(sh, 0, km.HookLines(params, sh.buf).flagged)
        return sorted(set(exp.keys) | exp.optional), 0
    exp = km.expect(sh, mode, km.GlibcLines(params, sh.buf))
    if mode == 1:
        return exp.keys, exp.device_lines
    return sorted(exp.keys + list(exp.prefix_lines)), 0


def build_row(sh, mode, keys, device_lines=0):
    """The row of shard sh (a regex_kernel_model.Shard) whose scan emitted `keys` in `mode`."""
    shift = km.REGEX_MATCH_SHIFT if mode == 2 else km.LIT_TAG_BITS
    G, buf, avail = sh.global_offset, sh.buf, sh.avail
    own_end = min(sh.own_end, avail)
    segs = []
    for k in keys:
        if mode == 2 and k & 1:
            continue
        p = (k >> shift) - G
        nl = buf.find(b"\n", p)
        e = nl + 1 if nl >= 0 else avail
        if segs and segs[-1][1] == p:
            segs[-1][1] = e
        else:
            segs.append([p, e])
    before = sh.prev_byte if sh.own_begin == 0 else buf[sh.own_begin - 1]
    flags, head = 0, b""
    if before >= 0 and before != 10:
        nl = buf.find(b"\n", sh.own_begin, own_end)
        head = buf[sh.own_begin:nl + 1 if nl >= 0 else own_end]
        flags |= ROW_HEAD
    if sh.next_byte < 0 and own_end >= avail:
        flags |= ROW_LAST | ((buf[avail - 1] if avail else 0) << 8)
    open_end = sh.next_byte >= 0 and avail and buf[avail - 1] != 10
    tab = b"".join(struct.pack("<2Q", G + b, ((e - b) << 1) | (1 if open_end and e == avail else 0)) for b, e in segs)
    fixed = HEADER + r16(8 * len(keys) + len(tab))
    data = pad16(head) + b"".join(pad16(buf[b:e]) for b, e in segs)
    hdr = struct.pack("<16Q", MAGIC, mode, fixed + len(data), device_lines, len(keys), len(segs), len(head), flags,
                      G + sh.own_begin, G + own_end, G + avail, 0, 0, 0, 0, 0)
    body = struct.pack("<%dQ" % len(keys), *keys) + tab
    return hdr + body + b"\0" * (fixed - HEADER - len(body)) + data


def twin_row(params, sh):
    mode = call_mode(params)
    keys, dl = twin_keys(params, sh, mode)
    return build_row(sh, mode, keys, dl)


def parse_row(row):
    """-> dict(header fields, keys, segs=[(start, len, cont, bytes)], head)"""
    h = struct.unpack_from("<16Q", row, 0)
    out = dict(magic=h[0], mode=h[1], row_bytes=h[2], device_lines=h[3], nkeys=h[4], nseg=h[5], head_len=h[6], flags=h[7],
               own_begin=h[8], own_end=h[9], avail_end=h[10])
    nk, ns = h[4], h[5]
    out["keys"] = list(struct.unpack_from("<%dQ" % nk, row, HEADER))
    tab = struct.unpack_from("<%dQ" % (2 * ns), row, HEADER + 8 * nk)
    p = HEADER + r16(8 * nk + 16 * ns)
    out["head"] = bytes(row[p:p + h[6]])
    p += r16(h[6])
    segs = []
    for i in range(ns):
        start, lc = tab[2 * i], tab[2 * i + 1]
        ln = lc >> 1
        segs.append((start, ln, lc & 1, bytes(row[p:p + ln])))
        p += r16(ln)
    out["segs"] = segs
    return out


def tile(text, cuts, halo):
    """Shards over text cut at `cuts` with a readable halo of `halo` bytes past each owned range: d_text at each cut
    rounded down to 16 (own_begin the remainder). -> [regex_kernel_model.Shard]"""
    n = len(text)
    bounds = [0] + sorted(cuts) + [n]
    out = []
    for b, e in zip(bounds, bounds[1:]):
        d = b & ~15
        end = min(n, e + halo)
        out.append(km.Shard(text[d:end], b - d, e - d, d, text[d - 1] if d else -1, text[end] if end < n else -1))
    return out
