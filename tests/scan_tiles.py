"""Texts that put literal and pattern-set occurrences on every lane and tile edge of the scan kernels' streaming loops.

Pure numpy, deterministic seeds.  tests/test_gpu_scan_tiles.py scans them on the GPU and holds every key to
tests/scan_model.py; tests/test_scan_tiles_layout.py checks without a GPU that the texts reach what that file claims.

Tile geometry of the kernels (a change to a kernel's tile must change these constants; the layout test then shows
whether the texts still reach every edge):

* k_lit_aligned4 / k_lit_window4 (csrc/scan_literal.cu: launch_literal, UNROLL = 4, 256 threads): vector u of thread t
  is group g0 + 256u + t, so a warp reads 512 contiguous bytes, a CTA tile is 16 KiB and the grid stride is
  grid x 16 KiB with grid = min(tiles, SMs x occupancy).
* k_ac_scan (csrc/scan_multi.cu: launch_ac, THREADS = 640, UNROLL = 4): the same layout with 640 threads, a 40 KiB
  tile; grid = min(tiles, SMs).
* k_ac_tri4 (csrc/scan_multi.cu: k_ac_tri4, TILE = THREADS * 4): warp w owns groups [128w, 128w + 128) of a tile and
  vector u of lane l is group 128w + 32u + l; 640 threads (40 KiB tile) by default, 768 (48 KiB) under
  KREP_B200_AC_THREADS=768; grid = min(tiles, SMs).

Every grid-stride edge, for any occupancy from 1 to 8, is a multiple k x SMs x tile (k = 1..8): the builders plant there.
"""
import random

import numpy as np

import scan_model as sm
from test_gpu_scan_keys import FULL_BYTE_ALPHABETS, KINDS, cased, is_letter, partner

VEC = 16                        # bytes per lane vector (one LDG.128)
WARP_VEC = 32 * VEC             # 512: one warp-wide vector load, contiguous in every kernel here
LIT_TILE = 256 * 4 * VEC        # 16 KiB: k_lit_aligned4 / k_lit_window4
AC_TILE = 640 * 4 * VEC         # 40 KiB: k_ac_scan, and k_ac_tri4 at its default 640 threads
TRI4_768_TILE = 768 * 4 * VEC   # 48 KiB: k_ac_tri4 under KREP_B200_AC_THREADS=768
TRI4_WARP_TILE = 128 * VEC      # 2 KiB: a k_ac_tri4 warp's share of a tile
TILES = {"lit": LIT_TILE, "ac": AC_TILE, "tri768": TRI4_768_TILE}
MAX_OCCUPANCY = 8
AC_TAIL = 24                    # a pattern-set group needs 24 readable bytes (tri4: its next word, 20)
H100_SMS = 132                  # H100 SXM; the GPU tests read the device's count
TEXT_LEN = 19 * (1 << 20) + 4567  # > 8 x SMs x 16 KiB and > 3 x SMs x 40 KiB; not near a multiple of any tile
CONTEXT_BYTES = b"a_0Z \n\x00\xe9\xff@"  # word, non-word, NUL and high bytes around planted occurrences (-w tags)
NON_WORD = CONTEXT_BYTES[4:]


def kind_case(kind, seed):
    """(func, patterns, cs, ww, only_matching) of a KINDS entry, as test_gpu_scan_keys.make_plan draws it."""
    _, func, mk, cs, ww, o = kind
    rng = random.Random(seed)
    pats = mk(rng)
    if func == "aho_corasick" and rng.random() < 0.5:
        pats = pats + [pats[0]]
    return func, (pats if func == "aho_corasick" else pats[:1]), cs, ww, o


def periodic(length, ww, period):
    """A self-overlapping needle: every byte offset of a run of it (period 1) or every other one (period 2) starts an
    occurrence.  Under -w its bytes are non-word bytes, so the occurrences inside a run keep both word-boundary bits."""
    base = (b"@", b"@\xe9")[period - 1] if ww else (b"a", b"ab")[period - 1]
    return (base * length)[:length]


def dense_case(kind):
    """The KINDS entry with each pattern replaced by a periodic needle of the same length: the same kernel (its choice
    depends on the lengths and flags only), now with occurrences at nearly every offset of a run."""
    func, pats, cs, ww, o = kind_case(kind, 7)
    period = 1 + KINDS.index(kind) % 2
    return func, [periodic(len(p), ww, period) if p else b"" for p in pats], cs, ww, o


# dense-only cases: long periodic needles for boyer_moore (k_lit_aligned4 verifies 64 and 1024 bytes at every offset)
DENSE_EXTRA = [("bm-64", ("boyer_moore", [b"ab" * 32], True, False, False)),
               ("bm-1024-fold", ("boyer_moore", [b"aB" * 512], False, False, False))]


def _noise(nrng, n, pats):
    """Background bytes: uniform for needles of 1..3 bytes (which a small alphabet would match everywhere), else one of
    the alias alphabets of test_scan_model (every byte the -i word fold confuses with a pattern byte)."""
    lmin = min(len(p) for p in pats if p)
    alpha = FULL_BYTE_ALPHABETS[0 if lmin <= 3 else 1 + int(nrng.integers(0, 4))]
    return np.frombuffer(alpha, np.uint8)[nrng.integers(0, len(alpha), n)]


def _near_miss(rng, p, cs, i):
    """p with byte i swapped for its fold alias or bit-7 partner; under -i a letter takes its bit-7 partner (its other
    case would still match)."""
    b = bytearray(p)
    b[i] = b[i] ^ 0x80 if (not cs and is_letter(b[i])) else partner(rng, b[i])
    return bytes(b)


def _put(t, pos, data, rng, ctx=CONTEXT_BYTES):
    t[pos:pos + len(data)] = np.frombuffer(data, np.uint8)
    if ctx:
        if pos > 0:
            t[pos - 1] = rng.choice(ctx)
        if pos + len(data) < t.size:
            t[pos + len(data)] = rng.choice(ctx)


def sweep_offset(j):
    """Offset inside warp vector j of the occurrence planted there.  Round q = j // 512 walks all 512 (lane, residue)
    pairs once (129 is odd; neighbouring vectors' offsets lie 129 apart, so items never touch), shifted by 7q, so
    across 32 rounds every pair also lands in every warp vector of a 16 KiB tile (129 = 1 mod 32): lane 31 with
    residues 13..15 reaches into the next warp, the next vector row of the same thread and the next CTA tile."""
    return (129 * j + 7 * (j // 512)) % WARP_VEC


def lane_sweep(pats, cs, n, seed):
    """-> (text, near-miss starts).  Noise with one occurrence per 512-byte warp vector at sweep_offset(j), and a near
    miss (one byte swapped, at every position of the pattern in turn) 256 bytes further on; context bytes around both.
    Items that would overlap the previous one are left out."""
    rng = random.Random(seed)
    nrng = np.random.default_rng(seed)
    live = [p for p in pats if p]
    t = _noise(nrng, n, live)
    items = []
    for j in range(n // WARP_VEC):
        o = sweep_offset(j)
        p = live[j % len(live)]
        ctx = CONTEXT_BYTES if j % 3 == 0 else NON_WORD  # under -w drop mode two in three occurrences keep their key
        items.append((j * WARP_VEC + o, cased(rng, p, cs), False, ctx))
        items.append((j * WARP_VEC + (o + 256) % WARP_VEC, _near_miss(rng, p, cs, (j // 2) % len(p)), True, ctx))
    items.sort(key=lambda x: x[0])
    misses, end = [], 0
    for pos, data, miss, ctx in items:
        if pos - 1 <= end or pos + len(data) + 1 > n:
            continue
        _put(t, pos, data, rng, ctx)
        end = pos + len(data)
        if miss:
            misses.append(pos)
    _put(t, n - len(live[0]), live[0], rng, ctx=b"")  # one ends on the last byte
    return t.tobytes(), np.array(misses, dtype=np.int64)


def named_edges(n, sms):
    """{name: byte offset} of the edges the dense runs straddle: group 0, CTA-tile edges, grid-stride edges
    k x SMs x tile (k = 1..8), the start of the ragged tile of every tile size, and the end of the text."""
    e = {"group0": 0, "end": n}
    for name, tile in TILES.items():
        for k in (1, 2, 3):
            e[f"{name}-tile{k}"] = k * tile
        for k in range(1, MAX_OCCUPANCY + 1):
            if k * sms * tile < n - 8192:
                e[f"{name}-stride{k}"] = k * sms * tile
        e[f"{name}-ragged"] = (n - AC_TAIL) // tile * tile
    return e


def ac_full_tile(sms):
    """(tile, carried-from tile) of the k_ac_scan CTA tile dense_blocks fills for pattern sets.  Tile sms + 5 is the
    second tile of CTA 5 (grid = SMs), so its warps come to it with the candidates their first tile, tile 5, left
    queued."""
    return sms + 5, 5


def _ac_scan_group(tile, warp, u, lane):
    """Group index of vector u of lane `lane` in warp `warp` of k_ac_scan CTA tile `tile` (640 threads x 4 vectors)."""
    return tile * (AC_TILE // VEC) + 640 * u + 32 * warp + lane


def dense_blocks(pats, cs, n, sms, seed, is_set=False):
    """-> (text, edges).  Sparse noise (an occurrence of the shortest needle every 256..1280 bytes, so queues carry
    entries across tiles) and a run of back-to-back needles around every named edge: 8 KiB at group 0 and at the end,
    2..8 KiB elsewhere (2..3.5 KiB for pattern sets, whose needles all match at every offset of a run).  One warp
    vector emits up to 512 keys and k_ac_tri4's queue fills in one push.

    For pattern sets also one whole k_ac_scan CTA tile (ac_full_tile) with an occurrence at the start of every 16-byte
    group, so all four vectors of every lane park in one iteration: 128 entries per warp on top of the 5 each warp
    carries over from its previous tile, where 5 of its groups hold one.  That is what AcQueue::CAP (a remainder of
    up to 31 plus one full iteration) is sized for.

    Newlines stay in the noise only, so no newline-free stretch reaches 64 KiB (k_line_bounds searches the whole line
    around every set key)."""
    rng = random.Random(seed)
    nrng = np.random.default_rng(seed)
    live = [p for p in pats if p]
    t = _noise(nrng, n, live)
    short = min(live, key=len)
    pos = 0
    while pos < n - 2048 - len(short):
        pos += len(short) + rng.randint(256, 1280)
        _put(t, pos, cased(rng, short, cs), rng)
    if is_set:
        full, carried = ac_full_tile(sms)
        groups = [_ac_scan_group(carried, w, u, 7 * u + 3) for w in range(AC_TILE // WARP_VEC // 4) for u in range(4)]
        groups += [_ac_scan_group(carried, w, 0, 29) for w in range(AC_TILE // WARP_VEC // 4)]
        groups += list(range(full * (AC_TILE // VEC), (full + 1) * (AC_TILE // VEC)))
        for g in groups:
            _put(t, 16 * g, cased(rng, short, cs), rng, NON_WORD)
    unit = short[:1] if len(set(short)) == 1 else short[:2]  # the needles' period
    edges = named_edges(n, sms)
    for name, e in edges.items():
        half = 4096 if name in ("group0", "end") else rng.randint(1024, 1792 if is_set else 4096)
        lo, hi = max(0, e - half), min(n, e + half)
        run = (unit * ((hi - lo) // len(unit) + 1))[:hi - lo]
        t[lo:hi] = np.frombuffer(cased(rng, run, cs), np.uint8)
        if 0 < lo:
            t[lo - 1] = rng.choice(CONTEXT_BYTES)
    return t.tobytes(), edges


def text_for(builder, pats, cs, n, sms, seed, is_set=False):
    if builder == "sweep":
        return lane_sweep(pats, cs, n, seed)[0]
    return dense_blocks(pats, cs, n, sms, seed, is_set)[0]


def where(name, start, group_begin=0, sms=H100_SMS, tri4_tile=AC_TILE):
    """Where a key's start falls in the streaming loop of the kernel `name` (a plan's filter name) runs."""
    rel = start - 16 * group_begin
    if "/" not in name:  # the literal filters: aligned4, window4 and their -fold forms
        kern, tile = "k_lit", LIT_TILE
    elif "tri4" in name or "aligned-word" in name:
        kern, tile = "k_ac_tri4", tri4_tile
    else:
        kern, tile = "k_ac_scan", AC_TILE
    o = rel % tile
    if kern == "k_ac_tri4":
        warp, u = o // TRI4_WARP_TILE, o % TRI4_WARP_TILE // WARP_VEC
    else:
        row = tile // 4  # one vector per thread of the CTA
        u, warp = o // row, o % row // WARP_VEC
    return (f"{kern} ({name}): start {start} = lane {o % WARP_VEC // VEC}, residue {o % VEC}, warp {warp}, vector row {u},"
            f" CTA tile {rel // tile} (+{o}), {rel / (sms * tile):.3f} x SMs x tile (grid-stride edges at whole numbers)")


def model_keys(case, buf, avail, ob, oe, go=0, prev=-1, nxt=-1):
    func, pats, cs, ww, o = case
    return sm.shard_keys(sm.plan_shape(func, pats, cs, ww, o), pats, cs, buf, avail, ob, oe, go, prev, nxt, ww)
