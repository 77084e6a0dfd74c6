"""The texts of tests/test_gpu_scan_tiles.py reach what that file claims (no GPU: the builders and scan_model only).

Each text is built as the GPU file builds it, its keys come from scan_model, and the coverage is counted against the
tile geometry in tests/scan_tiles.py: every (lane, residue) pair of a warp vector holds a key and a near miss in the
main-loop region, every named edge has keys on both sides, a warp vector holds >= 256 keys, a k_ac_tri4 warp tile has
all 128 groups occupied, a k_ac_scan warp parks all 128 of its groups in one iteration with entries left over from its
previous tile, and a group holds keys of two patterns at different distances from its aligned words."""
import numpy as np
import pytest

import scan_model as sm
import scan_tiles as st
from test_gpu_scan_keys import KIND_IDS, KINDS

N = st.TEXT_LEN
SMS = st.H100_SMS
MAIN_END = min((N - st.AC_TAIL) // t * t for t in st.TILES.values())  # below this every kernel is in its main loop


def starts_of(case, buf):
    keys = st.model_keys(case, buf, N, 0, N)
    return keys, sm.key_starts(keys, case[0] == "aho_corasick").astype(np.int64)


def pairs(starts):
    """Set of (lane, residue) pairs, as lane * 16 + residue, of starts in the main-loop region past warp vector 0."""
    s = starts[(starts >= st.WARP_VEC) & (starts < MAIN_END)]
    return set(np.unique(s % st.WARP_VEC).tolist())


@pytest.mark.parametrize("kind", KINDS, ids=KIND_IDS)
def test_lane_sweep_covers_every_lane_and_residue(kind):
    case = st.kind_case(kind, 11)
    buf, misses = st.lane_sweep(case[1], case[2], N, 1 + KINDS.index(kind))
    keys, starts = starts_of(case, buf)
    assert pairs(starts) == set(range(st.WARP_VEC)), sorted(set(range(st.WARP_VEC)) - pairs(starts))[:8]
    missed = misses[~np.isin(misses, starts)]
    assert pairs(missed) == set(range(st.WARP_VEC)), sorted(set(range(st.WARP_VEC)) - pairs(missed))[:8]
    # lane 31's last residues reach into the next warp, the next vector row and the next 16 KiB tile
    last = starts[(starts % st.WARP_VEC >= 31 * 16 + 13) & (starts < MAIN_END)]
    chunk_in_tile = set((last % st.LIT_TILE // st.WARP_VEC).tolist())
    assert chunk_in_tile == set(range(st.LIT_TILE // st.WARP_VEC)), sorted(chunk_in_tile)
    assert sm.PACK_KEYS < keys.size < 6 * 10 ** 5


DENSE = [(st.dense_case(k), 1 + KINDS.index(k)) for k in KINDS] + [(c, 77) for _, c in st.DENSE_EXTRA]


@pytest.mark.parametrize("case,seed", DENSE, ids=KIND_IDS + [i for i, _ in st.DENSE_EXTRA])
def test_dense_blocks_straddle_every_named_edge(case, seed):
    is_set = case[0] == "aho_corasick"
    buf, edges = st.dense_blocks(case[1], case[2], N, SMS, seed, is_set)
    keys, starts = starts_of(case, buf)
    assert 3 * sm.PACK_KEYS <= keys.size <= 1 << 19, keys.size  # well past CUB's threshold, half the 2^20-key list
    for k in range(1, st.MAX_OCCUPANCY + 1):
        assert f"lit-stride{k}" in edges
    for name, e in edges.items():
        if name == "group0":
            assert (starts < 16).any(), name
        elif name == "end":
            lens = np.array([len(p) for p in case[1] if p])
            assert (starts + lens.min() > N - st.AC_TAIL).any(), name
        else:
            assert ((starts >= e - 64) & (starts < e)).any() and ((starts >= e) & (starts < e + 64)).any(), (name, e)
    per_vec = np.bincount(starts // st.WARP_VEC)
    assert per_vec.max() >= 256, per_vec.max()
    if is_set:
        pattern = (keys & np.uint64(sm.AC_MAX_PATTERNS - 1)).astype(np.int64)
        a = (starts + 3) // 4 * 4                   # the aligned word a lookup finds the start by: p = a - d
        d, group = a - starts, a // 16
        if min(len(p) for p in case[1] if p) >= 6:  # k_ac_tri4: a warp tile with all 128 groups occupied
            occupied = np.bincount(np.unique(group) // 128)
            assert occupied.max() == 128, occupied.max()
        # k_ac_scan: a warp whose four vectors all park in one iteration (128 queue entries), after a tile of the same
        # CTA (SMs tiles earlier) that left it a remainder
        g = np.unique(starts // st.VEC)
        tile_groups = st.AC_TILE // st.VEC
        tile, o = g // tile_groups, g % tile_groups
        warps = tile_groups // 4 // 32  # 640 threads: 20 warps, a row of 640 groups per vector
        warp_id = tile * warps + o % (tile_groups // 4) // 32
        per_warp = np.bincount(warp_id)
        full = np.flatnonzero(per_warp == 128)
        carried = full - warps * SMS
        carried = carried[carried >= 0]
        assert carried.size and (per_warp[carried] > 0).all(), (full[:8], per_warp[carried][:8])
        assert (per_warp[carried] >= 5).all(), per_warp[carried][:8]
        # one group holding keys of >= 2 patterns at different d: several passed lookups, the re-push path
        g2 = np.unique(np.stack([group, pattern, d]), axis=1)
        ok = False
        for g in np.unique(g2[0][np.flatnonzero(np.diff(g2[0]) == 0)])[:64]:
            sel = g2[:, g2[0] == g]
            ok |= np.unique(sel[1]).size >= 2 and np.unique(sel[2]).size >= 2
        assert ok


def test_where_names_the_edge():
    """The failure message's decoding of a start: a lane-31 start at residue 13 of the last vector of a literal tile."""
    s = st.LIT_TILE - 3
    w = st.where("window4-fold", s)
    assert "lane 31, residue 13, warp 7, vector row 3, CTA tile 0" in w, w
    w = st.where("window3/stride4 tri4+byte-select fold", st.AC_TILE + 2048 + 512 + 17)
    assert "k_ac_tri4" in w and "lane 1, residue 1, warp 1, vector row 1, CTA tile 1" in w, w
    w = st.where("window4/stride2 paired", 2 * SMS * st.AC_TILE)
    assert "k_ac_scan" in w and "2.000 x SMs x tile" in w, w
