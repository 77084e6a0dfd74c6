"""Multi-GPU plumbing for the scan path (one process per GPU): shard geometry and the single gather of per-shard
counts + occurrence keys to rank 0, followed by the key merge.

This is the analogue of krep's chunker + merge (krep.c:2816-2905, 2928-3004) with two differences that make
the result equal to the reference's single-chunk run instead of its multi-thread artefacts (SURVEY §8 a12):
a match belongs to the shard that contains its START, and -w context bytes come from the neighbouring shards.

Order of the gathered lists.  Literal keys are ordered AND owned by start offset, so the per-rank lists concatenate
into a globally ascending list.  Pattern-set keys are ordered by END offset (aho_corasick_search's emission order,
aho_corasick.c:353-431) but still owned by start offset: a long match that starts just before a cut belongs to the
earlier rank yet ends after a short match owned by the later rank.  Rank 0 therefore always MERGES the per-rank lists
by key (krep_b200_merge_keys, C); the disorder is confined to max_pattern_len bytes around each cut, so the merge is
one linear pass per cut.

Works on any torch.distributed backend (nccl on the GPUs, gloo in the CPU tests).

-E plans take another exchange (regex_resolve_ranks, RegexRanks; DESIGN §12.6): each rank resolves the lines its own
shard owns from its own row, and only counts and positions travel to rank 0.
"""
import ctypes as C

import torch
import torch.distributed as dist

from . import lib


def shard_bounds(total_len, world, rank, halo, align=16):
    """-> (begin, own_len, avail_len): the shard owns [begin, begin+own_len) and can read avail_len bytes from begin.

    own ranges tile [0, total_len) exactly; every shard but the last reads `halo` bytes past its owned range
    (longest pattern + 1, so an occurrence starting on the last owned byte and the byte after it are visible)."""
    per = -(-total_len // world)
    per = -(-per // align) * align
    begin = min(rank * per, total_len)
    end = min(begin + per, total_len)
    avail_end = min(end + halo, total_len)
    return begin, end - begin, avail_end - begin


def merge_rows(rows, counts, out=None):
    """rows: 2-D int64 CPU tensor, row r = [count_r, key_0 .. ] (contiguous); counts: list of valid keys per row.
    -> 1-D int64 tensor with all keys in ascending key order (krep_b200_merge_keys)."""
    L = lib.load()
    world = rows.shape[0]
    total = int(sum(counts))
    if out is None or out.numel() < max(total, 1):
        out = torch.empty(max(total, 1), dtype=torch.int64)
    stride = rows.stride(0) * 8
    base = rows.data_ptr()
    lists = (C.c_void_p * world)(*[base + r * stride + 8 for r in range(world)])
    cnts = (C.c_uint64 * world)(*[int(c) for c in counts])
    n = L.krep_b200_merge_keys(lists, cnts, world, C.c_void_p(out.data_ptr()))
    assert n == total
    return out[:total]


def gather_keys(local_keys, world, rank, device):
    """One all_gather of per-rank counts + one gather of the (padded) sorted key lists to rank 0, merged by key.

    local_keys: 1-D int64 tensor on `device` (sorted, global offsets).  Returns the merged, globally ascending key
    tensor on rank 0 (CPU), None elsewhere, plus the list of per-rank counts."""
    cnt = torch.tensor([local_keys.numel()], dtype=torch.int64, device=device)
    counts = [torch.zeros_like(cnt) for _ in range(world)]
    dist.all_gather(counts, cnt)
    counts = [int(c.item()) for c in counts]
    mx = max(max(counts), 1)
    mine = torch.zeros(mx + 1, dtype=torch.int64, device=device)
    mine[0] = local_keys.numel()
    mine[1: 1 + local_keys.numel()] = local_keys
    gathered = [torch.empty_like(mine) for _ in range(world)] if rank == 0 else None
    dist.gather(mine, gathered, dst=0)
    if rank != 0:
        return None, counts
    rows = torch.stack([g.cpu() for g in gathered]).contiguous()
    return merge_rows(rows, counts).clone(), counts


class KeyGatherer:
    """The same exchange with persistent buffers and ONE collective per step, for a steady state of many steps.

    Every rank owns a fixed-capacity row [count, key_0 .. key_{cap-1}] on its device (krep_b200_export_packed fills it
    in one device-to-device copy); post() gathers the rows to rank 0 — a gather, not an all_gather: ranks other than 0
    only send, so nothing on their GPUs waits for rank 0 — and rank 0 starts an asynchronous copy of the gathered rows
    into one of two pinned host buffers.  fetch() (rank 0) waits for that copy and merges the rows by key.  The two
    host buffers let rank 0 post step i+1 (and run its scan) before it fetches and replays step i.

    Capacity: negotiate() is the checked form used while warming up — every rank learns the largest count through a
    MAX all_reduce and all ranks grow their buffers in lockstep when it does not fit.  In the unchecked steady state a
    row that does not fit is truncated but still carries its exact count, so rank 0 notices; it does not raise in the
    middle of the run (the other ranks would hang in the next collective) but sets `overflowed`, which the caller
    turns into a collective error after the loop."""

    def __init__(self, world, rank, device, capacity=1 << 14):
        self.world, self.rank, self.device = world, rank, device
        self.overflowed = False
        self._alloc(capacity)

    def _alloc(self, capacity):
        self.cap = int(capacity)
        pin = self.device != "cpu" and torch.cuda.is_available()
        self.row = torch.zeros(self.cap + 1, dtype=torch.int64, device=self.device)
        if self.rank == 0:
            self.rows = torch.zeros((self.world, self.cap + 1), dtype=torch.int64, device=self.device)
            self.host = [torch.zeros((self.world, self.cap + 1), dtype=torch.int64, pin_memory=pin) for _ in range(2)]
            self.merged = torch.empty(self.world * self.cap + 1, dtype=torch.int64)
            self.events = [torch.cuda.Event() if pin else None for _ in range(2)]
        self._mx = torch.zeros(1, dtype=torch.int64, device=self.device)

    def row_ptr(self):
        """Device pointer of this rank's row (what krep_b200_export_packed writes: count + up to `cap` keys)."""
        return self.row.data_ptr()

    def negotiate(self, count):
        """Checked form: True if every rank's count fits, else grows the buffers on all ranks and returns False."""
        self._mx[0] = int(count)
        dist.all_reduce(self._mx, op=dist.ReduceOp.MAX)
        mx = int(self._mx.item())
        if mx <= self.cap:
            return True
        cap = self.cap
        while cap < mx:
            cap *= 2
        self._alloc(cap * 2)
        return False

    def post(self, slot=0):
        """Gather the rows to rank 0; rank 0 also starts the device-to-host copy into host buffer `slot`."""
        if self.rank == 0:
            dist.gather(self.row, list(self.rows.unbind(0)), dst=0)
            self.host[slot].copy_(self.rows, non_blocking=True)
            if self.events[slot] is not None:
                self.events[slot].record()
        else:
            dist.gather(self.row, None, dst=0)

    def fetch(self, slot=0):
        """Rank 0: -> (merged keys as a 1-D int64 CPU tensor, per-rank counts)."""
        assert self.rank == 0
        if self.events[slot] is not None:
            self.events[slot].synchronize()
        rows = self.host[slot]
        counts = [int(c) for c in rows[:, 0].tolist()]
        if max(counts) > self.cap:
            self.overflowed = True
            counts = [min(c, self.cap) for c in counts]
        return merge_rows(rows, counts, self.merged), counts


# ---- -E over rank-resident shards (DESIGN §12.6) ----

def _result_positions(res):
    """The positions of a match_result_t as an int64 [k, 2] CPU tensor (one copy, no per-position Python)."""
    import numpy as np
    r = res.contents
    if r.count == 0:
        return torch.zeros((0, 2), dtype=torch.int64)
    flat = np.ctypeslib.as_array(C.cast(r.positions, C.POINTER(C.c_uint64)), shape=(2 * r.count,))
    return torch.from_numpy(flat.astype(np.int64)).view(-1, 2)


def regex_resolve_ranks(params, row, rank, world, device="cpu", group=None, times=None):
    """One -E answer from rows spread over the ranks: every rank passes its own shard's row and resolves the lines that
    shard owns; only counts and positions travel to rank 0.

    row: this rank's row (krep_b200_regex_export_shard) in a uint8 CPU tensor (it may be longer than the row).  The
    shards of ranks 0 .. world-1 must tile one text in rank order.  device: where the collectives' tensors live — "cpu"
    for gloo, the rank's CUDA device for NCCL.  times (a dict, optional) receives exchange_ms and resolve_ms.
    Returns (count, positions as an int64 [k, 2] tensor in the reference's order) on rank 0, None elsewhere.

      1. one all_gather of the 128-byte row headers: from them every rank knows the tiling, the text's last byte, which
         rank decides the end of the text, and which heads it receives (krep_b200_regex_tiling).  A tiling error is
         raised on every rank alike, before any further collective, so none is left waiting;
      2. every shard that starts mid-line sends its head-only row (krep_b200_regex_row_head) to the rank that owns the
         line it continues, point to point (the sizes are known from the headers);
      3. every rank resolves its part (krep_b200_regex_resolve_part) with the full -m budget;
      4. one all_gather of (count, positions), then the positions are gathered to rank 0, which concatenates them in
         rank order and cuts them to max_count: each part's answer is the first max_count items of its own unbounded
         answer, so this is the whole answer."""
    import time
    L = lib.load()
    t0 = time.perf_counter()
    hb = lib.REGEX_ROW_HEADER
    mine = row[:hb].to(device)
    heads = [torch.empty_like(mine) for _ in range(world)]
    dist.all_gather(heads, mine, group=group)
    headers = torch.cat([h.cpu() for h in heads]).contiguous()
    tiling, head_to, head_bytes = lib.regex_tiling(headers.data_ptr(), world)
    ops, recv = [], []
    if head_to[rank] >= 0:
        out = torch.empty(head_bytes[rank], dtype=torch.uint8)
        n = L.krep_b200_regex_row_head(C.c_void_p(row.data_ptr()), C.c_void_p(out.data_ptr()), out.numel())
        lib.check(L)
        assert n == out.numel(), (n, out.numel())
        ops.append(dist.isend(out.to(device), head_to[rank], group=group))
    for j in range(world):
        if head_to[j] == rank:
            buf = torch.empty(head_bytes[j], dtype=torch.uint8, device=device)
            recv.append(buf)
            ops.append(dist.irecv(buf, j, group=group))
    for op in ops:
        op.wait()
    rows = [row] + [b.cpu() for b in recv]  # the heads of the shards after this one, in text order
    t1 = time.perf_counter()
    arr = (C.c_void_p * len(rows))(*[r.data_ptr() for r in rows])
    res = L.krep_b200_match_result_init(16)
    try:
        cnt = L.krep_b200_regex_resolve_part(params.ref(), arr, len(rows), 1, tiling.text_len, tiling.last_byte,
                                             int(tiling.decider == rank), res)
        err = L.krep_b200_last_error()
        msg = L.krep_b200_last_error_string().decode() if err else ""
        pos = _result_positions(res)
    finally:
        L.krep_b200_match_result_free(res)
    t2 = time.perf_counter()
    # an error of one part travels with the counts, so every rank raises it and none waits in the gather below
    meta = torch.tensor([int(cnt), pos.shape[0], err], dtype=torch.int64, device=device)
    metas = [torch.empty_like(meta) for _ in range(world)]
    dist.all_gather(metas, meta, group=group)
    metas = torch.stack([m.cpu() for m in metas])
    bad = [r for r in range(world) if metas[r, 2] != 0]
    if bad:
        raise RuntimeError(f"krep_b200_regex_resolve_part failed on rank(s) {bad}" + (f": {msg}" if msg else ""))
    counts, npos = metas[:, 0].tolist(), metas[:, 1].tolist()
    mx = max(npos)
    parts = [pos]
    if mx:
        padded = torch.zeros((mx, 2), dtype=torch.int64, device=device)
        padded[:pos.shape[0]] = pos.to(device)
        got = [torch.empty_like(padded) for _ in range(world)] if rank == 0 else None
        dist.gather(padded, got, dst=0, group=group)
        if rank == 0:
            parts = [g[:k].cpu() for g, k in zip(got, npos)]
    t3 = time.perf_counter()
    if times is not None:
        times["exchange_ms"] = ((t1 - t0) + (t3 - t2)) * 1e3
        times["resolve_ms"] = (t2 - t1) * 1e3
    if rank != 0:
        return None
    max_count = int(params.struct.max_count)
    return min(sum(counts), max_count), torch.cat(parts)[:max_count]


class RegexRanks:
    """-E search of this rank's resident shard as one part of a text tiled across the ranks: the export into a
    persistent host buffer (grown when a row does not fit), then regex_resolve_ranks.  The row, the heads and the
    answers live on the host, so a gloo group is the natural transport; bench_regex_ranks.py uses one.  NCCL works too
    (device = the rank's GPU): every message is then staged through it."""

    def __init__(self, rank, world, device="cpu", group=None, capacity=1 << 20):
        self.rank, self.world, self.device, self.group = rank, world, device, group
        self.row = torch.empty(capacity, dtype=torch.uint8, pin_memory=torch.cuda.is_available())
        self.times = {}

    def export(self, plan, params, shard):
        """This rank's row into self.row; -> its size in bytes."""
        import time
        L = lib.load()
        t0 = time.perf_counter()
        nb = C.c_uint64(0)
        rc = L.krep_b200_regex_export_shard(plan, params.ref(), C.byref(shard), None, C.c_void_p(self.row.data_ptr()),
                                            self.row.numel(), C.byref(nb), None)
        if rc == -5:  # the row needs more room: grow and export again
            L.krep_b200_last_error()
            self.row = torch.empty(nb.value + nb.value // 4, dtype=torch.uint8, pin_memory=torch.cuda.is_available())
            rc = L.krep_b200_regex_export_shard(plan, params.ref(), C.byref(shard), None, C.c_void_p(self.row.data_ptr()),
                                                self.row.numel(), C.byref(nb), None)
        if rc != 0:
            raise RuntimeError("krep_b200: " + L.krep_b200_last_error_string().decode())
        self.times["export_ms"] = (time.perf_counter() - t0) * 1e3
        return nb.value

    def search(self, plan, params, shard):
        """-> (count, int64 [k, 2] positions) on rank 0, None elsewhere.

        Every rank must call it with the same plan and params.  An export that fails on one rank (a refused pattern, a
        CUDA error) still takes part in the exchange with a header no tiling accepts, so every rank raises."""
        try:
            self.export(plan, params, shard)
        except RuntimeError:
            self.row[:lib.REGEX_ROW_HEADER].zero_()
            try:
                regex_resolve_ranks(params, self.row, self.rank, self.world, self.device, self.group)
            except RuntimeError:
                pass
            raise
        return regex_resolve_ranks(params, self.row, self.rank, self.world, self.device, self.group, self.times)
