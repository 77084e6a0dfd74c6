"""-E over rank-sharded rows, on the host: every part of a tiling resolved on its own (krep_b200_regex_resolve_part with
only the heads krep_b200_regex_tiling routes to it), the answers concatenated in text order and cut to max_count, must
equal the reference loop over glibc and krep_b200_regex_resolve on all rows — count, every position and their order.
Rows come from the host twin of the export (tests/regex_rows_util.py).  The exchange of krep_b200/sharding.py runs on
such rows at gloo world sizes 2 and 3."""
import os
import queue
import random
import socket
import time

import pytest
import torch

import regex_kernel_model as km
import regex_ranks_util as rk
import regex_rows_util as rr
import regex_util as ru
from krep_b200 import lib, sharding


def want_of(P, text):
    w = ru.ref_regex_search(P, text)
    return (w[0], w[1] if P.struct.track_positions else [])


def groups_of(n_rows, k):
    """k consecutive groups of rows (k <= n_rows) -> [(first, end)]"""
    b = [n_rows * i // k for i in range(k + 1)]
    return [(x, y) for x, y in zip(b, b[1:]) if y > x]


def check(P, text, cuts, halo, what=""):
    if ru.filter_host(P, text) is None:
        return
    rows = rk.tiling_rows(P, text, cuts, halo)
    want = want_of(P, text)
    # krep_b200_regex_resolve takes a tiling without the empty shards after the end of the text
    whole = [r for i, r in enumerate(rows) if i == 0 or rr.parse_row(rows[i - 1])["own_end"] < len(text)]
    assert lib.regex_resolve(P, whole) == want, what
    got = rk.parts_answer(P, rows, [(i, i + 1) for i in range(len(rows))])
    assert got == want, (what, P.patterns, cuts, halo, got[0], want[0], got[1][:6], want[1][:6])
    if len(rows) > 2:  # parts of several rows (n_own > 1)
        assert rk.parts_answer(P, rows, groups_of(len(rows), 2)) == want, (what, "two parts")


def _cuts(rng, text, k):
    n = len(text)
    return sorted(rng.sample(range(1, n), min(k - 1, n - 1))) if n >= 2 and k > 1 else []


@pytest.mark.parametrize("world", [1, 2, 3, 7])
@pytest.mark.parametrize("pat,opts", rk.PATTERNS)
def test_cut_kinds(world, pat, opts):
    for mode in rk.MODES:
        P = rk.params(pat, **opts, **mode)
        for name, text, cuts in rk.cut_texts(world):
            for halo in rk.HALOS:
                check(P, text, cuts, halo, what=(name, mode, halo))


def test_random_regexes_tilings():
    rng = random.Random(17)
    done = 0
    while done < 80:
        pat = ru.random_regex(rng)
        case = rng.choice(ru.CASES + [dict(max_count=7), dict(count=True, only_matching=True, max_count=2)])
        try:
            P = rk.params(pat, **case)
        except ValueError:
            continue
        if ru.filter_host(P, b"") is None:
            continue
        text = ru.random_text(rng, rng.randint(0, 700))
        if rng.random() < 0.5:
            text = text.rstrip(b"\n") + b"\n"
        check(P, text, _cuts(rng, text, rng.choice([1, 2, 3, 7])), rng.choice(rk.HALOS), what=(pat, case))
        done += 1


@pytest.mark.parametrize("tail", [b"", b"\n", b"\n\n", b"x", b"X\n"])
def test_end_of_text(tail):
    """The empty string at n is decided by one part only, whichever shard holds the last line start."""
    rng = random.Random(len(tail) + 3)
    text = b"ab\nxx\n\nthe x\n" * 40 + tail
    for pat, case in [("^$", dict()), ("^$", dict(count=True)), ("x*", dict()), ("x*", dict(count=True, only_matching=True)),
                      ("x$", dict(case_sensitive=False)), ("$", dict()), ("^", dict(count=True))]:
        P = rk.params(pat, **case)
        for k in (2, 3, 7):
            for halo in rk.HALOS:
                check(P, text, _cuts(rng, text, k), halo, what=(pat, case, k, halo))
                # every cut in the last 3 bytes: the last shards hold no line start
                n = len(text)
                check(P, text, sorted({max(1, n - 3), max(1, n - 2), max(1, n - 1)})[:k - 1], halo, what=(pat, case, "tail"))


def test_long_text_modes():
    rng = random.Random(5)
    text = km.random_lines_text(rng, 12000).replace(b"x", b"the", 100)
    for pat, opts in rk.PATTERNS:
        for mode in rk.MODES:
            P = rk.params(pat, **opts, **mode)
            for k in (2, 3, 7):
                check(P, text, _cuts(rng, text, k), rng.choice(rk.HALOS), what=(pat, mode, k))


def test_empty_text():
    for pat in ["^$", "a", "x*"]:
        for case in [dict(), dict(count=True)]:
            P = rk.params(pat, **case)
            rows = [rr.twin_row(P, km.Shard(b""))] * 3
            assert rk.parts_answer(P, rows, [(0, 1), (1, 2), (2, 3)]) == want_of(P, b""), (pat, case)


def test_tiling_routes_heads():
    P = rk.params("the")
    text = b"the a\nthe b\nthe " + b"b" * 40 + b"\nthe c\n"
    # shard 1 starts mid-line and holds the line start 12; shard 2 lies inside that line, shard 3 starts in it
    rows = rk.tiling_rows(P, text, [8, 20, 30], 4)
    t, head_to, nb = lib.regex_tiling(b"".join(r[:lib.REGEX_ROW_HEADER] for r in rows), len(rows))
    assert (t.text_len, t.last_byte, t.decider) == (len(text), 10, 3)
    assert head_to == [-1, 0, 1, 1]
    assert nb[0] == 0 and all(b == lib.REGEX_ROW_HEADER + rr.r16(len(rr.parse_row(r)["head"])) for b, r in zip(nb[1:], rows[1:]))
    head = rr.parse_row(lib.regex_row_head(rows[2]))
    full = rr.parse_row(rows[2])
    assert head["nkeys"] == head["nseg"] == 0 and head["head"] == full["head"] and head["own_begin"] == full["own_begin"]


def test_bad_tilings_refused():
    P = rk.params("the")
    text = b"the a\nthe b\nthe c\n"
    rows = rk.tiling_rows(P, text, [6, 12], 4)
    hdr = lambda rs: b"".join(r[:lib.REGEX_ROW_HEADER] for r in rs)  # noqa: E731
    lib.regex_tiling(hdr(rows), 3)
    for bad in (rows[1:], [rows[0], rows[2]], rows[:2], [rows[1], rows[0], rows[2]], [b"\0" * 128] + rows[1:]):
        with pytest.raises(RuntimeError):
            lib.regex_tiling(hdr(bad), len(bad))
    # a part whose line runs past the heads it is given
    rows = rk.tiling_rows(P, text, [3, 9], 0)
    with pytest.raises(RuntimeError):
        lib.regex_resolve_part(P, rows[:1], 1, len(text), 10, False)
    # rows that are not consecutive shards
    with pytest.raises(RuntimeError):
        lib.regex_resolve_part(P, [rows[0], rows[2]], 1, len(text), 10, False)
    lib.load().krep_b200_last_error()


# ---- the exchange of krep_b200/sharding.py over gloo ----

def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def exchange_cases(world):
    rng = random.Random(world)
    out = []
    for name, text, cuts in rk.cut_texts(world):
        for pat, opts in rk.PATTERNS:
            out.append((name, pat, dict(opts, **rng.choice(rk.MODES)), text, cuts, rng.choice(rk.HALOS)))
    text = km.random_lines_text(rng, 6000)
    for pat, opts in rk.PATTERNS:
        for mode in rk.MODES:
            out.append(("random", pat, dict(opts, **mode), text, sorted(rng.sample(range(1, len(text)), world - 1)),
                        rng.choice(rk.HALOS)))
    return out


def exchange_worker(rank, world, port, q):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    bad = []
    try:
        for name, pat, opts, text, cuts, halo in exchange_cases(world):
            P = rk.params(pat, **opts)
            sh = rr.tile(text, cuts, halo)[rank]
            row = torch.frombuffer(bytearray(rr.twin_row(P, sh)), dtype=torch.uint8)
            got = sharding.regex_resolve_ranks(P, row, rank, world)
            if rank == 0:
                got = (got[0], [tuple(x) for x in got[1].tolist()])
                if got != want_of(P, text):
                    bad.append((name, pat, opts, halo, got[0], want_of(P, text)[0]))
            elif got is not None:
                bad.append(("rank answered", rank))
        # a bad tiling (this rank's row shifted by one byte on the last rank) fails on every rank, none waits
        P = rk.params("the")
        text = b"the a\nthe b\nthe c\n" * 5
        cuts = [16 * i for i in range(1, world)]
        sh = rr.tile(text, cuts, 4)[rank]
        if rank == world - 1:
            sh = km.Shard(sh.buf, sh.own_begin + 1, sh.own_end, sh.global_offset, sh.prev_byte, sh.next_byte)
        row = torch.frombuffer(bytearray(rr.twin_row(P, sh)), dtype=torch.uint8)
        try:
            sharding.regex_resolve_ranks(P, row, rank, world)
            bad.append(("bad tiling accepted", rank))
        except RuntimeError as e:
            if "tile" not in str(e):
                bad.append(("unexpected error", rank, str(e)))
        dist.barrier()
    finally:
        dist.destroy_process_group()
    q.put((rank, bad))


def run_spawned(target, world, timeout=300):
    """Runs target(rank, world, port, q) in `world` spawned processes; joins them with a timeout and terminates them on
    failure (a worker that died, or the timeout), so no process outlives the test. -> {rank: what it put on the queue}"""
    ctx = torch.multiprocessing.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=target, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    out = {}
    deadline = time.monotonic() + timeout
    try:
        while len(out) < world and time.monotonic() < deadline:
            try:
                r, v = q.get(timeout=1)
                out[r] = v
            except queue.Empty:
                if any(p.exitcode not in (None, 0) for p in procs):
                    break
        for p in procs:
            p.join(max(1.0, min(60.0, deadline - time.monotonic())))
    finally:
        for p in procs:
            if p.is_alive():
                p.terminate()
                p.join(10)
    assert all(p.exitcode == 0 for p in procs), [p.exitcode for p in procs]
    assert sorted(out) == list(range(world)), out
    return out


@pytest.mark.parametrize("world", [2, 3])
def test_exchange_gloo(world):
    out = run_spawned(exchange_worker, world)
    assert all(v == [] for v in out.values()), out
