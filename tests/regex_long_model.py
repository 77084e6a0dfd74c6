"""A plain restatement of what the -E long-line pass adds to one k_regex_lines scan of a shard (scan_regex_long.cu,
DESIGN §12.8), on top of regex_kernel_model, for tests.

The pass takes an owned line that k_regex_lines leaves out of reach (its '\\n' at or beyond the owner's limit) when

  * its '\\n' lies within avail_len,
  * it is not the text's last line ('\\n' at avail_len - 1 with next_byte -1),
  * it is shorter than 2^30 bytes,

and decides it as the kernel would with unbounded reach:

  filter : the key stays exactly when the line automaton flags the line (a set of flagged starts, as for
           regex_kernel_model.expect);
  count  : the key goes, and a line with a match is counted;
  match  : the key goes and every match of the line is emitted, unless a match is REGEX_LONG_MAX_MATCH bytes or longer:
           then the line keeps its key, with the matches before that one.  A line over the step budget keeps its key
           and a prefix of its matches (the prefix form of regex_kernel_model.check).

Every other line is as in regex_kernel_model.expect.
"""
import collections

import numpy as np

import regex_kernel_model as km

MAX_LINE = 1 << 30
MAX_MATCH = 8192
SLICE, CKPT = 4096, 256  # production sizes (csrc/common.h)
REC_BYTES = 64 << 20     # slice records of one round (scan_regex_long.cu)

Sizes = collections.namedtuple("Sizes", "nck pick_cap owner_cap round_slices rounds")


def width(ngroups):
    """G of the pass's instantiation for a plan of ngroups automata: 1, 2, 4 or 8."""
    return 1 if ngroups <= 1 else 2 if ngroups <= 2 else 4 if ngroups <= 4 else 8


def sizes(avail, own, ngroups, slice=SLICE, ckpt=CKPT):
    """The pass's scratch sizing (sizes_of): checkpoints per slice record, work-list and slice-map capacities, slices
    per round (records of (S/C + 1) x G rows of 2 bytes, at most REC_BYTES a round) and the rounds launched."""
    nck = (slice + ckpt - 1) // ckpt + 1
    pick_cap = own // (km.REGEX_HALO + 1) + 2
    owner_cap = (avail + slice - 1) // slice + pick_cap
    round_slices = min(owner_cap, REC_BYTES // (nck * width(ngroups) * 2))
    return Sizes(nck, pick_cap, owner_cap, round_slices, -(-owner_cap // round_slices))


def slices_needed(sh, slice=SLICE):
    """Slices the pass hands out for shard sh: ceil((nl - p) / slice) per taken line."""
    return sum(-(-(nl - p) // slice) for p, nl in taken_lines(sh))


def taken_lines(sh):
    """[(p, nl)] of the lines the pass takes, in order."""
    a = np.frombuffer(sh.buf, dtype=np.uint8)
    nls = np.flatnonzero(a == 10)
    out = []
    for ln in km.owned_lines(sh):
        if ln.nl is not None:
            continue
        k = int(np.searchsorted(nls, ln.p))
        if k == len(nls):
            continue  # the line runs past avail_len
        nl = int(nls[k])
        if nl + 1 == sh.avail and sh.next_byte == -1:
            continue  # the text's last line
        if nl - ln.p >= MAX_LINE:
            continue
        out.append((ln.p, nl))
    return out


def expect(sh, mode, oracle, budget_free=False):
    """regex_kernel_model.expect with the pass applied.  oracle as there; in match mode the taken lines always take the
    prefix form unless budget_free.  The result has must_flag: match-mode line keys that must be present."""
    exp = km.expect(sh, mode, oracle, budget_free)
    exp.must_flag = set()
    G = sh.global_offset
    taken = taken_lines(sh)
    if mode == 0:
        for p, _ in taken:
            k = (G + p) << km.LIT_TAG_BITS
            exp.optional.discard(k)
            if p in oracle:
                exp.keys.append(k)
        exp.keys.sort()
        return exp
    if mode == 1:
        gone = {(G + p) << km.LIT_TAG_BITS for p, _ in taken}
        exp.keys = [k for k in exp.keys if k not in gone]
        exp.device_lines += sum(1 for p, nl in taken if oracle.verdict(p, nl))
        return exp
    gone = set()
    for p, nl in taken:
        lk = (G + p) << km.REGEX_MATCH_SHIFT
        gone.add(lk)
        ms = oracle.matches(p, nl)
        long_at = next((i for i, (s, e) in enumerate(ms) if e - s >= MAX_MATCH), None)
        keys = [((G + s) << km.REGEX_MATCH_SHIFT) | ((e - s) << km.LIT_TAG_BITS) | 1 for s, e in ms[:long_at]]
        if long_at is not None:
            exp.must_flag.add(lk)
            exp.prefix_lines[lk] = keys
        elif budget_free:
            exp.keys += keys
        elif keys:
            exp.prefix_lines[lk] = keys
    exp.keys = sorted(k for k in exp.keys if k not in gone)
    return exp


def check(exp, keys, device_lines, what=""):
    """regex_kernel_model.check, and the match-mode keys that must stay."""
    km.check(exp, keys, device_lines, what)
    if exp.mode == 2:
        missing = exp.must_flag - set(keys)
        assert not missing, (what, [hex(k) for k in sorted(missing)[:5]])


def long_lines_text(rng, n, alphabet=b"abcx ,", lens=(4000, 4097, 4352, 4353, 5000, 8192, 9000, 20000)):
    """Text with many lines longer than the reach: random short lines (regex_util.random_text) between long lines of
    random bytes from alphabet, with lengths around the reach, the slice size and its multiples."""
    parts = []
    while sum(map(len, parts)) < n:
        if rng.random() < 0.4:
            L = rng.choice(lens) + rng.randint(-3, 3)
            parts.append(bytes(rng.choice(alphabet) for _ in range(max(L, 1))) + b"\n")
        else:
            parts.append(km.ru.random_text(rng, rng.randint(1, 300)))
    text = b"".join(parts)[:n]
    return text if rng.random() < 0.5 else text.rstrip(b"\n") + b"\n"
