"""Helpers shared by the -E tests: a Python restatement of the reference's regex_search (krep.c:1389-1579) over glibc's
regexec, a random ERE generator for the supported grammar, and the library's host-side line-filter hook."""
import ctypes as C

from krep_b200 import lib
from krep_b200.abi import REG_ICASE, REG_NEWLINE, REG_NOTBOL, REG_STARTEND


def _is_word(b):
    return (48 <= b <= 57) or (65 <= b <= 90) or (97 <= b <= 122) or b == 95


def ref_regex_search(params, text):
    """krep.c:1389-1579 restated line for line. -> (count, [(start, end), ...])"""
    P = params.struct
    rx = params.regex
    n = len(text)
    if P.max_count == 0 and (P.count_lines_mode or P.track_positions):
        return 0, []
    if rx is None:
        return 0, []
    buf = C.create_string_buffer(text, n + 1)
    pos = []
    if n == 0:
        if rx.search(buf, 0, 0, 0) is not None:
            if P.count_lines_mode:
                return 1, []
            if P.track_positions:
                pos.append((0, 0))
            return 1, pos
        return 0, []
    # compilation flags passed as execution flags, as krep.c:1422 does (REG_NEWLINE == REG_STARTEND, REG_ICASE == REG_NOTEOL)
    base = REG_STARTEND | REG_NEWLINE | (0 if P.case_sensitive else REG_ICASE)
    cur, last_line, count, max_count = 0, None, 0, P.max_count
    while cur < n:
        at_ls = cur == 0 or text[cur - 1] == 10
        r = rx.search(buf, cur, n, base | (0 if at_ls else REG_NOTBOL))
        if r is None:
            break
        so, eo = r
        start, end = cur + so, cur + eo
        if P.whole_word and ((start > 0 and _is_word(text[start - 1])) or (end < n and _is_word(text[end]))):
            cur = min(cur + so + 1, n)
            continue
        if P.count_lines_mode:
            ls = text.rfind(b"\n", 0, start) + 1
            if ls != last_line:
                count += 1
                last_line = ls
                if count >= max_count:
                    break
                le = text.find(b"\n", ls)
                cur = le + 1 if le >= 0 else n
                continue
        else:
            count += 1
            if P.track_positions:
                pos.append((start, end))
        if count >= max_count:
            break
        cur = min(cur + (so + 1 if so == eo else eo), n)
    return count, pos


def line_starts(text):
    out, p, n = [], 0, len(text)
    while p < n:
        out.append(p)
        q = text.find(b"\n", p)
        if q < 0:
            break
        p = q + 1
    return out


def filter_host(params, text):
    """The library's line filter for params, run on the host. -> (flagged line starts, widened) or None when refused."""
    L = lib.load()
    cap = max(len(text), 1)
    out = (C.c_uint64 * cap)()
    wid = C.c_int(0)
    buf = C.create_string_buffer(text, len(text) + 1)
    k = L.krep_b200_regex_filter_host(params.ref(), buf, len(text), out, cap, C.byref(wid))
    if k < 0:
        return None
    return list(out[:k]), bool(wid.value)


def replay(params, keys, text):
    """krep_b200_replay with KREP_B200_ALGO_REGEX on host keys (flagged line starts << 3)."""
    L = lib.load()
    arr = (C.c_uint64 * max(len(keys), 1))(*keys)
    buf = C.create_string_buffer(text, len(text) + 1)
    res = L.krep_b200_match_result_init(16)
    try:
        cnt = L.krep_b200_replay(9, params.ref(), False, arr, len(keys), buf, len(text), res)
        lib.check(L)
        r = res.contents
        return int(cnt), [(r.positions[i].start_offset, r.positions[i].end_offset) for i in range(r.count)]
    finally:
        L.krep_b200_match_result_free(res)


ATOMS = ["a", "b", "c", "ab", ".", "[ab]", "[^a]", "[a-c]", "[[:alpha:]]", "[[:digit:]]", "x", "A", "\\.", " ", "\\w",
         "[^ ]", "0", "[0-9]"]
ZERO_WIDTH = ["^", "$", "\\b", "\\B", "\\<", "\\>"]


def random_regex(rng, depth=0):
    parts = []
    for _ in range(rng.randint(1, 3)):
        r = rng.random()
        if r < 0.12 and depth < 2:
            alts = [random_regex(rng, depth + 1) for _ in range(rng.randint(1, 3))]
            if rng.random() < 0.15:
                alts.append("")
            atom = "(" + "|".join(alts) + ")"
        elif r < 0.22:
            parts.append(rng.choice(ZERO_WIDTH))
            continue
        else:
            atom = rng.choice(ATOMS)
            if len(atom) == 2 and atom[0] != "\\" and atom[0] not in ".[":
                atom = "(" + atom + ")"
        q = rng.random()
        if q < 0.12:
            atom += "*"
        elif q < 0.2:
            atom += "+"
        elif q < 0.27:
            atom += "?"
        elif q < 0.33:
            lo = rng.randint(0, 2)
            atom += rng.choice(["{%d}" % lo, "{%d,}" % lo, "{%d,%d}" % (lo, lo + rng.randint(0, 2)), "{,%d}" % (lo + 1)])
        parts.append(atom)
    return "".join(parts)


def random_text(rng, n):
    alphabet = b"aabbcxA0. \n\n_"
    return bytes(rng.choice(alphabet) for _ in range(n))


CASES = [dict(), dict(case_sensitive=False), dict(whole_word=True), dict(count=True), dict(max_count=1),
         dict(max_count=2), dict(max_count=3), dict(count=True, max_count=2), dict(count=True, only_matching=True),
         dict(case_sensitive=False, whole_word=True)]

