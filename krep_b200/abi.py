"""ctypes mirror of include/krep_b200.h (the types restated from krep.h:49-101).

Plumbing only: tests and bench.py use these to call the C ABI of libkrep_b200.so,
the oracle port and the compiled reference with the very same structs.
"""
import ctypes as C
import locale

SIZE_MAX = (1 << 64) - 1


class MatchPosition(C.Structure):  # krep.h:49-53
    _fields_ = [("start_offset", C.c_size_t), ("end_offset", C.c_size_t)]


class MatchResult(C.Structure):  # krep.h:55-60
    _fields_ = [("positions", C.POINTER(MatchPosition)), ("count", C.c_uint64), ("capacity", C.c_uint64)]


class SearchParams(C.Structure):  # krep.h:65-94
    _fields_ = [
        ("pattern", C.c_char_p),
        ("pattern_len", C.c_size_t),
        ("patterns", C.POINTER(C.c_char_p)),
        ("pattern_lens", C.POINTER(C.c_size_t)),
        ("num_patterns", C.c_size_t),
        ("case_sensitive", C.c_bool),
        ("use_regex", C.c_bool),
        ("count_lines_mode", C.c_bool),
        ("count_matches_mode", C.c_bool),
        ("track_positions", C.c_bool),
        ("whole_word", C.c_bool),
        ("compiled_regex", C.c_void_p),
        ("ac_trie", C.c_void_p),
        ("max_count", C.c_size_t),
    ]


SEARCH_FUNC = C.CFUNCTYPE(C.c_uint64, C.POINTER(SearchParams), C.c_void_p, C.c_size_t, C.POINTER(MatchResult))


class Shard(C.Structure):  # krep_b200_shard_t
    _fields_ = [
        ("d_text", C.c_void_p),
        ("avail_len", C.c_uint64),
        ("own_begin", C.c_uint64),
        ("own_end", C.c_uint64),
        ("global_offset", C.c_uint64),
        ("prev_byte", C.c_int32),
        ("next_byte", C.c_int32),
    ]


class DeviceResult(C.Structure):  # krep_b200_device_result_t
    _fields_ = [
        ("count", C.c_uint64),
        ("stored", C.c_uint64),
        ("d_keys", C.c_void_p),
        ("overflow", C.c_int),
        ("text_len", C.c_uint64),
        ("d_line_bounds", C.c_void_p),
        ("device", C.c_int32),
        ("slot", C.c_int32),
        ("serial", C.c_uint64),
    ]


REGEX_ROW_HEADER = 128  # KREP_B200_REGEX_ROW_HEADER


class RegexTiling(C.Structure):  # krep_b200_regex_tiling_t
    _fields_ = [("text_len", C.c_uint64), ("last_byte", C.c_int32), ("decider", C.c_uint32)]


class CorpusSpec(C.Structure):  # krep_b200_corpus_spec_t
    _fields_ = [
        ("seed", C.c_uint64),
        ("plant_seed", C.c_uint64),
        ("plant_period", C.c_uint64),
        ("needle", C.c_char_p),
        ("needle_len", C.c_uint32),
        ("flags", C.c_uint32),
    ]


CORPUS_RANDOM_CASE = 1
CORPUS_EMBED_HALF = 2

ALGO_BMH, ALGO_KMP, ALGO_MEMCHR, ALGO_MEMCHR_SHORT, ALGO_SSE42, ALGO_AVX2, ALGO_AVX512, ALGO_AC, ALGO_NEON, ALGO_REGEX = range(10)

# <regex.h> (glibc): regcomp / regexec flags, regmatch_t with 32-bit regoff_t
REG_EXTENDED, REG_ICASE, REG_NEWLINE = 1, 2, 4
REG_NOTBOL, REG_NOTEOL, REG_STARTEND = 1, 2, 4
REGEX_T_BYTES = 256  # >= sizeof(regex_t) (64 on x86-64 glibc)


class RegMatch(C.Structure):
    _fields_ = [("rm_so", C.c_int), ("rm_eo", C.c_int)]


_libc = None


def libc():
    global _libc
    if _libc is None:
        _libc = C.CDLL("libc.so.6")
        _libc.regcomp.argtypes = [C.c_void_p, C.c_char_p, C.c_int]
        _libc.regexec.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.POINTER(RegMatch), C.c_int]
        _libc.regfree.argtypes = [C.c_void_p]
    return _libc


def c_locale():
    """krep never calls setlocale, so its regexes are C-locale regexes; Python starts in the user's LC_CTYPE.  Regexes
    compiled here (and the library's line automaton, which refuses multibyte locales) need the C locale."""
    locale.setlocale(locale.LC_CTYPE, "C")


def krep_regex_source(patterns, whole_word):
    """The string krep hands to regcomp (krep.c:2081-2145): patterns read as C strings."""
    pats = [p.split(b"\0", 1)[0] for p in patterns]
    if len(pats) > 1:
        return b"|".join((b"(\\b" + p + b"\\b)") if whole_word else (b"(" + p + b")") for p in pats)
    return (b"\\b" + pats[0] + b"\\b") if whole_word else pats[0]


class Regex:
    """A glibc regex_t compiled with krep's flags (REG_EXTENDED | REG_NEWLINE | REG_ICASE for -i)."""

    def __init__(self, source, case_sensitive=True):
        c_locale()
        self.buf = C.create_string_buffer(REGEX_T_BYTES)
        rc = libc().regcomp(self.buf, source, REG_EXTENDED | REG_NEWLINE | (0 if case_sensitive else REG_ICASE))
        if rc != 0:
            self.buf = None
            raise ValueError(f"regcomp failed ({rc}) for {source!r}")

    def ptr(self):
        return C.cast(self.buf, C.c_void_p)

    def search(self, text, start, end, eflags):
        """regexec with REG_STARTEND on text[start:end] (text: a ctypes buffer or bytes). -> (so, eo) relative to start, or None."""
        m = (RegMatch * 1)()
        m[0].rm_so, m[0].rm_eo = 0, end - start
        base = C.cast(text, C.c_void_p).value if not isinstance(text, bytes) else C.cast(C.c_char_p(text), C.c_void_p).value
        rc = libc().regexec(self.buf, C.c_void_p(base + start), 1, m, eflags | REG_STARTEND)
        return None if rc else (m[0].rm_so, m[0].rm_eo)

    def __del__(self):
        if getattr(self, "buf", None) is not None and _libc is not None:
            _libc.regfree(self.buf)
            self.buf = None


class Params:
    """Owns the Python-side buffers behind one search_params_t.

    Mirrors the reference tests' create_literal_params (test/test_krep.c:208-249):
    count_lines_mode = -c && !-o, count_matches_mode = -c && -o,
    track_positions = !(-c && !-o)   (krep.c:3811-3814).
    regex=True is -E: use_regex is set and compiled_regex points at a regex_t compiled from the patterns as krep does.
    """

    def __init__(self, patterns, case_sensitive=True, count=False, only_matching=False,
                 whole_word=False, max_count=SIZE_MAX, track_positions=None, regex=False):
        if isinstance(patterns, (bytes, bytearray)):
            patterns = [bytes(patterns)]
        self.patterns = [bytes(p) for p in patterns]
        n = len(self.patterns)
        # c_char_p would stop at NUL bytes when read back, but the struct only stores pointers.
        self._bufs = [C.create_string_buffer(p, len(p) + 16) for p in self.patterns]  # +16: krep.c:4725 over-read
        self._arr = (C.c_char_p * max(n, 1))(*[C.cast(b, C.c_char_p) for b in self._bufs])
        self._lens = (C.c_size_t * max(n, 1))(*[len(p) for p in self.patterns])
        s = SearchParams()
        s.patterns = C.cast(self._arr, C.POINTER(C.c_char_p))
        s.pattern_lens = C.cast(self._lens, C.POINTER(C.c_size_t))
        s.num_patterns = n
        if n:
            s.pattern = C.cast(self._bufs[0], C.c_char_p)
            s.pattern_len = len(self.patterns[0])
        s.case_sensitive = case_sensitive
        s.use_regex = bool(regex)
        s.count_lines_mode = bool(count and not only_matching)
        s.count_matches_mode = bool(count and only_matching)
        s.track_positions = (not (count and not only_matching)) if track_positions is None else track_positions
        s.whole_word = whole_word
        self.regex = Regex(krep_regex_source(self.patterns, whole_word), case_sensitive) if regex else None
        s.compiled_regex = self.regex.ptr() if regex else None
        s.ac_trie = None
        s.max_count = max_count
        self.only_matching = only_matching
        self.struct = s

    def ref(self):
        return C.byref(self.struct)
