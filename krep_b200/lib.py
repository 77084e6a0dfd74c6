"""ctypes binding of libkrep_b200.so — plumbing for tests and bench.py, not a second implementation.

The library is loaded from krep_b200/libkrep_b200.so (built in-tree by krep_b200/build.py).  Loading
never falls back to anything else: if the .so is missing this raises, and if no sm_90 device is
usable every search call reports an error through krep_b200_last_error().
"""
import ctypes as C
import os

from .abi import (REGEX_ROW_HEADER, CorpusSpec, DeviceResult, MatchResult, Params, RegexTiling, SearchParams, Shard,  # noqa: F401
                  SEARCH_FUNC, SIZE_MAX)

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("KREP_B200_LIB") or os.path.join(_HERE, "libkrep_b200.so")  # override: kernel-variant builds

SEARCH_ENTRIES = {
    "boyer_moore": "krep_b200_boyer_moore_search",
    "kmp": "krep_b200_kmp_search",
    "memchr": "krep_b200_memchr_search",
    "memchr_short": "krep_b200_memchr_short_search",
    "sse42": "krep_b200_simd_sse42_search",
    "avx2": "krep_b200_simd_avx2_search",
    "avx512": "krep_b200_simd_avx512_search",
    "aho_corasick": "krep_b200_aho_corasick_search",
    "neon": "krep_b200_neon_search",
    "regex": "krep_b200_regex_search",
}

_lib = None


def load():
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(f"{LIB_PATH} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                           "(there is no fallback implementation)")
    L = C.CDLL(LIB_PATH)
    sig = [C.POINTER(SearchParams), C.c_void_p, C.c_size_t, C.POINTER(MatchResult)]
    for name in SEARCH_ENTRIES.values():
        f = getattr(L, name)
        f.argtypes = sig
        f.restype = C.c_uint64
    L.krep_b200_init.argtypes = [C.c_int]
    L.krep_b200_init.restype = C.c_int
    L.krep_b200_last_error.restype = C.c_int
    L.krep_b200_last_error_string.restype = C.c_char_p
    L.krep_b200_version.restype = C.c_char_p
    L.krep_b200_set_only_matching.argtypes = [C.c_bool]
    L.krep_b200_get_only_matching.restype = C.c_bool
    L.krep_b200_set_force_no_simd.argtypes = [C.c_bool]
    L.krep_b200_set_algo_override.argtypes = [C.c_char_p]
    L.krep_b200_select_search_algorithm.argtypes = [C.POINTER(SearchParams)]
    L.krep_b200_select_search_algorithm.restype = C.c_void_p
    L.krep_b200_get_algorithm_name.argtypes = [C.c_void_p]
    L.krep_b200_get_algorithm_name.restype = C.c_char_p
    L.krep_b200_ac_trie_build.argtypes = [C.POINTER(SearchParams)]
    L.krep_b200_ac_trie_build.restype = C.c_void_p
    L.krep_b200_ac_trie_free.argtypes = [C.c_void_p]
    L.krep_b200_ac_trie_root_has_outputs.argtypes = [C.c_void_p]
    L.krep_b200_ac_trie_root_has_outputs.restype = C.c_bool
    L.krep_b200_match_result_init.argtypes = [C.c_uint64]
    L.krep_b200_match_result_init.restype = C.POINTER(MatchResult)
    L.krep_b200_match_result_add.argtypes = [C.POINTER(MatchResult), C.c_size_t, C.c_size_t]
    L.krep_b200_match_result_add.restype = C.c_bool
    L.krep_b200_match_result_free.argtypes = [C.POINTER(MatchResult)]
    L.krep_b200_match_result_merge.argtypes = [C.POINTER(MatchResult), C.POINTER(MatchResult), C.c_size_t]
    L.krep_b200_match_result_merge.restype = C.c_bool
    L.krep_b200_plan_create.argtypes = [C.POINTER(SearchParams), C.c_int]
    L.krep_b200_plan_create.restype = C.c_void_p
    L.krep_b200_plan_destroy.argtypes = [C.c_void_p]
    L.krep_b200_plan_filter_name.argtypes = [C.c_void_p]
    L.krep_b200_plan_filter_name.restype = C.c_char_p
    L.krep_b200_scan_shard.argtypes = [C.c_void_p, C.POINTER(Shard), C.c_int, C.c_void_p, C.POINTER(DeviceResult)]
    L.krep_b200_scan_shard.restype = C.c_int
    L.krep_b200_collect.argtypes = [C.c_void_p, C.POINTER(SearchParams), C.POINTER(DeviceResult), C.POINTER(MatchResult)]
    L.krep_b200_collect.restype = C.c_uint64
    L.krep_b200_replay.argtypes = [C.c_int, C.POINTER(SearchParams), C.c_bool, C.POINTER(C.c_uint64), C.c_uint64,
                                   C.c_void_p, C.c_size_t, C.POINTER(MatchResult)]
    L.krep_b200_replay.restype = C.c_uint64
    L.krep_b200_replay_lines.argtypes = [C.c_int, C.POINTER(SearchParams), C.c_bool, C.POINTER(C.c_uint64), C.c_uint64,
                                         C.POINTER(C.c_uint64), C.c_size_t, C.POINTER(MatchResult)]
    L.krep_b200_replay_lines.restype = C.c_uint64
    L.krep_b200_search_batch.argtypes = [C.c_void_p, C.POINTER(SearchParams), C.POINTER(C.c_char_p), C.POINTER(C.c_size_t), C.c_size_t,
                                         C.POINTER(C.c_uint64), C.POINTER(C.POINTER(MatchResult))]
    L.krep_b200_search_batch.restype = C.c_int
    L.krep_b200_regex_search_batch.argtypes = [C.POINTER(SearchParams), C.POINTER(C.c_char_p), C.POINTER(C.c_size_t), C.c_size_t,
                                               C.POINTER(C.c_uint64), C.POINTER(C.POINTER(MatchResult))]
    L.krep_b200_regex_search_batch.restype = C.c_int
    L.krep_b200_regex_batch_stats.argtypes = [C.POINTER(C.c_double), C.POINTER(C.c_double)]
    L.krep_b200_regex_batch_stats.restype = None
    L.krep_b200_regex_search_batch_raw.argtypes = [C.POINTER(SearchParams), C.POINTER(C.c_char_p), C.POINTER(C.c_size_t), C.c_size_t,
                                                   C.c_int, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64), C.c_uint64,
                                                   C.POINTER(C.c_uint64)]
    L.krep_b200_regex_search_batch_raw.restype = C.c_int64
    L.krep_b200_regex_search_batch_long_raw.argtypes = [C.POINTER(SearchParams), C.POINTER(C.c_char_p), C.POINTER(C.c_size_t),
                                                        C.c_size_t, C.c_int, C.c_uint32, C.c_uint32, C.POINTER(C.c_uint64),
                                                        C.POINTER(C.c_uint64), C.c_uint64, C.POINTER(C.c_uint64)]
    L.krep_b200_regex_search_batch_long_raw.restype = C.c_int64
    L.krep_b200_search_batch_resident.argtypes = [C.c_void_p, C.POINTER(SearchParams), C.c_void_p, C.POINTER(C.c_uint64),
                                                  C.POINTER(C.c_size_t), C.c_size_t, C.POINTER(C.c_uint64),
                                                  C.POINTER(C.POINTER(MatchResult))]
    L.krep_b200_search_batch_resident.restype = C.c_int
    L.krep_b200_regex_search_batch_resident.argtypes = [C.POINTER(SearchParams), C.c_void_p, C.POINTER(C.c_uint64),
                                                        C.POINTER(C.c_size_t), C.c_size_t, C.POINTER(C.c_uint64),
                                                        C.POINTER(C.POINTER(MatchResult))]
    L.krep_b200_regex_search_batch_resident.restype = C.c_int
    L.krep_b200_batch_resident_stats.argtypes = [C.POINTER(C.c_float), C.POINTER(C.c_float), C.POINTER(C.c_double)]
    L.krep_b200_batch_resident_stats.restype = None
    L.krep_b200_batch_gather_raw.argtypes = [C.c_void_p, C.POINTER(C.c_uint64), C.POINTER(C.c_size_t), C.c_size_t, C.c_int,
                                             C.c_size_t, C.c_void_p, C.c_uint64]
    L.krep_b200_batch_gather_raw.restype = C.c_int64
    L.krep_b200_scan_shard_begin.argtypes = [C.c_void_p, C.POINTER(Shard), C.c_int, C.c_void_p, C.POINTER(C.c_int)]
    L.krep_b200_scan_shard_begin.restype = C.c_int
    L.krep_b200_scan_shard_end.argtypes = [C.c_int, C.POINTER(DeviceResult)]
    L.krep_b200_scan_shard_end.restype = C.c_int
    L.krep_b200_export_packed.argtypes = [C.POINTER(DeviceResult), C.c_void_p, C.c_uint64, C.c_void_p]
    L.krep_b200_export_packed.restype = C.c_int
    L.krep_b200_export_packed_async.argtypes = [C.c_int, C.c_void_p, C.c_uint64]
    L.krep_b200_export_packed_async.restype = C.c_int
    L.krep_b200_merge_keys.argtypes = [C.POINTER(C.c_void_p), C.POINTER(C.c_uint64), C.c_uint32, C.c_void_p]
    L.krep_b200_merge_keys.restype = C.c_uint64
    L.krep_b200_set_devices.argtypes = [C.POINTER(C.c_int), C.c_int]
    L.krep_b200_device_count.restype = C.c_int
    L.krep_b200_search_shards.argtypes = [C.c_void_p, C.POINTER(SearchParams), C.POINTER(Shard), C.c_uint32, C.POINTER(MatchResult)]
    L.krep_b200_search_shards.restype = C.c_uint64
    L.krep_b200_export_keys.argtypes = [C.POINTER(DeviceResult), C.c_void_p, C.c_uint64, C.c_void_p]
    L.krep_b200_export_keys.restype = C.c_int
    L.krep_b200_regex_filter_host.argtypes = [C.POINTER(SearchParams), C.c_void_p, C.c_size_t, C.POINTER(C.c_uint64), C.c_uint64,
                                              C.POINTER(C.c_int)]
    L.krep_b200_regex_filter_host.restype = C.c_int64
    L.krep_b200_regex_count_mode.argtypes = [C.POINTER(SearchParams)]
    L.krep_b200_regex_count_mode.restype = C.c_int
    L.krep_b200_regex_count_host.argtypes = [C.POINTER(SearchParams), C.c_void_p, C.c_size_t, C.c_uint64]
    L.krep_b200_regex_count_host.restype = C.c_int64
    L.krep_b200_regex_match_mode.argtypes = [C.POINTER(SearchParams)]
    L.krep_b200_regex_match_mode.restype = C.c_int
    L.krep_b200_regex_matches_host.argtypes = [C.POINTER(SearchParams), C.c_void_p, C.c_size_t, C.c_uint64, C.POINTER(MatchResult)]
    L.krep_b200_regex_matches_host.restype = C.c_int64
    L.krep_b200_regex_scan_shard_raw.argtypes = [C.c_void_p, C.POINTER(Shard), C.c_int, C.POINTER(C.c_uint64), C.c_uint64,
                                                 C.POINTER(C.c_uint64)]
    L.krep_b200_regex_scan_shard_raw.restype = C.c_int64
    L.krep_b200_regex_scan_shard_long_raw.argtypes = [C.c_void_p, C.POINTER(Shard), C.c_int, C.c_uint32, C.c_uint32,
                                                      C.POINTER(C.c_uint64), C.c_uint64, C.POINTER(C.c_uint64)]
    L.krep_b200_regex_scan_shard_long_raw.restype = C.c_int64
    L.krep_b200_regex_automata.argtypes = [C.POINTER(SearchParams)]
    L.krep_b200_regex_automata.restype = C.c_int
    L.krep_b200_regex_plan_split.argtypes = [C.POINTER(SearchParams), C.c_uint32]
    L.krep_b200_regex_plan_split.restype = C.c_void_p
    L.krep_b200_regex_plan_host.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_size_t, C.c_uint64, C.POINTER(C.c_uint64),
                                            C.c_uint64, C.POINTER(C.c_uint64)]
    L.krep_b200_regex_plan_host.restype = C.c_int64
    L.krep_b200_regex_export_shard.argtypes = [C.c_void_p, C.POINTER(SearchParams), C.POINTER(Shard), C.c_void_p, C.c_void_p,
                                               C.c_uint64, C.POINTER(C.c_uint64), C.POINTER(C.c_void_p)]
    L.krep_b200_regex_export_shard.restype = C.c_int
    L.krep_b200_regex_resolve.argtypes = [C.POINTER(SearchParams), C.POINTER(C.c_void_p), C.c_uint32, C.POINTER(MatchResult)]
    L.krep_b200_regex_resolve.restype = C.c_uint64
    L.krep_b200_regex_resolve_part.argtypes = [C.POINTER(SearchParams), C.POINTER(C.c_void_p), C.c_uint32, C.c_uint32, C.c_uint64,
                                               C.c_int, C.c_int, C.POINTER(MatchResult)]
    L.krep_b200_regex_resolve_part.restype = C.c_uint64
    L.krep_b200_regex_row_head.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64]
    L.krep_b200_regex_row_head.restype = C.c_uint64
    L.krep_b200_regex_tiling.argtypes = [C.c_void_p, C.c_uint32, C.POINTER(RegexTiling), C.POINTER(C.c_int32),
                                         C.POINTER(C.c_uint64)]
    L.krep_b200_regex_tiling.restype = C.c_int
    L.krep_b200_regex_export_stats.argtypes = [C.POINTER(C.c_float), C.POINTER(C.c_float), C.POINTER(C.c_uint64)]
    L.krep_b200_last_kernel_ms.restype = C.c_float
    L.krep_b200_launch_count.restype = C.c_uint64
    for n in ("krep_b200_ac_key_end", "krep_b200_ac_key_start"):
        getattr(L, n).argtypes = [C.c_uint64]
        getattr(L, n).restype = C.c_uint64
    L.krep_b200_ac_key_pattern.argtypes = [C.c_uint64]
    L.krep_b200_ac_key_pattern.restype = C.c_uint32
    L.krep_b200_corpus_generate.argtypes = [C.POINTER(CorpusSpec), C.c_void_p, C.c_uint64, C.c_uint64, C.c_void_p]
    L.krep_b200_corpus_generate.restype = C.c_int
    L.krep_b200_corpus_generate_host.argtypes = [C.POINTER(CorpusSpec), C.c_void_p, C.c_uint64, C.c_uint64]
    L.krep_b200_corpus_generate_host.restype = C.c_int
    _lib = L
    return L


def check(L=None):
    L = L or load()
    if L.krep_b200_last_error() != 0:
        raise RuntimeError("krep_b200: " + L.krep_b200_last_error_string().decode())


def search(func, params, text, with_result=True, text_ptr=None, text_len=None):
    """Calls one search_func_t entry point on host text. -> (count, [(start, end), ...]).

    `text` is bytes (or pass text_ptr/text_len for a raw host buffer, e.g. pinned memory).
    Raises if the library reported an error (missing GPU, CUDA failure): there is no fallback.
    """
    L = load()
    L.krep_b200_set_only_matching(bool(params.only_matching))
    own_trie = False
    if func == "aho_corasick" and not params.struct.ac_trie:
        params.struct.ac_trie = L.krep_b200_ac_trie_build(params.ref())
        own_trie = True
    res = L.krep_b200_match_result_init(16) if with_result else None
    try:
        if text_ptr is None:
            buf = C.cast(C.c_char_p(text), C.c_void_p)
            n = len(text)
        else:
            buf, n = C.c_void_p(text_ptr), text_len
        cnt = getattr(L, SEARCH_ENTRIES[func])(params.ref(), buf, n, res)
        check(L)
        pos = []
        if res:
            r = res.contents
            pos = [(r.positions[i].start_offset, r.positions[i].end_offset) for i in range(r.count)]
        return int(cnt), pos
    finally:
        if res:
            L.krep_b200_match_result_free(res)
        if own_trie:
            L.krep_b200_ac_trie_free(params.struct.ac_trie)
            params.struct.ac_trie = None
        L.krep_b200_set_only_matching(False)


def make_spec(seed, plant_seed=0, plant_period=0, needle=b"", flags=0):
    s = CorpusSpec()
    s.seed = seed
    s.plant_seed = plant_seed
    s.plant_period = plant_period
    s._needle_keepalive = C.create_string_buffer(needle, max(len(needle), 1))
    s.needle = C.cast(s._needle_keepalive, C.c_char_p)
    s.needle_len = len(needle)
    s.flags = flags
    return s


def corpus_host(spec, offset, length):
    L = load()
    buf = C.create_string_buffer(length)
    rc = L.krep_b200_corpus_generate_host(C.byref(spec), buf, offset, length)
    if rc != 0:
        raise RuntimeError("corpus_generate_host failed")
    return buf.raw


def search_batch(func, params, texts, with_result=True):
    """krep_b200_search_batch on a list of bytes objects. -> [(count, [(start, end), ...]), ...]"""
    L = load()
    L.krep_b200_set_only_matching(bool(params.only_matching))
    own_trie = False
    if func == "aho_corasick" and not params.struct.ac_trie:
        params.struct.ac_trie = L.krep_b200_ac_trie_build(params.ref())
        own_trie = True
    n = len(texts)
    bufs = [C.create_string_buffer(t, max(len(t), 1)) for t in texts]
    tarr = (C.c_char_p * max(n, 1))(*[C.cast(b, C.c_char_p) for b in bufs])
    larr = (C.c_size_t * max(n, 1))(*[len(t) for t in texts])
    counts = (C.c_uint64 * max(n, 1))()
    res = [L.krep_b200_match_result_init(16) for _ in range(n)] if with_result else []
    rarr = (C.POINTER(MatchResult) * max(n, 1))(*res) if with_result else None
    try:
        entry = C.cast(getattr(L, SEARCH_ENTRIES[func]), C.c_void_p)
        rc = L.krep_b200_search_batch(entry, params.ref(), tarr, larr, n, counts, rarr)
        check(L)
        assert rc == 0, rc
        out = []
        for i in range(n):
            pos = []
            if with_result:
                r = res[i].contents
                pos = [(r.positions[k].start_offset, r.positions[k].end_offset) for k in range(r.count)]
            out.append((int(counts[i]), pos))
        return out
    finally:
        for r in res:
            L.krep_b200_match_result_free(r)
        if own_trie:
            L.krep_b200_ac_trie_free(params.struct.ac_trie)
            params.struct.ac_trie = None
        L.krep_b200_set_only_matching(False)


def text_array(texts):
    """(keep-alive buffers, char* array, size_t array) for a list of bytes objects."""
    n = len(texts)
    bufs = [C.create_string_buffer(t, max(len(t), 1)) for t in texts]
    tarr = (C.c_char_p * max(n, 1))(*[C.cast(b, C.c_char_p) for b in bufs])
    larr = (C.c_size_t * max(n, 1))(*[len(t) for t in texts])
    return bufs, tarr, larr


def regex_search_batch(params, texts, with_result=True):
    """krep_b200_regex_search_batch on a list of bytes objects. -> [(count, [(start, end), ...]), ...]"""
    L = load()
    n = len(texts)
    _bufs, tarr, larr = text_array(texts)
    counts = (C.c_uint64 * max(n, 1))()
    res = [L.krep_b200_match_result_init(16) for _ in range(n)] if with_result else []
    rarr = (C.POINTER(MatchResult) * max(n, 1))(*res) if with_result else None
    try:
        rc = L.krep_b200_regex_search_batch(params.ref(), tarr, larr, n, counts, rarr)
        check(L)
        assert rc == 0, rc
        return [(int(counts[i]), _positions(res[i]) if with_result else []) for i in range(n)]
    finally:
        for r in res:
            L.krep_b200_match_result_free(r)


def _resident_args(tensor, offsets, lens):
    """(d_base, offsets array, lens array, n) for a uint8 CUDA tensor (any view) and int sequences or CPU int64 tensors."""
    if not getattr(tensor, "is_cuda", False) or tensor.dtype.itemsize != 1:
        raise ValueError("texts must be a uint8 CUDA tensor")
    offs = [int(x) for x in (offsets.tolist() if hasattr(offsets, "tolist") else offsets)]
    ls = [int(x) for x in (lens.tolist() if hasattr(lens, "tolist") else lens)]
    if len(offs) != len(ls):
        raise ValueError("offsets and lens differ in length")
    n = len(ls)
    if any(o < 0 or l < 0 or o + l > tensor.numel() for o, l in zip(offs, ls)):
        raise ValueError("a text lies outside the tensor")
    if not tensor.is_contiguous():
        raise ValueError("the tensor must be contiguous")
    # the library reads the texts on its own stream: whatever torch has queued that writes them must be done first
    import torch
    torch.cuda.current_stream(tensor.device).synchronize()
    return tensor.data_ptr(), (C.c_uint64 * max(n, 1))(*offs), (C.c_size_t * max(n, 1))(*ls), n


def search_batch_resident(func, params, tensor, offsets, lens, with_result=True):
    """krep_b200_search_batch_resident on texts tensor[offsets[i] : offsets[i] + lens[i]] of a uint8 CUDA tensor.
    -> [(count, [(start, end), ...]), ...], as search_batch on host copies of the texts."""
    L = load()
    base, oarr, larr, n = _resident_args(tensor, offsets, lens)
    L.krep_b200_set_only_matching(bool(params.only_matching))
    own_trie = False
    if func == "aho_corasick" and not params.struct.ac_trie:
        params.struct.ac_trie = L.krep_b200_ac_trie_build(params.ref())
        own_trie = True
    counts = (C.c_uint64 * max(n, 1))()
    res = [L.krep_b200_match_result_init(16) for _ in range(n)] if with_result else []
    rarr = (C.POINTER(MatchResult) * max(n, 1))(*res) if with_result else None
    try:
        entry = C.cast(getattr(L, SEARCH_ENTRIES[func]), C.c_void_p)
        rc = L.krep_b200_search_batch_resident(entry, params.ref(), base, oarr, larr, n, counts, rarr)
        check(L)
        assert rc == 0, rc
        return [(int(counts[i]), _positions(res[i]) if with_result else []) for i in range(n)]
    finally:
        for r in res:
            L.krep_b200_match_result_free(r)
        if own_trie:
            L.krep_b200_ac_trie_free(params.struct.ac_trie)
            params.struct.ac_trie = None
        L.krep_b200_set_only_matching(False)


def regex_search_batch_resident(params, tensor, offsets, lens, with_result=True):
    """krep_b200_regex_search_batch_resident on texts tensor[offsets[i] : offsets[i] + lens[i]] of a uint8 CUDA tensor.
    -> [(count, [(start, end), ...]), ...], as regex_search_batch on host copies of the texts."""
    L = load()
    base, oarr, larr, n = _resident_args(tensor, offsets, lens)
    counts = (C.c_uint64 * max(n, 1))()
    res = [L.krep_b200_match_result_init(16) for _ in range(n)] if with_result else []
    rarr = (C.POINTER(MatchResult) * max(n, 1))(*res) if with_result else None
    try:
        rc = L.krep_b200_regex_search_batch_resident(params.ref(), base, oarr, larr, n, counts, rarr)
        check(L)
        assert rc == 0, rc
        return [(int(counts[i]), _positions(res[i]) if with_result else []) for i in range(n)]
    finally:
        for r in res:
            L.krep_b200_match_result_free(r)


def batch_resident_stats():
    """(gather_ms, scan_ms, resolve_ms) of the calling thread's most recent resident batch call."""
    L = load()
    g, s, r = C.c_float(), C.c_float(), C.c_double()
    L.krep_b200_batch_resident_stats(C.byref(g), C.byref(s), C.byref(r))
    return g.value, s.value, r.value


def _positions(res):
    r = res.contents
    return [(r.positions[i].start_offset, r.positions[i].end_offset) for i in range(r.count)]


def search_shards(plan, params, shards, with_result=True):
    """krep_b200_search_shards on a list of Shard structs (text order). -> (count, [(start, end), ...])"""
    L = load()
    arr = (Shard * max(len(shards), 1))(*shards)
    res = L.krep_b200_match_result_init(16) if with_result else None
    try:
        cnt = L.krep_b200_search_shards(plan, params.ref(), arr, len(shards), res)
        check(L)
        return int(cnt), (_positions(res) if res else [])
    finally:
        if res:
            L.krep_b200_match_result_free(res)


def regex_resolve(params, rows, with_result=True):
    """krep_b200_regex_resolve over host rows (bytes objects, text order). -> (count, [(start, end), ...])"""
    L = load()
    bufs = [C.create_string_buffer(bytes(r), max(len(r), 1)) for r in rows]
    arr = (C.c_void_p * max(len(rows), 1))(*[C.cast(b, C.c_void_p) for b in bufs])
    res = L.krep_b200_match_result_init(16) if with_result else None
    try:
        cnt = L.krep_b200_regex_resolve(params.ref(), arr, len(rows), res)
        check(L)
        return int(cnt), (_positions(res) if res else [])
    finally:
        if res:
            L.krep_b200_match_result_free(res)


def regex_resolve_part(params, rows, n_own, text_len, last_byte, decides_end, with_result=True):
    """krep_b200_regex_resolve_part over host rows (bytes-like objects, text order): the answer of the lines rows[:n_own]
    own. -> (count, [(start, end), ...])"""
    L = load()
    bufs = [C.create_string_buffer(bytes(r), max(len(r), 1)) for r in rows]
    arr = (C.c_void_p * max(len(rows), 1))(*[C.cast(b, C.c_void_p) for b in bufs])
    res = L.krep_b200_match_result_init(16) if with_result else None
    try:
        cnt = L.krep_b200_regex_resolve_part(params.ref(), arr, len(rows), n_own, text_len, last_byte, int(decides_end), res)
        check(L)
        return int(cnt), (_positions(res) if res else [])
    finally:
        if res:
            L.krep_b200_match_result_free(res)


def regex_row_head(row):
    """krep_b200_regex_row_head: the head-only row of a row (bytes-like). -> bytes"""
    L = load()
    src = C.create_string_buffer(bytes(row), max(len(row), 1))
    n = L.krep_b200_regex_row_head(src, None, 0)
    check(L)
    dst = C.create_string_buffer(n)
    assert L.krep_b200_regex_row_head(src, dst, n) == n
    return dst.raw


def regex_tiling(headers, n):
    """krep_b200_regex_tiling over n row headers packed in `headers` (a buffer address or bytes-like).
    -> (RegexTiling, head_to list, head_bytes list); raises RuntimeError when the rows do not tile one text."""
    L = load()
    if not isinstance(headers, int):
        keep = C.create_string_buffer(bytes(headers), max(len(headers), 1))
        headers = C.addressof(keep)
    out = RegexTiling()
    to = (C.c_int32 * n)()
    nb = (C.c_uint64 * n)()
    rc = L.krep_b200_regex_tiling(C.c_void_p(headers), n, C.byref(out), to, nb)
    if rc != 0:
        raise RuntimeError("krep_b200: " + L.krep_b200_last_error_string().decode())
    return out, list(to), list(nb)
