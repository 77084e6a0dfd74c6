/* krep_b200.h — C ABI of the H100-native scan engine that drops in behind krep's
 * search_func_t boundary.
 *
 * Every entry point below names the reference interface it replaces as
 * (file:line) into davidesantangelo/krep v2.2.0.  The data types are restated
 * byte-for-byte from krep.h:49-101 so that a krep host can pass its own
 * search_params_t / match_result_t straight through; if krep.h was included
 * first (KREP_H defined) the restatement is skipped and krep's own types are used.
 *
 * Nothing in this header mentions torch, CUDA runtime types or C++: plain
 * pointers and sizes only.  Device pointers are passed as const void* and
 * streams as void* (a cudaStream_t).
 */
#ifndef KREP_B200_H
#define KREP_B200_H

#include <stdbool.h>
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ------------------------------------------------------------------------- */
/* Types restated from krep.h (layout-identical; checked by tests/test_abi.py, */
/* which also drives the compiled reference with the very same structs)       */
/* ------------------------------------------------------------------------- */
#ifndef KREP_H

/* krep.h:49-53 */
typedef struct
{
   size_t start_offset; /* first byte of the match, relative to text_start   */
   size_t end_offset;   /* one past the last byte                             */
} match_position_t;

/* krep.h:55-60 — positions must be malloc-family memory (krep.c:244-251)     */
typedef struct match_result_t
{
   match_position_t *positions;
   uint64_t count;
   uint64_t capacity;
} match_result_t;

struct ac_trie;
typedef struct ac_trie ac_trie_t; /* krep.h:22-23, opaque */

/* krep.h:65-94 */
typedef struct search_params
{
   const char *pattern; /* single-literal kernels read these two (krep.c:1271) */
   size_t pattern_len;

   const char **patterns; /* multi-literal kernel reads these three            */
   size_t *pattern_lens;
   size_t num_patterns;

   bool case_sensitive;
   bool use_regex;
   bool count_lines_mode;   /* -c   */
   bool count_matches_mode; /* -co  */
   bool track_positions;    /* !(-c && !-o) */
   bool whole_word;         /* -w   */

   const void *compiled_regex; /* const regex_t* in krep.h; used by krep_b200_regex_search only */
   ac_trie_t *ac_trie;
   size_t max_count; /* SIZE_MAX = unlimited */
} search_params_t;

/* krep.h:98-101 */
typedef uint64_t (*search_func_t)(const search_params_t *params,
                                  const char *text_start,
                                  size_t text_len,
                                  match_result_t *result);
#endif /* KREP_H */

/* ------------------------------------------------------------------------- */
/* Lifetime                                                                  */
/* ------------------------------------------------------------------------- */

/* Make `device` the process's primary CUDA device and create its engine context
 * (streams, result buffers).  Optional: every entry point initialises lazily,
 * with the calling thread's current device as the primary one.  One process can
 * drive several devices: host-text searches spread over the devices chosen by
 * krep_b200_set_devices / KREP_B200_DEVICES (see below), and the resident-shard
 * API runs each shard on the device that owns its memory.  Returns 0, or a
 * negative value after printing "krep: ..." to stderr (the reference's error
 * convention, krep.c:1933).  There is no CPU fallback: without a usable sm_90
 * device every search entry point prints an error and aborts the call with
 * count 0 and krep_b200_last_error() != 0. */
int krep_b200_init(int device);
int krep_b200_device_count(void);          /* CUDA devices visible to the process */
/* Non-blocking: starts CUDA initialisation and the primary device's context on a background thread and returns.  A
 * host calls it as soon as it knows a literal search is coming (krep: after option parsing, before search_file opens
 * and maps the file, krep.c:3818), so the driver start-up overlaps the host's own file handling; the first entry point
 * that needs the GPU waits for it (and meanwhile pre-faults the caller's text with the staging threads). */
void krep_b200_warmup(void);
/* The devices a search_func_t call spreads the caller's text over — the analogue of krep's thread count
 * (krep.c:2851-2905 cuts the file into one chunk per pool thread; here into one contiguous range per GPU, each range
 * streamed over that GPU's own PCIe link and scanned there, per-device occurrence lists merged by key on the host).
 * devices == NULL or n == 0 restores the default: KREP_B200_DEVICES=<count> from the environment, else ONE device (from a
 * pageable file mapping more devices add nothing: the host's page faults and staging copies are the limit; they pay for
 * pinned text).  Start-up note: a process in which this library is the first user of CUDA hides the GPUs it will not use
 * from the driver before CUDA initialises (cuInit enumerates every visible GPU: 6.8 s on an 8-GPU box against 0.4 s for
 * one) — so choose the devices (this call, krep_b200_init, or KREP_B200_DEVICES / KREP_B200_KEEP_VISIBLE in the
 * environment) before the first search. */
void krep_b200_set_devices(const int *devices, int n);
void krep_b200_shutdown(void);
int krep_b200_last_error(void);           /* 0 = last call succeeded          */
const char *krep_b200_last_error_string(void);
const char *krep_b200_version(void);

/* ------------------------------------------------------------------------- */
/* The file-static globals of krep.c that the kernels read (krep.c:117-120). */
/* A host that links this library mirrors its own flags into these.          */
/* ------------------------------------------------------------------------- */
void krep_b200_set_only_matching(bool on); /* -o            krep.c:117 */
bool krep_b200_get_only_matching(void);
void krep_b200_set_force_no_simd(bool on); /* --no-simd     krep.c:118 */
void krep_b200_set_algo_override(const char *name); /* --algo=auto|bm|kmp krep.c:120; NULL = auto */

/* ------------------------------------------------------------------------- */
/* search_func_t replacements (host text in, match_result_t out).            */
/* Each reproduces the count, the offsets and their order of the named       */
/* reference function called once on the whole buffer (krep -t 1 semantics,  */
/* SURVEY §8 a12), including its overlap policy, -w/-c/-m behaviour.          */
/* ------------------------------------------------------------------------- */
uint64_t krep_b200_boyer_moore_search(const search_params_t *, const char *, size_t, match_result_t *);  /* krep.c:1260 */
uint64_t krep_b200_kmp_search(const search_params_t *, const char *, size_t, match_result_t *);          /* krep.c:1628 */
uint64_t krep_b200_memchr_search(const search_params_t *, const char *, size_t, match_result_t *);       /* krep.c:3891 */
uint64_t krep_b200_memchr_short_search(const search_params_t *, const char *, size_t, match_result_t *); /* krep.c:4371 */
uint64_t krep_b200_simd_sse42_search(const search_params_t *, const char *, size_t, match_result_t *);   /* krep.c:4702 */
uint64_t krep_b200_simd_avx2_search(const search_params_t *, const char *, size_t, match_result_t *);    /* krep.c:4877 */
uint64_t krep_b200_simd_avx512_search(const search_params_t *, const char *, size_t, match_result_t *);  /* krep.c:5108 */
uint64_t krep_b200_aho_corasick_search(const search_params_t *, const char *, size_t, match_result_t *); /* aho_corasick.c:299 */
/* the ARM build's kernel; never chosen by krep_b200_select_search_algorithm (which stands in for the x86 AVX2 build) */
uint64_t krep_b200_neon_search(const search_params_t *, const char *, size_t, match_result_t *);          /* krep.c:4506 */
/* -E: regex_search (krep.c:1389).  The GPU flags every line the regex can match in (a byte automaton built from the
 * regex string krep compiles, krep.c:2081-2145, read as a C-locale POSIX ERE under REG_NEWLINE); glibc's regexec on
 * params->compiled_regex (a const regex_t *) then runs on the flagged lines only, clipped to each run of consecutive
 * flagged lines.  Count, offsets, -w / -c / -m and every glibc detail are regexec's own (or, on the two paths below,
 * computed on the GPU and bit for bit the same).  Only for patterns that
 * krep_b200_select_search_algorithm accepts; any other pattern makes this entry fail (count 0, krep_b200_last_error).
 * Accepted: literals and escaped punctuation, '.', bracket expressions with ranges, negation and the classes alpha,
 * digit, alnum, upper, lower, blank, punct, print, graph, xdigit; ^ $ ( ) | * + ? {m} {m,} {m,n} {,n} (counts <= 255);
 * \w; \b \B \< \> (the filter treats them as empty: a wider answer, never a narrower one).
 * -c without -w (count_lines_mode) on a pattern whose line automaton is exact (no word assertion, no -i bracket that
 * case folding widens, no anchor inside a repeated group) is counted on the GPU: lines the automaton decides there are
 * counted in the scan, and regexec sees only the lines it cannot decide (a line longer than the scan's reach, and the
 * text's last line).  The count is the same; KREP_B200_NO_FUSED_COUNT=1 turns this off
 * (krep_b200_regex_count_mode tells which path a call takes).
 * Positions and -co (track_positions without count_lines_mode), without -w, on such a pattern compute their match
 * offsets on the GPU when the pattern's anchored match automaton fits the scan's shared memory next to the line
 * automaton: every line the scan decides is walked again there, leftmost-longest, as the reference's loop walks it,
 * and regexec sees only the lines it cannot decide (those above, and a line whose walk runs over a step budget of a
 * few automaton steps per byte).  Count, positions and their order are the same; KREP_B200_NO_DEVICE_MATCHES=1 turns
 * this off (krep_b200_regex_match_mode tells which path a call takes).
 * Refused (the pattern stays with the host's regex_search): back-references, \` \', \s \S \W, [[:space:]],
 * [[:cntrl:]], collating elements, any character set that holds '\n' or a newline in the pattern, non-ASCII pattern
 * bytes, unknown escapes, a process running in a multibyte locale (krep itself never calls setlocale), and automata
 * above 4096 states or 32 KiB of transition table (or 8192 NFA states, or 255 byte classes).  A regex whose top level
 * is an alternation (krep's (p1)|...|(pk) of several -e or -f patterns, or one pattern with a top-level |) and whose
 * one automaton is too large is split instead: its branches, in order, go to up to 8 automata that the scan walks
 * together (a split plan).  The size refusal then applies to a single branch that no automaton holds, and to sets whose
 * automata need more than 224 KiB of shared memory together (about 500 patterns of 8-12 lowercase letters); a split
 * plan computes offsets on the GPU only when its match automata fit in the same 224 KiB as well. */
uint64_t krep_b200_regex_search(const search_params_t *, const char *, size_t, match_result_t *);

/* Many texts, one launch — what search_directory_recursive (krep.c:3310) calling search_file once per small file
 * becomes when the per-call copy and launch latency matters.  `entry` is one of the literal and pattern-set functions
 * above (not krep_b200_regex_search, which is refused with an error: -E batches go through
 * krep_b200_regex_search_batch); text i gets
 * exactly the count (counts[i]) and positions (results[i], may be NULL, or results == NULL) that
 * entry(params, texts[i], lens[i], results[i]) would have produced.  Returns 0, or a negative error. */
int krep_b200_search_batch(search_func_t entry, const search_params_t *params, const char *const *texts,
                           const size_t *lens, size_t n_texts, uint64_t *counts, match_result_t *const *results);

/* -E over many texts in one pack, one copy and one scan.  For every i, counts[i] and results[i] (results or results[i]
 * may be NULL) are exactly what krep_b200_regex_search(params, texts[i], lens[i], results[i]) returns: the count, the
 * positions and their order, on each of its three paths (fused -c, offsets on the GPU, line filter + regexec), chosen
 * once per call from params and switched by the same KREP_B200_NO_FUSED_COUNT / KREP_B200_NO_DEVICE_MATCHES.  Per text:
 * its own -m budget, -w, -i, -c, -co, and the early returns (max_count == 0, no compiled_regex, the empty text), which
 * are answered on the host without a launch.  The texts are packed at 16-byte aligned offsets with '\n' gaps, so no line
 * crosses from one text into the next; every text still costs at least one regexec call on its last line on the -c and
 * offsets paths.  Lines longer than the line kernel's reach are decided on the GPU by the long-line pass, as in
 * krep_b200_regex_search, except each text's last line and lines cut by a chunk edge; KREP_B200_NO_LONG_LINES=1 leaves
 * them to regexec.  A pattern krep_b200_regex_search refuses fails the call with -3 and every count 0.  Returns 0, or a
 * negative error. */
int krep_b200_regex_search_batch(const search_params_t *params, const char *const *texts, const size_t *lens,
                                 size_t n_texts, uint64_t *counts, match_result_t *const *results);
/* Host-clock times of the calling thread's most recent krep_b200_regex_search_batch: packing the texts (with the text
 * table) and the per-text replays.  The scan itself is krep_b200_last_kernel_ms. */
void krep_b200_regex_batch_stats(double *pack_ms, double *resolve_ms);

/* Many texts that already live in HBM, one call (DESIGN §12.9): text i is d_base[offsets[i] .. offsets[i] + lens[i]).
 * d_base is device memory of one CUDA device, of any alignment (a torch tensor with a storage offset is fine); offsets
 * and lens are host arrays; texts may come in any order, overlap or repeat.  counts[i] and results[i] are exactly what
 * krep_b200_search_batch / krep_b200_regex_search_batch return for host copies of the same texts, with the same knobs.
 * The texts are gathered on the device that owns d_base into one packed buffer (the host batch's layout), scanned there
 * as one shard and resolved per text on the host from the keys (and, for -E, from one row of the lines glibc must
 * see), so no text is copied to the host.  The packed buffer needs about the texts' total size in extra HBM; it is kept
 * across calls and grown on demand, and a batch that cannot get it fails with -2.  Errors: -3 for a refused regex
 * (every count 0), krep_b200_regex_search as entry (or any foreign entry), a d_base that is not device memory, or
 * a span from the lowest text start to the highest text end that is not all mapped device memory; -2 for CUDA failures.
 * The texts are read on the library's own stream: work that writes them on another stream must be complete before the
 * call (synchronise that stream or the device).  Speed on an H100: README (bench_batch_resident.py). */
int krep_b200_search_batch_resident(search_func_t entry, const search_params_t *params, const void *d_base,
                                    const uint64_t *offsets, const size_t *lens, size_t n_texts, uint64_t *counts,
                                    match_result_t *const *results);
int krep_b200_regex_search_batch_resident(const search_params_t *params, const void *d_base, const uint64_t *offsets,
                                          const size_t *lens, size_t n_texts, uint64_t *counts,
                                          match_result_t *const *results);
/* Times of the calling thread's most recent resident batch call: the gather kernel and the scan (with its sort and, for
 * -E, the row pack) in device time, and the per-text replays on the host clock. */
void krep_b200_batch_resident_stats(float *gather_ms, float *scan_ms, double *resolve_ms);
/* Test hook: the packed buffer of a resident batch.  gap_kind 0: zero gaps of at least max_gap + 16 bytes (the literal
 * and pattern-set batch, max_gap = the longest pattern); 1: '\n' gaps of at least one byte (the -E batch).  With base in
 * device memory the texts are gathered by k_batch_gather; with base in host memory the host batch's own pack builds the
 * buffer instead, for comparison.  Copies min(total, cap) bytes to dst_host and returns the total, or a negative error.
 * No search entry point calls it. */
int64_t krep_b200_batch_gather_raw(const void *base, const uint64_t *offsets, const size_t *lens, size_t n, int gap_kind,
                                   size_t max_gap, void *dst_host, uint64_t cap);

/* krep.c:1771 — same decision order, same globals.  For use_regex it returns
 * krep_b200_regex_search when the pattern's line automaton compiles, and
 * NULL when it is refused (the caller keeps its own regex_search then). */
search_func_t krep_b200_select_search_algorithm(const search_params_t *params);
/* krep.c:1964 */
const char *krep_b200_get_algorithm_name(search_func_t func);

/* aho_corasick.c:111 / 274 / 287.  The returned object is this library's own
 * device automaton (patterns folded, filter tables and verify tables resident
 * in HBM); krep_b200_aho_corasick_search also accepts a params->ac_trie that
 * was built by the reference's ac_trie_build (it only tests it for NULL, as
 * aho_corasick.c:306 does) and then compiles and caches its own automaton
 * from params->patterns. */
ac_trie_t *krep_b200_ac_trie_build(const search_params_t *params);
void krep_b200_ac_trie_free(ac_trie_t *trie);
bool krep_b200_ac_trie_root_has_outputs(const ac_trie_t *trie);

/* krep.c:139 / 175 / 244 / 256 — for hosts that do not link krep.c. */
match_result_t *krep_b200_match_result_init(uint64_t initial_capacity);
bool krep_b200_match_result_add(match_result_t *result, size_t start_offset, size_t end_offset);
void krep_b200_match_result_free(match_result_t *result);
bool krep_b200_match_result_merge(match_result_t *dest, const match_result_t *src, size_t chunk_offset);

/* ------------------------------------------------------------------------- */
/* HBM-resident shard API — what search_chunk_thread (krep.c:1919) becomes   */
/* when the chunk already lives on the GPU: one shard per device, owned      */
/* range + halo, matches owned by start offset (SURVEY §8e).                 */
/* ------------------------------------------------------------------------- */

/* Emulated reference kernel: selects the overlap / -w / -m policy applied to
 * the raw occurrence list. */
enum
{
   KREP_B200_ALGO_BMH = 0,          /* boyer_moore_search  krep.c:1260 */
   KREP_B200_ALGO_KMP = 1,          /* kmp_search          krep.c:1628 */
   KREP_B200_ALGO_MEMCHR = 2,       /* memchr_search       krep.c:3891 */
   KREP_B200_ALGO_MEMCHR_SHORT = 3, /* memchr_short_search krep.c:4371 */
   KREP_B200_ALGO_SSE42 = 4,        /* simd_sse42_search   krep.c:4702 */
   KREP_B200_ALGO_AVX2 = 5,         /* simd_avx2_search    krep.c:4877 */
   KREP_B200_ALGO_AVX512 = 6,       /* simd_avx512_search  krep.c:5108 */
   KREP_B200_ALGO_AC = 7,           /* aho_corasick_search aho_corasick.c:299 */
   KREP_B200_ALGO_NEON = 8,         /* neon_search         krep.c:4506 */
   KREP_B200_ALGO_REGEX = 9         /* regex_search        krep.c:1389: keys are flagged line starts */
};

typedef struct krep_b200_plan krep_b200_plan_t; /* compiled pattern set, device-resident */

/* Compile params->pattern (literal algos), params->patterns[] (algo == AC) or the
 * regex krep compiles from params->patterns[] (algo == REGEX) into filter
 * constants / tables on the current device. NULL on error (or refused regex).
 * A REGEX plan's scan emits one key per line the regex may match in,
 * (global line start << 3); lines longer than about 4 KiB past a thread's
 * 256-byte segment, or cut by the shard's end, are flagged without a verdict.
 * Such keys are confirmed by krep_b200_replay(KREP_B200_ALGO_REGEX, ...) with
 * the host text, or, for resident shards without one, by
 * krep_b200_search_shards (krep_b200_regex_export_shard + _regex_resolve);
 * krep_b200_collect refuses regex plans. */
krep_b200_plan_t *krep_b200_plan_create(const search_params_t *params, int algo);
void krep_b200_plan_destroy(krep_b200_plan_t *plan);
/* Which device filter the plan uses (for bench/config reporting). */
const char *krep_b200_plan_filter_name(const krep_b200_plan_t *plan);

/* One shard of a corpus that is resident in device memory. */
typedef struct
{
   const void *d_text;     /* device pointer, 16-byte aligned                       */
   uint64_t avail_len;     /* bytes readable at d_text: owned range + halo            */
   uint64_t own_begin;     /* report matches whose start is in [own_begin, own_end)   */
   uint64_t own_end;       /*   (offsets relative to d_text)                          */
   uint64_t global_offset; /* added to every reported offset                          */
   int32_t prev_byte;      /* byte preceding d_text[0] in the whole text, -1 = none   */
   int32_t next_byte;      /* byte following d_text[avail_len-1], -1 = end of text    */
} krep_b200_shard_t;

/* Result of a device scan, left in device memory (sorted ascending). */
typedef struct
{
   uint64_t count;          /* occurrences found (exact even if capacity was exceeded) */
   uint64_t stored;         /* entries actually stored = min(count, capacity)           */
   const uint64_t *d_keys;  /* device: literal: start offset (global); AC: packed key   */
   int overflow;            /* 1 if count > capacity: call again with a larger capacity */
   uint64_t text_len;       /* global_offset + avail_len of the scanned shard: the length of the whole text when
                               the shard is the last (or only) one — what the window kernels' tail logic needs */
   const uint64_t *d_line_bounds; /* device, 2 words per stored key, only for plans created with count_lines_mode (-c):
                               global offset of the first byte of the occurrence's line, and of the line's newline (or
                               the text length) — find_line_start / find_line_end (krep.c:363, 401) computed on the GPU */
   int32_t device;          /* CUDA device that holds the lists                                                      */
   int32_t slot;            /* which of the device's result buffers the scan used                                    */
   uint64_t serial;         /* scan number on that device: the lists stay valid until the next scan of that device   */
} krep_b200_device_result_t;

/* Scan one shard on `stream` (cudaStream_t, NULL = engine stream) of the device that owns shard->d_text: launches
 * the filter+verify kernel and sorts the occurrence list on the device (lists of up to 16 384 occurrences by the
 * one-CTA finish kernel, which also hands count and list to the host in the scan's single synchronisation; longer
 * ones by a radix sort that is still running on `stream` when the call returns — krep_b200_collect /
 * krep_b200_export_* order themselves after it). For a
 * literal plan every key is (global start offset << 3 | tag bits) of one occurrence
 * that passed the plan's -w filter (tags: see csrc/common.h).  For an AC plan every key packs
 * (end_offset << 24 | (1023 - (len-1)) << 10 ... see krep_b200_ac_key_* below) so
 * that ascending key order is aho_corasick_search's emission order.
 * `want_positions` = 0 counts only (no list is written).
 * Blocks until the count is known. Returns 0 or a negative error. */
int krep_b200_scan_shard(const krep_b200_plan_t *plan, const krep_b200_shard_t *shard,
                         int want_positions, void *stream, krep_b200_device_result_t *out);
/* The same scan in two halves: _begin enqueues it and returns a ticket without waiting, _end waits for it.  A host
 * that has work of its own per scan (rank 0 of a multi-GPU job replaying the previous step's gathered list) does it
 * between the two.  At most two scans per device may be in flight, and _end only waits for its own scan: a host that
 * begins scan i+1 before it ends scan i keeps the GPU busy back to back (lists of up to 16 384 occurrences, which come
 * back through pinned memory; a longer list must be ended before the next scan begins). */
int krep_b200_scan_shard_begin(const krep_b200_plan_t *plan, const krep_b200_shard_t *shard,
                               int want_positions, void *stream, int *ticket);
int krep_b200_scan_shard_end(int ticket, krep_b200_device_result_t *out);

/* Copy the first min(out->stored, max_keys) sorted keys of a shard result into another device
 * buffer (device-to-device, on `stream`), e.g. a torch tensor that is then gathered with NCCL. */
int krep_b200_export_keys(const krep_b200_device_result_t *dev, void *d_dst, uint64_t max_keys, void *stream);
/* The row a multi-GPU host gathers: d_dst[0] = the shard's exact occurrence count, d_dst[1..] = its first
 * min(stored, max_keys) sorted keys — one device-to-device copy on `stream`. */
int krep_b200_export_packed(const krep_b200_device_result_t *dev, void *d_dst, uint64_t max_keys, void *stream);
/* The same row for a scan that is still in flight (its ticket): enqueued on the scan's stream behind the finish kernel,
 * always the whole fixed-size row (max_keys <= 16384); a longer list arrives as count > max_keys. */
int krep_b200_export_packed_async(int ticket, void *d_dst, uint64_t max_keys);
/* Merge step of a sharded search (krep.c:2928-3004 without its chunk-edge artefacts): n_lists ascending key lists
 * (one per shard, shards in text order) -> one ascending list in dst (room for the sum of counts; may alias the
 * first list).  Literal keys (ordered and owned by start offset) are already globally ordered after concatenation;
 * pattern-set keys are ordered by END offset (aho_corasick.c:353-431) but owned by START offset, so around every cut
 * a long match owned by the earlier shard can end after a short match owned by the later one — the merge puts them
 * back into emission order.  Returns the total. */
uint64_t krep_b200_merge_keys(const uint64_t *const *lists, const uint64_t *counts, uint32_t n_lists, uint64_t *dst);

/* Timing hook for bench.py: device time in milliseconds of the scan kernel(s)
 * of the most recent krep_b200_scan_shard / search call on this thread,
 * measured with CUDA events on the launching stream (kernel only, no sort). */
float krep_b200_last_kernel_ms(void);
/* Number of launches of this library's own (hand-written) kernels since the last reset; the CUB radix-sort
 * launches behind krep_b200_scan_shard are library code and are not included. */
uint64_t krep_b200_launch_count(void);
void krep_b200_reset_launch_count(void);

/* Fused -c (count_lines_mode): the lines that hold an occurrence are counted on the device, so only this record leaves
 * the GPU.  Single literals count in the scan itself (krep.c:1331-1351 and the equivalent branches of the other literal
 * kernels); pattern sets (aho_corasick.c:390-403) count from their sorted occurrence keys, which stay on the device, and a
 * shard whose occurrences overflow the occurrence list is counted in pieces instead of growing the list.
 * A shard that cuts lines still gives an exact total: records of shards in text order are folded with
 * krep_b200_combine_line_counts, which subtracts a line counted on both sides of a cut. */
typedef struct
{
   uint64_t lines;    /* lines of this shard that hold an occurrence it owns                                     */
   uint32_t flags;    /* KREP_B200_LINES_*                                                                        */
   uint32_t reserved;
} krep_b200_line_count_t;
enum
{
   KREP_B200_LINES_HAS_HIT = 1,      /* the shard owns at least one occurrence                                       */
   KREP_B200_LINES_FIRST_OPEN = 2,   /* its first occurrence lies before its first newline (the line began earlier)  */
   KREP_B200_LINES_LAST_PENDING = 4, /* no newline between its last occurrence and its end (the line goes on)         */
   KREP_B200_LINES_HAS_NL = 8        /* the shard holds a newline (computed for shards without an occurrence)         */
};
/* Plans created from params with count_lines_mode set, single literals and pattern sets; not for needles of 17..64 bytes
 * taken by the window kernels, patterns containing a newline (a set with one such pattern) or -w plans in tag mode (those
 * need krep_b200_scan_shard + krep_b200_collect): returns -3 for them.  A pattern set's call waits for its scan's
 * occurrence count before it enqueues the count itself, and fails with -3 while both scan slots of the device are held
 * by krep_b200_scan_shard_begin. */
int krep_b200_count_lines_shard(const krep_b200_plan_t *plan, const search_params_t *params, const krep_b200_shard_t *shard,
                                void *stream, krep_b200_line_count_t *out);
uint64_t krep_b200_combine_line_counts(const krep_b200_line_count_t *recs, size_t n, size_t max_count);

/* Apply the emulated reference kernel's policy (overlap rule, -w, -c, -m) to a
 * shard result and deliver it as krep's match_result_t (host, malloc memory).
 * Count-lines mode (-c) uses the line bounds the scan computed on the device
 * (plan created from params with count_lines_mode set, single shard: the
 * shard must not cut a line, i.e. prev_byte = next_byte = -1 or newline-aligned).
 * Returns the count the reference would return.  Regex plans are refused (error -3): a device result does not carry
 * its shard's text, which glibc needs; use krep_b200_search_shards. */
uint64_t krep_b200_collect(const krep_b200_plan_t *plan, const search_params_t *params,
                           const krep_b200_device_result_t *dev, match_result_t *result);

/* Several resident shards (text order; on one GPU or spread over the GPUs of this process), one answer: search_file's
 * chunk loop and merge (krep.c:2851-3004) for text that already lives in HBM.  Shards on distinct devices are scanned
 * concurrently, the per-shard lists merged by key, and the policy replayed ONCE over the whole list, so overlap rules,
 * -m and the emission order are those of the reference's single-chunk run.  -c is answered by the fused line count
 * (single literals and pattern sets without a newline in a pattern; line cuts between shards are resolved, shards on
 * distinct devices are counted concurrently).
 *
 * Regex plans (-E): returns the count and positions krep_b200_regex_search(params, text, n, result) returns on the text
 * the shards hold — the same path (fused -c, offsets on the device, or the line filter + regexec), the same knobs
 * (KREP_B200_NO_FUSED_COUNT, KREP_B200_NO_DEVICE_MATCHES), the same early returns and -m / -w / -i / -o / -c behaviour —
 * without a host copy of the text: each shard's row (krep_b200_regex_export_shard) brings back the bytes of the lines
 * glibc must see, and krep_b200_regex_resolve answers from the rows.  The shards must tile one whole text: the first
 * has global_offset + own_begin == 0 and prev_byte == -1, consecutive owned ranges abut, the last has next_byte == -1
 * and own_end == avail_len; any other geometry fails with error -3.  The halo (avail_len - own_end) may be anything
 * from 0: a smaller one only leaves more lines to glibc.  Offsets on the device keep the match keys' limit: a call that
 * takes that path fails with error -3 when a shard ends at or beyond 2^48 bytes of global offset (set
 * KREP_B200_NO_DEVICE_MATCHES for the filter path there). */
uint64_t krep_b200_search_shards(const krep_b200_plan_t *plan, const search_params_t *params,
                                 const krep_b200_shard_t *shards, uint32_t n_shards, match_result_t *result);

/* -E over resident shards in two steps, so that one code path serves one process and several ranks (each rank exports
 * its shard's row and resolves its own lines with krep_b200_regex_resolve_part below; rank 0 gathers the answers).
 * krep_b200_regex_export_shard: one k_regex_lines scan of the shard in the mode krep_b200_regex_search would use for
 * params, then the pack kernels: the shard's row (layout: csrc/common.h, RegexRowHeader) in engine-owned device memory
 * of the shard's device — *d_row (may be NULL), valid until the next export on that device — and *row_bytes.  When dst
 * is not NULL the row is also copied there (host or device memory, dst_cap bytes of room; -5 and nothing copied when
 * the row does not fit).  Work queued on `stream` (may be NULL) is waited for first.  Returns 0 or a negative error. */
int krep_b200_regex_export_shard(const krep_b200_plan_t *plan, const search_params_t *params, const krep_b200_shard_t *shard,
                                 void *stream, void *dst, uint64_t dst_cap, uint64_t *row_bytes, const void **d_row);
/* The answer of the search from the rows (host memory, text order) of shards that tile the text: what
 * krep_b200_search_shards returns.  Host only; 0 with error -3 when the rows are not rows of one tiling. */
uint64_t krep_b200_regex_resolve(const search_params_t *params, const void *const *rows, uint32_t n_rows, match_result_t *result);
/* -E over shards resident on several ranks (one process per GPU, krep_b200/sharding.py; DESIGN §12.6): each rank resolves
 * the lines its own shard owns, and only counts and positions travel.
 * krep_b200_regex_resolve_part: the answer of the lines owned by rows[0 .. n_own) — consecutive shards of one tiling of
 * a text of text_len bytes whose last byte is last_byte (-1 when empty) — capped at params->max_count.
 * rows[n_own .. n_rows) are the shards that follow, in order; only their heads are read (full rows or head-only rows).
 * decides_end: this part decides the end of the text (the empty string at text_len); exactly one part of a tiling does,
 * the owner of the last line start (krep_b200_regex_tiling's decider).  Each part's answer is the first max_count items
 * of its unbounded answer, so the search's answer is the parts' positions concatenated in text order and cut to
 * max_count, with count min(sum of counts, max_count).  krep_b200_regex_resolve is the case n_own == n_rows,
 * decides_end = 1.  Same early returns as krep_b200_regex_resolve; 0 with error -3 when the rows are not consecutive
 * shards of such a text or a line the part owns runs past the heads it is given. */
uint64_t krep_b200_regex_resolve_part(const search_params_t *params, const void *const *rows, uint32_t n_rows, uint32_t n_own,
                                      uint64_t text_len, int last_byte, int decides_end, match_result_t *result);
/* A head-only row: the row's header with nkeys = nseg = 0, followed by its head.  Returns its size, or the size needed
 * (nothing copied) when dst is NULL or cap is too small; 0 with error -3 when row is not a regex row. */
uint64_t krep_b200_regex_row_head(const void *row, void *dst, uint64_t cap);
/* A row's header: its first KREP_B200_REGEX_ROW_HEADER bytes, all that krep_b200_regex_tiling reads. */
#define KREP_B200_REGEX_ROW_HEADER 128
typedef struct
{
   uint64_t text_len;  /* the text the rows tile                                                                  */
   int32_t last_byte;  /* its last byte, -1 when it is empty                                                      */
   uint32_t decider;   /* the shard that decides the end of the text: the last one that holds a line start (0 for
                          the empty text)                                                                         */
} krep_b200_regex_tiling_t;
/* The geometry of n rows' headers (shard i's at i * KREP_B200_REGEX_ROW_HEADER bytes, text order): whether they tile
 * one text — the first owns from 0 at a line start, owned ranges abut, the last ends the text, and only empty shards
 * follow a shard that ends it — and which part reads which head.  A shard holds a line start when it is not empty and
 * either starts at one (no head) or its head ends before its owned range does.  head_to[i] (may be NULL): the shard
 * whose part reads shard i's head — the last earlier shard that holds a line start, the owner of the line shard i's
 * head continues — or -1 when shard i has no head; head_bytes[i] (may be NULL): the size of shard i's head-only row
 * (krep_b200_regex_row_head), 0 when it sends none.  Returns 0, or -3 when the rows do not tile one text. */
int krep_b200_regex_tiling(const void *headers, uint32_t n, krep_b200_regex_tiling_t *out, int32_t *head_to,
                           uint64_t *head_bytes);
/* Timing of the most recent krep_b200_search_shards (regex plan) or krep_b200_regex_export_shard call on this thread,
 * summed over its shards: device ms of the scans (with their sort) and of the pack kernels, and the row bytes. */
void krep_b200_regex_export_stats(float *scan_ms, float *pack_ms, uint64_t *packed_bytes);

/* Policy replay over a caller-supplied, ascending occurrence-key list in HOST memory (what
 * krep_b200_collect does after reading the device list back).  A multi-GPU host gathers the
 * per-shard lists, merges them with krep_b200_merge_keys and calls this once.  `text` may be NULL unless params->count_lines_mode is set; `text_len` (the length of the
 * whole text) may be 0 = unknown, except for the AVX2 / AVX-512 window kernels with needles > 16 bytes, whose tail
 * handling (krep.c:5059, 5260) depends on it.
 * `algo` is a KREP_B200_ALGO_* value; `only_matching` is the -o global to emulate. */
uint64_t krep_b200_replay(int algo, const search_params_t *params, bool only_matching,
                          const uint64_t *keys, uint64_t nkeys,
                          const char *text, size_t text_len, match_result_t *result);
/* (KREP_B200_ALGO_REGEX: `keys` are flagged line starts of the whole text, `text` / `text_len` the whole host text —
 * required — and glibc's regexec on params->compiled_regex decides every match, exactly as krep_b200_regex_search.) */

/* Test hook, host only: runs the line automaton that krep_b200_regex_search would use for params over `text` on the
 * CPU (no long-line bound) and stores the start offsets of the flagged lines in line_starts[0 .. min(result, cap)).
 * Returns the number of flagged lines, or -1 when the pattern is refused.  *widened (may be NULL) = 1 when the
 * automaton accepts more than the regex.  No search entry point calls it. */
int64_t krep_b200_regex_filter_host(const search_params_t *params, const char *text, size_t n, uint64_t *line_starts,
                                    uint64_t cap, int *widened);

/* Test hook: which path a -E -c call with params takes — 1 when it is a -c call counted on the device (see
 * krep_b200_regex_search), 0 when its lines go through regexec (every call that is not such a -c call), -1 when the
 * pattern is refused. */
int krep_b200_regex_count_mode(const search_params_t *params);
/* Test hook, host only: the fused -E -c on the CPU — the line automaton decides every line it can within `reach` bytes
 * of the line's start (UINT64_MAX: no bound), and the lines it leaves uncertain (out of reach, or holding the text's
 * last byte) go to regexec as in krep_b200_regex_search.  Returns the count, or -1 when the pattern is refused or a
 * -c call with params would not be counted on the device whatever KREP_B200_NO_FUSED_COUNT says. */
int64_t krep_b200_regex_count_host(const search_params_t *params, const char *text, size_t n, uint64_t reach);
/* Test hook: where a -E positions or -co call with params gets its offsets — 1 when the device computes them (see
 * krep_b200_regex_search), 0 when they come from regexec, -1 when the pattern is refused. */
int krep_b200_regex_match_mode(const search_params_t *params);
/* Test hook, host only: device offsets on the CPU — the line automaton decides every line it can within `reach` bytes
 * of the line's start (UINT64_MAX: no bound), the match automaton enumerates the matches of each line decided MATCHED
 * within the same step budget as the scan, and the lines left uncertain go to regexec as in krep_b200_regex_search.
 * Fills res (may be NULL) and returns the count, or -1 when the pattern is refused or a call with params would not
 * compute its offsets on the device whatever KREP_B200_NO_DEVICE_MATCHES says. */
int64_t krep_b200_regex_matches_host(const search_params_t *params, const char *text, size_t n, uint64_t reach,
                                     match_result_t *res);
/* Test hook: one k_regex_lines scan of a resident shard in `mode` (0 = line filter, 1 = fused -c count,
 * 2 = match offsets). The keys, sorted ascending, go to keys[0 .. min(result, cap)), in the layout of that mode
 * (csrc/common.h). *device_lines (may be NULL) receives the count mode's counter of lines decided MATCHED (0 in the
 * other modes). Returns the exact number of keys, or a negative error. Errors: plan not a regex plan; mode 1 on a plan
 * that is not count_exact; mode 2 on a plan that is not offsets_exact; global_offset + avail_len >= 2^48 in mode 2.
 * No search entry point calls it. */
int64_t krep_b200_regex_scan_shard_raw(const krep_b200_plan_t *plan, const krep_b200_shard_t *shard, int mode,
                                       uint64_t *keys, uint64_t cap, uint64_t *device_lines);
/* Test hook: krep_b200_regex_scan_shard_raw followed by the long-line pass of the search entry points (DESIGN §12.8):
 * the uncertain keys of lines whose '\n' lies beyond the kernel's reach but within avail_len (not the text's last line,
 * shorter than 2^30 bytes) are decided on the device as the kernel would with unbounded reach.  slice_bytes and
 * ckpt_bytes set the slice and checkpoint sizes (0: the production 4096 / 256); the output does not depend on them.
 * Under KREP_B200_NO_LONG_LINES=1 it returns what krep_b200_regex_scan_shard_raw returns.  Errors as that hook's, and
 * -3 for sizes outside 1 <= ckpt_bytes <= slice_bytes <= 2^20 with at most 1024 checkpoints per slice. */
int64_t krep_b200_regex_scan_shard_long_raw(const krep_b200_plan_t *plan, const krep_b200_shard_t *shard, int mode,
                                            uint32_t slice_bytes, uint32_t ckpt_bytes, uint64_t *keys, uint64_t cap,
                                            uint64_t *device_lines);
/* Test hook: how many automata the -E plan of params has — G >= 2 for a split plan (see krep_b200_regex_search), 1 for
 * a plan of one automaton, -1 when the pattern is refused. */
int krep_b200_regex_automata(const search_params_t *params);
/* Test hook: a -E plan of params compiled with a cap of max_states (3 .. 4096) states per automaton instead of 4096,
 * so that small regexes with a top-level alternation become split plans.  The plan is not cached and no search entry
 * point uses it; scan it with krep_b200_regex_scan_shard_raw, run it with krep_b200_regex_plan_host, and free it with
 * krep_b200_plan_destroy.  NULL (error -3) when the regex is refused under that cap. */
krep_b200_plan_t *krep_b200_regex_plan_split(const search_params_t *params, uint32_t max_states);
/* Test hook, host only: the host twin of one krep_b200_regex_scan_shard_raw scan of the whole `text` (one shard from
 * offset 0, nothing after it) with `plan`, every line walked at most `reach` bytes (UINT64_MAX: no bound) in modes 1
 * and 2; mode 0 has no bound.  Keys, in the layout of the mode, sorted, go to keys[0 .. min(result, cap)) and
 * *device_lines (may be NULL) gets the count mode's lines decided MATCHED.  Returns the number of keys, or -3 when the
 * plan does not admit the mode. */
int64_t krep_b200_regex_plan_host(const krep_b200_plan_t *plan, int mode, const char *text, size_t n, uint64_t reach,
                                  uint64_t *keys, uint64_t cap, uint64_t *device_lines);
/* Test hook: one batch scan of krep_b200_regex_search_batch in `mode` (0, 1, 2 as above) over the texts with lens[i] > 0.
 * offsets[i] (may be NULL): text i's packed offset (UINT64_MAX for a text not packed); keys[0 .. min(result, cap)):
 * the sorted keys in packed coordinates; text_lines[i] (may be NULL): in mode 1 the lines of text i decided MATCHED on
 * the device (else 0).  Returns the exact number of keys, or a negative error (refused pattern, or a mode the pattern
 * does not admit).  No search entry point calls it. */
int64_t krep_b200_regex_search_batch_raw(const search_params_t *params, const char *const *texts, const size_t *lens,
                                         size_t n_texts, int mode, uint64_t *offsets, uint64_t *keys, uint64_t cap,
                                         uint64_t *text_lines);
/* Test hook: krep_b200_regex_search_batch_raw followed, after each chunk's scan, by the long-line pass of
 * krep_b200_regex_search_batch (DESIGN §12.8) in the batch rules: a line is taken when its '\n' lies beyond the
 * kernel's reach but within the chunk's readable bytes, it is not its own text's last line, and it is shorter than 2^30
 * bytes.  In mode 1 its count goes to its text's text_lines.  slice_bytes and ckpt_bytes as for
 * krep_b200_regex_scan_shard_long_raw (0: the production 4096 / 256); the output does not depend on them.  Under
 * KREP_B200_NO_LONG_LINES=1 it returns what krep_b200_regex_search_batch_raw returns.  Errors as that hook's, and -3 for
 * the sizes krep_b200_regex_scan_shard_long_raw refuses. */
int64_t krep_b200_regex_search_batch_long_raw(const search_params_t *params, const char *const *texts, const size_t *lens,
                                              size_t n_texts, int mode, uint32_t slice_bytes, uint32_t ckpt_bytes,
                                              uint64_t *offsets, uint64_t *keys, uint64_t cap, uint64_t *text_lines);

/* The same replay without any host text: `bounds` holds two words per key — the global offset of the first byte of
 * the occurrence's line and of that line's newline (or the text length) — as krep_b200_scan_shard computes them on
 * the device for -c plans (krep_b200_device_result_t.d_line_bounds, markers resolved).  A host that gathers keys from
 * several newline-aligned shards gathers the bounds with them. */
uint64_t krep_b200_replay_lines(int algo, const search_params_t *params, bool only_matching,
                                const uint64_t *keys, uint64_t nkeys, const uint64_t *bounds,
                                size_t text_len, match_result_t *result);

/* AC key layout helpers */
uint64_t krep_b200_ac_key_end(uint64_t key);
uint64_t krep_b200_ac_key_start(uint64_t key);
uint32_t krep_b200_ac_key_pattern(uint64_t key);

/* ------------------------------------------------------------------------- */
/* Synthetic corpus (SURVEY §8d): byte[i] is a pure function of (seed, i), so */
/* any shard can be materialised in place on any GPU without transfers.      */
/* ------------------------------------------------------------------------- */
typedef struct
{
   uint64_t seed;            /* text seed                                          */
   uint64_t plant_seed;      /* needle placement seed                              */
   uint64_t plant_period;    /* one planted needle per this many bytes (0 = none)  */
   const char *needle;       /* host pointer, needle_len bytes (copied)            */
   uint32_t needle_len;      /* <= 64                                              */
   uint32_t flags;           /* KREP_B200_CORPUS_*                                 */
} krep_b200_corpus_spec_t;

enum
{
   KREP_B200_CORPUS_RANDOM_CASE = 1, /* planted needles get per-letter pseudo-random case   */
   KREP_B200_CORPUS_EMBED_HALF = 2   /* odd-numbered plants are glued inside a longer word  */
};

/* Fill d_dst[0..len) with corpus bytes [global_offset, global_offset+len). */
int krep_b200_corpus_generate(const krep_b200_corpus_spec_t *spec, void *d_dst,
                              uint64_t global_offset, uint64_t len, void *stream);
/* Host twin of the generator (same bytes), for tests and the CPU baseline. */
int krep_b200_corpus_generate_host(const krep_b200_corpus_spec_t *spec, void *dst,
                                   uint64_t global_offset, uint64_t len);

#ifdef __cplusplus
}
#endif
#endif /* KREP_B200_H */
