// common.h — internal declarations shared by the engine's translation units.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stddef.h>
#include <string>
#include <vector>
#include "../../include/krep_b200.h"

namespace kb {

// ---------------------------------------------------------------------------------------------
// Occurrence keys.  Every occurrence the device reports is one 64-bit key; ascending key order is
// the order the emulated reference kernel would have produced.
//   literal plans : key = (global_start << 3) | (full << 2) | (ws_ok << 1) | we_ok
//                   full  = all pattern_len bytes match (always 1 unless the plan emits prefix hits,
//                           which only memchr_short_search's -o walk needs, krep.c:4495)
//                   ws_ok / we_ok = the two halves of is_whole_word_match(start, start+len) (krep.h:312):
//                           no word character before the start / after the end — both 1 when -w is off.
//                           Kept apart because the tail sub-search of simd_avx2_search / simd_avx512_search
//                           (krep.c:5068, 5268) cannot see the byte before its sub-buffer.
//   AC plans      : key = (global_end << 24) | ((1023 - (len-1)) << 14) | pattern_index
//                   (end ascending, then longest first, then pattern-list order: aho_corasick.c:353-431)
// ---------------------------------------------------------------------------------------------
static constexpr int LIT_TAG_BITS = 3;
static constexpr int AC_END_SHIFT = 24;
static constexpr int AC_LEN_SHIFT = 14;
static constexpr uint32_t AC_MAX_PATTERNS = 1u << 14;

enum FilterKind : int
{
    FILTER_ALIGNED4 = 0, // pattern_len >= 7: every occurrence contains one aligned 32-bit word; test each
                         // aligned text word against the 4 pattern words P[d..d+4), d = 0..3
    FILTER_WINDOW4 = 1,  // pattern_len < 7 (or prefix plans): test the 4-byte window at every byte offset
};

struct LitDevParams
{
    const uint8_t *text; // 16-byte aligned
    uint64_t avail_len;
    uint64_t own_begin, own_end;
    uint64_t global_offset;
    int32_t prev_byte, next_byte;
    uint64_t group_begin, group_end; // 16-byte groups [group_begin, group_end) are scanned by the vector loop
    uint64_t tail_start;             // starts >= tail_start are checked byte-wise by the tail warp
    uint32_t m;                      // full pattern length
    uint32_t emit_len;               // bytes that must match for a key to be emitted (== m, or 1 for prefix plans)
    uint32_t K[4];                   // filter constants (already folded)
    uint32_t fold;                   // AND-mask applied to text words before comparing (0xFFFFFFFF or 0xDFDFDFDF)
    uint32_t win_mask;               // WINDOW4: mask of the low min(4, emit_len) bytes
    uint32_t mulc[3];                // WINDOW4: 2^24, 2^16, 2^8 — window extraction on the FMA pipe (scan_literal.cu)
    const uint8_t *pat_val;          // device: pattern[k] & pat_mask[k]
    const uint8_t *pat_mask;         // device: 0xDF where case folds, else 0xFF
    uint64_t *out;                   // device key buffer (may be null when !want_positions)
    uint64_t cap;
    unsigned long long *counter;     // [0] = occurrences emitted (exact, also past cap)
    uint32_t whole_word;             // 0 none, 1 drop failures on device, 2 tag only
    uint32_t want_positions;
};

// -E plans (regex_dfa.cpp): the line automaton of the regex.  Rows are addressed by offset (state * nclasses), and so
// are the table entries: next_row = trans[row + cls[byte]].  Row 0 is MATCHED (the line is flagged), row nclasses is
// DEAD (nothing can match in the rest of the line); the '\n' column holds 0 for states that accept at the end of a line.
//   regex keys : key = global_line_start << LIT_TAG_BITS (tag bits zero), one per flagged line
static constexpr uint32_t REGEX_TABLE_BYTES = 32768; // transition table budget: shared memory of k_regex_lines
static constexpr uint32_t REGEX_MAX_STATES = 4096;
static constexpr uint32_t REGEX_HALO = 4096; // a line may run this far past its thread's segment before it is flagged unverified
static constexpr uint32_t REGEX_SEG = 256;   // bytes of owned range per thread of k_regex_lines
// The long-line pass (scan_regex_long.cu, DESIGN §12.8): a line whose '\n' lies beyond the reach of k_regex_lines is cut
// into slices of REGEX_LONG_SLICE bytes walked in parallel, each recording its rows every REGEX_LONG_CKPT bytes.
static constexpr uint32_t REGEX_LONG_SLICE = 4096;
static constexpr uint32_t REGEX_LONG_CKPT = 256;
static constexpr uint64_t REGEX_LONG_MAX_LINE = 1ull << 30; // longer lines stay with glibc (replay_regex cuts runs there)
static constexpr uint32_t REGEX_LONG_MAX_MATCH = 8192;      // a match this long does not fit the match key's length field

// Match mode of k_regex_lines (offsets on the device, DESIGN §12.2): one key per match of a line the device decides, one
// per line it leaves to regexec.  Ascending key order is the reference's emission order; a line's uncertain key sorts
// before any match key in it.
//   match key     : (global_start << 16) | (len << 3) | 1    (len <= REGEX_SEG + REGEX_HALO < 2^13)
//   uncertain key : global_line_start << 16
static constexpr int REGEX_MATCH_SHIFT = 16;
static constexpr uint64_t REGEX_MATCH_MAX_OFFSET = 1ull << 48;
// The three modes of k_regex_lines.  The values are the C ABI's `int mode` and RegexRowHeader::mode (DESIGN §12.4).
enum RegexMode : int
{
    RX_FILTER = 0,  // one key per flagged line; glibc confirms them
    RX_COUNT = 1,   // fused -c: lines decided MATCHED are counted, uncertain lines leave keys
    RX_OFFSETS = 2, // offsets: one key per match of a line decided MATCHED, uncertain lines leave keys
};
// Where a mode's keys hold the line or match start: LIT_TAG_BITS, or REGEX_MATCH_SHIFT in the offsets mode.
inline int regex_key_shift(RegexMode mode) { return mode == RX_OFFSETS ? REGEX_MATCH_SHIFT : LIT_TAG_BITS; }
// The anchored match automaton shares the kernel's default dynamic shared memory with the line table and the class map.
static constexpr uint32_t REGEX_SMEM_BYTES = 48 * 1024;
// Enumeration budget of one line in match mode: automaton steps (plus one per start position tried) before the line is
// left to regexec.  Keeps patterns such as [a-c]*d on long a-c runs linear.
static constexpr uint32_t REGEX_MATCH_STEPS_PER_BYTE = 8;
static constexpr uint32_t REGEX_MATCH_STEPS_BASE = 256;

struct RegexDfa
{
    uint32_t nstates = 0, nclasses = 0, nl_class = 0;
    uint32_t start = 0; // row of the line-start state
    uint8_t cls[256];
    std::vector<uint16_t> trans;
    bool widened = false; // the automaton accepts more than the regex (word assertions, -i brackets)
    bool count_exact = false; // its per-line answer is glibc's: -c may be counted on the device (DESIGN §12.1)
    // offsets_exact: match offsets may be computed on the device (DESIGN §12.2).  Then `match` holds the anchored match
    // automaton over the same byte classes: row 0 is DEAD, entries are row offsets (next = match[row + cls[byte]]), and
    // the '\n' column holds the row's accept bits instead of a transition: 1 = a match ends here, 2 = a match ends here
    // if the line ends here (the '$' before '\n').  match_bol starts a match at the line's first byte, match_mid anywhere
    // else.
    bool offsets_exact = false;
    std::vector<uint16_t> match;
    uint32_t match_bol = 0, match_mid = 0;
    // A split plan (DESIGN §12.7) holds the automata of its groups here, each compiled as a regex of its own, and only
    // the three flags above (the union's); a plan of one automaton leaves it empty.
    std::vector<RegexDfa> groups;
};
// Is `mode` (any int, as the C ABI passes it) one the plan of D can run?  The count and offsets modes need the exact flags.
inline bool regex_mode_available(const RegexDfa &D, int mode)
{
    return mode == RX_FILTER || (mode == RX_COUNT && D.count_exact) || (mode == RX_OFFSETS && D.offsets_exact);
}
static constexpr uint16_t RX_ACC = 1, RX_ACC_EOL = 2;
// Padded size in 16-bit words of the table image the kernel copies to shared memory: line table, class map, match table.
__host__ __device__ inline uint32_t regex_tab_words(uint32_t ntrans) { return (ntrans + 7) & ~7u; }

// Split plans (DESIGN §12.7).  A regex whose one automaton is refused for size, and whose top level is an alternation
// B1|...|Bk (krep's (p1)|...|(pk) of -f / several -e), is compiled as up to REGEX_MAX_GROUPS automata, one per group
// of consecutive branches, that k_regex_lines walks together.  The whole image lives in the shared memory of one CTA,
// at most REGEX_SET_SMEM_BYTES (a constant: plans are built before any device is known; sm_90 lets a block opt in to
// 227 KiB).  The line tables and class maps must fit, or the plan is refused; offsets stay on the device only when the
// match tables fit as well.  Measured envelope: 200 lowercase literals of 8-12 bytes fit with offsets (about 95 KiB of
// line tables and 95 KiB of match tables), 200 alphanumeric ones without (176 KiB of line tables), 500 lowercase ones
// not at all (235 KiB of line tables).
static constexpr uint32_t REGEX_MAX_GROUPS = 8;
static constexpr uint32_t REGEX_SET_SMEM_BYTES = 224 * 1024;
// One automaton of a plan's image as the kernel reads it: 16-bit word offsets of its line table, class map and match
// table in the image, and its RegexDfa numbers.
struct RegexGroup
{
    uint32_t trans, cls, match;
    uint32_t nclasses, nl_class, start, match_bol, match_mid;
};
// The image of a plan: every automaton's line table (padded to 16 bytes) and class map, in order, then every match table
// (padded).  A plan of one automaton gives the layout k_regex_lines reads.  grp[REGEX_MAX_GROUPS]: the automata, and in
// the slots past *ngroups the first one started DEAD; *line_words: the words the filter and count modes read.
void regex_layout(const RegexDfa &D, RegexGroup *grp, uint32_t *ngroups, uint32_t *line_words, uint32_t *image_words);
std::vector<uint16_t> regex_image(const RegexDfa &D);
bool regex_source(const search_params_t *P, std::string *out); // the string krep compiles (krep.c:2081-2145)
// 0, or -1 = refused (*why).  max_states: the state cap of each automaton (tests lower it to force split plans).
int regex_compile(const std::string &re, bool icase, RegexDfa *D, std::string *why, uint32_t max_states = REGEX_MAX_STATES);
void regex_lines_host(const RegexDfa &D, const char *text, size_t n, std::vector<uint64_t> *line_starts);
// The count mode of k_regex_lines on the host, every line walked at most `reach` bytes: returns the lines decided
// MATCHED and stores the uncertain line starts (live at the bound, or holding the text's last byte) in *uncertain.
uint64_t regex_count_lines_host(const RegexDfa &D, const char *text, size_t n, uint64_t reach, std::vector<uint64_t> *uncertain);
// The match mode of k_regex_lines on the host (offsets_exact plans), every line walked at most `reach` bytes: stores the
// match-mode keys (see REGEX_MATCH_SHIFT) in ascending order in *keys.
void regex_matches_host(const RegexDfa &D, const char *text, size_t n, uint64_t reach, std::vector<uint64_t> *keys);

// A shard's -E row (krep_b200_regex_export_shard, DESIGN §12.4): what the host needs of one resident shard to finish a
// regex search without the text.  One flat, 16-byte aligned buffer, every part padded to 16 bytes:
//   RegexRowHeader                      128 bytes
//   keys[nkeys]                         the shard's sorted keys, in the layout of its mode (filter / count: line start
//                                       << LIT_TAG_BITS; match: REGEX_MATCH_SHIFT layout)
//   segs[nseg]                          RegexRowSeg: global start, (length << 1) | cont
//   head bytes                          head_len bytes (ROW_HEAD only)
//   segment bytes                       one per segment, in order
// A segment is a maximal run of consecutive lines glibc must see (filter and count mode: every key's line; match mode:
// the uncertain lines, keys with low bit 0), from its first line start up to and including its last line's '\n'.  The
// '\n' is searched up to avail_len; a segment whose last line runs past avail_len is cut there and has cont = 1 (the
// line goes on in the next shards).  The head is the shard's own bytes from own_begin up to and including its first
// '\n' (the whole owned range when it holds none), present when the shard starts mid-line: the resolver continues a cut
// line with the heads of the shards that follow it, through as many shards as the line spans.
static constexpr uint64_t REGEX_ROW_MAGIC = 0x31776f725f78726bull; // "krx_row1"
static constexpr uint64_t ROW_HEAD = 1;  // the head is present (the shard starts mid-line)
static constexpr uint64_t ROW_LAST = 2;  // the shard ends the text: last_byte holds the text's last byte
static constexpr uint64_t ROW_LAST_BYTE_SHIFT = 8;
struct RegexRowHeader
{
    uint64_t magic;
    uint64_t mode;         // RegexMode
    uint64_t row_bytes;    // the whole row, a multiple of 16
    uint64_t device_lines; // count mode: lines of the shard decided MATCHED on the device
    uint64_t nkeys, nseg, head_len;
    uint64_t flags;        // ROW_HEAD | ROW_LAST | last byte << ROW_LAST_BYTE_SHIFT
    uint64_t own_begin, own_end, avail_end; // global offsets of the owned range and of the end of the readable bytes
    uint64_t reserved[5];
};
static_assert(sizeof(RegexRowHeader) == 128, "row header layout");
struct RegexRowSeg
{
    uint64_t start;    // global offset of the segment's first byte (a line start)
    uint64_t len_cont; // (bytes << 1) | cont
};
__host__ __device__ inline uint64_t round16(uint64_t v) { return (v + 15) & ~15ull; }
__host__ __device__ inline uint64_t regex_row_fixed_bytes(uint64_t nkeys, uint64_t nseg)
{
    return sizeof(RegexRowHeader) + round16(nkeys * 8 + nseg * sizeof(RegexRowSeg));
}

struct RegexLaunch
{
    const uint8_t *text;
    uint64_t avail_len, own_begin, own_end, global_offset;
    int32_t prev_byte, next_byte;
    const uint16_t *trans; // device copy of RegexDfa::trans followed by the 256-byte class map
    uint32_t ntrans, nclasses, start, nl_class;
    uint64_t *out;
    uint64_t cap;
    unsigned long long *counter;
    unsigned long long *line_count; // count mode (-c): lines decided MATCHED on the device; nullptr = filter mode
    // match mode (offsets on the device) when set: the match table follows the class map in `trans`
    uint32_t matches, nmtrans, match_bol, match_mid;
    // batch mode when text_end is set (krep_b200_regex_search_batch, DESIGN §12.5): the text holds many texts packed at
    // 16-byte aligned global offsets, each followed by '\n' bytes up to the next text; a line belongs to the text it
    // starts in, and its uncertain-line rule and -c counter are that text's own
    const uint64_t *text_start, *text_end; // global [start, end) of packed text i, ascending
    const uint32_t *seg_text;              // per global 256-byte segment g: the first text i with text_end[i] > g * 256
    unsigned long long *text_lines;        // count mode: lines of text i decided MATCHED (replaces line_count)
    uint32_t n_texts;
    // split plans (ngroups >= 2): the automata of the image at `trans` (regex_layout); line_words of it are
    // copied to shared memory in the filter and count modes, image_words in match mode
    uint32_t ngroups, line_words, image_words;
    RegexGroup grp[REGEX_MAX_GROUPS];
};
static_assert(REGEX_SEG == 256, "RegexLaunch::seg_text has one entry per 256 bytes");
// The device copies of a batch's text table (RegexLaunch batch fields), handed to launch_scan.
struct RegexBatchDev
{
    const uint64_t *text_start, *text_end;
    const uint32_t *seg_text;
    uint32_t n_texts;
};

struct AcDevTables;  // scan_multi.cu: one device's copy of a pattern set's tables
struct AcHostTables; // scan_multi.cu: the tables as compiled on the host (uploaded to each device on first use)

static constexpr int MAX_DEV = 16; // CUDA devices one process can drive

// Device-resident half of a plan, one per CUDA device that has run it (uploaded lazily by plan_on_device()).
struct PlanDev
{
    bool ready = false;
    uint8_t *d_pat_val = nullptr, *d_pat_mask = nullptr; // literal
    AcDevTables *ac = nullptr;                           // pattern set
    uint16_t *d_regex = nullptr;                         // regex: the plan's image (regex_layout)
};

struct Plan
{
    int algo = 0;
    bool is_ac = false;
    // literal
    std::string pattern;
    bool case_sensitive = true;
    uint32_t m = 0, emit_len = 0;
    FilterKind filter = FILTER_ALIGNED4;
    uint32_t K[4] = {0, 0, 0, 0};
    uint32_t fold = 0xFFFFFFFFu, win_mask = 0xFFFFFFFFu;
    uint32_t whole_word = 0;
    std::vector<uint8_t> h_val, h_msk; // pattern[k] & mask[k], mask[k] (0xDF where case folds, else 0xFF)
    bool border_free = true; // no proper prefix is also a suffix: occurrences cannot overlap
    bool built_only_matching = false; // value of the -o global the plan was compiled for
    bool count_lines = false;         // -c: scan_shard also computes the line bounds of every occurrence on the device
    // AC
    std::vector<std::string> patterns;
    std::vector<uint32_t> pat_lens;
    uint32_t min_len = 0, max_len = 0;
    AcHostTables *ach = nullptr;
    // regex (-E)
    bool is_regex = false;
    std::string regex;       // the string krep compiled
    RegexDfa *rx = nullptr;
    std::string filter_name;
    PlanDev dev[MAX_DEV];
    uint64_t magic = 0x6b7265705f623230ull; // "krep_b20"
};

// engine.cu
struct DevCtx;
void set_error(int code, const char *fmt, ...);
void clear_error();

struct ScanOut
{
    uint64_t count = 0, stored = 0;
    const uint64_t *d_keys = nullptr;
    int overflow = 0;
    const uint64_t *d_bounds = nullptr; // -c plans: 2 words per stored key (line start, line end), see k_line_bounds
    const uint64_t *h_sorted = nullptr; // host copy of the sorted keys when the list was small enough to come back with the
                                        // count (k_finish, engine.cu); valid until the next scan on the same device slot
    int device = 0;
    uint64_t serial = 0;                // scan number on that device (stale-result detection in krep_b200_collect)
};

// Line bounds of an occurrence, global offsets: [0] = first byte of its line, [1] = position of the line's '\n' (or
// the text length).  The device writes these markers where the answer lies outside what one warp looked at:
static constexpr uint64_t LB_SAME_AS_PREV = ~0ull;     // no newline between the previous occurrence and this one
static constexpr uint64_t LB_SAME_AS_NEXT = ~0ull - 1; // no newline between this occurrence and the next one
static constexpr uint64_t LB_OUTSIDE_SHARD = ~0ull - 2; // the line continues into a neighbouring shard

// Slice and checkpoint sizes of the long-line pass (0: REGEX_LONG_SLICE / REGEX_LONG_CKPT).
struct LongLineOpts
{
    uint32_t slice_bytes = 0, ckpt_bytes = 0;
};

// Launch one shard scan on `stream` of the device context; appends to that device's key list (no counter reset).
// regex_lines (regex plans only): run k_regex_lines in count mode, adding the lines it decides MATCHED there.
// regex_matches (offsets_exact regex plans, with want_positions): run it in match mode (match and uncertain-line keys).
// regex_batch: the shard is (a chunk of) a packed batch of texts; regex_lines then has one counter per text.
// long_lines (regex plans): after k_regex_lines, decide the lines longer than its reach on the device
// (scan_regex_long.cu, DESIGN §12.8), batches included; nullptr leaves them uncertain.
int launch_scan(DevCtx &C, const Plan *plan, const krep_b200_shard_t *sh, int want_positions, cudaStream_t stream, int slot = 0,
                unsigned long long *regex_lines = nullptr, bool regex_matches = false, const RegexBatchDev *regex_batch = nullptr,
                const LongLineOpts *long_lines = nullptr);
// literal kernels (scan_literal.cu)
void launch_literal(const Plan *plan, const LitDevParams &p, int sm_count, cudaStream_t s);
// multi kernels (scan_multi.cu)
int ac_build_tables(Plan *plan);                 // host side only: filter tables, exact table, pattern pool
void ac_free_tables(Plan *plan);                 // host tables (device copies are freed by ac_free_device)
AcDevTables *ac_upload_tables(const Plan *plan); // copies the host tables to the current device; nullptr on CUDA errors
void ac_free_device(AcDevTables *T);
struct AcLaunch
{
    const uint8_t *text;
    uint64_t avail_len, own_begin, own_end, global_offset;
    int32_t prev_byte, next_byte;
    uint64_t *out;
    uint64_t cap;
    unsigned long long *counter;
    uint32_t whole_word, want_positions;
};
void launch_ac(const Plan *plan, const AcDevTables *T, const AcLaunch &a, int sm_count, cudaStream_t s);
void count_launch(int n = 1);
// regex kernel (scan_regex.cu)
int launch_regex(const RegexLaunch &a, int sm_count, cudaStream_t s); // 0, or -2 with the error set
// long-line pass (scan_regex_long.cu): long_lines_begin before launch_regex (scratch + list snapshot), launch_long_lines
// after it, both on the scan's stream; 0, or the error set
int long_lines_begin(DevCtx &C, const RegexLaunch &a, const LongLineOpts &o, cudaStream_t s);
int launch_long_lines(DevCtx &C, const RegexLaunch &a, const LongLineOpts &o, cudaStream_t s);
const LongLineOpts *long_lines_default(); // production sizes, or nullptr when KREP_B200_NO_LONG_LINES is set (read per call)
// the sizes of the long-line test hooks (0: production); 0, or -3 with the error set for sizes outside
// 1 <= ckpt <= slice <= 2^20 with at most 1024 checkpoints per slice
int long_lines_opts(const char *who, uint32_t slice_bytes, uint32_t ckpt_bytes, LongLineOpts *o);

// semantics.cpp — reference control flow replayed over the sorted occurrence list
struct Replay
{
    const uint64_t *keys;
    size_t n;
    const char *text; // host text (for -c line logic); may be null when `bounds` is given or -c is off
    size_t text_len;
    uint64_t base; // global offset subtracted from key offsets
    const uint64_t *bounds = nullptr; // resolved line bounds, 2 per key (device-side -c): used when text is null
    // replay_regex: the text from `stop` on (a line start below text_len) belongs to another decider — no regexec call
    // reaches past it, and a match found there ends the replay (SIZE_MAX: the whole text is the replay's)
    size_t stop = SIZE_MAX;
    // replay_regex over a window of the text (resident shards, DESIGN §12.4): `text` holds the bytes of global
    // [origin, origin + window_len), whole lines starting at a line start, while text_len stays the whole text's length.
    // window_len SIZE_MAX: `text` is the whole text.  last_byte: the text's last byte when the window does not hold it.
    size_t origin = 0;
    size_t window_len = SIZE_MAX;
    int last_byte = -1;
};
// One window of a windowed replay: global [origin, origin + len), whole lines.
struct RegexWindow
{
    size_t origin;
    const char *bytes;
    size_t len;
};
uint64_t replay_literal(int algo, const search_params_t *P, bool only_matching, uint32_t m,
                        const Replay &r, match_result_t *res);
uint64_t replay_ac(const search_params_t *P, const Replay &r, match_result_t *res);
uint64_t replay_regex(const search_params_t *P, const Replay &r, match_result_t *res); // needs r.text
// Offsets on the device (match-mode keys, ascending): match keys become positions, uncertain lines go to replay_regex.
uint64_t replay_regex_matches(const search_params_t *P, const Replay &r, match_result_t *res);
// The same two replays over windows of the text instead of the whole text (ascending, disjoint; every key's line lies in
// one): window by window in order, the -m budget carried.  n: the whole text's length, last_byte its last byte.
// replay_regex_windows takes LIT_TAG_BITS keys; at_end: also decide the empty string at n after the last window.
uint64_t replay_regex_windows(const search_params_t *P, const uint64_t *keys, size_t nkeys, const RegexWindow *w, size_t nw,
                              size_t n, int last_byte, bool at_end, match_result_t *res);
uint64_t replay_regex_matches_windows(const search_params_t *P, const uint64_t *keys, size_t nkeys, const RegexWindow *w,
                                      size_t nw, size_t n, int last_byte, match_result_t *res);
// The -E call is answered 0 before the text is looked at: -m 0 with -c or positions (krep.c:1395), or no compiled regex
// (krep.c:1399).
bool regex_returns_early(const search_params_t *P);
// The answer on an empty text (krep.c:1403-1416) of a call that did not return early: whether the regex matches the
// empty string.
uint64_t regex_empty_text(const search_params_t *P, match_result_t *res);
// The answer of a -E call from the keys of a scan in `mode`; device_lines: the lines the count mode decided MATCHED.
uint64_t regex_answer(const search_params_t *P, RegexMode mode, uint64_t device_lines, const Replay &r, match_result_t *res);
// The same over windows of the text (replay_regex_windows); at_end: the filter and count modes decide the empty string
// at n after the last window.
uint64_t regex_answer_windows(const search_params_t *P, RegexMode mode, uint64_t device_lines, const std::vector<uint64_t> &keys,
                              const std::vector<RegexWindow> &w, size_t n, int last_byte, bool at_end, match_result_t *res);
// regex_rows.cpp: the answer of a -E search from the rows of the shards that tile the text (text order).  *err: 0, or
// -3 with the error set.
uint64_t regex_resolve_rows(const search_params_t *P, const void *const *rows, uint32_t n_rows, match_result_t *res, int *err);
// The answers of a packed -E batch from its one row (DESIGN §12.9).  Text i (packed order) is [lo[i], lo[i] + len[i]) of
// the packed buffer, len[i] > 0, with last byte last[i] and, in count mode, text_lines[i] lines decided on the device;
// counts[i] and res[i] (res or res[i] may be null) get krep_b200_regex_search's answer for it.  Returns 0, or -3 with
// the error set.
int regex_resolve_batch(const search_params_t *P, const void *row, size_t n_texts, const uint64_t *lo, const size_t *len,
                        const uint8_t *last, const uint64_t *text_lines, uint64_t *counts, match_result_t *const *res);
bool result_push(match_result_t *r, size_t s, size_t e);

// C-locale helpers shared by host code (krep.c:125-134, krep.h:298-301)
static inline unsigned char lower_c(unsigned char c) { return (c >= 'A' && c <= 'Z') ? (unsigned char)(c + 32) : c; }
static inline bool is_alpha_c(unsigned char c) { return (c >= 'A' && c <= 'Z') || (c >= 'a' && c <= 'z'); }
static inline bool is_word_c(int c)
{
    return (c >= '0' && c <= '9') || (c >= 'A' && c <= 'Z') || (c >= 'a' && c <= 'z') || c == '_';
}

} // namespace kb
