// engine.cu — process-wide engine context, plan compilation, shard scan (launch + device sort),
// synthetic corpus generator, and the device-level half of the C ABI (include/krep_b200.h).
#include <cub/device/device_radix_sort.cuh>
#include <algorithm>
#include <chrono>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <thread>
#include "common.h"
#include "corpus.h"
#include "engine.h"

namespace kb {

// ---------------------------------------------------------------------------------------------
// errors (reference convention: "krep: ..." on stderr, no in-band channel — krep.c:1933)
// ---------------------------------------------------------------------------------------------
static thread_local int t_err = 0;
static thread_local char t_errmsg[512] = "";

void set_error(int code, const char *fmt, ...)
{
    t_err = code;
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(t_errmsg, sizeof t_errmsg, fmt, ap);
    va_end(ap);
    fprintf(stderr, "krep: %s\n", t_errmsg);
}
void clear_error()
{
    t_err = 0;
    t_errmsg[0] = 0;
}

#define CK(call)                                                                                   \
    do                                                                                             \
    {                                                                                              \
        cudaError_t e_ = (call);                                                                   \
        if (e_ != cudaSuccess)                                                                     \
        {                                                                                          \
            set_error(-2, "CUDA error %s at %s:%d (%s)", cudaGetErrorName(e_), __FILE__, __LINE__, \
                      cudaGetErrorString(e_));                                                     \
            return -2;                                                                             \
        }                                                                                          \
    } while (0)

static DevCtx g_ctx[MAX_DEV];
static std::recursive_mutex g_mu;
static std::mutex g_ctx_mu;
static int g_primary = -1;
static int g_visible = -1;
static bool g_keep_visible = false; // the host chose its devices itself: leave CUDA_VISIBLE_DEVICES alone
static uint64_t g_launches = 0;
static thread_local float t_kernel_ms = 0.f;
static const std::chrono::steady_clock::time_point g_t0 = std::chrono::steady_clock::now();

std::recursive_mutex &engine_mutex() { return g_mu; }
void count_launch(int n) { __atomic_fetch_add(&g_launches, (uint64_t)n, __ATOMIC_RELAXED); }
void add_kernel_ms(float ms) { t_kernel_ms += ms; }
void reset_kernel_ms() { t_kernel_ms = 0.f; }
float get_kernel_ms() { return t_kernel_ms; }
void set_kernel_ms(float ms) { t_kernel_ms = ms; }
void get_error(ErrState *e)
{
    e->code = t_err;
    memcpy(e->msg, t_errmsg, sizeof e->msg);
}
void adopt_error(const ErrState &e)
{
    t_err = e.code;
    memcpy(t_errmsg, e.msg, sizeof t_errmsg);
}

void trace(const char *fmt, ...)
{
    static const bool on = getenv("KREP_B200_TRACE") != nullptr;
    if (!on) return;
    char buf[400];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    const double ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - g_t0).count();
    fprintf(stderr, "[krep_b200 +%.1f ms] %s\n", ms, buf);
}

// Asynchronous start-up (krep_b200_warmup): CUDA initialisation and the primary context are created on a background
// thread while the host is still busy opening and mapping its file; the first entry point that needs the GPU joins it.
static std::thread *g_warm = nullptr; // heap object on purpose: never destroyed behind a still-running thread
static std::mutex g_warm_mu;
void warm_join()
{
    std::lock_guard<std::mutex> lk(g_warm_mu);
    if (g_warm && g_warm->joinable() && g_warm->get_id() != std::this_thread::get_id()) g_warm->join();
}
bool warm_running()
{
    std::lock_guard<std::mutex> lk(g_warm_mu);
    return g_warm && g_warm->joinable();
}
static void warm_start()
{
    std::lock_guard<std::mutex> lk(g_warm_mu);
    if (g_warm || g_visible >= 0) return; // already started, or CUDA is already up
    g_warm = new std::thread([] {
        trace("warm-up thread: start");
        if (visible_devices() > 0)
            if (DevCtx *C = ctx_primary()) prewarm_host_path(*C);
        trace("warm-up thread: done");
    });
}
__attribute__((destructor)) static void warm_at_exit()
{
    warm_join(); // a process that exits without searching must not tear CUDA down under the thread
    trace("library destructor (process exit)");
}

void keep_devices_visible() { g_keep_visible = true; }

int visible_devices()
{
    if (g_visible >= 0) return g_visible;
    static std::mutex mu;
    std::lock_guard<std::mutex> lk(mu);
    if (g_visible >= 0) return g_visible;
    // A process in which this library is the FIRST user of CUDA (the krep CLI) hides the GPUs it is not going to use from
    // the driver before CUDA initialises: cuInit enumerates every visible GPU, which on an 8-GPU box costs seconds
    // more than with one device visible.  It will use KREP_B200_DEVICES devices (default
    // 1) — the first ones of CUDA_VISIBLE_DEVICES if that is set.  Not done when the host manages devices itself
    // (krep_b200_init / krep_b200_set_devices called first, or KREP_B200_KEEP_VISIBLE set); harmless when something else
    // (torch) has initialised CUDA already — the variable is only read at initialisation.
    if (!g_keep_visible && !getenv("KREP_B200_KEEP_VISIBLE"))
    {
        const char *v = getenv("KREP_B200_DEVICES");
        const int k = v && atoi(v) > 0 ? atoi(v) : 1;
        std::string list;
        if (const char *cur = getenv("CUDA_VISIBLE_DEVICES"))
        {
            int taken = 0;
            for (const char *q = cur; *q && taken < k;)
            {
                const char *e = strchr(q, ',');
                const size_t len = e ? (size_t)(e - q) : strlen(q);
                if (len)
                {
                    list += (taken ? "," : "") + std::string(q, len);
                    taken++;
                }
                q += len + (e ? 1 : 0);
            }
        }
        else
            for (int d = 0; d < k && d < MAX_DEV; d++) list += (d ? "," : "") + std::to_string(d);
        if (!list.empty())
        {
            setenv("CUDA_VISIBLE_DEVICES", list.c_str(), 1);
            trace("CUDA_VISIBLE_DEVICES=%s", list.c_str());
        }
    }
    int n = 0;
    trace("cudaGetDeviceCount ...");
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess)
    {
        cudaGetLastError();
        n = 0;
    }
    trace("cudaGetDeviceCount -> %d", n);
    g_visible = n > MAX_DEV ? MAX_DEV : n;
    return g_visible;
}

int primary_device()
{
    if (g_primary >= 0) return g_primary;
    if (visible_devices() == 0)
    {
        set_error(-1, "no CUDA device available; this engine has no CPU fallback");
        return -1;
    }
    int d = 0;
    if (cudaGetDevice(&d) != cudaSuccess) d = 0;
    g_primary = d;
    return d;
}

static int ctx_create(DevCtx &E, int device)
{
    trace("device %d: creating context", device);
    CK(cudaSetDevice(device));
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9 || prop.minor != 0) // sm_90a code loads on compute capability 9.0 only
    {
        set_error(-1, "device %d (%s, sm_%d%d) is not an sm_90 part; kernels are built for sm_90a only", device,
                  prop.name, prop.major, prop.minor);
        return -1;
    }
    E.device = device;
    E.sm_count = prop.multiProcessorCount;
    CK(cudaStreamCreateWithFlags(&E.scan_stream, cudaStreamNonBlocking));
    CK(cudaStreamCreateWithFlags(&E.copy_stream, cudaStreamNonBlocking));
    CK(cudaStreamCreateWithFlags(&E.fin_stream, cudaStreamNonBlocking));
    CK(cudaMalloc(&E.d_counter, 64 * SCAN_SLOTS));
    CK(cudaMemset(E.d_counter, 0, 64 * SCAN_SLOTS));
    CK(cudaEventCreate(&E.ev_ca));
    CK(cudaEventCreate(&E.ev_cb));
    for (int s = 0; s < SCAN_SLOTS; s++)
    {
        CK(cudaMalloc(&E.d_pack[s], (PACK_KEYS + 1) * sizeof(uint64_t)));
        CK(cudaHostAlloc(&E.h_pack[s], (PACK_KEYS + 1) * sizeof(uint64_t), cudaHostAllocMapped | cudaHostAllocPortable));
        E.h_pack[s][0] = 0;
        CK(cudaEventCreate(&E.ev_a[s]));
        CK(cudaEventCreate(&E.ev_b[s]));
        CK(cudaEventCreateWithFlags(&E.ev_done[s], cudaEventDisableTiming));
        CK(cudaEventCreateWithFlags(&E.ev_scanned[s], cudaEventDisableTiming));
        E.counter_clean[s] = true;
    }
    E.ready = true;
    trace("device %d: context ready (%s, %d SMs)", device, prop.name, E.sm_count);
    return 0;
}

DevCtx *ctx_get(int device)
{
    if (device < 0 || device >= MAX_DEV || device >= visible_devices())
    {
        set_error(-1, visible_devices() == 0 ? "no CUDA device available; this engine has no CPU fallback"
                                               : "CUDA device %d is not visible to this process",
                  device);
        return nullptr;
    }
    DevCtx &E = g_ctx[device];
    if (E.ready)
    {
        cudaSetDevice(device);
        return &E;
    }
    static std::mutex mu[MAX_DEV]; // per device: contexts of different GPUs may be created concurrently
    std::lock_guard<std::mutex> lk(mu[device]);
    if (!E.ready && ctx_create(E, device) != 0) return nullptr;
    return &E;
}

DevCtx *ctx_primary()
{
    const int d = primary_device();
    return d < 0 ? nullptr : ctx_get(d);
}

// a single process may hold shards on several GPUs; a failed lookup's error is cleared
DevCtx *ctx_of_pointer(const void *d_ptr)
{
    cudaPointerAttributes a;
    if (cudaPointerGetAttributes(&a, d_ptr) == cudaSuccess && a.type == cudaMemoryTypeDevice) return ctx_get(a.device);
    cudaGetLastError();
    return ctx_primary();
}

static std::vector<Plan *> g_all_plans; // every live plan (device copies are released at shutdown)
static std::mutex g_plans_mu;

static void ctx_destroy(DevCtx &E)
{
    if (!E.ready) return;
    cudaSetDevice(E.device);
    cudaDeviceSynchronize();
    for (int s = 0; s < SCAN_SLOTS; s++) cudaFree(E.d_list[s]);
    cudaFree(E.d_alt);
    cudaFree(E.d_sort_tmp);
    cudaFree(E.d_bounds);
    cudaFreeHost(E.h_bounds);
    cudaFreeHost(E.h_batch);
    cudaFree(E.d_rx_batch);
    cudaFree(E.d_gather);
    cudaFree(E.d_gather_tab);
    cudaFree(E.d_counter);
    cudaFree(E.d_ring);
    cudaFree(E.d_line_recs);
    cudaFree(E.d_line_out);
    cudaFreeHost(E.h_line_out);
    cudaFree(E.d_set_acc);
    cudaFreeHost(E.h_keys);
    regex_pack_free(E);
    long_lines_free(E);
    for (int s = 0; s < SCAN_SLOTS; s++)
    {
        cudaFree(E.d_pack[s]);
        cudaFreeHost(E.h_pack[s]);
        cudaEventDestroy(E.ev_a[s]);
        cudaEventDestroy(E.ev_b[s]);
        cudaEventDestroy(E.ev_done[s]);
        cudaEventDestroy(E.ev_scanned[s]);
    }
    for (auto &s : E.stage) cudaFreeHost(s.buf);
    for (auto &s : E.stage)
        if (s.ev) cudaEventDestroy(s.ev);
    for (auto ev : E.ev_pool) cudaEventDestroy(ev);
    for (auto ev : E.ring_landed) cudaEventDestroy(ev);
    for (auto ev : E.ring_scanned) cudaEventDestroy(ev);
    cudaEventDestroy(E.ev_ca);
    cudaEventDestroy(E.ev_cb);
    cudaStreamDestroy(E.scan_stream);
    cudaStreamDestroy(E.copy_stream);
    cudaStreamDestroy(E.fin_stream);
    E = DevCtx();
}

void plan_cache_clear(); // host_api.cu

void engine_shutdown()
{
    std::lock_guard<std::recursive_mutex> lk(g_mu);
    DeviceGuard guard;
    plan_cache_clear();
    {
        std::lock_guard<std::mutex> lp(g_plans_mu);
        for (Plan *p : g_all_plans) // plans still held by the host keep their host half; device halves go with the contexts
            for (int d = 0; d < MAX_DEV; d++)
            {
                PlanDev &pd = p->dev[d];
                if (!pd.ready) continue;
                cudaSetDevice(d);
                cudaFree(pd.d_pat_val);
                cudaFree(pd.d_pat_mask);
                if (pd.ac) ac_free_device(pd.ac);
                pd = PlanDev();
            }
    }
    for (int d = 0; d < MAX_DEV; d++) ctx_destroy(g_ctx[d]);
    g_primary = -1;
}

int ensure_keys(DevCtx &E, uint64_t cap)
{
    if (cap <= E.key_cap) return 0;
    uint64_t ncap = E.key_cap ? E.key_cap : (1ull << 20);
    while (ncap < cap) ncap *= 2;
    CK(cudaDeviceSynchronize());
    for (int s = 0; s < SCAN_SLOTS; s++)
    {
        cudaFree(E.d_list[s]);
        E.d_list[s] = nullptr;
    }
    cudaFree(E.d_alt);
    E.d_alt = nullptr;
    E.key_cap = 0;
    for (int s = 0; s < SCAN_SLOTS; s++) CK(cudaMalloc(&E.d_list[s], ncap * sizeof(uint64_t)));
    CK(cudaMalloc(&E.d_alt, ncap * sizeof(uint64_t)));
    E.key_cap = ncap;
    return 0;
}

unsigned long long *slot_counter(DevCtx &E, int slot) { return E.d_counter + 8 * slot; }

// ---------------------------------------------------------------------------------------------
// plan compilation
// ---------------------------------------------------------------------------------------------
static uint32_t le32(const uint8_t *b, uint32_t n)
{
    uint32_t v = 0;
    for (uint32_t k = 0; k < n && k < 4; k++) v |= (uint32_t)b[k] << (8 * k);
    return v;
}

void plan_free(Plan *p)
{
    if (!p) return;
    {
        std::lock_guard<std::mutex> lp(g_plans_mu);
        for (size_t i = 0; i < g_all_plans.size(); i++)
            if (g_all_plans[i] == p)
            {
                g_all_plans.erase(g_all_plans.begin() + i);
                break;
            }
    }
    DeviceGuard guard;
    for (int d = 0; d < MAX_DEV; d++)
    {
        PlanDev &pd = p->dev[d];
        if (!pd.ready) continue;
        cudaSetDevice(d);
        cudaFree(pd.d_pat_val);
        cudaFree(pd.d_pat_mask);
        if (pd.ac) ac_free_device(pd.ac);
        cudaFree(pd.d_regex);
    }
    if (p->ach) ac_free_tables(p);
    delete p->rx;
    p->magic = 0;
    delete p;
}

// The device half of a plan on the context's device: uploaded the first time that device runs the plan.
const PlanDev *plan_on_device(const Plan *plan, DevCtx &C)
{
    static std::mutex mu;
    PlanDev &pd = const_cast<Plan *>(plan)->dev[C.device];
    if (pd.ready) return &pd;
    std::lock_guard<std::mutex> lk(mu);
    if (pd.ready) return &pd;
    cudaSetDevice(C.device);
    if (plan->is_ac)
    {
        pd.ac = ac_upload_tables(plan);
        if (!pd.ac) return nullptr;
    }
    else if (plan->is_regex)
    {
        // the plan's image (regex_layout): the kernel copies what its mode reads to shared memory as vectors
        const std::vector<uint16_t> img = regex_image(*plan->rx);
        if (cudaMalloc(&pd.d_regex, img.size() * 2) != cudaSuccess ||
            cudaMemcpy(pd.d_regex, img.data(), img.size() * 2, cudaMemcpyHostToDevice) != cudaSuccess)
        {
            set_error(-2, "CUDA allocation failed while uploading the regex automaton to device %d", C.device);
            cudaFree(pd.d_regex);
            pd = PlanDev();
            return nullptr;
        }
    }
    else
    {
        const size_t m = plan->h_val.size();
        if (cudaMalloc(&pd.d_pat_val, m) != cudaSuccess || cudaMalloc(&pd.d_pat_mask, m) != cudaSuccess ||
            cudaMemcpy(pd.d_pat_val, plan->h_val.data(), m, cudaMemcpyHostToDevice) != cudaSuccess ||
            cudaMemcpy(pd.d_pat_mask, plan->h_msk.data(), m, cudaMemcpyHostToDevice) != cudaSuccess)
        {
            set_error(-2, "CUDA allocation failed while uploading the pattern to device %d", C.device);
            cudaFree(pd.d_pat_val);
            cudaFree(pd.d_pat_mask);
            pd = PlanDev();
            return nullptr;
        }
    }
    pd.ready = true;
    return &pd;
}

static bool border_free(const std::string &s, bool cs)
{
    const size_t m = s.size();
    if (m < 2) return true;
    std::vector<int> pi(m, 0);
    auto ch = [&](size_t i) { return cs ? (unsigned char)s[i] : lower_c((unsigned char)s[i]); };
    for (size_t i = 1; i < m; i++)
    {
        int k = pi[i - 1];
        while (k > 0 && ch(i) != ch((size_t)k)) k = pi[(size_t)k - 1];
        if (ch(i) == ch((size_t)k)) k++;
        pi[i] = k;
    }
    return pi[m - 1] == 0;
}

// -E: the line automaton of the regex krep compiled from params->patterns (or the automata of a split plan).  nullptr and
// *why when the compiler refuses the pattern (no error is raised: a refused regex simply stays on the host's
// regex_search).  max_states: the state cap of each automaton, REGEX_MAX_STATES but for test plans.
Plan *regex_plan_build(const search_params_t *P, std::string *why, uint32_t max_states)
{
    std::string re;
    if (!regex_source(P, &re))
    {
        *why = "no pattern";
        return nullptr;
    }
    RegexDfa *D = new RegexDfa();
    if (regex_compile(re, !P->case_sensitive, D, why, max_states) != 0)
    {
        delete D;
        return nullptr;
    }
    Plan *pl = new Plan();
    pl->algo = KREP_B200_ALGO_REGEX;
    pl->is_regex = true;
    pl->case_sensitive = P->case_sensitive;
    pl->whole_word = P->whole_word ? 1 : 0;
    pl->regex = re;
    pl->rx = D;
    pl->filter_name = std::string(D->groups.empty() ? "regex-lines" : "regex-lines-split") + (D->widened ? "-widened" : "");
    std::lock_guard<std::mutex> lp(g_plans_mu);
    g_all_plans.push_back(pl);
    return pl;
}

// Maps (reference function, params) to what the device has to enumerate.
Plan *plan_build(const search_params_t *P, int algo, bool only_matching)
{
    if (!P) return nullptr;
    if (algo == KREP_B200_ALGO_REGEX)
    {
        std::string why;
        Plan *pl = regex_plan_build(P, &why);
        if (!pl) set_error(-3, "this regex is not run on the GPU (%s); use the host's regex_search", why.c_str());
        return pl;
    }
    Plan *pl = new Plan();
    pl->algo = algo;
    pl->case_sensitive = P->case_sensitive;
    pl->count_lines = P->count_lines_mode;
    if (algo == KREP_B200_ALGO_AC)
    {
        pl->is_ac = true;
        if (P->num_patterns > AC_MAX_PATTERNS)
        {
            set_error(-3, "too many patterns (%zu > %u)", (size_t)P->num_patterns, AC_MAX_PATTERNS);
            delete pl;
            return nullptr;
        }
        for (size_t k = 0; k < P->num_patterns; k++)
        {
            const size_t len = P->pattern_lens[k];
            if (len > 1024)
            {
                set_error(-3, "pattern %zu longer than 1024 bytes (krep.c:77)", k);
                delete pl;
                return nullptr;
            }
            pl->patterns.emplace_back(P->patterns[k] ? P->patterns[k] : "", len);
            pl->pat_lens.push_back((uint32_t)len);
        }
        pl->whole_word = P->whole_word ? 1 : 0;
        if (ac_build_tables(pl) != 0)
        {
            delete pl;
            return nullptr;
        }
        std::lock_guard<std::mutex> lp(g_plans_mu);
        g_all_plans.push_back(pl);
        return pl;
    }
    // ---- single literal ----
    size_t m = P->pattern_len;
    if (algo == KREP_B200_ALGO_MEMCHR) m = m ? 1 : 0; // memchr_search reads pattern[0] only (krep.c:3902)
    if (m == 0 || m > 1024 || !P->pattern)
    {
        set_error(-3, "literal plan needs 1..1024 pattern bytes (got %zu)", m);
        delete pl;
        return nullptr;
    }
    pl->pattern.assign(P->pattern, m);
    pl->m = (uint32_t)m;
    // memchr_short_search -o walks first-byte hits, not occurrences (krep.c:4495)
    pl->emit_len = (algo == KREP_B200_ALGO_MEMCHR_SHORT && only_matching) ? 1u : (uint32_t)m;
    pl->border_free = border_free(pl->pattern, pl->case_sensitive);
    pl->built_only_matching = only_matching;
    if (P->whole_word)
    {
        // Kernels whose cursor also moves past a -w reject (kmp krep.c:1686, sse4.2 krep.c:4839-4848) need the
        // rejected occurrences in the list — but only if occurrences can overlap at all.  Prefix plans always tag.
        bool tag = pl->emit_len != pl->m;
        // the window kernels' tail sub-search re-evaluates -w against its sub-buffer (krep.c:5068): needs both halves
        if (algo == KREP_B200_ALGO_AVX2 || algo == KREP_B200_ALGO_AVX512 || algo == KREP_B200_ALGO_NEON) tag = true;
        if (!tag && !pl->border_free)
            tag = algo == KREP_B200_ALGO_KMP || (algo == KREP_B200_ALGO_SSE42 && !only_matching);
        pl->whole_word = tag ? 2 : 1;
    }
    pl->h_val.resize(m);
    pl->h_msk.resize(m);
    const uint8_t *pb = (const uint8_t *)pl->pattern.data();
    for (size_t k = 0; k < m; k++)
    {
        pl->h_msk[k] = (!pl->case_sensitive && is_alpha_c(pb[k])) ? 0xDF : 0xFF;
        pl->h_val[k] = pb[k] & pl->h_msk[k];
    }
    pl->fold = pl->case_sensitive ? 0xFFFFFFFFu : 0xDFDFDFDFu;
    if (pl->emit_len >= 7)
    {
        pl->filter = FILTER_ALIGNED4;
        for (int d = 0; d < 4; d++) pl->K[d] = le32(pb + d, 4) & pl->fold;
        pl->win_mask = 0xFFFFFFFFu;
        pl->filter_name = pl->case_sensitive ? "aligned4" : "aligned4-fold";
    }
    else
    {
        pl->filter = FILTER_WINDOW4;
        const uint32_t wl = pl->emit_len < 4 ? pl->emit_len : 4;
        pl->win_mask = wl == 4 ? 0xFFFFFFFFu : ((1u << (8 * wl)) - 1);
        pl->K[0] = le32(pb, wl) & pl->fold & pl->win_mask;
        pl->filter_name = pl->case_sensitive ? "window4" : "window4-fold";
    }
    std::lock_guard<std::mutex> lp(g_plans_mu);
    g_all_plans.push_back(pl);
    return pl;
}

// ---------------------------------------------------------------------------------------------
// shard scan
// ---------------------------------------------------------------------------------------------
int launch_scan(DevCtx &E, const Plan *plan, const krep_b200_shard_t *sh, int want_positions, cudaStream_t stream, int slot,
                unsigned long long *regex_lines, bool regex_matches, const RegexBatchDev *regex_batch, const LongLineOpts *long_lines)
{
    if (((uintptr_t)sh->d_text & 15) != 0)
    {
        set_error(-3, "shard text pointer must be 16-byte aligned");
        return -3;
    }
    const PlanDev *pd = plan_on_device(plan, E);
    if (!pd) return -2;
    uint64_t own_end = sh->own_end < sh->avail_len ? sh->own_end : sh->avail_len;
    if (plan->is_regex)
    {
        if (regex_matches && (!plan->rx->offsets_exact || !want_positions))
        {
            set_error(-3, "regex match mode needs an offsets_exact plan and the occurrence list");
            return -3;
        }
        // match keys pack (global start << 16): 48 bits of offset
        if (regex_matches && sh->global_offset + sh->avail_len >= REGEX_MATCH_MAX_OFFSET)
        {
            set_error(-3, "regex match offsets must stay below 2^48 bytes of global offset (key layout, csrc/common.h)");
            return -3;
        }
        RegexLaunch a;
        a.text = (const uint8_t *)sh->d_text;
        a.avail_len = sh->avail_len;
        a.own_begin = sh->own_begin;
        a.own_end = own_end;
        a.global_offset = sh->global_offset;
        a.prev_byte = sh->prev_byte;
        a.next_byte = sh->next_byte;
        a.trans = pd->d_regex;
        a.ntrans = (uint32_t)plan->rx->trans.size();
        a.nclasses = plan->rx->nclasses;
        a.start = plan->rx->start;
        a.nl_class = plan->rx->nl_class;
        a.out = E.d_list[slot];
        a.cap = want_positions ? E.key_cap : 0;
        a.counter = slot_counter(E, slot);
        a.line_count = regex_batch ? nullptr : regex_lines;
        a.matches = regex_matches ? 1u : 0u;
        a.nmtrans = (uint32_t)plan->rx->match.size();
        a.match_bol = plan->rx->match_bol;
        a.match_mid = plan->rx->match_mid;
        a.text_start = regex_batch ? regex_batch->text_start : nullptr;
        a.text_end = regex_batch ? regex_batch->text_end : nullptr;
        a.seg_text = regex_batch ? regex_batch->seg_text : nullptr;
        a.text_lines = regex_batch ? regex_lines : nullptr;
        a.n_texts = regex_batch ? regex_batch->n_texts : 0u;
        regex_layout(*plan->rx, a.grp, &a.ngroups, &a.line_words, &a.image_words);
        // the long-line pass works on the keys this scan appends (a batch's in the batch rules of k_regex_lines)
        const bool long_pass = long_lines && a.cap > 0;
        if (long_pass && long_lines_begin(E, a, *long_lines, stream) != 0) return -2;
        const int rc = launch_regex(a, E.sm_count, stream);
        if (rc != 0 || !long_pass) return rc;
        return launch_long_lines(E, a, *long_lines, stream);
    }
    if (plan->is_ac)
    {
        // the key packs (global end offset << 24): 40 bits of offset
        if (sh->global_offset + sh->avail_len >= (1ull << 40))
        {
            set_error(-3, "pattern-set shards must end below 2^40 bytes of global offset (key layout, csrc/common.h)");
            return -3;
        }
        AcLaunch a;
        a.text = (const uint8_t *)sh->d_text;
        a.avail_len = sh->avail_len;
        a.own_begin = sh->own_begin;
        a.own_end = own_end;
        a.global_offset = sh->global_offset;
        a.prev_byte = sh->prev_byte;
        a.next_byte = sh->next_byte;
        a.out = E.d_list[slot];
        a.cap = want_positions ? E.key_cap : 0;
        a.counter = slot_counter(E, slot);
        a.whole_word = plan->whole_word;
        a.want_positions = (uint32_t)want_positions;
        launch_ac(plan, pd->ac, a, E.sm_count, stream);
        return 0;
    }
    LitDevParams p;
    memset(&p, 0, sizeof p);
    p.text = (const uint8_t *)sh->d_text;
    p.avail_len = sh->avail_len;
    p.own_begin = sh->own_begin;
    p.own_end = own_end;
    p.global_offset = sh->global_offset;
    p.prev_byte = sh->prev_byte;
    p.next_byte = sh->next_byte;
    uint64_t total_groups;
    if (plan->filter == FILTER_ALIGNED4)
    {
        total_groups = sh->avail_len / 16;
        p.tail_start = total_groups ? total_groups * 16 - 3 : 0;
    }
    else
    {
        total_groups = sh->avail_len >= 20 ? (sh->avail_len - 20) / 16 + 1 : 0; // vector + next word readable
        p.tail_start = total_groups * 16;
    }
    p.group_begin = sh->own_begin / 16;
    p.group_end = (own_end + 2) / 16 + 1;
    if (p.group_end > total_groups) p.group_end = total_groups;
    if (p.group_begin > p.group_end) p.group_begin = p.group_end;
    p.m = plan->m;
    p.emit_len = plan->emit_len;
    for (int d = 0; d < 4; d++) p.K[d] = plan->K[d];
    p.fold = plan->fold;
    p.win_mask = plan->win_mask;
    p.mulc[0] = 1u << 24;
    p.mulc[1] = 1u << 16;
    p.mulc[2] = 1u << 8;
    p.pat_val = pd->d_pat_val;
    p.pat_mask = pd->d_pat_mask;
    p.out = E.d_list[slot];
    p.cap = want_positions ? E.key_cap : 0;
    p.counter = slot_counter(E, slot);
    p.whole_word = plan->whole_word;
    p.want_positions = (uint32_t)want_positions;
    launch_literal(plan, p, E.sm_count, stream);
    return 0;
}

int reset_counter(DevCtx &E, int slot, cudaStream_t stream)
{
    if (E.counter_clean[slot]) return 0;
    CK(cudaMemsetAsync(slot_counter(E, slot), 0, 64, stream));
    E.counter_clean[slot] = true;
    return 0;
}

// ---------------------------------------------------------------------------------------------
// k_finish — the tail of every scan: publishes the occurrence count, and when the list is short (<= PACK_KEYS, the
// normal case on low-hit-rate corpora: 10 240 occurrences in the 10 GiB benchmark shard) sorts it into d_pack (the
// device copy later stages and a multi-GPU host's gather read), from where it goes to the host's pinned
// memory — one fixed-size copy of the packed row behind the kernel — so that count AND sorted occurrences reach the host
// with the one synchronisation the scan needs anyway: no CUB launches, no second read-back.
//
// The sort is a RANK sort spread over the GPU: a CTA owns 32 keys, streams the whole list through shared memory in
// 2048-key pieces and counts, for each of its keys, the keys that order before it (16 lanes per key, each taking every
// 16th list entry; lanes of one slice read the same word — a broadcast); that count is the key's final position.  n^2
// compares, 10^8 for 10 240 keys, on 320 CTAs x 16 warps — instead of the 105 barrier-separated passes of a one-CTA
// bitonic network: with ~10^4 keys the quadratic algorithm is the one that uses the machine.
// The last CTA to finish zeroes the scan counter and the done-counter for the slot's next scan.
// ---------------------------------------------------------------------------------------------
static constexpr int FIN_THREADS = 512, FIN_SLICES = 16, FIN_KEYS = FIN_THREADS / FIN_SLICES, FIN_PIECE = 2048;

__global__ void __launch_bounds__(FIN_THREADS) k_finish(unsigned long long *counter, const uint64_t *__restrict__ keys, uint64_t cap,
                                                        uint64_t *d_pack, int want_sort)
{
    __shared__ uint64_t s_keys[FIN_PIECE];
    __shared__ unsigned long long s_cnt;
    if (threadIdx.x == 0) s_cnt = counter[0];
    __syncthreads();
    const unsigned long long cnt = s_cnt;
    if (blockIdx.x == 0 && threadIdx.x == 0) d_pack[0] = cnt;
    const bool sorting = want_sort && cnt != 0 && cnt <= PACK_KEYS && cnt <= cap;
    const uint32_t n = sorting ? (uint32_t)cnt : 0u;
    // a CTA owns FIN_KEYS consecutive keys; FIN_SLICES neighbouring lanes share one key and each ranks it against every
    // FIN_SLICES-th key of the list (lanes of one slice read the same shared-memory word: broadcast; the slices read
    // consecutive words)
    const uint32_t idx = blockIdx.x * FIN_KEYS + threadIdx.x / FIN_SLICES, slice = threadIdx.x % FIN_SLICES;
    if (blockIdx.x * FIN_KEYS < n) // this CTA owns at least one key
    {
        const uint64_t mine = idx < n ? keys[idx] : ~0ull;
        uint32_t rank = 0;
        for (uint32_t base = 0; base < n; base += FIN_PIECE)
        {
            const uint32_t m = n - base < FIN_PIECE ? n - base : FIN_PIECE;
            for (uint32_t j = threadIdx.x; j < FIN_PIECE; j += FIN_THREADS) s_keys[j] = j < m ? keys[base + j] : ~0ull;
            __syncthreads();
            // keys are distinct (an occurrence key is unique), so "<" alone is a total order; padding (~0) never counts
            const uint32_t mr = (m + 63u) & ~63u;
#pragma unroll 8
            for (uint32_t j = slice; j < mr; j += FIN_SLICES) rank += s_keys[j] < mine ? 1u : 0u;
            __syncthreads();
        }
#pragma unroll
        for (int o = 1; o < FIN_SLICES; o <<= 1) rank += __shfl_xor_sync(0xffffffffu, rank, o);
        if (idx < n && slice == 0) d_pack[1 + rank] = mine;
    }
    // the last CTA out resets the counters (counter[1] counts finished CTAs)
    __syncthreads();
    if (threadIdx.x == 0)
    {
        __threadfence();
        const unsigned long long done = atomicAdd(&counter[1], 1ULL);
        if (done == gridDim.x - 1)
        {
            counter[0] = 0;
            counter[1] = 0;
        }
    }
}

// k_finish of the scan whose kernels were just enqueued on `stream`, on the same stream: being short, it is cheaper to run
// it between two scans than beside one (a CTA that needs registers on an SM the scan's persistent CTAs already fill only
// gets there when they exit, so an overlapped finish serialises anyway and slows the scan's tail).
int finish_scan(DevCtx &E, int slot, int want_sort, cudaStream_t stream, bool keys_to_host)
{
    k_finish<<<PACK_KEYS / FIN_KEYS, FIN_THREADS, 0, stream>>>(slot_counter(E, slot), E.d_list[slot], E.key_cap, E.d_pack[slot],
                                                                 (want_sort && E.d_list[slot]) ? 1 : 0);
    CK(cudaGetLastError());
    // count + (possibly) sorted keys to the host in one DMA of the whole packed row: 128 KiB over PCIe is ~5 us, cheaper than
    // having the sort's scattered 8-byte stores go through mapped memory
    const size_t words = want_sort && keys_to_host ? PACK_KEYS + 1 : 1;
    CK(cudaMemcpyAsync(E.h_pack[slot], E.d_pack[slot], words * sizeof(uint64_t), cudaMemcpyDeviceToHost, stream));
    CK(cudaEventRecord(E.ev_done[slot], stream));
    count_launch();
    E.counter_clean[slot] = true;
    return 0;
}

// Sorts the first n keys of the slot's list; the sorted list ends up in *sorted (the list or the alternate buffer).
int sort_keys(DevCtx &E, int slot, uint64_t n, int end_bit, cudaStream_t stream, const uint64_t **sorted)
{
    *sorted = E.d_list[slot];
    if (n < 2) return 0;
    cub::DoubleBuffer<uint64_t> db(E.d_list[slot], E.d_alt);
    size_t need = 0;
    CK(cub::DeviceRadixSort::SortKeys(nullptr, need, db, (int64_t)n, 0, end_bit, stream));
    if (need > E.sort_tmp_bytes)
    {
        CK(cudaStreamSynchronize(stream));
        cudaFree(E.d_sort_tmp);
        E.d_sort_tmp = nullptr;
        E.sort_tmp_bytes = 0;
        CK(cudaMalloc(&E.d_sort_tmp, need));
        E.sort_tmp_bytes = need;
    }
    CK(cub::DeviceRadixSort::SortKeys(E.d_sort_tmp, need, db, (int64_t)n, 0, end_bit, stream));
    // (CUB's own launches — histogram, scan, one onesweep pass per 8 key bits — are library kernels and are not counted
    // by krep_b200_launch_count, which reports this library's hand-written kernels only)
    *sorted = db.Current();
    return 0;
}

static int bits_for(uint64_t v)
{
    int b = 1;
    while (b < 64 && (v >> b)) b++;
    return b;
}

int key_end_bit(const Plan *plan, uint64_t max_offset, RegexMode mode)
{
    const int shift = plan->is_ac ? AC_END_SHIFT : regex_key_shift(mode);
    int b = bits_for(max_offset) + shift;
    return b > 64 ? 64 : b;
}

// ---------------------------------------------------------------------------------------------
// -c on the device: line bounds of every occurrence (find_line_start / find_line_end, krep.c:363-408), so that the
// line-counting replay needs no host copy of the text.  One warp per (sorted) occurrence.  For literal plans the keys
// are sorted by start, so the backward scan stops at the previous occurrence and the forward scan at the next one
// (markers LB_SAME_AS_* are resolved by one pass on the host): the total work is O(text), however long the lines are.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_line_bounds(const uint8_t *__restrict__ text, uint64_t avail, uint64_t go,
                                                     const uint64_t *__restrict__ keys, uint64_t n, int is_ac, int has_prev,
                                                     int has_next, uint64_t *__restrict__ out)
{
    const uint64_t i = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (i >= n) return;
    auto start_of = [&](uint64_t key) -> uint64_t {
        if (!is_ac) return (key >> LIT_TAG_BITS) - go;
        return (key >> AC_END_SHIFT) - (1024 - ((key >> AC_LEN_SHIFT) & 1023)) - go;
    };
    const uint64_t s = start_of(keys[i]);
    const uint64_t lb = (!is_ac && i > 0) ? start_of(keys[i - 1]) : 0;       // backward scan covers [lb, s)
    const uint64_t ub = (!is_ac && i + 1 < n) ? start_of(keys[i + 1]) : avail; // forward scan covers [s, ub)
    // backward: last '\n' in [lb, s), 128 bytes per step (4 per lane)
    uint64_t ls = (!is_ac && i > 0) ? LB_SAME_AS_PREV : (has_prev ? LB_OUTSIDE_SHARD : go);
    for (uint64_t hi = s; hi > lb;)
    {
        const uint64_t w0 = hi >= lb + 128 ? hi - 128 : lb; // window [w0, hi)
        int best = -1;
#pragma unroll
        for (int k = 0; k < 4; k++)
        {
            const uint64_t p = w0 + (uint64_t)lane * 4 + k;
            if (p < hi && text[p] == '\n') best = lane * 4 + k;
        }
        best = __reduce_max_sync(0xffffffffu, best);
        if (best >= 0)
        {
            ls = go + w0 + (uint64_t)best + 1;
            break;
        }
        hi = w0;
    }
    // forward: first '\n' in [s, ub)
    uint64_t le = (!is_ac && i + 1 < n) ? LB_SAME_AS_NEXT : (has_next ? LB_OUTSIDE_SHARD : go + avail);
    for (uint64_t lo = s; lo < ub; lo += 128)
    {
        int best = 1 << 20;
#pragma unroll
        for (int k = 3; k >= 0; k--)
        {
            const uint64_t p = lo + (uint64_t)lane * 4 + k;
            if (p < ub && text[p] == '\n') best = lane * 4 + k;
        }
        best = __reduce_min_sync(0xffffffffu, best);
        if (best < (1 << 20))
        {
            le = go + lo + (uint64_t)best;
            break;
        }
    }
    if (lane == 0)
    {
        out[2 * i] = ls;
        out[2 * i + 1] = le;
    }
}

static int line_bounds(DevCtx &E, const Plan *plan, const krep_b200_shard_t *sh, const uint64_t *d_sorted, uint64_t n,
                       cudaStream_t stream, const uint64_t **d_bounds)
{
    *d_bounds = nullptr;
    if (n == 0) return 0;
    if (2 * n > E.bounds_cap)
    {
        CK(cudaStreamSynchronize(stream));
        cudaFree(E.d_bounds);
        E.d_bounds = nullptr;
        E.bounds_cap = 0;
        const uint64_t cap = 2 * n + n / 4 + 1024;
        CK(cudaMalloc(&E.d_bounds, cap * sizeof(uint64_t)));
        E.bounds_cap = cap;
    }
    const uint64_t threads = n * 32;
    // a shard that begins right after a newline (or ends right before one) does not cut a line
    const int has_prev = sh->prev_byte >= 0 && sh->prev_byte != '\n';
    const int has_next = sh->next_byte >= 0 && sh->next_byte != '\n';
    k_line_bounds<<<(unsigned)((threads + 255) / 256), 256, 0, stream>>>((const uint8_t *)sh->d_text, sh->avail_len, sh->global_offset,
                                                                        d_sorted, n, plan->is_ac ? 1 : 0, has_prev, has_next, E.d_bounds);
    CK(cudaGetLastError());
    count_launch();
    *d_bounds = E.d_bounds;
    return 0;
}

// One shard scan = counter reset (only if the previous scan did not leave it clean), filter+verify kernel, k_finish.
// scan_begin enqueues all three and returns; scan_end waits for them (the scan's single synchronisation), and only
// if the list was too long for k_finish runs the radix sort (or, if it overflowed the list, grows it and rescans).
int scan_begin(DevCtx &E, const Plan *plan, const krep_b200_shard_t *sh, int want_positions, cudaStream_t stream, int *slot_out)
{
    if (!stream) stream = E.scan_stream;
    if (want_positions && ensure_keys(E, 1) != 0) return -2;
    const int slot = E.next_slot;
    if (E.pend[slot].active)
    {
        set_error(-3, "krep_b200_scan_shard_begin: %d scans are already in flight on device %d", SCAN_SLOTS, E.device);
        return -3;
    }
    // the slot's previous occupant: its k_finish (finish stream) must be done with the list and the counter
    CK(cudaStreamWaitEvent(stream, E.ev_done[slot], 0));
    if (reset_counter(E, slot, stream) != 0) return -2;
    CK(cudaEventRecord(E.ev_a[slot], stream));
    int rc = launch_scan(E, plan, sh, want_positions, stream, slot);
    if (rc != 0) return rc;
    CK(cudaEventRecord(E.ev_b[slot], stream));
    CK(cudaGetLastError());
    if (finish_scan(E, slot, want_positions, stream) != 0) return -2;
    PendingScan &P = E.pend[slot];
    P.active = true;
    P.plan = plan;
    P.shard = *sh;
    P.want_positions = want_positions;
    P.stream = stream;
    E.next_slot = (slot + 1) % SCAN_SLOTS;
    *slot_out = slot;
    return 0;
}

int scan_end(DevCtx &E, int slot, ScanOut *out)
{
    PendingScan &P = E.pend[slot];
    if (slot < 0 || slot >= SCAN_SLOTS || !P.active)
    {
        set_error(-3, "krep_b200_scan_shard_end: no scan in flight in slot %d", slot);
        return -3;
    }
    P.active = false;
    const Plan *plan = P.plan;
    const krep_b200_shard_t *sh = &P.shard;
    cudaStream_t stream = P.stream;
    reset_kernel_ms();
    for (int attempt = 0; attempt < 3; attempt++)
    {
        // wait for this scan's k_finish only (not for the stream: the next scan may already be running behind it)
        CK(cudaEventSynchronize(E.ev_done[slot]));
        const uint64_t cnt = E.h_pack[slot][0];
        float ms = 0.f;
        cudaEventElapsedTime(&ms, E.ev_a[slot], E.ev_b[slot]);
        add_kernel_ms(ms);
        *out = ScanOut();
        out->count = cnt;
        out->device = E.device;
        out->serial = ++E.serial;
        E.result_stream = stream;
        if (!P.want_positions) return 0;
        if (cnt <= E.key_cap)
        {
            int rc = 0;
            out->stored = cnt;
            if (cnt <= PACK_KEYS)
            {
                out->d_keys = E.d_pack[slot] + 1; // the rank sort writes the ordered list here (the slot's list stays raw)
                out->h_sorted = E.h_pack[slot] + 1;
            }
            else
                rc = sort_keys(E, slot, cnt, key_end_bit(plan, sh->global_offset + sh->avail_len), stream, &out->d_keys);
            if (rc == 0 && plan->count_lines) rc = line_bounds(E, plan, sh, out->d_keys, cnt, stream, &out->d_bounds);
            return rc;
        }
        // the list overflowed (the counter stays exact past capacity): grow it and scan again
        out->overflow = 1;
        for (int s2 = 0; s2 < SCAN_SLOTS; s2++)
            if (s2 != slot && E.pend[s2].active)
            {
                set_error(-3, "krep_b200_scan_shard_end: the occurrence list overflowed while another scan is in flight; end each "
                              "scan before beginning the next until the list has grown");
                return -3;
            }
        if (ensure_keys(E, cnt + cnt / 8 + 1024) != 0) return -2;
        if (reset_counter(E, slot, stream) != 0) return -2;
        CK(cudaEventRecord(E.ev_a[slot], stream));
        int rc = launch_scan(E, plan, sh, 1, stream, slot);
        if (rc != 0) return rc;
        CK(cudaEventRecord(E.ev_b[slot], stream));
        if (finish_scan(E, slot, 1, stream) != 0) return -2;
    }
    set_error(-4, "occurrence list kept overflowing");
    return -4;
}

int scan_shard(DevCtx &E, const Plan *plan, const krep_b200_shard_t *sh, int want_positions, cudaStream_t stream, ScanOut *out)
{
    int slot = 0;
    int rc = scan_begin(E, plan, sh, want_positions, stream, &slot);
    if (rc != 0) return rc;
    return scan_end(E, slot, out);
}

// Sorted keys on the host: already there when they came back packed with the count, else one copy on the stream that
// produced them (so the copy is ordered after the sort whatever stream the caller scanned on).
int fetch_keys(DevCtx &E, const ScanOut &so, const uint64_t **h)
{
    *h = nullptr;
    if (so.stored == 0) return 0;
    if (so.h_sorted)
    {
        *h = so.h_sorted;
        return 0;
    }
    if (so.stored > E.h_keys_cap)
    {
        cudaFreeHost(E.h_keys);
        E.h_keys = nullptr;
        E.h_keys_cap = 0;
        uint64_t cap = so.stored + so.stored / 4;
        if (cap < (1u << 16)) cap = 1u << 16;
        CK(cudaMallocHost(&E.h_keys, cap * sizeof(uint64_t)));
        E.h_keys_cap = cap;
    }
    cudaStream_t s = E.result_stream ? E.result_stream : E.scan_stream;
    CK(cudaMemcpyAsync(E.h_keys, so.d_keys, so.stored * sizeof(uint64_t), cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    *h = E.h_keys;
    return 0;
}

// Ascending lists -> one ascending list.  Concatenation first (the common case is already ordered: literal keys of
// rank-ordered shards), then one in-place merge per list boundary that is out of order.
uint64_t merge_key_lists(const uint64_t *const *lists, const uint64_t *counts, uint32_t n_lists, uint64_t *dst)
{
    uint64_t total = 0;
    std::vector<uint64_t> cut;
    for (uint32_t i = 0; i < n_lists; i++)
    {
        if (counts[i] == 0) continue;
        if (dst + total != lists[i]) memmove(dst + total, lists[i], counts[i] * sizeof(uint64_t));
        cut.push_back(total);
        total += counts[i];
    }
    for (size_t i = 1; i < cut.size(); i++)
        if (dst[cut[i] - 1] > dst[cut[i]]) std::inplace_merge(dst, dst + cut[i], dst + (i + 1 < cut.size() ? cut[i + 1] : total));
    return total;
}

// ---------------------------------------------------------------------------------------------
// synthetic corpus
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_corpus(const __grid_constant__ CorpusParams c, uint8_t *dst, uint64_t global_offset,
                                                uint64_t len)
{
    // dst[k] = byte(global_offset + k); global_offset is a multiple of 16 (checked on the host)
    const uint64_t groups = (len + 15) / 16;
    for (uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; g < groups; g += (uint64_t)gridDim.x * blockDim.x)
    {
        alignas(16) uint8_t b[16];
        corpus_fill16(c, global_offset + g * 16, b);
        const uint64_t off = g * 16;
        if (off + 16 <= len && (((uintptr_t)(dst + off)) & 15) == 0)
            *reinterpret_cast<uint4 *>(dst + off) = *reinterpret_cast<const uint4 *>(b);
        else
            for (int k = 0; k < 16 && off + k < len; k++) dst[off + k] = b[k];
    }
}

static int corpus_params(const krep_b200_corpus_spec_t *spec, CorpusParams *c)
{
    memset(c, 0, sizeof *c);
    c->seed = spec->seed;
    c->plant_seed = spec->plant_seed;
    c->plant_period = spec->plant_period;
    c->needle_len = spec->needle_len;
    c->flags = spec->flags;
    if (spec->needle_len > 64)
    {
        set_error(-3, "corpus needle longer than 64 bytes");
        return -3;
    }
    if (spec->plant_period && (spec->plant_period % 16 != 0 || spec->plant_period < 4ull * spec->needle_len + 32))
    {
        set_error(-3, "corpus plant_period must be a multiple of 16 and >= 4*needle_len+32");
        return -3;
    }
    if (spec->needle_len) memcpy(c->needle, spec->needle, spec->needle_len);
    return 0;
}

} // namespace kb

using namespace kb;

// ---------------------------------------------------------------------------------------------
// C ABI: lifetime, plans, shard scan, corpus
// ---------------------------------------------------------------------------------------------
extern "C" {

int krep_b200_init(int device)
{
    g_keep_visible = true;
    warm_join();
    std::lock_guard<std::recursive_mutex> lk(engine_mutex());
    clear_error();
    if (visible_devices() == 0)
    {
        set_error(-1, "no CUDA device available; this engine has no CPU fallback");
        return -1;
    }
    if (device < 0)
    {
        device = primary_device();
        if (device < 0) return -1;
    }
    if (!ctx_get(device)) return krep_b200_last_error() ? krep_b200_last_error() : -1;
    g_primary = device;
    return 0;
}
void krep_b200_shutdown(void) { engine_shutdown(); }
int krep_b200_last_error(void) { return t_err; }
const char *krep_b200_last_error_string(void) { return t_errmsg; }
const char *krep_b200_version(void) { return "krep_b200 0.2.0 (sm_90a)"; }
int krep_b200_device_count(void)
{
    warm_join();
    return visible_devices();
}
void krep_b200_warmup(void) { warm_start(); }

float krep_b200_last_kernel_ms(void) { return t_kernel_ms; }
uint64_t krep_b200_launch_count(void) { return g_launches; }
void krep_b200_reset_launch_count(void) { g_launches = 0; }

krep_b200_plan_t *krep_b200_plan_create(const search_params_t *params, int algo)
{
    warm_join();
    std::lock_guard<std::recursive_mutex> lk(engine_mutex());
    clear_error();
    if (!params) return nullptr;
    if (visible_devices() == 0)
    {
        set_error(-1, "no CUDA device available; this engine has no CPU fallback");
        return nullptr;
    }
    return reinterpret_cast<krep_b200_plan_t *>(plan_build(params, resolve_algo(params, algo), krep_b200_get_only_matching()));
}
void krep_b200_plan_destroy(krep_b200_plan_t *plan)
{
    std::lock_guard<std::recursive_mutex> lk(engine_mutex());
    plan_free(reinterpret_cast<Plan *>(plan));
}
const char *krep_b200_plan_filter_name(const krep_b200_plan_t *plan)
{
    return plan ? reinterpret_cast<const Plan *>(plan)->filter_name.c_str() : "";
}

static void fill_result(const ScanOut &so, const krep_b200_shard_t *shard, int slot, krep_b200_device_result_t *out)
{
    out->count = so.count;
    out->stored = so.stored;
    out->d_keys = so.d_keys;
    out->overflow = so.overflow;
    out->text_len = shard->global_offset + shard->avail_len;
    out->d_line_bounds = so.d_bounds;
    out->device = so.device;
    out->slot = slot;
    out->serial = so.serial;
}

int krep_b200_scan_shard_begin(const krep_b200_plan_t *plan, const krep_b200_shard_t *shard, int want_positions, void *stream,
                               int *ticket)
{
    std::lock_guard<std::recursive_mutex> lk(engine_mutex());
    clear_error();
    if (!plan || !shard || !ticket)
    {
        set_error(-3, "krep_b200_scan_shard_begin: null argument");
        return -3;
    }
    DeviceGuard guard;
    DevCtx *C = ctx_of_pointer(shard->d_text);
    if (!C) return -1;
    int slot = 0;
    int rc = scan_begin(*C, reinterpret_cast<const Plan *>(plan), shard, want_positions, (cudaStream_t)stream, &slot);
    *ticket = C->device * SCAN_SLOTS + slot;
    return rc;
}

int krep_b200_scan_shard_end(int ticket, krep_b200_device_result_t *out)
{
    std::lock_guard<std::recursive_mutex> lk(engine_mutex());
    clear_error();
    if (!out || ticket < 0 || ticket >= MAX_DEV * SCAN_SLOTS)
    {
        set_error(-3, "krep_b200_scan_shard_end: bad argument");
        return -3;
    }
    DeviceGuard guard;
    DevCtx *C = ctx_get(ticket / SCAN_SLOTS);
    if (!C) return -1;
    const int slot = ticket % SCAN_SLOTS;
    const krep_b200_shard_t shard = C->pend[slot].shard;
    ScanOut so;
    int rc = scan_end(*C, slot, &so);
    fill_result(so, &shard, slot, out);
    return rc;
}

int krep_b200_scan_shard(const krep_b200_plan_t *plan, const krep_b200_shard_t *shard, int want_positions,
                         void *stream, krep_b200_device_result_t *out)
{
    int ticket = 0;
    int rc = krep_b200_scan_shard_begin(plan, shard, want_positions, stream, &ticket);
    if (rc != 0) return rc;
    if (!out)
    {
        set_error(-3, "krep_b200_scan_shard: null argument");
        return -3;
    }
    return krep_b200_scan_shard_end(ticket, out);
}

} // extern "C"

// One k_regex_lines scan of a shard in the given mode on the device's scan stream, its keys sorted on the device:
// *d_sorted (device, *cnt keys; short lists sorted by k_finish into d_pack, longer ones by the radix sort, enqueued on
// the stream) and the count mode's line counter.  Unlike scan_end's retry, an overflow re-scan keeps the
// mode and zeroes the line counter again, so the keys and the count are those of one complete scan.  The lists stay valid
// until the next scan on the device.  long_lines: the long-line pass follows the scan (DESIGN §12.8).
int kb::regex_scan_keys(DevCtx &E, const Plan *plan, const krep_b200_shard_t *shard, RegexMode mode, const char *who, uint64_t *cnt_out,
                        const uint64_t **d_sorted, uint64_t *device_lines, const LongLineOpts *long_lines, const RegexBatchDev *batch)
{
    for (int s = 0; s < SCAN_SLOTS; s++)
        if (E.pend[s].active)
        {
            set_error(-3, "%s: a scan is in flight on device %d", who, E.device);
            return -3;
        }
    const uint64_t n_lines = batch ? batch->n_texts : 1; // line counters: one per text of a batch
    if (ensure_keys(E, 1) != 0 || (mode == RX_COUNT && ensure_line_out(E, (n_lines + 1) / 2) != 0)) return -2;
    unsigned long long *d_lines = mode == RX_COUNT ? (unsigned long long *)E.d_line_out : nullptr;
    const int slot = 0;
    cudaStream_t st = E.scan_stream;
    ++E.serial; // slot 0's lists are overwritten: a device result handed out earlier no longer passes the stale check
    for (int attempt = 0; attempt < 3; attempt++)
    {
        CK(cudaStreamWaitEvent(st, E.ev_done[slot], 0));
        if (reset_counter(E, slot, st) != 0) return -2;
        if (d_lines) CK(cudaMemsetAsync(d_lines, 0, n_lines * sizeof(unsigned long long), st));
        int rc = launch_scan(E, plan, shard, 1, st, slot, d_lines, mode == RX_OFFSETS, batch, long_lines);
        if (rc != 0) return rc;
        if (finish_scan(E, slot, 1, st) != 0) return -2;
        if (d_lines) CK(cudaMemcpyAsync(E.h_line_out, d_lines, n_lines * sizeof(uint64_t), cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
        const uint64_t cnt = E.h_pack[slot][0];
        if (cnt > E.key_cap)
        {
            if (ensure_keys(E, cnt + cnt / 8 + 1024) != 0) return -2;
            continue;
        }
        *d_sorted = E.d_pack[slot] + 1;
        if (cnt > PACK_KEYS)
        {
            rc = sort_keys(E, slot, cnt, key_end_bit(plan, shard->global_offset + shard->avail_len, mode), st, d_sorted);
            if (rc != 0) return rc;
        }
        *cnt_out = cnt;
        if (device_lines)
            for (uint64_t i = 0; i < n_lines; i++) device_lines[i] = d_lines ? E.h_line_out[i] : 0;
        return 0;
    }
    set_error(-4, "occurrence list kept overflowing");
    return -4;
}

extern "C" {

// One k_regex_lines scan in the given mode (followed by the long-line pass when long_lines is set), its keys sorted and
// read back.
static int64_t regex_scan_raw(const char *who, const krep_b200_plan_t *plan_, const krep_b200_shard_t *shard, int mode,
                              const LongLineOpts *long_lines, uint64_t *keys, uint64_t cap, uint64_t *device_lines)
{
    std::lock_guard<std::recursive_mutex> lk(engine_mutex());
    clear_error();
    const Plan *plan = reinterpret_cast<const Plan *>(plan_);
    if (!plan || !shard || (cap && !keys))
    {
        set_error(-3, "%s: null argument", who);
        return -3;
    }
    if (!plan->is_regex || !regex_mode_available(*plan->rx, mode))
    {
        set_error(-3, "%s: mode %d is not available for this plan", who, mode);
        return -3;
    }
    DeviceGuard guard;
    DevCtx *Cp = ctx_of_pointer(shard->d_text);
    if (!Cp) return -1;
    DevCtx &E = *Cp;
    uint64_t cnt = 0;
    const uint64_t *d_sorted = nullptr;
    const int rc = regex_scan_keys(E, plan, shard, (RegexMode)mode, who, &cnt, &d_sorted, device_lines, long_lines);
    if (rc != 0) return rc;
    const uint64_t n = cnt < cap ? cnt : cap;
    if (cnt <= PACK_KEYS)
    {
        if (n) memcpy(keys, E.h_pack[0] + 1, n * sizeof(uint64_t));
    }
    else if (n)
    {
        CK(cudaMemcpyAsync(keys, d_sorted, n * sizeof(uint64_t), cudaMemcpyDeviceToHost, E.scan_stream));
        CK(cudaStreamSynchronize(E.scan_stream));
    }
    return (int64_t)cnt;
}

int64_t krep_b200_regex_scan_shard_raw(const krep_b200_plan_t *plan, const krep_b200_shard_t *shard, int mode, uint64_t *keys,
                                       uint64_t cap, uint64_t *device_lines)
{
    return regex_scan_raw("krep_b200_regex_scan_shard_raw", plan, shard, mode, nullptr, keys, cap, device_lines);
}

int64_t krep_b200_regex_scan_shard_long_raw(const krep_b200_plan_t *plan, const krep_b200_shard_t *shard, int mode,
                                            uint32_t slice_bytes, uint32_t ckpt_bytes, uint64_t *keys, uint64_t cap,
                                            uint64_t *device_lines)
{
    const char *who = "krep_b200_regex_scan_shard_long_raw";
    LongLineOpts o;
    if (long_lines_opts(who, slice_bytes, ckpt_bytes, &o) != 0) return -3;
    return regex_scan_raw(who, plan, shard, mode, long_lines_default() ? &o : nullptr, keys, cap, device_lines);
}

int krep_b200_export_keys(const krep_b200_device_result_t *dev, void *d_dst, uint64_t max_keys, void *stream)
{
    std::lock_guard<std::recursive_mutex> lk(engine_mutex());
    clear_error();
    if (!dev || !d_dst) return -3;
    const uint64_t n = dev->stored < max_keys ? dev->stored : max_keys;
    if (n == 0) return 0;
    DeviceGuard guard;
    DevCtx *C = ctx_get(dev->device);
    if (!C) return -1;
    cudaStream_t s = stream ? (cudaStream_t)stream : (C->result_stream ? C->result_stream : C->scan_stream);
    CK(cudaMemcpyAsync(d_dst, dev->d_keys, n * sizeof(uint64_t), cudaMemcpyDeviceToDevice, s));
    if (!stream) CK(cudaStreamSynchronize(s));
    return 0;
}

// [count, key_0 .. key_{k-1}] with k = min(stored, max_keys) in one device-to-device copy: the row a multi-GPU host
// hands to its gather (krep_b200/sharding.py).  count is the exact occurrence count even when k < count.
int krep_b200_export_packed(const krep_b200_device_result_t *dev, void *d_dst, uint64_t max_keys, void *stream)
{
    std::lock_guard<std::recursive_mutex> lk(engine_mutex());
    clear_error();
    if (!dev || !d_dst) return -3;
    DeviceGuard guard;
    DevCtx *C = ctx_get(dev->device);
    if (!C) return -1;
    cudaStream_t s = stream ? (cudaStream_t)stream : (C->result_stream ? C->result_stream : C->scan_stream);
    const uint64_t n = dev->stored < max_keys ? dev->stored : max_keys;
    if (dev->serial == C->serial && dev->stored <= PACK_KEYS && dev->slot >= 0 && dev->slot < SCAN_SLOTS)
        CK(cudaMemcpyAsync(d_dst, C->d_pack[dev->slot], (n + 1) * sizeof(uint64_t), cudaMemcpyDeviceToDevice, s));
    else
    {
        CK(cudaMemcpyAsync(d_dst, C->d_pack[dev->slot & (SCAN_SLOTS - 1)], sizeof(uint64_t), cudaMemcpyDeviceToDevice, s));
        if (n) CK(cudaMemcpyAsync((uint64_t *)d_dst + 1, dev->d_keys, n * sizeof(uint64_t), cudaMemcpyDeviceToDevice, s));
    }
    if (!stream) CK(cudaStreamSynchronize(s));
    return 0;
}

// The same row for a scan that is still in flight (ticket of krep_b200_scan_shard_begin): enqueued on the scan's own
// stream behind its finish kernel, so the host does not have to know the count first — the whole fixed-size row
// [count, key_0 .. key_{max_keys-1}] is copied (max_keys <= 16384: only lists that short are sorted by the finish kernel;
// a longer list shows up at the receiver as count > max_keys).
int krep_b200_export_packed_async(int ticket, void *d_dst, uint64_t max_keys)
{
    std::lock_guard<std::recursive_mutex> lk(engine_mutex());
    clear_error();
    if (!d_dst || ticket < 0 || ticket >= MAX_DEV * SCAN_SLOTS || max_keys > PACK_KEYS)
    {
        set_error(-3, "krep_b200_export_packed_async: bad argument");
        return -3;
    }
    DeviceGuard guard;
    DevCtx *C = ctx_get(ticket / SCAN_SLOTS);
    if (!C) return -1;
    const int slot = ticket % SCAN_SLOTS;
    if (!C->pend[slot].active)
    {
        set_error(-3, "krep_b200_export_packed_async: no scan in flight for this ticket");
        return -3;
    }
    cudaStream_t s = C->pend[slot].stream;
    CK(cudaStreamWaitEvent(s, C->ev_done[slot], 0)); // the finish kernel runs on its own stream
    CK(cudaMemcpyAsync(d_dst, C->d_pack[slot], (max_keys + 1) * sizeof(uint64_t), cudaMemcpyDeviceToDevice, s));
    return 0;
}

uint64_t krep_b200_merge_keys(const uint64_t *const *lists, const uint64_t *counts, uint32_t n_lists, uint64_t *dst)
{
    if (!lists || !counts || !dst) return 0;
    return merge_key_lists(lists, counts, n_lists, dst);
}

uint64_t krep_b200_ac_key_end(uint64_t key) { return key >> AC_END_SHIFT; }
uint64_t krep_b200_ac_key_start(uint64_t key)
{
    const uint64_t len = 1024 - ((key >> AC_LEN_SHIFT) & 1023);
    return (key >> AC_END_SHIFT) - len;
}
uint32_t krep_b200_ac_key_pattern(uint64_t key) { return (uint32_t)(key & (AC_MAX_PATTERNS - 1)); }

int krep_b200_corpus_generate(const krep_b200_corpus_spec_t *spec, void *d_dst, uint64_t global_offset, uint64_t len,
                              void *stream)
{
    std::lock_guard<std::recursive_mutex> lk(engine_mutex());
    clear_error();
    DeviceGuard guard;
    DevCtx *C = ctx_of_pointer(d_dst);
    if (!C) return -1;
    CorpusParams c;
    if (corpus_params(spec, &c) != 0) return -3;
    if (global_offset % 16 != 0)
    {
        set_error(-3, "corpus global_offset must be a multiple of 16");
        return -3;
    }
    if (len == 0) return 0;
    cudaStream_t s = stream ? (cudaStream_t)stream : C->scan_stream;
    const uint64_t groups = (len + 15) / 16;
    uint64_t blocks = (groups + 255) / 256;
    const uint64_t maxb = (uint64_t)C->sm_count * 16;
    if (blocks > maxb) blocks = maxb;
    k_corpus<<<(unsigned)blocks, 256, 0, s>>>(c, (uint8_t *)d_dst, global_offset, len);
    CK(cudaGetLastError());
    if (!stream) CK(cudaStreamSynchronize(s));
    return 0;
}

int krep_b200_corpus_generate_host(const krep_b200_corpus_spec_t *spec, void *dst, uint64_t global_offset, uint64_t len)
{
    CorpusParams c;
    if (corpus_params(spec, &c) != 0) return -3;
    uint8_t *o = (uint8_t *)dst;
    uint64_t i = global_offset, end = global_offset + len;
    while (i < end)
    {
        const uint64_t g0 = i & ~15ull;
        uint8_t b[16];
        corpus_fill16(c, g0, b);
        for (uint64_t k = i - g0; k < 16 && g0 + k < end; k++) o[g0 + k - global_offset] = b[k];
        i = g0 + 16;
    }
    return 0;
}

} // extern "C"
