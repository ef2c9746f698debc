// tsfx_api.cu -- the C ABI of libtsfx.so (include/tsfx.h): context, plan, extraction entry points, and the native
// runtime around the kernels: pinned host pool, threaded pageable->pinned staging ring, the row-block pipeline of the
// long-frame path (stage (a) + kernels + result transfer on three streams), multi-GPU result placement.
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <condition_variable>
#include <functional>
#include <map>
#include <mutex>
#include <new>
#include <string>
#include <thread>
#include <unordered_map>
#include <vector>

#include "tsfx_common.cuh"
#include "tsfx_kernels.h"
#include "tsfx_csr.h"
#include "tsfx_roll.cuh"
#include "tsfx_impute.h"
#include "tsfx_select.h"

using namespace tsfx;

static std::string g_create_error;

namespace tsfx {
int grid_waves(int dflt) {
    static int v = -1;
    if (v < 0) { const char* e = getenv("TSFX_GRID_WAVES"); v = e ? atoi(e) : 0; }
    return v > 0 ? v : dflt;
}
int global_above() {
    static int v = -1;
    if (v < 0) { const char* e = getenv("TSFX_GLOBAL_ABOVE"); v = e ? atoi(e) : 0; if (v > 227 * 1024 || v < 0) v = 0; }
    return v;
}
int global_ctas_env() {
    static int v = -1;
    if (v < 0) { const char* e = getenv("TSFX_GLOBAL_CTAS"); v = e ? atoi(e) : 0; if (v < 1 || v > 16) v = 0; }
    return v;
}
cudaError_t undeclared_geometry(const char* grp, const Geometry& G, const char** variant) {
    static thread_local std::string name;
    name = std::string(grp) + "/w" + std::to_string(G.wpc) + (G.gscratch ? "/global" : "/shared");
    *variant = name.c_str();
    return cudaErrorNotSupported;
}
}  // namespace tsfx

static int env_streams() {
    static int v = -1;
    if (v < 0) { const char* e = getenv("TSFX_STREAMS"); v = e ? atoi(e) : 1; if (v < 1) v = 1; if (v > 4) v = 4; }
    return v;
}

struct DevBuf {
    void* p = nullptr;
    size_t cap = 0;
    cudaError_t reserve(size_t bytes) {
        if (bytes <= cap) return cudaSuccess;
        if (p) cudaFree(p);
        p = nullptr;
        cap = 0;
        cudaError_t e = cudaMalloc(&p, bytes);
        if (e == cudaSuccess) cap = bytes;
        return e;
    }
    void release() { if (p) cudaFree(p); p = nullptr; cap = 0; }
};

// ---------------------------------------------------------------------------------- pinned host memory pool
// Page-locking is slow (a few GB/s), so blocks handed back with tsfx_host_free are cached and reused.
struct HostPool {
    std::mutex mu;
    std::multimap<size_t, void*> idle;
    std::unordered_map<void*, size_t> live;
    void* alloc(size_t bytes) {
        if (bytes == 0) bytes = 1;
        const size_t want = (bytes + ((size_t)2 << 20) - 1) & ~(((size_t)2 << 20) - 1);
        {
            std::lock_guard<std::mutex> g(mu);
            auto it = idle.lower_bound(want);
            if (it != idle.end() && it->first <= want + want / 2 + ((size_t)64 << 20)) {
                void* p = it->second;
                live[p] = it->first;
                idle.erase(it);
                return p;
            }
        }
        void* p = nullptr;
        if (cudaHostAlloc(&p, want, cudaHostAllocPortable) != cudaSuccess) {
            cudaGetLastError();
            trim();                                  // give cached blocks back and retry once
            if (cudaHostAlloc(&p, want, cudaHostAllocPortable) != cudaSuccess) { cudaGetLastError(); return nullptr; }
        }
        std::lock_guard<std::mutex> g(mu);
        live[p] = want;
        return p;
    }
    bool free(void* p) {
        std::lock_guard<std::mutex> g(mu);
        auto it = live.find(p);
        if (it == live.end()) return false;
        idle.emplace(it->second, p);
        live.erase(it);
        return true;
    }
    void trim() {
        std::lock_guard<std::mutex> g(mu);
        for (auto& kv : idle) cudaFreeHost(kv.second);
        idle.clear();
    }
    void release_all() {
        // blocks still handed out (a DataFrame may live on one) are deliberately NOT freed when the context goes away:
        // they stay valid until the process exits
        trim();
        std::lock_guard<std::mutex> g(mu);
        live.clear();
    }
};

// ---------------------------------------------------------------------------------- pageable -> device staging
// Host buffers that are not page-locked (numpy / pandas columns) are copied chunk by chunk into a ring of pinned
// slots by a few worker threads (one memcpy thread cannot feed PCIe gen5) and sent with cudaMemcpyAsync, so the
// transfer overlaps both the next chunk's memcpy and the kernels already queued.
struct Stager {
    static const int SLOTS = 3;
    size_t slot_bytes = (size_t)32 << 20;
    void* slot[SLOTS] = {nullptr, nullptr, nullptr};
    cudaEvent_t ev[SLOTS] = {nullptr, nullptr, nullptr};
    bool busy[SLOTS] = {false, false, false};
    int next = 0;
    // worker pool
    std::vector<std::thread> workers;
    std::mutex mu;
    std::condition_variable cv, cv_done;
    const char* src = nullptr;
    char* dst = nullptr;
    size_t total = 0, piece = 0;
    int next_piece = 0, n_pieces = 0, pending = 0;
    uint64_t generation = 0;
    bool stop = false;

    void worker() {
        uint64_t seen = 0;
        for (;;) {
            std::unique_lock<std::mutex> lk(mu);
            cv.wait(lk, [&] { return stop || (generation != seen && next_piece < n_pieces); });
            if (stop) return;
            while (next_piece < n_pieces) {
                const int k = next_piece++;
                lk.unlock();
                const size_t off = (size_t)k * piece;
                memcpy(dst + off, src + off, std::min(piece, total - off));
                lk.lock();
                if (--pending == 0) cv_done.notify_all();
            }
            seen = generation;
        }
    }
    void start(int n) {
        if (!workers.empty()) return;
        for (int i = 0; i < n; ++i) workers.emplace_back([this] { worker(); });
    }
    void parallel_copy(void* d, const void* s_, size_t bytes) {
        if (workers.empty() || bytes < ((size_t)1 << 20)) { memcpy(d, s_, bytes); return; }
        std::unique_lock<std::mutex> lk(mu);
        src = (const char*)s_; dst = (char*)d; total = bytes;
        n_pieces = (int)std::min<size_t>(workers.size() * 2, (bytes + ((size_t)1 << 20) - 1) >> 20);
        piece = ((bytes + n_pieces - 1) / n_pieces + 63) & ~(size_t)63;
        n_pieces = (int)((bytes + piece - 1) / piece);
        next_piece = 0; pending = n_pieces; ++generation;
        cv.notify_all();
        cv_done.wait(lk, [&] { return pending == 0; });
    }
    cudaError_t init() {
        if (slot[0]) return cudaSuccess;
        for (int i = 0; i < SLOTS; ++i) {
            cudaError_t e = cudaHostAlloc(&slot[i], slot_bytes, cudaHostAllocDefault);
            if (e != cudaSuccess) return e;
            e = cudaEventCreateWithFlags(&ev[i], cudaEventDisableTiming);
            if (e != cudaSuccess) return e;
        }
        int n = (int)std::thread::hardware_concurrency();
        const char* env = getenv("TSFX_COPY_THREADS");
        n = env ? atoi(env) : std::min(8, std::max(1, n / 2));
        if (n > 1) start(n);
        return cudaSuccess;
    }
    void release() {
        {
            std::lock_guard<std::mutex> g(mu);
            stop = true;
        }
        cv.notify_all();
        for (auto& t : workers) t.join();
        workers.clear();
        for (int i = 0; i < SLOTS; ++i) { if (slot[i]) cudaFreeHost(slot[i]); if (ev[i]) cudaEventDestroy(ev[i]); slot[i] = nullptr; ev[i] = nullptr; }
    }
    // host (pageable or pinned) -> device, asynchronous with respect to the device; returns when the LAST chunk's
    // cudaMemcpyAsync has been issued (pageable source: the source buffer is no longer needed by then)
    cudaError_t h2d(void* d, const void* h, size_t bytes, cudaStream_t st) {
        if (bytes == 0) return cudaSuccess;
        cudaPointerAttributes at;
        bool pinned = false;
        if (cudaPointerGetAttributes(&at, h) == cudaSuccess) pinned = (at.type == cudaMemoryTypeHost || at.type == cudaMemoryTypeManaged);
        else cudaGetLastError();
        if (pinned) return cudaMemcpyAsync(d, h, bytes, cudaMemcpyHostToDevice, st);
        cudaError_t e = init();
        if (e != cudaSuccess) return e;
        for (size_t off = 0; off < bytes; off += slot_bytes) {
            const size_t cnt = std::min(slot_bytes, bytes - off);
            const int k = next;
            next = (next + 1) % SLOTS;
            if (busy[k]) { e = cudaEventSynchronize(ev[k]); if (e != cudaSuccess) return e; }
            parallel_copy(slot[k], (const char*)h + off, cnt);
            e = cudaMemcpyAsync((char*)d + off, slot[k], cnt, cudaMemcpyHostToDevice, st);
            if (e != cudaSuccess) return e;
            e = cudaEventRecord(ev[k], st);
            if (e != cudaSuccess) return e;
            busy[k] = true;
        }
        return cudaSuccess;
    }
};

static const char* kGroupNames[G_EVENTS] = {"basic", "sorted", "spectral", "la", "entropy", "seq", "peaks", "assemble"};

struct tsfx_ctx {
    int device = 0;
    cudaStream_t stream = nullptr;        // where calls are enqueued (tsfx_ctx_set_stream)
    cudaStream_t home_stream = nullptr;   // the stream of tsfx_ctx_create
    bool own_stream = false;              // home_stream was created by the library
    cudaEvent_t ev_rebind = nullptr;
    int sm_count = 132;                   // replaced by the device's multiProcessorCount in tsfx_create
    std::string err;
    DevBuf values, begin, len, out, misc, stage;
    double* d_dec = nullptr;
    double2* d_tw = nullptr;
    int tw_n = 0;
    double* d_ricker = nullptr;           // number_cwt_peaks tap table (TSFX_RICKER_W x TSFX_RICKER_K), filled on first use
    cudaEvent_t ev[G_EVENTS][2];
    bool ev_used[G_EVENTS];
    float ms[G_EVENTS];
    int launches = 0;
    const char* kernels[G_COUNT];         // variant each group of the last pass ran (tsfx_last_kernels)
    int n_kernels = 0;
    CsrWorkspace csr;
    StackedWorkspace stacked;    // tsfx_stage_long_stacked: the staged rows the next tsfx_extract_staged consumes
    ImputeWorkspace imp;
    SelectWorkspace sel;
    DevBuf sel_x, sel_y, sel_out;
    bool used_moments = false;   // the last pass ran k_moments in place of k_basic (reported as "moments")
    DevBuf kvals, kvals_sorted;  // value columns of kinds 1 .. K-1 of a wide frame (input order / CSR order)
    DevBuf times, times_sorted;  // tsfx_set_row_times: row timestamps of the next extract call (linear_trend_timewise)
    const int64_t* times_ptr = nullptr;
    int64_t times_rows = -1;
    int max_len_hint = 0;        // tsfx_set_max_len_hint: longest series of the coming device-pointer CSR calls
    int out_ld = 0;              // tsfx_set_out_ld: row stride of `out` of the coming device-pointer calls (0: n_cols)
    // TSFX_FLAG_DEFER_CHECK: the largest shape tsfx_prepare made ready, the caller's status words (tsfx_set_status) and
    // the check's buffers: first series per reason, then per series its private view and its reject reason
    int64_t prep_series = 0;
    int prep_len = 0;
    int64_t* status = nullptr;
    DevBuf defer;
    // tsfx_prepare_long: the prepared long shape, its plans, its slot and check buffers and its per-kind staging blocks
    int long_kinds = 0;
    int64_t long_rows = 0, long_ids = 0;
    int long_len = 0;
    const tsfx_plan* long_plans[TSFX_MAX_KINDS];
    DevBuf long_slots, long_out;
    HostPool pool;
    Stager stager;
    // multi-GPU result placement (tsfx_set_peer_outputs): peers' mapped result matrices
    std::vector<uint64_t> peer_out;
    int peer_self = -1, peer_mode = 0;
    uint64_t peer_mc = 0;
    cudaStream_t s_peer = nullptr;
    cudaEvent_t ev_peer = nullptr;
    cudaStream_t s_in = nullptr, s_out = nullptr;   // copy streams of the pipelined host path
    cudaStream_t s_side[3] = {nullptr, nullptr, nullptr};   // optional side streams so kernel groups can overlap
    cudaEvent_t ev_fork = nullptr, ev_join[3] = {nullptr, nullptr, nullptr};
    cudaEvent_t ev_in[2] = {nullptr, nullptr}, ev_done[2] = {nullptr, nullptr};
};

struct tsfx_plan {
    tsfx_ctx* ctx = nullptr;
    std::vector<Desc> host[G_COUNT];
    Desc* dev[G_COUNT] = {nullptr};
    int32_t* d_final_col = nullptr;   // final column of every staged column, groups concatenated
    double2* d_cq = nullptr;          // (ql, qh) of the distinct change_quantiles corridors (SortedArgs::cq)
    bool sorted_cq_own = false;       // SORTED runs the instantiation with cq_own_passes (launch_sorted)
    bool basic_vocab = false;         // BASIC runs the instantiation with basic_vocabulary (launch_basic)
    bool la_tstat = false;            // LA runs the instantiations with the t-stat lag search (launch_la)
    bool basic_moments_only = false;  // the BASIC group is reductions only: k_moments replaces k_basic
    int moments_need_high = 0;
    int n_groups_used = 0;
    int cum[G_COUNT + 1] = {0};
    int ncols = 0;
    int need_times = 0;               // linear_trend_timewise columns: the extract call needs tsfx_set_row_times
    // each group's kernel arguments as far as the plan fixes them (run_groups adds the call's series and buffers)
    BasicArgs basic = {};
    SortedArgs sorted = {};
    SpectralArgs spectral = {};
    LaArgs la = {};
    EntropyArgs entropy = {};
    SeqArgs seq = {};
    PeaksArgs peaks = {};
    double* d_tables = nullptr;
    int64_t* d_toff = nullptr;
    int32_t* d_thalf = nullptr;
    int n_tables = 0;
    std::vector<int64_t> toff;
    std::vector<int32_t> thalf;
};

static int fail(tsfx_ctx* c, int code, const std::string& msg) {
    if (c) c->err = msg; else g_create_error = msg;
    return code;
}
#define CK(call)                                                                                  \
    do {                                                                                          \
        cudaError_t e__ = (call);                                                                 \
        if (e__ != cudaSuccess)                                                                   \
            return fail(ctx, TSFX_E_CUDA, std::string(#call) + ": " + cudaGetErrorString(e__));  \
    } while (0)

static int group_of(int calc) {
    switch (calc) {
        case TSFX_SYMMETRY_LOOKING: case TSFX_HAS_DUPLICATE: case TSFX_MEDIAN:
        case TSFX_PERCENTAGE_OF_REOCCURRING_VALUES_TO_ALL_VALUES:
        case TSFX_PERCENTAGE_OF_REOCCURRING_DATAPOINTS_TO_ALL_DATAPOINTS:
        case TSFX_SUM_OF_REOCCURRING_VALUES: case TSFX_SUM_OF_REOCCURRING_DATA_POINTS:
        case TSFX_RATIO_VALUE_NUMBER_TO_TIME_SERIES_LENGTH: case TSFX_QUANTILE:
        case TSFX_MEAN_N_ABSOLUTE_MAX: case TSFX_CHANGE_QUANTILES: case TSFX_FRIEDRICH_COEFFICIENTS:
        case TSFX_MAX_LANGEVIN_FIXED_POINT:
            return G_SORTED;
        case TSFX_FFT_COEFFICIENT: case TSFX_FFT_AGGREGATED: case TSFX_SPKT_WELCH_DENSITY:
        case TSFX_FOURIER_ENTROPY: case TSFX_CWT_COEFFICIENTS:
            return G_SPECTRAL;
        case TSFX_AR_COEFFICIENT: case TSFX_AUGMENTED_DICKEY_FULLER:
            return G_LA;
        case TSFX_SAMPLE_ENTROPY: case TSFX_APPROXIMATE_ENTROPY:
            return G_ENTROPY;
        case TSFX_LEMPEL_ZIV_COMPLEXITY: case TSFX_PERMUTATION_ENTROPY:
            return G_SEQ;
        case TSFX_NUMBER_CWT_PEAKS:
            return G_PEAKS;
        default:
            return G_BASIC;
    }
}

extern "C" int tsfx_version(void) { return TSFX_VERSION; }

extern "C" int tsfx_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
    return n;
}

extern "C" const char* tsfx_last_error(const tsfx_ctx* ctx) { return ctx ? ctx->err.c_str() : g_create_error.c_str(); }

extern "C" int tsfx_ctx_create(int device, void* cuda_stream, tsfx_ctx** out) {
    if (!out) return fail(nullptr, TSFX_E_INVALID, "out is NULL");
    *out = nullptr;
    tsfx_ctx* ctx = nullptr;
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || ndev == 0)
        return fail(nullptr, TSFX_E_CUDA, std::string("no CUDA device: ") + cudaGetErrorString(e));
    if (device < 0 || device >= ndev) return fail(nullptr, TSFX_E_INVALID, "device index out of range");
    ctx = new (std::nothrow) tsfx_ctx();
    if (!ctx) return fail(nullptr, TSFX_E_NOMEM, "out of host memory");
    ctx->device = device;
    for (int g = 0; g < G_EVENTS; ++g) { ctx->ev_used[g] = false; ctx->ms[g] = 0.f; ctx->ev[g][0] = ctx->ev[g][1] = nullptr; }
#define CKC(call)                                                                                     \
    do {                                                                                              \
        cudaError_t e__ = (call);                                                                     \
        if (e__ != cudaSuccess) {                                                                     \
            std::string m = std::string(#call) + ": " + cudaGetErrorString(e__);                     \
            delete ctx;                                                                               \
            return fail(nullptr, TSFX_E_CUDA, m);                                                     \
        }                                                                                             \
    } while (0)
    CKC(cudaSetDevice(device));
    cudaDeviceProp prop;
    CKC(cudaGetDeviceProperties(&prop, device));
    ctx->sm_count = prop.multiProcessorCount;
    if (cuda_stream) { ctx->stream = (cudaStream_t)cuda_stream; ctx->own_stream = false; }
    else { CKC(cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking)); ctx->own_stream = true; }
    ctx->home_stream = ctx->stream;
    CKC(cudaEventCreateWithFlags(&ctx->ev_rebind, cudaEventDisableTiming));
    for (int g = 0; g < G_EVENTS; ++g) { CKC(cudaEventCreate(&ctx->ev[g][0])); CKC(cudaEventCreate(&ctx->ev[g][1])); }
    CKC(cudaStreamCreateWithFlags(&ctx->s_in, cudaStreamNonBlocking));
    CKC(cudaStreamCreateWithFlags(&ctx->s_out, cudaStreamNonBlocking));
    CKC(cudaEventCreateWithFlags(&ctx->ev_fork, cudaEventDisableTiming));
    CKC(cudaStreamCreateWithFlags(&ctx->s_peer, cudaStreamNonBlocking));
    CKC(cudaEventCreateWithFlags(&ctx->ev_peer, cudaEventDisableTiming));
    for (int i = 0; i < 3; ++i) { CKC(cudaStreamCreateWithFlags(&ctx->s_side[i], cudaStreamNonBlocking)); CKC(cudaEventCreateWithFlags(&ctx->ev_join[i], cudaEventDisableTiming)); }
    for (int i = 0; i < 2; ++i) { CKC(cudaEventCreateWithFlags(&ctx->ev_in[i], cudaEventDisableTiming)); CKC(cudaEventCreateWithFlags(&ctx->ev_done[i], cudaEventDisableTiming)); }
    // decimal threshold table d * 10^k (correctly rounded literals via strtod)
    {
        std::vector<double> dec((TSFX_DEC_MAX - TSFX_DEC_MIN + 1) * 9);
        for (int k = TSFX_DEC_MIN; k <= TSFX_DEC_MAX; ++k)
            for (int d = 1; d <= 9; ++d) {
                char buf[32];
                snprintf(buf, sizeof buf, "%de%d", d, k);
                dec[(k - TSFX_DEC_MIN) * 9 + (d - 1)] = strtod(buf, nullptr);
            }
        CKC(cudaMalloc(&ctx->d_dec, dec.size() * sizeof(double)));
        CKC(cudaMemcpy(ctx->d_dec, dec.data(), dec.size() * sizeof(double), cudaMemcpyHostToDevice));
    }
#undef CKC
    *out = ctx;
    return TSFX_OK;
}

extern "C" void tsfx_ctx_destroy(tsfx_ctx* ctx) {
    if (!ctx) return;
    cudaSetDevice(ctx->device);
    cudaStreamSynchronize(ctx->stream);
    cudaStreamSynchronize(ctx->home_stream);
    ctx->values.release(); ctx->begin.release(); ctx->len.release(); ctx->out.release(); ctx->misc.release(); ctx->stage.release();
    ctx->times.release(); ctx->times_sorted.release(); ctx->kvals.release(); ctx->kvals_sorted.release();
    ctx->defer.release();
    ctx->long_slots.release(); ctx->long_out.release();
    ctx->csr.release();
    ctx->stacked.release();
    ctx->imp.release();
    ctx->sel.release();
    ctx->sel_x.release(); ctx->sel_y.release(); ctx->sel_out.release();
    ctx->stager.release();
    ctx->pool.release_all();
    if (ctx->s_peer) cudaStreamDestroy(ctx->s_peer);
    if (ctx->ev_peer) cudaEventDestroy(ctx->ev_peer);
    if (ctx->d_dec) cudaFree(ctx->d_dec);
    if (ctx->d_tw) cudaFree(ctx->d_tw);
    if (ctx->d_ricker) cudaFree(ctx->d_ricker);
    for (int g = 0; g < G_EVENTS; ++g) { if (ctx->ev[g][0]) cudaEventDestroy(ctx->ev[g][0]); if (ctx->ev[g][1]) cudaEventDestroy(ctx->ev[g][1]); }
    for (int i = 0; i < 3; ++i) { if (ctx->s_side[i]) cudaStreamDestroy(ctx->s_side[i]); if (ctx->ev_join[i]) cudaEventDestroy(ctx->ev_join[i]); }
    if (ctx->ev_fork) cudaEventDestroy(ctx->ev_fork);
    if (ctx->s_in) cudaStreamDestroy(ctx->s_in);
    if (ctx->s_out) cudaStreamDestroy(ctx->s_out);
    for (int i = 0; i < 2; ++i) { if (ctx->ev_in[i]) cudaEventDestroy(ctx->ev_in[i]); if (ctx->ev_done[i]) cudaEventDestroy(ctx->ev_done[i]); }
    if (ctx->ev_rebind) cudaEventDestroy(ctx->ev_rebind);
    if (ctx->own_stream && ctx->home_stream) cudaStreamDestroy(ctx->home_stream);
    delete ctx;
}

// a stream that is capturing a CUDA graph (or whose capture has been invalidated)
static bool capturing(cudaStream_t s) {
    cudaStreamCaptureStatus st = cudaStreamCaptureStatusNone;
    if (cudaStreamIsCapturing(s, &st) != cudaSuccess) { cudaGetLastError(); return true; }
    return st != cudaStreamCaptureStatusNone;
}

extern "C" int tsfx_ctx_set_stream(tsfx_ctx* ctx, void* cuda_stream) {
    if (!ctx) return TSFX_E_INVALID;
    cudaStream_t next = cuda_stream ? (cudaStream_t)cuda_stream : ctx->home_stream;
    if (next == ctx->stream) return TSFX_OK;
    CK(cudaSetDevice(ctx->device));
    // the next calls reuse the scratch (and twiddle / Ricker tables) the work on the old stream may still be using; an
    // event cannot order work across the boundary of a graph capture, so there the caller orders it
    if (!capturing(ctx->stream) && !capturing(next)) {
        CK(cudaEventRecord(ctx->ev_rebind, ctx->stream));
        CK(cudaStreamWaitEvent(next, ctx->ev_rebind, 0));
    }
    ctx->stream = next;
    return TSFX_OK;
}

extern "C" int tsfx_sync(tsfx_ctx* ctx) {
    if (!ctx) return TSFX_E_INVALID;
    CK(cudaSetDevice(ctx->device));
    CK(cudaStreamSynchronize(ctx->stream));
    return TSFX_OK;
}

// ------------------------------------------------------------------------------------------ plan
static int even(int v) { return (v + 1) & ~1; }

// f_agg codes of agg_autocorrelation and change_quantiles: TSFX_AGG_MEAN .. TSFX_AGG_PROD, each also with TSFX_AGG_NANSKIP
// (np.average is TSFX_AGG_MEAN; there is no nanptp or nanaverage in numpy)
static bool numpy_agg_code(int a) {
    const int op = a & ~TSFX_AGG_NANSKIP;
    if (a < 0 || op > TSFX_AGG_PROD) return false;
    return !(a & TSFX_AGG_NANSKIP) || op != TSFX_AGG_PTP;
}

extern "C" int tsfx_plan_create(tsfx_ctx* ctx, const tsfx_feature_desc* descs, int32_t n_descs, int32_t n_cols,
                                const double* tables, const int64_t* table_off, const int32_t* table_half,
                                int32_t n_tables, tsfx_plan** out) {
    if (!ctx) return TSFX_E_INVALID;
    if (!out || (!descs && n_descs > 0) || n_descs < 0 || n_cols < 0)
        return fail(ctx, TSFX_E_INVALID, "tsfx_plan_create: bad arguments");
    *out = nullptr;
    CK(cudaSetDevice(ctx->device));
    tsfx_plan* P = new (std::nothrow) tsfx_plan();
    if (!P) return fail(ctx, TSFX_E_NOMEM, "out of host memory");
    P->ctx = ctx;
    P->ncols = n_cols;
    int lag_needed = 0, pacf_want = -1, basic_bins = 0, fourier_bins = 0, need_fft = 0, need_welch = 0, max_ar_k = 0;
    int max_lz_bins = 0, max_perm_dim = 0, max_cwt_peaks_n = 0, n_lz = 0, friedrich_r = 0;
    int basic_nfin = 0, sorted_nfin = 0, spectral_nfft = 0;     // leading finisher / fft_coefficient descriptors
    for (int i = 0; i < n_descs; ++i) {
        const Desc& d = descs[i];
        if (d.calc < 0 || d.calc >= TSFX_N_CALCS || d.col < 0 || d.col >= n_cols) {
            delete P;
            return fail(ctx, TSFX_E_INVALID, "tsfx_plan_create: descriptor " + std::to_string(i) + " out of range");
        }
        P->host[group_of(d.calc)].push_back(d);
        switch (d.calc) {
            case TSFX_AUTOCORRELATION: lag_needed = std::max(lag_needed, d.i0); break;
            case TSFX_AGG_AUTOCORRELATION:
                if (!numpy_agg_code(d.attr)) { delete P; return fail(ctx, TSFX_E_UNSUPPORTED, "agg_autocorrelation: unknown f_agg code"); }
                lag_needed = std::max(lag_needed, d.i0);
                break;
            case TSFX_CHANGE_QUANTILES:
                if (!numpy_agg_code(d.attr)) { delete P; return fail(ctx, TSFX_E_UNSUPPORTED, "change_quantiles: unknown f_agg code"); }
                break;
            case TSFX_LINEAR_TREND:
                if (d.attr < 0 || d.attr > TSFX_LR_INTERCEPT_STDERR) { delete P; return fail(ctx, TSFX_E_UNSUPPORTED, "linear_trend: unknown attr code"); }
                break;
            case TSFX_AGG_LINEAR_TREND:
                if (d.attr < 0 || d.attr > TSFX_LR_INTERCEPT_STDERR || d.i1 < TSFX_AGG_MEAN || d.i1 > TSFX_AGG_MIN) {
                    delete P;
                    return fail(ctx, TSFX_E_UNSUPPORTED, "agg_linear_trend: unknown attr or f_agg code");
                }
                break;
            case TSFX_AUGMENTED_DICKEY_FULLER:
                if (d.i0 < TSFX_AUTOLAG_AIC || d.i0 > TSFX_AUTOLAG_TSTAT) { delete P; return fail(ctx, TSFX_E_UNSUPPORTED, "augmented_dickey_fuller: unknown autolag code"); }
                break;
            case TSFX_PARTIAL_AUTOCORRELATION:
                lag_needed = std::max(lag_needed, d.i1);
                pacf_want = std::max(pacf_want, d.i1);
                break;
            case TSFX_BINNED_ENTROPY: basic_bins = std::max(basic_bins, d.i0); break;
            case TSFX_FOURIER_ENTROPY: fourier_bins = std::max(fourier_bins, d.i0); need_welch = 1; break;
            case TSFX_SPKT_WELCH_DENSITY: need_welch = 1; break;
            case TSFX_FFT_COEFFICIENT: case TSFX_FFT_AGGREGATED: need_fft = 1; break;
            case TSFX_CWT_COEFFICIENTS:
                if (d.i1 < 0 || d.i1 >= n_tables) { delete P; return fail(ctx, TSFX_E_INVALID, "cwt table index out of range"); }
                break;
            case TSFX_AR_COEFFICIENT:
                if (d.i1 < 1 || d.i1 > 32) { delete P; return fail(ctx, TSFX_E_UNSUPPORTED, "ar_coefficient: k must be in 1..32"); }
                max_ar_k = std::max(max_ar_k, d.i1);
                break;
            case TSFX_LINEAR_TREND_TIMEWISE:
                if (d.attr < 0 || d.attr > TSFX_LR_INTERCEPT_STDERR) { delete P; return fail(ctx, TSFX_E_UNSUPPORTED, "linear_trend_timewise: unknown attr code"); }
                P->need_times = 1;
                break;
            case TSFX_APPROXIMATE_ENTROPY:
                if (d.i0 != 2) { delete P; return fail(ctx, TSFX_E_UNSUPPORTED, "approximate_entropy: only m=2"); }
                break;
            case TSFX_LEMPEL_ZIV_COMPLEXITY:
                // symbols 0 .. bins - 1 are stored in 16 bits, and key (root 0xffff << 16 | symbol 0xffff) is the empty slot
                if (d.i0 < 1 || d.i0 > TSFX_LZ_MAX_BINS) { delete P; return fail(ctx, TSFX_E_UNSUPPORTED, "lempel_ziv_complexity: bins must be in 1..65535"); }
                max_lz_bins = std::max(max_lz_bins, d.i0); n_lz += 1;
                break;
            case TSFX_PERMUTATION_ENTROPY:
                if (d.i1 < 2 || d.i1 > 8 || d.i0 < 1) { delete P; return fail(ctx, TSFX_E_UNSUPPORTED, "permutation_entropy: dimension 2..8, tau >= 1"); }
                max_perm_dim = std::max(max_perm_dim, d.i1);
                break;
            case TSFX_NUMBER_CWT_PEAKS:
                if (d.i0 < 1 || d.i0 > 16) { delete P; return fail(ctx, TSFX_E_UNSUPPORTED, "number_cwt_peaks: n must be in 1..16"); }
                max_cwt_peaks_n = std::max(max_cwt_peaks_n, d.i0);
                break;
            case TSFX_FRIEDRICH_COEFFICIENTS: case TSFX_MAX_LANGEVIN_FIXED_POINT:
                if (d.i1 != 3 || d.i2 < 1 || d.i2 > 256) { delete P; return fail(ctx, TSFX_E_UNSUPPORTED, "friedrich: only m=3, r in 1..256"); }
                friedrich_r = std::max(friedrich_r, d.i2);
                break;
            default: break;
        }
    }
    if (lag_needed > 4096) { delete P; return fail(ctx, TSFX_E_UNSUPPORTED, "lag > 4096"); }
    // k_basic keeps the whole descriptor table in shared memory, wherever the per-warp working sets live
    if (P->host[G_BASIC].size() > TSFX_BASIC_MAX_COLS &&
        !std::all_of(P->host[G_BASIC].begin(), P->host[G_BASIC].end(), [](const Desc& d) { return moments_only_calc(d.calc); })) {
        delete P;
        return fail(ctx, TSFX_E_UNSUPPORTED, "more than " + std::to_string(TSFX_BASIC_MAX_COLS) + " columns of the BASIC kernel group in one plan");
    }
    std::vector<int32_t> final_col;
    for (int g = 0; g < G_COUNT; ++g) {
        std::stable_sort(P->host[g].begin(), P->host[g].end(), [g](const Desc& a, const Desc& b) {
            if (g == G_BASIC) {               // O(1) finishers first (evaluated lane-parallel)
                const bool fa = basic_finisher_calc(a.calc), fb = basic_finisher_calc(b.calc);
                if (fa != fb) return fa;
            }
            if (g == G_SORTED) {
                const bool fa = sorted_finisher_calc(a.calc), fb = sorted_finisher_calc(b.calc);
                if (fa != fb) return fa;
            }
            if (g == G_SPECTRAL) {            // fft_coefficient first, grouped by attribute
                const bool fa = a.calc == TSFX_FFT_COEFFICIENT, fb = b.calc == TSFX_FFT_COEFFICIENT;
                if (fa != fb) return fa;
                if (fa && a.attr != b.attr) return a.attr < b.attr;
            }
            if (a.calc != b.calc) return a.calc < b.calc;
            if (a.i1 != b.i1) return a.i1 < b.i1;
            if (a.i2 != b.i2) return a.i2 < b.i2;
            if (a.p0 != b.p0) return a.p0 < b.p0;
            if (a.p1 != b.p1) return a.p1 < b.p1;
            if (a.i0 != b.i0) return a.i0 < b.i0;
            return a.col < b.col;
        });
        if (g == G_BASIC)
            for (const Desc& d : P->host[g]) basic_nfin += basic_finisher_calc(d.calc) ? 1 : 0;
        if (g == G_SORTED)
            for (const Desc& d : P->host[g]) sorted_nfin += sorted_finisher_calc(d.calc) ? 1 : 0;
        if (g == G_SPECTRAL)
            for (const Desc& d : P->host[g]) spectral_nfft += (d.calc == TSFX_FFT_COEFFICIENT) ? 1 : 0;
        P->cum[g + 1] = P->cum[g] + (int)P->host[g].size();
        for (size_t j = 0; j < P->host[g].size(); ++j) {      // col becomes the index inside the group's staging row
            final_col.push_back(P->host[g][j].col);
            P->host[g][j].col = (int32_t)j;
        }
        if (!P->host[g].empty()) {
            size_t bytes = P->host[g].size() * sizeof(Desc);
            cudaError_t e = cudaMalloc(&P->dev[g], bytes);
            if (e == cudaSuccess) e = cudaMemcpy(P->dev[g], P->host[g].data(), bytes, cudaMemcpyHostToDevice);
            if (e != cudaSuccess) { tsfx_plan_destroy(P); return fail(ctx, TSFX_E_CUDA, cudaGetErrorString(e)); }
        }
    }
    P->basic_moments_only = !P->host[G_BASIC].empty();
    for (const Desc& d : P->host[G_BASIC]) {
        if (!moments_only_calc(d.calc)) P->basic_moments_only = false;
        if (d.calc == TSFX_SKEWNESS || d.calc == TSFX_KURTOSIS) P->moments_need_high = 1;
    }
    for (int g = 0; g < G_COUNT; ++g) P->n_groups_used += P->host[g].empty() ? 0 : 1;
    if (!final_col.empty()) {
        cudaError_t e = cudaMalloc(&P->d_final_col, final_col.size() * sizeof(int32_t));
        if (e == cudaSuccess) e = cudaMemcpy(P->d_final_col, final_col.data(), final_col.size() * sizeof(int32_t), cudaMemcpyHostToDevice);
        if (e != cudaSuccess) { tsfx_plan_destroy(P); return fail(ctx, TSFX_E_CUDA, cudaGetErrorString(e)); }
    }
    if (n_tables > 0) {
        if (!tables || !table_off || !table_half) { tsfx_plan_destroy(P); return fail(ctx, TSFX_E_INVALID, "cwt tables missing"); }
        P->n_tables = n_tables;
        P->toff.assign(table_off, table_off + n_tables + 1);
        P->thalf.assign(table_half, table_half + n_tables);
        size_t tb = (size_t)table_off[n_tables] * sizeof(double);
        cudaError_t e = cudaMalloc(&P->d_tables, std::max<size_t>(tb, 8));
        if (e == cudaSuccess) e = cudaMemcpy(P->d_tables, tables, tb, cudaMemcpyHostToDevice);
        if (e == cudaSuccess) e = cudaMalloc(&P->d_toff, (n_tables + 1) * sizeof(int64_t));
        if (e == cudaSuccess) e = cudaMemcpy(P->d_toff, table_off, (n_tables + 1) * sizeof(int64_t), cudaMemcpyHostToDevice);
        if (e == cudaSuccess) e = cudaMalloc(&P->d_thalf, n_tables * sizeof(int32_t));
        if (e == cudaSuccess) e = cudaMemcpy(P->d_thalf, table_half, n_tables * sizeof(int32_t), cudaMemcpyHostToDevice);
        if (e != cudaSuccess) { tsfx_plan_destroy(P); return fail(ctx, TSFX_E_CUDA, cudaGetErrorString(e)); }
    }
    auto group = [&](GroupArgs& A, int g) { A.descs = P->dev[g]; A.nd = A.ncols = (int)P->host[g].size(); };
    BasicArgs& B = P->basic;
    group(B, G_BASIC);
    B.lag_needed = lag_needed;
    B.nfin = basic_nfin;
    B.pacf_off = lag_needed + 1;
    B.nlag = even(lag_needed + 1 + (pacf_want >= 0 ? 4 * (pacf_want + 1) : 0));
    B.nscr = even(std::max(64, (basic_bins + 1) / 2));      // launch_basic raises it to the series length
    for (int q = 0, prev = -1; q < (int)P->host[G_BASIC].size(); ++q) {       // distinct agg_linear_trend keys
        const Desc& d = P->host[G_BASIC][q];
        const int key = (d.i0 << 4) | d.i1;
        if (d.calc == TSFX_AGG_LINEAR_TREND && key != prev) { ++B.nalt; prev = key; }
        if (((d.calc == TSFX_LINEAR_TREND || d.calc == TSFX_LINEAR_TREND_TIMEWISE || d.calc == TSFX_AGG_LINEAR_TREND) &&
             d.attr == TSFX_LR_INTERCEPT_STDERR) || (d.calc == TSFX_AGG_AUTOCORRELATION && d.attr > TSFX_AGG_STD))
            P->basic_vocab = true;
    }
    B.dec = ctx->d_dec;
    B.lt_pcol = -1;
    for (int q = 0; q < (int)P->host[G_BASIC].size(); ++q)
        if (P->host[G_BASIC][q].calc == TSFX_LINEAR_TREND && P->host[G_BASIC][q].attr == TSFX_LR_PVALUE) B.lt_pcol = q;
    SortedArgs& S = P->sorted;
    group(S, G_SORTED);
    S.nscr = even(4 * (friedrich_r + 2) + 16);
    S.nfin = sorted_nfin;
    double pl = -1.0, ph = -1.0;                                 // distinct change_quantiles corridors
    std::vector<double2> cq;
    for (const Desc& d : P->host[G_SORTED])
        if (d.calc == TSFX_CHANGE_QUANTILES && !(d.p0 == pl && d.p1 == ph)) { cq.push_back(make_double2(d.p0, d.p1)); pl = d.p0; ph = d.p1; }
    S.ncq = (int)cq.size();
    for (const Desc& d : P->host[G_SORTED])
        if (d.calc == TSFX_CHANGE_QUANTILES && d.attr != TSFX_AGG_MEAN && d.attr != TSFX_AGG_VAR && d.attr != TSFX_AGG_STD)
            P->sorted_cq_own = true;
    if (!cq.empty()) {
        cudaError_t e = cudaMalloc(&P->d_cq, cq.size() * sizeof(double2));
        if (e == cudaSuccess) e = cudaMemcpy(P->d_cq, cq.data(), cq.size() * sizeof(double2), cudaMemcpyHostToDevice);
        if (e != cudaSuccess) { tsfx_plan_destroy(P); return fail(ctx, TSFX_E_CUDA, cudaGetErrorString(e)); }
    }
    S.cq = P->d_cq;
    SpectralArgs& F = P->spectral;
    group(F, G_SPECTRAL);
    F.tables = P->d_tables; F.table_off = P->d_toff; F.table_half = P->d_thalf;
    F.need_fft = need_fft; F.need_welch = need_welch;
    F.max_hist = fourier_bins;
    F.nfft = spectral_nfft;
    group(P->la, G_LA);
    P->la.max_ar_k = max_ar_k;
    for (const Desc& d : P->host[G_LA])
        if (d.calc == TSFX_AUGMENTED_DICKEY_FULLER && d.i0 == TSFX_AUTOLAG_TSTAT) P->la_tstat = true;
    group(P->entropy, G_ENTROPY);
    SeqArgs& Q = P->seq;
    group(Q, G_SEQ);
    Q.need_lz = max_lz_bins > 0; Q.need_perm = max_perm_dim > 0;
    Q.n_lz = n_lz; Q.max_lz_bins = max_lz_bins;
    group(P->peaks, G_PEAKS);
    P->peaks.cwt_n = max_cwt_peaks_n;
    *out = P;
    return TSFX_OK;
}

extern "C" void tsfx_plan_destroy(tsfx_plan* P) {
    if (!P) return;
    if (P->ctx) cudaSetDevice(P->ctx->device);
    for (int g = 0; g < G_COUNT; ++g) if (P->dev[g]) cudaFree(P->dev[g]);
    if (P->d_final_col) cudaFree(P->d_final_col);
    if (P->d_cq) cudaFree(P->d_cq);
    if (P->d_tables) cudaFree(P->d_tables);
    if (P->d_toff) cudaFree(P->d_toff);
    if (P->d_thalf) cudaFree(P->d_thalf);
    delete P;
}

// ------------------------------------------------------------------------------------------ launch all groups

static int ensure_twiddle(tsfx_ctx* ctx, int n_pow2) {
    if (n_pow2 <= ctx->tw_n) return TSFX_OK;
    if (ctx->d_tw) { cudaStreamSynchronize(ctx->stream); cudaFree(ctx->d_tw); ctx->d_tw = nullptr; ctx->tw_n = 0; }
    CK(cudaMalloc(&ctx->d_tw, (size_t)(n_pow2 / 2 + 1) * sizeof(double2)));
    CK(launch_fill_twiddle(ctx->d_tw, n_pow2, ctx->stream));
    ctx->tw_n = n_pow2;
    return TSFX_OK;
}

static int ensure_ricker(tsfx_ctx* ctx) {
    if (ctx->d_ricker) return TSFX_OK;
    CK(cudaMalloc(&ctx->d_ricker, (size_t)TSFX_RICKER_W * TSFX_RICKER_K * sizeof(double)));
    CK(launch_fill_ricker(ctx->d_ricker, ctx->stream));
    return TSFX_OK;
}

// row timestamps handed over with tsfx_set_row_times for a call whose `values` array has `rows` rows (consumed)
static int take_times(tsfx_ctx* ctx, const tsfx_plan* P, int64_t rows, const int64_t** out) {
    *out = nullptr;
    const bool have = ctx->times_rows >= 0;
    const int64_t got = ctx->times_rows;
    const int64_t* p = ctx->times_ptr;
    ctx->times_rows = -1;
    ctx->times_ptr = nullptr;
    if (!P->need_times) return TSFX_OK;
    if (!have) return fail(ctx, TSFX_E_INVALID, "linear_trend_timewise needs the row timestamps (tsfx_set_row_times)");
    if (got != rows) return fail(ctx, TSFX_E_INVALID, "tsfx_set_row_times: " + std::to_string(got) + " timestamps for " + std::to_string(rows) + " rows");
    *out = p;
    return TSFX_OK;
}

extern "C" int tsfx_set_row_times(tsfx_ctx* ctx, const int64_t* row_time_ns, int64_t n_rows, uint32_t flags) {
    if (!ctx) return TSFX_E_INVALID;
    if (n_rows < 0 || (n_rows > 0 && !row_time_ns)) return fail(ctx, TSFX_E_INVALID, "tsfx_set_row_times: bad arguments");
    CK(cudaSetDevice(ctx->device));
    if (flags & TSFX_FLAG_DEVICE_PTRS) ctx->times_ptr = row_time_ns;
    else {
        CK(ctx->times.reserve(std::max<size_t>((size_t)n_rows * 8, 8)));
        CK(ctx->stager.h2d(ctx->times.p, row_time_ns, (size_t)n_rows * 8, ctx->stream));
        ctx->times_ptr = (const int64_t*)ctx->times.p;
    }
    ctx->times_rows = n_rows;
    return TSFX_OK;
}

// TSFX_E_TOO_LONG when a series of max_len samples exceeds the limit of one of the plan's kernel groups
static int check_lengths(tsfx_ctx* ctx, const tsfx_plan* P, int max_len) {
    for (int g = 0; g < G_COUNT; ++g)
        if (!P->host[g].empty() && max_len > group_max_len(g))
            return fail(ctx, TSFX_E_TOO_LONG, std::string("series length ") + std::to_string(max_len) +
                                                  " exceeds the shared-memory staging of kernel group " + kGroupNames[g] +
                                                  " (limit " + std::to_string(group_max_len(g)) + " samples)");
    return TSFX_OK;
}

// the working memory and tables the groups of P need for n_series series of at most max_len samples (tsfx_prepare
// makes them ready ahead of time)
static int reserve_groups(tsfx_ctx* ctx, const tsfx_plan* P, int64_t n_series, int max_len) {
    CK(ctx->stage.reserve((size_t)n_series * P->cum[G_COUNT] * sizeof(double)));
    CK(ctx->misc.reserve(max_len > 1024 ? ((size_t)1 << 30) : ((size_t)256 << 20)));      // global working regions for series too long for shared memory
    if (!P->host[G_SPECTRAL].empty()) {      // FFT twiddle table (filled once, on the main stream, before any fork)
        int p2 = 1;
        if (max_len > TSFX_SHORT_L_MAX) {
            while (p2 < 2 * max_len - 1) p2 <<= 1;      // Bluestein convolution length of the longest series
        } else {
            while (p2 < max_len) p2 <<= 1;
            if (p2 > max_len) p2 >>= 1;        // largest power of two <= max_len
        }
        p2 = std::max(p2, 256);
        int rc = ensure_twiddle(ctx, p2);
        if (rc) return rc;
    }
    if (!P->host[G_PEAKS].empty()) {         // Ricker taps (filled once, on the main stream, before any fork)
        int rc = ensure_ricker(ctx);
        if (rc) return rc;
    }
    return TSFX_OK;
}

static int run_groups(tsfx_ctx* ctx, const tsfx_plan* P, const SeriesRef& R, int max_len, double* d_out, uint32_t flags, int ld = 0) {
    if (ld <= 0) ld = P->ncols;          // row stride of the caller's matrix
    const bool timing = (flags & TSFX_FLAG_TIMING) != 0;
    for (int g = 0; g < G_EVENTS; ++g) ctx->ev_used[g] = false;
    ctx->launches = 0;
    ctx->n_kernels = 0;
    if (R.n_series == 0) return TSFX_OK;
    const int staged = P->cum[G_COUNT];
    if (staged == 0) return TSFX_OK;
    if (int rc = check_lengths(ctx, P, max_len)) return rc;      // every group's length limit before any group runs
    if (int rc = reserve_groups(ctx, P, R.n_series, max_len)) return rc;
    // kernel groups are independent (own staging matrix): optionally spread them over side streams
    const int nstreams = timing ? 1 : env_streams();
    if (nstreams > 1) {
        CK(cudaEventRecord(ctx->ev_fork, ctx->stream));
        for (int i = 0; i < nstreams - 1; ++i) CK(cudaStreamWaitEvent(ctx->s_side[i], ctx->ev_fork, 0));
    }
    int launched = 0;
    bool direct = false;          // the only group wrote the final matrix itself
    ctx->used_moments = false;
    if (max_len < 1) return fail(ctx, TSFX_E_INVALID, "series of length < 1");
    auto too_long = [&](const char* g) {
        return fail(ctx, TSFX_E_TOO_LONG, std::string("series length ") + std::to_string(max_len) +
                                              " exceeds the shared-memory staging of kernel group " + g);
    };
    for (int g = 0; g < G_COUNT; ++g) {
        if (P->host[g].empty()) continue;
        if (timing) { CK(cudaEventRecord(ctx->ev[g][0], ctx->stream)); }
        cudaError_t e = cudaSuccess;
        const char* variant = nullptr;
        double* const stage_g = (double*)ctx->stage.p + (size_t)R.n_series * P->cum[g];      // this group's staging matrix
        const int sidx = launched++ % nstreams;
        cudaStream_t gs = (sidx == 0) ? ctx->stream : ctx->s_side[sidx - 1];
        const int g_ncols = (int)P->host[g].size();
        // global working region: the whole buffer when the groups run back to back, a private slice per group when
        // they overlap on side streams (concurrent groups must not share working sets)
        const size_t slice = (nstreams > 1) ? (ctx->misc.cap / G_COUNT) & ~(size_t)255 : ctx->misc.cap;
        unsigned char* const gs_base = (unsigned char*)ctx->misc.p + (nstreams > 1 ? (size_t)g * slice : 0);
        // the plan's arguments of the group with this call's series, working region and staging matrix
        auto call = [&](auto A) {
            A.R = R; A.gscratch = gs_base; A.gscratch_bytes = slice; A.out = stage_g;
            return A;
        };
        switch (g) {
            case G_BASIC: {
                if (P->basic_moments_only) {
                    // reductions only: stream the series from HBM; with no other group in the plan the rows go
                    // straight into the caller's matrix (no staging, no assemble pass)
                    MomentsArgs M;
                    M.R = R; M.descs = P->dev[g]; M.nd = g_ncols; M.need_high = P->moments_need_high;
                    direct = (P->n_groups_used == 1) && ctx->peer_out.empty() && (P->ncols == g_ncols);
                    M.out = direct ? d_out : stage_g;
                    M.ncols = direct ? ld : g_ncols;
                    M.colmap = direct ? P->d_final_col + P->cum[g] : nullptr;
                    e = launch_moments(M, gs, ctx->sm_count, &variant);
                    ctx->used_moments = true;
                    break;
                }
                e = launch_basic(call(P->basic), P->basic_vocab, max_len, gs, ctx->sm_count, &variant);
                break;
            }
            case G_SORTED: e = launch_sorted(call(P->sorted), P->sorted_cq_own, max_len, gs, ctx->sm_count, &variant); break;
            case G_SPECTRAL: {
                SpectralArgs A = call(P->spectral);
                A.twiddle = ctx->d_tw; A.tw_n = ctx->tw_n;
                e = launch_spectral(A, max_len, gs, ctx->sm_count, &variant);
                break;
            }
            case G_LA: e = launch_la(call(P->la), P->la_tstat, max_len, gs, ctx->sm_count, &variant); break;
            case G_ENTROPY: e = launch_entropy(call(P->entropy), max_len, gs, ctx->sm_count, &variant); break;
            case G_SEQ: e = launch_seq(call(P->seq), max_len, gs, ctx->sm_count, &variant); break;
            case G_PEAKS: {
                PeaksArgs A = call(P->peaks);
                A.ricker = ctx->d_ricker;
                e = launch_peaks(A, max_len, gs, ctx->sm_count, &variant);
                break;
            }
        }
        if (e == cudaErrorInvalidConfiguration) return too_long(kGroupNames[g]);
        if (e != cudaSuccess)      // the variant names the geometry of a launch that failed, or one not compiled
            return fail(ctx, TSFX_E_CUDA, std::string("launch ") + kGroupNames[g] + (variant ? std::string(" (") + variant + ")" : "") +
                                              ": " + cudaGetErrorString(e));
        ctx->launches += 1;
        ctx->kernels[ctx->n_kernels++] = variant;
        if (timing) { CK(cudaEventRecord(ctx->ev[g][1], ctx->stream)); ctx->ev_used[g] = true; }
    }
    if (nstreams > 1)
        for (int i = 0; i < nstreams - 1; ++i) {
            CK(cudaEventRecord(ctx->ev_join[i], ctx->s_side[i]));
            CK(cudaStreamWaitEvent(ctx->stream, ctx->ev_join[i], 0));
        }
    if (!direct) {   // scatter the staging matrices into the caller's [n_series x ncols] matrix
        if (timing) { CK(cudaEventRecord(ctx->ev[G_COUNT][0], ctx->stream)); }
        AssembleArgs A;
        A.stage = (const double*)ctx->stage.p; A.out = d_out; A.n_series = R.n_series; A.ncols = P->ncols; A.ld = ld;
        if (ld != P->ncols && !ctx->peer_out.empty()) return fail(ctx, TSFX_E_UNSUPPORTED, "peer placement of a strided matrix");
        A.n_groups = G_COUNT;
        for (int g = 0; g <= G_COUNT; ++g) A.cum[g] = P->cum[g];
        A.final_col = P->d_final_col;
        A.n_extra = 0;
        A.out_mc = nullptr;
        // multi-GPU placement: where does this row block live inside the peers' copies of the result matrix?
        int64_t peer_off = -1;                 // byte offset of d_out inside this rank's mapped matrix
        if (!ctx->peer_out.empty()) {
            const uint64_t self = ctx->peer_out[ctx->peer_self];
            if ((uint64_t)d_out < self) return fail(ctx, TSFX_E_INVALID, "out is not inside the matrix registered with tsfx_set_peer_outputs");
            peer_off = (int64_t)((uint64_t)d_out - self);
            if (ctx->peer_mode == TSFX_PEER_MULTICAST) A.out_mc = (double*)(ctx->peer_mc + (uint64_t)peer_off);
            else if (ctx->peer_mode == TSFX_PEER_STORE)
                for (size_t p = 0; p < ctx->peer_out.size(); ++p)
                    if ((int)p != ctx->peer_self) A.extra[A.n_extra++] = (double*)(ctx->peer_out[p] + (uint64_t)peer_off);
        }
        cudaError_t e = launch_assemble(A, ctx->stream, ctx->sm_count);
        if (e != cudaSuccess) return fail(ctx, TSFX_E_CUDA, std::string("launch assemble: ") + cudaGetErrorString(e));
        ctx->launches += 1;
        if (timing) { CK(cudaEventRecord(ctx->ev[G_COUNT][1], ctx->stream)); ctx->ev_used[G_COUNT] = true; }
        if (peer_off >= 0 && ctx->peer_mode == TSFX_PEER_COPY) {
            // copy engines push the finished row block to every peer while the next block's kernels run
            const size_t bytes = (size_t)R.n_series * P->ncols * sizeof(double);
            CK(cudaEventRecord(ctx->ev_peer, ctx->stream));
            CK(cudaStreamWaitEvent(ctx->s_peer, ctx->ev_peer, 0));
            const size_t np = ctx->peer_out.size();
            for (size_t k = 1; k < np; ++k) {          // start with the next rank so the ranks do not all hit one peer
                const size_t p = ((size_t)ctx->peer_self + k) % np;
                CK(cudaMemcpyAsync((void*)(ctx->peer_out[p] + (uint64_t)peer_off), d_out, bytes, cudaMemcpyDeviceToDevice, ctx->s_peer));
            }
        }
    }
    return TSFX_OK;
}

static int impute_after_extract(tsfx_ctx* ctx, double* d_out, int64_t rows, int cols);
static int nan_error(tsfx_ctx* ctx);

static int check_args(tsfx_ctx* ctx, const tsfx_plan* plan, const void* values, const void* out, int64_t n_series) {
    if (!ctx) return TSFX_E_INVALID;
    if (!plan || plan->ctx != ctx) return fail(ctx, TSFX_E_INVALID, "plan does not belong to this context");
    if (n_series < 0) return fail(ctx, TSFX_E_INVALID, "n_series < 0");
    if (n_series > 0 && (!values || !out)) return fail(ctx, TSFX_E_INVALID, "NULL values/out");
    return TSFX_OK;
}

// TSFX_FLAG_CHECK_DEVICE_INPUT: one pass over the caller's device input (views when begin != nullptr, else n_values
// values of a dense batch) and one synchronisation, before any kernel group can see the input
static int check_device_input(tsfx_ctx* ctx, const float* values, int64_t n_values, const int64_t* begin, const int32_t* len,
                              int64_t n_series, int* max_len) {
    ctx->launches = 0;
    ctx->n_kernels = 0;
    CsrWorkspace& W = ctx->csr;
    CK(W.init_info());
    CK(cudaMemsetAsync(W.d_info, 0, sizeof(CsrInfo), ctx->stream));
    if (begin) csr_check_views(W, values, n_values, begin, len, n_series, ctx->stream);
    else csr_check_nan(W, values, n_values, ctx->stream);
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(W.h_info, W.d_info, sizeof(CsrInfo), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    const CsrInfo& I = *W.h_info;
    if (I.bad_view_rev)
        return fail(ctx, TSFX_E_INVALID, "series " + std::to_string(n_series - (int64_t)I.bad_view_rev) +
                                             " has an invalid (begin, len): len < 1, begin < 0 or begin + len > n_values");
    if (I.has_nan) return nan_error(ctx);
    if (begin) *max_len = I.max_len;
    return TSFX_OK;
}

// TSFX_FLAG_DEFER_CHECK buffers, laid out for ctx->prep_series series
struct DeferBufs {
    unsigned long long* first;   // n_series - s of the first rejected series s per reason (0: none)
    int64_t* vbegin;             // private views (CSR)
    int32_t* vlen;
    uint8_t* reject;             // reject reason per series
};
static size_t defer_bytes(int64_t n_series) { return 64 + (size_t)n_series * 13; }
static DeferBufs defer_bufs(tsfx_ctx* ctx) {
    char* p = (char*)ctx->defer.p;
    const size_t n = (size_t)ctx->prep_series;
    return {(unsigned long long*)p, (int64_t*)(p + 64), (int32_t*)(p + 64 + 8 * n), (uint8_t*)(p + 64 + 12 * n)};
}

// TSFX_FLAG_DEFER_CHECK (tsfx.h "Deferred input check"): the validation pass, the groups on the private views (CSR) or
// on the input as it is (dense), then the NaN rows and the report.  Only enqueues: a prepared shape needs no allocation.
static int extract_deferred(tsfx_ctx* ctx, const tsfx_plan* plan, SeriesRef R, int64_t n_values, int max_len, double* out,
                            uint32_t flags, int ld) {
    if (flags & (TSFX_FLAG_CHECK_DEVICE_INPUT | TSFX_FLAG_IMPUTE))
        return fail(ctx, TSFX_E_INVALID, "TSFX_FLAG_DEFER_CHECK excludes TSFX_FLAG_CHECK_DEVICE_INPUT and TSFX_FLAG_IMPUTE");
    if (!ctx->status) return fail(ctx, TSFX_E_INVALID, "TSFX_FLAG_DEFER_CHECK needs a status buffer (tsfx_set_status)");
    if (max_len < 1) return fail(ctx, TSFX_E_INVALID, "TSFX_FLAG_DEFER_CHECK needs the longest series (tsfx_set_max_len_hint)");
    if (R.n_series > ctx->prep_series || max_len > ctx->prep_len)
        return fail(ctx, TSFX_E_INVALID, "TSFX_FLAG_DEFER_CHECK: " + std::to_string(R.n_series) + " series of up to " +
                                             std::to_string(max_len) + " samples, more than tsfx_prepare made ready");
    if (n_values < 1) return fail(ctx, TSFX_E_INVALID, "TSFX_FLAG_DEFER_CHECK: no values");
    const DeferBufs B = defer_bufs(ctx);
    const bool csr = R.begin != nullptr;
    CK(cudaMemsetAsync(B.first, 0, 3 * sizeof(unsigned long long), ctx->stream));
    CK(defer_check(R.values, n_values, R.begin, R.len, R.n_series, max_len, csr ? B.vbegin : nullptr, B.vlen, B.reject,
                   B.first, ctx->stream));
    if (csr) { R.begin = B.vbegin; R.len = B.vlen; }
    if (int rc = run_groups(ctx, plan, R, max_len, out, flags, ld)) return rc;
    CK(defer_finish(out, R.n_series, plan->ncols, ld, B.reject, B.first, ctx->status, ctx->stream));
    ctx->launches += 2;
    return TSFX_OK;
}

extern "C" int tsfx_prepare(tsfx_ctx* ctx, const tsfx_plan* plan, int64_t n_series, int32_t max_len) {
    int rc = check_args(ctx, plan, nullptr, nullptr, 0);
    if (rc) return rc;
    if (n_series < 1 || max_len < 1) return fail(ctx, TSFX_E_INVALID, "tsfx_prepare: n_series and max_len must be >= 1");
    CK(cudaSetDevice(ctx->device));
    if ((rc = check_lengths(ctx, plan, max_len))) return rc;
    if ((rc = reserve_groups(ctx, plan, n_series, max_len))) return rc;
    const int64_t n = std::max(n_series, ctx->prep_series);
    CK(ctx->defer.reserve(defer_bytes(n)));
    ctx->prep_series = n;
    ctx->prep_len = std::max(ctx->prep_len, (int)max_len);
    CK(cudaStreamSynchronize(ctx->stream));     // the tables are filled before a captured call, which cannot wait for them
    return TSFX_OK;
}

extern "C" int tsfx_set_status(tsfx_ctx* ctx, int64_t* status) {
    if (!ctx) return TSFX_E_INVALID;
    ctx->status = status;
    return TSFX_OK;
}

extern "C" int32_t tsfx_plan_max_len(const tsfx_feature_desc* descs, int32_t n_descs) {
    if (n_descs < 0 || (n_descs > 0 && !descs)) return TSFX_E_INVALID;
    int32_t m = 0x7fffffff;
    for (int i = 0; i < n_descs; ++i) {
        if (descs[i].calc < 0 || descs[i].calc >= TSFX_N_CALCS) return TSFX_E_INVALID;
        m = std::min(m, (int32_t)group_max_len(group_of(descs[i].calc)));
    }
    return m;
}

// row stride of a device-pointer call's `out` (tsfx_set_out_ld)
static int device_out_ld(tsfx_ctx* ctx, const tsfx_plan* plan, uint32_t flags, int* ld) {
    *ld = ctx->out_ld > 0 ? ctx->out_ld : plan->ncols;
    if (*ld < plan->ncols)
        return fail(ctx, TSFX_E_INVALID, "tsfx_set_out_ld: row stride " + std::to_string(*ld) + " < " + std::to_string(plan->ncols) + " columns");
    if (*ld != plan->ncols && (flags & TSFX_FLAG_IMPUTE))
        return fail(ctx, TSFX_E_INVALID, "TSFX_FLAG_IMPUTE needs a contiguous result matrix (tsfx_set_out_ld)");
    return TSFX_OK;
}

extern "C" int tsfx_extract_csr(tsfx_ctx* ctx, const tsfx_plan* plan, const float* values, int64_t n_values,
                                const int64_t* begin, const int32_t* len, int64_t n_series, double* out,
                                uint32_t flags) {
    int rc = check_args(ctx, plan, values, out, n_series);
    if (rc) return rc;
    if (n_series == 0) return TSFX_OK;
    if (!begin || !len) return fail(ctx, TSFX_E_INVALID, "NULL begin/len");
    CK(cudaSetDevice(ctx->device));
    SeriesRef R;
    R.dense_len = 0;
    R.n_series = n_series;
    rc = take_times(ctx, plan, n_values, &R.times);
    if (rc) return rc;
    int max_len = 0;
    if (flags & TSFX_FLAG_DEVICE_PTRS) {
        R.values = values; R.begin = begin; R.len = len;
        int ld = 0;
        rc = device_out_ld(ctx, plan, flags, &ld);
        if (rc) return rc;
        if (flags & TSFX_FLAG_DEFER_CHECK) return extract_deferred(ctx, plan, R, n_values, ctx->max_len_hint, out, flags, ld);
        if (flags & TSFX_FLAG_CHECK_DEVICE_INPUT) {
            rc = check_device_input(ctx, values, n_values, begin, len, n_series, &max_len);
            if (rc) return rc;
        } else if (ctx->max_len_hint > 0) max_len = ctx->max_len_hint;       // stays asynchronous
        else {
            int rc2 = csr_max_len(ctx->csr, len, n_series, ctx->stream, &max_len);
            if (rc2) return fail(ctx, TSFX_E_CUDA, "max-length reduction failed");
        }
        rc = run_groups(ctx, plan, R, max_len, out, flags, ld);
        if (!rc && (flags & TSFX_FLAG_IMPUTE)) rc = impute_after_extract(ctx, out, n_series, plan->ncols);
        return rc;
    }
    for (int64_t s = 0; s < n_series; ++s) {
        if (len[s] < 1 || begin[s] < 0 || begin[s] + len[s] > n_values)
            return fail(ctx, TSFX_E_INVALID, "series " + std::to_string(s) + " has an invalid (begin, len)");
        max_len = std::max(max_len, (int)len[s]);
    }
    size_t ob = (size_t)n_series * plan->ncols * sizeof(double);
    CK(ctx->values.reserve((size_t)n_values * sizeof(float) + 16));
    CK(ctx->begin.reserve((size_t)n_series * sizeof(int64_t)));
    CK(ctx->len.reserve((size_t)n_series * sizeof(int32_t)));
    CK(ctx->out.reserve(std::max<size_t>(ob, 8)));
    CK(cudaMemcpyAsync(ctx->values.p, values, (size_t)n_values * sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemcpyAsync(ctx->begin.p, begin, (size_t)n_series * sizeof(int64_t), cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemcpyAsync(ctx->len.p, len, (size_t)n_series * sizeof(int32_t), cudaMemcpyHostToDevice, ctx->stream));
    R.values = (const float*)ctx->values.p; R.begin = (const int64_t*)ctx->begin.p; R.len = (const int32_t*)ctx->len.p;
    const bool check_nan = !(flags & TSFX_FLAG_NO_NAN_CHECK);
    if (check_nan) {
        CK(ctx->csr.init_info());
        CK(cudaMemsetAsync(ctx->csr.d_info, 0, sizeof(CsrInfo), ctx->stream));
        csr_check_nan(ctx->csr, R.values, n_values, ctx->stream);
        CK(cudaMemcpyAsync(ctx->csr.h_info, ctx->csr.d_info, sizeof(CsrInfo), cudaMemcpyDeviceToHost, ctx->stream));
    }
    rc = run_groups(ctx, plan, R, max_len, (double*)ctx->out.p, flags);
    if (rc) return rc;
    if (flags & TSFX_FLAG_IMPUTE) { rc = impute_after_extract(ctx, (double*)ctx->out.p, n_series, plan->ncols); if (rc) return rc; }
    CK(cudaMemcpyAsync(out, ctx->out.p, ob, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    if (check_nan && ctx->csr.h_info->has_nan) return nan_error(ctx);
    return TSFX_OK;
}

extern "C" int tsfx_extract_dense(tsfx_ctx* ctx, const tsfx_plan* plan, const float* values, int64_t n_series,
                                  int32_t len, double* out, uint32_t flags) {
    int rc = check_args(ctx, plan, values, out, n_series);
    if (rc) return rc;
    if (n_series == 0) return TSFX_OK;
    if (len < 1) return fail(ctx, TSFX_E_INVALID, "len < 1");
    CK(cudaSetDevice(ctx->device));
    SeriesRef R;
    R.begin = nullptr; R.len = nullptr; R.dense_len = len; R.n_series = n_series;
    const int64_t* all_times = nullptr;
    rc = take_times(ctx, plan, n_series * (int64_t)len, &all_times);
    if (rc) return rc;
    R.times = all_times;
    if (flags & TSFX_FLAG_DEVICE_PTRS) {
        R.values = values;
        int ld = 0;
        rc = device_out_ld(ctx, plan, flags, &ld);
        if (rc) return rc;
        if (flags & TSFX_FLAG_DEFER_CHECK) return extract_deferred(ctx, plan, R, n_series * (int64_t)len, len, out, flags, ld);
        if (flags & TSFX_FLAG_CHECK_DEVICE_INPUT) {
            int max_len = len;
            rc = check_device_input(ctx, values, n_series * (int64_t)len, nullptr, nullptr, n_series, &max_len);
            if (rc) return rc;
        }
        rc = run_groups(ctx, plan, R, len, out, flags, ld);
        if (!rc && (flags & TSFX_FLAG_IMPUTE)) rc = impute_after_extract(ctx, out, n_series, plan->ncols);
        return rc;
    }
    // host path: pipelined over row blocks -- the H2D copy of block b+1 and the D2H copy of block b-1 run on
    // their own streams while the kernels of block b execute (pinned host buffers make the copies truly async)
    const size_t ncols = (size_t)plan->ncols;
    const size_t vb = (size_t)n_series * len * sizeof(float), ob = (size_t)n_series * ncols * sizeof(double);
    CK(ctx->values.reserve(vb + 16));
    CK(ctx->out.reserve(std::max<size_t>(ob, 8)));
    int64_t block = std::max<int64_t>(16384, (n_series + 15) / 16);
    if (flags & TSFX_FLAG_TIMING) block = n_series;            // per-group events describe one whole pass
    float* dv = (float*)ctx->values.p;
    double* dout = (double*)ctx->out.p;
    const bool check_nan = !(flags & TSFX_FLAG_NO_NAN_CHECK);
    if (check_nan) { CK(ctx->csr.init_info()); CK(cudaMemsetAsync(ctx->csr.d_info, 0, sizeof(CsrInfo), ctx->stream)); }
    int nb = 0;
    for (int64_t lo = 0; lo < n_series; lo += block, ++nb) {
        const int64_t cnt = std::min<int64_t>(block, n_series - lo);
        const int slot = nb & 1;
        CK(ctx->stager.h2d(dv + (size_t)lo * len, values + (size_t)lo * len, (size_t)cnt * len * sizeof(float), ctx->s_in));
        CK(cudaEventRecord(ctx->ev_in[slot], ctx->s_in));
        CK(cudaStreamWaitEvent(ctx->stream, ctx->ev_in[slot], 0));
        if (check_nan) csr_check_nan(ctx->csr, dv + (size_t)lo * len, cnt * len, ctx->stream);
        R.values = dv + (size_t)lo * len;
        R.times = all_times ? all_times + (size_t)lo * len : nullptr;
        R.n_series = cnt;
        rc = run_groups(ctx, plan, R, len, dout + (size_t)lo * ncols, flags);
        if (rc) return rc;
        if (flags & TSFX_FLAG_IMPUTE) continue;         // column statistics need every row: one copy at the end
        CK(cudaEventRecord(ctx->ev_done[slot], ctx->stream));
        CK(cudaStreamWaitEvent(ctx->s_out, ctx->ev_done[slot], 0));
        CK(cudaMemcpyAsync(out + (size_t)lo * ncols, dout + (size_t)lo * ncols, (size_t)cnt * ncols * sizeof(double),
                           cudaMemcpyDeviceToHost, ctx->s_out));
    }
    if (flags & TSFX_FLAG_IMPUTE) {
        rc = impute_after_extract(ctx, dout, n_series, plan->ncols);
        if (rc) return rc;
        CK(cudaMemcpyAsync(out, dout, ob, cudaMemcpyDeviceToHost, ctx->stream));
    }
    if (check_nan) CK(cudaMemcpyAsync(ctx->csr.h_info, ctx->csr.d_info, sizeof(CsrInfo), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->s_out));
    CK(cudaStreamSynchronize(ctx->stream));
    if (check_nan && ctx->csr.h_info->has_nan) return nan_error(ctx);
    return TSFX_OK;
}

// impute the device matrix of the extract call that just ran (TSFX_FLAG_IMPUTE)
static int impute_after_extract(tsfx_ctx* ctx, double* d_out, int64_t rows, int cols) {
    int n = 0;
    cudaError_t e = impute_device(ctx->imp, d_out, rows, cols, TSFX_IMPUTE_RANGE, false, nullptr, ctx->sm_count, ctx->stream, &n);
    if (e != cudaSuccess) return fail(ctx, TSFX_E_CUDA, std::string("impute: ") + cudaGetErrorString(e));
    ctx->launches += n;
    return TSFX_OK;
}

extern "C" int tsfx_impute(tsfx_ctx* ctx, double* matrix, int64_t n_rows, int32_t n_cols, int32_t mode, double* col_stats,
                           uint32_t flags) {
    if (!ctx) return TSFX_E_INVALID;
    if (n_rows < 0 || n_cols < 0 || mode < TSFX_IMPUTE_RANGE || mode > TSFX_IMPUTE_STATS)
        return fail(ctx, TSFX_E_INVALID, "tsfx_impute: bad arguments");
    if (n_rows == 0 || n_cols == 0) return TSFX_OK;
    if (!matrix) return fail(ctx, TSFX_E_INVALID, "tsfx_impute: NULL matrix");
    if ((mode == TSFX_IMPUTE_GIVEN || mode == TSFX_IMPUTE_STATS) && !col_stats)
        return fail(ctx, TSFX_E_INVALID, "tsfx_impute: col_stats is required for this mode");
    if (mode == TSFX_IMPUTE_GIVEN)
        for (int64_t i = 0; i < (int64_t)3 * n_cols; ++i)
            if (!std::isfinite(col_stats[i]))       // dataframe_functions.py:147-156 raises ValueError
                return fail(ctx, TSFX_E_INVALID, "tsfx_impute: non-finite replacement value");
    CK(cudaSetDevice(ctx->device));
    const size_t bytes = (size_t)n_rows * n_cols * sizeof(double);
    double* d_m = matrix;
    const bool host = !(flags & TSFX_FLAG_DEVICE_PTRS);
    if (host) {
        CK(ctx->out.reserve(bytes));
        d_m = (double*)ctx->out.p;
        CK(cudaMemcpyAsync(d_m, matrix, bytes, cudaMemcpyHostToDevice, ctx->stream));
    }
    int n = 0;
    cudaError_t e = impute_device(ctx->imp, d_m, n_rows, n_cols, mode, (flags & TSFX_FLAG_ALL_MEDIANS) != 0 || mode == TSFX_IMPUTE_STATS,
                                  col_stats, ctx->sm_count, ctx->stream, &n);
    if (e != cudaSuccess) return fail(ctx, TSFX_E_CUDA, std::string("impute: ") + cudaGetErrorString(e));
    ctx->launches = n;
    if (host) {
        if (mode != TSFX_IMPUTE_STATS) CK(cudaMemcpyAsync(matrix, d_m, bytes, cudaMemcpyDeviceToHost, ctx->stream));
        CK(cudaStreamSynchronize(ctx->stream));
    }
    return TSFX_OK;
}

extern "C" int tsfx_get_timings(tsfx_ctx* ctx, float* ms_out, const char** names_out, int32_t cap) {
    if (!ctx) return TSFX_E_INVALID;
    CK(cudaSetDevice(ctx->device));
    CK(cudaStreamSynchronize(ctx->stream));
    int k = 0;
    for (int g = 0; g < G_EVENTS && k < cap; ++g) {
        if (!ctx->ev_used[g]) continue;
        float ms = 0.f;
        CK(cudaEventElapsedTime(&ms, ctx->ev[g][0], ctx->ev[g][1]));
        if (ms_out) ms_out[k] = ms;
        if (names_out) names_out[k] = (g == G_BASIC && ctx->used_moments) ? "moments" : kGroupNames[g];
        ++k;
    }
    return k;
}

extern "C" int tsfx_last_launch_count(const tsfx_ctx* ctx) { return ctx ? ctx->launches : 0; }

extern "C" int tsfx_last_kernels(const tsfx_ctx* ctx, const char** names_out, int32_t cap) {
    if (!ctx || cap < 0 || (cap > 0 && !names_out)) return TSFX_E_INVALID;
    const int k = std::min<int>(ctx->n_kernels, cap);
    for (int i = 0; i < k; ++i) names_out[i] = ctx->kernels[i];
    return k;
}

// every name a launcher can report: its fixed-geometry kernels and its declared geometries (tsfx_kernels.h)
static const char* const kKernelVariants[] = {
    "moments/dense", "moments/general",
    TSFX_GEOMS_BASIC(TSFX_GEOM_NAME, "basic")
    TSFX_GEOMS_ALL(TSFX_GEOM_NAME, "sorted")
    TSFX_GEOMS_ALL(TSFX_GEOM_NAME, "spectral") TSFX_GEOMS_ALL(TSFX_GEOM_NAME, "spectral/pow2")
    "la/small", TSFX_GEOMS_ALL(TSFX_GEOM_NAME, "la")
    "entropy/rank-g1", "entropy/rank-g4", "entropy/rank-g16", TSFX_GEOMS_ENTROPY(TSFX_GEOM_NAME, "entropy/tiles")
    "seq/small", TSFX_GEOMS_SEQ(TSFX_GEOM_NAME, "seq/general")
    "peaks/small", TSFX_GEOMS_PEAKS(TSFX_GEOM_NAME, "peaks/general") TSFX_GEOMS_PEAKS(TSFX_GEOM_NAME, "peaks/general/hybrid")
};

extern "C" int tsfx_kernel_variants(const char** names_out, int32_t cap) {
    const int n = (int)(sizeof(kKernelVariants) / sizeof(kKernelVariants[0]));
    for (int i = 0; i < n && i < cap && names_out; ++i) names_out[i] = kKernelVariants[i];
    return n;
}

// ------------------------------------------------------------------------------------------ stage (a)
// Long frame on the host -> device CSR -> kernels, pipelined.  See tsfx_csr.h for the two paths.  The columns are copied
// through Stager::h2d (pinned sources go straight to cudaMemcpyAsync, pageable ones through the pinned ring) into the
// workspace's W.ids() / W.keys() / W.vals(), and the value columns of kinds 1.. into ctx->kvals.
struct LongIn {
    const int64_t* ids;
    const void* keys;
    int is_f64;
    const float* values;           // value column of kind 0
    int64_t n;
    const float* const* more = nullptr;   // value columns of kinds 1 .. n_kinds-1 (wide format: the kinds share ids and sort keys)
    int n_kinds = 1;
    const float* col(int k) const { return k == 0 ? values : more[k - 1]; }
};

static inline size_t kind_stride(int64_t n) { return ((size_t)n + 3) & ~(size_t)3; }   // floats between the kinds' device columns

static int nan_error(tsfx_ctx* ctx) { return fail(ctx, TSFX_E_NAN, "the value column contains NaN"); }

// Copies the id column to the device and runs the ids pass; one synchronisation for the sizes (*info).  The key and
// value columns are then streamed by run_blocks (ids ascending) or copied whole by stage_a_sort.
static int stage_a(tsfx_ctx* ctx, const LongIn& in, int max_blocks, CsrInfo* info) {
    CsrWorkspace& W = ctx->csr;
    const int64_t n = in.n;
    CK(W.reserve(0, (size_t)n * 8));
    CK(W.reserve(2, (size_t)n * 4 + 16));
    if (in.keys) CK(W.reserve(1, (size_t)n * 8));
    CK(ctx->stager.h2d(W.ids(), in.ids, (size_t)n * 8, ctx->stream));
    std::string msg;
    int rc = csr_ids_pass(W, W.ids(), n, 16384, max_blocks, ctx->stream, &msg);
    if (rc) return fail(ctx, rc, msg);
    CK(cudaStreamSynchronize(ctx->stream));
    *info = *W.h_info;
    return TSFX_OK;
}

// rows in arbitrary order: (copy the key and value columns unless they are resident,) sort, rebuild the CSR
static int stage_a_sort(tsfx_ctx* ctx, const LongIn& in, bool resident, int max_blocks, bool check_nan, CsrInfo* info) {
    CsrWorkspace& W = ctx->csr;
    if (!resident) {
        if (in.keys) CK(ctx->stager.h2d(W.keys(), in.keys, (size_t)in.n * 8, ctx->stream));
        CK(ctx->stager.h2d(W.vals(), in.values, (size_t)in.n * 4, ctx->stream));
    }
    std::string msg;
    int rc = csr_sort_pass(W, W.ids(), in.keys ? W.keys() : nullptr, in.is_f64, W.vals(), in.n, 16384, max_blocks, check_nan,
                           ctx->stream, &msg);
    if (rc) return fail(ctx, rc, msg);
    CK(cudaStreamSynchronize(ctx->stream));
    *info = *W.h_info;
    if (info->has_nan) return nan_error(ctx);
    return TSFX_OK;
}

// the kinds of one call: plan, device value column (CSR order) and first output column of each
struct KindSet {
    int n = 1;
    const tsfx_plan* plan[TSFX_MAX_KINDS];
    const float* dvals[TSFX_MAX_KINDS];
    int col0[TSFX_MAX_KINDS];
    int total_cols = 0;
};

// kernels + result transfer over the row blocks of the device CSR: results go through ctx->out and are copied to `out`
// (host) block by block on the D2H stream.  stream_in (rows ordered by id, only the ids on the device): the key / value
// rows of a block are copied from the host right before the block's kernels and checked for sort keys that decrease
// inside an id and for NaN.  Several kinds (wide format) share the CSR: every block runs each kind's plan on that kind's
// value column and writes its own column block of the one result matrix.
static int run_blocks(tsfx_ctx* ctx, const KindSet& K, const CsrInfo& info, const LongIn* stream_in, bool check_nan,
                      double* out, uint32_t flags, const int64_t* row_times) {
    CsrWorkspace& W = ctx->csr;
    const size_t ncols = (size_t)K.total_cols;
    const int64_t ns = info.n_series;
    CK(ctx->out.reserve(std::max<size_t>((size_t)ns * ncols * sizeof(double), 8)));
    double* dout = (double*)ctx->out.p;
    const bool impute = (flags & TSFX_FLAG_IMPUTE) != 0;
    for (int b = 0; b < info.n_blocks; ++b) {
        const int64_t s0 = info.series_lo[b], s1 = info.series_lo[b + 1];
        const int64_t r0 = info.row_lo[b], r1 = info.row_lo[b + 1];
        const int slot = b & 1;
        if (stream_in) {
            const uint64_t* d_keys = stream_in->keys ? W.keys() : nullptr;
            if (d_keys) CK(ctx->stager.h2d(W.keys() + r0, (const uint64_t*)stream_in->keys + r0, (size_t)(r1 - r0) * 8, ctx->s_in));
            for (int k = 0; k < K.n; ++k)
                CK(ctx->stager.h2d(const_cast<float*>(K.dvals[k]) + r0, stream_in->col(k) + r0, (size_t)(r1 - r0) * 4, ctx->s_in));
            CK(cudaEventRecord(ctx->ev_in[slot], ctx->s_in));
            CK(cudaStreamWaitEvent(ctx->stream, ctx->ev_in[slot], 0));
            csr_check_rows(W, W.ids(), d_keys, stream_in->is_f64, K.dvals[0], r0, r1, check_nan, ctx->stream);
            if (check_nan) for (int k = 1; k < K.n; ++k) csr_check_nan(W, K.dvals[k] + r0, r1 - r0, ctx->stream);
        }
        for (int k = 0; k < K.n; ++k) {
            if (K.plan[k]->ncols == 0) continue;
            SeriesRef R;
            R.values = K.dvals[k]; R.begin = W.d_begin + s0; R.len = W.d_len + s0; R.dense_len = 0; R.n_series = s1 - s0;
            R.times = row_times;
            int rc = run_groups(ctx, K.plan[k], R, info.max_len, dout + (size_t)s0 * ncols + K.col0[k], flags, K.total_cols);
            if (rc) return rc;
        }
        if (impute) continue;
        CK(cudaEventRecord(ctx->ev_done[slot], ctx->stream));
        CK(cudaStreamWaitEvent(ctx->s_out, ctx->ev_done[slot], 0));
        CK(cudaMemcpyAsync(out + (size_t)s0 * ncols, dout + (size_t)s0 * ncols, (size_t)(s1 - s0) * ncols * sizeof(double),
                           cudaMemcpyDeviceToHost, ctx->s_out));
    }
    if (impute) {
        int rc = impute_after_extract(ctx, dout, ns, K.total_cols);
        if (rc) return rc;
        CK(cudaMemcpyAsync(out, dout, (size_t)ns * ncols * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    }
    return TSFX_OK;
}

// Rows with ascending ids take one streamed pass; if it finds a sort key that decreases inside an id, the columns it left
// on the device are sorted and the kernels run again.  Rows in any other order are copied whole and sorted first.
static int extract_long_impl(tsfx_ctx* ctx, const tsfx_plan* const* plans, const LongIn& in, int64_t* out_ids, double* out,
                             int64_t out_capacity, int64_t** out_ids_alloc, double** out_alloc, int64_t* n_series_out,
                             uint32_t flags) {
    CsrWorkspace& W = ctx->csr;
    const tsfx_plan* plan = plans[0];
    KindSet K;
    K.n = in.n_kinds;
    if (K.n < 1 || K.n > TSFX_MAX_KINDS) return fail(ctx, TSFX_E_INVALID, "between 1 and 64 kinds per call");
    for (int k = 0; k < K.n; ++k) {
        if (!plans[k] || plans[k]->ctx != ctx) return fail(ctx, TSFX_E_INVALID, "plan does not belong to this context");
        K.plan[k] = plans[k];
        K.col0[k] = K.total_cols;
        K.total_cols += plans[k]->ncols;
    }
    for (int k = 0; k < K.n; ++k) if (plans[k]->need_times) plan = plans[k];      // take_times looks at one plan's flag
    const size_t kstride = kind_stride(in.n);
    if (K.n > 1) CK(ctx->kvals.reserve((size_t)(K.n - 1) * kstride * 4 + 16));
    auto kind_in = [&](int k) { return (float*)ctx->kvals.p + (size_t)(k - 1) * kstride; };   // kind k >= 1, input row order
    const bool check_nan = !(flags & TSFX_FLAG_NO_NAN_CHECK);
    const int max_blocks = (flags & TSFX_FLAG_TIMING) ? 1 : 16;
    const int64_t* times_in = nullptr;           // row timestamps (input row order), device
    int rc = take_times(ctx, plan, in.n, &times_in);
    if (rc) return rc;
    // the result: blocks from the pinned pool (out_alloc) or the caller's buffers, once the number of series is known
    auto size_result = [&](const CsrInfo& info) -> int {
        const int64_t ns = info.n_series;
        *n_series_out = ns;
        if (out_alloc) {
            *out_alloc = (double*)ctx->pool.alloc(std::max<size_t>((size_t)ns * K.total_cols * sizeof(double), 8));
            *out_ids_alloc = (int64_t*)ctx->pool.alloc(std::max<size_t>((size_t)ns * 8, 8));
            if (!*out_alloc || !*out_ids_alloc) return fail(ctx, TSFX_E_NOMEM, "pinned host allocation failed");
            out = *out_alloc;
            out_ids = *out_ids_alloc;
        } else if (ns > out_capacity) {
            return fail(ctx, TSFX_E_INVALID, "out_capacity too small: " + std::to_string(ns) + " series");
        }
        if (info.max_len < 1 && ns > 0) return fail(ctx, TSFX_E_INVALID, "empty series");
        return TSFX_OK;
    };
    CsrInfo info;
    rc = stage_a(ctx, in, max_blocks, &info);
    if (rc) return rc;
    bool streamed = false;         // the streamed pass ran: the result is sized and every column is on the device
    if (!info.unsorted_ids) {
        W.d_values = W.vals();
        K.dvals[0] = W.d_values;
        for (int k = 1; k < K.n; ++k) K.dvals[k] = kind_in(k);
        rc = size_result(info);
        if (rc) return rc;
        rc = run_blocks(ctx, K, info, &in, check_nan, out, flags, times_in);
        if (rc) return rc;
        if (out_ids) CK(cudaMemcpyAsync(out_ids, W.d_uid, (size_t)info.n_series * sizeof(int64_t), cudaMemcpyDeviceToHost, ctx->stream));
        CK(cudaMemcpyAsync(W.h_info, W.d_info, sizeof(CsrInfo), cudaMemcpyDeviceToHost, ctx->stream));
        CK(cudaStreamSynchronize(ctx->s_out));
        CK(cudaStreamSynchronize(ctx->stream));
        if (W.h_info->has_nan) return nan_error(ctx);
        if (!W.h_info->unsorted_keys) return TSFX_OK;
        streamed = true;           // some sort key decreases inside an id
    }
    rc = stage_a_sort(ctx, in, /*resident=*/streamed, max_blocks, check_nan, &info);
    if (rc) return rc;
    // the rows were sorted on the device: the other kinds and the row timestamps follow the permutation
    K.dvals[0] = W.d_values;
    if (K.n > 1) {
        CK(ctx->kvals_sorted.reserve((size_t)(K.n - 1) * kstride * 4 + 16));
        for (int k = 1; k < K.n; ++k) {
            if (!streamed) CK(ctx->stager.h2d(kind_in(k), in.col(k), (size_t)in.n * 4, ctx->stream));
            if (check_nan) csr_check_nan(W, kind_in(k), in.n, ctx->stream);
            float* dst = (float*)ctx->kvals_sorted.p + (size_t)(k - 1) * kstride;
            csr_gather_f32(W, kind_in(k), dst, in.n, ctx->stream);
            K.dvals[k] = dst;
        }
    }
    if (!streamed) {
        rc = size_result(info);
        if (rc) return rc;
    }
    const int64_t* row_times = nullptr;
    if (times_in) {
        CK(ctx->times_sorted.reserve((size_t)in.n * 8));
        csr_gather_i64(W, times_in, (int64_t*)ctx->times_sorted.p, in.n, ctx->stream);
        row_times = (const int64_t*)ctx->times_sorted.p;
    }
    rc = run_blocks(ctx, K, info, nullptr, check_nan, out, flags, row_times);
    if (rc) return rc;
    if (out_ids) CK(cudaMemcpyAsync(out_ids, W.d_uid, (size_t)info.n_series * sizeof(int64_t), cudaMemcpyDeviceToHost, ctx->stream));
    // the NaN scans of the other kinds' columns were queued after the sort pass read its flags: read them again
    const bool late_nan_flags = K.n > 1 && check_nan;
    if (late_nan_flags) CK(cudaMemcpyAsync(W.h_info, W.d_info, sizeof(CsrInfo), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->s_out));
    CK(cudaStreamSynchronize(ctx->stream));
    if (late_nan_flags && W.h_info->has_nan) return nan_error(ctx);
    return TSFX_OK;
}

extern "C" int tsfx_extract_long(tsfx_ctx* ctx, const tsfx_plan* plan, const int64_t* ids, const void* sort_keys,
                                 int32_t sort_key_is_f64, const float* values, int64_t n_rows, int64_t* out_ids,
                                 double* out, int64_t out_capacity, int64_t* n_series_out, uint32_t flags) {
    if (!ctx) return TSFX_E_INVALID;
    if (!plan || plan->ctx != ctx) return fail(ctx, TSFX_E_INVALID, "plan does not belong to this context");
    if (flags & TSFX_FLAG_DEVICE_PTRS)
        return fail(ctx, TSFX_E_INVALID, "tsfx_extract_long takes host pointers (device rows: tsfx_stage_long_stacked, tsfx_extract_staged)");
    if (n_rows < 0 || !n_series_out || (n_rows > 0 && (!ids || !values)) || !out)
        return fail(ctx, TSFX_E_INVALID, "tsfx_extract_long: bad arguments");
    CK(cudaSetDevice(ctx->device));
    *n_series_out = 0;
    if (n_rows == 0) return TSFX_OK;
    LongIn in{ids, sort_keys, sort_key_is_f64, values, n_rows};
    return extract_long_impl(ctx, &plan, in, out_ids, out, out_capacity, nullptr, nullptr, n_series_out, flags);
}

// tsfx_extract_long_alloc / _kinds after their argument checks: the result comes from the pinned pool, and goes back to
// it when the call fails
static int extract_long_pooled(tsfx_ctx* ctx, const tsfx_plan* const* plans, const LongIn& in, int64_t** out_ids,
                               double** out, int64_t* n_series_out, uint32_t flags) {
    CK(cudaSetDevice(ctx->device));
    *n_series_out = 0;
    *out = nullptr;
    *out_ids = nullptr;
    if (in.n == 0) return TSFX_OK;
    int rc = extract_long_impl(ctx, plans, in, nullptr, nullptr, 0, out_ids, out, n_series_out, flags);
    if (rc) {
        if (*out) ctx->pool.free(*out);
        if (*out_ids) ctx->pool.free(*out_ids);
        *out = nullptr; *out_ids = nullptr;
    }
    return rc;
}

extern "C" int tsfx_extract_long_alloc(tsfx_ctx* ctx, const tsfx_plan* plan, const int64_t* ids, const void* sort_keys,
                                       int32_t sort_key_is_f64, const float* values, int64_t n_rows, int64_t** out_ids,
                                       double** out, int64_t* n_series_out, uint32_t flags) {
    if (!ctx) return TSFX_E_INVALID;
    if (!plan || plan->ctx != ctx) return fail(ctx, TSFX_E_INVALID, "plan does not belong to this context");
    if (flags & TSFX_FLAG_DEVICE_PTRS) return fail(ctx, TSFX_E_INVALID, "tsfx_extract_long_alloc takes host pointers");
    if (n_rows < 0 || !n_series_out || !out || !out_ids || (n_rows > 0 && (!ids || !values)))
        return fail(ctx, TSFX_E_INVALID, "tsfx_extract_long_alloc: bad arguments");
    return extract_long_pooled(ctx, &plan, LongIn{ids, sort_keys, sort_key_is_f64, values, n_rows}, out_ids, out,
                               n_series_out, flags);
}

extern "C" int tsfx_extract_long_kinds(tsfx_ctx* ctx, const tsfx_plan* const* plans, const int64_t* ids, const void* sort_keys,
                                       int32_t sort_key_is_f64, const float* const* values, int32_t n_kinds, int64_t n_rows,
                                       int64_t** out_ids, double** out, int64_t* n_series_out, uint32_t flags) {
    if (!ctx) return TSFX_E_INVALID;
    if (flags & TSFX_FLAG_DEVICE_PTRS) return fail(ctx, TSFX_E_INVALID, "tsfx_extract_long_kinds takes host pointers");
    if (n_kinds < 1 || n_kinds > TSFX_MAX_KINDS || !plans || !values || n_rows < 0 || !n_series_out || !out || !out_ids ||
        (n_rows > 0 && !ids))
        return fail(ctx, TSFX_E_INVALID, "tsfx_extract_long_kinds: bad arguments");
    for (int k = 0; k < n_kinds; ++k)
        if (!plans[k] || (n_rows > 0 && !values[k])) return fail(ctx, TSFX_E_INVALID, "tsfx_extract_long_kinds: NULL plan / column");
    LongIn in{ids, sort_keys, sort_key_is_f64, values[0], n_rows};
    in.more = values + 1;
    in.n_kinds = n_kinds;
    return extract_long_pooled(ctx, plans, in, out_ids, out, n_series_out, flags);
}

// ------------------------------------------------------------------------------------------ stacked long format
// the rows and their alignment gaps are counted in int (CUB scans)
static const int64_t kMaxStackedRows = ((int64_t)1 << 31) - 2 - TSFX_MAX_KINDS * TSFX_STACK_ALIGN;
extern "C" int tsfx_stage_long_stacked(tsfx_ctx* ctx, const int64_t* ids, const void* sort_keys, int32_t sort_key_is_f64,
                                       const float* values, const void* kind_codes, int32_t kind_code_is_i64, int32_t n_kinds,
                                       const int64_t* row_time_ns, int64_t n_rows, int64_t* n_ids_out, int64_t* rows_per_kind,
                                       int32_t* max_len_per_kind, uint32_t flags) {
    if (!ctx) return TSFX_E_INVALID;
    StackedWorkspace& S = ctx->stacked;
    S.pending = false;
    ctx->launches = 0;
    ctx->n_kernels = 0;
    if (!(flags & TSFX_FLAG_DEVICE_PTRS)) return fail(ctx, TSFX_E_INVALID, "tsfx_stage_long_stacked takes device pointers");
    if (n_kinds < 1 || n_kinds > TSFX_MAX_KINDS) return fail(ctx, TSFX_E_INVALID, "between 1 and 64 kinds per call");
    if (n_rows < 0 || !n_ids_out || !rows_per_kind || !max_len_per_kind || (n_rows > 0 && (!ids || !values)))
        return fail(ctx, TSFX_E_INVALID, "tsfx_stage_long_stacked: bad arguments");
    if (n_rows > kMaxStackedRows) return fail(ctx, TSFX_E_UNSUPPORTED, "more than 2^31 - 4 098 rows in one call");
    CK(cudaSetDevice(ctx->device));
    *n_ids_out = 0;
    for (int k = 0; k < n_kinds; ++k) { rows_per_kind[k] = 0; max_len_per_kind[k] = 0; }
    S.n_kinds = n_kinds;
    S.n_union = 0;
    S.d_times = nullptr;
    S.d_keys = nullptr;
    S.d_src = nullptr;
    S.has_keys = false;
    S.staged = Staged::Rows;
    if (n_rows > 0) {
        std::string msg;
        int rc = stacked_stage(S, ctx->csr, ids, (const uint64_t*)sort_keys, sort_keys && sort_key_is_f64, values, kind_codes,
                               kind_code_is_i64, n_kinds, row_time_ns, n_rows, (flags & TSFX_FLAG_KEEP_SORT_KEYS) != 0,
                               (flags & TSFX_FLAG_KEEP_ROW_NUMBERS) != 0, ctx->stream, &msg);
        if (rc) return fail(ctx, rc, msg);
        CK(cudaStreamSynchronize(ctx->stream));
        const StackedInfo& I = *S.h_info;
        if (I.bad_kind) return fail(ctx, TSFX_E_INVALID, "a kind code is outside 0 .. " + std::to_string(n_kinds - 1));
        if (I.nan_values) return nan_error(ctx);
        if (I.nan_keys) return fail(ctx, TSFX_E_NAN, "the float64 sort keys contain NaN");
        CK(S.keep_ids(ctx->csr.d_uid, I.n_union, ctx->stream));
        S.n_union = I.n_union;
        for (int k = 0; k < n_kinds; ++k) {
            rows_per_kind[k] = I.kind_rows[k];
            max_len_per_kind[k] = I.kind_max_len[k];
        }
    }
    *n_ids_out = S.n_union;
    S.pending = true;
    return TSFX_OK;
}

extern "C" int tsfx_extract_staged(tsfx_ctx* ctx, const tsfx_plan* const* plans, int64_t* out_ids, double* out, int32_t ld,
                                   uint32_t flags) {
    if (!ctx) return TSFX_E_INVALID;
    StackedWorkspace& S = ctx->stacked;
    ctx->launches = 0;
    ctx->n_kernels = 0;
    if (!S.pending) return fail(ctx, TSFX_E_INVALID, "tsfx_extract_staged: no rows staged (tsfx_stage_long_stacked)");
    S.pending = false;
    const int64_t U = S.n_union;
    if (U == 0) return TSFX_OK;
    if (!plans || !out_ids) return fail(ctx, TSFX_E_INVALID, "tsfx_extract_staged: bad arguments");
    const StackedInfo& I = *S.h_info;
    int col0[TSFX_MAX_KINDS], total = 0;
    size_t block = 0;             // largest staging block of a kind that covers only some of the union rows
    bool holes = false;
    for (int k = 0; k < S.n_kinds; ++k) {
        col0[k] = total;
        if (I.kind_rows[k] == 0) continue;          // a kind without rows has no columns
        const tsfx_plan* P = plans[k];
        if (!P || P->ctx != ctx) return fail(ctx, TSFX_E_INVALID, "plan does not belong to this context");
        total += P->ncols;
        if (P->ncols == 0) continue;
        if (int rc = check_lengths(ctx, P, I.kind_max_len[k])) return rc;
        if (P->need_times && !S.d_times) return fail(ctx, TSFX_E_INVALID, "linear_trend_timewise needs the row timestamps");
        const int64_t ns = I.kind_series[k + 1] - I.kind_series[k];
        if (ns < U) { holes = true; block = std::max(block, (size_t)ns * P->ncols * sizeof(double)); }
    }
    if (total > 0 && !out) return fail(ctx, TSFX_E_INVALID, "tsfx_extract_staged: NULL out");
    if (ld < total) return fail(ctx, TSFX_E_INVALID, "tsfx_extract_staged: row stride " + std::to_string(ld) + " < " + std::to_string(total) + " columns");
    if (ld != total && (flags & TSFX_FLAG_IMPUTE)) return fail(ctx, TSFX_E_INVALID, "TSFX_FLAG_IMPUTE needs a contiguous result matrix");
    CK(cudaSetDevice(ctx->device));
    int launched = 0;
    if (holes) {              // cells of an (id, kind) pair without rows stay NaN
        CK(ctx->out.reserve(block));
        CK(stacked_fill_nan(out, U, total, ld, ctx->stream));
        launched += 1;
    }
    for (int k = 0; k < S.n_kinds; ++k) {
        if (I.kind_rows[k] == 0 || plans[k]->ncols == 0) continue;
        const tsfx_plan* P = plans[k];
        const int64_t s0 = I.kind_series[k], ns = I.kind_series[k + 1] - s0;
        SeriesRef R;
        R.values = S.d_values; R.begin = S.d_begin + s0; R.len = S.d_len + s0; R.dense_len = 0; R.n_series = ns;
        R.times = S.d_times;
        // a kind with a series for every union row fills its columns in place; the others go through a staging block
        // and are scattered to their union rows
        double* dst = ns == U ? out + col0[k] : (double*)ctx->out.p;
        int rc = run_groups(ctx, P, R, I.kind_max_len[k], dst, flags, ns == U ? ld : P->ncols);
        if (rc) return rc;
        launched += ctx->launches;
        if (ns < U) {
            CK(stacked_scatter(dst, ns, P->ncols, S.d_row + s0, out + col0[k], ld, ctx->stream));
            launched += 1;
        }
    }
    CK(cudaMemcpyAsync(out_ids, S.d_uid, (size_t)U * sizeof(int64_t), cudaMemcpyDeviceToDevice, ctx->stream));
    ctx->launches = launched;
    if (flags & TSFX_FLAG_IMPUTE) return impute_after_extract(ctx, out, U, total);
    return TSFX_OK;
}

// ------------------------------------------------------------------------------------------ deferred long format
// tsfx_prepare_long's slot and check buffers for n = n_kinds x max_ids slots: per slot its view and union row
// (stacked_slots), its private view and reject reason (defer_check); the first rejected slot per reason, the live
// series of every kind and the first id past max_ids
struct LongSlots {
    unsigned long long* first;
    int64_t *sbegin, *vbegin, *live, *id_past;
    int32_t *slen, *vlen, *srow;
    uint8_t* reject;
};
static size_t long_slot_bytes(int64_t n) { return 64 + 8 * (TSFX_MAX_KINDS + 1) + (size_t)n * 29; }
static LongSlots long_slots(tsfx_ctx* ctx) {
    char* p = (char*)ctx->long_slots.p;
    const size_t n = (size_t)ctx->long_kinds * ctx->long_ids;
    LongSlots B;
    B.first = (unsigned long long*)p;
    B.live = (int64_t*)(p + 64);
    B.id_past = B.live + TSFX_MAX_KINDS;
    p += 64 + 8 * (TSFX_MAX_KINDS + 1);
    B.sbegin = (int64_t*)p;
    B.vbegin = B.sbegin + n;
    B.slen = (int32_t*)(B.vbegin + n);
    B.vlen = B.slen + n;
    B.srow = B.vlen + n;
    B.reject = (uint8_t*)(B.srow + n);
    return B;
}

extern "C" int tsfx_prepare_long(tsfx_ctx* ctx, const tsfx_plan* const* plans, int32_t n_kinds, int64_t max_rows, int64_t max_ids,
                                 int32_t max_len) {
    if (!ctx) return TSFX_E_INVALID;
    if (n_kinds < 1 || n_kinds > TSFX_MAX_KINDS || !plans) return fail(ctx, TSFX_E_INVALID, "between 1 and 64 kinds per call");
    if (max_rows < 1 || max_rows > kMaxStackedRows || max_ids < 1 || max_ids > 0x7fffffff || max_len < 1)
        return fail(ctx, TSFX_E_INVALID, "tsfx_prepare_long: max_rows in 1 .. 2^31 - 4 098, max_ids in 1 .. 2^31 - 1 and "
                                         "max_len >= 1");
    int64_t cols = 0;
    for (int k = 0; k < n_kinds; ++k) {
        if (plans[k] && plans[k]->ctx != ctx) return fail(ctx, TSFX_E_INVALID, "plan does not belong to this context");
        if (plans[k]) cols += plans[k]->ncols;
    }
    CK(cudaSetDevice(ctx->device));
    ctx->long_kinds = 0;                  // unprepared until every step succeeded
    for (int k = 0; k < n_kinds; ++k) {
        if (!plans[k] || plans[k]->ncols == 0) continue;
        if (int rc = check_lengths(ctx, plans[k], max_len)) return rc;
        if (int rc = reserve_groups(ctx, plans[k], max_ids, max_len)) return rc;
    }
    std::string msg;
    ctx->stacked.frozen = ctx->csr.frozen = false;
    if (int rc = stacked_defer_reserve(ctx->stacked, ctx->csr, max_rows, n_kinds, &msg)) return fail(ctx, rc, msg);
    CK(ctx->long_slots.reserve(long_slot_bytes((int64_t)n_kinds * max_ids)));
    CK(ctx->long_out.reserve(std::max<size_t>((size_t)max_ids * cols * sizeof(double), 8)));
    for (int k = 0; k < n_kinds; ++k) ctx->long_plans[k] = plans[k] && plans[k]->ncols > 0 ? plans[k] : nullptr;
    ctx->long_kinds = n_kinds;
    ctx->long_rows = max_rows;
    ctx->long_ids = max_ids;
    ctx->long_len = max_len;
    CK(cudaStreamSynchronize(ctx->stream));     // the tables are filled before a captured call, which cannot wait for them
    return TSFX_OK;
}

// While a deferred call enqueues, the stage's workspaces fail instead of growing (a graph holds their addresses)
struct FreezeStage {
    tsfx_ctx* ctx;
    explicit FreezeStage(tsfx_ctx* c) : ctx(c) { ctx->stacked.frozen = ctx->csr.frozen = true; }
    ~FreezeStage() { ctx->stacked.frozen = ctx->csr.frozen = false; }
};

// stage -> slots -> deferred check -> every kind's groups on its slots -> report -> NaN matrix and scatter of the live
// slots -> ids and status (tsfx.h "Deferred long format")
extern "C" int tsfx_extract_long_deferred(tsfx_ctx* ctx, const int64_t* ids, const void* sort_keys, int32_t sort_key_is_f64,
                                          const float* values, const void* kind_codes, int32_t kind_code_is_i64, int64_t n_rows,
                                          const int64_t* n_rows_live, int64_t* out_ids, int64_t* n_ids, double* out, int32_t ld,
                                          uint32_t flags) {
    if (!ctx) return TSFX_E_INVALID;
    ctx->launches = 0;
    ctx->n_kernels = 0;
    if (flags != TSFX_FLAG_DEVICE_PTRS) return fail(ctx, TSFX_E_INVALID, "tsfx_extract_long_deferred takes TSFX_FLAG_DEVICE_PTRS alone");
    const int K = ctx->long_kinds;
    const int64_t M = ctx->long_ids;
    if (K == 0) return fail(ctx, TSFX_E_INVALID, "tsfx_extract_long_deferred: no shape prepared (tsfx_prepare_long)");
    if (!ctx->status) return fail(ctx, TSFX_E_INVALID, "tsfx_extract_long_deferred needs a status buffer (tsfx_set_status)");
    if (n_rows < 0 || n_rows > ctx->long_rows)
        return fail(ctx, TSFX_E_INVALID, "tsfx_extract_long_deferred: " + std::to_string(n_rows) + " rows, more than the " +
                                             std::to_string(ctx->long_rows) + " tsfx_prepare_long made ready");
    int col0[TSFX_MAX_KINDS], total = 0;
    for (int k = 0; k < K; ++k) { col0[k] = total; if (ctx->long_plans[k]) total += ctx->long_plans[k]->ncols; }
    if ((n_rows > 0 && (!ids || !values)) || !out_ids || !n_ids || (total > 0 && !out))
        return fail(ctx, TSFX_E_INVALID, "tsfx_extract_long_deferred: bad arguments");
    if (ld < total) return fail(ctx, TSFX_E_INVALID, "tsfx_extract_long_deferred: row stride " + std::to_string(ld) + " < " +
                                                       std::to_string(total) + " columns");
    CK(cudaSetDevice(ctx->device));
    StackedWorkspace& S = ctx->stacked;
    FreezeStage freeze(ctx);
    std::string msg;
    // the sizes first, so that a call beyond the prepared buffers fails before it enqueues anything
    if (int rc = stacked_defer_reserve(S, ctx->csr, std::max<int64_t>(n_rows, 1), K, &msg)) return fail(ctx, rc, msg);
    const LongSlots B = long_slots(ctx);
    const cudaStream_t st = ctx->stream;
    CK(cudaMemsetAsync(B.first, 0, 3 * sizeof(unsigned long long), st));
    if (int rc = stacked_stage_deferred(S, ctx->csr, ids, (const uint64_t*)sort_keys, sort_keys && sort_key_is_f64, values,
                                        kind_codes, kind_code_is_i64, K, n_rows, n_rows_live, M, out_ids, B.id_past, st, &msg))
        return fail(ctx, rc, msg);
    CK(stacked_slots(S, K, M, B.sbegin, B.slen, B.srow, B.reject, B.live, st));
    const int64_t n_pad = n_rows + (int64_t)K * TSFX_STACK_ALIGN;      // the staged values, alignment gaps included
    CK(defer_check(S.d_values, n_pad, B.sbegin, B.slen, K * M, ctx->long_len, B.vbegin, B.vlen, B.reject, B.first, st, true));
    int launched = 3;
    double* block = (double*)ctx->long_out.p;
    for (int k = 0; k < K; ++k) {
        const tsfx_plan* P = ctx->long_plans[k];
        if (!P) continue;
        SeriesRef R;
        R.values = S.d_values; R.begin = B.vbegin + k * M; R.len = B.vlen + k * M; R.dense_len = 0; R.n_series = M;
        R.times = nullptr;
        if (int rc = run_groups(ctx, P, R, ctx->long_len, block + M * col0[k], 0, P->ncols)) return rc;
        launched += ctx->launches;
    }
    // the report only (no columns: the rejected slots are left out of the scatter, so their cells keep the NaN fill)
    CK(defer_finish(nullptr, K * M, 0, 0, B.reject, B.first, ctx->status, st));
    CK(stacked_fill_nan(out, M, total, ld, st));
    launched += 2;
    for (int k = 0; k < K; ++k) {
        const tsfx_plan* P = ctx->long_plans[k];
        if (!P) continue;
        CK(stacked_scatter(block + M * col0[k], M, P->ncols, B.srow + k * M, out + col0[k], ld, st, B.live + k, B.reject + k * M));
        launched += 1;
    }
    CK(stacked_defer_report(S, M, B.id_past, B.srow, out_ids, n_ids, ctx->status, st));
    ctx->launches = launched + 1;
    return TSFX_OK;
}

// The steps tsfx_roll_staged and tsfx_sub_staged share before they replace the staged series by pieces of them (`to`):
// the state check, then the caller's argument error `bad` (nullptr: none), the outputs zeroed and the stage consumed
// until the call succeeds.  *empty: no rows are staged, so the call is complete.
static int regroup_begin(tsfx_ctx* ctx, const char* call, Staged to, const char* bad, int64_t* n_rows_out,
                         int32_t* max_len_per_kind, bool* empty) {
    StackedWorkspace& S = ctx->stacked;
    ctx->launches = 0;
    ctx->n_kernels = 0;
    if (!S.pending || S.staged != Staged::Rows)
        return fail(ctx, TSFX_E_INVALID, std::string(call) + ": no unrolled, unpackaged rows staged (tsfx_stage_long_stacked)");
    if (bad) return fail(ctx, TSFX_E_INVALID, bad);
    S.pending = false;
    *n_rows_out = 0;
    for (int k = 0; k < S.n_kinds; ++k) max_len_per_kind[k] = 0;
    *empty = S.n_union == 0;
    if (*empty) { S.staged = to; S.pending = true; return TSFX_OK; }
    CK(cudaSetDevice(ctx->device));
    return TSFX_OK;
}

// The steps they share once the regrouping is enqueued: the new stage state, one synchronisation, then the pieces'
// sizes published and the stage ready for tsfx_extract_staged.
static int regroup_end(tsfx_ctx* ctx, Staged to, int64_t* n_rows_out, int32_t* max_len_per_kind) {
    StackedWorkspace& S = ctx->stacked;
    S.staged = to;
    CK(cudaStreamSynchronize(ctx->stream));
    const StackedInfo& I = *S.h_info;
    if (I.dup_names)
        return fail(ctx, TSFX_E_INVALID, "two windows of one kind have the same name (id, sort key): the sort keys tie at "
                                         "the rows that name them");
    S.n_union = I.n_union;
    for (int k = 0; k < S.n_kinds; ++k) max_len_per_kind[k] = I.kind_max_len[k];
    *n_rows_out = S.n_union;
    S.pending = true;
    return TSFX_OK;
}

extern "C" int tsfx_roll_staged(tsfx_ctx* ctx, int32_t rolling_direction, int32_t max_timeshift, int32_t min_timeshift,
                                int64_t* n_rows_out, int32_t* max_len_per_kind, uint32_t flags) {
    if (!ctx) return TSFX_E_INVALID;
    const bool forecast = (flags & TSFX_FLAG_FORECAST) != 0;
    const Staged to = forecast ? Staged::ForecastWindows : Staged::Windows;
    StackedWorkspace& S = ctx->stacked;
    const char* bad = nullptr;
    if (!n_rows_out || !max_len_per_kind || rolling_direction == 0 || max_timeshift < 0 || min_timeshift < 0)
        bad = "tsfx_roll_staged: bad arguments";
    else if (S.has_keys && !S.d_keys)
        bad = "tsfx_roll_staged: the rows were staged without TSFX_FLAG_KEEP_SORT_KEYS";
    else if (forecast && S.n_union > 0 && !S.d_src)
        bad = "tsfx_roll_staged: TSFX_FLAG_FORECAST needs rows staged with TSFX_FLAG_KEEP_ROW_NUMBERS";
    bool empty = false;
    if (int rc = regroup_begin(ctx, "tsfx_roll_staged", to, bad, n_rows_out, max_len_per_kind, &empty)) return rc;
    if (empty) return TSFX_OK;
    const StackedInfo& I = *S.h_info;
    // the shifts are anchored to the longest (kind, id) series; a window never has more rows than its series, and a
    // series of L rows has at most one window per shift <= L
    int32_t Lmax = 0;
    int64_t rows = 0;
    for (int k = 0; k < S.n_kinds; ++k) { Lmax = std::max(Lmax, I.kind_max_len[k]); rows += I.kind_rows[k]; }
    if (max_timeshift == 0) max_timeshift = Lmax;
    const RollSpec R = roll_spec(rolling_direction, max_timeshift, min_timeshift, Lmax);
    const int64_t shifts = (Lmax - R.first) / R.amount + 1;
    const int64_t series = I.kind_series[S.n_kinds];
    const int64_t bound = std::min(rows, series > rows / shifts ? rows : series * shifts);
    std::string msg;
    int rc = stacked_roll(S, ctx->csr, rolling_direction, max_timeshift, min_timeshift, Lmax, bound, forecast, ctx->stream,
                          &msg);
    if (rc) return fail(ctx, rc, msg);
    return regroup_end(ctx, to, n_rows_out, max_len_per_kind);
}

extern "C" int tsfx_sub_staged(tsfx_ctx* ctx, int64_t sub_length, int64_t* n_rows_out, int32_t* max_len_per_kind,
                               uint32_t flags) {
    (void)flags;
    if (!ctx) return TSFX_E_INVALID;
    StackedWorkspace& S = ctx->stacked;
    const char* bad = !n_rows_out || !max_len_per_kind || sub_length < 1 ? "tsfx_sub_staged: bad arguments" : nullptr;
    bool empty = false;
    if (int rc = regroup_begin(ctx, "tsfx_sub_staged", Staged::Packages, bad, n_rows_out, max_len_per_kind, &empty))
        return rc;
    if (empty) return TSFX_OK;
    const StackedInfo& I = *S.h_info;
    // every series has fewer than 2^31 rows, so a longer sub_length gives the same packages: whole series
    const int32_t L = (int32_t)std::min<int64_t>(sub_length, 0x7fffffff);
    // a kind of r rows in s series has at most r / L full packages and one shorter package per series, and every
    // package has a row
    int64_t rows = 0, bound = 0;
    for (int k = 0; k < S.n_kinds; ++k) {
        rows += I.kind_rows[k];
        bound += I.kind_rows[k] / L + (I.kind_series[k + 1] - I.kind_series[k]);
    }
    bound = std::min(bound, rows);
    std::string msg;
    int rc = stacked_sub(S, ctx->csr, L, bound, ctx->stream, &msg);
    if (rc) return fail(ctx, rc, msg);
    return regroup_end(ctx, Staged::Packages, n_rows_out, max_len_per_kind);
}

extern "C" int tsfx_staged_row_keys(tsfx_ctx* ctx, void* out_keys) {
    if (!ctx) return TSFX_E_INVALID;
    StackedWorkspace& S = ctx->stacked;
    if (S.staged == Staged::Rows)
        return fail(ctx, TSFX_E_INVALID, "tsfx_staged_row_keys: no windows or packages staged (tsfx_roll_staged, tsfx_sub_staged)");
    if (S.n_union == 0) return TSFX_OK;
    if (!out_keys) return fail(ctx, TSFX_E_INVALID, "tsfx_staged_row_keys: NULL out_keys");
    CK(cudaSetDevice(ctx->device));
    CK(cudaMemcpyAsync(out_keys, S.d_ukey, (size_t)S.n_union * 8, cudaMemcpyDeviceToDevice, ctx->stream));
    return TSFX_OK;
}

extern "C" int tsfx_staged_targets(tsfx_ctx* ctx, int64_t* out_rows) {
    if (!ctx) return TSFX_E_INVALID;
    StackedWorkspace& S = ctx->stacked;
    if (S.staged != Staged::ForecastWindows)
        return fail(ctx, TSFX_E_INVALID, "tsfx_staged_targets: no forecasting windows staged (tsfx_roll_staged, TSFX_FLAG_FORECAST)");
    if (S.n_union == 0) return TSFX_OK;
    if (!out_rows) return fail(ctx, TSFX_E_INVALID, "tsfx_staged_targets: NULL out_rows");
    CK(cudaSetDevice(ctx->device));
    CK(cudaMemcpyAsync(out_rows, S.d_utarget, (size_t)S.n_union * 8, cudaMemcpyDeviceToDevice, ctx->stream));
    return TSFX_OK;
}

extern "C" void* tsfx_host_alloc(tsfx_ctx* ctx, size_t bytes) {
    if (!ctx) return nullptr;
    cudaSetDevice(ctx->device);
    return ctx->pool.alloc(bytes);
}
extern "C" void tsfx_host_free(tsfx_ctx* ctx, void* p) {
    if (ctx && p) ctx->pool.free(p);
}

// ------------------------------------------------------------------------------------------ feature selection
extern "C" int tsfx_select_classification(tsfx_ctx* ctx, const double* X, int64_t n_rows, int32_t n_cols, const int32_t* y_codes,
                                          int32_t n_classes, double* out, uint32_t flags) {
    if (!ctx) return TSFX_E_INVALID;
    if (n_rows < 1 || n_cols < 0 || n_classes < 1 || !y_codes || !out || (n_cols > 0 && !X))
        return fail(ctx, TSFX_E_INVALID, "tsfx_select_classification: bad arguments");
    if (n_cols == 0) return TSFX_OK;
    CK(cudaSetDevice(ctx->device));
    std::vector<int64_t> counts(n_classes, 0);
    for (int64_t i = 0; i < n_rows; ++i) {
        if (y_codes[i] < 0 || y_codes[i] >= n_classes) return fail(ctx, TSFX_E_INVALID, "class code out of range");
        counts[y_codes[i]] += 1;
    }
    const double* d_X = X;
    if (!(flags & TSFX_FLAG_DEVICE_PTRS)) {
        CK(ctx->sel_x.reserve((size_t)n_rows * n_cols * 8));
        CK(ctx->stager.h2d(ctx->sel_x.p, X, (size_t)n_rows * n_cols * 8, ctx->stream));
        d_X = (const double*)ctx->sel_x.p;
    }
    CK(ctx->sel_y.reserve((size_t)n_rows * 4));
    CK(ctx->stager.h2d(ctx->sel_y.p, y_codes, (size_t)n_rows * 4, ctx->stream));
    const size_t ob = (size_t)n_classes * n_cols * TSFX_SEL_NSTAT * sizeof(double);
    CK(ctx->sel_out.reserve(ob));
    std::string msg;
    int has_nan = 0;
    int rc = select_class_stats(ctx->sel, d_X, n_rows, n_cols, (const int32_t*)ctx->sel_y.p, n_classes, counts.data(),
                                (double*)ctx->sel_out.p, &has_nan, ctx->stream, &msg);
    if (rc) return fail(ctx, rc, msg);
    CK(cudaMemcpyAsync(out, ctx->sel_out.p, ob, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    if (has_nan) return fail(ctx, TSFX_E_NAN, "the feature matrix contains NaN");
    return TSFX_OK;
}

extern "C" int tsfx_select_regression(tsfx_ctx* ctx, const double* X, int64_t n_rows, int32_t n_cols, const double* y, double* out,
                                      uint32_t flags) {
    if (!ctx) return TSFX_E_INVALID;
    if (n_rows < 1 || n_cols < 0 || !y || !out || (n_cols > 0 && !X))
        return fail(ctx, TSFX_E_INVALID, "tsfx_select_regression: bad arguments");
    if (n_cols == 0) return TSFX_OK;
    CK(cudaSetDevice(ctx->device));
    const double* d_X = X;
    if (!(flags & TSFX_FLAG_DEVICE_PTRS)) {
        CK(ctx->sel_x.reserve((size_t)n_rows * n_cols * 8));
        CK(ctx->stager.h2d(ctx->sel_x.p, X, (size_t)n_rows * n_cols * 8, ctx->stream));
        d_X = (const double*)ctx->sel_x.p;
    }
    CK(ctx->sel_y.reserve((size_t)n_rows * 8));
    CK(ctx->stager.h2d(ctx->sel_y.p, y, (size_t)n_rows * 8, ctx->stream));
    const size_t ob = ((size_t)n_cols * TSFX_SEL_NSTAT + 4) * sizeof(double);
    CK(ctx->sel_out.reserve(ob));
    std::string msg;
    int has_nan = 0;
    int rc = select_regression_stats(ctx->sel, d_X, n_rows, n_cols, (const double*)ctx->sel_y.p, (double*)ctx->sel_out.p, &has_nan,
                                     ctx->stream, &msg);
    if (rc) return fail(ctx, rc, msg);
    CK(cudaMemcpyAsync(out, ctx->sel_out.p, ob, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    if (has_nan) return fail(ctx, TSFX_E_NAN, "the feature matrix or the target contains NaN");
    return TSFX_OK;
}

// ------------------------------------------------------------------------------------------ multi-GPU placement
extern "C" int tsfx_set_peer_outputs(tsfx_ctx* ctx, const uint64_t* peer_out, int32_t n_peers, int32_t self_index,
                                     uint64_t multicast_out, int32_t mode) {
    if (!ctx) return TSFX_E_INVALID;
    CK(cudaSetDevice(ctx->device));
    CK(cudaStreamSynchronize(ctx->s_peer));
    ctx->peer_out.clear();
    ctx->peer_self = -1;
    ctx->peer_mc = 0;
    if (n_peers <= 0) return TSFX_OK;
    if (!peer_out || self_index < 0 || self_index >= n_peers || n_peers > 8 || mode < TSFX_PEER_AUTO || mode > TSFX_PEER_MULTICAST)
        return fail(ctx, TSFX_E_INVALID, "tsfx_set_peer_outputs: bad arguments (at most 8 ranks)");
    if (mode == TSFX_PEER_AUTO) mode = TSFX_PEER_COPY;      // copy engines: no SM time taken from the kernels (include/tsfx.h)
    if (mode == TSFX_PEER_MULTICAST && !multicast_out) return fail(ctx, TSFX_E_INVALID, "no multicast mapping was supplied");
    ctx->peer_out.assign(peer_out, peer_out + n_peers);
    ctx->peer_self = self_index;
    ctx->peer_mc = multicast_out;
    ctx->peer_mode = mode;
    return TSFX_OK;
}

extern "C" int tsfx_set_max_len_hint(tsfx_ctx* ctx, int32_t max_len) {
    if (!ctx || max_len < 0) return TSFX_E_INVALID;
    ctx->max_len_hint = max_len;
    return TSFX_OK;
}

extern "C" int tsfx_set_out_ld(tsfx_ctx* ctx, int32_t ld) {
    if (!ctx || ld < 0) return TSFX_E_INVALID;
    ctx->out_ld = ld;
    return TSFX_OK;
}

extern "C" int tsfx_peer_flush(tsfx_ctx* ctx) {
    if (!ctx) return TSFX_E_INVALID;
    CK(cudaSetDevice(ctx->device));
    CK(cudaEventRecord(ctx->ev_peer, ctx->s_peer));
    CK(cudaStreamWaitEvent(ctx->stream, ctx->ev_peer, 0));
    return TSFX_OK;
}

// ------------------------------------------------------------------------------------------ roll_time_series views
extern "C" int64_t tsfx_roll_windows(const int64_t* begin, const int32_t* len, int64_t n_series,
                                     int32_t rolling_direction, int32_t max_timeshift, int32_t min_timeshift,
                                     int64_t* win_begin, int32_t* win_len, int64_t* win_parent,
                                     int32_t* win_end_index, int64_t capacity) {
    // the window arithmetic (dataframe_functions.py:340-373, 548-562) is tsfx_roll.cuh's, shared with tsfx_roll_staged;
    // win_end_index is "the row whose sort value names the window": last row (positive) / first row (negative).
    if (!begin || !len || n_series < 0 || rolling_direction == 0 || max_timeshift < 0 || min_timeshift < 0)
        return TSFX_E_INVALID;
    int32_t Lmax = 0;
    for (int64_t s = 0; s < n_series; ++s) { if (len[s] < 1) return TSFX_E_INVALID; Lmax = std::max(Lmax, len[s]); }
    const RollSpec R = roll_spec(rolling_direction, max_timeshift, min_timeshift, Lmax);
    int64_t k = 0;
    for (int64_t s = 0; s < n_series; ++s) {
        const int32_t L = len[s];
        int32_t t0;
        const int64_t n = roll_kept(R, L, &t0);
        for (int64_t j = 0; j < n; ++j) {
            const int32_t t = (int32_t)(t0 + j * R.amount);
            int32_t lo;
            const int32_t wl = roll_window(R, L, t, &lo);
            if (win_begin) {
                if (k >= capacity) return TSFX_E_INVALID;
                win_begin[k] = begin[s] + lo;
                win_len[k] = wl;
                if (win_parent) win_parent[k] = s;
                if (win_end_index) win_end_index[k] = t - 1;
            }
            ++k;
        }
    }
    return k;
}
