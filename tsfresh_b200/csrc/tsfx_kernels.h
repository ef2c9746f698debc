// tsfx_kernels.h -- argument blocks and launchers of the kernel groups (internal to libtsfx.so).
#pragma once
#include <cuda_runtime.h>
#include <algorithm>
#include "tsfx_common.cuh"

#define TSFX_DEC_MIN (-46)
#define TSFX_DEC_MAX 39

namespace tsfx {

// CTAs per SM in a launch (each CTA loops over its share of the series).  TSFX_GRID_WAVES overrides the
// per-kernel default (tuning knob, read once).
int grid_waves(int dflt);
int global_above();
int global_ctas_env();

struct Geometry { int wpc; size_t smem; int grid; unsigned char* gscratch; };

// CTAs of a launch with `per_cta` series per CTA: one per per_cta series, at most `cap`
inline int cta_grid(int64_t n_series, int per_cta, int64_t cap) {
    const int64_t ctas = (n_series + per_cta - 1) / per_cta;
    return (int)(ctas < cap ? (ctas < 1 ? 1 : ctas) : cap);
}

// Chooses warps per CTA / grid for a warp-per-series kernel needing `per` bytes per warp.  Shared memory when it
// fits (budget = target bytes per CTA so several CTAs stay resident), else the global scratch buffer.  `cta_bytes` of
// shared memory in front of the per-warp regions are needed in either placement (k_basic's descriptor table): they
// count against the 227 KB of one CTA, and G->smem includes them.
inline bool plan_geometry(size_t per, size_t budget, int maxw, int64_t n_series, int sm_count, unsigned char* gs,
                          size_t gs_bytes, Geometry* G, size_t prefer_global_above = 227 * 1024,
                          int global_ctas = 0, size_t cta_bytes = 0) {
    // Working sets above `prefer_global_above` bytes per warp run from the global (L2-resident) region even though
    // they would fit in shared memory: shared memory would limit the latency-bound PEAKS / SEQ kernels to 2-4 warps per
    // SM -- measured on H100 SXM (700 W) at 250 000 x 1024, PEAKS 61 ms against 266 ms, SEQ 67 ms against 143 ms.
    // TSFX_GLOBAL_ABOVE=<bytes> lowers every kernel's threshold to at most that (it never raises one: the launchers
    // compile only the geometries their own thresholds can give).
    const size_t thr = global_above() > 0 ? std::min((size_t)global_above(), prefer_global_above) : prefer_global_above;
    if (per <= thr && per + cta_bytes <= 227 * 1024) {
        size_t w = budget / per;
        int wpc = w >= 8 ? 8 : w >= 4 ? 4 : w >= 2 ? 2 : 1;
        while (wpc > maxw) wpc >>= 1;
        G->wpc = wpc;
        G->smem = per * wpc + cta_bytes;
        G->grid = cta_grid(n_series, wpc, (int64_t)sm_count * grid_waves(4096));
        G->gscratch = nullptr;
        return true;
    }
    int wpc = maxw >= 4 ? 4 : 1;
    size_t max_ctas = gs ? gs_bytes / (per * wpc) : 0;
    if (max_ctas < 1) { wpc = 1; max_ctas = gs ? gs_bytes / per : 0; }
    if (max_ctas < 1) return false;
    // CTAs per SM in global-region mode: TSFX_GLOBAL_CTAS, else the kernel's own choice, else 4
    int64_t cap = (int64_t)sm_count * (global_ctas_env() > 0 ? global_ctas_env() : global_ctas > 0 ? global_ctas : 4);
    if ((int64_t)max_ctas < cap) cap = (int64_t)max_ctas;
    G->wpc = wpc;
    G->smem = cta_bytes;
    G->grid = cta_grid(n_series, wpc, cap);
    G->gscratch = gs;
    return true;
}

// kernel<<<grid, threads, smem, st>>>(args...), after raising the kernel's dynamic shared-memory limit to smem
template <class... P, class... Args>
cudaError_t launch_kernel(void (*kernel)(P...), int grid, int threads, size_t smem, cudaStream_t st, const Args&... args) {
    if (smem) {
        cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return e;
    }
    kernel<<<grid, threads, smem, st>>>(args...);
    return cudaGetLastError();
}
// a geometry from plan_geometry
template <class... P, class... Args>
cudaError_t launch_kernel(void (*kernel)(P...), const Geometry& G, cudaStream_t st, const Args&... args) {
    return launch_kernel(kernel, G.grid, G.wpc * 32, G.smem, st, args...);
}
// a fixed geometry: CTAs of `threads` threads serving `per_cta` series each, at most `cap` CTAs
template <class... P, class... Args>
cudaError_t launch_fixed(void (*kernel)(P...), int threads, int per_cta, size_t smem, int64_t cap, int64_t n_series,
                         cudaStream_t st, const Args&... args) {
    return launch_kernel(kernel, cta_grid(n_series, per_cta, cap), threads, smem, st, args...);
}

// The geometries a warp-per-series launcher can run, declared once per launcher as LIST(X, a) = X(a, warps per CTA,
// shared | global) ...  Only the listed instantiations are compiled (TSFX_LAUNCH_DECLARED), and with a group prefix the
// same list gives the variant names "<group>/w<warps per CTA>/<shared | global>" that tsfx_last_kernels reports and
// tsfx_kernel_variants lists.  Every global list keeps w1: the fallback when the working region holds fewer than four
// warps' working sets.
#define TSFX_GEOMS_ALL(X, a) X(a, 8, shared) X(a, 4, shared) X(a, 2, shared) X(a, 1, shared) X(a, 4, global) X(a, 1, global)
// BASIC: the 8-warp shared geometry runs as 12-warp CTAs (launch_basic)
#define TSFX_GEOMS_BASIC(X, a) X(a, 12, shared) X(a, 4, shared) X(a, 2, shared) X(a, 1, shared) X(a, 4, global) X(a, 1, global)
// ENTROPY tiles (at most 4 warps per CTA): the rank kernel takes every series whose tile working set fits four warps
#define TSFX_GEOMS_ENTROPY(X, a) X(a, 2, shared) X(a, 1, shared) X(a, 4, global) X(a, 1, global)
// general SEQ kernel: shared memory only up to 16 KB per warp, so its 72 KB budget always holds four warps
#define TSFX_GEOMS_SEQ(X, a) X(a, 8, shared) X(a, 4, shared) X(a, 4, global) X(a, 1, global)
// general PEAKS kernel: whenever it runs (k_peaks_small takes the short series), its working set exceeds the 16 KB per
// warp below which it would stay in shared memory
#define TSFX_GEOMS_PEAKS(X, a) X(a, 4, global) X(a, 1, global)

template <int W, bool GS> struct Geo { static constexpr int wpc = W; static constexpr bool global = GS; };
#define TSFX_GEOM_IS_shared false
#define TSFX_GEOM_IS_global true
#define TSFX_GEOM_NAME(grp, W, P) grp "/w" #W "/" #P,
#define TSFX_GEOM_CASE(grp, W, P)                                              \
    if (G__.wpc == W && (G__.gscratch != nullptr) == TSFX_GEOM_IS_##P) {       \
        *variant__ = grp "/w" #W "/" #P;                                       \
        return launch__(Geo<W, TSFX_GEOM_IS_##P>());                           \
    }
// Runs launch(Geo<W, GS>()) for the geometry G, which must be one of LIST, and reports its variant name.  Any other
// geometry fails with cudaErrorNotSupported and *variant naming it: a launcher never falls back to another geometry.
#define TSFX_LAUNCH_DECLARED(LIST, grp, G, variant, launch) \
    do {                                                    \
        const Geometry& G__ = (G);                          \
        const char** const variant__ = (variant);           \
        auto&& launch__ = (launch);                         \
        LIST(TSFX_GEOM_CASE, grp)                           \
        return undeclared_geometry(grp, G__, variant__);    \
    } while (0)
cudaError_t undeclared_geometry(const char* grp, const Geometry& G, const char** variant);

enum Group { G_BASIC = 0, G_SORTED, G_SPECTRAL, G_LA, G_ENTROPY, G_SEQ, G_PEAKS, G_COUNT };

// Longest series a call may hold (TSFX_E_TOO_LONG beyond), checked for every group of a plan before any is launched.
// ENTROPY's pair work is O(n^2) per series, so it keeps the old cap; SPECTRAL, LA, SEQ and PEAKS have layouts up to
// TSFX_L_MAX; BASIC (and its reduction-only kernel) and SORTED have no length limit of their own.  Calls whose longest
// series exceeds TSFX_SHORT_L_MAX select the long-series layouts (wide Lempel-Ziv keys, 32-bit ridge-line columns,
// Bluestein FFT).
#define TSFX_L_MAX 131072
#define TSFX_SHORT_L_MAX 21000
inline int group_max_len(int g) {
    return g == G_ENTROPY ? TSFX_SHORT_L_MAX : (g == G_BASIC || g == G_SORTED) ? 0x7fffffff : TSFX_L_MAX;
}
#define G_EVENTS (G_COUNT + 1)      // + the assemble pass

// Plan limits that follow from a layout (tsfx_plan_create refuses larger values with TSFX_E_UNSUPPORTED).
// lempel_ziv_complexity: symbols are 16-bit and the all-ones key marks an empty slot of the 32-bit key table.
// BASIC: the CTA-wide descriptor table (40 bytes per column) must fit one CTA's 227 KB next to 1 KB of static shared
// memory in every placement: 5 632 columns are 220 KB.
#define TSFX_LZ_MAX_BINS 65535
#define TSFX_BASIC_MAX_COLS 5632

// Result assembly: every kernel group writes its own dense [n_series x ncols_g] staging matrix (so each
// 32-byte sector is completed by the warp that owns the row, while it is still in L2); this pass
// scatters the staging rows into the final row-major [n_series x ncols] matrix in column order.
struct AssembleArgs {
    const double* stage;          // group g starts at stage + n_series * cum[g]
    double* out;
    int64_t n_series;
    int ncols;                    // columns of this plan
    int ld;                       // row stride of `out` (>= ncols: several kinds share one matrix, each its own column block)
    int n_groups;
    int cum[G_COUNT + 1];         // columns before group g (cum[n_groups] = total staged columns)
    const int32_t* final_col;     // device: final column of staged column (cum[g] + j)
    // multi-GPU result placement (tsfx_set_peer_outputs): the finished row is ALSO stored at the same offset of
    // every peer's mapped result matrix (plain P2P stores over NVLink), or -- when the result matrix has a multicast
    // mapping -- stored once through it (the NVSwitch replicates the store to every GPU, including this one)
    int n_extra;
    double* extra[7];
    double* out_mc;               // non-null: store through the multicast mapping instead of `out`
};
cudaError_t launch_assemble(const AssembleArgs& A, cudaStream_t st, int sm_count);

// What every warp-per-series group's arguments start with.  tsfx_plan_create fills one *Args per group from the plan;
// an extract call sets R, gscratch, gscratch_bytes and out, and the launcher the fields that depend on the longest series.
struct GroupArgs {
    SeriesRef R;
    unsigned char* gscratch;     // global working region -> set to nullptr by the launcher when shared memory is used
    size_t gscratch_bytes;
    const Desc* descs;           // device, this group's descriptors
    int nd;
    double* out;                 // this group's staging matrix
    int ncols;
};

struct BasicArgs : GroupArgs {
    int npad, nscr, nlag, bytes_per_warp;   // shared-memory carve-up (doubles / doubles / doubles / bytes)
    int lag_tiles;       // > 0: lag products by DMMA (mma.sync m8n8k4 f64) with this many 8 x 8 tiles; 0: FMA path
    int desc_bytes;      // CTA-wide copy of the descriptor table in front of the per-warp regions (set by the launcher)
    int nxc, nalt;       // doubles of the centred copy incl. its zero tail; distinct agg_linear_trend (f_agg, chunk_len) keys
    int nfin;            // the first nfin descriptors are O(1) "finishers" (see k_basic.cu)
    int lag_needed;      // largest lag product any descriptor reads (0 = none)
    int pacf_off;        // offset (doubles) of the pacf staging area inside lagS
    const double* dec;   // device table d*10^k, k = TSFX_DEC_MIN..TSFX_DEC_MAX, 9 per decade
    int lt_pcol;         // staging column of linear_trend's p-value (k_basic leaves the t statistic there and
                         // k_basic_pvalue finishes it, see k_basic.cu); -1: the plan has no such column
};
// vocab: the plan has a column basic_vocabulary (k_basic.cu) finishes: agg_autocorrelation with a reducer other than
// mean / median / var / std, or linregress attr intercept_stderr
cudaError_t launch_basic(const BasicArgs& A, bool vocab, int max_len, cudaStream_t st, int sm_count, const char** variant);
bool basic_finisher_calc(int calc);
bool sorted_finisher_calc(int calc);    // same for the SORTED group     // host: is this calculator evaluated by the lane-parallel finisher stage?

// reduction-only fast path of the BASIC group (k_moments.cu)
struct MomentsArgs {
    SeriesRef R;
    const Desc* descs;   // device, the BASIC group's descriptors (all moments_only_calc)
    int nd;
    double* out;         // staging matrix (colmap == nullptr: column = descriptor index) or the final matrix
    int ncols;           // row stride of `out`
    const int32_t* colmap;   // device: final column of descriptor j (direct write, no assemble pass), or nullptr
    int need_high;       // third / fourth centred moments are needed (skewness, kurtosis)
};
cudaError_t launch_moments(const MomentsArgs& A, cudaStream_t st, int sm_count, const char** variant);
bool moments_only_calc(int calc);       // host: can the reduction-only kernel evaluate this calculator?

struct SortedArgs : GroupArgs {
    int npad, npow2, nscr, bytes_per_warp;
    int nfin, ncq;       // leading O(1) descriptors (lane-parallel); distinct change_quantiles corridors
    const double2* cq;   // device: (ql, qh) of every distinct corridor, in descriptor order
};
// cq_own: some change_quantiles column's reducer is not mean / var / std (cq_own_passes, k_sorted.cu)
cudaError_t launch_sorted(const SortedArgs& A, bool cq_own, int max_len, cudaStream_t st, int sm_count, const char** variant);

struct SpectralArgs : GroupArgs {
    int npad, nspec, bytes_per_warp;
    const double2* twiddle;    // device: exp(-2 pi i k / tw_n), k = 0 .. tw_n/2
    int tw_n;                  // power of two >= largest power-of-two FFT length in use
    const double* tables;      // cwt tables (device)
    const int64_t* table_off;
    const int32_t* table_half;
    int need_fft, need_welch;
    int max_hist;
    int nfft;                  // the first nfft descriptors are fft_coefficient (lane-parallel stage)
};
cudaError_t launch_spectral(const SpectralArgs& A, int max_len, cudaStream_t st, int sm_count, const char** variant);

struct LaArgs : GroupArgs {
    int npad, max_ar_k, bytes_per_warp;    // max_ar_k: the plan's largest ar_coefficient order k
};
// tstat: some augmented_dickey_fuller column uses autolag "t-stat"
cudaError_t launch_la(const LaArgs& A, bool tstat, int max_len, cudaStream_t st, int sm_count, const char** variant);

struct EntropyArgs : GroupArgs {
    int xpad;                  // tile kernel: padded sample count
    int npad, bytes_per_warp;
};
cudaError_t launch_entropy(const EntropyArgs& A, int max_len, cudaStream_t st, int sm_count, const char** variant);

struct SeqArgs : GroupArgs {
    int npad, bytes_per_warp;
    int need_lz, need_perm;    // the plan has lempel_ziv_complexity / permutation_entropy columns
    int n_lz, max_lz_bins;     // lempel_ziv_complexity columns; their largest bin count
};
cudaError_t launch_seq(const SeqArgs& A, int max_len, cudaStream_t st, int sm_count, const char** variant);

struct PeaksArgs : GroupArgs {
    int npad, bytes_per_warp;
    int cwt_n;                 // largest n of the number_cwt_peaks columns: CWT rows 1..cwt_n
    const double* ricker;      // device Ricker tap table (launch_fill_ricker)
};
cudaError_t launch_peaks(const PeaksArgs& A, int max_len, cudaStream_t st, int sm_count, const char** variant);

// Ricker tap table of number_cwt_peaks: widths 1..TSFX_RICKER_W, entry (w - 1) * TSFX_RICKER_K + |2 v - (points - 1)|
// is tap v of ricker(points, w) for every points <= 10 w (filled once per context, on the device)
#define TSFX_RICKER_W 16
#define TSFX_RICKER_K 160
cudaError_t launch_fill_ricker(double* tab, cudaStream_t st);

// plain fill of a column set with NaN is done by BASIC (TSFX_CONST_NAN)

// twiddle table fill: tw[k] = exp(-2 pi i k / n), k = 0..n/2
cudaError_t launch_fill_twiddle(double2* tw, int n, cudaStream_t st);

}  // namespace tsfx
