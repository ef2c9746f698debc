// k_peaks.cu -- kernel group PEAKS: number_cwt_peaks (feature_calculators.py:1320-1339; scipy.signal.find_peaks_cwt with
// _ricker :1307).  Both kernels read the Ricker taps from a per-context table (launch_fill_ricker).
//
// One warp per series.  k_peaks_small (series <= 256 samples, register-blocked CWT): row0 (float64), float32 copies of the
// wider rows, the maxima bits and a skewed float32 copy of the series that the packed ridge-line records and int16
// column map reuse after the CWT (8.3 KB per warp at 256 samples and n = 5, all in shared memory, 24 warps per SM).
// k_peaks (longer series): row0[npad], tmp[npad] (cwt rows, float64), noise[npad], float32 copies of the wider rows, a
// zero-padded float64 copy of the series in the working region; the ridge-line tables (5 int16 + 3 int32 per line), the
// column map and the local-maximum bit masks in shared memory.
#include <algorithm>

#include "tsfx_common.cuh"
#include "tsfx_kernels.h"

namespace tsfx {

#define TSFX_MAXW_PTS 160

struct PeaksLayout {
    int hot_bytes, hot_lines, hot_map, hot_bits;     // k_peaks from the global working region: the small, latency-critical
                                                     // tables (ridge lines, column map, maxima bits) stay in shared memory
    int npad, nwords, nxd;
    int off_rowsf, off_noise, off_bits, off_lines, off_map, off_xs, off_xd;   // byte offsets
};

// ---------------------------------------------------------------------------- find_peaks_cwt pieces
// _ricker(points, a) (:1307-1316) depends on tap v only through vec = v - (points - 1) / 2, and on vec only through
// vec^2, so one table row per width holds every tap of every points <= 10 w <= TSFX_RICKER_K: entry |2 vec|.  Filled
// once per context on the device with scipy's expression (a host fill could round exp differently).
__global__ void k_fill_ricker(double* tab) {
    const int w = blockIdx.x + 1, k = threadIdx.x;
    const double a = (double)w;
    const double A = 2.0 / (sqrt(3.0 * a) * pow(3.14159265358979323846, 0.25));
    const double wsq = a * a;
    const double vec = 0.5 * (double)k;          // exact, as v - (points - 1) / 2 is
    const double xsq = vec * vec;
    const double mod = 1.0 - xsq / wsq;
    const double gauss = exp(-xsq / (2.0 * wsq));
    tab[(size_t)(w - 1) * TSFX_RICKER_K + k] = A * mod * gauss;
}
cudaError_t launch_fill_ricker(double* tab, cudaStream_t st) {
    k_fill_ricker<<<TSFX_RICKER_W, TSFX_RICKER_K, 0, st>>>(tab);
    return cudaGetLastError();
}

// k_peaks: cwt row of width w, dst[i] = sum_u h[u] x[i + c0 - u] as below, lane-interleaved (i = lane + 32 m).  xd is
// the series as float64 with TSFX_MAXW_PTS zeros in front and zeros up to a whole 256-sample chunk (+ the same margin)
// behind, so no tap needs a bounds test.  One broadcast load of the tap serves 8 outputs.  (From the global working
// region the register-blocked form below measured slower: PEAKS 277 against 265 ms at 1 M x 1024 on an H100 SXM
// with a 400 W power limit.)
__device__ __forceinline__ void cwt_row(const double* xd, int n, const double* __restrict__ taps, int npts, double* dst, int lane) {
    const int c0 = (npts - 1) / 2;
    for (int i0 = 0; i0 < n; i0 += 256) {
        double acc[8];
#pragma unroll
        for (int m = 0; m < 8; ++m) acc[m] = 0.0;
        const double* xb = xd + TSFX_MAXW_PTS + i0 + lane + c0;
        for (int u = 0; u < npts; ++u) {
            const double h = __ldg(taps + abs(2 * u - (npts - 1)));
#pragma unroll
            for (int m = 0; m < 8; ++m) acc[m] = fma(xb[32 * m - u], h, acc[m]);
        }
#pragma unroll
        for (int m = 0; m < 8; ++m) {
            const int i = i0 + lane + 32 * m;
            if (i < n) dst[i] = acc[m];
        }
    }
}

// k_peaks_small: CWT row of width w, register-blocked: the lane forms the 8 consecutive outputs i0 .. i0+7 of
//   convolve(x, ricker(npts, w), mode="same")[i] = sum_u h[u] x[i + c0 - u],  c0 = (npts - 1) / 2,
// each one fma-accumulated over u = 0 .. npts-1 from 0.0.  The 8 outputs' inputs slide down by one sample per tap, so a
// window of 8 samples in registers costs one load per tap (and one tap load per 8 fma).  x(t) is sample t as float64,
// zero outside 0 .. n-1; it is called for t = i0 + c0 - (npts - 1) .. i0 + 7 + c0.  taps = the width's table row.
template <typename X>
__device__ __forceinline__ void cwt_run8(X x, int i0, int npts, const double* __restrict__ taps, double (&acc)[8]) {
    const int c0 = (npts - 1) / 2, base = i0 + c0;
    double win[8];
#pragma unroll
    for (int m = 0; m < 8; ++m) acc[m] = 0.0;
#pragma unroll
    for (int m = 1; m < 8; ++m) win[m - 1] = x(base + m);      // moved into place by the first tap
    win[7] = 0.0;
    auto tap = [&](int u) {
#pragma unroll
        for (int m = 7; m > 0; --m) win[m] = win[m - 1];
        win[0] = x(base - u);                                   // win[m] = x(i0 + m + c0 - u)
        const double h = __ldg(taps + abs(2 * u - (npts - 1)));
#pragma unroll
        for (int m = 0; m < 8; ++m) acc[m] = fma(win[m], h, acc[m]);
    };
    int u = 0;
    for (; u + 8 <= npts; u += 8) {
#pragma unroll
        for (int q = 0; q < 8; ++q) tap(u + q);
    }
    for (; u < npts; ++u) tap(u);
}

// scipy.stats.scoreatpercentile(win[0..wlen), 10): the order statistics i = floor(0.1 (wlen-1)) and i+1 are
// found by successive minima over (value, index) pairs -- no scratch, read-only window, O(wlen * (i+2)).
__device__ __forceinline__ double percentile10(const double* win, int wlen) {
    const double idx = 10.0 / 100.0 * (double)(wlen - 1);
    const int i = (int)idx;
    double pv = 0.0, v0 = 0.0, v1 = 0.0;
    int pi = -1;
    if (i <= 1) {                       // windows of up to 20 samples: the three smallest in one pass
        double m0 = dinf(), m1 = dinf(), m2 = dinf();
        for (int a = 0; a < wlen; ++a) {
            const double va = win[a];
            if (va < m0) { m2 = m1; m1 = m0; m0 = va; }
            else if (va < m1) { m2 = m1; m1 = va; }
            else if (va < m2) m2 = va;
        }
        v0 = i == 0 ? m0 : m1;
        v1 = i == 0 ? m1 : m2;
    } else
    for (int r = 0; r <= i + 1 && r < wlen; ++r) {
        double bv = 0.0;
        int bi = -1;
        for (int a = 0; a < wlen; ++a) {
            const double va = win[a];
            const bool after = (pi < 0) || (va > pv) || (va == pv && a > pi);
            if (after && (bi < 0 || va < bv)) { bv = va; bi = a; }
        }
        pv = bv; pi = bi;
        if (r == i) v0 = bv;
        if (r == i + 1) v1 = bv;
    }
    if ((double)i == idx) return v0;
    const double w0 = (double)(i + 1) - idx, w1 = idx - (double)i;
    return (v0 * w0 + v1 * w1) / (w0 + w1);
}

template <int WPC, bool GS>
__global__ void __launch_bounds__(WPC * 32) k_peaks(PeaksArgs A, PeaksLayout Y) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    unsigned char* base = warp_region<GS>(smem_raw, A.gscratch, A.bytes_per_warp, WPC, warp);
    double* row0 = reinterpret_cast<double*>(base);                       // npad : width-1 row (float64)
    double* tmp = row0 + Y.npad;                                           // npad : the row being formed
    double* noise = reinterpret_cast<double*>(base + Y.off_noise);         // npad : memoised noise floor (NaN = not yet)
    float* rowsf = reinterpret_cast<float*>(base + Y.off_rowsf);           // (cwt_n - 1) x npad : wider rows, float32 copies
    // ridge-line bookkeeping is a chain of dependent small-table lookups: from the global region every one of them is
    // an L2 round trip (the hottest stalls of the kernel), so these tables get their own shared-memory slice
    unsigned char* hot = (GS && Y.hot_bytes > 0) ? smem_raw + (size_t)warp * Y.hot_bytes : nullptr;
    unsigned* maxbits = hot ? reinterpret_cast<unsigned*>(hot + Y.hot_bits) : reinterpret_cast<unsigned*>(base + Y.off_bits);
    short* lines = hot ? reinterpret_cast<short*>(hot + Y.hot_lines) : reinterpret_cast<short*>(base + Y.off_lines);
    int* colmap = hot ? reinterpret_cast<int*>(hot + Y.hot_map) : reinterpret_cast<int*>(base + Y.off_map);
    float* xs = reinterpret_cast<float*>(base + Y.off_xs);
    double* xd = reinterpret_cast<double*>(base + Y.off_xd);               // zero-padded float64 copy for the convolutions
    const int64_t warps_total = (int64_t)gridDim.x * WPC;
    const int LCAP = Y.npad + Y.npad / 2 + 32;   // alive (<= maxima of the two previous rows <= n) + new in this row (<= n/2)

    for (int64_t s = (int64_t)blockIdx.x * WPC + warp; s < A.R.n_series; s += warps_total) {
        const int n = load_series(A.R, s, xs, lane);
        double* orow = A.out + (size_t)s * A.ncols;
        bool cwt_ready = false;

        int j = 0;
        while (j < A.nd) {
            const Desc d0 = A.descs[j];
            if (d0.calc == TSFX_NUMBER_CWT_PEAKS) {
                if (!cwt_ready) {
                    for (int p = lane; p < Y.nxd; p += 32) {
                        const int t = p - TSFX_MAXW_PTS;
                        xd[p] = (t >= 0 && t < n) ? (double)xs[t] : 0.0;
                    }
                    __syncwarp();
                    // all rows 1..cwt_n once (kept in shared memory) + local-maximum bit masks per row
                    for (int w = 1; w <= A.cwt_n; ++w) {
                        const int npts = min(10 * w, n);
                        double* dst = (w == 1) ? row0 : tmp;
                        cwt_row(xd, n, A.ricker + (size_t)(w - 1) * TSFX_RICKER_K, npts, dst, lane);
                        __syncwarp();
                        unsigned* bits = maxbits + (size_t)(w - 1) * Y.nwords;
                        for (int b0 = 0; b0 < n; b0 += 32) {
                            int i = b0 + lane;
                            bool mx = false;
                            if (i < n) {
                                double v = dst[i];
                                double pl = dst[min(i + 1, n - 1)], mi = dst[max(i - 1, 0)];
                                mx = (v > pl) && (v > mi);
                                if (w > 1) rowsf[(size_t)(w - 2) * Y.npad + i] = (float)v;   // only read for the SNR test
                            }
                            unsigned word = __ballot_sync(FULL, mx);
                            if (lane == 0) bits[b0 >> 5] = word;
                        }
                        __syncwarp();
                    }
                    for (int c = lane; c < n; c += 32) noise[c] = dnan();
                    __syncwarp();
                    cwt_ready = true;
                }
                const int nrows = d0.i0;
                // ---- ridge lines (scipy _identify_ridge_lines + _filter_ridge_lines), warp-parallel ----
                // line table (list order = creation order, as in scipy's Python list)
                short* l_last = lines;                 // last attached column
                short* l_gap = lines + LCAP;
                short* l_len = lines + 2 * LCAP;
                short* l_minrow = lines + 3 * LCAP;    // smallest row so far
                short* l_mincol = lines + 4 * LCAP;    // first column attached at that row
                int* t_max = reinterpret_cast<int*>(lines + 5 * LCAP);   // per-row attachment summaries
                int* t_min = t_max + LCAP;
                int* t_cnt = t_min + LCAP;
                const int min_length = (nrows + 3) / 4;                       // ceil(nrows / 4)
                const unsigned lt = (1u << lane) - 1u;
                const int NONE = 0x7fffffff;
                int result = 0, nl = 0, start = -1;
                for (int r = nrows - 1; r >= 0 && start < 0; --r) {             // largest row with any maximum
                    const unsigned* bits = maxbits + (size_t)r * Y.nwords;
                    unsigned any = 0;
                    for (int wd = lane; wd * 32 < n; wd += 32) any |= bits[wd];
                    if (__any_sync(FULL, any != 0)) start = r;
                }
                if (start >= 0) {
                    const unsigned* bits = maxbits + (size_t)start * Y.nwords;
                    for (int b0 = 0; b0 < n; b0 += 32) {
                        const unsigned word = bits[b0 >> 5];
                        const int idx = nl + __popc(word & lt);
                        if (((word >> lane) & 1u) && idx < LCAP) {
                            const int c = b0 + lane;
                            l_last[idx] = (short)c; l_gap[idx] = 0; l_len[idx] = 1; l_minrow[idx] = (short)start; l_mincol[idx] = (short)c;
                        }
                        nl = min(nl + __popc(word), LCAP);
                    }
                }
                __syncwarp();
                // filter of _filter_ridge_lines for one finished line
                const int window = (n + 19) / 20, hf = window / 2, odd = window & 1;
                auto accept = [&](int len, int rr, int cc) -> bool {
                    if (len < min_length) return false;
                    double nz = noise[cc];
                    if (nz != nz) {                 // 10th percentile of row 0 around cc, formed on first use
                        const int ws = max(cc - hf, 0), we = min(cc + hf + odd, n);
                        nz = percentile10(row0 + ws, we - ws);
                        noise[cc] = nz;
                    }
                    const double val = (rr == 0) ? row0[cc] : (double)rowsf[(size_t)(rr - 1) * Y.npad + cc];
                    const double snr = fabs(val / nz);
                    return !(snr < 1.0);
                };
                for (int r = start - 1; r >= 0; --r) {
                    const unsigned* bits = maxbits + (size_t)r * Y.nwords;
                    const int maxd = (r + 1) / 4;                  // floor(widths[r] / 4); distances are integers
                    for (int c = lane; c < n; c += 32) colmap[c] = NONE;
                    for (int li = lane; li < nl; li += 32) { t_max[li] = -1; t_min[li] = NONE; t_cnt[li] = 0; l_gap[li] += 1; }
                    __syncwarp();
                    // snapshot: column -> first line (list order) whose last column is that column
                    for (int li = lane; li < nl; li += 32) atomicMin(&colmap[l_last[li]], li);
                    __syncwarp();
                    const int nl_snapshot = nl;
                    for (int b0 = 0; b0 < n; b0 += 32) {
                        const unsigned word = bits[b0 >> 5];
                        const bool mine = (word >> lane) & 1u;
                        const int c = b0 + lane;
                        int best = -1;
                        if (mine && nl_snapshot > 0) {
                            // np.argmin(|c - prev|): smallest distance, first in list order on ties; attach only
                            // when that distance is <= max_distances[row]
                            for (int dd = 0; dd <= maxd && best < 0; ++dd) {
                                const int a = (c - dd >= 0) ? colmap[c - dd] : NONE;
                                const int b = (dd > 0 && c + dd < n) ? colmap[c + dd] : NONE;
                                const int m = min(a, b);
                                if (m != NONE) best = m;
                            }
                        }
                        if (mine && best >= 0) { atomicMax(&t_max[best], c); atomicMin(&t_min[best], c); atomicAdd(&t_cnt[best], 1); }
                        const unsigned newm = __ballot_sync(FULL, mine && best < 0);
                        if (mine && best < 0) {
                            const int idx = nl + __popc(newm & lt);
                            if (idx < LCAP) { l_last[idx] = (short)c; l_gap[idx] = 0; l_len[idx] = 1; l_minrow[idx] = (short)r; l_mincol[idx] = (short)c; }
                        }
                        nl = min(nl + __popc(newm), LCAP);
                    }
                    __syncwarp();
                    for (int li = lane; li < nl_snapshot; li += 32) {
                        const int cnt = t_cnt[li];
                        if (cnt > 0) {      // points are appended in ascending column order within a row
                            l_last[li] = (short)t_max[li]; l_gap[li] = 0; l_len[li] = (short)(l_len[li] + cnt);
                            l_minrow[li] = (short)r; l_mincol[li] = (short)t_min[li];
                        }
                    }
                    __syncwarp();
                    // retire lines whose gap exceeds gap_thresh = ceil(widths[0]) = 1; survivors keep their order
                    int keep = 0;
                    for (int b0 = 0; b0 < nl; b0 += 32) {
                        const int li = b0 + lane;
                        const bool valid = li < nl;
                        short f_last = 0, f_gap = 0, f_len = 0, f_row = 0, f_col = 0;
                        if (valid) { f_last = l_last[li]; f_gap = l_gap[li]; f_len = l_len[li]; f_row = l_minrow[li]; f_col = l_mincol[li]; }
                        const bool retire = valid && f_gap > 1;
                        const bool ok = retire && accept(f_len, f_row, f_col);
                        result += __popc(__ballot_sync(FULL, ok));
                        const unsigned keepm = __ballot_sync(FULL, valid && !retire);
                        __syncwarp();
                        if (valid && !retire) {
                            const int dst = keep + __popc(keepm & lt);
                            l_last[dst] = f_last; l_gap[dst] = f_gap; l_len[dst] = f_len; l_minrow[dst] = f_row; l_mincol[dst] = f_col;
                        }
                        keep += __popc(keepm);
                        __syncwarp();
                    }
                    nl = keep;
                }
                for (int b0 = 0; b0 < nl; b0 += 32) {
                    const int li = b0 + lane;
                    const bool ok = li < nl && accept(l_len[li], l_minrow[li], l_mincol[li]);
                    result += __popc(__ballot_sync(FULL, ok));
                }
                if (lane == 0) orow[d0.col] = (double)result;
                __syncwarp();
                ++j;
            } else {
                if (lane == 0) orow[d0.col] = dnan();
                ++j;
            }
        }
        __syncwarp();
    }
}

// ---------------------------------------------------------------------------- k_peaks_small: series <= 256 samples
// One register-blocked pass per CWT row (32 lanes x 8 outputs), everything in shared memory:
//   row0     float64[npad]            width-1 row (noise floor and the SNR of lines ending in row 0)
//   rowsf    float32[(cwt_n-1) npad]  wider rows, read only for the SNR test (float32, as k_peaks)
//   bits     uint32[cwt_n][8]         local-maximum masks, one byte per lane
//   union    the series as float32, skewed (xz_at) with PK_XZ_FRONT zeros in front and zeros behind, while the rows
//            are formed; then the ridge lines (one packed uint32 per line, LCAP of them) and the int16 column map
// The noise floor is recomputed per accepted-length line instead of memoised: windows are <= 13 samples here.
#define PK_SMALL_LEN 256
#define PK_XZ_FRONT 80                  // widest tap reach behind an output: 160 taps, c0 = 79
#define PK_XZ_LOGICAL (PK_XZ_FRONT + PK_SMALL_LEN + 79)       // t = -80 .. 334
#define PK_XZ_FLOATS 428                // xz_at(PK_XZ_LOGICAL - 1) + 1, rounded up to 16 bytes
// A lane reads samples 8 apart; one unused float per 32 spreads a warp's 32 reads over distinct banks
__device__ __forceinline__ int xz_at(int p) { return p + (p >> 5); }

// line record: last column | first column of the latest row << 8 | latest row << 16 | gap << 20 | length << 24.  The
// length saturates at 255: it is only compared with min_length = ceil(n / 4) <= 4.
#define LN_REC(last, col, row, len) ((unsigned)(last) | ((unsigned)(col) << 8) | ((unsigned)(row) << 16) | ((unsigned)(len) << 24))
#define LN_LAST(r) ((int)((r) & 0xffu))
#define LN_COL(r) ((int)(((r) >> 8) & 0xffu))
#define LN_ROW(r) ((int)(((r) >> 16) & 0xfu))
#define LN_GAP(r) ((int)(((r) >> 20) & 0xfu))
#define LN_LEN(r) ((int)((r) >> 24))

template <int WPC>
__global__ void __launch_bounds__(WPC * 32, 24 / WPC) k_peaks_small(PeaksArgs A, PeaksLayout Y) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    unsigned char* base = smem_raw + (size_t)warp * A.bytes_per_warp;
    double* row0 = reinterpret_cast<double*>(base);
    float* rowsf = reinterpret_cast<float*>(base + Y.off_rowsf);
    unsigned* maxbits = reinterpret_cast<unsigned*>(base + Y.off_bits);
    float* xz = reinterpret_cast<float*>(base + Y.off_xs);                 // while the rows are formed
    unsigned* lines = reinterpret_cast<unsigned*>(base + Y.off_lines);     // afterwards, over the same bytes
    short* colmap = reinterpret_cast<short*>(base + Y.off_map);
    const int64_t warps_total = (int64_t)gridDim.x * WPC;
    const int LCAP = Y.npad + Y.npad / 2 + 32;   // alive (<= maxima of the two previous rows <= n) + new in this row (<= n/2)
    const unsigned lt = (1u << lane) - 1u;
    const int NONE = 0x7fff;
    auto xat = [&](int t) { return (double)xz[xz_at(t + PK_XZ_FRONT)]; };

    for (int64_t s = (int64_t)blockIdx.x * WPC + warp; s < A.R.n_series; s += warps_total) {
        int64_t b;
        int n;
        if (A.R.begin) { b = A.R.begin[s]; n = A.R.len[s]; } else { b = s * (int64_t)A.R.dense_len; n = A.R.dense_len; }
        // all rows 1..cwt_n first (every descriptor of the group is number_cwt_peaks)
        const float* src = A.R.values + b;
        for (int p = lane; p < PK_XZ_LOGICAL; p += 32) {
            const int t = p - PK_XZ_FRONT;
            xz[xz_at(p)] = (t >= 0 && t < n) ? __ldg(src + t) : 0.f;
        }
        __syncwarp();
        const int i0 = 8 * lane;
        for (int w = 1; w <= A.cwt_n; ++w) {
            double v[8];
            cwt_run8(xat, i0, min(10 * w, n), A.ricker + (size_t)(w - 1) * TSFX_RICKER_K, v);
            // strict local maxima, the ends excluded (scipy compares them with themselves)
            const double vl = __shfl_up_sync(FULL, v[7], 1), vr = __shfl_down_sync(FULL, v[0], 1);
            unsigned mb = 0;
#pragma unroll
            for (int m = 0; m < 8; ++m) {
                const double l = m > 0 ? v[m - 1] : vl, r = m < 7 ? v[m + 1] : vr;
                const int i = i0 + m;
                if (i >= 1 && i <= n - 2 && v[m] > l && v[m] > r) mb |= 1u << m;
            }
            reinterpret_cast<unsigned char*>(maxbits + (w - 1) * 8)[lane] = (unsigned char)mb;
            if (w == 1) {
                if (i0 + 8 <= n) {
#pragma unroll
                    for (int m = 0; m < 8; m += 2) *reinterpret_cast<double2*>(row0 + i0 + m) = make_double2(v[m], v[m + 1]);
                } else {
#pragma unroll
                    for (int m = 0; m < 8; ++m) if (i0 + m < n) row0[i0 + m] = v[m];
                }
            } else {
                float* rf = rowsf + (size_t)(w - 2) * Y.npad;
                if (i0 + 8 <= n) {
                    *reinterpret_cast<float4*>(rf + i0) = make_float4((float)v[0], (float)v[1], (float)v[2], (float)v[3]);
                    *reinterpret_cast<float4*>(rf + i0 + 4) = make_float4((float)v[4], (float)v[5], (float)v[6], (float)v[7]);
                } else {
#pragma unroll
                    for (int m = 0; m < 8; ++m) if (i0 + m < n) rf[i0 + m] = (float)v[m];
                }
            }
        }
        __syncwarp();                   // xz is dead from here on: its bytes hold the lines
        double* orow = A.out + (size_t)s * A.ncols;
        int j = 0;
        while (j < A.nd) {
            const Desc d0 = A.descs[j];
            if (d0.calc == TSFX_NUMBER_CWT_PEAKS) {
                const int nrows = d0.i0;
                // ---- ridge lines (scipy _identify_ridge_lines + _filter_ridge_lines), as k_peaks ----
                const int min_length = (nrows + 3) / 4;                       // ceil(nrows / 4)
                int result = 0, nl = 0, start = -1;
                for (int r = nrows - 1; r >= 0 && start < 0; --r) {             // largest row with any maximum
                    const unsigned* bits = maxbits + r * 8;
                    unsigned any = 0;
                    for (int wd = lane; wd * 32 < n; wd += 32) any |= bits[wd];
                    if (__any_sync(FULL, any != 0)) start = r;
                }
                if (start >= 0) {
                    const unsigned* bits = maxbits + start * 8;
                    for (int b0 = 0; b0 < n; b0 += 32) {
                        const unsigned word = bits[b0 >> 5];
                        const int idx = nl + __popc(word & lt);
                        if (((word >> lane) & 1u) && idx < LCAP) lines[idx] = LN_REC(b0 + lane, b0 + lane, start, 1);
                        nl = min(nl + __popc(word), LCAP);
                    }
                }
                __syncwarp();
                const int window = (n + 19) / 20, hf = window / 2, odd = window & 1;
                auto accept = [&](unsigned rec) -> bool {
                    if (LN_LEN(rec) < min_length) return false;
                    const int rr = LN_ROW(rec), cc = LN_COL(rec);
                    const int ws = max(cc - hf, 0), we = min(cc + hf + odd, n);
                    const double nz = percentile10(row0 + ws, we - ws);
                    const double val = (rr == 0) ? row0[cc] : (double)rowsf[(size_t)(rr - 1) * Y.npad + cc];
                    const double snr = fabs(val / nz);
                    return !(snr < 1.0);
                };
                for (int r = start - 1; r >= 0; --r) {
                    const unsigned* bits = maxbits + r * 8;
                    const int maxd = (r + 1) / 4;                  // floor(widths[r] / 4); distances are integers
                    for (int c = lane; c < n; c += 32) colmap[c] = (short)NONE;
                    for (int li = lane; li < nl; li += 32) lines[li] += 1u << 20;      // gap + 1
                    __syncwarp();
                    // snapshot: column -> first line (list order) whose last column is that column.  Chunks from the
                    // back, the lowest lane of equal columns stores: the smallest line index is written last
                    for (int b0 = (nl - 1) & ~31; b0 >= 0; b0 -= 32) {
                        const int li = b0 + lane;
                        const int key = li < nl ? LN_LAST(lines[li]) : -1;
                        const unsigned grp = __match_any_sync(FULL, key);
                        if (key >= 0 && (grp & lt) == 0) colmap[key] = (short)li;
                        __syncwarp();
                    }
                    const int nl_snapshot = nl;
                    for (int b0 = 0; b0 < n; b0 += 32) {
                        const unsigned word = bits[b0 >> 5];
                        const bool mine = (word >> lane) & 1u;
                        const int c = b0 + lane;
                        int best = -1;
                        if (mine && nl_snapshot > 0) {
                            // np.argmin(|c - prev|): smallest distance, first in list order on ties; attach only
                            // when that distance is <= max_distances[row]
                            for (int dd = 0; dd <= maxd && best < 0; ++dd) {
                                const int a = (c - dd >= 0) ? colmap[c - dd] : NONE;
                                const int bb = (dd > 0 && c + dd < n) ? colmap[c + dd] : NONE;
                                const int m = min(a, bb);
                                if (m != NONE) best = m;
                            }
                        }
                        // columns of this chunk that attach to one line: the lowest lane updates the record (columns
                        // ascend, so the first attachment of the row sets the row's first column, the last one `last`)
                        const unsigned grp = __match_any_sync(FULL, best);
                        if (best >= 0 && (grp & lt) == 0) {
                            const unsigned rec = lines[best];
                            const int col = LN_GAP(rec) != 0 ? c : LN_COL(rec);       // gap 0: attached earlier in this row
                            lines[best] = LN_REC(b0 + 31 - __clz(grp), col, r, min(LN_LEN(rec) + __popc(grp), 255));
                        }
                        const unsigned newm = __ballot_sync(FULL, mine && best < 0);
                        if (mine && best < 0) {
                            const int idx = nl + __popc(newm & lt);
                            if (idx < LCAP) lines[idx] = LN_REC(c, c, r, 1);
                        }
                        nl = min(nl + __popc(newm), LCAP);
                        __syncwarp();
                    }
                    // retire lines whose gap exceeds gap_thresh = ceil(widths[0]) = 1; survivors keep their order
                    int keep = 0;
                    for (int b0 = 0; b0 < nl; b0 += 32) {
                        const int li = b0 + lane;
                        const bool valid = li < nl;
                        const unsigned rec = valid ? lines[li] : 0u;
                        const bool retire = valid && LN_GAP(rec) > 1;
                        const bool ok = retire && accept(rec);
                        result += __popc(__ballot_sync(FULL, ok));
                        const unsigned keepm = __ballot_sync(FULL, valid && !retire);
                        __syncwarp();
                        if (valid && !retire) lines[keep + __popc(keepm & lt)] = rec;
                        keep += __popc(keepm);
                        __syncwarp();
                    }
                    nl = keep;
                }
                for (int b0 = 0; b0 < nl; b0 += 32) {
                    const int li = b0 + lane;
                    const bool ok = li < nl && accept(lines[li]);
                    result += __popc(__ballot_sync(FULL, ok));
                }
                if (lane == 0) orow[d0.col] = (double)result;
                __syncwarp();
                ++j;
            } else {
                if (lane == 0) orow[d0.col] = dnan();
                ++j;
            }
        }
        __syncwarp();
    }
}

cudaError_t launch_peaks(const PeaksArgs& A0, int max_len, cudaStream_t st, int sm_count, const char** variant) {
    PeaksArgs A = A0;
    A.npad = (max_len + 3) & ~3;
    if (max_len > 32000) return cudaErrorInvalidConfiguration;      // int16 line tables
    if (!A.ricker) return cudaErrorInvalidValue;
    PeaksLayout Y = {};
    Y.npad = A.npad;
    if (A.cwt_n < 1 || A.cwt_n > TSFX_RICKER_W) return cudaErrorInvalidValue;
    if (max_len <= PK_SMALL_LEN) {
        // k_peaks_small while its footprint keeps at least 16 warps per SM resident (at 256 samples: n <= 10)
        const size_t lcap = (size_t)A.npad + A.npad / 2 + 32;
        size_t o = (size_t)A.npad * 8;                                       // row0
        Y.off_rowsf = (int)o; o += (size_t)(A.cwt_n - 1) * A.npad * 4;
        Y.nwords = PK_SMALL_LEN / 32;
        Y.off_bits = (int)o;  o += (size_t)A.cwt_n * Y.nwords * 4;
        o = (o + 15) & ~(size_t)15;
        Y.off_xs = Y.off_lines = (int)o;
        Y.off_map = (int)(o + lcap * 4);
        o += std::max((size_t)PK_XZ_FLOATS * 4, lcap * 4 + (size_t)A.npad * 2);
        const size_t per = (o + 15) & ~(size_t)15;
        if (4 * (4 * per + 1024) <= 228 * 1024) {
            A.bytes_per_warp = (int)per;
            A.gscratch = nullptr;
            *variant = "peaks/small";
            return launch_fixed(k_peaks_small<4>, 4 * 32, 4, per * 4, (int64_t)sm_count * grid_waves(4096), A.R.n_series, st, A, Y);
        }
    }
    Y.nwords = (A.npad + 31) / 32 + 1;
    size_t off = 0;
    off += (size_t)2 * A.npad * 8;                          // row0 + tmp (float64)
    Y.off_noise = (int)off; off += (size_t)A.npad * 8;
    Y.off_bits = (int)off;  off += (size_t)A.cwt_n * Y.nwords * 4;
    off = (off + 3) & ~(size_t)3;
    Y.off_rowsf = (int)off; off += (size_t)std::max(A.cwt_n - 1, 0) * A.npad * 4;
    Y.off_lines = (int)off; off += (size_t)(A.npad + A.npad / 2 + 32) * (5 * 2 + 3 * 4);    // 5 int16 + 3 int32 tables of LCAP lines
    Y.off_map = (int)off;   off += (size_t)A.npad * 4;
    off = (off + 15) & ~(size_t)15;
    Y.off_xs = (int)off;    off += (size_t)A.npad * 4;
    off = (off + 15) & ~(size_t)15;
    Y.nxd = ((max_len + 255) / 256) * 256 + 2 * TSFX_MAXW_PTS;
    Y.off_xd = (int)off;    off += (size_t)Y.nxd * 8;
    size_t per = (off + 15) & ~(size_t)15;
    A.bytes_per_warp = (int)per;
    Geometry G;
    if (!plan_geometry(per, 72 * 1024, 8, A.R.n_series, sm_count, A.gscratch, A.gscratch_bytes, &G, 16 * 1024)) return cudaErrorInvalidConfiguration;
    A.gscratch = G.gscratch;
    if (G.gscratch) {
        // hybrid placement: bulk rows in the global (L2-resident) region, hot tables in shared memory when four CTAs
        // per SM still fit
        const size_t lines_b = (size_t)(A.npad + A.npad / 2 + 32) * (5 * 2 + 3 * 4);
        const size_t map_b = (size_t)A.npad * 4, bits_b = (size_t)A.cwt_n * Y.nwords * 4;
        size_t hot = ((lines_b + 15) & ~(size_t)15) + ((map_b + 15) & ~(size_t)15) + ((bits_b + 15) & ~(size_t)15);
        if (hot * G.wpc <= 54 * 1024) {
            Y.hot_lines = 0;
            Y.hot_map = (int)((lines_b + 15) & ~(size_t)15);
            Y.hot_bits = Y.hot_map + (int)((map_b + 15) & ~(size_t)15);
            Y.hot_bytes = (int)hot;
            G.smem = hot * G.wpc;
        }
    }
    auto launch = [&](auto g) { return launch_kernel(k_peaks<decltype(g)::wpc, decltype(g)::global>, G, st, A, Y); };
    if (Y.hot_bytes)         // global region with the hot tables in shared memory
        TSFX_LAUNCH_DECLARED(TSFX_GEOMS_PEAKS, "peaks/general/hybrid", G, variant, launch);
    TSFX_LAUNCH_DECLARED(TSFX_GEOMS_PEAKS, "peaks/general", G, variant, launch);
}

}  // namespace tsfx
