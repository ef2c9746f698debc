// k_la.cu -- kernel group LA: small dense least-squares problems per series.
//   ar_coefficient          (feature_calculators.py:1459-1507; statsmodels AutoReg(lags=k, trend="c") OLS)
//   augmented_dickey_fuller (feature_calculators.py:499-544; statsmodels adfuller(regression="c"),
//                            autolag AIC / BIC / None) -- restated in oracle/thirdparty.py
//
// One warp per series.  Normal equations are formed cooperatively (one Gram entry per lane, looping over
// the rows) on mean-centred regressors, then solved by lane 0 with a float64 Cholesky.  The nested ADF
// lag search needs ONE factorisation: with columns ordered [const, level, dlag1, dlag2, ...] the
// residual sum of squares of the model using the first q columns is y'y - sum_{i<q} z_i^2, z = L^-1 X'y.
// Calls whose series all have at most 256 samples run k_la_small instead (below).
#include <algorithm>

#include "tsfx_common.cuh"
#include "tsfx_kernels.h"
#include "tsfx_math.cuh"

namespace tsfx {

__host__ __device__ inline int adf_maxlag(int n) {
    // ceil(12 * (n/100)^(1/4)); sqrt(sqrt()) is correctly rounded, so the perfect-fourth-power lengths
    // (100, 1600, 8100, ...) land exactly on the integer like a correctly rounded pow() does
    int m = (int)ceil(12.0 * sqrt(sqrt((double)n / 100.0)));
    int cap = n / 2 - 2;
    return m < cap ? m : cap;
}

// Lag-product block of one sequence over the row window [t0, T):
//   P[i*ldp + j] = sum_t seq[t-i] * seq[t-j]   (0 <= j <= i <= M),   C[i] = sum_t seq[t-i],
//   and, when `lev` is given, Lv[i] = sum_t lev[t] * seq[t-i].
// Lane d forms the three full sums of lag distance d once; every other entry on that diagonal follows
// from the sliding-window identity S_d(i+1) = S_d(i) + seq[t0-i-1] seq[t0-i-1-d] - seq[T-1-i] seq[T-1-i-d],
// so the whole block costs O(M * rows + M^2) instead of O(M^2 * rows).  Requires t0 >= M.
__device__ __forceinline__ void lag_gram(const double* seq, const double* lev, int t0, int T, int M, double* P, int ldp,
                                         double* C, double* Lv, int lane) {
    for (int d = lane; d <= M; d += 32) {
        double s = 0.0, c = 0.0, l = 0.0;
        for (int t = t0; t < T; ++t) {
            const double v = seq[t - d];
            s = fma(seq[t], v, s);
            c += v;
            if (lev) l = fma(lev[t], v, l);
        }
        C[d] = c;
        if (lev) Lv[d] = l;
        P[d * ldp + 0] = s;                          // (i, j) = (d, 0)
        for (int i = 0; i + 1 + d <= M; ++i) {       // slide the window one step back in time
            s += seq[t0 - i - 1] * seq[t0 - i - 1 - d] - seq[T - 1 - i] * seq[T - 1 - i - d];
            P[(i + 1 + d) * ldp + (i + 1)] = s;
        }
    }
    __syncwarp();
}

// ---- warp-cooperative dense SPD kernels (row-major lower triangle in shared memory) -----------------
// In-place Cholesky; returns the number of columns factorised before a non-positive pivot (q if none).
__device__ __forceinline__ int warp_cholesky(double* G, int q, int lda, int lane) {
    for (int j = 0; j < q; ++j) {
        double s = 0.0;
        for (int k = lane; k < j; k += 32) { double v = G[j * lda + k]; s = fma(v, v, s); }
        double d = G[j * lda + j] - wsum(s);
        if (!(d > 0.0)) return j;
        d = sqrt(d);
        __syncwarp();
        if (lane == 0) G[j * lda + j] = d;
        for (int i = j + 1 + lane; i < q; i += 32) {
            double t = G[i * lda + j];
            for (int k = 0; k < j; ++k) t = fma(-G[i * lda + k], G[j * lda + k], t);
            G[i * lda + j] = t / d;
        }
        __syncwarp();
    }
    return q;
}
// L z = b in place (column oriented: after z_k is known every lane retires it from its own row)
__device__ __forceinline__ void warp_forward(const double* L, int q, int lda, double* b, int lane) {
    for (int k = 0; k < q; ++k) {
        double zk = b[k] / L[k * lda + k];
        __syncwarp();
        if (lane == 0) b[k] = zk;
        for (int i = k + 1 + lane; i < q; i += 32) b[i] = fma(-L[i * lda + k], zk, b[i]);
        __syncwarp();
    }
}
// L^T x = z in place
__device__ __forceinline__ void warp_backward(const double* L, int q, int lda, double* b, int lane) {
    for (int i = q - 1; i >= 0; --i) {
        double xi = b[i] / L[i * lda + i];
        __syncwarp();
        if (lane == 0) b[i] = xi;
        for (int k = lane; k < i; k += 32) b[k] = fma(-L[i * lda + k], xi, b[k]);
        __syncwarp();
    }
}

template <int WPC, bool GS>
__global__ void __launch_bounds__(WPC * 32) k_la(LaArgs A, int pmax) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    unsigned char* base = warp_region<GS>(smem_raw, A.gscratch, A.bytes_per_warp, WPC, warp);
    double* xc = reinterpret_cast<double*>(base);          // npad : centred series (level)
    double* dx = xc + A.npad;                              // npad : first differences
    double* G = dx + A.npad;                               // pmax*pmax
    double* bvec = G + pmax * pmax;                        // pmax
    double* res = bvec + pmax;                             // 8 : staged results
    double* Pm = res + 8;                                  // pmax*pmax : lag-product block
    double* Cv = Pm + pmax * pmax;                         // pmax
    double* Lv = Cv + pmax;                                // pmax
    float* xs = reinterpret_cast<float*>(Lv + pmax);
    const int64_t warps_total = (int64_t)gridDim.x * WPC;

    for (int64_t s = (int64_t)blockIdx.x * WPC + warp; s < A.R.n_series; s += warps_total) {
        const int n = load_series(A.R, s, xs, lane);
        const Moments M = moments(xs, n, xc, lane);
        for (int i = lane; i + 1 < n; i += 32) dx[i] = (double)xs[i + 1] - (double)xs[i];
        __syncwarp();
        double* orow = A.out + (size_t)s * A.ncols;
        int ar_k = -1; bool ar_ok = false;
        int adf_mode = -1;

        for (int j = 0; j < A.nd; ++j) {
            const Desc d = A.descs[j];
            double r = dnan();
            if (d.calc == TSFX_AR_COEFFICIENT) {
                const int k = d.i1, p = d.i0;
                if (k != ar_k) {
                    ar_k = k;
                    const int rows = n - k;
                    ar_ok = (k < n) && (rows >= k + 1);
                    if (ar_ok) {
                        const int q = k + 1;
                        // columns: 0 const, j>=1: xc[t-j]; target xc[t]; rows t = k..n-1
                        lag_gram(xc, nullptr, k, n, k, Pm, pmax, Cv, nullptr, lane);
                        for (int e = lane; e < q * q; e += 32) {
                            const int a = e / q, c = e - a * q;
                            if (c > a) continue;
                            G[a * q + c] = (a == 0) ? (double)rows : (c == 0 ? Cv[a] : Pm[a * pmax + c]);
                        }
                        for (int a = lane; a < q; a += 32) bvec[a] = (a == 0) ? Cv[0] : Pm[a * pmax + 0];
                        __syncwarp();
                        int good = 0;
                        if (M.vmax == M.vmin) {
                            // rank-one design (constant series): numpy pinv's minimum-norm solution
                            double cst = M.vmin, sc = cst / (1.0 + (double)k * cst * cst);
                            for (int a = lane; a < q; a += 32) bvec[a] = (a == 0) ? sc : sc * cst;
                            good = 2;
                        } else if (warp_cholesky(G, q, q, lane) == q) {
                            warp_forward(G, q, q, bvec, lane);
                            warp_backward(G, q, q, bvec, lane);
                            // undo the centring: const = c~ + mean * (1 - sum phi)
                            double sphi = 0.0;
                            for (int a = 1 + lane; a < q; a += 32) sphi += bvec[a];
                            sphi = wsum(sphi);
                            if (lane == 0) bvec[0] = bvec[0] + M.mean * (1.0 - sphi);
                            good = 1;
                        }
                        __syncwarp();
                        if (!good) { ar_ok = true; for (int a = lane; a <= k; a += 32) bvec[a] = dnan(); __syncwarp(); }
                    }
                }
                if (p > k) r = dnan();
                else if (!ar_ok) r = (p < k) ? dnan() : 0.0;       // params = [nan]*k ; index k -> IndexError -> 0
                else r = bvec[p];
            } else if (d.calc == TSFX_AUGMENTED_DICKEY_FULLER) {
                if (adf_mode != d.i0) {
                    adf_mode = d.i0;
                    __syncwarp();
                    double stat = dnan(), pval = dnan(), ulag = dnan();
                    const int M0 = adf_maxlag(n);
                    if (M.vmax != M.vmin && M0 >= 0) {
                        const int nd_ = n - 1;
                        int used = M0;
                        if (adf_mode != TSFX_AUTOLAG_NONE) {
                            const int p = M0 + 2, t0 = M0, nobs = nd_ - M0;
                            double* yy = res + 7;
                            // columns [const, level, dlag1..dlagM]; y = dx[t] = "dlag0"
                            lag_gram(dx, xc, t0, nd_, M0, Pm, pmax, Cv, Lv, lane);
                            {
                                double l1 = 0.0, l2 = 0.0;
                                for (int t = t0 + lane; t < nd_; t += 32) { double v = xc[t]; l1 += v; l2 = fma(v, v, l2); }
                                l1 = wsum(l1); l2 = wsum(l2);
                                for (int e = lane; e < p * p; e += 32) {
                                    const int a = e / p, c = e - a * p;
                                    if (c > a) continue;
                                    double v;
                                    if (a == 0) v = (double)nobs;
                                    else if (a == 1) v = (c == 0) ? l1 : l2;
                                    else v = (c == 0) ? Cv[a - 1] : (c == 1 ? Lv[a - 1] : Pm[(a - 1) * pmax + (c - 1)]);
                                    G[a * p + c] = v;
                                }
                                for (int a = lane; a < p; a += 32) bvec[a] = (a == 0) ? Cv[0] : (a == 1 ? Lv[0] : Pm[(a - 1) * pmax + 0]);
                                if (lane == 0) *yy = Pm[0];
                                __syncwarp();
                            }
                            int best_q = 2;
                            {
                                // factorise as far as the pivots stay positive (the models are nested)
                                const int okq = warp_cholesky(G, p, p, lane);
                                double ssr = *yy;
                                double ssr_a = 0.0, ssr_b = 0.0;        // residual sum of squares of model q = lane+1 / lane+33
                                const double dnobs = (double)nobs;
                                for (int i = 0; i < okq; ++i) {
                                    double z = bvec[i] / G[i * p + i];
                                    __syncwarp();
                                    for (int r2 = i + 1 + lane; r2 < okq; r2 += 32) bvec[r2] = fma(-G[r2 * p + i], z, bvec[r2]);
                                    __syncwarp();
                                    ssr -= z * z;
                                    if ((i & 31) == lane) { if (i < 32) ssr_a = ssr; else ssr_b = ssr; }
                                }
                                // information criterion of every nested model, one model per lane (the logarithms are
                                // the expensive part), then the reference's first-minimum scan in model order
                                double ic_a = 0.0, ic_b = 0.0;
#pragma unroll
                                for (int c = 0; c < 2; ++c) {
                                    const int q = c * 32 + lane + 1;
                                    if (q >= 2 && q <= okq) {
                                        const double sq = c ? ssr_b : ssr_a;
                                        const double llf = -dnobs / 2.0 * log(2.0 * 3.14159265358979323846) -
                                                           dnobs / 2.0 * log(sq / dnobs) - dnobs / 2.0;
                                        const double pen = (adf_mode == TSFX_AUTOLAG_AIC) ? 2.0 * (double)q : log(dnobs) * (double)q;
                                        const double ic = -2.0 * llf + pen;
                                        if (c) ic_b = ic; else ic_a = ic;
                                    }
                                }
                                double best_ic = 0.0;
                                bool have = false;
                                for (int q = 2; q <= okq; ++q) {
                                    const double ic = __shfl_sync(FULL, (q > 32) ? ic_b : ic_a, (q - 1) & 31);
                                    if (!have || ic < best_ic) { have = true; best_ic = ic; best_q = q; }
                                }
                            }
                            best_q = __shfl_sync(FULL, best_q, 0);
                            used = best_q - 2;
                            __syncwarp();
                        }
                        // final regression on the longer sample, columns [const, dlag1..dlagU, level]
                        const int q = used + 2, t0 = used, nobs = nd_ - used;
                        double* yy = res + 7;
                        lag_gram(dx, xc, t0, nd_, used, Pm, pmax, Cv, Lv, lane);
                        {
                            double l1 = 0.0, l2 = 0.0;
                            for (int t = t0 + lane; t < nd_; t += 32) { double v = xc[t]; l1 += v; l2 = fma(v, v, l2); }
                            l1 = wsum(l1); l2 = wsum(l2);
                            for (int e = lane; e < q * q; e += 32) {
                                const int a = e / q, c = e - a * q;
                                if (c > a) continue;
                                double v;
                                if (a == 0) v = (double)nobs;
                                else if (a < q - 1) v = (c == 0) ? Cv[a] : Pm[a * pmax + c];
                                else v = (c == 0) ? l1 : (c == q - 1 ? l2 : Lv[c]);
                                G[a * q + c] = v;
                            }
                            for (int a = lane; a < q; a += 32) bvec[a] = (a == 0) ? Cv[0] : (a < q - 1 ? Pm[a * pmax + 0] : Lv[0]);
                            if (lane == 0) *yy = Pm[0];
                            __syncwarp();
                        }
                        if (warp_cholesky(G, q, q, lane) == q) {
                            warp_forward(G, q, q, bvec, lane);
                            double ssr = 0.0;
                            for (int i = lane; i < q; i += 32) ssr = fma(bvec[i], bvec[i], ssr);
                            ssr = *yy - wsum(ssr);
                            double s2 = ssr / (double)(nobs - q);
                            stat = bvec[q - 1] / sqrt(s2);
                            pval = m_mackinnon_p_c(stat);
                            ulag = (double)used;
                        }
                        __syncwarp();
                        if (lane == 0) { res[0] = stat; res[1] = pval; res[2] = ulag; }
                    } else if (lane == 0) { res[0] = stat; res[1] = pval; res[2] = ulag; }
                    __syncwarp();
                }
                r = (d.attr >= 0 && d.attr <= 2) ? res[d.attr] : dnan();
            }
            if (lane == 0) orow[d.col] = r;
        }
        __syncwarp();
    }
}

// ---------------------------------------------------------------------------- k_la_small: series <= 256 samples
// Only the series stays in shared memory, converted once to float64 (centred values and differences are recomputed
// from it), next to one Gram matrix being assembled.  Lag sums are formed with the lanes going over rows and combined by
// a warp reduce-scatter; the off-diagonal entries follow from lag_gram's sliding-window identity.  Every solve runs on
// the augmented Gram [X'X X'y; y'X y'y] held one row per lane in registers (chol_rows): its last row carries
// z = L^-1 X'y, so the SSR of every nested ADF model comes out of the factorisation, and the final ADF regression is the
// autolag Gram with its columns permuted to [const, dlag1..dlagU, level, y] plus the M0 - U rows the autolag sample
// left out, added as rank-one updates.  Results match k_la up to summation order.
#define LA_SMALL_LEN 256
#define LA_SMALL_KMAX 15      // largest AR order: lag sums S_0..S_15 in lanes 0-15 of the reduce-scatter, C_0 in lane 16
#define LA_SMALL_P 19         // largest augmented Gram: ADF autolag at 256 samples, [const, level, dlag1..dlag16, y]
#define LA_SMALL_LD 19        // odd row stride: the lanes' row loads fall in distinct banks
#define LA_SMALL_WPC 8
#define LA_SMALL_CB (LA_SMALL_P + 64)    // chol_rows' pivots and two column buffers

// 1 / sqrt(d) for a finite d > 0: the hardware approximation refined by two Newton steps (within an ulp or two).
// sqrt() and division would bring their slow-path subroutine calls, and with them register spills.
__device__ __forceinline__ double rsqrt_pos(double d) {
    double y;
    asm("rsqrt.approx.ftz.f64 %0, %1;" : "=d"(y) : "d"(d));
#pragma unroll
    for (int it = 0; it < 2; ++it) y = fma(0.5 * y, fma(-d * y, y, 1.0), y);
    return y;
}

// lane i receives the warp-wide sum of v[i]: five butterfly stages, each lane keeping the half its partner drops
// (one template per stage, so that every index into v is a compile-time constant and v stays in registers)
template <int O>
__device__ __forceinline__ void reduce_scatter_stage(double (&v)[32], int lane) {
    const bool up = lane & O;
#pragma unroll
    for (int i = 0; i < O; ++i) {
        const double lo = v[i], hi = v[i + O];
        const double send = up ? lo : hi;
        const double keep = up ? hi : lo;
        v[i] = keep + __shfl_xor_sync(FULL, send, O);
    }
    if constexpr (O > 1) reduce_scatter_stage<O / 2>(v, lane);
}
__device__ __forceinline__ double reduce_scatter32(double (&v)[32], int lane) {
    reduce_scatter_stage<16>(v, lane);
    return v[0];
}

// g[i] for a warp-uniform runtime index (register arrays are indexed at compile time only)
__device__ __forceinline__ double pick(const double (&g)[LA_SMALL_P], int i) {
    double r = 0.0;
#pragma unroll
    for (int c = 0; c < LA_SMALL_P; ++c)
        if (c == i) r = g[c];
    return r;
}

// Right-looking Cholesky of a symmetric matrix of order na held one full row per lane (lane i: g[c] = G[i][c]; lanes
// >= na hold zeros).  Factorises columns 0 .. nf-1 (nf < na) while the pivots stay positive; returns how many it did.
// Lane i < (returned count) then holds L[i][c] for c < i, L[i][i], L[c][i] for c > i (its column of L, so that the
// back-substitution needs no transpose) and inv = 1 / L[i][i]; the rows past it hold L[i][c] for the factorised c and
// their Schur complement after it.  With y as the last column, row na-1 carries z = L^-1 X'y and ends in y'y - z'z.
// Pivots and columns of L are broadcast through shared memory (cb: LA_SMALL_P pivots, then two 32-entry column
// buffers used in turn, so that one __syncwarp per hand-off suffices); under the descriptor branches every shuffle
// would be wrapped in a convergence sequence.
__device__ __forceinline__ int chol_rows(double (&g)[LA_SMALL_P], int na, int nf, double& inv, double* cb, int lane) {
    double* piv = cb;
    int done = nf;
    if (lane == 0) piv[0] = g[0];
#pragma unroll
    for (int j = 0; j < LA_SMALL_P - 1; ++j) {
        if (j < done) {
            __syncwarp();
            const double d = piv[j];
            if (!(d > 0.0)) {
                done = j;
            } else {
                double* col = cb + LA_SMALL_P + 32 * (j & 1);
                const double rinv = rsqrt_pos(d), r = d * rinv;
                const double l = (lane == j) ? r : g[j] * rinv;
                if (lane == j) inv = rinv;
                if (lane >= j) g[j] = l;
                col[lane] = l;
                __syncwarp();
#pragma unroll
                for (int c = j + 1; c < LA_SMALL_P; ++c) {     // columns >= na: zero rows, zero entries of L
                    const double lc = col[c];
                    g[c] = (lane > j) ? fma(-l, lc, g[c]) : (lane == j ? lc : g[c]);
                }
                if (j + 1 < LA_SMALL_P && lane == j + 1) piv[j + 1] = g[j + 1];
            }
        }
    }
    __syncwarp();
    return done;
}

// lane < na: row `lane` of the Gram in shared memory, row and column indices mapped by col()
template <typename F>
__device__ __forceinline__ void load_rows(double (&g)[LA_SMALL_P], const double* Gs, int na, F col, int lane) {
    const double* row = Gs + (lane < na ? col(lane) : 0) * LA_SMALL_LD;
#pragma unroll
    for (int c = 0; c < LA_SMALL_P; ++c) g[c] = (c < na && lane < na) ? row[col(c)] : 0.0;
}

// Lane-over-rows sums of the AR fit: v[d] = sum_t xc[t] xc[t-d] for d < NL, v[16] = sum_t xc[t], rows t = k .. n-1.
// Lags k < d < NL are formed too (from a clamped index) and never read: a fixed lag count keeps the loop
// branch-free instead of being specialised for every k.
template <int NL>
__device__ __forceinline__ void ar_sums(double (&v)[32], const double* xs, int n, int k, double mean, int lane) {
#pragma unroll 1
    for (int t = k + lane; t < n; t += 32) {
        const double w = xs[t] - mean;
        v[16] += w;
#pragma unroll
        for (int d = 0; d < NL; ++d) v[d] = fma(w, xs[max(t - d, 0)] - mean, v[d]);
    }
}

// AR(k) Gram over rows t = k .. n-1, columns [const, xc[t-1] .. xc[t-k], y = xc[t]]
__device__ __forceinline__ void ar_gram(const double* xs, int n, int k, double mean, double* Gs, int lane) {
    double v[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) v[i] = 0.0;
    if (k <= 10) ar_sums<11>(v, xs, n, k, mean, lane);        // ComprehensiveFCParameters: k = 10
    else ar_sums<LA_SMALL_KMAX + 1>(v, xs, n, k, mean, lane);
    const double tot = reduce_scatter32(v, lane);       // lane d: S_d = sum xc[t] xc[t-d]; lane 16: C_0 = sum xc[t]
    const double c0 = __shfl_sync(FULL, tot, 16);
    __syncwarp();                                       // every lane is done reading the previous Gram
    const int q = k + 1;
    auto col = [&](int i) { return i == 0 ? q : i; };
    auto xc = [&](int i) { return xs[i] - mean; };
    if (lane <= k) {
        const int d = lane;
        double s = tot, c = c0;
        Gs[col(d) * LA_SMALL_LD + col(0)] = s;
        Gs[col(0) * LA_SMALL_LD + col(d)] = s;
        for (int m = 0; m + 1 + d <= k; ++m) {         // slide the window one step back in time
            s += xc(k - m - 1) * xc(k - m - 1 - d) - xc(n - 1 - m) * xc(n - 1 - m - d);
            Gs[col(m + 1 + d) * LA_SMALL_LD + col(m + 1)] = s;
            Gs[col(m + 1) * LA_SMALL_LD + col(m + 1 + d)] = s;
        }
        for (int m = 0; m < d; ++m) c += xc(k - 1 - m) - xc(n - 1 - m);   // C_d = sum_t xc[t-d], slid the same way
        Gs[col(d)] = c;
        Gs[col(d) * LA_SMALL_LD] = c;
    }
    if (lane == 0) Gs[0] = (double)(n - k);
    __syncwarp();
}

// ADF autolag Gram over rows t = M0 .. n-2, columns [const, level xc[t], dlag1..dlagM0, y = dx[t]]
__device__ __forceinline__ void adf_gram(const double* xs, int n, int M0, double mean, double* Gs, int lane) {
    const int nd = n - 1, t0 = M0, p = M0 + 2;
    auto xd = [&](int i) { return xs[i]; };
    auto dx = [&](int i) { return xd(i + 1) - xd(i); };
    auto col = [&](int i) { return i == 0 ? p : i + 1; };
    // pass 1: S_d = sum dx[t] dx[t-d] (lane d), l1 = sum xc[t] (lane 17), l2 = sum xc[t]^2 (lane 18)
    // pass 2: Lv_d = sum xc[t] dx[t-d] (lane d)          (two passes keep the accumulators within the register budget)
    double sums[2];
#pragma unroll
    for (int pass = 0; pass < 2; ++pass) {
        double v[32];
#pragma unroll
        for (int i = 0; i < 32; ++i) v[i] = 0.0;
#pragma unroll 1
        for (int t = t0 + lane; t < nd; t += 32) {
            double hi = xd(t + 1), lo = xd(t);
            const double y = hi - lo, lev = lo - mean;
            const double w = pass ? lev : y;
            if (!pass) { v[17] += lev; v[18] = fma(lev, lev, v[18]); }
#pragma unroll
            for (int d = 0; d <= 16; ++d) {               // lags past M0 (clamped index) are never read
                if (d > 0) { hi = lo; lo = xd(max(t - d, 0)); }
                v[d] = fma(w, hi - lo, v[d]);              // w * dx[t-d]
            }
        }
        sums[pass] = reduce_scatter32(v, lane);
    }
    const double tot = sums[0], lv = sums[1];
    const double l1 = __shfl_sync(FULL, tot, 17), l2 = __shfl_sync(FULL, tot, 18);
    __syncwarp();                                       // every lane is done reading the previous Gram
    if (lane <= M0) {
        const int d = lane;
        double s = tot;
        Gs[col(d) * LA_SMALL_LD + col(0)] = s;
        Gs[col(0) * LA_SMALL_LD + col(d)] = s;
        for (int m = 0; m + 1 + d <= M0; ++m) {
            s += dx(t0 - m - 1) * dx(t0 - m - 1 - d) - dx(nd - 1 - m) * dx(nd - 1 - m - d);
            Gs[col(m + 1 + d) * LA_SMALL_LD + col(m + 1)] = s;
            Gs[col(m + 1) * LA_SMALL_LD + col(m + 1 + d)] = s;
        }
        const double c = xd(nd - d) - xd(t0 - d);      // sum_t dx[t-d] telescopes
        Gs[col(d)] = c;
        Gs[col(d) * LA_SMALL_LD] = c;
        Gs[LA_SMALL_LD + col(d)] = lv;
        Gs[col(d) * LA_SMALL_LD + 1] = lv;
    }
    if (lane == 0) {
        Gs[0] = (double)(nd - M0);
        Gs[1] = Gs[LA_SMALL_LD] = l1;
        Gs[LA_SMALL_LD + 1] = l2;
    }
    __syncwarp();
}

template <int WPC, int MINB>
__global__ void __launch_bounds__(WPC * 32, MINB) k_la_small(LaArgs A) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    unsigned char* base = smem_raw + (size_t)warp * A.bytes_per_warp;
    double* xs = reinterpret_cast<double*>(base);                         // LA_SMALL_LEN : the series, as float64
    double* Gs = xs + LA_SMALL_LEN;                                       // LA_SMALL_P x LA_SMALL_LD : Gram
    double* cb = Gs + LA_SMALL_P * LA_SMALL_LD;                           // LA_SMALL_CB : broadcasts between the lanes
    double* arb = cb + LA_SMALL_CB;                    // 32 : AR coefficients 0..15, ADF teststat / pvalue / usedlag at 16..18

    for (int64_t s = (int64_t)blockIdx.x * WPC + warp; s < A.R.n_series; s += (int64_t)gridDim.x * WPC) {
        // staged as float32 over the Gram, converted once: float64 conversions issue at a quarter of the FP64 rate,
        // and the sweeps would otherwise convert every sample about 20 times
        float* stage = reinterpret_cast<float*>(Gs);
        const int n = load_series(A.R, s, stage, lane);
        const Moments M = moments(stage, n, nullptr, lane);
        for (int i = lane; i < n; i += 32) xs[i] = (double)stage[i];
        __syncwarp();
        const bool flat = M.vmax == M.vmin;
        int ar_k = -1; bool ar_ok = false;
        int adf_mode = -1; bool adf_gram_ok = false;  // Gs holds this series' ADF autolag Gram

        for (int j = 0; j < A.nd; ++j) {
            const Desc d = A.descs[j];
            double r = dnan();
            if (d.calc == TSFX_AR_COEFFICIENT) {
                const int k = d.i1, p = d.i0;
                if (k != ar_k) {
                    ar_k = k;
                    const int rows = n - k;
                    ar_ok = (k < n) && (rows >= k + 1);
                    if (ar_ok) {
                        const int q = k + 1;
                        if (flat) {
                            // rank-one design (constant series): numpy pinv's minimum-norm solution
                            const double cst = M.vmin, sc = cst / (1.0 + (double)k * cst * cst);
                            if (lane < q) arb[lane] = (lane == 0) ? sc : sc * cst;
                        } else {
                            ar_gram(xs, n, k, M.mean, Gs, lane);
                            adf_gram_ok = false;
                            double g[LA_SMALL_P], inv = 0.0;
                            load_rows(g, Gs, q + 1, [](int i) { return i; }, lane);
                            if (chol_rows(g, q + 1, q, inv, cb, lane) == q) {
                                // L^T beta = z, z_i = L[y][i] (lane i: column i of L holds it); lane i publishes beta_i
                                double b = pick(g, q);
#pragma unroll
                                for (int i = LA_SMALL_P - 2; i >= 0; --i) {
                                    if (i < q) {
                                        if (lane == i) arb[i] = b * inv;
                                        __syncwarp();
                                        if (lane < i) b = fma(-g[i], arb[i], b);
                                    }
                                }
                                // undo the centring: const = c~ + mean * (1 - sum phi)
                                if (lane == 0) {
                                    double sphi = 0.0;
                                    for (int a = 1; a < q; ++a) sphi += arb[a];
                                    arb[0] = arb[0] + M.mean * (1.0 - sphi);
                                }
                            } else if (lane < q) {
                                arb[lane] = dnan();
                            }
                        }
                        __syncwarp();
                    }
                }
                if (p > k) r = dnan();
                else if (!ar_ok) r = (p < k) ? dnan() : 0.0;       // params = [nan]*k ; index k -> IndexError -> 0
                else r = arb[p];
            } else if (d.calc == TSFX_AUGMENTED_DICKEY_FULLER) {
                if (adf_mode != d.i0) {
                    adf_mode = d.i0;
                    double stat = dnan(), pval = dnan(), ulag = dnan();
                    const int M0 = adf_maxlag(n);
                    if (!flat && M0 >= 0) {
                        const int nd_ = n - 1, p = M0 + 2;
                        if (!adf_gram_ok) { adf_gram(xs, n, M0, M.mean, Gs, lane); adf_gram_ok = true; }
                        int used = M0;
                        if (adf_mode != TSFX_AUTOLAG_NONE) {
                            double g[LA_SMALL_P], inv = 0.0;
                            load_rows(g, Gs, p + 1, [](int i) { return i; }, lane);
                            // factorise as far as the pivots stay positive (the models are nested); the SSR of the
                            // model with the first q columns is y'y - sum_{i<q} z_i^2, z_i = L[y][i]
                            const int okq = chol_rows(g, p + 1, p, inv, cb, lane);
                            if (lane == p) {
#pragma unroll
                                for (int c = 0; c < LA_SMALL_P - 1; ++c) cb[c] = g[c];
                            }
                            __syncwarp();
                            const double dnobs = (double)(nd_ - M0);
                            double ssr = Gs[p * LA_SMALL_LD + p], ssr_q = 0.0;   // lane q-1: SSR of model q
                            for (int i = 0; i < okq; ++i) {
                                const double z = cb[i];
                                ssr -= z * z;
                                if (lane == i) ssr_q = ssr;
                            }
                            // information criterion of every nested model, one model per lane, then the reference's
                            // first-minimum scan in model order
                            double ic = 0.0;
                            const int q = lane + 1;
                            if (q >= 2 && q <= okq) {
                                const double llf = -dnobs / 2.0 * log(2.0 * 3.14159265358979323846) -
                                                   dnobs / 2.0 * log(ssr_q / dnobs) - dnobs / 2.0;
                                const double pen = (adf_mode == TSFX_AUTOLAG_AIC) ? 2.0 * (double)q : log(dnobs) * (double)q;
                                ic = -2.0 * llf + pen;
                            }
                            __syncwarp();
                            cb[lane] = ic;
                            __syncwarp();
                            int best_q = 2;
                            double best_ic = 0.0;
                            bool have = false;
                            for (int qq = 2; qq <= okq; ++qq) {
                                const double icq = cb[qq - 1];
                                if (!have || icq < best_ic) { have = true; best_ic = icq; best_q = qq; }
                            }
                            __syncwarp();
                            used = best_q - 2;
                        }
                        // final regression on the longer sample [used, nd_): the autolag Gram's columns
                        // [const, dlag1..dlagU, level, y] plus the rows t = used .. M0-1 as rank-one updates
                        const int q = used + 2, na = q + 1;
                        auto fcol = [&](int f) { return f == 0 ? 0 : f <= used ? f + 1 : f == used + 1 ? 1 : p; };
                        double g[LA_SMALL_P], inv = 0.0;
                        load_rows(g, Gs, na, fcol, lane);
                        for (int t = used; t < M0; ++t) {
                            double v = 0.0;                     // lane f: entry of final column f on row t
                            if (lane == 0) v = 1.0;
                            else if (lane <= used) v = xs[t - lane + 1] - xs[t - lane];
                            else if (lane == used + 1) v = xs[t] - M.mean;
                            else if (lane == used + 2) v = xs[t + 1] - xs[t];
                            cb[lane] = v;
                            __syncwarp();
#pragma unroll
                            for (int c = 0; c < LA_SMALL_P; ++c)
                                if (c < na) g[c] = fma(v, cb[c], g[c]);
                            __syncwarp();
                        }
                        if (chol_rows(g, na, q, inv, cb, lane) == q) {
                            if (lane == q) { cb[0] = pick(g, q - 1); cb[1] = pick(g, q); }
                            __syncwarp();
                            const double z = cb[0], ssr = cb[1];                  // L[y][level], y'y - z'z
                            const double s2 = ssr / (double)(nd_ - used - q);
                            stat = z / sqrt(s2);
                            pval = m_mackinnon_p_c(stat);
                            ulag = (double)used;
                        }
                    }
                    __syncwarp();
                    if (lane == 0) { arb[16] = stat; arb[17] = pval; arb[18] = ulag; }
                    __syncwarp();
                }
                r = (d.attr >= 0 && d.attr <= 2) ? arb[16 + d.attr] : dnan();
            }
            if (lane == 0) A.out[(size_t)s * A.ncols + d.col] = r;
        }
        __syncwarp();
    }
}

cudaError_t launch_la(const LaArgs& A0, int max_len, cudaStream_t st, int sm_count, const char** variant) {
    LaArgs A = A0;
    if (max_len <= LA_SMALL_LEN && A.max_ar_k <= LA_SMALL_KMAX) {
        A.npad = LA_SMALL_LEN;
        A.bytes_per_warp = (LA_SMALL_LEN + LA_SMALL_P * LA_SMALL_LD + LA_SMALL_CB + 32) * 8;
        A.gscratch = nullptr;
        *variant = "la/small";
        return launch_fixed(k_la_small<LA_SMALL_WPC, 3>, LA_SMALL_WPC * 32, LA_SMALL_WPC, (size_t)A.bytes_per_warp * LA_SMALL_WPC,
                            (int64_t)sm_count * grid_waves(4096), A.R.n_series, st, A);
    }
    A.npad = (max_len + 3) & ~3;
    if (adf_maxlag(max_len) + 2 > 64) return cudaErrorInvalidConfiguration;     // autolag keeps one model per lane, two rounds
    int pmax = std::max(adf_maxlag(max_len) + 2, A.max_ar_k + 1);
    pmax = (pmax + 1) & ~1;
    size_t per = (size_t)A.npad * 16 + (size_t)pmax * pmax * 16 + (size_t)pmax * 24 + 64 + (size_t)A.npad * 4;
    per = (per + 15) & ~(size_t)15;
    A.bytes_per_warp = (int)per;
    Geometry G;
    if (!plan_geometry(per, 100 * 1024, 8, A.R.n_series, sm_count, A.gscratch, A.gscratch_bytes, &G)) return cudaErrorInvalidConfiguration;
    A.gscratch = G.gscratch;
    auto launch = [&](auto g) { return launch_kernel(k_la<decltype(g)::wpc, decltype(g)::global>, G, st, A, pmax); };
    TSFX_LAUNCH_DECLARED(TSFX_GEOMS_ALL, "la", G, variant, launch);
}

}  // namespace tsfx
