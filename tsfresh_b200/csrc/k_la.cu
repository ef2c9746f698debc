// k_la.cu -- kernel group LA: small dense least-squares problems per series.
//   ar_coefficient          (feature_calculators.py:1459-1507; statsmodels AutoReg(lags=k, trend="c") OLS)
//   augmented_dickey_fuller (feature_calculators.py:499-544; statsmodels adfuller(regression="c"),
//                            autolag AIC / BIC / None) -- restated in oracle/thirdparty.py
//
// One warp per series.  Normal equations are formed cooperatively (one Gram entry per lane, looping over
// the rows) on mean-centred regressors, then solved by lane 0 with a float64 Cholesky.  The nested ADF
// lag search needs ONE factorisation: with columns ordered [const, level, dlag1, dlag2, ...] the
// residual sum of squares of the model using the first q columns is y'y - sum_{i<q} z_i^2, z = L^-1 X'y.
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

cudaError_t launch_la(const LaArgs& A0, int max_len, cudaStream_t st, int sm_count, const char** variant) {
    static const char* const names[6] = TSFX_GEOM_NAMES("la");
    LaArgs A = A0;
    A.npad = (max_len + 3) & ~3;
    if (adf_maxlag(max_len) + 2 > 64) return cudaErrorInvalidConfiguration;     // autolag keeps one model per lane, two rounds
    int pmax = std::max(adf_maxlag(max_len) + 2, A.nscr + 1);   // nscr carries the plan's largest AR order k
    pmax = (pmax + 1) & ~1;
    size_t per = (size_t)A.npad * 16 + (size_t)pmax * pmax * 16 + (size_t)pmax * 24 + 64 + (size_t)A.npad * 4;
    per = (per + 15) & ~(size_t)15;
    A.bytes_per_warp = (int)per;
    Geometry G;
    if (!plan_geometry(per, 100 * 1024, 8, A.R.n_series, sm_count, A.gscratch, A.gscratch_bytes, &G)) return cudaErrorInvalidConfiguration;
    A.gscratch = G.gscratch;
    *variant = geom_variant(names, G);
    TSFX_DISPATCH(k_la, G, st, A, pmax)
    return cudaGetLastError();
}

}  // namespace tsfx
