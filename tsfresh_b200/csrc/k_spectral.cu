// k_spectral.cu -- kernel group SPECTRAL: fft_coefficient, fft_aggregated, spkt_welch_density,
// fourier_entropy, cwt_coefficients ("class FFT" / "class CONV" rows of SURVEY.md section 8a).
//
// One warp per series, float64 throughout.  The real FFT of a power-of-two length n is an in-place
// radix-2 complex FFT of length n/2 in shared memory followed by the real-split step; other lengths up to
// TSFX_SHORT_L_MAX use a direct DFT against a per-series twiddle table (exact index arithmetic, no accumulated rotation),
// longer ones Bluestein's chirp-z convolution over radix-2 FFTs of length M >= 2n - 1 (rfft_bluestein).
// Twiddles come from a device table filled once with sincospi().
#include <algorithm>

#include "tsfx_common.cuh"
#include "tsfx_kernels.h"
#include "tsfx_math.cuh"

namespace tsfx {

__device__ __forceinline__ double2 cmul(double2 a, double2 b) {
    return make_double2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x);
}

__global__ void k_fill_twiddle(double2* tw, int n) {
    int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k <= n / 2) {
        double s, c;
        sincospi(2.0 * (double)k / (double)n, &s, &c);
        tw[k] = make_double2(c, -s);
    }
}
cudaError_t launch_fill_twiddle(double2* tw, int n, cudaStream_t st) {
    int threads = 256, blocks = (n / 2 + 1 + threads - 1) / threads;
    k_fill_twiddle<<<blocks, threads, 0, st>>>(tw, n);
    return cudaGetLastError();
}

// Real FFT of m samples f(0..m-1) -> X[0..m/2] (double2) in shared memory.  m is a power of two >= 4.
template <typename F>
__device__ __forceinline__ void rfft_pow2(F f, int m, double2* X, const double2* tw, int tw_n, int lane) {
    const int h = m >> 1;
    int lg = 31 - __clz(h);
    // load z[j] = f(2j) + i f(2j+1) at the bit-reversed position
    for (int j = lane; j < h; j += 32) {
        int rj = (int)(__brev((unsigned)j) >> (32 - lg));
        if (lg == 0) rj = 0;
        X[rj] = make_double2(f(2 * j), f(2 * j + 1));
    }
    __syncwarp();
    for (int len = 2; len <= h; len <<= 1) {
        const int half = len >> 1;
        const int tstep = tw_n / len;
        for (int t = lane; t < (h >> 1); t += 32) {
            int j = t & (half - 1);
            int i = ((t - j) << 1) + j;
            int l = i + half;
            double2 w = tw[j * tstep];
            double2 u = X[i], v = cmul(X[l], w);
            X[i] = make_double2(u.x + v.x, u.y + v.y);
            X[l] = make_double2(u.x - v.x, u.y - v.y);
        }
        __syncwarp();
    }
    // real split: X[k] = (Z[k] + conj(Z[h-k]))/2 - i W_m^k (Z[k] - conj(Z[h-k]))/2
    const int sstep = tw_n / m;
    double2 z0 = X[0];
    __syncwarp();
    for (int k = 1 + lane; k <= (h >> 1); k += 32) {
        double2 a = X[k], b = X[h - k];
        double2 e = make_double2(0.5 * (a.x + b.x), 0.5 * (a.y - b.y));      // even part
        double2 o = make_double2(0.5 * (a.x - b.x), 0.5 * (a.y + b.y));      // (Z[k]-conj(Z[h-k]))/2
        double2 w = tw[k * sstep];
        double2 wo = cmul(w, o);                                              // W * o
        // -i * wo = (wo.y, -wo.x)
        double2 xk = make_double2(e.x + wo.y, e.y - wo.x);
        // mirrored bin h-k: even' = conj(e), odd' = -conj(o), W_m^{h-k} = -conj(W_m^k)
        double2 w2 = make_double2(-w.x, w.y);
        double2 o2 = make_double2(-o.x, o.y);
        double2 wo2 = cmul(w2, o2);
        double2 xh = make_double2(e.x + wo2.y, -e.y - wo2.x);
        X[k] = xk;
        if (k != h - k) X[h - k] = xh;
    }
    if (lane == 0) {
        X[0] = make_double2(z0.x + z0.y, 0.0);
        X[h] = make_double2(z0.x - z0.y, 0.0);
    }
    __syncwarp();
}

// Direct real DFT for arbitrary m: X[k] = sum_t f(t) w[(k t) mod m], w[j] = exp(-2 pi i j / m) in wtab.
template <typename F>
__device__ __forceinline__ void rdft_any(F f, int m, double2* X, double2* wtab, int lane) {
    for (int j = lane; j < m; j += 32) {
        double s, c;
        sincospi(2.0 * (double)j / (double)m, &s, &c);
        wtab[j] = make_double2(c, -s);
    }
    __syncwarp();
    const int nb = m / 2 + 1;
    for (int k = lane; k < nb; k += 32) {
        double re = 0.0, im = 0.0;
        int idx = 0;
        for (int t = 0; t < m; ++t) {
            double v = f(t);
            double2 w = wtab[idx];
            re = fma(v, w.x, re);
            im = fma(v, w.y, im);
            idx += k;
            if (idx >= m) idx -= m;
        }
        if (k == 0 || ((m & 1) == 0 && k == m / 2)) im = 0.0;
        X[k] = make_double2(re, im);
    }
    __syncwarp();
}

// In-place complex FFT of the power of two M <= tw_n.  Forward: decimation in frequency, natural order in, bit-reversed
// order out.  Inverse (conjugate twiddles, unscaled): decimation in time, bit-reversed in, natural out.  Chained, they
// need no permutation pass.
__device__ __forceinline__ void cfft_dif(double2* X, int M, const double2* tw, int tw_n, int lane) {
    for (int len = M; len >= 2; len >>= 1) {
        const int half = len >> 1, tstep = tw_n / len;
        for (int t = lane; t < (M >> 1); t += 32) {
            const int j = t & (half - 1), i = ((t - j) << 1) + j, l = i + half;
            const double2 u = X[i], v = X[l];
            X[i] = make_double2(u.x + v.x, u.y + v.y);
            X[l] = cmul(make_double2(u.x - v.x, u.y - v.y), tw[j * tstep]);
        }
        __syncwarp();
    }
}
__device__ __forceinline__ void cifft_dit(double2* X, int M, const double2* tw, int tw_n, int lane) {
    for (int len = 2; len <= M; len <<= 1) {
        const int half = len >> 1, tstep = tw_n / len;
        for (int t = lane; t < (M >> 1); t += 32) {
            const int j = t & (half - 1), i = ((t - j) << 1) + j, l = i + half;
            const double2 w = tw[j * tstep];
            const double2 u = X[i], v = cmul(X[l], make_double2(w.x, -w.y));
            X[i] = make_double2(u.x + v.x, u.y + v.y);
            X[l] = make_double2(u.x - v.x, u.y - v.y);
        }
        __syncwarp();
    }
}

// exp(i pi j^2 / m), the angle reduced exactly: j^2 mod 2m in 64-bit integers
__device__ __forceinline__ double2 chirp(int j, int m) {
    const long long r = ((long long)j * j) % (2LL * m);
    double s, c;
    sincospi((double)r / (double)m, &s, &c);
    return make_double2(c, s);
}
// Real DFT of any m by Bluestein: with c_j = exp(i pi j^2 / m), kt = (k^2 + t^2 - (k - t)^2) / 2 gives
//   X[k] = conj(c_k) * sum_t (f(t) conj(c_t)) c_(k-t),
// a circular convolution of length M (power of two >= 2m - 1) done by two forward FFTs and one inverse.  X and B hold M
// values each; X[0..m/2] is the result.
template <typename F>
__device__ __forceinline__ void rfft_bluestein(F f, int m, double2* X, double2* B, const double2* tw, int tw_n, int lane) {
    int M = 2;
    while (M < 2 * m - 1) M <<= 1;
    for (int j = lane; j < M; j += 32) {
        double2 a = make_double2(0.0, 0.0), b = a;
        if (j < m) {
            b = chirp(j, m);
            const double v = f(j);
            a = make_double2(v * b.x, -v * b.y);
        } else if (j > M - m) b = chirp(M - j, m);
        X[j] = a;
        B[j] = b;
    }
    __syncwarp();
    cfft_dif(X, M, tw, tw_n, lane);
    cfft_dif(B, M, tw, tw_n, lane);
    for (int j = lane; j < M; j += 32) X[j] = cmul(X[j], B[j]);
    __syncwarp();
    cifft_dit(X, M, tw, tw_n, lane);
    const double inv = 1.0 / (double)M;          // exact: M is a power of two
    for (int k = lane; k <= m / 2; k += 32) {
        const double2 c = chirp(k, m);
        double2 z = cmul(X[k], make_double2(c.x * inv, -c.y * inv));
        if (k == 0 || ((m & 1) == 0 && k == m / 2)) z.y = 0.0;
        X[k] = z;
    }
    __syncwarp();
}

// Series longer than TSFX_SHORT_L_MAX only run from the global working region (GS), so only those instantiations carry
// the Bluestein path.
template <bool GS, typename F>
__device__ __forceinline__ void rfft_dispatch(F f, int m, double2* X, double2* wtab, const double2* tw, int tw_n, int lane) {
    if (m >= 4 && (m & (m - 1)) == 0 && m <= tw_n) rfft_pow2(f, m, X, tw, tw_n, lane);
    else if (GS && m > TSFX_SHORT_L_MAX) rfft_bluestein(f, m, X, wtab, tw, tw_n, lane);
    else rdft_any(f, m, X, wtab, lane);
}

__device__ __forceinline__ int hist_bin_s(double v, double first, double last, double denom, double step, int nb) {
    double f = __dmul_rn(__ddiv_rn(__dsub_rn(v, first), denom), (double)nb);
    int idx = (int)f;
    if (idx == nb) idx -= 1;
    double e_lo = __dadd_rn(__dmul_rn((double)idx, step), first);
    if (v < e_lo) idx -= 1;
    double e_hi = (idx + 1 == nb) ? last : __dadd_rn(__dmul_rn((double)(idx + 1), step), first);
    if (v >= e_hi && idx != nb - 1) idx += 1;
    return idx;
}

template <int WPC, bool GS>
__global__ void __launch_bounds__(WPC * 32) k_spectral(SpectralArgs A, int nwtab, int nhist) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    unsigned char* base = warp_region<GS>(smem_raw, A.gscratch, A.bytes_per_warp, WPC, warp);
    double2* X = reinterpret_cast<double2*>(base);                // nspec
    double2* wtab = X + A.nspec;                                  // nwtab
    double* pxx = reinterpret_cast<double*>(wtab + nwtab);        // 130
    int* hist = reinterpret_cast<int*>(pxx + 130);                // nhist
    float* xs = reinterpret_cast<float*>(hist + nhist);           // npad
    const int64_t warps_total = (int64_t)gridDim.x * WPC;

    // (no lock-step barrier here: measured slower -- the FFT stages dominate and are the same code for every warp)
    for (int64_t s = (int64_t)blockIdx.x * WPC + warp; s < A.R.n_series; s += warps_total) {
        const int n = load_series(A.R, s, xs, lane);
        double* orow = A.out + (size_t)s * A.ncols;

        // ---------------- Welch periodogram (scipy.signal.welch(x, nperseg=min(n,256))) -> pxx[0..m/2]
        int wm = n < 256 ? n : 256;
        const int wnb = wm / 2 + 1;
        double pmax = 0.0, pmin = 0.0;
        if (A.need_welch) {
            const int hop = wm - wm / 2;
            const int nseg = (n - wm) / hop + 1;
            double wss = 0.0;                        // sum w^2
            for (int k = lane; k < wm; k += 32) {
                double w = 0.5 - 0.5 * cospi(2.0 * (double)k / (double)wm);
                wss = fma(w, w, wss);
            }
            wss = wsum(wss);
            for (int k = lane; k < wnb; k += 32) pxx[k] = 0.0;
            __syncwarp();
            for (int g = 0; g < nseg; ++g) {
                const float* seg = xs + g * hop;
                double sm = 0.0;
                for (int k = lane; k < wm; k += 32) sm += (double)seg[k];
                const double mu = wsum(sm) / (double)wm;
                auto f = [&](int t) {
                    double w = 0.5 - 0.5 * cospi(2.0 * (double)t / (double)wm);
                    return ((double)seg[t] - mu) * w;
                };
                rfft_dispatch<GS>(f, wm, X, wtab, A.twiddle, A.tw_n, lane);
                for (int k = lane; k < wnb; k += 32) {
                    double2 z = X[k];
                    double p = (z.x * z.x + z.y * z.y) / wss;
                    bool edge = (k == 0) || ((wm & 1) == 0 && k == wm / 2);
                    if (!edge) p *= 2.0;
                    pxx[k] += p;
                }
                __syncwarp();
            }
            double lmax = -dinf(), lmin = dinf();
            for (int k = lane; k < wnb; k += 32) {
                double p = pxx[k] / (double)nseg;
                if (wm == 1) {      // scipy's one-sample window is 1 where the Hann formula gives 0: the detrended sample, squared
                    const double d0 = (double)xs[0] - (double)xs[0];
                    p = d0 * d0;
                }
                pxx[k] = p;
                lmax = fmax(lmax, p);
                lmin = fmin(lmin, p);
            }
            pmax = wmax(lmax);
            pmin = wmin(lmin);
            __syncwarp();
        }
        // ---------------- full-series real FFT -> X[0..n/2]
        const int nb = n / 2 + 1;
        double am0 = 0, am1 = 0, am2 = 0, am3 = 0, am4 = 0;
        if (A.need_fft) {
            auto f = [&](int t) { return (double)xs[t]; };
            rfft_dispatch<GS>(f, n, X, wtab, A.twiddle, A.tw_n, lane);
            for (int k = lane; k < nb; k += 32) {
                double2 z = X[k];
                double y = hypot(z.x, z.y);
                double kk = (double)k, k2 = kk * kk;
                am0 += y; am1 = fma(y, kk, am1); am2 = fma(y, k2, am2); am3 = fma(y, k2 * kk, am3); am4 = fma(y, k2 * k2, am4);
            }
            am0 = wsum(am0); am1 = wsum(am1); am2 = wsum(am2); am3 = wsum(am3); am4 = wsum(am4);
        }

        // fft_coefficient columns are O(1) reads of the spectrum: evaluated LANE-PARALLEL (the descriptors are
        // the first A.nfft of the group, ordered by attr so a round of 32 lanes mostly shares one branch)
        for (int j = lane; j < A.nfft; j += 32) {
            const Desc d = A.descs[j];
            double r = dnan();
            if (d.i0 < nb) {
                const double2 z = X[d.i0];
                switch (d.attr) {
                    case TSFX_FFT_REAL: r = z.x; break;
                    case TSFX_FFT_IMAG: r = z.y; break;
                    case TSFX_FFT_ABS: r = hypot(z.x, z.y); break;
                    default: r = atan2(z.y, z.x) * (180.0 / 3.14159265358979323846); break;
                }
            }
            orow[d.col] = r;
        }
        for (int j = A.nfft; j < A.nd; ++j) {
            const Desc d = A.descs[j];
            double r = dnan();
            bool stored = false;
            switch (d.calc) {
                case TSFX_FFT_AGGREGATED: {
                    double m1 = am1 / am0, m2 = am2 / am0, m3 = am3 / am0, m4 = am4 / am0;
                    double var = m2 - m1 * m1;
                    switch (d.attr) {
                        case TSFX_SPEC_CENTROID: r = m1; break;
                        case TSFX_SPEC_VARIANCE: r = var; break;
                        case TSFX_SPEC_SKEW:
                            r = (var < 0.5) ? dnan() : (m3 - 3.0 * m1 * var - m1 * m1 * m1) / pow(var, 1.5);
                            break;
                        default:
                            r = (var < 0.5) ? dnan() : (m4 - 4.0 * m1 * m3 + 6.0 * m2 * m1 * m1 - 3.0 * m1) / (var * var);
                            break;
                    }
                    if (var != var) r = dnan();
                    break;
                }
                case TSFX_SPKT_WELCH_DENSITY: r = (d.i0 < wnb) ? pxx[d.i0] : dnan(); break;
                case TSFX_FOURIER_ENTROPY: {
                    // binned_entropy(pxx / max(pxx), bins)
                    const int nbins = d.i0;
                    double first = pmin / pmax, last = pmax / pmax;
                    if (first != first || last != last) { r = dnan(); break; }
                    if (first == last) { first -= 0.5; last += 0.5; }
                    double denom = __dsub_rn(last, first);
                    double step = __ddiv_rn(denom, (double)nbins);
                    for (int b = lane; b < nbins; b += 32) hist[b] = 0;
                    __syncwarp();
                    for (int k = lane; k < wnb; k += 32) {
                        int idx = hist_bin_s(pxx[k] / pmax, first, last, denom, step, nbins);
                        atomicAdd(&hist[idx], 1);
                    }
                    __syncwarp();
                    double a = 0.0;
                    for (int b = lane; b < nbins; b += 32) {
                        int c = hist[b];
                        if (c > 0) { double p = (double)c / (double)wnb; a += p * log(p); }
                    }
                    r = -wsum(a);
                    __syncwarp();
                    break;
                }
                case TSFX_CWT_COEFFICIENTS: {
                    // the whole run of cwt_coefficients descriptors (sorted by width, descriptor j writes column j):
                    // one coefficient per lane, each lane walks the taps of its wavelet row serially -- no warp
                    // sum and one trip through this loop instead of one per column
                    int run = 0;
                    for (;;) {
                        const int jj = j + run + lane;
                        const unsigned same = __ballot_sync(FULL, jj < A.nd && A.descs[jj].calc == TSFX_CWT_COEFFICIENTS);
                        if (same == FULL) { run += 32; continue; }
                        run += __ffs(~same) - 1;
                        break;
                    }
                    for (int t = lane; t < run; t += 32) {
                        const Desc e = A.descs[j + t];
                        const int c = e.i0;
                        double a = dnan();
                        if (n > c) {
                            const double* D = A.tables + A.table_off[e.i1];
                            const int dl = (int)(A.table_off[e.i1 + 1] - A.table_off[e.i1]);
                            const int top = c + A.table_half[e.i1];        // D index for k = 0
                            int k0 = top - (dl - 1);
                            if (k0 < 0) k0 = 0;
                            const int k1 = top < n - 1 ? top : n - 1;
                            a = 0.0;
                            for (int k = k0; k <= k1; ++k) a = fma((double)xs[k], __ldg(D + (top - k)), a);
                        }
                        orow[j + t] = a;
                    }
                    stored = true;
                    j += run - 1;
                    break;
                }
                default: break;
            }
            if (!stored && lane == 0) orow[d.col] = r;
        }
        __syncwarp();
    }
}

cudaError_t launch_spectral(const SpectralArgs& A0, int max_len, cudaStream_t st, int sm_count, const char** variant) {
    SpectralArgs A = A0;
    A.npad = (max_len + 3) & ~3;
    A.nspec = A.npad / 2 + 2;
    bool dense_pow2 = (A.R.begin == nullptr) && max_len >= 4 && (max_len & (max_len - 1)) == 0;
    int nwtab = dense_pow2 ? 0 : A.npad;
    if (max_len > TSFX_L_MAX) return cudaErrorInvalidConfiguration;
    if (!dense_pow2 && max_len > TSFX_SHORT_L_MAX) {
        // Bluestein: the spectrum and the chirp each take M complex values (M >= 2 max_len - 1, twiddle table >= M)
        int M = 2;
        while (M < 2 * max_len - 1) M <<= 1;
        if (M > A.tw_n) return cudaErrorInvalidValue;
        A.nspec = nwtab = M;
    }
    int nhist = (std::max(A.max_hist, 4) + 3) & ~3;
    size_t per = (size_t)A.nspec * 16 + (size_t)nwtab * 16 + 130 * 8 + (size_t)nhist * 4 + (size_t)A.npad * 4;
    per = (per + 15) & ~(size_t)15;
    A.bytes_per_warp = (int)per;
    Geometry G;
    if (!plan_geometry(per, 100 * 1024, 8, A.R.n_series, sm_count, A.gscratch, A.gscratch_bytes, &G)) return cudaErrorInvalidConfiguration;
    A.gscratch = G.gscratch;
    auto launch = [&](auto g) { return launch_kernel(k_spectral<decltype(g)::wpc, decltype(g)::global>, G, st, A, nwtab, nhist); };
    if (dense_pow2)          // dense power-of-two length: no twiddle-word table
        TSFX_LAUNCH_DECLARED(TSFX_GEOMS_ALL, "spectral/pow2", G, variant, launch);
    TSFX_LAUNCH_DECLARED(TSFX_GEOMS_ALL, "spectral", G, variant, launch);
}

}  // namespace tsfx
