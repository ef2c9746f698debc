// k_seq.cu -- kernel group SEQ: the inherently sequential / dictionary calculators
//   lempel_ziv_complexity (feature_calculators.py:1825-1862)   lane-per-parameter trie parse
//   permutation_entropy   (feature_calculators.py:1866-1915)   rank codes -> bitonic sort -> run lengths
//
// One warp per series.  k_seq: general layout = uint32 codes[npow2], one uint32 open-addressing key table per Lempel-Ziv
// parameter, uint16 symbols, float xs[npad] (17.8 KB per warp at 256 samples, run from the global working region);
// compact layout k_seq_small (series <= 256, alphabets <= 127) = packed 16-bit histogram counters, 16-bit keys in
// 256-slot tables, byte symbols (6.5 KB per warp, shared memory, 32 warps per SM).
#include <algorithm>

#include "tsfx_common.cuh"
#include "tsfx_kernels.h"

namespace tsfx {

#define LZ_LANES 8

struct SeqLayout {
    int hist_cap;                                    // permutation-histogram bins the `codes` area can hold
    int npad, npow2, lz_lanes, lz_hash, lz_stride;
    int off_codes, off_trie, off_sym, off_xs;        // byte offsets
};

// ---------------------------------------------------------------------------- Lempel-Ziv
// symbol = np.searchsorted(np.linspace(min, max, bins+1)[1:], x, side="left")
__device__ __forceinline__ int lz_symbol(double v, double vmin, double vmax, double step, int bins) {
    int c = (int)__ddiv_rn(__dsub_rn(v, vmin), step);      // NaN (step == 0) converts to 0
    if (c < 0) c = 0;
    if (c > bins) c = bins;
    // edge(i) = i*step + vmin for i < bins, edge(bins) = vmax ; count edges i in 1..bins with edge(i) < v
    while (c < bins) {
        double e = (c + 1 == bins) ? vmax : __dadd_rn(__dmul_rn((double)(c + 1), step), vmin);
        if (e < v) ++c; else break;
    }
    while (c > 0) {
        double e = (c == bins) ? vmax : __dadd_rn(__dmul_rn((double)c, step), vmin);
        if (!(e < v)) --c; else break;
    }
    return c;
}

// ---------------------------------------------------------------------------- bitonic sort on uint32
__device__ __forceinline__ void warp_bitonic_sort_u32(unsigned* s, int m, int lane) {
    for (int k = 2; k <= m; k <<= 1) {
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int t = lane; t < (m >> 1); t += 32) {
                int i = 2 * t - (t & (j - 1));
                int l = i + j;
                unsigned a = s[i], b = s[l];
                bool up = (i & k) == 0;
                if ((a > b) == up) { s[i] = b; s[l] = a; }
            }
            __syncwarp();
        }
    }
}

// ---------------------------------------------------------------------------- permutation patterns
// A window's rank pattern is fixed by its pairwise order bits b(p,q) = [w_q < w_p], p < q (ties: the earlier
// sample counts as smaller = stable ranks).  With the bits laid out q-major (bit q(q-1)/2 + p) the pattern of
// the first D samples is the low D(D-1)/2 bits, so ONE pass over a window serves every dimension.  The dense
// index used for counting is the Lehmer code: digit p = popcount(bits & PE_MASK[D][p]).
struct PeMasks { unsigned m[9][8]; };
__host__ __device__ constexpr PeMasks make_pe_masks() {
    PeMasks M = {};
    for (int D = 2; D <= 8; ++D)
        for (int p = 0; p < D - 1; ++p) {
            unsigned v = 0;
            for (int q = p + 1; q < D; ++q) v |= 1u << (q * (q - 1) / 2 + p);
            M.m[D][p] = v;
        }
    return M;
}
__constant__ PeMasks PE_MASKS = make_pe_masks();

__device__ __forceinline__ unsigned pe_order_bits(const float* w, int m) {      // m = samples available (<= 8)
    float v[8];
#pragma unroll
    for (int q = 0; q < 8; ++q) v[q] = q < m ? w[q] : 0.f;
    unsigned bits = 0;
#pragma unroll
    for (int q = 1; q < 8; ++q)
#pragma unroll
        for (int p = 0; p < q; ++p)
            if (q < m) bits |= (v[q] < v[p]) ? (1u << (q * (q - 1) / 2 + p)) : 0u;
    return bits;
}
__device__ __forceinline__ unsigned pe_lehmer(unsigned bits, int D) {
    unsigned code = 0;
    for (int p = 0; p < D - 1; ++p) code = code * (unsigned)(D - p) + (unsigned)__popc(bits & PE_MASKS.m[D][p]);
    return code;            // digit D-1 is always 0 (radix 1)
}

// SMALL = compact shared-memory working set for series of at most 256 samples and alphabets of at most 127 symbols (the
// BASELINE shapes): byte symbols, 16-bit trie keys (node << 7 | symbol, 256 slots per parse) and permutation histograms
// with two 16-bit counters per word -- 6.5 KB per warp, so 32 warps per SM run entirely from shared memory.  The general
// layout (uint32 keys, uint16 symbols, uint32 counters) needs 17.8 KB per warp and runs from the global working region,
// where every probe of the sequential parse and every histogram update is an L2 round trip.
template <int WPC, bool GS, bool SMALL>
__device__ __forceinline__ void seq_body(const SeqArgs& A, const SeqLayout& Y) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    __shared__ double clogc_small[64];            // c ln c for small counts (permutation histograms are mostly tiny)
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x < 64) clogc_small[threadIdx.x] = threadIdx.x > 1 ? (double)threadIdx.x * log((double)threadIdx.x) : 0.0;
    if (WPC * 32 < 64 && threadIdx.x < 32) clogc_small[32 + threadIdx.x] = (double)(32 + threadIdx.x) * log((double)(32 + threadIdx.x));
    __syncthreads();
    unsigned char* base = warp_region<GS>(smem_raw, A.gscratch, A.bytes_per_warp, WPC, warp);
    unsigned* codes = reinterpret_cast<unsigned*>(base + Y.off_codes);
    unsigned short* trie = reinterpret_cast<unsigned short*>(base + Y.off_trie);
    unsigned short* symbuf = reinterpret_cast<unsigned short*>(base + Y.off_sym);
    unsigned char* symbuf8 = base + Y.off_sym;
    float* xs = reinterpret_cast<float*>(base + Y.off_xs);
    const int64_t warps_total = (int64_t)gridDim.x * WPC;

    for (int64_t s = (int64_t)blockIdx.x * WPC + warp; s < A.R.n_series; s += warps_total) {
        const int n = load_series(A.R, s, xs, lane);
        double* orow = A.out + (size_t)s * A.ncols;
        float lo = INFINITY, hi = -INFINITY;
        for (int i = lane; i < n; i += 32) { lo = fminf(lo, xs[i]); hi = fmaxf(hi, xs[i]); }
        const double vmin = (double)wminf(lo), vmax = (double)wmaxf(hi);

        int j = 0;
        while (j < A.nd) {
            const Desc d0 = A.descs[j];
            if (d0.calc == TSFX_LEMPEL_ZIV_COMPLEXITY) {
                // up to lz_lanes consecutive LZ descriptors, one per lane
                int cnt = 0;
                while (j + cnt < A.nd && cnt < Y.lz_lanes && A.descs[j + cnt].calc == TSFX_LEMPEL_ZIV_COMPLEXITY) ++cnt;
                for (int q = 0; q < cnt; ++q) {                      // symbols of every position, all lanes
                    const int bins = A.descs[j + q].i0;
                    const double step = __ddiv_rn(__dsub_rn(vmax, vmin), (double)bins);
                    if (SMALL) {
                        unsigned char* sb = symbuf8 + (size_t)q * Y.npad;
                        for (int pos = lane; pos < n; pos += 32) sb[pos] = (unsigned char)lz_symbol((double)xs[pos], vmin, vmax, step, bins);
                    } else {
                        unsigned short* sb = symbuf + (size_t)q * Y.npad;
                        for (int pos = lane; pos < n; pos += 32) sb[pos] = (unsigned short)lz_symbol((double)xs[pos], vmin, vmax, step, bins);
                    }
                }
                __syncwarp();
                // phrase dictionary = prefix-closed trie stored as ONE open-addressing table of keys
                // (parent slot << 16 | symbol); a node's id is the slot its key lives in, the root is 0xffff
                {
                    unsigned* tab = reinterpret_cast<unsigned*>(trie);       // SMALL: two 16-bit keys per word
                    const int words = SMALL ? (cnt * Y.lz_hash) >> 1 : cnt * Y.lz_hash;
                    for (int q = lane; q < words; q += 32) tab[q] = 0xffffffffu;
                }
                __syncwarp();
                if (lane < cnt) {
                    const Desc d = A.descs[j + lane];
                    int phrases = 0;
                    if (SMALL) {
                        const unsigned char* sb = symbuf8 + (size_t)lane * Y.npad;
                        unsigned short* hkey = trie + (size_t)lane * Y.lz_hash;
                        const unsigned mask = (unsigned)Y.lz_hash - 1u;          // 256 slots: node ids fit 8 bits, the root is 256
                        unsigned node = 256u;
                        for (int pos = 0; pos < n; ++pos) {
                            const unsigned key = (node << 7) | (unsigned)sb[pos];
                            unsigned h = ((key * 0x9E3779B1u) >> 20) & mask;
                            unsigned k;
                            while ((k = hkey[h]) != key && k != 0xffffu) h = (h + 1u) & mask;
                            if (k == key) node = h;
                            else { hkey[h] = (unsigned short)key; ++phrases; node = 256u; }
                        }
                    } else {
                        const unsigned short* sb = symbuf + (size_t)lane * Y.npad;
                        unsigned* hkey = reinterpret_cast<unsigned*>(trie) + (size_t)lane * Y.lz_hash;
                        const unsigned mask = (unsigned)Y.lz_hash - 1u;
                        unsigned node = 0xffffu;
                        for (int pos = 0; pos < n; ++pos) {
                            const unsigned key = (node << 16) | (unsigned)sb[pos];
                            unsigned h = (key * 0x9E3779B1u) >> 15;
                            h &= mask;
                            unsigned k;
                            while ((k = hkey[h]) != key && k != 0xffffffffu) h = (h + 1u) & mask;
                            if (k == key) node = h;                      // phrase seen: extend it
                            else { hkey[h] = key; ++phrases; node = 0xffffu; }
                        }
                    }
                    orow[d.col] = (double)phrases / (double)n;
                }
                __syncwarp();
                j += cnt;
            } else if (d0.calc == TSFX_PERMUTATION_ENTROPY) {
                // run of permutation_entropy descriptors sharing tau: one pass over the windows serves all of
                // them (dimensions <= 6 through shared-memory histograms over the D! Lehmer indices)
                const int tau = d0.i0;
                int cnt = 0, bins_total = 0, Dh = 0;
                while (j + cnt < A.nd && A.descs[j + cnt].calc == TSFX_PERMUTATION_ENTROPY && A.descs[j + cnt].i0 == tau) {
                    const int D = A.descs[j + cnt].i1;
                    if (D <= 6) {
                        int f = 1;
                        for (int q = 2; q <= D; ++q) f *= q;
                        if (bins_total + f > Y.hist_cap) break;
                        bins_total += f;
                        Dh = max(Dh, D);
                    }
                    ++cnt;
                }
                if (cnt == 0) {             // a histogram that does not fit the `codes` area at all: cannot happen for
                    if (lane == 0) orow[d0.col] = dnan();      // dimensions <= 6 (720 bins <= hist_cap); never loop in place
                    ++j;
                    continue;
                }
                if (Dh > 0) {
                    for (int b = lane; b < (SMALL ? (bins_total + 1) >> 1 : bins_total); b += 32) codes[b] = 0u;
                    __syncwarp();
                    const int Wmax = (n >= 2) ? (n - 2) / tau + 1 : 0;          // windows of the smallest dimension
                    for (int k = lane; k < Wmax; k += 32) {
                        const int st = k * tau;
                        const unsigned bits = pe_order_bits(xs + st, min(8, n - st));
                        int off = 0;
                        for (int t = 0; t < cnt; ++t) {
                            const int D = A.descs[j + t].i1;
                            if (D > 6) continue;
                            int f = 1;
                            for (int q = 2; q <= D; ++q) f *= q;
                            if (st + D <= n) {
                                const unsigned bin = off + pe_lehmer(bits, D);
                                if (SMALL) atomicAdd(&codes[bin >> 1], (bin & 1u) ? 0x10000u : 1u);
                                else atomicAdd(&codes[bin], 1u);
                            }
                            off += f;
                        }
                    }
                    __syncwarp();
                    int off = 0;
                    for (int t = 0; t < cnt; ++t) {
                        const Desc d = A.descs[j + t];
                        const int D = d.i1;
                        if (D > 6) continue;
                        int f = 1;
                        for (int q = 2; q <= D; ++q) f *= q;
                        double r = dnan();
                        if (n >= D) {
                            const int W = (n - D) / tau + 1;
                            // -sum p ln p = ln W - (1/W) sum c ln c  (bins with c = 1 contribute nothing)
                            double acc = 0.0;
                            for (int b = lane; b < f; b += 32) {
                                const unsigned c = SMALL ? (codes[(off + b) >> 1] >> (16 * ((off + b) & 1))) & 0xffffu : codes[off + b];
                                if (c > 1u) acc += c < 64u ? clogc_small[c] : (double)c * log((double)c);
                            }
                            r = log((double)W) - wsum(acc) / (double)W;
                        }
                        if (lane == 0) orow[d.col] = r;
                        off += f;
                    }
                    __syncwarp();
                }
                for (int t = 0; t < cnt; ++t) {             // dimensions 7, 8: sort the indices, count run lengths
                    const Desc d = A.descs[j + t];
                    const int D = d.i1;
                    if (D <= 6) continue;
                    double r = dnan();
                    if (n >= D) {
                        const int W = (n - D) / tau + 1;
                        int m = 2;
                        while (m < W) m <<= 1;
                        for (int k = lane; k < m; k += 32)
                            codes[k] = (k < W) ? pe_lehmer(pe_order_bits(xs + k * tau, D), D) : 0xffffffffu;
                        __syncwarp();
                        warp_bitonic_sort_u32(codes, m, lane);
                        double acc = 0.0;
                        for (int k = lane; k < W; k += 32) {
                            const unsigned c = codes[k];
                            if ((k == 0 || codes[k - 1] != c) && k + 1 < W && codes[k + 1] == c) {
                                int len = 2;
                                while (k + len < W && codes[k + len] == c) ++len;
                                acc += len < 64 ? clogc_small[len] : (double)len * log((double)len);
                            }
                        }
                        r = log((double)W) - wsum(acc) / (double)W;
                        __syncwarp();
                    }
                    if (lane == 0) orow[d.col] = r;
                }
                j += cnt;
            } else {
                if (lane == 0) orow[d0.col] = dnan();
                ++j;
            }
        }
        __syncwarp();
    }
}

template <int WPC, bool GS>
__global__ void __launch_bounds__(WPC * 32) k_seq(SeqArgs A, SeqLayout Y) { seq_body<WPC, GS, false>(A, Y); }

template <int WPC, bool GS>
__global__ void __launch_bounds__(WPC * 32, (WPC == 4 ? 8 : 1)) k_seq_small(SeqArgs A, SeqLayout Y) { seq_body<WPC, GS, true>(A, Y); }

cudaError_t launch_seq(const SeqArgs& A0, int max_len, cudaStream_t st, int sm_count, const char** variant) {
    SeqArgs A = A0;
    A.npad = (max_len + 3) & ~3;
    if (max_len > 21000) return cudaErrorInvalidConfiguration;      // LZ node ids are 15-bit slot indices
    SeqLayout Y = {};
    Y.npad = A.npad;
    Y.lz_lanes = A.need_lz ? std::min(LZ_LANES, std::max(1, A.n_lz)) : 0;
    if (max_len <= 256 && A.max_lz_bins <= 127) {
        // compact shared-memory layout (k_seq_small)
        Y.lz_hash = 256;
        Y.npow2 = 256;                                   // sort path of dimensions 7, 8: <= 256 windows
        Y.hist_cap = 896;                                // 1792 bytes of packed 16-bit counters
        size_t o = 0;
        Y.off_codes = (int)o; o += A.need_perm ? (size_t)1792 : 0;   // 870 packed 16-bit bins (dimensions 3..6), or 256 sort keys
        Y.off_trie = (int)o;  o += (size_t)Y.lz_lanes * Y.lz_hash * 2;
        Y.off_sym = (int)o;   o += (size_t)Y.lz_lanes * A.npad;
        o = (o + 15) & ~(size_t)15;
        Y.off_xs = (int)o;    o += (size_t)A.npad * 4;
        const size_t per = (o + 15) & ~(size_t)15;
        A.bytes_per_warp = (int)per;
        A.gscratch = nullptr;
        *variant = "seq/small";
        return launch_fixed(k_seq_small<4, false>, 4 * 32, 4, per * 4, (int64_t)sm_count * grid_waves(4096), A.R.n_series, st, A, Y);
    }
    int p2 = 2;
    while (p2 < max_len) p2 <<= 1;
    Y.npow2 = std::max(p2, 1024);                 // >= 6! = 720 so dimensions up to 6 use the histogram path
    Y.hist_cap = Y.npow2;
    Y.lz_hash = 4;
    while (Y.lz_hash < A.npad + A.npad / 2 + 2) Y.lz_hash <<= 1;      // load factor <= 2/3 in the worst case
    Y.lz_stride = 2 * Y.lz_hash;                  // uint16 units: one uint32 key per slot
    size_t off = 0;
    Y.off_codes = (int)off; off += A.need_perm ? (size_t)Y.npow2 * 4 : 0;
    Y.off_trie = (int)off;  off += (size_t)Y.lz_lanes * Y.lz_stride * 2;
    off = (off + 3) & ~(size_t)3;
    Y.off_sym = (int)off;   off += (size_t)Y.lz_lanes * A.npad * 2;
    off = (off + 15) & ~(size_t)15;
    Y.off_xs = (int)off;    off += (size_t)A.npad * 4;
    size_t per = (off + 15) & ~(size_t)15;
    A.bytes_per_warp = (int)per;
    Geometry G;
    if (!plan_geometry(per, 72 * 1024, 8, A.R.n_series, sm_count, A.gscratch, A.gscratch_bytes, &G, 16 * 1024, 8)) return cudaErrorInvalidConfiguration;
    A.gscratch = G.gscratch;
    auto launch = [&](auto g) { return launch_kernel(k_seq<decltype(g)::wpc, decltype(g)::global>, G, st, A, Y); };
    TSFX_LAUNCH_DECLARED(TSFX_GEOMS_SEQ, "seq/general", G, variant, launch);
}

}  // namespace tsfx
