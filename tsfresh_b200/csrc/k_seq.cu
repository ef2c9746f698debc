// k_seq.cu -- kernel group SEQ: the inherently sequential / dictionary calculators
//   lempel_ziv_complexity (feature_calculators.py:1825-1862)   lane-per-parameter trie parse
//   permutation_entropy   (feature_calculators.py:1866-1915)   order bits -> histograms of Lehmer codes (dimensions <= 6),
//                                                                sorted Lehmer codes -> run lengths (dimensions 7, 8)
//
// One warp per series.  k_seq: general layout = uint32 codes[npow2], one uint32 open-addressing key table per Lempel-Ziv
// parameter (uint64 keys past TSFX_SHORT_L_MAX samples), uint16 symbols, float xs[npad] (17.8 KB per warp at 256 samples,
// run from the global working region);
// compact layout k_seq_small (series <= 256, alphabets <= 127) = packed 16-bit histogram counters, 16-bit keys in
// 384-slot tables (256 with more than five Lempel-Ziv columns) sharing their area with the histograms, byte symbols
// (6 KB per warp at five Lempel-Ziv columns, shared memory, 32 warps per SM); its windows are sorted once in
// registers, and the histograms are filled one run of equal patterns at a time.
#include <algorithm>

#include "tsfx_common.cuh"
#include "tsfx_kernels.h"
#include "tsfx_warp_sort.cuh"

// Builds for profiles/scripts/time_seq_phases.py: -DTSFX_SEQ_SKIP=k leaves phase k of k_seq_small out (1 load + min/max,
// 2 Lempel-Ziv symbols, 3 Lempel-Ziv parse, 4 permutation counts of dimensions <= 6, 5 dimensions 7 and 8, 6 order bits
// and the window sort, 7 the entropy finish of dimensions <= 6), so the group's time splits by phase.  Their results
// are wrong; the library build never sets it.
#ifndef TSFX_SEQ_SKIP
#define TSFX_SEQ_SKIP 0
#endif
#define SEQ_SKIP(k) (SMALL && TSFX_SEQ_SKIP == (k))

namespace tsfx {

#define LZ_LANES 8

struct SeqLayout {
    int hist_cap;                                    // permutation-histogram bins the `codes` area can hold
    int npad, npow2, lz_lanes, lz_hash, lz_stride;
    int wide;                                        // series longer than TSFX_SHORT_L_MAX: 64-bit Lempel-Ziv keys
    int off_codes, off_trie, off_sym, off_xs;        // byte offsets
};

// ---------------------------------------------------------------------------- Lempel-Ziv
// symbol = np.searchsorted(np.linspace(min, max, bins+1)[1:], x, side="left")
// c is an estimate of the symbol; the loops below move it to the number of edges below v.  The edges are
// nondecreasing in i (for float32-origin min and max, edge(bins - 1) stays below max by about step), so that number
// is the one c where both loops stop, whatever the estimate: the estimate only sets how many steps they take.
__device__ __forceinline__ int lz_symbol(int c, double v, double vmin, double vmax, double step, int bins) {
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
// BASELINE shapes): byte symbols, 16-bit trie keys (node << 7 | symbol, 384 or 256 slots per parse) and permutation histograms
// with two 16-bit counters per word -- at most 6.75 KB per warp, so 32 warps per SM run entirely from shared memory.  The general
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
        double* orow = A.out + (size_t)s * A.ncols;
        int n;
        double vmin, vmax;
        if (SEQ_SKIP(1)) {          // a hashed series in [0, 1) in place of the load and the min/max
            n = A.R.begin ? A.R.len[s] : A.R.dense_len;
            for (int i = lane; i < n; i += 32) xs[i] = (float)((unsigned)(i + s) * 2654435761u >> 8) * 0x1p-24f;
            __syncwarp();
            vmin = 0.0; vmax = 1.0;
        } else {
            n = load_series(A.R, s, xs, lane);
            float lo = INFINITY, hi = -INFINITY;
            for (int i = lane; i < n; i += 32) { lo = fminf(lo, xs[i]); hi = fmaxf(hi, xs[i]); }
            vmin = (double)wminf(lo); vmax = (double)wmaxf(hi);
        }

        int j = 0;
        while (j < A.nd) {
            const Desc d0 = A.descs[j];
            if (d0.calc == TSFX_LEMPEL_ZIV_COMPLEXITY) {
                // up to lz_lanes consecutive LZ descriptors, one per lane
                int cnt = 0;
                while (j + cnt < A.nd && cnt < Y.lz_lanes && A.descs[j + cnt].calc == TSFX_LEMPEL_ZIV_COMPLEXITY) ++cnt;
                for (int q = 0; q < (SEQ_SKIP(2) ? 0 : cnt); ++q) {   // symbols of every position, all lanes
                    const int bins = A.descs[j + q].i0;
                    const double step = __ddiv_rn(__dsub_rn(vmax, vmin), (double)bins);
                    if (SMALL) {
                        // (v - vmin) * (1 / step) is within a few units in the last place of the quotient (v - vmin) / step,
                        // so its truncation is the division's or one off (lz_symbol's loops then take one more step);
                        // step == 0 gives 0 * inf = NaN, which converts to 0 like the division's NaN
                        const double rstep = __drcp_rn(step);
                        unsigned char* sb = symbuf8 + (size_t)q * Y.npad;
                        for (int pos = lane; pos < n; pos += 32) {
                            const double v = (double)xs[pos];
                            sb[pos] = (unsigned char)lz_symbol((int)__dmul_rn(__dsub_rn(v, vmin), rstep), v, vmin, vmax, step, bins);
                        }
                    } else {
                        unsigned short* sb = symbuf + (size_t)q * Y.npad;
                        for (int pos = lane; pos < n; pos += 32) {
                            const double v = (double)xs[pos];
                            sb[pos] = (unsigned short)lz_symbol((int)__ddiv_rn(__dsub_rn(v, vmin), step), v, vmin, vmax, step, bins);
                        }
                    }
                }
                __syncwarp();
                // phrase dictionary = prefix-closed trie stored as ONE open-addressing table of keys
                // (parent slot << 16 | symbol); a node's id is the slot its key lives in, the root is 0xffff
                {
                    unsigned* tab = reinterpret_cast<unsigned*>(trie);       // SMALL: two 16-bit keys per word
                    const int words = SMALL ? (cnt * Y.lz_hash) >> 1 : cnt * Y.lz_hash * (Y.wide ? 2 : 1);
                    for (int q = lane; q < words; q += 32) tab[q] = 0xffffffffu;
                }
                __syncwarp();
                if (lane < cnt) {
                    const Desc d = A.descs[j + lane];
                    int phrases = 0;
                    if (SEQ_SKIP(3)) {
                    } else if (SMALL) {
                        const unsigned char* sb = symbuf8 + (size_t)lane * Y.npad;
                        // slots = 256 or 384: node ids are below it, the root is `slots`, so a key (node << 7 | symbol)
                        // stays below 0xffff, the empty mark
                        const unsigned slots = (unsigned)Y.lz_hash;
                        unsigned short* hkey = trie + (size_t)lane * slots;
                        unsigned node = slots;
                        for (int pos = 0; pos < n; ++pos) {
                            const unsigned key = (node << 7) | (unsigned)sb[pos];
                            unsigned h = __umulhi(key * 0x9E3779B1u, slots);
                            unsigned k;
                            while ((k = hkey[h]) != key && k != 0xffffu) h = (h + 1u == slots) ? 0u : h + 1u;
                            if (k == key) node = h;
                            else { hkey[h] = (unsigned short)key; ++phrases; node = slots; }
                        }
                    } else if (Y.wide) {
                        // more than 2^16 slots: node ids need 18 bits, so keys (parent slot << 16 | symbol) are
                        // 64-bit and the root is 0xffffffff
                        const unsigned short* sb = symbuf + (size_t)lane * Y.npad;
                        unsigned long long* hkey = reinterpret_cast<unsigned long long*>(trie) + (size_t)lane * Y.lz_hash;
                        const unsigned mask = (unsigned)Y.lz_hash - 1u;
                        unsigned long long node = 0xffffffffull;
                        for (int pos = 0; pos < n; ++pos) {
                            const unsigned long long key = (node << 16) | (unsigned long long)sb[pos];
                            unsigned h = (unsigned)((key * 0x9E3779B97F4A7C15ull) >> 40) & mask;
                            unsigned long long k;
                            while ((k = hkey[h]) != key && k != ~0ull) h = (h + 1u) & mask;
                            if (k == key) node = h;
                            else { hkey[h] = key; ++phrases; node = 0xffffffffull; }
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
                const int Wmax = (n >= 2) ? (n - 2) / tau + 1 : 0;              // windows of the smallest dimension
                // SMALL: the windows sorted once, in registers (lane L holds sorted positions 8L .. 8L + 7), by the key
                // brev(order bits) | (8 - m), m = min(8, samples from the window's start).  The order bits use bits
                // 0 .. 27, so brev puts the pattern of every dimension D, its low D(D-1)/2 bits, at the top of the key:
                // equal patterns of every dimension sit in contiguous runs.  A window counts for D when m >= D, i.e.
                // (key & 15) <= 8 - D; the padding keys 0xffffffff count for none.
                unsigned v[8];
                if constexpr (SMALL) {
#pragma unroll
                    for (int e = 0; e < 8; ++e) {
                        const int k = lane + 32 * e, st = k * tau, m = min(8, n - st);
                        v[e] = k < Wmax ? (SEQ_SKIP(6) ? (unsigned)(k * 2654435761u) & ~15u : __brev(pe_order_bits(xs + st, m))) | (unsigned)(8 - m)
                                        : 0xffffffffu;
                    }
                    if (!SEQ_SKIP(6)) warp_sort256(v, lane);
                }
                if (Dh > 0) {
                    for (int b = lane; b < (SMALL ? (bins_total + 1) >> 1 : bins_total); b += 32) codes[b] = 0u;
                    __syncwarp();
                    if constexpr (SMALL) {
                        // one atomic per run boundary instead of one per window: with V(a) the valid windows at sorted
                        // positions < a, a run [a0, a1] adds V(a1 + 1) - V(a0) to its Lehmer bin (packed 16-bit counters:
                        // the words wrap modulo 2^32 on the way and end exact)
                        int off = 0;
                        for (int t = 0; t < (SEQ_SKIP(4) ? 0 : cnt); ++t) {
                            const int D = A.descs[j + t].i1;
                            if (D > 6) continue;
                            int f = 1;
                            for (int q = 2; q <= D; ++q) f *= q;
                            const unsigned pm = ~0u << (32 - D * (D - 1) / 2), lim = 8u - D;
                            int c[8], run = 0;
#pragma unroll
                            for (int e = 0; e < 8; ++e) { run += (v[e] & 15u) <= lim; c[e] = run; }
                            int before = run;                                    // warp inclusive scan of the lane totals
#pragma unroll
                            for (int o = 1; o < 32; o <<= 1) {
                                const int y = __shfl_up_sync(FULL, before, o);
                                if (lane >= o) before += y;
                            }
                            before -= run;
                            const unsigned prev = __shfl_up_sync(FULL, v[7] & pm, 1), next = __shfl_down_sync(FULL, v[0] & pm, 1);
#pragma unroll
                            for (int e = 0; e < 8; ++e) {
                                const unsigned pe = v[e] & pm;
                                const bool first = e ? (v[e - 1] & pm) != pe : (lane == 0 || prev != pe);
                                const bool last = e < 7 ? (v[e + 1] & pm) != pe : (lane == 31 || next != pe);
                                const int delta = (last ? before + c[e] : 0) - (first ? before + (e ? c[e - 1] : 0) : 0);
                                if (delta != 0) {
                                    const unsigned bin = off + pe_lehmer(__brev(v[e]), D);
                                    atomicAdd(&codes[bin >> 1], (unsigned)delta << (16 * (bin & 1u)));
                                }
                            }
                            off += f;
                        }
                    } else {
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
                                    atomicAdd(&codes[off + pe_lehmer(bits, D)], 1u);
                                }
                                off += f;
                            }
                        }
                    }
                    __syncwarp();
                    int off = 0;
                    for (int t = 0; t < (SEQ_SKIP(7) ? 0 : cnt); ++t) {
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
                    if (n >= D && !SEQ_SKIP(5)) {
                        const int W = (n - D) / tau + 1;
                        if constexpr (SMALL) {          // the W windows valid for D, their Lehmer codes sorted in registers
                            unsigned c[8];
#pragma unroll
                            for (int e = 0; e < 8; ++e) c[e] = (v[e] & 15u) <= 8u - D ? pe_lehmer(__brev(v[e]), D) : 0xffffffffu;
                            warp_sort256(c, lane);
                            reinterpret_cast<uint4*>(codes)[2 * lane] = make_uint4(c[0], c[1], c[2], c[3]);
                            reinterpret_cast<uint4*>(codes)[2 * lane + 1] = make_uint4(c[4], c[5], c[6], c[7]);
                            __syncwarp();
                        } else {
                            int m = 2;
                            while (m < W) m <<= 1;
                            for (int k = lane; k < m; k += 32)
                                codes[k] = (k < W) ? pe_lehmer(pe_order_bits(xs + k * tau, D), D) : 0xffffffffu;
                            __syncwarp();
                            warp_bitonic_sort_u32(codes, m, lane);
                        }
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
    if (max_len > TSFX_L_MAX) return cudaErrorInvalidConfiguration;
    SeqLayout Y = {};
    Y.npad = A.npad;
    Y.lz_lanes = A.need_lz ? std::min(LZ_LANES, std::max(1, A.n_lz)) : 0;
    if (max_len <= 256 && A.max_lz_bins <= 127) {
        // compact shared-memory layout (k_seq_small)
        // The permutation histograms and the Lempel-Ziv tables are never live at the same time (a series runs its
        // descriptor runs one after another, with a __syncwarp between them), so they share one area.  Each parse
        // gets 384 table slots where the warp's working set still lets 32 warps run per SM (8 CTAs of 4 warps: at
        // most 6 912 bytes per warp beside the 512 static and 1 024 reserved bytes per CTA), 256 slots otherwise.
        // The fuller a table, the longer its linear probes, and a warp waits for the longest of its parses' probes.
        Y.npow2 = 256;                                   // sort path of dimensions 7, 8: <= 256 windows
        Y.hist_cap = 896;                                // 1792 bytes of packed 16-bit counters
        size_t per = 0;
        for (int slots : {384, 256}) {
            Y.lz_hash = slots;
            size_t o = std::max(A.need_perm ? (size_t)1792 : 0,            // 870 packed 16-bit bins (dimensions 3..6), or 256 sort keys
                                (size_t)Y.lz_lanes * Y.lz_hash * 2);
            Y.off_codes = 0;
            Y.off_trie = 0;
            o = (o + 15) & ~(size_t)15;
            Y.off_sym = (int)o;   o += (size_t)Y.lz_lanes * A.npad;
            o = (o + 15) & ~(size_t)15;
            Y.off_xs = (int)o;    o += (size_t)A.npad * 4;
            per = (o + 15) & ~(size_t)15;
            if (per <= 6912) break;
        }
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
    // up to TSFX_SHORT_L_MAX samples the table has at most 2^15 slots, so a slot id and a 16-bit symbol pack into one
    // uint32 key; longer series take uint64 keys (at TSFX_L_MAX: 2^18 slots, 2 MB per Lempel-Ziv lane)
    Y.wide = max_len > TSFX_SHORT_L_MAX;
    Y.lz_stride = (Y.wide ? 4 : 2) * Y.lz_hash;   // uint16 units per lane
    size_t off = 0;
    Y.off_codes = (int)off; off += A.need_perm ? (size_t)Y.npow2 * 4 : 0;
    off = (off + 7) & ~(size_t)7;
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
