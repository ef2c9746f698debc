// tsfx_warp_sort.cuh -- bitonic sort of 256 keys held in the registers of one warp (ENTROPY's rank space, SEQ's
// permutation patterns).
#pragma once

#include "tsfx_common.cuh"

namespace tsfx {

// Lane L holds positions 8L .. 8L + 7: strides below 8 run inside the lane's registers, the larger ones by shuffle.
// Ascending; keys that compare equal are indistinguishable, so the sorted sequence is the one any sorting network gives.
template <typename K>
__device__ __forceinline__ void cmpx_regs(K (&v)[8], int e, int f, bool up) {
    const K a = v[e], c = v[f];
    if ((a > c) == up) { v[e] = c; v[f] = a; }
}
template <typename K>
__device__ __forceinline__ void warp_sort256(K (&v)[8], int lane) {
#pragma unroll
    for (int k = 2; k <= 8; k <<= 1) {                 // blocks of 8 inside the lane (direction from position 8L + e)
#pragma unroll
        for (int j = k >> 1; j > 0; j >>= 1) {
#pragma unroll
            for (int e = 0; e < 8; ++e)
                if (!(e & j)) cmpx_regs(v, e, e | j, ((8 * lane + e) & k) == 0);
        }
    }
#pragma unroll 1
    for (int k = 16; k <= 256; k <<= 1) {              // from here the direction is the lane's
        const bool up = (lane & (k >> 3)) == 0;
#pragma unroll 1
        for (int jl = k >> 4; jl > 0; jl >>= 1) {      // strides 8 jl: partner lane ^ jl
            const bool keep_min = up != ((lane & jl) != 0);
#pragma unroll
            for (int e = 0; e < 8; ++e) {
                const K o = __shfl_xor_sync(FULL, v[e], jl);
                v[e] = keep_min ? (o < v[e] ? o : v[e]) : (o > v[e] ? o : v[e]);
            }
        }
#pragma unroll
        for (int j = 4; j > 0; j >>= 1) {
#pragma unroll
            for (int e = 0; e < 8; ++e)
                if (!(e & j)) cmpx_regs(v, e, e | j, up);
        }
    }
}

}  // namespace tsfx
