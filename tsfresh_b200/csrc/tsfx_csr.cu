// tsfx_csr.cu -- device CSR build (stage (a) of the hot path); see tsfx_csr.h.
#include <cub/cub.cuh>
#include <thrust/iterator/counting_iterator.h>
#include <thrust/iterator/transform_iterator.h>
#include <algorithm>

#include "../../include/tsfx.h"
#include "tsfx_csr.h"

namespace tsfx {

enum { S_IDS = 0, S_KEYS, S_VALS, S_PERM_A, S_PERM_B, S_KEY_A, S_KEY_B, S_TEMP, S_FLAG, S_OUT_UID, S_OUT_BEGIN, S_OUT_LEN, S_IDS_SORTED };

cudaError_t CsrWorkspace::reserve(int slot, size_t bytes) {
    if (bytes <= caps[slot]) return cudaSuccess;
    if (bufs[slot]) cudaFree(bufs[slot]);
    bufs[slot] = nullptr;
    caps[slot] = 0;
    cudaError_t e = cudaMalloc(&bufs[slot], bytes);
    if (e == cudaSuccess) caps[slot] = bytes;
    return e;
}
cudaError_t CsrWorkspace::init_info() {
    if (h_info) return cudaSuccess;
    cudaError_t e = cudaHostAlloc((void**)&h_info, sizeof(CsrInfo), cudaHostAllocDefault);
    if (e != cudaSuccess) return e;
    e = cudaMalloc((void**)&d_info, sizeof(CsrInfo));
    return e;
}
void CsrWorkspace::release() {
    for (int i = 0; i < 16; ++i) { if (bufs[i]) cudaFree(bufs[i]); bufs[i] = nullptr; caps[i] = 0; }
    if (h_info) cudaFreeHost(h_info);
    if (d_info) cudaFree(d_info);
    h_info = nullptr; d_info = nullptr;
    d_uid = nullptr; d_begin = nullptr; d_len = nullptr; d_values = nullptr;
}

__device__ __forceinline__ uint64_t key_i64(int64_t v) { return (uint64_t)v ^ 0x8000000000000000ull; }
__device__ __forceinline__ uint64_t key_f64(uint64_t b) { return (b & 0x8000000000000000ull) ? ~b : (b | 0x8000000000000000ull); }

__global__ void k_check_sorted_ids(const int64_t* __restrict__ ids, int64_t n, CsrInfo* info) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    int bad = 0;
    for (; i + 1 < n; i += stride) bad |= ids[i] > ids[i + 1];
    if (__any_sync(0xffffffffu, bad) && (threadIdx.x & 31) == 0) atomicOr(&info->unsorted_ids, 1);
}

// pairs (i-1, i), i in [max(lo,1), hi): same id and decreasing key -> unsorted_keys; NaN value in [lo, hi) -> has_nan
__global__ void k_check_rows(const int64_t* __restrict__ ids, const uint64_t* __restrict__ keys, int is_f64,
                             const float* __restrict__ values, int64_t lo, int64_t hi, int check_nan, CsrInfo* info) {
    int64_t i = lo + (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    int badk = 0, nan = 0;
    for (; i < hi; i += stride) {
        if (keys && i > 0 && ids[i - 1] == ids[i]) {
            uint64_t ka = keys[i - 1], kb = keys[i];
            if (is_f64) { ka = key_f64(ka); kb = key_f64(kb); } else { ka = key_i64((int64_t)ka); kb = key_i64((int64_t)kb); }
            badk |= ka > kb;
        }
        if (check_nan) { const float v = values[i]; nan |= v != v; }
    }
    if (__any_sync(0xffffffffu, badk) && (threadIdx.x & 31) == 0) atomicOr(&info->unsorted_keys, 1);
    if (__any_sync(0xffffffffu, nan) && (threadIdx.x & 31) == 0) atomicOr(&info->has_nan, 1);
}

__global__ void k_check_nan(const float* __restrict__ values, int64_t n, CsrInfo* info) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    int nan = 0;
    for (; i < n; i += stride) { const float v = values[i]; nan |= v != v; }
    if (__any_sync(0xffffffffu, nan) && (threadIdx.x & 31) == 0) atomicOr(&info->has_nan, 1);
}

// One warp per view: bounds and length of the view, then its samples (coalesced) for NaN.  Views may overlap (rolled
// windows), so the scan follows the views rather than the value array: a NaN no series covers is not an error.
__global__ void k_check_views(const float* __restrict__ values, int64_t n_values, const int64_t* __restrict__ begin,
                              const int32_t* __restrict__ len, int64_t n_series, CsrInfo* info) {
    const int lane = threadIdx.x & 31;
    int64_t w = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t n_warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    int mx = 0, nan = 0;
    for (; w < n_series; w += n_warps) {                  // warp-uniform
        const int64_t b = begin[w];
        const int32_t l = len[w];
        if (l < 1 || b < 0 || b > n_values - l) {
            if (lane == 0) atomicMax((unsigned long long*)&info->bad_view_rev, (unsigned long long)(n_series - w));
            continue;
        }
        mx = max(mx, (int)l);
        for (int32_t i = lane; i < l; i += 32) { const float v = values[b + i]; nan |= v != v; }
    }
    if (lane == 0 && mx > 0) atomicMax(&info->max_len, mx);
    if (__any_sync(0xffffffffu, nan) && lane == 0) atomicOr(&info->has_nan, 1);
}

// len[s] = begin[s+1] - begin[s] (begin[n_series] = n_rows), longest series, row-block boundaries
__global__ void k_len_info(const int64_t* __restrict__ begin, const int* __restrict__ d_nruns, int64_t n_rows,
                           int32_t* __restrict__ len, int64_t min_block, int max_blocks, CsrInfo* info) {
    const int64_t ns = *d_nruns;
    int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    int mx = 0;
    for (; s < ns; s += stride) {
        const int64_t e = (s + 1 < ns) ? begin[s + 1] : n_rows;
        const int64_t l = e - begin[s];
        len[s] = (int32_t)l;
        mx = max(mx, (int)min(l, (int64_t)0x7fffffff));
    }
    mx = __reduce_max_sync(0xffffffffu, mx);
    if ((threadIdx.x & 31) == 0 && mx > 0) atomicMax(&info->max_len, mx);
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        info->n_series = ns;
        int64_t blk = (ns + max_blocks - 1) / max_blocks;
        if (blk < min_block) blk = min_block;
        if (blk < 1) blk = 1;
        int nb = 0;
        for (int64_t lo = 0; lo < ns && nb < TSFX_CSR_MAX_BLOCKS; lo += blk, ++nb) {
            info->series_lo[nb] = lo;
            info->row_lo[nb] = begin[lo];
        }
        info->series_lo[nb] = ns;
        info->row_lo[nb] = n_rows;
        info->n_blocks = nb;
    }
}

__global__ void k_make_keys(const uint64_t* raw, int is_f64, int64_t n, uint64_t* key, uint32_t* perm) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; i < n; i += stride) {
        if (key) key[i] = is_f64 ? key_f64(raw[i]) : key_i64((int64_t)raw[i]);
        perm[i] = (uint32_t)i;
    }
}
__global__ void k_gather_id_keys(const int64_t* ids, const uint32_t* perm, int64_t n, uint64_t* key) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; i < n; i += stride) key[i] = key_i64(ids[perm[i]]);
}
__global__ void k_gather_final(const uint64_t* idkey_sorted, const float* values, const uint32_t* perm, int64_t n,
                               int64_t* ids_out, float* vals_out) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; i < n; i += stride) {
        ids_out[i] = (int64_t)(idkey_sorted[i] ^ 0x8000000000000000ull);
        vals_out[i] = values[perm[i]];
    }
}

#define CKE(call, what)                                                                    \
    do {                                                                                   \
        cudaError_t e__ = (call);                                                          \
        if (e__ != cudaSuccess) {                                                          \
            if (msg) *msg = std::string(what) + ": " + cudaGetErrorString(e__);           \
            return TSFX_E_CUDA;                                                            \
        }                                                                                  \
    } while (0)

static inline int grid_for(int64_t n, int threads) { return (int)std::max<int64_t>(1, std::min<int64_t>((n + threads - 1) / threads, 132 * 16)); }   // grid-stride, 16 CTAs per SM of an H100

// unique ids + begin offsets + lengths + info from ids that are non-decreasing (garbage otherwise: the caller checks
// info.unsorted_ids first)
static int csr_from_sorted_ids(CsrWorkspace& W, const int64_t* d_ids_sorted, int64_t n, int64_t min_block, int max_blocks,
                               cudaStream_t st, std::string* msg) {
    CKE(W.reserve(S_OUT_UID, n * 8), "alloc uid");
    CKE(W.reserve(S_OUT_BEGIN, n * 8 + 8), "alloc begin");
    CKE(W.reserve(S_OUT_LEN, n * 4 + 64), "alloc len");
    CKE(W.reserve(S_FLAG, 64), "alloc flag");
    W.d_uid = (int64_t*)W.bufs[S_OUT_UID];
    W.d_begin = (int64_t*)W.bufs[S_OUT_BEGIN];
    W.d_len = (int32_t*)W.bufs[S_OUT_LEN];
    int* d_nruns = (int*)W.bufs[S_FLAG];
    thrust::counting_iterator<int64_t> rows(0);
    size_t tb = 0;
    CKE(cub::DeviceSelect::UniqueByKey(nullptr, tb, d_ids_sorted, rows, W.d_uid, W.d_begin, d_nruns, (int)n, st), "unique size");
    CKE(W.reserve(S_TEMP, tb), "alloc temp");
    CKE(cub::DeviceSelect::UniqueByKey(W.bufs[S_TEMP], tb, d_ids_sorted, rows, W.d_uid, W.d_begin, d_nruns, (int)n, st), "unique by key");
    k_len_info<<<grid_for(n / 64 + 1, 256), 256, 0, st>>>(W.d_begin, d_nruns, n, W.d_len, min_block, max_blocks, W.d_info);
    CKE(cudaGetLastError(), "len kernel");
    return TSFX_OK;
}

__global__ void k_gather_i64(const int64_t* __restrict__ src, const uint32_t* __restrict__ perm, int64_t n, int64_t* __restrict__ dst) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; i < n; i += stride) dst[i] = src[perm[i]];
}
__global__ void k_gather_f32(const float* __restrict__ src, const uint32_t* __restrict__ perm, int64_t n, float* __restrict__ dst) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; i < n; i += stride) dst[i] = src[perm[i]];
}
void csr_gather_f32(CsrWorkspace& W, const float* src, float* dst, int64_t n, cudaStream_t st) {
    if (n > 0 && W.d_perm) k_gather_f32<<<grid_for(n, 256), 256, 0, st>>>(src, W.d_perm, n, dst);
}
void csr_gather_i64(CsrWorkspace& W, const int64_t* src, int64_t* dst, int64_t n, cudaStream_t st) {
    if (n > 0 && W.d_perm) k_gather_i64<<<grid_for(n, 256), 256, 0, st>>>(src, W.d_perm, n, dst);
}

int csr_ids_pass(CsrWorkspace& W, const int64_t* d_ids, int64_t n, int64_t min_block, int max_blocks, cudaStream_t st,
                 std::string* msg) {
    W.d_perm = nullptr;
    if (n >= (int64_t)1 << 31) { if (msg) *msg = "more than 2^31-1 rows in one call"; return TSFX_E_UNSUPPORTED; }
    CKE(W.init_info(), "alloc info");
    CKE(cudaMemsetAsync(W.d_info, 0, sizeof(CsrInfo), st), "memset info");
    k_check_sorted_ids<<<grid_for(n, 256), 256, 0, st>>>(d_ids, n, W.d_info);
    int rc = csr_from_sorted_ids(W, d_ids, n, min_block, max_blocks, st, msg);
    if (rc) return rc;
    CKE(cudaMemcpyAsync(W.h_info, W.d_info, sizeof(CsrInfo), cudaMemcpyDeviceToHost, st), "D2H info");
    return TSFX_OK;
}

void csr_check_rows(CsrWorkspace& W, const int64_t* d_ids, const uint64_t* d_keys, int is_f64, const float* d_values,
                    int64_t row_lo, int64_t row_hi, bool check_nan, cudaStream_t st) {
    if (row_hi <= row_lo || (!d_keys && !check_nan)) return;
    k_check_rows<<<grid_for(row_hi - row_lo, 256), 256, 0, st>>>(d_ids, d_keys, is_f64, d_values, row_lo, row_hi, check_nan ? 1 : 0, W.d_info);
}

void csr_check_nan(CsrWorkspace& W, const float* d_values, int64_t n, cudaStream_t st) {
    if (n <= 0) return;
    k_check_nan<<<grid_for(n, 256), 256, 0, st>>>(d_values, n, W.d_info);
}

void csr_check_views(CsrWorkspace& W, const float* d_values, int64_t n_values, const int64_t* d_begin, const int32_t* d_len,
                     int64_t n_series, cudaStream_t st) {
    if (n_series <= 0) return;
    k_check_views<<<grid_for(n_series * 32, 256), 256, 0, st>>>(d_values, n_values, d_begin, d_len, n_series, W.d_info);
}

int csr_sort_pass(CsrWorkspace& W, const int64_t* d_ids, const uint64_t* d_keys, int is_f64, const float* d_values,
                  int64_t n, int64_t min_block, int max_blocks, bool check_nan, cudaStream_t st, std::string* msg) {
    const int threads = 256;
    const int blocks = grid_for(n, threads);
    CKE(W.init_info(), "alloc info");
    CKE(cudaMemsetAsync(W.d_info, 0, sizeof(CsrInfo), st), "memset info");
    if (check_nan) csr_check_nan(W, d_values, n, st);
    CKE(W.reserve(S_PERM_A, n * 4), "alloc perm");
    CKE(W.reserve(S_PERM_B, n * 4), "alloc perm");
    CKE(W.reserve(S_KEY_A, n * 8), "alloc key");
    CKE(W.reserve(S_KEY_B, n * 8), "alloc key");
    CKE(W.reserve(S_IDS_SORTED, n * 8), "alloc ids sorted");
    uint32_t *pa = (uint32_t*)W.bufs[S_PERM_A], *pb = (uint32_t*)W.bufs[S_PERM_B];
    uint64_t *ka = (uint64_t*)W.bufs[S_KEY_A], *kb = (uint64_t*)W.bufs[S_KEY_B];
    size_t tb = 0;
    CKE(cub::DeviceRadixSort::SortPairs(nullptr, tb, ka, kb, pa, pb, (int)n, 0, 64, st), "radix size");
    CKE(W.reserve(S_TEMP, tb), "alloc temp");
    const uint32_t* perm = pa;
    k_make_keys<<<blocks, threads, 0, st>>>(d_keys, is_f64, n, d_keys ? ka : nullptr, pa);
    if (d_keys) {      // pass A: stable sort of row indices by sort key
        CKE(cub::DeviceRadixSort::SortPairs(W.bufs[S_TEMP], tb, ka, kb, pa, pb, (int)n, 0, 64, st), "radix sort A");
        perm = pb;
    }
    // pass B: stable sort by id, carrying the pass-A order
    k_gather_id_keys<<<blocks, threads, 0, st>>>(d_ids, perm, n, ka);
    uint32_t* perm_out = (perm == pa) ? pb : pa;
    CKE(cub::DeviceRadixSort::SortPairs(W.bufs[S_TEMP], tb, ka, kb, perm, perm_out, (int)n, 0, 64, st), "radix sort B");
    // gather: sorted ids, sorted values (into pass-A key storage, free by now)
    k_gather_final<<<blocks, threads, 0, st>>>(kb, d_values, perm_out, n, (int64_t*)W.bufs[S_IDS_SORTED], (float*)ka);
    W.d_values = (float*)ka;
    W.d_perm = perm_out;
    int rc = csr_from_sorted_ids(W, (const int64_t*)W.bufs[S_IDS_SORTED], n, min_block, max_blocks, st, msg);
    if (rc) return rc;
    CKE(cudaMemcpyAsync(W.h_info, W.d_info, sizeof(CsrInfo), cudaMemcpyDeviceToHost, st), "D2H info");
    return TSFX_OK;
}

int csr_max_len(CsrWorkspace& W, const int32_t* d_len, int64_t n, cudaStream_t st, int* out) {
    std::string* msg = nullptr;
    CKE(W.reserve(S_FLAG, 64), "alloc");
    int* d_out = (int*)W.bufs[S_FLAG] + 8;
    size_t tb = 0;
    CKE(cub::DeviceReduce::Max(nullptr, tb, d_len, d_out, (int)n, st), "max size");
    CKE(W.reserve(S_TEMP, tb), "alloc temp");
    CKE(cub::DeviceReduce::Max(W.bufs[S_TEMP], tb, d_len, d_out, (int)n, st), "max");
    CKE(cudaMemcpyAsync(out, d_out, sizeof(int), cudaMemcpyDeviceToHost, st), "D2H");
    CKE(cudaStreamSynchronize(st), "sync");
    return TSFX_OK;
}

}  // namespace tsfx
