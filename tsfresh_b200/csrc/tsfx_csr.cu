// tsfx_csr.cu -- device CSR build (stage (a) of the hot path); see tsfx_csr.h.
#include <cub/cub.cuh>
#include <thrust/iterator/counting_iterator.h>
#include <thrust/iterator/transform_iterator.h>
#include <algorithm>
#include <cstddef>

#include "../../include/tsfx.h"
#include "tsfx_csr.h"
#include "tsfx_roll.cuh"

namespace tsfx {

enum { S_IDS = 0, S_KEYS, S_VALS, S_PERM_A, S_PERM_B, S_KEY_A, S_KEY_B, S_TEMP, S_FLAG, S_OUT_UID, S_OUT_BEGIN, S_OUT_LEN, S_IDS_SORTED };

cudaError_t CsrWorkspace::reserve(int slot, size_t bytes) {
    if (bytes <= caps[slot]) return cudaSuccess;
    if (frozen) return cudaErrorMemoryAllocation;
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

// Stable sort of the row index by (id, sort key) (sort key nullptr: by id alone): *perm_out = input row of every sorted
// row, and S_KEY_B holds the sorted ids as ordered keys (key_i64).
// the buffers of sort_rows over n rows; *tb = the radix sort's temporary storage
static int sort_reserve(CsrWorkspace& W, int64_t n, size_t* tb, cudaStream_t st, std::string* msg) {
    CKE(W.reserve(S_PERM_A, n * 4), "alloc perm");
    CKE(W.reserve(S_PERM_B, n * 4), "alloc perm");
    CKE(W.reserve(S_KEY_A, n * 8), "alloc key");
    CKE(W.reserve(S_KEY_B, n * 8), "alloc key");
    uint32_t *pa = (uint32_t*)W.bufs[S_PERM_A], *pb = (uint32_t*)W.bufs[S_PERM_B];
    uint64_t *ka = (uint64_t*)W.bufs[S_KEY_A], *kb = (uint64_t*)W.bufs[S_KEY_B];
    *tb = 0;
    CKE(cub::DeviceRadixSort::SortPairs(nullptr, *tb, ka, kb, pa, pb, (int)n, 0, 64, st), "radix size");
    CKE(W.reserve(S_TEMP, *tb), "alloc temp");
    return TSFX_OK;
}

static int sort_rows(CsrWorkspace& W, const int64_t* d_ids, const uint64_t* d_keys, int is_f64, int64_t n, cudaStream_t st,
                     std::string* msg, uint32_t** perm_out_) {
    const int threads = 256;
    const int blocks = grid_for(n, threads);
    size_t tb = 0;
    if (int rc = sort_reserve(W, n, &tb, st, msg)) return rc;
    uint32_t *pa = (uint32_t*)W.bufs[S_PERM_A], *pb = (uint32_t*)W.bufs[S_PERM_B];
    uint64_t *ka = (uint64_t*)W.bufs[S_KEY_A], *kb = (uint64_t*)W.bufs[S_KEY_B];
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
    *perm_out_ = perm_out;
    return TSFX_OK;
}

int csr_sort_pass(CsrWorkspace& W, const int64_t* d_ids, const uint64_t* d_keys, int is_f64, const float* d_values,
                  int64_t n, int64_t min_block, int max_blocks, bool check_nan, cudaStream_t st, std::string* msg) {
    const int threads = 256;
    const int blocks = grid_for(n, threads);
    CKE(W.init_info(), "alloc info");
    CKE(cudaMemsetAsync(W.d_info, 0, sizeof(CsrInfo), st), "memset info");
    if (check_nan) csr_check_nan(W, d_values, n, st);
    uint32_t* perm_out = nullptr;
    if (int rc = sort_rows(W, d_ids, d_keys, is_f64, n, st, msg, &perm_out)) return rc;
    CKE(W.reserve(S_IDS_SORTED, n * 8), "alloc ids sorted");
    uint64_t *ka = (uint64_t*)W.bufs[S_KEY_A], *kb = (uint64_t*)W.bufs[S_KEY_B];
    // gather: sorted ids, sorted values (into pass-A key storage, free by now)
    k_gather_final<<<blocks, threads, 0, st>>>(kb, d_values, perm_out, n, (int64_t*)W.bufs[S_IDS_SORTED], (float*)ka);
    W.d_values = (float*)ka;
    W.d_perm = perm_out;
    int rc = csr_from_sorted_ids(W, (const int64_t*)W.bufs[S_IDS_SORTED], n, min_block, max_blocks, st, msg);
    if (rc) return rc;
    CKE(cudaMemcpyAsync(W.h_info, W.d_info, sizeof(CsrInfo), cudaMemcpyDeviceToHost, st), "D2H info");
    return TSFX_OK;
}

// ---------------------------------------------------------------------------------------------------------------------
// stacked long format (tsfx_csr.h)
enum { T_CODE = 0, T_UROW, T_COUNTS, T_TEMP, T_VALS, T_SROW, T_TIMES, T_BEGIN, T_LEN, T_ROW, T_UID, T_INFO, T_KEYS,
       // stacked_roll / stacked_sub: per-series piece offsets, per-piece (window or package) begin / len / union row /
       // parent id / name key, scanned name flags, union pieces' names
       G_OFF, G_BEGIN, G_LEN, G_ROW, G_ID, G_KEY, G_SCAN, G_UID, G_UKEY,
       // stacked_sub: begin / len / union row of every package in union order inside its kind
       P_BEGIN, P_LEN, P_ROW,
       // input row number of every staged row; stacked_roll with forecast: target row of every window and union window
       T_SRC, R_TGT, R_UTGT, T_SLOTS };
static_assert(T_SLOTS <= 32, "StackedWorkspace::bufs");

cudaError_t StackedWorkspace::reserve(int slot, size_t bytes) {
    if (bytes <= caps[slot]) return cudaSuccess;
    if (frozen) return cudaErrorMemoryAllocation;
    if (bufs[slot]) cudaFree(bufs[slot]);
    bufs[slot] = nullptr;
    caps[slot] = 0;
    cudaError_t e = cudaMalloc(&bufs[slot], bytes);
    if (e == cudaSuccess) caps[slot] = bytes;
    return e;
}
cudaError_t StackedWorkspace::keep_ids(const int64_t* d_src, int64_t n, cudaStream_t st) {
    cudaError_t e = reserve(T_UID, std::max<size_t>((size_t)n * 8, 8));
    if (e != cudaSuccess) return e;
    d_uid = (int64_t*)bufs[T_UID];
    return cudaMemcpyAsync(d_uid, d_src, (size_t)n * 8, cudaMemcpyDeviceToDevice, st);
}
void StackedWorkspace::release() {
    for (int i = 0; i < T_SLOTS; ++i) { if (bufs[i]) cudaFree(bufs[i]); bufs[i] = nullptr; caps[i] = 0; }
    if (h_info) cudaFreeHost(h_info);
    h_info = nullptr; d_info = nullptr;
    d_values = nullptr; d_times = nullptr; d_begin = nullptr; d_len = nullptr; d_row = nullptr; d_uid = nullptr;
    d_keys = nullptr; d_ukey = nullptr; d_src = nullptr; d_utarget = nullptr;
    staged = Staged::Rows; pending = false;
}

// the device's sizes and flags (d_info) to the host's copy (h_info), asynchronously: the caller synchronises
static int stacked_publish(StackedWorkspace& S, cudaStream_t st, std::string* msg) {
    CKE(cudaMemcpyAsync(S.h_info, S.d_info, sizeof(StackedInfo), cudaMemcpyDeviceToHost, st), "D2H info");
    return TSFX_OK;
}

#define STACK_TILE 4096          // rows per CTA of the counting sort
#define STACK_THREADS 256
#define STACK_NO_KIND 0xFFu

// Counting-sort histogram over the rows in CSR order: kind code of every row (STACK_NO_KIND when out of range), rows per
// (kind, tile) into counts[k * n_tiles + tile]; NaN float64 sort keys (input order) are flagged on the way.  n_live
// (deferred stage; nullptr: every row counts): input rows from *n_live on are STACK_NO_KIND too, without a flag.
__global__ void __launch_bounds__(STACK_THREADS) k_stack_count(const uint32_t* __restrict__ perm, const void* kinds, int kinds_i64,
                                                               int n_kinds, const uint64_t* __restrict__ keys_f64, int64_t n,
                                                               uint8_t* __restrict__ code, int* __restrict__ counts, StackedInfo* info,
                                                               const int64_t* __restrict__ n_live) {
    __shared__ int hist[TSFX_MAX_KINDS];
    for (int k = threadIdx.x; k < TSFX_MAX_KINDS; k += blockDim.x) hist[k] = 0;
    __syncthreads();
    const int64_t lo = (int64_t)blockIdx.x * STACK_TILE, hi = min(lo + STACK_TILE, n);
    const int64_t live = n_live ? *n_live : n;
    int bad = 0, nan = 0;
    for (int64_t i = lo + threadIdx.x; i < hi; i += blockDim.x) {
        const uint32_t src = perm[i];
        const bool dropped = (int64_t)src >= live;
        int64_t c = 0;
        if (kinds && !dropped) c = kinds_i64 ? ((const int64_t*)kinds)[src] : (int64_t)((const int32_t*)kinds)[src];
        const bool ok = !dropped && c >= 0 && c < n_kinds;
        code[i] = ok ? (uint8_t)c : (uint8_t)STACK_NO_KIND;
        if (ok) atomicAdd(&hist[c], 1);
        bad |= !ok && !dropped;
        if (keys_f64) { const double v = __longlong_as_double((long long)keys_f64[i]); nan |= v != v; }
    }
    if (__any_sync(0xffffffffu, bad) && (threadIdx.x & 31) == 0) atomicOr(&info->bad_kind, 1);
    if (__any_sync(0xffffffffu, nan) && (threadIdx.x & 31) == 0) atomicOr(&info->nan_keys, 1);
    __syncthreads();
    for (int k = threadIdx.x; k < n_kinds; k += blockDim.x) counts[(int64_t)k * gridDim.x + blockIdx.x] = hist[k];
}

// Stable scatter of the counting sort: each tile walks its rows in order, 256 at a time; a row's destination is its
// kind's running base in this tile + the rows of that kind in earlier warps of the step + its rank among its warp's
// rows of the same kind (__match_any_sync).  Gathers the value (already in CSR order), the union row, the time, the
// sort key and the input row number (the last three when asked for).
__global__ void __launch_bounds__(STACK_THREADS) k_stack_scatter(const uint8_t* __restrict__ code, const int* __restrict__ offs,
                                                                 int n_kinds, int64_t n, const float* __restrict__ vals,
                                                                 const int32_t* __restrict__ urow, const int64_t* __restrict__ times,
                                                                 const uint64_t* __restrict__ keys,
                                                                 const uint32_t* __restrict__ perm, const StackedInfo* info,
                                                                 float* __restrict__ out_vals, int32_t* __restrict__ out_row,
                                                                 int64_t* __restrict__ out_times, uint64_t* __restrict__ out_keys,
                                                                 uint32_t* __restrict__ out_src) {
    constexpr int W = STACK_THREADS / 32;
    __shared__ int64_t base[TSFX_MAX_KINDS];
    __shared__ int cnt[W][TSFX_MAX_KINDS];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int k = threadIdx.x; k < n_kinds; k += blockDim.x)        // the scan packs the kinds; their starts are aligned
        base[k] = offs[(int64_t)k * gridDim.x + blockIdx.x] - offs[(int64_t)k * gridDim.x] + info->kind_row[k];
    const int64_t lo = (int64_t)blockIdx.x * STACK_TILE, hi = min(lo + STACK_TILE, n);
    for (int64_t c0 = lo; c0 < hi; c0 += STACK_THREADS) {
        for (int j = threadIdx.x; j < W * TSFX_MAX_KINDS; j += blockDim.x) (&cnt[0][0])[j] = 0;
        __syncthreads();
        const int64_t i = c0 + threadIdx.x;
        const unsigned k = i < hi ? code[i] : STACK_NO_KIND;
        const unsigned peers = __match_any_sync(0xffffffffu, k);
        const int rank = __popc(peers & ((1u << lane) - 1));
        if (k != STACK_NO_KIND && rank == 0) cnt[warp][k] = __popc(peers);
        __syncthreads();
        if (k != STACK_NO_KIND) {
            int64_t dst = base[k] + rank;
            for (int w = 0; w < warp; ++w) dst += cnt[w][k];
            out_vals[dst] = vals[i];
            out_row[dst] = urow[i];
            if (times) out_times[dst] = times[perm[i]];
            if (keys) out_keys[dst] = keys[perm[i]];
            if (out_src) out_src[dst] = perm[i];
        }
        __syncthreads();
        for (int kk = threadIdx.x; kk < n_kinds; kk += blockDim.x) {
            int add = 0;
            for (int w = 0; w < W; ++w) add += cnt[w][kk];
            base[kk] += add;
        }
        __syncthreads();
    }
}

// rows and aligned first row of every kind
__global__ void k_stack_kind_rows(const int* __restrict__ offs, int n_kinds, int n_tiles, StackedInfo* info) {
    int64_t at = 0;
    for (int k = 0; k < n_kinds; ++k) {
        const int64_t rows = offs[(int64_t)(k + 1) * n_tiles] - offs[(int64_t)k * n_tiles];
        info->kind_row[k] = at;
        info->kind_rows[k] = rows;
        at += (rows + TSFX_STACK_ALIGN - 1) / TSFX_STACK_ALIGN * TSFX_STACK_ALIGN;
    }
    info->kind_row[n_kinds] = at;
}

// kind whose aligned row range holds partitioned row j (the last of kinds that start at the same row is the only one
// that can have rows)
__device__ __forceinline__ int kind_at(const StackedInfo* info, int n_kinds, int64_t j) {
    int lo = 0, hi = n_kinds;
    while (hi - lo > 1) { const int m = (lo + hi) >> 1; if (info->kind_row[m] <= j) lo = m; else hi = m; }
    return lo;
}

// 1 where row i of the sorted ids starts a new id (row 0 excluded): the inclusive scan is the union row of every row
struct IdChange {
    const int64_t* ids;
    __device__ int operator()(int64_t i) const { return i > 0 && ids[i] != ids[i - 1]; }
};

// 1 where partitioned row j starts a series: the first row of a kind, or a new union row (0 in the alignment gaps)
struct SeriesStart {
    const int32_t* row;
    const StackedInfo* info;
    int n_kinds;
    __device__ int operator()(int64_t j) const {
        if (j >= info->kind_row[n_kinds]) return 0;
        const int k = kind_at(info, n_kinds, j);
        if (j >= info->kind_row[k] + info->kind_rows[k]) return 0;
        return j == info->kind_row[k] || row[j] != row[j - 1];
    }
};

__global__ void k_stack_series(const int32_t* __restrict__ sidx, SeriesStart start, int64_t n, int64_t* __restrict__ begin,
                               int32_t* __restrict__ series_row) {
    int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; j < n; j += stride)
        if (start(j)) { const int32_t s = sidx[j]; begin[s] = j; series_row[s] = start.row[j]; }
}

// series lengths, each kind's first series and longest series
__global__ void k_stack_lengths(const int32_t* __restrict__ sidx, int64_t n, int n_kinds, const int64_t* __restrict__ begin,
                                int32_t* __restrict__ len, StackedInfo* info) {
    __shared__ int mx[TSFX_MAX_KINDS];
    for (int k = threadIdx.x; k < n_kinds; k += blockDim.x) mx[k] = 0;
    __syncthreads();
    const int64_t ns = sidx[n];
    if (blockIdx.x == 0)
        for (int k = threadIdx.x; k <= n_kinds; k += blockDim.x) info->kind_series[k] = sidx[info->kind_row[k]];
    int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; s < ns; s += stride) {
        const int64_t b = begin[s];
        const int k = kind_at(info, n_kinds, b);
        int64_t e = info->kind_row[k] + info->kind_rows[k];
        if (s + 1 < ns) e = min(e, begin[s + 1]);
        const int32_t l = (int32_t)(e - b);
        len[s] = l;
        atomicMax(&mx[k], l);
    }
    __syncthreads();
    for (int k = threadIdx.x; k < n_kinds; k += blockDim.x) if (mx[k]) atomicMax(&info->kind_max_len[k], mx[k]);
}

__global__ void k_stack_finish(const CsrInfo* csr, StackedInfo* info) {
    info->n_union = csr->n_series;
    info->nan_values = csr->has_nan;
}

// the device info of a stage, zeroed
static int stack_info(StackedWorkspace& S, cudaStream_t st, std::string* msg) {
    CKE(S.reserve(T_INFO, sizeof(StackedInfo)), "alloc info");
    S.d_info = (StackedInfo*)S.bufs[T_INFO];
    CKE(cudaMemsetAsync(S.d_info, 0, sizeof(StackedInfo), st), "memset info");
    return TSFX_OK;
}

// The partition's buffers for n rows of n_kinds kinds (row times, kept sort keys and row numbers when asked for) and the
// temporary storage of its three scans (sizes into tb[3]; the scans read the sorted ids at ids_sorted)
static int stack_reserve(StackedWorkspace& S, int64_t n, int n_kinds, bool times, bool keep_keys, bool keep_rows,
                         const int64_t* ids_sorted, size_t* tb, cudaStream_t st, std::string* msg) {
    const int n_tiles = (int)((n + STACK_TILE - 1) / STACK_TILE);
    const int64_t n_pad = n + (int64_t)n_kinds * TSFX_STACK_ALIGN;       // partitioned rows and alignment gaps
    const size_t n_counts = (size_t)n_kinds * n_tiles + 1;
    CKE(S.reserve(T_CODE, n), "alloc codes");
    CKE(S.reserve(T_UROW, (size_t)(n_pad + 1) * 4), "alloc rows");
    CKE(S.reserve(T_COUNTS, n_counts * 4), "alloc counts");
    CKE(S.reserve(T_VALS, (size_t)n_pad * 4), "alloc values");
    CKE(S.reserve(T_SROW, (size_t)n_pad * 4), "alloc rows");
    CKE(S.reserve(T_BEGIN, (size_t)n * 8), "alloc begin");
    CKE(S.reserve(T_LEN, (size_t)n * 4), "alloc len");
    CKE(S.reserve(T_ROW, (size_t)n * 4), "alloc map");
    if (times) CKE(S.reserve(T_TIMES, (size_t)n_pad * 8), "alloc times");
    if (keep_keys) CKE(S.reserve(T_KEYS, (size_t)n_pad * 8), "alloc keys");
    if (keep_rows) CKE(S.reserve(T_SRC, (size_t)n_pad * 4), "alloc row numbers");
    int32_t* urow = (int32_t*)S.bufs[T_UROW];
    int* counts = (int*)S.bufs[T_COUNTS];
    thrust::counting_iterator<int64_t> rows(0);
    auto id_change = thrust::make_transform_iterator(rows, IdChange{ids_sorted});
    auto series_start = thrust::make_transform_iterator(rows, SeriesStart{(int32_t*)S.bufs[T_SROW], S.d_info, n_kinds});
    CKE(cub::DeviceScan::InclusiveSum(nullptr, tb[0], id_change, urow, (int)n, st), "scan size");
    CKE(cub::DeviceScan::ExclusiveSum(nullptr, tb[1], counts, counts, (int)n_counts, st), "scan size");
    CKE(cub::DeviceScan::ExclusiveSum(nullptr, tb[2], series_start, urow, (int)(n_pad + 1), st), "scan size");
    CKE(S.reserve(T_TEMP, std::max(tb[0], std::max(tb[1], tb[2]))), "alloc temp");
    return TSFX_OK;
}

// Deferred stage: the union size, union ids below max_ids and first id past them (stacked_stage_deferred)
struct DeferredUnion {
    const int64_t* n_live;
    int64_t max_ids;
    int64_t* out_ids;
    int64_t* id_past;
};

// Union rows of the live rows [0, *n_live) of the sorted ids (the dropped rows sort after them): the union size into
// info->n_union, the id of union row u into out_ids[u] below max_ids, the id of union row max_ids into *id_past
__global__ void k_defer_union(const int32_t* __restrict__ urow, const int64_t* __restrict__ ids_sorted, int64_t n,
                              DeferredUnion U, StackedInfo* info) {
    const int64_t live = U.n_live ? max((int64_t)0, min(*U.n_live, n)) : n;
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    if (i == 0) info->n_union = live > 0 ? (int64_t)urow[live - 1] + 1 : 0;
    for (; i < live; i += stride)
        if (i == 0 || urow[i] != urow[i - 1]) {
            const int64_t u = urow[i];
            if (u < U.max_ids) U.out_ids[u] = ids_sorted[i];
            else if (u == U.max_ids) *U.id_past = ids_sorted[i];
        }
}

// The sorted rows (W.d_perm, W.d_values, W's sorted ids) partitioned by kind: union rows, the kind counting sort, the
// series' views, union rows and lengths (tsfx_csr.h).  D (deferred stage; nullptr: stacked_stage): the rows from
// *D->n_live on are dropped, and the union is taken from the live rows.
static int stack_partition(StackedWorkspace& S, CsrWorkspace& W, const uint64_t* d_keys, int keys_f64, const void* d_kinds,
                           int kinds_i64, int n_kinds, const int64_t* d_times, int64_t n, bool keep_keys, bool keep_rows,
                           const DeferredUnion* D, cudaStream_t st, std::string* msg) {
    const int n_tiles = (int)((n + STACK_TILE - 1) / STACK_TILE);
    const int64_t n_pad = n + (int64_t)n_kinds * TSFX_STACK_ALIGN;       // partitioned rows and alignment gaps
    const size_t n_counts = (size_t)n_kinds * n_tiles + 1;
    keep_keys = keep_keys && d_keys;
    const int64_t* ids_sorted = (const int64_t*)W.bufs[S_IDS_SORTED];
    size_t tb[3] = {0, 0, 0};
    if (int rc = stack_reserve(S, n, n_kinds, d_times != nullptr, keep_keys, keep_rows, ids_sorted, tb, st, msg)) return rc;
    uint8_t* code = (uint8_t*)S.bufs[T_CODE];
    int32_t* urow = (int32_t*)S.bufs[T_UROW];      // union row of every CSR row; later the series index of every staged row
    int* counts = (int*)S.bufs[T_COUNTS];
    int32_t* srow = (int32_t*)S.bufs[T_SROW];
    S.d_values = (float*)S.bufs[T_VALS];
    S.d_times = d_times ? (int64_t*)S.bufs[T_TIMES] : nullptr;
    S.d_keys = keep_keys ? (uint64_t*)S.bufs[T_KEYS] : nullptr;
    S.d_src = keep_rows ? (uint32_t*)S.bufs[T_SRC] : nullptr;
    S.d_begin = (int64_t*)S.bufs[T_BEGIN];
    S.d_len = (int32_t*)S.bufs[T_LEN];
    S.d_row = (int32_t*)S.bufs[T_ROW];
    thrust::counting_iterator<int64_t> rows(0);
    auto id_change = thrust::make_transform_iterator(rows, IdChange{ids_sorted});
    SeriesStart start{srow, S.d_info, n_kinds};
    auto series_start = thrust::make_transform_iterator(rows, start);
    CKE(cub::DeviceScan::InclusiveSum(S.bufs[T_TEMP], tb[0], id_change, urow, (int)n, st), "union rows");
    if (D) {
        k_defer_union<<<grid_for(n, 256), 256, 0, st>>>(urow, ids_sorted, n, *D, S.d_info);
        CKE(cudaGetLastError(), "union kernel");
    }
    k_stack_count<<<n_tiles, STACK_THREADS, 0, st>>>(W.d_perm, d_kinds, kinds_i64, n_kinds, keys_f64 ? d_keys : nullptr, n,
                                                     code, counts, S.d_info, D ? D->n_live : nullptr);
    CKE(cudaGetLastError(), "kind count kernel");
    CKE(cudaMemsetAsync(counts + n_counts - 1, 0, 4, st), "memset counts");
    CKE(cub::DeviceScan::ExclusiveSum(S.bufs[T_TEMP], tb[1], counts, counts, (int)n_counts, st), "kind offsets");
    k_stack_kind_rows<<<1, 1, 0, st>>>(counts, n_kinds, n_tiles, S.d_info);
    k_stack_scatter<<<n_tiles, STACK_THREADS, 0, st>>>(code, counts, n_kinds, n, W.d_values, urow, d_times,
                                                       keep_keys ? d_keys : nullptr, W.d_perm, S.d_info, S.d_values, srow,
                                                       S.d_times, S.d_keys, S.d_src);
    CKE(cudaGetLastError(), "kind scatter kernel");
    CKE(cub::DeviceScan::ExclusiveSum(S.bufs[T_TEMP], tb[2], series_start, urow, (int)(n_pad + 1), st), "series index");
    k_stack_series<<<grid_for(n_pad, 256), 256, 0, st>>>(urow, start, n_pad, S.d_begin, S.d_row);
    k_stack_lengths<<<grid_for(n / 4 + 1, 256), 256, 0, st>>>(urow, n_pad, n_kinds, S.d_begin, S.d_len, S.d_info);
    CKE(cudaGetLastError(), "series kernels");
    return TSFX_OK;
}

int stacked_stage(StackedWorkspace& S, CsrWorkspace& W, const int64_t* d_ids, const uint64_t* d_keys, int keys_f64,
                  const float* d_values, const void* d_kinds, int kinds_i64, int n_kinds, const int64_t* d_times,
                  int64_t n, bool keep_keys, bool keep_rows, cudaStream_t st, std::string* msg) {
    S.n_kinds = n_kinds;
    S.has_keys = d_keys != nullptr;
    S.keys_f64 = d_keys && keys_f64;
    if (!S.h_info) CKE(cudaHostAlloc((void**)&S.h_info, sizeof(StackedInfo), cudaHostAllocDefault), "alloc info");
    if (int rc = stack_info(S, st, msg)) return rc;
    // stage (a) over every row: (id, sort key) order, union of the ids, NaN scan of the values
    int rc = csr_sort_pass(W, d_ids, d_keys, keys_f64, d_values, n, n, 1, true, st, msg);
    if (rc) return rc;
    rc = stack_partition(S, W, d_keys, keys_f64, d_kinds, kinds_i64, n_kinds, d_times, n, keep_keys, keep_rows, nullptr, st, msg);
    if (rc) return rc;
    k_stack_finish<<<1, 1, 0, st>>>(W.d_info, S.d_info);
    CKE(cudaGetLastError(), "series kernels");
    return stacked_publish(S, st, msg);
}

// Deferred stage: the id and sort-key columns with the rows from *n_live on made to sort after every live row: id
// INT64_MAX and the largest key that is not NaN (int64 INT64_MAX, float64 +inf), so the stable sorts keep them behind the
// live rows with the same id and key.  A live NaN key rejects the call, so its place does not matter.
__global__ void k_defer_rows(const int64_t* __restrict__ ids, const uint64_t* __restrict__ keys, int keys_f64, int64_t n,
                             const int64_t* __restrict__ n_live, int64_t* __restrict__ ids_out, uint64_t* __restrict__ keys_out) {
    const int64_t live = n_live ? *n_live : n;
    const uint64_t last_key = keys_f64 ? 0x7ff0000000000000ull : 0x7fffffffffffffffull;
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; i < n; i += stride) {
        const bool dropped = i >= live;
        ids_out[i] = dropped ? INT64_MAX : ids[i];
        if (keys) keys_out[i] = dropped ? last_key : keys[i];
    }
}

int stacked_defer_reserve(StackedWorkspace& S, CsrWorkspace& W, int64_t n, int n_kinds, std::string* msg) {
    cudaStream_t st = 0;          // size queries only
    CKE(W.reserve(S_IDS, (size_t)n * 8), "alloc ids");
    CKE(W.reserve(S_KEYS, (size_t)n * 8), "alloc keys");
    CKE(W.reserve(S_IDS_SORTED, (size_t)n * 8), "alloc ids sorted");
    size_t tb = 0;
    if (int rc = sort_reserve(W, n, &tb, st, msg)) return rc;
    CKE(S.reserve(T_INFO, sizeof(StackedInfo)), "alloc info");
    S.d_info = (StackedInfo*)S.bufs[T_INFO];
    size_t tbs[3] = {0, 0, 0};
    return stack_reserve(S, n, n_kinds, false, false, false, (const int64_t*)W.bufs[S_IDS_SORTED], tbs, st, msg);
}

int stacked_stage_deferred(StackedWorkspace& S, CsrWorkspace& W, const int64_t* d_ids, const uint64_t* d_keys, int keys_f64,
                           const float* d_values, const void* d_kinds, int kinds_i64, int n_kinds, int64_t n,
                           const int64_t* d_n_live, int64_t max_ids, int64_t* out_ids, int64_t* id_past, cudaStream_t st,
                           std::string* msg) {
    S.n_kinds = n_kinds;
    S.has_keys = d_keys != nullptr;
    S.keys_f64 = d_keys && keys_f64;
    S.d_times = nullptr;
    S.d_keys = nullptr;
    S.d_src = nullptr;
    S.staged = Staged::Rows;
    S.pending = false;
    if (int rc = stack_info(S, st, msg)) return rc;
    if (n == 0) {                         // the zeroed info: no union row, no series (the slots still view the values)
        S.d_values = (float*)S.bufs[T_VALS];
        S.d_begin = (int64_t*)S.bufs[T_BEGIN];
        S.d_len = (int32_t*)S.bufs[T_LEN];
        S.d_row = (int32_t*)S.bufs[T_ROW];
        return TSFX_OK;
    }
    CKE(W.reserve(S_IDS, (size_t)n * 8), "alloc ids");
    if (d_keys) CKE(W.reserve(S_KEYS, (size_t)n * 8), "alloc keys");
    CKE(W.reserve(S_IDS_SORTED, (size_t)n * 8), "alloc ids sorted");
    k_defer_rows<<<grid_for(n, 256), 256, 0, st>>>(d_ids, d_keys, keys_f64, n, d_n_live, W.ids(), W.keys());
    CKE(cudaGetLastError(), "row kernel");
    const uint64_t* keys = d_keys ? W.keys() : nullptr;
    uint32_t* perm = nullptr;
    if (int rc = sort_rows(W, W.ids(), keys, keys_f64, n, st, msg, &perm)) return rc;
    uint64_t *ka = (uint64_t*)W.bufs[S_KEY_A], *kb = (uint64_t*)W.bufs[S_KEY_B];
    k_gather_final<<<grid_for(n, 256), 256, 0, st>>>(kb, d_values, perm, n, (int64_t*)W.bufs[S_IDS_SORTED], (float*)ka);
    CKE(cudaGetLastError(), "gather kernel");
    W.d_values = (float*)ka;
    W.d_perm = perm;
    const DeferredUnion D{d_n_live, max_ids, out_ids, id_past};
    return stack_partition(S, W, keys, keys_f64, d_kinds, kinds_i64, n_kinds, nullptr, n, false, false, &D, st, msg);
}

// kind k's series into the slots [k * max_ids, (k + 1) * max_ids) (stacked_slots)
__global__ void k_defer_slots(const int64_t* __restrict__ begin, const int32_t* __restrict__ len, const int32_t* __restrict__ row,
                              const StackedInfo* info, int n_kinds, int64_t max_ids, int64_t* __restrict__ sbegin,
                              int32_t* __restrict__ slen, int32_t* __restrict__ srow, uint8_t* __restrict__ reject,
                              int64_t* __restrict__ live) {
    const bool whole = info->bad_kind || info->nan_keys || info->n_union > max_ids;
    int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; j < (int64_t)n_kinds * max_ids; j += stride) {
        const int k = (int)(j / max_ids);
        const int64_t i = j - (int64_t)k * max_ids;
        const int64_t s0 = info->kind_series[k];
        const int64_t ns = whole ? 0 : info->kind_series[k + 1] - s0;        // <= n_union <= max_ids
        if (i < ns) {
            sbegin[j] = begin[s0 + i];
            slen[j] = len[s0 + i];
            srow[j] = row[s0 + i];
            reject[j] = 0;
        } else {
            sbegin[j] = 0;
            slen[j] = 1;
            srow[j] = 0;
            reject[j] = DEFER_UNUSED;
        }
        if (i == 0) live[k] = ns;
    }
}

cudaError_t stacked_slots(const StackedWorkspace& S, int n_kinds, int64_t max_ids, int64_t* sbegin, int32_t* slen,
                          int32_t* srow, uint8_t* reject, int64_t* live, cudaStream_t st) {
    k_defer_slots<<<grid_for((int64_t)n_kinds * max_ids, 256), 256, 0, st>>>(S.d_begin, S.d_len, S.d_row, S.d_info, n_kinds,
                                                                             max_ids, sbegin, slen, srow, reject, live);
    return cudaGetLastError();
}

__global__ void k_defer_report(const StackedInfo* info, int64_t max_ids, const int64_t* __restrict__ id_past,
                               const int32_t* __restrict__ srow, int64_t* __restrict__ out_ids, int64_t* n_ids, int64_t* status) {
    const bool over = info->n_union > max_ids;
    const bool whole = info->bad_kind || info->nan_keys || over;
    const int64_t U = whole ? 0 : info->n_union;
    int64_t u = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (u == 0) {                         // one thread: the calls on a status buffer are stream-ordered
        *n_ids = U;
        const int64_t call = status[TSFX_STATUS_CALLS];       // counted by k_defer_finish
        if (whole && status[TSFX_STATUS_BAD] == 0) {
            status[TSFX_STATUS_BAD] = call;
            for (int r = 0; r < 3; ++r) status[TSFX_STATUS_VIEW + r] = -1;
        }
        if (status[TSFX_STATUS_BAD] == call) {
            status[TSFX_STATUS_KIND] = info->bad_kind != 0;
            status[TSFX_STATUS_KEY_NAN] = info->nan_keys != 0;
            status[TSFX_STATUS_IDS] = over ? info->n_union : 0;
            const int64_t s = status[TSFX_STATUS_LONG];
            status[TSFX_STATUS_ID] = over ? *id_past : (!whole && s >= 0) ? out_ids[srow[s]] : -1;
        }
    }
    for (const int64_t stride = (int64_t)gridDim.x * blockDim.x; u < max_ids; u += stride)
        if (u >= U) out_ids[u] = INT64_MAX;
}

cudaError_t stacked_defer_report(const StackedWorkspace& S, int64_t max_ids, const int64_t* id_past, const int32_t* srow,
                                 int64_t* out_ids, int64_t* n_ids, int64_t* status, cudaStream_t st) {
    k_defer_report<<<grid_for(max_ids, 256), 256, 0, st>>>(S.d_info, max_ids, id_past, srow, out_ids, n_ids, status);
    return cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------------------------------
// rolled windows of the staged series (stacked_roll), and the regrouping that fixed-length packages (stacked_sub)
// share with them: pieces of the staged series replace them, named, with a union of the names

// kind whose series range holds series s (the last of kinds that start at the same series is the only one with series)
__device__ __forceinline__ int kind_of_series(const StackedInfo* info, int n_kinds, int64_t s) {
    int lo = 0, hi = n_kinds;
    while (hi - lo > 1) { const int m = (lo + hi) >> 1; if (info->kind_series[m] <= s) lo = m; else hi = m; }
    return lo;
}

// name of the window whose naming row is row r of the series at staged row b: the row's sort key (float64 -0.0 made
// +0.0, which pandas holds equal to it), or r itself without sort keys
__device__ __forceinline__ uint64_t window_name(const uint64_t* __restrict__ keys, int keys_f64, int64_t b, int32_t r) {
    if (!keys) return (uint64_t)r;
    const uint64_t k = keys[b + r];
    return keys_f64 && k == 0x8000000000000000ull ? 0ull : k;
}

// A cut gives the number of pieces of a series of L rows and, in *longest, its longest piece.  Windows: the window
// lengths are monotone in the shift, so a series' longest window is its first or its last; Forecast: every window loses
// its last row.
template <bool Forecast>
struct RollCut {
    RollSpec R;
    __device__ int32_t operator()(int32_t L, int32_t* longest) const {
        int32_t t0, lo;
        const int64_t n = roll_kept(R, L, &t0);
        *longest = 0;
        if (n > 0) {
            const int32_t first = roll_window(R, L, t0, &lo);
            const int32_t last = roll_window(R, L, (int32_t)(t0 + (n - 1) * R.amount), &lo);
            *longest = max(first, last) - (int32_t)Forecast;
        }
        return (int32_t)n;
    }
};

// packages of L rows, the last one shorter
struct SubCut {
    int32_t L;
    __device__ int32_t operator()(int32_t n, int32_t* longest) const {
        *longest = min(n, L);
        return n / L + (n % L != 0);
    }
};

// pieces of every series into cnt[s]; each kind's longest piece into info->kind_max_len (zeroed by the caller)
template <class Cut>
__global__ void k_piece_count(const int32_t* __restrict__ len, int64_t n_series, Cut cut, int n_kinds,
                              int32_t* __restrict__ cnt, StackedInfo* info) {
    __shared__ int mx[TSFX_MAX_KINDS];
    for (int k = threadIdx.x; k < n_kinds; k += blockDim.x) mx[k] = 0;
    __syncthreads();
    int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; s < n_series; s += stride) {
        int32_t longest;
        cnt[s] = cut(len[s], &longest);
        if (longest > 0) atomicMax(&mx[kind_of_series(info, n_kinds, s)], longest);
    }
    __syncthreads();
    for (int k = threadIdx.x; k < n_kinds; k += blockDim.x) if (mx[k]) atomicMax(&info->kind_max_len[k], mx[k]);
}

// 1 when shift u, outside the run of kept shifts, is a window of the roll with min_timeshift given_min_ts and is named
// `name` too
__device__ __forceinline__ int dropped_twin(const RollSpec& R, int32_t L, int64_t u, int32_t given_min_ts,
                                           const uint64_t* __restrict__ keys, int keys_f64, int64_t b, uint64_t name) {
    if (u < R.first || u > L) return 0;
    int32_t lo;
    if (roll_window(R, L, (int32_t)u, &lo) < given_min_ts + 1) return 0;
    return name == window_name(keys, keys_f64, b, (int32_t)(u - 1));
}

// One warp per series, one lane per window: the window's view on the staged values, its parent id and its name.  Two
// windows of one series with the same name (sort keys tied at their naming rows) set info->dup_names.  The slots
// [off[n_series], bound) get the name that sorts after every real one (id INT64_MAX, key 0x7fff...f: the largest
// int64, or a NaN above every float64 key).  Forecast: the view loses its last row, and the window's target is the input
// row number src[] of its naming row, -1 for input row 0.  The reference rolls with the caller's min_timeshift (given_min_ts)
// and only then drops the last rows, so it also names the one-row windows that R.min_ts >= 1 leaves out here (the shift
// before the first kept one, or after the last), and merges such a window with a kept neighbour of the same name: that
// name is flagged too.
template <bool Forecast>
__global__ void k_roll_fill(const int64_t* __restrict__ begin, const int32_t* __restrict__ len, const int32_t* __restrict__ row,
                            const int64_t* __restrict__ uid, const uint64_t* __restrict__ keys, int keys_f64,
                            const int32_t* __restrict__ off, int64_t n_series, int64_t bound, RollSpec R,
                            int64_t* __restrict__ wbegin, int32_t* __restrict__ wlen, int64_t* __restrict__ wid,
                            uint64_t* __restrict__ wkey, StackedInfo* info, const uint32_t* __restrict__ src,
                            int64_t* __restrict__ wtarget, int32_t given_min_ts) {
    const int lane = threadIdx.x & 31;
    int64_t s = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t n_warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    int dup = 0;
    for (; s < n_series; s += n_warps) {                  // warp-uniform
        const int64_t b = begin[s];
        const int32_t L = len[s];
        const int64_t id = uid[row[s]];
        const int32_t o = off[s], n = off[s + 1] - o;
        int32_t t0;
        roll_kept(R, L, &t0);
        for (int32_t j = lane; j < n; j += 32) {
            const int32_t t = (int32_t)(t0 + (int64_t)j * R.amount);
            int32_t lo;
            const int32_t wl = roll_window(R, L, t, &lo);
            const uint64_t name = window_name(keys, keys_f64, b, t - 1);
            wbegin[o + j] = b + lo;
            wlen[o + j] = wl - (int32_t)Forecast;
            wid[o + j] = id;
            wkey[o + j] = name;
            if (Forecast) {
                const uint32_t r = src[b + t - 1];
                wtarget[o + j] = r == 0 ? -1 : (int64_t)r;
            }
            if (j > 0 && keys) dup |= name == window_name(keys, keys_f64, b, t - R.amount - 1);
            if (Forecast && keys) {
                if (j == 0) dup |= dropped_twin(R, L, (int64_t)t - R.amount, given_min_ts, keys, keys_f64, b, name);
                if (j == n - 1) dup |= dropped_twin(R, L, (int64_t)t + R.amount, given_min_ts, keys, keys_f64, b, name);
            }
        }
    }
    if (__any_sync(0xffffffffu, dup) && lane == 0) atomicOr(&info->dup_names, 1);
    int64_t i = off[n_series] + (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    for (const int64_t stride = (int64_t)gridDim.x * blockDim.x; i < bound; i += stride) {
        wid[i] = INT64_MAX;
        wkey[i] = 0x7fffffffffffffffull;
    }
}

// 1 where sorted window i starts a new name (window 0 excluded, the sentinel slots from *n_windows on are 0): the
// inclusive scan is the union row of every sorted window
struct NameChange {
    const int64_t* wid;
    const uint64_t* wkey;
    const uint32_t* perm;
    const int32_t* n_windows;
    __device__ int operator()(int64_t i) const {
        if (i == 0 || i >= *n_windows) return 0;
        const uint32_t a = perm[i - 1], b = perm[i];
        return wid[a] != wid[b] || wkey[a] != wkey[b];
    }
};

// union row of every window, name of every union row, the union size; Forecast: the target of every union row, from its
// first window in name order (the lowest kind's)
template <bool Forecast>
__global__ void k_roll_union(const uint32_t* __restrict__ perm, const int32_t* __restrict__ scan, const int32_t* __restrict__ n_windows,
                             const int64_t* __restrict__ wid, const uint64_t* __restrict__ wkey, int32_t* __restrict__ wrow,
                             int64_t* __restrict__ uid, uint64_t* __restrict__ ukey, StackedInfo* info,
                             const int64_t* __restrict__ wtarget, int64_t* __restrict__ utarget) {
    const int64_t nw = *n_windows;
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    if (i == 0) info->n_union = nw > 0 ? (int64_t)scan[nw - 1] + 1 : 0;
    for (; i < nw; i += stride) {
        const uint32_t w = perm[i];
        const int32_t u = scan[i];
        wrow[w] = u;
        if (i == 0 || u != scan[i - 1]) {
            uid[u] = wid[w];
            ukey[u] = wkey[w];
            if (Forecast) utarget[u] = wtarget[w];
        }
    }
}

// each kind's series range becomes its window range
__global__ void k_roll_kinds(const int32_t* __restrict__ off, int n_kinds, StackedInfo* info) {
    for (int k = threadIdx.x; k <= n_kinds; k += blockDim.x) info->kind_series[k] = off[info->kind_series[k]];
}

// The working arrays of a regrouping (slots G_*): `bound` piece slots for the ns staged series
struct Pieces {
    int64_t ns, bound;
    int32_t* off;                 // first piece of every series; off[ns] = the number of pieces
    int64_t* begin;               // view of every piece on the staged values
    int32_t* len;
    int32_t* row;                 // union row of every piece
    int64_t* id;                  // name of every piece: its parent id and a key
    uint64_t* key;
    int32_t* scan;                // the scanned name changes
    size_t tb_off, tb_union;      // temporary storage of the two scans
};

static auto name_changes(const Pieces& P, const uint32_t* perm) {
    return thrust::make_transform_iterator(thrust::counting_iterator<int64_t>(0), NameChange{P.id, P.key, perm, P.off + P.ns});
}

// Setup: the piece slots, the temporary storage of both scans, kind_max_len and off[ns] zeroed
static int pieces_setup(StackedWorkspace& S, int64_t bound, Pieces* P, cudaStream_t st, std::string* msg) {
    const int64_t ns = S.h_info->kind_series[S.n_kinds];
    const size_t nb = (size_t)std::max<int64_t>(bound, 1);
    CKE(S.reserve(G_OFF, (size_t)(ns + 1) * 4), "alloc offsets");
    CKE(S.reserve(G_BEGIN, nb * 8), "alloc pieces");
    CKE(S.reserve(G_LEN, nb * 4), "alloc pieces");
    CKE(S.reserve(G_ROW, nb * 4), "alloc pieces");
    CKE(S.reserve(G_ID, nb * 8), "alloc pieces");
    CKE(S.reserve(G_KEY, nb * 8), "alloc pieces");
    CKE(S.reserve(G_SCAN, nb * 4), "alloc pieces");
    CKE(S.reserve(G_UID, nb * 8), "alloc pieces");
    CKE(S.reserve(G_UKEY, nb * 8), "alloc pieces");
    *P = Pieces{ns, bound, (int32_t*)S.bufs[G_OFF], (int64_t*)S.bufs[G_BEGIN], (int32_t*)S.bufs[G_LEN], (int32_t*)S.bufs[G_ROW],
                (int64_t*)S.bufs[G_ID], (uint64_t*)S.bufs[G_KEY], (int32_t*)S.bufs[G_SCAN], 0, 0};
    CKE(cub::DeviceScan::ExclusiveSum(nullptr, P->tb_off, P->off, P->off, (int)(ns + 1), st), "scan size");
    CKE(cub::DeviceScan::InclusiveSum(nullptr, P->tb_union, name_changes(*P, nullptr), P->scan, (int)bound, st), "scan size");
    CKE(S.reserve(T_TEMP, std::max(P->tb_off, P->tb_union)), "alloc temp");
    CKE(cudaMemsetAsync((char*)S.d_info + offsetof(StackedInfo, kind_max_len), 0, sizeof(StackedInfo::kind_max_len), st),
        "memset info");
    CKE(cudaMemsetAsync(P->off + ns, 0, 4, st), "memset offsets");
    return TSFX_OK;
}

// Offsets: the pieces of every series and each kind's longest piece, then the exclusive scan of the counts
template <class Cut>
static int pieces_count(StackedWorkspace& S, const Pieces& P, Cut cut, cudaStream_t st, std::string* msg) {
    k_piece_count<<<grid_for(P.ns, 256), 256, 0, st>>>(S.d_len, P.ns, cut, S.n_kinds, P.off, S.d_info);
    CKE(cudaGetLastError(), "piece count kernel");
    size_t tb = P.tb_off;
    CKE(cub::DeviceScan::ExclusiveSum(S.bufs[T_TEMP], tb, P.off, P.off, (int)(P.ns + 1), st), "piece offsets");
    return TSFX_OK;
}

// Union: sort_rows over the names as (major, minor) pairs (minor float64 bits when minor_f64), the distinct names
// flagged and scanned into the union row of every piece and the name (id, key) of every union row (S.d_uid / S.d_ukey);
// each kind's series range becomes its piece range.  utarget (forecasting windows, with their targets): the target of
// every union row.
static int pieces_union(StackedWorkspace& S, CsrWorkspace& W, const Pieces& P, const int64_t* major, const uint64_t* minor,
                        int minor_f64, const int64_t* target, int64_t* utarget, cudaStream_t st, std::string* msg) {
    uint32_t* perm = nullptr;
    if (int rc = sort_rows(W, major, minor, minor_f64, P.bound, st, msg, &perm)) return rc;
    size_t tb = P.tb_union;
    CKE(cub::DeviceScan::InclusiveSum(S.bufs[T_TEMP], tb, name_changes(P, perm), P.scan, (int)P.bound, st), "union rows");
    S.d_uid = (int64_t*)S.bufs[G_UID];
    S.d_ukey = (uint64_t*)S.bufs[G_UKEY];
    (utarget ? k_roll_union<true> : k_roll_union<false>)<<<grid_for(P.bound, 256), 256, 0, st>>>(
        perm, P.scan, P.off + P.ns, P.id, P.key, P.row, S.d_uid, S.d_ukey, S.d_info, target, utarget);
    k_roll_kinds<<<1, 128, 0, st>>>(P.off, S.n_kinds, S.d_info);
    CKE(cudaGetLastError(), "union kernels");
    return TSFX_OK;
}

int stacked_roll(StackedWorkspace& S, CsrWorkspace& W, int32_t rolling_direction, int32_t max_timeshift, int32_t min_timeshift,
                 int32_t Lmax, int64_t bound, bool forecast, cudaStream_t st, std::string* msg) {
    const int32_t given_min_ts = min_timeshift;
    if (forecast) min_timeshift = std::max(min_timeshift, 1);     // a window of one row is empty without its last row
    const RollSpec R = roll_spec(rolling_direction, max_timeshift, min_timeshift, Lmax);
    Pieces P;
    if (int rc = pieces_setup(S, bound, &P, st, msg)) return rc;
    int64_t *wtarget = nullptr, *utarget = nullptr;
    if (forecast) {
        const size_t nb = (size_t)std::max<int64_t>(bound, 1);
        CKE(S.reserve(R_TGT, nb * 8), "alloc targets");
        CKE(S.reserve(R_UTGT, nb * 8), "alloc targets");
        wtarget = (int64_t*)S.bufs[R_TGT];
        utarget = (int64_t*)S.bufs[R_UTGT];
    }
    const int keys_f64 = S.d_keys && S.keys_f64;
    if (int rc = forecast ? pieces_count(S, P, RollCut<true>{R}, st, msg) : pieces_count(S, P, RollCut<false>{R}, st, msg))
        return rc;
    (forecast ? k_roll_fill<true> : k_roll_fill<false>)<<<grid_for(std::max<int64_t>(P.ns * 32, bound), 256), 256, 0, st>>>(
        S.d_begin, S.d_len, S.d_row, S.d_uid, S.d_keys, keys_f64, P.off, P.ns, bound, R, P.begin, P.len, P.id, P.key,
        S.d_info, S.d_src, wtarget, given_min_ts);
    CKE(cudaGetLastError(), "window fill kernel");
    // windows are named (parent id, key)
    if (int rc = pieces_union(S, W, P, P.id, P.key, keys_f64, wtarget, utarget, st, msg)) return rc;
    S.d_begin = P.begin;
    S.d_len = P.len;
    S.d_row = P.row;
    S.d_utarget = utarget;
    return stacked_publish(S, st, msg);
}

// ---------------------------------------------------------------------------------------------------------------------
// fixed-length packages of the staged series (stacked_sub)

// Sort key of package slot i that puts every kind's packages in the order of their union rows: (kind, union row), or
// INT64_MAX for the slots from *n_packages on.  Reads the kinds' package ranges (info->kind_series after k_roll_kinds).
__global__ void k_sub_layout_key(const int32_t* __restrict__ prow, const int32_t* __restrict__ n_packages, int64_t bound,
                                 int n_kinds, const StackedInfo* info, int64_t* __restrict__ key) {
    const int64_t np = *n_packages;
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    for (const int64_t stride = (int64_t)gridDim.x * blockDim.x; i < bound; i += stride)
        key[i] = i < np ? ((int64_t)kind_of_series(info, n_kinds, i) << 32) | prow[i] : INT64_MAX;
}

// package slot i takes the package perm[i]
__global__ void k_sub_gather(const uint32_t* __restrict__ perm, const int32_t* __restrict__ n_packages,
                             const int64_t* __restrict__ begin, const int32_t* __restrict__ len, const int32_t* __restrict__ row,
                             int64_t* __restrict__ obegin, int32_t* __restrict__ olen, int32_t* __restrict__ orow) {
    const int64_t np = *n_packages;
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    for (const int64_t stride = (int64_t)gridDim.x * blockDim.x; i < np; i += stride) {
        const uint32_t p = perm[i];
        obegin[i] = begin[p];
        olen[i] = len[p];
        orow[i] = row[p];
    }
}

// One warp per series, one lane per package: package j is rows [j * L, min((j + 1) * L, n)) of the series, named
// (package number j, parent id).  The slots [off[n_series], bound) get the name that sorts after every real one
// (INT64_MAX, INT64_MAX).
__global__ void k_sub_fill(const int64_t* __restrict__ begin, const int32_t* __restrict__ len, const int32_t* __restrict__ row,
                           const int64_t* __restrict__ uid, const int32_t* __restrict__ off, int64_t n_series, int64_t bound,
                           int32_t L, int64_t* __restrict__ pbegin, int32_t* __restrict__ plen, int64_t* __restrict__ pid,
                           int64_t* __restrict__ pnum) {
    const int lane = threadIdx.x & 31;
    int64_t s = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t n_warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (; s < n_series; s += n_warps) {                  // warp-uniform
        const int64_t b = begin[s];
        const int32_t n = len[s];
        const int64_t id = uid[row[s]];
        const int32_t o = off[s], np = off[s + 1] - o;
        for (int32_t j = lane; j < np; j += 32) {
            const int64_t lo = (int64_t)j * L;
            pbegin[o + j] = b + lo;
            plen[o + j] = (int32_t)min((int64_t)L, n - lo);
            pid[o + j] = id;
            pnum[o + j] = j;
        }
    }
    int64_t i = off[n_series] + (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    for (const int64_t stride = (int64_t)gridDim.x * blockDim.x; i < bound; i += stride) {
        pid[i] = INT64_MAX;
        pnum[i] = INT64_MAX;
    }
}

int stacked_sub(StackedWorkspace& S, CsrWorkspace& W, int32_t L, int64_t bound, cudaStream_t st, std::string* msg) {
    Pieces P;
    if (int rc = pieces_setup(S, bound, &P, st, msg)) return rc;
    const size_t nb = (size_t)std::max<int64_t>(bound, 1);
    CKE(S.reserve(P_BEGIN, nb * 8), "alloc packages");
    CKE(S.reserve(P_LEN, nb * 4), "alloc packages");
    CKE(S.reserve(P_ROW, nb * 4), "alloc packages");
    if (int rc = pieces_count(S, P, SubCut{L}, st, msg)) return rc;
    int64_t* pnum = (int64_t*)P.key;
    k_sub_fill<<<grid_for(std::max<int64_t>(P.ns * 32, bound), 256), 256, 0, st>>>(S.d_begin, S.d_len, S.d_row, S.d_uid, P.off,
                                                                                   P.ns, bound, L, P.begin, P.len, P.id, pnum);
    CKE(cudaGetLastError(), "package fill kernel");
    // packages are named (package number, parent id)
    if (int rc = pieces_union(S, W, P, pnum, (const uint64_t*)P.id, 0, nullptr, nullptr, st, msg)) return rc;
    // The packages were filled series by series, (parent id, package number) order inside a kind, but the union rows
    // ascend in (package number, parent id).  Reorder every kind's packages by union row, so that a kind with a package
    // for every union row fills its columns in place, as tsfx_extract_staged expects.  The names are no longer needed:
    // the sort key goes into their storage.
    int64_t* key = pnum;
    k_sub_layout_key<<<grid_for(bound, 256), 256, 0, st>>>(P.row, P.off + P.ns, bound, S.n_kinds, S.d_info, key);
    CKE(cudaGetLastError(), "package layout kernel");
    uint32_t* perm = nullptr;
    if (int rc = sort_rows(W, key, nullptr, 0, bound, st, msg, &perm)) return rc;
    S.d_begin = (int64_t*)S.bufs[P_BEGIN];
    S.d_len = (int32_t*)S.bufs[P_LEN];
    S.d_row = (int32_t*)S.bufs[P_ROW];
    k_sub_gather<<<grid_for(bound, 256), 256, 0, st>>>(perm, P.off + P.ns, P.begin, P.len, P.row, S.d_begin, S.d_len, S.d_row);
    CKE(cudaGetLastError(), "package gather kernel");
    return stacked_publish(S, st, msg);
}

__global__ void k_fill_nan(double* __restrict__ out, int64_t n_rows, int n_cols, int ld) {
    int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x, total = n_rows * n_cols;
    for (; e < total; e += stride) out[(e / n_cols) * ld + e % n_cols] = __longlong_as_double(0x7ff8000000000000LL);
}

cudaError_t stacked_fill_nan(double* out, int64_t n_rows, int n_cols, int ld, cudaStream_t st) {
    if (n_rows <= 0 || n_cols <= 0) return cudaSuccess;
    k_fill_nan<<<grid_for(n_rows * n_cols, 256), 256, 0, st>>>(out, n_rows, n_cols, ld);
    return cudaGetLastError();
}

__global__ void k_scatter_rows(const double* __restrict__ block, int64_t n_series, int n_cols, const int32_t* __restrict__ row,
                               double* __restrict__ out, int ld, const int64_t* __restrict__ count,
                               const uint8_t* __restrict__ skip) {
    const int lane = threadIdx.x & 31;
    int64_t s = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t n_warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    if (count) n_series = min(n_series, *count);
    for (; s < n_series; s += n_warps) {
        if (skip && skip[s]) continue;    // warp-uniform
        const double* src = block + (size_t)s * n_cols;
        double* dst = out + (size_t)row[s] * ld;
        for (int c = lane; c < n_cols; c += 32) __stcs(dst + c, __ldcs(src + c));
    }
}

cudaError_t stacked_scatter(const double* block, int64_t n_series, int n_cols, const int32_t* row, double* out, int ld,
                            cudaStream_t st, const int64_t* count, const uint8_t* skip) {
    if (n_series <= 0 || n_cols <= 0) return cudaSuccess;
    k_scatter_rows<<<grid_for(n_series * 32, 256), 256, 0, st>>>(block, n_series, n_cols, row, out, ld, count, skip);
    return cudaGetLastError();
}

// One warp per series, as k_check_views, but every series gets its own verdict instead of the call getting one
__global__ void k_defer_check(const float* __restrict__ values, int64_t n_values, const int64_t* __restrict__ begin,
                              const int32_t* __restrict__ len, int64_t n_series, int32_t max_len, int64_t* __restrict__ vbegin,
                              int32_t* __restrict__ vlen, uint8_t* __restrict__ reject, unsigned long long* first,
                              int keep_unused) {
    const int lane = threadIdx.x & 31;
    int64_t w = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t n_warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (; w < n_series; w += n_warps) {                  // warp-uniform
        if (keep_unused && reject[w] == DEFER_UNUSED) {
            if (lane == 0) { vbegin[w] = 0; vlen[w] = 1; }
            continue;
        }
        int64_t b = w * (int64_t)max_len;
        int32_t l = max_len;
        int why = 0;
        if (begin) {
            b = begin[w];
            l = len[w];
            if (l < 1 || b < 0 || b > n_values - l) why = DEFER_VIEW;
            else if (l > max_len) why = DEFER_LONG;
        }
        if (!why) {
            int nan = 0;
            for (int32_t i = lane; i < l; i += 32) { const float v = values[b + i]; nan |= v != v; }
            if (__any_sync(0xffffffffu, nan)) why = DEFER_NAN;
        }
        if (lane == 0) {
            reject[w] = (uint8_t)why;
            if (why) atomicMax(first + (why - 1), (unsigned long long)(n_series - w));
            if (vbegin) { vbegin[w] = why ? 0 : b; vlen[w] = why ? 1 : l; }
        }
    }
}

cudaError_t defer_check(const float* d_values, int64_t n_values, const int64_t* d_begin, const int32_t* d_len,
                        int64_t n_series, int32_t max_len, int64_t* vbegin, int32_t* vlen, uint8_t* reject,
                        unsigned long long* first, cudaStream_t st, bool keep_unused) {
    if (n_series <= 0) return cudaSuccess;
    k_defer_check<<<grid_for(n_series * 32, 256), 256, 0, st>>>(d_values, n_values, d_begin, d_len, n_series, max_len,
                                                                vbegin, vlen, reject, first, keep_unused ? 1 : 0);
    return cudaGetLastError();
}

__global__ void k_defer_finish(double* __restrict__ out, int64_t n_series, int n_cols, int ld, const uint8_t* __restrict__ reject,
                               const unsigned long long* __restrict__ first, int64_t* status) {
    if (blockIdx.x == 0 && threadIdx.x == 0) {           // one thread: the calls on a status buffer are stream-ordered
        const int64_t call = status[TSFX_STATUS_CALLS] + 1;
        status[TSFX_STATUS_CALLS] = call;
        if (status[TSFX_STATUS_BAD] == 0 && (first[0] | first[1] | first[2])) {
            status[TSFX_STATUS_BAD] = call;
            for (int r = 0; r < 3; ++r) status[TSFX_STATUS_VIEW + r] = first[r] ? n_series - (int64_t)first[r] : -1;
        }
    }
    int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; s < n_series; s += stride)
        if (reject[s])
            for (int c = 0; c < n_cols; ++c) out[s * ld + c] = __longlong_as_double(0x7ff8000000000000LL);
}

cudaError_t defer_finish(double* out, int64_t n_series, int n_cols, int ld, const uint8_t* reject,
                         const unsigned long long* first, int64_t* status, cudaStream_t st) {
    k_defer_finish<<<grid_for(n_series, 256), 256, 0, st>>>(out, n_series, n_cols, ld, reject, first, status);
    return cudaGetLastError();
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
