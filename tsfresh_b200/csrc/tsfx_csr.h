// tsfx_csr.h -- stage (a): long (id, sort key, value) frame -> CSR [ids, begin, len, values] on the device.
// Restates what the reference's adapters do per series on the host (tsfresh/feature_extraction/data.py:
// groupby(id) :217/:280, per-group sort_values(sort) :226/:289, value column slice :230/:291) as device passes.
//
// Fast path (rows already ordered by (id, sort key), the layout the reference's own benchmarks produce): ONE pass
// over the id column (sortedness check + unique-by-key with the row index as payload -> unique ids and begin
// offsets, lengths, longest series, row-block boundaries) and ONE host synchronisation to learn the sizes; the
// sort-key / value columns are then streamed in row blocks while the kernels of earlier blocks run.
// Slow path (any other order): two stable 64-bit radix sorts of the row index (by sort key, then by id), gather.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <string>

namespace tsfx {

#define TSFX_CSR_MAX_BLOCKS 32

struct CsrInfo {                  // written by the device, mirrored in pinned host memory
    int32_t unsorted_ids;         // some id is smaller than its predecessor
    int32_t unsorted_keys;        // inside one id, some sort key is smaller than its predecessor
    int32_t has_nan;              // a value is NaN (data.py:148-167 raises ValueError)
    int32_t max_len;
    int64_t n_series;
    int32_t n_blocks;
    int32_t pad;
    int64_t series_lo[TSFX_CSR_MAX_BLOCKS + 1];   // block b covers series [series_lo[b], series_lo[b+1])
    int64_t row_lo[TSFX_CSR_MAX_BLOCKS + 1];      //             and rows [row_lo[b], row_lo[b+1])
    uint64_t bad_view_rev;        // csr_check_views: n_series - s for the first series s with an invalid view (0: none)
};

struct CsrWorkspace {
    // outputs (device)
    int64_t* d_uid = nullptr;     // unique ids, ascending
    int64_t* d_begin = nullptr;
    int32_t* d_len = nullptr;
    float* d_values = nullptr;    // values in (id, sort key) order
    const uint32_t* d_perm = nullptr;   // after csr_sort_pass: input row of every CSR row (nullptr: rows were in order)
    // internals
    void* bufs[16] = {nullptr};
    size_t caps[16] = {0};
    CsrInfo* h_info = nullptr;    // pinned
    CsrInfo* d_info = nullptr;
    bool frozen = false;          // reserve() fails instead of growing a buffer (a prepared, enqueue-only call)
    void release();
    cudaError_t reserve(int slot, size_t bytes);
    cudaError_t init_info();
    // device copies of the input columns (host-pointer stage (a): tsfx_extract_long[_alloc|_kinds])
    int64_t* ids() const { return (int64_t*)bufs[0]; }
    uint64_t* keys() const { return (uint64_t*)bufs[1]; }
    float* vals() const { return (float*)bufs[2]; }
};

// Pass over the id column (already on the device): fills d_uid / d_begin / d_len for the case the ids are
// non-decreasing, and d_info (copied to h_info asynchronously; the caller synchronises).  min_block = smallest number
// of series per row block, max_blocks <= TSFX_CSR_MAX_BLOCKS.
int csr_ids_pass(CsrWorkspace& W, const int64_t* d_ids, int64_t n_rows, int64_t min_block, int max_blocks,
                 cudaStream_t st, std::string* msg);

// Rows [row_lo, row_hi): flags sort keys that decrease inside one id (pairs (i-1, i)) and NaN values.
void csr_check_rows(CsrWorkspace& W, const int64_t* d_ids, const uint64_t* d_keys, int is_f64, const float* d_values,
                    int64_t row_lo, int64_t row_hi, bool check_nan, cudaStream_t st);

// Slow path: ids / keys / values are on the device in arbitrary row order; sorts and rebuilds the CSR (d_values then
// points at the gathered copy), refreshes d_info / h_info (caller synchronises).
int csr_sort_pass(CsrWorkspace& W, const int64_t* d_ids, const uint64_t* d_keys, int is_f64, const float* d_values,
                  int64_t n_rows, int64_t min_block, int max_blocks, bool check_nan, cudaStream_t st, std::string* msg);

// dst[i] = src[d_perm[i]] (row timestamps follow the sort)
void csr_gather_i64(CsrWorkspace& W, const int64_t* src, int64_t* dst, int64_t n, cudaStream_t st);

void csr_gather_f32(CsrWorkspace& W, const float* src, float* dst, int64_t n, cudaStream_t st);

// longest series of a device CSR (synchronises the stream)
int csr_max_len(CsrWorkspace& W, const int32_t* d_len, int64_t n, cudaStream_t st, int* out);

// NaN scan of a device float array; result lands in d_info->has_nan (async)
void csr_check_nan(CsrWorkspace& W, const float* d_values, int64_t n, cudaStream_t st);

// ---------------------------------------------------------------------------------------------------------------------
// Stacked long format: rows (id, sort key, kind code, value[, time]) in any order, several kinds in one frame
// (data.py:233-291 LongTsFrameAdapter, whose pivot makes one row per id of ANY kind, data.py:86-121).
//
// One csr_sort_pass over all rows orders them by (id, sort key) and yields the union of the ids of every kind as its
// unique ids.  A stable counting sort by kind code then partitions the rows in that order, so each kind's rows land
// contiguous and still ordered by (id, sort key), each carrying the union row of its id.  Series start where the union
// row or the kind changes; every series keeps (begin, len) into the partitioned values and the union row it fills.
// Every kind's rows start at a multiple of TSFX_STACK_ALIGN rows: its series then have the alignment they have when the
// kind is extracted on its own, and kernels whose summation order follows the alignment of the loads (k_moments) give
// the same bits.
#define TSFX_MAX_KINDS 64
#define TSFX_STACK_ALIGN 64

struct StackedInfo {              // written by the device, read once by the host
    int32_t bad_kind;             // a kind code outside 0 .. n_kinds-1
    int32_t nan_values;
    int32_t nan_keys;             // a float64 sort key is NaN
    int32_t dup_names;            // stacked_roll: two windows of one kind have the same name
    int64_t n_union;              // distinct ids over all kinds
    int64_t kind_row[TSFX_MAX_KINDS + 1];      // kind k's rows are [kind_row[k], + kind_rows[k]) of the partitioned arrays
    int64_t kind_rows[TSFX_MAX_KINDS];
    int64_t kind_series[TSFX_MAX_KINDS + 1];   // kind k's series are [kind_series[k], kind_series[k+1])
    int32_t kind_max_len[TSFX_MAX_KINDS];
};

// what the staged series are: the (kind, id) series of the staged rows, or what stacked_roll / stacked_sub replaced them by
enum class Staged : uint8_t { Rows, Windows, ForecastWindows, Packages };

struct StackedWorkspace {
    // the staged input: partitioned rows and per-series views (device), and what the host learnt about them
    float* d_values = nullptr;    // row values, kind-major, (id, sort key) order inside a kind
    int64_t* d_times = nullptr;   // row timestamps in the same order (nullptr: none were given)
    int64_t* d_begin = nullptr;   // series s = d_values[d_begin[s] .. + d_len[s])
    int32_t* d_len = nullptr;
    int32_t* d_row = nullptr;     // union row of series s
    int64_t* d_uid = nullptr;     // union ids, ascending (keep_ids); after stacked_roll / stacked_sub the parent id of
                                  // every union window / package
    uint64_t* d_keys = nullptr;   // sort keys (raw bits) in the order of d_values (stacked_stage with keep_keys)
    uint64_t* d_ukey = nullptr;   // after stacked_roll: naming sort key of every union window (raw bits); after
                                  // stacked_sub: package number of every union package (int64)
    uint32_t* d_src = nullptr;    // input row number of every staged row (stacked_stage with keep_rows)
    int64_t* d_utarget = nullptr; // after stacked_roll with forecast: target row of every union window (-1: none)
    StackedInfo* h_info = nullptr;   // pinned
    StackedInfo* d_info = nullptr;
    int n_kinds = 0;
    int64_t n_union = 0;
    Staged staged = Staged::Rows;
    bool pending = false;         // staged and not yet consumed by tsfx_extract_staged (staged outlives it: the row keys
                                  // and targets stay readable)
    bool has_keys = false;        // the rows came with sort keys
    bool keys_f64 = false;        //   float64 ones
    void* bufs[32] = {nullptr};
    size_t caps[32] = {0};
    bool frozen = false;          // reserve() fails instead of growing a buffer (a prepared, enqueue-only call)
    cudaError_t reserve(int slot, size_t bytes);
    cudaError_t keep_ids(const int64_t* d_src, int64_t n, cudaStream_t st);   // d_uid = a copy of n union ids
    void release();
};

// Stages n_rows device rows (ids, sort keys (nullptr: input order), float32 values, kind codes (int32 / int64; nullptr:
// every row is kind 0), optional int64 row times) into S, then copies S.d_info to S.h_info.  Asynchronous: the caller
// synchronises and checks the flags before it relies on the sizes.  Uses W's sort buffers as scratch.  keep_keys: the
// sort keys follow the rows into S.d_keys (stacked_roll names its windows by them).  keep_rows: every staged row's input
// row number goes to S.d_src (stacked_roll with forecast finds the targets by them).
int stacked_stage(StackedWorkspace& S, CsrWorkspace& W, const int64_t* d_ids, const uint64_t* d_keys, int keys_f64,
                  const float* d_values, const void* d_kinds, int kinds_i64, int n_kinds, const int64_t* d_times,
                  int64_t n_rows, bool keep_keys, bool keep_rows, cudaStream_t st, std::string* msg);

// Rolled windows (roll_time_series, tsfx_roll.cuh) of the staged series, as new staged series: every window is a view
// (d_begin, d_len) on the unchanged d_values, so each kind keeps its aligned rows.  Per series a count of its windows, a
// scan, then a fill of one warp per series; the windows' names (parent id, sort key of the naming row, or its row number
// without sort keys) are sorted with W's radix passes, and the distinct names, flagged and scanned, are the union rows:
// d_row of every window, d_uid / d_ukey of every union row.  d_info gets the window ranges of the kinds (kind_series),
// their longest windows (kind_max_len), n_union and dup_names, and is copied to h_info (the caller synchronises).
// Lmax = the longest staged series (the shifts' anchor); bound >= the number of windows.
// forecast (make_forecasting_frame, needs S.d_src): only windows of at least max(min_timeshift, 1) + 1 rows are kept,
// every one of them loses its last row (so none is empty), and its target is the input row number of its naming row (-1
// for input row 0, which the reference's y = x[1:] leaves out); the first window of every union row passes its target on
// to d_utarget.  A name shared with a one-row window that min_timeshift keeps but the drop empties sets dup_names too.
int stacked_roll(StackedWorkspace& S, CsrWorkspace& W, int32_t rolling_direction, int32_t max_timeshift, int32_t min_timeshift,
                 int32_t Lmax, int64_t bound, bool forecast, cudaStream_t st, std::string* msg);

// Fixed-length packages (add_sub_time_series_index) of the staged series, as new staged series: package j of a series
// of n rows is the view on its rows [j * L, min((j + 1) * L, n)), so each kind keeps its aligned rows.  The count, scan
// and union are stacked_roll's (one code path for both), the fill is its own; a package is named (package number, parent
// id) and the union rows ascend in that order, and one more sort puts every kind's packages in union-row order.  d_uid /
// d_ukey get the parent id / package number of every union row; d_info the package ranges of the kinds, their longest
// packages and n_union, copied to h_info (the caller synchronises).  bound >= the number of packages.
int stacked_sub(StackedWorkspace& S, CsrWorkspace& W, int32_t L, int64_t bound, cudaStream_t st, std::string* msg);

// Deferred stage (tsfx_extract_long_deferred): stacked_stage of n rows of which only [0, *n_live) count (n_live
// nullptr: all n), enqueue-only.  The rows from *n_live on are made to sort after every live row, so the live rows
// take the order, union rows and staged layout that stacked_stage gives them alone; the kind counting sort drops them
// with the rows whose code is out of range (the bad_kind flag stays on the device, as nan_keys does).  The union size
// goes to S.d_info->n_union, the union ids below max_ids to out_ids[0 .. n_union), the first id past them to *id_past.
// Nothing is copied to the host, and S and W must hold what stacked_defer_reserve reserved for at least n rows.
int stacked_stage_deferred(StackedWorkspace& S, CsrWorkspace& W, const int64_t* d_ids, const uint64_t* d_keys, int keys_f64,
                           const float* d_values, const void* d_kinds, int kinds_i64, int n_kinds, int64_t n,
                           const int64_t* d_n_live, int64_t max_ids, int64_t* out_ids, int64_t* id_past, cudaStream_t st,
                           std::string* msg);

// Every buffer stacked_stage_deferred of n rows and n_kinds kinds uses, with or without sort keys
int stacked_defer_reserve(StackedWorkspace& S, CsrWorkspace& W, int64_t n, int n_kinds, std::string* msg);

// After stacked_stage_deferred: kind k's series in the fixed slots [k * max_ids, (k + 1) * max_ids), in series order.  A
// live series gets its view (sbegin, slen) and union row (srow); the other slots, and every slot of a call the stage
// rejects (a kind code out of range, a NaN sort key, more than max_ids union rows), get reject reason DEFER_UNUSED.
// live[k] = kind k's live series.
cudaError_t stacked_slots(const StackedWorkspace& S, int n_kinds, int64_t max_ids, int64_t* sbegin, int32_t* slen,
                          int32_t* srow, uint8_t* reject, int64_t* live, cudaStream_t st);

// Last step of a deferred long call: *n_ids (0 for a rejected call), INT64_MAX in out_ids[*n_ids .. max_ids), and, if
// the status words record this call (tsfx.h "Deferred input check"), its call-wide reasons and the id its report names.
cudaError_t stacked_defer_report(const StackedWorkspace& S, int64_t max_ids, const int64_t* id_past, const int32_t* srow,
                                 int64_t* out_ids, int64_t* n_ids, int64_t* status, cudaStream_t st);

// out[r * ld + c] = NaN for r < n_rows, c < n_cols
cudaError_t stacked_fill_nan(double* out, int64_t n_rows, int n_cols, int ld, cudaStream_t st);

// out[row[s] * ld + c] = block[s * n_cols + c] for s < n_series, c < n_cols (one warp per row).  count (device, may be
// nullptr): only s < *count; skip (may be nullptr): not the series with skip[s] != 0.
cudaError_t stacked_scatter(const double* block, int64_t n_series, int n_cols, const int32_t* row, double* out, int ld,
                            cudaStream_t st, const int64_t* count = nullptr, const uint8_t* skip = nullptr);

// Checked pass over caller-supplied device views (TSFX_FLAG_CHECK_DEVICE_INPUT), one launch: the longest series into
// d_info->max_len, the first view with len < 1, begin < 0 or begin + len > n_values into d_info->bad_view_rev, and a NaN
// among the values of the valid views into d_info->has_nan (async; d_info zeroed by the caller)
void csr_check_views(CsrWorkspace& W, const float* d_values, int64_t n_values, const int64_t* d_begin, const int32_t* d_len,
                     int64_t n_series, cudaStream_t st);

// Deferred input check (TSFX_FLAG_DEFER_CHECK), one launch: per series (dense: row s of max_len samples at
// values + s * max_len, begin == nullptr; CSR: the caller's view) its reject reason into reject[s] (DEFER_VIEW, DEFER_LONG
// or DEFER_NAN, 0: none) and, per reason r, n_series - s of the first rejected series into first[r - 1] (atomicMax,
// zeroed by the caller).  CSR: the private view of every series into vbegin / vlen, (0, 1) for a rejected one.
// keep_unused: a series whose reject[s] is already DEFER_UNUSED (stacked_slots) keeps it, unreported.
enum { DEFER_VIEW = 1, DEFER_LONG, DEFER_NAN, DEFER_UNUSED };
cudaError_t defer_check(const float* d_values, int64_t n_values, const int64_t* d_begin, const int32_t* d_len,
                        int64_t n_series, int32_t max_len, int64_t* vbegin, int32_t* vlen, uint8_t* reject,
                        unsigned long long* first, cudaStream_t st, bool keep_unused = false);

// After the groups of a deferred-check call: NaN in every column of every rejected series (out[s * ld + c], c < n_cols),
// then the call's report into the caller's status words (tsfx.h TSFX_STATUS_*).
cudaError_t defer_finish(double* out, int64_t n_series, int n_cols, int ld, const uint8_t* reject,
                         const unsigned long long* first, int64_t* status, cudaStream_t st);

}  // namespace tsfx
