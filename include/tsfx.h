/* tsfx.h -- C ABI of libtsfx.so: the H100 (sm_90a) implementation of tsfresh's feature-extraction
 * hot path.
 *
 * There is no native interface in the reference (tsfresh is pure Python); the entry points below are
 * what a ctypes binding for the path replaces:
 *
 *   tsfx_plan_create      <- the settings dict walked by _do_extraction_on_chunk
 *                            (tsfresh/feature_extraction/extraction.py:339-378, settings.py:133-294):
 *                            one tsfx_feature_desc per output column, in column order.
 *   tsfx_extract_csr      <- _do_extraction_on_chunk over every (id, kind) series of a chunk list
 *   tsfx_extract_dense       (extraction.py:308-386; distribution.py:173-245 map_reduce): all series in
 *                            one call, results as the dense [n_series x n_features] float64 matrix that
 *                            PartitionedTsData.pivot (data.py:86-121) would assemble.
 *   tsfx_extract_long     <- LongTsFrameAdapter / WideTsFrameAdapter iteration (data.py:181-291):
 *                            group by id, sort each group by the sort column, then the above.
 *   tsfx_roll_windows     <- roll_time_series window enumeration
 *                            (utilities/dataframe_functions.py:376-603), expressed as CSR views.
 *
 * Conventions: plain C, no exceptions cross the boundary.  Return 0 on success, a negative TSFX_E_*
 * code otherwise (text via tsfx_last_error).  The caller owns every buffer it passes; the library owns
 * only the device scratch inside the context.  Pointers are host pointers unless TSFX_FLAG_DEVICE_PTRS
 * is set, in which case `values`, `begin`, `len` and `out` are device pointers on the context's device
 * and the call is asynchronous on the context's stream (use tsfx_sync).  NaN results that the
 * reference defines (short series, zero variance, ...) are values, not errors.  Values are float32
 * (BASELINE.json north_star); all arithmetic is float64.
 */
#ifndef TSFX_H_
#define TSFX_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define TSFX_VERSION 2

/* error codes */
#define TSFX_OK 0
#define TSFX_E_INVALID (-1)     /* bad argument / malformed plan */
#define TSFX_E_CUDA (-2)        /* CUDA runtime failure (message has the cudaError string) */
#define TSFX_E_UNSUPPORTED (-3) /* parameter combination without a GPU implementation */
#define TSFX_E_TOO_LONG (-4)    /* a series does not fit the per-warp shared-memory staging */
#define TSFX_E_NOMEM (-5)
#define TSFX_E_NAN (-6)         /* NaN in the value column (data.py:148-167 raises ValueError) */

/* flags */
#define TSFX_FLAG_DEVICE_PTRS 1u /* values/begin/len/out are device pointers; async on ctx stream */
#define TSFX_FLAG_TIMING 2u      /* record CUDA events around every kernel group (tsfx_get_timings) */
#define TSFX_FLAG_NO_NAN_CHECK 4u /* host-pointer extract calls scan the values for NaN and return TSFX_E_NAN (the reference
                                  * raises ValueError, data.py:148-167); this flag skips the scan.  Device-pointer calls
                                  * (asynchronous) never scan. */
#define TSFX_FLAG_IMPUTE 8u      /* extract calls: impute the feature matrix on the device before it is returned
                                  * (extract_features(impute_function=impute), extraction.py:179-181, 286-287) */
#define TSFX_FLAG_ALL_MEDIANS 16u /* tsfx_impute: compute every column's median, not only those a NaN needs */

/* tsfx_impute modes (tsfresh/utilities/dataframe_functions.py) */
#define TSFX_IMPUTE_RANGE 0      /* impute :49-78: +inf -> max, -inf -> min, NaN -> median of the finite values */
#define TSFX_IMPUTE_ZERO 1       /* impute_dataframe_zero :81-101: every non-finite value -> 0 */
#define TSFX_IMPUTE_GIVEN 2      /* impute_dataframe_range :104-167: replacement values supplied by the caller */
#define TSFX_IMPUTE_STATS 3      /* get_range_values_per_column :170-212: statistics only, matrix untouched */

/* calculator ids: one per reference calculator (feature_calculators.py line in the comment) */
enum tsfx_calc {
    TSFX_VARIANCE_LARGER_THAN_STANDARD_DEVIATION = 0, /* :239 */
    TSFX_RATIO_BEYOND_R_SIGMA,                         /* :256  p0=r */
    TSFX_LARGE_STANDARD_DEVIATION,                     /* :273  p0=r */
    TSFX_SYMMETRY_LOOKING,                             /* :299  p0=r */
    TSFX_HAS_DUPLICATE_MAX,                            /* :325 */
    TSFX_HAS_DUPLICATE_MIN,                            /* :340 */
    TSFX_HAS_DUPLICATE,                                /* :355 */
    TSFX_SUM_VALUES,                                   /* :371 */
    TSFX_AGG_AUTOCORRELATION,                          /* :387  attr=f_agg i0=maxlag */
    TSFX_PARTIAL_AUTOCORRELATION,                      /* :440  i0=lag i1=max lag over the param list */
    TSFX_AUGMENTED_DICKEY_FULLER,                      /* :499  attr=teststat|pvalue|usedlag i0=autolag */
    TSFX_ABS_ENERGY,                                   /* :548 */
    TSFX_CID_CE,                                       /* :567  i0=normalize */
    TSFX_MEAN_ABS_CHANGE,                              /* :604 */
    TSFX_MEAN_CHANGE,                                  /* :624 */
    TSFX_MEAN_SECOND_DERIVATIVE_CENTRAL,               /* :644 */
    TSFX_MEDIAN,                                       /* :663 */
    TSFX_MEAN,                                         /* :677 */
    TSFX_LENGTH,                                       /* :691 */
    TSFX_STANDARD_DEVIATION,                           /* :705 */
    TSFX_VARIATION_COEFFICIENT,                        /* :718 */
    TSFX_VARIANCE,                                     /* :735 */
    TSFX_SKEWNESS,                                     /* :749 */
    TSFX_KURTOSIS,                                     /* :766 */
    TSFX_ROOT_MEAN_SQUARE,                             /* :783 */
    TSFX_ABSOLUTE_SUM_OF_CHANGES,                      /* :796 */
    TSFX_LONGEST_STRIKE_BELOW_MEAN,                    /* :813 */
    TSFX_LONGEST_STRIKE_ABOVE_MEAN,                    /* :828 */
    TSFX_COUNT_ABOVE_MEAN,                             /* :843 */
    TSFX_COUNT_BELOW_MEAN,                             /* :857 */
    TSFX_LAST_LOCATION_OF_MAXIMUM,                     /* :871 */
    TSFX_FIRST_LOCATION_OF_MAXIMUM,                    /* :886 */
    TSFX_LAST_LOCATION_OF_MINIMUM,                     /* :902 */
    TSFX_FIRST_LOCATION_OF_MINIMUM,                    /* :917 */
    TSFX_PERCENTAGE_OF_REOCCURRING_VALUES_TO_ALL_VALUES,         /* :933 */
    TSFX_PERCENTAGE_OF_REOCCURRING_DATAPOINTS_TO_ALL_DATAPOINTS, /* :961 */
    TSFX_SUM_OF_REOCCURRING_VALUES,                    /* :992 */
    TSFX_SUM_OF_REOCCURRING_DATA_POINTS,               /* :1020 */
    TSFX_RATIO_VALUE_NUMBER_TO_TIME_SERIES_LENGTH,     /* :1045 */
    TSFX_FFT_COEFFICIENT,                              /* :1067 attr=real|imag|abs|angle i0=coeff */
    TSFX_FFT_AGGREGATED,                               /* :1123 attr=centroid|variance|skew|kurtosis */
    TSFX_NUMBER_PEAKS,                                 /* :1235 i0=n */
    TSFX_INDEX_MASS_QUANTILE,                          /* :1275 p0=q */
    TSFX_NUMBER_CWT_PEAKS,                             /* :1320 i0=n */
    TSFX_LINEAR_TREND,                                 /* :1343 attr=pvalue|rvalue|intercept|slope|stderr */
    TSFX_CWT_COEFFICIENTS,                             /* :1370 i0=coeff i1=table index of scale w */
    TSFX_SPKT_WELCH_DENSITY,                           /* :1418 i0=coeff */
    TSFX_AR_COEFFICIENT,                               /* :1459 i0=coeff i1=k */
    TSFX_CHANGE_QUANTILES,                             /* :1511 p0=ql p1=qh i0=isabs attr=f_agg */
    TSFX_TIME_REVERSAL_ASYMMETRY_STATISTIC,            /* :1557 i0=lag */
    TSFX_C3,                                           /* :1600 i0=lag */
    TSFX_MEAN_N_ABSOLUTE_MAX,                          /* :1643 i0=number_of_maxima */
    TSFX_BINNED_ENTROPY,                               /* :1666 i0=max_bins */
    TSFX_SAMPLE_ENTROPY,                               /* :1701 */
    TSFX_APPROXIMATE_ENTROPY,                          /* :1759 i0=m p0=r */
    TSFX_FOURIER_ENTROPY,                              /* :1809 i0=bins */
    TSFX_LEMPEL_ZIV_COMPLEXITY,                        /* :1825 i0=bins */
    TSFX_PERMUTATION_ENTROPY,                          /* :1866 i0=tau i1=dimension */
    TSFX_AUTOCORRELATION,                              /* :1919 i0=lag */
    TSFX_QUANTILE,                                     /* :1963 p0=q */
    TSFX_NUMBER_CROSSING_M,                            /* :1980 p0=m */
    TSFX_MAXIMUM,                                      /* :2003 */
    TSFX_ABSOLUTE_MAXIMUM,                             /* :2017 */
    TSFX_MINIMUM,                                      /* :2031 */
    TSFX_VALUE_COUNT,                                  /* :2044 p0=value */
    TSFX_RANGE_COUNT,                                  /* :2065 p0=min p1=max */
    TSFX_FRIEDRICH_COEFFICIENTS,                       /* :2082 i0=coeff i1=m i2=r */
    TSFX_MAX_LANGEVIN_FIXED_POINT,                     /* :2134 i1=m i2=r */
    TSFX_AGG_LINEAR_TREND,                             /* :2171 attr=linregress attr i0=chunk_len i1=f_agg */
    TSFX_ENERGY_RATIO_BY_CHUNKS,                       /* :2226 i0=num_segments i1=segment_focus */
    TSFX_COUNT_ABOVE,                                  /* :2309 p0=t */
    TSFX_COUNT_BELOW,                                  /* :2325 p0=t */
    TSFX_BENFORD_CORRELATION,                          /* :2341 */
    TSFX_QUERY_SIMILARITY_COUNT,                       /* :2475 default query=None -> NaN */
    TSFX_LINEAR_TREND_TIMEWISE,                        /* :2274 attr=linregress attr; regressor = row time in hours
                                                        * since the first row of the series (tsfx_set_row_times) */
    TSFX_CONST_NAN,                                    /* a column the reference defines as NaN */
    TSFX_N_CALCS
};

/* attr codes */
enum { TSFX_AGG_MEAN = 0, TSFX_AGG_MEDIAN, TSFX_AGG_VAR, TSFX_AGG_STD, TSFX_AGG_MAX, TSFX_AGG_MIN };
enum { TSFX_FFT_REAL = 0, TSFX_FFT_IMAG, TSFX_FFT_ABS, TSFX_FFT_ANGLE };
enum { TSFX_SPEC_CENTROID = 0, TSFX_SPEC_VARIANCE, TSFX_SPEC_SKEW, TSFX_SPEC_KURTOSIS };
enum { TSFX_LR_PVALUE = 0, TSFX_LR_RVALUE, TSFX_LR_INTERCEPT, TSFX_LR_SLOPE, TSFX_LR_STDERR };
enum { TSFX_ADF_TESTSTAT = 0, TSFX_ADF_PVALUE, TSFX_ADF_USEDLAG, TSFX_ADF_BADATTR };
enum { TSFX_AUTOLAG_AIC = 0, TSFX_AUTOLAG_BIC, TSFX_AUTOLAG_NONE };

/* One output column. `col` is its index in the row-major [n_series x n_cols] result. */
typedef struct tsfx_feature_desc {
    int32_t calc; /* enum tsfx_calc */
    int32_t attr;
    int32_t i0, i1, i2;
    int32_t col;
    double p0, p1;
} tsfx_feature_desc;

typedef struct tsfx_ctx tsfx_ctx;
typedef struct tsfx_plan tsfx_plan;

/* Context: one per process and device.  `cuda_stream` may be NULL (library creates its own stream) or
 * a cudaStream_t the caller owns (e.g. torch's current stream) so caller-side CUDA events see the work. */
int tsfx_ctx_create(int device, void* cuda_stream, tsfx_ctx** out);
void tsfx_ctx_destroy(tsfx_ctx* ctx);
const char* tsfx_last_error(const tsfx_ctx* ctx); /* ctx may be NULL: last creation error */
int tsfx_sync(tsfx_ctx* ctx);
int tsfx_version(void);
int tsfx_device_count(void);   /* CUDA devices visible to this process (0 when there is none) */

/* Plan: the compiled settings dict.  `tables` holds the concatenated float64 convolution kernels for
 * cwt_coefficients (one per distinct scale, table t = tables[table_off[t] .. table_off[t+1])),
 * scaled so that coefficient c of scale t is sum_k x[k] * table_t[c + half_t - k]; `table_half[t]` is
 * half_t.  n_cols is the row stride of the output (>= max col + 1). */
int tsfx_plan_create(tsfx_ctx* ctx, const tsfx_feature_desc* descs, int32_t n_descs, int32_t n_cols,
                     const double* tables, const int64_t* table_off, const int32_t* table_half,
                     int32_t n_tables, tsfx_plan** out);
void tsfx_plan_destroy(tsfx_plan* plan);

/* CSR: series s is values[begin[s] .. begin[s]+len[s]).  out is [n_series x n_cols] float64 row-major. */
int tsfx_extract_csr(tsfx_ctx* ctx, const tsfx_plan* plan, const float* values, int64_t n_values,
                     const int64_t* begin, const int32_t* len, int64_t n_series, double* out,
                     uint32_t flags);

/* Device-pointer CSR calls size their working sets by the longest series.  Without a hint the library reduces `len` on
 * the device and synchronises the stream once per call; a caller that knows an upper bound (e.g. max_timeshift + 1 for
 * rolled windows) passes it here and the calls stay asynchronous.  The bound must hold for every series of the
 * following device-pointer tsfx_extract_csr calls; 0 removes the hint. */
int tsfx_set_max_len_hint(tsfx_ctx* ctx, int32_t max_len);

/* Row timestamps for linear_trend_timewise (feature_calculators.py:2274-2306: the regressor is the series' DatetimeIndex,
 * hours since its first row).  row_time_ns[i] is the timestamp (int64 nanoseconds) of row i of the `values` array of the
 * NEXT extract call on this context (host pointer, or device pointer with TSFX_FLAG_DEVICE_PTRS); that call consumes
 * them (tsfx_extract_long carries them through its sort).  A plan with linear_trend_timewise columns and no row times
 * is TSFX_E_INVALID. */
int tsfx_set_row_times(tsfx_ctx* ctx, const int64_t* row_time_ns, int64_t n_rows, uint32_t flags);

/* Dense fast path: n_series series of identical length `len`, back to back. */
int tsfx_extract_dense(tsfx_ctx* ctx, const tsfx_plan* plan, const float* values, int64_t n_series,
                       int32_t len, double* out, uint32_t flags);

/* Long frame (stage (a)): rows (ids[i], sort_keys[i], values[i]) in any order.  Groups rows by id,
 * orders each group by sort key (stable for equal keys; sort_keys may be NULL = keep row order), then
 * extracts.  Series come out in ascending id order: out_ids[s] and row s of out.
 * sort_key_is_f64: 0 = int64 keys, 1 = float64 keys.  Returns the number of series in *n_series_out;
 * TSFX_E_INVALID if it exceeds out_capacity.
 * Rows that already arrive ordered by (id, sort key) take the pipelined path: one pass over the id column, one host
 * synchronisation for the sizes, then the sort-key / value columns are copied in row blocks while the kernels of the
 * previous blocks run and their result rows travel back.  Any other order is sorted on the device first.
 * Host pointers may be pageable (staged through pinned memory by worker threads) or page-locked.  With
 * TSFX_FLAG_DEVICE_PTRS every pointer (ids, sort_keys, values, out_ids, out) is a device pointer; the call still
 * synchronises once to learn the sizes.
 * Two-step use: call tsfx_build_csr with all output pointers NULL (it counts the series and keeps the CSR on the
 * device), size `out`, then call tsfx_extract_long with ids == values == NULL to extract from the held CSR. */
int tsfx_extract_long(tsfx_ctx* ctx, const tsfx_plan* plan, const int64_t* ids, const void* sort_keys,
                      int32_t sort_key_is_f64, const float* values, int64_t n_rows, int64_t* out_ids,
                      double* out, int64_t out_capacity, int64_t* n_series_out, uint32_t flags);

/* Same, but the library sizes the result itself: *out ([n_series x n_cols] float64) and *out_ids come from the context's
 * pinned host pool and must be handed back with tsfx_host_free (a numpy array can wrap them without a copy). */
int tsfx_extract_long_alloc(tsfx_ctx* ctx, const tsfx_plan* plan, const int64_t* ids, const void* sort_keys,
                            int32_t sort_key_is_f64, const float* values, int64_t n_rows, int64_t** out_ids,
                            double** out, int64_t* n_series_out, uint32_t flags);

/* Wide format with a KIND dimension (data.py:181-230 WideTsFrameAdapter: several value columns share the id and sort
 * columns): stage (a) runs once, every kind k is then evaluated with its own plan (kind_to_fc_parameters, extraction.py:
 * 333-336) on its own value column values[k], and the result is ONE matrix [n_series x sum_k n_cols(k)] whose column
 * blocks follow the order of the kinds -- the frame PartitionedTsData.pivot builds (data.py:86-121).  Result buffers come
 * from the pinned pool (tsfx_host_free).  Up to 64 kinds per call. */
int tsfx_extract_long_kinds(tsfx_ctx* ctx, const tsfx_plan* const* plans, const int64_t* ids, const void* sort_keys,
                            int32_t sort_key_is_f64, const float* const* values, int32_t n_kinds, int64_t n_rows,
                            int64_t** out_ids, double** out, int64_t* n_series_out, uint32_t flags);

/* Page-locked host memory from the context's pool (freed blocks are cached: page-locking is slow). */
void* tsfx_host_alloc(tsfx_ctx* ctx, size_t bytes);
void tsfx_host_free(tsfx_ctx* ctx, void* p);

/* Multi-GPU result placement -- replaces the single all-gather of the feature matrix (SURVEY.md section 8e; the
 * reference's workers return their rows to the parent process, distribution.py:471-486).  peer_out[p] is rank p's copy
 * of the full result matrix as mapped into THIS process (CUDA IPC / symmetric memory), peer_out[self_index] the local
 * one.  Afterwards every device-pointer extract call whose `out` lies inside the local matrix also places its rows at
 * the same offset of every peer's matrix:
 *   TSFX_PEER_COPY       copy engines (cudaMemcpyAsync over NVLink on a side stream, no SM time), per row block
 *   TSFX_PEER_STORE      the assemble kernel stores each finished row to every peer (P2P stores over NVLink)
 *   TSFX_PEER_MULTICAST  the assemble kernel stores each row once through `multicast_out`, the multicast mapping of the
 *                        matrix (NVSwitch replicates the store to all ranks, this one included)
 *   TSFX_PEER_AUTO       COPY (copy engines take no SM time, and 8-byte multicast stores do not fill NVLink packets;
 *                        the three modes have not been timed against each other on H100)
 * tsfx_peer_flush makes the context's stream wait for the copies in flight; the caller then synchronises the ranks
 * (barrier) before reading its matrix.  n_peers = 0 switches the placement off. */
#define TSFX_PEER_AUTO 0
#define TSFX_PEER_COPY 1
#define TSFX_PEER_STORE 2
#define TSFX_PEER_MULTICAST 3
int tsfx_set_peer_outputs(tsfx_ctx* ctx, const uint64_t* peer_out, int32_t n_peers, int32_t self_index,
                          uint64_t multicast_out, int32_t mode);
int tsfx_peer_flush(tsfx_ctx* ctx);

/* Stage (a) alone: builds the CSR on the device (it stays held by the context until the next stage-(a)
 * call) and copies back whichever outputs are non-NULL. */
int tsfx_build_csr(tsfx_ctx* ctx, const int64_t* ids, const void* sort_keys, int32_t sort_key_is_f64,
                   const float* values, int64_t n_rows, int64_t* out_ids, int64_t* out_begin,
                   int32_t* out_len, float* sorted_values, int64_t out_capacity, int64_t* n_series_out);

/* roll_time_series as views: for every series s of the input CSR and every shift t of
 * dataframe_functions.py:340-373, 548-562 (positive rolling_direction: windows END at row t-1; negative: windows
 * START at row t-1) emits win_begin/win_len over the SAME values buffer plus (parent, index of the row whose sort
 * value names the window: its last row for positive, its first row for negative direction).  max_timeshift is the
 * reference's value (window length - 1; pass a number >= the longest series for "None").  Returns the number of
 * windows (or a negative error); pass NULL outputs to only count. */
int64_t tsfx_roll_windows(const int64_t* begin, const int32_t* len, int64_t n_series,
                          int32_t rolling_direction, int32_t max_timeshift, int32_t min_timeshift,
                          int64_t* win_begin, int32_t* win_len, int64_t* win_parent,
                          int32_t* win_end_index, int64_t capacity);

/* Column-wise imputation of a row-major float64 matrix [n_rows x n_cols], in place (replaces the reference's
 * tsfresh.utilities.dataframe_functions.impute / impute_dataframe_zero / impute_dataframe_range /
 * get_range_values_per_column, dataframe_functions.py:49-212, on the matrix extract_features returns).
 * `matrix` is a host pointer (copied to the device and back) or, with TSFX_FLAG_DEVICE_PTRS, a device pointer.
 * col_stats: host array of 3*n_cols doubles laid out min | max | median -- output for RANGE / STATS (may be NULL
 * for RANGE), input for GIVEN, ignored for ZERO.  Columns without any finite value report 0 for all three.
 * Without TSFX_FLAG_ALL_MEDIANS the median of a column that holds no NaN is not computed and reported as NaN. */
int tsfx_impute(tsfx_ctx* ctx, double* matrix, int64_t n_rows, int32_t n_cols, int32_t mode, double* col_stats,
                uint32_t flags);

/* Feature selection on the feature matrix (tsfresh/feature_selection/relevance.py:31-322, significance_tests.py:43-132),
 * classification targets: for every column of X ([n_rows x n_cols] row-major float64; host pointer, or device pointer with
 * TSFX_FLAG_DEVICE_PTRS) and every class k (one-vs-rest, y_codes[i] in 0 .. n_classes-1, host) the sufficient statistics of
 * the reference's univariate tests, from one sort of the column:
 *   out[(k * n_cols + c) * TSFX_SEL_NSTAT + ...] =
 *     0: feature type (0 constant, 1 binary, 2 real; get_feature_type relevance.py:325-345)   1: n1 = rows of class k   2: n0
 *     real feature:    3: Mann-Whitney U of the class-k sample   4: tie term sum(t^3 - t)   5: two-sample KS statistic
 *                      6: number of distinct values
 *     binary feature:  3: n(y = k, x = larger value)  4: n(y = k, x = smaller)  5: n(y != k, x = larger)  6: n(y != k, x = smaller)
 * (the contingency table of target_binary_feature_binary_test, significance_tests.py:70-79).  p-values and the
 * Benjamini-Hochberg / -Yekutieli decision are O(n_cols) host work (tsfresh_b200/feature_selection.py).
 * TSFX_E_NAN when X holds a NaN (the reference raises ValueError, significance_tests.py:266-289). */
#define TSFX_SEL_NSTAT 8
int tsfx_select_classification(tsfx_ctx* ctx, const double* X, int64_t n_rows, int32_t n_cols, const int32_t* y_codes,
                               int32_t n_classes, double* out, uint32_t flags);

/* Same for REGRESSION targets (relevance.py:282-296; significance_tests.py:135-188): y is the float64 target of every row.
 * out: n_cols x TSFX_SEL_NSTAT doubles + 4 trailing doubles { sum t(t-1)/2, sum t(t-1)(t-2), sum t(t-1)(2t+5) over the
 * tie groups of y, n_rows }:
 *     0: feature type   1: n_rows
 *     real feature (Kendall's tau, scipy.stats.kendalltau method="asymptotic"):  2: discordant pairs   3..5: the three tie
 *                      sums of the feature   6: joint ties sum c(c-1)/2 of (x, y)
 *     binary feature (two-sample KS of the target, scipy.stats.ks_2samp):  2: KS statistic   3: rows with the larger value
 *                      4: rows with the smaller value */
int tsfx_select_regression(tsfx_ctx* ctx, const double* X, int64_t n_rows, int32_t n_cols, const double* y, double* out,
                           uint32_t flags);

/* Per-kernel-group device time (ms) of the last extract call made with TSFX_FLAG_TIMING.
 * names_out[i] points at a static string.  Returns the number of groups written (<= cap). */
int tsfx_get_timings(tsfx_ctx* ctx, float* ms_out, const char** names_out, int32_t cap);
/* Number of kernels the last extract call launched. */
int tsfx_last_launch_count(const tsfx_ctx* ctx);
/* Which kernel variant each kernel group of the last extract call ran, e.g. "entropy/rank-g4", "basic/w12/shared",
 * "spectral/w4/global", "peaks/general/hybrid", "moments/dense" (entry points that work in row blocks: the last
 * block).  names_out[i] points at a static string.  Returns the number of groups written (<= cap). */
int tsfx_last_kernels(const tsfx_ctx* ctx, const char** names_out, int32_t cap);
/* Every variant name tsfx_last_kernels can report, including those only A/B tuning variables select.  Returns the
 * number of names; writes at most cap of them to names_out (may be NULL). */
int tsfx_kernel_variants(const char** names_out, int32_t cap);

#ifdef __cplusplus
}
#endif
#endif /* TSFX_H_ */
