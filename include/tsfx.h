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

#define TSFX_VERSION 4

/* error codes */
#define TSFX_OK 0
#define TSFX_E_INVALID (-1)     /* bad argument / malformed plan */
#define TSFX_E_CUDA (-2)        /* CUDA runtime failure (message has the cudaError string) */
#define TSFX_E_UNSUPPORTED (-3) /* parameter combination without a GPU implementation */
#define TSFX_E_TOO_LONG (-4)    /* the longest series exceeds a kernel group's limit: 21 000 samples for a plan with
                                   sample_entropy / approximate_entropy, else 131 072 unless every calculator of the plan
                                   is in BASIC / SORTED (no limit); checked before any group runs */
#define TSFX_E_NOMEM (-5)
#define TSFX_E_NAN (-6)         /* NaN in the value column (data.py:148-167 raises ValueError) */

/* flags */
#define TSFX_FLAG_DEVICE_PTRS 1u /* values/begin/len/out are device pointers; async on ctx stream */
#define TSFX_FLAG_TIMING 2u      /* record CUDA events around every kernel group (tsfx_get_timings) */
#define TSFX_FLAG_NO_NAN_CHECK 4u /* host-pointer extract calls scan the values for NaN and return TSFX_E_NAN (the reference
                                  * raises ValueError, data.py:148-167); this flag skips the scan.  Device-pointer calls
                                  * (asynchronous) scan only with TSFX_FLAG_CHECK_DEVICE_INPUT. */
#define TSFX_FLAG_IMPUTE 8u      /* extract calls: impute the feature matrix on the device before it is returned
                                  * (extract_features(impute_function=impute), extraction.py:179-181, 286-287) */
#define TSFX_FLAG_ALL_MEDIANS 16u /* tsfx_impute: compute every column's median, not only those a NaN needs */
#define TSFX_FLAG_CHECK_DEVICE_INPUT 32u /* with TSFX_FLAG_DEVICE_PTRS, tsfx_extract_csr / tsfx_extract_dense first make ONE
                                  * pass over the input on the device and synchronise the stream once to read its result:
                                  * the longest series (tsfx_set_max_len_hint is ignored), every (begin, len) view inside
                                  * [0, n_values) with len >= 1 (else TSFX_E_INVALID), and no NaN among the values the
                                  * series cover (else TSFX_E_NAN).  No kernel group runs on input that fails the pass,
                                  * so tsfx_last_launch_count is 0 after such an error. */
#define TSFX_FLAG_KEEP_SORT_KEYS 64u /* tsfx_stage_long_stacked: keep every staged row's sort key, which tsfx_roll_staged
                                  * names its windows by (without the flag the call does no extra work) */
#define TSFX_FLAG_KEEP_ROW_NUMBERS 128u /* tsfx_stage_long_stacked: keep every staged row's input row number (4 bytes per row),
                                  * which tsfx_roll_staged with TSFX_FLAG_FORECAST finds the targets by */
#define TSFX_FLAG_FORECAST 256u  /* tsfx_roll_staged: make_forecasting_frame's windows (see tsfx_staged_targets) */
#define TSFX_FLAG_DEFER_CHECK 512u /* with TSFX_FLAG_DEVICE_PTRS, tsfx_extract_csr / tsfx_extract_dense validate the input on
                                  * the device and report to the status buffer of tsfx_set_status instead of returning an
                                  * error; see "Deferred input check" below */

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
    TSFX_AUGMENTED_DICKEY_FULLER,                      /* :499  attr=teststat|pvalue|usedlag i0=autolag (TSFX_AUTOLAG_*) */
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
    TSFX_LINEAR_TREND,                                 /* :1343 attr=pvalue|rvalue|intercept|slope|stderr|intercept_stderr */
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
/* f_agg: numpy reducers (var and std with ddof 0; ptp = max - min).  agg_linear_trend takes mean, median, var, std, max
 * and min.  agg_autocorrelation and change_quantiles take every code, and OR'ed with TSFX_AGG_NANSKIP the np.nan*
 * variant, which skips NaN: on no value left nansum gives 0, nanprod 1 and the others NaN. */
enum { TSFX_AGG_MEAN = 0, TSFX_AGG_MEDIAN, TSFX_AGG_VAR, TSFX_AGG_STD, TSFX_AGG_MAX, TSFX_AGG_MIN, TSFX_AGG_PTP,
       TSFX_AGG_SUM, TSFX_AGG_PROD };
#define TSFX_AGG_NANSKIP 16
enum { TSFX_FFT_REAL = 0, TSFX_FFT_IMAG, TSFX_FFT_ABS, TSFX_FFT_ANGLE };
enum { TSFX_SPEC_CENTROID = 0, TSFX_SPEC_VARIANCE, TSFX_SPEC_SKEW, TSFX_SPEC_KURTOSIS };
/* linregress attributes; intercept_stderr = stderr * sqrt(ssxm + xmean^2) (scipy.stats.linregress) */
enum { TSFX_LR_PVALUE = 0, TSFX_LR_RVALUE, TSFX_LR_INTERCEPT, TSFX_LR_SLOPE, TSFX_LR_STDERR, TSFX_LR_INTERCEPT_STDERR };
enum { TSFX_ADF_TESTSTAT = 0, TSFX_ADF_PVALUE, TSFX_ADF_USEDLAG, TSFX_ADF_BADATTR };
/* adfuller autolag: AIC / BIC (smallest criterion), TSTAT ("t-stat": from the longest model down, the first whose last
 * lag has |t| >= 1.6448536269514722, else no lag), NONE (maxlag) */
enum { TSFX_AUTOLAG_AIC = 0, TSFX_AUTOLAG_BIC, TSFX_AUTOLAG_NONE, TSFX_AUTOLAG_TSTAT };

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
/* Rebinds the stream the context's calls are enqueued on, so one context (and its working memory) serves whichever
 * stream the caller is on.  cuda_stream is a stream of the context's device, or NULL for the stream the context was
 * created with; pass cudaStreamLegacy ((void*)1) for the legacy default stream.  The new stream first waits for
 * everything already enqueued on the old one (the calls reuse the context's scratch); the side streams, copy streams
 * and timing events of later calls fork from and join to the new stream.  Does not block the host.  When the old or the
 * new stream is capturing a CUDA graph, the new stream does not wait (an event recorded on one side of a capture cannot
 * order work on the other): ordering the graph's launches against other work on the context is then the caller's. */
int tsfx_ctx_set_stream(tsfx_ctx* ctx, void* cuda_stream);
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

/* Row stride (in doubles) of `out` for the following device-pointer tsfx_extract_csr / tsfx_extract_dense calls, so
 * that several plans (one per kind) fill column blocks of one matrix: row s of a call goes to out + s * ld.  ld must be
 * >= the plan's n_cols (else the call returns TSFX_E_INVALID); 0 removes the setting (ld = n_cols).  A strided call
 * cannot take TSFX_FLAG_IMPUTE (imputation needs every column of the matrix: impute it afterwards with tsfx_impute). */
int tsfx_set_out_ld(tsfx_ctx* ctx, int32_t ld);

/* Row timestamps for linear_trend_timewise (feature_calculators.py:2274-2306: the regressor is the series' DatetimeIndex,
 * hours since its first row).  row_time_ns[i] is the timestamp (int64 nanoseconds) of row i of the `values` array of the
 * NEXT extract call on this context (host pointer, or device pointer with TSFX_FLAG_DEVICE_PTRS); that call consumes
 * them (tsfx_extract_long carries them through its sort).  A plan with linear_trend_timewise columns and no row times
 * is TSFX_E_INVALID. */
int tsfx_set_row_times(tsfx_ctx* ctx, const int64_t* row_time_ns, int64_t n_rows, uint32_t flags);

/* Deferred input check, for calls that only enqueue work (no allocation, copy to the host or synchronisation), so that
 * they overlap other work and can be captured in a CUDA graph:
 *   tsfx_prepare       does ahead of time every lazy step a device-pointer call of `plan` with at most n_series series of
 *                      at most max_len samples takes: the length check (TSFX_E_TOO_LONG), the working memory (256 MB, or
 *                      1 GB for max_len > 1 024, plus the staging matrices and the check's per-series buffers) and the
 *                      FFT / Ricker tables.  Blocks until the tables are filled.  Prepare every plan a context will run, before
 *                      capturing any call in a graph: a later, larger tsfx_prepare may move the working memory.
 *   tsfx_set_status    the caller's device buffer of TSFX_STATUS_WORDS int64 words (zeroed by the caller) that the
 *                      following TSFX_FLAG_DEFER_CHECK calls report to; NULL removes it.
 * A TSFX_FLAG_DEFER_CHECK call (needs TSFX_FLAG_DEVICE_PTRS and a prepared shape, and excludes
 * TSFX_FLAG_CHECK_DEVICE_INPUT and TSFX_FLAG_IMPUTE) makes one pass over its input that rejects a series for a NaN value,
 * an invalid view (len < 1, begin < 0 or begin + len > n_values) or a view longer than the declared max_len (CSR: the
 * tsfx_set_max_len_hint value, which is then required; dense: len).  CSR calls hand the groups private views, in which a
 * rejected view is the one-sample view (0, 1); dense calls hand them the input as it is.  After the groups, every column
 * of a rejected series is set to NaN in `out` (honouring tsfx_set_out_ld).  The call then counts itself in
 * status[TSFX_STATUS_CALLS] and, if no earlier call since the caller last zeroed status[TSFX_STATUS_BAD] rejected a
 * series and this one did, stores the count in status[TSFX_STATUS_BAD] and the call's first series of each reason in the
 * three reason words (-1: none). */
#define TSFX_STATUS_CALLS 0
#define TSFX_STATUS_BAD 1
#define TSFX_STATUS_VIEW 2       /* first series with an invalid view */
#define TSFX_STATUS_LONG 3       /* first valid series longer than max_len */
#define TSFX_STATUS_NAN 4        /* first other series with a NaN value */
#define TSFX_STATUS_KIND 5       /* tsfx_extract_long_deferred: 1 when a kind code is outside 0 .. n_kinds-1 */
#define TSFX_STATUS_KEY_NAN 6    /* tsfx_extract_long_deferred: 1 when a float64 sort key is NaN */
#define TSFX_STATUS_IDS 7        /* tsfx_extract_long_deferred: the number of distinct ids when it exceeds max_ids, else 0 */
#define TSFX_STATUS_ID 2         /* tsfx_extract_long_deferred (whose slot views are never invalid): the id its report
                                  * names -- the first id past max_ids, else the id of the first series longer than max_len,
                                  * else -1 */
#define TSFX_STATUS_WORDS 8
int tsfx_prepare(tsfx_ctx* ctx, const tsfx_plan* plan, int64_t n_series, int32_t max_len);
int tsfx_set_status(tsfx_ctx* ctx, int64_t* status);

/* Deferred long format: tsfx_stage_long_stacked + tsfx_extract_staged in one call that only enqueues work, for a prepared
 * shape, so that it overlaps other work and can be captured in a CUDA graph:
 *   tsfx_prepare_long          plans[k] is kind k's plan (NULL: the kind has no columns), 1 <= n_kinds <= 64; the calls
 *                              take at most max_rows rows (<= 2^31 - 4 098) with at most max_ids distinct ids and
 *                              series of at most max_len samples (TSFX_E_TOO_LONG beyond a plan's limit).  Reserves every
 *                              buffer of the stage for max_rows rows, the slot and check buffers of n_kinds x max_ids
 *                              series, a staging block of max_ids x n_cols(k) doubles per kind, and calls tsfx_prepare for
 *                              every plan with (max_ids, max_len).  Blocks.  The plans must outlive the calls; a later
 *                              tsfx_prepare_long, tsfx_prepare or stage call on the context may move the working memory.
 *   tsfx_extract_long_deferred n_rows device rows (ids, sort_keys, values, kind_codes as tsfx_stage_long_stacked takes them,
 *                              TSFX_FLAG_DEVICE_PTRS required, no other flag), of which rows [0, *n_rows_live) count
 *                              (n_rows_live: a device int64, clamped to 0 .. n_rows; NULL: all n_rows).  Fills out
 *                              ([max_ids x ld] row-major float64, ld >= the total column count of all kinds, blocks in
 *                              kind order): rows [0, *n_ids) are tsfx_extract_staged's rows for the live rows, every
 *                              other cell NaN -- a kind without rows has NaN columns; out_ids (max_ids int64) gets the
 *                              union ids ascending, then INT64_MAX; *n_ids (device int64) the union size.  Errors are
 *                              the deferred input check's, reported to the tsfx_set_status words (required): a kind
 *                              code out of range, a NaN float64 sort key or more than max_ids distinct ids reject the
 *                              call (out all NaN, *n_ids 0, TSFX_STATUS_KIND / _KEY_NAN / _IDS); a NaN value, or more
 *                              than max_len samples, in the series of one (id, kind) makes that series' cells NaN
 *                              (TSFX_STATUS_NAN / _LONG: its slot k * max_ids + i, the i-th series of kind k in id
 *                              order; TSFX_STATUS_ID: the id).  One call counts once in TSFX_STATUS_CALLS.  The call
 *                              makes no allocation, no copy to the host and no synchronisation; a call that would need
 *                              more than was prepared returns TSFX_E_INVALID (n_rows) or TSFX_E_CUDA before any work. */
int tsfx_prepare_long(tsfx_ctx* ctx, const tsfx_plan* const* plans, int32_t n_kinds, int64_t max_rows, int64_t max_ids,
                      int32_t max_len);
int tsfx_extract_long_deferred(tsfx_ctx* ctx, const int64_t* ids, const void* sort_keys, int32_t sort_key_is_f64,
                               const float* values, const void* kind_codes, int32_t kind_code_is_i64, int64_t n_rows,
                               const int64_t* n_rows_live, int64_t* out_ids, int64_t* n_ids, double* out, int32_t ld,
                               uint32_t flags);
/* Longest series a plan of these columns accepts (TSFX_E_TOO_LONG beyond; 2^31 - 1 when no group limits it), or
 * TSFX_E_INVALID for an unknown calculator.  Needs no context or device. */
int32_t tsfx_plan_max_len(const tsfx_feature_desc* descs, int32_t n_descs);

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
 * Host pointers may be pageable (staged through pinned memory by worker threads) or page-locked; TSFX_FLAG_DEVICE_PTRS
 * is TSFX_E_INVALID.  Rows already on the device go through tsfx_stage_long_stacked + tsfx_extract_staged: with
 * kind_codes NULL and n_kinds 1 they give the same ids and matrix. */
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

/* Long format with a KIND column (data.py:233-291 LongTsFrameAdapter): rows (ids[i], sort_keys[i], kind_codes[i],
 * values[i]) in any order, all of them device pointers (TSFX_FLAG_DEVICE_PTRS is required).  The result has one row per
 * id of ANY kind, ids ascending, and one column block per kind -- the frame PartitionedTsData.pivot builds (data.py:
 * 86-121) -- so its row count is only known after grouping.  Extraction therefore takes two calls on the context:
 *   tsfx_stage_long_stacked  partitions the rows by kind code (kind_codes int32, or int64 with kind_code_is_i64; NULL:
 *                            every row is kind 0) with a stable counting sort, orders every kind's rows by (id, sort key)
 *                            as tsfx_extract_long does (sort_keys NULL = keep row order; stable for equal keys), takes
 *                            the union of the kinds' ids, synchronises the stream once and returns the union size
 *                            in *n_ids_out, and per kind its row count and longest series (arrays of n_kinds entries,
 *                            host).  row_time_ns (optional, int64 ns per row) follows the rows for linear_trend_timewise.
 *                            TSFX_E_INVALID for a code outside 0 .. n_kinds-1 (1 <= n_kinds <= 64), TSFX_E_NAN for a
 *                            NaN value or float64 sort key, TSFX_E_UNSUPPORTED for more than 2^31 - 4 098 rows.  The staged rows
 *                            live in the context's working region until the next stage call.
 *   tsfx_extract_staged      consumes what the last stage call staged: plans[k] is kind k's plan (may be NULL for a
 *                            kind without rows, which contributes no columns).  Checks every kind's length limit
 *                            (TSFX_E_TOO_LONG) before any kernel runs, then fills out ([n_ids x ld] row-major float64,
 *                            device) with NaN where an id has no rows of a kind, writes each kind's columns at its
 *                            column offset (blocks in kind order) and the union ids to out_ids (device).  ld >= the
 *                            total column count; TSFX_FLAG_IMPUTE (needs ld == that count) imputes the matrix after.
 *                            Asynchronous on the context's stream. */
int tsfx_stage_long_stacked(tsfx_ctx* ctx, const int64_t* ids, const void* sort_keys, int32_t sort_key_is_f64,
                            const float* values, const void* kind_codes, int32_t kind_code_is_i64, int32_t n_kinds,
                            const int64_t* row_time_ns, int64_t n_rows, int64_t* n_ids_out, int64_t* rows_per_kind,
                            int32_t* max_len_per_kind, uint32_t flags);
int tsfx_extract_staged(tsfx_ctx* ctx, const tsfx_plan* const* plans, int64_t* out_ids, double* out, int32_t ld,
                        uint32_t flags);

/* Rolled windows of staged rows (extract_features(roll_time_series(df, column_kind=...)), dataframe_functions.py:
 * 376-603), between the two calls above:
 *   tsfx_roll_staged      turns the staged series into staged windows, with the window arithmetic of tsfx_roll_windows:
 *                         every kind rolls on its own, the shifts anchored to the longest (kind, id) series of the call.
 *                         max_timeshift 0 means None (the longest series).  A window is a view on the staged values, so
 *                         each kind keeps its row alignment.  A window is named (id, sort key of its naming row: last
 *                         row for a positive direction, first for a negative one), or (id, row number of that row in
 *                         its series) when the rows were staged without sort keys; the staged rows are the union of
 *                         the names over all kinds, ascending.  Needs TSFX_FLAG_KEEP_SORT_KEYS on the stage call when
 *                         sort keys were given.  Synchronises the stream once and returns the number of union windows
 *                         in *n_rows_out and the longest window of every kind in max_len_per_kind (host, n_kinds
 *                         entries; the exact longest window, which tsfx_extract_staged checks against each plan's
 *                         limit).  TSFX_E_INVALID when two windows of one kind have the same name (sort keys tied at
 *                         their naming rows; the reference would merge them into one series).  No feature kernel runs.
 *                         flags: 0, or TSFX_FLAG_FORECAST (below).  TSFX_E_INVALID when the staged rows are already
 *                         rolled or packaged (tsfx_sub_staged).
 *   tsfx_staged_row_keys  copies the naming sort keys (raw int64 / float64 bits as staged, float64 -0.0 as +0.0; row
 *                         numbers as int64 without sort keys) of the n_rows_out staged windows to out_keys (device, 8
 *                         bytes each), asynchronously.  Valid until the next stage call.  After tsfx_sub_staged it
 *                         copies the package numbers (int64) of the staged packages instead.
 * tsfx_extract_staged then extracts the windows: out_ids receives the id of every union window. */
int tsfx_roll_staged(tsfx_ctx* ctx, int32_t rolling_direction, int32_t max_timeshift, int32_t min_timeshift,
                     int64_t* n_rows_out, int32_t* max_len_per_kind, uint32_t flags);
int tsfx_staged_row_keys(tsfx_ctx* ctx, void* out_keys);

/* Forecasting windows (make_forecasting_frame, dataframe_functions.py:606-680): tsfx_roll_staged with TSFX_FLAG_FORECAST,
 * on rows staged with TSFX_FLAG_KEEP_ROW_NUMBERS (else TSFX_E_INVALID), rolls as above and then drops every window's last
 * row, leaving out the windows that this empties (those of one row; the kept windows have at least
 * max(min_timeshift, 1) + 1 rows before the drop).  Names, union rows and the one synchronisation are as without the flag;
 * max_len_per_kind is the longest window after the drop.  Two windows of one kind with the same name are TSFX_E_INVALID
 * as without the flag, counting the one-row windows that the drop empties: the reference names them too and merges each
 * with a window of the same name before it drops a row.
 *   tsfx_staged_targets   copies the target of each of the n_rows_out staged windows to out_rows (device, int64),
 *                         asynchronously: the input row number of the row that names the window (the row the window
 *                         forecasts is that row's value), or -1 when that is input row 0 (the reference's y = x[1:] has
 *                         no entry for it).  A union row that several kinds' windows share takes the target of its
 *                         lowest kind's window.  TSFX_E_INVALID unless the last roll had TSFX_FLAG_FORECAST; valid until
 *                         the next stage call.
 * The targets are row numbers, so the caller gathers the target values from its own copy of the input in any dtype. */
int tsfx_staged_targets(tsfx_ctx* ctx, int64_t* out_rows);

/* Fixed-length packages of staged rows (extract_features(add_sub_time_series_index(df, sub_length, ...)),
 * dataframe_functions.py:683-784), between tsfx_stage_long_stacked and tsfx_extract_staged:
 *   tsfx_sub_staged       cuts every staged (kind, id) series, in (id, sort key) order, into packages of sub_length rows,
 *                         the last one shorter: package k is rows [k * sub_length, min((k + 1) * sub_length, n)).  A
 *                         package is a view on the staged values, so each kind keeps its row alignment.  A package is
 *                         named (package number, parent id); the staged rows become the union of the names over all
 *                         kinds, ascending in (package number, parent id).  Synchronises the stream once and returns the
 *                         number of union packages in *n_rows_out and the longest package of every kind in
 *                         max_len_per_kind (host, n_kinds entries; checked by tsfx_extract_staged against each plan's
 *                         limit).  TSFX_E_INVALID for sub_length < 1, and when the staged rows are already rolled or
 *                         packaged (stage them again).  No feature kernel runs.  No flags are defined for it yet: pass 0.
 * tsfx_staged_row_keys then gives the package numbers (int64), and tsfx_extract_staged's out_ids the parent ids. */
int tsfx_sub_staged(tsfx_ctx* ctx, int64_t sub_length, int64_t* n_rows_out, int32_t* max_len_per_kind, uint32_t flags);

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
