// tsfx_roll.cuh -- the window arithmetic of roll_time_series (dataframe_functions.py:340-373, 548-562), shared by the
// host enumeration (tsfx_roll_windows) and the device one (tsfx_roll_staged).
//
// rolling_direction > 0: the shifts are reversed(range(Lmax, 0, -rolling_direction)) where Lmax is the LONGEST series
// of the frame (:555-560), so window ends are anchored to Lmax for every series; shift t applies to a series of length
// L when t <= L, the window is rows [max(t-max_timeshift-1, 0), t), kept when it has at least min_timeshift+1 rows, and
// its id is (parent id, time of row t-1).
// rolling_direction < 0 (:351-356, 365-366): shifts range(1, Lmax+1, |rolling_direction|), the window is rows
// [t-1, min(t+max_timeshift, L)), same minimum length, id = (parent id, time of row t-1) -- the window's FIRST row.
// Row t-1 is therefore "the row whose sort value names the window": last row (positive) / first row (negative).
#pragma once
#include <stdint.h>

namespace tsfx {

struct RollSpec {
    int32_t dir;          // rolling_direction (!= 0)
    int32_t amount;       // |rolling_direction|
    int32_t first;        // smallest shift; the others follow every `amount`
    int32_t max_ts;       // max_timeshift (>= 0)
    int32_t min_ts;       // min_timeshift (>= 0)
};

__host__ __device__ inline RollSpec roll_spec(int32_t rolling_direction, int32_t max_timeshift, int32_t min_timeshift,
                                              int32_t Lmax) {
    RollSpec R;
    R.dir = rolling_direction;
    R.amount = rolling_direction > 0 ? rolling_direction : -rolling_direction;
    R.first = rolling_direction > 0 ? (Lmax > 0 ? Lmax - ((Lmax - 1) / R.amount) * R.amount : 1) : 1;
    R.max_ts = max_timeshift;
    R.min_ts = min_timeshift;
    return R;
}

// Window of shift t (1 <= t <= L) of a series of L rows: rows [*lo, *lo + length); returns the length.  The length
// grows with t for a positive direction and shrinks with t for a negative one.
__host__ __device__ inline int32_t roll_window(const RollSpec& R, int32_t L, int32_t t, int32_t* lo) {
    if (R.dir > 0) {
        const int32_t b = t - R.max_ts - 1;
        *lo = b < 0 ? 0 : b;
        return t - *lo;
    }
    *lo = t - 1;
    const int64_t hi = (int64_t)*lo + R.max_ts + 1;
    return (int32_t)((hi < L ? hi : (int64_t)L) - *lo);
}

// The kept shifts of a series of L rows (windows of at least min_timeshift + 1 rows): returns their number, *t0 is the
// first and the others follow every R.amount.  By the monotone lengths above, the dropped shifts are a prefix (positive
// direction: t < min_timeshift + 1) or a suffix (negative: t > L - min_timeshift); none is kept when
// max_timeshift < min_timeshift.
__host__ __device__ inline int64_t roll_kept(const RollSpec& R, int32_t L, int32_t* t0) {
    *t0 = R.first;
    if (R.max_ts < R.min_ts) return 0;
    int64_t lo = R.first, hi = L;
    if (R.dir > 0) lo = lo > (int64_t)R.min_ts + 1 ? lo : (int64_t)R.min_ts + 1;
    else hi = (int64_t)L - R.min_ts;
    lo = R.first + (lo - R.first + R.amount - 1) / R.amount * R.amount;      // first shift >= lo
    if (lo > hi) return 0;
    *t0 = (int32_t)lo;
    return (hi - lo) / R.amount + 1;
}

}  // namespace tsfx
