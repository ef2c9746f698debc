"""CPU emulations (numpy) of the two reformulations in the short-series SEQ kernel (csrc/k_seq.cu, k_seq_small):

  * permutation patterns: the windows are sorted once by the key brev(order bits) | (8 - m), m = min(8, samples from
    the window's start).  Equal patterns of every dimension then sit in contiguous runs, and adding, per run,
    V(last + 1) - V(first) (V = windows valid for D before a sorted position, valid meaning m >= D) to the run's Lehmer
    bin gives exactly the per-dimension histograms; the valid keys' Lehmer codes, sorted, are the codes of the
    dimension-7 and -8 run-length loop;
  * Lempel-Ziv symbols: truncating (v - vmin) * (1 / step) instead of (v - vmin) / step as the estimate that lz_symbol
    corrects against the exact edges gives the same symbols, and the two estimates differ by at most one.
"""
import math

import numpy as np
import pytest

PAD = 0xFFFFFFFF
PAIRS = [(p, q) for q in range(1, 8) for p in range(q)]          # bit q(q-1)/2 + p is [w_q < w_p]
_REV8 = np.array([int("{:08b}".format(i)[::-1], 2) for i in range(256)], dtype=np.uint64)


def brev32(u):
    u = np.asarray(u, dtype=np.uint64)
    return ((_REV8[u & 0xFF] << 24) | (_REV8[(u >> 8) & 0xFF] << 16) | (_REV8[(u >> 16) & 0xFF] << 8)
            | _REV8[(u >> 24) & 0xFF])


def order_bits(x, starts):
    """pe_order_bits of every window: pairwise order bits of the first m = min(8, n - start) samples"""
    n = len(x)
    xp = np.concatenate([x, np.zeros(8, x.dtype)])
    w = xp[starts[:, None] + np.arange(8)[None, :]]
    m = np.minimum(8, n - starts)
    bits = np.zeros(len(starts), dtype=np.uint64)
    for p, q in PAIRS:
        bits |= ((q < m) & (w[:, q] < w[:, p])).astype(np.uint64) << np.uint64(q * (q - 1) // 2 + p)
    return bits, m


def lehmer_of_bits(bits, D):
    code = np.zeros(len(bits), dtype=np.int64)
    for p in range(D - 1):
        mask = sum(1 << (q * (q - 1) // 2 + p) for q in range(p + 1, D))
        digit = np.array([bin(int(b) & mask).count("1") for b in bits], dtype=np.int64)
        code = code * (D - p) + digit
    return code


def lehmer_direct(x, st, D):
    """the Lehmer code of the window's stable ranks: digit p = #{q > p : w_q < w_p}"""
    w = x[st:st + D]
    code = 0
    for p in range(D - 1):
        code = code * (D - p) + int(np.sum(w[p + 1:] < w[p]))
    return code


def sorted_keys(x, tau):
    n = len(x)
    wmax = (n - 2) // tau + 1 if n >= 2 else 0
    starts = np.arange(wmax) * tau
    bits, m = order_bits(x, starts)
    keys = brev32(bits) | (8 - m).astype(np.uint64)
    return np.sort(np.concatenate([keys, np.full(256 - wmax, PAD, np.uint64)]))


def histogram_by_runs(keys, D):
    L = D * (D - 1) // 2
    pm = np.uint64((0xFFFFFFFF << (32 - L)) & 0xFFFFFFFF)
    pre = keys & pm
    valid = ((keys & np.uint64(15)) <= np.uint64(8 - D)).astype(np.int64)
    incl = np.cumsum(valid)
    excl = incl - valid
    first = np.r_[True, pre[1:] != pre[:-1]]
    last = np.r_[pre[1:] != pre[:-1], True]
    delta = np.where(last, incl, 0) - np.where(first, excl, 0)
    hist = np.zeros(math.factorial(D), dtype=np.int64)
    nz = delta != 0
    np.add.at(hist, lehmer_of_bits(brev32(keys[nz]), D), delta[nz])
    return hist, lehmer_of_bits(brev32(keys[valid == 1]), D)


SERIES = {
    "random": lambda rng, n: rng.standard_normal(n).astype(np.float32),
    "tied": lambda rng, n: rng.integers(0, 3, n).astype(np.float32),
    "constant": lambda rng, n: np.full(n, 0.25, np.float32),
}


@pytest.mark.parametrize("kind", list(SERIES))
@pytest.mark.parametrize("tau", [1, 2, 3])
def test_runs_of_sorted_keys_give_the_lehmer_histograms(kind, tau):
    rng = np.random.default_rng(7 + tau)
    for n in range(1, 257):
        x = SERIES[kind](rng, n)
        keys = sorted_keys(x, tau)
        for D in range(2, 9):
            want = np.zeros(math.factorial(D), dtype=np.int64)
            codes = [lehmer_direct(x, st, D) for st in range(0, n - D + 1, tau)]
            np.add.at(want, np.array(codes, dtype=np.int64), 1)
            hist, valid_codes = histogram_by_runs(keys, D)
            assert np.array_equal(hist, want), (kind, tau, n, D)
            assert np.array_equal(np.sort(valid_codes), np.sort(np.array(codes, dtype=np.int64))), (kind, tau, n, D)


def _to_int(q):
    """cvt.rzi.s32.f64: truncation toward zero, NaN to 0"""
    return 0 if math.isnan(q) else int(max(min(q, 2.0 ** 31 - 1), -2.0 ** 31))


def lz_symbol(c, v, vmin, vmax, step, bins):
    c = min(max(c, 0), bins)
    edge = lambda i: vmax if i == bins else np.float64(i) * step + vmin
    while c < bins and edge(c + 1) < v:
        c += 1
    while c > 0 and not (edge(c) < v):
        c -= 1
    return c


def test_reciprocal_estimate_gives_the_division_symbols():
    rng = np.random.default_rng(3)
    ranges = [(np.float32(-1.7), np.float32(2.3)), (np.float32(0), np.float32(1)), (np.float32(1e8), np.float32(1e8 + 64)),
              (np.float32(-3e-30), np.float32(5e-30)), (np.float32(7.5), np.float32(7.5))]
    ranges += [tuple(np.sort(rng.standard_normal(2).astype(np.float32) * np.float32(10.0 ** rng.integers(-3, 4))))
               for _ in range(20)]
    for lo32, hi32 in ranges:
        vmin, vmax = np.float64(lo32), np.float64(hi32)
        for bins in range(1, 128):
            step = (vmax - vmin) / np.float64(bins)
            with np.errstate(divide="ignore", invalid="ignore"):
                rstep = np.float64(1.0) / step
            # float32 samples on, just below and just above every edge, and the ends
            vals = {lo32, hi32}
            for i in range(1, bins + 1):
                e = np.float32(vmax if i == bins else np.float64(i) * step + vmin)
                vals |= {e, np.nextafter(e, np.float32(-np.inf)), np.nextafter(e, np.float32(np.inf))}
            vals = [v for v in vals if lo32 <= v <= hi32]
            edges = np.linspace(vmin, vmax, bins + 1)[1:]
            for v32 in vals:
                v = np.float64(v32)
                with np.errstate(divide="ignore", invalid="ignore"):
                    c_div = _to_int((v - vmin) / step)
                    c_rcp = _to_int((v - vmin) * rstep)
                assert abs(c_rcp - c_div) <= 1, (lo32, hi32, bins, v32)
                want = lz_symbol(c_div, v, vmin, vmax, step, bins)
                assert lz_symbol(c_rcp, v, vmin, vmax, step, bins) == want, (lo32, hi32, bins, v32)
                assert want == int(np.searchsorted(edges, v, side="left")), (lo32, hi32, bins, v32)
