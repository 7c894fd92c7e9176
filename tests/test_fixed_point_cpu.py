"""CPU model of the CSR K1's two-word fixed-point gradient accumulation (ml-ease_b200/csrc/k1_score_grad.cu,
k1_csr_fx_kernel): the same float32 operations in numpy, against an exact (fp64) column sum.  It pins the scale
selection (no 32-bit overflow at the worst-case bound) and the resolution claim in DESIGN.md, and shows that the result
does not depend on the order in which contributions arrive (integer addition commutes), which is what makes the
pass deterministic on the GPU."""
import numpy as np


def _scales(rows_per_cta, wmax, vmax, has_bias=True):
    bound = np.float32(rows_per_cta) * np.float32(wmax) * np.float32(max(vmax, 1.0 if has_bias else 0.0))
    if not (bound > 0) or not np.isfinite(bound):
        bound = np.float32(1.0)
    e_hi = 29 - (int(np.floor(np.log2(float(bound)))) + 1)           # ilogbf(bound) + 1 = number of integer bits
    kbits = 30 - int(rows_per_cta).bit_length()                       # 64 - clzll(per)
    kbits = max(0, min(kbits, 24))
    return e_hi, kbits


def _accumulate(contrib, e_hi, kbits):
    """contrib: float32 contributions c to ONE column.  Returns (hi_sum, lo_sum) as Python ints (checked for int32 range)."""
    s_hi = np.float32(2.0) ** np.float32(e_hi)
    s_k = np.float32(2.0) ** np.float32(kbits)
    ts = (contrib.astype(np.float32) * s_hi).astype(np.float32)       # exact: power-of-two scaling
    h = np.rint(ts).astype(np.float32)
    lo = np.rint(((ts - h).astype(np.float32) * s_k).astype(np.float32)).astype(np.int64)
    hi = h.astype(np.int64)
    run_hi, run_lo = np.cumsum(hi), np.cumsum(lo)                     # every prefix must fit 32 bits, whatever the order
    assert np.abs(run_hi).max(initial=0) < 2 ** 31 and np.abs(run_lo).max(initial=0) < 2 ** 31
    return int(hi.sum()), int(lo.sum())


def _value(hi, lo, e_hi, kbits):
    return (hi + lo * 2.0 ** -kbits) * 2.0 ** -e_hi


def test_worst_case_bound_does_not_overflow_and_is_order_independent():
    rng = np.random.default_rng(0)
    for rows, wmax, vmax in ((6757, 1.0, 5.3), (20409, 2.0, 1.0), (131072, 7.5, 1e3), (64, 1e-4, 1e-3), (1_000_000, 1.0, 10.0)):
        e_hi, kbits = _scales(rows, wmax, vmax)
        worst = np.full(rows, np.float32(wmax) * np.float32(vmax), np.float32)   # every row hits the column with the largest value
        hi, lo = _accumulate(worst, e_hi, kbits)
        exact = float(np.sum(worst.astype(np.float64)))
        assert abs(_value(hi, lo, e_hi, kbits) - exact) <= rows * 2.0 ** -(e_hi + kbits)
        c = (rng.normal(size=rows) * wmax * vmax / 4).astype(np.float32).clip(-wmax * vmax, wmax * vmax)
        a = _accumulate(c, e_hi, kbits)
        b = _accumulate(c[rng.permutation(rows)], e_hi, kbits)
        assert a == b                                                  # bit-identical sums in any arrival order


def test_resolution_is_below_float32_rounding_of_the_contributions():
    rng = np.random.default_rng(1)
    rows, wmax, vmax = 7576, 1.0, 5.0                                  # config 3: 1M rows over 132 CTAs, N(0,1) values
    e_hi, kbits = _scales(rows, wmax, vmax)
    assert kbits >= 16
    n_hit = 76                                                          # ~1 % of the CTA's rows touch a given column
    c = (rng.normal(size=n_hit) * 0.5).astype(np.float32)
    hi, lo = _accumulate(c, e_hi, kbits)
    exact = float(np.sum(c.astype(np.float64)))
    err = abs(_value(hi, lo, e_hi, kbits) - exact)
    quantum = 2.0 ** -(e_hi + kbits)
    assert err <= 0.5 * quantum * n_hit
    assert quantum < 2.0 ** -24 * np.abs(c).max()                       # finer than the fp32 spacing of the contributions themselves
    # a float32 running sum (what float atomics would give) is no better than this
    f32 = np.float32(0)
    for x in c:
        f32 = np.float32(f32 + x)
    assert err <= abs(float(f32) - exact) + 0.5 * quantum * n_hit
