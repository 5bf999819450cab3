"""Executable version of the argument behind quantize_scan_kernel's arithmetic (csrc/cdf.cuh): the fixed-point weight
q = floor(w * 2^e), with e from the largest weight and the particle count (oracle/beluga_oracle.hpp: fixed_point_exponent,
quantize_weight -- std::ldexp), is computed on the device as floor((w * 2^e1) * 2^(e - e1)), e1 = e / 2: two multiplications
by exact powers of two instead of scalbn.  The claims checked here, with exact rationals:

* the two-step product equals ldexp(w, e) for every weight 0 <= w <= wmax, subnormals and huge values included (a power-of-two
  multiplication is exact unless the result is subnormal, and where the first step can lose bits the result is below 1 anyway);
* both factors are normal doubles for every exponent the rule can produce (the kernel builds them from the exponent field);
* n quantised weights never overflow 64 bits: every q < 2^min(52, 62 - ceil_log2 n), so the total stays below 2^62.

CPU only; it models the arithmetic, it does not run the kernel."""
import math
import sys
from fractions import Fraction

import numpy as np
import pytest


def ceil_log2(n: int) -> int:
    b = 0
    while (1 << b) < n:
        b += 1
    return b


def fixed_point_exponent(wmax: float, n_total: int) -> int:
    return min(52, 62 - ceil_log2(n_total)) - math.frexp(wmax)[1]


def pow2_double(e: int) -> float:
    """cdf.cuh: pow2_double -- the bit pattern (e + 1023) << 52; needs a normal result."""
    assert -1022 <= e <= 1023, e
    return math.ldexp(1.0, e)


DBL_MAX = sys.float_info.max
U64_MAX = (1 << 64) - 1


def double2ull_rd(x: float) -> int:
    """__double2ull_rd (PTX cvt.rmi.u64.f64): round towards -inf, then saturate to [0, 2^64 - 1]; NaN converts to 0."""
    if math.isnan(x) or x <= 0.0:
        return 0
    if x >= 2.0 ** 64:  # +inf included
        return U64_MAX
    return math.floor(x)


def weight_selectable(w: float) -> bool:
    """device_common.cuh: weight_selectable -- the rule weight_order_bits and quantize_mul share."""
    return 0.0 < w <= DBL_MAX


def kernel_quantize(w: float, exponent: int) -> int:
    """cdf.cuh: quantize_mul with the factors quantize_scan_tile builds."""
    if not weight_selectable(w):
        return 0
    e1 = int(exponent / 2)  # C++ integer division truncates towards zero
    return double2ull_rd((w * pow2_double(e1)) * pow2_double(exponent - e1))


def kernel_cdf(weights, n_total: int):
    """quantize_scan_tile over a whole weight set: the exponent from the largest selectable weight (weight_order_bits),
    the uniform fallback (2^20 per particle) when there is none, 64-bit wrap-around sums.  -> (cdf, exponent, valid)."""
    selectable = [w for w in weights if weight_selectable(w)]
    valid = bool(selectable)
    ex = fixed_point_exponent(max(selectable), n_total) if valid else min(52, 62 - ceil_log2(n_total))
    cdf, acc = [], 0
    for w in weights:
        acc = (acc + (kernel_quantize(w, ex) if valid else 1 << 20)) & U64_MAX
        cdf.append(acc)
    return cdf, ex, valid


def oracle_quantize(w: float, exponent: int) -> int:
    if not (w > 0.0):
        return 0
    return math.floor(Fraction(w) * Fraction(2) ** exponent)  # what floor(ldexp(w, e)) is when ldexp is exact -- checked below


WMAX = [1.0, 4205.0, 1e-12, 1e-300, 5e-324, 2.2250738585072014e-308, 1e300, 1.7976931348623157e308, 0.75, 3.0000000000000004, 2.0 ** -1000,
        2.0 ** 1000]


@pytest.mark.parametrize("n_total", [1, 2, 1000, 1_000_000, 12_500_000, 100_000_000, 1 << 31])
@pytest.mark.parametrize("wmax", WMAX)
def test_two_power_of_two_multiplications_equal_ldexp(wmax, n_total):
    e = fixed_point_exponent(wmax, n_total)
    e1 = int(e / 2)
    assert -1022 <= e1 <= 1023 and -1022 <= e - e1 <= 1023  # both factors are normal doubles
    rng = np.random.default_rng(abs(hash((wmax, n_total))) % (1 << 32))
    ws = [wmax, wmax * 0.5, wmax * (1 - 2 ** -53), math.nextafter(wmax, 0.0), 0.0, 5e-324, 2.2250738585072014e-308]
    ws += list(wmax * rng.random(200)) + list(wmax * 2.0 ** -rng.integers(0, 1100, 100).astype(float))
    limit = 1 << min(52, 62 - ceil_log2(n_total))
    for w in ws:
        if not (0.0 <= w <= wmax):
            continue
        q = kernel_quantize(w, e)
        assert q == oracle_quantize(w, e), (w, e)
        assert q == (math.floor(math.ldexp(w, e)) if w > 0.0 else 0)  # and ldexp itself was exact wherever it matters
        assert q < limit or (w == wmax and q <= limit)
    # the largest weight lands in the top octave of the range: the resolution the exponent rule promises
    assert kernel_quantize(wmax, e) >= limit // 2


def test_weights_that_are_never_selected():
    for w in (0.0, -0.0, -1.0, float("nan"), -float("inf"), float("inf")):
        assert kernel_quantize(w, 10) == 0


def test_saturating_conversion():
    assert double2ull_rd(float("inf")) == U64_MAX and double2ull_rd(2.0 ** 64) == U64_MAX and double2ull_rd(2.0 ** 70) == U64_MAX
    assert double2ull_rd(float("nan")) == 0 and double2ull_rd(-float("inf")) == 0 and double2ull_rd(-0.5) == 0
    assert double2ull_rd(2.0 ** 64 - 2048) == (1 << 64) - 2048 and double2ull_rd(1.999) == 1


SPECIAL = [0.0, -0.0, 5e-324, 1e-320, 2.2250738585072009e-308, 2.2250738585072014e-308, 1e-300, 1.0, 3.0, 1e300, DBL_MAX,
           float("inf"), -float("inf"), float("nan"), -1.0, -5e-324, -DBL_MAX]


@pytest.mark.parametrize("n_total", [0, 1 << 20, 1 << 40])
def test_cdf_of_special_values_never_decreases(orc, n_total):
    """Every special double in one weight set, in several orders and with a few of them removed: the modelled kernel CDF
    never goes down, selects only positive finite weights, and equals the oracle's fixed_point_cdf bit for bit."""
    rng = np.random.default_rng(7)
    sets = [list(SPECIAL), SPECIAL[::-1]] + [list(rng.permutation(np.array(SPECIAL, dtype=object))) for _ in range(20)]
    sets += [[w for w in s if not (w == DBL_MAX or w == 1e300)] for s in sets[:6]]  # the largest weight moves down
    sets += [[w for w in s if not weight_selectable(w)] for s in sets[:4]]  # nothing selectable: the uniform fallback
    for ws in sets:
        ws = [float(w) for w in ws]
        cdf, ex, valid = kernel_cdf(ws, n_total or len(ws))
        assert all(b >= a for a, b in zip([0] + cdf, cdf)), ws
        assert cdf[-1] < 1 << 62
        assert valid == any(weight_selectable(w) for w in ws)
        if valid:
            assert all(weight_selectable(w) for a, b, w in zip([0] + cdf, cdf, ws) if b > a)
        _, want, want_ex, want_valid = orc.resample_indices(ws, orc.SYSTEMATIC, seed=1, step=1, n_total=n_total, return_valid=True)
        assert (ex, valid) == (want_ex, want_valid)
        assert [int(v) for v in want] == cdf


@pytest.mark.parametrize("n_total", [1, 3, 1 << 20, (1 << 20) + 1, 100_000_000, 1 << 40])
def test_total_cannot_overflow(n_total):
    per_weight = 1 << min(52, 62 - ceil_log2(n_total))
    assert n_total * per_weight <= 1 << 62
