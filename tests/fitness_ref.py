"""Plain exact restatement of the matcher's fitness arithmetic, for tests/test_fitness_division.py.

div(x, y) is IEEE 754 binary64 division written out: the exact quotient as a Fraction, rounded to nearest with
ties to even, through the subnormal range, with overflow to +-inf and the sign rules of zeros, infinities and
NaN.  fitness() is Fenzo's cpuMemBinPacker as the oracle's eval_pair states it: IEEE sums in its association,
each division correctly rounded, the mean of the two fits, and 0.0 when the request does not fit.
"""
import math
from fractions import Fraction

import numpy as np

MANT = 52                 # stored significand bits of binary64
EMIN = -1022              # exponent of the smallest normal
EMAX = 1023               # exponent of the largest finite binade
TINY = 2.0 ** (EMIN - MANT)   # the smallest subnormal


def _sign(x):
    return math.copysign(1.0, x) < 0


def round_rn(q, negative=False):
    """The binary64 nearest the exact non-negative rational q, ties to even; +-inf past the largest finite."""
    assert q >= 0
    if q == 0:
        return -0.0 if negative else 0.0
    p, r = q.numerator, q.denominator
    e = p.bit_length() - r.bit_length()           # 2^e <= q < 2^(e+1) after the adjustment below
    if (p << max(0, -e)) < (r << max(0, e)):
        e -= 1
    qe = max(e, EMIN) - MANT                       # exponent of one unit in the last place
    scaled = q / Fraction(2) ** qe if qe >= 0 else q * (1 << -qe)
    n, rem = divmod(scaled.numerator, scaled.denominator)
    twice = 2 * rem
    if twice > scaled.denominator or (twice == scaled.denominator and n % 2 == 1):
        n += 1
    if n == 0:
        return -0.0 if negative else 0.0
    if n.bit_length() + qe > EMAX + 1:            # the rounded value reaches 2^1024
        return -math.inf if negative else math.inf
    v = math.ldexp(float(n), qe)                   # n < 2^54 and n 2^qe representable: both exact
    return -v if negative else v


def div(x, y):
    """x / y in binary64, correctly rounded, computed exactly rather than with the float operator."""
    x, y = float(x), float(y)
    neg = _sign(x) != _sign(y)
    if math.isnan(x) or math.isnan(y):
        return math.nan
    if math.isinf(x):
        return math.nan if math.isinf(y) else (-math.inf if neg else math.inf)
    if math.isinf(y):
        return -0.0 if neg else 0.0
    if y == 0.0:
        return math.nan if x == 0.0 else (-math.inf if neg else math.inf)
    return round_rn(abs(Fraction(x)) / abs(Fraction(y)), neg)


def fitness(jc, jm, ac, am, lc, lm, rc, rm):
    """eval_pair's fitness of request (jc, jm) on a VM with (ac, am) assigned this cycle, lease (lc, lm) and
    running (rc, rm): ((req + assigned) + running) / (lease + running) per resource, their mean, and 0.0 when
    assigned + request exceeds the lease in either resource."""
    jc, jm, ac, am, lc, lm, rc, rm = map(float, (jc, jm, ac, am, lc, lm, rc, rm))
    if ac + jc > lc or am + jm > lm:
        return 0.0
    cpu_fit = div((jc + ac) + rc, lc + rc)
    mem_fit = div((jm + am) + rm, lm + rm)
    return div(cpu_fit + mem_fit, 2.0)


# ---- the device's shortcut, restated: what fit_fitness computes when both reciprocals are set -----------------
def fma(a, b, c):
    """a * b + c rounded once."""
    exact = Fraction(a) * Fraction(b) + Fraction(c)
    if exact == 0:
        return -0.0 if (_sign(a) != _sign(b)) and _sign(c) else 0.0
    return round_rn(abs(exact), exact < 0)


def safe_rcp(den):
    """fitness.cuh's safe_rcp: RN(1 / den) for den in (1e-100, 1e100) without an all-ones significand, else 0."""
    frac = int(np.float64(den).view(np.int64)) & ((1 << MANT) - 1)
    return div(1.0, den) if 1e-100 < den < 1e100 and frac != (1 << MANT) - 1 else 0.0


def shortcut_div(x, den, y=None):
    """div_y(x, den, y): q0 = x y, q = fma(fma(-den, q0, x), y, q0); IEEE division when y is 0."""
    y = safe_rcp(den) if y is None else y
    if y == 0.0:
        return div(x, den)
    q0 = float(x) * y
    return fma(fma(-float(den), q0, x), y, q0)


def shortcut_fitness(jc, jm, ac, am, lc, lm, rc, rm):
    """fit_fitness with both reciprocals from safe_rcp: the matcher's fitness without a guard on the dividends."""
    jc, jm, ac, am, lc, lm, rc, rm = map(float, (jc, jm, ac, am, lc, lm, rc, rm))
    if ac + jc > lc or am + jm > lm:
        return 0.0
    return (shortcut_div((jc + ac) + rc, lc + rc) + shortcut_div((jm + am) + rm, lm + rm)) * 0.5
