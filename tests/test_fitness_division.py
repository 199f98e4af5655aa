"""The matcher's fitness arithmetic (cook_b200/csrc/fitness.cuh) against the exact reference of fitness_ref.py.

Without a GPU: fitness_ref.div is pinned on hand cases and against numpy's IEEE division on every family below.
With one (-m gpu, through tests/fold_probe.cu built with the product's flags): the dividend guard fit_guard flips
exactly at its bounds, div_y(x, den, safe_rcp(den)) is bit for bit exact division inside the range it states (and
not below it), and fit_fitness, with the reciprocals init_dyn_kernel sets for a cycle of that one job and VM, is
bit for bit the reference over non-negative finite amounts.

Each family draws the amounts of a (job, VM) pair: request (jc, jm), assigned this cycle (ac, am), lease (lc, lm)
and running (rc, rm).  The cpu side takes the family's operands; the mem side takes them or a grid pair.
"""
import ctypes as C
import math
import os

import numpy as np
import pytest

import fitness_ref as R

HERE = os.path.dirname(os.path.abspath(__file__))
PROBE = os.path.join(HERE, "libfoldprobe.so")

GUARD_MIN, GUARD_MAX = 2.0 ** -600, 2.0 ** 600   # the amounts that keep the reciprocal shortcut (fitness.cuh)
N = 4096                                          # pairs per family on the GPU


def _rd(rng, n, emin, emax):
    """Normal doubles, exponent uniform in [emin, emax], significand uniform."""
    e = rng.integers(emin, emax + 1, n).astype(np.uint64)
    m = rng.integers(0, 1 << 52, n, dtype=np.uint64)
    return (((e + np.uint64(1023)) << np.uint64(52)) | m).view(np.float64)


def _sub(rng, n):
    """Subnormal doubles."""
    return rng.integers(1, 1 << 52, n, dtype=np.uint64).view(np.float64)


def _under(rng, lc):
    """A request or assigned amount at most lc (a uniform share, rounded)."""
    return lc * rng.uniform(0.0, 1.0, len(lc))


def _grid(rng, n, q, lmax):
    """Cook's amounts on a grid of quantum q: leases up to lmax quanta, running up to twice that, the assigned
    share and the request within the lease (one quantum past it now and then)."""
    l = q * rng.integers(1, lmax + 1, n)
    r = q * rng.integers(0, 2 * lmax + 1, n)
    a = q * np.floor(rng.uniform(0, 1, n) * (l / q))
    j = q * rng.integers(0, (l - a) / q + 2)
    return j, a, l, r


def _ulps(x, k):
    return (np.asarray(x, np.float64).view(np.int64) + k).view(np.float64)


def _side(fam, rng, n):
    """(j, a, l, r) of one resource in family `fam`."""
    z = np.zeros(n)
    if fam == "grid-half":
        return _grid(rng, n, 0.5, 512)
    if fam == "grid-512":
        return _grid(rng, n, 512.0, 2048)
    if fam == "grid-2^-10":
        return _grid(rng, n, 2.0 ** -10, 1 << 20)
    if fam in ("den-1e-100", "den-1e100"):       # lease one ulp either side of the bound, or on it
        l = _ulps(np.full(n, 1e-100 if fam == "den-1e-100" else 1e100), rng.integers(-1, 2, n))
        return _under(rng, l), z, l, z
    if fam == "all-ones":                        # significand all ones at every 16th exponent
        e = rng.choice(np.arange(-1022, 1024, 16), n)
        l = np.ldexp(np.full(n, 2.0 - 2.0 ** -52), e)
        return _under(rng, l), z, l, z
    if fam == "pow2":                            # powers of two, and den == 0 (nothing leased, nothing asked)
        l = np.ldexp(1.0, rng.integers(-1022, 1024, n))
        j = _under(rng, l)
        zero = rng.random(n) < 0.1
        return np.where(zero, 0.0, j), z, np.where(zero, 0.0, l), z
    if fam == "tiny-quotient":                   # quotients in the last 60 binades above underflow and below
        l = _rd(rng, n, -300, 300)
        q = np.ldexp(rng.uniform(1.0, 2.0, n), rng.integers(-1074, -962, n))
        return q * l, z, l, z
    if fam == "subnormal-dividend":
        j = _sub(rng, n)
        return j, np.where(rng.random(n) < 0.3, _sub(rng, n), 0.0), np.maximum(_rd(rng, n, -30, 30), 2 * j), z
    if fam == "near-min-normal":                 # dividends within 2^60 of the smallest normal
        j = _rd(rng, n, -1022, -962)
        return j, z, _rd(rng, n, -30, 30), z
    if fam == "fit-edge":                        # ac + jc == lc exactly, or one ulp below it (no fit)
        j, a, r = _rd(rng, n, -20, 30), _rd(rng, n, -20, 30), _rd(rng, n, -20, 30)
        return j, a, _ulps(a + j, -rng.integers(0, 2, n)), r
    if fam == "near-one":                        # fitness within a few ulps of 1
        l, r = _rd(rng, n, -10, 30), _rd(rng, n, -10, 30)
        a = _under(rng, l)
        return _ulps(l - a, -rng.integers(0, 4, n)), a, l, r
    if fam == "guard":                           # one amount on either side of the guard's bounds
        j, a, l, r = _rd(rng, n, -10, 10), z.copy(), _rd(rng, n, 11, 20), _rd(rng, n, -10, 10)
        edge = rng.choice(np.array([GUARD_MIN, _ulps(GUARD_MIN, -1), GUARD_MAX, _ulps(GUARD_MAX, 1)]), n)
        slot = rng.integers(0, 4, n)
        j = np.where(slot == 0, np.minimum(edge, l), j)
        a = np.where(slot == 1, np.minimum(edge, l - j), a)
        l = np.where(slot == 2, np.maximum(edge, j), l)
        r = np.where(slot == 3, edge, r)
        return j, a, l, r
    raise KeyError(fam)


FAMILIES = ("grid-half", "grid-512", "grid-2^-10", "den-1e-100", "den-1e100", "all-ones", "pow2", "tiny-quotient",
            "subnormal-dividend", "near-min-normal", "fit-edge", "near-one", "guard")
TINY_FAMILIES = ("tiny-quotient", "subnormal-dividend", "near-min-normal")


def family(fam, n, seed=0):
    """Columns jc, jm, ac, am, lc, lm, rc, rm of n pairs: every amount non-negative and finite."""
    rng = np.random.default_rng([seed, FAMILIES.index(fam)])
    jc, ac, lc, rc = _side(fam, rng, n)
    jm, am, lm, rm = _side(fam, rng, n)
    gj, ga, gl, gr = _side("grid-half", rng, n)
    keep = rng.random(n) < 0.5
    jm, am, lm, rm = (np.where(keep, x, g) for x, g in ((jm, gj), (am, ga), (lm, gl), (rm, gr)))
    cols = [np.asarray(x, np.float64) for x in (jc, jm, ac, am, lc, lm, rc, rm)]
    for x in cols:
        assert np.isfinite(x).all() and (x >= 0).all() and not np.signbit(x).any(), fam
    return cols


def pairs(cols):
    """The two divisions of each pair: dividends (req + assigned) + running, denominators lease + running."""
    jc, jm, ac, am, lc, lm, rc, rm = cols
    return np.concatenate([(jc + ac) + rc, (jm + am) + rm]), np.concatenate([lc + rc, lm + rm])


def in_div_range(x):
    """div_y's stated range for the dividend: +0.0, or within [2^-600, 2^602) (a sum of three guarded amounts)."""
    return ((x >= GUARD_MIN) & (x < 4 * GUARD_MAX)) | (x.view(np.int64) == 0)


def _bits_equal(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return (a.view(np.int64) == b.view(np.int64)) | (np.isnan(a) & np.isnan(b))


# ---- CPU: the exact reference ----------------------------------------------------------------------------------
def test_exact_division_hand_cases():
    T = R.TINY
    h = float.fromhex
    assert R.div(1.0, 3.0) == h("0x1.5555555555555p-2")
    assert R.div(2.0, 3.0) == h("0x1.5555555555555p-1")
    # exact midpoints between subnormals round to even: 3 T / 2 -> 2 T, 5 T / 2 -> 2 T, 7 T / 2 -> 4 T
    assert R.div(3 * T, 2.0) == 2 * T and R.div(5 * T, 2.0) == 2 * T and R.div(7 * T, 2.0) == 4 * T
    assert R.div(T, 2.0) == 0.0 and not math.copysign(1.0, R.div(T, 2.0)) < 0     # half the least: ties to 0
    assert R.div(T, h("0x1.fffffffffffffp0")) == T                                # just over half rounds up
    assert R.div(h("0x1p-1022"), 2.0) == h("0x0.8p-1022")                         # into the subnormals, exact
    assert R.div(4 * T, h("0x1.bf17257e3aa5p+0")) == 2 * T
    # the overflow edge: the largest finite and its rounding to 2^1024
    big = h("0x1.fffffffffffffp1023")
    assert R.div(big, 1.0) == big and R.div(big, 0.5) == math.inf
    assert R.div(big, h("0x1.fffffffffffffp-1")) == math.inf
    assert R.div(h("0x1p1023"), h("0x1.0000000000001p-1")) == h("0x1.ffffffffffffep1023")
    # zeros, signs, 0/0 and division by zero
    assert math.isnan(R.div(0.0, 0.0)) and math.isnan(R.div(-0.0, 0.0))
    assert R.div(1.0, 0.0) == math.inf and R.div(-1.0, 0.0) == -math.inf and R.div(1.0, -0.0) == -math.inf
    for x, y, neg in ((0.0, 3.0, False), (-0.0, 3.0, True), (0.0, -3.0, True), (-0.0, -3.0, False),
                      (-T, 4.0, True)):
        z = R.div(x, y)
        assert z == 0.0 and (math.copysign(1.0, z) < 0) == neg, (x, y)
    assert R.div(1.0, math.inf) == 0.0 and math.isnan(R.div(math.inf, math.inf))


def test_exact_division_equals_ieee_division():
    """10^5 random pairs of every family against numpy's IEEE `/`: the reference is IEEE division."""
    for fam in FAMILIES:
        x, den = pairs(family(fam, 100_000 // 2, seed=1))
        with np.errstate(divide="ignore", invalid="ignore"):
            want = x / den
        got = np.array([R.div(a, b) for a, b in zip(x.tolist(), den.tolist())])
        assert _bits_equal(got, want).all(), fam


def test_reference_fitness_is_eval_pairs():
    """fitness(): 0.0 past the lease, else the mean of the two correctly rounded fits (numpy's IEEE operations in
    eval_pair's association)."""
    for fam in FAMILIES:
        cols = family(fam, 2000, seed=2)
        jc, jm, ac, am, lc, lm, rc, rm = cols
        with np.errstate(divide="ignore", invalid="ignore"):
            want = np.where((ac + jc > lc) | (am + jm > lm), 0.0, (((jc + ac) + rc) / (lc + rc) + ((jm + am) + rm) / (lm + rm)) / 2.0)
        got = np.array([R.fitness(*p) for p in zip(*(c.tolist() for c in cols))])
        assert _bits_equal(got, want).all(), fam


def test_families_reach_their_edges():
    """The families hold what they are named for: fits and misfits at the fit edge, fitnesses next to 1, the three
    reasons safe_rcp rejects a denominator, tiny dividends below the guard and amounts on both sides of it."""
    fit = lambda c: ~((c[2] + c[0] > c[4]) | (c[3] + c[1] > c[5]))
    c = family("fit-edge", N)
    f = fit(c)
    assert f.any() and (~f).any() and ((c[2] + c[0] == c[4]) & f).any()
    c = family("near-one", N)
    fits = np.array([R.fitness(*p) for p in zip(*(x[:500].tolist() for x in c))])
    assert (np.abs(fits - 1.0) <= 4 * 2.0 ** -52).sum() > 100
    rcp = lambda fam: np.array([R.safe_rcp(d) for d in pairs(family(fam, N))[1][:N].tolist()])
    assert (rcp("den-1e-100") == 0).any() and (rcp("den-1e-100") != 0).any()
    assert (rcp("den-1e100") == 0).any() and (rcp("den-1e100") != 0).any()
    assert (rcp("all-ones") == 0).all()
    assert (pairs(family("pow2", N))[1] == 0).any()
    for fam in TINY_FAMILIES:
        x = pairs(family(fam, N))[0][:N]
        assert ((x > 0) & (x < GUARD_MIN)).mean() > 0.5, fam
    c = np.concatenate(family("guard", N))
    for v in (GUARD_MIN, _ulps(GUARD_MIN, -1), GUARD_MAX, _ulps(GUARD_MAX, 1)):
        assert (c == v).any()


# ---- GPU: the device code against the reference ------------------------------------------------------------------
@pytest.fixture(scope="module")
def probe():
    if not os.path.exists(PROBE):
        raise FileNotFoundError(f"{PROBE} not built: run __graft_entry__.build() (nvcc, sm_90a)")
    lib = C.CDLL(PROBE)
    for name in ("fp_div", "fp_fitness"):
        getattr(lib, name).restype = C.c_int
    return lib


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


def device_div(probe, x, den):
    x, den = np.ascontiguousarray(x, np.float64), np.ascontiguousarray(den, np.float64)
    out = np.empty_like(x)
    assert probe.fp_div(_ptr(x), _ptr(den), C.c_int(len(x)), _ptr(out)) == 0
    return out


def device_fitness(probe, cols):
    cols = [np.ascontiguousarray(c, np.float64) for c in cols]
    out = np.empty_like(cols[0])
    assert probe.fp_fitness(*(_ptr(c) for c in cols), C.c_int(len(out)), _ptr(out)) == 0
    return out


def _mismatches(got, want, *inputs):
    bad = np.flatnonzero(~_bits_equal(got, want))
    return [tuple(float(x[i]).hex() for x in inputs) + (float(got[i]).hex(), float(want[i]).hex())
            for i in bad[:5]], len(bad)


@pytest.mark.gpu
@pytest.mark.parametrize("fam", FAMILIES)
def test_div_y_is_exact_in_its_range(probe, fam):
    """div_y(x, den, safe_rcp(den)) == RN(x / den) for every dividend in its stated range, any denominator."""
    x, den = pairs(family(fam, N))
    keep = in_div_range(x)
    x, den = x[keep], den[keep]
    got = device_div(probe, x, den)
    want = np.array([R.div(a, b) for a, b in zip(x.tolist(), den.tolist())])
    ex, n = _mismatches(got, want, x, den)
    assert n == 0, (n, ex)


@pytest.mark.gpu
@pytest.mark.parametrize("fam", TINY_FAMILIES[:2])
def test_div_y_needs_its_range(probe, fam):
    """Below the range the shortcut is not exact: why the guard exists."""
    x, den = pairs(family(fam, N))
    keep = ~in_div_range(x) & (den > 0)
    got = device_div(probe, x[keep], den[keep])
    want = np.array([R.div(a, b) for a, b in zip(x[keep].tolist(), den[keep].tolist())])
    assert (~_bits_equal(got, want)).sum() > 0


@pytest.mark.gpu
@pytest.mark.parametrize("fam", FAMILIES)
def test_fit_fitness_is_exact(probe, fam):
    """fit_fitness as the matcher evaluates one (job, VM) pair == the exact reference, bit for bit."""
    cols = family(fam, N)
    got = device_fitness(probe, cols)
    want = np.array([R.fitness(*p) for p in zip(*(c.tolist() for c in cols))])
    ex, n = _mismatches(got, want, *cols)
    assert n == 0, (n, ex)


@pytest.mark.gpu
def test_guard_bounds(probe):
    """fit_guard keeps +0.0 and [2^-600, 2^600] on the shortcut and flags everything else, per resource."""
    h = float.fromhex
    vals = np.array([0.0, -0.0, GUARD_MIN, _ulps(GUARD_MIN, -1), GUARD_MAX, _ulps(GUARD_MAX, 1), R.TINY,
                     h("0x1p-1022"), 1.0, 2.0 ** -10, 393216.0, math.inf, math.nan, -1.0, -GUARD_MIN])
    ok = [True, False, True, False, True, False, False, False, True, True, True, False, False, False, False]
    one = np.ones(len(vals))
    probe.fp_fit_guard.restype = C.c_int
    for c, m, bit in ((vals, one, 1), (one, vals, 2)):
        out = np.empty(len(vals), np.int32)
        assert probe.fp_fit_guard(_ptr(c), _ptr(m), C.c_int(len(vals)), _ptr(out)) == 0
        assert ((out & bit) == 0).tolist() == ok and (out & ~bit == 0).all()
