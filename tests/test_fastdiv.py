"""CPU check of the arithmetic shortcut the CUDA kernels use: division by the
fitness denominators through their correctly rounded reciprocals plus one fused
correction step must equal IEEE division bit for bit (DESIGN.md, "exactness of f64"),
for every dividend a cycle that passes the dividend guard (cook_b200/csrc/fitness.cuh)
can form, and it does not for dividends below the guard."""
import ctypes as C


def test_reciprocal_division_equals_ieee_division(oracle):
    fn = oracle.lib.oracle_check_fastdiv
    fn.restype = C.c_int64
    fn.argtypes = [C.c_int64, C.c_uint64]
    assert fn(20_000_000, 12345) == 0


def _guard_check(oracle):
    fn = oracle.lib.oracle_check_fastdiv_guard
    fn.restype = C.c_int64
    fn.argtypes = [C.c_int64, C.c_uint64, C.c_int]
    return fn


def test_reciprocal_division_is_exact_at_the_guards_edges(oracle):
    """Dividends 0 and in [2^-600, 2^602) by every denominator safe_rcp accepts, quotients from 2^-933 to 2^934."""
    assert _guard_check(oracle)(20_000_000, 12345, 0) == 0


def test_reciprocal_division_is_not_exact_below_the_guard(oracle):
    """Subnormal dividends and normal ones up to 2^-960: the shortcut is off by an ulp on some, so a cycle with
    such an amount must divide with IEEE division."""
    assert _guard_check(oracle)(1_000_000, 777, 1) > 0
