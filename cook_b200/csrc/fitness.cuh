// fitness.cuh — Fenzo's cpuMemBinPacker fitness as the matcher computes it, and the division shortcut under it.
//
// The fitness divides by the two denominators lc + rc and lm + rm of a VM.  They are static in a cycle, so
// init_dyn_kernel sets their correctly rounded reciprocals once per VM (safe_rcp) and every evaluation divides
// through them (div_y).  Bit for bit the oracle's eval_pair, which divides with IEEE `/`, for any input: a
// denominator safe_rcp rejects, and every VM of a cycle whose amounts fit_guard flags, divide with IEEE division.
#pragma once

namespace {   // one copy per translation unit, like the kernels that use it

// What one fitness evaluation reads about a VM: cpus / mem assigned this cycle, lease, running, and the
// reciprocals of the two denominators (0 = divide with IEEE division).  fit_fitness takes any struct with
// these fields (the matcher's VmState).
struct FitState {
  double ac, am, lc, lm, rc, rm, yc, ym;
};

// x / den with y = RN(1 / den) (or 0 => plain division): three dependent f64 ops
// instead of the ~10 of div.rn.f64, same correctly rounded result.  Precondition (y = safe_rcp(den) != 0): x is
// +0.0 or within [2^-600, 2^602).  Markstein's correction is exact while q0 and the residual fma(-den, q0, x) are
// normal; with den in (1e-100, 1e100) such an x keeps q0 and q within (2^-933, 2^935) and the residual at least
// 2^-104 |x|.  A smaller x, a subnormal one above all, can be off by an ulp; fit_guard keeps those away.
__device__ __forceinline__ double div_y(double x, double den, double y) {
  if (y == 0.0) return x / den;
  const double q0 = x * y;
  return fma(fma(-den, q0, x), y, q0);
}
// (y = 0 selects the IEEE division in div_y.)  The Markstein correction is proven for a faithful q0 and a
// denominator whose significand is not all ones; such denominators take the plain division as well.  This guards
// the denominator only: the dividend's range is fit_guard's.
__device__ __forceinline__ double safe_rcp(double den) {
  const unsigned long long frac = (unsigned long long)__double_as_longlong(den) & 0x000fffffffffffffULL;
  return (den > 1e-100 && den < 1e100 && frac != 0x000fffffffffffffULL) ? 1.0 / den : 0.0;
}

// The dividend guard.  A cycle keeps the shortcut for a resource only while every amount it divides with -- each
// considerable job's request, each VM's lease and running usage -- is +0.0 or within [2^-600, 2^600].  The
// dividend (jc + ac) + rc is then 0 or in [2^-600, 2^602): non-negative sums are at least their largest term, and
// ac + jc <= lc for every placement made.  fit_guard gives the resources whose amount breaks that (NaN, infinite,
// negative, -0.0 and the tiny ones included); init_dyn_kernel then sets that reciprocal to 0 on every VM.
constexpr double FIT_AMOUNT_MIN = 0x1p-600, FIT_AMOUNT_MAX = 0x1p600;
enum { FIT_IEEE_CPU = 1, FIT_IEEE_MEM = 2 };
__device__ __forceinline__ bool fit_amount_ok(double x) {
  return (x >= FIT_AMOUNT_MIN && x <= FIT_AMOUNT_MAX) || __double_as_longlong(x) == 0;
}
__device__ __forceinline__ int fit_guard(double cpus, double mem) {
  return (fit_amount_ok(cpus) ? 0 : FIT_IEEE_CPU) | (fit_amount_ok(mem) ? 0 : FIT_IEEE_MEM);
}

// FENZO 3a + 4 (see oracle): resource fit then cpuMemBinPacker fitness.
// The usual case (both reciprocals usable) takes no branch between the two divisions, so their
// dependent chains interleave: on the commit chain that is one 7-op f64 path instead of two 5-op ones
// each fenced by a branch to the IEEE division.  Same operations, same results.
template <class State>
__device__ __forceinline__ double fit_fitness(double jc, double jm, const State& st) {
  const bool no = (st.ac + jc > st.lc) | (st.am + jm > st.lm);
  double cpu_fit, mem_fit;
  if (st.yc != 0.0 && st.ym != 0.0) {
    const double xc = (jc + st.ac) + st.rc, xm = (jm + st.am) + st.rm;
    const double qc = xc * st.yc, qm = xm * st.ym;
    cpu_fit = fma(fma(-(st.lc + st.rc), qc, xc), st.yc, qc);
    mem_fit = fma(fma(-(st.lm + st.rm), qm, xm), st.ym, qm);
  } else {
    cpu_fit = div_y((jc + st.ac) + st.rc, st.lc + st.rc, st.yc);
    mem_fit = div_y((jm + st.am) + st.rm, st.lm + st.rm, st.ym);
  }
  return no ? 0.0 : (cpu_fit + mem_fit) * 0.5;
}

}  // namespace
