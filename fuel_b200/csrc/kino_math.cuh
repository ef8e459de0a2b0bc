// kino_math.cuh -- the arithmetic of KinodynamicAstar (path_searching/src/kinodynamic_astar.cpp) that is not plain IEEE
// +, -, *, /, sqrt: cbrt, the powers and the three-real-root branch of cubic().  Host and device; compiled without
// contraction (-fmad=false on the device, -ffp-contract=off on the host) so every operation rounds as written.
//   km_cbrt      glibc's x86-64 cbrt (sysdeps/ieee754/dbl-64/s_cbrt.c) restated operation for operation: equal to the
//                host libm bit for bit.  It is not correctly rounded, so the device's own cbrt would not match.
//   km_cube      t^3 correctly rounded (an fma error-free product); t^2 is t * t.  They replace pow(t, 2) and pow(t, 3)
//                outside the search, where glibc's pow is not always correctly rounded (DESIGN.md 4.14).  Inside the
//                search the powers come from host tables computed with the host's pow.
//   km_acos_cr   acos correctly rounded, km_cos_cr cos correctly rounded on |z| <= pi/2: double-double arithmetic, then
//                one rounding.  Only cubic()'s D < 0 branch uses them.
#pragma once

#include <math.h>

#ifdef __CUDACC__
#define KM_HD __host__ __device__ __forceinline__
#else
#define KM_HD static inline
#endif

KM_HD double km_cbrt(double x) {
  int xe;
  const double xm = frexp(fabs(x), &xe);
  if (xe == 0 && (x == 0.0 || !isfinite(x))) return x + x;
  const double u = (0.354895765043919860 +
                    ((1.50819193781584896 +
                      ((-2.11499494167371287 +
                        ((2.44693122563534430 + ((-1.83469277483613086 + (0.784932344976639262 - 0.145263899385486377 * xm) * xm) * xm)) *
                         xm)) *
                       xm)) *
                     xm));
  const double t2 = u * u * u;
  double f;
  switch (2 + xe % 3) {  // 1 / 2^(2/3), 1 / 2^(1/3), 1, 2^(1/3), 2^(2/3)
    case 0: f = 1.0 / 1.5874010519681994748; break;
    case 1: f = 1.0 / 1.2599210498948731648; break;
    case 2: f = 1.0; break;
    case 3: f = 1.2599210498948731648; break;
    default: f = 1.5874010519681994748; break;
  }
  const double ym = u * (t2 + 2.0 * xm) / (2.0 * t2 + xm) * f;
  return ldexp(x > 0.0 ? ym : -ym, xe / 3);
}

KM_HD double km_cube(double t) {
  const double p = t * t, e = fma(t, t, -p);  // t^2 = p + e exactly
  const double h = p * t;
  if (!isfinite(h) || h == 0.0) return h;
  const double l = fma(p, t, -h);  // p * t = h + l exactly
  return h + (l + e * t);
}

// ---- double-double: value hi + lo, |lo| <= ulp(hi) / 2 ----
struct km_dd {
  double hi, lo;
};
KM_HD km_dd km_two_sum(double a, double b) {
  const double s = a + b, bb = s - a;
  return km_dd{ s, (a - (s - bb)) + (b - bb) };
}
KM_HD km_dd km_fast_sum(double a, double b) {
  const double s = a + b;
  return km_dd{ s, b - (s - a) };
}
KM_HD km_dd km_add(km_dd a, km_dd b) {
  km_dd s = km_two_sum(a.hi, b.hi);
  const km_dd t = km_two_sum(a.lo, b.lo);
  s.lo += t.hi;
  s = km_fast_sum(s.hi, s.lo);
  s.lo += t.lo;
  return km_fast_sum(s.hi, s.lo);
}
KM_HD km_dd km_neg(km_dd a) { return km_dd{ -a.hi, -a.lo }; }
KM_HD km_dd km_mul(km_dd a, km_dd b) {
  const double p = a.hi * b.hi;
  const double e = fma(a.hi, b.hi, -p) + (a.hi * b.lo + a.lo * b.hi);
  return km_fast_sum(p, e);
}
KM_HD km_dd km_div(km_dd a, km_dd b) {
  const double q1 = a.hi / b.hi;
  km_dd r = km_add(a, km_neg(km_mul(b, km_dd{ q1, 0.0 })));
  const double q2 = r.hi / b.hi;
  r = km_add(r, km_neg(km_mul(b, km_dd{ q2, 0.0 })));
  const double q3 = r.hi / b.hi;
  return km_add(km_fast_sum(q1, q2), km_dd{ q3, 0.0 });
}

// sin(x) and cos(x) in double-double by their Taylor series, |x| <= pi/2: every term is below the first in magnitude,
// and 26 terms leave a remainder below 2^-120 of the sum
KM_HD km_dd km_dd_sin(km_dd x) {
  const km_dd x2 = km_mul(x, x);
  km_dd term = x, sum = x;
  for (int k = 1; k < 26; ++k) {
    term = km_div(km_mul(term, km_neg(x2)), km_dd{ (double)((2 * k) * (2 * k + 1)), 0.0 });
    sum = km_add(sum, term);
  }
  return sum;
}
KM_HD km_dd km_dd_cos(km_dd x) {
  const km_dd x2 = km_mul(x, x);
  km_dd term = km_dd{ 1.0, 0.0 }, sum = term;
  for (int k = 1; k < 26; ++k) {
    term = km_div(km_mul(term, km_neg(x2)), km_dd{ (double)((2 * k - 1) * (2 * k)), 0.0 });
    sum = km_add(sum, term);
  }
  return sum;
}

// cos(z) correctly rounded for |z| <= pi/2 (there cos(z) >= 0 and the series' absolute error is far below its ulp
// wherever cos(z) >= 2^-50; below that the argument is within 2^-50 of pi/2, which cubic() never passes)
KM_HD double km_cos_cr(double z) {
  if (!(fabs(z) <= 1.5707963267948966)) return cos(z);
  const km_dd c = km_dd_cos(km_dd{ z, 0.0 });
  return c.hi + c.lo;
}

// acos(x) correctly rounded: Newton's method on y from the double acos, in double-double, on f(y) = cos(y) - x written
// without cancellation: (1 - x) - 2 sin^2(y/2) for x >= 0, 2 cos^2(y/2) - (1 + x) for x < 0, with
// cos(y/2) = sin(pi/2 - y/2) and f'(y) = -sin(y) = -2 sin(y/2) cos(y/2)
KM_HD double km_acos_cr(double x) {
  if (!(fabs(x) <= 1.0)) return acos(x);
  if (x == 1.0) return 0.0;
  if (x == -1.0) return 3.141592653589793;
  const km_dd half_pi = km_dd{ 1.5707963267948966, 6.123233995736766e-17 };
  km_dd y = km_dd{ acos(x), 0.0 };
  for (int it = 0; it < 3; ++it) {
    const km_dd h = km_dd{ 0.5 * y.hi, 0.5 * y.lo };
    const km_dd s = km_dd_sin(h);
    const km_dd c = km_dd_sin(km_add(half_pi, km_neg(h)));
    km_dd f;
    if (x >= 0.0) {
      const km_dd s2 = km_mul(s, s);
      f = km_add(km_two_sum(1.0, -x), km_neg(km_dd{ 2.0 * s2.hi, 2.0 * s2.lo }));
    } else {
      const km_dd c2 = km_mul(c, c);
      f = km_add(km_dd{ 2.0 * c2.hi, 2.0 * c2.lo }, km_neg(km_two_sum(1.0, x)));
    }
    const km_dd sc = km_mul(s, c);
    y = km_add(y, km_div(f, km_dd{ 2.0 * sc.hi, 2.0 * sc.lo }));
  }
  return y.hi + y.lo;
}
