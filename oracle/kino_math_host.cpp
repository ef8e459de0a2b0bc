// The host build of fuel_b200/csrc/kino_math.cuh (-ffp-contract=off, as the device build runs with -fmad=false), for
// tests/test_kino_math.py.  TEST INFRASTRUCTURE ONLY.
#include <math.h>
#include <stdint.h>

#include "kino_math.cuh"

extern "C" void orc_kino_math(int32_t f, int64_t n, const double* in, double* out) {
  for (int64_t i = 0; i < n; ++i) {
    const double x = in[i];
    switch (f) {
      case 0: out[i] = km_cbrt(x); break;
      case 1: out[i] = km_cube(x); break;
      case 2: out[i] = km_acos_cr(x); break;
      case 3: out[i] = km_cos_cr(x); break;
      default: out[i] = cbrt(x); break;
    }
  }
}
