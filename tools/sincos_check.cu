// Host harness for sincos_fast (csrc/fastmath.cuh): max absolute error of sin against long double libm over the argument
// ranges of the random-Fourier-feature kernels, and its cosine bit for bit equal to cos_fast (the paired trajectory kernel's values
// must not depend on whether it also computes the gradient).
//   g++ -O2 -x c++ -o build/sincos_check tools/sincos_check.cu && build/sincos_check
#include <cmath>
#include <cstdio>
#include <cstring>
#include <random>
#include "../trieste_b200/csrc/fastmath.cuh"
#ifndef FM_ITERS
#define FM_ITERS 20000000
#endif
int main() {
  const tb::fm::TrigConsts TC;
  std::mt19937_64 rng(2);
  std::uniform_real_distribution<double> u(0.0, 1.0);
  double worst = 0, at = 0;
  long long cos_mismatch = 0;
  for (int i = 0; i < FM_ITERS; ++i) {
    const double a = (i % 2 ? 60.0 : 3000.0) * (2.0 * u(rng) - 1.0);
    double s;
    const double c = tb::fm::sincos_fast(a, TC, s);
    const double c0 = tb::fm::cos_fast(a, TC);
    if (std::memcmp(&c, &c0, sizeof(double)) != 0) ++cos_mismatch;
    const double err = (double)fabsl((long double)s - sinl((long double)a));
    if (err > worst) { worst = err; at = a; }
  }
  double s0, s_half, s_pi;
  tb::fm::sincos_fast(0.0, TC, s0);
  tb::fm::sincos_fast(1.5707963267948966, TC, s_half);
  tb::fm::sincos_fast(3.141592653589793, TC, s_pi);
  printf("sincos_fast: max ABS err %.3e at a = %.17g; sin(0) = %.17g, sin(pi/2) = %.17g, sin(pi) = %.17g\n", worst, at, s0, s_half,
         s_pi);
  printf("sincos_fast: cos differs from cos_fast at %lld of %d arguments\n", cos_mismatch, FM_ITERS);
  return (worst < 1e-13 && cos_mismatch == 0) ? 0 : 1;
}
