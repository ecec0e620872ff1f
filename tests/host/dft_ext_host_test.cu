// Host-side check of the prime butterflies of the extended master kernels (Dft<11> .. Dft<23>, fft_radix.cuh), compiled
// for the host where the add / multiply / fma primitives round like the device's __fadd_rn / __fmul_rn / __fmaf_rn.
// Each radix, forward and inverse, on several random inputs against a float64 DFT, at the bound of dft_host_test.cu.
// Built and run by tests/test_extended_primes_cpu.py.
#include <cmath>
#include <complex>
#include <cstdio>
#include <cuda_runtime.h>
#include "../../ka9q_radio_b200/csrc/fft_radix.cuh"
using namespace kfft;
static unsigned long long rng_state = 0x9E3779B97F4A7C15ULL;
static float frand() {
  rng_state ^= rng_state << 13; rng_state ^= rng_state >> 7; rng_state ^= rng_state << 17;
  return (float)((double)(rng_state >> 11) / 9007199254740992.0 * 2.0 - 1.0);
}
template <int R, bool INV> static double check() {
  double worst_rel = 0;
  for (int trial = 0; trial < 64; trial++) {
    float2 x[R];
    std::complex<double> in[R];
    for (int i = 0; i < R; i++) {
      // trial 0: a unit impulse at n = 1, which reads every constant of the butterfly exactly once per output
      x[i] = trial == 0 ? make_float2(i == 1 ? 1.f : 0.f, 0.f) : make_float2(frand(), frand());
      in[i] = {x[i].x, x[i].y};
    }
    Dft<R, INV>::run(x);
    double worst = 0, mag = 0;
    for (int k = 0; k < R; k++) {
      std::complex<double> s = 0;
      for (int n = 0; n < R; n++) s += in[n] * std::polar(1.0, (INV ? 2.0 : -2.0) * M_PI * (double)((long)n * k % R) / R);
      worst = std::fmax(worst, std::abs(s - std::complex<double>(x[k].x, x[k].y)));
      mag = std::fmax(mag, std::abs(s));
    }
    worst_rel = std::fmax(worst_rel, worst / mag);
  }
  return worst_rel;
}
template <int R> static int both() {
  double const f = check<R, false>(), i = check<R, true>();
  bool const ok = f < 2e-6 && i < 2e-6;
  printf("radix %2d  forward %.2e  inverse %.2e  %s\n", R, f, i, ok ? "ok" : "FAIL");
  return ok ? 0 : 1;
}

int main() {
  int bad = both<11>() + both<13>() + both<17>() + both<19>() + both<23>();
  printf(bad ? "FAILED (%d)\n" : "all prime butterflies ok\n", bad);
  return bad ? 1 : 0;
}
