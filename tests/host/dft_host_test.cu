// Host-side check of the butterfly templates (fft_radix.cuh): on the host the add / multiply / fma primitives are
// plain scalar code with the rounding of the device's __fadd_rn / __fmul_rn / __fmaf_rn, so the algebra (index maps, signs, quarter turns,
// Good-Thomas / Cooley-Tukey splits) is verified without a GPU.  Built and run by tests/test_capi_cpu.py.
#include <cmath>
#include <complex>
#include <cstdio>
#include <cuda_runtime.h>
#include "../../ka9q_radio_b200/csrc/fft_radix.cuh"
using namespace kfft;
static unsigned long long rng_state = 88172645463325252ULL;
static float frand() {
  rng_state ^= rng_state << 13; rng_state ^= rng_state >> 7; rng_state ^= rng_state << 17;
  return (float)((double)(rng_state >> 11) / 9007199254740992.0 * 2.0 - 1.0);
}
template <int R, bool INV> static double check() {
  float2 x[R];
  std::complex<double> in[R];
  for (int i = 0; i < R; i++) { x[i] = make_float2(frand(), frand()); in[i] = {x[i].x, x[i].y}; }
  Dft<R, INV>::run(x);
  double worst = 0, mag = 0;
  for (int k = 0; k < R; k++) {
    std::complex<double> s = 0;
    for (int n = 0; n < R; n++) s += in[n] * std::polar(1.0, (INV ? 2.0 : -2.0) * M_PI * (double)((long)n * k % R) / R);
    worst = std::fmax(worst, std::abs(s - std::complex<double>(x[k].x, x[k].y)));
    mag = std::fmax(mag, std::abs(s));
  }
  return worst / mag;
}
template <int R> static int both() {
  double const f = check<R, false>(), i = check<R, true>();
  bool const ok = f < 2e-6 && i < 2e-6;
  printf("radix %2d  forward %.2e  inverse %.2e  %s\n", R, f, i, ok ? "ok" : "FAIL");
  return ok ? 0 : 1;
}
// The two-fat-stage decomposition of fwd_cols_r36 / fwd_2s restated on the host: stage 0 takes x[j + RD m],
// m < RC, output t times W_N^{j t} goes to slot t RD + j; stage 1 transforms slots t RD .. t RD + RD - 1 and its output k' is
// X[t + RC k'].  The twiddle W^{j t} is formed as the kernels form it: t = Q a + b, one product of two float-rounded powers.
template <int RC, int RD> static int two_stage() {
  constexpr int N = RC * RD;
  static float2 x[N], y[N];
  static std::complex<double> in[N];
  for (int i = 0; i < N; i++) { x[i] = make_float2(frand(), frand()); in[i] = {x[i].x, x[i].y}; }
  int Q = 1;
  while (Q * Q < RC) Q++;
  auto root = [](long e, long n) {
    double const a = -2.0 * M_PI * (double)(e % n) / (double)n;
    return make_float2((float)std::cos(a), (float)std::sin(a));
  };
  for (int j = 0; j < RD; j++) {
    float2 a[RC];
    for (int m = 0; m < RC; m++) a[m] = x[j + RD * m];
    Dft<RC, false>::run(a);
    for (int t = 0; t < RC; t++) {
      int const qa = t / Q, qb = t % Q;
      float2 w = make_float2(1.f, 0.f);
      if (qa && qb) w = cmul(root((long)j * Q * qa, N), root((long)j * qb, N));
      else if (qa) w = root((long)j * Q * qa, N);
      else if (qb) w = root((long)j * qb, N);
      y[t * RD + j] = t ? cmul(a[t], w) : a[0];
    }
  }
  double worst = 0, mag = 0;
  for (int t = 0; t < RC; t++) {
    float2 b[RD];
    for (int m = 0; m < RD; m++) b[m] = y[t * RD + m];
    Dft<RD, false>::run(b);
    for (int kp = 0; kp < RD; kp++) {
      int const k = t + RC * kp;
      std::complex<double> s = 0;
      for (int n = 0; n < N; n++) s += in[n] * std::polar(1.0, -2.0 * M_PI * (double)((long)n * k % N) / N);
      worst = std::fmax(worst, std::abs(s - std::complex<double>(b[kp].x, b[kp].y)));
      mag = std::fmax(mag, std::abs(s));
    }
  }
  bool const ok = worst / mag < 3e-6;
  printf("two-stage %2d x %2d  %.2e  %s\n", RC, RD, worst / mag, ok ? "ok" : "FAIL");
  return ok ? 0 : 1;
}

int main() {
  int bad = 0;
  bad += both<40>() + both<45>() + both<48>() + both<50>();
  bad += two_stage<36, 36>() + two_stage<50, 25>() + two_stage<25, 32>() + two_stage<25, 25>();
  bad += both<2>() + both<3>() + both<4>() + both<5>() + both<6>() + both<7>() + both<8>() + both<9>() + both<10>();
  bad += both<12>() + both<14>() + both<15>() + both<16>() + both<18>() + both<20>() + both<21>() + both<24>() + both<25>();
  bad += both<27>() + both<28>() + both<30>() + both<32>() + both<35>() + both<36>();
  // complex products
  for (int t = 0; t < 1000; t++) {
    float2 a = make_float2(frand(), frand()), b = make_float2(frand(), frand());
    std::complex<double> A(a.x, a.y), B(b.x, b.y);
    float2 p = cmul(a, b), q = cmulc(a, b);
    if (std::abs(A * B - std::complex<double>(p.x, p.y)) > 3e-7 || std::abs(A * std::conj(B) - std::complex<double>(q.x, q.y)) > 3e-7) bad++;
    float2 r0 = rot90<false>(a), r1 = rot90<true>(a);
    if (r0.x != a.y || r0.y != -a.x || r1.x != -a.y || r1.y != a.x) bad++;
  }
  printf(bad ? "FAILED (%d)\n" : "all butterflies ok\n", bad);
  return bad ? 1 : 0;
}
