// fft_radix.cuh -- in-register DFT butterflies for the Stockham/DIF stages (sm_90a).
//
// Everything here works on a thread-private float2 x[R] that the compiler keeps in registers
// (all indices are literals after unrolling).  Primitive radices 2,3,4,5,7 are written out, and
// the primes 11, 13, 17, 19, 23 of the extended master kernels share one pair-form template;
// a radix with two coprime factors (6, 10, 12, 15, 20, 24, 36 ...) is a Good-Thomas prime-factor
// split R = R1*R2 -- index maps only, no twiddles between the two levels -- and a prime power
// (8, 9, 16, 25 ...) a two-level Cooley-Tukey split with compile-time twiddles from wconst.cuh.  INV selects exp(+i..) (the reference's FFTW_BACKWARD, filter.c:359).
#pragma once
#include <cuda_runtime.h>
#include "wconst.cuh"
#ifndef KFFT_HD
#define KFFT_HD __host__ __device__ __forceinline__
#endif

namespace kfft {

// ---- complex arithmetic on float2 pairs -------------------------------------------------------
// Every butterfly is built from three per-half primitives: add, multiply and fused multiply-add,
// one rounding each.  Hopper has no two-wide fp32 instructions, so each is two scalar instructions;
// on the device they are the _rn intrinsics, which the compiler never contracts or reassociates, so
// the rounding of every result is fixed by the source (the host build used by the tests matches it).
KFFT_HD float2 p_add(float2 a, float2 b) {
#if defined(__CUDA_ARCH__)
  return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y));
#else
  return make_float2(a.x + b.x, a.y + b.y);
#endif
}
KFFT_HD float2 p_mul(float2 a, float2 b) {
#if defined(__CUDA_ARCH__)
  return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y));
#else
  return make_float2(a.x * b.x, a.y * b.y);
#endif
}
KFFT_HD float2 p_fma(float2 a, float2 b, float2 c) {  // a*b + c per half, one rounding each
#if defined(__CUDA_ARCH__)
  return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y));
#else
  return make_float2(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y));
#endif
}
KFFT_HD float2 bb(float s) { return make_float2(s, s); }  // scalar broadcast operand

KFFT_HD float2 cadd(float2 a, float2 b) { return p_add(a, b); }
KFFT_HD float2 csub(float2 a, float2 b) { return p_add(a, make_float2(-b.x, -b.y)); }
KFFT_HD float2 cmul(float2 a, float2 b) {  // (ax bx - ay by, ay bx + ax by)
  return p_fma(a, bb(b.x), p_mul(make_float2(-a.y, a.x), bb(b.y)));
}
KFFT_HD float2 cmulc(float2 a, float2 b) {  // a * conj(b) = (ax bx + ay by, ay bx - ax by)
  return p_fma(a, bb(b.x), p_mul(make_float2(a.y, -a.x), bb(b.y)));
}
KFFT_HD float2 cconj(float2 a) { return make_float2(a.x, -a.y); }
// multiply by -i (forward quarter turn) or +i
template <bool INV> KFFT_HD float2 rot90(float2 a) {
  return INV ? make_float2(-a.y, a.x) : make_float2(a.y, -a.x);
}
// c + s * (-i or +i) * a  and  c - s * (-/+ i) * a : the quarter turn rides on the operand modifiers
template <bool INV> KFFT_HD float2 fma_rot(float2 a, float s, float2 c) { return p_fma(rot90<INV>(a), bb(s), c); }
template <bool INV> KFFT_HD float2 fms_rot(float2 a, float s, float2 c) { return p_fma(rot90<!INV>(a), bb(s), c); }

template <int R, bool INV> struct Dft;

template <bool INV> struct Dft<1, INV> {
  static KFFT_HD void run(float2 (&)[1]) {}
};
template <bool INV> struct Dft<2, INV> {
  static KFFT_HD void run(float2 (&x)[2]) {
    float2 const a = x[0], b = x[1];
    x[0] = cadd(a, b);
    x[1] = csub(a, b);
  }
};
template <bool INV> struct Dft<3, INV> {
  static KFFT_HD void run(float2 (&x)[3]) {
    constexpr float S = 0.86602540378443864676f;
    float2 const a = x[0], t1 = cadd(x[1], x[2]), d = csub(x[1], x[2]);
    float2 const t2 = p_fma(t1, bb(-0.5f), a);
    // forward: X1 = t2 - i*S*d, X2 = t2 + i*S*d
    x[0] = cadd(a, t1);
    x[1] = fma_rot<INV>(d, S, t2);
    x[2] = fms_rot<INV>(d, S, t2);
  }
};
template <bool INV> struct Dft<4, INV> {
  static KFFT_HD void run(float2 (&x)[4]) {
    float2 const apc = cadd(x[0], x[2]), amc = csub(x[0], x[2]);
    float2 const bpd = cadd(x[1], x[3]), bmd = csub(x[1], x[3]);
    x[0] = cadd(apc, bpd);
    x[1] = fma_rot<INV>(bmd, 1.0f, amc);
    x[2] = csub(apc, bpd);
    x[3] = fms_rot<INV>(bmd, 1.0f, amc);
  }
};
template <bool INV> struct Dft<5, INV> {
  static KFFT_HD void run(float2 (&x)[5]) {
    constexpr float C1 = 0.30901699437494742410f, C2 = -0.80901699437494742410f;
    constexpr float S1 = 0.95105651629515357212f, S2 = 0.58778525229247312917f;
    float2 const a = x[0];
    float2 const t1 = cadd(x[1], x[4]), t2 = cadd(x[2], x[3]);
    float2 const t3 = csub(x[1], x[4]), t4 = csub(x[2], x[3]);
    float2 const u1 = p_fma(t2, bb(C2), p_fma(t1, bb(C1), a));
    float2 const u2 = p_fma(t2, bb(C1), p_fma(t1, bb(C2), a));
    float2 const w1 = p_fma(t4, bb(S2), p_mul(t3, bb(S1)));   // v1 = (-/+ i) w1
    float2 const w2 = p_fma(t4, bb(-S1), p_mul(t3, bb(S2)));  // v2 = (-/+ i) w2
    x[0] = cadd(a, cadd(t1, t2));
    x[1] = fma_rot<INV>(w1, 1.0f, u1);
    x[2] = fma_rot<INV>(w2, 1.0f, u2);
    x[3] = fms_rot<INV>(w2, 1.0f, u2);
    x[4] = fms_rot<INV>(w1, 1.0f, u1);
  }
};
template <bool INV> struct Dft<7, INV> {
  static KFFT_HD void run(float2 (&x)[7]) {
    constexpr float C1 = 0.62348980185873353053f, C2 = -0.22252093395631440429f, C3 = -0.90096886790241912624f;
    constexpr float S1 = 0.78183148246802980871f, S2 = 0.97492791218182360702f, S3 = 0.43388373911755812048f;
    float2 const a = x[0];
    float2 const p1 = cadd(x[1], x[6]), p2 = cadd(x[2], x[5]), p3 = cadd(x[3], x[4]);
    float2 const m1 = csub(x[1], x[6]), m2 = csub(x[2], x[5]), m3 = csub(x[3], x[4]);
    auto comb = [&](float c1, float c2, float c3) { return p_fma(p3, bb(c3), p_fma(p2, bb(c2), p_fma(p1, bb(c1), a))); };
    auto sinc = [&](float s1, float s2, float s3) { return p_fma(m3, bb(s3), p_fma(m2, bb(s2), p_mul(m1, bb(s1)))); };
    float2 const u1 = comb(C1, C2, C3), u2 = comb(C2, C3, C1), u3 = comb(C3, C1, C2);
    float2 const w1 = sinc(S1, S2, S3), w2 = sinc(S2, -S3, -S1), w3 = sinc(S3, -S1, S2);  // v = (-/+ i) w
    x[0] = cadd(a, cadd(p1, cadd(p2, p3)));
    x[1] = fma_rot<INV>(w1, 1.0f, u1);
    x[6] = fms_rot<INV>(w1, 1.0f, u1);
    x[2] = fma_rot<INV>(w2, 1.0f, u2);
    x[5] = fms_rot<INV>(w2, 1.0f, u2);
    x[3] = fma_rot<INV>(w3, 1.0f, u3);
    x[4] = fms_rot<INV>(w3, 1.0f, u3);
  }
};

// Odd prime P >= 11 (the extended master kernels only): Dft<7>'s symmetric pair form written as loops.
//   p_j = x_j + x_{P-j}, m_j = x_j - x_{P-j}  (j = 1 .. H, H = (P-1)/2)
//   u_k = x_0 + sum_j p_j cos(2 pi jk/P),  w_k = sum_j m_j sin(2 pi jk/P),  X_k = u_k -/+ i w_k,  X_{P-k} = u_k +/- i w_k
// The cosines and sines are wroot<P> entries (generated, correctly rounded); each sum is one fma chain in j order.
template <int P, bool INV> struct DftPair {
  static constexpr int H = (P - 1) / 2;
  static KFFT_HD void run(float2 (&x)[P]) {
    float2 const a = x[0];
    float2 p[H], m[H];
#pragma unroll
    for (int j = 0; j < H; j++) {
      p[j] = cadd(x[j + 1], x[P - 1 - j]);
      m[j] = csub(x[j + 1], x[P - 1 - j]);
    }
    float2 s = p[H - 1];
#pragma unroll
    for (int j = H - 2; j >= 0; j--) s = cadd(p[j], s);
    x[0] = cadd(a, s);
#pragma unroll
    for (int k = 1; k <= H; k++) {
      float2 u = a, w = p_mul(m[0], bb(-wroot<P>(k).y));
#pragma unroll
      for (int j = 0; j < H; j++) u = p_fma(p[j], bb(wroot<P>((j + 1) * k % P).x), u);
#pragma unroll
      for (int j = 1; j < H; j++) w = p_fma(m[j], bb(-wroot<P>((j + 1) * k % P).y), w);
      x[k] = fma_rot<INV>(w, 1.0f, u);
      x[P - k] = fms_rot<INV>(w, 1.0f, u);
    }
  }
};
template <bool INV> struct Dft<11, INV> : DftPair<11, INV> {};
template <bool INV> struct Dft<13, INV> : DftPair<13, INV> {};
template <bool INV> struct Dft<17, INV> : DftPair<17, INV> {};
template <bool INV> struct Dft<19, INV> : DftPair<19, INV> {};
template <bool INV> struct Dft<23, INV> : DftPair<23, INV> {};

// first factor of the two-level split for composite radices
constexpr int split_first(int r) {
  return (r % 4 == 0 && r > 4) ? 4
         : (r % 5 == 0 && r > 5) ? 5
         : (r % 3 == 0 && r > 3) ? 3
         : (r % 2 == 0 && r > 2) ? 2
         : (r % 7 == 0 && r > 7) ? 7
                                 : 1;
}

// multiply by the compile-time root exp(-/+ 2*pi*i*e/R); trivial cases cost nothing or a swap
template <int R, bool INV> KFFT_HD float2 mul_root(float2 a, int e) {
  e %= R;
  if (e == 0) return a;
  if (2 * e == R) return make_float2(-a.x, -a.y);
  if (4 * e == R) return rot90<INV>(a);
  if (4 * e == 3 * R) return rot90<!INV>(a);
  float2 const w = wroot<R>(e);
  return INV ? cmulc(a, w) : cmul(a, w);
}

// R1 of the prime-factor split: the full power of the smallest prime in r (== r for a prime power)
constexpr int prime_power_first(int r) {
  int const p = (r % 2 == 0) ? 2 : (r % 3 == 0) ? 3 : (r % 5 == 0) ? 5 : (r % 7 == 0) ? 7 : 1;
  if (p == 1) return 1;
  int q = 1;
  while (r % p == 0) {
    q *= p;
    r /= p;
  }
  return q;
}
constexpr int inv_mod(int a, int m) {  // a^-1 mod m, gcd(a, m) = 1, m > 1
  for (int i = 1; i < m; i++)
    if ((a * i) % m == 1) return i;
  return 0;
}

template <int R, bool INV> struct Dft {
  static constexpr int Q = prime_power_first(R);
  static constexpr bool PFA = (Q != R);  // two coprime factors
  static constexpr int R1 = PFA ? Q : split_first(R);
  static constexpr int R2 = R / R1;
  static_assert(R1 > 1, "radix has an unsupported prime factor");
  // x natural order in, natural order out
  static KFFT_HD void run(float2 (&x)[R]) {
    float2 y[R];
    if constexpr (PFA) {
      // Good-Thomas: n = (R2 n1 + R1 n2) mod R,  k = (R2 (R2^-1 mod R1) k1 + R1 (R1^-1 mod R2) k2) mod R
      //   => W_R^{nk} = W_R1^{n1 k1} W_R2^{n2 k2}: R2 DFTs of length R1, then R1 of length R2, nothing between
      constexpr int A = R2 * inv_mod(R2 % R1, R1), B = R1 * inv_mod(R1 % R2, R2);
#pragma unroll
      for (int n2 = 0; n2 < R2; n2++) {
        float2 a[R1];
#pragma unroll
        for (int n1 = 0; n1 < R1; n1++) a[n1] = x[(R2 * n1 + R1 * n2) % R];
        Dft<R1, INV>::run(a);
#pragma unroll
        for (int k1 = 0; k1 < R1; k1++) y[k1 * R2 + n2] = a[k1];
      }
#pragma unroll
      for (int k1 = 0; k1 < R1; k1++) {
        float2 b[R2];
#pragma unroll
        for (int n2 = 0; n2 < R2; n2++) b[n2] = y[k1 * R2 + n2];
        Dft<R2, INV>::run(b);
#pragma unroll
        for (int k2 = 0; k2 < R2; k2++) x[(A * k1 + B * k2) % R] = b[k2];
      }
    } else {
      // Cooley-Tukey: n = n1*R2 + n2 ; k = k1 + R1*k2
#pragma unroll
      for (int n2 = 0; n2 < R2; n2++) {
        float2 a[R1];
#pragma unroll
        for (int n1 = 0; n1 < R1; n1++) a[n1] = x[n1 * R2 + n2];
        Dft<R1, INV>::run(a);
#pragma unroll
        for (int k1 = 0; k1 < R1; k1++) y[k1 * R2 + n2] = mul_root<R, INV>(a[k1], n2 * k1);
      }
#pragma unroll
      for (int k1 = 0; k1 < R1; k1++) {
        float2 b[R2];
#pragma unroll
        for (int n2 = 0; n2 < R2; n2++) b[n2] = y[k1 * R2 + n2];
        Dft<R2, INV>::run(b);
#pragma unroll
        for (int k2 = 0; k2 < R2; k2++) x[k1 + R1 * k2] = b[k2];
      }
    }
  }
};

}  // namespace kfft
