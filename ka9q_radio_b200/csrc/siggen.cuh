// siggen.cuh -- sig_gen.c's CW source (proc_sig_gen, sig_gen.c:286-346) generated on the device: a carrier from the
// reference's oscillator (set_osc / step_osc, osc.c:28-70) plus the noise of real_gauss (gauss.c:103-111), stored as the
// driver's loop stores it, (float)(samp * scale).
//
// Noise.  Draw d of the stream (REAL: d = sample index; COMPLEX: re = 2s, im = 2s + 1, as complex_gauss in misc.h draws
// them) is xoshiro256** jumped d steps from its seeded state.  The generator's state transition is linear over GF(2), so
// a jump of j steps is a 256 x 256 bit matrix T^j.  Each thread produces a run of kGenRun consecutive draws: its start is
// the launch's base state (computed on the host) times T^(kGenRun t), applied as one matrix T^(kGenRun 2^b) per set bit b
// of its thread index t.  A matrix is held as 64 tables of 16 entries, one per nibble of the state: the product is the
// XOR of 64 table entries.  The Gaussian is real_gauss's popcount construction with explicitly rounded doubles in the
// reference's operation order, so the floats are bitwise the driver's.
//
// Carrier.  The reference's phasor is a chain of complex products by the rounded step cispi(2 freq), renormalised every
// 16384 steps.  Sample n is modelled as exp(2 pi i phi_n), phi_n = n F + n (n + 1) / 2 R (mod 1), where F and R are the
// exact angles, in cycles, of the rounded step and sweep phasors (computed on the host), held as 128-bit fractions of a
// cycle; the phase is exact modular integer arithmetic.  The chain's own rounding walks away from this by about 1e-12
// rad after 1e8 samples, which flips the float rounding of a few samples in 1e5 by one ulp, and next to a zero of the
// signal, where a float ulp is smaller than that, by more ulps (tests/test_siggen_cpu.py).
//
// AM and DSB (sig_gen.c:297-314, :327-344).  The modulated instantiation multiplies the carrier by dc + m, m the envelope
// float libsamplerate produced for the sample (read from GenArgs::mod; dc = 1 for AM, 0 for DSB), with the products and
// sums the reference's compiled loop performs, in its order and contraction (found in its disassembly, pinned by
// tests/test_siggen_mod_cpu.py):
//   REAL     samp = fma(amplitude * cr, dc + m, noise * g)
//   COMPLEX  k = (dc + m) * amplitude;  re = fma(k, cr, noise * g),  im = k * ci
// The reference draws one Gaussian per sample there, for COMPLEX too (noise on I only), so draw d is sample d and each
// thread's run of kGenRun draws is kGenRun samples.
#pragma once
#include <stdint.h>

#include "raw_ingest.cuh"  // ScaleChange, scale_at

namespace kfft {

constexpr int kGenThreads = 128;
constexpr int kGenRun = 64;       // draws per thread: REAL 64 samples, COMPLEX 32 pairs
constexpr int kGenJumpBits = 24;  // threads per launch < 2^24: up to 2^30 draws
constexpr int kGf2Table = 64 * 16 * 4;  // uint64 words of one jump matrix

struct U128 {
  unsigned long long lo, hi;
};
__device__ __forceinline__ U128 add128(U128 a, U128 b) {
  U128 r;
  r.lo = a.lo + b.lo;
  r.hi = a.hi + b.hi + (r.lo < a.lo);
  return r;
}
// (n * x) mod 2^128
__device__ __forceinline__ U128 mul128(unsigned long long n, U128 x) {
  U128 r;
  r.lo = n * x.lo;
  r.hi = __umul64hi(n, x.lo) + n * x.hi;
  return r;
}
// (a * x) mod 2^128, a and x both 128-bit
__device__ __forceinline__ U128 mul128x(U128 a, U128 x) {
  U128 r = mul128(a.lo, x);
  r.hi += a.hi * x.lo;
  return r;
}

struct GenArgs {
  unsigned long long base[4];  // xoshiro256** state before draw a0 * C
  U128 F, R;                   // step and sweep angles, cycles * 2^128
  double amplitude, noise, scale;
  ScaleChange const *chg;
  int nchg;
  long long a0;  // absolute sample of out[0], >= 0
  long count, history, L;
  unsigned long long const *tabs;  // kGenJumpBits jump matrices T^(kGenRun 2^b)
  float *out;
  double *part;  // 2 per thread: energy in the block of its first new sample, and in the next one
  double dc;             // modulated: the carrier component (AM 1, DSB 0)
  float const *mod;      // modulated: one envelope float per sample of out
};

__device__ __forceinline__ unsigned long long rotl64(unsigned long long x, int k) { return (x << k) | (x >> (64 - k)); }
// xoshiro256ss_next (gauss.c:47-61)
__device__ __forceinline__ unsigned long long xo_next(unsigned long long s[4]) {
  unsigned long long const r = rotl64(s[1] * 5, 7) * 9;
  unsigned long long const t = s[1] << 17;
  s[2] ^= s[0];
  s[3] ^= s[1];
  s[1] ^= s[2];
  s[0] ^= s[3];
  s[2] ^= t;
  s[3] = rotl64(s[3], 45);
  return r;
}
// real_gauss (gauss.c:103-111) of one draw u
__device__ __forceinline__ double gauss_of(unsigned long long u) {
  int const p = __popcll(u * 0x2c1b3c6dULL) + __popcll(u * 0x297a2d39ULL) - 64;
  double const x = __dadd_rn((double)p, __dmul_rn(__ll2double_rn((long long)u), 0x1p-63));
  return __dmul_rn(x, 0.1765469659009499);
}
// s = M s, M a jump matrix in nibble-table form: entry (w * 16 + q) * 16 + v is the XOR of the columns selected by
// nibble value v at nibble q of word w
__device__ __forceinline__ void gf2_apply(unsigned long long const *__restrict__ tab, unsigned long long s[4]) {
  unsigned long long y0 = 0, y1 = 0, y2 = 0, y3 = 0;
#pragma unroll
  for (int w = 0; w < 4; w++) {
    unsigned long long const x = s[w];
#pragma unroll
    for (int q = 0; q < 16; q++) {
      ulonglong2 const *e = (ulonglong2 const *)(tab + (((w * 16 + q) * 16 + (int)((x >> (4 * q)) & 15)) * 4));
      ulonglong2 const a = __ldg(e), b = __ldg(e + 1);
      y0 ^= a.x;
      y1 ^= a.y;
      y2 ^= b.x;
      y3 ^= b.y;
    }
  }
  s[0] = y0;
  s[1] = y1;
  s[2] = y2;
  s[3] = y3;
}

// MOD: the AM / DSB instantiation (one draw per sample, the envelope from a.mod)
template <bool CPLX, bool MOD>
__global__ void __launch_bounds__(kGenThreads) siggen_kernel(GenArgs a) {
  constexpr int C = CPLX ? 2 : 1;
  constexpr int S = MOD ? kGenRun : kGenRun / C;  // samples per thread
  long const t = (long)blockIdx.x * kGenThreads + threadIdx.x;
  long const i0 = t * S;
  double e_lo = 0, e_hi = 0;
  if (i0 < a.count) {
    unsigned long long s[4] = {a.base[0], a.base[1], a.base[2], a.base[3]};
    for (int b = 0; b < kGenJumpBits; b++)
      if ((t >> b) & 1) gf2_apply(a.tabs + (size_t)b * kGf2Table, s);
    unsigned long long const n0 = (unsigned long long)(a.a0 + i0);
    bool const carrier = a.amplitude != 0;
    U128 ph = {0, 0}, inc = {0, 0};
    if (carrier) {  // phi_n0 = n0 F + n0 (n0 + 1) / 2 R, and the step to n0 + 1: F + (n0 + 1) R
      U128 tri;
      tri.lo = n0 * (n0 + 1);
      tri.hi = __umul64hi(n0, n0 + 1);
      tri.lo = (tri.lo >> 1) | (tri.hi << 63);
      tri.hi >>= 1;
      ph = add128(mul128(n0, a.F), mul128x(tri, a.R));
      inc = add128(a.F, mul128(n0 + 1, a.R));
    }
    long const blk0 = i0 < a.history ? 0 : (i0 - a.history) / a.L;
    long const end = i0 + S < a.count ? i0 + S : a.count;
    for (long i = i0; i < end; i++) {
      double const sc = a.nchg ? scale_at(a.chg, a.nchg, a.scale, a.a0 + i) : a.scale;
      double cr = 0, ci = 0;
      if (carrier) {
        double const phi = __dmul_rn(__ull2double_rn(ph.hi), 0x1p-63);  // 2 phi, in [0, 2]
        sincospi(phi, &ci, &cr);
        ph = add128(ph, inc);
        inc = add128(inc, a.R);
      }
      double re, e;
      if constexpr (MOD) {
        double const m = (double)a.mod[i];
        double const ng = __dmul_rn(a.noise, gauss_of(xo_next(s)));
        if constexpr (CPLX) {
          double const k = __dmul_rn(__dadd_rn(m, a.dc), a.amplitude);
          re = __fma_rn(k, cr, ng);
          double const im = __dmul_rn(k, ci);
          e = __fma_rn(im, im, __dmul_rn(re, re));
          a.out[2 * i + 1] = __double2float_rn(__dmul_rn(im, sc));
        } else {
          re = __fma_rn(__dmul_rn(a.amplitude, cr), __dadd_rn(m, a.dc), ng);
          e = __dmul_rn(re, re);
        }
        a.out[i * C] = __double2float_rn(__dmul_rn(re, sc));
      } else {
        // samp = amplitude * step_osc() + noise * gauss, the product by the carrier contracted into an FMA
        re = carrier ? __fma_rn(a.amplitude, cr, __dmul_rn(a.noise, gauss_of(xo_next(s))))
                     : __dmul_rn(a.noise, gauss_of(xo_next(s)));
        e = __dmul_rn(re, re);
        a.out[i * C] = __double2float_rn(__dmul_rn(re, sc));
        if constexpr (CPLX) {
          double const im = carrier ? __fma_rn(a.amplitude, ci, __dmul_rn(a.noise, gauss_of(xo_next(s))))
                                    : __dmul_rn(a.noise, gauss_of(xo_next(s)));
          e = __fma_rn(im, im, e);
          a.out[i * C + 1] = __double2float_rn(__dmul_rn(im, sc));
        }
      }
      if (i >= a.history) {
        if ((i - a.history) / a.L == blk0) e_lo += e;
        else e_hi += e;
      }
    }
  }
  if (a.part) {
    a.part[2 * t] = e_lo;
    a.part[2 * t + 1] = e_hi;
  }
}

// Block j's energy: the partial sums of the threads whose runs meet its L new samples, in thread order per lane, then
// a fixed tree across the CTA, so the result does not depend on timing.
__global__ void __launch_bounds__(256) siggen_energy_kernel(double const *__restrict__ part, long history, long L, int S,
                                                            long nthreads, double *__restrict__ energy) {
  int const j = blockIdx.x;
  long const lo = history + (long)j * L, hi = lo + L;  // samples [lo, hi)
  long const t0 = lo / S, t1 = (hi - 1) / S;
  double sum = 0;
  for (long t = t0 + threadIdx.x; t <= t1 && t < nthreads; t += 256) {
    long const first = t * S > history ? t * S : history;  // the thread's first new sample
    long const blk0 = (first - history) / L;
    sum += part[2 * t + (blk0 == j ? 0 : 1)];
  }
  __shared__ double red[256];
  red[threadIdx.x] = sum;
  __syncthreads();
  for (int k = 128; k > 0; k >>= 1) {
    if (threadIdx.x < k) red[threadIdx.x] += red[threadIdx.x + k];
    __syncthreads();
  }
  if (threadIdx.x == 0) energy[j] = red[0];
}

}  // namespace kfft
