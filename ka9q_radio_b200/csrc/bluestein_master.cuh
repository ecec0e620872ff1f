// bluestein_master.cuh -- forward transform of masters whose complex length nc has no split the two-pass pair runs
// (a prime factor >= 29, or a 23-smooth length without a split that fits shared memory).  Around two unchanged
// kgpu_forward passes of an internal 7-smooth COMPLEX master of length P >= 2 nc - 1, per chunk of blocks:
//   bluestein_in_kernel    window (float or int16 pairs, the master's hop) -> a = z w, zero-padded to P; int16 statistics
//   kgpu_forward           A = DFT_P(a)
//   bluestein_mul_kernel   conj(A B), B = DFT_P of the conjugate chirp
//   kgpu_forward           y = DFT_P(conj(A B)) = P conj(a (*) conj w)
//   bluestein_out_kernel   Z_k = w_k conj(y_k) / P, k < nc; REAL masters: the real split to bins 0 .. nc
// w_n = exp(-i pi n^2 / nc), from n^2 mod 2 nc in 64-bit integers and one double sincospi, rounded once.
// z is the master's complex sequence: REAL windows as packed pairs z[n] = x[2n] + i x[2n+1], COMPLEX as (re, im).
#pragma once
#include <cuda_runtime.h>

#include "fwd_kernels.cuh"

namespace kfft {

constexpr int kBluesteinThreads = 256;

// exp(-i pi (k^2 mod 2 nc) / nc) * mul, in double, rounded once
__device__ __forceinline__ float2 bluestein_chirp(long k, long nc, double mul) {
  long const r = (k * k) % (2 * nc);
  double s, c;
  sincospi((double)r / (double)nc, &s, &c);
  return make_float2((float)(c * mul), (float)(-s * mul));
}

// out[s][k] = conj(spec[s][k] * B[k]) for k < P: the input of the second pass.  Every Bluestein transform (masters,
// channels, the spectrum analyzer) runs it between its two passes.
__global__ void __launch_bounds__(kBluesteinThreads) bluestein_mul_kernel(float2 const *__restrict__ spec, long spec_stride,
                                                                          float2 const *__restrict__ B, int P,
                                                                          float2 *__restrict__ out) {
  long const k = (long)blockIdx.x * kBluesteinThreads + threadIdx.x;
  if (k >= P) return;
  int const seg = blockIdx.y;
  float2 const a = spec[(long)seg * spec_stride + k], b = B[k];
  out[(long)seg * P + k] = make_float2(a.x * b.x - a.y * b.y, -(a.x * b.y + a.y * b.x));
}

struct BluesteinInArgs {
  void const *in;       // block 0's window: float2 or short2 pairs
  long hop;             // pairs between consecutive windows (L/2 REAL, L COMPLEX)
  long nc, P;
  long first_new;       // pair index of a window's first new sample (statistics)
  int nblocks;
  int i16, derandomize;
  float scale;          // int16: scale * (float)x after the randomizer flip, as the column passes
  IngestStats *stats;   // int16 only, or nullptr: [nblocks]
  float2 *out;          // [nblocks][P]
};

// One thread per point k < P, looping over the chunk's blocks so the chirp is computed once.
__global__ void __launch_bounds__(kBluesteinThreads) bluestein_in_kernel(BluesteinInArgs a) {
  long const k = (long)blockIdx.x * kBluesteinThreads + threadIdx.x;
  bool const live = k < a.nc;
  float2 const w = live ? bluestein_chirp(k, a.nc, 1.0) : make_float2(0.f, 0.f);
  bool const counted = live && k >= a.first_new;
  for (int b = 0; b < a.nblocks; b++) {
    float re = 0.f, im = 0.f;
    unsigned long long energy = 0;
    unsigned int clips = 0;
    if (live) {
      if (a.i16) {
        short2 const v = reinterpret_cast<short2 const *>(a.in)[(long)b * a.hop + k];
        short lo = v.x, hi = v.y;
        if (a.derandomize) {  // lsb set -> flip bits 1..15 (rx888.c:707-712)
          lo ^= (short)((lo & 1) ? 0xfffe : 0);
          hi ^= (short)((hi & 1) ? 0xfffe : 0);
        }
        if (counted) {
          energy = (unsigned long long)((int)lo * lo) + (unsigned long long)((int)hi * hi);
          clips = (lo > 32766 || lo < -32766) + (hi > 32766 || hi < -32766);
        }
        re = (float)lo * a.scale;
        im = (float)hi * a.scale;
      } else {
        float2 const v = reinterpret_cast<float2 const *>(a.in)[(long)b * a.hop + k];
        re = v.x;
        im = v.y;
      }
    }
    if (k < a.P) a.out[(long)b * a.P + k] = make_float2(re * w.x - im * w.y, re * w.y + im * w.x);
    if (a.stats) {
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        energy += __shfl_xor_sync(0xffffffffu, energy, o);
        clips += __shfl_xor_sync(0xffffffffu, clips, o);
      }
      if ((threadIdx.x & 31) == 0 && (energy | clips)) {
        atomicAdd(&a.stats[b].energy, energy);
        atomicAdd(&a.stats[b].clips, clips);
      }
    }
  }
}

struct BluesteinOutArgs {
  float2 const *y;      // [nblocks][y_stride]: the second pass's spectra
  long y_stride;
  long nc;
  double inv_p;         // 1 / P
  int real_split;       // REAL master: bins 0 .. nc of the real split; COMPLEX: bins 0 .. nc-1
  int nblocks;
  float2 *spec;         // [nblocks][spec_stride], bins only
  long spec_stride;
};

// Z_k = w_k conj(y_k) / P for k mod nc
__device__ __forceinline__ float2 bluestein_z(float2 const *y, float2 w, long k) {
  float2 const v = y[k];
  return make_float2(v.x * w.x + v.y * w.y, v.x * w.y - v.y * w.x);
}

// One thread per output bin, looping over the chunk's blocks.  REAL: X[k] = E - i W_{2nc}^k O with
// E = (Z[k] + conj Z[nc-k]) / 2, O = (Z[k] - conj Z[nc-k]) / 2 (indices mod nc), as the row passes split.
__global__ void __launch_bounds__(kBluesteinThreads) bluestein_out_kernel(BluesteinOutArgs a) {
  long const k = (long)blockIdx.x * kBluesteinThreads + threadIdx.x;
  long const bins = a.real_split ? a.nc + 1 : a.nc;
  if (k >= bins) return;
  long const ka = k == a.nc ? 0 : k;
  float2 const wa = bluestein_chirp(ka, a.nc, a.inv_p);
  if (!a.real_split) {
    for (int b = 0; b < a.nblocks; b++) a.spec[(long)b * a.spec_stride + k] = bluestein_z(a.y + (long)b * a.y_stride, wa, ka);
    return;
  }
  long const kb = ka == 0 ? 0 : a.nc - ka;
  float2 const wb = bluestein_chirp(kb, a.nc, a.inv_p);
  float2 const rc = unit_root_f(k, 2 * a.nc);  // W_{2nc}^k
  for (int b = 0; b < a.nblocks; b++) {
    float2 const *y = a.y + (long)b * a.y_stride;
    float2 const za = bluestein_z(y, wa, ka), zb = bluestein_z(y, wb, kb);
    float2 const E = make_float2(0.5f * (za.x + zb.x), 0.5f * (za.y - zb.y));
    float2 const O = make_float2(0.5f * (za.x - zb.x), 0.5f * (za.y + zb.y));
    float2 const P = cmul(rc, O);
    a.spec[(long)b * a.spec_stride + k] = make_float2(E.x + P.y, E.y - P.x);
  }
}

}  // namespace kfft
