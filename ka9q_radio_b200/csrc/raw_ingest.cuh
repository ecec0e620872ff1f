// raw_ingest.cuh -- the 8-bit front ends' sample conversion (rtlsdr.c:316-343, hydrasdr.c:759-830) and the per-block A/D
// statistics of every raw ingest format (energy, components at the limits, samples with a component at the limits).
//
// Both kernels walk one overlap-save launch: a window of `history` samples followed by nblocks blocks of L new samples.
// grid.y picks the segment: y < nblocks is block y's new samples, whose statistics go to stats[y]; for the 8-bit unpack
// y == nblocks is the history, converted but never counted (the drivers count each sample once).  A sample is one value
// (REAL) or one I/Q pair (COMPLEX); every component counts in the energy and in the component count.
#pragma once
#include <stdint.h>

namespace kfft {

constexpr int kRawThreads = 256;

struct BlockStats {  // = struct kgpu_block_stats
  unsigned long long energy;
  unsigned int overs;         // components at the format's limits
  unsigned int over_samples;  // samples with at least one component at the limits
};

// Warp sums of one thread's counts into *s (every lane of the warp calls it).
__device__ __forceinline__ void block_stats_add(BlockStats *s, unsigned long long e, unsigned o, unsigned os) {
#pragma unroll
  for (int k = 16; k > 0; k >>= 1) {
    e += __shfl_xor_sync(0xffffffffu, e, k);
    o += __shfl_xor_sync(0xffffffffu, o, k);
    os += __shfl_xor_sync(0xffffffffu, os, k);
  }
  if ((threadIdx.x & 31) == 0) {
    if (e) atomicAdd(&s->energy, e);
    if (o) {
      atomicAdd(&s->overs, o);
      atomicAdd(&s->over_samples, os);
    }
  }
}

// u8 (excess-128) or s8 words -> float, one thread per sample.  The value is (float)(scale * (double)x) as the drivers'
// loops store it: a double product rounded once more to float (no float multiply, no FMA).  At the limits: x >= 127 or
// x <= -128, i.e. bytes 0 and 255 of u8 (rtlsdr.c:324-333) and 127, -128 of s8 (hydrasdr.c:781).
template <bool SIGNED, bool CPLX>
__global__ void __launch_bounds__(kRawThreads) unpack8_kernel(uint8_t const *__restrict__ in, long history, long L, int nblocks,
                                                              double scale, float *__restrict__ out, BlockStats *stats) {
  int const seg = blockIdx.y;
  long const len = seg < nblocks ? L : history;
  if ((long)blockIdx.x * kRawThreads >= len) return;  // the whole CTA lies past its segment
  long const base = seg < nblocks ? history + (long)seg * L : 0;
  long const i = (long)blockIdx.x * kRawThreads + threadIdx.x;
  unsigned long long e = 0;
  unsigned o = 0;
  if (i < len) {
    constexpr int C = CPLX ? 2 : 1;
    long const s = (base + i) * C;
#pragma unroll
    for (int c = 0; c < C; c++) {
      uint8_t const b = in[s + c];
      int const x = SIGNED ? (int)(int8_t)b : (int)b - 128;
      out[s + c] = __double2float_rn(__dmul_rn(scale, (double)x));
      e += (unsigned)(x * x);
      o += (x >= 127 || x <= -128);
    }
  }
  if (stats && seg < nblocks) block_stats_add(stats + seg, e, o, o != 0);
}

// Statistics of int16 words already on the device, one thread per sample of block y's new samples: the RX888's words
// after the optional derandomization (rx888.c:707-712, 759-762), or Airspy packed-12 values after the unpack
// (airspy-unpack.c:121-124).  At the limits: |x| >= limit (32767 for int16, 2047 for packed-12).
template <bool CPLX>
__global__ void __launch_bounds__(kRawThreads) block_stats_i16_kernel(short const *__restrict__ in, long history, long L,
                                                                      int derandomize, int limit, BlockStats *stats) {
  if ((long)blockIdx.x * kRawThreads >= L) return;
  long const i = (long)blockIdx.x * kRawThreads + threadIdx.x;
  unsigned long long e = 0;
  unsigned o = 0;
  if (i < L) {
    constexpr int C = CPLX ? 2 : 1;
    long const s = (history + (long)blockIdx.y * L + i) * C;
#pragma unroll
    for (int c = 0; c < C; c++) {
      short v = in[s + c];
      if (derandomize) v ^= (short)((v & 1) ? 0xfffe : 0);
      int const x = v;
      e += (unsigned)(x * x);
      o += (x >= limit || x <= -limit);
    }
  }
  block_stats_add(stats + blockIdx.y, e, o, o != 0);
}

}  // namespace kfft
