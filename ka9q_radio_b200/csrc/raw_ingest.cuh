// raw_ingest.cuh -- the 8- and 16-bit front ends' sample conversion (rtlsdr.c:316-343, hydrasdr.c:681-716, :729-747,
// :759-830, bladerf.c:215-246, sdrplay.c:1234-1246) and the per-block A/D statistics of every raw ingest format (energy,
// components at the limits, samples with a component at the limits).
//
// Both kernels walk one overlap-save launch: a window of `history` samples followed by nblocks blocks of L new samples.
// grid.y picks the segment: y < nblocks is block y's new samples, whose statistics go to stats[y]; for the unpack
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

struct ScaleChange {  // = struct kgpu_scale_change
  long long at;
  double scale;
};

// The scale of absolute sample a: that of the last of the n changes (sorted by at) at or before a, `base` before the first.
__device__ __forceinline__ double scale_at(ScaleChange const *chg, int n, double base, long long a) {
  int lo = 0, hi = n;
  while (lo < hi) {
    int const mid = (lo + hi) >> 1;
    if (chg[mid].at <= a) lo = mid + 1;
    else hi = mid;
  }
  return lo ? chg[lo - 1].scale : base;
}

// The word decodes of unpack_kernel: each gives a word's integer x and whether x is at the format's limits.
struct DecodeU8 {  // excess-128 bytes: RTL-SDR (rtlsdr.c:316-343), HydraSDR UINT8_* (hydrasdr.c:759-775, :793-811)
  using Word = uint8_t;
  static __device__ __forceinline__ int x(Word w) { return (int)w - 128; }
  static __device__ __forceinline__ bool over(int x) { return x >= 127 || x <= -128; }
};
struct DecodeS8 {  // signed bytes: HydraSDR INT8_* (hydrasdr.c:776-791, :812-830)
  using Word = uint8_t;
  static __device__ __forceinline__ int x(Word w) { return (int)(int8_t)w; }
  static __device__ __forceinline__ bool over(int x) { return x >= 127 || x <= -128; }
};
struct DecodeS16 {  // int16: HydraSDR INT16_REAL / INT16_IQ (hydrasdr.c:700-716, :729-747), SDRplay (sdrplay.c:1238-1242)
  using Word = uint16_t;
  static __device__ __forceinline__ int x(Word w) { return (int)(int16_t)w; }
  static __device__ __forceinline__ bool over(int x) { return x >= 32767 || x <= -32768; }
};
struct DecodeU16 {  // offset-binary uint16: HydraSDR UINT16_REAL at 16 bits per sample (hydrasdr.c:681-699, :265-267)
  using Word = uint16_t;
  static __device__ __forceinline__ int x(Word w) { return (int)w - 32768; }
  static __device__ __forceinline__ bool over(int x) { return x >= 32767 || x <= -32768; }
};
struct DecodeSC16Q11 {  // bladeRF SC16_Q11 (bladerf.c:226-235): bits 0-11 sign-extended from bit 11, bits 12-15 ignored
  using Word = uint16_t;
  static __device__ __forceinline__ int x(Word w) { return (int)((w & 0xfffu) ^ 0x800u) - 0x800; }
  static __device__ __forceinline__ bool over(int x) { return x == 2047 || x == -2048; }  // s == 0x7ff || s == 0x800
};

// Raw words -> float, one thread per sample.  The value is (float)(scale * (double)x) as the drivers' loops store it: a
// double product rounded once more to float (no float multiply, no FMA), with the sample's own scale where nchg changes
// are given (in[0] being absolute sample a0).  D decodes each word (above).
template <class D, bool CPLX>
__global__ void __launch_bounds__(kRawThreads) unpack_kernel(typename D::Word const *__restrict__ in, long history, long L,
                                                             int nblocks, double scale, ScaleChange const *__restrict__ chg,
                                                             int nchg, long long a0, float *__restrict__ out, BlockStats *stats) {
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
    double const sc = nchg ? scale_at(chg, nchg, scale, a0 + base + i) : scale;
#pragma unroll
    for (int c = 0; c < C; c++) {
      int const x = D::x(in[s + c]);
      out[s + c] = __double2float_rn(__dmul_rn(sc, (double)x));
      e += (unsigned)(x * x);
      o += D::over(x);
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

// int16 words -> float for a window that holds more than one scale, one thread per sample (in[0] being absolute sample
// a0): (float)x * (float)s after the optional derandomization, s the sample's own scale -- what fwd_cols' fused
// conversion computes with one scale (rx888.c:765, airspy-unpack.c:124), so kgpu_forward then runs on floats.
template <bool CPLX>
__global__ void __launch_bounds__(kRawThreads) scale_i16_kernel(short const *__restrict__ in, long count, long long a0, double base,
                                                                ScaleChange const *__restrict__ chg, int nchg, int derandomize,
                                                                float *__restrict__ out) {
  long const i = (long)blockIdx.x * kRawThreads + threadIdx.x;
  if (i >= count) return;
  float const sc = (float)scale_at(chg, nchg, base, a0 + i);
  constexpr int C = CPLX ? 2 : 1;
#pragma unroll
  for (int c = 0; c < C; c++) {
    short v = in[i * C + c];
    if (derandomize) v ^= (short)((v & 1) ? 0xfffe : 0);
    out[i * C + c] = __fmul_rn((float)v, sc);
  }
}

}  // namespace kfft
