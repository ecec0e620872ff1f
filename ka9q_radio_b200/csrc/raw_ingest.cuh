// raw_ingest.cuh -- the 8-bit, 16-bit and float front ends' sample conversion (rtlsdr.c:316-343, hydrasdr.c:681-830,
// bladerf.c:215-246, sdrplay.c:1234-1246, airspyhf.c:308-318, fobos.c:410-420) and the per-block A/D statistics of every
// raw ingest format (energy, components at the limits, samples with a component at the limits).
//
// Both kernels walk one overlap-save launch: a window of `history` samples followed by nblocks blocks of L new samples.
// grid.y picks the segment: y < nblocks is block y's new samples, whose statistics go to stats[y]; for the unpack
// y == nblocks is the history, converted but never counted (the drivers count each sample once).  A sample is one value
// (REAL) or one I/Q pair (COMPLEX); every component counts in the energy and in the component count.
#pragma once
#include <stdint.h>
#include <cooperative_groups.h>
#include <type_traits>

namespace kfft {

constexpr int kRawThreads = 256;

struct BlockStats {  // = struct kgpu_block_stats
  union {
    unsigned long long energy;  // integer formats
    double fenergy;             // float formats (float_energy_kernel)
  };
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
// The float decodes store a value of their own rule and count nothing: the float drivers test no limits, and their
// energy is a double that float_energy_kernel sums (below).
struct DecodeF32 {  // (float)(scale * (double)x): hydrasdr.c:724, :753-754, airspyhf.c:315-317
  using Word = float;
  static __device__ __forceinline__ float store(float x, double sc) { return __double2float_rn(__dmul_rn(sc, (double)x)); }
};
struct DecodeF32FScale {  // x * (float)scale, a float product: fobos.c:419
  using Word = float;
  static __device__ __forceinline__ float store(float x, double sc) { return __fmul_rn(x, __double2float_rn(sc)); }
};

// Raw words -> float, one thread per sample.  The value is (float)(scale * (double)x) as the drivers' loops store it: a
// double product rounded once more to float (no float multiply, no FMA), with the sample's own scale where nchg changes
// are given (in[0] being absolute sample a0).  D decodes each word (above); a float decode stores by its own rule.
template <class D, bool CPLX>
__global__ void __launch_bounds__(kRawThreads) unpack_kernel(typename D::Word const *__restrict__ in, long history, long L,
                                                             int nblocks, double scale, ScaleChange const *__restrict__ chg,
                                                             int nchg, long long a0, float *__restrict__ out, BlockStats *stats) {
  int const seg = blockIdx.y;
  long const len = seg < nblocks ? L : history;
  if ((long)blockIdx.x * kRawThreads >= len) return;  // the whole CTA lies past its segment
  long const base = seg < nblocks ? history + (long)seg * L : 0;
  long const i = (long)blockIdx.x * kRawThreads + threadIdx.x;
  constexpr int C = CPLX ? 2 : 1;
  if constexpr (std::is_same<typename D::Word, float>::value) {  // float decodes: stores only (float_energy_kernel counts)
    if (i < len) {
      long const s = (base + i) * C;
      double const sc = nchg ? scale_at(chg, nchg, scale, a0 + base + i) : scale;
#pragma unroll
      for (int c = 0; c < C; c++) out[s + c] = D::store(in[s + c], sc);
    }
  } else {
    unsigned long long e = 0;
    unsigned o = 0;
    if (i < len) {
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
}

// The energy terms of the float drivers' loops, each computed as the loop's source writes it before adding it to its
// sum: one term per component (kComps 1) or per I/Q pair (2).  One deliberate departure: the reference builds airspyhf.c
// with -ffp-contract=fast, which contracts cnrmf's re*re + im*im into a fused multiply-add; EnergyCnrmf rounds both
// products, as the source says, and differs from the contracted term by at most a float rounding (2^-24 relative).  A
// NaN or Inf sample, or a square past FLT_MAX in a float term, gives a non-finite term, so the block's energy is
// non-finite as the loop's transfer energy is (its isfinite guard); filter_ingest_stats adds every drained block's
// energy, so one such block makes the whole drained batch non-finite.
struct EnergySq {  // float x * x: hydrasdr.c:725, fobos.c:418
  static constexpr int kComps = 1;
  static __device__ __forceinline__ double term(float const *p) { return (double)__fmul_rn(p[0], p[0]); }
};
struct EnergyCnrmf {  // cnrmf, a float sum of float squares, uncontracted: airspyhf.c:316, misc.h:279-281
  static constexpr int kComps = 2;
  static __device__ __forceinline__ double term(float const *p) {
    return (double)__fadd_rn(__fmul_rn(p[0], p[0]), __fmul_rn(p[1], p[1]));
  }
};
struct EnergyCnrm {  // cnrm of the pair as doubles (exact squares, one rounding): hydrasdr.c:755, misc.h:282-284
  static constexpr int kComps = 2;
  static __device__ __forceinline__ double term(float const *p) {
    double const a = p[0], b = p[1];
    return __dadd_rn(__dmul_rn(a, a), __dmul_rn(b, b));
  }
};

constexpr int kEnergyCluster = 8, kEnergyThreads = 1024;
// Block y's energy over its L new samples (in[0] the launch's first history sample, C components per sample), summed in
// double in a fixed order, so it does not depend on timing: lane t = blockIdx.x * kEnergyThreads + threadIdx.x adds
// terms t, t + kLanes, t + 2 kLanes, ... in turn; each CTA halves its lanes' sums pairwise (red[i] += red[i + h], h =
// 512 .. 1); CTA 0 of the cluster adds the eight CTA sums in rank order into stats[y].fenergy (tests/float_ingest_ref.py
// restates it).  The drivers' own sums are reassociated by their compiler, and fobos.c's is a float sum.
template <class E>
__global__ void __cluster_dims__(kEnergyCluster, 1, 1) __launch_bounds__(kEnergyThreads)
    float_energy_kernel(float const *__restrict__ in, long history, long L, int C, BlockStats *stats) {
  namespace cg = cooperative_groups;
  constexpr long kLanes = (long)kEnergyCluster * kEnergyThreads;
  long const n = L * C / E::kComps;
  float const *const p = in + (history + (long)blockIdx.y * L) * C;
  double sum = 0;
#pragma unroll 4
  for (long t = (long)blockIdx.x * kEnergyThreads + threadIdx.x; t < n; t += kLanes) sum = __dadd_rn(sum, E::term(p + t * E::kComps));
  __shared__ double red[kEnergyThreads];
  red[threadIdx.x] = sum;
  __syncthreads();
#pragma unroll
  for (int h = kEnergyThreads / 2; h > 0; h >>= 1) {
    if (threadIdx.x < h) red[threadIdx.x] = __dadd_rn(red[threadIdx.x], red[threadIdx.x + h]);
    __syncthreads();
  }
  cg::cluster_group cl = cg::this_cluster();
  cl.sync();  // every CTA's red[0] is final
  if (cl.block_rank() == 0 && threadIdx.x == 0) {
    double e = 0;
    for (int r = 0; r < kEnergyCluster; r++) e = __dadd_rn(e, *cl.map_shared_rank(red, r));
    stats[blockIdx.y].fenergy = e;
  }
  cl.sync();  // no CTA leaves while CTA 0 reads its shared memory
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
