// chan_kernels.cuh -- the per-channel half of the fast convolver, batched: for every channel
// (slave) and block, gather its bins from the master spectrum, multiply by the channel's
// frequency response, run the small inverse transform and keep the last olen samples.
// Replaces execute_filter_output's arithmetic (reference filter.c:728-921): the four slicing
// loops (:728-893), ISB (:895-909), Nyquist zero (:911), fftwf_execute(rev_plan) (:914) and the
// "output = buffer + points - olen" discard (:357).
//
// One warp owns one (channel, block): the 600-point NBFM case is two fat in-register stages
// (radix 24 then 25) with only __syncwarp between them; hundreds of channels x several blocks
// go out as one grid.
#pragma once
#include "fft_tile.cuh"

namespace kfft {

constexpr int kChanWarps = 4;  // (channel, block) pairs per CTA

// Longest channel transform: chan_kernel holds kChanWarps columns of (points rounded up to 4) + 2 float2 in shared
// memory, which must fit the 227 KB a block may opt into on sm_90.  7260 points.
constexpr int kChanSmemLimit = 227 * 1024;
constexpr int kMaxChanPoints = (kChanSmemLimit / (8 * kChanWarps) - 2) / 4 * 4;

// Host-resolved description of how output bin t (in the reference's walk order, starting at the
// most negative output bin) maps onto the master spectrum.  Covers filter.c:810-893 (REAL
// master, upright or inverted) and :728-793 (COMPLEX master with circular wrap).
struct ChanDesc {
  int plan;        // registry index of the length-`points` inverse plan (kPlanExt, kPlanBluestein: none), < 0: disabled
  int points;      // Ns
  int olen;        // Ls
  int zlead;       // walk positions t < zlead are zero
  int ncopy;       // then ncopy bins are taken from the master ...
  int q0;          // ... starting at master bin q0 ...
  int dir;         // ... stepping +1 or -1 (inverted spectrum => conjugate, filter.c:876)
  int flags;       // kChanIsb | kChanRealOut | kChanBeam | kChanOsc
  long resp_off;   // float2 offset of this channel's response
  long out_off;    // float2 offset of this channel's output inside a block's output row
};

// ChanDesc::plan of a channel whose length has a prime factor 11 .. 23 (kgpu_bank_define_ext): runnable, but not a
// registry index, so it must never reach a kernel that reads c_plans[d.plan]; its plan reaches chan_kernel_ext or
// chan_wide_ext by value.
constexpr int kPlanExt = kMaxPlans;
// ChanDesc::plan of a channel served by a Bluestein transform (kgpu_bank_define_any, bluestein_chan.cuh): runnable for
// the noise estimator and huge_power_kernel, and never a registry index either.
constexpr int kPlanBluestein = kMaxPlans + 1;

enum : int {
  kChanIsb = 1,      // filter_out.isb (filter.c:895-909)
  kChanRealOut = 2,  // REAL-output slave: positive-frequency slice + c2r inverse, olen floats (filter.c:794-809, :386); q0 = shift
  kChanBeam = 4,     // beam synthesis on a COMPLEX master (filter.c:756-775), weights in ChanAux
  kChanOsc = 8       // fine-tuning oscillator + block phase on the output, power per block (radio.c:1476-1501, :1515-1520)
};

// Per-channel parameters that only the flagged variants read.
struct ChanAux {
  double osc_phase;  // cycles at the epoch, before any block adjustment
  double osc_freq;   // cycles per output sample (= -remainder / output rate, radio.c:1481)
  double osc_rate;   // cycles per sample^2 (doppler rate)
  double osc_adj;    // cycles added at the start of every block: (shift % V) / V (radio.c:1493,1497)
  long osc_epoch;    // bank block counter at which osc_phase holds
  double are, aim, bre, bim;  // beam weights alpha, beta (filter.c:926-927)
};

// Phase (cycles, reduced to [-0.5, 0.5]) of output sample n of the block that is k blocks past the epoch:
// step_osc hands out the phasor BEFORE stepping, phasor_step is multiplied by phasor_step_step before each step
// (osc.c:60-70), and the block adjustment is applied before the block's first sample (radio.c:1497).
__device__ __forceinline__ double osc_phase_cycles(ChanAux const &x, long k, int olen, int n) {
  double const m = (double)(k * (long)olen + n);
  double ph = fma((double)(k + 1), x.osc_adj, x.osc_phase);
  ph = fma(m, x.osc_freq, ph);
  if (x.osc_rate != 0.0) ph = fma(0.5 * m * (m + 1.0), x.osc_rate, ph);
  return ph - rint(ph);
}
__device__ __forceinline__ float2 osc_rotate(float2 v, double ph_cycles) {
  float sn, cs;
  sincospif(2.0f * (float)ph_cycles, &sn, &cs);
  return make_float2(v.x * cs - v.y * sn, v.x * sn + v.y * cs);
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

struct ChanArgs {
  float2 const *spec;
  long spec_stride;
  int m_bins;        // master bins (wrap modulus for COMPLEX masters)
  int wrap;          // 1: COMPLEX master (q wraps mod m_bins), 0: REAL
  ChanDesc const *desc;
  int const *order;  // descriptor indices to process (one launch per plan), or nullptr:
  int norder;        //   then descriptors chan_base .. chan_base+norder-1
  int chan_base;
  float2 const *resp;
  float2 *out;
  long out_stride;
  int pitch;         // shared-memory floats2 per warp
  ChanAux const *aux;  // [descriptor index], read only for flagged channels
  long block0;         // bank block counter of this launch's block 0 (oscillator epoch arithmetic)
  float *power;        // nullptr or [block][power_stride]: mean |y|^2 of each kChanOsc channel's block (radio.c:1515-1520)
  long power_stride;
};

}  // namespace kfft
#include "chan_slice.cuh"
namespace kfft {

__global__ void __launch_bounds__(kChanWarps * 32) chan_kernel(ChanArgs const a) {
#define KFFT_CHAN_EXT false
#include "chan_body.cuh"
#undef KFFT_CHAN_EXT
}
// The channels of one extended length (prime factors up to 23), every variant chan_kernel serves.
__global__ void __launch_bounds__(kChanWarps * 32) chan_kernel_ext(ChanArgs const a, __grid_constant__ TilePlan const xpl) {
#define KFFT_CHAN_EXT true
#include "chan_body.cuh"
#undef KFFT_CHAN_EXT
}

// Forward transform of one response in place (set_filter's fftwf_execute, filter.c:1030):
// one warp, data staged through shared memory.
template <bool EXT>
__device__ __forceinline__ void response_fft_body(float2 *resp, TilePlan const &pl) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  float2 *col = reinterpret_cast<float2 *>(smem_raw);
  int const lane = threadIdx.x;
  for (int i = lane; i < pl.len; i += 32) col[i] = resp[i];
  __syncwarp();
  tile_fft<false, EXT>(pl, col, lane, 32, [] { __syncwarp(); });
  for (int k = lane; k < pl.len; k += 32) resp[k] = col[pl.perm[k]];
}
__global__ void __launch_bounds__(32) response_fft_kernel(float2 *resp, int plan) { response_fft_body<false>(resp, c_plans[plan]); }
__global__ void __launch_bounds__(32) response_fft_ext(float2 *resp, __grid_constant__ TilePlan const pl) {
  response_fft_body<true>(resp, pl);
}

}  // namespace kfft
