// bluestein_chan.cuh -- channels whose point count Ns has no transform of their own: a prime factor >= 29, or a prime
// factor 11 .. 23 above kMaxWideChanPoints (kgpu_bank_define_any).  The inverse transform runs as a forward Bluestein
// transform of the conjugate slice, IDFT(S) = conj(DFT(conj S)), so it reuses the masters' chirp w_n = exp(-i pi n^2 / Ns)
// and B = DFT_P of the conjugate chirp (bluestein_master.cuh) exactly.  Per chunk of (channel, block) rows:
//   bluestein_chan_in      a_k = conj(S_k) w_k, S = slice x response (huge_slice: every variant), zero-padded to P
//   kgpu_forward           A = DFT_P(a)                       (an internal 7-smooth COMPLEX master, L = P, M = 1)
//   bluestein_mul_kernel   conj(A B)                          (bluestein_master.cuh)
//   kgpu_forward           y = DFT_P(conj(A B))
//   bluestein_chan_out     Z_n = w_n conj(y_n) / P; output conj(Z_n) for the last olen n, with the plain, oscillator
//                          and REAL-output stores of chan_huge_rows
// A row of the scratch is one (channel, block): row = block * channels + channel, as chan_huge's slots.  The block
// power of an oscillator channel is summed per CTA in a fixed order and huge_power_kernel adds the CTAs' partial sums in
// a fixed order, so a (channel, block) gets bitwise the same power whichever launch computes it.
#pragma once
#include "bluestein_master.cuh"
#include "chan_huge.cuh"

namespace kfft {

// grid (P / kBluesteinThreads tiles, channels, blocks); out: [row][P]
__global__ void __launch_bounds__(kBluesteinThreads) bluestein_chan_in(ChanArgs const a, long P, float2 *out) {
  long const k = (long)blockIdx.x * kBluesteinThreads + threadIdx.x;
  if (k >= P) return;
  int const oi = blockIdx.y;
  int const ci = chan_index(a, oi);
  ChanDesc const d = a.desc[ci];
  if (d.plan < 0) return;
  int const blk = blockIdx.z;
  float2 v = make_float2(0.f, 0.f);
  if (k < d.points) {
    ChanAux ax{};
    if (d.flags & kChanBeam) ax = a.aux[ci];
    float2 const s = huge_slice(a, d, ax, a.spec + (long)blk * a.spec_stride, a.resp + d.resp_off, (int)k);
    float2 const w = bluestein_chirp(k, d.points, 1.0);
    v = make_float2(s.x * w.x + s.y * w.y, s.x * w.y - s.y * w.x);  // conj(s) w
  }
  out[((long)blk * gridDim.y + oi) * P + k] = v;
}

// grid (olen / kBluesteinThreads tiles, channels, blocks); y: [row][y_stride], the second pass's spectra.
// partial: [row][gridDim.x] per-CTA power sums of kChanOsc channels.
__global__ void __launch_bounds__(kBluesteinThreads) bluestein_chan_out(ChanArgs const a, double inv_p, float2 const *y, long y_stride,
                                                                       float *partial) {
  int const oi = blockIdx.y;
  int const ci = chan_index(a, oi);
  ChanDesc const d = a.desc[ci];
  if (d.plan < 0) return;
  int const blk = blockIdx.z, tid = threadIdx.x;
  long const row = (long)blk * gridDim.y + oi;
  int const i = blockIdx.x * kBluesteinThreads + tid;  // output sample; n = Ns - olen + i
  bool const live = i < d.olen;
  float2 v = make_float2(0.f, 0.f);
  if (live) {
    long const n = (long)(d.points - d.olen) + i;
    float2 const z = bluestein_z(y + row * y_stride, bluestein_chirp(n, d.points, inv_p), n);
    v = make_float2(z.x, -z.y);
  }
  float2 *dst = a.out + (long)blk * a.out_stride + d.out_off;
  if (d.flags & kChanRealOut) {  // c2r: the real part, olen floats packed in the channel's float2 run
    if (live) reinterpret_cast<float *>(dst)[i] = v.x;
    return;
  }
  if (d.flags & kChanOsc) {
    ChanAux const ax = a.aux[ci];
    float pw = 0.f;
    if (live) dst[i] = osc_sample(ax, a.block0 + blk - ax.osc_epoch, d.olen, i, v, pw);
    float const s = cta_power_sum<kBluesteinThreads>(pw);
    if (partial && tid == 0) partial[row * gridDim.x + blockIdx.x] = s;
    return;
  }
  if (live) dst[i] = v;
}

}  // namespace kfft
