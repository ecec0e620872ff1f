// noise_kernel.cuh -- per-channel noise-density estimate straight from the device-resident master spectrum.
// Replaces estimate_noise() (reference radio.c:1783-1866, quantile/quickselect :1722-1775): the energies of >= 1000
// master bins around the channel, their 10 % quantile q (linear interpolation between order statistics), the mean of
// the bins <= 1.5 q, a closed-form bias correction, scaled to 1 Hz.  The reference reads master->fdomain on the host,
// which forces a 13 MB device->host copy of every block's spectrum; here one double per channel and block leaves the GPU.
//
// One CTA per (channel, block).  Order statistics by an exact 4 x 8-bit radix select on the float bit patterns
// (energies are >= 0, so the unsigned order is the numeric order): no sort, O(n) per pass.  noise_kernel keeps the
// window's energies in dynamic shared memory of noise_window() words of the bank's widest channel whose window has at
// most kNoiseSmemBins; windows above that (huge channels from 57 088 bins, chan_huge.cuh) are estimated by
// noise_kernel_gm, which runs the same body on kNoiseGmThreads threads over energies kept in a global scratch slot.
#pragma once
#include "chan_kernels.cuh"

namespace kfft {

constexpr int kNoiseThreads = 128;
constexpr int kNoiseGmThreads = 512;
constexpr int kMinNoiseBins = 1000;   // radio.c:76
// the largest window noise_kernel holds in shared memory: 227 KB less 4 KB for its static arrays
constexpr int kNoiseSmemBins = (227 * 1024 - 4096) / 4;

// bins estimate_noise takes around a runnable channel: max(slave->bins, Min_noise_bins) (radio.c:1794-1797)
__host__ __device__ inline int noise_window(ChanDesc const &d) {
  int const s_bins = (d.flags & kChanRealOut) ? d.points / 2 + 1 : d.points;  // slave->bins (filter.c:347,374)
  return s_bins < kMinNoiseBins ? kMinNoiseBins : s_bins;
}

struct NoiseArgs {
  float2 const *spec;
  long spec_stride;
  int m_bins;
  int wrap;          // COMPLEX master
  ChanDesc const *desc;
  int const *shift;  // [descriptor index] the shift execute_filter_output was called with
  int nchan;
  double scale;      // correction / (m_bins * samprate)
  double *n0;        // [block][n0_stride]
  long n0_stride;
};

// k-th smallest (0-based) of e[0..n): returns its bit pattern; *n_le = number of elements <= that value
template <int NT>
__device__ inline unsigned radix_select(unsigned const *e, int n, int k, unsigned *hist /*256*/, int *sh /*4 ints*/) {
  unsigned prefix = 0, mask = 0;
  int kk = k;
  for (int pass = 3; pass >= 0; pass--) {
    for (int i = threadIdx.x; i < 256; i += NT) hist[i] = 0;
    __syncthreads();
    int const sft = 8 * pass;
    for (int i = threadIdx.x; i < n; i += NT) {
      unsigned const v = e[i];
      if ((v & mask) == prefix) atomicAdd(&hist[(v >> sft) & 255u], 1u);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      int acc = 0, d = 0;
      for (; d < 256; d++) {
        int const c = (int)hist[d];
        if (acc + c > kk) break;
        acc += c;
      }
      sh[0] = d;
      sh[1] = kk - acc;
    }
    __syncthreads();
    prefix |= (unsigned)sh[0] << sft;
    mask |= 255u << sft;
    kk = sh[1];
    __syncthreads();
  }
  return prefix;
}

// The estimate of channel ci in block blk, with NT threads and the window's energies in e[noise_window(d)].
template <int NT>
__device__ __forceinline__ void noise_body(NoiseArgs const &a, unsigned *e, int ci, int blk) {
  __shared__ unsigned hist[256];
  __shared__ int sh[4];
  __shared__ double red_s[NT / 32];
  __shared__ int red_c[NT / 32];
  __shared__ unsigned red_m[NT / 32];
  int const tid = threadIdx.x;
  ChanDesc const d = a.desc[ci];
  double *out = a.n0 + (long)blk * a.n0_stride + ci;
  if (d.plan < 0 || d.points <= 0) {
    if (tid == 0) *out = 0.0;
    return;
  }
  int const nbins = noise_window(d);
  int const shift = a.shift[ci], m = a.m_bins;
  float2 const *X = a.spec + (long)blk * a.spec_stride;
  int filled = nbins;
  if (!a.wrap) {  // radio.c:1805-1820
    int mbin = abs(shift) - nbins / 2;
    if (mbin < 0) mbin = 0;
    else if (mbin + nbins > m) mbin = m - nbins;
    if (nbins > m) {  // master smaller than the window: the reference would read out of bounds; use what exists
      mbin = 0;
      filled = m;
    }
    for (int i = tid; i < nbins; i += NT) {
      float v = 0.f;
      if (i < filled) {
        float2 const x = __ldg(X + mbin + i);
        v = x.x * x.x + x.y * x.y;
      }
      e[i] = __float_as_uint(v);
    }
  } else {  // radio.c:1821-1836
    int mbin = shift - nbins / 2;
    if (mbin < 0) mbin += m;
    else if (mbin >= m) mbin -= m;
    if (mbin < 0 || mbin >= m) {
      if (tid == 0) *out = 0.0;
      return;
    }
    // the reference stops filling when the walk reaches the master's Nyquist bin; what it leaves is zero here
    int const to_nyq = ((m / 2 - mbin) % m + m) % m;  // steps until mbin == m/2 (0 -> a full turn)
    filled = (to_nyq == 0 || to_nyq > nbins) ? nbins : to_nyq;
    for (int i = tid; i < nbins; i += NT) {
      float v = 0.f;
      if (i < filled) {
        int q = mbin + i;
        if (q >= m) q -= m;
        float2 const x = __ldg(X + q);
        v = x.x * x.x + x.y * x.y;
      }
      e[i] = __float_as_uint(v);
    }
  }
  __syncthreads();
  // quantile(energies, nbins, 0.10): pos = 0.1 (n-1), q1 = order statistic floor(pos), q2 the next one (radio.c:1761-1775)
  double const pos = 0.10 * (double)(nbins - 1);
  int const k = (int)floor(pos);
  double const frac = pos - (double)k;
  unsigned const b1 = radix_select<NT>(e, nbins, k, hist, sh);
  // the next order statistic: b1 again if enough duplicates, else the smallest element above it
  int cnt_le = 0;
  unsigned next = 0xffffffffu;
  for (int i = tid; i < nbins; i += NT) {
    unsigned const v = e[i];
    cnt_le += (v <= b1);
    if (v > b1 && v < next) next = v;
  }
  for (int o = 16; o > 0; o >>= 1) {
    cnt_le += __shfl_xor_sync(0xffffffffu, cnt_le, o);
    next = min(next, __shfl_xor_sync(0xffffffffu, next, o));
  }
  if ((tid & 31) == 0) {
    red_c[tid >> 5] = cnt_le;
    red_m[tid >> 5] = next;
  }
  __syncthreads();
  cnt_le = 0;
  next = 0xffffffffu;
  for (int w = 0; w < NT / 32; w++) {
    cnt_le += red_c[w];
    next = min(next, red_m[w]);
  }
  __syncthreads();
  double const q1 = (double)__uint_as_float(b1);
  double q = q1;
  if (frac != 0.0) {
    double const q2 = (cnt_le > k + 1 || next == 0xffffffffu) ? q1 : (double)__uint_as_float(next);
    q = q1 + frac * (q2 - q1);
  }
  double const en = 1.5 * q;  // N_cutoff, radio.c:74
  double sum = 0.0;
  int nb = 0;
  for (int i = tid; i < nbins; i += NT) {
    double const v = (double)__uint_as_float(e[i]);
    if (v <= en) {
      sum += v;
      nb++;
    }
  }
  for (int o = 16; o > 0; o >>= 1) {
    sum += __shfl_xor_sync(0xffffffffu, sum, o);
    nb += __shfl_xor_sync(0xffffffffu, nb, o);
  }
  if ((tid & 31) == 0) {
    red_s[tid >> 5] = sum;
    red_c[tid >> 5] = nb;
  }
  __syncthreads();
  if (tid == 0) {
    sum = 0.0;
    nb = 0;
    for (int w = 0; w < NT / 32; w++) {
      sum += red_s[w];
      nb += red_c[w];
    }
    *out = nb == 0 ? 0.0 : sum / (double)nb * a.scale;
  }
}

__global__ void __launch_bounds__(kNoiseThreads) noise_kernel(NoiseArgs const a) {
  extern __shared__ unsigned e[];  // [noise_window(d)]
  int const ci = blockIdx.x;
  ChanDesc const d = a.desc[ci];
  if (d.plan >= 0 && d.points > 0 && noise_window(d) > kNoiseSmemBins) return;  // noise_kernel_gm's
  noise_body<kNoiseThreads>(a, e, ci, blockIdx.y);
}

// grid (listed channels, blocks): channel list[blockIdx.x], its energies in scratch slot blockIdx.y * gridDim.x + blockIdx.x
// of `stride` words
__global__ void __launch_bounds__(kNoiseGmThreads) noise_kernel_gm(NoiseArgs const a, int const *list, unsigned *scratch, long stride) {
  noise_body<kNoiseGmThreads>(a, scratch + ((long)blockIdx.y * gridDim.x + blockIdx.x) * stride, list[blockIdx.x], blockIdx.y);
}

// ------------------------------------------------------------------ FM discriminator front half -----------------------
// Replaces the per-sample loops at the top of demod_fm (reference fm.c:104-131 and :205-231, plain discriminator): for every
// channel and block, baseband[n] = arg(y[n] conj y[n-1]) / pi with y[-1] carried over from the previous block, the mean
// amplitude and the sum of squared amplitude deviations (two passes, as the reference).  Reads the channel kernel's output
// rows in place; one CTA per (channel, block).
constexpr int kFmThreads = 128;
struct FmArgs {
  float2 const *out;   // channel outputs [block][out_pitch]
  long out_pitch;
  ChanDesc const *desc;
  int nblocks;
  float2 const *mem_in;  // [channel] last sample of the block before this launch (0 at start)
  float2 *mem_out;       // [channel] last sample of this launch's last block
  float *baseband;       // [block][bb_pitch], channel i's olen floats at 2 * desc[i].out_off (same packing as the outputs)
  long bb_pitch;
  double2 *stats;        // [block][stats_stride]: (.x mean amplitude, .y sum of squared deviations)
  long stats_stride;
};
__global__ void __launch_bounds__(kFmThreads) fm_front_kernel(FmArgs const a) {
  __shared__ double red[kFmThreads / 32];
  __shared__ double mean_sh;
  int const ci = blockIdx.x, blk = blockIdx.y, tid = threadIdx.x;
  ChanDesc const d = a.desc[ci];
  if (d.plan < 0 || (d.flags & kChanRealOut) || d.olen <= 0) {
    // the memory buffers alternate per launch: a skipped channel carries its y[-1] to the one the next launch reads
    if (tid == 0 && blk == a.nblocks - 1) a.mem_out[ci] = a.mem_in[ci];
    return;
  }
  float2 const *y = a.out + (long)blk * a.out_pitch + d.out_off;
  float2 const first_prev = blk > 0 ? a.out[(long)(blk - 1) * a.out_pitch + d.out_off + d.olen - 1] : a.mem_in[ci];
  float *bb = a.baseband + (long)blk * a.bb_pitch + 2 * d.out_off;
  double sum = 0;
  for (int n = tid; n < d.olen; n += kFmThreads) {
    float2 const v = y[n];
    float2 const p = n > 0 ? y[n - 1] : first_prev;
    double const re = (double)v.x * p.x + (double)v.y * p.y, im = (double)v.y * p.x - (double)v.x * p.y;  // v * conj(p)
    bb[n] = (float)(atan2(im, re) * 0.31830988618379067154);
    sum += (double)hypotf(v.x, v.y);
  }
  auto block_sum = [&](double v) -> double {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    __syncthreads();
    if ((tid & 31) == 0) red[tid >> 5] = v;
    __syncthreads();
    double t = 0;
    for (int w = 0; w < kFmThreads / 32; w++) t += red[w];
    return t;
  };
  double const mean = block_sum(sum) / (double)d.olen;
  double dev = 0;
  for (int n = tid; n < d.olen; n += kFmThreads) {
    float2 const v = y[n];
    double const e = (double)hypotf(v.x, v.y) - mean;
    dev += e * e;
  }
  dev = block_sum(dev);
  if (tid == 0) {
    a.stats[(long)blk * a.stats_stride + ci] = make_double2(mean, dev);
    if (blk == a.nblocks - 1) a.mem_out[ci] = y[d.olen - 1];
  }
  (void)mean_sh;
}

}  // namespace kfft
