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
  int plan;        // registry index of the length-`points` inverse plan, < 0: channel disabled
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

__global__ void __launch_bounds__(kChanWarps * 32) chan_kernel(ChanArgs const a) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  int const lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int const oi = blockIdx.x * kChanWarps + warp;
  if (oi >= a.norder) return;
  ChanDesc const d = a.desc[a.order ? a.order[oi] : a.chan_base + oi];
  if (d.plan < 0) return;
  int const blk = blockIdx.y;
  float2 *col = reinterpret_cast<float2 *>(smem_raw) + warp * a.pitch;
  TilePlan const &pl = c_plans[d.plan];
  int const ns = d.points;
  int const top = (ns + 1) / 2;  // index of the most negative output bin == Nyquist slot

  float2 const *X = a.spec + (long)blk * a.spec_stride;
  float2 const *R = a.resp + d.resp_off;
  auto src_of = [&](int wp, bool &live, bool &cj) -> int {
    int t = wp - top;
    if (t < 0) t += ns;
    int const u = t - d.zlead;
    live = (u >= 0 && u < d.ncopy && wp != top);  // Nyquist slot is forced to zero (filter.c:911)
    cj = d.dir < 0;
    int q = d.q0 + d.dir * u;
    if (a.wrap && q >= a.m_bins) q -= a.m_bins;
    return live ? q : 0;
  };
  int const ci = a.order ? a.order[oi] : a.chan_base + oi;
  if (d.flags & kChanRealOut) {
    // REAL-output slave (filter.c:794-809): bins 0..ns/2 of the slave = master bins si + shift, then the Hermitian
    // extension the c2r inverse implies (FFTW ignores the imaginary parts of DC and Nyquist).  The reference's
    // "Nyquist zero" (filter.c:911) lands on index (s_bins+1)/2 of the HALF spectrum; so does ours.
    int const shift = d.q0, sb = ns / 2 + 1, zero_at = (sb + 1) / 2, m = a.m_bins;
    for (int si = lane; si < sb; si += 32) {
      int const mi = si + shift;
      float2 v = make_float2(0.f, 0.f);
      if (!a.wrap) {
        if (mi >= 0 && mi < m) v = cmul(__ldg(X + mi), __ldg(R + si));
      } else if (mi >= -(m / 2) && mi < m / 2) {
        int q1 = mi % m, q2 = (m - mi) % m;
        if (q1 < 0) q1 += m;
        if (q2 < 0) q2 += m;
        float2 const xa = __ldg(X + q1), xb = __ldg(X + q2);
        v = cmul(__ldg(R + si), make_float2(xa.x + xb.x, xa.y - xb.y));
      }
      if (si == zero_at) v = make_float2(0.f, 0.f);
      if (si == 0 || 2 * si == ns) {
        col[si] = make_float2(v.x, 0.f);
      } else {
        col[si] = v;
        col[ns - si] = make_float2(v.x, -v.y);
      }
    }
  } else if (d.flags & kChanBeam) {
    // filter.c:756-775: alpha X[q] + beta conj(X[m-q]) (at q = 0 or m/2: Re(X) alpha + Im(X) beta), times the response,
    // in double complex as the reference's mixed float/double expression evaluates, rounded to float once
    ChanAux const ax = a.aux[ci];
    int const m = a.m_bins;
    for (int wq = lane; wq < ns; wq += 32) {
      bool live, cj;
      int const q = src_of(wq, live, cj);
      float2 const r = __ldg(R + wq);
      float2 const x = __ldg(X + q);
      double sr, si_;
      if (q == 0 || q == m / 2) {
        sr = (double)x.x * ax.are + (double)x.y * ax.bre;
        si_ = (double)x.x * ax.aim + (double)x.y * ax.bim;
      } else {
        float2 const y = __ldg(X + (m - q));
        sr = ax.are * x.x - ax.aim * x.y + ax.bre * y.x + ax.bim * y.y;
        si_ = ax.are * x.y + ax.aim * x.x - ax.bre * y.y + ax.bim * y.x;
      }
      float2 const v = make_float2((float)(sr * r.x - si_ * r.y), (float)(sr * r.y + si_ * r.x));
      col[wq] = live ? v : make_float2(0.f, 0.f);
    }
  } else {
    constexpr int U = 4;
    int wp = lane;
    for (; wp + (U - 1) * 32 < ns; wp += U * 32) {
      float2 x[U], rr[U];
      bool live[U], cj[U];
#pragma unroll
      for (int u = 0; u < U; u++) {
        int const q = src_of(wp + u * 32, live[u], cj[u]);
        x[u] = __ldg(X + q);
        rr[u] = __ldg(R + wp + u * 32);
      }
#pragma unroll
      for (int u = 0; u < U; u++) {
        if (cj[u]) x[u].y = -x[u].y;
        float2 const v = cmul(x[u], rr[u]);
        col[wp + u * 32] = live[u] ? v : make_float2(0.f, 0.f);
      }
    }
    for (; wp < ns; wp += 32) {
      bool live, cj;
      int const q = src_of(wp, live, cj);
      float2 x = __ldg(X + q);
      if (cj) x.y = -x.y;
      float2 const v = cmul(x, __ldg(R + wp));
      col[wp] = live ? v : make_float2(0.f, 0.f);
    }
  }
  __syncwarp();
  if (d.flags & kChanIsb) {  // ISB: (S[p], S[ns-p]) <- (S[p]+conj S[ns-p], S[ns-p]-conj S[p]); S[0]=0
    for (int p = 1 + lane; p < ns / 2; p += 32) {
      float2 const pos = col[p], neg = col[ns - p];
      col[p] = make_float2(pos.x + neg.x, pos.y - neg.y);
      col[ns - p] = make_float2(neg.x - pos.x, neg.y + pos.y);
    }
    if (lane == 0) {
      col[0] = make_float2(0.f, 0.f);
      col[top] = make_float2(0.f, 0.f);
    }
    __syncwarp();
  }
  tile_fft<true>(pl, col, lane, 32, [] { __syncwarp(); });
  float2 *dst = a.out + (long)blk * a.out_stride + d.out_off;
  int const first = ns - d.olen;
  if (d.flags & kChanRealOut) {  // the c2r result is the real part; olen floats, packed in the channel's float2 run
    float *dr = reinterpret_cast<float *>(dst);
    for (int i = lane; i < d.olen; i += 32) dr[i] = col[__ldg(pl.perm + first + i)].x;
    return;
  }
  if (d.flags & kChanOsc) {
    ChanAux const ax = a.aux[ci];
    long const k = a.block0 + blk - ax.osc_epoch;
    float pw = 0.f;
    for (int i = lane; i < d.olen; i += 32) {
      float2 const v = osc_rotate(col[__ldg(pl.perm + first + i)], osc_phase_cycles(ax, k, d.olen, i));
      dst[i] = v;
      pw += v.x * v.x + v.y * v.y;
    }
    pw = warp_sum(pw);
    if (a.power && lane == 0) a.power[(long)blk * a.power_stride + ci] = pw / (float)d.olen;
    return;
  }
  {
    constexpr int V = 4;
    int i = lane;
    for (; i + (V - 1) * 32 < d.olen; i += V * 32) {
      int slot[V];
      float2 v[V];
#pragma unroll
      for (int u = 0; u < V; u++) slot[u] = __ldg(pl.perm + first + i + u * 32);
#pragma unroll
      for (int u = 0; u < V; u++) v[u] = col[slot[u]];
#pragma unroll
      for (int u = 0; u < V; u++) dst[i + u * 32] = v[u];
    }
    for (; i < d.olen; i += 32) dst[i] = col[__ldg(pl.perm + first + i)];
  }
}

// Forward transform of one response in place (set_filter's fftwf_execute, filter.c:1030):
// one warp, data staged through shared memory.
__global__ void __launch_bounds__(32) response_fft_kernel(float2 *resp, int plan) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  float2 *col = reinterpret_cast<float2 *>(smem_raw);
  TilePlan const &pl = c_plans[plan];
  int const lane = threadIdx.x;
  for (int i = lane; i < pl.len; i += 32) col[i] = resp[i];
  __syncwarp();
  tile_fft<false>(pl, col, lane, 32, [] { __syncwarp(); });
  for (int k = lane; k < pl.len; k += 32) resp[k] = col[pl.perm[k]];
}

}  // namespace kfft
