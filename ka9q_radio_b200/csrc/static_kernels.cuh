// static_kernels.cuh -- shared pieces of the compile-time specialised kernels (fft_static.cuh) and the v1 channel kernel
// (chan_static: 1200-point and other three-stage plans; the 600 / 300-point channels use chan_v2).  Same arithmetic, same
// tables and the same argument structs as the generic kernels in fwd_kernels.cuh / chan_kernels.cuh, so parity
// tests cover both; what changes is everything around the butterflies:
//   * literal strides / trip counts, unrolled stage loops, arithmetic digit reversal
//   * rows and channel inputs arrive by TMA bulk copies (cp.async.bulk -> mbarrier) straight into
//     shared memory: no register staging, whole rows / slices in flight at once
//   * inter-pass twiddles come from small precomputed tables instead of double-precision sincospi
#pragma once
#include "chan_kernels.cuh"
#include "fft_static.cuh"
#include "fwd_kernels.cuh"

namespace kfft {

struct FwdTables {
  float2 const *rootC;  // [n1/2+1]   W_{2nc}^{k1}   (REAL split only)
};

// ------------------------------------------------------------------ channels ------------------
// `order` lists the descriptors that share this plan (mixed output rates are launched per plan).
template <class P>
__global__ void __launch_bounds__(kChanWarps * 32) chan_static(ChanArgs const a) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  __shared__ __align__(8) uint64_t bars[kChanWarps];
  constexpr int NS = P::len, TOP = (NS + 1) / 2;
  static_assert(NS % 2 == 0, "bulk copies need 16-byte multiples");
  constexpr int XS = NS + 4;  // staged slice: up to NS bins + alignment slack
  int const lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int const oi = blockIdx.x * kChanWarps + warp;
  float2 *s_tw = reinterpret_cast<float2 *>(smem_raw) + kChanWarps * (NS + XS);
  bool const active = oi < a.norder;
  ChanDesc d;
  d.plan = -1;
  if (active) d = a.desc[a.order ? a.order[oi] : a.chan_base + oi];
  // stage twiddles of this plan: one TMA bulk copy per CTA (every descriptor of the launch shares the plan)
  __shared__ __align__(8) uint64_t tbar;
  __shared__ int plan_sh;
  if (threadIdx.x == 0) {
    int p0 = -1;
    for (int w = 0; w < kChanWarps && p0 < 0; w++) {
      int const o = blockIdx.x * kChanWarps + w;
      if (o < a.norder) p0 = a.desc[a.order ? a.order[o] : a.chan_base + o].plan;
    }
    plan_sh = p0;
    mbar_init(&tbar, 1);
    mbar_fence_init();
    if (p0 >= 0) {
      constexpr uint32_t TWB = (uint32_t)((static_tw_count<P>() + 1) & ~1) * 8u;
      mbar_expect_tx(&tbar, TWB);
      bulk_g2s(s_tw, c_plans[p0].tw, TWB, &tbar);
    }
  }
  __syncthreads();
  if (!active || d.plan < 0) return;
  int const blk = blockIdx.y;
  float2 *col = reinterpret_cast<float2 *>(smem_raw) + warp * (NS + XS);
  float2 *xs = col + NS;
  float2 const *X = a.spec + (long)blk * a.spec_stride;
  float2 const *R = a.resp + d.resp_off;
  float2 *dst = a.out + (long)blk * a.out_stride + d.out_off;

  if (d.ncopy <= 0) {  // nothing of this channel overlaps the master spectrum: zeros (filter.c:823-832)
    for (int i = lane; i < d.olen; i += 32) dst[i] = make_float2(0.f, 0.f);
    if ((d.flags & kChanOsc) && a.power && lane == 0) a.power[(long)blk * a.power_stride + (a.order ? a.order[oi] : a.chan_base + oi)] = 0.f;
    mbar_wait(&tbar, 0);  // never retire the CTA with its twiddle copy still in flight
    return;
  }
  int const qlo = d.dir > 0 ? d.q0 : d.q0 - (d.ncopy - 1);
  bool const wraps = a.wrap && (d.q0 + d.ncopy > a.m_bins);
  int const qa = qlo & ~1;
  if (!wraps) {
    int const qhi = qlo + d.ncopy - 1;
    uint32_t const nx = (uint32_t)(((qhi - qa + 1) + 1) & ~1);
    if (lane == 0) {
      mbar_init(&bars[warp], 1);
      mbar_fence_init();
      mbar_expect_tx(&bars[warp], nx * 8 + NS * 8);
      bulk_g2s(xs, X + qa, nx * 8, &bars[warp]);
      bulk_g2s(col, R, NS * 8, &bars[warp]);
    }
    __syncwarp();
    mbar_wait(&bars[warp], 0);
  } else {  // circular wrap of a COMPLEX master (filter.c:771-772): two pieces, plain loads
    for (int i = lane; i < NS; i += 32) col[i] = __ldg(R + i);
    for (int u = lane; u < d.ncopy; u += 32) {
      int q = d.q0 + u;
      if (q >= a.m_bins) q -= a.m_bins;
      xs[u] = __ldg(X + q);
    }
    __syncwarp();
  }
  // S[wp] = X[q(wp)] * R[wp] in place over the staged response
#pragma unroll 4
  for (int wp = lane; wp < NS; wp += 32) {
    int t = wp - TOP;
    if (t < 0) t += NS;
    int const u = t - d.zlead;
    bool const live = (u >= 0 && u < d.ncopy && wp != TOP);
    int const xi = wraps ? u : (d.q0 + d.dir * u - qa);
    float2 x = xs[live ? xi : 0];
    if (d.dir < 0) x.y = -x.y;
    float2 const v = cmul(x, col[wp]);
    col[wp] = live ? v : make_float2(0.f, 0.f);
  }
  __syncwarp();
  if (d.flags & kChanIsb) {
    for (int p = 1 + lane; p < NS / 2; p += 32) {
      float2 const pos = col[p], neg = col[NS - p];
      col[p] = make_float2(pos.x + neg.x, pos.y - neg.y);
      col[NS - p] = make_float2(neg.x - pos.x, neg.y + pos.y);
    }
    if (lane == 0) {
      col[0] = make_float2(0.f, 0.f);
      col[TOP] = make_float2(0.f, 0.f);
    }
    __syncwarp();
  }
  mbar_wait(&tbar, 0);
  StaticFft<P, true, true>::run(col, s_tw, lane);
  int const first = NS - d.olen;
  if (d.flags & kChanOsc) {  // fine-tuning rotation + block power (radio.c:1476-1501, :1515-1520)
    int const ci = a.order ? a.order[oi] : a.chan_base + oi;
    ChanAux const ax = a.aux[ci];
    long const k = a.block0 + blk - ax.osc_epoch;
    float pw = 0.f;
    for (int i = lane; i < d.olen; i += 32) {
      float2 const v = osc_rotate(col[static_slot<P>(first + i)], osc_phase_cycles(ax, k, d.olen, i));
      dst[i] = v;
      pw += v.x * v.x + v.y * v.y;
    }
    pw = warp_sum(pw);
    if (a.power && lane == 0) a.power[(long)blk * a.power_stride + ci] = pw / (float)d.olen;
    return;
  }
#pragma unroll 4
  for (int i = lane; i < d.olen; i += 32) dst[i] = col[static_slot<P>(first + i)];
}

// does the registry plan have exactly the radices of static plan P?
template <class P> inline bool plan_is(TilePlan const *p) {
  if (p->len != P::len || p->nstages != P::nst) return false;
  for (int i = 0; i < P::nst; i++)
    if (p->radix[i] != P::rad(i)) return false;
  return true;
}

using S600 = SPlan<600, 24, 25>;
using S300 = SPlan<300, 20, 15>;
using S1200 = SPlan<1200, 12, 10, 10>;

}  // namespace kfft
