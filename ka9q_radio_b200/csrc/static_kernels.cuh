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
// What chan_static and chan_v2 share: one warp per (channel, block); the warp's column holds the staged response (then
// the slice) in col[NS] and the staged master bins in xs[XS]; the plan's twiddles follow the kChanWarps columns.
// `order` lists the descriptors that share this plan (mixed output rates are launched per plan).
template <class P>
struct StaticChan {
  static constexpr int NS = P::len, TOP = (NS + 1) / 2;
  static_assert(NS % 2 == 0, "bulk copies need 16-byte multiples");
  static constexpr int XS = NS + 4;  // staged slice: up to NS bins + alignment slack
  static constexpr uint32_t TWB = (uint32_t)((static_tw_count<P>() + 1) & ~1) * 8u;
  static constexpr size_t smem = sizeof(float2) * ((size_t)(NS + XS) * kChanWarps + static_tw_count<P>() + 2);
  ChanDesc d;
  int lane, oi, blk;
  float2 *col, *xs, *s_tw, *dst;
  int qa;      // master bin of xs[0] (bulk copies start at an even bin)
  bool wraps;  // a COMPLEX master wraps inside the slice: xs holds walk positions 0 .. ncopy-1 instead
  // S[w] = X[q(w)] * R[w] from the staged copies, zero outside the master (filter.c:728-911)
  __device__ __forceinline__ float2 product(int w) const {
    bool live;
    int const u = walk_pos(d, NS, TOP, w, live);
    float2 const v = slice_product(d, xs[live ? (wraps ? u : d.q0 + d.dir * u - qa) : 0], col[w]);
    return live ? v : make_float2(0.f, 0.f);
  }
};

// The prologue of chan_static and chan_v2.  Thread 0 issues the CTA's twiddle bulk copy into s_tw (tbar; every
// descriptor of the launch shares the plan) when some warp of the CTA has a runnable descriptor.  Each warp then stages
// its slice: one pair of bulk copies (bars[warp]), or plain loads when a COMPLEX master wraps.  A channel with no overlap
// at all gets its zero output here.  Returns false when the warp has nothing more to do.  Every warp with a runnable
// descriptor waits on tbar before it retires (here for a zero channel, in the kernel otherwise), so no CTA can retire
// with its twiddle copy still in flight.
template <class P>
__device__ __forceinline__ bool static_prologue(ChanArgs const &a, uint64_t *bars, uint64_t &tbar, StaticChan<P> &s) {
  using S = StaticChan<P>;
  constexpr int NS = S::NS;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  int const lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int const oi = blockIdx.x * kChanWarps + warp;
  float2 *s_tw = reinterpret_cast<float2 *>(smem_raw) + kChanWarps * (NS + S::XS);
  bool const active = oi < a.norder;
  ChanDesc d;
  d.plan = -1;
  if (active) d = a.desc[chan_index(a, oi)];
  if (threadIdx.x == 0) {
    int p0 = -1;
    for (int w = 0; w < kChanWarps && p0 < 0; w++) {
      int const o = blockIdx.x * kChanWarps + w;
      if (o < a.norder) p0 = a.desc[chan_index(a, o)].plan;
    }
    mbar_init(&tbar, 1);
    mbar_fence_init();
    if (p0 >= 0) {
      mbar_expect_tx(&tbar, S::TWB);
      bulk_g2s(s_tw, c_plans[p0].tw, S::TWB, &tbar);
    }
  }
  __syncthreads();
  if (!active || d.plan < 0) return false;
  int const blk = blockIdx.y;
  float2 *col = reinterpret_cast<float2 *>(smem_raw) + warp * (NS + S::XS);
  float2 *xs = col + NS;
  float2 const *X = a.spec + (long)blk * a.spec_stride;
  float2 const *R = a.resp + d.resp_off;
  float2 *dst = a.out + (long)blk * a.out_stride + d.out_off;
  if (d.ncopy <= 0) {  // nothing of this channel overlaps the master spectrum: zeros (filter.c:823-832)
    for (int i = lane; i < d.olen; i += 32) dst[i] = make_float2(0.f, 0.f);
    if ((d.flags & kChanOsc) && a.power && lane == 0) a.power[(long)blk * a.power_stride + chan_index(a, oi)] = 0.f;
    mbar_wait(&tbar, 0);
    return false;
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
  s.d = d;
  s.lane = lane;
  s.oi = oi;
  s.blk = blk;
  s.col = col;
  s.xs = xs;
  s.s_tw = s_tw;
  s.dst = dst;
  s.qa = qa;
  s.wraps = wraps;
  return true;
}

// chan_static: the 1200-point and other three-stage plans (the 600 / 300-point channels use chan_v2)
template <class P>
__global__ void __launch_bounds__(kChanWarps * 32) chan_static(ChanArgs const a) {
  __shared__ __align__(8) uint64_t bars[kChanWarps];
  __shared__ __align__(8) uint64_t tbar;
  using S = StaticChan<P>;
  S s;
  if (!static_prologue<P>(a, bars, tbar, s)) return;
  ChanDesc const &d = s.d;
  float2 *col = s.col;
  int const lane = s.lane;
  // the product in place over the staged response
#pragma unroll 4
  for (int wp = lane; wp < S::NS; wp += 32) col[wp] = s.product(wp);
  __syncwarp();
  if (d.flags & kChanIsb) isb_fold_warp(col, S::NS, S::TOP, lane);
  mbar_wait(&tbar, 0);
  StaticFft<P, true, true>::run(col, s.s_tw, lane);
  int const first = S::NS - d.olen;
  if (d.flags & kChanOsc) {  // fine-tuning rotation + block power (radio.c:1476-1501, :1515-1520)
    int const ci = chan_index(a, s.oi);
    ChanAux const ax = a.aux[ci];
    long const k = a.block0 + s.blk - ax.osc_epoch;
    float pw = 0.f;
    for (int i = lane; i < d.olen; i += 32) s.dst[i] = osc_sample(ax, k, d.olen, i, col[static_slot<P>(first + i)], pw);
    pw = warp_sum(pw);
    if (a.power && lane == 0) a.power[(long)s.blk * a.power_stride + ci] = pw / (float)d.olen;
    return;
  }
#pragma unroll 4
  for (int i = lane; i < d.olen; i += 32) s.dst[i] = col[static_slot<P>(first + i)];
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
