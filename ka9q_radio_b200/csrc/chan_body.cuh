// chan_body.cuh -- the body of the generic channel kernel, included by chan_kernels.cuh into chan_kernel (registry
// plan c_plans[d.plan], KFFT_CHAN_EXT false) and chan_kernel_ext (a length with a prime factor 11 .. 23, its plan `xpl`
// by value, KFFT_CHAN_EXT true: tile_fft also dispatches the extended radices).  Not a header of its own: it expects
// `a` (ChanArgs) in scope.  Written out in each kernel rather than called as an inline function because that keeps
// chan_kernel's machine code exactly what it was before the extended kernel existed (as a call, the compiler
// allocates the registers of the store loops differently).  The per-channel steps are chan_slice.cuh's.
  extern __shared__ __align__(16) unsigned char smem_raw[];
  int const lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int const oi = blockIdx.x * kChanWarps + warp;
  if (oi >= a.norder) return;
  ChanDesc const d = a.desc[chan_index(a, oi)];
  if (d.plan < 0) return;
  int const blk = blockIdx.y;
  float2 *col = reinterpret_cast<float2 *>(smem_raw) + warp * a.pitch;
#if KFFT_CHAN_EXT
  TilePlan const &pl = xpl;
#else
  TilePlan const &pl = c_plans[d.plan];
#endif
  int const ns = d.points;
  int const top = (ns + 1) / 2;  // index of the most negative output bin == Nyquist slot

  float2 const *X = a.spec + (long)blk * a.spec_stride;
  float2 const *R = a.resp + d.resp_off;
  int const ci = chan_index(a, oi);
  if (d.flags & kChanRealOut) {
    for (int si = lane; si < ns / 2 + 1; si += 32) {
      float2 const v = real_half(a, d, X, R, si);
      if (si == 0 || 2 * si == ns) {
        col[si] = make_float2(v.x, 0.f);
      } else {
        col[si] = v;
        col[ns - si] = make_float2(v.x, -v.y);
      }
    }
  } else if (d.flags & kChanBeam) {
    ChanAux const ax = a.aux[ci];
    for (int wq = lane; wq < ns; wq += 32) {
      bool live;
      int const u = walk_pos(d, ns, top, wq, live);
      float2 const v = beam_product(ax, X, a.m_bins, live ? walk_bin(a, d, u) : 0, __ldg(R + wq));
      col[wq] = live ? v : make_float2(0.f, 0.f);
    }
  } else {
    constexpr int U = 4;  // four gathers in flight
    int wp = lane;
    for (; wp + (U - 1) * 32 < ns; wp += U * 32) {
      float2 x[U], rr[U];
      bool live[U];
#pragma unroll
      for (int k = 0; k < U; k++) {
        int const u = walk_pos(d, ns, top, wp + k * 32, live[k]);
        x[k] = __ldg(X + (live[k] ? walk_bin(a, d, u) : 0));
        rr[k] = __ldg(R + wp + k * 32);
      }
#pragma unroll
      for (int k = 0; k < U; k++) {
        float2 const v = slice_product(d, x[k], rr[k]);
        col[wp + k * 32] = live[k] ? v : make_float2(0.f, 0.f);
      }
    }
    for (; wp < ns; wp += 32) {
      bool live;
      int const u = walk_pos(d, ns, top, wp, live);
      float2 const v = slice_product(d, __ldg(X + (live ? walk_bin(a, d, u) : 0)), __ldg(R + wp));
      col[wp] = live ? v : make_float2(0.f, 0.f);
    }
  }
  __syncwarp();
  if (d.flags & kChanIsb) isb_fold_warp(col, ns, top, lane);
  tile_fft<true, KFFT_CHAN_EXT>(pl, col, lane, 32, [] { __syncwarp(); });
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
    for (int i = lane; i < d.olen; i += 32) dst[i] = osc_sample(ax, k, d.olen, i, col[__ldg(pl.perm + first + i)], pw);
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
