// chan_body.cuh -- the body of the generic channel kernel, included by chan_kernels.cuh into chan_kernel (registry
// plan c_plans[d.plan], KFFT_CHAN_EXT false) and chan_kernel_ext (a length with a prime factor 11 .. 23, its plan `xpl`
// by value, KFFT_CHAN_EXT true: tile_fft also dispatches the extended radices).  Not a header of its own: it expects
// `a` (ChanArgs) in scope.  Written out in each kernel rather than called as an inline function because that keeps
// chan_kernel's machine code exactly what it was before the extended kernel existed (as a call, the compiler
// allocates the registers of the store loops differently).
  extern __shared__ __align__(16) unsigned char smem_raw[];
  int const lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int const oi = blockIdx.x * kChanWarps + warp;
  if (oi >= a.norder) return;
  ChanDesc const d = a.desc[a.order ? a.order[oi] : a.chan_base + oi];
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
