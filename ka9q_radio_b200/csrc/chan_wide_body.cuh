// chan_wide_body.cuh -- the body of the wide channel kernel, included by chan_wide.cuh into chan_wide (registry plans,
// KFFT_WIDE_EXT false) and chan_wide_ext (an extended length, KFFT_WIDE_EXT true: its plans by value, and wide_fft also
// dispatches the extended radices).  Not a header of its own: it expects `a` (ChanArgs) and `g` (WideGeom) in scope,
// and with KFFT_WIDE_EXT `x` (WideGeomExt, x.g is g).  Written out in each kernel rather than called as an inline
// function because that keeps chan_wide's machine code exactly what it was before the extended kernel existed.
  extern __shared__ __align__(16) unsigned char smem_raw[];
  __shared__ float red[kWideThreads / 32];
  int const oi = blockIdx.x;
  int const ci = a.order ? a.order[oi] : a.chan_base + oi;
  ChanDesc const d = a.desc[ci];
  if (d.plan < 0) return;
  int const blk = blockIdx.y, tid = threadIdx.x, nt = blockDim.x;
  float2 *col = reinterpret_cast<float2 *>(smem_raw);
  int const ns = d.points;
  int const top = (ns + 1) / 2;  // index of the most negative output bin == Nyquist slot

  float2 const *X = a.spec + (long)blk * a.spec_stride;
  float2 const *R = a.resp + d.resp_off;
  auto src_of = [&](int wp, bool &live) -> int {  // chan_kernel's walk
    int t = wp - top;
    if (t < 0) t += ns;
    int const u = t - d.zlead;
    live = (u >= 0 && u < d.ncopy && wp != top);  // Nyquist slot is forced to zero (filter.c:911)
    int q = d.q0 + d.dir * u;
    if (a.wrap && q >= a.m_bins) q -= a.m_bins;
    return live ? q : 0;
  };
  if (d.flags & kChanRealOut) {
    // REAL-output slave (filter.c:794-809), as chan_kernel: half spectrum, zero at (sb+1)/2, Hermitian extension
    int const shift = d.q0, sb = ns / 2 + 1, zero_at = (sb + 1) / 2, m = a.m_bins;
    for (int si = tid; si < sb; si += nt) {
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
        col[wide_in_slot(g, si)] = make_float2(v.x, 0.f);
      } else {
        col[wide_in_slot(g, si)] = v;
        col[wide_in_slot(g, ns - si)] = make_float2(v.x, -v.y);
      }
    }
  } else if (d.flags & kChanBeam) {
    // filter.c:756-775 in double complex, rounded to float once (as chan_kernel)
    ChanAux const ax = a.aux[ci];
    int const m = a.m_bins;
    for (int wq = tid; wq < ns; wq += nt) {
      bool live;
      int const q = src_of(wq, live);
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
      col[wide_in_slot(g, wq)] = live ? v : make_float2(0.f, 0.f);
    }
  } else {
    bool const cj = d.dir < 0;  // inverted REAL spectrum => conjugate (filter.c:876)
    for (int wp = tid; wp < ns; wp += nt) {
      bool live;
      int const q = src_of(wp, live);
      float2 x = __ldg(X + q);
      if (cj) x.y = -x.y;
      float2 const v = cmul(x, __ldg(R + wp));
      col[wide_in_slot(g, wp)] = live ? v : make_float2(0.f, 0.f);
    }
  }
  __syncthreads();
  if (d.flags & kChanIsb) {  // filter.c:895-909, pairs p with ns-p: only after the whole slice is in place
    for (int p = 1 + tid; p < ns / 2; p += nt) {
      int const sp = wide_in_slot(g, p), sn = wide_in_slot(g, ns - p);
      float2 const pos = col[sp], neg = col[sn];
      col[sp] = make_float2(pos.x + neg.x, pos.y - neg.y);
      col[sn] = make_float2(neg.x - pos.x, neg.y + pos.y);
    }
    if (tid == 0) {
      col[wide_in_slot(g, 0)] = make_float2(0.f, 0.f);
      col[wide_in_slot(g, top)] = make_float2(0.f, 0.f);
    }
    __syncthreads();
  }
#if KFFT_WIDE_EXT
  wide_transform<true, true>(g, col, &x);
  uint16_t const *perm1 = x.p1.perm, *perm2 = x.p2.perm;
#else
  wide_transform<true>(g, col);
  uint16_t const *perm1 = c_plans[g.plan1].perm, *perm2 = c_plans[g.plan2].perm;
#endif
  float2 *dst = a.out + (long)blk * a.out_stride + d.out_off;
  int const first = ns - d.olen;
  if (d.flags & kChanRealOut) {  // c2r: the real part, olen floats packed in the channel's float2 run
    float *dr = reinterpret_cast<float *>(dst);
    for (int i = tid; i < d.olen; i += nt) dr[i] = col[wide_out_slot(g, perm1, perm2, first + i)].x;
    return;
  }
  if (d.flags & kChanOsc) {
    ChanAux const ax = a.aux[ci];
    long const k = a.block0 + blk - ax.osc_epoch;
    float pw = 0.f;
    for (int i = tid; i < d.olen; i += nt) {
      float2 const v = osc_rotate(col[wide_out_slot(g, perm1, perm2, first + i)], osc_phase_cycles(ax, k, d.olen, i));
      dst[i] = v;
      pw += v.x * v.x + v.y * v.y;
    }
    pw = warp_sum(pw);
    if ((tid & 31) == 0) red[tid >> 5] = pw;
    __syncthreads();
    if (a.power && tid == 0) {
      float s = 0.f;
      for (int w = 0; w < nt / 32; w++) s += red[w];
      a.power[(long)blk * a.power_stride + ci] = s / (float)d.olen;
    }
    return;
  }
  for (int i = tid; i < d.olen; i += nt) dst[i] = col[wide_out_slot(g, perm1, perm2, first + i)];
