// chan_slice.cuh -- the per-channel steps of execute_filter_output (reference filter.c:728-921) and of the channel's
// output (radio.c:1476-1520), stated once for every channel kernel.  Each helper computes one element, index or value;
// the loops, the tiling and the mapping of slice slots onto shared memory stay in the kernels.  Included by
// chan_kernels.cuh after ChanDesc, ChanAux and ChanArgs.
#pragma once

namespace kfft {

// Descriptor index of launch item oi: the launch's own list of descriptors, or the run chan_base, chan_base + 1, ...
__device__ __forceinline__ int chan_index(ChanArgs const &a, int oi) { return a.order ? a.order[oi] : a.chan_base + oi; }

// The walk (filter.c:728-893): slot w of an ns-point slice is walk position u = ((w - top) mod ns) - zlead, counted from
// the most negative output bin; top = (ns + 1) / 2.  The slot takes a master bin when 0 <= u < ncopy, except the
// Nyquist slot top, which filter.c:911 zeroes.
__device__ __forceinline__ int walk_pos(ChanDesc const &d, int ns, int top, int w, bool &live) {
  int t = w - top;
  if (t < 0) t += ns;
  int const u = t - d.zlead;
  live = (u >= 0 && u < d.ncopy && w != top);
  return u;
}

// Master bin of walk position u, wrapping around a COMPLEX master (filter.c:771-772).
__device__ __forceinline__ int walk_bin(ChanArgs const &a, ChanDesc const &d, int u) {
  int q = d.q0 + d.dir * u;
  if (a.wrap && q >= a.m_bins) q -= a.m_bins;
  return q;
}

// Master bin x times response r; a walk down an inverted REAL spectrum takes the conjugate (filter.c:876).
__device__ __forceinline__ float2 slice_product(ChanDesc const &d, float2 x, float2 r) {
  if (d.dir < 0) x.y = -x.y;
  return cmul(x, r);
}

// Beam synthesis at master bin q of the m-bin COMPLEX spectrum X, times response r (filter.c:756-775):
// alpha X[q] + beta conj(X[m-q]), at q = 0 or m/2 Re(X) alpha + Im(X) beta, in double complex as the reference's mixed
// float/double expression evaluates, rounded to float once.
__device__ __forceinline__ float2 beam_product(ChanAux const &ax, float2 const *X, int m, int q, float2 r) {
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
  return make_float2((float)(sr * r.x - si_ * r.y), (float)(sr * r.y + si_ * r.x));
}

// REAL-output slave (filter.c:794-809): element si (0 <= si <= ns/2) of the half spectrum is master bin si + shift
// (d.q0) times the response.  The c2r inverse implies the Hermitian extension: slot si takes it (with the imaginary part
// dropped at si = 0 and 2 si = ns, as FFTW ignores it), slot ns - si its conjugate.  The reference's "Nyquist zero"
// (filter.c:911) lands on index (sb+1)/2 of the HALF spectrum; so does ours.  x(q) loads master bin q.
template <class LoadX>
__device__ __forceinline__ float2 real_half_at(ChanArgs const &a, ChanDesc const &d, LoadX x, float2 const *R, int si) {
  int const sb = d.points / 2 + 1, m = a.m_bins, mi = si + d.q0;
  float2 v = make_float2(0.f, 0.f);
  if (!a.wrap) {
    if (mi >= 0 && mi < m) v = cmul(x(mi), __ldg(R + si));
  } else if (mi >= -(m / 2) && mi < m / 2) {
    int q1 = mi % m, q2 = (m - mi) % m;
    if (q1 < 0) q1 += m;
    if (q2 < 0) q2 += m;
    float2 const xa = x(q1), xb = x(q2);
    v = cmul(__ldg(R + si), make_float2(xa.x + xb.x, xa.y - xb.y));
  }
  if (si == (sb + 1) / 2) v = make_float2(0.f, 0.f);
  return v;
}
// The same from a spectrum no kernel of the launch writes (read-only loads).
__device__ __forceinline__ float2 real_half(ChanArgs const &a, ChanDesc const &d, float2 const *X, float2 const *R, int si) {
  return real_half_at(a, d, [X](int q) { return __ldg(X + q); }, R, si);
}

// ISB (filter.c:895-909), for 0 < p < ns/2: (S[p], S[ns-p]) <- (S[p] + conj S[ns-p], S[ns-p] - conj S[p]).  The
// kernels also zero S[0] and S[top].
__device__ __forceinline__ void isb_fold(float2 &pos, float2 &neg) {
  float2 const p = pos, n = neg;
  pos = make_float2(p.x + n.x, p.y - n.y);
  neg = make_float2(n.x - p.x, n.y + p.y);
}
// The whole ISB step on a slice that one warp holds in order at col, once the slice is complete; ends with __syncwarp.
__device__ __forceinline__ void isb_fold_warp(float2 *col, int ns, int top, int lane) {
  for (int p = 1 + lane; p < ns / 2; p += 32) isb_fold(col[p], col[ns - p]);
  if (lane == 0) {
    col[0] = make_float2(0.f, 0.f);
    col[top] = make_float2(0.f, 0.f);
  }
  __syncwarp();
}

// Oscillator store of output sample i of a block k blocks past the epoch (radio.c:1476-1501): the rotated v, whose
// power term is added to pw (radio.c:1515-1520).
__device__ __forceinline__ float2 osc_sample(ChanAux const &ax, long k, int olen, int i, float2 v, float &pw) {
  v = osc_rotate(v, osc_phase_cycles(ax, k, olen, i));
  pw += v.x * v.x + v.y * v.y;
  return v;
}

// Sum of every thread's pw over a CTA of NT threads in a fixed order: warp sums, then the warps in order.  Every
// thread must call it (it holds a CTA barrier); the sum is returned to thread 0.
template <int NT>
__device__ __forceinline__ float cta_power_sum(float pw) {
  __shared__ float red[NT / 32];
  pw = warp_sum(pw);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = pw;
  __syncthreads();
  float s = 0.f;
  if (threadIdx.x == 0)
    for (int w = 0; w < NT / 32; w++) s += red[w];
  return s;
}

}  // namespace kfft
