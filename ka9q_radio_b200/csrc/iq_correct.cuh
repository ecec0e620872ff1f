// iq_correct.cuh -- the DC removal and I/Q gain and phase correction of the HackRF and FUNcube drivers
// (hackrf.c:297-375, funcube.c:194-310) on the device, by exact moments.
//
// A driver corrects each write (one USB transfer, or one PortAudio block) with the state the previous write left, then
// updates the state from sums over the write.  Those sums follow from five exact integer moments of the write's words
// (Si, Sq, Sii, Sqq, Siq), so the device:
//   iq_moments_kernel  sums the moments, the components at the limits and the last of them per write, in int64, over
//                      a launch's new samples (a write that straddles launches completes in the later one);
//   iq_scan_kernel     one thread: per completed write, in order, its record and the state after it, which is the
//                      coefficient set of the next write;
//   iq_apply_kernel    the corrected floats of a window, each sample with its own write's coefficients and scale.
// Writes live in a ring table indexed by write number modulo its capacity; `first` is the absolute index of a write's
// first sample (0 = the first sample ever written).  Samples before it (the first window's history) are 0.0f.
// All double arithmetic is rounded per operation (__dmul_rn, __dadd_rn, ...): no contraction, so the records, states
// and floats are bitwise those of the restatement in tests/iq_correction_ref.py.
#pragma once
#include <stdint.h>

namespace kfft {

constexpr int kIqThreads = 256;
constexpr int kIqChunk = 2048;  // samples per CTA

struct IqWrite {  // = struct kgpu_iq_write
  long long first, n;
  double scale;
  long long m[5];  // Si, Sq, Sii, Sqq, Siq
  long long overs;
  long long last_over;  // absolute component index (2 * sample + 0 for I, 1 for Q), -1 if none
};
struct IqState {  // = struct kgpu_iq_state
  double dc_i, dc_q, sinphi, imbalance, gain_i, gain_q, secphi, tanphi;
};
struct IqRecord {  // = struct kgpu_iq_record
  long long seq, n, sum_i, sum_q;
  double i_energy, q_energy, dotprod;
  long long overs, since_over;
  IqState state;
};

// One I/Q pair at index s of the raw words.  S8: HackRF's -128 -> -127, counted (hackrf.c:325-332); S16: FUNcube's
// words as they are, |x| >= 32767 counted (funcube.c:256-266).
template <bool S16>
__device__ __forceinline__ void iq_load(void const *__restrict__ raw, long s, int &i, int &q, bool &oi, bool &oq) {
  if (S16) {
    short2 const v = reinterpret_cast<short2 const *>(raw)[s];
    i = v.x;
    q = v.y;
    oi = i >= 32767 || i <= -32767;
    oq = q >= 32767 || q <= -32767;
  } else {
    char2 const v = reinterpret_cast<char2 const *>(raw)[s];
    i = v.x;
    q = v.y;
    oi = i == -128;
    oq = q == -128;
    if (oi) i = -127;
    if (oq) q = -127;
  }
}

// the write among [w_lo, w_lo + nw) holding absolute sample a (the last whose first sample is <= a)
__device__ __forceinline__ long long iq_find(IqWrite const *tab, int cap, long long w_lo, int nw, long long a) {
  long long lo = w_lo, hi = w_lo + nw - 1;
  while (lo < hi) {
    long long const mid = (lo + hi + 1) >> 1;
    if (tab[mid % cap].first <= a) lo = mid;
    else hi = mid - 1;
  }
  return lo;
}

// samples [a0, a0 + count) at raw[0 ..]: every one lies in a write of [w_lo, w_lo + nw)
template <bool S16>
__global__ void __launch_bounds__(kIqThreads) iq_moments_kernel(void const *__restrict__ raw, long long a0, long count,
                                                                IqWrite *tab, int cap, long long w_lo, int nw) {
  __shared__ long long red[kIqThreads / 32][7];
  __shared__ long long w0;
  long long const c0 = a0 + (long long)blockIdx.x * kIqChunk;
  long long const c1 = min(c0 + kIqChunk, a0 + count);
  if (threadIdx.x == 0) w0 = iq_find(tab, cap, w_lo, nw, c0);
  __syncthreads();
  int const lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (long long w = w0; w < w_lo + nw; w++) {
    IqWrite *const t = &tab[w % cap];
    long long const f = t->first;
    if (f >= c1) break;
    long long const s0 = max(c0, f), s1 = min(c1, f + t->n);
    long long v[7] = {0, 0, 0, 0, 0, 0, -1};  // Si, Sq, Sii, Sqq, Siq, overs, last over
    for (long long a = s0 + threadIdx.x; a < s1; a += kIqThreads) {
      int i, q;
      bool oi, oq;
      iq_load<S16>(raw, (long)(a - a0), i, q, oi, oq);
      v[0] += i;
      v[1] += q;
      v[2] += (long long)(i * i);
      v[3] += (long long)(q * q);
      v[4] += (long long)(i * q);
      v[5] += (int)oi + (int)oq;
      if (oq) v[6] = 2 * a + 1;
      else if (oi) v[6] = 2 * a;
    }
#pragma unroll
    for (int k = 16; k > 0; k >>= 1) {
#pragma unroll
      for (int j = 0; j < 6; j++) v[j] += __shfl_xor_sync(0xffffffffu, v[j], k);
      v[6] = max(v[6], __shfl_xor_sync(0xffffffffu, v[6], k));
    }
    if (lane == 0)
#pragma unroll
      for (int j = 0; j < 7; j++) red[warp][j] = v[j];
    __syncthreads();
    if (threadIdx.x == 0) {
      for (int u = 1; u < kIqThreads / 32; u++) {
#pragma unroll
        for (int j = 0; j < 6; j++) v[j] += red[u][j];
        v[6] = max(v[6], red[u][6]);
      }
#pragma unroll
      for (int j = 0; j < 5; j++)
        if (v[j]) atomicAdd(reinterpret_cast<unsigned long long *>(&t->m[j]), (unsigned long long)v[j]);
      if (v[5]) {
        atomicAdd(reinterpret_cast<unsigned long long *>(&t->overs), (unsigned long long)v[5]);
        atomicMax(&t->last_over, v[6]);
      }
    }
    __syncthreads();
  }
}

struct IqParams {  // the scan's constants (struct kgpu_iq_params less the initial state)
  int kind;        // 1: HackRF (weight gp * n, DC held when n == 0), 2: FUNcube (weight gp)
  double dc_alpha, gp;
};

// writes [w_from, w_from + nw), all complete, in order: coef[w % cap] is the state write w was corrected with; its
// record goes to rec[w % cap] and the state after it to coef[(w + 1) % cap].  Expression order of hackrf.c:356-374 and
// funcube.c:295-307; 2 * dotprod / (i + q) == dotprod / (0.5 * (i + q)) in IEEE double, so one form serves both.
__global__ void iq_scan_kernel(IqWrite const *tab, IqState *coef, int cap, long long w_from, int nw, IqParams p,
                               IqRecord *rec) {
  for (long long w = w_from; w < w_from + nw; w++) {
    IqWrite const t = tab[w % cap];
    IqState const st = coef[w % cap];
    double const nd = __ll2double_rn(t.n);
    double const Si = __ll2double_rn(t.m[0]), Sq = __ll2double_rn(t.m[1]);
    double const Sii = __ll2double_rn(t.m[2]), Sqq = __ll2double_rn(t.m[3]), Siq = __ll2double_rn(t.m[4]);
    double const r = st.dc_i, c = st.dc_q;
    double const ie = __dadd_rn(__dsub_rn(Sii, __dmul_rn(__dmul_rn(2.0, r), Si)), __dmul_rn(__dmul_rn(nd, r), r));
    double const qe = __dadd_rn(__dsub_rn(Sqq, __dmul_rn(__dmul_rn(2.0, c), Sq)), __dmul_rn(__dmul_rn(nd, c), c));
    double const cross = __dadd_rn(__dsub_rn(__dsub_rn(Siq, __dmul_rn(c, Si)), __dmul_rn(r, Sq)), __dmul_rn(__dmul_rn(nd, r), c));
    double const dot = __dmul_rn(__dmul_rn(st.gain_i, st.gain_q), cross);
    IqState s = st;
    if (t.n != 0 || p.kind != 1) {  // hackrf.c:359
      s.dc_i = __dadd_rn(r, __dmul_rn(p.dc_alpha, __dsub_rn(Si, __dmul_rn(nd, r))));
      s.dc_q = __dadd_rn(c, __dmul_rn(p.dc_alpha, __dsub_rn(Sq, __dmul_rn(nd, c))));
    }
    double const be = __dmul_rn(0.5, __dadd_rn(ie, qe));
    if (be > 0) {
      double const w8 = p.kind == 1 ? __dmul_rn(p.gp, nd) : p.gp;
      s.imbalance = __dadd_rn(s.imbalance, __dmul_rn(w8, __dsub_rn(__ddiv_rn(ie, qe), s.imbalance)));
      double const dpn = __ddiv_rn(dot, be);
      s.sinphi = __dadd_rn(s.sinphi, __dmul_rn(w8, __dsub_rn(dpn, s.sinphi)));
      s.gain_q = __dsqrt_rn(__dmul_rn(0.5, __dadd_rn(1.0, s.imbalance)));
      s.gain_i = __dsqrt_rn(__dmul_rn(0.5, __dadd_rn(1.0, __ddiv_rn(1.0, s.imbalance))));
      s.secphi = __ddiv_rn(1.0, __dsqrt_rn(__dsub_rn(1.0, __dmul_rn(s.sinphi, s.sinphi))));
      s.tanphi = __dmul_rn(s.sinphi, s.secphi);
    }
    coef[(w + 1) % cap] = s;
    IqRecord &o = rec[w % cap];
    o.seq = w;
    o.n = t.n;
    o.sum_i = t.m[0];
    o.sum_q = t.m[1];
    o.i_energy = ie;
    o.q_energy = qe;
    o.dotprod = dot;
    o.overs = t.overs;
    o.since_over = t.last_over < 0 ? -1 : 2 * (t.first + t.n) - 1 - t.last_over;
    o.state = s;
  }
}

// the corrected floats of samples [a0, a0 + count) (raw[0 ..] and out[0 ..] hold sample a0); samples a >= 0 lie in
// writes of [w_lo, w_lo + nw) whose coefficients are known, samples a < 0 precede the first write and are 0.0f.
template <bool S16>
__global__ void __launch_bounds__(kIqThreads) iq_apply_kernel(void const *__restrict__ raw, long long a0, long count,
                                                              IqWrite const *tab, IqState const *coef, int cap,
                                                              long long w_lo, int nw, float2 *__restrict__ out) {
  __shared__ long long w0;
  long long const c0 = a0 + (long long)blockIdx.x * kIqChunk;
  long long const c1 = min(c0 + kIqChunk, a0 + count);
  for (long long a = c0 + threadIdx.x; a < min(c1, 0LL); a += kIqThreads) out[a - a0] = make_float2(0.f, 0.f);
  if (c1 <= 0) return;
  if (threadIdx.x == 0) w0 = iq_find(tab, cap, w_lo, nw, max(c0, 0LL));
  __syncthreads();
  for (long long w = w0; w < w_lo + nw; w++) {
    long long const f = tab[w % cap].first;
    if (f >= c1) break;
    long long const s0 = max(max(c0, f), 0LL), s1 = min(c1, f + tab[w % cap].n);
    double const scale = tab[w % cap].scale;
    IqState const k = coef[w % cap];
    for (long long a = s0 + threadIdx.x; a < s1; a += kIqThreads) {
      int i, q;
      bool oi, oq;
      iq_load<S16>(raw, (long)(a - a0), i, q, oi, oq);
      double const xi = __dmul_rn(__dsub_rn((double)i, k.dc_i), k.gain_i);
      double const yq = __dmul_rn(__dsub_rn((double)q, k.dc_q), k.gain_q);
      double const y = __dsub_rn(__dmul_rn(k.secphi, yq), __dmul_rn(k.tanphi, xi));
      out[a - a0] = make_float2(__double2float_rn(__dmul_rn(scale, xi)), __double2float_rn(__dmul_rn(scale, y)));
    }
  }
}

}  // namespace kfft
