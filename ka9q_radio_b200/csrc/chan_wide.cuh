// chan_wide.cuh -- channels whose inverse transform is longer than kMaxChanPoints (the 384 kHz `wfm` downconverter,
// wide spectrum-mode slaves).  One CTA owns one (channel, block) and holds the whole Ns-point slice in shared memory;
// the transform is a four-step split Ns = n1 * n2 (both factors <= kMaxTileLen, registry plans, the same choice
// choose_split makes for masters), computed in place:
//   input  k = k1 + n1*k2  sits at  row k1, column k2   (row pitch `pitch` = n2 rounded up to odd)
//   pass 1: every row, length n2 over k2            -> j2 at column perm2[j2]
//   twiddle W_Ns^{+-k1*j2}                         (host table in column order, long double, rounded once)
//   pass 2: every column, length n1 over k1 (stride pitch) -> j1 at row perm1[j1]
//   output n = n2*j1 + j2  sits at  row perm1[j1], column perm2[j2]
// The load stage forms slice x response with chan_kernel's semantics and writes each product straight into its
// row/column, so there is no separate transpose; the epilogue resolves both digit reversals while it stores the last
// olen samples in natural order.  No cluster, no inter-CTA traffic: one launch, grid (channels, blocks).
#pragma once
#include "chan_kernels.cuh"

namespace kfft {

constexpr int kWideThreads = 256;

// Every length in (kMaxChanPoints, kMaxWideChanPoints] with factors 2, 3, 5, 7 splits into two plannable factors, and
// its n1 rows of pitch (n2 | 1) float2 fit the 227 KB a block may opt into: 28812 = 196 x 147 needs 225 KB, while the
// next such length, 29160 = 180 x 162, needs 229 KB.  kgpu.cu asserts both at compile time.
constexpr int kMaxWideChanPoints = 28812;
static_assert(kMaxWideChanPoints >= 15360, "wfm (384 kHz) at the default block time at overlap 2 needs 15360 points");

__host__ __device__ constexpr int wide_pitch(int n2) { return n2 | 1; }  // odd: rows and columns both bank-conflict free
__host__ __device__ constexpr long wide_smem_bytes(int n1, int n2) { return 8L * n1 * wide_pitch(n2); }

// One length's four-step geometry (host registry in kgpu.cu, passed by value to every launch of that length).
struct WideGeom {
  int n1, n2, pitch;
  int plan1, plan2;  // registry plans of length n1 (pass 2) and n2 (pass 1)
  float2 const *tw;  // [k1 * n2 + c] = W_Ns^{k1 * j2}, j2 = the output index pass 1 leaves in column c (forward sign)
};

// shared-memory slot of input point k / of output point n after both passes
__device__ __forceinline__ int wide_in_slot(WideGeom const &g, int k) {
  int const k2 = k / g.n1;
  return (k - k2 * g.n1) * g.pitch + k2;
}
__device__ __forceinline__ int wide_out_slot(WideGeom const &g, uint16_t const *perm1, uint16_t const *perm2, int n) {
  int const j1 = n / g.n2;
  return (int)__ldg(perm1 + j1) * g.pitch + (int)__ldg(perm2 + (n - j1 * g.n2));
}

// dif_stage over `ncols` columns at once, the whole CTA cooperating: column c starts at base + c*cs, its elements are
// es apart.  Consecutive threads take consecutive columns, so with an odd pitch neither pass has bank conflicts.
template <int R, bool INV>
__device__ __forceinline__ void wide_stage(float2 *__restrict__ base, int ncols, int cs, int es, int len, int nsub, int s,
                                           uint32_t magic, float2 const *__restrict__ tw) {
  int const total = (len / R) * ncols;
  for (int w = threadIdx.x; w < total; w += blockDim.x) {
    int const u = w / ncols, c = w - u * ncols;
    int b, j;
    if (s == 1) {
      b = u;
      j = 0;
    } else {
      b = (int)__umulhi((uint32_t)u, magic);
      j = u - b * s;
    }
    float2 *p = base + c * cs + (b * nsub + j) * es;
    int const step = s * es;
    float2 x[R];
#pragma unroll
    for (int m = 0; m < R; m++) x[m] = p[m * step];
    Dft<R, INV>::run(x);
    if (s > 1) {
#pragma unroll
      for (int t = 1; t < R; t++) {
        float2 const wt = __ldg(tw + (t - 1) * s + j);
        x[t] = INV ? cmulc(x[t], wt) : cmul(x[t], wt);
      }
    }
#pragma unroll
    for (int t = 0; t < R; t++) p[t * step] = x[t];
  }
}

// All stages of a registry plan on ncols columns; ends with a CTA barrier.
template <bool INV>
__device__ __forceinline__ void wide_fft(TilePlan const &pl, float2 *base, int ncols, int cs, int es) {
  for (int i = 0; i < pl.nstages; i++) {
    int const r = pl.radix[i], n = pl.sub[i], s = pl.stride[i];
    uint32_t const mg = pl.magic[i];
    float2 const *tw = pl.tw + pl.tw_off[i];
    switch (r) {
#define KFFT_WIDE_CASE(RR) \
  case RR: wide_stage<RR, INV>(base, ncols, cs, es, pl.len, n, s, mg, tw); break;
      KFFT_WIDE_CASE(2)
      KFFT_WIDE_CASE(3)
      KFFT_WIDE_CASE(4)
      KFFT_WIDE_CASE(5)
      KFFT_WIDE_CASE(6)
      KFFT_WIDE_CASE(7)
      KFFT_WIDE_CASE(8)
      KFFT_WIDE_CASE(9)
      KFFT_WIDE_CASE(10)
      KFFT_WIDE_CASE(12)
      KFFT_WIDE_CASE(15)
      KFFT_WIDE_CASE(16)
      KFFT_WIDE_CASE(20)
      KFFT_WIDE_CASE(24)
      KFFT_WIDE_CASE(25)
      KFFT_WIDE_CASE(36)
#undef KFFT_WIDE_CASE
      default: break;
    }
    __syncthreads();
  }
}

// The four-step transform of the slice the CTA loaded (caller's barrier done); ends with a CTA barrier.
template <bool INV>
__device__ __forceinline__ void wide_transform(WideGeom const &g, float2 *col) {
  wide_fft<INV>(c_plans[g.plan2], col, g.n1, g.pitch, 1);
  int const nn = g.n1 * g.n2;
  for (int i = threadIdx.x; i < nn; i += blockDim.x) {
    int const k1 = i / g.n2;
    float2 *p = col + k1 * g.pitch + (i - k1 * g.n2);
    float2 const w = __ldg(g.tw + i);
    *p = INV ? cmulc(*p, w) : cmul(*p, w);
  }
  __syncthreads();
  wide_fft<INV>(c_plans[g.plan1], col, g.n2, 1, g.pitch);
}

__global__ void __launch_bounds__(kWideThreads) chan_wide(ChanArgs const a, WideGeom const g) {
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
  wide_transform<true>(g, col);

  uint16_t const *perm1 = c_plans[g.plan1].perm, *perm2 = c_plans[g.plan2].perm;
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
}

// Forward transform of one wide response in place (set_filter's fftwf_execute, filter.c:1030), the same engine.
// A single CTA: it may take every register (at two CTAs per SM the forward radix-36 stage would spill).
__global__ void __launch_bounds__(kWideThreads, 1) response_wide_kernel(float2 *resp, WideGeom const g) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  float2 *col = reinterpret_cast<float2 *>(smem_raw);
  int const ns = g.n1 * g.n2;
  for (int k = threadIdx.x; k < ns; k += blockDim.x) col[wide_in_slot(g, k)] = resp[k];
  __syncthreads();
  wide_transform<false>(g, col);
  uint16_t const *perm1 = c_plans[g.plan1].perm, *perm2 = c_plans[g.plan2].perm;
  for (int k = threadIdx.x; k < ns; k += blockDim.x) resp[k] = col[wide_out_slot(g, perm1, perm2, k)];
}

}  // namespace kfft
