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

// The four-step geometry of a length with a prime factor 11 .. 23: the plans of n1 and n2 by value (g.plan1 / g.plan2
// are unused), because such a length's plans never enter the registry.
struct WideGeomExt {
  WideGeom g;
  TilePlan p1, p2;
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

// The stages of the extended radices (primes 11 .. 23), which only the extended kernels compile in.
template <bool INV>
__device__ __forceinline__ void wide_stage_ext(int r, float2 *__restrict__ base, int ncols, int cs, int es, int len, int nsub,
                                               int s, uint32_t magic, float2 const *__restrict__ tw) {
  switch (r) {
    case 11: wide_stage<11, INV>(base, ncols, cs, es, len, nsub, s, magic, tw); break;
    case 13: wide_stage<13, INV>(base, ncols, cs, es, len, nsub, s, magic, tw); break;
    case 17: wide_stage<17, INV>(base, ncols, cs, es, len, nsub, s, magic, tw); break;
    case 19: wide_stage<19, INV>(base, ncols, cs, es, len, nsub, s, magic, tw); break;
    case 23: wide_stage<23, INV>(base, ncols, cs, es, len, nsub, s, magic, tw); break;
    default: break;
  }
}

// All stages of a plan on ncols columns; ends with a CTA barrier.  EXT also dispatches the extended radices, as in
// tile_fft.
template <bool INV, bool EXT = false>
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
      default:
        if constexpr (EXT) wide_stage_ext<INV>(r, base, ncols, cs, es, pl.len, n, s, mg, tw);
        break;
    }
    __syncthreads();
  }
}

// The four-step transform of the slice the CTA loaded (caller's barrier done); ends with a CTA barrier.  The plans are
// the registry's, or with EXT those of the extended geometry `xp` (whose .g is g).
template <bool INV, bool EXT = false>
__device__ __forceinline__ void wide_transform(WideGeom const &g, float2 *col, WideGeomExt const *xp = nullptr) {
  wide_fft<INV, EXT>(EXT ? xp->p2 : c_plans[g.plan2], col, g.n1, g.pitch, 1);
  int const nn = g.n1 * g.n2;
  for (int i = threadIdx.x; i < nn; i += blockDim.x) {
    int const k1 = i / g.n2;
    float2 *p = col + k1 * g.pitch + (i - k1 * g.n2);
    float2 const w = __ldg(g.tw + i);
    *p = INV ? cmulc(*p, w) : cmul(*p, w);
  }
  __syncthreads();
  wide_fft<INV, EXT>(EXT ? xp->p1 : c_plans[g.plan1], col, g.n2, 1, g.pitch);
}

__global__ void __launch_bounds__(kWideThreads) chan_wide(ChanArgs const a, WideGeom const g) {
#define KFFT_WIDE_EXT false
#include "chan_wide_body.cuh"
#undef KFFT_WIDE_EXT
}

// The wide channels of one extended length, every variant chan_wide serves.
__global__ void __launch_bounds__(kWideThreads) chan_wide_ext(ChanArgs const a, __grid_constant__ WideGeomExt const x) {
  WideGeom const &g = x.g;
#define KFFT_WIDE_EXT true
#include "chan_wide_body.cuh"
#undef KFFT_WIDE_EXT
}

// Forward transform of one wide response in place (set_filter's fftwf_execute, filter.c:1030), the same engine, on the
// registry's plans or, with EXT, on those of `xp`.
template <bool EXT>
__device__ __forceinline__ void response_wide_body(float2 *resp, WideGeom const &g, WideGeomExt const *xp) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  float2 *col = reinterpret_cast<float2 *>(smem_raw);
  int const ns = g.n1 * g.n2;
  for (int k = threadIdx.x; k < ns; k += blockDim.x) col[wide_in_slot(g, k)] = resp[k];
  __syncthreads();
  wide_transform<false, EXT>(g, col, xp);
  uint16_t const *perm1 = EXT ? xp->p1.perm : c_plans[g.plan1].perm, *perm2 = EXT ? xp->p2.perm : c_plans[g.plan2].perm;
  for (int k = threadIdx.x; k < ns; k += blockDim.x) resp[k] = col[wide_out_slot(g, perm1, perm2, k)];
}
// A single CTA: it may take every register (at two CTAs per SM the forward radix-36 stage would spill).
__global__ void __launch_bounds__(kWideThreads, 1) response_wide_kernel(float2 *resp, WideGeom const g) {
  response_wide_body<false>(resp, g, nullptr);
}
__global__ void __launch_bounds__(kWideThreads, 1) response_wide_ext(float2 *resp, __grid_constant__ WideGeomExt const x) {
  response_wide_body<true>(resp, x.g, &x);
}

}  // namespace kfft
