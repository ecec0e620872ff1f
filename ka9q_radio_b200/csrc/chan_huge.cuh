// chan_huge.cuh -- channels whose inverse transform is longer than kMaxWideChanPoints, up to kMaxHugeChanPoints (the
// 1.536 MS/s websdr channels of an RX888 at 64.8 MS/s: 38 400 points at overlap 5).  Such a slice does not fit one
// CTA's shared memory, so the four-step transform Ns = n1 * n2 (choose_split, both factors registry plans) goes through
// a scratch buffer in global memory, in two kernels shaped like the generic master pair (fwd_cols_body /
// fwd_rows_body.cuh): a tile of kTile adjacent columns or rows per CTA, one warp per column, tile_fft on registry plans.
//   input  k = n2*k1 + k2,  output n = j1 + n1*j2
//   pass A (chan_huge_cols): for every k2, length n1 over k1; times W_Ns^{-+j1*k2}   -> scratch[slot][j1][k2]
//   pass B (chan_huge_rows): for every j1, length n2 over k2 (contiguous)          -> output n = j1 + n1*j2
// Pass A forms slice x response element by element with chan_wide's semantics and rounding: every variant (conjugate
// walk, COMPLEX wrap, beam, ISB, the REAL-output Hermitian extension) is a function of the master spectrum at that one
// element, so the load needs no barrier across the slice.  Pass B keeps only the last olen outputs, at their natural
// positions, with the plain, oscillator and REAL-output stores.  The block power of an oscillator channel is summed per
// CTA in a fixed order, and huge_power_kernel adds the CTAs' partial sums in a fixed order, so a (channel, block) gets
// bitwise the same power whichever launch computes it.
// A slot of the scratch is one (channel, block): Ns float2.  The bank owns the buffer and loops over chunks of
// channels and blocks so that it stays below kHugeScratchCap (kgpu.cu).
#pragma once
#include "chan_kernels.cuh"
#include "fwd_kernels.cuh"

namespace kfft {

constexpr int kMaxHugeChanPoints = 1 << 20;
constexpr int kHugeThreads = kTile * 32;
constexpr int kHugeRowsPerIt = kHugeThreads / kTile;  // 32

// column_pitch (plan.cuh) in constexpr form: the smallest p >= len with p % 16 == 2
__host__ __device__ constexpr int huge_pitch(int len) { return len + ((2 - len % 16) + 16) % 16; }
__host__ __device__ constexpr long huge_smem_bytes(int len) { return 8L * kTile * huge_pitch(len); }

// One length's four-step geometry (host registry in kgpu.cu, passed by value to every launch of that length).
struct HugeGeom {
  int n1, n2;
  int pitch1, pitch2;  // shared-memory column pitch of pass A (n1) and pass B (n2)
  int plan1, plan2;    // registry plans of length n1 (pass A) and n2 (pass B)
};

// Element w of the slice chan_wide hands its inverse transform, computed from the spectrum alone (chan_slice.cuh's
// steps, element by element).
__device__ __forceinline__ float2 huge_slice(ChanArgs const &a, ChanDesc const &d, ChanAux const &ax, float2 const *X,
                                             float2 const *R, int w) {
  int const ns = d.points, top = (ns + 1) / 2, half = ns / 2;
  if (d.flags & kChanRealOut) {  // the Hermitian extension the c2r inverse implies
    if (w <= half) {
      float2 const v = real_half(a, d, X, R, w);
      return (w == 0 || 2 * w == ns) ? make_float2(v.x, 0.f) : v;
    }
    float2 const v = real_half(a, d, X, R, ns - w);
    return make_float2(v.x, -v.y);
  }
  auto base = [&](int v) {  // slot v before the ISB fold
    bool live;
    int const u = walk_pos(d, ns, top, v, live);
    if (!live) return make_float2(0.f, 0.f);
    int const q = walk_bin(a, d, u);
    float2 const r = __ldg(R + v);
    return (d.flags & kChanBeam) ? beam_product(ax, X, a.m_bins, q, r) : slice_product(d, __ldg(X + q), r);
  };
  if (!(d.flags & kChanIsb)) return base(w);
  if (w == 0 || w == top) return make_float2(0.f, 0.f);
  bool const lower = w < half;
  if (!lower && ns - w >= half) return base(w);  // the middle slot, which the fold leaves alone
  float2 pos = base(lower ? w : ns - w), neg = base(lower ? ns - w : w);
  isb_fold(pos, neg);
  return lower ? pos : neg;
}

// Pass A after the tile's columns k2 = c0 .. c0+ncols-1 are loaded (tile[c * pitch1 + k1]): transform each column,
// multiply by the inter-pass twiddle (double precision, rounded once) and store scratch slot `dst` as [j1][k2].
template <bool INV>
__device__ __forceinline__ void huge_cols_finish(HugeGeom const &g, float2 *tile, float2 *dst, int c0, int ncols) {
  int const tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, c = tid % kTile, r = tid / kTile;
  long const ns = (long)g.n1 * g.n2;
  TilePlan const &pl = c_plans[g.plan1];
  __syncthreads();
  if (warp < ncols) tile_fft<INV>(pl, tile + warp * g.pitch1, lane, 32, [] { __syncwarp(); });
  __syncthreads();
  if (c >= ncols) return;
  long const k2 = c0 + c;
  float2 const *colp = tile + c * g.pitch1;
  for (int j1 = r; j1 < g.n1; j1 += kHugeRowsPerIt) {
    float2 const w = unit_root_f((long)j1 * k2 % ns, ns);
    float2 const v = colp[__ldg(pl.perm + j1)];
    dst[(long)j1 * g.n2 + k2] = INV ? cmulc(v, w) : cmul(v, w);
  }
}

// Pass B's head: warp w streams row j1 = r0 + w of scratch slot `src` into its column and transforms it.
template <bool INV>
__device__ __forceinline__ void huge_rows_start(HugeGeom const &g, float2 *tile, float2 const *src, int r0, int nrows) {
  int const tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (warp < nrows) {
    float2 const *row = src + (long)(r0 + warp) * g.n2;
    float2 *colp = tile + warp * g.pitch2;
    for (int k2 = lane; k2 < g.n2; k2 += 32) colp[k2] = row[k2];
    __syncwarp();
    tile_fft<INV>(c_plans[g.plan2], colp, lane, 32, [] { __syncwarp(); });
  }
  __syncthreads();
}

// grid (n2 column tiles, channels, blocks); scratch slot (block, channel) = blockIdx.z * gridDim.y + blockIdx.y
__global__ void __launch_bounds__(kHugeThreads, 2) chan_huge_cols(ChanArgs const a, HugeGeom const g, float2 *scratch) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  float2 *tile = reinterpret_cast<float2 *>(smem_raw);  // [kTile][pitch1]
  int const oi = blockIdx.y;
  int const ci = chan_index(a, oi);
  ChanDesc const d = a.desc[ci];
  if (d.plan < 0) return;
  int const blk = blockIdx.z, tid = threadIdx.x, c = tid % kTile, r = tid / kTile;
  int const c0 = blockIdx.x * kTile, ncols = min(kTile, g.n2 - c0);
  ChanAux ax{};
  if (d.flags & kChanBeam) ax = a.aux[ci];
  float2 const *X = a.spec + (long)blk * a.spec_stride;
  float2 const *R = a.resp + d.resp_off;
  if (c < ncols)
    for (int k1 = r; k1 < g.n1; k1 += kHugeRowsPerIt) tile[c * g.pitch1 + k1] = huge_slice(a, d, ax, X, R, g.n2 * k1 + c0 + c);
  long const slot = (long)blk * gridDim.y + oi;
  huge_cols_finish<true>(g, tile, scratch + slot * d.points, c0, ncols);
}

// grid (n1 row tiles, channels, blocks).  partial: [slot][gridDim.x] per-CTA power sums of kChanOsc channels.
__global__ void __launch_bounds__(kHugeThreads, 2) chan_huge_rows(ChanArgs const a, HugeGeom const g, float2 const *scratch,
                                                               float *partial) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  float2 *tile = reinterpret_cast<float2 *>(smem_raw);  // [kTile][pitch2]
  int const oi = blockIdx.y;
  int const ci = chan_index(a, oi);
  ChanDesc const d = a.desc[ci];
  if (d.plan < 0) return;
  int const blk = blockIdx.z, tid = threadIdx.x;
  int const r0 = blockIdx.x * kTile, nrows = min(kTile, g.n1 - r0);
  long const slot = (long)blk * gridDim.y + oi;
  huge_rows_start<true>(g, tile, scratch + slot * d.points, r0, nrows);

  uint16_t const *perm2 = c_plans[g.plan2].perm;
  int const i = tid % kTile, q = tid / kTile, j1 = r0 + i;
  bool const row_ok = i < nrows;
  float2 const *colp = tile + i * g.pitch2;
  int const first = d.points - d.olen;
  float2 *dst = a.out + (long)blk * a.out_stride + d.out_off;
  // the first j2 whose output n = j1 + n1*j2 is among the last olen
  int const j2lo = first > j1 ? (first - j1 + g.n1 - 1) / g.n1 : 0;
  if (d.flags & kChanRealOut) {  // c2r: the real part, olen floats packed in the channel's float2 run
    float *dr = reinterpret_cast<float *>(dst);
    if (row_ok)
      for (int j2 = j2lo + q; j2 < g.n2; j2 += kHugeRowsPerIt) dr[j1 + g.n1 * j2 - first] = colp[__ldg(perm2 + j2)].x;
    return;
  }
  if (d.flags & kChanOsc) {
    ChanAux const ax = a.aux[ci];
    long const k = a.block0 + blk - ax.osc_epoch;
    float pw = 0.f;
    if (row_ok)
      for (int j2 = j2lo + q; j2 < g.n2; j2 += kHugeRowsPerIt) {
        int const n = j1 + g.n1 * j2 - first;
        dst[n] = osc_sample(ax, k, d.olen, n, colp[__ldg(perm2 + j2)], pw);
      }
    float const s = cta_power_sum<kHugeThreads>(pw);
    if (partial && tid == 0) partial[slot * gridDim.x + blockIdx.x] = s;
    return;
  }
  if (row_ok)
    for (int j2 = j2lo + q; j2 < g.n2; j2 += kHugeRowsPerIt) dst[j1 + g.n1 * j2 - first] = colp[__ldg(perm2 + j2)];
}

// grid (channels, blocks), one warp: the block power of each kChanOsc channel from pass B's ntiles partial sums
__global__ void __launch_bounds__(32) huge_power_kernel(ChanArgs const a, float const *partial, int ntiles) {
  int const oi = blockIdx.x, blk = blockIdx.y, lane = threadIdx.x;
  int const ci = chan_index(a, oi);
  ChanDesc const d = a.desc[ci];
  if (d.plan < 0 || !(d.flags & kChanOsc) || (d.flags & kChanRealOut)) return;
  float const *p = partial + ((long)blk * gridDim.x + oi) * ntiles;
  float s = 0.f;
  for (int t = lane; t < ntiles; t += 32) s += p[t];
  s = warp_sum(s);
  if (lane == 0) a.power[(long)blk * a.power_stride + ci] = s / (float)d.olen;
}

// Forward transform of one huge response in place (set_filter's fftwf_execute, filter.c:1030), the same pair of passes
// through a scratch slot: response_huge_cols, then response_huge_rows.
__global__ void __launch_bounds__(kHugeThreads, 2) response_huge_cols(float2 const *resp, HugeGeom const g, float2 *scratch) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  float2 *tile = reinterpret_cast<float2 *>(smem_raw);
  int const tid = threadIdx.x, c = tid % kTile, r = tid / kTile;
  int const c0 = blockIdx.x * kTile, ncols = min(kTile, g.n2 - c0);
  if (c < ncols)
    for (int k1 = r; k1 < g.n1; k1 += kHugeRowsPerIt) tile[c * g.pitch1 + k1] = resp[(long)g.n2 * k1 + c0 + c];
  huge_cols_finish<false>(g, tile, scratch, c0, ncols);
}
__global__ void __launch_bounds__(kHugeThreads, 2) response_huge_rows(float2 *resp, HugeGeom const g, float2 const *scratch) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  float2 *tile = reinterpret_cast<float2 *>(smem_raw);
  int const tid = threadIdx.x, r0 = blockIdx.x * kTile, nrows = min(kTile, g.n1 - r0);
  huge_rows_start<false>(g, tile, scratch, r0, nrows);
  int const i = tid % kTile, q = tid / kTile;
  if (i >= nrows) return;
  uint16_t const *perm2 = c_plans[g.plan2].perm;
  float2 const *colp = tile + i * g.pitch2;
  for (int j2 = q; j2 < g.n2; j2 += kHugeRowsPerIt) resp[r0 + i + (long)g.n1 * j2] = colp[__ldg(perm2 + j2)];
}

}  // namespace kfft
