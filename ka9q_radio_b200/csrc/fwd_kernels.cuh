// fwd_kernels.cuh -- the wideband forward transform (replaces fftwf_execute_dft_r2c /
// fftwf_execute_dft at reference filter.c:505-508) as two shared-memory passes.
//
// REAL master, N = 2*Nc real samples: z[n] = x[2n] + i*x[2n+1], Z = DFT_Nc(z) by the two passes,
// then the split  X[k] = E - i*W_N^k*O,  E = (Z[k]+conj Z[Nc-k])/2, O = (Z[k]-conj Z[Nc-k])/2
// fused into pass 2's epilogue.  COMPLEX master: plain DFT_N, no split.
//
// Index maps (Nc = N1*N2):  n = N2*n1 + n2,  k = k1 + N1*k2
//   pass 1 (cols): for each n2, DFT_N1 over n1 (stride N2), times W_Nc^{n2*k1}  -> mid[k1][n2]
//   pass 2 (rows): for each k1, DFT_N2 over n2 (contiguous)                     -> Z[k1 + N1*k2]
//
// Both kernels give one warp one column of the tile; the only block-wide barriers are around
// the cooperative (coalesced) global loads/stores.  int16 -> float (rx888.c:753-767) and the
// overlap-save window addressing (filter.c:631-635) are part of pass 1's load.
#pragma once
#include "fft_tile.cuh"

namespace kfft {

constexpr int kTile = 8;              // columns (warps) per CTA
constexpr int kFwdThreads = kTile * 32;

struct IngestStats {
  unsigned long long energy;
  unsigned int clips;
  unsigned int pad;
};

struct Pass1Args {
  void const *in;       // block 0 window start
  long hop;             // complex elements (pairs) between consecutive block windows = L/2 (REAL) or L
  int n1, n2;           // column length, number of columns
  long nc;              // n1*n2
  int plan;             // registry index of the length-n1 column plan
  int pitch;            // shared-memory column pitch
  float scale;          // int16 scale
  int derandomize;
  long first_new;       // index (in complex elements) of the first NEW element of a window, for stats
  float2 *mid;          // [block][k1][n2]
  IngestStats *stats;   // or nullptr
  float out_scale;      // specialised kernels: factor folded into the inter-pass twiddle (int16 scale, x0.5 when the split is pre-halved)
  int mid_ld;           // elements between consecutive k1 rows of `mid` (>= n2; padded to 128 bytes for the specialised pairs)
};

// exp(-2*pi*i*e/n) from a double-precision sincospi, rounded once
__device__ __forceinline__ float2 unit_root_f(long e, long n) {
  double s, c;
  sincospi(2.0 * (double)e / (double)n, &s, &c);
  return make_float2((float)c, (float)-s);
}

template <int FMT /*0: float pairs, 1: int16 pairs*/>
__global__ void __launch_bounds__(kFwdThreads, 2) fwd_cols_kernel(Pass1Args const a) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  float2 *tile = reinterpret_cast<float2 *>(smem_raw);             // [kTile][pitch]
  int const rows_per_it = kFwdThreads / kTile;                      // 32
  int const nit = (a.n1 + rows_per_it - 1) / rows_per_it;
  float2 *twA = tile + kTile * a.pitch;                             // [kTile][nit]

  TilePlan const &pl = c_plans[a.plan];
  int const tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  int const c = tid % kTile, r = tid / kTile;
  int const c0 = blockIdx.x * kTile;
  int const blk = blockIdx.y;
  int const ncols = min(kTile, a.n2 - c0);
  bool const col_ok = c < ncols;
  long const n2g = c0 + c;  // this thread's global column in the cooperative phases

  // ---- cooperative load: kTile adjacent columns x 32 rows per step ----------------------
  unsigned long long energy = 0;
  unsigned int clips = 0;
  constexpr int U = 8;  // independent global loads in flight per thread
  if (FMT == 1) {
    int const *src = reinterpret_cast<int const *>(a.in) + (long)blk * a.hop + n2g;
    auto put = [&](int n1, int w) {
      short lo = (short)(w & 0xffff), hi = (short)((unsigned)w >> 16);
      if (a.derandomize) {  // lsb set -> flip bits 1..15 (rx888.c:707-712)
        lo ^= (short)((lo & 1) ? 0xfffe : 0);
        hi ^= (short)((hi & 1) ? 0xfffe : 0);
      }
      if (a.stats && (long)n1 * a.n2 + n2g >= a.first_new) {
        energy += (unsigned long long)((int)lo * lo) + (unsigned long long)((int)hi * hi);
        clips += (lo > 32766 || lo < -32766) + (hi > 32766 || hi < -32766);
      }
      tile[c * a.pitch + n1] = make_float2((float)lo * a.scale, (float)hi * a.scale);
    };
    int n1 = r;
    if (col_ok) {
      for (; n1 + (U - 1) * rows_per_it < a.n1; n1 += U * rows_per_it) {
        int w[U];
#pragma unroll
        for (int u = 0; u < U; u++) w[u] = __ldg(src + (long)(n1 + u * rows_per_it) * a.n2);
#pragma unroll
        for (int u = 0; u < U; u++) put(n1 + u * rows_per_it, w[u]);
      }
      for (; n1 < a.n1; n1 += rows_per_it) put(n1, __ldg(src + (long)n1 * a.n2));
    } else {
      for (; n1 < a.n1; n1 += rows_per_it) tile[c * a.pitch + n1] = make_float2(0.f, 0.f);
    }
  } else {
    float2 const *src = reinterpret_cast<float2 const *>(a.in) + (long)blk * a.hop + n2g;
    int n1 = r;
    if (col_ok) {
      for (; n1 + (U - 1) * rows_per_it < a.n1; n1 += U * rows_per_it) {
        float2 w[U];
#pragma unroll
        for (int u = 0; u < U; u++) w[u] = __ldg(src + (long)(n1 + u * rows_per_it) * a.n2);
#pragma unroll
        for (int u = 0; u < U; u++) tile[c * a.pitch + n1 + u * rows_per_it] = w[u];
      }
      for (; n1 < a.n1; n1 += rows_per_it) tile[c * a.pitch + n1] = __ldg(src + (long)n1 * a.n2);
    } else {
      for (; n1 < a.n1; n1 += rows_per_it) tile[c * a.pitch + n1] = make_float2(0.f, 0.f);
    }
  }
  // inter-pass twiddle factors W_nc^{n2*k1}, k1 = r + 32*it, as B(n2,r) * A(n2,it)
  float2 twB = make_float2(1.f, 0.f);
  if (col_ok) twB = unit_root_f((n2g * r) % a.nc, a.nc);
  for (int i = tid; i < kTile * nit; i += kFwdThreads) {
    int const cc = i / nit, it = i - cc * nit;
    long const e = ((long)(c0 + cc) * rows_per_it * it) % a.nc;
    twA[i] = unit_root_f(e, a.nc);
  }
  if (FMT == 1 && a.stats) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      energy += __shfl_xor_sync(0xffffffffu, energy, o);
      clips += __shfl_xor_sync(0xffffffffu, clips, o);
    }
    if (lane == 0 && (energy | clips)) {
      atomicAdd(&a.stats[blk].energy, energy);
      atomicAdd(&a.stats[blk].clips, clips);
    }
  }
  __syncthreads();

  // ---- one warp per column: length-n1 transform in shared memory -------------------------
  if (warp < ncols) tile_fft<false>(pl, tile + warp * a.pitch, lane, 32, [] { __syncwarp(); });
  __syncthreads();

  // ---- cooperative store with the inter-pass twiddle: mid[k1][n2] ------------------------
  if (col_ok) {
    float2 *dst = a.mid + (long)blk * a.nc + n2g;
    float2 const *colp = tile + c * a.pitch;
    float2 const *twc = twA + c * nit;
    constexpr int V = 4;
    int it = 0, k1 = r;
    for (; k1 + (V - 1) * rows_per_it < a.n1; k1 += V * rows_per_it, it += V) {
      int slot[V];
      float2 v[V];
#pragma unroll
      for (int u = 0; u < V; u++) slot[u] = __ldg(pl.perm + k1 + u * rows_per_it);
#pragma unroll
      for (int u = 0; u < V; u++) v[u] = cmul(colp[slot[u]], cmul(twB, twc[it + u]));
#pragma unroll
      for (int u = 0; u < V; u++) dst[(long)(k1 + u * rows_per_it) * a.n2] = v[u];
    }
    for (; k1 < a.n1; k1 += rows_per_it, it++)
      dst[(long)k1 * a.n2] = cmul(colp[__ldg(pl.perm + k1)], cmul(twB, twc[it]));
  }
}

// ---------------------------------------------------------------------------------------------
enum RowKind : int { kRowEmpty = 0, kRowPair = 1, kRowSelf0 = 2, kRowSelfMid = 3, kRowPlain = 4 };
struct RowItem {   // one unit of pass-2 work: a row, or a mirrored pair of rows
  int kind;
  int row_a;       // k1 of the first row (column 2*i of the tile, or column i for plain rows)
  int row_b;       // k1 of the mirror row N1-row_a (column 2*i+1), pairs only
};

// Pass-2 work item p.  REAL: row 0 | pairs (k1, n1-k1) | row n1/2 (n1 even) | empty padding, n1/2 + 1 items in all.
// COMPLEX: row p | empty padding.
__device__ __forceinline__ RowItem row_item(int p, int n1, bool real_split) {
  RowItem it;
  if (!real_split) {
    it.kind = p < n1 ? kRowPlain : kRowEmpty;
    it.row_a = p;
    it.row_b = 0;
    return it;
  }
  it.row_a = p;
  it.row_b = n1 - p;
  if (p == 0) it.kind = kRowSelf0, it.row_b = 0;
  else if (2 * p < n1) it.kind = kRowPair;
  else if (2 * p == n1) it.kind = kRowSelfMid, it.row_b = p;
  else it.kind = kRowEmpty, it.row_a = it.row_b = 0;
  return it;
}

struct Pass2Args {
  float2 const *mid;    // [block][k1][n2]
  int n1, n2;
  long nc;              // n1*n2
  int plan;             // registry index of the length-n2 row plan
  int pitch;
  int real_split;       // 1: REAL master epilogue, 0: plain complex rows
  float2 const *rootD;  // REAL only: W_{2*nc}^{n1*k2} = exp(-i*pi*k2/n2), k2 < n2
  float2 *spec;         // [block][spec_stride]
  long spec_stride;
  int mid_ld;           // see Pass1Args
};

__global__ void __launch_bounds__(kFwdThreads, 2) fwd_rows_kernel(Pass2Args const a) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  float2 *tile = reinterpret_cast<float2 *>(smem_raw);  // [kTile][pitch]
  TilePlan const &pl = c_plans[a.plan];
  int const tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  int const blk = blockIdx.y;
  int const item0 = blockIdx.x * (a.real_split ? kTile / 2 : kTile);  // items per CTA: 4 row pairs or 8 plain rows

  // ---- each warp streams its own row into its column (contiguous 8-byte loads) ------------
  {
    RowItem const it = row_item(item0 + (a.real_split ? warp >> 1 : warp), a.n1, a.real_split);
    int row = -1;
    if (a.real_split) {
      if ((warp & 1) == 0 && it.kind != kRowEmpty) row = it.row_a;
      if ((warp & 1) == 1 && it.kind == kRowPair) row = it.row_b;
    } else if (it.kind == kRowPlain) {
      row = it.row_a;
    }
    if (row >= 0) {
      float2 const *src = a.mid + (long)blk * a.nc + (long)row * a.n2;
      float2 *colp = tile + warp * a.pitch;
      constexpr int U = 8;
      int n2 = lane;
      for (; n2 + (U - 1) * 32 < a.n2; n2 += U * 32) {
        float2 w[U];
#pragma unroll
        for (int u = 0; u < U; u++) w[u] = __ldg(src + n2 + u * 32);
#pragma unroll
        for (int u = 0; u < U; u++) colp[n2 + u * 32] = w[u];
      }
      for (; n2 < a.n2; n2 += 32) colp[n2] = __ldg(src + n2);
      __syncwarp();
      tile_fft<false>(pl, colp, lane, 32, [] { __syncwarp(); });
    }
  }
  __syncthreads();

  float2 *spec = a.spec + (long)blk * a.spec_stride;
  if (!a.real_split) {
    // plain rows: X[k1 + n1*k2] = Z; 8 adjacent rows -> 64-byte segments
    int const i = tid % kTile, q0 = tid / kTile;
    RowItem const it = row_item(item0 + i, a.n1, false);
    if (it.kind == kRowPlain) {
      float2 const *colp = tile + i * a.pitch;
      constexpr int V = 4, QS = kFwdThreads / kTile;
      int k2 = q0;
      for (; k2 + (V - 1) * QS < a.n2; k2 += V * QS) {
        int slot[V];
        float2 v[V];
#pragma unroll
        for (int u = 0; u < V; u++) slot[u] = __ldg(pl.perm + k2 + u * QS);
#pragma unroll
        for (int u = 0; u < V; u++) v[u] = colp[slot[u]];
#pragma unroll
        for (int u = 0; u < V; u++) spec[(long)it.row_a + (long)a.n1 * (k2 + u * QS)] = v[u];
      }
      for (; k2 < a.n2; k2 += QS) spec[(long)it.row_a + (long)a.n1 * k2] = colp[__ldg(pl.perm + k2)];
    }
    return;
  }
  // ---- REAL epilogue: split the packed transform, 4 adjacent rows -> 32-byte segments -----
  int const i = tid % (kTile / 2), q0 = tid / (kTile / 2);
  int const qstep = kFwdThreads / (kTile / 2);
  RowItem const it = row_item(item0 + i, a.n1, true);
  if (it.kind == kRowEmpty) return;
  float2 const *ca = tile + (2 * i) * a.pitch;
  float2 const *cb = (it.kind == kRowPair) ? tile + (2 * i + 1) * a.pitch : ca;
  float2 const rootC = unit_root_f(it.row_a, 2 * a.nc);  // W_N^{k1}
  int const kend = (it.kind == kRowPair) ? a.n2 : (it.kind == kRowSelf0 ? a.n2 / 2 + 1 : (a.n2 + 1) / 2);
  constexpr int V = 4;
  auto partner = [&](int k2) { return (it.kind == kRowSelf0) ? (k2 == 0 ? 0 : a.n2 - k2) : a.n2 - 1 - k2; };
  auto emit = [&](int k2, float2 za, float2 zb, float2 rd) {
    long const k = (long)it.row_a + (long)a.n1 * k2;
    float2 const w = cmul(rootC, rd);  // W_N^k
    float2 const E = make_float2(0.5f * (za.x + zb.x), 0.5f * (za.y - zb.y));
    float2 const O = make_float2(0.5f * (za.x - zb.x), 0.5f * (za.y + zb.y));
    float2 const P = cmul(w, O);
    // X[k] = E - i*P ;  X[Nc-k] = conj(E + i*P)
    spec[k] = make_float2(E.x + P.y, E.y - P.x);
    long const km = a.nc - k;
    if (km != k) spec[km] = make_float2(E.x - P.y, -(E.y + P.x));
  };
  int k2 = q0;
  for (; k2 + (V - 1) * qstep < kend; k2 += V * qstep) {
    int sa[V], sb[V];
    float2 za[V], zb[V], rd[V];
#pragma unroll
    for (int u = 0; u < V; u++) {
      sa[u] = __ldg(pl.perm + k2 + u * qstep);
      sb[u] = __ldg(pl.perm + partner(k2 + u * qstep));
      rd[u] = __ldg(a.rootD + k2 + u * qstep);
    }
#pragma unroll
    for (int u = 0; u < V; u++) {
      za[u] = ca[sa[u]];
      zb[u] = cb[sb[u]];
    }
#pragma unroll
    for (int u = 0; u < V; u++) emit(k2 + u * qstep, za[u], zb[u], rd[u]);
  }
  for (; k2 < kend; k2 += qstep)
    emit(k2, ca[__ldg(pl.perm + k2)], cb[__ldg(pl.perm + partner(k2))], __ldg(a.rootD + k2));
}

// ---------------------------------------------------------------------------------------------
// apply_notch_filters (filter.c:464-474): per listed bin a double-complex EWMA that is
// subtracted from the bin.  One thread per notch entry, blocks in time order.
struct NotchDev {
  int bin;
  int pad;
  double re, im;   // state
  double alpha;
};
__global__ void notch_kernel(NotchDev *list, int n, int sequential, float2 *spec, long spec_stride, int nblocks) {
  int const i = blockIdx.x * blockDim.x + threadIdx.x;
  if (sequential) {  // duplicate bins in the list: keep the reference's in-order semantics
    if (i != 0) return;
    for (int b = 0; b < nblocks; b++)
      for (int e = 0; e < n; e++) {
        float2 *p = spec + (long)b * spec_stride + list[e].bin;
        float2 v = *p;
        list[e].re += list[e].alpha * ((double)v.x - list[e].re);
        list[e].im += list[e].alpha * ((double)v.y - list[e].im);
        *p = make_float2((float)((double)v.x - list[e].re), (float)((double)v.y - list[e].im));
      }
    return;
  }
  if (i >= n) return;
  NotchDev nd = list[i];
  for (int b = 0; b < nblocks; b++) {
    float2 *p = spec + (long)b * spec_stride + nd.bin;
    float2 v = *p;
    nd.re += nd.alpha * ((double)v.x - nd.re);
    nd.im += nd.alpha * ((double)v.y - nd.im);
    *p = make_float2((float)((double)v.x - nd.re), (float)((double)v.y - nd.im));
  }
  list[i].re = nd.re;
  list[i].im = nd.im;
}

}  // namespace kfft
