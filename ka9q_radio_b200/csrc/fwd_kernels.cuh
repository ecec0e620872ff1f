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

// The generic pair is written once: fwd_cols_body here, the row pass in fwd_rows_body.cuh.  fwd_cols_kernel /
// fwd_rows_kernel run them on registry plans with the radix switch of every other kernel; the extended pair
// (fwd_cols_ext / fwd_rows_ext) runs them on plans the master passes by value, with EXT adding the prime radices
// 11 .. 23 to tile_fft.
template <int FMT /*0: float pairs, 1: int16 pairs*/, bool EXT>
__device__ __forceinline__ void fwd_cols_body(Pass1Args const &a, TilePlan const &pl) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  float2 *tile = reinterpret_cast<float2 *>(smem_raw);             // [kTile][pitch]
  int const rows_per_it = kFwdThreads / kTile;                      // 32
  int const nit = (a.n1 + rows_per_it - 1) / rows_per_it;
  float2 *twA = tile + kTile * a.pitch;                             // [kTile][nit]

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
  if (warp < ncols) tile_fft<false, EXT>(pl, tile + warp * a.pitch, lane, 32, [] { __syncwarp(); });
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

template <int FMT>
__global__ void __launch_bounds__(kFwdThreads, 2) fwd_cols_kernel(Pass1Args const a) {
  fwd_cols_body<FMT, false>(a, c_plans[a.plan]);
}
template <int FMT>
__global__ void __launch_bounds__(kFwdThreads, 2) fwd_cols_ext(Pass1Args const a, __grid_constant__ TilePlan const pl) {
  fwd_cols_body<FMT, true>(a, pl);
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
__host__ __device__ __forceinline__ RowItem row_item(int p, int n1, bool real_split) {
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
  TilePlan const &pl = c_plans[a.plan];
#define KFFT_ROWS_EXT false
#include "fwd_rows_body.cuh"
#undef KFFT_ROWS_EXT
}
__global__ void __launch_bounds__(kFwdThreads, 2) fwd_rows_ext(Pass2Args const a, __grid_constant__ TilePlan const pl) {
#define KFFT_ROWS_EXT true
#include "fwd_rows_body.cuh"
#undef KFFT_ROWS_EXT
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
