// fwd_rows_r50.cuh -- row pass of a REAL master's n1 x 1250 two-pass transform with TWO fat stages (50 x 25) and the
// real-input split fused into the second.
//
// fwd_rows_v2 (10 x 25 x 5) moves every point through shared memory five times (stage 0 load + store, stage 1 load + store,
// stage 2 load) on top of the TMA fill and is paced by exactly that traffic.  1250 = 50 x 25 needs three:
//   stage 0, in place:  butterfly j < 25 takes x[j + 25 m], m < 50; output t, times W_1250^{j t}, goes back to x[25 t + j];
//   stage 1 + split:    the thread of (row pair i, sub-transform t) transforms block t of row a = k1 and block 49 - t of
//                       row b = n1 - k1 (25 contiguous points each).  Output k' of the first is Z[k], k = k1 + n1 (t + 50 k'),
//                       and output 24 - k' of the second is Z[nc - k]: the split X[k] = E - i W_N^k O, X[nc-k] = conj(E + i W_N^k O)
//                       happens in registers and both go straight to the spectrum.
// Thread budget: 8 rows x 25 butterflies = 4 pairs x 50 sub-transforms = 200 threads, every one busy in both stages; a
// 50-point butterfly (Good-Thomas 2 x 25) and two 25-point ones are ~100 live data registers either way.
// Rows k1 = 0 and k1 = n1/2 pair with themselves: two CTAs per block take the slow path at the end (as in fwd_rows_v2).
#pragma once
#include "fwd_2s.cuh"

namespace kfft {

struct RowsR50Shape {
  static constexpr int N2 = 1250, RC = 50, RD = 25, T = 200, PITCH = 1250;  // 1250 = 2 (mod 16)
  static constexpr int NP0 = Pow<RC>::NP;                                   // 13 loaded powers
  static constexpr int TW0 = (NP0 * RD + 1) & ~1;
  static constexpr size_t smem = sizeof(float2) * (size_t)(8 * PITCH + TW0);
};

template <int N1C, bool HALVED>
__global__ void __launch_bounds__(200, 2) fwd_rows_r50(Pass2Args const a, FwdTables const tb, float2 const *tw0) {
  using S = RowsR50Shape;
  constexpr int N2 = S::N2, RC = S::RC, RD = S::RD, PITCH = S::PITCH, T = S::T;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  float2 *tile = reinterpret_cast<float2 *>(smem_raw);  // [8][PITCH]: column 2i = row a of item i, 2i + 1 = row b
  float2 *s_tw0 = tile + 8 * PITCH;                     // [13][25]  W_1250^{j e}
  __shared__ __align__(8) uint64_t bars[8];
  __shared__ __align__(8) uint64_t tbar;
  int const tid = threadIdx.x;
  int const blk = a.rev ? gridDim.y - 1 - blockIdx.y : blockIdx.y;
  int const n1 = N1C ? N1C : a.n1;
  int const item0 = blockIdx.x * 4;
  auto row_of = [&](int col, int first = -1) -> int {
    RowItem const it = row_item((first < 0 ? item0 : first) + (col >> 1), n1, true);
    if ((col & 1) == 0) return it.kind != kRowEmpty ? it.row_a : -1;
    return it.kind == kRowPair ? it.row_b : -1;
  };
  if (tid < 8) {  // one TMA bulk copy per (contiguous) row
    int const row = row_of(tid);
    mbar_init(&bars[tid], 1);
    if (tid == 0) mbar_init(&tbar, 1);
    mbar_fence_init();
    if (row >= 0) {
      mbar_expect_tx(&bars[tid], N2 * 8);
      bulk_g2s(tile + tid * PITCH, a.mid + ((long)blk * n1 + row) * a.mid_ld, N2 * 8, &bars[tid]);
    }
    if (tid == 0) {
      mbar_expect_tx(&tbar, S::TW0 * 8);
      bulk_g2s(s_tw0, tw0, S::TW0 * 8, &tbar);
    }
    if (a.pf_ctas) {  // pull the rows of a CTA that starts later into L2 now
      int const lin = blockIdx.y * gridDim.x + blockIdx.x + a.pf_ctas;
      int const ty = lin / gridDim.x, tx = lin - ty * gridDim.x;
      if (ty < gridDim.y) {
        int const prow = row_of(tid, tx * 4);
        int const pblk = a.rev ? gridDim.y - 1 - ty : ty;
        if (prow >= 0) bulk_prefetch_l2(a.mid + ((long)pblk * n1 + prow) * a.mid_ld, N2 * 8);
      }
    }
  }
  __syncthreads();
  // ---- stage 0: radix 50, in place ----------------------------------------------------------------------------------
  {
    int const c = tid & 7, j = tid >> 3;  // row of the tile, butterfly 0..24
    bool const ok = row_of(c) >= 0;
    mbar_wait(&tbar, 0);
    if (ok) {
      mbar_wait(&bars[c], 0);
      float2 *p = tile + c * PITCH + j;
      float2 x[RC];
#pragma unroll
      for (int m = 0; m < RC; m++) x[m] = p[m * RD];
      Dft<RC, false>::run(x);
      Pow<RC> w;
      w.load(s_tw0 + j, RD);
      p[0] = x[0];
#pragma unroll
      for (int t = 1; t < RC; t++) p[t * RD] = cmul(x[t], w.get(t));
    }
  }
  // table factors of the split, requested before the barrier
  int const i = tid & 3, t = tid >> 2;  // item (row pair) 0..3, sub-transform 0..49
  RowItem const it = row_item(item0 + i, n1, true);
  bool const self_item = it.kind == kRowSelf0 || it.kind == kRowSelfMid;
  float2 wkb = make_float2(1.f, 0.f);
  if (it.kind == kRowPair) wkb = cmul(__ldg(tb.rootC + it.row_a), __ldg(a.rootD + t));  // W_N^{k1 + n1 t}
  int const has_self = __syncthreads_or(self_item);

  float2 *spec = a.spec + (long)blk * a.spec_stride;
  int const nc = N1C ? N1C * N2 : (int)a.nc;
  // ---- stage 1 fused with the real split --------------------------------------------------------------------------
  if (it.kind == kRowPair) {
    float2 za[RD], zb[RD];
    float2 const *pa = tile + (2 * i) * PITCH + t * RD, *pb = tile + (2 * i + 1) * PITCH + (RC - 1 - t) * RD;
#pragma unroll
    for (int m = 0; m < RD; m++) za[m] = pa[m];
    Dft<RD, false>::run(za);
#pragma unroll
    for (int m = 0; m < RD; m++) zb[m] = pb[m];
    Dft<RD, false>::run(zb);
    float2 *pk = spec + (it.row_a + n1 * t), *pm = spec + (nc - it.row_a - n1 * t);  // k = k1 + n1 (t + 50 k')
#pragma unroll
    for (int k = 0; k < RD; k++) {
      float2 const A = za[k], B = zb[RD - 1 - k];
      float2 const w = (k == 0) ? wkb : cmul(wkb, wroot<2 * RD>(k));  // exp(-i pi (t + 50 k') / 1250) = D[t] W_50^{k'}
      float2 const E = HALVED ? make_float2(A.x + B.x, A.y - B.y) : make_float2(0.5f * (A.x + B.x), 0.5f * (A.y - B.y));
      float2 const O = HALVED ? make_float2(A.x - B.x, A.y + B.y) : make_float2(0.5f * (A.x - B.x), 0.5f * (A.y + B.y));
      float2 const Pp = cmul(w, O);
      pk[(long)n1 * RC * k] = make_float2(E.x + Pp.y, E.y - Pp.x);       // X[k]    = E - i P
      pm[-(long)n1 * RC * k] = make_float2(E.x - Pp.y, -(E.y + Pp.x));  // X[nc-k] = conj(E + i P)
    }
  }
  if (!has_self) return;  // CTA-uniform
  // ---- rows that pair with themselves (k1 = 0, k1 = n1/2): last stage in place, then a plain epilogue ------------------
  float const hf = HALVED ? 1.0f : 0.5f;
  for (int s = 0; s < 4; s++) {
    RowItem const its = row_item(item0 + s, n1, true);
    if (its.kind != kRowSelf0 && its.kind != kRowSelfMid) continue;
    float2 *col = tile + (2 * s) * PITCH;
    for (int u = tid; u < RC; u += T) {
      float2 x[RD];
#pragma unroll
      for (int m = 0; m < RD; m++) x[m] = col[u * RD + m];
      Dft<RD, false>::run(x);
#pragma unroll
      for (int m = 0; m < RD; m++) col[u * RD + m] = x[m];  // Z[u + 50 m]
    }
  }
  __syncthreads();
  for (int s = 0; s < 4; s++) {
    RowItem const its = row_item(item0 + s, n1, true);
    if (its.kind != kRowSelf0 && its.kind != kRowSelfMid) continue;
    float2 const *col = tile + (2 * s) * PITCH;
    float2 const rC = __ldg(tb.rootC + its.row_a);
    bool const self0 = its.kind == kRowSelf0;
    int const kend = self0 ? N2 / 2 + 1 : (N2 + 1) / 2;
    for (int k2 = tid; k2 < kend; k2 += T) {
      int const k2m = self0 ? (k2 == 0 ? 0 : N2 - k2) : N2 - 1 - k2;
      float2 const A = col[(k2 % RC) * RD + k2 / RC], B = col[(k2m % RC) * RD + k2m / RC];
      float2 const w = cmul(rC, __ldg(a.rootD + k2));
      float2 const E = make_float2(hf * (A.x + B.x), hf * (A.y - B.y));
      float2 const O = make_float2(hf * (A.x - B.x), hf * (A.y + B.y));
      float2 const Pp = cmul(w, O);
      int const k = its.row_a + n1 * k2;
      spec[k] = make_float2(E.x + Pp.y, E.y - Pp.x);
      if (nc - k != k) spec[nc - k] = make_float2(E.x - Pp.y, -(E.y + Pp.x));
    }
  }
}

}  // namespace kfft
