// static_kernels_v2.cuh -- forward passes with the first and last butterfly stage fused into the
// global load / store.
//
// The v1 kernels are bound by the L1/shared-memory LSU data pipe: an
// in-shared-memory DIF moves every point through shared memory twice per stage plus once on the
// way in and once on the way out.  Here the lanes of a warp are interleaved over the tile's 8
// columns (lane = 8*u' + column), so a warp-wide global access still covers 8 adjacent columns
// (one 32/64-byte segment per row) -- which lets
//   * stage 0 read its R0 inputs straight from global memory (int16 -> float in registers),
//   * the last stage write its outputs (times the inter-pass twiddle / through the real split)
//     straight to global memory,
// leaving one store, one load+store and one load per point in shared memory instead of eight
// accesses.  With 288 threads the 8 x 1296 tile divides evenly (864 and 1152 butterflies per
// stage): no idle lanes.  Column pitch = 2 mod 16 keeps every access pattern here free of bank
// conflicts (8 even column offsets x 2 consecutive butterflies per half-warp).
#pragma once
#include "static_kernels.cuh"

namespace kfft {

using S1250v2 = SPlan<1250, 10, 25, 5>;

// twiddles W^{j*t}, t = 1..R-1, for one butterfly: 4 table loads + products (see static_stage TWC)
template <int R, int S> __device__ __forceinline__ void load_stage_twiddles(float2 const *twi, int j, float2 (&w)[R]) {
#pragma unroll
  for (int t = 1; t < R; t <<= 1) w[t] = twi[(t - 1) * S + j];
#pragma unroll
  for (int t = 3; t < R; t++) {
    int const hb = (t >= 16) ? 16 : (t >= 8) ? 8 : (t >= 4) ? 4 : 2;
    if (t != hb) w[t] = cmul(w[hb], w[t - hb]);
  }
}

// pass-2 work item p of the list kgpu.cu builds (row 0 | pairs (k1, n1-k1) | row n1/2 | padding),
// computed instead of loaded: the row fetch of a CTA does not wait for a table read
__device__ __forceinline__ RowItem row_item(int p, int n1, bool real_split) {
  RowItem it;
  it.pad = 0;
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

struct ColsV2Tables {
  float2 const *twU;  // [n2][144]  W_nc^{n2 * kbase(u)}, kbase(u) = u/12 + 12*(u%12)   (u = t0*12 + t1)
  float2 const *twT;  // [n2][9]    W_nc^{n2 * 144 * t2}
};

// ------------------------------------------------------------------ pass 1: columns -----------
// FMT 0: float pairs; 1: int16 pairs; 2: int16 pairs + de-randomise + energy/clip statistics.
// N2C: number of columns as a compile-time constant (0 = read it from the arguments): with it every
// global address of a thread is one base register plus an immediate.
// int16 pair -> two floats.  `(float)(short)` compiles to I2F.S16, which issues through the MIO
// queue to the quarter-rate conversion unit -- the queue the 36 loads and 72 shared-memory accesses
// of a thread also need (ncu: mio_throttle was the top stall of this kernel).  Sign-extend with
// PRMT / SHF and convert with I2FP.F32.S32 on the integer pipe instead.
__device__ __forceinline__ void unpack_i16(int raw, int &lo, int &hi) {
  asm("prmt.b32 %0, %1, 0, 0x9910;" : "=r"(lo) : "r"(raw));  // bytes b0 b1 sign sign
  hi = raw >> 16;
}
__device__ __forceinline__ float i32_to_f32(int v) {
  float f;
  asm("cvt.rn.f32.s32 %0, %1;" : "=f"(f) : "r"(v));
  return f;
}

// Round-1 column pass (12 x 12 x 9, two and a half trips through shared memory); fwd_cols_r36.cuh replaced it as the default,
// it stays selectable (kgpu_set_tuning(13, 4)) as the A/B partner.  Variants tried on it and removed again: 16- and 6-column
// tiles, a TMA tensor store of the tile, table twiddles, an L2 prefetch of the next block's input.
template <int FMT, int N2C = 0>
__global__ void __launch_bounds__(288, 2) fwd_cols_v2(Pass1Args const a, ColsV2Tables const tb) {
  using P = SPlan<1296, 12, 12, 9>;
  constexpr int TC = 8;
  constexpr int N1 = 1296, PITCH = 1298, UPI = 36 /*butterflies per column per iteration*/;
  constexpr int R0 = 12, S0 = 108, R1 = 12, NSUB1 = 108, S1 = 9, R2 = 9;
  constexpr int XS = 1, CS = PITCH;  // element (column c, index X) at tile[X*XS + c*CS]
  extern __shared__ __align__(16) unsigned char smem_raw[];
  float2 *tile = reinterpret_cast<float2 *>(smem_raw);  // [8][PITCH]
  float2 *s_tw = tile + TC * PITCH + (TC * PITCH) % 2;  // stage twiddles (1287 entries, padded to 1288), 16-byte aligned
  float2 *s_twT = s_tw + 1288;                          // [TC][9] (padded to 10 TC)
  __shared__ __align__(8) uint64_t tbar;
  TilePlan const &pl = c_plans[a.plan];
  int const tid = threadIdx.x;
  int const c = tid % TC, ul = tid / TC;  // column of the tile, butterfly lane 0..35
  int const c0 = blockIdx.x * TC, blk = blockIdx.y;
  int const n2 = N2C ? N2C : a.n2;
  long const nc = N2C ? (long)N1 * N2C : a.nc;
  unsigned long long *dbg = a.dbg ? a.dbg + 6 * ((long)blockIdx.y * gridDim.x + blockIdx.x) : nullptr;
  if (dbg && tid == 0) {
    dbg[0] = gtimer();
    dbg[5] = sm_id();
  }
  int const ncols = min(TC, n2 - c0);
  bool const col_ok = c < ncols;
  int const n2g = c0 + c;
  float2 *mycol = tile + c * CS;
  if (tid == 0) {
    mbar_init(&tbar, 1);
    mbar_fence_init();
    mbar_expect_tx(&tbar, 1288 * 8 + 10 * TC * 8);
    bulk_g2s(s_tw, pl.tw, 1288 * 8, &tbar);
    bulk_g2s(s_twT, tb.twT + (long)c0 * 9, 10 * TC * 8, &tbar);  // table padded by 16 columns + 16 entries
  }
  __syncthreads();  // barrier initialised before anybody waits on it
  // inter-pass factors B'(n2, u) for this thread's four stage-2 butterflies: issued now, used last
  float2 twU[4];
#pragma unroll
  for (int it = 0; it < 4; it++)
    twU[it] = col_ok ? ldg_stream_f2(tb.twU + (long)n2g * 144 + ul + UPI * it) : make_float2(1.f, 0.f);

  // ---- stage 0 fused with the load: x[j + 108 m], m = 0..11, straight from global ------------
  unsigned long long energy = 0;
  unsigned int clips = 0;
  if (col_ok) {
    // row of butterfly j = ul + 36 it, input m: j + 108 m  ->  element (ul + 36 it + 108 m) * n2
    if (FMT == 0) {
      float2 const *src = reinterpret_cast<float2 const *>(a.in) + (long)blk * a.hop + n2g + (long)ul * n2;
      float2 x[3][R0];
#pragma unroll
      for (int it = 0; it < 3; it++) {
#pragma unroll
        for (int m = 0; m < R0; m++) x[it][m] = ldg_stream_f2(src + (long)(UPI * it + S0 * m) * n2);
      }
      mbar_wait(&tbar, 0);
#pragma unroll
      for (int it = 0; it < 3; it++) {
        int const j = ul + UPI * it;
        Dft<R0, false>::run(x[it]);
        float2 w[R0];
        load_stage_twiddles<R0, S0>(s_tw, j, w);
        float2 *d = mycol + j * XS;
        d[0] = x[it][0];
#pragma unroll
        for (int t = 1; t < R0; t++) d[t * S0 * XS] = cmul(x[it][t], w[t]);
      }
    } else {
      int const *src = reinterpret_cast<int const *>(a.in) + (long)blk * a.hop + n2g + (long)ul * n2;
      int raw[3][R0];
#pragma unroll
      for (int it = 0; it < 3; it++) {
#pragma unroll
        for (int m = 0; m < R0; m++) raw[it][m] = ldg_stream_b32(src + (long)(UPI * it + S0 * m) * n2);
      }
      mbar_wait(&tbar, 0);
#pragma unroll
      for (int it = 0; it < 3; it++) {
        int const j = ul + UPI * it;
        float2 x[R0];
#pragma unroll
        for (int m = 0; m < R0; m++) {
          int lo, hi;
          unpack_i16(raw[it][m], lo, hi);
          if (FMT == 2) {
            if (a.derandomize) {  // lsb set -> flip bits 1..15 (rx888.c:707-712); on the sign-extended word: bits 1..31
              lo ^= (lo & 1) ? 0xfffffffe : 0;
              hi ^= (hi & 1) ? 0xfffffffe : 0;
            }
            if (a.stats && (long)(j + S0 * m) * n2 + n2g >= a.first_new) {
              energy += (unsigned long long)(lo * lo) + (unsigned long long)(hi * hi);
              clips += (lo > 32766 || lo < -32766) + (hi > 32766 || hi < -32766);
            }
          }
          x[m] = make_float2(i32_to_f32(lo), i32_to_f32(hi));  // the int16 scale rides on the inter-pass twiddle
        }
        Dft<R0, false>::run(x);
        float2 w[R0];
        load_stage_twiddles<R0, S0>(s_tw, j, w);
        float2 *d = mycol + j * XS;
        d[0] = x[0];
#pragma unroll
        for (int t = 1; t < R0; t++) d[t * S0 * XS] = cmul(x[t], w[t]);
      }
    }
  } else {
    mbar_wait(&tbar, 0);
  }
  if (FMT == 2 && a.stats) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      energy += __shfl_xor_sync(0xffffffffu, energy, o);
      clips += __shfl_xor_sync(0xffffffffu, clips, o);
    }
    if ((tid & 31) == 0 && (energy | clips)) {
      atomicAdd(&a.stats[blk].energy, energy);
      atomicAdd(&a.stats[blk].clips, clips);
    }
  }
  __syncthreads();
  if (dbg && tid == 0) dbg[1] = gtimer();

  // ---- stage 1 in shared memory: 12 blocks of 108, stride 9 -----------------------------------
  if (col_ok) {
    float2 const *tw1 = s_tw + P::tw_off(1);
    // j = u mod 9 with u = ul + 36 it: the same for the three butterflies -> twiddles formed once
    int const b0 = ul / S1, j = ul - b0 * S1;
    float2 w[R1];
    load_stage_twiddles<R1, S1>(tw1, j, w);
#pragma unroll 1
    for (int it = 0; it < 3; it++) {
      float2 *p = mycol + ((b0 + (UPI / S1) * it) * NSUB1 + j) * XS;
      float2 x[R1];
#pragma unroll
      for (int m = 0; m < R1; m++) x[m] = p[m * S1 * XS];
      Dft<R1, false>::run(x);
      p[0] = x[0];
#pragma unroll
      for (int t = 1; t < R1; t++) p[t * S1 * XS] = cmul(x[t], w[t]);
    }
  }
  __syncthreads();
  if (dbg && tid == 0) dbg[2] = gtimer();

  // ---- stage 2 fused with the store: X[k1] * W_nc^{n2 k1} -> mid[k1][n2] ------------------------
  {
    float2 wT[R2];
#pragma unroll
    for (int t = 0; t < R2; t++) wT[t] = s_twT[c * 9 + t];
    // u = ul + 36 it = t0*12 + t1 -> k1 = kbase + 144 t2 with kbase = t0 + 12 t1 = kbase(ul) + 3 it
    int const kb0 = ul / 12 + 12 * (ul % 12);
    float2 *dst = a.mid + (long)blk * nc + n2g + (long)kb0 * n2;
    float const os = a.out_scale;
#pragma unroll
    for (int it = 0; it < 4; it++) {
      if (col_ok) {
        int const u = ul + UPI * it;
        float2 *p = mycol + u * R2 * XS;
        float2 x[R2];
#pragma unroll
        for (int m = 0; m < R2; m++) x[m] = p[m * XS];
        Dft<R2, false>::run(x);
        float2 const wb = make_float2(twU[it].x * os, twU[it].y * os);
#pragma unroll
        for (int t = 0; t < R2; t++) {
          dst[(long)(3 * it + 144 * t) * n2] = cmul(x[t], cmul(wb, wT[t]));
        }
      }
    }
  }
  if (dbg && tid == 0) dbg[3] = gtimer();
}

// ------------------------------------------------------------------ pass 2: rows --------------
// 1250 = 10 * 25 * 5.  Rows arrive by TMA; stages 0 and 1 run in shared memory with the lanes
// interleaved over the 8 columns; the radix-5 last stage is fused with the real split: the thread
// that owns butterfly u of row k1 also takes butterfly 249-u of the mirror row N1-k1, which holds
// exactly the partners Z[Nc-k] of its five outputs (digit complement: 1249-k2 <-> (9-t0,24-t1,4-t2)).
// N1C: row count as a compile-time constant (0 = from the arguments).  HALVED: the 1/2 of the real
// split was already folded into the column pass (Pass1Args::out_scale).
// W_1250^{32 it t} literals for stage 0 of the row pass
__device__ constexpr float kRowsTw0[3][4][2] = {
    {{9.870916009e-01f, -1.601568460e-01f}, {9.486995935e-01f, -3.161789477e-01f}, {8.000617623e-01f, -5.999176502e-01f}, {2.801976204e-01f, -9.599423409e-01f}},
    {{9.486995935e-01f, -3.161789477e-01f}, {8.000617623e-01f, -5.999176502e-01f}, {2.801976204e-01f, -9.599423409e-01f}, {-8.429785967e-01f, -5.379471183e-01f}},
    {{8.858151436e-01f, -4.640382826e-01f}, {5.693368912e-01f, -8.221042752e-01f}, {-3.517109454e-01f, -9.361086488e-01f}, {-7.525988221e-01f, 6.584793329e-01f}},
};

// Stage-0 twiddles W^{j t}, j = ul + 32 it, are (4 values loaded once per thread) x (literal W^{32 it t}) instead of 4 loads per
// butterfly.  Variants tried and removed again: warp-per-column stages 0/1, stage-0 butterflies in groups of 2 / 4,
// stage-1 twiddles by products, a persistent double-buffered form.
// For REAL masters fwd_rows_r50.cuh is the default now; this kernel serves COMPLEX 1296 x 1250 masters and
// kgpu_set_tuning(10, 6).
template <bool REAL_SPLIT, int N1C = 0, bool HALVED = false>
__global__ void __launch_bounds__(256, 2) fwd_rows_v2(Pass2Args const a, FwdTables const tb) {
  using P = S1250v2;
  constexpr int N2 = 1250, PITCH = 1250, T = 256;
  constexpr int R0 = 10, S0 = 125, R1 = 25, NSUB1 = 125, S1 = 5, R2 = 5;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  float2 *tile = reinterpret_cast<float2 *>(smem_raw);  // [8][PITCH]
  float2 *s_tw = tile + 8 * PITCH;
  __shared__ __align__(8) uint64_t bars[8];
  __shared__ __align__(8) uint64_t tbar;
  TilePlan const &pl = c_plans[a.plan];
  int const tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  int const blk = a.rev ? gridDim.y - 1 - blockIdx.y : blockIdx.y;
  constexpr int IPC = REAL_SPLIT ? 4 : 8;
  int const n1 = N1C ? N1C : a.n1;
  int const item0 = blockIdx.x * IPC;
  unsigned long long *dbg = a.dbg ? a.dbg + 6 * ((long)blockIdx.y * gridDim.x + blockIdx.x) : nullptr;
  if (dbg && tid == 0) {
    dbg[0] = gtimer();
    dbg[5] = sm_id();
  }
  // which global row sits in which tile column
  auto row_of = [&](int col, int first = -1) -> int {
    RowItem const it = row_item((first < 0 ? item0 : first) + (REAL_SPLIT ? col >> 1 : col), n1, REAL_SPLIT);
    if (REAL_SPLIT) {
      if ((col & 1) == 0) return it.kind != kRowEmpty ? it.row_a : -1;
      return it.kind == kRowPair ? it.row_b : -1;
    }
    return it.kind == kRowPlain ? it.row_a : -1;
  };
  if (lane == 0) {  // warp w fetches column w: one TMA bulk copy of the whole (contiguous) row
    int const row = row_of(warp);
    mbar_init(&bars[warp], 1);
    if (warp == 0) mbar_init(&tbar, 1);
    mbar_fence_init();
    if (row >= 0) {
      mbar_expect_tx(&bars[warp], N2 * 8);
      bulk_g2s(tile + warp * PITCH, a.mid + ((long)blk * n1 + row) * a.mid_ld, N2 * 8, &bars[warp]);
    }
    if (warp == 0) {
      constexpr uint32_t TWB = (uint32_t)((static_tw_count<P>() + 1) & ~1) * 8u;
      mbar_expect_tx(&tbar, TWB);
      bulk_g2s(s_tw, pl.tw, TWB, &tbar);
    }
    if (a.pf_ctas) {  // pull the rows of a CTA that starts about one wave later into L2 now
      int const lin = blockIdx.y * gridDim.x + blockIdx.x + a.pf_ctas;
      int const ty = lin / gridDim.x, tx = lin - ty * gridDim.x;
      if (ty < gridDim.y) {
        int const prow = row_of(warp, tx * IPC);
        int const pblk = a.rev ? gridDim.y - 1 - ty : ty;
        if (prow >= 0) bulk_prefetch_l2(a.mid + ((long)pblk * n1 + prow) * a.mid_ld, N2 * 8);
      }
    }
  }
  __syncthreads();
  int const c = tid & 7, ul = tid >> 3;  // column, butterfly lane 0..31
  bool const col_ok = row_of(c) >= 0;
  mbar_wait(&tbar, 0);
  if (col_ok) mbar_wait(&bars[c], 0);
  if (dbg && tid == 0) dbg[1] = gtimer();
  float2 *mycol = tile + c * PITCH;

  // ---- stage 0: radix 10, stride 125 (125 butterflies per column) ------------------------------
  if (col_ok) {
    float2 base[4];
#pragma unroll
    for (int q = 0; q < 4; q++) base[q] = s_tw[((1 << q) - 1) * S0 + ul];  // W^{ul t}, t = 1, 2, 4, 8
#pragma unroll
    for (int it = 0; it < 4; it++) {
      int const j = ul + (T / 8) * it;
      if (it < 3 || j < S0) {
        float2 *p = mycol + j;
        float2 x[R0], w[R0];
#pragma unroll
        for (int m = 0; m < R0; m++) x[m] = p[m * S0];
#pragma unroll
        for (int q = 0; q < 4; q++)
          w[1 << q] = it == 0 ? base[q] : cmul(base[q], make_float2(kRowsTw0[it > 0 ? it - 1 : 0][q][0], kRowsTw0[it > 0 ? it - 1 : 0][q][1]));
        w[3] = cmul(w[2], w[1]);
        w[5] = cmul(w[4], w[1]);
        w[6] = cmul(w[4], w[2]);
        w[7] = cmul(w[4], w[3]);
        w[9] = cmul(w[8], w[1]);
        Dft<R0, false>::run(x);
        p[0] = x[0];
#pragma unroll
        for (int t = 1; t < R0; t++) p[t * S0] = cmul(x[t], w[t]);
      }
    }
  }
  __syncthreads();
  // ---- stage 1: radix 25, 10 blocks of 125, stride 5 (50 butterflies per column) ---------------
  if (col_ok) {
    float2 const *tw1 = s_tw + P::tw_off(1);
#pragma unroll 1
    for (int u = ul; u < N2 / R1; u += T / 8) {
      int const b = u / S1, j = u - b * S1;
      float2 *p = mycol + b * NSUB1 + j;
      float2 x[R1];
#pragma unroll
      for (int m = 0; m < R1; m++) x[m] = p[m * S1];
      Dft<R1, false>::run(x);
#pragma unroll
      for (int t = 1; t < R1; t++) x[t] = cmul(x[t], tw1[(t - 1) * S1 + j]);
#pragma unroll
      for (int t = 0; t < R1; t++) p[t * S1] = x[t];
    }
  }
  // REAL: table factors of this thread's four split butterflies, requested before the barrier
  int const i = tid & 3, uq = tid >> 2;  // item (row pair) 0..3, butterfly lane 0..63
  RowItem const it = row_item(item0 + i, n1, REAL_SPLIT);
  float2 rootC = make_float2(1.f, 0.f), rd[4];
  bool self_item = false;
  if (REAL_SPLIT) {
    self_item = it.kind == kRowSelf0 || it.kind == kRowSelfMid;
    if (it.kind == kRowPair) rootC = __ldg(tb.rootC + it.row_a);
#pragma unroll
    for (int q = 0; q < 4; q++) {
      int const u = uq + (T / 4) * q;
      int const t0 = u / 25, t1 = u - t0 * 25;
      rd[q] = (it.kind == kRowPair && u < N2 / R2) ? __ldg(a.rootD + t0 + 10 * t1) : make_float2(1.f, 0.f);
    }
  }
  int const has_self = __syncthreads_or(self_item);
  if (dbg && tid == 0) dbg[2] = gtimer();

  float2 *spec = a.spec + (long)blk * a.spec_stride;
  float const hf = HALVED ? 1.0f : 0.5f;
  if (!REAL_SPLIT) {
    // ---- stage 2 fused with the plain store: X[k1 + n1*k2], k2 = t0 + 10 t1 + 250 t2 ---------
    if (col_ok) {
      float2 *dst = spec + row_of(c);
#pragma unroll 1
      for (int u = ul; u < N2 / R2; u += T / 8) {
        int const t0 = u / 25, t1 = u - t0 * 25;
        int const kb = t0 + 10 * t1;
        float2 const *p = mycol + u * R2;
        float2 x[R2];
#pragma unroll
        for (int m = 0; m < R2; m++) x[m] = p[m];
        Dft<R2, false>::run(x);
        float2 *d = dst + (long)n1 * kb;
#pragma unroll
        for (int t = 0; t < R2; t++) d[(long)n1 * 250 * t] = x[t];
      }
    }
    return;
  }
  // ---- stage 2 fused with the real split -----------------------------------------------------
  // W_N^{n1*k2} = exp(-i*pi*k2/1250); k2 = kb + 250 t2 -> D[kb] * exp(-i*pi*t2/5)
  int const nc = N1C ? N1C * N2 : (int)a.nc;
  if (it.kind == kRowPair) {
    float2 const *ca = tile + (2 * i) * PITCH, *cb = tile + (2 * i + 1) * PITCH;
#pragma unroll
    for (int q = 0; q < 4; q++) {
      int const u = uq + (T / 4) * q;
      if (u >= N2 / R2) break;
      int const t0 = u / 25, t1 = u - t0 * 25;
      int const kb = t0 + 10 * t1;
      float2 const wkb = cmul(rootC, rd[q]);  // W_N^{row_a + n1*kb}
      float2 za[R2], zb[R2];
      float2 const *pa = ca + u * R2, *pb = cb + (N2 / R2 - 1 - u) * R2;
      float2 *pk = spec + (it.row_a + n1 * kb), *pm = spec + (nc - it.row_a - n1 * kb);  // k = row_a + n1 (kb + 250 t)
#pragma unroll
      for (int m = 0; m < R2; m++) {
        za[m] = pa[m];
        zb[m] = pb[m];
      }
      Dft<R2, false>::run(za);
      Dft<R2, false>::run(zb);
#pragma unroll
      for (int t = 0; t < R2; t++) {
        float2 const A = za[t], B = zb[R2 - 1 - t];
        float2 const w = (t == 0) ? wkb : cmul(wkb, wroot<10>(t));  // exp(-i*pi*t/5) = W_10^t
        float2 const E = HALVED ? make_float2(A.x + B.x, A.y - B.y) : make_float2(0.5f * (A.x + B.x), 0.5f * (A.y - B.y));
        float2 const O = HALVED ? make_float2(A.x - B.x, A.y + B.y) : make_float2(0.5f * (A.x - B.x), 0.5f * (A.y + B.y));
        float2 const Pp = cmul(w, O);
        pk[(long)n1 * 250 * t] = make_float2(E.x + Pp.y, E.y - Pp.x);       // X[k]    = E - i P
        pm[-(long)n1 * 250 * t] = make_float2(E.x - Pp.y, -(E.y + Pp.x));  // X[Nc-k] = conj(E + i P)
      }
    }
  }
  // rows that pair with themselves (k1 = 0 and k1 = n1/2): last stage in place, then the v1 epilogue
  if (dbg && tid == 0) dbg[3] = gtimer();
  if (!has_self) return;  // CTA-uniform
  for (int s = 0; s < 4; s++) {
    RowItem const its = row_item(item0 + s, n1, true);
    if (its.kind != kRowSelf0 && its.kind != kRowSelfMid) continue;
    float2 *col = tile + (2 * s) * PITCH;
    for (int u = tid; u < N2 / R2; u += T) {
      float2 x[R2];
#pragma unroll
      for (int m = 0; m < R2; m++) x[m] = col[u * R2 + m];
      Dft<R2, false>::run(x);
#pragma unroll
      for (int m = 0; m < R2; m++) col[u * R2 + m] = x[m];
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
      float2 const A = col[static_slot<P>(k2)], B = col[static_slot<P>(k2m)];
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

// ------------------------------------------------------------------ channels ------------------
// Two-stage plans (600 = 24*25, 300 = 20*15): the bin-slice x response product is formed in
// registers as stage 0 loads its inputs, and the last stage writes the kept samples (the last
// olen of Ns, reference filter.c:357) straight to global memory: output n = u + R0*t, so the 24
// (20) lanes of a warp write contiguous runs.  Shared-memory traffic per point drops from eight
// accesses to three.  ISB channels need the whole product first and take the v1 path.
// OSC: instantiated twice so that the default path carries none of the oscillator's registers
// Tried and removed again: stage-0 twiddles by products (more registers, no gain), an L2 prefetch of a later CTA's slices.
template <class P, bool OSC = false>
__global__ void __launch_bounds__(kChanWarps * 32) chan_v2(ChanArgs const a) {
  static_assert(P::nst == 2, "two-stage plans only");
  extern __shared__ __align__(16) unsigned char smem_raw[];
  __shared__ __align__(8) uint64_t bars[kChanWarps];
  __shared__ __align__(8) uint64_t tbar;
  constexpr int NS = P::len, TOP = (NS + 1) / 2, R0 = P::rad(0), R1 = P::rad(1), S0 = NS / R0;
  static_assert(S0 == R1 && NS % 2 == 0, "plan shape");
  constexpr int XS = NS + 4;
  int const lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int const oi = blockIdx.x * kChanWarps + warp;
  float2 *s_tw = reinterpret_cast<float2 *>(smem_raw) + kChanWarps * (NS + XS);
  bool const active = oi < a.norder;
  ChanDesc d;
  d.plan = -1;
  if (active) d = a.desc[a.order ? a.order[oi] : a.chan_base + oi];
  if (threadIdx.x == 0) {
    int p0 = -1;
    for (int w = 0; w < kChanWarps && p0 < 0; w++) {
      int const o = blockIdx.x * kChanWarps + w;
      if (o < a.norder) p0 = a.desc[a.order ? a.order[o] : a.chan_base + o].plan;
    }
    mbar_init(&tbar, 1);
    mbar_fence_init();
    if (p0 >= 0) {
      constexpr uint32_t TWB = (uint32_t)((static_tw_count<P>() + 1) & ~1) * 8u;
      mbar_expect_tx(&tbar, TWB);
      bulk_g2s(s_tw, c_plans[p0].tw, TWB, &tbar);
    }
  }
  __syncthreads();
  if (!active || d.plan < 0) return;
  int const blk = blockIdx.y;
  float2 *col = reinterpret_cast<float2 *>(smem_raw) + warp * (NS + XS);
  float2 *xs = col + NS;
  float2 const *X = a.spec + (long)blk * a.spec_stride;
  float2 const *R = a.resp + d.resp_off;
  float2 *dst = a.out + (long)blk * a.out_stride + d.out_off;
  if (d.ncopy <= 0) {
    for (int i = lane; i < d.olen; i += 32) dst[i] = make_float2(0.f, 0.f);
    if ((d.flags & kChanOsc) && a.power && lane == 0) a.power[(long)blk * a.power_stride + (a.order ? a.order[oi] : a.chan_base + oi)] = 0.f;
    mbar_wait(&tbar, 0);  // the CTA's twiddle copy targets this CTA's shared memory: never retire with it in flight
    return;
  }
  int const qlo = d.dir > 0 ? d.q0 : d.q0 - (d.ncopy - 1);
  bool const wraps = a.wrap && (d.q0 + d.ncopy > a.m_bins);
  int const qa = qlo & ~1;
  if (!wraps) {
    int const qhi = qlo + d.ncopy - 1;
    uint32_t const nx = (uint32_t)(((qhi - qa + 1) + 1) & ~1);
    if (lane == 0) {
      mbar_init(&bars[warp], 1);
      mbar_fence_init();
      mbar_expect_tx(&bars[warp], nx * 8 + NS * 8);
      bulk_g2s(xs, X + qa, nx * 8, &bars[warp]);
      bulk_g2s(col, R, NS * 8, &bars[warp]);
    }
    __syncwarp();
    mbar_wait(&bars[warp], 0);
  } else {
    for (int i = lane; i < NS; i += 32) col[i] = __ldg(R + i);
    for (int u = lane; u < d.ncopy; u += 32) {
      int q = d.q0 + u;
      if (q >= a.m_bins) q -= a.m_bins;
      xs[u] = __ldg(X + q);
    }
    __syncwarp();
  }
  mbar_wait(&tbar, 0);
  auto product = [&](int wp) -> float2 {  // S[wp] = X[q(wp)] * R[wp], zero outside the master (filter.c:728-911)
    int t = wp - TOP;
    if (t < 0) t += NS;
    int const u = t - d.zlead;
    bool const live = (u >= 0 && u < d.ncopy && wp != TOP);
    int const xi = wraps ? u : (d.q0 + d.dir * u - qa);
    float2 x = xs[live ? xi : 0];
    if (d.dir < 0) x.y = -x.y;
    float2 const v = cmul(x, col[wp]);
    return live ? v : make_float2(0.f, 0.f);
  };
  if (d.flags & kChanIsb) {  // ISB: whole product in shared memory first, then the plain two stages
    for (int wp = lane; wp < NS; wp += 32) col[wp] = product(wp);  // same lane reads R[wp] and writes S[wp]
    __syncwarp();
    for (int p = 1 + lane; p < NS / 2; p += 32) {
      float2 const pos = col[p], neg = col[NS - p];
      col[p] = make_float2(pos.x + neg.x, pos.y - neg.y);
      col[NS - p] = make_float2(neg.x - pos.x, neg.y + pos.y);
    }
    if (lane == 0) {
      col[0] = make_float2(0.f, 0.f);
      col[TOP] = make_float2(0.f, 0.f);
    }
    __syncwarp();
    static_stage<P, true, 0, true, 1>(col, s_tw, lane);
    __syncwarp();
  } else if (lane < S0) {
    // ---- stage 0 with the product formed on the fly ------------------------------------------
    float2 x[R0];
#pragma unroll
    for (int m = 0; m < R0; m++) x[m] = product(lane + S0 * m);
    Dft<R0, true>::run(x);
    col[lane] = x[0];
#pragma unroll
    for (int t = 1; t < R0; t++) col[lane + S0 * t] = cmulc(x[t], s_tw[(t - 1) * S0 + lane]);
  }
  __syncwarp();
  // ---- stage 1 fused with the store: y[n], n = u + R0*t, keep n >= NS - olen ---------------------
  bool const osc = OSC && (d.flags & kChanOsc) != 0;  // warp-uniform
  float pw = 0.f;
  int const ci = a.order ? a.order[oi] : a.chan_base + oi;
  if (lane < R0) {
    float2 x[R1];
#pragma unroll
    for (int m = 0; m < R1; m++) x[m] = col[R1 * lane + m];
    Dft<R1, true>::run(x);
    int const first = NS - d.olen;
    if (!OSC || !osc) {
#pragma unroll
      for (int t = 0; t < R1; t++) {
        int const n = lane + R0 * t;
        if (n >= first) dst[n - first] = x[t];
      }
    } else if (OSC) {  // fine-tuning rotation + block power fused into the store (radio.c:1476-1501, :1515-1520)
      ChanAux const ax = a.aux[ci];
      long const k = a.block0 + blk - ax.osc_epoch;
#pragma unroll
      for (int t = 0; t < R1; t++) {
        int const n = lane + R0 * t;
        if (n >= first) {
          float2 const v = osc_rotate(x[t], osc_phase_cycles(ax, k, d.olen, n - first));
          dst[n - first] = v;
          pw += v.x * v.x + v.y * v.y;
        }
      }
    }
  }
  if (OSC && osc && a.power) {
    pw = warp_sum(pw);
    if (lane == 0) a.power[(long)blk * a.power_stride + ci] = pw / (float)d.olen;
  }
}

}  // namespace kfft
