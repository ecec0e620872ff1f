// static_kernels_v3.cuh -- persistent forward passes.
//
// The per-CTA timeline of the v2 kernels (tools/phase_trace.py) shows each 8-row / 8-column tile
// waiting for its input (rows: TMA, columns: gather) before a single butterfly issues, and with two CTAs per SM about half of the time only one of them is past that
// wait.  Here one CTA stays on each SM and walks over the tiles:
//   cols  : 288 threads x 2 CTAs per SM as before, but the 36 raw int16 words a thread needs for the
//           NEXT tile are requested into the (by then dead) registers right after stage 0 of the
//           current tile, so the gather latency hides behind stages 1 and 2.
//   rows  : 512 threads, two 80 kB tile buffers; the rows of tile k+1 arrive by TMA while tile k
//           is being transformed, so all 16 warps always have butterflies to issue; the stage
//           twiddles, barriers and row-item decoding are set up once per CTA instead of per tile.
#pragma once
#include "static_kernels_v2.cuh"

namespace kfft {

__device__ __forceinline__ void mbar_arrive(uint64_t *bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void fence_proxy_async() { fence_proxy_async_smem(); }


// ------------------------------------------------------------------ pass 1: columns, persistent --
template <int FMT, int N2C>
__device__ __forceinline__ void cols_v3_request(int (&raw)[3][12], int const *src, int n2) {
#pragma unroll
  for (int it = 0; it < 3; it++) {
#pragma unroll
    for (int m = 0; m < 12; m++) raw[it][m] = ldg_stream_b32(src + (long)(36 * it + 108 * m) * (N2C ? N2C : n2));
  }
}

// int16 formats only (FMT 1, 2): the float format would need 72 look-ahead registers.
template <int FMT, int N2C = 0>
__global__ void __launch_bounds__(288, 2) fwd_cols_v3(Pass1Args const a, ColsV2Tables const tb, int tiles_per_block, int ntiles) {
  static_assert(FMT == 1 || FMT == 2, "int16 input");
  using P = SPlan<1296, 12, 12, 9>;
  constexpr int N1 = 1296, PITCH = 1298, T = 288, UPI = T / 8;
  constexpr int R0 = 12, S0 = 108, R1 = 12, NSUB1 = 108, S1 = 9, R2 = 9;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  float2 *tile = reinterpret_cast<float2 *>(smem_raw);  // [8][PITCH]
  float2 *s_tw = tile + 8 * PITCH;                      // stage twiddles (1287 entries, padded to 1288)
  float2 *s_twT = s_tw + 1288;                          // [8][9] (padded to 80), per tile
  __shared__ __align__(8) uint64_t tbar;
  TilePlan const &pl = c_plans[a.plan];
  int const tid = threadIdx.x;
  int const c = tid & 7, ul = tid >> 3;  // column of the tile, butterfly lane 0..35
  int const n2 = N2C ? N2C : a.n2;
  long const nc = N2C ? (long)N1 * N2C : a.nc;
  int const G = gridDim.x;
  if (tid == 0) {
    mbar_init(&tbar, 1);
    mbar_fence_init();
    mbar_expect_tx(&tbar, 1288 * 8);
    bulk_g2s(s_tw, pl.tw, 1288 * 8, &tbar);
  }
  __syncthreads();
  float2 *mycol = tile + c * PITCH;
  float2 const *tw1 = s_tw + P::tw_off(1);
  int const b0 = ul / S1, j1 = ul - b0 * S1;      // stage-1 butterfly of iteration 0
  int const kb0 = ul / 12 + 12 * (ul % 12);       // stage-2 output row of iteration 0
  int const *in = reinterpret_cast<int const *>(a.in);

  int raw[3][R0];
  int t = blockIdx.x;
  {
    int const blk = t / tiles_per_block, x = t - blk * tiles_per_block;
    if (t < ntiles && 8 * x + c < n2) cols_v3_request<FMT, N2C>(raw, in + (long)blk * a.hop + 8 * x + c + (long)ul * n2, n2);
  }
  mbar_wait(&tbar, 0);
  for (; t < ntiles; t += G) {
    int const blk = t / tiles_per_block, x = t - blk * tiles_per_block;
    int const mblk = a.mid_mod ? blk % a.mid_mod : blk;
    int const n2g = 8 * x + c;
    bool const col_ok = n2g < n2;
    // ---- stage 0 on the words requested one tile ago -------------------------------------------
    unsigned long long energy = 0;
    unsigned int clips = 0;
    if (col_ok) {
#pragma unroll
      for (int it = 0; it < 3; it++) {
        int const j = ul + UPI * it;
        float2 xv[R0];
#pragma unroll
        for (int m = 0; m < R0; m++) {
          short lo = (short)(raw[it][m] & 0xffff), hi = (short)((unsigned)raw[it][m] >> 16);
          if (FMT == 2) {
            if (a.derandomize) {  // lsb set -> flip bits 1..15 (rx888.c:707-712)
              lo ^= (short)((lo & 1) ? 0xfffe : 0);
              hi ^= (short)((hi & 1) ? 0xfffe : 0);
            }
            if (a.stats && (long)(j + S0 * m) * n2 + n2g >= a.first_new) {
              energy += (unsigned long long)((int)lo * lo) + (unsigned long long)((int)hi * hi);
              clips += (lo > 32766 || lo < -32766) + (hi > 32766 || hi < -32766);
            }
          }
          xv[m] = make_float2((float)lo, (float)hi);  // the int16 scale rides on the inter-pass twiddle
        }
        Dft<R0, false>::run(xv);
        float2 *d = mycol + j;
        d[0] = xv[0];
#pragma unroll
        for (int q = 1; q < R0; q++) d[q * S0] = cmul(xv[q], s_tw[(q - 1) * S0 + j]);  // twiddles straight from the table:
                                                                                      // the look-ahead words own the registers
      }
    }
    // ---- the next tile's words: in flight during stages 1 and 2 -----------------------------------
    {
      int const tn = t + G;
      int const blkn = tn / tiles_per_block, xn = tn - blkn * tiles_per_block;
      if (tn < ntiles && 8 * xn + c < n2) cols_v3_request<FMT, N2C>(raw, in + (long)blkn * a.hop + 8 * xn + c + (long)ul * n2, n2);
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
    // ---- stage 1 in shared memory: 12 blocks of 108, stride 9 -----------------------------------
    if (col_ok) {
#pragma unroll 1
      for (int it = 0; it < 3; it++) {
        float2 *p = mycol + (b0 + (UPI / S1) * it) * NSUB1 + j1;
        float2 xv[R1];
#pragma unroll
        for (int m = 0; m < R1; m++) xv[m] = p[m * S1];
        Dft<R1, false>::run(xv);
        p[0] = xv[0];
#pragma unroll
        for (int q = 1; q < R1; q++) p[q * S1] = cmul(xv[q], tw1[(q - 1) * S1 + j1]);
      }
    }
    // inter-pass factors of this tile: requested before the barrier, used after it
    float2 twU[4];
    if (col_ok) {
#pragma unroll
      for (int it = 0; it < 4; it++) twU[it] = __ldg(tb.twU + (long)n2g * 144 + ul + UPI * it);
    }
    if (tid < 72) s_twT[tid] = __ldg(tb.twT + (long)(8 * x) * 9 + tid);  // [8][9], table padded by 8 columns
    __syncthreads();
    // ---- stage 2 fused with the store: X[k1] * W_nc^{n2 k1} -> mid[k1][n2] ------------------------
    if (col_ok) {
      float2 *dst = a.mid + (long)mblk * nc + n2g + (long)kb0 * n2;
      float const os = a.out_scale;
#pragma unroll
      for (int it = 0; it < 4; it++) {
        int const u = ul + UPI * it;
        float2 const *p = mycol + u * R2;
        float2 xv[R2];
#pragma unroll
        for (int m = 0; m < R2; m++) xv[m] = p[m];
        Dft<R2, false>::run(xv);
        float2 const wb = make_float2(twU[it].x * os, twU[it].y * os);
#pragma unroll
        for (int q = 0; q < R2; q++) dst[(long)(3 * it + 144 * q) * n2] = cmul(xv[q], cmul(wb, s_twT[c * 9 + q]));
      }
    }
    __syncthreads();  // the tile buffer is rewritten by the next stage 0
  }
}

// ------------------------------------------------------------------ pass 2: rows, persistent ---
template <bool REAL_SPLIT, int N1C = 0, bool HALVED = false>
__global__ void __launch_bounds__(512, 1) fwd_rows_v3(Pass2Args const a, FwdTables const tb, int tiles_per_block, int ntiles) {
  using P = S1250v2;
  constexpr int N2 = 1250, PITCH = 1250, T = 512, LPC = T / 8 /*lanes per column*/;
  constexpr int R0 = 10, S0 = 125, R1 = 25, NSUB1 = 125, S1 = 5, R2 = 5;
  constexpr int IPC = REAL_SPLIT ? 4 : 8;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  float2 *bufs = reinterpret_cast<float2 *>(smem_raw);  // [2][8][PITCH]
  float2 *s_tw = bufs + 2 * 8 * PITCH;
  __shared__ __align__(16) RowItem s_items[2][8];
  __shared__ __align__(8) uint64_t bars[2];
  __shared__ __align__(8) uint64_t tbar;
  TilePlan const &pl = c_plans[a.plan];
  int const tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  int const n1 = N1C ? N1C : a.n1;
  int const nc = N1C ? N1C * N2 : (int)a.nc;
  int const G = gridDim.x;

  // warp 0: fetch the rows of tile t into buffer b (lanes 0..7 = tile columns)
  auto issue = [&](int t, int b) {
    int const blk = t / tiles_per_block, x = t - blk * tiles_per_block;
    int const mblk = a.mid_mod ? blk % a.mid_mod : blk;
    RowItem it;
    it.kind = kRowEmpty;
    it.row_a = it.row_b = it.pad = 0;
    if (lane < IPC) {
      it = row_item(x * IPC + lane, n1, REAL_SPLIT);
      s_items[b][lane] = it;
    }
    int const src = REAL_SPLIT ? (lane >> 1) & 3 : lane & 7;
    int const kind = __shfl_sync(0xffffffffu, it.kind, src);
    int const ra = __shfl_sync(0xffffffffu, it.row_a, src), rb = __shfl_sync(0xffffffffu, it.row_b, src);
    if (lane < 8) {
      int row;
      if (REAL_SPLIT)
        row = (lane & 1) == 0 ? (kind != kRowEmpty ? ra : -1) : (kind == kRowPair ? rb : -1);
      else
        row = kind == kRowPlain ? ra : -1;
      if (row >= 0) {
        mbar_expect_tx(&bars[b], N2 * 8);
        bulk_g2s(bufs + (b * 8 + lane) * PITCH, a.mid + (long)mblk * nc + (long)row * N2, N2 * 8, &bars[b]);
      } else
        mbar_arrive(&bars[b]);
    }
  };

  if (tid == 0) {
    mbar_init(&bars[0], 8);
    mbar_init(&bars[1], 8);
    mbar_init(&tbar, 1);
    mbar_fence_init();
    constexpr uint32_t TWB = (uint32_t)((static_tw_count<P>() + 1) & ~1) * 8u;
    mbar_expect_tx(&tbar, TWB);
    bulk_g2s(s_tw, pl.tw, TWB, &tbar);
  }
  __syncthreads();
  if (warp == 0 && (int)blockIdx.x < ntiles) issue(blockIdx.x, 0);
  mbar_wait(&tbar, 0);

  int const c = tid & 7, ul = tid >> 3;  // column, butterfly lane 0..63
  float2 const *tw1 = s_tw + P::tw_off(1);
  int k = 0;
  for (int t = blockIdx.x; t < ntiles; t += G, k++) {
    int const b = k & 1;
    if (warp == 0 && t + G < ntiles) {  // buffer b^1 was released by the barrier that ended tile k-1
      fence_proxy_async();
      issue(t + G, b ^ 1);
    }
    mbar_wait(&bars[b], (k >> 1) & 1);
    int const blk = t / tiles_per_block;
    float2 *tile = bufs + b * 8 * PITCH;
    RowItem const itc = s_items[b][REAL_SPLIT ? c >> 1 : c];
    bool col_ok;
    if (REAL_SPLIT)
      col_ok = (c & 1) == 0 ? itc.kind != kRowEmpty : itc.kind == kRowPair;
    else
      col_ok = itc.kind == kRowPlain;
    float2 *mycol = tile + c * PITCH;

    // ---- stage 0: radix 10, stride 125 (125 butterflies per column, 64 lanes) -------------------
    if (col_ok) {
#pragma unroll
      for (int jj = 0; jj < 2; jj++) {
        int const j = ul + LPC * jj;
        if (j < S0) {
          float2 *p = mycol + j;
          float2 x[R0], w[R0];
#pragma unroll
          for (int m = 0; m < R0; m++) x[m] = p[m * S0];
          load_stage_twiddles<R0, S0>(s_tw, j, w);
          Dft<R0, false>::run(x);
          p[0] = x[0];
#pragma unroll
          for (int t2 = 1; t2 < R0; t2++) p[t2 * S0] = cmul(x[t2], w[t2]);
        }
      }
    }
    __syncthreads();
    // ---- stage 1: radix 25, 10 blocks of 125, stride 5 (50 butterflies per column) ---------------
    if (col_ok && ul < N2 / R1) {
      int const bb = ul / S1, j = ul - bb * S1;
      float2 *p = mycol + bb * NSUB1 + j;
      float2 x[R1];
#pragma unroll
      for (int m = 0; m < R1; m++) x[m] = p[m * S1];
      Dft<R1, false>::run(x);
#pragma unroll
      for (int t2 = 1; t2 < R1; t2++) x[t2] = cmul(x[t2], tw1[(t2 - 1) * S1 + j]);
#pragma unroll
      for (int t2 = 0; t2 < R1; t2++) p[t2 * S1] = x[t2];
    }

    float2 *spec = a.spec + (long)blk * a.spec_stride;
    if (!REAL_SPLIT) {
      __syncthreads();
      // ---- stage 2 fused with the plain store: X[k1 + n1*k2], k2 = t0 + 10 t1 + 250 t2 ---------
      if (col_ok) {
        float2 *dst = spec + itc.row_a;
#pragma unroll 2
        for (int u = ul; u < N2 / R2; u += LPC) {
          int const t0 = u / 25, t1 = u - t0 * 25;
          int const kb = t0 + 10 * t1;
          float2 const *p = mycol + u * R2;
          float2 x[R2];
#pragma unroll
          for (int m = 0; m < R2; m++) x[m] = p[m];
          Dft<R2, false>::run(x);
          float2 *d = dst + (long)n1 * kb;
#pragma unroll
          for (int t2 = 0; t2 < R2; t2++) d[(long)n1 * 250 * t2] = x[t2];
        }
      }
      __syncthreads();  // tile buffer free again
      continue;
    }
    // ---- stage 2 fused with the real split -----------------------------------------------------
    // W_N^{n1*k2} = exp(-i*pi*k2/1250); k2 = kb + 250 t2 -> D[kb] * exp(-i*pi*t2/5)
    int const i = tid & 3, uq = tid >> 2;  // item (row pair) 0..3, butterfly lane 0..127
    RowItem const it = s_items[b][i];
    bool const self_item = it.kind == kRowSelf0 || it.kind == kRowSelfMid;
    // table factors of this thread's two butterflies: requested before the barrier, used after it
    float2 rootC = make_float2(1.f, 0.f), rd[2];
    if (it.kind == kRowPair) rootC = __ldg(tb.rootC + it.row_a);
#pragma unroll
    for (int q = 0; q < 2; q++) {
      int const u = uq + (T / 4) * q;
      int const t0 = u / 25, t1 = u - t0 * 25;
      rd[q] = (it.kind == kRowPair && u < N2 / R2) ? __ldg(a.rootD + t0 + 10 * t1) : make_float2(1.f, 0.f);
    }
    int const has_self = __syncthreads_or(self_item);
    if (it.kind == kRowPair) {
      float2 const *ca = tile + (2 * i) * PITCH, *cb = tile + (2 * i + 1) * PITCH;
#pragma unroll
      for (int q = 0; q < 2; q++) {
        int const u = uq + (T / 4) * q;
        if (u < N2 / R2) {
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
          for (int t2 = 0; t2 < R2; t2++) {
            float2 const A = za[t2], B = zb[R2 - 1 - t2];
            float2 const w = (t2 == 0) ? wkb : cmul(wkb, wroot<10>(t2));  // exp(-i*pi*t/5) = W_10^t
            float2 const E = HALVED ? make_float2(A.x + B.x, A.y - B.y) : make_float2(0.5f * (A.x + B.x), 0.5f * (A.y - B.y));
            float2 const O = HALVED ? make_float2(A.x - B.x, A.y + B.y) : make_float2(0.5f * (A.x - B.x), 0.5f * (A.y + B.y));
            float2 const Pp = cmul(w, O);
            pk[(long)n1 * 250 * t2] = make_float2(E.x + Pp.y, E.y - Pp.x);       // X[k]    = E - i P
            pm[-(long)n1 * 250 * t2] = make_float2(E.x - Pp.y, -(E.y + Pp.x));  // X[Nc-k] = conj(E + i P)
          }
        }
      }
    }
    if (has_self) {  // CTA-uniform: rows that pair with themselves (k1 = 0 and k1 = n1/2)
      float const hf = HALVED ? 1.0f : 0.5f;
      for (int s = 0; s < 4; s++) {
        RowItem const its = s_items[b][s];
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
        RowItem const its = s_items[b][s];
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
          int const kk = its.row_a + n1 * k2;
          spec[kk] = make_float2(E.x + Pp.y, E.y - Pp.x);
          if (nc - kk != kk) spec[nc - kk] = make_float2(E.x - Pp.y, -(E.y + Pp.x));
        }
      }
    }
    __syncthreads();  // tile buffer free again
  }
}

}  // namespace kfft

namespace kfft {

// ------------------------------------------------------------------ channels, lane-packed --------
// chan_v2 gives one warp to a (channel, block) task and keeps only S0 = 25 of its lanes busy in stage 0 and
// R0 = 24 in stage 1 (600 = 24 * 25); ncu shows the kernel issue-bound (69 %).  Here a 4-warp CTA takes
// TPC = 128 / S0 tasks (5 for the 600-point plan): thread t works for task t / S0 as lane t % S0 in stage 0
// and for task t / R0 as lane t % R0 in stage 1, so 125 / 120 of the 128 lanes carry butterflies.  Tasks no
// longer coincide with warps, hence block barriers instead of __syncwarp.  REAL masters without ISB channels
// only (the launcher falls back to chan_v2 otherwise).
template <class P>
__global__ void __launch_bounds__(128) chan_v3(ChanArgs const a) {
  static_assert(P::nst == 2, "two-stage plans only");
  constexpr int NS = P::len, TOP = (NS + 1) / 2, R0 = P::rad(0), R1 = P::rad(1), S0 = NS / R0;
  static_assert(S0 == R1 && NS % 2 == 0, "plan shape");
  constexpr int TPC = 128 / (S0 > R0 ? S0 : R0);  // tasks per CTA
  constexpr int XS = NS + 4, TP = NS + XS + 2;      // per-task pitch: even (16-byte TMA alignment)
  extern __shared__ __align__(16) unsigned char smem_raw[];
  __shared__ __align__(8) uint64_t bars[TPC];
  __shared__ __align__(8) uint64_t tbar;
  float2 *base = reinterpret_cast<float2 *>(smem_raw);
  float2 *s_tw = base + TPC * TP;
  int const tid = threadIdx.x, blk = blockIdx.y;
  int const first_task = blockIdx.x * TPC;
  float2 const *X = a.spec + (long)blk * a.spec_stride;

  auto load_desc = [&](int tk, ChanDesc &d) -> bool {  // false: no such task / disabled channel
    int const oi = first_task + tk;
    d.plan = -1;
    if (tk >= TPC || oi >= a.norder) return false;
    d = a.desc[a.order ? a.order[oi] : a.chan_base + oi];
    return d.plan >= 0;
  };

  // ---- fetch: thread tk < TPC issues the two bulk copies of task tk --------------------------------------
  if (tid == 0) {
    mbar_init(&tbar, 1);
    for (int i = 0; i < TPC; i++) mbar_init(&bars[i], 1);
    mbar_fence_init();
    constexpr uint32_t TWB = (uint32_t)((static_tw_count<P>() + 1) & ~1) * 8u;
    int p0 = -1;
    for (int i = 0; i < TPC && p0 < 0; i++) {
      ChanDesc d;
      if (load_desc(i, d)) p0 = d.plan;
    }
    if (p0 >= 0) {
      mbar_expect_tx(&tbar, TWB);
      bulk_g2s(s_tw, c_plans[p0].tw, TWB, &tbar);
    } else
      mbar_arrive(&tbar);
  }
  __syncthreads();
  if (tid < TPC) {
    ChanDesc d;
    if (load_desc(tid, d) && d.ncopy > 0) {
      int const qlo = d.dir > 0 ? d.q0 : d.q0 - (d.ncopy - 1);
      int const qa = qlo & ~1, qhi = qlo + d.ncopy - 1;
      uint32_t const nx = (uint32_t)(((qhi - qa + 1) + 1) & ~1);
      float2 *col = base + tid * TP, *xs = col + NS;
      mbar_expect_tx(&bars[tid], nx * 8 + NS * 8);
      bulk_g2s(xs, X + qa, nx * 8, &bars[tid]);
      bulk_g2s(col, a.resp + d.resp_off, NS * 8, &bars[tid]);
    } else
      mbar_arrive(&bars[tid]);
  }
  mbar_wait(&tbar, 0);

  // ---- stage 0 with the slice x response product formed on the fly ------------------------------------------
  {
    int const tk = tid / S0, lane = tid - tk * S0;
    ChanDesc d;
    if (load_desc(tk, d) && d.ncopy > 0) {
      float2 *col = base + tk * TP;
      float2 const *xs = col + NS;
      int const qlo = d.dir > 0 ? d.q0 : d.q0 - (d.ncopy - 1);
      int const qa = qlo & ~1;
      mbar_wait(&bars[tk], 0);
      float2 x[R0];
#pragma unroll
      for (int m = 0; m < R0; m++) {  // S[wp] = X[q(wp)] * R[wp], zero outside the master (filter.c:728-911)
        int const wp = lane + S0 * m;
        int t = wp - TOP;
        if (t < 0) t += NS;
        int const u = t - d.zlead;
        bool const live = (u >= 0 && u < d.ncopy && wp != TOP);
        float2 xv = xs[live ? (d.q0 + d.dir * u - qa) : 0];
        if (d.dir < 0) xv.y = -xv.y;
        float2 const v = cmul(xv, col[wp]);
        x[m] = live ? v : make_float2(0.f, 0.f);
      }
      Dft<R0, true>::run(x);
      // every response word of this task is consumed above by the lane that overwrites it below (wp = lane + S0 m)
      col[lane] = x[0];
#pragma unroll
      for (int t = 1; t < R0; t++) col[lane + S0 * t] = cmulc(x[t], s_tw[(t - 1) * S0 + lane]);
    }
  }
  __syncthreads();
  // ---- stage 1 fused with the store: y[n], n = u + R0*t, keep n >= NS - olen --------------------------------
  {
    int const tk = tid / R0, lane = tid - tk * R0;
    ChanDesc d;
    if (load_desc(tk, d)) {
      float2 *dst = a.out + (long)blk * a.out_stride + d.out_off;
      if (d.ncopy <= 0) {
        for (int i = lane; i < d.olen; i += R0) dst[i] = make_float2(0.f, 0.f);
      } else {
        float2 const *col = base + tk * TP;
        float2 x[R1];
#pragma unroll
        for (int m = 0; m < R1; m++) x[m] = col[R1 * lane + m];
        Dft<R1, true>::run(x);
        int const first = NS - d.olen;
#pragma unroll
        for (int t = 0; t < R1; t++) {
          int const n = lane + R0 * t;
          if (n >= first) dst[n - first] = x[t];
        }
      }
    }
  }
}

}  // namespace kfft
