// static_kernels_v2.cuh -- the 1250-point row pass and the two-stage channel kernels, with the first and last butterfly
// stage fused into the fill and the global store.
//
// An in-shared-memory DIF moves every point through shared memory twice per stage plus once on the way in and once on the
// way out, and kernels built that way are bound by the L1/shared-memory LSU data pipe.  Here the lanes of a warp are
// interleaved over the tile's 8 columns (lane = 8*u' + column), the first stage works on the data as it arrives and the last
// stage writes its outputs (through the real split, or into the kept samples of a channel) straight to global memory.
// Column pitch = 2 mod 16 keeps every access pattern free of bank conflicts (8 even column offsets x 2 consecutive
// butterflies per half-warp).
#pragma once
#include "static_kernels.cuh"

namespace kfft {

// ---- int16 ingest of the specialised column kernels (fwd_cols_r36.cuh, fwd_2s.cuh) -----------
// FMT 0: float pairs; 1: int16 pairs; 2: int16 pairs + de-randomise + energy/clip statistics.
// int16 pair -> two floats.  `(float)(short)` compiles to I2F.S16, which issues through the MIO
// queue to the quarter-rate conversion unit -- the queue the 36 loads and 72 shared-memory accesses
// of a thread also need (ncu: mio_throttle was the top stall of the column pass).  Sign-extend with
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

// ------------------------------------------------------------------ pass 2: rows --------------
// 1250 = 10 * 25 * 5.  Rows arrive by TMA; stages 0 and 1 run in shared memory with the lanes
// interleaved over the 8 columns; the radix-5 last stage is fused with the real split: the thread
// that owns butterfly u of row k1 also takes butterfly 249-u of the mirror row N1-k1, which holds
// exactly the partners Z[Nc-k] of its five outputs (digit complement: 1249-k2 <-> (9-t0,24-t1,4-t2)).
// N1C: row count as a compile-time constant (0 = from the arguments).  HALVED: the 1/2 of the real
// split was already folded into the column pass (Pass1Args::out_scale).
// The row pass of every master with 1250 columns, REAL and COMPLEX.  On H100 it beat a two-stage 50 x 25 row kernel
// (DESIGN.md section 4).  Blocks are taken last-to-first: the column pass wrote the last ones most recently, so their
// rows are the likeliest to be still in L2.
// Tiling: a group of 256 threads runs stages 0 and 1 on 8 tile columns.  COMPLEX: one group, 8 rows per CTA.  REAL: two
// groups, 16 columns = 8 mirrored pairs per CTA (pair i in columns 2i, 2i+1; group g holds pairs 4g..4g+3), so that a
// warp's split stores cover 8 consecutive k1: 64-byte runs X[k1 + n1 k2] and their mirrors, instead of 32-byte runs
// from 4 pairs.  One 512-thread CTA per SM holds about as many rows and warps as two 4-pair CTAs did.
// Shared-memory banks, in float2 slots (bank pair = offset mod 16), PITCH = 1250 = 2 mod 16:
//  * stages 0 and 1 touch only their group's 8 columns, at 2c mod 16: conflict-free as in the one-group form.
//  * stage 2 reads slot col_off(2i) + 5u + m (forward row) and col_off(2i+1) - 5u + m (mirror), lane = 8 (u - u0) + i.
//    A half-warp holds i = 0..7 at two consecutive u.  Without a skew, 2i*PITCH = 4i mod 16 puts pairs i and i+4 on the
//    same slots (2-way).  The second group's columns start SKEW = 2 slots later: pairs 0..3 take the slots
//    {4a + 5b} = {0,1,4,5,8,9,12,13}, pairs 4..7 the slots {2,3,6,7,10,11,14,15}, and the mirror reads
//    {4a + 2 - 5b} likewise split into two disjoint halves: every stage-2 read is conflict-free.  SKEW = 2 float2s
//    = 16 bytes keeps every TMA destination 16-byte aligned (PITCH * 8 = 10000 bytes is a multiple of 16).
template <bool REAL_SPLIT>
struct RowsV2Shape {
  using P = SPlan<1250, 10, 25, 5>;  // what choose_radices(1250) picks: the kernel reads that registry plan's stage twiddles
  static constexpr int N2 = 1250, PITCH = 1250, GT = 256, SKEW = 2;
  static constexpr int NG = REAL_SPLIT ? 2 : 1, T = GT * NG, COLS = 8 * NG;
  static constexpr int IPC = REAL_SPLIT ? COLS / 2 : COLS;  // work items (row pairs or rows) per CTA
  static constexpr int TW = (static_tw_count<P>() + 1) & ~1;  // stage twiddles, even (bulk copies move 16-byte multiples)
  static constexpr int TILE = COLS * PITCH + (NG - 1) * SKEW;
  static constexpr size_t smem = sizeof(float2) * (size_t)(TILE + TW);
  static __host__ __device__ constexpr int col_off(int c) { return c * PITCH + (c >> 3) * SKEW; }
};

// W_1250^{32 it t} literals for stage 0 of the row pass
__device__ constexpr float kRowsTw0[3][4][2] = {
    {{9.870916009e-01f, -1.601568460e-01f}, {9.486995935e-01f, -3.161789477e-01f}, {8.000617623e-01f, -5.999176502e-01f}, {2.801976204e-01f, -9.599423409e-01f}},
    {{9.486995935e-01f, -3.161789477e-01f}, {8.000617623e-01f, -5.999176502e-01f}, {2.801976204e-01f, -9.599423409e-01f}, {-8.429785967e-01f, -5.379471183e-01f}},
    {{8.858151436e-01f, -4.640382826e-01f}, {5.693368912e-01f, -8.221042752e-01f}, {-3.517109454e-01f, -9.361086488e-01f}, {-7.525988221e-01f, 6.584793329e-01f}},
};

// Stage-0 twiddles W^{j t}, j = ul + 32 it, are (4 values loaded once per thread) x (literal W^{32 it t}) instead of 4 loads per
// butterfly.  Variants tried and removed again: warp-per-column stages 0/1, stage-0 butterflies in groups of 2 / 4,
// stage-1 twiddles by products, a persistent double-buffered form, an L2 prefetch of a later CTA's rows, blocks first-to-last,
// REAL with 4 row pairs per 256-thread CTA (32-byte store runs; 18.2 against 13.5 us per cfg-2 block, DESIGN.md section 4).
// The 128-byte lines of the inter-pass buffer (rows of mid_ld points, a multiple of 16): line l of row `row` of block
// blk, counted from the buffer's start
__host__ __device__ constexpr int mid_row_lines(int mid_ld) { return mid_ld * 8 / 128; }
__host__ __device__ constexpr long mid_line(int blk, int n1, int row, int mid_ld, int l) {
  return ((long)blk * n1 + row) * mid_row_lines(mid_ld) + l;
}

// The row tile of items item0 .. item0+IPC-1 of block blk, by the S::T threads tid = 0..T-1, in S::smem bytes of shared
// memory at smem_raw with the mbarriers bars[COLS] and tbar.  sync / sync_or: a barrier (and its OR reduction) of exactly
// those threads; the groups' barriers are 1 and 2.  FUSED (fwd_fused.cuh): the caller has acquired the block's inter-pass
// rows, written by other SMs; each row's copy is ordered after that through the async proxy, and the row's L2 lines are
// discarded once it is in shared memory (nothing reads them again, so they never have to be written back to DRAM).
template <bool REAL_SPLIT, int N1C, bool HALVED, bool FUSED, class Sync, class SyncOr>
__device__ __forceinline__ void fwd_rows_v2_body(Pass2Args const &a, FwdTables const &tb, unsigned char *smem_raw,
                                                 uint64_t *bars, uint64_t &tbar, int tid, int blk, int item0,
                                                 Sync const &sync, SyncOr const &sync_or, bool discard = false) {
  using S = RowsV2Shape<REAL_SPLIT>;
  using P = typename S::P;
  constexpr int N2 = S::N2, T = S::T, GT = S::GT, COLS = S::COLS, IPC = S::IPC;
  constexpr int R0 = 10, S0 = 125, R1 = 25, NSUB1 = 125, S1 = 5, R2 = 5;
  float2 *tile = reinterpret_cast<float2 *>(smem_raw);  // COLS columns at S::col_off(c)
  float2 *s_tw = tile + S::TILE;
  TilePlan const &pl = c_plans[a.plan];
  int const lane = tid & 31, warp = tid >> 5;
  int const n1 = N1C ? N1C : a.n1;
  // which global row sits in which tile column
  auto row_of = [&](int col) -> int {
    RowItem const it = row_item(item0 + (REAL_SPLIT ? col >> 1 : col), n1, REAL_SPLIT);
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
      if (FUSED) fence_proxy_async_global();
      mbar_expect_tx(&bars[warp], N2 * 8);
      bulk_g2s(tile + S::col_off(warp), a.mid + ((long)blk * n1 + row) * a.mid_ld, N2 * 8, &bars[warp]);
    }
    if (warp == 0) {
      constexpr uint32_t TWB = (uint32_t)S::TW * 8u;
      mbar_expect_tx(&tbar, TWB);
      bulk_g2s(s_tw, pl.tw, TWB, &tbar);
    }
  }
  sync();
  int const g = tid / GT;                                  // group
  int const c = (tid & 7) + 8 * g, ul = (tid % GT) >> 3;  // column, butterfly lane 0..31
  // stages 0 and 1 of a group touch only its own columns: the groups meet only before stage 2
  auto group_sync = [&] {
    if (S::NG == 1) sync();
    else asm volatile("bar.sync %0, %1;" ::"r"(1 + g), "n"(GT) : "memory");
  };
  bool const col_ok = row_of(c) >= 0;
  mbar_wait(&tbar, 0);
  if (col_ok) mbar_wait(&bars[c], 0);
  if (FUSED && discard && col_ok) {  // the 32 threads of column c discard its row's lines (scratch: no result changes)
    char *const mid = const_cast<char *>(reinterpret_cast<char const *>(a.mid));
    for (int l = ul; l < mid_row_lines(a.mid_ld); l += GT / 8) discard_l2_line(mid + 128 * mid_line(blk, n1, row_of(c), a.mid_ld, l));
  }
  float2 *mycol = tile + S::col_off(c);

  // ---- stage 0: radix 10, stride 125 (125 butterflies per column) ------------------------------
  if (col_ok) {
    float2 base[4];
#pragma unroll
    for (int q = 0; q < 4; q++) base[q] = s_tw[((1 << q) - 1) * S0 + ul];  // W^{ul t}, t = 1, 2, 4, 8
#pragma unroll
    for (int it = 0; it < 4; it++) {
      int const j = ul + (GT / 8) * it;
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
  group_sync();
  // ---- stage 1: radix 25, 10 blocks of 125, stride 5 (50 butterflies per column) ---------------
  if (col_ok) {
    float2 const *tw1 = s_tw + P::tw_off(1);
#pragma unroll 1
    for (int u = ul; u < N2 / R1; u += GT / 8) {
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
  constexpr int UQ = T / IPC;               // REAL: 64 butterfly lanes per row pair
  int const i = tid % IPC, uq = tid / IPC;  // item (row pair) 0..7, butterfly lane 0..63
  RowItem const it = row_item(item0 + i, n1, REAL_SPLIT);
  float2 rootC = make_float2(1.f, 0.f), rd[4];
  bool self_item = false;
  if (REAL_SPLIT) {
    self_item = it.kind == kRowSelf0 || it.kind == kRowSelfMid;
    if (it.kind == kRowPair) rootC = __ldg(tb.rootC + it.row_a);
#pragma unroll
    for (int q = 0; q < 4; q++) {
      int const u = uq + UQ * q;
      int const t0 = u / 25, t1 = u - t0 * 25;
      rd[q] = (it.kind == kRowPair && u < N2 / R2) ? __ldg(a.rootD + t0 + 10 * t1) : make_float2(1.f, 0.f);
    }
  }
  int const has_self = sync_or(self_item);

  float2 *spec = a.spec + (long)blk * a.spec_stride;
  float const hf = HALVED ? 1.0f : 0.5f;
  if (!REAL_SPLIT) {
    // ---- stage 2 fused with the plain store: X[k1 + n1*k2], k2 = t0 + 10 t1 + 250 t2 ---------
    if (col_ok) {
      float2 *dst = spec + row_of(c);
#pragma unroll 1
      for (int u = ul; u < N2 / R2; u += GT / 8) {
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
    float2 const *ca = tile + S::col_off(2 * i), *cb = tile + S::col_off(2 * i + 1);
#pragma unroll
    for (int q = 0; q < 4; q++) {
      int const u = uq + UQ * q;
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
  if (!has_self) return;  // CTA-uniform
  for (int s = 0; s < IPC; s++) {
    RowItem const its = row_item(item0 + s, n1, true);
    if (its.kind != kRowSelf0 && its.kind != kRowSelfMid) continue;
    float2 *col = tile + S::col_off(2 * s);
    for (int u = tid; u < N2 / R2; u += T) {
      float2 x[R2];
#pragma unroll
      for (int m = 0; m < R2; m++) x[m] = col[u * R2 + m];
      Dft<R2, false>::run(x);
#pragma unroll
      for (int m = 0; m < R2; m++) col[u * R2 + m] = x[m];
    }
  }
  sync();
  for (int s = 0; s < IPC; s++) {
    RowItem const its = row_item(item0 + s, n1, true);
    if (its.kind != kRowSelf0 && its.kind != kRowSelfMid) continue;
    float2 const *col = tile + S::col_off(2 * s);
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

template <bool REAL_SPLIT, int N1C = 0, bool HALVED = false>
__global__ void __launch_bounds__(RowsV2Shape<REAL_SPLIT>::T, REAL_SPLIT ? 1 : 2) fwd_rows_v2(Pass2Args const a, FwdTables const tb) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  __shared__ __align__(8) uint64_t bars[RowsV2Shape<REAL_SPLIT>::COLS];
  __shared__ __align__(8) uint64_t tbar;
  fwd_rows_v2_body<REAL_SPLIT, N1C, HALVED, false>(a, tb, smem_raw, bars, tbar, threadIdx.x, gridDim.y - 1 - blockIdx.y,
                                                   blockIdx.x * RowsV2Shape<REAL_SPLIT>::IPC, [] { __syncthreads(); },
                                                   [](int p) { return __syncthreads_or(p); });
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
  __shared__ __align__(8) uint64_t bars[kChanWarps];
  __shared__ __align__(8) uint64_t tbar;
  using S = StaticChan<P>;
  constexpr int NS = S::NS, R0 = P::rad(0), R1 = P::rad(1), S0 = NS / R0;
  static_assert(S0 == R1, "plan shape");
  S s;
  if (!static_prologue<P>(a, bars, tbar, s)) return;
  ChanDesc const &d = s.d;
  float2 *col = s.col;
  int const lane = s.lane;
  mbar_wait(&tbar, 0);
  if (d.flags & kChanIsb) {  // ISB: whole product in shared memory first, then the plain two stages
    for (int wp = lane; wp < NS; wp += 32) col[wp] = s.product(wp);  // same lane reads R[wp] and writes S[wp]
    __syncwarp();
    isb_fold_warp(col, NS, S::TOP, lane);
    static_stage<P, true, 0, true, 1>(col, s.s_tw, lane);
    __syncwarp();
  } else if (lane < S0) {
    // ---- stage 0 with the product formed on the fly ------------------------------------------
    float2 x[R0];
#pragma unroll
    for (int m = 0; m < R0; m++) x[m] = s.product(lane + S0 * m);
    Dft<R0, true>::run(x);
    col[lane] = x[0];
#pragma unroll
    for (int t = 1; t < R0; t++) col[lane + S0 * t] = cmulc(x[t], s.s_tw[(t - 1) * S0 + lane]);
  }
  __syncwarp();
  // ---- stage 1 fused with the store: y[n], n = u + R0*t, keep n >= NS - olen ---------------------
  bool const osc = OSC && (d.flags & kChanOsc) != 0;  // warp-uniform
  float pw = 0.f;
  int const ci = chan_index(a, s.oi);
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
        if (n >= first) s.dst[n - first] = x[t];
      }
    } else if (OSC) {  // fine-tuning rotation + block power fused into the store (radio.c:1476-1501, :1515-1520)
      ChanAux const ax = a.aux[ci];
      long const k = a.block0 + s.blk - ax.osc_epoch;
#pragma unroll
      for (int t = 0; t < R1; t++) {
        int const n = lane + R0 * t;
        if (n >= first) s.dst[n - first] = osc_sample(ax, k, d.olen, n - first, x[t], pw);
      }
    }
  }
  if (OSC && osc && a.power) {
    pw = warp_sum(pw);
    if (lane == 0) a.power[(long)s.blk * a.power_stride + ci] = pw / (float)d.olen;
  }
}

}  // namespace kfft
