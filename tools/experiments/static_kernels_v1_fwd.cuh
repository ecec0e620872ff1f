// NOT BUILT.  Round-1 forward kernels (in-shared-memory DIF, every stage through shared memory), superseded by
// static_kernels_v2.cuh.  Kept for the record.
#pragma once
namespace kfft {
// largest divisor of n that is <= cap (compile-time batch sizes without remainders)
constexpr int batch_of(int n, int cap) {
  int b = 1;
  for (int d = 1; d <= cap; d++)
    if (n % d == 0) b = d;
  return b;
}
constexpr int static_pitch(int len) {
  int p = len;
  while (p % 16 != 2) p++;
  return p;
}

// ------------------------------------------------------------------ pass 1: columns -----------
// FMT 0: float pairs; 1: int16 pairs, plain; 2: int16 pairs with de-randomise + energy/clip stats.
// TILE columns per CTA, WPC warps per column, LAY: shared-memory layout variant (see below).
template <int FMT, class P, int TILE, int WPC, int LAY = 0, int MINB = 2, bool TWC = false>
__global__ void __launch_bounds__(TILE * 32 * WPC, MINB) fwd_cols_static(Pass1Args const a, FwdTables const tb) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  // Column c starts at c*PITCH + e(c), PITCH = 0 mod 16 and e = {0,1,2,3,8,9,10,11}: then both the
  // transposing load (a half-warp holds 8 columns x rows {r, r+4}) and the digit-reversed read of
  // the store phase (8 columns x slots {s, s+108 = s+12 mod 16}) touch 16 distinct bank pairs.
  static_assert(TILE == 8, "column base table is written for 8 columns");
  constexpr int N1 = P::len, PITCH = LAY ? (N1 + 12 + 15) / 16 * 16 : static_pitch(phys_len<P>()), NT = TILE * 32 * WPC;
  constexpr int RPI = NT / TILE /*rows per step*/, FULL = N1 / RPI, REM = N1 % RPI;
  auto colbase = [](int cc) { return LAY ? cc * PITCH + (cc < 4 ? cc : cc + 4) : cc * PITCH; };
  float2 *tile = reinterpret_cast<float2 *>(smem_raw);  // [TILE][PITCH]
  float2 *s_tw = tile + TILE * PITCH;                   // stage twiddles, shared by the columns
  float2 *s_twA = s_tw + ((static_tw_count<P>() + 1) & ~1);  // [TILE][FULL+1] inter-pass factors A(n2, it)
  TilePlan const &pl = c_plans[a.plan];
  int const tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  int const c = tid % TILE, r = tid / TILE;  // store phase: rows r, r+1 share a half-warp
  // load phase: rows r, r+4 share a half-warp (warp pairs cover 8 consecutive rows)
  int const rl = LAY ? 8 * (warp >> 1) + 2 * (warp & 1) + 4 * ((lane >> 3) & 1) + (lane >> 4) : r;
  int const c0 = blockIdx.x * TILE;
  int const blk = blockIdx.y;
  int const ncols = min(TILE, a.n2 - c0);
  bool const col_ok = c < ncols;
  int const n2g = c0 + c;
  float2 *mycol = tile + colbase(c);
  unsigned long long *dbg = a.dbg ? a.dbg + 6 * ((long)blockIdx.y * gridDim.x + blockIdx.x) : nullptr;
  if (dbg && tid == 0) {
    dbg[0] = gtimer();
    unsigned smid;
    asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
    dbg[5] = smid;
  }
  // stage twiddles and the tile's inter-pass factors arrive by TMA bulk copies (tables are padded)
  __shared__ __align__(8) uint64_t tbar;
  constexpr uint32_t TWB = (uint32_t)((static_tw_count<P>() + 1) & ~1) * 8u, TAB = (uint32_t)(TILE * (FULL + 1)) * 8u;
  static_assert((TILE * (FULL + 1)) % 2 == 0, "inter-pass factor tile must be a 16-byte multiple");
  if (tid == 0) {
    mbar_init(&tbar, 1);
    mbar_fence_init();
    mbar_expect_tx(&tbar, TWB + TAB);
    bulk_g2s(s_tw, pl.tw, TWB, &tbar);
    bulk_g2s(s_twA, tb.twA + (long)c0 * (FULL + 1), TAB, &tbar);
  }
  float2 const twB = col_ok ? __ldg(tb.twB + n2g * RPI + r) : make_float2(1.f, 0.f);

  unsigned long long energy = 0;
  unsigned int clips = 0;
  if (col_ok) {
    long const step = (long)RPI * a.n2;
    constexpr int U = batch_of(FULL, 20);  // rows in flight per thread
    if (FMT == 0) {
      float2 const *src = reinterpret_cast<float2 const *>(a.in) + (long)blk * a.hop + (long)rl * a.n2 + n2g;
#pragma unroll 1
      for (int it0 = 0; it0 < FULL; it0 += U) {
        float2 w[U];
#pragma unroll
        for (int u = 0; u < U; u++, src += step) w[u] = ldg_stream_f2(src);
#pragma unroll
        for (int u = 0; u < U; u++) mycol[phys_of<P>(rl + RPI * (it0 + u))] = w[u];
      }
      if (REM && rl < REM) mycol[phys_of<P>(rl + RPI * FULL)] = ldg_stream_f2(src);
    } else {
      int const *src = reinterpret_cast<int const *>(a.in) + (long)blk * a.hop + (long)rl * a.n2 + n2g;
      float const sc = a.scale;
      auto conv = [&](int w, int n1) -> float2 {
        short lo = (short)(w & 0xffff), hi = (short)((unsigned)w >> 16);
        if (FMT == 2) {
          if (a.derandomize) {  // lsb set -> flip bits 1..15 (rx888.c:707-712)
            lo ^= (short)((lo & 1) ? 0xfffe : 0);
            hi ^= (short)((hi & 1) ? 0xfffe : 0);
          }
          if (a.stats && (long)n1 * a.n2 + n2g >= a.first_new) {
            energy += (unsigned long long)((int)lo * lo) + (unsigned long long)((int)hi * hi);
            clips += (lo > 32766 || lo < -32766) + (hi > 32766 || hi < -32766);
          }
        }
        return make_float2((float)lo * sc, (float)hi * sc);
      };
#pragma unroll 1
      for (int it0 = 0; it0 < FULL; it0 += U) {
        int w[U];
#pragma unroll
        for (int u = 0; u < U; u++, src += step) w[u] = ldg_stream_b32(src);
#pragma unroll
        for (int u = 0; u < U; u++) mycol[phys_of<P>(rl + RPI * (it0 + u))] = conv(w[u], rl + RPI * (it0 + u));
      }
      if (REM && rl < REM) mycol[phys_of<P>(rl + RPI * FULL)] = conv(ldg_stream_b32(src), rl + RPI * FULL);
    }
  }
  if (FMT == 2 && a.stats) {
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
  if (dbg && tid == 0) dbg[1] = gtimer();
  __syncthreads();
  mbar_wait(&tbar, 0);
  if (dbg && tid == 0) dbg[2] = gtimer();
  {
    int const fc = warp / WPC;  // the column this warp transforms
    if (fc < ncols) StaticFftGroup<P, false, WPC, TWC>::run(tile + colbase(fc), s_tw, (warp % WPC) * 32 + lane, 1 + fc);
  }
  __syncthreads();
  if (dbg && tid == 0) dbg[3] = gtimer();
  if (col_ok) {
    long const step = (long)RPI * a.n2;
    float2 *dst = a.mid + (long)blk * a.nc + (long)r * a.n2 + n2g;
    float2 const *twA = s_twA + c * (FULL + 1);
    constexpr int V = batch_of(FULL, 10);
#pragma unroll 1
    for (int it0 = 0; it0 < FULL; it0 += V) {
      float2 v[V], w[V];
#pragma unroll
      for (int u = 0; u < V; u++) {
        w[u] = twA[it0 + u];
        v[u] = mycol[phys_of<P>(static_slot<P>(r + RPI * (it0 + u)))];
      }
#pragma unroll
      for (int u = 0; u < V; u++, dst += step) *dst = cmul(v[u], cmul(twB, w[u]));
    }
    if (REM && r < REM) *dst = cmul(mycol[phys_of<P>(static_slot<P>(r + RPI * FULL))], cmul(twB, twA[FULL]));
  }
  if (dbg && tid == 0) dbg[4] = gtimer();
}

// ------------------------------------------------------------------ pass 2: rows --------------
// WPC warps per row (column of the tile).
template <class P, bool REAL_SPLIT, int WPC, bool TWC = false>
__global__ void __launch_bounds__(kTile * 32 * WPC, 2) fwd_rows_static(Pass2Args const a, FwdTables const tb) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  constexpr int N2 = P::len, PITCH = static_pitch(N2), NT = kTile * 32 * WPC;
  static_assert(N2 % 2 == 0, "bulk row copies need 16-byte multiples");
  float2 *tile = reinterpret_cast<float2 *>(smem_raw);  // [kTile][PITCH]
  float2 *s_tw = tile + kTile * PITCH;
  __shared__ __align__(8) uint64_t bars[kTile];
  __shared__ __align__(8) uint64_t tbar;
  TilePlan const &pl = c_plans[a.plan];
  int const tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  int const blk = blockIdx.y;
  constexpr int IPC = REAL_SPLIT ? kTile / 2 : kTile;
  RowItem const *items = a.items + (long)blockIdx.x * IPC;
  unsigned long long *dbg = a.dbg ? a.dbg + 6 * ((long)blockIdx.y * gridDim.x + blockIdx.x) : nullptr;
  if (dbg && tid == 0) dbg[0] = gtimer();
  {
    int const colw = warp / WPC, sub = warp % WPC;  // tile column this warp works on
    RowItem const it = items[REAL_SPLIT ? colw >> 1 : colw];
    int row = -1;
    if (REAL_SPLIT) {
      if ((colw & 1) == 0 && it.kind != kRowEmpty) row = it.row_a;
      if ((colw & 1) == 1 && it.kind == kRowPair) row = it.row_b;
    } else if (it.kind == kRowPlain) {
      row = it.row_a;
    }
    float2 *colp = tile + colw * PITCH;
    if (row >= 0 && sub == 0 && lane == 0) {
      // one TMA bulk copy brings the whole (contiguous) row; completion lands on this column's mbarrier
      mbar_init(&bars[colw], 1);
      mbar_fence_init();
      mbar_expect_tx(&bars[colw], N2 * 8);
      bulk_g2s(colp, a.mid + (long)blk * a.nc + (long)row * N2, N2 * 8, &bars[colw]);
    }
    // the stage twiddles come the same way, on their own barrier
    if (tid == 0) {
      constexpr uint32_t TWB = (uint32_t)((static_tw_count<P>() + 1) & ~1) * 8u;
      mbar_init(&tbar, 1);
      mbar_fence_init();
      mbar_expect_tx(&tbar, TWB);
      bulk_g2s(s_tw, pl.tw, TWB, &tbar);
    }
    __syncthreads();
    mbar_wait(&tbar, 0);
    if (row >= 0) {
      mbar_wait(&bars[colw], 0);
      if (dbg && tid == 0) dbg[1] = gtimer();
      StaticFftGroup<P, false, WPC, TWC>::run(colp, s_tw, sub * 32 + lane, 1 + colw);
    }
  }
  __syncthreads();
  if (dbg && tid == 0) dbg[2] = gtimer();

  float2 *spec = a.spec + (long)blk * a.spec_stride;
  int const n1 = a.n1;
  if (!REAL_SPLIT) {
    int const i = tid % kTile, q0 = tid / kTile;
    RowItem const it = items[i];
    if (it.kind == kRowPlain) {
      float2 const *colp = tile + i * PITCH;
      constexpr int QS = NT / kTile, V = 8;
      float2 *dst = spec + it.row_a;
#pragma unroll 1
      for (int k0 = q0; k0 < N2; k0 += V * QS) {
        float2 v[V];
#pragma unroll
        for (int u = 0; u < V; u++)
          if (k0 + u * QS < N2) v[u] = colp[static_slot<P>(k0 + u * QS)];
#pragma unroll
        for (int u = 0; u < V; u++)
          if (k0 + u * QS < N2) dst[(long)n1 * (k0 + u * QS)] = v[u];
      }
    }
    return;
  }
  // REAL epilogue.  X[k] = E - i*P, X[Nc-k] = conj(E + i*P) with E/O the even/odd parts of the
  // (Z[k], conj Z[Nc-k]) pair and P = W_N^k * O.  4 adjacent rows per warp quad -> 32-byte segments.
  constexpr int HALF = kTile / 2, QS = NT / HALF;
  int const i = tid % HALF, q0 = tid / HALF;
  RowItem const it = items[i];
  if (it.kind == kRowEmpty) return;
  float2 const *ca = tile + (2 * i) * PITCH;
  float2 const rootC = __ldg(tb.rootC + it.row_a);
  int const nc = (int)a.nc;
  auto emit = [&](int k2, float2 za, float2 zb, float2 rd) {
    int const k = it.row_a + n1 * k2;
    float2 const w = cmul(rootC, rd);
    float2 const E = make_float2(0.5f * (za.x + zb.x), 0.5f * (za.y - zb.y));
    float2 const O = make_float2(0.5f * (za.x - zb.x), 0.5f * (za.y + zb.y));
    float2 const Pp = cmul(w, O);
    spec[k] = make_float2(E.x + Pp.y, E.y - Pp.x);
    spec[nc - k] = make_float2(E.x - Pp.y, -(E.y + Pp.x));
  };
  constexpr int V = 4;
  if (it.kind == kRowPair) {
    float2 const *cb = tile + (2 * i + 1) * PITCH;
    constexpr int NFULL = (N2 / QS) / V * V;  // iterations valid for every q0
#pragma unroll 1
    for (int j0 = 0; j0 < NFULL; j0 += V) {
      float2 za[V], zb[V], rd[V];
#pragma unroll
      for (int u = 0; u < V; u++) {
        int const k2 = q0 + (j0 + u) * QS;
        rd[u] = __ldg(a.rootD + k2);
        za[u] = ca[static_slot<P>(k2)];
        zb[u] = cb[static_slot<P>(N2 - 1 - k2)];
      }
#pragma unroll
      for (int u = 0; u < V; u++) emit(q0 + (j0 + u) * QS, za[u], zb[u], rd[u]);
    }
    for (int k2 = q0 + NFULL * QS; k2 < N2; k2 += QS)
      emit(k2, ca[static_slot<P>(k2)], cb[static_slot<P>(N2 - 1 - k2)], __ldg(a.rootD + k2));
  } else if (it.kind == kRowSelf0) {  // row 0 pairs with itself: k2 <-> N2-k2 (k2 = 0 -> bins 0 and Nc)
    for (int k2 = q0; k2 <= N2 / 2; k2 += QS) {
      float2 const za = ca[static_slot<P>(k2)], zb = ca[static_slot<P>(k2 == 0 ? 0 : N2 - k2)];
      if (2 * k2 == N2) {  // bin Nc/2 pairs with itself: one write
        float2 const w = cmul(rootC, __ldg(a.rootD + k2));
        float2 const E = make_float2(0.5f * (za.x + zb.x), 0.5f * (za.y - zb.y));
        float2 const O = make_float2(0.5f * (za.x - zb.x), 0.5f * (za.y + zb.y));
        float2 const Pp = cmul(w, O);
        spec[n1 * k2] = make_float2(E.x + Pp.y, E.y - Pp.x);
      } else {
        emit(k2, za, zb, __ldg(a.rootD + k2));
      }
    }
  } else {  // middle row n1/2 pairs with itself: k2 <-> N2-1-k2
    for (int k2 = q0; k2 < (N2 + 1) / 2; k2 += QS) {
      float2 const za = ca[static_slot<P>(k2)], zb = ca[static_slot<P>(N2 - 1 - k2)];
      if (2 * k2 == N2 - 1) {
        float2 const w = cmul(rootC, __ldg(a.rootD + k2));
        float2 const E = make_float2(0.5f * (za.x + zb.x), 0.5f * (za.y - zb.y));
        float2 const O = make_float2(0.5f * (za.x - zb.x), 0.5f * (za.y + zb.y));
        float2 const Pp = cmul(w, O);
        spec[it.row_a + n1 * k2] = make_float2(E.x + Pp.y, E.y - Pp.x);
      } else {
        emit(k2, za, zb, __ldg(a.rootD + k2));
      }
    }
  }
  if (dbg && tid < HALF) dbg[3] = gtimer();
}

}  // namespace kfft
