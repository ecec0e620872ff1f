// fwd_rows_body.cuh -- the body of the generic row pass, included by fwd_kernels.cuh into fwd_rows_kernel (registry
// plan, KFFT_ROWS_EXT false) and fwd_rows_ext (the master's own plan, KFFT_ROWS_EXT true).  Not a header of its own:
// it expects `a` (Pass2Args) and `pl` (TilePlan) in scope.  Written out in each kernel rather than called as an
// inline function because that keeps fwd_rows_kernel's machine code exactly what it was before the extended pair
// existed (as a call, the compiler reorders the address arithmetic of the split loop).
  extern __shared__ __align__(16) unsigned char smem_raw[];
  float2 *tile = reinterpret_cast<float2 *>(smem_raw);  // [kTile][pitch]
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
      tile_fft<false, KFFT_ROWS_EXT>(pl, colp, lane, 32, [] { __syncwarp(); });
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
