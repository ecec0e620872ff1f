// fwd_2s.cuh -- both passes of the two-pass forward transform with TWO fat stages each, for any n1 = RA x RB, n2 = RC x RD.
//
// fwd_cols_r36.cuh showed (cfg-2, 1296 = 36 x 36) that these kernels are paced by trips through shared memory, not by
// arithmetic: with two stages a point crosses shared memory once per pass.  This file is the same design with the radices
// as template parameters, instantiated for the c2c front ends of BASELINE.json (cfg-4, Airspy-class 20 MS/s I/Q:
// 500 000 = 800 x 625 = (25 x 32) x (25 x 25)), which otherwise run on the runtime-plan kernels of fwd_kernels.cuh.
//
// Column pass  fwd_cols_2s<FMT, RA, RB>:  column n2 of the n1 x n2 matrix, n1 = RA x RB
//   stage 0 (fused with the global load, int16 pairs -> float in registers): butterfly j < RB takes x[j + RB m], m < RA,
//     output t is multiplied by W_n1^{j t} and stored to block t of the column (RB points per block);
//   stage 1 (fused with the global store): sub-transform t < RA reads its RB contiguous points, output k' is
//     X[t + RA k'] * W_nc^{n2 (t + RA k')} -> row t + RA k' of the inter-pass buffer.
// Row pass  fwd_rows_2s<RC, RD>:  row k1 (n2 = RC x RD contiguous points, fetched by one TMA bulk copy)
//   stage 0 in place: butterfly j < RD takes x[j + RD m], m < RC, output t * W_n2^{j t} -> x[t RD + j];
//   stage 1 fused with the store: sub-transform t reads x[t RD + m], output k' is X[k1 + n1 (t + RC k')].
// A thread needs the powers w^e, e = 1..R-1, of one base w; Q - 1 + (R-1)/Q of them are loaded (e = 1..Q-1 and Q, 2Q, ..),
// the others are one product each (Pow<R>), as in the 36 x 36 kernel.
// Shared-memory layout (both passes): 8 columns (rows) per CTA at a pitch = 2 mod 16 elements, so that the 8 B accesses of a
// half warp (8 columns x 2 consecutive butterflies) and the 16 B accesses of a quarter warp (8 columns) hit all banks once.
#pragma once
#include "static_kernels_v2.cuh"

namespace kfft {

constexpr int ceil_sqrt(int r) {
  int q = 1;
  while (q * q < r) q++;
  return q;
}
constexpr int pitch_2mod16(int n) { return (n + 13) / 16 * 16 + 2; }  // smallest p >= n with p = 2 (mod 16)

// powers of one base: exponents 1..Q-1 ("b") and Q, 2Q, .. ("a"); w^t = a[t / Q] * b[t % Q]
template <int R> struct Pow {
  static constexpr int Q = ceil_sqrt(R), NB = Q - 1, NA = (R - 1) / Q, NP = NB + NA;
  static_assert(NA * Q + NB >= R - 1, "power split does not cover the radix");
  static constexpr int exponent(int i) { return i < NB ? i + 1 : Q * (i - NB + 1); }
  float2 b[Q], a[NA + 1];
  // p[i * stride] = w^{exponent(i)}
  __device__ __forceinline__ void load(float2 const *p, int stride) {
#pragma unroll
    for (int i = 0; i < NB; i++) b[i + 1] = p[i * stride];
#pragma unroll
    for (int i = 0; i < NA; i++) a[i + 1] = p[(NB + i) * stride];
  }
  __device__ __forceinline__ float2 get(int t) const {
    int const qa = t / Q, qb = t - Q * qa;
    if (qa == 0) return b[qb];
    if (qb == 0) return a[qa];
    return cmul(a[qa], b[qb]);
  }
};

struct Cols2sTables {
  float2 const *tw0;   // [Pow<RA>::NP][RB]       W_n1^{j e}
  float2 const *twA;   // [n2][RA]                W_nc^{n2 t}
  float2 const *twB;   // [n2 + 8][Pow<RB>::NP]   (W_nc^{RA n2})^e
};

template <int RA, int RB> struct Cols2sShape {
  static constexpr int TPC = RA > RB ? RA : RB;                // threads per column
  static constexpr bool V128 = (RB % 2 == 0);                  // stage 1 reads with LDS.128
  static constexpr int BLK = V128 ? RB : (RB | 1);             // odd block pitch keeps the LDS.64 path conflict free
  static constexpr int CP = pitch_2mod16(RA * BLK);
  static constexpr int T = 8 * TPC;
  static constexpr int NP0 = Pow<RA>::NP, NP1 = Pow<RB>::NP;
  static constexpr int TW0 = (NP0 * RB + 1) & ~1;              // elements, even (bulk copies move multiples of 16 bytes)
  static constexpr size_t smem = sizeof(float2) * (size_t)(8 * CP + TW0 + 8 * NP1);
};

template <int FMT, int RA, int RB>
__global__ void __launch_bounds__((Cols2sShape<RA, RB>::T), 2) fwd_cols_2s(Pass1Args const a, Cols2sTables const tb) {
  using S = Cols2sShape<RA, RB>;
  constexpr int BLK = S::BLK, CP = S::CP, NP1 = S::NP1, N1 = RA * RB;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  float2 *tile = reinterpret_cast<float2 *>(smem_raw);  // [8][CP]
  float2 *s_tw0 = tile + 8 * CP;                        // [NP0][RB]
  float2 *s_twB = s_tw0 + S::TW0;                       // [8][NP1]
  __shared__ __align__(8) uint64_t tbar;
  int const tid = threadIdx.x;
  int const c = tid & 7, ul = tid >> 3;
  int const c0 = blockIdx.x * 8, blk = blockIdx.y;
  int const n2 = a.n2, ld = a.mid_ld;
  bool const col_ok = c < min(8, n2 - c0);
  int const n2g = c0 + c;
  float2 *mycol = tile + c * CP;
  if (tid == 0) {
    mbar_init(&tbar, 1);
    mbar_fence_init();
    mbar_expect_tx(&tbar, S::TW0 * 8 + 8 * NP1 * 8);
    bulk_g2s(s_tw0, tb.tw0, S::TW0 * 8, &tbar);
    bulk_g2s(s_twB, tb.twB + (long)c0 * NP1, 8 * NP1 * 8, &tbar);  // table padded by 8 columns
  }
  __syncthreads();
  float2 const twA = (col_ok && ul < RA) ? ldg_stream_f2(tb.twA + (long)n2g * RA + ul) : make_float2(1.f, 0.f);

  // ---- stage 0 fused with the load ---------------------------------------------------------------------------------
  unsigned long long energy = 0;
  unsigned int clips = 0;
  if (col_ok && ul < RB) {
    float2 x[RA];
    if (FMT == 0) {
      float2 const *src = reinterpret_cast<float2 const *>(a.in) + (long)blk * a.hop + n2g + (long)ul * n2;
#pragma unroll
      for (int m = 0; m < RA; m++) x[m] = ldg_stream_f2(src + (long)(RB * m) * n2);
    } else {
      int const *src = reinterpret_cast<int const *>(a.in) + (long)blk * a.hop + n2g + (long)ul * n2;
      int raw[RA];
#pragma unroll
      for (int m = 0; m < RA; m++) raw[m] = ldg_stream_b32(src + (long)(RB * m) * n2);
#pragma unroll
      for (int m = 0; m < RA; m++) {
        int lo, hi;
        unpack_i16(raw[m], lo, hi);
        if (FMT == 2) {
          if (a.derandomize) {  // rx888.c:707-712 on the sign-extended words
            lo ^= (lo & 1) ? 0xfffffffe : 0;
            hi ^= (hi & 1) ? 0xfffffffe : 0;
          }
          if (a.stats && (long)(ul + RB * m) * n2 + n2g >= a.first_new) {
            energy += (unsigned long long)(lo * lo) + (unsigned long long)(hi * hi);
            clips += (lo > 32766 || lo < -32766) + (hi > 32766 || hi < -32766);
          }
        }
        x[m] = make_float2(i32_to_f32(lo), i32_to_f32(hi));  // the int16 scale rides on the inter-pass twiddle
      }
    }
    mbar_wait(&tbar, 0);
    Dft<RA, false>::run(x);
    Pow<RA> w;
    w.load(s_tw0 + ul, RB);
    float2 *d = mycol + ul;
    d[0] = x[0];
#pragma unroll
    for (int t = 1; t < RA; t++) d[t * BLK] = cmul(x[t], w.get(t));
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

  // ---- stage 1 fused with the store --------------------------------------------------------------------------------
  if (col_ok && ul < RA) {
    float2 x[RB];
    float2 const *p = mycol + ul * BLK;
    if (S::V128) {
      float4 const *p4 = reinterpret_cast<float4 const *>(p);
#pragma unroll
      for (int m = 0; m < RB / 2; m++) {
        float4 const v = p4[m];
        x[2 * m] = make_float2(v.x, v.y);
        x[2 * m + 1] = make_float2(v.z, v.w);
      }
    } else {
#pragma unroll
      for (int m = 0; m < RB; m++) x[m] = p[m];
    }
    Dft<RB, false>::run(x);
    Pow<RB> w;
    w.load(s_twB + c * NP1, 1);
    float2 const w0 = make_float2(twA.x * a.out_scale, twA.y * a.out_scale);
    float2 *dst = a.mid + (long)blk * N1 * ld + n2g + (long)ul * ld;
    dst[0] = cmul(x[0], w0);
#pragma unroll
    for (int k = 1; k < RB; k++) dst[(long)(RA * k) * ld] = cmul(x[k], cmul(w0, w.get(k)));
  }
}

// ---- row pass, plain complex rows (COMPLEX masters) -------------------------------------------------------------------
template <int RC, int RD> struct Rows2sShape {
  static constexpr int N2 = RC * RD;
  static constexpr int TPC = RC > RD ? RC : RD;
  static constexpr int T = 8 * TPC;
  static constexpr int PITCH = pitch_2mod16(N2 + 1);           // + 1: the bulk copy moves an even number of elements
  static constexpr int NP0 = Pow<RC>::NP;
  static constexpr int TW0 = (NP0 * RD + 1) & ~1;
  static constexpr uint32_t ROW_BYTES = (uint32_t)((N2 + 1) & ~1) * 8u;
  static constexpr size_t smem = sizeof(float2) * (size_t)(8 * PITCH + TW0);
};

template <int RC, int RD>
__global__ void __launch_bounds__((Rows2sShape<RC, RD>::T), 3) fwd_rows_2s(Pass2Args const a, float2 const *tw0) {
  using S = Rows2sShape<RC, RD>;
  constexpr int PITCH = S::PITCH;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  float2 *tile = reinterpret_cast<float2 *>(smem_raw);  // [8][PITCH]
  float2 *s_tw0 = tile + 8 * PITCH;                     // [NP0][RD]  W_n2^{j e}
  __shared__ __align__(8) uint64_t bars[8];
  __shared__ __align__(8) uint64_t tbar;
  int const tid = threadIdx.x;
  int const c = tid & 7, ul = tid >> 3;
  int const blk = blockIdx.y, n1 = a.n1;
  int const row0 = blockIdx.x * 8;
  if (tid < 8) {  // one TMA bulk copy per (contiguous) row; rows of `mid` are padded so that the copy may run one element over
    int const row = row0 + tid;
    mbar_init(&bars[tid], 1);
    if (tid == 0) mbar_init(&tbar, 1);
    mbar_fence_init();
    if (row < n1) {
      mbar_expect_tx(&bars[tid], S::ROW_BYTES);
      bulk_g2s(tile + tid * PITCH, a.mid + ((long)blk * n1 + row) * a.mid_ld, S::ROW_BYTES, &bars[tid]);
    }
    if (tid == 0) {
      mbar_expect_tx(&tbar, S::TW0 * 8);
      bulk_g2s(s_tw0, tw0, S::TW0 * 8, &tbar);
    }
  }
  __syncthreads();
  bool const row_ok = row0 + c < n1;
  float2 *myrow = tile + c * PITCH;
  mbar_wait(&tbar, 0);
  if (row_ok) mbar_wait(&bars[c], 0);
  // ---- stage 0, in place -----------------------------------------------------------------------------------------
  if (row_ok && ul < RD) {
    float2 x[RC];
    float2 *p = myrow + ul;
#pragma unroll
    for (int m = 0; m < RC; m++) x[m] = p[m * RD];
    Dft<RC, false>::run(x);
    Pow<RC> w;
    w.load(s_tw0 + ul, RD);
    p[0] = x[0];
#pragma unroll
    for (int t = 1; t < RC; t++) p[t * RD] = cmul(x[t], w.get(t));
  }
  __syncthreads();
  // ---- stage 1 fused with the store: X[k1 + n1 (t + RC k')] ------------------------------------------------------------
  if (row_ok && ul < RC) {
    float2 x[RD];
    float2 const *p = myrow + ul * RD;
#pragma unroll
    for (int m = 0; m < RD; m++) x[m] = p[m];
    Dft<RD, false>::run(x);
    float2 *dst = a.spec + (long)blk * a.spec_stride + (row0 + c) + (long)n1 * ul;
#pragma unroll
    for (int k = 0; k < RD; k++) dst[(long)n1 * RC * k] = x[k];
  }
}

}  // namespace kfft
