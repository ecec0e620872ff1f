// fwd_cols_r36.cuh -- column pass of the 1296 x n2 two-pass forward transform with TWO fat stages (36 x 36).
//
// A three-stage 12 x 12 x 9 column pass is paced by the L1TEX data pipe, and most of its wavefronts are shared-memory
// traffic: one store, one load + store and one load per point, plus stage twiddles (on H100 it took 14.4 us per cfg-2 block
// against 9.8 for this kernel).  With 1296 = 36 x 36 a point crosses shared memory ONCE (stage 0 store, stage 1 load), there
// is one block barrier instead of two, and the 36-point butterfly is a Good-Thomas 4 x 9 split with no inner twiddles
// (fft_radix.cuh).  Stage 0 reads its 36 inputs straight from global memory (int16 pairs -> float in registers) and
// stage 1 stores X[k1] * W^{n2 k1} straight to the inter-pass buffer, 8 adjacent columns per warp row.
//
// Twiddles: a thread needs W^{j t}, t = 1..35.  Ten are loaded (t = 1..5 and 6, 12, .., 30), the other 25 are one product
// each (t = 6a + b): depth 1, so the rounding error stays at one multiply.  Same for the inter-pass factors
// W_nc^{n2 (t + 36 k')} = A[n2][t] * (W_nc^{36 n2})^{k'}.
// Shared-memory layout: a column is 36 blocks of 36 points padded to 38, column pitch = 2 mod 16: stage 0's stores
// (8 columns x 2 consecutive j) and stage 1's loads are bank-conflict free.  Stage 1 reads its 36 contiguous points with
// 18 LDS.128 (a quarter-warp = the 8 columns of one butterfly: 8 x 16 B at a column pitch of 4 banks = all 32 banks once)
// instead of 36 LDS.64.  Inter-pass rows are padded to 128 B when the row pass is fwd_rows_v2 (N2C = 1250).
#pragma once
#include "static_kernels_v2.cuh"

namespace kfft {

struct ColsR36Tables {
  float2 const *tw0;   // [10][36]  rows 0-4: W_1296^{j b}, b = 1..5; rows 5-9: W_1296^{6 j a}, a = 1..5
  float2 const *twA;   // [n2][36]  W_nc^{n2 t}
  float2 const *twB;   // [n2 + 8][10]  (W_nc^{36 n2})^e, e = 1,2,3,4,5,6,12,18,24,30
};

// w^{t}, t = 6a + b, from the ten loaded powers
__device__ __forceinline__ float2 r36_power(float2 const (&wb)[6], float2 const (&wa)[6], int t) {
  int const a = t / 6, b = t - 6 * a;
  if (a == 0) return wb[b];
  if (b == 0) return wa[a];
  return cmul(wa[a], wb[b]);
}

struct ColsR36Shape {
  static constexpr int BLK = 38, CP = 1378, T = 288;  // 36 * BLK <= CP, CP = 2 mod 16; 8 columns x 36 butterflies
  static constexpr size_t smem = sizeof(float2) * (size_t)(8 * CP + 360 + 80);  // tile, tw0, twB of the 8 columns
};

template <int FMT, int N2C>
__global__ void __launch_bounds__(ColsR36Shape::T, 2) fwd_cols_r36(Pass1Args const a, ColsR36Tables const tb) {
  constexpr int R = 36, BLK = ColsR36Shape::BLK, CP = ColsR36Shape::CP;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  float2 *tile = reinterpret_cast<float2 *>(smem_raw);  // [8][CP]
  float2 *s_tw0 = tile + 8 * CP;                        // [10][36]
  float2 *s_twB = s_tw0 + 360;                          // [8][10]
  __shared__ __align__(8) uint64_t tbar;
  int const tid = threadIdx.x;
  int const c = tid & 7, ul = tid >> 3;  // column of the tile, butterfly 0..35
  int const c0 = blockIdx.x * 8, blk = blockIdx.y;
  int const n2 = N2C ? N2C : a.n2;  // N2C: number of columns as a compile-time constant (0 = from the arguments)
  // rows of the inter-pass buffer padded to whole 128-byte lines: every 64-byte store piece of this kernel then lies in ONE
  // line (with the natural pitch of 10 000 bytes 3 of 8 pieces straddle two: +27 % L1TEX wavefronts for the stores)
  int const ld = N2C ? (N2C + 15) / 16 * 16 : a.mid_ld;
  int const ncols = min(8, n2 - c0);
  bool const col_ok = c < ncols;
  int const n2g = c0 + c;
  float2 *mycol = tile + c * CP;
  if (tid == 0) {
    mbar_init(&tbar, 1);
    mbar_fence_init();
    mbar_expect_tx(&tbar, 360 * 8 + 80 * 8);
    bulk_g2s(s_tw0, tb.tw0, 360 * 8, &tbar);
    bulk_g2s(s_twB, tb.twB + (long)c0 * 10, 80 * 8, &tbar);  // table padded by 8 columns
  }
  __syncthreads();  // barrier initialised before anybody waits on it
  float2 const twA = col_ok ? ldg_stream_f2(tb.twA + (long)n2g * 36 + ul) : make_float2(1.f, 0.f);

  // ---- stage 0 fused with the load: x[j + 36 m], m = 0..35, j = ul --------------------------------------------
  unsigned long long energy = 0;
  unsigned int clips = 0;
  if (col_ok) {
    float2 x[R];
    if (FMT == 0) {
      float2 const *src = reinterpret_cast<float2 const *>(a.in) + (long)blk * a.hop + n2g + (long)ul * n2;
#pragma unroll
      for (int m = 0; m < R; m++) x[m] = ldg_stream_f2(src + (long)(R * m) * n2);
    } else {
      int const *src = reinterpret_cast<int const *>(a.in) + (long)blk * a.hop + n2g + (long)ul * n2;
      int raw[R];
#pragma unroll
      for (int m = 0; m < R; m++) raw[m] = ldg_stream_b32(src + (long)(R * m) * n2);
#pragma unroll
      for (int m = 0; m < R; m++) {
        int lo, hi;
        unpack_i16(raw[m], lo, hi);
        if (FMT == 2) {
          if (a.derandomize) {  // rx888.c:707-712 on the sign-extended words
            lo ^= (lo & 1) ? 0xfffffffe : 0;
            hi ^= (hi & 1) ? 0xfffffffe : 0;
          }
          if (a.stats && (long)(ul + R * m) * n2 + n2g >= a.first_new) {
            energy += (unsigned long long)(lo * lo) + (unsigned long long)(hi * hi);
            clips += (lo > 32766 || lo < -32766) + (hi > 32766 || hi < -32766);
          }
        }
        x[m] = make_float2(i32_to_f32(lo), i32_to_f32(hi));  // the int16 scale rides on the inter-pass twiddle
      }
    }
    mbar_wait(&tbar, 0);
    Dft<R, false>::run(x);
    float2 wb[6], wa[6];
#pragma unroll
    for (int b = 1; b < 6; b++) {
      wb[b] = s_tw0[(b - 1) * 36 + ul];
      wa[b] = s_tw0[(4 + b) * 36 + ul];
    }
    float2 *d = mycol + ul;
    d[0] = x[0];
#pragma unroll
    for (int t = 1; t < R; t++) d[t * BLK] = cmul(x[t], r36_power(wb, wa, t));
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

  // ---- stage 1 fused with the store: sub-transform t = ul, X[t + 36 k'] * W_nc^{n2 (t + 36 k')} -> mid ------------
  if (col_ok) {
    float2 x[R];
    float4 const *p4 = reinterpret_cast<float4 const *>(mycol + ul * BLK);
#pragma unroll
    for (int m = 0; m < R / 2; m++) {
      float4 const v = p4[m];
      x[2 * m] = make_float2(v.x, v.y);
      x[2 * m + 1] = make_float2(v.z, v.w);
    }
    Dft<R, false>::run(x);
    float2 wb[6], wa[6];
#pragma unroll
    for (int b = 1; b < 6; b++) {
      wb[b] = s_twB[c * 10 + (b - 1)];
      wa[b] = s_twB[c * 10 + (4 + b)];
    }
    float2 const w0 = make_float2(twA.x * a.out_scale, twA.y * a.out_scale);
    float2 *dst = a.mid + (long)blk * 1296 * ld + n2g + (long)ul * ld;
    dst[0] = cmul(x[0], w0);
#pragma unroll
    for (int k = 1; k < R; k++) dst[(long)(R * k) * ld] = cmul(x[k], cmul(w0, r36_power(wb, wa, k)));
  }
}

}  // namespace kfft
