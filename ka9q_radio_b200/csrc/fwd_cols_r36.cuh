// fwd_cols_r36.cuh -- column pass of the 1296 x n2 two-pass forward transform with TWO fat stages (36 x 36).
//
// A three-stage 12 x 12 x 9 column pass is paced by the L1TEX data pipe, and most of its wavefronts are shared-memory
// traffic: one store, one load + store and one load per point, plus stage twiddles (on H100 it took 14.4 us per cfg-2 block
// against 9.8 for this kernel).  With 1296 = 36 x 36 a point crosses shared memory ONCE (stage 0 store, stage 1 load), there
// is one block barrier instead of two, and the 36-point butterfly is a Good-Thomas 4 x 9 split with no inner twiddles
// (fft_radix.cuh).  Stage 0 reads its 36 inputs from global memory, or from the tile tensor copies fetched
// (fwd_cols_r36_tma, below), converting int16 pairs to floats in registers, and
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
#include <cuda.h>  // CUtensorMap (a type only: the library does not link the driver)

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

// ---- the raw tile by tensor copies: fwd_cols_r36_tma ------------------------------------------------------------------
// With global loads a warp's stage-0 load reads 4 rows x 32 bytes (int16) or x 64 bytes (float); at the row pitch of n2
// points most of those pieces straddle a 32-byte sector, and all 36 loads of a thread occupy the LSU pipe that the
// shared-memory traffic of both stages also needs.  fwd_cols_r36_tma has the tensor-memory accelerator copy the CTA's
// 8 columns x 1296 rows into shared memory instead (tensor maps built by the host per launch, kgpu.cu cols_tma_map);
// stage 0 then reads its inputs from there and does exactly what the global-load form does with them.  Every box starts
// 16-byte aligned in global memory, inside the rows it covers.
//  * float (FMT 0): map [2 n2 floats][n1 rows][nblocks], 6 boxes of 16 floats x 216 rows, one 64-byte row after the
//    other.  A warp's rows ul = 4w .. 4w+3 are 256 contiguous bytes: LDS.64 without bank conflicts.
//  * int16 (FMT 1, 2): the row pitch 4 n2 bytes is not a multiple of 16, so the map's rows are row pairs of 32-bit words
//    (one int16 pair each): [2 n2 words][n1/2 pairs][nblocks].  Even rows are the first half of a pair (x = c0), odd rows
//    the second (x = n2 + c0), which starts 8 bytes off 16-byte alignment when n2 = 2 mod 4: their boxes start
//    s = n2 & 2 words earlier.  Both parities take boxes 12 words wide (48 bytes: the 8 columns and the s words before
//    them), 3 boxes of 216 pairs each.  A thread's rows ul + 36m all have the parity of ul.  At a pitch of 12 words the
//    even and odd pieces a warp reads share banks: its LDS.32 take 2 wavefronts, as the LDS.64 of the float form do.
// The raw tile lies in the float tile's memory: a CTA barrier separates the last raw read from stage 0's first store.
// Columns past n2 (the last group of 1250 = 156 * 8 + 2) hold zeros or the next row's first words and are never used.
struct ColsR36Tma {
  static constexpr int BOX_ROWS = 216;  // rows (float) or row pairs (int16) of a box: 1296 = 6 x 216 = 2 x 3 x 216
  static constexpr int F32_BOX_BYTES = BOX_ROWS * 64;
  static constexpr int I16_BOX_WORDS = 12, I16_BOX_BYTES = BOX_ROWS * I16_BOX_WORDS * 4;
  static constexpr int I16_ODD_OFF = 3 * I16_BOX_BYTES;  // the odd rows' boxes, after the even rows' ones
  static constexpr uint32_t bytes(int fmt) { return fmt == 0 ? 6 * F32_BOX_BYTES : 6 * I16_BOX_BYTES; }
};
static_assert(ColsR36Tma::bytes(0) + 112 <= sizeof(float2) * 8 * ColsR36Shape::CP &&
              ColsR36Tma::bytes(1) + 112 <= sizeof(float2) * 8 * ColsR36Shape::CP, "the raw tile lies in the float tile");
static_assert(ColsR36Tma::F32_BOX_BYTES % 128 == 0 && ColsR36Tma::I16_BOX_BYTES % 128 == 0, "box destinations 128-B aligned");

// one int16 pair of stage 0 -> float2, with de-randomisation and the statistics of FMT 2; row, col: its place in the window
template <int FMT>
__device__ __forceinline__ float2 r36_ingest(int raw, int row, int col, int n2, Pass1Args const &a, unsigned long long &energy,
                                             unsigned int &clips) {
  int lo, hi;
  unpack_i16(raw, lo, hi);
  if (FMT == 2) {
    if (a.derandomize) {  // rx888.c:707-712 on the sign-extended words
      lo ^= (lo & 1) ? 0xfffffffe : 0;
      hi ^= (hi & 1) ? 0xfffffffe : 0;
    }
    if (a.stats && (long)row * n2 + col >= a.first_new) {
      energy += (unsigned long long)(lo * lo) + (unsigned long long)(hi * hi);
      clips += (lo > 32766 || lo < -32766) + (hi > 32766 || hi < -32766);
    }
  }
  return make_float2(i32_to_f32(lo), i32_to_f32(hi));  // the int16 scale rides on the inter-pass twiddle
}

// stage 0's twiddles and its stores into the float tile
__device__ __forceinline__ void r36_stage0_store(float2 (&x)[36], float2 const *s_tw0, float2 *d, int ul) {
  constexpr int R = 36, BLK = ColsR36Shape::BLK;
  float2 wb[6], wa[6];
#pragma unroll
  for (int b = 1; b < 6; b++) {
    wb[b] = s_tw0[(b - 1) * 36 + ul];
    wa[b] = s_tw0[(4 + b) * 36 + ul];
  }
  d[0] = x[0];
#pragma unroll
  for (int t = 1; t < R; t++) d[t * BLK] = cmul(x[t], r36_power(wb, wa, t));
}

// One column tile: columns c0 .. c0+7 of block blk, by the 288 threads tid = 0..287 that `sync` (a barrier of exactly
// those threads) joins, in ColsR36Shape::smem bytes of shared memory at smem_raw (16-byte aligned), with tbar its
// copies' mbarrier.  The kernels below run one tile per CTA; fwd_fused_r36_v2 (fwd_fused.cuh) two side by side.
template <int FMT, int N2C, bool TMA, class Sync>
__device__ __forceinline__ void fwd_cols_r36_body(Pass1Args const &a, ColsR36Tables const &tb, CUtensorMap const *tmap,
                                                  unsigned char *smem_raw, uint64_t &tbar, int tid, int c0, int blk,
                                                  Sync const &sync) {
  constexpr int R = 36, BLK = ColsR36Shape::BLK, CP = ColsR36Shape::CP;
  float2 *tile = reinterpret_cast<float2 *>(smem_raw);  // [8][CP]
  float2 *s_tw0 = tile + 8 * CP;                        // [10][36]
  float2 *s_twB = s_tw0 + 360;                          // [8][10]
  int const c = tid & 7, ul = tid >> 3;  // column of the tile, butterfly 0..35
  int const n2 = N2C ? N2C : a.n2;  // N2C: number of columns as a compile-time constant (0 = from the arguments)
  // rows of the inter-pass buffer padded to whole 128-byte lines: every 64-byte store piece of this kernel then lies in ONE
  // line (with the natural pitch of 10 000 bytes 3 of 8 pieces straddle two: +27 % L1TEX wavefronts for the stores)
  int const ld = N2C ? (N2C + 15) / 16 * 16 : a.mid_ld;
  int const ncols = min(8, n2 - c0);
  bool const col_ok = c < ncols;
  int const n2g = c0 + c;
  float2 *mycol = tile + c * CP;
  // tensor copies land 128-byte aligned (an extern alignment of 128 would move every kernel's shared memory)
  unsigned char *const rtile = smem_raw + ((0u - smem_u32(smem_raw)) & 127u);
  if (tid == 0) {
    mbar_init(&tbar, 1);
    mbar_fence_init();
    if constexpr (TMA) {
      using T = ColsR36Tma;
      mbar_expect_tx(&tbar, 360 * 8 + 80 * 8 + T::bytes(FMT));
      if (FMT == 0) {
#pragma unroll
        for (int k = 0; k < 6; k++) tensor_g2s_3d(rtile + k * T::F32_BOX_BYTES, tmap, 2 * c0, k * T::BOX_ROWS, blk, &tbar);
      } else {
#pragma unroll
        for (int k = 0; k < 3; k++) {
          tensor_g2s_3d(rtile + k * T::I16_BOX_BYTES, tmap, c0, k * T::BOX_ROWS, blk, &tbar);
          tensor_g2s_3d(rtile + T::I16_ODD_OFF + k * T::I16_BOX_BYTES, tmap, n2 + c0 - (n2 & 2), k * T::BOX_ROWS, blk, &tbar);
        }
      }
    } else {
      mbar_expect_tx(&tbar, 360 * 8 + 80 * 8);
    }
    bulk_g2s(s_tw0, tb.tw0, 360 * 8, &tbar);
    bulk_g2s(s_twB, tb.twB + (long)c0 * 10, 80 * 8, &tbar);  // table padded by 8 columns
  }
  sync();  // barrier initialised before anybody waits on it
  float2 const twA = col_ok ? ldg_stream_f2(tb.twA + (long)n2g * 36 + ul) : make_float2(1.f, 0.f);

  // ---- stage 0 fused with the load: x[j + 36 m], m = 0..35, j = ul --------------------------------------------
  unsigned long long energy = 0;
  unsigned int clips = 0;
  if constexpr (TMA) {
    float2 x[R];
    mbar_wait(&tbar, 0);
    if (col_ok) {
      if (FMT == 0) {
        float2 const *src = reinterpret_cast<float2 const *>(rtile) + ul * 8 + c;
#pragma unroll
        for (int m = 0; m < R; m++) x[m] = src[R * 8 * m];
      } else {
        using T = ColsR36Tma;
        int const odd = ul & 1;
        int const *src = reinterpret_cast<int const *>(rtile + odd * T::I16_ODD_OFF) + (ul >> 1) * T::I16_BOX_WORDS + c +
                         odd * (n2 & 2);
#pragma unroll
        for (int m = 0; m < R; m++)
          x[m] = r36_ingest<FMT>(src[(R / 2) * T::I16_BOX_WORDS * m], ul + R * m, n2g, n2, a, energy, clips);
      }
      Dft<R, false>::run(x);
    }
    sync();  // the raw tile is read: stage 0 may overwrite it
    if (col_ok) r36_stage0_store(x, s_tw0, mycol + ul, ul);
  } else if (col_ok) {
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
      for (int m = 0; m < R; m++) x[m] = r36_ingest<FMT>(raw[m], ul + R * m, n2g, n2, a, energy, clips);
    }
    mbar_wait(&tbar, 0);
    Dft<R, false>::run(x);
    r36_stage0_store(x, s_tw0, mycol + ul, ul);
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
  sync();

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

// stage 0 from global loads: any input layout
template <int FMT, int N2C>
__global__ void __launch_bounds__(ColsR36Shape::T, 2) fwd_cols_r36(Pass1Args const a, ColsR36Tables const tb) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  __shared__ __align__(8) uint64_t tbar;
  fwd_cols_r36_body<FMT, N2C, false>(a, tb, nullptr, smem_raw, tbar, threadIdx.x, blockIdx.x * 8, blockIdx.y,
                                     [] { __syncthreads(); });
}
// stage 0 from the raw tile the tensor copies fetch: inputs whose tensor map the host could build (kgpu.cu cols_tma_fits)
template <int FMT, int N2C>
__global__ void __launch_bounds__(ColsR36Shape::T, 2)
    fwd_cols_r36_tma(Pass1Args const a, ColsR36Tables const tb, const __grid_constant__ CUtensorMap tmap) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  __shared__ __align__(8) uint64_t tbar;
  fwd_cols_r36_body<FMT, N2C, true>(a, tb, &tmap, smem_raw, tbar, threadIdx.x, blockIdx.x * 8, blockIdx.y,
                                    [] { __syncthreads(); });
}

}  // namespace kfft
