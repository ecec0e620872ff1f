// fft_tile.cuh -- shared-memory FFT engine: in-place decimation-in-frequency stages over one
// column of `len` complex points held contiguously in shared memory.
//
// A column is transformed by a group of `nl` cooperating threads (one warp in every kernel of
// this library) that only needs a group-wide barrier between stages, because each butterfly
// reads and writes the same R slots.  After the last stage X[k] sits at the digit-reversed slot
//     k = t0 + r0*t1 + r0*r1*t2 + ...   ->   slot = t0*s0 + t1*s1 + ...,   s_i = len/(r0*..*r_i)
// which the caller resolves through the plan's `perm` table when it streams results out.
#pragma once
#include <stdint.h>
#include "fft_radix.cuh"

namespace kfft {

constexpr int kMaxStages = 8;

// Device-resident description of one column transform (built on the host, see plan.cu).
struct TilePlan {
  int len;                  // transform length
  int nstages;
  int radix[kMaxStages];    // r_i
  int sub[kMaxStages];      // n_i  = length of the sub-transform entering stage i (n_0 = len)
  int stride[kMaxStages];   // s_i  = n_i / r_i
  uint32_t magic[kMaxStages];  // ceil(2^32 / s_i) for the u / s_i split (unused when s_i == 1)
  int tw_off[kMaxStages];   // offset (float2 units) of stage i's twiddles inside `tw`
  float2 const *tw;         // stage twiddles, forward sign: tw[off + (t-1)*s_i + j] = W_{n_i}^{j*t}
  uint16_t const *perm;     // perm[k] = slot holding X[k] after the last stage
};

// Process-wide registry of column plans (filled by get_tile_plan() in kgpu.cu; this header is
// included by exactly one translation unit).  One entry per distinct transform length, never freed:
// every master uses two, every channel rate one.  320 entries hold all 304 lengths the planner can
// ever be asked for (1 .. 7260 points, factors 2, 3, 5, 7; kgpu.cu asserts it), so the registry
// cannot fill.  The table (57.5 KB) is the library's only __constant__ data and must stay inside
// the 64 KB constant bank.
constexpr int kMaxPlans = 320;
static_assert(sizeof(TilePlan) * kMaxPlans <= 60 * 1024, "plan registry must fit the 64 KB constant bank");
__constant__ TilePlan c_plans[kMaxPlans];

// One DIF stage of radix R on one column.  `lane`/`nl`: index and size of the cooperating group.
template <int R, bool INV>
__device__ __forceinline__ void dif_stage(float2 *__restrict__ col, int len, int nsub, int s, uint32_t magic,
                                          float2 const *__restrict__ tw, int lane, int nl) {
  int const nb = len / R;
  for (int u = lane; u < nb; u += nl) {
    int b, j;
    if (s == 1) {
      b = u;
      j = 0;
    } else {
      b = (int)__umulhi((uint32_t)u, magic);
      j = u - b * s;
    }
    float2 *p = col + b * nsub + j;
    float2 x[R];
    constexpr bool kPrefetchTw = (R <= 12);  // bigger radices have no registers to spare
    float2 w[kPrefetchTw ? R : 1];
    if (kPrefetchTw && s > 1) {  // twiddles first: their (L1-resident) latency overlaps the butterfly
#pragma unroll
      for (int t = 1; t < R; t++) w[kPrefetchTw ? t : 0] = __ldg(tw + (t - 1) * s + j);
    }
#pragma unroll
    for (int m = 0; m < R; m++) x[m] = p[m * s];
    Dft<R, INV>::run(x);
    if (s > 1) {
#pragma unroll
      for (int t = 1; t < R; t++) {
        float2 const wt = kPrefetchTw ? w[kPrefetchTw ? t : 0] : __ldg(tw + (t - 1) * s + j);
        x[t] = INV ? cmulc(x[t], wt) : cmul(x[t], wt);
      }
    }
#pragma unroll
    for (int t = 0; t < R; t++) p[t * s] = x[t];
  }
}

// The stages of the extended radices (primes 11 .. 23), which only the extended master kernels compile in.
template <bool INV>
__device__ __forceinline__ void dif_stage_ext(int r, float2 *__restrict__ col, int len, int nsub, int s, uint32_t magic,
                                              float2 const *__restrict__ tw, int lane, int nl) {
  switch (r) {
    case 11: dif_stage<11, INV>(col, len, nsub, s, magic, tw, lane, nl); break;
    case 13: dif_stage<13, INV>(col, len, nsub, s, magic, tw, lane, nl); break;
    case 17: dif_stage<17, INV>(col, len, nsub, s, magic, tw, lane, nl); break;
    case 19: dif_stage<19, INV>(col, len, nsub, s, magic, tw, lane, nl); break;
    case 23: dif_stage<23, INV>(col, len, nsub, s, magic, tw, lane, nl); break;
    default: break;
  }
}

// All stages of a plan on one column.  SYNC() is the group barrier (e.g. __syncwarp).  EXT also dispatches the
// extended radices; without it the switch is exactly the one every registry-plan kernel inlines.
template <bool INV, bool EXT = false, typename Sync>
__device__ __forceinline__ void tile_fft(TilePlan const &pl, float2 *col, int lane, int nl, Sync sync) {
  for (int i = 0; i < pl.nstages; i++) {
    int const r = pl.radix[i], n = pl.sub[i], s = pl.stride[i];
    uint32_t const mg = pl.magic[i];
    float2 const *tw = pl.tw + pl.tw_off[i];
    switch (r) {
#define KFFT_CASE(RR) \
  case RR: dif_stage<RR, INV>(col, pl.len, n, s, mg, tw, lane, nl); break;
      KFFT_CASE(2)
      KFFT_CASE(3)
      KFFT_CASE(4)
      KFFT_CASE(5)
      KFFT_CASE(6)
      KFFT_CASE(7)
      KFFT_CASE(8)
      KFFT_CASE(9)
      KFFT_CASE(10)
      KFFT_CASE(12)
      KFFT_CASE(15)
      KFFT_CASE(16)
      KFFT_CASE(20)
      KFFT_CASE(24)
      KFFT_CASE(25)
      KFFT_CASE(36)
#undef KFFT_CASE
      default:
        if constexpr (EXT) dif_stage_ext<INV>(r, col, pl.len, n, s, mg, tw, lane, nl);
        break;
    }
    sync();
  }
}

}  // namespace kfft
