// fft_static.cuh -- compile-time specialised version of the shared-memory column transform.
//
// Same algorithm and table layout as fft_tile.cuh (in-place DIF, digit-reversed result, stage
// twiddles tw[off_i + (t-1)*s_i + j]) but the length and radix sequence are template
// parameters: strides, loop trip counts and the index splits are literals, the stage loop is
// unrolled, and the digit reversal is arithmetic instead of a table load.  Used by the kernels
// instantiated for the sizes the configured workloads hit; every other size takes the generic
// (runtime-plan) kernels.
#pragma once
#include "fft_radix.cuh"

namespace kfft {

template <int LEN, int... RS> struct SPlan {
  static constexpr int len = LEN;
  static constexpr int nst = sizeof...(RS);
  static constexpr int rad_arr[sizeof...(RS) > 0 ? sizeof...(RS) : 1] = {RS...};
  static constexpr int rad(int i) { return rad_arr[i]; }
  static constexpr int nsub(int i) {  // length of the sub-transform entering stage i
    int n = LEN;
    for (int k = 0; k < i; k++) n /= rad_arr[k];
    return n;
  }
  static constexpr int stride(int i) { return nsub(i) / rad_arr[i]; }
  static constexpr int tw_off(int i) {
    int o = 0;
    for (int k = 0; k < i; k++)
      if (stride(k) > 1) o += (rad_arr[k] - 1) * stride(k);
    return o;
  }
  static constexpr bool valid() {
    int p = 1;
    for (int k = 0; k < nst; k++) p *= rad_arr[k];
    return p == LEN;
  }
};

// slot holding X[k] after the last stage: digits of k in the mixed radix (r0, r1, ...)
template <class P, int I = 0> struct SlotOf {
  static __device__ __forceinline__ int run(int rem) {
    constexpr int R = P::rad(I), S = P::stride(I);
    int const q = rem / R;
    return (rem - q * R) * S + SlotOf<P, I + 1>::run(q);
  }
};
template <class P> struct SlotOf<P, P::nst> {
  static __device__ __forceinline__ int run(int) { return 0; }
};
template <class P> __device__ __forceinline__ int static_slot(int k) { return SlotOf<P>::run(k); }

// number of stage-twiddle entries of plan P (same layout as the registry table)
template <class P> constexpr int static_tw_count() { return P::tw_off(P::nst); }

// streaming global load that does not displace the L1-resident tables
__device__ __forceinline__ int ldg_stream_b32(int const *p) {
  int v;
  asm volatile("ld.global.nc.L1::no_allocate.b32 %0, [%1];" : "=r"(v) : "l"(p));
  return v;
}
__device__ __forceinline__ float2 ldg_stream_f2(float2 const *p) {
  float2 v;
  asm volatile("ld.global.nc.L1::no_allocate.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "l"(p));
  return v;
}

// One butterfly of stage I at butterfly index u: load / transform / twiddle / store helpers.
template <class P, int I> struct StageGeom {
  static constexpr int R = P::rad(I), NSUB = P::nsub(I), S = P::stride(I), NB = P::len / R;
  static __device__ __forceinline__ void split(int u, int &b, int &j) {
    if (S == 1) {
      b = u;
      j = 0;
    } else {
      b = u / S;
      j = u - b * S;
    }
  }
};

// TWS: the twiddle table pointer is in shared memory (plain loads) instead of global (__ldg).
// ILP: butterflies of consecutive loop iterations handled together (loads of all first, then the
// arithmetic, then the stores) so one warp keeps ILP independent chains in flight.
template <class P, bool INV, int I, bool TWS, int ILP>
__device__ __forceinline__ void static_stage(float2 *__restrict__ col, float2 const *__restrict__ tw, int lane) {
  using G = StageGeom<P, I>;
  constexpr int R = G::R, NSUB = G::NSUB, S = G::S, NB = G::NB, NL = 32;
  constexpr int ITERS = (NB + NL - 1) / NL;
  float2 const *twi = tw + P::tw_off(I);
#pragma unroll
  for (int it0 = 0; it0 < ITERS; it0 += ILP) {
    float2 x[ILP][R];
    float2 *p[ILP];
    int jj[ILP];
    bool ok[ILP];
#pragma unroll
    for (int q = 0; q < ILP; q++) {
      int const u = lane + NL * (it0 + q);
      ok[q] = (it0 + q < ITERS) && ((NB % NL == 0) || it0 + q + 1 < ITERS || u < NB);
      int b, j;
      G::split(ok[q] ? u : 0, b, j);
      jj[q] = j;
      p[q] = col + b * NSUB + j;
      if (ok[q]) {
#pragma unroll
        for (int m = 0; m < R; m++) x[q][m] = p[q][m * S];
      }
    }
#pragma unroll
    for (int q = 0; q < ILP; q++) {
      if (ok[q]) {
        Dft<R, INV>::run(x[q]);
        if (S > 1) {
#pragma unroll
          for (int t = 1; t < R; t++) {
            float2 const w = TWS ? twi[(t - 1) * S + jj[q]] : __ldg(twi + (t - 1) * S + jj[q]);
            x[q][t] = INV ? cmulc(x[q][t], w) : cmul(x[q][t], w);
          }
        }
      }
    }
#pragma unroll
    for (int q = 0; q < ILP; q++) {
      if (ok[q]) {
#pragma unroll
        for (int t = 0; t < R; t++) p[q][t * S] = x[q][t];
      }
    }
  }
}

template <class P, bool INV, bool TWS = false, int ILP = 1, int I = 0> struct StaticFft {
  static __device__ __forceinline__ void run(float2 *col, float2 const *tw, int lane) {
    // big radices have no registers for a second butterfly
    static_stage<P, INV, I, TWS, (P::rad(I) <= 12 ? ILP : 1)>(col, tw, lane);
    __syncwarp();
    StaticFft<P, INV, TWS, ILP, I + 1>::run(col, tw, lane);
  }
};
template <class P, bool INV, bool TWS, int ILP> struct StaticFft<P, INV, TWS, ILP, P::nst> {
  static __device__ __forceinline__ void run(float2 *, float2 const *, int) {}
};

// ---- shared-memory bulk copies (TMA, 1-D): cp.async.bulk + mbarrier -------------------------
__device__ __forceinline__ uint32_t smem_u32(void const *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t *bar, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void *dst, void const *src, uint32_t bytes, uint64_t *bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)),
               "l"(src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
// a box of a 3-D tensor map into shared memory (128-byte aligned); coordinates in elements, outside the tensor zero-filled
__device__ __forceinline__ void tensor_g2s_3d(void *dst, void const *map, int x, int y, int z, uint64_t *bar) {
  asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];"
               ::"r"(smem_u32(dst)), "l"(map), "r"(x), "r"(y), "r"(z), "r"(smem_u32(bar))
               : "memory");
}
// orders this thread's earlier generic-proxy view of global memory (what an acquire made visible) before its later
// async-proxy accesses (bulk and tensor copies)
__device__ __forceinline__ void fence_proxy_async_global() { asm volatile("fence.proxy.async.global;" ::: "memory"); }
// drops one 128-byte L2 line (128-byte aligned) without writing it back: its contents become undefined
__device__ __forceinline__ void discard_l2_line(void *p) { asm volatile("discard.global.L2 [%0], 128;" ::"l"(p) : "memory"); }
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "WAIT_%=:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra DONE_%=;\n\t"
      "bra WAIT_%=;\n\t"
      "DONE_%=:\n\t}" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}

}  // namespace kfft
