// small_master.cuh -- a whole small master in one kernel: radiod's per-channel secondary masters (filter2 of CW and ISB
// channels, the wfm / stereod / rdsd composite, packetd, ctcss) write a few thousand samples per block and read their
// slaves back at once, so the front end's machinery (two forward passes, a channel bank, one launch per path class,
// powers, spectrum windows) is mostly overhead for them.  Here one CTA owns one block of one master:
//   1. its window -> the forward transform in shared memory, on chan_wide's four-step geometry (WideGeom, registry
//      plans); a REAL master transforms Nc = N/2 packed points and splits them as the forward passes do, giving the
//      bin layout of kgpu_master_spec_stride (N/2 + 1 bins, rows padded to 4)
//   2. the spectrum -> the master's ring slot, which the recompute-one-slave entry reads after a retune
//   3. each slave in turn: chan_slice's walk x response (ISB fold, Nyquist zero, REAL Hermitian half), the inverse in
//      shared memory, the last olen samples into the output row
// With `only` >= 0 it skips steps 1-2 and runs step 3 for that slave alone, from the spectrum stored in the slot.  The
// spectrum is read back with plain loads: this kernel wrote it, so the read-only (non-coherent) path is not used.
#pragma once
#include "chan_wide.cuh"

namespace kfft {

constexpr int kSmallMaxSlaves = 8;

struct SmallSlave {
  ChanDesc d;          // plan < 0: not run; points, olen, walk, flags (kChanIsb, kChanRealOut), out_off
  WideGeom g;          // the inverse's four-step geometry
  float2 const *resp;  // the response in set_filter's layout
};

struct SmallArgs {
  void const *in;     // block 0's window: N floats (REAL, read as Nc packed pairs) or N float2 (COMPLEX)
  long hop;           // float2 between consecutive windows: L/2 (REAL), L (COMPLEX)
  WideGeom fg;        // the forward transform's geometry, Nc = fg.n1 * fg.n2 points
  int real;           // REAL master: real split after the forward transform
  float2 *spec;       // [block][spec_stride]: this launch's ring slots
  long spec_stride;
  int m_bins;         // N/2 + 1 (REAL) or N (COMPLEX)
  float2 *out;        // [block][out_stride]: output rows, slave i at s[i].d.out_off
  long out_stride;
  int nslaves;
  int only;           // >= 0: step 3 for slave `only` from the stored spectrum
  SmallSlave s[kSmallMaxSlaves];
};

// Step 1-2 for one block: the forward transform of the window at `in` into X (bins m_bins).
__device__ __forceinline__ void small_forward(SmallArgs const &a, float2 const *in, float2 *X, float2 *col) {
  WideGeom const &g = a.fg;
  int const nc = g.n1 * g.n2, tid = threadIdx.x, nt = blockDim.x;
  for (int k = tid; k < nc; k += nt) col[wide_in_slot(g, k)] = in[k];
  __syncthreads();
  wide_transform<false>(g, col);
  uint16_t const *perm1 = c_plans[g.plan1].perm, *perm2 = c_plans[g.plan2].perm;
  if (!a.real) {
    for (int k = tid; k < nc; k += nt) X[k] = col[wide_out_slot(g, perm1, perm2, k)];
    return;
  }
  // z[n] = x[2n] + i x[2n+1], Z = DFT_Nc(z):  X[k] = E - i W_N^k O,  E = (Z[k] + conj Z[Nc-k]) / 2,
  // O = (Z[k] - conj Z[Nc-k]) / 2, for k = 0 .. Nc (fwd_kernels.cuh's split, one bin per thread step)
  for (int k = tid; k <= nc; k += nt) {
    float2 const za = col[wide_out_slot(g, perm1, perm2, k == nc ? 0 : k)];
    float2 const zb = col[wide_out_slot(g, perm1, perm2, k == 0 ? 0 : nc - k)];
    float2 const w = unit_root_f(k, 2L * nc);
    float2 const E = make_float2(0.5f * (za.x + zb.x), 0.5f * (za.y - zb.y));
    float2 const O = make_float2(0.5f * (za.x - zb.x), 0.5f * (za.y + zb.y));
    float2 const P = cmul(w, O);
    X[k] = make_float2(E.x + P.y, E.y - P.x);
  }
}

// Step 3 for one slave and one block: X is this block's spectrum, dst the slave's run of the output row.
__device__ __forceinline__ void small_slave(SmallArgs const &a, SmallSlave const &s, float2 const *X, float2 *col, float2 *dst) {
  ChanDesc const &d = s.d;
  WideGeom const &g = s.g;
  int const ns = d.points, top = (ns + 1) / 2, tid = threadIdx.x, nt = blockDim.x;
  ChanArgs ca{};
  ca.m_bins = a.m_bins;
  ca.wrap = !a.real;
  float2 const *R = s.resp;
  if (d.flags & kChanRealOut) {
    for (int si = tid; si < ns / 2 + 1; si += nt) {
      float2 const v = real_half_at(ca, d, [X](int q) { return X[q]; }, R, si);
      if (si == 0 || 2 * si == ns) {
        col[wide_in_slot(g, si)] = make_float2(v.x, 0.f);
      } else {
        col[wide_in_slot(g, si)] = v;
        col[wide_in_slot(g, ns - si)] = make_float2(v.x, -v.y);
      }
    }
  } else {
    for (int w = tid; w < ns; w += nt) {
      bool live;
      int const u = walk_pos(d, ns, top, w, live);
      col[wide_in_slot(g, w)] = live ? slice_product(d, X[walk_bin(ca, d, u)], __ldg(R + w)) : make_float2(0.f, 0.f);
    }
  }
  __syncthreads();
  if (d.flags & kChanIsb) {
    for (int p = 1 + tid; p < ns / 2; p += nt) isb_fold(col[wide_in_slot(g, p)], col[wide_in_slot(g, ns - p)]);
    if (tid == 0) {
      col[wide_in_slot(g, 0)] = make_float2(0.f, 0.f);
      col[wide_in_slot(g, top)] = make_float2(0.f, 0.f);
    }
    __syncthreads();
  }
  wide_transform<true>(g, col);
  uint16_t const *perm1 = c_plans[g.plan1].perm, *perm2 = c_plans[g.plan2].perm;
  int const first = ns - d.olen;
  if (d.flags & kChanRealOut) {  // c2r: the real part, olen floats packed in the slave's float2 run
    float *dr = reinterpret_cast<float *>(dst);
    for (int i = tid; i < d.olen; i += nt) dr[i] = col[wide_out_slot(g, perm1, perm2, first + i)].x;
  } else {
    for (int i = tid; i < d.olen; i += nt) dst[i] = col[wide_out_slot(g, perm1, perm2, first + i)];
  }
}

// grid = the launch's blocks, one CTA each; dynamic shared memory = the largest geometry's wide_smem_bytes.
__global__ void __launch_bounds__(kWideThreads, 1) small_master_kernel(__grid_constant__ SmallArgs const a) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  float2 *col = reinterpret_cast<float2 *>(smem_raw);
  int const blk = blockIdx.x;
  float2 *X = a.spec + (long)blk * a.spec_stride;
  if (a.only < 0) {
    small_forward(a, reinterpret_cast<float2 const *>(a.in) + (long)blk * a.hop, X, col);
    __syncthreads();  // the spectrum (global) is complete and the shared memory free for the slaves
  }
  int const lo = a.only < 0 ? 0 : a.only, hi = a.only < 0 ? a.nslaves : a.only + 1;
  for (int i = lo; i < hi; i++) {
    SmallSlave const &s = a.s[i];
    if (s.d.plan < 0) continue;
    small_slave(a, s, X, col, a.out + (long)blk * a.out_stride + s.d.out_off);
    __syncthreads();
  }
}

}  // namespace kfft
