// fwd_fused.cuh -- the column and row passes of REAL 1296 x 1250 masters (fwd_cols_r36_tma + fwd_rows_v2<true, 1296,
// true>) as ONE launch, so that each block's inter-pass buffer is read back from L2 while it is still there.
//
// Run as two launches, the column pass writes all B blocks' inter-pass rows (13.1 MB per block) before the row pass reads
// the first of them: the buffer goes to DRAM and comes back, 26 of the ~55 MB that cross HBM per cfg-2 block.  Here
// the launch's CTAs are work items of two kinds, taken in ticket order:
//   C(b, x)  column tiles 2x and 2x+1 of block b: fwd_cols_r36_body, two 288-thread tiles side by side;
//   R(b, y)  row pairs 8y .. 8y+7 of block b: fwd_rows_v2_body (REAL, halved), 512 threads, the other 64 leave.
// Ticket order: C(0, *), then for each block b, R(b, *) interleaved with C(b+1, *) (fused_item), so that a block's rows
// are read while about one block of inter-pass rows is in L2.  Optionally (FusedArgs::discard) each row's lines are
// discarded from L2 once its copy has landed, so that they are never written back; on H100 that measured slower.
// Same bodies, same instructions on the same values as the two-kernel pair: spectra and IngestStats are bitwise equal.
#pragma once
#include "fwd_cols_r36.cuh"
#include "static_kernels_v2.cuh"

namespace kfft {

struct FusedShape {
  static constexpr int N1 = 1296, N2 = 1250;
  static constexpr int TILES = (N2 + 7) / 8;                       // column tiles per block: 157
  static constexpr int NC = (TILES + 1) / 2;                       // C items per block: 79
  static constexpr int NR = (N1 / 2 + 1 + RowsV2Shape<true>::IPC - 1) / RowsV2Shape<true>::IPC;  // R items per block: 82
  static constexpr int T = 2 * ColsR36Shape::T;                    // 576 threads, 1 CTA per SM: 18 warps, 5 on some of the 4 SM sub-partitions, so <= 96 registers
  static constexpr int RT = RowsV2Shape<true>::T;                  // threads of an R item: 512
  static constexpr size_t smem = 2 * ColsR36Shape::smem > RowsV2Shape<true>::smem ? 2 * ColsR36Shape::smem : RowsV2Shape<true>::smem;
  static constexpr int DEFAULT_LEAD = 40;
  static_assert(ColsR36Shape::smem % 16 == 0, "the second tile's memory 16-byte aligned");
  static_assert(T % 32 == 0 && ColsR36Shape::T % 32 == 0 && RT % 32 == 0, "whole warps per tile and per R item");
};

enum FusedKind : int { kFusedCol = 0, kFusedRow = 1 };
struct FusedItem {
  int kind, blk, idx;  // C(blk, idx) or R(blk, idx)
};

// The item of ticket t (0 <= t < nblocks * (NC + NR)).  Tickets 0 .. NC-1 are C(0, *).  Then, for b = 0 .. nblocks-1,
// a phase of NR + NC tickets (NR in the last): `lead` items C(b+1, 0 .. lead-1) first, then R(b, y) and C(b+1, lead + y)
// alternately, then the rest of R(b, *).  lead (0 .. NC) spaces R(b, 0) from the last C(b, *) by NR - NC + 2 lead + 1
// tickets, so that the CTAs that take the first rows of a block seldom find its columns still running.
// Only R(b, *) waits, on every C(b, *), and all of those come in an earlier phase: every wait is on smaller tickets.
__host__ __device__ __forceinline__ FusedItem fused_item(int t, int nblocks, int lead) {
  using F = FusedShape;
  if (t < F::NC) return {kFusedCol, 0, t};
  t -= F::NC;
  int const b = t / (F::NR + F::NC), p = t - b * (F::NR + F::NC);
  if (b >= nblocks - 1) return {kFusedRow, nblocks - 1, t - (nblocks - 1) * (F::NR + F::NC)};
  if (p < lead) return {kFusedCol, b + 1, p};
  int const q = p - lead, m = F::NC - lead;
  if (q < 2 * m) return (q & 1) ? FusedItem{kFusedCol, b + 1, lead + q / 2} : FusedItem{kFusedRow, b, q / 2};
  return {kFusedRow, b, q - m};
}

struct FusedArgs {
  unsigned *ctr;  // [0]: tickets taken; [1 + b]: C items of block b done.  Zeroed before each launch.
  int nblocks, lead;
  int discard;    // discard each inter-pass row from L2 once read (measured slower on H100: off by default)
};

__device__ __forceinline__ void red_release_gpu_add(unsigned *p, unsigned v) {
  asm volatile("red.release.gpu.global.add.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ unsigned ld_acquire_gpu(unsigned const *p) {
  unsigned v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}

// Progress.  A CTA takes its ticket with one atomicAdd after it is resident, so every smaller ticket is held by a CTA
// that is resident or has finished.  C items wait on nothing, so they finish.  An R item waits only on C items of
// smaller tickets (fused_item), which by induction all finish.  So every wait ends, whatever order the hardware
// dispatches the CTAs in and however many fit at once.  There is no reuse of inter-pass memory between items (one slot
// per block), so there are no write-after-read waits.
// Ordering.  A C item's threads meet at a CTA barrier; one thread then releases (fence + red.release.gpu) the block's
// done counter.  One thread of an R item acquires it (ld.acquire.gpu) until it reaches NC, its 512 threads meet at a
// barrier, and each thread that issues a row's bulk copy orders it after the acquire through fence.proxy.async.global:
// the copies read through the async proxy what other SMs stored through the generic proxy.
// Barriers: 0 (all 576 threads) around the ticket and at the end of a C item; 1 and 2 the column tiles' (288 each);
// in an R item 1 and 2 the row groups' (256 each), 3 the 512 threads'.
template <int FMT>
__global__ void __launch_bounds__(FusedShape::T, 1)
    fwd_fused_r36_v2(Pass1Args const a1, ColsR36Tables const t1, Pass2Args const a2, FwdTables const t2, FusedArgs const f,
                     const __grid_constant__ CUtensorMap tmap) {
  using F = FusedShape;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  __shared__ __align__(8) uint64_t bars[RowsV2Shape<true>::COLS];
  __shared__ __align__(8) uint64_t tbar[2];
  __shared__ int s_ticket;
  int const tid = threadIdx.x;
  if (tid == 0) s_ticket = (int)atomicAdd(f.ctr, 1u);
  __syncthreads();
  FusedItem const it = fused_item(s_ticket, f.nblocks, f.lead);
  if (it.kind == kFusedCol) {
    int const h = tid >= ColsR36Shape::T, tile = 2 * it.idx + h;
    if (tile < F::TILES)
      fwd_cols_r36_body<FMT, F::N2, true>(a1, t1, &tmap, smem_raw + h * ColsR36Shape::smem, tbar[h], tid - h * ColsR36Shape::T,
                                           tile * 8, it.blk, [h] {
                                             asm volatile("bar.sync %0, %1;" ::"r"(1 + h), "n"(ColsR36Shape::T) : "memory");
                                           });
    __syncthreads();
    if (tid == 0) {  // the item again from its ticket: nothing of it stays live across the tiles
      __threadfence();
      red_release_gpu_add(f.ctr + 1 + fused_item(s_ticket, f.nblocks, f.lead).blk, 1u);
    }
    return;
  }
  if (tid >= F::RT) return;  // reaches no barrier that counts it
  auto sync = [] { asm volatile("bar.sync 3, %0;" ::"n"(F::RT) : "memory"); };
  auto sync_or = [](int p) {
    int r;
    asm volatile("{\n\t.reg .pred q, o;\n\tsetp.ne.s32 q, %1, 0;\n\tbar.red.or.pred o, 3, %2, q;\n\tselp.s32 %0, 1, 0, o;\n\t}"
                 : "=r"(r)
                 : "r"(p), "n"(F::RT)
                 : "memory");
    return r;
  };
  if (tid == 0)
    while (ld_acquire_gpu(f.ctr + 1 + it.blk) < (unsigned)F::NC) __nanosleep(64);
  sync();
  fwd_rows_v2_body<true, F::N1, true, true>(a2, t2, smem_raw, bars, tbar[0], tid, it.blk, it.idx * RowsV2Shape<true>::IPC,
                                            sync, sync_or, f.discard);
}

}  // namespace kfft
