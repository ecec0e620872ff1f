// plan.cuh -- host-side planning for the shared-memory column transforms and the two-pass
// forward transform.  All tables are computed in double precision on the host and rounded once
// (the reference gets its twiddles from FFTW's planner, filter.c:101-163; there is no wisdom here,
// a plan is a pure function of the length).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <vector>
#include "fft_tile.cuh"

namespace kfft {

constexpr int kMaxTileLen = 4096;

// Factor n into supported in-register radices: fewest stages, then smallest radix sum; even
// radices first (large strides are bank-conflict free), odd ones last.  Empty result = unsupported.
std::vector<int> choose_radices(int n);
// The same search over the extended set (today's radices plus the primes 11, 13, 17, 19, 23) that masters created with
// kgpu_master_create_ex use.  On a length with factors 2, 3, 5, 7 only it returns exactly choose_radices(n).
std::vector<int> choose_radices_ext(int n);

// Returns the registry index of the column plan for `len` (creating and uploading it on first
// use), or -1 if len cannot be planned.  Thread-safe.
int get_tile_plan(int len);
TilePlan const *host_tile_plan(int idx);  // host copy (device pointers inside)

// Pitch (in float2) of a column of `len` points inside shared memory: len rounded up so that
// pitch % 16 == 2, which keeps both the transposing loads (T columns x consecutive rows) and the
// per-column butterflies free of 64-bit bank conflicts.
inline int column_pitch(int len) {
  int p = len;
  while (p % 16 != 2) p++;
  return p;
}

// Split of a long transform into columns (len n1, stride n2) and rows (len n2).
struct Split2 {
  int n1, n2;
};
bool choose_split(long n, Split2 *out);
// choose_split with choose_radices_ext deciding what is plannable (equal to choose_split where n has factors 2, 3, 5, 7).
// Its plans never enter the registry: an extended master builds and owns them.
bool choose_split_ext(long n, Split2 *out);

}  // namespace kfft
