// spectrum_kernels.cuh -- the wideband spectrum analyzer (wideband_poll, reference spectrum.c:308-522) around the forward
// transform pair.  One poll of fft_avg segments of fft_n samples runs, per chunk of segments:
//   spectrum_window_kernel   ring (float or int16, REAL or COMPLEX, modular) -> windowed segments the forward pass reads
//   kgpu_forward             r2c (REAL, even fft_n), c2c of length fft_n, or the first Bluestein pass of length P
//   bluestein_mul_kernel     Bluestein only: conj(A * B), B the stored transform of the conjugate chirp; second pass
//                            (bluestein_master.cuh)
//   spectrum_power_kernel    one thread per output bin: index mapping, bin += gain * |X|^2 over the chunk's segments
// The narrowband analyzer (narrowband_poll, spectrum.c:206-306) runs the same chain on a ring of a COMPLEX slave's
// delivered blocks (nb_ring_append_kernel), with narrowband_power_kernel's bin mapping in place of the last step.
// Bluestein: X_k = w_k sum_n (x_n w_n) conj(w_{k-n}) with w_n = exp(-i pi n^2 / fft_n), so with a = x w zero-padded to P,
// y = DFT_P(conj(DFT_P(a) B)) = P conj(conv(a, conj w)) and |X_k|^2 = |y_k|^2 / P^2 (|w_k| = 1: no post-chirp).
#pragma once
#include <cuda_runtime.h>

#include "bluestein_master.cuh"
#include "raw_ingest.cuh"

namespace kfft {

constexpr int kSpecThreads = 256;

struct SpecWindowArgs {
  void const *ring;  // float / int16 samples (REAL) or float / int16 pairs (COMPLEX)
  long cap;          // ring capacity in samples (>= fft_n)
  long start0;       // ring position of segment 0's first sample, in [0, cap)
  long step;         // signed distance between consecutive segments (REAL +hop, COMPLEX -hop)
  int seg0;          // global index of the chunk's first segment
  int fft_n;
  int out_len;       // elements per segment in `out` (fft_n, or P for Bluestein: zeros past fft_n)
  int complex_in, i16, derandomize;
  int flip;          // REAL with shift < 0: odd samples negated, odd fft_n's last sample zeroed (spectrum.c:385-390)
  int complex_out;   // float2 output (c2c and Bluestein); float for the r2c
  int chirp;         // multiply by w_n = exp(-i pi n^2 / fft_n)
  float scale;       // int16 samples: scale * (float)x (rx888.c:765) ...
  ScaleChange const *chg;  // ... or, with nchg > 0, each sample's own scale: `scale` before chg[0].at
  int nchg;
  long end;          // ring position just past the newest sample, which is absolute sample end_index - 1
  long long end_index;
  float const *window;
  void *out;         // [segment][out_len]
};

// rx888.c:707-712: lsb set -> flip bits 1..15 (what fwd_cols_body does, fwd_kernels.cuh:80-82)
__device__ __forceinline__ float spec_i16(short v, int derandomize, float scale) {
  if (derandomize) v ^= (short)((v & 1) ? 0xfffe : 0);
  return (float)v * scale;
}

__global__ void __launch_bounds__(kSpecThreads) spectrum_window_kernel(SpecWindowArgs a) {
  long const k = (long)blockIdx.x * kSpecThreads + threadIdx.x;
  if (k >= a.out_len) return;
  int const seg = blockIdx.y;
  float re = 0.f, im = 0.f;
  if (k < a.fft_n) {
    long base = (a.start0 + (long)(a.seg0 + seg) * a.step) % a.cap;
    if (base < 0) base += a.cap;
    long pos = base + k;
    if (pos >= a.cap) pos -= a.cap;
    float const w = a.window[k];
    float scale = a.scale;
    if (a.nchg) {
      long const back = a.end > pos ? a.end - pos : a.end - pos + a.cap;  // 1 for the newest sample
      scale = (float)scale_at(a.chg, a.nchg, (double)a.scale, a.end_index - back);
    }
    if (a.complex_in) {
      float xr, xi;
      if (a.i16) {
        short2 const v = reinterpret_cast<short2 const *>(a.ring)[pos];
        xr = spec_i16(v.x, a.derandomize, scale);
        xi = spec_i16(v.y, a.derandomize, scale);
      } else {
        float2 const v = reinterpret_cast<float2 const *>(a.ring)[pos];
        xr = v.x;
        xi = v.y;
      }
      re = __fmul_rn(w, xr);
      im = __fmul_rn(w, xi);
    } else {
      float const x = a.i16 ? spec_i16(reinterpret_cast<short const *>(a.ring)[pos], a.derandomize, scale)
                            : reinterpret_cast<float const *>(a.ring)[pos];
      re = __fmul_rn(w, x);
      if (a.flip) {
        if (k & 1) re = -re;
        if ((a.fft_n & 1) && k == a.fft_n - 1) re = 0.f;
      }
    }
    if (a.chirp) {
      float2 const w = bluestein_chirp(k, a.fft_n, 1.0);
      float const pr = re * w.x - im * w.y, pi = re * w.y + im * w.x;
      re = pr;
      im = pi;
    }
  }
  long const o = (long)seg * a.out_len + k;
  if (a.complex_out) reinterpret_cast<float2 *>(a.out)[o] = make_float2(re, im);
  else reinterpret_cast<float *>(a.out)[o] = re;
}

struct SpecPowerArgs {
  float2 const *spec;  // [segment][spec_stride]
  long spec_stride;
  int nseg;            // segments of this chunk, in the reference's order
  int first;           // first chunk of the poll: the bins start from 0
  int real_walk;       // REAL front end: the r2c walk of spectrum.c:396-406; else the KE5GDB mapping (:477-488)
  int fft_n, shift, bin_count;
  double norm;         // 1, or 1/P^2 after Bluestein
  double gain;         // 2/(fft_avg fft_n^2) REAL, 1/(fft_avg fft_n^2) COMPLEX
  float *bins;
};

// Source bin of output bin i, or -1 where the reference adds nothing (or, for a negative REAL walk index, reads outside
// its array: contributes 0 here).
__device__ __forceinline__ long spec_source(SpecPowerArgs const &a, int i) {
  int const half = a.bin_count / 2;
  if (a.real_walk) {
    long const b0 = a.shift >= 0 ? a.shift : a.fft_n / 2 + a.shift, top = a.fft_n / 2 + 1;
    // the walk checks binp < top before the step back at i == bin_count/2 and stops at the first failure
    if (i < half) return (b0 + i < top && b0 + i >= 0) ? b0 + i : -1;
    if (b0 + half >= top) return -1;
    long const b = b0 + i - a.bin_count;
    return b >= 0 ? b : -1;
  }
  long const off = i < half ? i : (long)i - a.bin_count;
  long const b = a.shift + off;
  if (b < -(long)(a.fft_n / 2) || b >= (long)((a.fft_n + 1) / 2)) return -1;
  return b >= 0 ? b : b + a.fft_n;
}

// bins[i] += gain * |X[src]|^2 over the chunk's segments in order, in double and stored as float after every segment;
// src = Source(a, i), -1 for a bin that gets nothing
template <long (*Source)(SpecPowerArgs const &, int)>
__device__ __forceinline__ void spec_accumulate(SpecPowerArgs const &a, int i) {
  float acc = a.first ? 0.f : a.bins[i];
  long const src = Source(a, i);
  if (src >= 0)
    for (int s = 0; s < a.nseg; s++) {
      float2 const v = a.spec[(long)s * a.spec_stride + src];
      double const p = __dmul_rn(__dadd_rn(__dmul_rn(v.x, v.x), __dmul_rn(v.y, v.y)), a.norm);
      if (isfinite(p)) acc = (float)__dadd_rn((double)acc, __dmul_rn(a.gain, p));
    }
  a.bins[i] = acc;
}

__global__ void __launch_bounds__(kSpecThreads) spectrum_power_kernel(SpecPowerArgs a) {
  int const i = blockIdx.x * kSpecThreads + threadIdx.x;
  if (i >= a.bin_count) return;
  spec_accumulate<spec_source>(a, i);
}

// ---- the narrowband analyzer (narrowband_poll, reference spectrum.c:206-306) ------------------------------------------
// Its segments are spectrum_window_kernel's COMPLEX float walk with a forward step; only the bin mapping differs.
// narrowband_poll's bin mapping (spectrum.c:267-271): bin i < bin_count/2 reads X[i], bin i >= bin_count/2 reads
// X[fft_n - 2 (bin_count/2) + i].  With an odd bin_count the last bin would read X[fft_n], past the transform: 0 here.
// shift and real_walk of the arguments are unused.
__device__ __forceinline__ long nb_source(SpecPowerArgs const &a, int i) {
  int const half = a.bin_count / 2;
  long const src = i < half ? (long)i : (long)a.fft_n - 2L * half + i;
  return src < a.fft_n ? src : -1;
}

__global__ void __launch_bounds__(kSpecThreads) narrowband_power_kernel(SpecPowerArgs a) {
  int const i = blockIdx.x * kSpecThreads + threadIdx.x;
  if (i >= a.bin_count) return;
  spec_accumulate<nb_source>(a, i);
}

// One delivered block of olen samples (src, or zeros when src is NULL: a lapped slave's block) into a ring of ring_size
// samples from position ring_idx on, wrapping (spectrum.c:147-151).  When the block is longer than the ring only its last
// ring_size samples survive the sample-by-sample loop, so only they are written.
__global__ void __launch_bounds__(kSpecThreads) nb_ring_append_kernel(float2 *ring, long ring_size, long ring_idx,
                                                                      float2 const *src, long olen) {
  long const first = olen > ring_size ? olen - ring_size : 0;
  long const i = first + (long)blockIdx.x * kSpecThreads + threadIdx.x;
  if (i >= olen) return;
  ring[(ring_idx + i) % ring_size] = src ? src[i] : make_float2(0.f, 0.f);
}

}  // namespace kfft
