/* oracle/spectrum_oracle.c -- restatement of the wideband spectrum analyzer's poll (wideband_poll, reference
 * spectrum.c:308-522) on a ring of float samples.  TEST INFRASTRUCTURE, NOT PRODUCT.
 *
 * It transforms with oracle/fft_cpu.c, the same transform the FFTW shim (fftw_shim.c) gives the reference, so with the
 * same flags it computes what the reference computes; the one deviation is the one the library makes: a REAL walk
 * index below 0 (an out-of-bounds read in the reference, e.g. 0 <= shift < bin_count/2) contributes 0.
 */
#include <complex.h>
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "fft_cpu.h"

/* cnrm (misc.h:282-284): the float bin promoted to double complex */
static inline double cnrm_d(float complex x) {
  double const re = crealf(x), im = cimagf(x);
  return re * re + im * im;
}

/* ring: cap floats (REAL) or cap float complex (COMPLEX); `end` the position just past the newest sample.  Writes
 * bin_data[0 .. bin_count).  Returns 0, or -1 on bad arguments. */
int ko_wideband_spectrum(int is_real, int fft_n, int bin_count, float const *window, int shift, int fft_avg,
                         double overlap, void const *ring, long cap, long end, float *bin_data) {
  if (fft_n < 2 || bin_count < 1 || fft_avg < 1 || cap < fft_n)
    return -1;
  memset(bin_data, 0, (size_t)bin_count * sizeof *bin_data);
  int const adjust = lrint(fft_n * (1 + (fft_avg - 1) * (1 - overlap))); /* spectrum.c:364, :422 */
  long const hop = lrint(fft_n * (1. - overlap));                          /* spectrum.c:407, :491 */
  long pos = ((end - adjust) % cap + cap) % cap;
  kfft_plan *half = NULL, *full = NULL;
  if (is_real) {
    float *fft_in = malloc(sizeof(float) * (size_t)fft_n);
    float complex *fft_out = malloc(sizeof(float complex) * (size_t)(fft_n / 2 + 1));
    float complex *tmp = NULL;
    if (fft_n % 2 == 0)
      half = kfft_plan_create(fft_n / 2);
    else {
      full = kfft_plan_create(fft_n);
      tmp = malloc(sizeof(float complex) * (size_t)fft_n);
    }
    float const *in = ring;
    double const gain = 2. / (double)((int64_t)fft_avg * fft_n * fft_n);
    for (int iter = 0; iter < fft_avg; iter++) {
      for (int i = 0; i < fft_n; i++) {
        long p = pos + i;
        if (p >= cap)
          p -= cap;
        fft_in[i] = window[i] * in[p];
      }
      if (shift < 0) { /* spectrum.c:385-390 */
        for (int i = 1; i < fft_n; i += 2)
          fft_in[i] = -fft_in[i];
        if (fft_n & 1)
          fft_in[fft_n - 1] = 0;
      }
      if (half)
        kfft_r2c_f(half, fft_in, fft_out);
      else { /* the shim's odd r2c (fftw_shim.c) */
        for (int i = 0; i < fft_n; i++)
          tmp[i] = fft_in[i];
        kfft_exec_f(full, tmp, tmp, -1);
        for (int i = 0; i <= fft_n / 2; i++)
          fft_out[i] = tmp[i];
      }
      int binp = shift >= 0 ? shift : fft_n / 2 + shift; /* spectrum.c:396-406 */
      for (int i = 0; i < bin_count && binp < fft_n / 2 + 1; i++, binp++) {
        if (i == bin_count / 2)
          binp -= bin_count;
        if (binp < 0)
          continue; /* the reference reads fft_out[binp < 0] here */
        double const p = cnrm_d(fft_out[binp]);
        if (isfinite(p))
          bin_data[i] += gain * p;
      }
      pos += hop;
      if (pos >= cap)
        pos -= cap;
    }
    free(fft_in);
    free(fft_out);
    free(tmp);
  } else {
    float complex const *in = ring;
    float complex *fft_in = malloc(sizeof(float complex) * (size_t)fft_n);
    float complex *fft_out = malloc(sizeof(float complex) * (size_t)fft_n);
    full = kfft_plan_create(fft_n);
    double const gain = 1. / (double)((int64_t)fft_avg * fft_n * fft_n);
    for (int iter = 0; iter < fft_avg; iter++) {
      for (int i = 0; i < fft_n; i++) {
        long p = pos + i;
        if (p >= cap)
          p -= cap;
        fft_in[i] = window[i] * in[p];
      }
      kfft_exec_f(full, fft_in, fft_out, -1);
      for (int i = 0; i < bin_count; i++) { /* spectrum.c:477-488 */
        int const offset = i < bin_count / 2 ? i : i - bin_count;
        int const b = shift + offset;
        if (b < -fft_n / 2 || b >= (fft_n + 1) / 2)
          continue;
        int const binp = b >= 0 ? b : b + fft_n;
        double const p = cnrm_d(fft_out[binp]);
        if (isfinite(p))
          bin_data[i] += gain * p;
      }
      pos -= hop;
      if (pos < 0)
        pos += cap;
    }
    free(fft_in);
    free(fft_out);
  }
  kfft_plan_destroy(half);
  kfft_plan_destroy(full);
  return 0;
}
