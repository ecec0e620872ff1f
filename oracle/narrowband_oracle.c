/* oracle/narrowband_oracle.c -- restatement of the narrowband spectrum analyzer (reference spectrum.c:123-155 and
 * narrowband_poll, :206-306) on a ring of float complex samples.  TEST INFRASTRUCTURE, NOT PRODUCT.
 *
 * It transforms with oracle/fft_cpu.c, the same transform the FFTW shim (fftw_shim.c) gives the reference, so with the
 * same flags it computes what the reference computes.  The one deviation is the library's: with an odd bin_count the last
 * bin, which the reference reads from fft_out[fft_n] (one past its transform), is 0.
 */
#include <complex.h>
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include "fft_cpu.h"

/* cnrm (misc.h:282-284): the float bin promoted to double complex */
static inline double cnrm_d(float complex x) {
  double const re = crealf(x), im = cimagf(x);
  return re * re + im * im;
}

/* One poll of the ring (ring_size samples, next write position ring_idx): writes bin_data[0 .. bin_count) and returns
 * the fft_avg the clamp left, or -1 on bad arguments. */
int ko_narrowband_spectrum(int fft_n, int bin_count, float const *window, int fft_avg, double overlap,
                           float complex const *ring, int ring_size, int ring_idx, float *bin_data) {
  if (fft_n < 1 || bin_count < 1 || bin_count > fft_n || fft_avg < 1 || ring_size < fft_n || ring_idx < 0 ||
      ring_idx >= ring_size || !(overlap >= 0 && overlap < 1))
    return -1;
  memset(bin_data, 0, (size_t)bin_count * sizeof *bin_data);
  double const avg_limit = floor(1 + ((ring_size / fft_n) - 1) / (1 - overlap)); /* spectrum.c:244-246 */
  int const avg = fft_avg > avg_limit ? lrint(avg_limit) : fft_avg;
  int rp = ring_idx - lrint(fft_n * (1 + (avg - 1) * (1 - overlap))); /* spectrum.c:247-249 */
  if (rp < 0)
    rp += ring_size;
  int const back = lrint(fft_n * overlap); /* spectrum.c:278 */
  double const gain = 1.0 / ((double)fft_n * fft_n * avg);
  float complex *fft_in = malloc(sizeof(float complex) * (size_t)fft_n);
  float complex *fft_out = malloc(sizeof(float complex) * (size_t)fft_n);
  kfft_plan *plan = kfft_plan_create(fft_n);
  int const half = bin_count / 2;
  for (int iter = 0; iter < avg; iter++) {
    for (int i = 0; i < fft_n; i++) {
      fft_in[i] = ring[rp++] * window[i];
      if (rp >= ring_size)
        rp -= ring_size;
    }
    kfft_exec_f(plan, fft_in, fft_out, -1);
    for (int i = 0; i < bin_count; i++) { /* spectrum.c:267-276 */
      int const fr = i < half ? i : fft_n - 2 * half + i;
      if (fr >= fft_n)
        continue; /* odd bin_count: the reference reads fft_out[fft_n] here */
      double const p = cnrm_d(fft_out[fr]);
      if (isfinite(p))
        bin_data[i] += gain * p;
    }
    rp -= back;
    if (rp < 0)
      rp += ring_size;
  }
  kfft_plan_destroy(plan);
  free(fft_in);
  free(fft_out);
  return avg;
}

/* One pass of demod_spectrum's narrowband ring upkeep (spectrum.c:124-151) for a block of n samples: create or grow the
 * ring to fft_avg * fft_n samples (new space zeroed, the index reset only when the ring is created), then append the
 * block sample by sample with wrap.  ring has room for cap samples; *ring_size is 0 for "no ring yet".  Returns 0, or -1
 * when cap is too small. */
int ko_nb_ring_step(float complex *ring, long cap, int *ring_size, int *ring_idx, int fft_avg, int fft_n,
                    float complex const *block, int n) {
  if (*ring_size == 0 || *ring_size < fft_avg * fft_n) {
    if (*ring_size == 0)
      *ring_idx = 0;
    int const old = *ring_size;
    int const size = fft_avg * fft_n;
    if (size > cap || size < old)
      return -1;
    memset(ring + old, 0, sizeof *ring * (size_t)(size - old));
    *ring_size = size;
  }
  for (int i = 0; i < n; i++) {
    ring[(*ring_idx)++] = block ? block[i] : 0;
    if (*ring_idx == *ring_size)
      *ring_idx = 0;
  }
  return 0;
}
