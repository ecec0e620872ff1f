/* oracle/ref_narrowband.c -- drives the reference's OWN narrowband_poll (spectrum.c:206-306) for the oracle.
 *
 * TEST INFRASTRUCTURE, NOT PRODUCT.  The reference's src/spectrum.c is #included unmodified from where it lies (never
 * copied), as oracle/ref_spectrum.c does for wideband_poll, so its static narrowband_poll is reachable here on a prepared
 * chan_t.  It plans through the reference's filter.c (plan_complex) onto fftw_shim.c, the same oracle/fft_cpu.c transform
 * the restatement (oracle/narrowband_oracle.c) uses.  Compiled only into oracle/_ref/libka9qnarrowband.so
 * (oracle/narrowband.mk).
 *
 * The allocators hand out one zeroed element past the requested length: with an odd bin_count narrowband_poll's last bin
 * reads fft_out[fft_n], one past its transform, and this makes that read defined and 0 (what the library gives that bin).
 */
#define _GNU_SOURCE 1
#include <stddef.h>
#include <stdlib.h>
#include <string.h>
#include <fftw3.h> /* the declaration-only stub: it lacks the three allocators spectrum.c calls */
float *fftwf_alloc_real(size_t n);
fftwf_complex *fftwf_alloc_complex(size_t n);
void fftwf_free(void *p);

#include "spectrum.c"

float *fftwf_alloc_real(size_t n) { return calloc(n + 1, sizeof(float)); }
fftwf_complex *fftwf_alloc_complex(size_t n) { return calloc(n + 1, sizeof(fftwf_complex)); }
void fftwf_free(void *p) { free(p); }

/* One narrowband_poll of a ring of ring_size float complex samples whose next write position is ring_idx.  bin_data
 * receives bin_count floats.  Returns the fft_avg its clamp used (spectrum.c:244-246), the same expression re-evaluated
 * here since the reference keeps it in a local. */
int rs_narrowband_poll(int fft_n, int bin_count, float const *window, int fft_avg, double overlap, void const *ring,
                       int ring_size, int ring_idx, float *bin_data) {
  static struct frontend fe;
  static chan_t chan;
  memset(&fe, 0, sizeof fe);
  memset(&chan, 0, sizeof chan);
  chan.frontend = &fe;
  chan.spectrum.fft_n = fft_n;
  chan.spectrum.bin_count = bin_count;
  chan.spectrum.bin_data = bin_data;
  chan.spectrum.fft_avg = fft_avg;
  chan.spectrum.overlap = overlap;
  chan.spectrum.ring = malloc(sizeof(float complex) * (size_t)ring_size);
  memcpy(chan.spectrum.ring, ring, sizeof(float complex) * (size_t)ring_size);
  chan.spectrum.ring_size = ring_size;
  chan.spectrum.ring_idx = ring_idx;
  chan.spectrum.window = malloc(sizeof(float) * ((size_t)fft_n + 1));
  memcpy(chan.spectrum.window, window, sizeof(float) * (size_t)fft_n);
  narrowband_poll(&chan);
  destroy_plan(&chan.spectrum.plan);
  free(chan.spectrum.window);
  free(chan.spectrum.ring);
  double const avg_limit = floor(1 + ((ring_size / fft_n) - 1) / (1 - overlap));
  return fft_avg > avg_limit ? (int)lrint(avg_limit) : fft_avg;
}
