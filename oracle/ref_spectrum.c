/* oracle/ref_spectrum.c -- drives the reference's OWN wideband_poll (spectrum.c:308-522) for the oracle.
 *
 * TEST INFRASTRUCTURE, NOT PRODUCT.  The reference's src/spectrum.c is #included unmodified from where it lies (never
 * copied), so its static wideband_poll is reachable here on a prepared chan_t and frontend.  It plans through the
 * reference's filter.c (plan_r2c / plan_complex) onto fftw_shim.c, the same oracle/fft_cpu.c transform the restatement
 * uses.  Compiled only into oracle/_ref/libka9qspectrum.so (oracle/spectrum.mk).
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

float *fftwf_alloc_real(size_t n) { return malloc(sizeof(float) * (n ? n : 1)); }
fftwf_complex *fftwf_alloc_complex(size_t n) { return malloc(sizeof(fftwf_complex) * (n ? n : 1)); }
void fftwf_free(void *p) { free(p); }

/* One wideband_poll on a ring of cap samples (float, or float complex when !is_real) whose newest sample ends at
 * position `end`.  The ring is laid out twice in a row, as the reference's mirrored input buffer shows it.  The shift is
 * passed through bin_shift with master->points = fft_n (spectrum.c:347).  Returns the fft_avg the poll used (its
 * avg_limit clamp, :359 / :417). */
int rs_wideband_poll(int is_real, int fft_n, int bin_count, float const *window, int shift, int fft_avg, double overlap,
                     void const *ring, long cap, long end, float *bin_data) {
  static struct frontend fe;
  static chan_t chan;
  memset(&fe, 0, sizeof fe);
  memset(&chan, 0, sizeof chan);
  size_t const esz = is_real ? sizeof(float) : sizeof(float complex);
  char *buf = malloc(2 * (size_t)cap * esz);
  memcpy(buf, ring, (size_t)cap * esz);
  memcpy(buf + (size_t)cap * esz, ring, (size_t)cap * esz);
  long const e = ((end % cap) + cap) % cap;
  fe.isreal = is_real;
  fe.in.input_buffer = buf;
  fe.in.input_buffer_size = (size_t)cap * esz;
  fe.in.points = fft_n;
  if (is_real)
    fe.in.input_write_pointer.r = (float *)buf + e;
  else
    fe.in.input_write_pointer.c = (float complex *)buf + e;
  chan.frontend = &fe;
  chan.filter.out.master = &fe.in;
  chan.filter.bin_shift = shift;
  chan.spectrum.fft_n = fft_n;
  chan.spectrum.bin_count = bin_count;
  chan.spectrum.bin_data = bin_data;
  chan.spectrum.fft_avg = fft_avg;
  chan.spectrum.overlap = overlap;
  chan.spectrum.window = malloc(sizeof(float) * ((size_t)fft_n + 1));
  memcpy(chan.spectrum.window, window, sizeof(float) * (size_t)fft_n);
  wideband_poll(&chan);
  destroy_plan(&chan.spectrum.plan);
  free(chan.spectrum.window);
  free(buf);
  return chan.spectrum.fft_avg;
}
