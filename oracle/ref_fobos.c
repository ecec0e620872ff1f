/* oracle/ref_fobos.c -- drives the reference's OWN Fobos sample callback (rx_callback, fobos.c:395-426) for the float
 * ingest checks (tests/test_float_ingest_cpu.py, tools/float_ingest_bench.py).
 *
 * TEST INFRASTRUCTURE, NOT PRODUCT.  The reference's src/fobos.c is #included unmodified from where it lies (never
 * copied), so its static rx_callback is reachable on a prepared sdrstate and frontend whose master is the reference's
 * own filter.c.  libfobos is a declaration-only header (stubs/fobos.h); the callback's thread naming is a no-op here.
 * Compiled only into oracle/_ref/libka9qfloat.so (oracle/float.mk).
 */
#define _GNU_SOURCE 1
#include <limits.h>
#include <time.h>
#include "misc.h"
#undef pthread_setname
#define pthread_setname(x) ((void)(x)) /* rx_callback names its thread once: not the oracle's to do */

#include "fobos.c"

static struct frontend Rf_frontend;
static struct sdrstate Rf_sdr;

/* a COMPLEX master of L, M on the reference's filter.c and the sdrstate fobos_startup leaves, with the given scale;
 * samprate sets Power_alpha at the first transfer (fobos.c:405-409), which keeps it from then on */
int rf_open(int L, int M, double scale, double samprate) {
  memset(&Rf_frontend, 0, sizeof Rf_frontend);
  memset(&Rf_sdr, 0, sizeof Rf_sdr);
  N_worker_threads = 0; /* blocks run inline on the calling thread (filter.c:44) */
  Rf_frontend.isreal = false;
  if (create_filter_input(&Rf_frontend.in, L, M, COMPLEX) != 0)
    return -1;
  Rf_frontend.samprate = samprate;
  Rf_frontend.context = &Rf_sdr;
  Rf_sdr.frontend = &Rf_frontend;
  Rf_sdr.scale = scale;
  Power_alpha = 0;
  return 0;
}
void rf_set_scale(double scale) { Rf_sdr.scale = scale; }

/* One transfer of `count` I/Q pairs (count > 0) through rx_callback, with if_power 0 before it.  floats: the 2 * count
 * floats it stored; *if_power as it left it (Power_alpha * energy / count, or 0 where its isfinite guard skipped the
 * update); *alpha: Power_alpha. */
int rf_transfer(float const *iq, int count, float *floats, double *if_power, double *alpha) {
  float *copy = malloc(sizeof(float) * 2 * (size_t)count);
  memcpy(copy, iq, sizeof(float) * 2 * (size_t)count);
  float const *wptr = (float const *)Rf_frontend.in.input_write_pointer.c;
  Rf_frontend.if_power = 0;
  rx_callback(copy, (unsigned)count, &Rf_sdr);
  free(copy);
  memcpy(floats, wptr, sizeof(float) * 2 * (size_t)count); /* the mirrored ring keeps them contiguous */
  *if_power = Rf_frontend.if_power;
  *alpha = Power_alpha;
  return 0;
}

/* host wall time of n calls of rx_callback on the same transfer, in seconds, with the master's
 * write refused so that only the conversion loop runs (tools/float_ingest_bench.py).  The write pointer advances by
 * the transfer after each call and wraps as write_*filter would move it, so the loop stores into the whole ring as it
 * does in a running radiod rather than into one cache-hot spot. */
double rf_time(float const *iq, int count, int n) {
  float *copy = malloc(sizeof(float) * 2 * (size_t)count);
  memcpy(copy, iq, sizeof(float) * 2 * (size_t)count);
  struct timespec a, b;
  int const wcnt = Rf_frontend.in.wcnt;
  Rf_frontend.in.wcnt = INT_MAX / 16; /* the closing write_cfilter is refused at once: no block fires, no FFT runs */
  clock_gettime(CLOCK_MONOTONIC, &a);
  struct rc const wp = Rf_frontend.in.input_write_pointer;
  for (int i = 0; i < n; i++) {
    rx_callback(copy, (unsigned)count, &Rf_sdr);
    Rf_frontend.in.input_write_pointer.c += count; /* mirrored ring: a transfer across the end stays contiguous */
    if ((char *)Rf_frontend.in.input_write_pointer.c >= (char *)Rf_frontend.in.input_buffer + Rf_frontend.in.input_buffer_size)
      Rf_frontend.in.input_write_pointer.c -= Rf_frontend.in.input_buffer_size / sizeof(float complex);
  }
  clock_gettime(CLOCK_MONOTONIC, &b);
  Rf_frontend.in.input_write_pointer = wp;
  Rf_frontend.in.wcnt = wcnt;
  free(copy);
  return (double)(b.tv_sec - a.tv_sec) + 1e-9 * (double)(b.tv_nsec - a.tv_nsec);
}

void rf_close(void) { delete_filter_input(&Rf_frontend.in); }
