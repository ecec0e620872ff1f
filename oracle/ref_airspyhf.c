/* oracle/ref_airspyhf.c -- drives the reference's OWN AirspyHF+ sample callback (rx_callback, airspyhf.c:292-325) for the
 * float ingest checks (tests/test_float_ingest_cpu.py, tools/float_ingest_bench.py).
 *
 * TEST INFRASTRUCTURE, NOT PRODUCT.  The reference's src/airspyhf.c is #included unmodified from where it lies (never
 * copied), so its static rx_callback is reachable on a prepared sdrstate and frontend whose master is the reference's
 * own filter.c.  libairspyhf is a declaration-only header (stubs/libairspyhf/airspyhf.h); the callback's thread naming,
 * priority and core pinning are no-ops here.  Compiled only into oracle/_ref/libka9qfloat.so (oracle/float.mk).
 */
#define _GNU_SOURCE 1
#include <limits.h>
#include <time.h>
#include "misc.h"
#undef pthread_setname
#define pthread_setname(x) ((void)(x)) /* rx_callback names its thread once: not the oracle's to do */

#include "airspyhf.c"

static struct frontend Rh_frontend;
static struct sdrstate Rh_sdr;

/* a COMPLEX master of L, M on the reference's filter.c and the sdrstate airspyhf_startup leaves, with the given scale */
int rh_open(int L, int M, double scale) {
  memset(&Rh_frontend, 0, sizeof Rh_frontend);
  memset(&Rh_sdr, 0, sizeof Rh_sdr);
  N_worker_threads = 0; /* blocks run inline on the calling thread (filter.c:44) */
  Rh_frontend.isreal = false;
  if (create_filter_input(&Rh_frontend.in, L, M, COMPLEX) != 0)
    return -1;
  Rh_frontend.context = &Rh_sdr;
  Rh_sdr.frontend = &Rh_frontend;
  Rh_sdr.scale = scale;
  return 0;
}
void rh_set_scale(double scale) { Rh_sdr.scale = scale; }

/* One transfer of `count` I/Q pairs through rx_callback, with if_power 0 before it.  floats: the 2 * count floats it
 * stored; *if_power as it left it (Power_alpha * energy / count, or 0 where its isfinite guard skipped the update);
 * *alpha: Power_alpha. */
int rh_transfer(float const *iq, int count, float *floats, double *if_power, double *alpha) {
  airspyhf_complex_float_t *copy = malloc(count > 0 ? sizeof *copy * (size_t)count : sizeof *copy);
  memcpy(copy, iq, sizeof *copy * (size_t)count);
  float const *wptr = (float const *)Rh_frontend.in.input_write_pointer.c;
  Rh_frontend.if_power = 0;
  airspyhf_transfer_t t = {.ctx = &Rh_sdr, .samples = copy, .sample_count = count};
  int const r = rx_callback(&t);
  free(copy);
  memcpy(floats, wptr, sizeof(float) * 2 * (size_t)count); /* the mirrored ring keeps them contiguous */
  *if_power = Rh_frontend.if_power;
  *alpha = Power_alpha;
  return r;
}

/* host wall time of n calls of rx_callback on the same transfer, in seconds, with the master's
 * write refused so that only the conversion loop runs (tools/float_ingest_bench.py).  The write pointer advances by
 * the transfer after each call and wraps as write_*filter would move it, so the loop stores into the whole ring as it
 * does in a running radiod rather than into one cache-hot spot. */
double rh_time(float const *iq, int count, int n) {
  airspyhf_complex_float_t *copy = malloc(sizeof *copy * (size_t)count);
  memcpy(copy, iq, sizeof *copy * (size_t)count);
  airspyhf_transfer_t t = {.ctx = &Rh_sdr, .samples = copy, .sample_count = count};
  struct timespec a, b;
  int const wcnt = Rh_frontend.in.wcnt;
  Rh_frontend.in.wcnt = INT_MAX / 16; /* the closing write_cfilter is refused at once: no block fires, no FFT runs */
  clock_gettime(CLOCK_MONOTONIC, &a);
  struct rc const wp = Rh_frontend.in.input_write_pointer;
  for (int i = 0; i < n; i++) {
    rx_callback(&t);
    Rh_frontend.in.input_write_pointer.c += count; /* mirrored ring: a transfer across the end stays contiguous */
    if ((char *)Rh_frontend.in.input_write_pointer.c >= (char *)Rh_frontend.in.input_buffer + Rh_frontend.in.input_buffer_size)
      Rh_frontend.in.input_write_pointer.c -= Rh_frontend.in.input_buffer_size / sizeof(float complex);
  }
  clock_gettime(CLOCK_MONOTONIC, &b);
  Rh_frontend.in.input_write_pointer = wp;
  Rh_frontend.in.wcnt = wcnt;
  free(copy);
  return (double)(b.tv_sec - a.tv_sec) + 1e-9 * (double)(b.tv_nsec - a.tv_nsec);
}

void rh_close(void) { delete_filter_input(&Rh_frontend.in); }
