/* oracle/ref_hydrasdr_float.c -- drives the reference's OWN HydraSDR sample callback (rx_callback, hydrasdr.c:641-867) in
 * its float formats for the float ingest checks (tests/test_float_ingest_cpu.py, tools/float_ingest_bench.py).
 *
 * TEST INFRASTRUCTURE, NOT PRODUCT.  The reference's src/hydrasdr.c is #included unmodified from where it lies (never
 * copied), as oracle/ref_hydrasdr.c does for the 16-bit formats, into a library of its own (oracle/_ref/libka9qfloat.so,
 * oracle/float.mk).  The software AGC is off; the callback's thread naming is a no-op here.
 */
#define _GNU_SOURCE 1
#include <limits.h>
#include <time.h>
#include "misc.h"
#undef pthread_setname
#define pthread_setname(x) ((void)(x)) /* rx_callback names its thread once: not the oracle's to do */

#include "hydrasdr.c"

static struct frontend Ryf_frontend;
static struct sdrstate Ryf_sdr;

/* iq 0: FLOAT32_REAL on a REAL master, 1: FLOAT32_IQ on a COMPLEX one, of L, M on the reference's filter.c, software AGC
 * off, the given scale */
int ryf_open(int iq, int L, int M, double scale) {
  memset(&Ryf_frontend, 0, sizeof Ryf_frontend);
  memset(&Ryf_sdr, 0, sizeof Ryf_sdr);
  N_worker_threads = 0; /* blocks run inline on the calling thread (filter.c:44) */
  Ryf_frontend.isreal = !iq;
  if (create_filter_input(&Ryf_frontend.in, L, M, iq ? COMPLEX : REAL) != 0)
    return -1;
  Ryf_frontend.bitspersample = 1;
  Ryf_frontend.context = &Ryf_sdr;
  Ryf_sdr.frontend = &Ryf_frontend;
  Ryf_sdr.sample_type = iq ? HYDRASDR_SAMPLE_FLOAT32_IQ : HYDRASDR_SAMPLE_FLOAT32_REAL;
  Ryf_sdr.software_agc = false;
  Ryf_sdr.scale = scale;
  return 0;
}
void ryf_set_scale(double scale) { Ryf_sdr.scale = scale; }

/* One transfer of `count` samples (REAL) or I/Q pairs through rx_callback, with if_power 0 before it.  floats: the
 * floats it stored; *if_power as it left it (Power_alpha * energy / count, or 0 where its isfinite guard skipped the
 * update); *alpha: Power_alpha. */
int ryf_transfer(float const *x, int count, float *floats, double *if_power, double *alpha) {
  size_t const comps = (size_t)count * (Ryf_frontend.isreal ? 1 : 2);
  float *copy = malloc(comps ? sizeof(float) * comps : sizeof(float));
  memcpy(copy, x, sizeof(float) * comps);
  float const *wptr = Ryf_frontend.isreal ? Ryf_frontend.in.input_write_pointer.r : (float const *)Ryf_frontend.in.input_write_pointer.c;
  Ryf_frontend.if_power = 0;
  hydrasdr_transfer t = {.ctx = &Ryf_sdr, .samples = copy, .sample_count = count, .sample_type = Ryf_sdr.sample_type};
  int const r = rx_callback(&t);
  free(copy);
  memcpy(floats, wptr, sizeof(float) * comps); /* the mirrored ring keeps them contiguous */
  *if_power = Ryf_frontend.if_power;
  *alpha = Power_alpha;
  return r;
}

/* host wall time of n calls of rx_callback on the same transfer, in seconds, with the master's
 * write refused so that only the conversion loop runs (tools/float_ingest_bench.py).  The write pointer advances by
 * the transfer after each call and wraps as write_*filter would move it, so the loop stores into the whole ring as it
 * does in a running radiod rather than into one cache-hot spot. */
double ryf_time(float const *x, int count, int n) {
  size_t const comps = (size_t)count * (Ryf_frontend.isreal ? 1 : 2);
  float *copy = malloc(sizeof(float) * comps);
  memcpy(copy, x, sizeof(float) * comps);
  hydrasdr_transfer t = {.ctx = &Ryf_sdr, .samples = copy, .sample_count = count, .sample_type = Ryf_sdr.sample_type};
  struct timespec a, b;
  int const wcnt = Ryf_frontend.in.wcnt;
  Ryf_frontend.in.wcnt = INT_MAX / 16; /* the closing write_*filter is refused at once: no block fires, no FFT runs */
  clock_gettime(CLOCK_MONOTONIC, &a);
  struct rc const wp = Ryf_frontend.in.input_write_pointer;
  size_t const step = sizeof(float) * comps;
  for (int i = 0; i < n; i++) {
    rx_callback(&t);
    char *p = (Ryf_frontend.isreal ? (char *)Ryf_frontend.in.input_write_pointer.r : (char *)Ryf_frontend.in.input_write_pointer.c) + step;
    if (p >= (char *)Ryf_frontend.in.input_buffer + Ryf_frontend.in.input_buffer_size)
      p -= Ryf_frontend.in.input_buffer_size;
    if (Ryf_frontend.isreal) /* only the master type's pointer is set (filter.c:186-269) */
      Ryf_frontend.in.input_write_pointer.r = (float *)p;
    else
      Ryf_frontend.in.input_write_pointer.c = (float complex *)p;
  }
  clock_gettime(CLOCK_MONOTONIC, &b);
  Ryf_frontend.in.input_write_pointer = wp;
  Ryf_frontend.in.wcnt = wcnt;
  free(copy);
  return (double)(b.tv_sec - a.tv_sec) + 1e-9 * (double)(b.tv_nsec - a.tv_nsec);
}

void ryf_close(void) { delete_filter_input(&Ryf_frontend.in); }
