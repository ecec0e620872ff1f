/* oracle/ref_bladerf.c -- drives the reference's OWN bladeRF sample loop (bladerf_process, bladerf.c:215-246) for the
 * raw 16-bit ingest checks (tests/test_raw16_ingest_cpu.py, tools/raw16_ingest_bench.py).
 *
 * TEST INFRASTRUCTURE, NOT PRODUCT.  The reference's src/bladerf.c is #included unmodified from where it lies (never
 * copied), so its static bladerf_process is reachable on a prepared frontend whose master is the reference's own
 * filter.c.  libbladeRF is a declaration-only header (stubs/libbladeRF.h).  Compiled only into oracle/_ref/libka9qraw16.so
 * (oracle/raw16.mk).
 */
#define _GNU_SOURCE 1
#include <limits.h>
#include "misc.h"
#undef pthread_setname
#define pthread_setname(x) ((void)(x))

#include "bladerf.c"

static struct frontend Rb_frontend;

/* a COMPLEX master of L, M on the reference's filter.c, as bladerf_setup leaves the frontend (bladerf.c:124-125) */
int rb_open(int L, int M) {
  memset(&Rb_frontend, 0, sizeof Rb_frontend);
  N_worker_threads = 0; /* blocks run inline on the calling thread (filter.c:44) */
  if (create_filter_input(&Rb_frontend.in, L, M, COMPLEX) != 0)
    return -1;
  Rb_frontend.isreal = false;
  Rb_frontend.bitspersample = 12;
  return 0;
}

/* One buffer of `count` SC16_Q11 I/Q pairs through bladerf_process.  floats: the 2 * count floats it stored;
 * *overranges and *if_power as it left them. */
void rb_transfer(int16_t const *words, int count, float *floats, uint64_t *overranges, double *if_power) {
  int16_t *copy = malloc(count > 0 ? sizeof(int16_t) * 2 * (size_t)count : 2);
  memcpy(copy, words, sizeof(int16_t) * 2 * (size_t)count);
  float const *wptr = (float const *)Rb_frontend.in.input_write_pointer.c;
  bladerf_process(&Rb_frontend, copy, (size_t)count);
  free(copy);
  memcpy(floats, wptr, sizeof(float) * 2 * (size_t)count); /* the mirrored ring keeps them contiguous */
  *overranges = Rb_frontend.overranges;
  *if_power = Rb_frontend.if_power;
}

/* host wall time of n calls of bladerf_process on the same buffer, in seconds, with the master's
 * write refused so that only the conversion loop runs (tools/raw16_ingest_bench.py) */
double rb_time(int16_t const *words, int count, int n) {
  int16_t *copy = malloc(sizeof(int16_t) * 2 * (size_t)count);
  memcpy(copy, words, sizeof(int16_t) * 2 * (size_t)count);
  struct timespec a, b;
  int const wcnt = Rb_frontend.in.wcnt;
  Rb_frontend.in.wcnt = INT_MAX / 16; /* the closing write_*filter is refused at once: no block fires, no FFT runs */
  clock_gettime(CLOCK_MONOTONIC, &a);
  for (int i = 0; i < n; i++)
    bladerf_process(&Rb_frontend, copy, (size_t)count);
  clock_gettime(CLOCK_MONOTONIC, &b);
  Rb_frontend.in.wcnt = wcnt;
  free(copy);
  return (double)(b.tv_sec - a.tv_sec) + 1e-9 * (double)(b.tv_nsec - a.tv_nsec);
}

void rb_close(void) { delete_filter_input(&Rb_frontend.in); }
