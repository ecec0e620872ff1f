/* oracle/ref_hydrasdr.c -- drives the reference's OWN HydraSDR sample callback (rx_callback, hydrasdr.c:641-867) in its
 * 16-bit formats for the raw 16-bit ingest checks (tests/test_raw16_ingest_cpu.py, tools/raw16_ingest_bench.py).
 *
 * TEST INFRASTRUCTURE, NOT PRODUCT.  The reference's src/hydrasdr.c is #included unmodified from where it lies (never
 * copied), so its static rx_callback is reachable on a prepared sdrstate and frontend whose master is the reference's
 * own filter.c.  libhydrasdr is a declaration-only header (stubs/libhydrasdr/hydrasdr.h).  The software AGC is off (it
 * would call the device's gain setters); the callback's thread naming is a no-op here.  Compiled only into
 * oracle/_ref/libka9qraw16.so (oracle/raw16.mk).
 */
#define _GNU_SOURCE 1
#include <limits.h>
#include "misc.h"
#undef pthread_setname
#define pthread_setname(x) ((void)(x)) /* rx_callback names its thread once: not the oracle's to do */

#include "hydrasdr.c"

static struct frontend Ry_frontend;
static struct sdrstate Ry_sdr;

/* kind 0: INT16_REAL, 1: UINT16_REAL, 2: INT16_IQ.  A master of L, M on the reference's filter.c (REAL for 0 and 1,
 * COMPLEX for 2) and the sdrstate hydrasdr_setup leaves for that sample type (hydrasdr.c:265-276): bitspersample 16,
 * software AGC off, the given scale. */
int ry_open(int kind, int L, int M, double scale) {
  static enum hydrasdr_sample_type const types[3] = {HYDRASDR_SAMPLE_INT16_REAL, HYDRASDR_SAMPLE_UINT16_REAL,
                                                     HYDRASDR_SAMPLE_INT16_IQ};
  if (kind < 0 || kind > 2)
    return -1;
  memset(&Ry_frontend, 0, sizeof Ry_frontend);
  memset(&Ry_sdr, 0, sizeof Ry_sdr);
  N_worker_threads = 0; /* blocks run inline on the calling thread (filter.c:44) */
  Ry_frontend.isreal = kind != 2;
  if (create_filter_input(&Ry_frontend.in, L, M, Ry_frontend.isreal ? REAL : COMPLEX) != 0)
    return -1;
  Ry_frontend.bitspersample = 16;
  Ry_frontend.context = &Ry_sdr;
  Ry_sdr.frontend = &Ry_frontend;
  Ry_sdr.sample_type = types[kind];
  Ry_sdr.software_agc = false;
  Ry_sdr.scale = scale;
  return 0;
}
void ry_set_scale(double scale) { Ry_sdr.scale = scale; }

/* One transfer of `count` samples (REAL) or I/Q pairs (INT16_IQ) through rx_callback.  floats: the floats it stored
 * (count, or 2 * count for I/Q); counts[0] overranges, counts[1] samp_since_over; *if_power as it left it. */
int ry_transfer(void const *words, int count, float *floats, uint64_t *counts, double *if_power) {
  size_t const comps = (size_t)count * (Ry_frontend.isreal ? 1 : 2);
  void *copy = malloc(comps ? comps * 2 : 2);
  memcpy(copy, words, comps * 2);
  void const *wptr = Ry_frontend.isreal ? (void const *)Ry_frontend.in.input_write_pointer.r
                                        : (void const *)Ry_frontend.in.input_write_pointer.c;
  hydrasdr_transfer t = {.ctx = &Ry_sdr, .samples = copy, .sample_count = count, .sample_type = Ry_sdr.sample_type};
  int const r = rx_callback(&t);
  free(copy);
  memcpy(floats, wptr, sizeof(float) * comps); /* the mirrored ring keeps them contiguous */
  counts[0] = Ry_frontend.overranges;
  counts[1] = Ry_frontend.samp_since_over;
  *if_power = Ry_frontend.if_power;
  return r;
}

/* host wall time of n calls of rx_callback on the same transfer, in seconds, with the master's
 * write refused so that only the conversion loop runs (tools/raw16_ingest_bench.py) */
double ry_time(void const *words, int count, int n) {
  size_t const comps = (size_t)count * (Ry_frontend.isreal ? 1 : 2);
  void *copy = malloc(comps * 2);
  memcpy(copy, words, comps * 2);
  hydrasdr_transfer t = {.ctx = &Ry_sdr, .samples = copy, .sample_count = count, .sample_type = Ry_sdr.sample_type};
  struct timespec a, b;
  int const wcnt = Ry_frontend.in.wcnt;
  Ry_frontend.in.wcnt = INT_MAX / 16; /* the closing write_*filter is refused at once: no block fires, no FFT runs */
  clock_gettime(CLOCK_MONOTONIC, &a);
  for (int i = 0; i < n; i++)
    rx_callback(&t);
  clock_gettime(CLOCK_MONOTONIC, &b);
  Ry_frontend.in.wcnt = wcnt;
  free(copy);
  return (double)(b.tv_sec - a.tv_sec) + 1e-9 * (double)(b.tv_nsec - a.tv_nsec);
}

void ry_close(void) { delete_filter_input(&Ry_frontend.in); }
