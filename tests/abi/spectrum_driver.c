/* tests/abi/spectrum_driver.c -- one master with one SPECTRUM slave through the filter.h surface, for
 * tests/test_gpu_spectrum.py: the producer (write_rfilter / write_cfilter / write_i16filter, optionally from a thread of
 * its own) and the device wideband analyzer (filter_spectrum_setup / filter_spectrum_poll). */
#define _GNU_SOURCE 1
#include <pthread.h>
#include <stdlib.h>
#include <string.h>

#include "ka9q_gpu_filter.h"

static struct filter_in In;
static struct filter_out Spec;
static int Type;

int sd_open(int L, int M, int complex_in) {
  memset(&In, 0, sizeof In);
  memset(&Spec, 0, sizeof Spec);
  Type = complex_in ? COMPLEX : REAL;
  if (create_filter_input(&In, L, M, Type) != 0)
    return -1;
  return create_filter_output(&Spec, &In, 0, SPECTRUM);
}
long sd_ring_samples(void) { return (long)(In.input_buffer_size / (Type == COMPLEX ? sizeof(float complex) : sizeof(float))); }
int sd_write_float(void const *x, int n) { /* float samples (REAL) or float complex (COMPLEX) */
  return Type == COMPLEX ? write_cfilter(&In, x, n) : write_rfilter(&In, x, n);
}
int sd_write_i16(int16_t const *x, int n, float scale, int derandomize) { return write_i16filter(&In, x, n, scale, derandomize); }
int sd_setup(int fft_n, int bin_count, float const *window) { return filter_spectrum_setup(&Spec, fft_n, bin_count, window); }
int sd_poll(int shift, int fft_avg, double overlap, float *bins, uint64_t *end_sample) {
  return filter_spectrum_poll(&Spec, shift, fft_avg, overlap, bins, end_sample);
}

/* a producer thread writing `blocks` chunks of n samples (float, or int16 when i16) while the caller polls */
static struct {
  pthread_t th;
  void const *x;
  int n, blocks, i16;
  float scale;
} P;
static void *producer(void *arg) {
  (void)arg;
  size_t const esz = P.i16 ? (Type == COMPLEX ? 4 : 2) : (Type == COMPLEX ? 8 : 4);
  for (int b = 0; b < P.blocks; b++) {
    void const *p = (char const *)P.x + (size_t)b * (size_t)P.n * esz;
    if (P.i16)
      write_i16filter(&In, p, P.n, P.scale, false);
    else
      sd_write_float(p, P.n);
  }
  return NULL;
}
int sd_producer_start(void const *x, int n, int blocks, int i16, float scale) {
  P.x = x;
  P.n = n;
  P.blocks = blocks;
  P.i16 = i16;
  P.scale = scale;
  return pthread_create(&P.th, NULL, producer, NULL);
}
int sd_producer_join(void) { return pthread_join(P.th, NULL); }

void sd_close(void) {
  delete_filter_output(&Spec);
  delete_filter_input(&In);
}
