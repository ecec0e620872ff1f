/* tests/abi/nbspectrum_driver.c -- one master and a few COMPLEX slaves through the filter.h surface, for
 * tests/test_gpu_narrowband_spectrum.py: the producer (write_i16filter, optionally from a thread of its own), deliveries
 * (execute_filter_output_tuned, execute_filter_output, execute_filter_output_batch) with a copy of every delivered block,
 * and the device narrowband analyzer (filter_spectrum_narrow_*). */
#define _GNU_SOURCE 1
#include <pthread.h>
#include <stdlib.h>
#include <string.h>

#include "ka9q_gpu_filter.h"

#define NS 8
static struct filter_in In;
static struct filter_out Out[NS];
static int Nout;

int nd_open(int L, int M) {
  memset(&In, 0, sizeof In);
  memset(Out, 0, sizeof Out);
  Nout = 0;
  return create_filter_input(&In, L, M, REAL);
}
/* a COMPLEX slave of olen samples per block with its filter; returns its index */
int nd_add(int olen, double low, double high, double beta) {
  if (Nout >= NS || create_filter_output(&Out[Nout], &In, olen, COMPLEX) != 0 || set_filter(&Out[Nout], low, high, beta) != 0)
    return -1;
  return Nout++;
}
int nd_write_i16(int16_t const *x, int n, float scale) { return write_i16filter(&In, x, n, scale, false); }

/* delivery of the next block to slave k, copied to y (olen float complex) */
int nd_tuned(int k, int shift, double remainder, double samprate, float complex *y) {
  double pw = 0;
  int const rc = execute_filter_output_tuned(&Out[k], shift, remainder, samprate, 0.0, &pw);
  memcpy(y, Out[k].output.c, sizeof *y * (size_t)Out[k].olen);
  return rc;
}
int nd_plain(int k, int shift, float complex *y) {
  int const rc = execute_filter_output(&Out[k], shift);
  memcpy(y, Out[k].output.c, sizeof *y * (size_t)Out[k].olen);
  return rc;
}
/* slaves ks[0 .. n) in one execute_filter_output_batch; ys[i] receives slave ks[i]'s block */
int nd_batch(int n, int const *ks, int const *shifts, float complex **ys) {
  struct filter_out *s[NS] = {0};
  if (n < 1 || n > NS)
    return -1;
  for (int i = 0; i < n; i++)
    s[i] = &Out[ks[i]];
  int const rc = execute_filter_output_batch(s, shifts, n);
  for (int i = 0; i < n; i++)
    memcpy(ys[i], Out[ks[i]].output.c, sizeof(float complex) * (size_t)Out[ks[i]].olen);
  return rc;
}
unsigned nd_drops(int k) { return Out[k].block_drops; }

int nd_setup(int k, int fft_n, int bin_count, float const *window) {
  return filter_spectrum_narrow_setup(&Out[k], fft_n, bin_count, window);
}
int nd_reserve(int k, long ring_samples) { return filter_spectrum_narrow_reserve(&Out[k], ring_samples); }
int nd_poll(int k, int fft_avg, double overlap, float *bins) { return filter_spectrum_narrow_poll(&Out[k], fft_avg, overlap, bins); }
long nd_ring(int k, float complex *ring, long cap, long *ring_idx) { return filter_spectrum_narrow_ring(&Out[k], ring, cap, ring_idx); }
int nd_delete(int k) { return delete_filter_output(&Out[k]); }

/* a producer thread writing `blocks` int16 blocks of n samples; with `ahead` > 0 it waits until no more than `ahead`
 * blocks are written but not yet released by nd_release(), so a consumer on another thread is never lapped */
static struct {
  pthread_t th;
  int16_t const *x;
  int n, blocks, ahead;
  float scale;
  int written, released;
  pthread_mutex_t mu;
  pthread_cond_t cv;
} P = {.mu = PTHREAD_MUTEX_INITIALIZER, .cv = PTHREAD_COND_INITIALIZER};
static void *producer(void *arg) {
  (void)arg;
  for (int b = 0; b < P.blocks; b++) {
    pthread_mutex_lock(&P.mu);
    while (P.ahead > 0 && P.written - P.released >= P.ahead)
      pthread_cond_wait(&P.cv, &P.mu);
    pthread_mutex_unlock(&P.mu);
    write_i16filter(&In, P.x + (size_t)b * (size_t)P.n, P.n, P.scale, false);
    pthread_mutex_lock(&P.mu);
    P.written++;
    pthread_cond_broadcast(&P.cv);
    pthread_mutex_unlock(&P.mu);
  }
  return NULL;
}
/* with ahead > 0 it returns once the first block is issued: until then the calling thread still owns the master, and
 * execute_filter_output would take "the latest block" (filter.c:681-683) instead of waiting for block 0 */
int nd_producer_start(int16_t const *x, int n, int blocks, int ahead, float scale) {
  P.x = x;
  P.n = n;
  P.blocks = blocks;
  P.ahead = ahead;
  P.scale = scale;
  P.written = P.released = 0;
  int const rc = pthread_create(&P.th, NULL, producer, NULL);
  if (rc == 0 && ahead > 0) {
    pthread_mutex_lock(&P.mu);
    while (P.written < 1)
      pthread_cond_wait(&P.cv, &P.mu);
    pthread_mutex_unlock(&P.mu);
  }
  return rc;
}
void nd_release(void) {
  pthread_mutex_lock(&P.mu);
  P.released++;
  pthread_cond_broadcast(&P.cv);
  pthread_mutex_unlock(&P.mu);
}
int nd_producer_join(void) { return pthread_join(P.th, NULL); }

void nd_close(void) {
  for (int k = 0; k < Nout; k++)
    delete_filter_output(&Out[k]);
  delete_filter_input(&In);
}
