/* tests/abi/iqcorr_driver.c -- HackRF and FUNcube I/Q correction through the filter.h surface, for
 * tests/test_gpu_iq_correction.py and tools/iq_correction_bench.py: sessions of one master with COMPLEX slaves
 * and an optional SPECTRUM slave, fed corrected raw words (filter_iq_correction_setup, write_rawfilter) or floats
 * (write_cfilter), and the per-write records (filter_iq_records).
 *
 * Compiled twice: against include/ka9q_gpu_filter.h (tests/abi/_build/iqcorr_driver.so, by build()) and against the
 * reference's own src/filter.h (oracle/_ref/iqcorr_driver_refhdr.so, oracle/iqcorr.mk, where the reference sources
 * exist).  The second declares the extensions itself, as a patched radiod would. */
#define _GNU_SOURCE 1
#include <complex.h>
#include <pthread.h>
#include <stdbool.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>
#ifndef FILTER_HEADER
#define FILTER_HEADER "ka9q_gpu_filter.h"
#endif
#include FILTER_HEADER

#ifndef KA9Q_GPU_FILTER_H
int Verbose = 0; /* the reference's misc.h declares it extern */
enum { FILTER_RAW_S8_IQCORR = 4, FILTER_RAW_S16_IQCORR = 5 };
struct filter_iq_params {
  double dc_alpha, gp_rate, gp_alpha;
  double dc_i, dc_q, sinphi, imbalance, gain_i, gain_q, secphi, tanphi;
};
struct filter_iq_record {
  int64_t seq, n, sum_i, sum_q;
  double i_energy, q_energy, dotprod;
  int64_t overs, since_over;
  double dc_i, dc_q, sinphi, imbalance, gain_i, gain_q, secphi, tanphi;
};
struct filter_ingest_stats {
  uint64_t blocks, samples, energy, overranges, overrange_samples, since_over;
};
int filter_iq_correction_setup(struct filter_in *master, int format, struct filter_iq_params const *params);
int filter_iq_records(struct filter_in *master, struct filter_iq_record *recs, int max);
int write_rawfilter(struct filter_in *master, void const *samples, int n, int format, double scale);
int filter_ingest_stats(struct filter_in *master, struct filter_ingest_stats *stats);
int execute_filter_output_tuned(struct filter_out *slave, int shift, double remainder, double samprate, double doppler_rate,
                                double *bb_power);
int filter_input_enable_noise(struct filter_in *master, double samprate);
double filter_noise_estimate(struct filter_out const *slave);
int filter_spectrum_setup(struct filter_out *slave, int fft_n, int bin_count, float const *window);
int filter_spectrum_poll(struct filter_out *slave, int shift, int fft_avg, double overlap, float *bin_data, uint64_t *end_sample);
#endif

#define IQ_MAX 16
struct iq_session {
  struct filter_in in;
  struct filter_out out[IQ_MAX];
  int nchan;
  struct filter_out spec;
  bool has_spec;
};

struct iq_session *iq_open(int L, int M, int complex_in, int nworkers) {
  struct iq_session *s = calloc(1, sizeof *s);
  N_worker_threads = nworkers;
  if (create_filter_input(&s->in, L, M, complex_in ? COMPLEX : REAL) != 0) {
    free(s);
    return NULL;
  }
  return s;
}
/* p: dc_alpha, gp_rate, gp_alpha, then the initial dc_i, dc_q, sinphi, imbalance, gain_i, gain_q, secphi, tanphi */
int iq_setup(struct iq_session *s, int format, double const *p) {
  struct filter_iq_params q;
  memcpy(&q, p, sizeof q);
  return filter_iq_correction_setup(&s->in, format, &q);
}
int iq_add_channel(struct iq_session *s, int olen, double low, double high, double beta) {
  if (s->nchan == IQ_MAX)
    return -1;
  struct filter_out *o = &s->out[s->nchan];
  if (create_filter_output(o, &s->in, olen, COMPLEX) != 0 || set_filter(o, low, high, beta) != 0)
    return -1;
  return s->nchan++;
}
int iq_write_raw(struct iq_session *s, void const *x, int n, int format, double scale) {
  return write_rawfilter(&s->in, x, n, format, scale);
}
int iq_write_float(struct iq_session *s, float complex const *x, int n) { return write_cfilter(&s->in, x, n); }
/* records as the library returns them (struct filter_iq_record, 17 eight-byte fields each) */
int iq_records(struct iq_session *s, void *recs, int max) { return filter_iq_records(&s->in, recs, max); }
int iq_stats(struct iq_session *s) {
  struct filter_ingest_stats st;
  return filter_ingest_stats(&s->in, &st);
}

/* chunks writes of n pairs (chunk_bytes apart) from a thread of their own, joined before returning, so that the caller
 * is not the master's owner and its slaves can be lapped (filter.c:681-701); kind 0 floats, 1 raw */
struct iq_prod {
  struct iq_session *s;
  void const *x;
  int n, chunks, kind, format;
  double scale;
  size_t esz;
};
static void *iq_producer(void *p) {
  struct iq_prod *a = p;
  for (int i = 0; i < a->chunks; i++) {
    void const *x = (char const *)a->x + (size_t)i * a->esz;
    if (a->kind == 1)
      iq_write_raw(a->s, x, a->n, a->format, a->scale);
    else
      iq_write_float(a->s, x, a->n);
  }
  return NULL;
}
int iq_write_from_thread(struct iq_session *s, void const *x, int n, int chunks, size_t chunk_bytes, int kind, int format,
                         double scale) {
  struct iq_prod a = {s, x, n, chunks, kind, format, scale, chunk_bytes};
  pthread_t t;
  if (pthread_create(&t, NULL, iq_producer, &a) != 0)
    return -1;
  return pthread_join(t, NULL);
}

int iq_execute(struct iq_session *s, int ch, int shift, float complex *dst) {
  struct filter_out *o = &s->out[ch];
  int const r = execute_filter_output(o, shift);
  memcpy(dst, o->output.c, sizeof(float complex) * (size_t)o->olen);
  return r;
}
int iq_execute_tuned(struct iq_session *s, int ch, int shift, double remainder, double samprate, float complex *dst,
                     double *bb_power) {
  struct filter_out *o = &s->out[ch];
  int const r = execute_filter_output_tuned(o, shift, remainder, samprate, 0.0, bb_power);
  memcpy(dst, o->output.c, sizeof(float complex) * (size_t)o->olen);
  return r;
}
unsigned iq_drops(struct iq_session *s, int ch) { return s->out[ch].block_drops; }
int iq_enable_noise(struct iq_session *s, double samprate) { return filter_input_enable_noise(&s->in, samprate); }
double iq_noise(struct iq_session *s, int ch) { return filter_noise_estimate(&s->out[ch]); }
int iq_spec_setup(struct iq_session *s, int fft_n, int bin_count, float const *window) {
  if (!s->has_spec && create_filter_output(&s->spec, &s->in, 0, SPECTRUM) != 0)
    return -1;
  s->has_spec = true;
  return filter_spectrum_setup(&s->spec, fft_n, bin_count, window);
}
int iq_spec_poll(struct iq_session *s, int shift, int fft_avg, double overlap, float *bins, uint64_t *end_sample) {
  return filter_spectrum_poll(&s->spec, shift, fft_avg, overlap, bins, end_sample);
}

/* wall time of `writes` writes of n pairs each (raw when kind 1, floats when 0) and every channel's output of each block
 * they fire, in seconds (tools/iq_correction_bench.py) */
double iq_time(struct iq_session *s, void const *x, int n, int writes, size_t write_bytes, int kind, int format, double scale) {
  struct timespec a, b;
  clock_gettime(CLOCK_MONOTONIC, &a);
  for (int w = 0; w < writes; w++) {
    void const *p = (char const *)x + (size_t)w * write_bytes;
    int const fired = kind == 1 ? iq_write_raw(s, p, n, format, scale) : iq_write_float(s, p, n);
    if (fired == 1)
      for (int c = 0; c < s->nchan; c++)
        execute_filter_output(&s->out[c], 0);
  }
  clock_gettime(CLOCK_MONOTONIC, &b);
  return (double)(b.tv_sec - a.tv_sec) + 1e-9 * (double)(b.tv_nsec - a.tv_nsec);
}

void iq_close(struct iq_session *s) {
  if (!s)
    return;
  for (int i = 0; i < s->nchan; i++)
    delete_filter_output(&s->out[i]);
  if (s->has_spec)
    delete_filter_output(&s->spec);
  delete_filter_input(&s->in);
  free(s);
}
