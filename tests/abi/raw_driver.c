/* tests/abi/raw_driver.c -- raw 8-bit / packed 12-bit / int16 ingest through the filter.h surface, for
 * tests/test_gpu_raw_ingest.py: sessions of one master with COMPLEX slaves (plain, fine-tuned, noise) and an optional
 * SPECTRUM slave, fed raw words (write_rawfilter, write_i16filter) or floats (write_rfilter / write_cfilter), and the
 * A/D statistics (filter_ingest_stats).
 *
 * Compiled twice: against include/ka9q_gpu_filter.h (tests/abi/_build/raw_driver.so, by build()) and against the
 * reference's own src/filter.h (oracle/_ref/raw_driver_refhdr.so, oracle/raw.mk, where the reference sources exist).
 * The second declares the extensions itself, as a patched radiod would. */
#define _GNU_SOURCE 1
#include <complex.h>
#include <pthread.h>
#include <stdbool.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#ifndef FILTER_HEADER
#define FILTER_HEADER "ka9q_gpu_filter.h"
#endif
#include FILTER_HEADER

#ifndef KA9Q_GPU_FILTER_H
int Verbose = 0; /* the reference's misc.h declares it extern */
enum { FILTER_RAW_PACKED12 = 1, FILTER_RAW_U8 = 2, FILTER_RAW_S8 = 3 };
struct filter_ingest_stats {
  uint64_t blocks, samples, energy, overranges, overrange_samples, since_over;
};
int write_rawfilter(struct filter_in *master, void const *samples, int n, int format, double scale);
int filter_ingest_stats(struct filter_in *master, struct filter_ingest_stats *stats);
int write_i16filter(struct filter_in *master, int16_t const *samples, int n, float scale, bool derandomize);
int execute_filter_output_tuned(struct filter_out *slave, int shift, double remainder, double samprate, double doppler_rate,
                                double *bb_power);
int filter_input_enable_noise(struct filter_in *master, double samprate);
double filter_noise_estimate(struct filter_out const *slave);
int filter_spectrum_setup(struct filter_out *slave, int fft_n, int bin_count, float const *window);
int filter_spectrum_poll(struct filter_out *slave, int shift, int fft_avg, double overlap, float *bin_data, uint64_t *end_sample);
#endif

#define RD_MAX 16
struct rd_session {
  struct filter_in in;
  struct filter_out out[RD_MAX];
  int nchan;
  struct filter_out spec;
  bool has_spec;
};

struct rd_session *rd_open(int L, int M, int complex_in, int nworkers) {
  struct rd_session *s = calloc(1, sizeof *s);
  N_worker_threads = nworkers;
  if (create_filter_input(&s->in, L, M, complex_in ? COMPLEX : REAL) != 0) {
    free(s);
    return NULL;
  }
  return s;
}
int rd_add_channel(struct rd_session *s, int olen, double low, double high, double beta) {
  if (s->nchan == RD_MAX)
    return -1;
  struct filter_out *o = &s->out[s->nchan];
  if (create_filter_output(o, &s->in, olen, COMPLEX) != 0 || set_filter(o, low, high, beta) != 0)
    return -1;
  return s->nchan++;
}
int rd_write_raw(struct rd_session *s, void const *x, int n, int format, double scale) {
  return write_rawfilter(&s->in, x, n, format, scale);
}
int rd_write_i16(struct rd_session *s, int16_t const *x, int n, float scale, int derandomize) {
  return write_i16filter(&s->in, x, n, scale, derandomize != 0);
}
int rd_write_float(struct rd_session *s, void const *x, int n) {
  return s->in.in_type == COMPLEX ? write_cfilter(&s->in, x, n) : write_rfilter(&s->in, x, n);
}

/* the same writes from a thread of their own (joined before returning), so that the caller is not the master's owner
 * and its slaves can be lapped (filter.c:681-701), or are served their blocks in order; kind 0 floats, 1 raw, 2 int16,
 * 3 int16 derandomized */
struct rd_prod {
  struct rd_session *s;
  void const *x;
  int n, chunks, kind, format;
  double scale;
  size_t esz; /* bytes per chunk */
  int rc;     /* the last write's return */
};
static void *rd_producer(void *p) {
  struct rd_prod *a = p;
  for (int i = 0; i < a->chunks; i++) {
    void const *x = (char const *)a->x + (size_t)i * a->esz;
    if (a->kind == 1)
      a->rc = rd_write_raw(a->s, x, a->n, a->format, a->scale);
    else if (a->kind == 2 || a->kind == 3)
      a->rc = rd_write_i16(a->s, x, a->n, (float)a->scale, a->kind == 3);
    else
      a->rc = rd_write_float(a->s, x, a->n);
  }
  return NULL;
}
int rd_write_from_thread(struct rd_session *s, void const *x, int n, int chunks, size_t chunk_bytes, int kind, int format,
                         double scale) {
  struct rd_prod a = {s, x, n, chunks, kind, format, scale, chunk_bytes, 0};
  pthread_t t;
  if (pthread_create(&t, NULL, rd_producer, &a) != 0)
    return -1;
  return pthread_join(t, NULL);
}
/* one write from a thread of its own: its return (-2 if the thread could not run) */
int rd_write_once_from_thread(struct rd_session *s, void const *x, int n, int kind, int format, double scale) {
  struct rd_prod a = {s, x, n, 1, kind, format, scale, 0, 0};
  pthread_t t;
  if (pthread_create(&t, NULL, rd_producer, &a) != 0 || pthread_join(t, NULL) != 0)
    return -2;
  return a.rc;
}

int rd_execute(struct rd_session *s, int ch, int shift, float complex *dst) {
  struct filter_out *o = &s->out[ch];
  int const r = execute_filter_output(o, shift);
  memcpy(dst, o->output.c, sizeof(float complex) * (size_t)o->olen);
  return r;
}
int rd_execute_tuned(struct rd_session *s, int ch, int shift, double remainder, double samprate, float complex *dst,
                     double *bb_power) {
  struct filter_out *o = &s->out[ch];
  int const r = execute_filter_output_tuned(o, shift, remainder, samprate, 0.0, bb_power);
  memcpy(dst, o->output.c, sizeof(float complex) * (size_t)o->olen);
  return r;
}
unsigned rd_drops(struct rd_session *s, int ch) { return s->out[ch].block_drops; }
/* the master's host copy of job `job`'s spectrum (master->fdomain[], filter.c:640); returns its bins */
int rd_fdomain(struct rd_session *s, unsigned job, float complex *dst) {
  memcpy(dst, s->in.fdomain[job % ND], sizeof(float complex) * (size_t)s->in.bins);
  return s->in.bins;
}
int rd_enable_noise(struct rd_session *s, double samprate) { return filter_input_enable_noise(&s->in, samprate); }
double rd_noise(struct rd_session *s, int ch) { return filter_noise_estimate(&s->out[ch]); }
/* out[6]: blocks, samples, energy, overranges, overrange_samples, since_over */
int rd_stats(struct rd_session *s, uint64_t *out) {
  struct filter_ingest_stats st;
  int const r = filter_ingest_stats(&s->in, &st);
  if (r == 0) {
    out[0] = st.blocks;
    out[1] = st.samples;
    out[2] = st.energy;
    out[3] = st.overranges;
    out[4] = st.overrange_samples;
    out[5] = st.since_over;
  }
  return r;
}
/* a SPECTRUM slave with the wideband analyzer */
int rd_spec_setup(struct rd_session *s, int fft_n, int bin_count, float const *window) {
  if (!s->has_spec && create_filter_output(&s->spec, &s->in, 0, SPECTRUM) != 0)
    return -1;
  s->has_spec = true;
  return filter_spectrum_setup(&s->spec, fft_n, bin_count, window);
}
int rd_spec_poll(struct rd_session *s, int shift, int fft_avg, double overlap, float *bins, uint64_t *end_sample) {
  return filter_spectrum_poll(&s->spec, shift, fft_avg, overlap, bins, end_sample);
}
void rd_close(struct rd_session *s) {
  if (!s)
    return;
  for (int i = 0; i < s->nchan; i++)
    delete_filter_output(&s->out[i]);
  if (s->has_spec)
    delete_filter_output(&s->spec);
  delete_filter_input(&s->in);
  free(s);
}
