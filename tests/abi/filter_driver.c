/* tests/abi/filter_driver.c -- flat, ctypes-friendly driver over the filter.h surface.
 *
 * Compiled twice:
 *   driver_gpuhdr.so  against include/ka9q_gpu_filter.h (our header; tests/abi/Makefile)
 *   driver_refhdr.so  against the REFERENCE's own src/filter.h (oracle/Makefile, into oracle/_ref/, only where
 *                     the reference sources exist) -- proves that code built with the reference header, i.e. the
 *                     untouched radiod sources, binds to libka9qgpu.so unchanged.
 * Both link libka9qgpu.so.  Function names match oracle/ref_driver.c so the same Python session
 * class drives the reference library and the GPU library: the parity tests read like the
 * reference's own usage (radio.c:582-620, fm.c:27-34, radio.c:1460).
 */
#define _GNU_SOURCE 1
#include <complex.h>
#include <pthread.h>
#include <stdbool.h>
#include <stddef.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include FILTER_HEADER

#ifndef KA9Q_GPU_FILTER_H
int Verbose = 0; /* the reference's misc.h declares it extern */
#endif

struct ref_session {
  struct filter_in in;
  int nchan, cap;
  struct filter_out **out;
  struct notch_state *notches;
};

struct ref_session *ref_open(int L, int M, int in_type, int nworkers) {
  struct ref_session *s = calloc(1, sizeof *s);
  N_worker_threads = nworkers;
  if (create_filter_input(&s->in, L, M, (enum filtertype)in_type) != 0) {
    free(s);
    return NULL;
  }
  return s;
}
int ref_set_notches(struct ref_session *s, int const *bins, int nbins, double alpha) {
  free(s->notches);
  s->notches = calloc((size_t)nbins + 1, sizeof *s->notches);
  for (int i = 0; i < nbins; i++) {
    s->notches[i].bin = bins[i];
    s->notches[i].alpha = alpha;
  }
  s->notches[nbins].bin = 0;
  s->notches[nbins].alpha = alpha;
  s->in.notches = s->notches;
  return 0;
}
int ref_add_channel(struct ref_session *s, int olen, int out_type, double low, double high, double beta) {
  if (s->nchan == s->cap) {
    s->cap = s->cap ? 2 * s->cap : 64;
    s->out = realloc(s->out, sizeof(*s->out) * (size_t)s->cap);
  }
  struct filter_out *o = calloc(1, sizeof *o);
  if (create_filter_output(o, &s->in, olen, (enum filtertype)out_type) != 0) {
    free(o);
    return -1;
  }
  if (out_type != SPECTRUM && set_filter(o, low, high, beta) != 0) {
    delete_filter_output(o);
    free(o);
    return -1;
  }
  s->out[s->nchan] = o;
  return s->nchan++;
}
int ref_retune_channel(struct ref_session *s, int ch, double low, double high, double beta) {
  return set_filter(s->out[ch], low, high, beta);
}
int ref_channel_points(struct ref_session *s, int ch) { return s->out[ch]->points; }
int ref_get_response(struct ref_session *s, int ch, float complex *dst) {
  memcpy(dst, s->out[ch]->response, sizeof(float complex) * (size_t)s->out[ch]->bins);
  return s->out[ch]->bins;
}
int ref_set_isb(struct ref_session *s, int ch, int isb) {
  s->out[ch]->isb = isb != 0;
  return 0;
}
int ref_write_real(struct ref_session *s, float const *x, int n) { return write_rfilter(&s->in, x, n); }
int ref_write_complex(struct ref_session *s, float complex const *x, int n) { return write_cfilter(&s->in, x, n); }
/* the way front-end drivers really do it (rx888.c:800-826): write through the ring pointer, then
 * publish with a NULL buffer */
int ref_write_real_inplace(struct ref_session *s, float const *x, int n) {
  memcpy(s->in.input_write_pointer.r, x, sizeof(float) * (size_t)n);
  return write_rfilter(&s->in, NULL, n);
}
#ifdef KA9Q_GPU_FILTER_H
int ref_write_i16(struct ref_session *s, int16_t const *x, int n, float scale, int derand) {
  return write_i16filter(&s->in, x, n, scale, derand != 0);
}
#endif
int ref_get_spectrum(struct ref_session *s, float complex *dst) {
  unsigned const job = s->in.next_jobnum - 1;
  memcpy(dst, s->in.fdomain[job % ND], sizeof(float complex) * (size_t)s->in.bins);
  return s->in.bins;
}
int ref_master_bins(struct ref_session *s) { return s->in.bins; }
int ref_execute_channel(struct ref_session *s, int ch, int shift, float complex *dst, float complex *full,
                        float complex *fdom) {
  struct filter_out *o = s->out[ch];
  int const r = execute_filter_output(o, shift);
  if (dst && o->output.c)
    memcpy(dst, o->output.c, sizeof(float complex) * (size_t)o->olen);
  (void)full;
  (void)fdom;
  return r;
}
unsigned ref_channel_drops(struct ref_session *s, int ch) { return s->out[ch]->block_drops; }
int ref_set_beam(struct ref_session *s, int ch, int beam, double ire, double iim, double qre, double qim) {
  s->out[ch]->beam = beam != 0;
  return set_filter_weights(s->out[ch], ire + I * iim, qre + I * qim);
}
/* REAL-output slave (wfm.c:76-77,188): dst receives olen floats */
int ref_execute_channel_real(struct ref_session *s, int ch, int shift, float *dst) {
  struct filter_out *o = s->out[ch];
  int const r = execute_filter_output(o, shift);
  if (dst && o->output.r)
    memcpy(dst, o->output.r, sizeof(float) * (size_t)o->olen);
  return r;
}
/* the consumer falls `skip` blocks behind before it asks again: lap semantics of filter.c:690-701.
 * Returns block_drops afterwards; dst receives what that execute_filter_output left in output.c */
unsigned ref_lap_probe(struct ref_session *s, int ch, int shift, float const *x, int skip, float complex *dst) {
  struct filter_out *o = s->out[ch];
  int const L = s->in.ilen;
  /* written from another thread context than the consumer: the producer must not be `owner` of this call's thread
   * (filter.c:681-683 would hand it the latest block instead); ref_lap_producer below runs the writes */
  (void)x;
  (void)skip;
  (void)L;
  execute_filter_output(o, shift);
  if (dst && o->output.c)
    memcpy(dst, o->output.c, sizeof(float complex) * (size_t)o->olen);
  return o->block_drops;
}
struct lap_arg {
  struct ref_session *s;
  float const *x;
  int nblocks;
};
static void *lap_producer(void *p) {
  struct lap_arg *a = p;
  int const L = a->s->in.ilen;
  for (int b = 0; b < a->nblocks; b++)
    write_rfilter(&a->s->in, a->x + (size_t)b * L, L);
  return NULL;
}
/* nblocks blocks written by a separate producer thread (joined before returning) */
int ref_produce_from_thread(struct ref_session *s, float const *x, int nblocks) {
  struct lap_arg a = {s, x, nblocks};
  pthread_t t;
  if (pthread_create(&t, NULL, lap_producer, &a) != 0)
    return -1;
  pthread_join(t, NULL);
  return 0;
}
unsigned ref_channel_next_job(struct ref_session *s, int ch) { return s->out[ch]->next_jobnum; }
#ifdef KA9Q_GPU_FILTER_H
/* extensions of the GPU library */
int ref_execute_tuned(struct ref_session *s, int ch, int shift, double remainder, double samprate, double doppler_rate,
                      float complex *dst, double *bb_power) {
  struct filter_out *o = s->out[ch];
  int const r = execute_filter_output_tuned(o, shift, remainder, samprate, doppler_rate, bb_power);
  if (dst && o->output.c)
    memcpy(dst, o->output.c, sizeof(float complex) * (size_t)o->olen);
  return r;
}
int ref_enable_noise(struct ref_session *s, double samprate) { return filter_input_enable_noise(&s->in, samprate); }
double ref_noise(struct ref_session *s, int ch) { return filter_noise_estimate(s->out[ch]); }
/* all channels of the session with one call; dst: nchan pointers to olen complex each */
int ref_execute_batch(struct ref_session *s, int const *shifts, float complex **dst) {
  int const r = execute_filter_output_batch((struct filter_out *const *)s->out, shifts, s->nchan);
  for (int i = 0; i < s->nchan; i++)
    if (dst && dst[i] && s->out[i]->output.c)
      memcpy(dst[i], s->out[i]->output.c, sizeof(float complex) * (size_t)s->out[i]->olen);
  return r;
}
int ref_write_i16_inplace(struct ref_session *s, int16_t const *x, int n, float scale) {
  int16_t *w = filter_i16_write_pointer(&s->in);
  if (!w)
    return -1;
  memcpy(w, x, sizeof(int16_t) * (size_t)n);
  return write_i16filter(&s->in, NULL, n, scale, false);
}
#endif
unsigned long long ref_channel_sample_index(struct ref_session *s, int ch) { return s->out[ch]->sample_index; }
void ref_close(struct ref_session *s) {
  if (!s)
    return;
  for (int i = 0; i < s->nchan; i++) {
    delete_filter_output(s->out[i]);
    free(s->out[i]);
  }
  free(s->out);
  s->in.notches = NULL;
  delete_filter_input(&s->in);
  free(s->notches);
  free(s);
}

/* ---- radiod-style threading: one producer, one pthread per channel (radio.c:996,1460) -------- */
struct chan_job {
  struct filter_out *o;
  int shift, nblocks;
  float complex *dst; /* nblocks*olen */
};
static void *chan_main(void *p) {
  struct chan_job *j = p;
  for (int b = 0; b < j->nblocks; b++) {
    execute_filter_output(j->o, j->shift);
    memcpy(j->dst + (size_t)b * j->o->olen, j->o->output.c, sizeof(float complex) * (size_t)j->o->olen);
  }
  return NULL;
}
/* feeds nblocks*L real samples from a separate producer thread context (this thread) while every
 * channel runs in its own thread; returns total dropped blocks */
int ref_threaded_run(struct ref_session *s, float const *x, int nblocks, int const *shifts, float complex **dsts) {
  int const n = s->nchan, L = s->in.ilen;
  pthread_t *t = calloc((size_t)n, sizeof *t);
  struct chan_job *jobs = calloc((size_t)n, sizeof *jobs);
  for (int i = 0; i < n; i++) {
    jobs[i] = (struct chan_job){s->out[i], shifts[i], nblocks, dsts[i]};
    s->out[i]->next_jobnum = s->in.next_jobnum;
    pthread_create(&t[i], NULL, chan_main, &jobs[i]);
  }
  for (int b = 0; b < nblocks; b++) {
    memcpy(s->in.input_write_pointer.r, x + (size_t)b * L, sizeof(float) * (size_t)L);
    write_rfilter(&s->in, NULL, L);
    /* pace like an ADC would: never more than ND-1 blocks ahead of the slowest channel */
    for (;;) {
      unsigned lag = 0;
      for (int i = 0; i < n; i++) {
        unsigned const d = s->in.next_jobnum - *(volatile unsigned *)&s->out[i]->next_jobnum;
        if (d > lag)
          lag = d;
      }
      if (lag < ND - 1)
        break;
      struct timespec ts = {0, 50000};
      nanosleep(&ts, NULL);
    }
  }
  unsigned drops = 0;
  for (int i = 0; i < n; i++) {
    pthread_join(t[i], NULL);
    drops += s->out[i]->block_drops;
  }
  free(t);
  free(jobs);
  return (int)drops;
}

/* ---- struct layout report: same text from either header => binary compatible --------------- */
#define OFF(T, f) n += snprintf(buf + n, (size_t)(len - n), #T "." #f " %zu %zu\n", offsetof(struct T, f), sizeof(((struct T *)0)->f))
int ref_layout_report(char *buf, int len) {
  int n = 0;
  n += snprintf(buf + n, (size_t)(len - n), "sizeof filter_in %zu filter_out %zu rc %zu notch_state %zu ND %d\n",
                sizeof(struct filter_in), sizeof(struct filter_out), sizeof(struct rc), sizeof(struct notch_state), ND);
  n += snprintf(buf + n, (size_t)(len - n), "enum %d %d %d %d\n", (int)NONE, (int)COMPLEX, (int)REAL, (int)SPECTRUM);
  OFF(filter_in, in_type); OFF(filter_in, points); OFF(filter_in, ilen); OFF(filter_in, bins);
  OFF(filter_in, impulse_length); OFF(filter_in, wcnt); OFF(filter_in, input_buffer); OFF(filter_in, input_buffer_size);
  OFF(filter_in, input_write_pointer); OFF(filter_in, input_read_pointer); OFF(filter_in, fwd_plan);
  OFF(filter_in, filter_mutex); OFF(filter_in, filter_cond); OFF(filter_in, notches); OFF(filter_in, fdomain);
  OFF(filter_in, next_jobnum); OFF(filter_in, completed_jobs); OFF(filter_in, perform_inline);
  OFF(filter_in, sample_index); OFF(filter_in, samples_by_job); OFF(filter_in, init); OFF(filter_in, owner);
  OFF(filter_out, master); OFF(filter_out, out_type); OFF(filter_out, points); OFF(filter_out, olen);
  OFF(filter_out, bins); OFF(filter_out, alpha); OFF(filter_out, beta); OFF(filter_out, fdomain);
  OFF(filter_out, response); OFF(filter_out, response_mutex); OFF(filter_out, output_buffer); OFF(filter_out, output);
  OFF(filter_out, rev_plan); OFF(filter_out, next_jobnum); OFF(filter_out, block_drops); OFF(filter_out, rcnt);
  OFF(filter_out, sample_index); OFF(filter_out, beam); OFF(filter_out, isb); OFF(filter_out, init);
  OFF(notch_state, bin); OFF(notch_state, state); OFF(notch_state, alpha);
  OFF(rc, r); OFF(rc, c);
  return n;
}
