/* tests/abi/small_driver.c -- filter_driver.c's sessions, whose masters are made by create_filter_input_small after
 * small_set_mode(1) (falling back to create_filter_input outside its envelope, as the patched radiod callers do), plus
 * P threads that each own a master and its slaves, for tests/test_gpu_small_masters.py and tools/small_master_bench.py.
 *
 * Compiled twice: against include/ka9q_gpu_filter.h (tests/abi/_build/small_driver.so, by build()) and against the
 * reference's own src/filter.h (oracle/_ref/small_driver_refhdr.so, oracle/small.mk, where the reference sources exist).
 * The second declares the extension itself, as a patched radiod would. */
#define _GNU_SOURCE 1
#include <complex.h>
#include <pthread.h>
#include <stdbool.h>
#include <stdint.h>
#include <string.h>
#include <time.h>
#ifndef FILTER_HEADER
#define FILTER_HEADER "ka9q_gpu_filter.h"
#endif
#include FILTER_HEADER

#ifndef KA9Q_GPU_FILTER_H
int create_filter_input_small(struct filter_in *master, int L, int M, enum filtertype in_type);
#endif

static int small_mode;
static __thread int small_taken;
static int drv_create_filter_input(struct filter_in *master, int L, int M, enum filtertype in_type) {
  small_taken = small_mode && create_filter_input_small(master, L, M, in_type) == 0;
  return small_taken ? 0 : create_filter_input(master, L, M, in_type);
}
#define create_filter_input drv_create_filter_input
#include "filter_driver.c"
#undef create_filter_input

int small_set_mode(int on) {
  small_mode = on != 0;
  return 0;
}
/* whether the calling thread's last ref_open made a small master */
int small_last_taken(void) { return small_taken; }

/* P threads, each with a master of its own (L, M, in_type) and ns slaves (olen, out_type, low, high, beta, shift), all
 * fed the same nb blocks of x (L floats or float pairs each) and read block by block as radiod's channel threads do
 * (perform_inline, the owner shortcut).  out: per thread, per block, per slave 2 * olen[i] floats (REAL slaves use the
 * first olen).  Returns the largest thread's wall time of the write / read loop in ns, after all threads have set up
 * (a barrier), or -1 if any call failed; *small_count: how many masters took the small path. */
struct st_arg {
  int L, M, in_type, ns, nb;
  int const *olen, *otype, *shift;
  double const *lo, *hi, *beta;
  void const *x;
  float *out;
  long per_thread;
  pthread_barrier_t *bar;
  long long ns_elapsed;
  int rc, small;
};
static long long now_ns(void) {
  struct timespec t;
  clock_gettime(CLOCK_MONOTONIC, &t);
  return (long long)t.tv_sec * 1000000000LL + t.tv_nsec;
}
static void *st_main(void *p) {
  struct st_arg *a = p;
  struct filter_in in;
  struct filter_out outs[8];
  memset(&in, 0, sizeof in);
  memset(outs, 0, sizeof outs);
  int rc = drv_create_filter_input(&in, a->L, a->M, (enum filtertype)a->in_type);
  a->small = small_taken;
  in.perform_inline = true;
  for (int i = 0; rc == 0 && i < a->ns; i++) {
    rc = create_filter_output(&outs[i], &in, a->olen[i], (enum filtertype)a->otype[i]);
    rc = rc ? rc : set_filter(&outs[i], a->lo[i], a->hi[i], a->beta[i]);
  }
  pthread_barrier_wait(a->bar);
  long long const t0 = now_ns();
  size_t const esz = a->in_type == COMPLEX ? sizeof(float complex) : sizeof(float);
  float *o = a->out;
  for (int b = 0; rc == 0 && b < a->nb; b++) {
    void const *blk = (char const *)a->x + (size_t)b * (size_t)a->L * esz;
    if ((a->in_type == COMPLEX ? write_cfilter(&in, blk, a->L) : write_rfilter(&in, blk, a->L)) != 1)
      rc = -1;
    for (int i = 0; rc == 0 && i < a->ns; i++) {
      rc = execute_filter_output(&outs[i], a->shift[i]);
      if (o)
        memcpy(o, a->otype[i] == REAL ? (void const *)outs[i].output.r : (void const *)outs[i].output.c,
               (a->otype[i] == REAL ? sizeof(float) : sizeof(float complex)) * (size_t)a->olen[i]);
      if (o)
        o += 2 * a->olen[i];
    }
  }
  a->ns_elapsed = now_ns() - t0;
  for (int i = 0; i < a->ns; i++)
    delete_filter_output(&outs[i]);
  delete_filter_input(&in);
  a->rc = rc;
  return NULL;
}
long long small_threads(int P, int L, int M, int in_type, int ns, int const *olen, int const *otype, double const *lo,
                        double const *hi, double const *beta, int const *shift, int nb, void const *x, float *out,
                        int *small_count) {
  if (P < 1 || ns < 0 || ns > 8)
    return -1;
  N_worker_threads = 0;
  long per = 0;
  for (int i = 0; i < ns; i++)
    per += 2L * olen[i];
  per *= nb;
  struct st_arg *a = calloc((size_t)P, sizeof *a);
  pthread_t *t = calloc((size_t)P, sizeof *t);
  pthread_barrier_t bar;
  pthread_barrier_init(&bar, NULL, (unsigned)P);
  for (int p = 0; p < P; p++) {
    a[p] = (struct st_arg){L, M, in_type, ns, nb, olen, otype, shift, lo, hi, beta, x, out ? out + (size_t)p * (size_t)per : NULL,
                           per, &bar, 0, 0, 0};
    pthread_create(&t[p], NULL, st_main, &a[p]);
  }
  long long worst = 0;
  int bad = 0, nsmall = 0;
  for (int p = 0; p < P; p++) {
    pthread_join(t[p], NULL);
    bad |= a[p].rc != 0;
    nsmall += a[p].small;
    if (a[p].ns_elapsed > worst)
      worst = a[p].ns_elapsed;
  }
  pthread_barrier_destroy(&bar);
  free(a);
  free(t);
  if (small_count)
    *small_count = nsmall;
  return bad ? -1 : worst;
}

#ifdef KA9Q_GPU_FILTER_H
/* Every extension a small master refuses, called on the session's master and its slave ch; returns a bit per call that
 * did NOT refuse (0: all refused). */
int small_refusals(struct ref_session *s, int ch) {
  struct filter_in *f = &s->in;
  struct filter_out *o = s->out[ch];
  int bad = 0, bit = 0;
  double pw;
  int16_t w[16] = {0};
  float win[64] = {0}, bins[64];
  uint64_t end;
  struct filter_ingest_stats is;
  struct filter_iq_params iqp = {1e-6, 0, 0, 0, 0, 0, 0, 1, 1, 1, 0};
  struct filter_iq_record rec;
  struct filter_siggen_params gp = {0.1, 0, 1, 0, 1};
  struct filter_siggen_stats gs;
  float complex ring[4];
  long idx;
  struct filter_out spec;
  memset(&spec, 0, sizeof spec);
#define REFUSED(call) bad |= ((call) != -1) << bit++
  REFUSED(execute_filter_output_tuned(o, 0, 0.0, 48000.0, 0.0, &pw));
  REFUSED(filter_output_untune(o));
  REFUSED(filter_input_enable_noise(f, 48000.0));
  REFUSED(filter_spectrum_setup(o, 64, 64, win));
  REFUSED(filter_spectrum_poll(o, 0, 1, 0.5, bins, &end));
  REFUSED(filter_spectrum_narrow_setup(o, 64, 64, win));
  REFUSED(filter_spectrum_narrow_reserve(o, 1024));
  REFUSED(filter_spectrum_narrow_poll(o, 1, 0.5, bins));
  REFUSED(filter_spectrum_narrow_ring(o, ring, 4, &idx));
  REFUSED(write_i16filter(f, w, 16, 1.0f, false));
  bad |= (filter_i16_write_pointer(f) != NULL) << bit++;
  REFUSED(write_rawfilter(f, w, 16, FILTER_RAW_S16, 1.0));
  REFUSED(write_rawfilter_planar(f, w, w, 8, 1.0));
  REFUSED(filter_ingest_stats(f, &is));
  REFUSED(filter_iq_correction_setup(f, FILTER_RAW_S16_IQCORR, &iqp));
  REFUSED(filter_iq_records(f, &rec, 1));
  REFUSED(filter_siggen_setup(f, &gp));
  REFUSED(write_genfilter(f, 16, 1.0));
  REFUSED(filter_siggen_modulate(f, 1.0));
  bad |= (filter_siggen_mod_pointer(f) != NULL) << bit++;
  REFUSED(filter_siggen_stats(f, &gs));
  REFUSED(create_filter_output(&spec, f, 0, SPECTRUM));
  bool const beam = o->beam;
  o->beam = true; /* beam synthesis: refused when the slave is next served */
  REFUSED(execute_filter_output(o, 0));
  o->beam = beam;
#undef REFUSED
  return bad;
}
long small_master_bytes(int L, int M, int in_type, int max_slaves) {
  return filter_small_master_bytes(L, M, (enum filtertype)in_type, max_slaves);
}
#endif
