/* tests/abi/siggen_driver.c -- a master that generates its own input (filter_siggen_setup, write_genfilter) through
 * the filter.h surface, for tests/test_gpu_siggen.py and tools/siggen_bench.py: raw_driver.c's sessions (channels,
 * floats, the wideband analyzer, writes from a thread of their own) plus the generator's calls.
 *
 * Compiled twice: against include/ka9q_gpu_filter.h (tests/abi/_build/siggen_driver.so, by build()) and against the
 * reference's own src/filter.h (oracle/_ref/siggen_driver_refhdr.so, oracle/siggen.mk, where the reference sources
 * exist).  The second declares the extensions itself, as a patched radiod would. */
#include "raw_driver.c"

#ifndef KA9Q_GPU_FILTER_H
struct filter_siggen_params {
  double freq, rate;
  double amplitude, noise;
  uint64_t seed;
};
struct filter_siggen_stats {
  uint64_t blocks, samples;
  double energy;
};
int filter_siggen_setup(struct filter_in *master, struct filter_siggen_params const *params);
int write_genfilter(struct filter_in *master, int n, double scale);
int filter_siggen_stats(struct filter_in *master, struct filter_siggen_stats *stats);
int execute_filter_output_batch(struct filter_out *const *slaves, int const *shifts, int n);
#endif

int sg_setup(struct rd_session *s, double freq, double rate, double amplitude, double noise, uint64_t seed) {
  struct filter_siggen_params const p = {freq, rate, amplitude, noise, seed};
  return filter_siggen_setup(&s->in, &p);
}
int sg_write(struct rd_session *s, int n, double scale) { return write_genfilter(&s->in, n, scale); }
/* out: blocks, samples; *energy */
int sg_stats(struct rd_session *s, uint64_t *out, double *energy) {
  struct filter_siggen_stats st;
  int const r = filter_siggen_stats(&s->in, &st);
  if (r == 0) {
    out[0] = st.blocks;
    out[1] = st.samples;
    *energy = st.energy;
  }
  return r;
}
/* fill the master's host float ring (both views are the same pages) with `v` */
void sg_fill_host_ring(struct rd_session *s, float v) {
  float *p = s->in.input_buffer;
  for (size_t i = 0; i < s->in.input_buffer_size / sizeof *p; i++)
    p[i] = v;
}
/* writes of n samples each, `chunks` times, from a thread of its own (joined): the caller is not the master's owner */
struct sg_prod {
  struct rd_session *s;
  int n, chunks;
  double scale;
};
static void *sg_producer(void *p) {
  struct sg_prod *a = p;
  for (int i = 0; i < a->chunks; i++)
    write_genfilter(&a->s->in, a->n, a->scale);
  return NULL;
}
int sg_write_from_thread(struct rd_session *s, int n, int chunks, double scale) {
  struct sg_prod a = {s, n, chunks, scale};
  pthread_t t;
  if (pthread_create(&t, NULL, sg_producer, &a) != 0)
    return -1;
  return pthread_join(t, NULL);
}
/* a lone execute_filter_output on channel ch with the master's jobs served in order (the batch of one slave) */
int sg_execute_batch(struct rd_session *s, int ch, int shift, float complex *dst) {
  struct filter_out *o = &s->out[ch];
  struct filter_out *const v[1] = {o};
  int const r = execute_filter_output_batch(v, &shift, 1);
  memcpy(dst, o->output.c, sizeof(float complex) * (size_t)o->olen);
  return r;
}
