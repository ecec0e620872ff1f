/* tests/abi/siggen_mod_driver.c -- a master that generates sig_gen's AM or DSB source (filter_siggen_setup,
 * filter_siggen_modulate, filter_siggen_mod_pointer, write_genfilter) through the filter.h surface, for
 * tests/test_gpu_siggen_mod.py and tools/siggen_mod_bench.py: siggen_driver.c's sessions plus the envelope writes a
 * patched sig_gen.c makes (src_callback_read into the library's envelope ring, then write_genfilter).
 *
 * Compiled twice: against include/ka9q_gpu_filter.h (tests/abi/_build/siggen_mod_driver.so, by build()) and against the
 * reference's own src/filter.h (oracle/_ref/siggen_mod_driver_refhdr.so, oracle/siggen_mod.mk, where the reference
 * sources exist).  The second declares the extensions itself, as a patched radiod would. */
#include "siggen_driver.c"

#ifndef KA9Q_GPU_FILTER_H
int filter_siggen_modulate(struct filter_in *master, double dc);
float *filter_siggen_mod_pointer(struct filter_in *master);
#endif

int sgm_modulate(struct rd_session *s, double dc) { return filter_siggen_modulate(&s->in, dc); }
int sgm_has_pointer(struct rd_session *s) { return filter_siggen_mod_pointer(&s->in) != NULL; }
/* the driver's iteration: n envelope floats where the library wants them (as src_callback_read would write them), then
 * write_genfilter; -2 when the master has no envelope pointer */
int sgm_write(struct rd_session *s, float const *env, int n, double scale) {
  float *p = filter_siggen_mod_pointer(&s->in);
  if (p == NULL)
    return -2;
  memcpy(p, env, sizeof(float) * (size_t)n);
  return write_genfilter(&s->in, n, scale);
}
/* `chunks` such iterations of n floats each, from env onwards, from a thread of its own (joined) */
struct sgm_prod {
  struct rd_session *s;
  float const *env;
  int n, chunks;
  double scale;
};
static void *sgm_producer(void *p) {
  struct sgm_prod *a = p;
  for (int i = 0; i < a->chunks; i++)
    sgm_write(a->s, a->env + (size_t)i * (size_t)a->n, a->n, a->scale);
  return NULL;
}
int sgm_write_from_thread(struct rd_session *s, float const *env, int n, int chunks, double scale) {
  struct sgm_prod a = {s, env, n, chunks, scale};
  pthread_t t;
  if (pthread_create(&t, NULL, sgm_producer, &a) != 0)
    return -1;
  return pthread_join(t, NULL);
}
