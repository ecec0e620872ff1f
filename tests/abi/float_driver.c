/* tests/abi/float_driver.c -- float ingest through the filter.h surface, for tests/test_gpu_float_ingest.py and
 * tools/float_ingest_bench.py: raw_driver.c's sessions (write_rawfilter with FILTER_RAW_F32 / CF32 / CF32_CNRMF /
 * CF32_FSCALE, floats, channels, the wideband analyzer), plus the statistics with their double energy.
 *
 * Compiled twice: against include/ka9q_gpu_filter.h (tests/abi/_build/float_driver.so, by build()) and against the
 * reference's own src/filter.h (oracle/_ref/float_driver_refhdr.so, oracle/float.mk, where the reference sources exist).
 * The second declares the extensions itself, as a patched radiod would. */
#include "raw_driver.c"

#ifndef KA9Q_GPU_FILTER_H
enum { FILTER_RAW_F32 = 9, FILTER_RAW_CF32 = 10, FILTER_RAW_CF32_CNRMF = 11, FILTER_RAW_CF32_FSCALE = 12 };
#define FENERGY(st) (*(double const *)&(st).energy) /* the union's double member, in the same 8 bytes */
#else
#define FENERGY(st) ((st).fenergy)
#endif

/* counts[5]: blocks, samples, overranges, overrange_samples, since_over; *energy: fenergy */
int rd_fstats(struct rd_session *s, uint64_t *counts, double *energy) {
  struct filter_ingest_stats st;
  int const r = filter_ingest_stats(&s->in, &st);
  if (r == 0) {
    counts[0] = st.blocks;
    counts[1] = st.samples;
    counts[2] = st.overranges;
    counts[3] = st.overrange_samples;
    counts[4] = st.since_over;
    memcpy(energy, &FENERGY(st), sizeof *energy);
  }
  return r;
}
/* the format numbers this build was compiled with: F32, CF32, CF32_CNRMF, CF32_FSCALE */
void rd_float_formats(int *out) {
  out[0] = FILTER_RAW_F32;
  out[1] = FILTER_RAW_CF32;
  out[2] = FILTER_RAW_CF32_CNRMF;
  out[3] = FILTER_RAW_CF32_FSCALE;
}
