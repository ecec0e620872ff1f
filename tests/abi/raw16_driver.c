/* tests/abi/raw16_driver.c -- raw 16-bit ingest through the filter.h surface, for tests/test_gpu_raw16_ingest.py and
 * tools/raw16_ingest_bench.py: raw_driver.c's sessions (write_rawfilter with FILTER_RAW_S16 / U16 / SC16Q11, floats,
 * channels, statistics, the wideband analyzer), plus SDRplay's separate I and Q arrays (write_rawfilter_planar).
 *
 * Compiled twice: against include/ka9q_gpu_filter.h (tests/abi/_build/raw16_driver.so, by build()) and against the
 * reference's own src/filter.h (oracle/_ref/raw16_driver_refhdr.so, oracle/raw16.mk, where the reference sources exist).
 * The second declares the extensions itself, as a patched radiod would. */
#include "raw_driver.c"

#ifndef KA9Q_GPU_FILTER_H
enum { FILTER_RAW_S16 = 6, FILTER_RAW_U16 = 7, FILTER_RAW_SC16Q11 = 8 };
int write_rawfilter_planar(struct filter_in *master, int16_t const *i, int16_t const *q, int n, double scale);
#endif

int rd_write_planar(struct rd_session *s, int16_t const *i, int16_t const *q, int n, double scale) {
  return write_rawfilter_planar(&s->in, i, q, n, scale);
}
/* the format numbers this build was compiled with: S16, U16, SC16Q11 */
void rd_raw16_formats(int *out) {
  out[0] = FILTER_RAW_S16;
  out[1] = FILTER_RAW_U16;
  out[2] = FILTER_RAW_SC16Q11;
}
