/* oracle/ref_hackrf.c -- drives the reference's OWN HackRF sample callback (hackrf.c:297-375) for the I/Q correction
 * checks (tests/test_iq_correction_cpu.py, tests/test_gpu_iq_correction.py).
 *
 * TEST INFRASTRUCTURE, NOT PRODUCT.  The reference's src/hackrf.c is #included unmodified from where it lies (never
 * copied), so its static rx_callback is reachable here on a prepared sdrstate and frontend whose master is the
 * reference's own filter.c.  libhackrf is a declaration-only header (stubs/libhackrf/hackrf.h).  The callback's
 * thread naming, real-time priority and core pinning are no-ops here: the oracle never changes how the host schedules
 * it.  Compiled only into oracle/_ref/libka9qiqcorr.so (oracle/iqcorr.mk).
 */
#define _GNU_SOURCE 1
#include "misc.h"
#undef pthread_setname
#define pthread_setname(x) ((void)(x)) /* rx_callback names its thread once: not the oracle's to do */

#include "hackrf.c"

static struct frontend Rh_frontend;
static struct sdrstate Rh_sdr;

/* A master of L, M on the reference's filter.c and the sdrstate hackrf_setup / hackrf_startup leave (hackrf.c:100,
 * :223, :239-241): calloc'd, then secphi = gain_i = gain_q = 1 and the sample scale. */
int rh_open(double samprate, int L, int M, double scale) {
  memset(&Rh_frontend, 0, sizeof Rh_frontend);
  memset(&Rh_sdr, 0, sizeof Rh_sdr);
  N_worker_threads = 0; /* blocks run inline on the calling thread (filter.c:44) */
  if (create_filter_input(&Rh_frontend.in, L, M, COMPLEX) != 0)
    return -1;
  Rh_frontend.samprate = samprate;
  Rh_frontend.context = &Rh_sdr;
  Rh_sdr.frontend = &Rh_frontend;
  Rh_sdr.secphi = 1;
  Rh_sdr.gain_i = 1;
  Rh_sdr.gain_q = 1;
  Rh_sdr.scale = scale;
  return 0;
}
void rh_set_scale(double scale) { Rh_sdr.scale = scale; }

/* One USB transfer of `bytes` signed bytes through rx_callback.  floats: the bytes/2 complex floats it stored; state:
 * DC (re, im), sinphi, imbalance, gain_i, gain_q, secphi, tanphi after the transfer; clips and if_power as it left them. */
int rh_transfer(uint8_t const *buf, int bytes, float complex *floats, double *state, int *clips, double *if_power) {
  uint8_t *copy = malloc(bytes > 0 ? (size_t)bytes : 1);
  memcpy(copy, buf, (size_t)bytes);
  float complex const *wptr = Rh_frontend.in.input_write_pointer.c;
  hackrf_transfer t = {.buffer = copy, .buffer_length = bytes, .valid_length = bytes, .rx_ctx = &Rh_sdr};
  int const r = rx_callback(&t);
  free(copy);
  memcpy(floats, wptr, sizeof(float complex) * (size_t)(bytes / 2)); /* the mirrored ring keeps them contiguous */
  double const s[8] = {creal(Rh_sdr.DC), cimag(Rh_sdr.DC), Rh_sdr.sinphi, Rh_sdr.imbalance,
                       Rh_sdr.gain_i,    Rh_sdr.gain_q,    Rh_sdr.secphi, Rh_sdr.tanphi};
  memcpy(state, s, sizeof s);
  *clips = Rh_sdr.clips;
  *if_power = Rh_frontend.if_power;
  return r;
}

/* host CPU time of n calls of rx_callback on the same transfer, in seconds (tools/iq_correction_bench.py) */
double rh_time(uint8_t const *buf, int bytes, int n) {
  uint8_t *copy = malloc((size_t)bytes);
  memcpy(copy, buf, (size_t)bytes);
  hackrf_transfer t = {.buffer = copy, .buffer_length = bytes, .valid_length = bytes, .rx_ctx = &Rh_sdr};
  struct timespec a, b;
  clock_gettime(CLOCK_THREAD_CPUTIME_ID, &a);
  for (int i = 0; i < n; i++)
    rx_callback(&t);
  clock_gettime(CLOCK_THREAD_CPUTIME_ID, &b);
  free(copy);
  return (double)(b.tv_sec - a.tv_sec) + 1e-9 * (double)(b.tv_nsec - a.tv_nsec);
}

void rh_close(void) { delete_filter_input(&Rh_frontend.in); }
