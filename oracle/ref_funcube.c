/* oracle/ref_funcube.c -- drives the reference's OWN FUNcube sample loop (proc_funcube, funcube.c:194-310) for the I/Q
 * correction checks (tests/test_iq_correction_cpu.py, tests/test_gpu_iq_correction.py).
 *
 * TEST INFRASTRUCTURE, NOT PRODUCT.  The reference's src/funcube.c is #included unmodified from where it lies (never
 * copied), so its static proc_funcube is reachable.  PortAudio is a declaration-only header (stubs/portaudio.h):
 * Pa_ReadStream below hands over the caller's next block and, after the last one, sets the state to STOPPING, so
 * proc_funcube's loop runs on the calling thread and returns.  Its thread naming and real-time priority are no-ops here.
 * The master is the reference's own filter.c.  Compiled only into oracle/_ref/libka9qiqcorr.so (oracle/iqcorr.mk).
 */
#define _GNU_SOURCE 1
#include "misc.h"
#undef pthread_setname
#define pthread_setname(x) ((void)(x)) /* proc_funcube names its thread: not the oracle's to do */

#include "funcube.c"

static struct frontend Rf_frontend;
static struct sdrstate Rf_sdr;
/* the blocks proc_funcube reads, and what it left after each */
static int16_t const *Rf_words;
static int Rf_blocks, Rf_next, Rf_blocksize;
static float complex *Rf_floats;
static double *Rf_state;
static uint64_t *Rf_counts;
static double *Rf_if_power;
static float complex const *Rf_wptr;

/* what proc_funcube left after the block just processed (called at the next read, or after the loop) */
static void rf_collect(void) {
  int const b = Rf_next - 1;
  if (b < 0)
    return;
  memcpy(Rf_floats + (size_t)b * (size_t)Rf_blocksize, Rf_wptr, sizeof(float complex) * (size_t)Rf_blocksize);
  double const s[8] = {creal(Rf_sdr.DC), cimag(Rf_sdr.DC), Rf_sdr.sinphi, Rf_sdr.imbalance, 0, 0, 0, 0};
  memcpy(Rf_state + 8 * (size_t)b, s, sizeof s); /* the gains are proc_funcube's locals: not observable */
  Rf_counts[2 * b] = Rf_frontend.overranges;
  Rf_counts[2 * b + 1] = Rf_frontend.samp_since_over;
  Rf_if_power[b] = Rf_frontend.if_power;
}

PaError Pa_StartStream(PaStream *stream) { return paNoError; }
PaError Pa_StopStream(PaStream *stream) { return paNoError; }
const char *Pa_GetErrorText(PaError errorCode) { return "oracle"; }
PaError Pa_ReadStream(PaStream *stream, void *buffer, unsigned long frames) {
  rf_collect();
  memcpy(buffer, Rf_words + 2 * (size_t)Rf_next * frames, 2 * sizeof(int16_t) * frames);
  Rf_wptr = Rf_frontend.in.input_write_pointer.c;
  if (++Rf_next == Rf_blocks)
    atomic_store(&Rf_sdr.state, STOPPING); /* proc_funcube processes this block, then leaves its loop */
  return paNoError;
}

/* nblocks blocks of blocksize I/Q pairs (int16) through proc_funcube on a master of L, M (reference filter.c), with the
 * sdrstate funcube_setup leaves (calloc'd, scale).  Per block: the floats stored; DC (re, im), sinphi, imbalance (then
 * four zeros); overranges and samp_since_over; if_power. */
int rf_run(int16_t const *words, int nblocks, int blocksize, double scale, int L, int M, float complex *floats, double *state,
           uint64_t *counts, double *if_power) {
  memset(&Rf_frontend, 0, sizeof Rf_frontend);
  memset(&Rf_sdr, 0, sizeof Rf_sdr);
  N_worker_threads = 0; /* blocks run inline on the calling thread (filter.c:44) */
  if (create_filter_input(&Rf_frontend.in, L, M, COMPLEX) != 0)
    return -1;
  Rf_frontend.samprate = ADC_samprate;
  Rf_frontend.context = &Rf_sdr;
  Rf_sdr.frontend = &Rf_frontend;
  Rf_sdr.scale = scale;
  atomic_store(&Rf_sdr.state, RUNNING);
  Blocktime = (blocksize + 0.5) / ADC_samprate; /* funcube.c:207 truncates Blocktime * ADC_samprate to blocksize */
  Rf_words = words;
  Rf_blocks = nblocks;
  Rf_next = 0;
  Rf_blocksize = blocksize;
  Rf_floats = floats;
  Rf_state = state;
  Rf_counts = counts;
  Rf_if_power = if_power;
  proc_funcube(&Rf_sdr);
  rf_collect();
  delete_filter_input(&Rf_frontend.in);
  return 0;
}
