/* oracle/ref_siggen_mod.c -- drives the reference's OWN signal generator loop (proc_sig_gen, sig_gen.c:211-372) through
 * its AM and DSB branches (sig_gen.c:297-314, :327-344) for the modulated generator checks (tests/test_siggen_mod_cpu.py,
 * tests/test_gpu_siggen_mod.py, tools/siggen_mod_bench.py).
 *
 * TEST INFRASTRUCTURE, NOT PRODUCT.  As oracle/ref_siggen.c does for the CW loop, the reference's src/sig_gen.c is
 * #included unmodified from where it lies (never copied) and its static proc_sig_gen runs on a prepared sdrstate and
 * frontend whose master is the reference's own filter.c.  The calls the AM / DSB set-up and loop make outside the
 * reference are renamed here to stand-ins:
 *   gps_time_ns, nanosleep   script each iteration's blocksize and scale and stop the loop after the last one (with
 *                            samprate = 1e9 a clock step of n nanoseconds is a blocksize of n);
 *   popen, pclose            open and close a dummy stream (the audio source is never read);
 *   src_callback_new         returns a dummy converter state;
 *   src_callback_read        copies the iteration's scripted number r <= blocksize of scripted envelope floats: what
 *                            libsamplerate would have produced;
 *   src_error, src_delete    no error; nothing to free.
 * The thread naming and real-time priority calls are no-ops.  Compiled only into oracle/_ref/libka9qsiggenmod.so
 * (oracle/siggen_mod.mk).
 */
#define _GNU_SOURCE 1
#include <stdint.h>
#include <stdio.h>
#include <time.h>

#include "misc.h"
#undef pthread_setname
#define pthread_setname(x) ((void)(x))
#define gps_time_ns rm_gps_time_ns
#define nanosleep rm_nanosleep
#define popen rm_popen
#define pclose rm_pclose
#define src_callback_new rm_src_callback_new
#define src_callback_read rm_src_callback_read
#define src_error rm_src_error
#define src_delete rm_src_delete
static int64_t rm_gps_time_ns(void);
static int rm_nanosleep(struct timespec const *req, struct timespec *rem);
static FILE *rm_popen(char const *cmd, char const *mode);
static int rm_pclose(FILE *f);

#include "sig_gen.c"

#undef gps_time_ns
#undef nanosleep
#undef popen
#undef pclose

static struct frontend Rm_frontend;
static struct sdrstate Rm_sdr;
static int const *Rm_sizes;  /* the scripted blocksize of each iteration */
static int const *Rm_reads;  /* the scripted src_callback_read count of each iteration */
static double const *Rm_scales;
static float const *Rm_env;  /* the scripted envelope, Rm_reads[k] floats per iteration */
static size_t Rm_env_pos;
static int Rm_n, Rm_k;
static long Rm_r;            /* this iteration's count, what the loop took as its blocksize */
static bool Rm_started;
static int64_t Rm_snap;
static void *Rm_wptr;
static float *Rm_out;
static double *Rm_energy;
static size_t Rm_pos;
static double Rm_cpu;
static struct timespec Rm_t0;
static char Rm_stream; /* the dummy audio source */
static char Rm_source[] = "scripted envelope";
static char Rm_state;  /* the dummy converter state */

static double rm_now(void) {
  struct timespec t;
  clock_gettime(CLOCK_THREAD_CPUTIME_ID, &t);
  return (double)t.tv_sec + 1e-9 * (double)t.tv_nsec;
}

static FILE *rm_popen(char const *cmd, char const *mode) {
  (void)cmd;
  (void)mode;
  return (FILE *)&Rm_stream;
}
static int rm_pclose(FILE *f) { return f == (FILE *)&Rm_stream ? 0 : -1; }
SRC_STATE *rm_src_callback_new(src_callback_t func, int converter_type, int channels, int *error, void *cb_data) {
  (void)func;
  (void)converter_type;
  (void)channels;
  (void)cb_data;
  *error = 0;
  return (SRC_STATE *)&Rm_state;
}
long rm_src_callback_read(SRC_STATE *state, double src_ratio, long frames, float *data) {
  (void)state;
  (void)src_ratio;
  long r = Rm_reads[Rm_k];
  if (r > frames)
    r = frames;
  memcpy(data, Rm_env + Rm_env_pos, sizeof(float) * (size_t)r);
  Rm_env_pos += (size_t)r;
  Rm_r = r;
  return r;
}
int rm_src_error(SRC_STATE *state) {
  (void)state;
  return 0;
}
SRC_STATE *rm_src_delete(SRC_STATE *state) {
  (void)state;
  return NULL;
}

/* the first call sets timesnap one Blocktime back (sig_gen.c:266); each later one starts an iteration: the interval
 * since timesnap is the scripted blocksize, and timesnap moves on by exactly that much (sig_gen.c:279-280) */
static int64_t rm_gps_time_ns(void) {
  if (!Rm_started) {
    Rm_started = true;
    Rm_snap = -lrint(Blocktime * BILLION);
    return 0;
  }
  Rm_sdr.scale = Rm_scales[Rm_k];
  Rm_frontend.if_power = 0; /* with Power_alpha 1, if_power becomes in_energy / blocksize */
  Rm_wptr = Rm_frontend.isreal ? (void *)Rm_frontend.in.input_write_pointer.r : (void *)Rm_frontend.in.input_write_pointer.c;
  Rm_r = 0;
  Rm_snap += Rm_sizes[Rm_k];
  clock_gettime(CLOCK_THREAD_CPUTIME_ID, &Rm_t0);
  return Rm_snap;
}
/* the end of an iteration: take the r floats (pairs) it stored and its in_energy; stop the loop after the last one */
static int rm_nanosleep(struct timespec const *req, struct timespec *rem) {
  (void)req;
  (void)rem;
  Rm_cpu += rm_now() - ((double)Rm_t0.tv_sec + 1e-9 * (double)Rm_t0.tv_nsec);
  size_t const c = Rm_frontend.isreal ? 1 : 2;
  if (Rm_out)
    memcpy(Rm_out + Rm_pos * c, Rm_wptr, sizeof(float) * c * (size_t)Rm_r); /* the mirrored ring keeps them contiguous */
  if (Rm_energy)
    Rm_energy[Rm_k] = Rm_r ? Rm_frontend.if_power * (double)Rm_r : 0.0;
  Rm_pos += (size_t)Rm_r;
  if (++Rm_k == Rm_n)
    atomic_store(&Rm_sdr.state, STOPPING);
  return 0;
}

static void *rm_thread(void *arg) { return proc_sig_gen(arg); }

/* One run of proc_sig_gen's AM (am != 0) or DSB loop from rand_init, on a master of L, M on the reference's filter.c:
 * n iterations of blocksize sizes[i], of which src_callback_read delivers reads[i] <= sizes[i] samples (REAL) or pairs
 * (COMPLEX) of the envelope env (sum of reads floats), with sdr->scale = scales[i].  freq = carrier / 1e9.  out: the
 * floats stored (sum of reads, times 2 for COMPLEX), energy: each iteration's in_energy (either may be NULL).  *cpu (if
 * not NULL): the thread CPU seconds spent in the iterations, the stand-in's copy of the envelope included.  Returns 0,
 * or -1 with a message. */
int rs_run_mod(int isreal, int L, int M, double carrier, double amplitude, double noise, int am, int const *sizes,
               int const *reads, double const *scales, int n, float const *env, float *out, double *energy, double *cpu) {
  memset(&Rm_frontend, 0, sizeof Rm_frontend);
  memset(&Rm_sdr, 0, sizeof Rm_sdr);
  memset(&Input_state, 0, sizeof Input_state); /* is->source survives pclose (sig_gen.c:365-366) */
  N_worker_threads = 0; /* blocks run inline on the loop's thread (filter.c:44) */
  for (int k = 0; k < n; k++)
    if (reads[k] < 0 || reads[k] > sizes[k]) {
      fprintf(stderr, "rs_run_mod: iteration %d reads %d of %d\n", k, reads[k], sizes[k]);
      return -1;
    }
  if (n < 1 || create_filter_input(&Rm_frontend.in, L, M, isreal ? REAL : COMPLEX) != 0) {
    fprintf(stderr, "rs_run_mod: create_filter_input(L=%d, M=%d) failed\n", L, M);
    return -1;
  }
  /* output_size = 1.5 Blocktime samprate (sig_gen.c:232) caps a blocksize and sizes the loop's dac_modulation buffer,
   * which the loop never frees: 1.5 times the largest scripted blocksize */
  int most = 1;
  for (int k = 0; k < n; k++)
    most = sizes[k] > most ? sizes[k] : most;
  Blocktime = 1e-9 * most;
  Power_alpha = 1.0;
  Rm_frontend.samprate = 1e9;
  Rm_frontend.isreal = isreal != 0;
  Rm_frontend.frequency = 0;
  Rm_frontend.context = &Rm_sdr;
  Rm_sdr.frontend = &Rm_frontend;
  Rm_sdr.carrier = carrier;
  Rm_sdr.amplitude = amplitude;
  Rm_sdr.noise = noise;
  Rm_sdr.modulation = am ? AM : DSB;
  Rm_sdr.source = Rm_source;
  Rm_sdr.state = RUNNING;
  Rm_sizes = sizes;
  Rm_reads = reads;
  Rm_scales = scales;
  Rm_env = env;
  Rm_env_pos = 0;
  Rm_n = n;
  Rm_k = 0;
  Rm_started = false;
  Rm_out = out;
  Rm_energy = energy;
  Rm_pos = 0;
  Rm_cpu = 0;
  pthread_t t; /* a thread of its own: rand_init seeds the thread-local generator once per thread (gauss.c:95-101) */
  int rc = pthread_create(&t, NULL, rm_thread, &Rm_sdr) == 0 && pthread_join(t, NULL) == 0 ? 0 : -1;
  if (rc != 0)
    fprintf(stderr, "rs_run_mod: the loop's thread could not run\n");
  else if (Rm_k != n || Rm_sdr.modulation != (am ? AM : DSB)) {
    fprintf(stderr, "rs_run_mod: the loop ran %d of %d iterations\n", Rm_k, n);
    rc = -1;
  }
  delete_filter_input(&Rm_frontend.in);
  if (cpu)
    *cpu = Rm_cpu;
  return rc;
}
