/* oracle/ref_siggen.c -- drives the reference's OWN signal generator loop (proc_sig_gen, sig_gen.c:211-372) for the
 * generator checks (tests/test_siggen_cpu.py, tests/test_gpu_siggen.py, tools/siggen_bench.py).
 *
 * TEST INFRASTRUCTURE, NOT PRODUCT.  The reference's src/sig_gen.c is #included unmodified from where it lies (never
 * copied), so its static proc_sig_gen runs here on a prepared sdrstate and frontend whose master is the reference's own
 * filter.c.  libsamplerate is a declaration-only header (stubs/samplerate.h); only the CW loop runs.  The loop paces
 * itself by gps_time_ns and nanosleep: both are renamed here to stand-ins that script each iteration's blocksize and
 * scale and stop the loop after the last one.  With samprate = 1e9 a clock step of n nanoseconds is a blocksize of n.
 * The thread naming and real-time priority calls are no-ops.  Compiled only into oracle/_ref/libka9qsiggen.so
 * (oracle/siggen.mk).
 */
#define _GNU_SOURCE 1
#include <stdint.h>
#include <time.h>

#include "misc.h"
#undef pthread_setname
#define pthread_setname(x) ((void)(x)) /* proc_sig_gen names its thread: not the oracle's to do */
#define gps_time_ns rs_gps_time_ns
#define nanosleep rs_nanosleep
static int64_t rs_gps_time_ns(void);
static int rs_nanosleep(struct timespec const *req, struct timespec *rem);

#include "sig_gen.c"

#undef gps_time_ns
#undef nanosleep

static struct frontend Rs_frontend;
static struct sdrstate Rs_sdr;
static int const *Rs_sizes; /* the scripted blocksize of each iteration */
static double const *Rs_scales;
static int Rs_n, Rs_k;
static bool Rs_started;
static int64_t Rs_snap; /* proc_sig_gen's timesnap, tracked */
static void *Rs_wptr;   /* where the current iteration writes */
static float *Rs_out;   /* every float the loop stored, in order */
static double *Rs_energy;
static size_t Rs_pos;
static double Rs_cpu; /* thread CPU seconds inside the iterations */
static struct timespec Rs_t0;

static double rs_now(void) {
  struct timespec t;
  clock_gettime(CLOCK_THREAD_CPUTIME_ID, &t);
  return (double)t.tv_sec + 1e-9 * (double)t.tv_nsec;
}

/* the first call sets timesnap one Blocktime back (sig_gen.c:266); each later one starts an iteration: the interval
 * since timesnap is the scripted blocksize, and timesnap moves on by exactly that much (sig_gen.c:279-280) */
static int64_t rs_gps_time_ns(void) {
  if (!Rs_started) {
    Rs_started = true;
    Rs_snap = -lrint(Blocktime * BILLION);
    return 0;
  }
  Rs_sdr.scale = Rs_scales[Rs_k];
  Rs_frontend.if_power = 0; /* with Power_alpha 1, if_power becomes in_energy / blocksize */
  Rs_wptr = Rs_frontend.isreal ? (void *)Rs_frontend.in.input_write_pointer.r : (void *)Rs_frontend.in.input_write_pointer.c;
  Rs_snap += Rs_sizes[Rs_k];
  clock_gettime(CLOCK_THREAD_CPUTIME_ID, &Rs_t0);
  return Rs_snap;
}
/* the end of an iteration: take its floats and in_energy; stop the loop after the last one */
static int rs_nanosleep(struct timespec const *req, struct timespec *rem) {
  (void)req;
  (void)rem;
  Rs_cpu += rs_now() - ((double)Rs_t0.tv_sec + 1e-9 * (double)Rs_t0.tv_nsec);
  int const n = Rs_sizes[Rs_k];
  size_t const c = Rs_frontend.isreal ? 1 : 2;
  if (Rs_out)
    memcpy(Rs_out + Rs_pos * c, Rs_wptr, sizeof(float) * c * (size_t)n); /* the mirrored ring keeps them contiguous */
  if (Rs_energy)
    Rs_energy[Rs_k] = n ? Rs_frontend.if_power * n : 0.0;
  Rs_pos += (size_t)n;
  if (++Rs_k == Rs_n)
    atomic_store(&Rs_sdr.state, STOPPING);
  return 0;
}

static void *rs_thread(void *arg) { return proc_sig_gen(arg); }

/* One run of proc_sig_gen's CW loop from rand_init, on a master of L, M on the reference's filter.c: n iterations of
 * sizes[i] samples (REAL) or pairs (COMPLEX) with sdr->scale = scales[i].  freq = carrier / 1e9 (the sample rate).
 * out: the floats stored (sum of sizes, times 2 for COMPLEX), energy: each iteration's in_energy (either may be NULL).
 * *cpu (if not NULL): the thread CPU seconds spent in the iterations.  Returns 0, or -1 with a message. */
int rs_run(int isreal, int L, int M, double carrier, double amplitude, double noise, int const *sizes, double const *scales,
           int n, float *out, double *energy, double *cpu) {
  memset(&Rs_frontend, 0, sizeof Rs_frontend);
  memset(&Rs_sdr, 0, sizeof Rs_sdr);
  N_worker_threads = 0; /* blocks run inline on the loop's thread (filter.c:44) */
  if (n < 1 || create_filter_input(&Rs_frontend.in, L, M, isreal ? REAL : COMPLEX) != 0) {
    fprintf(stderr, "rs_run: create_filter_input(L=%d, M=%d) failed\n", L, M);
    return -1;
  }
  Blocktime = 1.0; /* output_size (sig_gen.c:232) then caps a blocksize at 1.5e9 */
  Power_alpha = 1.0;
  Rs_frontend.samprate = 1e9;
  Rs_frontend.isreal = isreal != 0;
  Rs_frontend.frequency = 0;
  Rs_frontend.context = &Rs_sdr;
  Rs_sdr.frontend = &Rs_frontend;
  Rs_sdr.carrier = carrier;
  Rs_sdr.amplitude = amplitude;
  Rs_sdr.noise = noise;
  Rs_sdr.modulation = CW;
  Rs_sdr.state = RUNNING;
  Rs_sizes = sizes;
  Rs_scales = scales;
  Rs_n = n;
  Rs_k = 0;
  Rs_started = false;
  Rs_out = out;
  Rs_energy = energy;
  Rs_pos = 0;
  Rs_cpu = 0;
  pthread_t t; /* a thread of its own: rand_init seeds the thread-local generator once per thread (gauss.c:95-101) */
  int const rc = pthread_create(&t, NULL, rs_thread, &Rs_sdr) == 0 && pthread_join(t, NULL) == 0 ? 0 : -1;
  if (rc != 0)
    fprintf(stderr, "rs_run: the loop's thread could not run\n");
  delete_filter_input(&Rs_frontend.in);
  if (cpu)
    *cpu = Rs_cpu;
  return rc;
}

/* the reference's xoshiro256** state after `steps` plain steps from xoshiro256ss_seed(seed) (gauss.c:32-61) */
void rs_state_after(uint64_t seed, uint64_t steps, uint64_t *out) {
  xoshiro256ss_state st;
  xoshiro256ss_seed(&st, seed);
  for (uint64_t i = 0; i < steps; i++)
    (void)xoshiro256ss_next(&st);
  memcpy(out, st.s, sizeof st.s);
}

/* the step phasor set_osc(f) stores (osc.c:37-40): out = {re, im} */
void rs_step_phasor(double f, double *out) {
  struct osc o = {0};
  set_osc(&o, f, 0.0);
  out[0] = creal(o.phasor_step);
  out[1] = cimag(o.phasor_step);
}
