/* include/ka9q_gpu.h -- low-level C-ABI of libka9qgpu.so: the H100 overlap-save channelizer.
 *
 * Plain pointers and sizes only; no CUDA or torch types in the signatures (streams are passed
 * as void* holding a cudaStream_t, device buffers as void*).  The reference-compatible
 * filter.h surface (include/ka9q_gpu_filter.h) is implemented on top of these calls; bench.py
 * and the multi-GPU harness call them directly so that device buffers owned by the caller
 * (e.g. torch tensors that an NCCL broadcast fills) can be used in place.
 *
 * Every entry point names the reference code it replaces (paths relative to the ka9q-radio
 * tree, commit 4e0033b4).  All functions return 0 on success, -1 on error (the reference's
 * convention, filter.h:99-118) unless stated; kgpu_last_error() gives the text.
 * There is NO CPU fallback: if no sm_90 device is usable the calls fail.
 */
#ifndef KA9Q_GPU_H
#define KA9Q_GPU_H 1
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

enum kgpu_type { KGPU_COMPLEX = 1, KGPU_REAL = 2 }; /* same values as enum filtertype, filter.h:29-34 */
enum kgpu_format {
  KGPU_FMT_F32 = 0, /* float samples (REAL master) or float I/Q pairs (COMPLEX master): what drivers
                       leave in the ring today (rx888.c:800-809, sig_gen.c:290-296) */
  KGPU_FMT_I16 = 1  /* raw int16 samples / int16 I/Q pairs: the fused ingest (rx888.c:753-767) */
};
enum kgpu_chan_flags {
  KGPU_CHAN_ISB = 1, /* filter_out.isb, filter.c:895-909 */
  KGPU_CHAN_BEAM = 4 /* filter_out.beam on a COMPLEX master, filter.c:756-775; weights: kgpu_bank_set_weights */
  /* 2 (REAL output) and 8 (oscillator) are owned by kgpu_bank_define_ex / kgpu_bank_set_osc */
};

typedef struct kgpu_master kgpu_master; /* geometry + plans of one struct filter_in */
typedef struct kgpu_bank kgpu_bank;     /* a batch of struct filter_out sharing one master */

struct kgpu_ingest_stats { /* per block, only for KGPU_FMT_I16: rx888.c:759-762 */
  unsigned long long energy; /* sum of x*x over the L new samples */
  unsigned int clips;        /* |x| > 32766 */
  unsigned int pad;
};

const char *kgpu_last_error(void);
/* Number of this library's own kernels launched by the calling process so far (bench.py's
 * "gpu_launches" claim is read from here, not estimated). */
unsigned long long kgpu_launch_count(void);
/* Per-launch profiling: when enabled every kernel launch is bracketed by CUDA events on its own
 * stream; totals per kernel kind (index < kgpu_profile_kernels()) are read back after a sync. */
int kgpu_profile_enable(int on);
int kgpu_profile_reset(void);
int kgpu_profile_kernels(void);
const char *kgpu_profile_name(int kernel);
int kgpu_profile_get(int kernel, double *total_ms, long *count);
int kgpu_device_count(void);
int kgpu_set_device(int device);

/* ---- master: replaces create_filter_input's planning (filter.c:186-269) ------------------- */
/* L new samples per block, impulse length M, N = L+M-1 (radio.c:582-587).  REAL needs even N. */
kgpu_master *kgpu_master_create(int L, int M, int in_type);
/* Same, for complex transform lengths Nc (N for COMPLEX, N/2 for REAL) whose prime factors are 2, 3, 5, 7, 11, 13,
 * 17, 19 and 23, e.g. the AirspyHF+ at 912 kS/s (N = 22800 = 2^4 3 5^2 19); the reference transforms any N
 * (filter.c:201).  Where Nc has factors 2, 3, 5, 7 only it is kgpu_master_create: the same kernels, plans and
 * kgpu_master_describe string.  Otherwise the master runs the extended generic pair fwd_cols_ext + fwd_rows_ext on two
 * column plans of its own (radices 2 .. 25 and the five primes), freed by kgpu_master_destroy; kgpu_use_static_kernels
 * has no effect on it.  Fails for a prime factor >= 29, or when Nc has no split n1 x n2 into plannable factors of at
 * most 4096 points, or when that split does not fit shared memory. */
kgpu_master *kgpu_master_create_ex(int L, int M, int in_type);
/* Same, for any transform length, as the reference plans (filter.c:201), e.g. an RX888 at 62 MS/s (REAL, N = 1550000,
 * Nc = 775000 = 2^3 5^5 31) or a COMPLEX front end at 2.9 MS/s (N = 72500 = 2^2 5^4 29).  Where kgpu_master_create_ex
 * succeeds it returns exactly that master.  Otherwise it builds a Bluestein transform: the window times the chirp
 * exp(-i pi n^2 / Nc), zero-padded to the smallest P >= 2 Nc - 1 with factors 2, 3, 5, 7 whose split the forward pair
 * runs, two forward passes of an internal COMPLEX master of length P around the product with the chirp's transform
 * (computed in double on the host), then the output chirp and, for REAL masters, the real split.  The spectrum layout,
 * int16 ingest, statistics and every other master call are those of any master.  The master owns scratch of at most
 * about 128 MB per buffer; launches of more blocks run in chunks.  Fails for REAL input with odd L or odd N, and when
 * P would exceed 3500 x 3500 (Nc > 6125000). */
kgpu_master *kgpu_master_create_any(int L, int M, int in_type);
/* Pure host code: the master kgpu_master_create_any would build (0 kgpu_master_create's, 1 kgpu_master_create_ex's
 * extended pair, 2 Bluestein; -1 when it would fail) and, if buf is not NULL, the string kgpu_master_describe would
 * print for it. */
int kgpu_master_plan(int L, int M, int in_type, char *buf, int buflen);
void kgpu_master_destroy(kgpu_master *m);
int kgpu_master_points(kgpu_master const *m);       /* N */
int kgpu_master_bins(kgpu_master const *m);         /* REAL: N/2+1, COMPLEX: N (filter.c:197) */
long kgpu_master_spec_stride(kgpu_master const *m); /* float2 elements between consecutive block spectra */
/* Plan description for logs/DESIGN.md: "n1 x n2, radices ..."; a Bluestein master of kgpu_master_create_any:
 * "N=... real|complex, bluestein P=...: <the internal master's transform and kernels> around bluestein_in_kernel, ..." */
int kgpu_master_describe(kgpu_master const *m, char *buf, int buflen);

/* Forward transform of `nblocks` consecutive overlap-save windows (replaces run_fft's
 * fftwf_execute_dft_r2c / fftwf_execute_dft, filter.c:505-508, fused with the int16->float
 * conversion rx888.c:753-767 when fmt == KGPU_FMT_I16).
 *   d_in   device pointer to the first sample of block 0's WINDOW, i.e. M-1 samples before block
 *          0's first new sample; window b starts b*L samples later (overlap-save, filter.c:631-635).
 *          Units: float / int16 for REAL masters, (re,im) pairs for COMPLEX masters.
 *   scale  multiplies int16 samples (rx888.c:765); ignored for float input.
 *   d_spec nblocks * spec_stride float2; bins 0..bins-1 of each block, unnormalised, sign -1.
 *   d_stats NULL or nblocks kgpu_ingest_stats (int16 only), zeroed by the call. */
int kgpu_forward(kgpu_master *m, const void *d_in, int fmt, float scale, int derandomize, int nblocks,
                 void *d_spec, void *d_stats, void *stream);

/* Airspy R2 / HydraSDR packed 12-bit ingest (replaces airspy_unpack / airspy_unpack_avx2, airspy-unpack.c:17-130, called at
 * airspy.c:416-419): `sampcount` (multiple of 8) offset-binary samples, 8 per three 32-bit words, -> int16 (s - 2048) at
 * d_i16 (16-byte aligned), ready for kgpu_forward(..., KGPU_FMT_I16, scale, ...) which applies `scale * (float)x`.
 * d_stats: NULL or ONE kgpu_ingest_stats receiving the energy and the clip count (x == 2047 || x <= -2047). */
int kgpu_unpack_airspy12(const void *d_packed, long sampcount, void *d_i16, void *d_stats, void *stream);

/* 8-bit, 16-bit and float sample words of kgpu_unpack8.  Kept apart from kgpu_format: kgpu_forward does not read them. */
enum kgpu_raw8 {
  KGPU_RAW_U8 = 1,  /* excess-128 bytes: RTL-SDR (rtlsdr.c:316-343), HydraSDR UINT8_REAL / UINT8_IQ (hydrasdr.c:759-775, :793-811) */
  KGPU_RAW_S8 = 2,  /* signed bytes: HydraSDR INT8_REAL / INT8_IQ (hydrasdr.c:776-791, :812-830) */
  KGPU_RAW_S16 = 3, /* int16: HydraSDR INT16_REAL / INT16_IQ (hydrasdr.c:700-716, :729-747), SDRplay (sdrplay.c:1238-1242) */
  KGPU_RAW_U16 = 4, /* offset-binary uint16, x = w - 32768, REAL only: HydraSDR UINT16_REAL (hydrasdr.c:681-699) */
  KGPU_RAW_SC16Q11 = 5, /* bladeRF SC16_Q11, COMPLEX only: x = bits 0-11 sign-extended from bit 11 (bladerf.c:226-235) */
  /* floats (4-byte aligned).  Energy per block: the sum of the loop's terms as its source writes them, in double in a fixed order. */
  KGPU_RAW_F32 = 6,         /* REAL only: (float)(scale * (double)x), terms x * x in float (hydrasdr.c:717-728) */
  KGPU_RAW_CF32 = 7,        /* COMPLEX only: (float)(scale * (double)x), terms cnrm in double (hydrasdr.c:748-758) */
  KGPU_RAW_CF32_CNRMF = 8,  /* COMPLEX only: (float)(scale * (double)x), terms cnrmf in float (airspyhf.c:313-318) */
  KGPU_RAW_CF32_FSCALE = 9  /* COMPLEX only: x * (float)scale in float, terms x * x in float (fobos.c:410-420) */
};
/* A/D statistics of one block's L new samples (never its M-1 history samples).  A sample is one value (REAL) or one I/Q
 * pair (COMPLEX). */
struct kgpu_block_stats {
  union {
    unsigned long long energy; /* integer formats: sum of x*x over every component */
    double fenergy;            /* float formats: the sum of the driver loop's energy terms, non-finite if one is */
  };
  unsigned int overs;        /* components at the format's limits (float formats: 0) */
  unsigned int over_samples; /* samples with at least one component at the limits (float formats: 0) */
};
/* A front end's change of scale between two writes: from absolute sample `at` on (0 = the first sample a master was
 * written), samples take `scale`.  The conversions that take a device array of n of them, sorted by `at`, give each
 * sample the scale of the last change at or before it, or their `scale` argument before the first. */
struct kgpu_scale_change {
  long long at;
  double scale;
};
/* 8-bit, 16-bit and float ingest (replaces the conversion loops cited at kgpu_raw8): the words of an overlap-save launch
 * -- `history` samples, then nblocks blocks of L new samples, laid out as kgpu_forward's d_in (16-bit words 2-byte
 * aligned, floats 4-byte aligned) -- to floats at d_out (4-byte aligned), each (float)(scale * (double)x) with x the
 * word's integer as kgpu_raw8 gives it, or the float formats' own rule, bitwise what the drivers' loops store; then
 * kgpu_forward(..., KGPU_FMT_F32, ...) reads d_out.  d_chg: NULL, or nchg scale changes, the first history sample being
 * absolute sample a0.  d_stats: NULL or nblocks kgpu_block_stats, zeroed by the call; at the limits: x >= 127 or x <= -128
 * (U8, S8), x >= 32767 or x <= -32768 (S16, U16), x == 2047 or x == -2048 (SC16Q11); the float formats fill fenergy.
 * nblocks may be 0 (conversion only: history samples). */
int kgpu_unpack8(const void *d_raw, int fmt, int in_type, long history, long L, int nblocks, double scale,
                 const struct kgpu_scale_change *d_chg, int nchg, long long a0, void *d_out, void *d_stats, void *stream);
/* int16 words laid out as kgpu_forward's KGPU_FMT_I16 d_in (count samples, the first being absolute sample a0) to floats
 * at d_out, each (float)x * (float)s after the optional derandomization (rx888.c:707-712, 764-765; airspy-unpack.c:124
 * for kgpu_unpack_airspy12's words), s its own scale: `scale` before the first of the nchg changes at d_chg, else the
 * last change at or before it.  For windows that hold more than one scale; kgpu_forward(..., KGPU_FMT_F32, ...) then
 * reads d_out. */
int kgpu_scale_i16(const void *d_in, int in_type, long count, long long a0, double scale, const struct kgpu_scale_change *d_chg,
                   int nchg, int derandomize, float *d_out, void *stream);
/* Per-block statistics of int16 words on the device, laid out as kgpu_forward's KGPU_FMT_I16 d_in (history samples, then
 * nblocks blocks of L): the RX888's words after the optional derandomization (rx888.c:707-712, 759-762; limit 32767, i.e.
 * x > 32766 or x < -32766), or kgpu_unpack_airspy12's output (airspy-unpack.c:121-124; limit 2047).  A component is at the
 * limits when |x| >= limit.  d_stats: nblocks kgpu_block_stats, zeroed by the call. */
int kgpu_block_stats_i16(const void *d_in, int in_type, long history, long L, int nblocks, int derandomize, int limit,
                         void *d_stats, void *stream);

/* I/Q correction of the HackRF and FUNcube drivers (hackrf.c:297-375, funcube.c:194-310) by exact moments; see
 * csrc/iq_correct.cuh.  Words of kgpu_iq_moments / kgpu_iq_apply, apart from kgpu_format and kgpu_raw8: */
enum kgpu_iq_fmt {
  KGPU_IQ_S8 = 1, /* HackRF: signed byte pairs, -128 clipped to -127 and counted (hackrf.c:325-332) */
  KGPU_IQ_S16 = 2 /* FUNcube: int16 pairs as they are, |x| >= 32767 counted (funcube.c:256-266) */
};
/* One write (one transfer) in the device's ring table of writes, indexed by write number modulo the table's capacity.
 * The caller fills first, n and scale and zeroes the rest (last_over = -1); kgpu_iq_moments accumulates the rest. */
struct kgpu_iq_write {
  long long first;     /* absolute index of its first I/Q pair (0 = the first pair ever written) */
  long long n;         /* I/Q pairs */
  double scale;        /* the scale of exactly these pairs */
  long long m[5];      /* sum i, sum q, sum i*i, sum q*q, sum i*q over the (clipped) words */
  long long overs;     /* components at the limits */
  long long last_over; /* absolute component index (2 * pair, + 1 for Q) of the last one, -1 if none */
};
/* The correction state: what a write is corrected with (the state its predecessor left), and what it leaves. */
struct kgpu_iq_state {
  double dc_i, dc_q, sinphi, imbalance, gain_i, gain_q, secphi, tanphi;
};
/* The state update's constants: kind 1 (HackRF) weighs gain and phase by gp * n and holds DC when n == 0
 * (hackrf.c:317, :359, :367-369); kind 2 (FUNcube) by gp = gainphase_alpha (funcube.c:209). */
struct kgpu_iq_params {
  int kind;
  double dc_alpha; /* per sample: 1e-7 (hackrf.c:34), 1e-6 (funcube.c:28) */
  double gp;
};
/* What a driver's state block computes for one write, and the state after it. */
struct kgpu_iq_record {
  long long seq;        /* write number */
  long long n, sum_i, sum_q;
  double i_energy, q_energy, dotprod; /* the drivers' sums over the write */
  long long overs;      /* HackRF clips, FUNcube components at the limits */
  long long since_over; /* components after the last one at the limits, -1 if none */
  struct kgpu_iq_state state;
};
/* Moments of I/Q pairs [a0, a0 + count) whose words start at d_raw, into the table entries of writes
 * [w_lo, w_lo + nw), which must hold every one of those pairs; a write may be summed over several calls. */
int kgpu_iq_moments(const void *d_raw, int fmt, long long a0, long count, struct kgpu_iq_write *d_tab, int cap,
                    long long w_lo, int nw, void *stream);
/* Writes [w_from, w_from + nw), complete, in order: d_coef[w % cap] is the state write w was corrected with; its record
 * goes to d_rec[w % cap] and the state after it to d_coef[(w + 1) % cap].  One thread. */
int kgpu_iq_scan(const struct kgpu_iq_write *d_tab, struct kgpu_iq_state *d_coef, int cap, long long w_from, int nw,
                 const struct kgpu_iq_params *params, struct kgpu_iq_record *d_rec, void *stream);
/* Corrected float I/Q of pairs [a0, a0 + count) to d_out (float2 per pair); pairs a >= 0 lie in writes [w_lo, w_lo + nw)
 * whose coefficients d_coef holds, pairs a < 0 precede the first write and are 0.0f. */
int kgpu_iq_apply(const void *d_raw, int fmt, long long a0, long count, const struct kgpu_iq_write *d_tab,
                  const struct kgpu_iq_state *d_coef, int cap, long long w_lo, int nw, void *d_out, void *stream);

/* sig_gen.c's CW, AM and DSB sources (proc_sig_gen, sig_gen.c:286-346) on the device; see csrc/siggen.cuh.  freq and rate are cycles
 * per sample and per sample^2, what set_osc receives (sig_gen.c:221-224); amplitude and noise sdr->amplitude and
 * sdr->noise; seed rand_init's xoshiro256** seed (1). */
struct kgpu_siggen_params {
  double freq, rate, amplitude, noise;
  uint64_t seed;
};
typedef struct kgpu_siggen kgpu_siggen;
/* A generator of REAL samples or COMPLEX pairs (pure host code; the device's jump matrices are copied at the first
 * generate); NULL and kgpu_last_error() on failure. */
kgpu_siggen *kgpu_siggen_create(int in_type, const struct kgpu_siggen_params *params);
void kgpu_siggen_destroy(kgpu_siggen *g);
/* The floats of samples [a0, a0 + count) at d_out (float per REAL sample, float2 per pair), each (float)(samp * scale) as
 * the driver's loop stores it, scale that of the sample (`scale` before the first of the nchg changes at d_chg, else the
 * last change at or before it); samples a < 0 precede the stream and are 0.0f (they must lie in the history).  The window is laid out as kgpu_forward's
 * d_in: `history` samples, then nblocks blocks of L (L >= 64 when nblocks > 0).  d_block_energy: NULL or nblocks
 * doubles, block j's sum of |samp|^2 (unscaled) over its L new samples.  Enqueued on `stream`; calls of one generator go
 * on one stream (its scratch is reused). */
int kgpu_siggen_generate(kgpu_siggen *g, long long a0, long count, double scale, const struct kgpu_scale_change *d_chg, int nchg,
                         void *d_out, double *d_block_energy, int nblocks, long L, long history, void *stream);
/* sig_gen.c's AM and DSB sources (sig_gen.c:297-314, :327-344): turns g into a generator of
 * (dc + m) * amplitude * carrier + noise * real_gauss, m the envelope libsamplerate produces at the front end's rate
 * (dc: AM 1.0, DSB 0.0; -1 for a non-finite dc).  One draw per sample, for COMPLEX pairs too (the noise is on I only),
 * so kgpu_siggen_state's draw d is then sample d.  A modulated generator is driven by kgpu_siggen_generate_mod only. */
int kgpu_siggen_set_modulation(kgpu_siggen *g, double dc);
/* kgpu_siggen_generate's window of a modulated generator: d_mod holds one envelope float per sample (REAL) or pair
 * (COMPLEX) of the window, laid out as d_out; the entries of samples before the stream are not read. */
int kgpu_siggen_generate_mod(kgpu_siggen *g, long long a0, long count, double scale, const struct kgpu_scale_change *d_chg,
                             int nchg, void *d_out, const float *d_mod, double *d_block_energy, int nblocks, long L,
                             long history, void *stream);
/* Pure host code: the xoshiro256** state before draw `draw` (out[4]), by GF(2) jumps from the seeded state; and the
 * step and sweep angles the carrier uses, in cycles as 128-bit fractions: out[4] = {F low, F high, R low, R high}. */
int kgpu_siggen_state(const kgpu_siggen *g, unsigned long long draw, uint64_t *out);
int kgpu_siggen_angles(const kgpu_siggen *g, uint64_t *out);

/* Notch EWMA on listed bins (apply_notch_filters, filter.c:464-474); list ends with bin 0. The state
 * lives in the master; blocks are processed in order. */
int kgpu_master_set_notches(kgpu_master *m, int const *bins, double const *alpha, int n);
int kgpu_apply_notches(kgpu_master *m, void *d_spec, int nblocks, void *stream);

/* ---- bank: replaces create_filter_output / set_filter / execute_filter_output ------------- */
kgpu_bank *kgpu_bank_create(kgpu_master *m, int capacity);
void kgpu_bank_destroy(kgpu_bank *b);
/* (Re)define channel idx: olen output samples per block (points = olen*N/L must be integral,
 * filter.c:312-316), COMPLEX output.  Returns points, or -1. */
int kgpu_bank_define(kgpu_bank *b, int idx, int olen);
/* Same with the output type of create_filter_output (filter.c:345-392): KGPU_COMPLEX, or KGPU_REAL for the
 * REAL-output slaves of wfm.c:76 / stereod.c:387 (slice filter.c:794-809, c2r inverse filter.c:386,914): olen FLOATS
 * per block, packed into (olen+1)/2 float2 of the output row.  points must be even for KGPU_REAL. */
int kgpu_bank_define_ex(kgpu_bank *b, int idx, int olen, int out_type);
/* Same, without the 7260-point limit of the two calls above (the reference plans any length, filter.c:298-415): at
 * most 7260 points it is kgpu_bank_define_ex; up to 28812 points (e.g. the 384 kHz wfm downconverter, wfm.c:37-38, at
 * 9600 or 15360 points) the channel runs a four-step inverse transform, one CTA per channel and block, provided
 * points splits into two factors of at most 4096 with factors 2, 3, 5, 7 (every such length in range does).  Every
 * other bank call treats such a channel like any other. */
int kgpu_bank_define_wide(kgpu_bank *b, int idx, int olen, int out_type);
/* Same, up to 1048576 points (e.g. the 1.536 MS/s websdr channels of an RX888 at 64.8 MS/s: 38400 points at overlap 5,
 * 368640 at 120 ms blocks): at most 28812 points it is kgpu_bank_define_wide; above that the channel runs a four-step
 * inverse transform in two kernels through a scratch buffer in global memory that the bank owns (grown on demand, at
 * most about 128 MB per stream), provided points has factors 2, 3, 5, 7 only (every such length in range then splits
 * into two factors of at most 4096).  Every other bank call treats such a channel like any other. */
int kgpu_bank_define_huge(kgpu_bank *b, int idx, int olen, int out_type);
/* Same, also for lengths of at most 28812 points whose prime factors reach 11, 13, 17, 19 or 23 (e.g. the 220 kHz and
 * 277.2 kHz channels of the HFDL bank: 5500 = 2^2 5^3 11 and 6930 = 2 3^2 5 7 11 points at 20 ms and overlap 5).  Where
 * points has factors 2, 3, 5, 7 only it is kgpu_bank_define_huge: the same result, kernels and messages.  Otherwise
 * the channel runs the generic channel kernel (up to 7260 points) or the four-step wide kernel on plans of its own,
 * which never take a slot of the plan registry.  Fails for a prime factor >= 29, and for a factor 11 .. 23 above 28812
 * points.  Every other bank call treats such a channel like any other. */
int kgpu_bank_define_ext(kgpu_bank *b, int idx, int olen, int out_type);
/* Same, for any point count up to 1048576, as the reference plans (filter.c:298-415), e.g. a 29 kHz (725 = 5^2 29
 * points), 62 kHz (1550 = 2 5^2 31) or 1.76 MS/s (44000 = 2^5 5^3 11) channel at 20 ms and overlap 5.  Where
 * kgpu_bank_define_ext succeeds it is that call: the same result, kernels and messages.  Otherwise (a prime factor >= 29,
 * or a factor 11 .. 23 above 28812 points) the channel runs a Bluestein transform: the conjugate slice x response times
 * the chirp exp(-i pi n^2 / points), zero-padded to the smallest P >= 2 points - 1 with factors 2, 3, 5, 7 whose split the
 * forward pair runs, two forward passes of an internal COMPLEX master of length P (one per bank and stream) around the
 * product with the chirp's transform (computed in double on the host once per length and process), then the output
 * chirp and 1/P.  The scratch is the bank's, at most about 128 MB per buffer and stream; launches of more channels and
 * blocks run in chunks.  Every other bank call treats such a channel like any other.  Fails above 1048576 points, and
 * for an odd point count with KGPU_REAL output. */
int kgpu_bank_define_any(kgpu_bank *b, int idx, int olen, int out_type);
/* Pure host code: the path kgpu_bank_define_any takes for a channel of `points` points (0 direct, 1 wide, 2 huge,
 * 3 extended, 4 Bluestein; -1 when it would fail) and, if buf is not NULL, a description: the radices or the split, the
 * kernels and, for Bluestein, P and the internal master's split. */
int kgpu_chan_plan(int points, int out_type, char *buf, int buflen);
/* set_filter (filter.c:968-1045): Kaiser-windowed sinc designed on the host in double, forward
 * transformed on the device.  low/high are fractions of the output rate. */
int kgpu_bank_set_filter(kgpu_bank *b, int idx, double low, double high, double kaiser_beta);
/* Same, synchronising only `stream` (on which the caller orders every launch that reads this bank) instead of the device. */
int kgpu_bank_set_filter_on(kgpu_bank *b, int idx, double low, double high, double kaiser_beta, void *stream);
/* Caller-supplied frequency response (points complex floats), e.g. for tests. */
int kgpu_bank_set_response(kgpu_bank *b, int idx, float const *response);
int kgpu_bank_get_response(kgpu_bank *b, int idx, float *response); /* device -> host copy */
/* shift as passed to execute_filter_output (filter.c:663); flags = kgpu_chan_flags. */
int kgpu_bank_set_shift(kgpu_bank *b, int idx, int shift);
int kgpu_bank_set_flags(kgpu_bank *b, int idx, int flags);
int kgpu_bank_enable(kgpu_bank *b, int idx, int enabled);
/* Beam weights alpha, beta as set_filter_weights leaves them in struct filter_out (filter.c:922-929):
 * alpha = i_weight/2 - j q_weight, beta = i_weight/2 + j q_weight.  Used when KGPU_CHAN_BEAM is set. */
int kgpu_bank_set_weights(kgpu_bank *b, int idx, double alpha_re, double alpha_im, double beta_re, double beta_im);
/* Fine-tuning oscillator fused into the channel kernel's store (replaces the per-sample loop radio.c:1499-1501 with
 * step_osc, osc.c:60-70, and the block phase of radio.c:1491-1497).  Output sample n of the k-th block processed after
 * this call is multiplied by exp(2 pi j (phase + (k+1) block_adj + m freq + rate m (m+1) / 2)), m = k*olen + n.
 * phase in cycles, freq in cycles/sample (= -remainder / output rate, radio.c:1481), rate in cycles/sample^2
 * (doppler_rate / rate^2), block_adj in cycles (= (shift % V) / V, radio.c:1493).  enable = 0 switches it off.
 * With the oscillator on, kgpu_bank_run_ex also writes the block's mean |y|^2 (radio.c:1515-1520). */
int kgpu_bank_set_osc(kgpu_bank *b, int idx, int enable, double phase_cycles, double freq_cps, double rate_cps2,
                      double block_adj_cycles);
/* Phase (cycles, [0,1)) the oscillator will have at the first sample of the next block, before that block's adjustment. */
int kgpu_bank_get_osc_phase(kgpu_bank *b, int idx, double *phase_cycles);
/* Index of the block the next run processes (advanced by every kgpu_bank_run*; the filter.h layer sets it to the job number). */
int kgpu_bank_set_block_counter(kgpu_bank *b, long counter);
long kgpu_bank_block_counter(kgpu_bank const *b);
int kgpu_bank_channels(kgpu_bank const *b);          /* highest defined idx + 1 */
long kgpu_bank_out_stride(kgpu_bank const *b);        /* float2 per block of the packed output row */
long kgpu_bank_out_offset(kgpu_bank const *b, int idx); /* float2 offset of channel idx inside a row */
/* Batched slice x response -> inverse transform -> keep last olen (filter.c:728-921) for every
 * enabled channel and `nblocks` spectra.  d_out: nblocks * out_stride float2. */
int kgpu_bank_run(kgpu_bank *b, const void *d_spec, int nblocks, void *d_out, void *stream);
/* Same, plus out_pitch: float2 between consecutive blocks' output rows (0 = packed, kgpu_bank_out_stride), and
 * d_power: NULL or nblocks * capacity floats; [block*capacity + idx] receives the mean |y|^2 of every channel whose
 * oscillator is on (chan->sig.bb_power, radio.c:1515-1520). */
int kgpu_bank_run_ex(kgpu_bank *b, const void *d_spec, int nblocks, void *d_out, long out_pitch, float *d_power, void *stream);
/* Single channel, single block (the retune slow path of the filter.h layer). d_out: olen float2. */
int kgpu_bank_run_one(kgpu_bank *b, int idx, const void *d_spec, void *d_out, void *stream);
int kgpu_bank_run_one_ex(kgpu_bank *b, int idx, const void *d_spec, void *d_out, float *d_power /* NULL or 1 float */, void *stream);
/* Noise density estimate per channel and block from the device-resident spectrum (estimate_noise, radio.c:1783-1866,
 * quantile :1722-1775) with the shift each channel was last given: d_n0[block*capacity + idx], doubles, in the
 * reference's scaling (energy per bin / (bins * samprate)).  Saves the 13 MB/block spectrum read-back. */
int kgpu_bank_noise(kgpu_bank *b, const void *d_spec, int nblocks, double samprate, double *d_n0, void *stream);

/* FM discriminator front half on the outputs a kgpu_bank_run* just produced (replaces the per-sample loops of demod_fm,
 * fm.c:104-131 amplitude statistics and fm.c:205-231 plain quadrature discriminator): for every COMPLEX channel and block
 *   d_baseband[block * 2*out_pitch + 2*out_offset(idx) + n] = arg(y[n] conj y[n-1]) / pi     (olen floats, y[-1] carried across calls)
 *   d_stats[(block * capacity + idx) * 2 + {0,1}]           = mean |y|, sum (|y| - mean)^2   (doubles)
 * out_pitch as given to kgpu_bank_run_ex (0 = packed). */
int kgpu_bank_fm_front(kgpu_bank *b, const void *d_out, long out_pitch, int nblocks, float *d_baseband, double *d_stats, void *stream);

/* Push pending channel changes (shift/filter/enable) to the device now, ordered after `stream`. */
int kgpu_bank_commit(kgpu_bank *b, void *stream);

/* A small master (small_master.cuh): the forward transform and every slave of one block in one CTA, one kernel launch per
 * write, for radiod's per-channel secondary masters (filter2, the wfm / stereod / rdsd composite, packetd, ctcss).  Its
 * envelope: Nc (N for COMPLEX, N/2 for REAL, with L and N even) has factors 2, 3, 5, 7 and at most 28 812 points; at most
 * KGPU_SMALL_MAX_SLAVES slaves, each of a point count with the same bounds.  The caller owns the window, the spectrum
 * slots (kgpu_small_spec_stride float2 per block, kgpu_master_spec_stride's layout) and the output rows. */
#define KGPU_SMALL_MAX_SLAVES 8
typedef struct kgpu_small kgpu_small;
long kgpu_small_smem(int L, int M, int in_type); /* host only: the forward's shared memory in bytes, -1 outside the envelope */
kgpu_small *kgpu_small_create(int L, int M, int in_type);
void kgpu_small_destroy(kgpu_small *m);
long kgpu_small_spec_stride(kgpu_small const *m);
int kgpu_small_define(kgpu_small *m, int idx, int olen, int out_type); /* the slave's points, or -1 */
int kgpu_small_undefine(kgpu_small *m, int idx);
/* set_filter's design and response transform, bitwise kgpu_bank_set_filter's; the response (points float2) is copied to
 * `response`.  Synchronises `stream` first: launches queued on it may still read the old response. */
int kgpu_small_set_filter(kgpu_small *m, int idx, double low, double high, double kaiser_beta, float *response, void *stream);
int kgpu_small_set_slave(kgpu_small *m, int idx, int shift, int isb); /* used by the next kgpu_small_run */
long kgpu_small_out_offset(kgpu_small const *m, int idx); /* float2 offset of slave idx in an output row */
long kgpu_small_out_stride(kgpu_small const *m);          /* float2 of one output row */
/* nblocks blocks from d_win (block b's window starts L samples after block b-1's): spectra into d_spec, every slave with a
 * response into d_out (rows out_pitch float2 apart).  only >= 0: d_win is not read and slave `only` alone is recomputed
 * from the spectra already in d_spec (after a retune). */
int kgpu_small_run(kgpu_small *m, const void *d_win, int nblocks, void *d_spec, void *d_out, long out_pitch, int only,
                   void *stream);
/* Testing aid: 0 forces the generic runtime-plan kernels even where a compile-time specialised
 * kernel exists (both are parity-tested); it takes effect at the next launch, also for existing masters. Default 1.
 * Masters running the extended pair (kgpu_master_create_ex) have no specialised kernels and ignore it.
 * A master's forward kernel pair (specialised where its split has one, generic otherwise) is chosen when it is created;
 * kgpu_master_describe prints it.  Kernel variants that lost on H100 are not in the library. */
int kgpu_use_static_kernels(int on);
/* fwd_cols_r36, the column pass of masters split 1296 x n2, copies each CTA's input tile into shared memory with tensor
 * copies (TMA) where the input allows a tensor map: d_in 16-byte aligned, the hop between windows and the row pitch of
 * n2 points multiples of 16 bytes.  Any other input, or on = 0, runs the same kernel reading its inputs with global loads;
 * the spectra and statistics are bitwise the same.  The default is on, or what the environment variable KA9Q_COLS_TMA
 * (0 / 1) says when the first launch reads it; a call takes effect at the next launch, also for existing masters. */
int kgpu_use_cols_tma(int on);
/* Pure host code: 1 if kgpu_forward of the master kgpu_master_create_any(L, M, in_type) builds, fed `fmt` input at d_in,
 * runs fwd_cols_r36 on tensor copies (with kgpu_use_cols_tma on), 0 if it does not, -1 for a length with no master. */
int kgpu_cols_tma_fits(int L, int M, int in_type, int fmt, const void *d_in);
/* REAL masters split 1296 x 1250 run their column and row passes as one launch, fwd_fused_r36_v2, wherever the column
 * pass could take its tile by tensor copies (kgpu_cols_tma_fits, with kgpu_use_cols_tma on), in launches of 2 or more
 * blocks: each block's row pass then overlaps the next block's column pass and reads its inter-pass rows from L2.  Every other master and input runs the two-kernel pair.  The
 * spectra and statistics are bitwise the same either way.  The default is on, or what the environment variable
 * KA9Q_FUSED_FWD (0 / 1) says when the first launch reads it; a call takes effect at the next launch. */
int kgpu_use_fused_forward(int on);
/* Pure host code: 1 if kgpu_forward of the master kgpu_master_create_any(L, M, in_type), fed `fmt` input at d_in, runs
 * the fused launch for 2 or more blocks (with kgpu_use_fused_forward and kgpu_use_cols_tma on), 0 if not, -1 for a length with no master. */
int kgpu_fused_forward_fits(int L, int M, int in_type, int fmt, const void *d_in);
/* Testing and measuring aids of the fused launch.  kgpu_fused_forward_options: `lead` (0 .. the C items per block) column
 * items of the next block go before a block's first row item; discard = 1 drops each inter-pass row from L2 once it is
 * read (default 0).  Takes effect at the next launch.  kgpu_fused_shape fills out[5] = {C items per block,
 * R items per block, n1, inter-pass row pitch in points, default lead}.  kgpu_fused_schedule fills out[5] = {kind
 * (0 C, 1 R), block, item, the block whose C items it waits for (-1: none), how many} for a ticket of a launch of
 * nblocks blocks.  kgpu_fused_discards writes the 128-byte lines (from the inter-pass buffer's start) that item R(blk, idx)
 * discards to lines[0 .. max-1] and returns their count.  All pure host code. */
int kgpu_fused_forward_options(int lead, int discard);
int kgpu_fused_shape(int *out);
int kgpu_fused_schedule(int nblocks, int lead, int ticket, int *out);
long kgpu_fused_discards(int blk, int idx, long *lines, long max);

/* Planner introspection, pure host code (works without a GPU): the in-register radices chosen for
 * a column transform of length len (returns their count, -1 if unplannable) and the two-pass split
 * n = n1*n2 of a long transform. */
int kgpu_plan_radices(int len, int *radices, int max);
int kgpu_plan_split(long n, int *n1, int *n2);
/* The same for the plans of kgpu_master_create_ex: the radix search also takes 11, 13, 17, 19, 23, and the split
 * accepts factors so planned.  Where len (n) has factors 2, 3, 5, 7 only they return what the two calls above return. */
int kgpu_plan_radices_ex(int len, int *radices, int max);
int kgpu_plan_split_ex(long n, int *n1, int *n2);

/* Multi-GPU hand-off of the block spectra (SURVEY.md 8e; replaces the per-block multicast the
 * reference leaves to the network, multicast.c): copy `bytes` (multiple of 16) from this GPU's
 * `d_src` to `mc_dst`, an NVSwitch MULTICAST address that maps the same symmetric buffer on every
 * GPU of the group (obtained by the caller, e.g. torch symmetric memory), with multimem.st -- one
 * NVLink egress serves all peers.  `nctas` thread blocks of 256 threads (0 = default) so the copy
 * co-resides with the forward kernels of the next step. */
int kgpu_multicast_copy(const void *d_src, void *mc_dst, unsigned long long bytes, int nctas, void *stream);

/* ---- wideband spectrum analyzer: replaces wideband_poll's fft_avg loops (spectrum.c:354-497) -------------------- */
typedef struct kgpu_spectrum kgpu_spectrum;
/* An analyzer of fft_n-point segments of a REAL or COMPLEX front end's raw samples into bin_count float bins.  The
 * transform is chosen from fft_n alone: REAL with even fft_n and fft_n/2 23-smooth runs the r2c of a REAL master
 * (L = fft_n, M = 1); COMPLEX 23-smooth, or REAL odd 23-smooth, a COMPLEX master of length fft_n; any other length a
 * Bluestein transform through a COMPLEX master of the smallest 7-smooth length P >= 2 fft_n - 1 whose split the
 * forward pair runs (both factors fit shared memory, so P <= 3500 x 3500 and fft_n <= 6 125 000); NULL and
 * kgpu_last_error() otherwise. */
kgpu_spectrum *kgpu_spectrum_create(int fft_n, int in_type, int bin_count);
/* fft_n floats, as generate_window() leaves them (spectrum.c:548-606); the default is all ones. */
int kgpu_spectrum_set_window(kgpu_spectrum *s, float const *window);
/* One poll (spectrum.c:354-497): d_bins[0 .. bin_count) = sum over fft_avg segments of gain |X|^2 in the reference's bin
 * mapping and order; bins the reference leaves 0 are 0, nothing past bin_count is written.
 *   d_ring        device ring of ring_samples samples (>= fft_n): float / int16 (fmt) samples (REAL) or pairs (COMPLEX)
 *   end           ring position just past the newest sample (taken modulo ring_samples); segments start at
 *                 end - adjust + i*hop (REAL) or end - adjust - i*hop (COMPLEX), adjust and hop as spectrum.c:364,407
 *   scale, derandomize  int16 samples are scale * (float)x after the randomizer flip (rx888.c:707-712,765)
 *   d_chg, nchg, end_index  NULL, or nchg scale changes of an int16 ring: the sample just before ring position end is
 *                 absolute sample end_index - 1, samples before the first change take `scale`
 *   shift         spectrum.c:347; fft_avg >= 1; 0 <= overlap < 1
 * Enqueued on `stream`; the analyzer's scratch is reused by the next run, so runs of one analyzer go on one stream.
 * A REAL walk index the reference would take below 0 (out of its array) contributes 0. */
int kgpu_spectrum_run(kgpu_spectrum *s, const void *d_ring, long ring_samples, long end, int fmt, float scale,
                      const struct kgpu_scale_change *d_chg, int nchg, long long end_index, int derandomize, int shift, int fft_avg, double overlap, float *d_bins, void *stream);
/* One narrowband poll (narrowband_poll, spectrum.c:206-306) on an analyzer created with in_type KGPU_COMPLEX:
 *   d_ring        device ring of ring_size float2 samples (>= fft_n), the channel's delivered blocks as spectrum.c:147-151
 *                 appends them (kgpu_spectrum_ring_append); ring_idx the position the next sample would take
 *   fft_avg       clamped as spectrum.c:244-246 does; *fft_avg_used (if not NULL) receives the count the poll used
 *   overlap       0 <= overlap < 1; segments start at ring_idx - lrint(fft_n (1 + (fft_avg-1)(1-overlap))) and step
 *                 fft_n - lrint(fft_n overlap)
 * d_bins[0 .. bin_count) = sum of |X|^2 / (fft_n^2 fft_avg) in narrowband_poll's mapping (bin i < bin_count/2 from X[i],
 * the others from X[fft_n - 2 (bin_count/2) + i]) and order; with an odd bin_count the last bin, which the reference reads
 * past its transform, is 0.  -1 if bin_count > fft_n or ring_size < fft_n.  Enqueued on `stream`, as kgpu_spectrum_run. */
int kgpu_spectrum_run_narrow(kgpu_spectrum *s, const void *d_ring, long ring_size, long ring_idx, int fft_avg,
                             double overlap, float *d_bins, int *fft_avg_used, void *stream);
/* olen float2 samples from d_src (device), or zeros when d_src is NULL, into the device ring d_ring of ring_size samples
 * starting at position ring_idx and wrapping (spectrum.c:147-151).  The new position is (ring_idx + olen) % ring_size. */
int kgpu_spectrum_ring_append(void *d_ring, long ring_size, long ring_idx, const void *d_src, long olen, void *stream);
/* "r2c|complex|bluestein fft_n=... real|complex P=...: <nc>-point complex two-pass n1 x n2" */
int kgpu_spectrum_describe(kgpu_spectrum const *s, char *buf, int buflen);
void kgpu_spectrum_destroy(kgpu_spectrum *s);
/* Pure host code: the path kgpu_spectrum_create would take for fft_n (0 r2c, 1 complex, 2 Bluestein; -1 when it would
 * fail) and, if buf is not NULL, the string kgpu_spectrum_describe would print. */
int kgpu_spectrum_plan(int fft_n, int in_type, char *buf, int buflen);

/* Algorithmic bytes per block of one forward + all enabled channels (SURVEY.md 8d). */
double kgpu_algorithmic_bytes(kgpu_master const *m, kgpu_bank const *b, int fmt);

#ifdef __cplusplus
}
#endif
#endif
