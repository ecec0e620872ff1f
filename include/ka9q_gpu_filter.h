/* include/ka9q_gpu_filter.h -- the reference-facing surface of libka9qgpu.so.
 *
 * This header is layout- and name-compatible with ka9q-radio's src/filter.h (commit 4e0033b4):
 * a program built against the reference header (radiod's radio.c / fm.c / linear.c, the front-end
 * drivers) links against libka9qgpu.so instead of filter.o and runs unmodified; tests/
 * test_filter_abi.py checks every field offset against the reference header where it is present.
 * Use this header only when building NEW code without the ka9q-radio tree.
 *
 *   entry point                   replaces (reference file:line)
 *   create_filter_input           filter.c:186-269   master: ring + forward plan  -> device plans
 *   create_filter_input_small     (EXTENSION) the same for a small secondary master: one kernel per write, no bank
 *   create_filter_output          filter.c:298-415   slave: response/ifft plan    -> bank slot
 *   execute_filter_input          filter.c:558-651   queue forward FFT            -> H2D + 2 kernels
 *   execute_filter_output         filter.c:663-921   wait, slice*response, IFFT   -> batched kernel
 *   set_filter                    filter.c:968-1045  Kaiser design + FFT          -> host design + device FFT
 *   set_filter_weights            filter.c:922-929
 *   write_rfilter / write_cfilter filter.c:1093-1134 ring advance, fire blocks
 *   delete_filter_input/output    filter.c:930-957
 *   write_i16filter               (EXTENSION, not in the reference) raw int16 ingest: fuses
 *                                 rx888.c:753-767 convert() into the first FFT pass
 *   write_rawfilter               (EXTENSION) raw 8-bit, packed 12-bit, 16-bit and float ingest: the conversion loops
 *                                 of rtlsdr.c, hydrasdr.c, airspy-unpack.c, bladerf.c, sdrplay.c, airspyhf.c and
 *                                 fobos.c on the device
 *   write_rawfilter_planar        (EXTENSION) SDRplay's separate int16 I and Q arrays as FILTER_RAW_S16 pairs
 *   filter_ingest_stats           (EXTENSION) the A/D energy and overranges those loops return, per drained block
 *   filter_iq_correction_setup    (EXTENSION) HackRF's and FUNcube's DC and I/Q gain and phase correction on the device
 *   filter_iq_records             (EXTENSION) the per-transfer sums and state those drivers' loops produce
 *   filter_siggen_setup           (EXTENSION) sig_gen.c's carrier and noise generated on the device
 *   write_genfilter               (EXTENSION) advance a generated master, replacing sig_gen.c's sample loop
 *   filter_siggen_stats           (EXTENSION) the energy that loop sums, per drained block
 *   filter_siggen_modulate        (EXTENSION) sig_gen.c's AM and DSB: the carrier times the driver's resampled envelope
 *   filter_siggen_mod_pointer     (EXTENSION) where src_callback_read puts that envelope
 *
 * Semantics kept: return 0 / -1 (write_*: 1 if a block fired), ND-deep spectrum ring with
 * lap -> zeros + block_drops++ (filter.c:690-701), owner-thread shortcut (filter.c:681-683),
 * missing response -> 0 with stale output (filter.c:715-718), caller-owned structs zeroed by
 * delete_*.  COMPLEX and REAL output slaves (filter.c:345-392), ISB and beam synthesis (filter.c:756-775) all run in
 * the master's batched launch.
 */
#ifndef KA9Q_GPU_FILTER_H
#define KA9Q_GPU_FILTER_H 1
#include <assert.h>
#include <complex.h>
#include <pthread.h>
#include <stdbool.h>
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
#error "C header (uses C99 complex); bind through include/ka9q_gpu.h from C++"
#endif

/* FFTW's opaque plan handle appears in the reference structs; the GPU library reuses the two
 * slots for its own context pointers.  Same typedef FFTW itself uses, so both may be included. */
typedef struct fftwf_plan_s *fftwf_plan;

enum filtertype { NONE, COMPLEX, REAL, SPECTRUM };

struct rc {
  float *r;
  float complex *c;
};
struct notch_state {
  int bin;
  double complex state;
  double alpha;
};

#define ND 4 /* depth of the spectrum ring */

struct filter_in {
  enum filtertype in_type;
  int points;         /* N = L + M - 1 */
  int ilen;           /* L */
  int bins;           /* N (complex) or N/2+1 (real) */
  int impulse_length; /* M */
  int wcnt;
  void *input_buffer; /* mirrored host ring the drivers write through input_write_pointer */
  size_t input_buffer_size;
  struct rc input_write_pointer;
  struct rc input_read_pointer;
  fftwf_plan fwd_plan; /* GPU library: master context */
  pthread_mutex_t filter_mutex;
  pthread_cond_t filter_cond;
  struct notch_state *notches; /* assigned by the caller (radio.c:601) */
  float complex *fdomain[ND];  /* host copies of the block spectra (pinned) */
  unsigned int next_jobnum;
  unsigned int completed_jobs[ND];
  bool perform_inline;
  uint64_t sample_index;
  uint64_t samples_by_job[ND];
  bool init;
  pthread_t owner;
};

struct filter_out {
  struct filter_in *master;
  enum filtertype out_type;
  int points;
  int olen;
  int bins;
  double complex alpha;
  double complex beta;
  float complex *fdomain;
  float complex *response; /* host copy of the device response */
  pthread_mutex_t response_mutex;
  struct rc output_buffer;
  struct rc output;
  fftwf_plan rev_plan; /* GPU library: slave context */
  unsigned next_jobnum;
  unsigned block_drops;
  int rcnt;
  uint64_t sample_index;
  bool beam;
  bool isb;
  bool init;
};

/* globals the reference's filter.c owns and radio.c/main.c touch (filter.h:17-24, filter.c:476-479) */
extern char const *Wisdom_file;
extern int N_worker_threads;
extern int N_internal_threads;
extern int FFTW_planning_level;
extern double FFTW_plan_timelimit;
extern int64_t Min_fft_time, Max_fft_time, Avg_fft_time, Mean_dev;

int create_filter_input(struct filter_in *master, int L, int M, enum filtertype in_type);
/* EXTENSION: create_filter_input for a master small enough for one CTA: radiod's per-channel secondary masters (filter2
 * of CW and ISB channels, radio.c:1583; the wfm / stereod / rdsd composite, wfm.c:70; packetd; ctcss).  Each write that
 * completes k blocks costs the window's H2D, one kernel, one D2H of the slaves' outputs and one event per block, and the
 * host state is sized to the master: no channel bank, nothing per KGF_MAX_SLAVES.  Envelope: Nc (N for COMPLEX, N/2 for
 * REAL, which needs even L and N) has factors 2, 3, 5, 7 and at most 28 812 points; outside it -1 is returned without
 * touching *master, and the caller calls create_filter_input as before.  The filter_in fields mean what they always mean,
 * and create_filter_output, set_filter, execute_filter_output(_batch), write_rfilter / write_cfilter, put_*filter and
 * delete_filter_* keep the reference's semantics (laps, no response, hot response swaps, k-block writes).  The slaves'
 * responses are bitwise a default master's.  On such a master:
 *   - at most 8 slaves, COMPLEX or REAL output, each of a point count (olen N / L) with the same bounds as Nc;
 *   - these return -1 with a message: SPECTRUM slaves, beam slaves (execute_filter_output), execute_filter_output_tuned,
 *     filter_output_untune, filter_input_enable_noise, both spectrum analyzers, and every int16, raw, I/Q corrected and
 *     generated ingest entry point (pointer-returning ones return NULL); filter_noise_estimate returns NAN;
 *   - in.notches is not read (only the front end has notches, radio.c:601), and fdomain[] is allocated but never written
 *     (only estimate_noise reads it, and only on the front end). */
int create_filter_input_small(struct filter_in *master, int L, int M, enum filtertype in_type);
/* Pure host code: the host and device bytes a create_filter_input_small master of this geometry allocates with max_slaves
 * slaves of olen <= L (an upper bound: ring, fdomain[], context, window, ND spectra, ND output rows, responses and the
 * slaves' own buffers), or -1 outside the envelope or for max_slaves outside 0..8. */
long filter_small_master_bytes(int L, int M, enum filtertype in_type, int max_slaves);
int create_filter_output(struct filter_out *slave, struct filter_in *master, int olen, enum filtertype out_type);
int execute_filter_input(struct filter_in *master);
int execute_filter_output(struct filter_out *slave, int shift);
int delete_filter_input(struct filter_in *master);
int delete_filter_output(struct filter_out *slave);
int set_filter(struct filter_out *slave, double low, double high, double kaiser_beta);
int set_filter_weights(struct filter_out *slave, double complex i_weight, double complex q_weight);
int write_cfilter(struct filter_in *master, float complex const *samples, int n);
int write_rfilter(struct filter_in *master, float const *samples, int n);
/* EXTENSION: raw ADC words.  n int16 samples (REAL master) or n I/Q pairs (COMPLEX master); a
 * master fed this way must not also be fed through write_rfilter/write_cfilter.  Each sample becomes
 * (float)x * scale with the scale of its own write, as rx888.c:764 converts each transfer (see FILTER_SCALE_CHANGES
 * for gain changes between writes).  derandomize is a per-device constant (rx888.c): the last write's applies to every
 * launch from then on. */
int write_i16filter(struct filter_in *master, int16_t const *samples, int n, float scale, bool derandomize);
/* Where a driver may deposit the next raw samples itself (pinned, mirrored ring: a block's worth stays contiguous),
 * e.g. as the libusb transfer buffer of rx888.c:797-826; publish with write_i16filter(master, NULL, n, scale, derand). */
int16_t *filter_i16_write_pointer(struct filter_in *master);
/* EXTENSION: raw 8-bit and packed 12-bit ADC words, unpacked on the device (airspy-unpack.c:105-129 for Airspy R2 and
 * HydraSDR RAW; rtlsdr.c:316-343 and hydrasdr.c:759-830 for the 8-bit formats).  n samples (REAL master) or I/Q pairs
 * (COMPLEX master) are copied into a pinned, mirrored ring of their own and fire blocks as write_i16filter does; each
 * launch sends the raw bytes of its windows to the device, unpacks them there, then runs the usual forward, notch,
 * channel and noise work.  U8 and S8 give floats bitwise equal to the drivers' (float)(scale * x) with a double scale;
 * PACKED12 (REAL masters only) gives (float)scale * (float)x, the drivers' float scale.  Each write's scale applies to
 * exactly its own samples.  PACKED12 needs n a multiple of 8 (whole groups of three 32-bit words), and
 * L and M - 1 multiples of 8 so every window starts on a group boundary (Airspy R2: L = 400000 / 200000, M - 1 = L/4);
 * other geometries are rejected with -1 and a message at the first write.  A master fed one format (raw, int16,
 * float or generated) rejects writes in another with -1: a raw, int16 or generated master refuses write_rfilter and
 * write_cfilter, and a float master refuses write_i16filter and filter_i16_write_pointer.  Returns -1 on error, 1 if
 * a block fired, else 0. */
enum filter_raw_format {
  FILTER_RAW_PACKED12 = 1,
  FILTER_RAW_U8 = 2,
  FILTER_RAW_S8 = 3,
  FILTER_RAW_S8_IQCORR = 4,  /* HackRF: signed byte I/Q with the driver's DC and I/Q correction (filter_iq_correction_setup) */
  FILTER_RAW_S16_IQCORR = 5, /* FUNcube: int16 I/Q with the same correction */
  FILTER_RAW_S16 = 6,        /* int16, REAL or I/Q: HydraSDR INT16_REAL / INT16_IQ; SDRplay through write_rawfilter_planar */
  FILTER_RAW_U16 = 7,        /* offset-binary uint16 (x = w - 32768), REAL only: HydraSDR UINT16_REAL */
  FILTER_RAW_SC16Q11 = 8,    /* bladeRF SC16_Q11 I/Q, COMPLEX only: bits 0-11 of each word, sign-extended from bit 11 */
  FILTER_RAW_F32 = 9,        /* float, REAL only: HydraSDR FLOAT32_REAL */
  FILTER_RAW_CF32 = 10,      /* float I/Q, COMPLEX only: HydraSDR FLOAT32_IQ */
  FILTER_RAW_CF32_CNRMF = 11, /* float I/Q, COMPLEX only: AirspyHF+ */
  FILTER_RAW_CF32_FSCALE = 12 /* float I/Q, COMPLEX only: Fobos */
};
/* The 16-bit formats (hydrasdr.c:681-716, :729-747, bladerf.c:215-246, sdrplay.c:1234-1246) give floats bitwise equal to
 * the drivers' (float)(scale * x) with a double scale; bladerf.c stores (float)x, i.e. scale 1.0.  Their limits, as the
 * drivers test them: x >= 32767 or x <= -32768 (S16, U16), x == 2047 or x == -2048 (SC16Q11).  Samples before the first
 * write are 0.0f (the U16 ring is prefilled with 0x8000 words). */
/* The float formats take the floats the vendor libraries deliver and store each driver's own value, bitwise:
 * (float)(scale * (double)x) with a double scale for F32, CF32 and CF32_CNRMF (hydrasdr.c:717-728, :748-758,
 * airspyhf.c:313-318), x * (float)scale in float for CF32_FSCALE (fobos.c:410-420).  They test no limits.  Their energy
 * (filter_ingest_stats' fenergy) sums the terms as each loop's source writes them: x * x in float (F32, CF32_FSCALE),
 * cnrm in double (CF32), cnrmf in float with both products rounded (CF32_CNRMF; the reference's build contracts it into a
 * fused multiply-add), added in double in a fixed order; the drivers' sums differ from it by their compiler's
 * reassociation (fobos.c's is a float sum).  A block with a NaN or Inf sample, or a float term past FLT_MAX, has a
 * non-finite energy, and so has every filter_ingest_stats result whose drained blocks include it: a driver's isfinite
 * guard on that result skips all of that call's blocks (draining after each write that fires a block keeps that to the
 * blocks the write fired).  Samples before the first write are 0.0f. */
int write_rawfilter(struct filter_in *master, void const *samples, int n, int format, double scale);
/* EXTENSION: SDRplay's separate I and Q arrays (sdrplay.c:1210-1246): n pairs i[k], q[k] interleaved into the raw ring of
 * a COMPLEX master fed FILTER_RAW_S16, then exactly a write_rawfilter(..., FILTER_RAW_S16, scale) of those pairs.  -1 on a
 * REAL master or one fed any other format. */
int write_rawfilter_planar(struct filter_in *master, int16_t const *i, int16_t const *q, int n, double scale);
/* Pure host code: the byte size of the raw ring write_rawfilter allocates for a master of this geometry and format (a
 * whole number of pages, and for PACKED12 of 12-byte groups, holding at least the master's float ring of samples), or -1
 * where write_rawfilter would reject the geometry. */
long filter_raw_ring_bytes(int L, int M, enum filtertype in_type, int format);
/* Scale changes of write_i16filter and write_rawfilter (every format without I/Q correction): a write whose scale differs from the previous
 * write's records a change at its first sample, in a table of FILTER_SCALE_CHANGES(L, S) entries, S the samples of the
 * master's float ring (input_buffer_size over the sample size).  A change leaves the table once S samples have been
 * launched after it (the wideband analyzer's device ring holds S samples).  A write whose change would overflow the
 * table returns -1 with a message and stores nothing.  A launch whose window holds one scale converts inside the first
 * FFT pass as before; one that holds more converts each sample with its own scale in a kernel of its own. */
#define FILTER_SCALE_CHANGES(L, S) (64 + 16 * (((S) + (L)-1) / (L)))
/* EXTENSION: the A/D statistics the drivers' conversion loops return (in_energy, overranges, samp_since_over), for masters
 * fed through write_rawfilter or write_i16filter.  Never blocks: sums over the blocks whose device work completed since
 * the previous call, each block counted once however rarely the caller asks.  Collection starts with the first call on
 * a master, which returns zeros; a master never asked launches nothing extra.  -1 for a master fed floats. */
struct filter_ingest_stats {
  uint64_t blocks;            /* blocks summed by this call */
  uint64_t samples;           /* their new samples (blocks * L): samples (REAL) or I/Q pairs (COMPLEX) */
  union {
    uint64_t energy;          /* integer formats: sum of x * x over every component of those samples */
    double fenergy;           /* float formats (FILTER_RAW_F32 ..): the sum of the driver loop's energy terms */
  };
  uint64_t overranges;        /* components at the format's limits (float formats: 0) */
  uint64_t overrange_samples; /* samples with at least one component at the limits */
  uint64_t since_over;        /* samples after the last summed block that had an overrange (over all calls) */
};
int filter_ingest_stats(struct filter_in *master, struct filter_ingest_stats *stats);
/* EXTENSION: the DC removal and I/Q gain and phase correction of hackrf.c:297-375 and funcube.c:194-310 on the device, for
 * COMPLEX masters fed FILTER_RAW_S8_IQCORR (HackRF: -128 is clipped to -127 and counted) or FILTER_RAW_S16_IQCORR
 * (FUNcube: words as they are; |x| >= 32767 is counted).  Each write_rawfilter call is one transfer: its samples are
 * corrected with the state the previous write left, and its scale applies to exactly its own samples.  The state update
 * after each write is the drivers', in their expression order, from exact integer moments of the write's words.
 * Call filter_iq_correction_setup once, before the first write; a write in these formats without it returns -1.
 *   dc_alpha  per sample: 1e-7 (hackrf.c:34), 1e-6 (funcube.c:28)
 *   gp_rate   HackRF: gain/phase weight gp_rate * n per write (rate_factor, hackrf.c:317): 1 / samprate;  else 0
 *   gp_alpha  FUNcube: the fixed weight per write (gainphase_alpha, funcube.c:209), with gp_rate 0
 *   dc_i .. tanphi: the driver's initial state (HackRF: imbalance 0, gains and secphi 1; FUNcube: the same)
 * Writes shorter than FILTER_IQ_MIN_WRITE pairs are rejected with -1 and a message (FUNcube at a 5 ms Blocktime writes
 * 960).  filter_ingest_stats returns -1 on such a master: filter_iq_records replaces it.  Samples before the first write
 * (the first window's M-1 history) are 0.0f. */
#define FILTER_IQ_MIN_WRITE 512
struct filter_iq_params {
  double dc_alpha, gp_rate, gp_alpha;
  double dc_i, dc_q, sinphi, imbalance, gain_i, gain_q, secphi, tanphi;
};
int filter_iq_correction_setup(struct filter_in *master, int format, struct filter_iq_params const *params);
/* Pure host code: the writes the device table of a master of this geometry holds (every write the raw ring can hold, at
 * FILTER_IQ_MIN_WRITE pairs each, and the launches in flight), or -1 where the format cannot feed it. */
long filter_iq_table_writes(int L, int M, enum filtertype in_type, int format);
/* One write's record: what the driver's state block computes, and the state after it.  The driver keeps its own
 * if_power rule (hackrf.c:364, funcube.c:293-294) and counters (clips, overranges, samp_since_over) from these. */
struct filter_iq_record {
  int64_t seq;        /* write number, from 0 */
  int64_t n;          /* I/Q pairs */
  int64_t sum_i, sum_q; /* samp_sum */
  double i_energy, q_energy, dotprod; /* as the drivers' loops sum them */
  int64_t overs;      /* HackRF clips, FUNcube components at the limits */
  int64_t since_over; /* components after the last one at the limits, -1 if none (funcube.c:256-267's samp_since_over) */
  double dc_i, dc_q, sinphi, imbalance, gain_i, gain_q, secphi, tanphi; /* after the update */
};
/* Never blocks: up to max records of the writes whose last sample's launch has completed, in write order, each once.
 * Records arrive up to one launch after their write.  A caller that falls more than the table's writes behind loses the
 * oldest.  Returns the count, or -1 on a master without I/Q correction. */
int filter_iq_records(struct filter_in *master, struct filter_iq_record *recs, int max);
/* EXTENSION: sig_gen.c's CW source (proc_sig_gen, sig_gen.c:286-346) generated on the device: no samples cross PCIe and
 * the host float ring is never written.  Call filter_siggen_setup once, before the first write (-1 on a master already
 * fed floats, int16 or raw words).  The master then rejects write_rfilter, write_cfilter, write_i16filter and
 * write_rawfilter with -1.  write_genfilter(master, n, scale) replaces the driver's per-sample loop and its
 * write_rfilter / write_cfilter: it advances the stream by n samples (REAL) or pairs (COMPLEX), each the loop's
 * (float)(samp * scale) with this write's scale, and fires blocks as write_rfilter does (1 if a block fired).  Samples
 * before the first write are 0.0f.  The noise is bitwise the reference's (xoshiro256** seeded by rand_init through
 * splitmix64, real_gauss); the carrier is within 1 ulp of its phasor chain.  CW is served (FM is CW in the reference),
 * and AM and DSB through filter_siggen_modulate.
 *   freq, rate  cycles per sample and per sample^2, what set_osc receives: carrier / samprate (REAL),
 *               (carrier - frequency) / samprate (COMPLEX), sig_gen.c:221-224
 *   amplitude, noise  sdr->amplitude, sdr->noise;  seed  rand_init's (1) */
struct filter_siggen_params {
  double freq, rate;
  double amplitude, noise;
  uint64_t seed;
};
int filter_siggen_setup(struct filter_in *master, struct filter_siggen_params const *params);
int write_genfilter(struct filter_in *master, int n, double scale);
/* EXTENSION: sig_gen.c's AM and DSB sources (sig_gen.c:297-314, :327-344).  libsamplerate stays with the driver; the
 * device multiplies the carrier by (dc + m), m the envelope floats src_callback_read produces at the front end's rate.
 * filter_siggen_modulate turns a master just set up by filter_siggen_setup into an AM (dc = 1) or DSB (dc = 0)
 * generator: -1 after its first write_genfilter, on a master that is not generated, or for a non-finite dc.  As in the
 * reference, a COMPLEX master then draws one Gaussian per pair and puts the noise on I only.
 * filter_siggen_mod_pointer is where the next write's envelope goes: one float per sample (REAL) or pair (COMPLEX), in a
 * pinned, mirrored host ring the library owns, with contiguous room for the largest n write_genfilter accepts (NULL on a
 * master that is not modulated).  The driver passes it straight to src_callback_read; write_genfilter(master, r, scale)
 * then commits the r envelope floats written there and generates those samples. */
int filter_siggen_modulate(struct filter_in *master, double dc);
float *filter_siggen_mod_pointer(struct filter_in *master);
/* The generated energy, as filter_ingest_stats counts its statistics: never blocks, sums over the blocks whose device
 * work completed since the previous call, each block once; the first call starts collection and returns zeros.  energy
 * is the sum of samp^2 (REAL, as sig_gen.c:294) or |samp|^2 (COMPLEX) of the unscaled samples; the reference's COMPLEX
 * loop adds re^2 - im^2 (sig_gen.c:324).  -1 on a master that is not generated. */
struct filter_siggen_stats {
  uint64_t blocks;  /* blocks summed by this call */
  uint64_t samples; /* their new samples (blocks * L) */
  double energy;
};
int filter_siggen_stats(struct filter_in *master, struct filter_siggen_stats *stats);
/* EXTENSION: serve many slaves with one call (what 1024 channel threads would each do): one wait per block. */
int execute_filter_output_batch(struct filter_out *const *slaves, int const *shifts, int n);
/* EXTENSION (downconvert()'s per-sample work, radio.c:1476-1501 and :1515-1520, on the device): execute_filter_output
 * plus the fine-tuning oscillator (set_osc / step_osc, osc.c:28-70), the block phase correction for shifts that are
 * not multiples of the overlap factor, and the baseband power.  shift, remainder: compute_tuning's results
 * (radio.c:1175-1199); samprate: the slave's output rate; doppler_rate: Hz/s.  *bb_power = chan->sig.bb_power.
 * output.c then holds what radio.c:1499-1501 would have left there; the caller skips that loop. */
int execute_filter_output_tuned(struct filter_out *slave, int shift, double remainder, double samprate, double doppler_rate,
                                double *bb_power);
int filter_output_untune(struct filter_out *slave); /* back to plain execute_filter_output semantics */
/* EXTENSION (estimate_noise, radio.c:1783-1866, on the device): once enabled (samprate = Frontend.samprate), every block
 * carries one noise-density estimate per slave; filter_noise_estimate() returns the one belonging to the block the
 * slave's last execute_filter_output* delivered (NAN if that block had to be recomputed alone after a retune). */
int filter_input_enable_noise(struct filter_in *master, double samprate);
double filter_noise_estimate(struct filter_out const *slave);

/* EXTENSION (spectrum.c:308-522 on the device) for a SPECTRUM slave: wideband_poll's fft_avg loops read a device copy of
 * the master's input ring (float or int16, as it is fed), created and seeded from the host ring by the first setup on
 * that master and appended by every block from then on.  setup: where setup_wideband / generate_window run, with fft_n
 * window floats; -1 for a length the device cannot serve (the caller keeps its CPU loop).  poll: bin_count floats as
 * wideband_poll leaves them, for the segments ending at the end of the last issued block, whose sample index goes to
 * *end_sample (the reference reads up to the live write pointer, up to one block newer).  One poller per slave. */
int filter_spectrum_setup(struct filter_out *slave, int fft_n, int bin_count, float const *window);
int filter_spectrum_poll(struct filter_out *slave, int shift, int fft_avg, double overlap, float *bin_data,
                         uint64_t *end_sample);

/* EXTENSION (spectrum.c:123-155 and narrowband_poll, :206-306, on the device) for a COMPLEX slave: its delivered blocks
 * are appended to a device ring exactly as the slave receives them (batched, recomputed after a retune, or zeros after a
 * lap), so with execute_filter_output_tuned the ring is spectrum.c's ring of chan->baseband; with plain
 * execute_filter_output it holds the untuned samples.  Slaves without an analyzer append nothing.
 *   setup    where setup_narrowband runs (after set_filter), with fft_n window floats as generate_window leaves them;
 *            -1 when the device cannot serve the slave (the caller keeps its CPU loop)
 *   reserve  spectrum.c:124-145, before downconvert() delivers the block: the first call creates ring_samples zeros
 *            with the write index at 0, a larger size keeps [0, old) and zeroes the rest, a smaller one does nothing
 *   poll     bin_count floats as narrowband_poll leaves them before its base / step scaling; one poller per slave
 *   ring     host copy of up to cap ring samples and the write index; returns the ring size (0 before reserve)
 * delete_filter_output frees the analyzer and its ring. */
int filter_spectrum_narrow_setup(struct filter_out *slave, int fft_n, int bin_count, float const *window);
int filter_spectrum_narrow_reserve(struct filter_out *slave, long ring_samples);
int filter_spectrum_narrow_poll(struct filter_out *slave, int fft_avg, double overlap, float *bin_data);
long filter_spectrum_narrow_ring(struct filter_out *slave, float complex *ring, long cap, long *ring_idx);

/* housekeeping the reference exports from filter.c */
void *run_fft(void *);
void suggest(int size, int dir, int clex);
long gcd(long a, long b);
long lcm(long a, long b);
bool goodchoice(long n);
int ceil_pow2(uint32_t x);
/* spectrum.c plans its own analysis FFTs through these; served by libfftw3f.so.3 when the host
 * has it (dlopen), NULL otherwise */
fftwf_plan plan_complex(int N, float complex *in, float complex *out, int direction);
fftwf_plan plan_r2c(int N, float *in, float complex *out);
fftwf_plan plan_c2r(int N, float complex *in, float *out);
void destroy_plan(fftwf_plan *plan);

/* ---- header-inline sample interface (filter.h:121-163) -------------------------------------- */
static inline void kgf_ring_wrap(void **p, void *base, size_t size) {
  if ((uint8_t *)*p >= (uint8_t *)base + size)
    *p = (uint8_t *)*p - size;
}
static inline int put_cfilter(struct filter_in *f, float complex s) {
  *f->input_write_pointer.c++ = s;
  kgf_ring_wrap((void **)&f->input_write_pointer.c, f->input_buffer, f->input_buffer_size);
  if (++f->wcnt < f->ilen)
    return 0;
  f->wcnt -= f->ilen;
  execute_filter_input(f);
  return 1;
}
static inline int put_rfilter(struct filter_in *f, float s) {
  *f->input_write_pointer.r++ = s;
  kgf_ring_wrap((void **)&f->input_write_pointer.r, f->input_buffer, f->input_buffer_size);
  if (++f->wcnt < f->ilen)
    return 0;
  f->wcnt -= f->ilen;
  execute_filter_input(f);
  return 1;
}
static inline float complex read_cfilter(struct filter_out *f, int rotate) {
  if (f->rcnt == 0) {
    execute_filter_output(f, rotate);
    f->rcnt = f->olen;
  }
  return f->output.c[f->olen - f->rcnt--];
}
static inline float read_rfilter(struct filter_out *f, int rotate) {
  if (f->rcnt == 0) {
    execute_filter_output(f, rotate);
    f->rcnt = f->olen;
  }
  return f->output.r[f->olen - f->rcnt--];
}
#endif
