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
void kgpu_master_destroy(kgpu_master *m);
int kgpu_master_points(kgpu_master const *m);       /* N */
int kgpu_master_bins(kgpu_master const *m);         /* REAL: N/2+1, COMPLEX: N (filter.c:197) */
long kgpu_master_spec_stride(kgpu_master const *m); /* float2 elements between consecutive block spectra */
/* Plan description for logs/DESIGN.md: "n1 x n2, radices ..." */
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
/* Testing aid: 0 forces the generic runtime-plan kernels even where a compile-time specialised
 * kernel exists (both are parity-tested). Default 1. */
int kgpu_use_static_kernels(int on);

/* A/B knobs (0 = shipped default everywhere).  key 13: 4 = column pass of the 1296 x n2 transform on the round-1 12 x 12 x 9
 * kernel instead of the 36 x 36 one; key 10: 5 = row pass of a REAL n1 x 1250 transform on the 50 x 25 kernel instead of the
 * 10 x 25 x 5 one; key 14: 1 = row pass takes the blocks first-to-last (default last-to-first: L2 reuse of the column pass's
 * output); key 15: n > 0 = row pass prefetches the rows of the CTA n later into L2 (default off).  The experiments that lost
 * (tile widths, TMA tile store, sub-batched forward, prefetches elsewhere ...) are no longer in the library. */
int kgpu_set_tuning(int key, int value);

/* Diagnostics: device buffer (6 uint64 per CTA of the cols kernel) receiving globaltimer stamps
 * at the phase boundaries; NULL (default) disables. */
int kgpu_set_debug_buffer(void *d_buf);
int kgpu_set_debug_buffer_rows(void *d_buf); /* same for the rows kernel */

/* Planner introspection, pure host code (works without a GPU): the in-register radices chosen for
 * a column transform of length len (returns their count, -1 if unplannable) and the two-pass split
 * n = n1*n2 of a long transform. */
int kgpu_plan_radices(int len, int *radices, int max);
int kgpu_plan_split(long n, int *n1, int *n2);

/* Multi-GPU hand-off of the block spectra (SURVEY.md 8e; replaces the per-block multicast the
 * reference leaves to the network, multicast.c): copy `bytes` (multiple of 16) from this GPU's
 * `d_src` to `mc_dst`, an NVSwitch MULTICAST address that maps the same symmetric buffer on every
 * GPU of the group (obtained by the caller, e.g. torch symmetric memory), with multimem.st -- one
 * NVLink egress serves all peers.  `nctas` thread blocks of 256 threads (0 = default) so the copy
 * co-resides with the forward kernels of the next step. */
int kgpu_multicast_copy(const void *d_src, void *mc_dst, unsigned long long bytes, int nctas, void *stream);

/* Algorithmic bytes per block of one forward + all enabled channels (SURVEY.md 8d). */
double kgpu_algorithmic_bytes(kgpu_master const *m, kgpu_bank const *b, int fmt);

#ifdef __cplusplus
}
#endif
#endif
