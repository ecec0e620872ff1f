/* filter_abi.c -- the reference's filter.h surface served by the H100 kernels.
 *
 * Host code stays C, exactly as north_star asks: this file owns the caller-visible state the
 * untouched ka9q-radio sources expect (mirrored input ring, ND-deep job bookkeeping, per-slave
 * output buffers, mutex/condvar hand-off) and forwards the arithmetic to the C-ABI in
 * include/ka9q_gpu.h.  One master = one device pipeline on one stream:
 *
 *   execute_filter_input  : H2D(window[s]) -> fwd_cols -> fwd_rows -> notch -> chan (ALL slaves,
 *                           batched with their last shifts) [-> noise] -> D2H(outputs) [-> D2H(spectrum windows)]
 *                           When the producer hands over k > 1 blocks at once (write_*filter with n >= 2L) they go
 *                           out as ONE launch sequence of k blocks (k <= ND-1).
 *   execute_filter_output : wait for that block's event, hand the slave its slice of the pinned
 *                           batch buffer; a slave whose shift/filter changed since the
 *                           block was issued is recomputed alone (retunes are rare, radio.c:1491)
 *
 * The two FFTW plan slots of the reference structs (fwd_plan / rev_plan, only ever touched by
 * filter.c itself) carry the contexts.  Reference lines are cited per function.
 */
#define _GNU_SOURCE 1
#include <cuda_runtime_api.h>
#include <dlfcn.h>
#include <errno.h>
#include <limits.h>
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <sys/mman.h>
#include <unistd.h>

#include "ka9q_gpu.h"
#include "ka9q_gpu_filter.h"

/* globals filter.c owns in the reference (filter.c:40-48, :476-479) */
char const *Wisdom_file;
int N_worker_threads = 1;
int N_internal_threads = 1;
int FFTW_planning_level = (1 << 5); /* FFTW_PATIENT; meaningless here, kept for radio.c:310-318 */
int64_t Min_fft_time = INT64_MAX;
int64_t Max_fft_time = 0;
int64_t Avg_fft_time = 0;
int64_t Mean_dev = 0;

#define KGF_MAX_SLAVES 2048 /* radiod allows 2000 channels (radio.h:356) */
#define KGF_MAX_RANGES 64

struct slave_ctx {
  int idx; /* bank slot */
  void *own;        /* the slave's private output buffer (output_buffer.{c,r}): lap zeros, copy mode */
  /* fine tuning fused into the channel kernel (extension, radio.c:1476-1497) */
  bool ft_on;
  int ft_shift;
  double ft_remainder, ft_freq, ft_rate, ft_adj;
  unsigned ft_ver; /* bumped whenever the oscillator parameters change */
  float last_power;
  double last_n0;
  struct nb_spec *nb; /* narrowband analyzer (filter_spectrum_narrow_*), NULL for every other slave */
};

/* the narrowband analyzer of a COMPLEX slave (extension): a device ring of the blocks it was delivered, appended as
 * spectrum.c:147-151 appends chan->baseband; every field is guarded by the master's c->mu */
struct nb_spec {
  kgpu_spectrum *ks;
  int bin_count;
  float complex *d_ring; /* NULL until the first filter_spectrum_narrow_reserve */
  long ring_size, ring_idx;
  float *d_bins, *h_bins;
  cudaEvent_t ev;
};

struct snap { /* what the batched launch of one ring slot used for one slave */
  int shift;
  unsigned ver, ft_ver;
  long off;
  bool isb, beam, ok;
  double complex alpha, beta;
};

/* a SPECTRUM slave served by filter_spectrum_setup / filter_spectrum_poll (extension) */
struct spec_slave {
  struct filter_out *slave;
  kgpu_spectrum *ks;
  int bin_count;
  float *d_bins, *h_bins;
  cudaEvent_t ev;
  struct spec_slave *next;
};

/* What feeds a master: nothing yet, floats, int16 words, raw words, or its own generator.  Floats are never recorded:
 * the header-inline put_rfilter / put_cfilter store them without calling the library, so a master holds floats once
 * its float ring has taken or launched a sample (ingest_of). */
enum ingest { INGEST_NONE, INGEST_FLOAT, INGEST_INT16, INGEST_RAW, INGEST_GEN };

/* The int16 or raw words, or the AM / DSB envelope floats, of a master's stream: a mirrored, pinned host ring of `size` bytes, `group` bytes to every 8
 * samples (REAL) or I/Q pairs, written at wp; rp is the first sample (history included) of the next launch's window. */
struct word_ring {
  char *base, *wp, *rp;
  size_t size, group;
};

struct master_ctx {
  bool small; /* false; a small master's context (struct small_ctx) starts with true */
  kgpu_master *km;
  kgpu_bank *bank;
  cudaStream_t st, st_one, st_d2h; /* pipeline, single-channel recompute, device->host copies */
  cudaEvent_t kev;                 /* kernels of the current launch done */
  size_t esz; /* bytes per input element (float: 4, float complex: 8) */
  void *d_win[ND];
  size_t win_bytes;
  float complex *d_spec; /* ND * spec_stride */
  long spec_stride;
  float complex *d_out, *h_out; /* ND rows of out_pitch float2 */
  long out_pitch;
  float *d_pw, *h_pw;   /* ND * KGF_MAX_SLAVES block powers (oscillator channels) */
  double *d_n0, *h_n0;  /* ND * KGF_MAX_SLAVES noise estimates */
  float complex *d_one, *h_one;
  float *d_one_pw, *h_one_pw;
  int one_cap;
  cudaEvent_t t0[ND], done[ND];
  bool timed[ND];
  pthread_mutex_t mu;
  struct filter_out *slots[KGF_MAX_SLAVES];
  unsigned ver[KGF_MAX_SLAVES];
  int cur_shift[KGF_MAX_SLAVES]; /* shift / isb / beam last pushed into the bank */
  bool cur_isb[KGF_MAX_SLAVES], cur_beam[KGF_MAX_SLAVES];
  double complex cur_alpha[KGF_MAX_SLAVES], cur_beta[KGF_MAX_SLAVES];
  struct snap snap[ND][KGF_MAX_SLAVES];
  int nslots; /* highest used + 1 */
  int spectrum_d2h; /* 0 none, 1 windows around the channels (what radio.c:1799-1831 reads), 2 everything */
  bool zero_copy;
  bool noise_on;
  double noise_samprate;
  int nranges;
  long range_lo[KGF_MAX_RANGES], range_hi[KGF_MAX_RANGES];
  bool ranges_dirty;
  struct notch_state *notches_seen;
  unsigned notch_hash;
  /* what feeds the master (see check_mode); int16 and raw words go through `ring`, raw ones are then unpacked on the
   * device from d_raw into d_win[slot]; a modulated generator's envelope goes through `ring` and d_raw too */
  enum ingest mode;
  int raw_fmt; /* INGEST_RAW: the enum filter_raw_format, its row of raw_formats; else 0 */
  struct word_ring ring;
  void *d_raw;
  bool i16_derand;
  /* the scale of every int16, 8-bit and packed-12 sample (the I/Q corrected formats keep theirs per write): samples
   * before chg[0].at take chg_base, those from chg[i].at on chg[i].scale.  A change enters where a write's scale differs
   * from the previous write's; changes leave once no launch, analyzer seeding or poll can read their samples.  d_chg takes
   * the changes of one launch's or poll's samples, copied from pinned staging h_stg (ND + 1 regions of chg_cap: one per
   * ring slot for the launches, one for the seedings and polls, whose reuse waits on stg_ev); d_conv the floats of a
   * window that holds more than one scale. */
  bool chg_started;
  double chg_base;
  struct kgpu_scale_change *chg, *d_chg, *h_stg;
  cudaEvent_t stg_ev;
  int nchg, chg_cap;
  float *d_conv;
  /* A/D statistics (filter_ingest_stats): one kgpu_block_stats per ring slot, folded in job order into `acc` */
  bool stats_on;
  struct kgpu_block_stats *d_bstats, *h_bstats;
  unsigned long long folded; /* blocks folded (or, before stats_on, skipped) so far */
  struct filter_ingest_stats acc;
  /* I/Q correction (the RAW_IQ formats): a ring table of the writes (host copy, device copy), the device's coefficient
   * set and record of each write, and the pinned copy of the records */
  struct kgpu_iq_params iq_par;
  int iq_cap; /* 0 until filter_iq_correction_setup has succeeded */
  struct kgpu_iq_write *h_iqw, *d_iqw;
  struct kgpu_iq_state *d_iqc;
  struct kgpu_iq_record *d_iqr, *h_iqr;
  unsigned long long iq_writes;          /* writes so far */
  long long iq_total;                    /* their I/Q pairs */
  unsigned long long iq_sent;            /* writes whose table entry is on the device */
  unsigned long long iq_scanned;         /* writes whose record a launch computes */
  unsigned long long iq_rec_from;        /* iq_scanned before the current launch */
  unsigned long long iq_job_done[ND];    /* iq_scanned after the launch of each ring slot's job */
  unsigned long long iq_checked;         /* jobs whose completion filter_iq_records has taken in */
  unsigned long long iq_avail, iq_given; /* records complete on the host; records handed to the caller */
  unsigned long long issued; /* blocks issued to the device so far */
  /* wideband spectrum analyzer (extension): a device copy of the input ring, in the ingest format, with the host float
   * ring's capacity and positions; created by the first filter_spectrum_setup, then appended by every launch */
  struct spec_slave *specs;
  void *d_sring;
  long sring_cap; /* samples */
  long sring_pos; /* just past the newest issued sample */
  bool sring_i16;
  /* sig_gen's source (filter_siggen_setup): the device generates every window, the host ring is never written.
   * d_gen_energy / h_gen_energy: each ring slot's block energies, folded in job order into gen_acc once asked for.
   * gen_mod: AM or DSB (filter_siggen_modulate), the envelope floats in `ring` */
  kgpu_siggen *gen;
  bool gen_mod;
  double *d_gen_energy, *h_gen_energy;
  bool gen_stats_on;
  unsigned long long gen_folded;
  struct filter_siggen_stats gen_acc;
};

/* ---------------------------------------------------------------- mirrored ring ------------- */
/* Same contract as the reference's mirror_alloc (misc.c:635-682): `size` bytes followed by a
 * second mapping of the same pages, so a window that starts near the end stays contiguous. */
static size_t page_round(size_t n) {
  size_t const pg = (size_t)sysconf(_SC_PAGESIZE);
  return (n + pg - 1) / pg * pg;
}
static void *ring_alloc(size_t size) {
  int const fd = memfd_create("ka9q-gpu-ring", 0);
  if (fd < 0)
    return NULL;
  if (ftruncate(fd, (off_t)size) != 0) {
    close(fd);
    return NULL;
  }
  char *base = mmap(NULL, 2 * size, PROT_NONE, MAP_PRIVATE | MAP_ANONYMOUS, -1, 0);
  if (base == MAP_FAILED) {
    close(fd);
    return NULL;
  }
  void *a = mmap(base, size, PROT_READ | PROT_WRITE, MAP_SHARED | MAP_FIXED, fd, 0);
  void *b = mmap(base + size, size, PROT_READ | PROT_WRITE, MAP_SHARED | MAP_FIXED, fd, 0);
  close(fd);
  if (a == MAP_FAILED || b == MAP_FAILED) {
    munmap(base, 2 * size);
    return NULL;
  }
  memset(base, 0, size);
  /* pin the primary view so the per-block H2D is a true async DMA (the copy never reads through
   * the mirror view, see window_h2d); harmless if the driver refuses */
  if (cudaHostRegister(base, size, cudaHostRegisterPortable) != cudaSuccess)
    (void)cudaGetLastError();
  return base;
}
static void ring_free(void *base, size_t size) {
  if (!base)
    return;
  if (cudaHostUnregister(base) != cudaSuccess)
    (void)cudaGetLastError();
  munmap(base, 2 * size);
}

static size_t wring_bytes(struct word_ring const *r, size_t n) { return n * r->group / 8; } /* packed-12: n % 8 == 0 */
static long wring_samples(struct word_ring const *r, size_t bytes) { return (long)(bytes * 8 / r->group); }
/* a ring of `size` bytes prefilled with the three-word `zero`, so the history samples and whatever the wideband
 * analyzer's seeding reads before the stream reaches it are 0.0 as in the float ring; wp past the M-1 history samples */
static int wring_open(struct word_ring *r, size_t size, size_t group, long history, uint32_t const zero[3]) {
  r->base = ring_alloc(size);
  if (!r->base)
    return -1;
  r->size = size;
  r->group = group;
  if (zero[0] | zero[1] | zero[2]) /* size is a multiple of the zero's period: 4 bytes, or 12 for packed-12 */
    for (size_t o = 0; o < size; o += sizeof *zero)
      memcpy(r->base + o, &zero[o / sizeof *zero % 3], sizeof *zero);
  r->rp = r->base;
  r->wp = r->base + wring_bytes(r, (size_t)history);
  return 0;
}
/* publish the n samples just stored at wp (the mirror view keeps a write across the end contiguous) */
static void wring_push(struct word_ring *r, size_t n) {
  r->wp += wring_bytes(r, n);
  kgf_ring_wrap((void **)&r->wp, r->base, r->size);
}
/* the window of the launch about to be issued, whose n new samples then leave the ring */
static char const *wring_advance(struct word_ring *r, size_t n) {
  char const *const win = r->rp;
  r->rp += wring_bytes(r, n);
  kgf_ring_wrap((void **)&r->rp, r->base, r->size);
  return win;
}

static int kgf_fail(char const *where) {
  fprintf(stderr, "ka9q-gpu filter: %s failed: kgpu: \"%s\" cuda: %s\n", where, kgpu_last_error(),
          cudaGetErrorString(cudaGetLastError()));
  return -1;
}

/* H2D of FFT window(s) that start inside the primary view and may run past its end: the part
 * beyond the end is the start of the ring again (that is what the mirror view shows the CPU). */
static int window_h2d(void *dst, void const *src, size_t bytes, void const *ring, size_t ring_size, cudaStream_t st) {
  char const *end = (char const *)ring + ring_size;
  if ((char const *)src + bytes <= end)
    return cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, st) == cudaSuccess ? 0 : -1;
  size_t const first = (size_t)(end - (char const *)src);
  if (cudaMemcpyAsync(dst, src, first, cudaMemcpyHostToDevice, st) != cudaSuccess)
    return -1;
  return cudaMemcpyAsync((char *)dst + first, ring, bytes - first, cudaMemcpyHostToDevice, st) == cudaSuccess ? 0 : -1;
}

static void *cache_aligned(size_t bytes) {
  void *p = NULL;
  return posix_memalign(&p, 64, bytes ? bytes : 64) == 0 ? p : NULL;
}

static void spec_slave_free(struct spec_slave *sp) {
  kgpu_spectrum_destroy(sp->ks);
  cudaFree(sp->d_bins);
  cudaFreeHost(sp->h_bins);
  if (sp->ev)
    cudaEventDestroy(sp->ev);
  free(sp);
}
/* unlink and free the analyzer of `slave` on master context c, if any (caller holds c->mu) */
static void spec_slave_drop(struct master_ctx *c, struct filter_out const *slave) {
  for (struct spec_slave **pp = &c->specs; *pp; pp = &(*pp)->next)
    if ((*pp)->slave == slave) {
      struct spec_slave *sp = *pp;
      *pp = sp->next;
      cudaStreamSynchronize(c->st);
      spec_slave_free(sp);
      return;
    }
}

static void nb_free(struct nb_spec *nb) {
  if (!nb)
    return;
  kgpu_spectrum_destroy(nb->ks);
  cudaFree(nb->d_ring);
  cudaFree(nb->d_bins);
  cudaFreeHost(nb->h_bins);
  if (nb->ev)
    cudaEventDestroy(nb->ev);
  free(nb);
}
/* the block a slave with a narrowband analyzer was just delivered (device samples, or NULL for a lap's zeros) onto its
 * ring, on stream st (caller holds c->mu) */
static int nb_append(struct slave_ctx *sc, void const *d_src, int olen, cudaStream_t st) {
  struct nb_spec *nb = sc->nb;
  if (!nb || !nb->d_ring)
    return 0;
  if (kgpu_spectrum_ring_append(nb->d_ring, nb->ring_size, nb->ring_idx, d_src, olen, st) != 0)
    return kgf_fail("narrowband spectrum ring append");
  nb->ring_idx = (nb->ring_idx + olen) % nb->ring_size;
  return 0;
}

static void small_teardown(struct filter_in *master);
static void master_teardown(struct filter_in *master) {
  struct master_ctx *c = (struct master_ctx *)master->fwd_plan;
  if (c && c->small) {
    small_teardown(master);
  } else if (c) {
    cudaStreamSynchronize(c->st);
    cudaStreamSynchronize(c->st_one);
    cudaStreamSynchronize(c->st_d2h);
    for (int i = 0; i < ND; i++) {
      cudaFree(c->d_win[i]);
      cudaEventDestroy(c->t0[i]);
      cudaEventDestroy(c->done[i]);
    }
    cudaFree(c->d_out);
    cudaFreeHost(c->h_out);
    cudaFree(c->d_pw);
    cudaFreeHost(c->h_pw);
    cudaFree(c->d_n0);
    cudaFreeHost(c->h_n0);
    cudaFree(c->d_spec);
    cudaFree(c->d_one);
    cudaFreeHost(c->h_one);
    cudaFree(c->d_one_pw);
    cudaFreeHost(c->h_one_pw);
    kgpu_bank_destroy(c->bank);
    kgpu_master_destroy(c->km);
    cudaStreamDestroy(c->st);
    cudaStreamDestroy(c->st_one);
    cudaStreamDestroy(c->st_d2h);
    cudaEventDestroy(c->kev);
    ring_free(c->ring.base, c->ring.size);
    cudaFree(c->d_raw);
    free(c->chg);
    cudaFree(c->d_chg);
    cudaFreeHost(c->h_stg);
    if (c->stg_ev)
      cudaEventDestroy(c->stg_ev);
    cudaFree(c->d_conv);
    cudaFree(c->d_bstats);
    cudaFreeHost(c->h_bstats);
    cudaFreeHost(c->h_iqw);
    cudaFree(c->d_iqw);
    cudaFree(c->d_iqc);
    cudaFree(c->d_iqr);
    cudaFreeHost(c->h_iqr);
    while (c->specs) {
      struct spec_slave *sp = c->specs;
      c->specs = sp->next;
      spec_slave_free(sp);
    }
    cudaFree(c->d_sring);
    kgpu_siggen_destroy(c->gen);
    cudaFree(c->d_gen_energy);
    cudaFreeHost(c->h_gen_energy);
    pthread_mutex_destroy(&c->mu);
    free(c);
    master->fwd_plan = NULL;
  }
  for (int i = 0; i < ND; i++) {
    if (master->fdomain[i])
      cudaFreeHost(master->fdomain[i]);
    master->fdomain[i] = NULL;
  }
  ring_free(master->input_buffer, master->input_buffer_size);
  master->input_buffer = NULL;
}

/* ---------------------------------------------------------------- small masters ------------- */
/* A master made by create_filter_input_small: one small_master_kernel launch per write (kgpu_small_run), no channel bank.
 * Its host state is what the filter.h semantics need and nothing sized by KGF_MAX_SLAVES: the float ring, a stream, ND
 * events, ND pinned output rows for its (at most KGPU_SMALL_MAX_SLAVES) slaves, and what each slot's launch used per
 * slave.  Device: one window, ND spectrum slots, ND output rows, the slaves' responses. */
struct small_ctx {
  bool small; /* true: see master_ctx */
  kgpu_small *ks;
  cudaStream_t st;
  cudaEvent_t done[ND];
  pthread_mutex_t mu;
  size_t esz;
  void *d_win;
  float complex *d_spec; /* ND * spec_stride */
  long spec_stride;
  float complex *d_out, *h_out; /* ND rows of out_pitch float2 */
  long out_pitch;
  struct filter_out *slots[KGPU_SMALL_MAX_SLAVES];
  unsigned ver[KGPU_SMALL_MAX_SLAVES];
  int cur_shift[KGPU_SMALL_MAX_SLAVES];
  bool cur_isb[KGPU_SMALL_MAX_SLAVES];
  struct snap snap[ND][KGPU_SMALL_MAX_SLAVES];
};

static bool is_small(struct filter_in const *f) { return f && f->fwd_plan && *(bool const *)f->fwd_plan; }
/* -1 with a message: `who` is not served on a small master (see create_filter_input_small) */
static int small_refuses(char const *who) {
  fprintf(stderr, "%s: not served on a master made by create_filter_input_small\n", who);
  return -1;
}

/* the window bytes one launch sends: up to ND-1 consecutive blocks (fire_ready_blocks) */
static size_t small_win_bytes(int L, int M, size_t esz) { return esz * ((size_t)(ND - 2) * (size_t)L + (size_t)(L + M - 1)); }
/* output row pitch for slaves of at most `points` points each (olen <= points) */
static long small_row_pitch(int nslaves, long points) { return ((long)nslaves * points + 3) / 4 * 4; }

long filter_small_master_bytes(int L, int M, enum filtertype in_type, int max_slaves) {
  if ((in_type != REAL && in_type != COMPLEX) || max_slaves < 0 || max_slaves > KGPU_SMALL_MAX_SLAVES ||
      kgpu_small_smem(L, M, in_type == REAL ? KGPU_REAL : KGPU_COMPLEX) < 0)
    return -1;
  long const N = (long)L + M - 1, bins = in_type == COMPLEX ? N : N / 2 + 1, stride = (bins + 3) / 4 * 4;
  size_t const esz = in_type == COMPLEX ? sizeof(float complex) : sizeof(float);
  long const pitch = small_row_pitch(max_slaves, N); /* a slave of olen <= L has at most N points */
  long const host = (long)sizeof(struct small_ctx) + (long)page_round((size_t)ND * (size_t)N * esz) /* float ring */
                    + ND * bins * (long)sizeof(float complex)                                      /* fdomain[] */
                    + ND * pitch * (long)sizeof(float complex)                                     /* output rows */
                    + (long)max_slaves * N * (long)(sizeof(float complex) + sizeof(float complex) + 2 * sizeof(float complex));
                    /* per slave: response, fdomain, own output buffer (upper bound) */
  long const dev = (long)small_win_bytes(L, M, esz) + ND * stride * (long)sizeof(float complex) +
                   ND * pitch * (long)sizeof(float complex) + (long)max_slaves * N * (long)sizeof(float complex);
  return host + dev;
}

static void small_teardown(struct filter_in *master) {
  struct small_ctx *c = (struct small_ctx *)master->fwd_plan;
  cudaStreamSynchronize(c->st);
  for (int i = 0; i < ND; i++)
    cudaEventDestroy(c->done[i]);
  cudaFree(c->d_win);
  cudaFree(c->d_spec);
  cudaFree(c->d_out);
  cudaFreeHost(c->h_out);
  kgpu_small_destroy(c->ks);
  cudaStreamDestroy(c->st);
  pthread_mutex_destroy(&c->mu);
  free(c);
  master->fwd_plan = NULL;
}

/* create_filter_input for a master one CTA serves (filter.c:186-269 semantics); -1 without touching *master outside
 * the envelope of kgpu_small_smem */
int create_filter_input_small(struct filter_in *master, int const L, int const M, enum filtertype const in_type) {
  if (master == NULL || (in_type != REAL && in_type != COMPLEX) ||
      kgpu_small_smem(L, M, in_type == REAL ? KGPU_REAL : KGPU_COMPLEX) < 0)
    return -1;
  if (master->init && is_small(master) && master->ilen == L && master->impulse_length == M && in_type == master->in_type)
    return 0; /* unchanged (filter.c:191) */
  struct small_ctx *c = calloc(1, sizeof *c);
  if (!c)
    return -1;
  c->small = true;
  c->ks = kgpu_small_create(L, M, in_type == REAL ? KGPU_REAL : KGPU_COMPLEX);
  if (!c->ks) {
    fprintf(stderr, "create_filter_input_small(L=%d M=%d): %s\n", L, M, kgpu_last_error());
    free(c);
    return -1;
  }
  if (master->init && master->fwd_plan)
    master_teardown(master);
  int const N = L + M - 1;
  int const bins = (in_type == COMPLEX) ? N : N / 2 + 1;
  c->esz = (in_type == COMPLEX) ? sizeof(float complex) : sizeof(float);
  c->spec_stride = kgpu_small_spec_stride(c->ks);
  pthread_mutex_init(&c->mu, NULL);
  bool ok = cudaStreamCreateWithFlags(&c->st, cudaStreamNonBlocking) == cudaSuccess;
  ok = ok && cudaMalloc(&c->d_win, small_win_bytes(L, M, c->esz)) == cudaSuccess;
  ok = ok && cudaMalloc((void **)&c->d_spec, sizeof(float complex) * (size_t)c->spec_stride * ND) == cudaSuccess;
  for (int i = 0; ok && i < ND; i++)
    ok = cudaEventCreateWithFlags(&c->done[i], cudaEventDisableTiming) == cudaSuccess;
  master->fwd_plan = (fftwf_plan)c;
  master->points = N;
  master->perform_inline = (N_worker_threads == 0);
  master->bins = bins;
  master->ilen = L;
  master->impulse_length = M;
  master->in_type = in_type;
  master->wcnt = 0;
  master->next_jobnum = 0;
  master->sample_index = 0;
  for (int i = 0; i < ND; i++) { /* allocated for the caller's layout; no launch copies the spectrum back */
    ok = ok && cudaHostAlloc((void **)&master->fdomain[i], sizeof(float complex) * (size_t)bins, cudaHostAllocPortable) ==
                   cudaSuccess;
    if (ok)
      memset(master->fdomain[i], 0, sizeof(float complex) * (size_t)bins);
    master->completed_jobs[i] = UINT_MAX; /* filter.c:214 */
  }
  master->input_buffer_size = page_round((size_t)ND * N * c->esz);
  master->input_buffer = ok ? ring_alloc(master->input_buffer_size) : NULL;
  ok = ok && master->input_buffer != NULL;
  if (!ok) {
    fprintf(stderr, "create_filter_input_small(L=%d M=%d): device/host allocation failed: %s\n", L, M,
            cudaGetErrorString(cudaGetLastError()));
    master_teardown(master);
    return -1;
  }
  if (in_type == COMPLEX) { /* filter.c:243-244 */
    master->input_read_pointer.c = master->input_buffer;
    master->input_write_pointer.c = master->input_read_pointer.c + (M - 1);
    master->input_read_pointer.r = master->input_write_pointer.r = NULL;
  } else {
    master->input_read_pointer.r = master->input_buffer;
    master->input_write_pointer.r = master->input_read_pointer.r + (M - 1);
    master->input_read_pointer.c = master->input_write_pointer.c = NULL;
  }
  if (!master->init) {
    pthread_mutex_init(&master->filter_mutex, NULL);
    pthread_cond_init(&master->filter_cond, NULL);
    master->init = true;
  }
  master->owner = pthread_self();
  return 0;
}

/* the output rows for the slaves now defined (c->mu held) */
static int small_rows(struct small_ctx *c) {
  long const need = kgpu_small_out_stride(c->ks);
  if (need <= c->out_pitch)
    return 0;
  cudaStreamSynchronize(c->st);
  cudaFree(c->d_out);
  cudaFreeHost(c->h_out);
  c->d_out = NULL;
  c->h_out = NULL;
  c->out_pitch = 0;
  for (int s = 0; s < ND; s++)
    for (int i = 0; i < KGPU_SMALL_MAX_SLAVES; i++)
      c->snap[s][i].ok = false;
  if (cudaMalloc((void **)&c->d_out, sizeof(float complex) * (size_t)need * ND) != cudaSuccess ||
      cudaHostAlloc((void **)&c->h_out, sizeof(float complex) * (size_t)need * ND, cudaHostAllocPortable) != cudaSuccess)
    return -1;
  c->out_pitch = need;
  return 0;
}

/* create_filter_output on a small master: a slot among its KGPU_SMALL_MAX_SLAVES (filter.c:298-415 semantics) */
static int small_create_output(struct filter_out *slave, struct filter_in *master, int len, enum filtertype out_type) {
  if (out_type != COMPLEX && out_type != REAL)
    return small_refuses("create_filter_output (SPECTRUM)");
  struct small_ctx *c = (struct small_ctx *)master->fwd_plan;
  struct slave_ctx *sc = (struct slave_ctx *)slave->rev_plan;
  if (slave->init && slave->master != master) /* a slave moves between masters only through delete_filter_output */
    return -1;
  if (!slave->init) {
    pthread_mutex_init(&slave->response_mutex, NULL);
    slave->init = true;
  }
  pthread_mutex_lock(&c->mu);
  if (!sc) {
    int idx = -1;
    for (int i = 0; i < KGPU_SMALL_MAX_SLAVES && idx < 0; i++)
      if (c->slots[i] == NULL)
        idx = i;
    if (idx < 0) {
      pthread_mutex_unlock(&c->mu);
      fprintf(stderr, "create_filter_output: a small master serves at most %d slaves\n", KGPU_SMALL_MAX_SLAVES);
      return -1;
    }
    sc = calloc(1, sizeof *sc);
    if (!sc) {
      pthread_mutex_unlock(&c->mu);
      return -1;
    }
    sc->idx = idx;
    c->slots[idx] = slave;
    slave->rev_plan = (fftwf_plan)sc;
  }
  cudaStreamSynchronize(c->st);
  int const pts = kgpu_small_define(c->ks, sc->idx, len, out_type == REAL ? KGPU_REAL : KGPU_COMPLEX);
  c->ver[sc->idx]++;
  int const rows = pts > 0 ? small_rows(c) : 0;
  pthread_mutex_unlock(&c->mu);
  if (pts <= 0 || rows != 0) {
    fprintf(stderr, "create_filter_output: %s\n", kgpu_last_error());
    return -1;
  }
  pthread_mutex_lock(&slave->response_mutex);
  free(slave->response);
  slave->response = NULL;
  pthread_mutex_unlock(&slave->response_mutex);
  free(slave->fdomain);
  free(sc->own);
  slave->olen = len;
  slave->points = pts;
  slave->master = master;
  slave->out_type = out_type;
  set_filter_weights(slave, 1.0, 0.0);
  slave->bins = out_type == COMPLEX ? pts : pts / 2 + 1;
  size_t const osz = out_type == COMPLEX ? sizeof(float complex) : sizeof(float);
  sc->own = cache_aligned(osz * (size_t)pts);
  slave->fdomain = cache_aligned(sizeof(float complex) * (size_t)slave->bins);
  if (!slave->fdomain || !sc->own)
    return -1;
  memset(sc->own, 0, osz * (size_t)pts);
  if (out_type == COMPLEX) {
    slave->output_buffer.c = sc->own;
    slave->output.c = slave->output_buffer.c + slave->bins - len; /* filter.c:357 */
    slave->output_buffer.r = slave->output.r = NULL;
  } else {
    slave->output_buffer.r = sc->own;
    slave->output.r = slave->output_buffer.r + slave->points - len; /* filter.c:385 */
    slave->output_buffer.c = slave->output.c = NULL;
  }
  slave->next_jobnum = master->next_jobnum;
  return 0;
}

/* k consecutive blocks as one launch: the window's H2D (two copies at the ring's end), small_master_kernel, one D2H of
 * the output rows, one event per block */
static int small_execute(struct filter_in *const f, int const k) {
  struct small_ctx *c = (struct small_ctx *)f->fwd_plan;
  pthread_mutex_lock(&c->mu);
  unsigned const jobnum = f->next_jobnum;
  int const slot = (int)(jobnum % ND);
  for (int j = 0; j < k; j++) { /* the slots' previous occupants (job - ND) must have drained */
    cudaEventSynchronize(c->done[slot + j]);
    for (int i = 0; i < KGPU_SMALL_MAX_SLAVES; i++)
      c->snap[slot + j][i].ok = false;
  }
  void **const rp = f->in_type == COMPLEX ? (void **)&f->input_read_pointer.c : (void **)&f->input_read_pointer.r;
  char const *const src = *rp;
  *rp = (char *)*rp + c->esz * (size_t)f->ilen * (size_t)k;
  kgf_ring_wrap(rp, f->input_buffer, f->input_buffer_size);
  size_t const span = (size_t)(k - 1) * (size_t)f->ilen + (size_t)f->points;
  float complex *spec = c->d_spec + (size_t)slot * (size_t)c->spec_stride;
  float complex *d_row = c->d_out ? c->d_out + (size_t)slot * (size_t)c->out_pitch : NULL;
  float complex *h_row = c->h_out ? c->h_out + (size_t)slot * (size_t)c->out_pitch : NULL;
  int rc = 0;
  if (window_h2d(c->d_win, src, c->esz * span, f->input_buffer, f->input_buffer_size, c->st) != 0)
    rc = kgf_fail("execute_filter_input: H2D of the window");
  /* a master without slaves still transforms: a slave created later recomputes from the stored spectrum */
  float complex dummy_row;
  if (rc == 0 && kgpu_small_run(c->ks, c->d_win, k, spec, d_row ? (void *)d_row : (void *)&dummy_row, c->out_pitch, -1, c->st) != 0)
    rc = kgf_fail("execute_filter_input: kgpu_small_run");
  if (rc == 0 && h_row &&
      cudaMemcpyAsync(h_row, d_row, sizeof(float complex) * (size_t)(k * c->out_pitch), cudaMemcpyDeviceToHost, c->st) !=
          cudaSuccess)
    rc = kgf_fail("execute_filter_input: D2H of the outputs");
  if (rc == 0)
    for (int i = 0; i < KGPU_SMALL_MAX_SLAVES; i++) {
      struct filter_out *o = c->slots[i];
      if (!o || !o->response)
        continue;
      for (int j = 0; j < k; j++) {
        struct snap *s = &c->snap[slot + j][i];
        s->shift = c->cur_shift[i];
        s->isb = c->cur_isb[i];
        s->ver = c->ver[i];
        s->off = kgpu_small_out_offset(c->ks, i);
        s->ok = true;
      }
    }
  for (int j = 0; j < k; j++)
    cudaEventRecord(c->done[slot + j], c->st);
  pthread_mutex_unlock(&c->mu);

  pthread_mutex_lock(&f->filter_mutex);
  f->owner = pthread_self();
  for (int j = 0; j < k; j++) {
    f->samples_by_job[slot + j] = f->sample_index;
    f->completed_jobs[slot + j] = jobnum + (unsigned)j; /* "complete" == issued; consumers wait on the slot's event */
    f->sample_index += (uint64_t)f->ilen;
  }
  f->next_jobnum += (unsigned)k;
  pthread_cond_broadcast(&f->filter_cond);
  pthread_mutex_unlock(&f->filter_mutex);
  if (f->perform_inline)
    cudaEventSynchronize(c->done[slot + k - 1]);
  return rc;
}

/* ---------------------------------------------------------------- create_filter_input ------- */
/* filter.c:186-269 */
int create_filter_input(struct filter_in *master, int const L, int const M, enum filtertype const in_type) {
  if (master == NULL || L <= 0 || M <= 0)
    return -1;
  if (master->init && master->ilen == L && master->impulse_length == M && in_type == master->in_type)
    return 0; /* unchanged (filter.c:191) */
  if (in_type != REAL && in_type != COMPLEX)
    return -1;
  int const N = L + M - 1;
  int const bins = (in_type == COMPLEX) ? N : N / 2 + 1;
  if (bins < 2)
    return -1;
  if (master->init && master->fwd_plan)
    master_teardown(master);

  struct master_ctx *c = calloc(1, sizeof *c);
  if (!c)
    return -1;
  /* any N, as filter.c:201 plans: where kgpu_master_create_ex serves N this is exactly its master (and a 7-smooth N
   * gets kgpu_master_create's); other lengths run a Bluestein transform with the same spectrum layout */
  c->km = kgpu_master_create_any(L, M, in_type == REAL ? KGPU_REAL : KGPU_COMPLEX);
  if (!c->km) {
    fprintf(stderr, "create_filter_input(L=%d M=%d): %s\n", L, M, kgpu_last_error());
    free(c);
    return -1;
  }
  c->bank = kgpu_bank_create(c->km, KGF_MAX_SLAVES);
  c->esz = (in_type == COMPLEX) ? sizeof(float complex) : sizeof(float);
  c->spec_stride = kgpu_master_spec_stride(c->km);
  /* What of each block's spectrum goes back to master->fdomain[] on the host (radio.c:1799-1831 and spectrum.c:318
   * read it there): "windows" (default) = the bins estimate_noise reads around every slave's shift; "all"/"1" = the
   * whole spectrum; "0" = nothing (callers use kgf_noise_estimate / the device spectrum). */
  char const *env = getenv("KA9Q_GPU_SPECTRUM_D2H");
  c->spectrum_d2h = 1;
  if (env && (env[0] == '0' || env[0] == 'n'))
    c->spectrum_d2h = 0;
  else if (env && (env[0] == '1' || env[0] == 'a'))
    c->spectrum_d2h = 2;
  env = getenv("KA9Q_GPU_ZEROCOPY");
  c->zero_copy = env && env[0] == '1';
  c->ranges_dirty = true;
  pthread_mutex_init(&c->mu, NULL);
  bool ok = c->bank != NULL;
  ok = ok && cudaStreamCreateWithFlags(&c->st, cudaStreamNonBlocking) == cudaSuccess;
  ok = ok && cudaStreamCreateWithFlags(&c->st_one, cudaStreamNonBlocking) == cudaSuccess;
  ok = ok && cudaStreamCreateWithFlags(&c->st_d2h, cudaStreamNonBlocking) == cudaSuccess;
  ok = ok && cudaEventCreateWithFlags(&c->kev, cudaEventDisableTiming) == cudaSuccess;
  ok = ok && cudaMalloc((void **)&c->d_spec, sizeof(float complex) * (size_t)c->spec_stride * ND) == cudaSuccess;
  ok = ok && cudaMalloc((void **)&c->d_pw, sizeof(float) * ND * KGF_MAX_SLAVES) == cudaSuccess;
  ok = ok && cudaHostAlloc((void **)&c->h_pw, sizeof(float) * ND * KGF_MAX_SLAVES, cudaHostAllocPortable) == cudaSuccess;
  ok = ok && cudaMalloc((void **)&c->d_n0, sizeof(double) * ND * KGF_MAX_SLAVES) == cudaSuccess;
  ok = ok && cudaHostAlloc((void **)&c->h_n0, sizeof(double) * ND * KGF_MAX_SLAVES, cudaHostAllocPortable) == cudaSuccess;
  ok = ok && cudaMalloc((void **)&c->d_one_pw, sizeof(float)) == cudaSuccess;
  ok = ok && cudaHostAlloc((void **)&c->h_one_pw, sizeof(float), cudaHostAllocPortable) == cudaSuccess;
  c->win_bytes = c->esz * ((size_t)(ND - 2) * (size_t)L + (size_t)N); /* up to ND-1 consecutive windows */
  for (int i = 0; ok && i < ND; i++) {
    ok = ok && cudaMalloc(&c->d_win[i], c->win_bytes) == cudaSuccess;
    ok = ok && cudaEventCreate(&c->t0[i]) == cudaSuccess;
    ok = ok && cudaEventCreate(&c->done[i]) == cudaSuccess;
  }
  master->points = N;
  master->perform_inline = (N_worker_threads == 0);
  master->bins = bins;
  master->ilen = L;
  master->impulse_length = M;
  master->in_type = in_type;
  master->wcnt = 0;
  master->next_jobnum = 0;
  master->sample_index = 0;
  for (int i = 0; ok && i < ND; i++) {
    ok = ok && cudaHostAlloc((void **)&master->fdomain[i], sizeof(float complex) * (size_t)bins, cudaHostAllocPortable) ==
                   cudaSuccess;
    if (ok)
      memset(master->fdomain[i], 0, sizeof(float complex) * (size_t)bins);
    master->completed_jobs[i] = UINT_MAX; /* filter.c:214 */
  }
  master->input_buffer_size = page_round((size_t)ND * N * c->esz);
  master->input_buffer = ok ? ring_alloc(master->input_buffer_size) : NULL;
  ok = ok && master->input_buffer != NULL;
  master->fwd_plan = (fftwf_plan)c;
  if (!ok) {
    fprintf(stderr, "create_filter_input(L=%d M=%d): device/host allocation failed: %s\n", L, M,
            cudaGetErrorString(cudaGetLastError()));
    master_teardown(master);
    return -1;
  }
  /* read pointer at the start, write pointer M-1 samples in: the zero history (filter.c:243-244) */
  if (in_type == COMPLEX) {
    master->input_read_pointer.c = master->input_buffer;
    master->input_write_pointer.c = master->input_read_pointer.c + (M - 1);
    master->input_read_pointer.r = master->input_write_pointer.r = NULL;
  } else {
    master->input_read_pointer.r = master->input_buffer;
    master->input_write_pointer.r = master->input_read_pointer.r + (M - 1);
    master->input_read_pointer.c = master->input_write_pointer.c = NULL;
  }
  if (!master->init) {
    pthread_mutex_init(&master->filter_mutex, NULL);
    pthread_cond_init(&master->filter_cond, NULL);
    master->init = true;
  }
  master->owner = pthread_self();
  return 0;
}

/* ---------------------------------------------------------------- create_filter_output ------ */
/* filter.c:298-415 */
int create_filter_output(struct filter_out *slave, struct filter_in *master, int len, enum filtertype out_type) {
  if (master == NULL || slave == NULL || (out_type != SPECTRUM && len <= 0) || master->fwd_plan == NULL)
    return -1;
  if (slave->master == master && slave->olen == len && slave->out_type == out_type && slave->init)
    goto done;
  if (is_small(master))
    return small_create_output(slave, master, len, out_type);
  if (out_type == SPECTRUM)
    len = 0;
  struct master_ctx *c = (struct master_ctx *)master->fwd_plan;
  int const N = master->ilen + master->impulse_length - 1, L = master->ilen;
  if (((long)len * N % L) != 0) {
    fprintf(stderr, "Invalid filter output length %d for input N=%d, L=%d\n", len, N, L);
    return -1;
  }
  struct slave_ctx *sc = (struct slave_ctx *)slave->rev_plan;
  if (!slave->init) {
    pthread_mutex_init(&slave->response_mutex, NULL);
    slave->init = true;
  } else {
    if (slave->out_type == SPECTRUM && slave->master && slave->master->fwd_plan) {
      struct master_ctx *old = (struct master_ctx *)slave->master->fwd_plan;
      pthread_mutex_lock(&old->mu);
      spec_slave_drop(old, slave);
      pthread_mutex_unlock(&old->mu);
    }
    pthread_mutex_lock(&slave->response_mutex);
    free(slave->response);
    slave->response = NULL;
    pthread_mutex_unlock(&slave->response_mutex);
    free(slave->fdomain);
    slave->fdomain = NULL;
    if (sc) {
      free(sc->own);
      sc->own = NULL;
    }
    slave->output_buffer.c = NULL;
    slave->output_buffer.r = NULL;
    slave->output.c = NULL;
    slave->output.r = NULL;
  }
  slave->olen = len;
  slave->points = (int)((long)len * N / L);
  slave->master = master;
  slave->out_type = out_type;
  set_filter_weights(slave, 1.0, 0.0);
  pthread_mutex_lock(&c->mu);
  c->ranges_dirty = true;
  if (out_type == COMPLEX || out_type == REAL) {
    if (!sc) {
      int idx = -1;
      for (int i = 0; i < KGF_MAX_SLAVES; i++)
        if (c->slots[i] == NULL) {
          idx = i;
          break;
        }
      if (idx < 0) {
        pthread_mutex_unlock(&c->mu);
        return -1;
      }
      sc = calloc(1, sizeof *sc);
      sc->idx = idx;
      sc->ft_shift = -1000999; /* modes.c:266 */
      sc->ft_remainder = NAN;  /* modes.c:265 */
      c->slots[idx] = slave;
      if (idx + 1 > c->nslots)
        c->nslots = idx + 1;
      slave->rev_plan = (fftwf_plan)sc;
    }
    cudaStreamSynchronize(c->st);
    int const pts = kgpu_bank_define_any(c->bank, sc->idx, len, out_type == REAL ? KGPU_REAL : KGPU_COMPLEX);
    c->ver[sc->idx]++;
    pthread_mutex_unlock(&c->mu);
    if (pts != slave->points) {
      fprintf(stderr, "create_filter_output: %s\n", kgpu_last_error());
      return -1;
    }
    if (out_type == COMPLEX) { /* filter.c:345-366 */
      slave->bins = slave->points;
      sc->own = cache_aligned(sizeof(float complex) * (size_t)slave->points);
    } else { /* filter.c:372-392 */
      slave->bins = slave->points / 2 + 1;
      sc->own = cache_aligned(sizeof(float) * (size_t)slave->points);
    }
    slave->fdomain = cache_aligned(sizeof(float complex) * (size_t)slave->bins);
    if (!slave->fdomain || !sc->own)
      return -1;
    memset(sc->own, 0, (out_type == COMPLEX ? sizeof(float complex) : sizeof(float)) * (size_t)slave->points);
    if (out_type == COMPLEX) {
      slave->output_buffer.c = sc->own;
      slave->output.c = slave->output_buffer.c + slave->bins - len; /* filter.c:357 */
    } else {
      slave->output_buffer.r = sc->own;
      slave->output.r = slave->output_buffer.r + slave->points - len; /* filter.c:385 */
    }
  } else
    pthread_mutex_unlock(&c->mu);
done:;
  slave->next_jobnum = master->next_jobnum;
  return 0;
}

/* ---------------------------------------------------------------- execute_filter_input ------ */
static int grow_out(struct master_ctx *c, long need) {
  if (need <= c->out_pitch)
    return 0;
  cudaStreamSynchronize(c->st);
  long const pitch = (need + need / 4 + 1024 + 3) / 4 * 4;
  cudaFree(c->d_out);
  cudaFreeHost(c->h_out);
  c->d_out = NULL;
  c->h_out = NULL;
  c->out_pitch = 0;
  for (int i = 0; i < ND; i++)
    for (int k = 0; k < KGF_MAX_SLAVES; k++)
      c->snap[i][k].ok = false;
  if (cudaMalloc((void **)&c->d_out, sizeof(float complex) * (size_t)pitch * ND) != cudaSuccess ||
      cudaHostAlloc((void **)&c->h_out, sizeof(float complex) * (size_t)pitch * ND, cudaHostAllocPortable) != cudaSuccess)
    return -1;
  c->out_pitch = pitch;
  return 0;
}

/* The notch list belongs to the caller (radio.c:601-620) and may be edited in place: re-upload when its identity or
 * its (bin, alpha) contents change.  The EWMA state lives on the device. */
static void sync_notches(struct filter_in *f, struct master_ctx *c) {
  int bins[64];
  double alpha[64];
  int n = 0;
  unsigned h = 2166136261u;
  if (f->notches)
    for (struct notch_state *p = f->notches; n < 64; p++) { /* list ends at bin 0 (filter.c:470) */
      bins[n] = p->bin;
      alpha[n] = p->alpha;
      unsigned long long bits;
      memcpy(&bits, &p->alpha, sizeof bits);
      h = (h ^ (unsigned)p->bin) * 16777619u;
      h = (h ^ (unsigned)(bits ^ (bits >> 32))) * 16777619u;
      n++;
      if (p->bin == 0)
        break;
    }
  if (f->notches == c->notches_seen && h == c->notch_hash)
    return;
  c->notches_seen = f->notches;
  c->notch_hash = h;
  cudaStreamSynchronize(c->st);
  kgpu_master_set_notches(c->km, bins, alpha, n);
}

/* bins of the master spectrum the untouched estimate_noise() reads for each slave (radio.c:1805-1836), merged */
static void rebuild_ranges(struct filter_in *f, struct master_ctx *c) {
  c->ranges_dirty = false;
  c->nranges = 0;
  long lo[KGF_MAX_SLAVES], hi[KGF_MAX_SLAVES];
  int n = 0;
  long const m = f->bins;
  for (int i = 0; i < c->nslots; i++) {
    struct filter_out *o = c->slots[i];
    if (!o)
      continue;
    long nb = o->bins < 1000 ? 1000 : o->bins;
    if (nb > m)
      nb = m;
    long a;
    if (f->in_type == REAL) {
      a = labs((long)c->cur_shift[i]) - nb / 2;
      if (a < 0)
        a = 0;
      else if (a + nb > m)
        a = m - nb;
    } else {
      a = (long)c->cur_shift[i] - nb / 2;
      if (a < 0)
        a += m;
      else if (a >= m)
        a -= m;
      if (a < 0 || a >= m)
        continue;
      if (a + nb > m) { /* wraps: two pieces */
        lo[n] = 0;
        hi[n++] = a + nb - m;
        nb = m - a;
      }
    }
    lo[n] = a;
    hi[n++] = a + nb;
  }
  /* merge (insertion sort by lo; n <= 2 * 2048) */
  for (int i = 1; i < n; i++) {
    long const l = lo[i], h = hi[i];
    int j = i - 1;
    while (j >= 0 && lo[j] > l) {
      lo[j + 1] = lo[j];
      hi[j + 1] = hi[j];
      j--;
    }
    lo[j + 1] = l;
    hi[j + 1] = h;
  }
  for (int i = 0; i < n; i++) {
    if (c->nranges && lo[i] <= c->range_hi[c->nranges - 1] + 4096) { /* close enough: one copy */
      if (hi[i] > c->range_hi[c->nranges - 1])
        c->range_hi[c->nranges - 1] = hi[i];
    } else if (c->nranges < KGF_MAX_RANGES) {
      c->range_lo[c->nranges] = lo[i];
      c->range_hi[c->nranges++] = hi[i];
    } else { /* too fragmented: everything from here up */
      c->range_hi[c->nranges - 1] = m;
      break;
    }
  }
}

/* ---------------------------------------------------------------- ingest modes and formats -- */
/* Every raw format (enum filter_raw_format) in one row: its words, the masters it serves, its ring's zero, how the device
 * decodes it, what the device window then holds, and its block statistics. */
enum raw_path { RAW_UNPACK, RAW_AIRSPY12, RAW_IQ }; /* kgpu_unpack8 (code KGPU_RAW_*), _unpack_airspy12, _iq_apply (KGPU_IQ_*) */
enum raw_stats { STATS_NONE, STATS_INT, STATS_FLOAT }; /* none: I/Q correction, whose records replace them */
struct raw_format {
  unsigned char group; /* bytes of 8 components: 1, 2 or 4 per component, or packed-12's 8 samples in three words */
  bool real, cplx;     /* the masters it serves */
  enum raw_path path;
  int code;
  bool i16; /* the device window holds int16 words, which kgpu_forward scales, rather than floats */
  enum raw_stats stats;
  char const *why;  /* why a master it does not serve is refused */
  uint32_t zero[3]; /* the ring's zero word(s), repeated */
};
static struct raw_format const raw_formats[] = {
    [FILTER_RAW_PACKED12] = {12, true, false, RAW_AIRSPY12, 0, true, STATS_INT,
                             " (packed 12-bit needs a REAL master with L and M-1 multiples of 8)",
                             {0x80080080u, 0x08008008u, 0x00800800u}}, /* eight offset-binary 2048s (airspy-unpack.c:110-117) */
    [FILTER_RAW_U8] = {8, true, true, RAW_UNPACK, KGPU_RAW_U8, false, STATS_INT, "", {0x80808080u, 0x80808080u, 0x80808080u}},
    [FILTER_RAW_S8] = {8, true, true, RAW_UNPACK, KGPU_RAW_S8, false, STATS_INT, ""},
    [FILTER_RAW_S8_IQCORR] = {8, false, true, RAW_IQ, KGPU_IQ_S8, false, STATS_NONE, " (I/Q correction needs COMPLEX)"},
    [FILTER_RAW_S16_IQCORR] = {16, false, true, RAW_IQ, KGPU_IQ_S16, false, STATS_NONE, " (I/Q correction needs COMPLEX)"},
    [FILTER_RAW_S16] = {16, true, true, RAW_UNPACK, KGPU_RAW_S16, false, STATS_INT, ""},
    [FILTER_RAW_U16] = {16, true, false, RAW_UNPACK, KGPU_RAW_U16, false, STATS_INT, " (real)",
                        {0x80008000u, 0x80008000u, 0x80008000u}}, /* offset binary: 0x8000 is 0 */
    [FILTER_RAW_SC16Q11] = {16, false, true, RAW_UNPACK, KGPU_RAW_SC16Q11, false, STATS_INT, " (I/Q)"},
    [FILTER_RAW_F32] = {32, true, false, RAW_UNPACK, KGPU_RAW_F32, false, STATS_FLOAT, " (real)"},
    [FILTER_RAW_CF32] = {32, false, true, RAW_UNPACK, KGPU_RAW_CF32, false, STATS_FLOAT, " (I/Q)"},
    [FILTER_RAW_CF32_CNRMF] = {32, false, true, RAW_UNPACK, KGPU_RAW_CF32_CNRMF, false, STATS_FLOAT, " (I/Q)"},
    [FILTER_RAW_CF32_FSCALE] = {32, false, true, RAW_UNPACK, KGPU_RAW_CF32_FSCALE, false, STATS_FLOAT, " (I/Q)"},
};
/* the row of a format number; NULL for a number that names no format */
static struct raw_format const *format_row(int fmt) {
  return fmt >= 1 && fmt < (int)(sizeof raw_formats / sizeof *raw_formats) ? &raw_formats[fmt] : NULL;
}
/* the row of the raw format a master is fed (row 0, all zero, for the other modes) */
static struct raw_format const *fed_row(struct master_ctx const *c) { return &raw_formats[c->raw_fmt]; }
/* the device window holds int16 words (int16 ingest, or packed-12 after the unpack) rather than floats */
static bool ingest_i16(struct master_ctx const *c) { return c->mode == INGEST_INT16 || fed_row(c)->i16; }
/* the master's blocks carry A/D statistics (filter_ingest_stats) */
static bool ingest_counted(struct master_ctx const *c) {
  return c->mode == INGEST_INT16 || (c->mode == INGEST_RAW && fed_row(c)->stats != STATS_NONE);
}

static enum ingest ingest_of(struct filter_in const *f, struct master_ctx const *c) {
  return c->mode == INGEST_NONE && (f->wcnt != 0 || c->issued != 0) ? INGEST_FLOAT : c->mode;
}
/* May the master be fed mode m?  0 if it holds nothing yet or m already (for a setup, which starts m, only nothing);
 * else -1 and a message.  The caller records m in c->mode once the mode's state exists. */
static int check_mode(struct filter_in const *f, struct master_ctx const *c, enum ingest m, bool setup, char const *who) {
  static char const *const name[] = {"nothing", "floats", "int16 words", "raw words", "generated samples"};
  enum ingest const held = ingest_of(f, c);
  if (held == INGEST_NONE || (held == m && !setup))
    return 0;
  fprintf(stderr, "%s: %s on a master already fed %s\n", who, name[m], name[held]);
  return -1;
}

long filter_raw_ring_bytes(int L, int M, enum filtertype in_type, int format) {
  struct raw_format const *rf = format_row(format);
  if (rf == NULL || L <= 0 || M <= 0 || !(in_type == REAL ? rf->real : in_type == COMPLEX && rf->cplx))
    return -1;
  bool const cplx = in_type == COMPLEX;
  size_t unit = page_round(1);
  if (rf->group % 8 != 0) { /* packed-12: whole groups, so a group never straddles the end of the ring */
    if (L % 8 != 0 || (M - 1) % 8 != 0)
      return -1;
    unit = unit / (size_t)gcd((long)unit, rf->group) * rf->group;
  }
  size_t const fsz = cplx ? sizeof(float complex) : sizeof(float);
  size_t const samples = page_round((size_t)ND * (size_t)(L + M - 1) * fsz) / fsz; /* the float ring's capacity */
  size_t const need = (samples + 7) / 8 * rf->group * (cplx ? 2 : 1);
  return (long)((need + unit - 1) / unit * unit);
}

/* the first write_rawfilter on a master, or its filter_iq_correction_setup: its ring and device window */
static int raw_start(struct filter_in *f, struct master_ctx *c, int format, bool setup, char const *who) {
  long const size = filter_raw_ring_bytes(f->ilen, f->impulse_length, f->in_type, format);
  if (size < 0) {
    fprintf(stderr, "%s(L=%d M=%d): format %d cannot feed this master%s\n", who, f->ilen, f->impulse_length, format,
            raw_formats[format].why);
    return -1;
  }
  if (check_mode(f, c, INGEST_RAW, setup, who) != 0)
    return -1;
  struct raw_format const *rf = &raw_formats[format];
  size_t const group = rf->group * (f->in_type == COMPLEX ? 2u : 1u);
  if (wring_open(&c->ring, (size_t)size, group, f->impulse_length - 1, rf->zero) != 0)
    return -1;
  size_t const span = (size_t)(ND - 2) * (size_t)f->ilen + (size_t)f->points;
  if (cudaMalloc(&c->d_raw, wring_bytes(&c->ring, span)) != cudaSuccess) {
    c->d_raw = NULL;
    ring_free(c->ring.base, c->ring.size);
    c->ring.base = NULL;
    return kgf_fail("write_rawfilter: device buffer");
  }
  c->raw_fmt = format;
  c->mode = INGEST_RAW;
  return 0;
}

/* ---------------------------------------------------------------- scale changes ------------- */
/* FILTER_SCALE_CHANGES entries, S the samples of the master's float ring: every consumer reads samples from (blocks
 * issued) L - S on (the analyzer's device ring holds S samples, a window M - 1 + k L of them), so a change leaves the
 * table once S samples have been issued after it. */
static int chg_capacity(struct filter_in const *f, struct master_ctx const *c) {
  return (int)FILTER_SCALE_CHANGES((long)f->ilen, (long)(f->input_buffer_size / c->esz));
}
/* drop the changes whose samples no launch, seeding or poll can still read, folding them into chg_base */
static void chg_prune(struct filter_in const *f, struct master_ctx *c) {
  long long const oldest = (long long)f->ilen * (long long)c->issued - (long long)(f->input_buffer_size / c->esz);
  int i = 0;
  while (i < c->nchg && c->chg[i].at <= oldest)
    c->chg_base = c->chg[i++].scale;
  if (i > 0) {
    memmove(c->chg, c->chg + i, sizeof *c->chg * (size_t)(c->nchg - i));
    c->nchg -= i;
  }
}
/* the scale of the write about to be stored, whose first sample is the next one; -1 (and a message) when its change
 * would overflow the table.  Caller holds c->mu. */
static int chg_note(struct filter_in const *f, struct master_ctx *c, double scale, char const *who) {
  long long const at = (long long)f->ilen * (long long)c->issued + f->wcnt;
  if (!c->chg_started) { /* the first write: the samples before it are zeros */
    c->chg_started = true;
    c->chg_base = scale;
    return 0;
  }
  if (c->nchg > 0 && c->chg[c->nchg - 1].at == at)
    c->nchg--; /* the previous write was empty: its change covers no sample */
  if (scale == (c->nchg > 0 ? c->chg[c->nchg - 1].scale : c->chg_base))
    return 0;
  if (c->chg == NULL) {
    c->chg_cap = chg_capacity(f, c);
    c->chg = malloc(sizeof *c->chg * (size_t)c->chg_cap);
    if (!c->chg || cudaMalloc((void **)&c->d_chg, sizeof *c->chg * (size_t)c->chg_cap) != cudaSuccess ||
        cudaHostAlloc((void **)&c->h_stg, sizeof *c->chg * (size_t)c->chg_cap * (ND + 1), cudaHostAllocPortable) != cudaSuccess ||
        cudaEventCreateWithFlags(&c->stg_ev, cudaEventDisableTiming) != cudaSuccess ||
        (ingest_i16(c) && cudaMalloc((void **)&c->d_conv, c->win_bytes) != cudaSuccess)) {
      free(c->chg);
      c->chg = NULL;
      cudaFree(c->d_chg);
      c->d_chg = NULL;
      cudaFreeHost(c->h_stg);
      c->h_stg = NULL;
      if (c->stg_ev)
        cudaEventDestroy(c->stg_ev);
      c->stg_ev = NULL;
      return kgf_fail(who);
    }
  }
  if (c->nchg == c->chg_cap)
    chg_prune(f, c);
  if (c->nchg == c->chg_cap) {
    fprintf(stderr, "%s: a scale change at sample %lld would overflow the table of %d changes of the last %ld samples\n", who, at,
            c->chg_cap, (long)(f->input_buffer_size / c->esz));
    return -1;
  }
  c->chg[c->nchg].at = at;
  c->chg[c->nchg].scale = scale;
  c->nchg++;
  return 0;
}
/* samples [lo, hi): *scale that of sample lo, and the *n changes after it that fall inside, copied to d_chg on the
 * pipeline stream through staging region `stage`: a launch's first ring slot (whose previous user the launch has already
 * waited for), or ND for seedings and polls.  Caller holds c->mu. */
static int chg_span(struct master_ctx const *c, int stage, long long lo, long long hi, double *scale, int *n) {
  int i = 0;
  while (i < c->nchg && c->chg[i].at <= lo)
    i++;
  *scale = i > 0 ? c->chg[i - 1].scale : c->chg_base;
  int j = i;
  while (j < c->nchg && c->chg[j].at < hi)
    j++;
  *n = j - i;
  if (*n == 0)
    return 0;
  struct kgpu_scale_change *const stg = c->h_stg + (size_t)stage * (size_t)c->chg_cap;
  if (stage == ND && cudaEventSynchronize(c->stg_ev) != cudaSuccess) /* the previous seeding's or poll's copy has read it */
    return -1;
  memcpy(stg, c->chg + i, sizeof *c->chg * (size_t)*n);
  if (cudaMemcpyAsync(c->d_chg, stg, sizeof *c->chg * (size_t)*n, cudaMemcpyHostToDevice, c->st) != cudaSuccess)
    return -1;
  return stage == ND && cudaEventRecord(c->stg_ev, c->st) != cudaSuccess ? -1 : 0;
}

/* raw bytes on the device (history samples, then nblocks blocks of L) -> the master's device samples at d_dst: floats for
 * the 8-bit, 16-bit, float and I/Q corrected formats, int16 for packed-12, which kgpu_forward then scales.  d_stats: NULL
 * or nblocks block statistics (not for I/Q correction, whose records replace them). */
static int iq_apply(struct master_ctx const *c, void const *d_src, long long a0, long count, void *d_dst, cudaStream_t st);
static int raw_unpack(struct filter_in const *f, struct master_ctx const *c, int stage, void const *d_src, long long a0,
                      long history, int nblocks, void *d_dst, void *d_stats, cudaStream_t st) {
  int const type = f->in_type == COMPLEX ? KGPU_COMPLEX : KGPU_REAL;
  long const count = history + (long)nblocks * f->ilen;
  if (fed_row(c)->path == RAW_IQ) /* a0: the absolute index of the first sample (whose write it is) */
    return iq_apply(c, d_src, a0, count, d_dst, st);
  if (fed_row(c)->path == RAW_AIRSPY12) {
    if (kgpu_unpack_airspy12(d_src, count, d_dst, NULL, st) != 0)
      return -1;
    return d_stats ? kgpu_block_stats_i16(d_dst, type, history, f->ilen, nblocks, 0, 2047, d_stats, st) : 0;
  }
  double scale;
  int n;
  if (chg_span(c, stage, a0, a0 + count, &scale, &n) != 0)
    return -1;
  return kgpu_unpack8(d_src, fed_row(c)->code, type, history, f->ilen, nblocks, scale, n ? c->d_chg : NULL, n, a0, d_dst,
                      d_stats, st);
}

/* ---------------------------------------------------------------- I/Q correction ------------ */
/* Writes live in a ring table of iq_cap entries (write w at w % iq_cap), on the host and on the device.  It holds twice
 * the writes the raw ring can hold at FILTER_IQ_MIN_WRITE pairs each, plus the writes of the launches that may be in
 * flight: the writes of the analyzer's seeding window and those written but not yet launched both fit, so no entry is
 * overwritten while a launch or the seeding can still read it. */
long filter_iq_table_writes(int L, int M, enum filtertype in_type, int format) {
  struct raw_format const *rf = format_row(format);
  long const bytes = rf && rf->path == RAW_IQ ? filter_raw_ring_bytes(L, M, in_type, format) : -1;
  if (bytes < 0)
    return -1;
  return 2 * (bytes * 8 / (2 * rf->group) / FILTER_IQ_MIN_WRITE) + 2 * ND + 2;
}

/* the newest write among [lo, hi) whose first pair is at or before absolute pair a (lo if none) */
static unsigned long long iq_find(struct master_ctx const *c, unsigned long long lo, unsigned long long hi, long long a) {
  while (hi - lo > 1) {
    unsigned long long const mid = lo + (hi - lo) / 2;
    if (c->h_iqw[mid % (unsigned long long)c->iq_cap].first <= a)
      lo = mid;
    else
      hi = mid;
  }
  return lo;
}
/* the oldest write the table still holds, of the first `upto` */
static unsigned long long iq_oldest(struct master_ctx const *c, unsigned long long upto) {
  return upto > (unsigned long long)c->iq_cap ? upto - (unsigned long long)c->iq_cap : 0;
}

/* corrected floats of pairs [a0, a0 + count) from their raw words at d_src, into d_dst; every write they lie in has
 * been sent to the device (c->iq_sent) and its predecessor scanned */
static int iq_apply(struct master_ctx const *c, void const *d_src, long long a0, long count, void *d_dst, cudaStream_t st) {
  unsigned long long w_lo = 0, w_hi = 0;
  if (a0 + count > 0 && c->iq_sent > 0) {
    unsigned long long const old = iq_oldest(c, c->iq_sent);
    w_lo = iq_find(c, old, c->iq_sent, a0 > 0 ? a0 : 0);
    w_hi = iq_find(c, old, c->iq_sent, a0 + count - 1);
  }
  return kgpu_iq_apply(d_src, fed_row(c)->code, a0, count, c->d_iqw, c->d_iqc, c->iq_cap, (long long)w_lo,
                       (int)(w_hi - w_lo + 1), d_dst, st);
}

/* the table entries, moments and records of the k blocks about to be issued (new pairs [issued L, (issued + k) L)),
 * whose raw window is in d_raw, on the pipeline stream; the apply follows in raw_unpack */
static int iq_launch(struct filter_in const *f, struct master_ctx *c, int k) {
  long long const a = (long long)f->ilen * (long long)c->issued, end = a + (long long)k * f->ilen;
  unsigned long long const cap = (unsigned long long)c->iq_cap, old = iq_oldest(c, c->iq_writes);
  unsigned long long const last = iq_find(c, old, c->iq_writes, end - 1); /* the write of the launch's last pair */
  for (unsigned long long w = c->iq_sent; w <= last;) { /* the writes that start in this launch */
    unsigned long long const n = last + 1 - w < cap - w % cap ? last + 1 - w : cap - w % cap;
    if (cudaMemcpyAsync(c->d_iqw + w % cap, c->h_iqw + w % cap, sizeof *c->h_iqw * (size_t)n, cudaMemcpyHostToDevice, c->st) !=
        cudaSuccess)
      return -1;
    w += n;
  }
  c->iq_sent = last + 1;
  unsigned long long const first = iq_find(c, old, c->iq_writes, a);
  char const *d_new = (char const *)c->d_raw + wring_bytes(&c->ring, (size_t)(f->impulse_length - 1));
  if (kgpu_iq_moments(d_new, fed_row(c)->code, a, (long)(end - a), c->d_iqw, c->iq_cap, (long long)first, (int)(last - first + 1),
                      c->st) != 0)
    return -1;
  struct kgpu_iq_write const *lw = &c->h_iqw[last % cap];
  unsigned long long const done = lw->first + lw->n <= end ? last + 1 : last; /* writes complete at the launch's end */
  c->iq_rec_from = c->iq_scanned;
  if (kgpu_iq_scan(c->d_iqw, c->d_iqc, c->iq_cap, (long long)c->iq_scanned, (int)(done - c->iq_scanned), &c->iq_par, c->d_iqr,
                   c->st) != 0)
    return -1;
  c->iq_scanned = done;
  return 0;
}

/* the block statistics of job c->folded into c->acc (its slot's device work has completed) */
static void fold_one(struct filter_in const *f, struct master_ctx *c) {
  struct kgpu_block_stats const *s = &c->h_bstats[c->folded % ND];
  c->acc.blocks++;
  c->acc.samples += (uint64_t)f->ilen;
  if (fed_row(c)->stats == STATS_FLOAT)
    c->acc.fenergy += s->fenergy;
  else
    c->acc.energy += s->energy;
  c->acc.overranges += s->overs;
  c->acc.overrange_samples += s->over_samples;
  c->acc.since_over = s->over_samples ? 0 : c->acc.since_over + (uint64_t)f->ilen;
  c->folded++;
}

/* the generated energy of job c->gen_folded into c->gen_acc (its slot's device work has completed) */
static void gen_fold_one(struct filter_in const *f, struct master_ctx *c) {
  c->gen_acc.blocks++;
  c->gen_acc.samples += (uint64_t)f->ilen;
  c->gen_acc.energy += c->h_gen_energy[c->gen_folded % ND];
  c->gen_folded++;
}

/* the generator's floats of samples [a0, a0 + count) at d_out (kgpu_siggen_generate's arguments), from the envelope
 * at d_mod (one float per sample of the window) on a modulated master */
static int gen_window(struct master_ctx *c, long long a0, long count, double scale, struct kgpu_scale_change const *chg,
                      int nchg, void *d_out, float const *d_mod, double *d_energy, int nblocks, long L, long history) {
  return c->gen_mod ? kgpu_siggen_generate_mod(c->gen, a0, count, scale, chg, nchg, d_out, d_mod, d_energy, nblocks, L,
                                               history, c->st)
                    : kgpu_siggen_generate(c->gen, a0, count, scale, chg, nchg, d_out, d_energy, nblocks, L, history, c->st);
}

/* ---------------------------------------------------------------- spectrum device ring ------ */
/* n samples of esz bytes from a ring (src_cap samples, position src) to the device ring at position dst, both modular */
static int sring_copy(struct master_ctx *c, char const *src_base, long src_cap, long src, long dst, long n, size_t esz,
                      enum cudaMemcpyKind kind) {
  while (n > 0) {
    long len = n;
    if (len > src_cap - src)
      len = src_cap - src;
    if (len > c->sring_cap - dst)
      len = c->sring_cap - dst;
    if (cudaMemcpyAsync((char *)c->d_sring + (size_t)dst * esz, src_base + (size_t)src * esz, (size_t)len * esz, kind,
                        c->st) != cudaSuccess)
      return -1;
    n -= len;
    src = (src + len) % src_cap;
    dst = (dst + len) % c->sring_cap;
  }
  return 0;
}
/* (Re)create the device ring in the master's current ingest format and seed it from the host ring: the sring_cap samples
 * up to the end of the last issued block.  Caller holds c->mu. */
static int sring_seed(struct filter_in *f, struct master_ctx *c) {
  cudaStreamSynchronize(c->st);
  cudaFree(c->d_sring);
  c->d_sring = NULL;
  c->sring_i16 = ingest_i16(c);
  c->sring_cap = (long)(f->input_buffer_size / c->esz);
  size_t const esz = c->sring_i16 ? (f->in_type == COMPLEX ? 2 * sizeof(int16_t) : sizeof(int16_t)) : c->esz;
  if (cudaMalloc(&c->d_sring, (size_t)c->sring_cap * esz) != cudaSuccess) {
    c->d_sring = NULL;
    return kgf_fail("filter_spectrum_setup: device ring");
  }
  long const M1 = f->impulse_length - 1, n = c->sring_cap;
  c->sring_pos = (long)((M1 + (unsigned long long)f->ilen * c->issued) % (unsigned long long)c->sring_cap);
  long const dst = c->sring_pos, first = n - dst;                 /* (sring_pos - n) modulo sring_cap, n being sring_cap */
  long long const a0 = (long long)f->ilen * (long long)c->issued - n; /* the absolute index of the first seeded sample */
  struct word_ring const *r = &c->ring;
  int rc = 0;
  switch (c->mode) {
  case INGEST_GEN: { /* the host float ring holds nothing: generate the last sring_cap samples again */
    double scale;
    int nc;
    rc = chg_span(c, ND, a0, a0 + n, &scale, &nc);
    struct kgpu_scale_change const *chg = nc ? c->d_chg : NULL;
    float *mod = NULL; /* modulated: those samples' envelope, sent over from the envelope ring */
    if (rc == 0 && c->gen_mod) {
      long const cap = wring_samples(r, r->size), end = wring_samples(r, (size_t)(r->rp - r->base)) + M1;
      long const src = ((end - n) % cap + cap) % cap;
      rc = cudaMalloc((void **)&mod, wring_bytes(r, (size_t)n)) == cudaSuccess ? 0 : -1;
      rc = rc ? rc : window_h2d(mod, r->base + wring_bytes(r, (size_t)src), wring_bytes(r, (size_t)n), r->base, r->size, c->st);
    }
    rc = rc ? rc : gen_window(c, a0, first, scale, chg, nc, (char *)c->d_sring + (size_t)dst * esz, mod, NULL, 0, 0, first);
    if (rc == 0 && dst > 0)
      rc = gen_window(c, a0 + first, dst, scale, chg, nc, c->d_sring, mod ? mod + first : NULL, NULL, 0, 0, dst);
    if (cudaStreamSynchronize(c->st) != cudaSuccess)
      rc = -1;
    cudaFree(mod);
    return rc ? kgf_fail("filter_spectrum_setup: generating the device ring") : 0;
  }
  case INGEST_RAW: { /* the host ring holds raw bytes: send the last sring_cap samples' bytes over and unpack them there */
    long const cap = wring_samples(r, r->size), end = wring_samples(r, (size_t)(r->rp - r->base)) + M1;
    long const src = ((end - n) % cap + cap) % cap;
    void *tmp = NULL;
    rc = cudaMalloc(&tmp, wring_bytes(r, (size_t)n)) == cudaSuccess ? 0 : -1;
    rc = rc ? rc : window_h2d(tmp, r->base + wring_bytes(r, (size_t)src), wring_bytes(r, (size_t)n), r->base, r->size, c->st);
    rc = rc ? rc : raw_unpack(f, c, ND, tmp, a0, first, 0, (char *)c->d_sring + (size_t)dst * esz, NULL, c->st);
    if (rc == 0 && dst > 0)
      rc = raw_unpack(f, c, ND, (char *)tmp + wring_bytes(r, (size_t)first), a0 + first, dst, 0, c->d_sring, NULL, c->st);
    if (cudaStreamSynchronize(c->st) != cudaSuccess)
      rc = -1;
    cudaFree(tmp);
    return rc ? kgf_fail("filter_spectrum_setup: seeding the device ring from the raw ring") : 0;
  }
  default: { /* int16 words or floats: the samples as they are (the int16 ring holds at least as many as the float ring) */
    bool const words = c->mode == INGEST_INT16;
    char const *const base = words ? r->base : (char const *)f->input_buffer;
    char const *const rp =
        words ? r->rp : f->in_type == COMPLEX ? (char const *)f->input_read_pointer.c : (char const *)f->input_read_pointer.r;
    long const src_cap = words ? wring_samples(r, r->size) : c->sring_cap;
    long const src_end = (long)((size_t)(rp - base) / esz) + M1;
    long const src = ((src_end - n) % src_cap + src_cap) % src_cap;
    if (sring_copy(c, base, src_cap, src, dst, n, esz, cudaMemcpyHostToDevice) != 0 ||
        cudaStreamSynchronize(c->st) != cudaSuccess)
      return kgf_fail("filter_spectrum_setup: seeding the device ring");
    return 0;
  }
  }
}
/* the k*L new samples of the launch just issued from d_win[slot] (after its M-1 history samples), on the pipeline stream */
static int sring_append(struct filter_in *f, struct master_ctx *c, int k) {
  if (c->sring_i16 != ingest_i16(c)) { /* the ingest format changed: the next poll seeds a new ring */
    cudaStreamSynchronize(c->st);
    cudaFree(c->d_sring);
    c->d_sring = NULL;
    return 0;
  }
  size_t const esz = c->sring_i16 ? (f->in_type == COMPLEX ? 2 * sizeof(int16_t) : sizeof(int16_t)) : c->esz;
  long const n = (long)k * f->ilen;
  void const *win = c->d_win[f->next_jobnum % ND];
  if (sring_copy(c, (char const *)win + (size_t)(f->impulse_length - 1) * esz, LONG_MAX, 0, c->sring_pos, n, esz,
                 cudaMemcpyDeviceToDevice) != 0)
    return kgf_fail("execute_filter_input: spectrum ring append");
  c->sring_pos = (c->sring_pos + n) % c->sring_cap;
  return 0;
}

/* The forward pass's input for the k blocks about to be issued from ring slot `slot`, in stages on the pipeline stream:
 * H2D of the window (floats or int16 words into d_win[slot], raw words into d_raw), I/Q correction's launch, generation,
 * unpack, int16 statistics into bst (NULL: none), and the conversion of an int16 window that holds more than one scale. */
static int launch_input(struct filter_in *f, struct master_ctx *c, int slot, int k, struct kgpu_block_stats *bst,
                        void const **fwd_in, int *fmt, float *scale) {
  int const type = f->in_type == COMPLEX ? KGPU_COMPLEX : KGPU_REAL;
  long const M1 = f->impulse_length - 1;
  size_t const span = (size_t)(k - 1) * (size_t)f->ilen + (size_t)f->points; /* samples covered by k overlapping windows */
  long long const a0 = (long long)f->ilen * (long long)c->issued - M1;     /* the window's first sample */
  void *const win = c->d_win[slot];
  *fwd_in = win;
  *fmt = ingest_i16(c) ? KGPU_FMT_I16 : KGPU_FMT_F32; /* packed-12 goes on as int16 with the drivers' float scale */
  *scale = 1.0f;
  if (c->chg)
    chg_prune(f, c);
  if (c->mode == INGEST_NONE) { /* floats */
    void **const rp = f->in_type == COMPLEX ? (void **)&f->input_read_pointer.c : (void **)&f->input_read_pointer.r;
    char const *const src = *rp;
    *rp = (char *)*rp + c->esz * (size_t)f->ilen * (size_t)k;
    kgf_ring_wrap(rp, f->input_buffer, f->input_buffer_size);
    if (window_h2d(win, src, c->esz * span, f->input_buffer, f->input_buffer_size, c->st) != 0)
      return kgf_fail("execute_filter_input: H2D of the window");
    return 0;
  }
  double s;
  int n;
  if (c->mode == INGEST_GEN) { /* generated on the device: only a modulated master's envelope crosses PCIe */
    if (c->gen_mod && window_h2d(c->d_raw, wring_advance(&c->ring, (size_t)f->ilen * (size_t)k), wring_bytes(&c->ring, span),
                                 c->ring.base, c->ring.size, c->st) != 0)
      return kgf_fail("execute_filter_input: H2D of the envelope");
    if (chg_span(c, slot, a0, a0 + (long long)span, &s, &n) != 0 ||
        gen_window(c, a0, (long)span, s, n ? c->d_chg : NULL, n, win, c->d_raw, c->gen_stats_on ? c->d_gen_energy + slot : NULL,
                   k, f->ilen, M1) != 0)
      return kgf_fail("execute_filter_input: generating the window");
    return 0;
  }
  bool const raw = c->mode == INGEST_RAW;
  char const *const src = wring_advance(&c->ring, (size_t)f->ilen * (size_t)k);
  if (window_h2d(raw ? c->d_raw : win, src, wring_bytes(&c->ring, span), c->ring.base, c->ring.size, c->st) != 0)
    return kgf_fail("execute_filter_input: H2D of the window");
  if (raw && fed_row(c)->path == RAW_IQ && iq_launch(f, c, k) != 0)
    return kgf_fail("execute_filter_input: I/Q correction");
  if (raw && raw_unpack(f, c, slot, c->d_raw, a0, M1, k, win, bst, c->st) != 0)
    return kgf_fail("execute_filter_input: raw unpack");
  if (!raw && bst && kgpu_block_stats_i16(win, type, M1, f->ilen, k, c->i16_derand, 32767, bst, c->st) != 0)
    return kgf_fail("execute_filter_input: kgpu_block_stats_i16");
  if (*fmt != KGPU_FMT_I16)
    return 0;
  if (chg_span(c, slot, a0, a0 + (long long)span, &s, &n) != 0)
    return kgf_fail("execute_filter_input: scale changes");
  if (n == 0) { /* one scale: fwd_cols converts; more: floats with each sample's own scale */
    *scale = (float)s;
    return 0;
  }
  if (kgpu_scale_i16(win, type, (long)span, a0, s, c->d_chg, n, c->i16_derand, c->d_conv, c->st) != 0)
    return kgf_fail("execute_filter_input: kgpu_scale_i16");
  *fwd_in = c->d_conv;
  *fmt = KGPU_FMT_F32;
  return 0;
}

/* k consecutive blocks (jobs next_jobnum .. +k-1, ring slots without wrap) as one device launch sequence.
 * filter.c:558-651 (+ run_fft :485-555) */
static int execute_filter_input_n(struct filter_in *const f, int const k) {
  if (is_small(f))
    return small_execute(f, k);
  struct master_ctx *c = (struct master_ctx *)f->fwd_plan;
  pthread_mutex_lock(&c->mu);
  unsigned const jobnum = f->next_jobnum;
  int const slot = (int)(jobnum % ND);
  /* the ring slots' previous occupants (job - ND) must have drained */
  for (int j = 0; j < k; j++)
    cudaEventSynchronize(c->done[slot + j]);
  if (c->stats_on && !ingest_counted(c))
    c->stats_on = false; /* fed floats (the driver counts in its own loop), generated or I/Q corrected */
  while (c->stats_on && c->folded + ND < c->issued + (unsigned long long)k)
    fold_one(f, c); /* the statistics of the slots about to be reused */
  while (c->gen_stats_on && c->gen_folded + ND < c->issued + (unsigned long long)k)
    gen_fold_one(f, c);
  bool const iq = fed_row(c)->path == RAW_IQ;
  while (iq && c->iq_checked + ND < c->issued + (unsigned long long)k)
    c->iq_avail = c->iq_job_done[c->iq_checked++ % ND]; /* the records of the slots about to be reused have arrived */
  struct kgpu_block_stats *const bst = c->stats_on ? c->d_bstats + slot : NULL;
  if (c->timed[slot]) { /* forward+channels device time of that older job, for main.c:154-164 */
    float ms = 0;
    if (cudaEventElapsedTime(&ms, c->t0[slot], c->done[slot]) == cudaSuccess) {
      int64_t const ns = (int64_t)(ms * 1e6f);
      if (ns > Max_fft_time)
        Max_fft_time = ns;
      if (ns < Min_fft_time)
        Min_fft_time = ns;
      int64_t const dev = ns - Avg_fft_time;
      Avg_fft_time += dev >> 4;
      Mean_dev += (llabs(dev) - Mean_dev) >> 4;
    }
  }
  sync_notches(f, c);
  cudaEventRecord(c->t0[slot], c->st);
  float complex *spec = c->d_spec + (size_t)slot * (size_t)c->spec_stride;
  for (int j = 0; j < k; j++) /* nothing of the previous occupants may be served for these jobs */
    for (int i = 0; i < c->nslots; i++)
      c->snap[slot + j][i].ok = false;
  void const *fwd_in;
  int fmt;
  float scale;
  int rc = launch_input(f, c, slot, k, bst, &fwd_in, &fmt, &scale);
  if (rc == 0 && kgpu_forward(c->km, fwd_in, fmt, scale, fmt == KGPU_FMT_I16 && c->i16_derand, k, spec, NULL, c->st) != 0)
    rc = kgf_fail("execute_filter_input: kgpu_forward");
  if (rc == 0 && c->d_sring)
    rc = sring_append(f, c, k);
  c->issued += (unsigned long long)k;
  if (rc == 0 && f->notches && kgpu_apply_notches(c->km, spec, k, c->st) != 0)
    rc = kgf_fail("execute_filter_input: kgpu_apply_notches");
  /* every slave, batched, with the shift it used last (radio.c:1491: shifts move only on retune) */
  if (rc == 0 && c->nslots > 0) {
    kgpu_bank_set_block_counter(c->bank, (long)jobnum);
    if (kgpu_bank_commit(c->bank, c->st) != 0)
      rc = kgf_fail("execute_filter_input: kgpu_bank_commit");
    long const stride = rc == 0 ? kgpu_bank_out_stride(c->bank) : 0;
    if (rc == 0 && stride > 0) {
      if (grow_out(c, stride) != 0)
        rc = kgf_fail("execute_filter_input: output buffers");
      float complex *d_row = c->d_out + (size_t)slot * (size_t)c->out_pitch;
      float complex *h_row = c->h_out + (size_t)slot * (size_t)c->out_pitch;
      if (rc == 0 && kgpu_bank_run_ex(c->bank, spec, k, d_row, c->out_pitch, c->d_pw + (size_t)slot * KGF_MAX_SLAVES, c->st) != 0)
        rc = kgf_fail("execute_filter_input: kgpu_bank_run");
      if (rc == 0 && c->noise_on &&
          kgpu_bank_noise(c->bank, spec, k, c->noise_samprate, c->d_n0 + (size_t)slot * KGF_MAX_SLAVES, c->st) != 0)
        rc = kgf_fail("execute_filter_input: kgpu_bank_noise");
      if (rc == 0) { /* device->host copies on their own stream: they overlap the next launch's H2D and kernels */
        cudaEventRecord(c->kev, c->st);
        cudaStreamWaitEvent(c->st_d2h, c->kev, 0);
        size_t const row_bytes = sizeof(float complex) * ((size_t)(k - 1) * (size_t)c->out_pitch + (size_t)stride);
        if (cudaMemcpyAsync(h_row, d_row, row_bytes, cudaMemcpyDeviceToHost, c->st_d2h) != cudaSuccess ||
            cudaMemcpyAsync(c->h_pw + (size_t)slot * KGF_MAX_SLAVES, c->d_pw + (size_t)slot * KGF_MAX_SLAVES,
                            sizeof(float) * (size_t)k * KGF_MAX_SLAVES, cudaMemcpyDeviceToHost, c->st_d2h) != cudaSuccess ||
            (c->noise_on &&
             cudaMemcpyAsync(c->h_n0 + (size_t)slot * KGF_MAX_SLAVES, c->d_n0 + (size_t)slot * KGF_MAX_SLAVES,
                             sizeof(double) * (size_t)k * KGF_MAX_SLAVES, cudaMemcpyDeviceToHost, c->st_d2h) != cudaSuccess))
          rc = kgf_fail("execute_filter_input: D2H of the channel outputs");
      }
      if (rc == 0)
        for (int i = 0; i < c->nslots; i++) {
          struct filter_out *o = c->slots[i];
          if (!o || (o->out_type != COMPLEX && o->out_type != REAL) || !o->response)
            continue;
          struct slave_ctx *sc = (struct slave_ctx *)o->rev_plan;
          long const off = kgpu_bank_out_offset(c->bank, i);
          for (int j = 0; j < k; j++) {
            struct snap *s = &c->snap[slot + j][i];
            s->shift = c->cur_shift[i];
            s->isb = c->cur_isb[i];
            s->beam = c->cur_beam[i];
            s->alpha = c->cur_alpha[i];
            s->beta = c->cur_beta[i];
            s->off = off;
            s->ver = c->ver[i];
            s->ft_ver = sc ? sc->ft_ver : 0;
            s->ok = true;
          }
        }
    }
  }
  cudaEventRecord(c->kev, c->st);
  cudaStreamWaitEvent(c->st_d2h, c->kev, 0);
  if (rc == 0 && bst && cudaMemcpyAsync(c->h_bstats + slot, bst, sizeof *bst * (size_t)k, cudaMemcpyDeviceToHost, c->st_d2h) != cudaSuccess)
    rc = kgf_fail("execute_filter_input: D2H of the A/D statistics");
  if (rc == 0 && c->gen_stats_on &&
      cudaMemcpyAsync(c->h_gen_energy + slot, c->d_gen_energy + slot, sizeof(double) * (size_t)k, cudaMemcpyDeviceToHost,
                      c->st_d2h) != cudaSuccess)
    rc = kgf_fail("execute_filter_input: D2H of the generated energies");
  if (iq) {
    unsigned long long const from = c->iq_rec_from, to = c->iq_scanned;
    for (unsigned long long w = from; rc == 0 && w < to;) { /* the records of the writes this launch completed */
      unsigned long long const n = to - w < (unsigned long long)c->iq_cap - w % (unsigned long long)c->iq_cap
                                       ? to - w
                                       : (unsigned long long)c->iq_cap - w % (unsigned long long)c->iq_cap;
      size_t const at = (size_t)(w % (unsigned long long)c->iq_cap);
      if (cudaMemcpyAsync(c->h_iqr + at, c->d_iqr + at, sizeof *c->h_iqr * (size_t)n, cudaMemcpyDeviceToHost, c->st_d2h) !=
          cudaSuccess)
        rc = kgf_fail("execute_filter_input: D2H of the I/Q records");
      w += n;
    }
    for (int j = 0; j < k; j++)
      c->iq_job_done[slot + j] = to;
  }
  if (rc == 0 && c->spectrum_d2h) {
    if (c->spectrum_d2h == 1 && c->ranges_dirty)
      rebuild_ranges(f, c);
    for (int j = 0; j < k; j++) {
      float complex const *sp = spec + (size_t)j * (size_t)c->spec_stride;
      if (c->spectrum_d2h == 2) {
        if (cudaMemcpyAsync(f->fdomain[slot + j], sp, sizeof(float complex) * (size_t)f->bins, cudaMemcpyDeviceToHost,
                            c->st_d2h) != cudaSuccess)
          rc = kgf_fail("execute_filter_input: D2H of the spectrum");
      } else
        for (int r = 0; r < c->nranges; r++)
          if (cudaMemcpyAsync(f->fdomain[slot + j] + c->range_lo[r], sp + c->range_lo[r],
                              sizeof(float complex) * (size_t)(c->range_hi[r] - c->range_lo[r]), cudaMemcpyDeviceToHost,
                              c->st_d2h) != cudaSuccess)
            rc = kgf_fail("execute_filter_input: D2H of the spectrum windows");
    }
  }
  for (int j = 0; j < k; j++) {
    cudaEventRecord(c->done[slot + j], c->st_d2h);
    c->timed[slot + j] = (j == 0);
  }
  pthread_mutex_unlock(&c->mu);

  pthread_mutex_lock(&f->filter_mutex);
  f->owner = pthread_self();
  for (int j = 0; j < k; j++) {
    f->samples_by_job[slot + j] = f->sample_index;
    f->completed_jobs[slot + j] = jobnum + (unsigned)j; /* "complete" == issued; consumers wait on the slot's event */
    f->sample_index += (uint64_t)f->ilen;
  }
  f->next_jobnum += (unsigned)k;
  pthread_cond_broadcast(&f->filter_cond);
  pthread_mutex_unlock(&f->filter_mutex);
  if (f->perform_inline)
    cudaEventSynchronize(c->done[slot + k - 1]);
  return rc;
}

int execute_filter_input(struct filter_in *const f) {
  if (f == NULL || f->fwd_plan == NULL)
    return -1;
  return execute_filter_input_n(f, 1);
}

/* as many launches as the ready blocks need: up to ND-1 blocks each, never across the end of the ND-slot ring */
static int fire_ready_blocks(struct filter_in *f) {
  int fired = 0;
  while (f->wcnt >= f->ilen) {
    int k = f->wcnt / f->ilen;
    int const to_wrap = ND - (int)(f->next_jobnum % ND);
    if (k > ND - 1)
      k = ND - 1;
    if (k > to_wrap)
      k = to_wrap;
    f->wcnt -= k * f->ilen;
    execute_filter_input_n(f, k);
    fired = 1;
  }
  return fired;
}

/* ---------------------------------------------------------------- execute_filter_output ----- */
static int ensure_one(struct master_ctx *c, int olen) {
  if (olen <= c->one_cap)
    return 0;
  cudaStreamSynchronize(c->st_one);
  cudaFree(c->d_one);
  cudaFreeHost(c->h_one);
  c->d_one = NULL;
  c->h_one = NULL;
  c->one_cap = 0;
  if (cudaMalloc((void **)&c->d_one, sizeof(float complex) * (size_t)olen) != cudaSuccess ||
      cudaHostAlloc((void **)&c->h_one, sizeof(float complex) * (size_t)olen, cudaHostAllocPortable) != cudaSuccess)
    return -1;
  c->one_cap = olen;
  return 0;
}

static void own_output(struct filter_out *slave, struct slave_ctx *sc) { /* point the slave back at its private buffer */
  if (slave->out_type == REAL) {
    slave->output_buffer.r = sc->own;
    slave->output.r = slave->output_buffer.r + slave->points - slave->olen;
  } else {
    slave->output_buffer.c = sc->own;
    slave->output.c = slave->output_buffer.c + slave->bins - slave->olen;
  }
}

/* wait / lap logic of filter.c:680-707; returns 1 = lapped (zeros delivered), 0 = job taken, -1 error */
static int take_job(struct filter_out *slave, struct filter_in *master, unsigned *job_out) {
  pthread_mutex_lock(&master->filter_mutex);
  if (pthread_equal(master->owner, pthread_self())) {
    slave->next_jobnum = master->next_jobnum - 1; /* same thread wrote the input: take the latest (filter.c:681-683) */
  } else {
    while ((int)(slave->next_jobnum - master->completed_jobs[slave->next_jobnum % ND]) > 0)
      pthread_cond_wait(&master->filter_cond, &master->filter_mutex);
    int const behind = (int)(master->completed_jobs[slave->next_jobnum % ND] - slave->next_jobnum);
    if (behind >= ND) { /* lapped: a block of zeros and a drop (filter.c:690-701) */
      pthread_mutex_unlock(&master->filter_mutex);
      slave->block_drops++;
      slave->next_jobnum++;
      struct slave_ctx *sc = (struct slave_ctx *)slave->rev_plan;
      if (sc && sc->own) {
        own_output(slave, sc);
        memset(sc->own, 0, (slave->out_type == REAL ? sizeof(float) : sizeof(float complex)) * (size_t)slave->points);
      }
      if (sc && sc->nb) {
        struct master_ctx *c = (struct master_ctx *)master->fwd_plan;
        pthread_mutex_lock(&c->mu);
        int const rc = nb_append(sc, NULL, slave->olen, c->st);
        pthread_mutex_unlock(&c->mu);
        if (rc != 0)
          return -1;
      }
      return 1;
    }
  }
  *job_out = slave->next_jobnum;
  slave->sample_index = master->samples_by_job[*job_out % ND];
  slave->next_jobnum++;
  pthread_mutex_unlock(&master->filter_mutex);
  return 0;
}

/* push the slave's current parameters into the bank; c->mu held */
static void push_params(struct master_ctx *c, struct filter_out *slave, int i, int shift) {
  c->cur_shift[i] = shift;
  c->cur_isb[i] = slave->isb;
  c->cur_beam[i] = slave->beam;
  c->cur_alpha[i] = slave->alpha;
  c->cur_beta[i] = slave->beta;
  c->ranges_dirty = true;
  kgpu_bank_set_shift(c->bank, i, shift);
  kgpu_bank_set_flags(c->bank, i, (slave->isb ? KGPU_CHAN_ISB : 0) | (slave->beam ? KGPU_CHAN_BEAM : 0));
  kgpu_bank_set_weights(c->bank, i, creal(slave->alpha), cimag(slave->alpha), creal(slave->beta), cimag(slave->beta));
}

/* Deliver job `job` to the slave: from the batch if the batched launch used exactly these parameters, else recomputed
 * alone.  filter.c:703-921 */
static int deliver(struct filter_out *slave, struct master_ctx *c, unsigned job, int shift) {
  struct slave_ctx *sc = (struct slave_ctx *)slave->rev_plan;
  int const slot = (int)(job % ND), i = sc->idx;
  size_t const obytes = (slave->out_type == REAL ? sizeof(float) : sizeof(float complex)) * (size_t)slave->olen;
  int rc = 0;
  pthread_mutex_lock(&c->mu);
  struct snap const *s = &c->snap[slot][i];
  bool const hit = s->ok && s->shift == shift && s->ver == c->ver[i] && s->isb == slave->isb && s->beam == slave->beam &&
                   s->ft_ver == sc->ft_ver && (!slave->beam || (s->alpha == slave->alpha && s->beta == slave->beta));
  if (hit) {
    void const *src = c->h_out + (size_t)slot * (size_t)c->out_pitch + s->off;
    sc->last_power = c->h_pw[(size_t)slot * KGF_MAX_SLAVES + i];
    sc->last_n0 = c->h_n0[(size_t)slot * KGF_MAX_SLAVES + i];
    /* the device row of h_out's copy, enqueued before the producer can issue job + ND into it (it issues under c->mu) */
    if (sc->nb)
      rc = nb_append(sc, c->d_out + (size_t)slot * (size_t)c->out_pitch + s->off, slave->olen, c->st);
    pthread_mutex_unlock(&c->mu);
    if (rc != 0)
      return rc;
    if (c->zero_copy) { /* the pinned row stays untouched until job + ND is issued */
      if (slave->out_type == REAL)
        slave->output.r = (float *)src;
      else
        slave->output.c = (float complex *)src;
    } else {
      own_output(slave, sc);
      memcpy(slave->out_type == REAL ? (void *)slave->output.r : (void *)slave->output.c, src, obytes);
    }
    return 0;
  }
  /* this slave's parameters moved after the block was issued (or it is new): redo it alone
   * from the block's spectrum, and let the next batched launches use the new values */
  cudaStreamSynchronize(c->st);
  push_params(c, slave, i, shift);
  float complex const *spec = c->d_spec + (size_t)slot * (size_t)c->spec_stride;
  long const saved = kgpu_bank_block_counter(c->bank);
  kgpu_bank_set_block_counter(c->bank, (long)job);
  if (ensure_one(c, slave->olen) != 0)
    rc = kgf_fail("execute_filter_output: scratch allocation");
  else if (kgpu_bank_run_one_ex(c->bank, i, spec, c->d_one, c->d_one_pw, c->st_one) != 0)
    rc = kgf_fail("execute_filter_output: kgpu_bank_run_one");
  else if (nb_append(sc, c->d_one, slave->olen, c->st_one) != 0) /* d_one is reused by the next recompute */
    rc = -1;
  else if (cudaMemcpyAsync(c->h_one, c->d_one, obytes, cudaMemcpyDeviceToHost, c->st_one) != cudaSuccess ||
           cudaMemcpyAsync(c->h_one_pw, c->d_one_pw, sizeof(float), cudaMemcpyDeviceToHost, c->st_one) != cudaSuccess ||
           cudaStreamSynchronize(c->st_one) != cudaSuccess)
    rc = kgf_fail("execute_filter_output: D2H of the recomputed channel");
  else {
    own_output(slave, sc);
    memcpy(slave->out_type == REAL ? (void *)slave->output.r : (void *)slave->output.c, c->h_one, obytes);
    sc->last_power = *c->h_one_pw;
    sc->last_n0 = NAN; /* not recomputed for a single retuned block; the next batched block has it */
  }
  kgpu_bank_set_block_counter(c->bank, saved);
  pthread_mutex_unlock(&c->mu);
  return rc;
}

/* Deliver job `job` of a small master to the slave: from the launch's output row if it used exactly these parameters,
 * else that slave recomputed alone from the job's stored spectrum into its run of the row.  filter.c:703-921 */
static int small_deliver(struct filter_out *slave, unsigned job, int shift) {
  struct small_ctx *c = (struct small_ctx *)slave->master->fwd_plan;
  if (cudaEventSynchronize(c->done[job % ND]) != cudaSuccess)
    return kgf_fail("execute_filter_output: waiting for the block");
  struct slave_ctx *sc = (struct slave_ctx *)slave->rev_plan;
  if (sc == NULL || sc->own == NULL)
    return -1;
  if (slave->beam)
    return small_refuses("execute_filter_output (beam)");
  if (slave->response == NULL) /* no filter yet: leave the output alone (filter.c:715-718) */
    return 0;
  int const slot = (int)(job % ND), i = sc->idx;
  size_t const obytes = (slave->out_type == REAL ? sizeof(float) : sizeof(float complex)) * (size_t)slave->olen;
  int rc = 0;
  pthread_mutex_lock(&c->mu);
  struct snap *s = &c->snap[slot][i];
  if (!(s->ok && s->shift == shift && s->ver == c->ver[i] && s->isb == slave->isb)) {
    c->cur_shift[i] = shift; /* the next launches use them too */
    c->cur_isb[i] = slave->isb;
    long const off = kgpu_small_out_offset(c->ks, i);
    float complex *d_row = c->d_out + (size_t)slot * (size_t)c->out_pitch;
    if (kgpu_small_set_slave(c->ks, i, shift, slave->isb) != 0 ||
        kgpu_small_run(c->ks, NULL, 1, c->d_spec + (size_t)slot * (size_t)c->spec_stride, d_row, c->out_pitch, i, c->st) != 0 ||
        cudaMemcpyAsync(c->h_out + (size_t)slot * (size_t)c->out_pitch + off, d_row + off, obytes, cudaMemcpyDeviceToHost,
                        c->st) != cudaSuccess ||
        cudaStreamSynchronize(c->st) != cudaSuccess) {
      rc = kgf_fail("execute_filter_output: recomputing the slave");
    } else {
      s->shift = shift;
      s->isb = slave->isb;
      s->ver = c->ver[i];
      s->off = off;
      s->ok = true;
    }
  }
  if (rc == 0) {
    own_output(slave, sc);
    memcpy(slave->out_type == REAL ? (void *)slave->output.r : (void *)slave->output.c,
           c->h_out + (size_t)slot * (size_t)c->out_pitch + s->off, obytes);
  }
  pthread_mutex_unlock(&c->mu);
  return rc;
}

/* filter.c:663-921 */
int execute_filter_output(struct filter_out *const slave, int const shift) {
  if (slave == NULL)
    return -1;
  struct filter_in *const master = slave->master;
  if (master == NULL || master->fwd_plan == NULL) /* transient, filter.c:670-671 */
    return -1;
  struct master_ctx *c = (struct master_ctx *)master->fwd_plan;
  unsigned job = 0;
  int const t = take_job(slave, master, &job);
  if (t != 0)
    return t < 0 ? -1 : 0;
  if (c->small)
    return small_deliver(slave, job, shift);
  if (cudaEventSynchronize(c->done[job % ND]) != cudaSuccess)
    return kgf_fail("execute_filter_output: waiting for the block");
  if (slave->out_type == SPECTRUM)
    return 0; /* the caller reads master->fdomain[] itself (filter.c:368-371, spectrum.c:318) */
  struct slave_ctx *sc = (struct slave_ctx *)slave->rev_plan;
  if (sc == NULL || sc->own == NULL)
    return -1;
  if (slave->response == NULL) /* no filter yet: leave the output alone (filter.c:715-718) */
    return 0;
  return deliver(slave, c, job, shift);
}

/* EXTENSION: what n channel threads would each do, in one pass: one wait per distinct block instead of n. */
int execute_filter_output_batch(struct filter_out *const *slaves, int const *shifts, int n) {
  int rc = 0;
  unsigned waited_job = 0;
  struct master_ctx *waited = NULL;
  for (int i = 0; i < n; i++) {
    struct filter_out *slave = slaves[i];
    if (slave == NULL || slave->master == NULL || slave->master->fwd_plan == NULL) {
      rc = -1;
      continue;
    }
    struct master_ctx *c = (struct master_ctx *)slave->master->fwd_plan;
    unsigned job = 0;
    int const t = take_job(slave, slave->master, &job);
    if (t != 0) {
      if (t < 0)
        rc = -1;
      continue;
    }
    if (c->small) {
      if (small_deliver(slave, job, shifts[i]) != 0)
        rc = -1;
      continue;
    }
    if (waited != c || waited_job != job) {
      if (cudaEventSynchronize(c->done[job % ND]) != cudaSuccess) {
        rc = kgf_fail("execute_filter_output_batch: waiting for the block");
        continue;
      }
      waited = c;
      waited_job = job;
    }
    if (slave->out_type == SPECTRUM)
      continue;
    struct slave_ctx *sc = (struct slave_ctx *)slave->rev_plan;
    if (sc == NULL || sc->own == NULL) {
      rc = -1;
      continue;
    }
    if (slave->response == NULL)
      continue;
    if (deliver(slave, c, job, shifts[i]) != 0)
      rc = -1;
  }
  return rc;
}

/* ---------------------------------------------------------------- extensions: fine tuning, noise ---------- */
/* EXTENSION (SURVEY 8f-1): execute_filter_output with the fine-tuning oscillator, the block phase correction and
 * the baseband power of downconvert() (radio.c:1476-1501, :1515-1520) done on the device in the channel kernel's
 * store.  shift/remainder are compute_tuning's results (radio.c:1175-1199), samprate the channel's output rate,
 * doppler_rate in Hz/s.  *bb_power receives chan->sig.bb_power.  The caller then skips its own step_osc loop. */
int execute_filter_output_tuned(struct filter_out *slave, int shift, double remainder, double samprate, double doppler_rate,
                                double *bb_power) {
  if (slave && is_small(slave->master))
    return small_refuses("execute_filter_output_tuned");
  if (slave == NULL || slave->master == NULL || slave->master->fwd_plan == NULL || !(samprate > 0))
    return -1;
  struct filter_in *master = slave->master;
  struct master_ctx *c = (struct master_ctx *)master->fwd_plan;
  struct slave_ctx *sc = (struct slave_ctx *)slave->rev_plan;
  if (sc == NULL || slave->out_type != COMPLEX)
    return -1;
  bool changed = false;
  double jump = 0;
  if (shift != sc->ft_shift || isnan(sc->ft_remainder) || remainder != sc->ft_remainder) {
    sc->ft_freq = -remainder / samprate; /* set_osc(&chan->fine, -remainder/samprate, rate/samprate^2), radio.c:1481 */
    sc->ft_rate = doppler_rate / (samprate * samprate);
    sc->ft_remainder = remainder;
    changed = true;
  }
  if (shift != sc->ft_shift) {
    int const V = 1 + master->ilen / (master->impulse_length - 1);   /* radio.c:1492 */
    sc->ft_adj = (double)(shift % V) / (double)V;                     /* cispi(2 (shift % V) / V), in cycles */
    jump = fmod((double)(shift - sc->ft_shift) / (-2.0 * (V - 1)) / 2.0, 1.0); /* radio.c:1494, cispi(x) = x/2 cycles */
    sc->ft_shift = shift;
    changed = true;
  }
  if (changed) {
    /* the new parameters take effect with the block this call is about to deliver: epoch = that job */
    pthread_mutex_lock(&master->filter_mutex);
    unsigned const job = pthread_equal(master->owner, pthread_self()) ? master->next_jobnum - 1 : slave->next_jobnum;
    pthread_mutex_unlock(&master->filter_mutex);
    pthread_mutex_lock(&c->mu);
    cudaStreamSynchronize(c->st);
    long const saved = kgpu_bank_block_counter(c->bank);
    kgpu_bank_set_block_counter(c->bank, (long)job);
    double phase = 0; /* set_osc starts an uninitialised phasor at 1 (osc.c:29-36) */
    if (sc->ft_on)
      kgpu_bank_get_osc_phase(c->bank, sc->idx, &phase);
    kgpu_bank_set_osc(c->bank, sc->idx, 1, phase + jump, sc->ft_freq, sc->ft_rate, sc->ft_adj);
    kgpu_bank_set_block_counter(c->bank, saved);
    sc->ft_on = true;
    sc->ft_ver++;
    pthread_mutex_unlock(&c->mu);
  }
  int const rc = execute_filter_output(slave, shift);
  if (bb_power)
    *bb_power = sc->last_power;
  return rc;
}
/* back to the plain filter.h behaviour for this slave */
int filter_output_untune(struct filter_out *slave) {
  if (slave && is_small(slave->master))
    return small_refuses("filter_output_untune");
  if (slave == NULL || slave->master == NULL || slave->master->fwd_plan == NULL || slave->rev_plan == NULL)
    return -1;
  struct master_ctx *c = (struct master_ctx *)slave->master->fwd_plan;
  struct slave_ctx *sc = (struct slave_ctx *)slave->rev_plan;
  pthread_mutex_lock(&c->mu);
  cudaStreamSynchronize(c->st);
  kgpu_bank_set_osc(c->bank, sc->idx, 0, 0, 0, 0, 0);
  sc->ft_on = false;
  sc->ft_shift = -1000999;
  sc->ft_remainder = NAN;
  sc->ft_ver++;
  pthread_mutex_unlock(&c->mu);
  return 0;
}

/* EXTENSION (SURVEY 8f-2): have every block's noise-density estimate (estimate_noise, radio.c:1783-1866) computed on the
 * device for all slaves; samprate = Frontend.samprate.  filter_noise_estimate() then returns the value for the block
 * the slave's last execute_filter_output delivered (NAN for a block that had to be recomputed alone). */
int filter_input_enable_noise(struct filter_in *master, double samprate) {
  if (is_small(master))
    return small_refuses("filter_input_enable_noise");
  if (master == NULL || master->fwd_plan == NULL)
    return -1;
  struct master_ctx *c = (struct master_ctx *)master->fwd_plan;
  pthread_mutex_lock(&c->mu);
  c->noise_on = samprate > 0;
  c->noise_samprate = samprate;
  pthread_mutex_unlock(&c->mu);
  return 0;
}
double filter_noise_estimate(struct filter_out const *slave) {
  if (slave && is_small(slave->master)) {
    small_refuses("filter_noise_estimate");
    return NAN;
  }
  if (slave == NULL || slave->rev_plan == NULL)
    return NAN;
  return ((struct slave_ctx const *)slave->rev_plan)->last_n0;
}

/* ---------------------------------------------------------------- set_filter ---------------- */
/* filter.c:968-1045 */
int set_filter(struct filter_out *const slave, double low, double high, double const kaiser_beta) {
  if (slave == NULL || low != low || high != high || kaiser_beta != kaiser_beta || slave->master == NULL)
    return -1;
  struct master_ctx *c = (struct master_ctx *)slave->master->fwd_plan;
  struct slave_ctx *sc = (struct slave_ctx *)slave->rev_plan;
  if (c == NULL || sc == NULL)
    return -1;
  float complex *host = cache_aligned(sizeof(float complex) * (size_t)slave->points);
  if (!host)
    return -1;
  int rc;
  if (c->small) {
    struct small_ctx *k = (struct small_ctx *)c;
    pthread_mutex_lock(&k->mu);
    rc = kgpu_small_set_filter(k->ks, sc->idx, low, high, kaiser_beta, (float *)host, k->st);
    if (rc == 0)
      k->ver[sc->idx]++;
    pthread_mutex_unlock(&k->mu);
  } else {
    pthread_mutex_lock(&c->mu);
    /* only this master's pipeline stream is synchronised: a retune of one channel must not stall other masters
     * (filter2 / wfm composite masters of other channel threads) the way a device-wide synchronisation would */
    rc = kgpu_bank_set_filter_on(c->bank, sc->idx, low, high, kaiser_beta, c->st);
    if (rc == 0)
      rc = kgpu_bank_get_response(c->bank, sc->idx, (float *)host) > 0 ? 0 : -1;
    if (rc == 0)
      c->ver[sc->idx]++;
    pthread_mutex_unlock(&c->mu);
  }
  if (rc != 0) {
    free(host);
    return -1;
  }
  pthread_mutex_lock(&slave->response_mutex); /* hot swap (filter.c:1039-1043) */
  float complex *old = slave->response;
  slave->response = host;
  pthread_mutex_unlock(&slave->response_mutex);
  free(old);
  return 0;
}

int set_filter_weights(struct filter_out *out, double complex i_weight, double complex q_weight) { /* filter.c:922-929 */
  if (out == NULL)
    return -1;
  out->alpha = 0.5 * i_weight - I * q_weight;
  out->beta = 0.5 * i_weight + I * q_weight;
  return 0;
}

/* ---------------------------------------------------------------- wideband spectrum -------- */
/* EXTENSION: wideband_poll (spectrum.c:308-522) on the device for a SPECTRUM slave.  fft_n floats of window, as
 * generate_window() leaves them.  -1 (and the CPU loop stays with the caller) for lengths the analyzer cannot serve. */
int filter_spectrum_setup(struct filter_out *slave, int fft_n, int bin_count, float const *window) {
  if (slave && is_small(slave->master))
    return small_refuses("filter_spectrum_setup");
  if (slave == NULL || slave->out_type != SPECTRUM || slave->master == NULL || slave->master->fwd_plan == NULL ||
      window == NULL || bin_count < 1)
    return -1;
  struct filter_in *f = slave->master;
  struct master_ctx *c = (struct master_ctx *)f->fwd_plan;
  struct spec_slave *sp = calloc(1, sizeof *sp);
  if (!sp)
    return -1;
  sp->slave = slave;
  sp->bin_count = bin_count;
  sp->ks = kgpu_spectrum_create(fft_n, f->in_type == COMPLEX ? KGPU_COMPLEX : KGPU_REAL, bin_count);
  if (!sp->ks) {
    fprintf(stderr, "filter_spectrum_setup(fft_n=%d): %s\n", fft_n, kgpu_last_error());
    free(sp);
    return -1;
  }
  bool ok = kgpu_spectrum_set_window(sp->ks, window) == 0;
  ok = ok && cudaMalloc((void **)&sp->d_bins, sizeof(float) * (size_t)bin_count) == cudaSuccess;
  ok = ok && cudaHostAlloc((void **)&sp->h_bins, sizeof(float) * (size_t)bin_count, cudaHostAllocPortable) == cudaSuccess;
  ok = ok && cudaEventCreateWithFlags(&sp->ev, cudaEventDisableTiming) == cudaSuccess;
  if (!ok) {
    spec_slave_free(sp);
    return kgf_fail("filter_spectrum_setup");
  }
  pthread_mutex_lock(&c->mu);
  spec_slave_drop(c, slave);
  int rc = c->d_sring ? 0 : sring_seed(f, c);
  if (rc == 0) {
    sp->next = c->specs;
    c->specs = sp;
  }
  pthread_mutex_unlock(&c->mu);
  if (rc != 0)
    spec_slave_free(sp);
  return rc;
}

/* EXTENSION: one poll of the fft_avg segments ending at the end of the last block issued to the device (the reference
 * reads up to the live write pointer, which may be up to one block newer); *end_sample = that sample index
 * (frontend->samples at spectrum.c:365 / :425).  bin_data: bin_count floats, as wideband_poll leaves them. */
int filter_spectrum_poll(struct filter_out *slave, int shift, int fft_avg, double overlap, float *bin_data,
                         uint64_t *end_sample) {
  if (slave && is_small(slave->master))
    return small_refuses("filter_spectrum_poll");
  if (slave == NULL || slave->master == NULL || slave->master->fwd_plan == NULL || bin_data == NULL)
    return -1;
  struct filter_in *f = slave->master;
  struct master_ctx *c = (struct master_ctx *)f->fwd_plan;
  pthread_mutex_lock(&c->mu);
  struct spec_slave *sp = c->specs;
  while (sp && sp->slave != slave)
    sp = sp->next;
  int rc = sp ? 0 : -1;
  if (rc == 0 && (c->d_sring == NULL || c->sring_i16 != ingest_i16(c)))
    rc = sring_seed(f, c);
  uint64_t const end = (uint64_t)f->ilen * c->issued;
  double scale = 1.0; /* int16 rings: that of the ring's oldest sample, then each change (packed-12: the drivers' float scale) */
  int n = 0;
  if (rc == 0 && c->sring_i16 && chg_span(c, ND, (long long)end - c->sring_cap, (long long)end, &scale, &n) != 0)
    rc = kgf_fail("filter_spectrum_poll: scale changes");
  if (rc == 0 && kgpu_spectrum_run(sp->ks, c->d_sring, c->sring_cap, c->sring_pos, c->sring_i16 ? KGPU_FMT_I16 : KGPU_FMT_F32,
                                   (float)scale, n ? c->d_chg : NULL, n, (long long)end, c->mode == INGEST_INT16 && c->i16_derand, shift,
                                   fft_avg, overlap, sp->d_bins, c->st) != 0)
    rc = kgf_fail("filter_spectrum_poll: kgpu_spectrum_run");
  if (rc == 0 && (cudaMemcpyAsync(sp->h_bins, sp->d_bins, sizeof(float) * (size_t)sp->bin_count, cudaMemcpyDeviceToHost,
                                  c->st) != cudaSuccess ||
                  cudaEventRecord(sp->ev, c->st) != cudaSuccess))
    rc = kgf_fail("filter_spectrum_poll: D2H of the bins");
  pthread_mutex_unlock(&c->mu);
  if (rc == 0 && cudaEventSynchronize(sp->ev) != cudaSuccess)
    rc = kgf_fail("filter_spectrum_poll: wait");
  if (rc != 0)
    return -1;
  memcpy(bin_data, sp->h_bins, sizeof(float) * (size_t)sp->bin_count);
  if (end_sample)
    *end_sample = end;
  return 0;
}

/* ---------------------------------------------------------------- narrowband spectrum ------ */
/* EXTENSION: narrowband_poll (spectrum.c:206-306) on the device for a COMPLEX slave.  fft_n floats of window, as
 * generate_window() leaves them.  -1 (and the CPU loop stays with the caller) when the device cannot serve the slave. */
int filter_spectrum_narrow_setup(struct filter_out *slave, int fft_n, int bin_count, float const *window) {
  if (slave && is_small(slave->master))
    return small_refuses("filter_spectrum_narrow_setup");
  if (slave == NULL || slave->out_type != COMPLEX || slave->rev_plan == NULL || slave->master == NULL ||
      slave->master->fwd_plan == NULL || window == NULL || bin_count < 1 || bin_count > fft_n)
    return -1;
  struct master_ctx *c = (struct master_ctx *)slave->master->fwd_plan;
  struct slave_ctx *sc = (struct slave_ctx *)slave->rev_plan;
  struct nb_spec *nb = calloc(1, sizeof *nb);
  if (!nb)
    return -1;
  nb->bin_count = bin_count;
  nb->ks = kgpu_spectrum_create(fft_n, KGPU_COMPLEX, bin_count);
  if (!nb->ks) {
    fprintf(stderr, "filter_spectrum_narrow_setup(fft_n=%d): %s\n", fft_n, kgpu_last_error());
    free(nb);
    return -1;
  }
  bool ok = kgpu_spectrum_set_window(nb->ks, window) == 0;
  ok = ok && cudaMalloc((void **)&nb->d_bins, sizeof(float) * (size_t)bin_count) == cudaSuccess;
  ok = ok && cudaHostAlloc((void **)&nb->h_bins, sizeof(float) * (size_t)bin_count, cudaHostAllocPortable) == cudaSuccess;
  ok = ok && cudaEventCreateWithFlags(&nb->ev, cudaEventDisableTiming) == cudaSuccess;
  if (!ok) {
    nb_free(nb);
    return kgf_fail("filter_spectrum_narrow_setup");
  }
  pthread_mutex_lock(&c->mu);
  struct nb_spec *old = sc->nb;
  if (old) {
    cudaStreamSynchronize(c->st);
    nb_free(old);
  }
  sc->nb = nb;
  pthread_mutex_unlock(&c->mu);
  return 0;
}

/* EXTENSION: the ring of spectrum.c:124-145 before a block is appended: the first call creates ring_samples zeros with
 * the write index at 0; a larger size keeps [0, old size), zeroes the rest and leaves the index; a smaller one does
 * nothing.  Call it where demod_spectrum would grow its ring, before downconvert() delivers the block. */
int filter_spectrum_narrow_reserve(struct filter_out *slave, long ring_samples) {
  if (slave && is_small(slave->master))
    return small_refuses("filter_spectrum_narrow_reserve");
  if (slave == NULL || slave->rev_plan == NULL || slave->master == NULL || slave->master->fwd_plan == NULL ||
      ring_samples < 1)
    return -1;
  struct master_ctx *c = (struct master_ctx *)slave->master->fwd_plan;
  struct nb_spec *nb = ((struct slave_ctx *)slave->rev_plan)->nb;
  if (nb == NULL)
    return -1;
  int rc = 0;
  pthread_mutex_lock(&c->mu);
  if (nb->d_ring == NULL || ring_samples > nb->ring_size) {
    float complex *ring = NULL;
    size_t const old = nb->d_ring ? sizeof(float complex) * (size_t)nb->ring_size : 0;
    cudaStreamSynchronize(c->st); /* pending appends and polls read the old ring */
    if (cudaMalloc((void **)&ring, sizeof(float complex) * (size_t)ring_samples) != cudaSuccess ||
        cudaMemsetAsync((char *)ring + old, 0, sizeof(float complex) * (size_t)ring_samples - old, c->st) != cudaSuccess ||
        (old && cudaMemcpyAsync(ring, nb->d_ring, old, cudaMemcpyDeviceToDevice, c->st) != cudaSuccess) ||
        cudaStreamSynchronize(c->st) != cudaSuccess) {
      cudaFree(ring);
      rc = kgf_fail("filter_spectrum_narrow_reserve");
    } else {
      cudaFree(nb->d_ring);
      nb->d_ring = ring;
      nb->ring_size = ring_samples;
    }
  }
  pthread_mutex_unlock(&c->mu);
  return rc;
}

/* EXTENSION: one narrowband_poll of the slave's ring as its delivered blocks have left it: bin_count floats into
 * bin_data, as narrowband_poll leaves them before its base / step scaling (spectrum.c:284-305), which stays with the
 * caller.  -1 before the first reserve.  One poller per slave. */
int filter_spectrum_narrow_poll(struct filter_out *slave, int fft_avg, double overlap, float *bin_data) {
  if (slave && is_small(slave->master))
    return small_refuses("filter_spectrum_narrow_poll");
  if (slave == NULL || slave->rev_plan == NULL || slave->master == NULL || slave->master->fwd_plan == NULL ||
      bin_data == NULL)
    return -1;
  struct master_ctx *c = (struct master_ctx *)slave->master->fwd_plan;
  struct slave_ctx *sc = (struct slave_ctx *)slave->rev_plan;
  pthread_mutex_lock(&c->mu);
  struct nb_spec *nb = sc->nb;
  int rc = nb && nb->d_ring ? 0 : -1;
  if (rc == 0 && kgpu_spectrum_run_narrow(nb->ks, nb->d_ring, nb->ring_size, nb->ring_idx, fft_avg, overlap, nb->d_bins,
                                          NULL, c->st) != 0)
    rc = kgf_fail("filter_spectrum_narrow_poll: kgpu_spectrum_run_narrow");
  if (rc == 0 && (cudaMemcpyAsync(nb->h_bins, nb->d_bins, sizeof(float) * (size_t)nb->bin_count, cudaMemcpyDeviceToHost,
                                  c->st) != cudaSuccess ||
                  cudaEventRecord(nb->ev, c->st) != cudaSuccess))
    rc = kgf_fail("filter_spectrum_narrow_poll: D2H of the bins");
  pthread_mutex_unlock(&c->mu);
  if (rc == 0 && cudaEventSynchronize(nb->ev) != cudaSuccess)
    rc = kgf_fail("filter_spectrum_narrow_poll: wait");
  if (rc != 0)
    return -1;
  memcpy(bin_data, nb->h_bins, sizeof(float) * (size_t)nb->bin_count);
  return 0;
}

/* EXTENSION: a host copy of the slave's ring (up to cap samples) with its size and write index, e.g. for a caller that
 * hands the analysis back to its CPU loop.  Returns the ring size, 0 before the first reserve, -1 on error. */
long filter_spectrum_narrow_ring(struct filter_out *slave, float complex *ring, long cap, long *ring_idx) {
  if (slave && is_small(slave->master))
    return (long)small_refuses("filter_spectrum_narrow_ring");
  if (slave == NULL || slave->rev_plan == NULL || slave->master == NULL || slave->master->fwd_plan == NULL)
    return -1;
  struct master_ctx *c = (struct master_ctx *)slave->master->fwd_plan;
  struct nb_spec *nb = ((struct slave_ctx *)slave->rev_plan)->nb;
  if (nb == NULL)
    return -1;
  long rc = 0;
  pthread_mutex_lock(&c->mu);
  if (nb->d_ring) {
    rc = nb->ring_size;
    if (ring_idx)
      *ring_idx = nb->ring_idx;
    long const n = cap < nb->ring_size ? cap : nb->ring_size;
    if (ring && n > 0 &&
        (cudaMemcpyAsync(ring, nb->d_ring, sizeof(float complex) * (size_t)n, cudaMemcpyDeviceToHost, c->st) != cudaSuccess ||
         cudaStreamSynchronize(c->st) != cudaSuccess))
      rc = kgf_fail("filter_spectrum_narrow_ring");
  }
  pthread_mutex_unlock(&c->mu);
  return rc;
}

/* ---------------------------------------------------------------- delete -------------------- */
int delete_filter_output(struct filter_out *slave) { /* filter.c:943-957 */
  if (slave == NULL)
    return -1;
  struct slave_ctx *sc = (struct slave_ctx *)slave->rev_plan;
  if (sc && is_small(slave->master)) {
    struct small_ctx *c = (struct small_ctx *)slave->master->fwd_plan;
    pthread_mutex_lock(&c->mu);
    cudaStreamSynchronize(c->st);
    kgpu_small_undefine(c->ks, sc->idx);
    c->slots[sc->idx] = NULL;
    c->ver[sc->idx]++;
    for (int s = 0; s < ND; s++)
      c->snap[s][sc->idx].ok = false;
    pthread_mutex_unlock(&c->mu);
  } else if (slave->out_type == SPECTRUM && slave->master && slave->master->fwd_plan) {
    struct master_ctx *c = (struct master_ctx *)slave->master->fwd_plan;
    pthread_mutex_lock(&c->mu);
    spec_slave_drop(c, slave);
    pthread_mutex_unlock(&c->mu);
  }
  if (sc && slave->master && slave->master->fwd_plan && !is_small(slave->master)) {
    struct master_ctx *c = (struct master_ctx *)slave->master->fwd_plan;
    pthread_mutex_lock(&c->mu);
    cudaStreamSynchronize(c->st);
    kgpu_bank_enable(c->bank, sc->idx, 0);
    kgpu_bank_set_osc(c->bank, sc->idx, 0, 0, 0, 0, 0);
    c->slots[sc->idx] = NULL;
    c->ranges_dirty = true;
    for (int s = 0; s < ND; s++)
      c->snap[s][sc->idx].ok = false;
    nb_free(sc->nb); /* after the synchronise above: no append or poll still reads it */
    sc->nb = NULL;
    pthread_mutex_unlock(&c->mu);
  }
  if (sc) {
    nb_free(sc->nb); /* the master was deleted first */
    free(sc->own);
  }
  free(sc);
  if (slave->init)
    pthread_mutex_destroy(&slave->response_mutex);
  free(slave->response);
  free(slave->fdomain);
  memset(slave, 0, sizeof *slave);
  return 0;
}
int delete_filter_input(struct filter_in *master) { /* filter.c:930-942 */
  if (master == NULL)
    return -1;
  master_teardown(master);
  if (master->init) {
    pthread_mutex_destroy(&master->filter_mutex);
    pthread_cond_destroy(&master->filter_cond);
  }
  memset(master, 0, sizeof *master);
  return 0;
}

/* ---------------------------------------------------------------- write_*filter ------------- */
/* filter.c:1093-1134: n floats or float pairs of esz bytes to the float ring at its write pointer *wp */
static int write_floats(struct filter_in *f, void **wp, void const *buffer, int size, size_t esz, char const *who) {
  if (f->fwd_plan == NULL || (!is_small(f) && check_mode(f, (struct master_ctx *)f->fwd_plan, INGEST_FLOAT, false, who) != 0))
    return -1;
  if ((f->wcnt + size) * esz >= f->input_buffer_size)
    return -1;
  if (buffer != NULL)
    memcpy(*wp, buffer, (size_t)size * esz);
  *wp = (char *)*wp + (ptrdiff_t)size * (ptrdiff_t)esz;
  kgf_ring_wrap(wp, f->input_buffer, f->input_buffer_size);
  f->wcnt += size;
  return fire_ready_blocks(f);
}
int write_cfilter(struct filter_in *f, float complex const *buffer, int size) {
  return f ? write_floats(f, (void **)&f->input_write_pointer.c, buffer, size, sizeof *buffer, "write_cfilter") : -1;
}
int write_rfilter(struct filter_in *f, float const *buffer, int size) {
  return f ? write_floats(f, (void **)&f->input_write_pointer.r, buffer, size, sizeof *buffer, "write_rfilter") : -1;
}
/* EXTENSION: raw ADC words straight to the device; conversion (rx888.c:753-767) happens in fwd_cols.
 * samples == NULL: the caller already wrote them through filter_i16_write_pointer() (the zero-copy driver path). */
int write_i16filter(struct filter_in *f, int16_t const *samples, int n, float scale, bool derandomize) {
  if (is_small(f))
    return small_refuses("write_i16filter");
  if (f == NULL || f->fwd_plan == NULL || n < 0)
    return -1;
  struct master_ctx *c = (struct master_ctx *)f->fwd_plan;
  if (c->mode != INGEST_INT16 && filter_i16_write_pointer(f) == NULL)
    return -1;
  if (wring_bytes(&c->ring, (size_t)f->wcnt + (size_t)n) >= c->ring.size)
    return -1;
  pthread_mutex_lock(&c->mu);
  int const rc = chg_note(f, c, scale, "write_i16filter");
  pthread_mutex_unlock(&c->mu);
  if (rc != 0)
    return -1;
  c->i16_derand = derandomize;
  if (samples != NULL)
    memcpy(c->ring.wp, samples, wring_bytes(&c->ring, (size_t)n));
  wring_push(&c->ring, (size_t)n);
  f->wcnt += n;
  return fire_ready_blocks(f);
}
/* where a driver may deposit the next raw samples itself (mirrored, pinned ring: up to one block contiguous),
 * e.g. as the libusb transfer buffer of rx888.c:797-826; publish with write_i16filter(f, NULL, n, ...) */
int16_t *filter_i16_write_pointer(struct filter_in *f) {
  if (is_small(f)) {
    small_refuses("filter_i16_write_pointer");
    return NULL;
  }
  if (f == NULL || f->fwd_plan == NULL)
    return NULL;
  struct master_ctx *c = (struct master_ctx *)f->fwd_plan;
  if (c->mode != INGEST_INT16) {
    static uint32_t const zero[3];
    size_t const group = 8 * ((f->in_type == COMPLEX) ? 2 * sizeof(int16_t) : sizeof(int16_t));
    if (check_mode(f, c, INGEST_INT16, false, "filter_i16_write_pointer") != 0 ||
        wring_open(&c->ring, page_round((size_t)ND * (size_t)f->points * group / 8), group, f->impulse_length - 1, zero) != 0)
      return NULL;
    c->mode = INGEST_INT16;
  }
  return (int16_t *)c->ring.wp;
}

/* the checks, table entry and scale of a write of n samples in `format` about to be stored at the ring's write pointer
 * (starting the raw ring at a master's first write); 0, or -1 with nothing stored */
static int raw_admit(struct filter_in *f, struct master_ctx *c, int n, int format, double scale, char const *who) {
  struct raw_format const *rf = format_row(format);
  if (rf == NULL) {
    fprintf(stderr, "%s: unknown format %d\n", who, format);
    return -1;
  }
  bool const iq = rf->path == RAW_IQ;
  if (iq && c->iq_cap == 0) {
    fprintf(stderr, "%s: format %d needs filter_iq_correction_setup first\n", who, format);
    return -1;
  }
  if (c->mode != INGEST_RAW && raw_start(f, c, format, false, who) != 0)
    return -1;
  if (format != c->raw_fmt) {
    fprintf(stderr, "%s: format %d on a master fed format %d\n", who, format, c->raw_fmt);
    return -1;
  }
  if (rf->group % 8 != 0 && n % 8 != 0) {
    fprintf(stderr, "%s: %d packed 12-bit samples: not a multiple of 8\n", who, n);
    return -1;
  }
  if (wring_bytes(&c->ring, (size_t)f->wcnt + (size_t)n) >= c->ring.size)
    return -1;
  if (iq) { /* one transfer: its table entry */
    if (n < FILTER_IQ_MIN_WRITE) {
      fprintf(stderr, "%s: %d I/Q pairs: writes with I/Q correction take at least %d\n", who, n, FILTER_IQ_MIN_WRITE);
      return -1;
    }
    struct kgpu_iq_write *w = &c->h_iqw[c->iq_writes % (unsigned long long)c->iq_cap];
    memset(w, 0, sizeof *w);
    w->first = c->iq_total;
    w->n = n;
    w->scale = scale;
    w->last_over = -1;
    c->iq_writes++;
    c->iq_total += n;
    return 0;
  }
  pthread_mutex_lock(&c->mu);
  int const rc = chg_note(f, c, scale, who);
  pthread_mutex_unlock(&c->mu);
  return rc;
}
/* publish the n samples just stored at the ring's write pointer, and fire the blocks they complete */
static int raw_commit(struct filter_in *f, struct master_ctx *c, int n) {
  wring_push(&c->ring, (size_t)n);
  f->wcnt += n;
  return fire_ready_blocks(f);
}

/* EXTENSION: raw packed 12-bit, 8-bit or 16-bit ADC words, or floats, converted on the device (see
 * include/ka9q_gpu_filter.h).  The drivers (airspy.c:388-434, hydrasdr.c:663-830, rtlsdr.c:316-343, bladerf.c:215-246,
 * airspyhf.c:292-325, fobos.c:395-426) get their buffers from their vendor libraries, so there is no zero-copy write
 * pointer: the bytes are copied into the raw ring. */
int write_rawfilter(struct filter_in *f, void const *samples, int n, int format, double scale) {
  if (is_small(f))
    return small_refuses("write_rawfilter");
  if (f == NULL || f->fwd_plan == NULL || samples == NULL || n < 0)
    return -1;
  struct master_ctx *c = (struct master_ctx *)f->fwd_plan;
  if (raw_admit(f, c, n, format, scale, "write_rawfilter") != 0)
    return -1;
  memcpy(c->ring.wp, samples, wring_bytes(&c->ring, (size_t)n)); /* the mirror view keeps a write across the end contiguous */
  return raw_commit(f, c, n);
}

/* EXTENSION: SDRplay's separate I and Q arrays (sdrplay.c:1234-1246), interleaved into the FILTER_RAW_S16 ring: a copy
 * like write_rawfilter's memcpy, after which the pairs are an S16 write like any other. */
int write_rawfilter_planar(struct filter_in *f, int16_t const *i, int16_t const *q, int n, double scale) {
  if (is_small(f))
    return small_refuses("write_rawfilter_planar");
  if (f == NULL || f->fwd_plan == NULL || i == NULL || q == NULL || n < 0)
    return -1;
  if (f->in_type != COMPLEX) {
    fprintf(stderr, "write_rawfilter_planar: the master is not COMPLEX\n");
    return -1;
  }
  struct master_ctx *c = (struct master_ctx *)f->fwd_plan;
  if (raw_admit(f, c, n, FILTER_RAW_S16, scale, "write_rawfilter_planar") != 0)
    return -1;
  int16_t *restrict const w = (int16_t *)c->ring.wp; /* the mirror view keeps a write across the end contiguous */
  for (int k = 0; k < n; k++) {
    w[2 * k] = i[k];
    w[2 * k + 1] = q[k];
  }
  return raw_commit(f, c, n);
}

/* EXTENSION: the A/D statistics of the blocks whose device work completed since the previous call (see
 * include/ka9q_gpu_filter.h).  The slots about to be reused are folded in by execute_filter_input_n, which has already
 * waited for them; this call folds, in job order, whatever else has completed, without waiting. */
int filter_ingest_stats(struct filter_in *f, struct filter_ingest_stats *stats) {
  if (is_small(f))
    return small_refuses("filter_ingest_stats");
  if (f == NULL || f->fwd_plan == NULL || stats == NULL)
    return -1;
  struct master_ctx *c = (struct master_ctx *)f->fwd_plan;
  int rc = 0;
  pthread_mutex_lock(&c->mu);
  if (ingest_of(f, c) != INGEST_NONE && !ingest_counted(c))
    rc = -1; /* floats: the driver counts them; generated: filter_siggen_stats; I/Q corrected: filter_iq_records */
  else if (!c->stats_on) {
    if (c->d_bstats == NULL &&
        (cudaMalloc((void **)&c->d_bstats, sizeof *c->d_bstats * ND) != cudaSuccess ||
         cudaHostAlloc((void **)&c->h_bstats, sizeof *c->h_bstats * ND, cudaHostAllocPortable) != cudaSuccess)) {
      cudaFree(c->d_bstats);
      c->d_bstats = NULL;
      rc = kgf_fail("filter_ingest_stats: buffers");
    } else {
      c->stats_on = true;
      c->folded = c->issued; /* blocks already issued carry no statistics */
      memset(&c->acc, 0, sizeof c->acc);
      memset(stats, 0, sizeof *stats);
    }
  } else {
    while (c->folded < c->issued && cudaEventQuery(c->done[c->folded % ND]) == cudaSuccess)
      fold_one(f, c);
    *stats = c->acc;
    uint64_t const since = c->acc.since_over;
    memset(&c->acc, 0, sizeof c->acc);
    c->acc.since_over = since;
  }
  pthread_mutex_unlock(&c->mu);
  return rc;
}

/* EXTENSION: HackRF's and FUNcube's DC and I/Q correction on the device (see include/ka9q_gpu_filter.h): the raw ring,
 * the table of writes and the initial coefficient set, before the first write. */
int filter_iq_correction_setup(struct filter_in *f, int format, struct filter_iq_params const *p) {
  if (is_small(f))
    return small_refuses("filter_iq_correction_setup");
  struct raw_format const *rf = format_row(format);
  if (f == NULL || f->fwd_plan == NULL || p == NULL || rf == NULL || rf->path != RAW_IQ)
    return -1;
  struct master_ctx *c = (struct master_ctx *)f->fwd_plan;
  if (raw_start(f, c, format, true, "filter_iq_correction_setup") != 0)
    return -1;
  size_t const nw = (size_t)filter_iq_table_writes(f->ilen, f->impulse_length, f->in_type, format);
  bool ok = cudaHostAlloc((void **)&c->h_iqw, sizeof *c->h_iqw * nw, cudaHostAllocPortable) == cudaSuccess;
  ok = ok && cudaMalloc((void **)&c->d_iqw, sizeof *c->d_iqw * nw) == cudaSuccess;
  ok = ok && cudaMalloc((void **)&c->d_iqc, sizeof *c->d_iqc * nw) == cudaSuccess;
  ok = ok && cudaMalloc((void **)&c->d_iqr, sizeof *c->d_iqr * nw) == cudaSuccess;
  ok = ok && cudaHostAlloc((void **)&c->h_iqr, sizeof *c->h_iqr * nw, cudaHostAllocPortable) == cudaSuccess;
  struct kgpu_iq_state const init = {p->dc_i, p->dc_q, p->sinphi, p->imbalance, p->gain_i, p->gain_q, p->secphi, p->tanphi};
  ok = ok && cudaMemcpy(c->d_iqc, &init, sizeof init, cudaMemcpyHostToDevice) == cudaSuccess; /* write 0's coefficients */
  if (!ok)
    return kgf_fail("filter_iq_correction_setup: table buffers"); /* freed with the master, whose writes are refused */
  c->iq_cap = (int)nw;
  c->iq_par.kind = p->gp_rate != 0 ? 1 : 2;
  c->iq_par.dc_alpha = p->dc_alpha;
  c->iq_par.gp = p->gp_rate != 0 ? p->gp_rate : p->gp_alpha;
  return 0;
}

/* EXTENSION: the records of the writes whose launch has completed (see include/ka9q_gpu_filter.h).  The launches' slots
 * about to be reused are taken in by execute_filter_input_n, which has already waited for them; this call takes in, in
 * job order, whatever else has completed, without waiting. */
int filter_iq_records(struct filter_in *f, struct filter_iq_record *recs, int max) {
  if (is_small(f))
    return small_refuses("filter_iq_records");
  if (f == NULL || f->fwd_plan == NULL || (recs == NULL && max > 0))
    return -1;
  struct master_ctx *c = (struct master_ctx *)f->fwd_plan;
  if (c->iq_cap == 0)
    return -1;
  pthread_mutex_lock(&c->mu);
  while (c->iq_checked < c->issued && cudaEventQuery(c->done[c->iq_checked % ND]) == cudaSuccess)
    c->iq_avail = c->iq_job_done[c->iq_checked++ % ND];
  unsigned long long const cap = (unsigned long long)c->iq_cap;
  if (c->iq_scanned > cap && c->iq_given < c->iq_scanned - cap)
    c->iq_given = c->iq_scanned - cap; /* overwritten by later launches' records */
  int n = 0;
  for (; n < max && c->iq_given < c->iq_avail; n++, c->iq_given++) {
    struct kgpu_iq_record const *r = &c->h_iqr[c->iq_given % cap];
    struct filter_iq_record *o = &recs[n];
    o->seq = r->seq;
    o->n = r->n;
    o->sum_i = r->sum_i;
    o->sum_q = r->sum_q;
    o->i_energy = r->i_energy;
    o->q_energy = r->q_energy;
    o->dotprod = r->dotprod;
    o->overs = r->overs;
    o->since_over = r->since_over;
    o->dc_i = r->state.dc_i;
    o->dc_q = r->state.dc_q;
    o->sinphi = r->state.sinphi;
    o->imbalance = r->state.imbalance;
    o->gain_i = r->state.gain_i;
    o->gain_q = r->state.gain_q;
    o->secphi = r->state.secphi;
    o->tanphi = r->state.tanphi;
  }
  pthread_mutex_unlock(&c->mu);
  return n;
}

/* ---------------------------------------------------------------- sig_gen ------------------- */
/* EXTENSION: sig_gen's source on the device (see include/ka9q_gpu_filter.h), before the first write. */
int filter_siggen_setup(struct filter_in *f, struct filter_siggen_params const *p) {
  if (is_small(f))
    return small_refuses("filter_siggen_setup");
  if (f == NULL || f->fwd_plan == NULL || p == NULL)
    return -1;
  struct master_ctx *c = (struct master_ctx *)f->fwd_plan;
  if (check_mode(f, c, INGEST_GEN, true, "filter_siggen_setup") != 0)
    return -1;
  struct kgpu_siggen_params const kp = {p->freq, p->rate, p->amplitude, p->noise, p->seed};
  kgpu_siggen *g = kgpu_siggen_create(f->in_type == COMPLEX ? KGPU_COMPLEX : KGPU_REAL, &kp);
  if (!g) {
    fprintf(stderr, "filter_siggen_setup: %s\n", kgpu_last_error());
    return -1;
  }
  if (cudaMalloc((void **)&c->d_gen_energy, sizeof(double) * ND) != cudaSuccess ||
      cudaHostAlloc((void **)&c->h_gen_energy, sizeof(double) * ND, cudaHostAllocPortable) != cudaSuccess) {
    kgpu_siggen_destroy(g);
    return kgf_fail("filter_siggen_setup: energy buffers"); /* freed with the master */
  }
  pthread_mutex_lock(&c->mu);
  c->gen = g;
  c->mode = INGEST_GEN;
  pthread_mutex_unlock(&c->mu);
  return 0;
}

/* EXTENSION: advance a generated master by n samples (REAL) or pairs (COMPLEX), stored with this write's scale; fires
 * the blocks they complete as write_rfilter does. */
int write_genfilter(struct filter_in *f, int n, double scale) {
  if (is_small(f))
    return small_refuses("write_genfilter");
  if (f == NULL || f->fwd_plan == NULL || n < 0)
    return -1;
  struct master_ctx *c = (struct master_ctx *)f->fwd_plan;
  if (check_mode(f, c, INGEST_GEN, false, "write_genfilter") != 0 || c->mode != INGEST_GEN)
    return -1; /* only filter_siggen_setup starts a generated master */
  if (((size_t)f->wcnt + (size_t)n) * c->esz >= f->input_buffer_size)
    return -1;
  pthread_mutex_lock(&c->mu);
  int const rc = chg_note(f, c, scale, "write_genfilter");
  pthread_mutex_unlock(&c->mu);
  if (rc != 0)
    return -1;
  if (c->gen_mod)
    wring_push(&c->ring, (size_t)n); /* the envelope the driver wrote at filter_siggen_mod_pointer */
  f->wcnt += n;
  return fire_ready_blocks(f);
}

/* EXTENSION: sig_gen's AM and DSB sources (see include/ka9q_gpu_filter.h), after filter_siggen_setup and before the
 * first write.  The envelope ring holds the host float ring's samples for the wideband analyzer's seeding (sring_seed
 * regenerates them), plus the largest write that may be pending or being written behind them; the device window of
 * the envelope is d_raw, sized as raw_start sizes it. */
int filter_siggen_modulate(struct filter_in *f, double dc) {
  if (is_small(f))
    return small_refuses("filter_siggen_modulate");
  if (f == NULL || f->fwd_plan == NULL || !isfinite(dc))
    return -1;
  struct master_ctx *c = (struct master_ctx *)f->fwd_plan;
  if (c->mode != INGEST_GEN || c->chg_started) {
    fprintf(stderr, "filter_siggen_modulate: %s\n", c->mode != INGEST_GEN ? "the master is not generated" : "after the first write");
    return -1;
  }
  if (!c->gen_mod) {
    static uint32_t const zero[3];
    size_t const samples = f->input_buffer_size / c->esz; /* the host float ring's */
    size_t const span = (size_t)(ND - 2) * (size_t)f->ilen + (size_t)f->points;
    if (wring_open(&c->ring, page_round(2 * samples * sizeof(float)), 8 * sizeof(float), f->impulse_length - 1, zero) != 0)
      return kgf_fail("filter_siggen_modulate: envelope ring");
    if (cudaMalloc(&c->d_raw, span * sizeof(float)) != cudaSuccess) {
      c->d_raw = NULL;
      ring_free(c->ring.base, c->ring.size);
      c->ring.base = NULL;
      return kgf_fail("filter_siggen_modulate: device buffer");
    }
  }
  if (kgpu_siggen_set_modulation(c->gen, dc) != 0)
    return kgf_fail("filter_siggen_modulate");
  pthread_mutex_lock(&c->mu);
  c->gen_mod = true;
  pthread_mutex_unlock(&c->mu);
  return 0;
}

float *filter_siggen_mod_pointer(struct filter_in *f) {
  if (is_small(f)) {
    small_refuses("filter_siggen_mod_pointer");
    return NULL;
  }
  if (f == NULL || f->fwd_plan == NULL)
    return NULL;
  struct master_ctx *c = (struct master_ctx *)f->fwd_plan;
  return c->mode == INGEST_GEN && c->gen_mod ? (float *)c->ring.wp : NULL;
}

/* EXTENSION: the generated energy of the blocks whose device work completed since the previous call, as
 * filter_ingest_stats counts them. */
int filter_siggen_stats(struct filter_in *f, struct filter_siggen_stats *stats) {
  if (is_small(f))
    return small_refuses("filter_siggen_stats");
  if (f == NULL || f->fwd_plan == NULL || stats == NULL)
    return -1;
  struct master_ctx *c = (struct master_ctx *)f->fwd_plan;
  if (c->mode != INGEST_GEN)
    return -1;
  pthread_mutex_lock(&c->mu);
  if (!c->gen_stats_on) {
    c->gen_stats_on = true;
    c->gen_folded = c->issued; /* blocks already issued carry no energy */
    memset(&c->gen_acc, 0, sizeof c->gen_acc);
    memset(stats, 0, sizeof *stats);
  } else {
    while (c->gen_folded < c->issued && cudaEventQuery(c->done[c->gen_folded % ND]) == cudaSuccess)
      gen_fold_one(f, c);
    *stats = c->gen_acc;
    memset(&c->gen_acc, 0, sizeof c->gen_acc);
  }
  pthread_mutex_unlock(&c->mu);
  return 0;
}

/* ---------------------------------------------------------------- housekeeping -------------- */
void *run_fft(void *p) { /* filter.c:485: the CPU FFT worker pool has no GPU counterpart */
  (void)p;
  return NULL;
}
void suggest(int size, int dir, int clex) { /* filter.c:1136-1144: wisdom hints are meaningless here */
  (void)size;
  (void)dir;
  (void)clex;
}
long gcd(long a, long b) {
  while (b != 0) {
    long const t = a % b;
    a = b;
    b = t;
  }
  return a;
}
long lcm(long a, long b) {
  if (a <= 0 || b <= 0)
    return 0;
  return a / gcd(a, b) * b;
}
/* "good" now means: plannable by the device transform (factors 2,3,5,7) */
bool goodchoice(long n) {
  if (n <= 0)
    return false;
  static int const primes[4] = {2, 3, 5, 7};
  for (int i = 0; i < 4; i++)
    while (n % primes[i] == 0)
      n /= primes[i];
  return n == 1;
}
int ceil_pow2(uint32_t x) {
  uint32_t p = 1;
  while (p < x && p < 0x80000000u)
    p <<= 1;
  return (int)p;
}

/* spectrum.c's own analysis FFTs (filter.h:112-115): forwarded to the host's FFTW when present */
static void *fftw_handle(void) {
  static void *h;
  static int tried;
  if (!tried) {
    tried = 1;
    h = dlopen("libfftw3f.so.3", RTLD_NOW | RTLD_GLOBAL);
  }
  return h;
}
fftwf_plan plan_complex(int N, float complex *in, float complex *out, int direction) {
  void *h = fftw_handle();
  fftwf_plan (*fn)(int, float complex *, float complex *, int, unsigned) = h ? dlsym(h, "fftwf_plan_dft_1d") : NULL;
  return fn ? fn(N, in, out, direction, 1u << 6 /* FFTW_ESTIMATE */) : NULL;
}
fftwf_plan plan_r2c(int N, float *in, float complex *out) {
  void *h = fftw_handle();
  fftwf_plan (*fn)(int, float *, float complex *, unsigned) = h ? dlsym(h, "fftwf_plan_dft_r2c_1d") : NULL;
  return fn ? fn(N, in, out, 1u << 6) : NULL;
}
fftwf_plan plan_c2r(int N, float complex *in, float *out) {
  void *h = fftw_handle();
  fftwf_plan (*fn)(int, float complex *, float *, unsigned) = h ? dlsym(h, "fftwf_plan_dft_c2r_1d") : NULL;
  return fn ? fn(N, in, out, 1u << 6) : NULL;
}
void destroy_plan(fftwf_plan *plan) {
  if (plan == NULL || *plan == NULL)
    return;
  void *h = fftw_handle();
  void (*fn)(fftwf_plan) = h ? dlsym(h, "fftwf_destroy_plan") : NULL;
  if (fn)
    fn(*plan);
  *plan = NULL;
}
