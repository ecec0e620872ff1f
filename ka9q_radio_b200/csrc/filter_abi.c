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

struct master_ctx {
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
  /* raw int16 ingest (extension) */
  bool i16_mode;
  void *i16_ring;
  size_t i16_ring_size, i16_esz;
  char *i16_wp, *i16_rp;
  bool i16_derand;
  /* raw 8-bit / packed 12-bit ingest (extension): the bytes in a mirrored ring of their own, unpacked on the device from
   * d_raw into d_win[slot] */
  int raw_fmt; /* 0, or the enum filter_raw_format the master is fed */
  void *raw_ring;
  size_t raw_ring_size;
  char *raw_wp, *raw_rp;
  void *d_raw;
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
  /* I/Q correction (FILTER_RAW_*_IQCORR): a ring table of the writes (host copy, device copy), the device's coefficient
   * set and record of each write, and the pinned copy of the records */
  bool iq_on;
  struct kgpu_iq_params iq_par;
  int iq_cap;
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

static void master_teardown(struct filter_in *master) {
  struct master_ctx *c = (struct master_ctx *)master->fwd_plan;
  if (c) {
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
    ring_free(c->i16_ring, c->i16_ring_size);
    ring_free(c->raw_ring, c->raw_ring_size);
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

/* ---------------------------------------------------------------- raw ingest ---------------- */
/* bytes of n samples (REAL) or I/Q pairs (COMPLEX) in a raw format; a packed-12 n is a multiple of 8 (three words) */
static bool iq_format(int fmt) { return fmt == FILTER_RAW_S8_IQCORR || fmt == FILTER_RAW_S16_IQCORR; }
/* bytes per component */
static size_t raw_word(int fmt) { return fmt == FILTER_RAW_S16_IQCORR ? 2 : 1; }
static size_t raw_bytes(int fmt, bool cplx, size_t n) {
  return fmt == FILTER_RAW_PACKED12 ? n / 8 * 12 : n * (cplx ? 2 : 1) * raw_word(fmt);
}
static long raw_samples(int fmt, bool cplx, size_t bytes) {
  return (long)(fmt == FILTER_RAW_PACKED12 ? bytes / 12 * 8 : bytes / ((cplx ? 2 : 1) * raw_word(fmt)));
}
/* the device window holds int16 words (int16 ingest, or packed-12 after the unpack) rather than floats */
static bool ingest_i16(struct master_ctx const *c) { return c->i16_mode || c->raw_fmt == FILTER_RAW_PACKED12; }

long filter_raw_ring_bytes(int L, int M, enum filtertype in_type, int format) {
  if (L <= 0 || M <= 0 || (in_type != REAL && in_type != COMPLEX))
    return -1;
  bool const cplx = in_type == COMPLEX;
  size_t unit = page_round(1);
  if (format == FILTER_RAW_PACKED12) { /* whole groups, so a group never straddles the end of the ring */
    if (cplx || L % 8 != 0 || (M - 1) % 8 != 0)
      return -1;
    unit = unit / (size_t)gcd((long)unit, 12) * 12;
  } else if (iq_format(format)) {
    if (!cplx)
      return -1;
  } else if (format != FILTER_RAW_U8 && format != FILTER_RAW_S8)
    return -1;
  size_t const fsz = cplx ? sizeof(float complex) : sizeof(float);
  size_t const samples = page_round((size_t)ND * (size_t)(L + M - 1) * fsz) / fsz; /* the float ring's capacity */
  size_t const need = raw_bytes(format, cplx, (samples + 7) / 8 * 8);
  return (long)((need + unit - 1) / unit * unit);
}

/* the first write_rawfilter on a master: its ring, prefilled with the format's zero so the M-1 history samples (and
 * whatever the wideband analyzer's seeding reads before the stream reaches it) are 0.0 as in the float ring */
static int raw_start(struct filter_in *f, struct master_ctx *c, int format) {
  long const size = filter_raw_ring_bytes(f->ilen, f->impulse_length, f->in_type, format);
  if (size < 0) {
    fprintf(stderr, "write_rawfilter(L=%d M=%d): format %d cannot feed this master%s\n", f->ilen, f->impulse_length, format,
            format == FILTER_RAW_PACKED12 ? " (packed 12-bit needs a REAL master with L and M-1 multiples of 8)"
            : iq_format(format)          ? " (I/Q correction needs a COMPLEX master)"
                                         : "");
    return -1;
  }
  if (c->i16_mode || f->wcnt != 0 || c->issued != 0) {
    fprintf(stderr, "write_rawfilter: the master is already fed int16 or float samples\n");
    return -1;
  }
  bool const cplx = f->in_type == COMPLEX;
  c->raw_ring = ring_alloc((size_t)size);
  if (!c->raw_ring)
    return -1;
  c->raw_ring_size = (size_t)size;
  if (format == FILTER_RAW_U8)
    memset(c->raw_ring, 128, c->raw_ring_size);
  else if (format == FILTER_RAW_PACKED12) { /* eight offset-binary 2048s per three words (airspy-unpack.c:110-117) */
    uint32_t const g[3] = {0x80080080u, 0x08008008u, 0x00800800u};
    for (size_t o = 0; o < c->raw_ring_size; o += sizeof g)
      memcpy((char *)c->raw_ring + o, g, sizeof g);
  }
  size_t const span = (size_t)(ND - 2) * (size_t)f->ilen + (size_t)f->points;
  if (cudaMalloc(&c->d_raw, raw_bytes(format, cplx, span)) != cudaSuccess) {
    c->d_raw = NULL;
    ring_free(c->raw_ring, c->raw_ring_size);
    c->raw_ring = NULL;
    return kgf_fail("write_rawfilter: device buffer");
  }
  c->raw_rp = c->raw_ring;
  c->raw_wp = c->raw_rp + raw_bytes(format, cplx, (size_t)(f->impulse_length - 1));
  c->raw_fmt = format;
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
 * the 8-bit and I/Q corrected formats, int16 for packed-12, which kgpu_forward then scales.  d_stats: NULL or nblocks
 * block statistics (not for I/Q correction, whose records replace them). */
static int iq_apply(struct master_ctx const *c, void const *d_src, long long a0, long count, void *d_dst, cudaStream_t st);
static int raw_unpack(struct filter_in const *f, struct master_ctx const *c, int stage, void const *d_src, long long a0,
                      long history, int nblocks, void *d_dst, void *d_stats, cudaStream_t st) {
  int const type = f->in_type == COMPLEX ? KGPU_COMPLEX : KGPU_REAL;
  if (c->iq_on) /* a0: the absolute index of the first sample (I/Q correction needs to know whose write it is) */
    return iq_apply(c, d_src, a0, history + (long)nblocks * f->ilen, d_dst, st);
  if (c->raw_fmt != FILTER_RAW_PACKED12) {
    double scale;
    int n;
    if (chg_span(c, stage, a0, a0 + history + (long long)nblocks * f->ilen, &scale, &n) != 0)
      return -1;
    return kgpu_unpack8(d_src, c->raw_fmt == FILTER_RAW_U8 ? KGPU_RAW_U8 : KGPU_RAW_S8, type, history, f->ilen, nblocks, scale,
                        n ? c->d_chg : NULL, n, a0, d_dst, d_stats, st);
  }
  if (kgpu_unpack_airspy12(d_src, history + (long)nblocks * f->ilen, d_dst, NULL, st) != 0)
    return -1;
  return d_stats ? kgpu_block_stats_i16(d_dst, type, history, f->ilen, nblocks, 0, 2047, d_stats, st) : 0;
}

/* ---------------------------------------------------------------- I/Q correction ------------ */
/* Writes live in a ring table of iq_cap entries (write w at w % iq_cap), on the host and on the device.  It holds twice
 * the writes the raw ring can hold at FILTER_IQ_MIN_WRITE pairs each, plus the writes of the launches that may be in
 * flight: the writes of the analyzer's seeding window and those written but not yet launched both fit, so no entry is
 * overwritten while a launch or the seeding can still read it. */
long filter_iq_table_writes(int L, int M, enum filtertype in_type, int format) {
  if (!iq_format(format))
    return -1;
  long const bytes = filter_raw_ring_bytes(L, M, in_type, format);
  if (bytes < 0)
    return -1;
  return 2 * (raw_samples(format, true, (size_t)bytes) / FILTER_IQ_MIN_WRITE) + 2 * ND + 2;
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
  return kgpu_iq_apply(d_src, c->raw_fmt == FILTER_RAW_S8_IQCORR ? KGPU_IQ_S8 : KGPU_IQ_S16, a0, count, c->d_iqw, c->d_iqc,
                       c->iq_cap, (long long)w_lo, (int)(w_hi - w_lo + 1), d_dst, st);
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
  int const fmt = c->raw_fmt == FILTER_RAW_S8_IQCORR ? KGPU_IQ_S8 : KGPU_IQ_S16;
  unsigned long long const first = iq_find(c, old, c->iq_writes, a);
  char const *d_new = (char const *)c->d_raw + raw_bytes(c->raw_fmt, true, (size_t)(f->impulse_length - 1));
  if (kgpu_iq_moments(d_new, fmt, a, (long)(end - a), c->d_iqw, c->iq_cap, (long long)first, (int)(last - first + 1), c->st) != 0)
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
  c->acc.energy += s->energy;
  c->acc.overranges += s->overs;
  c->acc.overrange_samples += s->over_samples;
  c->acc.since_over = s->over_samples ? 0 : c->acc.since_over + (uint64_t)f->ilen;
  c->folded++;
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
  long const M1 = f->impulse_length - 1;
  c->sring_pos = (long)((M1 + (unsigned long long)f->ilen * c->issued) % (unsigned long long)c->sring_cap);
  if (c->raw_fmt) { /* the host ring holds raw bytes: send the last sring_cap samples' bytes over and unpack them there */
    bool const cplx = f->in_type == COMPLEX;
    long const n = c->sring_cap, cap = raw_samples(c->raw_fmt, cplx, c->raw_ring_size);
    long const end = raw_samples(c->raw_fmt, cplx, (size_t)(c->raw_rp - (char *)c->raw_ring)) + M1;
    long const src = ((end - n) % cap + cap) % cap;
    long const dst = c->sring_pos; /* (sring_pos - n) modulo sring_cap, n being sring_cap */
    long const first = n - dst;
    void *tmp = NULL;
    int rc = cudaMalloc(&tmp, raw_bytes(c->raw_fmt, cplx, (size_t)n)) == cudaSuccess ? 0 : -1;
    rc = rc ? rc
            : window_h2d(tmp, (char *)c->raw_ring + raw_bytes(c->raw_fmt, cplx, (size_t)src), raw_bytes(c->raw_fmt, cplx, (size_t)n),
                         c->raw_ring, c->raw_ring_size, c->st);
    long long const a0 = (long long)f->ilen * (long long)c->issued - n; /* the absolute index of the first seeded sample */
    rc = rc ? rc : raw_unpack(f, c, ND, tmp, a0, first, 0, (char *)c->d_sring + (size_t)dst * esz, NULL, c->st);
    if (rc == 0 && dst > 0)
      rc = raw_unpack(f, c, ND, (char *)tmp + raw_bytes(c->raw_fmt, cplx, (size_t)first), a0 + first, dst, 0, c->d_sring, NULL,
                      c->st);
    if (cudaStreamSynchronize(c->st) != cudaSuccess)
      rc = -1;
    cudaFree(tmp);
    return rc ? kgf_fail("filter_spectrum_setup: seeding the device ring from the raw ring") : 0;
  }
  char const *base;
  long src_cap, src_end;
  if (c->sring_i16) {
    base = c->i16_ring;
    src_cap = (long)(c->i16_ring_size / c->i16_esz);
    src_end = (long)((c->i16_rp - (char *)c->i16_ring) / (long)c->i16_esz) + M1;
  } else {
    base = f->input_buffer;
    src_cap = c->sring_cap;
    src_end = (long)(((char *)(f->in_type == COMPLEX ? (void *)f->input_read_pointer.c : (void *)f->input_read_pointer.r) -
                      (char *)f->input_buffer) / (long)c->esz) + M1;
  }
  long const n = c->sring_cap; /* the i16 ring holds at least as many samples as the float ring */
  long const src = ((src_end - n) % src_cap + src_cap) % src_cap;
  long const dst = ((c->sring_pos - n) % c->sring_cap + c->sring_cap) % c->sring_cap;
  if (sring_copy(c, base, src_cap, src, dst, n, esz, cudaMemcpyHostToDevice) != 0 || cudaStreamSynchronize(c->st) != cudaSuccess)
    return kgf_fail("filter_spectrum_setup: seeding the device ring");
  return 0;
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

/* k consecutive blocks (jobs next_jobnum .. +k-1, ring slots without wrap) as one device launch sequence.
 * filter.c:558-651 (+ run_fft :485-555) */
static int execute_filter_input_n(struct filter_in *const f, int const k) {
  struct master_ctx *c = (struct master_ctx *)f->fwd_plan;
  int const N = f->points;
  pthread_mutex_lock(&c->mu);
  unsigned const jobnum = f->next_jobnum;
  int const slot = (int)(jobnum % ND);
  /* the ring slots' previous occupants (job - ND) must have drained */
  for (int j = 0; j < k; j++)
    cudaEventSynchronize(c->done[slot + j]);
  if (c->stats_on && !c->i16_mode && !c->raw_fmt)
    c->stats_on = false; /* fed floats: the driver counts in its own loop */
  while (c->stats_on && c->folded + ND < c->issued + (unsigned long long)k)
    fold_one(f, c); /* the statistics of the slots about to be reused */
  while (c->iq_on && c->iq_checked + ND < c->issued + (unsigned long long)k)
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
  int rc = 0;
  cudaEventRecord(c->t0[slot], c->st);
  void const *src;
  int fmt = KGPU_FMT_F32;
  float scale = 1.0f;
  size_t bytes;
  size_t const span = (size_t)(k - 1) * (size_t)f->ilen + (size_t)N; /* samples covered by k overlapping windows */
  if (c->i16_mode) {
    src = c->i16_rp;
    bytes = c->i16_esz * span;
    fmt = KGPU_FMT_I16;
    c->i16_rp += c->i16_esz * (size_t)f->ilen * (size_t)k;
    if (c->i16_rp >= (char *)c->i16_ring + c->i16_ring_size)
      c->i16_rp -= c->i16_ring_size;
  } else if (c->raw_fmt) { /* packed-12 goes on as int16 with the drivers' float scale; 8-bit as floats */
    bool const cplx = f->in_type == COMPLEX;
    src = c->raw_rp;
    bytes = raw_bytes(c->raw_fmt, cplx, span);
    fmt = c->raw_fmt == FILTER_RAW_PACKED12 ? KGPU_FMT_I16 : KGPU_FMT_F32;
    c->raw_rp += raw_bytes(c->raw_fmt, cplx, (size_t)f->ilen * (size_t)k);
    if (c->raw_rp >= (char *)c->raw_ring + c->raw_ring_size)
      c->raw_rp -= c->raw_ring_size;
  } else if (f->in_type == COMPLEX) {
    src = f->input_read_pointer.c;
    bytes = sizeof(float complex) * span;
    f->input_read_pointer.c += (size_t)f->ilen * (size_t)k;
    kgf_ring_wrap((void **)&f->input_read_pointer.c, f->input_buffer, f->input_buffer_size);
  } else {
    src = f->input_read_pointer.r;
    bytes = sizeof(float) * span;
    f->input_read_pointer.r += (size_t)f->ilen * (size_t)k;
    kgf_ring_wrap((void **)&f->input_read_pointer.r, f->input_buffer, f->input_buffer_size);
  }
  float complex *spec = c->d_spec + (size_t)slot * (size_t)c->spec_stride;
  for (int j = 0; j < k; j++) /* nothing of the previous occupants may be served for these jobs */
    for (int i = 0; i < c->nslots; i++)
      c->snap[slot + j][i].ok = false;
  void const *const ring = c->i16_mode ? c->i16_ring : c->raw_fmt ? c->raw_ring : f->input_buffer;
  size_t const ring_size = c->i16_mode ? c->i16_ring_size : c->raw_fmt ? c->raw_ring_size : f->input_buffer_size;
  if (window_h2d(c->raw_fmt ? c->d_raw : c->d_win[slot], src, bytes, ring, ring_size, c->st) != 0)
    rc = kgf_fail("execute_filter_input: H2D of the window");
  long const M1 = f->impulse_length - 1;
  long long const a0 = (long long)f->ilen * (long long)c->issued - M1; /* the window's first sample */
  if (c->chg)
    chg_prune(f, c);
  if (rc == 0 && c->iq_on && iq_launch(f, c, k) != 0)
    rc = kgf_fail("execute_filter_input: I/Q correction");
  if (rc == 0 && c->raw_fmt && raw_unpack(f, c, slot, c->d_raw, a0, M1, k, c->d_win[slot], bst, c->st) != 0)
    rc = kgf_fail("execute_filter_input: raw unpack");
  if (rc == 0 && c->i16_mode && bst &&
      kgpu_block_stats_i16(c->d_win[slot], f->in_type == COMPLEX ? KGPU_COMPLEX : KGPU_REAL, M1, f->ilen, k, c->i16_derand, 32767,
                           bst, c->st) != 0)
    rc = kgf_fail("execute_filter_input: kgpu_block_stats_i16");
  void const *fwd_in = c->d_win[slot];
  if (rc == 0 && fmt == KGPU_FMT_I16) { /* one scale: fwd_cols converts; more: floats with each sample's own scale */
    double s;
    int n;
    if (chg_span(c, slot, a0, a0 + (long long)span, &s, &n) != 0)
      rc = kgf_fail("execute_filter_input: scale changes");
    else if (n == 0)
      scale = (float)s;
    else if (kgpu_scale_i16(c->d_win[slot], f->in_type == COMPLEX ? KGPU_COMPLEX : KGPU_REAL, (long)span, a0, s, c->d_chg, n,
                            c->i16_mode && c->i16_derand, c->d_conv, c->st) != 0)
      rc = kgf_fail("execute_filter_input: kgpu_scale_i16");
    else {
      fwd_in = c->d_conv;
      fmt = KGPU_FMT_F32;
    }
  }
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
  if (c->iq_on) {
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
  pthread_mutex_lock(&c->mu);
  /* only this master's pipeline stream is synchronised: a retune of one channel must not stall other masters
   * (filter2 / wfm composite masters of other channel threads) the way a device-wide synchronisation would */
  int rc = kgpu_bank_set_filter_on(c->bank, sc->idx, low, high, kaiser_beta, c->st);
  if (rc == 0)
    rc = kgpu_bank_get_response(c->bank, sc->idx, (float *)host) > 0 ? 0 : -1;
  if (rc == 0)
    c->ver[sc->idx]++;
  pthread_mutex_unlock(&c->mu);
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
                                   (float)scale, n ? c->d_chg : NULL, n, (long long)end, c->i16_mode && c->i16_derand, shift,
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
  if (slave->out_type == SPECTRUM && slave->master && slave->master->fwd_plan) {
    struct master_ctx *c = (struct master_ctx *)slave->master->fwd_plan;
    pthread_mutex_lock(&c->mu);
    spec_slave_drop(c, slave);
    pthread_mutex_unlock(&c->mu);
  }
  if (sc && slave->master && slave->master->fwd_plan) {
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
/* a master fed raw words takes no floats */
static bool raw_fed(struct filter_in const *f) { return f->fwd_plan && ((struct master_ctx const *)f->fwd_plan)->raw_fmt; }
int write_cfilter(struct filter_in *f, float complex const *buffer, int size) { /* filter.c:1093-1113 */
  if (f == NULL || raw_fed(f))
    return -1;
  if ((f->wcnt + size) * sizeof *buffer >= f->input_buffer_size)
    return -1;
  if (buffer != NULL)
    memcpy(f->input_write_pointer.c, buffer, (size_t)size * sizeof *buffer);
  f->input_write_pointer.c += size;
  kgf_ring_wrap((void **)&f->input_write_pointer.c, f->input_buffer, f->input_buffer_size);
  f->wcnt += size;
  return fire_ready_blocks(f);
}
int write_rfilter(struct filter_in *f, float const *buffer, int size) { /* filter.c:1114-1134 */
  if (f == NULL || raw_fed(f))
    return -1;
  if ((f->wcnt + size) * sizeof *buffer >= f->input_buffer_size)
    return -1;
  if (buffer != NULL)
    memcpy(f->input_write_pointer.r, buffer, (size_t)size * sizeof *buffer);
  f->input_write_pointer.r += size;
  kgf_ring_wrap((void **)&f->input_write_pointer.r, f->input_buffer, f->input_buffer_size);
  f->wcnt += size;
  return fire_ready_blocks(f);
}
/* EXTENSION: raw ADC words straight to the device; conversion (rx888.c:753-767) happens in fwd_cols.
 * samples == NULL: the caller already wrote them through filter_i16_write_pointer() (the zero-copy driver path). */
int write_i16filter(struct filter_in *f, int16_t const *samples, int n, float scale, bool derandomize) {
  if (f == NULL || f->fwd_plan == NULL || n < 0)
    return -1;
  struct master_ctx *c = (struct master_ctx *)f->fwd_plan;
  if (!c->i16_mode && filter_i16_write_pointer(f) == NULL)
    return -1;
  if (((size_t)f->wcnt + (size_t)n) * c->i16_esz >= c->i16_ring_size)
    return -1;
  pthread_mutex_lock(&c->mu);
  int const rc = chg_note(f, c, scale, "write_i16filter");
  pthread_mutex_unlock(&c->mu);
  if (rc != 0)
    return -1;
  c->i16_derand = derandomize;
  if (samples != NULL)
    memcpy(c->i16_wp, samples, (size_t)n * c->i16_esz);
  c->i16_wp += (size_t)n * c->i16_esz;
  if (c->i16_wp >= (char *)c->i16_ring + c->i16_ring_size)
    c->i16_wp -= c->i16_ring_size;
  f->wcnt += n;
  return fire_ready_blocks(f);
}
/* where a driver may deposit the next raw samples itself (mirrored, pinned ring: up to one block contiguous),
 * e.g. as the libusb transfer buffer of rx888.c:797-826; publish with write_i16filter(f, NULL, n, ...) */
int16_t *filter_i16_write_pointer(struct filter_in *f) {
  if (f == NULL || f->fwd_plan == NULL || raw_fed(f))
    return NULL;
  struct master_ctx *c = (struct master_ctx *)f->fwd_plan;
  if (!c->i16_mode) {
    c->i16_esz = (f->in_type == COMPLEX) ? 2 * sizeof(int16_t) : sizeof(int16_t);
    c->i16_ring_size = page_round((size_t)ND * (size_t)f->points * c->i16_esz);
    c->i16_ring = ring_alloc(c->i16_ring_size);
    if (!c->i16_ring)
      return NULL;
    c->i16_rp = c->i16_ring;
    c->i16_wp = c->i16_rp + c->i16_esz * (size_t)(f->impulse_length - 1);
    c->i16_mode = true;
  }
  return (int16_t *)c->i16_wp;
}

/* EXTENSION: raw packed 12-bit or 8-bit ADC words, unpacked on the device (see include/ka9q_gpu_filter.h).  The drivers
 * (airspy.c:388-434, hydrasdr.c:663-679, :759-830, rtlsdr.c:316-343) get their buffers from their vendor libraries, so
 * there is no zero-copy write pointer: the bytes are copied into the raw ring. */
int write_rawfilter(struct filter_in *f, void const *samples, int n, int format, double scale) {
  if (f == NULL || f->fwd_plan == NULL || samples == NULL || n < 0)
    return -1;
  struct master_ctx *c = (struct master_ctx *)f->fwd_plan;
  if (format != FILTER_RAW_PACKED12 && format != FILTER_RAW_U8 && format != FILTER_RAW_S8 && !iq_format(format)) {
    fprintf(stderr, "write_rawfilter: unknown format %d\n", format);
    return -1;
  }
  if (iq_format(format) && !c->iq_on) {
    fprintf(stderr, "write_rawfilter: format %d needs filter_iq_correction_setup first\n", format);
    return -1;
  }
  if (!c->raw_fmt && raw_start(f, c, format) != 0)
    return -1;
  if (format != c->raw_fmt) {
    fprintf(stderr, "write_rawfilter: format %d on a master fed format %d\n", format, c->raw_fmt);
    return -1;
  }
  if (format == FILTER_RAW_PACKED12 && n % 8 != 0) {
    fprintf(stderr, "write_rawfilter: %d packed 12-bit samples: not a multiple of 8\n", n);
    return -1;
  }
  bool const cplx = f->in_type == COMPLEX;
  if (raw_bytes(format, cplx, (size_t)f->wcnt + (size_t)n) >= c->raw_ring_size)
    return -1;
  if (c->iq_on) { /* one transfer: its table entry */
    if (n < FILTER_IQ_MIN_WRITE) {
      fprintf(stderr, "write_rawfilter: %d I/Q pairs: writes with I/Q correction take at least %d\n", n, FILTER_IQ_MIN_WRITE);
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
  }
  if (!c->iq_on) {
    pthread_mutex_lock(&c->mu);
    int const rc = chg_note(f, c, scale, "write_rawfilter");
    pthread_mutex_unlock(&c->mu);
    if (rc != 0)
      return -1;
  }
  size_t const bytes = raw_bytes(format, cplx, (size_t)n);
  memcpy(c->raw_wp, samples, bytes); /* the mirror view keeps a write across the end contiguous */
  c->raw_wp += bytes;
  if (c->raw_wp >= (char *)c->raw_ring + c->raw_ring_size)
    c->raw_wp -= c->raw_ring_size;
  f->wcnt += n;
  return fire_ready_blocks(f);
}

/* EXTENSION: the A/D statistics of the blocks whose device work completed since the previous call (see
 * include/ka9q_gpu_filter.h).  The slots about to be reused are folded in by execute_filter_input_n, which has already
 * waited for them; this call folds, in job order, whatever else has completed, without waiting. */
int filter_ingest_stats(struct filter_in *f, struct filter_ingest_stats *stats) {
  if (f == NULL || f->fwd_plan == NULL || stats == NULL)
    return -1;
  struct master_ctx *c = (struct master_ctx *)f->fwd_plan;
  if (c->iq_on)
    return -1; /* I/Q corrected: filter_iq_records replaces the block statistics */
  int rc = 0;
  pthread_mutex_lock(&c->mu);
  if (!c->i16_mode && !c->raw_fmt && (c->issued > 0 || f->wcnt > 0))
    rc = -1; /* fed floats */
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
  if (f == NULL || f->fwd_plan == NULL || p == NULL || !iq_format(format))
    return -1;
  struct master_ctx *c = (struct master_ctx *)f->fwd_plan;
  if (c->raw_fmt || c->iq_on) {
    fprintf(stderr, "filter_iq_correction_setup: the master is already fed raw words\n");
    return -1;
  }
  long const cap = filter_iq_table_writes(f->ilen, f->impulse_length, f->in_type, format);
  if (cap < 0) {
    fprintf(stderr, "filter_iq_correction_setup(L=%d M=%d): I/Q correction needs a COMPLEX master\n", f->ilen, f->impulse_length);
    return -1;
  }
  if (raw_start(f, c, format) != 0)
    return -1;
  c->iq_cap = (int)cap;
  size_t const nw = (size_t)cap;
  bool ok = cudaHostAlloc((void **)&c->h_iqw, sizeof *c->h_iqw * nw, cudaHostAllocPortable) == cudaSuccess;
  ok = ok && cudaMalloc((void **)&c->d_iqw, sizeof *c->d_iqw * nw) == cudaSuccess;
  ok = ok && cudaMalloc((void **)&c->d_iqc, sizeof *c->d_iqc * nw) == cudaSuccess;
  ok = ok && cudaMalloc((void **)&c->d_iqr, sizeof *c->d_iqr * nw) == cudaSuccess;
  ok = ok && cudaHostAlloc((void **)&c->h_iqr, sizeof *c->h_iqr * nw, cudaHostAllocPortable) == cudaSuccess;
  struct kgpu_iq_state const init = {p->dc_i, p->dc_q, p->sinphi, p->imbalance, p->gain_i, p->gain_q, p->secphi, p->tanphi};
  ok = ok && cudaMemcpy(c->d_iqc, &init, sizeof init, cudaMemcpyHostToDevice) == cudaSuccess; /* write 0's coefficients */
  if (!ok)
    return kgf_fail("filter_iq_correction_setup: table buffers"); /* freed with the master */
  c->iq_par.kind = p->gp_rate != 0 ? 1 : 2;
  c->iq_par.dc_alpha = p->dc_alpha;
  c->iq_par.gp = p->gp_rate != 0 ? p->gp_rate : p->gp_alpha;
  c->iq_on = true;
  return 0;
}

/* EXTENSION: the records of the writes whose launch has completed (see include/ka9q_gpu_filter.h).  The launches' slots
 * about to be reused are taken in by execute_filter_input_n, which has already waited for them; this call takes in, in
 * job order, whatever else has completed, without waiting. */
int filter_iq_records(struct filter_in *f, struct filter_iq_record *recs, int max) {
  if (f == NULL || f->fwd_plan == NULL || (recs == NULL && max > 0))
    return -1;
  struct master_ctx *c = (struct master_ctx *)f->fwd_plan;
  if (!c->iq_on)
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
