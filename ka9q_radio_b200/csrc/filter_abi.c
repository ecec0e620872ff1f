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
};

struct snap { /* what the batched launch of one ring slot used for one slave */
  int shift;
  unsigned ver, ft_ver;
  long off;
  bool isb, beam, ok;
  double complex alpha, beta;
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
  float i16_scale;
  bool i16_derand;
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
  c->km = kgpu_master_create(L, M, in_type == REAL ? KGPU_REAL : KGPU_COMPLEX);
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
    int const pts = kgpu_bank_define_ex(c->bank, sc->idx, len, out_type == REAL ? KGPU_REAL : KGPU_COMPLEX);
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
    scale = c->i16_scale;
    c->i16_rp += c->i16_esz * (size_t)f->ilen * (size_t)k;
    if (c->i16_rp >= (char *)c->i16_ring + c->i16_ring_size)
      c->i16_rp -= c->i16_ring_size;
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
  if (window_h2d(c->d_win[slot], src, bytes, c->i16_mode ? c->i16_ring : f->input_buffer,
                 c->i16_mode ? c->i16_ring_size : f->input_buffer_size, c->st) != 0)
    rc = kgf_fail("execute_filter_input: H2D of the window");
  if (rc == 0 && kgpu_forward(c->km, c->d_win[slot], fmt, scale, c->i16_derand, k, spec, NULL, c->st) != 0)
    rc = kgf_fail("execute_filter_input: kgpu_forward");
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
    pthread_mutex_unlock(&c->mu);
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

/* ---------------------------------------------------------------- delete -------------------- */
int delete_filter_output(struct filter_out *slave) { /* filter.c:943-957 */
  if (slave == NULL)
    return -1;
  struct slave_ctx *sc = (struct slave_ctx *)slave->rev_plan;
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
    pthread_mutex_unlock(&c->mu);
  }
  if (sc)
    free(sc->own);
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
int write_cfilter(struct filter_in *f, float complex const *buffer, int size) { /* filter.c:1093-1113 */
  if (f == NULL)
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
  if (f == NULL)
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
  c->i16_scale = scale;
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
  if (f == NULL || f->fwd_plan == NULL)
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
