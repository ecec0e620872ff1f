// kgpu.cu -- host side of libka9qgpu.so: plan registry, forward-transform and channel-bank
// launchers behind the C-ABI declared in include/ka9q_gpu.h.  No CPU fallback anywhere: every
// entry point either launches the sm_90a kernels or fails with -1.
#include <cuda_runtime.h>
#include <math.h>
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <algorithm>
#include <atomic>
#include <mutex>
#include <string>
#include <vector>

#include "../../include/ka9q_gpu.h"
#include "chan_kernels.cuh"
#include "fwd_kernels.cuh"
#include "noise_kernel.cuh"
#include "plan.cuh"
#include "static_kernels.cuh"
#include "static_kernels_v2.cuh"
#include "fwd_cols_r36.cuh"
#include "fwd_2s.cuh"
#include "fwd_rows_r50.cuh"

using namespace kfft;

// ------------------------------------------------------------------------------------------
static thread_local std::string g_err;
static std::atomic<unsigned long long> g_launches{0};

static std::atomic<int> g_tuning[16];
static int sm_count() {
  static int n = 0;
  if (!n) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    if (n <= 0) n = 132;  // H100 SXM
  }
  return n;
}      // experiment knobs (kgpu_set_tuning), 0 = default
extern "C" int kgpu_set_tuning(int key, int value) {
  if (key < 0 || key >= 16) return -1;
  g_tuning[key].store(value);
  return 0;
}
static void *g_dbg_buf = nullptr, *g_dbg_buf2 = nullptr;  // per-CTA phase timestamps (tools/phase_trace.py)
extern "C" int kgpu_set_debug_buffer(void *d_buf) {
  g_dbg_buf = d_buf;
  return 0;
}
extern "C" int kgpu_set_debug_buffer_rows(void *d_buf) {
  g_dbg_buf2 = d_buf;
  return 0;
}
static std::atomic<int> g_static_on{1};  // tests can force the generic kernels
extern "C" int kgpu_use_static_kernels(int on) {
  g_static_on.store(on != 0);
  return 0;
}

static int fail(char const *fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof buf, fmt, ap);
  va_end(ap);
  g_err = buf;
  return -1;
}
#define CUDA_OK(expr)                                                                    \
  do {                                                                                   \
    cudaError_t e_ = (expr);                                                             \
    if (e_ != cudaSuccess) return fail("%s: %s (%s:%d)", #expr, cudaGetErrorString(e_), __FILE__, __LINE__); \
  } while (0)
#define CUDA_OKP(expr)                                                                   \
  do {                                                                                   \
    cudaError_t e_ = (expr);                                                             \
    if (e_ != cudaSuccess) {                                                             \
      fail("%s: %s (%s:%d)", #expr, cudaGetErrorString(e_), __FILE__, __LINE__);         \
      return nullptr;                                                                    \
    }                                                                                    \
  } while (0)

// ------------------------------------------------------------------ per-launch profiling -----
// When enabled, every kernel launch is bracketed by CUDA events on the launching stream; bench.py
// reads the per-kernel totals for its roofline line (events are markers, they do not serialise).
enum KernelId { K_FWD_COLS = 0, K_FWD_ROWS, K_CHAN, K_NOTCH, K_RESPONSE, K_NOISE, K_COUNT };
static char const *const kKernelNames[K_COUNT] = {"fwd_cols", "fwd_rows", "chan", "notch", "response_fft", "noise"};
struct ProfRec {
  cudaEvent_t a, b;
  int kid;
};
static std::atomic<int> g_prof_on{0};
static std::mutex g_prof_mu;
static std::vector<ProfRec> g_prof_pending;
static std::vector<cudaEvent_t> g_prof_pool;
static double g_prof_ms[K_COUNT];
static long g_prof_cnt[K_COUNT];

static cudaEvent_t prof_event() {
  if (!g_prof_pool.empty()) {
    cudaEvent_t e = g_prof_pool.back();
    g_prof_pool.pop_back();
    return e;
  }
  cudaEvent_t e;
  cudaEventCreate(&e);
  return e;
}
struct ProfScope {
  ProfRec r;
  cudaStream_t st;
  bool on;
  ProfScope(int kid, cudaStream_t s) : st(s), on(g_prof_on.load() != 0) {
    if (!on) return;
    std::lock_guard<std::mutex> lk(g_prof_mu);
    r.a = prof_event();
    r.b = prof_event();
    r.kid = kid;
    cudaEventRecord(r.a, st);
  }
  ~ProfScope() {
    if (!on) return;
    cudaEventRecord(r.b, st);
    std::lock_guard<std::mutex> lk(g_prof_mu);
    g_prof_pending.push_back(r);
  }
};
static void prof_drain() {
  std::lock_guard<std::mutex> lk(g_prof_mu);
  for (ProfRec &r : g_prof_pending) {
    float ms = 0;
    if (cudaEventSynchronize(r.b) == cudaSuccess && cudaEventElapsedTime(&ms, r.a, r.b) == cudaSuccess) {
      g_prof_ms[r.kid] += ms;
      g_prof_cnt[r.kid]++;
    }
    g_prof_pool.push_back(r.a);
    g_prof_pool.push_back(r.b);
  }
  g_prof_pending.clear();
}
extern "C" int kgpu_profile_enable(int on) {
  g_prof_on.store(on != 0);
  return 0;
}
extern "C" int kgpu_profile_reset(void) {
  prof_drain();
  for (int i = 0; i < K_COUNT; i++) {
    g_prof_ms[i] = 0;
    g_prof_cnt[i] = 0;
  }
  return 0;
}
extern "C" int kgpu_profile_kernels(void) { return K_COUNT; }
extern "C" const char *kgpu_profile_name(int kid) { return (kid >= 0 && kid < K_COUNT) ? kKernelNames[kid] : ""; }
extern "C" int kgpu_profile_get(int kid, double *total_ms, long *count) {
  if (kid < 0 || kid >= K_COUNT) return -1;
  prof_drain();
  if (total_ms) *total_ms = g_prof_ms[kid];
  if (count) *count = g_prof_cnt[kid];
  return 0;
}

extern "C" const char *kgpu_last_error(void) { return g_err.c_str(); }
extern "C" unsigned long long kgpu_launch_count(void) { return g_launches.load(); }
// ---- spectrum hand-off over NVSwitch multicast ---------------------------------------------------
// Streaming copy local HBM -> multicast address: 16-byte no-allocate loads, multimem.st stores (the
// switch replicates each store to every GPU bound to the multicast object).  256 threads and <= 32
// registers per CTA so that the CTAs fit beside two resident forward CTAs on an SM.
__global__ void __launch_bounds__(256) mc_push_kernel(float4 const *__restrict__ src, float4 *mc_dst, size_t n16) {
  size_t const stride = (size_t)gridDim.x * 256;
  size_t i = (size_t)blockIdx.x * 256 + threadIdx.x;
  for (; i + 3 * stride < n16; i += 4 * stride) {
    float4 v[4];
#pragma unroll
    for (int q = 0; q < 4; q++)
      asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
                   : "=f"(v[q].x), "=f"(v[q].y), "=f"(v[q].z), "=f"(v[q].w)
                   : "l"(src + i + q * stride));
#pragma unroll
    for (int q = 0; q < 4; q++)
      asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(mc_dst + i + q * stride), "f"(v[q].x),
                   "f"(v[q].y), "f"(v[q].z), "f"(v[q].w)
                   : "memory");
  }
  for (; i < n16; i += stride) {
    float4 v;
    asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(src + i));
    asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(mc_dst + i), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w)
                 : "memory");
  }
  __threadfence_system();  // this thread's multicast stores are performed system-wide before the kernel retires
}
extern "C" int kgpu_multicast_copy(const void *d_src, void *mc_dst, unsigned long long bytes, int nctas, void *stream) {
  if (!d_src || !mc_dst || (bytes & 15) || ((uintptr_t)d_src & 15) || ((uintptr_t)mc_dst & 15))
    return fail("kgpu_multicast_copy: pointers and size must be multiples of 16 bytes");
  if (bytes == 0) return 0;
  if (nctas <= 0) nctas = 64;
  mc_push_kernel<<<nctas, 256, 0, (cudaStream_t)stream>>>((float4 const *)d_src, (float4 *)mc_dst, (size_t)(bytes / 16));
  g_launches++;
  CUDA_OK(cudaGetLastError());
  return 0;
}

// ---- Airspy R2 / HydraSDR packed 12-bit ingest (airspy-unpack.c:17-130) ------------------------------------------
// 8 offset-binary 12-bit samples in three 32-bit words -> 8 int16 (s - 2048), which the forward transform's fused
// int16 ingest then scales exactly as the reference's `scale * (float)x`.  One thread per group: 12 contiguous bytes in,
// one 16-byte store out.  Energy and clip count (x == 2047 || x <= -2047) as the reference returns them.
__global__ void __launch_bounds__(256) airspy_unpack_kernel(uint32_t const *__restrict__ up, long ngroups, uint4 *__restrict__ out,
                                                            IngestStats *stats) {
  long const g = (long)blockIdx.x * 256 + threadIdx.x;
  unsigned long long energy = 0;
  unsigned int clips = 0;
  if (g < ngroups) {
    uint32_t const w0 = __ldg(up + 3 * g), w1 = __ldg(up + 3 * g + 1), w2 = __ldg(up + 3 * g + 2);
    uint32_t s[8] = {w0 >> 20, w0 >> 8, (w0 << 4) | (w1 >> 28), w1 >> 16, w1 >> 4, (w1 << 8) | (w2 >> 24), w2 >> 12, w2};
    int x[8];
#pragma unroll
    for (int j = 0; j < 8; j++) {
      x[j] = (int)(s[j] & 0xfffu) - 2048;
      clips += (x[j] == 2047 || x[j] <= -2047);
      energy += (unsigned long long)(x[j] * x[j]);
    }
    uint4 o;
    o.x = (uint32_t)(x[0] & 0xffff) | ((uint32_t)x[1] << 16);
    o.y = (uint32_t)(x[2] & 0xffff) | ((uint32_t)x[3] << 16);
    o.z = (uint32_t)(x[4] & 0xffff) | ((uint32_t)x[5] << 16);
    o.w = (uint32_t)(x[6] & 0xffff) | ((uint32_t)x[7] << 16);
    out[g] = o;
  }
  if (stats) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      energy += __shfl_xor_sync(0xffffffffu, energy, o);
      clips += __shfl_xor_sync(0xffffffffu, clips, o);
    }
    if ((threadIdx.x & 31) == 0 && (energy | clips)) {
      atomicAdd(&stats->energy, energy);
      atomicAdd(&stats->clips, clips);
    }
  }
}
extern "C" int kgpu_unpack_airspy12(const void *d_packed, long sampcount, void *d_i16, void *d_stats, void *stream) {
  if (!d_packed || !d_i16 || sampcount < 0 || (sampcount & 7)) return fail("kgpu_unpack_airspy12: sample count must be a multiple of 8");
  if (((uintptr_t)d_i16 & 15) || ((uintptr_t)d_packed & 3)) return fail("kgpu_unpack_airspy12: output must be 16-byte aligned");
  if (sampcount == 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  if (d_stats) CUDA_OK(cudaMemsetAsync(d_stats, 0, sizeof(IngestStats), st));
  long const ng = sampcount / 8;
  airspy_unpack_kernel<<<(unsigned)((ng + 255) / 256), 256, 0, st>>>((uint32_t const *)d_packed, ng, (uint4 *)d_i16, (IngestStats *)d_stats);
  g_launches++;
  CUDA_OK(cudaGetLastError());
  return 0;
}

extern "C" int kgpu_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) return 0;
  return n;
}
extern "C" int kgpu_set_device(int device) {
  CUDA_OK(cudaSetDevice(device));
  return 0;
}

// ------------------------------------------------------------------ radix selection ---------
namespace kfft {

static int const kRadixSet[] = {25, 24, 20, 16, 15, 12, 10, 9, 8, 7, 6, 5, 4, 3, 2};

// exhaustive search over multisets of supported radices (depth <= kMaxStages): fewest stages,
// then smallest sum.
static void search(int n, int start, std::vector<int> &cur, std::vector<int> &best, int &best_sum) {
  if (n == 1) {
    int sum = 0;
    for (int r : cur) sum += r;
    if (best.empty() || cur.size() < best.size() || (cur.size() == best.size() && sum < best_sum)) {
      best = cur;
      best_sum = sum;
    }
    return;
  }
  if ((int)cur.size() >= kMaxStages) return;
  if (!best.empty() && cur.size() + 1 > best.size()) return;
  for (int i = start; i < (int)(sizeof kRadixSet / sizeof kRadixSet[0]); i++) {
    int const r = kRadixSet[i];
    if (n % r) continue;
    cur.push_back(r);
    search(n / r, i, cur, best, best_sum);
    cur.pop_back();
  }
}

std::vector<int> choose_radices(int n) {
  std::vector<int> cur, best;
  int best_sum = 0;
  if (n < 2) return best;
  search(n, 0, cur, best, best_sum);
  // even radices first (descending): power-of-two strides stay away from the unit-stride stages;
  // odd ones last, descending: the last (unit-stride) stage gets the smallest radix, which is the
  // one the v2 kernels fuse with the global store / real split (fewest registers per butterfly)
  std::stable_sort(best.begin(), best.end(), [](int a, int b) {
    bool const ea = (a % 2 == 0), eb = (b % 2 == 0);
    if (ea != eb) return ea;
    return a > b;
  });
  return best;
}

struct PlanSlot {
  int len = 0;
  TilePlan host;  // device pointers inside
};
static std::mutex g_plan_mu;
static std::vector<PlanSlot> g_plans;

int get_tile_plan(int len) {
  std::lock_guard<std::mutex> lk(g_plan_mu);
  for (size_t i = 0; i < g_plans.size(); i++)
    if (g_plans[i].len == len) return (int)i;
  if ((int)g_plans.size() >= kMaxPlans || len < 1 || len > 65535) return -1;
  std::vector<int> rad;
  if (len > 1) {
    rad = choose_radices(len);
    if (rad.empty()) return -1;
  }
  TilePlan p;
  memset(&p, 0, sizeof p);
  p.len = len;
  p.nstages = (int)rad.size();
  std::vector<float2> tw;
  int n = len;
  for (int i = 0; i < p.nstages; i++) {
    int const r = rad[i], s = n / r;
    p.radix[i] = r;
    p.sub[i] = n;
    p.stride[i] = s;
    p.magic[i] = (s > 1) ? (uint32_t)(((1ull << 32) + (unsigned)s - 1) / (unsigned)s) : 0u;
    p.tw_off[i] = (int)tw.size();
    if (s > 1)
      for (int t = 1; t < r; t++)
        for (int j = 0; j < s; j++) {
          long double const ang = -2.0L * M_PIl * (long double)((long)j * t % n) / (long double)n;
          tw.push_back(make_float2((float)cosl(ang), (float)sinl(ang)));
        }
    n = s;
  }
  std::vector<uint16_t> perm((size_t)len);
  for (int k = 0; k < len; k++) {
    int rem = k, slot = 0;
    for (int i = 0; i < p.nstages; i++) {
      int const t = rem % p.radix[i];
      rem /= p.radix[i];
      slot += t * p.stride[i];
    }
    perm[k] = (uint16_t)slot;
  }
  float2 *d_tw = nullptr;
  uint16_t *d_perm = nullptr;
  tw.push_back(make_float2(0.f, 0.f));  // padding: bulk (16-byte granular) copies may read one entry past the end
  tw.push_back(make_float2(0.f, 0.f));
  if (cudaMalloc(&d_tw, sizeof(float2) * std::max<size_t>(tw.size(), 1)) != cudaSuccess) return -1;
  if (cudaMalloc(&d_perm, sizeof(uint16_t) * (size_t)len) != cudaSuccess) return -1;
  if (!tw.empty()) cudaMemcpy(d_tw, tw.data(), sizeof(float2) * tw.size(), cudaMemcpyHostToDevice);
  cudaMemcpy(d_perm, perm.data(), sizeof(uint16_t) * (size_t)len, cudaMemcpyHostToDevice);
  p.tw = d_tw;
  p.perm = d_perm;
  int const idx = (int)g_plans.size();
  if (cudaMemcpyToSymbol(c_plans, &p, sizeof p, sizeof(TilePlan) * (size_t)idx) != cudaSuccess) return -1;
  PlanSlot sl;
  sl.len = len;
  sl.host = p;
  g_plans.push_back(sl);
  return idx;
}
TilePlan const *host_tile_plan(int idx) { return &g_plans[(size_t)idx].host; }

static bool plannable(int len) { return len == 1 || (len <= kMaxTileLen && !choose_radices(len).empty()); }

bool choose_split(long n, Split2 *out) {
  long best = -1;
  for (long d = (long)floor(sqrt((double)n) + 1e-9); d >= 1; d--) {
    if (n % d) continue;
    long const a = n / d;  // a >= d
    if (a > kMaxTileLen) break;
    if (plannable((int)a) && plannable((int)d)) {
      best = d;
      break;
    }
  }
  if (best < 0) return false;
  out->n1 = (int)(n / best);
  out->n2 = (int)best;
  return true;
}
}  // namespace kfft

// ------------------------------------------------------------------ master ------------------
struct kgpu_master {
  int L, M, N, in_type, bins;
  long nc;           // complex points of the two-pass transform (N/2 for REAL, N for COMPLEX)
  Split2 sp;
  int plan1, plan2, pitch1, pitch2;
  long spec_stride;
  RowItem *d_items = nullptr;
  int n_item_ctas = 0;
  float2 *d_rootD = nullptr;
  float2 *d_rootC = nullptr;                                      // split roots of the row pass
  float2 *d_twU = nullptr, *d_twT = nullptr;                      // v2 cols kernel (1296 columns)
  float2 *d_r36_tw0 = nullptr, *d_r36_A = nullptr, *d_r36_B = nullptr;  // 36 x 36 cols kernel
  int static_cols = 0, static_rows = 0;  // which specialised kernels apply (0 = generic)
  int static_2s = 0;                     // 1: COMPLEX 800 x 625 on the two-fat-stage kernels of fwd_2s.cuh
  float2 *d_2s_tw0 = nullptr, *d_2s_A = nullptr, *d_2s_B = nullptr, *d_2s_rtw0 = nullptr;
  float2 *d_r50_tw0 = nullptr;           // 50 x 25 row kernel (REAL masters with 1250 columns)
  float2 *d_mid = nullptr;
  int mid_blocks = 0;
  size_t smem1 = 0, smem2 = 0;
  // notches
  NotchDev *d_notch = nullptr;
  int n_notch = 0;
  int notch_sequential = 0;
};

static int set_smem(const void *func, size_t bytes) {
  if (bytes > 48 * 1024)
    CUDA_OK(cudaFuncSetAttribute(func, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
  return 0;
}

extern "C" kgpu_master *kgpu_master_create(int L, int M, int in_type) {
  if (L < 1 || M < 1 || (in_type != KGPU_REAL && in_type != KGPU_COMPLEX)) {
    fail("kgpu_master_create: bad arguments L=%d M=%d type=%d", L, M, in_type);
    return nullptr;
  }
  int const N = L + M - 1;
  if (in_type == KGPU_REAL && ((N & 1) || (L & 1))) {
    fail("kgpu_master_create: REAL input needs even L and even N=L+M-1 (got L=%d N=%d)", L, N);
    return nullptr;
  }
  kgpu_master *m = new kgpu_master;
  m->L = L;
  m->M = M;
  m->N = N;
  m->in_type = in_type;
  m->bins = (in_type == KGPU_COMPLEX) ? N : N / 2 + 1;
  m->nc = (in_type == KGPU_COMPLEX) ? N : N / 2;
  if (!choose_split(m->nc, &m->sp)) {
    fail("kgpu_master_create: %ld points cannot be split into two plannable lengths (factors 2,3,5,7; <= %d)",
         m->nc, kMaxTileLen);
    delete m;
    return nullptr;
  }
  m->plan1 = get_tile_plan(m->sp.n1);
  m->plan2 = get_tile_plan(m->sp.n2);
  if (m->plan1 < 0 || m->plan2 < 0) {
    fail("kgpu_master_create: plan registry full or length unsupported");
    delete m;
    return nullptr;
  }
  m->pitch1 = column_pitch(m->sp.n1);
  m->pitch2 = column_pitch(m->sp.n2);
  int const nit = (m->sp.n1 + 31) / 32;
  m->smem1 = sizeof(float2) * ((size_t)kTile * m->pitch1 + (size_t)kTile * nit);
  m->smem2 = sizeof(float2) * ((size_t)kTile * m->pitch2);
  m->spec_stride = ((long)m->bins + 3) / 4 * 4;

  // pass-2 work items
  std::vector<RowItem> items;
  int const n1 = m->sp.n1;
  if (in_type == KGPU_REAL) {
    items.push_back({kRowSelf0, 0, 0, 0});
    for (int k1 = 1; 2 * k1 < n1; k1++) items.push_back({kRowPair, k1, n1 - k1, 0});
    if (n1 % 2 == 0 && n1 > 1) items.push_back({kRowSelfMid, n1 / 2, n1 / 2, 0});
    int const ipc = kTile / 2;
    while (items.size() % ipc) items.push_back({kRowEmpty, 0, 0, 0});
    m->n_item_ctas = (int)items.size() / ipc;
  } else {
    for (int k1 = 0; k1 < n1; k1++) items.push_back({kRowPlain, k1, 0, 0});
    while (items.size() % kTile) items.push_back({kRowEmpty, 0, 0, 0});
    m->n_item_ctas = (int)items.size() / kTile;
  }
  CUDA_OKP(cudaMalloc(&m->d_items, sizeof(RowItem) * items.size()));
  CUDA_OKP(cudaMemcpy(m->d_items, items.data(), sizeof(RowItem) * items.size(), cudaMemcpyHostToDevice));
  if (in_type == KGPU_REAL) {
    std::vector<float2> rootD((size_t)m->sp.n2);
    for (int k2 = 0; k2 < m->sp.n2; k2++) {
      long double const ang = -M_PIl * (long double)k2 / (long double)m->sp.n2;
      rootD[(size_t)k2] = make_float2((float)cosl(ang), (float)sinl(ang));
    }
    CUDA_OKP(cudaMalloc(&m->d_rootD, sizeof(float2) * rootD.size()));
    CUDA_OKP(cudaMemcpy(m->d_rootD, rootD.data(), sizeof(float2) * rootD.size(), cudaMemcpyHostToDevice));
  }
  // specialised kernels for the lengths the configured workloads use
  {
    TilePlan const *p1 = host_tile_plan(m->plan1), *p2 = host_tile_plan(m->plan2);
    if (plan_is<S1296>(p1)) m->static_cols = 1296;
    if (plan_is<S1250>(p2)) m->static_rows = 1250;
    int const n2 = m->sp.n2;
    std::vector<float2> tC((size_t)n1 / 2 + 1);
    auto root = [](long e, long n) {
      long double const ang = -2.0L * M_PIl * (long double)(e % n) / (long double)n;
      return make_float2((float)cosl(ang), (float)sinl(ang));
    };
    for (int k1 = 0; k1 <= n1 / 2; k1++) tC[(size_t)k1] = root(k1, 2 * m->nc);
    if (m->static_cols == 1296) {  // inter-pass factors in the v2 kernel's (u, t2) split
      std::vector<float2> tU((size_t)(n2 + 8) * 144, make_float2(0.f, 0.f)), tT((size_t)(n2 + 16) * 9 + 32, make_float2(0.f, 0.f));
      for (long c = 0; c < n2; c++) {
        for (int u = 0; u < 144; u++) tU[(size_t)c * 144 + u] = root(c * (u / 12 + 12 * (u % 12)), m->nc);
        for (int t = 0; t < 9; t++) tT[(size_t)c * 9 + t] = root(c * 144 * t, m->nc);
      }
      CUDA_OKP(cudaMalloc(&m->d_twU, sizeof(float2) * tU.size()));
      CUDA_OKP(cudaMalloc(&m->d_twT, sizeof(float2) * tT.size()));
      CUDA_OKP(cudaMemcpy(m->d_twU, tU.data(), sizeof(float2) * tU.size(), cudaMemcpyHostToDevice));
      CUDA_OKP(cudaMemcpy(m->d_twT, tT.data(), sizeof(float2) * tT.size(), cudaMemcpyHostToDevice));
      // 36 x 36 variant: stage-0 powers, inter-pass factors A[n2][t] and the ten powers of W_nc^{36 n2}
      static int const kPow[10] = {1, 2, 3, 4, 5, 6, 12, 18, 24, 30};
      std::vector<float2> t0(360), tA36((size_t)n2 * 36), tB10((size_t)(n2 + 8) * 10, make_float2(0.f, 0.f));
      for (int e = 0; e < 10; e++)
        for (int j = 0; j < 36; j++) t0[(size_t)e * 36 + j] = root((long)j * kPow[e], 1296);
      for (long c = 0; c < n2; c++) {
        for (int t = 0; t < 36; t++) tA36[(size_t)c * 36 + t] = root(c * t, m->nc);
        for (int e = 0; e < 10; e++) tB10[(size_t)c * 10 + e] = root(c * 36 * kPow[e], m->nc);
      }
      CUDA_OKP(cudaMalloc(&m->d_r36_tw0, sizeof(float2) * t0.size()));
      CUDA_OKP(cudaMalloc(&m->d_r36_A, sizeof(float2) * tA36.size()));
      CUDA_OKP(cudaMalloc(&m->d_r36_B, sizeof(float2) * tB10.size()));
      CUDA_OKP(cudaMemcpy(m->d_r36_tw0, t0.data(), sizeof(float2) * t0.size(), cudaMemcpyHostToDevice));
      CUDA_OKP(cudaMemcpy(m->d_r36_A, tA36.data(), sizeof(float2) * tA36.size(), cudaMemcpyHostToDevice));
      CUDA_OKP(cudaMemcpy(m->d_r36_B, tB10.data(), sizeof(float2) * tB10.size(), cudaMemcpyHostToDevice));
    }
    if (in_type == KGPU_COMPLEX && n1 == 800 && n2 == 625) {  // cfg-4: (25 x 32) x (25 x 25), fwd_2s.cuh
      using CS = Cols2sShape<25, 32>;
      using RS = Rows2sShape<25, 25>;
      constexpr int RA = 25, RB = 32, RC = 25, RD = 25;
      std::vector<float2> t0((size_t)CS::TW0, make_float2(0.f, 0.f)), tA((size_t)n2 * RA),
          tB((size_t)(n2 + 8) * CS::NP1, make_float2(0.f, 0.f)), r0((size_t)RS::TW0, make_float2(0.f, 0.f));
      for (int e = 0; e < CS::NP0; e++)
        for (int j = 0; j < RB; j++) t0[(size_t)e * RB + j] = root((long)j * Pow<RA>::exponent(e), n1);
      for (long c = 0; c < n2; c++) {
        for (int t = 0; t < RA; t++) tA[(size_t)c * RA + t] = root(c * t, m->nc);
        for (int e = 0; e < CS::NP1; e++) tB[(size_t)c * CS::NP1 + e] = root(c * RA * Pow<RB>::exponent(e), m->nc);
      }
      for (int e = 0; e < RS::NP0; e++)
        for (int j = 0; j < RD; j++) r0[(size_t)e * RD + j] = root((long)j * Pow<RC>::exponent(e), n2);
      auto up = [](float2 **d, std::vector<float2> const &v) {
        if (cudaMalloc(d, sizeof(float2) * v.size()) != cudaSuccess) return 1;
        return cudaMemcpy(*d, v.data(), sizeof(float2) * v.size(), cudaMemcpyHostToDevice) != cudaSuccess ? 1 : 0;
      };
      if (up(&m->d_2s_tw0, t0) || up(&m->d_2s_A, tA) || up(&m->d_2s_B, tB) || up(&m->d_2s_rtw0, r0) ||
          set_smem((const void *)fwd_cols_2s<0, 25, 32>, CS::smem) || set_smem((const void *)fwd_cols_2s<1, 25, 32>, CS::smem) ||
          set_smem((const void *)fwd_cols_2s<2, 25, 32>, CS::smem) || set_smem((const void *)fwd_rows_2s<25, 25>, RS::smem)) {
        fail("kgpu_master_create: tables of the 800 x 625 kernels: %s", cudaGetErrorString(cudaGetLastError()));
        kgpu_master_destroy(m);
        return nullptr;
      }
      m->static_2s = 1;
    }
    if (in_type == KGPU_REAL && m->static_rows == 1250) {  // fwd_rows_r50.cuh
      using RS = RowsR50Shape;
      std::vector<float2> r0((size_t)RS::TW0, make_float2(0.f, 0.f));
      for (int e = 0; e < RS::NP0; e++)
        for (int j = 0; j < RS::RD; j++) r0[(size_t)e * RS::RD + j] = root((long)j * Pow<RS::RC>::exponent(e), 1250);
      CUDA_OKP(cudaMalloc(&m->d_r50_tw0, sizeof(float2) * r0.size()));
      CUDA_OKP(cudaMemcpy(m->d_r50_tw0, r0.data(), sizeof(float2) * r0.size(), cudaMemcpyHostToDevice));
      if (set_smem((const void *)fwd_rows_r50<1296, true>, RS::smem) || set_smem((const void *)fwd_rows_r50<0, false>, RS::smem)) {
        kgpu_master_destroy(m);
        return nullptr;
      }
    }
    CUDA_OKP(cudaMalloc(&m->d_rootC, sizeof(float2) * tC.size()));
    CUDA_OKP(cudaMemcpy(m->d_rootC, tC.data(), sizeof(float2) * tC.size(), cudaMemcpyHostToDevice));
    size_t const sv1 = sizeof(float2) * (8 * 1298 + 1288 + 80), sv2 = sizeof(float2) * (8 * 1250 + 1246);
    if (set_smem((const void *)fwd_cols_v2<0>, sv1) || set_smem((const void *)fwd_cols_v2<1>, sv1) ||
        set_smem((const void *)fwd_cols_v2<2>, sv1) || set_smem((const void *)fwd_rows_v2<true>, sv2) ||
        set_smem((const void *)fwd_rows_v2<false>, sv2) ||
        set_smem((const void *)fwd_cols_v2<0, 1250>, sv1) || set_smem((const void *)fwd_cols_v2<1, 1250>, sv1) ||
        set_smem((const void *)fwd_cols_v2<2, 1250>, sv1) || set_smem((const void *)fwd_rows_v2<true, 1296, true>, sv2) ||
        set_smem((const void *)fwd_cols_r36<0, 1250>, sizeof(float2) * (8 * 1378 + 440)) ||
        set_smem((const void *)fwd_cols_r36<1, 1250>, sizeof(float2) * (8 * 1378 + 440)) ||
        set_smem((const void *)fwd_cols_r36<2, 1250>, sizeof(float2) * (8 * 1378 + 440)) ||
        set_smem((const void *)fwd_cols_r36<0, 0>, sizeof(float2) * (8 * 1378 + 440)) ||
        set_smem((const void *)fwd_cols_r36<1, 0>, sizeof(float2) * (8 * 1378 + 440)) ||
        set_smem((const void *)fwd_cols_r36<2, 0>, sizeof(float2) * (8 * 1378 + 440)) ||
        set_smem((const void *)fwd_rows_v2<false, 1296, false>, sv2)) {
      kgpu_master_destroy(m);
      return nullptr;
    }
  }
  if (set_smem((const void *)fwd_cols_kernel<0>, m->smem1) || set_smem((const void *)fwd_cols_kernel<1>, m->smem1) ||
      set_smem((const void *)fwd_rows_kernel, m->smem2)) {
    kgpu_master_destroy(m);
    return nullptr;
  }
  return m;
}

extern "C" void kgpu_master_destroy(kgpu_master *m) {
  if (!m) return;
  cudaFree(m->d_items);
  cudaFree(m->d_rootD);
  cudaFree(m->d_rootC);
  cudaFree(m->d_twU);
  cudaFree(m->d_r36_tw0);
  cudaFree(m->d_r36_A);
  cudaFree(m->d_r36_B);
  cudaFree(m->d_2s_tw0);
  cudaFree(m->d_2s_A);
  cudaFree(m->d_2s_B);
  cudaFree(m->d_2s_rtw0);
  cudaFree(m->d_r50_tw0);
  cudaFree(m->d_twT);
  cudaFree(m->d_mid);
  cudaFree(m->d_notch);
  delete m;
}
extern "C" int kgpu_master_points(kgpu_master const *m) { return m ? m->N : -1; }
extern "C" int kgpu_master_bins(kgpu_master const *m) { return m ? m->bins : -1; }
extern "C" long kgpu_master_spec_stride(kgpu_master const *m) { return m ? m->spec_stride : -1; }
extern "C" int kgpu_master_describe(kgpu_master const *m, char *buf, int buflen) {
  if (!m || !buf) return -1;
  std::string s;
  char tmp[128];
  snprintf(tmp, sizeof tmp, "N=%d %s, %ld-point complex two-pass %d x %d; cols radices [", m->N,
           m->in_type == KGPU_REAL ? "real" : "complex", m->nc, m->sp.n1, m->sp.n2);
  s += tmp;
  TilePlan const *p1 = host_tile_plan(m->plan1), *p2 = host_tile_plan(m->plan2);
  if (m->static_2s) s += "25,32";
  else if (m->static_cols == 1296) s += "36,36";  // fwd_cols_r36 (the tile plan is what the generic kernels would run)
  else
    for (int i = 0; i < p1->nstages; i++) s += std::to_string(p1->radix[i]) + (i + 1 < p1->nstages ? "," : "");
  s += "] rows radices [";
  if (m->in_type == KGPU_REAL && m->static_rows == 1250) s += "50,25";
  else
  for (int i = 0; i < p2->nstages; i++) s += std::to_string(p2->radix[i]) + (i + 1 < p2->nstages ? "," : "");
  snprintf(tmp, sizeof tmp, "]; smem %zu/%zu B; grids %d/%d CTAs per block",
           m->static_2s ? Cols2sShape<25, 32>::smem : m->static_cols == 1296 ? sizeof(float2) * (8 * 1378 + 440) : m->smem1,
           m->static_2s ? Rows2sShape<25, 25>::smem : (m->in_type == KGPU_REAL && m->static_rows == 1250) ? RowsR50Shape::smem : m->smem2,
           (m->sp.n2 + kTile - 1) / kTile, m->n_item_ctas);
  s += tmp;
  snprintf(buf, (size_t)buflen, "%s", s.c_str());
  return 0;
}

// One launch pair (column pass, row pass) over `nblocks` consecutive blocks on stream `st`, inter-pass data in `mid`.
static int forward_span(kgpu_master *m, const void *d_in, int fmt, float scale, int derandomize, int nblocks, void *d_spec,
                        void *d_stats, cudaStream_t st, float2 *mid) {
  Pass1Args a1;
  a1.in = d_in;
  a1.hop = (m->in_type == KGPU_REAL) ? m->L / 2 : m->L;
  a1.n1 = m->sp.n1;
  a1.n2 = m->sp.n2;
  a1.nc = m->nc;
  a1.plan = m->plan1;
  a1.pitch = m->pitch1;
  a1.scale = scale;
  a1.derandomize = derandomize;
  a1.first_new = (m->in_type == KGPU_REAL) ? (m->M - 1) / 2 : (m->M - 1);
  a1.mid = mid;
  a1.stats = (fmt == KGPU_FMT_I16) ? (IngestStats *)d_stats : nullptr;
  a1.dbg = (unsigned long long *)g_dbg_buf;
  a1.mid_ld = m->sp.n2;
  dim3 const g1((unsigned)((m->sp.n2 + kTile - 1) / kTile), (unsigned)nblocks);
  FwdTables tb;
  tb.rootC = m->d_rootC;
  bool const use_static = g_static_on.load() != 0;
  bool halved = false;
  {
    ProfScope ps(K_FWD_COLS, st);
    if (use_static && m->static_2s) {
      int const f = (fmt != KGPU_FMT_I16) ? 0 : ((derandomize || a1.stats) ? 2 : 1);
      using CS = Cols2sShape<25, 32>;
      Cols2sTables t4;
      t4.tw0 = m->d_2s_tw0;
      t4.twA = m->d_2s_A;
      t4.twB = m->d_2s_B;
      a1.out_scale = (fmt == KGPU_FMT_I16) ? scale : 1.0f;
      a1.mid_ld = (m->sp.n2 + 15) / 16 * 16;
      if (f == 0) fwd_cols_2s<0, 25, 32><<<g1, CS::T, CS::smem, st>>>(a1, t4);
      else if (f == 1) fwd_cols_2s<1, 25, 32><<<g1, CS::T, CS::smem, st>>>(a1, t4);
      else fwd_cols_2s<2, 25, 32><<<g1, CS::T, CS::smem, st>>>(a1, t4);
    } else if (use_static && m->static_cols == 1296) {
      int const f = (fmt != KGPU_FMT_I16) ? 0 : ((derandomize || a1.stats) ? 2 : 1);
      size_t const sv1 = sizeof(float2) * (8 * 1298 + 1288 + 80);
      ColsV2Tables t2;
      t2.twU = m->d_twU;
      t2.twT = m->d_twT;
      // the int16 scale (and the 1/2 of the real split when the row pass is the v2 kernel too) is
      // folded into the inter-pass twiddle
      halved = (m->in_type == KGPU_REAL) && m->static_rows == 1250;
      a1.out_scale = (fmt == KGPU_FMT_I16 ? scale : 1.0f) * (halved ? 0.5f : 1.0f);
      if (g_tuning[13].load() == 0) {  // default: two fat stages (36 x 36), one trip through shared memory
        if (m->sp.n2 == 1250 && m->static_rows == 1250) a1.mid_ld = (m->sp.n2 + 15) / 16 * 16;  // rows padded to 128 B (both kernels know)
        size_t const sr = sizeof(float2) * (8 * 1378 + 440);
        ColsR36Tables t3;
        t3.tw0 = m->d_r36_tw0;
        t3.twA = m->d_r36_A;
        t3.twB = m->d_r36_B;
        if (m->sp.n2 == 1250 && m->static_rows == 1250) {
          if (f == 0) fwd_cols_r36<0, 1250><<<g1, 288, sr, st>>>(a1, t3);
          else if (f == 1) fwd_cols_r36<1, 1250><<<g1, 288, sr, st>>>(a1, t3);
          else fwd_cols_r36<2, 1250><<<g1, 288, sr, st>>>(a1, t3);
        } else {
          if (f == 0) fwd_cols_r36<0, 0><<<g1, 288, sr, st>>>(a1, t3);
          else if (f == 1) fwd_cols_r36<1, 0><<<g1, 288, sr, st>>>(a1, t3);
          else fwd_cols_r36<2, 0><<<g1, 288, sr, st>>>(a1, t3);
        }
      } else if (m->sp.n2 == 1250) {
        if (f == 0) fwd_cols_v2<0, 1250><<<g1, 288, sv1, st>>>(a1, t2);
        else if (f == 1) fwd_cols_v2<1, 1250><<<g1, 288, sv1, st>>>(a1, t2);
        else fwd_cols_v2<2, 1250><<<g1, 288, sv1, st>>>(a1, t2);
      } else {
        if (f == 0) fwd_cols_v2<0><<<g1, 288, sv1, st>>>(a1, t2);
        else if (f == 1) fwd_cols_v2<1><<<g1, 288, sv1, st>>>(a1, t2);
        else fwd_cols_v2<2><<<g1, 288, sv1, st>>>(a1, t2);
      }
    } else if (fmt == KGPU_FMT_I16)
      fwd_cols_kernel<1><<<g1, kFwdThreads, m->smem1, st>>>(a1);
    else
      fwd_cols_kernel<0><<<g1, kFwdThreads, m->smem1, st>>>(a1);
  }
  g_launches++;
  Pass2Args a2;
  a2.mid = mid;
  a2.n1 = m->sp.n1;
  a2.n2 = m->sp.n2;
  a2.nc = m->nc;
  a2.plan = m->plan2;
  a2.pitch = m->pitch2;
  a2.real_split = (m->in_type == KGPU_REAL);
  a2.items = m->d_items;
  a2.rootD = m->d_rootD;
  a2.spec = (float2 *)d_spec;
  a2.spec_stride = m->spec_stride;
  a2.dbg = g_dbg_buf2 ? (unsigned long long *)g_dbg_buf2 : nullptr;
  a2.mid_ld = a1.mid_ld;
  // The row pass reads what the column pass has just written: taking the blocks last-to-first finds the most recent ones
  // still in L2.  Key 15 = n makes every CTA pull the rows of the CTA n later in launch order into L2 while it works; on
  // H100 that prefetch costs row-pass time at every distance tried (tools/kbench.py), so it is off by default.
  a2.rev = g_tuning[14].load() != 1;                   // 14=1: first-to-last (A/B)
  a2.pf_ctas = std::max(0, g_tuning[15].load());       // 15=n: prefetch n CTAs ahead (A/B)
  dim3 const g2((unsigned)m->n_item_ctas, (unsigned)nblocks);
  {
    ProfScope ps(K_FWD_ROWS, st);
    if (use_static && m->static_2s) {
      using RS = Rows2sShape<25, 25>;
      dim3 const g2s((unsigned)((m->sp.n1 + 7) / 8), (unsigned)nblocks);
      fwd_rows_2s<25, 25><<<g2s, RS::T, RS::smem, st>>>(a2, m->d_2s_rtw0);
    } else if (use_static && m->static_rows == 1250) {
      size_t const sv2 = sizeof(float2) * (8 * 1250 + 1246);
      if (a2.real_split && g_tuning[10].load() == 5) {  // 10=5: two fat stages (50 x 25) (A/B); default: the 10 x 25 x 5 kernel
        using RS = RowsR50Shape;
        if (halved) fwd_rows_r50<1296, true><<<g2, RS::T, RS::smem, st>>>(a2, tb, m->d_r50_tw0);  // halved <=> 36 x 36 columns in front
        else fwd_rows_r50<0, false><<<g2, RS::T, RS::smem, st>>>(a2, tb, m->d_r50_tw0);
      } else if (a2.real_split && halved) fwd_rows_v2<true, 1296, true><<<g2, 256, sv2, st>>>(a2, tb);
      else if (a2.real_split) fwd_rows_v2<true><<<g2, 256, sv2, st>>>(a2, tb);
      else if (m->sp.n1 == 1296) fwd_rows_v2<false, 1296, false><<<g2, 256, sv2, st>>>(a2, tb);
      else fwd_rows_v2<false><<<g2, 256, sv2, st>>>(a2, tb);
    } else
      fwd_rows_kernel<<<g2, kFwdThreads, m->smem2, st>>>(a2);
  }
  g_launches++;
  CUDA_OK(cudaGetLastError());
  return 0;
}

extern "C" int kgpu_forward(kgpu_master *m, const void *d_in, int fmt, float scale, int derandomize, int nblocks,
                            void *d_spec, void *d_stats, void *stream) {
  if (!m || !d_in || !d_spec || nblocks < 1) return fail("kgpu_forward: bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  if (m->mid_blocks < nblocks) {
    CUDA_OK(cudaStreamSynchronize(st));
    cudaFree(m->d_mid);
    m->d_mid = nullptr;
    m->mid_blocks = 0;
    CUDA_OK(cudaMalloc(&m->d_mid, sizeof(float2) * (size_t)m->sp.n1 * (size_t)((m->sp.n2 + 15) / 16 * 16) * (size_t)nblocks));
    m->mid_blocks = nblocks;
  }
  if (fmt == KGPU_FMT_I16 && d_stats) CUDA_OK(cudaMemsetAsync(d_stats, 0, sizeof(IngestStats) * (size_t)nblocks, st));
  return forward_span(m, d_in, fmt, scale, derandomize, nblocks, d_spec, d_stats, st, m->d_mid);
}

extern "C" int kgpu_master_set_notches(kgpu_master *m, int const *bins, double const *alpha, int n) {
  if (!m || n < 0) return fail("kgpu_master_set_notches: bad arguments");
  cudaFree(m->d_notch);
  m->d_notch = nullptr;
  m->n_notch = 0;
  if (n == 0) return 0;
  std::vector<NotchDev> v((size_t)n);
  m->notch_sequential = 0;
  for (int i = 0; i < n; i++) {
    if (bins[i] < 0 || bins[i] >= m->bins) return fail("kgpu_master_set_notches: bin %d out of range", bins[i]);
    v[(size_t)i] = {bins[i], 0, 0.0, 0.0, alpha[i]};
    for (int j = 0; j < i; j++)
      if (bins[j] == bins[i]) m->notch_sequential = 1;
  }
  CUDA_OK(cudaMalloc(&m->d_notch, sizeof(NotchDev) * (size_t)n));
  CUDA_OK(cudaMemcpy(m->d_notch, v.data(), sizeof(NotchDev) * (size_t)n, cudaMemcpyHostToDevice));
  m->n_notch = n;
  return 0;
}
extern "C" int kgpu_apply_notches(kgpu_master *m, void *d_spec, int nblocks, void *stream) {
  if (!m || !d_spec) return fail("kgpu_apply_notches: bad arguments");
  if (m->n_notch == 0) return 0;
  {
    ProfScope ps(K_NOTCH, (cudaStream_t)stream);
    notch_kernel<<<1, 32 * ((m->n_notch + 31) / 32), 0, (cudaStream_t)stream>>>(
        m->d_notch, m->n_notch, m->notch_sequential, (float2 *)d_spec, m->spec_stride, nblocks);
  }
  g_launches++;
  CUDA_OK(cudaGetLastError());
  return 0;
}

// ------------------------------------------------------------------ response design ----------
// set_filter's host half (filter.c:968-1029, window.c:217-254, misc.c:416-427, misc.h:217-221,
// sincospi.c:24-66): Kaiser-windowed sinc, complex-shifted to the passband centre, normalised for
// window loss, the master's unnormalised forward transform and the half-power of a real input.
namespace {
double bessel_i0(double z) {
  double const q = z * z / 4;
  double sum = 1 + q, term = q;
  for (int k = 2; k < 40; k++) {
    term *= q / ((double)k * (double)k);
    sum += term;
    if (term < 1e-12 * sum) break;
  }
  return sum;
}
void cis_revolutions(double x, double *re, double *im) {  // exp(i*pi*x), exact reduction
  double y = fmod(x, 2.0);
  if (y < 0) y += 2.0;
  int const quad = (int)floor(2.0 * y) & 3;
  double z = y - 0.5 * quad;
  bool const fold = z > 0.25;
  if (fold) z = 0.5 - z;
  double s = sin(M_PI * z), c = cos(M_PI * z);
  if (fold) std::swap(s, c);
  switch (quad) {
    case 0: *re = c; *im = s; break;
    case 1: *re = -s; *im = c; break;
    case 2: *re = -c; *im = -s; break;
    default: *re = s; *im = -c; break;
  }
}
// taps[0..points) complex float (interleaved), first M = points-olen+1 non-zero
int design_taps(int points, int olen, int master_points, bool master_real, double low, double high, double beta,
                std::vector<float2> &taps) {
  if (isnan(low) || isnan(high) || isnan(beta)) return -1;
  if (low > high) std::swap(low, high);
  low = std::min(std::max(low, -0.5), 0.5);
  high = std::min(std::max(high, -0.5), 0.5);
  int const M = points - olen + 1;
  if (M < 2) return -1;
  double const half_bw = (high == low) ? 1e-4 : fabs(high - low) / 2;
  double const centre = (high + low) / 2;
  std::vector<float> win((size_t)M);
  double const norm0 = 1.0 / bessel_i0(beta), step = 2.0 / (M - 1);
  for (int n = 0; n < M / 2; n++) {
    double const p = step * n - 1;
    win[(size_t)n] = win[(size_t)(M - 1 - n)] = (float)(bessel_i0(beta * sqrt(1 - p * p)) * norm0);
  }
  if (M & 1) win[(size_t)((M - 1) / 2)] = 1.0f;
  double wsum = 0;
  for (float w : win) wsum += w;
  if (wsum == 0 || !std::isfinite(wsum)) return -1;
  float const wgain = (float)(M / wsum);
  for (float &w : win) w *= wgain;
  taps.assign((size_t)points, make_float2(0.f, 0.f));
  std::vector<double> rr((size_t)M), cr((size_t)M), ci((size_t)M);
  double tap_sum = 0;
  for (int i = 0; i < M; i++) {
    double const n = i - (double)(M - 1) / 2;
    double const arg = 2 * half_bw * n;
    double const snc = (arg == 0) ? 1.0 : sin(M_PI * arg) / (M_PI * arg);
    rr[(size_t)i] = win[(size_t)i] * 2 * half_bw * snc;
    tap_sum += rr[(size_t)i];
    cis_revolutions(2 * centre * n, &cr[(size_t)i], &ci[(size_t)i]);
  }
  double const gain = (master_real ? M_SQRT2 : 1.0) / (tap_sum * master_points);
  for (int i = 0; i < M; i++) {
    // the reference rounds the un-normalised tap to float first, then scales (filter.c:1015,1028)
    float const tr = (float)(cr[(size_t)i] * rr[(size_t)i]), ti = (float)(ci[(size_t)i] * rr[(size_t)i]);
    taps[(size_t)i] = make_float2((float)((double)tr * gain), (float)((double)ti * gain));
  }
  return 0;
}
}  // namespace

// ------------------------------------------------------------------ bank --------------------
struct ChanHost {
  bool defined = false, enabled = false, has_response = false;
  bool real_out = false;  // REAL-output slave (filter.c:370-390): olen floats per block
  int olen = 0, points = 0, plan = -1, shift = 0, flags = 0;
  long resp_off = 0, resp_cap = 0;  // region of the response arena owned by this slot
  ChanAux aux{};          // oscillator / beam parameters (zero = unused)
};
struct kgpu_bank {
  kgpu_master *m;
  int capacity;
  std::vector<ChanHost> ch;
  int nchan = 0;  // highest defined + 1
  float2 *d_resp = nullptr;
  long resp_cap = 0, resp_used = 0;
  ChanDesc *d_desc = nullptr;
  std::vector<ChanDesc> desc;
  std::vector<long> out_off;
  long out_stride = 0;
  bool dirty = true;
  int max_points = 0;
  struct Group {
    int plan, points, off, count;
    bool generic;  // REAL-output / beam channels: served by the runtime-plan kernel only
  };
  std::vector<Group> groups;  // enabled channels grouped by inverse-transform plan
  int *d_order = nullptr;
  ChanAux *d_aux = nullptr;   // [capacity]
  int *d_shift = nullptr;     // [capacity] shifts, for the noise estimator
  float2 *d_fm_mem[2] = {nullptr, nullptr};  // [capacity] discriminator phase memory, ping-pong per launch
  int fm_parity = 0;
  std::vector<ChanAux> aux;
  long block_counter = 0;     // index of the next block a run will process (oscillator epoch arithmetic)
  long last_rebase = 0;
  bool any_osc = false;
};

static void resolve_walk(kgpu_master const *m, ChanHost const &c, ChanDesc &d) {
  int const ns = c.points, mb = m->bins, half = ns / 2;
  long const shift = c.shift;
  d.zlead = 0;
  d.ncopy = 0;
  d.q0 = 0;
  d.dir = 1;
  if (c.real_out) {  // filter.c:794-809: the kernel indexes the master by si + shift itself
    d.q0 = (int)shift;
    d.ncopy = 1;
    return;
  }
  if (m->in_type == KGPU_REAL) {
    if (shift >= 0) {  // filter.c:819-855
      long const start = shift - half;
      long const z = std::min<long>(std::max<long>(0, -start), ns);
      long const q0 = start + z;
      long const nc = std::max<long>(0, std::min<long>(ns - z, (long)mb - q0));
      d.zlead = (int)z;
      d.q0 = (int)std::max<long>(0, std::min<long>(q0, mb - 1));
      d.ncopy = (int)nc;
    } else {  // filter.c:856-892
      long const start = -(shift - half);
      long const z = std::min<long>(std::max<long>(0, start - (mb - 1)), ns);
      long const q0 = start - z;
      long const nc = std::max<long>(0, std::min<long>(ns - z, q0 + 1));
      d.zlead = (int)z;
      d.q0 = (int)std::max<long>(0, std::min<long>(q0, mb - 1));
      d.ncopy = (int)nc;
      d.dir = -1;
    }
  } else {  // filter.c:728-793, the walk in closed form
    long const nyq = (mb + 1) / 2;
    long rp = shift - half;
    long const z = std::min<long>(std::max<long>(0, -nyq - rp), ns);
    d.zlead = (int)z;
    if (z < ns) {
      rp += z;
      if (rp < 0) rp += mb;
      if (rp >= 0 && rp < mb) {
        long dist = ((nyq - rp - 1) % mb + mb) % mb + 1;
        d.q0 = (int)rp;
        d.ncopy = (int)std::min<long>(ns - z, dist);
      }
    }
  }
}

static int bank_commit(kgpu_bank *b, cudaStream_t st) {
  if (!b->dirty) return 0;
  b->desc.assign((size_t)std::max(b->nchan, 1), ChanDesc{});
  b->out_off.assign((size_t)std::max(b->nchan, 1), 0);
  long off = 0;
  b->max_points = 1;
  for (int i = 0; i < b->nchan; i++) {
    ChanHost const &c = b->ch[(size_t)i];
    ChanDesc &d = b->desc[(size_t)i];
    memset(&d, 0, sizeof d);
    d.plan = -1;
    b->out_off[(size_t)i] = off;
    if (!c.defined) continue;
    d.points = c.points;
    d.olen = c.olen;
    d.flags = (c.flags & (kChanIsb | kChanBeam | kChanOsc)) | (c.real_out ? kChanRealOut : 0);
    if (c.real_out) d.flags &= ~(kChanIsb | kChanBeam | kChanOsc);  // the reference applies none of them to REAL slaves
    if (b->m->in_type != KGPU_COMPLEX) d.flags &= ~kChanBeam;       // beam exists for COMPLEX masters only (filter.c:756)
    d.resp_off = c.resp_off;
    d.out_off = off;
    off += c.real_out ? (c.olen + 1) / 2 : c.olen;
    if (c.enabled && c.has_response) {
      d.plan = c.plan;
      resolve_walk(b->m, c, d);
      b->max_points = std::max(b->max_points, c.points);
    }
  }
  b->out_stride = (off + 3) / 4 * 4;
  // one launch per distinct plan: order[] lists that plan's descriptors
  std::vector<int> order;
  b->groups.clear();
  auto generic_only = [&](int i) { return (b->desc[(size_t)i].flags & (kChanRealOut | kChanBeam)) != 0; };
  for (int i = 0; i < b->nchan; i++) {
    if (b->desc[(size_t)i].plan < 0) continue;
    bool const gen = generic_only(i);
    bool found = false;
    for (auto &g : b->groups)
      if (g.plan == b->desc[(size_t)i].plan && g.generic == gen) found = true;
    if (found) continue;
    kgpu_bank::Group g{b->desc[(size_t)i].plan, b->desc[(size_t)i].points, (int)order.size(), 0, gen};
    for (int k = i; k < b->nchan; k++)
      if (b->desc[(size_t)k].plan == g.plan && generic_only(k) == gen) order.push_back(k);
    g.count = (int)order.size() - g.off;
    b->groups.push_back(g);
  }
  // oscillator epochs move up to the current block so the device-side phase arithmetic stays small
  b->any_osc = false;
  b->aux.assign((size_t)std::max(b->nchan, 1), ChanAux{});
  for (int i = 0; i < b->nchan; i++) {
    ChanHost &c = b->ch[(size_t)i];
    if (c.defined && (c.flags & kChanOsc) && !c.real_out) {
      b->any_osc = true;
      long const K = b->block_counter - c.aux.osc_epoch;
      if (K > 0) {
        double const D = (double)K * (double)c.olen;
        double ph = c.aux.osc_phase + (double)K * c.aux.osc_adj + D * c.aux.osc_freq + 0.5 * D * (D + 1.0) * c.aux.osc_rate;
        c.aux.osc_phase = ph - floor(ph);
        c.aux.osc_freq += c.aux.osc_rate * D;
        c.aux.osc_epoch = b->block_counter;
      }
    }
    b->aux[(size_t)i] = c.aux;
  }
  b->last_rebase = b->block_counter;
  CUDA_OK(cudaStreamSynchronize(st));
  CUDA_OK(cudaMemcpy(b->d_aux, b->aux.data(), sizeof(ChanAux) * b->aux.size(), cudaMemcpyHostToDevice));
  {
    std::vector<int> sh((size_t)std::max(b->nchan, 1), 0);
    for (int i = 0; i < b->nchan; i++) sh[(size_t)i] = b->ch[(size_t)i].shift;
    CUDA_OK(cudaMemcpy(b->d_shift, sh.data(), sizeof(int) * sh.size(), cudaMemcpyHostToDevice));
  }
  if (!order.empty())
    CUDA_OK(cudaMemcpy(b->d_order, order.data(), sizeof(int) * order.size(), cudaMemcpyHostToDevice));
  CUDA_OK(cudaMemcpy(b->d_desc, b->desc.data(), sizeof(ChanDesc) * b->desc.size(), cudaMemcpyHostToDevice));
  b->dirty = false;
  return 0;
}

extern "C" kgpu_bank *kgpu_bank_create(kgpu_master *m, int capacity) {
  if (!m || capacity < 1) {
    fail("kgpu_bank_create: bad arguments");
    return nullptr;
  }
  kgpu_bank *b = new kgpu_bank;
  b->m = m;
  b->capacity = capacity;
  b->ch.resize((size_t)capacity);
  CUDA_OKP(cudaMalloc(&b->d_desc, sizeof(ChanDesc) * (size_t)capacity));
  CUDA_OKP(cudaMalloc(&b->d_order, sizeof(int) * (size_t)capacity));
  CUDA_OKP(cudaMalloc(&b->d_aux, sizeof(ChanAux) * (size_t)capacity));
  CUDA_OKP(cudaMalloc(&b->d_shift, sizeof(int) * (size_t)capacity));
  for (int i = 0; i < 2; i++) {
    CUDA_OKP(cudaMalloc(&b->d_fm_mem[i], sizeof(float2) * (size_t)capacity));
    CUDA_OKP(cudaMemset(b->d_fm_mem[i], 0, sizeof(float2) * (size_t)capacity));
  }
  return b;
}
extern "C" void kgpu_bank_destroy(kgpu_bank *b) {
  if (!b) return;
  cudaFree(b->d_resp);
  cudaFree(b->d_desc);
  cudaFree(b->d_order);
  cudaFree(b->d_aux);
  cudaFree(b->d_shift);
  cudaFree(b->d_fm_mem[0]);
  cudaFree(b->d_fm_mem[1]);
  delete b;
}
static bool bad_idx(kgpu_bank const *b, int idx) { return !b || idx < 0 || idx >= b->capacity; }

static int bank_define(kgpu_bank *b, int idx, int olen, bool real_out);
extern "C" int kgpu_bank_define(kgpu_bank *b, int idx, int olen) { return bank_define(b, idx, olen, false); }
extern "C" int kgpu_bank_define_ex(kgpu_bank *b, int idx, int olen, int out_type) {
  if (out_type != KGPU_COMPLEX && out_type != KGPU_REAL) return fail("kgpu_bank_define_ex: out_type must be KGPU_COMPLEX or KGPU_REAL");
  return bank_define(b, idx, olen, out_type == KGPU_REAL);
}
static int bank_define(kgpu_bank *b, int idx, int olen, bool real_out) {
  if (bad_idx(b, idx) || olen < 1) return fail("kgpu_bank_define: bad arguments");
  long const num = (long)olen * b->m->N;
  if (num % b->m->L) return fail("invalid output length %d for N=%d L=%d (filter.c:312-316)", olen, b->m->N, b->m->L);
  int const points = (int)(num / b->m->L);
  if (real_out && (points & 1)) return fail("kgpu_bank_define: REAL-output slaves need an even number of points (got %d)", points);
  int const plan = get_tile_plan(points);
  if (plan < 0) return fail("kgpu_bank_define: %d-point inverse transform cannot be planned", points);
  ChanHost &c = b->ch[(size_t)idx];
  c.real_out = real_out;
  if (!(c.defined && c.points == points)) {
    long const need = (points + 3) / 4 * 4;
    if (need <= c.resp_cap) {
      // the slot's old region is large enough: reuse it (a long-running radiod re-creates channels at other rates)
    } else if (b->resp_used + need > b->resp_cap) {
      long const ncap = std::max<long>(2 * b->resp_cap, b->resp_used + std::max<long>(need, 64L * 1024));
      float2 *nb = nullptr;
      CUDA_OK(cudaMalloc(&nb, sizeof(float2) * (size_t)ncap));
      CUDA_OK(cudaDeviceSynchronize());
      if (b->resp_used)
        CUDA_OK(cudaMemcpy(nb, b->d_resp, sizeof(float2) * (size_t)b->resp_used, cudaMemcpyDeviceToDevice));
      cudaFree(b->d_resp);
      b->d_resp = nb;
      b->resp_cap = ncap;
    }
    if (need > c.resp_cap) {
      c.resp_off = b->resp_used;
      c.resp_cap = need;
      b->resp_used += need;
    }
    c.has_response = false;
  }
  c.defined = true;
  c.enabled = true;
  c.olen = olen;
  c.points = points;
  c.plan = plan;
  b->nchan = std::max(b->nchan, idx + 1);
  b->dirty = true;
  return points;
}

// st == nullptr: legacy entry points, whole-device synchronisation (any stream may be using the response);
// otherwise only `st` is synchronised: the caller guarantees that every launch reading this bank is ordered on it
static int upload_taps_and_transform(kgpu_bank *b, ChanHost &c, float2 const *host, bool transform, cudaStream_t st = nullptr,
                                     bool on_stream = false) {
  float2 *dst = b->d_resp + c.resp_off;
  // the response may be in use by a queued run: wait, then swap (the reference takes
  // response_mutex for the same reason, filter.c:1039-1043)
  if (on_stream) CUDA_OK(cudaStreamSynchronize(st));
  else CUDA_OK(cudaDeviceSynchronize());
  CUDA_OK(cudaMemcpyAsync(dst, host, sizeof(float2) * (size_t)c.points, cudaMemcpyHostToDevice, st));
  if (transform) {
    size_t const sm = sizeof(float2) * (size_t)c.points;
    if (set_smem((const void *)response_fft_kernel, sm)) return -1;
    response_fft_kernel<<<1, 32, sm, st>>>(dst, c.plan);
    g_launches++;
    CUDA_OK(cudaGetLastError());
  }
  if (on_stream) CUDA_OK(cudaStreamSynchronize(st));
  else CUDA_OK(cudaDeviceSynchronize());
  c.has_response = true;
  b->dirty = true;
  return 0;
}

static int bank_set_filter(kgpu_bank *b, int idx, double low, double high, double kaiser_beta, cudaStream_t st, bool on_stream);
extern "C" int kgpu_bank_set_filter(kgpu_bank *b, int idx, double low, double high, double kaiser_beta) {
  return bank_set_filter(b, idx, low, high, kaiser_beta, nullptr, false);
}
extern "C" int kgpu_bank_set_filter_on(kgpu_bank *b, int idx, double low, double high, double kaiser_beta, void *stream) {
  return bank_set_filter(b, idx, low, high, kaiser_beta, (cudaStream_t)stream, true);
}
static int bank_set_filter(kgpu_bank *b, int idx, double low, double high, double kaiser_beta, cudaStream_t st, bool on_stream) {
  if (bad_idx(b, idx) || !b->ch[(size_t)idx].defined) return fail("kgpu_bank_set_filter: channel not defined");
  ChanHost &c = b->ch[(size_t)idx];
  std::vector<float2> taps;
  if (c.real_out) {  // filter edges may not cross DC for a real output (filter.c:971-975)
    low = fabs(low);
    high = fabs(high);
  }
  if (design_taps(c.points, c.olen, b->m->N, b->m->in_type == KGPU_REAL, low, high, kaiser_beta, taps))
    return fail("kgpu_bank_set_filter: rejected (NaN or M < 2), cf. filter.c:969,989");
  return upload_taps_and_transform(b, c, taps.data(), true, st, on_stream);
}
extern "C" int kgpu_bank_set_response(kgpu_bank *b, int idx, float const *response) {
  if (bad_idx(b, idx) || !b->ch[(size_t)idx].defined || !response) return fail("kgpu_bank_set_response: bad arguments");
  return upload_taps_and_transform(b, b->ch[(size_t)idx], (float2 const *)response, false);
}
extern "C" int kgpu_bank_get_response(kgpu_bank *b, int idx, float *response) {
  if (bad_idx(b, idx) || !b->ch[(size_t)idx].has_response || !response) return fail("kgpu_bank_get_response: none");
  ChanHost &c = b->ch[(size_t)idx];
  // written by a synchronised upload (above) and never modified by kernels: a plain blocking copy is ordered correctly
  CUDA_OK(cudaMemcpy(response, b->d_resp + c.resp_off, sizeof(float2) * (size_t)c.points, cudaMemcpyDeviceToHost));
  return c.points;
}
extern "C" int kgpu_bank_set_shift(kgpu_bank *b, int idx, int shift) {
  if (bad_idx(b, idx) || !b->ch[(size_t)idx].defined) return fail("kgpu_bank_set_shift: channel not defined");
  if (b->ch[(size_t)idx].shift != shift) {
    b->ch[(size_t)idx].shift = shift;
    b->dirty = true;
  }
  return 0;
}
extern "C" int kgpu_bank_set_flags(kgpu_bank *b, int idx, int flags) {
  if (bad_idx(b, idx) || !b->ch[(size_t)idx].defined) return fail("kgpu_bank_set_flags: channel not defined");
  int const keep = b->ch[(size_t)idx].flags & kChanOsc;  // the oscillator bit belongs to kgpu_bank_set_osc
  flags = (flags & ~kChanOsc) | keep;
  if (b->ch[(size_t)idx].flags != flags) {
    b->ch[(size_t)idx].flags = flags;
    b->dirty = true;
  }
  return 0;
}
extern "C" int kgpu_bank_set_weights(kgpu_bank *b, int idx, double alpha_re, double alpha_im, double beta_re, double beta_im) {
  if (bad_idx(b, idx) || !b->ch[(size_t)idx].defined) return fail("kgpu_bank_set_weights: channel not defined");
  ChanAux &x = b->ch[(size_t)idx].aux;
  x.are = alpha_re;
  x.aim = alpha_im;
  x.bre = beta_re;
  x.bim = beta_im;
  b->dirty = true;
  return 0;
}
extern "C" int kgpu_bank_set_osc(kgpu_bank *b, int idx, int enable, double phase_cycles, double freq_cps, double rate_cps2,
                                 double block_adj_cycles) {
  if (bad_idx(b, idx) || !b->ch[(size_t)idx].defined) return fail("kgpu_bank_set_osc: channel not defined");
  ChanHost &c = b->ch[(size_t)idx];
  if (!std::isfinite(phase_cycles) || !std::isfinite(freq_cps) || !std::isfinite(rate_cps2) || !std::isfinite(block_adj_cycles))
    return fail("kgpu_bank_set_osc: non-finite parameter");
  c.flags = enable ? (c.flags | kChanOsc) : (c.flags & ~kChanOsc);
  c.aux.osc_phase = phase_cycles - floor(phase_cycles);
  c.aux.osc_freq = freq_cps;
  c.aux.osc_rate = rate_cps2;
  c.aux.osc_adj = block_adj_cycles;
  c.aux.osc_epoch = b->block_counter;
  b->dirty = true;
  return 0;
}
extern "C" int kgpu_bank_get_osc_phase(kgpu_bank *b, int idx, double *phase_cycles) {
  if (bad_idx(b, idx) || !b->ch[(size_t)idx].defined || !phase_cycles) return fail("kgpu_bank_get_osc_phase: bad arguments");
  ChanHost const &c = b->ch[(size_t)idx];
  long const K = b->block_counter - c.aux.osc_epoch;
  double const D = (double)K * (double)c.olen;
  double const ph = c.aux.osc_phase + (double)K * c.aux.osc_adj + D * c.aux.osc_freq + 0.5 * D * (D + 1.0) * c.aux.osc_rate;
  *phase_cycles = ph - floor(ph);
  return 0;
}
extern "C" int kgpu_bank_set_block_counter(kgpu_bank *b, long counter) {
  if (!b) return fail("kgpu_bank_set_block_counter: bad arguments");
  b->block_counter = counter;
  return 0;
}
extern "C" long kgpu_bank_block_counter(kgpu_bank const *b) { return b ? b->block_counter : -1; }
extern "C" int kgpu_bank_enable(kgpu_bank *b, int idx, int enabled) {
  if (bad_idx(b, idx) || !b->ch[(size_t)idx].defined) return fail("kgpu_bank_enable: channel not defined");
  if (b->ch[(size_t)idx].enabled != (enabled != 0)) {
    b->ch[(size_t)idx].enabled = enabled != 0;
    b->dirty = true;
  }
  return 0;
}
extern "C" int kgpu_bank_channels(kgpu_bank const *b) { return b ? b->nchan : -1; }
extern "C" long kgpu_bank_out_stride(kgpu_bank const *b) {
  if (!b) return -1;
  if (b->dirty) bank_commit(const_cast<kgpu_bank *>(b), 0);
  return b->out_stride;
}
extern "C" long kgpu_bank_out_offset(kgpu_bank const *b, int idx) {
  if (bad_idx(b, idx)) return -1;
  if (b->dirty) bank_commit(const_cast<kgpu_bank *>(b), 0);
  return idx < b->nchan ? b->out_off[(size_t)idx] : -1;
}

template <class P> static int launch_chan_v2(ChanArgs const &a, int n, int nblocks, cudaStream_t st, bool osc) {
  size_t const sm = sizeof(float2) * ((size_t)(2 * P::len + 4) * kChanWarps + static_tw_count<P>() + 2);
  static bool attr_done = false;
  if (!attr_done) {
    if (set_smem((const void *)chan_v2<P, false>, sm) || set_smem((const void *)chan_v2<P, true>, sm)) return -1;
    attr_done = true;
  }
  dim3 const g((unsigned)((n + kChanWarps - 1) / kChanWarps), (unsigned)nblocks);
  if (osc) chan_v2<P, true><<<g, kChanWarps * 32, sm, st>>>(a);
  else chan_v2<P, false><<<g, kChanWarps * 32, sm, st>>>(a);
  return 0;
}

template <class P> static int launch_chan_static(ChanArgs const &a, int n, int nblocks, cudaStream_t st) {
  size_t const sm = sizeof(float2) * ((size_t)(2 * P::len + 4) * kChanWarps + static_tw_count<P>() + 2);
  static bool attr_done = false;
  if (!attr_done) {
    if (set_smem((const void *)chan_static<P>, sm)) return -1;
    attr_done = true;
  }
  dim3 const g((unsigned)((n + kChanWarps - 1) / kChanWarps), (unsigned)nblocks);
  chan_static<P><<<g, kChanWarps * 32, sm, st>>>(a);
  return 0;
}

// one (plan, descriptor list) launch
static int launch_chan(kgpu_bank *b, const void *d_spec, int nblocks, void *d_out, long out_stride, int plan,
                       int points, int const *d_order, int base, int n, cudaStream_t st, bool generic = false,
                       float *d_power = nullptr) {
  ChanArgs a;
  a.spec = (float2 const *)d_spec;
  a.spec_stride = b->m->spec_stride;
  a.m_bins = b->m->bins;
  a.wrap = (b->m->in_type == KGPU_COMPLEX);
  a.desc = b->d_desc;
  a.order = d_order;
  a.norder = n;
  a.chan_base = base;
  a.resp = b->d_resp;
  a.out = (float2 *)d_out;
  a.out_stride = out_stride;
  a.pitch = (points + 3) / 4 * 4 + 2;
  a.aux = b->d_aux;
  a.block0 = b->block_counter;
  a.power = d_power;
  a.power_stride = b->capacity;
  ProfScope ps(K_CHAN, st);
  g_launches++;
  TilePlan const *tp = host_tile_plan(plan);
  if (g_static_on.load() && !generic) {
    if (plan_is<S600>(tp)) return launch_chan_v2<S600>(a, n, nblocks, st, b->any_osc);
    if (plan_is<S300>(tp)) return launch_chan_v2<S300>(a, n, nblocks, st, b->any_osc);
    if (plan_is<S1200>(tp)) return launch_chan_static<S1200>(a, n, nblocks, st);
  }
  size_t const sm = sizeof(float2) * (size_t)a.pitch * kChanWarps;
  if (set_smem((const void *)chan_kernel, sm)) return -1;
  dim3 const g((unsigned)((n + kChanWarps - 1) / kChanWarps), (unsigned)nblocks);
  chan_kernel<<<g, kChanWarps * 32, sm, st>>>(a);
  return 0;
}

extern "C" int kgpu_bank_run_ex(kgpu_bank *b, const void *d_spec, int nblocks, void *d_out, long out_pitch, float *d_power, void *stream) {
  if (!b || !d_spec || !d_out || nblocks < 1 || out_pitch < 0) return fail("kgpu_bank_run: bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  if (b->any_osc && b->block_counter - b->last_rebase > 4096) b->dirty = true;  // keep oscillator phases small
  if (bank_commit(b, st)) return -1;
  if (out_pitch && out_pitch < b->out_stride) return fail("kgpu_bank_run_ex: out_pitch %ld < packed row %ld", out_pitch, b->out_stride);
  for (auto const &g : b->groups)
    if (launch_chan(b, d_spec, nblocks, d_out, out_pitch ? out_pitch : b->out_stride, g.plan, g.points, b->d_order + g.off, 0, g.count,
                    st, g.generic, d_power))
      return -1;
  b->block_counter += nblocks;
  CUDA_OK(cudaGetLastError());
  return 0;
}
extern "C" int kgpu_bank_run(kgpu_bank *b, const void *d_spec, int nblocks, void *d_out, void *stream) {
  return kgpu_bank_run_ex(b, d_spec, nblocks, d_out, 0, nullptr, stream);
}
extern "C" int kgpu_bank_run_one_ex(kgpu_bank *b, int idx, const void *d_spec, void *d_out, float *d_power, void *stream);
extern "C" int kgpu_bank_run_one(kgpu_bank *b, int idx, const void *d_spec, void *d_out, void *stream) {
  return kgpu_bank_run_one_ex(b, idx, d_spec, d_out, nullptr, stream);
}
// d_power: nullptr or one float; the block is taken to be block_counter (set it with kgpu_bank_set_block_counter)
extern "C" int kgpu_bank_run_one_ex(kgpu_bank *b, int idx, const void *d_spec, void *d_out, float *d_power, void *stream) {
  if (bad_idx(b, idx) || !d_spec || !d_out) return fail("kgpu_bank_run_one: bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  if (bank_commit(b, st)) return -1;
  ChanHost const &c = b->ch[(size_t)idx];
  if (!c.defined || !c.has_response || !c.enabled) return fail("kgpu_bank_run_one: channel %d not runnable", idx);
  // write this channel's olen samples at d_out[0..olen): shift the row origin back by out_off
  float2 *origin = (float2 *)d_out - b->out_off[(size_t)idx];
  bool const gen = (b->desc[(size_t)idx].flags & (kChanRealOut | kChanBeam)) != 0;
  if (launch_chan(b, d_spec, 1, origin, 0, c.plan, c.points, nullptr, idx, 1, st, gen, d_power ? d_power - idx : nullptr)) return -1;
  CUDA_OK(cudaGetLastError());
  return 0;
}
// Noise density per channel and block from the device-resident spectrum (estimate_noise, radio.c:1783-1866).
extern "C" int kgpu_bank_noise(kgpu_bank *b, const void *d_spec, int nblocks, double samprate, double *d_n0, void *stream) {
  if (!b || !d_spec || !d_n0 || nblocks < 1 || !(samprate > 0)) return fail("kgpu_bank_noise: bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  if (bank_commit(b, st)) return -1;
  if (b->nchan == 0) return 0;
  double const NQ = 0.10, N_cutoff = 1.5;  // radio.c:73-74
  double const z = N_cutoff * (-log(1 - NQ));
  double const correction = 1 / (1 - z * exp(-z) / (1 - exp(-z)));  // radio.c:1842-1843
  NoiseArgs a;
  a.spec = (float2 const *)d_spec;
  a.spec_stride = b->m->spec_stride;
  a.m_bins = b->m->bins;
  a.wrap = (b->m->in_type == KGPU_COMPLEX);
  a.desc = b->d_desc;
  a.shift = b->d_shift;
  a.nchan = b->nchan;
  a.scale = correction / ((double)b->m->bins * samprate);
  a.n0 = d_n0;
  a.n0_stride = b->capacity;
  {
    ProfScope ps(K_NOISE, st);
    noise_kernel<<<dim3((unsigned)b->nchan, (unsigned)nblocks), kNoiseThreads, 0, st>>>(a);
  }
  g_launches++;
  CUDA_OK(cudaGetLastError());
  return 0;
}
// FM discriminator front half on the channel outputs of the run that just filled d_out (fm.c:104-131, :205-231).
extern "C" int kgpu_bank_fm_front(kgpu_bank *b, const void *d_out, long out_pitch, int nblocks, float *d_baseband, double *d_stats,
                                  void *stream) {
  if (!b || !d_out || !d_baseband || !d_stats || nblocks < 1 || out_pitch < 0) return fail("kgpu_bank_fm_front: bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  if (bank_commit(b, st)) return -1;
  if (b->nchan == 0) return 0;
  FmArgs a;
  a.out = (float2 const *)d_out;
  a.out_pitch = out_pitch ? out_pitch : b->out_stride;
  a.desc = b->d_desc;
  a.nblocks = nblocks;
  a.mem_in = b->d_fm_mem[b->fm_parity];
  a.mem_out = b->d_fm_mem[b->fm_parity ^ 1];
  a.baseband = d_baseband;
  a.bb_pitch = 2 * a.out_pitch;
  a.stats = (double2 *)d_stats;
  a.stats_stride = b->capacity;
  b->fm_parity ^= 1;
  {
    ProfScope ps(K_NOISE, st);
    fm_front_kernel<<<dim3((unsigned)b->nchan, (unsigned)nblocks), kFmThreads, 0, st>>>(a);
  }
  g_launches++;
  CUDA_OK(cudaGetLastError());
  return 0;
}
/* make the descriptor table current now (e.g. before reading out_stride) and order it after `stream` */
extern "C" int kgpu_bank_commit(kgpu_bank *b, void *stream) {
  if (!b) return fail("kgpu_bank_commit: bad arguments");
  return bank_commit(b, (cudaStream_t)stream);
}

// pure host helpers (usable without a GPU): what the planner would pick
extern "C" int kgpu_plan_radices(int len, int *radices, int max) {
  std::vector<int> r = choose_radices(len);
  if (len != 1 && r.empty()) return -1;
  for (int i = 0; i < (int)r.size() && i < max; i++) radices[i] = r[(size_t)i];
  return (int)r.size();
}
extern "C" int kgpu_plan_split(long n, int *n1, int *n2) {
  Split2 sp;
  if (!choose_split(n, &sp)) return -1;
  *n1 = sp.n1;
  *n2 = sp.n2;
  return 0;
}

extern "C" double kgpu_algorithmic_bytes(kgpu_master const *m, kgpu_bank const *b, int fmt) {
  if (!m) return 0;
  double const s_in = (m->in_type == KGPU_REAL) ? (fmt == KGPU_FMT_I16 ? 2.0 : 4.0) : (fmt == KGPU_FMT_I16 ? 4.0 : 8.0);
  double bytes = (double)m->N * s_in + (double)m->bins * 8.0;
  if (b)
    for (int i = 0; i < b->nchan; i++) {
      ChanHost const &c = b->ch[(size_t)i];
      if (c.defined && c.enabled && c.has_response) bytes += 8.0 * (2.0 * c.points + c.olen);
    }
  return bytes;
}
