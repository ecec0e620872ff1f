// kgpu.cu -- host side of libka9qgpu.so: plan registry, forward-transform and channel-bank
// launchers behind the C-ABI declared in include/ka9q_gpu.h.  No CPU fallback anywhere: every
// entry point either launches the sm_90a kernels or fails with -1.
#include <cuda_runtime.h>
#include <cudaTypedefs.h>  // PFN_cuTensorMapEncodeTiled: taken from the runtime, the library does not link the driver
#include <math.h>
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <algorithm>
#include <complex>
#include <atomic>
#include <map>
#include <mutex>
#include <string>
#include <vector>

#include "../../include/ka9q_gpu.h"
#include "chan_kernels.cuh"
#include "chan_huge.cuh"
#include "chan_wide.cuh"
#include "small_master.cuh"
#include "fwd_kernels.cuh"
#include "noise_kernel.cuh"
#include "plan.cuh"
#include "static_kernels.cuh"
#include "static_kernels_v2.cuh"
#include "fwd_cols_r36.cuh"
#include "fwd_fused.cuh"
#include "fwd_2s.cuh"
#include "spectrum_kernels.cuh"
#include "bluestein_master.cuh"
#include "bluestein_chan.cuh"
#include "raw_ingest.cuh"
#include "iq_correct.cuh"
#include "siggen.cuh"

using namespace kfft;

// ------------------------------------------------------------------------------------------
static thread_local std::string g_err;
static std::atomic<unsigned long long> g_launches{0};

static std::atomic<int> g_static_on{1};  // tests can force the generic kernels
extern "C" int kgpu_use_static_kernels(int on) {
  g_static_on.store(on != 0);
  return 0;
}
// fwd_cols_r36 fetches its raw tile by tensor copies wherever the input allows (kgpu_use_cols_tma); -1: not yet read
// from KA9Q_COLS_TMA
static std::atomic<int> g_cols_tma{-1};
extern "C" int kgpu_use_cols_tma(int on) {
  g_cols_tma.store(on != 0);
  return 0;
}
static bool cols_tma_on() {
  int v = g_cols_tma.load();
  if (v < 0) {
    char const *e = getenv("KA9Q_COLS_TMA");
    g_cols_tma.compare_exchange_strong(v, (e && *e) ? (atoi(e) != 0) : 1);
    v = g_cols_tma.load();
  }
  return v != 0;
}
// REAL 1296 x 1250 masters run both passes as one launch (fwd_fused_r36_v2) wherever the column pass could take its
// tile by tensor copies (kgpu_use_fused_forward); -1: not yet read from KA9Q_FUSED_FWD
static std::atomic<int> g_fused{-1};
// The L2 discard of the inter-pass rows is off by default: on H100 it cost 0.6 us per cfg-2 block (DESIGN.md section 4).
static std::atomic<int> g_fused_lead{FusedShape::DEFAULT_LEAD}, g_fused_discard{0};
extern "C" int kgpu_use_fused_forward(int on) {
  g_fused.store(on != 0);
  return 0;
}
static bool fused_on() {
  int v = g_fused.load();
  if (v < 0) {
    char const *e = getenv("KA9Q_FUSED_FWD");
    g_fused.compare_exchange_strong(v, (e && *e) ? (atoi(e) != 0) : 1);
    v = g_fused.load();
  }
  return v != 0;
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

// Lets `func` launch with up to `bytes` of dynamic shared memory.  The limit is one value per kernel and device for the
// whole process, shared by every master and bank, so it is only ever raised: a smaller request must not take away what
// another caller already relies on.  It is a ceiling; each launch still asks for its own size, so occupancy is unchanged.
static int allow_smem(const void *func, size_t bytes) {
  if (bytes <= 48 * 1024) return 0;
  static std::mutex mu;
  static std::map<std::pair<int, const void *>, size_t> granted;
  int dev = 0;
  CUDA_OK(cudaGetDevice(&dev));
  std::lock_guard<std::mutex> lk(mu);
  size_t &g = granted[{dev, func}];
  if (bytes <= g) return 0;
  CUDA_OK(cudaFuncSetAttribute(func, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
  g = bytes;
  return 0;
}

// A device buffer used by the launches of one stream, grown on demand by grow(); its owner frees `p`.
struct StreamBuf {
  void *p = nullptr;
  size_t bytes = 0;
};
// Makes `s` at least `bytes` long.  Earlier launches on `st` may still use the old buffer, so it waits for the stream
// before freeing it.  `who` begins the messages.
static int grow(StreamBuf &s, size_t bytes, cudaStream_t st, char const *who) {
  if (s.bytes >= bytes) return 0;
  if (cudaStreamSynchronize(st) != cudaSuccess)
    return fail("%s: cudaStreamSynchronize: %s", who, cudaGetErrorString(cudaGetLastError()));
  cudaFree(s.p);
  s.p = nullptr;
  s.bytes = 0;
  cudaError_t const e = cudaMalloc(&s.p, bytes);
  if (e != cudaSuccess) {
    s.p = nullptr;
    return fail("%s: cudaMalloc(%zu): %s", who, bytes, cudaGetErrorString(e));
  }
  s.bytes = bytes;
  return 0;
}

// ------------------------------------------------------------------ per-launch profiling -----
// When enabled, every kernel launch is bracketed by CUDA events on the launching stream; bench.py
// reads the per-kernel totals for its roofline line (events are markers, they do not serialise).
enum KernelId { K_FWD_COLS = 0, K_FWD_ROWS, K_CHAN, K_NOTCH, K_RESPONSE, K_NOISE, K_FWD_FUSED, K_COUNT };
static char const *const kKernelNames[K_COUNT] = {"fwd_cols", "fwd_rows", "chan", "notch", "response_fft", "noise", "fwd_fused"};
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

// ---- 8-bit, 16-bit and float ingest and per-block statistics of raw ingest (raw_ingest.cuh) ---------------------------
static_assert(sizeof(ScaleChange) == sizeof(kgpu_scale_change), "raw_ingest.cuh mirrors include/ka9q_gpu.h");
// REAL_OK / CPLX_OK: the master types the format exists for (only those kernels are instantiated)
template <class D, bool REAL_OK = true, bool CPLX_OK = true>
static void launch_unpack(dim3 g, cudaStream_t st, bool cplx, const void *d_raw, long history, long L, int nblocks, double scale,
                          ScaleChange const *chg, int nchg, long long a0, float *out, BlockStats *stats) {
  auto const *w = (typename D::Word const *)d_raw;
  if constexpr (CPLX_OK)
    if (cplx) unpack_kernel<D, true><<<g, kRawThreads, 0, st>>>(w, history, L, nblocks, scale, chg, nchg, a0, out, stats);
  if constexpr (REAL_OK)
    if (!cplx) unpack_kernel<D, false><<<g, kRawThreads, 0, st>>>(w, history, L, nblocks, scale, chg, nchg, a0, out, stats);
}
extern "C" int kgpu_unpack8(const void *d_raw, int fmt, int in_type, long history, long L, int nblocks, double scale,
                            const kgpu_scale_change *d_chg, int nchg, long long a0, void *d_out, void *d_stats, void *stream) {
  if (!d_raw || !d_out || history < 0 || nblocks < 0 || (nblocks > 0 && L < 1) || nblocks >= 65535 || nchg < 0 || (nchg && !d_chg) ||
      fmt < KGPU_RAW_U8 || fmt > KGPU_RAW_CF32_FSCALE || (in_type != KGPU_REAL && in_type != KGPU_COMPLEX) ||
      ((fmt == KGPU_RAW_U16 || fmt == KGPU_RAW_F32) && in_type != KGPU_REAL) ||
      ((fmt == KGPU_RAW_SC16Q11 || fmt >= KGPU_RAW_CF32) && in_type != KGPU_COMPLEX) ||
      (fmt >= KGPU_RAW_S16 && ((uintptr_t)d_raw & 1)) || (fmt >= KGPU_RAW_F32 && ((uintptr_t)d_raw & 3)))
    return fail("kgpu_unpack8: bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  BlockStats *stats = (BlockStats *)d_stats;
  if (stats && nblocks) CUDA_OK(cudaMemsetAsync(stats, 0, sizeof(BlockStats) * (size_t)nblocks, st));
  long const longest = std::max(nblocks ? L : 0L, history);
  if (longest == 0) return 0;
  dim3 const g((unsigned)((longest + kRawThreads - 1) / kRawThreads), (unsigned)nblocks + 1);
  bool const cplx = in_type == KGPU_COMPLEX;
  auto const *chg = (ScaleChange const *)d_chg;
  auto *out = (float *)d_out;
#define KGPU_UNPACK(...) launch_unpack<__VA_ARGS__>(g, st, cplx, d_raw, history, L, nblocks, scale, chg, nchg, a0, out, stats)
  switch (fmt) {
    case KGPU_RAW_U8: KGPU_UNPACK(DecodeU8); break;
    case KGPU_RAW_S8: KGPU_UNPACK(DecodeS8); break;
    case KGPU_RAW_S16: KGPU_UNPACK(DecodeS16); break;
    case KGPU_RAW_U16: KGPU_UNPACK(DecodeU16, true, false); break;    // REAL only
    case KGPU_RAW_SC16Q11: KGPU_UNPACK(DecodeSC16Q11, false, true); break;  // COMPLEX only
    case KGPU_RAW_F32: KGPU_UNPACK(DecodeF32, true, false); break;     // REAL only
    case KGPU_RAW_CF32_FSCALE: KGPU_UNPACK(DecodeF32FScale, false, true); break;  // COMPLEX only
    default: KGPU_UNPACK(DecodeF32, false, true); break;               // CF32, CF32_CNRMF: COMPLEX only
  }
#undef KGPU_UNPACK
  g_launches++;
  CUDA_OK(cudaGetLastError());
  if (fmt >= KGPU_RAW_F32 && stats && nblocks) {  // the float formats' energies: a double sum in a fixed order
    dim3 const ge(kEnergyCluster, (unsigned)nblocks);
    auto const *f = (float const *)d_raw;
    int const C = cplx ? 2 : 1;
    if (fmt == KGPU_RAW_CF32) float_energy_kernel<EnergyCnrm><<<ge, kEnergyThreads, 0, st>>>(f, history, L, C, stats);
    else if (fmt == KGPU_RAW_CF32_CNRMF) float_energy_kernel<EnergyCnrmf><<<ge, kEnergyThreads, 0, st>>>(f, history, L, C, stats);
    else float_energy_kernel<EnergySq><<<ge, kEnergyThreads, 0, st>>>(f, history, L, C, stats);
    g_launches++;
    CUDA_OK(cudaGetLastError());
  }
  return 0;
}

extern "C" int kgpu_scale_i16(const void *d_in, int in_type, long count, long long a0, double scale, const kgpu_scale_change *d_chg,
                              int nchg, int derandomize, float *d_out, void *stream) {
  if (!d_in || !d_out || count < 0 || nchg < 0 || (nchg && !d_chg) || (in_type != KGPU_REAL && in_type != KGPU_COMPLEX))
    return fail("kgpu_scale_i16: bad arguments");
  if (count == 0) return 0;
  auto const k = in_type == KGPU_COMPLEX ? scale_i16_kernel<true> : scale_i16_kernel<false>;
  k<<<(unsigned)((count + kRawThreads - 1) / kRawThreads), kRawThreads, 0, (cudaStream_t)stream>>>(
      (short const *)d_in, count, a0, scale, (ScaleChange const *)d_chg, nchg, derandomize != 0, d_out);
  g_launches++;
  CUDA_OK(cudaGetLastError());
  return 0;
}

extern "C" int kgpu_block_stats_i16(const void *d_in, int in_type, long history, long L, int nblocks, int derandomize, int limit,
                                    void *d_stats, void *stream) {
  if (!d_in || !d_stats || history < 0 || L < 1 || nblocks < 1 || nblocks >= 65535 || limit < 1 ||
      (in_type != KGPU_REAL && in_type != KGPU_COMPLEX))
    return fail("kgpu_block_stats_i16: bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  CUDA_OK(cudaMemsetAsync(d_stats, 0, sizeof(BlockStats) * (size_t)nblocks, st));
  dim3 const g((unsigned)((L + kRawThreads - 1) / kRawThreads), (unsigned)nblocks);
  auto const k = in_type == KGPU_COMPLEX ? block_stats_i16_kernel<true> : block_stats_i16_kernel<false>;
  k<<<g, kRawThreads, 0, st>>>((short const *)d_in, history, L, derandomize != 0, limit, (BlockStats *)d_stats);
  g_launches++;
  CUDA_OK(cudaGetLastError());
  return 0;
}

// ---- I/Q correction of the HackRF and FUNcube drivers (iq_correct.cuh) ----------------------------------------------
static_assert(sizeof(IqWrite) == sizeof(kgpu_iq_write) && sizeof(IqState) == sizeof(kgpu_iq_state) &&
                  sizeof(IqRecord) == sizeof(kgpu_iq_record),
              "iq_correct.cuh mirrors include/ka9q_gpu.h");
static bool iq_args(const void *d_raw, int fmt, long count, const void *d_tab, int cap, int nw) {
  return d_raw && d_tab && count >= 0 && cap > 0 && nw > 0 && nw <= cap && (fmt == KGPU_IQ_S8 || fmt == KGPU_IQ_S16) &&
         (count + kIqChunk - 1) / kIqChunk < 0x7fffffffL;
}

extern "C" int kgpu_iq_moments(const void *d_raw, int fmt, long long a0, long count, kgpu_iq_write *d_tab, int cap,
                               long long w_lo, int nw, void *stream) {
  if (!iq_args(d_raw, fmt, count, d_tab, cap, nw) || a0 < 0 || w_lo < 0) return fail("kgpu_iq_moments: bad arguments");
  if (count == 0) return 0;
  auto const k = fmt == KGPU_IQ_S16 ? iq_moments_kernel<true> : iq_moments_kernel<false>;
  k<<<(unsigned)((count + kIqChunk - 1) / kIqChunk), kIqThreads, 0, (cudaStream_t)stream>>>(d_raw, a0, count, (IqWrite *)d_tab,
                                                                                           cap, w_lo, nw);
  g_launches++;
  CUDA_OK(cudaGetLastError());
  return 0;
}

extern "C" int kgpu_iq_scan(const kgpu_iq_write *d_tab, kgpu_iq_state *d_coef, int cap, long long w_from, int nw,
                            const kgpu_iq_params *params, kgpu_iq_record *d_rec, void *stream) {
  if (!d_tab || !d_coef || !d_rec || !params || cap < 2 || nw < 0 || nw >= cap || w_from < 0 ||
      (params->kind != 1 && params->kind != 2))
    return fail("kgpu_iq_scan: bad arguments");
  if (nw == 0) return 0;
  IqParams const p = {params->kind, params->dc_alpha, params->gp};
  iq_scan_kernel<<<1, 1, 0, (cudaStream_t)stream>>>((IqWrite const *)d_tab, (IqState *)d_coef, cap, w_from, nw, p,
                                                    (IqRecord *)d_rec);
  g_launches++;
  CUDA_OK(cudaGetLastError());
  return 0;
}

extern "C" int kgpu_iq_apply(const void *d_raw, int fmt, long long a0, long count, const kgpu_iq_write *d_tab,
                             const kgpu_iq_state *d_coef, int cap, long long w_lo, int nw, void *d_out, void *stream) {
  if (!iq_args(d_raw, fmt, count, d_tab, cap, nw) || !d_coef || !d_out || w_lo < 0) return fail("kgpu_iq_apply: bad arguments");
  if (count == 0) return 0;
  auto const k = fmt == KGPU_IQ_S16 ? iq_apply_kernel<true> : iq_apply_kernel<false>;
  k<<<(unsigned)((count + kIqChunk - 1) / kIqChunk), kIqThreads, 0, (cudaStream_t)stream>>>(
      d_raw, a0, count, (IqWrite const *)d_tab, (IqState const *)d_coef, cap, w_lo, nw, (float2 *)d_out);
  g_launches++;
  CUDA_OK(cudaGetLastError());
  return 0;
}

// ---- sig_gen.c's CW, AM and DSB sources (siggen.cuh) -----------------------------------------------------------------
extern "C" void kgpu_siggen_angle128(double f, uint64_t *out);  // siggen_host.c
namespace {
// T^(2^b), b = 0 .. 63, of xoshiro256**'s state transition, in siggen.cuh's nibble-table form; built once per process
std::vector<unsigned long long> g_jump;
std::once_flag g_jump_once;
void xo_step_host(unsigned long long s[4]) {
  unsigned long long const t = s[1] << 17;
  s[2] ^= s[0];
  s[3] ^= s[1];
  s[1] ^= s[2];
  s[0] ^= s[3];
  s[2] ^= t;
  s[3] = (s[3] << 45) | (s[3] >> 19);
}
void gf2_apply_host(unsigned long long const *tab, unsigned long long s[4]) {
  unsigned long long y[4] = {0, 0, 0, 0};
  for (int w = 0; w < 4; w++)
    for (int q = 0; q < 16; q++) {
      unsigned long long const *e = tab + ((w * 16 + q) * 16 + (int)((s[w] >> (4 * q)) & 15)) * 4;
      for (int k = 0; k < 4; k++) y[k] ^= e[k];
    }
  for (int k = 0; k < 4; k++) s[k] = y[k];
}
// nibble tables of the matrix whose column j (the image of state bit j = bit j % 64 of word j / 64) is cols[j]
void gf2_tables(unsigned long long const (*cols)[4], unsigned long long *tab) {
  for (int w = 0; w < 4; w++)
    for (int q = 0; q < 16; q++)
      for (int v = 0; v < 16; v++) {
        unsigned long long *e = tab + ((w * 16 + q) * 16 + v) * 4;
        e[0] = e[1] = e[2] = e[3] = 0;
        for (int i = 0; i < 4; i++)
          if ((v >> i) & 1)
            for (int k = 0; k < 4; k++) e[k] ^= cols[w * 64 + 4 * q + i][k];
      }
}
void build_jumps() {
  g_jump.assign((size_t)64 * kGf2Table, 0);
  static unsigned long long cols[256][4];
  for (int j = 0; j < 256; j++) {
    for (int k = 0; k < 4; k++) cols[j][k] = 0;
    cols[j][j / 64] = 1ULL << (j % 64);
    xo_step_host(cols[j]);
  }
  gf2_tables(cols, g_jump.data());
  for (int b = 1; b < 64; b++) {  // T^(2^b) = T^(2^(b-1)) applied to each column of itself
    for (int j = 0; j < 256; j++) gf2_apply_host(g_jump.data() + (size_t)(b - 1) * kGf2Table, cols[j]);
    gf2_tables(cols, g_jump.data() + (size_t)b * kGf2Table);
  }
}
unsigned long long splitmix64(unsigned long long *x) {  // gauss.c:24-29
  unsigned long long z = (*x += 0x9E3779B97F4A7C15ULL);
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ULL;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBULL;
  return z ^ (z >> 31);
}
}  // namespace

struct kgpu_siggen {
  bool cplx;
  bool mod;   // AM / DSB (kgpu_siggen_set_modulation): one draw per sample, the envelope from kgpu_siggen_generate_mod
  double dc;  // and its carrier component
  kgpu_siggen_params p;
  unsigned long long seeded[4];  // xoshiro256ss_seed (gauss.c:32-44)
  U128 F, R;
  unsigned long long *d_tabs;  // T^(kGenRun 2^b), b < kGenJumpBits
  double *d_part;
  long part_cap;
};
constexpr int kGenLog2Run = 6;
static_assert(kGenRun == 64, "kGenLog2Run");

extern "C" kgpu_siggen *kgpu_siggen_create(int in_type, const kgpu_siggen_params *p) {
  if (!p || (in_type != KGPU_REAL && in_type != KGPU_COMPLEX) || !std::isfinite(p->freq) || !std::isfinite(p->rate) ||
      !std::isfinite(p->amplitude) || !std::isfinite(p->noise)) {
    fail("kgpu_siggen_create: bad arguments");
    return nullptr;
  }
  std::call_once(g_jump_once, build_jumps);
  auto *g = new kgpu_siggen();
  g->cplx = in_type == KGPU_COMPLEX;
  g->p = *p;
  unsigned long long x = p->seed;
  for (int k = 0; k < 4; k++) g->seeded[k] = splitmix64(&x);
  if ((g->seeded[0] | g->seeded[1] | g->seeded[2] | g->seeded[3]) == 0) g->seeded[0] = 1;
  uint64_t a[2];
  kgpu_siggen_angle128(p->freq, a);
  g->F = {a[0], a[1]};
  kgpu_siggen_angle128(p->rate, a);
  g->R = {a[0], a[1]};
  return g;
}

extern "C" void kgpu_siggen_destroy(kgpu_siggen *g) {
  if (!g) return;
  cudaFree(g->d_tabs);
  cudaFree(g->d_part);
  delete g;
}

extern "C" int kgpu_siggen_state(const kgpu_siggen *g, unsigned long long draw, uint64_t *out) {
  if (!g || !out) return fail("kgpu_siggen_state: bad arguments");
  unsigned long long s[4] = {g->seeded[0], g->seeded[1], g->seeded[2], g->seeded[3]};
  for (int b = 0; b < 64; b++)
    if ((draw >> b) & 1) gf2_apply_host(g_jump.data() + (size_t)b * kGf2Table, s);
  for (int k = 0; k < 4; k++) out[k] = s[k];
  return 0;
}

extern "C" int kgpu_siggen_angles(const kgpu_siggen *g, uint64_t *out) {
  if (!g || !out) return fail("kgpu_siggen_angles: bad arguments");
  out[0] = g->F.lo;
  out[1] = g->F.hi;
  out[2] = g->R.lo;
  out[3] = g->R.hi;
  return 0;
}

extern "C" int kgpu_siggen_set_modulation(kgpu_siggen *g, double dc) {
  if (!g || !std::isfinite(dc)) return fail("kgpu_siggen_set_modulation: bad arguments");
  g->mod = true;
  g->dc = dc;
  return 0;
}

// kgpu_siggen_generate and _generate_mod: d_mod is NULL exactly when the generator is not modulated
static int siggen_launch(kgpu_siggen *g, long long a0, long count, double scale, const kgpu_scale_change *d_chg, int nchg,
                         void *d_out, const float *d_mod, double *d_block_energy, int nblocks, long L, long history,
                         void *stream, char const *who) {
  int const C = g && g->cplx ? 2 : 1;                   // floats per sample
  int const D = g && g->cplx && !g->mod ? 2 : 1;        // draws per sample
  int const S = kGenRun / D;                            // samples per thread
  if (!g || !d_out || (g->mod != (d_mod != nullptr)) || count < 0 || history < 0 || nblocks < 0 || nchg < 0 ||
      (nchg && !d_chg) || (nblocks > 0 && (L < S || count != history + (long)nblocks * L)) ||
      (a0 < 0 && std::min(-a0, (long long)count) > history))
    return fail("%s: bad arguments", who);
  cudaStream_t st = (cudaStream_t)stream;
  float *out = (float *)d_out;
  if (a0 < 0) {  // the samples before the stream's first: zeros, all inside the history
    long const z = (long)std::min(-a0, (long long)count);
    CUDA_OK(cudaMemsetAsync(out, 0, sizeof(float) * (size_t)C * (size_t)z, st));
    out += (size_t)C * (size_t)z;
    if (d_mod) d_mod += z;
    count -= z;
    history -= z;
    a0 = 0;
  }
  long const nthreads = (count + S - 1) / S;
  if (nthreads >= (1L << kGenJumpBits)) return fail("%s: %ld samples exceed one launch", who, count);
  if (count == 0) return 0;
  long const grid = (nthreads + kGenThreads - 1) / kGenThreads;
  if (!g->d_tabs) {  // the device's jump matrices, at the first launch (create is pure host code)
    size_t const bytes = sizeof(unsigned long long) * (size_t)kGenJumpBits * kGf2Table;
    CUDA_OK(cudaMalloc((void **)&g->d_tabs, bytes));
    CUDA_OK(cudaMemcpy(g->d_tabs, g_jump.data() + (size_t)kGenLog2Run * kGf2Table, bytes, cudaMemcpyHostToDevice));
  }
  if (d_block_energy && nblocks > 0 && 2 * grid * kGenThreads > g->part_cap) {
    CUDA_OK(cudaStreamSynchronize(st));  // the previous launch may still write the old scratch
    cudaFree(g->d_part);
    g->d_part = nullptr;
    g->part_cap = 0;
    CUDA_OK(cudaMalloc((void **)&g->d_part, sizeof(double) * 2 * (size_t)grid * kGenThreads));
    g->part_cap = 2 * grid * kGenThreads;
  }
  GenArgs a;
  uint64_t base[4];
  kgpu_siggen_state(g, (unsigned long long)a0 * (unsigned long long)D, base);
  for (int k = 0; k < 4; k++) a.base[k] = base[k];
  a.F = g->F;
  a.R = g->R;
  a.amplitude = g->p.amplitude;
  a.noise = g->p.noise;
  a.scale = scale;
  a.chg = (ScaleChange const *)d_chg;
  a.nchg = nchg;
  a.a0 = a0;
  a.count = count;
  a.history = history;
  a.L = nblocks > 0 ? L : 1;
  a.tabs = g->d_tabs;
  a.out = out;
  a.part = d_block_energy && nblocks > 0 ? g->d_part : nullptr;
  a.dc = g->dc;
  a.mod = d_mod;
  auto const k = g->mod ? (g->cplx ? siggen_kernel<true, true> : siggen_kernel<false, true>)
                        : (g->cplx ? siggen_kernel<true, false> : siggen_kernel<false, false>);
  k<<<(unsigned)grid, kGenThreads, 0, st>>>(a);
  g_launches++;
  CUDA_OK(cudaGetLastError());
  if (a.part) {
    siggen_energy_kernel<<<nblocks, 256, 0, st>>>(a.part, history, L, S, nthreads, d_block_energy);
    g_launches++;
    CUDA_OK(cudaGetLastError());
  }
  return 0;
}

extern "C" int kgpu_siggen_generate(kgpu_siggen *g, long long a0, long count, double scale, const kgpu_scale_change *d_chg, int nchg,
                                    void *d_out, double *d_block_energy, int nblocks, long L, long history, void *stream) {
  return siggen_launch(g, a0, count, scale, d_chg, nchg, d_out, nullptr, d_block_energy, nblocks, L, history, stream,
                       "kgpu_siggen_generate");
}

extern "C" int kgpu_siggen_generate_mod(kgpu_siggen *g, long long a0, long count, double scale, const kgpu_scale_change *d_chg,
                                        int nchg, void *d_out, const float *d_mod, double *d_block_energy, int nblocks, long L,
                                        long history, void *stream) {
  return siggen_launch(g, a0, count, scale, d_chg, nchg, d_out, d_mod, d_block_energy, nblocks, L, history, stream,
                       "kgpu_siggen_generate_mod");
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
// The extended set of masters created with kgpu_master_create_ex: the same radices, then the five primes.  A prime
// above 7 divides no radix of kRadixSet, so every factorisation carries each of them as its own stage, and on a length
// with factors 2, 3, 5, 7 only the search visits exactly what it visits with kRadixSet.
static int const kRadixSetExt[] = {25, 24, 20, 16, 15, 12, 10, 9, 8, 7, 6, 5, 4, 3, 2, 23, 19, 17, 13, 11};

// Every length the registry accepts has prime factors 2, 3, 5, 7 only and is at most kMaxChanPoints: masters split into
// lengths <= kMaxTileLen and kgpu_bank_define rejects channels whose transform the channel kernel cannot hold.  If all
// of them fit, the registry can never fill, and which lengths a process has used (master rates, channel rates, test
// order) cannot make a creation fail.
static_assert(kMaxChanPoints >= kMaxTileLen, "every tile length must also be a valid channel length");
constexpr int plannable_lengths(int max) {
  int count = 0;
  for (int n = 1; n <= max; n++) {
    int v = n;
    for (int p : {2, 3, 5, 7})
      while (v % p == 0) v /= p;
    count += (v == 1);
  }
  return count;
}
static_assert(plannable_lengths(kMaxChanPoints) <= kMaxPlans, "the plan registry must hold every plannable length");

// exhaustive search over multisets of the radices set[0 .. nset) (depth <= kMaxStages): fewest stages,
// then smallest sum.
static void search(int const *set, int nset, int n, int start, std::vector<int> &cur, std::vector<int> &best,
                   int &best_sum) {
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
  for (int i = start; i < nset; i++) {
    int const r = set[i];
    if (n % r) continue;
    cur.push_back(r);
    search(set, nset, n / r, i, cur, best, best_sum);
    cur.pop_back();
  }
}

static std::vector<int> radices_from(int const *set, int nset, int n) {
  std::vector<int> cur, best;
  int best_sum = 0;
  if (n < 2) return best;
  search(set, nset, n, 0, cur, best, best_sum);
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

std::vector<int> choose_radices(int n) { return radices_from(kRadixSet, (int)(sizeof kRadixSet / sizeof kRadixSet[0]), n); }
std::vector<int> choose_radices_ext(int n) {
  return radices_from(kRadixSetExt, (int)(sizeof kRadixSetExt / sizeof kRadixSetExt[0]), n);
}

struct PlanSlot {
  int len = 0;
  TilePlan host;  // device pointers inside
};
static std::mutex g_plan_mu;
static std::vector<PlanSlot> g_plans;

// Builds the column plan of `len` with stages `rad` and uploads its twiddle and perm tables (freed with free_tile_plan).
static int make_tile_plan(int len, std::vector<int> const &rad, TilePlan &p) {
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
  p.tw = nullptr;
  p.perm = nullptr;
  auto upload = [&]() -> int {
    CUDA_OK(cudaMalloc(&d_tw, sizeof(float2) * tw.size()));
    CUDA_OK(cudaMalloc(&d_perm, sizeof(uint16_t) * (size_t)len));
    CUDA_OK(cudaMemcpy(d_tw, tw.data(), sizeof(float2) * tw.size(), cudaMemcpyHostToDevice));
    CUDA_OK(cudaMemcpy(d_perm, perm.data(), sizeof(uint16_t) * (size_t)len, cudaMemcpyHostToDevice));
    return 0;
  };
  if (upload()) {  // the CUDA error is in kgpu_last_error()
    cudaFree(d_tw);
    cudaFree(d_perm);
    return -1;
  }
  p.tw = d_tw;
  p.perm = d_perm;
  return 0;
}
static void free_tile_plan(TilePlan &p) {
  cudaFree((void *)p.tw);
  cudaFree((void *)p.perm);
  p.tw = nullptr;
  p.perm = nullptr;
}

int get_tile_plan(int len) {
  std::lock_guard<std::mutex> lk(g_plan_mu);
  for (size_t i = 0; i < g_plans.size(); i++)
    if (g_plans[i].len == len) return (int)i;
  std::vector<int> rad;
  if (len > 1) rad = choose_radices(len);
  if (len < 1 || len > kMaxChanPoints || (len > 1 && rad.empty()))
    return fail("%d-point transform cannot be planned (factors 2, 3, 5, 7; at most %d points)", len, kMaxChanPoints);
  if ((int)g_plans.size() >= kMaxPlans) return fail("plan registry full (%d plans)", kMaxPlans);
  TilePlan p;
  if (make_tile_plan(len, rad, p)) return -1;
  int const idx = (int)g_plans.size();
  cudaError_t const e = cudaMemcpyToSymbol(c_plans, &p, sizeof p, sizeof(TilePlan) * (size_t)idx);
  if (e != cudaSuccess) {
    free_tile_plan(p);
    return fail("cudaMemcpyToSymbol(c_plans): %s", cudaGetErrorString(e));
  }
  PlanSlot sl;
  sl.len = len;
  sl.host = p;
  g_plans.push_back(sl);
  return idx;
}
TilePlan const *host_tile_plan(int idx) { return &g_plans[(size_t)idx].host; }

static bool plannable(int len) { return len == 1 || (len <= kMaxTileLen && !choose_radices(len).empty()); }
static bool plannable_ext(int len) { return len == 1 || (len <= kMaxTileLen && !choose_radices_ext(len).empty()); }

// the largest d <= sqrt(n) with n = (n / d) * d, n / d <= kMaxTileLen and both factors plannable
template <bool (*Plannable)(int)> static bool split_with(long n, Split2 *out) {
  long best = -1;
  for (long d = (long)floor(sqrt((double)n) + 1e-9); d >= 1; d--) {
    if (n % d) continue;
    long const a = n / d;  // a >= d
    if (a > kMaxTileLen) break;
    if (Plannable((int)a) && Plannable((int)d)) {
      best = d;
      break;
    }
  }
  if (best < 0) return false;
  out->n1 = (int)(n / best);
  out->n2 = (int)best;
  return true;
}
bool choose_split(long n, Split2 *out) { return split_with<plannable>(n, out); }
bool choose_split_ext(long n, Split2 *out) { return split_with<plannable_ext>(n, out); }

// choose_split restated at compile time (a length <= kMaxTileLen is plannable iff its factors are 2, 3, 5, 7), to pin
// kMaxWideChanPoints: every such length above kMaxChanPoints up to it fits chan_wide's shared memory, the next does not.
constexpr bool smooth7(long n) {
  for (long p : {2, 3, 5, 7})
    while (n % p == 0) n /= p;
  return n == 1;
}
constexpr bool wide_fits(long n) {
  long d = 1;
  while ((d + 1) * (d + 1) <= n) d++;
  for (; d >= 1; d--) {
    if (n % d) continue;
    if (n / d > kMaxTileLen) return false;
    if (smooth7(n / d) && smooth7(d)) return wide_smem_bytes((int)(n / d), (int)d) <= kChanSmemLimit;
  }
  return false;
}
constexpr bool all_wide_fit(long lo, long hi) {
  for (long n = lo; n <= hi; n++)
    if (smooth7(n) && !wide_fits(n)) return false;
  return true;
}
constexpr long next_smooth7(long n) {
  while (!smooth7(n)) n++;
  return n;
}
static_assert(all_wide_fit(kMaxChanPoints + 1, kMaxWideChanPoints), "a wide length up to the maximum does not fit");
static_assert(!wide_fits(next_smooth7(kMaxWideChanPoints + 1)), "kMaxWideChanPoints is below what shared memory holds");

static int plan_slot(TilePlan const &p, int k) {  // slot holding X[k] after the plan's last stage (its perm[k])
  int slot = 0;
  for (int i = 0; i < p.nstages; i++) {
    slot += (k % p.radix[i]) * p.stride[i];
    k /= p.radix[i];
  }
  return slot;
}

// Sets g.tw, the device table of W_Ns^{k1 j2}: pass 1 leaves output j2 in column plan_slot(p2, j2), so it is tabulated
// in column order.  p2: the plan of length g.n2.
static int wide_twiddles(WideGeom &g, TilePlan const &p2) {
  long const points = (long)g.n1 * g.n2;
  std::vector<float2> tw((size_t)points);
  for (int j2 = 0; j2 < g.n2; j2++) {
    int const c = plan_slot(p2, j2);
    for (int k1 = 0; k1 < g.n1; k1++) {
      long double const ang = -2.0L * M_PIl * (long double)((long)k1 * j2) / (long double)points;
      tw[(size_t)k1 * g.n2 + c] = make_float2((float)cosl(ang), (float)sinl(ang));
    }
  }
  float2 *d_tw = nullptr;
  if (cudaMalloc(&d_tw, sizeof(float2) * tw.size()) != cudaSuccess ||
      cudaMemcpy(d_tw, tw.data(), sizeof(float2) * tw.size(), cudaMemcpyHostToDevice) != cudaSuccess) {
    cudaFree(d_tw);
    return fail("%ld-point transform: twiddle upload failed", points);
  }
  g.tw = d_tw;
  return 0;
}

// Pins kMaxHugeChanPoints: every length with factors 2, 3, 5, 7 in (kMaxWideChanPoints, kMaxHugeChanPoints] splits
// into two plannable factors whose kTile-column tiles fit shared memory (the largest factor is 2401, for 823 543 =
// 2401 x 343), and there are 806 of them.  The lengths are enumerated by their exponents to keep the evaluation short.
constexpr bool huge_fits(long n) {
  long d = 1;
  while ((d + 1) * (d + 1) <= n) d++;
  for (; d >= 1; d--) {
    if (n % d) continue;
    if (n / d > kMaxTileLen) return false;
    if (smooth7(n / d) && smooth7(d)) return huge_smem_bytes((int)(n / d)) <= kChanSmemLimit && huge_smem_bytes((int)d) <= kChanSmemLimit;
  }
  return false;
}
constexpr long huge_lengths(long lo, long hi) {  // how many 7-smooth lengths in (lo, hi]; -1 if one does not fit
  long count = 0;
  for (long a = 1; a <= hi; a *= 2)
    for (long b = a; b <= hi; b *= 3)
      for (long c = b; c <= hi; c *= 5)
        for (long e = c; e <= hi; e *= 7)
          if (e > lo) {
            if (!huge_fits(e)) return -1;
            count++;
          }
  return count;
}
static_assert(huge_lengths(kMaxWideChanPoints, kMaxHugeChanPoints) == 806, "a huge length does not split or fit");

// ---- channels whose length has a prime factor 11 .. 23 (kgpu_bank_define_ext) ----
// They keep their plans out of the registry: c_plans holds exactly the 7-smooth lengths, whose count kMaxPlans is
// sized for.  Their kernels, chan_kernel_ext and chan_wide_ext, take the plans by value instead.
constexpr bool smooth23(long n) {
  for (long p : {2, 3, 5, 7, 11, 13, 17, 19, 23})
    while (n % p == 0) n /= p;
  return n == 1;
}
constexpr bool extended(long n) { return smooth23(n) && !smooth7(n); }
// choose_split_ext restated as wide_fits is (a length <= kMaxTileLen is plannable_ext iff its factors reach 23 at most)
constexpr bool wide_fits_ext(long n) {
  long d = 1;
  while ((d + 1) * (d + 1) <= n) d++;
  for (; d >= 1; d--) {
    if (n % d) continue;
    if (n / d > kMaxTileLen) return false;
    if (smooth23(n / d) && smooth23(d)) return wide_smem_bytes((int)(n / d), (int)d) <= kChanSmemLimit;
  }
  return false;
}
constexpr long ext_lengths(long lo, long hi, bool wide) {  // extended lengths in [lo, hi]; -1 if a wide one does not fit
  long count = 0;
  for (long n = lo; n <= hi; n++)
    if (extended(n)) {
      if (wide && !wide_fits_ext(n)) return -1;
      count++;
    }
  return count;
}
// 863 extended lengths run chan_kernel_ext (7260 = 2^2 3 5 11^2 is one of them), and 1032 more, up to 28798 =
// 2 7 11^2 17, split into two factors of at most kMaxTileLen whose chan_wide_ext footprint fits shared memory.
static_assert(ext_lengths(2, kMaxChanPoints, false) == 863, "extended channel lengths up to kMaxChanPoints");
static_assert(ext_lengths(kMaxChanPoints + 1, kMaxWideChanPoints, true) == 1032, "an extended wide length does not split or fit");

// The largest prime factor of n above 7, or 1 if n has none.
static long factor_above7(long n) {
  long big = 1;
  for (long p = 2; p * p <= n; p++)
    while (n % p == 0) {
      n /= p;
      if (p > 7) big = p;
    }
  return n > 7 ? std::max(big, n) : big;
}

// the split kgpu_master_create(_ex) would run for nc complex points, if its kernels fit shared memory
static bool forward_split(long nc, bool ext, Split2 *sp) {
  if (!(ext ? choose_split_ext(nc, sp) : choose_split(nc, sp))) return false;
  size_t const smem1 = sizeof(float2) * ((size_t)kTile * column_pitch(sp->n1) + (size_t)kTile * ((sp->n1 + 31) / 32));
  size_t const smem2 = sizeof(float2) * ((size_t)kTile * column_pitch(sp->n2));
  return smem1 <= (size_t)kChanSmemLimit && smem2 <= (size_t)kChanSmemLimit;
}

// A Bluestein transform of n points (bluestein_master.cuh), as masters, channels and the spectrum analyzer run it: two
// passes of an internal 7-smooth COMPLEX master of length P around bluestein_mul_kernel.  bluestein_shape fills n, P and
// the split without a device; bluestein_upload computes B and puts it on the device, where its owner frees it.
struct Bluestein {
  long n = 0;
  long P = 0;             // the smallest length >= 2n - 1 with factors 2, 3, 5, 7 whose split the forward pair runs
  Split2 sp{};            // the split of P
  float2 *d_b = nullptr;  // B = DFT_P of the conjugate chirp
};
// The largest P is 3500 x 3500; false if n needs more.
static bool bluestein_shape(long n, Bluestein *b) {
  long const limit = (long)kMaxTileLen * kMaxTileLen;
  for (long p = 2 * n - 1; p <= limit; p++)
    if (smooth7(p) && forward_split(p, false, &b->sp)) {
      b->n = n;
      b->P = p;
      return true;
    }
  return false;
}

// Forward DFT of n points (factors 2, 3, 5, 7) in place, in double: decimation in time, radix = smallest factor.
// tw[e * d] = exp(-2 pi i e / n) (d: the stride of this sub-transform in the top-level table).
static void host_dft(std::complex<double> *x, long n, std::complex<double> const *tw, long d) {
  if (n == 1) return;
  int const r = n % 2 == 0 ? 2 : n % 3 == 0 ? 3 : n % 5 == 0 ? 5 : 7;
  long const m = n / r;
  std::vector<std::complex<double>> t((size_t)n);
  for (long j = 0; j < m; j++)
    for (int q = 0; q < r; q++) t[(size_t)(q * m + j)] = x[j * r + q];
  for (int q = 0; q < r; q++) host_dft(t.data() + q * m, m, tw, d * r);
  for (long k = 0; k < m; k++)
    for (int s = 0; s < r; s++) {
      long const kk = k + s * m;
      std::complex<double> acc = t[(size_t)k];
      for (int q = 1; q < r; q++) acc += t[(size_t)(q * m + k)] * tw[(size_t)(((long)q * kk) % n * d)];
      x[kk] = acc;
    }
}

// B = DFT_P(b), b_m = conj(w_m) on -(n-1) .. n-1 wrapped modulo P, w_m = exp(-i pi m^2 / n): transformed in double on
// the host and rounded once, since a float transform here would add a third float transform's error to every result.
static std::vector<float2> bluestein_bspec(long n, long P) {
  std::vector<std::complex<double>> bd((size_t)P), tw((size_t)P);
  for (long m = 0; m < n; m++) {
    long double const ang = M_PIl * (long double)((m * m) % (2 * n)) / (long double)n;
    std::complex<double> const v((double)cosl(ang), (double)sinl(ang));  // conj(exp(-i ang))
    bd[(size_t)m] = v;
    if (m) bd[(size_t)(P - m)] = v;
  }
  for (long e2 = 0; e2 < P; e2++) {
    long double const ang = -2.0L * M_PIl * (long double)e2 / (long double)P;
    tw[(size_t)e2] = std::complex<double>((double)cosl(ang), (double)sinl(ang));
  }
  host_dft(bd.data(), P, tw.data(), 1);
  std::vector<float2> b((size_t)P);
  for (long k = 0; k < P; k++) b[(size_t)k] = make_float2((float)bd[(size_t)k].real(), (float)bd[(size_t)k].imag());
  return b;
}
}  // namespace kfft

// ------------------------------------------------------------------ master ------------------
// The kernel pair of a master is chosen once, in kgpu_master_create, from its split n1 x n2:
//   COMPLEX 800 x 625       fwd_cols_2s<f, 25, 32> + fwd_rows_2s<25, 25>     (fwd_2s.cuh)
//   n1 = 1296               column pass fwd_cols_r36                           (fwd_cols_r36.cuh)
//   n2 = 1250               row pass fwd_rows_v2                               (static_kernels_v2.cuh)
//   anything else           the runtime-plan kernels fwd_cols_kernel / fwd_rows_kernel (fwd_kernels.cuh)
// When both passes of a REAL master are specialised (1296 x 1250) the 1/2 of the real split rides on the column pass's
// inter-pass twiddle, and the inter-pass rows of a specialised pair are padded to 128 bytes.  kgpu_use_static_kernels(0)
// runs the generic pair instead, at launch time.
// fwd_cols_r36 comes in two forms with the same arithmetic, chosen per launch (forward_span): fwd_cols_r36_tma has its
// input tile copied into shared memory by tensor copies, wherever cols_tma_fits finds the input's base and strides 16-byte
// aligned; fwd_cols_r36 reads it with global loads for any other input, or with kgpu_use_cols_tma(0) / KA9Q_COLS_TMA=0.
enum ColsKernel { COLS_GENERIC, COLS_R36, COLS_2S };
enum RowsKernel { ROWS_GENERIC, ROWS_V2, ROWS_2S };

struct kgpu_master {
  int L, M, N, in_type, bins;
  long nc;           // complex points of the two-pass transform (N/2 for REAL, N for COMPLEX)
  Split2 sp;
  int plan1, plan2, pitch1, pitch2;
  long spec_stride;
  int n_item_ctas = 0;             // CTAs per block of fwd_rows_kernel (row_item(): 4 pairs or 8 rows)
  int n_rows_ctas = 0;             // CTAs per block of the master's own row kernel (fwd_rows_v2 REAL: 8 pairs)
  ColsKernel cols = COLS_GENERIC;
  RowsKernel rows = ROWS_GENERIC;
  bool halved = false;             // the 1/2 of the real split is folded into the column pass
  int n1c = 0, n2c = 0;            // compile-time n1 of fwd_rows_v2, n2 of fwd_cols_r36 (0 = from the arguments)
  int mid_ld = 0;                  // row pitch of the inter-pass buffer for the chosen pair
  float2 *d_rootD = nullptr;       // REAL: split roots of the row pass
  float2 *d_rootC = nullptr;       // REAL with fwd_rows_v2: W_{2nc}^{k1}
  float2 *d_tw0 = nullptr, *d_twA = nullptr, *d_twB = nullptr;  // tables of fwd_cols_r36 / fwd_cols_2s
  float2 *d_rtw0 = nullptr;        // stage-0 powers of fwd_rows_2s
  StreamBuf mid;                   // the inter-pass buffer
  StreamBuf fused_ctr;             // fwd_fused_r36_v2's ticket and done counters (FusedArgs::ctr)
  size_t smem1 = 0, smem2 = 0;     // generic kernels
  // kgpu_master_create_ex with a prime factor 11 .. 23: the master owns its two plans (plan1 / plan2 stay -1) and runs
  // the extended pair fwd_cols_ext / fwd_rows_ext, which take them by value
  bool ext = false;
  TilePlan xplan1{}, xplan2{};
  // kgpu_master_create_any with a Bluestein transform of nc points: the internal COMPLEX master of length blue.P, and
  // the chirped input and the passes' spectra of chunks of at most b_chunk blocks
  kgpu_master *bs = nullptr;
  Bluestein blue;
  StreamBuf b_in, b_out;
  int b_chunk = 0;
  // notches
  NotchDev *d_notch = nullptr;
  int n_notch = 0;
  int notch_sequential = 0;
};

// the specialised kernels of a master's pair; f: 0 float input, 1 int16, 2 int16 with de-randomisation or statistics
using ColsR36Fn = void (*)(Pass1Args, ColsR36Tables);
using ColsR36TmaFn = void (*)(Pass1Args, ColsR36Tables, CUtensorMap);
using Cols2sFn = void (*)(Pass1Args, Cols2sTables);
using RowsV2Fn = void (*)(Pass2Args, FwdTables);
using Cols2s = Cols2sShape<25, 32>;
using Rows2s = Rows2sShape<25, 25>;
static ColsR36Fn cols_r36_kernel(kgpu_master const *m, int f) {
  static ColsR36Fn const k[2][3] = {{fwd_cols_r36<0, 0>, fwd_cols_r36<1, 0>, fwd_cols_r36<2, 0>},
                                    {fwd_cols_r36<0, 1250>, fwd_cols_r36<1, 1250>, fwd_cols_r36<2, 1250>}};
  return k[m->n2c == 1250][f];
}
static ColsR36TmaFn cols_r36_tma_kernel(kgpu_master const *m, int f) {
  static ColsR36TmaFn const k[2][3] = {{fwd_cols_r36_tma<0, 0>, fwd_cols_r36_tma<1, 0>, fwd_cols_r36_tma<2, 0>},
                                       {fwd_cols_r36_tma<0, 1250>, fwd_cols_r36_tma<1, 1250>, fwd_cols_r36_tma<2, 1250>}};
  return k[m->n2c == 1250][f];
}
static Cols2sFn cols_2s_kernel(int f) {
  static Cols2sFn const k[3] = {fwd_cols_2s<0, 25, 32>, fwd_cols_2s<1, 25, 32>, fwd_cols_2s<2, 25, 32>};
  return k[f];
}
static RowsV2Fn rows_v2_kernel(kgpu_master const *m) {
  if (m->in_type == KGPU_REAL) return m->halved ? fwd_rows_v2<true, 1296, true> : fwd_rows_v2<true, 0, false>;
  return m->n1c ? fwd_rows_v2<false, 1296, false> : fwd_rows_v2<false, 0, false>;
}
// Whether a master's pair can run as one launch (fwd_fused.cuh): REAL with the 1296 x 1250 pair and the real split's 1/2
// folded into the column pass.  The input decides the rest (fused_fits).
static bool fused_pair(kgpu_master const *m) {
  return m->in_type == KGPU_REAL && m->cols == COLS_R36 && m->rows == ROWS_V2 && m->halved && m->n2c == FusedShape::N2 &&
         m->n1c == FusedShape::N1 && m->mid_ld % 16 == 0;
}
using FusedFn = void (*)(Pass1Args, ColsR36Tables, Pass2Args, FwdTables, FusedArgs, CUtensorMap);
static FusedFn fused_kernel(int f) {
  static FusedFn const k[3] = {fwd_fused_r36_v2<0>, fwd_fused_r36_v2<1>, fwd_fused_r36_v2<2>};
  return k[f];
}
static int rows_v2_threads(kgpu_master const *m) { return m->in_type == KGPU_REAL ? RowsV2Shape<true>::T : RowsV2Shape<false>::T; }
static size_t rows_v2_smem(kgpu_master const *m) {
  return m->in_type == KGPU_REAL ? RowsV2Shape<true>::smem : RowsV2Shape<false>::smem;
}

static int upload(float2 **d, std::vector<float2> const &v) {
  CUDA_OK(cudaMalloc(d, sizeof(float2) * v.size()));
  CUDA_OK(cudaMemcpy(*d, v.data(), sizeof(float2) * v.size(), cudaMemcpyHostToDevice));
  return 0;
}

// The device step of a Bluestein record: B = DFT_P of the conjugate chirp, computed on the host and uploaded to b->d_b
// (nothing stays allocated on failure).
static int bluestein_upload(Bluestein *b) {
  if (upload(&b->d_b, bluestein_bspec(b->n, b->P)) == 0) return 0;
  cudaFree(b->d_b);
  b->d_b = nullptr;
  return -1;
}

// A master's outer geometry: what it takes in and the spectrum it writes, whichever transform computes it.
static void master_geometry(kgpu_master *m, int L, int M, int in_type) {
  m->L = L;
  m->M = M;
  m->N = L + M - 1;
  m->in_type = in_type;
  m->bins = (in_type == KGPU_COMPLEX) ? m->N : m->N / 2 + 1;
  m->nc = (in_type == KGPU_COMPLEX) ? m->N : m->N / 2;
  m->spec_stride = ((long)m->bins + 3) / 4 * 4;
}

// The part of a master that needs no device: geometry, shared-memory sizes, the kernel pair and its launch shape.
// kgpu_master_create(_ex) and the host-only kgpu_master_plan share it, so the plan describes what creation builds.
static void master_shape(kgpu_master *m, int L, int M, int in_type, Split2 const &sp, bool ext) {
  master_geometry(m, L, M, in_type);
  m->sp = sp;
  m->ext = ext;
  m->pitch1 = column_pitch(sp.n1);
  m->pitch2 = column_pitch(sp.n2);
  int const nit = (sp.n1 + 31) / 32;
  m->smem1 = sizeof(float2) * ((size_t)kTile * m->pitch1 + (size_t)kTile * nit);
  m->smem2 = sizeof(float2) * ((size_t)kTile * m->pitch2);
  int const n1 = sp.n1, n2 = sp.n2;
  bool const real = in_type == KGPU_REAL;
  if (ext) {  // the extended generic pair only
    m->mid_ld = n2;
    m->n_item_ctas = m->n_rows_ctas = real ? (n1 / 2 + 1 + 3) / 4 : (n1 + 7) / 8;
    return;
  }
  if (!real && n1 == 800 && n2 == 625) {
    m->cols = COLS_2S;
    m->rows = ROWS_2S;
  } else {
    if (n1 == 1296) m->cols = COLS_R36, m->n2c = (n2 == 1250) ? 1250 : 0;
    if (n2 == 1250) m->rows = ROWS_V2, m->n1c = (n1 == 1296) ? 1296 : 0;
  }
  m->halved = real && m->cols == COLS_R36 && m->rows == ROWS_V2;
  bool const padded = m->cols == COLS_2S || (m->cols == COLS_R36 && m->rows == ROWS_V2);  // both kernels know the pitch
  m->mid_ld = padded ? (n2 + 15) / 16 * 16 : n2;
  m->n_item_ctas = real ? (n1 / 2 + 1 + 3) / 4 : (n1 + 7) / 8;
  int const ipc = m->rows == ROWS_V2 ? (real ? RowsV2Shape<true>::IPC : RowsV2Shape<false>::IPC) : 0;
  m->n_rows_ctas = ipc ? ((real ? n1 / 2 + 1 : n1) + ipc - 1) / ipc : m->rows == ROWS_2S ? (n1 + 7) / 8 : m->n_item_ctas;
}

// tables and shared-memory limits of a master whose shape and plans are set
static int master_setup(kgpu_master *m) {
  int const n1 = m->sp.n1, n2 = m->sp.n2;
  bool const real = m->in_type == KGPU_REAL;
  auto root = [](long e, long n) {
    long double const ang = -2.0L * M_PIl * (long double)(e % n) / (long double)n;
    return make_float2((float)cosl(ang), (float)sinl(ang));
  };
  if (real) {
    std::vector<float2> rootD((size_t)n2);
    for (int k2 = 0; k2 < n2; k2++) {
      long double const ang = -M_PIl * (long double)k2 / (long double)n2;
      rootD[(size_t)k2] = make_float2((float)cosl(ang), (float)sinl(ang));
    }
    if (upload(&m->d_rootD, rootD)) return -1;
  }
  if (real && m->rows == ROWS_V2) {
    std::vector<float2> tC((size_t)n1 / 2 + 1);
    for (int k1 = 0; k1 <= n1 / 2; k1++) tC[(size_t)k1] = root(k1, 2 * m->nc);
    if (upload(&m->d_rootC, tC)) return -1;
  }
  if (m->cols == COLS_R36) {  // stage-0 powers, inter-pass factors A[n2][t] and the ten powers of W_nc^{36 n2}
    static int const kPow[10] = {1, 2, 3, 4, 5, 6, 12, 18, 24, 30};
    std::vector<float2> t0(360), tA((size_t)n2 * 36), tB((size_t)(n2 + 8) * 10, make_float2(0.f, 0.f));
    for (int e = 0; e < 10; e++)
      for (int j = 0; j < 36; j++) t0[(size_t)e * 36 + j] = root((long)j * kPow[e], 1296);
    for (long c = 0; c < n2; c++) {
      for (int t = 0; t < 36; t++) tA[(size_t)c * 36 + t] = root(c * t, m->nc);
      for (int e = 0; e < 10; e++) tB[(size_t)c * 10 + e] = root(c * 36 * kPow[e], m->nc);
    }
    if (upload(&m->d_tw0, t0) || upload(&m->d_twA, tA) || upload(&m->d_twB, tB)) return -1;
    for (int f = 0; f < 3; f++)
      if (allow_smem((const void *)cols_r36_kernel(m, f), ColsR36Shape::smem) ||
          allow_smem((const void *)cols_r36_tma_kernel(m, f), ColsR36Shape::smem))
        return -1;
  }
  if (m->cols == COLS_2S) {  // (25 x 32) x (25 x 25)
    constexpr int RA = 25, RB = 32, RC = 25, RD = 25;
    std::vector<float2> t0((size_t)Cols2s::TW0, make_float2(0.f, 0.f)), tA((size_t)n2 * RA),
        tB((size_t)(n2 + 8) * Cols2s::NP1, make_float2(0.f, 0.f)), r0((size_t)Rows2s::TW0, make_float2(0.f, 0.f));
    for (int e = 0; e < Cols2s::NP0; e++)
      for (int j = 0; j < RB; j++) t0[(size_t)e * RB + j] = root((long)j * Pow<RA>::exponent(e), n1);
    for (long c = 0; c < n2; c++) {
      for (int t = 0; t < RA; t++) tA[(size_t)c * RA + t] = root(c * t, m->nc);
      for (int e = 0; e < Cols2s::NP1; e++) tB[(size_t)c * Cols2s::NP1 + e] = root(c * RA * Pow<RB>::exponent(e), m->nc);
    }
    for (int e = 0; e < Rows2s::NP0; e++)
      for (int j = 0; j < RD; j++) r0[(size_t)e * RD + j] = root((long)j * Pow<RC>::exponent(e), n2);
    if (upload(&m->d_tw0, t0) || upload(&m->d_twA, tA) || upload(&m->d_twB, tB) || upload(&m->d_rtw0, r0)) return -1;
    for (int f = 0; f < 3; f++)
      if (allow_smem((const void *)cols_2s_kernel(f), Cols2s::smem)) return -1;
    if (allow_smem((const void *)fwd_rows_2s<25, 25>, Rows2s::smem)) return -1;
  }
  if (m->rows == ROWS_V2 && allow_smem((const void *)rows_v2_kernel(m), rows_v2_smem(m))) return -1;
  if (fused_pair(m))
    for (int f = 0; f < 3; f++)
      if (allow_smem((const void *)fused_kernel(f), FusedShape::smem)) return -1;
  // an extended master runs the extended pair; the generic pair can run for every other one (kgpu_use_static_kernels(0))
  if (m->ext) {
    if (allow_smem((const void *)fwd_cols_ext<0>, m->smem1) || allow_smem((const void *)fwd_cols_ext<1>, m->smem1) ||
        allow_smem((const void *)fwd_rows_ext, m->smem2))
      return -1;
  } else if (allow_smem((const void *)fwd_cols_kernel<0>, m->smem1) || allow_smem((const void *)fwd_cols_kernel<1>, m->smem1) ||
             allow_smem((const void *)fwd_rows_kernel, m->smem2)) {
    return -1;
  }
  return 0;
}

extern "C" void kgpu_master_destroy(kgpu_master *m) {
  if (!m) return;
  if (m->ext) {
    free_tile_plan(m->xplan1);
    free_tile_plan(m->xplan2);
  }
  cudaFree(m->d_rootD);
  cudaFree(m->d_rootC);
  cudaFree(m->d_tw0);
  cudaFree(m->d_twA);
  cudaFree(m->d_twB);
  cudaFree(m->d_rtw0);
  cudaFree(m->mid.p);
  cudaFree(m->fused_ctr.p);
  cudaFree(m->d_notch);
  kgpu_master_destroy(m->bs);
  cudaFree(m->blue.d_b);
  cudaFree(m->b_in.p);
  cudaFree(m->b_out.p);
  delete m;
}
extern "C" int kgpu_master_points(kgpu_master const *m) { return m ? m->N : -1; }
extern "C" int kgpu_master_bins(kgpu_master const *m) { return m ? m->bins : -1; }
extern "C" long kgpu_master_spec_stride(kgpu_master const *m) { return m ? m->spec_stride : -1; }

// What kgpu_master_describe prints for a master of this shape (master_shape: no device state is read).  The radices
// are the planner's, which are what the tile plans of the generic kernels hold.
static std::string describe_text(kgpu_master const *m) {
  auto radices = [](std::vector<int> const &v) {
    std::string r;
    for (size_t i = 0; i < v.size(); i++) r += std::to_string(v[i]) + (i + 1 < v.size() ? "," : "");
    return r;
  };
  auto plan_of = [m](int len) { return m->ext ? choose_radices_ext(len) : choose_radices(len); };
  std::string const rc = m->cols == COLS_2S ? "25,32" : m->cols == COLS_R36 ? "36,36" : radices(plan_of(m->sp.n1));
  std::string const rr = m->rows == ROWS_2S ? "25,25" : m->rows == ROWS_V2 ? "10,25,5" : radices(plan_of(m->sp.n2));
  size_t const s1 = m->cols == COLS_2S ? Cols2s::smem : m->cols == COLS_R36 ? ColsR36Shape::smem : m->smem1;
  size_t const s2 = m->rows == ROWS_2S ? Rows2s::smem : m->rows == ROWS_V2 ? rows_v2_smem(m) : m->smem2;
  char const *kc = m->ext ? "fwd_cols_ext" : m->cols == COLS_2S ? "fwd_cols_2s" : m->cols == COLS_R36 ? "fwd_cols_r36" : "fwd_cols_kernel";
  char const *kr = m->ext ? "fwd_rows_ext" : m->rows == ROWS_2S ? "fwd_rows_2s" : m->rows == ROWS_V2 ? "fwd_rows_v2" : "fwd_rows_kernel";
  char buf[512];
  snprintf(buf, sizeof buf, "N=%d %s, %ld-point complex two-pass %d x %d; cols radices [%s] rows radices [%s]; smem %zu/%zu B; "
           "grids %d/%d CTAs per block; kernels %s + %s", m->N, m->in_type == KGPU_REAL ? "real" : "complex", m->nc, m->sp.n1,
           m->sp.n2, rc.c_str(), rr.c_str(), s1, s2, (m->sp.n2 + kTile - 1) / kTile, m->n_rows_ctas, kc, kr);
  return buf;
}
// A Bluestein transform: its internal master's description from the transform on, then the kernels around it (`in` and
// `out`, the master's or the channels').
static std::string bluestein_text(Bluestein const &b, char const *in, char const *out) {
  kgpu_master inner;
  master_shape(&inner, (int)b.P, 1, KGPU_COMPLEX, b.sp, false);
  std::string const t = describe_text(&inner);
  return t.substr(t.find(", ") + 2) + " around " + in + ", bluestein_mul_kernel, " + out;
}
// A Bluestein master: its own length, then bluestein_text.
static std::string describe_bluestein(int N, int in_type, Bluestein const &b) {
  return "N=" + std::to_string(N) + (in_type == KGPU_REAL ? " real" : " complex") + ", bluestein P=" + std::to_string(b.P) +
         ": " + bluestein_text(b, "bluestein_in_kernel", "bluestein_out_kernel");
}

extern "C" int kgpu_master_describe(kgpu_master const *m, char *buf, int buflen) {
  if (!m || !buf) return -1;
  std::string const t = m->bs ? describe_bluestein(m->N, m->in_type, m->blue) : describe_text(m);
  snprintf(buf, (size_t)buflen, "%s", t.c_str());
  return 0;
}

// ---- the path of a master, chosen from L, M and the input type alone ----
// Bound on each of a Bluestein master's scratch buffers (the chirped input, the passes' spectra, and the internal
// master's inter-pass buffer), as the bank bounds its huge-channel scratch: longer launches run in chunks of blocks.
static constexpr long kBluesteinScratchCap = 128L << 20;
enum MasterPath { MP_DIRECT = 0, MP_EXTENDED = 1, MP_BLUESTEIN = 2 };
struct MasterPlan {
  MasterPath path;
  long nc;
  Split2 sp;       // direct, extended: the split of nc
  Bluestein blue;  // Bluestein: its shape
};
#define KGPU_EXT_FACTORS "2, 3, 5, 7, 11, 13, 17, 19, 23"
// The one place a master's path is decided: the direct pair for a 7-smooth length whose split fits shared memory, else
// the extended pair for a 23-smooth one, else a Bluestein transform; the first of them at or below `ceiling`, the highest
// path the caller serves (kgpu_master_create: direct, _ex: extended, _any and kgpu_master_plan: Bluestein).  `who` names
// the caller in its messages.  A length above the ceiling is refused as kgpu_master_create words it for a 7-smooth
// length and as kgpu_master_create_ex words it for any other.
static int master_plan(int L, int M, int in_type, MasterPath ceiling, char const *who, MasterPlan *pl) {
  if (L < 1 || M < 1 || (in_type != KGPU_REAL && in_type != KGPU_COMPLEX))
    return fail("%s: bad arguments L=%d M=%d type=%d", who, L, M, in_type);
  long const N = (long)L + M - 1;
  if (N > INT32_MAX) return fail("%s: N=L+M-1 is too large (L=%d M=%d)", who, L, M);
  if (in_type == KGPU_REAL && ((N & 1) || (L & 1)))
    return fail("%s: REAL input needs even L and even N=L+M-1 (got L=%d N=%ld)", who, L, N);
  long const nc = (in_type == KGPU_COMPLEX) ? N : N / 2;
  pl->nc = nc;
  if (smooth7(nc) && forward_split(nc, false, &pl->sp)) {
    pl->path = MP_DIRECT;
    return 0;
  }
  if (ceiling >= MP_EXTENDED && smooth23(nc) && forward_split(nc, true, &pl->sp)) {
    pl->path = MP_EXTENDED;
    return 0;
  }
  if (ceiling == MP_BLUESTEIN) {
    if (bluestein_shape(nc, &pl->blue)) {
      pl->path = MP_BLUESTEIN;
      return 0;
    }
    return fail("%s: %ld points need a Bluestein transform of at least %ld points, more than the forward pair splits (at "
                "most 3500 x 3500)", who, nc, 2 * nc - 1);
  }
  bool const ext = ceiling == MP_EXTENDED && !smooth7(nc);
  char const *const name = ext ? "kgpu_master_create_ex" : "kgpu_master_create";
  char const *const factors = ext ? KGPU_EXT_FACTORS : "2,3,5,7";
  if (ext) {
    long rest = nc;
    for (long p : {2, 3, 5, 7, 11, 13, 17, 19, 23})
      while (rest % p == 0) rest /= p;
    if (rest != 1) {
      long q = 29;  // the smallest prime factor left
      while (q * q <= rest && rest % q) q++;
      if (rest % q) q = rest;
      return fail("%s: %ld points have the prime factor %ld (accepted factors %s)", name, nc, q, factors);
    }
  }
  Split2 sp;
  if (!(ext ? choose_split_ext(nc, &sp) : choose_split(nc, &sp)))
    return fail("%s: %ld points cannot be split into two plannable lengths (factors %s; <= %d)", name, nc, factors, kMaxTileLen);
  kgpu_master m;
  master_shape(&m, L, M, in_type, sp, ext);
  return fail("%s: %ld points split as %d x %d, which needs %zu / %zu B of shared memory (at most %d; factors %s)", name, nc,
              sp.n1, sp.n2, m.smem1, m.smem2, kChanSmemLimit, factors);
}

// The master master_plan chooses, built.  An extended master keeps its two plans out of the registry, which keeps room
// for every length a 7-smooth master or channel can ask for.
static kgpu_master *master_create(int L, int M, int in_type, MasterPath ceiling, char const *who) {
  MasterPlan pl;
  if (master_plan(L, M, in_type, ceiling, who, &pl)) return nullptr;
  kgpu_master *m = new kgpu_master;
  bool ok;
  if (pl.path == MP_BLUESTEIN) {
    master_geometry(m, L, M, in_type);
    m->blue = pl.blue;
    m->b_chunk = (int)std::max(1L, kBluesteinScratchCap / (long)(sizeof(float2) * (size_t)(pl.blue.P + 3)));
    m->bs = kgpu_master_create((int)pl.blue.P, 1, KGPU_COMPLEX);
    ok = m->bs && bluestein_upload(&m->blue) == 0;
  } else {
    master_shape(m, L, M, in_type, pl.sp, pl.path == MP_EXTENDED);
    if (m->ext) {
      m->plan1 = m->plan2 = -1;
      ok = make_tile_plan(pl.sp.n1, choose_radices_ext(pl.sp.n1), m->xplan1) == 0 &&
           make_tile_plan(pl.sp.n2, choose_radices_ext(pl.sp.n2), m->xplan2) == 0;
    } else {
      m->plan1 = get_tile_plan(pl.sp.n1);
      m->plan2 = get_tile_plan(pl.sp.n2);
      ok = m->plan1 >= 0 && m->plan2 >= 0;
    }
    ok = ok && master_setup(m) == 0;
  }
  if (!ok) {
    fail("%s: %s", who, std::string(g_err).c_str());
    kgpu_master_destroy(m);
    return nullptr;
  }
  return m;
}

extern "C" kgpu_master *kgpu_master_create(int L, int M, int in_type) {
  return master_create(L, M, in_type, MP_DIRECT, "kgpu_master_create");
}
// kgpu_master_create for transform lengths whose prime factors go up to 23.  A length with factors 2, 3, 5, 7 only
// gets exactly kgpu_master_create's master; any other the extended generic pair.
extern "C" kgpu_master *kgpu_master_create_ex(int L, int M, int in_type) {
  return master_create(L, M, in_type, MP_EXTENDED, "kgpu_master_create_ex");
}
// Any length: kgpu_master_create_ex's master wherever that succeeds, a Bluestein transform otherwise.
extern "C" kgpu_master *kgpu_master_create_any(int L, int M, int in_type) {
  return master_create(L, M, in_type, MP_BLUESTEIN, "kgpu_master_create_any");
}

extern "C" int kgpu_master_plan(int L, int M, int in_type, char *buf, int buflen) {
  MasterPlan pl;
  if (master_plan(L, M, in_type, MP_BLUESTEIN, "kgpu_master_plan", &pl)) return -1;
  if (buf && buflen > 0) {
    std::string t;
    if (pl.path == MP_BLUESTEIN) {
      t = describe_bluestein(L + M - 1, in_type, pl.blue);
    } else {
      kgpu_master m;
      master_shape(&m, L, M, in_type, pl.sp, pl.path == MP_EXTENDED);
      t = describe_text(&m);
    }
    snprintf(buf, (size_t)buflen, "%s", t.c_str());
  }
  return (int)pl.path;
}

// Whether fwd_cols_r36 can take its raw tile by tensor copies (fwd_cols_r36.cuh): a tensor map needs a 16-byte aligned
// base and strides that are multiples of 16 bytes.  Its rows are n2 points apart (8 n2 bytes: a row of floats, or a pair of
// int16 rows, which also needs n1 even) and its windows hop points apart.  Any other input runs the global-load form.
static bool cols_tma_fits(kgpu_master const *m, void const *d_in, int fmt) {
  long const point = fmt == KGPU_FMT_I16 ? 4 : 8;  // bytes of a complex input point
  long const hop = m->in_type == KGPU_REAL ? m->L / 2 : m->L;
  return m->cols == COLS_R36 && (uintptr_t)d_in % 16 == 0 && hop * point % 16 == 0 && 8L * m->sp.n2 % 16 == 0 &&
         m->sp.n1 % 2 == 0;
}

extern "C" int kgpu_cols_tma_fits(int L, int M, int in_type, int fmt, const void *d_in) {
  MasterPlan pl;
  if (master_plan(L, M, in_type, MP_BLUESTEIN, "kgpu_cols_tma_fits", &pl)) return -1;
  if (pl.path != MP_DIRECT) return 0;
  kgpu_master m;
  master_shape(&m, L, M, in_type, pl.sp, false);
  return cols_tma_fits(&m, d_in, fmt) ? 1 : 0;
}

// Whether both passes run as one launch (fwd_fused.cuh): a master whose pair allows it and an input the column pass can
// take by tensor copies.
static bool fused_fits(kgpu_master const *m, void const *d_in, int fmt) { return fused_pair(m) && cols_tma_fits(m, d_in, fmt); }

extern "C" int kgpu_fused_forward_fits(int L, int M, int in_type, int fmt, const void *d_in) {
  MasterPlan pl;
  if (master_plan(L, M, in_type, MP_BLUESTEIN, "kgpu_fused_forward_fits", &pl)) return -1;
  if (pl.path != MP_DIRECT) return 0;
  kgpu_master m;
  master_shape(&m, L, M, in_type, pl.sp, false);
  return fused_fits(&m, d_in, fmt) ? 1 : 0;
}

extern "C" int kgpu_fused_forward_options(int lead, int discard) {
  if (lead < 0 || lead > FusedShape::NC) return fail("kgpu_fused_forward_options: lead %d outside 0..%d", lead, FusedShape::NC);
  g_fused_lead.store(lead);
  g_fused_discard.store(discard != 0);
  return 0;
}

extern "C" int kgpu_fused_shape(int *out) {
  if (!out) return fail("kgpu_fused_shape: bad arguments");
  out[0] = FusedShape::NC;
  out[1] = FusedShape::NR;
  out[2] = FusedShape::N1;
  out[3] = (FusedShape::N2 + 15) / 16 * 16;
  out[4] = FusedShape::DEFAULT_LEAD;
  return 0;
}

extern "C" int kgpu_fused_schedule(int nblocks, int lead, int ticket, int *out) {
  if (nblocks < 1 || lead < 0 || lead > FusedShape::NC || ticket < 0 || ticket >= nblocks * (FusedShape::NC + FusedShape::NR) ||
      !out)
    return fail("kgpu_fused_schedule: bad arguments");
  FusedItem const it = fused_item(ticket, nblocks, lead);
  out[0] = it.kind;
  out[1] = it.blk;
  out[2] = it.idx;
  out[3] = it.kind == kFusedRow ? it.blk : -1;  // the done counter it waits on, and for what count
  out[4] = it.kind == kFusedRow ? FusedShape::NC : 0;
  return 0;
}

extern "C" long kgpu_fused_discards(int blk, int idx, long *lines, long max) {
  using S = RowsV2Shape<true>;
  if (blk < 0 || idx < 0 || idx >= FusedShape::NR || max < 0) return fail("kgpu_fused_discards: bad arguments");
  int const ld = (FusedShape::N2 + 15) / 16 * 16;
  long n = 0;
  for (int col = 0; col < S::COLS; col++) {  // the rows fwd_rows_v2_body's tile columns hold
    RowItem const it = row_item(idx * S::IPC + (col >> 1), FusedShape::N1, true);
    int const row = (col & 1) == 0 ? (it.kind != kRowEmpty ? it.row_a : -1) : (it.kind == kRowPair ? it.row_b : -1);
    if (row < 0) continue;
    for (int l = 0; l < mid_row_lines(ld); l++, n++)
      if (lines && n < max) lines[n] = mid_line(blk, FusedShape::N1, row, ld, l);
  }
  return n;
}

// The tensor map of the windows of `nblocks` blocks from d_in that fwd_cols_r36_tma reads, for a master and input that
// cols_tma_fits accepts.  L2 fills in 128-byte pieces: on H100 the column pass took 7.9 us per cfg-2 block so, 8.1 with
// 256-byte pieces and 8.2 without promotion (int16, tools/cols_tma_ab.py).
static int cols_tma_map(kgpu_master const *m, void const *d_in, int fmt, int nblocks, CUtensorMap *map) {
  static PFN_cuTensorMapEncodeTiled const encode = [] {
    void *fn = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q) != cudaSuccess ||
        q != cudaDriverEntryPointSuccess)
      fn = nullptr;
    return (PFN_cuTensorMapEncodeTiled)fn;
  }();
  if (!encode) return fail("kgpu_forward: the driver has no cuTensorMapEncodeTiled");
  bool const i16 = fmt == KGPU_FMT_I16;
  cuuint64_t const n1 = (cuuint64_t)m->sp.n1, n2 = (cuuint64_t)m->sp.n2;
  cuuint64_t const hop = (cuuint64_t)(m->in_type == KGPU_REAL ? m->L / 2 : m->L);
  cuuint64_t const dim[3] = {2 * n2, i16 ? n1 / 2 : n1, (cuuint64_t)nblocks};
  cuuint64_t const stride[2] = {8 * n2, hop * (i16 ? 4 : 8)};
  cuuint32_t const box[3] = {(cuuint32_t)(i16 ? ColsR36Tma::I16_BOX_WORDS : 16), ColsR36Tma::BOX_ROWS, 1};
  cuuint32_t const unit[3] = {1, 1, 1};
  CUresult const r = encode(map, i16 ? CU_TENSOR_MAP_DATA_TYPE_UINT32 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, const_cast<void *>(d_in),
                            dim, stride, box, unit, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
                            CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail("kgpu_forward: cuTensorMapEncodeTiled failed (%d)", (int)r);
  return 0;
}

// The Pass2Args of the row pass, for the Pass1Args a1 of the same launch
static Pass2Args rows_args(kgpu_master const *m, Pass1Args const &a1, void *d_spec) {
  Pass2Args a2;
  a2.mid = a1.mid;
  a2.n1 = m->sp.n1;
  a2.n2 = m->sp.n2;
  a2.nc = m->nc;
  a2.plan = m->plan2;
  a2.pitch = m->pitch2;
  a2.real_split = (m->in_type == KGPU_REAL);
  a2.rootD = m->d_rootD;
  a2.spec = (float2 *)d_spec;
  a2.spec_stride = m->spec_stride;
  a2.mid_ld = a1.mid_ld;
  return a2;
}

// Both passes over `nblocks` blocks as one launch of fwd_fused_r36_v2, for a master and input fused_fits accepts.
static int fused_span(kgpu_master *m, const void *d_in, int fmt, int f, int nblocks, void *d_spec, cudaStream_t st,
                      Pass1Args const &a1) {
  using F = FusedShape;
  size_t const ctr_bytes = sizeof(unsigned) * (size_t)(1 + nblocks);
  if (grow(m->fused_ctr, ctr_bytes, st, "kgpu_forward")) return -1;
  CUtensorMap map;
  if (cols_tma_map(m, d_in, fmt, nblocks, &map)) return -1;
  FusedArgs fa;
  fa.ctr = (unsigned *)m->fused_ctr.p;
  fa.nblocks = nblocks;
  fa.lead = g_fused_lead.load();
  fa.discard = g_fused_discard.load();
  CUDA_OK(cudaMemsetAsync(fa.ctr, 0, ctr_bytes, st));
  {
    ProfScope ps(K_FWD_FUSED, st);
    fused_kernel(f)<<<(unsigned)(nblocks * (F::NC + F::NR)), F::T, F::smem, st>>>(a1, ColsR36Tables{m->d_tw0, m->d_twA, m->d_twB},
                                                                       rows_args(m, a1, d_spec), FwdTables{m->d_rootC}, fa, map);
  }
  g_launches++;
  CUDA_OK(cudaGetLastError());
  return 0;
}

// One launch pair (column pass, row pass) over `nblocks` consecutive blocks on stream `st`, inter-pass data in `mid`.
static int forward_span(kgpu_master *m, const void *d_in, int fmt, float scale, int derandomize, int nblocks, void *d_spec,
                        void *d_stats, cudaStream_t st, float2 *mid) {
  bool const use_static = g_static_on.load() != 0;
  ColsKernel const cols = use_static ? m->cols : COLS_GENERIC;
  RowsKernel const rows = use_static ? m->rows : ROWS_GENERIC;
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
  // the specialised column kernels take the int16 scale (and the folded 1/2) on the inter-pass twiddle
  a1.out_scale = (fmt == KGPU_FMT_I16 ? scale : 1.0f) * (m->halved ? 0.5f : 1.0f);
  a1.mid_ld = use_static ? m->mid_ld : m->sp.n2;
  int const f = (fmt != KGPU_FMT_I16) ? 0 : ((derandomize || a1.stats) ? 2 : 1);
  // one block has nothing to overlap: its row items could only wait for its column items, so it runs the pair
  if (nblocks >= 2 && use_static && cols_tma_on() && fused_on() && fused_fits(m, d_in, fmt)) return fused_span(m, d_in, fmt, f, nblocks, d_spec, st, a1);
  dim3 const g1((unsigned)((m->sp.n2 + kTile - 1) / kTile), (unsigned)nblocks);
  {
    ProfScope ps(K_FWD_COLS, st);
    switch (cols) {
      case COLS_2S:
        cols_2s_kernel(f)<<<g1, Cols2s::T, Cols2s::smem, st>>>(a1, Cols2sTables{m->d_tw0, m->d_twA, m->d_twB});
        break;
      case COLS_R36:
        if (cols_tma_on() && cols_tma_fits(m, d_in, fmt)) {
          CUtensorMap map;
          if (cols_tma_map(m, d_in, fmt, nblocks, &map)) return -1;
          cols_r36_tma_kernel(m, f)<<<g1, ColsR36Shape::T, ColsR36Shape::smem, st>>>(a1, ColsR36Tables{m->d_tw0, m->d_twA, m->d_twB}, map);
        } else {
          cols_r36_kernel(m, f)<<<g1, ColsR36Shape::T, ColsR36Shape::smem, st>>>(a1, ColsR36Tables{m->d_tw0, m->d_twA, m->d_twB});
        }
        break;
      case COLS_GENERIC:
        if (m->ext && f) fwd_cols_ext<1><<<g1, kFwdThreads, m->smem1, st>>>(a1, m->xplan1);
        else if (m->ext) fwd_cols_ext<0><<<g1, kFwdThreads, m->smem1, st>>>(a1, m->xplan1);
        else if (f) fwd_cols_kernel<1><<<g1, kFwdThreads, m->smem1, st>>>(a1);
        else fwd_cols_kernel<0><<<g1, kFwdThreads, m->smem1, st>>>(a1);
        break;
    }
  }
  g_launches++;
  Pass2Args const a2 = rows_args(m, a1, d_spec);
  dim3 const g2((unsigned)(rows == ROWS_GENERIC ? m->n_item_ctas : m->n_rows_ctas), (unsigned)nblocks);
  {
    ProfScope ps(K_FWD_ROWS, st);
    switch (rows) {
      case ROWS_2S:
        fwd_rows_2s<25, 25><<<g2, Rows2s::T, Rows2s::smem, st>>>(a2, m->d_rtw0);
        break;
      case ROWS_V2:
        rows_v2_kernel(m)<<<g2, rows_v2_threads(m), rows_v2_smem(m), st>>>(a2, FwdTables{m->d_rootC});
        break;
      case ROWS_GENERIC:
        if (m->ext) fwd_rows_ext<<<g2, kFwdThreads, m->smem2, st>>>(a2, m->xplan2);
        else fwd_rows_kernel<<<g2, kFwdThreads, m->smem2, st>>>(a2);
        break;
    }
  }
  g_launches++;
  CUDA_OK(cudaGetLastError());
  return 0;
}

// The convolution of every Bluestein transform, over `rows` rows on stream st: A = DFT_P(a) of the chirped input a
// ([rows][P]) into y ([rows][im->spec_stride]), conj(A B) back into a, then y = DFT_P(conj(A B)).  im: the internal
// master, a COMPLEX master of length b.P.
static int bluestein_conv(kgpu_master *im, Bluestein const &b, float2 *a, int rows, float2 *y, cudaStream_t st) {
  if (kgpu_forward(im, a, KGPU_FMT_F32, 1.0f, 0, rows, y, nullptr, st) != 0) return -1;
  {
    ProfScope ps(K_FWD_COLS, st);
    bluestein_mul_kernel<<<dim3((unsigned)((b.P + kBluesteinThreads - 1) / kBluesteinThreads), (unsigned)rows), kBluesteinThreads, 0,
                           st>>>(y, im->spec_stride, b.d_b, (int)b.P, a);
  }
  g_launches++;
  return kgpu_forward(im, a, KGPU_FMT_F32, 1.0f, 0, rows, y, nullptr, st);
}

// A forward Bluestein transform of b.n points over a.nblocks blocks (bluestein_master.cuh): bluestein_in_kernel into
// bin ([nblocks][P]), the convolution into bout ([nblocks][im->spec_stride]), bluestein_out_kernel.  The caller sets
// a's input fields and o's output fields; the transform's own are set here.
static int bluestein_chain(kgpu_master *im, Bluestein const &b, BluesteinInArgs a, BluesteinOutArgs o, float2 *bin, float2 *bout,
                           cudaStream_t st) {
  a.nc = o.nc = b.n;
  a.P = b.P;
  a.out = bin;
  o.y = bout;
  o.y_stride = im->spec_stride;
  o.inv_p = 1.0 / (double)b.P;
  o.nblocks = a.nblocks;
  long const bins = o.real_split ? b.n + 1 : b.n;
  {
    ProfScope ps(K_FWD_COLS, st);
    bluestein_in_kernel<<<(unsigned)((b.P + kBluesteinThreads - 1) / kBluesteinThreads), kBluesteinThreads, 0, st>>>(a);
  }
  g_launches++;
  if (bluestein_conv(im, b, bin, a.nblocks, bout, st)) return -1;
  {
    ProfScope ps(K_FWD_ROWS, st);
    bluestein_out_kernel<<<(unsigned)((bins + kBluesteinThreads - 1) / kBluesteinThreads), kBluesteinThreads, 0, st>>>(o);
  }
  g_launches++;
  return 0;
}

// kgpu_forward of a Bluestein master, in chunks of at most b_chunk blocks.
static int bluestein_forward(kgpu_master *m, const void *d_in, int fmt, float scale, int derandomize, int nblocks, void *d_spec,
                             void *d_stats, cudaStream_t st) {
  int const chunk = std::min(nblocks, m->b_chunk);
  if (grow(m->b_in, sizeof(float2) * (size_t)m->blue.P * (size_t)chunk, st, "kgpu_forward") ||
      grow(m->b_out, sizeof(float2) * (size_t)m->bs->spec_stride * (size_t)chunk, st, "kgpu_forward"))
    return -1;
  bool const i16 = fmt == KGPU_FMT_I16;
  if (i16 && d_stats) CUDA_OK(cudaMemsetAsync(d_stats, 0, sizeof(IngestStats) * (size_t)nblocks, st));
  bool const real = m->in_type == KGPU_REAL;
  BluesteinInArgs a{};
  a.hop = real ? m->L / 2 : m->L;
  a.first_new = real ? (m->M - 1) / 2 : (m->M - 1);
  a.i16 = i16;
  a.derandomize = i16 && derandomize;
  a.scale = scale;
  BluesteinOutArgs o{};
  o.real_split = real;
  o.spec_stride = m->spec_stride;
  size_t const pair = i16 ? sizeof(short2) : sizeof(float2);
  for (int b0 = 0; b0 < nblocks; b0 += chunk) {
    a.in = (char const *)d_in + pair * (size_t)a.hop * (size_t)b0;
    a.nblocks = std::min(chunk, nblocks - b0);
    a.stats = (i16 && d_stats) ? (IngestStats *)d_stats + b0 : nullptr;
    o.spec = (float2 *)d_spec + (size_t)m->spec_stride * (size_t)b0;
    if (bluestein_chain(m->bs, m->blue, a, o, (float2 *)m->b_in.p, (float2 *)m->b_out.p, st)) return -1;
  }
  CUDA_OK(cudaGetLastError());
  return 0;
}

extern "C" int kgpu_forward(kgpu_master *m, const void *d_in, int fmt, float scale, int derandomize, int nblocks,
                            void *d_spec, void *d_stats, void *stream) {
  if (!m || !d_in || !d_spec || nblocks < 1) return fail("kgpu_forward: bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  if (m->bs) return bluestein_forward(m, d_in, fmt, scale, derandomize, nblocks, d_spec, d_stats, st);
  size_t const mid = sizeof(float2) * (size_t)m->sp.n1 * (size_t)((m->sp.n2 + 15) / 16 * 16);
  if (grow(m->mid, mid * (size_t)nblocks, st, "kgpu_forward")) return -1;
  if (fmt == KGPU_FMT_I16 && d_stats) CUDA_OK(cudaMemsetAsync(d_stats, 0, sizeof(IngestStats) * (size_t)nblocks, st));
  return forward_span(m, d_in, fmt, scale, derandomize, nblocks, d_spec, d_stats, st, (float2 *)m->mid.p);
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
// ---- the path of a channel's inverse transform, chosen from its point count alone ----
//   CP_DIRECT     factors 2, 3, 5, 7, at most kMaxChanPoints: one warp per channel on a registry plan (chan_kernel, or
//                 a specialised kernel of chan_v2 / chan_static)
//   CP_WIDE       factors 2, 3, 5, 7, at most kMaxWideChanPoints: chan_wide, one CTA per channel on a four-step split
//                 into two registry lengths
//   CP_HUGE       factors 2, 3, 5, 7, at most kMaxHugeChanPoints: chan_huge's two passes through the bank's scratch
//   CP_EXTENDED   a prime factor 11 .. 23, at most kMaxWideChanPoints: chan_kernel_ext, or chan_wide_ext above
//                 kMaxChanPoints, on plans outside the registry
//   CP_BLUESTEIN  every other length up to kMaxHugeChanPoints: a Bluestein transform (bluestein_chan.cuh)
// The values are kgpu_chan_plan's.  Each kgpu_bank_define* entry point serves the paths up to its own (its ceiling), and
// kDefineName[path] is the entry point that introduced a path, which names it in messages.
enum ChanPath { CP_DIRECT = 0, CP_WIDE = 1, CP_HUGE = 2, CP_EXTENDED = 3, CP_BLUESTEIN = 4 };
static char const *const kDefineName[] = {"kgpu_bank_define", "kgpu_bank_define_wide", "kgpu_bank_define_huge",
                                          "kgpu_bank_define_ext", "kgpu_bank_define_any"};
struct ChanRoute {
  ChanPath path;
  bool narrow;  // at most kMaxChanPoints: the transform fits one warp (direct, extended; Bluestein only for grouping)
  Split2 sp;       // wide, huge, extended above kMaxChanPoints: the four-step split
  Bluestein blue;  // Bluestein: its shape, and B once chan_geom has built the length's record
};

// The route of a channel of `points` points, without a device.  A length above `ceiling`, or above every path, is
// refused with the message each entry point has always given; `who` names the caller when it is above every path.
static int chan_route(int points, ChanPath ceiling, char const *who, ChanRoute *r) {
  long const big = factor_above7(points);  // 1: factors 2, 3, 5, 7 only
  // the path a 7-smooth length of this size takes
  ChanPath const size = points <= kMaxChanPoints ? CP_DIRECT : points <= kMaxWideChanPoints ? CP_WIDE : CP_HUGE;
  bool const too_long = points > kMaxHugeChanPoints;
  *r = ChanRoute{};
  r->path = big == 1 ? size : (big <= 23 && size != CP_HUGE) ? CP_EXTENDED : CP_BLUESTEIN;
  r->narrow = size == CP_DIRECT;
  if (too_long && ceiling == CP_BLUESTEIN)
    return fail("%s: %d-point inverse transform exceeds the %d-point maximum", who, points, kMaxHugeChanPoints);
  if (r->path == CP_BLUESTEIN && ceiling == CP_EXTENDED) {
    if (big > 23)
      return fail("kgpu_bank_define_ext: %d-point inverse transform has the prime factor %ld (prime factors up to 23 are served)",
                  points, big);
    return fail("kgpu_bank_define_ext: %d-point inverse transform has the prime factor %ld, served up to %d points only",
                points, big, kMaxWideChanPoints);
  }
  if (r->path > ceiling || too_long) {  // a 7-smooth length too long for define_ext gets define_huge's message
    static int const kMaxPoints[] = {kMaxChanPoints, kMaxWideChanPoints, kMaxHugeChanPoints};
    ChanPath const c = std::min(ceiling, CP_HUGE);
    if (size > c || too_long)
      return fail("%s: %d-point inverse transform exceeds the %d-point maximum", kDefineName[c], points, kMaxPoints[c]);
    if (size == CP_DIRECT)
      return fail("kgpu_bank_define: %d-point transform cannot be planned (factors 2, 3, 5, 7; at most %d points)", points,
                  kMaxChanPoints);
    return fail("%s: %d-point transform cannot be split into two plannable lengths (factors 2, 3, 5, 7; each at most %d)",
                kDefineName[size], points, kMaxTileLen);
  }
  // the static_asserts on wide_fits, huge_lengths and ext_lengths pin that every split below exists and fits
  bool ok = true;
  if (r->path == CP_BLUESTEIN) ok = bluestein_shape(points, &r->blue);
  else if (!r->narrow) ok = r->path == CP_EXTENDED ? choose_split_ext(points, &r->sp) : choose_split(points, &r->sp);
  if (!ok) return fail("%s: %d-point transform has no split", who, points);
  return 0;
}

// A channel length's route and the device state its kernels read, per device and length: built by the first
// kgpu_bank_define* of the length, never freed (like the plan registry).  Map nodes are stable, so channels keep a
// pointer.  Bluestein's B is read-only and its host transform takes about 1 s at P = 1.5 M, so it is computed once per
// length, not per channel or bank.  DESIGN.md section 4 states the device memory the extended plans can reach.
struct ChanGeom {
  ChanRoute r;
  int points = 0;
  int plan = -1;          // ChanDesc::plan: the registry plan of the length (direct) or of n1 (wide, huge); kPlanExt,
                          // kPlanBluestein
  WideGeom wide{};        // CP_WIDE
  HugeGeom huge{};        // CP_HUGE (no tables: the kernels compute their twiddles)
  TilePlan ext{};         // CP_EXTENDED, narrow
  WideGeomExt wide_ext{}; // CP_EXTENDED above kMaxChanPoints: chan_wide's split and twiddles, the factor plans by value
};
static std::recursive_mutex g_geom_mu;  // recursive: an extended wide length builds the records of its factors
static std::map<std::pair<int, int>, ChanGeom> g_geom;

static ChanGeom const *chan_geom(int points, ChanRoute const &r);
// The plan of a factor (<= kMaxTileLen) of an extended wide length by value: the registry's for a 7-smooth factor,
// the factor's own extended plan otherwise.
static int factor_plan(int len, TilePlan *out) {
  ChanRoute r;
  if (chan_route(len, CP_EXTENDED, "factor_plan", &r)) return -1;
  ChanGeom const *g = chan_geom(len, r);
  if (!g) return -1;
  if (r.path == CP_EXTENDED) {
    *out = g->ext;
    return 0;
  }
  std::lock_guard<std::mutex> lk(g_plan_mu);
  *out = g_plans[(size_t)g->plan].host;
  return 0;
}

static ChanGeom const *chan_geom(int points, ChanRoute const &r) {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) {
    fail("cudaGetDevice: %s", cudaGetErrorString(cudaGetLastError()));
    return nullptr;
  }
  std::lock_guard<std::recursive_mutex> lk(g_geom_mu);
  auto it = g_geom.find({dev, points});
  if (it != g_geom.end()) return &it->second;
  ChanGeom g;
  g.r = r;
  g.points = points;
  int const n1 = r.sp.n1, n2 = r.sp.n2;
  bool ok = true;
  switch (r.path) {
    case CP_DIRECT:
      g.plan = get_tile_plan(points);
      ok = g.plan >= 0;
      break;
    case CP_WIDE:
      g.wide = WideGeom{n1, n2, wide_pitch(n2), get_tile_plan(n1), get_tile_plan(n2), nullptr};
      ok = g.wide.plan1 >= 0 && g.wide.plan2 >= 0 && !wide_twiddles(g.wide, *host_tile_plan(g.wide.plan2));
      g.plan = g.wide.plan1;
      break;
    case CP_HUGE:
      g.huge = HugeGeom{n1, n2, huge_pitch(n1), huge_pitch(n2), get_tile_plan(n1), get_tile_plan(n2)};
      ok = g.huge.plan1 >= 0 && g.huge.plan2 >= 0;
      g.plan = g.huge.plan1;
      break;
    case CP_EXTENDED:
      g.plan = kPlanExt;
      if (r.narrow) {
        ok = make_tile_plan(points, choose_radices_ext(points), g.ext) == 0;
      } else {
        g.wide_ext.g = WideGeom{n1, n2, wide_pitch(n2), -1, -1, nullptr};
        ok = !factor_plan(n1, &g.wide_ext.p1) && !factor_plan(n2, &g.wide_ext.p2) && !wide_twiddles(g.wide_ext.g, g.wide_ext.p2);
      }
      break;
    case CP_BLUESTEIN:
      g.plan = kPlanBluestein;
      ok = bluestein_upload(&g.r.blue) == 0;
      break;
  }
  if (!ok) return nullptr;
  return &(g_geom[{dev, points}] = g);
}

struct ChanHost {
  bool defined = false, enabled = false, has_response = false;
  bool real_out = false;  // REAL-output slave (filter.c:370-390): olen floats per block
  int olen = 0, points = 0, shift = 0, flags = 0;
  ChanGeom const *geom = nullptr;  // the path and geometry of `points` (set by kgpu_bank_define*)
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
    ChanGeom const *geom;
    int off, count;
    bool generic;  // runtime_plan_only
  };
  std::vector<Group> groups;  // enabled channels grouped by length
  int *d_order = nullptr;
  ChanAux *d_aux = nullptr;   // [capacity]
  int *d_shift = nullptr;     // [capacity] shifts, for the noise estimator
  float2 *d_fm_mem[2] = {nullptr, nullptr};  // [capacity] discriminator phase memory, ping-pong per launch
  int fm_parity = 0;
  std::vector<ChanAux> aux;
  long block_counter = 0;     // index of the next block a run will process (oscillator epoch arithmetic)
  long last_rebase = 0;
  bool any_osc = false;
  // global scratch of the huge channels (chan_huge.cuh) and of noise_kernel_gm, one buffer per stream so that launches
  // on different streams (a batched run and a run_one) never share one; grown on demand, freed in kgpu_bank_destroy
  std::mutex scratch_mu;
  std::map<cudaStream_t, StreamBuf> scratch;
  // the internal COMPLEX masters of the Bluestein channels, by (stream, P): kgpu_forward keeps its inter-pass buffer in
  // the master, so launches on two streams must never share one; created on first use, freed in kgpu_bank_destroy
  std::map<std::pair<cudaStream_t, long>, kgpu_master *> bmaster;
};

// Bound on one launch's huge-channel scratch: chan_huge loops over chunks of channels and blocks to stay below it.
static constexpr long kHugeScratchCap = 128L << 20;
// Bound on the (channel, block) rows of one Bluestein chunk: they are the blocks (grid.y) of one kgpu_forward.
static constexpr long kMaxBluesteinRows = 65535;

// the internal master of length P for the Bluestein channels launched on stream `st` (nullptr and kgpu_last_error())
static kgpu_master *bank_bluestein_master(kgpu_bank *b, cudaStream_t st, long P) {
  std::lock_guard<std::mutex> lk(b->scratch_mu);
  kgpu_master *&m = b->bmaster[{st, P}];
  if (!m) m = kgpu_master_create((int)P, 1, KGPU_COMPLEX);
  return m;
}

// the scratch buffer of stream `st`, at least `bytes` long (nullptr and kgpu_last_error() on failure)
static void *bank_scratch(kgpu_bank *b, cudaStream_t st, size_t bytes) {
  std::lock_guard<std::mutex> lk(b->scratch_mu);
  StreamBuf &s = b->scratch[st];
  return grow(s, bytes, st, "bank scratch") ? nullptr : s.p;
}

// in_type, mb: the master's type and bins
static void resolve_walk(int in_type, int mb, ChanHost const &c, ChanDesc &d) {
  int const ns = c.points, half = ns / 2;
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
  if (in_type == KGPU_REAL) {
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

// REAL-output and beam channels of at most kMaxChanPoints: a direct one is served by the runtime-plan kernel only, and
// the other narrow paths keep them in groups of their own as well.
static bool runtime_plan_only(kgpu_bank const *b, int i) {
  return b->ch[(size_t)i].geom->r.narrow && (b->desc[(size_t)i].flags & (kChanRealOut | kChanBeam)) != 0;
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
      d.plan = c.geom->plan;
      resolve_walk(b->m->in_type, b->m->bins, c, d);
      b->max_points = std::max(b->max_points, c.points);
    }
  }
  b->out_stride = (off + 3) / 4 * 4;
  // one launch per distinct length (and runtime_plan_only flag): order[] lists that group's descriptors
  std::vector<int> order;
  b->groups.clear();
  auto same_group = [&](kgpu_bank::Group const &g, int k) {
    return b->desc[(size_t)k].plan >= 0 && b->ch[(size_t)k].geom == g.geom && runtime_plan_only(b, k) == g.generic;
  };
  for (int i = 0; i < b->nchan; i++) {
    if (b->desc[(size_t)i].plan < 0) continue;
    bool found = false;
    for (auto &g : b->groups)
      if (same_group(g, i)) found = true;
    if (found) continue;
    kgpu_bank::Group g{b->ch[(size_t)i].geom, (int)order.size(), 0, runtime_plan_only(b, i)};
    for (int k = i; k < b->nchan; k++)
      if (same_group(g, k)) order.push_back(k);
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
  for (auto &s : b->scratch) cudaFree(s.second.p);
  for (auto &m : b->bmaster) kgpu_master_destroy(m.second);
  delete b;
}
static bool bad_idx(kgpu_bank const *b, int idx) { return !b || idx < 0 || idx >= b->capacity; }

// Defines channel idx with the path chan_route chooses, if it lies at or below `ceiling`.  who: the entry point.
static int bank_define(char const *who, kgpu_bank *b, int idx, int olen, int out_type, ChanPath ceiling) {
  if (out_type != KGPU_COMPLEX && out_type != KGPU_REAL) return fail("%s: out_type must be KGPU_COMPLEX or KGPU_REAL", who);
  if (bad_idx(b, idx) || olen < 1) return fail("kgpu_bank_define: bad arguments");
  bool const real_out = out_type == KGPU_REAL;
  long const num = (long)olen * b->m->N;
  if (num % b->m->L) return fail("invalid output length %d for N=%d L=%d (filter.c:312-316)", olen, b->m->N, b->m->L);
  int const points = (int)(num / b->m->L);
  if (real_out && (points & 1)) return fail("kgpu_bank_define: REAL-output slaves need an even number of points (got %d)", points);
  ChanRoute r;
  if (chan_route(points, ceiling, who, &r)) return -1;
  ChanGeom const *geom = chan_geom(points, r);
  if (!geom) return fail("%s: %s", kDefineName[r.path], std::string(g_err).c_str());
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
  c.geom = geom;
  b->nchan = std::max(b->nchan, idx + 1);
  b->dirty = true;
  return points;
}
extern "C" int kgpu_bank_define(kgpu_bank *b, int idx, int olen) {
  return bank_define("kgpu_bank_define", b, idx, olen, KGPU_COMPLEX, CP_DIRECT);
}
extern "C" int kgpu_bank_define_ex(kgpu_bank *b, int idx, int olen, int out_type) {
  return bank_define("kgpu_bank_define_ex", b, idx, olen, out_type, CP_DIRECT);
}
extern "C" int kgpu_bank_define_wide(kgpu_bank *b, int idx, int olen, int out_type) {
  return bank_define("kgpu_bank_define_wide", b, idx, olen, out_type, CP_WIDE);
}
extern "C" int kgpu_bank_define_huge(kgpu_bank *b, int idx, int olen, int out_type) {
  return bank_define("kgpu_bank_define_huge", b, idx, olen, out_type, CP_HUGE);
}
extern "C" int kgpu_bank_define_ext(kgpu_bank *b, int idx, int olen, int out_type) {
  return bank_define("kgpu_bank_define_ext", b, idx, olen, out_type, CP_EXTENDED);
}
extern "C" int kgpu_bank_define_any(kgpu_bank *b, int idx, int olen, int out_type) {
  return bank_define("kgpu_bank_define_any", b, idx, olen, out_type, CP_BLUESTEIN);
}

// The forward transform of one response in place on stream st (set_filter's fftwf_execute, filter.c:1030), for the paths
// whose transform runs in one CTA: direct, wide and extended.  1: another path (the caller's own code).
static int response_transform_cta(float2 *dst, ChanGeom const &g, int points, cudaStream_t st) {
  size_t const sm = sizeof(float2) * (size_t)points;  // the narrow paths' transform in shared memory
  switch (g.r.path) {
    case CP_DIRECT:
      if (allow_smem((const void *)response_fft_kernel, sm)) return -1;
      response_fft_kernel<<<1, 32, sm, st>>>(dst, g.plan);
      break;
    case CP_WIDE: {
      size_t const smw = (size_t)wide_smem_bytes(g.wide.n1, g.wide.n2);
      if (allow_smem((const void *)response_wide_kernel, smw)) return -1;
      response_wide_kernel<<<1, kWideThreads, smw, st>>>(dst, g.wide);
      break;
    }
    case CP_EXTENDED:
      if (g.r.narrow) {
        if (allow_smem((const void *)response_fft_ext, sm)) return -1;
        response_fft_ext<<<1, 32, sm, st>>>(dst, g.ext);
      } else {
        size_t const smw = (size_t)wide_smem_bytes(g.wide_ext.g.n1, g.wide_ext.g.n2);
        if (allow_smem((const void *)response_wide_ext, smw)) return -1;
        response_wide_ext<<<1, kWideThreads, smw, st>>>(dst, g.wide_ext);
      }
      break;
    default:
      return 1;
  }
  g_launches++;
  return 0;
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
    ChanGeom const &g = *c.geom;
    switch (g.r.path) {
      case CP_DIRECT:
      case CP_WIDE:
      case CP_EXTENDED:
        if (response_transform_cta(dst, g, c.points, st)) return -1;
        break;
      case CP_HUGE: {
        float2 *scr = (float2 *)bank_scratch(b, st, sizeof(float2) * (size_t)c.points);
        if (!scr) return -1;
        size_t const sm1 = (size_t)huge_smem_bytes(g.huge.n1), sm2 = (size_t)huge_smem_bytes(g.huge.n2);
        if (allow_smem((const void *)response_huge_cols, sm1) || allow_smem((const void *)response_huge_rows, sm2)) return -1;
        response_huge_cols<<<(unsigned)((g.huge.n2 + kTile - 1) / kTile), kHugeThreads, sm1, st>>>(dst, g.huge, scr);
        response_huge_rows<<<(unsigned)((g.huge.n1 + kTile - 1) / kTile), kHugeThreads, sm2, st>>>(dst, g.huge, scr);
        g_launches += 2;
        break;
      }
      case CP_BLUESTEIN: {  // one block of the masters' chain: a COMPLEX master of `points` with hop 0, in place
        kgpu_master *im = bank_bluestein_master(b, st, g.r.blue.P);
        if (!im) return -1;
        long const in_len = (g.r.blue.P + 31) / 32 * 32;
        float2 *bin = (float2 *)bank_scratch(b, st, sizeof(float2) * (size_t)(in_len + im->spec_stride));
        if (!bin) return -1;
        BluesteinInArgs a{};
        a.in = dst;
        a.nblocks = 1;
        a.scale = 1.0f;
        BluesteinOutArgs o{};
        o.spec = dst;
        if (bluestein_chain(im, g.r.blue, a, o, bin, bin + in_len, st)) return -1;
        break;
      }
    }
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

// The specialised channel kernel of static plan P: chan_v2 (with the oscillator compiled in when `osc`) for a two-stage
// plan, chan_static for the others.
template <class P> static int launch_chan_static(ChanArgs const &a, int n, int nblocks, cudaStream_t st, bool osc) {
  void (*k)(ChanArgs);
  if constexpr (P::nst == 2) k = osc ? chan_v2<P, true> : chan_v2<P, false>;
  else k = chan_static<P>;
  if (allow_smem((const void *)k, StaticChan<P>::smem)) return -1;
  k<<<dim3((unsigned)((n + kChanWarps - 1) / kChanWarps), (unsigned)nblocks), kChanWarps * 32, StaticChan<P>::smem, st>>>(a);
  return 0;
}

// The chunks of channels and blocks of the multi-kernel paths (huge, Bluestein): at most `per` (channel, block) rows
// each, as many channels as fit, then as many blocks.  for_each runs launch(x, nc, nb) on each chunk of nc channels and
// nb blocks, x being its ChanArgs.
struct ChanChunks {
  int n, nblocks, cch, cbl;  // channels and blocks in all, per chunk
  ChanChunks(int n_, int nblocks_, long per)
      : n(n_), nblocks(nblocks_), cch((int)std::min<long>(n_, per)), cbl((int)std::max(1L, std::min<long>(nblocks_, per / cch))) {}
  size_t rows() const { return (size_t)cch * (size_t)cbl; }
  template <class F> int for_each(ChanArgs const &a, F launch) const {
    for (int c0 = 0; c0 < n; c0 += cch)
      for (int b0 = 0; b0 < nblocks; b0 += cbl) {
        ChanArgs x = a;
        if (x.order) x.order += c0;
        else x.chan_base += c0;
        x.norder = std::min(cch, n - c0);
        x.spec += (long)b0 * x.spec_stride;
        x.out += (long)b0 * x.out_stride;
        x.block0 += b0;
        if (x.power) x.power += (long)b0 * x.power_stride;
        if (launch(x, x.norder, std::min(cbl, nblocks - b0))) return -1;
      }
    return 0;
  }
};

// The huge channels of one length (chan_huge.cuh): pass A, pass B and, with d_power, the power reduction, in chunks of
// channels and blocks whose scratch stays within kHugeScratchCap.
static int launch_huge(kgpu_bank *b, ChanArgs const &a, ChanGeom const &geom, int n, int nblocks, cudaStream_t st) {
  HugeGeom const &g = geom.huge;
  long const slot = (long)geom.points * (long)sizeof(float2);
  ChanChunks const ch(n, nblocks, std::max(1L, kHugeScratchCap / slot));
  int const tiles_a = (g.n2 + kTile - 1) / kTile, tiles_b = (g.n1 + kTile - 1) / kTile;
  size_t const data = ch.rows() * (size_t)slot;
  char *scr = (char *)bank_scratch(b, st, data + ch.rows() * (size_t)tiles_b * sizeof(float));
  if (!scr) return -1;
  float *partial = a.power ? (float *)(scr + data) : nullptr;
  size_t const sm1 = (size_t)huge_smem_bytes(g.n1), sm2 = (size_t)huge_smem_bytes(g.n2);
  if (allow_smem((const void *)chan_huge_cols, sm1) || allow_smem((const void *)chan_huge_rows, sm2)) return -1;
  return ch.for_each(a, [&](ChanArgs const &x, int nc, int nb) {
    chan_huge_cols<<<dim3((unsigned)tiles_a, (unsigned)nc, (unsigned)nb), kHugeThreads, sm1, st>>>(x, g, (float2 *)scr);
    chan_huge_rows<<<dim3((unsigned)tiles_b, (unsigned)nc, (unsigned)nb), kHugeThreads, sm2, st>>>(x, g, (float2 const *)scr, partial);
    g_launches += 2;
    if (partial) {
      huge_power_kernel<<<dim3((unsigned)nc, (unsigned)nb), 32, 0, st>>>(x, partial, tiles_b);
      g_launches++;
    }
    return 0;
  });
}

// The Bluestein channels of one length (bluestein_chan.cuh): bluestein_chan_in, bluestein_conv on the stream's internal
// master, bluestein_chan_out and, with d_power, the power reduction, in chunks of channels
// and blocks whose two scratch buffers stay within kHugeScratchCap each.
static int launch_bluestein(kgpu_bank *b, ChanArgs const &a, ChanGeom const &geom, int n, int nblocks, cudaStream_t st) {
  long const P = geom.r.blue.P;
  kgpu_master *im = bank_bluestein_master(b, st, P);
  if (!im) return -1;
  long const ld = im->spec_stride;  // rows of P points in, rows of ld between the passes' spectra
  int const olen = (int)((long)geom.points * b->m->L / b->m->N);
  ChanChunks const ch(n, nblocks, std::min(kMaxBluesteinRows, std::max(1L, kHugeScratchCap / (ld * (long)sizeof(float2)))));
  int const tiles_in = (int)((P + kBluesteinThreads - 1) / kBluesteinThreads), tiles_out = (olen + kBluesteinThreads - 1) / kBluesteinThreads;
  size_t const rows = ch.rows();
  size_t const in_bytes = (rows * (size_t)P * sizeof(float2) + 255) / 256 * 256, out_bytes = rows * (size_t)ld * sizeof(float2);
  char *scr = (char *)bank_scratch(b, st, in_bytes + out_bytes + rows * (size_t)tiles_out * sizeof(float));
  if (!scr) return -1;
  float2 *bin = (float2 *)scr, *bout = (float2 *)(scr + in_bytes);
  float *partial = a.power ? (float *)(scr + in_bytes + out_bytes) : nullptr;
  return ch.for_each(a, [&](ChanArgs const &x, int nc, int nb) {
    bluestein_chan_in<<<dim3((unsigned)tiles_in, (unsigned)nc, (unsigned)nb), kBluesteinThreads, 0, st>>>(x, P, bin);
    if (bluestein_conv(im, geom.r.blue, bin, nc * nb, bout, st)) return -1;
    bluestein_chan_out<<<dim3((unsigned)tiles_out, (unsigned)nc, (unsigned)nb), kBluesteinThreads, 0, st>>>(x, 1.0 / (double)P, bout,
                                                                                                          ld, partial);
    g_launches += 2;
    if (partial) {
      huge_power_kernel<<<dim3((unsigned)nc, (unsigned)nb), 32, 0, st>>>(x, partial, tiles_out);
      g_launches++;
    }
    return 0;
  });
}

// one launch of the channels of one group
static int launch_chan(kgpu_bank *b, const void *d_spec, int nblocks, void *d_out, long out_stride, ChanGeom const &g,
                       int const *d_order, int base, int n, cudaStream_t st, bool generic = false, float *d_power = nullptr) {
  int const points = g.points;
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
  dim3 const ctas((unsigned)n, (unsigned)nblocks);  // chan_wide(_ext): one CTA per channel and block
  dim3 const warps((unsigned)((n + kChanWarps - 1) / kChanWarps), (unsigned)nblocks);  // chan_kernel(_ext): one warp each
  size_t const warp_smem = sizeof(float2) * (size_t)a.pitch * kChanWarps;
  // the paths other than direct run the same kernels whatever the static-kernel setting (they serve every variant)
  switch (g.r.path) {
    case CP_BLUESTEIN:
      return launch_bluestein(b, a, g, n, nblocks, st);
    case CP_HUGE:
      return launch_huge(b, a, g, n, nblocks, st);
    case CP_WIDE: {
      g_launches++;
      size_t const sm = (size_t)wide_smem_bytes(g.wide.n1, g.wide.n2);
      if (allow_smem((const void *)chan_wide, sm)) return -1;
      chan_wide<<<ctas, kWideThreads, sm, st>>>(a, g.wide);
      return 0;
    }
    case CP_EXTENDED: {
      g_launches++;
      if (!g.r.narrow) {
        size_t const sm = (size_t)wide_smem_bytes(g.wide_ext.g.n1, g.wide_ext.g.n2);
        if (allow_smem((const void *)chan_wide_ext, sm)) return -1;
        chan_wide_ext<<<ctas, kWideThreads, sm, st>>>(a, g.wide_ext);
        return 0;
      }
      if (allow_smem((const void *)chan_kernel_ext, warp_smem)) return -1;
      chan_kernel_ext<<<warps, kChanWarps * 32, warp_smem, st>>>(a, g.ext);
      return 0;
    }
    case CP_DIRECT:
      break;
  }
  g_launches++;
  TilePlan const *tp = host_tile_plan(g.plan);
  if (g_static_on.load() && !generic) {
    if (plan_is<S600>(tp)) return launch_chan_static<S600>(a, n, nblocks, st, b->any_osc);
    if (plan_is<S300>(tp)) return launch_chan_static<S300>(a, n, nblocks, st, b->any_osc);
    if (plan_is<S1200>(tp)) return launch_chan_static<S1200>(a, n, nblocks, st, b->any_osc);
  }
  if (allow_smem((const void *)chan_kernel, warp_smem)) return -1;
  chan_kernel<<<warps, kChanWarps * 32, warp_smem, st>>>(a);
  return 0;
}

extern "C" int kgpu_bank_run_ex(kgpu_bank *b, const void *d_spec, int nblocks, void *d_out, long out_pitch, float *d_power, void *stream) {
  if (!b || !d_spec || !d_out || nblocks < 1 || out_pitch < 0) return fail("kgpu_bank_run: bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  if (b->any_osc && b->block_counter - b->last_rebase > 4096) b->dirty = true;  // keep oscillator phases small
  if (bank_commit(b, st)) return -1;
  if (out_pitch && out_pitch < b->out_stride) return fail("kgpu_bank_run_ex: out_pitch %ld < packed row %ld", out_pitch, b->out_stride);
  for (auto const &g : b->groups)
    if (launch_chan(b, d_spec, nblocks, d_out, out_pitch ? out_pitch : b->out_stride, *g.geom, b->d_order + g.off, 0, g.count, st,
                    g.generic, d_power))
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
  if (launch_chan(b, d_spec, 1, origin, 0, *c.geom, nullptr, idx, 1, st, runtime_plan_only(b, idx), d_power ? d_power - idx : nullptr))
    return -1;
  CUDA_OK(cudaGetLastError());
  return 0;
}
// Noise density per channel and block from the device-resident spectrum (estimate_noise, radio.c:1783-1866).
static_assert(kNoiseSmemBins >= kMaxWideChanPoints, "every wide channel's noise window must fit shared memory");
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
  // windows of at most kNoiseSmemBins live in noise_kernel's shared memory whole, sized for the widest of them; the
  // wider ones (huge channels) go to noise_kernel_gm, which keeps them in the bank's scratch
  int window = 0, big_window = 0;
  std::vector<int> big;
  for (int i = 0; i < b->nchan; i++) {
    if (b->desc[(size_t)i].plan < 0 || b->desc[(size_t)i].points <= 0) continue;
    int const w = noise_window(b->desc[(size_t)i]);
    if (w <= kNoiseSmemBins) {
      window = std::max(window, w);
    } else {
      big.push_back(i);
      big_window = std::max(big_window, w);
    }
  }
  size_t const sm = sizeof(unsigned) * (size_t)window;
  if (allow_smem((const void *)noise_kernel, sm)) return -1;
  {
    ProfScope ps(K_NOISE, st);
    noise_kernel<<<dim3((unsigned)b->nchan, (unsigned)nblocks), kNoiseThreads, sm, st>>>(a);
  }
  g_launches++;
  if (!big.empty()) {
    long const stride = ((long)big_window + 31) / 32 * 32, nbig = (long)big.size();
    long const per = std::max(1L, kHugeScratchCap / (stride * (long)sizeof(unsigned)));  // (channel, block) slots per chunk
    int const cbl = (int)std::max(1L, std::min<long>(nblocks, per / nbig));
    size_t const list_off = (size_t)nbig * (size_t)cbl * (size_t)stride * sizeof(unsigned);
    char *scr = (char *)bank_scratch(b, st, list_off + sizeof(int) * big.size());
    if (!scr) return -1;
    CUDA_OK(cudaMemcpyAsync(scr + list_off, big.data(), sizeof(int) * big.size(), cudaMemcpyHostToDevice, st));
    ProfScope ps(K_NOISE, st);
    for (int b0 = 0; b0 < nblocks; b0 += cbl) {
      NoiseArgs x = a;
      x.spec += (long)b0 * x.spec_stride;
      x.n0 += (long)b0 * x.n0_stride;
      noise_kernel_gm<<<dim3((unsigned)nbig, (unsigned)std::min(cbl, nblocks - b0)), kNoiseGmThreads, 0, st>>>(
          x, (int const *)(scr + list_off), (unsigned *)scr, stride);
      g_launches++;
    }
  }
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

// ------------------------------------------------------------------ small masters -------------
// A master whose forward transform and every slave's inverse fit one CTA (small_master.cuh): radiod's per-channel
// secondary masters.  It owns its slaves' responses and geometry; the caller (filter_abi.c) owns the ring, the spectrum
// slots and the output rows.  No bank: each launch passes every slave's walk by value.
struct SmallSlaveHost {
  bool defined = false, real_out = false, has_response = false, isb = false;
  int olen = 0, points = 0, shift = 0;
  WideGeom const *g = nullptr;  // the inverse's four-step geometry
  float2 *d_resp = nullptr;     // points float2
};
struct kgpu_small {
  int L, M, N, in_type, bins, nc;
  long spec_stride;
  WideGeom const *fg;
  SmallSlaveHost s[kSmallMaxSlaves];
};

// A length one CTA transforms: factors 2, 3, 5, 7, at most kMaxWideChanPoints, a four-step split that fits shared memory.
// The shared memory it needs, or -1.  Host only.
static long small_len_smem(long n) {
  Split2 sp;
  if (n < 2 || n > kMaxWideChanPoints || !smooth7(n) || !choose_split(n, &sp) || sp.n1 < 2 || sp.n2 < 2) return -1;
  long const bytes = wide_smem_bytes(sp.n1, sp.n2);
  return bytes <= kChanSmemLimit ? bytes : -1;
}
// The four-step geometry of a length small_len_smem accepts, per device, built once and never freed (like g_geom).
static WideGeom const *small_geom(int points) {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) {
    fail("cudaGetDevice: %s", cudaGetErrorString(cudaGetLastError()));
    return nullptr;
  }
  static std::mutex mu;
  static std::map<std::pair<int, int>, WideGeom> geoms;
  std::lock_guard<std::mutex> lk(mu);
  auto it = geoms.find({dev, points});
  if (it != geoms.end()) return &it->second;
  Split2 sp;
  if (small_len_smem(points) < 0 || !choose_split(points, &sp)) {
    fail("%d points: not a one-CTA transform length", points);
    return nullptr;
  }
  WideGeom g{sp.n1, sp.n2, wide_pitch(sp.n2), get_tile_plan(sp.n1), get_tile_plan(sp.n2), nullptr};
  if (g.plan1 < 0 || g.plan2 < 0 || wide_twiddles(g, *host_tile_plan(g.plan2))) return nullptr;
  return &(geoms[{dev, points}] = g);
}

extern "C" long kgpu_small_smem(int L, int M, int in_type) {
  if (L < 1 || M < 1 || (in_type != KGPU_REAL && in_type != KGPU_COMPLEX)) return -1;
  long const N = (long)L + M - 1;
  if (in_type == KGPU_REAL && ((L & 1) || (N & 1))) return -1;
  return small_len_smem(in_type == KGPU_REAL ? N / 2 : N);
}

extern "C" kgpu_small *kgpu_small_create(int L, int M, int in_type) {
  if (kgpu_small_smem(L, M, in_type) < 0) {
    fail("kgpu_small_create(L=%d M=%d): outside the one-CTA envelope (Nc with factors 2, 3, 5, 7, at most %d points)", L, M,
         kMaxWideChanPoints);
    return nullptr;
  }
  kgpu_small *m = new kgpu_small;
  m->L = L;
  m->M = M;
  m->N = L + M - 1;
  m->in_type = in_type;
  m->bins = in_type == KGPU_COMPLEX ? m->N : m->N / 2 + 1;
  m->nc = in_type == KGPU_COMPLEX ? m->N : m->N / 2;
  m->spec_stride = ((long)m->bins + 3) / 4 * 4;
  m->fg = small_geom(m->nc);
  if (!m->fg) {
    delete m;
    return nullptr;
  }
  return m;
}
extern "C" void kgpu_small_destroy(kgpu_small *m) {
  if (!m) return;
  for (auto &s : m->s) cudaFree(s.d_resp);
  delete m;
}
extern "C" long kgpu_small_spec_stride(kgpu_small const *m) { return m ? m->spec_stride : -1; }

static bool small_bad(kgpu_small const *m, int idx) { return !m || idx < 0 || idx >= kSmallMaxSlaves; }

extern "C" int kgpu_small_define(kgpu_small *m, int idx, int olen, int out_type) {
  if (small_bad(m, idx) || olen < 1 || (out_type != KGPU_COMPLEX && out_type != KGPU_REAL))
    return fail("kgpu_small_define: bad arguments");
  long const num = (long)olen * m->N;
  if (num % m->L) return fail("invalid output length %d for N=%d L=%d (filter.c:312-316)", olen, m->N, m->L);
  int const points = (int)(num / m->L);
  if (out_type == KGPU_REAL && (points & 1))
    return fail("kgpu_small_define: REAL-output slaves need an even number of points (got %d)", points);
  WideGeom const *g = small_geom(points);
  if (!g) return fail("kgpu_small_define: %d-point slave is outside the one-CTA envelope", points);
  SmallSlaveHost &s = m->s[idx];
  if (!(s.defined && s.points == points)) {
    cudaFree(s.d_resp);
    s.d_resp = nullptr;
    CUDA_OK(cudaMalloc(&s.d_resp, sizeof(float2) * (size_t)points));
    s.has_response = false;
  }
  s.defined = true;
  s.real_out = out_type == KGPU_REAL;
  s.olen = olen;
  s.points = points;
  s.g = g;
  return points;
}
extern "C" int kgpu_small_undefine(kgpu_small *m, int idx) {
  if (small_bad(m, idx)) return fail("kgpu_small_undefine: bad arguments");
  cudaFree(m->s[idx].d_resp);
  m->s[idx] = SmallSlaveHost{};
  return 0;
}

// set_filter for slave idx on stream st: the bank's Kaiser design and response transform (bitwise the bank's response),
// copied to `response` (points float2).  Waits for st before the swap: queued launches may still read the old one.
extern "C" int kgpu_small_set_filter(kgpu_small *m, int idx, double low, double high, double kaiser_beta, float *response,
                                     void *stream) {
  if (small_bad(m, idx) || !m->s[idx].defined || !response) return fail("kgpu_small_set_filter: slave not defined");
  SmallSlaveHost &s = m->s[idx];
  cudaStream_t const st = (cudaStream_t)stream;
  if (s.real_out) {  // filter edges may not cross DC for a real output (filter.c:971-975)
    low = fabs(low);
    high = fabs(high);
  }
  std::vector<float2> taps;
  if (design_taps(s.points, s.olen, m->N, m->in_type == KGPU_REAL, low, high, kaiser_beta, taps))
    return fail("kgpu_small_set_filter: rejected (NaN or M < 2), cf. filter.c:969,989");
  ChanRoute r;
  if (chan_route(s.points, CP_EXTENDED, "kgpu_small_set_filter", &r)) return -1;
  ChanGeom const *g = chan_geom(s.points, r);
  if (!g) return -1;
  CUDA_OK(cudaStreamSynchronize(st));
  CUDA_OK(cudaMemcpyAsync(s.d_resp, taps.data(), sizeof(float2) * taps.size(), cudaMemcpyHostToDevice, st));
  if (response_transform_cta(s.d_resp, *g, s.points, st)) return fail("kgpu_small_set_filter: no one-CTA response transform");
  CUDA_OK(cudaGetLastError());
  CUDA_OK(cudaMemcpyAsync(response, s.d_resp, sizeof(float2) * (size_t)s.points, cudaMemcpyDeviceToHost, st));
  CUDA_OK(cudaStreamSynchronize(st));
  s.has_response = true;
  return 0;
}
extern "C" int kgpu_small_set_slave(kgpu_small *m, int idx, int shift, int isb) {
  if (small_bad(m, idx) || !m->s[idx].defined) return fail("kgpu_small_set_slave: slave not defined");
  m->s[idx].shift = shift;
  m->s[idx].isb = isb != 0;
  return 0;
}
// Output rows: slave i's olen float2 (COMPLEX) or olen floats in (olen + 1) / 2 float2 (REAL) at kgpu_small_out_offset,
// in slave order; a row is kgpu_small_out_stride float2.
extern "C" long kgpu_small_out_offset(kgpu_small const *m, int idx) {
  if (small_bad(m, idx)) return -1;
  long off = 0;
  for (int i = 0; i < idx; i++)
    if (m->s[i].defined) off += m->s[i].real_out ? (m->s[i].olen + 1) / 2 : m->s[i].olen;
  return off;
}
extern "C" long kgpu_small_out_stride(kgpu_small const *m) {
  if (!m) return -1;
  long off = 0;
  for (auto const &s : m->s)
    if (s.defined) off += s.real_out ? (s.olen + 1) / 2 : s.olen;
  return (off + 3) / 4 * 4;
}

extern "C" int kgpu_small_run(kgpu_small *m, const void *d_win, int nblocks, void *d_spec, void *d_out, long out_pitch, int only,
                              void *stream) {
  if (!m || nblocks < 1 || !d_spec || !d_out || only >= kSmallMaxSlaves || (only < 0 && !d_win))
    return fail("kgpu_small_run: bad arguments");
  SmallArgs a{};
  a.in = d_win;
  a.hop = m->in_type == KGPU_REAL ? m->L / 2 : m->L;
  a.fg = *m->fg;
  a.real = m->in_type == KGPU_REAL;
  a.spec = (float2 *)d_spec;
  a.spec_stride = m->spec_stride;
  a.m_bins = m->bins;
  a.out = (float2 *)d_out;
  a.out_stride = out_pitch;
  a.nslaves = kSmallMaxSlaves;
  a.only = only;
  long smem = only < 0 ? wide_smem_bytes(a.fg.n1, a.fg.n2) : 0, off = 0;
  for (int i = 0; i < kSmallMaxSlaves; i++) {
    SmallSlaveHost const &h = m->s[i];
    SmallSlave &s = a.s[i];
    s.d.plan = -1;
    if (!h.defined) continue;
    s.d.out_off = off;
    off += h.real_out ? (h.olen + 1) / 2 : h.olen;
    if (!h.has_response || (only >= 0 && i != only)) continue;
    ChanHost c;
    c.points = h.points;
    c.shift = h.shift;
    c.real_out = h.real_out;
    resolve_walk(m->in_type, m->bins, c, s.d);
    s.d.plan = 0;
    s.d.points = h.points;
    s.d.olen = h.olen;
    s.d.flags = h.real_out ? kChanRealOut : (h.isb ? kChanIsb : 0);
    s.g = *h.g;
    s.resp = h.d_resp;
    smem = std::max(smem, wide_smem_bytes(h.g->n1, h.g->n2));
  }
  if (only >= 0 && a.s[only].d.plan < 0) return fail("kgpu_small_run: slave %d has no response", only);
  if (allow_smem((const void *)small_master_kernel, (size_t)smem)) return -1;
  small_master_kernel<<<(unsigned)nblocks, kWideThreads, (size_t)smem, (cudaStream_t)stream>>>(a);
  g_launches++;
  CUDA_OK(cudaGetLastError());
  return 0;
}

// pure host helpers (usable without a GPU): what the planner would pick
extern "C" int kgpu_plan_radices(int len, int *radices, int max) {
  std::vector<int> r = choose_radices(len);
  if (len != 1 && r.empty()) return -1;
  for (int i = 0; i < (int)r.size() && i < max; i++) radices[i] = r[(size_t)i];
  return (int)r.size();
}
extern "C" int kgpu_plan_radices_ex(int len, int *radices, int max) {
  std::vector<int> r = choose_radices_ext(len);
  if (len != 1 && r.empty()) return -1;
  for (int i = 0; i < (int)r.size() && i < max; i++) radices[i] = r[(size_t)i];
  return (int)r.size();
}
extern "C" int kgpu_plan_split_ex(long n, int *n1, int *n2) {
  Split2 sp;
  if (!choose_split_ext(n, &sp)) return -1;
  *n1 = sp.n1;
  *n2 = sp.n2;
  return 0;
}
extern "C" int kgpu_plan_split(long n, int *n1, int *n2) {
  Split2 sp;
  if (!choose_split(n, &sp)) return -1;
  *n1 = sp.n1;
  *n2 = sp.n2;
  return 0;
}

// The path kgpu_bank_define_any takes for a channel of `points` points (chan_route), described without a device.
extern "C" int kgpu_chan_plan(int points, int out_type, char *buf, int buflen) {
  if (points < 1 || (out_type != KGPU_COMPLEX && out_type != KGPU_REAL)) return fail("kgpu_chan_plan: bad arguments");
  if (out_type == KGPU_REAL && (points & 1))
    return fail("kgpu_bank_define: REAL-output slaves need an even number of points (got %d)", points);
  ChanRoute r;
  if (chan_route(points, CP_BLUESTEIN, "kgpu_chan_plan", &r)) return -1;
  auto list = [](std::vector<int> const &v) {
    std::string s;
    for (size_t i = 0; i < v.size(); i++) s += std::to_string(v[i]) + (i + 1 < v.size() ? "," : "");
    return s;
  };
  bool const ext = r.path == CP_EXTENDED;
  char text[512];
  if (r.path == CP_BLUESTEIN) {
    snprintf(text, sizeof text, "bluestein: %d points, P=%ld: %s", points, r.blue.P,
             bluestein_text(r.blue, "bluestein_chan_in", "bluestein_chan_out").c_str());
  } else if (r.narrow) {
    std::vector<int> const rad = ext ? choose_radices_ext(points) : choose_radices(points);
    snprintf(text, sizeof text, "%s: %d points, radices [%s]; kernel %s", ext ? "extended" : "direct", points, list(rad).c_str(),
             ext ? "chan_kernel_ext" : "chan_kernel");
  } else {
    bool const huge = r.path == CP_HUGE;
    snprintf(text, sizeof text, "%s: %d points, four-step %d x %d; kernels %s", ext ? "extended" : huge ? "huge" : "wide", points,
             r.sp.n1, r.sp.n2, ext ? "chan_wide_ext" : huge ? "chan_huge_cols + chan_huge_rows" : "chan_wide");
  }
  if (buf && buflen > 0) snprintf(buf, (size_t)buflen, "%s", text);
  return (int)r.path;
}

// ------------------------------------------------------------------ wideband spectrum analyzer ----------
// wideband_poll (spectrum.c:308-522) on the device: spectrum_kernels.cuh around a forward master of its own.  The path
// is a function of fft_n and the input type alone:
//   SP_R2C        REAL, even fft_n, fft_n/2 23-smooth: the r2c pair of a REAL master L = fft_n, M = 1
//   SP_C2C        COMPLEX 23-smooth fft_n, or REAL odd 23-smooth fft_n: a COMPLEX master of length fft_n
//   SP_BLUESTEIN  anything else: two passes of a COMPLEX master of the smallest 7-smooth length P >= 2 fft_n - 1
enum SpecPath { SP_R2C, SP_C2C, SP_BLUESTEIN };
struct SpecPlan {
  SpecPath path;
  long nc;  // complex points of the forward master (fft_n/2, fft_n or P)
  long P;   // transform length of the master (fft_n or P)
  Split2 sp;
  Bluestein blue;  // SP_BLUESTEIN: its shape, and B once kgpu_spectrum_create has uploaded it
};

// Bound on the scratch of one poll (per buffer): longer polls run in chunks of segments.
static constexpr long kSpectrumScratchCap = 64L << 20;

static int spectrum_plan(int fft_n, int in_type, SpecPlan *pl) {
  if (fft_n < 2 || (in_type != KGPU_REAL && in_type != KGPU_COMPLEX))
    return fail("kgpu_spectrum: bad arguments fft_n=%d type=%d", fft_n, in_type);
  bool const real = in_type == KGPU_REAL;
  if (real && !(fft_n & 1) && smooth23(fft_n / 2) && forward_split(fft_n / 2, true, &pl->sp)) {
    pl->path = SP_R2C;
    pl->nc = fft_n / 2;
    pl->P = fft_n;
    return 0;
  }
  if ((!real || (fft_n & 1)) && smooth23(fft_n) && forward_split(fft_n, true, &pl->sp)) {
    pl->path = SP_C2C;
    pl->nc = pl->P = fft_n;
    return 0;
  }
  if (bluestein_shape(fft_n, &pl->blue)) {
    pl->path = SP_BLUESTEIN;
    pl->nc = pl->P = pl->blue.P;
    pl->sp = pl->blue.sp;
    return 0;
  }
  return fail("kgpu_spectrum: %d points have a prime factor >= 29 and need a Bluestein transform of at least %ld points, "
              "more than the forward pair splits", fft_n, 2L * fft_n - 1);
}
static void spectrum_plan_text(int fft_n, int in_type, SpecPlan const &pl, char *buf, int buflen) {
  char const *path = pl.path == SP_R2C ? "r2c" : pl.path == SP_C2C ? "complex" : "bluestein";
  snprintf(buf, (size_t)buflen, "%s fft_n=%d %s P=%ld: %ld-point complex two-pass %d x %d", path, fft_n,
           in_type == KGPU_REAL ? "real" : "complex", pl.P, pl.nc, pl.sp.n1, pl.sp.n2);
}

struct kgpu_spectrum {
  int fft_n, in_type, bin_count;
  SpecPlan pl;
  kgpu_master *m = nullptr;
  float *d_window = nullptr;
  void *d_in = nullptr;       // chunk windowed segments (float fft_n for the r2c, float2 P otherwise)
  float2 *d_spec = nullptr;   // chunk spectra, master spec_stride apart
  long in_len = 0;            // elements per segment of d_in
  long spec_stride = 0;
  int chunk = 0;              // segments per chunk
};

extern "C" int kgpu_spectrum_plan(int fft_n, int in_type, char *buf, int buflen) {
  SpecPlan pl;
  if (spectrum_plan(fft_n, in_type, &pl)) return -1;
  if (buf && buflen > 0) spectrum_plan_text(fft_n, in_type, pl, buf, buflen);
  return (int)pl.path;
}

extern "C" void kgpu_spectrum_destroy(kgpu_spectrum *s) {
  if (!s) return;
  kgpu_master_destroy(s->m);
  cudaFree(s->d_window);
  cudaFree(s->pl.blue.d_b);
  cudaFree(s->d_in);
  cudaFree(s->d_spec);
  delete s;
}

extern "C" kgpu_spectrum *kgpu_spectrum_create(int fft_n, int in_type, int bin_count) {
  SpecPlan pl;
  if (bin_count < 1) {
    fail("kgpu_spectrum_create: bad bin_count %d", bin_count);
    return nullptr;
  }
  if (spectrum_plan(fft_n, in_type, &pl)) return nullptr;
  kgpu_spectrum *s = new kgpu_spectrum;
  s->fft_n = fft_n;
  s->in_type = in_type;
  s->bin_count = bin_count;
  s->pl = pl;
  bool const r2c = pl.path == SP_R2C;
  s->m = r2c ? kgpu_master_create_ex(fft_n, 1, KGPU_REAL)
             : pl.path == SP_C2C ? kgpu_master_create_ex(fft_n, 1, KGPU_COMPLEX) : kgpu_master_create((int)pl.P, 1, KGPU_COMPLEX);
  if (!s->m) {
    fail("kgpu_spectrum_create: %s", std::string(g_err).c_str());
    kgpu_spectrum_destroy(s);
    return nullptr;
  }
  s->spec_stride = s->m->spec_stride;
  s->in_len = r2c ? fft_n : pl.P;
  size_t const in_bytes = r2c ? sizeof(float) * (size_t)fft_n : sizeof(float2) * (size_t)pl.P;
  size_t const spec_bytes = sizeof(float2) * (size_t)s->spec_stride;
  size_t const mid_bytes = sizeof(float2) * (size_t)s->m->sp.n1 * (size_t)((s->m->sp.n2 + 15) / 16 * 16);
  s->chunk = (int)std::min(32768L, std::max(1L, kSpectrumScratchCap / (long)std::max(in_bytes, std::max(spec_bytes, mid_bytes))));
  std::vector<float> ones((size_t)fft_n, 1.0f);
  cudaError_t e = cudaMalloc(&s->d_window, sizeof(float) * (size_t)fft_n);
  if (e == cudaSuccess) e = cudaMemcpy(s->d_window, ones.data(), sizeof(float) * (size_t)fft_n, cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaMalloc(&s->d_in, in_bytes * (size_t)s->chunk);
  if (e == cudaSuccess) e = cudaMalloc(&s->d_spec, spec_bytes * (size_t)s->chunk);
  if (e != cudaSuccess)
    fail("kgpu_spectrum_create(%d): %s", fft_n, cudaGetErrorString(e));
  else if (pl.path == SP_BLUESTEIN && bluestein_upload(&s->pl.blue))
    fail("kgpu_spectrum_create(%d): %s", fft_n, std::string(g_err).c_str());
  else
    return s;
  kgpu_spectrum_destroy(s);
  return nullptr;
}

extern "C" int kgpu_spectrum_set_window(kgpu_spectrum *s, float const *window) {
  if (!s || !window) return fail("kgpu_spectrum_set_window: bad arguments");
  CUDA_OK(cudaMemcpy(s->d_window, window, sizeof(float) * (size_t)s->fft_n, cudaMemcpyHostToDevice));
  return 0;
}

extern "C" int kgpu_spectrum_describe(kgpu_spectrum const *s, char *buf, int buflen) {
  if (!s || !buf || buflen < 1) return -1;
  spectrum_plan_text(s->fft_n, s->in_type, s->pl, buf, buflen);
  return 0;
}

// One poll in chunks of at most s->chunk segments: window, transform, then the wideband or narrowband bin mapping.  The
// bins carry over from chunk to chunk, so they accumulate in the reference's segment order.
static int spectrum_chunks(kgpu_spectrum *s, SpecWindowArgs w, SpecPowerArgs p, int fft_avg, bool narrow, cudaStream_t st) {
  for (int seg0 = 0; seg0 < fft_avg; seg0 += s->chunk) {
    int const nseg = std::min(s->chunk, fft_avg - seg0);
    w.seg0 = seg0;
    spectrum_window_kernel<<<dim3((unsigned)((s->in_len + kSpecThreads - 1) / kSpecThreads), (unsigned)nseg), kSpecThreads, 0,
                             st>>>(w);
    g_launches++;
    if (s->pl.path == SP_BLUESTEIN ? bluestein_conv(s->m, s->pl.blue, (float2 *)s->d_in, nseg, s->d_spec, st)
                                   : kgpu_forward(s->m, s->d_in, KGPU_FMT_F32, 1.0f, 0, nseg, s->d_spec, nullptr, st))
      return -1;
    p.nseg = nseg;
    p.first = seg0 == 0;
    unsigned const grid = (unsigned)((s->bin_count + kSpecThreads - 1) / kSpecThreads);
    if (narrow)
      narrowband_power_kernel<<<grid, kSpecThreads, 0, st>>>(p);
    else
      spectrum_power_kernel<<<grid, kSpecThreads, 0, st>>>(p);
    g_launches++;
  }
  CUDA_OK(cudaGetLastError());
  return 0;
}

extern "C" int kgpu_spectrum_run(kgpu_spectrum *s, const void *d_ring, long ring_samples, long end, int fmt, float scale,
                                 const kgpu_scale_change *d_chg, int nchg, long long end_index, int derandomize, int shift,
                                 int fft_avg, double overlap, float *d_bins, void *stream) {
  if (!s || !d_ring || !d_bins || fft_avg < 1 || !(overlap >= 0.0 && overlap < 1.0) || nchg < 0 || (nchg && !d_chg) ||
      (fmt != KGPU_FMT_F32 && fmt != KGPU_FMT_I16))
    return fail("kgpu_spectrum_run: bad arguments");
  int const fft_n = s->fft_n;
  if (ring_samples < fft_n) return fail("kgpu_spectrum_run: a ring of %ld samples is shorter than fft_n=%d", ring_samples, fft_n);
  cudaStream_t st = (cudaStream_t)stream;
  bool const real = s->in_type == KGPU_REAL;
  // spectrum.c:364,407 (REAL) and :422,491 (COMPLEX), in double as there
  long const adjust = lrint(fft_n * (1 + (fft_avg - 1) * (1 - overlap)));
  long const hop = lrint(fft_n * (1. - overlap));
  long start0 = (end - adjust) % ring_samples;
  if (start0 < 0) start0 += ring_samples;
  SpecWindowArgs w;
  w.ring = d_ring;
  w.cap = ring_samples;
  w.start0 = start0;
  w.step = real ? hop : -hop;
  w.fft_n = fft_n;
  w.out_len = (int)s->in_len;
  w.complex_in = !real;
  w.i16 = fmt == KGPU_FMT_I16;
  w.derandomize = derandomize != 0;
  w.flip = real && shift < 0;
  w.complex_out = s->pl.path != SP_R2C;
  w.chirp = s->pl.path == SP_BLUESTEIN;
  w.scale = scale;
  w.chg = (ScaleChange const *)d_chg;
  w.nchg = w.i16 ? nchg : 0;
  w.end = (end % ring_samples + ring_samples) % ring_samples;
  w.end_index = end_index;
  w.window = s->d_window;
  w.out = s->d_in;
  SpecPowerArgs p;
  p.spec = s->d_spec;
  p.spec_stride = s->spec_stride;
  p.real_walk = real;
  p.fft_n = fft_n;
  p.shift = shift;
  p.bin_count = s->bin_count;
  p.norm = s->pl.path == SP_BLUESTEIN ? 1.0 / ((double)s->pl.blue.P * (double)s->pl.blue.P) : 1.0;
  p.gain = (real ? 2. : 1.) / (double)((int64_t)fft_avg * fft_n * fft_n);  // spectrum.c:373, :431
  p.bins = d_bins;
  return spectrum_chunks(s, w, p, fft_avg, false, st);
}

extern "C" int kgpu_spectrum_run_narrow(kgpu_spectrum *s, const void *d_ring, long ring_size, long ring_idx, int fft_avg,
                                        double overlap, float *d_bins, int *fft_avg_used, void *stream) {
  if (!s || s->in_type != KGPU_COMPLEX || !d_ring || !d_bins || fft_avg < 1 || !(overlap >= 0.0 && overlap < 1.0))
    return fail("kgpu_spectrum_run_narrow: bad arguments");
  int const fft_n = s->fft_n;
  if (s->bin_count > fft_n) return fail("kgpu_spectrum_run_narrow: bin_count %d > fft_n %d", s->bin_count, fft_n);
  if (ring_size < fft_n) return fail("kgpu_spectrum_run_narrow: a ring of %ld samples is shorter than fft_n=%d", ring_size, fft_n);
  if (ring_idx < 0 || ring_idx >= ring_size) return fail("kgpu_spectrum_run_narrow: ring_idx %ld outside the ring", ring_idx);
  // spectrum.c:244-249, :278: the clamp with an integer ring_size / fft_n, the start, and the hop as the walk takes it
  // (fft_n forward, then lrint(fft_n overlap) back)
  double const avg_limit = floor(1 + ((ring_size / fft_n) - 1) / (1 - overlap));
  int const avg = fft_avg > avg_limit ? (int)lrint(avg_limit) : fft_avg;
  long rp = ring_idx - lrint(fft_n * (1 + (avg - 1) * (1 - overlap)));
  if (rp < 0) rp += ring_size;
  if (fft_avg_used) *fft_avg_used = avg;
  SpecWindowArgs w;
  w.ring = d_ring;
  w.cap = ring_size;
  w.start0 = ((rp % ring_size) + ring_size) % ring_size;
  w.step = fft_n - lrint(fft_n * overlap);
  w.fft_n = fft_n;
  w.out_len = (int)s->in_len;
  w.complex_in = 1;
  w.i16 = 0;
  w.derandomize = 0;
  w.flip = 0;
  w.complex_out = 1;
  w.chirp = s->pl.path == SP_BLUESTEIN;
  w.scale = 1.0f;
  w.nchg = 0;
  w.window = s->d_window;
  w.out = s->d_in;
  SpecPowerArgs p;
  p.spec = s->d_spec;
  p.spec_stride = s->spec_stride;
  p.real_walk = 0;
  p.fft_n = fft_n;
  p.shift = 0;
  p.bin_count = s->bin_count;
  p.norm = s->pl.path == SP_BLUESTEIN ? 1.0 / ((double)s->pl.blue.P * (double)s->pl.blue.P) : 1.0;
  p.gain = 1.0 / ((double)fft_n * fft_n * avg);  // spectrum.c:255
  p.bins = d_bins;
  return spectrum_chunks(s, w, p, avg, true, (cudaStream_t)stream);
}

extern "C" int kgpu_spectrum_ring_append(void *d_ring, long ring_size, long ring_idx, const void *d_src, long olen,
                                         void *stream) {
  if (!d_ring || ring_size < 1 || ring_idx < 0 || ring_idx >= ring_size || olen < 0)
    return fail("kgpu_spectrum_ring_append: bad arguments");
  long const n = std::min(olen, ring_size);
  if (n == 0) return 0;
  nb_ring_append_kernel<<<(unsigned)((n + kSpecThreads - 1) / kSpecThreads), kSpecThreads, 0, (cudaStream_t)stream>>>(
      (float2 *)d_ring, ring_size, ring_idx, (float2 const *)d_src, olen);
  g_launches++;
  CUDA_OK(cudaGetLastError());
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
