// Shared helpers for the sm_90a kernels of libvalle_b200.so.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_fp8.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/valle_b200.h"

#define VB_API extern "C" __attribute__((visibility("default")))

namespace vb {

// ---- error slot (thread-local, SURVEY 8b: no global mutable state but this) -------------
void set_error(const char *fmt, ...);
extern thread_local int64_t g_launches_tls;
void count_launch();
int tune(const char *name, int dflt);  // tuning knob: vb_tune_set() override, else environment variable, else dflt

#define VB_CHECK_ARG(cond, ...)            \
  do {                                     \
    if (!(cond)) {                         \
      vb::set_error(__VA_ARGS__);          \
      return VB_ERR_ARG;                   \
    }                                      \
  } while (0)

#define VB_CUDA(expr)                                                                  \
  do {                                                                                 \
    cudaError_t _e = (expr);                                                           \
    if (_e != cudaSuccess) {                                                           \
      vb::set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e)); \
      return VB_ERR_CUDA;                                                              \
    }                                                                                  \
  } while (0)

#define VB_LAUNCH_CHECK()      \
  do {                         \
    vb::count_launch();        \
    VB_CUDA(cudaGetLastError()); \
  } while (0)

#define VB_TRY(expr)            \
  do {                          \
    int _s = (expr);            \
    if (_s != VB_OK) return _s; \
  } while (0)

// ---- dtype helpers ------------------------------------------------------------------------
typedef __nv_bfloat16 bf16;

__device__ __forceinline__ float to_f32(float v) { return v; }
__device__ __forceinline__ float to_f32(bf16 v) { return __bfloat162float(v); }
template <typename T> __device__ __forceinline__ T from_f32(float v);
template <> __device__ __forceinline__ float from_f32<float>(float v) { return v; }
template <> __device__ __forceinline__ bf16 from_f32<bf16>(float v) { return __float2bfloat16_rn(v); }

// 16-byte vector of T: 4 floats or 8 bf16
template <typename T> struct Vec16;
template <> struct Vec16<float> {
  static constexpr int N = 4;
  float4 raw;
  __device__ __forceinline__ void unpack(float (&f)[4]) const {
    f[0] = raw.x; f[1] = raw.y; f[2] = raw.z; f[3] = raw.w;
  }
};
template <> struct Vec16<bf16> {
  static constexpr int N = 8;
  uint4 raw;
  __device__ __forceinline__ void unpack(float (&f)[8]) const {
    const uint32_t w[4] = {raw.x, raw.y, raw.z, raw.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      // bf16 -> f32 is a 16-bit left shift
      f[2 * i] = __uint_as_float(w[i] << 16);
      f[2 * i + 1] = __uint_as_float(w[i] & 0xffff0000u);
    }
  }
};

// streaming (read-once) 16-byte global load that does not pollute L1
__device__ __forceinline__ uint4 ldg_stream16(const void *p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p));
  return r;
}
template <typename T> __device__ __forceinline__ Vec16<T> load_stream(const T *p);
template <> __device__ __forceinline__ Vec16<float> load_stream<float>(const float *p) {
  Vec16<float> v;
  uint4 r = ldg_stream16(p);
  v.raw = make_float4(__uint_as_float(r.x), __uint_as_float(r.y), __uint_as_float(r.z),
                      __uint_as_float(r.w));
  return v;
}
template <> __device__ __forceinline__ Vec16<bf16> load_stream<bf16>(const bf16 *p) {
  Vec16<bf16> v;
  v.raw = ldg_stream16(p);
  return v;
}
template <typename T> __device__ __forceinline__ Vec16<T> load_vec(const T *p);
template <> __device__ __forceinline__ Vec16<float> load_vec<float>(const float *p) {
  Vec16<float> v;
  v.raw = *reinterpret_cast<const float4 *>(p);
  return v;
}
template <> __device__ __forceinline__ Vec16<bf16> load_vec<bf16>(const bf16 *p) {
  Vec16<bf16> v;
  v.raw = *reinterpret_cast<const uint4 *>(p);
  return v;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// ---- FP8 (e4m3) KV cache rows, one power-of-two scale per 64-element row (include/valle_b200.h,
//      "FP8 (e4m3) KV cache").  Exponents travel biased: eb = e + 127, eb in [0, 254].
// eb of a row with max |r| = a: the smallest integer e with a <= 448 * 2^e (frexpf: a = m 2^x, m in [0.5, 1); e = x - 9
// when m <= 0.875 = 448 / 2^9, else x - 8), clamped to [-127, 127]; an all-zero row gets e = -127
__device__ __forceinline__ int kv8_exp_biased(float a) {
  if (!(a > 0.f)) return 0;
  int x;
  const float m = frexpf(a, &x);
  const int e = m <= 0.875f ? x - 9 : x - 8;
  return min(max(e, -127), 127) + 127;
}
// 2^(eb - 127) in fp32 (eb = 0: the subnormal 2^-127); 2^-(eb - 127) = kv8_scale(254 - eb)
__device__ __forceinline__ float kv8_scale(int eb) { return __int_as_float(eb > 0 ? eb << 23 : 0x00400000); }
// cvt.rn.satfinite.e4m3 of r * 2^-e (the product is exact: a power-of-two scale)
__device__ __forceinline__ uint8_t kv8_quant(float r, int eb) {
  return (uint8_t)__nv_cvt_float_to_fp8(r * kv8_scale(254 - eb), __NV_SATFINITE, __NV_E4M3);
}
// 8 e4m3 bytes -> 8 floats (exact: e4m3 -> f16 -> f32)
__device__ __forceinline__ void kv8_unpack(uint2 raw, float (&f)[8]) {
  const uint32_t w[2] = {raw.x, raw.y};
#pragma unroll
  for (int i = 0; i < 2; ++i) {
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const __half2_raw hr = __nv_cvt_fp8x2_to_halfraw2((__nv_fp8x2_storage_t)(w[i] >> (16 * j)), __NV_E4M3);
      const float2 p = __half22float2(__half2(hr));
      f[4 * i + 2 * j] = p.x;
      f[4 * i + 2 * j + 1] = p.y;
    }
  }
}
// streaming 8-byte global load (half a bf16 row chunk: 8 e4m3 elements)
__device__ __forceinline__ uint2 ldg_stream8(const void *p) {
  uint2 r;
  asm volatile("ld.global.nc.L1::no_allocate.v2.u32 {%0,%1}, [%2];" : "=r"(r.x), "=r"(r.y) : "l"(p));
  return r;
}

// ---- grid-wide barrier of a cooperative launch (every CTA resident).  `ctr` is a monotonic arrival counter zeroed
// before the launch, together with the generation word 32 words behind it; `target` (thread 0) advances by gridDim.x
// per barrier.  The LAST arriver publishes the target as the generation word, which the others poll: the counter line
// sees one atomic per CTA, where ~150 CTAs polling the counter itself would hammer that L2 line and delay the late
// arrivals' atomics.
__device__ __forceinline__ void grid_barrier_sync(unsigned *ctr, unsigned &target) {
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned G = gridDim.x * gridDim.y * gridDim.z;
    target += G;
    unsigned *gen = ctr + 32;   // a different 128-byte line
    unsigned prev;
    asm volatile("atom.add.acq_rel.gpu.global.u32 %0, [%1], 1;" : "=r"(prev) : "l"(ctr) : "memory");
    if (prev + 1 == target) {
      asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(gen), "r"(target) : "memory");
    } else {
      unsigned v;
      do {
        __nanosleep(20);
        asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(gen) : "memory");
      } while ((int)(v - target) < 0);
    }
  }
  __syncthreads();
}

// ---- programmatic dependent launch (no-ops unless the launch carries the PDL attribute) -------
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() {
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
}

template <typename... KArgs, typename... Args>
inline cudaError_t launch_kernel_cluster(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t s,
                                         bool pdl, dim3 cluster, Args... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = s;
  cudaLaunchAttribute attr[2];
  int n = 0;
  if (pdl) {
    attr[n].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[n].val.programmaticStreamSerializationAllowed = 1;
    ++n;
  }
  if (cluster.x * cluster.y * cluster.z > 1) {
    attr[n].id = cudaLaunchAttributeClusterDimension;
    attr[n].val.clusterDim.x = cluster.x;
    attr[n].val.clusterDim.y = cluster.y;
    attr[n].val.clusterDim.z = cluster.z;
    ++n;
  }
  cfg.attrs = attr;
  cfg.numAttrs = n;
  return cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
}
template <typename... KArgs, typename... Args>
inline cudaError_t launch_kernel(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t s,
                                 bool pdl, Args... args) {
  return launch_kernel_cluster(kern, grid, block, smem, s, pdl, dim3(1, 1, 1), args...);
}

// SM count of the CURRENT device (cached per device: a process may drive several GPUs)
inline int sm_count() {
  static int n[64] = {0};
  int dev = 0;
  cudaGetDevice(&dev);
  const int slot = dev & 63;
  if (n[slot] == 0) {
    int v = 0;
    cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev);
    n[slot] = v > 0 ? v : 132;
  }
  return n[slot];
}
// L2 size in bytes of the CURRENT device (cached per device)
inline int64_t l2_bytes() {
  static int64_t n[64] = {0};
  int dev = 0;
  cudaGetDevice(&dev);
  const int slot = dev & 63;
  if (n[slot] == 0) {
    int v = 0;
    cudaDeviceGetAttribute(&v, cudaDevAttrL2CacheSize, dev);
    n[slot] = v > 0 ? v : (int64_t)50 << 20;
  }
  return n[slot];
}

// cudaFuncSetAttribute(MaxDynamicSharedMemorySize) is per (function, device): remember which devices were done
struct PerDeviceOnce {
  bool done[64] = {false};
  // true exactly once per device (callers then set their function attributes)
  bool first() {
    int dev = 0;
    cudaGetDevice(&dev);
    const int slot = dev & 63;
    if (done[slot]) return false;
    done[slot] = true;
    return true;
  }
};

// ---- device timeline (profiling builds only: -DVB_TRACE, libvalle_b200_trace.so) ----------------
// Thread 0 of block (0,0,0) of a traced kernel appends (globaltimer << 8 | id) to a ring bound with
// vb_trace_bind() (the ring keeps the most recent `cap` stamps); ids: kernel kind * 2 + (0 = dependency resolved, 1 = block 0 done).
#ifdef VB_TRACE
static __device__ unsigned long long *g_trace_buf = nullptr;
static __device__ unsigned int *g_trace_cnt = nullptr;
static __device__ unsigned int g_trace_cap = 0;
static __device__ unsigned int g_trace_all = 0;   // 1: only vb_trace_cta stamps (every CTA of the traced kernel)
// every CTA's thread 0: (low 40 bits of globaltimer << 24) | (linear block id, 16 bits) << 8 | id  (tools/trace_attn_ctas.py)
__device__ __forceinline__ void vb_trace_cta(int id) {
  if (threadIdx.x == 0 && g_trace_all != 0 && g_trace_buf != nullptr) {
    unsigned long long t;
    asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
    const unsigned bid = blockIdx.x + gridDim.x * (blockIdx.y + gridDim.y * blockIdx.z);
    const unsigned i = atomicAdd(g_trace_cnt, 1u);
    g_trace_buf[i % g_trace_cap] = ((t & ((1ull << 40) - 1)) << 24) | ((unsigned long long)(bid & 0xffff) << 8) |
                                   (unsigned long long)(id & 0xff);
  }
}
__device__ __forceinline__ void vb_trace(int id) {
  if ((blockIdx.x | blockIdx.y | blockIdx.z | threadIdx.x) == 0 && g_trace_buf != nullptr && g_trace_all == 0) {
    unsigned long long t;
    asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
    const unsigned i = atomicAdd(g_trace_cnt, 1u);
    g_trace_buf[i % g_trace_cap] = (t << 8) | (unsigned long long)(id & 0xff);  // ring: the last cap stamps survive
  }
}
typedef int (*trace_bind_fn)(unsigned long long *, unsigned int *, unsigned int);
void trace_register(trace_bind_fn f);
static int trace_bind_tu(unsigned long long *buf, unsigned int *cnt, unsigned int cap) {
  if (cudaMemcpyToSymbol(g_trace_buf, &buf, sizeof(buf)) != cudaSuccess) return 1;
  if (cudaMemcpyToSymbol(g_trace_cnt, &cnt, sizeof(cnt)) != cudaSuccess) return 1;
  const unsigned int all = cap >> 31;   // top bit of the capacity: per-CTA stamps of the attention kernel only
  cap &= 0x7fffffffu;
  if (cudaMemcpyToSymbol(g_trace_cap, &cap, sizeof(cap)) != cudaSuccess) return 1;
  if (cudaMemcpyToSymbol(g_trace_all, &all, sizeof(all)) != cudaSuccess) return 1;
  return 0;
}
namespace {
struct TraceReg {
  TraceReg() { trace_register(trace_bind_tu); }
};
static TraceReg g_trace_reg;
}  // namespace
#else
#define vb_trace(id) ((void)0)
#define vb_trace_cta(id) ((void)0)
#endif
enum { TR_LN = 1, TR_GEMM = 2, TR_ATTN = 3, TR_RELU = 4, TR_SAMPLE = 5, TR_COMBINE = 6, TR_FUSED = 7 };

static inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

}  // namespace vb
