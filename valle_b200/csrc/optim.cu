// Optimizer steps of the trainer (include/valle_b200.h f3): ScaledAdam and Eve, valle/modules/optim.py.
//   * sadam_reduce_kernel: per chunk of VB_OPTIM_CHUNK elements, sum g^2, sum p*g and sum p^2 (p and g read once).
//   * sadam_coef_kernel: one CTA.  Per-tensor sums in chunk order, the model norm and the clip scale, model_norms and
//     the clipping counters, scale_grads / param_rms / scale_exp_avg_sq, and one (alpha, scale_step) pair per tensor.
//   * sadam_update_kernel: the elementwise update of delta, exp_avg_sq and p (optim.py:479-661).
//   * eve_reduce_kernel / eve_update_kernel: per-chunk sum p^2, then the Eve update with the per-tensor norm test.
// The gradient pointers (which change every step under zero_grad(set_to_none=True)) travel by value in the kernel
// parameters (CUDA 12.1+: up to 32 KB on sm_90), so the host never uploads a table and never waits.
#include <math.h>

#include "common.cuh"

namespace vb {
namespace {

constexpr int OPT_THREADS = 256;
constexpr int OPT_CHUNK = VB_OPTIM_CHUNK;
constexpr int OPT_MAXT = VB_OPTIM_MAX_TENSORS;
constexpr int EVE_MAXT = VB_OPTIM_EVE_MAX_TENSORS;
constexpr int COEF_THREADS = 1024;

// the gradient pointers and chunk offsets of tensors [t0, t0 + nt) of the table
struct GradSlice {
  const float *g[OPT_MAXT];
  int32_t chunk0[OPT_MAXT + 1];  // absolute chunk offsets; chunk0[nt] ends the slice
  int32_t t0, nt;
};
static_assert(sizeof(GradSlice) < 32000, "kernel parameters are limited to 32764 bytes");

struct EveSlice {
  vb_eve_tensor e[EVE_MAXT];
  int32_t chunk0[EVE_MAXT + 1];
  int32_t nt;
};
static_assert(sizeof(EveSlice) < 32000, "kernel parameters are limited to 32764 bytes");

__host__ __device__ __forceinline__ int64_t n_chunks_of(int64_t numel) { return (numel + OPT_CHUNK - 1) / OPT_CHUNK; }

// the slice entry j whose chunks contain absolute chunk c: the last j with chunk0[j] <= c (empty tensors skipped)
__device__ __forceinline__ int find_entry(const int32_t *chunk0, int nt, int c) {
  int lo = 0, hi = nt;  // chunk0[lo] <= c < chunk0[hi]
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (chunk0[mid] <= c) lo = mid; else hi = mid;
  }
  return lo;
}

__device__ __forceinline__ bool aligned16(const void *a) { return (reinterpret_cast<uintptr_t>(a) & 15) == 0; }

// sum of N values over the CTA in a fixed order (deterministic); the result is valid in thread 0
template <int N, int THREADS>
__device__ __forceinline__ void block_sum(float (&v)[N], float *sh /* [N][THREADS / 32] */) {
  constexpr int W = THREADS / 32;
#pragma unroll
  for (int k = 0; k < N; ++k) v[k] = warp_sum(v[k]);
  if ((threadIdx.x & 31) == 0)
#pragma unroll
    for (int k = 0; k < N; ++k) sh[k * W + (threadIdx.x >> 5)] = v[k];
  __syncthreads();
  if (threadIdx.x == 0)
#pragma unroll
    for (int k = 0; k < N; ++k) {
      float s = 0.f;
      for (int w = 0; w < W; ++w) s += sh[k * W + w];
      v[k] = s;
    }
}

// ---- ScaledAdam -----------------------------------------------------------------------------------------------------
// The clip scale reaches the update only through scale_grads: _step and _step_scalar read the unclipped p.grad
// (optim.py:611, 648), while _step_one_batch scales its local copy (optim.py:495-509).
__global__ void __launch_bounds__(OPT_THREADS) sadam_reduce_kernel(const vb_scaled_adam_tensor *__restrict__ tab,
                                                                   const __grid_constant__ GradSlice gs,
                                                                   float *__restrict__ partials) {
  __shared__ float sh[3 * OPT_THREADS / 32];
  const int c = gs.chunk0[0] + blockIdx.x;
  const int j = find_entry(gs.chunk0, gs.nt, c);
  const float *p = tab[gs.t0 + j].param;
  const int64_t numel = tab[gs.t0 + j].numel;
  const float *g = gs.g[j];
  const int64_t begin = (int64_t)(c - gs.chunk0[j]) * OPT_CHUNK;
  const int64_t end = min(begin + (int64_t)OPT_CHUNK, numel);
  float v[3] = {0.f, 0.f, 0.f};  // g^2, p*g, p^2
  int64_t i = begin;
  if (aligned16(p) && (g == nullptr || aligned16(g))) {
    const int64_t end4 = begin + ((end - begin) & ~(int64_t)3);
    for (int64_t k = begin + 4 * threadIdx.x; k < end4; k += 4 * OPT_THREADS) {
      float pf[4], gf[4] = {0.f, 0.f, 0.f, 0.f};
      load_stream(p + k).unpack(pf);
      if (g != nullptr) load_stream(g + k).unpack(gf);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        v[0] = fmaf(gf[e], gf[e], v[0]);
        v[1] = fmaf(pf[e], gf[e], v[1]);
        v[2] = fmaf(pf[e], pf[e], v[2]);
      }
    }
    i = end4;
  }
  for (int64_t k = i + threadIdx.x; k < end; k += OPT_THREADS) {
    const float pf = p[k], gf = g != nullptr ? g[k] : 0.f;
    v[0] = fmaf(gf, gf, v[0]);
    v[1] = fmaf(pf, gf, v[1]);
    v[2] = fmaf(pf, pf, v[2]);
  }
  block_sum<3, OPT_THREADS>(v, sh);
  if (threadIdx.x == 0) {
    partials[3 * (int64_t)c + 0] = v[0];
    partials[3 * (int64_t)c + 1] = v[1];
    partials[3 * (int64_t)c + 2] = v[2];
  }
}

struct CoefArgs {
  int n_tensors;
  int clip_mode, log_step, clip_period, norm_slot;
  double clipping_scale;
  int init, sg_slot, size_period, refresh_rms, size_update;
  float beta2_corr, omb2_corr, size_coef, min_rms, max_rms, max_fill, eps, alpha_coef;
};

__global__ void __launch_bounds__(COEF_THREADS) sadam_coef_kernel(const vb_scaled_adam_tensor *__restrict__ tab,
                                                                  const float *__restrict__ partials,
                                                                  float *__restrict__ coef, float *model_norms,
                                                                  vb_clip_state *clip, const CoefArgs a) {
  __shared__ float sh[COEF_THREADS / 32];
  __shared__ float s_scale, s_median;
  // 1. per-tensor sums in chunk order; this tensor's share of tot_sumsq with the param_rms before this step
  float tot[1] = {0.f};
  for (int t = threadIdx.x; t < a.n_tensors; t += COEF_THREADS) {
    const vb_scaled_adam_tensor e = tab[t];
    const int64_t c1 = e.chunk0 + n_chunks_of(e.numel);
    float gg = 0.f, pp = 0.f;
    for (int64_t c = e.chunk0; c < c1; ++c) {
      gg += partials[3 * c + 0];
      pp += partials[3 * c + 2];
    }
    if (a.init && e.param_rms != nullptr) *e.param_rms = sqrtf(pp / (float)e.numel);
    if (e.scalar) {
      tot[0] += gg;
    } else {
      const float r = *e.param_rms;
      tot[0] += gg * (r * r);
    }
  }
  // 2. the model norm and the clip scale (optim.py:342-412)
  block_sum<1, COEF_THREADS>(tot, sh);
  if (threadIdx.x == 0) {
    s_scale = 1.f;
    s_median = 0.f;
  }
  __syncthreads();
  const float norm = sqrtf(tot[0]);  // thread 0 only
  if (a.clip_mode >= 1 && threadIdx.x == 0) model_norms[a.norm_slot] = norm;
  __syncthreads();
  if (a.clip_mode >= 1 && a.log_step) {
    // the element at sorted index k of model_norms: its rank among them, ties broken by index (exact, no sort)
    const int P = a.clip_period;
    const int k = min(P - 1, (P / 4) * 2);
    for (int i = threadIdx.x; i < P; i += COEF_THREADS) {
      const float vi = model_norms[i];
      int rank = 0;
      for (int j = 0; j < P; ++j) {
        const float vj = model_norms[j];
        rank += (vj < vi) || (vj == vi && j < i);
      }
      if (rank == k) s_median = vi;
    }
    __syncthreads();
  }
  if (threadIdx.x == 0 && a.clip_mode >= 1) {
    if (a.log_step) {
      clip->threshold = a.clipping_scale * (double)s_median;
      clip->has_threshold = 1;
      clip->prev_clipped = clip->num_clipped;
      clip->num_clipped = 0;
      clip->prev_min_scale = clip->min_scale;
      clip->min_scale = 1.f;
    }
    float s = 1.f;
    if (a.clip_mode == 2 && clip->has_threshold) {
      // Python float / fp32 tensor is reciprocal(tensor) * float
      const float r = (1.f / (norm + 1.0e-20f)) * (float)clip->threshold;
      s = fminf(1.f, r);
      if (s < 1.f) {
        clip->num_clipped += 1;
        clip->min_scale = fminf(clip->min_scale, s);
      }
    }
    clip->scale = s;
    s_scale = s;
  }
  __syncthreads();
  const float s = s_scale;
  if (blockIdx.x == 0 && threadIdx.x == 0) coef[2 * a.n_tensors] = s;
  // 3. scale_grads, param_rms, the size update (optim.py:504-596) and the per-tensor coefficients
  for (int t = threadIdx.x; t < a.n_tensors; t += COEF_THREADS) {
    const vb_scaled_adam_tensor e = tab[t];
    float alpha = 0.f, sstep = 0.f;
    if (!e.scalar) {
      const int64_t c1 = e.chunk0 + n_chunks_of(e.numel);
      float pg = 0.f, pp = 0.f;
      for (int64_t c = e.chunk0; c < c1; ++c) {
        pg += partials[3 * c + 1];
        pp += partials[3 * c + 2];
      }
      float *sg = e.scale_grads;
      const int64_t st = e.sg_stride;
      sg[a.sg_slot * st] = pg * s;
      float rms = *e.param_rms;
      if (a.refresh_rms) {
        rms = sqrtf(pp / (float)e.numel);
        *e.param_rms = rms;
      }
      if (a.size_update) {
        float sq = 0.f, sum = 0.f;
        for (int k = 0; k < a.size_period; ++k) {
          const float x = sg[k * st];
          sq += x * x;
          sum += x;
        }
        const float seas = *e.scale_exp_avg_sq * a.beta2_corr + a.omb2_corr * (sq / (float)a.size_period);
        *e.scale_exp_avg_sq = seas;
        sstep = a.size_coef * sum / (sqrtf(seas) + a.eps);
        if (rms < a.min_rms) sstep = 0.f;
        if (rms > a.max_rms) sstep = a.max_fill;
      }
      alpha = a.alpha_coef * fmaxf(rms, a.min_rms);
    }
    coef[2 * t] = alpha;
    coef[2 * t + 1] = sstep;
  }
}

struct UpdateArgs {
  float beta1, beta2, omb1, omb2, eps;
  int bias_correct;
  float inv_bc2;       // (float)(1 / bias_correction2), non-scalar tensors
  float inv_bc2_s;     // 1 / (float)bias_correction2, scalars (Tensor / Python float multiplies by the reciprocal)
  float scalar_alpha;  // -lr * scalar_lr_scale * (1 - beta1)
  float scalar_max;
  int size_step;
};

struct SadamElem {
  float beta1, beta2, omb1, omb2, eps, vscale, alpha, sstep;
  bool size_step, bias_correct;
  __device__ __forceinline__ void run(float &p, float g, float &d, float &v) const {
    d = d * beta1;
    if (size_step) d = d + omb1 * (p * sstep);
    v = v * beta2 + omb2 * (g * g);
    const float vv = bias_correct ? v * vscale : v;
    d = d + (g / (sqrtf(vv) + eps)) * alpha;
    p = p + d;
  }
};

__global__ void __launch_bounds__(OPT_THREADS) sadam_update_kernel(const vb_scaled_adam_tensor *__restrict__ tab,
                                                                   const __grid_constant__ GradSlice gs,
                                                                   const float *__restrict__ coef, const int n_tensors,
                                                                   const UpdateArgs a) {
  const int c = gs.chunk0[0] + blockIdx.x;
  const int j = find_entry(gs.chunk0, gs.nt, c);
  const int t = gs.t0 + j;
  const vb_scaled_adam_tensor e = tab[t];
  const float *g = gs.g[j];
  const int64_t begin = (int64_t)(c - gs.chunk0[j]) * OPT_CHUNK;
  const int64_t end = min(begin + (int64_t)OPT_CHUNK, e.numel);
  if (e.scalar) {
    // _step_scalar (optim.py:639-661): one element per parameter
    for (int64_t k = begin + threadIdx.x; k < end; k += OPT_THREADS) {
      const float gf = g != nullptr ? g[k] : 0.f;
      float d = e.delta[k] * a.beta1;
      float v = e.exp_avg_sq[k] * a.beta2 + a.omb2 * (gf * gf);
      d = d + a.scalar_alpha * (gf / (sqrtf(v * a.inv_bc2_s) + a.eps));
      const float p = fminf(fmaxf(e.param[k], -a.scalar_max), a.scalar_max) + d;
      e.delta[k] = d;
      e.exp_avg_sq[k] = v;
      e.param[k] = p;
    }
    return;
  }
  SadamElem op{a.beta1, a.beta2, a.omb1, a.omb2, a.eps, a.inv_bc2, coef[2 * t], coef[2 * t + 1], a.size_step != 0,
               a.bias_correct != 0};
  int64_t i = begin;
  if (aligned16(e.param) && aligned16(e.delta) && aligned16(e.exp_avg_sq) && (g == nullptr || aligned16(g))) {
    const int64_t end4 = begin + ((end - begin) & ~(int64_t)3);
    for (int64_t k = begin + 4 * threadIdx.x; k < end4; k += 4 * OPT_THREADS) {
      float4 p4 = *reinterpret_cast<const float4 *>(e.param + k);
      float4 d4 = *reinterpret_cast<const float4 *>(e.delta + k);
      float4 v4 = *reinterpret_cast<const float4 *>(e.exp_avg_sq + k);
      float gf[4] = {0.f, 0.f, 0.f, 0.f};
      if (g != nullptr) load_stream(g + k).unpack(gf);
      op.run(p4.x, gf[0], d4.x, v4.x);
      op.run(p4.y, gf[1], d4.y, v4.y);
      op.run(p4.z, gf[2], d4.z, v4.z);
      op.run(p4.w, gf[3], d4.w, v4.w);
      *reinterpret_cast<float4 *>(e.param + k) = p4;
      *reinterpret_cast<float4 *>(e.delta + k) = d4;
      *reinterpret_cast<float4 *>(e.exp_avg_sq + k) = v4;
    }
    i = end4;
  }
  for (int64_t k = i + threadIdx.x; k < end; k += OPT_THREADS) {
    float p = e.param[k], d = e.delta[k], v = e.exp_avg_sq[k];
    op.run(p, g != nullptr ? g[k] : 0.f, d, v);
    e.param[k] = p;
    e.delta[k] = d;
    e.exp_avg_sq[k] = v;
  }
}

// ---- Eve ------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(OPT_THREADS) eve_reduce_kernel(const __grid_constant__ EveSlice es,
                                                                 float *__restrict__ partials) {
  __shared__ float sh[OPT_THREADS / 32];
  const int c = es.chunk0[0] + blockIdx.x;
  const int j = find_entry(es.chunk0, es.nt, c);
  const float *p = es.e[j].param;
  const int64_t begin = (int64_t)(c - es.chunk0[j]) * OPT_CHUNK;
  const int64_t end = min(begin + (int64_t)OPT_CHUNK, es.e[j].numel);
  float v[1] = {0.f};
  int64_t i = begin;
  if (aligned16(p)) {
    const int64_t end4 = begin + ((end - begin) & ~(int64_t)3);
    for (int64_t k = begin + 4 * threadIdx.x; k < end4; k += 4 * OPT_THREADS) {
      const float4 p4 = *reinterpret_cast<const float4 *>(p + k);
      v[0] = fmaf(p4.x, p4.x, v[0]);
      v[0] = fmaf(p4.y, p4.y, v[0]);
      v[0] = fmaf(p4.z, p4.z, v[0]);
      v[0] = fmaf(p4.w, p4.w, v[0]);
    }
    i = end4;
  }
  for (int64_t k = i + threadIdx.x; k < end; k += OPT_THREADS) v[0] = fmaf(p[k], p[k], v[0]);
  block_sum<1, OPT_THREADS>(v, sh);
  if (threadIdx.x == 0) partials[c] = v[0];
}

struct EveArgs {
  float beta1, beta2, omb1, omb2, eps, decay;  // decay = 1 - weight_decay (fp32)
};

struct EveElem {
  float beta1, beta2, omb1, omb2, eps, bc2r, mult, neg_step;
  __device__ __forceinline__ void run(float &p, float g, float &m, float &v) const {
    m = m * beta1 + omb1 * g;
    v = v * beta2 + omb2 * (g * g);
    const float den = sqrtf(v) * bc2r + eps;
    p = p * mult;
    p = p + neg_step * (m / den);
  }
};

__global__ void __launch_bounds__(OPT_THREADS) eve_update_kernel(const __grid_constant__ EveSlice es,
                                                                 const float *__restrict__ partials,
                                                                 const EveArgs a) {
  __shared__ float s_mult;
  const int c = es.chunk0[0] + blockIdx.x;
  const int j = find_entry(es.chunk0, es.nt, c);
  const vb_eve_tensor &e = es.e[j];
  if (threadIdx.x == 0) {
    float mult = 1.f;
    if (e.numel > 1) {
      float ss = 0.f;
      for (int k = es.chunk0[j]; k < es.chunk0[j + 1]; ++k) ss += partials[k];
      if (sqrtf(ss) > e.norm_limit) mult = a.decay;
    }
    s_mult = mult;
  }
  __syncthreads();
  const EveElem op{a.beta1, a.beta2, a.omb1, a.omb2, a.eps, e.bc2_rsqrt, s_mult, -e.step_size};
  float *p = e.param, *m = e.exp_avg, *v = e.exp_avg_sq;
  const float *g = e.grad;
  const int64_t begin = (int64_t)(c - es.chunk0[j]) * OPT_CHUNK;
  const int64_t end = min(begin + (int64_t)OPT_CHUNK, e.numel);
  int64_t i = begin;
  if (aligned16(p) && aligned16(m) && aligned16(v) && aligned16(g)) {
    const int64_t end4 = begin + ((end - begin) & ~(int64_t)3);
    for (int64_t k = begin + 4 * threadIdx.x; k < end4; k += 4 * OPT_THREADS) {
      float4 p4 = *reinterpret_cast<const float4 *>(p + k);
      float4 m4 = *reinterpret_cast<const float4 *>(m + k);
      float4 v4 = *reinterpret_cast<const float4 *>(v + k);
      float gf[4];
      load_stream(g + k).unpack(gf);
      op.run(p4.x, gf[0], m4.x, v4.x);
      op.run(p4.y, gf[1], m4.y, v4.y);
      op.run(p4.z, gf[2], m4.z, v4.z);
      op.run(p4.w, gf[3], m4.w, v4.w);
      *reinterpret_cast<float4 *>(p + k) = p4;
      *reinterpret_cast<float4 *>(m + k) = m4;
      *reinterpret_cast<float4 *>(v + k) = v4;
    }
    i = end4;
  }
  for (int64_t k = i + threadIdx.x; k < end; k += OPT_THREADS) {
    float pf = p[k], mf = m[k], vf = v[k];
    op.run(pf, g[k], mf, vf);
    p[k] = pf;
    m[k] = mf;
    v[k] = vf;
  }
}

struct SadamWs {
  float *partials, *coef;
};
SadamWs carve_sadam(void *base, int n_tensors, int n_chunks, size_t *bytes) {
  char *b = static_cast<char *>(base);
  SadamWs w;
  size_t off = 0;
  w.partials = reinterpret_cast<float *>(b + off);
  off += align_up((size_t)n_chunks * 3 * sizeof(float), 256);
  w.coef = reinterpret_cast<float *>(b + off);
  off += align_up(((size_t)n_tensors * 2 + 1) * sizeof(float), 256);
  *bytes = off;
  return w;
}

int64_t eve_chunks(const vb_eve_tensor *tensors, int n) {
  int64_t c = 0;
  for (int i = 0; i < n; ++i) c += n_chunks_of(tensors[i].numel);
  return c;
}

}  // namespace
}  // namespace vb

using namespace vb;

VB_API size_t vb_scaled_adam_workspace(int n_tensors, int n_chunks) {
  size_t bytes = 0;
  carve_sadam(nullptr, n_tensors < 0 ? 0 : n_tensors, n_chunks < 0 ? 0 : n_chunks, &bytes);
  return bytes;
}

VB_API int vb_scaled_adam_step(const vb_scaled_adam_tensor *tensors, const float *const *grads, const int32_t *chunk0,
                               const vb_scaled_adam_args *args, float *model_norms, vb_clip_state *clip,
                               void *workspace, size_t ws_bytes, vb_stream_t stream) {
  VB_CHECK_ARG(args != nullptr && tensors != nullptr && grads != nullptr && chunk0 != nullptr,
               "vb_scaled_adam_step: NULL table or args");
  const vb_scaled_adam_args &A = *args;
  const int T = A.n_tensors;
  VB_CHECK_ARG(T > 0, "vb_scaled_adam_step: n_tensors = %d", T);
  VB_CHECK_ARG(chunk0[0] == 0 && chunk0[T] == A.n_chunks, "vb_scaled_adam_step: chunk0[0] = %d, chunk0[%d] = %d != "
               "n_chunks = %d", chunk0[0], T, chunk0[T], A.n_chunks);
  // a zero-element parameter has no param_rms / scale_grads slot for sadam_coef_kernel to read and write
  for (int t = 0; t < T; ++t)
    VB_CHECK_ARG(chunk0[t + 1] > chunk0[t], "vb_scaled_adam_step: tensor %d has no elements (chunk0[%d] = %d, "
                 "chunk0[%d] = %d)", t, t, chunk0[t], t + 1, chunk0[t + 1]);
  VB_CHECK_ARG(A.size_period >= 1 && A.step >= 0, "vb_scaled_adam_step: size_period = %d, step = %d", A.size_period,
               A.step);
  VB_CHECK_ARG(A.clip_mode >= 0 && A.clip_mode <= 2, "vb_scaled_adam_step: clip_mode = %d", A.clip_mode);
  VB_CHECK_ARG(A.clip_mode == 0 || (A.clip_period >= 1 && model_norms != nullptr && clip != nullptr),
               "vb_scaled_adam_step: clipping needs clip_period >= 1, model_norms and the clip state");
  size_t need = 0;
  const SadamWs ws = carve_sadam(workspace, T, A.n_chunks, &need);
  VB_CHECK_ARG(workspace != nullptr && ws_bytes >= need, "vb_scaled_adam_step: workspace %zu < %zu bytes", ws_bytes,
               need);
  cudaStream_t st = static_cast<cudaStream_t>(stream);

  const double beta1 = A.beta1, beta2 = A.beta2;
  const int step = A.step;
  CoefArgs ca{};
  ca.n_tensors = T;
  ca.clip_mode = A.clip_mode;
  ca.clip_period = A.clip_mode ? A.clip_period : 1;
  ca.log_step = A.clip_mode >= 1 && step % ca.clip_period == 0;
  ca.norm_slot = step % ca.clip_period;
  ca.clipping_scale = A.clipping_scale;
  ca.init = A.init;
  ca.sg_slot = step % A.size_period;
  ca.size_period = A.size_period;
  ca.refresh_rms = ca.sg_slot == A.size_period - 1;
  ca.size_update = ca.refresh_rms && step > 0;
  // _size_update (optim.py:548-596), Python doubles rounded to fp32 where they meet a tensor
  const double size_lr = A.lr * A.scalar_lr_scale;
  const double beta2_corr = pow(beta2, (double)A.size_period);
  const double size_bc2 = 1.0 - pow(beta2_corr, (double)((step + 1) / A.size_period));
  ca.beta2_corr = (float)beta2_corr;
  ca.omb2_corr = (float)(1.0 - beta2_corr);
  ca.size_coef = (float)(-size_lr * pow(size_bc2, 0.5));
  ca.min_rms = (float)A.param_min_rms;
  ca.max_rms = (float)A.param_max_rms;
  ca.max_fill = (float)(-size_lr * A.size_period);
  ca.eps = (float)A.eps;
  ca.alpha_coef = (float)(-A.lr * (1.0 - beta1));

  UpdateArgs ua{};
  ua.beta1 = (float)beta1;
  ua.beta2 = (float)beta2;
  ua.omb1 = (float)(1.0 - beta1);
  ua.omb2 = (float)(1.0 - beta2);
  ua.eps = (float)A.eps;
  const double bc2 = 1.0 - pow(beta2, (double)(step - A.zero_step + 1));
  ua.bias_correct = bc2 < 0.99;
  ua.inv_bc2 = (float)(1.0 / bc2);
  ua.inv_bc2_s = 1.0f / (float)(1.0 - pow(beta2, (double)(step + 1)));
  ua.scalar_alpha = (float)(-size_lr * (1.0 - beta1));
  ua.scalar_max = (float)A.scalar_max;
  ua.size_step = ca.size_update;

  GradSlice gs;
  for (int t0 = 0; t0 < T; t0 += OPT_MAXT) {
    const int nt = T - t0 < OPT_MAXT ? T - t0 : OPT_MAXT;
    gs.t0 = t0;
    gs.nt = nt;
    for (int j = 0; j <= nt; ++j) gs.chunk0[j] = chunk0[t0 + j];
    for (int j = 0; j < nt; ++j) gs.g[j] = grads[t0 + j];
    const int blocks = chunk0[t0 + nt] - chunk0[t0];
    if (blocks == 0) continue;
    sadam_reduce_kernel<<<blocks, OPT_THREADS, 0, st>>>(tensors, gs, ws.partials);
    VB_LAUNCH_CHECK();
  }
  sadam_coef_kernel<<<1, COEF_THREADS, 0, st>>>(tensors, ws.partials, ws.coef, model_norms, clip, ca);
  VB_LAUNCH_CHECK();
  for (int t0 = 0; t0 < T; t0 += OPT_MAXT) {
    const int nt = T - t0 < OPT_MAXT ? T - t0 : OPT_MAXT;
    gs.t0 = t0;
    gs.nt = nt;
    for (int j = 0; j <= nt; ++j) gs.chunk0[j] = chunk0[t0 + j];
    for (int j = 0; j < nt; ++j) gs.g[j] = grads[t0 + j];
    const int blocks = chunk0[t0 + nt] - chunk0[t0];
    if (blocks == 0) continue;
    sadam_update_kernel<<<blocks, OPT_THREADS, 0, st>>>(tensors, gs, ws.coef, T, ua);
    VB_LAUNCH_CHECK();
  }
  return VB_OK;
}

VB_API size_t vb_eve_workspace(const vb_eve_tensor *tensors, int n_tensors) {
  if (tensors == nullptr || n_tensors <= 0) return 256;
  return align_up((size_t)eve_chunks(tensors, n_tensors) * sizeof(float), 256);
}

VB_API int vb_eve_step(const vb_eve_tensor *tensors, int n_tensors, float beta1, float beta2, float eps,
                       float weight_decay, void *workspace, size_t ws_bytes, vb_stream_t stream) {
  VB_CHECK_ARG(n_tensors >= 0 && (n_tensors == 0 || tensors != nullptr), "vb_eve_step: n_tensors = %d", n_tensors);
  if (n_tensors == 0) return VB_OK;
  const size_t need = vb_eve_workspace(tensors, n_tensors);
  VB_CHECK_ARG(workspace != nullptr && ws_bytes >= need, "vb_eve_step: workspace %zu < %zu bytes", ws_bytes, need);
  for (int i = 0; i < n_tensors; ++i)
    VB_CHECK_ARG(tensors[i].param && tensors[i].grad && tensors[i].exp_avg && tensors[i].exp_avg_sq &&
                 tensors[i].numel >= 0, "vb_eve_step: tensor %d has a NULL pointer or a negative size", i);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  EveArgs ea{beta1, beta2, 1.f - beta1, 1.f - beta2, eps, 1.f - weight_decay};
  float *partials = static_cast<float *>(workspace);
  EveSlice es;
  int64_t c = 0;
  for (int t0 = 0; t0 < n_tensors; t0 += EVE_MAXT) {
    const int nt = n_tensors - t0 < EVE_MAXT ? n_tensors - t0 : EVE_MAXT;
    es.nt = nt;
    for (int j = 0; j < nt; ++j) {
      es.e[j] = tensors[t0 + j];
      es.chunk0[j] = (int32_t)c;
      c += n_chunks_of(tensors[t0 + j].numel);
    }
    es.chunk0[nt] = (int32_t)c;
    const int blocks = es.chunk0[nt] - es.chunk0[0];
    if (blocks == 0) continue;
    eve_reduce_kernel<<<blocks, OPT_THREADS, 0, st>>>(es, partials);
    VB_LAUNCH_CHECK();
    eve_update_kernel<<<blocks, OPT_THREADS, 0, st>>>(es, partials, ea);
    VB_LAUNCH_CHECK();
  }
  return VB_OK;
}
