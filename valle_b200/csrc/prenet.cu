// Text pre-net training (valle/models/valle.py:96-123,181-213): BatchNorm1d over the Conv1d(k=5, 'same') output with
// batch statistics, ReLU and Dropout(0.5), forward and backward, and the im2col / col2im of the convolution.
//
// Geometry: rows are the padded text batch, utterance after utterance, `seg_len` rows each (M = N * seg_len), C
// channels.  The convolutions are vb_linear over an im2col operand [M, 5C] whose column block k holds row
// r + k - 2 of the same utterance (zero outside it: padding="same"), with the shift-major weight [Cout, 5 Cin].
//
// Reductions: one CTA per (32 columns, kRows rows) writes its partial column statistics to the workspace; every CTA of
// the following kernel adds the partials of its columns in block order 0..nblk-1 (the same order in every CTA), so
// the results do not depend on scheduling: no atomics, the same bits in every run.
//
// Accuracy when |mean| >> sigma: the batch statistics are taken of h - s, with the shift s = h[0, c] (a value of the
// channel, so h - s is of the size of sigma and exact in fp32), and combined as (count, mean, sum of squared deviations
// from the block mean) pairs (Chan et al.).  The mean is kept relative to s: xhat = ((h - s) - mean_s) * rstd never
// forms the fp32 mean itself, whose rounding alone would shift xhat by |mean| / sigma * 2^-24.
#include <algorithm>

#include "kernels.cuh"

namespace vb {
namespace pn {

constexpr int kRows = 64;  // rows per statistics block
constexpr int kTy = 8;     // thread rows of a 32 x 8 CTA

struct BnCfg {
  const float *gamma, *beta;  // NULL: no BatchNorm / ReLU / dropout (plain im2col or col2im)
  const float *mean, *rstd;   // per channel, written by bn_apply_kernel: mean - shift, 1 / sqrt(var + eps)
  DropCfg drop;
};

// shift of channel c: h[0, c] with batch statistics, 0 with the running ones
__device__ __forceinline__ float bn_shift(const float *__restrict__ h, int training, int c) {
  return training ? h[c] : 0.f;
}

// y[r, c] of the block output: dropout(relu(gamma * ((h - shift) - mean) * rstd + beta)), mask index r * C + c
__device__ __forceinline__ float bn_act(const BnCfg &b, float h, float shift, float mean, float rstd, float g,
                                        float be, int64_t r, int C, int c) {
  const float z = fmaf(g, ((h - shift) - mean) * rstd, be);
  if (!(z > 0.f)) return 0.f;
  if (b.drop.thresh == 0) return z;
  return drop_keep(b.drop, (uint64_t)(r * C + c)) ? z * b.drop.inv_keep : 0.f;
}

// ---- forward statistics: partial (mean of h - shift, M2) of block blockIdx.y over columns [32 bx, 32 bx + 32) ------
__global__ void __launch_bounds__(256) bn_stats_kernel(const float *__restrict__ h, int64_t M, int C,
                                                       float2 *__restrict__ part) {
  __shared__ float red[kTy][33];
  __shared__ float bmean[32];
  const int tx = threadIdx.x, ty = threadIdx.y;
  const int c = blockIdx.x * 32 + tx;
  const int64_t r0 = (int64_t)blockIdx.y * kRows, r1 = min(M, r0 + kRows);
  const float cnt = (float)(r1 - r0);
  const float sh = bn_shift(h, 1, c);
  float s = 0.f;
  for (int64_t r = r0 + ty; r < r1; r += kTy) s += h[r * C + c] - sh;
  red[ty][tx] = s;
  __syncthreads();
  if (ty == 0) {
    float t = 0.f;
#pragma unroll
    for (int i = 0; i < kTy; ++i) t += red[i][tx];
    bmean[tx] = t / cnt;
  }
  __syncthreads();
  const float mu = bmean[tx];
  float q = 0.f;
  for (int64_t r = r0 + ty; r < r1; r += kTy) {
    const float e = (h[r * C + c] - sh) - mu;
    q = fmaf(e, e, q);
  }
  __syncthreads();
  red[ty][tx] = q;
  __syncthreads();
  if (ty == 0) {
    float t = 0.f;
#pragma unroll
    for (int i = 0; i < kTy; ++i) t += red[i][tx];
    part[(int64_t)blockIdx.y * C + c] = make_float2(mu, t);
  }
}

// ---- forward apply: statistics of the CTA's columns (partials combined in block order), running-statistics update by
// the CTAs of row block 0, then out[r, k C + c] = y[r + k - 2, c] (taps 5, zero outside the utterance) or y[r, c]
// (taps 1) in TO.  gamma == NULL: y = h (the im2col of the first convolution's input).
template <typename TO>
__global__ void __launch_bounds__(256)
bn_apply_kernel(const float *__restrict__ h, int64_t M, int C, int seg_len, int taps, BnCfg b,
                const float2 *__restrict__ part, int nblk, int training, float *running_mean, float *running_var,
                float eps, float momentum, float *save_mean, float *save_rstd, TO *__restrict__ out) {
  __shared__ float s_mean[32], s_rstd[32], s_g[32], s_b[32], s_sh[32];
  const int tx = threadIdx.x, ty = threadIdx.y;
  const int c = blockIdx.x * 32 + tx;
  if (b.gamma != nullptr && ty == 0) {
    float mean, rstd;
    if (training) {
      float n_a = 0.f, mean_a = 0.f, m2_a = 0.f;   // counts below 2^24 are exact in fp32
      for (int i = 0; i < nblk; ++i) {
        const float2 p = part[(int64_t)i * C + c];
        const float n_b = (float)(min(M, (int64_t)(i + 1) * kRows) - (int64_t)i * kRows);
        const float n_ab = n_a + n_b;
        const float delta = p.x - mean_a;
        mean_a = fmaf(delta, n_b / n_ab, mean_a);
        m2_a = m2_a + p.y + delta * delta * (n_a * n_b / n_ab);
        n_a = n_ab;
      }
      const float var = m2_a / (float)M;
      mean = mean_a;
      rstd = rsqrtf(var + eps);
      if (blockIdx.y == 0) {
        running_mean[c] = (1.f - momentum) * running_mean[c] + momentum * (bn_shift(h, 1, c) + mean);
        running_var[c] = (1.f - momentum) * running_var[c] + momentum * (m2_a / (float)(M - 1));
      }
    } else {
      mean = running_mean[c];
      rstd = rsqrtf(running_var[c] + eps);
    }
    s_mean[tx] = mean;
    s_rstd[tx] = rstd;
    s_sh[tx] = bn_shift(h, training, c);
    s_g[tx] = b.gamma[c];
    s_b[tx] = b.beta[c];
    if (blockIdx.y == 0) {
      save_mean[c] = mean;
      save_rstd[c] = rstd;
    }
  }
  __syncthreads();
  const int64_t r0 = (int64_t)blockIdx.y * kRows, r1 = min(M, r0 + kRows);
  const float mean = b.gamma ? s_mean[tx] : 0.f, rstd = b.gamma ? s_rstd[tx] : 1.f;
  const float g = b.gamma ? s_g[tx] : 1.f, be = b.gamma ? s_b[tx] : 0.f, shift = b.gamma ? s_sh[tx] : 0.f;
  const int64_t ldo = (int64_t)taps * C;
  for (int64_t r = r0 + ty; r < r1; r += kTy) {
    const int pos = (int)(r % seg_len);
    for (int k = 0; k < taps; ++k) {
      const int sh = taps == 1 ? 0 : k - 2;
      float v = 0.f;
      if (pos + sh >= 0 && pos + sh < seg_len) {
        const int64_t rs = r + sh;
        const float x = h[rs * C + c];
        v = b.gamma ? bn_act(b, x, shift, mean, rstd, g, be, rs, C, c) : x;
      }
      out[r * ldo + (int64_t)k * C + c] = from_f32<TO>(v);
    }
  }
}

// gradient w.r.t. y[r, c]: the col2im sum over the taps in fixed order k = 0..4 (row r feeds out[r - k + 2, k C + c])
__device__ __forceinline__ float col2im_load(const float *__restrict__ dy, int64_t r, int C, int c, int seg_len,
                                             int taps) {
  if (taps == 1) return dy[r * C + c];
  const int pos = (int)(r % seg_len);
  const int64_t ld = 5ll * C;
  float s = 0.f;
#pragma unroll
  for (int k = 0; k < 5; ++k) {
    const int p = pos - k + 2;
    if (p >= 0 && p < seg_len) s += dy[(r - k + 2) * ld + (int64_t)k * C + c];
  }
  return s;
}

// dL/dz of z = gamma * xhat + beta (through the dropout mask and the ReLU gate), and xhat
__device__ __forceinline__ float bn_grad_z(const BnCfg &b, float gy, float h, float shift, float mean, float rstd,
                                           float g, float be, int64_t r, int C, int c, float &xhat) {
  xhat = ((h - shift) - mean) * rstd;
  const float z = fmaf(g, xhat, be);
  if (!(z > 0.f)) return 0.f;
  if (b.drop.thresh == 0) return gy;
  return drop_keep(b.drop, (uint64_t)(r * C + c)) ? gy * b.drop.inv_keep : 0.f;
}

// ---- backward partials: per block, sum gz, sum gz * xhat, sum xhat ------------------------------------------------
__global__ void __launch_bounds__(256)
bn_bwd_stats_kernel(const float *__restrict__ dy, int taps, const float *__restrict__ h, int64_t M, int C, int seg_len,
                    BnCfg b, int training, float4 *__restrict__ part) {
  __shared__ float red[3][kTy][33];
  const int tx = threadIdx.x, ty = threadIdx.y;
  const int c = blockIdx.x * 32 + tx;
  const float mean = b.mean[c], rstd = b.rstd[c], g = b.gamma[c], be = b.beta[c], shift = bn_shift(h, training, c);
  const int64_t r0 = (int64_t)blockIdx.y * kRows, r1 = min(M, r0 + kRows);
  float sg = 0.f, sgx = 0.f, sx = 0.f;
  for (int64_t r = r0 + ty; r < r1; r += kTy) {
    float xh;
    const float gz = bn_grad_z(b, col2im_load(dy, r, C, c, seg_len, taps), h[r * C + c], shift, mean, rstd, g, be, r, C, c,
                               xh);
    sg += gz;
    sgx = fmaf(gz, xh, sgx);
    sx += xh;
  }
  red[0][ty][tx] = sg;
  red[1][ty][tx] = sgx;
  red[2][ty][tx] = sx;
  __syncthreads();
  if (ty == 0) {
    float a = 0.f, e = 0.f, f = 0.f;
#pragma unroll
    for (int i = 0; i < kTy; ++i) {
      a += red[0][i][tx];
      e += red[1][i][tx];
      f += red[2][i][tx];
    }
    part[(int64_t)blockIdx.y * C + c] = make_float4(a, e, f, 0.f);
  }
}

// ---- backward apply: dh = gamma rstd (gz - training (sum gz + xhat sum gz xhat) / M) in TO; the CTAs of row block 0
// write dgamma = sum gz xhat, dbeta = sum gz and the conv bias gradient sum_r dh (exact column sum of the formula).
// gamma == NULL: dh = the col2im of dy (gradient w.r.t. the first convolution's input).
template <typename TO>
__global__ void __launch_bounds__(256)
bn_bwd_apply_kernel(const float *__restrict__ dy, int taps, const float *__restrict__ h, int64_t M, int C, int seg_len,
                    BnCfg b, const float4 *__restrict__ part, int nblk, int training, float *dgamma, float *dbeta,
                    float *dbias, TO *__restrict__ dh) {
  __shared__ float s_sg[32], s_sgx[32];
  const int tx = threadIdx.x, ty = threadIdx.y;
  const int c = blockIdx.x * 32 + tx;
  float mean = 0.f, rstd = 1.f, g = 1.f, be = 0.f, shift = 0.f;
  if (b.gamma != nullptr) {
    shift = bn_shift(h, training, c);
    mean = b.mean[c];
    rstd = b.rstd[c];
    g = b.gamma[c];
    be = b.beta[c];
    if (ty == 0) {
      float sg = 0.f, sgx = 0.f, sx = 0.f;
      for (int i = 0; i < nblk; ++i) {
        const float4 p = part[(int64_t)i * C + c];
        sg += p.x;
        sgx += p.y;
        sx += p.z;
      }
      s_sg[tx] = sg;
      s_sgx[tx] = sgx;
      if (blockIdx.y == 0) {
        if (dgamma) dgamma[c] = sgx;
        if (dbeta) dbeta[c] = sg;
        if (dbias)
          dbias[c] = training ? -g * rstd * sx * sgx / (float)M : g * rstd * sg;
      }
    }
    __syncthreads();
  }
  const float inv_n = 1.f / (float)M;
  const float sg = b.gamma ? s_sg[tx] : 0.f, sgx = b.gamma ? s_sgx[tx] : 0.f;
  const int64_t r0 = (int64_t)blockIdx.y * kRows, r1 = min(M, r0 + kRows);
  for (int64_t r = r0 + ty; r < r1; r += kTy) {
    const float gy = col2im_load(dy, r, C, c, seg_len, taps);
    float v = gy;
    if (b.gamma) {
      float xh;
      const float gz = bn_grad_z(b, gy, h[r * C + c], shift, mean, rstd, g, be, r, C, c, xh);
      v = training ? g * rstd * (gz - (sg + xh * sgx) * inv_n) : g * rstd * gz;
    }
    dh[r * C + c] = from_f32<TO>(v);
  }
}

// ---- audio pre-net: dz = keep(i) && h[i] > 0 ? dy[i] / (1 - p) : 0 (Dropout after a ReLU, backward) -----------------
template <typename T>
__global__ void relu_dropout_bwd_kernel(const T *__restrict__ dy, const T *__restrict__ h, T *__restrict__ dz,
                                        int64_t n, DropCfg cfg) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    float v = 0.f;
    if (to_f32(h[i]) > 0.f && (cfg.thresh == 0 || drop_keep(cfg, (uint64_t)i)))
      v = cfg.thresh == 0 ? to_f32(dy[i]) : to_f32(dy[i]) * cfg.inv_keep;
    dz[i] = from_f32<T>(v);
  }
}

}  // namespace pn
}  // namespace vb

using namespace vb;

static int bn_geometry(const char *who, int64_t M, int C, int seg_len, int taps) {
  VB_CHECK_ARG(M > 0 && C > 0 && C % 32 == 0, "%s: bad shape M=%lld C=%d (C must be a multiple of 32)", who,
               (long long)M, C);
  VB_CHECK_ARG(seg_len > 0 && M % seg_len == 0, "%s: M=%lld is not a multiple of seg_len=%d", who, (long long)M,
               seg_len);
  VB_CHECK_ARG(taps == 1 || taps == 5, "%s: taps=%d not in {1, 5}", who, taps);
  return VB_OK;
}

VB_API size_t vb_batchnorm_workspace(int64_t M, int C) {
  return (size_t)((M + pn::kRows - 1) / pn::kRows) * C * sizeof(float4) + 256;
}

VB_API int vb_batchnorm_forward(const float *h, int64_t M, int C, int seg_len, const float *gamma, const float *beta,
                                float *running_mean, float *running_var, float eps, float momentum, int training,
                                float *save_mean, float *save_rstd, float dropout_p, uint64_t dropout_seed,
                                uint32_t dropout_stream, void *out, int out_dtype, int taps, void *workspace,
                                size_t workspace_bytes, vb_stream_t stream) {
  VB_TRY(bn_geometry("vb_batchnorm_forward", M, C, seg_len, taps));
  VB_CHECK_ARG(h && out && (out_dtype == VB_F32 || out_dtype == VB_BF16), "vb_batchnorm_forward: bad argument");
  VB_CHECK_ARG(dropout_p >= 0.f && dropout_p < 1.f, "vb_batchnorm_forward: dropout_p=%g not in [0, 1)",
               (double)dropout_p);
  const int nblk = (int)((M + pn::kRows - 1) / pn::kRows);
  pn::BnCfg b{gamma, beta, nullptr, nullptr, make_drop(dropout_p, dropout_seed, dropout_stream)};
  cudaStream_t s = (cudaStream_t)stream;
  const dim3 block(32, pn::kTy), grid((unsigned)(C / 32), (unsigned)nblk);
  if (gamma) {
    VB_CHECK_ARG(beta && running_mean && running_var && save_mean && save_rstd,
                 "vb_batchnorm_forward: gamma needs beta, the running statistics and the save buffers");
    if (training) {
      VB_CHECK_ARG(M > 1, "vb_batchnorm_forward: expected more than 1 value per channel when training (M=%lld)",
                   (long long)M);
      VB_CHECK_ARG(workspace && workspace_bytes >= vb_batchnorm_workspace(M, C),
                   "vb_batchnorm_forward: workspace too small");
      pn::bn_stats_kernel<<<grid, block, 0, s>>>(h, M, C, (float2 *)workspace);
      VB_LAUNCH_CHECK();
    }
  }
  if (out_dtype == VB_F32)
    pn::bn_apply_kernel<float><<<grid, block, 0, s>>>(h, M, C, seg_len, taps, b, (const float2 *)workspace, nblk,
                                                      training, running_mean, running_var, eps, momentum, save_mean,
                                                      save_rstd, (float *)out);
  else
    pn::bn_apply_kernel<bf16><<<grid, block, 0, s>>>(h, M, C, seg_len, taps, b, (const float2 *)workspace, nblk,
                                                     training, running_mean, running_var, eps, momentum, save_mean,
                                                     save_rstd, (bf16 *)out);
  VB_LAUNCH_CHECK();
  return VB_OK;
}

VB_API int vb_batchnorm_backward(const float *dy, int taps, const float *h, int64_t M, int C, int seg_len,
                                 const float *gamma, const float *beta, const float *save_mean, const float *save_rstd,
                                 int training, float dropout_p, uint64_t dropout_seed, uint32_t dropout_stream,
                                 void *dh, int dh_dtype, float *dgamma, float *dbeta, float *dbias, void *workspace,
                                 size_t workspace_bytes, vb_stream_t stream) {
  VB_TRY(bn_geometry("vb_batchnorm_backward", M, C, seg_len, taps));
  VB_CHECK_ARG(dy && dh && (dh_dtype == VB_F32 || dh_dtype == VB_BF16), "vb_batchnorm_backward: bad argument");
  VB_CHECK_ARG(dropout_p >= 0.f && dropout_p < 1.f, "vb_batchnorm_backward: dropout_p=%g not in [0, 1)",
               (double)dropout_p);
  const int nblk = (int)((M + pn::kRows - 1) / pn::kRows);
  pn::BnCfg b{gamma, beta, save_mean, save_rstd, make_drop(dropout_p, dropout_seed, dropout_stream)};
  cudaStream_t s = (cudaStream_t)stream;
  const dim3 block(32, pn::kTy), grid((unsigned)(C / 32), (unsigned)nblk);
  if (gamma) {
    VB_CHECK_ARG(h && beta && save_mean && save_rstd, "vb_batchnorm_backward: gamma needs h, beta and the statistics");
    VB_CHECK_ARG(!training || M > 1, "vb_batchnorm_backward: M=%lld", (long long)M);
    VB_CHECK_ARG(workspace && workspace_bytes >= vb_batchnorm_workspace(M, C),
                 "vb_batchnorm_backward: workspace too small");
    pn::bn_bwd_stats_kernel<<<grid, block, 0, s>>>(dy, taps, h, M, C, seg_len, b, training, (float4 *)workspace);
    VB_LAUNCH_CHECK();
  }
  if (dh_dtype == VB_F32)
    pn::bn_bwd_apply_kernel<float><<<grid, block, 0, s>>>(dy, taps, h, M, C, seg_len, b, (const float4 *)workspace,
                                                          nblk, training, dgamma, dbeta, dbias, (float *)dh);
  else
    pn::bn_bwd_apply_kernel<bf16><<<grid, block, 0, s>>>(dy, taps, h, M, C, seg_len, b, (const float4 *)workspace,
                                                         nblk, training, dgamma, dbeta, dbias, (bf16 *)dh);
  VB_LAUNCH_CHECK();
  return VB_OK;
}

VB_API int vb_relu_dropout_backward(const void *dy, const void *h, void *dz, int dtype, int64_t n, float dropout_p,
                                    uint64_t dropout_seed, uint32_t dropout_stream, vb_stream_t stream) {
  VB_CHECK_ARG(dy && h && dz && (dtype == VB_F32 || dtype == VB_BF16), "vb_relu_dropout_backward: bad argument");
  VB_CHECK_ARG(dropout_p >= 0.f && dropout_p < 1.f, "vb_relu_dropout_backward: dropout_p=%g not in [0, 1)",
               (double)dropout_p);
  if (n == 0) return VB_OK;
  const DropCfg cfg = make_drop(dropout_p, dropout_seed, dropout_stream);
  const unsigned grid = (unsigned)std::min<int64_t>((n + 255) / 256, 132 * 16);
  cudaStream_t s = (cudaStream_t)stream;
  if (dtype == VB_F32)
    pn::relu_dropout_bwd_kernel<float><<<grid, 256, 0, s>>>((const float *)dy, (const float *)h, (float *)dz, n, cfg);
  else
    pn::relu_dropout_bwd_kernel<bf16><<<grid, 256, 0, s>>>((const bf16 *)dy, (const bf16 *)h, (bf16 *)dz, n, cfg);
  VB_LAUNCH_CHECK();
  return VB_OK;
}
