// Consumer kernels of the split-K decode projections (gemm_decode.cu).
//   ln_reduce_kernel: x[b,:] += bias + sum_s partials[s][b][:]   (residual add of
//   valle/modules/transformer.py:297-302, partial sums in fixed order), then
//   out16[b,:] = bf16(LayerNorm(x[b,:]))  (transformer.py:57-74) -- the activation rows of the next
//   tensor-core projection.  One warp per row, the row stays in registers.
#include "common.cuh"
#include "kernels.cuh"

namespace vb {

// one CTA (256 threads) per row: every thread owns 4 consecutive features per 1024-wide slab, sums the
// S partials with independent loads in flight, then the block reduces the LayerNorm moments.
// kPost: the post-norm of a post-LN layer (transformer.py:304-308, `x = norm(x + block(x))`): the normalised row
// replaces x[b,:] as well (with or without partials), not the pre-norm sum.
template <int kSlabs, bool kPost>
__global__ void __launch_bounds__(256)
ln_reduce_kernel(float *__restrict__ x, int64_t ldx, int B, int d, const float *__restrict__ partials, int splits,
                 int ldp, const float *__restrict__ bias, const float *__restrict__ gamma,
                 const float *__restrict__ beta, float eps, bf16 *__restrict__ out16) {
  __shared__ float red[2][8];
  pdl_launch_dependents();
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  // parameters do not depend on the previous kernel: fetch them ahead of the dependency wait
  float4 g[kSlabs], be[kSlabs], bb[kSlabs];
#pragma unroll
  for (int i = 0; i < kSlabs; ++i) {
    const int c = (i * 256 + tid) * 4;
    g[i] = be[i] = bb[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    if (c < d) {
      g[i] = *reinterpret_cast<const float4 *>(gamma + c);
      be[i] = *reinterpret_cast<const float4 *>(beta + c);
      if (partials && bias) bb[i] = *reinterpret_cast<const float4 *>(bias + c);
    }
  }
  pdl_wait();
  vb_trace(TR_LN * 2);
  float *xr = x + (int64_t)b * ldx;
  float4 v[kSlabs];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < kSlabs; ++i) {
    const int c = (i * 256 + tid) * 4;
    v[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    if (c < d) {
      v[i] = *reinterpret_cast<const float4 *>(xr + c);
      if (partials) {
        const float *p = partials + (int64_t)b * ldp + c;
        float4 a = __ldcg(reinterpret_cast<const float4 *>(p));
#pragma unroll 6
        for (int sidx = 1; sidx < splits; ++sidx) {
          const float4 t = __ldcg(reinterpret_cast<const float4 *>(p + (int64_t)sidx * 64 * ldp));
          a.x += t.x; a.y += t.y; a.z += t.z; a.w += t.w;
        }
        if (bias) {
          a.x += bb[i].x; a.y += bb[i].y; a.z += bb[i].z; a.w += bb[i].w;
        }
        v[i].x += a.x; v[i].y += a.y; v[i].z += a.z; v[i].w += a.w;
        if constexpr (!kPost) *reinterpret_cast<float4 *>(xr + c) = v[i];
      }
      s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
    }
  }
  s = warp_sum(s);
  if (lane == 0) red[0][warp] = s;
  __syncthreads();
  float tot = 0.f;
#pragma unroll
  for (int w = 0; w < 8; ++w) tot += red[0][w];
  const float mean = tot / (float)d;
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < kSlabs; ++i) {
    const int c = (i * 256 + tid) * 4;
    if (c < d) {
      const float a = v[i].x - mean, bq = v[i].y - mean, e = v[i].z - mean, f = v[i].w - mean;
      q += (a * a + bq * bq) + (e * e + f * f);
    }
  }
  q = warp_sum(q);
  if (lane == 0) red[1][warp] = q;
  __syncthreads();
  float qt = 0.f;
#pragma unroll
  for (int w = 0; w < 8; ++w) qt += red[1][w];
  const float rstd = rsqrtf(qt / (float)d + eps);
  bf16 *orow = out16 + (int64_t)b * d;
#pragma unroll
  for (int i = 0; i < kSlabs; ++i) {
    const int c = (i * 256 + tid) * 4;
    if (c < d) {
      const float y0 = (v[i].x - mean) * rstd * g[i].x + be[i].x, y1 = (v[i].y - mean) * rstd * g[i].y + be[i].y;
      const float y2 = (v[i].z - mean) * rstd * g[i].z + be[i].z, y3 = (v[i].w - mean) * rstd * g[i].w + be[i].w;
      if constexpr (kPost) *reinterpret_cast<float4 *>(xr + c) = make_float4(y0, y1, y2, y3);
      __nv_bfloat162 p0 = __floats2bfloat162_rn(y0, y1);
      __nv_bfloat162 p1 = __floats2bfloat162_rn(y2, y3);
      uint2 pk;
      pk.x = *reinterpret_cast<uint32_t *>(&p0);
      pk.y = *reinterpret_cast<uint32_t *>(&p1);
      *reinterpret_cast<uint2 *>(orow + c) = pk;
    }
  }
  vb_trace(TR_LN * 2 + 1);
}

// out16[b, n] = bf16(relu(bias[n] + sum_s partials[s][b][n]))  -- FFN hidden activation
// (valle/modules/transformer.py:332-334: linear1 -> ReLU), input rows of the linear2 projection.
__global__ void __launch_bounds__(256)
relu_reduce_kernel(const float *__restrict__ partials, int splits, int ldp, const float *__restrict__ bias, int N,
                   bf16 *__restrict__ out16, int64_t ldo, LnFoldStats fold) {
  pdl_launch_dependents();
  const int b = blockIdx.y;
  const int c = (blockIdx.x * 256 + threadIdx.x) * 4;
  const float4 bb = c < N ? *reinterpret_cast<const float4 *>(bias + c) : make_float4(0.f, 0.f, 0.f, 0.f);  // ahead of the wait
  float4 cc = make_float4(0.f, 0.f, 0.f, 0.f);
  if (fold.stats && c < N) cc = *reinterpret_cast<const float4 *>(fold.c + c);
  pdl_wait();
  vb_trace(TR_RELU * 2);
  // (whole warps: no early exit ahead of the shuffles; the pair is in flight together with the partial sums below)
  float2 mraw = make_float2(0.f, 0.f);
  if (fold.stats) mraw = ln_fold_moments_load(fold, b, blockIdx.x * 8 + (threadIdx.x >> 5));
  const bool live = c < N;
  const float *p = partials + (int64_t)b * ldp + (live ? c : 0);
  // every split's slab requested before the first add: ONE L2 round trip (a loop with a run-time trip count ends up as
  // one dependent round trip per split in its remainder iterations)
  float4 t[8];
#pragma unroll
  for (int s = 0; s < 8; ++s)
    t[s] = s < splits ? __ldcg(reinterpret_cast<const float4 *>(p + (int64_t)s * 64 * ldp)) : make_float4(0.f, 0.f, 0.f, 0.f);
  float4 a = t[0];
#pragma unroll
  for (int s = 1; s < 8; ++s) {   // fixed order 0..S-1 (the tail adds exact zeros)
    a.x += t[s].x; a.y += t[s].y; a.z += t[s].z; a.w += t[s].w;
  }
  for (int s = 8; s < splits; ++s) {
    const float4 u = __ldcg(reinterpret_cast<const float4 *>(p + (int64_t)s * 64 * ldp));
    a.x += u.x; a.y += u.y; a.z += u.z; a.w += u.w;
  }
  float mean = 0.f, rstd = 1.f;
  if (fold.stats) ln_fold_moments_finish(fold, mraw, mean, rstd);
  if (!live) return;
  if (fold.stats) {  // LayerNorm folded into linear1: relu(rstd (x W'^T - mean c) + bias')
    a.x = rstd * (a.x - mean * cc.x); a.y = rstd * (a.y - mean * cc.y);
    a.z = rstd * (a.z - mean * cc.z); a.w = rstd * (a.w - mean * cc.w);
  }
  __nv_bfloat162 p0 = __floats2bfloat162_rn(fmaxf(a.x + bb.x, 0.f), fmaxf(a.y + bb.y, 0.f));
  __nv_bfloat162 p1 = __floats2bfloat162_rn(fmaxf(a.z + bb.z, 0.f), fmaxf(a.w + bb.w, 0.f));
  uint2 pk;
  pk.x = *reinterpret_cast<uint32_t *>(&p0);
  pk.y = *reinterpret_cast<uint32_t *>(&p1);
  *reinterpret_cast<uint2 *>(out16 + (int64_t)b * ldo + c) = pk;
}

int launch_relu_reduce(const SplitK &in, int B, int N, bf16 *out16, int64_t ldo, bool pdl, cudaStream_t s) {
  VB_CHECK_ARG(N % 4 == 0 && ldo % 4 == 0, "relu_reduce: N %% 4 != 0");
  VB_CUDA(launch_kernel(relu_reduce_kernel, dim3((N / 4 + 255) / 256, B), dim3(256), 0, s, pdl, in.part, in.splits,
                        in.ldp, in.bias, N, out16, ldo, in.fold));
  count_launch();
  return VB_OK;
}

template <bool kPost>
static int launch_ln_reduce_t(float *x, int64_t ldx, int B, int d, const float *partials, int splits, int ldp,
                              const float *bias, const float *gamma, const float *beta, float eps, bf16 *out16,
                              bool pdl, cudaStream_t s) {
  VB_CHECK_ARG(d % 4 == 0 && ldx % 4 == 0 && d <= 4096, "ln_reduce: bad d=%d", d);
  const dim3 grid(B), block(256);
  const int slabs = (d + 1023) / 1024;
  if (slabs <= 1)
    VB_CUDA(launch_kernel(ln_reduce_kernel<1, kPost>, grid, block, 0, s, pdl, x, ldx, B, d, partials, splits, ldp, bias,
                          gamma, beta, eps, out16));
  else if (slabs <= 2)
    VB_CUDA(launch_kernel(ln_reduce_kernel<2, kPost>, grid, block, 0, s, pdl, x, ldx, B, d, partials, splits, ldp, bias,
                          gamma, beta, eps, out16));
  else
    VB_CUDA(launch_kernel(ln_reduce_kernel<4, kPost>, grid, block, 0, s, pdl, x, ldx, B, d, partials, splits, ldp, bias,
                          gamma, beta, eps, out16));
  count_launch();
  return VB_OK;
}

int launch_ln_reduce(float *x, int64_t ldx, int B, int d, const SplitK &in, const float *gamma, const float *beta,
                     float eps, bf16 *out16, bool pdl, cudaStream_t s, bool post) {
  const auto launch = post ? launch_ln_reduce_t<true> : launch_ln_reduce_t<false>;
  return launch(x, ldx, B, d, in.part, in.splits, in.ldp, in.bias, gamma, beta, eps, out16, pdl, s);
}

}  // namespace vb
