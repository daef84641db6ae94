// CUDA-core (FFMA) linear layers:
//   * gemm_simt_kernel : C[M,N] = epi(A[M,K] W[N,K]^T + b), fp32 accumulate in fixed k order.
//     This is the exact-order path used for fp32 parity (greedy tokens bit-exact vs the
//     reference) and for shapes the wgmma kernel does not take (N=1025 head, tiny K).
//   * gemv_kernel      : skinny M (decode rows, M<=64), weight-streaming, HBM-bound.  One warp
//     per output column, 16-byte streaming loads of W, activations (optionally LayerNorm'ed in
//     the prologue) staged in shared memory, warp-shuffle reduction.
//
// Reference arithmetic: F.linear at valle/modules/transformer.py:332-334 (FFN),
// valle/modules/activation.py:408 (packed in-proj / out-proj), valle/models/valle.py:1039,1128
// (predict layers); residual adds transformer.py:297-302.
#include "common.cuh"
#include "kernels.cuh"

namespace vb {

// ------------------------------------------------------------------------------------------
// Tiled SIMT GEMM.  64x64 tile, BK=16, 256 threads, 4x4 micro-tile.
// ------------------------------------------------------------------------------------------
template <typename T> __device__ __forceinline__ void load4(const T *p, float (&f)[4]);
template <> __device__ __forceinline__ void load4<float>(const float *p, float (&f)[4]) {
  const float4 v = *reinterpret_cast<const float4 *>(p);
  f[0] = v.x; f[1] = v.y; f[2] = v.z; f[3] = v.w;
}
template <> __device__ __forceinline__ void load4<bf16>(const bf16 *p, float (&f)[4]) {
  const uint2 v = *reinterpret_cast<const uint2 *>(p);
  f[0] = __uint_as_float(v.x << 16);
  f[1] = __uint_as_float(v.x & 0xffff0000u);
  f[2] = __uint_as_float(v.y << 16);
  f[3] = __uint_as_float(v.y & 0xffff0000u);
}

template <typename TA, typename TC, int kEpi>
__global__ void __launch_bounds__(256)
gemm_simt_kernel(const TA *__restrict__ A, int64_t lda, const TA *__restrict__ W,
                 const float *__restrict__ bias, TC *__restrict__ C, int64_t ldc, int64_t M, int N,
                 int K) {
  constexpr int BM = 64, BN = 64, BK = 16;
  __shared__ __align__(16) float As[BK][BM + 4];
  __shared__ __align__(16) float Ws[BK][BN + 4];
  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;
  const int64_t m0 = (int64_t)blockIdx.y * BM;
  const int n0 = blockIdx.x * BN;
  // loader mapping: thread -> (row = tid/4, k4 = (tid%4)*4)
  const int lrow = tid >> 2, lk = (tid & 3) * 4;
  const int64_t am = m0 + lrow;
  const int wn = n0 + lrow;
  const TA *ap = A + (am < M ? am : 0) * lda + lk;
  const TA *wp = W + (int64_t)(wn < N ? wn : 0) * K + lk;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  float ra[4], rw[4];
  load4<TA>(ap, ra);
  load4<TA>(wp, rw);
  for (int k0 = 0; k0 < K; k0 += BK) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      As[lk + i][lrow] = (am < M) ? ra[i] : 0.f;
      Ws[lk + i][lrow] = (wn < N) ? rw[i] : 0.f;
    }
    __syncthreads();
    if (k0 + BK < K) {  // prefetch next slab into registers
      load4<TA>(ap + k0 + BK, ra);
      load4<TA>(wp + k0 + BK, rw);
    }
#pragma unroll
    for (int k = 0; k < BK; ++k) {
      const float4 a = *reinterpret_cast<const float4 *>(&As[k][ty * 4]);
      const float4 w = *reinterpret_cast<const float4 *>(&Ws[k][tx * 4]);
      const float av[4] = {a.x, a.y, a.z, a.w};
      const float wv[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], wv[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int64_t m = m0 + ty * 4 + i;
    if (m >= M) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int n = n0 + tx * 4 + j;
      if (n >= N) continue;
      float v = acc[i][j];
      if (bias) v += bias[n];
      TC *cp = C + m * ldc + n;
      if constexpr (kEpi == VB_EPI_RELU) v = fmaxf(v, 0.f);
      if constexpr (kEpi == VB_EPI_RESIDUAL) v = to_f32(*cp) + v;
      *cp = from_f32<TC>(v);
    }
  }
}

template <typename TA, typename TC>
static int launch_gemm_simt_t(const TA *A, int64_t lda, const TA *W, const float *bias, TC *C,
                              int64_t ldc, int64_t M, int N, int K, int epi, cudaStream_t s) {
  dim3 grid((N + 63) / 64, (unsigned)((M + 63) / 64));
  if (epi == VB_EPI_NONE)
    gemm_simt_kernel<TA, TC, VB_EPI_NONE><<<grid, 256, 0, s>>>(A, lda, W, bias, C, ldc, M, N, K);
  else if (epi == VB_EPI_RELU)
    gemm_simt_kernel<TA, TC, VB_EPI_RELU><<<grid, 256, 0, s>>>(A, lda, W, bias, C, ldc, M, N, K);
  else
    gemm_simt_kernel<TA, TC, VB_EPI_RESIDUAL><<<grid, 256, 0, s>>>(A, lda, W, bias, C, ldc, M, N, K);
  VB_LAUNCH_CHECK();
  return VB_OK;
}

int launch_gemm_simt(const void *A, int a_dtype, int64_t lda, const void *W, const float *bias, void *C,
                     int c_dtype, int64_t ldc, int64_t M, int N, int K, int epi, cudaStream_t s) {
  VB_CHECK_ARG(K % 16 == 0, "gemm_simt: K=%d must be a multiple of 16", K);
  VB_CHECK_ARG(lda % 4 == 0, "gemm_simt: lda must be a multiple of 4");
  if (M == 0) return VB_OK;
  if (epi == VB_EPI_RESIDUAL) VB_CHECK_ARG(c_dtype == VB_F32, "gemm: residual epilogue needs fp32 C");
  if (a_dtype == VB_F32 && c_dtype == VB_F32)
    return launch_gemm_simt_t<float, float>((const float *)A, lda, (const float *)W, bias, (float *)C, ldc, M, N, K, epi, s);
  if (a_dtype == VB_BF16 && c_dtype == VB_F32)
    return launch_gemm_simt_t<bf16, float>((const bf16 *)A, lda, (const bf16 *)W, bias, (float *)C, ldc, M, N, K, epi, s);
  if (a_dtype == VB_BF16 && c_dtype == VB_BF16)
    return launch_gemm_simt_t<bf16, bf16>((const bf16 *)A, lda, (const bf16 *)W, bias, (bf16 *)C, ldc, M, N, K, epi, s);
  set_error("gemm_simt: unsupported dtype combination a=%d c=%d", a_dtype, c_dtype);
  return VB_ERR_UNSUPPORTED;
}

// ------------------------------------------------------------------------------------------
// Skinny GEMV for decode rows.
//   out[b, n] = epi( sum_k xin[b,k] * W[n,k] + bias[n] ),  b < B (processed in chunks of BT rows)
//   xin = x or LayerNorm(x) (prologue, per CTA, from L2-resident rows)
// Shared-memory layout of the activation rows: 16-byte groups of a row are stored so that the
// float4 reads of consecutive lanes are contiguous (bank-conflict free) for both fp32 weights
// (lane owns 4 k) and bf16 weights (lane owns 8 k = two groups).
// ------------------------------------------------------------------------------------------
template <int VEC> __device__ __forceinline__ int xs_phys(int k, int K) {
  if constexpr (VEC == 4) return k;
  // VEC == 8: even 4-groups in the first half, odd groups in the second half
  return ((k >> 2) & 1) * (K >> 1) + ((k >> 3) << 2) + (k & 3);
}

struct GemvEpi {
  int mode;  // 0 none, 1 relu, 2 residual (out += ), 3 qkv-scatter
  QkvScatter qkv;  // mode 3: n in [0,d) -> q[b,n]; [d,2d) -> the K cache; [2d,3d) -> the V cache
};

template <typename TW, int BT, int NPW>
__global__ void __launch_bounds__(512)
gemv_kernel(const float *__restrict__ x, int64_t ldx, int B, const TW *__restrict__ W,
            const float *__restrict__ bias, int N, int K, float *__restrict__ out, int64_t ldo,
            const float *__restrict__ ln_g, const float *__restrict__ ln_b,
            const float *__restrict__ ada_wb, float eps, GemvEpi epi) {
  constexpr int VEC = Vec16<TW>::N;
  extern __shared__ __align__(16) float xs[];  // [BT][K]
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int nwarps = blockDim.x >> 5;
  const int gw = blockIdx.x * nwarps + warp;
  const int GW = gridDim.x * nwarps;

  for (int b0 = 0; b0 < B; b0 += BT) {
    const int nb = min(BT, B - b0);
    if (b0 > 0) __syncthreads();
    // ---- stage activation rows (+ optional LayerNorm) -----------------------------------
    for (int i = threadIdx.x * 4; i < BT * K; i += blockDim.x * 4) {
      const int b = i / K, k = i - b * K;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (b < nb) v = *reinterpret_cast<const float4 *>(x + (int64_t)(b0 + b) * ldx + k);
      *reinterpret_cast<float4 *>(&xs[b * K + xs_phys<VEC>(k, K)]) = v;
    }
    __syncthreads();
    if (ln_g != nullptr) {
      if (warp < nb) {
        float *row = xs + warp * K;
        float s = 0.f;
        for (int k = lane; k < K; k += 32) s += row[k];
        const float mean = warp_sum(s) / (float)K;
        float q = 0.f;
        for (int k = lane; k < K; k += 32) {
          const float dlt = row[k] - mean;
          q += dlt * dlt;
        }
        const float rstd = rsqrtf(warp_sum(q) / (float)K + eps);
        for (int k = lane; k < K; k += 32) {
          const int p = xs_phys<VEC>(k, K);
          float y = (row[p] - mean) * rstd * ln_g[k] + ln_b[k];
          if (ada_wb) y = ada_wb[k] * y + ada_wb[K + k];
          row[p] = y;
        }
      }
      __syncthreads();
    }
    // ---- stream weights ---------------------------------------------------------------------
    for (int n0 = gw * NPW; n0 < N; n0 += GW * NPW) {
      float acc[NPW][BT];
#pragma unroll
      for (int j = 0; j < NPW; ++j)
#pragma unroll
        for (int b = 0; b < BT; ++b) acc[j][b] = 0.f;
#pragma unroll 2
      for (int k = lane * VEC; k < K; k += 32 * VEC) {
        Vec16<TW> wv[NPW];
#pragma unroll
        for (int j = 0; j < NPW; ++j) {
          const int n = min(n0 + j, N - 1);
          wv[j] = load_stream<TW>(W + (int64_t)n * K + k);
        }
        float xv[BT][VEC];
#pragma unroll
        for (int b = 0; b < BT; ++b) {
          if constexpr (VEC == 4) {
            const float4 t = *reinterpret_cast<const float4 *>(&xs[b * K + k]);
            xv[b][0] = t.x; xv[b][1] = t.y; xv[b][2] = t.z; xv[b][3] = t.w;
          } else {
            const int p = (k >> 3) << 2;
            const float4 t0 = *reinterpret_cast<const float4 *>(&xs[b * K + p]);
            const float4 t1 = *reinterpret_cast<const float4 *>(&xs[b * K + (K >> 1) + p]);
            xv[b][0] = t0.x; xv[b][1] = t0.y; xv[b][2] = t0.z; xv[b][3] = t0.w;
            xv[b][4] = t1.x; xv[b][5] = t1.y; xv[b][6] = t1.z; xv[b][7] = t1.w;
          }
        }
#pragma unroll
        for (int j = 0; j < NPW; ++j) {
          float wf[VEC];
          wv[j].unpack(wf);
#pragma unroll
          for (int b = 0; b < BT; ++b)
#pragma unroll
            for (int i = 0; i < VEC; ++i) acc[j][b] = fmaf(wf[i], xv[b][i], acc[j][b]);
        }
      }
#pragma unroll
      for (int j = 0; j < NPW; ++j)
#pragma unroll
        for (int b = 0; b < BT; ++b) acc[j][b] = warp_sum(acc[j][b]);
      if (lane == 0) {
#pragma unroll
        for (int j = 0; j < NPW; ++j) {
          const int n = n0 + j;
          if (n >= N) continue;
          const float bn = bias ? bias[n] : 0.f;
#pragma unroll
          for (int b = 0; b < BT; ++b) {
            if (b >= nb) continue;
            const int bb = b0 + b;
            float v = acc[j][b] + bn;
            if (epi.mode == 3) {
              const QkvScatter &q = epi.qkv;
              const int part = n / q.d, c = n - part * q.d;
              if (part == 0) {
                q.q[(int64_t)bb * q.d + c] = v;
              } else if (q.rows.finished == nullptr || q.rows.finished[bb] == 0) {
                const int h = c / q.head_dim, e = c - h * q.head_dim;
                const int64_t off = q.kv.row(bb, h, q.rows.cur(bb, q.rows.n_gen[bb], q.kv.cap)) + e;
                TW *cache = reinterpret_cast<TW *>(part == 1 ? q.kv.k : q.kv.v);
                cache[off] = from_f32<TW>(v);
              }
            } else {
              float *o = out + (int64_t)bb * ldo + n;
              if (epi.mode == 1) v = fmaxf(v, 0.f);
              if (epi.mode == 2) v = *o + v;
              *o = v;
            }
          }
        }
      }
    }
  }
}

template <typename TW, int BT>
static int launch_gemv_bt(const float *x, int64_t ldx, int B, const TW *W, const float *bias, int N,
                          int K, float *out, int64_t ldo, const float *ln_g, const float *ln_b,
                          const float *ada_wb, float eps, const GemvEpi &epi, cudaStream_t s) {
  const int threads = 512, nwarps = threads / 32;
  const size_t smem = (size_t)BT * K * sizeof(float);
  const int sms = sm_count();
  const int per_sm = smem <= 48 * 1024 ? 2 : 1;
  const int total_warps = sms * per_sm * nwarps;
  const bool two = (N / 2) >= total_warps;
  int grid;
  if (two) {
    grid = min(sms * per_sm, (N / 2 + nwarps - 1) / nwarps);
    auto kern = gemv_kernel<TW, BT, 2>;
    if (smem > 48 * 1024) VB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kern<<<grid, threads, smem, s>>>(x, ldx, B, W, bias, N, K, out, ldo, ln_g, ln_b, ada_wb, eps, epi);
  } else {
    grid = min(sms * per_sm, (N + nwarps - 1) / nwarps);
    auto kern = gemv_kernel<TW, BT, 1>;
    if (smem > 48 * 1024) VB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kern<<<grid, threads, smem, s>>>(x, ldx, B, W, bias, N, K, out, ldo, ln_g, ln_b, ada_wb, eps, epi);
  }
  VB_LAUNCH_CHECK();
  return VB_OK;
}

template <typename TW>
static int launch_gemv_t(const float *x, int64_t ldx, int B, const TW *W, const float *bias, int N, int K,
                         float *out, int64_t ldo, const float *ln_g, const float *ln_b,
                         const float *ada_wb, float eps, const GemvEpi &epi, cudaStream_t s) {
  // rows per pass: keep BT*K*4 bytes within shared memory (<= 128 KB)
  int bt = B >= 8 ? 8 : (B >= 4 ? 4 : (B >= 2 ? 2 : 1));
  while ((size_t)bt * K * 4 > 160 * 1024 && bt > 1) bt >>= 1;
  switch (bt) {
    case 8: return launch_gemv_bt<TW, 8>(x, ldx, B, W, bias, N, K, out, ldo, ln_g, ln_b, ada_wb, eps, epi, s);
    case 4: return launch_gemv_bt<TW, 4>(x, ldx, B, W, bias, N, K, out, ldo, ln_g, ln_b, ada_wb, eps, epi, s);
    case 2: return launch_gemv_bt<TW, 2>(x, ldx, B, W, bias, N, K, out, ldo, ln_g, ln_b, ada_wb, eps, epi, s);
    default: return launch_gemv_bt<TW, 1>(x, ldx, B, W, bias, N, K, out, ldo, ln_g, ln_b, ada_wb, eps, epi, s);
  }
}

int launch_gemv(const float *x, int64_t ldx, int B, const void *W, int w_dtype, const float *bias,
                int N, int K, float *out, int64_t ldo, const LnParams *ln, int epi_mode,
                const QkvScatter *qkv, cudaStream_t s) {
  VB_CHECK_ARG(K % 256 == 0, "gemv: K=%d must be a multiple of 256", K);
  VB_CHECK_ARG(ldx % 4 == 0, "gemv: ldx must be a multiple of 4");
  if (B == 0) return VB_OK;
  GemvEpi epi{};
  epi.mode = epi_mode;
  if (epi_mode == 3) {
    VB_CHECK_ARG(qkv != nullptr, "gemv: qkv scatter parameters missing");
    epi.qkv = *qkv;
  }
  const float *g = ln ? ln->gamma : nullptr, *bt = ln ? ln->beta : nullptr, *ada = ln ? ln->ada_wb : nullptr;
  const float eps = ln ? ln->eps : 0.f;
  if (w_dtype == VB_F32)
    return launch_gemv_t<float>(x, ldx, B, (const float *)W, bias, N, K, out, ldo, g, bt, ada, eps, epi, s);
  if (w_dtype == VB_BF16)
    return launch_gemv_t<bf16>(x, ldx, B, (const bf16 *)W, bias, N, K, out, ldo, g, bt, ada, eps, epi, s);
  set_error("gemv: bad weight dtype %d", w_dtype);
  return VB_ERR_ARG;
}

}  // namespace vb
