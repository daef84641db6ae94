// bf16 GEMM on the Hopper tensor cores (sm_90a): C[M,N] = epi(A[M,K] W[N,K]^T + bias).
//
// Hand-written wgmma / TMA kernel for the dense QKV / out-proj / FFN / head projections
// of the NAR passes, the AR prefill and the training forward (F.linear at
// valle/modules/activation.py:408, valle/modules/transformer.py:332-334, valle/models/valle.py:1128).
//
// Structure (one CTA per 128 x 128 output tile, 384 threads = 3 warpgroups):
//   warpgroup 0    TMA producer (one thread): cp.async.bulk.tensor 2D loads of a 128 x 64 A box and a
//                  128 x 64 W box (both K-major, 128-byte swizzle) into a kStages-deep shared-memory ring,
//                  mbarrier complete_tx signalling.
//   warpgroups 1-2 consumers: warpgroup g owns rows [64 g, 64 g + 64) of the tile and issues
//                  wgmma.m64n128k16 x 4 per stage, fp32 accumulators in registers; one k-block of MMAs
//                  stays in flight while the previous stage is handed back to the producer.  Epilogue
//                  straight from the accumulator fragments: + bias, ReLU / residual, convert, store.
#include <cuda.h>
#include <stdlib.h>

#include "common.cuh"
#include "kernels.cuh"
#include "sm90_ptx.cuh"

namespace vb {

namespace tc {

constexpr int BM = 128, BN = 128;
constexpr int kThreads = 384;
constexpr int kStages = 6;
constexpr int kABytes = BM * BK * 2;  // 16 KB
constexpr int kBBytes = BN * BK * 2;  // 16 KB
constexpr int kStageBytes = kABytes + kBBytes;
constexpr int kSmemBytes = kStages * kStageBytes + 1024 /*align slack*/ + 256 /*barriers*/;
static_assert(kSmemBytes <= 227 * 1024, "shared memory of one CTA");

template <int kEpi, typename TC>
__global__ void __launch_bounds__(kThreads, 1)
gemm_wgmma_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                  const float *__restrict__ bias, TC *__restrict__ C, int64_t ldc, int M, int K) {
  extern __shared__ uint8_t smem_raw[];
  // 1024-byte alignment for the 128B-swizzled tiles
  uint8_t *tiles = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint64_t *bars = reinterpret_cast<uint64_t *>(tiles + kStages * kStageBytes);
  uint64_t *full_bar = bars;             // [kStages]
  uint64_t *empty_bar = bars + kStages;  // [kStages]

  const int wg = threadIdx.x >> 7, t = threadIdx.x & 127;
  const int n_blk = blockIdx.x, m_blk = blockIdx.y;
  const int num_kb = K / BK;

  if (threadIdx.x == 0) {
    prefetch_tmap(&tmap_a);
    prefetch_tmap(&tmap_b);
    for (int i = 0; i < kStages; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 8);  // one arrive per consumer warp
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (wg == 0) {
    // ===== TMA producer =====
    if (t == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait(&empty_bar[stage], phase ^ 1);
        uint8_t *a_dst = tiles + stage * kStageBytes;
        mbar_expect_tx(&full_bar[stage], kStageBytes);
        tma_load_2d(&tmap_a, &full_bar[stage], a_dst, kb * BK, m_blk * BM);
        tma_load_2d(&tmap_b, &full_bar[stage], a_dst + kABytes, kb * BK, n_blk * BN);
        if (++stage == kStages) {
          stage = 0;
          phase ^= 1;
        }
      }
    }
    return;
  }

  // ===== consumers: rows [64 (wg-1), +64) of the tile =====
  const int half = wg - 1;
  float acc[BN / 2];  // written first by the scale-d = 0 MMA of k-block 0 (K > 0)
  int stage = 0, prev = -1;
  uint32_t phase = 0;
  for (int kb = 0; kb < num_kb; ++kb) {
    mbar_wait(&full_bar[stage], phase);
    const uint32_t a_addr = smem_u32(tiles + stage * kStageBytes) + half * (64 * 128);
    const uint32_t b_addr = smem_u32(tiles + stage * kStageBytes) + kABytes;
    const uint64_t adesc = make_smem_desc(a_addr), bdesc = make_smem_desc(b_addr);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < BK / WGMMA_K; ++k) wgmma_m64n128k16(acc, adesc + (uint64_t)(k * 2), bdesc + (uint64_t)(k * 2), (kb | k) != 0);
    wgmma_commit();
    wgmma_wait<1>();  // the MMAs of the previous k-block have retired: its stage goes back to the producer
    if (prev >= 0 && (t & 31) == 0) mbar_arrive(&empty_bar[prev]);
    prev = stage;
    if (++stage == kStages) {
      stage = 0;
      phase ^= 1;
    }
  }
  wgmma_wait<0>();
  wgmma_fence_regs(acc);

  // ===== epilogue: + bias, ReLU / residual (fp32 read-modify-write of C, one owner per element) =====
  const int n0 = n_blk * BN;
#pragma unroll
  for (int i = 0; i < BN / 2; i += 2) {
    const int row = m_blk * BM + half * 64 + wg_row(t, i);
    const int col = n0 + wg_col(t, i);
    if (row >= M) continue;
    float v0 = acc[i], v1 = acc[i + 1];
    if (bias) {
      v0 += __ldg(bias + col);
      v1 += __ldg(bias + col + 1);
    }
    if constexpr (kEpi == VB_EPI_RELU) {
      v0 = fmaxf(v0, 0.f);
      v1 = fmaxf(v1, 0.f);
    }
    TC *dst = C + (int64_t)row * ldc + col;
    if constexpr (sizeof(TC) == 4) {
      float2 *d2 = reinterpret_cast<float2 *>(dst);
      if constexpr (kEpi == VB_EPI_RESIDUAL) {
        const float2 o = *d2;
        v0 = o.x + v0;
        v1 = o.y + v1;
      }
      *d2 = make_float2(v0, v1);
    } else {
      *reinterpret_cast<__nv_bfloat162 *>(dst) = __floats2bfloat162_rn(v0, v1);
    }
  }
}

template <int kEpi, typename TC>
static int launch_t(const CUtensorMap &ta, const CUtensorMap &tb, const float *bias, TC *C, int64_t ldc, int M,
                    int N, int K, cudaStream_t s) {
  auto kern = gemm_wgmma_kernel<kEpi, TC>;
  static PerDeviceOnce once;  // per template instantiation and device
  if (once.first()) VB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBytes));
  const dim3 grid(N / BN, (M + BM - 1) / BM);
  kern<<<grid, kThreads, kSmemBytes, s>>>(ta, tb, bias, C, ldc, M, K);
  VB_LAUNCH_CHECK();
  return VB_OK;
}

}  // namespace tc

bool wgmma_gemm_supported(int64_t M, int N, int K, int64_t lda, int64_t ldc) {
  return M >= 1 && (M + tc::BM - 1) / tc::BM <= 65535 && N % tc::BN == 0 && K % tc::BK == 0 && K > 0 &&
         lda % 8 == 0 && ldc % 8 == 0 && getenv("VB_DISABLE_WGMMA") == nullptr;
}

int launch_gemm_wgmma(const bf16 *A, int64_t lda, const bf16 *W, const float *bias, void *C, int c_dtype,
                      int64_t ldc, int64_t M, int N, int K, int epi, cudaStream_t s) {
  VB_CHECK_ARG((reinterpret_cast<uintptr_t>(A) & 15) == 0 && (reinterpret_cast<uintptr_t>(W) & 15) == 0 &&
                   (reinterpret_cast<uintptr_t>(C) & 15) == 0,
               "wgmma gemm: operands must be 16-byte aligned");
  CUtensorMap ta, tb;
  VB_TRY(tc::make_tmap(&ta, A, M, K, lda, tc::BM));
  VB_TRY(tc::make_tmap(&tb, W, N, K, K, tc::BN));
  const int m = (int)M;
  if (epi == VB_EPI_RESIDUAL) return tc::launch_t<VB_EPI_RESIDUAL, float>(ta, tb, bias, (float *)C, ldc, m, N, K, s);
  if (epi == VB_EPI_RELU) {
    if (c_dtype == VB_BF16) return tc::launch_t<VB_EPI_RELU, bf16>(ta, tb, bias, (bf16 *)C, ldc, m, N, K, s);
    return tc::launch_t<VB_EPI_RELU, float>(ta, tb, bias, (float *)C, ldc, m, N, K, s);
  }
  if (c_dtype == VB_BF16) return tc::launch_t<VB_EPI_NONE, bf16>(ta, tb, bias, (bf16 *)C, ldc, m, N, K, s);
  return tc::launch_t<VB_EPI_NONE, float>(ta, tb, bias, (float *)C, ldc, m, N, K, s);
}

}  // namespace vb
