// bf16 GEMM on the Hopper tensor cores (sm_90a): C[M,N] = epi(A[M,K] W[N,K]^T + bias).
//
// Hand-written wgmma / TMA kernel for the dense QKV / out-proj / FFN / head projections
// of the NAR passes, the AR prefill and the training forward (F.linear at
// valle/modules/activation.py:408, valle/modules/transformer.py:332-334, valle/models/valle.py:1128).
//
// Structure (persistent: min(tiles, SMs) CTAs walk the 128 x 256 output tiles round-robin, n fastest within an
// m-block, so one layer's W stays in L2 and A is read from HBM once; 384 threads = 3 warpgroups):
//   warpgroup 0    TMA producer (one thread): cp.async.bulk.tensor 2D loads of a 128 x 64 A box and a
//                  256 x 64 W box (both K-major, 128-byte swizzle) into a kStages-deep shared-memory ring,
//                  mbarrier complete_tx signalling.  Its ring position runs on across tiles, so the next
//                  tile's k-blocks stream in while the consumers run the epilogue.
//   warpgroups 1-2 consumers: warpgroup g owns rows [64 g, 64 g + 64) of the tile and issues
//                  wgmma.m64n256k16 x 4 per stage, fp32 accumulators in registers; one k-block of MMAs
//                  stays in flight while the previous stage is handed back to the producer.
//   epilogue       per 64-row x 128-byte sub-tile: + bias, ReLU / residual, convert, write into a 128B-swizzled
//                  staging buffer (two per consumer warpgroup), then one cp.async.bulk.tensor store.  The
//                  residual x of the tile is TMA-loaded through the ring behind the tile's last k-block and
//                  added as x + (acc + bias), one plain fp32 add per element.  (The bulk reduce-add would save
//                  that load, but the PTX ISA does not promise that its .f32 add keeps subnormals, and a
//                  flushed subnormal would change the output bits.)
#include <cuda.h>
#include <stdlib.h>

#include "common.cuh"
#include "kernels.cuh"
#include "sm90_ptx.cuh"

namespace vb {

namespace tc {

constexpr int BM = 128, BN = 256;
constexpr int kThreads = 384;
constexpr int kStages = 4;
constexpr int kABytes = BM * BK * 2;            // 16 KB
constexpr int kBBytes = BN * BK * 2;            // 32 KB
constexpr int kStageBytes = kABytes + kBBytes;  // 48 KB
constexpr int kStgBytes = 64 * 128;             // staging sub-tile: 64 rows x 128 bytes (32 fp32 / 64 bf16 columns)
// residual: x of a tile fills ring stages as 128-row x 32-column fp32 boxes, kXPerStage boxes per stage
constexpr int kXBoxBytes = BM * 128;
constexpr int kXBoxes = BN / 32;
constexpr int kXPerStage = kStageBytes / kXBoxBytes;
constexpr int kXStages = (kXBoxes + kXPerStage - 1) / kXPerStage;
constexpr int kSmemBytes = kStages * kStageBytes + 4 * kStgBytes + 1024 /*align slack*/ + 256 /*barriers*/;
static_assert(kSmemBytes <= 227 * 1024, "shared memory of one CTA");
static_assert(kXStages <= kStages, "x of a tile fits the ring");

template <int kEpi, typename TC>
__global__ void __launch_bounds__(kThreads, 1)
gemm_wgmma_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                  const __grid_constant__ CUtensorMap tmap_c, const __grid_constant__ CUtensorMap tmap_x,
                  const float *__restrict__ bias, int M, int N, int K) {
  constexpr bool kRes = kEpi == VB_EPI_RESIDUAL;
  constexpr int SUBN = 128 / (int)sizeof(TC);  // columns of one staging sub-tile
  static_assert(!kRes || SUBN == 32, "residual sub-tiles are the x boxes' columns");
  extern __shared__ uint8_t smem_raw[];
  // 1024-byte alignment for the 128B-swizzled tiles
  uint8_t *tiles = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t *stg = tiles + kStages * kStageBytes;  // [consumer warpgroup][2][kStgBytes]
  uint64_t *bars = reinterpret_cast<uint64_t *>(stg + 4 * kStgBytes);
  uint64_t *full_bar = bars;             // [kStages]
  uint64_t *empty_bar = bars + kStages;  // [kStages]

  const int wg = threadIdx.x >> 7, t = threadIdx.x & 127;
  const int n_tiles = (N + BN - 1) / BN;
  const int num_tiles = ((M + BM - 1) / BM) * n_tiles;
  const int num_kb = K / BK;

  if (threadIdx.x == 0) {
    prefetch_tmap(&tmap_a);
    prefetch_tmap(&tmap_b);
    prefetch_tmap(&tmap_c);
    if constexpr (kRes) prefetch_tmap(&tmap_x);
    for (int i = 0; i < kStages; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 8);  // one arrive per consumer warp
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  int stage = 0;
  uint32_t phase = 0;
  auto advance = [&] {
    if (++stage == kStages) {
      stage = 0;
      phase ^= 1;
    }
  };

  if (wg == 0) {
    // ===== TMA producer =====
    setmaxnreg_dec<40>();
    if (t == 0) {
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int m0 = (tile / n_tiles) * BM, n0 = (tile % n_tiles) * BN;
        for (int kb = 0; kb < num_kb; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          uint8_t *a_dst = tiles + stage * kStageBytes;
          mbar_expect_tx(&full_bar[stage], kStageBytes);
          tma_load_2d(&tmap_a, &full_bar[stage], a_dst, kb * BK, m0);
          tma_load_2d(&tmap_b, &full_bar[stage], a_dst + kABytes, kb * BK, n0);
          advance();
        }
        if constexpr (kRes) {
          for (int q = 0; q < kXStages; ++q) {
            mbar_wait(&empty_bar[stage], phase ^ 1);
            int nbox = 0;  // boxes of columns < N (a half tile at N % 256 == 128 has only the first four)
            for (int j = 0; j < kXPerStage; ++j) {
              const int b = q * kXPerStage + j;
              nbox += (b < kXBoxes && n0 + 32 * b < N);
            }
            mbar_expect_tx(&full_bar[stage], nbox * kXBoxBytes);
            for (int j = 0; j < nbox; ++j)
              tma_load_2d(&tmap_x, &full_bar[stage], tiles + stage * kStageBytes + j * kXBoxBytes,
                          n0 + 32 * (q * kXPerStage + j), m0);
            advance();
          }
        }
      }
    }
    return;
  }

  // ===== consumers: rows [64 (wg-1), +64) of each tile =====
  setmaxnreg_inc<232>();
  const int half = wg - 1;
  uint8_t *my_stg = stg + half * 2 * kStgBytes;
  int sbuf = 0;  // staging buffer the next sub-tile goes through
  float acc[BN / 2];  // written first by the scale-d = 0 MMA of k-block 0 (K > 0)
  for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
    const int m0 = (tile / n_tiles) * BM, n0 = (tile % n_tiles) * BN;
    int prev = 0;
    for (int kb = 0; kb < num_kb; ++kb) {
      mbar_wait(&full_bar[stage], phase);
      const uint32_t a_addr = smem_u32(tiles + stage * kStageBytes) + half * (64 * 128);
      const uint32_t b_addr = smem_u32(tiles + stage * kStageBytes) + kABytes;
      const uint64_t adesc = make_smem_desc(a_addr), bdesc = make_smem_desc(b_addr);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < BK / WGMMA_K; ++k)
        wgmma_m64n256k16(acc, adesc + (uint64_t)(k * 2), bdesc + (uint64_t)(k * 2), (kb | k) != 0);
      wgmma_commit();
      wgmma_wait<1>();  // the MMAs of the previous k-block have retired: its stage goes back to the producer
      if (kb > 0 && (t & 31) == 0) mbar_arrive(&empty_bar[prev]);
      prev = stage;
      advance();
    }
    wgmma_wait<0>();
    wgmma_fence_regs(acc);
    if ((t & 31) == 0) mbar_arrive(&empty_bar[prev]);

    // ===== epilogue: + bias, ReLU / residual, convert; staged sub-tiles leave through TMA stores =====
    const int row0 = m0 + half * 64;
#pragma unroll
    for (int sub = 0; sub < BN / SUBN; ++sub) {
      const int c0 = n0 + sub * SUBN;
      if constexpr (kRes) {
        if (sub % kXPerStage == 0) mbar_wait(&full_bar[stage], phase);
      }
      if (c0 < N && row0 < M) {  // uniform over the warpgroup; N % 128 == 0, so every column of the sub-tile is < N
        uint8_t *buf = my_stg + sbuf * kStgBytes;
        if (t == 0) bulk_wait_read<1>();  // the store that last read `buf` is done with it
        named_bar_sync(1 + half, 128);
#pragma unroll
        for (int i = sub * (SUBN / 2); i < (sub + 1) * (SUBN / 2); i += 2) {
          const int r = wg_row(t, i), cc = wg_col(t, i) - sub * SUBN;
          const int byte = cc * (int)sizeof(TC);
          const int off = r * 128 + ((((byte >> 4) ^ r) & 7) << 4) + (byte & 15);  // 128B swizzle
          float v0 = acc[i], v1 = acc[i + 1];
          if (bias) {
            v0 += __ldg(bias + c0 + cc);
            v1 += __ldg(bias + c0 + cc + 1);
          }
          if constexpr (kEpi == VB_EPI_RELU) {
            v0 = fmaxf(v0, 0.f);
            v1 = fmaxf(v1, 0.f);
          }
          if constexpr (sizeof(TC) == 4) {
            if constexpr (kRes) {
              const float2 o = *reinterpret_cast<const float2 *>(
                  tiles + stage * kStageBytes + (sub % kXPerStage) * kXBoxBytes + half * (64 * 128) + off);
              v0 = o.x + v0;
              v1 = o.y + v1;
            }
            *reinterpret_cast<float2 *>(buf + off) = make_float2(v0, v1);
          } else {
            *reinterpret_cast<__nv_bfloat162 *>(buf + off) = __floats2bfloat162_rn(v0, v1);
          }
        }
        fence_proxy_async_smem();
        named_bar_sync(1 + half, 128);
        if (t == 0) {
          tma_store_2d(&tmap_c, buf, c0, row0);
          bulk_commit();
        }
        sbuf ^= 1;
      }
      if constexpr (kRes) {
        if (sub % kXPerStage == kXPerStage - 1 || sub == BN / SUBN - 1) {  // x stage read: back to the producer
          __syncwarp();
          if ((t & 31) == 0) mbar_arrive(&empty_bar[stage]);
          advance();
        }
      }
    }
  }
  if (t == 0) bulk_wait<0>();  // every store has landed before the CTA exits
}

template <int kEpi, typename TC>
static int launch_t(const CUtensorMap &ta, const CUtensorMap &tb, const CUtensorMap &tc_, const CUtensorMap &tx,
                    const float *bias, int M, int N, int K, cudaStream_t s) {
  auto kern = gemm_wgmma_kernel<kEpi, TC>;
  static PerDeviceOnce once;  // per template instantiation and device
  if (once.first()) VB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBytes));
  const int tiles = ((M + BM - 1) / BM) * ((N + BN - 1) / BN);
  const int grid = tiles < sm_count() ? tiles : sm_count();
  kern<<<grid, kThreads, kSmemBytes, s>>>(ta, tb, tc_, tx, bias, M, N, K);
  VB_LAUNCH_CHECK();
  return VB_OK;
}

}  // namespace tc

bool wgmma_gemm_supported(int64_t M, int N, int K, int64_t lda, int64_t ldc) {
  return M >= 1 && (M + tc::BM - 1) / tc::BM <= 65535 && N % 128 == 0 && K % tc::BK == 0 && K > 0 &&
         lda % 8 == 0 && ldc % 8 == 0 && tune("VB_DISABLE_WGMMA", 0) == 0;
}

int launch_gemm_wgmma(const bf16 *A, int64_t lda, const bf16 *W, const float *bias, void *C, int c_dtype,
                      int64_t ldc, int64_t M, int N, int K, int epi, cudaStream_t s) {
  VB_CHECK_ARG((reinterpret_cast<uintptr_t>(A) & 15) == 0 && (reinterpret_cast<uintptr_t>(W) & 15) == 0 &&
                   (reinterpret_cast<uintptr_t>(C) & 15) == 0,
               "wgmma gemm: operands must be 16-byte aligned");
  const bool f32 = epi == VB_EPI_RESIDUAL || c_dtype != VB_BF16;
  CUtensorMap ta, tb, tcm, tx;
  VB_TRY(tc::make_tmap(&ta, A, M, K, lda, tc::BM));
  VB_TRY(tc::make_tmap(&tb, W, N, K, K, tc::BN));
  VB_TRY(tc::make_tmap_swz128(&tcm, C, f32, M, N, ldc, 64));
  tx = tcm;
  if (epi == VB_EPI_RESIDUAL) VB_TRY(tc::make_tmap_swz128(&tx, C, true, M, N, ldc, tc::BM));
  const int m = (int)M;
  if (epi == VB_EPI_RESIDUAL) return tc::launch_t<VB_EPI_RESIDUAL, float>(ta, tb, tcm, tx, bias, m, N, K, s);
  if (epi == VB_EPI_RELU) {
    if (c_dtype == VB_BF16) return tc::launch_t<VB_EPI_RELU, bf16>(ta, tb, tcm, tx, bias, m, N, K, s);
    return tc::launch_t<VB_EPI_RELU, float>(ta, tb, tcm, tx, bias, m, N, K, s);
  }
  if (c_dtype == VB_BF16) return tc::launch_t<VB_EPI_NONE, bf16>(ta, tb, tcm, tx, bias, m, N, K, s);
  return tc::launch_t<VB_EPI_NONE, float>(ta, tb, tcm, tx, bias, m, N, K, s);
}

}  // namespace vb
