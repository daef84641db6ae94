// bf16 flash attention for packed ragged sequences (head_dim 64) on the Hopper tensor cores (wgmma / TMA /
// mbarrier) -- the L x L attention of the 7 NAR passes, the AR prefill (which also fills the KV cache here) and the
// training forward in bf16 mode: softmax(q k^T / 8 + mask) v with online softmax
// (F.multi_head_attention_forward, valle/modules/activation.py:408-427; no mask for NAR
// valle/models/valle.py:1125-1127, key-padding / causal rules of valle.py:835-861,921-925, kv_len(i) = max(S, i + 1)).
//
// One CTA = 128 query rows of one (sequence, head); 256 threads, two CTAs per SM (one CTA's softmax overlaps the
// other's MMAs):
//   warpgroups 0-1 query rows [64 g, 64 g + 64): S = Q K^T by wgmma m64n64k16 (both operands K-major in shared memory),
//                  mask + online softmax on the accumulator fragments, O += P V by wgmma with P straight from
//                  registers as the A operand and V as the MN-major B operand exactly as TMA lands it.  Key tiles
//                  that every row of the warpgroup sees skip the mask tests; a warp whose row maxima did not move
//                  skips the rescale of O; a warpgroup whose 64 rows all lie past the sequence exits at once.
//   thread 0       also issues the TMA: the Q boxes once, then 64-key K and V boxes (128B-swizzled 64 x 64 boxes of
//                  the packed [M, 3d] qkv matrix) through a kStages-deep mbarrier ring.  Without a separate producer
//                  warp the CTA is 8 warps, so two CTAs per SM may use 128 registers per thread (no spills).
// Every query row gets the arithmetic of the plain masked loop (same tiles, mask decisions, expressions and wgmma
// order), so the outputs are bitwise those of that loop; tests/test_attention_bitwise_gpu.py pins them.
#include <math_constants.h>

#include "common.cuh"
#include "kernels.cuh"
#include "sm90_ptx.cuh"

namespace vb {
namespace fa3 {

using namespace tc;

constexpr int HD = 64, BQ = 128, BKV = 64;
constexpr int kThreads = 256;
constexpr int kStages = 4;
constexpr int kBoxBytes = 64 * HD * 2;        // 8 KB: one 64-row x 64-column bf16 box
constexpr int kQBytes = 2 * kBoxBytes;        // 16 KB
constexpr int kStageBytes = 2 * kBoxBytes;    // K + V
constexpr int kSmemBytes = kQBytes + kStages * kStageBytes + 1024 /*align slack*/ + 256 /*barriers*/;

// MN-major, 128-byte swizzle descriptor: a [K rows x 64 MN] tile stored as rows of 128 bytes (8 rows = one
// 1024-byte swizzle atom); 1024 B between 8-row groups along K (the single 128-byte atom column along MN needs no
// second stride)
__device__ __forceinline__ uint64_t make_smem_desc_mn(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr & 0x3FFFF) >> 4);
  d |= (uint64_t)(1024 >> 4) << 16;
  d |= (uint64_t)(1024 >> 4) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}
__device__ __forceinline__ float ex2(float x) {  // 2^x; ex2(-inf) = 0
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ uint32_t pack_bf16(float lo, float hi) {
  __nv_bfloat162 p = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t *>(&p);
}

// Scale (and, for kMask, mask) one 64-key tile of scores, then the online-softmax update of the thread's two rows:
// s becomes P = 2^(s sc - m), l the per-thread partial row sums; corr is the factor O has to be rescaled by.
// Register i of s holds row (i >> 1) & 1 ? b : a, key j0 + wg_col(t, i).  The scale is a separate rounded multiply
// (never contracted with the subtraction that follows).
template <bool kMask>
__device__ __forceinline__ void online_softmax(float (&s)[32], int j0, int t, const RowMask &lim_a,
                                               const RowMask &lim_b, float &m_a, float &m_b, float &l_a, float &l_b,
                                               float &corr_a, float &corr_b) {
  const float sc = 0.125f * 1.4426950408889634f;  // 1/sqrt(64) * log2(e)
  float mx_a = -CUDART_INF_F, mx_b = -CUDART_INF_F;
#pragma unroll
  for (int i = 0; i < 32; ++i) {
    const int c = j0 + wg_col(t, i);
    if ((i >> 1) & 1) {
      s[i] = (!kMask || lim_b.ok(c)) ? __fmul_rn(s[i], sc) : -CUDART_INF_F;
      mx_b = fmaxf(mx_b, s[i]);
    } else {
      s[i] = (!kMask || lim_a.ok(c)) ? __fmul_rn(s[i], sc) : -CUDART_INF_F;
      mx_a = fmaxf(mx_a, s[i]);
    }
  }
  mx_a = fmaxf(mx_a, __shfl_xor_sync(0xffffffffu, mx_a, 1));
  mx_a = fmaxf(mx_a, __shfl_xor_sync(0xffffffffu, mx_a, 2));
  mx_b = fmaxf(mx_b, __shfl_xor_sync(0xffffffffu, mx_b, 1));
  mx_b = fmaxf(mx_b, __shfl_xor_sync(0xffffffffu, mx_b, 2));
  const float mn_a = fmaxf(m_a, mx_a), mn_b = fmaxf(m_b, mx_b);
  const float mu_a = mn_a == -CUDART_INF_F ? 0.f : mn_a, mu_b = mn_b == -CUDART_INF_F ? 0.f : mn_b;
  corr_a = ex2(m_a - mu_a);
  corr_b = ex2(m_b - mu_b);
  m_a = mn_a;
  m_b = mn_b;
  float rs_a = 0.f, rs_b = 0.f;
#pragma unroll
  for (int i = 0; i < 32; ++i) {
    if ((i >> 1) & 1) {
      s[i] = ex2(s[i] - mu_b);
      rs_b += s[i];
    } else {
      s[i] = ex2(s[i] - mu_a);
      rs_a += s[i];
    }
  }
  l_a = l_a * corr_a + rs_a;  // per-thread partial row sums (quad-reduced at the end)
  l_b = l_b * corr_b + rs_b;
}

// kF8: the KV cache is the FP8 one (include/valle_b200.h, "FP8 (e4m3) KV cache"): e4m3 rows and their exponents;
// the attention itself computes on the bf16 tiles either way
template <bool kF8>
__global__ void __launch_bounds__(kThreads, 2)
attn_wgmma_kernel(const __grid_constant__ CUtensorMap tmap_qkv, int n_head, const Packed pk,
                  bf16 *__restrict__ out, const __grid_constant__ KvCache kv) {
  const int b = blockIdx.z, h = blockIdx.y;
  const Packed::Seq sb = pk.seq(b);
  const int r0 = sb.r0, L = sb.L;
  const int q0 = blockIdx.x * BQ;
  if (q0 >= L) return;
  const int d = n_head * HD;
  const int n_tiles = (pk.kv_max(sb, min(q0 + BQ, L)) + BKV - 1) / BKV;

  extern __shared__ uint8_t smem_raw[];
  uint8_t *sq = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t *ring = sq + kQBytes;
  uint64_t *bars = reinterpret_cast<uint64_t *>(ring + kStages * kStageBytes);
  uint64_t *q_bar = bars, *full_bar = bars + 1, *empty_bar = bars + 1 + kStages;

  const int wg = threadIdx.x >> 7, t = threadIdx.x & 127, lane = threadIdx.x & 31;
  const int n_wg = q0 + 64 < L ? 2 : 1;  // consumer warpgroups with at least one query row
  if (threadIdx.x == 0) {
    prefetch_tmap(&tmap_qkv);
    mbar_init(q_bar, 1);
    for (int i = 0; i < kStages; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 4 * n_wg);  // one arrive per working consumer warp
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  // TMA of key tile `k` into ring stage k % kStages, once every warp has released the tile kStages before it
  auto load_tile = [&](int k) {
    const int stg = k % kStages;
    mbar_wait(&empty_bar[stg], ((k / kStages) & 1) ^ 1);
    uint8_t *dst = ring + stg * kStageBytes;
    mbar_expect_tx(&full_bar[stg], kStageBytes);
    tma_load_2d(&tmap_qkv, &full_bar[stg], dst, d + h * HD, r0 + k * BKV);
    tma_load_2d(&tmap_qkv, &full_bar[stg], dst + kBoxBytes, 2 * d + h * HD, r0 + k * BKV);
  };
  if (threadIdx.x == 0) {
    mbar_expect_tx(q_bar, n_wg * kBoxBytes);
    tma_load_2d(&tmap_qkv, q_bar, sq, h * HD, r0 + q0);
    if (n_wg == 2) tma_load_2d(&tmap_qkv, q_bar, sq + kBoxBytes, h * HD, r0 + q0 + 64);
    for (int k = 0; k < min(kStages, n_tiles); ++k) load_tile(k);
  }
  // no rows, and no key tile of the KV cache to copy (that is tile q0 + 64 >= L)
  if (wg >= n_wg) return;

  // ===== consumers =====
  const int half = wg;
  const int row_a = q0 + half * 64 + wg_row(t, 0), row_b = row_a + 8;  // the two query rows of this thread
  const RowMask lim_a = pk.row_mask(sb, row_a), lim_b = pk.row_mask(sb, row_b);
  // every row of the warpgroup sees keys [0, kfree): lim0 does not decrease with the row in any mask mode, so the
  // warpgroup's first row has the smallest.  Tiles below it skip the mask tests (they would all pass).
  const int kfree = pk.row_mask(sb, q0 + half * 64).lim0;
  const uint64_t qdesc = make_smem_desc(smem_u32(sq + half * kBoxBytes));

  float o[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) o[i] = 0.f;
  float m_a = -CUDART_INF_F, m_b = -CUDART_INF_F, l_a = 0.f, l_b = 0.f;
  uint32_t pa[4][4];  // P as bf16 pairs (k-step ks = keys 16 ks .. +16 = s[8 ks .. 8 ks + 7])

  // S = Q K^T of one tile (64 query rows x 64 keys per warpgroup)
  auto issue_qk = [&](float (&s)[32], const uint8_t *sk) {
    const uint64_t kdesc = make_smem_desc(smem_u32(sk));
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < HD / WGMMA_K; ++k) wgmma_m64n64k16(s, qdesc + (uint64_t)(k * 2), kdesc + (uint64_t)(k * 2), k != 0);
    wgmma_commit();
  };
  // O += P V of the tile in ring stage `stg` (P from registers, pa)
  auto issue_pv = [&](int stg) {
    const uint64_t vdesc = make_smem_desc_mn(smem_u32(ring + stg * kStageBytes + kBoxBytes));
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) wgmma_m64n64k16_rs_tb(o, pa[ks], vdesc + (uint64_t)(ks * (16 * 128 >> 4)));
    wgmma_commit();
  };
  // the prefill fills the KV cache: warpgroup `half` copies key tile q0 + 64 half (rows < L)
  auto fill_cache = [&](int j0, const uint8_t *sk) {
    if (kv.k == nullptr || j0 != q0 + half * 64) return;
    const uint8_t *sv = sk + kBoxBytes;
    const int cb = pk.cache_seq(b);
    if constexpr (kF8) {
      // 8 consecutive lanes hold one row (16 bytes = 8 bf16 each): the row's max |.| is one 8-lane shuffle reduction
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int idx = t + i * 128;
        const int r = idx >> 3, c = idx & 7;
        const int so = r * 128 + ((c ^ (r & 7)) << 4);
        Vec16<bf16> kt, vt;
        kt.raw = *reinterpret_cast<const uint4 *>(sk + so);
        vt.raw = *reinterpret_cast<const uint4 *>(sv + so);
        float kf[8], vf[8];
        kt.unpack(kf);
        vt.unpack(vf);
        float ak = 0.f, av = 0.f;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          ak = fmaxf(ak, fabsf(kf[j]));
          av = fmaxf(av, fabsf(vf[j]));
        }
#pragma unroll
        for (int o = 4; o > 0; o >>= 1) {
          ak = fmaxf(ak, __shfl_xor_sync(0xffffffffu, ak, o));
          av = fmaxf(av, __shfl_xor_sync(0xffffffffu, av, o));
        }
        if (j0 + r < L) {
          const int ek = kv8_exp_biased(ak), ev = kv8_exp_biased(av);
          uint32_t kq[2] = {0u, 0u}, vq[2] = {0u, 0u};
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            kq[j >> 2] |= (uint32_t)kv8_quant(kf[j], ek) << (8 * (j & 3));
            vq[j >> 2] |= (uint32_t)kv8_quant(vf[j], ev) << (8 * (j & 3));
          }
          const int64_t e = kv.exp_index(cb, h, j0 + r), off = e * HD + c * 8;   // row(b, h, p) = 64 exp_index(b, h, p)
          *reinterpret_cast<uint2 *>((uint8_t *)kv.k + off) = make_uint2(kq[0], kq[1]);
          *reinterpret_cast<uint2 *>((uint8_t *)kv.v + off) = make_uint2(vq[0], vq[1]);
          if (c == 0) {
            kv.kexp[e] = (uint8_t)ek;
            kv.vexp[e] = (uint8_t)ev;
          }
        }
      }
    } else {
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int idx = t + i * 128;
        const int r = idx >> 3, c = idx & 7;
        if (j0 + r < L) {
          const int64_t off = kv.row(cb, h, j0 + r) + c * 8;
          const int so = r * 128 + ((c ^ (r & 7)) << 4);
          *reinterpret_cast<uint4 *>((bf16 *)kv.k + off) = *reinterpret_cast<const uint4 *>(sk + so);
          *reinterpret_cast<uint4 *>((bf16 *)kv.v + off) = *reinterpret_cast<const uint4 *>(sv + so);
        }
      }
    }
  };
  auto softmax = [&](float (&s)[32], int j0, float &corr_a, float &corr_b) {
    if (j0 + BKV <= kfree)
      online_softmax<false>(s, j0, t, lim_a, lim_b, m_a, m_b, l_a, l_b, corr_a, corr_b);
    else
      online_softmax<true>(s, j0, t, lim_a, lim_b, m_a, m_b, l_a, l_b, corr_a, corr_b);
  };
  auto pack_p = [&](const float (&s)[32]) {
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
      pa[ks][0] = pack_bf16(s[8 * ks + 0], s[8 * ks + 1]);
      pa[ks][1] = pack_bf16(s[8 * ks + 2], s[8 * ks + 3]);
      pa[ks][2] = pack_bf16(s[8 * ks + 4], s[8 * ks + 5]);
      pa[ks][3] = pack_bf16(s[8 * ks + 6], s[8 * ks + 7]);
    }
  };

  mbar_wait(q_bar, 0);
  int stage = 0;
  uint32_t phase = 0;
  for (int it = 0; it < n_tiles; ++it) {
    const int j0 = it * BKV;
    // refill the stage of tile it - 2: a warpgroup running up to a tile behind the other does not stall thread 0
    if (threadIdx.x == 0 && it >= 2 && it - 2 + kStages < n_tiles) load_tile(it - 2 + kStages);
    __syncwarp();
    mbar_wait(&full_bar[stage], phase);
    uint8_t *sk = ring + stage * kStageBytes;
    // The tail tile's box runs past the sequence: into the next one's rows, or TMA's zero fill past M.  P is 0 there,
    // but 0 * inf and 0 * NaN are NaN in P V, so the working warpgroups zero those V rows (whole 128-byte rows: the
    // swizzle stays within a row) and make the zeros visible to the wgmma before either warpgroup's P V reads them.
    // Only the last tile can be the tail tile (n_tiles <= ceil(L / 64)).
    if (j0 + BKV > L) {
      uint4 *sv = reinterpret_cast<uint4 *>(sk + kBoxBytes);
      for (int i = (L - j0) * 8 + threadIdx.x; i < BKV * 8; i += 128 * n_wg) sv[i] = make_uint4(0u, 0u, 0u, 0u);
      fence_proxy_async_smem();
      named_bar_sync(1, 128 * n_wg);
    }
    float s[32], corr_a, corr_b;
    issue_qk(s, sk);
    wgmma_wait<0>();
    wgmma_fence_regs(s);
    fill_cache(j0, sk);
    softmax(s, j0, corr_a, corr_b);
    // o * 1.0f == o: a warp whose row maxima all stayed put skips the rescale
    if (__any_sync(0xffffffffu, corr_a != 1.f || corr_b != 1.f)) {
#pragma unroll
      for (int i = 0; i < 32; ++i) o[i] *= ((i >> 1) & 1) ? corr_b : corr_a;
    }
    pack_p(s);
    wgmma_fence();
    issue_pv(stage);
    wgmma_wait<0>();
    wgmma_fence_regs(o);
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty_bar[stage]);
    if (++stage == kStages) {
      stage = 0;
      phase ^= 1;
    }
  }
  l_a += __shfl_xor_sync(0xffffffffu, l_a, 1);
  l_a += __shfl_xor_sync(0xffffffffu, l_a, 2);
  l_b += __shfl_xor_sync(0xffffffffu, l_b, 1);
  l_b += __shfl_xor_sync(0xffffffffu, l_b, 2);
  const float inv_a = 1.f / l_a, inv_b = 1.f / l_b;
#pragma unroll
  for (int i = 0; i < 32; i += 2) {
    const bool rb = (i >> 1) & 1;
    const int row = rb ? row_b : row_a;
    if (row >= L) continue;
    const float inv = rb ? inv_b : inv_a;
    *reinterpret_cast<uint32_t *>(out + (int64_t)(r0 + row) * d + h * HD + wg_col(t, i)) =
        pack_bf16(o[i] * inv, o[i + 1] * inv);
  }
}

}  // namespace fa3

template <bool kF8>
static int launch_wgmma(const CUtensorMap &tm, int n_head, const Packed &pk, bf16 *out, const KvCache &kv,
                        cudaStream_t s) {
  static PerDeviceOnce once;
  if (once.first())
    VB_CUDA(cudaFuncSetAttribute(fa3::attn_wgmma_kernel<kF8>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 fa3::kSmemBytes));
  const dim3 grid((pk.max_seqlen + fa3::BQ - 1) / fa3::BQ, n_head, pk.B);
  fa3::attn_wgmma_kernel<kF8><<<grid, fa3::kThreads, fa3::kSmemBytes, s>>>(tm, n_head, pk, out, kv);
  VB_LAUNCH_CHECK();
  return VB_OK;
}

int launch_attention_wgmma(const bf16 *qkv, int64_t M, int n_head, const Packed &pk, bf16 *out, const KvCache &kv,
                           cudaStream_t s) {
  if (M == 0 || pk.B == 0) return VB_OK;
  VB_CHECK_ARG((reinterpret_cast<uintptr_t>(qkv) & 15) == 0, "wgmma attention: qkv must be 16-byte aligned");
  CUtensorMap tm;
  VB_TRY(tc::make_tmap(&tm, qkv, M, 3 * n_head * fa3::HD, 3 * (int64_t)n_head * fa3::HD, 64));
  return kv.kexp != nullptr ? launch_wgmma<true>(tm, n_head, pk, out, kv, s)
                            : launch_wgmma<false>(tm, n_head, pk, out, kv, s);
}

}  // namespace vb
