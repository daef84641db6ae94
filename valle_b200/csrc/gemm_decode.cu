// Skinny (decode) projections on the tensor cores: out[b, n] = epi( sum_k act[b,k] W[n,k] + bias[n] ),
// b < B <= 64 rows of the AR decode step, bf16 operands, fp32 accumulate.
//
// HBM-bound weight streaming (AI <= 64 FLOP/B): the weight matrix is the M operand of wgmma
// ("swap-AB"), the B <= 64 activation rows are the N=64 operand, so every weight byte is
// read exactly once per step at full TMA throughput and the 132 SMs are filled by split-K:
//   grid = (N_out/128 tiles, S splits); CTA (t, s) streams W[t*128 .. +128, k-range(s)] through a
//   TMA/mbarrier ring into wgmma (2 x m64n64k16 per k-step), accumulates in registers, and
//   either applies the fused epilogue itself (S == 1: +bias, ReLU -> bf16, residual, QKV scatter) or
//   writes its fp32 partial tile to partials[split][b][n]; the CONSUMER kernel (residual + LayerNorm,
//   the KV-cache attention prologue, the sampler) sums the S partials in fixed order 0..S-1, which
//   keeps the result deterministic and costs no extra launch.  A residual update of the folded chain has no
//   consumer: the S splits of a tile form a thread-block cluster and add their tiles over DSMEM in fixed order.
//   Programmatic dependent launch: barrier setup and the first kStages WEIGHT tiles (which do
//   not depend on the previous kernel) are issued before griddepcontrol.wait, so weight streaming
//   overlaps the tail of the previous kernel in the CUDA graph.
//
// Replaces F.linear at valle/modules/activation.py:408 (in/out-proj), valle/modules/transformer.py:332-334
// (FFN) and valle/models/valle.py:1039 (ar_predict_layer) for the batched decode step.
#include <algorithm>

#include "common.cuh"
#include "kernels.cuh"
#include "sm90_ptx.cuh"

namespace vb {
namespace dg {

constexpr int kMaxClusterSplits = 8;  // portable thread-block cluster size

using namespace tc;

constexpr int TM = 128;      // weight rows per tile (two wgmma M=64 halves)
constexpr int TN = 64;       // activation rows (wgmma N)
constexpr int kStages = 6;
constexpr int kWBytes = TM * BK * 2;  // 16 KB
constexpr int kXBytes = TN * BK * 2;  // 8 KB
constexpr int kStageBytes = kWBytes + kXBytes;
constexpr int kSmemBytes = kStages * kStageBytes + 1024 + 256;
constexpr int kThreads = 256;
static_assert(kStages * kStageBytes >= TN * TM * 4, "the epilogue stages the fp32 tile in the ring");

struct Epi {
  int mode;  // DG_* below
  int red;   // DG_RESIDUAL with split-K, no partials: the splits of a tile are a thread-block cluster and add their
             // tiles into out_f32 over DSMEM in fixed order 0..S-1 (run-to-run identical)
  int N, B;  // valid output features / rows
  const float *bias;
  float *out_f32;      // [B, ld_out] (RESIDUAL: in/out; F32: out; QKV: q)
  bf16 *out_bf16;      // [B, ld_out] (RELU_BF16)
  int64_t ld_out;
  QkvScatter qkv;      // DG_QKV
};

__device__ __forceinline__ void apply_epi(const Epi &e, int n, int b, float v) {
  if (e.bias) v += e.bias[n];
  if (e.mode == DG_F32) {
    e.out_f32[(int64_t)b * e.ld_out + n] = v;
  } else if (e.mode == DG_RESIDUAL) {
    float *o = e.out_f32 + (int64_t)b * e.ld_out + n;
    *o = *o + v;
  } else if (e.mode == DG_RELU_BF16) {
    e.out_bf16[(int64_t)b * e.ld_out + n] = __float2bfloat16_rn(fmaxf(v, 0.f));
  } else {
    const QkvScatter &q = e.qkv;
    const int part = n / q.d, c = n - part * q.d;
    if (part == 0) {
      q.q[(int64_t)b * q.d + c] = v;
    } else if (q.rows.finished == nullptr || q.rows.finished[b] == 0) {
      const int h = c / q.head_dim, el = c - h * q.head_dim;
      const int64_t off = q.kv.row(b, h, q.rows.cur(b, q.rows.n_gen[b], q.kv.cap)) + el;
      ((bf16 *)(part == 1 ? q.kv.k : q.kv.v))[off] = __float2bfloat16_rn(v);
    }
  }
}

// swap-AB on wgmma: the weight tile is the A operand (two m64 halves), the activation rows the N = 64 B operand
__device__ __forceinline__ void decode_mma_stage(float (&acc0)[32], float (&acc1)[32], uint32_t w_addr, uint32_t x_addr) {
  const uint64_t a0 = make_smem_desc(w_addr), a1 = make_smem_desc(w_addr + 64 * 128), bd = make_smem_desc(x_addr);
  wgmma_fence();
#pragma unroll
  for (int k = 0; k < BK / WGMMA_K; ++k) {
    wgmma_m64n64k16(acc0, a0 + (uint64_t)(k * 2), bd + (uint64_t)(k * 2), 1);
    wgmma_m64n64k16(acc1, a1 + (uint64_t)(k * 2), bd + (uint64_t)(k * 2), 1);
  }
  wgmma_commit();
}
// accumulator fragments -> sv[b][feature] ([TN][TM] fp32, row b = activation row)
__device__ __forceinline__ void decode_stage_tile(const float (&acc0)[32], const float (&acc1)[32], float *sv, int t) {
#pragma unroll
  for (int i = 0; i < 32; ++i) {
    const int nl = wg_row(t, i), b = wg_col(t, i);
    sv[b * TM + nl] = acc0[i];
    sv[b * TM + 64 + nl] = acc1[i];
  }
}

// 256 threads: warp 0 TMA producer, warps 1-3 KV-cache L2 prefetch, warps 4-7 the MMA warpgroup and the epilogue
__global__ void __launch_bounds__(kThreads, 1)
gemm_decode_kernel(const __grid_constant__ CUtensorMap tmap_w, const __grid_constant__ CUtensorMap tmap_x, int num_kb, float *__restrict__ partials, int ldp,
                   Epi epi, KvPrefetch pf) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t *tiles = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint64_t *bars = reinterpret_cast<uint64_t *>(tiles + kStages * kStageBytes);
  uint64_t *full_bar = bars, *empty_bar = bars + kStages;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tile = blockIdx.x, split = blockIdx.y, splits = gridDim.y;
  // k-block range of this split (balanced, contiguous)
  const int base = num_kb / splits, rem = num_kb % splits;
  const int kb0 = split * base + min(split, rem);
  const int nkb = base + (split < rem ? 1 : 0);

  pdl_launch_dependents();
  if (warp == 0 && lane == 0) {
    prefetch_tmap(&tmap_w);
    prefetch_tmap(&tmap_x);
  }
  if (warp == 1 && lane == 0) {
    for (int i = 0; i < kStages; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 4);  // one arrive per MMA warp
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp == 0) {
    if (lane == 0) {
      // weights do not depend on the previous kernel: fill the ring with W tiles first ...
      const int pre = min(nkb, kStages);
      for (int i = 0; i < pre; ++i) {
        mbar_expect_tx(&full_bar[i], kStageBytes);
        tma_load_2d(&tmap_w, &full_bar[i], tiles + i * kStageBytes, (kb0 + i) * BK, tile * TM);
      }
      pdl_wait();  // ... the activations do
      vb_trace(TR_GEMM * 2);
      for (int i = 0; i < pre; ++i)
        tma_load_2d(&tmap_x, &full_bar[i], tiles + i * kStageBytes + kWBytes, (kb0 + i) * BK, 0);
      int stage = 0;
      uint32_t phase = 1;  // the ring has wrapped once
      for (int i = pre; i < nkb; ++i) {
        mbar_wait(&empty_bar[stage], phase ^ 1);
        uint8_t *w_dst = tiles + stage * kStageBytes;
        mbar_expect_tx(&full_bar[stage], kStageBytes);
        tma_load_2d(&tmap_w, &full_bar[stage], w_dst, (kb0 + i) * BK, tile * TM);
        tma_load_2d(&tmap_x, &full_bar[stage], w_dst + kWBytes, (kb0 + i) * BK, 0);
        if (++stage == kStages) {
          stage = 0;
          phase ^= 1;
        }
      }
    }
    __syncwarp();
  } else if (warp < 4) {
    // idle until the accumulator is complete: pull a slice of an upcoming layer's KV cache into L2
    kv_prefetch(pf, (blockIdx.y * gridDim.x + blockIdx.x) * 3 + (warp - 1), gridDim.x * gridDim.y * 3);
    pdl_wait();
  } else {
    const int t = threadIdx.x - 128;
    float acc0[32], acc1[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) acc0[i] = acc1[i] = 0.f;
    int stage = 0, prev = -1;
    uint32_t phase = 0;
    for (int i = 0; i < nkb; ++i) {
      mbar_wait(&full_bar[stage], phase);
      const uint32_t w_addr = smem_u32(tiles + stage * kStageBytes);
      decode_mma_stage(acc0, acc1, w_addr, w_addr + kWBytes);
      wgmma_wait<1>();
      if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
      prev = stage;
      if (++stage == kStages) {
        stage = 0;
        phase ^= 1;
      }
    }
    wgmma_wait<0>();
    wgmma_fence_regs(acc0);
    wgmma_fence_regs(acc1);
    pdl_wait();
    // every TMA load has landed and every MMA has retired: the ring is free for the [TN][TM] fp32 tile
    float *sv = reinterpret_cast<float *>(tiles);
    decode_stage_tile(acc0, acc1, sv, t);
    asm volatile("bar.sync 1, 128;" ::: "memory");
    const int nl = t;  // feature within the tile
    const int n = tile * TM + nl;
    if (splits == 1) {
      if (n < epi.N)
        for (int b = 0; b < epi.B; ++b) apply_epi(epi, n, b, sv[b * TM + nl]);
    } else if (!epi.red) {
      // partials[split][b][n]: for a fixed row b consecutive threads write consecutive features
      float *mine = partials + (int64_t)split * TN * ldp + n;
#pragma unroll 8
      for (int b = 0; b < TN; ++b) mine[(int64_t)b * ldp] = sv[b * TM + nl];
    }
    // epi.red: the tile stays in shared memory for the cluster reduction below
  }
  __syncwarp();
  // residual update x[0:B, tile] += sum of the splits' tiles + bias: the CTAs of a tile (its `splits` splits) form a
  // thread-block cluster; every CTA has parked its tile in shared memory, CTA r adds up rows [r R, (r+1) R) of all the
  // tiles over DSMEM in fixed order 0..S-1 and updates those residual rows itself (plain read-modify-write, no atomics),
  // so the result does not depend on which split finishes first
  if (epi.red && splits > 1) {
    asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
    if (warp >= 4) {
      const int nl = (warp & 3) * 32 + lane, n = tile * TM + nl;
      const int R = (TN + splits - 1) / splits;
      const int b_lo = split * R, b_hi = min(min(b_lo + R, TN), epi.B);
      const uint32_t sv_addr = smem_u32(tiles) + (uint32_t)nl * 4u;
      const float bias = (epi.bias && n < epi.N) ? epi.bias[n] : 0.f;
      // remote address of this thread's column in every rank's tile (rank j == split j: the cluster is a y column)
      uint32_t ra[kMaxClusterSplits];
#pragma unroll
      for (int j = 0; j < kMaxClusterSplits; ++j)
        asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(ra[j]) : "r"(sv_addr), "r"(min(j, splits - 1)));
#pragma unroll 2
      for (int b = b_lo; b < b_hi; ++b) {
        float t[kMaxClusterSplits];
#pragma unroll
        for (int j = 0; j < kMaxClusterSplits; ++j) {   // all ranks' values requested before the first add (DSMEM latency ~200 clocks)
          t[j] = 0.f;
          if (j < splits)
            asm volatile("ld.shared::cluster.f32 %0, [%1];" : "=f"(t[j]) : "r"(ra[j] + (uint32_t)(b * TM * 4)) : "memory");
        }
        float acc = t[0];
#pragma unroll
        for (int j = 1; j < kMaxClusterSplits; ++j) acc += t[j];   // fixed order 0..S-1
        if (n < epi.N) {
          float *o = epi.out_f32 + (int64_t)b * epi.ld_out + n;
          *o = *o + (acc + bias);
        }
      }
    }
    // nobody leaves while its tile may still be read
    asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
  }
  vb_trace(TR_GEMM * 2 + 1);
}

// ---- the same projection fed from the fp32 residual stream, LayerNorm folded into the weights ----------------
// LayerNorm(x) W^T = rstd (x (gamma o W)^T - mean c) + (beta W^T),  c[n] = sum_k gamma[k] W[n,k]: the tensor cores
// multiply the RAW rows by the pre-scaled weights, every CTA turns the fp32 rows of its k-range into the bf16
// 128B-swizzled operand tile itself (TMA brings the fp32 box, 8 warps convert it), and the moments of the rows
// (sum x, sum x^2 over the k-range) ride along as two more partial sums per split.  The consumer of the partials
// (attention prologue / ReLU reduce / sampler) applies rstd, mean, c and the folded bias -- the separate
// residual + LayerNorm launch between two projections (transformer.py:296-302,57-74) disappears from the chain.
constexpr int kStagesX = 4;   // the launcher picks the split count so that a CTA has <= 4 k-blocks where the split cap
                              // allows (d_model <= 4096): every tile in flight at once; beyond that the ring wraps
constexpr int kXfBytes = TN * BK * 4;  // 16 KB fp32 box
constexpr int kStageBytesX = kWBytes + kXBytes + kXfBytes;  // 40 KB
constexpr int kSmemBytesX = kStagesX * kStageBytesX + 1024 + 512;   // + alignment slack, barriers

constexpr int kThreadsX = 384;  // warp 0 TMA, 1..3 KV prefetch, 4..11 converters = the two MMA warpgroups + epilogue

__global__ void __launch_bounds__(kThreadsX, 1)
gemm_decode_x_kernel(const __grid_constant__ CUtensorMap tmap_w, const __grid_constant__ CUtensorMap tmap_xf,
                     int num_kb, float *__restrict__ partials, int ldp, float *__restrict__ stats, KvPrefetch pf) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t *tiles = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint64_t *bars = reinterpret_cast<uint64_t *>(tiles + kStagesX * kStageBytesX);
  uint64_t *wfull = bars, *xfull = bars + kStagesX, *bfull = bars + 2 * kStagesX, *empty_bar = bars + 3 * kStagesX;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tile = blockIdx.x, split = blockIdx.y, splits = gridDim.y;
  const int base = num_kb / splits, rem = num_kb % splits;
  const int kb0 = split * base + min(split, rem);
  const int nkb = base + (split < rem ? 1 : 0);

  pdl_launch_dependents();
  if (warp == 0 && lane == 0) {
    prefetch_tmap(&tmap_w);
    prefetch_tmap(&tmap_xf);
  }
  if (warp == 1 && lane == 0) {
    for (int i = 0; i < kStagesX; ++i) {
      mbar_init(&wfull[i], 1);
      mbar_init(&xfull[i], 1);
      mbar_init(&bfull[i], 8);
      mbar_init(&empty_bar[i], 8);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp == 0) {
    if (lane == 0) {
      const int pre = min(nkb, kStagesX);
      for (int i = 0; i < pre; ++i) {  // weights: independent of the previous kernel
        mbar_expect_tx(&wfull[i], kWBytes);
        tma_load_2d(&tmap_w, &wfull[i], tiles + i * kStageBytesX, (kb0 + i) * BK, tile * TM);
      }
      pdl_wait();
      vb_trace(TR_GEMM * 2);
      for (int i = 0; i < pre; ++i) {
        mbar_expect_tx(&xfull[i], kXfBytes);
        tma_load_2d(&tmap_xf, &xfull[i], tiles + i * kStageBytesX + kWBytes + kXBytes, (kb0 + i) * BK, 0);
      }
      int stage = 0;
      uint32_t phase = 1;
      for (int i = pre; i < nkb; ++i) {
        mbar_wait(&empty_bar[stage], phase ^ 1);
        uint8_t *dst = tiles + stage * kStageBytesX;
        mbar_expect_tx(&wfull[stage], kWBytes);
        tma_load_2d(&tmap_w, &wfull[stage], dst, (kb0 + i) * BK, tile * TM);
        mbar_expect_tx(&xfull[stage], kXfBytes);
        tma_load_2d(&tmap_xf, &xfull[stage], dst + kWBytes + kXBytes, (kb0 + i) * BK, 0);
        if (++stage == kStagesX) {
          stage = 0;
          phase ^= 1;
        }
      }
    }
    __syncwarp();
  } else if (warp < 4) {
    // idle warps: pull a slice of an upcoming layer's KV cache into L2 while the weight tiles stream
    kv_prefetch(pf, (blockIdx.y * gridDim.x + blockIdx.x) * 3 + (warp - 1), gridDim.x * gridDim.y * 3);
    pdl_wait();
  } else {
    // ---- converters: warp cw owns rows cw*8 .. +8 of every k-block; lane = (row parity, float4 of the row).
    //      Once all 8 warps have converted a stage, warpgroup h (warps 4 + 4h ..) multiplies weight rows [64 h, +64).
    const int cw = warp - 4, h = cw >> 2, t = threadIdx.x & 127;
    const int rsub = lane >> 4, f = lane & 15;
    float s1[4] = {0.f, 0.f, 0.f, 0.f}, s2[4] = {0.f, 0.f, 0.f, 0.f};
    float acc[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) acc[i] = 0.f;
    pdl_wait();
    int stage = 0, prev = -1;
    uint32_t phase = 0;
    for (int i = 0; i < nkb; ++i) {
      mbar_wait(&xfull[stage], phase);
      const uint8_t *xf = tiles + stage * kStageBytesX + kWBytes + kXBytes;
      uint8_t *xb = tiles + stage * kStageBytesX + kWBytes;
#pragma unroll
      for (int it = 0; it < 4; ++it) {
        const int r = cw * 8 + it * 2 + rsub;
        const float4 v = *reinterpret_cast<const float4 *>(xf + r * (BK * 4) + f * 16);
        s1[it] += (v.x + v.y) + (v.z + v.w);
        s2[it] = fmaf(v.x, v.x, fmaf(v.y, v.y, fmaf(v.z, v.z, fmaf(v.w, v.w, s2[it]))));
        __nv_bfloat162 p0 = __floats2bfloat162_rn(v.x, v.y), p1 = __floats2bfloat162_rn(v.z, v.w);
        uint2 pk;
        pk.x = *reinterpret_cast<uint32_t *>(&p0);
        pk.y = *reinterpret_cast<uint32_t *>(&p1);
        // 128B swizzle of a K-major row: 16-byte chunk c of row r lives at chunk c ^ (r & 7)
        *reinterpret_cast<uint2 *>(xb + r * 128 + ((((f >> 1) ^ (r & 7))) << 4) + (f & 1) * 8) = pk;
      }
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
      __syncwarp();
      if (lane == 0) mbar_arrive(&bfull[stage]);
      mbar_wait(&bfull[stage], phase);
      mbar_wait(&wfull[stage], phase);
      const uint32_t w_addr = smem_u32(tiles + stage * kStageBytesX) + h * (64 * 128);
      const uint64_t adesc = make_smem_desc(w_addr), bdesc = make_smem_desc(smem_u32(xb));
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < BK / WGMMA_K; ++k)
        wgmma_m64n64k16(acc, adesc + (uint64_t)(k * 2), bdesc + (uint64_t)(k * 2), 1);
      wgmma_commit();
      wgmma_wait<1>();
      if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
      prev = stage;
      if (++stage == kStagesX) {
        stage = 0;
        phase ^= 1;
      }
    }
    wgmma_wait<0>();
    wgmma_fence_regs(acc);
    if (tile < kLnFoldMaxCopies && stats != nullptr) {  // moments of this split's k-range: stats[tile][split][row][2]
#pragma unroll
      for (int it = 0; it < 4; ++it) {
#pragma unroll
        for (int o = 8; o > 0; o >>= 1) {
          s1[it] += __shfl_xor_sync(0xffffffffu, s1[it], o);
          s2[it] += __shfl_xor_sync(0xffffffffu, s2[it], o);
        }
        if (f == 0) {
          const int r = cw * 8 + it * 2 + rsub;
          *reinterpret_cast<float2 *>(stats + (((int64_t)tile * splits + split) * TN + r) * 2) =
              make_float2(s1[it], s2[it]);
        }
      }
    }
    // ---- epilogue: fp32 partial tile of this split, partials[split][b][n], straight from the fragments ----
    float *mine = partials + (int64_t)split * TN * ldp + tile * TM + h * 64;
#pragma unroll
    for (int i = 0; i < 32; ++i) mine[(int64_t)wg_col(t, i) * ldp + wg_row(t, i)] = acc[i];
  }
  vb_trace(TR_GEMM * 2 + 1);
}


}  // namespace dg

size_t gemm_decode_workspace(int d_model, int d_ff) {
  // fp32 partials [splits][64][ldp], ldp = tiles * 128: the automatic split count keeps tiles * splits <= #SMs;
  // the forced / tuned counts of the decode chain (api.cu, VB_SPLITS_*) are capped at kMaxForcedSplits per
  // projection, whose widest output is max(3 * d_model, d_ff) features
  const size_t tiles_max = ((size_t)std::max(3 * d_model, d_ff) + dg::TM - 1) / dg::TM;
  const size_t slabs = std::max((size_t)sm_count() + 32, tiles_max * kMaxForcedSplits);
  return slabs * dg::TN * dg::TM * sizeof(float);
}

static int pick_splits(int tiles, int num_kb) {
  int s = sm_count() / tiles;
  s = max(1, min(s, num_kb / 2));
  return max(1, min(s, kMaxForcedSplits));   // the consumers keep up to kMaxForcedSplits slabs of a column in flight
}

int launch_gemm_decode(const bf16 *act, int B, int64_t ld_act, const bf16 *W, int N, int K, int force_splits,
                       const float *bias, int mode, float *out_f32, bf16 *out_bf16, int64_t ld_out,
                       const QkvScatter *qkv, float *partials, size_t partial_bytes, SplitK *out,
                       const KvPrefetch *pf, bool pdl, cudaStream_t s, bool red_add) {
  VB_CHECK_ARG(B >= 1 && B <= dg::TN, "gemm_decode: B=%d not in [1,64]", B);
  VB_CHECK_ARG(!red_add || mode == DG_RESIDUAL, "gemm_decode: red_add needs the residual epilogue");
  VB_CHECK_ARG(K % tc::BK == 0 && ld_act % 8 == 0, "gemm_decode: K %% 64 != 0 or unaligned activations");
  const int tiles = (N + dg::TM - 1) / dg::TM;
  const int num_kb = K / tc::BK;
  int splits = force_splits > 0 ? std::min(force_splits, std::min(kMaxForcedSplits, num_kb)) : pick_splits(tiles, num_kb);
  // the splits of a residual update form one thread-block cluster: at most the portable cluster size
  if (red_add) splits = std::min(splits, dg::kMaxClusterSplits);
  const int ldp = tiles * dg::TM;
  if (splits > 1 && !red_add)
    VB_CHECK_ARG(partials && partial_bytes >= (size_t)splits * dg::TN * ldp * sizeof(float),
                 "gemm_decode: partial buffer too small");
  // a residual update adds its splits up in the cluster: nothing left for a consumer, and the partials stay unused
  if (red_add) partials = nullptr;
  *out = SplitK{splits > 1 ? partials : nullptr, red_add ? 1 : splits, ldp, bias};
  CUtensorMap tw, tx;
  VB_TRY(tc::make_tmap(&tw, W, N, K, K, dg::TM));
  VB_TRY(tc::make_tmap(&tx, act, B, K, ld_act, dg::TN));
  dg::Epi e{};
  e.mode = mode; e.N = N; e.B = B; e.bias = bias;
  e.red = red_add && splits > 1;
  e.out_f32 = out_f32; e.out_bf16 = out_bf16; e.ld_out = ld_out;
  if (mode == DG_QKV && splits == 1) {
    VB_CHECK_ARG(qkv != nullptr, "gemm_decode: qkv scatter parameters missing");
    e.qkv = *qkv;
  }
  static PerDeviceOnce once;
  if (once.first()) {
    VB_CUDA(cudaFuncSetAttribute(dg::gemm_decode_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 dg::kSmemBytes));
  }
  KvPrefetch pf0{};
  if (pf) pf0 = *pf;
  VB_CUDA(launch_kernel_cluster(dg::gemm_decode_kernel, dim3(tiles, splits), dim3(dg::kThreads), dg::kSmemBytes, s, pdl,
                                dim3(1, e.red ? splits : 1, 1), tw, tx, num_kb, partials, ldp, e, pf0));
  count_launch();
  return VB_OK;
}

// projection of the fp32 rows x[B, K] by LayerNorm-folded weights: fp32 partial tiles + the rows' moments per split
int launch_gemm_decode_x(const float *x, int B, int64_t ldx, const vb_ln_fold &F, int N, int K, int force_splits,
                         float *partials, size_t partial_bytes, float *stats, SplitK *out, const KvPrefetch *pf,
                         bool pdl, cudaStream_t s) {
  VB_CHECK_ARG(B >= 1 && B <= dg::TN, "gemm_decode_x: B=%d not in [1,64]", B);
  VB_CHECK_ARG(K % tc::BK == 0 && ldx % 4 == 0, "gemm_decode_x: K %% 64 != 0 or unaligned rows");
  const int tiles = (N + dg::TM - 1) / dg::TM;
  const int num_kb = K / tc::BK;
  int splits = force_splits > 0 ? std::min(force_splits, std::min(kMaxForcedSplits, num_kb)) : pick_splits(tiles, num_kb);
  // keep a CTA's k-range inside the ring where the split cap allows it (wider models: more splits rather than a
  // wrapping ring, whose later fp32 boxes would wait for the first MMAs)
  splits = std::max(splits, std::min(kMaxForcedSplits, (num_kb + dg::kStagesX - 1) / dg::kStagesX));
  const int ldp = tiles * dg::TM;
  VB_CHECK_ARG(partials && stats && partial_bytes >= (size_t)splits * dg::TN * ldp * sizeof(float),
               "gemm_decode_x: partial buffer too small");
  *out = SplitK{partials, splits, ldp, F.dvec,
                LnFoldStats{stats, F.c, splits, K, 1e-5f, std::min(tiles, kLnFoldMaxCopies)}};
  CUtensorMap tw, tx;
  VB_TRY(tc::make_tmap(&tw, (const bf16 *)F.wf, N, K, K, dg::TM));
  VB_TRY(tc::make_tmap_f32_dense(&tx, x, B, K, ldx, dg::TN, tc::BK));
  static PerDeviceOnce once;
  if (once.first())
    VB_CUDA(cudaFuncSetAttribute(dg::gemm_decode_x_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 dg::kSmemBytesX));
  KvPrefetch pf0{};
  if (pf) pf0 = *pf;
  VB_CUDA(launch_kernel(dg::gemm_decode_x_kernel, dim3(tiles, splits), dim3(dg::kThreadsX), dg::kSmemBytesX, s, pdl,
                        tw, tx, num_kb, partials, ldp, stats, pf0));
  count_launch();
  return VB_OK;
}

// ---- LayerNorm folding (host API vb_ln_fold_build): wf[n,k] = bf16(W[n,k] gamma[k]), c[n] = sum_k wf[n,k],
//      dvec[n] = bias[n] + sum_k beta[k] W[n,k]; one warp per output feature --------------------------------------
__global__ void __launch_bounds__(256)
ln_fold_kernel(const bf16 *__restrict__ W, int N, int K, const float *__restrict__ gamma,
               const float *__restrict__ beta, const float *__restrict__ bias, bf16 *__restrict__ wf,
               float *__restrict__ c, float *__restrict__ dvec) {
  const int n = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (n >= N) return;
  float cs = 0.f, ds = 0.f;
  for (int k = lane; k < K; k += 32) {
    const float w = __bfloat162float(W[(int64_t)n * K + k]);
    const bf16 f = __float2bfloat16_rn(w * gamma[k]);
    wf[(int64_t)n * K + k] = f;
    cs += __bfloat162float(f);
    ds = fmaf(beta[k], w, ds);
  }
  cs = warp_sum(cs);
  ds = warp_sum(ds);
  if (lane == 0) {
    c[n] = cs;
    dvec[n] = ds + (bias ? bias[n] : 0.f);
  }
}
int launch_ln_fold(const bf16 *W, int N, int K, const float *gamma, const float *beta, const float *bias, bf16 *wf,
                   float *c, float *dvec, cudaStream_t s) {
  VB_CUDA(launch_kernel(ln_fold_kernel, dim3((N + 7) / 8), dim3(256), 0, s, false, W, N, K, gamma, beta, bias, wf, c,
                        dvec));
  count_launch();
  return VB_OK;
}

}  // namespace vb
