// Attention kernels (head_dim = 64).
//   * attn_varlen_simt : softmax(q k^T / 8 + mask) v over packed ragged sequences, fp32 math in a
//     fixed order -- prefill of the AR decoder, NAR passes and the training forward in fp32
//     parity mode.  Also fills the KV cache.
//   * attn_decode      : one query row per (utterance, head) against the growing KV cache.
//     HBM-bound: 16-byte coalesced K/V reads, warp-shuffle dot products and softmax
//     reductions, split-KV across CTAs when B*H is too small to fill 132 SMs.
//
// Reference arithmetic: F.multi_head_attention_forward as called from
// valle/modules/activation.py:408-427; masks valle/models/valle.py:1010-1033 (AR) / none (NAR).
#include <math_constants.h>

#include <type_traits>

#include "common.cuh"
#include "kernels.cuh"

namespace vb {

static constexpr int HD = 64;

// ------------------------------------------------------------------------------------------
// Ragged multi-query attention, 64x64 tiles, 256 threads, 4x4 micro-tiles.
// ------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(256)
attn_varlen_simt_kernel(const T *__restrict__ qkv, int n_head, const Packed pk, T *__restrict__ out,
                        KvCache kv, const uint8_t *__restrict__ dmask, int64_t dld, DropCfg drop) {
  constexpr int LDT = 68;  // padded leading dim (floats), keeps float4 alignment
  extern __shared__ __align__(16) float smem[];
  float *Qt = smem;             // [64 e][LDT rows]
  float *Kt = Qt + 64 * LDT;    // [64 e][LDT keys]
  float *Vs = Kt + 64 * LDT;    // [64 keys][LDT e]
  float *Pt = Vs + 64 * LDT;    // [64 keys][LDT rows]

  const int b = blockIdx.z, h = blockIdx.y;
  const Packed::Seq sb = pk.seq(b);
  const int r0 = sb.r0, L = sb.L;
  const int q0 = blockIdx.x * 64;
  if (q0 >= L) return;
  const int d = n_head * HD;
  const int64_t ld = 3 * (int64_t)d;
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int lrow = tid >> 2, le0 = (tid & 3) * 16;

  // load Q tile (transposed)
  {
    const int qr = q0 + lrow;
    const T *src = qkv + (int64_t)(r0 + min(qr, L - 1)) * ld + h * HD + le0;
#pragma unroll
    for (int i = 0; i < 16; ++i) Qt[(le0 + i) * LDT + lrow] = (qr < L) ? to_f32(src[i]) : 0.f;
  }
  RowMask lim[4];  // visibility rule per owned row
#pragma unroll
  for (int i = 0; i < 4; ++i) lim[i] = pk.row_mask(sb, q0 + ty * 4 + i);
  const int kv_max = pk.kv_max(sb, min(q0 + 64, L));

  float m_run[4], l_run[4], o[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    m_run[i] = -CUDART_INF_F;
    l_run[i] = 0.f;
#pragma unroll
    for (int j = 0; j < 4; ++j) o[i][j] = 0.f;
  }

  for (int j0 = 0; j0 < kv_max; j0 += 64) {
    __syncthreads();  // previous tile fully consumed (also covers the Q store above)
    {
      const int kr = j0 + lrow;
      const bool ok = kr < L;
      const T *ksrc = qkv + (int64_t)(r0 + min(kr, L - 1)) * ld + d + h * HD + le0;
      const T *vsrc = ksrc + d;
      T kraw[16], vraw[16];
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        kraw[i] = ksrc[i];
        vraw[i] = vsrc[i];
      }
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        Kt[(le0 + i) * LDT + lrow] = ok ? to_f32(kraw[i]) : 0.f;
        Vs[lrow * LDT + le0 + i] = ok ? to_f32(vraw[i]) : 0.f;
      }
      if (kv.k != nullptr && j0 == q0 && ok) {  // this CTA owns rows [q0, q0+64) of the cache
        const int64_t off = kv.row(pk.cache_seq(b), h, kr) + le0;
        T *kc = (T *)kv.k + off, *vc = (T *)kv.v + off;
#pragma unroll
        for (int i = 0; i < 16; ++i) {
          kc[i] = kraw[i];
          vc[i] = vraw[i];
        }
      }
    }
    __syncthreads();
    // S = Q K^T
    float s[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) s[i][j] = 0.f;
#pragma unroll 8
    for (int e = 0; e < HD; ++e) {
      const float4 qa = *reinterpret_cast<const float4 *>(&Qt[e * LDT + ty * 4]);
      const float4 kb = *reinterpret_cast<const float4 *>(&Kt[e * LDT + tx * 4]);
      const float qv[4] = {qa.x, qa.y, qa.z, qa.w};
      const float kv[4] = {kb.x, kb.y, kb.z, kb.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) s[i][j] = fmaf(qv[i], kv[j], s[i][j]);
    }
    // online softmax per row (16 lanes share a row)
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      float mx = -CUDART_INF_F;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int c = j0 + tx * 4 + j;
        bool seen = lim[i].ok(c);
        if (dmask != nullptr && seen) seen = dmask[(int64_t)(q0 + ty * 4 + i) * dld + c] == 0;  // True = blocked
        s[i][j] = seen ? s[i][j] * 0.125f : -CUDART_INF_F;
        mx = fmaxf(mx, s[i][j]);
      }
#pragma unroll
      for (int off = 8; off > 0; off >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, off));
      const float m_new = fmaxf(m_run[i], mx);
      const float m_use = (m_new == -CUDART_INF_F) ? 0.f : m_new;
      const float corr = expf(m_run[i] - m_use);  // exp(-inf) = 0 on the first tile
      float rs = 0.f;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        s[i][j] = expf(s[i][j] - m_use);
        rs += s[i][j];
      }
#pragma unroll
      for (int off = 8; off > 0; off >>= 1) rs += __shfl_xor_sync(0xffffffffu, rs, off);
      l_run[i] = l_run[i] * corr + rs;
      m_run[i] = m_new;
#pragma unroll
      for (int j = 0; j < 4; ++j) o[i][j] *= corr;
      if (drop.thresh != 0) {   // training: dropout on the normalised probabilities = on p~ with the full row sum kept
        const uint64_t base = ((uint64_t)(b * n_head + h) * drop.lmax + (q0 + ty * 4 + i)) * drop.lmax + j0 + tx * 4;
#pragma unroll
        for (int j = 0; j < 4; ++j) s[i][j] = drop_keep(drop, base + j) ? s[i][j] * drop.inv_keep : 0.f;
      }
    }
    // P^T to shared: Pt[key][row]
#pragma unroll
    for (int j = 0; j < 4; ++j)
      *reinterpret_cast<float4 *>(&Pt[(tx * 4 + j) * LDT + ty * 4]) =
          make_float4(s[0][j], s[1][j], s[2][j], s[3][j]);
    __syncthreads();
    // O += P V
#pragma unroll 8
    for (int c = 0; c < 64; ++c) {
      const float4 pa = *reinterpret_cast<const float4 *>(&Pt[c * LDT + ty * 4]);
      const float4 vb4 = *reinterpret_cast<const float4 *>(&Vs[c * LDT + tx * 4]);
      const float pv[4] = {pa.x, pa.y, pa.z, pa.w};
      const float vv[4] = {vb4.x, vb4.y, vb4.z, vb4.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) o[i][j] = fmaf(pv[i], vv[j], o[i][j]);
    }
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int qr = q0 + ty * 4 + i;
    if (qr >= L) continue;
    const float inv = 1.f / l_run[i];
    T *dst = out + (int64_t)(r0 + qr) * d + h * HD + tx * 4;
#pragma unroll
    for (int j = 0; j < 4; ++j) dst[j] = from_f32<T>(o[i][j] * inv);
  }
}

int launch_attention_varlen(const void *qkv, int dtype, int64_t M, int n_head, int head_dim, const Packed &pk,
                            void *out, const KvCache &kv, const uint8_t *dense_mask, int64_t dense_ld, cudaStream_t s,
                            const DropCfg *drop) {
  VB_CHECK_ARG(head_dim == HD, "attention: head_dim=%d, only 64 is built", head_dim);
  DropCfg dc{};
  if (drop) dc = *drop;
  dc.lmax = pk.max_seqlen;
  Packed p = pk;
  if (p.mask_mode == VB_MASK_DENSE) {
    VB_CHECK_ARG(dense_mask != nullptr && dense_ld >= p.max_seqlen, "attention: VB_MASK_DENSE needs a [>=L, >=L] byte mask");
    p.mask_mode = VB_MASK_FULL;  // every key of the sequence, minus the blocked entries of the dense mask
  } else {
    dense_mask = nullptr;
  }
  VB_TRY(check_packed(p, "attention"));
  if (M == 0 || p.B == 0) return VB_OK;
  // attention-probability dropout and the dense mask are carried by the CUDA-core kernel only
  const bool wgmma = dtype == VB_BF16 && dc.thresh == 0 && dense_mask == nullptr && tune("VB_ATTN_SIMT", 0) == 0;
  if (kv.kexp != nullptr) {   // an FP8 cache is filled by the wgmma kernel only
    if (!wgmma) {
      set_error("attention: an FP8 KV cache is filled by the bf16 wgmma prefill only (no dropout, no dense mask, not VB_ATTN_SIMT)");
      return VB_ERR_UNSUPPORTED;
    }
    VB_CHECK_ARG(kv.k && kv.v && kv.vexp, "attention: FP8 cache: kcache, vcache, k_exp and v_exp are all needed");
  }
  if (wgmma) return launch_attention_wgmma((const bf16 *)qkv, M, n_head, p, (bf16 *)out, kv, s);
  VB_CHECK_ARG(dtype == VB_F32 || dtype == VB_BF16, "attention: bad dtype %d", dtype);
  auto simt = [&](auto elem) -> int {
    using T = decltype(elem);
    const size_t smem = 4 * 64 * 68 * sizeof(float);
    auto k = attn_varlen_simt_kernel<T>;
    VB_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k<<<dim3((p.max_seqlen + 63) / 64, n_head, p.B), 256, smem, s>>>((const T *)qkv, n_head, p, (T *)out, kv,
                                                                     dense_mask, dense_ld, dc);
    VB_LAUNCH_CHECK();
    return VB_OK;
  };
  return dtype == VB_F32 ? simt(float{}) : simt(bf16{});
}

// ------------------------------------------------------------------------------------------
// Single-query decode attention over the KV cache.
//   grid (H, B, nsplit), 128 threads.  kv_len[b] = S_b + Tp_b + n_gen[b].
//   kShared (kv_parent != NULL, best-of-n decoding; bf16 and fp32 caches): the rows below P_b come from the parent
//   row's streams (KvStreamRows); the same values in the same order as from the row's own copy of them.
//   kBeam (beam search; bf16 and fp32 caches): the generated rows below the current one come from the streams the
//   beam ancestry names, every row through a table of stream offsets the CTA stages in shared memory behind its
//   other buffers; again the same values in the same order as from a stream that holds them all.
// ------------------------------------------------------------------------------------------
static constexpr int kDecMaxChunk = 4096;

// 8 consecutive elements of an fp32 cache row
__device__ __forceinline__ void kv_row8_f32(const float *p, float (&f)[8]) {
  const uint4 a = ldg_stream16(p), b = ldg_stream16(p + 4);
  f[0] = __uint_as_float(a.x); f[1] = __uint_as_float(a.y); f[2] = __uint_as_float(a.z); f[3] = __uint_as_float(a.w);
  f[4] = __uint_as_float(b.x); f[5] = __uint_as_float(b.y); f[6] = __uint_as_float(b.z); f[7] = __uint_as_float(b.w);
}

// A finished utterance (stop rule fired, vb_ar_state.finished != 0) takes no further part in the step: its KV
// cache stays as it is (nothing appended, nothing streamed) and its attention output row is zero.  Uniform
// over the CTA.  Returns true if the CTA is done.
__device__ __forceinline__ bool decode_row_finished(const int32_t *finished, int b, int h, int sp, int d, int tid,
                                                    int nsplit, int n_head, float *out, bf16 *out16, float *part_o,
                                                    float *part_ml) {
  if (finished == nullptr || finished[b] == 0) return false;
  if (tid < HD) {
    if (nsplit == 1) {
      out[(int64_t)b * d + h * HD + tid] = 0.f;
      if (out16) out16[(int64_t)b * d + h * HD + tid] = __float2bfloat16_rn(0.f);
    } else {
      const int64_t pi = ((int64_t)b * n_head + h) * nsplit + sp;
      part_o[pi * HD + tid] = 0.f;
      if (tid == 0) {
        part_ml[pi * 2] = -CUDART_INF_F;
        part_ml[pi * 2 + 1] = 0.f;
      }
    }
  }
  return true;
}

// fp32 cache (the fp32 parity chain): q of the current token and its k / v row are already in place, written by the
// QKV projection.  Single pass, no block-level synchronisation inside the loop: each 8-lane group owns every 16th key
// of the chunk, streams the K row and the V row of its keys together (4 keys = 16 x 16-byte loads in flight per lane),
// and keeps its OWN online-softmax state (m, l, 8 output elements per lane).  The 16 groups are merged once at the end
// (flash-decoding style).
template <bool kShared = false, bool kBeam = false>
__global__ void __launch_bounds__(128)
attn_decode_kernel(const float *__restrict__ q, int n_head, KvCache kv, KvRows rows, float *__restrict__ out,
                   float *__restrict__ part_o, float *__restrict__ part_ml, int nsplit,
                   const int32_t *__restrict__ kv_parent, BeamAnc beam) {
  __shared__ __align__(16) float qs[HD];
  __shared__ float g_o[16][HD + 1];
  __shared__ float g_m[16], g_l[16];
  pdl_launch_dependents();
  const int h = blockIdx.x, b = blockIdx.y, sp = blockIdx.z;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int d = n_head * HD;
  pdl_wait();
  if (decode_row_finished(rows.finished, b, h, sp, d, threadIdx.x, nsplit, n_head, out, nullptr, part_o, part_ml)) return;
  const int pos = rows.cur(b, rows.n_gen[b], kv.cap);  // cache row of the current token
  const int kv_len = pos + 1;
  const int chunk = ((kv_len + nsplit - 1) / nsplit + 15) & ~15;
  const int c0 = sp * chunk, c1 = min(kv_len, c0 + chunk);
  const int n = max(0, c1 - c0);
  const float *kb = (const float *)kv.k + kv.row(b, h, 0);
  const float *vb_ = (const float *)kv.v + kv.row(b, h, 0);
  KvStreamRows<kShared, kBeam> sr(kv_parent, rows, kv, b);
  if constexpr (kBeam) {   // read after the __syncthreads below
    extern __shared__ __align__(16) int16_t beam_dl[];
    sr.stage_beam(beam_dl, kv_parent, rows, beam, b, c0, n, pos);
  }
  if (tid < HD) qs[tid] = q[(int64_t)b * d + h * HD + tid] * 0.125f;
  __syncthreads();

  const int grp = warp * 4 + (lane >> 3);  // 0..15
  const int j8 = (lane & 7) * 8;           // this lane's 8 head dims
  float qf[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) qf[i] = qs[j8 + i];
  float m = -CUDART_INF_F, l = 0.f, acc[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) acc[i] = 0.f;

  // The K and V rows of a tile are requested at the end of the tile before it, so that all 16 loads are in flight
  // together: requested at the top of the tile, the V loads would be scheduled behind the K dot products, one more
  // round trip to memory per tile.
  float kf[4][8], vf[4][8];
  auto load_tile = [&](int base) {
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int kk = min(base + u * 16 + grp, n - 1);
      kv_row8_f32(kb + sr.row(c0 + kk) + j8, kf[u]);
      kv_row8_f32(vb_ + sr.row(c0 + kk) + j8, vf[u]);
    }
  };
  if (n > 0) load_tile(0);
  for (int base = 0; base < n; base += 64) {
    float s[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int key = base + u * 16 + grp;
      float dot = 0.f;
#pragma unroll
      for (int i = 0; i < 8; ++i) dot = fmaf(qf[i], kf[u][i], dot);
      dot += __shfl_xor_sync(0xffffffffu, dot, 4);
      dot += __shfl_xor_sync(0xffffffffu, dot, 2);
      dot += __shfl_xor_sync(0xffffffffu, dot, 1);
      s[u] = key < n ? dot : -CUDART_INF_F;
    }
    const float mt = fmaxf(fmaxf(s[0], s[1]), fmaxf(s[2], s[3]));
    const float mn = fmaxf(m, mt);  // finite: key `base + grp` < n whenever this group has work ...
    if (mn != -CUDART_INF_F) {      // ... otherwise the group has no key in this tile at all
      const float corr = expf(m - mn);
      float p[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) p[u] = expf(s[u] - mn);
      l = l * corr + ((p[0] + p[1]) + (p[2] + p[3]));
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        float a = acc[i] * corr;
#pragma unroll
        for (int u = 0; u < 4; ++u) a = fmaf(p[u], vf[u][i], a);
        acc[i] = a;
      }
      m = mn;
    }
    if (base + 64 < n) load_tile(base + 64);
  }
  // ---- merge the 16 groups ------------------------------------------------------------------------
#pragma unroll
  for (int i = 0; i < 8; ++i) g_o[grp][j8 + i] = acc[i];
  if ((lane & 7) == 0) {
    g_m[grp] = m;
    g_l[grp] = l;
  }
  __syncthreads();
  if (tid < HD) {
    float mm = -CUDART_INF_F;
#pragma unroll
    for (int g = 0; g < 16; ++g) mm = fmaxf(mm, g_m[g]);
    float lt = 0.f, ot = 0.f;
#pragma unroll
    for (int g = 0; g < 16; ++g) {
      if (g_m[g] == -CUDART_INF_F) continue;
      const float w = expf(g_m[g] - mm);
      lt += g_l[g] * w;
      ot += g_o[g][tid] * w;
    }
    if (nsplit == 1) {
      out[(int64_t)b * d + h * HD + tid] = ot / lt;
    } else {
      const int64_t pi = ((int64_t)b * n_head + h) * nsplit + sp;
      part_o[pi * HD + tid] = ot;
      if (tid == 0) {
        part_ml[pi * 2] = n > 0 ? mm : -CUDART_INF_F;
        part_ml[pi * 2 + 1] = n > 0 ? lt : 0.f;
      }
    }
  }
}

// bf16 two-phase kernel (scores of the whole chunk to shared memory, block softmax, then P.V) with the FIRST batch
// of K rows fetched ahead of the q/k/v prologue (and, with the fused QKV prologue, ahead of the dependency wait)
// and the first batch of V rows fetched ahead of the block softmax: all CTAs of the single wave run their phases
// in lock step, so without this the HBM pipe idles through every prologue / softmax / epilogue of the launch.
// 8 CTAs per SM (<= 64 registers, which holds U = 4 K / V rows per thread without spilling): the 1,024 CTAs of B=64 x
// 16 heads are then resident at once on the H100's 132 SMs.  At 7 per SM (U = 8, 72 registers) 100 of them waited for
// the first wave to drain and then streamed their whole K and V alone.
// Fused QKV prologue (qp.part != nullptr): q/k/v of the CURRENT token arrive as split-K partials of the QKV
// projection (gemm_decode.cu); the CTA sums them in fixed order, adds the bias, appends k/v to the cache (split 0)
// and serves the new key/value from shared memory.  qp.fold.stats != NULL: the partials are x (gamma o W)^T of the
// raw rows (gemm_decode_x_kernel).
// CT = uint8_t: the FP8 cache (e4m3 rows, exponent bytes kexp / vexp; the fused QKV prologue is required).  A lane
// then loads 8 bytes (its 8 elements) per row, so U = 8 rows keep the same bytes and registers in flight as U = 4 bf16
// rows.  The exponents of the chunk come into shared memory by cp.async; 2^e is applied once per row: to the score
// (K) and to p_j ahead of P.V (V).  The current token's k / v are the unquantized bf16 rows, served from shared
// memory; split 0 appends their quantized rows.
template <int U, typename CT, bool kShared = false, bool kBeam = false>
__global__ void __launch_bounds__(128, 8)
attn_decode_2phase_pf_kernel(const float *__restrict__ q, SplitK qp, int n_head, KvCache kv, KvRows rows,
                   float *__restrict__ out, bf16 *__restrict__ out16,
                   float *__restrict__ part_o, float *__restrict__ part_ml, int nsplit,
                   const int32_t *__restrict__ kv_parent, BeamAnc beam) {
  constexpr bool kF8 = sizeof(CT) == 1;
  using Raw = typename std::conditional<kF8, uint2, uint4>::type;
  auto ld_raw = [](const CT *p) -> Raw {
    if constexpr (kF8) return ldg_stream8(p);
    else return ldg_stream16(p);
  };
  auto unpack_raw = [](const Raw &r, float (&f)[8]) {
    if constexpr (kF8) {
      kv8_unpack(r, f);
    } else {
      Vec16<bf16> v;
      v.raw = r;
      v.unpack(f);
    }
  };
  // score buffer of the chunk: dynamic shared memory sized by the launch (cache_cap / nsplit keys), so that the
  // kernel's footprint -- and with it the shared-memory carve-out the driver picks, i.e. how much L1 is left to land
  // the ~64 KB of K / V loads an SM keeps in flight -- follows the actual context instead of the 4096-key maximum
  extern __shared__ float sc[];
  __shared__ __align__(16) float qs[HD];
  __shared__ __align__(16) float knew[HD];
  __shared__ __align__(16) float vnew[HD];
  __shared__ float red[16][HD + 1];
  __shared__ float wred[8];
  __shared__ float pex[3][HD];
  pdl_launch_dependents();
  vb_trace_cta(16);   // CTA resident
  const int h = blockIdx.x, b = blockIdx.y, sp = blockIdx.z;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int d = n_head * HD;
  using T = bf16;
  CT *kb = (CT *)kv.k + kv.row(b, h, 0);
  CT *vb_ = (CT *)kv.v + kv.row(b, h, 0);
  KvStreamRows<kShared, kBeam> sr(kv_parent, rows, kv, b);
  const bool has_new = qp.part != nullptr;
  const int g = lane >> 3, j8 = (lane & 7) * 8;
  // The K rows of earlier tokens and the lengths do not depend on the kernels of THIS step that precede the
  // launch (the QKV projection only produces the current token), so the chunk geometry is worked out and the
  // first K batch is requested ahead of the dependency wait; the generated-token count is read again after
  // the wait and the batch re-requested should it have moved (it cannot when steps are separate graph launches).
  int kv_len, pos, c0, c1, n;
  Raw kraw[U];
  auto setup = [&](int n_generated) {
    pos = rows.cur(b, n_generated, kv.cap);  // cache row of the current token
    kv_len = pos + 1;
    const int chunk = ((kv_len + nsplit - 1) / nsplit + 15) & ~15;
    c0 = sp * chunk;
    c1 = min(kv_len, c0 + chunk);
    n = max(0, c1 - c0);
    if constexpr (kBeam) {   // the row table behind the score buffer (only after the dependency wait: see below)
      const int sc_len = ((kv.cap + nsplit - 1) / nsplit + 32 + 15) & ~15;
      sr.stage_beam(reinterpret_cast<int16_t *>(sc + sc_len), kv_parent, rows, beam, b, c0, n, pos);
      __syncthreads();
    }
    if (n > 0) {
#pragma unroll
      for (int u = 0; u < U; ++u)
        kraw[u] = ld_raw(kb + sr.row(c0 + min(u * 16 + warp * 4 + g, n - 1)) + j8);
    }
  };
  // (only with the fused QKV prologue: there the current token's row is served from shared memory; without it the
  // row was written to the cache by the kernel this launch depends on and nothing may be read ahead of the wait.
  // kBeam: the ancestry is written by the previous step's tail, so the rows are located only after the wait.)
  const int n_gen_early = (has_new && !kBeam) ? rows.n_gen[b] : -1;
  if (has_new && !kBeam) setup(n_gen_early);
  float qbias[3] = {0.f, 0.f, 0.f}, qc[3] = {0.f, 0.f, 0.f};
  if (tid < HD && has_new) {
#pragma unroll
    for (int j = 0; j < 3; ++j) {
      qbias[j] = qp.bias[j * d + h * HD + tid];
      if (qp.fold.stats) qc[j] = qp.fold.c[j * d + h * HD + tid];
    }
  }
  pdl_wait();
  vb_trace(TR_ATTN * 2);
  vb_trace_cta(17);   // dependency resolved
  if (decode_row_finished(rows.finished, b, h, sp, d, tid, nsplit, n_head, out, out16, part_o, part_ml)) return;
  int n_gen_now;
  asm volatile("ld.global.cg.s32 %0, [%1];" : "=r"(n_gen_now) : "l"(rows.n_gen + b) : "memory");
  if (n_gen_now != n_gen_early) setup(n_gen_now);  // uniform over the CTA
  // FP8: the chunk's exponent bytes -> shared memory (16-byte cp.async: c0 and kv.cap are multiples of 16), behind
  // the score buffer; read once the scores are in
  uint8_t *kes = nullptr, *ves = nullptr;
  if constexpr (kF8) {
    const int sc_len = ((kv.cap + nsplit - 1) / nsplit + 32 + 15) & ~15;
    kes = reinterpret_cast<uint8_t *>(sc + sc_len);
    ves = kes + sc_len;
    const int64_t e0 = kv.exp_index(b, h, c0);
    for (int i = tid; i < (n + 15) / 16; i += 128) {
      asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"((uint32_t)__cvta_generic_to_shared(kes + 16 * i)),
                   "l"(kv.kexp + e0 + 16 * i) : "memory");
      asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"((uint32_t)__cvta_generic_to_shared(ves + 16 * i)),
                   "l"(kv.vexp + e0 + 16 * i) : "memory");
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
  }
  if (has_new) {
    // q / k / v of the current token = sum of the projection's split-K partial tiles (+ folded LayerNorm, bias).  All 128
    // threads fetch: thread = (column c of the head, parity of the split), <= 3 splits x 3 columns each in ONE round
    // trip; the odd half hands its sums over through shared memory.  (A per-thread loop over the splits costs one
    // dependent L2 round trip per split.)
    const int c = tid & (HD - 1), hf = tid >> 6;
    float2 mraw = make_float2(0.f, 0.f);
    if (qp.fold.stats && hf == 0) mraw = ln_fold_moments_load(qp.fold, b, h);   // warps 0 and 1, complete
    float pv[3][3];   // (<= 6 splits in the one round trip; the chain uses 5)
#pragma unroll
    for (int j = 0; j < 3; ++j) {
      const float *p = qp.part + (int64_t)b * qp.ldp + j * d + h * HD + c;
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        const int s = hf + 2 * k;
        pv[j][k] = s < qp.splits ? __ldcg(p + (int64_t)s * 64 * qp.ldp) : 0.f;
      }
    }
    float mean = 0.f, rstd = 1.f;
    if (qp.fold.stats && hf == 0) ln_fold_moments_finish(qp.fold, mraw, mean, rstd);
    float acc[3];
#pragma unroll
    for (int j = 0; j < 3; ++j) {
      acc[j] = (pv[j][0] + pv[j][1]) + pv[j][2];
      const float *p = qp.part + (int64_t)b * qp.ldp + j * d + h * HD + c;
      for (int s = 6 + hf; s < qp.splits; s += 2) acc[j] += __ldcg(p + (int64_t)s * 64 * qp.ldp);
      if (hf == 1) pex[j][c] = acc[j];
    }
    __syncthreads();
    if (hf == 0) {
      float a[3];
#pragma unroll
      for (int j = 0; j < 3; ++j) a[j] = rstd * ((acc[j] + pex[j][c]) - mean * qc[j]) + qbias[j];
      qs[tid] = a[0] * 0.125f;
      const T k16 = from_f32<T>(a[1]), v16 = from_f32<T>(a[2]);
      knew[tid] = to_f32(k16);  // exactly what later steps will read back from the cache
      vnew[tid] = to_f32(v16);
      if constexpr (kF8) {   // the rows' max |.| over the head's 64 columns (warps 0 and 1)
        const float ak = warp_max(fabsf(to_f32(k16))), av = warp_max(fabsf(to_f32(v16)));
        if (lane == 0) {
          wred[warp] = ak;
          wred[2 + warp] = av;
        }
      } else if (sp == 0) {
        kb[(int64_t)pos * HD + tid] = k16;
        vb_[(int64_t)pos * HD + tid] = v16;
      }
    }
    if constexpr (kF8) {
      __syncthreads();
      if (hf == 0 && sp == 0) {   // append the quantized rows and their exponents
        const int ek = kv8_exp_biased(fmaxf(wred[0], wred[1])), ev = kv8_exp_biased(fmaxf(wred[2], wred[3]));
        kb[(int64_t)pos * HD + tid] = kv8_quant(knew[tid], ek);
        vb_[(int64_t)pos * HD + tid] = kv8_quant(vnew[tid], ev);
        if (tid == 0) {
          const int64_t e0 = kv.exp_index(b, h, pos);
          kv.kexp[e0] = (uint8_t)ek;
          kv.vexp[e0] = (uint8_t)ev;
        }
      }
    }
  } else if (tid < HD) {
    qs[tid] = q[(int64_t)b * d + h * HD + tid] * 0.125f;
  }
  __syncthreads();

  // ---- scores: 8 lanes per key, 4 keys per warp-iteration, 16 keys per CTA-iteration ----
  float qf[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) qf[i] = qs[j8 + i];
  float lmax = -CUDART_INF_F;
  const bool new_here = has_new && pos >= c0 && pos < c1;  // the current token's key lives in smem
  for (int base = 0; base < n; base += 16 * U) {
    if (base > 0) {
#pragma unroll
      for (int u = 0; u < U; ++u)
        kraw[u] = ld_raw(kb + sr.row(c0 + min(base + u * 16 + warp * 4 + g, n - 1)) + j8);
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int key = base + u * 16 + warp * 4 + g;
      float kf[8];
      unpack_raw(kraw[u], kf);
      float dot = 0.f;
#pragma unroll
      for (int i = 0; i < 8; ++i) dot = fmaf(qf[i], kf[i], dot);
      dot += __shfl_xor_sync(0xffffffffu, dot, 4);
      dot += __shfl_xor_sync(0xffffffffu, dot, 2);
      dot += __shfl_xor_sync(0xffffffffu, dot, 1);
      if ((lane & 7) == 0 && key < n && !(new_here && c0 + key == pos)) {
        sc[key] = dot;
        if constexpr (!kF8) lmax = fmaxf(lmax, dot);
      }
    }
  }
  // first batch of V rows in flight across the block softmax
  const int eg = (tid & 7) * 8, jl = tid >> 3;
  Raw vraw[U];
  if (n > 0) {
#pragma unroll
    for (int u = 0; u < U; ++u) vraw[u] = ld_raw(vb_ + sr.row(c0 + min(u * 16 + jl, n - 1)) + eg);
  }
  if (new_here && warp == 0) {  // score of the current token from the shared-memory key (never from the cache)
    float dot = 0.f;
    if (lane < 8) {
#pragma unroll
      for (int i = 0; i < 8; ++i) dot = fmaf(qf[i], knew[j8 + i], dot);
    }
    dot += __shfl_xor_sync(0xffffffffu, dot, 4);
    dot += __shfl_xor_sync(0xffffffffu, dot, 2);
    dot += __shfl_xor_sync(0xffffffffu, dot, 1);
    if (lane == 0) {
      sc[pos - c0] = dot;
      if constexpr (!kF8) lmax = fmaxf(lmax, dot);
    }
  }
  if constexpr (kF8) {   // the scores of the cached keys times 2^e_k (the current token's is exact as it stands)
    asm volatile("cp.async.wait_all;" ::: "memory");
    __syncthreads();
    for (int i = tid; i < n; i += 128) {
      float sv = sc[i];
      if (!(new_here && c0 + i == pos)) sv *= kv8_scale(kes[i]);
      sc[i] = sv;
      lmax = fmaxf(lmax, sv);
    }
  }
  lmax = warp_max(lmax);
  if (lane == 0) wred[warp] = lmax;
  __syncthreads();
  const float m = fmaxf(fmaxf(wred[0], wred[1]), fmaxf(wred[2], wred[3]));
  float lsum = 0.f;
  for (int i = tid; i < n; i += 128) {
    const float p = expf(sc[i] - m);
    if constexpr (kF8) sc[i] = (new_here && c0 + i == pos) ? p : p * kv8_scale(ves[i]);   // p_j 2^e_v for P.V
    else sc[i] = p;
    lsum += p;
  }
  lsum = warp_sum(lsum);
  if (lane == 0) wred[4 + warp] = lsum;
  __syncthreads();
  const float l = (wred[4] + wred[5]) + (wred[6] + wred[7]);

  // ---- O = P V : thread = (element group eg, key lane jl) --------------------------------
  float acc[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) acc[i] = 0.f;
  for (int base = 0; base < n; base += 16 * U) {
    if (base > 0) {
#pragma unroll
      for (int u = 0; u < U; ++u)
        vraw[u] = ld_raw(vb_ + sr.row(c0 + min(base + u * 16 + jl, n - 1)) + eg);
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int key = base + u * 16 + jl;
      const float pv = (key < n && !(new_here && c0 + key == pos)) ? sc[min(key, n - 1)] : 0.f;
      float vf[8];
      unpack_raw(vraw[u], vf);
#pragma unroll
      for (int i = 0; i < 8; ++i) acc[i] = fmaf(pv, vf[i], acc[i]);
    }
  }
  if (new_here && jl == 0) {
    const float pn = sc[pos - c0];
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[i] = fmaf(pn, vnew[eg + i], acc[i]);
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) red[jl][eg + i] = acc[i];
  __syncthreads();
  if (tid < HD) {
    float s = 0.f;
#pragma unroll
    for (int r = 0; r < 16; ++r) s += red[r][tid];
    if (nsplit == 1) {
      out[(int64_t)b * d + h * HD + tid] = s / l;
      if (out16) out16[(int64_t)b * d + h * HD + tid] = __float2bfloat16_rn(s / l);
    } else {
      const int64_t pi = ((int64_t)b * n_head + h) * nsplit + sp;
      part_o[pi * HD + tid] = s;
      if (tid == 0) {
        part_ml[pi * 2] = n > 0 ? m : -CUDART_INF_F;
        part_ml[pi * 2 + 1] = n > 0 ? l : 0.f;
      }
    }
  }
  vb_trace(TR_ATTN * 2 + 1);
  vb_trace_cta(18);   // CTA done
}

__global__ void attn_decode_combine_kernel(const float *__restrict__ part_o,
                                           const float *__restrict__ part_ml, int n_head, int nsplit,
                                           float *__restrict__ out, bf16 *__restrict__ out16) {
  pdl_launch_dependents();
  pdl_wait();
  vb_trace(TR_COMBINE * 2);
  const int h = blockIdx.x, b = blockIdx.y, e = threadIdx.x;
  const int64_t p0 = ((int64_t)b * n_head + h) * nsplit;
  float m = -CUDART_INF_F;
  for (int s = 0; s < nsplit; ++s) m = fmaxf(m, part_ml[(p0 + s) * 2]);
  float l = 0.f, o = 0.f;
  for (int s = 0; s < nsplit; ++s) {
    const float ms = part_ml[(p0 + s) * 2];
    if (ms == -CUDART_INF_F) continue;
    const float w = expf(ms - m);
    l += part_ml[(p0 + s) * 2 + 1] * w;
    o += part_o[(p0 + s) * HD + e] * w;
  }
  const float r = l > 0.f ? o / l : 0.f;  // l == 0: a finished utterance (every split empty)
  out[(int64_t)b * n_head * HD + h * HD + e] = r;
  if (out16) out16[(int64_t)b * n_head * HD + h * HD + e] = __float2bfloat16_rn(r);
}

static int decode_nsplit(int B, int n_head, int cache_cap) {
  const int forced = tune("VB_DECODE_NSPLIT", 0);
  if (forced > 0) return forced;
  int ns = (2 * sm_count() + B * n_head - 1) / (B * n_head);
  ns = max(1, min(ns, 32));
  ns = min(ns, max(1, cache_cap / 64));              // keep chunks >= 64 keys
  ns = max(ns, (cache_cap + kDecMaxChunk - 1) / kDecMaxChunk);  // chunk must fit the score buffer
  return ns;
}

size_t attn_decode_workspace(int B, int n_head, int head_dim, int cache_cap) {
  const int ns = decode_nsplit(B, n_head, cache_cap);
  return (size_t)B * n_head * ns * (head_dim + 2) * sizeof(float) + 256;
}

// VB_ATTN_CARVEOUT: shared-memory carve-out (percent) preferred for the two-phase decode kernels; -1 = the driver's
// choice.  A fixed carve-out keeps the SMs from re-partitioning on the way in and out of every attention launch of the
// chain; the largest carve-out leaves no L1 for the loads in flight.  (Default not re-tuned on H100.)  Set on the
// current device whenever the knob differs from what kernel `kKernel` last got there; the driver's choice needs no
// call until another value has been set.
template <auto kKernel>
static int set_attn_carveout() {
  static int set[64];
  static bool init = false;
  if (!init) {
    for (int i = 0; i < 64; ++i) set[i] = -2;
    init = true;
  }
  int dev = 0;
  cudaGetDevice(&dev);
  const int carve = tune("VB_ATTN_CARVEOUT", 72);
  if (set[dev & 63] != carve) {
    const int want = carve >= 0 ? carve : (int)cudaSharedmemCarveoutDefault;
    if (carve >= 0 || set[dev & 63] != -2)
      VB_CUDA(cudaFuncSetAttribute(kKernel, cudaFuncAttributePreferredSharedMemoryCarveout, want));
    set[dev & 63] = carve;
  }
  return VB_OK;
}

int launch_attn_decode(const QkvScatter &kv, const SplitK &qkv, int B, int n_head, int dtype, float *out, void *out16,
                       void *workspace, bool pdl, cudaStream_t s, const int32_t *kv_parent, const BeamAnc &beam) {
  VB_CHECK_ARG(kv.head_dim == HD, "attn_decode: head_dim=%d, only 64 is built", kv.head_dim);
  const int cache_cap = kv.kv.cap;
  const int ns = decode_nsplit(B, n_head, cache_cap);
  VB_CHECK_ARG((cache_cap + ns - 1) / ns + 16 <= kDecMaxChunk, "attn_decode: cache_cap %d too large", cache_cap);
  float *part_o = (float *)workspace;
  float *part_ml = part_o + (size_t)B * n_head * ns * HD;
  dim3 grid(n_head, B, ns);
  // beam search: the chunk's row table, int16 per row, behind the score buffer of the two-phase kernel (sized as the
  // kernel sizes it) or alone (fp32 kernel); kBeam instantiations take kShared = true
  const bool bm = beam.anc != nullptr;
  const int dl_len = ((cache_cap + ns - 1) / ns + 32 + 15) & ~15;
  if (dtype == VB_E4M3) {
    VB_CHECK_ARG(qkv.part != nullptr && kv.kv.kexp != nullptr && kv.kv.vexp != nullptr && cache_cap % 16 == 0,
                 "attn_decode: the FP8 cache needs the fused QKV prologue, exponent arrays and cache_cap %% 16 == 0");
    // score buffer as for bf16 (rounded to 16 floats), then the chunk's K and V exponent bytes
    const int sc_len = ((cache_cap + ns - 1) / ns + 32 + 15) & ~15;
    const size_t smem = align_up((size_t)sc_len * (sizeof(float) + 2), 1024);
    constexpr auto k = attn_decode_2phase_pf_kernel<8, uint8_t>;
    VB_TRY(set_attn_carveout<k>());
    VB_CUDA(launch_kernel(k, grid, dim3(128), smem, s, pdl, (const float *)kv.q, qkv, n_head, kv.kv, kv.rows, out,
                          (bf16 *)out16, part_o, part_ml, ns, nullptr, BeamAnc{}));   // no shared rows (vb_ar_decode_step)
  } else if (dtype == VB_F32) {
    VB_CHECK_ARG(qkv.part == nullptr && out16 == nullptr,
                 "attn_decode: the fp32 cache takes q and the k / v rows in place, and writes fp32 rows only");
    const auto k = bm ? attn_decode_kernel<true, true> : kv_parent ? attn_decode_kernel<true> : attn_decode_kernel<>;
    VB_CUDA(launch_kernel(k, grid, dim3(128), bm ? dl_len * sizeof(int16_t) : 0, s, pdl, (const float *)kv.q, n_head,
                          kv.kv, kv.rows, out, part_o, part_ml, ns, kv_parent, beam));
  } else if (bm) {
    constexpr auto k_bm = attn_decode_2phase_pf_kernel<4, bf16, true, true>;
    VB_TRY(set_attn_carveout<k_bm>());
    VB_CUDA(launch_kernel(k_bm, grid, dim3(128), align_up((size_t)dl_len * (sizeof(float) + sizeof(int16_t)), 1024),
                          s, pdl, (const float *)kv.q, qkv, n_head, kv.kv, kv.rows, out, (bf16 *)out16, part_o, part_ml,
                          ns, kv_parent, beam));
  } else {
    // score buffer: the chunk of one split, rounded as the kernel rounds it (+16), in 1 KB steps
    const size_t sc_bytes = align_up((size_t)((cache_cap + ns - 1) / ns + 32) * sizeof(float), 1024);
    constexpr auto k = attn_decode_2phase_pf_kernel<4, bf16>;
    constexpr auto k_sh = attn_decode_2phase_pf_kernel<4, bf16, true>;
    if (kv_parent) VB_TRY(set_attn_carveout<k_sh>());
    else VB_TRY(set_attn_carveout<k>());
    VB_CUDA(launch_kernel(kv_parent ? k_sh : k, grid, dim3(128), sc_bytes, s, pdl, (const float *)kv.q, qkv, n_head,
                          kv.kv, kv.rows, out, (bf16 *)out16, part_o, part_ml, ns, kv_parent, beam));
  }
  count_launch();
  if (ns > 1) {
    VB_CUDA(launch_kernel(attn_decode_combine_kernel, dim3(n_head, B), dim3(HD), 0, s, pdl, (const float *)part_o,
                          (const float *)part_ml, n_head, ns, out, (bf16 *)out16));
    count_launch();
  }
  return VB_OK;
}

}  // namespace vb

VB_API int vb_attention(const void *qkv, int dtype, int64_t M, int B, int n_head, int head_dim,
                        const int32_t *cu_seqlens, const int32_t *text_lens, const int32_t *seg1_lens, int seg1_start,
                        int max_seqlen, int mask_mode, void *out, void *kcache, void *vcache,
                        int64_t cache_seq_stride, int cache_cap, const uint8_t *dense_mask, int64_t dense_ld,
                        vb_stream_t stream) {
  const vb::KvCache kv{kcache, vcache, nullptr, nullptr, cache_seq_stride, cache_cap, (int)vb::elem_size(dtype)};
  const vb::Packed pk{cu_seqlens, text_lens, seg1_lens, B, max_seqlen, seg1_start, mask_mode};
  return vb::launch_attention_varlen(qkv, dtype, M, n_head, head_dim, pk, out, kv, dense_mask, dense_ld,
                                     (cudaStream_t)stream);
}
