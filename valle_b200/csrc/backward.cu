// Backward pass of the training forward (VALLE.forward, valle/models/valle.py:762-959 -> loss.backward() at
// valle/bin/trainer.py:674): the gradients torch.autograd would produce for the reference's modules, computed by
// hand-written kernels behind the C ABI.
//
//   * GEMM gradients reuse the forward GEMM kernels (wgmma for bf16 operands, exact-order CUDA-core for fp32):
//       dgrad  dX[M,K] = dY[M,N] W[N,K]        = linear(dY, W^T)          (W^T kept by the caller per step)
//       wgrad  dW[N,K] += dY^T[N,M] X[M,K]     = linear(dY^T, X^T) with the fp32 accumulate epilogue
//     the two activation transposes are explicit memory-bound passes (transpose_pad_kernel);
//   * LayerNorm / AdaptiveLayerNorm backward (transformer.py:57-108), ReLU mask, bias column sums,
//     cross-entropy backward (softmax - onehot), embedding scatter-add, sine-PE alpha gradient;
//   * attention backward (F.multi_head_attention_forward, activation.py:408-427) as two fp32 CUDA-core passes over
//     64 x 64 tiles with recomputed probabilities: per query block (log-sum-exp, D = rowsum(dO o O), dQ) and per key
//     block (dK, dV) -- no atomics, deterministic.
#include <math_constants.h>

#include <algorithm>

#include "common.cuh"
#include "kernels.cuh"

namespace vb {
namespace bw {

// ---- out[c][r] = in[r][c], rows r >= R of the padded leading dimension are zero ---------------------------
template <typename T>
__global__ void transpose_pad_kernel(const T *__restrict__ in, int64_t ld_in, int64_t R, int C, T *__restrict__ out,
                                     int64_t ld_out) {
  __shared__ T tile[32][33];
  const int64_t r0 = (int64_t)blockIdx.x * 32;
  const int c0 = blockIdx.y * 32;
  for (int i = threadIdx.y; i < 32; i += 8) {
    const int64_t r = r0 + i;
    const int c = c0 + threadIdx.x;
    tile[i][threadIdx.x] = (r < R && c < C) ? in[r * ld_in + c] : from_f32<T>(0.f);
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += 8) {
    const int c = c0 + i;
    const int64_t r = r0 + threadIdx.x;
    if (c < C && r < ld_out) out[(int64_t)c * ld_out + r] = tile[threadIdx.x][i];
  }
}

// ---- out[n] += sum_r in[r][n]  (bias gradients) ------------------------------------------------------------
template <typename T>
__global__ void colsum_kernel(const T *__restrict__ in, int64_t ld, int64_t R, int N, float *__restrict__ out,
                              int64_t rows_per_cta) {
  __shared__ float red[8][33];
  const int n = blockIdx.x * 32 + threadIdx.x;
  const int64_t r0 = (int64_t)blockIdx.y * rows_per_cta, r1 = min(R, r0 + rows_per_cta);
  float s = 0.f;
  if (n < N)
    for (int64_t r = r0 + threadIdx.y; r < r1; r += 8) s += to_f32(in[r * ld + n]);
  red[threadIdx.y][threadIdx.x] = s;
  __syncthreads();
  if (threadIdx.y == 0 && n < N) {
    float t = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) t += red[i][threadIdx.x];
    atomicAdd(out + n, t);
  }
}

// ---- dh = (h > 0) ? dh * scale : 0   (scale = 1 / keep when h went through dropout: dropped entries are 0 in h) ------
template <typename T>
__global__ void relu_bwd_kernel(T *__restrict__ dh, const T *__restrict__ h, int64_t n, float scale) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    if (!(to_f32(h[i]) > 0.f)) dh[i] = from_f32<T>(0.f);
    else if (scale != 1.f) dh[i] = from_f32<T>(to_f32(dh[i]) * scale);
  }
}

// ---- dropout (element index = linear offset into the contiguous tensor) ------------------------------------------
template <typename T>
__global__ void dropout_kernel(const T *__restrict__ in, T *__restrict__ out, int64_t n, DropCfg cfg) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    out[i] = drop_keep(cfg, (uint64_t)i) ? from_f32<T>(to_f32(in[i]) * cfg.inv_keep) : from_f32<T>(0.f);
}
__global__ void dropout_add_kernel(float *__restrict__ x, const float *__restrict__ t, int64_t n, DropCfg cfg) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    if (drop_keep(cfg, (uint64_t)i)) x[i] += t[i] * cfg.inv_keep;
}

// ---- LayerNorm / AdaptiveLayerNorm backward --------------------------------------------------------------------
// forward: y = a_w * (gamma * xhat + beta) + a_b   (a_w = 1, a_b = 0 without AdaLN), xhat = (x - mu) * rstd
// One warp per row; dx_io[xrow] += dLN/dx; optional dt copy of the updated dx row; parameter gradients are summed
// per CTA in shared memory and added to the fp32 gradient vectors with one atomic per column and CTA.
template <typename TD>
__global__ void __launch_bounds__(256)
ln_bwd_kernel(const float *__restrict__ x, int64_t ldx, const int32_t *__restrict__ rows, int64_t n_rows, int d,
              const float *__restrict__ gamma, const float *__restrict__ beta, const float *__restrict__ ada_wb,
              float eps, const float *__restrict__ dy, int64_t ld_dy, float *__restrict__ dx_io, int64_t ld_dx,
              TD *__restrict__ dx_copy, float *__restrict__ dgamma, float *__restrict__ dbeta,
              float *__restrict__ dada_wb, int rows_per_cta) {
  extern __shared__ float sm[];  // [4][d]: dgamma, dbeta, dada_w, dada_b partial sums of this CTA
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int i = threadIdx.x; i < 4 * d; i += 256) sm[i] = 0.f;
  __syncthreads();
  const int64_t r_begin = (int64_t)blockIdx.x * rows_per_cta;
  const int64_t r_end = min(n_rows, r_begin + rows_per_cta);
  for (int64_t r = r_begin + warp; r < r_end; r += 8) {
    const int64_t xr = rows ? (int64_t)rows[r] : r;
    const float *xp = x + xr * ldx;
    const float *dyp = dy + r * ld_dy;
    float s = 0.f;
    for (int c = lane; c < d; c += 32) s += xp[c];
    const float mu = warp_sum(s) / (float)d;
    float q = 0.f;
    for (int c = lane; c < d; c += 32) {
      const float t = xp[c] - mu;
      q += t * t;
    }
    const float rstd = rsqrtf(warp_sum(q) / (float)d + eps);
    float m1 = 0.f, m2 = 0.f;
    for (int c = lane; c < d; c += 32) {
      const float xhat = (xp[c] - mu) * rstd;
      const float aw = ada_wb ? ada_wb[c] : 1.f;
      const float g = dyp[c] * aw * gamma[c];
      m1 += g;
      m2 += g * xhat;
    }
    m1 = warp_sum(m1) / (float)d;
    m2 = warp_sum(m2) / (float)d;
    float *dxp = dx_io + xr * ld_dx;
    for (int c = lane; c < d; c += 32) {
      const float xhat = (xp[c] - mu) * rstd;
      const float aw = ada_wb ? ada_wb[c] : 1.f;
      const float dyv = dyp[c];
      const float g = dyv * aw * gamma[c];
      const float v = dxp[c] + rstd * (g - m1 - xhat * m2);
      dxp[c] = v;
      if (dx_copy) dx_copy[xr * (int64_t)d + c] = from_f32<TD>(v);
      atomicAdd(&sm[c], dyv * aw * xhat);
      atomicAdd(&sm[d + c], dyv * aw);
      if (ada_wb) {
        atomicAdd(&sm[2 * d + c], dyv * (gamma[c] * xhat + beta[c]));
        atomicAdd(&sm[3 * d + c], dyv);
      }
    }
  }
  __syncthreads();
  for (int c = threadIdx.x; c < d; c += 256) {
    if (dgamma) atomicAdd(dgamma + c, sm[c]);
    if (dbeta) atomicAdd(dbeta + c, sm[d + c]);
    if (dada_wb && ada_wb) {
      atomicAdd(dada_wb + c, sm[2 * d + c]);
      atomicAdd(dada_wb + d + c, sm[3 * d + c]);
    }
  }
}

// ---- cross-entropy backward: dlogits[r, :] = g[r] * (softmax(logits[r, :]) - onehot(target[r])) -----------------
template <typename TD>
__global__ void ce_bwd_kernel(const float *__restrict__ logits, int64_t ld, const int64_t *__restrict__ targets,
                              int64_t n_rows, int n_vocab, int64_t ignore_index, const float *__restrict__ grad_rows,
                              float grad_scale, TD *__restrict__ dlogits, int64_t ld_out, int n_out) {
  const int64_t r = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (r >= n_rows) return;
  const int lane = threadIdx.x & 31;
  const float *row = logits + r * ld;
  const int64_t tg = targets[r];
  const bool skip = (tg == ignore_index || tg < 0 || tg >= n_vocab);
  const float g = skip ? 0.f : grad_scale * (grad_rows ? grad_rows[r] : 1.f);
  float mx = -CUDART_INF_F;
  for (int i = lane; i < n_vocab; i += 32) mx = fmaxf(mx, row[i]);
  mx = warp_max(mx);
  float s = 0.f;
  for (int i = lane; i < n_vocab; i += 32) s += expf(row[i] - mx);
  s = warp_sum(s);
  const float inv = 1.f / s;
  TD *o = dlogits + r * ld_out;
  for (int i = lane; i < n_out; i += 32) {
    float v = 0.f;
    if (i < n_vocab) v = g * (expf(row[i] - mx) * inv - ((int64_t)i == tg ? 1.f : 0.f));
    o[i] = from_f32<TD>(v);
  }
}

// ---- embedding backward: table_grad[j][ids[r, j], :] += dy[orow(r), :] ---------------------------------------
constexpr int kMaxTables = 8;
struct GradTables {
  float *t[kMaxTables];
  int rows[kMaxTables];
};
__global__ void embed_bwd_kernel(const int64_t *__restrict__ tokens, int64_t tok_row_stride, int64_t tok_tab_stride,
                                 GradTables tabs, int n_tables, int64_t n_rows, int d, const float *__restrict__ dy,
                                 int64_t dy_row_stride, const int32_t *__restrict__ dy_rows) {
  const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= n_rows) return;
  const int lane = threadIdx.x & 31;
  const float *g = dy + (dy_rows ? (int64_t)dy_rows[row] : row) * dy_row_stride;
  for (int j = 0; j < n_tables; ++j) {
    int64_t id = tokens[row * tok_row_stride + j * tok_tab_stride];
    if (id < 0 || id >= tabs.rows[j]) continue;  // flagged by the forward pass
    float *dst = tabs.t[j] + id * d;
    for (int c = lane; c < d; c += 32) atomicAdd(dst + c, g[c]);
  }
}

// ---- out[0] += sum_r <a[r, :], b[pos(r), :]>   (gradient of the sine-PE alpha, embedding.py:93-97) -------------
__global__ void rowdot_kernel(const float *__restrict__ a, int64_t lda, const float *__restrict__ b, int64_t pos0,
                              const int32_t *__restrict__ positions, int64_t n_rows, int d, float *__restrict__ out) {
  __shared__ float red[8];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float s = 0.f;
  for (int64_t r = (int64_t)blockIdx.x * 8 + warp; r < n_rows; r += (int64_t)gridDim.x * 8) {
    const float *ap = a + r * lda;
    const float *bp = b + (positions ? (int64_t)positions[r] : pos0 + r) * d;
    for (int c = lane; c < d; c += 32) s += ap[c] * bp[c];
  }
  s = warp_sum(s);
  if (lane == 0) red[warp] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int i = 0; i < 8; ++i) t += red[i];
    atomicAdd(out, t);
  }
}

// ---- AdaLN projection backward: wb[2d] = W[2d, d] e[d] + b[2d] (transformer.py:96-100) -----------------------
// dW[i, k] += dwb[i] e[k]; db[i] += dwb[i]; de[k] += sum_i W[i, k] dwb[i]
__global__ void adaln_proj_bwd_kernel(const float *__restrict__ W, const float *__restrict__ e,
                                      const float *__restrict__ dwb, int d, float *__restrict__ dW,
                                      float *__restrict__ db, float *__restrict__ de) {
  const int i = blockIdx.x;  // row of W (0 .. 2d)
  const float g = dwb[i];
  if (threadIdx.x == 0 && db) atomicAdd(db + i, g);
  for (int k = threadIdx.x; k < d; k += blockDim.x) {
    if (dW) atomicAdd(dW + (int64_t)i * d + k, g * e[k]);
    if (de) atomicAdd(de + k, W[(int64_t)i * d + k] * g);
  }
}

// ------------------------------------------------------------------------------------------------------------
// Attention backward, 64 x 64 tiles, 256 threads, 4 x 4 micro-tiles (same tiling as attn_varlen_simt_kernel).
// qkv [M, 3d] (Q|K|V), o [M, d] forward output, dout [M, d]; dqkv [M, 3d] written (every element exactly once).
// ------------------------------------------------------------------------------------------------------------
constexpr int HD = 64, LDT = 68;

template <typename T>
__device__ __forceinline__ void load_tile_t(float *dst /*[64 e][LDT]*/, const T *src, int64_t ld, int r0, int L, int col0,
                                            int tid) {
  // dst[e][row] = src[(r0 + row) * ld + col0 + e], rows >= L zero
  const int lrow = tid >> 2, le0 = (tid & 3) * 16;
  const int r = r0 + lrow;
  const T *p = src + (int64_t)min(r, L - 1) * ld + col0 + le0;
#pragma unroll
  for (int i = 0; i < 16; ++i) dst[(le0 + i) * LDT + lrow] = (r < L) ? to_f32(p[i]) : 0.f;
}
template <typename T>
__device__ __forceinline__ void load_tile_n(float *dst /*[64 row][LDT]*/, const T *src, int64_t ld, int r0, int L, int col0,
                                            int tid) {
  const int lrow = tid >> 2, le0 = (tid & 3) * 16;
  const int r = r0 + lrow;
  const T *p = src + (int64_t)min(r, L - 1) * ld + col0 + le0;
#pragma unroll
  for (int i = 0; i < 16; ++i) dst[lrow * LDT + le0 + i] = (r < L) ? to_f32(p[i]) : 0.f;
}
// acc[i][j] = sum_e A[e][ty*4+i] * B[e][tx*4+j]   (both operands stored e-major)
__device__ __forceinline__ void mm_tt(const float *A, const float *B, int ty, int tx, float (&acc)[4][4]) {
#pragma unroll 8
  for (int e = 0; e < HD; ++e) {
    const float4 a = *reinterpret_cast<const float4 *>(&A[e * LDT + ty * 4]);
    const float4 b = *reinterpret_cast<const float4 *>(&B[e * LDT + tx * 4]);
    const float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
  }
}

// pass 1: per (query block, head, sequence): lse, D = rowsum(dO o O), dQ
template <typename T>
__global__ void __launch_bounds__(256)
attn_bwd_dq_kernel(const T *__restrict__ qkv, const T *__restrict__ o, const T *__restrict__ dout, int n_head,
                   const Packed pk, T *__restrict__ dqkv, float *__restrict__ lse_out,
                   float *__restrict__ dsum_out, DropCfg drop) {
  extern __shared__ __align__(16) float smem[];
  float *Qt = smem;              // [e][q]
  float *dOt = Qt + 64 * LDT;    // [e][q]
  float *Kt = dOt + 64 * LDT;    // [e][key]
  float *Vt = Kt + 64 * LDT;     // [e][key]
  float *Kn = Vt + 64 * LDT;     // [key][e]
  float *dSt = Kn + 64 * LDT;    // [key][q]
  __shared__ float s_lse[64], s_D[64];
  const int b = blockIdx.z, h = blockIdx.y;
  const Packed::Seq sb = pk.seq(b);
  const int r0 = sb.r0, L = sb.L;
  const int q0 = blockIdx.x * 64;
  if (q0 >= L) return;
  const int d = n_head * HD;
  const int64_t ld = 3 * (int64_t)d;
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const T *qb = qkv + (int64_t)r0 * ld;
  load_tile_t(Qt, qb, ld, q0, L, h * HD, tid);
  load_tile_t(dOt, dout + (int64_t)r0 * d, (int64_t)d, q0, L, h * HD, tid);
  {  // D[row] = sum_e dO * O : 4 threads per row
    const int lrow = tid >> 2, le0 = (tid & 3) * 16;
    const int r = q0 + lrow;
    float s = 0.f;
    if (r < L) {
      const T *op = o + (int64_t)(r0 + r) * d + h * HD + le0;
      const T *gp = dout + (int64_t)(r0 + r) * d + h * HD + le0;
#pragma unroll
      for (int i = 0; i < 16; ++i) s += to_f32(op[i]) * to_f32(gp[i]);
    }
    s += __shfl_xor_sync(0xffffffffu, s, 1);
    s += __shfl_xor_sync(0xffffffffu, s, 2);
    if ((tid & 3) == 0) s_D[lrow] = s;
  }
  RowMask lim[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) lim[i] = pk.row_mask(sb, q0 + ty * 4 + i);
  const int kv_max = pk.kv_max(sb, min(q0 + 64, L));
  // ---- sweep 1: log-sum-exp of every query row ----
  float m_run[4], l_run[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    m_run[i] = -CUDART_INF_F;
    l_run[i] = 0.f;
  }
  for (int j0 = 0; j0 < kv_max; j0 += 64) {
    __syncthreads();
    load_tile_t(Kt, qb, ld, j0, L, d + h * HD, tid);
    __syncthreads();
    float s[4][4] = {};
    mm_tt(Qt, Kt, ty, tx, s);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      float mx = -CUDART_INF_F;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        s[i][j] = lim[i].ok(j0 + tx * 4 + j) ? s[i][j] * 0.125f : -CUDART_INF_F;
        mx = fmaxf(mx, s[i][j]);
      }
#pragma unroll
      for (int off = 8; off > 0; off >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, off));
      const float m_new = fmaxf(m_run[i], mx);
      const float m_use = (m_new == -CUDART_INF_F) ? 0.f : m_new;
      float rs = 0.f;
#pragma unroll
      for (int j = 0; j < 4; ++j) rs += expf(s[i][j] - m_use);
#pragma unroll
      for (int off = 8; off > 0; off >>= 1) rs += __shfl_xor_sync(0xffffffffu, rs, off);
      l_run[i] = l_run[i] * expf(m_run[i] - m_use) + rs;
      m_run[i] = m_new;
    }
  }
  if (tx == 0) {
#pragma unroll
    for (int i = 0; i < 4; ++i) s_lse[ty * 4 + i] = (l_run[i] > 0.f) ? m_run[i] + logf(l_run[i]) : CUDART_INF_F;
  }
  __syncthreads();
  if (tid < 64 && q0 + tid < L) {
    lse_out[((int64_t)(r0 + q0 + tid)) * n_head + h] = s_lse[tid];
    dsum_out[((int64_t)(r0 + q0 + tid)) * n_head + h] = s_D[tid];
  }
  // ---- sweep 2: dQ = sum_keys dS K * scale, dS = P o (dP - D) ----
  float dq[4][4] = {};
  for (int j0 = 0; j0 < kv_max; j0 += 64) {
    __syncthreads();
    load_tile_t(Kt, qb, ld, j0, L, d + h * HD, tid);
    load_tile_t(Vt, qb, ld, j0, L, 2 * d + h * HD, tid);
    load_tile_n(Kn, qb, ld, j0, L, d + h * HD, tid);
    __syncthreads();
    float s[4][4] = {}, dp[4][4] = {};
    mm_tt(Qt, Kt, ty, tx, s);
    mm_tt(dOt, Vt, ty, tx, dp);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float lse = s_lse[ty * 4 + i], Dv = s_D[ty * 4 + i];
      const uint64_t base = ((uint64_t)(b * n_head + h) * drop.lmax + (q0 + ty * 4 + i)) * drop.lmax + j0 + tx * 4;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float p = lim[i].ok(j0 + tx * 4 + j) ? expf(s[i][j] * 0.125f - lse) : 0.f;
        float dpm = dp[i][j];   // with dropout O = (m / keep o P) V: dP reaches P through the same mask
        if (drop.thresh != 0) dpm = drop_keep(drop, base + j) ? dpm * drop.inv_keep : 0.f;
        dSt[(tx * 4 + j) * LDT + ty * 4 + i] = p * (dpm - Dv);
      }
    }
    __syncthreads();
    // dq[i][e-col] += sum_key dS[key][q] * K[key][e] : A = dSt (key-major, q fastest), B = Kn (key-major, e fastest)
#pragma unroll 8
    for (int c = 0; c < 64; ++c) {
      const float4 a = *reinterpret_cast<const float4 *>(&dSt[c * LDT + ty * 4]);
      const float4 k4 = *reinterpret_cast<const float4 *>(&Kn[c * LDT + tx * 4]);
      const float av[4] = {a.x, a.y, a.z, a.w}, kv[4] = {k4.x, k4.y, k4.z, k4.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) dq[i][j] = fmaf(av[i], kv[j], dq[i][j]);
    }
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int qr = q0 + ty * 4 + i;
    if (qr >= L) continue;
    T *dst = dqkv + (int64_t)(r0 + qr) * ld + h * HD + tx * 4;
#pragma unroll
    for (int j = 0; j < 4; ++j) dst[j] = from_f32<T>(dq[i][j] * 0.125f);
  }
}

// pass 2: per (key block, head, sequence): dK, dV
template <typename T>
__global__ void __launch_bounds__(256)
attn_bwd_dkv_kernel(const T *__restrict__ qkv, const T *__restrict__ dout, int n_head, const Packed pk,
                    T *__restrict__ dqkv, const float *__restrict__ lse_in, const float *__restrict__ dsum_in,
                    DropCfg drop) {
  extern __shared__ __align__(16) float smem[];
  float *Kt = smem;              // [e][key]
  float *Vt = Kt + 64 * LDT;     // [e][key]
  float *Qt = Vt + 64 * LDT;     // [e][q]
  float *dOt = Qt + 64 * LDT;    // [e][q]
  float *Qn = dOt + 64 * LDT;    // [q][e]
  float *dOn = Qn + 64 * LDT;    // [q][e]
  float *Pt = dOn + 64 * LDT;    // [q][key]  probabilities
  float *dSt = Pt + 64 * LDT;    // [q][key]
  __shared__ float s_lse[64], s_D[64];
  const int b = blockIdx.z, h = blockIdx.y;
  const Packed::Seq sb = pk.seq(b);
  const int r0 = sb.r0, L = sb.L;
  const int k0 = blockIdx.x * 64;
  if (k0 >= L) return;
  const int d = n_head * HD;
  const int64_t ld = 3 * (int64_t)d;
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;   // here: ty -> 4 keys, tx -> 4 head dims
  const T *qb = qkv + (int64_t)r0 * ld;
  load_tile_t(Kt, qb, ld, k0, L, d + h * HD, tid);
  load_tile_t(Vt, qb, ld, k0, L, 2 * d + h * HD, tid);
  float dk[4][4] = {}, dv[4][4] = {};
  for (int q0 = 0; q0 < L; q0 += 64) {
    __syncthreads();
    load_tile_t(Qt, qb, ld, q0, L, h * HD, tid);
    load_tile_t(dOt, dout + (int64_t)r0 * d, (int64_t)d, q0, L, h * HD, tid);
    load_tile_n(Qn, qb, ld, q0, L, h * HD, tid);
    load_tile_n(dOn, dout + (int64_t)r0 * d, (int64_t)d, q0, L, h * HD, tid);
    if (tid < 64) {
      const bool ok = q0 + tid < L;
      s_lse[tid] = ok ? lse_in[((int64_t)(r0 + q0 + tid)) * n_head + h] : CUDART_INF_F;
      s_D[tid] = ok ? dsum_in[((int64_t)(r0 + q0 + tid)) * n_head + h] : 0.f;
    }
    __syncthreads();
    // scores of (4 queries of this thread's row group) x (4 keys): reuse the q-major tiling: rows = queries
    float s[4][4] = {}, dp[4][4] = {};
    mm_tt(Qt, Kt, ty, tx, s);    // s[i][j]: query ty*4+i, key tx*4+j
    mm_tt(dOt, Vt, ty, tx, dp);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int qr = q0 + ty * 4 + i;
      const RowMask lim = pk.row_mask(sb, qr);
      const float lse = s_lse[ty * 4 + i], Dv = s_D[ty * 4 + i];
      const uint64_t base = ((uint64_t)(b * n_head + h) * drop.lmax + qr) * drop.lmax + k0 + tx * 4;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float p = lim.ok(k0 + tx * 4 + j) ? expf(s[i][j] * 0.125f - lse) : 0.f;
        float pm = p, dpm = dp[i][j];
        if (drop.thresh != 0) {
          const float mk = drop_keep(drop, base + j) ? drop.inv_keep : 0.f;
          pm *= mk;
          dpm *= mk;
        }
        Pt[(ty * 4 + i) * LDT + tx * 4 + j] = pm;               // dV = (m / keep o P)^T dO
        dSt[(ty * 4 + i) * LDT + tx * 4 + j] = p * (dpm - Dv);
      }
    }
    __syncthreads();
    // dV[key][e] += sum_q P[q][key] dO[q][e];  dK[key][e] += sum_q dS[q][key] Q[q][e]
#pragma unroll 8
    for (int c = 0; c < 64; ++c) {
      const float4 p4 = *reinterpret_cast<const float4 *>(&Pt[c * LDT + ty * 4]);
      const float4 s4 = *reinterpret_cast<const float4 *>(&dSt[c * LDT + ty * 4]);
      const float4 g4 = *reinterpret_cast<const float4 *>(&dOn[c * LDT + tx * 4]);
      const float4 q4 = *reinterpret_cast<const float4 *>(&Qn[c * LDT + tx * 4]);
      const float pv[4] = {p4.x, p4.y, p4.z, p4.w}, sv[4] = {s4.x, s4.y, s4.z, s4.w};
      const float gv[4] = {g4.x, g4.y, g4.z, g4.w}, qv[4] = {q4.x, q4.y, q4.z, q4.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          dv[i][j] = fmaf(pv[i], gv[j], dv[i][j]);
          dk[i][j] = fmaf(sv[i], qv[j], dk[i][j]);
        }
    }
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int kr = k0 + ty * 4 + i;
    if (kr >= L) continue;
    T *dkp = dqkv + (int64_t)(r0 + kr) * ld + d + h * HD + tx * 4;
    T *dvp = dkp + d;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      dkp[j] = from_f32<T>(dk[i][j] * 0.125f);
      dvp[j] = from_f32<T>(dv[i][j]);
    }
  }
}

}  // namespace bw

template <typename TD>
__global__ void cast_kernel(const float *__restrict__ in, TD *__restrict__ out, int64_t n) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    out[i] = from_f32<TD>(in[i]);
}

int launch_cast_from_f32(const float *in, void *out, int dtype, int64_t n, cudaStream_t s) {
  if (n == 0) return VB_OK;
  const unsigned grid = (unsigned)std::min<int64_t>((n + 255) / 256, 132 * 16);
  if (dtype == VB_F32)
    cast_kernel<float><<<grid, 256, 0, s>>>(in, (float *)out, n);
  else
    cast_kernel<bf16><<<grid, 256, 0, s>>>(in, (bf16 *)out, n);
  VB_LAUNCH_CHECK();
  return VB_OK;
}

// ---- host launchers (dtype dispatch) ---------------------------------------------------------------------------
int launch_transpose_pad(const void *in, int dtype, int64_t ld_in, int64_t R, int C, void *out, int64_t ld_out,
                         cudaStream_t s) {
  VB_CHECK_ARG(ld_out >= R, "transpose: ld_out < rows");
  if (C == 0 || ld_out == 0) return VB_OK;
  dim3 grid((unsigned)((ld_out + 31) / 32), (unsigned)((C + 31) / 32)), block(32, 8);
  if (dtype == VB_F32)
    bw::transpose_pad_kernel<float><<<grid, block, 0, s>>>((const float *)in, ld_in, R, C, (float *)out, ld_out);
  else
    bw::transpose_pad_kernel<bf16><<<grid, block, 0, s>>>((const bf16 *)in, ld_in, R, C, (bf16 *)out, ld_out);
  VB_LAUNCH_CHECK();
  return VB_OK;
}

int launch_colsum(const void *in, int dtype, int64_t ld, int64_t R, int N, float *out, cudaStream_t s) {
  if (R == 0 || N == 0) return VB_OK;
  const int64_t rows_per_cta = 256;
  dim3 grid((unsigned)((N + 31) / 32), (unsigned)((R + rows_per_cta - 1) / rows_per_cta)), block(32, 8);
  if (dtype == VB_F32)
    bw::colsum_kernel<float><<<grid, block, 0, s>>>((const float *)in, ld, R, N, out, rows_per_cta);
  else
    bw::colsum_kernel<bf16><<<grid, block, 0, s>>>((const bf16 *)in, ld, R, N, out, rows_per_cta);
  VB_LAUNCH_CHECK();
  return VB_OK;
}

int launch_dropout(const void *in, void *out, int dtype, int64_t n, const DropCfg &cfg, cudaStream_t s) {
  if (n == 0) return VB_OK;
  const unsigned grid = (unsigned)std::min<int64_t>((n + 255) / 256, 132 * 16);
  if (dtype == VB_F32)
    bw::dropout_kernel<float><<<grid, 256, 0, s>>>((const float *)in, (float *)out, n, cfg);
  else
    bw::dropout_kernel<bf16><<<grid, 256, 0, s>>>((const bf16 *)in, (bf16 *)out, n, cfg);
  VB_LAUNCH_CHECK();
  return VB_OK;
}

int launch_dropout_add(float *x, const float *t, int64_t n, const DropCfg &cfg, cudaStream_t s) {
  if (n == 0) return VB_OK;
  const unsigned grid = (unsigned)std::min<int64_t>((n + 255) / 256, 132 * 16);
  bw::dropout_add_kernel<<<grid, 256, 0, s>>>(x, t, n, cfg);
  VB_LAUNCH_CHECK();
  return VB_OK;
}

int launch_relu_bwd(void *dh, const void *h, int dtype, int64_t n, float scale, cudaStream_t s) {
  if (n == 0) return VB_OK;
  const unsigned grid = (unsigned)std::min<int64_t>((n + 255) / 256, 132 * 16);
  if (dtype == VB_F32)
    bw::relu_bwd_kernel<float><<<grid, 256, 0, s>>>((float *)dh, (const float *)h, n, scale);
  else
    bw::relu_bwd_kernel<bf16><<<grid, 256, 0, s>>>((bf16 *)dh, (const bf16 *)h, n, scale);
  VB_LAUNCH_CHECK();
  return VB_OK;
}

}  // namespace vb

using namespace vb;

VB_API int vb_layernorm_backward(const float *x, int64_t x_row_stride, const int32_t *rows, int64_t n_rows, int d,
                                 const float *gamma, const float *beta, const float *ada_wb, float eps,
                                 const float *dy, int64_t dy_row_stride, float *dx, int64_t dx_row_stride,
                                 void *dx_copy, int copy_dtype, float *dgamma, float *dbeta, float *dada_wb,
                                 vb_stream_t stream) {
  VB_CHECK_ARG(x && dy && dx && gamma && beta, "vb_layernorm_backward: null argument");
  VB_CHECK_ARG(d <= 8192, "vb_layernorm_backward: d=%d too large", d);
  if (n_rows == 0) return VB_OK;
  const int rows_per_cta = 64;
  const unsigned grid = (unsigned)((n_rows + rows_per_cta - 1) / rows_per_cta);
  const size_t smem = (size_t)4 * d * sizeof(float);
  cudaStream_t s = (cudaStream_t)stream;
  if (dx_copy && copy_dtype == VB_BF16) {
    auto k = bw::ln_bwd_kernel<bf16>;
    if (smem > 48 * 1024) VB_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k<<<grid, 256, smem, s>>>(x, x_row_stride, rows, n_rows, d, gamma, beta, ada_wb, eps, dy, dy_row_stride, dx,
                              dx_row_stride, (bf16 *)dx_copy, dgamma, dbeta, dada_wb, rows_per_cta);
  } else {
    auto k = bw::ln_bwd_kernel<float>;
    if (smem > 48 * 1024) VB_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k<<<grid, 256, smem, s>>>(x, x_row_stride, rows, n_rows, d, gamma, beta, ada_wb, eps, dy, dy_row_stride, dx,
                              dx_row_stride, (float *)dx_copy, dgamma, dbeta, dada_wb, rows_per_cta);
  }
  VB_LAUNCH_CHECK();
  return VB_OK;
}

VB_API int vb_cross_entropy_backward(const float *logits, int64_t ld_logits, const int64_t *targets, int64_t n_rows,
                                     int n_vocab, int64_t ignore_index, const float *grad_rows, float grad_scale,
                                     void *dlogits, int out_dtype, int64_t ld_out, int n_out, vb_stream_t stream) {
  VB_CHECK_ARG(n_out >= n_vocab && ld_out >= n_out, "vb_cross_entropy_backward: bad output geometry");
  if (n_rows == 0) return VB_OK;
  const int wpb = 4;
  const unsigned grid = (unsigned)((n_rows + wpb - 1) / wpb);
  if (out_dtype == VB_BF16)
    bw::ce_bwd_kernel<bf16><<<grid, wpb * 32, 0, (cudaStream_t)stream>>>(logits, ld_logits, targets, n_rows, n_vocab,
                                                                         ignore_index, grad_rows, grad_scale,
                                                                         (bf16 *)dlogits, ld_out, n_out);
  else
    bw::ce_bwd_kernel<float><<<grid, wpb * 32, 0, (cudaStream_t)stream>>>(logits, ld_logits, targets, n_rows, n_vocab,
                                                                          ignore_index, grad_rows, grad_scale,
                                                                          (float *)dlogits, ld_out, n_out);
  VB_LAUNCH_CHECK();
  return VB_OK;
}

VB_API int vb_embed_backward(const int64_t *tokens, int64_t tok_row_stride, int64_t tok_tab_stride,
                             float *const *table_grads, const int32_t *table_rows, int n_tables, int64_t n_rows, int d,
                             const float *dy, int64_t dy_row_stride, const int32_t *dy_rows, vb_stream_t stream) {
  VB_CHECK_ARG(n_tables >= 1 && n_tables <= bw::kMaxTables && table_rows, "vb_embed_backward: bad tables");
  if (n_rows == 0) return VB_OK;
  bw::GradTables gt;
  for (int j = 0; j < bw::kMaxTables; ++j) {
    gt.t[j] = j < n_tables ? table_grads[j] : nullptr;
    gt.rows[j] = j < n_tables ? table_rows[j] : 0;
  }
  const int wpb = 4;
  bw::embed_bwd_kernel<<<(unsigned)((n_rows + wpb - 1) / wpb), wpb * 32, 0, (cudaStream_t)stream>>>(
      tokens, tok_row_stride, tok_tab_stride, gt, n_tables, n_rows, d, dy, dy_row_stride, dy_rows);
  VB_LAUNCH_CHECK();
  return VB_OK;
}

VB_API int vb_rowdot_accumulate(const float *a, int64_t a_row_stride, const float *b, int64_t pos0,
                                const int32_t *positions, int64_t n_rows, int d, float *out, vb_stream_t stream) {
  if (n_rows == 0) return VB_OK;
  const unsigned grid = (unsigned)std::min<int64_t>((n_rows + 7) / 8, 1024);
  bw::rowdot_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(a, a_row_stride, b, pos0, positions, n_rows, d, out);
  VB_LAUNCH_CHECK();
  return VB_OK;
}

VB_API int vb_adaln_project_backward(const float *W, const float *emb, const float *dwb, int d, float *dW, float *db,
                                     float *demb, vb_stream_t stream) {
  bw::adaln_proj_bwd_kernel<<<2 * d, 128, 0, (cudaStream_t)stream>>>(W, emb, dwb, d, dW, db, demb);
  VB_LAUNCH_CHECK();
  return VB_OK;
}

VB_API size_t vb_linear_backward_workspace(int dtype, int64_t M, int N, int K) {
  const size_t ts = dtype == VB_BF16 ? 2 : 4;
  const size_t Mp = align_up((size_t)M, 64);
  return (align_up((size_t)N * Mp * ts, 256) + align_up((size_t)K * Mp * ts, 256)) + 256;
}

// Gradients of Y[M,N] = X[M,K] W[N,K]^T + b:  dX = dY W (through Wt = W^T [K,N]), dW += dY^T X, db += colsum(dY).
// dX may be NULL (no input gradient), dW / db may be NULL.  dx_epilogue: VB_EPI_NONE (dX = ...) or VB_EPI_RESIDUAL
// (fp32 dX += ...).  workspace: vb_linear_backward_workspace(dtype, M, N, K) bytes.
VB_API int vb_linear_backward(const void *X, int dtype, int64_t ldx, const void *Wt, const void *dY, int64_t lddy,
                              void *dX, int dx_dtype, int64_t lddx, int dx_epilogue, float *dW, float *db, int64_t M,
                              int N, int K, void *workspace, size_t workspace_bytes, vb_stream_t stream) {
  VB_CHECK_ARG(dtype == VB_F32 || dtype == VB_BF16, "vb_linear_backward: bad dtype");
  if (M == 0) return VB_OK;
  cudaStream_t s = (cudaStream_t)stream;
  if (dX) {
    VB_CHECK_ARG(Wt != nullptr, "vb_linear_backward: dX needs the transposed weight");
    VB_TRY(vb_linear(dY, dtype, lddy, Wt, dtype, nullptr, dX, dx_dtype, lddx, M, K, N, dx_epilogue, nullptr, 0, stream));
  }
  if (db) VB_TRY(launch_colsum(dY, dtype, lddy, M, N, db, s));
  if (dW) {
    VB_CHECK_ARG(workspace && workspace_bytes >= vb_linear_backward_workspace(dtype, M, N, K),
                 "vb_linear_backward: workspace too small");
    const size_t ts = dtype == VB_BF16 ? 2 : 4;
    const int64_t Mp = (int64_t)align_up((size_t)M, 64);
    char *ws = (char *)workspace;
    void *dYt = ws;
    void *Xt = ws + align_up((size_t)N * Mp * ts, 256);
    VB_TRY(launch_transpose_pad(dY, dtype, lddy, M, N, dYt, Mp, s));
    VB_TRY(launch_transpose_pad(X, dtype, ldx, M, K, Xt, Mp, s));
    // dW[N, K] += dYt[N, Mp] Xt[K, Mp]^T
    VB_TRY(vb_linear(dYt, dtype, Mp, Xt, dtype, nullptr, dW, VB_F32, K, N, K, (int)Mp, VB_EPI_RESIDUAL, nullptr, 0, stream));
  }
  return VB_OK;
}

VB_API int vb_dropout(const void *in, void *out, int dtype, int64_t n, float p, uint64_t seed, uint32_t stream_id,
                      vb_stream_t stream) {
  VB_CHECK_ARG(in && out && (dtype == VB_F32 || dtype == VB_BF16), "vb_dropout: bad argument");
  VB_CHECK_ARG(p >= 0.f && p < 1.f, "vb_dropout: p=%g not in [0, 1)", (double)p);
  if (p == 0.f) {
    if (in != out) VB_CUDA(cudaMemcpyAsync(out, in, (size_t)n * (dtype == VB_F32 ? 4 : 2), cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
    return VB_OK;
  }
  return launch_dropout(in, out, dtype, n, make_drop(p, seed, stream_id), (cudaStream_t)stream);
}

VB_API size_t vb_attention_backward_workspace(int64_t M, int n_head) { return (size_t)M * n_head * 2 * sizeof(float) + 256; }

VB_API int vb_attention_backward(const void *qkv, const void *out, const void *dout, int dtype, int64_t M, int B,
                                 int n_head, int head_dim, const int32_t *cu_seqlens, const int32_t *text_lens,
                                 const int32_t *seg1_lens, int seg1_start, int max_seqlen, int mask_mode, void *dqkv,
                                 void *workspace, size_t workspace_bytes, vb_stream_t stream) {
  const vb::Packed pk{cu_seqlens, text_lens, seg1_lens, B, max_seqlen, seg1_start, mask_mode};
  return vb::attention_backward(qkv, out, dout, dtype, M, n_head, head_dim, pk, dqkv, workspace, workspace_bytes, nullptr,
                                (cudaStream_t)stream);
}

int vb::attention_backward(const void *qkv, const void *out, const void *dout, int dtype, int64_t M, int n_head,
                           int head_dim, const Packed &pk, void *dqkv, void *workspace, size_t workspace_bytes,
                           const DropCfg *drop, cudaStream_t s) {
  DropCfg dc{};
  if (drop) dc = *drop;
  dc.lmax = pk.max_seqlen;
  VB_CHECK_ARG(head_dim == bw::HD, "vb_attention_backward: head_dim=%d, only 64 is built", head_dim);
  VB_TRY(check_packed(pk, "vb_attention_backward"));
  VB_CHECK_ARG(workspace && workspace_bytes >= vb_attention_backward_workspace(M, n_head),
               "vb_attention_backward: workspace too small");
  if (M == 0 || pk.B == 0) return VB_OK;
  VB_CHECK_ARG(dtype == VB_F32 || dtype == VB_BF16, "vb_attention_backward: bad dtype %d", dtype);
  float *lse = (float *)workspace;
  float *dsum = lse + (size_t)M * n_head;
  auto launch = [&](auto elem) -> int {
    using T = decltype(elem);
    const dim3 grid((pk.max_seqlen + 63) / 64, n_head, pk.B);
    const size_t smem_q = (size_t)6 * 64 * bw::LDT * sizeof(float), smem_k = (size_t)8 * 64 * bw::LDT * sizeof(float);
    auto kq = bw::attn_bwd_dq_kernel<T>;
    auto kk = bw::attn_bwd_dkv_kernel<T>;
    VB_CUDA(cudaFuncSetAttribute(kq, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_q));
    VB_CUDA(cudaFuncSetAttribute(kk, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_k));
    kq<<<grid, 256, smem_q, s>>>((const T *)qkv, (const T *)out, (const T *)dout, n_head, pk, (T *)dqkv, lse, dsum, dc);
    VB_LAUNCH_CHECK();
    kk<<<grid, 256, smem_k, s>>>((const T *)qkv, (const T *)dout, n_head, pk, (T *)dqkv, lse, dsum, dc);
    VB_LAUNCH_CHECK();
    return VB_OK;
  };
  return dtype == VB_F32 ? launch(float{}) : launch(bf16{});
}
