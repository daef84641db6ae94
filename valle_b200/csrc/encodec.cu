// EnCodec 24 kHz (SEANet encoder/decoder + 2-layer LSTM + 8-stage residual VQ) building blocks, fp32.
//
// The reference reaches this arithmetic through the un-vendored PyPI package `encodec`
// (valle/data/tokenizer.py:219-242: EncodecModel.encodec_model_24khz(), set_target_bandwidth(6.0),
// codec.encode / codec.decode; weight-norm stripped at load, :181-208).  The published architecture is
// restated here (causal SConv1d with reflect padding, ELU pre-activations, residual blocks with 1x1
// shortcut, strided down/up-sampling convs, LSTM with skip, Euclidean-codebook RVQ) and checked
// against transformers' EncodecModel, the only implementation available offline (parity
// "unpinned" w.r.t. the PyPI package, see DESIGN.md).
//
// Layout: activations [B, C, T] fp32, time contiguous (PyTorch conv layout).
#include <math_constants.h>

#include "common.cuh"
#include "kernels.cuh"

namespace vb {
namespace ec {

__device__ __forceinline__ float elu1(float x) { return x > 0.f ? x : expm1f(x); }

// ---- causal / asymmetric-padded Conv1d as a register-tiled implicit GEMM (+pre-ELU, +bias, +residual) -------
//   out[b, co, t] = bias[co] + sum_{ci,k} W[co, ci, k] * act(x)[b, ci, t*stride - pad_left + k*dil]
// Reflect padding maps g < 0 to -g and g >= Te to 2 (Te - 1) - g over x zero-extended to Te samples (vb_conv1d).
// One CTA = CO_T output channels x T_T time steps of one utterance; a thread owns 8 channels x 8 time steps
// (64 accumulators; per (ci, k): 2 broadcast LDS.128 of weights + 8 conflict-free LDS of inputs for 64 FFMA).
// The weights arrive pre-packed as wp[Cin][K][Cout] (channel-fastest) so a chunk of CI_T input channels is one
// contiguous slab.  `phase` > 1 serves the transposed up-sampling convolutions: output channel c' = co * phase + r
// is stored to out[b, co, t * phase + r] (a ConvTranspose1d with K = 2 * stride, causal trim, is a stride-1 K=2
// convolution onto Cout * stride phase channels, see vb_conv1d in the header).
constexpr int CI_T = 8, TH_CO = 8, TH_T = 8;

template <int CO_T>
__global__ void __launch_bounds__(256, 2)
conv1d_tiled_kernel(const float *__restrict__ x, int Cin, int Tin, const float *__restrict__ wp,
                    const float *__restrict__ bias, int Cout, int K, int stride, int dil, int pad_left, int reflect,
                    int Te, int pre_elu, const float *__restrict__ residual, float *__restrict__ out, int Tout,
                    int in_w, int phase) {
  constexpr int TYN = CO_T / TH_CO;   // thread rows (channel groups)
  constexpr int TXN = 256 / TYN;      // thread columns; time steps of a thread: tx + j * TXN
  constexpr int T_T = TXN * TH_T;
  extern __shared__ __align__(16) float smem[];
  float *ws = smem;                      // [CI_T][K][CO_T]
  float *xs = smem + CI_T * K * CO_T;    // [CI_T][in_w]
  const int b = blockIdx.z, co0 = blockIdx.y * CO_T, t0 = blockIdx.x * T_T;
  const int tid = threadIdx.x, tx = tid % TXN, ty = tid / TXN;
  const float *xb = x + (int64_t)b * Cin * Tin;
  float acc[TH_CO][TH_T];
#pragma unroll
  for (int i = 0; i < TH_CO; ++i)
#pragma unroll
    for (int j = 0; j < TH_T; ++j) acc[i][j] = 0.f;
  const int g0 = t0 * stride - pad_left;  // global time index of xs[.][0]
  for (int ci0 = 0; ci0 < Cin; ci0 += CI_T) {
    const int cin = min(CI_T, Cin - ci0);
    // weights of this chunk: rows (ci, k) of wp are Cout floats wide
    for (int idx = tid; idx < cin * K * CO_T; idx += 256) {
      const int row = idx / CO_T, co = idx & (CO_T - 1);   // CO_T is a power of two
      ws[idx] = (co0 + co < Cout) ? wp[((int64_t)ci0 * K + row) * Cout + co0 + co] : 0.f;
    }
    for (int ci = 0; ci < cin; ++ci) {   // (no integer division in the staging loop: it runs once per input element)
      const float *xrow = xb + (int64_t)(ci0 + ci) * Tin;
      float *xd = xs + ci * in_w;
      for (int i = tid; i < in_w; i += 256) {
        int g = g0 + i;
        float v = 0.f;
        if (reflect) {  // F.pad(mode="reflect") of x zero-extended to Te = max(Tin, max pad + 1) samples
          if (g < 0) g = -g;
          if (g >= Te) g = 2 * (Te - 1) - g;
        }
        if (g >= 0 && g < Tin) {
          v = xrow[g];
          if (pre_elu) v = elu1(v);
        }
        xd[i] = v;
      }
    }
    __syncthreads();
    for (int ci = 0; ci < cin; ++ci) {
      const float *xr = xs + ci * in_w + tx * stride;
      const float *wr = ws + (ci * K) * CO_T + ty * TH_CO;
      for (int k = 0; k < K; ++k) {
        const float4 w0 = *reinterpret_cast<const float4 *>(wr + k * CO_T);
        const float4 w1 = *reinterpret_cast<const float4 *>(wr + k * CO_T + 4);
        const float wv[TH_CO] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
        float xv[TH_T];
#pragma unroll
        for (int j = 0; j < TH_T; ++j) xv[j] = xr[j * TXN * stride + k * dil];
#pragma unroll
        for (int i = 0; i < TH_CO; ++i)
#pragma unroll
          for (int j = 0; j < TH_T; ++j) acc[i][j] = fmaf(wv[i], xv[j], acc[i][j]);
      }
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < TH_CO; ++i) {
    const int co = co0 + ty * TH_CO + i;
    if (co >= Cout) continue;
    const float bv = bias ? bias[co / phase] : 0.f;
#pragma unroll
    for (int j = 0; j < TH_T; ++j) {
      const int t = t0 + tx + j * TXN;
      if (t >= Tout) continue;
      int64_t o;
      if (phase == 1) o = ((int64_t)b * Cout + co) * Tout + t;
      else o = ((int64_t)b * (Cout / phase) + co / phase) * ((int64_t)Tout * phase) + (int64_t)t * phase + co % phase;
      float v = acc[i][j] + bv;
      if (residual) v += residual[o];
      out[o] = v;
    }
  }
}

// ---- LSTM time step: 128 hidden units x 4 batch rows per CTA --------------------------------------
// gates = xproj[t] (W_ih x + b_ih + b_hh, precomputed) + W_hh h_{t-1}; PyTorch gate order i,f,g,o
__global__ void __launch_bounds__(128)
lstm_step_kernel(const float *__restrict__ xproj_t, const float *__restrict__ whh_t /*[H][4H]*/,
                 const float *__restrict__ h_prev /*[B][H] or null*/, float *__restrict__ c /*[B][H]*/,
                 float *__restrict__ h_out /*[B][H]*/, int B, int H) {
  extern __shared__ float hs[];  // [4][H]
  const int j = blockIdx.x * 128 + threadIdx.x;
  const int b0 = blockIdx.y * 4;
  for (int i = threadIdx.x; i < 4 * H; i += 128) {
    const int bb = i / H, k = i - bb * H;
    hs[i] = (h_prev && b0 + bb < B) ? h_prev[(int64_t)(b0 + bb) * H + k] : 0.f;
  }
  __syncthreads();
  if (j >= H) return;
  float acc[4][4];
#pragma unroll
  for (int g = 0; g < 4; ++g)
#pragma unroll
    for (int bb = 0; bb < 4; ++bb) acc[g][bb] = 0.f;
  if (h_prev) {
    for (int k = 0; k < H; ++k) {
      const float *wr = whh_t + (int64_t)k * 4 * H + j;
      const float w0 = wr[0], w1 = wr[H], w2 = wr[2 * H], w3 = wr[3 * H];
#pragma unroll
      for (int bb = 0; bb < 4; ++bb) {
        const float hv = hs[bb * H + k];
        acc[0][bb] = fmaf(w0, hv, acc[0][bb]);
        acc[1][bb] = fmaf(w1, hv, acc[1][bb]);
        acc[2][bb] = fmaf(w2, hv, acc[2][bb]);
        acc[3][bb] = fmaf(w3, hv, acc[3][bb]);
      }
    }
  }
#pragma unroll
  for (int bb = 0; bb < 4; ++bb) {
    const int b = b0 + bb;
    if (b >= B) continue;
    const float *xp = xproj_t + (int64_t)b * 4 * H;
    const float gi = acc[0][bb] + xp[j], gf = acc[1][bb] + xp[H + j];
    const float gg = acc[2][bb] + xp[2 * H + j], go = acc[3][bb] + xp[3 * H + j];
    const float si = 1.f / (1.f + expf(-gi)), sf = 1.f / (1.f + expf(-gf)), so = 1.f / (1.f + expf(-go));
    const float cprev = h_prev ? c[(int64_t)b * H + j] : 0.f;
    const float cn = sf * cprev + si * tanhf(gg);
    c[(int64_t)b * H + j] = cn;
    h_out[(int64_t)b * H + j] = so * tanhf(cn);
  }
}

// ---- one LSTM layer, all T steps in ONE persistent cooperative kernel --------------------------------------
// CTA j owns LSTM_U hidden units = 4 * LSTM_U gate columns; its slice of W_hh^T ([H][4*LSTM_U], 32 KB at H=512)
// stays in shared memory for the whole sequence.  Per step: load h_{t-1} [B][H] (L2), the [B x 16] gate slice as
// register-tiled dot products split over k-groups, cell update for its units, write h_t, one grid barrier.
// The launch per time step of lstm_step_kernel (2 x 750 launches per 10 s utterance batch) becomes 2 launches.
constexpr int LSTM_U = 4, LSTM_C = 4 * LSTM_U, LSTM_MAXB = 64;


__global__ void __launch_bounds__(256, 1)
lstm_layer_persistent_kernel(const float *__restrict__ xproj /*[T][B][4H]*/, const float *__restrict__ whh_t /*[H][4H]*/,
                             int T, int B, int H, float *__restrict__ h_seq /*[T][B][H]*/, unsigned *__restrict__ sync) {
  extern __shared__ __align__(16) float sm[];
  const int HP = H + 1;                      // padded row of the h tile (bank spread over batch rows)
  float *wsl = sm;                           // [H][LSTM_C]  column c = gate * LSTM_U + u
  float *hs = wsl + H * LSTM_C;              // [Bp][HP]
  const int Bp = (B + 3) & ~3;
  float *red = hs + Bp * HP;                 // [kgroups][Bp * LSTM_C]
  float *cst = red + 256 * 16;               // [Bp][LSTM_U] cell state
  const int tid = threadIdx.x;
  const int u0 = blockIdx.x * LSTM_U;
  for (int i = tid; i < H * LSTM_C; i += 256) {
    const int k = i / LSTM_C, c = i - k * LSTM_C;
    const int g = c / LSTM_U, u = c - g * LSTM_U;
    wsl[i] = whh_t[(int64_t)k * 4 * H + g * H + u0 + u];
  }
  for (int i = tid; i < Bp * LSTM_U; i += 256) cst[i] = 0.f;
  for (int i = tid; i < Bp * HP; i += 256) hs[i] = 0.f;
  const int tiles = (Bp / 4) * (LSTM_C / 4);   // 4 batch rows x 4 gate columns per thread
  const int kgroups = 256 / tiles;             // B <= 64 -> tiles <= 64, kgroups >= 4
  const int kper = (H + kgroups - 1) / kgroups;
  const int tile = tid % tiles, kg = tid / tiles;
  const int bt = tile / (LSTM_C / 4), ct = tile - bt * (LSTM_C / 4);
  unsigned bar_target = 0;
  __syncthreads();
  for (int t = 0; t < T; ++t) {
    float acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
    if (t > 0) {
      const float *hp = h_seq + (int64_t)(t - 1) * B * H;
      for (int i = tid; i < B * H; i += 256) {
        const int b = i / H, k = i - b * H;
        hs[b * HP + k] = __ldcg(hp + i);
      }
      __syncthreads();
      if (kg < kgroups) {
        const int k0 = kg * kper, k1 = min(H, k0 + kper);
        const float *h0 = hs + (bt * 4) * HP;
        for (int k = k0; k < k1; ++k) {
          const float4 w = *reinterpret_cast<const float4 *>(wsl + k * LSTM_C + ct * 4);
          const float hv[4] = {h0[k], h0[HP + k], h0[2 * HP + k], h0[3 * HP + k]};
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            acc[i][0] = fmaf(hv[i], w.x, acc[i][0]);
            acc[i][1] = fmaf(hv[i], w.y, acc[i][1]);
            acc[i][2] = fmaf(hv[i], w.z, acc[i][2]);
            acc[i][3] = fmaf(hv[i], w.w, acc[i][3]);
          }
        }
      }
    }
    if (kg < kgroups) {
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) red[kg * (Bp * LSTM_C) + (bt * 4 + i) * LSTM_C + ct * 4 + j] = acc[i][j];
    }
    __syncthreads();
    // cell update: thread = (batch row, unit)
    for (int i = tid; i < B * LSTM_U; i += 256) {
      const int b = i / LSTM_U, u = i - b * LSTM_U;
      float g4[4];
#pragma unroll
      for (int g = 0; g < 4; ++g) {
        float v = 0.f;
        for (int q = 0; q < kgroups; ++q) v += red[q * (Bp * LSTM_C) + b * LSTM_C + g * LSTM_U + u];
        g4[g] = v + xproj[((int64_t)t * B + b) * 4 * H + g * H + u0 + u];
      }
      const float si = 1.f / (1.f + expf(-g4[0])), sf = 1.f / (1.f + expf(-g4[1])), so = 1.f / (1.f + expf(-g4[3]));
      const float cn = sf * cst[i] + si * tanhf(g4[2]);
      cst[i] = cn;
      h_seq[((int64_t)t * B + b) * H + u0 + u] = so * tanhf(cn);
    }
    if (t + 1 < T) grid_barrier_sync(sync, bar_target);
  }
}

// ---- residual vector quantisation: 8 frames per CTA, all stages in one launch ---------------------
// per stage: idx = argmax_j -(|r|^2 - 2 r.e_j + |e_j|^2) (first maximum), r -= e_idx
constexpr int RVQ_ROWS = 8;
__global__ void __launch_bounds__(256)
rvq_encode_kernel(const float *__restrict__ x, int64_t n_rows, int dim, int n_q, int n_codes,
                  const float *__restrict__ cb /*[nq][n_codes][dim]*/, const float *__restrict__ cb_t /*[nq][dim][n_codes]*/,
                  const float *__restrict__ cb_sq /*[nq][n_codes]*/, int64_t *__restrict__ codes, int64_t code_row_stride,
                  int64_t code_q_stride, int64_t rows_per_seq, int64_t code_seq_stride) {
  extern __shared__ float sm[];
  float *rs = sm;                     // [RVQ_ROWS][dim] residuals
  float *xx = rs + RVQ_ROWS * dim;    // [RVQ_ROWS]
  float *bv = xx + RVQ_ROWS;          // [8 warps][RVQ_ROWS] best value
  int *bi = reinterpret_cast<int *>(bv + 8 * RVQ_ROWS);  // [8 warps][RVQ_ROWS]
  int *sel = bi + 8 * RVQ_ROWS;       // [RVQ_ROWS]
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int64_t r0 = (int64_t)blockIdx.x * RVQ_ROWS;
  for (int i = tid; i < RVQ_ROWS * dim; i += 256) {
    const int r = i / dim, k = i - r * dim;
    rs[i] = (r0 + r < n_rows) ? x[(r0 + r) * dim + k] : 0.f;
  }
  __syncthreads();
  for (int q = 0; q < n_q; ++q) {
    if (tid < RVQ_ROWS) {
      float s = 0.f;
      for (int k = 0; k < dim; ++k) s += rs[tid * dim + k] * rs[tid * dim + k];
      xx[tid] = s;
    }
    __syncthreads();
    float best[RVQ_ROWS];
    int besti[RVQ_ROWS];
#pragma unroll
    for (int r = 0; r < RVQ_ROWS; ++r) {
      best[r] = -CUDART_INF_F;
      besti[r] = 0x7fffffff;
    }
    const float *et = cb_t + (int64_t)q * dim * n_codes;
    for (int j = tid; j < n_codes; j += 256) {
      float dot[RVQ_ROWS];
#pragma unroll
      for (int r = 0; r < RVQ_ROWS; ++r) dot[r] = 0.f;
      for (int k = 0; k < dim; ++k) {
        const float e = et[(int64_t)k * n_codes + j];
#pragma unroll
        for (int r = 0; r < RVQ_ROWS; ++r) dot[r] = fmaf(rs[r * dim + k], e, dot[r]);
      }
      const float ee = cb_sq[(int64_t)q * n_codes + j];
#pragma unroll
      for (int r = 0; r < RVQ_ROWS; ++r) {
        const float dist = -(xx[r] - 2.f * dot[r] + ee);
        if (dist > best[r] || (dist == best[r] && j < besti[r])) {
          best[r] = dist;
          besti[r] = j;
        }
      }
    }
#pragma unroll
    for (int r = 0; r < RVQ_ROWS; ++r) {
      float v = best[r];
      int ix = besti[r];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        const float v2 = __shfl_xor_sync(0xffffffffu, v, o);
        const int i2 = __shfl_xor_sync(0xffffffffu, ix, o);
        if (v2 > v || (v2 == v && i2 < ix)) {
          v = v2;
          ix = i2;
        }
      }
      if (lane == 0) {
        bv[warp * RVQ_ROWS + r] = v;
        bi[warp * RVQ_ROWS + r] = ix;
      }
    }
    __syncthreads();
    if (tid < RVQ_ROWS) {
      float v = bv[tid];
      int ix = bi[tid];
      for (int w = 1; w < 8; ++w) {
        const float v2 = bv[w * RVQ_ROWS + tid];
        const int i2 = bi[w * RVQ_ROWS + tid];
        if (v2 > v || (v2 == v && i2 < ix)) {
          v = v2;
          ix = i2;
        }
      }
      sel[tid] = ix;
      if (r0 + tid < n_rows) {
        const int64_t r = r0 + tid, sq = r / rows_per_seq;
        codes[sq * code_seq_stride + (r - sq * rows_per_seq) * code_row_stride + q * code_q_stride] = ix;
      }
    }
    __syncthreads();
    for (int i = tid; i < RVQ_ROWS * dim; i += 256) {
      const int r = i / dim, k = i - r * dim;
      rs[i] -= cb[((int64_t)q * n_codes + sel[r]) * dim + k];
    }
    __syncthreads();
  }
}

// ---- generic 3-D permute: out[i_p0][i_p1][i_p2] = in[i0][i1][i2] ---------------------------------
__global__ void permute3_kernel(const float *__restrict__ in, int d0, int d1, int d2, int p0, int p1, int p2,
                                float *__restrict__ out) {
  const int64_t n = (int64_t)d0 * d1 * d2;
  const int dims[3] = {d0, d1, d2};
  const int od1 = dims[p1], od2 = dims[p2];
  for (int64_t o = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; o < n; o += (int64_t)gridDim.x * blockDim.x) {
    int idx[3];
    const int64_t a = o / ((int64_t)od1 * od2);
    const int64_t rem = o - a * od1 * od2;
    idx[p0] = (int)a;
    idx[p1] = (int)(rem / od2);
    idx[p2] = (int)(rem - (int64_t)idx[p1] * od2);
    out[o] = in[((int64_t)idx[0] * d1 + idx[1]) * d2 + idx[2]];
  }
}

}  // namespace ec
}  // namespace vb

using namespace vb;

template <int CO_T>
static int launch_conv1d(const float *x, int B, int Cin, int Tin, const float *wp, const float *bias, int Cout, int K,
                         int stride, int dil, int pad_left, int reflect, int Te, int pre_elu, const float *residual,
                         float *out, int Tout, int phase, cudaStream_t s) {
  constexpr int TXN = 256 / (CO_T / ec::TH_CO), T_T = TXN * ec::TH_T;
  const int in_w = (T_T - 1) * stride + (K - 1) * dil + 1;
  const size_t smem = (size_t)(ec::CI_T * K * CO_T + ec::CI_T * in_w) * sizeof(float);
  VB_CHECK_ARG(smem <= 200 * 1024, "vb_conv1d: tile needs %zu bytes of shared memory", smem);
  auto kern = ec::conv1d_tiled_kernel<CO_T>;
  static PerDeviceOnce once;
  if (once.first()) VB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
  dim3 grid((Tout + T_T - 1) / T_T, (Cout + CO_T - 1) / CO_T, B);
  kern<<<grid, 256, smem, s>>>(x, Cin, Tin, wp, bias, Cout, K, stride, dil, pad_left, reflect, Te, pre_elu, residual,
                               out, Tout, in_w, phase);
  VB_LAUNCH_CHECK();
  return VB_OK;
}

VB_API int vb_conv1d(const float *x, int B, int Cin, int Tin, const float *wp, const float *bias, int Cout, int K,
                     int stride, int dilation, int pad_left, int pad_right, int reflect, int pre_elu,
                     const float *residual, float *out, int Tout, int phase, vb_stream_t stream) {
  VB_CHECK_ARG(K >= 1 && K <= 16 && stride >= 1 && stride <= 8, "vb_conv1d: K=%d stride=%d unsupported", K, stride);
  VB_CHECK_ARG(Tout == (Tin + pad_left + pad_right - (K - 1) * dilation - 1) / stride + 1,
               "vb_conv1d: Tout=%d inconsistent with Tin=%d pads=(%d,%d) K=%d stride=%d dil=%d", Tout, Tin, pad_left,
               pad_right, K, stride, dilation);
  VB_CHECK_ARG(phase >= 1 && Cout % phase == 0 && (phase == 1 || (stride == 1 && residual == nullptr)),
               "vb_conv1d: bad phase %d", phase);
  if (B == 0 || Tout <= 0) return VB_OK;
  cudaStream_t s = (cudaStream_t)stream;
  // a reflect pad as long as the input reflects over the input zero-extended to max pad + 1 samples (EnCodec's pad1d)
  const int Te = max(Tin, max(pad_left, pad_right) + 1);
  if (Cout > 32)
    return launch_conv1d<64>(x, B, Cin, Tin, wp, bias, Cout, K, stride, dilation, pad_left, reflect, Te, pre_elu,
                             residual, out, Tout, phase, s);
  if (Cout > 16)
    return launch_conv1d<32>(x, B, Cin, Tin, wp, bias, Cout, K, stride, dilation, pad_left, reflect, Te, pre_elu,
                             residual, out, Tout, phase, s);
  return launch_conv1d<16>(x, B, Cin, Tin, wp, bias, Cout, K, stride, dilation, pad_left, reflect, Te, pre_elu,
                           residual, out, Tout, phase, s);
}

VB_API int vb_lstm_layer(const float *xproj, const float *whh_t, int T, int B, int H, float *h_seq, float *c_state,
                         vb_stream_t stream) {
  VB_CHECK_ARG(H % 128 == 0 && H <= 2048, "vb_lstm_layer: H=%d must be a multiple of 128", H);
  if (T == 0 || B == 0) return VB_OK;
  cudaStream_t s = (cudaStream_t)stream;
  const int grid_p = H / ec::LSTM_U;
  const int Bp = (B + 3) & ~3;
  const size_t smem_p = ((size_t)H * ec::LSTM_C + (size_t)Bp * (H + 1) + 256 * 16 + (size_t)Bp * ec::LSTM_U) * sizeof(float);
  if (B <= ec::LSTM_MAXB && grid_p <= sm_count() && smem_p <= 200 * 1024 && tune("VB_LSTM_STEPWISE", 0) == 0) {
    // all T steps in one cooperative launch; the grid-barrier word lives behind the cell-state scratch
    unsigned *sync = reinterpret_cast<unsigned *>(c_state + (size_t)B * H);
    VB_CUDA(cudaMemsetAsync(sync, 0, 64 * sizeof(unsigned), s));
    auto kern = ec::lstm_layer_persistent_kernel;
    static PerDeviceOnce once;
    if (once.first()) VB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    void *args[] = {(void *)&xproj, (void *)&whh_t, (void *)&T, (void *)&B, (void *)&H, (void *)&h_seq, (void *)&sync};
    VB_CUDA(cudaLaunchCooperativeKernel((const void *)kern, dim3(grid_p), dim3(256), args, smem_p, s));
    count_launch();
    return VB_OK;
  }
  const size_t smem = (size_t)4 * H * sizeof(float);
  dim3 grid(H / 128, (B + 3) / 4);
  for (int t = 0; t < T; ++t) {
    const float *hp = t == 0 ? nullptr : h_seq + (int64_t)(t - 1) * B * H;
    ec::lstm_step_kernel<<<grid, 128, smem, s>>>(xproj + (int64_t)t * B * 4 * H, whh_t, hp, c_state,
                                                 h_seq + (int64_t)t * B * H, B, H);
    VB_LAUNCH_CHECK();
  }
  return VB_OK;
}

VB_API int vb_rvq_encode(const float *x, int64_t n_rows, int dim, int n_q, int n_codes, const float *codebooks,
                         const float *codebooks_t, const float *codebook_sq, int64_t *codes, int64_t code_row_stride,
                         int64_t code_q_stride, int64_t rows_per_seq, int64_t code_seq_stride, vb_stream_t stream) {
  VB_CHECK_ARG(dim <= 512 && n_q >= 1, "vb_rvq_encode: bad dim/n_q");
  if (rows_per_seq <= 0) {
    rows_per_seq = n_rows > 0 ? n_rows : 1;
    code_seq_stride = 0;
  }
  if (n_rows == 0) return VB_OK;
  const size_t smem = (size_t)(ec::RVQ_ROWS * dim + ec::RVQ_ROWS + 8 * ec::RVQ_ROWS) * sizeof(float) +
                      (size_t)(8 * ec::RVQ_ROWS + ec::RVQ_ROWS) * sizeof(int);
  const unsigned grid = (unsigned)((n_rows + ec::RVQ_ROWS - 1) / ec::RVQ_ROWS);
  ec::rvq_encode_kernel<<<grid, 256, smem, (cudaStream_t)stream>>>(x, n_rows, dim, n_q, n_codes, codebooks, codebooks_t,
                                                                  codebook_sq, codes, code_row_stride, code_q_stride, rows_per_seq,
                                                                  code_seq_stride);
  VB_LAUNCH_CHECK();
  return VB_OK;
}

VB_API int vb_permute3(const float *in, int d0, int d1, int d2, int p0, int p1, int p2, float *out, vb_stream_t stream) {
  VB_CHECK_ARG(((1 << p0) | (1 << p1) | (1 << p2)) == 7, "vb_permute3: not a permutation");
  const int64_t n = (int64_t)d0 * d1 * d2;
  if (n == 0) return VB_OK;
  const unsigned grid = (unsigned)((n + 255) / 256 > 65535 * 8 ? 65535 * 8 : (n + 255) / 256);
  ec::permute3_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(in, d0, d1, d2, p0, p1, p2, out);
  VB_LAUNCH_CHECK();
  return VB_OK;
}
