// Memory-bound row kernels: TokenEmbedding gather(+8-codebook sum), sine-PE add, LayerNorm /
// AdaptiveLayerNorm, row gather.  One warp per row, 16-byte accesses, grid sized by rows.
//
// Reference arithmetic: valle/modules/embedding.py:21-47,93-97; valle/modules/transformer.py:57-108;
// valle/models/valle.py:1064,1110-1113,1134.
#include "common.cuh"

namespace vb {

static constexpr int kMaxTables = 8;
struct TablePtrs {
  const float *t[kMaxTables];
  int rows[kMaxTables];  // vocabulary size of each table, 0 = unknown (no check)
};

// out[r,:] (=|+=) sum_j tables[j][tok[r, j], :]   -- sum in order j = 0..n-1
__global__ void embed_sum_kernel(const int64_t *__restrict__ tokens, int64_t tok_row_stride,
                                 int64_t tok_tab_stride, TablePtrs tabs, int n_tables, int64_t n_rows,
                                 int d, float *__restrict__ out, int64_t out_row_stride,
                                 const int32_t *__restrict__ out_rows, int accumulate,
                                 int32_t *__restrict__ err_flag) {
  const int warps_per_block = blockDim.x >> 5;
  const int64_t row = (int64_t)blockIdx.x * warps_per_block + (threadIdx.x >> 5);
  if (row >= n_rows) return;
  const int lane = threadIdx.x & 31;
  int64_t ids[kMaxTables];
#pragma unroll
  for (int j = 0; j < kMaxTables; ++j) {
    ids[j] = (j < n_tables) ? tokens[row * tok_row_stride + j * tok_tab_stride] : 0;
    // nn.Embedding raises IndexError for an id outside the table (embedding.py:46); here the read is clamped
    // (never out of bounds) and the caller's flag is raised so the host can report it
    if (j < n_tables && tabs.rows[j] > 0 && (ids[j] < 0 || ids[j] >= tabs.rows[j])) {
      if (err_flag != nullptr && lane == 0) atomicOr(err_flag, 1);
      ids[j] = ids[j] < 0 ? 0 : tabs.rows[j] - 1;
    }
  }
  float *orow = out + (out_rows ? (int64_t)out_rows[row] : row) * out_row_stride;
  for (int c = lane * 4; c < d; c += 128) {
    float4 acc;
    int j0 = 0;
    if (accumulate) {
      acc = *reinterpret_cast<const float4 *>(orow + c);
    } else {
      acc = *reinterpret_cast<const float4 *>(tabs.t[0] + ids[0] * d + c);
      j0 = 1;
    }
#pragma unroll
    for (int j = 0; j < kMaxTables; ++j) {
      if (j >= j0 && j < n_tables) {
        const float4 v = *reinterpret_cast<const float4 *>(tabs.t[j] + ids[j] * d + c);
        acc.x = __fadd_rn(acc.x, v.x);
        acc.y = __fadd_rn(acc.y, v.y);
        acc.z = __fadd_rn(acc.z, v.z);
        acc.w = __fadd_rn(acc.w, v.w);
      }
    }
    *reinterpret_cast<float4 *>(orow + c) = acc;
  }
}

// out = in + alpha * pe[pos0 + r]   (product rounded, then sum rounded: embedding.py:96)
__global__ void add_pe_kernel(const float *__restrict__ in, int64_t in_row_stride,
                              const float *__restrict__ pe, int64_t pos0,
                              const int32_t *__restrict__ positions,
                              const float *__restrict__ alpha, int64_t n_rows, int d,
                              float *__restrict__ out, int64_t out_row_stride,
                              const int32_t *__restrict__ out_rows) {
  const int warps_per_block = blockDim.x >> 5;
  const int64_t row = (int64_t)blockIdx.x * warps_per_block + (threadIdx.x >> 5);
  if (row >= n_rows) return;
  const int lane = threadIdx.x & 31;
  const float a = alpha[0];
  const float *irow = in + row * in_row_stride;
  const float *prow = pe + (positions ? (int64_t)positions[row] : pos0 + row) * d;
  float *orow = out + (out_rows ? (int64_t)out_rows[row] : row) * out_row_stride;
  for (int c = lane * 4; c < d; c += 128) {
    const float4 x = *reinterpret_cast<const float4 *>(irow + c);
    const float4 p = *reinterpret_cast<const float4 *>(prow + c);
    float4 o;
    o.x = __fadd_rn(x.x, __fmul_rn(a, p.x));
    o.y = __fadd_rn(x.y, __fmul_rn(a, p.y));
    o.z = __fadd_rn(x.z, __fmul_rn(a, p.z));
    o.w = __fadd_rn(x.w, __fmul_rn(a, p.w));
    *reinterpret_cast<float4 *>(orow + c) = o;
  }
}

// One warp per row; the row lives in registers (d <= 32*4*kMaxVec).  Two-pass moments.
// kPost: the post-norm of a post-LN layer (transformer.py:304-308, `x = norm(x + block(x))`): the normalised row also
// replaces the fp32 residual row it was read from (xpost, in place; `x` is unused), and `out` (the next GEMM's
// operand) may be NULL.
template <typename TO, int kVecs, bool kPost>
__global__ void layernorm_kernel(const float *__restrict__ x, int64_t x_row_stride,
                                 const int32_t *__restrict__ rows, int64_t n_rows, int d,
                                 const float *__restrict__ gamma, const float *__restrict__ beta,
                                 const float *__restrict__ ada_wb, float eps, TO *__restrict__ out,
                                 float *__restrict__ xpost) {
  const int warps_per_block = blockDim.x >> 5;
  const int64_t r = (int64_t)blockIdx.x * warps_per_block + (threadIdx.x >> 5);
  if (r >= n_rows) return;
  const int lane = threadIdx.x & 31;
  const int64_t src = rows ? (int64_t)rows[r] : r;
  const float *xr = (kPost ? xpost : x) + src * x_row_stride;
  float4 v[kVecs];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < kVecs; ++i) {
    const int c = (i * 32 + lane) * 4;
    if (c < d) {
      v[i] = *reinterpret_cast<const float4 *>(xr + c);
      s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
    } else {
      v[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
  }
  const float mean = warp_sum(s) / (float)d;
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < kVecs; ++i) {
    const int c = (i * 32 + lane) * 4;
    if (c < d) {
      const float a = v[i].x - mean, b = v[i].y - mean, e = v[i].z - mean, f = v[i].w - mean;
      q += (a * a + b * b) + (e * e + f * f);
    }
  }
  const float rstd = rsqrtf(warp_sum(q) / (float)d + eps);
  TO *orow = out + r * (int64_t)d;
#pragma unroll
  for (int i = 0; i < kVecs; ++i) {
    const int c = (i * 32 + lane) * 4;
    if (c < d) {
      const float4 g = *reinterpret_cast<const float4 *>(gamma + c);
      const float4 b = *reinterpret_cast<const float4 *>(beta + c);
      float y[4];
      y[0] = (v[i].x - mean) * rstd * g.x + b.x;
      y[1] = (v[i].y - mean) * rstd * g.y + b.y;
      y[2] = (v[i].z - mean) * rstd * g.z + b.z;
      y[3] = (v[i].w - mean) * rstd * g.w + b.w;
      if (ada_wb) {  // weight * LN(x) + bias, transformer.py:101
        const float4 w = *reinterpret_cast<const float4 *>(ada_wb + c);
        const float4 bb = *reinterpret_cast<const float4 *>(ada_wb + d + c);
        y[0] = w.x * y[0] + bb.x;
        y[1] = w.y * y[1] + bb.y;
        y[2] = w.z * y[2] + bb.z;
        y[3] = w.w * y[3] + bb.w;
      }
      if constexpr (kPost) {
        *reinterpret_cast<float4 *>(xpost + src * x_row_stride + c) = make_float4(y[0], y[1], y[2], y[3]);
        if (out == nullptr) continue;
      }
      if constexpr (sizeof(TO) == 4) {
        *reinterpret_cast<float4 *>(orow + c) = make_float4(y[0], y[1], y[2], y[3]);
      } else {
        __nv_bfloat162 p0 = __floats2bfloat162_rn(y[0], y[1]);
        __nv_bfloat162 p1 = __floats2bfloat162_rn(y[2], y[3]);
        uint2 pk;
        pk.x = *reinterpret_cast<uint32_t *>(&p0);
        pk.y = *reinterpret_cast<uint32_t *>(&p1);
        *reinterpret_cast<uint2 *>(orow + c) = pk;
      }
    }
  }
}

// out[n] = W[n,:] . emb + b[n]   (fp32, one warp per output)
__global__ void adaln_project_kernel(const float *__restrict__ W, const float *__restrict__ b,
                                     const float *__restrict__ emb, int d, float *__restrict__ out) {
  const int n = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (n >= 2 * d) return;
  const int lane = threadIdx.x & 31;
  const float *w = W + (int64_t)n * d;
  float acc = 0.f;
  for (int c = lane * 4; c < d; c += 128) {
    const float4 a = *reinterpret_cast<const float4 *>(w + c);
    const float4 e = *reinterpret_cast<const float4 *>(emb + c);
    acc += a.x * e.x + a.y * e.y + a.z * e.z + a.w * e.w;
  }
  acc = warp_sum(acc);
  if (lane == 0) out[n] = acc + b[n];
}

__global__ void gather_rows_kernel(const float *__restrict__ src, int64_t src_row_stride,
                                   const int32_t *__restrict__ rows, int64_t n_rows, int d,
                                   float *__restrict__ dst, int64_t dst_row_stride) {
  const int64_t r = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (r >= n_rows) return;
  const int lane = threadIdx.x & 31;
  const int32_t sr = rows[r];
  const float *s = src + (int64_t)sr * src_row_stride;
  float *o = dst + r * dst_row_stride;
  for (int c = lane * 4; c < d; c += 128)   // a negative index yields a zero row (the 'same' padding of the pre-net convs)
    *reinterpret_cast<float4 *>(o + c) = sr >= 0 ? *reinterpret_cast<const float4 *>(s + c) : make_float4(0.f, 0.f, 0.f, 0.f);
}

}  // namespace vb

using namespace vb;

VB_API int vb_embed_sum(const int64_t *tokens, int64_t tok_row_stride, int64_t tok_tab_stride,
                            const float *const *tables, const int32_t *table_rows, int n_tables,
                            int64_t n_rows, int d, float *out, int64_t out_row_stride, const int32_t *out_rows,
                            int accumulate, int32_t *err_flag, vb_stream_t stream) {
  VB_CHECK_ARG(n_tables >= 1 && n_tables <= kMaxTables, "vb_embed_sum: n_tables=%d not in [1,8]", n_tables);
  VB_CHECK_ARG(d % 4 == 0 && out_row_stride % 4 == 0, "vb_embed_sum: d and stride must be multiples of 4");
  if (n_rows == 0) return VB_OK;
  TablePtrs tp;
  for (int j = 0; j < kMaxTables; ++j) {
    tp.t[j] = j < n_tables ? tables[j] : nullptr;
    tp.rows[j] = (j < n_tables && table_rows) ? table_rows[j] : 0;
  }
  const int wpb = 4;
  embed_sum_kernel<<<(unsigned)((n_rows + wpb - 1) / wpb), wpb * 32, 0, (cudaStream_t)stream>>>(
      tokens, tok_row_stride, tok_tab_stride, tp, n_tables, n_rows, d, out, out_row_stride, out_rows, accumulate,
      err_flag);
  VB_LAUNCH_CHECK();
  return VB_OK;
}

VB_API int vb_add_pe(const float *in, int64_t in_row_stride, const float *pe, int64_t pos0,
                         const int32_t *positions, const float *alpha, int64_t n_rows, int d, float *out,
                         int64_t out_row_stride, const int32_t *out_rows, vb_stream_t stream) {
  VB_CHECK_ARG(d % 4 == 0 && in_row_stride % 4 == 0 && out_row_stride % 4 == 0,
               "vb_add_pe: d and strides must be multiples of 4");
  if (n_rows == 0) return VB_OK;
  const int wpb = 4;
  add_pe_kernel<<<(unsigned)((n_rows + wpb - 1) / wpb), wpb * 32, 0, (cudaStream_t)stream>>>(
      in, in_row_stride, pe, pos0, positions, alpha, n_rows, d, out, out_row_stride, out_rows);
  VB_LAUNCH_CHECK();
  return VB_OK;
}

template <typename TO, bool kPost = false>
static int launch_ln(const float *x, int64_t x_row_stride, const int32_t *rows, int64_t n_rows, int d,
                     const float *gamma, const float *beta, const float *ada_wb, float eps, TO *out,
                     cudaStream_t s, float *xpost = nullptr) {
  const int wpb = 4;
  const unsigned grid = (unsigned)((n_rows + wpb - 1) / wpb);
  const int vecs = (d + 127) / 128;
#define VB_LN_CASE(V)                                                                                  \
  layernorm_kernel<TO, V, kPost><<<grid, wpb * 32, 0, s>>>(x, x_row_stride, rows, n_rows, d, gamma, beta, \
                                                           ada_wb, eps, out, xpost)
  if (vecs <= 2) VB_LN_CASE(2);
  else if (vecs <= 4) VB_LN_CASE(4);
  else if (vecs <= 8) VB_LN_CASE(8);
  else if (vecs <= 16) VB_LN_CASE(16);
  else {
    set_error("vb_layernorm: d=%d > 2048 unsupported", d);
    return VB_ERR_UNSUPPORTED;
  }
#undef VB_LN_CASE
  VB_LAUNCH_CHECK();
  return VB_OK;
}

VB_API int vb_layernorm(const float *x, int64_t x_row_stride, const int32_t *rows, int64_t n_rows,
                            int d, const float *gamma, const float *beta, const float *ada_wb,
                            float eps, void *out, int out_dtype, vb_stream_t stream) {
  VB_CHECK_ARG(d % 4 == 0 && x_row_stride % 4 == 0, "vb_layernorm: d and stride must be multiples of 4");
  if (n_rows == 0) return VB_OK;
  if (out_dtype == VB_F32)
    return launch_ln<float>(x, x_row_stride, rows, n_rows, d, gamma, beta, ada_wb, eps, (float *)out,
                            (cudaStream_t)stream);
  if (out_dtype == VB_BF16)
    return launch_ln<bf16>(x, x_row_stride, rows, n_rows, d, gamma, beta, ada_wb, eps, (bf16 *)out,
                           (cudaStream_t)stream);
  set_error("vb_layernorm: bad out_dtype %d", out_dtype);
  return VB_ERR_ARG;
}

namespace vb {
int launch_post_norm(float *x, int64_t n_rows, int d, const float *gamma, const float *beta, const float *ada_wb,
                     float eps, void *out, int out_dtype, cudaStream_t s) {
  VB_CHECK_ARG(d % 4 == 0, "post_norm: d %% 4 != 0");
  if (n_rows == 0) return VB_OK;
  if (out_dtype == VB_BF16)
    return launch_ln<bf16, true>(nullptr, d, nullptr, n_rows, d, gamma, beta, ada_wb, eps, (bf16 *)out, s, x);
  return launch_ln<float, true>(nullptr, d, nullptr, n_rows, d, gamma, beta, ada_wb, eps, (float *)out, s, x);
}
}  // namespace vb

VB_API int vb_adaln_project(const float *W, const float *b, const float *emb, int d, float *out,
                                vb_stream_t stream) {
  VB_CHECK_ARG(d % 4 == 0, "vb_adaln_project: d %% 4 != 0");
  const int wpb = 8;
  adaln_project_kernel<<<(2 * d + wpb - 1) / wpb, wpb * 32, 0, (cudaStream_t)stream>>>(W, b, emb, d, out);
  VB_LAUNCH_CHECK();
  return VB_OK;
}

VB_API int vb_gather_rows(const float *src, int64_t src_row_stride, const int32_t *rows,
                              int64_t n_rows, int d, float *dst, int64_t dst_row_stride,
                              vb_stream_t stream) {
  VB_CHECK_ARG(d % 4 == 0, "vb_gather_rows: d %% 4 != 0");
  if (n_rows == 0) return VB_OK;
  const int wpb = 4;
  gather_rows_kernel<<<(unsigned)((n_rows + wpb - 1) / wpb), wpb * 32, 0, (cudaStream_t)stream>>>(
      src, src_row_stride, rows, n_rows, d, dst, dst_row_stride);
  VB_LAUNCH_CHECK();
  return VB_OK;
}
