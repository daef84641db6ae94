// Device-side tails of the AR loop and of a NAR stage.
//   * ar_sample_kernel: argmax over the 1025 logits, the stop rule of valle/models/valle.py:1044-1048
//     (argmax==EOS or sample==EOS or n_new > 16*S), the append of :1057 and the embedding + sine PE
//     of the appended token (:1013-1015) so the next decode step needs no host round trip
//     (the reference syncs to the host once per token).
//     ar_sample_kernel<true> draws the token with the seeded sampler (sample_row) instead of taking the argmax;
//     ar_sample_kernel<true, true> also adds the drawn token's log-probability under the raw logits to the row's score.
//   * sample_logits_kernel: the same sampler on caller-given logits (vb_sample_logits, vb_sample_logits_ex).
//   * nar_argmax_accumulate_kernel: samples = argmax(logits) (:1130) and
//     y_emb[:, Tp:] += nar_audio_embeddings[i+1](samples) (:1133-1134).
#include <math_constants.h>

#include <vector>

#include "common.cuh"
#include "kernels.cuh"

namespace vb {

struct ArgMax {
  float v;
  int i;
};
__device__ __forceinline__ ArgMax better(ArgMax a, ArgMax b) {
  // larger value wins; on ties the smaller index (torch.argmax returns the first maximum).  torch.argmax also takes
  // NaN as the maximum, the first NaN first: a NaN beats any number, and the smaller index wins between NaNs.  Without
  // that rule a row of NaN would keep the initial {-inf, 0x7fffffff} and the NAR tail would read next_emb far out of
  // bounds.  For rows without NaN the result is the same as the plain comparison.
  const bool an = a.v != a.v, bn = b.v != b.v;
  if (an || bn) return (bn && (!an || b.i < a.i)) ? b : a;
  return (b.v > a.v || (b.v == a.v && b.i < a.i)) ? b : a;
}
__device__ __forceinline__ ArgMax warp_argmax(ArgMax a) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    ArgMax b;
    b.v = __shfl_xor_sync(0xffffffffu, a.v, o);
    b.i = __shfl_xor_sync(0xffffffffu, a.i, o);
    a = better(a, b);
  }
  return a;
}

// ---- seeded top-k / temperature / nucleus sampler with repetition-aware fallback (include/valle_b200.h
// vb_sample_logits_ex), one CTA of 256 threads per row, the row held in registers as 5 values per thread
// (element i = threadIdx.x + 256 j, V <= 1280)
struct SamplerArgs {
  const uint64_t *seed;
  const int32_t *top_k;
  const float *temperature;
  const float *top_p;         // NULL: 1 (no nucleus)
  const int32_t *ras_window;  // NULL: 0 (no repetition-aware fallback)
  const int32_t *ras_max;
};
// one row's sampler parameters; hist: the utterance's generated ids [0, step) (read only when ras_window > 0)
struct RowSampler {
  uint64_t seed;
  int step, k;
  float temp, top_p;
  int ras_window, ras_max;
  const int32_t *hist;
};
__device__ __forceinline__ RowSampler row_sampler(const SamplerArgs &sa, int64_t r, int step, const int32_t *hist) {
  return RowSampler{sa.seed[r], step, sa.top_k[r], sa.temperature[r], sa.top_p ? sa.top_p[r] : 1.f,
                    sa.ras_window ? sa.ras_window[r] : 0, sa.ras_max ? sa.ras_max[r] : 0, hist};
}
constexpr int kSortMax = 2048;  // power of two >= 5 * 256
constexpr int kRasStream = 2048;  // the fallback draw hashes id i at index i + 2^11 (disjoint from the first draw's)
struct SamplerSmem {
  unsigned hist[256];
  unsigned wsum[8];
  ArgMax wbest[8];
  int sel_bin, sel_k;
  float wsumf[8];
  int count, cut, ras_count;
  unsigned long long keys[kSortMax];  // nucleus: (float_key(l'), ~id) of the kept tokens, sorted descending
};
// order-preserving float <-> uint32 (larger float, larger key)
__device__ __forceinline__ uint32_t float_key(float f) {
  const uint32_t u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float key_float(uint32_t k) {
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}
// the row's maximum (smallest index on ties), returned to every thread
__device__ __forceinline__ ArgMax block_argmax(ArgMax a, ArgMax *wbest) {
  a = warp_argmax(a);
  if ((threadIdx.x & 31) == 0) wbest[threadIdx.x >> 5] = a;
  __syncthreads();
  a = wbest[0];
#pragma unroll
  for (int w = 1; w < 8; ++w) a = better(a, wbest[w]);
  return a;
}
// exact k-th largest of the n valid values (0 < k < n): radix select over the order-preserving keys, 4 passes of 8
// bits, each a 256-bin histogram of the keys that match the digits chosen so far plus a suffix scan over the bins
__device__ float radix_kth(const float (&x)[5], int n, int k, SamplerSmem &sm) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  uint32_t key[5];
#pragma unroll
  for (int j = 0; j < 5; ++j) key[j] = float_key(x[j]);
  uint32_t prefix = 0, mask = 0;
#pragma unroll 1
  for (int shift = 24; shift >= 0; shift -= 8) {
    sm.hist[tid] = 0;
    __syncthreads();
#pragma unroll
    for (int j = 0; j < 5; ++j)
      if (tid + j * 256 < n && (key[j] & mask) == prefix) atomicAdd(&sm.hist[(key[j] >> shift) & 255u], 1u);
    __syncthreads();
    // thread t owns bin 255 - t: the inclusive prefix sum over t is the count of keys whose digit is >= that bin
    const int bin = 255 - tid;
    const unsigned c = sm.hist[bin];
    unsigned s = c;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const unsigned t = __shfl_up_sync(0xffffffffu, s, o);
      if (lane >= o) s += t;
    }
    if (lane == 31) sm.wsum[warp] = s;
    __syncthreads();
    for (int w = 0; w < warp; ++w) s += sm.wsum[w];
    if (s >= (unsigned)k && s - c < (unsigned)k) {  // exactly one bin holds the k-th key
      sm.sel_bin = bin;
      sm.sel_k = k - (int)(s - c);
    }
    __syncthreads();
    prefix |= (uint32_t)sm.sel_bin << shift;
    mask |= 255u << shift;
    k = sm.sel_k;
  }
  return key_float(prefix);
}
// Gumbel noise g_i of (seed, step, hash index): 23 bits, m + 0.5 fits fp32's 24-bit significand, so u is exact, in
// [2^-24, 1 - 2^-24] and g finite (a 24-bit m + 0.5 would round 2^24 - 0.5 up to 2^24: u = 1, g = +inf)
__device__ __forceinline__ float gumbel(uint64_t seed, int step, int idx) {
  const uint64_t h = mix64(seed, (uint64_t)(int64_t)step, (uint64_t)idx);
  const float u = ((float)(uint32_t)(h >> 41) + 0.5f) * 1.1920928955078125e-7f;
  return -logf(-logf(u));
}
// (value, ascending id) order of the nucleus as one integer: a larger key comes first
__device__ __forceinline__ unsigned long long order_key(float v, int i) {
  return ((unsigned long long)float_key(v) << 32) | (0xFFFFFFFFu - (uint32_t)i);
}
// Nucleus of the kept set (include/valle_b200.h vb_sample_logits_ex): sorts the kept tokens by order_key (bitonic, in
// shared memory, over the next power of two >= their count), sums e = expf(l' - max) over sorted positions in the
// association order the header states (5 positions per thread in sequence, a Hillis-Steele warp scan, the warp
// totals in sequence) and returns the order key of the first position whose prefix sum exceeds top_p * Z (of the last
// kept token if none does): the nucleus is every kept token whose order key is >= it.
__device__ unsigned long long nucleus_cut(const float (&x)[5], const bool (&kept)[5], float top_p, SamplerSmem &sm) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  // gather the kept keys into keys[0, m) (in any order: the keys are distinct, so the sort fixes the result), zeros up
  // to N
  if (tid == 0) sm.count = 0;
  __syncthreads();
#pragma unroll
  for (int j = 0; j < 5; ++j)
    if (kept[j]) sm.keys[atomicAdd(&sm.count, 1)] = order_key(x[j], tid + j * 256);
  __syncthreads();
  const int m = sm.count;
  int N = 2;
  while (N < m) N <<= 1;
  for (int i = m + tid; i < N; i += 256) sm.keys[i] = 0ull;
  if (tid == 0) sm.cut = m - 1;
  __syncthreads();
#pragma unroll 1
  for (int size = 2; size <= N; size <<= 1) {
#pragma unroll 1
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      for (int t = tid; t < (N >> 1); t += 256) {
        const int lo = 2 * t - (t & (stride - 1)), hi = lo + stride;
        const unsigned long long a = sm.keys[lo], b = sm.keys[hi];
        if ((a < b) == ((lo & size) == 0)) {  // descending where bit `size` of lo is clear
          sm.keys[lo] = b;
          sm.keys[hi] = a;
        }
      }
      __syncthreads();
    }
  }
  const float mx = key_float((uint32_t)(sm.keys[0] >> 32));
  float c[5], s = 0.f;
#pragma unroll
  for (int q = 0; q < 5; ++q) {
    const int p = tid * 5 + q;
    const float e = p < m ? expf(__fsub_rn(key_float((uint32_t)(sm.keys[p] >> 32)), mx)) : 0.f;
    s = __fadd_rn(s, e);
    c[q] = s;
  }
  float ws = s;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const float t = __shfl_up_sync(0xffffffffu, ws, o);
    if (lane >= o) ws = __fadd_rn(ws, t);
  }
  float ex = __shfl_up_sync(0xffffffffu, ws, 1);
  if (lane == 0) ex = 0.f;
  if (lane == 31) sm.wsumf[warp] = ws;
  __syncthreads();
  float off = 0.f, Z = 0.f;
#pragma unroll
  for (int w = 0; w < 8; ++w) {
    if (w == warp) off = Z;
    Z = __fadd_rn(Z, sm.wsumf[w]);
  }
  const float thr = __fmul_rn(top_p, Z), base = __fadd_rn(off, ex);
#pragma unroll
  for (int q = 0; q < 5; ++q) {
    const int p = tid * 5 + q;
    if (p < m && __fadd_rn(base, c[q]) > thr) {
      atomicMin(&sm.cut, p);
      break;
    }
  }
  __syncthreads();
  return sm.keys[sm.cut];
}
// Gumbel-max draw over the top-k set of l / T, narrowed to its nucleus when top_p < 1; `amax` = argmax(l), the draw
// for k == 1.  With ras_window > 0, a draw that fills more than ras_max of the last ras_window ids of `hist` is
// replaced by a Gumbel-max draw over all of l / T.  Called by all 256 threads, returns the id to every thread.
__device__ int sample_row(const float (&l)[5], int n, int amax, const RowSampler &r, SamplerSmem &sm) {
  const bool ras = r.ras_window > 0;
  if (r.k == 1 && !ras) return amax;
  const int tid = threadIdx.x;
  float x[5];
#pragma unroll
  for (int j = 0; j < 5; ++j) x[j] = r.temp != 1.f ? __fdiv_rn(l[j], r.temp) : l[j];
  int d = amax;
  if (r.k != 1) {
    const float kth = (r.k > 0 && r.k < n) ? radix_kth(x, n, r.k, sm) : -CUDART_INF_F;
    bool kept[5];
#pragma unroll
    for (int j = 0; j < 5; ++j) kept[j] = tid + j * 256 < n && x[j] >= kth;
    if (r.top_p < 1.f) {
      const unsigned long long cut = nucleus_cut(x, kept, r.top_p, sm);
#pragma unroll
      for (int j = 0; j < 5; ++j) kept[j] = kept[j] && order_key(x[j], tid + j * 256) >= cut;
    }
    ArgMax best{-CUDART_INF_F, 0x7fffffff};
#pragma unroll
    for (int j = 0; j < 5; ++j) {
      const int i = tid + j * 256;
      if (kept[j]) best = better(best, ArgMax{__fadd_rn(x[j], gumbel(r.seed, r.step, i)), i});
    }
    d = block_argmax(best, sm.wbest).i;
  }
  if (ras) {
    // count of d among the utterance's last ras_window ids (warp 0), then the unfiltered redraw if it is too high
    if (tid < 32) {
      int c = 0;
      for (int j = max(0, r.step - r.ras_window) + tid; j < r.step; j += 32) c += r.hist[j] == d;
      c = __reduce_add_sync(0xffffffffu, c);
      if (tid == 0) sm.ras_count = c;
    }
    __syncthreads();  // also orders the reads of sm.wbest above before the writes below
    if (sm.ras_count > r.ras_max) {
      ArgMax best{-CUDART_INF_F, 0x7fffffff};
#pragma unroll
      for (int j = 0; j < 5; ++j) {
        const int i = tid + j * 256;
        if (i < n) best = better(best, ArgMax{__fadd_rn(x[j], gumbel(r.seed, r.step, i + kRasStream)), i});
      }
      d = block_argmax(best, sm.wbest).i;
    }
  }
  return d;
}

// log-sum-exp of one row of logits as a 256-thread CTA holds it (element tid + 256 j, -inf padding), mx its maximum:
// mx + logf(z), z = sum expf(l - mx), each thread's 5 terms in order, a warp sum, then the 8 warps' sums in order.
// vb_ar_state.logprob and the beam scores both use it.  wz: 8 floats of shared memory.
__device__ __forceinline__ float row_logsumexp(const float (&lv)[5], float mx, float *wz, int lane, int warp) {
  float z = 0.f;
#pragma unroll
  for (int j = 0; j < 5; ++j) z += expf(lv[j] - mx);
  z = warp_sum(z);
  if (lane == 0) wz[warp] = z;
  __syncthreads();
  z = 0.f;
#pragma unroll
  for (int w = 0; w < 8; ++w) z += wz[w];
  return mx + logf(z);
}

// kMixed (vb_ar_head.greedy == 4): the rows of beam groups (beam_first[b] >= 0) only reduce their logits, the beam tail
// that follows takes them
template <bool kSample, bool kScore = false, bool kMixed = false>
__global__ void __launch_bounds__(256)
ar_sample_kernel(float *__restrict__ logits, int64_t ld_logits, const float *__restrict__ partials, int splits,
                 int ldp, int n_vocab, int eos_id,
                 const float *__restrict__ audio_emb, const float *__restrict__ alpha,
                 const float *__restrict__ pe, int pe_rows, const int32_t *__restrict__ text_len,
                 const int32_t *__restrict__ prompt_len, const int32_t *__restrict__ max_new,
                 int32_t *__restrict__ n_gen, int32_t *__restrict__ finished,
                 int32_t *__restrict__ tokens, int tok_stride, float *__restrict__ x_cur, int d,
                 const int64_t *__restrict__ forced, int reduce_only, LnFoldStats fold, const float *__restrict__ fold_d,
                 SamplerArgs sa, float *__restrict__ logprob, const int32_t *__restrict__ beam_first) {
  __shared__ ArgMax wbest[8];
  __shared__ int s_tok, s_pos;
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  pdl_launch_dependents();
  pdl_wait();
  vb_trace(TR_SAMPLE * 2);
  if constexpr (kMixed) reduce_only |= beam_first[b] >= 0;
  if (finished[b] != 0 && !reduce_only) {  // uniform per CTA
    // a stopped utterance still rides through the batched step: give it a fixed, bounded input row (its residual
    // stream is updated in place by the layer chain and would otherwise drift step over step); the scatter and
    // attention kernels skip its KV cache
    float *xo = x_cur + (int64_t)b * d;
    for (int c = tid * 4; c < d; c += 1024) *reinterpret_cast<float4 *>(xo + c) = make_float4(0.f, 0.f, 0.f, 0.f);
    return;
  }
  // scalars of the stop rule: in flight together with the logits instead of after the argmax
  const int n_new = n_gen[b], p_len = prompt_len[b], cap_new = max_new[b];
  const int forced_tok = forced ? (int)forced[b] : -1;
  RowSampler rs{};
  if constexpr (kSample) rs = row_sampler(sa, b, n_new, tokens + (int64_t)b * tok_stride);
  float *row = logits + (int64_t)b * ld_logits;
  float lv[5];  // kSample: the row in registers, element tid + 256 j
  ArgMax best{-CUDART_INF_F, 0x7fffffff};
  // final LayerNorm folded into ar_predict_layer (gemm_decode_x_kernel): logit = rstd (acc - mean c[i]) + (beta W^T)[i]
  float f_mean = 0.f, f_rstd = 1.f;
  const bool folded = fold.stats != nullptr && partials != nullptr;
  if (folded) ln_fold_moments(fold, b, b, f_mean, f_rstd);
  if (partials && n_vocab <= 5 * 256 && splits <= 8) {
    // head projection split-K partials, summed in fixed order; all loads of the row issued at once
    float v[5][8];
#pragma unroll
    for (int j = 0; j < 5; ++j) {
      const int i = tid + j * 256;
      const float *p = partials + (int64_t)b * ldp + min(i, n_vocab - 1);
#pragma unroll
      for (int s = 0; s < 8; ++s) v[j][s] = s < splits ? __ldcg(p + (int64_t)s * 64 * ldp) : 0.f;
    }
#pragma unroll
    for (int j = 0; j < 5; ++j) {
      const int i = tid + j * 256;
      float a = v[j][0];
#pragma unroll
      for (int s = 1; s < 8; ++s)
        if (s < splits) a += v[j][s];
      if (i < n_vocab) {
        if (folded) a = f_rstd * (a - f_mean * fold.c[i]) + fold_d[i];
        row[i] = a;
        best = better(best, ArgMax{a, i});
      }
      if constexpr (kSample) lv[j] = i < n_vocab ? a : -CUDART_INF_F;
    }
  } else {
    for (int i = tid; i < n_vocab; i += 256) {
      float v;
      if (partials) {
        const float *p = partials + (int64_t)b * ldp + i;
        v = __ldcg(p);
#pragma unroll 8
        for (int s = 1; s < splits; ++s) v += __ldcg(p + (int64_t)s * 64 * ldp);
        if (folded) v = f_rstd * (v - f_mean * fold.c[i]) + fold_d[i];
        row[i] = v;
      } else {
        v = row[i];
      }
      best = better(best, ArgMax{v, i});
    }
    if constexpr (kSample) {  // read back this thread's elements of the row (its own writes)
#pragma unroll
      for (int j = 0; j < 5; ++j) lv[j] = tid + j * 256 < n_vocab ? row[tid + j * 256] : -CUDART_INF_F;
    }
  }
  if constexpr (!kSample || kMixed) {
    if (reduce_only) return;
  }
  int draw = -1;
  float lse = 0.f;   // kScore: logsumexp of the raw logits
  if constexpr (kSample) {
    __shared__ SamplerSmem smp;
    best = block_argmax(best, wbest);
    draw = sample_row(lv, n_vocab, best.i, rs, smp);
    if constexpr (kScore) {
      __shared__ float wz[8];
      lse = row_logsumexp(lv, best.v, wz, lane, warp);
    }
  } else {
    best = warp_argmax(best);
    if (lane == 0) wbest[warp] = best;
    __syncthreads();
  }
  if (tid == 0) {
    ArgMax a = wbest[0];
#pragma unroll
    for (int w = 1; w < 8; ++w) a = better(a, wbest[w]);
    const int samp = kSample ? draw : (forced ? forced_tok : a.i);
    const bool stop = (a.i == eos_id) || (samp == eos_id) || (n_new > cap_new) || (n_new >= tok_stride);
    if (stop) {
      finished[b] = (n_new == 0) ? 2 : 1;
      s_tok = -1;
    } else {
      tokens[(int64_t)b * tok_stride + n_new] = samp;
      if constexpr (kScore) logprob[b] += row[samp] - lse;
      n_gen[b] = n_new + 1;
      s_tok = samp;
      s_pos = min(p_len + n_new, pe_rows - 1);
    }
  }
  __syncthreads();
  const int tok = s_tok;
  if (tok < 0) {  // stopped at this step: same fixed input row as above
    float *xo = x_cur + (int64_t)b * d;
    for (int c = tid * 4; c < d; c += 1024) *reinterpret_cast<float4 *>(xo + c) = make_float4(0.f, 0.f, 0.f, 0.f);
    return;
  }
  const float a = alpha[0];
  const float *e = audio_emb + (int64_t)tok * d;
  const float *p = pe + (int64_t)s_pos * d;
  float *xo = x_cur + (int64_t)b * d;
  for (int c = tid * 4; c < d; c += 1024) {
    const float4 ev = *reinterpret_cast<const float4 *>(e + c);
    const float4 pv = *reinterpret_cast<const float4 *>(p + c);
    float4 o;
    o.x = __fadd_rn(ev.x, __fmul_rn(a, pv.x));
    o.y = __fadd_rn(ev.y, __fmul_rn(a, pv.y));
    o.z = __fadd_rn(ev.z, __fmul_rn(a, pv.z));
    o.w = __fadd_rn(ev.w, __fmul_rn(a, pv.w));
    *reinterpret_cast<float4 *>(xo + c) = o;
  }
}

int launch_ar_sample(float *logits, int64_t ld_logits, const SplitK &in, const vb_ar_head *head, vb_ar_state *st,
                     int d, const int64_t *forced, int reduce_only, bool pdl, cudaStream_t s) {
  const bool sample = (head->greedy == 2 || head->greedy == 4) && forced == nullptr && !reduce_only;
  const bool score = sample && st->logprob != nullptr;
  const bool mixed = sample && head->greedy == 4;
  SamplerArgs sa{};
  if (sample) {
    VB_CHECK_ARG(st->sample_seed && st->top_k && st->temperature,
                 "vb_ar_head.greedy == %d: sampler arrays not set", head->greedy);
    VB_CHECK_ARG(head->n_vocab <= 5 * 256, "device sampler: n_vocab %d > 1280", head->n_vocab);
    sa = SamplerArgs{st->sample_seed, st->top_k, st->temperature, st->top_p, st->ras_window, st->ras_max};
  }
  const auto k = mixed ? (score ? ar_sample_kernel<true, true, true> : ar_sample_kernel<true, false, true>)
                 : score ? ar_sample_kernel<true, true> : sample ? ar_sample_kernel<true> : ar_sample_kernel<false>;
  VB_CUDA(launch_kernel(k, dim3(st->B), dim3(256), 0, s, pdl,
                        logits, ld_logits, in.part, in.splits, in.ldp, head->n_vocab, head->eos_id, head->audio_emb,
                        head->alpha, head->pe, head->pe_rows, (const int32_t *)st->text_len,
                        (const int32_t *)st->prompt_len, (const int32_t *)st->max_new, st->n_gen, st->finished,
                        st->tokens, st->tok_stride, st->x_cur, d, forced, reduce_only, in.fold, in.bias, sa,
                        score ? st->logprob : nullptr, mixed ? st->beam_first : nullptr));
  count_launch();
  return VB_OK;
}

// ---- beam search tail (include/valle_b200.h "Beam search"), one CTA of 256 threads per group of n <= 16 rows.
// The ranking (c desc, l desc, j asc, v asc) restricted to one row j is (l desc, v asc): c = fl(s_j + fl(l - lse_j)) is
// non-decreasing in l.  So each row's 2n best by order_key (warp per row) hold the group's 2n best, which hold the n
// first non-EOS candidates (a row has one EOS candidate) and every candidate of rank < n; warp 0 merges the rows'
// sorted lists into the group's ranking.
constexpr int kBeamMax = 16;
struct BeamCand {
  float c, l;
  int v;
};
// -0 ranks as +0 (the ranking compares values)
__device__ __forceinline__ uint32_t rank_key(float f) { return float_key(f == 0.f ? 0.f : f); }

__global__ void __launch_bounds__(256)
ar_beam_kernel(const float *__restrict__ logits, int64_t ld_logits, int n_vocab, int eos_id, int n,
               const float *__restrict__ audio_emb, const float *__restrict__ alpha, const float *__restrict__ pe,
               int pe_rows, const int32_t *__restrict__ prompt_len, const int32_t *__restrict__ max_new,
               int32_t *__restrict__ n_gen, int32_t *__restrict__ finished, int32_t *__restrict__ tokens,
               int tok_stride, float *__restrict__ x_cur, int d, uint8_t *__restrict__ anc,
               float *__restrict__ score, float *__restrict__ fin_score, int32_t *__restrict__ fin_len,
               uint8_t *__restrict__ fin_anc, float *__restrict__ lse_out, const int32_t *__restrict__ first,
               const int32_t *__restrict__ width) {
  __shared__ ArgMax wbest[8];
  __shared__ float wz[8];
  __shared__ float lse[kBeamMax];
  __shared__ BeamCand cand[kBeamMax][2 * kBeamMax];
  __shared__ int ranked[2 * kBeamMax];                       // j * 2n + index in row j's list
  __shared__ int npar[kBeamMax], ntok[kBeamMax];
  __shared__ float nsc[kBeamMax];
  __shared__ int s_stop, s_fpar, s_len, s_from_fin;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  pdl_launch_dependents();
  pdl_wait();
  // per-row groups: one CTA per row, the first row of a group runs it (and indexes its finished hypothesis); a width
  // out of range, or a group past the last row, is refused on the host and never read out of bounds here
  const int g = blockIdx.x;
  int r0 = g * n;
  if (first != nullptr) {
    if (first[g] != g) return;
    r0 = g;
    n = width[g];
    if (n < 2 || n > kBeamMax || g + n > (int)gridDim.x) return;
  }
  const int K = 2 * n;
  if (finished[r0] != 0) {   // a stopped group rides along with fixed input rows, as ar_sample_kernel's rows do
    for (int j = 0; j < n; ++j) {
      float *xo = x_cur + (int64_t)(r0 + j) * d;
      for (int c = tid * 4; c < d; c += 1024) *reinterpret_cast<float4 *>(xo + c) = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    return;
  }
  const int t = n_gen[r0];
  const bool cap = t > max_new[r0] || t >= tok_stride;
  if (!cap) {
    // every row's log-sum-exp, as the logprob path computes it
    for (int j = 0; j < n; ++j) {
      const float *row = logits + (int64_t)(r0 + j) * ld_logits;
      float lv[5];
      ArgMax best{-CUDART_INF_F, 0x7fffffff};
#pragma unroll
      for (int q = 0; q < 5; ++q) {
        const int i = tid + q * 256;
        lv[q] = i < n_vocab ? row[i] : -CUDART_INF_F;
        if (i < n_vocab) best = better(best, ArgMax{lv[q], i});
      }
      best = block_argmax(best, wbest);
      const float l = row_logsumexp(lv, best.v, wz, lane, warp);
      if (tid == 0) {
        lse[j] = l;
        if (lse_out != nullptr) lse_out[r0 + j] = l;
      }
    }
    __syncthreads();
    // each row's K best (l desc, v asc), one warp per row, the row in registers (element lane + 32 q)
    for (int j = warp; j < n; j += 8) {
      const float *row = logits + (int64_t)(r0 + j) * ld_logits;
      float x[40];
#pragma unroll
      for (int q = 0; q < 40; ++q) x[q] = lane + 32 * q < n_vocab ? row[lane + 32 * q] : 0.f;
      uint64_t taken = 0;
      auto mine = [&]() {
        unsigned long long k = 0;
#pragma unroll
        for (int q = 0; q < 40; ++q) {
          const int v = lane + 32 * q;
          const unsigned long long kq = ((unsigned long long)rank_key(x[q]) << 32) | (0xFFFFFFFFu - (uint32_t)v);
          if (v < n_vocab && !((taken >> q) & 1) && kq > k) k = kq;
        }
        return k;
      };
      unsigned long long km = mine();
      const float sj = score[r0 + j], lj = lse[j];
      for (int r = 0; r < K; ++r) {
        unsigned long long w = km;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
          const unsigned long long ow = __shfl_xor_sync(0xffffffffu, w, o);
          w = ow > w ? ow : w;
        }
        const int v = (int)(0xFFFFFFFFu - (uint32_t)w);
        if (lane == (v & 31)) {
          taken |= 1ull << (v >> 5);
          km = mine();
        }
        if (lane == 0) {
          const float l = key_float((uint32_t)(w >> 32));
          cand[j][r] = BeamCand{__fadd_rn(sj, __fsub_rn(l, lj)), l, v};
        }
      }
    }
    __syncthreads();
    // the group's K best: merge of the rows' sorted lists (c desc, l desc; ties to the smaller j)
    if (warp == 0) {
      int idx = 0;
      for (int r = 0; r < K; ++r) {
        unsigned long long w = 0;
        if (lane < n && idx < K) {
          const BeamCand &c = cand[lane][idx];
          w = ((unsigned long long)rank_key(c.c) << 32) | rank_key(c.l);
        }
        int wl = lane;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
          const unsigned long long ow = __shfl_xor_sync(0xffffffffu, w, o);
          const int ol = __shfl_xor_sync(0xffffffffu, wl, o);
          if (ow > w || (ow == w && ol < wl)) {
            w = ow;
            wl = ol;
          }
        }
        if (lane == wl) {
          ranked[r] = lane * K + idx;
          ++idx;
        }
      }
    }
    __syncthreads();
  }
  if (tid == 0) {
    float fc = fin_score[2 * g], fo = fin_score[2 * g + 1];
    int fpar = -1, stop = 1, from_fin = 0, len = t;
    if (cap) {
      from_fin = fc > -CUDART_INF_F && fc >= score[r0];
    } else {
      int live = 0;
      for (int r = 0; r < K && live < n; ++r) {
        const int j = ranked[r] / K;
        const BeamCand c = cand[j][ranked[r] % K];
        if (c.v == eos_id) {
          if (r < n && c.c > fc) {
            fc = c.c;
            fo = score[r0 + j];
            fpar = j;
          }
        } else {
          npar[live] = j;
          ntok[live] = c.v;
          nsc[live] = c.c;
          ++live;
        }
      }
      if (fpar >= 0) {
        fin_score[2 * g] = fc;
        fin_score[2 * g + 1] = fo;
        fin_len[g] = t;
      }
      stop = fc > -CUDART_INF_F && fc >= nsc[0];
      from_fin = stop;
    }
    if (stop) {
      len = from_fin ? (fpar >= 0 ? t : fin_len[g]) : t;
      score[r0] = from_fin ? fo : score[r0];
    }
    s_stop = stop;
    s_fpar = fpar;
    s_len = len;
    s_from_fin = from_fin;
  }
  __syncthreads();
  const int stop = s_stop, fpar = s_fpar;
  const int64_t ld = tok_stride;
  // ancestry pass, thread per position: the n rows' old entries, then the finished hypothesis's copy and (going on)
  // the new beams' entries
  for (int i = tid; i < t && (fpar >= 0 || !stop); i += 256) {
    unsigned long long lo = 0, hi = 0;
    for (int j = 0; j < n; ++j) {
      const unsigned long long a = anc[(r0 + j) * ld + i];
      if (j < 8) lo |= a << (8 * j);
      else hi |= a << (8 * (j - 8));
    }
    auto old = [&](int j) { return (uint8_t)(((j < 8) ? lo : hi) >> (8 * (j & 7))); };
    if (fpar >= 0) fin_anc[g * ld + i] = old(fpar);
    if (!stop)
      for (int k = 0; k < n; ++k) anc[(r0 + k) * ld + i] = old(npar[k]);
  }
  if (stop) {
    __syncthreads();   // fin_anc is complete
    const int len = s_len;
    const uint8_t *src = s_from_fin ? fin_anc + g * ld : anc + r0 * ld;
    for (int i = tid; i < len; i += 256) tokens[r0 * ld + i] = tokens[(r0 + src[i]) * ld + i];
    for (int j = 0; j < n; ++j) {
      float *xo = x_cur + (int64_t)(r0 + j) * d;
      for (int c = tid * 4; c < d; c += 1024) *reinterpret_cast<float4 *>(xo + c) = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    if (tid < n) finished[r0 + tid] = len == 0 ? 2 : 1;
    if (tid == 0) n_gen[r0] = len;
    return;
  }
  if (tid < n) {
    anc[(r0 + tid) * ld + t] = (uint8_t)tid;
    tokens[(r0 + tid) * ld + t] = ntok[tid];
    score[r0 + tid] = nsc[tid];
    n_gen[r0 + tid] = t + 1;
  }
  // the new beams' input rows: embedding + alpha * PE, as ar_sample_kernel
  const float a = alpha[0];
  const float *p = pe + (int64_t)min(prompt_len[r0] + t, pe_rows - 1) * d;
  for (int k = 0; k < n; ++k) {
    const float *e = audio_emb + (int64_t)ntok[k] * d;
    float *xo = x_cur + (int64_t)(r0 + k) * d;
    for (int c = tid * 4; c < d; c += 1024) {
      const float4 ev = *reinterpret_cast<const float4 *>(e + c);
      const float4 pv = *reinterpret_cast<const float4 *>(p + c);
      float4 o;
      o.x = __fadd_rn(ev.x, __fmul_rn(a, pv.x));
      o.y = __fadd_rn(ev.y, __fmul_rn(a, pv.y));
      o.z = __fadd_rn(ev.z, __fmul_rn(a, pv.z));
      o.w = __fadd_rn(ev.w, __fmul_rn(a, pv.w));
      *reinterpret_cast<float4 *>(xo + c) = o;
    }
  }
}

int launch_beam_tail(const vb_ar_head *head, vb_ar_state *st, int d, bool pdl, cudaStream_t s, float *lse) {
  const bool per_row = st->beam_first != nullptr;
  const int n = per_row ? kBeamMax : st->beam_width;   // per-row groups: the widest group
  VB_CHECK_ARG(head->n_vocab <= 40 * 32 && 2 * n <= head->n_vocab, "beam tail: n_vocab %d not in [2n, 1280]",
               head->n_vocab);
  const int64_t ldl = (head->n_vocab + 3) & ~3;
  VB_CUDA(launch_kernel(ar_beam_kernel, dim3(per_row ? st->B : st->B / n), dim3(256), 0, s, pdl,
                        (const float *)st->logits, ldl, head->n_vocab, head->eos_id, n, head->audio_emb, head->alpha,
                        head->pe, head->pe_rows, st->prompt_len, st->max_new, st->n_gen, st->finished, st->tokens,
                        st->tok_stride, st->x_cur, d, st->beam_anc, st->beam_score, st->beam_fin_score,
                        st->beam_fin_len, st->beam_fin_anc, lse, st->beam_first, st->beam_n));
  count_launch();
  return VB_OK;
}

// one CTA per admitted row i, slot = slots[i] (launch_ar_admit_copy)
__global__ void __launch_bounds__(256)
ar_admit_copy_kernel(vb_ar_state st, vb_ar_state cs, const int32_t *__restrict__ slots, int d, int ldl, int n_vocab,
                     int scatter) {
  const int i = blockIdx.x, tid = threadIdx.x;
  const int s = slots[i];
  if (!scatter) {
    if (tid == 0) {
      const_cast<int32_t *>(cs.text_len)[i] = st.text_len[s];
      const_cast<int32_t *>(cs.prompt_len)[i] = st.prompt_len[s];
      const_cast<int32_t *>(cs.max_new)[i] = st.max_new[s];
      cs.n_gen[i] = 0;
      cs.finished[i] = 0;
      cs.tokens[i] = 0;
      if (cs.logprob) cs.logprob[i] = 0.f;
      if (st.sample_seed) {
        const_cast<uint64_t *>(cs.sample_seed)[i] = st.sample_seed[s];
        const_cast<int32_t *>(cs.top_k)[i] = st.top_k[s];
        const_cast<float *>(cs.temperature)[i] = st.temperature[s];
        const_cast<float *>(cs.top_p)[i] = st.top_p ? st.top_p[s] : 1.f;
        const_cast<int32_t *>(cs.ras_window)[i] = st.ras_window ? st.ras_window[s] : 0;
        const_cast<int32_t *>(cs.ras_max)[i] = st.ras_max ? st.ras_max[s] : 0;
      }
      if (cs.beam_first) {   // greedy == 4: a group's rows start as a fresh beam state's (include/valle_b200.h)
        const int f = st.beam_first[s];
        const_cast<int32_t *>(cs.beam_first)[i] = f < 0 ? -1 : i - (s - f);
        const_cast<int32_t *>(cs.beam_n)[i] = f < 0 ? 0 : st.beam_n[s];
        cs.beam_anc[i] = 0;
        cs.beam_score[i] = s == f ? 0.f : -CUDART_INF_F;
        cs.beam_fin_score[2 * i] = -CUDART_INF_F;
        cs.beam_fin_score[2 * i + 1] = st.beam_fin_score[2 * s + 1];
        cs.beam_fin_len[i] = st.beam_fin_len[s];
      }
    }
    return;
  }
  if (tid == 0) {
    st.n_gen[s] = cs.n_gen[i];
    st.finished[s] = cs.finished[i];
    st.tokens[(int64_t)s * st.tok_stride] = cs.tokens[i];
    if (cs.logprob) st.logprob[s] = cs.logprob[i];
    if (cs.beam_first && st.beam_first[s] >= 0) {
      st.beam_anc[(int64_t)s * st.tok_stride] = cs.beam_anc[i];
      st.beam_score[s] = cs.beam_score[i];
      if (st.beam_first[s] == s) {
        st.beam_fin_score[2 * s] = cs.beam_fin_score[2 * i];
        st.beam_fin_score[2 * s + 1] = cs.beam_fin_score[2 * i + 1];
        st.beam_fin_len[s] = cs.beam_fin_len[i];
      }
    }
  }
  for (int c = tid; c < d; c += 256) st.x_cur[(int64_t)s * d + c] = cs.x_cur[(int64_t)i * d + c];
  for (int c = tid; c < n_vocab; c += 256) st.logits[(int64_t)s * ldl + c] = cs.logits[(int64_t)i * ldl + c];
}

int launch_ar_admit_copy(vb_ar_state *st, const vb_ar_state *cs, const int32_t *slots, int d, int ldl, int n_vocab,
                         bool scatter, cudaStream_t s) {
  ar_admit_copy_kernel<<<cs->B, 256, 0, s>>>(*st, *cs, slots, d, ldl, n_vocab, scatter ? 1 : 0);
  VB_LAUNCH_CHECK();
  return VB_OK;
}

// vb_ar_fork_prefix: one CTA per (row i, layer, head).  Row b = slots[i] gets the rows [P_b, S_b + Tp_b) of its K and V
// streams of that layer and head from its parent's, the rows the shared prompt prefix (kv_shared_rows) leaves to its
// own streams: at most 15 rows of 64 elements each, copied as 16-byte vectors.  A row that is its own parent is left.
__global__ void __launch_bounds__(128)
ar_fork_prefix_kernel(KvCache cache, int64_t layer_stride, const int32_t *__restrict__ slots,
                      const int32_t *__restrict__ kv_parent, KvRows rows) {
  const int b = slots[blockIdx.x], l = blockIdx.y, h = blockIdx.z;
  int par;
  const int lo = kv_shared_rows(kv_parent, rows, b, par);
  if (par == b) return;
  const int hi = min(rows.text_len[b] + rows.prompt_len[b], cache.cap);
  if (hi <= lo) return;
  const int vec_row = 64 * cache.elem / 16;      // 16-byte vectors per cached row
  const int n = (hi - lo) * vec_row;             // of one stream
  const int64_t layer = (int64_t)l * layer_stride;
  const int64_t dst = (layer + cache.row(b, h, lo)) * cache.elem / 16, src = (layer + cache.row(par, h, lo)) * cache.elem / 16;
  for (int t = threadIdx.x; t < 2 * n; t += blockDim.x) {
    uint4 *base = reinterpret_cast<uint4 *>(t < n ? cache.k : cache.v);
    const int j = t < n ? t : t - n;
    base[dst + j] = base[src + j];
  }
}

int launch_ar_fork_prefix(const vb_ar_state *st, int n_layer, int n_head, int elem, const int32_t *slots, int k,
                          cudaStream_t s) {
  const KvCache cache{st->kcache, st->vcache, nullptr, nullptr, st->cache_seq_stride, st->cache_cap, elem};
  const KvRows rows{st->text_len, st->prompt_len, st->n_gen, st->finished};
  ar_fork_prefix_kernel<<<dim3(k, n_layer, n_head), 128, 0, s>>>(cache, st->cache_layer_stride, slots, st->kv_parent,
                                                                 rows);
  VB_LAUNCH_CHECK();
  return VB_OK;
}

__global__ void __launch_bounds__(256)
sample_logits_kernel(const float *__restrict__ logits, int64_t ld, int n_vocab, SamplerArgs sa,
                     const int32_t *__restrict__ steps, const int32_t *__restrict__ tokens, int64_t tok_ld,
                     int64_t *__restrict__ out_ids) {
  __shared__ SamplerSmem sm;
  const int64_t r = blockIdx.x;
  const int tid = threadIdx.x;
  const float *row = logits + r * ld;
  float l[5];
  ArgMax best{-CUDART_INF_F, 0x7fffffff};
#pragma unroll
  for (int j = 0; j < 5; ++j) {
    const int i = tid + j * 256;
    l[j] = i < n_vocab ? row[i] : -CUDART_INF_F;
    if (i < n_vocab) best = better(best, ArgMax{l[j], i});
  }
  best = block_argmax(best, sm.wbest);
  __syncthreads();  // sm.wbest is reused by the draw
  const int id = sample_row(l, n_vocab, best.i, row_sampler(sa, r, steps[r], tokens + r * tok_ld), sm);
  if (tid == 0) out_ids[r] = id;
}

__global__ void nar_argmax_accumulate_kernel(const float *__restrict__ logits, int64_t n_rows, int n_vocab,
                                             int64_t ld_logits, int64_t *__restrict__ codes,
                                             int64_t code_row_stride, const float *__restrict__ next_emb,
                                             float *__restrict__ y_emb, int64_t y_row_stride,
                                             const int32_t *__restrict__ y_rows, int d) {
  const int64_t r = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (r >= n_rows) return;
  const int lane = threadIdx.x & 31;
  const float *row = logits + r * ld_logits;
  ArgMax best{-CUDART_INF_F, 0x7fffffff};
  for (int i = lane; i < n_vocab; i += 32) best = better(best, ArgMax{row[i], i});
  best = warp_argmax(best);
  if (lane == 0) codes[r * code_row_stride] = best.i;
  if (next_emb != nullptr) {
    const float *e = next_emb + (int64_t)best.i * d;
    float *y = y_emb + (y_rows ? (int64_t)y_rows[r] : r) * y_row_stride;
    for (int c = lane * 4; c < d; c += 128) {
      float4 yv = *reinterpret_cast<float4 *>(y + c);
      const float4 ev = *reinterpret_cast<const float4 *>(e + c);
      yv.x = __fadd_rn(yv.x, ev.x);
      yv.y = __fadd_rn(yv.y, ev.y);
      yv.z = __fadd_rn(yv.z, ev.z);
      yv.w = __fadd_rn(yv.w, ev.w);
      *reinterpret_cast<float4 *>(y + c) = yv;
    }
  }
}

}  // namespace vb

using namespace vb;

VB_API int vb_nar_argmax_accumulate(const float *logits, int64_t n_rows, int n_vocab, int64_t ld_logits,
                                        int64_t *codes, int64_t code_row_stride, const float *next_emb,
                                        float *y_emb, int64_t y_row_stride, const int32_t *y_rows, int d,
                                        vb_stream_t stream) {
  VB_CHECK_ARG(d % 4 == 0, "vb_nar_argmax_accumulate: d %% 4 != 0");
  if (n_rows == 0) return VB_OK;
  const int wpb = 4;
  nar_argmax_accumulate_kernel<<<(unsigned)((n_rows + wpb - 1) / wpb), wpb * 32, 0, (cudaStream_t)stream>>>(
      logits, n_rows, n_vocab, ld_logits, codes, code_row_stride, next_emb, y_emb, y_row_stride, y_rows, d);
  VB_LAUNCH_CHECK();
  return VB_OK;
}

VB_API int vb_sample_logits(const float *logits, int64_t ld, int64_t n_rows, int n_vocab, const uint64_t *seeds,
                            const int32_t *steps, const int32_t *top_k, const float *temperature, int64_t *out_ids,
                            vb_stream_t stream) {
  return vb_sample_logits_ex(logits, ld, n_rows, n_vocab, seeds, steps, top_k, temperature, nullptr, nullptr, nullptr,
                             nullptr, 0, out_ids, stream);
}

namespace {
// copies n device values to the host (on `s`, waiting for them) to check the per-row sampler parameters
template <class T>
int fetch_rows(const T *dev, int64_t n, std::vector<T> &host, cudaStream_t s) {
  host.resize((size_t)n);
  VB_CUDA(cudaMemcpyAsync(host.data(), dev, (size_t)n * sizeof(T), cudaMemcpyDeviceToHost, s));
  VB_CUDA(cudaStreamSynchronize(s));
  return VB_OK;
}
}  // namespace

VB_API int vb_sample_logits_ex(const float *logits, int64_t ld, int64_t n_rows, int n_vocab, const uint64_t *seeds,
                               const int32_t *steps, const int32_t *top_k, const float *temperature,
                               const float *top_p, const int32_t *ras_window, const int32_t *ras_max,
                               const int32_t *tokens, int64_t tok_ld, int64_t *out_ids, vb_stream_t stream) {
  VB_CHECK_ARG(n_vocab >= 1 && n_vocab <= 5 * 256, "vb_sample_logits: n_vocab %d not in [1, 1280]", n_vocab);
  VB_CHECK_ARG(n_rows >= 0 && n_rows < (1ll << 31), "vb_sample_logits: n_rows out of range");
  if (n_rows == 0) return VB_OK;
  VB_CHECK_ARG(logits && seeds && steps && top_k && temperature && out_ids, "vb_sample_logits: null argument");
  VB_CHECK_ARG(!ras_window || (ras_max && tokens), "vb_sample_logits_ex: ras_window needs ras_max and tokens");
  cudaStream_t s = (cudaStream_t)stream;
  if (top_p) {
    std::vector<float> p;
    VB_TRY(fetch_rows(top_p, n_rows, p, s));
    for (int64_t r = 0; r < n_rows; ++r)
      VB_CHECK_ARG(p[r] > 0.f && p[r] <= 1.f, "vb_sample_logits_ex: top_p[%lld] = %g not in (0, 1]", (long long)r,
                   (double)p[r]);
  }
  if (ras_window) {
    std::vector<int32_t> w, mx;
    VB_TRY(fetch_rows(ras_window, n_rows, w, s));
    VB_TRY(fetch_rows(ras_max, n_rows, mx, s));
    for (int64_t r = 0; r < n_rows; ++r) {
      VB_CHECK_ARG(w[r] >= 0 && w[r] <= 256, "vb_sample_logits_ex: ras_window[%lld] = %d not in [0, 256]",
                   (long long)r, w[r]);
      VB_CHECK_ARG(mx[r] >= 0, "vb_sample_logits_ex: ras_max[%lld] = %d < 0", (long long)r, mx[r]);
    }
  }
  sample_logits_kernel<<<(unsigned)n_rows, 256, 0, s>>>(
      logits, ld, n_vocab, SamplerArgs{seeds, top_k, temperature, top_p, ras_window, ras_max}, steps, tokens, tok_ld,
      out_ids);
  VB_LAUNCH_CHECK();
  return VB_OK;
}

// F.cross_entropy per row (valle/models/valle.py:877,936-941): loss[r] = logsumexp(logits[r,:]) -
// logits[r, target[r]]; rows whose target == ignore_index contribute 0.  One warp per row, fp32.
namespace vb {
__global__ void cross_entropy_kernel(const float *__restrict__ logits, int64_t ld, const int64_t *__restrict__ targets,
                                     int64_t n_rows, int n_vocab, int64_t ignore_index, float *__restrict__ loss) {
  const int64_t r = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (r >= n_rows) return;
  const int lane = threadIdx.x & 31;
  const float *row = logits + r * ld;
  const int64_t tg = targets[r];
  float mx = -CUDART_INF_F;
  for (int i = lane; i < n_vocab; i += 32) mx = fmaxf(mx, row[i]);
  mx = warp_max(mx);
  float s = 0.f;
  for (int i = lane; i < n_vocab; i += 32) s += expf(row[i] - mx);
  s = warp_sum(s);
  if (lane == 0) loss[r] = (tg == ignore_index || tg < 0 || tg >= n_vocab) ? 0.f : (logf(s) + mx - row[tg]);
}
}  // namespace vb

VB_API int vb_cross_entropy(const float *logits, int64_t ld_logits, const int64_t *targets, int64_t n_rows,
                            int n_vocab, int64_t ignore_index, float *loss, vb_stream_t stream) {
  if (n_rows == 0) return VB_OK;
  const int wpb = 4;
  vb::cross_entropy_kernel<<<(unsigned)((n_rows + wpb - 1) / wpb), wpb * 32, 0, (cudaStream_t)stream>>>(
      logits, ld_logits, targets, n_rows, n_vocab, ignore_index, loss);
  VB_LAUNCH_CHECK();
  return VB_OK;
}
