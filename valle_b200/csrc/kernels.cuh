// Internal launcher declarations shared by the translation units of libvalle_b200.so.
#pragma once
#include "common.cuh"

namespace vb {

// Training-mode dropout (valle/modules/transformer.py:329,333-334, activation.py attention dropout, embedding.py:97):
// a stateless Bernoulli mask keyed by (seed of the forward call, stream id of the site, element index), so the backward
// pass regenerates the mask of the forward pass instead of storing it.  splitmix64 finaliser; keep <=> hash >= thresh
// with thresh = p * 2^32.  tests/test_backward_gpu.py holds the same function in numpy.
struct DropCfg {
  uint64_t seed;
  uint32_t stream;     // site id: (layer << 2) | {0 attention probabilities, 1 after out-proj, 2 FFN hidden, 3 after FFN}
  uint32_t thresh;     // 0 = dropout off
  float inv_keep;      // 1 / (1 - p)
  int64_t lmax;        // attention only: index = ((b * H + h) * lmax + q) * lmax + k
};
// Counter-based hash of (seed, stream, index): splitmix64 finaliser over seed + stream * C1 + index * C2.  Shared by
// the dropout masks and the device sampler (sample.cu); tests restate it in numpy.
__host__ __device__ __forceinline__ uint64_t mix64(uint64_t seed, uint64_t stream, uint64_t idx) {
  uint64_t z = seed + stream * 0x9E3779B97F4A7C15ull + idx * 0xD1342543DE82EF95ull;
  z ^= z >> 30;
  z *= 0xBF58476D1CE4E5B9ull;
  z ^= z >> 27;
  z *= 0x94D049BB133111EBull;
  z ^= z >> 31;
  return z;
}
__host__ __device__ __forceinline__ bool drop_keep(const DropCfg &c, uint64_t idx) {
  return (uint32_t)(mix64(c.seed, (uint64_t)c.stream, idx) >> 32) >= c.thresh;
}
inline DropCfg make_drop(float p, uint64_t seed, uint32_t stream, int64_t lmax = 0) {
  DropCfg c{};
  if (p > 0.f) {
    c.seed = seed;
    c.stream = stream;
    const double t = (double)p * 4294967296.0;
    c.thresh = t >= 4294967295.0 ? 0xFFFFFFFFu : (uint32_t)t;
    c.inv_keep = 1.f / (1.f - p);
    c.lmax = lmax;
  }
  return c;
}

// Visibility rule of one query row: key c is seen iff c < lim0 or s1 <= c < hi1.
struct RowMask {
  int lim0, s1, hi1;
  __device__ __forceinline__ bool ok(int c) const { return c < lim0 || (c >= s1 && c < hi1); }
};
// A batch of packed ragged sequences and the attention mask over them (vb_mask_mode VB_MASK_FULL .. VB_MASK_PADDED).
// Sequence b is rows [r0, r0 + L) of the packed [M, .] matrices, r0 = cu_seqlens[b], L = cu_seqlens[b + 1] - r0 <=
// max_seqlen; its rows and keys are counted from 0.  S = text_lens[b] is read in every mode but FULL, c1 = seg1_lens[b]
// in the padded modes (a padded sequence is [text padded to seg1_start | audio padded]).  Query row qr < L sees key c
// iff c < lim0 or s1 <= c < hi1, with
//   FULL       lim0 = L                        (NAR: the whole sequence)
//   VALLE_AR   lim0 = max(S, qr + 1)           (AR inference: all text, causal audio)
//   PADDED_AR  lim0 = S; s1 = seg1_start, hi1 = seg1_start + clamp(qr - seg1_start + 1, 0, c1)
//                                              (AR training: text, and the audio causally)
//   PADDED     lim0 = S; s1 = seg1_start, hi1 = seg1_start + c1
//                                              (NAR training: key padding only)
// and a row qr >= L sees nothing.  A prefill that fills a KV cache writes sequence b's rows into the cache's stream
// cache_seq(b): cache_slot[b] when a slot map is given (continuous batching refills one slot of a running batch),
// else b.
struct Packed {
  const int32_t *cu_seqlens, *text_lens, *seg1_lens;
  int B, max_seqlen, seg1_start, mask_mode;
  const int32_t *cache_slot = nullptr;
  struct Seq {
    int r0, L, S, c1;
  };
  // read-only loads (ld.global.nc): no kernel writes the length arrays
  __device__ __forceinline__ Seq seq(int b) const {
    Seq q;
    q.r0 = __ldg(cu_seqlens + b);
    q.L = __ldg(cu_seqlens + b + 1) - q.r0;
    q.S = mask_mode != VB_MASK_FULL ? __ldg(text_lens + b) : 0;
    q.c1 = mask_mode >= VB_MASK_PADDED_AR ? __ldg(seg1_lens + b) : 0;
    return q;
  }
  __device__ __forceinline__ RowMask row_mask(const Seq &q, int qr) const {
    RowMask m{0, 0, 0};
    if (qr >= q.L) return m;
    if (mask_mode == VB_MASK_FULL) {
      m.lim0 = q.L; m.s1 = q.L; m.hi1 = q.L;
    } else if (mask_mode == VB_MASK_VALLE_AR) {
      m.lim0 = max(q.S, qr + 1); m.s1 = q.L; m.hi1 = q.L;
    } else if (mask_mode == VB_MASK_PADDED_AR) {
      m.lim0 = q.S; m.s1 = seg1_start;
      m.hi1 = qr >= seg1_start ? seg1_start + min(q.c1, qr - seg1_start + 1) : seg1_start;
    } else {  // VB_MASK_PADDED
      m.lim0 = q.S; m.s1 = seg1_start; m.hi1 = seg1_start + q.c1;
    }
    return m;
  }
  // keys [0, kv_max) hold every key that the query rows below q_hi (<= L) see
  __device__ __forceinline__ int kv_max(const Seq &q, int q_hi) const {
    return mask_mode == VB_MASK_VALLE_AR ? max(q.S, q_hi) : q.L;
  }
  __device__ __forceinline__ int cache_seq(int b) const { return cache_slot ? __ldg(cache_slot + b) : b; }
};
// the mask mode, and the length arrays it reads (fn: the caller, for the message)
inline int check_packed(const Packed &p, const char *fn) {
  VB_CHECK_ARG(p.mask_mode >= VB_MASK_FULL && p.mask_mode <= VB_MASK_PADDED, "%s: bad mask mode %d", fn, p.mask_mode);
  VB_CHECK_ARG(p.mask_mode == VB_MASK_FULL || p.text_lens != nullptr, "%s: this mask mode needs text_lens", fn);
  VB_CHECK_ARG(p.mask_mode < VB_MASK_PADDED_AR || p.seg1_lens != nullptr, "%s: padded mask modes need seg1_lens", fn);
  return VB_OK;
}

// bytes per element of a VB_* dtype
inline size_t elem_size(int dtype) { return dtype == VB_E4M3 ? 1 : dtype == VB_BF16 ? 2 : 4; }

// The KV cache of the AR decoder, seen one layer at a time.  The whole cache is two arrays, K and V, of
// [n_layer, B, H, cap, 64] rows (one row = one token's key or value of one head): layer l starts l * layer_stride
// elements in, utterance b of a layer b * seq_stride elements in, and the cap rows of one (utterance, head) stream are
// contiguous.  The elements are fp32, bf16 (the decoder's dtype) or, for the FP8 cache, e4m3 bytes; an FP8 row has one
// exponent byte e + 127 as well and reads back as e4m3 * 2^e (kv8_* in common.cuh), and the exponent arrays
// [n_layer, B, H, cap] have the cache's strides divided by 64 (both strides are multiples of 1024 there, so a row's
// element offset is 64 times its exponent index).  Utterance b's stream holds KvRows::count rows, the current
// token's being KvRows::cur.
struct KvCache {
  void *k, *v;            // this layer's K and V rows, or nullptr (no cache)
  uint8_t *kexp, *vexp;   // this layer's exponent bytes (FP8 cache), else nullptr
  int64_t seq_stride;     // elements between utterances
  int cap;                // rows per (utterance, head) stream
  int elem;               // bytes per element
  // element offset of row `pos` of stream (b, h) from k / v
  __host__ __device__ __forceinline__ int64_t row(int b, int h, int pos) const {
    return (int64_t)b * seq_stride + ((int64_t)h * cap + pos) * 64;
  }
  // index of that row's exponent byte in kexp / vexp
  __host__ __device__ __forceinline__ int64_t exp_index(int b, int h, int pos) const {
    return (int64_t)b * (seq_stride / 64) + (int64_t)h * cap + pos;
  }
};
// layer l's view, from the whole cache (the view whose pointers are the arrays' bases) and the elements between
// layers; a null pointer stays null
inline KvCache kv_cache_layer(KvCache c, int64_t layer_stride, int l) {
  const size_t off = (size_t)l * layer_stride * c.elem, eoff = (size_t)l * layer_stride / 64;
  if (c.k) c.k = (char *)c.k + off;
  if (c.v) c.v = (char *)c.v + off;
  if (c.kexp) c.kexp += eoff;
  if (c.vexp) c.vexp += eoff;
  return c;
}
// The rows of each utterance's cache streams during AR decoding (vb_ar_state): text_len[b] + prompt_len[b] + n_gen[b]
// once n_gen[b] tokens are generated, at most cap.  n_gen[b] is an argument: the decode attention reads it twice.
struct KvRows {
  const int32_t *text_len, *prompt_len, *n_gen;
  const int32_t *finished;  // NULL or [B]: rows that have stopped keep their cache untouched
  __device__ __forceinline__ int count(int b, int n_gen_b, int cap) const {
    return min(text_len[b] + prompt_len[b] + n_gen_b, cap);
  }
  // the current token's row, max(count, 1) - 1, written as a clamp: spelled with count, the QKV epilogue of
  // gemv_kernel takes more registers and spills more
  __device__ __forceinline__ int cur(int b, int n_gen_b, int cap) const {
    return max(0, min(text_len[b] + prompt_len[b] + n_gen_b - 1, cap - 1));
  }
};
// Shared prompt prefix of best-of-n decoding (vb_ar_state.kv_parent): row b reads its cache rows below
// P_b = 16 floor((text_len[b] + prompt_len[b]) / 16) from the streams of row parent[b], which holds the same text and
// prompt, and every other row from its own streams.  A row that is its own parent shares nothing (P = 0).  P_b is a
// multiple of 16, as is every KV split boundary; the current token's row is always >= S_b + Tp_b >= P_b, so every write
// goes to the row's own streams.  bf16 and fp32 caches only: on the FP8 cache the shared read was measured slower than
// every row reading its own copy (DESIGN section 7), so vb_ar_decode_step refuses it there.
__device__ __forceinline__ int kv_shared_rows(const int32_t *parent, const KvRows &rows, int b, int &par) {
  par = parent[b];
  return par == b ? 0 : (rows.text_len[b] + rows.prompt_len[b]) & ~15;
}
// Beam search (vb_ar_state.beam_width > 1, or the per-row groups beam_first): the ancestry table the decode attention
// follows.  Row b's generated cache row S_b + Tp_b + t, below its current row, lives in the streams of row
// g_b + anc[b * ld + t], g_b the first row of b's group: b - b % width, or first[b] (-1: b is in no group and reads
// its own streams).
struct BeamAnc {
  const uint8_t *anc = nullptr;  // [B, ld]
  int ld = 0, width = 0;
  const int32_t *first = nullptr;  // [B] or NULL (groups of `width` rows)
};
// The rows of one (utterance, head) stream as a decode kernel reads them: element offset of row `pos` from the
// stream's row 0.  kShared = false: the stream's own rows, nothing else is
// computed.  kShared: rows below `shared` are the parent's, `poff` elements away (the parent's stream minus the own).
// kBeam: every row of the CTA's chunk [c0, c0 + n) comes from the stream `dl[pos - c0]` rows away, a table the CTA
// stages in shared memory once (stage_beam) from the prefix parent (when kv_parent is set) and the ancestry.
template <bool kShared, bool kBeam = false>
struct KvStreamRows {
  int64_t poff = 0;
  int shared = 0;
  const int16_t *dl = nullptr;
  int c0 = 0;
  int64_t stride = 0;
  __device__ __forceinline__ KvStreamRows() {}
  __device__ __forceinline__ KvStreamRows(const int32_t *parent, const KvRows &rows, const KvCache &kv, int b) {
    if constexpr (kBeam) {
      stride = kv.seq_stride;
    } else if constexpr (kShared) {
      int par;
      shared = kv_shared_rows(parent, rows, b, par);
      poff = (int64_t)(par - b) * kv.seq_stride;
    }
  }
  // kBeam: row deltas of the chunk [c0, c0 + n) of row b, whose current row is `cur`, into dl_s (shared memory, n
  // entries), by every thread of the CTA; the caller synchronises the CTA before the first row() call
  __device__ __forceinline__ void stage_beam(int16_t *dl_s, const int32_t *parent, const KvRows &rows,
                                             const BeamAnc &ba, int b, int c0_, int n, int cur) {
    const int gen0 = rows.text_len[b] + rows.prompt_len[b];
    int pre = 0, pd = 0;
    if (parent != nullptr) {
      int par;
      pre = kv_shared_rows(parent, rows, b, par);
      pd = par - b;
    }
    const int g0 = ba.first != nullptr ? ba.first[b] : b - b % ba.width;
    const int jb = b - g0;
    const int gen_end = g0 >= 0 ? cur : gen0;   // a row in no group: no generated row comes from elsewhere
    const uint8_t *a = ba.anc + (int64_t)b * ba.ld;
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
      const int p = c0_ + i;
      dl_s[i] = (int16_t)(p < pre ? pd : (p >= gen0 && p < gen_end) ? (int)a[p - gen0] - jb : 0);
    }
    dl = dl_s;
    c0 = c0_;
  }
  __device__ __forceinline__ int64_t row(int pos) const {
    if constexpr (kBeam) return (int64_t)pos * 64 + (int64_t)dl[pos - c0] * stride;
    else if constexpr (kShared) return (int64_t)pos * 64 + (pos < shared ? poff : 0);
    else return (int64_t)pos * 64;
  }
};

// L2 prefetch of a slice of an upcoming layer's K and V cache, issued by the otherwise idle warps of the
// split-K decode projections (gemm_decode.cu) while their weight tiles stream: the projection chain is latency
// bound and leaves HBM mostly idle, the KV-cache attention that follows is HBM bound -- rows [row_lo, row_hi) of
// every (utterance, head) stream (the leading rows, where every CTA of the attention starts) are pulled into L2
// ahead of it.  Only a hint: the lengths may be one step stale (read before the dependency wait),
// which changes what is prefetched, never what is computed.  A row whose parent (kv_parent) is another row skips the
// shared rows: its parent's streams hold them and its parent fetches them.
struct KvPrefetch {
  KvCache kv;   // the target layer (kv.k == nullptr: nothing to prefetch)
  KvRows rows;
  int B, H;
  int row_lo, row_hi;
  const int32_t *kv_parent = nullptr;   // vb_ar_state.kv_parent, or nullptr
};
// worker = one warp; `n_workers` warps of the grid share the streams.  Lane i of a warp fetches the lengths of the
// warp's i-th stream up front (the three dependent global loads per stream would otherwise serialise the loop).
__device__ __forceinline__ void kv_prefetch(const KvPrefetch &pf, int worker, int n_workers) {
  if (pf.kv.k == nullptr) return;
  const int lane = threadIdx.x & 31;
  const int n_streams = 2 * pf.B * pf.H;
  int kv_mine = 0;
  {
    const int s_mine = worker + lane * n_workers;
    if (s_mine < n_streams) {
      const int b = (s_mine >> 1) / pf.H;
      kv_mine = pf.rows.count(b, pf.rows.n_gen[b], pf.kv.cap);
    }
  }
  const int row_bytes = 64 * pf.kv.elem;
  for (int i = 0, sidx = worker; sidx < n_streams; ++i, sidx += n_workers) {
    int kv;
    if (i < 32) {
      kv = __shfl_sync(0xffffffffu, kv_mine, i);
    } else {
      const int b = (sidx >> 1) / pf.H;
      kv = pf.rows.count(b, pf.rows.n_gen[b], pf.kv.cap);
    }
    const int pair = sidx >> 1;
    const int b = pair / pf.H, h = pair - b * pf.H;
    int lo = pf.row_lo;
    if (pf.kv_parent != nullptr) {
      int par;
      lo = max(lo, kv_shared_rows(pf.kv_parent, pf.rows, b, par));
    }
    const int r_lo = min(kv, lo), r_hi = min(kv, pf.row_hi);
    const char *p = (const char *)((sidx & 1) ? pf.kv.v : pf.kv.k) + pf.kv.row(b, h, r_lo) * pf.kv.elem;
    const int lines = ((r_hi - r_lo) * row_bytes) >> 7;  // 128-byte lines
    for (int l = lane; l < lines; l += 32) asm volatile("prefetch.global.L2 [%0];" ::"l"(p + ((int64_t)l << 7)));
    if (pf.kv.kexp != nullptr && lane == 0 && r_hi > r_lo) {  // the rows' exponent bytes: one or two lines
      const char *e = (const char *)((sidx & 1) ? pf.kv.vexp : pf.kv.kexp) + pf.kv.exp_index(b, h, 0);
      const int64_t l0 = (r_lo + ((int64_t)(uintptr_t)e & 127)) >> 7, l1 = (r_hi - 1 + ((int64_t)(uintptr_t)e & 127)) >> 7;
      const char *e0 = (const char *)((uintptr_t)e & ~(uintptr_t)127);
      for (int64_t l = l0; l <= l1; ++l) asm volatile("prefetch.global.L2 [%0];" ::"l"(e0 + (l << 7)));
    }
  }
}

struct LnParams {
  const float *gamma, *beta, *ada_wb;  // ada_wb: NULL or [2d] (weight | bias)
  float eps;
};

// The QKV projection of a decode step: q of the current token to q, its k and v appended to the layer's cache
struct QkvScatter {
  int d, head_dim;
  float *q;  // [B, d] fp32
  KvCache kv;
  KvRows rows;
};

// gemm_simt.cu
int launch_gemm_simt(const void *A, int a_dtype, int64_t lda, const void *W, const float *bias, void *C,
                     int c_dtype, int64_t ldc, int64_t M, int N, int K, int epi, cudaStream_t s);
int launch_gemv(const float *x, int64_t ldx, int B, const void *W, int w_dtype, const float *bias,
                int N, int K, float *out, int64_t ldo, const LnParams *ln, int epi_mode,
                const QkvScatter *qkv, cudaStream_t s);

// gemm_wgmma.cu
bool wgmma_gemm_supported(int64_t M, int N, int K, int64_t lda, int64_t ldc);
int launch_gemm_wgmma(const bf16 *A, int64_t lda, const bf16 *W, const float *bias, void *C,
                      int c_dtype, int64_t ldc, int64_t M, int N, int K, int epi, cudaStream_t s);

// gemm_decode.cu (swap-AB split-K wgmma projections for B <= 64 decode rows, bf16)
enum { DG_F32 = 0, DG_RESIDUAL = 1, DG_RELU_BF16 = 2, DG_QKV = 3 };
constexpr int kMaxForcedSplits = 16;  // cap of a caller-chosen split-K count (sizes the partial workspace)
size_t gemm_decode_workspace(int d_model, int d_ff);
// LayerNorm folded into the projection (decode chain without the residual + LayerNorm launches):
//   moments of the fp32 rows, stats[split][64][2] = (sum x, sum x^2) over the split's k-range, next to the partials
struct LnFoldStats {
  const float *stats;  // NULL: the partials are plain (no folded LayerNorm)
  const float *c;      // [N]  sum_k wf[n,k]
  int splits, d;       // splits of the producing projection, LayerNorm width
  float eps;
  int copies;          // every tile row of the producing grid stores its own copy of the moments:
                       // stats[copy][split][64][2]; consumers spread over the copies (no L2 hot spot)
};
constexpr int kLnFoldMaxCopies = 32;
// Called by every lane of a (converged) warp whose threads share the row b: lane s fetches split s's pair, the warp
// adds them up by shuffles -- ONE L2 round trip.  (A per-thread loop over the splits, however it is unrolled, ends up
// as `splits` dependent round trips under the register caps of the consumer kernels.)
__device__ __forceinline__ float2 ln_fold_moments_load(const LnFoldStats &f, int b, int which) {
  const int lane = threadIdx.x & 31;
  const float *st = f.stats + (int64_t)(which % f.copies) * f.splits * 64 * 2;
  float2 m = make_float2(0.f, 0.f);
  if (lane < f.splits) m = __ldcg(reinterpret_cast<const float2 *>(st + ((int64_t)lane * 64 + b) * 2));
  return m;
}
__device__ __forceinline__ void ln_fold_moments_finish(const LnFoldStats &f, float2 m, float &mean, float &rstd) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    m.x += __shfl_xor_sync(0xffffffffu, m.x, o);
    m.y += __shfl_xor_sync(0xffffffffu, m.y, o);
  }
  mean = m.x / (float)f.d;
  rstd = rsqrtf(fmaxf(m.y / (float)f.d - mean * mean, 0.f) + f.eps);
}
__device__ __forceinline__ void ln_fold_moments(const LnFoldStats &f, int b, int which, float &mean, float &rstd) {
  ln_fold_moments_finish(f, ln_fold_moments_load(f, b, which), mean, rstd);
}
// What a decode projection hands to the kernel that consumes it: fp32 partial tiles [splits][64][ldp] for the
// consumer to add up in fixed order 0..splits-1, then `bias`; with a folded LayerNorm (fold.stats != NULL) the rows'
// moments as well, and `bias` is the folded bias.  part == NULL: nothing is pending, the projection applied its own
// epilogue (one split, the QKV scatter, the in-cluster residual update).
struct SplitK {
  const float *part = nullptr;
  int splits = 0, ldp = 0;
  const float *bias = nullptr;
  LnFoldStats fold{};
};
// out receives the hand-over: the partials when the projection leaves any, and its bias
int launch_gemm_decode(const bf16 *act, int B, int64_t ld_act, const bf16 *W, int N, int K, int force_splits,
                       const float *bias, int mode, float *out_f32, bf16 *out_bf16, int64_t ld_out,
                       const QkvScatter *qkv, float *partials, size_t partial_bytes, SplitK *out,
                       const KvPrefetch *pf, bool pdl, cudaStream_t s, bool red_add = false);
// projection of the fp32 rows by the weights of F (vb_ln_fold): out receives the partials, F's c and folded bias, and
// the moments the kernel leaves in stats
int launch_gemm_decode_x(const float *x, int B, int64_t ldx, const vb_ln_fold &F, int N, int K, int force_splits,
                         float *partials, size_t partial_bytes, float *stats, SplitK *out, const KvPrefetch *pf,
                         bool pdl, cudaStream_t s);
int launch_ln_fold(const bf16 *W, int N, int K, const float *gamma, const float *beta, const float *bias, bf16 *wf,
                   float *c, float *dvec, cudaStream_t s);

// attention.cu
// fills the layer's KV cache `kv` when kv.k != nullptr (kv.kexp != nullptr: the FP8 cache)
// pk.mask_mode may also be VB_MASK_DENSE, with the byte mask dense_mask
int launch_attention_varlen(const void *qkv, int dtype, int64_t M, int n_head, int head_dim, const Packed &pk,
                            void *out, const KvCache &kv, const uint8_t *dense_mask, int64_t dense_ld, cudaStream_t s,
                            const DropCfg *drop = nullptr);
// attention_wgmma.cu (bf16 flash attention on wgmma / TMA; fills the KV cache when kv.k != nullptr: bf16, or with
// kv.kexp != nullptr the FP8 cache, e4m3 rows + exponent bytes)
int launch_attention_wgmma(const bf16 *qkv, int64_t M, int n_head, const Packed &pk, bf16 *out, const KvCache &kv,
                           cudaStream_t s);
size_t attn_decode_workspace(int B, int n_head, int head_dim, int cache_cap);
// the current token's q, k, v (kv.q, or pending in qkv) against the layer's cache kv.kv.  dtype VB_E4M3: the FP8
// cache; q, k, v must then be pending in qkv.  kv_parent: vb_ar_state.kv_parent (NULL: every row reads its own streams)
// beam.anc != NULL: the generated rows follow the beam ancestry (bf16 and fp32 caches)
int launch_attn_decode(const QkvScatter &kv, const SplitK &qkv, int B, int n_head, int dtype, float *out, void *out16,
                       void *workspace, bool pdl, cudaStream_t s, const int32_t *kv_parent, const BeamAnc &beam);

// decode_fused.cu
int launch_relu_reduce(const SplitK &in, int B, int N, bf16 *out16, int64_t ldo, bool pdl, cudaStream_t s);
// post = true: the post-norm of a post-LN layer, x[b,:] = LayerNorm(x[b,:] + bias + partials) (normalised in place)
int launch_ln_reduce(float *x, int64_t ldx, int B, int d, const SplitK &in, const float *gamma, const float *beta,
                     float eps, bf16 *out16, bool pdl, cudaStream_t s, bool post = false);

// embed_norm.cu: the post-norm of a post-LN layer over the rows x[n_rows, d] (fp32, dense): x = LayerNorm(x) (AdaLN with
// ada_wb != NULL) in place, and the same rows in out_dtype into `out` (may be NULL)
int launch_post_norm(float *x, int64_t n_rows, int d, const float *gamma, const float *beta, const float *ada_wb,
                     float eps, void *out, int out_dtype, cudaStream_t s);

// backward.cu
int launch_transpose_pad(const void *in, int dtype, int64_t ld_in, int64_t R, int C, void *out, int64_t ld_out,
                         cudaStream_t s);
int launch_colsum(const void *in, int dtype, int64_t ld, int64_t R, int N, float *out, cudaStream_t s);
int launch_relu_bwd(void *dh, const void *h, int dtype, int64_t n, float scale, cudaStream_t s);
int attention_backward(const void *qkv, const void *out, const void *dout, int dtype, int64_t M, int n_head,
                       int head_dim, const Packed &pk, void *dqkv, void *workspace, size_t workspace_bytes,
                       const DropCfg *drop, cudaStream_t s);
// out[i] = keep(i) ? in[i] / (1 - p) : 0 (in place allowed); x[i] += keep(i) ? t[i] / (1 - p) : 0
int launch_dropout(const void *in, void *out, int dtype, int64_t n, const DropCfg &cfg, cudaStream_t s);
int launch_dropout_add(float *x, const float *t, int64_t n, const DropCfg &cfg, cudaStream_t s);
int launch_cast_from_f32(const float *in, void *out, int dtype, int64_t n, cudaStream_t s);

// sample.cu
// head->greedy == 2 (and neither `forced` nor `reduce_only`) launches the seeded device sampler, which reads
// st->sample_seed / top_k / temperature; every other call the argmax / push / reduce kernel
// in: the head projection's pending partials (in.part == NULL: the logits are complete)
int launch_ar_sample(float *logits, int64_t ld_logits, const SplitK &in, const vb_ar_head *head, vb_ar_state *st,
                     int d, const int64_t *forced, int reduce_only, bool pdl, cudaStream_t s);
// head->greedy == 3: one beam-search step (include/valle_b200.h "Beam search") over the complete logits st->logits,
// one CTA per group of st->beam_width rows; lse: NULL or [B], each row's log-sum-exp (vb_ar_beam_step)
int launch_beam_tail(const vb_ar_head *head, vb_ar_state *st, int d, bool pdl, cudaStream_t s, float *lse = nullptr);
// vb_ar_admit: row i of the k-row state cs <-> row slots[i] of the running state st.  Gather (scatter = false): the
// lengths and sampler parameters into cs, n_gen / finished / tokens of cs zeroed.  Scatter: n_gen, finished,
// tokens[., 0], x_cur and logits[., 0:n_vocab] back into the slots; with cs->logprob, logprob too (zeroed by the gather)
int launch_ar_admit_copy(vb_ar_state *st, const vb_ar_state *cs, const int32_t *slots, int d, int ldl, int n_vocab,
                         bool scatter, cudaStream_t s);
// vb_ar_fork_prefix on a bf16 / fp32 cache of `elem`-byte elements: the k rows slots[i] whose kv_parent is another row
// copy their cache rows [P, S + Tp) of every layer and head, K and V, from the parent's streams
int launch_ar_fork_prefix(const vb_ar_state *st, int n_layer, int n_head, int elem, const int32_t *slots, int k,
                          cudaStream_t s);

}  // namespace vb
