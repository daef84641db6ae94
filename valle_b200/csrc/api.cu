// C-ABI entry points and host-side orchestration (layer loops) of libvalle_b200.so.
// See include/valle_b200.h for the contract of every function.
#include <stdarg.h>
#include <string.h>

#include <new>

#include <algorithm>
#include <vector>

#include "common.cuh"
#include "kernels.cuh"

namespace vb {

static thread_local char g_err[1024] = "";
static int64_t g_launches = 0;  // process-wide counter (relaxed; bench reads it when idle)

void set_error(const char *fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
void count_launch() { __atomic_fetch_add(&g_launches, 1, __ATOMIC_RELAXED); }

// Tuning knobs: vb_tune_set() overrides > environment variable of the same name > built-in default.  Read at
// launch time (a captured CUDA graph keeps the values it was captured with).
namespace {
struct TuneEntry {
  char name[48];
  int value;
};
TuneEntry g_tune[32];
int g_n_tune = 0;
}  // namespace
int tune(const char *name, int dflt) {
  for (int i = 0; i < g_n_tune; ++i)
    if (strcmp(g_tune[i].name, name) == 0) return g_tune[i].value;
  const char *e = getenv(name);
  return e ? atoi(e) : dflt;
}

#ifdef VB_TRACE
static trace_bind_fn g_trace_binders[32];
static int g_n_trace_binders = 0;
void trace_register(trace_bind_fn f) {
  if (g_n_trace_binders < 32) g_trace_binders[g_n_trace_binders++] = f;
}
#endif

}  // namespace vb

using namespace vb;

struct vb_decoder {
  vb_decoder_desc desc;
  vb_layer_params *layers;  // owned host copy
  vb_ln_fold *fold_qkv = nullptr, *fold_ffn1 = nullptr;  // owned host copies [n_layer] or NULL (vb_decoder_set_decode_fold)
};

VB_API int vb_abi_version(void) { return VB_ABI_VERSION; }
VB_API const char *vb_last_error(void) { return g_err; }
VB_API int64_t vb_launch_count(void) { return __atomic_load_n(&g_launches, __ATOMIC_RELAXED); }

VB_API int vb_tune_set(const char *name, int value) {
  VB_CHECK_ARG(name && strlen(name) < sizeof(g_tune[0].name), "vb_tune_set: bad name");
  for (int i = 0; i < g_n_tune; ++i)
    if (strcmp(g_tune[i].name, name) == 0) {
      g_tune[i].value = value;
      return VB_OK;
    }
  VB_CHECK_ARG(g_n_tune < 32, "vb_tune_set: table full");
  strcpy(g_tune[g_n_tune].name, name);
  g_tune[g_n_tune++].value = value;
  return VB_OK;
}

VB_API int vb_trace_bind(unsigned long long *buf, unsigned int *counter, unsigned int cap) {
#ifdef VB_TRACE
  for (int i = 0; i < g_n_trace_binders; ++i)
    if (g_trace_binders[i](buf, counter, cap) != 0) {
      set_error("vb_trace_bind: cudaMemcpyToSymbol failed");
      return VB_ERR_CUDA;
    }
  return VB_OK;
#else
  (void)buf; (void)counter; (void)cap;
  set_error("vb_trace_bind: not a profiling build (compile with -DVB_TRACE: python -m valle_b200.build --trace)");
  return VB_ERR_UNSUPPORTED;
#endif
}

VB_API int vb_linear(const void *A, int a_dtype, int64_t lda, const void *W, int w_dtype,
                         const float *bias, void *C, int c_dtype, int64_t ldc, int64_t M, int N, int K,
                         int epilogue, void *workspace, size_t workspace_bytes, vb_stream_t stream) {
  (void)workspace;
  (void)workspace_bytes;
  VB_CHECK_ARG(a_dtype == w_dtype, "vb_linear: a_dtype (%d) must equal w_dtype (%d)", a_dtype, w_dtype);
  VB_CHECK_ARG(epilogue >= VB_EPI_NONE && epilogue <= VB_EPI_RESIDUAL, "vb_linear: bad epilogue %d", epilogue);
  VB_CHECK_ARG(M >= 0 && N > 0 && K > 0, "vb_linear: bad shape M=%lld N=%d K=%d", (long long)M, N, K);
  cudaStream_t s = (cudaStream_t)stream;
  if (a_dtype == VB_BF16 && wgmma_gemm_supported(M, N, K, lda, ldc))
    return launch_gemm_wgmma((const bf16 *)A, lda, (const bf16 *)W, bias, C, c_dtype, ldc, M, N, K,
                               epilogue, s);
  return launch_gemm_simt(A, a_dtype, lda, W, bias, C, c_dtype, ldc, M, N, K, epilogue, s);
}

VB_API int vb_decoder_create(const vb_decoder_desc *desc, vb_decoder_t *out) {
  VB_CHECK_ARG(desc && out, "vb_decoder_create: null argument");
  VB_CHECK_ARG(desc->n_layer > 0 && desc->n_head > 0 && desc->d_model % desc->n_head == 0,
               "vb_decoder_create: bad geometry d=%d H=%d L=%d", desc->d_model, desc->n_head, desc->n_layer);
  VB_CHECK_ARG(desc->d_model / desc->n_head == 64, "vb_decoder_create: head_dim must be 64 (got %d)",
               desc->d_model / desc->n_head);
  VB_CHECK_ARG(desc->d_model % 256 == 0 && desc->d_ff % 256 == 0, "vb_decoder_create: d_model and d_ff must be multiples of 256");
  VB_CHECK_ARG(desc->wdtype == VB_F32 || desc->wdtype == VB_BF16, "vb_decoder_create: bad wdtype");
  VB_CHECK_ARG(desc->norm_first == 0 || desc->norm_first == 1, "vb_decoder_create: norm_first=%d not in {0, 1}",
               desc->norm_first);
  VB_CHECK_ARG(!desc->final_norm_w == !desc->final_norm_b, "vb_decoder_create: final_norm_w / final_norm_b: both or neither");
  vb_decoder *d = new (std::nothrow) vb_decoder;
  if (!d) {
    set_error("vb_decoder_create: out of host memory");
    return VB_ERR_ARG;
  }
  d->desc = *desc;
  d->layers = new (std::nothrow) vb_layer_params[desc->n_layer];
  if (!d->layers) {
    delete d;
    set_error("vb_decoder_create: out of host memory");
    return VB_ERR_ARG;
  }
  memcpy(d->layers, desc->layers, sizeof(vb_layer_params) * desc->n_layer);
  d->desc.layers = d->layers;
  *out = d;
  return VB_OK;
}

VB_API void vb_decoder_destroy(vb_decoder_t dec) {
  if (!dec) return;
  delete[] dec->layers;
  delete[] dec->fold_qkv;
  delete[] dec->fold_ffn1;
  delete dec;
}

VB_API int vb_ln_fold_build(const void *W, int N, int K, const float *gamma, const float *beta, const float *bias,
                            void *wf, float *c, float *dvec, vb_stream_t stream) {
  VB_CHECK_ARG(W && gamma && beta && wf && c && dvec && N > 0 && K > 0, "vb_ln_fold_build: null argument / bad shape");
  return launch_ln_fold((const bf16 *)W, N, K, gamma, beta, bias, (bf16 *)wf, c, dvec, (cudaStream_t)stream);
}

VB_API int vb_decoder_set_decode_fold(vb_decoder_t dec, const vb_ln_fold *qkv, const vb_ln_fold *ffn1) {
  VB_CHECK_ARG(dec, "vb_decoder_set_decode_fold: null decoder");
  delete[] dec->fold_qkv;
  delete[] dec->fold_ffn1;
  dec->fold_qkv = dec->fold_ffn1 = nullptr;
  if (!qkv && !ffn1) return VB_OK;
  VB_CHECK_ARG(qkv && ffn1, "vb_decoder_set_decode_fold: both arrays or neither");
  VB_CHECK_ARG(dec->desc.wdtype == VB_BF16, "vb_decoder_set_decode_fold: bf16 decoders only");
  VB_CHECK_ARG(dec->desc.norm_first, "vb_decoder_set_decode_fold: pre-LN decoders only (post-LN norms do not feed a projection)");
  const int n = dec->desc.n_layer;
  for (int l = 0; l < n; ++l)
    VB_CHECK_ARG(qkv[l].wf && qkv[l].c && qkv[l].dvec && ffn1[l].wf && ffn1[l].c && ffn1[l].dvec,
                 "vb_decoder_set_decode_fold: layer %d has a null pointer", l);
  dec->fold_qkv = new (std::nothrow) vb_ln_fold[n];
  dec->fold_ffn1 = new (std::nothrow) vb_ln_fold[n];
  if (!dec->fold_qkv || !dec->fold_ffn1) {
    delete[] dec->fold_qkv;
    delete[] dec->fold_ffn1;
    dec->fold_qkv = dec->fold_ffn1 = nullptr;
    set_error("vb_decoder_set_decode_fold: out of host memory");
    return VB_ERR_ARG;
  }
  memcpy(dec->fold_qkv, qkv, sizeof(vb_ln_fold) * n);
  memcpy(dec->fold_ffn1, ffn1, sizeof(vb_ln_fold) * n);
  return VB_OK;
}

// ------------------------------------------------------------------------------------------
// Decoder stack: the forward of inference and training, and the backward pass
// ------------------------------------------------------------------------------------------
namespace {
// Bump allocator: 256-byte aligned slots in the order they are taken.  Carved from a null base it hands out null slots
// and only adds up the layout, so every workspace size below is its own layout carved from nullptr.
struct Carve {
  char *base;
  size_t used = 0;
  explicit Carve(const void *b) : base((char *)b) {}
  template <class T = void>
  T *take(size_t n) {
    T *r = base ? (T *)(base + used) : nullptr;
    used += align_up(n, 256);
    return r;
  }
};
// bytes of a buffer laid out by layout(c, a...): the layout carved from a null base
template <class Layout, class... A>
size_t carved_bytes(Layout layout, const A &...a) {
  Carve c(nullptr);
  layout(c, a...);
  return c.used + 256;
}

// One layer's activations.  x_in / x_mid: fp32 [M, d] copies of the residual stream as norm1 / norm2 read it, what
// the LayerNorm backward needs (null: not kept).  Storage dtype: xn1 (the QKV operand), q|k|v, attention out, xn2 (the
// FFN1 operand), FFN hidden (post-ReLU, post-dropout).
struct LayerSave {
  float *x_in, *x_mid;
  void *xn1, *qkv, *att, *xn2, *hb;
};
// the scratch of vb_decoder_forward: one set of slots that every layer reuses, no fp32 copies
LayerSave carve_forward_ws(Carve &c, const vb_decoder_desc &D, int64_t M) {
  const size_t ts = elem_size(D.wdtype), d = D.d_model, Mp = align_up((size_t)M, 128);
  LayerSave s{};
  s.xn1 = s.xn2 = c.take(Mp * d * ts);
  s.qkv = c.take(Mp * 3 * d * ts);
  s.att = c.take(Mp * d * ts);
  s.hb = c.take(Mp * D.d_ff * ts);
  return s;
}
LayerSave carve_layer_save(Carve &c, const vb_decoder_desc &D, int64_t M) {
  const size_t ts = elem_size(D.wdtype), d = D.d_model, Mp = align_up((size_t)M, 128);
  LayerSave s;
  s.x_in = c.take<float>(Mp * d * 4);
  s.x_mid = c.take<float>(Mp * d * 4);
  s.xn1 = c.take(Mp * d * ts);
  s.att = c.take(Mp * d * ts);
  s.xn2 = c.take(Mp * d * ts);
  s.qkv = c.take(Mp * 3 * d * ts);
  s.hb = c.take(Mp * D.d_ff * ts);
  return s;
}
// The training save buffer: one LayerSave block per layer, then an fp32 [M, d] scratch for the sub-layer output that
// dropout scales ahead of the residual add (returned).
float *carve_train_save(Carve &c, const vb_decoder_desc &D, int64_t M) {
  for (int l = 0; l < D.n_layer; ++l) carve_layer_save(c, D, M);
  return c.take<float>((size_t)M * D.d_model * 4);
}
// layer l's block of the training save buffer
LayerSave layer_save(const vb_decoder_desc &D, int64_t M, const void *save, int l) {
  Carve block(nullptr);
  carve_layer_save(block, D, M);
  Carve c((const char *)save + (size_t)l * block.used);
  return carve_layer_save(c, D, M);
}

// norm k (1 or 2) of layer l: its row of an AdaLN (weight|bias) table [*, 2d] or of the table's gradient (null: LayerNorm)
template <class T>
T *ada_row(T *wb, int l, int k, int d) {
  return wb ? wb + (size_t)(2 * l + k - 1) * 2 * d : nullptr;
}
// training-mode dropout of layer l (transformer.py:329,333-334, activation.py:199 `dropout=`) at site 0 (attention
// probabilities), 1 (attention output), 2 (FFN hidden) or 3 (FFN output): the stateless hash of kernels.cuh on stream
// (l << 2) | site, regenerated by the backward
DropCfg layer_drop(float p, uint64_t seed, int l, int site) { return make_drop(p, seed, (uint32_t)(l << 2) | (uint32_t)site); }

// The layer loop of vb_decoder_forward and vb_decoder_forward_train.  slots(l): layer l's activation slots; cache:
// the whole KV cache the attention fills (cache.k == nullptr: none); sub: the fp32 [M, d] scratch of the sub-layer
// outputs when dropout_p > 0.  Pre-LN (transformer.py:297-302): x += SA(norm1(x)); x += FF(norm2(x)).  Post-LN (:303-308):
// x = norm1(x + SA(x)); x = norm2(x + FF(x)); a post-norm writes the normalised rows back into x and into the
// storage-dtype operand of the next GEMM, and layer 0 reads a plain cast.
template <class Slots>
int stack_forward(const vb_decoder *dec, float *x, int64_t M, const Packed &pk, const float *ada_wb, Slots slots,
                  const KvCache &cache, int64_t cache_layer_stride, float *sub, float dropout_p, uint64_t dropout_seed,
                  cudaStream_t s) {
  const vb_decoder_desc &D = dec->desc;
  const int d = D.d_model, dff = D.d_ff, dt = D.wdtype;
  const vb_stream_t stream = (vb_stream_t)s;
  if (!D.norm_first) VB_TRY(launch_cast_from_f32(x, slots(0).xn1, dt, M * d, s));
  for (int l = 0; l < D.n_layer; ++l) {
    const vb_layer_params &P = dec->layers[l];
    const LayerSave sv = slots(l);
    // norm k reads x, copied first into the layer's fp32 slot if it has one, and writes the operand `out`
    auto norm = [&](int k, void *out) -> int {
      float *keep = k == 1 ? sv.x_in : sv.x_mid;
      if (keep) VB_CUDA(cudaMemcpyAsync(keep, x, (size_t)M * d * 4, cudaMemcpyDeviceToDevice, s));
      const float *w = k == 1 ? P.norm1_w : P.norm2_w, *b = k == 1 ? P.norm1_b : P.norm2_b;
      if (D.norm_first) return vb_layernorm(x, d, nullptr, M, d, w, b, ada_row(ada_wb, l, k, d), 1e-5f, out, dt, stream);
      return launch_post_norm(x, M, d, w, b, ada_row(ada_wb, l, k, d), 1e-5f, out, dt, s);
    };
    // x += in W^T + b, the sum ahead of the add through the dropout at `site`
    auto residual = [&](const void *in, int K, const void *W, const float *b, int site) -> int {
      if (dropout_p > 0.f) {
        VB_TRY(vb_linear(in, dt, K, W, dt, b, sub, VB_F32, d, M, d, K, VB_EPI_NONE, nullptr, 0, stream));
        return launch_dropout_add(x, sub, M * d, layer_drop(dropout_p, dropout_seed, l, site), s);
      }
      return vb_linear(in, dt, K, W, dt, b, x, VB_F32, d, M, d, K, VB_EPI_RESIDUAL, nullptr, 0, stream);
    };
    auto attn = [&]() -> int {
      VB_TRY(vb_linear(sv.xn1, dt, d, P.in_proj_w, dt, P.in_proj_b, sv.qkv, dt, 3 * d, M, 3 * d, d, VB_EPI_NONE, nullptr,
                       0, stream));
      const DropCfg dc = layer_drop(dropout_p, dropout_seed, l, 0);
      VB_TRY(launch_attention_varlen(sv.qkv, dt, M, D.n_head, d / D.n_head, pk, sv.att,
                                     kv_cache_layer(cache, cache_layer_stride, l), nullptr, 0, s, &dc));
      return residual(sv.att, d, P.out_proj_w, P.out_proj_b, 1);
    };
    auto ffn = [&]() -> int {
      VB_TRY(vb_linear(sv.xn2, dt, d, P.lin1_w, dt, P.lin1_b, sv.hb, dt, dff, M, dff, d, VB_EPI_RELU, nullptr, 0, stream));
      if (dropout_p > 0.f)
        VB_TRY(launch_dropout(sv.hb, sv.hb, dt, M * dff, layer_drop(dropout_p, dropout_seed, l, 2), s));
      return residual(sv.hb, dff, P.lin2_w, P.lin2_b, 3);
    };
    if (D.norm_first) {
      VB_TRY(norm(1, sv.xn1));
      VB_TRY(attn());
      VB_TRY(norm(2, sv.xn2));
      VB_TRY(ffn());
    } else {
      VB_TRY(attn());
      VB_TRY(norm(1, sv.xn2));
      VB_TRY(ffn());
      VB_TRY(norm(2, l + 1 < D.n_layer ? slots(l + 1).xn1 : nullptr));
    }
  }
  return VB_OK;
}

struct BackwardWs {
  void *dx_dt;          // dx in the storage dtype
  void *dy;             // dx through the mask of a sub-layer's output dropout
  void *dh, *dO, *dqkv;
  float *dn;            // pre-LN: the gradient of a norm's output
  float *dr;            // post-LN: the gradient between the two post-norms (null for pre-LN)
  void *attn_ws, *lin_ws;
  size_t attn_ws_bytes, lin_ws_bytes;
};
BackwardWs carve_backward_ws(Carve &c, const vb_decoder_desc &D, int64_t M) {
  const size_t ts = elem_size(D.wdtype), d = D.d_model, dff = D.d_ff, Mp = align_up((size_t)M, 128);
  BackwardWs w{};
  w.dx_dt = c.take(Mp * d * ts);
  w.dy = c.take(Mp * d * ts);
  w.dh = c.take(Mp * dff * ts);
  w.dn = c.take<float>(Mp * d * 4);
  w.dO = c.take(Mp * d * ts);
  w.dqkv = c.take(Mp * 3 * d * ts);
  w.attn_ws_bytes = vb_attention_backward_workspace(M, D.n_head);
  w.attn_ws = c.take(w.attn_ws_bytes);
  w.lin_ws_bytes = vb_linear_backward_workspace(D.wdtype, M, std::max(D.d_ff, 3 * D.d_model), std::max(D.d_ff, D.d_model));
  w.lin_ws = c.take(w.lin_ws_bytes);
  if (!D.norm_first) w.dr = c.take<float>(Mp * d * 4);
  return w;
}
}  // namespace

VB_API size_t vb_decoder_forward_workspace(const vb_decoder_desc *desc, int64_t M) {
  return carved_bytes(carve_forward_ws, *desc, M);
}

// The one check of an FP8 cache against a decoder (fn: the entry point's name, for the message): a bf16 decoder, both
// exponent arrays, and their layout.  The exponent rows are read 16 bytes at a time (cp.async in the decode attention):
// every (layer, utterance, head) stream of k_exp / v_exp, at offset stride / 64, and every 16-key chunk of it must
// start 16-byte aligned.
static int check_kv8(const char *fn, const vb_decoder_desc &D, const uint8_t *k_exp, const uint8_t *v_exp,
                     int64_t cache_layer_stride, int64_t cache_seq_stride, int cache_cap) {
  if (D.wdtype != VB_BF16) {
    set_error("%s: the FP8 KV cache needs a bf16 decoder", fn);
    return VB_ERR_UNSUPPORTED;
  }
  VB_CHECK_ARG(k_exp && v_exp, "%s: FP8 cache: k_exp / v_exp missing", fn);
  VB_CHECK_ARG(cache_layer_stride % 1024 == 0 && cache_seq_stride % 1024 == 0 && cache_cap % 16 == 0 &&
                   (reinterpret_cast<uintptr_t>(k_exp) & 15) == 0 && (reinterpret_cast<uintptr_t>(v_exp) & 15) == 0,
               "%s: FP8 cache: strides must be multiples of 1024, cache_cap a multiple of 16 and "
               "k_exp / v_exp 16-byte aligned", fn);
  return VB_OK;
}

VB_API int vb_decoder_forward(vb_decoder_t dec, float *x, int64_t M, int B, const int32_t *cu_seqlens,
                              const int32_t *text_lens, const int32_t *seg1_lens, int seg1_start, int max_seqlen,
                              int mask_mode, const float *ada_wb, void *kcache, void *vcache, uint8_t *k_exp,
                              uint8_t *v_exp, int64_t cache_layer_stride, int64_t cache_seq_stride, int cache_cap,
                              const int32_t *cache_slots, void *workspace, size_t workspace_bytes, vb_stream_t stream) {
  VB_CHECK_ARG(dec && x && cu_seqlens, "vb_decoder_forward: null argument");
  VB_CHECK_ARG(!kcache == !vcache, "vb_decoder_forward: kcache / vcache: both or neither");
  VB_CHECK_ARG(!k_exp == !v_exp, "vb_decoder_forward: k_exp / v_exp: both or neither");
  VB_CHECK_ARG(kcache || (!k_exp && !cache_slots), "vb_decoder_forward: k_exp / v_exp and cache_slots need a cache");
  const vb_decoder_desc &D = dec->desc;
  const bool f8 = k_exp != nullptr;
  if (f8) VB_TRY(check_kv8("vb_decoder_forward", D, k_exp, v_exp, cache_layer_stride, cache_seq_stride, cache_cap));
  VB_CHECK_ARG(workspace_bytes >= vb_decoder_forward_workspace(&D, M),
               "vb_decoder_forward: workspace too small (%zu < %zu)", workspace_bytes,
               vb_decoder_forward_workspace(&D, M));
  if (M == 0) return VB_OK;
  const KvCache cache{kcache, vcache, k_exp, v_exp, cache_seq_stride, cache_cap, (int)elem_size(f8 ? VB_E4M3 : D.wdtype)};
  const Packed pk{cu_seqlens, text_lens, seg1_lens, B, max_seqlen, seg1_start, mask_mode, cache_slots};
  Carve c(workspace);
  const LayerSave ws = carve_forward_ws(c, D, M);
  return stack_forward(dec, x, M, pk, ada_wb, [&](int) { return ws; }, cache, cache_layer_stride, nullptr, 0.f, 0,
                       (cudaStream_t)stream);
}

VB_API size_t vb_decoder_train_save_bytes(const vb_decoder_desc *desc, int64_t M) {
  return carved_bytes(carve_train_save, *desc, M);
}

VB_API int vb_decoder_forward_train(vb_decoder_t dec, float *x, int64_t M, int B, const int32_t *cu_seqlens,
                                    const int32_t *text_lens, const int32_t *seg1_lens, int seg1_start, int max_seqlen,
                                    int mask_mode, const float *ada_wb, void *save, size_t save_bytes,
                                    float dropout_p, uint64_t dropout_seed, vb_stream_t stream) {
  VB_CHECK_ARG(dec && x && cu_seqlens && save, "vb_decoder_forward_train: null argument");
  VB_CHECK_ARG(dropout_p >= 0.f && dropout_p < 1.f, "vb_decoder_forward_train: dropout_p=%g not in [0, 1)", (double)dropout_p);
  const vb_decoder_desc &D = dec->desc;
  VB_CHECK_ARG(save_bytes >= vb_decoder_train_save_bytes(&D, M), "vb_decoder_forward_train: save buffer too small");
  if (M == 0) return VB_OK;
  Carve c(save);
  float *sub = carve_train_save(c, D, M);
  const Packed pk{cu_seqlens, text_lens, seg1_lens, B, max_seqlen, seg1_start, mask_mode};
  return stack_forward(dec, x, M, pk, ada_wb, [&](int l) { return layer_save(D, M, save, l); }, KvCache{}, 0, sub,
                       dropout_p, dropout_seed, (cudaStream_t)stream);
}

VB_API size_t vb_decoder_backward_workspace(const vb_decoder_desc *desc, int64_t M) {
  return carved_bytes(carve_backward_ws, *desc, M);
}

VB_API int vb_decoder_backward(vb_decoder_t dec, float *dx, int64_t M, int B, const int32_t *cu_seqlens,
                               const int32_t *text_lens, const int32_t *seg1_lens, int seg1_start, int max_seqlen,
                               int mask_mode, const float *ada_wb, float *dada_wb, const void *save,
                               const vb_layer_wt *wt, const vb_layer_grads *grads, void *workspace,
                               size_t workspace_bytes, float dropout_p, uint64_t dropout_seed, vb_stream_t stream) {
  VB_CHECK_ARG(dec && dx && cu_seqlens && save && wt && grads, "vb_decoder_backward: null argument");
  VB_CHECK_ARG(dropout_p >= 0.f && dropout_p < 1.f, "vb_decoder_backward: dropout_p=%g not in [0, 1)", (double)dropout_p);
  const vb_decoder_desc &D = dec->desc;
  VB_CHECK_ARG(workspace_bytes >= vb_decoder_backward_workspace(&D, M), "vb_decoder_backward: workspace too small");
  VB_CHECK_ARG(!ada_wb || dada_wb, "vb_decoder_backward: AdaLN stack needs dada_wb");
  if (M == 0) return VB_OK;
  cudaStream_t s = (cudaStream_t)stream;
  const int d = D.d_model, dff = D.d_ff, dt = D.wdtype;
  Carve c(workspace);
  const BackwardWs w = carve_backward_ws(c, D, M);
  const Packed pk{cu_seqlens, text_lens, seg1_lens, B, max_seqlen, seg1_start, mask_mode};
  const bool drop = dropout_p > 0.f;
  const float inv_keep = drop ? 1.f / (1.f - dropout_p) : 1.f;
  // dx holds the gradient of the stack output on entry.  dx_dt, the residual stream's gradient in the storage dtype
  // (refreshed by each LayerNorm backward), is the gradient of the output of the sub-layer handled next; dy is that
  // gradient through the mask of the sub-layer's output dropout
  const void *dy = drop ? w.dy : w.dx_dt;
  if (D.norm_first) VB_TRY(launch_cast_from_f32(dx, w.dx_dt, dt, M * d, s));
  for (int l = D.n_layer - 1; l >= 0; --l) {
    const vb_layer_params &P = dec->layers[l];
    const vb_layer_grads &G = grads[l];
    const vb_layer_wt &T = wt[l];
    const LayerSave sv = layer_save(D, M, save, l);
    // norm k: from the gradient dout of its output, the gradient of its input added into dst and copied into dx_dt
    auto norm = [&](int k, const float *dout, float *dst) -> int {
      const bool n1 = k == 1;
      return vb_layernorm_backward(n1 ? sv.x_in : sv.x_mid, d, nullptr, M, d, n1 ? P.norm1_w : P.norm2_w,
                                   n1 ? P.norm1_b : P.norm2_b, ada_row(ada_wb, l, k, d), 1e-5f, dout, d, dst, d, w.dx_dt,
                                   dt, n1 ? G.norm1_w : G.norm2_w, n1 ? G.norm1_b : G.norm2_b, ada_row(dada_wb, l, k, d),
                                   stream);
    };
    // FFN block x + linear2(drop(relu(linear1(xn2)))): the input gradient into dst by the epilogue epi (with dropout
    // the saved hidden is post-dropout, zero where dropped)
    auto ffn = [&](float *dst, int epi) -> int {
      if (drop) VB_TRY(launch_dropout(w.dx_dt, w.dy, dt, M * d, layer_drop(dropout_p, dropout_seed, l, 3), s));
      VB_TRY(vb_linear_backward(sv.hb, dt, dff, T.lin2_wt, dy, d, w.dh, dt, dff, VB_EPI_NONE, G.lin2_w, G.lin2_b, M, d, dff,
                                w.lin_ws, w.lin_ws_bytes, stream));
      VB_TRY(launch_relu_bwd(w.dh, sv.hb, dt, M * dff, inv_keep, s));
      return vb_linear_backward(sv.xn2, dt, d, T.lin1_wt, w.dh, dff, dst, VB_F32, d, epi, G.lin1_w, G.lin1_b, M, dff, d,
                                w.lin_ws, w.lin_ws_bytes, stream);
    };
    // attention block x + out_proj(Attn(in_proj(xn1))): input gradient into dst by the epilogue epi
    auto attn = [&](float *dst, int epi) -> int {
      if (drop) VB_TRY(launch_dropout(w.dx_dt, w.dy, dt, M * d, layer_drop(dropout_p, dropout_seed, l, 1), s));
      VB_TRY(vb_linear_backward(sv.att, dt, d, T.out_proj_wt, dy, d, w.dO, dt, d, VB_EPI_NONE, G.out_proj_w, G.out_proj_b,
                                M, d, d, w.lin_ws, w.lin_ws_bytes, stream));
      const DropCfg dc = layer_drop(dropout_p, dropout_seed, l, 0);
      VB_TRY(attention_backward(sv.qkv, sv.att, w.dO, dt, M, D.n_head, d / D.n_head, pk, w.dqkv, w.attn_ws,
                                w.attn_ws_bytes, &dc, s));
      return vb_linear_backward(sv.xn1, dt, d, T.in_proj_wt, w.dqkv, 3 * d, dst, VB_F32, d, epi, G.in_proj_w,
                                G.in_proj_b, M, 3 * d, d, w.lin_ws, w.lin_ws_bytes, stream);
    };
    if (D.norm_first) {
      // each block's input gradient goes to dn, and its norm's backward adds it to the residual gradient in dx
      VB_TRY(ffn(w.dn, VB_EPI_NONE));
      VB_TRY(norm(2, w.dn, dx));
      VB_TRY(attn(w.dn, VB_EPI_NONE));
      VB_TRY(norm(1, w.dn, dx));
    } else {
      // y = norm2(r2), r2 = x1 + drop(FF(x1)), x1 = norm1(r1), r1 = x + drop(SA(x)): dr = norm2^T(dy), the FFN input
      // gradient is added to dr (= dx1), dx = norm1^T(dx1), the attention input gradient is added to dx
      VB_CUDA(cudaMemsetAsync(w.dr, 0, (size_t)M * d * 4, s));
      VB_TRY(norm(2, dx, w.dr));
      VB_TRY(ffn(w.dr, VB_EPI_RESIDUAL));
      VB_CUDA(cudaMemsetAsync(dx, 0, (size_t)M * d * 4, s));
      VB_TRY(norm(1, w.dr, dx));
      VB_TRY(attn(dx, VB_EPI_RESIDUAL));
    }
  }
  return VB_OK;
}

// ------------------------------------------------------------------------------------------
// AR decode
// ------------------------------------------------------------------------------------------
namespace {
struct StepWs {
  float *q, *att, *hb;
  void *attn_ws;
  bf16 *xn16, *att16, *hb16;
  void *gemm_ws;
  float *stats;  // moments of the folded-LayerNorm projections: [kMaxForcedSplits][64][2]
  size_t gemm_ws_bytes;
};
StepWs carve_step_ws(Carve &c, const vb_decoder_desc &D, int B, int cache_cap) {
  const size_t d = D.d_model, dff = D.d_ff;
  StepWs w{};
  w.q = c.take<float>((size_t)B * d * 4);
  w.att = c.take<float>((size_t)B * d * 4);
  w.hb = c.take<float>((size_t)B * dff * 4);
  w.attn_ws = c.take(attn_decode_workspace(B, D.n_head, (int)(d / D.n_head), cache_cap));
  w.xn16 = c.take<bf16>((size_t)64 * d * 2);
  w.att16 = c.take<bf16>((size_t)64 * d * 2);
  w.hb16 = c.take<bf16>((size_t)64 * dff * 2);
  w.gemm_ws_bytes = gemm_decode_workspace((int)d, (int)dff);
  w.gemm_ws = c.take(w.gemm_ws_bytes);
  w.stats = c.take<float>((size_t)kLnFoldMaxCopies * kMaxForcedSplits * 64 * 2 * sizeof(float));
  return w;
}
// tensor-core decode path: bf16 storage, up to 64 rows (one UMMA N tile)
bool use_tc_decode(const vb_decoder_desc &D, int B) {
  return D.wdtype == VB_BF16 && B >= 1 && B <= 64 && tune("VB_DECODE_SIMT", 0) == 0;
}
// the LayerNorm-folded chain: the decoder's norms (vb_decoder_set_decode_fold) and the head's final norm are folded
bool use_fold(const vb_decoder *dec, const vb_ar_head *head) { return dec->fold_qkv && head->fold.wf; }
bool use_pdl() { return tune("VB_NO_PDL", 0) == 0; }

// split-K counts of the four decode projections.  Split-K wide enough to fill the SMs (0) is not the optimum for the
// projections whose partial sums a reduce kernel has to add up again, hence fixed counts (not re-tuned on H100;
// VB_SPLITS_* override them).  The folded chain has no reduce kernel that pays for more slabs, and with <= 6 k-blocks
// per CTA its weight ring never wraps.
struct DecodeSplits {
  int qkv, out, ffn1, ffn2;
};
DecodeSplits decode_splits(const vb_decoder_desc &D, bool fold) {
  const int kb = D.d_model / 128, fb = D.d_ff / 128;
  auto upto = [](int n, int cap) { return std::max(1, std::min(cap, n)); };
  auto knob = [](const char *name, int dflt) {
    const int v = tune(name, 0);
    return v > 0 ? v : dflt;
  };
  return {knob("VB_SPLITS_QKV", upto(kb, 5)), knob("VB_SPLITS_OUT", fold ? 8 : 0),
          knob("VB_SPLITS_FFN1", upto(kb, fold ? 4 : 2)), knob("VB_SPLITS_FFN2", upto(fb, fold ? 8 : 9))};
}

bool kv_fp8(const vb_ar_state *st) { return st->kv_dtype == VB_E4M3; }
// layer l's cache and the rows' lengths: where the QKV projection leaves q and appends k / v, what the attention
// reads and what the KV prefetch pulls into L2
QkvScatter layer_kv(const vb_decoder_desc &D, const vb_ar_state *st, int l, float *q) {
  const bool f8 = kv_fp8(st);
  const KvCache cache{st->kcache, st->vcache, f8 ? st->k_exp : nullptr, f8 ? st->v_exp : nullptr, st->cache_seq_stride,
                      st->cache_cap, (int)elem_size(f8 ? VB_E4M3 : D.wdtype)};
  return QkvScatter{D.d_model, D.d_model / D.n_head, q, kv_cache_layer(cache, st->cache_layer_stride, l),
                    KvRows{st->text_len, st->prompt_len, st->n_gen, st->finished}};
}

// the beam ancestry the decode attention follows (beam_width > 1, or per-row groups), or none
BeamAnc beam_anc(const vb_ar_state *st) {
  if (st->beam_first) return BeamAnc{st->beam_anc, st->tok_stride, 0, st->beam_first};
  return st->beam_width > 1 ? BeamAnc{st->beam_anc, st->tok_stride, st->beam_width} : BeamAnc{};
}
// The per-row beam groups (vb_ar_state.beam_first / beam_n) as the header states them, read back on `s` unless `s`
// is capturing a graph (a captured call reads no host values: there the caller guarantees them).  slots / k:
// vb_ar_admit's slots, which must pass every admitted group's rows together and in order.
int check_groups(const char *fn, const vb_ar_state *st, const int32_t *slots, int k, cudaStream_t s) {
  cudaStreamCaptureStatus cap;
  VB_CUDA(cudaStreamIsCapturing(s, &cap));
  if (cap != cudaStreamCaptureStatusNone) return VB_OK;
  const int B = st->B;
  std::vector<int32_t> f(B), w(B), sl(k);
  VB_CUDA(cudaMemcpyAsync(f.data(), st->beam_first, B * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
  VB_CUDA(cudaMemcpyAsync(w.data(), st->beam_n, B * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
  if (k > 0) VB_CUDA(cudaMemcpyAsync(sl.data(), slots, k * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
  VB_CUDA(cudaStreamSynchronize(s));
  for (int b = 0; b < B; ++b) {
    const int g = f[b], n = w[b];
    if (g == -1) continue;
    VB_CHECK_ARG(n >= 2 && n <= 16, "%s: beam_n[%d] = %d not in [2, 16]", fn, b, n);
    VB_CHECK_ARG(g >= 0 && g <= b && b < g + n && g + n <= B && f[g] == g && w[g] == n,
                 "%s: row %d: beam_first %d / beam_n %d is not a group of rows [first, first + n) within B = %d", fn,
                 b, g, n, B);
    if (g == b)
      for (int j = 1; j < n; ++j)
        VB_CHECK_ARG(f[b + j] == b, "%s: row %d of the group at row %d has beam_first %d", fn, b + j, b, f[b + j]);
  }
  for (int i = 0; i < k; ++i) {
    VB_CHECK_ARG(sl[i] >= 0 && sl[i] < B, "%s: slots[%d] = %d not in [0, B = %d)", fn, i, sl[i], B);
    const int g = f[sl[i]], j = sl[i] - g, i0 = i - j;
    if (g < 0) continue;
    bool whole = i0 >= 0 && i0 + w[g] <= k;
    for (int q = 0; whole && q < w[g]; ++q) whole = sl[i0 + q] == g + q;
    VB_CHECK_ARG(whole, "%s: slots[%d] = %d: the group at row %d is not admitted whole and in order", fn, i, sl[i], g);
  }
  return VB_OK;
}
// the beam-search fields a step with this head reads (include/valle_b200.h "Beam search")
int check_beam(const char *fn, const vb_ar_head *head, const vb_ar_state *st, cudaStream_t s,
               const int32_t *slots = nullptr, int k = 0) {
  const bool per_row = st->beam_first != nullptr;
  if (per_row || head->greedy == 4) {
    VB_CHECK_ARG(st->beam_width <= 1, "%s: per-row beam groups (beam_first) with beam_width %d > 1", fn,
                 st->beam_width);
    VB_CHECK_ARG(head->greedy == 4, "%s: per-row beam groups run with vb_ar_head.greedy == 4 (got %d)", fn,
                 head->greedy);
    VB_CHECK_ARG(per_row && st->beam_n && st->beam_anc, "%s: vb_ar_head.greedy == 4 needs beam_first, beam_n and "
                 "beam_anc", fn);
  }
  if (head->greedy == 3 || st->beam_width > 1) {
    VB_CHECK_ARG(st->beam_width >= 1 && st->beam_width <= 16 && st->B % st->beam_width == 0,
                 "%s: beam_width %d not in [1, 16] or not dividing B = %d", fn, st->beam_width, st->B);
    VB_CHECK_ARG(st->beam_anc != nullptr, "%s: beam search needs beam_anc", fn);
  }
  if (head->greedy >= 3)
    VB_CHECK_ARG(st->beam_score && st->beam_fin_score && st->beam_fin_len && st->beam_fin_anc,
                 "%s: vb_ar_head.greedy == %d: beam arrays not set", fn, head->greedy);
  if (per_row) VB_TRY(check_groups(fn, st, slots, k, s));
  return VB_OK;
}
// the step's tail on the head's logits (in: their pending partials): the argmax / seeded draw, the reduce alone
// (greedy == 0), the reduce and the beam step (greedy == 3), or the seeded draw of the rows in no group and the beam
// step of every group (greedy == 4)
int ar_tail(int ldl, const SplitK &in, const vb_ar_head *head, vb_ar_state *st, int d, bool pdl, cudaStream_t s) {
  if (head->greedy == 4) {
    VB_TRY(launch_ar_sample(st->logits, ldl, in, head, st, d, nullptr, 0, pdl, s));
    return launch_beam_tail(head, st, d, pdl, s);
  }
  if (head->greedy != 3)
    return launch_ar_sample(st->logits, ldl, in, head, st, d, nullptr, head->greedy ? 0 : 1, pdl, s);
  if (in.part) VB_TRY(launch_ar_sample(st->logits, ldl, in, head, st, d, nullptr, 1, pdl, s));
  return launch_beam_tail(head, st, d, pdl, s);
}

// final LayerNorm (adding the pending partials of the last FFN2) + ar_predict_layer + sampler on the tensor-core
// path.  fold: the final norm is folded into ar_predict_layer, the projection reads the fp32 rows and the sampler
// applies the moments.  A stack without a final norm (post-LN) feeds the head the bf16 rows of x: w.xn16 as the
// decode chain's last post-norm left it (xn_ready), else a cast of x.
int tc_head(const vb_decoder_desc &D, const vb_ar_head *head, float *x, vb_ar_state *st, const StepWs &w, bool fold,
            const SplitK &pend, cudaStream_t s, bool xn_ready = false) {
  const int d = D.d_model, B = st->B;
  const int ldl = (head->n_vocab + 3) & ~3;
  const bool pdl = use_pdl();
  SplitK logits;
  if (fold) {
    VB_TRY(launch_gemm_decode_x(x, B, d, head->fold, head->n_vocab, d, 0, (float *)w.gemm_ws, w.gemm_ws_bytes, w.stats,
                                &logits, nullptr, pdl, s));
    return ar_tail(ldl, logits, head, st, d, pdl, s);
  }
  if (D.final_norm_w)
    VB_TRY(launch_ln_reduce(x, d, B, d, pend, D.final_norm_w, D.final_norm_b, 1e-5f, w.xn16, pdl, s));
  else if (!xn_ready)
    VB_TRY(launch_cast_from_f32(x, w.xn16, VB_BF16, (int64_t)B * d, s));
  VB_TRY(launch_gemm_decode(w.xn16, B, d, (const bf16 *)head->predict_w, head->n_vocab, d, 0, nullptr, DG_F32,
                            st->logits, nullptr, ldl, nullptr, (float *)w.gemm_ws, w.gemm_ws_bytes, &logits, nullptr,
                            pdl, s));
  // logits only (host-side sampling follows) and split: just reduce the partials
  if (head->greedy || logits.part) VB_TRY(ar_tail(ldl, logits, head, st, d, pdl, s));
  return VB_OK;
}
}  // namespace

VB_API size_t vb_ar_step_workspace(const vb_decoder_desc *desc, int B, int cache_cap) {
  return carved_bytes(carve_step_ws, *desc, B, cache_cap);
}

namespace {
// vb_ar_head_step once its arguments are checked (vb_ar_decode_step's CUDA-core chain ends with it)
int head_step(vb_decoder_t dec, const vb_ar_head *head, const float *h, vb_ar_state *st, void *workspace,
              size_t workspace_bytes, cudaStream_t s) {
  const vb_decoder_desc &D = dec->desc;
  const int d = D.d_model;
  const int ldl = (head->n_vocab + 3) & ~3;
  if (use_tc_decode(D, st->B)) {
    VB_CHECK_ARG(workspace && workspace_bytes >= vb_ar_step_workspace(&D, st->B, st->cache_cap),
                 "vb_ar_head_step: workspace too small");
    Carve c(workspace);
    const StepWs w = carve_step_ws(c, D, st->B, st->cache_cap);
    return tc_head(D, head, const_cast<float *>(h), st, w, use_fold(dec, head), SplitK{}, s);
  }
  LnParams ln{D.final_norm_w, D.final_norm_b, nullptr, 1e-5f};
  VB_TRY(launch_gemv(h, d, st->B, head->predict_w, D.wdtype, nullptr, head->n_vocab, d, st->logits, ldl,
                     D.final_norm_w ? &ln : nullptr, 0, nullptr, s));
  if (head->greedy) VB_TRY(ar_tail(ldl, SplitK{}, head, st, d, false, s));
  return VB_OK;
}
}  // namespace

VB_API int vb_ar_head_step(vb_decoder_t dec, const vb_ar_head *head, const float *h, vb_ar_state *st,
                           void *workspace, size_t workspace_bytes, vb_stream_t stream) {
  VB_CHECK_ARG(dec && head && h && st, "vb_ar_head_step: null argument");
  VB_CHECK_ARG(head->greedy >= 0 && head->greedy <= 4, "vb_ar_head_step: greedy %d not in {0, 1, 2, 3, 4}",
               head->greedy);
  VB_TRY(check_beam("vb_ar_head_step", head, st, (cudaStream_t)stream));
  VB_CHECK_ARG(!dec->desc.norm_first || dec->desc.final_norm_w, "vb_ar_head_step: a pre-LN decoder needs its final norm");
  return head_step(dec, head, h, st, workspace, workspace_bytes, (cudaStream_t)stream);
}

namespace {
// vb_ar_admit's workspace: a k-row state (cs, tok_stride 1) for the head step of the admitted rows, then that head
// step's own workspace
struct AdmitWs {
  vb_ar_state cs;
  void *head_ws;
  size_t head_ws_bytes;
};
constexpr int kAdmitCap = 64;  // the k-row state holds no cache: the smallest capacity sizes the head's workspace
AdmitWs carve_admit_ws(Carve &c, const vb_decoder_desc &D, int k, int n_vocab) {
  AdmitWs w{};
  vb_ar_state &cs = w.cs;
  cs.B = k;
  cs.tok_stride = 1;
  cs.text_len = c.take<int32_t>(k * 4);
  cs.prompt_len = c.take<int32_t>(k * 4);
  cs.max_new = c.take<int32_t>(k * 4);
  cs.n_gen = c.take<int32_t>(k * 4);
  cs.finished = c.take<int32_t>(k * 4);
  cs.tokens = c.take<int32_t>(k * 4);
  cs.x_cur = c.take<float>((size_t)k * D.d_model * 4);
  cs.logits = c.take<float>((size_t)k * ((n_vocab + 3) & ~3) * 4);
  cs.cache_cap = kAdmitCap;
  cs.sample_seed = c.take<uint64_t>(k * 8);
  cs.top_k = c.take<int32_t>(k * 4);
  cs.temperature = c.take<float>(k * 4);
  cs.top_p = c.take<float>(k * 4);
  cs.ras_window = c.take<int32_t>(k * 4);
  cs.ras_max = c.take<int32_t>(k * 4);
  cs.beam_first = c.take<int32_t>(k * 4);   // the per-row beam groups (head->greedy == 4 only)
  cs.beam_n = c.take<int32_t>(k * 4);
  cs.beam_anc = c.take<uint8_t>(k);
  cs.beam_score = c.take<float>(k * 4);
  cs.beam_fin_score = c.take<float>(k * 8);
  cs.beam_fin_len = c.take<int32_t>(k * 4);
  cs.beam_fin_anc = c.take<uint8_t>(k);
  cs.logprob = c.take<float>(k * 4);        // the first draw's score (st->logprob set only)
  w.head_ws_bytes = vb_ar_step_workspace(&D, k, kAdmitCap);
  w.head_ws = c.take(w.head_ws_bytes);
  return w;
}
}  // namespace

VB_API size_t vb_ar_admit_workspace(const vb_decoder_desc *desc, int k, int n_vocab) {
  return carved_bytes(carve_admit_ws, *desc, k, n_vocab);
}

VB_API int vb_ar_admit(vb_decoder_t dec, const vb_ar_head *head, const float *h, int k, const int32_t *slots,
                       vb_ar_state *st, void *workspace, size_t workspace_bytes, vb_stream_t stream) {
  VB_CHECK_ARG(dec && head && h && slots && st, "vb_ar_admit: null argument");
  VB_CHECK_ARG(k >= 1 && k <= st->B, "vb_ar_admit: k=%d not in [1, B=%d]", k, st->B);
  VB_CHECK_ARG(head->greedy >= 0 && head->greedy <= 4 && head->greedy != 3, "vb_ar_admit: greedy %d not in {0, 1, 2, 4}",
               head->greedy);
  VB_CHECK_ARG(head->greedy < 2 || (st->sample_seed && st->top_k && st->temperature),
               "vb_ar_admit: vb_ar_head.greedy == %d: sampler arrays not set", head->greedy);
  VB_TRY(check_beam("vb_ar_admit", head, st, (cudaStream_t)stream, slots, k));
  const vb_decoder_desc &D = dec->desc;
  VB_CHECK_ARG(workspace && workspace_bytes >= vb_ar_admit_workspace(&D, k, head->n_vocab),
               "vb_ar_admit: workspace too small (%zu < %zu)", workspace_bytes,
               vb_ar_admit_workspace(&D, k, head->n_vocab));
  cudaStream_t s = (cudaStream_t)stream;
  Carve c(workspace);
  AdmitWs w = carve_admit_ws(c, D, k, head->n_vocab);
  if (head->greedy != 4)
    w.cs.beam_first = w.cs.beam_n = nullptr;
  if (!st->logprob) w.cs.logprob = nullptr;
  const int ldl = (head->n_vocab + 3) & ~3;
  VB_TRY(launch_ar_admit_copy(st, &w.cs, slots, D.d_model, ldl, head->n_vocab, false, s));
  VB_CHECK_ARG(!D.norm_first || D.final_norm_w, "vb_ar_admit: a pre-LN decoder needs its final norm");
  VB_TRY(head_step(dec, head, h, &w.cs, w.head_ws, w.head_ws_bytes, s));
  return launch_ar_admit_copy(st, &w.cs, slots, D.d_model, ldl, head->n_vocab, true, s);
}

VB_API int vb_ar_fork_prefix(vb_decoder_t dec, const int32_t *slots, int k, vb_ar_state *st, vb_stream_t stream) {
  VB_CHECK_ARG(dec && slots && st, "vb_ar_fork_prefix: null argument");
  if (kv_fp8(st)) {
    set_error("vb_ar_fork_prefix: kv_parent (shared prompt prefixes) is not supported on the FP8 KV cache");
    return VB_ERR_UNSUPPORTED;
  }
  VB_CHECK_ARG(k >= 1 && k <= st->B, "vb_ar_fork_prefix: k=%d not in [1, B=%d]", k, st->B);
  VB_CHECK_ARG(st->kv_parent && st->text_len && st->prompt_len && st->kcache && st->vcache,
               "vb_ar_fork_prefix: needs kv_parent, text_len, prompt_len and the cache");
  const vb_decoder_desc &D = dec->desc;
  return launch_ar_fork_prefix(st, D.n_layer, D.n_head, (int)elem_size(D.wdtype), slots, k, (cudaStream_t)stream);
}

VB_API int vb_cast_from_f32(const float *in, void *out, int dtype, int64_t n, vb_stream_t stream) {
  VB_CHECK_ARG(dtype == VB_F32 || dtype == VB_BF16, "vb_cast_from_f32: bad dtype %d", dtype);
  VB_CHECK_ARG(n >= 0 && (n == 0 || (in && out)), "vb_cast_from_f32: null argument / bad size");
  return launch_cast_from_f32(in, out, dtype, n, (cudaStream_t)stream);
}

VB_API int vb_ar_push_tokens(const vb_ar_head *head, vb_ar_state *st, const int64_t *sampled, int d,
                             vb_stream_t stream) {
  VB_CHECK_ARG(head && st && sampled, "vb_ar_push_tokens: null argument");
  const int ldl = (head->n_vocab + 3) & ~3;
  return launch_ar_sample(st->logits, ldl, SplitK{}, head, st, d, sampled, 0, false, (cudaStream_t)stream);
}

VB_API int vb_ar_beam_step(const vb_ar_head *head, vb_ar_state *st, int d, float *lse, vb_stream_t stream) {
  VB_CHECK_ARG(head && st, "vb_ar_beam_step: null argument");
  VB_CHECK_ARG(head->greedy == 3 || head->greedy == 4, "vb_ar_beam_step: vb_ar_head.greedy %d not in {3, 4}",
               head->greedy);
  VB_TRY(check_beam("vb_ar_beam_step", head, st, (cudaStream_t)stream));
  return launch_beam_tail(head, st, d, false, (cudaStream_t)stream, lse);
}

VB_API int vb_ar_decode_step(vb_decoder_t dec, const vb_ar_head *head, vb_ar_state *st, void *workspace,
                             size_t workspace_bytes, vb_stream_t stream) {
  VB_CHECK_ARG(dec && head && st, "vb_ar_decode_step: null argument");
  VB_CHECK_ARG(head->greedy >= 0 && head->greedy <= 4, "vb_ar_decode_step: greedy %d not in {0, 1, 2, 3, 4}",
               head->greedy);
  VB_TRY(check_beam("vb_ar_decode_step", head, st, (cudaStream_t)stream));
  const vb_decoder_desc &D = dec->desc;
  // the pre-LN chain leaves the last FFN2's partial sums to the final norm's reduce: without one they would be lost
  VB_CHECK_ARG(!D.norm_first || D.final_norm_w, "vb_ar_decode_step: a pre-LN decoder needs its final norm");
  VB_CHECK_ARG(workspace_bytes >= vb_ar_step_workspace(&D, st->B, st->cache_cap),
               "vb_ar_decode_step: workspace too small");
  const bool f8 = kv_fp8(st);
  if (f8 && !use_tc_decode(D, st->B)) {
    set_error("vb_ar_decode_step: the FP8 KV cache runs on the bf16 tensor-core chains only (bf16, B <= 64, not VB_DECODE_SIMT)");
    return VB_ERR_UNSUPPORTED;
  }
  if (f8)
    VB_TRY(check_kv8("vb_ar_decode_step", D, st->k_exp, st->v_exp, st->cache_layer_stride, st->cache_seq_stride,
                     st->cache_cap));
  if (f8 && st->kv_parent) {
    set_error("vb_ar_decode_step: kv_parent (shared prompt prefixes) is not supported on the FP8 KV cache");
    return VB_ERR_UNSUPPORTED;
  }
  if (f8 && (st->beam_width > 1 || st->beam_first)) {
    set_error("vb_ar_decode_step: beam search (beam_width > 1 or beam_first) is not supported on the FP8 KV cache");
    return VB_ERR_UNSUPPORTED;
  }
  cudaStream_t s = (cudaStream_t)stream;
  const int d = D.d_model, dff = D.d_ff, B = st->B, dt = D.wdtype, hd = d / D.n_head;
  const size_t ts = elem_size(dt);
  const int kv_dt = f8 ? VB_E4M3 : dt;
  const size_t kv_row_bytes = hd * elem_size(kv_dt) + (f8 ? 1 : 0);   // one cached row of K (or V), with its exponent byte
  Carve c(workspace);
  const StepWs w = carve_step_ws(c, D, B, st->cache_cap);
  float *x = st->x_cur;
  const bool post = !D.norm_first;
  if (use_tc_decode(D, B)) {
    // bf16 tensor-core path: swap-AB split-K wgmma projections whose partial sums are consumed by the next kernel in
    // the chain (PDL-chained).  Three chains share the layer loop:
    //   folded (6 launches per layer): QKV'(x) -> attention (+ moments, KV append) -> out-proj (+= x) -> FFN1'(x) ->
    //     ReLU reduce (+ moments) -> FFN2 (+= x).  The projections that consume the residual stream x read its fp32
    //     rows and carry the LayerNorm in their weights (vb_ln_fold), the rows' moments travel with the partial sums;
    //     the projections that produce x assemble it in place (the splits of a tile as a cluster, summed over DSMEM
    //     in fixed order).
    //   unfolded pre-LN (8): ln_reduce(+ the previous FFN2's partials, norm1) -> QKV -> attention -> out-proj ->
    //     ln_reduce(norm2) -> FFN1 -> ReLU reduce -> FFN2.
    //   post-LN (8; transformer.py:303-308, one cast of x ahead of layer 0 and none of the final norm): QKV ->
    //     attention -> out-proj -> ln_reduce<post>(norm1) -> FFN1 -> ReLU reduce -> FFN2 -> ln_reduce<post>(norm2),
    //     each post-norm writing the normalised rows into x as well.
    const bool pdl = use_pdl();
    const bool fold = use_fold(dec, head);
    const DecodeSplits sp = decode_splits(D, fold);
    // KV prefetch budget: a share of the L2 that one layer's weights, streaming through it at the same time, leave
    // free (VB_KV_PREFETCH_L2_PCT, DESIGN section 7), spread evenly over the B x H streams as their leading rows.
    // Lines evicted before the attention reads them would cost their HBM bytes twice.
    const int64_t layer_w_bytes = (4 * (int64_t)d * d + 2 * (int64_t)d * dff) * (int64_t)ts;
    const int64_t pf_budget = B >= 16 ? std::max<int64_t>(0, l2_bytes() - layer_w_bytes) *
                                            tune("VB_KV_PREFETCH_L2_PCT", 60) / 100 : 0;
    const int pf_rows = (int)std::min<int64_t>(st->cache_cap, pf_budget / (2 * (int64_t)B * D.n_head * kv_row_bytes));
    float *P = (float *)w.gemm_ws;
    // the four projections of the chain each prefetch a quarter of the first pf_rows rows of the KV streams that the
    // NEXT attention launch will read (QKV: this layer's, the other three: the following layer's)
    auto kv_slice = [&](int layer, int quarter) {
      if (pf_rows <= 0) return KvPrefetch{};
      const QkvScatter kv = layer_kv(D, st, layer % D.n_layer, w.q);
      return KvPrefetch{kv.kv, kv.rows, B, D.n_head, pf_rows * quarter / 4, pf_rows * (quarter + 1) / 4, st->kv_parent};
    };
    SplitK pend;  // the last FFN2's partial sums, for the next LayerNorm to add
    if (post) VB_TRY(launch_cast_from_f32(x, w.xn16, VB_BF16, (int64_t)B * d, s));
    for (int l = 0; l < D.n_layer; ++l) {
      const vb_layer_params &L = dec->layers[l];
      const QkvScatter kv = layer_kv(D, st, l, w.q);
      const KvPrefetch pf_qkv = kv_slice(l, 3), pf_out = kv_slice(l + 1, 0), pf_f1 = kv_slice(l + 1, 1),
                       pf_f2 = kv_slice(l + 1, 2);
      SplitK qkv, out, ffn1;
      if (fold) {
        VB_TRY(launch_gemm_decode_x(x, B, d, dec->fold_qkv[l], 3 * d, d, sp.qkv, P, w.gemm_ws_bytes, w.stats, &qkv,
                                    &pf_qkv, pdl, s));
      } else {
        if (!post) VB_TRY(launch_ln_reduce(x, d, B, d, pend, L.norm1_w, L.norm1_b, 1e-5f, w.xn16, pdl, s));
        if (f8) {
          // the FP8 append needs a head's 64 columns together: the projection always hands its product (the raw sums of
          // one split land as slab 0) to the attention prologue, which adds the bias and quantizes the rows
          VB_TRY(launch_gemm_decode(w.xn16, B, d, (const bf16 *)L.in_proj_w, 3 * d, d, sp.qkv, nullptr, DG_F32, P,
                                    nullptr, 3 * d, nullptr, P, w.gemm_ws_bytes, &qkv, &pf_qkv, pdl, s));
          qkv.part = P;
          qkv.ldp = 3 * d;
          qkv.bias = L.in_proj_b;
        } else {
          VB_TRY(launch_gemm_decode(w.xn16, B, d, (const bf16 *)L.in_proj_w, 3 * d, d, sp.qkv, L.in_proj_b, DG_QKV,
                                    nullptr, nullptr, d, &kv, P, w.gemm_ws_bytes, &qkv, &pf_qkv, pdl, s));
        }
      }
      VB_TRY(launch_attn_decode(kv, qkv, B, D.n_head, kv_dt, w.att, w.att16, w.attn_ws, pdl, s, st->kv_parent,
                                beam_anc(st)));
      VB_TRY(launch_gemm_decode(w.att16, B, d, (const bf16 *)L.out_proj_w, d, d, sp.out, L.out_proj_b, DG_RESIDUAL, x,
                                nullptr, d, nullptr, P, w.gemm_ws_bytes, &out, &pf_out, pdl, s, fold));
      if (fold) {
        VB_TRY(launch_gemm_decode_x(x, B, d, dec->fold_ffn1[l], dff, d, sp.ffn1, P, w.gemm_ws_bytes, w.stats, &ffn1,
                                    &pf_f1, pdl, s));
      } else {
        VB_TRY(launch_ln_reduce(x, d, B, d, out, post ? L.norm1_w : L.norm2_w, post ? L.norm1_b : L.norm2_b, 1e-5f,
                                w.xn16, pdl, s, post));
        VB_TRY(launch_gemm_decode(w.xn16, B, d, (const bf16 *)L.lin1_w, dff, d, sp.ffn1, L.lin1_b, DG_RELU_BF16,
                                  nullptr, w.hb16, dff, nullptr, P, w.gemm_ws_bytes, &ffn1, &pf_f1, pdl, s));
      }
      if (ffn1.part) VB_TRY(launch_relu_reduce(ffn1, B, dff, w.hb16, dff, pdl, s));
      VB_TRY(launch_gemm_decode(w.hb16, B, dff, (const bf16 *)L.lin2_w, d, dff, sp.ffn2, L.lin2_b, DG_RESIDUAL, x,
                                nullptr, d, nullptr, P, w.gemm_ws_bytes, &pend, &pf_f2, pdl, s, fold));
      if (post) {
        VB_TRY(launch_ln_reduce(x, d, B, d, pend, L.norm2_w, L.norm2_b, 1e-5f, w.xn16, pdl, s, true));
        pend = SplitK{};
      }
    }
    return tc_head(D, head, x, st, w, fold, pend, s, post);
  }
  // CUDA-core chain: pre-LN GEMVs normalise their input rows on the fly; post-LN GEMVs read x as it is, and each
  // residual GEMV is followed by the in-place post-norm of x's B rows
  for (int l = 0; l < D.n_layer; ++l) {
    const vb_layer_params &P = dec->layers[l];
    const QkvScatter kv = layer_kv(D, st, l, w.q);
    LnParams ln1{P.norm1_w, P.norm1_b, nullptr, 1e-5f};
    VB_TRY(launch_gemv(x, d, B, P.in_proj_w, dt, P.in_proj_b, 3 * d, d, nullptr, 0, post ? nullptr : &ln1, 3, &kv, s));
    VB_TRY(launch_attn_decode(kv, SplitK{}, B, D.n_head, dt, w.att, nullptr, w.attn_ws, false, s, st->kv_parent,
                              beam_anc(st)));
    VB_TRY(launch_gemv(w.att, d, B, P.out_proj_w, dt, P.out_proj_b, d, d, x, d, nullptr, 2, nullptr, s));
    if (post) VB_TRY(launch_post_norm(x, B, d, P.norm1_w, P.norm1_b, nullptr, 1e-5f, nullptr, VB_F32, s));
    LnParams ln2{P.norm2_w, P.norm2_b, nullptr, 1e-5f};
    VB_TRY(launch_gemv(x, d, B, P.lin1_w, dt, P.lin1_b, dff, d, w.hb, dff, post ? nullptr : &ln2, 1, nullptr, s));
    VB_TRY(launch_gemv(w.hb, dff, B, P.lin2_w, dt, P.lin2_b, d, dff, x, d, nullptr, 2, nullptr, s));
    if (post) VB_TRY(launch_post_norm(x, B, d, P.norm2_w, P.norm2_b, nullptr, 1e-5f, nullptr, VB_F32, s));
  }
  return head_step(dec, head, x, st, workspace, workspace_bytes, s);
}
