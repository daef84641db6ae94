"""LayerNorm / AdaptiveLayerNorm / TransformerEncoderLayer / TransformerEncoder with the
reference's constructor signatures, parameter names (checkpoint layout) and init order
(valle/modules/transformer.py:17-108,178-406).  Forward = libvalle_b200.so:
`NativeDecoder` packs the layer pointers into a `vb_decoder_t` and runs
`vb_decoder_forward` (LN/AdaLN -> QKV GEMM -> ragged attention -> out-proj+residual -> LN ->
FFN1+ReLU -> FFN2+residual per layer).  Pre-LN (`norm_first=True`, the VALL-E default) and post-LN
(`norm_first=False`: QKV GEMM -> attention -> out-proj+residual -> LN -> FFN1+ReLU -> FFN2+residual -> LN,
no final norm in VALLE) stacks.
"""
from __future__ import annotations

import copy
import ctypes as C
import numbers
from typing import Any, Callable, List, Optional, Tuple, Union

import torch
from torch import Tensor, nn
from torch.nn import functional as F

from .. import _lib as L
from .. import ops
from .activation import MultiheadAttention, ValleARMask, classify_attn_mask, pack_rows

_shape_t = Union[int, List[int], torch.Size]


class LayerNorm(nn.Module):
    """valle/modules/transformer.py:17-80: LayerNorm whose forward also accepts (input, embedding) tuples and passes
    the embedding through (:57-74); weight / bias parameters as in the reference.  forward -> vb_layernorm."""
    __constants__ = ["normalized_shape", "eps", "elementwise_affine"]

    def __init__(self, normalized_shape: _shape_t, eps: float = 1e-5, elementwise_affine: bool = True,
                 device=None, dtype=None) -> None:
        super().__init__()
        if isinstance(normalized_shape, numbers.Integral):
            normalized_shape = (normalized_shape,)
        self.normalized_shape = tuple(normalized_shape)
        self.eps = eps
        self.elementwise_affine = elementwise_affine
        if not elementwise_affine:
            raise NotImplementedError("valle_b200.LayerNorm: elementwise_affine=False is not on the VALL-E path")
        self.weight = nn.Parameter(torch.ones(self.normalized_shape, device=device, dtype=dtype))
        self.bias = nn.Parameter(torch.zeros(self.normalized_shape, device=device, dtype=dtype))

    def forward(self, input: Tensor, embedding: Any = None) -> Tensor:
        if isinstance(input, tuple):
            input, embedding = input
            return (_ln(input, self.weight, self.bias, self.eps), embedding)
        assert embedding is None
        return _ln(input, self.weight, self.bias, self.eps)

    def extra_repr(self) -> str:
        return f"{self.normalized_shape}, eps={self.eps}, elementwise_affine={self.elementwise_affine}"


def _ln(x: Tensor, w: Tensor, b: Tensor, eps: float, ada_wb: Optional[Tensor] = None) -> Tensor:
    shp = x.shape
    y = ops.layernorm(x.reshape(-1, shp[-1]).contiguous(), w.detach(), b.detach(), eps, ada_wb)
    return y.view(shp)


class AdaptiveLayerNorm(nn.Module):
    r"""Adaptive Layer Normalization (transformer.py:83-108)."""

    def __init__(self, d_model, norm) -> None:
        super().__init__()
        self.project_layer = nn.Linear(d_model, 2 * d_model)
        self.norm = norm
        self.d_model = d_model
        self.eps = self.norm.eps

    def forward(self, input: Tensor, embedding: Tensor = None) -> Tensor:
        is_tuple = isinstance(input, tuple)
        if is_tuple:
            input, embedding = input
        wb = ops.adaln_project(self.project_layer.weight.detach(), self.project_layer.bias.detach(),
                               embedding.detach().reshape(-1).contiguous())
        y = _ln(input, self.norm.weight, self.norm.bias, self.eps, wb)
        return (y, embedding) if is_tuple else y


class TransformerEncoderLayer(nn.Module):
    """valle/modules/transformer.py:178-334.  Pre-LN (`norm_first=True`, the VALL-E default):
    x += SA(norm1(x)); x += linear2(relu(linear1(norm2(x)))) (:297-302, _sa_block :315, _ff_block :332); post-LN
    (`norm_first=False`): x = norm1(x + SA(x)); x = norm2(x + linear2(relu(linear1(x)))) (:303-308); optional
    AdaptiveLayerNorm wrapping (:238-258).  Same sub-module and parameter names as the reference; a standalone
    forward runs the one-layer native stack, a TransformerEncoder drives all layers through one vb_decoder_t."""
    __constants__ = ["batch_first", "norm_first"]

    def __init__(self, d_model: int, nhead: int, dim_feedforward: int = 2048, dropout: float = 0.1,
                 activation: Union[str, Callable[[Tensor], Tensor]] = F.relu, batch_first: bool = False,
                 norm_first: bool = False, device=None, dtype=None,
                 linear1_self_attention_cls: nn.Module = nn.Linear,
                 linear2_self_attention_cls: nn.Module = nn.Linear,
                 linear1_feedforward_cls: nn.Module = nn.Linear,
                 linear2_feedforward_cls: nn.Module = nn.Linear,
                 layer_norm_cls: nn.Module = LayerNorm, layer_norm_eps: float = 1e-5,
                 adaptive_layer_norm=False) -> None:
        fk = {"device": device, "dtype": dtype}
        super().__init__()
        if activation not in (F.relu, "relu") or layer_norm_cls is not LayerNorm \
                or linear1_feedforward_cls is not nn.Linear or linear2_feedforward_cls is not nn.Linear:
            raise NotImplementedError("valle_b200.TransformerEncoderLayer: only ReLU / LayerNorm / nn.Linear "
                                      "(the configuration VALLE instantiates, valle.py:141-149) is built")
        self.self_attn = MultiheadAttention(d_model, nhead, dropout=dropout, batch_first=batch_first,
                                            linear1_cls=linear1_self_attention_cls,
                                            linear2_cls=linear2_self_attention_cls, **fk)
        self.linear1 = nn.Linear(d_model, dim_feedforward, **fk)
        self.dropout = nn.Dropout(dropout)
        self.linear2 = nn.Linear(dim_feedforward, d_model, **fk)
        self.norm_first = norm_first
        self.dropout1 = nn.Dropout(dropout)
        self.dropout2 = nn.Dropout(dropout)
        self.activation = F.relu
        norm1 = layer_norm_cls(d_model, eps=layer_norm_eps, **fk)
        norm2 = layer_norm_cls(d_model, eps=layer_norm_eps, **fk)
        if adaptive_layer_norm:
            self.norm1 = AdaptiveLayerNorm(d_model, norm1)
            self.norm2 = AdaptiveLayerNorm(d_model, norm2)
        else:
            self.norm1 = norm1
            self.norm2 = norm2

    def forward_packed(self, xp: Tensor, cu: Tensor, max_len: int, B: int, mode: int, tl, dense,
                       ada1: Optional[Tensor], ada2: Optional[Tensor]) -> Tensor:
        """transformer.py:296-308 on packed rows xp [M, d] fp32, operator by operator; returns the output rows.  Pre-LN,
        in place: x += out_proj(SA(norm1(x))); x += linear2(relu(linear1(norm2(x)))).  Post-LN:
        x = norm1(x + out_proj(SA(x))); x = norm2(x + linear2(relu(linear1(x))))."""
        n1 = self.norm1.norm if isinstance(self.norm1, AdaptiveLayerNorm) else self.norm1
        n2 = self.norm2.norm if isinstance(self.norm2, AdaptiveLayerNorm) else self.norm2
        if not self.norm_first:
            o = self.self_attn.attend_packed(xp, cu, max_len, B, mode, tl, dense)
            ops.linear(o, self.self_attn.out_proj.weight.detach(), self.self_attn.out_proj.bias.detach(),
                       epilogue=L.VB_EPI_RESIDUAL, out=xp)
            xp = ops.layernorm(xp, n1.weight.detach(), n1.bias.detach(), n1.eps, ada1)
            f = ops.linear(xp, self.linear1.weight.detach(), self.linear1.bias.detach(), epilogue=L.VB_EPI_RELU)
            ops.linear(f, self.linear2.weight.detach(), self.linear2.bias.detach(), epilogue=L.VB_EPI_RESIDUAL, out=xp)
            return ops.layernorm(xp, n2.weight.detach(), n2.bias.detach(), n2.eps, ada2)
        h = ops.layernorm(xp, n1.weight.detach(), n1.bias.detach(), n1.eps, ada1)
        o = self.self_attn.attend_packed(h, cu, max_len, B, mode, tl, dense)
        ops.linear(o, self.self_attn.out_proj.weight.detach(), self.self_attn.out_proj.bias.detach(),
                   epilogue=L.VB_EPI_RESIDUAL, out=xp)
        h = ops.layernorm(xp, n2.weight.detach(), n2.bias.detach(), n2.eps, ada2)
        f = ops.linear(h, self.linear1.weight.detach(), self.linear1.bias.detach(), epilogue=L.VB_EPI_RELU)
        ops.linear(f, self.linear2.weight.detach(), self.linear2.bias.detach(), epilogue=L.VB_EPI_RESIDUAL, out=xp)
        return xp

    def forward(self, src, src_mask=None, src_key_padding_mask: Optional[Tensor] = None):
        """One layer (transformer.py:296-308) -- runs a 1-layer native stack."""
        enc = TransformerEncoder.__new__(TransformerEncoder)
        nn.Module.__init__(enc)
        enc.layers = nn.ModuleList([self])
        enc.num_layers = 1
        enc.norm = None
        enc._native = {}
        enc.training = self.training
        return enc.forward(src, mask=src_mask, src_key_padding_mask=src_key_padding_mask)


class TransformerEncoder(nn.Module):
    """valle/modules/transformer.py:337-406: N deep-copied layers (+ optional final norm).  forward (:363-406) over
    padded [B, L, d] input maps to one vb_decoder_forward call on packed ragged rows (`NativeDecoder`)."""
    __constants__ = ["norm"]

    def __init__(self, encoder_layer, num_layers, norm=None):
        super().__init__()
        self.layers = nn.ModuleList([copy.deepcopy(encoder_layer) for _ in range(num_layers)])
        self.num_layers = num_layers
        self.norm = norm
        self._native = {}

    # ---- native handle -----------------------------------------------------------------
    def native(self, dtype: torch.dtype = torch.float32) -> "NativeDecoder":
        """the C-side handle of this stack for the given storage dtype (rebuilt when a parameter changed)"""
        nd = self._native.get(dtype)
        if nd is None or nd.stale():
            nd = NativeDecoder(self, dtype)
            self._native[dtype] = nd
        return nd

    def __getstate__(self):
        st = self.__dict__.copy()
        st["_native"] = {}
        return st

    def __deepcopy__(self, memo):
        cls = self.__class__
        new = cls.__new__(cls)
        memo[id(self)] = new
        for k, v in self.__dict__.items():
            new.__dict__[k] = {} if k == "_native" else copy.deepcopy(v, memo)
        return new

    def forward(self, src, mask=None, src_key_padding_mask: Optional[Tensor] = None,
                return_layer_states: bool = False):
        """transformer.py:363-406.  `src` is `x` or `(x, stage_embedding)`; `mask` is None, a ValleARMask or the
        reference's boolean [L, L] `attn_mask` tensor (True = blocked; the VALL-E AR pattern of valle.py:1019-1033
        is recognised and served by the structured kernels, any other pattern by the dense-mask kernel);
        `src_key_padding_mask` a bool [B, L] suffix-padding mask.  `return_layer_states=True` returns
        (layer_states, output) as transformer.py:368-381 does."""
        if self.training and torch.is_grad_enabled():
            raise NotImplementedError("valle_b200.TransformerEncoder: the module-level forward is inference only "
                                      "(training goes through VALLE.forward); call .eval()")
        is_tuple = isinstance(src, tuple)
        x, stage = src if is_tuple else (src, None)
        B, Lq, d = x.shape
        dev = x.device
        with torch.cuda.device(dev):
            idx, cu, lens = pack_rows(B, Lq, src_key_padding_mask, dev)
            xp = x.reshape(B * Lq, d).to(torch.float32).index_select(0, idx).contiguous()
            mode, tl, dense = classify_attn_mask(mask, Lq)
            max_len = int(lens.max())

            def unpack(t):
                out = torch.zeros((B * Lq, d), dtype=torch.float32, device=dev)
                out.index_copy_(0, idx, t)
                return out.view(B, Lq, d)

            nd = self.native(torch.float32)
            ada = nd.ada_table(stage) if stage is not None else None
            if mode != L.VB_MASK_DENSE and not return_layer_states:
                if mode == L.VB_MASK_VALLE_AR:
                    tl = (torch.full((B,), tl, dtype=torch.int32) if isinstance(tl, int) else tl).to(
                        device=dev, dtype=torch.int32)
                nd.forward(xp, cu, B, max_len, mode, tl, ada)   # the whole stack in one C call
                if self.norm is not None:
                    xp = nd.final_norm(xp, ada)
                out = unpack(xp)
                return (out, stage) if is_tuple else out
            # layer by layer through the operator surface (dense masks, per-layer states)
            states = []
            for i, lyr in enumerate(self.layers):
                xp = lyr.forward_packed(xp, cu, max_len, B, mode, tl, dense,
                                        None if ada is None else ada[2 * i], None if ada is None else ada[2 * i + 1])
                if return_layer_states:
                    states.append(unpack(xp))
            if self.norm is not None:
                xp = nd.final_norm(xp, ada)
            out = unpack(xp)
            if return_layer_states:
                return states, ((out, stage) if is_tuple else out)
            return (out, stage) if is_tuple else out


class NativeDecoder:
    """Owns a `vb_decoder_t` for one TransformerEncoder at one storage dtype.

    fp32: the handle points straight at the nn.Parameters (zero copy).  bf16: the four big
    matrices of every layer are kept as packed bf16 copies (re-made when a parameter changes)."""

    def __init__(self, enc: TransformerEncoder, dtype: torch.dtype):
        self.lib = L.load()
        self.dtype = dtype
        self.enc = enc
        l0 = enc.layers[0]
        self.d = l0.self_attn.embed_dim
        self.H = l0.self_attn.num_heads
        self.dff = l0.linear1.out_features
        self.n_layer = len(enc.layers)
        self.adaptive = isinstance(l0.norm1, AdaptiveLayerNorm)
        self.norm_first = bool(l0.norm_first)
        dev = l0.linear1.weight.device
        if dev.type != "cuda":
            raise L.VbError("valle_b200: the model must live on a CUDA device (no CPU fallback)")
        self.device = dev
        self._keep = []
        self._bf16 = {}   # data_ptr -> packed bf16 copy of a big matrix
        self._sig = self._signature()

        def big(p):
            t = p.detach()
            if t.dtype != torch.float32 or not t.is_contiguous():
                raise L.VbError("valle_b200: parameters must be contiguous fp32")
            if dtype == torch.bfloat16:
                t = t.to(torch.bfloat16).contiguous()
                self._bf16[t.data_ptr()] = t
            self._keep.append(t)
            return t.data_ptr()

        def small(p):
            t = p.detach()
            self._keep.append(t)
            return t.data_ptr()

        arr = (L.LayerParams * self.n_layer)()
        for i, lyr in enumerate(enc.layers):
            n1 = lyr.norm1.norm if self.adaptive else lyr.norm1
            n2 = lyr.norm2.norm if self.adaptive else lyr.norm2
            a = arr[i]
            a.in_proj_w = big(lyr.self_attn.in_proj_weight)
            a.in_proj_b = small(lyr.self_attn.in_proj_bias)
            a.out_proj_w = big(lyr.self_attn.out_proj.weight)
            a.out_proj_b = small(lyr.self_attn.out_proj.bias)
            a.lin1_w = big(lyr.linear1.weight)
            a.lin1_b = small(lyr.linear1.bias)
            a.lin2_w = big(lyr.linear2.weight)
            a.lin2_b = small(lyr.linear2.bias)
            a.norm1_w, a.norm1_b = small(n1.weight), small(n1.bias)
            a.norm2_w, a.norm2_b = small(n2.weight), small(n2.bias)
        self._layers = arr
        desc = L.DecoderDesc()
        desc.d_model, desc.n_head, desc.n_layer, desc.d_ff = self.d, self.H, self.n_layer, self.dff
        desc.wdtype = L.VB_BF16 if dtype == torch.bfloat16 else L.VB_F32
        desc.layers = arr
        desc.norm_first = int(self.norm_first)
        fn = enc.norm
        if fn is not None:
            inner = fn.norm if isinstance(fn, AdaptiveLayerNorm) else fn
            desc.final_norm_w, desc.final_norm_b = small(inner.weight), small(inner.bias)
            self.final_w, self.final_b, self.final_eps = inner.weight.detach(), inner.bias.detach(), inner.eps
        self.desc = desc
        h = C.c_void_p()
        L.check(self.lib.vb_decoder_create(C.byref(desc), C.byref(h)), "vb_decoder_create")
        self.handle = h
        self._ws = None

    def __del__(self):
        try:
            if getattr(self, "handle", None):
                self.lib.vb_decoder_destroy(self.handle)
                self.handle = None
        except Exception:
            pass

    def _signature(self):
        return tuple((p.data_ptr(), p._version) for p in self.enc.parameters())

    def fold_layernorm(self, w16: Tensor, gamma: Tensor, beta: Tensor, bias: Optional[Tensor]) -> "L.LnFold":
        """vb_ln_fold_build: LayerNorm(gamma, beta) folded into the bf16 projection w16 [N, K] (+ bias) that consumes
        it -- wf = w16 * gamma, c = row sums of wf, dvec = bias + w16 @ beta (include/valle_b200.h vb_ln_fold)"""
        N, K = w16.shape
        wf = torch.empty_like(w16)
        c = torch.empty(N, dtype=torch.float32, device=w16.device)
        dv = torch.empty(N, dtype=torch.float32, device=w16.device)
        with torch.cuda.device(self.device):
            L.check(self.lib.vb_ln_fold_build(w16.data_ptr(), N, K, gamma.data_ptr(), beta.data_ptr(), L.ptr(bias),
                                              wf.data_ptr(), c.data_ptr(), dv.data_ptr(), L.stream_ptr()),
                    "vb_ln_fold_build")
        self._keep += [wf, c, dv]
        f = L.LnFold()
        f.wf, f.c, f.dvec = wf.data_ptr(), c.data_ptr(), dv.data_ptr()
        return f

    def enable_decode_fold(self) -> bool:
        """bf16 AR decode chain without the residual + LayerNorm launches (valle/modules/transformer.py:296-302): norm1
        is folded into in_proj and norm2 into linear1 of every layer (plain LayerNorm only).  Returns False (chain left
        as it is) for fp32 storage, for AdaptiveLayerNorm stacks and for post-LN stacks (their norms follow the
        residual add instead of feeding a projection)."""
        if self.dtype != torch.bfloat16 or self.adaptive or not self.norm_first:
            return False
        qkv = (L.LnFold * self.n_layer)()
        ffn1 = (L.LnFold * self.n_layer)()
        for i, lyr in enumerate(self.enc.layers):
            a = self._layers[i]
            w_in = self._bf16[a.in_proj_w]
            w_l1 = self._bf16[a.lin1_w]
            qkv[i] = self.fold_layernorm(w_in, lyr.norm1.weight.detach(), lyr.norm1.bias.detach(),
                                         lyr.self_attn.in_proj_bias.detach())
            ffn1[i] = self.fold_layernorm(w_l1, lyr.norm2.weight.detach(), lyr.norm2.bias.detach(),
                                          lyr.linear1.bias.detach())
        L.check(self.lib.vb_decoder_set_decode_fold(self.handle, qkv, ffn1), "vb_decoder_set_decode_fold")
        return True

    def stale(self) -> bool:
        return self._sig != self._signature()

    # ---- AdaLN (weight|bias) rows for one stage embedding: [(2L+1), 2d] fp32 (2L rows without a final norm) ----
    def ada_table(self, stage_emb: Tensor) -> Tensor:
        assert self.adaptive
        e = stage_emb.detach().reshape(-1).contiguous()
        rows = 2 * self.n_layer + int(self.enc.norm is not None)
        tab = torch.empty((rows, 2 * self.d), dtype=torch.float32, device=self.device)
        r = 0
        for lyr in self.enc.layers:
            for nm in (lyr.norm1, lyr.norm2):
                ops.adaln_project(nm.project_layer.weight.detach(), nm.project_layer.bias.detach(), e, tab[r])
                r += 1
        fn = self.enc.norm
        if isinstance(fn, AdaptiveLayerNorm):
            ops.adaln_project(fn.project_layer.weight.detach(), fn.project_layer.bias.detach(), e, tab[r])
        return tab

    def transposed(self):
        """(vb_layer_wt array, keep-alive list): the four matrices of every layer transposed, in the storage dtype --
        the weight operands of the input-gradient GEMMs of vb_decoder_backward"""
        arr = (L.LayerWt * self.n_layer)()
        keep = []
        for i, lyr in enumerate(self.enc.layers):
            for name, p in (("in_proj_wt", lyr.self_attn.in_proj_weight), ("out_proj_wt", lyr.self_attn.out_proj.weight),
                            ("lin1_wt", lyr.linear1.weight), ("lin2_wt", lyr.linear2.weight)):
                t = p.detach().to(self.dtype).t().contiguous()
                keep.append(t)
                setattr(arr[i], name, t.data_ptr())
        self._wt_keep = keep
        return arr, keep

    def workspace(self, nbytes: int) -> Tensor:
        if self._ws is None or self._ws.numel() < nbytes:
            self._ws = torch.empty(nbytes, dtype=torch.uint8, device=self.device)
        return self._ws

    def forward(self, x: Tensor, cu_seqlens: Tensor, B: int, max_seqlen: int, mask_mode: int,
                text_lens: Optional[Tensor], ada: Optional[Tensor], kcache: Optional[Tensor] = None,
                vcache: Optional[Tensor] = None, cache_cap: int = 0, seg1_lens: Optional[Tensor] = None,
                seg1_start: int = 0, k_exp: Optional[Tensor] = None, v_exp: Optional[Tensor] = None,
                cache_slots: Optional[Tensor] = None) -> Tensor:
        """In-place stack forward over packed rows x [M, d] fp32 (no final norm): one vb_decoder_forward call.
        kcache / vcache ([n_layer, B, H, cap, hd]) given: the attention fills them.  k_exp / v_exp (uint8 [n_layer, B,
        H, cap]) given: kcache / vcache are the FP8 cache (torch.float8_e4m3fn, include/valle_b200.h "FP8 (e4m3) KV
        cache").  cache_slots (device int32 [B]) given: sequence b fills cache stream cache_slots[b]."""
        M = x.shape[0]
        ws = self.workspace(self.lib.vb_decoder_forward_workspace(C.byref(self.desc), M))
        ls, ss = (kcache.stride(0), kcache.stride(1)) if kcache is not None else (0, 0)
        L.check(self.lib.vb_decoder_forward(self.handle, x.data_ptr(), M, B, cu_seqlens.data_ptr(), L.ptr(text_lens),
                                            L.ptr(seg1_lens), seg1_start, max_seqlen, mask_mode, L.ptr(ada),
                                            L.ptr(kcache), L.ptr(vcache), L.ptr(k_exp), L.ptr(v_exp), ls, ss, cache_cap,
                                            L.ptr(cache_slots), ws.data_ptr(), ws.numel(), L.stream_ptr()),
                "vb_decoder_forward")
        return x

    def final_norm(self, x: Tensor, ada: Optional[Tensor], rows: Optional[Tensor] = None,
                   out_dtype: torch.dtype = torch.float32) -> Tensor:
        wb = ada[2 * self.n_layer] if ada is not None else None
        return ops.layernorm(x, self.final_w, self.final_b, self.final_eps, wb, rows, out_dtype)

    def head_rows(self, x: Tensor, ada: Optional[Tensor], rows: Tensor, out_dtype: torch.dtype) -> Tensor:
        """the prediction head's operand: the stack output rows x[rows], through the final norm if the stack has one
        (valle.py:1128), else as they are (post-LN, valle.py:242-246: no final norm), in out_dtype"""
        if self.enc.norm is not None:
            return self.final_norm(x, ada, rows, out_dtype)
        h = ops.gather_rows(x, rows)
        return h if out_dtype == torch.float32 else ops.cast_from_f32(h, out_dtype)
