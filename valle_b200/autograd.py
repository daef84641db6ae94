"""torch.autograd bridges for the training path (VALLE.forward -> loss.backward(), valle/bin/trainer.py:674).

Every Function runs the forward kernels of libvalle_b200.so and, in backward, the hand-written gradient kernels
(csrc/backward.cu, vb_decoder_backward): torch only records the graph, owns the tensors and accumulates `.grad`.
Dropout is not applied (p treated as 0): the reference's training-mode dropout draws from torch's RNG inside
kernels this engine replaces; see DESIGN.md.
"""
from __future__ import annotations

import ctypes as C
from typing import List, Optional, Sequence

import torch

from . import _lib as L
from . import ops

_DT = {torch.float32: L.VB_F32, torch.bfloat16: L.VB_BF16}


def _s() -> int:
    return torch.cuda.current_stream().cuda_stream


def _pad64(n: int) -> int:
    return (n + 63) // 64 * 64


class EmbedSum(torch.autograd.Function):
    """out[r] = sum_j tables[j][tokens[r, j]] (TokenEmbedding + the codebook sum of valle.py:335-393,1064)"""

    @staticmethod
    def forward(ctx, tokens, tok_row_stride, tok_tab_stride, n_rows, *tables):
        d = tables[0].shape[1]
        out = torch.empty((n_rows, d), dtype=torch.float32, device=tables[0].device)
        ops.embed_sum(tokens, tok_row_stride, tok_tab_stride, [t.detach() for t in tables], n_rows, out)
        ctx.save_for_backward(tokens)
        ctx.meta = (tok_row_stride, tok_tab_stride, n_rows, [tuple(t.shape) for t in tables], tables[0].device)
        return out

    @staticmethod
    def backward(ctx, dy):
        (tokens,) = ctx.saved_tensors
        rs, ts, n_rows, shapes, dev = ctx.meta
        dy = dy.contiguous()
        grads = [torch.zeros(s, dtype=torch.float32, device=dev) for s in shapes]
        arr = (C.c_void_p * len(grads))(*[g.data_ptr() for g in grads])
        rows = (C.c_int32 * len(grads))(*[s[0] for s in shapes])
        with torch.cuda.device(dev):
            L.check(L.load().vb_embed_backward(tokens.data_ptr(), rs, ts, arr, rows, len(grads), n_rows, shapes[0][1],
                                               dy.data_ptr(), dy.stride(0), 0, _s()), "vb_embed_backward")
        return (None, None, None, None, *grads)


class AddPe(torch.autograd.Function):
    """SinePositionalEmbedding.forward (embedding.py:93-97, scale=False): x [N, T, d] + alpha * pe[:T]"""

    @staticmethod
    def forward(ctx, x, pe, alpha):
        N, T, d = x.shape
        x = x.contiguous()
        out = torch.empty_like(x)
        for b in range(N):
            ops.add_pe(x[b], pe, alpha.detach(), out[b], T, pos0=0)
        ctx.save_for_backward(pe)
        ctx.alpha_grad = alpha.requires_grad
        return out

    @staticmethod
    def backward(ctx, dy):
        (pe,) = ctx.saved_tensors
        dalpha = None
        if ctx.alpha_grad:
            dy = dy.contiguous()
            N, T, d = dy.shape
            dalpha = torch.zeros(1, dtype=torch.float32, device=dy.device)
            with torch.cuda.device(dy.device):
                for b in range(N):
                    L.check(L.load().vb_rowdot_accumulate(dy[b].data_ptr(), d, pe.data_ptr(), 0, 0, T, d,
                                                          dalpha.data_ptr(), _s()), "vb_rowdot_accumulate")
        return dy, None, dalpha


class AdaTable(torch.autograd.Function):
    """(weight | bias) rows of every AdaptiveLayerNorm of a stack for one stage embedding (transformer.py:96-100):
    table[r] = W_r e + b_r, r = 2l (norm1 of layer l), 2l+1 (norm2), last = final norm"""

    @staticmethod
    def forward(ctx, emb, *wb):  # wb = W_0, b_0, W_1, b_1, ...
        e = emb.detach().reshape(-1).contiguous()
        n = len(wb) // 2
        d = e.numel()
        tab = torch.empty((n, 2 * d), dtype=torch.float32, device=e.device)
        for r in range(n):
            ops.adaln_project(wb[2 * r].detach(), wb[2 * r + 1].detach(), e, tab[r])
        ctx.save_for_backward(e, *[w.detach() for w in wb[0::2]])
        ctx.emb_shape = emb.shape
        return tab

    @staticmethod
    def backward(ctx, dtab):
        e, *Ws = ctx.saved_tensors
        d = e.numel()
        dtab = dtab.contiguous()
        de = torch.zeros(d, dtype=torch.float32, device=e.device)
        out = []
        lib = L.load()
        with torch.cuda.device(e.device):
            for r, W in enumerate(Ws):
                dW = torch.zeros_like(W)
                db = torch.zeros(2 * d, dtype=torch.float32, device=e.device)
                L.check(lib.vb_adaln_project_backward(W.data_ptr(), e.data_ptr(), dtab[r].data_ptr(), d, dW.data_ptr(),
                                                      db.data_ptr(), de.data_ptr(), _s()), "vb_adaln_project_backward")
                out += [dW, db]
        return (de.view(ctx.emb_shape), *out)


class LayerNormRows(torch.autograd.Function):
    """vb_layernorm over gathered rows (final LayerNorm / AdaptiveLayerNorm of a stack before the prediction head)"""

    @staticmethod
    def forward(ctx, x, gamma, beta, ada_wb, rows, eps, out_dtype):
        y = ops.layernorm(x, gamma.detach(), beta.detach(), eps, None if ada_wb is None else ada_wb.detach(), rows, out_dtype)
        ctx.save_for_backward(x, gamma.detach(), beta.detach(), ada_wb.detach() if ada_wb is not None else None, rows)
        ctx.eps = eps
        return y

    @staticmethod
    def backward(ctx, dy):
        x, gamma, beta, ada, rows = ctx.saved_tensors
        M, d = x.shape
        dy = dy.to(torch.float32).contiguous()
        n = dy.shape[0]
        dx = torch.zeros_like(x)
        dg, db = torch.zeros_like(gamma), torch.zeros_like(beta)
        dada = torch.zeros_like(ada) if ada is not None else None
        with torch.cuda.device(x.device):
            L.check(L.load().vb_layernorm_backward(x.data_ptr(), x.stride(0), L.ptr(rows), n, d, gamma.data_ptr(),
                                                   beta.data_ptr(), L.ptr(ada), ctx.eps, dy.data_ptr(), dy.stride(0),
                                                   dx.data_ptr(), dx.stride(0), 0, L.VB_F32, dg.data_ptr(), db.data_ptr(),
                                                   L.ptr(dada), _s()), "vb_layernorm_backward")
        return dx, dg, db, dada, None, None, None


class GatherRows(torch.autograd.Function):
    """the head operand of a stack without a final norm (post-LN): rows x[rows] in out_dtype; the gradient goes back to
    those rows (zero elsewhere)"""

    @staticmethod
    def forward(ctx, x, rows, out_dtype):
        y = ops.gather_rows(x, rows)
        if out_dtype != torch.float32:
            y = ops.cast_from_f32(y, out_dtype)
        ctx.save_for_backward(rows)
        ctx.n_src = x.shape[0]
        return y

    @staticmethod
    def backward(ctx, dy):
        (rows,) = ctx.saved_tensors
        src = torch.full((ctx.n_src,), -1, dtype=torch.int32, device=rows.device)   # -1: a zero row (vb_gather_rows)
        src[rows.long()] = torch.arange(rows.numel(), dtype=torch.int32, device=rows.device)
        return ops.gather_rows(dy.to(torch.float32).contiguous(), src), None, None


class Linear(torch.autograd.Function):
    """F.linear without bias for the prediction heads (valle.py:870,929): logits fp32 = a @ w^T, operands in the
    engine dtype"""

    @staticmethod
    def forward(ctx, a, w, dtype):
        wc = w.detach() if dtype == torch.float32 else w.detach().to(dtype)
        out = ops.linear(a, wc, None, out_dtype=torch.float32)
        ctx.save_for_backward(a, wc)
        ctx.dtype = dtype
        return out

    @staticmethod
    def backward(ctx, dy):
        a, wc = ctx.saved_tensors
        dtype = ctx.dtype
        M, K = a.shape
        N = wc.shape[0]
        Np = _pad64(N)
        dev = a.device
        dyp = torch.zeros((M, Np), dtype=dtype, device=dev)
        dyp[:, :N] = dy.to(dtype)
        wt = torch.zeros((K, Np), dtype=dtype, device=dev)
        wt[:, :N] = wc.t()
        da = torch.empty((M, K), dtype=torch.float32, device=dev)
        dw = torch.zeros((Np, K), dtype=torch.float32, device=dev)
        lib = L.load()
        with torch.cuda.device(dev):
            nb = lib.vb_linear_backward_workspace(_DT[dtype], M, Np, K)
            ws = torch.empty(nb, dtype=torch.uint8, device=dev)
            L.check(lib.vb_linear_backward(a.data_ptr(), _DT[dtype], a.stride(0), wt.data_ptr(), dyp.data_ptr(), Np,
                                           da.data_ptr(), L.VB_F32, K, L.VB_EPI_NONE, dw.data_ptr(), 0, M, Np, K,
                                           ws.data_ptr(), nb, _s()), "vb_linear_backward")
        return da.to(a.dtype), dw[:N], None


class CrossEntropySum(torch.autograd.Function):
    """F.cross_entropy(..., reduction="sum", ignore_index) over rows (valle.py:877,936-941)"""

    @staticmethod
    def forward(ctx, logits, targets, ignore_index):
        loss = ops.cross_entropy_rows(logits, targets, ignore_index=ignore_index).sum()
        ctx.save_for_backward(logits, targets)
        ctx.ignore = ignore_index
        return loss

    @staticmethod
    def backward(ctx, g):
        logits, targets = ctx.saved_tensors
        n, V = logits.shape
        dl = torch.empty_like(logits)
        grow = g.to(torch.float32).reshape(1).expand(n).contiguous()
        with torch.cuda.device(logits.device):
            L.check(L.load().vb_cross_entropy_backward(logits.data_ptr(), logits.stride(0), targets.data_ptr(), n, V,
                                                       ctx.ignore, grow.data_ptr(), 1.0, dl.data_ptr(), L.VB_F32,
                                                       dl.stride(0), V, _s()), "vb_cross_entropy_backward")
        return dl, None, None


_LAYER_PARAM_ORDER = ("in_proj_w", "in_proj_b", "out_proj_w", "out_proj_b", "lin1_w", "lin1_b", "lin2_w", "lin2_b",
                      "norm1_w", "norm1_b", "norm2_w", "norm2_b")


def layer_params(enc) -> List[torch.Tensor]:
    """the 12 tensors of every layer in vb_layer_params order (inner norm of an AdaptiveLayerNorm)"""
    from .modules.transformer import AdaptiveLayerNorm
    out = []
    for lyr in enc.layers:
        n1 = lyr.norm1.norm if isinstance(lyr.norm1, AdaptiveLayerNorm) else lyr.norm1
        n2 = lyr.norm2.norm if isinstance(lyr.norm2, AdaptiveLayerNorm) else lyr.norm2
        out += [lyr.self_attn.in_proj_weight, lyr.self_attn.in_proj_bias, lyr.self_attn.out_proj.weight,
                lyr.self_attn.out_proj.bias, lyr.linear1.weight, lyr.linear1.bias, lyr.linear2.weight, lyr.linear2.bias,
                n1.weight, n1.bias, n2.weight, n2.bias]
    return out


class DecoderStack(torch.autograd.Function):
    """TransformerEncoder layers (no final norm) over packed rows: vb_decoder_forward_train / vb_decoder_backward"""

    @staticmethod
    def forward(ctx, x, ada, nd, geom, *params):
        cu, B, max_len, mode, tl, seg1, seg1_start = geom[:7]
        drop_p, drop_seed = (geom[7], geom[8]) if len(geom) > 7 else (0.0, 0)   # training-mode dropout of the layers
        lib = L.load()
        x = x.detach().clone().contiguous()
        M = x.shape[0]
        with torch.cuda.device(x.device):
            nb = lib.vb_decoder_train_save_bytes(C.byref(nd.desc), M)
            save = torch.empty(nb, dtype=torch.uint8, device=x.device)
            L.check(lib.vb_decoder_forward_train(nd.handle, x.data_ptr(), M, B, cu.data_ptr(), L.ptr(tl), L.ptr(seg1),
                                                 seg1_start, max_len, mode, L.ptr(ada), save.data_ptr(), nb,
                                                 float(drop_p), int(drop_seed), _s()),
                    "vb_decoder_forward_train")
        ctx.nd, ctx.geom, ctx.save = nd, geom, save
        ctx.drop = (float(drop_p), int(drop_seed))
        ctx.ada = ada.detach() if ada is not None else None
        ctx.shapes = [tuple(p.shape) for p in params]
        return x

    @staticmethod
    def backward(ctx, dy):
        nd, (cu, B, max_len, mode, tl, seg1, seg1_start) = ctx.nd, ctx.geom[:7]
        lib = L.load()
        dev = dy.device
        dx = dy.detach().to(torch.float32).clone().contiguous()
        M = dx.shape[0]
        grads = [torch.zeros(s, dtype=torch.float32, device=dev) for s in ctx.shapes]
        garr = (L.LayerGrads * nd.n_layer)()
        for l in range(nd.n_layer):
            for j, name in enumerate(_LAYER_PARAM_ORDER):
                setattr(garr[l], name, grads[12 * l + j].data_ptr())
        dada = torch.zeros_like(ctx.ada) if ctx.ada is not None else None
        wt, keep = nd.transposed()
        with torch.cuda.device(dev):
            nb = lib.vb_decoder_backward_workspace(C.byref(nd.desc), M)
            ws = torch.empty(nb, dtype=torch.uint8, device=dev)
            L.check(lib.vb_decoder_backward(nd.handle, dx.data_ptr(), M, B, cu.data_ptr(), L.ptr(tl), L.ptr(seg1),
                                            seg1_start, max_len, mode, L.ptr(ctx.ada), L.ptr(dada), ctx.save.data_ptr(),
                                            wt, garr, ws.data_ptr(), nb, ctx.drop[0], ctx.drop[1], _s()),
                    "vb_decoder_backward")
        ctx.save = None
        return (dx, dada, None, None, *grads)


class Dropout(torch.autograd.Function):
    """nn.Dropout after the positional encoding (valle/modules/embedding.py:97) on the library's stateless mask:
    vb_dropout forward, the same call on the gradient backward."""

    @staticmethod
    def forward(ctx, x, p, seed, stream_id):
        x = x.contiguous()
        out = torch.empty_like(x)
        with torch.cuda.device(x.device):
            L.check(L.load().vb_dropout(x.data_ptr(), out.data_ptr(), _DT[x.dtype], x.numel(), float(p), int(seed),
                                        int(stream_id), _s()), "vb_dropout")
        ctx.cfg = (float(p), int(seed), int(stream_id))
        return out

    @staticmethod
    def backward(ctx, dy):
        dy = dy.contiguous()
        dx = torch.empty_like(dy)
        p, seed, sid = ctx.cfg
        with torch.cuda.device(dy.device):
            L.check(L.load().vb_dropout(dy.data_ptr(), dx.data_ptr(), _DT[dy.dtype], dy.numel(), p, seed, sid, _s()),
                    "vb_dropout")
        return dx, None, None, None
