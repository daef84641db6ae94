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


#: dropout site ids of the pre-nets (csrc/kernels.cuh::drop_keep): PRENET_STREAM | site << 4 | dropout index; the
#: decoder layers use (layer << 2) | k and the positional encodings 0x10000 + k
PRENET_STREAM = 0x20000
PRENET_SITES = {"ar_text": 0, "nar_text": 1, "ar_audio": 2, "nar_audio": 3}
_TEXT_BLOCKS = (1, 5, 9)   # Conv1d indices of the text pre-net Sequential (valle.py:97-113); BatchNorm1d at +1, Dropout +3


def text_prenet_params(seq) -> List[torch.Tensor]:
    """(conv weight, conv bias, BatchNorm weight, BatchNorm bias) of the three blocks, then the Linear's weight, bias"""
    out = []
    for i in _TEXT_BLOCKS:
        out += [seq[i].weight, seq[i].bias, seq[i + 1].weight, seq[i + 1].bias]
    return out + [seq[14].weight, seq[14].bias]


def audio_prenet_params(seq) -> List[torch.Tensor]:
    return [seq[0].weight, seq[0].bias, seq[3].weight, seq[3].bias, seq[6].weight, seq[6].bias]


def _linear_grads(x, w, dy, dx, dw, db):
    """vb_linear_backward of y = x w^T + b, x / w / dy in one dtype: dx = dy w (None: skipped), dw += dy^T x,
    db += column sums of dy (None: skipped)"""
    lib = L.load()
    M, K = x.shape
    N = w.shape[0]
    dt = _DT[x.dtype]
    wt = w.t().contiguous()
    nb = lib.vb_linear_backward_workspace(dt, M, N, K)
    ws = torch.empty(nb, dtype=torch.uint8, device=x.device)
    L.check(lib.vb_linear_backward(x.data_ptr(), dt, x.stride(0), wt.data_ptr(), dy.data_ptr(), dy.stride(0),
                                   L.ptr(dx), _DT[dx.dtype] if dx is not None else L.VB_F32,
                                   dx.stride(0) if dx is not None else K, L.VB_EPI_NONE, dw.data_ptr(), L.ptr(db), M, N,
                                   K, ws.data_ptr(), nb, _s()), "vb_linear_backward")


class TextPrenet(torch.autograd.Function):
    """The text pre-net (valle.py:96-113) over the embedded, padded text batch e [N * seg_len, C] fp32: three
    Conv1d(k=5, "same") -> BatchNorm1d -> ReLU -> Dropout blocks and a Linear, GEMM operands in `dtype`.  BatchNorm
    follows the module's mode: train() normalises by the batch statistics over all rows (padding included) and updates
    the running statistics in place, eval() uses the running statistics.  Dropout is live in train() with the
    library's stateless mask.  Backward: the gradients of every pre-net parameter and of e."""

    @staticmethod
    def forward(ctx, e, seq, seg_len, dtype, drop_seed, site, *params):
        lib = L.load()
        dev = e.device
        e = e.detach().contiguous()
        M, C_ = e.shape
        dt = _DT[dtype]
        training = bool(seq.training)
        if training and M < 2:
            raise ValueError(f"Expected more than 1 value per channel when training, got input size [1, {C_}, 1]")
        if any(seq[j + 1].momentum is None for j in _TEXT_BLOCKS):
            raise NotImplementedError("valle_b200: BatchNorm1d(momentum=None) is not built")
        nb = lib.vb_batchnorm_workspace(M, C_)
        ws = torch.empty(nb, dtype=torch.uint8, device=dev)
        col = torch.empty((M, 5 * C_), dtype=dtype, device=dev)
        blocks = []
        with torch.cuda.device(dev):
            L.check(lib.vb_batchnorm_forward(e.data_ptr(), M, C_, seg_len, 0, 0, 0, 0, 0.0, 0.0, 0, 0, 0, 0.0, 0, 0,
                                             col.data_ptr(), dt, 5, 0, 0, _s()), "vb_batchnorm_forward")
            for i, j in enumerate(_TEXT_BLOCKS):
                conv, bn, drop = seq[j], seq[j + 1], seq[j + 3]
                w = conv.weight.detach().permute(0, 2, 1).reshape(C_, 5 * C_).to(dtype).contiguous()
                h = ops.linear(col, w, conv.bias.detach(), out_dtype=torch.float32)
                mean = torch.empty(C_, dtype=torch.float32, device=dev)
                rstd = torch.empty_like(mean)
                taps = 5 if i < 2 else 1
                nxt = torch.empty((M, taps * C_), dtype=dtype, device=dev)
                p = float(drop.p) if training else 0.0
                sid = PRENET_STREAM | (site << 4) | i
                L.check(lib.vb_batchnorm_forward(h.data_ptr(), M, C_, seg_len, bn.weight.data_ptr(), bn.bias.data_ptr(),
                                                 bn.running_mean.data_ptr(), bn.running_var.data_ptr(), float(bn.eps),
                                                 float(bn.momentum), int(training), mean.data_ptr(), rstd.data_ptr(), p,
                                                 int(drop_seed), sid, nxt.data_ptr(), dt, taps, ws.data_ptr(), nb,
                                                 _s()), "vb_batchnorm_forward")
                if training:
                    # the running statistics changed in place; this bump also moves the engine's weight signature
                    bn.num_batches_tracked.add_(1)
                blocks.append((col, w, h, mean, rstd, p, sid))
                col = nxt
            wl = seq[14].weight.detach().to(dtype).contiguous()
            out = ops.linear(col, wl, seq[14].bias.detach(), out_dtype=torch.float32)
        ctx.blocks, ctx.last = blocks, (col, wl)
        ctx.cfg = (seq, seg_len, dtype, training, int(drop_seed))
        return out

    @staticmethod
    def backward(ctx, dout):
        lib = L.load()
        seq, seg_len, dtype, training, seed = ctx.cfg
        dev = dout.device
        col3, wl = ctx.last
        M, C_ = col3.shape
        dt = _DT[dtype]
        nb = lib.vb_batchnorm_workspace(M, C_)
        ws = torch.empty(nb, dtype=torch.uint8, device=dev)
        f32 = dict(dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            dl_w, dl_b = torch.zeros((C_, C_), **f32), torch.zeros(C_, **f32)
            dy, taps = torch.empty((M, C_), **f32), 1
            _linear_grads(col3, wl, ops.cast_from_f32(dout.to(torch.float32).contiguous(), dtype), dy, dl_w, dl_b)
            grads = [None] * 3
            for i in (2, 1, 0):
                col, w, h, mean, rstd, p, sid = ctx.blocks[i]
                bn = seq[_TEXT_BLOCKS[i] + 1]
                dh = torch.empty((M, C_), dtype=dtype, device=dev)
                dg, dbeta, dbias = (torch.empty(C_, **f32) for _ in range(3))
                L.check(lib.vb_batchnorm_backward(dy.data_ptr(), taps, h.data_ptr(), M, C_, seg_len, bn.weight.data_ptr(),
                                                  bn.bias.data_ptr(), mean.data_ptr(), rstd.data_ptr(), int(training), p,
                                                  seed, sid, dh.data_ptr(), dt, dg.data_ptr(), dbeta.data_ptr(),
                                                  dbias.data_ptr(), ws.data_ptr(), nb, _s()), "vb_batchnorm_backward")
                dcol, dw = torch.empty((M, 5 * C_), **f32), torch.zeros((C_, 5 * C_), **f32)
                _linear_grads(col, w, dh, dcol, dw, None)   # the conv bias gradient came from the BatchNorm kernel
                grads[i] = [dw.view(C_, 5, C_).permute(0, 2, 1).contiguous(), dbias, dg, dbeta]
                dy, taps = dcol, 5
            de = torch.empty((M, C_), **f32)
            L.check(lib.vb_batchnorm_backward(dy.data_ptr(), 5, 0, M, C_, seg_len, 0, 0, 0, 0, 0, 0.0, 0, 0,
                                              de.data_ptr(), L.VB_F32, 0, 0, 0, 0, 0, _s()), "vb_batchnorm_backward")
        ctx.blocks = ctx.last = None
        return (de, None, None, None, None, None, *grads[0], *grads[1], *grads[2], dl_w, dl_b)


class AudioPrenet(torch.autograd.Function):
    """The audio pre-net (valle.py:114-123) per row of x [R, C] fp32: Linear(C, 256) -> ReLU -> Dropout ->
    Linear(256, 256) -> ReLU -> Dropout -> Linear(256, C), GEMM operands in `dtype`, dropout live in train()."""

    @staticmethod
    def forward(ctx, x, seq, dtype, drop_seed, site, w1, b1, w2, b2, w3, b3):
        lib = L.load()
        dev = x.device
        x = x.detach().contiguous()
        a = x if dtype == torch.float32 else ops.cast_from_f32(x, dtype)
        ws_ = [w.detach().to(dtype).contiguous() for w in (w1, w2, w3)]
        saved = [a]
        drops = []
        with torch.cuda.device(dev):
            for j, (w, b) in enumerate(zip(ws_[:2], (b1, b2))):
                h = ops.linear(a, w, b.detach(), L.VB_EPI_RELU)
                p = float(seq[3 * j + 2].p) if seq.training else 0.0
                sid = PRENET_STREAM | (site << 4) | j
                a = h
                if p > 0:
                    a = torch.empty_like(h)
                    L.check(lib.vb_dropout(h.data_ptr(), a.data_ptr(), _DT[dtype], h.numel(), p, int(drop_seed), sid,
                                           _s()), "vb_dropout")
                saved += [h, a]
                drops.append((p, sid))
            out = ops.linear(a, ws_[2], b3.detach(), out_dtype=torch.float32)
        ctx.saved, ctx.ws, ctx.drops, ctx.seed, ctx.dtype = saved, ws_, drops, int(drop_seed), dtype
        return out

    @staticmethod
    def backward(ctx, dout):
        lib = L.load()
        a0, h1, a1, h2, a2 = ctx.saved
        dtype, dev = ctx.dtype, dout.device
        f32 = dict(dtype=torch.float32, device=dev)
        grads = [None] * 6
        with torch.cuda.device(dev):
            dy = ops.cast_from_f32(dout.to(torch.float32).contiguous(), dtype)
            for j, (x, h) in ((2, (a2, h2)), (1, (a1, h1)), (0, (a0, None))):
                w = ctx.ws[j]
                dw, db = torch.zeros(w.shape, **f32), torch.zeros(w.shape[0], **f32)
                dx = torch.empty((x.shape[0], w.shape[1]), dtype=dtype if j > 0 else torch.float32, device=dev)
                _linear_grads(x, w, dy, dx, dw, db)
                grads[2 * j], grads[2 * j + 1] = dw, db
                if j > 0:
                    p, sid = ctx.drops[j - 1]
                    L.check(lib.vb_relu_dropout_backward(dx.data_ptr(), h.data_ptr(), dx.data_ptr(), _DT[dtype],
                                                         dx.numel(), p, ctx.seed, sid, _s()), "vb_relu_dropout_backward")
                dy = dx
        ctx.saved = ctx.ws = None
        return (dy, None, None, None, None, *grads)


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
