"""The decoder stack of `vb_decoder_forward` restated once, over pluggable ops, with float64 ops and the rounding-error
bounds of the two kernels the stack adds to the attention: `layernorm_kernel` (csrc/embed_norm.cu) and `vb_linear`
(the wgmma GEMM of csrc/gemm_wgmma.cu for bf16, `gemm_simt_kernel` of csrc/gemm_simt.cu for fp32), plus the AdaLN
table of `vb_adaln_project`.

Everything here is plain torch and runs on whatever device its tensors live on.  Three facts, each checked on its
own, cover the stack:
  1. semantics: `layer_loop` over `Float64Ops()` (no rounding) is the model, `oracle.valle_oracle.encoder` without
     its final norm and `tests/postln_oracle.encoder_postln` (tests/test_stack_oracle64.py, CPU);
  2. composition: `layer_loop` over the library's public ops reproduces `vb_decoder_forward` bit for bit
     (tests/test_stack_oracle64_gpu.py);
  3. numerics: each op, fed the inputs it received in that run, is within `ln_bound` / `gemm_bound` /
     `attention_oracle64.bound` of its float64 value (same file).

`layer_loop` is written from the model (transformer.py:296-308, the oracle), not from csrc/api.cu:
  pre-LN   x += out_proj(SA(norm1(x)));  x += linear2(relu(linear1(norm2(x))))
  post-LN  x = norm1(x + out_proj(SA(x)));  x = norm2(x + linear2(relu(linear1(x))))
with an AdaLN stack's norm k of layer l reading row 2 l + k - 1 of the (weight | bias) table (NativeDecoder.ada_table
order: norm1, norm2 of each layer, then the final norm).  The storage dtype (bf16 or fp32) is where the library keeps
the GEMM operands, q | k | v, the attention output and the ReLU hidden; the residual stream stays fp32.  A post-norm's
fp32 output replaces the residual row and is cast to the storage dtype for the next projection.

Reading the ratios.  Each bound is a first-order bound on the fp32 arithmetic plus, for a bf16 output, half_ulp(out),
the most a round-to-nearest store can move a value.  That store takes up to its whole share, so a correct kernel's
worst error / bound on a bf16 output sits just under 1 by construction; the fp32 arithmetic shows on the fp32 outputs.
gemm_bound's gamma_K is the worst case that the unspecified order of the tensor cores' sums allows, while the
accumulation error actually made is a random walk of about sqrt(K) roundings, so fp32 outputs sit at a few hundredths
of it.  It still rejects one dropped 64-wide k-block at K = 4096 by more than 20 times (tests/test_stack_oracle64.py).

Backward.  `backward_loop` is the chain rule of `layer_loop` over pluggable ops (Float64Ops has the float64 backward
ops, with the same storage rounding), and the bounds below cover `vb_decoder_backward`'s kernels: `ln_bwd_bound` and
`ln_param_bounds` for `ln_bwd_kernel`, `wgrad_bound` / `dgrad_ratio` (gemm_bound) for the GEMMs of
`vb_linear_backward`, `colsum_bound` and `reduce_bound` for the atomically reduced vectors, `attn_bwd_ratio`
(attention_oracle64.bwd_bound) for the attention backward, `ce_bound` / `ce_bwd_bound` for the loss head.  They are
checked on the CPU by tests/test_stack_backward_oracle64.py and against the kernels by
tests/test_stack_backward_oracle64_gpu.py.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Callable, Dict, List, Optional, Tuple

import torch

import attention_oracle64 as A
from oracle import valle_oracle as O

U32, U_TC = 2.0 ** -24, 2.0 ** -23   # fp32 unit roundoff; the tensor cores' sums (order and rounding unspecified)
EPS = 1e-5
SLACK = 1 + 2.0 ** -5                # second-order terms of the first-order bounds below
TINY = 2.0 ** -120
CHUNK_ELEMS = 2 ** 26                # float64 temporaries of at most 512 MB


# ---------------------------------------------------------------------------------------------------- packed rows
@dataclass
class Pack:
    """packed ragged sequences as vb_decoder_forward takes them: lengths, mask mode (attention_oracle64.MODES), text
    lengths S (text_lens), real audio lengths c1 (seg1_lens) and seg1_start"""
    lens: List[int]
    mode: str
    S: List[int]
    c1: List[int]
    seg1_start: int = 0

    @property
    def cu(self) -> List[int]:
        c = [0]
        for n in self.lens:
            c.append(c[-1] + n)
        return c

    @property
    def M(self) -> int:
        return sum(self.lens)

    def vis(self, b: int) -> torch.Tensor:
        return A.visible(self.mode, self.lens[b], self.S[b], self.c1[b], self.seg1_start)

    def empty_rows(self) -> torch.Tensor:
        """bool [M]: packed rows that see no key"""
        e = torch.zeros(self.M, dtype=torch.bool)
        for b, r0 in enumerate(self.cu[:-1]):
            for r in A.empty_rows_rule(self.mode, self.lens[b], self.S[b], self.c1[b], self.seg1_start):
                e[r0 + r] = True
        return e


@dataclass
class Layer:
    """one layer's parameters as the library reads them (matrices in the storage dtype, vectors fp32)"""
    in_w: torch.Tensor
    in_b: torch.Tensor
    out_w: torch.Tensor
    out_b: torch.Tensor
    w1: torch.Tensor
    b1: torch.Tensor
    w2: torch.Tensor
    b2: torch.Tensor
    n1w: torch.Tensor
    n1b: torch.Tensor
    n2w: torch.Tensor
    n2b: torch.Tensor


def ada_row(ada: Optional[torch.Tensor], l: int, k: int) -> Optional[torch.Tensor]:
    """norm k (1 or 2) of layer l: its (weight | bias) row of the AdaLN table (None: LayerNorm)"""
    return None if ada is None else ada[2 * l + k - 1]


# ----------------------------------------------------------------------------------------------------- layer loop
EPI_NONE, EPI_RELU, EPI_RESIDUAL = 0, 1, 2


def layer_loop(ops, x: torch.Tensor, layers: List[Layer], pk: Pack, n_head: int, norm_first: bool,
               ada: Optional[torch.Tensor] = None, record: Optional[Callable[[int, Dict], None]] = None,
               drop: Optional[Tuple[float, int]] = None) -> torch.Tensor:
    """The stack over packed rows x [M, d] (fp32 or float64; not modified), through `ops`:
      ops.norm(x, w, b, wb, operand)   LayerNorm, then weight * LN + bias with wb = (weight | bias); operand=True: in
                                       the storage dtype (a pre-norm), False: fp32 (a post-norm's new residual)
      ops.linear(a, W, b, epi, res)    epi(a W^T + b), + res for EPI_RESIDUAL (fp32 out), else storage dtype
      ops.attention(qkv, pk, n_head, l)  masked softmax attention of layer l (which may fill layer l's KV cache)
      ops.cast(x)                      x rounded to the storage dtype
    record(l, ops_of_layer) gets, per layer, {op name: (inputs..., output)} for the ops norm1 / norm2 (x, w, b, wb),
    qkv / ffn1 (a, W, b), attn (qkv,), out / ffn2 (a, W, b, res) and, post-LN, cast1 / cast2 (x,).  Returns x.
    drop = (p, seed): training-mode dropout with the masks of `keep_mask` (transformer.py:329,333-334): layer l's
    attention probabilities (stream 4 l), the out-proj output ahead of its residual add (4 l + 1), the FFN hidden after
    the ReLU (4 l + 2) and the FFN2 output (4 l + 3).  Only Float64Ops takes it: ops.linear(..., scale) multiplies
    the (ReLU'd) product by the dropout scale tensor, ops.attention(..., drop) drops probabilities."""
    n = len(layers)
    h = ops.cast(x) if not norm_first else None
    for l, P in enumerate(layers):
        rec = {}

        def norm(k, xin, operand):
            w, b = (P.n1w, P.n1b) if k == 1 else (P.n2w, P.n2b)
            wb = ada_row(ada, l, k)
            out = ops.norm(xin, w, b, wb, operand)
            rec[f"norm{k}"] = (xin, w, b, wb, out)
            return out

        def lin(name, a, W, b, epi, res=None, site=None):
            if drop is None or site is None:
                out = ops.linear(a, W, b, epi, res)
            else:
                shape = (a.shape[0], W.shape[0])
                out = ops.linear(a, W, b, epi, res, dropout_scale(drop, (l << 2) | site, shape, a.device))
            rec[name] = (a, W, b, out) if res is None else (a, W, b, res, out)
            return out

        def attn(hin, xres):
            qkv = lin("qkv", hin, P.in_w, P.in_b, EPI_NONE)
            att = ops.attention(qkv, pk, n_head, l) if drop is None else ops.attention(qkv, pk, n_head, l, drop)
            rec["attn"] = (qkv, att)
            return lin("out", att, P.out_w, P.out_b, EPI_RESIDUAL, xres, site=1)

        def ffn(hin, xres):
            f = lin("ffn1", hin, P.w1, P.b1, EPI_RELU, site=2)
            return lin("ffn2", f, P.w2, P.b2, EPI_RESIDUAL, xres, site=3)

        def cast(name, xin):
            out = ops.cast(xin)
            rec[name] = (xin, out)
            return out

        if norm_first:
            x = attn(norm(1, x, True), x)
            x = ffn(norm(2, x, True), x)
        else:
            x = norm(1, attn(h, x), False)
            x = norm(2, ffn(cast("cast1", x), x), False)
            h = cast("cast2", x) if l + 1 < n else None
        if record is not None:
            record(l, rec)
    return x


class Float64Ops:
    """the ops of layer_loop in float64.  storage: None (no rounding anywhere: the model) or the dtype the library
    rounds the operands, q | k | v, the attention output and the ReLU hidden to; fp32_residual: round the residual
    stream (and a post-norm's output) to fp32 as the library stores it."""

    def __init__(self, storage: Optional[torch.dtype] = None, fp32_residual: bool = False):
        self.storage = storage
        self.fp32_residual = fp32_residual

    # a rounded value is kept in the dtype it was rounded to (exact there); every op reads its inputs as float64
    def _st(self, t):
        return t if self.storage is None else t.to(self.storage)

    def _res(self, t):
        return t.float() if self.fp32_residual else t

    def norm(self, x, w, b, wb, operand):
        y = norm64(x, w, b, wb)
        return self._st(y) if operand else self._res(y)

    def linear(self, a, W, b, epi, res, scale=None):
        """in row chunks, so that no float64 temporary exceeds CHUNK_ELEMS; scale: a dropout scale [M, N]"""
        Wd, bd = W.double().t(), b.double()
        step = max(1, CHUNK_ELEMS // W.shape[0])
        parts = []
        for r0 in range(0, a.shape[0], step):
            z = a[r0:r0 + step].double() @ Wd + bd
            if epi == EPI_RELU:
                z = torch.relu(z)
            if scale is not None:
                z = z * scale[r0:r0 + step]
            if epi == EPI_RESIDUAL:
                parts.append(self._res(res[r0:r0 + step].double() + z))
            else:
                parts.append(self._st(z))
        return torch.cat(parts)

    def attention(self, qkv, pk, n_head, l, drop=None):
        if drop is None:
            return self._st(attention_rows64(qkv, pk, n_head))
        d = qkv.shape[1] // 3
        out = torch.zeros(qkv.shape[0], d, dtype=torch.float64, device=qkv.device)
        for b, r0 in enumerate(pk.cu[:-1]):
            L = pk.lens[b]
            q, k, v = _heads(qkv, r0, L, n_head)
            w = attn_drop_scale(drop, l, b, n_head, L, max(pk.lens), qkv.device)
            P = softmax_rows64(q, k, pk.vis(b).to(qkv.device))
            out[r0:r0 + L] = ((P * w) @ v).transpose(0, 1).reshape(L, d)
        return self._st(out)

    def cast(self, x):
        return self._st(x)

    # ---- the backward ops of backward_loop (grads are float64 accumulators, added to in place) ----
    def linear_backward(self, a, W, dy, epi, dst, dW, db):
        """dX = dy W (chunked); dW += dy^T a; db += column sums of dy.  epi EPI_NONE: dX in the storage dtype (dst
        None) or fp32 (dst given; its contents are not read); EPI_RESIDUAL: dst + dX in fp32"""
        Wd = W.double()
        step = max(1, CHUNK_ELEMS // max(W.shape[0], W.shape[1]))
        dX = torch.cat([dy[r0:r0 + step].double() @ Wd for r0 in range(0, dy.shape[0], step)])
        if dW is not None:
            dW += dy.double().t() @ a.double()
        if db is not None:
            db += dy.double().sum(0)
        if dst is None:
            return self._st(dX)
        return self._res(dst.double() + dX if epi == EPI_RESIDUAL else dX)

    def relu_backward(self, dh, hb, scale):
        return self._st(torch.where(hb.double() > 0, dh.double() * scale, torch.zeros((), dtype=torch.float64,
                                                                                        device=dh.device)))

    def attention_backward(self, qkv, o, dO, pk, n_head, l, drop=None):
        """the gradient of qkv, D = rowsum(dO o) formed from the o given (the stored output, as the kernels do)"""
        d = qkv.shape[1] // 3
        out = torch.zeros(qkv.shape[0], 3 * d, dtype=torch.float64, device=qkv.device)
        for b, r0 in enumerate(pk.cu[:-1]):
            L = pk.lens[b]
            q, k, v = _heads(qkv, r0, L, n_head)
            ob, gb = (t[r0:r0 + L].reshape(L, n_head, A.HD).transpose(0, 1) for t in (o, dO))
            w = None if drop is None else attn_drop_scale(drop, l, b, n_head, L, max(pk.lens), qkv.device)
            g = A.attention_bwd64(q, k, v, ob, gb, pk.vis(b).to(qkv.device), w)
            for i, t in enumerate(g):
                out[r0:r0 + L, i * d:(i + 1) * d] = t.transpose(0, 1).reshape(L, d)
        return self._st(out)

    def norm_backward(self, x, w, b, wb, dout, dst, dg, dbeta, dwb):
        """dst + dLN/dx (fp32; dst None: 0); dg / dbeta / dwb += the parameter gradients"""
        dx, pg = norm_bwd64(x, w, b, wb, dout)
        dg += pg[0]
        dbeta += pg[1]
        if wb is not None:
            dwb += pg[2]
        return self._res(dx if dst is None else dst.double() + dx)

    def dropout(self, t, p, seed, stream):
        return self._st(t.double() * dropout_scale((p, seed), stream, t.shape, t.device))


def norm64(x, w, b, wb=None, eps: float = EPS):
    """LayerNorm (oracle.valle_oracle.layer_norm) and AdaLN weight * LN + bias, in float64"""
    y = O.layer_norm(x.double(), w.double(), b.double(), eps)
    if wb is not None:
        d = x.shape[-1]
        wb = wb.double()
        y = wb[:d] * y + wb[d:]
    return y


def attention_rows64(qkv: torch.Tensor, pk: Pack, n_head: int, head_chunk: int = 8) -> torch.Tensor:
    """attention_oracle64.attention64 over every sequence of a packed qkv [M, 3 d]; [M, d] float64 (0 on rows that
    see no key)"""
    d = qkv.shape[1] // 3
    out = torch.empty(qkv.shape[0], d, dtype=torch.float64, device=qkv.device)
    for b, r0 in enumerate(pk.cu[:-1]):
        L = pk.lens[b]
        q, k, v = (qkv[r0:r0 + L, i * d:(i + 1) * d].reshape(L, n_head, A.HD).transpose(0, 1) for i in range(3))
        ref = A.attention64(q, k, v, pk.vis(b).to(qkv.device), head_chunk=head_chunk)
        out[r0:r0 + L] = ref.O.transpose(0, 1).reshape(L, d)
    return out


def _heads(qkv, r0, L, n_head):
    d = qkv.shape[1] // 3
    return tuple(qkv[r0:r0 + L, i * d:(i + 1) * d].reshape(L, n_head, A.HD).transpose(0, 1) for i in range(3))


def softmax_rows64(q, k, vis):
    """float64 softmax(q k^T / 8 + mask) [H, L, L] (a row that sees no key: 0)"""
    s = (q.double() @ k.double().transpose(-1, -2)) * 0.125
    s = s.masked_fill(~vis, -math.inf)
    m = s.amax(-1, keepdim=True)
    m = torch.where(torch.isfinite(m), m, torch.zeros_like(m))
    p = torch.exp(s - m)
    return p / torch.clamp(p.sum(-1, keepdim=True), min=TINY)


# ---------------------------------------------------------------------------------------------------------- dropout
def keep_mask(seed: int, stream: int, n: int, p: float, idx=None) -> torch.Tensor:
    """the stateless mask of csrc/kernels.cuh::drop_keep restated in numpy: True = kept.  Element i of stream `stream`
    is kept iff the top 32 bits of splitmix64(seed + stream * golden + i * 0xD1342543DE82EF95) are >= p 2^32."""
    import numpy as np
    with np.errstate(over="ignore"):
        i = np.arange(n, dtype=np.uint64) if idx is None else idx.astype(np.uint64)
        z = np.uint64(seed) + np.uint64(stream) * np.uint64(0x9E3779B97F4A7C15) + i * np.uint64(0xD1342543DE82EF95)
        z ^= z >> np.uint64(30)
        z *= np.uint64(0xBF58476D1CE4E5B9)
        z ^= z >> np.uint64(27)
        z *= np.uint64(0x94D049BB133111EB)
        z ^= z >> np.uint64(31)
        return torch.from_numpy(((z >> np.uint64(32)) >= np.uint64(int(p * 4294967296.0))).astype(np.bool_))


def inv_keep(p: float) -> float:
    """1 / (1 - p) as the kernels (and torch's fp32 dropout) hold it: in fp32"""
    return float(torch.tensor(1.0 / (1.0 - p), dtype=torch.float32))


def dropout_scale(drop: Tuple[float, int], stream: int, shape, device) -> torch.Tensor:
    """float64 tensor of `shape`: inv_keep(p) where stream `stream` keeps the element (row-major index), else 0"""
    p, seed = drop
    n = int(math.prod(shape))
    return (keep_mask(seed, stream, n, p).view(shape).double() * inv_keep(p)).to(device)


def attn_drop_scale(drop: Tuple[float, int], l: int, b: int, n_head: int, L: int, lmax: int, device) -> torch.Tensor:
    """[H, L, L] dropout scale of layer l's attention probabilities of sequence b: element (h, q, k) is index
    ((b H + h) lmax + q) lmax + k of stream 4 l (lmax: the max_seqlen the library was given)"""
    import numpy as np
    p, seed = drop
    h, q, k = np.meshgrid(np.arange(n_head), np.arange(L), np.arange(L), indexing="ij")
    idx = ((b * n_head + h).astype(np.uint64) * lmax + q) * lmax + k
    return (keep_mask(seed, l << 2, idx.size, p, idx.reshape(-1)).view(n_head, L, L).double() * inv_keep(p)).to(device)


# -------------------------------------------------------------------------------------------------------- backward
def norm_bwd64(x, w, b, wb, dout, eps: float = EPS):
    """float64 gradients of norm64 (LayerNorm, then AdaLN): (dx, (dgamma, dbeta[, d(weight | bias)])) for the rows x
    and the output gradient dout"""
    xd, gy = x.double(), dout.double()
    d = xd.shape[-1]
    mu = xd.mean(-1, keepdim=True)
    rstd = 1.0 / torch.sqrt(((xd - mu) ** 2).mean(-1, keepdim=True) + eps)
    xh = (xd - mu) * rstd
    aw = wb.double()[:d] if wb is not None else torch.ones(d, dtype=torch.float64, device=xd.device)
    G = gy * aw * w.double()
    dx = rstd * (G - G.mean(-1, keepdim=True) - xh * (G * xh).mean(-1, keepdim=True))
    pg = [(gy * aw * xh).sum(0), (gy * aw).sum(0)]
    if wb is not None:
        pg.append(torch.cat([(gy * (w.double() * xh + b.double())).sum(0), gy.sum(0)]))
    return dx, pg


def saves_of(rec: Dict) -> Dict[str, torch.Tensor]:
    """layer_loop's record of one layer as the library's LayerSave (csrc/api.cu): x_in / x_mid the inputs of norm1 /
    norm2, xn1 / xn2 the QKV / FFN1 operands, qkv, att, and hb the FFN hidden after ReLU and dropout"""
    return dict(x_in=rec["norm1"][0], x_mid=rec["norm2"][0], xn1=rec["qkv"][0], qkv=rec["attn"][0],
                att=rec["attn"][1], xn2=rec["ffn1"][0], hb=rec["ffn2"][0])


GRAD_NAMES = ("in_w", "in_b", "out_w", "out_b", "w1", "b1", "w2", "b2", "n1w", "n1b", "n2w", "n2b")


def backward_loop(ops, saves: List[Dict[str, torch.Tensor]], dx: torch.Tensor, layers: List[Layer], pk: Pack,
                  n_head: int, norm_first: bool, grads: List[Dict[str, torch.Tensor]],
                  ada: Optional[torch.Tensor] = None, dada: Optional[torch.Tensor] = None,
                  drop: Optional[Tuple[float, int]] = None,
                  record: Optional[Callable[[int, Dict], None]] = None) -> torch.Tensor:
    """The chain rule of layer_loop, last layer first, through `ops`.  saves[l]: layer l's forward values (saves_of);
    dx [M, d]: the gradient of the stack output (not modified); grads[l]: {GRAD_NAMES: accumulator}, dada: the
    AdaLN table's gradient (accumulated into in place).  Returns the gradient of the stack input.
      ops.linear_backward(a, W, dy, epi, dst, dW, db)  dX = dy W (see Float64Ops), dW += dy^T a, db += colsum dy
      ops.relu_backward(dh, hb, scale)    dh where hb > 0 (times the dropout scale), else 0
      ops.attention_backward(qkv, o, dO, pk, n_head, l[, drop])   the gradient of qkv
      ops.norm_backward(x, w, b, wb, dout, dst, dg, dbeta, dwb)   dst + the norm's input gradient (fp32)
      ops.dropout(t, p, seed, stream), ops.cast(x)
    Pre-LN:  g is the residual gradient; per block: dy = drop(cast(g)); the block's input gradient dn (fp32) goes
             through the block's norm and is added to g.
    Post-LN: y = norm2(r2), r2 = x1 + drop(FF(x1)), x1 = norm1(r1), r1 = x + drop(SA(x)): dr = norm2^T(g), the FFN's
             input gradient is added to dr (= dx1), g = norm1^T(dr), the attention's input gradient is added to g.
    record(l, ops_of_layer) gets {op name: (inputs..., output)}."""
    p, seed = drop if drop is not None else (0.0, 0)
    scale = inv_keep(p) if drop is not None else 1.0
    g = dx
    for l in range(len(layers) - 1, -1, -1):
        P, sv, G = layers[l], saves[l], grads[l]
        rec = {}

        def dropped(name, t, site):
            if drop is None:
                return t
            out = ops.dropout(t, p, seed, (l << 2) | site)
            rec[name] = (t, out)
            return out

        def cast(name, t):
            out = ops.cast(t)
            rec[name] = (t, out)
            return out

        def lin(name, a, W, dy, epi, dst, wn, bn):
            out = ops.linear_backward(a, W, dy, epi, dst, G[wn], G[bn])
            rec[name] = (a, W, dy, dst, out, G[wn], G[bn])
            return out

        def norm(k, dout, dst):
            x = sv["x_in"] if k == 1 else sv["x_mid"]
            w, b = (P.n1w, P.n1b) if k == 1 else (P.n2w, P.n2b)
            wb, dwb = ada_row(ada, l, k), ada_row(dada, l, k)
            out = ops.norm_backward(x, w, b, wb, dout, dst, G[f"n{k}w"], G[f"n{k}b"], dwb)
            rec[f"norm{k}_bwd"] = (x, w, b, wb, dout, dst, out, G[f"n{k}w"], G[f"n{k}b"], dwb)
            return out

        def ffn(gd, dst, epi):
            dy = dropped("drop3", gd, 3)
            dh = lin("ffn2_bwd", sv["hb"], P.w2, dy, EPI_NONE, None, "w2", "b2")
            dr = ops.relu_backward(dh, sv["hb"], scale)
            rec["relu_bwd"] = (dh, sv["hb"], scale, dr)
            return lin("ffn1_bwd", sv["xn2"], P.w1, dr, epi, dst, "w1", "b1")

        def attn(gd, dst, epi):
            dy = dropped("drop1", gd, 1)
            dO = lin("out_bwd", sv["att"], P.out_w, dy, EPI_NONE, None, "out_w", "out_b")
            if drop is None:
                dqkv = ops.attention_backward(sv["qkv"], sv["att"], dO, pk, n_head, l)
            else:
                dqkv = ops.attention_backward(sv["qkv"], sv["att"], dO, pk, n_head, l, drop)
            rec["attn_bwd"] = (sv["qkv"], sv["att"], dO, dqkv)
            return lin("qkv_bwd", sv["xn1"], P.in_w, dqkv, epi, dst, "in_w", "in_b")

        if norm_first:
            dn = ffn(cast("cast2", g), g, EPI_NONE)
            g = norm(2, dn, g)
            dn = attn(cast("cast1", g), g, EPI_NONE)
            g = norm(1, dn, g)
        else:
            dr = norm(2, g, None)
            dr = ffn(cast("cast2", dr), dr, EPI_RESIDUAL)
            g = norm(1, dr, None)
            g = attn(cast("cast1", g), g, EPI_RESIDUAL)
        if record is not None:
            record(l, rec)
    return g


# ---------------------------------------------------------------------------------------------------------- bounds
def half_ulp(out: torch.Tensor) -> torch.Tensor:
    """half the spacing of out's dtype (bf16 or fp32) just above |out|, float64: a round-to-nearest result is within
    this of the value it rounded (0 maps to the smallest subnormal's half)"""
    p = 8 if out.dtype == torch.bfloat16 else 24
    o = out.double().abs()
    _, e = torch.frexp(o)                        # o = m 2^e, m in [0.5, 1): the spacing above is 2^(e - p)
    h = torch.ldexp(torch.ones_like(o), (e - 1 - p).to(torch.int32))
    return torch.where(o > 0, h, torch.full_like(o, 2.0 ** -150))


def ratio(got: torch.Tensor, ref: torch.Tensor, bnd: torch.Tensor, keep: Optional[torch.Tensor] = None) -> float:
    """max |got - ref| / bnd over the elements whose reference is finite (and, if given, rows `keep`); a non-finite
    `got` there counts as infinite"""
    dlt = got.double() - ref
    r = dlt.abs() / bnd
    r = torch.where(torch.isfinite(dlt), r, torch.full_like(r, math.inf))
    ok = torch.isfinite(ref)
    if keep is not None:
        ok = ok & keep.to(ok.device).reshape(-1, *([1] * (ok.dim() - 1)))
    r = r[ok]
    return float(r.max()) if r.numel() else 0.0


def sum_depth(d: int) -> int:
    """the most fp32 roundings one element goes through in the kernel's row sums: the pair sums of a float4 (2), the
    lane's running sum over its ceil(d / 128) float4s, the 5 butterfly steps of warp_sum, one for a product"""
    return -(-d // 128) + 8


def ln_bound(x: torch.Tensor, w: torch.Tensor, b: torch.Tensor, wb: Optional[torch.Tensor], out: torch.Tensor,
             eps: float = EPS):
    """(exact, bound) float64 [R, d] for the rows `out` [R, d] (bf16 or fp32) that `layernorm_kernel` made from the
    fp32 rows x [R, d] (already gathered), gamma w, beta b and the AdaLN (weight | bias) row wb (None: LayerNorm).

    The kernel, one warp per row, in fp32: s = sum x (each lane adds (x0 + x1) + (x2 + x3) of its float4s in order,
    then warp_sum's butterfly), mean = s / d; a_i = x_i - mean; q = sum a_i^2 the same way; r = rsqrtf(q / d + eps);
    y_i = a_i r g_i + b_i; AdaLN z_i = w_i y_i + bb_i; then the store rounds to the output type.  With n = sum_depth(d)
    roundings per element, S1 = sum |x_i|, mu, sigma^2 the exact moments and s_e = sqrt(sigma^2 + eps):
      mean:  |mean^ - mu| <= dm = gamma_{n+1} S1 / d (the sum, the division).  S1 / d <= |mu| + sigma, so dm / s_e
             carries the row offset |mu| / sigma: at |mu| / sigma = 4096 it is about 2^-8.
      var:   a_i = (x_i - mu - dm_i)(1 + e_i); sum (x_i - mu) = 0 cancels the linear term, so sum a_i^2 =
             d (sigma^2 + dm^2)(1 + 2u + u^2) at worst; the sum of positive terms adds gamma_n, / d and + eps one u
             each: q / d + eps = s_e^2 (1 + ev), ev <= (dm / s_e)^2 (1 + 3u) + 4u + gamma_n.
      rstd:  rsqrtf is within 2 ulp (2^-22 relative): r^ = (1 + t) / s_e, |t| <= ev / 2 + 2^-22.
      y:     t2 = fl(a_i r^) is off n_i = (x_i - mu) / s_e by en = dm / s_e + (2u + |t|) |n_i|; y = fl(t2 g + b)
             (one fma, or two roundings) is off Y = n g + b by ey = |g| en + 2u (|g n| + |b|).
      AdaLN: z = fl(w y + bb) is off Z = w Y + bb by |w| ey + 2u (|w Y| + |bb|).
      out:   a round-to-nearest store adds half_ulp(out) (bf16; fp32 stores y as it is).
    Bound: the first-order sum times SLACK, + half_ulp(out) for a bf16 out, + TINY."""
    xd = x.double()
    R, d = xd.shape
    n = sum_depth(d)
    mu = xd.mean(-1, keepdim=True)
    var = ((xd - mu) ** 2).mean(-1, keepdim=True)
    se = torch.sqrt(var + eps)
    dm = A.gamma(n + 1, U32) * xd.abs().sum(-1, keepdim=True) / d
    ev = (dm / se) ** 2 * (1 + 3 * U32) + 4 * U32 + A.gamma(n, U32)
    t = ev / 2 + 2.0 ** -22
    nn_ = (xd - mu) / se
    en = dm / se + (2 * U32 + t) * nn_.abs()
    g, bb = w.double(), b.double()
    Y = nn_ * g + bb
    e = g.abs() * en + 2 * U32 * ((g * nn_).abs() + bb.abs())
    if wb is not None:
        ww, wbias = wb.double()[:d], wb.double()[d:]
        e = ww.abs() * e + 2 * U32 * ((ww * Y).abs() + wbias.abs())
        Y = ww * Y + wbias
    bnd = e * SLACK + TINY
    if out.dtype == torch.bfloat16:
        bnd = bnd + half_ulp(out)
    return Y, bnd


def gemm_bound(a: torch.Tensor, W: torch.Tensor, b: Optional[torch.Tensor], epi: int, res: Optional[torch.Tensor],
               out: torch.Tensor, kind: str):
    """(exact, bound) float64 [R, N] for out = epi(a W^T + b) [+ res] from `vb_linear` (a [R, K], W [N, K] in the
    storage dtype, b fp32 or None, res fp32).  kind: "wgmma" (bf16 tensor cores) or "simt" (gemm_simt_kernel).

    With p = a W^T and S = |a| |W|^T, the kernel's fp32 accumulator acc = p + e_acc:
      wgmma: bf16 x bf16 products are exact in fp32; the order and rounding of the tensor cores' sums are not
             specified, so a K-term sum gets gamma_K with u = 2^-23 (twice the fp32 unit roundoff, as
             attention_oracle64.score_error assumes): |e_acc| <= gamma_K(2^-23) S.
      simt:  fmaf chains in k order: one rounding per term; gamma_{K+1}(2^-24) S also covers a product rounded on its
             own, should the compiler not contract.
    Epilogue: v = fl(acc + b) adds 2^-24 |p + b| (and the first-order e_acc); ReLU is 1-Lipschitz and exact; the
    residual fl(res + v) adds 2^-24 |res + z|; a bf16 store adds half_ulp(out), an fp32 store is the last rounding
    already counted.  Bound: (sum) times SLACK + TINY (+ half_ulp(out) for bf16)."""
    K = a.shape[1]
    ad, Wd = a.double(), W.double()
    p = ad @ Wd.t()
    S = ad.abs() @ Wd.abs().t()
    e = (A.gamma(K, U_TC) if kind == "wgmma" else A.gamma(K + 1, U32)) * S
    z = p if b is None else p + b.double()
    if b is not None:
        e = e + U32 * z.abs()
    if epi == EPI_RELU:
        z = torch.relu(z)
    if epi == EPI_RESIDUAL:
        z = res.double() + z
        e = e + U32 * z.abs()
    bnd = e * SLACK + TINY
    if out.dtype == torch.bfloat16:
        bnd = bnd + half_ulp(out)
    return z, bnd


def gemm_ratio(a, W, b, epi, res, out, kind, keep: Optional[torch.Tensor] = None) -> float:
    """max error / gemm_bound over all of out, in row chunks that keep each float64 temporary under CHUNK_ELEMS"""
    N = W.shape[0]
    step = max(1, CHUNK_ELEMS // max(N, a.shape[1]))
    worst = 0.0
    for r0 in range(0, a.shape[0], step):
        sl = slice(r0, r0 + step)
        z, bnd = gemm_bound(a[sl], W, b, epi, None if res is None else res[sl], out[sl], kind)
        worst = max(worst, ratio(out[sl], z, bnd, None if keep is None else keep[sl]))
    return worst


def ln_ratio(x, w, b, wb, out, keep: Optional[torch.Tensor] = None) -> float:
    step = max(1, CHUNK_ELEMS // (4 * x.shape[1]))
    worst = 0.0
    for r0 in range(0, x.shape[0], step):
        sl = slice(r0, r0 + step)
        y, bnd = ln_bound(x[sl], w, b, wb, out[sl])
        worst = max(worst, ratio(out[sl], y, bnd, None if keep is None else keep[sl]))
    return worst


def adaln_bound(W: torch.Tensor, b: torch.Tensor, emb: torch.Tensor, out: torch.Tensor):
    """(exact, bound) float64 [2 d] for the (weight | bias) row vb_adaln_project makes: out[n] = W[n] . emb + b[n],
    each lane an fp32 chain over its float4s, then warp_sum and the bias add: at most d + 6 roundings per term, so
    gamma_{d+6}(2^-24) (sum_c |W[n, c] emb[c]| + |b[n]|)."""
    d = W.shape[1]
    z = W.double() @ emb.double() + b.double()
    bnd = A.gamma(d + 6, U32) * (W.double().abs() @ emb.double().abs() + b.double().abs()) * SLACK + TINY
    return z, bnd


# ------------------------------------------------------------------------------------------------- backward bounds
def sum_depth_lanes(d: int) -> int:
    """the most fp32 roundings one element goes through in a row sum of ln_bwd_kernel / ce_bwd_kernel: the lane's
    running sum over its ceil(d / 32) elements, warp_sum's 5 butterfly steps, one for a product or the division"""
    return -(-d // 32) + 6


def reduce_bound(abs_sum: torch.Tensor, n: int, prior: Optional[torch.Tensor] = None,
                 term_err: Optional[torch.Tensor] = None) -> torch.Tensor:
    """bound on an fp32 sum of n terms reduced in an unspecified order (atomics): any order of n + 1 additions (the
    prior value included) is off by at most gamma_{n+1}(2^-24) (sum |terms| + |prior|); term_err: the sum of the
    terms' own errors.  Times SLACK, + TINY."""
    s = abs_sum if prior is None else abs_sum + prior.double().abs()
    e = A.gamma(n + 1, U32) * s
    if term_err is not None:
        e = e + term_err
    return e * SLACK + TINY


def _ln_terms(xd, eps):
    """moments and the error of xhat that ln_bwd_kernel's fp32 recomputation makes: (nn, rstd, en), see ln_bwd_bound"""
    d = xd.shape[-1]
    n = sum_depth_lanes(d)
    mu = xd.mean(-1, keepdim=True)
    se = torch.sqrt(((xd - mu) ** 2).mean(-1, keepdim=True) + eps)
    dm = A.gamma(n + 1, U32) * xd.abs().sum(-1, keepdim=True) / d
    ev = (dm / se) ** 2 * (1 + 3 * U32) + 4 * U32 + A.gamma(n, U32)
    t = ev / 2 + 2.0 ** -22
    nn_ = (xd - mu) / se
    en = dm / se + (2 * U32 + t) * nn_.abs()
    return nn_, 1.0 / se, en, t


def ln_bwd_bound(x, w, b, wb, dout, prior: Optional[torch.Tensor] = None, eps: float = EPS):
    """(exact, bound) float64 for what `ln_bwd_kernel` (csrc/backward.cu) leaves in the rows of dx: prior + dLN/dx,
    from the fp32 rows x [R, d] (gathered), gamma w, beta b, the AdaLN row wb (None: LayerNorm), the output gradient
    dout [R, d] and the rows' prior contents (None: 0).

    The kernel, one warp per row in fp32, sums in lane chains of ceil(d / 32) terms and warp_sum (n = sum_depth_lanes
    roundings): it recomputes mu and rstd as ln_bound derives (dm, ev, t, and en, the error of xhat = fl(fl(x - mu)
    rstd) against n_i = (x_i - mu) / s_e); G_i = dy_i aw_i g_i (two roundings, 2u |G|); two d-term means
    m1 = mean G (off by (gamma_{n+1} + 2u) mean |G|) and m2 = mean G xhat (off by mean(|G| en + 2u |G n|)
    + (gamma_{n+1} + u) mean |G n|); inner = G - m1 - xhat m2 (its error e_in: the errors of G, m1, xhat m2 plus
    three roundings, 3u (|G| + |m1| + |n m2|)); v = prior + rstd inner (rstd relative t, the product and the add one u
    each).  The cancellation in G - m1 - xhat m2 is covered: every error above is absolute.  Bound: the sum times
    SLACK + TINY; the output is fp32 (a bf16 dx_copy is bf16(v), checked bit for bit)."""
    xd, gy = x.double(), dout.double()
    d = xd.shape[-1]
    n = sum_depth_lanes(d)
    nn_, rstd, en, t = _ln_terms(xd, eps)
    aw = wb.double()[:d] if wb is not None else torch.ones(d, dtype=torch.float64, device=xd.device)
    G = gy * aw * w.double()
    m1, m2 = G.mean(-1, keepdim=True), (G * nn_).mean(-1, keepdim=True)
    em1 = (A.gamma(n + 1, U32) + 2 * U32) * G.abs().mean(-1, keepdim=True)
    em2 = (G.abs() * en + 2 * U32 * (G * nn_).abs()).mean(-1, keepdim=True) + \
        (A.gamma(n + 1, U32) + U32) * (G * nn_).abs().mean(-1, keepdim=True)
    inner = G - m1 - nn_ * m2
    e_in = 2 * U32 * G.abs() + em1 + en * m2.abs() + nn_.abs() * em2 + \
        3 * U32 * (G.abs() + m1.abs() + (nn_ * m2).abs())
    dx = rstd * inner
    z = dx if prior is None else prior.double() + dx
    e = t * dx.abs() + rstd * e_in + U32 * dx.abs() + U32 * z.abs()
    return z, e * SLACK + TINY


def ln_param_bounds(x, w, b, wb, dout, priors=None, eps: float = EPS):
    """{name: (exact, bound)} for the vectors ln_bwd_kernel adds up over the R rows with atomics (reduce_bound,
    n = R): dgamma = sum dy aw xhat, dbeta = sum dy aw and, with AdaLN, dada = (sum dy (g xhat + beta) | sum dy).
    Each term's own error: dgamma |dy aw| en + 2u |term|; dbeta u |term|; the AdaLN weight part
    |dy| (|g| en + 2u (|g n| + |beta|)) + u |term|; its bias part none.  priors: {name: the vector's prior value}."""
    xd, gy = x.double(), dout.double()
    R, d = xd.shape
    nn_, _, en, _ = _ln_terms(xd, eps)
    aw = wb.double()[:d] if wb is not None else torch.ones(d, dtype=torch.float64, device=xd.device)
    g, bb = w.double(), b.double()
    priors = priors or {}
    out = {}
    T = gy * aw * nn_
    terms = {"dgamma": (T, (gy * aw).abs() * en + 2 * U32 * T.abs()), "dbeta": (gy * aw, U32 * (gy * aw).abs())}
    if wb is not None:
        Tw = gy * (g * nn_ + bb)
        ew = gy.abs() * (g.abs() * en + 2 * U32 * ((g * nn_).abs() + bb.abs())) + U32 * Tw.abs()
        terms["dada"] = (torch.cat([Tw, gy], -1), torch.cat([ew, torch.zeros_like(gy)], -1))
    for k, (T, eT) in terms.items():
        z = T.sum(0)
        pr = priors.get(k)
        if pr is not None:
            z = z + pr.double()
        out[k] = (z, reduce_bound(T.abs().sum(0), R, pr, eT.sum(0)))
    return out


def colsum_bound(dy, prior=None):
    """(exact, bound) of the bias gradient prior + sum_r dy[r] (colsum_kernel: exact fp32 terms, added in per-thread
    chains, a shared-memory tree and one atomic per 256-row block, in an unspecified order: reduce_bound, n = R)"""
    t = dy.double()
    z = t.sum(0) if prior is None else t.sum(0) + prior.double()
    return z, reduce_bound(t.abs().sum(0), t.shape[0], prior)


def wgrad_bound(a, dy, prior, out, kind):
    """(exact, bound) of the weight gradient prior + dy^T a [N, K] that vb_linear_backward forms as the GEMM of the
    transposed, zero-padded dY^T [N, Mp] and X^T [K, Mp] with the fp32 residual epilogue: gemm_bound over K = Mp
    (the padded row count, padded with zeros), residual = prior"""
    M = a.shape[0]
    Mp = -(-M // 64) * 64
    pad = lambda t: torch.cat([t, t.new_zeros(Mp - M, t.shape[1])]) if Mp > M else t  # noqa: E731
    return gemm_bound(pad(dy).t(), pad(a).t(), None, EPI_RESIDUAL, prior, out, kind)


def dgrad_ratio(dy, W, epi, res, out, kind) -> float:
    """dX = dy W [+ res] of vb_linear_backward (the forward GEMM of dY with the transposed weight): gemm_ratio"""
    return gemm_ratio(dy, W.t(), None, epi, res, out, kind)


def attn_bwd_ratio(dqkv, qkv, o, dO, pk: Pack, n_head: int, l: int = 0, drop=None):
    """{dq, dk, dv: max error / bound} of dqkv [M, 3 d] from vb_attention_backward for every sequence of pk, with
    attention_oracle64.bwd_bound (+ half_ulp of the output for a bf16 dqkv)"""
    d = qkv.shape[1] // 3
    worst = {"dq": 0.0, "dk": 0.0, "dv": 0.0}
    for b, r0 in enumerate(pk.cu[:-1]):
        L = pk.lens[b]
        q, k, v = _heads(qkv, r0, L, n_head)
        ob, gb = (t[r0:r0 + L].reshape(L, n_head, A.HD).transpose(0, 1) for t in (o, dO))
        w = None if drop is None else attn_drop_scale(drop, l, b, n_head, L, max(pk.lens), qkv.device)
        exact, bnds = A.bwd_bound(q, k, v, ob, gb, pk.vis(b).to(qkv.device), w)
        got = _heads(dqkv, r0, L, n_head)
        for name, z, bnd, gt in zip(("dq", "dk", "dv"), exact, bnds, got):
            if dqkv.dtype == torch.bfloat16:
                bnd = bnd + half_ulp(gt)
            worst[name] = max(worst[name], ratio(gt, z, bnd))
    return worst


def ce_bound(logits, targets, n_vocab: int, ignore_index: int):
    """(exact, bound) float64 [R] of vb_cross_entropy's loss = logsumexp(x) - x[t] (0 on ignored rows).  The kernel
    (one warp per row, fp32): mx exact; s = sum expf(x_j - mx) in lane chains (n = sum_depth_lanes(V) roundings),
    each term off by u |x_j - mx| (the subtraction) and 2^-22 (expf): s is off by e_s = gamma_n + 2^-22 +
    u max_j |x_j - mx| relative; logf adds 2u |log s|, the two adds u |lse| and u |loss|."""
    x = logits[:, :n_vocab].double()
    mx = x.amax(-1, keepdim=True)
    z = x - mx
    ls = torch.log(torch.exp(z).sum(-1))
    lse = mx[:, 0] + ls
    t = targets.clamp(0, n_vocab - 1)
    loss = lse - x.gather(1, t[:, None])[:, 0]
    e_s = A.gamma(sum_depth_lanes(n_vocab), U32) + 2.0 ** -22 + U32 * z.abs().amax(-1)
    e = e_s + 2 * U32 * ls.abs() + U32 * lse.abs() + U32 * loss.abs()
    skip = (targets == ignore_index) | (targets < 0) | (targets >= n_vocab)
    loss = torch.where(skip, torch.zeros_like(loss), loss)
    return loss, torch.where(skip, torch.zeros_like(e), e * SLACK) + TINY


def ce_bwd_bound(logits, targets, n_vocab: int, ignore_index: int, grad_rows, grad_scale: float, n_out: int, out):
    """(exact, bound) float64 [R, n_out] of vb_cross_entropy_backward: dl = g (softmax(x) - onehot(t)) with
    g = grad_scale grad_rows[r] (0 on ignored rows), 0 in the columns [n_vocab, n_out).  The kernel recomputes mx and
    s as ce_bound derives (relative e_s); inv = 1 / s one more u; p^ = fl(expf(x_j - mx) inv) is off P_j by
    P_j (2^-22 + u |x_j - mx| + e_s + 2u); the onehot subtraction, the fp32 g and the product by g one u each.
    Bound: |g| P_j (...) + 3u |g (P_j - onehot)|, times SLACK, + TINY, + half_ulp(out) for bf16; ignored rows and
    padding columns must be exactly 0."""
    x = logits[:, :n_vocab].double()
    R = x.shape[0]
    mx = x.amax(-1, keepdim=True)
    z = x - mx
    P = torch.softmax(z, -1)
    skip = (targets == ignore_index) | (targets < 0) | (targets >= n_vocab)
    g = torch.full((R,), float(grad_scale), dtype=torch.float64, device=x.device)
    if grad_rows is not None:
        g = g * grad_rows.double()
    g = torch.where(skip, torch.zeros_like(g), g)[:, None]
    oh = torch.zeros_like(P)
    oh.scatter_(1, targets.clamp(0, n_vocab - 1)[:, None], 1.0)
    dl = g * (P - oh)
    e_s = A.gamma(sum_depth_lanes(n_vocab), U32) + 2.0 ** -22 + U32 * z.abs().amax(-1, keepdim=True)
    e = g.abs() * P * (2.0 ** -22 + U32 * z.abs() + e_s + 2 * U32) + 3 * U32 * dl.abs()
    exact = torch.zeros(R, n_out, dtype=torch.float64, device=x.device)
    bnd = torch.full((R, n_out), TINY, dtype=torch.float64, device=x.device)
    exact[:, :n_vocab] = dl
    bnd[:, :n_vocab] = e * SLACK + TINY
    if out.dtype == torch.bfloat16:
        bnd = bnd + half_ulp(out[:, :n_out])
    return exact, bnd
