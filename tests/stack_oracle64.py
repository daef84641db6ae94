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
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Callable, Dict, List, Optional

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
               ada: Optional[torch.Tensor] = None, record: Optional[Callable[[int, Dict], None]] = None) -> torch.Tensor:
    """The stack over packed rows x [M, d] (fp32 or float64; not modified), through `ops`:
      ops.norm(x, w, b, wb, operand)   LayerNorm, then weight * LN + bias with wb = (weight | bias); operand=True: in
                                       the storage dtype (a pre-norm), False: fp32 (a post-norm's new residual)
      ops.linear(a, W, b, epi, res)    epi(a W^T + b), + res for EPI_RESIDUAL (fp32 out), else storage dtype
      ops.attention(qkv, pk, n_head, l)  masked softmax attention of layer l (which may fill layer l's KV cache)
      ops.cast(x)                      x rounded to the storage dtype
    record(l, ops_of_layer) gets, per layer, {op name: (inputs..., output)} for the ops norm1 / norm2 (x, w, b, wb),
    qkv / ffn1 (a, W, b), attn (qkv,), out / ffn2 (a, W, b, res) and, post-LN, cast1 / cast2 (x,).  Returns x."""
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

        def lin(name, a, W, b, epi, res=None):
            out = ops.linear(a, W, b, epi, res)
            rec[name] = (a, W, b, out) if res is None else (a, W, b, res, out)
            return out

        def attn(hin, xres):
            qkv = lin("qkv", hin, P.in_w, P.in_b, EPI_NONE)
            att = ops.attention(qkv, pk, n_head, l)
            rec["attn"] = (qkv, att)
            return lin("out", att, P.out_w, P.out_b, EPI_RESIDUAL, xres)

        def ffn(hin, xres):
            f = lin("ffn1", hin, P.w1, P.b1, EPI_RELU)
            return lin("ffn2", f, P.w2, P.b2, EPI_RESIDUAL, xres)

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

    def linear(self, a, W, b, epi, res):
        """in row chunks, so that no float64 temporary exceeds CHUNK_ELEMS"""
        Wd, bd = W.double().t(), b.double()
        step = max(1, CHUNK_ELEMS // W.shape[0])
        parts = []
        for r0 in range(0, a.shape[0], step):
            z = a[r0:r0 + step].double() @ Wd + bd
            if epi == EPI_RELU:
                z = torch.relu(z)
            if epi == EPI_RESIDUAL:
                parts.append(self._res(res[r0:r0 + step].double() + z))
            else:
                parts.append(self._st(z))
        return torch.cat(parts)

    def attention(self, qkv, pk, n_head, l):
        return self._st(attention_rows64(qkv, pk, n_head))

    def cast(self, x):
        return self._st(x)


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
