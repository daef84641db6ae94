"""TEST INFRASTRUCTURE ONLY -- one batched AR decode step (`vb_ar_decode_step`, include/valle_b200.h) restated in
float64 from an explicit state, with the bf16 rounding points of each decode chain of the engine.

State: the decoder's weights (a state dict in the oracle's naming, `<prefix>.layers.<i>.*`, `<prefix>.norm.*`), the
input rows x [B, d], the K / V caches [n_layer, B, H, cap, 64], text_len, prompt_len, n_gen and finished.  Row b has
kv_len = clamp(text_len + prompt_len + n_gen, 1, cap) keys: the current token's key and value go to cache row
kv_len - 1, and its query attends to rows [0, kv_len).  A finished row appends nothing and its attention output is
zero (the kernels skip it); its other outputs are not meaningful.

Chains (where the operands are rounded to bf16; every sum is float64 here, fp32 in the kernels):
  fp32           no rounding: the CUDA-core GEMV chain and attn_decode_kernel, either layer order
  bf16_unfolded  pre-LN, VB_DECODE_FOLD=0: the projection operands bf16(LN(x)), bf16(attn_out), bf16(relu(.)); K and
                 V rounded to bf16 (the current token's too, as attention reads it); q unrounded; bf16(W); biases and
                 the residual stream fp32
  bf16_folded    pre-LN, LayerNorm folded into the projection that consumes it (vb_ln_fold): operand bf16(x) of the
                 raw rows, wf = bf16(fp32(bf16(W) gamma)), c = sum_k wf, dvec = b + bf16(W) beta, mean = sum x / d,
                 var = max(sum x^2 / d - mean^2, 0), consumer rstd (acc - mean c) + dvec
  bf16_postln    post-LN (DESIGN section 4): x cast to bf16 once ahead of layer 0, after that the operand of each
                 projection is the bf16 copy of the previous post-norm's output; no final norm
`rounding=False` keeps a chain's algebra (the fold, the layer order) and drops every rounding.
"""
from __future__ import annotations

from dataclasses import dataclass

import torch

from oracle import valle_oracle as O

CHAINS = ("fp32", "bf16_unfolded", "bf16_folded", "bf16_postln")
HD = 64
EPS = 1e-5


@dataclass
class StepOut:
    x: torch.Tensor       # [B, d] the stack output: residual rows before the final norm (post-LN: the last norm2's)
    k_new: torch.Tensor   # [n_layer, B, H, 64] the key row each layer appends at cache row kv_len - 1
    v_new: torch.Tensor   # [n_layer, B, H, 64]
    q: torch.Tensor       # [n_layer, B, H, 64] each layer's query (before the 1/8 scale)
    logits: torch.Tensor  # [B, n_vocab]
    kv_len: torch.Tensor  # [B]


def bf16(t: torch.Tensor) -> torch.Tensor:
    """float64 -> the kernels' fp32 value -> bf16 (round to nearest even), back in float64"""
    return t.to(torch.float32).to(torch.bfloat16).to(torch.float64)


def kv_lengths(text_len, prompt_len, n_gen, cap: int) -> torch.Tensor:
    return torch.clamp(torch.as_tensor(text_len, dtype=torch.int64) + torch.as_tensor(prompt_len, dtype=torch.int64)
                       + torch.as_tensor(n_gen, dtype=torch.int64), 1, cap)


class _Chain:
    def __init__(self, chain: str, rounding: bool):
        if chain not in CHAINS:
            raise ValueError(f"unknown chain {chain!r}")
        self.fold = chain == "bf16_folded"
        self.r = rounding and chain != "fp32"

    def rnd(self, t):
        return bf16(t) if self.r else t

    def ln_proj(self, x, g, beta, W, bias):
        """the projection of LayerNorm(x): LN(x) W^T + bias, as the chain computes it"""
        W16 = self.rnd(W)
        if not self.fold:
            y = self.rnd(O.layer_norm(x, g, beta, EPS)) @ W16.T
            return y if bias is None else y + bias
        if self.r:   # vb_ln_fold_build: the fp32 product of the bf16 weight and gamma, rounded to bf16
            wf = bf16((W16.to(torch.float32) * g.to(torch.float32)).to(torch.float64))
        else:
            wf = W16 * g
        c = wf.sum(1)
        dvec = W16 @ beta
        if bias is not None:
            dvec = dvec + bias
        d = x.shape[1]
        mean = x.sum(1, keepdim=True) / d
        var = torch.clamp((x * x).sum(1, keepdim=True) / d - mean * mean, min=0.0)
        rstd = 1.0 / torch.sqrt(var + EPS)
        return rstd * (self.rnd(x) @ wf.T - mean * c) + dvec


def _attend(q, k, v, kc, vc, kv_len, finished):
    """q, k, v [B, H, 64] of the current token; kc, vc [B, H, cap, 64]; row b attends to cache rows [0, kv_len[b])
    with row kv_len[b] - 1 replaced by (k, v)"""
    out = torch.zeros_like(q)
    for b in range(q.shape[0]):
        if finished[b]:
            continue
        n = int(kv_len[b])
        K = kc[b, :, :n].clone()
        V = vc[b, :, :n].clone()
        K[:, n - 1] = k[b]
        V[:, n - 1] = v[b]
        s = torch.einsum("hd,hnd->hn", q[b] * 0.125, K)
        out[b] = torch.einsum("hn,hnd->hd", torch.softmax(s, dim=-1), V)
    return out


def decode_step(sd, prefix: str, head_w: torch.Tensor, x, kcache, vcache, text_len, prompt_len, n_gen, finished,
                nhead: int, chain: str, norm_first: bool = True, rounding: bool = True) -> StepOut:
    """one vb_ar_decode_step (greedy = 0) of every row; see the module docstring"""
    if chain in ("bf16_unfolded", "bf16_folded") and not norm_first:
        raise ValueError(f"{chain} is a pre-LN chain")
    if chain == "bf16_postln" and norm_first:
        raise ValueError("bf16_postln is the post-LN chain")
    f64 = lambda t: t.detach().to(torch.float64)   # noqa: E731
    ch = _Chain(chain, rounding)
    x = f64(x)
    kc, vc = f64(kcache), f64(vcache)
    B, d = x.shape
    H = nhead
    n_layer = kc.shape[0]
    kv_len = kv_lengths(text_len, prompt_len, n_gen, kc.shape[3])
    fin = [bool(int(f)) for f in finished]
    ks, vs, qs = [], [], []
    if not norm_first:
        xn = ch.rnd(x)
    for i in range(n_layer):
        p = {k[len(f"{prefix}.layers.{i}."):]: f64(v) for k, v in sd.items() if k.startswith(f"{prefix}.layers.{i}.")}
        if norm_first:
            qkv = ch.ln_proj(x, p["norm1.weight"], p["norm1.bias"], p["self_attn.in_proj_weight"],
                             p["self_attn.in_proj_bias"])
        else:
            qkv = xn @ ch.rnd(p["self_attn.in_proj_weight"]).T + p["self_attn.in_proj_bias"]
        q = qkv[:, :d].reshape(B, H, HD)
        k = ch.rnd(qkv[:, d:2 * d]).reshape(B, H, HD)
        v = ch.rnd(qkv[:, 2 * d:]).reshape(B, H, HD)
        qs.append(q)
        ks.append(k)
        vs.append(v)
        o = _attend(q, k, v, kc[i], vc[i], kv_len, fin).reshape(B, d)
        sa = ch.rnd(o) @ ch.rnd(p["self_attn.out_proj.weight"]).T + p["self_attn.out_proj.bias"]
        if norm_first:
            x = x + sa
            h = ch.ln_proj(x, p["norm2.weight"], p["norm2.bias"], p["linear1.weight"], p["linear1.bias"])
            x = x + ch.rnd(torch.relu(h)) @ ch.rnd(p["linear2.weight"]).T + p["linear2.bias"]
        else:
            x = O.layer_norm(x + sa, p["norm1.weight"], p["norm1.bias"], EPS)
            h = ch.rnd(x) @ ch.rnd(p["linear1.weight"]).T + p["linear1.bias"]
            x = x + ch.rnd(torch.relu(h)) @ ch.rnd(p["linear2.weight"]).T + p["linear2.bias"]
            x = O.layer_norm(x, p["norm2.weight"], p["norm2.bias"], EPS)
            xn = ch.rnd(x)
    Wp = f64(head_w)
    if norm_first:
        logits = ch.ln_proj(x, f64(sd[f"{prefix}.norm.weight"]), f64(sd[f"{prefix}.norm.bias"]), Wp, None)
    else:
        logits = xn @ ch.rnd(Wp).T
    return StepOut(x, torch.stack(ks), torch.stack(vs), torch.stack(qs), logits, kv_len)
