"""TEST INFRASTRUCTURE ONLY -- the post-LN (`norm_first=False`) restatement of the reference's decoder stack, on top
of the pre-LN oracle in oracle/valle_oracle.py.

valle/modules/transformer.py:303-308 (post-LN layer):
    x = norm1(x + SA(x), stage_embedding);  x = norm2(x + FF(x), stage_embedding)
and valle/models/valle.py:151,242-246: VALLE builds its post-LN stacks without a final norm.

Every other step of inference, continual and the training loss is the pre-LN oracle's: its functions reach the stack
through the module attribute `encoder`, which `post_ln()` points at `encoder_postln` for the duration of a call.
"""
from __future__ import annotations

import contextlib
from typing import Dict, Optional

import torch
import torch.nn.functional as F

from oracle import valle_oracle as O


def encoder_postln(sd: Dict[str, torch.Tensor], prefix: str, x: torch.Tensor, cfg: O.OracleConfig,
                   blocked=None, key_padding=None, stage_emb: Optional[torch.Tensor] = None):
    """transformer.py:363-406 over post-LN layers; the final norm only if the state dict has one (VALLE's do not)"""
    adaptive = stage_emb is not None

    def norm(h, p):
        if adaptive:   # transformer.py:93-108; the (weight | bias) projection stays fp32, as in the engine
            wb = F.linear(stage_emb, sd[p + "project_layer.weight"], sd[p + "project_layer.bias"])
            d = h.shape[-1]
            return wb[..., :d] * O.layer_norm(h, sd[p + "norm.weight"], sd[p + "norm.bias"]) + wb[..., d:]
        return O.layer_norm(h, sd[p + "weight"], sd[p + "bias"])

    for i in range(cfg.num_layers):
        p = O._layer_keys(prefix, i)
        x = norm(x + O.mha(x, sd[p + "self_attn.in_proj_weight"], sd[p + "self_attn.in_proj_bias"],
                           sd[p + "self_attn.out_proj.weight"], sd[p + "self_attn.out_proj.bias"],
                           cfg.nhead, blocked, key_padding), p + "norm1.")
        x = norm(x + O.F.linear(F.relu(O.F.linear(x, sd[p + "linear1.weight"], sd[p + "linear1.bias"])),
                                sd[p + "linear2.weight"], sd[p + "linear2.bias"]), p + "norm2.")
    if any(k.startswith(prefix + ".norm.") for k in sd):
        x = norm(x, prefix + ".norm.")
    return x


def _no_postln_kv(*args, **kwargs):
    raise NotImplementedError("postln_oracle: ar_decode_kv restates pre-LN layers only")


@contextlib.contextmanager
def post_ln():
    """the pre-LN oracle's inference / continual / forward_train / nar_logits_forced with post-LN stacks inside the
    block (they reach the stack through the module attribute `encoder`); ar_decode_kv, which has its own pre-LN layer
    loop, raises there"""
    saved = O.encoder, O.ar_decode_kv
    O.encoder, O.ar_decode_kv = encoder_postln, _no_postln_kv
    try:
        yield
    finally:
        O.encoder, O.ar_decode_kv = saved


def inference(*args, **kwargs):
    with post_ln():
        return O.inference(*args, **kwargs)


def continual(*args, **kwargs):
    with post_ln():
        return O.continual(*args, **kwargs)


def forward_train(*args, **kwargs):
    with post_ln():
        return O.forward_train(*args, **kwargs)


def nar_logits_forced(sd, cfg: O.OracleConfig, x, y, codes):
    """valle.py:1063-1134 teacher-forced: the 7 NAR stages' logits [T, 1024] when the stages' ids are `codes` [1, T, 8]
    (the generated frames; the prompt y [1, Tp, 8]) instead of each stage's argmax (prefix_mode 1 layout)"""
    assert cfg.prefix_mode == 1
    S, Tp = x.shape[1], y.shape[1]
    yy = torch.cat([y[..., 0], codes[..., 0]], 1)
    y_emb = sd["nar_audio_embeddings.0.word_embeddings.weight"][yy].clone()
    for j in range(1, cfg.num_quantizers):
        y_emb[:, :Tp] += sd[f"nar_audio_embeddings.{j}.word_embeddings.weight"][y[..., j]]
    xe = O.pos_embed(sd["nar_text_embedding.word_embeddings.weight"][x], sd["nar_text_position.alpha"])
    out = []
    for i in range(cfg.num_quantizers - 1):
        xy = torch.cat([xe, O.pos_embed(y_emb, sd["nar_audio_position.alpha"])], dim=1)
        dec = O.encoder(sd, "nar_decoder", xy, cfg, stage_emb=sd[f"nar_stage_embeddings.{i}.word_embeddings.weight"])
        out.append(O.F.linear(dec[0, S + Tp:], sd[f"nar_predict_layers.{i}.weight"]))
        if i < cfg.num_quantizers - 2:
            y_emb[:, Tp:] += sd[f"nar_audio_embeddings.{i + 1}.word_embeddings.weight"][codes[..., i + 1]]
    return out


class _RoundBf16(torch.autograd.Function):
    """forward: the value rounded to bf16 (a GEMM operand the engine stores in bf16); backward: the gradient unchanged"""

    @staticmethod
    def forward(ctx, t):
        return t.to(torch.bfloat16).float()

    @staticmethod
    def backward(ctx, g):
        return g


class _RoundGradBf16(torch.autograd.Function):
    """forward: identity; backward: the gradient rounded to bf16 (the dY operand of the engine's dgrad / wgrad GEMMs)"""

    @staticmethod
    def forward(ctx, t):
        return t.clone()

    @staticmethod
    def backward(ctx, g):
        return g.to(torch.bfloat16).float()


class _Bf16Linear:
    """torch.nn.functional with `linear` on bf16-rounded operands (fp32 accumulation) and a bf16-rounded output gradient"""

    def __getattr__(self, name):
        return getattr(F, name)

    @staticmethod
    def linear(x, w, b=None):
        return _RoundGradBf16.apply(F.linear(_RoundBf16.apply(x), _RoundBf16.apply(w), b))


@contextlib.contextmanager
def bf16_gemm_operands():
    """the oracle's arithmetic with every GEMM operand rounded to bf16 and accumulated in fp32, and every GEMM's output
    gradient rounded to bf16 -- what bf16 storage does to the reference computation itself, independent of the engine's
    kernels.  The bf16 bars of the tests are this restatement's own error where it exceeds the fixed bars."""
    saved = O.F
    O.F = _Bf16Linear()
    try:
        yield
    finally:
        O.F = saved
