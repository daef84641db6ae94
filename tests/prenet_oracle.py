"""TEST INFRASTRUCTURE ONLY -- the pre-nets (`add_prenet=True`) in the training loss, on top of the oracle's
forward_train (oracle/valle_oracle.py).

valle/models/valle.py:96-123 / 181-213, applied between embedding and positional encoding (:829-831, :863-865,
:897-899, :918-919):
    text:  Transpose -> 3 x [Conv1d(C, C, 5, padding="same") -> BatchNorm1d(C) -> ReLU -> Dropout(0.5)] -> Transpose
           -> Linear(C, C), over the padded batch [N, Smax, C]
    audio: Linear(C, 256) -> ReLU -> Dropout(0.25) -> Linear(256, 256) -> ReLU -> Dropout(0.25) -> Linear(256, C)
Dropout is left out (the comparisons run every Dropout at p = 0).  In training mode BatchNorm normalises by the batch
statistics over all N * Smax positions, padding included (F.batch_norm(training=True)), and updates copies of the
running statistics, which forward_train returns.

Every other step is the oracle's: its forward_train reaches the positional encoding through the module attribute
`pos_embed`, which `forward_train` below points at a wrapper that applies the pre-net of the site first (the site is
told apart by its `*_position.alpha` tensor).  Combine with postln_oracle.post_ln() for post-LN stacks.
"""
from __future__ import annotations

from typing import Dict

import torch
import torch.nn.functional as F

from oracle import valle_oracle as O

BN_EPS, BN_MOMENTUM = 1e-5, 0.1   # nn.BatchNorm1d defaults, as the reference builds them
SITES = ("ar_text", "ar_audio", "nar_text", "nar_audio")
SAMPLES = 32   # gradient elements per parameter in tests/golden/prenet_train.pt


def sample_positions(name: str, numel: int) -> torch.Tensor:
    """SAMPLES element positions of a parameter's flattened gradient, seeded by its name"""
    g = torch.Generator().manual_seed(sum((i + 1) * ord(ch) for i, ch in enumerate(name)))
    return torch.randint(0, numel, (SAMPLES,), generator=g)


def _conv5(h, w, b):
    """Conv1d(k=5, padding="same") of h [N, T, C] as a linear over the five shifted copies (the engine's im2col form),
    through O.F.linear so that postln_oracle.bf16_gemm_operands() rounds its operands"""
    T = h.shape[1]
    hp = F.pad(h, (0, 0, 2, 2))
    col = torch.cat([hp[:, k:k + T] for k in range(5)], dim=2)
    return O.F.linear(col, w.permute(0, 2, 1).reshape(w.shape[0], -1), b)


def text_prenet(sd, prefix: str, x: torch.Tensor, training: bool, buffers: Dict[str, torch.Tensor]) -> torch.Tensor:
    """x [N, T, C] -> [N, T, C]; `buffers` holds (and receives the updates of) the running statistics"""
    h = x
    for i in (1, 5, 9):
        h = _conv5(h, sd[f"{prefix}.{i}.weight"], sd[f"{prefix}.{i}.bias"]).transpose(1, 2)
        k = f"{prefix}.{i + 1}."
        for b in ("running_mean", "running_var", "num_batches_tracked"):
            buffers.setdefault(k + b, sd[k + b].detach().clone())
        h = F.batch_norm(h, buffers[k + "running_mean"], buffers[k + "running_var"], sd[k + "weight"], sd[k + "bias"],
                         training=training, momentum=BN_MOMENTUM, eps=BN_EPS)
        if training:
            buffers[k + "num_batches_tracked"] += 1
        h = F.relu(h).transpose(1, 2)
    return O.F.linear(h, sd[f"{prefix}.14.weight"], sd[f"{prefix}.14.bias"])


def audio_prenet(sd, prefix: str, x: torch.Tensor) -> torch.Tensor:
    h = F.relu(O.F.linear(x, sd[f"{prefix}.0.weight"], sd[f"{prefix}.0.bias"]))
    h = F.relu(O.F.linear(h, sd[f"{prefix}.3.weight"], sd[f"{prefix}.3.bias"]))
    return O.F.linear(h, sd[f"{prefix}.6.weight"], sd[f"{prefix}.6.bias"])


def forward_train(sd, cfg: O.OracleConfig, *args, training: bool = True, **kwargs):
    """O.forward_train with the pre-nets of the state dict (plain O.forward_train when it has none); BatchNorm on batch
    statistics when `training`, else on the running statistics.  Returns (loss, aux, buffers after the call)."""
    if "ar_text_prenet.1.weight" not in sd:
        loss, aux = O.forward_train(sd, cfg, *args, **kwargs)
        return loss, aux, {}
    buffers: Dict[str, torch.Tensor] = {}
    site_of = {id(sd[f"{s}_position.alpha"]): s for s in SITES}
    plain = O.pos_embed

    def pos_embed(x, alpha, start=0):
        s = site_of.get(id(alpha))
        if s in ("ar_text", "nar_text"):
            x = text_prenet(sd, s + "_prenet", x, training, buffers)
        elif s is not None:
            x = audio_prenet(sd, s + "_prenet", x)
        return plain(x, alpha, start)

    O.pos_embed = pos_embed
    try:
        loss, aux = O.forward_train(sd, cfg, *args, **kwargs)
    finally:
        O.pos_embed = plain
    for k, v in sd.items():   # buffers of pre-nets the call did not reach stay as they were
        if k.endswith(("running_mean", "running_var", "num_batches_tracked")):
            buffers.setdefault(k, v.detach().clone())
    return loss, aux, buffers
