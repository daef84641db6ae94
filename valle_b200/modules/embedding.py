"""TokenEmbedding / SinePositionalEmbedding with the reference's constructor signatures,
parameter names (checkpoint layout) and init order -- forward runs on the sm_90a kernels.

Mirrors valle/modules/embedding.py:21-97 (interface); arithmetic: csrc/embed_norm.cu.
"""
from __future__ import annotations

import math

import torch
import torch.nn as nn

from .. import ops


def build_sine_pe(n: int, dim_model: int) -> torch.Tensor:
    """fp32 sin/cos table built on the CPU exactly as embedding.py:75-91 does (device sinf/cosf
    would drift by ULPs), then shipped to the device once."""
    pe = torch.zeros(n, dim_model)
    position = torch.arange(0, n, dtype=torch.float32).unsqueeze(1)
    div_term = torch.exp(torch.arange(0, dim_model, 2, dtype=torch.float32) * -(math.log(10000.0) / dim_model))
    pe[:, 0::2] = torch.sin(position * div_term)
    pe[:, 1::2] = torch.cos(position * div_term)
    return pe


class TokenEmbedding(nn.Module):
    """valle/modules/embedding.py:21-47: nn.Embedding under `word_embeddings` (same parameter name, so checkpoints
    load unchanged), `weight` / `embedding(i)` accessors, forward = lookup (+ dropout, identity in eval) -> vb_embed_sum."""
    def __init__(self, dim_model: int, vocab_size: int, dropout: float = 0.0):
        super().__init__()
        self.vocab_size = vocab_size
        self.dim_model = dim_model
        self.dropout = torch.nn.Dropout(p=dropout)
        self.word_embeddings = nn.Embedding(self.vocab_size, self.dim_model)

    @property
    def weight(self) -> torch.Tensor:
        return self.word_embeddings.weight

    def embedding(self, index: int) -> torch.Tensor:
        return self.word_embeddings.weight[index: index + 1]

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        if self.training and self.dropout.p > 0:
            raise NotImplementedError("valle_b200: the module-level forward is inference only (training-mode dropout "
                                      "is applied by VALLE.forward, valle_b200/train_forward.py); call .eval()")
        w = self.word_embeddings.weight
        tok = x.reshape(-1).to(torch.int64).contiguous()
        out = torch.empty((tok.numel(), self.dim_model), dtype=torch.float32, device=w.device)
        ops.embed_sum(tok, 1, 0, [w.detach()], tok.numel(), out)
        return out.view(*x.shape, self.dim_model)


class SinePositionalEmbedding(nn.Module):
    """valle/modules/embedding.py:50-97: x * x_scale + alpha * pe[:, :T] with the sine table of :68-91 (built on the
    CPU with the reference's own expression, kept as a plain attribute like :65, never in the checkpoint); `alpha`
    is the only parameter.  forward -> vb_add_pe."""
    def __init__(self, dim_model: int, dropout: float = 0.0, scale: bool = False, alpha: bool = False):
        super().__init__()
        self.dim_model = dim_model
        self.x_scale = math.sqrt(dim_model) if scale else 1.0
        self.alpha = nn.Parameter(torch.ones(1), requires_grad=alpha)
        self.dropout = torch.nn.Dropout(p=dropout)
        self.reverse = False
        self.pe = None  # plain attribute, NOT in the checkpoint (embedding.py:65)
        self._pe_rows = 0

    def table(self, n: int, device) -> torch.Tensor:
        """fp32 [rows >= n, d] table on `device` (auto-extends like embedding.py:68-91)."""
        if self.pe is None or self._pe_rows < n or self.pe.device != torch.device(device):
            rows = max(4000, int(n))
            self.pe = build_sine_pe(rows, self.dim_model).to(device)
            self._pe_rows = rows
        return self.pe

    def extend_pe(self, x: torch.Tensor) -> None:
        self.table(x.size(1), x.device)

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        if self.x_scale != 1.0:
            raise NotImplementedError("valle_b200: scale=True is not on the VALL-E path")
        if self.training and self.dropout.p > 0:
            raise NotImplementedError("valle_b200: the module-level forward is inference only (training-mode dropout "
                                      "is applied by VALLE.forward, valle_b200/train_forward.py); call .eval()")
        assert x.dim() == 3 and x.dtype == torch.float32
        B, T, d = x.shape
        pe = self.table(T, x.device)
        x = x.contiguous()
        out = torch.empty_like(x)
        for b in range(B):
            ops.add_pe(x[b], pe, self.alpha.detach(), out[b], T, pos0=0)
        return out
