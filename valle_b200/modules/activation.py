"""MultiheadAttention with the reference's constructor, parameter names and init order
(valle/modules/activation.py:12-197); forward = sm_90a kernels (packed in-proj GEMM,
ragged attention, out-proj GEMM).  Self-attention, batch_first, the masks of the VALL-E path.
"""
from __future__ import annotations

from typing import Optional, Tuple

import torch
from torch import Tensor, nn
from torch.nn.init import constant_, xavier_uniform_
from torch.nn.modules.linear import NonDynamicallyQuantizableLinear
from torch.nn.parameter import Parameter

from .. import _lib as L
from .. import ops


class ValleARMask:
    """Structured stand-in for the boolean [S+t, S+t] mask of valle.py:1010-1033: text rows see
    all text, audio rows see text + causal audio.  The kernels evaluate the rule
    kv_len(i) = max(S, i + 1) instead of reading a materialised mask."""

    def __init__(self, text_lens: Tensor):
        self.text_lens = text_lens


def classify_attn_mask(attn_mask, L_q: int):
    """Map the reference's `attn_mask` argument (activation.py:199-431) onto a kernel mask mode.

    None -> (VB_MASK_FULL, None, None); ValleARMask -> (VB_MASK_VALLE_AR, text_lens, None); a boolean [L, L] tensor
    (True = blocked, the form VALLE.inference builds at valle.py:1019-1033) is recognised as the VALL-E AR rule
    `kv_len(i) = max(S, i + 1)` when it has exactly that shape -> (VB_MASK_VALLE_AR, S, None); an all-False mask ->
    FULL; anything else -> (VB_MASK_DENSE, None, uint8 mask) served by the exact-order kernel."""
    if attn_mask is None:
        return L.VB_MASK_FULL, None, None
    if isinstance(attn_mask, ValleARMask):
        return L.VB_MASK_VALLE_AR, attn_mask.text_lens, None
    if not isinstance(attn_mask, Tensor) or attn_mask.dim() != 2 or attn_mask.shape != (L_q, L_q):
        raise NotImplementedError("valle_b200: attn_mask must be None, a ValleARMask or a boolean [L, L] tensor")
    if attn_mask.dtype != torch.bool:
        if attn_mask.is_floating_point():  # additive float mask: -inf = blocked (valle.py:852-861 builds these)
            if not bool(((attn_mask == 0) | (attn_mask == float("-inf"))).all()):
                raise NotImplementedError("valle_b200: float attn_mask must hold only 0 / -inf")
            attn_mask = attn_mask == float("-inf")
        else:
            attn_mask = attn_mask != 0
    if not bool(attn_mask.any()):
        return L.VB_MASK_FULL, None, None
    S = int((~attn_mask[0]).sum())
    rows = torch.arange(L_q, device=attn_mask.device)
    expect = rows[None, :] >= torch.clamp(rows + 1, min=S)[:, None]
    if torch.equal(attn_mask, expect):
        return L.VB_MASK_VALLE_AR, S, None
    return L.VB_MASK_DENSE, None, attn_mask.to(torch.uint8).contiguous()


def pack_rows(B: int, Lq: int, key_padding_mask: Optional[Tensor], device):
    """(row index of every valid position in the flattened [B*L] layout, cu_seqlens, lens) for a suffix-padding
    `key_padding_mask` (True = padding; make_pad_mask's form, valle.py:804-805)."""
    lens = torch.full((B,), Lq, dtype=torch.int32)
    if key_padding_mask is not None:
        kpm = key_padding_mask.to(torch.bool)
        lens = (~kpm).sum(dim=1).to(torch.int32).cpu()
        # suffix padding only: valid positions must be a prefix of every row
        pos = torch.arange(Lq, device=kpm.device)[None, :]
        if not torch.equal(kpm, pos >= lens.to(kpm.device)[:, None]):
            raise NotImplementedError("valle_b200: key_padding_mask must mark a padded suffix of every sequence")
    idx = torch.cat([torch.arange(int(n)) + b * Lq for b, n in enumerate(lens)]).to(device)
    cu = torch.zeros(B + 1, dtype=torch.int32)
    cu[1:] = torch.cumsum(lens, 0)
    return idx, cu.to(device), lens


class MultiheadAttention(nn.Module):
    """valle/modules/activation.py:12-431 restricted to what VALLE instantiates (:72-197: packed `in_proj_weight`
    [3d, d] + `in_proj_bias`, `out_proj` NonDynamicallyQuantizableLinear, xavier / zero init in the same order):
    forward (:199-431) = F.multi_head_attention_forward (:408-427) -> vb_linear / vb_attention / vb_linear."""
    __constants__ = ["batch_first"]

    def __init__(self, embed_dim, num_heads, dropout=0.0, bias=True, add_bias_kv=False, add_zero_attn=False,
                 kdim=None, vdim=None, batch_first=False, linear1_cls=nn.Linear, linear2_cls=nn.Linear,
                 device=None, dtype=None) -> None:
        super().__init__()
        if add_bias_kv or add_zero_attn or kdim not in (None, embed_dim) or vdim not in (None, embed_dim) \
                or linear1_cls is not nn.Linear or linear2_cls is not nn.Linear or not bias:
            raise NotImplementedError("valle_b200.MultiheadAttention: only the configuration VALLE "
                                      "instantiates (packed in-proj, bias, nn.Linear) is built")
        fk = {"device": device, "dtype": dtype}
        self.embed_dim = embed_dim
        self.kdim = self.vdim = embed_dim
        self._qkv_same_embed_dim = True
        self.num_heads = num_heads
        self.dropout = dropout
        self.batch_first = batch_first
        self.head_dim = embed_dim // num_heads
        assert self.head_dim * num_heads == embed_dim, "embed_dim must be divisible by num_heads"
        self.bias_k = self.bias_v = None
        self.in_proj_weight = Parameter(torch.empty((3 * embed_dim, embed_dim), **fk))
        self.register_parameter("q_proj_weight", None)
        self.register_parameter("k_proj_weight", None)
        self.register_parameter("v_proj_weight", None)
        self.in_proj_bias = Parameter(torch.empty(3 * embed_dim, **fk))
        self.out_proj = NonDynamicallyQuantizableLinear(embed_dim, embed_dim, bias=True, **fk)
        self.add_zero_attn = False
        xavier_uniform_(self.in_proj_weight)
        constant_(self.in_proj_bias, 0.0)
        constant_(self.out_proj.bias, 0.0)

    def forward(self, query: Tensor, key: Tensor, value: Tensor, key_padding_mask: Optional[Tensor] = None,
                need_weights: bool = True, attn_mask=None, average_attn_weights: bool = True
                ) -> Tuple[Tensor, Optional[Tensor]]:
        if not (query is key and key is value):
            raise NotImplementedError("valle_b200.MultiheadAttention: self-attention only")
        if not self.batch_first or need_weights:
            raise NotImplementedError("valle_b200.MultiheadAttention: batch_first=True, need_weights=False only")
        B, Lq, d = query.shape
        x = query.reshape(B * Lq, d).to(torch.float32).contiguous()
        idx, cu, lens = pack_rows(B, Lq, key_padding_mask, x.device)
        xp = x.index_select(0, idx)   # pack valid rows of every sequence
        mode, tl, dense = classify_attn_mask(attn_mask, Lq)
        o = self.attend_packed(xp, cu, int(lens.max()), B, mode, tl, dense)
        o = ops.linear(o, self.out_proj.weight.detach(), self.out_proj.bias.detach())
        out = torch.zeros_like(x)
        out.index_copy_(0, idx, o)
        return out.view(B, Lq, d), None

    def attend_packed(self, xp: Tensor, cu: Tensor, max_len: int, B: int, mode: int, tl, dense) -> Tensor:
        """in-proj + scaled-dot-product attention over packed rows (before out_proj)"""
        if mode == L.VB_MASK_VALLE_AR:
            if isinstance(tl, int):
                tl = torch.full((B,), tl, dtype=torch.int32)
            tl = tl.to(device=xp.device, dtype=torch.int32)
        qkv = ops.linear(xp, self.in_proj_weight.detach(), self.in_proj_bias.detach())
        return ops.attention(qkv, cu, max_len, self.num_heads, mode, tl, dense_mask=dense)
