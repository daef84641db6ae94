"""Op-level Python wrappers over the C ABI (torch tensors in, torch tensors out).

torch is used for allocation and stream selection only; every computation is a kernel of
libvalle_b200.so.  All tensors must be CUDA and contiguous; there is no CPU path.
"""
from __future__ import annotations

import ctypes as C
from typing import List, Optional, Sequence

import torch

from . import _lib as L

_DT = {torch.float32: L.VB_F32, torch.bfloat16: L.VB_BF16}


def _req_cuda(*ts):
    for t in ts:
        if t is not None and not t.is_cuda:
            raise L.VbError("valle_b200 kernels need CUDA tensors; there is no CPU fallback")


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def _dev_guard(fn):
    """Launch on the GPU the tensors live on: the first CUDA tensor argument's device becomes the current device for
    the call, so the stream, the per-device function attributes and the SM count all belong to that GPU even when
    the caller's current device is another one."""
    import functools

    @functools.wraps(fn)
    def wrapper(*args, **kwargs):
        for a in args:
            if isinstance(a, torch.Tensor) and a.is_cuda:
                if a.device.index == torch.cuda.current_device():
                    break
                with torch.cuda.device(a.device):
                    return fn(*args, **kwargs)
        return fn(*args, **kwargs)
    return wrapper


def table_array(tables: Sequence[torch.Tensor]):
    arr = (C.c_void_p * len(tables))(*[t.data_ptr() for t in tables])
    return arr


_OOB: dict = {}


def oob_flag(device) -> torch.Tensor:
    """per-device int32 flag the embedding kernels raise when a token id is outside its table"""
    device = torch.device(device)
    key = device.index if device.index is not None else torch.cuda.current_device()
    f = _OOB.get(key)
    if f is None:
        f = torch.zeros(1, dtype=torch.int32, device=torch.device("cuda", key))
        _OOB[key] = f
    return f


def check_oob(device) -> None:
    """nn.Embedding's contract (valle/modules/embedding.py:46): an id outside the table is an IndexError.
    The kernels clamp the read and raise the device flag; this reads it (one D2H sync) and reports."""
    f = oob_flag(device)
    if int(f.item()) != 0:
        f.zero_()
        raise IndexError("index out of range in self (token id outside its embedding table)")


@_dev_guard
def embed_sum(tokens: torch.Tensor, tok_row_stride: int, tok_tab_stride: int,
              tables: Sequence[torch.Tensor], n_rows: int, out: torch.Tensor,
              out_rows: Optional[torch.Tensor] = None, accumulate: bool = False) -> torch.Tensor:
    """out[orow(r)] (=|+=) sum_j tables[j][tokens[r*row_stride + j*tab_stride]]  (valle.py:1064,1110-1113).
    Ids outside a table are clamped and flagged (see check_oob)."""
    _req_cuda(tokens, out, *tables)
    assert tokens.dtype == torch.int64 and out.dtype == torch.float32
    d = out.shape[-1]
    lib = L.load()
    rows = (C.c_int32 * len(tables))(*[int(t.shape[0]) for t in tables])
    L.check(lib.vb_embed_sum(tokens.data_ptr(), tok_row_stride, tok_tab_stride, table_array(tables), rows,
                             len(tables), n_rows, d, out.data_ptr(), out.stride(-2) if out.dim() > 1 else d,
                             L.ptr(out_rows), int(accumulate), oob_flag(out.device).data_ptr(), _stream()),
            "vb_embed_sum")
    return out


@_dev_guard
def add_pe(inp: torch.Tensor, pe: torch.Tensor, alpha: torch.Tensor, out: torch.Tensor, n_rows: int,
           pos0: int = 0, positions: Optional[torch.Tensor] = None,
           out_rows: Optional[torch.Tensor] = None) -> torch.Tensor:
    """out[orow(r)] = inp[r] + alpha * pe[pos(r)]  (embedding.py:93-97)."""
    _req_cuda(inp, pe, alpha, out)
    d = inp.shape[-1]
    lib = L.load()
    L.check(lib.vb_add_pe(inp.data_ptr(), inp.stride(-2) if inp.dim() > 1 else d, pe.data_ptr(), pos0,
                          L.ptr(positions), alpha.data_ptr(), n_rows, d, out.data_ptr(),
                          out.stride(-2) if out.dim() > 1 else d, L.ptr(out_rows), _stream()), "vb_add_pe")
    return out


@_dev_guard
def layernorm(x: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, eps: float = 1e-5,
              ada_wb: Optional[torch.Tensor] = None, rows: Optional[torch.Tensor] = None,
              out_dtype: torch.dtype = torch.float32, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """LayerNorm / AdaptiveLayerNorm over the last dim of a [R, d] fp32 tensor (transformer.py:57-108)."""
    _req_cuda(x, gamma, beta)
    assert x.dtype == torch.float32 and x.dim() == 2
    d = x.shape[1]
    n = x.shape[0] if rows is None else rows.numel()
    if out is None:
        out = torch.empty((n, d), dtype=out_dtype, device=x.device)
    lib = L.load()
    L.check(lib.vb_layernorm(x.data_ptr(), x.stride(0), L.ptr(rows), n, d, gamma.data_ptr(), beta.data_ptr(),
                             L.ptr(ada_wb), eps, out.data_ptr(), _DT[out.dtype], _stream()), "vb_layernorm")
    return out


@_dev_guard
def adaln_project(W: torch.Tensor, b: torch.Tensor, emb: torch.Tensor, out: Optional[torch.Tensor] = None):
    """(weight | bias) = project_layer(stage_embedding)  (transformer.py:96-100)."""
    _req_cuda(W, b, emb)
    d = W.shape[1]
    if out is None:
        out = torch.empty(2 * d, dtype=torch.float32, device=W.device)
    L.check(L.load().vb_adaln_project(W.data_ptr(), b.data_ptr(), emb.data_ptr(), d, out.data_ptr(), _stream()),
            "vb_adaln_project")
    return out


@_dev_guard
def linear(a: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor] = None, epilogue: int = L.VB_EPI_NONE,
           out: Optional[torch.Tensor] = None, out_dtype: Optional[torch.dtype] = None) -> torch.Tensor:
    """C = epi(A W^T + b)  (F.linear; transformer.py:332-334, activation.py:408, valle.py:1039,1128)."""
    _req_cuda(a, w, bias)
    assert a.dim() == 2 and w.dim() == 2 and a.dtype == w.dtype and a.shape[1] == w.shape[1]
    M, K = a.shape
    N = w.shape[0]
    if out is None:
        assert epilogue != L.VB_EPI_RESIDUAL
        out = torch.empty((M, N), dtype=out_dtype or a.dtype, device=a.device)
    L.check(L.load().vb_linear(a.data_ptr(), _DT[a.dtype], a.stride(0), w.data_ptr(), _DT[w.dtype], L.ptr(bias),
                               out.data_ptr(), _DT[out.dtype], out.stride(0), M, N, K, epilogue, 0, 0,
                               _stream()), "vb_linear")
    return out


@_dev_guard
def attention(qkv: torch.Tensor, cu_seqlens: torch.Tensor, max_seqlen: int, n_head: int,
              mask_mode: int = L.VB_MASK_FULL, text_lens: Optional[torch.Tensor] = None,
              out: Optional[torch.Tensor] = None, seg1_lens: Optional[torch.Tensor] = None,
              seg1_start: int = 0, dense_mask: Optional[torch.Tensor] = None) -> torch.Tensor:
    """softmax(q k^T / sqrt(hd) + mask) v over packed ragged sequences (activation.py:408-427).
    dense_mask: bool / uint8 [L, L] `attn_mask` tensor (True = blocked) for mask_mode VB_MASK_DENSE."""
    _req_cuda(qkv, cu_seqlens, text_lens, dense_mask)
    dm_ptr, dm_ld = 0, 0
    if mask_mode == L.VB_MASK_DENSE:
        assert dense_mask is not None and dense_mask.dim() == 2
        dense_mask = dense_mask.to(torch.uint8).contiguous()
        dm_ptr, dm_ld = dense_mask.data_ptr(), dense_mask.stride(0)
    M, d3 = qkv.shape
    d = d3 // 3
    if out is None:
        out = torch.empty((M, d), dtype=qkv.dtype, device=qkv.device)
    B = cu_seqlens.numel() - 1
    L.check(L.load().vb_attention(qkv.data_ptr(), _DT[qkv.dtype], M, B, n_head, d // n_head, cu_seqlens.data_ptr(),
                                  L.ptr(text_lens), L.ptr(seg1_lens), seg1_start, max_seqlen, mask_mode, out.data_ptr(), 0, 0, 0, 0,
                                  dm_ptr, dm_ld, _stream()),
            "vb_attention")
    return out


@_dev_guard
def gather_rows(src: torch.Tensor, rows: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    _req_cuda(src, rows)
    d = src.shape[1]
    n = rows.numel()
    if out is None:
        out = torch.empty((n, d), dtype=torch.float32, device=src.device)
    L.check(L.load().vb_gather_rows(src.data_ptr(), src.stride(0), rows.data_ptr(), n, d, out.data_ptr(),
                                    out.stride(0), _stream()), "vb_gather_rows")
    return out


@_dev_guard
def cast_from_f32(x: torch.Tensor, dtype: torch.dtype) -> torch.Tensor:
    """x (contiguous fp32) rounded to `dtype` (a copy for fp32), vb_cast_from_f32"""
    _req_cuda(x)
    assert x.dtype == torch.float32 and x.is_contiguous()
    out = torch.empty(x.shape, dtype=dtype, device=x.device)
    L.check(L.load().vb_cast_from_f32(x.data_ptr(), out.data_ptr(), _DT[dtype], x.numel(), _stream()),
            "vb_cast_from_f32")
    return out


@_dev_guard
def nar_argmax_accumulate(logits: torch.Tensor, codes: torch.Tensor, code_row_stride: int,
                          next_emb: Optional[torch.Tensor], y_emb: Optional[torch.Tensor],
                          y_rows: Optional[torch.Tensor] = None) -> None:
    """samples = argmax(logits); y_emb += next_emb[samples]  (valle.py:1130-1134)."""
    _req_cuda(logits, codes, next_emb, y_emb)
    n, V = logits.shape
    d = y_emb.shape[1] if y_emb is not None else 4
    L.check(L.load().vb_nar_argmax_accumulate(logits.data_ptr(), n, V, logits.stride(0), codes.data_ptr(),
                                              code_row_stride, L.ptr(next_emb), L.ptr(y_emb),
                                              y_emb.stride(0) if y_emb is not None else 0, L.ptr(y_rows), d, _stream()),
            "vb_nar_argmax_accumulate")


@_dev_guard
def cross_entropy_rows(logits: torch.Tensor, targets: torch.Tensor, ignore_index: int = -1) -> torch.Tensor:
    """per-row F.cross_entropy (valle.py:877,936-941); ignored rows give 0."""
    _req_cuda(logits, targets)
    assert logits.dtype == torch.float32 and targets.dtype == torch.int64 and logits.dim() == 2
    n, V = logits.shape
    out = torch.empty(n, dtype=torch.float32, device=logits.device)
    L.check(L.load().vb_cross_entropy(logits.data_ptr(), logits.stride(0), targets.data_ptr(), n, V, ignore_index,
                                      out.data_ptr(), _stream()), "vb_cross_entropy")
    return out


@_dev_guard
def sample_logits(logits: torch.Tensor, top_k, temperature, seeds, steps, top_p=None, ras_window=None, ras_max=None,
                  tokens: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Seeded top-k / temperature draw per row of fp32 logits [R, V] (V <= 1280; a row stride of 0, e.g. from
    `expand`, draws R times from one row), vb_sample_logits: top_k / temperature / seeds / steps are one value or one
    per row; seeds are uint64 values (int64 bit patterns accepted).  Returns int64 ids [R].
    top_p, ras_window / ras_max (one value or one per row) and tokens (int32 [R, >= max step] history, row stride
    free) select vb_sample_logits_ex: nucleus filtering and repetition-aware sampling."""
    _req_cuda(logits)
    assert logits.dtype == torch.float32 and logits.dim() == 2 and logits.stride(1) == 1
    R, V = logits.shape
    dev = logits.device

    def rows(v, dtype):
        t = v.to(dev, dtype) if isinstance(v, torch.Tensor) else torch.as_tensor(v, dtype=dtype, device=dev)
        return t.expand(R).contiguous() if t.numel() == 1 else t.reshape(R).contiguous()

    if not isinstance(seeds, torch.Tensor):
        seeds = [int(x) - (1 << 64) if int(x) >= 1 << 63 else int(x) for x in
                 (seeds if isinstance(seeds, (list, tuple)) else [seeds])]
    sd, st = rows(seeds, torch.int64), rows(steps, torch.int32)
    k, t = rows(top_k, torch.int32), rows(temperature, torch.float32)
    out = torch.empty(R, dtype=torch.int64, device=dev)
    if top_p is not None or ras_window is not None:
        p = rows(top_p, torch.float32) if top_p is not None else None
        rw = rm = None
        tok_ld = 0
        if ras_window is not None:
            rw, rm = rows(ras_window, torch.int32), rows(ras_max, torch.int32)
            assert tokens is not None and tokens.dtype == torch.int32 and tokens.dim() == 2 and tokens.stride(1) == 1
            tokens = tokens.to(dev)
            tok_ld = tokens.stride(0)
        L.check(L.load().vb_sample_logits_ex(logits.data_ptr(), logits.stride(0), R, V, sd.data_ptr(), st.data_ptr(),
                                             k.data_ptr(), t.data_ptr(), L.ptr(p), L.ptr(rw), L.ptr(rm),
                                             L.ptr(tokens if rw is not None else None), tok_ld, out.data_ptr(),
                                             _stream()), "vb_sample_logits_ex")
        return out
    L.check(L.load().vb_sample_logits(logits.data_ptr(), logits.stride(0), R, V, sd.data_ptr(), st.data_ptr(),
                                      k.data_ptr(), t.data_ptr(), out.data_ptr(), _stream()), "vb_sample_logits")
    return out
