"""Float64 restatements of the EnCodec building blocks behind `csrc/encodec.cu`, written from their definitions.

Each function works on whatever device its tensors live on and in their dtype (the tests pass float64; the LSTM is
also run in float32 to size the error of an fp32 recurrence).  `tests/test_codec_oracle64.py` pins them against torch
(`F.conv1d`, `F.conv_transpose1d`, `nn.LSTM`) and the HF EnCodec modules on the CPU; `tests/test_codec_kernels_gpu.py`
compares the kernels with them.
"""
from __future__ import annotations

import math

import torch


def elu(x: torch.Tensor) -> torch.Tensor:
    return torch.where(x > 0, x, torch.expm1(x))


def pad_index(T: int, pad_left: int, pad_right: int, reflect: bool):
    """source index and validity of every sample of the padded signal (length T + pad_left + pad_right).

    Zero padding: sample g of x for 0 <= g < T, else 0.  Reflect (EnCodec's pad1d): x is zero-extended to
    Te = max(T, max pad + 1) samples, reflected over those (g < 0 -> -g, g >= Te -> 2 (Te - 1) - g), and the
    extension trimmed again; a reflected index that lands in the extension reads 0."""
    g = torch.arange(-pad_left, T + pad_right)
    if reflect:
        te = max(T, max(pad_left, pad_right) + 1)
        g = torch.where(g < 0, -g, g)
        g = torch.where(g >= te, 2 * (te - 1) - g, g)
    valid = (g >= 0) & (g < T)
    return g.clamp(0, max(T - 1, 0)), valid


def pad1d(x: torch.Tensor, pad_left: int, pad_right: int, reflect: bool) -> torch.Tensor:
    idx, valid = pad_index(x.shape[-1], pad_left, pad_right, reflect)
    return torch.where(valid.to(x.device), x[..., idx.to(x.device)], torch.zeros((), dtype=x.dtype, device=x.device))


def encodec_pads(T: int, K: int, stride: int = 1, dilation: int = 1, causal: bool = True):
    """(pad_left, pad_right) of EnCodec's SConv1d: padding_total = K_eff - stride, plus the extra right padding that
    completes the last window; causal puts padding_total on the left, otherwise it is split with the odd sample left."""
    k_eff = (K - 1) * dilation + 1
    total = k_eff - stride
    n = T - k_eff + total
    n_frames = -(-n // stride)                           # ceil((T - K_eff + total) / stride + 1) - 1
    extra = n_frames * stride + k_eff - total - T
    if causal:
        return total, extra
    right = total // 2
    return total - right, right + extra


def conv1d(x: torch.Tensor, w: torch.Tensor, bias=None, stride: int = 1, dilation: int = 1, pad_left: int = 0,
           pad_right: int = 0, reflect: bool = False, pre_elu: bool = False, residual=None, phase: int = 1):
    """y[b, co, t] = bias[co // phase] + sum_{ci,k} w[co, ci, k] act(x)[b, ci, t stride - pad_left + k dilation]
    (+ residual), act = ELU if pre_elu, padding per `pad_index`.  phase > 1 interleaves channel co = c phase + r
    into out[b, c, t phase + r].  Returns (y, s): s = sum |w act(x)| + |bias| + |residual| per output, the magnitude
    the kernel's rounding scales with."""
    B, Cin, T = x.shape
    Cout, _, K = w.shape
    a = elu(x) if pre_elu else x
    xp = pad1d(a, pad_left, pad_right, reflect)
    Tout = (xp.shape[-1] - (K - 1) * dilation - 1) // stride + 1
    y = x.new_zeros((B, Cout, Tout))
    s = x.new_zeros((B, Cout, Tout))
    for k in range(K):
        tap = xp[..., k * dilation: k * dilation + (Tout - 1) * stride + 1: stride]       # [B, Cin, Tout]
        y += torch.einsum("oc,bct->bot", w[:, :, k], tap)
        s += torch.einsum("oc,bct->bot", w[:, :, k].abs(), tap.abs())
    if bias is not None:
        bb = bias.repeat_interleave(phase)[None, :, None]
        y, s = y + bb, s + bb.abs()
    if phase > 1:
        def interleave(v):
            return v.view(B, Cout // phase, phase, Tout).permute(0, 1, 3, 2).reshape(B, Cout // phase, Tout * phase)
        y, s = interleave(y), interleave(s)
    if residual is not None:
        y, s = y + residual, s + residual.abs()
    return y, s


def sconv1d(x, w, bias, stride: int = 1, dilation: int = 1, causal: bool = True, pre_elu: bool = False, residual=None):
    """EnCodec's SConv1d (reflect padding, `encodec_pads`) -> (y, s) as `conv1d`."""
    pl, pr = encodec_pads(x.shape[-1], w.shape[-1], stride, dilation, causal)
    return conv1d(x, w, bias, stride, dilation, pl, pr, True, pre_elu, residual)


def sconv_transpose1d(x: torch.Tensor, w: torch.Tensor, bias, stride: int, pre_elu: bool = False):
    """EnCodec's causal SConvTranspose1d with the padding K - stride trimmed on the right:
    y[b, co, j] = bias[co] + sum_{ci, q, k: q stride + k = j} w[ci, co, k] act(x)[b, ci, q], j < T stride."""
    B, Cin, T = x.shape
    _, Cout, K = w.shape
    a = elu(x) if pre_elu else x
    full = x.new_zeros((B, Cout, (T - 1) * stride + K))
    for k in range(K):
        full[..., k: k + (T - 1) * stride + 1: stride] += torch.einsum("ioc,bit->bot", w[:, :, k:k + 1], a)
    y = full[..., : full.shape[-1] - (K - stride)]
    return y + bias[None, :, None] if bias is not None else y


def pack_conv_transpose(w: torch.Tensor, stride: int) -> torch.Tensor:
    """the phase-channel packing of a K = 2 stride transposed-conv weight [Cin, C, K] as a stride-1 K = 2 conv weight
    [C stride, Cin, 2]: output sample q stride + r of channel c is phase channel c stride + r at time q; tap 0 reads
    x[q - 1] with w[:, c, r + stride], tap 1 reads x[q] with w[:, c, r]."""
    Cin, C, K = w.shape
    assert K == 2 * stride
    out = w.new_empty((C * stride, Cin, 2))
    for c in range(C):
        for r in range(stride):
            out[c * stride + r, :, 0] = w[:, c, r + stride]
            out[c * stride + r, :, 1] = w[:, c, r]
    return out


def conv_transpose_as_phases(x, w, bias, stride: int, pre_elu: bool = False):
    """the causal transposed conv computed the way the kernel does: a stride-1 K = 2 conv with one zero on the left,
    onto C stride phase channels, interleaved -> (y, s)."""
    return conv1d(x, pack_conv_transpose(w, stride), bias, 1, 1, 1, 0, False, pre_elu, None, phase=stride)


def lstm_layer(xproj: torch.Tensor, w_hh: torch.Tensor) -> torch.Tensor:
    """one LSTM layer from zero state: xproj [T, B, 4H] = W_ih x + b_ih + b_hh, w_hh [4H, H], gate order i, f, g, o;
    returns h [T, B, H] in the dtype of the inputs."""
    T, B, H4 = xproj.shape
    H = H4 // 4
    h = xproj.new_zeros((B, H))
    c = xproj.new_zeros((B, H))
    out = xproj.new_empty((T, B, H))
    for t in range(T):
        gates = xproj[t] + h @ w_hh.t()
        i, f, g, o = gates.split(H, dim=1)
        c = torch.sigmoid(f) * c + torch.sigmoid(i) * torch.tanh(g)
        h = torch.sigmoid(o) * torch.tanh(c)
        out[t] = h
    return out


def rvq_distances(r: torch.Tensor, cb: torch.Tensor) -> torch.Tensor:
    """-(|r|^2 - 2 r.e + |e|^2) for rows r [n, dim] and codes cb [n_codes, dim] -> [n, n_codes]"""
    return -(r.pow(2).sum(1, keepdim=True) - 2 * r @ cb.t() + cb.pow(2).sum(1)[None])


def rvq_encode(x: torch.Tensor, cbs: torch.Tensor, picks=None):
    """residual VQ of rows x [n, dim] over codebooks cbs [n_q, n_codes, dim]: per stage the first index of the largest
    `rvq_distances`, then r -= e_idx.  With `picks` [n, n_q] the residual of stage q is rebuilt from picks[:, :q]
    instead of the own choices (teacher forcing).  Returns (codes [n, n_q], margins [n, n_q]: best minus second-best
    distance, inf with one code, residuals [n_q, n, dim]: the residual each stage saw)."""
    n = x.shape[0]
    r = x.clone()
    codes, margins, res = [], [], []
    for q in range(cbs.shape[0]):
        d = rvq_distances(r, cbs[q])
        idx = d.argmax(1)
        if d.shape[1] > 1:
            top = d.topk(2, dim=1).values
            margins.append(top[:, 0] - top[:, 1])
        else:
            margins.append(torch.full((n,), math.inf, dtype=d.dtype, device=d.device))
        codes.append(idx)
        res.append(r)
        r = r - cbs[q][idx if picks is None else picks[:, q]]
    return torch.stack(codes, 1), torch.stack(margins, 1), torch.stack(res)
