"""The decoder-stack backward restatement of tests/stack_oracle64.py and its bounds, checked without a GPU:
  * `backward_loop` over unrounded float64 ops is torch.autograd of `layer_loop` over the same ops, to about 1e-12:
    pre-LN and post-LN, LayerNorm and AdaLN, the four mask modes, and dropout with the documented hash masks;
  * `attention_oracle64.bwd_bound`, `ln_bwd_bound` / `ln_param_bounds`, `colsum_bound` and `ce_bwd_bound` accept
    fp32 / bf16 emulations of `attn_bwd_dq_kernel` / `attn_bwd_dkv_kernel`, `ln_bwd_kernel`, `colsum_kernel` and
    `ce_bwd_kernel`;
  * the same bounds reject planted mistakes by at least REJECT times.
The worst ratios and the rejection factors are printed (pytest -s)."""
import math
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

import attention_oracle64 as A  # noqa: E402
import stack_oracle64 as S  # noqa: E402
from test_stack_oracle64 import D, H, NL, _pack, _state  # noqa: E402

REJECT = 20.0


# ------------------------------------------------------------------------------------------------------ semantics
def _autograd_and_loop(norm_first, adaptive, mode, drop=None):
    _, _, layers, ada = _state(norm_first, adaptive)
    pk = _pack(mode)
    g = torch.Generator().manual_seed(8)
    x = torch.randn(pk.M, D, generator=g, dtype=torch.float64).requires_grad_()
    gout = torch.randn(pk.M, D, generator=g, dtype=torch.float64)
    leaves = [S.Layer(*[t.clone().requires_grad_() for t in vars(P).values()]) for P in layers]
    ada_l = ada.clone().requires_grad_() if ada is not None else None
    recs = {}
    out = S.layer_loop(S.Float64Ops(), x, leaves, pk, H, norm_first, ada_l, lambda l, r: recs.__setitem__(l, r), drop)
    (out * gout).sum().backward()
    saves = [{k: v.detach() for k, v in S.saves_of(recs[l]).items()} for l in range(NL)]
    grads = [{k: torch.zeros_like(getattr(P, k)) for k in S.GRAD_NAMES} for P in layers]
    dada = torch.zeros_like(ada) if ada is not None else None
    dx = S.backward_loop(S.Float64Ops(), saves, gout, layers, pk, H, norm_first, grads, ada, dada, drop)
    pairs = [("x", dx, x.grad)]
    for l, P in enumerate(leaves):
        pairs += [(f"layer {l} {k}", grads[l][k], getattr(P, k).grad) for k in S.GRAD_NAMES]
    if ada is not None:
        pairs.append(("ada", dada, ada_l.grad))
    return pairs


def _rel(a, b):
    return float((a - b).abs().max() / b.abs().max().clamp(min=1e-300))


@pytest.mark.parametrize("mode", A.MODES)
@pytest.mark.parametrize("variant", ["preln", "preln_adaln", "postln", "postln_adaln"])
def test_backward_loop_is_autograd(variant, mode):
    pairs = _autograd_and_loop(variant.startswith("preln"), variant.endswith("adaln"), mode)
    worst = max(_rel(a, b) for _, a, b in pairs)
    print(f"backward_loop {variant} {mode}: worst relative difference from autograd {worst:.2e}")
    for name, a, b in pairs:
        assert _rel(a, b) < 1e-11, (name, _rel(a, b))


@pytest.mark.parametrize("variant", ["preln", "postln_adaln"])
def test_backward_loop_with_dropout_is_autograd(variant):
    """p = 0.1 with the hash masks of keep_mask at all four sites; the loop's gradient differs from the p = 0 one"""
    drop = (0.1, 987654321)
    pairs = _autograd_and_loop(variant == "preln", variant.endswith("adaln"), "padded_ar", drop)
    for name, a, b in pairs:
        assert _rel(a, b) < 1e-11, (name, _rel(a, b))
    plain = _autograd_and_loop(variant == "preln", variant.endswith("adaln"), "padded_ar")
    assert _rel(pairs[0][1], plain[0][1]) > 1e-2


def test_keep_mask_rate_and_streams():
    m = S.keep_mask(12345, 7, 1 << 18, 0.1)
    assert abs(float(m.float().mean()) - 0.9) < 5e-3
    assert not torch.equal(m, S.keep_mask(12345, 8, 1 << 18, 0.1))
    idx = torch.arange(5, 1 << 18, 97).numpy()
    assert torch.equal(S.keep_mask(12345, 7, len(idx), 0.1, idx), m[5::97])


# -------------------------------------------------------------------------------------------- attention backward
def _attn_case(L, mode, S_, c1, seg1, st, hh=2, seed=0, drop=False):
    """q, k, v, stored O, dO [hh, L, 64] in the storage dtype st, vis and the dropout scale (or None)"""
    g = torch.Generator().manual_seed(seed + L)
    q, k, v = ((torch.randn(hh, L, A.HD, generator=g) * 0.7).to(st) for _ in range(3))
    vis = A.visible(mode, L, S_, c1, seg1)
    w = None
    if drop:
        w = (torch.rand(hh, L, L, generator=g) >= 0.1).double() * S.inv_keep(0.1)
    P = S.softmax_rows64(q, k, vis)
    O = ((P if w is None else P * w) @ v.double()).to(st)
    dO = (torch.randn(hh, L, A.HD, generator=g) * 0.3).to(st)
    return q, k, v, O, dO, vis, w


ATTN_CASES = [(1, "full", 0, 0, 0), (63, "valle_ar", 10, 0, 0), (65, "full", 0, 0, 0),
              (200, "valle_ar", 47, 0, 0), (193, "padded_ar", 30, 100, 60), (150, "padded", 17, 70, 60),
              (129, "padded_ar", 60, 69, 60)]


def _attn_ratio(case, got):
    q, k, v, O, dO, vis, w = case
    exact, bnds = A.bwd_bound(q, k, v, O, dO, vis, w)
    out = []
    for z, b, t in zip(exact, bnds, got):
        if t.dtype == torch.bfloat16:
            b = b + S.half_ulp(t)
        out.append(S.ratio(t, z, b))
    return out


def test_attn_bwd_bound_accepts_the_kernel_arithmetic():
    worst = {}
    for st in (torch.float32, torch.bfloat16):
        for drop in (False, True):
            for L, mode, S_, c1, seg1 in ATTN_CASES:
                case = _attn_case(L, mode, S_, c1, seg1, st, drop=drop)
                got = A.emulate_bwd(*case, out_dtype=st)
                for name, r in zip(("dq", "dk", "dv"), _attn_ratio(case, got)):
                    key = f"{name} {str(st).split('.')[-1]}"
                    worst[key] = max(worst.get(key, 0.0), r)
                    assert r <= 1.0, (st, drop, L, mode, name, r)
    print("attention backward bound: worst emulation error / bound " +
          ", ".join(f"{k} {v:.3g}" for k, v in worst.items()))


def test_attn_bwd_bound_rejects_planted_mistakes():
    """fp32 storage: dK / dV skipping the last partial query tile and dQ skipping the last key tile (L = 200, causal:
    the last keys are seen by the last rows only), D over 48 of the 64 head dims, and the dropout scale applied to P
    but not to dP"""
    found = {}
    st = torch.float32
    c = _attn_case(200, "valle_ar", 47, 0, 0, st)
    found["dK / dV skip the last partial query tile"] = max(_attn_ratio(c, A.emulate_bwd(*c, skip_last_q_tile=True))[1:])
    found["dQ skips the last key tile"] = _attn_ratio(c, A.emulate_bwd(*c, skip_last_k_tile=True))[0]
    c = _attn_case(193, "padded_ar", 30, 100, 60, st)
    found["D over 48 head dims"] = max(_attn_ratio(c, A.emulate_bwd(*c, d_dims=48)))
    c = _attn_case(150, "full", 0, 0, 0, st, drop=True)
    found["dropout mask on P but not on dP"] = max(_attn_ratio(c, A.emulate_bwd(*c, drop_dp=False)))
    print("attention backward rejection factors: " + ", ".join(f"{k} {v:.3g}" for k, v in found.items()))
    for k, v in found.items():
        assert v >= REJECT, (k, v)


# -------------------------------------------------------------------------------------------- LayerNorm backward
def _lane_sum(t):
    """ln_bwd_kernel / ce_bwd_kernel row sums in fp32: lane j adds elements j, j + 32, ... in order, then warp_sum"""
    R, d = t.shape
    n = -(-d // 32)
    v = torch.zeros(R, n * 32)
    v[:, :d] = t
    v = v.view(R, n, 32)
    s = torch.zeros(R, 32)
    for i in range(n):
        s = s + v[:, i]
    for o in (16, 8, 4, 2, 1):
        s = s + s[:, torch.arange(32) ^ o]
    return s[:, :1]


def _ln_bwd_emulate(x, w, b, wb, dy, prior, no_m2=False, no_aw_in_dgamma=False):
    """ln_bwd_kernel in fp32: moments recomputed, the two means, dx = prior + rstd (g - m1 - xhat m2), and the
    parameter sums (in torch's order).  The keyword arguments plant mistakes."""
    d = x.shape[1]
    fd = torch.tensor(float(d))
    mu = _lane_sum(x) / fd
    t = x - mu
    rstd = torch.rsqrt(_lane_sum(t * t) / fd + S.EPS)
    xh = t * rstd
    aw = wb[:d] if wb is not None else torch.ones(d)
    g = dy * aw * w
    m1 = _lane_sum(g) / fd
    m2 = _lane_sum(g * xh) / fd
    dx = prior + rstd * (g - m1 - (0 if no_m2 else xh * m2))
    pg = {"dgamma": ((dy if no_aw_in_dgamma else dy * aw) * xh).sum(0), "dbeta": (dy * aw).sum(0)}
    if wb is not None:
        pg["dada"] = torch.cat([(dy * (w * xh + b)).sum(0), dy.sum(0)])
    return dx, pg


def _ln_bwd_inputs(d, rho, seed=0, R=64):
    g = torch.Generator().manual_seed(seed + d + int(rho))
    sc = 10.0 ** (torch.rand(R, 1, generator=g) * 3 - 2)
    x = ((torch.randn(R, d, generator=g) + rho * torch.sign(torch.randn(R, 1, generator=g))) * sc).float()
    w = (1 + 0.2 * torch.randn(d, generator=g)).float()
    b = (0.1 * torch.randn(d, generator=g)).float()
    wb = torch.cat([1 + 0.1 * torch.randn(d, generator=g), 0.1 * torch.randn(d, generator=g)]).float()
    dy = torch.randn(R, d, generator=g).float()
    prior = (0.5 * torch.randn(R, d, generator=g)).float()
    return x, w, b, wb, dy, prior


def _ln_ratios(x, w, b, wb, dy, prior, dx, pg):
    z, bnd = S.ln_bwd_bound(x, w, b, wb, dy, prior)
    out = {"dx": S.ratio(dx, z, bnd)}
    for k, (z, bnd) in S.ln_param_bounds(x, w, b, wb, dy).items():
        out[k] = S.ratio(pg[k], z, bnd)
    return out


def test_ln_bwd_bound_accepts_the_kernel_arithmetic():
    worst = {}
    for d in (128, 256, 1024, 4096):
        for rho in (0, 16, 4096):
            x, w, b, wb, dy, prior = _ln_bwd_inputs(d, rho)
            for ada in (None, wb):
                dx, pg = _ln_bwd_emulate(x, w, b, ada, dy, prior)
                for k, r in _ln_ratios(x, w, b, ada, dy, prior, dx, pg).items():
                    worst[k] = max(worst.get(k, 0.0), r)
                    assert r <= 1.0, (d, rho, ada is not None, k, r)
    print("LayerNorm backward bounds: worst emulation error / bound " +
          ", ".join(f"{k} {v:.3g}" for k, v in worst.items()))


def test_ln_bwd_bound_rejects_planted_mistakes():
    found = {}
    for d in (256, 1024):
        for rho in (0, 16):
            x, w, b, wb, dy, prior = _ln_bwd_inputs(d, rho)
            dx, pg = _ln_bwd_emulate(x, w, b, wb, dy, prior, no_m2=True)
            r = _ln_ratios(x, w, b, wb, dy, prior, dx, pg)["dx"]
            found["dx without xhat mean(g xhat)"] = min(found.get("dx without xhat mean(g xhat)", math.inf), r)
            dx, pg = _ln_bwd_emulate(x, w, b, wb, dy, prior, no_aw_in_dgamma=True)
            r = _ln_ratios(x, w, b, wb, dy, prior, dx, pg)["dgamma"]
            found["dgamma without the AdaLN weight"] = min(found.get("dgamma without the AdaLN weight", math.inf), r)
    print("LayerNorm backward rejection factors: " + ", ".join(f"{k} {v:.3g}" for k, v in found.items()))
    for k, v in found.items():
        assert v >= REJECT, (k, v)


# ------------------------------------------------------------------------------------------------- bias colsum
def _colsum_emulate(dy, prior, drop_last_block=False):
    """colsum_kernel: 256-row blocks, each 8 strided per-thread chains then their sum; the blocks added in order"""
    R = dy.shape[0]
    out = prior.clone()
    blocks = list(range(0, R, 256))
    if drop_last_block:
        blocks = blocks[:-1]
    for r0 in blocks:
        blk = dy[r0:r0 + 256].float()
        part = torch.zeros(8, dy.shape[1])
        for i in range(0, blk.shape[0], 8):
            part = part + torch.nn.functional.pad(blk[i:i + 8], (0, 0, 0, 8 - blk[i:i + 8].shape[0]))
        t = torch.zeros(dy.shape[1])
        for i in range(8):
            t = t + part[i]
        out = out + t
    return out


def test_colsum_bound_accepts_and_rejects():
    g = torch.Generator().manual_seed(3)
    worst, found = 0.0, math.inf
    for R in (1, 63, 65, 1000, 3001):
        for st in (torch.float32, torch.bfloat16):
            dy = torch.randn(R, 96, generator=g).to(st)
            prior = torch.randn(96, generator=g)
            z, bnd = S.colsum_bound(dy, prior)
            worst = max(worst, S.ratio(_colsum_emulate(dy, prior), z, bnd))
            if R > 256:
                found = min(found, S.ratio(_colsum_emulate(dy, prior, drop_last_block=True), z, bnd))
    print(f"colsum bound: worst emulation error / bound {worst:.3g}; a dropped last row block rejected by {found:.3g}")
    assert worst <= 1.0 and found >= REJECT


# ------------------------------------------------------------------------------------------------ cross-entropy
def _ce_emulate(logits, targets, V, ignore, grad_rows, scale, n_out, out_dtype, onehot_shift=0):
    """ce_bwd_kernel and cross_entropy_kernel in fp32 (lane sums as _lane_sum); onehot_shift plants a mistake"""
    x = logits[:, :V]
    mx = x.amax(-1, keepdim=True)
    e = torch.exp(x - mx)
    s = _lane_sum(e)
    skip = (targets == ignore) | (targets < 0) | (targets >= V)
    t = targets.clamp(0, V - 1)
    loss = torch.log(s)[:, 0] + mx[:, 0] - x.gather(1, t[:, None])[:, 0]
    loss = torch.where(skip, torch.zeros_like(loss), loss)
    g = torch.full((x.shape[0],), scale) * (grad_rows if grad_rows is not None else 1.0)
    g = torch.where(skip, torch.zeros_like(g), g)[:, None]
    oh = torch.zeros_like(x)
    oh.scatter_(1, ((t + onehot_shift) % V)[:, None], 1.0)
    dl = torch.zeros(x.shape[0], n_out)
    dl[:, :V] = g * (e * (1.0 / s) - oh)
    return loss, dl.to(out_dtype)


def _ce_inputs(V, R=96, spread=80.0, seed=4):
    g = torch.Generator().manual_seed(seed + V)
    logits = (torch.rand(R, V, generator=g) * 2 - 1) * spread
    logits[: R // 2] = torch.randn(R // 2, V, generator=g) * 2
    targets = torch.randint(0, V, (R,), generator=g)
    targets[::7] = -100
    grad_rows = torch.rand(R, generator=g) + 0.5
    return logits.float(), targets, grad_rows.float()


def test_ce_bounds_accept_and_reject():
    worst, found = {}, math.inf
    for V, n_out in ((1025, 1088), (1024, 1024)):
        logits, targets, grad_rows = _ce_inputs(V)
        for st in (torch.float32, torch.bfloat16):
            loss, dl = _ce_emulate(logits, targets, V, -100, grad_rows, 0.5, n_out, st)
            z, bnd = S.ce_bound(logits, targets, V, -100)
            worst["loss"] = max(worst.get("loss", 0.0), S.ratio(loss, z, bnd))
            z, bnd = S.ce_bwd_bound(logits, targets, V, -100, grad_rows, 0.5, n_out, dl)
            key = f"dlogits {str(st).split('.')[-1]}"
            worst[key] = max(worst.get(key, 0.0), S.ratio(dl, z, bnd))
        _, dl = _ce_emulate(logits, targets, V, -100, grad_rows, 0.5, n_out, torch.float32, onehot_shift=-1)
        z, bnd = S.ce_bwd_bound(logits, targets, V, -100, grad_rows, 0.5, n_out, dl)
        found = min(found, S.ratio(dl, z, bnd))
    print("cross-entropy bounds: worst emulation error / bound " + ", ".join(f"{k} {v:.3g}" for k, v in worst.items())
          + f"; onehot at target - 1 rejected by {found:.3g}")
    assert max(worst.values()) <= 1.0 and found >= REJECT
