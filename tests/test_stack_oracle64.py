"""The decoder-stack restatement of tests/stack_oracle64.py, checked without a GPU:
  * `layer_loop` over unrounded float64 ops is the model: `oracle.valle_oracle.encoder` (pre-LN, LayerNorm and AdaLN)
    and `tests/postln_oracle.encoder_postln` (post-LN), in all four mask modes over packed batches;
  * `ln_bound` and `gemm_bound` accept fp32 / bf16 emulations of `layernorm_kernel` and of the GEMMs' sums in
    several orders and block sizes;
  * the same bounds reject planted mistakes by at least REJECT times;
  * the NAR argmax rule: a CPU restatement of `better` / `warp_argmax` (csrc/sample.cu) before and after NaN became
    the maximum, against torch.argmax.
The worst ratios are printed (pytest -s)."""
import math
import os
import sys

import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

import attention_oracle64 as A  # noqa: E402
import stack_oracle64 as S  # noqa: E402
from oracle import valle_oracle as O  # noqa: E402
from postln_oracle import encoder_postln  # noqa: E402

REJECT = 4.0
PREFIX = "enc"
D, H, DFF, NL = 128, 2, 256, 2
LENS = [1, 63, 64, 65, 127, 128, 129]
SEG1 = 60


# ------------------------------------------------------------------------------------------------------ semantics
def _state(norm_first, adaptive, seed=5):
    """a float64 state dict in the oracle's layout (final norm for pre-LN only, as VALLE builds it), the stage
    embedding, the Layer list and the AdaLN table in NativeDecoder.ada_table order"""
    g = torch.Generator().manual_seed(seed)
    r = lambda *s: torch.randn(*s, generator=g, dtype=torch.float64)  # noqa: E731
    sd = {}

    def norm(p):
        if adaptive:
            sd[p + "project_layer.weight"] = r(2 * D, D) * 0.1
            sd[p + "project_layer.bias"] = torch.cat([1 + 0.1 * r(D), 0.1 * r(D)])
            p = p + "norm."
        sd[p + "weight"] = 1 + 0.2 * r(D)
        sd[p + "bias"] = 0.1 * r(D)

    for i in range(NL):
        p = f"{PREFIX}.layers.{i}."
        sd[p + "self_attn.in_proj_weight"] = r(3 * D, D) / math.sqrt(D)
        sd[p + "self_attn.in_proj_bias"] = 0.1 * r(3 * D)
        sd[p + "self_attn.out_proj.weight"] = r(D, D) / math.sqrt(D)
        sd[p + "self_attn.out_proj.bias"] = 0.1 * r(D)
        sd[p + "linear1.weight"] = r(DFF, D) / math.sqrt(D)
        sd[p + "linear1.bias"] = 0.1 * r(DFF)
        sd[p + "linear2.weight"] = r(D, DFF) / math.sqrt(DFF)
        sd[p + "linear2.bias"] = 0.1 * r(D)
        norm(p + "norm1.")
        norm(p + "norm2.")
    if norm_first:
        norm(PREFIX + ".norm.")
    emb = r(1, D) if adaptive else None
    inner = "norm." if adaptive else ""
    layers = []
    for i in range(NL):
        p = f"{PREFIX}.layers.{i}."
        layers.append(S.Layer(sd[p + "self_attn.in_proj_weight"], sd[p + "self_attn.in_proj_bias"],
                              sd[p + "self_attn.out_proj.weight"], sd[p + "self_attn.out_proj.bias"],
                              sd[p + "linear1.weight"], sd[p + "linear1.bias"], sd[p + "linear2.weight"],
                              sd[p + "linear2.bias"], sd[p + "norm1." + inner + "weight"], sd[p + "norm1." + inner + "bias"],
                              sd[p + "norm2." + inner + "weight"], sd[p + "norm2." + inner + "bias"]))
    ada = None
    if adaptive:
        names = [f"{PREFIX}.layers.{i}.norm{k}." for i in range(NL) for k in (1, 2)]
        if norm_first:
            names.append(PREFIX + ".norm.")
        ada = torch.stack([F.linear(emb, sd[n + "project_layer.weight"], sd[n + "project_layer.bias"])[0]
                           for n in names])
    return sd, emb, layers, ada


def _pack(mode):
    n = len(LENS)
    if mode == "full":
        return S.Pack(LENS, mode, [0] * n, [0] * n)
    if mode == "valle_ar":
        return S.Pack(LENS, mode, [min(L, s) for L, s in zip(LENS, [1, 47, 64, 1, 65, 128, 60])], [0] * n)
    # every sequence has text (S >= 1): a row that sees no key is NaN in the model (softmax over nothing), and its
    # NaN K / V rows reach the other rows of its sequence through P V (0 NaN = NaN)
    S_ = [min(L, SEG1, s) for L, s in zip(LENS, [1, 5, 60, 1, 33, 60, 17])]
    c1 = [max(0, min(L - SEG1, c)) for L, c in zip(LENS, [0, 3, 4, 5, 0, 68, 30])]
    return S.Pack(LENS, mode, S_, c1, SEG1)


@pytest.mark.parametrize("mode", A.MODES)
@pytest.mark.parametrize("variant", ["preln", "preln_adaln", "postln", "postln_adaln"])
def test_layer_loop_is_the_model(variant, mode):
    norm_first, adaptive = variant.startswith("preln"), variant.endswith("adaln")
    sd, emb, layers, ada = _state(norm_first, adaptive)
    pk = _pack(mode)
    x = torch.randn(pk.M, D, generator=torch.Generator().manual_seed(6), dtype=torch.float64)
    got = S.layer_loop(S.Float64Ops(), x, layers, pk, H, norm_first, ada)
    cfg = O.OracleConfig(D, H, NL)
    worst = 0.0
    for b, r0 in enumerate(pk.cu[:-1]):
        L = pk.lens[b]
        xb = x[r0:r0 + L][None]
        blocked = ~pk.vis(b)
        if norm_first:
            ref = O.encoder(sd, PREFIX, xb, cfg, blocked=blocked, stage_emb=emb)[0]
            # the loop has no final norm: put the oracle's on top of it
            if adaptive:
                mine = O.ada_layer_norm(got[r0:r0 + L], emb, sd[PREFIX + ".norm.project_layer.weight"],
                                        sd[PREFIX + ".norm.project_layer.bias"], sd[PREFIX + ".norm.norm.weight"],
                                        sd[PREFIX + ".norm.norm.bias"])
            else:
                mine = O.layer_norm(got[r0:r0 + L], sd[PREFIX + ".norm.weight"], sd[PREFIX + ".norm.bias"])
        else:
            ref = encoder_postln(sd, PREFIX, xb, cfg, blocked=blocked, stage_emb=emb)[0]
            mine = got[r0:r0 + L]
        assert torch.isfinite(ref).all()
        worst = max(worst, float((mine - ref).abs().max()))
    print(f"layer_loop {variant} {mode}: worst |difference| from the model {worst:.2e}")
    assert worst < 1e-10


def test_layer_loop_ada_rows():
    """norm k of layer l reads table row 2 l + k - 1: a table whose rows are tagged by their index shows which"""
    seen = []

    class Probe(S.Float64Ops):
        def norm(self, x, w, b, wb, operand):
            seen.append(int(wb[0]))
            return super().norm(x, w, b, None, operand)

    _, _, layers, _ = _state(True, False)
    tab = torch.arange(2 * NL + 1, dtype=torch.float64)[:, None].expand(-1, 2 * D).contiguous()
    pk = S.Pack([3], "full", [0], [0])
    x = torch.randn(3, D, dtype=torch.float64)
    for norm_first in (True, False):
        seen.clear()
        S.layer_loop(Probe(), x, layers, pk, H, norm_first, tab)
        assert seen == list(range(2 * NL)), (norm_first, seen)


# ------------------------------------------------------------------------------------------ layernorm emulation
def _ln_emulate(x, w, b, wb, out_dtype, eps=S.EPS, var_div=None, eps_on=True, swap_ada=False):
    """layernorm_kernel in fp32: each lane sums (x0 + x1) + (x2 + x3) of its float4s in order (element
    (i * 32 + lane) * 4 + j of the row), warp_sum's butterfly, two-pass moments, rsqrt, affine, AdaLN, the store.
    The keyword arguments plant mistakes."""
    R, d = x.shape
    kv = -(-d // 128)
    xp = torch.zeros(R, kv * 128)
    xp[:, :d] = x
    v = xp.view(R, kv, 32, 4)

    def lane_sum(t):
        s = torch.zeros(R, 32)
        for i in range(kv):
            s = s + ((t[:, i, :, 0] + t[:, i, :, 1]) + (t[:, i, :, 2] + t[:, i, :, 3]))
        for o in (16, 8, 4, 2, 1):
            s = s + s[:, torch.arange(32) ^ o]
        return s[:, :1]

    mean = lane_sum(v) / torch.tensor(float(d))
    a = v - mean[:, :, None, None]
    valid = (torch.arange(kv * 128) < d).view(1, kv, 32, 4)
    a = torch.where(valid, a, torch.zeros(()))
    q = lane_sum(a * a)
    var = q / torch.tensor(float(var_div or d))
    r = torch.rsqrt(var + eps) if eps_on else torch.rsqrt(var)
    y = (a.reshape(R, -1)[:, :d] * r) * w + b
    if wb is not None:
        ww, bb = wb[:d], wb[d:]
        if swap_ada:
            ww, bb = bb, ww
        y = ww * y + bb
    return y.to(out_dtype)


def _ln_rows(d, rho, R=48, seed=0):
    """R fp32 rows of width d: scale 10^U(-2, 1), offset rho * scale; the last two rows constant"""
    g = torch.Generator().manual_seed(seed + d)
    sc = 10.0 ** (torch.rand(R, 1, generator=g) * 3 - 2)
    x = (torch.randn(R, d, generator=g) + rho * torch.sign(torch.randn(R, 1, generator=g))) * sc
    x[-2:] = torch.randn(2, 1, generator=g) * 3
    return x.float()


def _ln_params(d, seed=1):
    g = torch.Generator().manual_seed(seed)
    w = (1 + 0.2 * torch.randn(d, generator=g)).float()
    b = (0.1 * torch.randn(d, generator=g)).float()
    wb = torch.cat([1 + 0.1 * torch.randn(d, generator=g), 0.1 * torch.randn(d, generator=g)]).float()
    wb2 = torch.cat([1 + 0.1 * torch.randn(d, generator=g), 0.1 * torch.randn(d, generator=g)]).float()
    return w, b, wb, wb2


LN_DIMS = (4, 128, 132, 260, 1024, 2044)


def test_ln_bound_accepts_the_kernel_arithmetic():
    worst = {}
    for d in LN_DIMS:
        w, b, wb, _ = _ln_params(d)
        for rho in (0, 16, 256, 4096):
            x = _ln_rows(d, rho)
            for ada in (None, wb):
                for dt in (torch.float32, torch.bfloat16):
                    out = _ln_emulate(x, w, b, ada, dt)
                    y, bnd = S.ln_bound(x, w, b, ada, out)
                    r = S.ratio(out, y, bnd)
                    key = str(dt).split(".")[-1]
                    worst[key] = max(worst.get(key, 0.0), r)
                    assert r <= 1.0, (d, rho, ada is not None, dt, r)
    print(f"ln_bound: worst emulation error / bound {worst}")


def test_ln_bound_rejects_planted_mistakes():
    """each mistake at d = 1024 and d = 132, rows of offset 0 and 16, fp32 out (a bf16 out's rounding is 2^-9 of the
    value, larger than the smaller of these mistakes)"""
    found = {}
    for d in (132, 1024):
        w, b, wb, wb2 = _ln_params(d)
        for rho in (0, 16):
            x = _ln_rows(d, rho)
            planted = {
                "variance over d - 1": dict(out=_ln_emulate(x, w, b, wb, torch.float32, var_div=d - 1), wb=wb),
                "eps missing": dict(out=_ln_emulate(x, w, b, wb, torch.float32, eps_on=False), wb=wb),
                "AdaLN weight and bias swapped": dict(out=_ln_emulate(x, w, b, wb, torch.float32, swap_ada=True), wb=wb),
                "the next layer's AdaLN row": dict(out=_ln_emulate(x, w, b, wb2, torch.float32), wb=wb),
            }
            for name, c in planted.items():
                y, bnd = S.ln_bound(x, w, b, c["wb"], c["out"])
                r = S.ratio(c["out"], y, bnd)
                found[name] = min(found.get(name, math.inf), r)
    print("ln_bound rejection factors: " + ", ".join(f"{k} {v:.3g}" for k, v in found.items()))
    for k, v in found.items():
        assert v >= REJECT, (k, v)


# ------------------------------------------------------------------------------------------------ gemm emulation
def _gemm_inputs(M, N, K, seed=3, dtype=torch.bfloat16):
    g = torch.Generator().manual_seed(seed + K)
    a = torch.randn(M, K, generator=g).to(dtype)
    W = (torch.randn(N, K, generator=g) / math.sqrt(K)).to(dtype)
    b = (0.1 * torch.randn(N, generator=g)).float()
    res = torch.randn(M, N, generator=g).float()
    return a, W, b, res


def _acc(a, W, order, block=64):
    """fp32 a W^T in one of several orders: 'torch' (torch's fp32 matmul), 'chain' (one running sum in k order),
    'blocks' (fp32 sums of `block`-wide k-blocks, each a chain, added in order), 'pairwise' (a pairwise tree over k)"""
    af, Wf = a.float(), W.float()
    if order == "torch":
        return af @ Wf.t()
    K = a.shape[1]
    if order == "chain":
        acc = torch.zeros(a.shape[0], W.shape[0])
        for k in range(K):
            acc = acc + af[:, k:k + 1] * Wf[:, k][None]
        return acc
    if order == "blocks":
        acc = torch.zeros(a.shape[0], W.shape[0])
        for k0 in range(0, K, block):
            part = torch.zeros_like(acc)
            for k in range(k0, min(K, k0 + block)):
                part = part + af[:, k:k + 1] * Wf[:, k][None]
            acc = acc + part
        return acc
    terms = af[:, None, :] * Wf[None, :, :]           # exact products (bf16 x bf16 fit fp32)
    while terms.shape[-1] > 1:
        if terms.shape[-1] % 2:
            terms = torch.cat([terms, torch.zeros_like(terms[..., :1])], -1)
        terms = terms[..., 0::2] + terms[..., 1::2]
    return terms[..., 0]


def _epilogue(acc, b, epi, res, out_dtype):
    v = acc + b if b is not None else acc
    if epi == S.EPI_RELU:
        v = torch.relu(v)
    if epi == S.EPI_RESIDUAL:
        v = res + v
    return v.to(out_dtype)


def test_gemm_bound_accepts_fp32_sums():
    worst = {}
    for K in (64, 1024, 4096):
        M, N = (32, 64) if K == 4096 else (48, 128)
        a, W, b, res = _gemm_inputs(M, N, K)
        for order in ("torch", "chain", "blocks", "pairwise"):
            for block in ((16, 64) if order == "blocks" else (64,)):
                acc = _acc(a, W, order, block)
                for epi, dt in ((S.EPI_NONE, torch.bfloat16), (S.EPI_RELU, torch.bfloat16),
                                (S.EPI_RESIDUAL, torch.float32), (S.EPI_NONE, torch.float32)):
                    bias = None if (epi == S.EPI_NONE and dt == torch.float32) else b   # the NAR head: no bias
                    out = _epilogue(acc, bias, epi, res if epi == S.EPI_RESIDUAL else None, dt)
                    for kind in ("wgmma", "simt"):
                        z, bnd = S.gemm_bound(a, W, bias, epi, res if epi == S.EPI_RESIDUAL else None, out, kind)
                        r = S.ratio(out, z, bnd)
                        key = f"{kind} {['none', 'relu', 'residual'][epi]} {str(dt).split('.')[-1]}"
                        worst[key] = max(worst.get(key, 0.0), r)
                        assert r <= 1.0, (K, order, block, epi, dt, kind, r)
    # the fp32 CUDA-core path: fp32 operands, fmaf chains (and torch's order)
    for K in (256, 1024):
        a, W, b, res = _gemm_inputs(40, 64, K, dtype=torch.float32)
        for order in ("torch", "chain"):
            acc = _acc(a, W, order)
            for epi in (S.EPI_NONE, S.EPI_RELU, S.EPI_RESIDUAL):
                out = _epilogue(acc, b, epi, res if epi == S.EPI_RESIDUAL else None, torch.float32)
                z, bnd = S.gemm_bound(a, W, b, epi, res if epi == S.EPI_RESIDUAL else None, out, "simt")
                r = S.ratio(out, z, bnd)
                worst["simt fp32 operands"] = max(worst.get("simt fp32 operands", 0.0), r)
                assert r <= 1.0, (K, order, epi, r)
    print("gemm_bound: worst emulation error / bound " + ", ".join(f"{k} {v:.3g}" for k, v in worst.items()))


def test_gemm_bound_rejects_planted_mistakes():
    """the wgmma bound (the looser of the two) against: one 64-wide k-block dropped at K = 1024 and K = 4096, the
    bias shifted by one column, the rows of one 64-row half-tile taken from the neighbouring half-tile, the residual
    taken from the wrong row"""
    found = {}
    for K in (1024, 4096):
        M, N = 128, 256
        a, W, b, res = _gemm_inputs(M, N, K, seed=9)
        acc = a.float() @ W.float().t()
        a_drop = a.clone()
        a_drop[:, K - 64:] = 0
        drop = a_drop.float() @ W.float().t()
        b_shift = torch.roll(b, 1)
        acc_half = acc.clone()
        acc_half[64:128] = acc[0:64]
        res_row = torch.roll(res, 1, 0)
        planted = {
            f"k-block dropped (K={K})": (_epilogue(drop, b, S.EPI_RESIDUAL, res, torch.float32), S.EPI_RESIDUAL),
            f"k-block dropped, bf16 out (K={K})": (_epilogue(drop, b, S.EPI_NONE, None, torch.bfloat16), S.EPI_NONE),
            f"bias shifted one column (K={K})": (_epilogue(acc, b_shift, S.EPI_RELU, None, torch.bfloat16), S.EPI_RELU),
            f"half-tile rows from the next half-tile (K={K})": (_epilogue(acc_half, b, S.EPI_NONE, None, torch.bfloat16),
                                                                 S.EPI_NONE),
            f"residual from the wrong row (K={K})": (_epilogue(acc, b, S.EPI_RESIDUAL, res_row, torch.float32),
                                                     S.EPI_RESIDUAL),
        }
        for name, (out, epi) in planted.items():
            z, bnd = S.gemm_bound(a, W, b, epi, res if epi == S.EPI_RESIDUAL else None, out, "wgmma")
            found[name] = S.ratio(out, z, bnd)
    print("gemm_bound rejection factors: " + ", ".join(f"{k} {v:.3g}" for k, v in found.items()))
    for k, v in found.items():
        assert v >= REJECT, (k, v)


def test_adaln_bound_accepts_fp32_chains():
    g = torch.Generator().manual_seed(4)
    for d in (256, 1024):
        W = (torch.randn(2 * d, d, generator=g) * 0.05).float()
        bias = torch.randn(2 * d, generator=g).float()
        e = torch.randn(d, generator=g).float()
        acc = torch.zeros(2 * d, 32)
        for c0 in range(0, d, 128):         # lane l: columns c0 + 4 l .. + 3, one fma chain
            blk = (W[:, c0:c0 + 128] * e[c0:c0 + 128]).view(2 * d, 32, 4)
            acc = acc + blk[..., 0] + blk[..., 1] + blk[..., 2] + blk[..., 3]
        out = acc.sum(-1) + bias
        z, bnd = S.adaln_bound(W, bias, e, out)
        assert S.ratio(out, z, bnd) <= 1.0


# --------------------------------------------------------------------------------------------------- NAR argmax
INT_MAX = 0x7fffffff


def _better_old(a, b):
    return b if (b[0] > a[0] or (b[0] == a[0] and b[1] < a[1])) else a


def _better_new(a, b):
    an, bn = math.isnan(a[0]), math.isnan(b[0])
    if an or bn:
        return b if (bn and (not an or b[1] < a[1])) else a
    return _better_old(a, b)


def _warp_argmax(row, better):
    """nar_argmax_accumulate_kernel: lane l scans i = l, l + 32, ..., then the shfl_xor butterfly"""
    lanes = [(-math.inf, INT_MAX)] * 32
    for i, v in enumerate(row):
        lanes[i % 32] = better(lanes[i % 32], (v, i))
    for o in (16, 8, 4, 2, 1):
        lanes = [better(lanes[l], lanes[l ^ o]) for l in range(32)]
    assert all(x[1] == lanes[0][1] for x in lanes)
    return lanes[0][1]


def test_nar_argmax_nan_rule():
    nan = float("nan")
    g = torch.Generator().manual_seed(8)
    rows = [[nan] * 1024, [nan] * 7]
    r = torch.randn(1024, generator=g).tolist()
    r[517] = nan
    rows.append(r)
    r = torch.randn(1024, generator=g).tolist()
    r[900], r[33], r[2] = nan, nan, 50.0
    rows.append(r)
    # the old rule: an all-NaN row keeps the initial index (the kernel then read next_emb + 0x7fffffff d), a one-NaN
    # row returns the largest number's index where torch.argmax returns the NaN's
    assert _warp_argmax(rows[0], _better_old) == INT_MAX
    assert _warp_argmax(rows[2], _better_old) != int(torch.argmax(torch.tensor(rows[2])))
    for v in (1, 5, 31, 32, 33, 1024, 1025):
        x = torch.randn(v, generator=g)
        x[torch.randint(0, v, (1,), generator=g)] = x.max()            # a planted exact tie: the first index wins
        rows.append(x.tolist())
        rows.append([-math.inf] * v)
        y = x.clone()
        y[torch.randint(0, v, (2,), generator=g)] = nan
        rows.append(y.tolist())
        rows.append(([math.inf] + x.tolist())[:v])
    for row in rows:
        want = int(torch.argmax(torch.tensor(row)))
        assert _warp_argmax(row, _better_new) == want, row[:8]
        if not any(math.isnan(v) for v in row):
            assert _warp_argmax(row, _better_old) == want
