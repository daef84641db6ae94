"""The decoder-stack backward `vb_decoder_backward` and the training loss head against tests/stack_oracle64.py, at the
trainer's shapes (d = 1024, 16 heads, d_ff = 4096; AR training in bf16 on a padded batch of about 80 s, NAR training
in fp32 with AdaLN on about 40 s).

For each stack case (CASES) the layers come from valle_b200.modules.transformer with seeded random weights, and the
library runs vb_decoder_forward_train, then vb_decoder_backward with its workspace filled with NaN (as
autograd.DecoderStack does, without dropout).  Then:
  * composition: `backward_loop` over the library's public ops (vb_linear_backward, vb_attention_backward,
    vb_layernorm_backward, vb_cast_from_f32), fed the forward values from the library's save buffer, reproduces the
    input gradient and every weight gradient bit for bit; the atomically reduced vectors (biases, LayerNorm and AdaLN
    gradients) agree within twice their reordering bound;
  * numerics: in the layers CHECKED_LAYERS each op of that run -- the dgrad and wgrad GEMMs, the bias sums, the ReLU
    mask, the attention backward, the LayerNorm backward and its parameter sums, the casts -- is within its derived
    bound of its float64 value computed from the inputs it received;
  * whole stack (AR case and the dropout case, report only): the per-layer input gradient against backward_loop over
    float64 ops with the library's rounding points, fed the same saved forward values.
The edges get their own tests: packed sweeps of the attention backward in all four mask modes with NaN planted around
each sequence and masked keys that must get exactly no gradient; vb_linear_backward at M = 1, 63, 65 with NaN in its
workspace and accumulate semantics; vb_layernorm_backward's strided gather, dx_copy, 4096 sigma offsets and d = 4096;
the loss head (vb_cross_entropy and its backward at V = 1025 / 1024, vb_embed_backward over 8 tables,
vb_rowdot_accumulate, vb_adaln_project_backward).
The worst error / bound per op and case goes to stack_backward.json in $VB_REPORT_DIR (default: the system temporary
directory)."""
import ctypes as C
import json
import math
import os
import sys
import tempfile
from dataclasses import dataclass

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

import attention_oracle64 as A  # noqa: E402
import stack_oracle64 as S  # noqa: E402
from test_stack_oracle64_gpu import _bits, _mode, _model, _packed_tensors  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
REPORT = {}
NAN_BYTE = 0xFF          # a buffer of 0xFF bytes is NaN in fp32 and bf16


def _s():
    return torch.cuda.current_stream().cuda_stream


def _lib():
    from valle_b200 import _lib as L
    return L, L.load()


def _dt(dtype):
    L, _ = _lib()
    return L.VB_BF16 if dtype == torch.bfloat16 else L.VB_F32


def _nan_ws(nbytes):
    return torch.full((nbytes,), NAN_BYTE, dtype=torch.uint8, device=DEV)


# ---- the library's public backward ops ----------------------------------------------------------------------------
class LibOps:
    """backward_loop's ops through the C ABI, every workspace filled with NaN first.  relu_backward has no entry of
    its own: the mask is restated elementwise (where(h > 0, dh, 0), exact)."""

    def __init__(self, dtype):
        self.dtype = dtype

    def cast(self, x):
        from valle_b200 import ops
        return ops.cast_from_f32(x.contiguous(), self.dtype)

    def linear_backward(self, a, W, dy, epi, dst, dW, db):
        L, lib = _lib()
        M, K = a.shape
        N = W.shape[0]
        dt = _dt(a.dtype)
        Wt = W.t().contiguous()
        if dst is None:
            dX = torch.empty(M, K, dtype=self.dtype, device=DEV)
        elif epi == S.EPI_RESIDUAL:
            dX = dst.clone()
        else:
            dX = torch.empty(M, K, dtype=torch.float32, device=DEV)
        nb = lib.vb_linear_backward_workspace(dt, M, N, K)
        ws = _nan_ws(nb)
        L.check(lib.vb_linear_backward(a.data_ptr(), dt, a.stride(0), Wt.data_ptr(), dy.data_ptr(), dy.stride(0),
                                       dX.data_ptr(), _dt(dX.dtype), dX.stride(0), epi, L.ptr(dW), L.ptr(db), M, N, K,
                                       ws.data_ptr(), nb, _s()), "vb_linear_backward")
        return dX

    def relu_backward(self, dh, hb, scale):
        assert scale == 1.0
        return torch.where(hb > 0, dh, torch.zeros((), dtype=dh.dtype, device=DEV))

    def attention_backward(self, qkv, o, dO, pk, n_head, l):
        return attention_backward(qkv, o, dO, pk, n_head)

    def norm_backward(self, x, w, b, wb, dout, dst, dg, dbeta, dwb):
        """as vb_decoder_backward calls it: dx into dst (zeros for None) and a dx_copy in the storage dtype, which
        must be bf16(dx) / dx bit for bit"""
        L, lib = _lib()
        M, d = x.shape
        out = torch.zeros(M, d, device=DEV) if dst is None else dst.clone()
        copy = torch.empty(M, d, dtype=self.dtype, device=DEV)
        L.check(lib.vb_layernorm_backward(x.data_ptr(), x.stride(0), 0, M, d, w.data_ptr(), b.data_ptr(), L.ptr(wb),
                                          S.EPS, dout.data_ptr(), dout.stride(0), out.data_ptr(), d, copy.data_ptr(),
                                          _dt(self.dtype), dg.data_ptr(), dbeta.data_ptr(), L.ptr(dwb), _s()),
                "vb_layernorm_backward")
        assert torch.equal(_bits(copy), _bits(out.to(self.dtype))), "vb_layernorm_backward: dx_copy is not dx rounded"
        return out


def attention_backward(qkv, o, dO, pk, n_head, M=None, ws_fill=True):
    L, lib = _lib()
    M = qkv.shape[0] if M is None else M
    dq = torch.full_like(qkv, float("nan"))
    cu, tl, sl = _packed_tensors(pk)
    nb = lib.vb_attention_backward_workspace(M, n_head)
    ws = _nan_ws(nb) if ws_fill else torch.zeros(nb, dtype=torch.uint8, device=DEV)
    L.check(lib.vb_attention_backward(qkv.data_ptr(), o.data_ptr(), dO.data_ptr(), _dt(qkv.dtype), M, len(pk.lens),
                                      n_head, A.HD, cu.data_ptr(), L.ptr(tl), L.ptr(sl), pk.seg1_start, max(pk.lens),
                                      _mode(pk.mode), dq.data_ptr(), ws.data_ptr(), nb, _s()), "vb_attention_backward")
    return dq


# ---- cases -----------------------------------------------------------------------------------------------------------
@dataclass(frozen=True)
class Case:
    name: str
    d: int
    H: int
    dff: int
    n_layer: int
    norm_first: bool
    adaptive: bool
    dtype: torch.dtype
    pack: str
    whole: bool = False


BIG = (1024, 16, 4096)
CHECKED_LAYERS = 2           # the per-op numerics run on the last two layers (the first two the backward handles)
CASES = [
    Case("ar_padded_ar_bf16_l12", *BIG, 12, True, False, torch.bfloat16, "ar", whole=True),
    Case("nar_padded_fp32_adaln", *BIG, 2, True, True, torch.float32, "nar"),
    Case("postln_padded_ar_bf16", *BIG, 2, False, False, torch.bfloat16, "ar_small"),
]


def _pack(kind):
    g = torch.Generator().manual_seed(sum(ord(c) for c in kind))
    if kind == "ar":            # 8 utterances padded to 150 text + 1350 audio rows: about 80 s of audio
        B, seg1, Lp = 8, 150, 1500
    elif kind == "ar_small":
        B, seg1, Lp = 4, 60, 421
    else:                       # NAR: 4 utterances padded to 100 text + 600 audio rows: about 40 s of audio
        B, seg1, Lp = 4, 100, 700
    S_ = [seg1] + torch.randint(1, seg1, (B - 1,), generator=g).tolist()
    c1 = [Lp - seg1] + torch.randint(1, Lp - seg1, (B - 1,), generator=g).tolist()
    return S.Pack([Lp] * B, "padded_ar" if kind.startswith("ar") else "padded", S_, c1, seg1)


def _saves(save, case, M):
    """layer l's forward values in the save buffer of vb_decoder_forward_train: the LayerSave layout of csrc/api.cu
    (x_in, x_mid fp32; xn1, att, xn2, qkv, hb in the storage dtype; each [Mp, width] with Mp = M rounded up to 128)"""
    d, dff = case.d, case.dff
    ts = 2 if case.dtype == torch.bfloat16 else 4
    Mp = -(-M // 128) * 128
    fields = [("x_in", d, torch.float32), ("x_mid", d, torch.float32), ("xn1", d, case.dtype), ("att", d, case.dtype),
              ("xn2", d, case.dtype), ("qkv", 3 * d, case.dtype), ("hb", dff, case.dtype)]
    sizes = [Mp * w * (4 if dt == torch.float32 else ts) for _, w, dt in fields]
    assert all(s % 256 == 0 for s in sizes)
    out, off = [], 0
    for _ in range(case.n_layer):
        sv = {}
        for (name, w, dt), n in zip(fields, sizes):
            sv[name] = save[off:off + M * w * (4 if dt == torch.float32 else ts)].view(dt).view(M, w)
            off += n
        out.append(sv)
    return out


def _run_library(case, m, pk, x0, gout, ada, drop=(0.0, 0)):
    """vb_decoder_forward_train then vb_decoder_backward (NaN-filled workspace); (save, dx, grads [per layer dict],
    dada)"""
    L, lib = _lib()
    nd = m["nd"]
    cu, tl, sl = _packed_tensors(pk)
    M, B = pk.M, len(pk.lens)
    x = x0.clone()
    nb = lib.vb_decoder_train_save_bytes(C.byref(nd.desc), M)
    save = torch.empty(nb, dtype=torch.uint8, device=DEV)
    L.check(lib.vb_decoder_forward_train(nd.handle, x.data_ptr(), M, B, cu.data_ptr(), L.ptr(tl), L.ptr(sl),
                                         pk.seg1_start, max(pk.lens), _mode(pk.mode), L.ptr(ada), save.data_ptr(), nb,
                                         float(drop[0]), int(drop[1]), _s()), "vb_decoder_forward_train")
    grads = [{k: torch.zeros(getattr(P, k).shape, device=DEV) for k in S.GRAD_NAMES} for P in m["layers"]]
    garr = (L.LayerGrads * case.n_layer)()
    for l in range(case.n_layer):
        for j, name in enumerate(L.LayerGrads._fields_):
            setattr(garr[l], name[0], grads[l][S.GRAD_NAMES[j]].data_ptr())
    dada = torch.zeros_like(ada) if ada is not None else None
    wt, keep = nd.transposed()
    dx = gout.clone()
    nb = lib.vb_decoder_backward_workspace(C.byref(nd.desc), M)
    ws = _nan_ws(nb)
    L.check(lib.vb_decoder_backward(nd.handle, dx.data_ptr(), M, B, cu.data_ptr(), L.ptr(tl), L.ptr(sl), pk.seg1_start,
                                    max(pk.lens), _mode(pk.mode), L.ptr(ada), L.ptr(dada), save.data_ptr(), wt, garr,
                                    ws.data_ptr(), nb, float(drop[0]), int(drop[1]), _s()), "vb_decoder_backward")
    torch.cuda.synchronize()
    return save, dx, grads, dada


def _inputs(case, pk, g):
    x = torch.randn(pk.M, case.d, generator=g)
    x[::7] += 4.0 * torch.randn(pk.M, 1, generator=g)[::7]
    gout = torch.randn(pk.M, case.d, generator=g) * 0.05
    return x.to(DEV), gout.to(DEV)


def _setup(case):
    m = _model(case.d, case.H, case.dff, case.n_layer, case.norm_first, case.adaptive, case.dtype)
    pk = _pack(case.pack)
    g = torch.Generator().manual_seed(sum(ord(c) for c in case.name))
    x0, gout = _inputs(case, pk, g)
    ada = m["nd"].ada_table(torch.randn(1, case.d, generator=g).to(DEV)) if case.adaptive else None
    return m, pk, x0, gout, ada


# ---- the checks of one layer's backward ops ---------------------------------------------------------------------
def _check_layer(case, pk, l, ops_, worst):
    kind = "wgmma" if case.dtype == torch.bfloat16 else "simt"

    def note(op, r):
        worst[op] = max(worst.get(op, 0.0), r)
        assert r <= 1.0, f"{case.name} layer {l} {op}: error / bound {r:.3g}"

    for name in ("cast1", "cast2"):
        t, out = ops_[name]
        assert torch.equal(_bits(out), _bits(t.to(case.dtype))), f"{case.name} layer {l} {name}"
    for name in ("ffn2_bwd", "ffn1_bwd", "out_bwd", "qkv_bwd"):
        a, W, dy, dst, out, dW, db = ops_[name]
        res_epi = (not case.norm_first) and name in ("ffn1_bwd", "qkv_bwd")
        note(f"{name} dX", S.dgrad_ratio(dy, W, S.EPI_RESIDUAL if res_epi else S.EPI_NONE, dst if res_epi else None,
                                         out, kind))
        z, bnd = S.wgrad_bound(a, dy, torch.zeros_like(dW), dW, kind)
        note(f"{name} dW", S.ratio(dW, z, bnd))
        z, bnd = S.colsum_bound(dy)
        note(f"{name} db", S.ratio(db, z, bnd))
    dh, hb, _, out = ops_["relu_bwd"]
    assert torch.equal(_bits(out), _bits(torch.where(hb > 0, dh, torch.zeros_like(dh)))), f"{case.name} relu"
    qkv, att, dO, dqkv = ops_["attn_bwd"]
    for k, r in S.attn_bwd_ratio(dqkv, qkv, att, dO, pk, case.H).items():
        note(f"attention {k}", r)
    for k in (1, 2):
        x, w, b, wb, dout, dst, out, dg, dbeta, dwb = ops_[f"norm{k}_bwd"]
        z, bnd = S.ln_bwd_bound(x, w, b, wb, dout, dst)
        note(f"norm{k} dx", S.ratio(out, z, bnd))
        for nm, (z, bnd) in S.ln_param_bounds(x, w, b, wb, dout).items():
            got = {"dgamma": dg, "dbeta": dbeta, "dada": dwb}[nm]
            note(f"norm{k} {nm}", S.ratio(got, z, bnd))


def _reduced_agree(case, a, b, bnd, what):
    r = float(((a.double() - b.double()).abs() / (2 * bnd)).max())
    assert r <= 1.0, f"{case.name}: {what} differs by {r:.3g} x twice its reordering bound"
    return r


@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_stack_backward_composition_and_numerics(case):
    m, pk, x0, gout, ada = _setup(case)
    save, dx_lib, g_lib, dada_lib = _run_library(case, m, pk, x0, gout, ada)
    saves = _saves(save, case, pk.M)
    g_loop = [{k: torch.zeros_like(v) for k, v in G.items()} for G in g_lib]
    dada_loop = torch.zeros_like(ada) if ada is not None else None
    worst, recs, per_layer = {}, {}, {}

    def rec(l, ops_):
        if l >= case.n_layer - CHECKED_LAYERS:
            _check_layer(case, pk, l, ops_, worst)
        if case.whole:
            per_layer[l] = _layer_input_grad(case, ops_).clone()
        recs[l] = {k: ops_[f"norm{k}_bwd"][:5] for k in (1, 2)}
        recs[l].update({n: ops_[n][2] for n in ("ffn2_bwd", "ffn1_bwd", "out_bwd", "qkv_bwd")})

    dx_loop = S.backward_loop(LibOps(case.dtype), saves, gout, m["layers"], pk, case.H, case.norm_first, g_loop, ada,
                              dada_loop, None, rec)
    torch.cuda.synchronize()
    assert torch.equal(_bits(dx_lib), _bits(dx_loop)), \
        f"{case.name}: dx differs in {int((_bits(dx_lib) != _bits(dx_loop)).sum())} elements"
    reorder = 0.0
    for l in range(case.n_layer):
        for k in ("in_w", "out_w", "w1", "w2"):
            assert torch.equal(_bits(g_lib[l][k]), _bits(g_loop[l][k])), f"{case.name} layer {l} {k}"
        for k, op in (("in_b", "qkv_bwd"), ("out_b", "out_bwd"), ("b1", "ffn1_bwd"), ("b2", "ffn2_bwd")):
            _, bnd = S.colsum_bound(recs[l][op])
            reorder = max(reorder, _reduced_agree(case, g_lib[l][k], g_loop[l][k], bnd, f"layer {l} {k}"))
        for j in (1, 2):
            x, w, b, wb, dout = recs[l][j]
            pb = S.ln_param_bounds(x, w, b, wb, dout)
            reorder = max(reorder, _reduced_agree(case, g_lib[l][f"n{j}w"], g_loop[l][f"n{j}w"], pb["dgamma"][1],
                                                  f"layer {l} norm{j} weight"))
            reorder = max(reorder, _reduced_agree(case, g_lib[l][f"n{j}b"], g_loop[l][f"n{j}b"], pb["dbeta"][1],
                                                  f"layer {l} norm{j} bias"))
            if ada is not None:
                row = 2 * l + j - 1
                reorder = max(reorder, _reduced_agree(case, dada_lib[row], dada_loop[row], pb["dada"][1],
                                                      f"layer {l} AdaLN row {row}"))
    REPORT.setdefault(case.name, {})["worst_error_over_bound"] = worst
    REPORT[case.name]["reduced_vectors_difference_over_twice_bound"] = reorder
    print(f"{case.name}: bit for bit; reduced vectors within {reorder:.3g} x twice their bound; worst error / bound "
          + ", ".join(f"{k} {v:.3g}" for k, v in worst.items()))
    if case.whole:
        _whole_stack(case, m, pk, saves, gout, ada, per_layer, None)
    _write_report()


def _layer_input_grad(case, ops_):
    """the gradient of layer l's input from backward_loop's record: norm1's output (pre-LN) or the attention block's
    residual epilogue (post-LN)"""
    return ops_["norm1_bwd"][6] if case.norm_first else ops_["qkv_bwd"][4]


def _whole_stack(case, m, pk, saves, gout, ada, lib_layers, drop):
    """per layer: the library's input gradient against backward_loop over float64 ops that round where the library
    stores (storage dtype operands and gradients, fp32 residual gradient), from the same saved forward values.
    Report only: the relative max error per layer."""
    ref = {}
    grads = [{k: torch.zeros(getattr(P, k).shape, dtype=torch.float64, device=DEV) for k in S.GRAD_NAMES}
             for P in m["layers"]]
    dada = torch.zeros_like(ada, dtype=torch.float64) if ada is not None else None
    S.backward_loop(S.Float64Ops(case.dtype, fp32_residual=True), saves, gout, m["layers"], pk, case.H,
                    case.norm_first, grads, ada, dada, drop,
                    lambda l, o: ref.__setitem__(l, _layer_input_grad(case, o).double()))
    rows = []
    for l in sorted(lib_layers, reverse=True):
        err = float((lib_layers[l].double() - ref[l]).abs().max() / ref[l].abs().max())
        rows.append(dict(layer=l, max_error_over_max_gradient=err))
        print(f"{case.name} layer {l}: max |lib - restatement| / max |gradient| {err:.3g}")
    REPORT.setdefault(case.name, {})["whole_stack"] = rows
    return rows


def test_stack_backward_with_dropout():
    """p = 0.1 at all four dropout sites on the AR batch shape (2 layers, 4 utterances): the library's input gradient
    per layer against the float64 restatement given the hash masks (report), which must be much closer to it than
    the restatement without the masks"""
    case = Case("ar_dropout_bf16", *BIG, 2, True, False, torch.bfloat16, "ar_small")
    m, pk, x0, gout, _ = _setup(case)
    drop = (0.1, 987654321)
    save, dx_lib, _, _ = _run_library(case, m, pk, x0, gout, None, drop)
    saves = _saves(save, case, pk.M)
    with_mask = _whole_stack(case, m, pk, saves, gout, None, {0: dx_lib}, drop)
    ref = {}
    grads = [{k: torch.zeros(getattr(P, k).shape, dtype=torch.float64, device=DEV) for k in S.GRAD_NAMES}
             for P in m["layers"]]
    S.backward_loop(S.Float64Ops(case.dtype, fp32_residual=True), saves, gout, m["layers"], pk, case.H, True, grads,
                    None, None, None, lambda l, o: ref.__setitem__(l, _layer_input_grad(case, o).double()))
    e_mask = [r for r in with_mask if r["layer"] == 0][0]["max_error_over_max_gradient"]
    e_plain = float((dx_lib.double() - ref[0]).abs().max() / ref[0].abs().max())
    REPORT[case.name]["without_masks"] = e_plain
    print(f"{case.name}: input gradient vs restatement with the masks {e_mask:.3g}, without {e_plain:.3g}")
    _write_report()
    assert torch.isfinite(dx_lib).all()
    assert e_mask < 0.1 * e_plain, (e_mask, e_plain)


# ---- attention backward: packed sweeps, isolation, masked keys ------------------------------------------------------
SWEEP_LENS = [1, 2, 63, 64, 65, 127, 128, 129, 191, 192, 193, 200]


def _sweep_pack(mode):
    n = len(SWEEP_LENS)
    if mode == "full":
        return S.Pack(SWEEP_LENS, mode, [0] * n, [0] * n)
    if mode == "valle_ar":
        return S.Pack(SWEEP_LENS, mode, [min(L, s) for L, s in zip(SWEEP_LENS, [1, 1, 10, 64, 1, 65, 47, 128, 63, 1,
                                                                                 100, 47])], [0] * n)
    seg1 = 60
    S_ = [min(L, seg1, s) for L, s in zip(SWEEP_LENS, [1, 2, 5, 60, 33, 1, 60, 17, 47, 60, 1, 59])]
    c1 = [max(0, min(L - seg1, c)) for L, c in zip(SWEEP_LENS, [0, 0, 3, 4, 5, 0, 68, 30, 131, 64, 1, 140])]
    return S.Pack(SWEEP_LENS, mode, S_, c1, seg1)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("mode", A.MODES)
def test_attention_backward_packed_sweep(mode, dtype):
    from valle_b200 import ops
    hh = 4
    pk = _sweep_pack(mode)
    M, d = pk.M, hh * A.HD
    g = torch.Generator().manual_seed(17 + len(mode))
    pad = 64                                    # rows past M, NaN in the isolation runs
    qkv = torch.zeros(M + pad, 3 * d, dtype=dtype, device=DEV)
    qkv[:M] = (torch.randn(M, 3 * d, generator=g) * 0.7).to(dtype).to(DEV)
    cu, tl, sl = _packed_tensors(pk)
    o = torch.zeros(M + pad, d, dtype=dtype, device=DEV)
    o[:M] = ops.attention(qkv[:M].contiguous(), cu, max(pk.lens), hh, _mode(pk.mode), tl, seg1_lens=sl,
                          seg1_start=pk.seg1_start)
    dO = torch.zeros(M + pad, d, dtype=dtype, device=DEV)
    dO[:M] = (torch.randn(M, d, generator=g) * 0.3).to(dtype).to(DEV)
    dq = attention_backward(qkv, o, dO, pk, hh, M=M)[:M]
    torch.cuda.synchronize()
    worst = S.attn_bwd_ratio(dq, qkv[:M], o[:M], dO[:M], pk, hh)
    REPORT.setdefault(f"attention_sweep_{mode}_{str(dtype).split('.')[-1]}", {})["worst_error_over_bound"] = worst
    print(f"attention backward sweep {mode} {dtype}: worst error / bound " +
          ", ".join(f"{k} {v:.3g}" for k, v in worst.items()))
    for k, r in worst.items():
        assert r <= 1.0, (k, r)
    # masked keys: the rows of keys that no query of their sequence sees get exactly no dK / dV
    for b, r0 in enumerate(pk.cu[:-1]):
        unseen = ~pk.vis(b).any(0)
        if unseen.any():
            rows = r0 + torch.nonzero(unseen).flatten().to(DEV)
            assert bool((dq[rows, d:] == 0).all()), f"{mode} seq {b}: a masked key got a gradient"
    # isolation: NaN in every other sequence's qkv, O and dO rows and in the rows past M changes no bit of this one
    for b in (2, 4, 9, 11):
        r0, r1 = pk.cu[b], pk.cu[b + 1]
        q2, o2, g2 = (t.clone() for t in (qkv, o, dO))
        for t in (q2, o2, g2):
            t[:r0] = float("nan")
            t[r1:] = float("nan")
        dq2 = attention_backward(q2, o2, g2, pk, hh, M=M)
        assert torch.equal(_bits(dq2[r0:r1]), _bits(dq[r0:r1])), f"{mode} seq {b}: a neighbour's NaN leaked in"
    _write_report()


# ---- vb_linear_backward: scratch, partial tiles, accumulate ---------------------------------------------------------
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("M,N,K", [(1, 1024, 1024), (63, 3072, 1024), (65, 1024, 4096), (333, 4096, 1024),
                                   (4000, 1088, 1024)])
def test_linear_backward_scratch_tiles_and_accumulate(M, N, K, dtype):
    """NaN-filled workspace (the transposes' pad rows must be zeroed, not read); dW / db prefilled: the result is
    prior + gradient; dX both written (EPI_NONE) and added into a prefilled fp32 buffer (EPI_RESIDUAL).
    (4000, 1088, 1024): the AR head's backward, its 1025 logits padded to 1088 columns."""
    L, lib = _lib()
    kind = "wgmma" if dtype == torch.bfloat16 else "simt"
    g = torch.Generator().manual_seed(M + N + K)
    a = torch.randn(M, K, generator=g).to(dtype).to(DEV)
    W = (torch.randn(N, K, generator=g) / math.sqrt(K)).to(dtype).to(DEV)
    dy = (torch.randn(M, N, generator=g) * 0.1).to(dtype).to(DEV)
    dW0 = torch.randn(N, K, generator=g).to(DEV) * 0.01
    db0 = torch.randn(N, generator=g).to(DEV)
    worst = {}
    for epi in (L.VB_EPI_NONE, L.VB_EPI_RESIDUAL):
        dW, db = dW0.clone(), db0.clone()
        res = torch.randn(M, K, generator=g).to(DEV)
        dX = res.clone() if epi == L.VB_EPI_RESIDUAL else torch.full((M, K), float("nan"), device=DEV)
        Wt = W.t().contiguous()
        nb = lib.vb_linear_backward_workspace(_dt(dtype), M, N, K)
        ws = _nan_ws(nb)
        L.check(lib.vb_linear_backward(a.data_ptr(), _dt(dtype), K, Wt.data_ptr(), dy.data_ptr(), N, dX.data_ptr(),
                                       L.VB_F32, K, epi, dW.data_ptr(), db.data_ptr(), M, N, K, ws.data_ptr(), nb,
                                       _s()), "vb_linear_backward")
        torch.cuda.synchronize()
        worst["dX"] = max(worst.get("dX", 0.0), S.dgrad_ratio(dy, W, epi, res if epi == L.VB_EPI_RESIDUAL else None,
                                                              dX, kind))
        z, bnd = S.wgrad_bound(a, dy, dW0, dW, kind)
        worst["dW"] = max(worst.get("dW", 0.0), S.ratio(dW, z, bnd))
        z, bnd = S.colsum_bound(dy, db0)
        worst["db"] = max(worst.get("db", 0.0), S.ratio(db, z, bnd))
    REPORT.setdefault("linear_backward", {})[f"M{M}_N{N}_K{K}_{str(dtype).split('.')[-1]}"] = worst
    _write_report()
    for k, r in worst.items():
        assert r <= 1.0, (k, r)


# ---- vb_layernorm_backward edges ------------------------------------------------------------------------------------
@pytest.mark.parametrize("d", [1024, 4096])
@pytest.mark.parametrize("adaptive", [False, True])
def test_layernorm_backward_edges(d, adaptive):
    """the strided `rows` gather (x with a row stride of d + 64) with dx accumulated into a prefilled buffer, rows
    offset by up to 4096 sigma, a bf16 dx_copy that must be bf16(dx) bit for bit, prefilled dgamma / dbeta / dada;
    d = 4096 takes the > 48 KB shared-memory launch"""
    L, lib = _lib()
    g = torch.Generator().manual_seed(d + int(adaptive))
    Mx, n = 700, 450
    xs = torch.randn(Mx, d + 64, generator=g)
    rho = torch.tensor([0.0, 16.0, 256.0, 4096.0])[torch.randint(0, 4, (Mx, 1), generator=g)]
    xs = (xs + rho) * 10.0 ** (torch.rand(Mx, 1, generator=g) * 3 - 2)
    xs = xs.to(DEV)
    x = xs[:, :d]
    rows = torch.randperm(Mx, generator=g)[:n].to(torch.int32).to(DEV)
    w = (1 + 0.2 * torch.randn(d, generator=g)).to(DEV)
    b = (0.1 * torch.randn(d, generator=g)).to(DEV)
    wb = torch.cat([1 + 0.1 * torch.randn(d, generator=g), 0.1 * torch.randn(d, generator=g)]).to(DEV) if adaptive \
        else None
    dy = torch.randn(n, d, generator=g).to(DEV)
    dx0 = (0.5 * torch.randn(Mx, d, generator=g)).to(DEV)
    dx = dx0.clone()
    copy = torch.full((Mx, d), float("nan"), dtype=torch.bfloat16, device=DEV)
    pri = {"dgamma": torch.randn(d, generator=g).to(DEV), "dbeta": torch.randn(d, generator=g).to(DEV),
           "dada": torch.randn(2 * d, generator=g).to(DEV)}
    got = {k: v.clone() for k, v in pri.items()}
    L.check(lib.vb_layernorm_backward(xs.data_ptr(), xs.stride(0), rows.data_ptr(), n, d, w.data_ptr(), b.data_ptr(),
                                      L.ptr(wb), S.EPS, dy.data_ptr(), d, dx.data_ptr(), d, copy.data_ptr(), L.VB_BF16,
                                      got["dgamma"].data_ptr(), got["dbeta"].data_ptr(),
                                      got["dada"].data_ptr() if adaptive else 0, _s()), "vb_layernorm_backward")
    torch.cuda.synchronize()
    rl = rows.long()
    xr = x.index_select(0, rl)
    z, bnd = S.ln_bwd_bound(xr, w, b, wb, dy, dx0[rl])
    worst = {"dx": S.ratio(dx[rl], z, bnd)}
    untouched = torch.ones(Mx, dtype=torch.bool, device=DEV)
    untouched[rl] = False
    assert torch.equal(_bits(dx[untouched]), _bits(dx0[untouched])), "rows outside `rows` changed"
    assert torch.equal(_bits(copy[rl]), _bits(dx[rl].to(torch.bfloat16))), "dx_copy is not bf16(dx)"
    assert bool(torch.isnan(copy[untouched].float()).all()), "dx_copy written outside `rows`"
    for k, (z, bnd) in S.ln_param_bounds(xr, w, b, wb, dy, {k: v for k, v in pri.items()}).items():
        worst[k] = S.ratio(got[k], z, bnd)
    if not adaptive:
        assert torch.equal(got["dada"], pri["dada"])
    REPORT.setdefault("layernorm_backward", {})[f"d{d}_{'adaln' if adaptive else 'ln'}"] = worst
    _write_report()
    print(f"vb_layernorm_backward d={d} adaptive={adaptive}: worst error / bound {worst}")
    for k, r in worst.items():
        assert r <= 1.0, (k, r)


# ---- the loss head ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("V,n_out", [(1025, 1088), (1024, 1024)])
@pytest.mark.parametrize("out_dtype", [torch.float32, torch.bfloat16])
def test_cross_entropy_and_backward(V, n_out, out_dtype):
    """logits spread over +-80, every 7th row at ignore_index (loss and gradient exactly 0), grad_rows weights,
    n_out > n_vocab padding columns exactly 0"""
    L, lib = _lib()
    g = torch.Generator().manual_seed(V + n_out)
    R, ignore = 3000, V if V == 1025 else -100
    logits = (torch.rand(R, V, generator=g) * 2 - 1) * 80
    logits[: R // 2] = torch.randn(R // 2, V, generator=g) * 3
    logits = logits.to(DEV)
    tg = torch.randint(0, V, (R,), generator=g)
    tg[::7] = ignore
    tg = tg.to(DEV)
    grow = (torch.rand(R, generator=g) + 0.5).to(DEV)
    loss = torch.full((R,), float("nan"), device=DEV)
    L.check(lib.vb_cross_entropy(logits.data_ptr(), V, tg.data_ptr(), R, V, ignore, loss.data_ptr(), _s()),
            "vb_cross_entropy")
    dl = torch.full((R, n_out), float("nan"), dtype=out_dtype, device=DEV)
    L.check(lib.vb_cross_entropy_backward(logits.data_ptr(), V, tg.data_ptr(), R, V, ignore, grow.data_ptr(), 0.5,
                                          dl.data_ptr(), _dt(out_dtype), n_out, n_out, _s()),
            "vb_cross_entropy_backward")
    torch.cuda.synchronize()
    z, bnd = S.ce_bound(logits, tg, V, ignore)
    worst = {"loss": S.ratio(loss, z, bnd)}
    z, bnd = S.ce_bwd_bound(logits, tg, V, ignore, grow, 0.5, n_out, dl)
    worst["dlogits"] = S.ratio(dl, z, bnd)
    skip = tg == ignore
    assert bool((loss[skip] == 0).all()) and bool((dl[skip].float() == 0).all()), "ignored rows"
    assert bool((dl[:, V:].float() == 0).all()), "padding columns"
    REPORT.setdefault("cross_entropy", {})[f"V{V}_nout{n_out}_{str(out_dtype).split('.')[-1]}"] = worst
    _write_report()
    for k, r in worst.items():
        assert r <= 1.0, (k, r)


def test_embed_rowdot_adaln_backward_accumulate():
    """vb_embed_backward over 8 tables (n = the occurrences of an id), vb_rowdot_accumulate for the sine-PE alpha
    (n = M d) and vb_adaln_project_backward, each into prefilled gradients: prior + gradient within reduce_bound"""
    L, lib = _lib()
    g = torch.Generator().manual_seed(99)
    d, n_rows, V = 1024, 3000, 1025
    worst = {}
    tok = torch.randint(0, V, (n_rows, 8), generator=g)
    tok[:, 0] = torch.randint(0, 4, (n_rows,), generator=g)        # hot ids: many occurrences
    tok = tok.to(DEV)
    dy = torch.randn(n_rows, d, generator=g).to(DEV)
    priors = [torch.randn(V, d, generator=g).to(DEV) for _ in range(8)]
    tabs = [p.clone() for p in priors]
    arr = (C.c_void_p * 8)(*[t.data_ptr() for t in tabs])
    rws = (C.c_int32 * 8)(*[V] * 8)
    L.check(lib.vb_embed_backward(tok.data_ptr(), 8, 1, arr, rws, 8, n_rows, d, dy.data_ptr(), d, 0, _s()),
            "vb_embed_backward")
    torch.cuda.synchronize()
    r = 0.0
    for j in range(8):
        ids = tok[:, j]
        z = priors[j].double().index_add(0, ids, dy.double())
        absum = torch.zeros(V, d, dtype=torch.float64, device=DEV).index_add(0, ids, dy.double().abs())
        cnt = int(torch.bincount(ids, minlength=V).max())
        r = max(r, S.ratio(tabs[j], z, S.reduce_bound(absum, cnt, priors[j])))
    worst["embed"] = r
    # rowdot: out += sum_r <a[r], pe[pos0 + r]>
    a = torch.randn(n_rows, d, generator=g).to(DEV)
    pe = torch.randn(n_rows + 10, d, generator=g).to(DEV)
    out = torch.tensor([3.0], device=DEV)
    L.check(lib.vb_rowdot_accumulate(a.data_ptr(), d, pe.data_ptr(), 10, 0, n_rows, d, out.data_ptr(), _s()),
            "vb_rowdot_accumulate")
    torch.cuda.synchronize()
    prod = a.double() * pe[10:].double()
    z = prod.sum() + 3.0
    bnd = S.reduce_bound(prod.abs().sum(), n_rows * d, torch.tensor(3.0), S.U32 * prod.abs().sum())
    worst["rowdot"] = S.ratio(out[0], z, bnd)
    # AdaLN projection backward
    W = (torch.randn(2 * d, d, generator=g) / math.sqrt(d)).to(DEV)
    e = torch.randn(d, generator=g).to(DEV)
    dwb = torch.randn(2 * d, generator=g).to(DEV)
    pW, pb, pe_ = (torch.randn(2 * d, d, generator=g) * 0.1).to(DEV), torch.randn(2 * d, generator=g).to(DEV), \
        torch.randn(d, generator=g).to(DEV)
    dW, db, de = pW.clone(), pb.clone(), pe_.clone()
    L.check(lib.vb_adaln_project_backward(W.data_ptr(), e.data_ptr(), dwb.data_ptr(), d, dW.data_ptr(), db.data_ptr(),
                                          de.data_ptr(), _s()), "vb_adaln_project_backward")
    torch.cuda.synchronize()
    t = dwb.double()[:, None] * e.double()[None]
    z = pW.double() + t
    worst["adaln dW"] = S.ratio(dW, z, (S.U32 * t.abs() + S.U32 * z.abs()) * S.SLACK + S.TINY)
    z = pb.double() + dwb.double()
    worst["adaln db"] = S.ratio(db, z, S.U32 * z.abs() * S.SLACK + S.TINY)
    t = W.double() * dwb.double()[:, None]
    z = pe_.double() + t.sum(0)
    worst["adaln de"] = S.ratio(de, z, S.reduce_bound(t.abs().sum(0), 2 * d, pe_, S.U32 * t.abs().sum(0)))
    REPORT["head_accumulate"] = worst
    _write_report()
    print(f"head accumulators: worst error / bound {worst}")
    for k, r in worst.items():
        assert r <= 1.0, (k, r)


def _write_report():
    out_dir = os.environ.get("VB_REPORT_DIR", tempfile.gettempdir())
    os.makedirs(out_dir, exist_ok=True)
    with open(os.path.join(out_dir, "stack_backward.json"), "w") as f:
        json.dump(REPORT, f, indent=1)
