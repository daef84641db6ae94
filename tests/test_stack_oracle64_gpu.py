"""The decoder-stack forward `vb_decoder_forward` against tests/stack_oracle64.py, at the benchmark's shapes.

For each case (CASES) the stack is built from valle_b200.modules.transformer with seeded random weights and run by
NativeDecoder.forward.  Then:
  * composition: `layer_loop` over the library's public ops (vb_layernorm, vb_linear, vb_attention with the layer's
    cache pointers, vb_cast_from_f32) reproduces it bit for bit: the output rows, both KV caches and the sentinel in
    every cache row the prefill must not write;
  * numerics: in every layer each op of that run -- norm1 / norm2, the QKV projection, the attention, the out-proj
    residual, FFN1 + ReLU, the FFN2 residual -- is within its derived bound (stack_oracle64.ln_bound / gemm_bound,
    attention_oracle64.bound) of its float64 value computed on the GPU from the inputs it received.  Rows that see no
    key (the padded modes without text): the kernels write NaN there (0 * (1 / l) with l = 0), as
    F.multi_head_attention_forward does; every later op of that sequence reads it, so those elements (reference not
    finite) are left out of the bound checks, and the test asserts that the NaN stays in its sequence;
  * the NAR case also checks the 7 stages' AdaLN tables (vb_adaln_project), the head (the final AdaLN of the target
    rows to bf16, the [G, 1024] logits of vb_linear within gemm_bound) and vb_nar_argmax_accumulate: bit for bit
    against torch.argmax of the kernel's own logits with planted exact ties, the y_emb update and the code column,
    and against the float64 argmax wherever the logits' bound leaves no tie;
  * whole stack (NAR): the 12-layer output per layer against the float64 restatement with the same rounding points,
    under the same-chain bar of tests/test_decode_step_gpu.py (FP32_REL S + 2 E per row).  A report with a safety net;
    the tight checks are the two above.
The worst error / bound per op and case, and the whole-stack errors per layer, go to stack.json in $VB_REPORT_DIR
(default: the system temporary directory)."""
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

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
FP32_REL = 4096 * 2.0 ** -24
SENTINEL = 6144.0        # exact in bf16
N_AUDIO = 1024
REPORT = {}


# ---- models --------------------------------------------------------------------------------------------------------
_MODELS = {}


def _model(d, H, dff, n_layer, norm_first, adaptive, dtype):
    key = (d, H, dff, n_layer, norm_first, adaptive, dtype)
    if key in _MODELS:
        return _MODELS[key]
    _MODELS.clear()
    torch.cuda.empty_cache()
    from valle_b200.modules.transformer import (AdaptiveLayerNorm, LayerNorm, TransformerEncoder,
                                                TransformerEncoderLayer)
    torch.manual_seed(31)
    final = None
    if norm_first:
        final = AdaptiveLayerNorm(d, LayerNorm(d)) if adaptive else LayerNorm(d)
    enc = TransformerEncoder(TransformerEncoderLayer(d, H, dff, dropout=0.0, batch_first=True, norm_first=norm_first,
                                                     adaptive_layer_norm=adaptive), n_layer, norm=final)
    g = torch.Generator().manual_seed(32 + n_layer + 2 * int(norm_first) + 4 * int(adaptive))
    with torch.no_grad():
        for name, p in enc.named_parameters():
            if p.ndim == 2:
                p.copy_(torch.randn(p.shape, generator=g) / math.sqrt(p.shape[1]))
            elif "norm" in name and name.endswith("weight"):
                p.copy_(1.0 + 0.2 * torch.randn(p.shape, generator=g))
            else:
                p.copy_(0.1 * torch.randn(p.shape, generator=g))
    enc = enc.to(DEV).eval()
    nd = enc.native(dtype)

    def nrm(m):
        return m.norm if adaptive else m

    layers = [S.Layer(l.self_attn.in_proj_weight.detach().to(dtype), l.self_attn.in_proj_bias.detach(),
                      l.self_attn.out_proj.weight.detach().to(dtype), l.self_attn.out_proj.bias.detach(),
                      l.linear1.weight.detach().to(dtype), l.linear1.bias.detach(),
                      l.linear2.weight.detach().to(dtype), l.linear2.bias.detach(),
                      nrm(l.norm1).weight.detach(), nrm(l.norm1).bias.detach(),
                      nrm(l.norm2).weight.detach(), nrm(l.norm2).bias.detach()) for l in enc.layers]
    m = dict(enc=enc, nd=nd, layers=layers)
    _MODELS[key] = m
    return m


# ---- the library's public ops ----------------------------------------------------------------------------------------
class LibOps:
    """layer_loop's ops through valle_b200.ops / vb_attention; kc / vc [n_layer, B, H, cap, 64]: the KV cache"""

    def __init__(self, dtype, kc=None, vc=None):
        self.dtype, self.kc, self.vc = dtype, kc, vc

    def norm(self, x, w, b, wb, operand):
        from valle_b200 import ops
        return ops.layernorm(x, w, b, S.EPS, wb, out_dtype=self.dtype if operand else torch.float32)

    def linear(self, a, W, b, epi, res):
        from valle_b200 import ops
        if epi == S.EPI_RESIDUAL:
            out = res.clone()
            return ops.linear(a, W, b, epi, out=out)
        return ops.linear(a, W, b, epi)

    def attention(self, qkv, pk, n_head, l):
        from valle_b200 import _lib as L
        M, d = qkv.shape[0], qkv.shape[1] // 3
        out = torch.empty(M, d, dtype=qkv.dtype, device=DEV)
        cu, tl, sl = _packed_tensors(pk)
        kc = vc = None
        stride, cap = 0, 0
        if self.kc is not None:
            kc, vc = self.kc[l], self.vc[l]
            stride, cap = kc.stride(0), kc.shape[2]
        L.check(L.load().vb_attention(qkv.data_ptr(), L.VB_BF16 if qkv.dtype == torch.bfloat16 else L.VB_F32, M,
                                      len(pk.lens), n_head, A.HD, cu.data_ptr(), L.ptr(tl), L.ptr(sl), pk.seg1_start,
                                      max(pk.lens), _mode(pk.mode), out.data_ptr(), L.ptr(kc), L.ptr(vc), stride, cap,
                                      None, 0, torch.cuda.current_stream().cuda_stream), "vb_attention")
        return out

    def cast(self, x):
        from valle_b200 import ops
        return ops.cast_from_f32(x, self.dtype)


def _mode(name):
    from valle_b200 import _lib as L
    return dict(full=L.VB_MASK_FULL, valle_ar=L.VB_MASK_VALLE_AR, padded_ar=L.VB_MASK_PADDED_AR,
                padded=L.VB_MASK_PADDED)[name]


def _packed_tensors(pk):
    cu = torch.tensor(pk.cu, dtype=torch.int32, device=DEV)
    tl = torch.tensor(pk.S, dtype=torch.int32, device=DEV) if pk.mode != "full" else None
    sl = torch.tensor(pk.c1, dtype=torch.int32, device=DEV) if pk.mode.startswith("padded") else None
    return cu, tl, sl


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
    cache_cap: int = 0
    whole: bool = False            # the whole-stack report against the float64 restatement
    head: bool = False             # the NAR head and argmax for all 7 stages


BIG = (1024, 16, 4096, 12)
TINY = (256, 4, 1024)
CASES = [
    Case("nar_b64_l1025", *BIG, True, True, torch.bfloat16, "nar", whole=True, head=True),
    Case("nar_ragged28", *BIG, True, True, torch.bfloat16, "ragged_full"),
    Case("prefill_b64_l272", *BIG, True, False, torch.bfloat16, "prefill", cache_cap=288),
    Case("postln_ln_l3", *TINY, 3, False, False, torch.bfloat16, "sweep_valle_ar", cache_cap=264),
    Case("postln_adaln_l2", *TINY, 2, False, True, torch.bfloat16, "sweep_full"),
    Case("train_padded_ar", *TINY, 2, True, False, torch.bfloat16, "ragged_padded_ar"),
    Case("train_padded", *TINY, 2, True, False, torch.bfloat16, "ragged_padded"),
    Case("fp32_preln", *TINY, 2, True, False, torch.float32, "b8_valle_ar"),
    Case("fp32_postln", *TINY, 2, False, False, torch.float32, "b8_full"),
]


def _pack(kind):
    if kind == "nar":               # the benchmark's NAR passes: 47 text + 225 prompt + 753 frames
        return S.Pack([1025] * 64, "full", [0] * 64, [0] * 64)
    if kind == "prefill":           # the benchmark's AR prefill: 47 text + 225 prompt rows
        return S.Pack([272] * 64, "valle_ar", [47] * 64, [0] * 64)
    if kind.startswith("sweep_"):
        lens = list(A.SWEEP_L)
        return S.Pack(lens, kind[6:], [min(L, 47) for L in lens], [0] * len(lens))
    if kind.startswith("b8_"):
        lens = [300, 1, 64, 65, 129, 200, 17, 299]
        return S.Pack(lens, kind[3:], [min(L, 47) for L in lens], [0] * len(lens))
    lens, S_, c1 = A._ragged_lengths()
    mode = kind[len("ragged_"):]
    if mode == "full":
        return S.Pack(lens, mode, [0] * len(lens), [0] * len(lens))
    # training masks: text padded to 60 rows; sequence 2 has no text (PADDED_AR: its 60 text rows see no key),
    # sequence 3 no audio, sequence 5 neither
    S_, c1 = list(S_), list(c1)
    S_[2], c1[3], S_[5], c1[5] = 0, 0, 0, 0
    return S.Pack(lens, mode, S_, c1, A.SEG1_START)


def _inputs(case, pk, g):
    x = torch.randn(pk.M, case.d, generator=g)
    x[::7] += 4.0 * torch.randn(pk.M, 1, generator=g)[::7]       # some rows with a common offset
    return x.to(DEV)


# ---- the checks of one layer's ops ------------------------------------------------------------------------------------
def _check_layer(case, pk, l, ops_, worst, kc=None, vc=None):
    kind = "wgmma" if case.dtype == torch.bfloat16 else "simt"
    akind = "wgmma" if case.dtype == torch.bfloat16 else "simt_f32"

    def note(op, r):
        worst[op] = max(worst.get(op, 0.0), r)
        assert r <= 1.0, f"{case.name} layer {l} {op}: error / bound {r:.3g}"

    for k in (1, 2):
        x, w, b, wb, out = ops_[f"norm{k}"]
        note(f"norm{k}", S.ln_ratio(x, w, b, wb, out))
    for name in ("cast1", "cast2"):
        if name in ops_:
            x, out = ops_[name]
            assert torch.equal(out, x.to(case.dtype)), f"{case.name} layer {l} {name}: not x rounded to nearest"
    a, W, b, out = ops_["qkv"]
    note("qkv", S.gemm_ratio(a, W, b, S.EPI_NONE, None, out, kind))
    qkv, att = ops_["attn"]
    d, H = case.d, case.H
    ra = 0.0
    for s, r0 in enumerate(pk.cu[:-1]):
        L = pk.lens[s]
        q, k_, v = (qkv[r0:r0 + L, i * d:(i + 1) * d].reshape(L, H, A.HD).transpose(0, 1) for i in range(3))
        ref = A.attention64(q, k_, v, pk.vis(s).to(DEV), head_chunk=8)
        got = att[r0:r0 + L].view(L, H, A.HD).transpose(0, 1)
        if torch.isfinite(qkv[r0:r0 + L]).all():
            ra = max(ra, A.ratio(got, ref, A.bound(ref, akind)))
        if ref.empty:       # rows that see no key: 0 * (1 / 0)
            assert torch.isnan(got[:, sorted(ref.empty)]).all(), f"{case.name} layer {l}: seq {s} rows without keys"
        if kc is not None:  # the rows [0, L) of this layer's cache are the K / V columns of qkv
            assert torch.equal(kc[l, s, :, :L], k_.contiguous()) and torch.equal(vc[l, s, :, :L], v.contiguous())
    note("attention", ra)
    a, W, b, res, out = ops_["out"]
    note("out_proj_residual", S.gemm_ratio(a, W, b, S.EPI_RESIDUAL, res, out, kind))
    a, W, b, out = ops_["ffn1"]
    note("ffn1_relu", S.gemm_ratio(a, W, b, S.EPI_RELU, None, out, kind))
    a, W, b, res, out = ops_["ffn2"]
    note("ffn2_residual", S.gemm_ratio(a, W, b, S.EPI_RESIDUAL, res, out, kind))


def _bits(t):
    return t.view(torch.int16) if t.dtype == torch.bfloat16 else t.view(torch.int32)


@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_stack_composition_and_numerics(case):
    m = _model(case.d, case.H, case.dff, case.n_layer, case.norm_first, case.adaptive, case.dtype)
    pk = _pack(case.pack)
    g = torch.Generator().manual_seed(sum(ord(c) for c in case.name))
    x0 = _inputs(case, pk, g)
    ada = None
    if case.adaptive:
        emb = torch.randn(1, case.d, generator=g).to(DEV)
        ada = m["nd"].ada_table(emb)
    cu, tl, sl = _packed_tensors(pk)
    B, H = len(pk.lens), case.H
    caches = {}
    if case.cache_cap:
        for who in ("lib", "loop"):
            caches[who] = tuple(torch.full((case.n_layer, B, H, case.cache_cap, A.HD), sgn * SENTINEL,
                                           dtype=case.dtype, device=DEV) for sgn in (1, -1))
    # the library's stack
    x_lib = x0.clone()
    kc, vc = caches.get("lib", (None, None))
    m["nd"].forward(x_lib, cu, B, max(pk.lens), _mode(pk.mode), tl, ada, kc, vc, case.cache_cap, sl, pk.seg1_start)
    torch.cuda.synchronize()
    # the layer loop over the public ops, checking each layer's ops as it goes
    worst = {}
    kl, vl = caches.get("loop", (None, None))
    per_layer = []

    def rec(l, ops_):
        _check_layer(case, pk, l, ops_, worst, kl, vl)
        if case.whole:
            per_layer.append(ops_["ffn2" if case.norm_first else "norm2"][-1].clone())

    x_loop = S.layer_loop(LibOps(case.dtype, kl, vl), x0, m["layers"], pk, H, case.norm_first, ada, rec)
    torch.cuda.synchronize()
    assert torch.equal(_bits(x_lib), _bits(x_loop)), \
        f"{case.name}: vb_decoder_forward differs from the layer loop over the public ops in " \
        f"{int((_bits(x_lib) != _bits(x_loop)).sum())} elements"
    if case.cache_cap:
        for i, nm in enumerate(("K", "V")):
            assert torch.equal(_bits(caches["lib"][i]), _bits(caches["loop"][i])), f"{case.name}: {nm} cache differs"
            c = caches["lib"][i]
            for s, L in enumerate(pk.lens):
                assert bool((c[:, s, :, L:] == (1 - 2 * i) * SENTINEL).all()), f"{case.name}: {nm} cache row >= {L}"
    # a sequence's NaN (rows without keys) stays in it
    seq_nan = [s for s in range(B) if not torch.isfinite(x_lib[pk.cu[s]:pk.cu[s + 1]]).all()]
    bad = [s for s in seq_nan if not pk.empty_rows()[pk.cu[s]:pk.cu[s + 1]].any()]
    assert not bad, f"{case.name}: sequences {bad} have no row without keys but non-finite outputs"
    REPORT.setdefault(case.name, {})["worst_error_over_bound"] = worst
    print(f"{case.name}: bit for bit; worst error / bound " + ", ".join(f"{k} {v:.3g}" for k, v in worst.items()))
    if case.head:
        _check_head(case, m, x_lib, pk, g)
    if case.whole:
        _whole_stack(case, m, x0, pk, ada, per_layer)
    _write_report()


# ---- NAR head ----------------------------------------------------------------------------------------------------------
def _check_head(case, m, x, pk, g):
    from valle_b200 import ops
    nd, enc, d = m["nd"], m["enc"], case.d
    # the target rows: the 753 generated frames of each utterance (47 text + 225 prompt rows ahead of them)
    tgt = torch.cat([torch.arange(r0 + 272, r0 + 1025) for r0 in pk.cu[:-1]]).to(torch.int32).to(DEV)
    G = tgt.numel()
    head_w = (torch.randn(N_AUDIO, d, generator=g) / math.sqrt(d)).to(DEV).to(torch.bfloat16)
    next_emb = torch.randn(N_AUDIO, d, generator=g).to(DEV)
    worst = {}
    norms = [n for l in enc.layers for n in (l.norm1, l.norm2)] + [enc.norm]
    for stage in range(7):
        emb = torch.randn(1, d, generator=g).to(DEV)
        ada = nd.ada_table(emb)
        r = 0.0
        for i, nm in enumerate(norms):
            z, bnd = S.adaln_bound(nm.project_layer.weight.detach(), nm.project_layer.bias.detach(), emb[0], ada[i])
            r = max(r, S.ratio(ada[i], z, bnd))
        worst["adaln_table"] = max(worst.get("adaln_table", 0.0), r)
        assert r <= 1.0, f"stage {stage}: AdaLN table error / bound {r:.3g}"
        hn = nd.head_rows(x, ada, tgt, torch.bfloat16)
        xr = x.index_select(0, tgt.long())
        r = S.ln_ratio(xr, nd.final_w, nd.final_b, ada[2 * case.n_layer], hn)
        worst["head_norm"] = max(worst.get("head_norm", 0.0), r)
        assert r <= 1.0, f"stage {stage}: head norm error / bound {r:.3g}"
        logits = torch.empty(G, N_AUDIO, dtype=torch.float32, device=DEV)
        ops.linear(hn, head_w, None, S.EPI_NONE, out=logits)
        codes = torch.full((G, 8), -5, dtype=torch.int64, device=DEV)
        ops.nar_argmax_accumulate(logits, codes[:, stage + 1], codes.stride(0), None, None)
        # logits within gemm_bound; outside the tie band the code is the float64 argmax
        r, decided, agree = 0.0, 0, 0
        step = 8192
        for r0 in range(0, G, step):
            sl = slice(r0, r0 + step)
            z, bnd = S.gemm_bound(hn[sl], head_w, None, S.EPI_NONE, None, logits[sl], "wgmma")
            r = max(r, S.ratio(logits[sl], z, bnd))
            j = z.argmax(-1)
            lo = z.gather(1, j[:, None])[:, 0] - bnd.gather(1, j[:, None])[:, 0]
            hi = (z + bnd).scatter(1, j[:, None], -math.inf).amax(-1)
            sure = lo > hi
            decided += int(sure.sum())
            agree += int((codes[sl, stage + 1][sure] == j[sure]).sum())
        worst["head_logits"] = max(worst.get("head_logits", 0.0), r)
        assert r <= 1.0, f"stage {stage}: logits error / bound {r:.3g}"
        assert agree == decided, f"stage {stage}: {decided - agree} of {decided} decided rows differ from the f64 argmax"
        # bit for bit: planted exact ties (the first index wins), the code column, the y_emb update
        lg = logits.clone()
        rows = torch.arange(0, G, 97, device=DEV)
        amax = lg[rows].argmax(-1)
        early = torch.clamp(amax - 1 - (rows % 5), min=0)
        late = torch.clamp(amax + 1 + (rows % 7), max=N_AUDIO - 1)
        lg[rows, early] = lg[rows, amax]
        lg[rows, late] = lg[rows, amax]
        y_emb = torch.randn(pk.M, d, generator=g).to(DEV)
        y0 = y_emb.clone()
        codes = torch.full((G, 8), -5, dtype=torch.int64, device=DEV)
        ops.nar_argmax_accumulate(lg, codes[:, stage + 1], codes.stride(0), next_emb, y_emb, tgt)
        torch.cuda.synchronize()
        want = torch.argmax(lg, -1)
        assert torch.equal(codes[:, stage + 1], want)
        assert bool((codes[:, [c for c in range(8) if c != stage + 1]] == -5).all())
        expect = y0.clone()
        expect[tgt.long()] = y0[tgt.long()] + next_emb[want]
        assert torch.equal(y_emb.view(torch.int32), expect.view(torch.int32))
    REPORT.setdefault(case.name, {})["head"] = worst
    print(f"{case.name} head, 7 stages: worst error / bound " + ", ".join(f"{k} {v:.3g}" for k, v in worst.items()))


def test_nar_argmax_nan_rows_follow_torch():
    """a NaN is the maximum and the first NaN wins (torch.argmax): an all-NaN row, one-NaN rows, a two-NaN row; the
    embedding row added is next_emb[code]"""
    from valle_b200 import ops
    V, d = 1024, 64
    g = torch.Generator().manual_seed(41)
    lg = torch.randn(6, V, generator=g)
    lg[0] = float("nan")
    lg[1, 517] = float("nan")
    lg[2, 0] = float("nan")
    lg[3, 1023] = float("nan")
    lg[4, 900], lg[4, 33] = float("nan"), float("nan")
    lg = lg.to(DEV)
    next_emb = torch.randn(V, d, generator=g).to(DEV)
    y = torch.randn(6, d, generator=g).to(DEV)
    y0 = y.clone()
    codes = torch.full((6, 2), -5, dtype=torch.int64, device=DEV)
    ops.nar_argmax_accumulate(lg, codes[:, 1], codes.stride(0), next_emb, y)
    torch.cuda.synchronize()
    want = torch.argmax(lg, -1)
    assert want.tolist()[:5] == [0, 517, 0, 1023, 33]
    assert torch.equal(codes[:, 1], want) and bool((codes[:, 0] == -5).all())
    assert torch.equal(y.view(torch.int32), (y0 + next_emb[want]).view(torch.int32))


# ---- whole stack ---------------------------------------------------------------------------------------------------------
def _whole_stack(case, m, x0, pk, ada, lib_layers):
    """per layer: the library's rows against the float64 restatement with the same rounding points (bf16 storage, fp32
    residual), under FP32_REL S + 2 E per row (S: the row's largest |value| in the restatement, E: the row's largest
    |difference| between the restatement and the unrounded stack)"""
    exact, rounded = [], []
    S.layer_loop(S.Float64Ops(), x0, m["layers"], pk, case.H, case.norm_first, ada,
                 lambda l, o: exact.append(o["ffn2" if case.norm_first else "norm2"][-1].float()))
    rows = []

    def rec(l, o):
        ref = o["ffn2" if case.norm_first else "norm2"][-1].double()
        E = (ref - exact[l].double()).abs().amax(-1)
        Sx = ref.abs().amax(-1)
        err = (lib_layers[l].double() - ref).abs().amax(-1)
        bar = FP32_REL * Sx + 2 * E
        rows.append(dict(layer=l, max_error=float(err.max()), max_E=float(E.max()),
                         worst_error_over_bar=float((err / bar).max())))
        exact[l] = None

    S.layer_loop(S.Float64Ops(case.dtype, fp32_residual=True), x0, m["layers"], pk, case.H, case.norm_first, ada, rec)
    REPORT.setdefault(case.name, {})["whole_stack"] = rows
    for r in rows:
        print(f"{case.name} layer {r['layer']}: max |lib - restatement| {r['max_error']:.3g}, max E {r['max_E']:.3g}, "
              f"error / bar {r['worst_error_over_bar']:.3g}")
    worst = max(r["worst_error_over_bar"] for r in rows)
    assert worst <= 1.0, f"{case.name}: whole-stack error / bar {worst:.3g}"


def _write_report():
    out_dir = os.environ.get("VB_REPORT_DIR", tempfile.gettempdir())
    os.makedirs(out_dir, exist_ok=True)
    with open(os.path.join(out_dir, "stack.json"), "w") as f:
        json.dump(REPORT, f, indent=1)
