"""GPU checks of post-LN VALL-E (`norm_first=False`, valle/modules/transformer.py:303-308; no final norm,
valle/models/valle.py:151,242-246) on an H100: the engine against the reference's stored outputs (fp32 ids
bit-exact), bf16 against the fp32 engine, batching, the decode chain's launch count, the module surface and the
training gradients."""
import contextlib
import os
import random

import pytest
import torch
import torch.nn.functional as F

from conftest import load_golden
from oracle import valle_oracle as O
from test_backward_gpu import _keep_mask, _no_dropout, _rel
from test_post_ln import postln_model

import postln_oracle as P

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
# bf16 bars: the pre-LN bars (tests/test_parity_bf16_gpu.py, tests/test_backward_gpu.py), except where bf16 rounding
# alone moves the reference computation itself further.  postln_oracle.bf16_gemm_operands() restates the oracle with
# every GEMM operand (and output gradient) rounded to bf16 and fp32 accumulation; where its own error exceeds a bar,
# the bar is EMUL_FACTOR times that error.  The factor covers the rounding points the restatement leaves out (bf16 q,
# k, v and attention probabilities, accumulation order).  At d=1024/16h/12L the restatement's worst NAR frame is 5.5 % of
# its stage's logit std, and on the tiny training batch its worst gradient is 6.3 % (a ReLU gate that bf16 rounding
# flips on a row with a large upstream gradient); the same restatement of the pre-LN fixtures stays inside the bars
# (NAR 1.4 %, config0 gradients 4.3 %).
AR_TOL, NAR_TOL_REL, GRAD_TOL_BF16, EMUL_FACTOR = 0.03, 0.03, 6e-2, 1.25


def _model(g, dtype=torch.float32):
    m = postln_model(g["config"], g["weight_seed"])
    if g.get("buffers"):
        m.load_state_dict(g["buffers"], strict=False)
    got = O.weight_checksums(m.state_dict())
    assert all(torch.equal(got[k], g["checksums"][k]) for k in got)
    m = m.to(DEV)
    m.engine_dtype = dtype
    m.engine(dtype).quiet = True
    return m


def _xl(x):
    return torch.tensor([x.shape[1]], dtype=torch.int32)


def _utts(n, seed=3, S=(5, 12), Tp=(8, 30)):
    g = torch.Generator().manual_seed(seed)
    out = []
    for _ in range(n):
        s = int(torch.randint(S[0], S[1], (), generator=g))
        t = int(torch.randint(Tp[0], Tp[1], (), generator=g))
        out.append((torch.randint(3, 100, (s,), generator=g), torch.randint(0, 1024, (t, 8), generator=g)))
    return out


# ---------------------------------------------------------------- fp32 parity with the reference
@pytest.mark.parametrize("name", ["tiny_postln_pm0.pt", "tiny_postln_pm1.pt", "tiny_postln_prenet.pt",
                                  "big_short_postln.pt"])
def test_greedy_ids_bit_exact_vs_reference(name):
    g = load_golden(name)
    m = _model(g)
    x, y = g["x"].to(DEV), g["y"].to(DEV)
    codes, ref = m.inference(x, _xl(x), y, None, top_k=1).cpu(), g["codes"].long()
    assert codes.shape == ref.shape, (codes.shape, ref.shape)
    assert torch.equal(codes, ref), int((codes != ref).sum())


@pytest.mark.parametrize("name", ["tiny_postln_pm0.pt", "tiny_postln_pm1.pt"])
def test_continual_and_host_sampling_bit_exact(name):
    g = load_golden(name)
    m = _model(g)
    x, y = g["x"].to(DEV), g["y"].to(DEV)
    assert torch.equal(m.continual(x, _xl(x), y).cpu(), g["continual"].long())
    s = g["sampled"]
    eng = m.engine()
    eng.sample_on_host = True
    torch.manual_seed(s["torch_seed"])
    got = m.inference(x, _xl(x), y, None, top_k=s["top_k"], temperature=s["temperature"]).cpu()
    assert torch.equal(got, s["codes"].long())


def test_ar_logits_within_tolerance_big_short():
    g = load_golden("big_short_postln.pt")
    eng = _model(g).engine()
    steps = g["ar_logit_steps"].tolist()
    tr = {"steps": set(steps)}
    eng.generate([g["x"][0]], [g["y"][0]], top_k=1, trace=tr)
    for i, s in enumerate(steps):
        err = float((tr["ar_logits"][s][0].cpu() - g["ar_logits"][i]).abs().max())
        assert err < 2e-4, (s, err)


@pytest.mark.parametrize("name", ["tiny_postln_pm0.pt", "tiny_postln_pm1.pt"])
def test_training_losses_match_reference(name):
    g = load_golden(name)
    fw = g["forward"]
    for dtype, tol in ((torch.float32, 1e-4), (torch.bfloat16, 2e-2)):
        m = _model(g, dtype)
        for stage in (0, 1, 2):
            m.rng = random.Random(0)
            torch.manual_seed(int(fw["torch_seed"]))
            with torch.no_grad():
                (_, _), loss, _ = m(fw["x"].to(DEV), fw["x_lens"], fw["y"].long().to(DEV), fw["y_lens"], train_stage=stage)
            want = float(fw[f"loss_stage{stage}"])
            assert abs(float(loss) - want) <= tol * abs(want), (dtype, stage, float(loss), want)


# ---------------------------------------------------------------- batching
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_ragged_batch_equals_solo_decodes(dtype):
    g = load_golden("tiny_postln_pm1.pt")
    m = _model(g, dtype)
    utts = _utts(5)
    outs = m.inference_batch([u[0] for u in utts], [u[1] for u in utts], top_k=1, max_new_tokens=40, dtype=dtype)
    for (t, p), o in zip(utts, outs):
        solo = m.inference_batch([t], [p], top_k=1, max_new_tokens=40, dtype=dtype)[0]
        assert torch.equal(o, solo)


def test_bf16_seventy_utterances_equal_solo_decodes_and_seeds_are_per_utterance():
    g = load_golden("tiny_postln_pm1.pt")
    m = _model(g, torch.bfloat16)
    utts = _utts(70, seed=5)
    texts, prompts = [u[0] for u in utts], [u[1] for u in utts]
    outs = m.inference_batch(texts, prompts, top_k=1, max_new_tokens=12, dtype=torch.bfloat16)
    sampled = m.inference_batch(texts, prompts, top_k=5, temperature=0.9, max_new_tokens=12, dtype=torch.bfloat16,
                                seed=100)
    for b in (0, 1, 63, 64, 69):
        solo = m.inference_batch([texts[b]], [prompts[b]], top_k=1, max_new_tokens=12, dtype=torch.bfloat16)[0]
        assert torch.equal(outs[b], solo), b
        solo = m.inference_batch([texts[b]], [prompts[b]], top_k=5, temperature=0.9, max_new_tokens=12,
                                 dtype=torch.bfloat16, seed=100 + b)[0]
        assert torch.equal(sampled[b], solo), b


# ---------------------------------------------------------------- bf16 tensor-core path
def test_bf16_teacher_forced_logits_vs_fp32_engine_big_short():
    """d=1024/16h/12L, teacher-forced with the reference's ids: every bf16 AR step within 0.03 of the fp32 engine, argmax
    flips only at the reference's near-ties, NAR logits within 3 % of each stage's logit std, or EMUL_FACTOR times the
    worst error of the bf16-operand restatement of the reference where that is larger"""
    g = load_golden("big_short_postln.pt")
    ref = g["codes"][0].long()
    n = ref.shape[0]
    res = {}
    for dtype in (torch.float32, torch.bfloat16):
        eng = _model(g, dtype).engine()
        tr = {"steps": "all", "nar": True}
        out = eng.generate([g["x"][0]], [g["y"][0]], top_k=1, trace=tr, forced=[ref])[0].cpu()
        assert torch.equal(out, ref)
        res[dtype] = (torch.stack([tr["ar_logits"][i][0].cpu() for i in range(n + 1)]),
                      [t.cpu() for t in tr["nar_logits"]], [t.cpu() for t in tr["nar_argmax"]])
    ar32, nar32, _ = res[torch.float32]
    ar16, nar16, arg16 = res[torch.bfloat16]
    err = (ar16 - ar32).abs().amax(dim=1)
    assert float(err.max()) < AR_TOL, float(err.max())
    flips = ar16[:n].argmax(dim=1) != ref[:, 0]
    assert not bool((flips & (g["ar_margin"][:n] > 2 * err[:n])).any())
    c = g["config"]
    cfg = O.OracleConfig(c["d_model"], c["nhead"], c["num_layers"], c["prefix_mode"], c["num_quantizers"])
    sd = {k: v.detach() for k, v in postln_model(c, g["weight_seed"]).state_dict().items()}
    with torch.no_grad(), P.post_ln():
        exact = P.nar_logits_forced(sd, cfg, g["x"], g["y"], g["codes"].long())
        with P.bf16_gemm_operands():
            rounded = P.nar_logits_forced(sd, cfg, g["x"], g["y"], g["codes"].long())
    emul = max(float((a - b).abs().max() / b.std()) for a, b in zip(rounded, exact))
    bar = max(NAR_TOL_REL, EMUL_FACTOR * emul)
    for i in range(7):
        e = (nar16[i] - nar32[i]).abs().amax(dim=1)
        assert float(e.max()) < bar * float(nar32[i].std()), (i, float(e.max()) / float(nar32[i].std()), bar)
        f = arg16[i] != ref[:, i + 1]
        assert not bool((f & (g["nar_margin"][i] > 2 * e)).any()), i


def test_bf16_codes_identical_across_reruns_graphs_and_the_cuda_core_path():
    g = load_golden("big_short_postln.pt")
    m = _model(g, torch.bfloat16)
    eng = m.engine()
    x, y = g["x"][0], g["y"][0]
    a = eng.generate([x, x[:4]], [y, y[:20]], top_k=1, max_new_tokens=48)
    b = eng.generate([x, x[:4]], [y, y[:20]], top_k=1, max_new_tokens=48)
    assert all(torch.equal(p, q) for p, q in zip(a, b))
    eng.use_cuda_graph = False
    c = eng.generate([x, x[:4]], [y, y[:20]], top_k=1, max_new_tokens=48)
    eng.use_cuda_graph = True
    assert all(torch.equal(p, q) for p, q in zip(a, c))
    tr_tc, tr_simt = {"steps": "all"}, {"steps": "all"}
    eng.generate([x], [y], top_k=1, trace=tr_tc, forced=[a[0]])
    from valle_b200 import _lib as L
    lib = L.load()
    L.check(lib.vb_tune_set(b"VB_DECODE_SIMT", 1))
    try:
        eng.generate([x], [y], top_k=1, trace=tr_simt, forced=[a[0]])
    finally:
        L.check(lib.vb_tune_set(b"VB_DECODE_SIMT", 0))
    err = max(float((tr_tc["ar_logits"][k] - tr_simt["ar_logits"][k]).abs().max()) for k in tr_tc["ar_logits"])
    assert err < AR_TOL, err


def test_bf16_decode_step_launches_equal_the_unfolded_pre_ln_chain():
    from valle_b200.models import VALLE

    def per_step(norm_first):
        torch.manual_seed(0)
        m = VALLE(1024, 16, 4, norm_first=norm_first, prefix_mode=1, num_quantizers=8).eval().to(DEV)
        eng = m.engine(torch.bfloat16)
        eng.quiet = True
        eng.generate([torch.arange(3, 9)], [torch.randint(0, 1024, (12, 8))], top_k=1, max_new_tokens=20)
        counts = {k[-1]: n for buf in eng._bufs.values() for k, (_, n, _) in buf.graphs.items()}
        assert 8 in counts, counts
        return counts[8] / 8

    old = os.environ.get("VB_DECODE_FOLD")
    os.environ["VB_DECODE_FOLD"] = "0"
    try:
        pre = per_step(True)
    finally:
        if old is None:
            del os.environ["VB_DECODE_FOLD"]
        else:
            os.environ["VB_DECODE_FOLD"] = old
    post = per_step(False)
    assert post == pre, (post, pre)


# ---------------------------------------------------------------- module surface
@pytest.mark.parametrize("adaptive", [False, True])
def test_post_ln_transformer_encoder_matches_the_oracle(adaptive):
    from valle_b200.modules.transformer import (AdaptiveLayerNorm, LayerNorm, TransformerEncoder,
                                                TransformerEncoderLayer)
    torch.manual_seed(2)
    d, H, nl, B, Lq = 256, 4, 2, 3, 20
    norm = AdaptiveLayerNorm(d, torch.nn.LayerNorm(d)) if adaptive else LayerNorm(d)
    enc = TransformerEncoder(TransformerEncoderLayer(d, H, dim_feedforward=4 * d, batch_first=True, norm_first=False,
                                                     adaptive_layer_norm=adaptive), num_layers=nl, norm=norm)
    for q in enc.parameters():
        if q.dim() == 1:
            q.data.add_(torch.randn_like(q) * 0.05)
    enc = enc.eval().to(DEV)
    sd = {"enc." + k: v.detach().cpu() for k, v in enc.state_dict().items()}
    sd_nonorm = {k: v for k, v in sd.items() if not k.startswith("enc.norm.")}
    cfg = O.OracleConfig(d, H, nl, 1, 8)
    x = torch.randn(B, Lq, d)
    emb = torch.randn(1, d) if adaptive else None
    src = (x.to(DEV), emb.to(DEV)) if adaptive else x.to(DEV)
    lens = torch.tensor([20, 13, 7])
    kpm = torch.arange(Lq)[None, :] >= lens[:, None]
    dense = torch.rand(Lq, Lq) < 0.3
    dense.fill_diagonal_(False)
    for mask, kp in ((None, kpm), (dense, None)):
        with torch.no_grad():
            states, out = enc(src, mask=None if mask is None else mask.to(DEV),
                              src_key_padding_mask=None if kp is None else kp.to(DEV), return_layer_states=True)
            whole = enc(src, mask=None if mask is None else mask.to(DEV),
                        src_key_padding_mask=None if kp is None else kp.to(DEV))
        out = out[0] if adaptive else out
        whole = whole[0] if adaptive else whole
        ref = P.encoder_postln(sd, "enc", x, cfg, blocked=mask, key_padding=kp, stage_emb=emb)
        valid = ~kp if kp is not None else torch.ones(B, Lq, dtype=torch.bool)
        assert _rel(out.cpu()[valid], ref[valid]) < 2e-5
        assert _rel(whole.cpu()[valid], ref[valid]) < 2e-5
        one = P.encoder_postln(sd_nonorm, "enc", x, O.OracleConfig(d, H, 1, 1, 8), blocked=mask, key_padding=kp,
                               stage_emb=emb)
        assert _rel(states[0].cpu()[valid], one[valid]) < 2e-5


# ---------------------------------------------------------------- training
@pytest.mark.parametrize("stage", [0, 1, 2])
@pytest.mark.parametrize("dtype,tol", [(torch.float32, 1e-3), (torch.bfloat16, GRAD_TOL_BF16)])
def test_post_ln_gradients_match_autograd_of_the_oracle(stage, dtype, tol):
    """every parameter's gradient against torch.autograd of the oracle's post-LN forward_train (max-abs error relative to
    the gradient's max-abs); bf16: the pre-LN bar, or EMUL_FACTOR times the bf16-operand restatement's worst error"""
    g = load_golden("tiny_postln_pm1.pt")
    fw = g["forward"]
    c = g["config"]
    cfg = O.OracleConfig(c["d_model"], c["nhead"], c["num_layers"], c["prefix_mode"], c["num_quantizers"])

    def oracle_grads(rounded):
        sd = {k: v.detach().clone().requires_grad_() for k, v in postln_model(c, g["weight_seed"]).state_dict().items()}
        with P.bf16_gemm_operands() if rounded else contextlib.nullcontext():
            loss, _ = P.forward_train(sd, cfg, fw["x"], fw["x_lens"], fw["y"].long(), fw["y_lens"], int(fw["nar_stage"]),
                                      int(fw["prefix_len"]), train_stage=stage)
            loss.backward()
        return sd

    sd = oracle_grads(False)
    if dtype == torch.bfloat16:
        sr = oracle_grads(True)
        emul = max(_rel(sr[k].grad, v.grad) for k, v in sd.items() if v.grad is not None and float(v.grad.abs().max()) > 0)
        tol = max(tol, EMUL_FACTOR * emul)
    m = _no_dropout(_model(g, dtype).train())
    m.rng = random.Random(0)
    torch.manual_seed(int(fw["torch_seed"]))
    (_, _), loss, _ = m(fw["x"].to(DEV), fw["x_lens"], fw["y"].long().to(DEV), fw["y_lens"], train_stage=stage)
    loss.backward()
    by_ptr = {p.data_ptr(): n for n, p in m.named_parameters()}
    want = {}
    for k, v in m.state_dict().items():
        n = by_ptr[v.data_ptr()]
        want[n] = want.get(n, 0) + (sd[k].grad if sd[k].grad is not None else torch.zeros_like(sd[k]))
    checked = 0
    for n, p in m.named_parameters():
        if not p.requires_grad or float(want[n].abs().max()) == 0.0:
            continue
        assert p.grad is not None, n
        assert _rel(p.grad.float().cpu(), want[n]) < tol, (n, _rel(p.grad.float().cpu(), want[n]))
        checked += 1
    assert checked > 20


def test_post_ln_stack_with_dropout_matches_torch_given_the_same_masks():
    from valle_b200 import _lib as L
    from valle_b200 import autograd as AG
    from valle_b200.modules.transformer import TransformerEncoder, TransformerEncoderLayer
    torch.manual_seed(4)
    d, H, nl, N, Smax, Tmax, p, seed = 256, 4, 2, 3, 8, 40, 0.1, 123456789
    enc = TransformerEncoder(TransformerEncoderLayer(d, H, dim_feedforward=4 * d, dropout=p, batch_first=True,
                                                     norm_first=False), num_layers=nl, norm=None).to(DEV)
    for q in enc.parameters():
        if q.dim() == 1:
            q.data.add_(torch.randn_like(q) * 0.05)
    Lp = Smax + Tmax
    xl = torch.tensor([8, 5, 3], dtype=torch.int32, device=DEV)
    yl = torch.tensor([40, 29, 12], dtype=torch.int32, device=DEV)
    x0 = torch.randn(N, Lp, d, device=DEV)
    cu = (torch.arange(N + 1, dtype=torch.int32, device=DEV) * Lp).contiguous()
    params = AG.layer_params(enc)
    xa = x0.clone().reshape(N * Lp, d).requires_grad_()
    out = AG.DecoderStack.apply(xa, None, enc.native(torch.float32), (cu, N, Lp, L.VB_MASK_PADDED, xl, yl, Smax, p, seed),
                                *params)
    t = torch.arange(Lp, device=DEV)[None, :]
    key_ok = (t < xl[:, None]) | ((t >= Smax) & (t < Smax + yl[:, None]))
    w = torch.randn(N, Lp, d, device=DEV) * key_ok[..., None]
    (out.view(N, Lp, d) * w).sum().backward()
    got = [q.grad.clone() for q in params] + [xa.grad.clone()]
    for q in params:
        q.grad = None
    xr = x0.clone().requires_grad_()
    x, ks = xr, 1.0 / (1.0 - p)
    for l, lyr in enumerate(enc.layers):    # transformer.py:303-308 with the library's masks
        qkv = F.linear(x, lyr.self_attn.in_proj_weight, lyr.self_attn.in_proj_bias).view(N, Lp, 3, H, 64)
        q, k, v = (qkv[:, :, i].transpose(1, 2) for i in range(3))
        sc = ((q @ k.transpose(-1, -2)) * 0.125).masked_fill(~key_ok[:, None, None, :], float("-inf"))
        m0 = _keep_mask(seed, (l << 2) | 0, N * H * Lp * Lp, p).view(N, H, Lp, Lp).to(DEV)
        o = ((torch.softmax(sc, dim=-1) * m0 * ks) @ v).transpose(1, 2).reshape(N, Lp, d)
        o = F.linear(o, lyr.self_attn.out_proj.weight, lyr.self_attn.out_proj.bias)
        m1 = _keep_mask(seed, (l << 2) | 1, N * Lp * d, p).view(N, Lp, d).to(DEV)
        x = F.layer_norm(x + o * m1 * ks, (d,), lyr.norm1.weight, lyr.norm1.bias, 1e-5)
        f = F.relu(F.linear(x, lyr.linear1.weight, lyr.linear1.bias))
        m2 = _keep_mask(seed, (l << 2) | 2, N * Lp * f.shape[-1], p).view(N, Lp, -1).to(DEV)
        f = F.linear(f * m2 * ks, lyr.linear2.weight, lyr.linear2.bias)
        m3 = _keep_mask(seed, (l << 2) | 3, N * Lp * d, p).view(N, Lp, d).to(DEV)
        x = F.layer_norm(x + f * m3 * ks, (d,), lyr.norm2.weight, lyr.norm2.bias, 1e-5)
    (x * w).sum().backward()
    valid = key_ok[..., None].expand_as(x)
    assert _rel(out.view(N, Lp, d)[valid].detach(), x[valid].detach()) < 1e-3
    want = [q.grad for q in params] + [xr.grad.reshape(N * Lp, d)]
    for i, (a, b) in enumerate(zip(got, want)):
        if i == len(got) - 1:
            a, b = a.view(N, Lp, d)[valid], b.view(N, Lp, d)[valid]
        assert _rel(a, b) < 1e-3, (i, _rel(a, b))
