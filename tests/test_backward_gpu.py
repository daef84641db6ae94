"""Training backward (SURVEY 8f rank 2; valle/bin/trainer.py:674 `scaler.scale(loss).backward()`): the gradient kernels
behind the C ABI against torch.autograd -- operator by operator on the same inputs, then the whole VALLE.forward loss
against the oracle (the reference's forward restated in plain torch, differentiated by torch on the host)."""
import ctypes as C
import random

import pytest
import torch
import torch.nn.functional as F

from conftest import assert_checksums, build_model, load_golden
from oracle import valle_oracle as O
from stack_oracle64 import keep_mask as _keep_mask

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _rel(a, b):
    return float((a - b).abs().max() / b.abs().max().clamp(min=1e-12))


def _s():
    return torch.cuda.current_stream().cuda_stream


def _no_dropout(m):
    """train() mode with every Dropout site at p = 0 (comparisons against the dropout-free oracle)"""
    for mod in m.modules():
        if isinstance(mod, torch.nn.Dropout):
            mod.p = 0.0
    return m


@pytest.mark.parametrize("dtype,tol", [(torch.float32, 2e-5), (torch.bfloat16, 2e-2)])
def test_linear_backward_vs_autograd(dtype, tol):
    from valle_b200 import _lib as L
    lib = L.load()
    torch.manual_seed(0)
    M, N, K = 333, 3072, 1024
    x = (torch.randn(M, K) * 0.5).to(dtype)
    w = (torch.randn(N, K) / 32).to(dtype)
    dy = (torch.randn(M, N) * 0.1).to(dtype)
    xr, wr = x.float().requires_grad_(), w.float().requires_grad_()
    b = torch.zeros(N, requires_grad=True)
    (F.linear(xr, wr, b) * dy.float()).sum().backward()
    xd, dyd = x.to(DEV), dy.to(DEV)
    wt = w.t().contiguous().to(DEV)
    dx = torch.empty(M, K, device=DEV)
    dw = torch.zeros(N, K, device=DEV)
    db = torch.zeros(N, device=DEV)
    dt = L.VB_F32 if dtype == torch.float32 else L.VB_BF16
    nb = lib.vb_linear_backward_workspace(dt, M, N, K)
    ws = torch.empty(nb, dtype=torch.uint8, device=DEV)
    L.check(lib.vb_linear_backward(xd.data_ptr(), dt, K, wt.data_ptr(), dyd.data_ptr(), N, dx.data_ptr(), L.VB_F32, K,
                                   L.VB_EPI_NONE, dw.data_ptr(), db.data_ptr(), M, N, K, ws.data_ptr(), nb, _s()))
    assert _rel(dx.cpu(), xr.grad) < tol and _rel(dw.cpu(), wr.grad) < tol and _rel(db.cpu(), b.grad) < tol
    # accumulate semantics: a second call doubles dW / db
    L.check(lib.vb_linear_backward(xd.data_ptr(), dt, K, wt.data_ptr(), dyd.data_ptr(), N, 0, L.VB_F32, K,
                                   L.VB_EPI_NONE, dw.data_ptr(), db.data_ptr(), M, N, K, ws.data_ptr(), nb, _s()))
    assert _rel(dw.cpu(), 2 * wr.grad) < tol and _rel(db.cpu(), 2 * b.grad) < tol


@pytest.mark.parametrize("adaptive", [False, True])
def test_layernorm_backward_vs_autograd(adaptive):
    from valle_b200 import _lib as L
    lib = L.load()
    torch.manual_seed(1)
    M, d = 301, 1024
    x = (torch.randn(M, d) * 2 + 0.3).requires_grad_()
    g = (torch.randn(d) * 0.2 + 1).requires_grad_()
    b = (torch.randn(d) * 0.2).requires_grad_()
    wb = (torch.randn(2 * d) * 0.3 + 0.5).requires_grad_() if adaptive else None
    rows = torch.randperm(M)[:200].to(torch.int32)
    dy = torch.randn(200, d)
    y = F.layer_norm(x[rows.long()], (d,), g, b, 1e-5)
    if adaptive:
        y = wb[:d] * y + wb[d:]
    (y * dy).sum().backward()
    dx = torch.full((M, d), 0.25, device=DEV)                    # accumulate semantics: dx += ...
    dg, db_, dwb = torch.zeros(d, device=DEV), torch.zeros(d, device=DEV), torch.zeros(2 * d, device=DEV)
    # (device copies are kept in variables: a temporary's memory may be reused before the kernel runs)
    xd, rd, gd, bd, dyd = x.detach().to(DEV), rows.to(DEV), g.detach().to(DEV), b.detach().to(DEV), dy.to(DEV)
    wbd = wb.detach().to(DEV) if adaptive else None
    L.check(lib.vb_layernorm_backward(xd.data_ptr(), d, rd.data_ptr(), 200, d, gd.data_ptr(), bd.data_ptr(),
                                      wbd.data_ptr() if adaptive else 0, 1e-5, dyd.data_ptr(), d, dx.data_ptr(), d, 0,
                                      L.VB_F32, dg.data_ptr(), db_.data_ptr(), dwb.data_ptr() if adaptive else 0, _s()))
    torch.cuda.synchronize()
    assert _rel(dx.cpu() - 0.25, x.grad) < 2e-5
    assert _rel(dg.cpu(), g.grad) < 2e-5 and _rel(db_.cpu(), b.grad) < 2e-5
    if adaptive:
        assert _rel(dwb.cpu(), wb.grad) < 2e-5


@pytest.mark.parametrize("mode", ["full", "valle_ar", "padded_ar", "padded"])
@pytest.mark.parametrize("dtype,tol", [(torch.float32, 3e-5), (torch.bfloat16, 3e-2)])
def test_attention_backward_vs_autograd(mode, dtype, tol):
    from valle_b200 import _lib as L
    lib = L.load()
    torch.manual_seed(2)
    H, d = 4, 256
    if mode in ("padded_ar", "padded"):
        B, Lp, seg1_start = 3, 150, 40
        lens, S, A = [Lp] * B, [40, 22, 9], [110, 75, 31]
    else:
        lens, S, A, seg1_start = [70, 5, 129, 200], [9, 2, 64, 30], None, 0
        B = len(lens)
    M = sum(lens)
    qkv = (torch.randn(M, 3 * d) * 0.7).to(dtype)
    dout = (torch.randn(M, d) * 0.3).to(dtype)
    cu = torch.tensor([0] + list(torch.tensor(lens).cumsum(0)), dtype=torch.int32)
    mm = {"full": L.VB_MASK_FULL, "valle_ar": L.VB_MASK_VALLE_AR, "padded_ar": L.VB_MASK_PADDED_AR, "padded": L.VB_MASK_PADDED}[mode]
    tl = torch.tensor(S, dtype=torch.int32) if mode != "full" else None
    sl = torch.tensor(A, dtype=torch.int32) if A is not None else None
    # torch reference per sequence
    ref_d = torch.zeros(M, 3 * d)
    ref_o = torch.zeros(M, d)
    for b in range(B):
        r0, n = int(cu[b]), lens[b]
        blk = qkv[r0:r0 + n].float().clone().requires_grad_()
        q, k, v = blk[:, :d], blk[:, d:2 * d], blk[:, 2 * d:]
        qh, kh, vh = (t.reshape(n, H, 64).transpose(0, 1) for t in (q, k, v))
        sc = qh @ kh.transpose(-1, -2) * 0.125
        rows, cols = torch.arange(n)[:, None], torch.arange(n)[None, :]
        if mode == "valle_ar":
            ok = cols < torch.clamp(rows + 1, min=S[b])
        elif mode == "padded_ar":
            ok = (cols < S[b]) | ((rows >= seg1_start) & (cols >= seg1_start) & (cols < seg1_start + A[b]) & (cols <= rows))
            ok = ok | ((rows >= seg1_start + A[b]) & (cols >= seg1_start) & (cols < seg1_start + A[b]))
        elif mode == "padded":
            ok = ((cols < S[b]) | ((cols >= seg1_start) & (cols < seg1_start + A[b]))).expand(n, n)
        else:
            ok = torch.ones(n, n, dtype=torch.bool)
        sc = sc.masked_fill(~ok, float("-inf"))
        o = (torch.softmax(sc, -1) @ vh).transpose(0, 1).reshape(n, d)
        (o * dout[r0:r0 + n].float()).sum().backward()
        ref_d[r0:r0 + n] = blk.grad
        ref_o[r0:r0 + n] = o.detach()
    from valle_b200 import ops
    qd, cud, doutd = qkv.to(DEV), cu.to(DEV), dout.to(DEV)
    tld = tl.to(DEV) if tl is not None else None
    sld = sl.to(DEV) if sl is not None else None
    out = ops.attention(qd, cud, max(lens), H, mm, tld, seg1_lens=sld, seg1_start=seg1_start)
    assert _rel(out.float().cpu(), ref_o) < (3e-5 if dtype == torch.float32 else 2e-2)
    dq = torch.empty_like(qd)
    nb = lib.vb_attention_backward_workspace(M, H)
    ws = torch.empty(nb, dtype=torch.uint8, device=DEV)
    dt = L.VB_F32 if dtype == torch.float32 else L.VB_BF16
    L.check(lib.vb_attention_backward(qd.data_ptr(), out.data_ptr(), doutd.data_ptr(), dt, M, B, H, 64,
                                      cud.data_ptr(), tld.data_ptr() if tld is not None else 0,
                                      sld.data_ptr() if sld is not None else 0, seg1_start, max(lens), mm,
                                      dq.data_ptr(), ws.data_ptr(), nb, _s()))
    torch.cuda.synchronize()
    assert _rel(dq.float().cpu(), ref_d) < tol, _rel(dq.float().cpu(), ref_d)


def test_cross_entropy_and_embedding_backward_vs_autograd():
    from valle_b200 import autograd as AG
    torch.manual_seed(3)
    n, V = 77, 1025
    lg = (torch.randn(n, V) * 2).requires_grad_()
    tg = torch.randint(0, V, (n,))
    tg[::7] = 1024
    F.cross_entropy(lg, tg, ignore_index=1024, reduction="sum").mul(0.5).backward()
    l2 = lg.detach().to(DEV).requires_grad_()
    AG.CrossEntropySum.apply(l2, tg.to(DEV), 1024).mul(0.5).backward()
    assert _rel(l2.grad.cpu(), lg.grad) < 1e-5
    tabs = [torch.randn(1024, 256, requires_grad=True) for _ in range(3)]
    tok = torch.randint(0, 1024, (50, 3))
    ref = sum(t[tok[:, j]] for j, t in enumerate(tabs))
    dy = torch.randn(50, 256)
    (ref * dy).sum().backward()
    tabs_d = [t.detach().to(DEV).requires_grad_() for t in tabs]
    out = AG.EmbedSum.apply(tok.to(DEV), 3, 1, 50, *tabs_d)
    (out * dy.to(DEV)).sum().backward()
    for a, b in zip(tabs_d, tabs):
        assert _rel(a.grad.cpu(), b.grad) < 1e-5


def _oracle_grads(g, stage, nar_stage, prefix_len):
    m = build_model(g["config"], g["weight_seed"])
    sd = {k: v.detach().clone().requires_grad_() for k, v in m.state_dict().items()}
    c = g["config"]
    cfg = O.OracleConfig(c["d_model"], c["nhead"], c["num_layers"], c["prefix_mode"], c["num_quantizers"])
    fw = g["forward"]
    loss, _ = O.forward_train(sd, cfg, fw["x"], fw["x_lens"], fw["y"].long(), fw["y_lens"], nar_stage, prefix_len,
                              train_stage=stage)
    loss.backward()          # (forward_train already halves the stage-0 loss, valle.py:956-957)
    grads = {k: (v.grad if v.grad is not None else torch.zeros_like(v)) for k, v in sd.items()}
    return float(loss), grads


@pytest.mark.parametrize("stage", [0, 1, 2])
@pytest.mark.parametrize("dtype,tol", [(torch.float32, 1e-3), (torch.bfloat16, 6e-2)])
def test_valle_forward_backward_matches_reference_autograd(stage, dtype, tol):
    """BASELINE configs[0] training batch (3 padded utterances, 32 phonemes, 128 x 8 codec tokens): loss.backward()
    through VALLE.forward in train() mode; every parameter gradient against torch.autograd of the oracle's forward
    (max-abs error relative to the gradient's max-abs: fp32 1e-3, bf16 6e-2); tied weights receive the sum."""
    g = load_golden("config0.pt")
    fw = g["forward"]
    ref_loss, ref = _oracle_grads(g, stage, int(fw["nar_stage"]), int(fw["prefix_len"]))
    m = build_model(g["config"], g["weight_seed"])
    assert_checksums(m, g["checksums"])
    m = _no_dropout(m.to(DEV).train())     # the oracle differentiates the evaluation-mode forward
    m.engine_dtype = dtype
    m.rng = random.Random(0)
    torch.manual_seed(int(fw["torch_seed"]))
    (_, codes), loss, metrics = m(fw["x"].to(DEV), fw["x_lens"], fw["y"].long().to(DEV), fw["y_lens"], train_stage=stage)
    assert loss.requires_grad
    assert abs(float(loss) - ref_loss) <= (1e-4 if dtype == torch.float32 else 2e-2) * abs(ref_loss)
    loss.backward()
    names = dict(m.named_parameters())
    sd_keys = list(m.state_dict().keys())
    alias = {}                                             # state_dict key -> parameter name (tied weights)
    by_ptr = {p.data_ptr(): n for n, p in names.items()}
    for k, v in m.state_dict().items():
        alias[k] = by_ptr[v.data_ptr()]
    want = {}
    for k in sd_keys:
        want[alias[k]] = want.get(alias[k], 0) + ref[k]
    worst = ("", 0.0)
    checked = 0
    for n, p in names.items():
        if not p.requires_grad:          # e.g. the NAR positional alphas (alpha=False): frozen in the reference too
            assert p.grad is None
            continue
        gref = want[n]
        if float(gref.abs().max()) == 0.0:
            assert p.grad is None or float(p.grad.abs().max()) < 1e-6, n
            continue
        assert p.grad is not None, f"no gradient for {n}"
        e = _rel(p.grad.float().cpu(), gref)
        checked += 1
        if e > worst[1]:
            worst = (n, e)
    assert checked > 20
    assert worst[1] < tol, worst


def test_optimizer_step_changes_the_next_forward():
    """one SGD step on the gradients lowers the loss of the same batch (the engine re-packs changed parameters)"""
    g = load_golden("config0.pt")
    fw = g["forward"]
    m = _no_dropout(build_model(g["config"], g["weight_seed"]).to(DEV).train())
    opt = torch.optim.SGD(m.parameters(), lr=2e-6)   # sum-reduced loss over ~800 target positions: large gradients
    losses = []
    for _ in range(3):
        m.rng = random.Random(0)
        torch.manual_seed(int(fw["torch_seed"]))
        (_, _), loss, _ = m(fw["x"].to(DEV), fw["x_lens"], fw["y"].long().to(DEV), fw["y_lens"], train_stage=0)
        opt.zero_grad()
        loss.backward()
        opt.step()
        losses.append(float(loss))
    assert losses[2] < losses[1] < losses[0], losses


# ---------------------------------------------------------------- training-mode dropout
def test_dropout_mask_is_the_documented_hash_and_its_own_backward():
    """vb_dropout: survivors scaled by 1 / (1 - p), mask = the splitmix hash of (seed, stream, index) restated in
    numpy above, keep rate within 0.5 % of 1 - p, another stream gives another mask, backward = same mask on dy"""
    from valle_b200 import autograd as AG
    torch.manual_seed(0)
    n, p, seed = 1 << 20, 0.1, 0x1234567890ABCDEF % (1 << 62)
    x = (torch.randn(n, device=DEV) + 3.0).requires_grad_()
    y = AG.Dropout.apply(x, p, seed, 7)
    keep = _keep_mask(seed, 7, n, p).to(DEV)
    assert torch.equal(y != 0, keep)
    assert torch.allclose(y[keep], x.detach()[keep] / (1 - p), rtol=1e-6)
    assert abs(float(keep.float().mean()) - (1 - p)) < 5e-3
    assert not torch.equal(AG.Dropout.apply(x.detach(), p, seed, 8) != 0, keep)
    y.sum().backward()
    assert torch.allclose(x.grad, keep.float() / (1 - p), rtol=1e-6)
    xb = x.detach().bfloat16()
    yb = AG.Dropout.apply(xb, p, seed, 7)
    assert torch.equal(yb != 0, keep)


def _torch_stack_with_masks(x, layers, key_ok, p, seed, H):
    """pre-LN TransformerEncoderLayer stack (transformer.py:296-334) in plain torch with the dropout masks of the
    library's hash: x [N, L, d]; key_ok [N, L] bool (keys a row may attend to: the VB_MASK_PADDED rule)."""
    N, Lq, d = x.shape
    keep_scale = 1.0 / (1.0 - p)
    for l, P in enumerate(layers):
        h = F.layer_norm(x, (d,), P["n1w"], P["n1b"], 1e-5)
        qkv = F.linear(h, P["wi"], P["bi"]).view(N, Lq, 3, H, 64)
        q, k, v = (qkv[:, :, i].transpose(1, 2) for i in range(3))              # [N, H, L, 64]
        sc = (q @ k.transpose(-1, -2)) * 0.125
        sc = sc.masked_fill(~key_ok[:, None, None, :], float("-inf"))
        pr = torch.softmax(sc, dim=-1)
        m0 = _keep_mask(seed, (l << 2) | 0, N * H * Lq * Lq, p).view(N, H, Lq, Lq).to(x.device)
        o = ((pr * m0 * keep_scale) @ v).transpose(1, 2).reshape(N, Lq, d)
        o = F.linear(o, P["wo"], P["bo"])
        m1 = _keep_mask(seed, (l << 2) | 1, N * Lq * d, p).view(N, Lq, d).to(x.device)
        x = x + o * m1 * keep_scale
        h = F.layer_norm(x, (d,), P["n2w"], P["n2b"], 1e-5)
        f = F.relu(F.linear(h, P["w1"], P["b1"]))
        m2 = _keep_mask(seed, (l << 2) | 2, N * Lq * f.shape[-1], p).view(N, Lq, -1).to(x.device)
        f = F.linear(f * m2 * keep_scale, P["w2"], P["b2"])
        m3 = _keep_mask(seed, (l << 2) | 3, N * Lq * d, p).view(N, Lq, d).to(x.device)
        x = x + f * m3 * keep_scale
    return x


def test_decoder_stack_with_dropout_matches_torch_given_the_same_masks():
    """vb_decoder_forward_train / vb_decoder_backward with dropout_p = 0.1 (attention probabilities, both sub-layer
    outputs, FFN hidden) against the same layers in plain torch fed the masks of the documented hash: output and every
    gradient within 1e-3 (fp32); the padded-batch key rule of the NAR training pass."""
    from valle_b200 import _lib as L
    from valle_b200 import autograd as AG
    from valle_b200.modules.transformer import LayerNorm, TransformerEncoder, TransformerEncoderLayer
    torch.manual_seed(4)
    d, H, nl, N, Smax, Tmax, p, seed = 256, 4, 2, 3, 8, 40, 0.1, 987654321
    enc = TransformerEncoder(TransformerEncoderLayer(d, H, dim_feedforward=4 * d, dropout=p, batch_first=True,
                                                     norm_first=True), num_layers=nl, norm=LayerNorm(d)).to(DEV)
    for q in enc.parameters():          # non-trivial biases / norm weights
        if q.dim() == 1:
            q.data.add_(torch.randn_like(q) * 0.05)
    Lp = Smax + Tmax
    xl = torch.tensor([8, 5, 3], dtype=torch.int32, device=DEV)
    yl = torch.tensor([40, 29, 12], dtype=torch.int32, device=DEV)
    x0 = torch.randn(N, Lp, d, device=DEV)
    cu = (torch.arange(N + 1, dtype=torch.int32, device=DEV) * Lp).contiguous()
    nd = enc.native(torch.float32)
    params = AG.layer_params(enc)
    xa = x0.clone().reshape(N * Lp, d).requires_grad_()
    out = AG.DecoderStack.apply(xa, None, nd, (cu, N, Lp, L.VB_MASK_PADDED, xl, yl, Smax, p, seed), *params)
    t = torch.arange(Lp, device=DEV)[None, :]
    key_ok = (t < xl[:, None]) | ((t >= Smax) & (t < Smax + yl[:, None]))
    w = torch.randn(N, Lp, d, device=DEV) * key_ok[..., None]              # padded rows carry no loss
    (out.view(N, Lp, d) * w).sum().backward()
    got = [q.grad.clone() for q in params] + [xa.grad.clone()]
    for q in params:
        q.grad = None
    layers = []
    for lyr in enc.layers:
        layers.append(dict(wi=lyr.self_attn.in_proj_weight, bi=lyr.self_attn.in_proj_bias, wo=lyr.self_attn.out_proj.weight,
                           bo=lyr.self_attn.out_proj.bias, w1=lyr.linear1.weight, b1=lyr.linear1.bias, w2=lyr.linear2.weight,
                           b2=lyr.linear2.bias, n1w=lyr.norm1.weight, n1b=lyr.norm1.bias, n2w=lyr.norm2.weight,
                           n2b=lyr.norm2.bias))
    xr = x0.clone().requires_grad_()
    ref = _torch_stack_with_masks(xr, layers, key_ok, p, seed, H)
    (ref * w).sum().backward()
    valid = key_ok[..., None].expand_as(ref)
    assert _rel(out.view(N, Lp, d)[valid].detach(), ref[valid].detach()) < 1e-3
    want = [q.grad for q in params] + [xr.grad.reshape(N * Lp, d)]
    for i, (a, b) in enumerate(zip(got, want)):
        if i == len(got) - 1:             # input gradient: valid rows only (padded rows see only masked keys)
            a, b = a.view(N, Lp, d)[valid], b.view(N, Lp, d)[valid]
        assert _rel(a, b) < 1e-3, (i, _rel(a, b))
    # dropout really happened: the p = 0 result differs
    out0 = AG.DecoderStack.apply(x0.clone().reshape(N * Lp, d), None, nd, (cu, N, Lp, L.VB_MASK_PADDED, xl, yl, Smax), *params)
    assert _rel(out0.view(N, Lp, d)[valid].detach(), ref[valid].detach()) > 1e-2


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_training_mode_applies_dropout_reproducibly(dtype):
    """model.train() with the reference's default rates (0.1): the loss differs from the evaluation loss, repeats
    under the same torch.manual_seed (the mask seed comes from the device generator), changes with another seed, and
    loss.backward() yields finite gradients for every trainable parameter."""
    g = load_golden("config0.pt")
    fw = g["forward"]
    m = build_model(g["config"], g["weight_seed"]).to(DEV)
    m.engine_dtype = dtype
    args = (fw["x"].to(DEV), fw["x_lens"], fw["y"].long().to(DEV), fw["y_lens"])

    def run(seed, train=True):
        m.train(train)
        m.rng = random.Random(0)
        torch.manual_seed(seed)
        return m(*args, train_stage=0)[1]

    with torch.no_grad():
        le = float(run(5, train=False))
    l1 = run(5)
    l2 = float(run(5))
    l3 = float(run(6))
    assert float(l1) == l2 and l2 != l3
    assert abs(float(l1) - le) > 1e-3 * abs(le) and abs(float(l1) - le) < 0.5 * abs(le)
    for q in m.parameters():
        q.grad = None
    l1.backward()
    with_grad = 0
    for n, q in m.named_parameters():      # (only the NAR stage drawn for this call trains its head / stage embedding)
        if q.grad is not None:
            assert torch.isfinite(q.grad).all(), n
            with_grad += 1
    assert with_grad > 60
