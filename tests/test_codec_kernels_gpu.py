"""The EnCodec kernels of `csrc/encodec.cu`, one C entry point at a time, against the float64 restatements of
`tests/codec_oracle64.py`; then the engine's encoder / decoder layer by layer and end to end at the benchmark shape
(32 x 10 s) against HF's `EncodecModel` cast to float64.  The float64 references run on the GPU (plain float64 torch).
The fp32 yardsticks run on the CPU for the LSTM and on the GPU with TF32 off for whole HF stacks.

Error model (u = 2^-24, fp32 round-off):
* `vb_conv1d`: an output is bias + an FMA chain of n = Cin K terms w act(x) (+ residual).  With s = sum |w act(x)| +
  |bias| + |residual| (`codec_oracle64.conv1d`), a random-walk bound on the chain is 4 sqrt(n) u s, the ELU's
  `expm1f` adds 2 u s and the bias / residual adds 2 u |y|:  E = u (2 |y| + (4 sqrt(n) + 2) s).  Every element must
  be within E.  A dropped tap or input channel of a typical element moves it by s / n, which exceeds E for every
  n <= 8192 the sweep runs (asserted per case on the median element).
* `vb_lstm_layer`: the recurrence is not a single chain, so its bar is measured: every h_t must be within 4 x the
  error of an fp32 CPU restatement of the same recurrence (largest over the batch and units, running maximum over t)
  and never below 1e-6.  At T = 1 (h_prev = 0) the kernel is two sigmoids, two tanh and three products of the
  inputs: within 8 ulp.
* `vb_rvq_encode`: distances -(|r|^2 - 2 r.e + |e|^2) of code e carry u ((4 sqrt(dim) + 2) (2 sum |r e| + |e|^2) +
  2 (|r|^2 + 2 |r.e| + |e|^2)) (|r|^2 is shared by all codes, so its own chain cancels in the comparison), plus
  2 sum |r - e| D for the fp32 residual, D = u sum over the earlier stages of |residual|.  Two codes are tied when
  their float64 distances differ by less than the sum of their bounds (the band tau).  Checked teacher-forced: stage
  q's residual is rebuilt in float64 from the kernel's own picks of stages < q; each pick must be the float64 argmax
  where that is outside tau, and one of the tied codes inside it.  Exactly equal codebook rows must give the lowest.
* `vb_permute3`: bit for bit.

Each test prints its worst err / bar (pytest -s).
"""
import math

import pytest
import torch

import codec_oracle64 as C64
from oracle import encodec_oracle as E

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
F64 = torch.float64
GUARD = 4096                  # sentinel elements on each side of an output
SENT = -7777.0


def _L():
    from valle_b200 import _lib as L
    return L


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _guarded(n, dtype=torch.float32, fill=SENT):
    buf = torch.full((n + 2 * GUARD,), fill, dtype=dtype, device="cuda")
    return buf, buf[GUARD:GUARD + n]


def _guards_intact(buf, fill=SENT):
    return bool((buf[:GUARD] == fill).all()) and bool((buf[-GUARD:] == fill).all())


# ---------------------------------------------------------------------------------------------------------------
# vb_conv1d
# ---------------------------------------------------------------------------------------------------------------
def _t_in(t_out, K, stride, dil, pl, pr):
    return (t_out - 1) * stride + (K - 1) * dil + 1 - pl - pr


# (B, Cin, Tin, Cout, K, stride, dil, pad_left, pad_right, reflect, pre_elu, residual, bias, phase).  CO_T = 16 / 32 / 64
# tiles serve Cout <= 16 / <= 32 / more with T_T = 1024 / 512 / 256 time steps per CTA; Tout sits at T_T - 1, T_T and
# T_T + 1 of each.  Cin 1, 7, 8, 9, 512 cover the 8-channel chunks and their partial tail.
CONV_CASES = [
    (1, 1, _t_in(1023, 7, 1, 1, 6, 0), 1, 7, 1, 1, 6, 0, True, False, False, True, 1),
    (3, 7, _t_in(1024, 3, 1, 2, 4, 0), 15, 3, 1, 2, 4, 0, True, True, True, True, 1),
    (1, 9, _t_in(1025, 8, 4, 1, 4, 3), 16, 8, 4, 1, 4, 3, True, True, False, True, 1),
    (3, 9, _t_in(511, 2, 2, 1, 0, 0), 17, 2, 2, 1, 0, 0, False, False, False, False, 1),
    (1, 512, 512, 32, 1, 1, 1, 0, 0, True, True, True, True, 1),
    (3, 8, _t_in(513, 4, 2, 1, 2, 1), 32, 4, 2, 1, 2, 1, True, True, False, True, 1),
    (3, 7, _t_in(255, 7, 1, 3, 18, 0), 33, 7, 1, 3, 18, 0, True, True, True, True, 1),
    (1, 8, _t_in(256, 10, 5, 1, 5, 2), 64, 10, 5, 1, 5, 2, True, True, False, True, 1),
    (3, 9, _t_in(257, 6, 3, 2, 5, 5), 65, 6, 3, 2, 5, 5, False, False, True, True, 1),
    (1, 512, _t_in(257, 16, 8, 1, 8, 0), 130, 16, 8, 1, 8, 0, True, True, False, True, 1),
    (3, 512, _t_in(256, 3, 1, 1, 2, 0), 512, 3, 1, 1, 2, 0, True, True, True, True, 1),
    (1, 512, _t_in(255, 16, 4, 1, 12, 0), 512, 16, 4, 1, 12, 0, True, True, False, True, 1),
    (32, 7, _t_in(100, 7, 6, 1, 1, 0), 65, 7, 6, 1, 1, 0, True, False, False, False, 1),
    (3, 1, _t_in(300, 6, 3, 1, 3, 0), 15, 6, 3, 1, 3, 0, True, True, True, True, 1),
    (3, 8, _t_in(255, 14, 7, 1, 7, 0), 33, 14, 7, 1, 7, 0, True, True, True, True, 1),
    (1, 9, _t_in(600, 3, 1, 3, 6, 0), 33, 3, 1, 3, 6, 0, False, True, True, False, 1),
    # transposed up-sampling convs: stride-1 two-tap convs onto C * phase channels, one zero on the left
    (3, 512, 255, 512, 2, 1, 1, 1, 0, False, True, False, True, 2),
    (1, 9, 1025, 16, 2, 1, 1, 1, 0, False, True, False, False, 4),
    (3, 8, 257, 65, 2, 1, 1, 1, 0, False, True, False, True, 5),
    (1, 7, 512, 32, 2, 1, 1, 1, 0, False, True, False, True, 8),
    (3, 7, 300, 64, 3, 1, 2, 4, 0, True, False, False, True, 8),
    # reflect pads at, above and below the input length (EnCodec zero-extends the input before reflecting)
    (3, 7, 7, 15, 7, 1, 1, 6, 0, True, True, True, True, 1),
    (3, 7, 6, 15, 7, 1, 1, 6, 0, True, True, True, True, 1),
    (1, 8, 5, 33, 7, 1, 1, 6, 0, True, False, False, True, 1),
    (3, 9, 1, 17, 7, 1, 1, 6, 0, True, True, True, True, 1),
    (1, 7, 3, 64, 16, 8, 1, 8, 7, True, True, False, True, 1),
    (3, 512, 2, 65, 3, 1, 1, 0, 5, True, False, True, True, 1),
    (1, 9, 1, 16, 7, 1, 1, 6, 0, False, True, False, True, 1),
    # the first encoder conv at the benchmark's 32 x 240,000 samples
    (32, 1, 240000, 32, 7, 1, 1, 6, 0, True, False, False, True, 1),
]


def conv_case_inputs(case, seed):
    B, Cin, Tin, Cout, K, stride, dil, pl, pr, reflect, pre_elu, res, bias, phase = case
    g = torch.Generator().manual_seed(seed)
    Tout = (Tin + pl + pr - (K - 1) * dil - 1) // stride + 1
    x = torch.randn(B, Cin, Tin, generator=g)
    bound = 1.0 / math.sqrt(Cin * K)
    w = (torch.rand(Cout, Cin, K, generator=g) * 2 - 1) * bound
    b = (torch.rand(Cout // phase, generator=g) * 2 - 1) * bound if bias else None
    r = torch.randn(B, Cout // phase, Tout * phase, generator=g) if res else None
    return [t.cuda() if t is not None else None for t in (x, w, b, r)] + [Tout]


def run_conv(case, x, w, b, r, Tout):
    """vb_conv1d on `case` into a sentinel-guarded buffer -> (out [B, Cout / phase, Tout * phase], guards intact)"""
    B, Cin, Tin, Cout, K, stride, dil, pl, pr, reflect, pre_elu, res, bias, phase = case
    L = _L()
    wp = w.permute(1, 2, 0).contiguous()
    n = B * Cout * Tout
    buf, out = _guarded(n)
    L.check(L.load().vb_conv1d(x.data_ptr(), B, Cin, Tin, wp.data_ptr(), L.ptr(b), Cout, K, stride, dil, pl, pr,
                               int(reflect), int(pre_elu), L.ptr(r), out.data_ptr(), Tout, phase, _stream()), "vb_conv1d")
    torch.cuda.synchronize()
    return out.view(B, Cout // phase, Tout * phase), _guards_intact(buf)


def conv_bar(y, s, n):
    return U * (2 * y.abs() + (4 * math.sqrt(n) + 2) * s)


@pytest.mark.parametrize("ci", range(len(CONV_CASES)))
def test_conv1d_against_float64(ci):
    case = CONV_CASES[ci]
    B, Cin, Tin, Cout, K, stride, dil, pl, pr, reflect, pre_elu, res, bias, phase = case
    x, w, b, r, Tout = conv_case_inputs(case, 100 + ci)
    out, intact = run_conv(case, x, w, b, r, Tout)
    assert intact, "vb_conv1d wrote outside [B, Cout, Tout]"
    y, s = C64.conv1d(x.double(), w.double(), None if b is None else b.double(), stride, dil, pl, pr, reflect, pre_elu,
                      None if r is None else r.double(), phase)
    n = Cin * K
    bar = conv_bar(y, s, n)
    ratio = float(((out.double() - y).abs() / bar).max())
    sens = float((s / n / bar).median())
    print(f"conv {case[:9]} reflect={reflect} phase={phase}: worst err/E {ratio:.3f}, median dropped-term/E {sens:.1f}")
    assert ratio <= 1.0, ratio
    assert sens > 1.0, sens


# ---------------------------------------------------------------------------------------------------------------
# vb_lstm_layer
# ---------------------------------------------------------------------------------------------------------------
LSTM_CASES = [(512, 1, 1), (512, 3, 2), (512, 4, 75), (512, 5, 750), (512, 32, 750), (512, 64, 75), (512, 65, 75),
              (512, 70, 2), (512, 1, 1500), (128, 1, 2), (128, 4, 1500), (128, 64, 750), (128, 3, 75), (128, 70, 1),
              (128, 5, 1)]


def lstm_inputs(H, B, T, seed):
    g = torch.Generator().manual_seed(seed)
    w_hh = (torch.rand(4 * H, H, generator=g) * 2 - 1) / math.sqrt(H)
    xproj = torch.randn(T, B, 4 * H, generator=g)
    return xproj, w_hh


def run_lstm(xproj, w_hh, stepwise=False):
    L = _L()
    lib = L.load()
    T, B, H4 = xproj.shape
    H = H4 // 4
    xd, whh_t = xproj.cuda(), w_hh.t().contiguous().cuda()
    buf, h = _guarded(T * B * H)
    c = torch.empty(B * H + 64, device="cuda")
    L.check(lib.vb_tune_set(b"VB_LSTM_STEPWISE", int(stepwise)))
    try:
        L.check(lib.vb_lstm_layer(xd.data_ptr(), whh_t.data_ptr(), T, B, H, h.data_ptr(), c.data_ptr(), _stream()),
                "vb_lstm_layer")
        torch.cuda.synchronize()
    finally:
        lib.vb_tune_set(b"VB_LSTM_STEPWISE", 0)
    assert _guards_intact(buf), "vb_lstm_layer wrote outside h_seq"
    return h.view(T, B, H).cpu()


def lstm_bar(err32):
    """per step: 4 x the running maximum of the fp32 restatement's error, at least 1e-6"""
    return torch.clamp(4 * torch.cummax(err32, 0).values, min=1e-6)


@pytest.mark.parametrize("H,B,T", LSTM_CASES)
def test_lstm_layer_against_float64(H, B, T):
    xproj, w_hh = lstm_inputs(H, B, T, 7 * H + B + T)
    h64 = C64.lstm_layer(xproj.double(), w_hh.double())
    h32 = C64.lstm_layer(xproj, w_hh)
    bar = lstm_bar((h32.double() - h64).abs().amax((1, 2)))
    for stepwise in ((False, True) if B <= 64 else (True,)):
        h = run_lstm(xproj, w_hh, stepwise)
        err = (h.double() - h64).abs()
        ratio = float((err.amax((1, 2)) / bar).max())
        print(f"lstm H={H} B={B} T={T} {'stepwise' if stepwise else 'persistent'}: worst err/bar {ratio:.3f}")
        assert ratio <= 1.0, ratio
        if T == 1:          # h_prev = 0: within 8 ulp of |h|
            assert bool((err <= 8 * 2.0 ** -23 * h64.abs()).all()), float((err / h64.abs()).max())


def test_lstm_persistent_reruns_are_bitwise_equal():
    """the grid barrier only orders the steps: two runs give the same bits at the benchmark's B=32, T=750"""
    xproj, w_hh = lstm_inputs(512, 32, 750, 11)
    assert torch.equal(run_lstm(xproj, w_hh), run_lstm(xproj, w_hh))


# ---------------------------------------------------------------------------------------------------------------
# vb_rvq_encode
# ---------------------------------------------------------------------------------------------------------------
def rvq_check(x, cbs, codes):
    """teacher-forced float64 check of the picks codes [n, n_q] of rows x [n, dim] over cbs [n_q, n_codes, dim] (fp32,
    any device) -> (worst tie-band use, fraction of picks outside the band).  See the module docstring."""
    dev = "cuda" if torch.cuda.is_available() else "cpu"
    x, cbs, codes = x.to(dev, F64), cbs.to(dev, F64), codes.to(dev)
    n, dim = x.shape
    _, _, res = C64.rvq_encode(x, cbs, picks=codes)
    drift = torch.zeros_like(x)
    worst, outside = 0.0, 0
    for q in range(cbs.shape[0]):
        r, e = res[q], cbs[q]
        if q > 0:
            drift += U * res[q].abs()
        d = C64.rvq_distances(r, e)
        dot = r @ e.t()
        ee = e.pow(2).sum(1)[None]
        xx = r.pow(2).sum(1, keepdim=True)
        bound = U * ((4 * math.sqrt(dim) + 2) * (2 * (r.abs() @ e.abs().t()) + ee) + 2 * (xx + 2 * dot.abs() + ee))
        bound += 2 * ((r.abs() * drift).sum(1, keepdim=True) + drift @ e.abs().t())
        best, jstar = d.max(1)
        slack = best[:, None] - d                                     # >= 0
        band = bound + bound.gather(1, jstar[:, None])
        tied = slack <= band
        pick = codes[:, q]
        assert bool(tied.gather(1, pick[:, None]).all()), f"stage {q}: a pick outside the tie band of the argmax"
        single = tied.sum(1) == 1
        assert bool((pick[single] == jstar[single]).all())
        outside += int(single.sum())
        other = slack.gather(1, pick[:, None])[:, 0] / band.gather(1, pick[:, None])[:, 0]
        worst = max(worst, float(other.max()))
    return worst, outside / (n * cbs.shape[0])


def rvq_inputs(n_rows, n_codes, dim, n_q, seed):
    """codebooks with a shrinking scale per stage and exactly duplicated rows (lo, hi); half the rows are sums of
    codewords plus noise (some of them built on the duplicated rows), half plain noise"""
    g = torch.Generator().manual_seed(seed)
    cbs = torch.stack([torch.randn(n_codes, dim, generator=g) * 0.8 ** q for q in range(n_q)])
    dups = sorted({(lo, hi) for lo, hi in ((0, 1), (3, 256 + 3), (224, 225), (230, 1000), (255, n_codes - 1))
                   if hi < n_codes and lo < hi})
    for lo, hi in dups:
        cbs[:, hi] = cbs[:, lo]
    picks = torch.randint(0, n_codes, (n_rows, n_q), generator=g)
    if dups:
        on_dup = torch.rand(n_rows, n_q, generator=g) < 0.2
        on_dup[:2, 0] = True
        los = torch.tensor([lo for lo, _ in dups])[torch.randint(0, len(dups), (n_rows, n_q), generator=g)]
        picks = torch.where(on_dup, los, picks)
    x = sum(cbs[q][picks[:, q]] for q in range(n_q)) + 0.05 * torch.randn(n_rows, dim, generator=g)
    x[n_rows // 2:] = torch.randn(n_rows - n_rows // 2, dim, generator=g) * 2
    return x.contiguous(), cbs.contiguous(), dups


def run_rvq(x, cbs, layout, B=1):
    """vb_rvq_encode into a sentinel-filled int64 buffer -> codes [n_rows, n_q].  layout "bnt": [B, n_q, T] with a gap
    of 3 after every utterance; "rows": one sequence (rows_per_seq = 0), [n_rows, n_q + 1]"""
    L = _L()
    n, dim = x.shape
    n_q, n_codes, _ = cbs.shape
    xd, cb = x.cuda(), cbs.cuda()
    cb_t = cb.transpose(1, 2).contiguous()
    cb_sq = cb.pow(2).sum(2).contiguous()
    if layout == "bnt":
        T = n // B
        row_s, q_s, per_seq, seq_s = 1, T, T, n_q * T + 3
        size = B * seq_s
    else:
        row_s, q_s, per_seq, seq_s = n_q + 1, 1, 0, 12345
        size = n * (n_q + 1)
    buf, codes = _guarded(size, torch.int64, -7)
    L.check(L.load().vb_rvq_encode(xd.data_ptr(), n, dim, n_q, n_codes, cb.data_ptr(), cb_t.data_ptr(), cb_sq.data_ptr(),
                                   codes.data_ptr(), row_s, q_s, per_seq, seq_s, _stream()), "vb_rvq_encode")
    torch.cuda.synchronize()
    assert _guards_intact(buf, -7)
    rows = torch.arange(n, device="cuda")
    if layout == "bnt":
        idx = (rows // T)[:, None] * seq_s + (rows % T)[:, None] * row_s + torch.arange(n_q, device="cuda")[None] * q_s
    else:
        idx = rows[:, None] * row_s + torch.arange(n_q, device="cuda")[None] * q_s
    written = torch.zeros(size, dtype=torch.bool, device="cuda")
    written[idx.reshape(-1)] = True
    assert bool((codes[~written] == -7).all()), "vb_rvq_encode wrote outside its code slots"
    return codes[idx]


# (n_rows, n_codes, dim, n_q, layout, B)
RVQ_CASES = [(1, 1024, 128, 8, "bnt", 1), (7, 255, 128, 8, "rows", 1), (8, 256, 512, 1, "bnt", 2),
             (9, 257, 1, 32, "rows", 1), (9, 1, 128, 8, "bnt", 3), (8, 1024, 512, 32, "rows", 1),
             (7, 257, 512, 8, "bnt", 7), (1, 255, 1, 1, "rows", 1), (24000, 1024, 128, 8, "bnt", 32),
             (24000, 257, 512, 1, "rows", 1), (9, 1024, 128, 32, "bnt", 3)]


@pytest.mark.parametrize("n_rows,n_codes,dim,n_q,layout,B", RVQ_CASES)
def test_rvq_encode_against_float64(n_rows, n_codes, dim, n_q, layout, B):
    x, cbs, dups = rvq_inputs(n_rows, n_codes, dim, n_q, n_rows + n_codes + dim + n_q)
    codes = run_rvq(x, cbs, layout, B)
    assert int(codes.min()) >= 0 and int(codes.max()) < n_codes
    worst, outside = rvq_check(x, cbs, codes)
    for lo, hi in dups:
        assert not bool((codes == hi).any()), f"picked code {hi}, an exact copy of code {lo}"
    if dups and n_rows >= 8 and dim >= 128:      # rows 0 and 1 are built on a duplicated stage-0 code
        assert bool(torch.isin(codes[:, 0], torch.tensor([lo for lo, _ in dups], device="cuda")).any())
    print(f"rvq n={n_rows} codes={n_codes} dim={dim} n_q={n_q} {layout}: worst pick slack / tau {worst:.3f}, "
          f"{outside:.4f} of the picks outside tau")
    if n_codes > 1 and n_rows >= 8:
        assert outside > 0.5, outside


# ---------------------------------------------------------------------------------------------------------------
# vb_permute3
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape", [(3, 5, 7), (1, 13, 1), (9, 1, 257), (32, 512, 750)])
def test_permute3_bitwise(shape):
    L = _L()
    x = torch.randn(shape, device="cuda")
    for p in ((0, 1, 2), (0, 2, 1), (1, 0, 2), (1, 2, 0), (2, 0, 1), (2, 1, 0)):
        ref = x.permute(*p).contiguous()
        buf, out = _guarded(x.numel())
        L.check(L.load().vb_permute3(x.data_ptr(), *shape, *p, out.data_ptr(), _stream()), "vb_permute3")
        torch.cuda.synchronize()
        assert _guards_intact(buf)
        assert torch.equal(out.view(ref.shape), ref), p


# ---------------------------------------------------------------------------------------------------------------
# the engine's stacks, layer by layer and end to end
# ---------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def codec():
    from valle_b200.data.tokenizer import AudioTokenizer
    m = E.build_codec(0)
    tok = AudioTokenizer(device="cuda:0", weights=m.state_dict())
    m64 = E.build_codec(0).double().cuda()
    m32 = E.build_codec(0).cuda()
    return m32, m64, tok.codec, tok


@pytest.fixture(scope="module")
def bench_wav():
    g = torch.Generator().manual_seed(21)
    return (torch.randn(32, 1, 240000, generator=g) * 0.1).clamp(-1, 1).cuda()


SUBSET = [0, 17, 31]


def _groups(layers):
    """HF stack -> the engine's items: an ELU goes with the layer after it"""
    out, pend = [], []
    for layer in layers:
        pend.append(layer)
        if not isinstance(layer, torch.nn.ELU):
            out.append(pend)
            pend = []
    return out


def _conv_w(mod):
    return mod.conv.weight.detach(), mod.conv.bias.detach()


def _layer_bar(kind, hf, x64):
    """per-element bar of one engine item on its (float64) input, from the restated convs"""
    from transformers.models.encodec.modeling_encodec import EncodecConvTranspose1d
    mod = hf[-1]
    pre = len(hf) == 2
    if kind in ("conv", "conv_elu"):
        w, b = _conv_w(mod)
        y, s = C64.sconv1d(x64, w, b, int(mod.stride), mod.conv.dilation[0], pre_elu=pre)
        return conv_bar(y, s, w.shape[1] * w.shape[2])
    if kind == "convt_elu":
        assert isinstance(mod, EncodecConvTranspose1d)
        w, b = _conv_w(mod)
        y, s = C64.conv_transpose_as_phases(x64, w, b, mod.conv.stride[0], pre_elu=True)
        return conv_bar(y, s, w.shape[0] * 2)
    # residual block: sc(x) + c2(elu(c1(elu(x)))); c1's error reaches the output through |w2| (ELU is 1-Lipschitz)
    c1, c2, sc = mod.block[1], mod.block[3], mod.shortcut
    w1, b1 = _conv_w(c1)
    w2, b2 = _conv_w(c2)
    ws, bs = _conv_w(sc)
    y1, s1 = C64.sconv1d(x64, w1, b1, 1, c1.conv.dilation[0], pre_elu=True)
    e1 = conv_bar(y1, s1, w1.shape[1] * w1.shape[2])
    ysc, ssc = C64.sconv1d(x64, ws, bs)
    esc = conv_bar(ysc, ssc, ws.shape[1])
    y2, s2 = C64.sconv1d(y1, w2, b2, pre_elu=True, residual=ysc)
    e2 = conv_bar(y2, s2, w2.shape[1])
    return e2 + C64.sconv1d(e1, w2.abs(), None)[0] + esc


def _lstm_yardstick(hf_lstm, x):
    """the module in fp32 on the CPU against float64 -> per-step error [T] of the fp32 run, for `lstm_bar`"""
    import copy
    m32 = copy.deepcopy(hf_lstm).float().cpu()
    m64 = copy.deepcopy(hf_lstm).double().cpu()
    with torch.no_grad():
        y32 = m32(x.float().cpu())
        y64 = m64(x.double().cpu())
    return (y32.double() - y64).abs().amax((0, 1)), y64


def _stack_layer_by_layer(items, hf_layers, x, name):
    worst = 0.0
    groups = _groups(hf_layers)
    assert len(groups) == len(items)
    for (kind, mod), hf in zip(items, groups):
        if kind in ("conv_elu", "convt_elu"):
            y = mod(x, pre_elu=True)
        else:
            y = mod(x)
        xs = x[SUBSET].double()
        if kind == "lstm":
            err32, ref = _lstm_yardstick(hf[-1], x[SUBSET])
            err = (y[SUBSET].double().cpu() - ref).abs().amax((0, 1))
            ratio = float((err / lstm_bar(err32)).max())
        else:
            with torch.no_grad():
                ref = xs
                for layer in hf:
                    ref = layer(ref)
            ratio = float(((y[SUBSET].double() - ref).abs() / _layer_bar(kind, hf, xs)).max())
        print(f"{name} {kind}: worst err/bar {ratio:.3f}")
        assert ratio <= 1.0, (name, kind, ratio)
        worst = max(worst, ratio)
        x = y
    return x, worst


def test_encoder_and_decoder_layer_by_layer_at_the_benchmark_shape(codec, bench_wav):
    """each engine layer on the engine's own input to it, against the HF layer in float64, for 3 of 32 10 s clips"""
    _, m64, nat, _ = codec
    emb, w_enc = _stack_layer_by_layer(nat.enc, m64.encoder.layers, bench_wav, "encoder")
    _, w_dec = _stack_layer_by_layer(nat.dec, m64.decoder.layers, emb.contiguous(), "decoder")
    print(f"layer by layer: worst err/bar encoder {w_enc:.3f}, decoder {w_dec:.3f}")


def _fp32_yardstick(run32, run64, x32, x64):
    """error of an HF stack run in fp32 (TF32 off) against its float64 run -> (largest error, float64 output)"""
    with torch.no_grad():
        prev = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
        torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
        try:
            y32 = run32(x32)
        finally:
            torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = prev
        y64 = run64(x64)
    return (y32.double() - y64).abs().amax(), y64


def _against_fp32_yardstick(out, ref, err32, what):
    """4 x the error of the same HF stack run in fp32 (TF32 off), at least 2^-20 of the output's scale"""
    bar = max(4 * float(err32), 2.0 ** -20 * float(ref.abs().max()))
    err = float((out.double() - ref).abs().max())
    print(f"{what}: err {err:.3g}, bar {bar:.3g}, err/bar {err / bar:.3f}")
    assert err <= bar, (what, err, bar)


def test_encode_end_to_end_at_the_benchmark_shape(codec, bench_wav):
    """32 x 10 s: every (frame, stage) code of the batch against the float64 pick on the engine's own embeddings
    (outside tau), and 3 utterances' embeddings against HF's float64 encoder"""
    m32, m64, nat, tok = codec
    (codes, _), = tok.encode(bench_wav)
    emb = nat._run(nat.enc, bench_wav)                                  # what encode() quantised
    B, D, T = emb.shape
    assert codes.shape == (32, 8, 750) and T == 750
    rows = emb.permute(0, 2, 1).reshape(-1, D)
    worst, outside = rvq_check(rows, nat.cb, codes.permute(0, 2, 1).reshape(-1, 8))
    print(f"end to end codes: worst pick slack / tau {worst:.3f}, {outside:.4f} of the picks outside tau")
    err32, ref = _fp32_yardstick(m32.encoder, m64.encoder, bench_wav[SUBSET], bench_wav[SUBSET].double())
    _against_fp32_yardstick(emb[SUBSET], ref, err32, "end to end embeddings")


@pytest.mark.parametrize("N", [1, 2, 6, 7, 319, 320, 321, 1000, 1920, 1921])
def test_encode_short_inputs(codec, N):
    """inputs shorter than the reflect pads of the first or last conv (N <= 1920) encode like EnCodec's pad1d"""
    m32, m64, nat, tok = codec
    g = torch.Generator().manual_seed(N)
    wav = (torch.randn(2, 1, N, generator=g) * 0.1).clamp(-1, 1).cuda()
    (codes, _), = tok.encode(wav)
    emb = nat._run(nat.enc, wav)
    assert codes.shape == (2, 8, -(-N // 320))
    rvq_check(emb.permute(0, 2, 1).reshape(-1, emb.shape[1]), nat.cb, codes.permute(0, 2, 1).reshape(-1, 8))
    err32, ref = _fp32_yardstick(m32.encoder, m64.encoder, wav, wav.double())
    _against_fp32_yardstick(emb, ref, err32, f"encode N={N}")


@pytest.mark.parametrize("T", range(1, 8))
def test_decode_short_inputs(codec, T):
    """T' <= 6 frames are shorter than the reflect pad of the decoder's first conv"""
    m32, m64, nat, tok = codec
    g = torch.Generator().manual_seed(50 + T)
    codes = torch.randint(0, 1024, (2, 8, T), generator=g).cuda()
    wav = tok.decode([(codes, None)])
    assert wav.shape == (2, 1, 320 * T)
    err32, ref = _fp32_yardstick(lambda c: E.decode(m32, c), lambda c: E.decode(m64, c), codes, codes)
    _against_fp32_yardstick(wav, ref, err32, f"decode T'={T}")

