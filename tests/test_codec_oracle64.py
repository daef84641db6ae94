"""The float64 codec restatements of `tests/codec_oracle64.py` against torch and the HF EnCodec modules, on the CPU."""
import itertools

import pytest
import torch
import torch.nn.functional as F

import codec_oracle64 as C64

D = torch.float64


def _close(a, b, tol=1e-12):
    assert a.shape == b.shape, (a.shape, b.shape)
    err = float((a - b).abs().max()) if a.numel() else 0.0
    assert err <= tol * max(1.0, float(b.abs().max()) if b.numel() else 1.0), err


def test_pad1d_matches_hf_pad1d_for_every_short_length():
    from transformers.models.encodec.modeling_encodec import EncodecConv1d
    g = torch.Generator().manual_seed(0)
    for T in range(1, 21):
        x = torch.randn(2, 3, T, generator=g, dtype=D)
        for pl, pr in itertools.product(range(17), range(17)):
            for reflect in (False, True):
                ref = EncodecConv1d._pad1d(x, (pl, pr), "reflect" if reflect else "constant")
                out = C64.pad1d(x, pl, pr, reflect)
                assert torch.equal(out, ref), (T, pl, pr, reflect)


def test_encodec_pads_match_hf():
    from transformers import EncodecConfig
    from transformers.models.encodec.modeling_encodec import EncodecConv1d
    for causal in (True, False):
        cfg = EncodecConfig(use_causal_conv=causal)
        for K, stride, dil in ((7, 1, 1), (3, 1, 2), (16, 8, 1), (10, 5, 1), (4, 2, 1), (5, 3, 2)):
            m = EncodecConv1d(cfg, 1, 1, K, stride, dil)
            total = int(m.padding_total)
            for T in (1, 2, 6, 7, 8, 9, 33, 320, 321):
                extra = int(m._get_extra_padding_for_conv1d(torch.zeros(1, 1, T)))
                right = total // 2
                exp = (total, extra) if causal else (total - right, right + extra)
                assert C64.encodec_pads(T, K, stride, dil, causal) == exp, (causal, K, stride, dil, T)


@pytest.mark.parametrize("reflect", [False, True])
def test_conv1d_matches_torch(reflect):
    g = torch.Generator().manual_seed(1)
    for B, Cin, Cout, T, K, stride, dil, pl, pr, pre_elu in (
            (2, 3, 5, 40, 7, 1, 1, 6, 0, False), (1, 4, 2, 33, 3, 1, 3, 6, 0, True), (3, 2, 3, 50, 16, 8, 1, 8, 0, True),
            (2, 5, 4, 9, 4, 2, 2, 3, 2, False), (1, 1, 1, 1, 1, 1, 1, 0, 0, True), (2, 3, 2, 3, 7, 1, 1, 6, 0, True),
            (1, 2, 3, 5, 5, 3, 1, 2, 9, False)):
        x = torch.randn(B, Cin, T, generator=g, dtype=D)
        w = torch.randn(Cout, Cin, K, generator=g, dtype=D)
        b = torch.randn(Cout, generator=g, dtype=D)
        xp = F.elu(x) if pre_elu else x
        if reflect:
            from transformers.models.encodec.modeling_encodec import EncodecConv1d
            xp = EncodecConv1d._pad1d(xp, (pl, pr), "reflect")
        else:
            xp = F.pad(xp, (pl, pr))
        ref = F.conv1d(xp, w, b, stride=stride, dilation=dil)
        res = torch.randn(ref.shape, generator=g, dtype=D)
        y, s = C64.conv1d(x, w, b, stride, dil, pl, pr, reflect, pre_elu, res)
        _close(y, ref + res)
        # s bounds |y| and is the same conv on magnitudes
        assert (y.abs() <= s * (1 + 1e-12)).all()
        s_ref = F.conv1d(xp.abs(), w.abs(), b.abs(), stride=stride, dilation=dil) + res.abs()
        _close(s, s_ref)


def test_conv_transpose_and_its_phase_packing_match_torch():
    from valle_b200.data.tokenizer import _ConvT
    g = torch.Generator().manual_seed(2)
    for stride in (2, 4, 5, 8):
        for B, Cin, Cout, T in ((2, 3, 4, 11), (1, 1, 1, 1), (3, 8, 5, 2)):
            x = torch.randn(B, Cin, T, generator=g, dtype=D)
            w = torch.randn(Cin, Cout, 2 * stride, generator=g, dtype=D)
            b = torch.randn(Cout, generator=g, dtype=D)
            full = F.conv_transpose1d(F.elu(x), w, b, stride=stride)
            ref = full[..., : full.shape[-1] - stride]                  # causal: trim K - stride on the right
            y = C64.sconv_transpose1d(x, w, b, stride, pre_elu=True)
            _close(y, ref)
            yp, _ = C64.conv_transpose_as_phases(x, w, b, stride, pre_elu=True)
            _close(yp, ref)
            # the tokenizer's packing [Cin, 2, C stride] is the restated [C stride, Cin, 2], permuted
            packed = _ConvT(w, b, stride).wp
            assert torch.equal(packed, C64.pack_conv_transpose(w, stride).permute(1, 2, 0))


def test_sconv_layers_match_hf_modules_in_float64():
    """the restated SConv1d / SConvTranspose1d against HF's modules (weight-norm folded) at lengths at, below and
    above the pads"""
    from transformers import EncodecConfig
    from transformers.models.encodec.modeling_encodec import EncodecConv1d, EncodecConvTranspose1d
    torch.manual_seed(3)
    for causal in (True, False):
        cfg = EncodecConfig(use_causal_conv=causal)
        for cin, cout, K, stride, dil in ((2, 3, 7, 1, 1), (3, 2, 3, 1, 3), (2, 4, 16, 8, 1), (4, 2, 10, 5, 1)):
            m = EncodecConv1d(cfg, cin, cout, K, stride, dil).double()
            w = m.conv.weight.detach()
            for T in (1, 2, 5, 6, 7, 8, 17, 40):
                x = torch.randn(2, cin, T, dtype=D)
                with torch.no_grad():
                    ref = m(x)
                y, _ = C64.sconv1d(x, w, m.conv.bias.detach(), stride, dil, causal)
                _close(y, ref)
    cfg = EncodecConfig()
    for stride in (2, 4, 5, 8):
        m = EncodecConvTranspose1d(cfg, 3, 2, 2 * stride, stride).double()
        x = torch.randn(2, 3, 9, dtype=D)
        with torch.no_grad():
            ref = m(x)
        _close(C64.sconv_transpose1d(x, m.conv.weight.detach(), m.conv.bias.detach(), stride), ref)


def test_lstm_layer_matches_torch_lstm():
    g = torch.Generator().manual_seed(4)
    for H, B, T in ((8, 3, 17), (32, 1, 5), (16, 5, 1)):
        lstm = torch.nn.LSTM(H, H, 1).double()
        x = torch.randn(T, B, H, generator=g, dtype=D)
        with torch.no_grad():
            ref = lstm(x)[0]
        xproj = x @ lstm.weight_ih_l0.detach().t() + lstm.bias_ih_l0.detach() + lstm.bias_hh_l0.detach()
        _close(C64.lstm_layer(xproj, lstm.weight_hh_l0.detach()), ref)


def test_rvq_encode_matches_the_hf_quantizer_and_its_margins():
    from oracle import encodec_oracle as E
    m = E.build_codec(0).double()
    g = torch.Generator().manual_seed(5)
    emb = torch.randn(2, 128, 30, generator=g, dtype=D) * 3
    with torch.no_grad():
        ref_codes = m.quantizer.encode(emb, 6.0)                          # [8, B, T]
    margins_ref = E.rvq_margins(m, emb)                                   # [8, B, T]
    cbs = torch.stack([layer.codebook.embed for layer in m.quantizer.layers[:8]])
    rows = emb.permute(0, 2, 1).reshape(-1, 128)
    codes, margins, res = C64.rvq_encode(rows, cbs)
    assert torch.equal(codes, ref_codes.permute(1, 2, 0).reshape(-1, 8))
    _close(margins, margins_ref.permute(1, 2, 0).reshape(-1, 8), 1e-9)
    assert torch.equal(res[0], rows)
    # teacher forcing with the own picks is the free-running encode
    codes2, margins2, _ = C64.rvq_encode(rows, cbs, picks=codes)
    assert torch.equal(codes2, codes) and torch.equal(margins2, margins)


def test_rvq_encode_breaks_ties_toward_the_first_index():
    cb = torch.tensor([[[1.0, 0.0], [0.0, 1.0], [1.0, 0.0], [0.0, 1.0]]], dtype=D)
    x = torch.tensor([[1.0, 0.0], [0.0, 1.0], [0.5, 0.5]], dtype=D)
    codes, margins, _ = C64.rvq_encode(x, cb)
    assert codes[:, 0].tolist() == [0, 1, 0]
    assert margins[:, 0].tolist() == [0.0, 0.0, 0.0]
    one, m1, _ = C64.rvq_encode(x, cb[:, :1])
    assert one[:, 0].tolist() == [0, 0, 0] and torch.isinf(m1).all()
