"""CPU checks of post-LN VALL-E (`norm_first=False`, valle/modules/transformer.py:303-308; no final norm,
valle/models/valle.py:151,242-246): the oracle restatement against the reference's stored outputs, and the
checkpoint layout of the model class against the reference class's."""
import pytest
import torch

from conftest import load_golden
from oracle import valle_oracle as O

import postln_oracle as P

FIXTURES = ["tiny_postln_pm0.pt", "tiny_postln_pm1.pt"]


def postln_model(cfg, seed):
    """valle_b200 VALLE with norm_first=False and the reference's default init under torch.manual_seed(seed)"""
    from valle_b200.models import VALLE
    torch.manual_seed(seed)
    return VALLE(cfg["d_model"], cfg["nhead"], cfg["num_layers"], norm_first=False,
                 add_prenet=cfg.get("add_prenet", False), prefix_mode=cfg["prefix_mode"], share_embedding=True,
                 nar_scale_factor=cfg.get("nar_scale_factor", 1.0), prepend_bos=False,
                 num_quantizers=cfg["num_quantizers"]).eval()


def _cfg(g):
    c = g["config"]
    return O.OracleConfig(c["d_model"], c["nhead"], c["num_layers"], c["prefix_mode"], c["num_quantizers"])


def _sd(g):
    m = postln_model(g["config"], g["weight_seed"])
    got = O.weight_checksums(m.state_dict())
    assert list(got) == list(g["checksums"])
    for k in got:
        assert torch.equal(got[k], g["checksums"][k]), k
    return {k: v.detach() for k, v in m.state_dict().items()}


@pytest.mark.parametrize("name", FIXTURES)
def test_oracle_postln_inference_matches_the_reference(name):
    g = load_golden(name)
    sd, cfg = _sd(g), _cfg(g)
    x, y = g["x"], g["y"]
    xl = torch.tensor([x.shape[1]], dtype=torch.int32)
    tr = O.InferenceTrace([], [], [], [])
    with torch.no_grad():
        codes = P.inference(sd, cfg, x, xl, y, None, top_k=1, trace=tr)
        assert torch.equal(codes, g["codes"].long())
        assert torch.allclose(torch.tensor(tr.ar_margin), g["ar_margin"], atol=1e-5)
        assert torch.equal(P.continual(sd, cfg, x, xl, y), g["continual"].long())
        s = g["sampled"]
        torch.manual_seed(s["torch_seed"])
        got = P.inference(sd, cfg, x, xl, y, None, top_k=s["top_k"], temperature=s["temperature"])
        assert torch.equal(got, s["codes"].long())


@pytest.mark.parametrize("name", FIXTURES)
@pytest.mark.parametrize("stage", [0, 1, 2])
def test_oracle_postln_losses_match_the_reference(name, stage):
    g = load_golden(name)
    sd, cfg, fw = _sd(g), _cfg(g), g["forward"]
    with torch.no_grad():
        loss, _ = P.forward_train(sd, cfg, fw["x"], fw["x_lens"], fw["y"].long(), fw["y_lens"], int(fw["nar_stage"]),
                                  int(fw["prefix_len"]), train_stage=stage)
    want = float(fw[f"loss_stage{stage}"])
    assert abs(float(loss) - want) <= 1e-4 * abs(want), (float(loss), want)


def test_postln_checkpoint_layout_equals_the_reference_class():
    g = load_golden("tiny_postln_pm1.pt")
    lay = g["layout"]
    m = postln_model(g["config"], 0)
    sd = m.state_dict()
    assert list(sd.keys()) == lay["keys"]
    assert [tuple(v.shape) for v in sd.values()] == lay["shapes"]
    assert [n for n, _ in m.named_parameters()] == lay["params"]
    assert [n for n, _ in m.named_buffers()] == lay["buffers"]
    got = O.weight_checksums(sd)
    for k in lay["keys"]:
        assert torch.equal(got[k], lay["checksums"][k]), k
    assert not any(k.startswith(("ar_decoder.norm.", "nar_decoder.norm.")) for k in sd)


def test_get_model_norm_first_false_round_trips_a_checkpoint():
    from valle.models import get_model
    from valle.utils import AttributeDict
    params = AttributeDict(model_name="VALL-E", decoder_dim=256, nhead=4, num_decoder_layers=2, scale_factor=1.0,
                           norm_first=False, add_prenet=False, prefix_mode=1, share_embedding=True, prepend_bos=False,
                           num_quantizers=8)
    m = get_model(params)
    assert not m.ar_decoder.layers[0].norm_first and m.ar_decoder.norm is None and m.nar_decoder.norm is None
    src = postln_model(dict(d_model=256, nhead=4, num_layers=2, prefix_mode=1, num_quantizers=8), 7)
    ck = {k: v.clone() for k, v in src.state_dict().items()}
    m.load_state_dict(ck, strict=True)
    for k, v in m.state_dict().items():
        assert torch.equal(v, ck[k]), k
    pre = get_model(AttributeDict(dict(params, norm_first=True)))
    with pytest.raises(RuntimeError):     # a pre-LN model has the final-norm keys a post-LN checkpoint lacks
        pre.load_state_dict(ck, strict=True)


def test_decode_of_a_pre_ln_decoder_without_final_norm_is_refused(lib):
    """a pre-LN decode step leaves the last FFN2's split-K partials to the final norm's reduce, so the AR head and decode
    step refuse a pre-LN decoder without one (the checks run before any device pointer is used)"""
    import ctypes as C
    from valle_b200 import _lib as L
    layers = (L.LayerParams * 1)()
    for name, _ in L.LayerParams._fields_:
        setattr(layers[0], name, 256)      # never dereferenced
    desc = L.DecoderDesc(d_model=256, n_head=4, n_layer=1, d_ff=1024, wdtype=L.VB_BF16, layers=layers, norm_first=1)
    h = C.c_void_p()
    L.check(lib.vb_decoder_create(C.byref(desc), C.byref(h)), "vb_decoder_create")
    try:
        head, st = L.ArHead(greedy=1), L.ArState(B=1)
        assert lib.vb_ar_head_step(h, C.byref(head), 256, C.byref(st), None, 0, None) == 1
        assert b"final norm" in lib.vb_last_error()
        assert lib.vb_ar_decode_step(h, C.byref(head), C.byref(st), None, 0, None) == 1
        assert b"final norm" in lib.vb_last_error()
    finally:
        lib.vb_decoder_destroy(h)
