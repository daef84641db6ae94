"""CPU checks of the pre-net training restatement (tests/prenet_oracle.py) against the reference's own training step
(tests/golden/prenet_train.pt, written by tools/gen_golden_prenet_train.py): loss, BatchNorm buffers after the call and
the sampled gradient elements, for the configurations the oracle restates (prefix modes 0 / 1, both layer orders)."""
import contextlib
import random
import re

import pytest
import torch

import postln_oracle as P
import prenet_oracle as PN
from conftest import load_golden
from oracle import valle_oracle as O

CONV_BIAS = re.compile(r"_text_prenet\.(1|5|9)\.bias$")


def build(cfg, seed=0):
    """valle_b200 VALLE of a fixture configuration with the reference's init under torch.manual_seed(seed)"""
    from valle_b200.models import VALLE
    torch.manual_seed(seed)
    return VALLE(cfg["d_model"], cfg["nhead"], cfg["num_layers"], norm_first=cfg["norm_first"], add_prenet=True,
                 prefix_mode=cfg["prefix_mode"], share_embedding=True, nar_scale_factor=cfg["nar_scale_factor"],
                 prepend_bos=cfg["prepend_bos"], num_quantizers=cfg["num_quantizers"])


def check_init(m, rec):
    got = O.weight_checksums(m.state_dict())
    assert list(got) == rec["checksum_keys"]
    assert torch.equal(torch.stack(list(got.values())), rec["checksums"])


def sampled(name, t):
    return t.reshape(-1)[PN.sample_positions(name, t.numel())]


def draws(rec):
    """the nar_stage / prefix_len the reference drew (m.rng = random.Random(0), torch.manual_seed(torch_seed))"""
    nar_stage = random.Random(0).choices(list(range(1, 8)), weights=[1 / 7] * 7, k=1)[0]
    torch.manual_seed(5)
    int_low = (0.25 * rec["y_lens"].min()).type(torch.int64).item()
    return nar_stage, min(torch.randint(int_low, int_low * 2, size=()).item(), 225)


@pytest.fixture(scope="module")
def golden():
    return load_golden("prenet_train.pt")


@pytest.mark.parametrize("name", ["preln_pm1", "postln_pm0"])
@pytest.mark.parametrize("stage", [0, 1, 2])
def test_oracle_matches_reference_training_step(golden, name, stage):
    rec = golden["configs"][name]
    c = rec["config"]
    m = build(c)
    check_init(m, rec)
    sd = {k: v.detach().clone().requires_grad_(v.is_floating_point()) for k, v in m.state_dict().items()}
    cfg = O.OracleConfig(c["d_model"], c["nhead"], c["num_layers"], c["prefix_mode"], 8)
    nar_stage, prefix_len = draws(rec)
    with P.post_ln() if not c["norm_first"] else contextlib.nullcontext():
        loss, _, bufs = PN.forward_train(sd, cfg, rec["x"], rec["x_lens"], rec["y"].long(), rec["y_lens"], nar_stage,
                                         prefix_len, train_stage=stage)
    loss.backward()
    st = rec["stages"][stage]
    assert abs(float(loss.detach()) - st["loss"]) <= 1e-5 * abs(st["loss"])
    mean = torch.cat([bufs[k + ".running_mean"] for k in st["buffer_keys"]])
    var = torch.cat([bufs[k + ".running_var"] for k in st["buffer_keys"]])
    assert float((mean - st["running_mean"]).abs().max()) <= 1e-5 * float(st["running_mean"].abs().max())
    assert float((var - st["running_var"]).abs().max()) <= 1e-5 * float(st["running_var"].abs().max())
    assert [int(bufs[k + ".num_batches_tracked"]) for k in st["buffer_keys"]] == st["num_batches_tracked"]
    by_ptr = {}
    for k, v in m.state_dict().items():
        by_ptr.setdefault(v.data_ptr(), []).append(k)
    params = dict(m.named_parameters())
    g = st["grads"]
    assert len(g["names"]) > 40
    top = float(g["max_abs"].max())
    for i, n in enumerate(g["names"]):
        if CONV_BIAS.search(n):
            # BatchNorm on batch statistics subtracts the channel mean: the exact gradient of a conv bias is 0, and
            # both sides hold rounding residue of a sum over the batch
            assert float(g["max_abs"][i]) < 1e-6 * top, n
            continue
        want = sum(sd[k].grad for k in by_ptr[params[n].data_ptr()] if sd[k].grad is not None)
        err = float((sampled(n, want) - g["values"][i]).abs().max())
        assert err <= 1e-4 * float(g["max_abs"][i]) + 1e-12, (n, err, float(g["max_abs"][i]))
