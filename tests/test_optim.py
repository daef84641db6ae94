"""CPU checks of the optimizer surface (valle/modules/optim.py, scheduler.py): the plain-torch restatement
(tests/optim_oracle.py) reproduces the fixture the unmodified reference wrote, the shim imports without a GPU, the
schedulers reproduce the reference's learning rates exactly, and the native step refuses CPU parameters."""
import pytest
import torch

import optim_oracle as R
from conftest import load_golden


def _rel(a, b):
    return float((a - b).abs().max() / b.abs().max().clamp(min=1e-30))


def run_oracle_sadam(two_groups, device="cpu", start=None, upto=R.STEPS):
    params = R.make_params(device)
    groups = R.groups_of(params, two_groups)
    opt = R.ScaledAdamOracle([{"params": [params[n] for n in g]} for g in groups], lr=0.05, betas=(0.9, 0.95),
                             clipping_scale=2.0, clipping_update_period=R.PERIOD)
    first = 1
    if start is not None:
        first = start[0] + 1
        for n, v in start[1].items():
            params[n].data.copy_(v)
        opt.load_state_dict(start[2])
    snaps = {}
    for s in range(first, upto + 1):
        for n, g in R.make_grads(params, s).items():
            params[n].grad = None if g is None else g.to(device)
        lr = 0.05 if s == 1 else R.eden_lr(0.05, s - 1, 0, warmup_batches=200)  # Eden sets lr after each step
        for grp in opt.param_groups:
            grp["lr"] = lr
        opt.step()
        snaps[s] = {n: p.detach().clone() for n, p in params.items()}
    return params, opt, snaps


def test_restatement_reproduces_the_reference_fixture():
    gold = load_golden("optim_ref.pt")
    ref = gold["sadam"]
    params, opt, snaps = run_oracle_sadam(False)
    scales = [x for x in opt.clip_scales]
    assert len(scales) == R.STEPS
    for s, (a, b) in enumerate(zip(scales, [x[0] for x in ref["clip_scales"]])):
        assert abs(a - b) <= 1e-6 * b, (s, a, b)
    for s, d in ref["snap"].items():
        for n, v in d.items():
            assert _rel(snaps[s][n], v) <= 1e-6, (s, n)
    for n, v in ref["params40"].items():
        assert _rel(params[n].detach(), v) <= 1e-6, n
    sd = opt.state_dict()
    for i, st in ref["sd40"]["state"].items():
        assert list(sd["state"][i].keys()) == list(st.keys())
        for k, v in st.items():
            assert type(sd["state"][i][k]) is type(v), (i, k)
            if isinstance(v, torch.Tensor):
                assert sd["state"][i][k].shape == v.shape and _rel(sd["state"][i][k], v) <= 1e-6, (i, k)
            else:
                assert abs(sd["state"][i][k] - v) <= 1e-6 * abs(v), (i, k)


def test_restatement_eve_reproduces_the_reference_fixture():
    gold = load_golden("optim_ref.pt")
    params = R.make_params()
    opt = R.EveOracle(list(params.values()), lr=0.02, betas=(0.9, 0.98), target_rms=0.1)
    for s in range(1, R.STEPS + 1):
        for n, g in R.make_grads(params, s).items():
            params[n].grad = g
        opt.step()
    for n, v in gold["eve"]["params40"].items():
        assert _rel(params[n].detach(), v) <= 1e-6, n


def test_fixture_recipe_checksum():
    gold = load_golden("optim_ref.pt")
    g1 = R.make_grads(R.make_params(), 1)
    assert sum(float(g.double().sum()) for g in g1.values() if g is not None) == gold["grad_checksum_step1"]


def test_shim_imports_without_gpu():
    from valle.modules.optim import Eden, Eve, ScaledAdam  # noqa: F401
    from valle.modules.scheduler import get_scheduler  # noqa: F401
    from torch.optim import Optimizer
    assert issubclass(ScaledAdam, Optimizer) and issubclass(Eve, Optimizer)


def test_schedulers_match_the_reference_exactly():
    from valle.modules.optim import Eden
    from valle.modules.scheduler import calc_lr, get_scheduler
    gold = load_golden("optim_ref.pt")
    p = torch.nn.Parameter(torch.zeros(2))
    eden = Eden(torch.optim.SGD([p], lr=0.05), 5000, 4, warmup_batches=200)
    for b, epoch, lr in gold["eden_lr"]:
        eden.step_batch(b)
        if b % 301 == 0:
            eden.step_epoch()
        assert eden.epoch == epoch and eden.get_last_lr()[0] == lr
    for s, lr in gold["noam_lr"]:
        assert 0.05 * calc_lr(s, 1024, 200) == lr
    # the fixture's Eden sequence inside the ScaledAdam run (stepped with the batch index after each step)
    for s, lr in enumerate(gold["sadam"]["lr"], start=1):
        assert R.eden_lr(0.05, s, 0, warmup_batches=200) == lr
    params = type("P", (), dict(scheduler_name="Eden", warmup_steps=200, base_lr=0.05, decoder_dim=1024))()
    assert isinstance(get_scheduler(params, torch.optim.SGD([p], lr=0.05)), Eden)
    with pytest.raises(TypeError):
        Eden(object(), 5000, 4)


def test_native_step_refuses_cpu_parameters():
    from valle_b200 import _lib as L
    from valle.modules.optim import Eve, ScaledAdam
    p = torch.nn.Parameter(torch.zeros(4, 4))
    p.grad = torch.ones(4, 4)
    opt = ScaledAdam([p], parameters_names=[["w"]])
    with pytest.raises(L.VbError, match="w"):
        opt.step()
    with pytest.raises(L.VbError):
        Eve([p]).step()
