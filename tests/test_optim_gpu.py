"""The native ScaledAdam / Eve steps (vb_scaled_adam_step, vb_eve_step) against the fixture the unmodified reference
wrote (tests/golden/optim_ref.pt) and against the plain-torch restatement (tests/optim_oracle.py) on the benchmark
model's real gradients; resume across implementations, the engine's re-pack after a step, determinism, launch count,
no host syncs, and the trainer's GradScaler loop."""
import copy
import random

import pytest
import torch

import optim_oracle as R
from conftest import load_golden

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _rel(a, b):
    return float((a.float().cpu() - b.float().cpu()).abs().max() / b.float().abs().max().clamp(min=1e-30))


def _native_sadam(two_groups, start=None, upto=R.STEPS, period=R.PERIOD):
    from valle.modules.optim import Eden, ScaledAdam
    params = R.make_params(DEV)
    groups = R.groups_of(params, two_groups)
    opt = ScaledAdam([{"params": [params[n] for n in g]} for g in groups], lr=0.05, betas=(0.9, 0.95),
                     clipping_scale=2.0, clipping_update_period=period, parameters_names=groups,
                     show_dominant_parameters=False)
    sched = Eden(opt, 5000, 4, warmup_batches=200)
    first = 1
    if start is not None:
        first = start[0] + 1
        with torch.no_grad():
            for n, v in start[1].items():
                params[n].copy_(v)
        opt.load_state_dict(start[2])
        sched.step_batch(start[0])
    scales = []
    for s in range(first, upto + 1):
        for n, g in R.make_grads(params, s).items():
            params[n].grad = None if g is None else g.to(DEV)
        opt.step()
        scales.append([float(opt._read_clip(opt._clip[i]).scale) for i in range(len(groups))])
        sched.step_batch(s)
    return params, opt, scales


def _check_state(got, want, tol=1e-5):
    assert list(got["state"].keys()) == list(want["state"].keys())
    for i, st in want["state"].items():
        assert list(got["state"][i].keys()) == list(st.keys()), i
        for k, v in st.items():
            g = got["state"][i][k]
            assert type(g) is type(v), (i, k, type(g), type(v))
            if isinstance(v, torch.Tensor):
                assert g.shape == v.shape, (i, k)
                assert _rel(g, v) <= tol, (i, k, _rel(g, v))
            elif isinstance(v, float):
                assert abs(g - v) <= 1e-6 * abs(v), (i, k)
            else:
                assert g == v, (i, k)


@pytest.mark.parametrize("two_groups", [False, True])
def test_scaled_adam_matches_the_reference_fixture(two_groups):
    gold = load_golden("optim_ref.pt")
    ref = gold["sadam2" if two_groups else "sadam"]
    params, opt, scales = _native_sadam(two_groups)
    for s, (a, b) in enumerate(zip(scales, ref["clip_scales"])):
        for x, y in zip(a, b):
            assert abs(x - y) <= 1e-6 * y, (s + 1, x, y)
    for n, v in ref["params40"].items():
        assert _rel(params[n].detach(), v) <= 1e-5, n
    sd = opt.state_dict()
    assert [opt.state[g["params"][0]].get("num_clipped") for g in opt.param_groups] == ref["num_clipped"]
    if not two_groups:
        _check_state(sd, ref["sd40"])
        for s, d in ref["snap"].items():
            assert s in R.SNAP_STEPS


def test_scaled_adam_snapshots_match_the_fixture():
    gold = load_golden("optim_ref.pt")["sadam"]
    for s, d in gold["snap"].items():
        params, _, _ = _native_sadam(False, upto=s)
        for n, v in d.items():
            assert _rel(params[n].detach(), v) <= 1e-5, (s, n)


def test_eve_matches_the_reference_fixture():
    from valle.modules.optim import Eve
    gold = load_golden("optim_ref.pt")
    params = R.make_params(DEV)
    opt = Eve(list(params.values()), lr=0.02, betas=(0.9, 0.98), target_rms=0.1)
    for s in range(1, R.STEPS + 1):
        for n, g in R.make_grads(params, s).items():
            params[n].grad = None if g is None else g.to(DEV)
        opt.step()
    for n, v in gold["eve"]["params40"].items():
        assert _rel(params[n].detach(), v) <= 1e-5, n
    table = params["table"]
    assert opt.state[table]["step"] == R.STEPS - sum(R.table_grad_none(s) for s in range(1, R.STEPS + 1))


def test_resume_from_the_reference_state_and_back():
    gold = load_golden("optim_ref.pt")["sadam"]
    # the reference's step-20 parameters: replay the native run to 20, then load the reference's step-20 state
    p20, _, _ = _native_sadam(False, upto=20)
    start = (20, {n: p.detach().clone() for n, p in p20.items()}, gold["sd20"])
    params, opt, _ = _native_sadam(False, start=start)
    for n, v in gold["params40"].items():
        assert _rel(params[n].detach(), v) <= 1e-5, n
    _check_state(opt.state_dict(), gold["sd40"])
    # the native step-40 state loads into the restatement, which continues like the native class
    sd = copy.deepcopy(opt.state_dict())  # state_dict() holds the live state tensors
    ps = R.make_params(DEV)
    with torch.no_grad():
        for n in ps:
            ps[n].copy_(params[n])
    o = R.ScaledAdamOracle([ps[n] for n in ps], lr=0.05, betas=(0.9, 0.95), clipping_scale=2.0,
                           clipping_update_period=R.PERIOD)
    o.load_state_dict(sd)
    for n, g in R.make_grads(ps, 41).items():
        ps[n].grad = None if g is None else g.to(DEV)
        params[n].grad = None if g is None else g.to(DEV)
    lr = R.eden_lr(0.05, 40, 0, warmup_batches=200)
    o.param_groups[0]["lr"] = opt.param_groups[0]["lr"] = lr
    o.step()
    opt.step()
    for n in ps:
        assert _rel(params[n].detach(), ps[n].detach()) <= 1e-5, n


def _bench_model():
    import bench
    m = bench.build_model(DEV).train()
    for mod in m.modules():
        if isinstance(mod, torch.nn.Dropout):
            mod.p = 0.0
    m.engine_dtype = torch.bfloat16
    return m


def _batch(seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randint(3, 100, (2, 24), generator=g).to(DEV)
    y = torch.randint(0, 1024, (2, 60, 8), generator=g).to(DEV)
    return x, torch.tensor([24, 20], dtype=torch.int32), y, torch.tensor([60, 51], dtype=torch.int32)


def _loss(m, stage, seed):
    m.rng = random.Random(seed)
    torch.manual_seed(seed)
    return m(*_batch(seed), train_stage=stage)[1]


@pytest.mark.parametrize("stage", [0, 1, 2])
def test_full_model_matches_the_restatement(stage):
    from valle.modules.optim import ScaledAdam
    m = _bench_model()
    named = list(m.stage_named_parameters(stage)) if stage else list(m.named_parameters())
    names = [n for n, _ in named]
    params = [p for _, p in named]
    twin = [torch.nn.Parameter(p.detach().clone()) for p in params]
    opt = ScaledAdam(params, lr=0.05, betas=(0.9, 0.95), clipping_scale=2.0, clipping_update_period=4,
                     parameters_names=[names], show_dominant_parameters=False)
    o = R.ScaledAdamOracle(twin, lr=0.05, betas=(0.9, 0.95), clipping_scale=2.0, clipping_update_period=4)
    nones = 0
    for s in range(12):
        opt.zero_grad(set_to_none=True)
        loss = _loss(m, stage, s)
        loss.backward()
        for p, q in zip(params, twin):
            q.grad = None if p.grad is None else p.grad.detach().clone()
            nones += p.grad is None
        if s in (5, 9):  # clipped steps (the period closes at step 8): the gradients of these steps x50
            for p, q in zip(params, twin):
                if p.grad is not None:
                    p.grad.mul_(50)
                    q.grad.mul_(50)
        opt.step()
        o.step()
    worst = max(((_rel(p.detach(), q.detach()), n) for n, p, q in zip(names, params, twin)))
    assert worst[0] <= 1e-5, worst
    opt.state_dict()  # reads num_clipped back into the state of the first sorted batch
    fs = opt.state[R._batches(params)[0][0]]
    nc = opt._read_clip(opt._clip[0]).num_clipped
    ofs = [o.state[b[0]] for b in R._batches(twin)][0]
    assert nc == ofs.get("num_clipped", 0) and fs.get("num_clipped", 0) == ofs.get("num_clipped", 0)
    assert ofs.get("num_clipped", 0) >= 1


def test_stepped_weights_reach_the_next_forward():
    """After step() the engine re-packs its bf16 weights: the next loss equals a fresh model's loaded with the
    stepped state_dict, bit for bit."""
    from valle.modules.optim import ScaledAdam
    m = _bench_model()
    names = [n for n, _ in m.named_parameters()]
    opt = ScaledAdam(m.parameters(), lr=0.05, betas=(0.9, 0.95), clipping_scale=2.0, parameters_names=[names],
                     show_dominant_parameters=False)
    for s in range(2):
        opt.zero_grad()
        _loss(m, 0, 7).backward()
        opt.step()
    after = _loss(m, 0, 7)
    fresh = _bench_model()
    fresh.load_state_dict(m.state_dict())
    assert torch.equal(after.detach(), _loss(fresh, 0, 7).detach())


def test_deterministic_launch_count_and_no_syncs():
    from valle.modules.optim import ScaledAdam
    from valle_b200 import _lib as L
    lib = L.load()
    m = _bench_model()
    runs, counts = [], {}
    for stage in (0, 1):
        named = list(m.stage_named_parameters(stage)) if stage else list(m.named_parameters())
        for rep in range(2 if stage == 0 else 1):
            ps = [torch.nn.Parameter(p.detach().clone()) for _, p in named]
            opt = ScaledAdam(ps, lr=0.05, clipping_scale=2.0, clipping_update_period=4,
                             parameters_names=[[n for n, _ in named]], show_dominant_parameters=False)
            g = torch.Generator(device=DEV).manual_seed(3)
            for s in range(6):
                for p in ps:
                    p.grad = torch.randn(p.shape, device=DEV, generator=g) * 1e-3
                torch.cuda.synchronize()
                n0 = lib.vb_launch_count()
                if s in (2, 3, 5):   # not a period step (4): no host sync
                    torch.cuda.set_sync_debug_mode("error")
                try:
                    opt.step()
                finally:
                    torch.cuda.set_sync_debug_mode(0)
                counts.setdefault(stage, set()).add(lib.vb_launch_count() - n0)
            if stage == 0:
                runs.append([p.detach().clone() for p in ps])
    assert len(named) != len(list(m.named_parameters()))
    assert counts[0] == counts[1] == {3}, counts
    assert all(torch.equal(a, b) for a, b in zip(*runs))


def test_trainer_loop_with_grad_scaler_skips_inf_steps():
    """bin/trainer.py:659-697 as written: autocast, GradScaler, scaler.step, zero_grad, scheduler.step_batch."""
    from valle.modules.optim import Eden, ScaledAdam
    m = _bench_model()
    names = [n for n, _ in m.named_parameters()]
    opt = ScaledAdam(m.parameters(), lr=0.05, betas=(0.9, 0.95), clipping_scale=2.0, parameters_names=[names],
                     show_dominant_parameters=False, clipping_update_period=1000)
    sched = Eden(opt, 5000, 4, warmup_batches=200)
    scaler = torch.amp.GradScaler("cuda", enabled=True)
    for batch_idx in range(1, 4):
        with torch.autocast("cuda", dtype=torch.float16, enabled=True):
            loss = _loss(m, 0, batch_idx)
        scaler.scale(loss).backward()
        if batch_idx == 3:
            before = [p.detach().clone() for p in m.parameters()]
            step_before = opt.state[next(iter(opt.state))]["step"]
            next(p for p in m.parameters() if p.grad is not None).grad.view(-1)[0] = float("inf")
        scaler.step(opt)
        scaler.update()
        opt.zero_grad()
        sched.step_batch(batch_idx)
    assert all(torch.equal(a, p.detach()) for a, p in zip(before, m.parameters()))
    assert opt.state[next(iter(opt.state))]["step"] == step_before == 2
