"""Writes tests/golden/optim_ref.pt from the UNMODIFIED reference valle/modules/optim.py and scheduler.py.

    python tools/gen_golden_optim.py [--check]

The reference files are exec'd where they lie (oracle.ref_loader.REFERENCE_ROOT); `lhotse.utils.fix_random_seed`,
which optim.py imports but the optimizers never call, is stubbed.  The recipe (tests/optim_oracle.py make_params /
make_grads): VALLE's shape classes at d = 32 (three (1,) scalars, a (1, d) row, 2-deep stacks of [3d, d] and [3d], a
[1025, d] table whose gradient is None every 5th step), 40 steps with betas (0.9, 0.95), clipping_scale 2.0,
clipping_update_period 8 and Eden(opt, 5000, 4, warmup_batches=200); gradients from a seeded CPU generator, scaled
x10 at steps 13, 29 and x100 at steps 22, 37.  Every clip decision and every Eve norm test is asserted to lie more
than 1e-4 relative away from its boundary.  --check regenerates and compares with the stored file.
"""
from __future__ import annotations

import copy
import importlib.util
import os
import sys
import types

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from oracle.ref_loader import REFERENCE_ROOT  # noqa: E402
import optim_oracle as R  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "optim_ref.pt")
BASE_LR = 0.05


def load_reference():
    if "lhotse" not in sys.modules:
        lh = types.ModuleType("lhotse")
        lu = types.ModuleType("lhotse.utils")
        lu.fix_random_seed = lambda seed: None  # only _test_scaled_adam calls it
        lh.utils = lu
        sys.modules["lhotse"], sys.modules["lhotse.utils"] = lh, lu
    mods = {}
    saved = {k: v for k, v in sys.modules.items() if k == "valle" or k.startswith("valle.")}
    for k in saved:
        del sys.modules[k]
    try:
        for name in ("valle", "valle.modules"):
            m = types.ModuleType(name)
            m.__path__ = []
            sys.modules[name] = m
        for leaf in ("optim", "scheduler"):
            spec = importlib.util.spec_from_file_location(
                f"valle.modules.{leaf}", os.path.join(REFERENCE_ROOT, "valle", "modules", f"{leaf}.py"))
            m = importlib.util.module_from_spec(spec)
            sys.modules[f"valle.modules.{leaf}"] = m
            spec.loader.exec_module(m)
            mods[leaf] = m
    finally:
        for k in [k for k in sys.modules if k == "valle" or k.startswith("valle.")]:
            del sys.modules[k]
        sys.modules.update(saved)
    return mods["optim"], mods["scheduler"]


def run_scaled_adam(optim, two_groups):
    params = R.make_params()
    groups = R.groups_of(params, two_groups)
    opt = optim.ScaledAdam([{"params": [params[n] for n in g]} for g in groups], lr=BASE_LR, betas=(0.9, 0.95),
                           clipping_scale=2.0, clipping_update_period=R.PERIOD, parameters_names=groups,
                           show_dominant_parameters=False)
    sched = optim.Eden(opt, 5000, 4, warmup_batches=200)
    scales = []
    orig = opt._get_clipping_scale

    def wrapped(group, tuples):
        ans = orig(group, tuples)
        fs = tuples[0][1]
        step = fs["step"]
        if step >= R.PERIOD and "model_norm_threshold" in fs:
            ratio = fs["model_norm_threshold"] / fs["model_norms"][step % R.PERIOD].item()
            assert abs(ratio - 1.0) > 1e-4, f"clip decision at step {step} within 1e-4 of its boundary ({ratio})"
        scales[-1][opt.param_groups.index(group)] = ans
        return ans

    opt._get_clipping_scale = wrapped
    rec = {"clip_scales": [], "snap": {}, "lr": []}
    for s in range(1, R.STEPS + 1):
        for n, g in R.make_grads(params, s).items():
            params[n].grad = g
        scales.append([1.0] * len(groups))
        opt.step()
        sched.step_batch(s)
        rec["lr"].append(sched.get_last_lr()[0])
        if s in R.SNAP_STEPS:
            rec["snap"][s] = {n: p.detach().clone() for n, p in params.items() if n not in R.BIG}
        if s == 20:
            rec["sd20"] = copy.deepcopy(opt.state_dict())
    rec["clip_scales"] = scales
    rec["params40"] = {n: p.detach().clone() for n, p in params.items()}
    rec["sd40"] = copy.deepcopy(opt.state_dict())
    rec["num_clipped"] = [opt.state[opt.param_groups[i]["params"][0]].get("num_clipped") for i in range(len(groups))]
    assert min(min(x) for x in scales) < 0.1 and any(0.1 < x[0] < 1.0 for x in scales), scales
    return rec


def run_eve(optim):
    params = R.make_params()
    opt = optim.Eve(list(params.values()), lr=0.02, betas=(0.9, 0.98), target_rms=0.1)
    for s in range(1, R.STEPS + 1):
        for n, g in R.make_grads(params, s).items():
            params[n].grad = g
            p = params[n]
            if g is not None and p.numel() > 1:
                r = p.norm().item() / (0.1 * p.numel() ** 0.5)
                assert abs(r - 1.0) > 1e-4, f"Eve norm test of {n} at step {s} within 1e-4 of its boundary ({r})"
        opt.step()
    return {"params40": {n: p.detach().clone() for n, p in params.items()}}


def generate():
    optim, scheduler = load_reference()
    torch.manual_seed(0)
    g1 = R.make_grads(R.make_params(), 1)
    out = {
        "recipe": __doc__,
        "grad_checksum_step1": sum(float(g.double().sum()) for g in g1.values() if g is not None),
        "base_lr": BASE_LR,
        "sadam": run_scaled_adam(optim, False),
        "eve": run_eve(optim),
    }
    two = run_scaled_adam(optim, True)
    out["sadam2"] = {"clip_scales": two["clip_scales"], "num_clipped": two["num_clipped"],
                     "params40": {n: two["params40"][n] for n in two["params40"] if n not in R.BIG}}
    # schedulers: Eden on its own optimizer with an epoch step, Noam's calc_lr as the reference computes it
    p = torch.nn.Parameter(torch.zeros(2))
    opt = optim.Eve([p], lr=0.05)
    eden = optim.Eden(opt, 5000, 4, warmup_batches=200)
    seq = []
    for b in range(0, 1200, 7):
        eden.step_batch(b)
        if b % 301 == 0:
            eden.step_epoch()
        seq.append((b, eden.epoch, eden.get_last_lr()[0]))
    out["eden_lr"] = seq
    out["noam_lr"] = [(s, 0.05 * scheduler.calc_lr(s, 1024, 200)) for s in range(1, 1000, 3)]
    return out


def main():
    out = generate()
    if "--check" in sys.argv:
        old = torch.load(OUT, weights_only=False)

        def same(a, b):
            if isinstance(a, torch.Tensor):
                return torch.equal(a, b)
            if isinstance(a, dict):
                return a.keys() == b.keys() and all(same(a[k], b[k]) for k in a)
            if isinstance(a, (list, tuple)):
                return len(a) == len(b) and all(same(x, y) for x, y in zip(a, b))
            return a == b
        assert same(out, old), "regenerated fixture differs from tests/golden/optim_ref.pt"
        print("optim_ref.pt reproduced exactly")
        return
    torch.save(out, OUT)
    print(f"wrote {OUT}: {os.path.getsize(OUT)} bytes")


if __name__ == "__main__":
    main()
