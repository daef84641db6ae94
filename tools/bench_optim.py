"""Times one optimizer step on the benchmark model (d=1024/16h/12L), native ScaledAdam against the plain-torch
restatement of the reference (tests/optim_oracle.py), for training stages 0, 1 and 2, and a whole bf16 training step
(forward + backward + step) with each optimizer.

    python tools/bench_optim.py [--steps 20] [--warmup 5] [--reps 3] [--out results.json]

CUDA events; the repetitions alternate native and baseline.  Algorithmic bytes of the native step: 36 B per element
(reduction: p, g; update: p, g, delta, exp_avg_sq read, p, delta, exp_avg_sq written).
"""
from __future__ import annotations

import argparse
import json
import os
import random
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import bench  # noqa: E402
import optim_oracle as R  # noqa: E402
from valle.modules.optim import ScaledAdam  # noqa: E402

DEV = "cuda:0"
HBM = 3.35e12


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True).stdout.strip()
    except OSError:
        return torch.cuda.get_device_name(0)


def make_opt(kind, params, names):
    kw = dict(lr=0.05, betas=(0.9, 0.95), clipping_scale=2.0, clipping_update_period=1000)
    if kind == "native":
        return ScaledAdam(params, parameters_names=[names], show_dominant_parameters=False, **kw)
    return R.ScaledAdamOracle(params, **kw)


def time_steps(opt, params, steps, warmup):
    g = torch.Generator(device=DEV).manual_seed(0)
    for p in params:
        p.grad = torch.randn(p.shape, device=DEV, generator=g) * 1e-3
    for _ in range(warmup):
        opt.step()
    torch.cuda.synchronize()
    m0 = torch.cuda.max_memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        opt.step()
    e1.record()
    torch.cuda.synchronize()
    del m0
    return e0.elapsed_time(e1) / steps, (torch.cuda.max_memory_allocated() - base) / 1e6


def train_step_ms(kind, steps, warmup):
    m = bench.build_model(DEV).train()
    m.engine_dtype = torch.bfloat16
    names = [n for n, _ in m.named_parameters()]
    opt = make_opt(kind, list(m.parameters()), names)
    gen = torch.Generator().manual_seed(0)
    x = torch.randint(3, 100, (16, 47), generator=gen).to(DEV)
    y = torch.randint(0, 1024, (16, 753, 8), generator=gen).to(DEV)
    xl = torch.full((16,), 47, dtype=torch.int32)
    yl = torch.full((16,), 753, dtype=torch.int32)

    def one():
        m.rng = random.Random(0)
        opt.zero_grad(set_to_none=True)
        loss = m(x, xl, y, yl, train_stage=0)[1]
        loss.backward()
        opt.step()
    for _ in range(warmup):
        one()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        one()
    e1.record()
    torch.cuda.synchronize()
    del m, opt
    torch.cuda.empty_cache()
    return e0.elapsed_time(e1) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--train-steps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_optim needs a GPU"
    res = {"card": card(), "stages": {}}
    print("card, power limit:", res["card"])
    model = bench.build_model(DEV).train()
    for stage in (0, 1, 2):
        named = list(model.stage_named_parameters(stage)) if stage else list(model.named_parameters())
        numel = sum(p.numel() for _, p in named)
        row = {"tensors": len(named), "numel": numel, "native_ms": [], "oracle_ms": [], "native_mb": [], "oracle_mb": []}
        for _ in range(a.reps):
            for kind in ("native", "oracle"):
                ps = [torch.nn.Parameter(p.detach().clone()) for _, p in named]
                opt = make_opt(kind, ps, [n for n, _ in named])
                ms, mb = time_steps(opt, ps, a.steps, a.warmup)
                row[f"{kind}_ms"].append(round(ms, 3))
                row[f"{kind}_mb"].append(round(mb, 1))
                del opt, ps
                torch.cuda.empty_cache()
        best = min(row["native_ms"])
        row["native_gbs"] = round(36 * numel / best / 1e6, 1)
        row["native_share_of_3.35TBs"] = round(36 * numel / (best * 1e-3) / HBM, 3)
        res["stages"][stage] = row
        print(f"stage {stage}: {len(named)} tensors, {numel / 1e6:.1f} M elements: native {row['native_ms']} ms "
              f"({row['native_gbs']} GB/s at 36 B/elem, {row['native_share_of_3.35TBs']:.1%} of 3.35 TB/s), "
              f"restatement {row['oracle_ms']} ms; peak extra memory native {row['native_mb']} MB, "
              f"restatement {row['oracle_mb']} MB")
    del model
    torch.cuda.empty_cache()
    tr = {"native": [], "oracle": []}
    for _ in range(2):
        for kind in ("native", "oracle"):
            tr[kind].append(round(train_step_ms(kind, a.train_steps, 2), 2))
    res["train_step_ms"] = tr
    print(f"whole bf16 training step (16 x 47 text x 753 frames, stage 0): native optimizer {tr['native']} ms, "
          f"restatement {tr['oracle']} ms")
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        json.dump(res, open(a.out, "w"), indent=1)


if __name__ == "__main__":
    main()
