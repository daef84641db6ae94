"""Cost of the pre-nets in a bf16 training step (DESIGN.md section 7): VALLE.forward + loss.backward() at
d=1024 / 16 heads / 12 layers, 16 utterances x 47 phonemes x 753 frames, train_stage 0, dropout live, for twins with
add_prenet=True and False built from the same seed, timed alternately with CUDA events; then, in a separate
torch.profiler run, the device time of each pre-net kernel.

    python tools/bench_prenet_train.py [--runs 3] [--steps 5] [--warmup 2] [--out DIR]
"""
from __future__ import annotations

import argparse
import json
import os
import random
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

N, S, T, D, H, LAYERS = 16, 47, 753, 1024, 16, 12
PRENET_KERNELS = ("bn_stats_kernel", "bn_apply_kernel", "bn_bwd_stats_kernel", "bn_bwd_apply_kernel",
                  "relu_dropout_bwd_kernel")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name()


def make(add_prenet):
    from valle_b200.models import VALLE
    torch.manual_seed(0)
    m = VALLE(D, H, LAYERS, norm_first=True, add_prenet=add_prenet, prefix_mode=1, num_quantizers=8).cuda().train()
    m.engine_dtype = torch.bfloat16
    return m


def batch():
    g = torch.Generator().manual_seed(7)
    x = torch.randint(3, 100, (N, S), generator=g)
    y = torch.randint(0, 1024, (N, T, 8), generator=g)
    return x, torch.full((N,), S, dtype=torch.int32), y, torch.full((N,), T, dtype=torch.int32)


def step(m, inp):
    x, xl, y, yl = inp
    m.rng = random.Random(0)
    torch.manual_seed(5)
    m.zero_grad(set_to_none=True)
    (_, _), loss, _ = m(x.cuda(), xl, y.cuda(), yl, train_stage=0)
    loss.backward()


def timed(m, inp, steps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(steps):
        step(m, inp)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    inp = batch()
    models = {True: make(True), False: make(False)}
    for m in models.values():
        for _ in range(a.warmup):
            step(m, inp)
    ms = {True: [], False: []}
    for _ in range(a.runs):
        for k in (False, True):
            ms[k].append(timed(models[k], inp, a.steps))
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        step(models[True], inp)
        torch.cuda.synchronize()
    kern = {}
    for ev in prof.key_averages():
        if any(k in ev.key for k in PRENET_KERNELS):
            name = next(k for k in PRENET_KERNELS if k in ev.key)
            t = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0.0)
            c = kern.setdefault(name, {"us": 0.0, "calls": 0})
            c["us"] += t
            c["calls"] += ev.count
    res = {"card": card(), "shape": dict(N=N, S=S, T=T, d=D, heads=H, layers=LAYERS, dtype="bf16", train_stage=0),
           "step_ms_prenet": ms[True], "step_ms_plain": ms[False], "prenet_kernels_us_per_step": kern}
    print(json.dumps(res))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_prenet_train.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
