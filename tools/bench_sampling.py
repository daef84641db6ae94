"""AR decode cost of sampled decoding against greedy on bench.py's model and workload (d=1024/16h/12L, bf16, S=47,
225-frame prompt, up to 753 frames).

    python tools/bench_sampling.py [--batches 1,64] [--repeats 2] [--run-to-cap] [--profile-steps 64]

Modes, each warmed up first, then run in alternation `--repeats` times:
  greedy       top_k=1 (what bench.py times)
  torch        top_k=-100, seed=None: the per-step torch draw (topk_sampling + vb_ar_push_tokens), no graphs
  native       top_k=-100, seed=...: the seeded sampler in the decode step's tail, CUDA-graph replays
  native_k50   top_k=50, temperature=0.8, seed=...
  native_p09   top_k=-100, top_p=0.9, seed=...: the nucleus (sort and scan of the whole row in the sampler)
  native_p09_ras  native_p09 plus repetition-aware sampling, ras=(10, 0.1)
Per mode: AR us per decode step from the engine's device events, ar_steps, library kernels and graph replays per
step, frames generated (live rows), and the wall time of a synchronised generate().

Sampling can stop an utterance early, and a step with fewer live rows is not the same work.  --run-to-cap makes every
mode run to the cap: the EOS row of ar_predict_layer becomes -c and the final LayerNorm's bias +c', so the EOS logit is
the constant -c c' d (the normalised row sums to zero; the final norm's weight is 1 at init) and EOS is never drawn.
--profile-steps N adds a torch.profiler run of N native steps (a run of its own, after the timing) that reports the
device time of the decode tail's sampler kernel against the greedy tail's.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import bench  # noqa: E402

MODES = {
    "greedy": dict(top_k=1),
    "torch": dict(top_k=-100),
    "native": dict(top_k=-100, seed=1234),
    "native_k50": dict(top_k=50, temperature=0.8, seed=1234),
    "native_p09": dict(top_k=-100, top_p=0.9, seed=1234),
    "native_p09_ras": dict(top_k=-100, top_p=0.9, ras=(10, 0.1), seed=1234),
}


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def run(eng, texts, prompts, kw):
    n0, r0 = eng.kernel_launches(), eng.replayed_launches
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = eng.generate(texts, prompts, return_device=True, **kw)
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    st = eng.stats
    steps = max(1, st.ar_steps)
    return dict(ar_us_per_step=1e3 * st.ar_ms / steps, ar_steps=st.ar_steps, ar_ms=st.ar_ms,
                launches_per_step=(eng.kernel_launches() - n0) / steps,
                replayed_per_step=(eng.replayed_launches - r0) / steps,
                frames=sum(int(o.shape[0]) for o in out), wall_ms=1e3 * wall)


def profile(eng, texts, prompts, steps):
    from torch.profiler import ProfilerActivity, profile as prof
    res = {}
    for name in ("greedy", "native", "native_p09", "native_p09_ras"):
        eng.generate(texts, prompts, max_new_tokens=steps, **MODES[name])   # warm, captured
        with prof(activities=[ProfilerActivity.CUDA]) as p:
            eng.generate(texts, prompts, max_new_tokens=steps, **MODES[name])
            torch.cuda.synchronize()
        for e in p.key_averages():
            if "ar_sample_kernel" in e.key:
                t = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0)
                res[f"{name}:{'sample' if 'true' in e.key or 'Lb1' in e.key else 'argmax'}"] = \
                    dict(calls=e.count, us_per_call=t / max(1, e.count))
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="1,64")
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--run-to-cap", action="store_true")
    ap.add_argument("--profile-steps", type=int, default=0)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "tools/bench_sampling.py needs a GPU"
    dev = torch.device("cuda:0")
    m = bench.build_model(dev)
    if a.run_to_cap:
        with torch.no_grad():
            m.ar_predict_layer.weight[1024].fill_(-0.05)   # EOS row
            m.ar_decoder.norm.bias.fill_(1.0)
    eng = m.engine(torch.bfloat16)
    eng.quiet = True
    print(json.dumps(dict(card=card(), run_to_cap=a.run_to_cap)), flush=True)
    for B in [int(b) for b in a.batches.split(",")]:
        texts, prompts = bench.make_batch(B, 1, device=dev)
        for name, kw in MODES.items():       # warm-up: captures, allocations
            eng.generate(texts, prompts, max_new_tokens=40, **kw)
        rec = {n: [] for n in MODES}
        for _ in range(a.repeats):
            for name, kw in MODES.items():
                rec[name].append(run(eng, texts, prompts, kw))
        for name, rs in rec.items():
            out = dict(B=B, mode=name, ar_us_per_step=[round(r["ar_us_per_step"], 1) for r in rs],
                       ar_steps=[r["ar_steps"] for r in rs], frames=[r["frames"] for r in rs],
                       launches_per_step=round(statistics.mean(r["launches_per_step"] for r in rs), 2),
                       replayed_per_step=round(statistics.mean(r["replayed_per_step"] for r in rs), 2),
                       wall_ms=[round(r["wall_ms"], 1) for r in rs])
            print(json.dumps(out), flush=True)
        g = statistics.median(r["ar_us_per_step"] for r in rec["greedy"])
        for name in [n for n in MODES if n != "greedy"]:
            v = statistics.median(r["ar_us_per_step"] for r in rec[name])
            print(json.dumps(dict(B=B, mode=name, ar_us_per_step_vs_greedy=round(v / g - 1, 4))), flush=True)
        if a.profile_steps:
            print(json.dumps(dict(B=B, profile=profile(eng, texts, prompts, a.profile_steps))), flush=True)
        del texts, prompts
        eng._bufs.clear()
        torch.cuda.empty_cache()
    print(json.dumps(dict(card=card())), flush=True)


if __name__ == "__main__":
    main()
