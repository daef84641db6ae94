"""Continuous batching against static batches on bench.py's model (d=1024/16h/12L, bf16, 47-phoneme texts, 225-frame
prompts), N requests in 64 decode slots.

Two workloads: (1) a length mix, max_new_tokens drawn from a seeded U[75, 752] (1-10 s of audio); (2) bench.py's
uniform workload, every utterance cap-terminated at 753 frames, where the stream has nothing to gain and any loss is
admission or poll overhead.  Three schedules: inference_batch in input order (groups of 64), inference_batch
longest-first, inference_stream.  They alternate, three repetitions each; the stream's `poll` is the best of 8 / 16 /
32 on workload 1.  The three schedules must return identical codes.

    python tools/bench_stream.py [--n 256] [--reps 3] [--out results.json]
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
from valle_b200.engine import StreamRequest  # noqa: E402

SLOTS = 64


def card():
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        q = f"nvidia-smi unavailable ({e})"
    return {"torch_name": torch.cuda.get_device_name(0), "nvidia_smi": q}


def run(eng, sched, texts, prompts, mnt, poll):
    """one schedule over the whole workload: (codes in request order, wall ms, engine stats, decode steps, occupancy)"""
    n = len(texts)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    steps = ar = pre = nar = 0.0
    if sched == "stream":
        reqs = [StreamRequest(t, p, max_new_tokens=k) for t, p, k in zip(texts, prompts, mnt)]
        out = [None] * n
        for i, c in eng.generate_stream(reqs, slots=SLOTS, poll=poll):
            out[i] = c
        st = eng.stats
        steps, ar, pre, nar = st.ar_steps, st.ar_ms, st.prefill_ms, st.nar_ms
    else:
        order = list(range(n)) if sched == "input_order" else sorted(range(n), key=lambda i: -mnt[i])
        out = [None] * n
        for b0 in range(0, n, SLOTS):
            ids = order[b0:b0 + SLOTS]
            cs = eng.generate([texts[i] for i in ids], [prompts[i] for i in ids], top_k=1,
                              max_new_tokens=[mnt[i] for i in ids], return_device=True)
            for i, c in zip(ids, cs):
                out[i] = c
            steps += eng.stats.ar_steps
            ar += eng.stats.ar_ms
            pre += eng.stats.prefill_ms
            nar += eng.stats.nar_ms
    torch.cuda.synchronize()
    ms = (time.perf_counter() - t0) * 1000.0
    frames = sum(int(c.shape[0]) for c in out)
    return out, {"sched": sched, "poll": poll if sched == "stream" else None, "wall_ms": ms,
                 "audio_tokens_per_s": frames * bench.N_Q / (ms / 1000.0), "ar_ms": ar, "prefill_ms": pre,
                 "nar_ms": nar, "decode_steps": int(steps), "frames": frames,
                 "occupancy": frames / (steps * SLOTS) if steps else None}


def workload(eng, name, texts, prompts, mnt, reps, polls):
    res = {"workload": name, "runs": []}
    ref = None

    def check(out, sched):
        nonlocal ref
        if ref is None:
            ref = [c.cpu() for c in out]
            return
        bad = [i for i, (a, b) in enumerate(zip(out, ref)) if not torch.equal(a.cpu(), b)]
        assert not bad, f"{name}: {sched} differs from the first schedule at requests {bad[:8]}"

    # warm-up: every shape the timed runs use (graphs, cache buffers, GEMM shapes)
    for sched in ("input_order", "longest_first", "stream"):
        for p in (polls if sched == "stream" else [None]):
            check(run(eng, sched, texts, prompts, mnt, p)[0], sched)
    poll = polls[0]
    if len(polls) > 1:
        best = {p: run(eng, "stream", texts, prompts, mnt, p)[1] for p in polls}
        res["poll_sweep"] = {p: r["audio_tokens_per_s"] for p, r in best.items()}
        poll = max(best, key=lambda p: best[p]["audio_tokens_per_s"])
    res["poll"] = poll
    for _ in range(reps):
        for sched in ("input_order", "longest_first", "stream"):
            out, r = run(eng, sched, texts, prompts, mnt, poll)
            check(out, sched)
            res["runs"].append(r)
    summary = {}
    for sched in ("input_order", "longest_first", "stream"):
        rs = [r for r in res["runs"] if r["sched"] == sched]
        summary[sched] = {k: (statistics.median(r[k] for r in rs) if k != "sched" else sched)
                          for k in ("audio_tokens_per_s", "wall_ms", "ar_ms", "prefill_ms", "nar_ms", "decode_steps",
                                    "occupancy")}
        summary[sched]["tokens_per_s_min_max"] = [min(r["audio_tokens_per_s"] for r in rs),
                                                  max(r["audio_tokens_per_s"] for r in rs)]
    res["summary"] = summary
    res["codes_identical"] = True
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=256)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_stream.py measures on the GPU; no CUDA device found")
    dev = torch.device("cuda:0")
    model = bench.build_model(dev)
    eng = model.engine(torch.bfloat16)
    eng.quiet = True
    texts, prompts = bench.make_batch(a.n, 1, device=dev)
    g = torch.Generator().manual_seed(a.seed)
    mix = [int(v) for v in torch.randint(75, 753, (a.n,), generator=g)]
    out = {"card": card(), "n": a.n, "slots": SLOTS, "seed": a.seed,
           "mix_lower_bound_steps": sum(k - 1 for k in mix) / SLOTS}
    out["mix"] = workload(eng, "mix U[75, 752]", texts, prompts, mix, a.reps, [8, 16, 32])
    uni = [bench.FRAMES] * a.n
    out["uniform"] = workload(eng, "uniform, cap-terminated", texts, prompts, uni, a.reps, [out["mix"]["poll"]])
    line = json.dumps(out)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
