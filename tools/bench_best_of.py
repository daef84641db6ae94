"""Best-of-n decoding against the repeated list on bench.py's model and workload (d=1024/16h/12L, bf16, S=47,
225-frame prompt, up to 753 frames).

    python tools/bench_best_of.py [--ns 1,2,4,8] [--repeats 3] [--kv bf16,fp8]

For each KV cache and n: 64 / n utterances, n candidates each (64 decode rows), seeded top-k 50 / temperature 0.8.
  shared    generate(texts, prompts, seed=s, num_samples=n): on the bf16 cache the candidates read one copy of the
            prompt prefix; on the FP8 cache, where that is slower, the engine runs the repeated list's step
  repeated  generate() on the list with every utterance repeated n times and the same seeds: every row reads its own
Both are warmed up, then run in alternation `--repeats` times.  Every candidate runs to the cap: the EOS row of
ar_predict_layer becomes -c and the final LayerNorm's bias +c', so the EOS logit is a constant far below the others
and EOS is never drawn (tools/bench_sampling.py --run-to-cap).  Per run: AR us per decode step and NAR ms from the
engine's device events, audio tokens/s (codes of every codebook over the wall time of a synchronised generate()),
and whether the two modes' codes are identical.
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

KW = dict(top_k=50, temperature=0.8, seed=1234)


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def run(eng, texts, prompts, n, shared):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    if shared:
        out = eng.generate(texts, prompts, return_device=True, num_samples=n, **KW)
        out = [c for cands in out for c in cands] if n > 1 else out
    else:
        out = eng.generate([t for t in texts for _ in range(n)], [p for p in prompts for _ in range(n)],
                           return_device=True, **KW)
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    st = eng.stats
    tokens = sum(int(o.numel()) for o in out)
    return dict(ar_us_per_step=1e3 * st.ar_ms / max(1, st.ar_steps), ar_steps=st.ar_steps, nar_ms=st.nar_ms,
                tokens_per_s=tokens / wall, wall_ms=1e3 * wall), out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ns", default="1,2,4,8")
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--kv", default="bf16,fp8")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "tools/bench_best_of.py needs a GPU"
    dev = torch.device("cuda:0")
    m = bench.build_model(dev)
    with torch.no_grad():                        # run every candidate to the cap
        m.ar_predict_layer.weight[1024].fill_(-0.05)
        m.ar_decoder.norm.bias.fill_(1.0)
    eng = m.engine(torch.bfloat16)
    eng.quiet = True
    print(json.dumps(dict(card=card(), sampler=KW)), flush=True)
    for kv in a.kv.split(","):
        m.kv_cache_dtype = torch.float8_e4m3fn if kv == "fp8" else None
        for n in [int(x) for x in a.ns.split(",")]:
            texts, prompts = bench.make_batch(64 // n, 1, device=dev)
            for shared in (True, False):         # warm-up: captures, allocations
                run(eng, texts, prompts, n, shared)
            rec = {"shared": [], "repeated": []}
            same = True
            for _ in range(a.repeats):
                rs, cs = run(eng, texts, prompts, n, True)
                rr, cr = run(eng, texts, prompts, n, False)
                rec["shared"].append(rs)
                rec["repeated"].append(rr)
                same = same and len(cs) == len(cr) and all(torch.equal(x, y) for x, y in zip(cs, cr))
            for mode, rs in rec.items():
                print(json.dumps(dict(kv=kv, n=n, utterances=64 // n, mode=mode,
                                      ar_us_per_step=[round(r["ar_us_per_step"], 1) for r in rs],
                                      ar_steps=[r["ar_steps"] for r in rs],
                                      nar_ms=[round(r["nar_ms"], 1) for r in rs],
                                      tokens_per_s=[round(r["tokens_per_s"]) for r in rs],
                                      wall_ms=[round(r["wall_ms"], 1) for r in rs])), flush=True)
            s = statistics.median(r["ar_us_per_step"] for r in rec["shared"])
            r = statistics.median(r["ar_us_per_step"] for r in rec["repeated"])
            print(json.dumps(dict(kv=kv, n=n, ar_us_per_step_shared_vs_repeated=round(s / r - 1, 4),
                                  codes_identical=same)), flush=True)
            del texts, prompts
            eng._bufs.clear()
            torch.cuda.empty_cache()
    m.kv_cache_dtype = None
    print(json.dumps(dict(card=card())), flush=True)


if __name__ == "__main__":
    main()
