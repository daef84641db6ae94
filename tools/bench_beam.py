"""Beam search against independent greedy rows on bench.py's model and workload (d=1024/16h/12L, bf16, S=47,
225-frame prompt, up to 753 frames).

    python tools/bench_beam.py [--ns 1,2,4,8,16] [--repeats 3]

For each n: 64 / n utterances, n beams each (64 decode rows).
  beam    generate(texts, prompts, num_beams=n): the beams read one copy of the prompt prefix, follow their ancestry in
          the decode attention and are pruned by the beam tail inside the CUDA-graph step
  greedy  generate() on the list with every utterance repeated n times: the same 64 rows decoded as independent
          greedy rows
Both are warmed up, then run in alternation `--repeats` times.  Every row runs to the cap: the EOS row of
ar_predict_layer becomes -c and the final LayerNorm's bias +c', so the EOS logit is a constant far below the others
(tools/bench_best_of.py does the same).  Per run: AR us per decode step from the engine's device events and decoded
first-codebook tokens per second of AR time (64 rows per step, whichever mode).  Then the beam tail's own kernel time,
from torch.profiler over 50 tail launches on the beam run's rows.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import bench  # noqa: E402
from valle_b200 import _lib as L  # noqa: E402


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def run(eng, texts, prompts, n, beam):
    if beam:
        eng.generate(texts, prompts, return_device=True, num_beams=n)
    else:
        eng.generate([t for t in texts for _ in range(n)], [p for p in prompts for _ in range(n)], return_device=True)
    torch.cuda.synchronize()
    st = eng.stats
    return dict(ar_us_per_step=1e3 * st.ar_ms / max(1, st.ar_steps), ar_steps=st.ar_steps,
                ar_tokens_per_s=64 * st.ar_steps / (st.ar_ms / 1e3))


def tail_us(eng, n):
    """mean device time of the beam tail kernel over 50 launches on the last beam run's 64 rows (every group reset
    to a running mid-sequence step before each launch)"""
    buf = next(b for b in eng._bufs.values() if b.st.beam_width == n)
    head = eng._head_ref
    lib = eng.lib
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(50):
            buf.finished.zero_()
            buf.n_gen.fill_(400)
            L.check(lib.vb_ar_beam_step(C.byref(head), C.byref(buf.st), eng.d, None, L.stream_ptr()),
                    "vb_ar_beam_step")
        torch.cuda.synchronize()
    ts = [e.device_time_total / e.count for e in prof.key_averages() if "ar_beam_kernel" in e.key]
    return round(ts[0], 2) if ts else None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ns", default="1,2,4,8,16")
    ap.add_argument("--repeats", type=int, default=3)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "tools/bench_beam.py needs a GPU"
    dev = torch.device("cuda:0")
    m = bench.build_model(dev)
    with torch.no_grad():                        # run every row to the cap
        m.ar_predict_layer.weight[1024].fill_(-0.05)
        m.ar_decoder.norm.bias.fill_(1.0)
    eng = m.engine(torch.bfloat16)
    eng.quiet = True
    print(json.dumps(dict(card=card())), flush=True)
    for n in [int(x) for x in a.ns.split(",")]:
        texts, prompts = bench.make_batch(64 // n, 1, device=dev)
        for beam in (True, False):               # warm-up: captures, allocations
            run(eng, texts, prompts, n, beam)
        rec = {"beam": [], "greedy": []}
        for _ in range(a.repeats):
            rec["beam"].append(run(eng, texts, prompts, n, True))
            rec["greedy"].append(run(eng, texts, prompts, n, False))
        out = dict(n=n, utterances=64 // n)
        for mode, rs in rec.items():
            out[mode] = dict(ar_us_per_step=[round(r["ar_us_per_step"], 1) for r in rs],
                             ar_steps=[r["ar_steps"] for r in rs],
                             ar_tokens_per_s=[round(r["ar_tokens_per_s"]) for r in rs])
        b = statistics.median(r["ar_us_per_step"] for r in rec["beam"])
        g = statistics.median(r["ar_us_per_step"] for r in rec["greedy"])
        out["ar_us_per_step_beam_vs_greedy"] = round(b / g - 1, 4)
        if n > 1:
            eng.generate(texts, prompts, return_device=True, num_beams=n)
            out["beam_tail_us"] = tail_us(eng, n)
        print(json.dumps(out), flush=True)
        del texts, prompts
        eng._bufs.clear()
        torch.cuda.empty_cache()
    print(json.dumps(dict(card=card())), flush=True)


if __name__ == "__main__":
    main()
