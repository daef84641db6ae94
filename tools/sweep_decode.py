"""In-process A/B sweep of the AR decode step's tuning knobs (vb_tune_set): one model build, one engine, the CUDA graph
re-captured per configuration; prints the AR-phase time of a full decode per configuration.

    python tools/sweep_decode.py B FRAMES "K1=v,K2=v" "K1=v" ...      ("" = defaults)

The decode chain is the engine's choice, made once when it builds the weights: VB_DECODE_FOLD=0 in the environment
of the run sweeps the unfolded chain.
"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

import bench  # noqa: E402
from valle_b200 import _lib  # noqa: E402

B, frames = int(sys.argv[1]), int(sys.argv[2])
cfgs = sys.argv[3:] or [""]
lib = _lib.load()
dev = torch.device("cuda:0")
model = bench.build_model(dev)
eng = model.engine(torch.bfloat16)
eng.quiet = True
texts, prompts = bench.make_batch(B, 0, dev)
mnt = None if frames >= bench.FRAMES else frames
touched = {}
res = []
for rep in range(int(os.environ.get("SWEEP_REPS", "2"))):
    for c in cfgs:
        for k in touched:                      # back to defaults
            lib.vb_tune_set(k.encode(), touched[k])
        kv = dict(x.split("=") for x in c.split(",") if x)
        for k, v in kv.items():
            touched.setdefault(k, {"VB_KV_PREFETCH_L2_PCT": 60}.get(k, 0))
            lib.vb_tune_set(k.encode(), int(v))
        eng._bufs.clear()
        eng.generate(texts, prompts, top_k=1, max_new_tokens=min(40, frames), return_device=True)   # capture
        eng.generate(texts, prompts, top_k=1, max_new_tokens=mnt, return_device=True)
        torch.cuda.synchronize()
        r = dict(cfg=c, rep=rep, ar_ms=eng.stats.ar_ms, steps=eng.stats.ar_steps,
                 us_per_step=1000 * eng.stats.ar_ms / max(1, eng.stats.ar_steps), nar_ms=eng.stats.nar_ms)
        res.append(r)
        print(json.dumps(r), flush=True)
