"""Cost of post-LN VALL-E (`norm_first=False`) against pre-LN on bench.py's model and workload (d=1024/16h/12L, bf16,
S=47, 225-frame prompt): AR us per decode step at each batch size and the time of the 7 NAR passes.

    python tools/bench_post_ln.py [--batches 1,64] [--repeats 3] [--max-new 256]

Models (the same seed-0 init; the post-LN twin has no final norms):
  pre_fold      pre-LN, LayerNorm-folded decode chain (what bench.py times)
  pre_unfolded  pre-LN, VB_DECODE_FOLD=0 (8 launches per layer)
  post          post-LN chain (8 launches per layer)
Every model decodes to --max-new frames: the EOS row of ar_predict_layer is a constant -c and the norm that feeds the
head gets bias +c' (pre-LN: the final norm, post-LN: the last layer's norm2), so the EOS logit is -c c' d (the normalised
row sums to zero at init) and every step does the same work.  Each model is warmed up with one run of the timed length
(graph captures, cache capacity), then the models run in alternation `--repeats` times.  Per run: AR us per step from the engine's device events, launches per step, NAR ms.
"""
from __future__ import annotations

import argparse
import contextlib
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import bench  # noqa: E402


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


@contextlib.contextmanager
def decode_fold(on: bool):
    old = os.environ.get("VB_DECODE_FOLD")
    os.environ["VB_DECODE_FOLD"] = "1" if on else "0"
    try:
        yield
    finally:
        if old is None:
            del os.environ["VB_DECODE_FOLD"]
        else:
            os.environ["VB_DECODE_FOLD"] = old


def model(dev, norm_first: bool):
    from valle_b200.models import VALLE
    torch.manual_seed(0)
    m = VALLE(bench.D_MODEL, bench.N_HEAD, bench.N_LAYER, norm_first=norm_first, add_prenet=False, prefix_mode=1,
              share_embedding=True, nar_scale_factor=1.0, prepend_bos=False, num_quantizers=bench.N_Q).eval().to(dev)
    with torch.no_grad():
        m.ar_predict_layer.weight[1024].fill_(-0.05)     # EOS row: never drawn (see the module docstring)
        (m.ar_decoder.norm if norm_first else m.ar_decoder.layers[-1].norm2).bias.fill_(1.0)
    return m


def run(eng, fold, texts, prompts, max_new):
    n0 = eng.kernel_launches()
    with decode_fold(fold):
        out = eng.generate(texts, prompts, top_k=1, max_new_tokens=max_new, return_device=True)
    torch.cuda.synchronize()
    st = eng.stats
    steps = max(1, st.ar_steps)
    return dict(ar_us_per_step=1e3 * st.ar_ms / steps, ar_steps=st.ar_steps, nar_ms=st.nar_ms,
                launches_per_step=(eng.kernel_launches() - n0) / steps, frames=sum(int(o.shape[0]) for o in out))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="1,64")
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--max-new", type=int, default=256)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "tools/bench_post_ln.py needs a GPU"
    dev = torch.device("cuda:0")
    print(json.dumps(dict(card=card(), max_new=a.max_new)), flush=True)
    pre, post = model(dev, True), model(dev, False)
    with decode_fold(True):
        e_fold = pre.engine(torch.bfloat16)
    pre_u = model(dev, True)
    with decode_fold(False):
        e_unf = pre_u.engine(torch.bfloat16)
    e_post = post.engine(torch.bfloat16)
    engines = {"pre_fold": (e_fold, True), "pre_unfolded": (e_unf, False), "post": (e_post, True)}
    for e, _ in engines.values():
        e.quiet = True
    for B in [int(b) for b in a.batches.split(",")]:
        texts, prompts = bench.make_batch(B, 1, device=dev)
        for e, fold in engines.values():     # warm-up at the timed length: graph captures, cache capacity, allocations
            run(e, fold, texts, prompts, a.max_new)
        rec = {n: [] for n in engines}
        for _ in range(a.repeats):
            for name, (e, fold) in engines.items():
                rec[name].append(run(e, fold, texts, prompts, a.max_new))
        for name, rs in rec.items():
            print(json.dumps(dict(B=B, model=name, ar_us_per_step=[round(r["ar_us_per_step"], 1) for r in rs],
                                  nar_ms=[round(r["nar_ms"], 2) for r in rs], ar_steps=[r["ar_steps"] for r in rs],
                                  frames=[r["frames"] for r in rs],
                                  launches_per_step=round(statistics.mean(r["launches_per_step"] for r in rs), 2))),
                  flush=True)
        med = {n: statistics.median(r["ar_us_per_step"] for r in rs) for n, rs in rec.items()}
        print(json.dumps(dict(B=B, post_vs_pre_unfolded=round(med["post"] / med["pre_unfolded"] - 1, 4),
                              post_vs_pre_fold=round(med["post"] / med["pre_fold"] - 1, 4))), flush=True)
        for e, _ in engines.values():
            e._bufs.clear()
        torch.cuda.empty_cache()
    print(json.dumps(dict(card=card())), flush=True)


if __name__ == "__main__":
    main()
