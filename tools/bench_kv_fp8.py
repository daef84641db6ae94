"""FP8 (e4m3) against bf16 KV cache on the bf16 AR decode (VALLE.kv_cache_dtype), the two cache modes alternating
within one run, on the benchmark model (d=1024/16h/12L, bf16, seeded init as bench.py builds it).

    python tools/bench_kv_fp8.py [--reps 5] [--out results.json]

  * AR step time, B=64 at contexts ~300 / 700 / 1000: the prefill fills the cache, then CUDA-graph replays of 8 decode
    steps are timed with CUDA events (n_gen reset before every replay, so the context stays put); bytes per step from
    the shapes: W + B (KV_read(L) + KV_write), and the bytes/s that achieves.
  * Whole decode: the bench.py workload (64 x S=47, 225-frame prompt -> 753 frames) through inference_batch: audio
    tokens/s, AR ms, NAR ms.
  * Accuracy on that workload: teacher-forced AR logits of the FP8 cache against the bf16 cache (max / mean |d|, argmax
    agreement) and the first step at which free-running greedy codes diverge.
The card name and power limit are printed with the numbers."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import bench  # noqa: E402

F8 = torch.float8_e4m3fn
B = 64


def card():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader"],
                            capture_output=True, text=True, timeout=20).stdout.strip()
    except Exception:   # noqa: BLE001
        pl = "unknown"
    return name, pl


def step_bytes(model, ctx, kv):
    """W + B (KV_read(ctx) + KV_write) of one decode step, from the shapes"""
    d, L, H = bench.D_MODEL, bench.N_LAYER, bench.N_HEAD
    dff = 4 * d
    W = (L * (4 * d * d + 2 * d * dff) + 1025 * d) * 2
    per_tok = L * H * 64 * 2 * (1 if kv == F8 else 2) + (L * H * 2 if kv == F8 else 0)
    return W + B * (ctx * per_tok + per_tok)


def ar_step_times(model, ctxs, reps):
    eng = model.engine()
    out = {}
    for ctx in ctxs:
        g = torch.Generator().manual_seed(ctx)
        texts = [torch.randint(3, 100, (bench.S_TEXT,), generator=g) for _ in range(B)]
        prompts = [torch.randint(0, 1024, (ctx - bench.S_TEXT, bench.N_Q), generator=g) for _ in range(B)]
        res = {}
        for rep in range(reps):
            for kv in (None, F8):          # alternate the two modes
                model.kv_cache_dtype = kv
                eng._bufs.clear()              # the buffer generate() fills below is then the only one
                eng.generate(texts, prompts, top_k=1, max_new_tokens=40, return_device=True)
                (buf,) = eng._bufs.values()
                assert buf.kv_dtype == kv and int(buf.text_len[0] + buf.prompt_len[0]) == ctx
                head = eng._head_ref
                head.greedy = 1
                times = []
                for it in range(4):
                    buf.n_gen.zero_()
                    buf.finished.zero_()
                    buf.max_new.fill_(1 << 20)
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    eng._replay_steps(buf, head, 8)
                    e1.record()
                    e1.synchronize()
                    if it > 0:                 # the first call captures the graph
                        times.append(e0.elapsed_time(e1) / 8)
                live = int((buf.finished == 0).sum())   # a row that stopped would skip its attention
                assert live == B, f"{B - live} rows stopped during the timed steps"
                res.setdefault(str(kv), []).append(sorted(times)[len(times) // 2])
        out[ctx] = {}
        for kv in (None, F8):
            ms = sorted(res[str(kv)])[len(res[str(kv)]) // 2]   # median over the repetitions
            nb = step_bytes(model, ctx, kv)
            out[ctx]["fp8" if kv else "bf16"] = dict(step_us=ms * 1e3, all_us=[round(t * 1e3, 1) for t in res[str(kv)]],
                                                     bytes=nb, GBps=nb / (ms * 1e-3) / 1e9)
    model.kv_cache_dtype = None
    return out


def whole_decode(model, reps):
    eng = model.engine()
    texts, prompts = bench.make_batch(B, 1, torch.device("cuda:0"))
    out = {}
    for rep in range(reps + 1):
        for kv in (None, F8):
            model.kv_cache_dtype = kv
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            codes = model.inference_batch(texts, prompts, top_k=1, dtype=torch.bfloat16, return_device=True)
            e1.record()
            e1.synchronize()
            if rep == 0:
                continue            # warm-up (graph capture)
            ms = e0.elapsed_time(e1)
            n = sum(int(c.shape[0]) for c in codes)
            r = out.setdefault("fp8" if kv else "bf16", [])
            r.append(dict(tokens_per_s=n * bench.N_Q / (ms * 1e-3), wall_ms=ms, ar_ms=eng.stats.ar_ms,
                          nar_ms=eng.stats.nar_ms, frames=n))
    model.kv_cache_dtype = None
    return out


def accuracy(model):
    eng = model.engine()
    texts, prompts = bench.make_batch(B, 1, torch.device("cuda:0"))
    model.kv_cache_dtype = None
    free16 = eng.generate(texts, prompts, top_k=1, return_device=False)
    model.kv_cache_dtype = F8
    free8 = eng.generate(texts, prompts, top_k=1, return_device=False)
    first = []
    for a, b in zip(free16, free8):
        n = min(a.shape[0], b.shape[0])
        diff = (a[:n, 0] != b[:n, 0]).nonzero()
        first.append(int(diff[0]) if diff.numel() else n)
    # teacher forcing with the bf16 cache's codes, on a few utterances (forced decodes run one step per launch)
    errs, agree, tot = [], 0, 0
    for b in range(4):
        logits = {}
        for kv in (None, F8):
            model.kv_cache_dtype = kv
            tr = {"steps": "all"}
            eng.generate([texts[b]], [prompts[b]], top_k=1, trace=tr, forced=[free16[b]])
            logits[kv] = torch.stack([tr["ar_logits"][i][0].float().cpu() for i in sorted(tr["ar_logits"])])
        d = (logits[F8] - logits[None]).abs()
        errs.append(d)
        agree += int((logits[F8].argmax(1) == logits[None].argmax(1)).sum())
        tot += d.shape[0]
    model.kv_cache_dtype = None
    allerr = torch.cat(errs)
    return dict(tf_utterances=4, tf_steps=tot, max_abs_dlogit=float(allerr.max()), mean_abs_dlogit=float(allerr.mean()),
                argmax_agreement=agree / tot, free_running_first_divergence=first,
                identical_utterances=sum(int(torch.equal(a, b)) for a, b in zip(free16, free8)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    model = bench.build_model(dev)
    model.engine_dtype = torch.bfloat16
    model.engine().quiet = True
    name, pl = card()
    print(f"card: {name}, power limit {pl}")
    res = {"card": name, "power_limit": pl}
    res["ar_step"] = ar_step_times(model, (300, 700, 1000), a.reps)
    for ctx, r in res["ar_step"].items():
        print(f"ctx {ctx}: bf16 {r['bf16']['step_us']:.1f} us ({r['bf16']['bytes'] / 1e9:.3f} GB, "
              f"{r['bf16']['GBps']:.0f} GB/s) | fp8 {r['fp8']['step_us']:.1f} us ({r['fp8']['bytes'] / 1e9:.3f} GB, "
              f"{r['fp8']['GBps']:.0f} GB/s)")
    res["whole_decode"] = whole_decode(model, max(1, a.reps // 2))
    for k, rs in res["whole_decode"].items():
        print(f"whole decode {k}: " + "; ".join(f"{r['tokens_per_s'] / 1e3:.1f}k tok/s AR {r['ar_ms']:.1f} ms "
                                                 f"NAR {r['nar_ms']:.1f} ms" for r in rs))
    res["accuracy"] = accuracy(model)
    acc = res["accuracy"]
    print(f"accuracy: teacher-forced max |dlogit| {acc['max_abs_dlogit']:.4f} mean {acc['mean_abs_dlogit']:.5f} "
          f"argmax agreement {acc['argmax_agreement']:.4f} over {acc['tf_steps']} steps; free-running identical "
          f"{acc['identical_utterances']}/64, first divergence min {min(acc['free_running_first_divergence'])}")
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
