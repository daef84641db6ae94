"""Continuous batching against static batches on bench.py's model (d=1024/16h/12L, bf16, 47-phoneme texts, 225-frame
prompts), N requests in 64 decode slots.

Three workloads: (1) a length mix, max_new_tokens drawn from a seeded U[75, 752] (1-10 s of audio); (2) bench.py's
uniform workload, every utterance cap-terminated at 753 frames, where the stream has nothing to gain and any loss is
admission or poll overhead; (3) the length mix with every eighth request a num_beams=4 beam search.  Workloads 1 and 2
run three schedules: inference_batch in input order (groups of 64), inference_batch longest-first, inference_stream.
Workload 3 runs two: (a) one stream of every request, the beam groups decoding next to the other requests, and (b)
what a server did before the stream took beam requests: the stream over the other requests, then
generate(num_beams=4) over the beam requests (groups of 16 utterances, 64 rows).  The schedules alternate, three
repetitions each; the stream's `poll` is the best of 8 / 16 / 32 on workload 1.  Every schedule of a workload must
return identical codes.  Last, the decode step at 64 running slots, timed with CUDA events over graph replays: the
seeded head (vb_ar_head.greedy == 2) against the mixed head (4) with no beam group present, the cost a stream pays
from its first beam request on.

--only best_of: the length mix with every eighth request a seeded BestOfRequest(..., 4) (top-k 50, temperature 0.8),
three schedules alternating: (a) one stream, each best-of request prefilled once and its candidates reading that
prefix; (b) the same candidates as four independent seeded StreamRequests each (seeds s + j), which must return the
same codes; (c) the stream over the other requests, then generate(num_samples=4) over the best-of requests.  Then the
decode step at 64 running slots with and without scores (vb_ar_state.logprob), the cost return_scores=True adds.

    python tools/bench_stream.py [--n 256] [--reps 3] [--out results.json] [--only beams|best_of]
"""
from __future__ import annotations

import argparse
import ctypes as C
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
from valle_b200 import _lib as L  # noqa: E402
from valle_b200.engine import BestOfRequest, StreamRequest, _ArBuffers, _draws  # noqa: E402

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


def run_beams(eng, sched, texts, prompts, mnt, beam, poll):
    """workload 3: (a) "mixed", one stream of every request; (b) "separate", the stream over the requests not in
    `beam`, then generate(num_beams=4) over those in it"""
    n = len(texts)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = [None] * n
    reqs = [StreamRequest(t, p, max_new_tokens=k, num_beams=4 if i in beam else 1)
            for i, (t, p, k) in enumerate(zip(texts, prompts, mnt))]
    ids = list(range(n)) if sched == "mixed" else [i for i in range(n) if i not in beam]
    for j, c in eng.generate_stream([reqs[i] for i in ids], slots=SLOTS, poll=poll):
        out[ids[j]] = c
    if sched == "separate":
        bs = sorted(beam)
        cs = eng.generate([texts[i] for i in bs], [prompts[i] for i in bs], max_new_tokens=[mnt[i] for i in bs],
                          num_beams=4, return_device=True)
        for i, c in zip(bs, cs):
            out[i] = c
    torch.cuda.synchronize()
    ms = (time.perf_counter() - t0) * 1000.0
    frames = sum(int(c.shape[0]) for c in out)
    return out, {"sched": sched, "wall_ms": ms, "audio_tokens_per_s": frames * bench.N_Q / (ms / 1000.0),
                 "frames": frames}


def beam_workload(eng, texts, prompts, mnt, reps, poll):
    beam = {i for i in range(len(texts)) if i % 8 == 7}
    res = {"workload": "mix U[75, 752], every eighth request num_beams=4", "poll": poll, "beam_requests": len(beam),
           "runs": []}
    ref = {}
    for _ in range(reps + 1):               # the first round warms up every shape (graphs, buffers)
        for sched in ("mixed", "separate"):
            out, r = run_beams(eng, sched, texts, prompts, mnt, beam, poll)
            if ref:
                bad = [i for i, (a, b) in enumerate(zip(out, ref["codes"])) if not torch.equal(a.cpu(), b)]
                assert not bad, f"beams: {sched} differs from the mixed stream at requests {bad[:8]}"
            else:
                ref["codes"] = [c.cpu() for c in out]
            res["runs"].append(r)
    res["runs"] = res["runs"][2:]
    res["summary"] = {sched: {"audio_tokens_per_s": statistics.median(r["audio_tokens_per_s"] for r in rs),
                              "tokens_per_s_min_max": [min(r["audio_tokens_per_s"] for r in rs),
                                                       max(r["audio_tokens_per_s"] for r in rs)],
                              "wall_ms": statistics.median(r["wall_ms"] for r in rs)}
                      for sched in ("mixed", "separate")
                      for rs in [[r for r in res["runs"] if r["sched"] == sched]]}
    res["codes_identical"] = True
    return res


def run_best_of(eng, sched, texts, prompts, mnt, best, poll):
    """the best_of workload: (a) "stream", every request in one stream, best-of requests as BestOfRequest(r, 4); (b)
    "copies", each best-of request as 4 seeded StreamRequests; (c) "separate", the stream over the other requests,
    then generate(num_samples=4) over the best-of requests.  Codes: one [T, Q] per plain request, a list of 4 per
    best-of request."""
    n = len(texts)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = [None] * n
    reqs = [StreamRequest(t, p, max_new_tokens=k, seed=1000 * i if i in best else None, top_k=50 if i in best else 1,
                          temperature=0.8 if i in best else 1.0) for i, (t, p, k) in enumerate(zip(texts, prompts, mnt))]
    pre = 0.0
    if sched == "stream":
        items, owner = [BestOfRequest(r, 4) if i in best else r for i, r in enumerate(reqs)], list(range(n))
    elif sched == "copies":
        items, owner = [], []
        for i, r in enumerate(reqs):
            for j in range(4 if i in best else 1):
                items.append(r._replace(seed=r.seed + j) if i in best else r)
                owner.append(i)
    else:
        owner = [i for i in range(n) if i not in best]
        items = [reqs[i] for i in owner]
    for j, c in eng.generate_stream(items, slots=SLOTS, poll=poll):
        i = owner[j]
        if sched == "copies" and i in best:
            out[i] = (out[i] or []) + [(items[j].seed, c)]
        else:
            out[i] = c
    pre += eng.stats.prefill_ms
    if sched == "copies":
        out = [sorted(o, key=lambda sc: sc[0]) if isinstance(o, list) else o for o in out]
        out = [[c for _, c in o] if isinstance(o, list) else o for o in out]
    if sched == "separate":
        bs = sorted(best)
        cs = eng.generate([texts[i] for i in bs], [prompts[i] for i in bs], max_new_tokens=[mnt[i] for i in bs],
                          seed=[reqs[i].seed for i in bs], top_k=50, temperature=0.8, num_samples=4, return_device=True)
        pre += eng.stats.prefill_ms
        for i, c in zip(bs, cs):
            out[i] = c
    torch.cuda.synchronize()
    ms = (time.perf_counter() - t0) * 1000.0
    frames = sum(sum(int(x.shape[0]) for x in c) if isinstance(c, list) else int(c.shape[0]) for c in out)
    return out, {"sched": sched, "wall_ms": ms, "audio_tokens_per_s": frames * bench.N_Q / (ms / 1000.0),
                 "prefill_ms": pre, "frames": frames}


def best_of_workload(eng, texts, prompts, mnt, reps, poll):
    best = {i for i in range(len(texts)) if i % 8 == 7}
    scheds = ("stream", "copies", "separate")
    res = {"workload": "mix U[75, 752], every eighth request BestOfRequest(top_k=50, temperature=0.8, n=4)",
           "poll": poll, "best_of_requests": len(best), "runs": []}

    def flat(out):
        return [x.cpu() for c in out for x in (c if isinstance(c, list) else [c])]
    ref = None
    same_as_separate = True
    for rep in range(reps + 1):             # the first round warms up every shape (graphs, buffers)
        for sched in scheds:
            out, r = run_best_of(eng, sched, texts, prompts, mnt, best, poll)
            codes = flat(out)
            if ref is None:
                ref = codes
            elif sched == "separate":       # generate()'s decode groups may round a row's attention differently
                same_as_separate &= len(codes) == len(ref) and all(torch.equal(a, b) for a, b in zip(codes, ref))
            else:
                bad = [i for i, (a, b) in enumerate(zip(codes, ref)) if not torch.equal(a, b)]
                assert len(codes) == len(ref) and not bad, f"best_of: {sched} differs from the stream at {bad[:8]}"
            if rep:
                res["runs"].append(r)
    res["summary"] = {sched: {k: statistics.median(r[k] for r in rs) for k in ("audio_tokens_per_s", "wall_ms",
                                                                              "prefill_ms")}
                      | {"tokens_per_s_min_max": [min(r["audio_tokens_per_s"] for r in rs),
                                                  max(r["audio_tokens_per_s"] for r in rs)]}
                      for sched in scheds for rs in [[r for r in res["runs"] if r["sched"] == sched]]}
    res["codes_identical_stream_copies"] = True
    res["codes_identical_separate"] = bool(same_as_separate)
    return res


def step_times(eng, texts, prompts, reps, steps=128, cases=(("greedy2", 2, False), ("greedy4", 4, False))):
    """ms per decode step at SLOTS running rows (each capped at bench.FRAMES), graphs of 8 steps, alternating between
    the cases (label, head, scores): by default the seeded head (greedy == 2) and the mixed head (greedy == 4, every
    row in no group); scores: the state points at logprob"""
    m = eng.model
    dev = eng.device
    cap = (max(int(t.numel()) + int(p.shape[0]) for t, p in zip(texts, prompts)) + bench.FRAMES + 2 + 63) // 64 * 64
    ts = (bench.FRAMES + 2 + 7) // 8 * 8
    pe_a = eng._pe(m.ar_audio_position, cap + 2)
    runs = {}
    for label, greedy, scores in cases:
        buf = _ArBuffers(eng, SLOTS, cap, ts)
        p = eng._prefill_inputs(texts[:SLOTS], prompts[:SLOTS], [bench.FRAMES] * SLOTS)
        buf.load_rows(p, _draws(SLOTS, 0, 1, 1.0))
        buf.n_gen.zero_()
        buf.finished.zero_()
        buf.set_best_of(SLOTS, 1, scores)
        if greedy == 4:
            buf.set_groups()
        h = eng._prefill(buf, p, pe_a)
        head = eng._head(pe_a, greedy)
        L.check(eng.lib.vb_ar_head_step(eng.ar.handle, C.byref(head), h.data_ptr(), C.byref(buf.st),
                                        buf.ws.data_ptr(), buf.ws.numel(), L.stream_ptr()), "vb_ar_head_step")
        eng._device_steps(buf, head, 16)    # capture + warm-up
        runs[label] = (buf, head)
    out = {label: [] for label in runs}
    for _ in range(reps):
        for label, (buf, head) in runs.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            eng._device_steps(buf, head, steps)
            e1.record()
            e1.synchronize()
            out[label].append(e0.elapsed_time(e1) / steps)
    assert all(int(b.finished.sum()) == 0 for b, _ in runs.values()), "a row stopped inside the timed steps"
    torch.cuda.synchronize(dev)
    res = {"slots": SLOTS, "steps_per_rep": steps}
    for label, ms in out.items():
        res[f"ms_per_step_{label}"] = ms
        res[f"median_{label}"] = statistics.median(ms)
    return res


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
    ap.add_argument("--only", choices=["all", "beams", "best_of"], default="all",
                    help="beams: workload 3 and the decode-step times only; best_of: the best-of workload and the "
                         "decode step with and without scores (the stream's poll: --poll)")
    ap.add_argument("--poll", type=int, default=16)
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
    if a.only == "beams":
        out["beams"] = beam_workload(eng, texts, prompts, mix, a.reps, a.poll)
        out["decode_step"] = step_times(eng, texts, prompts, a.reps)
        out["card_after"] = card()
        return emit(out, a.out)
    if a.only == "best_of":
        out["best_of"] = best_of_workload(eng, texts, prompts, mix, a.reps, a.poll)
        out["decode_step"] = step_times(eng, texts, prompts, a.reps,
                                        cases=(("greedy2", 2, False), ("greedy2_scores", 2, True)))
        out["card_after"] = card()
        return emit(out, a.out)
    out["mix"] = workload(eng, "mix U[75, 752]", texts, prompts, mix, a.reps, [8, 16, 32])
    uni = [bench.FRAMES] * a.n
    out["uniform"] = workload(eng, "uniform, cap-terminated", texts, prompts, uni, a.reps, [out["mix"]["poll"]])
    out["beams"] = beam_workload(eng, texts, prompts, mix, a.reps, out["mix"]["poll"])
    out["decode_step"] = step_times(eng, texts, prompts, a.reps)
    emit(out, a.out)


def emit(out, path):
    line = json.dumps(out)
    print(line)
    if path:
        os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
        with open(path, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
