"""One engine.generate() call for profiling (ncu / launch lists): python tools/profile_decode.py B FRAMES [dtype] [nar [prof]]
`nar prof` records the timed NAR run with torch.profiler and prints the device time per kernel and per kernel group."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402

B = int(sys.argv[1]) if len(sys.argv) > 1 else 64
frames = int(sys.argv[2]) if len(sys.argv) > 2 else bench.FRAMES
dtype = torch.float32 if (len(sys.argv) > 3 and sys.argv[3] == "fp32") else torch.bfloat16
dev = torch.device("cuda", 0)
model = bench.build_model(dev)
if len(sys.argv) > 4 and sys.argv[4] == "ar_only":
    model.num_quantizers_saved = model.num_quantizers
eng = model.engine(dtype)
eng.quiet = True
if os.environ.get('VB_NO_GRAPH'):
    eng.use_cuda_graph = False
texts, prompts = bench.make_batch(B, 0, dev)
if len(sys.argv) > 4 and sys.argv[4] == 'nar':
    # NAR only: VALLE.continual on [prompt | 753 given first-codebook frames] -> the 7 NAR passes of the bench shape
    g = torch.Generator().manual_seed(1)
    ys = [torch.randint(0, 1024, (bench.T_PROMPT + frames, bench.N_Q), generator=g).to(dev) for _ in range(B)]
    eng.continual(texts, ys)
    torch.cuda.synchronize()
    if len(sys.argv) > 5 and sys.argv[5] == 'prof':
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            eng.continual(texts, ys)
            torch.cuda.synchronize()
        per = {}
        for ev in prof.events():
            if ev.device_type == torch.autograd.DeviceType.CUDA and ev.device_time > 0:
                n, us = per.get(ev.name, (0, 0.0))
                per[ev.name] = (n + 1, us + ev.device_time)
        total = sum(us for _, us in per.values())
        groups = {}
        print(f"{'ms':>9} {'share':>6} {'calls':>6}  kernel")
        for name, (n, us) in sorted(per.items(), key=lambda kv: -kv[1][1]):
            print(f"{us / 1e3:9.2f} {us / total:6.1%} {n:6d}  {name[:110]}")
            g = 'gemm_wgmma' if 'gemm_wgmma' in name else 'attention' if 'attn' in name or 'attention' in name else 'other'
            groups[g] = groups.get(g, 0.0) + us
        print('nar_kernel_ms', {g: round(us / 1e3, 2) for g, us in groups.items()}, 'total', round(total / 1e3, 2))
        sys.exit(0)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    eng.continual(texts, ys)
    e1.record()
    torch.cuda.synchronize()
    print('nar_only_ms', e0.elapsed_time(e1))
    sys.exit(0)
mnt = None if frames >= bench.FRAMES else frames
if os.environ.get('VB_WARM'):
    eng.generate(texts, prompts, top_k=1, max_new_tokens=mnt, return_device=True)
out = eng.generate(texts, prompts, top_k=1, max_new_tokens=mnt, return_device=True)
torch.cuda.synchronize()
print("frames", out[0].shape, "ar_ms", eng.stats.ar_ms, "steps", eng.stats.ar_steps, "nar_ms", eng.stats.nar_ms,
      "prefill_ms", eng.stats.prefill_ms)
