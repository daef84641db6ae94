"""Microbenchmark of the wgmma GEMM on the NAR projection shapes: python tools/bench_gemm.py [M]
M defaults to 48,000 (BASELINE.json configs[2], B=32 x L=1500); bench.py's NAR runs at M = 64 x 1,025 = 65,600.
CUDA-event timing, L2 flushed between iterations by the shapes themselves (A+C > 50 MB)."""
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from valle_b200 import _lib as L, ops  # noqa: E402

dev = "cuda:0"
M = int(sys.argv[1]) if len(sys.argv) > 1 else 48000
shapes = [("qkv", 3072, 1024, L.VB_EPI_NONE, torch.bfloat16), ("out_proj", 1024, 1024, L.VB_EPI_RESIDUAL, torch.float32),
          ("ffn1", 4096, 1024, L.VB_EPI_RELU, torch.bfloat16), ("ffn2", 1024, 4096, L.VB_EPI_RESIDUAL, torch.float32),
          ("head", 1024, 1024, L.VB_EPI_NONE, torch.float32)]
res = {}
for name, N, K, epi, cdt in shapes:
    a = torch.randn(M, K, device=dev).bfloat16()
    w = (torch.randn(N, K, device=dev) / 32).bfloat16()
    b = torch.randn(N, device=dev)
    c = torch.zeros(M, N, device=dev, dtype=cdt)
    for _ in range(3):
        ops.linear(a, w, b, epilogue=epi, out=c)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    n = 10
    e0.record()
    for _ in range(n):
        ops.linear(a, w, b, epilogue=epi, out=c)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / n
    tf = 2.0 * M * N * K / ms / 1e9
    # cuBLAS for context (library kernel, not the product)
    for _ in range(3):
        torch.matmul(a, w.t())
    e0.record()
    for _ in range(n):
        torch.matmul(a, w.t())
    e1.record()
    torch.cuda.synchronize()
    ms_cublas = e0.elapsed_time(e1) / n
    res[name] = dict(M=M, N=N, K=K, ms=ms, tflops=tf, cublas_ms=ms_cublas, cublas_tflops=2.0 * M * N * K / ms_cublas / 1e9)
    print(name, res[name], flush=True)
print(json.dumps(res))
