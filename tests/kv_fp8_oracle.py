"""TEST INFRASTRUCTURE ONLY -- the FP8 (e4m3) KV-cache row format of include/valle_b200.h ("FP8 (e4m3) KV cache"),
restated with torch on the CPU.

A cached row r is 64 values (the bf16 row the bf16 cache would hold).  a = max |r|; e = the smallest integer with
a <= 448 * 2^e, taken exactly from frexp(a) = m * 2^x (m in [0.5, 1)): e = x - 9 if m <= 0.875 else x - 8, clamped to
[-127, 127]; an all-zero row gets e = -127.  The row is stored as torch.float8_e4m3fn(r * 2^-e) (the scaling is exact:
a power of two) and the exponent as the byte e + 127.  It reads back as fp8 * 2^e."""
from __future__ import annotations

import torch

E4M3_MAX = 448.0


def row_exponent(rows: torch.Tensor) -> torch.Tensor:
    """e (int32) of every 64-element row of rows [..., 64]"""
    a = rows.float().abs().amax(dim=-1)
    m, x = torch.frexp(a)
    e = torch.where(m <= 0.875, x - 9, x - 8)
    e = torch.where(a > 0, e, torch.full_like(e, -127))
    return e.clamp(-127, 127).to(torch.int32)


def quantize(rows: torch.Tensor):
    """rows [..., 64] (bf16 values) -> (e4m3 bytes as torch.float8_e4m3fn [..., 64], biased exponents uint8 [...])"""
    e = row_exponent(rows)
    scaled = torch.ldexp(rows.float(), (-e)[..., None].float())
    return scaled.to(torch.float8_e4m3fn), (e + 127).to(torch.uint8)


def dequantize(q: torch.Tensor, eb: torch.Tensor) -> torch.Tensor:
    """(fp8 [..., 64], biased exponents [...]) -> fp32 [..., 64], exact"""
    return torch.ldexp(q.float(), (eb.to(torch.int32) - 127)[..., None].float())
