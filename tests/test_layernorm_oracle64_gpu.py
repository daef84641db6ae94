"""`vb_layernorm` (csrc/embed_norm.cu layernorm_kernel) at its edges, against float64 under
tests/stack_oracle64.ln_bound: widths that reach every register-tile instantiation (kVecs 2, 4, 8, 16) and its tail
(d % 128 != 0), rows whose |mean| / sigma is 0, 16, 256 or 4096, constant rows, the `rows` gather from a strided x,
fp32 and bf16 out, with and without an AdaLN row.  The rows around `out` hold a sentinel that must survive; d = 2052
is refused as unsupported and a width that is not a multiple of 4 as a bad argument."""
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

import stack_oracle64 as S  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
DIMS = (4, 128, 132, 256, 260, 512, 1020, 1024, 1028, 2044, 2048)
OFFSETS = (0.0, 16.0, 256.0, 4096.0)
VB_ERR_ARG, VB_ERR_UNSUPPORTED = 1, 3
SENTINEL = -7777.0   # exact in bf16


def _layernorm(x, ld, rows, n, d, w, b, wb, out_dtype, pad=3):
    """vb_layernorm into the middle of a sentinel-filled buffer: returns (status, out [n, d], the whole buffer)"""
    from valle_b200 import _lib as L
    buf = torch.full(((n + 2 * pad) * d,), SENTINEL, dtype=out_dtype, device=DEV)
    out = buf[pad * d:(pad + n) * d]
    st = L.load().vb_layernorm(x.data_ptr(), ld, L.ptr(rows), n, d, w.data_ptr(), b.data_ptr(), L.ptr(wb), 1e-5,
                               out.data_ptr(), L.VB_F32 if out_dtype == torch.float32 else L.VB_BF16,
                               torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return st, out.view(n, d), buf, pad * d


def _rows(d, gen):
    """fp32 rows: for each offset 24 rows of scale 10^U(-2, 1) and |mean| / sigma = offset, then 4 constant rows"""
    parts = []
    for rho in OFFSETS:
        sc = 10.0 ** (torch.rand(24, 1, generator=gen) * 3 - 2)
        sign = torch.sign(torch.randn(24, 1, generator=gen))
        parts.append((torch.randn(24, d, generator=gen) + rho * sign) * sc)
    parts.append(torch.randn(4, 1, generator=gen).expand(4, d) * 5)
    return torch.cat(parts).float()


@pytest.mark.parametrize("d", DIMS)
def test_layernorm_within_float64_bound(d):
    gen = torch.Generator().manual_seed(100 + d)
    x = _rows(d, gen)
    R = x.shape[0]
    w = (1 + 0.2 * torch.randn(d, generator=gen)).float().to(DEV)
    b = (0.1 * torch.randn(d, generator=gen)).float().to(DEV)
    wb = torch.cat([1 + 0.1 * torch.randn(d, generator=gen), 0.1 * torch.randn(d, generator=gen)]).float().to(DEV)
    # strided x: every row padded to d + 8 columns, the real rows scattered over 3 R rows; the gather reads them back
    ld = d + 8
    big = torch.full((3 * R, ld), float("nan"))
    where = torch.randperm(3 * R, generator=gen)[:R]
    big[where, :d] = x
    big = big.to(DEV)
    rows = where.to(torch.int32).to(DEV)
    xs = x.to(DEV)
    worst = {}
    for out_dtype in (torch.float32, torch.bfloat16):
        for ada in (None, wb):
            for gather in (False, True):
                src, ldx, rr = (big, ld, rows) if gather else (xs, d, None)
                st, out, buf, off = _layernorm(src, ldx, rr, R, d, w, b, ada, out_dtype)
                assert st == 0
                assert bool((buf[:off] == SENTINEL).all()) and bool((buf[off + R * d:] == SENTINEL).all()), \
                    "vb_layernorm wrote outside its output rows"
                y, bnd = S.ln_bound(xs, w, b, ada, out)
                r = S.ratio(out, y, bnd)
                key = f"{str(out_dtype).split('.')[-1]}{' adaln' if ada is not None else ''}"
                worst[key] = max(worst.get(key, 0.0), r)
                assert r <= 1.0, f"d={d} {key} gather={gather}: error / bound {r:.3g}"
    print(f"vb_layernorm d={d}: worst error / bound " + ", ".join(f"{k} {v:.3g}" for k, v in worst.items()))


def test_layernorm_refuses_unsupported_widths():
    from valle_b200 import _lib as L
    x = torch.randn(4, 2052, device=DEV)
    w, b = torch.ones(2052, device=DEV), torch.zeros(2052, device=DEV)
    st, *_ = _layernorm(x, 2052, None, 4, 2052, w, b, None, torch.float32)
    assert st == VB_ERR_UNSUPPORTED, (st, L.load().vb_last_error())
    for d in (6, 130, 1022):
        x = torch.randn(4, d, device=DEV)
        w, b = torch.ones(d, device=DEV), torch.zeros(d, device=DEV)
        st, *_ = _layernorm(x, d, None, 4, d, w, b, None, torch.bfloat16)
        assert st == VB_ERR_ARG, (d, st)
