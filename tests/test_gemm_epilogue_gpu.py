"""The wgmma GEMM's epilogues against its own plain fp32 output, bit for bit.

The NONE fp32 result is the k-ordered sum acc plus the bias.  Every other epilogue is one more
exactly specified fp32 step on that value, so it must match the torch op applied to it bitwise:
  RESIDUAL(res) == res + NONE_f32,  RELU_f32 == relu(NONE_f32),  NONE_bf16 == NONE_f32.bfloat16().
The output may be a column slice of a wider buffer (ldc > N); nothing outside it may change."""
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"

SHAPES = [(1, 128, 64), (127, 1024, 1024), (128, 3072, 1024), (300, 1024, 4096), (2049, 4096, 1024),
          (20000, 256, 256),
          # more 128 x 256 tiles than two per SM: CTAs walk several tiles each
          (40000, 1024, 1024), (9001, 3072, 512),
          # N % 256 == 128: the last tile column is a half tile
          (9000, 1152, 512), (777, 128, 192)]


def _run(M, N, K, ldc_pad):
    from valle_b200 import _lib as L, ops
    g = torch.Generator().manual_seed(M * 13 + N * 3 + K + ldc_pad)
    a = torch.randn(M, K, generator=g).bfloat16().to(DEV)
    w = (torch.randn(N, K, generator=g) / K ** 0.5).bfloat16().to(DEV)
    b = torch.randn(N, generator=g).to(DEV)
    res = torch.randn(M, N, generator=g).to(DEV)

    def out_buf(dtype, init=None):
        # [M, N] view of an [M + 2, N] buffer, or at column 8 of an [M + 2, N + 8 + ldc_pad] one, filled with a sentinel
        big = torch.full((M + 2, N + (8 + ldc_pad if ldc_pad else 0)), -7.0, device=DEV, dtype=dtype)
        view = big[:M, 8:8 + N] if ldc_pad else big[:M]
        if init is not None:
            view.copy_(init)
        return big, view

    def untouched_outside(big, view):
        mask = torch.ones_like(big, dtype=torch.bool)
        if ldc_pad:
            mask[:M, 8:8 + N] = False
        else:
            mask[:M, :N] = False
        return bool((big[mask] == -7.0).all())

    big, f32 = out_buf(torch.float32)
    ops.linear(a, w, b, out=f32)
    assert untouched_outside(big, f32)
    ref = f32.clone()
    assert torch.isfinite(ref).all()

    big, c = out_buf(torch.float32, res)
    ops.linear(a, w, b, epilogue=L.VB_EPI_RESIDUAL, out=c)
    assert untouched_outside(big, c)
    assert torch.equal(c, res + ref), (c - res - ref).abs().max()

    big, r = out_buf(torch.float32)
    ops.linear(a, w, b, epilogue=L.VB_EPI_RELU, out=r)
    assert untouched_outside(big, r)
    assert torch.equal(r, torch.relu(ref))

    big, h = out_buf(torch.bfloat16)
    ops.linear(a, w, b, out=h)
    assert untouched_outside(big, h)
    assert torch.equal(h, ref.bfloat16())

    big, hr = out_buf(torch.bfloat16)
    ops.linear(a, w, b, epilogue=L.VB_EPI_RELU, out=hr)
    assert untouched_outside(big, hr)
    assert torch.equal(hr, torch.relu(ref).bfloat16())

    # without a bias the NONE output is the bare accumulator
    big, nb = out_buf(torch.float32)
    ops.linear(a, w, None, out=nb)
    assert untouched_outside(big, nb)
    assert torch.equal(nb + b, ref)


@pytest.mark.parametrize("M,N,K", SHAPES)
def test_gemm_epilogues_bitwise(M, N, K):
    _run(M, N, K, 0)


@pytest.mark.parametrize("M,N,K", [(1, 128, 64), (3000, 1024, 1024), (9000, 1152, 512)])
def test_gemm_epilogues_bitwise_column_slice(M, N, K):
    _run(M, N, K, 136)
