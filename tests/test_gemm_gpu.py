"""wgmma GEMM (bf16; the test names keep the kernel's former tcgen05 name) against a torch fp32 reference of the same op on the same bf16-rounded
operands.  Tolerance: fp32 accumulation of bf16 products -> |err| <= 2e-3 * sqrt(K/1024) abs on
O(1) outputs (bf16 output rounding adds 2^-8 relative)."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.mark.parametrize("M,N,K", [(1, 128, 64), (127, 1024, 1024), (128, 3072, 1024), (300, 1024, 4096),
                                   (2049, 4096, 1024), (20000, 256, 256)])
@pytest.mark.parametrize("epi", ["none_bf16", "none_f32", "relu", "residual"])
def test_tcgen05_gemm_matches_fp32_reference(M, N, K, epi):
    from valle_b200 import _lib as L, ops
    g = torch.Generator().manual_seed(M * 7 + N + K)
    a = torch.randn(M, K, generator=g).bfloat16()
    w = (torch.randn(N, K, generator=g) / K ** 0.5).bfloat16()
    b = torch.randn(N, generator=g)
    ref = F.linear(a.float(), w.float(), b)
    tol = 3e-3 * max(1.0, (K / 1024) ** 0.5)
    ad, wd, bd = a.to(DEV), w.to(DEV), b.to(DEV)
    if epi == "none_bf16":
        out = ops.linear(ad, wd, bd).float().cpu()
        assert torch.allclose(out, ref, atol=tol + 0.02, rtol=1e-2)
    elif epi == "none_f32":
        out = ops.linear(ad, wd, bd, out_dtype=torch.float32).cpu()
        assert torch.allclose(out, ref, atol=tol, rtol=1e-3), (out - ref).abs().max()
    elif epi == "relu":
        out = ops.linear(ad, wd, bd, epilogue=L.VB_EPI_RELU, out_dtype=torch.float32).cpu()
        assert torch.allclose(out, F.relu(ref), atol=tol, rtol=1e-3)
    else:
        res = torch.randn(M, N, generator=g)
        c = res.to(DEV).clone()
        ops.linear(ad, wd, bd, epilogue=L.VB_EPI_RESIDUAL, out=c)
        assert torch.allclose(c.cpu(), res + ref, atol=tol, rtol=1e-3), (c.cpu() - res - ref).abs().max()


def test_tcgen05_matches_simt_kernel_bitwise_inputs():
    """same bf16 operands through the CUDA-core kernel (VB_DISABLE_WGMMA is read per call)."""
    from valle_b200 import _lib as L
    from valle_b200 import ops
    lib = L.load()
    g = torch.Generator().manual_seed(5)
    a = torch.randn(257, 1024, generator=g).bfloat16().to(DEV)
    w = (torch.randn(1024, 1024, generator=g) / 32).bfloat16().to(DEV)
    o1 = ops.linear(a, w, None, out_dtype=torch.float32)
    L.check(lib.vb_tune_set(b"VB_DISABLE_WGMMA", 1))
    try:
        o2 = ops.linear(a, w, None, out_dtype=torch.float32)
    finally:
        L.check(lib.vb_tune_set(b"VB_DISABLE_WGMMA", 0))
    assert torch.allclose(o1, o2, atol=1e-3, rtol=1e-4), (o1 - o2).abs().max()
