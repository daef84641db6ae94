"""CPU checks of the FP8 KV-cache row format (tests/kv_fp8_oracle.py, include/valle_b200.h "FP8 (e4m3) KV cache"):
the exponent rule puts every row's scaled maximum in (224, 448], the edge rows behave, and quantization is
torch.float8_e4m3fn rounding of the exactly scaled row."""
import torch

import kv_fp8_oracle as K


def _rows(n, seed):
    g = torch.Generator().manual_seed(seed)
    scale = torch.pow(2.0, torch.randint(-60, 60, (n, 1), generator=g).float())
    return (torch.randn(n, 64, generator=g) * scale).to(torch.bfloat16).float()


def test_scaled_row_maximum_lies_in_224_448():
    r = _rows(4096, 0)
    e = K.row_exponent(r)
    top = torch.ldexp(r.abs().amax(-1), (-e).float())
    assert bool((top > 224).all()) and bool((top <= 448).all()), (float(top.min()), float(top.max()))
    # e is the smallest such integer: one less would overflow 448
    assert bool((torch.ldexp(r.abs().amax(-1), (1 - e).float()) > 448).all())


def test_rows_at_powers_of_two_times_448():
    for k in (-100, -20, -1, 0, 1, 7, 60, 100):
        for sign in (1.0, -1.0):
            r = torch.zeros(1, 64)
            r[0, 5] = sign * 448.0 * 2.0 ** k          # exactly representable in bf16
            r[0, 9] = 0.5 * 2.0 ** k
            assert int(K.row_exponent(r)) == k
            q, eb = K.quantize(r)
            assert float(q.float()[0, 5]) == sign * 448.0 and int(eb) == k + 127
            assert torch.equal(K.dequantize(q, eb), r)
            # just above: the next exponent
            r2 = r.clone()
            r2[0, 5] = sign * 2.0 ** (k + 9) * (1 - 2 ** -8)   # 0.99609 * 2^(k+9) > 448 * 2^k, m > 0.875
            assert int(K.row_exponent(r2)) == k + 1


def test_zero_and_subnormal_rows():
    z = torch.zeros(3, 64)
    q, eb = K.quantize(z)
    assert bool((eb == 0).all()) and bool((q.float() == 0).all())
    assert torch.equal(K.dequantize(q, eb), z)
    # bf16 subnormals (< 2^-126): the exponent clamps at -127 and the row still reads back within e4m3 precision
    tiny = torch.zeros(2, 64)
    tiny[0, :4] = torch.tensor([2.0 ** -133, -(2.0 ** -130), 3 * 2.0 ** -131, 2.0 ** -127])
    tiny[1, 0] = 2.0 ** -120
    tiny = tiny.to(torch.bfloat16).float()
    e = K.row_exponent(tiny)
    assert e.tolist() == [-127, -127]
    q, eb = K.quantize(tiny)
    back = K.dequantize(q, eb)
    assert torch.equal(back[0, :4], tiny[0, :4])          # a few bits each: exact in e4m3 at this scale
    assert float(back[1, 0]) == 2.0 ** -120


def test_agrees_with_torch_float8_casting():
    r = _rows(2048, 1)
    q, eb = K.quantize(r)
    e = eb.to(torch.int32) - 127
    want = (r * torch.pow(2.0, -e.float())[:, None]).to(torch.float8_e4m3fn)
    assert torch.equal(q.view(torch.uint8), want.view(torch.uint8))
    # dequantization is exact and within half an e4m3 step (2^-4 relative, 2^(e-10) absolute) of the row
    back = K.dequantize(q, eb)
    assert torch.equal(back, q.float() * torch.pow(2.0, e.float())[:, None])
    tol = torch.maximum(r.abs() * 2.0 ** -4, torch.pow(2.0, e.float() - 10)[:, None])
    assert bool(((back - r).abs() <= tol).all())
