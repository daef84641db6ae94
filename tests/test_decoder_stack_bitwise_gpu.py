"""The native decoder stack (vb_decoder_forward, vb_decoder_forward_train, vb_decoder_backward), pinned bit for bit.

A small stack (d=256, 4 heads, d_ff=1024, 2 layers) is built through valle_b200.modules.transformer from a torch seed,
and every input is generated on the CPU.  Each case runs the stack through `NativeDecoder.forward` (inference) or
`autograd.DecoderStack` (training forward + backward) and compares with tests/golden/decoder_stack_bits.pt:
  - SHA-256 of the stack output, of both whole KV caches (pre-filled with a sentinel; with the FP8 cache, both
    exponent arrays as well), of the input gradient and of the four weight-matrix gradients of every layer;
  - the bias, LayerNorm-affine and AdaLN gradients within 1e-5 x the recorded tensor's max-abs: they are summed with
    atomicAdd, so their last bits vary from run to run;
  - the number of library launches of each call.
A change to the host-side layer loops that keeps every launch, its arguments and its order passes unchanged; one that
moves a slot, swaps two launches or drops a dropout site names the case and the value that moved.

    python tests/test_decoder_stack_bitwise_gpu.py --record     # rewrite the fixture from the library as built
"""
import hashlib
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
FIXTURE = os.path.join(ROOT, "tests", "golden", "decoder_stack_bits.pt")
D, H, DFF, NL = 256, 4, 1024, 2
TOL = 1e-5
SEED = 987654321
DTYPES = {"f32": torch.float32, "bf16": torch.bfloat16}


def _sha(t):
    return hashlib.sha256(t.detach().contiguous().cpu().reshape(-1).view(torch.uint8).numpy().tobytes()).hexdigest()


def _stack(norm_first, adaptive, seed):
    """the TransformerEncoder on cuda:0, with non-trivial biases and norm affines, and its AdaLN table [2*NL, 2d]"""
    from valle_b200.modules.transformer import TransformerEncoder, TransformerEncoderLayer
    torch.manual_seed(seed)
    enc = TransformerEncoder(TransformerEncoderLayer(D, H, dim_feedforward=DFF, dropout=0.1, batch_first=True,
                                                     norm_first=norm_first, adaptive_layer_norm=adaptive),
                             num_layers=NL)
    g = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():
        for p in enc.parameters():
            if p.dim() == 1:
                p.add_(torch.randn(p.shape, generator=g) * 0.05)
    ada = None
    if adaptive:
        ada = torch.cat([1.0 + 0.1 * torch.randn(2 * NL, D, generator=g), 0.1 * torch.randn(2 * NL, D, generator=g)], 1)
    return enc.to(DEV), ada


def _launches(fn):
    from valle_b200 import _lib as L
    lib = L.load()
    torch.cuda.synchronize()
    n0 = lib.vb_launch_count()
    r = fn()
    torch.cuda.synchronize()
    return r, lib.vb_launch_count() - n0


def _forward(name):
    """fwd_{pre,post}_{ln_prefill,adaln_nar}_{f32,bf16}: one vb_decoder_forward call; fwd_{pre,post}_ln_prefill_f8: the
    same call with the exponent rows (bf16 stack, FP8 cache)"""
    from valle_b200 import _lib as L
    _, order, norm, shape, dt = name.split("_")
    f8 = dt == "f8"
    enc, ada = _stack(order == "pre", norm == "adaln", 5)
    nd = enc.native(torch.bfloat16 if f8 else DTYPES[dt])
    g = torch.Generator().manual_seed(6)
    r = {}
    ke = ve = None
    if shape == "prefill":        # the AR prefill: text + prompt rows per utterance, KV caches filled for decoding
        lens, tl, cap = [40, 23, 61], [9, 5, 17], 64
        rows = (NL, len(lens), H, cap)
        if f8:                    # sentinel bytes in the e4m3 rows and in the exponent arrays
            cache = lambda v: torch.full(rows + (D // H,), v, dtype=torch.uint8, device=DEV).view(torch.float8_e4m3fn)
            kc, vc = cache(0x5A), cache(0xDA)
            ke, ve = (torch.full(rows, v, dtype=torch.uint8, device=DEV) for v in (0xAB, 0xCD))
        else:
            cache = lambda v: torch.full(rows + (D // H,), v, dtype=DTYPES[dt], device=DEV)
            kc, vc = cache(1234.0), cache(-1234.0)
        mode, tl = L.VB_MASK_VALLE_AR, torch.tensor(tl, dtype=torch.int32, device=DEV)
    else:                         # a NAR pass: whole sequences, AdaLN rows of one stage
        lens, kc, vc, cap = [57, 12, 90], None, None, 0
        mode, tl = L.VB_MASK_FULL, None
    x = torch.randn(sum(lens), D, generator=g).to(DEV)
    cu = torch.tensor([0] + torch.tensor(lens).cumsum(0).tolist(), dtype=torch.int32, device=DEV)
    ada = ada.to(DEV) if ada is not None else None
    _, r["launches"] = _launches(lambda: nd.forward(x, cu, len(lens), max(lens), mode, tl, ada, kc, vc, cap,
                                                    k_exp=ke, v_exp=ve))
    r["out"] = _sha(x)
    if kc is not None:
        r["kcache"], r["vcache"] = _sha(kc), _sha(vc)
    if ke is not None:
        r["k_exp"], r["v_exp"] = _sha(ke), _sha(ve)
    return r


def _train(name, mode=None):
    """train_{pre,post}_{ln,adaln}_{f32,bf16}_{p0,p01}: autograd.DecoderStack forward + backward on the padded batch of
    the NAR training pass (VB_MASK_PADDED, or the mask mode given)"""
    from valle_b200 import _lib as L
    from valle_b200 import autograd as AG
    mode = L.VB_MASK_PADDED if mode is None else mode
    _, order, norm, dt, pp = name.split("_")
    p = {"p0": 0.0, "p01": 0.1}[pp]
    enc, ada = _stack(order == "pre", norm == "adaln", 7)
    nd = enc.native(DTYPES[dt])
    params = AG.layer_params(enc)
    N, Smax, Tmax = 3, 8, 40
    Lp = Smax + Tmax
    xl = torch.tensor([8, 5, 3], dtype=torch.int32, device=DEV)
    yl = torch.tensor([40, 29, 12], dtype=torch.int32, device=DEV)
    cu = (torch.arange(N + 1, dtype=torch.int32) * Lp).to(DEV)
    g = torch.Generator().manual_seed(8)
    xa = torch.randn(N * Lp, D, generator=g).to(DEV).requires_grad_()
    w = torch.randn(N * Lp, D, generator=g).to(DEV)
    ada = ada.to(DEV).requires_grad_() if ada is not None else None
    geom = (cu, N, Lp, mode, xl, yl, Smax, p, SEED)
    r = {}
    out, r["launches_fwd"] = _launches(lambda: AG.DecoderStack.apply(xa, ada, nd, geom, *params))
    _, r["launches_bwd"] = _launches(lambda: (out * w).sum().backward())
    r["out"], r["dx"] = _sha(out), _sha(xa.grad)
    names = AG._LAYER_PARAM_ORDER
    tol = {}
    for i, q in enumerate(params):
        key = f"{i // len(names)}.{names[i % len(names)]}"
        if q.dim() == 2:
            r[key] = _sha(q.grad)
        else:
            tol[key] = q.grad.detach().cpu().clone()
    if ada is not None:
        tol["ada"] = ada.grad.detach().cpu().clone()
    r["tol"] = tol
    return r


CASES = ([f"fwd_{o}_{k}_{dt}" for o in ("pre", "post") for k in ("ln_prefill", "adaln_nar") for dt in DTYPES] +
         [f"fwd_{o}_ln_prefill_f8" for o in ("pre", "post")] +
         [f"train_{o}_{n}_{dt}_{p}" for o in ("pre", "post") for n in ("ln", "adaln") for dt in DTYPES
          for p in ("p0", "p01")])


def _run(name):
    return _forward(name) if name.startswith("fwd_") else _train(name)


def _diff(got, want):
    """the keys of `want` that `got` does not reproduce: exact values, and the "tol" tensors within TOL x max-abs"""
    assert set(got) == set(want), (sorted(got), sorted(want))
    moved = [k for k in want if k != "tol" and got[k] != want[k]]
    for k, t in want.get("tol", {}).items():
        err = float((got["tol"][k] - t).abs().max())
        if not err <= TOL * float(t.abs().max()):
            moved.append(f"{k} (max |diff| {err:.3g}, bound {TOL * float(t.abs().max()):.3g})")
    return moved


@pytest.mark.parametrize("name", CASES)
def test_decoder_stack_bits(name):
    want = torch.load(FIXTURE, weights_only=False)[name]
    moved = _diff(_run(name), want)
    assert not moved, f"{name}: differs from the recorded run in {moved}"


if __name__ == "__main__":
    if "--record" not in sys.argv:
        sys.exit("usage: python tests/test_decoder_stack_bitwise_gpu.py --record")
    rec = {name: _run(name) for name in CASES}
    # a second run must reproduce the first: the hashes exactly, the atomically summed gradients within the bound
    again = {name: _run(name) for name in CASES}
    bad = {name: m for name in CASES if (m := _diff(again[name], rec[name]))}
    if bad:
        sys.exit(f"two runs of the library disagree: {bad}")
    worst = max(float((again[n]["tol"][k] - t).abs().max() / t.abs().max().clamp_min(1e-30))
                for n in CASES if "tol" in rec[n] for k, t in rec[n]["tol"].items())
    print(f"atomically summed gradients: two runs differ by at most {worst:.3g} x max-abs (bound {TOL:g})")
    torch.save(rec, FIXTURE)
    print(f"recorded {len(CASES)} cases to {FIXTURE}")
