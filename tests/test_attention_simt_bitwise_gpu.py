"""The CUDA-core attention kernels and the AR training mask, pinned bit for bit.

tests/test_attention_bitwise_gpu.py pins the bf16 wgmma forward and tests/test_decoder_stack_bitwise_gpu.py the stacks
in VALLE_AR / FULL / PADDED.  This file pins the rest of the masked attention paths, on the ragged batch of
test_attention_bitwise_gpu._ragged (seeded on the CPU), against tests/golden/attn_simt_bits.pt:
  - fwd_*: `vb_attention` on the exact-order CUDA-core kernel, fp32 and bf16 (VB_ATTN_SIMT=1), in the four mask modes
    and VB_MASK_DENSE: SHA-256 of each sequence's output; the *_cache cases also hash both sentinel-filled KV caches;
  - bwd_*: `vb_attention_backward`, fp32 and bf16, four modes: SHA-256 of each sequence's dqkv rows (the backward
    kernels use no atomics, so their bits are fixed);
  - train_*: `autograd.DecoderStack` forward + backward with VB_MASK_PADDED_AR and dropout 0.1, hashed and compared as
    in test_decoder_stack_bitwise_gpu.py (the atomically summed gradients within its tolerance).

    python tests/test_attention_simt_bitwise_gpu.py --record     # rewrite the fixture from the library as built
"""
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import test_attention_bitwise_gpu as A  # noqa: E402
import test_decoder_stack_bitwise_gpu as S  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
FIXTURE = os.path.join(ROOT, "tests", "golden", "attn_simt_bits.pt")
H, D = A.H, A.D
DTYPES = {"f32": (torch.float32, 0), "bf16": (torch.bfloat16, 1)}   # torch dtype, VB_F32 / VB_BF16
MODES = ("full", "valle_ar", "padded_ar", "padded")


def _batch(mode, dtype):
    """qkv [M, 3D] on the device, lengths, mask mode, text_lens, seg1_lens (device int32 or None)"""
    from valle_b200 import _lib as L
    qkv, lens, tl, sl = A._ragged(mode)
    mm = dict(full=L.VB_MASK_FULL, valle_ar=L.VB_MASK_VALLE_AR, padded_ar=L.VB_MASK_PADDED_AR,
              padded=L.VB_MASK_PADDED, dense=L.VB_MASK_DENSE)[mode]
    tl = torch.tensor(tl, dtype=torch.int32, device=DEV) if mode not in ("full", "dense") else None
    sl = torch.tensor(sl, dtype=torch.int32, device=DEV) if mode.startswith("padded") else None
    return qkv.to(dtype).to(DEV), lens, mm, tl, sl


def _cu(lens):
    return torch.tensor([0] + torch.tensor(lens).cumsum(0).tolist(), dtype=torch.int32, device=DEV)


def _per_seq(t, cu):
    t = t.cpu()
    return [S._sha(t[int(cu[b]):int(cu[b + 1])]) for b in range(len(cu) - 1)]


def _attention(qkv, vdt, lens, mm, tl, sl, kc=None, vc=None, cap=0, dense=None):
    from valle_b200 import _lib as L
    M, B = qkv.shape[0], len(lens)
    cu = _cu(lens)
    out = torch.full((M, D), -3.0, dtype=qkv.dtype, device=DEV)
    L.check(L.load().vb_attention(qkv.data_ptr(), vdt, M, B, H, 64, cu.data_ptr(), L.ptr(tl), L.ptr(sl), A.SEG1_START,
                                  max(lens), mm, out.data_ptr(), L.ptr(kc), L.ptr(vc), H * cap * 64 if cap else 0, cap,
                                  L.ptr(dense), dense.shape[1] if dense is not None else 0,
                                  torch.cuda.current_stream().cuda_stream), "vb_attention")
    return out, cu


def _forward(name):
    """fwd_{f32,bf16}_{full,valle_ar,padded_ar,padded,dense}[_cache]"""
    from valle_b200 import _lib as L
    _, dt, *rest = name.split("_")
    cache = rest[-1] == "cache"
    mode = "_".join(rest[:-1] if cache else rest)
    dtype, vdt = DTYPES[dt]
    qkv, lens, mm, tl, sl = _batch(mode, dtype)
    dense = None
    if mode == "dense":   # ~30 % of the pairs blocked, never a row's own key
        n = max(lens)
        blocked = torch.rand(n, n, generator=torch.Generator().manual_seed(12)) < 0.3
        blocked.fill_diagonal_(False)
        dense = blocked.to(torch.uint8).to(DEV)
    kc = vc = None
    cap = max(lens) + 16 if cache else 0
    if cache:
        kc = torch.full((len(lens), H, cap, 64), 1234.0, dtype=dtype, device=DEV)
        vc = torch.full((len(lens), H, cap, 64), -1234.0, dtype=dtype, device=DEV)
    lib = L.load()
    if dt == "bf16":
        L.check(lib.vb_tune_set(b"VB_ATTN_SIMT", 1))
    try:
        out, cu = _attention(qkv, vdt, lens, mm, tl, sl, kc, vc, cap, dense)
        torch.cuda.synchronize()
    finally:
        lib.vb_tune_set(b"VB_ATTN_SIMT", 0)
    r = {"seq": _per_seq(out, cu)}
    if cache:
        r["kcache"], r["vcache"] = S._sha(kc), S._sha(vc)
    return r


def _backward(name):
    """bwd_{f32,bf16}_{full,valle_ar,padded_ar,padded}: the forward output of vb_attention, then vb_attention_backward"""
    from valle_b200 import _lib as L
    _, dt, mode = name.split("_", 2)
    dtype, vdt = DTYPES[dt]
    qkv, lens, mm, tl, sl = _batch(mode, dtype)
    M, B = qkv.shape[0], len(lens)
    dout = (torch.randn(M, D, generator=torch.Generator().manual_seed(13)) * 0.3).to(dtype).to(DEV)
    out, cu = _attention(qkv, vdt, lens, mm, tl, sl)
    lib = L.load()
    nb = lib.vb_attention_backward_workspace(M, H)
    ws = torch.empty(nb, dtype=torch.uint8, device=DEV)
    dqkv = torch.full((M, 3 * D), -5.0, dtype=dtype, device=DEV)
    L.check(lib.vb_attention_backward(qkv.data_ptr(), out.data_ptr(), dout.data_ptr(), vdt, M, B, H, 64, cu.data_ptr(),
                                      L.ptr(tl), L.ptr(sl), A.SEG1_START, max(lens), mm, dqkv.data_ptr(),
                                      ws.data_ptr(), nb, torch.cuda.current_stream().cuda_stream),
            "vb_attention_backward")
    torch.cuda.synchronize()
    return {"seq": _per_seq(dqkv, cu)}


def _train(name):
    """train_pre_ln_{f32,bf16}_p01: the stack of test_decoder_stack_bitwise_gpu.py trained on the AR mask"""
    from valle_b200 import _lib as L
    return S._train(name, mode=L.VB_MASK_PADDED_AR)


CASES = ([f"fwd_{dt}_{m}" for dt in DTYPES for m in MODES + ("dense",)] + [f"fwd_{dt}_valle_ar_cache" for dt in DTYPES] +
         [f"bwd_{dt}_{m}" for dt in DTYPES for m in MODES] +
         [f"train_pre_ln_{dt}_p01" for dt in DTYPES])


def _run(name):
    return {"fwd": _forward, "bwd": _backward, "train": _train}[name.split("_")[0]](name)


def _diff(got, want):
    """what of `want` `got` does not reproduce: the sequences whose hash moved, and the keys of S._diff"""
    if "seq" not in want:
        return S._diff(got, want)
    assert set(got) == set(want) and len(got["seq"]) == len(want["seq"])
    moved = [b for b, (x, y) in enumerate(zip(got["seq"], want["seq"])) if x != y]
    return ([f"sequences {moved}"] if moved else []) + [k for k in want if k != "seq" and got[k] != want[k]]


@pytest.mark.parametrize("name", CASES)
def test_attention_simt_bits(name):
    want = torch.load(FIXTURE, weights_only=False)[name]
    moved = _diff(_run(name), want)
    assert not moved, f"{name}: differs from the recorded run in {moved}"


if __name__ == "__main__":
    if "--record" not in sys.argv:
        sys.exit("usage: python tests/test_attention_simt_bitwise_gpu.py --record")
    rec = {name: _run(name) for name in CASES}
    # a second run must reproduce the first: the hashes exactly, the atomically summed gradients within the bound
    again = {name: _run(name) for name in CASES}
    bad = {name: m for name in CASES if (m := _diff(again[name], rec[name]))}
    if bad:
        sys.exit(f"two runs of the library disagree: {bad}")
    torch.save(rec, FIXTURE)
    print(f"recorded {len(CASES)} cases to {FIXTURE}")
