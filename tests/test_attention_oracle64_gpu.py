"""`vb_attention` against the float64 reference of tests/attention_oracle64.py, under its derived error bound, on all
three kernel paths: the bf16 wgmma flash kernel, the bf16 CUDA-core kernel (VB_ATTN_SIMT=1) and the fp32 CUDA-core
kernel.  The cases (attention_oracle64.case_names) are the benchmark's NAR passes (B=64, L=1025, H=16) and AR prefill
(B=64, L=272, S=47), config2 (B=4, L=1500) and the 28-sequence ragged set in all four mask modes, and packed sweeps of
L in {1, 2, 63, 64, 65, 127, 128, 129, 191, 192, 193, 256, 257} over text lengths and padded audio lengths; every case
carries planted keys, so a key the kernel skips or lets through costs it O(|v|), far over the bound.

Also: the KV cache the prefill fills (every row < L bit for bit, every other row untouched), and that NaN / inf in the
next packed sequence's K or V rows changes no output of a sequence.
"""
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

import attention_oracle64 as A  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
PATHS = {"wgmma": (torch.bfloat16, 0), "simt_bf16": (torch.bfloat16, 1), "simt_f32": (torch.float32, 0)}
_cache = {}


def _mode(name):
    from valle_b200 import _lib as L
    return dict(full=L.VB_MASK_FULL, valle_ar=L.VB_MASK_VALLE_AR, padded_ar=L.VB_MASK_PADDED_AR,
                padded=L.VB_MASK_PADDED)[name]


def _attention(qkv, lens, mode, S, c1, seg1_start, H, path, kc=None, vc=None, cap=0):
    """vb_attention on one kernel path: qkv [M, 3 H 64] on the device, in the path's dtype"""
    from valle_b200 import _lib as L
    dtype, simt = PATHS[path]
    assert qkv.dtype == dtype
    M, B, D = qkv.shape[0], len(lens), H * A.HD
    cu = torch.tensor([0] + torch.tensor(lens).cumsum(0).tolist(), dtype=torch.int32, device=DEV)
    tl = torch.tensor(S, dtype=torch.int32, device=DEV) if mode != "full" else None
    sl = torch.tensor(c1, dtype=torch.int32, device=DEV) if mode.startswith("padded") else None
    out = torch.full((M, D), -3.0, dtype=dtype, device=DEV)
    lib = L.load()
    L.check(lib.vb_tune_set(b"VB_ATTN_SIMT", simt))
    try:
        L.check(lib.vb_attention(qkv.data_ptr(), L.VB_BF16 if dtype == torch.bfloat16 else L.VB_F32, M, B, H, A.HD,
                                 cu.data_ptr(), L.ptr(tl), L.ptr(sl), seg1_start, max(lens), _mode(mode),
                                 out.data_ptr(), L.ptr(kc), L.ptr(vc), H * cap * A.HD if cap else 0, cap, None, 0,
                                 torch.cuda.current_stream().cuda_stream), "vb_attention")
        torch.cuda.synchronize()
    finally:
        lib.vb_tune_set(b"VB_ATTN_SIMT", 0)
    return out


def _batch(name):
    if name not in _cache:
        _cache.clear()
        _cache[name] = A.make_case(name, device=DEV)
    return _cache[name]


@pytest.mark.parametrize("path", list(PATHS))
@pytest.mark.parametrize("name", A.case_names())
def test_attention_within_float64_bound(name, path):
    b = _batch(name)
    qkv = b.qkv.to(PATHS[path][0])
    out = _attention(qkv, b.lens, b.mode, b.S, b.c1, b.seg1_start, b.H, path)
    worst, empty_rows = 0.0, 0
    for i in range(len(b.lens)):
        vis = b.vis(i)
        ref = A.attention64(*b.heads(qkv, i), vis.to(DEV), head_chunk=8)
        assert ref.empty == A.empty_rows_rule(b.mode, b.lens[i], b.S[i], b.c1[i], b.seg1_start)
        empty_rows += len(ref.empty)
        got = out[b.cu[i]:b.cu[i + 1]].view(b.lens[i], b.H, A.HD).transpose(0, 1)
        r = A.ratio(got, ref, A.bound(ref, path))
        assert r <= 1.0, f"{name} {path}: sequence {i} (L={b.lens[i]}, S={b.S[i]}, c1={b.c1[i]}) error / bound {r:.3g}"
        worst = max(worst, r)
    print(f"{name} {path}: max error / bound {worst:.3f} over {len(b.lens)} sequences, {len(b.beacons)} planted keys, "
          f"{empty_rows} rows without keys")


CACHE_LENS = [1, 63, 64, 65, 129, 320]


@pytest.mark.parametrize("path", list(PATHS))
def test_prefill_fills_the_kv_cache(path):
    """the prefill (VALLE_AR, S = min(47, L)) writes rows [0, L) of every stream (b, h) of a cap-320 cache from the
    K and V columns of qkv, bit for bit, and leaves every other row at its sentinel"""
    dtype = PATHS[path][0]
    H, cap, D = 16, 320, 16 * A.HD
    lens = CACHE_LENS
    S = [min(47, n) for n in lens]
    g = torch.Generator().manual_seed(21)
    qkv = (torch.randn(sum(lens), 3 * D, generator=g) * 0.5).to(dtype).to(DEV)
    kc = torch.full((len(lens), H, cap, A.HD), 1234.0, dtype=dtype, device=DEV)
    vc = torch.full((len(lens), H, cap, A.HD), -1234.0, dtype=dtype, device=DEV)
    sentinel_k, sentinel_v = kc[0, 0, 0, 0].clone(), vc[0, 0, 0, 0].clone()
    _attention(qkv, lens, "valle_ar", S, [0] * len(lens), 0, H, path, kc, vc, cap)
    r0 = 0
    bits = torch.int16 if dtype == torch.bfloat16 else torch.int32
    for b, n in enumerate(lens):
        k = qkv[r0:r0 + n, D:2 * D].reshape(n, H, A.HD).transpose(0, 1)
        v = qkv[r0:r0 + n, 2 * D:].reshape(n, H, A.HD).transpose(0, 1)
        assert torch.equal(kc[b, :, :n].view(bits), k.contiguous().view(bits)), (path, b, n, "K rows")
        assert torch.equal(vc[b, :, :n].view(bits), v.contiguous().view(bits)), (path, b, n, "V rows")
        assert bool((kc[b, :, n:] == sentinel_k).all()) and bool((vc[b, :, n:] == sentinel_v).all()), (path, b, n)
        r0 += n


ISO_LENS = [65, 1, 129, 200, 63, 64, 257, 100, 130]


@pytest.mark.parametrize("path", list(PATHS))
@pytest.mark.parametrize("mode", A.MODES)
def test_next_sequence_nan_does_not_leak(mode, path):
    """NaN in the K rows and inf / NaN in the V rows of the sequences of one parity leave every output of the others
    bit for bit as they were: the last key tile of a sequence reads into the next one, where P is 0, but 0 inf and
    0 NaN are NaN"""
    dtype = PATHS[path][0]
    H, D, seg1_start = 4, 4 * A.HD, 60
    lens = ISO_LENS
    S = [min(n, 47) for n in lens]
    c1 = [max(0, min(n - seg1_start, 50)) for n in lens]
    g = torch.Generator().manual_seed(22)
    qkv = (torch.randn(sum(lens), 3 * D, generator=g) * 0.5).to(dtype).to(DEV)
    cu = [0] + torch.tensor(lens).cumsum(0).tolist()
    clean = _attention(qkv, lens, mode, S, c1, seg1_start, H, path)
    assert torch.isfinite(clean).all()
    for parity in (0, 1):
        bad = qkv.clone()
        for b in range(parity, len(lens), 2):
            bad[cu[b]:cu[b + 1], D:2 * D] = float("nan")
            bad[cu[b]:cu[b + 1], 2 * D::2] = float("inf")
            bad[cu[b]:cu[b + 1], 2 * D + 1::2] = float("nan")
        out = _attention(bad, lens, mode, S, c1, seg1_start, H, path)
        bits = torch.int16 if dtype == torch.bfloat16 else torch.int32
        moved = [b for b in range(1 - parity, len(lens), 2)
                 if not torch.equal(out[cu[b]:cu[b + 1]].view(bits), clean[cu[b]:cu[b + 1]].view(bits))]
        assert not moved, f"{mode} {path}: sequences {moved} changed when the next sequence holds NaN / inf"
