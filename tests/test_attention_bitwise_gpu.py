"""The bf16 tensor-core flash attention (attention_wgmma.cu), pinned bit for bit.

Every case feeds seeded bf16 inputs (generated on the CPU) to `vb_attention` and compares the SHA-256 of each
sequence's output bytes with tests/golden/attn_wgmma_bits.pt.  The prefill case also passes real KV-cache pointers,
pre-filled with a sentinel, and hashes both whole caches: every key row < L is written, nothing else is.
A rewrite of the kernel that keeps its arithmetic (tile order, mask decisions, softmax expressions, wgmma shapes)
passes unchanged; one that rounds anything differently names the case and the sequences that moved.

    python tests/test_attention_bitwise_gpu.py --record     # rewrite the fixture from the library as built
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
FIXTURE = os.path.join(ROOT, "tests", "golden", "attn_wgmma_bits.pt")
H, D = 16, 1024
SEG1_START = 60


def _sha(t):
    return hashlib.sha256(t.contiguous().cpu().view(torch.int16).numpy().tobytes()).hexdigest()


def _ragged(mode):
    # the lengths and mask parameters of test_parity_gpu.py::test_bf16_flash_attention_persistent_schedule_all_masks:
    # 1-row and 1-key remainders, more (query tile, head, sequence) items than the grid holds at once
    g = torch.Generator().manual_seed(11)
    B = 28
    lens = [1, 129, 257, 400, 128, 256, 385] + torch.randint(2, 400, (B - 7,), generator=g).tolist()
    S = [min(n, int(v)) for n, v in zip(lens, torch.randint(1, 60, (B,), generator=g).tolist())]
    seg1 = [max(0, min(n - SEG1_START, int(v))) for n, v in zip(lens, torch.randint(0, 340, (B,), generator=g).tolist())]
    qkv = (torch.randn(sum(lens), 3 * D, generator=g) * 0.7).bfloat16()
    return qkv, lens, S, seg1


def _case(name):
    """(qkv [M, 3D] bf16 on the CPU, lengths, mask mode, text_lens, seg1_lens, cache_cap or 0)"""
    from valle_b200 import _lib as L
    if name == "nar_b64_l1025":      # the benchmark's NAR passes
        n, B = 1025, 64
        qkv = (torch.randn(B * n, 3 * D, generator=torch.Generator().manual_seed(1)) * 0.5).bfloat16()
        qkv[:n, :D] *= 6.0           # peaked scores in sequence 0: the row maximum grows, the rescale path runs
        return qkv, [n] * B, L.VB_MASK_FULL, None, None, 0
    if name == "config2_b4_l1500":   # L % 64 = 28, L % 128 = 92
        n, B = 1500, 4
        qkv = (torch.randn(B * n, 3 * D, generator=torch.Generator().manual_seed(2)) * 0.5).bfloat16()
        return qkv, [n] * B, L.VB_MASK_FULL, None, None, 0
    if name == "prefill_b64_l272":   # the AR prefill of the benchmark: 47 text + 225 prompt rows, fills the KV cache
        n, B, S = 272, 64, 47
        qkv = (torch.randn(B * n, 3 * D, generator=torch.Generator().manual_seed(3)) * 0.5).bfloat16()
        return qkv, [n] * B, L.VB_MASK_VALLE_AR, [S] * B, None, 320
    mode = name[len("ragged_"):]
    qkv, lens, S, seg1 = _ragged(mode)
    mm = dict(full=L.VB_MASK_FULL, valle_ar=L.VB_MASK_VALLE_AR, padded_ar=L.VB_MASK_PADDED_AR,
              padded=L.VB_MASK_PADDED)[mode]
    return (qkv, lens, mm, S if mode != "full" else None, seg1 if mode.startswith("padded") else None, 0)


CASES = ["nar_b64_l1025", "config2_b4_l1500", "ragged_full", "ragged_valle_ar", "ragged_padded_ar", "ragged_padded",
         "prefill_b64_l272"]


def _hashes(name):
    """{"seq": [sha of each sequence's [L, D] output], and with a cache: "kcache" / "vcache": sha of the whole cache}"""
    from valle_b200 import _lib as L
    qkv_h, lens, mode, S, seg1, cap = _case(name)
    qkv = qkv_h.to(DEV)
    B, M = len(lens), sum(lens)
    cu = torch.tensor([0] + torch.tensor(lens).cumsum(0).tolist(), dtype=torch.int32, device=DEV)
    tl = torch.tensor(S, dtype=torch.int32, device=DEV) if S is not None else None
    sl = torch.tensor(seg1, dtype=torch.int32, device=DEV) if seg1 is not None else None
    out = torch.full((M, D), -3.0, dtype=torch.bfloat16, device=DEV)
    kc = vc = None
    if cap:
        kc = torch.full((B, H, cap, 64), 1234.0, dtype=torch.bfloat16, device=DEV)
        vc = torch.full((B, H, cap, 64), -1234.0, dtype=torch.bfloat16, device=DEV)
    lib = L.load()
    L.check(lib.vb_attention(qkv.data_ptr(), L.VB_BF16, M, B, H, 64, cu.data_ptr(), L.ptr(tl), L.ptr(sl), SEG1_START,
                             max(lens), mode, out.data_ptr(), L.ptr(kc), L.ptr(vc), H * cap * 64 if cap else 0, cap,
                             None, 0, torch.cuda.current_stream().cuda_stream), "vb_attention")
    torch.cuda.synchronize()
    out = out.cpu()
    r = {"seq": [_sha(out[int(cu[b]):int(cu[b + 1])]) for b in range(B)]}
    if cap:
        r["kcache"], r["vcache"] = _sha(kc), _sha(vc)
    return r


@pytest.mark.parametrize("name", CASES)
def test_attention_wgmma_bits(name):
    want = torch.load(FIXTURE, weights_only=False)[name]
    got = _hashes(name)
    assert set(got) == set(want)
    moved = [b for b, (x, y) in enumerate(zip(got["seq"], want["seq"])) if x != y]
    assert len(got["seq"]) == len(want["seq"]) and not moved, f"{name}: output bits differ in sequences {moved}"
    for k in ("kcache", "vcache"):
        if k in want:
            assert got[k] == want[k], f"{name}: {k} bits differ"


if __name__ == "__main__":
    if "--record" not in sys.argv:
        sys.exit("usage: python tests/test_attention_bitwise_gpu.py --record")
    torch.save({name: _hashes(name) for name in CASES}, FIXTURE)
    print(f"recorded {len(CASES)} cases to {FIXTURE}")
