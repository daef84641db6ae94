"""The float64 attention reference of tests/attention_oracle64.py, checked without a GPU: its masks against the
kernels' RowMask rule, its error bound against float32 / bf16 emulations of each kernel path (which it must accept
with room to spare), and its planted keys against every single-key omission or leak and a dropped key tile (each of
which it must reject).  The cases are the GPU cases of tests/test_attention_oracle64_gpu.py with fewer sequences and
heads."""
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

import attention_oracle64 as A  # noqa: E402

# A correct kernel's arithmetic stays under the bound.  Long rows, where many roundings average out, stay near 0.1
# to 0.5 of it; on rows of one or two keys the bf16 rounding of P and of the output can line up and reach 0.85.
ACCEPT = 0.9
REJECT = 4.0       # every planted mistake exceeds the bound this many times over


def _small(name):
    """the CPU copy of a GPU case: 3 sequences (sweeps: all) and 4 heads (sweeps: 2)"""
    if name.startswith("sweep_"):
        return A.make_case(name, H=2)
    return A.make_case(name, B=3, H=4)


def _mask_params():
    for mode in A.MODES:
        for seg1_start in (0, 1, 60, 64, 65, 150):
            for L, S, c1 in A._sweep_seqs(mode, seg1_start) + [(1500, 47, 1350), (1500, 0, 700), (400, 59, 340)]:
                if mode.startswith("padded") and (S > seg1_start or c1 > max(L - seg1_start, 0)):
                    continue
                if mode in ("full", "valle_ar") and seg1_start:
                    continue
                yield mode, L, min(S, L), c1, seg1_start


def test_masks_match_the_row_mask_rule():
    n = 0
    for mode, L, S, c1, s1 in _mask_params():
        vis = A.visible(mode, L, S, c1, s1)
        rule = A.row_mask_rule(mode, L, S, c1, s1)
        assert torch.equal(vis, rule), (mode, L, S, c1, s1)
        empty = set(torch.nonzero(~vis.any(1)).flatten().tolist())
        assert empty == A.empty_rows_rule(mode, L, S, c1, s1), (mode, L, S, c1, s1)
        n += 1
    assert n > 500
    # a sequence with rows that see nothing: the reference returns them as a set, with O = A = 0
    vis = A.visible("padded_ar", 130, 0, 5, 64)
    q, k, v = (torch.randn(2, 130, 64) for _ in range(3))
    ref = A.attention64(q, k, v, vis)
    assert ref.empty == set(range(64))
    assert ref.O[:, :64].abs().max() == 0 and ref.A[:, :64].abs().max() == 0
    assert torch.isfinite(ref.O).all()


def test_reference_matches_torch_softmax():
    b = _small("ragged_padded_ar")
    for i in range(len(b.lens)):
        q, k, v = (t.double() for t in b.heads(b.qkv, i))
        vis = b.vis(i)
        s = (q @ k.transpose(-1, -2) / 8).masked_fill(~vis, float("-inf"))
        want = torch.softmax(s, -1) @ v
        got = A.attention64(q, k, v, vis).O
        assert torch.allclose(got, want, rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("name", A.case_names())
def test_bound_accepts_kernel_emulation(name):
    b = _small(name)
    worst = {}
    for kind in A.KINDS:
        src = b.qkv if kind == "simt_f32" else b.qkv.bfloat16().float()
        r = 0.0
        for i in range(len(b.lens)):
            q, k, v = b.heads(src, i)
            vis = b.vis(i)
            ref = A.attention64(q, k, v, vis)
            got = A.emulate(q.contiguous(), k.contiguous(), v.contiguous(), vis, kind)
            r = max(r, A.ratio(got, ref, A.bound(ref, kind)))
        worst[kind] = r
    print(f"{name}: emulated error / bound {worst}")
    assert all(r < ACCEPT for r in worst.values()), worst


def _row(q, k, v, keys):
    """float64 attention of one query row q [H, 64] over keys k, v [H, n, 64] where `keys` [n] is True"""
    s = (q[:, None, :] @ k.transpose(-1, -2))[:, 0] / 8
    s = s.masked_fill(~keys, float("-inf"))
    return (torch.softmax(s, -1)[:, None, :] @ v)[:, 0]


@pytest.mark.parametrize("name", A.case_names())
def test_bound_rejects_planted_mistakes(name):
    """every beacon's key omitted (visible) or let through (forbidden), alone, and the last key tile of every 128-row
    block dropped, exceed the bf16 bound (the loosest) REJECT times over"""
    b = _small(name)
    src = b.qkv.bfloat16().float()
    D = b.H * A.HD
    cu = b.cu
    per_seq = {}
    for bc in b.beacons:
        per_seq.setdefault(bc.seq, []).append(bc)
    least, n, n_drop, least_drop = float("inf"), 0, 0, float("inf")
    for i in range(len(b.lens)):
        L = b.lens[i]
        q, k, v = (t.double() for t in b.heads(src, i))
        vis = b.vis(i)
        ref = A.attention64(q, k, v, vis)
        bnd = A.bound(ref, "wgmma")
        nxt = src[cu[i] + L:cu[i] + L + 1].double() if i + 1 < len(b.lens) else torch.zeros(1, 3 * D, dtype=torch.float64)
        k1 = torch.cat([k, nxt[:, D:2 * D].view(1, b.H, A.HD).transpose(0, 1)], 1)
        v1 = torch.cat([v, nxt[:, 2 * D:].view(1, b.H, A.HD).transpose(0, 1)], 1)
        for bc in per_seq.get(i, []):
            got = _row(q[:, bc.row], k1, v1, A.beacon_vis(vis, bc))
            # a row left without keys is NaN: the kernels' 0 / 0 would be too
            r = float(((got - ref.O[:, bc.row]).abs() / bnd[:, bc.row]).nan_to_num(nan=float("inf")).max())
            assert r > REJECT, (name, i, bc, r)
            least, n = min(least, r), n + 1
        dropped = A.drop_last_tile(b.mode, vis, b.S[i])
        if not torch.equal(dropped, vis):
            got = A.attention64(q, k, v, dropped).O
            r = float(((got - ref.O).abs() / bnd).max())
            assert r > REJECT, (name, i, "dropped tile", r)
            least_drop, n_drop = min(least_drop, r), n_drop + 1
    assert n > 0 or all(not A.visible(b.mode, L, S, c, b.seg1_start).any()
                        for L, S, c in zip(b.lens, b.S, b.c1))
    print(f"{name}: {n} planted keys omitted / leaked, least error / bound {least:.1f}; "
          f"{n_drop} sequences with a dropped tile, least {least_drop:.1f}")
