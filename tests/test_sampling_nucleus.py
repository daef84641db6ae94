"""CPU checks of nucleus (top-p) filtering against the unmodified reference's `top_k_top_p_filtering`
(tests/golden/tiny_topp.pt, written by tools/gen_golden_top_p.py): the engine's torch filter and the numpy restatement
of the device sampler (tests/sampling_oracle.py) keep the reference's sets."""
import numpy as np
import torch

import sampling_oracle as S
from conftest import load_golden


def _rows():
    f = load_golden("tiny_topp.pt")["filter"]
    return f["logits"], f["top_k"].tolist(), f["top_p"].tolist(), f["mask"]


def test_torch_filter_reproduces_the_reference_masks():
    from valle_b200.models.valle import top_k_top_p_filtering
    lg, ks, ps, masks = _rows()
    for r in range(lg.shape[0]):
        out = top_k_top_p_filtering(lg[r:r + 1].clone(), top_k=ks[r], top_p=ps[r])
        assert torch.equal(torch.isfinite(out[0]), masks[r]), (r, ks[r], ps[r])


def test_restated_nucleus_keeps_the_reference_set():
    """The restatement keeps the reference's set on every row, except where the boundary mass lies within fp32
    rounding of top_p (the reference divides by the softmax sum, the restatement multiplies top_p by it)"""
    lg, ks, ps, masks = _rows()
    near = 0
    for r in range(lg.shape[0]):
        x = lg[r].numpy().astype(np.float32)
        keep = S.top_k_set(x, ks[r])
        order, j, slack = S.nucleus(x, keep, ps[r])
        got = np.zeros_like(keep)
        got[order[: j + 1]] = True
        if np.array_equal(got, masks[r].numpy()):
            continue
        assert slack < S.BOUNDARY, (r, ks[r], ps[r], slack)
        assert abs(int(got.sum()) - int(masks[r].sum())) == 1, r
        near += 1
    print(f"{near} of {lg.shape[0]} rows differ at a boundary within fp32 rounding of top_p")
    assert near <= lg.shape[0] // 20


def test_restated_nucleus_edges():
    x = np.array([3.0, 1.0, 3.0, -np.inf, 0.5], dtype=np.float32)
    keep = np.ones(5, dtype=bool)
    order, j, _ = S.nucleus(x, keep, 1e-6)
    assert order.tolist()[:3] == [0, 2, 1] and j == 0            # equal values in ascending id order; p -> 0: argmax
    order, j, _ = S.nucleus(x, keep, 1.0)
    assert j <= 4
    # p = 1 draws exactly what the top-k sampler draws
    g = torch.Generator().manual_seed(3)
    for r in range(20):
        l = (torch.randn(1025, generator=g) * 2).numpy()
        for k in (-100, 7):
            a = S.draw(l, 99 + r, r, k, 0.8, top_p=1.0)
            x = S.scaled(l, 0.8)
            sc = np.where(S.top_k_set(x, k), x + S.gumbel(99 + r, r, np.arange(1025)), -np.inf)
            assert a == int(np.argmax(sc))
