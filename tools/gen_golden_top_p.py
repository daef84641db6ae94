"""Writes tests/golden/tiny_topp.pt from the UNMODIFIED reference (loaded through oracle/ref_loader.py, run on the CPU in
fp32), in the manner of oracle/gen_golden.py::gen_topk.

    python tools/gen_golden_top_p.py

The reference's `inference` always calls `topk_sampling(..., top_p=1.0, ...)` (valle.py:1040-1043).  This script
wraps the loaded module's `topk_sampling` name so that those calls draw with a fixed top_p instead, and records the
codes of the tiny prefix_mode-1 model for a few (top_k, top_p, temperature, torch seed) cases.  It also stores the
masks the reference's `top_k_top_p_filtering` keeps on seeded logit rows without exact ties (one (top_k, top_p) per
row), for tests/test_sampling_nucleus.py.
"""
from __future__ import annotations

import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from oracle import ref_loader  # noqa: E402
from oracle.gen_golden import build_reference, checksums, make_inputs, save  # noqa: E402

CASES = ((-100, 0.9, 1.0, 11), (50, 0.8, 0.9, 12), (5, 0.5, 1.2, 13), (-100, 0.3, 1.0, 14))
ROW_TOPK = (0, 5, 50, 1025)
ROW_TOPP = (1e-4, 0.1, 0.5, 0.9, 0.99)


def _with_top_p(own, p):
    def topk_sampling(logits, top_k=10, top_p=1.0, temperature=1.0):
        return own(logits, top_k=top_k, top_p=p, temperature=temperature)
    return topk_sampling


def main():
    ref = ref_loader.load_reference()
    mod = sys.modules[ref_loader._PREFIX + ".models.valle"]
    own = mod.topk_sampling
    d, h, l, pm, seed = 256, 4, 2, 1, 0
    m = build_reference(ref, d, h, l, pm, seed)
    g = torch.Generator().manual_seed(23)
    x, y = make_inputs(g, 7, 18)
    xl = torch.tensor([x.shape[1]], dtype=torch.int32)
    cases = []
    try:
        for top_k, top_p, temp, tseed in CASES:
            mod.topk_sampling = _with_top_p(own, top_p)
            torch.manual_seed(tseed)
            with torch.no_grad():
                codes = m.inference(x, xl, y, None, top_k=top_k, temperature=temp)
            print(f"top_p case top_k={top_k} top_p={top_p} T={temp} seed={tseed}: {codes.shape[1]} frames")
            cases.append(dict(top_k=top_k, top_p=top_p, temperature=temp, torch_seed=tseed,
                              codes=codes.to(torch.int16)))
    finally:
        mod.topk_sampling = own

    # filter masks on seeded rows: no two logits of a row are equal, so the reference's (unstable) sort is one order
    gr = torch.Generator().manual_seed(29)
    rows, ks, ps, masks = [], [], [], []
    for r in range(120):
        scale = (0.5, 1.5, 4.0)[r % 3]
        while True:
            lg = torch.randn(1, 1025, generator=gr) * scale
            if torch.unique(lg).numel() == lg.numel():
                break
        k, p = ROW_TOPK[r % len(ROW_TOPK)], ROW_TOPP[(r // len(ROW_TOPK)) % len(ROW_TOPP)]
        out = mod.top_k_top_p_filtering(lg.clone(), top_k=k, top_p=p)
        rows.append(lg[0])
        ks.append(k)
        ps.append(p)
        masks.append(torch.isfinite(out[0]))
    save("tiny_topp.pt", dict(config=dict(d_model=d, nhead=h, num_layers=l, prefix_mode=pm, num_quantizers=8),
                              weight_seed=seed, checksums=checksums(m.state_dict()), x=x, y=y, cases=cases,
                              filter=dict(logits=torch.stack(rows), top_k=torch.tensor(ks, dtype=torch.int32),
                                          top_p=torch.tensor(ps, dtype=torch.float32), mask=torch.stack(masks))))


if __name__ == "__main__":
    main()
