import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (H100, sm_90a); select with -m gpu")


def load_golden(name):
    import torch
    return torch.load(os.path.join(GOLDEN, name), weights_only=False)


def build_model(cfg, seed, device="cpu"):
    """valle_b200 VALLE with the reference's default init under torch.manual_seed(seed)."""
    import torch
    from valle_b200.models import VALLE
    torch.manual_seed(seed)
    m = VALLE(cfg["d_model"], cfg["nhead"], cfg["num_layers"], norm_first=True, add_prenet=cfg.get("add_prenet", False),
              prefix_mode=cfg["prefix_mode"], share_embedding=True, nar_scale_factor=cfg.get("nar_scale_factor", 1.0),
              prepend_bos=cfg.get("prepend_bos", False), num_quantizers=cfg["num_quantizers"]).eval()
    return m.to(device)


def assert_checksums(model, ck):
    import torch
    from oracle.valle_oracle import weight_checksums
    got = weight_checksums(model.state_dict())
    assert list(got.keys()) == list(ck.keys())
    for k in got:
        assert torch.equal(got[k], ck[k]), f"weights differ from the reference init at {k}"


@pytest.fixture(scope="session")
def lib():
    from valle_b200 import _lib
    return _lib.load()
