"""Host logic of beam search (ValleEngine.generate(num_beams=)): the argument checks.  No GPU needed."""
import pytest
import torch

from valle_b200.engine import _candidates, _check_num_beams


def _check(n, seed=None, top_k=1, top_p=1.0, ras=None, num_samples=1, trace=None, forced=None, host=False,
           fp8=False):
    return _check_num_beams(n, seed, top_k, top_p, ras, num_samples, trace, forced, host, fp8)


def test_num_beams_checks():
    assert [_check(n) for n in (1, 2, 7, 16)] == [1, 2, 7, 16]
    # n = 1 is today's call: every sampler argument and hook stays allowed
    assert _check(1, seed=3, top_k=50, top_p=0.9, ras=(10, 0.2), num_samples=4, trace={}, host=True, fp8=True) == 1
    for bad in (0, -1, 17, 2.0, "2", True, None):
        with pytest.raises(ValueError, match="num_beams must be an int in"):
            _check(bad)
    for kw in (dict(seed=0), dict(top_k=5), dict(top_k=-100), dict(top_k=[1, 1]), dict(top_p=0.9),
               dict(top_p=[1.0, 1.0]), dict(ras=(10, 0.2))):
        with pytest.raises(ValueError, match="no seed, top_k, top_p or ras"):
            _check(4, **kw)
    for ns in (2, True, 1.0):
        with pytest.raises(ValueError, match="num_samples"):
            _check(2, num_samples=ns)
    with pytest.raises(ValueError, match="sample_on_host"):
        _check(2, host=True)
    with pytest.raises(ValueError, match="test hooks"):
        _check(2, trace={"steps": {0}})
    with pytest.raises(ValueError, match="test hooks"):
        _check(2, forced=[torch.zeros(3, 8)])
    with pytest.raises(ValueError, match="FP8"):
        _check(2, fp8=True)


def test_beams_expand_like_candidates():
    """the n beams of utterance b are rows b n .. b n + n - 1, each with the utterance's arguments"""
    B, n = 3, 4
    _, per, _ = _candidates(B, n, 0, dict(texts=["a", "b", "c"], max_new_tokens=[5, 6, 7], enroll_lens=None), None)
    assert per["texts"] == ["a"] * 4 + ["b"] * 4 + ["c"] * 4
    assert per["max_new_tokens"] == [5] * 4 + [6] * 4 + [7] * 4
    assert per["enroll_lens"] is None
