"""Host logic of best-of-n decoding (ValleEngine.generate(num_samples=, return_scores=)): the argument checks and the
repeated list that the candidates stand for.  No GPU needed."""
import pytest
import torch

from valle_b200.engine import _candidates, _check_num_samples, _draws


def _check(n, seed=1, scores=False, trace=None, forced=None, host=False, bf16_rows=64):
    return _check_num_samples(n, seed, scores, trace, forced, host, bf16_rows)


def test_num_samples_checks():
    assert _check(1) == 1 and _check(4) == 4 and _check(64) == 64
    assert _check(1, seed=None) == 1                       # n = 1 without scores is today's call
    assert _check(100, bf16_rows=None) == 100              # fp32: no group limit
    for bad in (0, -3, 2.0, "2", True, None):
        with pytest.raises(ValueError, match="num_samples"):
            _check(bad)
    with pytest.raises(ValueError, match="seed"):
        _check(2, seed=None)
    with pytest.raises(ValueError, match="seed"):
        _check(1, seed=None, scores=True)
    with pytest.raises(ValueError, match="sample_on_host"):
        _check(2, host=True)
    with pytest.raises(ValueError, match="sample_on_host"):
        _check(1, scores=True, host=True)
    with pytest.raises(ValueError, match="test hooks"):
        _check(2, trace={"steps": {0}})
    with pytest.raises(ValueError, match="test hooks"):
        _check(2, forced=[torch.zeros(3, 8)])
    with pytest.raises(ValueError, match="forced"):
        _check(1, scores=True, forced=[torch.zeros(3, 8)])
    assert _check(1, scores=True, trace={"steps": {0}}) == 1
    with pytest.raises(ValueError, match="at most 64"):
        _check(65)


def test_candidates_are_the_repeated_list():
    B, n = 3, 4
    seeds, per, ras = _candidates(B, n, 10, dict(top_k=[1, 5, 9], temperature=0.7, mnt=None), [None, (8, 0.5), None])
    assert seeds == 10                                      # an int seed: s + row, row = b n + j
    assert per == dict(top_k=[1] * 4 + [5] * 4 + [9] * 4, temperature=0.7, mnt=None)
    assert ras == [None] * 4 + [(8, 0.5)] * 4 + [None] * 4
    d = _draws(B * n, seeds, per["top_k"], per["temperature"], 1.0, ras)
    assert [x.seed for x in d] == [10 + b * n + j for b in range(B) for j in range(n)]
    seeds, _, ras = _candidates(B, n, [100, 200, 2**64 - 4], {}, (8, 0.5))
    assert seeds == [100 + j for j in range(n)] + [200 + j for j in range(n)] + [2**64 - 4 + j for j in range(n)]
    assert ras == (8, 0.5)                                  # one pair for every utterance stays one pair
    with pytest.raises(ValueError, match="seed"):           # seed[b] + j must stay below 2**64
        _draws(B * n, _candidates(B, n, [0, 0, 2**64 - 2], {}, None)[0], 1, 1.0)
    for bad in (dict(top_k=[1, 2]), dict(texts=[torch.zeros(3)] * 4)):
        with pytest.raises(ValueError, match="values for 3 utterances"):
            _candidates(B, n, 0, bad, None)
    with pytest.raises(ValueError, match="seed: 2 values"):
        _candidates(B, n, [1, 2], {}, None)
    with pytest.raises(ValueError, match="ras: 2 values"):
        _candidates(B, n, 1, {}, [None, None])
