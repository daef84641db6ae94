"""Host-side logic of the batched engine that needs no GPU: the packed index maps (rows / positions of the
text and audio segments of every utterance) that generate() / _nar() ship to the device in one copy, the validated
per-utterance draws of the seeded sampler, and the checks of an utterance's inputs."""
import math

import numpy as np
import pytest
import torch

from valle_b200.engine import _check_utt, _draws, _seg_ranges


def _naive(starts, lens):
    rows = [s + i for s, n in zip(starts, lens) for i in range(n)]
    pos = [i for n in lens for i in range(n)]
    return rows, pos


def test_seg_ranges_matches_python_loops():
    rng = np.random.default_rng(0)
    for _ in range(50):
        B = int(rng.integers(1, 9))
        lens = rng.integers(0, 40, size=B).tolist()   # ragged, empty segments included
        starts = rng.integers(0, 1000, size=B).tolist()
        rows, pos = _seg_ranges(starts, lens)
        exp_rows, exp_pos = _naive(starts, lens)
        assert rows.tolist() == exp_rows and pos.tolist() == exp_pos
        assert rows.dtype == np.int64 and pos.dtype == np.int64


def test_seg_ranges_empty_and_packed_layout():
    rows, pos = _seg_ranges([5, 9], [0, 0])
    assert rows.size == 0 and pos.size == 0
    # the packed [text_b | audio_b] layout of generate(): text rows then audio rows of each utterance
    S, T = [3, 2], [4, 1]
    cu = np.concatenate([[0], np.cumsum(np.add(S, T))])
    trow, tpos = _seg_ranges(cu[:-1], S)
    arow, apos = _seg_ranges(cu[:-1] + np.asarray(S), T)
    assert trow.tolist() == [0, 1, 2, 7, 8] and tpos.tolist() == [0, 1, 2, 0, 1]
    assert arow.tolist() == [3, 4, 5, 6, 9] and apos.tolist() == [0, 1, 2, 3, 0]
    assert sorted(trow.tolist() + arow.tolist()) == list(range(int(cu[-1])))


def test_draws_expand_one_seed_and_keep_per_utterance_values():
    d = _draws(3, 5, 8, 0.7, 0.9)
    assert [x.seed for x in d] == [5, 6, 7]   # utterance b draws from s + b, as it would alone with seed s + b
    assert {(x.top_k, x.temperature, x.top_p, x.ras_window, x.ras_max) for x in d} == {(8, 0.7, 0.9, 0, 0)}
    d = _draws(3, [9, 0, 2 ** 64 - 1], [1, 5, 1], [1.0, 0.8, 1.3], [1.0, 0.5, 0.95], [None, (4, 0.3), None])
    assert [x.seed for x in d] == [9, 0, 2 ** 64 - 1] and [x.top_k for x in d] == [1, 5, 1]
    assert [x.temperature for x in d] == [1.0, 0.8, 1.3] and [x.top_p for x in d] == [1.0, 0.5, 0.95]
    assert [(x.ras_window, x.ras_max) for x in d] == [(0, 0), (4, 1), (0, 0)]
    t = torch.tensor([3, 4])
    assert [x.seed for x in _draws(2, t, t, 1.0)] == [3, 4]   # tensors of values, one per utterance


def test_draw_seeds_map_to_their_int64_bit_patterns():
    for s in (0, 1, 2 ** 63 - 1, 2 ** 63, 2 ** 63 + 5, 2 ** 64 - 1):
        d = _draws(1, s, 5, 1.0)[0]
        assert d.seed == s
        want = int(np.array([s], dtype=np.uint64).view(np.int64)[0])
        assert d.seed_i64 == want and -2 ** 63 <= d.seed_i64 < 2 ** 63
    assert _draws(1, 2 ** 63, 5, 1.0)[0].seed_i64 == -2 ** 63
    assert _draws(1, 2 ** 64 - 1, 5, 1.0)[0].seed_i64 == -1


def test_draw_ras_max_is_the_python_count_test():
    for (w, t), want in (((100, 0.29), 29), ((3, 1 / 3), 1), ((7, 0.5), 3), ((10, 0.0), 0)):
        assert _draws(1, 0, 5, 1.0, ras=(w, t))[0].ras_max == want, (w, t)
    for w in (1, 2, 3, 7, 10, 64, 100, 256):   # count > ras_max exactly when count / K > t
        for t in (0.0, 0.1, 0.29, 1 / 3, 0.5, 0.7, 0.999):
            d = _draws(1, 0, 5, 1.0, ras=(w, t))[0]
            assert d.ras_window == w
            assert all((c > d.ras_max) == (c / w > t) for c in range(w + 1)), (w, t)


def test_draw_greedy_is_top_k_1_without_ras():
    assert _draws(1, 0, 1, 0.5, 0.3)[0].greedy
    assert not _draws(1, 0, 1, 1.0, ras=(8, 0.1))[0].greedy
    assert not _draws(1, 0, 5, 1.0)[0].greedy
    assert not _draws(1, 0, -100, 1.0)[0].greedy
    assert [x.greedy for x in _draws(2, 0, [1, 1], 1.0, ras=[None, (4, 0.5)])] == [True, False]


@pytest.mark.parametrize("kw, match", [
    (dict(seed=-1), "seed"), (dict(seed=2 ** 64), "seed"), (dict(seed=2 ** 64 - 2), "seed"),
    (dict(seed=[1, 2]), "seed"), (dict(top_k=[5, 5]), "top_k"),
    (dict(temperature=0.0), "temperature"), (dict(temperature=-1.0), "temperature"),
    (dict(temperature=math.inf), "temperature"), (dict(temperature=math.nan), "temperature"),
    (dict(temperature=[1.0, 1.0, 0.5]), "temperature"),
    (dict(top_p=0.0), "top_p"), (dict(top_p=1.01), "top_p"), (dict(top_p=-1.0), "top_p"),
    (dict(top_p=math.nan), "top_p"), (dict(top_p=[0.5, 0.5, 0.5, 2.0]), "top_p"),
    (dict(ras=(0, 0.1)), "window"), (dict(ras=(257, 0.1)), "window"), (dict(ras=(8.0, 0.1)), "window"),
    (dict(ras=(True, 0.1)), "window"), (dict(ras=(8, 1.0)), "threshold"), (dict(ras=(8, -0.1)), "threshold"),
    (dict(ras=(8, math.nan)), "threshold"), (dict(ras=[(8, 0.1)] * 3), "ras"), (dict(ras=(8, 0.1, 2)), "pair"),
])
def test_draw_argument_errors(kw, match):
    args = dict(seed=1, top_k=5, temperature=1.0, top_p=1.0, ras=None)
    args.update(kw)
    with pytest.raises(ValueError, match=match):
        _draws(2 if "ras" in kw else 4, **args)


def test_utterance_checks():
    text, prompt = torch.tensor([3, 4, 5]), torch.zeros((6, 8), dtype=torch.int64)
    _check_utt("utterance 0", text, prompt, 8)
    for t, p in ((text[None], prompt), (text[:0], prompt), (text, prompt[:, :7]), (text, prompt[0])):
        with pytest.raises(ValueError, match="utterance 0"):
            _check_utt("utterance 0", t, p, 8)
    bad_first = prompt.clone()
    bad_first[2, 0] = 1025
    bad_rest = prompt.clone()
    bad_rest[2, 3] = 1024
    for t, p, what in ((torch.tensor([3, 512]), prompt, "phoneme"), (torch.tensor([-1]), prompt, "phoneme"),
                       (text, bad_first, "first codebook"), (text, bad_rest, "prompt code id 1024")):
        with pytest.raises(IndexError, match=what):
            _check_utt("utterance 0", t, p, 8)
    prompt[:, 0] = 1024                       # <BOS> row of the first codebook's tables
    _check_utt("utterance 0", text, prompt, 8)


def test_layernorm_fold_identity_of_the_decode_chain():
    """The algebra behind vb_ln_fold (include/valle_b200.h): LayerNorm(x) W^T + b = rstd (x (W gamma)^T - mean c) + d with
    c = row sums of the folded weights and d = b + W beta, the moments taken over split k-ranges and added up -- what
    gemm_decode_x_kernel and its consumers compute on the device (here in torch fp64 against F.layer_norm, and with the
    bf16 roundings of the device path against its own tolerance)."""
    import torch
    import torch.nn.functional as F
    g = torch.Generator().manual_seed(3)
    B, K, N, eps = 5, 256, 96, 1e-5
    x = torch.randn(B, K, generator=g, dtype=torch.float64) * 1.7 + 0.3
    W = torch.randn(N, K, generator=g, dtype=torch.float64) / 16
    gamma = 1 + 0.1 * torch.randn(K, generator=g, dtype=torch.float64)
    beta = 0.1 * torch.randn(K, generator=g, dtype=torch.float64)
    b = torch.randn(N, generator=g, dtype=torch.float64)
    ref = F.linear(F.layer_norm(x, (K,), gamma, beta, eps), W, b)
    wf = W * gamma
    c, d = wf.sum(1), b + W @ beta
    # moments as per-split partial sums over k-ranges (4 splits), then added up
    s1 = sum(x[:, i:i + 64].sum(1) for i in range(0, K, 64))
    s2 = sum((x[:, i:i + 64] ** 2).sum(1) for i in range(0, K, 64))
    mean = s1 / K
    rstd = torch.rsqrt(s2 / K - mean * mean + eps)
    acc = sum(x[:, i:i + 64] @ wf[:, i:i + 64].T for i in range(0, K, 64))
    out = rstd[:, None] * (acc - mean[:, None] * c[None, :]) + d[None, :]
    assert torch.allclose(out, ref, atol=1e-10, rtol=1e-10)
    # device roundings: x and W gamma in bf16, c summed from the ROUNDED folded weights, fp32 accumulation
    xb, wfb = x.float().bfloat16().float(), wf.float().bfloat16().float()
    accb = xb @ wfb.T
    outb = rstd.float()[:, None] * (accb - mean.float()[:, None] * wfb.sum(1)[None, :]) + d.float()[None, :]
    assert (outb.double() - ref).abs().max() < 3e-2
