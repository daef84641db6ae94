"""CPU self-checks of the float64 decode-step restatement (tests/decode_step_oracle.py) that the GPU sweep
(tests/test_decode_step_gpu.py) compares the engine's decode kernels with."""
import pytest
import torch

from oracle import valle_oracle as O

import decode_step_oracle as D
import postln_oracle as P

PREFIX = "ar_decoder"


def random_state_dict(d, H, dff, n_layer, norm_first, seed, n_vocab=37):
    """float64 weights with non-trivial biases and LayerNorm affines; returns (sd, head weight)"""
    g = torch.Generator().manual_seed(seed)
    r = lambda *s: torch.randn(*s, generator=g, dtype=torch.float64)   # noqa: E731
    sd = {}
    for i in range(n_layer):
        p = f"{PREFIX}.layers.{i}."
        sd[p + "self_attn.in_proj_weight"] = r(3 * d, d) / d ** 0.5
        sd[p + "self_attn.in_proj_bias"] = 0.1 * r(3 * d)
        sd[p + "self_attn.out_proj.weight"] = r(d, d) / d ** 0.5
        sd[p + "self_attn.out_proj.bias"] = 0.1 * r(d)
        sd[p + "linear1.weight"] = r(dff, d) / d ** 0.5
        sd[p + "linear1.bias"] = 0.1 * r(dff)
        sd[p + "linear2.weight"] = r(d, dff) / dff ** 0.5
        sd[p + "linear2.bias"] = 0.1 * r(d)
        for n in ("norm1", "norm2"):
            sd[p + n + ".weight"] = 1.0 + 0.2 * r(d)
            sd[p + n + ".bias"] = 0.1 * r(d)
    if norm_first:
        sd[PREFIX + ".norm.weight"] = 1.0 + 0.2 * r(d)
        sd[PREFIX + ".norm.bias"] = 0.1 * r(d)
    return sd, r(n_vocab, d) / d ** 0.5


@pytest.mark.parametrize("norm_first", [True, False])
def test_growing_cache_matches_the_causal_encoder(norm_first):
    """fp32 chain, float64: grow the cache from empty one token at a time (n_gen = i + 1, no text or prompt); step i's
    output (after the final norm of a pre-LN stack) is row i of the whole sequence through the oracle's encoder under
    the causal mask ar_inference_mask(0, L)"""
    d, H, dff, n_layer, Lq = 128, 2, 256, 2, 9
    sd, head = random_state_dict(d, H, dff, n_layer, norm_first, seed=1)
    X = torch.randn(Lq, d, generator=torch.Generator().manual_seed(2), dtype=torch.float64)
    cfg = O.OracleConfig(d_model=d, nhead=H, num_layers=n_layer)
    enc = O.encoder if norm_first else P.encoder_postln
    ref = enc(sd, PREFIX, X[None], cfg, blocked=O.ar_inference_mask(0, Lq))[0]
    kc = torch.full((n_layer, 1, H, Lq, 64), float("nan"), dtype=torch.float64)   # never read before written
    vc = kc.clone()
    z = torch.zeros(1, dtype=torch.int32)
    for i in range(Lq):
        out = D.decode_step(sd, PREFIX, head, X[i:i + 1], kc, vc, z, z, torch.tensor([i + 1]), z, H, "fp32",
                            norm_first=norm_first)
        assert int(out.kv_len[0]) == i + 1
        kc[:, 0, :, i] = out.k_new[:, 0]
        vc[:, 0, :, i] = out.v_new[:, 0]
        y = out.x[0]
        if norm_first:
            y = O.layer_norm(y, sd[PREFIX + ".norm.weight"], sd[PREFIX + ".norm.bias"])
        assert torch.allclose(out.logits[0], y @ head.T, rtol=0, atol=1e-10)
        err = float((y - ref[i]).abs().max())
        assert err < 1e-10, f"step {i}: {err}"


def _random_step_state(d, H, n_layer, B, cap, seed, offsets=(0.0, 4.0, 16.0, 64.0)):
    g = torch.Generator().manual_seed(seed)
    z = torch.randn(B, d, generator=g, dtype=torch.float64)
    z = (z - z.mean(1, keepdim=True)) / z.std(1, unbiased=False, keepdim=True)
    x = (z + torch.tensor([offsets[b % len(offsets)] for b in range(B)], dtype=torch.float64)[:, None]).float()
    kc = torch.randn(n_layer, B, H, cap, 64, generator=g).to(torch.bfloat16).float()
    vc = torch.randn(n_layer, B, H, cap, 64, generator=g).to(torch.bfloat16).float()
    text = torch.randint(0, cap // 2, (B,), generator=g, dtype=torch.int32)
    prompt = torch.randint(0, cap // 4, (B,), generator=g, dtype=torch.int32)
    n_gen = torch.randint(0, cap // 4, (B,), generator=g, dtype=torch.int32)
    return x, kc, vc, text, prompt, n_gen, torch.zeros(B, dtype=torch.int32)


def test_fold_identity_without_rounding():
    """rstd (x (gamma o W)^T - mean c) + b + beta W^T == LayerNorm(x) W^T + b: the folded chain without its roundings
    is the unfolded chain, for rows with |mean| / sigma up to 64"""
    d, H, dff, n_layer, B, cap = 128, 2, 256, 2, 8, 40
    sd, head = random_state_dict(d, H, dff, n_layer, True, seed=3)
    st = _random_step_state(d, H, n_layer, B, cap, seed=4)
    a = D.decode_step(sd, PREFIX, head, *st, H, "bf16_folded", rounding=False)
    b = D.decode_step(sd, PREFIX, head, *st, H, "bf16_unfolded", rounding=False)
    for name in ("x", "k_new", "v_new", "q", "logits"):
        err = float((getattr(a, name) - getattr(b, name)).abs().max())
        assert err < 1e-10, f"{name}: {err}"


@pytest.mark.parametrize("chain", ["bf16_unfolded", "bf16_folded", "bf16_postln"])
def test_rounding_points_make_a_bf16_sized_difference(chain):
    """each bf16 chain differs from its own unrounded algebra by a bf16-sized amount -- neither zero (a rounding point
    that does nothing) nor O(1) (one that rounds the wrong thing) -- and its appended K / V rows are bf16 values"""
    norm_first = chain != "bf16_postln"
    d, H, dff, n_layer, B, cap = 128, 2, 256, 2, 4, 40
    sd, head = random_state_dict(d, H, dff, n_layer, norm_first, seed=5)
    st = _random_step_state(d, H, n_layer, B, cap, seed=6, offsets=(0.0,))
    got = D.decode_step(sd, PREFIX, head, *st, H, chain, norm_first=norm_first)
    ref = D.decode_step(sd, PREFIX, head, *st, H, chain, norm_first=norm_first, rounding=False)
    for name in ("x", "logits"):
        a, b = getattr(got, name), getattr(ref, name)
        rel = float((a - b).abs().max() / b.abs().max())
        assert 2.0 ** -14 < rel < 2.0 ** -4, f"{name}: relative difference {rel}"
    assert torch.equal(got.k_new, D.bf16(got.k_new)) and torch.equal(got.v_new, D.bf16(got.v_new))
    assert not torch.equal(ref.k_new, D.bf16(ref.k_new))
    # the fp32 chain has no rounding point at all
    f = D.decode_step(sd, PREFIX, head, *st, H, "fp32", norm_first=norm_first)
    f0 = D.decode_step(sd, PREFIX, head, *st, H, "fp32", norm_first=norm_first, rounding=False)
    assert torch.equal(f.logits, f0.logits)


def test_kv_length_clamp():
    """kv_len = clamp(text + prompt + n_gen, 1, cap), as the kernels take it"""
    got = D.kv_lengths([0, 0, 3, 10, 10], [0, 0, 4, 5, 5], [0, 1, 0, 10, 1], 16)
    assert got.tolist() == [1, 1, 7, 16, 16]
