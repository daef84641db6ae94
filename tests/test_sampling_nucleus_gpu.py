"""GPU tests of nucleus (top-p) and repetition-aware sampling (RAS) in the seeded device sampler
(vb_sample_logits_ex, vb_ar_state.top_p / ras_window / ras_max, ValleEngine.generate(top_p=, ras=)).

The ids are compared with the numpy restatement of include/valle_b200.h (tests/sampling_oracle.py).  Its expf / logf
may differ from the device's in the last bit, so a device id may differ from the restated one only where that decides
the draw (a near-tie of the perturbed scores, or a prefix sum within fp32 rounding of top_p * Z); such rows are
counted and bounded."""
import math

import numpy as np
import pytest
import torch

import sampling_oracle as S
from conftest import load_golden
from test_sampling_gpu import _batch, _model, _rows
from test_stream_gpu import _check_equal, _requests, _stream, tuned
from test_stream_gpu import _model as _stream_model
from valle_b200.engine import StreamRequest, _draws

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
EOS = 1024


def _ids(lg, k, T, seeds, steps, top_p=None, window=None, rmax=None, hist=None):
    from valle_b200 import ops
    return ops.sample_logits(lg.to(DEV), k, T, seeds, steps, top_p=top_p, ras_window=window, ras_max=rmax,
                             tokens=hist).cpu().tolist()


def _check_rows(ids, lg, seeds, steps, ks, ts, ps, ws=None, rms=None, hist=None):
    """every device id is the restated one, or one a last-bit difference of expf / logf may give; returns the count of
    the latter"""
    near = 0
    for r, d in enumerate(ids):
        h = () if hist is None else hist[r].numpy()
        want, others = S.candidates(lg[r].numpy(), seeds[r], int(steps[r]), ks[r], ts[r], ps[r],
                                    0 if ws is None else ws[r], 0 if rms is None else rms[r], h)
        assert d == want or d in others, (r, d, want, ks[r], ts[r], ps[r])
        near += d != want
    return near


# ------------------------------------------------------------------------------------------- 1. ids
@pytest.mark.parametrize("V", [1025, 1280])
def test_nucleus_ids_match_the_restatement(V):
    g = torch.Generator().manual_seed(V)
    R = 3072
    lg = torch.randn(R, V, generator=g) * torch.tensor([0.5, 2.0, 5.0])[torch.arange(R) % 3, None]
    lg[1::4] = torch.round(lg[1::4] * 2) / 2                 # many exact ties, some straddling the nucleus boundary
    lg[2::8, : V // 3] = -math.inf                           # -inf entries that top-k keeps when it keeps everything
    ks = [(-100, 1, 5, 50, 1024, V)[i % 6] for i in range(R)]
    ts = [(1.0, 0.7, 1.3)[i % 3] for i in range(R)]
    ps = [(1e-7, 0.3, 0.9, 0.99, 1.0)[(i // 7) % 5] for i in range(R)]
    seeds = [(i * 0x9E3779B97F4A7C15 + 11) % (1 << 64) for i in range(R)]
    steps = torch.randint(0, 3000, (R,), generator=g, dtype=torch.int32)
    kt, tt = torch.tensor(ks, dtype=torch.int32), torch.tensor(ts)
    ids = _ids(lg, kt, tt, seeds, steps, top_p=torch.tensor(ps))
    near = _check_rows(ids, lg, seeds, steps, ks, ts, ps)
    print(f"V={V}: {near} of {R} ids differ from numpy at a last-bit decision")
    assert near <= R // 100
    base = _ids(lg, kt, tt, seeds, steps)
    for r in range(R):
        if ps[r] == 1.0:                                     # p = 1: exactly vb_sample_logits's id
            assert ids[r] == base[r], r
        if ps[r] == 1e-7:                                    # p -> 0: the largest l' (smallest id on ties)
            l = lg[r].numpy()
            assert ids[r] == int(np.argmax(l if ks[r] == 1 else S.scaled(l, ts[r]))), r


def test_nucleus_boundary_ties_keep_the_lower_ids():
    """Tokens tied at the boundary value: the nucleus takes them in ascending id order, so a boundary that falls
    inside the tie keeps the lower ids only (a draw of a higher one is a bug)"""
    V = 1025
    l = torch.full((V,), -10.0)
    l[[40, 7, 900, 300]] = 2.0                               # four equal tokens of 1/4 each (the rest ~e-12)
    N = 4096
    seeds = list(range(N))
    ids = _ids(l[None].expand(N, V), -100, 1.0, seeds, [0] * N, top_p=0.6)
    assert set(ids) == {7, 40, 300}, sorted(set(ids))       # cumulative 0.25, 0.5, 0.75 > 0.6: ids 7, 40, 300


# ------------------------------------------------------------------------------------------- 2. distribution
@pytest.mark.parametrize("k,p", [(-100, 0.9), (50, 0.5), (-100, 0.2), (1025, 0.99)])
def test_nucleus_draws_from_the_renormalised_nucleus(k, p):
    from scipy.stats import chisquare
    rows, _ = _rows()
    N = 1 << 18
    idx = torch.arange(N, device=DEV)
    seeds, steps = (idx // 64) * 7919 + 5, (idx % 64).to(torch.int32)
    for r in range(rows.shape[0]):
        l = rows[r]
        ids = np.array(_ids(l[None].expand(N, l.numel()), k, 1.0, seeds, steps, top_p=p))
        x = l.numpy().astype(np.float32)
        order, j, _ = S.nucleus(x, S.top_k_set(x, k), p)
        keep = order[: j + 1]
        assert np.isin(ids, keep).all(), f"row {r}: a draw outside the nucleus"
        pr = torch.softmax(l.double()[keep], 0).numpy()
        counts = np.bincount(ids, minlength=l.numel())[keep].astype(np.float64)
        exp = pr * N
        big = exp >= 5
        obs, ex = np.append(counts[big], counts[~big].sum()), np.append(exp[big], exp[~big].sum())
        if ex[-1] == 0:
            obs, ex = obs[:-1], ex[:-1]
        if ex.size < 2:
            continue
        pv = chisquare(obs, ex * obs.sum() / ex.sum()).pvalue
        assert pv > 1e-4, (r, k, p, pv)


# ------------------------------------------------------------------------------------------- 3. RAS
def test_ras_falls_back_exactly_when_the_count_exceeds_ras_max():
    g = torch.Generator().manual_seed(17)
    R, V, W = 1536, 1025, 300
    lg = torch.randn(R, V, generator=g) * 3
    ks = [(-100, 5, 1, 40)[i % 4] for i in range(R)]
    ps = [(1.0, 0.8)[(i // 4) % 2] for i in range(R)]
    ts = [1.0] * R
    seeds = [i * 31 + 1 for i in range(R)]
    kt = torch.tensor(ks, dtype=torch.int32)
    steps = torch.tensor([(3, 9, 64, 200, 256, 299)[i % 6] for i in range(R)], dtype=torch.int32)
    first = _ids(lg, kt, 1.0, seeds, steps, top_p=torch.tensor(ps))
    windows = [(1, 8, 16, 100, 256)[(i // 8) % 5] for i in range(R)]
    rmax = [min(w - 1, (0, 1, 3)[i % 3]) for i, w in enumerate(windows)]
    hist = torch.randint(0, V, (R, W), generator=g, dtype=torch.int32)
    fallbacks = 0
    for r in range(R):
        d, n, w = first[r], int(steps[r]), windows[r]
        h = hist[r]
        h[h == d] = (d + 1) % V
        lo = max(0, n - w)
        c = int(torch.randint(0, min(w, n - lo) + 1, (1,), generator=g)) if r % 5 else min(rmax[r] + 1, n - lo)
        pos = lo + torch.randperm(n - lo, generator=g)[:c]
        h[pos] = d
        h[n:] = d                                            # a previous occupant's codes behind n_gen
        if lo > 0:
            h[: lo] = d                                      # and this utterance's own, outside the window
        fallbacks += S.ras_fallback(d, n, w, rmax[r], h.numpy())
    ids = _ids(lg, kt, 1.0, seeds, steps, top_p=torch.tensor(ps), window=torch.tensor(windows, dtype=torch.int32),
               rmax=torch.tensor(rmax, dtype=torch.int32), hist=hist)
    near = _check_rows(ids, lg, seeds, steps, ks, ts, ps, windows, rmax, hist)
    assert fallbacks >= 100 and R - fallbacks >= 100, fallbacks
    assert near <= R // 100
    # no fallback: the first draw, whatever the history outside the window holds
    for r in range(R):
        if not S.ras_fallback(first[r], int(steps[r]), windows[r], rmax[r], hist[r].numpy()):
            assert ids[r] == first[r], r


# ------------------------------------------------------------------------------------------- 4. traced decode
CHAINS = ["f32", "folded", "unfolded", "postln", "fp8"]


@pytest.mark.parametrize("chain", CHAINS)
def test_traced_native_decode_matches_the_restatement(chain, monkeypatch):
    """Every id of a native decode with top-p and RAS is the restated draw from that step's traced logits, seed, step
    and the codes before it; the decode ends where the stop rule fires"""
    name = "tiny_postln_pm1.pt" if chain == "postln" else "tiny_pm1.pt"
    dtype = torch.float32 if chain == "f32" else torch.bfloat16
    if chain == "unfolded":
        monkeypatch.setenv("VB_DECODE_FOLD", "0")
    g, m = _stream_model(name, dtype, torch.float8_e4m3fn if chain == "fp8" else None)
    eng = m.engine(dtype)
    x, y = g["x"][0], g["y"][0]
    seed, k, T, p, ras = 4242, 8, 1.0, 0.7, (6, 0.2)
    rmax = _draws(1, seed, k, T, p, ras)[0].ras_max
    tr = {"steps": "all"}
    out = eng.generate([x], [y], top_k=k, temperature=T, top_p=p, ras=ras, trace=tr, seed=seed)[0].cpu()
    n = out.shape[0]
    cap = 16 * x.numel() - int(eng.prepend_bos)
    hist = out[:, 0].numpy().astype(np.int32)
    near = fell = 0
    for j in range(n + 1):
        l = tr["ar_logits"][j][0].cpu().numpy()
        want, others = S.candidates(l, seed, j, k, T, p, ras[0], rmax, hist)
        if j < n:
            d = int(out[j, 0])
            assert d == want or d in others, (j, d, want)
            near += d != want
            first = S.candidates(l, seed, j, k, T, p)[0]
            fell += S.ras_fallback(first, j, ras[0], rmax, hist)
            assert int(np.argmax(l)) != EOS and d != EOS
        else:
            assert int(np.argmax(l)) == EOS or want == EOS or j > cap, (j, want)
    print(f"{chain}: {n} frames, {fell} RAS fallbacks, {near} last-bit mismatches")
    assert fell > 0
    assert near <= max(1, n // 50)


# ------------------------------------------------------------------------------------------- 5. invariance
KW = dict(top_k=[-100, 20, 1, 5], temperature=[1.0, 0.8, 1.0, 1.2], top_p=[0.9, 0.6, 1.0, 0.95],
          ras=[(10, 0.1), None, (4, 0.3), (32, 0.5)])


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_batch_equals_each_utterance_alone(dtype):
    g = load_golden("tiny_batch.pt")
    m = _model(g, dtype)
    eng = m.engine()
    texts, prompts = _batch(g)
    s = 99
    outs = eng.generate(texts, prompts, seed=s, **KW)
    for b in range(len(texts)):
        eng._bufs.clear()
        solo = eng.generate([texts[b]], [prompts[b]], seed=s + b, **{k: v[b] for k, v in KW.items()})[0]
        assert torch.equal(solo, outs[b]), b
    x = texts[0]
    one = m.inference(x[None].to(DEV), torch.tensor([x.numel()], dtype=torch.int32), prompts[0][None].to(DEV), None,
                      top_k=-100, temperature=1.0, seed=s, top_p=0.9, ras=(10, 0.1))[0].cpu()
    assert torch.equal(one, outs[0])
    again = m.inference_batch(texts, prompts, seed=s, **KW)
    assert all(torch.equal(a, b) for a, b in zip(again, outs))
    # a top_k == 1 row with RAS is not greedy: its repeats fall back to a draw
    greedy = eng.generate(texts[:1], prompts[:1], top_k=1)[0]
    ras1 = eng.generate(texts[:1], prompts[:1], top_k=1, seed=s, ras=(4, 0.0))[0]
    assert not torch.equal(greedy, ras1)


def test_codes_are_invariant_to_graphs_polling_groups_and_reruns():
    g = load_golden("tiny_batch.pt")
    m = _model(g, torch.bfloat16)
    eng = m.engine()
    texts, prompts = _batch(g)
    kw = dict(seed=7, **KW)
    ref = eng.generate(texts, prompts, **kw)
    assert all(torch.equal(a, b) for a, b in zip(ref, eng.generate(texts, prompts, **kw)))
    assert all(torch.equal(a, b) for a, b in zip(ref, eng.generate(texts, prompts, poll=1, **kw)))
    eng.use_cuda_graph = False
    try:
        assert all(torch.equal(a, b) for a, b in zip(ref, eng.generate(texts, prompts, **kw)))
    finally:
        eng.use_cuda_graph = True
    # B = 70 (two tensor-core groups) == its groups decoded on their own
    t70, p70 = (texts * 18)[:70], (prompts * 18)[:70]
    kw70 = {k: (v * 18)[:70] for k, v in KW.items()}
    out = eng.generate(t70, p70, max_new_tokens=12, seed=500, **kw70)
    a = eng.generate(t70[:64], p70[:64], max_new_tokens=12, seed=500, **{k: v[:64] for k, v in kw70.items()})
    b = eng.generate(t70[64:], p70[64:], max_new_tokens=12, seed=564, **{k: v[64:] for k, v in kw70.items()})
    assert len(out) == 70
    for i, (o, r) in enumerate(zip(out, a + b)):
        assert torch.equal(o, r), i


def _mixed(reqs):
    out = []
    for i, r in enumerate(reqs):
        if r.seed is None:
            out.append(r)
        else:
            out.append(r._replace(top_p=(0.9, 0.7, 1.0)[i % 3], ras=((8, 0.1), None, (3, 0.3))[i % 3]))
    return out


def _solo(m, r):
    x = r.text[None].to(DEV)
    el = None if r.enroll_len is None else torch.tensor([r.enroll_len], dtype=torch.int32)
    return m.inference(x, torch.tensor([x.shape[1]], dtype=torch.int32), r.prompt[None].to(DEV), el, top_k=r.top_k,
                       temperature=r.temperature, max_new_tokens=r.max_new_tokens, seed=r.seed, top_p=r.top_p,
                       ras=r.ras)[0].cpu()


@pytest.mark.parametrize("poll", [1, 32])
def test_stream_with_mixed_top_p_and_ras_equals_solo(poll):
    with tuned(VB_DECODE_NSPLIT=1):
        g, m = _stream_model("tiny_pm1.pt", torch.bfloat16)
        eng = m.engine(torch.bfloat16)
        reqs = _mixed(_requests(g, 10, seeded=True, seed=4))
        assert StreamRequest(*tuple(reqs[0])[:7]).top_p == 1.0           # the old positional field order still works
        eng._bufs.clear()
        n_cap = []
        got = {}
        for idx, codes in eng.generate_stream(reqs, slots=3, poll=poll):
            got[idx] = codes.cpu()
            n_cap.append(eng.captured_launches)
        assert len(set(n_cap)) == 1, n_cap                                # one graph capture for the whole stream
        _check_equal([got[i] for i in range(len(reqs))], [_solo(m, r) for r in reqs])
        _check_equal(_stream(m, reqs, slots=3, poll=poll), [got[i] for i in range(len(reqs))])   # a rerun


# ------------------------------------------------------------------------------------------- 6. reference
def test_host_draw_with_top_p_matches_the_reference_at_fixed_seed():
    """seed=None, sample_on_host: the reference's own topk_sampling with top_p, at the same torch seed, reproduces
    the unmodified reference's codes (tools/gen_golden_top_p.py) bit for bit"""
    g = load_golden("tiny_topp.pt")
    m = _model(g, torch.float32)
    eng = m.engine()
    eng.sample_on_host = True
    try:
        x, y = g["x"].to(DEV), g["y"].to(DEV)
        xl = torch.tensor([x.shape[1]], dtype=torch.int32)
        for c in g["cases"]:
            torch.manual_seed(int(c["torch_seed"]))
            out = m.inference(x, xl, y, None, top_k=int(c["top_k"]), temperature=float(c["temperature"]),
                              top_p=float(c["top_p"])).cpu()
            ref = c["codes"].long()
            assert out.shape == ref.shape and torch.equal(out, ref), (c["top_k"], c["top_p"])
    finally:
        eng.sample_on_host = False


# ------------------------------------------------------------------------------------------- 7. errors
def test_bad_top_p_and_ras_arguments_raise():
    from valle_b200 import _lib as L
    lg = torch.randn(4, 1025, device=DEV)
    hist = torch.zeros((4, 8), dtype=torch.int32)
    for kw in (dict(top_p=0.0), dict(top_p=1.5), dict(top_p=float("nan")), dict(top_p=[0.5, 0.5, 0.5, -0.1]),
               dict(window=257, rmax=0), dict(window=-1, rmax=0), dict(window=4, rmax=-1)):
        with pytest.raises(L.VbError):
            _ids(lg, 5, 1.0, [1] * 4, [3] * 4, hist=hist if "window" in kw else None, **kw)
    assert len(_ids(lg, 5, 1.0, [1] * 4, [3] * 4, top_p=1.0, window=256, rmax=0, hist=hist)) == 4

    g = load_golden("tiny_batch.pt")
    m = _model(g, torch.float32)
    eng = m.engine()
    texts, prompts = _batch(g)
    bad = [dict(seed=1, top_p=0.0), dict(seed=1, top_p=1.01), dict(seed=1, top_p=[0.5, 0.5]), dict(top_p=-1.0),
           dict(top_p=[0.9] * 4), dict(ras=(8, 0.1)), dict(seed=1, ras=(0, 0.1)), dict(seed=1, ras=(257, 0.1)),
           dict(seed=1, ras=(8.0, 0.1)), dict(seed=1, ras=(8, 1.0)), dict(seed=1, ras=(8, -0.1)),
           dict(seed=1, ras=[(8, 0.1)] * 3), dict(seed=1, ras=(8, 0.1, 2))]
    for kw in bad:
        kw.setdefault("top_k", 5)
        with pytest.raises(ValueError):
            eng.generate(texts, prompts, max_new_tokens=4, **kw)
    eng.sample_on_host = True
    try:
        with pytest.raises(ValueError):
            eng.generate(texts, prompts, top_k=5, max_new_tokens=4, ras=(8, 0.1))
    finally:
        eng.sample_on_host = False
    r = StreamRequest(texts[0], prompts[0], None, None, 1, 1.0, 4, 1.0, (8, 0.1))
    with pytest.raises(ValueError):
        list(eng.generate_stream([r]))
    out = eng.generate(texts, prompts, top_k=5, max_new_tokens=4, seed=1, top_p=0.9, ras=(8, 0.1))
    assert all(o.shape == (4, 8) for o in out)
