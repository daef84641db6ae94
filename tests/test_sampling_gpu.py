"""GPU tests of the seeded device sampler (vb_sample_logits, vb_ar_head.greedy == 2, ValleEngine.generate(seed=)).

The sampler's contract (include/valle_b200.h vb_sample_logits) is restated here in numpy: l' = l / T, the exact top-k
set (ties with the k-th value kept), u = ((h >> 41) + 0.5) 2^-23 from the splitmix64 hash of (seed, step, id),
Gumbel-max over the kept set.  The device's logf and numpy's log may differ in the last bit, so a restated id may
differ from the device's only where the two best perturbed scores are within 1e-6 of each other."""
import math

import numpy as np
import pytest
import torch

from conftest import assert_checksums, build_model, load_golden
from oracle import valle_oracle as O

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
EOS = 1024
V = 1025
NEAR_TIE = 1e-6


def _model(g, dtype):
    m = build_model(g["config"], g["weight_seed"])
    assert_checksums(m, g["checksums"])
    m = m.to(DEV)
    m.engine_dtype = dtype
    m.engine().quiet = True
    return m


def _batch(g):
    return [u["x"][0] for u in g["utts"]], [u["y"][0] for u in g["utts"]]


# ------------------------------------------------------------------------------------------- numpy restatement
def _mix64(seed, stream, idx):
    with np.errstate(over="ignore"):
        z = np.uint64(seed) + np.uint64(stream) * np.uint64(0x9E3779B97F4A7C15) + \
            idx.astype(np.uint64) * np.uint64(0xD1342543DE82EF95)
        z ^= z >> np.uint64(30)
        z *= np.uint64(0xBF58476D1CE4E5B9)
        z ^= z >> np.uint64(27)
        z *= np.uint64(0x94D049BB133111EB)
        z ^= z >> np.uint64(31)
    return z


def _scores(l, seed, step, k, T):
    """perturbed scores of one row (float32, -inf outside the top-k set)"""
    l = np.asarray(l, dtype=np.float32)
    n = l.size
    x = l if T == 1.0 else (l / np.float32(T)).astype(np.float32)
    keep = np.ones(n, dtype=bool)
    if 0 < k < n:
        kth = np.partition(x, n - k)[n - k]
        keep = x >= kth
    h = _mix64(seed, step, np.arange(n))
    u = ((h >> np.uint64(41)).astype(np.float32) + np.float32(0.5)) * np.float32(2.0 ** -23)
    g = -np.log(-np.log(u))
    assert bool(((u > 0) & (u < 1)).all()) and bool(np.isfinite(g).all())
    return np.where(keep, x + g, np.float32(-np.inf)).astype(np.float32)


def _draw(l, seed, step, k, T):
    if k == 1:
        return int(np.argmax(np.asarray(l, dtype=np.float32)))
    return int(np.argmax(_scores(l, seed, step, k, T)))


def _agrees(dev_id, l, seed, step, k, T):
    """(exact, allowed): the device id equals the restated one, or it is a near-tie of the best perturbed score"""
    ref = _draw(l, seed, step, k, T)
    if dev_id == ref:
        return True, True
    if k == 1:
        return False, False
    sc = _scores(l, seed, step, k, T)
    return False, bool(sc[dev_id] >= sc[ref] - NEAR_TIE * max(1.0, abs(float(sc[ref]))))


# ------------------------------------------------------------------------------------------- 1. distribution
CASES = [(-100, 1.0), (5, 1.0), (5, 0.7), (50, 1.3), (1025, 1.0), (2000, 1.0), (1, 1.0)]


def _rows():
    g = torch.Generator().manual_seed(5)
    rows = [torch.randn(V, generator=g) * 1.5 for _ in range(3)]
    tie = torch.randn(V, generator=g)
    kth = tie.topk(5)[0][-1]
    tie[[17, 600]] = kth                                   # two extra tokens tied with the 5th largest value
    dom = torch.randn(V, generator=g)
    dom[321] = 12.0                                        # one token holds almost all the mass
    return torch.stack(rows + [tie, dom]), [17, 600]


@pytest.mark.parametrize("k,T", CASES)
def test_sample_logits_draws_from_the_filtered_softmax(k, T):
    from scipy.stats import chisquare
    from valle_b200 import ops
    rows, tied = _rows()
    N = 1 << 18
    idx = torch.arange(N, device=DEV)
    seeds, steps = (idx // 64) * 7919 + 3, (idx % 64).to(torch.int32)
    for r in range(rows.shape[0]):
        l = rows[r]
        ids = ops.sample_logits(l.to(DEV)[None].expand(N, V), k, T, seeds, steps).cpu()
        assert int(ids.min()) >= 0 and int(ids.max()) < V
        if k == 1:
            assert bool((ids == int(l.argmax())).all()), r
            continue
        lt = l if T == 1.0 else l / T
        filt = O.top_k_top_p_filtering(lt[None].clone(), top_k=k)[0]
        kept = torch.isfinite(filt)
        assert bool(kept[ids].all()), f"row {r}: a draw outside the top-{k} set"
        counts = np.bincount(ids.numpy(), minlength=V).astype(np.float64)
        if r == 3 and 1 < k < 7:
            assert all(counts[t] > 0 for t in tied), "tokens tied with the k-th value are never drawn"
        p = torch.softmax(filt.double(), 0).numpy()
        exp = p * N
        big = exp >= 5
        obs = np.append(counts[big], counts[~big].sum())
        ex = np.append(exp[big], exp[~big].sum())
        if ex[-1] == 0:
            obs, ex = obs[:-1], ex[:-1]
        if ex.size < 2:
            continue
        pv = chisquare(obs, ex * obs.sum() / ex.sum()).pvalue
        assert pv > 1e-4, (r, k, T, pv)


# ------------------------------------------------------------------------------------------- 2. exact restatement
def test_sample_logits_matches_the_numpy_restatement():
    from valle_b200 import ops
    g = torch.Generator().manual_seed(9)
    R = 512
    lg = torch.randn(R, V, generator=g) * 2
    lg[::7, 40] = lg[::7].max(dim=1).values               # exact ties with the row maximum
    ks = torch.tensor([(-100, 1, 2, 5, 50, 1024, 1025, 0)[i % 8] for i in range(R)], dtype=torch.int32)
    ts = torch.tensor([(1.0, 0.7, 1.3, 0.25)[i % 4] for i in range(R)], dtype=torch.float32)
    seeds = [(i * 0x9E3779B97F4A7C15 + 5) % (1 << 64) for i in range(R)]     # includes seeds >= 2**63
    steps = torch.randint(0, 3000, (R,), generator=g, dtype=torch.int32)
    ids = ops.sample_logits(lg.to(DEV), ks, ts, seeds, steps).cpu().tolist()
    near = 0
    for r in range(R):
        exact, ok = _agrees(ids[r], lg[r].numpy(), seeds[r], int(steps[r]), int(ks[r]), float(ts[r]))
        assert ok, (r, ids[r], _draw(lg[r].numpy(), seeds[r], int(steps[r]), int(ks[r]), float(ts[r])))
        near += not exact
    print(f"sample_logits: {near} of {R} draws differ from numpy at a near-tie")
    assert near <= R // 100


def test_the_largest_hash_value_does_not_win_over_the_logits():
    """(seed 2024, step 12495947, id 7) hashes to h >> 40 == 2^24 - 1, the top of the uniform's range.  The draw must
    stay finite there: a token 60 below every other logit is never drawn.  (A 24-bit u = ((h >> 40) + 0.5) 2^-24 rounds
    to 1.0 in fp32 at this hash, giving g = +inf, so that token would win whatever its logit.)"""
    from valle_b200 import ops
    seed, step, tok = 2024, 12495947, 7
    assert int(_mix64(seed, step, np.array([tok]))[0]) >> 40 == (1 << 24) - 1
    l = torch.zeros(V)
    l[tok] = -60.0
    for k in (-100, 1025, 50):
        ids = ops.sample_logits(l.to(DEV)[None], k, 1.0, [seed], [step]).cpu()
        assert int(ids[0]) != tok, k
        assert int(ids[0]) == _draw(l.numpy(), seed, step, k, 1.0)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("k,T", [(-100, 1.0), (20, 0.8)])
def test_traced_native_decode_matches_the_restatement(dtype, k, T):
    """Every id of a native sampled decode is the restated draw from that step's traced logits with (seed, step), and
    the decode ends at the first step where the stop rule (argmax == EOS, draw == EOS, or the cap) fires."""
    g = load_golden("tiny_pm1.pt")
    m = _model(g, dtype)
    eng = m.engine()
    x, y = g["x"][0], g["y"][0]
    seed = 987654321
    tr = {"steps": "all"}
    out = eng.generate([x], [y], top_k=k, temperature=T, trace=tr, seed=seed)[0].cpu()
    n = out.shape[0]
    cap = 16 * x.numel() - int(eng.prepend_bos)
    near = 0
    for j in range(n + 1):
        l = tr["ar_logits"][j][0].cpu().numpy()
        amax = int(np.argmax(l))
        if j < n:
            exact, ok = _agrees(int(out[j, 0]), l, seed, j, k, T)
            assert ok, (j, int(out[j, 0]), _draw(l, seed, j, k, T))
            near += not exact
            assert amax != EOS and int(out[j, 0]) != EOS
        else:
            d = _draw(l, seed, j, k, T)
            assert amax == EOS or d == EOS or j > cap, (j, amax, d)
    print(f"{dtype} top_k={k} T={T}: {n} frames, {near} near-tie mismatches")
    assert near <= max(1, n // 50)


# ------------------------------------------------------------------------------------------- 3. invariance
def test_seeded_codes_are_invariant_to_graphs_polling_and_reruns():
    g = load_golden("tiny_batch.pt")
    m = _model(g, torch.bfloat16)
    eng = m.engine()
    texts, prompts = _batch(g)
    kw = dict(top_k=-100, seed=77)
    ref = eng.generate(texts, prompts, **kw)
    assert all(torch.equal(a, b) for a, b in zip(ref, eng.generate(texts, prompts, **kw)))
    assert all(torch.equal(a, b) for a, b in zip(ref, eng.generate(texts, prompts, poll=1, **kw)))
    eng.steps_per_graph = 1
    try:
        assert all(torch.equal(a, b) for a, b in zip(ref, eng.generate(texts, prompts, **kw)))
    finally:
        eng.steps_per_graph = 8
    eng.use_cuda_graph = False
    try:
        assert all(torch.equal(a, b) for a, b in zip(ref, eng.generate(texts, prompts, **kw)))
    finally:
        eng.use_cuda_graph = True
    # the torch default path is unaffected by the seed of an earlier call and still draws
    assert len(eng.generate(texts, prompts, top_k=-100, max_new_tokens=4)) == len(texts)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_batch_equals_each_utterance_alone(dtype):
    g = load_golden("tiny_batch.pt")
    m = _model(g, dtype)
    eng = m.engine()
    texts, prompts = _batch(g)
    s = 1 << 40
    outs = eng.generate(texts, prompts, top_k=50, temperature=0.9, seed=s)
    for b in range(len(texts)):
        eng._bufs.clear()
        solo = eng.generate([texts[b]], [prompts[b]], top_k=50, temperature=0.9, seed=s + b)[0]
        assert torch.equal(solo, outs[b]), b
    # VALLE.inference / inference_batch pass the seed through
    x, y = texts[1], prompts[1]
    one = m.inference(x[None].to(DEV), torch.tensor([x.numel()], dtype=torch.int32), y[None].to(DEV), None,
                      top_k=50, temperature=0.9, seed=s + 1)[0].cpu()
    assert torch.equal(one, outs[1])
    again = m.inference_batch(texts, prompts, top_k=50, temperature=0.9, seed=s)
    assert all(torch.equal(a, b) for a, b in zip(again, outs))


def test_bf16_groups_above_64_keep_their_absolute_seeds():
    g = load_golden("tiny_batch.pt")
    m = _model(g, torch.bfloat16)
    eng = m.engine()
    t4, p4 = _batch(g)
    texts, prompts = (t4 * 18)[:70], (p4 * 18)[:70]
    ks = [(-100, 5, 50, 1)[i % 4] for i in range(70)]
    out = eng.generate(texts, prompts, top_k=ks, max_new_tokens=12, seed=500)
    a = eng.generate(texts[:64], prompts[:64], top_k=ks[:64], max_new_tokens=12, seed=500)
    b = eng.generate(texts[64:], prompts[64:], top_k=ks[64:], max_new_tokens=12, seed=564)
    assert len(out) == 70
    for i, (o, r) in enumerate(zip(out, a + b)):
        assert torch.equal(o, r), i


# ------------------------------------------------------------------------------------------- 4. per-utterance parameters
def test_mixed_parameters_equal_solo_decodes():
    g = load_golden("tiny_batch.pt")
    m = _model(g, torch.float32)
    eng = m.engine()
    texts, prompts = _batch(g)
    ks, ts = [1, 5, -100, 50], [1.0, 0.7, 1.0, 1.3]
    outs = eng.generate(texts, prompts, top_k=ks, temperature=ts, seed=[11, 12, 13, 2 ** 64 - 1])
    for b, s in enumerate([11, 12, 13, 2 ** 64 - 1]):
        solo = eng.generate([texts[b]], [prompts[b]], top_k=ks[b], temperature=ts[b], seed=s)[0]
        assert torch.equal(solo, outs[b]), b
    greedy = eng.generate([texts[0]], [prompts[0]], top_k=1)[0]
    assert torch.equal(greedy, outs[0])
    assert torch.equal(greedy, g["utts"][0]["codes"][0].long())


# ------------------------------------------------------------------------------------------- 5. graphs, no push
class _Spy:
    def __init__(self, lib):
        self._lib, self.pushes = lib, 0

    def __getattr__(self, name):
        f = getattr(self._lib, name)
        if name != "vb_ar_push_tokens":
            return f

        def push(*a):
            self.pushes += 1
            return f(*a)
        return push


def test_native_sampling_runs_in_graphs_without_host_draws():
    g = load_golden("tiny_batch.pt")
    m = _model(g, torch.bfloat16)
    eng = m.engine()
    texts, prompts = _batch(g)

    def per_step(**kw):
        res = []
        for mnt in (4, 20):
            n0, r0 = eng.kernel_launches(), eng.replayed_launches
            eng.generate(texts, prompts, max_new_tokens=mnt, **kw)
            res.append((eng.kernel_launches() - n0, eng.stats.ar_steps, eng.replayed_launches - r0))
        (l1, s1, _), (l2, s2, rep) = res
        assert s2 > s1
        return (l2 - l1) / (s2 - s1), rep

    per_step(top_k=1)                                   # captures the greedy graphs
    per_step(top_k=-100, seed=3)                        # captures the sampled graphs
    greedy, _ = per_step(top_k=1)
    spy = _Spy(eng.lib)
    eng.lib = spy
    try:
        native, replayed = per_step(top_k=-100, seed=3)
        assert spy.pushes == 0
        eng.generate(texts, prompts, top_k=-100, max_new_tokens=4)   # the torch path still pushes its draws
        assert spy.pushes > 0
    finally:
        eng.lib = spy._lib
    assert replayed > 0
    assert greedy <= native <= greedy + 2, (greedy, native)


# ------------------------------------------------------------------------------------------- 6. validation
def test_bad_sampler_arguments_raise_value_error():
    g = load_golden("tiny_batch.pt")
    m = _model(g, torch.float32)
    eng = m.engine()
    texts, prompts = _batch(g)
    bad = [dict(seed=[1, 2, 3]), dict(seed=-1), dict(seed=2 ** 64), dict(seed=[0, 1, 2, 2 ** 64]),
           dict(seed=1, top_k=[5, 5]), dict(seed=1, temperature=0.0), dict(seed=1, temperature=-1.0),
           dict(seed=1, temperature=math.nan), dict(seed=1, temperature=math.inf),
           dict(seed=1, temperature=[1.0, 1.0, 1.0, 0.0]), dict(top_k=[5, 5, 5, 5])]
    for kw in bad:
        kw.setdefault("top_k", 5)
        with pytest.raises(ValueError):
            eng.generate(texts, prompts, max_new_tokens=4, **kw)
    eng.sample_on_host = True
    try:
        with pytest.raises(ValueError):
            eng.generate(texts, prompts, top_k=5, max_new_tokens=4, seed=1)
    finally:
        eng.sample_on_host = False
    out = eng.generate(texts, prompts, top_k=5, max_new_tokens=4, seed=1)   # still usable
    assert all(o.shape == (4, 8) for o in out)
