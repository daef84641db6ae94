"""Best-of-n decoding on the GPU: vb_ar_state.kv_parent (n candidates of one utterance read one copy of their prompt
prefix from the KV cache), vb_ar_state.logprob (the AR log-likelihood of what the seeded sampler drew) and
ValleEngine.generate(num_samples=, return_scores=).

1. One decode step with kv_parent set gives, bit for bit, the whole state of the same step without it, where every
   sibling holds a real copy of its parent's prefix rows.  In the shared run the siblings' rows below P_b are NaN, so
   any read of them would show.
2. generate(num_samples=n) gives the codes of generate() on the list with every utterance repeated n times.
3. The scores match a float64 restatement of their definition on teacher-forced logits.
4. The argument errors.
"""
import pytest
import torch

import kv_fp8_oracle as K
from test_decode_step_bitwise_gpu import D, EOS, LDL, N_VOCAB, NL, PE_ROWS, _model, _switches
from test_stream_gpu import _model as _engine_model
from test_stream_gpu import _requests, tuned

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
H = 16
CAP = 176
STEPS = 2


# ------------------------------------------------------------------------------------------- 1. decode step
# name: (chain, B, n, greedy, FP8 cache, switches).  The chains are those of tests/test_decode_step_bitwise_gpu.py.
STEP_CASES = {
    "folded_b2_n2_g1": ("folded", 2, 2, 1, False, ()),
    "folded_b17_n4_g2": ("folded", 17, 4, 2, False, ()),
    "folded_b64_n8_g0": ("folded", 64, 8, 0, False, ()),
    "folded_b64_n4_g2_ns1": ("folded", 64, 4, 2, False, (("VB_DECODE_NSPLIT", 1),)),
    "folded_b17_n2_g1_ns3": ("folded", 17, 2, 1, False, (("VB_DECODE_NSPLIT", 3),)),
    "folded_b64_n2_g2_ns7": ("folded", 64, 2, 2, False, (("VB_DECODE_NSPLIT", 7),)),
    "nofold_b17_n8_g0": ("unfolded", 17, 8, 0, False, ()),
    "nofold_b64_n4_g2_ns3": ("unfolded", 64, 4, 2, False, (("VB_DECODE_NSPLIT", 3),)),
    "nofold_b64_n2_g0_ns7": ("unfolded", 64, 2, 0, False, (("VB_DECODE_NSPLIT", 7),)),
    "postln_b17_n4_g1": ("postln", 17, 4, 1, False, ()),
    "postln_b64_n2_g2_ns7": ("postln", 64, 2, 2, False, (("VB_DECODE_NSPLIT", 7),)),
    "fp32_b17_n4_g2": ("fp32", 17, 4, 2, False, ()),
    "fp32_b64_n8_g1_ns3": ("fp32", 64, 8, 1, False, (("VB_DECODE_NSPLIT", 3),)),
    "simt_b17_n4_g1": ("folded", 17, 4, 1, False, (("VB_DECODE_SIMT", 1),)),
    "simt_postln_b2_n2_g2": ("postln", 2, 2, 2, False, (("VB_DECODE_SIMT", 1),)),
}
# the FP8 cache has no shared-prefix step: vb_ar_decode_step refuses kv_parent there
F8_CASES = {
    "f8_folded_b17_n4_g2": ("folded", 17, 4, 2, True, ()),
    "f8_postln_b64_n2_g1": ("postln", 64, 2, 1, True, ()),
}


def _step_inputs(name):
    """host-side inputs of one case: rows grouped in runs of n (the last run may be shorter), parent = first row of
    its run; text + prompt lengths of the forms 16k - 1, 16k, 16k + 1; generated counts that put some contexts on the
    KV split edges; a parent that has finished while its siblings run, and a finished sibling"""
    chain, B, n, greedy, f8, tune = {**STEP_CASES, **F8_CASES}[name]
    g = torch.Generator().manual_seed(sum(map(ord, name)))
    parent = torch.arange(B, dtype=torch.int32) // n * n
    ns = dict(tune).get("VB_DECODE_NSPLIT", 0)
    text, prompt, n_gen = (torch.zeros(B, dtype=torch.int32) for _ in range(3))
    for r in range(B):
        p = int(parent[r])
        if p == r:
            sp = 16 * int(torch.randint(1, 7, (1,), generator=g)) + (r // n) % 3 - 1
            text[r] = int(torch.randint(1, sp, (1,), generator=g))
            prompt[r] = sp - text[r]
        else:
            text[r], prompt[r] = text[p], prompt[p]
        sp = int(text[r] + prompt[r])
        if r % 3 == 0 and ns > 1:          # the context of the coming step ends on a split edge (or one past it)
            kv = max(sp + 1, 16 * ns * int(torch.randint(1, max(2, 170 // (16 * ns) + 1), (1,), generator=g)) + r % 2)
        else:
            kv = sp + int(torch.randint(1, 40, (1,), generator=g))
        n_gen[r] = min(kv, CAP - STEPS - 1) - sp
    fin = torch.zeros(B, dtype=torch.int32)
    if B > n:
        fin[n] = 1                          # the second run's parent has stopped; its siblings run on
        fin[2 * n - 1 if 2 * n - 1 < B else B - 1] = 1
    return chain, B, n, greedy, f8, tune, g, parent, text, prompt, n_gen, fin


def _run_step(name, shared, scores=True):
    from valle_b200 import _lib as L
    import ctypes as C
    lib = L.load()
    chain, B, n, greedy, f8, tune, g, parent, text, prompt, n_gen, fin = _step_inputs(name)
    dtype = torch.float32 if chain == "fp32" else torch.bfloat16
    m = _model(chain in ("folded", "unfolded", "fp32"), dtype)
    nd = m["nd"]
    i32 = dict(dtype=torch.int32, device=DEV)
    kc = torch.randn(NL, B, H, CAP, 64, generator=g).to(DEV, dtype)
    vc = torch.randn(NL, B, H, CAP, 64, generator=g).to(DEV, dtype)
    ke = ve = None
    if f8:
        (kc, ke), (vc, ve) = ((a.to(DEV) for a in K.quantize(c.cpu())) for c in (kc, vc))
    P = [int(text[r] + prompt[r]) // 16 * 16 for r in range(B)]
    arrays = [c.view(torch.uint8) for c in (kc, vc, ke, ve)] if f8 else [kc, vc]   # FP8: e4m3 and exponent bytes
    nan = [0x7F, 0x7F, 0xFF, 0xFF] if f8 else [float("nan")] * 2                     # 0x7f: an e4m3 NaN
    for r in range(B):                     # every sibling holds a copy of its parent's prompt rows ...
        p, sp = int(parent[r]), int(text[r] + prompt[r])
        for c, v in zip(arrays, nan):
            c[:, r, :, :sp] = c[:, p, :, :sp]
            if shared and p != r:          # ... which the shared run must never read below P
                c[:, r, :, :P[r]] = v
    t = dict(text=text.to(**i32), prompt=prompt.to(**i32), n_gen=n_gen.to(**i32), finished=fin.to(**i32),
             max_new=torch.full((B,), 1 << 20, **i32), tokens=torch.full((B, CAP + 8), -5, **i32),
             x=torch.randn(B, D, generator=g).to(DEV), logits=torch.full((B, LDL), 6144.0, device=DEV),
             seed=torch.arange(B, dtype=torch.int64).mul(7919).add(3).to(DEV),
             top_k=torch.randint(1, 60, (B,), generator=g).to(**i32),
             temperature=(0.6 + torch.rand(B, generator=g)).to(DEV), parent=parent.to(**i32),
             logprob=torch.full((B,), 0.25, device=DEV), kc=kc, vc=vc)
    if f8:
        t["ke"], t["ve"] = ke, ve
    pushed = torch.randint(0, N_VOCAB - 1, (STEPS, B), generator=g, dtype=torch.int64).to(DEV)
    s = L.ArState()
    s.B, s.tok_stride = B, CAP + 8
    s.text_len, s.prompt_len, s.max_new = t["text"].data_ptr(), t["prompt"].data_ptr(), t["max_new"].data_ptr()
    s.n_gen, s.finished, s.tokens = t["n_gen"].data_ptr(), t["finished"].data_ptr(), t["tokens"].data_ptr()
    s.x_cur, s.logits = t["x"].data_ptr(), t["logits"].data_ptr()
    s.kcache, s.vcache = kc.data_ptr(), vc.data_ptr()
    s.cache_layer_stride, s.cache_seq_stride, s.cache_cap = kc.stride(0), kc.stride(1), CAP
    if f8:
        s.kv_dtype, s.k_exp, s.v_exp = L.VB_E4M3, ke.data_ptr(), ve.data_ptr()
    s.sample_seed, s.top_k, s.temperature = t["seed"].data_ptr(), t["top_k"].data_ptr(), t["temperature"].data_ptr()
    if shared:
        s.kv_parent = t["parent"].data_ptr()
    if scores:
        s.logprob = t["logprob"].data_ptr()
    h = L.ArHead()
    h.predict_w, h.n_vocab, h.eos_id = m["head_w"].data_ptr(), N_VOCAB, EOS
    h.audio_emb, h.alpha, h.pe, h.pe_rows = m["audio_emb"].data_ptr(), m["alpha"].data_ptr(), m["pe"].data_ptr(), \
        PE_ROWS
    h.greedy = greedy
    if chain == "folded":
        h.fold = m["fold"]
    launches = []
    with _switches(lib, tune):
        nbytes = lib.vb_ar_step_workspace(C.byref(nd.desc), B, CAP)
        ws = torch.zeros(nbytes, dtype=torch.uint8, device=DEV)
        for step in range(STEPS):
            torch.cuda.synchronize()
            n0 = lib.vb_launch_count()
            L.check(lib.vb_ar_decode_step(nd.handle, C.byref(h), C.byref(s), ws.data_ptr(), nbytes, L.stream_ptr()),
                    "vb_ar_decode_step")
            torch.cuda.synchronize()
            launches.append(lib.vb_launch_count() - n0)
            if greedy == 0:
                L.check(lib.vb_ar_push_tokens(C.byref(h), C.byref(s), pushed[step].data_ptr(), D, L.stream_ptr()),
                        "vb_ar_push_tokens")
        torch.cuda.synchronize()
    return t, launches, P, parent


def _bits(x):
    return x.contiguous().view(torch.uint8)


@pytest.mark.parametrize("name", sorted(STEP_CASES))
def test_shared_prefix_step_equals_copied_prefix_step(name):
    want, l_want, _, _ = _run_step(name, shared=False)
    got, l_got, P, parent = _run_step(name, shared=True)
    assert l_got == l_want, "the shared step launches differently"
    for k in ("x", "logits", "tokens", "n_gen", "finished", "logprob"):
        assert torch.equal(_bits(got[k]), _bits(want[k])), f"{name}: {k} differs"
    for k in ("kc", "vc", "ke", "ve"):
        if k not in got:
            continue
        a, b = got[k].clone(), want[k].clone()
        for r in range(len(P)):
            if int(parent[r]) != r:        # the NaN rows below P stay exactly as they were: never written
                sent = a[:, r, :, :P[r]]
                if a.dtype == torch.uint8:
                    assert bool((sent == 0xFF).all()), (k, r)
                else:
                    assert bool(torch.isnan(sent.float()).all()), (k, r)
                a[:, r, :, :P[r]] = 0
                b[:, r, :, :P[r]] = 0
        assert torch.equal(_bits(a), _bits(b)), f"{name}: {k} differs outside the shared rows"
    # no score array: the same state and launches, and logprob untouched
    plain, l_plain, _, _ = _run_step(name, shared=True, scores=False)
    assert l_plain == l_want
    for k in ("x", "logits", "tokens", "n_gen", "finished"):
        assert torch.equal(_bits(plain[k]), _bits(got[k])), f"{name}: {k} depends on the score array"
    assert bool((plain["logprob"] == 0.25).all())
    if STEP_CASES[name][3] != 2:           # only the seeded sampler scores
        assert bool((got["logprob"] == 0.25).all())


@pytest.mark.parametrize("name", sorted(F8_CASES))
def test_fp8_cache_refuses_shared_prefixes(name):
    from valle_b200 import _lib as L
    with pytest.raises(L.VbError, match="FP8"):
        _run_step(name, shared=True)
    _run_step(name, shared=False)          # the same step without kv_parent runs


# ------------------------------------------------------------------------------------------- 2. engine
def _utts(g, B, seed):
    reqs = _requests(g, B, seed=seed)
    return [r.text for r in reqs], [r.prompt for r in reqs], [r.enroll_len for r in reqs]


def _rep(v, n):
    return [x for x in v for _ in range(n)]


# (golden model, engine dtype, FP8 cache)
ENGINE_MODELS = [("tiny_pm1.pt", torch.float32, None), ("tiny_pm1.pt", torch.bfloat16, None),
                 ("tiny_pm1.pt", torch.bfloat16, torch.float8_e4m3fn), ("tiny_postln_pm1.pt", torch.bfloat16, None),
                 ("tiny_postln_pm1.pt", torch.float32, None), ("tiny_bos.pt", torch.bfloat16, None),
                 ("tiny_prenet.pt", torch.float32, None), ("tiny_pm2.pt", torch.bfloat16, torch.float8_e4m3fn)]


@pytest.mark.parametrize("model,dtype,kv", ENGINE_MODELS, ids=lambda v: str(v).replace("torch.", ""))
@pytest.mark.parametrize("n", [2, 4])
def test_best_of_equals_the_repeated_list(model, dtype, kv, n):
    g, m = _engine_model(model, dtype, kv)
    eng = m.engine(dtype)
    B = 5
    texts, prompts, enroll = _utts(g, B, n)
    el = enroll if enroll[0] is not None else None
    mnt = [30 + 7 * b for b in range(B)]
    kw = dict(top_k=[1, 5, 40, 1, 20], temperature=[1.0, 0.8, 1.3, 1.0, 1.1], top_p=[1.0, 0.9, 1.0, 0.7, 1.0],
              ras=[None, (10, 0.2), None, (5, 0.5), None])
    got, sc = eng.generate(texts, prompts, el, max_new_tokens=mnt, seed=77, num_samples=n, return_scores=True, **kw)
    rep = {k: _rep(v, n) for k, v in kw.items()}
    want = eng.generate(_rep(texts, n), _rep(prompts, n), None if el is None else _rep(el, n),
                        max_new_tokens=_rep(mnt, n), seed=77, **rep)
    assert len(got) == B and all(len(c) == n for c in got)
    for b in range(B):
        for j in range(n):
            assert torch.equal(got[b][j], want[b * n + j]), (b, j)
    assert sc.shape == (B, n) and sc.dtype == torch.float32 and bool(torch.isfinite(sc).all())
    # B seeds: candidate j of utterance b draws from seed[b] + j
    seeds = [1000 * b + 3 for b in range(B)]
    got2 = eng.generate(texts, prompts, el, max_new_tokens=mnt, seed=seeds, num_samples=n, **kw)
    want2 = eng.generate(_rep(texts, n), _rep(prompts, n), None if el is None else _rep(el, n),
                         max_new_tokens=_rep(mnt, n), seed=[s + j for s in seeds for j in range(n)], **rep)
    for b in range(B):
        for j in range(n):
            assert torch.equal(got2[b][j], want2[b * n + j]), (b, j)


@pytest.mark.parametrize("kv", [None, torch.float8_e4m3fn], ids=["bf16", "fp8"])
@pytest.mark.parametrize("B,n", [(11, 8), (22, 3)])
def test_best_of_groups_whole_utterances_in_bf16(kv, B, n):
    """B * n > 64 rows: groups of floor(64 / n) utterances, all candidates of each in one group.  11 x 8: groups of
    64 + 24 rows, as the repeated list's; 22 x 3: 63 + 3 rows against the repeated list's 64 + 2, which gives the same
    codes once the KV split count no longer depends on the group's size"""
    g, m = _engine_model("tiny_pm1.pt", torch.bfloat16, kv)
    eng = m.engine(torch.bfloat16)
    with tuned(VB_DECODE_NSPLIT=1):     # one KV split at every batch size: a row's bits do not depend on B
        _check_groups(g, eng, B, n)


def _check_groups(g, eng, B, n):
    texts, prompts, _ = _utts(g, B, 5)
    got, sc = eng.generate(texts, prompts, max_new_tokens=40, top_k=30, temperature=0.9, seed=5, num_samples=n,
                           return_scores=True)
    # the bf16 cache reads the shared prefixes; the FP8 cache runs the repeated list's step
    assert all(bool(b.st.kv_parent) == (b.kv_dtype is None) for b in eng._bufs.values())
    want = eng.generate(_rep(texts, n), _rep(prompts, n), max_new_tokens=40, top_k=30, temperature=0.9, seed=5)
    for b in range(B):
        for j in range(n):
            assert torch.equal(got[b][j], want[b * n + j]), (b, j)
    # scores of the same rows decoded with n = 1 (one candidate per call, its own seed)
    one, sc1 = eng.generate(_rep(texts, n)[:16], _rep(prompts, n)[:16], max_new_tokens=40, top_k=30,
                            temperature=0.9, seed=5, return_scores=True)
    assert sc1.shape == (16, 1)
    assert torch.equal(sc1.view(-1), sc.view(-1)[:16])
    # the solo promise: candidate j of utterance b alone with seed s + b n + j
    for b, j in ((0, 0), (B // 2, n - 1), (B - 1, n // 2)):
        solo = eng.generate([texts[b]], [prompts[b]], max_new_tokens=40, top_k=30, temperature=0.9,
                            seed=5 + b * n + j)[0]
        assert torch.equal(solo, got[b][j]), (b, j)


# ------------------------------------------------------------------------------------------- 3. scores
def _restated(logits, codes):
    """float64 sum of log_softmax(l_i)[t_i] over the steps, and the partial sums"""
    part, s = [], 0.0
    for i, t in enumerate(codes):
        l = logits[i].double()
        s += float(l[t] - torch.logsumexp(l, 0))
        part.append(s)
    return s, part


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["fp32", "bf16"])
@pytest.mark.parametrize("greedy", [False, True], ids=["sampled", "greedy"])
def test_scores_match_the_float64_restatement(dtype, greedy):
    """Each term is l_t - (max + logf(sum expf(l_i - max))) in fp32.  The sum of 1025 terms each within [0, 1] carries
    a relative error of at most 1025 u (u = 2^-24, sequential fp32 sum) plus one ulp each for expf, logf and the two
    additions, so lse is within |lse| 2^-21 + 1025 * 2^-24 * (1 + 2^-21) / z of the exact value, z >= 1, i.e. below
    7e-5 + |lse| 5e-7.  The term adds one rounding of |term| u, and the running sum one of |sum| u per step.  With
    |l| < 60 every term is within 1e-4 + 60 * 6e-7 < 1.4e-4, so after k steps the sum is within
    k (1.4e-4 + |sum| 6e-8).  The logits the restatement reads are the teacher-forced ones of the same codes, which
    are the same fp32 values the decode saw (the engine's forced decode runs the same step kernels)."""
    g, m = _engine_model("tiny_pm1.pt", dtype)
    with tuned(VB_DECODE_NSPLIT=1):     # one KV split at every batch size: the solo logits are the batch's
        _check_scores(g, m.engine(dtype), greedy)


def _check_scores(g, eng, greedy):
    B, n = 3, 2
    texts, prompts, _ = _utts(g, B, 11)
    kw = dict(top_k=1) if greedy else dict(top_k=[40, 10, 200], temperature=[1.2, 0.7, 1.0], top_p=[1.0, 0.8, 1.0])
    codes, sc = eng.generate(texts, prompts, max_new_tokens=25, seed=9, num_samples=n, return_scores=True, **kw)
    for b in range(B):
        for j in range(n):
            c = codes[b][j]
            tr = {"steps": "all"}
            eng.generate([texts[b]], [prompts[b]], max_new_tokens=c.shape[0] + 1, forced=[c], trace=tr)
            lg = tr["ar_logits"]
            assert max(float(lg[i][0].abs().max()) for i in range(c.shape[0])) < 60, "the bar assumes |l| < 60"
            want, part = _restated([lg[i][0].cpu() for i in range(c.shape[0])], c[:, 0].tolist())
            bar = c.shape[0] * (1.4e-4 + abs(want) * 6e-8)
            assert abs(float(sc[b, j]) - want) <= bar, (b, j, float(sc[b, j]), want, bar)
            if greedy:
                assert all(int(c[i, 0]) == int(lg[i][0].argmax()) for i in range(c.shape[0]))
            # the sum of the first k terms: a decode capped after k codes
            k = max(1, c.shape[0] // 2)
            _, sk = eng.generate([texts[b]], [prompts[b]], max_new_tokens=k, seed=9 + b * n + j,
                                 return_scores=True, **({k_: (v[b] if isinstance(v, list) else v)
                                                         for k_, v in kw.items()}))
            assert abs(float(sk[0, 0]) - part[k - 1]) <= k * (1.4e-4 + abs(part[k - 1]) * 6e-8), (b, j, k)


# ------------------------------------------------------------------------------------------- 4. errors
def test_best_of_argument_errors():
    g, m = _engine_model("tiny_pm1.pt", torch.bfloat16)
    eng = m.engine(torch.bfloat16)
    texts, prompts, _ = _utts(g, 2, 1)
    with pytest.raises(ValueError, match="seed"):
        eng.generate(texts, prompts, max_new_tokens=5, num_samples=2)
    with pytest.raises(ValueError, match="seed"):
        eng.generate(texts, prompts, max_new_tokens=5, return_scores=True)
    for bad in (0, -1, 2.0, "2", True):
        with pytest.raises(ValueError, match="num_samples"):
            eng.generate(texts, prompts, max_new_tokens=5, seed=1, num_samples=bad)
    with pytest.raises(ValueError, match="at most 64"):
        eng.generate(texts, prompts, max_new_tokens=5, seed=1, num_samples=65)
    with pytest.raises(ValueError, match="test hooks"):
        eng.generate(texts, prompts, max_new_tokens=5, seed=1, num_samples=2, trace={"steps": {0}})
    with pytest.raises(ValueError, match="test hooks"):
        eng.generate(texts, prompts, max_new_tokens=5, seed=1, num_samples=2, forced=[p[:3] for p in prompts])
    eng.sample_on_host = True
    try:
        with pytest.raises(ValueError, match="sample_on_host"):
            eng.generate(texts, prompts, max_new_tokens=5, seed=1, num_samples=2)
    finally:
        eng.sample_on_host = False
    # n = 1 is today's call
    a = eng.generate(texts, prompts, max_new_tokens=8, seed=3, top_k=20, num_samples=1)
    b = eng.generate(texts, prompts, max_new_tokens=8, seed=3, top_k=20)
    assert all(torch.equal(x, y) for x, y in zip(a, b))
