"""The opt-in FP8 (e4m3) KV cache of bf16 AR decoding (`VALLE.kv_cache_dtype = torch.float8_e4m3fn`, include/valle_b200.h
"FP8 (e4m3) KV cache", vb_ar_state.kv_dtype), on the GPU.

  * prefill: the FP8 cache the prefill writes is, byte for byte and exponent for exponent, tests/kv_fp8_oracle.py applied
    to the bf16 cache the bf16 prefill writes; rows outside the sequences keep their sentinel;
  * decode step: with the cache quantized, each bf16 chain (folded, unfolded, post-LN) is the bf16 step run on the
    dequantized cache -- the current token attends as its unquantized bf16 row -- so the float64 restatement of
    tests/decode_step_oracle.py fed the dequantized cache checks it at the error-model bars of
    tests/test_decode_step_gpu.py; layer 0's appended row is the restatement of the bf16-cache run's row, bit for bit;
  * the decode invariances of the bf16 cache: reruns, poll, graphs, batch == solo, B > 64 groups, prepend_bos,
    add_prenet, post-LN, VB_DECODE_FOLD=0;
  * a bounded end-to-end deviation of the teacher-forced logits on big_short;
  * the errors and the buffer sizes."""
import ctypes as C
import math
import os

import pytest
import torch

from conftest import build_model, load_golden

import decode_step_oracle as D
import kv_fp8_oracle as K
import test_decode_step_gpu as T

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
F8 = torch.float8_e4m3fn
_c, OFF, NS, Q = T._c, T.OFF, T.NS, T.Q


# ---- decode step against the restatement ------------------------------------------------------------------------
CASES = [
    _c("f8_big_folded_b64", "big", "bf16_folded", 64, 1088, offsets=OFF),
    _c("f8_big_folded_b1_cap", "big", "bf16_folded", 1, 4160, lens=[4169], content="peak_last"),
    _c("f8_big_folded_b17_ns3", "big", "bf16_folded", 17, 304, finished=[3], tune=[(NS, 3)]),
    _c("f8_tiny_folded_b64_ns7", "tiny", "bf16_folded", 64, 512, offsets=OFF, content="peak_boundary", tune=[(NS, 7)]),
    _c("f8_big_unfolded_b17_qkv1", "big", "bf16_unfolded", 17, 208, finished=[1], tune=[(NS, 2), (Q, 1)]),
    _c("f8_tiny_unfolded_b64", "tiny", "bf16_unfolded", 64, 160, content="peak_current", tune=[(NS, 1), (Q, 4)]),
    _c("f8_tiny_unfolded_b1_qkv1", "tiny", "bf16_unfolded", 1, 3008, lens=[1501], tune=[(NS, 32), (Q, 1)]),
    _c("f8_big_postln_b17", "big", "bf16_postln", 17, 304, content="peak_first"),
    _c("f8_tiny_postln_b64_qkv1", "tiny", "bf16_postln", 64, 160, content="flat", tune=[(NS, 3), (Q, 1), T.NO_PDL]),
    _c("f8_tiny_postln_b1", "tiny", "bf16_postln", 1, 4160, lens=[4160], content="peak_current"),
]


def _run8(lib, case, m, st, kq, ke, vq, ve):
    """one vb_ar_decode_step on an FP8 cache (kq / vq float8 [L, B, H, cap, 64], ke / ve uint8 [L, B, H, cap])"""
    from valle_b200 import _lib as L
    B, cap = case.B, case.cap
    i32 = dict(dtype=torch.int32, device=DEV)
    t = dict(text=st["text"].to(**i32), prompt=st["prompt"].to(**i32), n_gen=st["n_gen"].to(**i32),
             finished=st["finished"].to(**i32), max_new=torch.full((B,), 1 << 20, **i32),
             tokens=torch.full((B, cap + 32), -5, **i32), x=st["x"].to(DEV),
             logits=torch.full((B, T.LDL), T.SENTINEL, device=DEV),
             kc=kq.to(DEV), vc=vq.to(DEV), ke=ke.to(DEV), ve=ve.to(DEV))
    s = L.ArState()
    s.B, s.tok_stride = B, cap + 32
    s.text_len, s.prompt_len, s.max_new = t["text"].data_ptr(), t["prompt"].data_ptr(), t["max_new"].data_ptr()
    s.n_gen, s.finished, s.tokens = t["n_gen"].data_ptr(), t["finished"].data_ptr(), t["tokens"].data_ptr()
    s.x_cur, s.logits = t["x"].data_ptr(), t["logits"].data_ptr()
    s.kcache, s.vcache = t["kc"].data_ptr(), t["vc"].data_ptr()
    s.cache_layer_stride, s.cache_seq_stride, s.cache_cap = t["kc"].stride(0), t["kc"].stride(1), cap
    s.kv_dtype, s.k_exp, s.v_exp = L.VB_E4M3, t["ke"].data_ptr(), t["ve"].data_ptr()
    h = L.ArHead()
    h.predict_w, h.n_vocab, h.eos_id = m["head_dev"].data_ptr(), T.N_VOCAB, T.EOS
    h.audio_emb, h.alpha, h.pe, h.pe_rows = m["audio_emb"].data_ptr(), m["alpha"].data_ptr(), m["pe"].data_ptr(), \
        m["pe_rows"]
    h.greedy = 0
    if m["fold"] is not None and case.chain == "bf16_folded":
        h.fold = m["fold"]
    nd = m["nd"]
    with T._knobs(lib, case):
        nbytes = lib.vb_ar_step_workspace(C.byref(nd.desc), B, cap)
        ws = torch.zeros(nbytes, dtype=torch.uint8, device=DEV)
        L.check(lib.vb_ar_decode_step(nd.handle, C.byref(h), C.byref(s), ws.data_ptr(), nbytes, L.stream_ptr()),
                "vb_ar_decode_step")
        torch.cuda.synchronize()
    return {k: v.cpu() for k, v in t.items()}


@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_fp8_decode_step_is_the_bf16_step_on_the_dequantized_cache(lib, case):
    m = T._model_for(case)
    st = T._state(case, m)                   # bf16 caches with sentinels past every row's current token
    kq, ke = K.quantize(st["kc"])
    vq, ve = K.quantize(st["vc"])
    st8 = dict(st, kc=K.dequantize(kq, ke), vc=K.dequantize(vq, ve))
    same = T._ref(case, m, st8)
    exact = T._ref(case, m, st8, rounding=False)
    bars = T._bars(case, st8, same, exact)
    run = _run8(lib, case, m, st, kq, ke, vq, ve)
    live = (st["finished"] == 0).nonzero().flatten()
    kv_len = same.kv_len
    for name, got in (("x", run["x"]), ("logits", run["logits"][:, :T.N_VOCAB])):
        bs, be = bars[name]
        es = T._row_err(got, getattr(same, name))[live]
        ee = T._row_err(got, getattr(exact, name))[live]
        rs, re_ = float((es / bs[live]).max()), float((ee / be[live]).max())
        print(f"{case.name} {name}: {rs:.3f} x the same-chain bar, {re_:.3f} x the rounding bar")
        assert rs <= 1.0, f"{name}: error {float(es.max()):.3g} vs the restatement, {rs:.2f} x its bar"
        assert re_ <= 1.0, f"{name}: error {float(ee.max()):.3g} vs the unrounded step, {re_:.2f} x its bar"
    assert torch.equal(run["logits"][:, T.N_VOCAB:], torch.full((case.B, T.LDL - T.N_VOCAB), T.SENTINEL))
    # layer 0's appended rows: the quantized row of the bf16-cache run (same inputs: x and the weights only)
    bf = T._run(lib, case, m, st, greedy=0)
    pos = kv_len - 1
    for key, q8, e8 in (("kc", "kc", "ke"), ("vc", "vc", "ve")):
        for b in live.tolist():
            want_q, want_e = K.quantize(bf[key][0, b, :, int(pos[b])].float())
            assert torch.equal(run[q8][0, b, :, int(pos[b])].view(torch.uint8), want_q.view(torch.uint8)), (key, b)
            assert torch.equal(run[e8][0, b, :, int(pos[b])], want_e), (key, b)
    # layer 1's appended rows: the restatement's row within its bar plus half an e4m3 step
    for name, q8, e8 in (("k_new", "kc", "ke"), ("v_new", "vc", "ve")):
        got = torch.stack([K.dequantize(run[q8][1, b, :, int(pos[b])], run[e8][1, b, :, int(pos[b])])
                           for b in range(case.B)]).double()                              # [B, H, 64]
        want = getattr(same, name)[1]
        tol = T._ulp_bf16(want) + bars[name][0][1][..., None] + 2.0 ** -4 * want.abs().amax(-1, keepdim=True)
        assert not bool(((got - want).abs() > tol)[live].any()), f"layer 1 {name}"
    # nothing else in the caches or the exponent arrays changed
    for q8, e8, src_q, src_e in (("kc", "ke", kq, ke), ("vc", "ve", vq, ve)):
        a, b_ = run[q8].view(torch.uint8).clone(), src_q.view(torch.uint8).clone()
        ea, eb = run[e8].clone(), src_e.clone()
        a[:, live, :, pos[live]] = 0
        b_[:, live, :, pos[live]] = 0
        ea[:, live, :, pos[live]] = 0
        eb[:, live, :, pos[live]] = 0
        assert torch.equal(a, b_) and torch.equal(ea, eb), f"{q8}: a cache row other than the appended one changed"
    again = _run8(lib, case, m, st, kq, ke, vq, ve)
    for k in ("x", "logits", "ke", "ve"):
        assert torch.equal(run[k], again[k]), f"{k}: a second run differs"
    for k in ("kc", "vc"):
        assert torch.equal(run[k].view(torch.uint8), again[k].view(torch.uint8))


# ---- prefill ---------------------------------------------------------------------------------------------------------
def _big_model():
    import bench
    m = bench.build_model(torch.device(DEV))
    m.engine_dtype = torch.bfloat16
    m.engine().quiet = True
    return m


_BIG = {}


def _big():
    if "m" not in _BIG:
        _BIG["m"] = _big_model()
    return _BIG["m"]


def test_prefill_writes_the_quantized_bf16_cache(lib):
    from valle_b200 import _lib as L
    m = _big()
    nd = m.engine().ar
    g = torch.Generator().manual_seed(5)
    S, Tp = [7, 40, 3], [90, 130, 1]
    lens = [s + t for s, t in zip(S, Tp)]
    B, cap, d = len(S), 256, nd.desc.d_model
    cu = torch.tensor([0] + list(torch.tensor(lens).cumsum(0)), dtype=torch.int32, device=DEV)
    S_d = torch.tensor(S, dtype=torch.int32, device=DEV)
    x0 = torch.randn(sum(lens), d, generator=g).to(DEV)
    shape = (nd.n_layer, B, nd.H, cap, 64)
    k16 = torch.full(shape, T.SENTINEL, dtype=torch.bfloat16, device=DEV)
    v16 = torch.full(shape, -T.SENTINEL, dtype=torch.bfloat16, device=DEV)
    nd.forward(x0.clone(), cu, B, max(lens), L.VB_MASK_VALLE_AR, S_d, None, k16, v16, cap)
    sq, se = K.quantize(torch.full((64,), T.SENTINEL))
    k8 = torch.full(shape, float(sq[0].float()), device=DEV).to(F8)
    v8 = torch.full(shape, -float(sq[0].float()), device=DEV).to(F8)
    ke = torch.full(shape[:-1], int(se), dtype=torch.uint8, device=DEV)
    ve = ke.clone()
    x8 = x0.clone()
    nd.forward(x8, cu, B, max(lens), L.VB_MASK_VALLE_AR, S_d, None, k8, v8, cap, k_exp=ke, v_exp=ve)
    torch.cuda.synchronize()
    x16 = x0.clone()
    nd.forward(x16, cu, B, max(lens), L.VB_MASK_VALLE_AR, S_d, None, torch.empty_like(k16), torch.empty_like(v16), cap)
    assert torch.equal(x8, x16), "the FP8 cache changed the prefill's arithmetic"
    for c16, c8, e8 in ((k16, k8, ke), (v16, v8, ve)):
        wq, we = K.quantize(c16.float().cpu())
        assert torch.equal(c8.cpu().view(torch.uint8), wq.view(torch.uint8))
        assert torch.equal(e8.cpu(), we)
    for b, n in enumerate(lens):    # the sentinel rows past every sequence survive (above: quantize(+-sentinel))
        assert bool((k8[:, b, :, n:].float() == float(sq[0].float())).all()) and bool((ke[:, b, :, n:] == int(se)).all())
        assert bool((v8[:, b, :, n:].float() == -float(sq[0].float())).all()) and bool((ve[:, b, :, n:] == int(se)).all())


# ---- invariances -------------------------------------------------------------------------------------------------
def _utts(n, seed=3, S=(5, 12), Tp=(8, 30)):
    g = torch.Generator().manual_seed(seed)
    out = []
    for _ in range(n):
        s = int(torch.randint(S[0], S[1], (), generator=g))
        t = int(torch.randint(Tp[0], Tp[1], (), generator=g))
        out.append((torch.randint(3, 100, (s,), generator=g), torch.randint(0, 1024, (t, 8), generator=g)))
    return out


def _tiny(name="tiny_pm1.pt"):
    g = load_golden(name)
    m = build_model(g["config"], g["weight_seed"])
    if g.get("buffers"):
        m.load_state_dict(g["buffers"], strict=False)
    m = m.to(DEV)
    m.engine_dtype = torch.bfloat16
    m.kv_cache_dtype = F8
    m.engine().quiet = True
    return m


def _gen(m, utts, **kw):
    kw.setdefault("max_new_tokens", 24)
    return m.engine().generate([u[0] for u in utts], [u[1] for u in utts], top_k=kw.pop("top_k", 1), **kw)


def test_reruns_poll_and_graphs_give_the_same_codes():
    m = _tiny()
    utts = _utts(5)
    ref = _gen(m, utts)
    eng = m.engine()
    for variant in ("rerun", "poll", "spg1", "nograph"):
        if variant == "poll":
            got = _gen(m, utts, poll=1)
        elif variant == "spg1":
            eng.steps_per_graph = 1
            got = _gen(m, utts)
            eng.steps_per_graph = 8
        elif variant == "nograph":
            eng.use_cuda_graph = False
            got = _gen(m, utts)
            eng.use_cuda_graph = True
        else:
            got = _gen(m, utts)
        assert all(torch.equal(a, b) for a, b in zip(got, ref)), variant


def test_batch_equals_solo_greedy_and_seeded():
    m = _tiny()
    utts = _utts(6, seed=7)
    texts, prompts = [u[0] for u in utts], [u[1] for u in utts]
    batch = m.inference_batch(texts, prompts, top_k=1, max_new_tokens=24)
    for b, (t, p) in enumerate(utts):
        solo = m.inference(t[None].to(DEV), torch.tensor([t.numel()], dtype=torch.int32), p[None].to(DEV), None,
                           top_k=1, max_new_tokens=24)[0].cpu()
        assert torch.equal(batch[b], solo), b
    ks, ts = [1, 5, 40, 3, 0, 12], [1.0, 0.7, 1.3, 1.0, 0.9, 2.0]
    batch = m.inference_batch(texts, prompts, top_k=ks, temperature=ts, max_new_tokens=24, seed=100)
    for b, (t, p) in enumerate(utts):
        solo = m.inference_batch([t], [p], top_k=ks[b], temperature=ts[b], max_new_tokens=24, seed=100 + b)[0]
        assert torch.equal(batch[b], solo), b


def test_b70_equals_its_two_groups():
    m = _tiny()
    utts = _utts(70, seed=9)
    whole = _gen(m, utts, max_new_tokens=10)
    first, second = _gen(m, utts[:64], max_new_tokens=10), _gen(m, utts[64:], max_new_tokens=10)
    assert all(torch.equal(a, b) for a, b in zip(whole, first + second))


@pytest.mark.parametrize("name", ["tiny_bos.pt", "tiny_prenet.pt", "tiny_postln_pm1.pt", "unfolded"])
def test_model_variants_run_and_keep_batch_equal_solo(name):
    if name == "tiny_postln_pm1.pt":
        from test_post_ln import postln_model
        g = load_golden(name)
        m = postln_model(g["config"], g["weight_seed"]).to(DEV)
        m.engine_dtype, m.kv_cache_dtype = torch.bfloat16, F8
        m.engine().quiet = True
    elif name == "unfolded":
        os.environ["VB_DECODE_FOLD"] = "0"
        try:
            m = _tiny()
            assert m.engine().ar_head_fold is None
        finally:
            del os.environ["VB_DECODE_FOLD"]
    else:
        m = _tiny(name)
    utts = _utts(4, seed=11)
    batch = _gen(m, utts, max_new_tokens=16)
    assert all(o.shape[1] == 8 and o.shape[0] >= 1 for o in batch)
    for b, u in enumerate(utts):
        assert torch.equal(batch[b], _gen(m, [u], max_new_tokens=16)[0]), (name, b)


# ---- bounded end-to-end deviation ------------------------------------------------------------------------------------
def test_teacher_forced_logits_stay_within_the_e4m3_bar_big_short():
    """big_short (d=1024/16h/12L, 97 frames), teacher-forced with the reference's ids, FP8 cache against the bf16 cache.

    Bar.  Every cached K / V element carries a relative error of at most 2^-4 (half an e4m3 step: 3 mantissa bits),
    the same form as the 2^-9 of a bf16 rounding in DESIGN section 2, 2^5 = 32 times larger.  Carried through a step as
    DESIGN section 2 carries the bf16 roundings -- independent per element, adding up as a random walk over the
    rounding points of a row's path -- two of the step's roundings (the cached K and V) grow by that factor.  The
    bf16 bar of an AR step against the fp32 reference is AR_TOL = 0.03 (tests/test_parity_bf16_gpu.py) for 22 bf16
    roundings; with 2 of them 32 times larger the walk grows by sqrt(20 + 2 * 32^2) / sqrt(22) = 9.7, so the bar on the
    FP8-versus-bf16 logits is 10 * AR_TOL = 0.3 per logit.  The observed figures are printed, not used as the bar.
    Being a worst-case walk over a whole decode, the bar sits far above the measured deviation (about 40 x on an H100)
    and guards against gross errors only; the per-step precision is checked by
    test_fp8_decode_step_is_the_bf16_step_on_the_dequantized_cache at the decode-step error model's bars."""
    g = load_golden("big_short.pt")
    m = build_model(g["config"], g["weight_seed"]).to(DEV)
    m.engine_dtype = torch.bfloat16
    m.engine().quiet = True
    ref = g["codes"][0].long()
    runs = {}
    for kv in (None, F8):
        m.kv_cache_dtype = kv
        tr = {"steps": "all"}
        m.engine().generate([g["x"][0]], [g["y"][0]], top_k=1, trace=tr, forced=[ref])
        runs[kv] = torch.stack([tr["ar_logits"][i][0].cpu() for i in range(ref.shape[0] + 1)])
    a, b = runs[F8], runs[None]
    assert bool(torch.isfinite(a).all())
    err = (a - b).abs()
    bar = 10 * 0.03
    agree = float((a.argmax(1) == b.argmax(1)).float().mean())
    print(f"FP8 vs bf16 cache, teacher-forced big_short: max |dlogit| {float(err.max()):.4f}, mean "
          f"{float(err.mean()):.5f}, argmax agreement {agree:.4f}; bar {bar}")
    assert float(err.max()) <= bar


# ---- errors and sizes ------------------------------------------------------------------------------------------------
def test_forward_and_step_argument_errors():
    from valle_b200 import _lib as L
    m = _tiny()
    utts = _utts(1)
    m.kv_cache_dtype = torch.float8_e5m2
    with pytest.raises(ValueError):
        _gen(m, utts)
    m.kv_cache_dtype = F8
    m.engine_dtype = torch.float32
    with pytest.raises(ValueError):
        _gen(m, utts)
    with pytest.raises(ValueError):
        m.inference(utts[0][0][None].to(DEV), torch.tensor([utts[0][0].numel()], dtype=torch.int32),
                    utts[0][1][None].to(DEV), None, top_k=1)
    # the ABI: an FP8 cache on the fp32 decoder is unsupported, in the prefill and in the decode step
    nd = m.engine(torch.float32).ar
    cap, B = 64, 1
    shape = (nd.n_layer, B, nd.H, cap, 64)
    k8 = torch.zeros(shape, dtype=F8, device=DEV)
    ke = torch.zeros(shape[:-1], dtype=torch.uint8, device=DEV)
    x = torch.zeros(4, nd.desc.d_model, device=DEV)
    cu = torch.tensor([0, 4], dtype=torch.int32, device=DEV)

    def forward(nd, kc, vc, ke, ve, slots=None):
        ws = torch.zeros(nd.lib.vb_decoder_forward_workspace(C.byref(nd.desc), 4), dtype=torch.uint8, device=DEV)
        return nd.lib.vb_decoder_forward(nd.handle, x.data_ptr(), 4, B, cu.data_ptr(), cu.data_ptr(), None, 0, 4,
                                         L.VB_MASK_VALLE_AR, None, kc, vc, ke, ve, k8.stride(0), k8.stride(1), cap,
                                         slots, ws.data_ptr(), ws.numel(), L.stream_ptr())

    k, e = k8.data_ptr(), ke.data_ptr()
    assert forward(nd, k, k, e, e) == 3
    s = L.ArState()
    s.B, s.cache_cap = B, cap
    s.kcache = s.vcache = k8.data_ptr()
    s.cache_layer_stride, s.cache_seq_stride = k8.stride(0), k8.stride(1)
    s.kv_dtype, s.k_exp, s.v_exp = L.VB_E4M3, ke.data_ptr(), ke.data_ptr()
    h = L.ArHead()
    nbytes = nd.lib.vb_ar_step_workspace(C.byref(nd.desc), B, cap)
    w2 = torch.zeros(nbytes, dtype=torch.uint8, device=DEV)
    assert nd.lib.vb_ar_decode_step(nd.handle, C.byref(h), C.byref(s), w2.data_ptr(), nbytes, L.stream_ptr()) == 3
    m.engine_dtype = torch.bfloat16
    # the layout the decode attention's 16-byte exponent reads need: a misaligned exponent array is refused up front
    nd = m.engine().ar
    nbytes = nd.lib.vb_ar_step_workspace(C.byref(nd.desc), B, cap)
    w3 = torch.zeros(nbytes, dtype=torch.uint8, device=DEV)
    s.k_exp = ke.data_ptr() + 1
    assert nd.lib.vb_ar_decode_step(nd.handle, C.byref(h), C.byref(s), w3.data_ptr(), nbytes, L.stream_ptr()) == 1
    assert b"16-byte" in nd.lib.vb_last_error()
    assert forward(nd, k, k, e, e + 1) == 1
    assert b"16-byte" in nd.lib.vb_last_error()
    # exponent rows and a slot map need a cache, and the cache and the exponent rows come in pairs
    assert forward(nd, None, None, None, None, cu.data_ptr()) == 1
    assert forward(nd, None, None, e, e) == 1
    assert forward(nd, k, k, e, None) == 1
    assert forward(nd, k, None, None, None) == 1


def test_fp8_buffers_take_half_the_cache_bytes():
    from valle_b200.engine import _ArBuffers
    m = _tiny()
    eng = m.engine()
    b16 = _ArBuffers(eng, 8, 256, 64)
    b8 = _ArBuffers(eng, 8, 256, 64, F8)
    nb = lambda t: t.numel() * t.element_size()   # noqa: E731
    assert b8.kcache.dtype == F8 and b8.k_exp.dtype == torch.uint8
    assert 2 * nb(b8.kcache) == nb(b16.kcache) and 2 * nb(b8.vcache) == nb(b16.vcache)
    assert nb(b8.k_exp) == nb(b8.kcache) // 64 and nb(b8.v_exp) == nb(b8.vcache) // 64
    assert b16.k_exp is None
