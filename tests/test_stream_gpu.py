"""GPU checks of continuous batching (ValleEngine.generate_stream / VALLE.inference_stream) on an H100: the slot-mapped
prefill (vb_decoder_forward with cache_slots) and the admission of rows into a running decode state (vb_ar_admit) at
the kernel level, then the streaming engine against solo decodes of every request, bit for bit.

Solo and streamed decodes run with different batch sizes and cache capacities.  The decode attention's KV split
count follows both (decode_nsplit), and its partial results are combined in split order, so the module pins
VB_DECODE_NSPLIT = 1: then every decode kernel computes each row independently of the batch it shares."""
import contextlib
import ctypes as C

import pytest
import torch

from conftest import build_model, load_golden
from test_post_ln import postln_model
from valle_b200 import _lib as L
from valle_b200.engine import StreamRequest, _ArBuffers, _draws

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
FIXTURES = ["tiny_batch.pt", "tiny_pm1.pt", "tiny_pm2.pt", "tiny_bos.pt", "tiny_prenet.pt", "tiny_postln_pm1.pt"]


@contextlib.contextmanager
def tuned(**knobs):
    lib = L.load()
    for k, v in knobs.items():
        L.check(lib.vb_tune_set(k.encode(), int(v)), "vb_tune_set")
    try:
        yield
    finally:
        for k in knobs:
            lib.vb_tune_set(k.encode(), 0)


@pytest.fixture(autouse=True)
def one_kv_split():
    with tuned(VB_DECODE_NSPLIT=1):
        yield


def _model(name, dtype=torch.float32, kv=None):
    g = load_golden(name)
    m = (postln_model if "postln" in name else build_model)(g["config"], g["weight_seed"])
    if g.get("buffers"):
        m.load_state_dict(g["buffers"], strict=False)
    m = m.to(DEV)
    m.engine_dtype = dtype
    m.kv_cache_dtype = kv
    m.engine(dtype).quiet = True
    return g, m


def _requests(g, n=10, seeded=False, seed=0):
    """the fixture's utterances first (reference codes without max_new_tokens), then random ones with mixed lengths"""
    gen = torch.Generator().manual_seed(seed)
    utts = g["utts"] if "utts" in g else [g]
    reqs = []
    for i in range(n):
        if i < len(utts):
            text, prompt, mnt = utts[i]["x"][0], utts[i]["y"][0], None
        else:
            S = int(torch.randint(4, 13, (1,), generator=gen))
            text = torch.randint(3, 100, (S,), generator=gen)
            prompt = torch.randint(0, 1024, (int(torch.randint(6, 30, (1,), generator=gen)), 8), generator=gen)
            mnt = int(torch.randint(5, 120, (1,), generator=gen))
        enroll = min(int(g.get("enroll", 3)), text.numel()) if g["config"]["prefix_mode"] in (2, 4) else None
        if seeded and i % 3 != 2:   # every third request stays greedy
            reqs.append(StreamRequest(text, prompt, enroll, 1000 + i, [5, 40][i % 2], [0.8, 1.3][i % 2], mnt))
        else:
            reqs.append(StreamRequest(text, prompt, enroll, None, 1, 1.0, mnt))
    return reqs


def _solo(m, r):
    x = r.text[None].to(DEV)
    el = None if r.enroll_len is None else torch.tensor([r.enroll_len], dtype=torch.int32)
    return m.inference(x, torch.tensor([x.shape[1]], dtype=torch.int32), r.prompt[None].to(DEV), el, top_k=r.top_k,
                       temperature=r.temperature, max_new_tokens=r.max_new_tokens, seed=r.seed)[0].cpu()


def _stream(m, reqs, **kw):
    got = {}
    for idx, codes in m.inference_stream(reqs, **kw):
        assert idx not in got, f"index {idx} yielded twice"
        assert codes.is_cuda and codes.dtype == torch.int64
        got[idx] = codes.cpu()
    assert sorted(got) == list(range(len(reqs)))
    return [got[i] for i in range(len(reqs))]


def _check_equal(outs, solos):
    for i, (o, s) in enumerate(zip(outs, solos)):
        assert o.shape == s.shape and torch.equal(o, s), f"request {i}: {tuple(o.shape)} vs solo {tuple(s.shape)}"


# ---------------------------------------------------------------- kernel level: slot-mapped prefill
def _forward(lib, nd, x, cu, S, B, maxlen, kc, vc, ke, ve, slots):
    ws = torch.empty(lib.vb_decoder_forward_workspace(C.byref(nd.desc), x.shape[0]), dtype=torch.uint8, device=DEV)
    ls, ss, cap = kc.stride(0), kc.stride(1), kc.shape[3]
    L.check(lib.vb_decoder_forward(nd.handle, x.data_ptr(), x.shape[0], B, cu.data_ptr(), S.data_ptr(), None, 0, maxlen,
                                   L.VB_MASK_VALLE_AR, None, kc.data_ptr(), vc.data_ptr(), L.ptr(ke), L.ptr(ve), ls, ss,
                                   cap, L.ptr(slots), ws.data_ptr(), ws.numel(), L.stream_ptr()), "vb_decoder_forward")


@pytest.mark.parametrize("kind", ["f32", "bf16", "fp8"])
@pytest.mark.parametrize("slots", [[5, 0, 3], [7, 2, 6, 1, 4]])
def test_slot_mapped_prefill_equals_unmapped_prefill(lib, kind, slots):
    dtype = torch.float32 if kind == "f32" else torch.bfloat16
    _, m = _model("tiny_pm1.pt", dtype)
    nd = m.ar_decoder.native(dtype)
    d, H, nl = 256, 4, 2
    gen = torch.Generator().manual_seed(len(slots))
    Ls = [int(v) for v in torch.randint(20, 150, (len(slots),), generator=gen)]
    Ss = [int(v) for v in torch.randint(3, 15, (len(slots),), generator=gen)]
    B, cap = len(slots), 192
    cu = torch.tensor([0] + list(torch.tensor(Ls).cumsum(0)), dtype=torch.int32, device=DEV)
    S = torch.tensor(Ss, dtype=torch.int32, device=DEV)
    x0 = torch.randn((sum(Ls), d), generator=gen).to(DEV)
    cdt = torch.uint8 if kind == "fp8" else dtype

    def caches(nb, fill):
        kc = torch.full((nl, nb, H, cap, 64), fill, dtype=torch.uint8, device=DEV)
        if cdt != torch.uint8:
            kc = torch.full((nl, nb, H, cap, 64 * torch.finfo(cdt).bits // 8), fill, dtype=torch.uint8,
                            device=DEV).view(cdt)
        ex = [torch.full((nl, nb, H, cap), fill + 1, dtype=torch.uint8, device=DEV) for _ in range(2)] \
            if kind == "fp8" else [None, None]
        return [kc, kc.clone()] + ex

    def raw(t):
        return t.contiguous().view(torch.uint8)

    ident = caches(B, 0x5A)
    xi = x0.clone()
    _forward(lib, nd, xi, cu, S, B, max(Ls), *ident, None)
    xe, explicit = x0.clone(), caches(B, 0x5A)
    _forward(lib, nd, xe, cu, S, B, max(Ls), *explicit, torch.arange(B, dtype=torch.int32, device=DEV))
    assert torch.equal(xe, xi)
    for a, b in zip(explicit, ident):
        if a is not None:
            assert torch.equal(raw(a), raw(b))
    sl = torch.tensor(slots, dtype=torch.int32, device=DEV)
    xs, mapped = x0.clone(), caches(8, 0x5A)
    before = [None if t is None else raw(t).clone() for t in mapped]
    _forward(lib, nd, xs, cu, S, B, max(Ls), *mapped, sl)
    torch.cuda.synchronize()
    assert torch.equal(xs, xi), "the residual rows depend on the slot map"
    for a, b, pre in zip(mapped, ident, before):
        if a is None:
            continue
        for i, s in enumerate(slots):
            assert torch.equal(raw(a[:, s]), raw(b[:, i])), f"slot {s} != identity stream {i}"
        others = [s for s in range(8) if s not in slots]
        assert torch.equal(raw(a[:, others]), pre[:, others]), "a stream outside the slot map was written"


# ---------------------------------------------------------------- kernel level: vb_ar_admit
def _rand_utts(n, seed, S=(4, 12), Tp=(8, 30)):
    gen = torch.Generator().manual_seed(seed)
    out = []
    for _ in range(n):
        s = int(torch.randint(*S, (1,), generator=gen))
        out.append((torch.randint(3, 100, (s,), generator=gen),
                    torch.randint(0, 1024, (int(torch.randint(*Tp, (1,), generator=gen)), 8), generator=gen)))
    return out


def _seeded(greedy, seeds):
    """the draws of the seeded head (greedy == 2): top_k 7, 8, ... and temperature 0.9"""
    return _draws(len(seeds), seeds, [7 + i for i in range(len(seeds))], 0.9) if greedy == 2 else None


STATE = ["n_gen", "finished", "tokens", "x_cur", "logits", "kcache", "vcache"]


@pytest.mark.parametrize("chain", ["fp32", "bf16_fold", "bf16_unfold", "postln_bf16"])
@pytest.mark.parametrize("greedy", [1, 2])
def test_admit_rows_into_running_state(lib, chain, greedy, monkeypatch):
    dtype = torch.float32 if chain == "fp32" else torch.bfloat16
    if chain == "bf16_unfold":
        monkeypatch.setenv("VB_DECODE_FOLD", "0")
    _, m = _model("tiny_postln_pm1.pt" if chain.startswith("postln") else "tiny_pm1.pt", dtype)
    eng = m.engine(dtype)
    eng._refresh()
    assert (eng.ar_head_fold is not None) == (chain == "bf16_fold")
    nv = eng.n_vocab
    cap, ts = 512, 264
    pe_a = eng._pe(m.ar_audio_position, cap + 2)
    head = eng._head(pe_a, greedy)
    old, new = _rand_utts(8, 1), _rand_utts(3, 2)
    buf = _ArBuffers(eng, 8, cap, ts)
    p = eng._prefill_inputs([u[0] for u in old], [u[1] for u in old], [100] * 8)
    buf.load_rows(p, _seeded(greedy, list(range(8))))
    h = eng._prefill(buf, p, pe_a)
    L.check(lib.vb_ar_head_step(eng.ar.handle, C.byref(head), h.data_ptr(), C.byref(buf.st), buf.ws.data_ptr(),
                                buf.ws.numel(), L.stream_ptr()))
    for _ in range(3):
        eng._launch_step(buf, head)
    twin = _ArBuffers(eng, 8, cap, ts)        # the same running state, decoded on without the admission
    for n in STATE + ["text_len", "prompt_len", "max_new", "sample_seed", "top_k", "temperature"]:
        getattr(twin, n).copy_(getattr(buf, n))
    slots = [5, 0, 3]
    sl = torch.tensor(slots, dtype=torch.int32, device=DEV)
    pn = eng._prefill_inputs([u[0] for u in new], [u[1] for u in new], [100] * 3, slots=slots)
    buf.load_rows(pn, _seeded(greedy, [50, 51, 52]))   # rows 5, 0, 3
    before = {n: getattr(buf, n).clone() for n in STATE}
    hn = eng._prefill(buf, pn, pe_a)
    ws = torch.empty(lib.vb_ar_admit_workspace(C.byref(eng.ar.desc), 3, nv), dtype=torch.uint8, device=DEV)
    L.check(lib.vb_ar_admit(eng.ar.handle, C.byref(head), hn.data_ptr(), 3, sl.data_ptr(), C.byref(buf.st),
                            ws.data_ptr(), ws.numel(), L.stream_ptr()), "vb_ar_admit")
    # the reference: the same 3 utterances as a fresh 3-row state
    fresh = _ArBuffers(eng, 3, cap, ts)
    pf = eng._prefill_inputs([u[0] for u in new], [u[1] for u in new], [100] * 3)
    fresh.load_rows(pf, _seeded(greedy, [50, 51, 52]))
    hf = eng._prefill(fresh, pf, pe_a)
    assert torch.equal(hf, hn)
    L.check(lib.vb_ar_head_step(eng.ar.handle, C.byref(head), hf.data_ptr(), C.byref(fresh.st), fresh.ws.data_ptr(),
                                fresh.ws.numel(), L.stream_ptr()))
    torch.cuda.synchronize()
    others = [s for s in range(8) if s not in slots]
    for n in STATE:
        a, b = getattr(buf, n), before[n]
        if n in ("kcache", "vcache"):
            assert torch.equal(a[:, others].view(torch.uint8), b[:, others].view(torch.uint8)), n
        else:
            assert torch.equal(a[others], b[others]), f"{n}: a row outside the admitted slots changed"
    for i, s in enumerate(slots):
        assert int(buf.n_gen[s]) == int(fresh.n_gen[i]) and int(buf.finished[s]) == int(fresh.finished[i])
        assert int(buf.tokens[s, 0]) == int(fresh.tokens[i, 0])
        assert torch.equal(buf.x_cur[s], fresh.x_cur[i])
        assert torch.equal(buf.logits[s, :nv], fresh.logits[i, :nv])
        assert torch.equal(buf.tokens[s, 1:], before["tokens"][s, 1:])
    eng._launch_step(buf, head)
    eng._launch_step(twin, head)
    torch.cuda.synchronize()
    assert torch.equal(buf.logits[others, :nv], twin.logits[others, :nv])
    assert torch.equal(buf.n_gen[others], twin.n_gen[others])


# ---------------------------------------------------------------- engine, end to end
@pytest.mark.parametrize("name", FIXTURES)
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["f32", "bf16"])
@pytest.mark.parametrize("seeded", [False, True], ids=["greedy", "seeded"])
def test_stream_equals_solo_decodes(name, dtype, seeded):
    g, m = _model(name, dtype)
    reqs = _requests(g, 10, seeded)
    outs = _stream(m, reqs, slots=3)
    st = m.engine(dtype).stats
    assert st.admissions == len(reqs) and 0 < st.slot_steps <= st.ar_steps * 3
    _check_equal(outs, [_solo(m, r) for r in reqs])
    if dtype == torch.float32 and not seeded:
        utts = g["utts"] if "utts" in g else [g]
        for i, u in enumerate(utts):
            assert torch.equal(outs[i], u["codes"][0].long()), f"request {i} differs from the reference's codes"


@pytest.mark.parametrize("variant", ["poll1", "poll8", "poll32", "no_graphs", "fp8", "slots_ge_n", "nar_batch2"])
def test_stream_schedules(variant):
    kv = torch.float8_e4m3fn if variant == "fp8" else None
    g, m = _model("tiny_pm1.pt", torch.bfloat16, kv)
    eng = m.engine(torch.bfloat16)
    reqs = _requests(g, 10, seeded=True, seed=3)
    kw = dict(slots=3)
    if variant.startswith("poll"):
        kw["poll"] = int(variant[4:])
    if variant == "nar_batch2":
        kw["nar_batch"] = 2
    if variant == "slots_ge_n":
        kw["slots"] = 12
    eng.use_cuda_graph = variant != "no_graphs"
    try:
        outs = _stream(m, reqs, **kw)
    finally:
        eng.use_cuda_graph = True
    if variant == "slots_ge_n":   # every request in the first admission: the static batch
        want = eng.generate([r.text for r in reqs], [r.prompt for r in reqs], top_k=[r.top_k for r in reqs],
                            temperature=[r.temperature for r in reqs], seed=[r.seed or 0 for r in reqs],
                            max_new_tokens=[r.max_new_tokens or 10 ** 6 for r in reqs])
    else:
        want = [_solo(m, r) for r in reqs]
    _check_equal(outs, want)


def test_bench_size_model_stream_equals_solo():
    import bench
    m = bench.build_model(DEV)
    m.engine_dtype = torch.bfloat16
    m.engine(torch.bfloat16).quiet = True
    texts, prompts = bench.make_batch(24, 11)
    gen = torch.Generator().manual_seed(5)
    mnt = [int(v) for v in torch.randint(20, 201, (24,), generator=gen)]
    reqs = [StreamRequest(t, p, max_new_tokens=n) for t, p, n in zip(texts, prompts, mnt)]
    outs = _stream(m, reqs, slots=8)
    _check_equal(outs, [_solo(m, r) for r in reqs])
    assert [o.shape[0] for o in outs] == mnt   # cap-terminated: random weights never stop early


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["f32", "bf16"])
def test_no_stale_reads_from_freed_slots(dtype):
    """NaN in the KV cache and in the x_cur / logits rows of every free slot, before each admission: a slot's earlier
    utterance, or never-written rows, must not reach the codes"""
    g, m = _model("tiny_pm1.pt", dtype)
    eng = m.engine(dtype)
    reqs = _requests(g, 10, seeded=True, seed=7)
    want = _stream(m, reqs, slots=3, poll=8)

    def poisoned():
        for r in reqs:
            for buf in eng._bufs.values():
                if buf.B != 3:
                    continue
                free = (buf.finished != 0).nonzero().flatten()
                buf.x_cur[free] = float("nan")
                buf.logits[free] = float("nan")
                buf.kcache[:, free] = float("nan")
                buf.vcache[:, free] = float("nan")
            yield r

    max_context = max(eng._context(r) for r in reqs)
    for buf in eng._bufs.values():
        buf.kcache.fill_(float("nan"))
        buf.vcache.fill_(float("nan"))
    got = {i: c.cpu() for i, c in m.inference_stream(poisoned(), slots=3, poll=8, max_context=max_context)}
    _check_equal([got[i] for i in range(len(reqs))], want)


def test_graphs_captured_once_and_same_kernels_per_step():
    g, m = _model("tiny_pm1.pt", torch.bfloat16)
    eng = m.engine(torch.bfloat16)
    reqs = _requests(g, 10)
    eng.generate([r.text for r in reqs[:3]], [r.prompt for r in reqs[:3]], top_k=1, max_new_tokens=40)
    static = [ent[1] for key, ent in eng._bufs[next(k for k in eng._bufs if k[0] == 3)].graphs.items() if key[-1] == 8]
    eng._bufs.clear()
    n_cap = []
    for _ in eng.generate_stream(reqs, slots=3, poll=16):
        n_cap.append(eng.captured_launches)
    assert len(set(n_cap)) == 1, n_cap          # one capture (8 steps), during the first poll window
    buf = next(b for b in eng._bufs.values() if b.B == 3)
    assert [ent[1] for ent in buf.graphs.values()] == static


def test_stream_argument_errors():
    g, m = _model("tiny_pm1.pt", torch.bfloat16)
    r = _requests(g, 1)[0]
    with pytest.raises(ValueError, match="seed"):
        list(m.inference_stream([r._replace(top_k=5)]))
    with pytest.raises(ValueError, match="64 slots"):
        m.inference_stream([r] * 2, slots=65)
    with pytest.raises(ValueError, match="max_context"):
        list(m.inference_stream([r], max_context=20))
    with pytest.raises(ValueError, match="max_context"):
        m.inference_stream(iter([r]))
    g2, m2 = _model("tiny_pm2.pt", torch.float32)
    with pytest.raises(ValueError, match="enroll_len"):
        list(m2.inference_stream([_requests(g2, 1)[0]._replace(enroll_len=None)]))
    m2.inference_stream([r._replace(enroll_len=3)] * 2, slots=70)   # fp32 takes any number of slots
