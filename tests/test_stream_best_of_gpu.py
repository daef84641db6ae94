"""Best-of-n requests and AR log-likelihood scores in the continuous-batching stream, on an H100.

1. The engine: mixed streams of greedy, seeded, beam and best-of (n = 2, 3, 4) requests in fewer slots than they need
   equal generate() on each request alone, codes and (return_scores) score bits, and the schedule covered a parent
   held while its siblings decoded and a request waited, and a sibling's freed slot refilled while its parent decoded.
2. The same on the FP8 KV cache, where each candidate is a row of its own.
3. No stale reads: the free slots and, after each prefix fork, the rows below P of every row reading a parent's
   prefix hold NaN; the codes do not change.
4. The C ABI: vb_ar_fork_prefix copies exactly the rows [P, S + Tp) and refuses the FP8 cache; vb_ar_admit scores the
   first draw into logprob; a greedy == 4 step adds to logprob what greedy == 2 adds for the rows in no group.
5. A bf16 best-of request is prefilled once, and the next plain stream runs plain again.

The test model's EOS row of ar_predict_layer is scaled so that utterances stop by EOS at varied steps (the random tiny
models hardly ever draw it); requests whose decode would stop before its first code are left out.  As in
tests/test_stream_gpu.py, VB_DECODE_NSPLIT = 1."""
import ctypes as C

import pytest
import torch

from test_stream_beam_gpu import _beam_requests
from test_stream_gpu import _model, _rand_utts, tuned

import valle_b200.engine as E
from valle_b200 import _lib as L
from valle_b200.engine import BestOfRequest, _ArBuffers, _draws

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
EOS = 1024


@pytest.fixture(autouse=True)
def one_kv_split():
    with tuned(VB_DECODE_NSPLIT=1):
        yield


@pytest.fixture(scope="module")
def lib():
    return L.load()


# the pre-net model's hidden rows draw EOS less often at the same scale
EOS_SCALE = {"tiny_prenet.pt": 6.0}


def _eos_model(name, dtype, kv=None):
    g, m = _model(name, dtype, kv)
    with torch.no_grad():
        m.ar_predict_layer.weight[EOS] *= EOS_SCALE.get(name, 3.0)
    return g, m


def _bits(t):
    return t.view(torch.int32) if t.dtype == torch.float32 else t


def _solo(eng, item, scores):
    """generate() on the request alone: codes (a list of n for a best-of request) and, with scores, its scores"""
    r, n = (item.request, item.num_samples) if isinstance(item, BestOfRequest) else (item, 1)
    kw = dict(enroll_lens=None if r.enroll_len is None else [r.enroll_len], max_new_tokens=r.max_new_tokens,
              return_device=True)
    if r.num_beams > 1:
        kw.update(num_beams=r.num_beams)
    elif r.seed is not None or scores:
        kw.update(seed=[0 if r.seed is None else r.seed], top_k=r.top_k, temperature=r.temperature, top_p=r.top_p,
                  ras=r.ras, num_samples=n)
    out = eng.generate([r.text], [r.prompt], return_scores=scores, **kw)
    codes, sc = out if scores else (out, None)
    codes = [c.cpu() for c in codes[0]] if n > 1 else codes[0].cpu()
    return codes, None if sc is None else sc[0].clone()


def _mix(g, eng, n_req, best_of, widths, seed=0, beams=True):
    """_beam_requests' greedy / seeded / beam mix, best_of[i % len] > 1 turning a seeded request into a BestOfRequest of
    that many candidates, then the solo results with and without scores; requests whose solo decode stops before its
    first code are left out"""
    reqs, want, want_sc = [], [], []
    for i, r in enumerate(_beam_requests(g, n_req, widths if beams else [1], seed=seed)):
        n = best_of[i % len(best_of)]
        item = BestOfRequest(r, n) if n > 1 and r.seed is not None else r
        try:
            codes, _ = _solo(eng, item, False)
            codes_sc, sc = _solo(eng, item, True)
        except SyntaxError:
            continue
        reqs.append(item)
        want.append(codes)
        want_sc.append((codes_sc, sc))
    return reqs, want, want_sc


def _check(got, want, reqs):
    for i, (o, w) in enumerate(zip(got, want)):
        if isinstance(reqs[i], BestOfRequest):
            assert isinstance(o, list) and len(o) == len(w) == reqs[i].num_samples, i
            for j, (a, b) in enumerate(zip(o, w)):
                assert a.shape == b.shape and torch.equal(a, b), (i, j, tuple(a.shape), tuple(b.shape))
        else:
            assert o.shape == w.shape and torch.equal(o, w), (i, tuple(o.shape), tuple(w.shape))


def _run(m, reqs, scores=False, lazy=False, **kw):
    """the stream's results in request order, and its log: ("take", free, widths, taken) for each admission,
    ("stop", candidates, slot, running before, freed) for each stopped candidate"""
    eng = m.engine(m.engine_dtype)
    log = []
    take, stop = E._take_slots, E._Candidates.stop

    def recording_take(free, widths):
        f = list(free)
        out = take(free, widths)
        log.append(("take", f, list(widths), out))
        return out

    def recording_stop(self, slot):
        before = set(self.running)
        freed = stop(self, slot)
        log.append(("stop", self, slot, before, list(freed)))
        return freed
    E._take_slots, E._Candidates.stop = recording_take, recording_stop
    try:
        if lazy:
            kw["max_context"] = max(eng._context(r.request if isinstance(r, BestOfRequest) else r) for r in reqs)
        got, sc = {}, {}
        for out in m.inference_stream(iter(reqs) if lazy else reqs, return_scores=scores, **kw):
            idx = out[0]
            assert idx not in got
            got[idx] = [c.cpu() for c in out[1]] if isinstance(out[1], list) else out[1].cpu()
            if scores:
                assert out[2].is_cuda and out[2].dtype == torch.float32
                sc[idx] = out[2]
    finally:
        E._take_slots, E._Candidates.stop = take, stop
    assert sorted(got) == list(range(len(reqs)))
    return [got[i] for i in range(len(reqs))], [sc.get(i) for i in range(len(reqs))], log


def _coverage(log):
    """(a parent held while its siblings decoded and a request queued for slots, a sibling's freed slot taken by
    another request while its parent still decoded)"""
    held, waiting_while_held, reused = set(), False, False
    sib_freed = {}                       # slot -> the candidates whose parent still decoded when it was freed
    parent_stopped = set()
    for ev in log:
        if ev[0] == "stop":
            _, c, slot, before, freed = ev
            if c.parent is None:
                continue
            if slot == c.parent:
                parent_stopped.add(id(c))
                if len(before) > 1:
                    held.add(id(c))
            elif c.parent in before:
                sib_freed[slot] = c
            if c.parent in freed:
                held.discard(id(c))
        else:
            _, _, widths, out = ev
            waiting_while_held |= bool(held) and len(widths) > 0
            for ss in out:
                for s in ss:
                    c = sib_freed.pop(s, None)
                    reused |= c is not None and id(c) not in parent_stopped
    return waiting_while_held, reused


def _check_scores(sc, want_sc, reqs):
    for i, (s, (_, w)) in enumerate(zip(sc, want_sc)):
        assert s.shape == w.shape, (i, tuple(s.shape), tuple(w.shape))
        assert torch.equal(_bits(s), _bits(w)), (i, s, w)


# ------------------------------------------------------------------------------------------- 1. the engine
STREAMS = [("tiny_pm1.pt", torch.float32, ""), ("tiny_pm1.pt", torch.bfloat16, ""), ("tiny_pm2.pt", torch.float32, ""),
           ("tiny_bos.pt", torch.bfloat16, "lazy"), ("tiny_postln_pm1.pt", torch.bfloat16, ""),
           ("tiny_prenet.pt", torch.float32, "")]


@pytest.mark.parametrize("name,dtype,variant", STREAMS, ids=lambda v: str(v).replace("torch.", ""))
def test_best_of_stream_equals_solo_decodes(name, dtype, variant):
    g, m = _eos_model(name, dtype)
    eng = m.engine(dtype)
    reqs, want, want_sc = _mix(g, eng, 32, [2, 1, 3, 4, 1], [1, 2, 1, 1, 4, 1, 1, 3, 1])
    assert sum(isinstance(r, BestOfRequest) for r in reqs) >= 6
    lazy = variant == "lazy"
    got, _, log = _run(m, reqs, lazy=lazy, slots=6, poll=2)
    _check(got, want, reqs)
    assert eng.stats.admissions == len(reqs)
    held, reused = _coverage(log)
    # the pre-net model's candidates of one request stop at the same step whenever requests queue: only the reuse of
    # a sibling's slot is covered there
    assert reused and (held or name == "tiny_prenet.pt"), (held, reused)
    got, sc, _ = _run(m, reqs, scores=True, lazy=lazy, slots=6, poll=2)
    _check(got, [c for c, _ in want_sc], reqs)
    _check_scores(sc, want_sc, reqs)


# ------------------------------------------------------------------------------------------- 2. FP8
def test_best_of_stream_on_fp8_cache():
    g, m = _eos_model("tiny_pm1.pt", torch.bfloat16, torch.float8_e4m3fn)
    eng = m.engine(torch.bfloat16)
    reqs, want, want_sc = _mix(g, eng, 14, [3, 1, 2, 1, 4, 1], [1], beams=False)
    got, _, _ = _run(m, reqs, slots=6, poll=4)
    _check(got, want, reqs)
    got, sc, _ = _run(m, reqs, scores=True, slots=6, poll=4)
    _check(got, [c for c, _ in want_sc], reqs)
    _check_scores(sc, want_sc, reqs)
    buf = next(b for b in eng._bufs.values() if b.B == 6 and b.kv_dtype is not None)
    assert not buf.st.kv_parent


# ------------------------------------------------------------------------------------------- 3. no stale reads
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["f32", "bf16"])
def test_no_stale_reads_with_forked_prefixes(lib, dtype):
    g, m = _eos_model("tiny_pm1.pt", dtype)
    eng = m.engine(dtype)
    reqs, want, _ = _mix(g, eng, 14, [3, 1, 2, 1, 4, 1], [1, 1, 2, 1, 1, 1, 3], seed=7)
    B = 5

    def buf5():
        return next(b for b in eng._bufs.values() if b.B == B and b.kv_dtype is None)

    def poisoned():
        for r in reqs:
            for buf in eng._bufs.values():
                if buf.B != B:
                    continue
                fin = buf.finished != 0
                if buf.st.kv_parent:   # a held parent is finished, but its candidates still read it
                    fin[buf.kv_parent[~fin].long()] = False
                free = fin.nonzero().flatten()
                for name in ("x_cur", "logits", "logprob", "beam_score", "beam_fin_score"):
                    getattr(buf, name)[free] = float("nan")
                buf.kcache[:, free] = float("nan")
                buf.vcache[:, free] = float("nan")
            yield r

    fork = lib.vb_ar_fork_prefix
    forks = []

    def poisoning_fork(dec, slots, k, st, stream):
        status = fork(dec, slots, k, st, stream)
        buf = buf5()
        par = buf.kv_parent.cpu()
        P = ((buf.text_len + buf.prompt_len) & ~15).cpu()
        for r in range(B):
            if int(par[r]) != r:     # a row reading its prompt prefix from another: its own rows below P are unused
                buf.kcache[:, r, :, :int(P[r])] = float("nan")
                buf.vcache[:, r, :, :int(P[r])] = float("nan")
        forks.append(k)
        return status

    for buf in eng._bufs.values():
        buf.kcache.fill_(float("nan"))
        buf.vcache.fill_(float("nan"))
    max_context = max(eng._context(r.request if isinstance(r, BestOfRequest) else r) for r in reqs)
    lib.vb_ar_fork_prefix = poisoning_fork
    try:
        got = {}
        for i, c in m.inference_stream(poisoned(), slots=B, poll=4, max_context=max_context):
            got[i] = [x.cpu() for x in c] if isinstance(c, list) else c.cpu()
    finally:
        lib.vb_ar_fork_prefix = fork
    assert forks
    _check([got[i] for i in range(len(reqs))], want, reqs)


# ------------------------------------------------------------------------------------------- 4. the C ABI
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["f32", "bf16"])
def test_fork_prefix_copies_the_prompt_tail(lib, dtype):
    _, m = _model("tiny_pm1.pt", dtype)
    eng = m.engine(dtype)
    eng._refresh()
    B, cap, ts = 7, 128, 72
    buf = _ArBuffers(eng, B, cap, ts)
    g = torch.Generator(device=DEV).manual_seed(3)
    for c in (buf.kcache, buf.vcache):
        c.copy_(torch.randn(c.shape, generator=g, device=DEV).to(dtype))
    # rows 0..2 one family (S + Tp = 37: P = 32), rows 3..4 another (S + Tp = 48 = P: nothing to copy), row 5 its own
    # parent, row 6 a family of its own parent 5 with S + Tp = 21 (P = 16)
    lens = [(12, 25)] * 3 + [(20, 28)] * 2 + [(7, 14), (7, 14)]
    buf.text_len.copy_(torch.tensor([s for s, _ in lens], dtype=torch.int32))
    buf.prompt_len.copy_(torch.tensor([t for _, t in lens], dtype=torch.int32))
    buf.set_parents()
    buf.kv_parent.copy_(torch.tensor([0, 0, 0, 3, 3, 5, 5], dtype=torch.int32))
    before = (buf.kcache.clone(), buf.vcache.clone())
    sl = torch.tensor([1, 2, 4, 5, 6, 0], dtype=torch.int32, device=DEV)
    L.check(lib.vb_ar_fork_prefix(eng.ar.handle, sl.data_ptr(), sl.numel(), C.byref(buf.st), L.stream_ptr()),
            "vb_ar_fork_prefix")
    torch.cuda.synchronize()
    for c, b in zip((buf.kcache, buf.vcache), before):
        want = b.clone()
        for r, p, lo, hi in ((1, 0, 32, 37), (2, 0, 32, 37), (6, 5, 16, 21)):
            want[:, r, :, lo:hi] = b[:, p, :, lo:hi]
        assert torch.equal(c.view(torch.uint8), want.view(torch.uint8))
    f8 = _ArBuffers(eng, B, cap, ts, torch.float8_e4m3fn) if dtype == torch.bfloat16 else None
    if f8 is not None:
        f8.set_parents()
        assert lib.vb_ar_fork_prefix(eng.ar.handle, sl.data_ptr(), 1, C.byref(f8.st), L.stream_ptr()) == 3
        assert b"FP8" in lib.vb_last_error()
    buf.st.kv_parent = None
    assert lib.vb_ar_fork_prefix(eng.ar.handle, sl.data_ptr(), 1, C.byref(buf.st), L.stream_ptr()) == 1
    assert lib.vb_ar_fork_prefix(eng.ar.handle, sl.data_ptr(), 0, C.byref(buf.st), L.stream_ptr()) == 1


@pytest.mark.parametrize("chain", ["fp32", "bf16"])
def test_admit_scores_the_first_draw(lib, chain):
    dtype = torch.float32 if chain == "fp32" else torch.bfloat16
    _, m = _model("tiny_pm1.pt", dtype)
    eng = m.engine(dtype)
    eng._refresh()
    nv, B, cap, ts = eng.n_vocab, 8, 512, 264
    pe_a = eng._pe(m.ar_audio_position, cap + 2)
    head = eng._head(pe_a, 2)
    old, new = _rand_utts(B, 1), _rand_utts(3, 2)
    buf = _ArBuffers(eng, B, cap, ts)
    p = eng._prefill_inputs([u[0] for u in old], [u[1] for u in old], [100] * B)
    buf.load_rows(p, _draws(B, 0, 7, 0.9))
    buf.n_gen.zero_()
    buf.finished.zero_()
    buf.set_best_of(B, 1, True)
    h = eng._prefill(buf, p, pe_a)
    L.check(lib.vb_ar_head_step(eng.ar.handle, C.byref(head), h.data_ptr(), C.byref(buf.st), buf.ws.data_ptr(),
                                buf.ws.numel(), L.stream_ptr()))
    for _ in range(3):
        eng._launch_step(buf, head)
    slots = [5, 0, 3]
    buf.logprob[slots] = float("nan")
    pn = eng._prefill_inputs([u[0] for u in new], [u[1] for u in new], [100] * 3, slots=slots)
    buf.load_rows(pn, _draws(3, 50, [7, 8, 9], 0.9))
    torch.cuda.synchronize()
    before = buf.logprob.clone()
    hn = eng._prefill(buf, pn, pe_a)
    sl = torch.tensor(slots, dtype=torch.int32, device=DEV)
    ws = torch.empty(lib.vb_ar_admit_workspace(C.byref(eng.ar.desc), 3, nv), dtype=torch.uint8, device=DEV)
    L.check(lib.vb_ar_admit(eng.ar.handle, C.byref(head), hn.data_ptr(), 3, sl.data_ptr(), C.byref(buf.st),
                            ws.data_ptr(), ws.numel(), L.stream_ptr()), "vb_ar_admit")
    fresh = _ArBuffers(eng, 3, cap, ts)
    pf = eng._prefill_inputs([u[0] for u in new], [u[1] for u in new], [100] * 3)
    fresh.load_rows(pf, _draws(3, 50, [7, 8, 9], 0.9))
    fresh.n_gen.zero_()
    fresh.finished.zero_()
    fresh.set_best_of(3, 1, True)
    hf = eng._prefill(fresh, pf, pe_a)
    L.check(lib.vb_ar_head_step(eng.ar.handle, C.byref(head), hf.data_ptr(), C.byref(fresh.st), fresh.ws.data_ptr(),
                                fresh.ws.numel(), L.stream_ptr()))
    torch.cuda.synchronize()
    others = [s for s in range(B) if s not in slots]
    assert torch.equal(_bits(buf.logprob[others]), _bits(before[others]))
    assert torch.equal(_bits(buf.logprob[slots]), _bits(fresh.logprob[:3]))
    lp = torch.log_softmax(fresh.logits[:, :nv].double(), -1)
    for i in range(3):   # the first draw's term: log_softmax(raw logits)[token]
        assert abs(float(fresh.logprob[i]) - float(lp[i, int(fresh.tokens[i, 0])])) < 1e-4
        assert float(fresh.logprob[i]) < 0
    # without logprob the admission writes none
    buf.st.logprob = None
    buf.logprob[slots] = 7.0
    L.check(lib.vb_ar_admit(eng.ar.handle, C.byref(head), hn.data_ptr(), 3, sl.data_ptr(), C.byref(buf.st),
                            ws.data_ptr(), ws.numel(), L.stream_ptr()), "vb_ar_admit")
    torch.cuda.synchronize()
    assert torch.all(buf.logprob[slots] == 7.0)


@pytest.mark.parametrize("chain", ["fp32", "bf16"])
def test_mixed_head_scores_single_rows_as_the_seeded_head(lib, chain):
    dtype = torch.float32 if chain == "fp32" else torch.bfloat16
    _, m = _model("tiny_pm1.pt", dtype)
    eng = m.engine(dtype)
    eng._refresh()
    cap, ts, n = 512, 264, 3
    pe_a = eng._pe(m.ar_audio_position, cap + 2)
    head2, head4 = eng._head(pe_a, 2), eng._head(pe_a, 4)
    utts = _rand_utts(4, 5)
    texts, prompts = [u[0] for u in utts[:3]] + [utts[3][0]] * n, [u[1] for u in utts[:3]] + [utts[3][1]] * n
    B = len(texts)
    mixed = _ArBuffers(eng, B, cap, ts)
    p = eng._prefill_inputs(texts, prompts, [60] * B)
    mixed.set_groups()
    mixed.load_rows(p, _draws(B, 20, [5, 1, 9, 1, 1, 1], 0.9), [(r, -1, 1) for r in range(3)] + [(3, 3, n)] * n)
    mixed.n_gen.zero_()
    mixed.finished.zero_()
    mixed.beam_score[3:] = torch.tensor([0.0] + [float("-inf")] * (n - 1), device=DEV)
    mixed.beam_fin_score[:, 0] = float("-inf")
    mixed.logprob.zero_()
    mixed.st.logprob = mixed.logprob.data_ptr()
    single = _ArBuffers(eng, 3, cap, ts)
    ps = eng._prefill_inputs(texts[:3], prompts[:3], [60] * 3)
    single.load_rows(ps, _draws(3, 20, [5, 1, 9], 0.9))
    single.n_gen.zero_()
    single.finished.zero_()
    single.set_best_of(3, 1, True)
    for buf, pp, head in ((mixed, p, head4), (single, ps, head2)):
        h = eng._prefill(buf, pp, pe_a)
        L.check(lib.vb_ar_head_step(eng.ar.handle, C.byref(head), h.data_ptr(), C.byref(buf.st), buf.ws.data_ptr(),
                                    buf.ws.numel(), L.stream_ptr()))
        for _ in range(6):
            eng._launch_step(buf, head)
    torch.cuda.synchronize()
    assert torch.equal(mixed.tokens[:3, :7], single.tokens[:, :7])
    assert torch.equal(_bits(mixed.logprob[:3]), _bits(single.logprob[:3]))
    assert torch.all(single.logprob[:3] < 0)
    assert torch.all(mixed.logprob[3:] == 0)     # beam rows only reduce: their score is beam_score


# ------------------------------------------------------------------------------------------- 5. prefill and reset
def test_best_of_prefills_once_and_streams_reset():
    g, m = _eos_model("tiny_pm1.pt", torch.bfloat16)
    eng = m.engine(torch.bfloat16)
    reqs, _, _ = _mix(g, eng, 10, [1, 4], [1], beams=False)
    b = next(x for x in reqs if isinstance(x, BestOfRequest))
    r = b.request
    plain = [x for x in reqs if not isinstance(x, BestOfRequest)]
    mc = max(eng._context(x.request if isinstance(x, BestOfRequest) else x) for x in reqs)   # one buffer for all
    rows = []
    inputs = eng._prefill_inputs

    def recording(texts, prompts, cap_new, slots=None, forks=None):
        rows.append(sum(int(t.numel()) for t in texts) + sum(int(p.shape[0]) for p in prompts))
        return inputs(texts, prompts, cap_new, slots=slots, forks=forks)
    eng._prefill_inputs = recording
    try:
        out = list(eng.generate_stream([b], slots=4, max_context=mc))
    finally:
        del eng._prefill_inputs
    assert rows == [int(r.text.numel()) + int(r.prompt.shape[0])]
    assert len(out) == 1 and len(out[0][1]) == 4
    list(eng.generate_stream(reqs, slots=4, poll=16, return_scores=True, max_context=mc))
    buf = eng._bufs[(4, (mc + 63) // 64 * 64, (mc + 2 + 7) // 8 * 8, None)]
    assert buf.st.kv_parent and buf.st.logprob
    buf.graphs.clear()
    list(eng.generate_stream(plain, slots=4, poll=16, max_context=mc))
    assert not buf.st.kv_parent and not buf.st.logprob and buf.st.beam_first is None
    keys = [k for k in buf.graphs if k[-1] == 8]
    assert keys and all(k[3] == 2 and not k[5] and not k[6] for k in keys), keys


def test_stream_best_of_argument_errors():
    g, m = _model("tiny_pm1.pt", torch.bfloat16)
    from test_stream_gpu import _requests
    r = _requests(g, 1)[0]
    with pytest.raises(ValueError, match="request 1: num_samples > 1 .* need seed="):
        list(m.inference_stream([r, BestOfRequest(r, 2)], slots=4))
    with pytest.raises(ValueError, match="request 0: num_samples=5 needs more than the 4 slots"):
        list(m.inference_stream([BestOfRequest(r._replace(seed=3), 5)], slots=4))
    with pytest.raises(ValueError, match="request 0: num_beams > 1 cannot be combined with num_samples"):
        list(m.inference_stream(iter([BestOfRequest(r._replace(num_beams=2), 2)]), slots=4, max_context=400))
    # default slots count the candidates
    out = list(m.inference_stream([BestOfRequest(r._replace(seed=3, top_k=5), 3)]))
    assert len(out) == 1 and len(out[0][1]) == 3
