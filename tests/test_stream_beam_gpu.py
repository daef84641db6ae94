"""Beam-search requests in the continuous-batching stream, on an H100.

1. Kernel level: a state of single rows (seeded and greedy) and per-row beam groups of widths 4 (at an unaligned row),
   2 and 16, decoded by the mixed tail (vb_ar_head.greedy == 4), equals bit for bit its parts decoded alone: the single
   rows in a greedy == 2 state, each group in a scalar beam_width = n, greedy == 3 state.  One group stops on its
   finished hypothesis after the first step, one at its length cap.
2. vb_ar_admit of a beam group next to a single row, into a running state whose other rows hold NaN: the group's rows
   get the bits of a fresh beam state's first head step, the single row those of a fresh seeded state, and nothing
   else changes.
3. The argument errors of per-row groups.
4. The engine: streams of greedy, seeded and beam requests equal solo decodes, bit for bit; a stream without beam
   requests runs the graphs it ran before; the ValueErrors of invalid num_beams.

As in tests/test_stream_gpu.py, VB_DECODE_NSPLIT = 1, so that every decode kernel computes a row independently of the
batch it shares."""
import ctypes as C

import pytest
import torch

from test_beam_gpu import CAP, DEV, H, NINF, TS, _bits, _head, _lib, _state
from test_decode_step_bitwise_gpu import D, EOS, LDL, NL, _model
from test_stream_gpu import _model as _engine_model
from test_stream_gpu import _rand_utts, _requests, tuned

import valle_b200.engine as E
from valle_b200 import _lib as L
from valle_b200.engine import StreamRequest, _ArBuffers, _draws

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def one_kv_split():
    with tuned(VB_DECODE_NSPLIT=1):
        yield


# ------------------------------------------------------------------------------------------- 1. the mixed step
# the rows of the mixed state: "s" a seeded single row, "g" a greedy one, (n, kind) a beam group of n rows; kinds:
# "run", "fin" (a finished hypothesis that beats every continuation: stops after the first step), "cap" (stops at its
# length cap after two steps)
LAYOUT = ["s", "g", "s", (4, "run"), "g", (2, "fin"), "s", (16, "run"), (2, "cap"), "g", (3, "run")]
STEPS = 5


def _layout():
    """(singles [(row, seeded)], groups [(first row, n, kind)], B)"""
    singles, groups, r = [], [], 0
    for e in LAYOUT:
        if isinstance(e, tuple):
            groups.append((r, e[0], e[1]))
            r += e[0]
        else:
            singles.append((r, e == "s"))
            r += 1
    return singles, groups, r


def _mixed_state(g, B, singles, groups, dtype):
    i32 = dict(dtype=torch.int32)
    text, prompt = torch.zeros(B, **i32), torch.zeros(B, **i32)
    n_gen, max_new = torch.zeros(B, **i32), torch.full((B,), 1 << 20, **i32)
    first, width, parent = torch.full((B,), -1, **i32), torch.zeros(B, **i32), torch.arange(B, **i32)
    score = torch.zeros(B)
    fin = torch.zeros(B, 2)
    fin[:, 0] = NINF
    fin_len = torch.zeros(B, **i32)
    anc = torch.zeros(B, TS, dtype=torch.uint8)
    units = [(r, 1, None) for r, _ in singles] + list(groups)
    for r0, n, kind in units:
        sp = 16 * int(torch.randint(1, 6, (1,), generator=g)) + r0 % 3 - 1
        tx = int(torch.randint(1, sp, (1,), generator=g))
        t = int(torch.randint(2, CAP - 8 - sp, (1,), generator=g))
        rr = slice(r0, r0 + n)
        text[rr], prompt[rr], n_gen[rr] = tx, sp - tx, t
        if kind is None:
            continue
        first[rr], width[rr], parent[rr] = r0, n, r0
        anc[rr] = torch.randint(0, n, (n, TS), generator=g, dtype=torch.uint8)
        score[rr] = -torch.sort(torch.rand(n, generator=g) * 4 * t).values
        if kind == "fin":
            fin[r0] = torch.tensor([float(score[r0]) + 0.5, float(score[r0]) - 1.0])
            fin_len[r0] = t - 2
        if kind == "cap":
            max_new[rr] = t + 1
    kc = torch.randn(NL, B, H, CAP, 64, generator=g).to(dtype)
    vc = torch.randn(NL, B, H, CAP, 64, generator=g).to(dtype)
    for r0, n, _ in groups:                  # a group's prompt rows, prefilled alike
        sp = int(text[r0] + prompt[r0])
        for c in (kc, vc):
            c[:, r0 + 1:r0 + n, :, :sp] = c[:, r0:r0 + 1, :, :sp]
    seeded = torch.zeros(B, dtype=torch.bool)
    for r, s in singles:
        seeded[r] = s
    t = dict(text=text, prompt=prompt, n_gen=n_gen, finished=torch.zeros(B, **i32), max_new=max_new,
             tokens=torch.randint(0, EOS, (B, TS), generator=g, **i32), x=torch.randn(B, D, generator=g),
             logits=torch.zeros(B, LDL), kc=kc, vc=vc, seed=torch.arange(B, dtype=torch.int64) * 7 + 3,
             top_k=torch.where(seeded, torch.arange(B) % 5 + 5, torch.ones(B, dtype=torch.int64)).to(torch.int32),
             temperature=torch.where(seeded, torch.full((B,), 0.9), torch.ones(B)), score=score, anc=anc, fin=fin,
             fin_len=fin_len, fin_anc=torch.randint(0, 2, (B, TS), generator=g, dtype=torch.uint8), first=first,
             width=width, parent=parent)
    return {k: v.to(DEV) for k, v in t.items()}


def _rows(t, rows, n=None):
    """the sub-state of the given rows; n: a scalar beam group (its finished hypothesis at index 0)"""
    out = {k: (v[:, rows] if k in ("kc", "vc") else v[rows]).clone() for k, v in t.items()}
    if n is not None:
        out["parent"] = torch.zeros(len(rows), dtype=torch.int32, device=DEV)
    return out


def _bind(t, B, greedy):
    s = _state(t, B)
    s.sample_seed, s.top_k, s.temperature = t["seed"].data_ptr(), t["top_k"].data_ptr(), t["temperature"].data_ptr()
    if greedy >= 3:
        s.beam_anc, s.beam_score = t["anc"].data_ptr(), t["score"].data_ptr()
        s.beam_fin_score, s.beam_fin_len, s.beam_fin_anc = t["fin"].data_ptr(), t["fin_len"].data_ptr(), \
            t["fin_anc"].data_ptr()
        s.kv_parent = t["parent"].data_ptr()
    if greedy == 4:
        s.beam_first, s.beam_n = t["first"].data_ptr(), t["width"].data_ptr()
    return s


def _decode(m, chain, t, B, greedy, beam_width=0):
    L, lib = _lib()
    s = _bind(t, B, greedy)
    s.beam_width = beam_width
    h = _head(m, chain, greedy)
    nbytes = lib.vb_ar_step_workspace(C.byref(m["nd"].desc), B, CAP)
    ws = torch.zeros(nbytes, dtype=torch.uint8, device=DEV)
    for _ in range(STEPS):
        L.check(lib.vb_ar_decode_step(m["nd"].handle, C.byref(h), C.byref(s), ws.data_ptr(), nbytes, L.stream_ptr()),
                "vb_ar_decode_step")
    torch.cuda.synchronize()
    return t


@pytest.mark.parametrize("chain", ["folded", "fp32", "postln", "unfolded"])
def test_mixed_step_equals_separate_steps(chain):
    singles, groups, B = _layout()
    g = torch.Generator().manual_seed(sum(map(ord, chain)))
    dtype = torch.float32 if chain == "fp32" else torch.bfloat16
    m = _model(chain in ("folded", "unfolded", "fp32"), dtype)
    t0 = _mixed_state(g, B, singles, groups, dtype)
    mixed = _decode(m, chain, {k: v.clone() for k, v in t0.items()}, B, 4)
    rows = [r for r, _ in singles]
    alone = _decode(m, chain, _rows(t0, rows), len(rows), 2)
    for k in ("tokens", "n_gen", "finished", "x"):
        assert torch.equal(_bits(mixed[k][rows]), _bits(alone[k])), (chain, "single rows", k)
    assert bool(mixed["finished"][rows].eq(0).any())
    for r0, n, kind in groups:
        rr = list(range(r0, r0 + n))
        sep = _decode(m, chain, _rows(t0, rr, n), n, 3, beam_width=n)
        for k in ("tokens", "n_gen", "finished", "x", "anc", "score"):
            assert torch.equal(_bits(mixed[k][rr]), _bits(sep[k])), (chain, r0, n, kind, k)
        assert torch.equal(_bits(mixed["fin"][r0]), _bits(sep["fin"][0])), (chain, r0, kind, "fin")
        if float(sep["fin"][0, 0]) > NINF:
            ln = int(sep["fin_len"][0])
            assert int(mixed["fin_len"][r0]) == ln
            assert torch.equal(mixed["fin_anc"][r0, :ln], sep["fin_anc"][0, :ln]), (chain, r0, kind)
        stopped = bool(sep["finished"][0])
        assert stopped == (kind in ("fin", "cap")), (chain, r0, kind)


# ------------------------------------------------------------------------------------------- 2. admission
ADMIT = ["n_gen", "finished", "tokens", "x_cur", "logits", "kcache", "vcache", "beam_anc", "beam_score",
         "beam_fin_score", "beam_fin_len", "beam_fin_anc"]


@pytest.mark.parametrize("chain", ["fp32", "bf16_fold", "postln_bf16"])
def test_admit_group_into_running_state(lib, chain):
    dtype = torch.float32 if chain == "fp32" else torch.bfloat16
    _, m = _engine_model("tiny_postln_pm1.pt" if chain.startswith("postln") else "tiny_pm1.pt", dtype)
    eng = m.engine(dtype)
    eng._refresh()
    nv, B, n = eng.n_vocab, 10, 3
    cap, ts = 512, 264
    pe_a = eng._pe(m.ar_audio_position, cap + 2)
    head4, head3, head2 = (eng._head(pe_a, gr) for gr in (4, 3, 2))
    old, new = _rand_utts(B, 1), _rand_utts(2, 2)
    buf = _ArBuffers(eng, B, cap, ts)
    p = eng._prefill_inputs([u[0] for u in old], [u[1] for u in old], [100] * B)
    buf.set_groups()
    buf.load_rows(p, _draws(B, 0, 7, 0.9), [(r, -1, 1) for r in range(B)])
    h = eng._prefill(buf, p, pe_a)
    L.check(lib.vb_ar_head_step(eng.ar.handle, C.byref(head4), h.data_ptr(), C.byref(buf.st), buf.ws.data_ptr(),
                                buf.ws.numel(), L.stream_ptr()))
    for _ in range(3):
        eng._launch_step(buf, head4)
    # slots: a single row, then a group of n at rows 6..8, in order
    slots = [2, 6, 7, 8]
    others = [s for s in range(B) if s not in slots]
    for name in ("x_cur", "logits", "kcache", "vcache"):
        t = getattr(buf, name)
        if name in ("kcache", "vcache"):
            t[:, others] = float("nan")
        else:
            t[others] = float("nan")
    buf.beam_score[others] = float("nan")
    texts, prompts = [new[0][0]] + [new[1][0]] * n, [new[0][1]] + [new[1][1]] * n
    pn = eng._prefill_inputs(texts, prompts, [100] * 4, slots=slots)
    buf.load_rows(pn, _draws(4, 50, 7, 0.9), [(2, -1, 1)] + [(6, 6, n)] * n)
    torch.cuda.synchronize()
    before = {k: getattr(buf, k).clone() for k in ADMIT}
    hn = eng._prefill(buf, pn, pe_a)
    sl = torch.tensor(slots, dtype=torch.int32, device=DEV)
    ws = torch.empty(lib.vb_ar_admit_workspace(C.byref(eng.ar.desc), 4, nv), dtype=torch.uint8, device=DEV)
    L.check(lib.vb_ar_admit(eng.ar.handle, C.byref(head4), hn.data_ptr(), 4, sl.data_ptr(), C.byref(buf.st),
                            ws.data_ptr(), ws.numel(), L.stream_ptr()), "vb_ar_admit")
    # the references: a fresh beam state holding the group alone, a fresh seeded state holding the single row
    grp = _ArBuffers(eng, n, cap, ts)
    pg = eng._prefill_inputs([new[1][0]] * n, [new[1][1]] * n, [100] * n)
    grp.load_rows(pg)
    grp.n_gen.zero_()
    grp.finished.zero_()
    grp.set_best_of(n, n, False, beams=True)
    hg = eng._prefill(grp, pg, pe_a)
    L.check(lib.vb_ar_head_step(eng.ar.handle, C.byref(head3), hg.data_ptr(), C.byref(grp.st), grp.ws.data_ptr(),
                                grp.ws.numel(), L.stream_ptr()))
    one = _ArBuffers(eng, 1, cap, ts)
    po = eng._prefill_inputs([new[0][0]], [new[0][1]], [100])
    one.load_rows(po, _draws(1, 50, 7, 0.9))
    ho = eng._prefill(one, po, pe_a)
    L.check(lib.vb_ar_head_step(eng.ar.handle, C.byref(head2), ho.data_ptr(), C.byref(one.st), one.ws.data_ptr(),
                                one.ws.numel(), L.stream_ptr()))
    torch.cuda.synchronize()
    assert torch.equal(hn[1:], hg) and torch.equal(hn[:1], ho)
    for k in ADMIT:
        a, b = getattr(buf, k), before[k]
        if k in ("kcache", "vcache"):
            assert torch.equal(_bits(a[:, others]), _bits(b[:, others])), k
        else:
            assert torch.equal(_bits(a[others]), _bits(b[others])), f"{k}: a row outside the admitted slots changed"
    assert int(buf.n_gen[2]) == int(one.n_gen[0]) and int(buf.finished[2]) == int(one.finished[0])
    assert int(buf.tokens[2, 0]) == int(one.tokens[0, 0])
    assert torch.equal(_bits(buf.x_cur[2]), _bits(one.x_cur[0]))
    assert torch.equal(_bits(buf.logits[2, :nv]), _bits(one.logits[0, :nv]))
    for k in ("beam_anc", "beam_score", "beam_fin_score", "beam_fin_len"):
        assert torch.equal(_bits(getattr(buf, k)[2:3]), _bits(before[k][2:3])), f"{k}: the single row's entry changed"
    g = slice(6, 9)
    assert torch.equal(buf.n_gen[g], grp.n_gen) and torch.equal(buf.finished[g], grp.finished)
    assert torch.equal(buf.tokens[g, 0], grp.tokens[:, 0]) and torch.equal(buf.beam_anc[g, 0], grp.beam_anc[:, 0])
    assert torch.equal(_bits(buf.beam_score[g]), _bits(grp.beam_score[:n]))
    assert torch.equal(_bits(buf.x_cur[g]), _bits(grp.x_cur))
    assert float(buf.beam_fin_score[6, 0]) == NINF == float(grp.beam_fin_score[0, 0])
    for s in slots:                          # only position 0 of the slots' token and ancestry rows is written
        assert torch.equal(buf.tokens[s, 1:], before["tokens"][s, 1:])
        assert torch.equal(buf.beam_anc[s, 1:], before["beam_anc"][s, 1:])
    # one more step of everything: the admitted group decodes on as the fresh one does
    buf.x_cur[others] = 0.0
    buf.finished[others] = 1
    eng._launch_step(buf, head4)
    eng._launch_step(grp, head3)
    torch.cuda.synchronize()
    assert torch.equal(buf.tokens[g, :2], grp.tokens[:, :2]) and torch.equal(_bits(buf.x_cur[g]), _bits(grp.x_cur))


# ------------------------------------------------------------------------------------------- 3. argument errors
def test_per_row_group_argument_errors(lib):
    _, m = _engine_model("tiny_pm1.pt", torch.bfloat16)
    eng = m.engine(torch.bfloat16)
    eng._refresh()
    pe_a = eng._pe(m.ar_audio_position, 130)
    head4, head3 = eng._head(pe_a, 4), eng._head(pe_a, 3)

    def status(buf, head, fn="step"):
        if fn == "step":
            return lib.vb_ar_decode_step(eng.ar.handle, C.byref(head), C.byref(buf.st), buf.ws.data_ptr(),
                                         buf.ws.numel(), L.stream_ptr())
        return lib.vb_ar_beam_step(C.byref(head), C.byref(buf.st), eng.d, None, L.stream_ptr())

    buf = _ArBuffers(eng, 8, 128, 136)
    buf.finished.fill_(1)
    buf.set_groups()
    buf.beam_first[2:6], buf.beam_n[2:6] = 2, 4
    assert status(buf, head4) == 0 and status(buf, head4, "beam") == 0
    buf.st.beam_width = 2                   # per-row groups and a scalar width
    assert status(buf, head4) == 1 and b"beam_width" in lib.vb_last_error()
    buf.st.beam_width = 0
    assert status(buf, head3) == 1 and status(buf, head3, "beam") == 1     # per-row groups need greedy == 4
    for bad in (1, 17):
        buf.beam_first[:], buf.beam_n[:] = -1, 0
        buf.beam_first[0:bad if bad < 8 else 8], buf.beam_n[0:8] = 0, bad
        assert status(buf, head4) == 1 and b"not in [2, 16]" in lib.vb_last_error(), bad
        assert status(buf, head4, "beam") == 1
    buf.beam_first[:], buf.beam_n[:] = -1, 0
    buf.beam_first[6:8], buf.beam_n[6:8] = 6, 3      # a group past the last row
    assert status(buf, head4) == 1
    buf.beam_first[:] = -1
    buf.beam_first[3:5], buf.beam_n[3:5] = 3, 2
    sl = torch.tensor([4, 3], dtype=torch.int32, device=DEV)   # the group's slots out of order
    h = torch.zeros((2, eng.d), device=DEV)
    ws = torch.empty(lib.vb_ar_admit_workspace(C.byref(eng.ar.desc), 2, eng.n_vocab), dtype=torch.uint8, device=DEV)
    assert lib.vb_ar_admit(eng.ar.handle, C.byref(head4), h.data_ptr(), 2, sl.data_ptr(), C.byref(buf.st),
                           ws.data_ptr(), ws.numel(), L.stream_ptr()) == 1
    assert b"whole and in order" in lib.vb_last_error()
    assert lib.vb_ar_admit(eng.ar.handle, C.byref(head3), h.data_ptr(), 2, sl.data_ptr(), C.byref(buf.st),
                           ws.data_ptr(), ws.numel(), L.stream_ptr()) == 1
    # the FP8 cache refuses per-row groups, as it refuses beam_width
    f8 = _ArBuffers(eng, 8, 128, 136, torch.float8_e4m3fn)
    f8.finished.fill_(1)
    f8.set_groups()
    f8.st.kv_parent = None                  # the groups alone
    assert status(f8, head4) == 3 and b"FP8" in lib.vb_last_error()
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------- 4. engine
def _beam_requests(g, n, widths, seed=0):
    """_requests' mix of greedy and seeded requests, some with top_p or ras, and every request i with widths[i] > 1 a
    beam request of that width"""
    reqs = _requests(g, n, seeded=True, seed=seed)
    out = []
    for i, r in enumerate(reqs):
        w = widths[i % len(widths)]
        if w > 1:
            r = r._replace(seed=None, top_k=1, temperature=1.0, num_beams=w)
        elif r.seed is not None and i % 4 == 1:
            r = r._replace(top_p=0.85)
        elif r.seed is not None and i % 4 == 3:
            r = r._replace(ras=(8, 0.25))
        out.append(r)
    return out


def _solo(eng, r):
    kw = dict(enroll_lens=None if r.enroll_len is None else [r.enroll_len], max_new_tokens=r.max_new_tokens,
              num_beams=r.num_beams)
    if r.seed is not None:
        kw.update(seed=[r.seed], top_k=r.top_k, temperature=r.temperature, top_p=r.top_p, ras=r.ras)
    return eng.generate([r.text], [r.prompt], **kw)[0].cpu()


def _run(m, reqs, lazy=False, **kw):
    eng = m.engine(m.engine_dtype)
    calls = []
    take = E._take_slots

    def recording(free, widths):
        f = list(free)
        out = take(free, widths)
        calls.append((f, list(widths), out))
        return out
    E._take_slots = recording
    try:
        src = iter(reqs) if lazy else reqs
        if lazy:
            kw["max_context"] = max(eng._context(r) for r in reqs)
        got = {}
        for idx, codes in m.inference_stream(src, **kw):
            assert idx not in got
            got[idx] = codes.cpu()
    finally:
        E._take_slots = take
    assert sorted(got) == list(range(len(reqs)))
    return [got[i] for i in range(len(reqs))], calls


def _check(outs, want, reqs):
    for i, (o, w) in enumerate(zip(outs, want)):
        assert o.shape == w.shape and torch.equal(o, w), (i, reqs[i].num_beams, tuple(o.shape), tuple(w.shape))


STREAMS = [("tiny_pm1.pt", torch.float32, ""), ("tiny_pm1.pt", torch.bfloat16, ""),
           ("tiny_pm1.pt", torch.bfloat16, "nofold"), ("tiny_pm2.pt", torch.float32, ""),
           ("tiny_bos.pt", torch.bfloat16, "lazy"), ("tiny_postln_pm1.pt", torch.bfloat16, ""),
           ("tiny_prenet.pt", torch.float32, "lazy")]


@pytest.mark.parametrize("name,dtype,variant", STREAMS, ids=lambda v: str(v).replace("torch.", ""))
def test_mixed_stream_equals_solo_decodes(name, dtype, variant, monkeypatch):
    if variant == "nofold":
        monkeypatch.setenv("VB_DECODE_FOLD", "0")
    g, m = _engine_model(name, dtype)
    eng = m.engine(dtype)
    reqs = _beam_requests(g, 14, [1, 2, 1, 4, 1, 1, 3, 1, 2])
    outs, calls = _run(m, reqs, lazy=variant == "lazy", slots=5, poll=8)
    assert eng.stats.admissions == len(reqs)
    # the schedule covered: a group waiting for a run while slots were free, a group in slots a single request held,
    # a single request in slots a group held
    assert any(f and len(out) < len(w) and w[len(out)] > 1 for f, w, out in calls)
    history = {}
    group_after_single = single_after_group = False
    for _, w, out in calls:
        for width_i, ss in zip(w, out):
            for s in ss:
                prev = history.get(s)
                group_after_single |= width_i > 1 and prev == 1
                single_after_group |= width_i == 1 and prev is not None and prev > 1
                history[s] = width_i
    assert group_after_single and single_after_group
    _check(outs, [_solo(eng, r) for r in reqs], reqs)


def test_sixteen_beams_in_a_stream():
    g, m = _engine_model("tiny_pm1.pt", torch.bfloat16)
    eng = m.engine(torch.bfloat16)
    reqs = _beam_requests(g, 20, [1, 1, 16, 1, 2, 1, 1, 1, 1, 4])
    outs, _ = _run(m, reqs, slots=18, poll=8)
    _check(outs, [_solo(eng, r) for r in reqs], reqs)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["f32", "bf16"])
def test_no_stale_reads_from_freed_beam_slots(dtype):
    """NaN in the KV cache, x_cur, logits and beam scores of every free slot, and wrong values in its ancestry and
    finished-hypothesis rows, before each admission: a slot's earlier utterance, or never-written rows, must not reach
    the codes"""
    g, m = _engine_model("tiny_pm1.pt", dtype)
    eng = m.engine(dtype)
    reqs = _beam_requests(g, 12, [1, 3, 1, 2, 1, 1, 4], seed=7)
    want, _ = _run(m, reqs, slots=5, poll=8)

    def poisoned():
        for r in reqs:
            for buf in eng._bufs.values():
                if buf.B != 5:
                    continue
                free = (buf.finished != 0).nonzero().flatten()
                for name in ("x_cur", "logits", "beam_score", "beam_fin_score"):
                    getattr(buf, name)[free] = float("nan")
                buf.kcache[:, free] = float("nan")
                buf.vcache[:, free] = float("nan")
                buf.beam_anc[free] = 1
                buf.beam_fin_anc[free] = 1
                buf.beam_fin_len[free] = 3
            yield r

    for buf in eng._bufs.values():
        buf.kcache.fill_(float("nan"))
        buf.vcache.fill_(float("nan"))
    max_context = max(eng._context(r) for r in reqs)
    got = {i: c.cpu() for i, c in m.inference_stream(poisoned(), slots=5, poll=8, max_context=max_context)}
    _check([got[i] for i in range(len(reqs))], want, reqs)


def test_stream_without_beams_is_unchanged_and_beams_add_one_launch():
    g, m = _engine_model("tiny_pm1.pt", torch.bfloat16)
    eng = m.engine(torch.bfloat16)
    reqs = _requests(g, 10, seeded=True)
    eng._bufs.clear()
    list(eng.generate_stream(reqs, slots=3, poll=16))
    buf = next(b for b in eng._bufs.values() if b.B == 3)
    assert buf.st.beam_first is None and not buf.st.kv_parent
    plain = {key[3]: ent[1] for key, ent in buf.graphs.items() if key[-1] == 8}
    assert set(plain) == {2}
    list(eng.generate_stream(reqs[:4] + [reqs[4]._replace(seed=None, top_k=1, num_beams=2)] + reqs[5:], slots=3,
                             poll=16))
    mixed = {key[3]: ent[1] for key, ent in buf.graphs.items() if key[-1] == 8}
    assert mixed[4] == plain[2] + 8, (mixed, plain)   # one launch more per step: the beam tail
    list(eng.generate_stream(reqs, slots=3, poll=16))   # the next stream without beams starts plain again
    assert buf.st.beam_first is None and not buf.st.kv_parent


def test_stream_beam_argument_errors():
    g, m = _engine_model("tiny_pm1.pt", torch.bfloat16)
    r = _requests(g, 1)[0]
    cases = [(dict(num_beams=0), "num_beams"), (dict(num_beams=17), "num_beams"), (dict(num_beams=2.0), "num_beams"),
             (dict(num_beams=2, seed=3), "seed"), (dict(num_beams=2, top_k=4), "top_k"),
             (dict(num_beams=2, top_p=0.9), "top_p"), (dict(num_beams=2, ras=(8, 0.2)), "ras")]
    for kw, what in cases:
        with pytest.raises(ValueError, match=f"request 1: .*{what}"):
            list(m.inference_stream([r, r._replace(**kw)], slots=4))
    with pytest.raises(ValueError, match="request 0: num_beams=4 needs more than the 3 slots"):
        list(m.inference_stream([r._replace(num_beams=4)], slots=3))
    list(m.inference_stream([r._replace(num_beams=1), r._replace(num_beams=3)], slots=3))   # n == slots runs
    _, m8 = _engine_model("tiny_pm1.pt", torch.bfloat16, torch.float8_e4m3fn)
    with pytest.raises(ValueError, match="request 0: .*FP8"):
        list(m8.inference_stream([r._replace(num_beams=2)], slots=4))
