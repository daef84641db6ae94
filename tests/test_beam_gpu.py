"""Beam search on the GPU: the decode attention that follows the beam ancestry, the beam tail (vb_ar_head.greedy == 3)
and ValleEngine.generate(num_beams=).

1. One decode step with the ancestry table equals, bit for bit, the step without it on a cache in which every row's
   streams physically hold its hypothesis's rows.  Cache rows that no hypothesis references are NaN in the beam run, so
   any read of them would show.
2. The tail's parents, tokens, scores, finished hypothesis and stop flags equal a numpy restatement of the spec in
   include/valle_b200.h ("Beam search"), fed with the device's per-row log-sum-exp so that every fp32 operation is the
   device's.
3. One beam is the seeded greedy tail with logprob: same codes and the same score bits, on every chain.
4. The engine: run-to-run and batch invariance, num_beams=1, scores against a float64 restatement, argument errors.
"""
import ctypes as C

import numpy as np
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
TS = CAP + 8
NINF = float("-inf")


def _lib():
    from valle_b200 import _lib as L
    return L, L.load()


def _bits(x):
    return x.contiguous().view(torch.uint8)


def _head(m, chain, greedy):
    L, _ = _lib()
    h = L.ArHead()
    h.predict_w, h.n_vocab, h.eos_id = m["head_w"].data_ptr(), N_VOCAB, EOS
    h.audio_emb, h.alpha, h.pe, h.pe_rows = m["audio_emb"].data_ptr(), m["alpha"].data_ptr(), m["pe"].data_ptr(), \
        PE_ROWS
    h.greedy = greedy
    if chain == "folded":
        h.fold = m["fold"]
    return h


def _state(t, B):
    L, _ = _lib()
    s = L.ArState()
    s.B, s.tok_stride = B, TS
    s.text_len, s.prompt_len, s.max_new = t["text"].data_ptr(), t["prompt"].data_ptr(), t["max_new"].data_ptr()
    s.n_gen, s.finished, s.tokens = t["n_gen"].data_ptr(), t["finished"].data_ptr(), t["tokens"].data_ptr()
    s.x_cur, s.logits = t["x"].data_ptr(), t["logits"].data_ptr()
    s.kcache, s.vcache = t["kc"].data_ptr(), t["vc"].data_ptr()
    s.cache_layer_stride, s.cache_seq_stride, s.cache_cap = t["kc"].stride(0), t["kc"].stride(1), CAP
    return s


# ------------------------------------------------------------------------------------------- 1. decode attention
# name: (chain, B, n, switches).  The chains are those of tests/test_decode_step_bitwise_gpu.py.  B < 17 rows take
# the split-KV path at the default split count.
STEP_CASES = {
    "folded_b2_n2": ("folded", 2, 2, ()),
    "folded_b16_n16_ns1": ("folded", 16, 16, (("VB_DECODE_NSPLIT", 1),)),
    "folded_b48_n4": ("folded", 48, 4, ()),
    "folded_b48_n16": ("folded", 48, 16, ()),
    "folded_b64_n4_ns3": ("folded", 64, 4, (("VB_DECODE_NSPLIT", 3),)),
    "folded_b64_n8": ("folded", 64, 8, ()),
    "nofold_b2_n2_ns7": ("unfolded", 2, 2, (("VB_DECODE_NSPLIT", 7),)),
    "nofold_b4_n4": ("unfolded", 4, 4, ()),
    "nofold_b48_n2_ns1": ("unfolded", 48, 2, (("VB_DECODE_NSPLIT", 1),)),
    "nofold_b64_n8_ns7": ("unfolded", 64, 8, (("VB_DECODE_NSPLIT", 7),)),
    "postln_b8_n8": ("postln", 8, 8, ()),
    "postln_b48_n2_ns3": ("postln", 48, 2, (("VB_DECODE_NSPLIT", 3),)),
    "postln_b64_n16_ns7": ("postln", 64, 16, (("VB_DECODE_NSPLIT", 7),)),
    "fp32_b16_n16": ("fp32", 16, 16, ()),
    "fp32_b48_n8_ns1": ("fp32", 48, 8, (("VB_DECODE_NSPLIT", 1),)),
    "fp32_b64_n4_ns7": ("fp32", 64, 4, (("VB_DECODE_NSPLIT", 7),)),
}


def _groups(g, B, n):
    """per group: text, prompt (text + prompt of the forms 16k - 1, 16k, 16k + 1) and a generated count t >= 2"""
    text, prompt, n_gen = (torch.zeros(B, dtype=torch.int32) for _ in range(3))
    for r0 in range(0, B, n):
        sp = 16 * int(torch.randint(1, 6, (1,), generator=g)) + (r0 // n) % 3 - 1
        tx = int(torch.randint(1, sp, (1,), generator=g))
        t = int(torch.randint(2, CAP - 4 - sp, (1,), generator=g))
        text[r0:r0 + n], prompt[r0:r0 + n], n_gen[r0:r0 + n] = tx, sp - tx, t
    return text, prompt, n_gen


def _run_step(name, beam, f8=False):
    """one logits-only step (greedy 0).  beam: the ancestry table and kv_parent are set, unreferenced rows are NaN;
    otherwise every row's streams hold its hypothesis's rows.  Returns the state before and after, and the launches."""
    L, lib = _lib()
    chain, B, n, tune = STEP_CASES[name] if name in STEP_CASES else name
    g = torch.Generator().manual_seed(sum(map(ord, str(name))))
    dtype = torch.float32 if chain == "fp32" else torch.bfloat16
    m = _model(chain in ("folded", "unfolded", "fp32"), dtype)
    text, prompt, n_gen = _groups(g, B, n)
    anc = torch.randint(0, n, (B, TS), generator=g, dtype=torch.uint8)
    fin = torch.zeros(B, dtype=torch.int32)
    if B > n:
        fin[n:2 * n] = 1                    # a stopped group
    kc = torch.randn(NL, B, H, CAP, 64, generator=g).to(dtype)
    vc = torch.randn(NL, B, H, CAP, 64, generator=g).to(dtype)
    for c in (kc, vc):
        for r in range(B):                  # the group's prompt rows, prefilled alike
            sp = int(text[r] + prompt[r])
            c[:, r, :, :sp] = c[:, r - r % n, :, :sp]
        if not beam:                        # gather each hypothesis's generated rows into its own streams
            src = c.clone()
            for r in range(B):
                gen0, t = int(text[r] + prompt[r]), int(n_gen[r])
                for i in range(t - 1):
                    c[:, r, :, gen0 + i] = src[:, r - r % n + int(anc[r, i]), :, gen0 + i]
        elif not f8:
            ref = torch.zeros(B, CAP, dtype=torch.bool)
            for r in range(B):              # the rows some hypothesis reads: its prompt rows (below P_b its
                gen0, t = int(text[r] + prompt[r]), int(n_gen[r])   # parent's), its current row ...
                ref[r - r % n, :gen0] = True
                ref[r, gen0 // 16 * 16 if r % n else 0:gen0] = True
                ref[r, gen0 + t - 1] = True
                for i in range(t - 1):      # ... and the generated rows its ancestry names
                    ref[r - r % n + int(anc[r, i]), gen0 + i] = True
            c.permute(1, 3, 0, 2, 4)[~ref] = float("nan")
    i32 = dict(dtype=torch.int32, device=DEV)
    t = dict(text=text.to(**i32), prompt=prompt.to(**i32), n_gen=n_gen.to(**i32), finished=fin.to(**i32),
             max_new=torch.full((B,), 1 << 20, **i32), tokens=torch.full((B, TS), -5, **i32),
             x=torch.randn(B, D, generator=g).to(DEV), logits=torch.full((B, LDL), 6144.0, device=DEV),
             kc=kc.to(DEV), vc=vc.to(DEV), anc=anc.to(DEV),
             parent=(torch.arange(B, dtype=torch.int32) // n * n).to(**i32))
    s = _state(t, B)
    if f8:
        (t["kc"], ke), (t["vc"], ve) = ((a.to(DEV) for a in K.quantize(c.cpu())) for c in (kc, vc))
        t["ke"], t["ve"] = ke, ve
        s = _state(t, B)
        s.kv_dtype, s.k_exp, s.v_exp = L.VB_E4M3, ke.data_ptr(), ve.data_ptr()
    if beam:
        s.beam_width, s.beam_anc = n, t["anc"].data_ptr()
        if not f8:                          # the FP8 cache refuses kv_parent on its own
            s.kv_parent = t["parent"].data_ptr()
    h = _head(m, chain, 0)
    before = {k: v.clone() for k, v in t.items()}
    with _switches(lib, tune):
        nbytes = lib.vb_ar_step_workspace(C.byref(m["nd"].desc), B, CAP)
        ws = torch.zeros(nbytes, dtype=torch.uint8, device=DEV)
        torch.cuda.synchronize()
        n0 = lib.vb_launch_count()
        L.check(lib.vb_ar_decode_step(m["nd"].handle, C.byref(h), C.byref(s), ws.data_ptr(), nbytes, L.stream_ptr()),
                "vb_ar_decode_step")
        torch.cuda.synchronize()
        launches = lib.vb_launch_count() - n0
    return before, t, launches


@pytest.mark.parametrize("name", sorted(STEP_CASES))
def test_beam_step_equals_gathered_step(name):
    b0, got, l_got = _run_step(name, beam=True)
    w0, want, l_want = _run_step(name, beam=False)
    assert l_got == l_want, "the beam step launches differently"
    for k in ("x", "logits", "tokens", "n_gen", "finished"):
        assert torch.equal(_bits(got[k]), _bits(want[k])), f"{name}: {k} differs"
    B = got["n_gen"].shape[0]
    cur = torch.zeros(B, CAP, dtype=torch.bool)
    for r in range(B):
        if int(got["finished"][r]) == 0:
            cur[r, int(got["text"][r] + got["prompt"][r] + got["n_gen"][r]) - 1] = True
    cur = cur.to(DEV)

    def rows(c, mask):
        return c.permute(1, 3, 0, 2, 4)[mask]
    for k in ("kc", "vc"):
        # the rows this step wrote are the same; every other row of either cache is as it was (NaN included)
        assert torch.equal(_bits(rows(got[k], cur)), _bits(rows(want[k], cur))), f"{name}: {k} appended rows differ"
        assert torch.equal(_bits(rows(got[k], ~cur)), _bits(rows(b0[k], ~cur))), f"{name}: {k} changed elsewhere"
        assert torch.equal(_bits(rows(want[k], ~cur)), _bits(rows(w0[k], ~cur)))


def test_fp8_cache_refuses_beams():
    """beam_width > 1 alone (kv_parent NULL) on the FP8 cache: VB_ERR_UNSUPPORTED, and the same step without the
    ancestry runs"""
    L, _ = _lib()
    case = ("folded", 16, 4, ())
    with pytest.raises(L.VbError, match="beam search") as e:
        _run_step(case, beam=True, f8=True)
    assert "status 3" in str(e.value), str(e.value)   # VB_ERR_UNSUPPORTED
    _run_step(case, beam=False, f8=True)


# ------------------------------------------------------------------------------------------- 2. beam tail
def _restate(lg, lse, s, t, cap_step, fin, anc, fin_anc, tokens, n):
    """include/valle_b200.h "Beam search" for one group, in numpy fp32.  lg [n, V] raw logits, lse [n] the device's
    log-sum-exps, s [n] scores, fin = (c, score, len).  Returns the group's expected outputs."""
    fc, fo, flen = fin
    out = dict(fin=(fc, fo, flen), fin_anc=fin_anc.copy())
    if cap_step:
        from_fin = fc > NINF and fc >= s[0]
        stop, par, tok, sc = True, None, None, None
    else:
        c = (s[:, None] + (lg - lse[:, None]).astype(np.float32)).astype(np.float32)
        V = lg.shape[1]
        jj, vv = np.meshgrid(np.arange(n), np.arange(V), indexing="ij")
        order = np.lexsort((vv.ravel(), jj.ravel(), -lg.ravel(), -c.ravel()))
        par, tok, sc = [], [], []
        for r, k in enumerate(order):
            j, v = int(jj.ravel()[k]), int(vv.ravel()[k])
            if len(par) == n:
                break
            if v == EOS:
                if r < n and c[j, v] > fc:
                    fc, fo, flen = c[j, v], s[j], t
                    out["fin_anc"][:t] = anc[j, :t]
            else:
                par.append(j)
                tok.append(v)
                sc.append(c[j, v])
        out["fin"] = (fc, fo, flen)
        stop = fc > NINF and fc >= sc[0]
        from_fin = stop
    out["stop"] = stop
    if stop:
        length = flen if from_fin else t
        src = out["fin_anc"] if from_fin else anc[0]
        out["len"] = length
        out["tokens0"] = np.array([tokens[src[i], i] for i in range(length)], dtype=np.int32)
        out["score0"] = fo if from_fin else s[0]
    else:
        out.update(par=par, tok=tok, sc=np.array(sc, dtype=np.float32))
        new = np.stack([anc[p] for p in par])
        new[:, t] = np.arange(n)
        out["anc"] = new
    return out


# per case: (n, groups).  Group kinds: "start" (t = 0, s = (0, -inf, ...)), "run" (random sorted scores), "ties"
# (exact ties within and across rows), "eos_in" (EOS at rank < n), "eos_out" (EOS at rank >= n), "fin_stop" (an
# earlier finished hypothesis that beats every continuation), "cap" and "cap_fin" (cap steps).
TAIL_CASES = {
    "n1": (1, ["start", "run", "eos_in", "cap", "ties"]),
    "n2": (2, ["start", "run", "ties", "eos_in", "eos_out", "fin_stop", "cap", "cap_fin"]),
    "n4": (4, ["start", "ties", "eos_in", "eos_out", "fin_stop", "run", "cap_fin"]),
    "n8": (8, ["ties", "eos_in", "run", "start", "cap"]),
    "n16": (16, ["ties", "eos_out", "eos_in", "fin_stop"]),
}


@pytest.mark.parametrize("case", sorted(TAIL_CASES))
def test_beam_tail_matches_restatement(case):
    L, lib = _lib()
    n, kinds = TAIL_CASES[case]
    G = len(kinds)
    B = G * n
    rng = np.random.default_rng(sum(map(ord, case)))
    lg = (rng.standard_normal((B, N_VOCAB)) * 3).astype(np.float32)
    score = np.zeros(B, np.float32)
    t = np.zeros(B, np.int32)
    max_new = np.full(B, 1000, np.int32)
    fin = np.zeros((G, 2), np.float32)
    fin[:, 0] = NINF
    fin_len = np.zeros(G, np.int32)
    for gi, kind in enumerate(kinds):
        r = slice(gi * n, gi * n + n)
        tg = 0 if kind == "start" else int(rng.integers(3, 20))
        t[r] = tg
        if kind == "start":
            score[r] = NINF
            score[gi * n] = 0.0
        else:
            score[r] = np.sort(-np.abs(rng.standard_normal(n) * 4 * tg)).astype(np.float32)[::-1]
        lg[r, EOS] = lg[r].min() - 1                              # EOS out of the way unless placed below
        if kind == "ties":
            top = lg[r].max(axis=1)
            for j in range(n):                                    # three equal maxima in every row ...
                lg[gi * n + j, [5, 77, 300]] = top[j] + 1
            if n > 1:                                             # ... and two identical rows with equal scores
                lg[gi * n + 1] = lg[gi * n]
                score[gi * n + 1] = score[gi * n]
        if kind == "eos_in":
            lg[gi * n, EOS] = lg[gi * n].max() + 0.5              # beam 0's EOS ranks first
        if kind == "eos_out":
            row = lg[gi * n + n - 1]
            row[EOS] = np.sort(row)[-(n + 1)]                     # the last beam's EOS: n of its row rank above it
            score[gi * n + n - 1] = score[gi * n:gi * n + n].min()
        if kind == "fin_stop":
            fin[gi] = (score[gi * n] + 0.5, score[gi * n] - 1.0)
            fin_len[gi] = tg - 2
        if kind in ("cap", "cap_fin"):
            max_new[r] = tg - 1
        if kind == "cap_fin":
            fin[gi] = (score[gi * n], score[gi * n] - 2.0)        # a tie goes to the finished hypothesis
            fin_len[gi] = tg - 1
    anc = rng.integers(0, n, (B, TS)).astype(np.uint8)
    fin_anc = rng.integers(0, n, (G, TS)).astype(np.uint8)
    tokens = rng.integers(0, EOS, (B, TS)).astype(np.int32)
    m = _model(True, torch.float32)
    i32 = dict(dtype=torch.int32, device=DEV)
    T = dict(text=torch.full((B,), 3, **i32), prompt=torch.full((B,), 7, **i32),
             max_new=torch.from_numpy(max_new).to(DEV), n_gen=torch.from_numpy(t).to(DEV),
             finished=torch.zeros(B, **i32), tokens=torch.from_numpy(tokens).to(DEV),
             x=torch.full((B, D), 9.0, device=DEV), logits=torch.zeros((B, LDL), device=DEV),
             kc=torch.zeros((1, 1), device=DEV), vc=torch.zeros((1, 1), device=DEV),
             anc=torch.from_numpy(anc).to(DEV), score=torch.from_numpy(score).to(DEV),
             fin=torch.from_numpy(np.concatenate([fin, np.zeros((B - G, 2), np.float32)])).to(DEV),
             fin_len=torch.from_numpy(np.concatenate([fin_len, np.zeros(B - G, np.int32)])).to(DEV),
             fin_anc=torch.from_numpy(np.concatenate([fin_anc, np.zeros((B - G, TS), np.uint8)])).to(DEV),
             lse=torch.full((B,), float("nan"), device=DEV))
    T["logits"][:, :N_VOCAB] = torch.from_numpy(lg).to(DEV)
    s = _state(T, B)
    s.beam_width, s.beam_anc, s.beam_score = n, T["anc"].data_ptr(), T["score"].data_ptr()
    s.beam_fin_score, s.beam_fin_len, s.beam_fin_anc = T["fin"].data_ptr(), T["fin_len"].data_ptr(), \
        T["fin_anc"].data_ptr()
    h = _head(m, "fp32", 3)
    L.check(lib.vb_ar_beam_step(C.byref(h), C.byref(s), D, T["lse"].data_ptr(), L.stream_ptr()), "vb_ar_beam_step")
    torch.cuda.synchronize()
    lse = T["lse"].cpu().numpy()
    emb, pe, alpha = m["audio_emb"].cpu().numpy(), m["pe"].cpu().numpy(), np.float32(m["alpha"].item())
    got = {k: v.cpu().numpy() for k, v in T.items()}
    for gi, kind in enumerate(kinds):
        r0, r = gi * n, slice(gi * n, gi * n + n)
        tg = int(t[r0])
        cap_step = tg > max_new[r0]
        want = _restate(lg[r], lse[r], score[r], tg, cap_step, (fin[gi, 0], fin[gi, 1], int(fin_len[gi])), anc[r],
                        fin_anc[gi], tokens[r], n)
        tag = (case, gi, kind)
        assert bool(want["stop"]) == bool(got["finished"][r0]), tag
        if kind == "fin_stop":
            assert want["stop"], tag
        if kind in ("eos_in",) and n > 1:
            assert want["fin"][2] == tg, tag              # the EOS hypothesis was taken
        wf = want["fin"]
        assert (got["fin"][gi, 0], got["fin"][gi, 1]) == (np.float32(wf[0]), np.float32(wf[1])) or \
            (wf[0] == NINF and got["fin"][gi, 0] == NINF), tag
        if wf[0] > NINF:
            assert got["fin_len"][gi] == wf[2], tag
            assert np.array_equal(got["fin_anc"][gi, :wf[2]], want["fin_anc"][:wf[2]]), tag
        if want["stop"]:
            ln = want["len"]
            assert (got["finished"][r] == (2 if ln == 0 else 1)).all(), tag
            assert got["n_gen"][r0] == ln, tag
            assert np.array_equal(got["tokens"][r0, :ln], want["tokens0"]), tag
            assert got["score"][r0].tobytes() == np.float32(want["score0"]).tobytes(), tag
            assert (got["x"][r] == 0).all(), tag
        else:
            assert (got["finished"][r] == 0).all() and (got["n_gen"][r] == tg + 1).all(), tag
            assert np.array_equal(got["tokens"][r, tg], np.array(want["tok"], np.int32)), tag
            assert got["score"][r].tobytes() == want["sc"].tobytes(), tag
            assert np.array_equal(got["anc"][r, :tg + 1], want["anc"][:, :tg + 1]), tag
            p = pe[min(7 + tg, PE_ROWS - 1)]
            x = emb[want["tok"]] + (alpha * p).astype(np.float32)
            assert got["x"][r].tobytes() == x.astype(np.float32).tobytes(), tag
            if kind == "eos_out":
                assert EOS not in want["tok"] and want["fin"][0] == NINF, tag


# ------------------------------------------------------------------------------------------- 3. one beam = greedy
@pytest.mark.parametrize("chain", ["folded", "unfolded", "postln", "fp32"])
def test_one_beam_is_greedy(chain):
    """beam_width = 1 (greedy == 3) against the seeded greedy tail with logprob (greedy == 2, top_k = 1), 8 steps of
    17 rows, some of which reach their cap on the way"""
    g, b = (_run_greedy(chain, beam) for beam in (False, True))
    for k in ("tokens", "n_gen", "finished", "x", "kc", "vc"):
        assert torch.equal(_bits(g[k]), _bits(b[k])), (chain, k)
    assert torch.equal(_bits(g["logprob"]), _bits(b["score"])), chain
    live = g["finished"] == 0
    assert torch.equal(_bits(g["logits"][live]), _bits(b["logits"][live])), chain
    assert bool((g["finished"] != 0).any()) and bool(live.any())


def _run_greedy(chain, beam):
    L, lib = _lib()
    B, steps = 17, 8
    g = torch.Generator().manual_seed(5)
    dtype = torch.float32 if chain == "fp32" else torch.bfloat16
    m = _model(chain in ("folded", "unfolded", "fp32"), dtype)
    text, prompt, n_gen = _groups(g, B, 1)
    n_gen //= 2                             # room for the steps in the cache
    max_new = n_gen + torch.randint(0, 2 * steps, (B,), generator=g, dtype=torch.int32)
    i32 = dict(dtype=torch.int32, device=DEV)
    t = dict(text=text.to(**i32), prompt=prompt.to(**i32), n_gen=n_gen.to(**i32), finished=torch.zeros(B, **i32),
             max_new=max_new.to(**i32), tokens=torch.full((B, TS), -5, **i32),
             x=torch.randn(B, D, generator=g).to(DEV), logits=torch.zeros((B, LDL), device=DEV),
             kc=torch.randn(NL, B, H, CAP, 64, generator=g).to(DEV, dtype),
             vc=torch.randn(NL, B, H, CAP, 64, generator=g).to(DEV, dtype),
             seed=torch.arange(B, dtype=torch.int64, device=DEV), top_k=torch.ones(B, **i32),
             temperature=torch.ones(B, device=DEV), logprob=torch.full((B,), 0.25, device=DEV),
             score=torch.full((B,), 0.25, device=DEV), anc=torch.zeros((B, TS), dtype=torch.uint8, device=DEV),
             fin=torch.full((B, 2), NINF, device=DEV), fin_len=torch.zeros(B, **i32),
             fin_anc=torch.zeros((B, TS), dtype=torch.uint8, device=DEV))
    s = _state(t, B)
    if beam:
        s.beam_width, s.beam_anc, s.beam_score = 1, t["anc"].data_ptr(), t["score"].data_ptr()
        s.beam_fin_score, s.beam_fin_len, s.beam_fin_anc = t["fin"].data_ptr(), t["fin_len"].data_ptr(), \
            t["fin_anc"].data_ptr()
    else:
        s.sample_seed, s.top_k, s.temperature = t["seed"].data_ptr(), t["top_k"].data_ptr(), t["temperature"].data_ptr()
        s.logprob = t["logprob"].data_ptr()
    h = _head(m, chain, 3 if beam else 2)
    nbytes = lib.vb_ar_step_workspace(C.byref(m["nd"].desc), B, CAP)
    ws = torch.zeros(nbytes, dtype=torch.uint8, device=DEV)
    for _ in range(steps):
        L.check(lib.vb_ar_decode_step(m["nd"].handle, C.byref(h), C.byref(s), ws.data_ptr(), nbytes, L.stream_ptr()),
                "vb_ar_decode_step")
    torch.cuda.synchronize()
    return t


# ------------------------------------------------------------------------------------------- 4. engine
def _utts(g, B, seed):
    reqs = _requests(g, B, seed=seed)
    return [r.text for r in reqs], [r.prompt for r in reqs], [r.enroll_len for r in reqs]


def _restated(logits, codes):
    """float64 sum of log_softmax(l_i)[t_i] over the steps"""
    s = 0.0
    for i, t in enumerate(codes):
        l = logits[i].double()
        s += float(l[t] - torch.logsumexp(l, 0))
    return s


ENGINE_MODELS = [("tiny_pm1.pt", torch.float32), ("tiny_pm1.pt", torch.bfloat16),
                 ("tiny_postln_pm1.pt", torch.bfloat16), ("tiny_postln_pm1.pt", torch.float32),
                 ("tiny_bos.pt", torch.bfloat16), ("tiny_prenet.pt", torch.float32), ("tiny_pm2.pt", torch.bfloat16)]


@pytest.mark.parametrize("model,dtype", ENGINE_MODELS, ids=lambda v: str(v).replace("torch.", ""))
@pytest.mark.parametrize("n", [2, 4])
def test_beam_engine_scores_and_reruns(model, dtype, n):
    """One code matrix per utterance; run-to-run identical; the score is the winner's AR log-likelihood over its
    codes, within the bar of tests/test_best_of_gpu.py's score test (each term within 1.4e-4 of the float64 value, the
    running sum one rounding of |sum| 2^-24 per step), restated on the teacher-forced logits of the returned codes."""
    g, m = _engine_model(model, dtype)
    eng = m.engine(dtype)
    B = 4
    texts, prompts, enroll = _utts(g, B, 3)
    el = enroll if enroll[0] is not None else None
    mnt = [20 + 9 * b for b in range(B)]
    with tuned(VB_DECODE_NSPLIT=1):
        codes, sc = eng.generate(texts, prompts, el, max_new_tokens=mnt, num_beams=n, return_scores=True)
        again = eng.generate(texts, prompts, el, max_new_tokens=mnt, num_beams=n)
        assert len(codes) == B and sc.shape == (B,) and sc.dtype == torch.float32
        for b in range(B):
            c = codes[b]
            assert c.ndim == 2 and c.shape[1] == prompts[b].shape[1] and 1 <= c.shape[0] <= mnt[b]
            assert torch.equal(c, again[b]), b
            tr = {"steps": "all"}
            eng.generate([texts[b]], [prompts[b]], None if el is None else [el[b]], max_new_tokens=c.shape[0] + 1,
                         forced=[c], trace=tr)
            lg = tr["ar_logits"]
            want = _restated([lg[i][0].cpu() for i in range(c.shape[0])], c[:, 0].tolist())
            bar = c.shape[0] * (1.4e-4 + abs(want) * 6e-8)
            assert abs(float(sc[b]) - want) <= bar, (b, float(sc[b]), want, bar)


def test_beam_batch_equals_solo_in_bf16():
    """23 utterances x 3 beams = 69 rows: groups of 21 utterances (63 rows) and 2; with one KV split an utterance's
    result does not depend on its batch.  num_beams=1 is the greedy call."""
    g, m = _engine_model("tiny_pm1.pt", torch.bfloat16)
    eng = m.engine(torch.bfloat16)
    B, n = 23, 3
    texts, prompts, _ = _utts(g, B, 8)
    with tuned(VB_DECODE_NSPLIT=1):
        got, sc = eng.generate(texts, prompts, max_new_tokens=40, num_beams=n, return_scores=True)
        for b in (0, 11, 20, 21, 22):
            solo, s1 = eng.generate([texts[b]], [prompts[b]], max_new_tokens=40, num_beams=n, return_scores=True)
            assert torch.equal(solo[0], got[b]), b
            assert torch.equal(_bits(s1), _bits(sc[b:b + 1])), b
        one = eng.generate(texts[:6], prompts[:6], max_new_tokens=40, num_beams=1)
        greedy = eng.generate(texts[:6], prompts[:6], max_new_tokens=40)
        assert all(torch.equal(a, c) for a, c in zip(one, greedy))


def test_beam_argument_errors():
    g, m = _engine_model("tiny_pm1.pt", torch.bfloat16)
    eng = m.engine(torch.bfloat16)
    texts, prompts, _ = _utts(g, 2, 1)
    for bad in (0, 17, 2.0, True):
        with pytest.raises(ValueError, match="num_beams"):
            eng.generate(texts, prompts, max_new_tokens=5, num_beams=bad)
    for kw in (dict(seed=1), dict(top_k=5), dict(top_p=0.9), dict(seed=1, ras=(10, 0.2))):
        with pytest.raises(ValueError, match="num_beams"):
            eng.generate(texts, prompts, max_new_tokens=5, num_beams=2, **kw)
    with pytest.raises(ValueError, match="num_samples"):
        eng.generate(texts, prompts, max_new_tokens=5, num_beams=2, num_samples=2)
    with pytest.raises(ValueError, match="test hooks"):
        eng.generate(texts, prompts, max_new_tokens=5, num_beams=2, trace={"steps": {0}})
    g8, m8 = _engine_model("tiny_pm1.pt", torch.bfloat16, torch.float8_e4m3fn)
    with pytest.raises(ValueError, match="FP8"):
        m8.engine(torch.bfloat16).generate(texts, prompts, max_new_tokens=5, num_beams=2)
    # VALLE.inference takes num_beams with its sampling default top_k
    x = texts[0][None].to(DEV)
    out = m.inference(x, torch.tensor([x.shape[1]], dtype=torch.int32), prompts[0][None].to(DEV), max_new_tokens=12,
                      num_beams=2)
    assert torch.equal(out[0].cpu(), eng.generate([texts[0]], [prompts[0]], max_new_tokens=12, num_beams=2)[0])


# ------------------------------------------------------------------------------------------- 5. reference oracle
def _oracle_cases():
    from conftest import load_golden
    return load_golden("tiny_beam.pt")


@pytest.mark.parametrize("model", ["tiny_pm1.pt", "tiny_postln_pm1.pt", "tiny_bos.pt", "tiny_prenet.pt",
                                   "tiny_pm2.pt"])
def test_beam_matches_oracle(model):
    """fp32 engine beam search against tests/beam_oracle.py's float64 search over the unmodified reference model
    (tests/golden/tiny_beam.pt, tools/gen_golden_beam.py): the same winner, EOS- and cap-stopped, n in {2, 4}.  Every
    decision of each case clears the fixture's margin bound (2e-3), so the fp32 search must take the same ones; the
    score agrees within 1e-3 (fp32 logits and running sum against float64, at most a few 1e-5 per step here)."""
    fx = _oracle_cases()
    cases = [c for c in fx["cases"] if c["model"] == model]
    assert {c["kind"] for c in cases} == {"eos", "cap"} and {c["n"] for c in cases} == {2, 4}
    _, m = _engine_model(model, torch.float32)
    with torch.no_grad():                   # the fixture's head: exact power-of-two scalings in fp32
        m.ar_predict_layer.weight.mul_(fx["head_scale"])
        m.ar_predict_layer.weight[EOS].mul_(cases[0]["eos_scale"])
    eng = m.engine(torch.float32)
    for c in cases:
        el = None if c["enroll"] is None else [c["enroll"]]
        codes, sc = eng.generate([c["x"][0]], [c["y"][0]], el, max_new_tokens=c["max_new_tokens"], num_beams=c["n"],
                                 return_scores=True)
        tag = (model, c["n"], c["kind"])
        assert torch.equal(codes[0][:, 0].cpu(), c["codes"].long()), tag
        assert codes[0].shape[1] == 8, tag
        assert abs(float(sc[0]) - c["score"]) <= 1e-3, (tag, float(sc[0]), c["score"])
