"""The AR decode step (`vb_ar_decode_step`) against its float64 restatement (tests/decode_step_oracle.py), one step per
case with no graph, across the decode chains, batch sizes, split counts, cache lengths and cache contents.

Every case builds the explicit state of one step -- a 2-layer stack with random weights, biases and LayerNorm affines,
random input rows (some with a large common offset), caches filled with random values and a sentinel in every row the
step must not touch, per-row lengths -- fills vb_ar_state / vb_ar_head directly and runs one step.  It then checks:
  * greedy = 0: the stack output left in x_cur and the logits of every running row against the restatement of the
    same chain (the same-chain bar below) and against the unrounded float64 step (the rounding bar below);
  * the appended K / V row of layer 0 within one bf16 ulp (the layer-0 check below); layer 1's within one bf16 ulp
    plus the same-chain bar; every other cache row, every finished row's cache and the logit padding columns
    [1025, 1028) bit for bit unchanged;
  * a second run of the same case is bitwise identical, and marking one more row finished changes no bit of the
    other rows' outputs;
  * greedy = 1: where the restatement's top-2 margin exceeds twice the same-chain bar, the appended token is its
    argmax (or the row stops on EOS), n_gen has advanced and x_cur is the next row's embedding
    audio_emb[tok] + alpha * pe[prompt_len + n_gen] (valle.py:1013-1015, oracle.ar_decode_kv), bit for bit.

Error model (per compared row; S = the row's largest |value| in the restatement, E = the largest |difference| between
the chain's restatement and the same step without any rounding, i.e. the chain's own bf16 rounding effect; rho = the
input row's |mean| / sigma):
  * fp32 accumulation: a K-term fp32 sum is within K 2^-24 of its exact value relative to the sum of |terms|; with
    K <= 4160 keys or 4096 features and the row's terms no larger than S, that is FP32_REL = 4096 * 2^-24 ~ 2.4e-4
    of S.  This is the whole bar of the fp32 chain.
  * bf16 flips: kernel and restatement round at the same points, but an operand whose fp32 and float64 values lie on
    opposite sides of a bf16 rounding boundary differs by one bf16 ulp.  A difference delta ahead of a rounding point
    flips it with probability delta / ulp and costs one ulp when it does, so flips multiply differences (to
    sqrt(delta ulp)) down the chain.  Once they reach the size of an ulp the kernel's roundings and the restatement's
    are independent: the kernel is then as far from the unrounded step as the restatement is, E, and the triangle
    inequality bounds their difference by 2 E.  Same-chain bar: FP32_REL S + 2 E.  This is the worst case over
    rows, not a tight per-row bar: a row whose roundings have not diverged sits far below it (the largest rounding of
    the folded chain, bf16 of the raw rows ahead of layer 0, is shared), the worst rows measured 0.9 E on an H100.
    On the logits 2 E is about 0.03 at rho = 0, no tighter than a plain bf16 tolerance; the tight check of the bf16
    arithmetic is the next one.
  * layer 0's appended K / V row: the QKV projection of layer 0 reads an operand that kernel and restatement share
    bit for bit in the folded and the post-LN chain (bf16 of the same fp32 rows) and the fp32 chain (the rows
    themselves), with the same bf16 weights and the same folded wf.  The only difference ahead of the one rounding
    of k / v is fp32 arithmetic: the K-term sums (a random walk, FP32_WALK = 64 * 2^-24 of the row's scale for K <=
    4096, times 1 + rho for the folded sum that cancels mean * c) and, in the folded chain, the variance taken as
    E[x^2] - mean^2 in fp32, whose relative error (1 + rho)^2 FP32_WALK becomes half that in rstd and in every
    output.  Bar per element: one bf16 ulp of the value (none for fp32) + 2 x that fp32 error.  This is one ulp up
    to rho = 16 and about two at rho = 64.  In the unfolded chain the operand is bf16 of an fp32 LayerNorm, so one
    operand in a row can land on the other side of a rounding boundary; the bar adds the effect of one such flip on
    each output, max_j ulp(a_j) |W[n, j]|.
  * the folded chain rounds the RAW rows to bf16, so its rounding effect grows with the row's offset: a relative
    2^-9 (|mean| + sigma) / sigma of the normalised operand, against 2^-9 for the unfolded chain.  Rounding bar
    (against the unrounded step, so that a wrong rounding point in the restatement cannot hide a kernel error):
    FP32_REL S + 2 * 2^-9 * sqrt(ROUNDINGS - RAW + RAW (1 + rho)^2) * U.  ROUNDINGS = 22 bf16 roundings lie on the
    path of a row through two layers and the head (13 operands, k, v and 9 weight matrices); RAW = 5 of them round the
    raw rows in the folded chain (the QKV and FFN1 operands of both layers, the head's) and 0 elsewhere; they add up as
    a random walk, with a factor 2 of headroom.  U is the size of what the bf16 arithmetic contributes: the logits'
    largest |value|, and for the residual rows of a pre-LN stack the largest |change| the step makes to them (their
    offset passes through the step in fp32 untouched).
The largest error / bar of every chain and the folded-versus-unfolded error at each row offset are written to
decode_step.json in $VB_REPORT_DIR (default: the system temporary directory).

Shapes: d=1024 / 16 heads / dff=4096 (the benchmark model) and d=256 / 4 / 1024 (the tiny fixtures).  d=192 is
refused by vb_decoder_create (d_model and d_ff must be multiples of 256), so the one-split QKV projection runs through
VB_SPLITS_QKV=1 instead of through a narrow model."""
import contextlib
import ctypes as C
import json
import math
import os
import tempfile
import zlib
from dataclasses import dataclass

import pytest
import torch

from oracle import valle_oracle as O

import decode_step_oracle as D

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
PREFIX = "ar_decoder"
N_VOCAB, EOS, LDL = 1025, 1024, 1028
SHAPES = {"big": (1024, 16, 4096), "tiny": (256, 4, 1024)}
FP32_REL = 4096 * 2.0 ** -24
FP32_WALK = 64 * 2.0 ** -24
ROUNDINGS, RAW = 22, 5
SENTINEL = 6144.0   # exact in bf16
REPORT = {}


# ---- model ---------------------------------------------------------------------------------------------------------
_MODELS = {}


def _model(shape, chain):
    """(encoder, NativeDecoder, head tensors, restatement state dict) of one shape and chain, built once"""
    norm_first = chain != "bf16_postln"
    dtype = torch.float32 if chain == "fp32" else torch.bfloat16
    key = (shape, norm_first, dtype)
    if key in _MODELS:
        return _MODELS[key]
    from valle_b200.modules.transformer import LayerNorm, TransformerEncoder, TransformerEncoderLayer
    d, H, dff = SHAPES[shape]
    torch.manual_seed(11)
    enc = TransformerEncoder(TransformerEncoderLayer(d, H, dff, dropout=0.0, batch_first=True, norm_first=norm_first),
                             2, norm=LayerNorm(d) if norm_first else None)
    g = torch.Generator().manual_seed(12 + 2 * int(norm_first))
    with torch.no_grad():
        for name, p in enc.named_parameters():
            if p.ndim == 2:     # the layers are deep copies of one layer: give each its own matrices
                p.copy_(torch.randn(p.shape, generator=g) / math.sqrt(p.shape[1]))
            elif "norm" in name and name.endswith("weight"):
                p.copy_(1.0 + 0.2 * torch.randn(p.shape, generator=g))
            else:
                p.copy_(0.1 * torch.randn(p.shape, generator=g))
    sd = {f"{PREFIX}.{k}": v.detach().clone() for k, v in enc.state_dict().items()}
    enc = enc.to(DEV).eval()
    nd = enc.native(dtype)
    head_w = torch.randn(N_VOCAB, d, generator=g) / math.sqrt(d)
    pe_rows = 4200
    m = dict(d=d, H=H, dff=dff, enc=enc, nd=nd, sd=sd, head_w=head_w, norm_first=norm_first,
             head_dev=head_w.to(DEV, dtype).contiguous(),
             audio_emb=torch.randn(N_VOCAB, d, generator=g).to(DEV),
             alpha=torch.tensor([0.7], device=DEV), pe=O.sine_pe(pe_rows, d).to(DEV), pe_rows=pe_rows, fold=None)
    if dtype == torch.bfloat16 and norm_first:
        assert nd.enable_decode_fold()
        fn = enc.norm
        m["fold"] = nd.fold_layernorm(m["head_dev"], fn.weight.detach(), fn.bias.detach(), None)
    _MODELS[key] = m
    return m


# ---- cases ---------------------------------------------------------------------------------------------------------
@dataclass(frozen=True)
class Case:
    name: str
    shape: str
    chain: str
    B: int
    cap: int
    lens: tuple = ()          # text + prompt + n_gen of each row, cycled over the batch; () = the standard mix
    content: str = "random"   # random | flat | peak_first | peak_last | peak_current | peak_boundary
    offsets: tuple = (0.0,)   # |mean| / sigma of row b: offsets[b % len(offsets)]
    finished: tuple = ()      # rows that have stopped
    tune: tuple = ()          # (name, value) through vb_tune_set


def _c(name, shape, chain, B, cap, **kw):
    return Case(name, shape, chain, B, cap, **{k: tuple(v) if isinstance(v, list) else v for k, v in kw.items()})


OFF = (0.0, 4.0, 16.0, 64.0)
NS = "VB_DECODE_NSPLIT"
Q, OUT, F1, F2 = "VB_SPLITS_QKV", "VB_SPLITS_OUT", "VB_SPLITS_FFN1", "VB_SPLITS_FFN2"
NO_PDL = ("VB_NO_PDL", 1)
CASES = [
    # ---- folded chain (the default) ----
    _c("big_folded_b1_clamp", "big", "bf16_folded", 1, 4160, lens=[4169], content="peak_last"),
    _c("big_folded_b1_peak_boundary", "big", "bf16_folded", 1, 2049, lens=[2049], content="peak_boundary",
       tune=[(NS, 2)]),
    _c("big_folded_b9_qkv7", "big", "bf16_folded", 9, 1100, offsets=OFF, finished=[4],
       tune=[(NS, 7), (Q, 7), (OUT, 3), (F1, 4), (F2, 9)]),
    _c("big_folded_b64_out3", "big", "bf16_folded", 64, 96, offsets=OFF,
       tune=[(NS, 1), (Q, 16), (OUT, 3), (F1, 16), (F2, 16)]),
    _c("big_folded_b17_ns32", "big", "bf16_folded", 17, 300, content="peak_current",
       tune=[(NS, 32), (Q, 5), (OUT, 16), (F1, 1), (F2, 1)]),
    _c("big_folded_b33_nopdl", "big", "bf16_folded", 33, 130, offsets=OFF,
       tune=[(NS, 3), (Q, 2), (OUT, 8), (F1, 16), (F2, 9), NO_PDL]),
    _c("tiny_folded_b1", "tiny", "bf16_folded", 1, 4160, lens=[4160], content="peak_first"),
    _c("tiny_folded_b2_flat", "tiny", "bf16_folded", 2, 700, content="flat", lens=[1, 699], tune=[(NS, 32)]),
    _c("tiny_folded_b9_offsets", "tiny", "bf16_folded", 9, 500, offsets=OFF, tune=[(NS, 7), (Q, 1), (OUT, 1)]),
    _c("tiny_folded_b17_peak_first", "tiny", "bf16_folded", 17, 600, content="peak_first", finished=[0, 5],
       tune=[(NS, 2), (Q, 4), (OUT, 3), (F1, 4), (F2, 9)]),
    _c("tiny_folded_b33_peak_current", "tiny", "bf16_folded", 33, 400, content="peak_current", offsets=OFF,
       tune=[(NS, 3), (OUT, 8), (F2, 16), NO_PDL]),
    _c("tiny_folded_b63", "tiny", "bf16_folded", 63, 200, offsets=OFF, tune=[(NS, 7), (OUT, 16), (F1, 16)]),
    _c("tiny_folded_b64_out3", "tiny", "bf16_folded", 64, 200, offsets=OFF[::-1], finished=[62],
       tune=[(NS, 1), (OUT, 3), (F2, 9)]),
    _c("tiny_folded_b64_default", "tiny", "bf16_folded", 64, 300, content="peak_boundary", tune=[(NS, 3)]),
    # ---- unfolded chain (the head's final norm not folded) ----
    _c("big_unfolded_b2_qkv16", "big", "bf16_unfolded", 2, 4160, lens=[4159, 33], content="peak_last", tune=[(Q, 16)]),
    _c("big_unfolded_b63_qkv1", "big", "bf16_unfolded", 63, 80, offsets=OFF, finished=[1],
       tune=[(NS, 2), (Q, 1), (OUT, 1), (F1, 1), (F2, 1)]),
    _c("big_unfolded_b9_qkv7", "big", "bf16_unfolded", 9, 700, content="peak_first",
       tune=[(NS, 7), (Q, 7), (OUT, 3), (F1, 4), (F2, 9)]),
    _c("tiny_unfolded_b1_qkv1", "tiny", "bf16_unfolded", 1, 3000, lens=[1501], tune=[(NS, 32), (Q, 1)]),
    _c("tiny_unfolded_b17", "tiny", "bf16_unfolded", 17, 500, offsets=OFF, content="peak_current",
       tune=[(NS, 7), (Q, 2), (OUT, 8), (F1, 4), (F2, 16), NO_PDL]),
    _c("tiny_unfolded_b64", "tiny", "bf16_unfolded", 64, 150, finished=[10, 20],
       tune=[(NS, 1), (Q, 4), (OUT, 16), (F2, 9)]),
    # ---- post-LN chain ----
    _c("big_postln_b17", "big", "bf16_postln", 17, 300, content="peak_first"),
    _c("big_postln_b2_qkv1", "big", "bf16_postln", 2, 1500, lens=[1, 1499], tune=[(NS, 7), (Q, 1), (OUT, 3)]),
    _c("tiny_postln_b9_qkv7", "tiny", "bf16_postln", 9, 400, finished=[3],
       tune=[(NS, 32), (Q, 7), (OUT, 1), (F1, 16), (F2, 9)]),
    _c("tiny_postln_b64", "tiny", "bf16_postln", 64, 150, content="flat", tune=[(NS, 3), (Q, 1), NO_PDL]),
    _c("tiny_postln_b1", "tiny", "bf16_postln", 1, 4160, lens=[4160], content="peak_current"),
    # ---- fp32 chain (CUDA-core GEMVs, attn_decode_kernel) ----
    _c("big_fp32_b9", "big", "fp32", 9, 300, offsets=OFF, finished=[2], tune=[(NS, 3)]),
    _c("big_fp32_b1", "big", "fp32", 1, 4160, lens=[4160]),
    _c("tiny_fp32_b33", "tiny", "fp32", 33, 500, content="peak_boundary", tune=[(NS, 7)]),
    _c("tiny_fp32_b2_postln", "tiny", "fp32_postln", 2, 800, lens=[17, 800], tune=[(NS, 32)]),
]


def _chain(case):
    return "fp32" if case.chain == "fp32_postln" else case.chain


def _norm_first(case):
    return case.chain not in ("bf16_postln", "fp32_postln")


def _model_for(case):
    return _model_fp32_postln(case.shape) if case.chain == "fp32_postln" else _model(case.shape, case.chain)


def _model_fp32_postln(shape):
    key = (shape, False, torch.float32)
    if key not in _MODELS:
        bf = _model(shape, "bf16_postln")   # the same weights, fp32 storage
        m = dict(bf)
        m["nd"] = bf["enc"].native(torch.float32)
        m["head_dev"] = bf["head_w"].to(DEV).contiguous()
        m["fold"] = None
        _MODELS[key] = m
    return _MODELS[key]


def _nsplit(case, m):
    """the attention split count of the case (decode_nsplit in attention.cu)"""
    forced = dict(case.tune).get(NS, 0)
    if forced > 0:
        return forced
    sm = torch.cuda.get_device_properties(DEV).multi_processor_count
    ns = min(max(1, (2 * sm + case.B * m["H"] - 1) // (case.B * m["H"])), 32)
    ns = min(ns, max(1, case.cap // 64))
    return max(ns, (case.cap + 4095) // 4096)


def _chunk(kv_len, ns):
    return ((kv_len + ns - 1) // ns + 15) & ~15


def _lengths(case, ns):
    if case.lens:
        return [case.lens[b % len(case.lens)] for b in range(case.B)]
    cap = case.cap
    mix = {0, 1, 15, 16, 17, 63, 64, 65, cap - 1, cap, cap + 9}
    for c in (16, 64, 256):   # split boundaries: the last split holds one key, or the chunks fill exactly, +-1
        mix |= {(ns - 1) * c + 1, ns * c - 1, ns * c, ns * c + 1}
    mix = sorted(v for v in mix if 0 <= v <= cap + 9)
    return [mix[(b * 7) % len(mix)] if case.B < len(mix) else mix[b % len(mix)] for b in range(case.B)]


def _state(case, m):
    """the explicit CPU state of one case: x rows, caches (bf16 values for the bf16 chains), lengths, finished"""
    d, H = m["d"], m["H"]
    g = torch.Generator().manual_seed(zlib.crc32(case.name.encode()))
    B, cap = case.B, case.cap
    ns = _nsplit(case, m)
    tot = _lengths(case, ns)
    text = torch.tensor([t // 3 for t in tot], dtype=torch.int32)
    prompt = torch.tensor([t // 4 for t in tot], dtype=torch.int32)
    n_gen = torch.tensor(tot, dtype=torch.int32) - text - prompt
    finished = torch.zeros(B, dtype=torch.int32)
    for b in case.finished:
        finished[b] = 1
    z = torch.randn(B, d, generator=g, dtype=torch.float64)
    z = (z - z.mean(1, keepdim=True)) / z.std(1, unbiased=False, keepdim=True)
    off = torch.tensor([case.offsets[b % len(case.offsets)] for b in range(B)], dtype=torch.float64)
    x = (z + off[:, None]).float()
    dt = torch.float32 if _chain(case) == "fp32" else torch.bfloat16
    kc = torch.randn(2, B, H, cap, 64, generator=g).to(dt).float()
    vc = torch.randn(2, B, H, cap, 64, generator=g).to(dt).float()
    kv_len = D.kv_lengths(text, prompt, n_gen, cap)
    for b in range(B):   # rows the step must not read: the current token's row and everything past it
        kc[:, b, :, int(kv_len[b]) - 1:] = SENTINEL
        vc[:, b, :, int(kv_len[b]) - 1:] = -SENTINEL
    st = dict(x=x, kc=kc, vc=vc, text=text, prompt=prompt, n_gen=n_gen, finished=finished, ns=ns)
    if case.content == "flat":   # every cached key zero: flat scores apart from the current token's
        for b in range(B):
            kc[:, b, :, :int(kv_len[b]) - 1] = 0.0
    elif case.content.startswith("peak"):
        for layer in range(2):   # the query of each layer from the restatement with the earlier layers' peaks in place
            q = _ref(case, m, st, rounding=False).q[layer]
            for b in range(B):
                n = int(kv_len[b])
                qh = q[b] / (q[b] * q[b]).sum(-1, keepdim=True)                    # [H, 64]: k = c qh scores c/8
                if case.content == "peak_current":
                    kc[layer, b, :, :n - 1] = (-96.0 * qh[:, None, :]).to(dt).float()
                else:
                    row = {"peak_first": 0, "peak_last": max(0, n - 2),
                           "peak_boundary": min(_chunk(n, ns), n - 1)}[case.content]
                    if row < n - 1:
                        kc[layer, b, :, row] = (96.0 * qh).to(dt).float()
    return st


def _ref(case, m, st, rounding=True):
    return D.decode_step(m["sd"], PREFIX, m["head_w"], st["x"], st["kc"], st["vc"], st["text"], st["prompt"],
                         st["n_gen"], st["finished"], m["H"], _chain(case), norm_first=_norm_first(case),
                         rounding=rounding)


# ---- one engine step -----------------------------------------------------------------------------------------------
@contextlib.contextmanager
def _knobs(lib, case):
    from valle_b200 import _lib as L
    try:
        for k, v in case.tune:
            L.check(lib.vb_tune_set(k.encode(), v), "vb_tune_set")
        yield
    finally:
        for k, _ in case.tune:
            lib.vb_tune_set(k.encode(), 0)


def _run(lib, case, m, st, greedy, finished=None):
    """one vb_ar_decode_step from the state st; returns the device state afterwards, on the CPU"""
    from valle_b200 import _lib as L
    B, cap, d = case.B, case.cap, m["d"]
    dt = torch.float32 if _chain(case) == "fp32" else torch.bfloat16
    i32 = dict(dtype=torch.int32, device=DEV)
    t = dict(text=st["text"].to(**i32), prompt=st["prompt"].to(**i32), n_gen=st["n_gen"].to(**i32),
             finished=(st["finished"] if finished is None else finished).to(**i32),
             max_new=torch.full((B,), 1 << 20, **i32), tokens=torch.full((B, cap + 32), -5, **i32),
             x=st["x"].to(DEV), logits=torch.full((B, LDL), SENTINEL, device=DEV),
             kc=st["kc"].to(DEV, dt), vc=st["vc"].to(DEV, dt))
    s = L.ArState()
    s.B, s.tok_stride = B, cap + 32
    s.text_len, s.prompt_len, s.max_new = t["text"].data_ptr(), t["prompt"].data_ptr(), t["max_new"].data_ptr()
    s.n_gen, s.finished, s.tokens = t["n_gen"].data_ptr(), t["finished"].data_ptr(), t["tokens"].data_ptr()
    s.x_cur, s.logits = t["x"].data_ptr(), t["logits"].data_ptr()
    s.kcache, s.vcache = t["kc"].data_ptr(), t["vc"].data_ptr()
    s.cache_layer_stride, s.cache_seq_stride, s.cache_cap = t["kc"].stride(0), t["kc"].stride(1), cap
    h = L.ArHead()
    h.predict_w, h.n_vocab, h.eos_id = m["head_dev"].data_ptr(), N_VOCAB, EOS
    h.audio_emb, h.alpha, h.pe, h.pe_rows = m["audio_emb"].data_ptr(), m["alpha"].data_ptr(), m["pe"].data_ptr(), \
        m["pe_rows"]
    h.greedy = greedy
    if m["fold"] is not None and case.chain == "bf16_folded":
        h.fold = m["fold"]
    nd = m["nd"]
    with _knobs(lib, case):
        nbytes = lib.vb_ar_step_workspace(C.byref(nd.desc), B, cap)   # after the knobs: it depends on the nsplit
        ws = torch.zeros(nbytes, dtype=torch.uint8, device=DEV)
        L.check(lib.vb_ar_decode_step(nd.handle, C.byref(h), C.byref(s), ws.data_ptr(), nbytes, L.stream_ptr()),
                "vb_ar_decode_step")
        torch.cuda.synchronize()
    return {k: v.cpu() for k, v in t.items()}


# ---- checks ----------------------------------------------------------------------------------------------------------
def _row_err(got, ref):
    return (got.double() - ref).abs().amax(dim=-1)


def _rho(case, st):
    """|mean| / sigma of each input row where the chain rounds the raw rows (the folded chain), else 0"""
    x = st["x"].double()
    return (x.mean(1).abs() / x.std(1, unbiased=False)) if case.chain == "bf16_folded" else torch.zeros(case.B)


def _bars(case, st, same, exact):
    """(same-chain bar, rounding bar) of the x and logit rows, same-chain bar of the k and v rows (module docstring)"""
    rho = _rho(case, st)
    bf = 0.0 if _chain(case) == "fp32" else 1.0
    raw = RAW if case.chain == "bf16_folded" else 0
    walk = 2 * 2.0 ** -9 * torch.sqrt(ROUNDINGS - raw + raw * (1.0 + rho) ** 2)
    out = {}
    for name in ("x", "logits", "k_new", "v_new"):
        a, b = getattr(same, name), getattr(exact, name)
        S = b.abs().amax(dim=-1)
        E = (a - b).abs().amax(dim=-1)
        out[name] = [FP32_REL * S + bf * 2.0 * E]
        if name == "x":
            U = (b - st["x"].double()).abs().amax(dim=-1) if _norm_first(case) else S
            out[name].append(FP32_REL * S + bf * walk * U)
        elif name == "logits":
            out[name].append(FP32_REL * S + bf * walk * S)
    return out


def _layer0_kv_tol(case, m, st, want, name):
    """per-element bar of layer 0's appended K or V rows [B, H, 64] (module docstring: layer 0's appended row)"""
    d, H = m["d"], m["H"]
    rho = _rho(case, st)[:, None, None]
    S = want.abs().amax(dim=-1, keepdim=True)
    fp32 = 2 * FP32_WALK * ((1.0 + rho) * S + 0.5 * (1.0 + rho) ** 2 * want.abs())
    if _chain(case) == "fp32":
        return fp32
    tol = _ulp_bf16(want) + fp32
    if case.chain == "bf16_unfolded":
        p = f"{PREFIX}.layers.0."
        sd = m["sd"]
        a = D.bf16(O.layer_norm(st["x"].double(), sd[p + "norm1.weight"].double(), sd[p + "norm1.bias"].double()))
        part = 1 if name == "k_new" else 2
        W = D.bf16(sd[p + "self_attn.in_proj_weight"].double()[part * d:(part + 1) * d]).abs()
        flip = torch.stack([(_ulp_bf16(a[b])[None, :] * W).amax(dim=1) for b in range(case.B)])   # [B, d]
        tol = tol + flip.reshape(case.B, H, 64)
    return tol


def _record(case, name, ratio_same, ratio_exact):
    rec = REPORT.setdefault(case.chain, {"same": 0.0, "exact": 0.0, "worst_same": "", "worst_exact": ""})
    if ratio_same > rec["same"]:
        rec["same"], rec["worst_same"] = ratio_same, f"{case.name}:{name}"
    if ratio_exact > rec["exact"]:
        rec["exact"], rec["worst_exact"] = ratio_exact, f"{case.name}:{name}"


def _write_report():
    out = os.environ.get("VB_REPORT_DIR", tempfile.gettempdir())
    os.makedirs(out, exist_ok=True)
    with open(os.path.join(out, "decode_step.json"), "w") as f:
        json.dump(REPORT, f, indent=1, sort_keys=True)


def _ulp_bf16(v):
    m, e = torch.frexp(v.abs().float())
    return torch.ldexp(torch.ones_like(m), e - 8).double()


@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_decode_step_matches_the_float64_restatement(lib, case):
    m = _model_for(case)
    st = _state(case, m)
    same = _ref(case, m, st)
    exact = _ref(case, m, st, rounding=False)
    bars = _bars(case, st, same, exact)
    run = _run(lib, case, m, st, greedy=0)
    live = (st["finished"] == 0).nonzero().flatten()
    kv_len = same.kv_len
    # stack output and logits
    for name, got in (("x", run["x"]), ("logits", run["logits"][:, :N_VOCAB])):
        bs, be = bars[name]
        es = _row_err(got, getattr(same, name))[live]
        ee = _row_err(got, getattr(exact, name))[live]
        rs, re_ = float((es / bs[live]).max()), float((ee / be[live]).max())
        _record(case, name, rs, re_)
        assert rs <= 1.0, f"{name}: error {float(es.max()):.3g} vs the {case.chain} restatement, {rs:.2f} x its bar"
        assert re_ <= 1.0, f"{name}: error {float(ee.max()):.3g} vs the unrounded step, {re_:.2f} x its bar"
    assert torch.equal(run["logits"][:, N_VOCAB:], torch.full((case.B, LDL - N_VOCAB), SENTINEL)), "logit padding"
    # the appended rows, and nothing else in the caches
    for name, key in (("k_new", "kc"), ("v_new", "vc")):
        got = torch.stack([run[key][:, b, :, int(kv_len[b]) - 1] for b in range(case.B)], 1).double()   # [L, B, H, 64]
        want = getattr(same, name)
        err = (got - want).abs()
        tol0 = _layer0_kv_tol(case, m, st, want[0], name)
        bad0 = (err[0] > tol0)[live]
        assert not bad0.any(), f"layer 0 {name}: {int(bad0.sum())} elements beyond one bf16 ulp + the fp32 error"
        if _chain(case) != "fp32":   # how many elements needed more than the one ulp, and by how much away from zero
            ulps = (err[0] / _ulp_bf16(want[0]))[live]
            away = (want[0].abs() >= want[0].abs().amax(dim=-1, keepdim=True) / 16)[live]
            rec = REPORT.setdefault("layer0_kv", {}).setdefault(case.chain, {"beyond_1ulp": 0, "elements": 0,
                                                                              "max_ulps_above_S/16": 0.0})
            rec["beyond_1ulp"] += int((ulps > 1.0).sum())
            rec["elements"] += ulps.numel()
            rec["max_ulps_above_S/16"] = max(rec["max_ulps_above_S/16"], float(ulps[away].max()))
        tol1 = _ulp_bf16(want[1]) * (_chain(case) != "fp32") + bars[name][0][1][..., None]
        bad1 = (err[1] > tol1)[live]
        assert not bad1.any(), f"layer 1 {name}: {int(bad1.sum())} elements beyond one bf16 ulp + the same-chain bar"
        before = st[key].clone()
        after = run[key].float().clone()
        before[:, live, :, kv_len[live] - 1] = 0.0
        after[:, live, :, kv_len[live] - 1] = 0.0
        assert torch.equal(after, before), f"{key}: a cache row other than the appended one changed"
    # run to run
    again = _run(lib, case, m, st, greedy=0)
    for k in ("x", "logits", "kc", "vc"):
        assert torch.equal(run[k], again[k]), f"{k}: a second run differs"
    # one more finished row changes nothing in the others
    if len(live) > 1:
        fin = st["finished"].clone()
        fin[live[0]] = 1
        other = live[1:]
        alt = _run(lib, case, m, st, greedy=0, finished=fin)
        for k in ("x", "logits"):
            assert torch.equal(alt[k][other], run[k][other]), f"{k}: marking row {int(live[0])} finished changed others"
        for k in ("kc", "vc"):
            assert torch.equal(alt[k][:, other], run[k][:, other])
            assert torch.equal(alt[k][:, live[0]].float(), st[k][:, live[0]]), "a finished row's cache changed"
    # greedy: the argmax, the stop rule and the next row
    gr = _run(lib, case, m, st, greedy=1)
    lg = same.logits
    top2 = lg.topk(2, dim=-1).values
    decided = (top2[:, 0] - top2[:, 1]) > 2 * bars["logits"][0]
    pe_row = lambda b: min(int(st["prompt"][b]) + int(st["n_gen"][b]), m["pe_rows"] - 1)   # noqa: E731
    n_checked = 0
    for b in range(case.B):
        n0 = int(st["n_gen"][b])
        if st["finished"][b]:
            assert int(gr["n_gen"][b]) == n0 and int(gr["finished"][b]) == 1
            assert torch.equal(gr["x"][b], torch.zeros(m["d"]))
            continue
        if not decided[b]:
            continue
        n_checked += 1
        tok = int(lg[b].argmax())
        if tok == EOS:
            assert int(gr["finished"][b]) == (2 if n0 == 0 else 1) and int(gr["n_gen"][b]) == n0
            assert torch.equal(gr["x"][b], torch.zeros(m["d"]))
        else:
            assert int(gr["finished"][b]) == 0 and int(gr["n_gen"][b]) == n0 + 1
            assert int(gr["tokens"][b, n0]) == tok, f"row {b}: token {int(gr['tokens'][b, n0])}, argmax {tok}"
            nxt = m["audio_emb"][tok].cpu() + m["alpha"].cpu() * m["pe"][pe_row(b)].cpu()
            assert torch.equal(gr["x"][b], nxt), f"row {b}: next-row embedding"
    assert n_checked > 0 or len(live) == 0
    _write_report()


def test_folded_chain_error_by_row_offset(lib):
    """The folded chain rounds the raw residual rows to bf16 ahead of the LayerNorm, the unfolded chain the normalised
    rows: on the benchmark model, rows with |mean| / sigma in {0, 4, 16, 64} through both chains against the unrounded
    float64 step.  Each chain stays within its rounding bar at every offset; the errors are reported."""
    rows = []
    for chain in ("bf16_folded", "bf16_unfolded"):
        case = _c(f"offsets_{chain}", "big", chain, 8, 300, offsets=OFF, tune=[(NS, 3)])
        m = _model_for(case)
        st = _state(case, m)
        exact = _ref(case, m, st, rounding=False)
        bars = _bars(case, st, _ref(case, m, st), exact)
        run = _run(lib, case, m, st, greedy=0)
        err = _row_err(run["logits"][:, :N_VOCAB], exact.logits)
        assert bool((err <= bars["logits"][1]).all()), f"{chain}: {err.tolist()} vs {bars['logits'][1].tolist()}"
        rows.append({str(o): float(err[[b for b in range(8) if OFF[b % 4] == o]].max()) for o in OFF})
    REPORT["logit_error_by_offset"] = {"bf16_folded": rows[0], "bf16_unfolded": rows[1]}
    _write_report()
