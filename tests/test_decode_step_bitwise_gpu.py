"""The AR decode step (vb_ar_head_step, vb_ar_decode_step), pinned bit for bit across its chains.

A 2-layer stack (d=1024, 16 heads, d_ff=4096: the benchmark model's layer shape, wide enough for every split-count
clamp) is built through valle_b200.modules.transformer from a torch seed, and every input is generated on the CPU.
Each case fills vb_ar_state / vb_ar_head directly, runs vb_ar_head_step and then three vb_ar_decode_step calls (with
greedy = 0 the host's draw is replaced by vb_ar_push_tokens of fixed ids between the calls) and compares with
tests/golden/decode_step_bits.pt:
  - SHA-256 of x_cur, logits, tokens, n_gen, finished and both whole KV caches (with the FP8 cache, both exponent
    arrays as well) after the last call, and of the logits after every call;
  - the number of library launches of every call.
The cases cover the LayerNorm-folded, unfolded and post-LN tensor-core chains on the bf16 and the FP8 cache, the
CUDA-core chain (fp32, and bf16 with VB_DECODE_SIMT), B = 1, 17 and 64 with finished rows, greedy = 0, 1 and 2, and the
switches that change what the chain launches.  A change to the host-side orchestration that keeps every launch, its arguments and its order passes
unchanged.

    python tests/test_decode_step_bitwise_gpu.py --record     # rewrite the fixture from the library as built
"""
import contextlib
import ctypes as C
import hashlib
import math
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import kv_fp8_oracle as K

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
FIXTURE = os.path.join(ROOT, "tests", "golden", "decode_step_bits.pt")
D, H, DFF, NL = 1024, 16, 4096, 2
N_VOCAB, EOS, LDL = 1025, 1024, 1028
CAP, PE_ROWS = 160, 256
STEPS = 3

# name: (chain, B, greedy, finished rows, switches set through vb_tune_set)
CASES = {
    "folded_b1_g1": ("folded", 1, 1, (), ()),
    "folded_b17_g2": ("folded", 17, 2, (3,), ()),
    "folded_b64_g0": ("folded", 64, 0, (5, 40), ()),
    "folded_b17_out16": ("folded", 17, 1, (), (("VB_SPLITS_OUT", 16),)),
    "folded_b64_nopdl": ("folded", 64, 1, (0,), (("VB_NO_PDL", 1),)),
    "unfolded_b1_g0": ("unfolded", 1, 0, (), ()),
    "unfolded_b17_g1": ("unfolded", 17, 1, (16,), ()),
    "unfolded_b64_g2": ("unfolded", 64, 2, (7, 63), ()),
    "unfolded_b17_ffn2_1": ("unfolded", 17, 1, (), (("VB_SPLITS_FFN2", 1),)),
    "postln_b1_g1": ("postln", 1, 1, (), ()),
    "postln_b17_g0": ("postln", 17, 0, (2,), ()),
    "postln_b64_g2": ("postln", 64, 2, (9, 33), ()),
    "postln_b17_nopdl": ("postln", 17, 1, (), (("VB_NO_PDL", 1),)),
    "fp32_b1_g2": ("fp32", 1, 2, (), ()),
    "fp32_b17_g1": ("fp32", 17, 1, (4,), ()),
    "fp32_b64_g0": ("fp32", 64, 0, (), ()),
    "fp32_postln_b17_g1": ("fp32_postln", 17, 1, (1,), ()),
    "simt_b17_g1": ("folded", 17, 1, (6,), (("VB_DECODE_SIMT", 1),)),
    "simt_postln_b64_g2": ("postln", 64, 2, (), (("VB_DECODE_SIMT", 1),)),
}
# the FP8 cache (vb_ar_state.kv_dtype = VB_E4M3): the caches start from tests/kv_fp8_oracle.py's quantization of the
# random bf16 caches, and the exponent arrays are hashed with them
F8_CASES = {
    "f8_folded_b1_g1": ("folded", 1, 1, (), ()),
    "f8_folded_b17_g2": ("folded", 17, 2, (3,), ()),
    "f8_folded_b64_g0": ("folded", 64, 0, (5, 40), ()),
    "f8_folded_b64_nopdl": ("folded", 64, 1, (0,), (("VB_NO_PDL", 1),)),
    "f8_unfolded_b1_g2": ("unfolded", 1, 2, (), ()),
    "f8_unfolded_b17_g0": ("unfolded", 17, 0, (16,), ()),
    "f8_unfolded_b64_g1": ("unfolded", 64, 1, (7, 63), ()),
    "f8_postln_b1_g0": ("postln", 1, 0, (), ()),
    "f8_postln_b17_g1": ("postln", 17, 1, (2,), ()),
    "f8_postln_b64_g2": ("postln", 64, 2, (9, 33), ()),
}
CASES.update(F8_CASES)


def _sha(t):
    return hashlib.sha256(t.detach().contiguous().cpu().reshape(-1).view(torch.uint8).numpy().tobytes()).hexdigest()


_MODELS = {}


def _model(norm_first, dtype):
    """NativeDecoder of the stack, the head's tables and (bf16 pre-LN) the final norm folded into the head"""
    key = (norm_first, dtype)
    if key in _MODELS:
        return _MODELS[key]
    from valle_b200.modules.transformer import LayerNorm, TransformerEncoder, TransformerEncoderLayer
    torch.manual_seed(21)
    enc = TransformerEncoder(TransformerEncoderLayer(D, H, DFF, dropout=0.0, batch_first=True, norm_first=norm_first),
                             NL, norm=LayerNorm(D) if norm_first else None)
    g = torch.Generator().manual_seed(22)
    with torch.no_grad():
        for name, p in enc.named_parameters():
            if p.ndim == 2:
                p.copy_(torch.randn(p.shape, generator=g) / math.sqrt(p.shape[1]))
            elif "norm" in name and name.endswith("weight"):
                p.copy_(1.0 + 0.2 * torch.randn(p.shape, generator=g))
            else:
                p.copy_(0.1 * torch.randn(p.shape, generator=g))
    enc = enc.to(DEV).eval()
    nd = enc.native(dtype)
    head_w = (torch.randn(N_VOCAB, D, generator=g) / math.sqrt(D)).to(DEV, dtype).contiguous()
    m = dict(nd=nd, head_w=head_w, audio_emb=torch.randn(N_VOCAB, D, generator=g).to(DEV),
             alpha=torch.tensor([0.7], device=DEV), pe=torch.randn(PE_ROWS, D, generator=g).to(DEV), fold=None)
    if dtype == torch.bfloat16 and norm_first:
        assert nd.enable_decode_fold()
        m["fold"] = nd.fold_layernorm(head_w, enc.norm.weight.detach(), enc.norm.bias.detach(), None)
    _MODELS[key] = m
    return m


@contextlib.contextmanager
def _switches(lib, tune):
    from valle_b200 import _lib as L
    try:
        for k, v in tune:
            L.check(lib.vb_tune_set(k.encode(), v), "vb_tune_set")
        yield
    finally:
        for k, _ in tune:
            lib.vb_tune_set(k.encode(), 0)


def _run(name):
    from valle_b200 import _lib as L
    lib = L.load()
    chain, B, greedy, finished, tune = CASES[name]
    norm_first = chain in ("folded", "unfolded")
    dtype = torch.float32 if chain.startswith("fp32") else torch.bfloat16
    nd = (m := _model(chain in ("folded", "unfolded", "fp32"), dtype))["nd"]
    g = torch.Generator().manual_seed(sum(map(ord, name)))
    i32 = dict(dtype=torch.int32, device=DEV)
    tot = torch.randint(4, CAP - STEPS - 1, (B,), generator=g)
    text = tot // 3
    prompt = tot // 4
    fin = torch.zeros(B, dtype=torch.int32)
    fin[list(finished)] = 1
    t = dict(text=text.to(**i32), prompt=prompt.to(**i32), n_gen=(tot - text - prompt).to(**i32),
             finished=fin.to(**i32), max_new=torch.full((B,), 1 << 20, **i32),
             tokens=torch.full((B, CAP + 8), -5, **i32), x=torch.randn(B, D, generator=g).to(DEV),
             logits=torch.full((B, LDL), 6144.0, device=DEV),
             kc=torch.randn(NL, B, H, CAP, 64, generator=g).to(DEV, dtype),
             vc=torch.randn(NL, B, H, CAP, 64, generator=g).to(DEV, dtype),
             seed=torch.arange(B, dtype=torch.int64).mul(7919).add(3).to(DEV),
             top_k=torch.randint(1, 60, (B,), generator=g).to(**i32),
             temperature=(0.6 + torch.rand(B, generator=g)).to(DEV))
    if name in F8_CASES:
        for c, e in (("kc", "ke"), ("vc", "ve")):
            t[c], t[e] = (a.to(DEV) for a in K.quantize(t[c].cpu()))
    h_in = torch.randn(B, D, generator=g).to(DEV)
    pushed = torch.randint(0, N_VOCAB - 1, (STEPS + 1, B), generator=g, dtype=torch.int64).to(DEV)
    s = L.ArState()
    s.B, s.tok_stride = B, CAP + 8
    s.text_len, s.prompt_len, s.max_new = t["text"].data_ptr(), t["prompt"].data_ptr(), t["max_new"].data_ptr()
    s.n_gen, s.finished, s.tokens = t["n_gen"].data_ptr(), t["finished"].data_ptr(), t["tokens"].data_ptr()
    s.x_cur, s.logits = t["x"].data_ptr(), t["logits"].data_ptr()
    s.kcache, s.vcache = t["kc"].data_ptr(), t["vc"].data_ptr()
    s.cache_layer_stride, s.cache_seq_stride, s.cache_cap = t["kc"].stride(0), t["kc"].stride(1), CAP
    if name in F8_CASES:
        s.kv_dtype, s.k_exp, s.v_exp = L.VB_E4M3, t["ke"].data_ptr(), t["ve"].data_ptr()
    s.sample_seed, s.top_k, s.temperature = t["seed"].data_ptr(), t["top_k"].data_ptr(), t["temperature"].data_ptr()
    h = L.ArHead()
    h.predict_w, h.n_vocab, h.eos_id = m["head_w"].data_ptr(), N_VOCAB, EOS
    h.audio_emb, h.alpha, h.pe, h.pe_rows = m["audio_emb"].data_ptr(), m["alpha"].data_ptr(), m["pe"].data_ptr(), \
        PE_ROWS
    h.greedy = greedy
    if chain == "folded":
        h.fold = m["fold"]
    r = {"launches": [], "logits_per_call": []}
    with _switches(lib, tune):
        nbytes = lib.vb_ar_step_workspace(C.byref(nd.desc), B, CAP)
        ws = torch.zeros(nbytes, dtype=torch.uint8, device=DEV)
        for step in range(STEPS + 1):
            torch.cuda.synchronize()
            n0 = lib.vb_launch_count()
            if step == 0:
                L.check(lib.vb_ar_head_step(nd.handle, C.byref(h), h_in.data_ptr(), C.byref(s), ws.data_ptr(),
                                            nbytes, L.stream_ptr()), "vb_ar_head_step")
            else:
                L.check(lib.vb_ar_decode_step(nd.handle, C.byref(h), C.byref(s), ws.data_ptr(), nbytes,
                                              L.stream_ptr()), "vb_ar_decode_step")
            torch.cuda.synchronize()
            r["launches"].append(lib.vb_launch_count() - n0)
            r["logits_per_call"].append(_sha(t["logits"]))
            if greedy == 0:
                L.check(lib.vb_ar_push_tokens(C.byref(h), C.byref(s), pushed[step].data_ptr(), D, L.stream_ptr()),
                        "vb_ar_push_tokens")
        torch.cuda.synchronize()
    for k in ("x", "logits", "tokens", "n_gen", "finished", "kc", "vc") + (("ke", "ve") if name in F8_CASES else ()):
        r[k] = _sha(t[k])
    return r


def _diff(got, want):
    assert set(got) == set(want), (sorted(got), sorted(want))
    return [k for k in want if got[k] != want[k]]


@pytest.mark.parametrize("name", sorted(CASES))
def test_decode_step_bits(name):
    want = torch.load(FIXTURE, weights_only=False)[name]
    moved = _diff(_run(name), want)
    assert not moved, f"{name}: differs from the recorded run in {moved}"


if __name__ == "__main__":
    if "--record" not in sys.argv:
        sys.exit("usage: python tests/test_decode_step_bitwise_gpu.py --record")
    rec = {name: _run(name) for name in CASES}
    bad = {name: m for name in CASES if (m := _diff(_run(name), rec[name]))}
    if bad:
        sys.exit(f"two runs of the library disagree: {bad}")
    torch.save(rec, FIXTURE)
    print(f"recorded {len(CASES)} cases to {FIXTURE}")
