"""Writes tests/golden/tiny_beam.pt: beam-search results of the UNMODIFIED reference model (loaded through
oracle/ref_loader.py, run on the CPU in float64), searched by tests/beam_oracle.py.

    python tools/gen_golden_beam.py

Models: the tiny fixtures' configurations and weights (the reference's default init under the fixture's weight seed,
plus tests/golden/tiny_prenet.pt's BatchNorm statistics): pre-LN and post-LN prefix mode 1, prepend_bos, add_prenet,
and prefix mode 2 with an enrolled prefix.  ar_predict_layer's weight (shared with the AR audio embedding) is scaled
by HEAD_SCALE = 4, exactly in fp32, as tiny_scale widens its margins: the logits spread and the search's decisions
are far from ties.  Its EOS row is scaled by EOS_SCALE more (4, or 8 for the pre-net model), so that an untrained model's EOS logit sometimes
dominates and the search can stop by EOS (the row is never embedded: EOS is never appended).  Per model and n in {2, 4}, random (text, prompt) inputs are drawn until one case stops by EOS and
one at its max_new_tokens cap, each with every decision margin of tests/beam_oracle.py at least MARGIN.

MARGIN: the fp32 engine's scores differ from these float64 ones by the fp32 rounding of the logits (relative 1e-6 of
|l| <= 60 per logit, through the tiny model's two layers a few 1e-5 at most) and of the running sum (one rounding of
|s| 2^-24 per step), summed over at most 100 steps: well below 2e-3, which a decision's margin must clear.
The fixture stores per case: the source fixture, the inputs, n, max_new_tokens, the winner's first-codebook ids, its
float64 score, the margin and how the search stopped.
"""
from __future__ import annotations

import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import torch.nn.functional as F  # noqa: E402

from beam_oracle import beam_search  # noqa: E402
from oracle import ref_loader  # noqa: E402
from oracle.gen_golden import make_inputs, save  # noqa: E402

HEAD_SCALE = 4.0
EOS_SCALE = {"tiny_prenet.pt": 8.0}   # 4.0 for the others
MARGIN = 2e-3
MODELS = ("tiny_pm1.pt", "tiny_postln_pm1.pt", "tiny_bos.pt", "tiny_prenet.pt", "tiny_pm2.pt")
NUM_AUDIO_TOKENS = 1024


def reference_model(ref, name):
    g = torch.load(os.path.join(ROOT, "tests", "golden", name), weights_only=False)
    c = g["config"]
    torch.manual_seed(g["weight_seed"])
    m = ref.VALLE(c["d_model"], c["nhead"], c["num_layers"], norm_first=c.get("norm_first", True),
                  add_prenet=c.get("add_prenet", False), prefix_mode=c["prefix_mode"], share_embedding=True,
                  nar_scale_factor=c.get("nar_scale_factor", 1.0), prepend_bos=c.get("prepend_bos", False),
                  num_quantizers=c["num_quantizers"]).eval()
    with torch.no_grad():
        for k, v in g.get("buffers", {}).items():
            m.get_buffer(k).copy_(v)
        m.ar_predict_layer.weight.mul_(HEAD_SCALE)
        m.ar_predict_layer.weight[NUM_AUDIO_TOKENS].mul_(EOS_SCALE.get(name, 4.0))
    return m.double(), c


def ar_logits_fn(m, x, y):
    """the reference's AR step (valle.py:993-1039) on text x [1, S] and prompt y [1, Tp, 8], as a function of the
    generated first-codebook ids"""
    xe = m.ar_text_position(m.ar_text_prenet(m.ar_text_embedding(x)))
    prompt = y[..., 0]
    if m.ar_audio_prepend_bos:
        prompt = F.pad(prompt, (1, 0), value=NUM_AUDIO_TOKENS + 1)
    S = x.shape[1]

    def fn(tokens):
        yy = torch.cat([prompt, torch.tensor([tokens], dtype=torch.int64).view(1, -1)], dim=1)
        y_pos = m.ar_audio_position(m.ar_audio_prenet(m.ar_audio_embedding(yy)))
        xy = torch.concat([xe, y_pos], dim=1)
        L = yy.shape[1]
        x_mask = F.pad(torch.zeros((S, S), dtype=torch.bool), (0, L), value=True)
        y_mask = F.pad(torch.triu(torch.ones(L, L, dtype=torch.bool), diagonal=1), (S, 0), value=False)
        dec, _ = m.ar_decoder((xy, None), mask=torch.concat([x_mask, y_mask], dim=0))
        return m.ar_predict_layer(dec[:, -1])[0]
    return fn


def main():
    ref = ref_loader.load_reference()
    cases = []
    for name in MODELS:
        m, c = reference_model(ref, name)
        for n in (2, 4):
            want = {"eos", "cap"}
            gen = torch.Generator().manual_seed(1000 + 10 * MODELS.index(name) + n)
            for attempt in range(40):
                if not want:
                    break
                S, Tp = int(torch.randint(4, 8, (1,), generator=gen)), int(torch.randint(6, 16, (1,), generator=gen))
                x, y = make_inputs(gen, S, Tp)
                kind_try = "cap" if "cap" in want and (attempt % 2 or "eos" not in want) else "eos"
                mnt = int(torch.randint(3, 9, (1,), generator=gen)) if kind_try == "cap" else None
                cap_new = 16 * S - (1 if c.get("prepend_bos") else 0)
                if mnt is not None:
                    cap_new = min(cap_new, mnt - 1)
                with torch.no_grad():
                    toks, score, margin, kind = beam_search(ar_logits_fn(m, x, y), n, cap_new)
                ok = kind in want and margin >= MARGIN and len(toks) > 0
                print(f"{name} n={n} S={S} Tp={Tp} mnt={mnt}: {kind} T={len(toks)} margin={margin:.4g}"
                      f"{'  kept' if ok else ''}")
                if ok:
                    want.discard(kind)
                    cases.append(dict(model=name, n=n, x=x, y=y, enroll=3 if c["prefix_mode"] in (2, 4) else None,
                                      max_new_tokens=mnt, codes=torch.tensor(toks, dtype=torch.int16),
                                      score=float(score), margin=float(margin), kind=kind,
                                      eos_scale=EOS_SCALE.get(name, 4.0)))
            assert not want, f"{name} n={n}: no {want} case clears the margin"
    save("tiny_beam.pt", dict(head_scale=HEAD_SCALE, margin_bound=MARGIN, cases=cases))


if __name__ == "__main__":
    main()
