"""Generate tests/golden/prenet_train.pt: VALLE.forward + loss.backward() of the UNMODIFIED reference (through
oracle/ref_loader.py) with add_prenet=True, in train() mode with every dropout at 0, on the CPU in fp32.  Needs the
reference checkout; the fixture travels, the reference does not.

    python tools/gen_golden_prenet_train.py

For train_stage 0 / 1 / 2 of each configuration it records the loss, the BatchNorm buffers after the call and, per
parameter with a gradient, the gradient's max-abs, its L2 norm and its values at the positions of
`prenet_oracle.sample_positions` (whole gradients would be tens of MB).  Before writing, the prefix-mode 0 / 1 configurations are
checked against the oracle restatement (tests/prenet_oracle.py) on every element of every gradient.
"""
from __future__ import annotations

import contextlib
import copy
import os
import random
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import torch  # noqa: E402

import postln_oracle as P  # noqa: E402
import prenet_oracle as PN  # noqa: E402
from oracle import gen_golden as G  # noqa: E402
from oracle import valle_oracle as O  # noqa: E402
from oracle.ref_loader import load_reference  # noqa: E402

TORCH_SEED = 5
# smallest |input| of a pre-net ReLU the fixture accepts: closer to 0, fp32 rounding may flip the gate and move a
# gradient by a whole row's contribution
RELU_MARGIN = 5e-6
# name, d, heads, layers, norm_first, prefix_mode, prepend_bos, nar_scale_factor
CONFIGS = [
    ("preln_pm1", 256, 4, 2, True, 1, False, 1.0),
    ("postln_pm0", 256, 4, 2, False, 0, False, 1.0),
    ("postln_pm2", 256, 4, 2, False, 2, False, 1.0),
    ("postln_pm4", 256, 4, 2, False, 4, False, 1.0),
    ("preln_bos", 256, 4, 2, True, 1, True, 1.0),
    ("postln_scale", 512, 8, 2, False, 1, False, 0.5),
]


def batch(pm: int, seed: int = 31):
    """3 padded utterances (the batch of tools/gen_golden_postln.py); prefix mode 4 also gets 10 prompt frames"""
    g = torch.Generator().manual_seed(seed)
    x = torch.randint(3, 100, (3, 12), generator=g)
    x_lens = torch.tensor([12, 9, 7], dtype=torch.int32)
    y = torch.randint(0, 1024, (3, 40, 8), generator=g)
    y_lens = torch.tensor([40, 31, 22], dtype=torch.int32)
    prompts = torch.randint(0, 1024, (3, 10, 8), generator=g) if pm == 4 else None
    return x, x_lens, y, y_lens, prompts


def no_dropout(m):
    for mod in m.modules():
        if isinstance(mod, torch.nn.Dropout):
            mod.p = 0.0
        if isinstance(getattr(mod, "dropout", None), float):   # MultiheadAttention's attention-probability dropout
            mod.dropout = 0.0
    return m


def run(ref, m0, pm, stage, seed):
    """one reference training call on a copy of m0: (loss, buffers after, {name: grad}, smallest |input| of a pre-net
    ReLU)"""
    m = copy.deepcopy(m0)
    margin = [float("inf")]

    def hook(mod, inp, out):
        margin[0] = min(margin[0], float(out.detach().abs().min()))

    for n, mod in m.named_modules():   # BatchNorm1d outputs and the audio pre-nets' first two Linear outputs
        if isinstance(mod, torch.nn.BatchNorm1d) or (("audio_prenet.0" in n or "audio_prenet.3" in n)
                                                     and isinstance(mod, torch.nn.Linear)):
            mod.register_forward_hook(hook)
    x, xl, y, yl, prompts = batch(pm, seed)
    if pm == 4:
        y, yl = ref.PromptedFeatures(prompts, y), ref.PromptedFeatures(torch.full((3,), 10, dtype=torch.int32), yl)
    m.rng = random.Random(0)
    torch.manual_seed(TORCH_SEED)
    (_, _), loss, _ = m(x, xl, y, yl, train_stage=stage)
    loss.backward()
    bufs = {k: v.detach().clone() for k, v in m.named_buffers()}
    grads = {n: p.grad.detach().clone() for n, p in m.named_parameters() if p.grad is not None}
    return float(loss.detach()), bufs, grads, margin[0]


def check_oracle(m0, cfg, stage, post_ln, loss, bufs, grads, seed):
    """the oracle restatement against the reference, every gradient element"""
    x, xl, y, yl, _ = batch(cfg.prefix_mode, seed)
    nar_stage = random.Random(0).choices(list(range(1, 8)), weights=[1 / 7] * 7, k=1)[0]
    torch.manual_seed(TORCH_SEED)
    int_low = (0.25 * yl.min()).type(torch.int64).item()
    prefix_len = min(torch.randint(int_low, int_low * 2, size=()).item(), 225)
    sd = {k: v.detach().clone().requires_grad_(v.is_floating_point()) for k, v in m0.state_dict().items()}
    with P.post_ln() if post_ln else contextlib.nullcontext():
        lo, _, ob = PN.forward_train(sd, cfg, x, xl, y, yl, nar_stage, prefix_len, train_stage=stage)
    lo.backward()
    assert abs(float(lo.detach()) - loss) <= 1e-5 * abs(loss), (float(lo.detach()), loss)
    for k, v in bufs.items():
        assert torch.allclose(ob[k].float(), v.float(), rtol=0, atol=1e-6 * max(1.0, float(v.abs().max()))), k
    by_ptr = {}
    for k, v in m0.state_dict().items():
        by_ptr.setdefault(v.data_ptr(), []).append(k)
    for n, p in m0.named_parameters():
        want = sum(sd[k].grad for k in by_ptr[p.data_ptr()] if sd[k].grad is not None)
        got = grads.get(n)
        if not p.requires_grad:   # the NAR positional alphas (alpha=False) are frozen
            continue
        if got is None:
            assert not torch.is_tensor(want) or float(want.abs().max()) == 0.0, n
            continue
        err = float((want - got).abs().max()) / max(float(got.abs().max()), 1e-30)
        assert err < 1e-4 or float(got.abs().max()) < 1e-6, (n, err)


def main():
    ref = load_reference()
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    out = {"samples": PN.SAMPLES, "torch_seed": TORCH_SEED, "configs": {}}
    for name, d, h, l, nf, pm, bos, scale in CONFIGS:
        torch.manual_seed(0)
        m0 = ref.VALLE(d, h, l, norm_first=nf, add_prenet=True, prefix_mode=pm, share_embedding=True,
                       nar_scale_factor=scale, prepend_bos=bos, num_quantizers=8)
        m0 = no_dropout(m0.train())
        # the first batch seed from 31 whose pre-net ReLU inputs keep RELU_MARGIN from 0 in every stage
        seed = next(sd for sd in range(31, 131) if all(run(ref, m0, pm, st, sd)[3] >= RELU_MARGIN for st in (0, 1, 2)))
        x, xl, y, yl, prompts = batch(pm, seed)
        ck = G.checksums(m0.state_dict())
        rec = dict(config=dict(d_model=d, nhead=h, num_layers=l, norm_first=nf, prefix_mode=pm, prepend_bos=bos,
                               nar_scale_factor=scale, num_quantizers=8, add_prenet=True),
                   weight_seed=0, checksum_keys=list(ck), checksums=torch.stack(list(ck.values())), x=x, x_lens=xl, y=y.to(torch.int16),
                   y_lens=yl, batch_seed=seed, prompts=None if prompts is None else prompts.to(torch.int16), stages={})
        for stage in (0, 1, 2):
            loss, bufs, grads, _ = run(ref, m0, pm, stage, seed)
            if pm in (0, 1) and not bos and scale == 1.0:
                check_oracle(m0, O.OracleConfig(d, h, l, pm, 8), stage, not nf, loss, bufs, grads, seed)
            names = sorted(grads)
            g = dict(names=names, max_abs=torch.tensor([float(grads[n].abs().max()) for n in names]),
                     l2=torch.tensor([float(grads[n].norm()) for n in names]),
                     values=torch.stack([grads[n].reshape(-1)[PN.sample_positions(n, grads[n].numel())] for n in names]))
            # the statistics of the pre-nets this stage ran (the others keep their initial 0 / 1 / 0)
            bn = [k[:-len(".num_batches_tracked")] for k, v in bufs.items() if k.endswith("num_batches_tracked") and v > 0]
            rec["stages"][stage] = dict(loss=loss, buffer_keys=bn, num_batches_tracked=[int(bufs[k + ".num_batches_tracked"]) for k in bn],
                                        running_mean=torch.cat([bufs[k + ".running_mean"] for k in bn]),
                                        running_var=torch.cat([bufs[k + ".running_var"] for k in bn]), grads=g)
            print(f"{name} (batch seed {seed}) stage {stage}: loss {loss:.6f}, {len(names)} gradients, {len(bn)} BatchNorms")
        out["configs"][name] = rec
    G.save("prenet_train.pt", out)


if __name__ == "__main__":
    main()
