"""CPU checks of the float64 optimizer restatement and its bounds (tests/optim_oracle64.py): replayed for 40 steps it
reproduces the fixture the unmodified reference wrote (tests/golden/optim_ref.pt); its bounds accept an fp32
emulation of the kernels' arithmetic and summation order, and reject that emulation with each of eight planted
mistakes by a wide margin.  Also: the kernels are built without fast-math, and vb_scaled_adam_step refuses a
zero-element tensor before it launches anything."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

import optim_oracle as R
import optim_oracle64 as O
from conftest import load_golden

HP = dict(lr=0.05, betas=(0.9, 0.95), eps=1e-8, scalar_lr_scale=0.1, param_min_rms=1e-5, param_max_rms=3.0,
          scalar_max=10.0, size_update_period=4, clipping_update_period=R.PERIOD, clipping_scale=2.0)
CLIP0 = dict(threshold=0.0, has_threshold=0, num_clipped=0, prev_clipped=0, scale=1.0, min_scale=1.0,
             prev_min_scale=1.0)


def _rel(a, b):
    return float((a.double() - b.double()).abs().max() / b.double().abs().max().clamp(min=1e-30))


def _x(v):
    return v.x.item() if isinstance(v, O.F) else v


# ---- the fixture replay -------------------------------------------------------------------------------------------------
class Replay:
    """ScaledAdam groups stepped by sadam_step64 alone, the state kept in fp32 between steps as the kernels keep it"""

    def __init__(self, params, groups, hp):
        self.params, self.hp = params, hp
        self.groups = []
        for names in groups:
            keys = sorted({(str(params[n].dtype), *params[n].shape) for n in names})
            batches = [[n for n in names if (str(params[n].dtype), *params[n].shape) == k] for k in keys]
            self.groups.append({"batches": batches, "states": None, "step": 0, "norms": None, "clip": dict(CLIP0)})

    def step(self, grads, lr):
        hp = dict(self.hp, lr=lr)
        scales = []
        for grp in self.groups:
            init = grp["states"] is None
            P = hp["clipping_update_period"]
            bs = []
            for i, names in enumerate(grp["batches"]):
                p = torch.stack([self.params[n] for n in names])
                g = torch.stack([torch.zeros_like(self.params[n]) if grads[n] is None else grads[n] for n in names])
                if init:
                    st = {"delta": torch.zeros_like(p), "exp_avg_sq": torch.zeros_like(p)}
                    if p.numel() > 1:
                        rs = (len(names),) + (1,) * (p.dim() - 1)
                        st.update(param_rms=torch.zeros(rs), scale_exp_avg_sq=torch.zeros(rs),
                                  scale_grads=torch.zeros(hp["size_update_period"], *rs))
                else:
                    st = grp["states"][i]
                bs.append((p, g, st))
            step = grp["step"]
            mode = O.clip_mode_of(step, P, hp["clipping_scale"], init, bool(grp["clip"]["has_threshold"]))
            if mode and grp["norms"] is None:
                grp["norms"] = torch.zeros(P)
            out = O.sadam_step64(bs, grp["norms"], grp["clip"], step, 0, init, mode, hp)
            new_states = []
            for i, (names, (p, g, st)) in enumerate(zip(grp["batches"], bs)):
                b = out["batches"][i]
                u = O.sadam_update64(out, i)
                n = len(names)
                ns = {"delta": u["delta"].x.float().view_as(p), "exp_avg_sq": u["exp_avg_sq"].x.float().view_as(p)}
                if "param_rms" in st:
                    rs = st["param_rms"].shape
                    ns["param_rms"] = b["param_rms"].x.float().view(rs)
                    ns["scale_exp_avg_sq"] = (b["scale_exp_avg_sq"].x.float().view(rs) if b.get("scale_exp_avg_sq")
                                              is not None else st["scale_exp_avg_sq"].clone())
                    sg = st["scale_grads"].clone()
                    if not b["scalar"]:
                        sg[out["slot"]] = b["scale_grads"].x.float().view(rs)
                    ns["scale_grads"] = sg
                new_states.append(ns)
                for k, nm in enumerate(names):
                    self.params[nm] = u["p"].x[k].float().view_as(p[k])
                assert n == p.shape[0]
            c = out["clip"]
            assert all(not isinstance(v, set) or len(v) == 1 for v in c.values()), "a clip decision inside its band"
            grp["clip"] = {k: (next(iter(v)) if isinstance(v, set) else _x(v)) for k, v in c.items()}
            if out["model_norms"] is not None:
                grp["norms"] = out["model_norms"].float()
            grp["states"], grp["step"] = new_states, step + 1
            scales.append(_x(out["scale"]))
        return scales


def _lr(s):
    return 0.05 if s == 1 else R.eden_lr(0.05, s - 1, 0, warmup_batches=200)


@pytest.mark.parametrize("two_groups", [False, True])
def test_replay_reproduces_the_reference_fixture(two_groups):
    gold = load_golden("optim_ref.pt")
    ref = gold["sadam2" if two_groups else "sadam"]
    params = {n: p.detach().clone() for n, p in R.make_params().items()}
    rp = Replay(params, R.groups_of(params, two_groups), HP)
    for s in range(1, R.STEPS + 1):
        scales = rp.step(R.make_grads(params, s), _lr(s))
        for x, y in zip(scales, ref["clip_scales"][s - 1]):
            assert abs(x - y) <= 1e-6 * y, (s, x, y)
        if not two_groups and s in ref["snap"]:
            for n, v in ref["snap"][s].items():
                assert _rel(rp.params[n], v) <= 1e-6, (s, n)
    for n, v in ref["params40"].items():
        assert _rel(rp.params[n], v) <= 1e-6, n
    assert [g["clip"]["num_clipped"] for g in rp.groups] == ref["num_clipped"]
    if two_groups:
        return
    names = list(params)
    grp = rp.groups[0]
    for names_b, st in zip(grp["batches"], grp["states"]):
        want = ref["sd40"]["state"][names.index(names_b[0])]
        assert want["step"] == grp["step"]
        for k, v in st.items():
            assert v.shape == want[k].shape and _rel(v, want[k]) <= 1e-6, (names_b[0], k)
        if "model_norms" in want:
            assert _rel(grp["norms"], want["model_norms"]) <= 1e-6
            assert abs(grp["clip"]["threshold"] - want["model_norm_threshold"]) <= 1e-6 * want["model_norm_threshold"]


def test_eve_replay_reproduces_the_reference_fixture():
    gold = load_golden("optim_ref.pt")["eve"]
    params = {n: p.detach().clone() for n, p in R.make_params().items()}
    hp = dict(lr=0.02, betas=(0.9, 0.98), eps=1e-8, weight_decay=1e-3, target_rms=0.1)
    state = {n: (0, torch.zeros_like(p), torch.zeros_like(p)) for n, p in params.items()}
    for s in range(1, R.STEPS + 1):
        for n, g in R.make_grads(params, s).items():
            if g is None:
                continue
            k, m, v = state[n]
            o = O.eve_step64(params[n], g, m, v, k + 1, hp)
            assert o["decay"] is not None
            params[n] = o["p"].x.float().view_as(g)
            state[n] = (k + 1, o["exp_avg"].x.float().view_as(g), o["exp_avg_sq"].x.float().view_as(g))
    for n, v in gold["params40"].items():
        assert _rel(params[n], v) <= 1e-6, n


# ---- an fp32 emulation of the kernels ---------------------------------------------------------------------------------
f32 = np.float32


def _fma(a, b, c):
    return (a.astype(np.float64) * b + c).astype(np.float32)


def _chunk_sum(a, b, mistake):
    """sadam_reduce_kernel's order for one chunk on the 16-byte path: 4 FMAs per thread per 1024 elements, the tail
    one element per thread, warp_sum's butterfly, then the 8 warp sums in order"""
    n = a.size
    n4 = n & ~3
    if mistake == "skip_last_group" and n4 >= 4:
        n4 -= 4
        a, b, n = a[:n4], b[:n4], n4
    v = np.zeros(O.THREADS, np.float32)
    if n4:
        pad = (-n4) % (4 * O.THREADS)
        A = np.concatenate([a[:n4], np.zeros(pad, np.float32)]).reshape(-1, O.THREADS, 4)
        B = np.concatenate([b[:n4], np.zeros(pad, np.float32)]).reshape(-1, O.THREADS, 4)
        for j in range(A.shape[0]):
            for e in range(4):
                v = _fma(A[j, :, e], B[j, :, e], v)
    for k in range(n4, n, O.THREADS):
        m = min(O.THREADS, n - k)
        v[:m] = _fma(a[k:k + m], b[k:k + m], v[:m])
    return _block_sum(v)


def _block_sum(v):
    w = v.reshape(-1, 32)
    lanes = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        w = (w + w[:, lanes ^ o]).astype(np.float32)
    s = f32(0)
    for k in range(w.shape[0]):
        s = f32(s + w[k, 0])
    return s


def _tensor_sum(a, b, mistake):
    chunks = range(0, a.size, O.CHUNK)
    if mistake == "skip_last_chunk" and len(chunks) > 1:
        chunks = chunks[:-1]
    s = f32(0)
    for c in chunks:
        s = f32(s + _chunk_sum(a[c:c + O.CHUNK], b[c:c + O.CHUNK], mistake))
    return s


def emulate_sadam32(batches, norms, clip, step, zero_step, init, mode, hp, mistake=None):
    """the kernels' fp32 step, op for op, with one planted mistake or none"""
    lr, (b1, b2), eps = hp["lr"], hp["betas"], hp["eps"]
    psz, size_lr = hp["size_update_period"], hp["lr"] * hp["scalar_lr_scale"]
    rows, terms = [], []
    for p, g, st in batches:
        n, per = p.shape[0], p[0].numel()
        P, G = p.reshape(n, per).numpy(), g.reshape(n, per).numpy()
        s = np.array([[_tensor_sum(G[i], G[i], mistake), _tensor_sum(P[i], G[i], mistake),
                       _tensor_sum(P[i], P[i], mistake)] for i in range(n)], np.float32)
        rms0 = None
        if "param_rms" in st:
            rms0 = np.sqrt(s[:, 2] / f32(per)) if init else st["param_rms"].reshape(n).numpy().copy()
        terms.append(s[:, 0] if per == 1 else s[:, 0] * (rms0 * rms0))
        rows.append((n, per, P, G, s, rms0))
    t = np.concatenate(terms).astype(np.float32)
    assert t.size <= O.COEF_THREADS
    tot = _block_sum(np.concatenate([t, np.zeros(O.COEF_THREADS - t.size, np.float32)]))
    norm = np.sqrt(tot)
    c, out = dict(clip), {"norm": norm, "sums": np.concatenate([r[4] for r in rows]), "batches": []}
    period = hp["clipping_update_period"] if mode else 1
    scale = f32(1)
    if mode >= 1:
        nn = norms.numpy().copy()
        nn[step % period] = norm
        out["model_norms"] = nn
        if step % period == 0:
            k = period // 2 if mistake == "median_p_half" else O.median_index(period)
            c.update(threshold=hp["clipping_scale"] * float(np.sort(nn)[k]), has_threshold=1)
        if mode == 2 and c["has_threshold"]:
            r = (f32(1) / (norm + f32(1e-20))) * f32(c["threshold"])
            scale = min(f32(1), r)
    out.update(scale=scale, threshold=c["threshold"])
    slot = step % psz
    b2c = b2 ** psz
    min_rms = f32(hp["param_min_rms"])
    bc2 = 1.0 - b2 ** (step - zero_step + 1)
    for (p, g, st), (n, per, P, G, s, rms0) in zip(batches, rows):
        o = {}
        D = st["delta"].reshape(n, per).numpy() * f32(b1)
        V = st["exp_avg_sq"].reshape(n, per).numpy() * f32(b2) + f32(1 - b2) * (G * G)
        if per > 1:
            sg_new = s[:, 1] if mistake == "sg_no_clip" else s[:, 1] * scale
            rms = np.sqrt(s[:, 2] / f32(per)) if slot == psz - 1 else rms0
            sstep = np.zeros(n, np.float32)
            if slot == psz - 1 and step > 0:
                sg = st["scale_grads"].reshape(psz, n).numpy().copy()
                sg[slot] = sg_new
                sq, sm = np.zeros(n, np.float32), np.zeros(n, np.float32)
                for k in range(psz):
                    sq, sm = sq + sg[k] * sg[k], sm + sg[k]
                seas = st["scale_exp_avg_sq"].reshape(n).numpy() * f32(b2c) + f32(1 - b2c) * (sq / f32(psz))
                coefs = f32(-size_lr * (1 - b2c ** ((step + 1) // psz)) ** 0.5)
                sstep = coefs * sm / (np.sqrt(seas) + f32(eps))
                sstep[rms < min_rms] = 0
                sstep[rms > f32(hp["param_max_rms"])] = f32(-size_lr * psz)
                o["scale_exp_avg_sq"] = seas
                if mistake != "no_size_step":
                    D = D + f32(1 - b1) * (P * sstep[:, None])
            alpha = f32(-lr * (1 - b1)) * np.maximum(rms, min_rms)
            VV = V * f32(1 / bc2) if bc2 < 0.99 else V
            D = D + (G / (np.sqrt(VV) + f32(eps))) * alpha[:, None]
            Pn = P + D
            if mistake == "rms_post_update" and slot == psz - 1:
                rms = np.sqrt((Pn.astype(np.float64) ** 2).mean(1)).astype(np.float32)
            o.update(scale_grads=sg_new, param_rms=rms, scale_step=sstep, alpha=alpha)
        else:
            k = step - zero_step if mistake == "zero_step_scalars" else step
            inv = f32(1) / f32(1.0 - b2 ** (k + 1))
            D = D + f32(-size_lr * (1 - b1)) * (G / (np.sqrt(V * inv) + f32(eps)))
            Pn = np.clip(P, f32(-hp["scalar_max"]), f32(hp["scalar_max"])) + D
        o.update(delta=D, exp_avg_sq=V, p=Pn)
        out["batches"].append(o)
    return out


def worst_ratios(emu, ref):
    """quantity -> the worst |emulated - float64| / bound"""
    r = {"sums": max(O.ratio(torch.from_numpy(emu["sums"][:, k].copy()), ref[q]) for k, q in
                     enumerate(("gg", "pg", "pp"))),
         "norm": O.ratio(torch.tensor(emu["norm"]), ref["norm"]),
         "scale": O.ratio(torch.tensor(emu["scale"]), ref["scale"])}
    if ref["threshold"] is not None:
        r["threshold"] = O.ratio(torch.tensor(emu["threshold"]), ref["threshold"])
    for i, (e, b) in enumerate(zip(emu["batches"], ref["batches"])):
        u = O.sadam_update64(ref, i)
        for k in ("scale_grads", "param_rms", "scale_exp_avg_sq", "scale_step", "alpha"):
            if k in e and b.get(k) is not None:
                r[k] = max(r.get(k, 0.0), O.ratio(torch.from_numpy(np.asarray(e[k])), b[k]))
        for k in ("delta", "exp_avg_sq", "p"):
            r[k] = max(r.get(k, 0.0), O.ratio(torch.from_numpy(e[k]), u[k]))
    return r


def _group(seed, clipped=False):
    """a small group: a batch of 3 scalars, a lone scalar, short tensors, tails, 2- and 4-chunk tensors, one tensor
    below param_min_rms and one above param_max_rms; state as after a few steps"""
    g = torch.Generator().manual_seed(seed)
    shapes = [((1,), 3), ((1, 1), 1), ((5,), 2), ((7, 3), 2), ((16385,), 1), ((3, 16384 + 1), 1), ((2, 24577), 1)]
    bs = []
    for shape, n in shapes:
        p = torch.randn((n, *shape), generator=g) * 0.3
        if shape == (5,):
            p[0] *= 1e-6    # rms ~3e-7 < param_min_rms
            p[1] *= 20.0    # rms ~6 > param_max_rms
        gr = torch.randn((n, *shape), generator=g) * (50.0 if clipped else 0.1)
        st = {"delta": torch.randn((n, *shape), generator=g) * 1e-3,
              "exp_avg_sq": torch.rand((n, *shape), generator=g) * 1e-2}
        if n * p[0].numel() > 1:
            rs = (n,) + (1,) * len(shape)
            st.update(param_rms=p.reshape(n, -1).pow(2).mean(1).sqrt().view(rs),
                      scale_exp_avg_sq=torch.rand(rs, generator=g) * 1e-2,
                      scale_grads=torch.randn((4, *rs), generator=g))
        bs.append((p, gr, st))
    return bs


CASES = {  # name: (step, zero_step, init, clip_mode, has_threshold, clipped)
    "init": (0, 0, True, 0, 0, False),
    "record": (1, 0, False, 1, 0, False),
    "size_update": (3, 0, False, 1, 0, False),
    "period_clipped": (24, 0, False, 2, 1, True),  # a period step at P = 8 and at P = 6
    "bias_corrected_zero_step": (91, 85, False, 2, 1, False),
    "no_bias_correction": (95, 0, False, 2, 1, True),
}


def _run(case, mistake=None, period=R.PERIOD):
    step, zero_step, init, mode, has_thr, clipped = CASES[case]
    bs = _group(step + 17, clipped)
    if init:
        for _, _, st in bs:
            st["delta"].zero_()
            st["exp_avg_sq"].zero_()
    hp = dict(HP, clipping_update_period=period)
    norms = torch.tensor([3.0, 1.0, 2.0, 2.0, 5.0, 4.0, 4.0, 0.5][:period] * (1 + period // 8))[:period]
    clip = dict(CLIP0, threshold=4.0 if has_thr else 0.0, has_threshold=has_thr)
    ref = O.sadam_step64(bs, norms, clip, step, zero_step, init, mode, hp)
    emu = emulate_sadam32(bs, norms, clip, step, zero_step, init, mode, hp, mistake)
    return worst_ratios(emu, ref)


@pytest.mark.parametrize("case", list(CASES))
def test_bounds_accept_the_fp32_emulation(case):
    r = _run(case)
    worst = max(r.items(), key=lambda kv: kv[1])
    print(case, {k: round(v, 3) for k, v in r.items()})
    assert worst[1] <= 1.0, (case, worst)


MISTAKES = {  # mistake: (case, period)
    "skip_last_chunk": ("record", R.PERIOD),
    "skip_last_group": ("record", R.PERIOD),
    "rms_post_update": ("size_update", R.PERIOD),
    "sg_no_clip": ("period_clipped", R.PERIOD),
    "median_p_half": ("period_clipped", 6),
    "zero_step_scalars": ("bias_corrected_zero_step", R.PERIOD),
    "no_size_step": ("size_update", R.PERIOD),
}


@pytest.mark.parametrize("mistake", list(MISTAKES))
def test_bounds_reject_planted_mistakes(mistake):
    case, period = MISTAKES[mistake]
    r = _run(case, mistake, period)
    worst = max(r.items(), key=lambda kv: kv[1])
    print(mistake, "worst error / bound", worst)
    assert worst[1] >= 10.0, (mistake, worst)


def test_bounds_reject_eve_decay_on_the_post_update_norm():
    g = torch.Generator().manual_seed(5)
    hp = dict(lr=0.02, betas=(0.9, 0.98), eps=1e-8, weight_decay=1e-3, target_rms=0.1)
    n = 4000
    q = torch.randn(n, generator=g)
    p = q / q.norm() * (0.1 * math.sqrt(n)) * (1 + 1e-3)  # ||p|| just above norm_limit
    grad = p.clone()                                       # the step shrinks every |p_i| by about lr
    m, v = torch.zeros(n), torch.zeros(n)
    right = O.eve_step64(p, grad, m, v, 1, hp)
    wrong = O.eve_step64(p, grad, m, v, 1, hp, post_update_norm=True)
    assert right["decay"] is True and wrong["decay"] is False
    r = O.ratio(wrong["p"].x.float(), right["p"])
    print("eve post-update norm: worst error / bound", r)
    assert r >= 10.0


def test_kernels_are_built_without_fast_math():
    from valle_b200 import build
    flags = " ".join(build.NVCC_FLAGS)
    for f in ("fast_math", "fast-math", "-ftz=true", "-prec-div=false", "-prec-sqrt=false"):
        assert f not in flags, f


def test_scaled_adam_step_refuses_an_empty_tensor_before_any_launch():
    from valle_b200 import _lib as L
    lib = L.load()
    chunk0 = (C.c_int32 * 4)(0, 1, 1, 2)  # tensor 1 has no chunks: no elements
    grads = (C.c_void_p * 3)()
    a = L.ScaledAdamArgs(n_tensors=3, n_chunks=2, step=1, size_period=4, lr=0.05, beta1=0.9, beta2=0.98, eps=1e-8,
                         scalar_lr_scale=0.1, param_min_rms=1e-5, param_max_rms=3.0, scalar_max=10.0)
    table = (C.c_uint8 * 64)()
    n0 = lib.vb_launch_count()
    # no workspace: should the empty-tensor check ever regress, the workspace check still refuses the call on the
    # host, so the host-memory table never reaches a kernel
    rc = lib.vb_scaled_adam_step(C.addressof(table), C.cast(grads, C.c_void_p), chunk0, C.byref(a), None, None,
                                 None, 0, None)
    assert rc != 0 and b"no elements" in lib.vb_last_error()
    assert lib.vb_launch_count() == n0
