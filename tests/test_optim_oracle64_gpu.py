"""The native ScaledAdam and Eve steps (csrc/optim.cu through valle.modules.optim) against the float64 restatement
of tests/optim_oracle64.py, one step at a time from a snapshot of the whole state, at the trainer's parameter table
and at the table's slice, chunk, alignment, clipping and magnitude edges.

Every step compares each output with the restatement run on the snapshot taken just before it: the per-tensor
coefficients (read from the step's workspace), model_norms and the clip state, scale_grads, param_rms,
scale_exp_avg_sq, delta, exp_avg_sq and p (the update p_after - p_before).  Each must lie within the bound the
restatement carries; decisions inside their band may go either way.  Every workspace is filled with NaN before a
step.  The worst error / bound of each quantity is printed at the end of the run."""
import collections
import math

import pytest
import torch

import optim_oracle64 as O

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
NAN = float("nan")
WORST = collections.defaultdict(float)


@pytest.fixture(autouse=True, scope="module")
def _report():
    yield
    print("\nworst error / bound:", {k: round(v, 3) for k, v in sorted(WORST.items())})


@pytest.fixture(autouse=True)
def _nan_workspaces(monkeypatch):
    from valle_b200.modules import optim
    init = optim._SadamPlan.__init__

    def nan_init(self, *a, **k):
        init(self, *a, **k)
        self.workspace.view(torch.float32).fill_(NAN)
    monkeypatch.setattr(optim._SadamPlan, "__init__", nan_init)


def _ok(name, r):
    WORST[name] = max(WORST[name], r)
    assert r <= 1.0, (name, r)


# ---- ScaledAdam ------------------------------------------------------------------------------------------------------
def _batches(opt, gi):
    from valle_b200.modules.optim import _sorted_batches
    return _sorted_batches(opt.param_groups[gi]["params"], opt.parameters_names[gi])


def _snapshot(opt, gi=0):
    group = opt.param_groups[gi]
    batches = _batches(opt, gi)
    states = [opt.state[ps[0]] for _, ps, _ in batches]
    init = len(states[0]) == 0
    bs = []
    for _, ps, _ in batches:
        p = torch.stack([q.detach() for q in ps])
        g = torch.stack([q.grad if q.grad is not None else torch.zeros_like(q) for q in ps])
        st = opt.state[ps[0]]
        if init:
            n = len(ps)
            c = {"delta": torch.zeros_like(p), "exp_avg_sq": torch.zeros_like(p)}
            if p.numel() > 1:
                rs = (n,) + (1,) * ps[0].dim()
                c.update(param_rms=torch.zeros(rs, device=DEV), scale_exp_avg_sq=torch.zeros(rs, device=DEV),
                         scale_grads=torch.zeros((group["size_update_period"], *rs), device=DEV))
        else:
            c = {k: v.clone() for k, v in st.items() if isinstance(v, torch.Tensor) and k != "model_norms"}
        bs.append((p, g, c))
    fs = states[0]
    step, zero_step = fs.get("step", 0), fs.get("zero_step", 0)
    if gi in opt._clip and gi not in opt._clip_stale:
        cs = opt._read_clip(opt._clip[gi])
        clip = {k: getattr(cs, k) for k, _ in cs._fields_}
    else:
        clip = dict(threshold=float(fs.get("model_norm_threshold", 0.0)), scale=1.0, min_scale=1.0,
                    prev_min_scale=1.0, num_clipped=int(fs.get("num_clipped", 0)), prev_clipped=0,
                    has_threshold=int("model_norm_threshold" in fs))
    P = group["clipping_update_period"]
    mode = O.clip_mode_of(step, P, group["clipping_scale"], init, "model_norm_threshold" in fs)
    norms = fs["model_norms"].clone() if "model_norms" in fs else (torch.zeros(P, device=DEV) if mode else None)
    hp = {k: group[k] for k in ("lr", "betas", "eps", "scalar_lr_scale", "param_min_rms", "param_max_rms",
                                "scalar_max", "size_update_period", "clipping_update_period", "clipping_scale")}
    return (bs, norms, clip, step, zero_step, init, mode, hp)


def _step_and_check(opt, gi=0):
    """one native step of group gi against sadam_step64 on the snapshot; returns (restatement, native outputs)"""
    plan = opt._plans.get(gi)
    if plan is not None:
        plan.workspace.view(torch.float32).fill_(NAN)
    snap = _snapshot(opt, gi)
    bs, norms0, clip0, step, _, init, mode, hp = snap
    opt.step()
    ref = O.sadam_step64(*snap)
    plan = opt._plans[gi]
    # the per-tensor coefficients: (alpha, scale_step) pairs after the partial sums in the workspace
    off = (plan.n_chunks * 3 * 4 + 255) // 256 * 256
    coef = plan.workspace[off:off + (2 * plan.n + 1) * 4].view(torch.float32)
    t = 0
    for b in ref["batches"]:
        n = b["n"]
        if not b["scalar"]:
            _ok("alpha", O.ratio(coef[2 * t:2 * (t + n):2], b["alpha"]))
            _ok("scale_step", O.ratio(coef[2 * t + 1:2 * (t + n):2], b["scale_step"]))
        else:
            assert bool((coef[2 * t:2 * (t + n)] == 0).all())
        t += n
    _ok("scale", O.ratio(coef[2 * t:2 * t + 1], ref["scale"]))
    # model_norms and the clip state
    batches = _batches(opt, gi)
    fs = opt.state[batches[0][1][0]]
    cs = opt._read_clip(opt._clip[gi])
    P = hp["clipping_update_period"]
    if mode >= 1:
        got = fs["model_norms"]
        slot = step % P
        _ok("model_norm", O.ratio(got[slot:slot + 1], ref["norm"]))
        others = torch.ones(P, dtype=torch.bool, device=DEV)
        others[slot] = False
        assert torch.equal(got[others], norms0[others])
        _ok("scale", O.ratio(torch.tensor([cs.scale]), ref["scale"]))
        c = ref["clip"]
        if ref["log_step"]:
            k = O.median_index(P)
            assert cs.threshold == hp["clipping_scale"] * float(got.sort()[0][k])
            _ok("threshold", O.ratio(torch.tensor([cs.threshold]), ref["threshold"]))
            assert cs.prev_clipped == clip0["num_clipped"] and cs.prev_min_scale == clip0["min_scale"]
            assert cs.has_threshold == 1
        assert cs.num_clipped in (c["num_clipped"] if isinstance(c["num_clipped"], set) else {c["num_clipped"]})
        before = 0 if ref["log_step"] else clip0["num_clipped"]
        assert cs.num_clipped - before == (1 if mode == 2 and cs.scale < 1.0 else 0)
        ms = c["min_scale"]
        if isinstance(ms, O.F):
            _ok("min_scale", O.ratio(torch.tensor([cs.min_scale]), ms))
        else:
            assert cs.min_scale == ms
    # the state and the parameters
    for i, ((_, ps, _), b) in enumerate(zip(batches, ref["batches"])):
        st = opt.state[ps[0]]
        n = b["n"]
        if not b["scalar"]:
            _ok("scale_grads", O.ratio(st["scale_grads"][ref["slot"]].reshape(n), b["scale_grads"]))
            if b.get("scale_exp_avg_sq") is not None:
                _ok("scale_exp_avg_sq", O.ratio(st["scale_exp_avg_sq"].reshape(n), b["scale_exp_avg_sq"]))
        if b.get("param_rms") is not None:
            _ok("param_rms", O.ratio(st["param_rms"].reshape(n), b["param_rms"]))
        u = O.sadam_update64(ref, i)
        _ok("delta", O.ratio(st["delta"], u["delta"]))
        _ok("exp_avg_sq", O.ratio(st["exp_avg_sq"], u["exp_avg_sq"]))
        pn = torch.stack([q.detach() for q in ps])
        _ok("update", O.ratio(pn.double() - bs[i][0].double(), u["update"]))
        del u
    return ref


def _set_step(opt, step, gi=0, zero_step=None):
    for _, ps, _ in _batches(opt, gi):
        opt.state[ps[0]]["step"] = step
        if zero_step is not None:
            opt.state[ps[0]]["zero_step"] = zero_step


def _sadam(params, names, **kw):
    from valle.modules.optim import ScaledAdam
    args = dict(lr=0.05, betas=(0.9, 0.95), clipping_scale=2.0, clipping_update_period=4,
                show_dominant_parameters=False)
    args.update(kw)
    return ScaledAdam(params, parameters_names=[names], **args)


@pytest.mark.parametrize("stage", [0, 1, 2])
def test_trainer_table(stage):
    """bench.build_model's parameters with real gradients: the init step, record-only steps, a size update, a period
    step, a clipped step (gradients x50), and steps 88 / 89 at beta2 = 0.95, where bias_correction2 < 0.99 flips
    (88: corrected, 89: not), then a size update at step 91 with zero_step = 85, which the non-scalar bias correction
    subtracts (corrected, where step 91 alone is not) and the scalars' does not."""
    from test_optim_gpu import _bench_model, _loss
    m = _bench_model()
    named = list(m.stage_named_parameters(stage)) if stage else list(m.named_parameters())
    names, params = [n for n, _ in named], [p for _, p in named]
    opt = _sadam(params, names)
    _loss(m, stage, stage).backward()
    grads = {p: None if p.grad is None else p.grad.clone() for p in params}
    for s, scale, jump in ((0, 1, None), (1, 1, None), (2, 1, None), (3, 1, None), (4, 1, None), (5, 50, None),
                           (88, 1, (88, None)), (89, 1, None), (91, 1, (91, 85))):
        if jump:
            _set_step(opt, jump[0], zero_step=jump[1])
        for p in params:
            if grads[p] is not None:
                p.grad = grads[p] * scale
        ref = _step_and_check(opt)
        if s == 5:
            assert ref["counted"] == {True}
        if s == 88:
            assert ref["bias_correct"]
        if s == 89:
            assert not ref["bias_correct"]
        if s == 91:
            assert ref["bias_correct"] and ref["size_update"] and 1.0 - 0.95 ** 92 >= 0.99
    del m, opt, params, grads
    torch.cuda.empty_cache()


def _slicing_layout():
    """> 2 x 1024 tensors in one group, sorted so that table indices 1023 / 1024 / 2047 / 2048 are multi-chunk"""
    return [((1,), 3), ((1, 1), 1), ((2,), 1019), ((2, 8193), 2), ((3,), 1021), ((3, 5461), 1), ((3, 5462), 2),
            ((5,), 40), ((5, 3277), 2), ((13, 3781), 1), ((16383,), 1), ((16384,), 2)]


def _make_params(layout, seed, offset=0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    params, names, bufs = [], [], []
    for shape, n in layout:
        for i in range(n):
            numel = math.prod(shape)
            buf = torch.empty(numel + offset, device=DEV)
            buf[offset:] = torch.randn(numel, device=DEV, generator=g) * 0.2
            params.append(torch.nn.Parameter(buf[offset:].view(shape)))
            names.append(f"{'x'.join(map(str, shape))}.{i}")
    return params, names


def test_slices_beyond_1024_tensors():
    layout = _slicing_layout()
    params, names = _make_params(layout, 1)
    T = len(params)
    assert T > 2048 and all(params[i].numel() > O.CHUNK for i in (1023, 1024, 2047, 2048))
    with torch.no_grad():
        params[2049].mul_(1e-6)   # a (5,) tensor below param_min_rms
        params[2050].mul_(30.0)   # one above param_max_rms
        params[0].fill_(-11.0)    # scalars beyond scalar_max: clamped before delta is added
        params[3].fill_(12.0)
    opt = _sadam(params, names, clipping_update_period=2)
    g = torch.Generator(device=DEV).manual_seed(2)
    for s in range(5):
        for i, p in enumerate(params):
            p.grad = None if i in (500, 1500, 2060) else torch.randn(p.shape, device=DEV, generator=g) * 0.1
        if s == 3:
            for p in params:
                if p.grad is not None:
                    p.grad.mul_(50)
        ref = _step_and_check(opt)
        if s == 3:
            assert ref["counted"] == {True} and ref["size_update"]
            # the planted tensors fall on both sides of the rms limits
            assert float(ref["batches"][7]["scale_step"].x[0]) == 0.0


def test_misaligned_parameters_and_gradients():
    """the same values with p and g placed 1, 2 and 3 floats into larger buffers, so every tensor takes the scalar
    fallback: each step within bound.  Step 1 starts every placement from the aligned run's state and refreshes no
    param_rms, so alpha is the same bits: exp_avg_sq and the scalars' update (the same instructions on both paths)
    must be bit-identical to the aligned run's; delta and p within the sum of both placements' bounds.  Those two
    differ in the last bit because nvcc contracts `d * beta1 + q * alpha` differently in the two loops: the 16-byte
    loop rounds d * beta1 and fuses q * alpha (FMUL, then FFMA q, alpha, d'), the fallback rounds q * alpha and fuses
    d * beta1 (FMUL, then FFMA d, beta1, q'), as `cuobjdump -sass` of sadam_update_kernel shows."""
    layout = [((1,), 2), ((5,), 3), ((7, 3), 2), ((16385,), 1), ((3, 16385), 1), ((49153,), 1)]
    start, outs = None, {}
    for off in (0, 1, 2, 3):
        params, names = _make_params(layout, 3, offset=off)
        assert off == 0 or all(p.data_ptr() % 16 for p in params)
        opt = _sadam(params, names)
        g = torch.Generator(device=DEV).manual_seed(4)
        gb = [torch.empty(p.numel() + off, device=DEV) for p in params]
        for s in range(2):
            for p, b in zip(params, gb):
                b[off:] = torch.randn(p.numel(), device=DEV, generator=g) * 0.1
                p.grad = b[off:].view(p.shape)
            if s == 1:
                if off == 0:
                    start = ([p.detach().clone() for p in params],
                             [{k: v.clone() for k, v in opt.state[ps[0]].items() if isinstance(v, torch.Tensor)}
                              for _, ps, _ in _batches(opt, 0)])
                with torch.no_grad():
                    for p, q in zip(params, start[0]):
                        p.copy_(q)
                for (_, ps, _), st in zip(_batches(opt, 0), start[1]):
                    for k, v in st.items():
                        opt.state[ps[0]][k].copy_(v)
            ref = _step_and_check(opt)
        outs[off] = []
        for i, (_, ps, _) in enumerate(_batches(opt, 0)):
            u = O.sadam_update64(ref, i)
            scalar = ref["batches"][i]["scalar"]
            outs[off] += [(torch.stack([q.detach() for q in ps]), u["p"].e, scalar),
                          (opt.state[ps[0]]["delta"].clone(), u["delta"].e, scalar),
                          (opt.state[ps[0]]["exp_avg_sq"].clone(), None, True)]
    for off in (1, 2, 3):
        for (a, ea, same), (b, eb, _) in zip(outs[0], outs[off]):
            if same:
                assert torch.equal(a, b), off
            else:
                diff = (a.double() - b.double()).abs().reshape(ea.shape)
                _ok("placements", float((diff / (ea + eb)).max()))


@pytest.mark.parametrize("P", [1, 2, 3, 5, 6, 8, 100])
def test_clipping_periods(P):
    """model_norms planted with exact ties; two periods: the period step's threshold, a clipped step, a step below
    the threshold, then the next period step's prev_clipped / prev_min_scale"""
    layout = [((1,), 2), ((5,), 3), ((64, 33), 2), ((20000,), 1)]
    params, names = _make_params(layout, 10 + P)
    opt = _sadam(params, names, clipping_update_period=P)
    g = torch.Generator(device=DEV).manual_seed(P)
    grads = [torch.randn(p.shape, device=DEV, generator=g) * 0.1 for p in params]
    for p, q in zip(params, grads):
        p.grad = q
    _step_and_check(opt)                          # init
    base = float(_step_and_check(opt)["norm"].x)  # step 1: record the norm (P = 1: a period step)
    fs = opt.state[_batches(opt, 0)[0][1][0]]
    planted = [base * x for x in (1.0, 1.0, 0.5, 2.0, 2.0, 0.5, 1.0, 3.0)]
    fs["model_norms"].copy_(torch.tensor((planted * (P // 8 + 1))[:P], device=DEV))
    for jump, scale in ((4 * P, 1.0), (None, 50.0), (None, 0.01), (8 * P, 1.0), (None, 50.0)):
        if jump is not None:
            _set_step(opt, jump)
        for p, q in zip(params, grads):
            p.grad = q * scale
        ref = _step_and_check(opt)
        if scale == 50.0 and P > 1:
            assert ref["counted"] == {True}


def test_magnitudes():
    """all-zero gradients, gradients near 1e-30 whose squares underflow in fp32, and a zero exp_avg_sq"""
    layout = [((1,), 2), ((5,), 3), ((7, 3), 2), ((16385,), 1)]
    params, names = _make_params(layout, 21)
    opt = _sadam(params, names, clipping_update_period=2)
    for s, gscale in enumerate((0.0, 1e-30, 0.0, 1e-30, 1e-30)):
        g = torch.Generator(device=DEV).manual_seed(s)
        for p in params:
            p.grad = torch.randn(p.shape, device=DEV, generator=g) * gscale
        if s == 4:
            for _, ps, _ in _batches(opt, 0):
                opt.state[ps[0]]["exp_avg_sq"].zero_()
        _step_and_check(opt)


def test_scaled_adam_refuses_a_zero_element_parameter_without_launching():
    from valle_b200 import _lib as L
    lib = L.load()
    params = [torch.nn.Parameter(torch.randn(4, 4, device=DEV)), torch.nn.Parameter(torch.zeros(0, 3, device=DEV))]
    for p in params:
        p.grad = torch.ones_like(p)
    opt = _sadam(params, ["w", "empty"])
    torch.cuda.synchronize()
    n0 = lib.vb_launch_count()
    with pytest.raises(L.VbError, match="empty"):
        opt.step()
    assert lib.vb_launch_count() == n0
    assert all(len(opt.state[p]) == 0 for p in params) and not opt._plans


# ---- Eve -------------------------------------------------------------------------------------------------------------
def test_eve_three_slices():
    """about 1,000 tensors (3 launches of each kernel), multi-chunk tensors at the 480 / 960 slice edges, numel-1
    tensors, ||p|| planted at norm_limit x (1 +- 1e-3), per-tensor step counts, misaligned placements and a
    zero-element parameter"""
    from valle.modules.optim import Eve
    g = torch.Generator(device=DEV).manual_seed(7)
    sizes = [3, 1, 5, 16, 17, 300] * 168
    sizes[479:481] = [16385, 3 * 16384 + 1]
    sizes[959:961] = [16384 * 2 + 3, 16385]
    sizes += [1, 2, 16383, 16384, 7] * 8
    # the empty parameter gets no table entry, so these are table indices: three slices of up to 480 tensors
    assert 960 < len(sizes) <= 3 * 480 and all(sizes[i] > O.CHUNK for i in (479, 480, 959, 960))
    hp = dict(lr=0.02, betas=(0.9, 0.98), eps=1e-8, weight_decay=1e-3, target_rms=0.1)
    params = []
    for i, n in enumerate(sizes):
        off = i % 4 if i % 7 == 0 else 0
        buf = torch.empty(n + off, device=DEV)
        buf[off:] = torch.randn(n, device=DEV, generator=g) * 0.12
        p = buf[off:]
        if n > 1 and i % 3 == 0:
            p.mul_(0.1 * n ** 0.5 * (1 + (1e-3 if i % 2 else -1e-3)) / p.norm())
        params.append(torch.nn.Parameter(p))
    empty = torch.nn.Parameter(torch.zeros(0, device=DEV))
    params.insert(700, empty)
    opt = Eve(params, **hp)
    ws_bytes = 4 * (sum(O.n_chunks(n) for n in sizes) + 64)
    opt._ws[torch.device(DEV)] = torch.full((ws_bytes // 4,), NAN, device=DEV).view(torch.uint8)
    for s in range(3):
        for i, p in enumerate(params):
            off = i % 4 if i % 5 == 0 else 0
            b = torch.empty(p.numel() + off, device=DEV)
            b[off:] = torch.randn(p.numel(), device=DEV, generator=g) * 0.1
            p.grad = b[off:].view(p.shape)
        if s == 1:  # per-tensor step counts, so step_size and bc2_rsqrt vary
            for i, p in enumerate(params):
                opt.state[p]["step"] = 1 + i % 13
        opt._ws[torch.device(DEV)].view(torch.float32).fill_(NAN)
        snap = [(p.detach().clone(), p.grad.clone(), opt.state[p].get("exp_avg"), opt.state[p].get("exp_avg_sq"),
                 opt.state[p].get("step", 0)) for p in params]
        snap = [(p0, g0, torch.zeros_like(p0) if m is None else m.clone(), torch.zeros_like(p0) if v is None
                 else v.clone(), k) for p0, g0, m, v, k in snap]
        opt.step()
        decided = 0
        for p, (p0, g0, m0, v0, k) in zip(params, snap):
            assert opt.state[p]["step"] == k + 1
            if p.numel() == 0:
                continue
            o = O.eve_step64(p0, g0, m0, v0, k + 1, hp)
            decided += o["decay"] is not None
            _ok("eve_exp_avg", O.ratio(opt.state[p]["exp_avg"], o["exp_avg"]))
            _ok("eve_exp_avg_sq", O.ratio(opt.state[p]["exp_avg_sq"], o["exp_avg_sq"]))
            _ok("eve_update", O.ratio(p.detach().double() - p0.double(), o["update"]))
        assert decided == len(sizes)  # the planted norms lie outside their bands
    # the zero-element parameter keeps its (empty) state and counts its steps like the others (checked above)
    assert opt.state[empty]["exp_avg"].numel() == 0 and opt.state[empty]["exp_avg_sq"].numel() == 0
