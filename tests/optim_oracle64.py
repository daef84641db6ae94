"""Float64 restatement of one ScaledAdam step and one Eve step from a given state, with the error bounds of the fp32
kernels in csrc/optim.cu (test infrastructure, like stack_oracle64.py).

Every computed quantity is an `F`: its float64 value x and a bound e on |fp32 kernel result - x|.  The bound grows
op by op as the kernels round, with u = 2^-24 and t = 2^-150 (the largest rounding error in fp32's subnormal range,
so that g * g underflowing for |g| < 1e-19 stays inside the bound):

    a + b    e_a + e_b + u|x| + t
    a * b    |a| e_b + |b| e_a + e_a e_b + u|x| + t
    a / b    (e_a + |x| e_b) / (|b| - e_b) + u|x| + t
    sqrt a   min(e_a / sqrt(a), sqrt(e_a)) + u sqrt(a) + t
    min/max  the larger of the operands' e (both are 1-Lipschitz)

`sqrtf` and `/` are IEEE in these kernels: build.py passes no fast-math flag (tests/test_optim_oracle64.py checks
that).  nvcc contracts a * b + c into one FMA, which only removes a rounding, so every bound holds for it too.

Coefficients the host rounds from double to fp32 once (`alpha_coef`, `size_coef`, `beta2_corr`, `inv_bc2`,
`scalar_alpha`, `max_fill`, Eve's `step_size`, `bc2_rsqrt`, `norm_limit`, ...) enter as their exact double with
e = u|c| (`coef`); `inv_bc2_s` is rounded twice (2u).  The restatement itself uses the exact doubles, so a wrong host
formula moves x, not e, and fails the comparison.

Sums (`sum_bound`) are γ_n Σ|terms| + 2 N t, γ_n = n u / (1 - n u), where n is the depth of the kernel's longest
addition chain and N the number of terms:
  * a chunk's sum (sadam_reduce_kernel, eve_reduce_kernel): 16384 / 256 = 64 FMAs per thread, 5 shuffle levels of
    `warp_sum` and 7 serial additions of the 8 warp sums (`block_sum`): 76;
  * a tensor's sum: its chunks added in order by one thread of sadam_coef_kernel (or eve_update_kernel): + n_chunks - 1;
  * tot_sumsq: ceil(T / 1024) terms per thread of sadam_coef_kernel, 5 shuffle levels and 31 serial additions of the
    32 warp sums; each term carries its own e from the tensor's Σg² and param_rms.

Discrete decisions (param_rms < param_min_rms, param_rms > param_max_rms, the clip scale below 1, Eve's
||p|| > norm_limit) are taken from x where x lies outside its band (the e of both sides); inside the band either
outcome is accepted, and the bound of everything downstream widens to cover both (`pick`).
"""
from __future__ import annotations

import torch

U = 2.0 ** -24
TINY = 2.0 ** -150
CHUNK = 16384          # VB_OPTIM_CHUNK
THREADS = 256          # OPT_THREADS
COEF_THREADS = 1024    # sadam_coef_kernel's CTA
CHUNK_DEPTH = CHUNK // THREADS + 5 + (THREADS // 32 - 1)


def gamma(n):
    return n * U / (1.0 - n * U)


def n_chunks(numel):
    return (numel + CHUNK - 1) // CHUNK


def tensor_depth(numel):
    """the longest addition chain of a tensor's sum: a chunk's 76, then its chunks added in order"""
    return CHUNK_DEPTH + n_chunks(numel) - 1


def tot_depth(n_tensors):
    return -(-n_tensors // COEF_THREADS) + 5 + (COEF_THREADS // 32 - 1)


def sum_bound(abs_sum, depth, n_terms):
    return gamma(depth) * abs_sum + 2 * n_terms * TINY


def _t(v):
    if isinstance(v, torch.Tensor):
        return v.double()
    return torch.tensor(float(v), dtype=torch.float64)


def _rnd(x):
    return U * x.abs() + TINY


class F:
    """x: the float64 value; e: a bound on |fp32 result - x| (see the module docstring)"""
    __slots__ = ("x", "e")

    def __init__(self, x, e=0.0):
        self.x = _t(x)
        self.e = _t(e) if not isinstance(e, torch.Tensor) else e.double()

    @staticmethod
    def of(v):
        return v if isinstance(v, F) else F(v)

    def __add__(a, b):
        b = F.of(b)
        x = a.x + b.x
        return F(x, a.e + b.e + _rnd(x))

    __radd__ = __add__

    def __neg__(a):
        return F(-a.x, a.e)

    def __sub__(a, b):
        return a + (-F.of(b))

    def __mul__(a, b):
        b = F.of(b)
        x = a.x * b.x
        return F(x, a.x.abs() * b.e + b.x.abs() * a.e + a.e * b.e + _rnd(x))

    __rmul__ = __mul__

    def __truediv__(a, b):
        b = F.of(b)
        x = a.x / b.x
        den = b.x.abs() - b.e
        assert bool((den > 0).all()), "a divisor's bound reaches 0"
        return F(x, (a.e + x.abs() * b.e) / den + _rnd(x))

    def __rtruediv__(a, b):
        return F.of(b) / a

    def sqrt(a):
        x = a.x.clamp(min=0).sqrt()
        prop = torch.where(x > 0, a.e / torch.where(x > 0, x, torch.ones_like(x)), a.e.sqrt())
        return F(x, torch.minimum(prop, a.e.sqrt()) + _rnd(x))

    def view(self, *shape):
        return F(self.x.reshape(*shape) if self.x.dim() else self.x,
                 self.e.reshape(*shape) if self.e.dim() else self.e)

    def __getitem__(self, i):
        return F(self.x[i], self.e[i] if self.e.dim() else self.e)


def coef(exact, roundings=1):
    """a host coefficient: the exact double, rounded to fp32 `roundings` times"""
    return F(exact, roundings * U * abs(exact))


def fmax(a, b):
    a, b = F.of(a), F.of(b)
    return F(torch.maximum(a.x, b.x), torch.maximum(a.e, b.e))


def exact_sum(terms, depth, dim=-1):
    """the sum of exact float64 products of fp32 values (Σg², Σp·g, Σp²) and its bound"""
    n = terms.shape[dim]
    return F(terms.sum(dim), sum_bound(terms.abs().sum(dim), depth, n))


def compare(a, b):
    """a, b: two F's.  Returns (decision of x, ambiguous): ambiguous where |a - b| <= e_a + e_b."""
    a, b = F.of(a), F.of(b)
    return a.x > b.x, (a.x - b.x).abs() <= a.e + b.e


def pick(cond, ambiguous, yes, no):
    """where(cond, yes, no); where the decision is ambiguous either outcome is accepted downstream"""
    yes, no = F.of(yes), F.of(no)
    x = torch.where(cond, yes.x, no.x)
    e = torch.where(cond, yes.e + 0 * x, no.e + 0 * x)
    both = torch.maximum(yes.e, no.e) + (yes.x - no.x).abs()
    return F(x, torch.where(ambiguous, both + 0 * x, e))


# ---- ScaledAdam -------------------------------------------------------------------------------------------------------
def clip_mode_of(step, period, clipping_scale, first_state_empty, has_threshold_key):
    """the reference's clipping decision of a step (optim.py:242-247, 342-412): 0 none, 1 record the norm, 2 clip"""
    if first_state_empty or clipping_scale is None or step == 0:
        return 0
    if step < period:
        return 1
    if not has_threshold_key and step % period != 0:
        return 1
    return 2


def median_index(period):
    return min(period - 1, (period // 4) * 2)


def sadam_step64(batches, model_norms, clip, step, zero_step, init, clip_mode, hp, median_at=median_index):
    """One ScaledAdam step of a parameter group in float64, every intermediate returned.

    batches: [(p, g, state)] in the reference's batch order (sorted (dtype, *shape) keys); p, g: [n, *shape] (g is
      zero where a gradient is None); state: the batch's stacked state before the step (delta, exp_avg_sq and, when
      n * numel > 1, param_rms, scale_exp_avg_sq, scale_grads); with init, delta / exp_avg_sq are zeros and
      param_rms is set here from p.
    model_norms: [P] before the step (None without clipping); clip: the vb_clip_state fields before the step.
    hp: the group's hyperparameters as Python floats (lr, betas, eps, scalar_lr_scale, param_min_rms,
      param_max_rms, scalar_max, size_update_period, clipping_update_period, clipping_scale).
    median_at: the sorted index of the median (a parameter so the CPU test can plant the wrong one).

    Returns a dict; the per-batch element-wise update is computed by `sadam_update64(out, i)`."""
    lr, (beta1, beta2), eps = hp["lr"], hp["betas"], hp["eps"]
    psz = hp["size_update_period"]
    size_lr = lr * hp["scalar_lr_scale"]
    out = {"batches": []}
    per_batch = []
    tot_terms = []
    for p, g, st in batches:
        n = p.shape[0]
        per = p[0].numel()
        P2, G2 = p.reshape(n, per).double(), g.reshape(n, per).double()
        d = tensor_depth(per)
        gg, pg, pp = exact_sum(G2 * G2, d), exact_sum(P2 * G2, d), exact_sum(P2 * P2, d)
        rms0 = None
        if "param_rms" in st:
            rms0 = (pp / F(per)).sqrt() if init else F(st["param_rms"].reshape(n).double())
        scalar = per == 1
        term = gg if scalar else gg * (rms0 * rms0)
        tot_terms.append(term)
        per_batch.append((n, per, P2, G2, gg, pg, pp, rms0, scalar))
    T = sum(b[0] for b in per_batch)
    allx = torch.cat([t.x.reshape(-1) for t in tot_terms])
    alle = torch.cat([(t.e + 0 * t.x).reshape(-1) for t in tot_terms])
    tot = F(allx.sum(), alle.sum() + sum_bound((allx.abs() + alle).sum(), tot_depth(T), T))
    norm = tot.sqrt()
    out.update(gg=_cat([b[4] for b in per_batch]), pg=_cat([b[5] for b in per_batch]),
               pp=_cat([b[6] for b in per_batch]), tot=tot, norm=norm, n_tensors=T)

    # the model norm and the clip scale (optim.py:342-412)
    c = dict(clip)
    period = hp["clipping_update_period"] if clip_mode else 1
    log_step = clip_mode >= 1 and step % period == 0
    norms = None
    if clip_mode >= 1:
        norms = model_norms.double().clone()
        norms[step % period] = norm.x.to(norms.device)
    threshold = None
    if log_step:
        med = float(norms.sort()[0][median_at(period)])
        # the k-th order statistic is 1-Lipschitz in the largest element error: only the new slot carries one
        threshold = F(hp["clipping_scale"] * med, hp["clipping_scale"] * float(norm.e))
        c.update(threshold=threshold.x.item(), has_threshold=1, prev_clipped=c["num_clipped"], num_clipped=0,
                 prev_min_scale=c["min_scale"], min_scale=1.0)
    scale = F(1.0)
    counted = {False}
    if clip_mode == 2 and c["has_threshold"]:
        thr = threshold if threshold is not None else F(c["threshold"])
        r = (1.0 / (norm + F(1.0e-20))) * F(thr.x, thr.e + _rnd(thr.x))  # (float) threshold
        below, amb = compare(F(1.0), r)
        scale = F(torch.minimum(r.x, torch.ones_like(r.x)), r.e)
        counted = {True, False} if bool(amb) else {bool(below)}
        ms = F(min(c["min_scale"], float(scale.x)), float(scale.e) + (abs(1.0 - float(r.x)) if bool(amb) else 0.0))
        c["min_scale"] = ms if True in counted else F(c["min_scale"])
        c["num_clipped"] = {c["num_clipped"] + int(k) for k in counted}
    if clip_mode >= 1:
        c["scale"] = scale
    out.update(model_norms=norms, threshold=threshold, scale=scale, counted=counted, clip=c, log_step=log_step)

    # scale_grads, param_rms, the size update (optim.py:504-596) and the per-tensor coefficients
    slot = step % psz
    refresh = slot == psz - 1
    size_update = refresh and step > 0
    b2c = beta2 ** psz
    size_bc2 = 1.0 - b2c ** ((step + 1) // psz)
    min_rms, max_rms = coef(hp["param_min_rms"]), coef(hp["param_max_rms"])
    for (p, g, st), (n, per, P2, G2, gg, pg, pp, rms0, scalar) in zip(batches, per_batch):
        b = {"n": n, "per": per, "scalar": scalar, "p0": p, "g": g, "state": st, "rms0": rms0}
        if not scalar:
            sg_new = pg * scale
            rms = (pp / F(per)).sqrt() if refresh else rms0
            sstep = F(0.0)
            seas = None
            if size_update:
                sg = st["scale_grads"].reshape(psz, n).double()
                sq, sm = F(0.0), F(0.0)
                for k in range(psz):
                    x = sg_new if k == slot else F(sg[k])
                    sq = sq + x * x
                    sm = sm + x
                seas = F(st["scale_exp_avg_sq"].reshape(n).double()) * coef(b2c) + coef(1.0 - b2c) * (sq / F(psz))
                sstep = coef(-size_lr * size_bc2 ** 0.5) * sm / (seas.sqrt() + coef(hp["eps"]))
                small, amb = compare(min_rms, rms)
                sstep = pick(small, amb, F(0.0), sstep)
                large, amb = compare(rms, max_rms)
                sstep = pick(large, amb, coef(-size_lr * psz), sstep)
            alpha = coef(-lr * (1.0 - beta1)) * fmax(rms, min_rms)
            b.update(scale_grads=sg_new, param_rms=rms, scale_exp_avg_sq=seas, scale_step=sstep, alpha=alpha)
        elif rms0 is not None:
            b.update(param_rms=rms0)
        out["batches"].append(b)
    bc2 = 1.0 - beta2 ** (step - zero_step + 1)
    out.update(slot=slot, refresh=refresh, size_update=size_update, bias_correct=bc2 < 0.99, inv_bc2=1.0 / bc2,
               inv_bc2_s=1.0 / (1.0 - beta2 ** (step + 1)), hp=hp)
    return out


def _cat(fs):
    return F(torch.cat([f.x.reshape(-1) for f in fs]), torch.cat([(f.e + 0 * f.x).reshape(-1) for f in fs]))


def sadam_update64(out, i, scalar_bc_step=None):
    """The element-wise update of batch i of `out` (optim.py:598-661): the new delta, exp_avg_sq and p, and the
    update p_after - p_before, each an F of the batch's stacked shape [n, numel]."""
    b, hp = out["batches"][i], out["hp"]
    beta1, beta2 = hp["betas"]
    n, per = b["n"], b["per"]
    st = b["state"]
    P0 = F(b["p0"].reshape(n, per).double())
    G = F(b["g"].reshape(n, per).double())
    d = F(st["delta"].reshape(n, per).double()) * coef(beta1)
    v = F(st["exp_avg_sq"].reshape(n, per).double()) * coef(beta2) + coef(1.0 - beta2) * (G * G)
    eps = coef(hp["eps"])
    if not b["scalar"]:
        if out["size_update"]:
            d = d + coef(1.0 - beta1) * (P0 * b["scale_step"].view(n, 1))
        vv = v * coef(out["inv_bc2"]) if out["bias_correct"] else v
        d = d + (G / (vv.sqrt() + eps)) * b["alpha"].view(n, 1)
        p = P0 + d
    else:
        size_lr = hp["lr"] * hp["scalar_lr_scale"]
        d = d + coef(-size_lr * (1.0 - beta1)) * (G / ((v * coef(out["inv_bc2_s"], 2)).sqrt() + eps))
        smax = hp["scalar_max"]
        clamped = P0.x.abs() > smax
        p = F(P0.x.clamp(-smax, smax), torch.where(clamped, U * smax, 0.0)) + d
    return {"delta": d, "exp_avg_sq": v, "p": p, "update": F(p.x - P0.x, p.e)}


# ---- Eve --------------------------------------------------------------------------------------------------------------
def eve_step64(p, g, m, v, step, hp, post_update_norm=False):
    """One Eve step of one tensor (optim.py:836-985) in float64; `step` is the state's step after the increment.
    Returns ||p|| before the update, the decay decision (None when inside its band; numel <= 1 never decays), and
    the new m, v, p and the update, as F's.  post_update_norm plants a mistake for the CPU test."""
    lr, (beta1, beta2), eps, wd = hp["lr"], hp["betas"], hp["eps"], hp["weight_decay"]
    n = p.numel()
    P0, G = F(p.reshape(-1).double()), F(g.reshape(-1).double())
    # the kernel's beta1, beta2, eps, weight_decay arrive as fp32; 1 - beta and 1 - weight_decay are formed in fp32
    b1, b2 = F(beta1, U * beta1), F(beta2, U * beta2)
    omb1, omb2 = F(1.0 - beta1, U), F(1.0 - beta2, U)
    M = F(m.reshape(-1).double()) * b1 + omb1 * G
    V = F(v.reshape(-1).double()) * b2 + omb2 * (G * G)
    bc1, bc2 = 1.0 - beta1 ** step, 1.0 - beta2 ** step
    den = V.sqrt() * coef(bc2 ** -0.5) + F(eps, U * eps)
    upd = coef(-lr / bc1) * (M / den)
    norm = exact_sum(P0.x * P0.x, tensor_depth(n)).sqrt()
    decay, mult = False, F(1.0)
    if n > 1:
        limit = coef(hp["target_rms"] * n ** 0.5)
        if post_update_norm:
            norm = F((P0.x + upd.x).norm(), norm.e)
        above, amb = compare(norm, limit)
        decay = None if bool(amb) else bool(above)
        mult = pick(above, amb, F(1.0 - wd, U), F(1.0))
    pn = P0 * mult + upd
    return {"norm": norm, "decay": decay, "exp_avg": M, "exp_avg_sq": V, "p": pn, "update": F(pn.x - P0.x, pn.e)}


def ratio(got, f):
    """the worst |got - x| / e of an F (got: the kernel's fp32 values, any shape that reshapes to f's)"""
    x = f.x.reshape(-1)
    g = got.double().reshape(-1).to(x.device)
    e = (f.e + 0 * f.x).reshape(-1)
    err = (g - x).abs()
    assert bool(torch.isfinite(g).all()), "non-finite output"
    return float((err / e.clamp(min=1e-300)).max()) if err.numel() else 0.0
