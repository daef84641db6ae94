"""Plain-torch restatement of the trainer's optimizers (valle/modules/optim.py:29-985) and schedulers
(valle/modules/scheduler.py:24-78), test infrastructure only.

It follows the reference's op order, stacking included: every step stacks each (dtype, *shape) batch of parameters and
gradients, runs the batch's update on the stacks and copies the parameters back.  It runs on any device, so it is
the pinned baseline on the GPU, where the reference itself is not available, and the baseline tools/bench_optim.py
times.  tests/test_optim.py checks it against the fixture the unmodified reference wrote (tests/golden/optim_ref.pt).
"""
from __future__ import annotations

from collections import defaultdict

import torch
from torch.optim import Optimizer


def _batches(params):
    groups = defaultdict(list)
    for p in params:
        groups[(str(p.dtype), *p.shape)].append(p)
    return [groups[k] for k in sorted(groups)]


class ScaledAdamOracle(Optimizer):
    """ScaledAdam with the reference's defaults, state layout and clipping; no logging."""

    def __init__(self, params, lr=3e-02, clipping_scale=None, betas=(0.9, 0.98), scalar_lr_scale=0.1, eps=1.0e-08,
                 param_min_rms=1.0e-05, param_max_rms=3.0, scalar_max=10.0, size_update_period=4,
                 clipping_update_period=100):
        super().__init__(params, dict(lr=lr, clipping_scale=clipping_scale, betas=betas,
                                      scalar_lr_scale=scalar_lr_scale, eps=eps, param_min_rms=param_min_rms,
                                      param_max_rms=param_max_rms, scalar_max=scalar_max,
                                      size_update_period=size_update_period,
                                      clipping_update_period=clipping_update_period))
        self.clip_scales = []  # the clip scale of every step of every group

    @torch.no_grad()
    def step(self):
        for group in self.param_groups:
            stacks = []
            for batch in _batches(group["params"]):
                p = torch.stack(batch)
                p.grad = torch.stack([torch.zeros_like(q) if q.grad is None else q.grad for q in batch])
                stacks.append((p, self.state[batch[0]], batch))
            scale = 1.0 if len(stacks[0][1]) == 0 else self._clip_scale(group, stacks)
            self.clip_scales.append(scale)
            for p, st, _ in stacks:
                if len(st) == 0:
                    self._init(group, p, st)
                self._one(group, p, st, scale)
            for p, _, batch in stacks:
                for i, q in enumerate(batch):
                    q.copy_(p[i])

    def _init(self, group, p, st):
        st["step"] = 0
        st["delta"] = torch.zeros_like(p)
        if p.numel() > 1:
            rms = (p ** 2).mean(dim=list(range(1, p.ndim)), keepdim=True).sqrt()
            st["param_rms"] = rms
            st["scale_exp_avg_sq"] = torch.zeros_like(rms)
            st["scale_grads"] = torch.zeros(group["size_update_period"], *rms.shape, device=p.device, dtype=p.dtype)
        st["exp_avg_sq"] = torch.zeros_like(p)

    def _clip_scale(self, group, stacks):
        cs = group["clipping_scale"]
        fs = stacks[0][1]
        step = fs["step"]
        if cs is None or step == 0:
            return 1.0
        P = group["clipping_update_period"]
        tot = torch.tensor(0.0, device=stacks[0][0].device)
        for p, st, _ in stacks:
            if p.numel() == p.shape[0]:
                tot += (p.grad ** 2).sum()
            else:
                tot += ((p.grad * st["param_rms"]) ** 2).sum()
        norm = tot.sqrt()
        if "model_norms" not in fs:
            fs["model_norms"] = torch.zeros(P, device=norm.device)
        fs["model_norms"][step % P] = norm
        if step % P == 0:
            srt = fs["model_norms"].sort()[0].to("cpu")
            fs["model_norm_threshold"] = cs * srt[min(P - 1, (P // 4) * 2)].item()
            fs["num_clipped"] = 0
        if step < P:
            return 1.0
        if "model_norm_threshold" not in fs:
            return 1.0
        ans = min(1.0, (fs["model_norm_threshold"] / (norm + 1.0e-20)).item())
        if ans < 1.0:
            fs["num_clipped"] += 1
        return ans

    def _one(self, group, p, st, scale):
        beta1, beta2 = group["betas"]
        P = group["size_update_period"]
        g = p.grad
        if scale != 1.0:
            g = g * scale
        step = st["step"]
        st["delta"].mul_(beta1)
        if p.numel() // p.shape[0] > 1:
            dims = list(range(1, p.ndim))
            st["scale_grads"][step % P] = (p * g).sum(dim=dims, keepdim=True)
            if step % P == P - 1:
                st["param_rms"].copy_((p ** 2).mean(dim=dims, keepdim=True).sqrt())
                if step > 0:
                    self._size(group, p, st)
            self._core(group, p, p.grad, st)
        else:
            self._scalar(group, p, p.grad, st)  # _step and _step_scalar read the unclipped p.grad
        st["step"] = step + 1

    def _size(self, group, p, st):
        beta1, beta2 = group["betas"]
        sg = st["scale_grads"]
        P = sg.shape[0]
        size_lr = group["lr"] * group["scalar_lr_scale"]
        b2c = beta2 ** P
        st["scale_exp_avg_sq"].mul_(b2c).add_((sg ** 2).mean(dim=0), alpha=1 - b2c)
        bc2 = 1 - b2c ** ((st["step"] + 1) // P)
        step = -size_lr * (bc2 ** 0.5) * sg.sum(dim=0) / (st["scale_exp_avg_sq"].sqrt() + group["eps"])
        step.masked_fill_(st["param_rms"] < group["param_min_rms"], 0.0)
        step.masked_fill_(st["param_rms"] > group["param_max_rms"], -size_lr * P)
        st["delta"].add_(p * step, alpha=1 - beta1)

    def _core(self, group, p, g, st):
        beta1, beta2 = group["betas"]
        v = st["exp_avg_sq"]
        v.mul_(beta2).addcmul_(g, g, value=1 - beta2)
        bc2 = 1 - beta2 ** (st["step"] - st.get("zero_step", 0) + 1)
        if bc2 < 0.99:
            v = v * (1.0 / bc2)
        den = v.sqrt()
        den += group["eps"]
        alpha = -group["lr"] * (1 - beta1) * st["param_rms"].clamp(min=group["param_min_rms"])
        st["delta"].add_((g / den) * alpha)
        p.add_(st["delta"])

    def _scalar(self, group, p, g, st):
        beta1, beta2 = group["betas"]
        lr = group["lr"] * group["scalar_lr_scale"]
        v = st["exp_avg_sq"]
        v.mul_(beta2).addcmul_(g, g, value=1 - beta2)
        den = (v / (1 - beta2 ** (st["step"] + 1))).sqrt() + group["eps"]
        st["delta"].add_(g / den, alpha=-lr * (1 - beta1))
        p.clamp_(min=-group["scalar_max"], max=group["scalar_max"])
        p.add_(st["delta"])


class EveOracle(Optimizer):
    def __init__(self, params, lr=1e-3, betas=(0.9, 0.98), eps=1e-8, weight_decay=1e-3, target_rms=0.1):
        super().__init__(params, dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay, target_rms=target_rms))

    @torch.no_grad()
    def step(self):
        for group in self.param_groups:
            beta1, beta2 = group["betas"]
            for p in group["params"]:
                if p.grad is None:
                    continue
                g = p.grad
                st = self.state[p]
                if len(st) == 0:
                    st["step"] = 0
                    st["exp_avg"] = torch.zeros_like(p)
                    st["exp_avg_sq"] = torch.zeros_like(p)
                st["step"] += 1
                bc1 = 1 - beta1 ** st["step"]
                bc2 = 1 - beta2 ** st["step"]
                st["exp_avg"].mul_(beta1).add_(g, alpha=1 - beta1)
                st["exp_avg_sq"].mul_(beta2).addcmul_(g, g, value=1 - beta2)
                den = (st["exp_avg_sq"].sqrt() * (bc2 ** -0.5)).add_(group["eps"])
                if p.numel() > 1:
                    above = p.norm() > (group["target_rms"] * (p.numel() ** 0.5))
                    p.mul_(1 - (group["weight_decay"] * above))
                p.addcdiv_(st["exp_avg"], den, value=-group["lr"] / bc1)


def eden_lr(base_lr, batch, epoch, lr_batches=5000, lr_epochs=4, warmup_batches=500.0):
    f = ((batch ** 2 + lr_batches ** 2) / lr_batches ** 2) ** -0.25 * (
        ((epoch ** 2 + lr_epochs ** 2) / lr_epochs ** 2) ** -0.25)
    return base_lr * f * (1.0 if batch >= warmup_batches else 0.5 + 0.5 * (batch / warmup_batches))


def noam_lr(base_lr, step, dim_embed, warmup_steps):
    return base_lr * dim_embed ** (-0.5) * min(step ** (-0.5), step * warmup_steps ** (-1.5))


# ---- the fixture's recipe (tools/gen_golden_optim.py) ------------------------------------------------------------------
D = 32
STEPS = 40
PERIOD = 8
SNAP_STEPS = (3, 4, 8, 9, 16, 17)
BIG = ("stack.0.weight", "stack.1.weight", "table")  # stored at step 40 only


def make_params(device="cpu"):
    """VALLE's shape classes at d = 32: names -> fp32 parameters (seeded)."""
    g = torch.Generator().manual_seed(1234)
    shapes = [("alpha.0", (1,)), ("alpha.1", (1,)), ("alpha.2", (1,)), ("row", (1, D)),
              ("stack.0.weight", (3 * D, D)), ("stack.1.weight", (3 * D, D)),
              ("stack.0.bias", (3 * D,)), ("stack.1.bias", (3 * D,)), ("table", (1025, D))]
    scales = {"alpha": 1.0, "row": 0.05, "stack.0.weight": 0.3, "stack.1.weight": 0.02, "stack.0.bias": 0.01,
              "stack.1.bias": 0.5, "table": 0.12}
    out = {}
    for n, s in shapes:
        sc = scales["alpha"] if n.startswith("alpha") else scales[n]
        out[n] = torch.nn.Parameter((torch.randn(s, generator=g) * sc).to(device))
    return out


def grad_scale(step):
    """steps 13 and 29 carry 10x gradients, step 22 and 37 100x: clipping fires below 1 and below 0.1"""
    return {13: 10.0, 29: 10.0, 22: 100.0, 37: 100.0}.get(step, 1.0)


def table_grad_none(step):
    return step % 5 == 2


def make_grads(params, step):
    """the gradients of step `step` (1-based), seeded per step on the CPU"""
    g = torch.Generator().manual_seed(10_000 + step)
    out = {}
    for n, p in params.items():
        x = torch.randn(p.shape, generator=g) * 0.1 * grad_scale(step)
        out[n] = None if (n == "table" and table_grad_none(step)) else x
    return out


def groups_of(params, two_groups):
    names = list(params)
    if not two_groups:
        return [names]
    return [[n for n in names if n.startswith("alpha") or n == "table"],
            [n for n in names if not (n.startswith("alpha") or n == "table")]]
