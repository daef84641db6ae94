"""valle/modules/optim.py surface: ScaledAdam, Eve, LRScheduler, Eden.

The constructor signatures, defaults, `param_groups` and the `state_dict()` layout are the reference's
(valle/modules/optim.py:129-986), so a checkpoint written by either implementation resumes in the other.  The step
itself runs in libvalle_b200.so (include/valle_b200.h f3):

* ScaledAdam keeps the reference's batching: the parameters of a group are grouped by `(str(dtype), *shape)`, the
  groups are sorted by that key, and the stacked state `[n, *shape]` of a batch lives in `self.state` of its first
  parameter.  Nothing is stacked at step time: `vb_scaled_adam_step` reads every real parameter and gradient in place
  and addresses its slot of the stacked state.  One step of a group is three launches (for up to 1024 tensors).
* Eve runs two launches per group (for up to 480 tensors with a gradient).
* Parameters must be fp32 CUDA tensors.  There is no CPU path.

`step()` does not synchronise with the device, with two exceptions.  Every `clipping_update_period` steps it reads
`model_norms` back to log the quartiles, as the reference does.  With `show_dominant_parameters=True` it reads the
clip scale back on every step and logs as the reference does.  With `show_dominant_parameters=False` (the trainer's
setting) the reference's per-step "Scaling gradients by ..." warning for a scale below 0.1 cannot be raised without a
sync; instead the device keeps the smallest scale of the period, and the period log warns with it when it is below
0.1.

The state keys hold what the reference's hold.  `step` is a Python int in every batch's state.  `num_clipped` is
counted on the device; `state_dict()` reads it back as an int.  `model_norm_threshold` is a Python float, set on the
period steps.  The engine's packed bf16 weights are keyed on each parameter's version counter, so `step()` bumps
the version of every parameter it updates.
"""
from __future__ import annotations

import ctypes as C
import logging
from collections import defaultdict
from typing import List, Optional, Union

import numpy as np
import torch
from torch import Tensor
from torch.optim import Optimizer

from .. import _lib as L

__all__ = ["ScaledAdam", "Eve", "LRScheduler", "Eden"]


def _check_param(p: Tensor, name: str, opt: str) -> None:
    if not (isinstance(p, Tensor) and p.is_cuda and p.dtype == torch.float32):
        dev = p.device if isinstance(p, Tensor) else type(p).__name__
        dt = p.dtype if isinstance(p, Tensor) else ""
        raise L.VbError(f"{opt}: parameter {name} is {dt} on {dev}; the native step takes fp32 CUDA parameters only "
                        "(there is no CPU or PyTorch fallback)")
    if not p.is_contiguous():
        raise L.VbError(f"{opt}: parameter {name} is not contiguous")


def _check_sadam_params(batches) -> None:
    """ScaledAdam keeps a param_rms and scale_grads slot per parameter; a zero-element one has none (the reference
    fails on it with a KeyError), so it is refused before any state or table is built."""
    for _, ps, ns in batches:
        for p, n in zip(ps, ns):
            _check_param(p, n, "ScaledAdam")
            if p.numel() == 0:
                raise L.VbError(f"ScaledAdam: parameter {n} has no elements; ScaledAdam cannot step a zero-element "
                                "parameter (it has no rms to scale its update by)")


def _check_grad(g: Tensor, p: Tensor, name: str, opt: str) -> None:
    if g.is_sparse:
        raise RuntimeError(f"{opt} optimizer does not support sparse gradients")
    if g.dtype != torch.float32 or g.device != p.device or g.shape != p.shape or not g.is_contiguous():
        raise L.VbError(f"{opt}: the gradient of {name} must be a contiguous fp32 tensor of the parameter's shape and "
                        f"device (got {g.dtype}, {tuple(g.shape)}, {g.device})")


def _sorted_batches(params, names):
    """The reference's batching (optim.py:76-96): [(key, [params], [names])] sorted by (str(dtype), *shape)."""
    by_key, by_key_names = defaultdict(list), defaultdict(list)
    for p, n in zip(params, names):
        key = (str(p.dtype), *p.shape)
        by_key[key].append(p)
        by_key_names[key].append(n)
    return [(k, by_key[k], by_key_names[k]) for k in sorted(by_key)]


class _SadamPlan:
    """The native tensor table of one parameter group: built when the group's parameters or state tensors move."""

    def __init__(self, batches, states, device):
        entries, chunk0, order, names = [], [0], [], []
        keep = []
        for (_, ps, ns), st in zip(batches, states):
            n = len(ps)
            scalar = ps[0].numel() == 1
            per = ps[0].numel()
            for k in ("delta", "exp_avg_sq", "param_rms", "scale_exp_avg_sq", "scale_grads"):
                if k in st and not st[k].is_contiguous():
                    st[k] = st[k].contiguous()
            keep.append([st[k] for k in ("delta", "exp_avg_sq", "param_rms", "scale_exp_avg_sq", "scale_grads")
                         if k in st])
            base = {k: (st[k].data_ptr() if k in st else 0)
                    for k in ("delta", "exp_avg_sq", "param_rms", "scale_exp_avg_sq", "scale_grads")}
            for i, p in enumerate(ps):
                e = L.ScaledAdamTensor()
                e.param = p.data_ptr()
                e.delta = base["delta"] + 4 * i * per
                e.exp_avg_sq = base["exp_avg_sq"] + 4 * i * per
                e.param_rms = base["param_rms"] + 4 * i if base["param_rms"] else None
                if not scalar:
                    e.scale_exp_avg_sq = base["scale_exp_avg_sq"] + 4 * i
                    e.scale_grads = base["scale_grads"] + 4 * i
                e.numel = per
                e.chunk0 = chunk0[-1]
                e.sg_stride = n
                e.scalar = 1 if scalar else 0
                entries.append(e)
                chunk0.append(chunk0[-1] + (per + L.OPTIM_CHUNK - 1) // L.OPTIM_CHUNK)
                order.append(p)
            names.extend(ns)
        self.params = order
        self.names = names
        self.n = len(order)
        self.n_chunks = chunk0[-1]
        self.chunk0 = (C.c_int32 * len(chunk0))(*chunk0)
        self.grads = np.zeros(self.n, dtype=np.int64)
        table = (L.ScaledAdamTensor * self.n)(*entries)
        host = torch.frombuffer(bytearray(bytes(table)), dtype=torch.uint8).pin_memory()
        self._host_table = host  # the upload below reads it asynchronously
        self.table = host.to(device, non_blocking=True)
        ws = L.load().vb_scaled_adam_workspace(self.n, self.n_chunks)
        self.workspace = torch.empty(ws, dtype=torch.uint8, device=device)
        self.key = self.signature(batches, states)
        self._keep = keep

    @staticmethod
    def signature(batches, states):
        return (tuple(p.data_ptr() for _, ps, _ in batches for p in ps),
                tuple(st[k].data_ptr() for st in states
                      for k in ("delta", "exp_avg_sq", "param_rms", "scale_exp_avg_sq", "scale_grads") if k in st))


class ScaledAdam(Optimizer):
    """valle/modules/optim.py:129-661 (ScaledAdam over BatchedOptimizer), stepped by vb_scaled_adam_step.

    Args are the reference's: lr, clipping_scale, betas, scalar_lr_scale, eps, param_min_rms, param_max_rms,
    scalar_max, size_update_period, clipping_update_period, parameters_names (one list of names per group) and
    show_dominant_parameters.  All batches of a group must be at the same `step` (they are unless a state dict mixes
    them)."""

    def __init__(self, params, lr=3e-02, clipping_scale=None, betas=(0.9, 0.98), scalar_lr_scale=0.1, eps=1.0e-08,
                 param_min_rms=1.0e-05, param_max_rms=3.0, scalar_max=10.0, size_update_period=4,
                 clipping_update_period=100, parameters_names=None, show_dominant_parameters=True):
        assert parameters_names is not None, (
            "Please prepare parameters_names, which is a List[List[str]]. Each List[str] is for a group and each str "
            "is for a parameter")
        defaults = dict(lr=lr, clipping_scale=clipping_scale, betas=betas, scalar_lr_scale=scalar_lr_scale, eps=eps,
                        param_min_rms=param_min_rms, param_max_rms=param_max_rms, scalar_max=scalar_max,
                        size_update_period=size_update_period, clipping_update_period=clipping_update_period)
        super().__init__(params, defaults)
        assert len(self.param_groups) == len(parameters_names)
        self.parameters_names = parameters_names
        self.show_dominant_parameters = show_dominant_parameters
        self._reset_native()

    def _reset_native(self):
        self._plans = {}   # group index -> _SadamPlan
        self._clip = {}    # group index -> device vb_clip_state (32 bytes), valid while not stale
        self._clip_stale = set()

    def __setstate__(self, state):
        super().__setstate__(state)
        self._reset_native()

    def load_state_dict(self, state_dict):
        super().load_state_dict(state_dict)
        self._plans = {}
        self._clip_stale = set(self._clip)

    def state_dict(self):
        self._flush_counters()
        return super().state_dict()

    # -- clipping state shared with the device ----------------------------------------------------------------------
    def _first_state(self, gi):
        group, names = self.param_groups[gi], self.parameters_names[gi]
        return self.state[_sorted_batches(group["params"], names)[0][1][0]]

    def _flush_counters(self):
        """num_clipped lives on the device between period steps: copy it into the state (a sync)."""
        for gi, buf in self._clip.items():
            if gi in self._clip_stale:
                continue
            fs = self._first_state(gi)
            if "num_clipped" in fs:
                fs["num_clipped"] = int(self._read_clip(buf).num_clipped)

    @staticmethod
    def _read_clip(buf) -> L.ClipState:
        return L.ClipState.from_buffer_copy(buf.cpu().numpy().tobytes())

    def _upload_clip(self, gi, fs, device):
        cs = L.ClipState()
        cs.threshold = float(fs.get("model_norm_threshold", 0.0))
        cs.has_threshold = 1 if "model_norm_threshold" in fs else 0
        cs.num_clipped = int(fs.get("num_clipped", 0))
        cs.scale = cs.min_scale = cs.prev_min_scale = 1.0
        host = torch.frombuffer(bytearray(bytes(cs)), dtype=torch.uint8)
        buf = self._clip.get(gi)
        if buf is None or buf.device != device:
            buf = torch.empty(C.sizeof(L.ClipState), dtype=torch.uint8, device=device)
            self._clip[gi] = buf
        buf.copy_(host)
        self._clip_stale.discard(gi)
        return buf

    # -- the step -----------------------------------------------------------------------------------------------------
    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        for gi, (group, names) in enumerate(zip(self.param_groups, self.parameters_names)):
            self._step_group(gi, group, names)
        return loss

    def _init_state(self, group, ps, state):
        """optim.py:265-314 for the stack of `ps`; param_rms is filled by the first native step (init flag)."""
        n = len(ps)
        dev = ps[0].device
        stacked = (n, *ps[0].shape)
        state["step"] = 0
        state["delta"] = torch.zeros(stacked, dtype=torch.float32, device=dev)
        if n * ps[0].numel() > 1:  # the reference tests numel of the whole stack (optim.py:295)
            rms_shape = (n,) + (1,) * ps[0].dim()
            state["param_rms"] = torch.zeros(rms_shape, dtype=torch.float32, device=dev)
            state["scale_exp_avg_sq"] = torch.zeros(rms_shape, dtype=torch.float32, device=dev)
            state["scale_grads"] = torch.zeros((group["size_update_period"], *rms_shape), dtype=torch.float32,
                                               device=dev)
        state["exp_avg_sq"] = torch.zeros(stacked, dtype=torch.float32, device=dev)

    def _step_group(self, gi, group, names):
        params = group["params"]
        if not params:
            return
        batches = _sorted_batches(params, names)
        states = [self.state[ps[0]] for _, ps, _ in batches]
        plan = self._plans.get(gi)
        first_empty = len(states[0]) == 0
        empty = [len(st) == 0 for st in states]
        if any(empty):
            if not all(empty):
                raise ValueError("ScaledAdam: some batches of a parameter group have state and others have none; "
                                 "the native step needs one step count per group")
            _check_sadam_params(batches)
            for (_, ps, _), st in zip(batches, states):
                self._init_state(group, ps, st)
            plan = None
        fs = states[0]
        step = fs["step"]
        zero_step = fs.get("zero_step", 0)
        for st in states:
            if st["step"] != step or st.get("zero_step", 0) != zero_step:
                raise ValueError(f"ScaledAdam: the batches of group {gi} are at different steps "
                                 f"({st['step']} vs {step}); the native step needs one step count per group")
        if plan is None or plan.key != _SadamPlan.signature(batches, states):
            _check_sadam_params(batches)
            plan = _SadamPlan(batches, states, params[0].device)
            self._plans[gi] = plan

        # clipping (optim.py:242-247, 316-412)
        cs = group["clipping_scale"]
        P = group["clipping_update_period"]
        clip_mode, log_step = 0, False
        dev = params[0].device
        if not (first_empty or cs is None or step == 0):
            if "model_norms" not in fs:
                fs["model_norms"] = torch.zeros(P, device=dev)
            log_step = step % P == 0
            if step < P:
                clip_mode = 1
            elif "model_norm_threshold" not in fs and not log_step:
                logging.info("Warning: model_norm_threshold not in state: possibly you changed config when "
                             "restarting, adding clipping_scale option?")
                clip_mode = 1
            else:
                clip_mode = 2
        buf = self._clip.get(gi)
        if buf is None or gi in self._clip_stale:
            buf = self._upload_clip(gi, fs, dev)
        norms = fs.get("model_norms")
        if clip_mode and (norms.dtype != torch.float32 or norms.numel() != P or not norms.is_contiguous()):
            raise ValueError(f"ScaledAdam: model_norms has shape {tuple(norms.shape)}, expected ({P},) fp32")

        grads = plan.grads
        for t, (p, name) in enumerate(zip(plan.params, plan.names)):
            g = p.grad
            if g is None:
                grads[t] = 0
            else:
                _check_grad(g, p, name, "ScaledAdam")
                grads[t] = g.data_ptr()

        beta1, beta2 = group["betas"]
        a = L.ScaledAdamArgs(n_tensors=plan.n, n_chunks=plan.n_chunks, step=step, zero_step=zero_step,
                             init=1 if first_empty else 0, clip_mode=clip_mode, clip_period=P,
                             size_period=group["size_update_period"],
                             clipping_scale=float(cs) if cs is not None else 0.0, lr=group["lr"],
                             scalar_lr_scale=group["scalar_lr_scale"], beta1=beta1, beta2=beta2, eps=group["eps"],
                             param_min_rms=group["param_min_rms"], param_max_rms=group["param_max_rms"],
                             scalar_max=group["scalar_max"])
        lib = L.load()
        L.check(lib.vb_scaled_adam_step(plan.table.data_ptr(), grads.ctypes.data, plan.chunk0, C.byref(a),
                                        L.ptr(norms) if clip_mode else None, buf.data_ptr(),
                                        plan.workspace.data_ptr(), plan.workspace.numel(), L.stream_ptr()),
                "vb_scaled_adam_step")
        torch.autograd.graph.increment_version(plan.params)
        for st in states:
            st["step"] = step + 1

        if log_step:
            self._log_period(fs, buf, cs, P)
        if clip_mode == 2 and self.show_dominant_parameters:
            scale = self._read_clip(buf).scale
            if scale < 0.1:
                logging.warning(f"Scaling gradients by {scale}, model_norm_threshold={fs['model_norm_threshold']}")
                self._show_gradient_dominating_parameter(plan, scale)

    def _log_period(self, fs, buf, cs, P):
        """The period step of optim.py:363-389 (a sync, as in the reference)."""
        sorted_norms = fs["model_norms"].sort()[0].to("cpu")
        quartiles = [sorted_norms[min(P - 1, (P // 4) * n)].item() for n in range(0, 5)]
        threshold = cs * quartiles[2]
        fs["model_norm_threshold"] = threshold
        st = self._read_clip(buf)
        percent_clipped = st.prev_clipped * 100.0 / P if "num_clipped" in fs else 0.0
        fs["num_clipped"] = int(st.num_clipped)
        q = " ".join(["%.3e" % x for x in quartiles])
        logging.info(f"Clipping_scale={cs}, grad-norm quartiles {q}, threshold={threshold:.3e}, "
                     f"percent-clipped={percent_clipped:.1f}")
        if not self.show_dominant_parameters and st.prev_min_scale < 0.1:
            logging.warning(f"Scaling gradients by {st.prev_min_scale} (the smallest clip scale of the last "
                            f"{P} steps), model_norm_threshold={threshold}")

    def _show_gradient_dominating_parameter(self, plan, scale):
        """optim.py:414-477: the parameter with the largest share of the clipped model norm (diagnostic, syncs)."""
        shares = {}
        for p, name in zip(plan.params, plan.names):
            g = p.grad if p.grad is not None else torch.zeros_like(p)
            shares[name] = (g, float((g.double() ** 2).sum()))
        tot = sum(v for _, v in shares.values()) or 1.0
        name, (g, v) = max(shares.items(), key=lambda kv: kv[1][1])
        logging.info(f"Parameter Dominanting tot_sumsq {name} with proportion {v / tot:.2f}, where "
                     f"dominant_sumsq=(grad_sumsq*orig_rms_sq)={v:.3e}, grad_sumsq = {(g ** 2).sum():.3e}, "
                     f"clip scale={scale:.3e}")


class LRScheduler(object):
    """valle/modules/optim.py:664-756: learning-rate schedule on the batch and the epoch."""

    def __init__(self, optimizer: Optimizer, verbose: bool = False):
        if not isinstance(optimizer, Optimizer):
            raise TypeError("{} is not an Optimizer".format(type(optimizer).__name__))
        self.optimizer = optimizer
        self.verbose = verbose
        for group in optimizer.param_groups:
            group.setdefault("base_lr", group["lr"])
        self.base_lrs = [group["base_lr"] for group in optimizer.param_groups]
        self.epoch = 0
        self.batch = 0

    def state_dict(self):
        return {"base_lrs": self.base_lrs, "epoch": self.epoch, "batch": self.batch}

    def load_state_dict(self, state_dict):
        self.__dict__.update(state_dict)

    def get_last_lr(self) -> List[float]:
        return self._last_lr

    def get_lr(self):
        raise NotImplementedError

    def step_batch(self, batch: Optional[int] = None) -> None:
        self.batch = batch if batch is not None else self.batch + 1
        self._set_lrs()

    def step_epoch(self, epoch: Optional[int] = None):
        self.epoch = epoch if epoch is not None else self.epoch + 1
        self._set_lrs()

    def _set_lrs(self):
        values = self.get_lr()
        assert len(values) == len(self.optimizer.param_groups)
        for i, (group, lr) in enumerate(zip(self.optimizer.param_groups, values)):
            group["lr"] = lr
            self.print_lr(self.verbose, i, lr)
        self._last_lr = [group["lr"] for group in self.optimizer.param_groups]

    def print_lr(self, is_verbose, group, lr):
        if is_verbose:
            logging.info(f"Epoch={self.epoch}, batch={self.batch}: adjusting learning rate of group {group} to "
                         f"{lr:.4e}.")


class Eden(LRScheduler):
    """valle/modules/optim.py:759-807: lr = base_lr * ((batch^2 + lr_batches^2) / lr_batches^2)^-0.25 *
    ((epoch^2 + lr_epochs^2) / lr_epochs^2)^-0.25 * warmup, warmup rising linearly from 0.5 to 1 over
    warmup_batches."""

    def __init__(self, optimizer: Optimizer, lr_batches: Union[int, float], lr_epochs: Union[int, float],
                 warmup_batches: Union[int, float] = 500.0, verbose: bool = False):
        super().__init__(optimizer, verbose)
        self.lr_batches = lr_batches
        self.lr_epochs = lr_epochs
        self.warmup_batches = warmup_batches

    def get_lr(self):
        b, e = self.batch, self.epoch
        factor = ((b ** 2 + self.lr_batches ** 2) / self.lr_batches ** 2) ** -0.25 * (
            ((e ** 2 + self.lr_epochs ** 2) / self.lr_epochs ** 2) ** -0.25)
        warmup = 1.0 if b >= self.warmup_batches else 0.5 + 0.5 * (b / self.warmup_batches)
        return [x * factor * warmup for x in self.base_lrs]


class Eve(Optimizer):
    """valle/modules/optim.py:836-985 (AdamW whose weight decay only applies while ||p|| > target_rms * sqrt(numel)),
    stepped by vb_eve_step.  Parameters with a None gradient are skipped and get no state; a zero-element parameter
    gets its state and its step count, and no table entry."""

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.98), eps=1e-8, weight_decay=1e-3, target_rms=0.1):
        if not 0.0 <= lr:
            raise ValueError("Invalid learning rate: {}".format(lr))
        if not 0.0 <= eps:
            raise ValueError("Invalid epsilon value: {}".format(eps))
        if not 0.0 <= betas[0] < 1.0:
            raise ValueError("Invalid beta parameter at index 0: {}".format(betas[0]))
        if not 0.0 <= betas[1] < 1.0:
            raise ValueError("Invalid beta parameter at index 1: {}".format(betas[1]))
        if not 0 <= weight_decay <= 0.1:
            raise ValueError("Invalid weight_decay value: {}".format(weight_decay))
        if not 0 < target_rms <= 10.0:
            raise ValueError("Invalid target_rms value: {}".format(target_rms))
        super().__init__(params, dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay, target_rms=target_rms))
        self._ws = {}

    def __setstate__(self, state):
        super().__setstate__(state)
        self._ws = {}

    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        lib = L.load()
        for group in self.param_groups:
            beta1, beta2 = group["betas"]
            rows, stepped = [], []
            for i, p in enumerate(group["params"]):
                if p.grad is None:
                    continue
                name = f"param_groups[{self.param_groups.index(group)}]['params'][{i}]"
                _check_param(p, name, "Eve")
                _check_grad(p.grad, p, name, "Eve")
                state = self.state[p]
                if len(state) == 0:
                    state["step"] = 0
                    state["exp_avg"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                    state["exp_avg_sq"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                state["step"] += 1
                n = p.numel()
                if n == 0:  # the reference's update of an empty tensor changes nothing but its step
                    continue
                bc1 = 1 - beta1 ** state["step"]
                bc2 = 1 - beta2 ** state["step"]
                rows.append((p.data_ptr(), p.grad.data_ptr(), state["exp_avg"].data_ptr(),
                             state["exp_avg_sq"].data_ptr(), n, group["lr"] / bc1, bc2 ** -0.5,
                             group["target_rms"] * (n ** 0.5) if n > 1 else float("inf")))
                stepped.append(p)
            if not rows:
                continue
            table = (L.EveTensor * len(rows))()
            for e, r in zip(table, rows):
                e.param, e.grad, e.exp_avg, e.exp_avg_sq, e.numel, e.step_size, e.bc2_rsqrt, e.norm_limit = r
            need = lib.vb_eve_workspace(table, len(rows))
            dev = stepped[0].device
            ws = self._ws.get(dev)
            if ws is None or ws.numel() < need:
                ws = torch.empty(need, dtype=torch.uint8, device=dev)
                self._ws[dev] = ws
            L.check(lib.vb_eve_step(table, len(rows), beta1, beta2, group["eps"], group["weight_decay"],
                                    ws.data_ptr(), ws.numel(), L.stream_ptr()), "vb_eve_step")
            torch.autograd.graph.increment_version(stepped)
        return loss
