"""valle/modules/scheduler.py surface: calc_lr, NoamScheduler, get_scheduler (valle/modules/scheduler.py:24-78).
Host-side learning-rate arithmetic only; the optimizers they drive are in valle_b200.modules.optim."""
from __future__ import annotations

import torch

from .optim import Eden

__all__ = ["calc_lr", "NoamScheduler", "get_scheduler"]


def calc_lr(step, dim_embed, warmup_steps):
    """Noam schedule: dim_embed^-0.5 * min(step^-0.5, step * warmup_steps^-1.5)."""
    return dim_embed ** (-0.5) * min(step ** (-0.5), step * warmup_steps ** (-1.5))


class NoamScheduler(torch.optim.lr_scheduler._LRScheduler):
    """base_lr * calc_lr(self._step_count, dim_embed, warmup_steps) for every parameter group."""

    def __init__(self, base_lr: float, optimizer: torch.optim.Optimizer, dim_embed: int, warmup_steps: int,
                 last_epoch: int = -1, verbose: bool = False) -> None:
        self.dim_embed = dim_embed
        self.base_lr = base_lr
        self.warmup_steps = warmup_steps
        self.num_param_groups = len(optimizer.param_groups)
        # torch 2.2+ deprecates `verbose`; it only ever printed, so it is not forwarded
        super().__init__(optimizer, last_epoch)

    def get_lr(self):
        return [self.base_lr * calc_lr(self._step_count, self.dim_embed, self.warmup_steps)] * self.num_param_groups

    def set_step(self, step: int):
        self._step_count = step


def get_scheduler(params, optimizer):
    """`params.scheduler_name`: "eden" -> Eden(optimizer, 5000, 4, warmup_batches=params.warmup_steps); "noam" ->
    NoamScheduler(params.base_lr, optimizer, params.decoder_dim, warmup_steps=params.warmup_steps); "cosine" ->
    torch's CosineAnnealingLR called with the reference's argument order."""
    name = params.scheduler_name.lower()
    if name == "eden":
        return Eden(optimizer, 5000, 4, warmup_batches=params.warmup_steps)
    if name == "noam":
        return NoamScheduler(params.base_lr, optimizer, params.decoder_dim, warmup_steps=params.warmup_steps)
    if name == "cosine":
        # the reference passes (warmup_steps, optimizer) in this order; kept as written
        return torch.optim.lr_scheduler.CosineAnnealingLR(params.warmup_steps, optimizer, eta_min=params.base_lr)
    raise NotImplementedError(f"{params.scheduler_name}")
