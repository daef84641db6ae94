"""valle/modules/optim.py surface: ScaledAdam, Eve, LRScheduler, Eden."""
from valle_b200.modules.optim import Eden, Eve, LRScheduler, ScaledAdam  # noqa: F401
