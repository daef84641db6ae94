"""valle/modules/scheduler.py surface: calc_lr, NoamScheduler, get_scheduler."""
from valle_b200.modules.scheduler import NoamScheduler, calc_lr, get_scheduler  # noqa: F401
