"""valle/modules operator surface."""
from . import activation, embedding, optim, scheduler, transformer  # noqa: F401
