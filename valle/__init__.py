"""`valle` -- the reference's package name, served by the H100 engine.

A user of lifeiteng/vall-e switches by putting this repository ahead of the reference on `sys.path`:
`from valle.models import get_model, add_model_arguments`, `from valle.data import AudioTokenizer,
tokenize_audio`, `from valle.modules.transformer import TransformerEncoder` ... resolve to the
`valle_b200` classes (same constructor signatures, parameter names and checkpoint layout,
valle/__init__.py:1 imports the same four sub-packages).  Everything here is a re-export; the code lives
in `valle_b200/`.
"""
from . import data, models, modules, utils  # noqa: F401
