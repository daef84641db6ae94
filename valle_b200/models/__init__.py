"""Model factory with the reference's flags (valle/models/__init__.py:18-136)."""
import argparse

import torch.nn as nn

from .macros import NUM_AUDIO_TOKENS, NUM_MEL_BINS, NUM_SPEAKER_CLASSES, NUM_TEXT_TOKENS, SPEAKER_EMBEDDING_DIM
from .valle import VALLE, PromptedFeatures


def str2bool(v):
    """icefall.utils.str2bool as used by the reference's flag definitions"""
    if isinstance(v, bool):
        return v
    if str(v).lower() in ("yes", "true", "t", "y", "1"):
        return True
    if str(v).lower() in ("no", "false", "f", "n", "0"):
        return False
    raise argparse.ArgumentTypeError("Boolean value expected.")


def add_model_arguments(parser: argparse.ArgumentParser):
    """the reference's model flags with the same names and defaults (valle/models/__init__.py:18-95)"""
    a = parser.add_argument
    a("--model-name", type=str, default="VALL-E", help="VALL-E (VALL-F / Transformer are not built here).")
    a("--decoder-dim", type=int, default=1024, help="Embedding dimension in the decoder model.")
    a("--nhead", type=int, default=16, help="Number of attention heads in the Decoder layers.")
    a("--num-decoder-layers", type=int, default=12, help="Number of Decoder layers.")
    a("--scale-factor", type=float, default=1.0, help="NAR scale factor (only 1.0 is built).")
    a("--norm-first", type=str2bool, default=True, help="Pre or Post Normalization.")
    a("--add-prenet", type=str2bool, default=False, help="Whether add PreNet after Inputs.")
    a("--prefix-mode", type=int, default=0,
      help="How to prefix the NAR decoder: 0 none, 1 0-to-random, 2 random-to-random, 4 chunk of pre/post utterance.")
    a("--share-embedding", type=str2bool, default=True,
      help="Share the output projection with the acoustic embedding.")
    a("--prepend-bos", type=str2bool, default=False, help="Prepend <BOS> to the AR decoder inputs.")
    a("--num-quantizers", type=int, default=8, help="Number of audio quantization layers.")
    a("--scaling-xformers", type=str2bool, default=False, help="(debug Transformer only; not built)")


def get_model(params) -> nn.Module:
    """valle/models/__init__.py:98-136 for model_name VALL-E: VALLE(decoder_dim, nhead, num_decoder_layers, ...)"""
    name = params.model_name.lower()
    if name not in ("vall-e", "valle"):
        raise NotImplementedError(
            f"valle_b200.get_model: model_name={params.model_name!r}: only VALL-E is on the H100 hot path "
            "(VALL-F and the debug Transformer are out of scope, SURVEY.md section 2 rows 1/7)")
    return VALLE(params.decoder_dim, params.nhead, params.num_decoder_layers, norm_first=params.norm_first,
                 add_prenet=params.add_prenet, prefix_mode=params.prefix_mode,
                 share_embedding=params.share_embedding, nar_scale_factor=params.scale_factor,
                 prepend_bos=params.prepend_bos, num_quantizers=params.num_quantizers)
