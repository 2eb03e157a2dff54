"""Drop-in installer: bind the GPU forwards onto the UNMODIFIED reference classes (class-level patch).

    import b200asr; b200asr.install()      # after `utils.constant` has parsed its flags

After this, the reference's own `Transformer` (models/asr/transformer.py), `Trainer` loop
(trainer/asr/trainer.py) and `test.py` run on libb200asr kernels: module tree, parameter names and checkpoints are
untouched; only `forward` attributes and the two loss functions are rebound (SURVEY.md §8b).
"""
from __future__ import annotations

import importlib
import sys

from . import metrics, modules

_PATCHED = {}


def install(reference_root: str = None):
    """Patch models.common_layers / models.asr.transformer / utils.metrics (+ trainer's imported name).
    Returns the dict of original attributes (pass it to uninstall())."""
    if reference_root and reference_root not in sys.path:
        sys.path.insert(0, reference_root)
    cl = importlib.import_module("models.common_layers")
    tr = importlib.import_module("models.asr.transformer")
    um = importlib.import_module("utils.metrics")
    targets = [
        (cl.ScaledDotProductAttention, "forward", modules.sdpa_forward),
        (cl.MultiHeadAttention, "forward", modules.mha_forward),
        (cl.PositionwiseFeedForwardWithConv, "forward", modules.ffn_forward),
        (tr.EncoderLayer, "forward", modules.encoder_layer_forward),
        (tr.DecoderLayer, "forward", modules.decoder_layer_forward),
        (tr.Encoder, "forward", modules.encoder_forward),
        (tr.Decoder, "forward", modules.decoder_forward),
        (tr.Transformer, "forward", modules.transformer_forward),
        (um, "calculate_loss", metrics.calculate_loss),
        (um, "calculate_metrics", metrics.calculate_metrics),
        (tr, "calculate_metrics", metrics.calculate_metrics),
    ]
    t_mod = sys.modules.get("trainer.asr.trainer")      # `from utils.metrics import calculate_metrics` binds by value
    if t_mod is not None:
        targets.append((t_mod, "calculate_metrics", metrics.calculate_metrics))
    for obj, name, new in targets:
        key = (id(obj), name)
        if key not in _PATCHED:
            _PATCHED[key] = (obj, name, getattr(obj, name))
        setattr(obj, name, new)
    return dict(_PATCHED)


def uninstall():
    for obj, name, old in _PATCHED.values():
        setattr(obj, name, old)
    _PATCHED.clear()
