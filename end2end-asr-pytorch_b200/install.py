"""Drop-in installer: bind the GPU forwards onto the UNMODIFIED reference classes (class-level patch).

    import b200asr; b200asr.install()      # after `utils.constant` has parsed its flags

After this, the reference's own `Transformer` (models/asr/transformer.py), `Trainer` loop
(trainer/asr/trainer.py), `test.py` and the LSTM LM's `RNNModel.forward` (utils/lstm_utils.py) run on libb200asr kernels:
module tree, parameter names and checkpoints are untouched; only `forward` attributes, `Decoder.beam_search`,
`Decoder.greedy_search`, `Transformer.evaluate`, the two loss functions and, when trainer/asr/trainer.py is imported,
`Trainer.train` (trainer.trainer_train: the CER / WER counts and the gradient clip on the device) and `NoamOpt.step`
(optim.noam_step: torch.optim.Adam's step on the device, in the optimizer's own state) are rebound (SURVEY.md §8b).  The replaced methods
stay reachable through original(): LM rescoring with an LM other than an LSTM LM still runs the reference's beam_search, a
GRU / RNN LM its own RNNModel.forward, an optimizer other than a plain fp32 CUDA torch.optim.Adam its own NoamOpt.step, greedy_search with lm_rescoring=True or in training mode and evaluate in training
mode the reference's own methods.

When utils/data_loader.py is imported before install(), `AudioDataLoader.__init__` / `__iter__` are bound too
(loader.audio_loader_init / audio_loader_iter): a loader over a SpectrogramDataset yields `_collate_fn`'s batches with
`inputs` computed on the device, its workers only reading audio and making the reference's random draws.  A loader over
another dataset, with the caller's own collate_fn, or with noise clips at another sample rate runs
original(AudioDataLoader, "__iter__").

Data-parallel training: when the environment of `python -m b200asr.launch` describes more than one rank (WORLD_SIZE > 1),
or `process_group=` is passed, install() joins that process group and the bound Trainer.train trains across it
(trainer.trainer_train, parallel.join).  The bound Transformer.evaluate in eval mode then decodes across it too: each rank
decodes its share of the batch and every rank returns the whole batch's strings (modules.evaluate_sharded), so test.py
runs data-parallel under the launcher.  Otherwise nothing about a single process changes.
"""
from __future__ import annotations

import importlib
import sys

from . import loader, metrics, modules, optim, parallel, trainer

_PATCHED = {}


def install(reference_root: str = None, process_group=None):
    """Patch models.common_layers / models.asr.transformer / utils.metrics (+ trainer's imported name).
    process_group: a torch.distributed group the bound Trainer.train trains across; without it the launcher's environment
    (WORLD_SIZE > 1) is joined, if present.  Returns the dict of original attributes (pass it to uninstall())."""
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
        (tr.Decoder, "beam_search", modules.beam_search),
        (tr.Decoder, "greedy_search", modules.greedy_search),
        (tr.Transformer, "forward", modules.transformer_forward),
        (tr.Transformer, "evaluate", modules.transformer_evaluate),
        (um, "calculate_loss", metrics.calculate_loss),
        (um, "calculate_metrics", metrics.calculate_metrics),
        (tr, "calculate_metrics", metrics.calculate_metrics),
    ]
    try:                                                # RNNModel.forward of the LSTM LM (training, LM.evaluate)
        lu = importlib.import_module("utils.lstm_utils")
    except ImportError:
        lu = None
    if lu is not None:
        targets.append((lu.RNNModel, "forward", modules.rnn_model_forward))
    try:                                                # NoamOpt.step: Adam on the device (optim.noam_step)
        uo = importlib.import_module("utils.optimizer")
    except ImportError:
        uo = None
    if uo is not None:
        targets.append((uo.NoamOpt, "step", optim.noam_step))
    t_mod = sys.modules.get("trainer.asr.trainer")      # `from utils.metrics import calculate_metrics` binds by value
    if t_mod is not None:
        targets.append((t_mod, "calculate_metrics", metrics.calculate_metrics))
        targets.append((t_mod.Trainer, "train", trainer.trainer_train))
    dl_mod = sys.modules.get("utils.data_loader")       # AudioDataLoader: the device feature front end (loader.py)
    if dl_mod is not None:
        targets.append((dl_mod.AudioDataLoader, "__init__", loader.audio_loader_init))
        targets.append((dl_mod.AudioDataLoader, "__iter__", loader.audio_loader_iter))
    for obj, name, new in targets:
        key = (id(obj), name)
        if key not in _PATCHED:                         # (.., own): `name` was in obj's own dict, not inherited
            _PATCHED[key] = (obj, name, getattr(obj, name), name in vars(obj))
        setattr(obj, name, new)
    parallel.join(process_group)
    return dict(_PATCHED)


def uninstall():
    for obj, name, old, own in _PATCHED.values():
        if own:
            setattr(obj, name, old)
        else:
            delattr(obj, name)
    _PATCHED.clear()
    parallel.leave()


def original(cls, name):
    """The reference's own attribute `name` of `cls` (or of the nearest patched base class) that install() replaced, or None."""
    for c in getattr(cls, "__mro__", (cls,)):
        hit = _PATCHED.get((id(c), name))
        if hit is not None:
            return hit[2]
    return None
