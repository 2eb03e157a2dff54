"""Import the UNMODIFIED reference (TEST INFRASTRUCTURE ONLY; used by tests/, bench.py's reference legs, make_golden).

The reference parses its command line when `utils.constant` is first imported (utils/constant.py:99) and imports
`Levenshtein` at module import (utils/metrics.py:3).  Neither is edited: this module
  * finds the checkout ($B200ASR_REFERENCE, or the copy oracle/make_ref.py stages in oracle/_ref),
  * registers a tiny pure-Python `Levenshtein.distance` (python-Levenshtein is not installed; it is only called by
    calculate_cer / calculate_wer, which the Trainer loop uses for logging),
  * sets sys.argv for the first import and, on later calls, re-parses the flags into `constant.args` (every reference
    module reads `constant.args.<flag>` at call time),
  * optionally applies the Q12 shim (SURVEY.md 8c): get_subsequent_mask(...).bool() so greedy/beam search run on torch >= 1.2.
"""
from __future__ import annotations

import os
import sys
import types

HERE = os.path.dirname(os.path.abspath(__file__))


def reference_root():
    for cand in (os.environ.get("B200ASR_REFERENCE"), os.path.join(HERE, "_ref")):
        if cand and os.path.isdir(os.path.join(cand, "models", "asr")):
            return cand
    return None


def available() -> bool:
    return reference_root() is not None


def _edit_distance(a: str, b: str) -> int:
    prev = list(range(len(b) + 1))
    for i, ca in enumerate(a, 1):
        cur = [i]
        for j, cb in enumerate(b, 1):
            cur.append(min(prev[j] + 1, cur[j - 1] + 1, prev[j - 1] + (ca != cb)))
        prev = cur
    return prev[-1]


def load(flags=(), q12_shim=False):
    """Returns a namespace with the reference modules: constant, functions, metrics, common_layers, transformer, trainer,
    optimizer.  `flags` are the reference's own command-line flags (utils/constant.py)."""
    root = reference_root()
    if root is None:
        raise RuntimeError("reference checkout not found (neither $B200ASR_REFERENCE nor oracle/_ref: run oracle/make_ref.py)")
    if root not in sys.path:
        sys.path.insert(0, root)
    if "Levenshtein" not in sys.modules:
        lev = types.ModuleType("Levenshtein")
        lev.distance = _edit_distance
        sys.modules["Levenshtein"] = lev
    flags = [str(f) for f in flags]
    if "utils.constant" not in sys.modules:
        argv, sys.argv = sys.argv, ["reference"] + flags
        try:
            from utils import constant
        finally:
            sys.argv = argv
    else:
        from utils import constant
        constant.args = constant.parser.parse_args(flags)
        constant.USE_CUDA = constant.args.cuda
    import importlib
    ns = types.SimpleNamespace(root=root, constant=constant)
    ns.functions = importlib.import_module("utils.functions")
    ns.metrics = importlib.import_module("utils.metrics")
    ns.optimizer = importlib.import_module("utils.optimizer")
    ns.common_layers = importlib.import_module("models.common_layers")
    ns.transformer = importlib.import_module("models.asr.transformer")
    ns.trainer = importlib.import_module("trainer.asr.trainer")
    if q12_shim and not getattr(ns.transformer.get_subsequent_mask, "_b200_q12", False):
        orig = ns.transformer.get_subsequent_mask

        def bool_mask(seq):
            return orig(seq).bool()

        bool_mask._b200_q12 = True
        ns.transformer.get_subsequent_mask = bool_mask
    return ns


def labels(vocab: int):
    """label2id / id2label with one distinct CJK character per id >= 3 (so greedy_search's strings map back to ids) and the
    reference's special characters for PAD/SOS/EOS (utils/constant.py:105-107)."""
    from utils import constant
    chars = [constant.PAD_CHAR, constant.SOS_CHAR, constant.EOS_CHAR] + [chr(0x4E00 + i) for i in range(vocab - 3)]
    return {c: i for i, c in enumerate(chars)}, {i: c for i, c in enumerate(chars)}
