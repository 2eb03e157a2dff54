"""Mirror of utils/metrics.py:78-154 (calculate_metrics / calculate_loss, CE and CTC branches) on the fused CE kernel and the
CTC kernels, and the training loop's CER / WER edit counts (LabelTable, edit_counts) on the edit-distance kernel."""
from __future__ import annotations

import torch

from . import _lib, ops


def loss_and_stats(pred, gold, smoothing=0.0, reduction="mean"):
    """(loss, stats) without any host synchronisation.  stats = [sum, n_tokens, n_correct, mean, 1/n_tokens]."""
    return ops.CrossEntropyFn.apply(pred, gold, float(smoothing), reduction)


def calculate_loss(pred, gold, input_lengths=None, target_lengths=None, smoothing=0.0, loss_type="ce"):
    """utils/metrics.py:102-154.  "ce": label-smoothed CE / CE over the non-PAD tokens.  "ctc": F.ctc_loss of
    log_softmax(pred) with blank 0 and the mean reduction, `smoothing` ignored, as the reference (ops.CtcLossFn)."""
    if loss_type == "ce":
        loss, _ = loss_and_stats(pred, gold, smoothing)
        return loss
    if loss_type == "ctc":
        return ops.CtcLossFn.apply(pred, gold, input_lengths, target_lengths)
    raise NotImplementedError(f"b200asr implements the 'ce' and 'ctc' losses only, not {loss_type!r}")


def calculate_metrics(pred, gold, input_lengths=None, target_lengths=None, smoothing=0.0, loss_type="ce"):
    """utils/metrics.py:78-99 -> (loss, num_correct).  For "ce", num_correct is a Python int as in the reference (one D2H
    sync, the reference has the same at :94); use loss_and_stats() to stay asynchronous.  For "ctc" it is None (:96-97)."""
    if loss_type == "ctc":
        return calculate_loss(pred, gold, input_lengths, target_lengths, smoothing, loss_type), None
    if loss_type != "ce":
        raise NotImplementedError(f"b200asr implements the 'ce' and 'ctc' losses only, not {loss_type!r}")
    loss, stats = loss_and_stats(pred, gold, smoothing)
    return loss, int(stats[2].item())


class LabelTable:
    """id2label in the form b200asr_edit_counts reads (include/b200asr.h): per id an offset and a length into one array of
    code points, a valid flag, and per code point bit 0 = ' ' and bit 1 = str.isspace().

    id2label must be a dict from ints >= 0 to str labels; V = max id + 1 and the ids in [0, V) missing from it are invalid.
    Every code point in `drop_chars` (single code points only) is removed from every label, which is the same as removing it
    from the joined string, as the trainer does with SOS_CHAR / EOS_CHAR (trainer/asr/trainer.py:97-98).  Anything else
    raises TypeError or ValueError.  The arrays are built once on the host; tensors(device) uploads them once per device."""

    def __init__(self, id2label, pad_id, drop_chars=()):
        if not isinstance(id2label, dict) or not id2label:
            raise TypeError("LabelTable: id2label must be a non-empty dict {id: label}")
        for k, lab in id2label.items():
            if type(k) is not int or k < 0:
                raise ValueError(f"LabelTable: ids must be ints >= 0, got {k!r}")
            if not isinstance(lab, str):
                raise TypeError(f"LabelTable: the label of id {k} is a {type(lab).__name__}, not a str")
        for c in drop_chars:
            if not isinstance(c, str) or len(c) != 1:
                raise ValueError(f"LabelTable: drop_chars must be single code points, got {c!r}")
        drop = set(drop_chars)
        self.V = max(id2label) + 1
        self.pad_id = int(pad_id)
        off, length, valid, cps = [], [], [], []
        for i in range(self.V):
            lab = id2label.get(i)
            off.append(len(cps))
            valid.append(lab is not None)
            kept = [c for c in (lab or "") if c not in drop]
            length.append(len(kept))
            cps.extend(kept)
        if len(cps) >= 2 ** 31:
            raise ValueError("LabelTable: more than 2^31 - 1 code points in all labels")
        self.max_label_len = max(length)
        self.off = torch.tensor(off, dtype=torch.int32)
        self.length = torch.tensor(length, dtype=torch.int32)
        self.valid = torch.tensor(valid, dtype=torch.uint8)
        self.code_points = torch.tensor([ord(c) for c in cps] or [0], dtype=torch.int32)
        self.flags = torch.tensor([int(c == " ") | int(c.isspace()) << 1 for c in cps] or [0], dtype=torch.uint8)
        self._on = {}

    def tensors(self, device):
        """(off, length, code_points, flags, valid) on `device`."""
        device = torch.device(device)
        if device not in self._on:
            self._on[device] = tuple(t.to(device) for t in (self.off, self.length, self.code_points, self.flags, self.valid))
        return self._on[device]


def edit_counts(hyp_seq, gold_seq, table: LabelTable):
    """b200asr_edit_counts: (per_utt [B, 4], totals [5]), int64 on the device of the ids, without a host synchronisation.

    Row b of per_utt = (cer_edits, wer_edits, gold_chars, gold_words) of hyp row b against gold row b, each joined from the
    table's labels up to its first pad id: the terms trainer/asr/trainer.py:99-104 adds to total_cer, total_wer, total_char
    and total_word.  totals = their column sums, then the first id the trainer's id2label lookup would fail on (gold rows
    first), or -1.  hyp_seq / gold_seq: [B, T] int64 or int32 CUDA tensors, any row stride."""
    ops._need_cuda(hyp_seq, gold_seq)
    if hyp_seq.dim() != 2 or gold_seq.dim() != 2 or hyp_seq.shape[0] != gold_seq.shape[0] or hyp_seq.shape[0] < 1:
        raise ValueError(f"edit_counts: hyp_seq {tuple(hyp_seq.shape)} and gold_seq {tuple(gold_seq.shape)} must be [B, T] "
                         "with the same B >= 1")
    if hyp_seq.device != gold_seq.device:
        raise ValueError("edit_counts: hyp_seq and gold_seq are on different devices")
    for t in (hyp_seq, gold_seq):
        if t.dtype not in (torch.int64, torch.int32):
            raise ValueError(f"edit_counts: ids must be int64 or int32, got {t.dtype}")
    hyp = hyp_seq if hyp_seq.stride(1) == 1 else hyp_seq.contiguous()
    gold = gold_seq if gold_seq.stride(1) == 1 else gold_seq.contiguous()
    B, T_h, T_g = hyp.shape[0], hyp.shape[1], gold.shape[1]
    off, length, cps, flags, valid = table.tensors(hyp.device)
    lib = _lib.load()
    ws = torch.empty(lib.b200asr_edit_counts_ws_bytes(B, T_h, T_g, table.max_label_len), dtype=torch.uint8,
                     device=hyp.device)
    if ws.numel() == 0:
        raise ValueError(f"edit_counts: B={B} T_h={T_h} T_g={T_g} with labels of up to {table.max_label_len} code points "
                         "are too large")
    per_utt = torch.empty(B, 4, dtype=torch.int64, device=hyp.device)
    totals = torch.empty(5, dtype=torch.int64, device=hyp.device)
    with torch.cuda.device(hyp.device):
        rc = lib.b200asr_edit_counts(_lib.ptr(hyp), int(hyp.dtype == torch.int64), hyp.stride(0), T_h, _lib.ptr(gold),
                                     int(gold.dtype == torch.int64), gold.stride(0), T_g, B, _lib.ptr(off), _lib.ptr(length),
                                     _lib.ptr(cps), _lib.ptr(flags), _lib.ptr(valid), table.V, table.max_label_len,
                                     table.pad_id, _lib.ptr(per_utt), _lib.ptr(totals), _lib.ptr(ws), ops._stream())
    _lib.check(rc, "edit_counts")
    return per_utt, totals
