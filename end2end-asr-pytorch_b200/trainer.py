"""Trainer.train (trainer/asr/trainer.py:21-213) with the CER / WER counts on the device.

The reference builds a gold and a hypothesis string per utterance with two `int(x)` per token -- a device-to-host copy and a
stream synchronisation each -- and takes their edit distances on the host.  trainer_train keeps the reference's loop, its
skips, its prints, logging lines, progress-bar texts, metrics and checkpoints, but gets the four sums it adds up per batch
(CER and WER edits, gold characters and words) from b200asr_edit_counts (metrics.edit_counts) in one read of a [5] row:
  * training: the row is read before the loss, because an id missing from id2label skips the batch before the loss is
    computed (:60-79); the loss is then read once, for the infinity check (:87) and for total_loss (:113);
  * validation: the loss comes first there (:145-151), so the loss and the row are read in one copy.
With --clip, the gradients are clipped by optim.clip_grad_norm_ on the device when every gradient is an fp32 CUDA tensor on
one device, by torch.nn.utils.clip_grad_norm_ otherwise (:108-109).
A batch with an id missing from id2label, or whose ids are not [B, T] integer CUDA tensors, builds its strings on the host
exactly as the reference does, which prints the same exception.

calculate_metrics, save_model, tqdm, constant, logging and Variable are looked up in the trainer module's globals at each use,
as the reference's own code resolves them.  The reference's train runs instead when id2label is not a dict of str labels
(metrics.LabelTable), when SOS_CHAR or EOS_CHAR is not a single code point, or when the trainer module's calculate_cer /
calculate_wer are not utils.metrics's.

Data-parallel (after install() joined a process group, parallel.join): the same loop on every rank, restating the
reference's --parallel (nn.DataParallel) semantics -- see _train_parallel.
"""
from __future__ import annotations

import contextlib
import sys

import numpy as np

import torch
import torch.distributed as dist

from . import _lib as L
from . import metrics, parallel
from .metrics import LabelTable, edit_counts
from .optim import FlatParams, clip_grads


def _device_totals(hyp_seq, gold_seq, table):
    """The [5] int64 totals row of edit_counts, or None when the batch takes the host path."""
    ids = (torch.int64, torch.int32)
    if not (torch.is_tensor(hyp_seq) and torch.is_tensor(gold_seq) and hyp_seq.is_cuda and gold_seq.is_cuda and
            hyp_seq.device == gold_seq.device and hyp_seq.dim() == 2 and gold_seq.dim() == 2 and
            hyp_seq.shape[0] == gold_seq.shape[0] >= 1 and hyp_seq.dtype in ids and gold_seq.dtype in ids):
        return None
    return edit_counts(hyp_seq, gold_seq, table)[1]


def _host_strings(gold_seq, hyp_seq, id2label, pad):
    """trainer.py:61-75 on host copies of the ids: (strs_gold, strs_hyps), raising where the reference raises."""
    gold_seq = gold_seq.cpu() if torch.is_tensor(gold_seq) else gold_seq
    hyp_seq = hyp_seq.cpu() if torch.is_tensor(hyp_seq) else hyp_seq

    def join(ut):
        s = ""
        for x in ut:
            if int(x) == pad:
                break
            s = s + id2label[int(x)]
        return s

    strs_gold = [join(ut) for ut in gold_seq]
    strs_hyps = [join(ut) for ut in hyp_seq]
    return strs_gold, strs_hyps


def _host_counts(strs_hyps, strs_gold, G):
    """trainer.py:96-104: (cer, wer, char, word) summed over the utterances."""
    constant = G["constant"]
    cer_sum, wer_sum, n_char, n_word = 0, 0, 0, 0
    for j in range(len(strs_hyps)):
        h = strs_hyps[j].replace(constant.SOS_CHAR, "").replace(constant.EOS_CHAR, "")
        g = strs_gold[j].replace(constant.SOS_CHAR, "").replace(constant.EOS_CHAR, "")
        cer_sum += G["calculate_cer"](h.replace(" ", ""), g.replace(" ", ""))
        wer_sum += G["calculate_wer"](h, g)
        n_char += len(g.replace(" ", ""))
        n_word += len(g.split(" "))
    return cer_sum, wer_sum, n_char, n_word


def _nan_predictions(G, e):
    print(e)
    G["logging"].info("NaN predictions")


def trainer_train(self, model, train_loader, train_sampler, valid_loader_list, opt, loss_type, start_epoch, num_epochs,
                  label2id, id2label, last_metrics=None):
    """Trainer.train with the string metrics on the device (module docstring)."""
    from .install import original
    ref = original(type(self), "train")
    if ref is None:
        raise RuntimeError("b200asr trainer_train: Trainer.train is not installed (b200asr.install())")
    G = ref.__globals__                                  # trainer/asr/trainer.py's module namespace, read at each use
    constant = G["constant"]
    um = sys.modules.get("utils.metrics")
    try:
        if um is None or G.get("calculate_cer") is not um.calculate_cer or G.get("calculate_wer") is not um.calculate_wer:
            raise ValueError("the trainer's calculate_cer / calculate_wer are not utils.metrics's")
        table = LabelTable(id2label, constant.PAD_TOKEN, (constant.SOS_CHAR, constant.EOS_CHAR))
    except (TypeError, ValueError):
        if parallel.joined() is not None:
            raise
        return ref(self, model, train_loader, train_sampler, valid_loader_list, opt, loss_type, start_epoch, num_epochs,
                   label2id, id2label, last_metrics)
    pad = constant.PAD_TOKEN
    p0 = next(iter(model.parameters()), None)
    if p0 is not None and p0.is_cuda:
        table.tensors(p0.device)                         # upload once, outside the loop
    if parallel.joined() is not None:
        return _train_parallel(G, table, parallel.joined(), model, train_loader, train_sampler, valid_loader_list, opt,
                               loss_type, start_epoch, num_epochs, label2id, id2label, last_metrics)

    history = []
    best_valid_loss = 1000000000 if last_metrics is None else last_metrics['valid_loss']
    smoothing = constant.args.label_smoothing

    G["logging"].info("name " + constant.args.name)

    for epoch in range(start_epoch, num_epochs):
        sys.stdout.flush()
        total_loss, total_cer, total_wer, total_char, total_word = 0, 0, 0, 0, 0

        G["logging"].info("TRAIN")
        model.train()
        pbar = G["tqdm"](iter(train_loader), leave=True, total=len(train_loader))
        for i, (data) in enumerate(pbar, start=0):
            src, tgt, src_percentages, src_lengths, tgt_lengths = data

            if constant.USE_CUDA:
                src = src.cuda()
                tgt = tgt.cuda()

            opt.zero_grad()

            pred, gold, hyp_seq, gold_seq = model(src, src_lengths, tgt, verbose=False)

            totals = _device_totals(hyp_seq, gold_seq, table)
            counts = None
            if totals is not None:
                t = totals.tolist()
                if t[4] == -1:
                    counts = t[:4]
            if counts is None:
                try:
                    strs_gold, strs_hyps = _host_strings(gold_seq, hyp_seq, id2label, pad)
                except Exception as e:
                    _nan_predictions(G, e)
                    continue

            seq_length = pred.size(1)
            sizes = G["Variable"](src_percentages.mul_(int(seq_length)).int(), requires_grad=False)

            loss, num_correct = G["calculate_metrics"](
                pred, gold, input_lengths=sizes, target_lengths=tgt_lengths, smoothing=smoothing, loss_type=loss_type)

            loss_value = loss.item()
            if loss_value == float('Inf'):
                G["logging"].info("Found infinity loss, masking")
                continue

            if counts is None:
                counts = _host_counts(strs_hyps, strs_gold, G)
            total_cer += counts[0]
            total_wer += counts[1]
            total_char += counts[2]
            total_word += counts[3]

            loss.backward()

            if constant.args.clip:
                clip_grads(model.parameters(), constant.args.max_norm)

            opt.step()

            total_loss += loss_value

            pbar.set_description("(Epoch {}) TRAIN LOSS:{:.4f} CER:{:.2f}% LR:{:.7f}".format(
                (epoch+1), total_loss/(i+1), total_cer*100/total_char, opt._rate))
        G["logging"].info("(Epoch {}) TRAIN LOSS:{:.4f} CER:{:.2f}% LR:{:.7f}".format(
            (epoch+1), total_loss/(len(train_loader)), total_cer*100/total_char, opt._rate))

        # evaluate
        print("")
        G["logging"].info("VALID")
        model.eval()

        for ind in range(len(valid_loader_list)):
            valid_loader = valid_loader_list[ind]

            total_valid_loss, total_valid_cer, total_valid_wer, total_valid_char, total_valid_word = 0, 0, 0, 0, 0
            valid_pbar = G["tqdm"](iter(valid_loader), leave=True, total=len(valid_loader))
            for i, (data) in enumerate(valid_pbar):
                src, tgt, src_percentages, src_lengths, tgt_lengths = data

                if constant.USE_CUDA:
                    src = src.cuda()
                    tgt = tgt.cuda()

                with torch.no_grad():
                    pred, gold, hyp_seq, gold_seq = model(src, src_lengths, tgt, verbose=False)

                seq_length = pred.size(1)
                sizes = G["Variable"](src_percentages.mul_(int(seq_length)).int(), requires_grad=False)

                loss, num_correct = G["calculate_metrics"](
                    pred, gold, input_lengths=sizes, target_lengths=tgt_lengths, smoothing=smoothing, loss_type=loss_type)

                totals = _device_totals(hyp_seq, gold_seq, table)
                counts = None
                if (totals is not None and torch.is_tensor(loss) and loss.numel() == 1 and loss.is_floating_point() and
                        loss.device == totals.device):
                    # one copy: float64 holds the float loss exactly, and the counts (far below 2^53) too
                    t = torch.cat([totals.to(torch.float64), loss.detach().reshape(1).to(torch.float64)]).tolist()
                    loss_value = t[5]
                    if t[4] == -1:
                        counts = [int(v) for v in t[:4]]
                else:
                    loss_value = loss.item()
                    if totals is not None:
                        t = totals.tolist()
                        if t[4] == -1:
                            counts = t[:4]

                if loss_value == float('Inf'):
                    G["logging"].info("Found infinity loss, masking")
                    continue

                if counts is None:
                    try:
                        strs_gold, strs_hyps = _host_strings(gold_seq, hyp_seq, id2label, pad)
                    except Exception as e:
                        _nan_predictions(G, e)
                        continue
                    counts = _host_counts(strs_hyps, strs_gold, G)
                total_valid_cer += counts[0]
                total_valid_wer += counts[1]
                total_valid_char += counts[2]
                total_valid_word += counts[3]

                total_valid_loss += loss_value
                valid_pbar.set_description("VALID SET {} LOSS:{:.4f} CER:{:.2f}%".format(ind,
                    total_valid_loss/(i+1), total_valid_cer*100/total_valid_char))
            G["logging"].info("VALID SET {} LOSS:{:.4f} CER:{:.2f}%".format(ind,
                    total_valid_loss/(len(valid_loader)), total_valid_cer*100/total_valid_char))

        metrics = {}
        metrics["train_loss"] = total_loss / len(train_loader)
        metrics["valid_loss"] = total_valid_loss / (len(valid_loader))
        metrics["train_cer"] = total_cer
        metrics["train_wer"] = total_wer
        metrics["valid_cer"] = total_valid_cer
        metrics["valid_wer"] = total_valid_wer
        metrics["history"] = history
        history.append(metrics)

        if epoch % constant.args.save_every == 0:
            G["save_model"](model, (epoch+1), opt, metrics,
                            label2id, id2label, best_model=False)

        # save the best model
        if best_valid_loss > total_valid_loss/len(valid_loader):
            best_valid_loss = total_valid_loss/len(valid_loader)
            G["save_model"](model, (epoch+1), opt, metrics,
                            label2id, id2label, best_model=True)

        if constant.args.shuffle:
            G["logging"].info("SHUFFLE")
            print("SHUFFLE")
            train_sampler.shuffle(epoch)


# ---------------------------------------------------------------------------------------------- data-parallel training
# One row per batch and rank, summed over the ranks by one all-reduce before anything is decided:
ROW = ("loss_sum", "normaliser", "cer", "wer", "char", "word", "missing")


def loss_value(row):
    """The reference's batch loss from the reduced row: the sum over the gathered batch / its normaliser (CE: the non-PAD
    tokens, label-smoothed or not, utils/metrics.py:102-131; CTC: the utterances, reduction="mean" of F.ctc_loss)."""
    return row[0] / row[1] if row[1] else float("nan")


def _shard_loss(pred, gold, sizes, tgt_lengths, smoothing, loss_type):
    """(loss to back-propagate, [2] device tensor (its value, normaliser)).  CE: the un-normalised token sum.  CTC: the
    shard's mean times its B, so that the sum over the ranks / the global B is reduction="mean" over the gathered batch."""
    if loss_type == "ce":
        loss_sum, stats = metrics.loss_and_stats(pred, gold, smoothing, reduction="sum")
        return loss_sum, stats[0:2]
    if loss_type == "ctc":
        B = pred.shape[0]
        loss_sum = metrics.calculate_loss(pred, gold, sizes, tgt_lengths, smoothing, loss_type) * B
        return loss_sum, torch.stack([loss_sum.detach().float(), loss_sum.new_tensor(float(B))])
    raise NotImplementedError(f"b200asr implements the 'ce' and 'ctc' losses only, not {loss_type!r}")


def _quiet(*a, **k):
    pass


class _NoBar:
    """The progress bar of a rank other than 0: iterates, draws nothing."""

    def __init__(self, it, leave=True, total=None):
        self.it = it

    def __iter__(self):
        return iter(self.it)

    def set_description(self, s):
        pass


class _Rank:
    """Per-rank state of the data-parallel loop: the flat gradient buffer, its all-reduce, the reduced row."""

    def __init__(self, G, table, group, model, id2label):
        self.G, self.table, self.model, self.id2label = G, table, model, id2label
        self.pg, self.rank, self.world = group
        self.lead = self.rank == 0
        flat = getattr(model, "_b200_flat", None)
        if flat is None:
            # parameters and their gradients become views of two flat buffers: names, state_dict and the optimizer's
            # parameter list and state are unchanged, the gradient all-reduce is one buffer
            flat = FlatParams(model, extra=0)
            model._b200_flat = flat
        self.flat = flat
        self.reducer = parallel.GradAllReduce(flat, self.pg)
        self.dev = flat.flat.device
        self.scale = torch.zeros(2, device=self.dev, dtype=torch.float32)
        parallel.broadcast_params(flat, self.pg)
        parallel.broadcast_module_state(model, flat, self.pg)
        parallel.seed_host_rngs(self.pg)
        parallel.fold_rank_into_dropout(self.rank)
        self.log = G["logging"].info if self.lead else _quiet
        self.say = print if self.lead else _quiet

    def shard(self, data):
        src, tgt, src_percentages, src_lengths, tgt_lengths = data
        a, b = parallel.shard_range(src.shape[0], self.rank, self.world)
        return tuple(t[a:b] for t in (src, tgt, src_percentages, src_lengths, tgt_lengths))

    def row(self, model, data, smoothing, loss_type, pad, no_grad):
        """Forward and loss of this rank's shard; the row reduced over the ranks (host list), the shard's loss and its
        (gold_seq, hyp_seq) -- None for an empty shard."""
        src, tgt, src_percentages, src_lengths, tgt_lengths = self.shard(data)
        row = torch.zeros(len(ROW), device=self.dev, dtype=torch.float64)
        loss, seqs = None, None
        if src.shape[0]:
            G = self.G
            if G["constant"].USE_CUDA:
                src = src.cuda()
                tgt = tgt.cuda()
            with torch.no_grad() if no_grad else contextlib.nullcontext():
                pred, gold, hyp_seq, gold_seq = model(src, src_lengths, tgt, verbose=False)
            seqs = (gold_seq, hyp_seq)
            sizes = G["Variable"](src_percentages.mul_(int(pred.size(1))).int(), requires_grad=False)
            loss, terms = _shard_loss(pred, gold, sizes, tgt_lengths, smoothing, loss_type)
            row[0:2] = terms
            totals = _device_totals(hyp_seq, gold_seq, self.table)
            if totals is not None:
                row[2:6] = totals[:4]
                row[6:7] = (totals[4:5] != -1)
            else:
                try:
                    strs_gold, strs_hyps = _host_strings(gold_seq, hyp_seq, self.id2label, pad)
                    row[2:6] = torch.tensor(_host_counts(strs_hyps, strs_gold, G), dtype=torch.float64)
                except Exception:
                    row[6] = 1
        dist.all_reduce(row, op=dist.ReduceOp.SUM, group=self.pg)
        return row.tolist(), loss, seqs

    def missing(self, seqs, pad):
        """A batch with an id missing from id2label on some rank: rank 0 prints what the reference prints for the gathered
        batch (the first failing lookup, gold rows first) and logs it."""
        part = None if seqs is None else tuple(t.cpu() if torch.is_tensor(t) else t for t in seqs)
        parts = [None] * self.world
        dist.all_gather_object(parts, part, group=self.pg)
        if self.lead:
            gold = [r for p in parts if p is not None for r in p[0]]
            hyp = [r for p in parts if p is not None for r in p[1]]
            try:
                _host_strings(gold, hyp, self.id2label, pad)
                e = KeyError("id missing from id2label")
            except Exception as exc:
                e = exc
            _nan_predictions(self.G, e)

    def step(self, loss, normaliser, clip, max_norm, opt):
        """Backward of the shard's un-normalised loss with the one gradient all-reduce, the 1 / global normaliser scale on
        the device, --clip over the global gradient and the bound NoamOpt.step."""
        if loss is not None:
            self.reducer.backward(loss)
            self.flat.ensure_grad_views()
        self.reducer.finish()
        f, stream = self.flat, torch.cuda.current_stream(self.dev).cuda_stream
        n = torch.full((1,), float(normaliser), device=self.dev, dtype=torch.float32)
        lib = L.load()
        L.check(lib.b200asr_grad_scale(None, f.numel, L.ptr(n), 0.0, None, L.ptr(self.scale), stream), "grad_scale")
        ptrs = np.array([f.flat_grad.data_ptr()], dtype=np.uint64)
        numel = np.array([f.numel], dtype=np.int64)
        L.check(lib.b200asr_scale_multi(ptrs.ctypes.data, numel.ctypes.data, 1, L.ptr(self.scale), stream), "scale_multi")
        torch._C._increment_version([f.flat_grad])
        if clip:
            clip_grads(self.model.parameters(), max_norm)
        opt.step()


def _train_parallel(G, table, group, model, train_loader, train_sampler, valid_loader_list, opt, loss_type, start_epoch,
                    num_epochs, label2id, id2label, last_metrics):
    """Trainer.train across the ranks of `group`, as the reference's --parallel would train on the gathered batch.

    Every rank's loader yields the global batch: at the start, rank 0 broadcasts a seed for Python's `random`, numpy's
    global generator and torch's CPU generator (parallel.seed_host_rngs), from which the reference's BucketingSampler, its
    SpectrogramDataset and the DataLoader draw the data order.  Rank r takes chunk r of each batch as
    nn.DataParallel.scatter does (parallel.shard_range; an empty shard still joins every collective with zeros).  Per
    training batch:
      * forward and loss of the shard, the un-normalised loss (_shard_loss), the CER / WER counts on the device;
      * ONE all-reduce of the row ROW -- every rank then takes the reference's skips identically: an id missing from
        id2label on any shard (:60-79), an infinite loss of the gathered batch (:87-90);
      * backward with ONE all-reduce of the flat gradient buffer (its head issued under the front end's backward,
        parallel.GradAllReduce), the scale 1 / global normaliser on the device (b200asr_grad_scale, b200asr_scale_multi),
        --clip over the global gradient (optim.clip_grads), the bound NoamOpt.step (torch Adam's state).
    Validation: one all-reduce of the row per batch.  Rank 0's parameters, frozen parameters and buffers are broadcast at
    the start (parallel.broadcast_params, broadcast_module_state); dropout draws differ per rank; from then on BatchNorm
    running statistics stay per rank.  Only rank 0 logs, draws progress bars, prints and calls
    save_model (rank 0's BatchNorm statistics are saved, as nn.DataParallel keeps device 0's); the metrics, and so the
    best-model decision, are the same on every rank.  The loss is computed by metrics.loss_and_stats (CE) and
    metrics.calculate_loss (CTC), not through the trainer module's calculate_metrics."""
    constant = G["constant"]
    if not constant.USE_CUDA:
        raise ValueError("b200asr data-parallel Trainer.train needs --cuda")
    r = _Rank(G, table, group, model, id2label)
    log, say = r.log, r.say
    tqdm = G["tqdm"] if r.lead else _NoBar
    pad = constant.PAD_TOKEN

    history = []
    best_valid_loss = 1000000000 if last_metrics is None else last_metrics['valid_loss']
    smoothing = constant.args.label_smoothing

    log("name " + constant.args.name)

    for epoch in range(start_epoch, num_epochs):
        sys.stdout.flush()
        total_loss, total_cer, total_wer, total_char, total_word = 0, 0, 0, 0, 0

        log("TRAIN")
        model.train()
        pbar = tqdm(iter(train_loader), leave=True, total=len(train_loader))
        for i, (data) in enumerate(pbar, start=0):
            r.flat.zero_grad()                           # opt.zero_grad(), keeping the gradients views of the flat buffer
            t, loss, seqs = r.row(model, data, smoothing, loss_type, pad, no_grad=False)
            if t[6]:
                r.missing(seqs, pad)
                continue
            value = loss_value(t)
            if value == float('Inf'):
                log("Found infinity loss, masking")
                continue

            total_cer += int(t[2])
            total_wer += int(t[3])
            total_char += int(t[4])
            total_word += int(t[5])

            r.step(loss, t[1], constant.args.clip, constant.args.max_norm, opt)

            total_loss += value

            pbar.set_description("(Epoch {}) TRAIN LOSS:{:.4f} CER:{:.2f}% LR:{:.7f}".format(
                (epoch+1), total_loss/(i+1), total_cer*100/total_char, opt._rate))
        log("(Epoch {}) TRAIN LOSS:{:.4f} CER:{:.2f}% LR:{:.7f}".format(
            (epoch+1), total_loss/(len(train_loader)), total_cer*100/total_char, opt._rate))

        # evaluate
        say("")
        log("VALID")
        model.eval()

        for ind in range(len(valid_loader_list)):
            valid_loader = valid_loader_list[ind]

            total_valid_loss, total_valid_cer, total_valid_wer, total_valid_char, total_valid_word = 0, 0, 0, 0, 0
            valid_pbar = tqdm(iter(valid_loader), leave=True, total=len(valid_loader))
            for i, (data) in enumerate(valid_pbar):
                t, _, seqs = r.row(model, data, smoothing, loss_type, pad, no_grad=True)
                value = loss_value(t)
                if value == float('Inf'):
                    log("Found infinity loss, masking")
                    continue
                if t[6]:
                    r.missing(seqs, pad)
                    continue
                total_valid_cer += int(t[2])
                total_valid_wer += int(t[3])
                total_valid_char += int(t[4])
                total_valid_word += int(t[5])

                total_valid_loss += value
                valid_pbar.set_description("VALID SET {} LOSS:{:.4f} CER:{:.2f}%".format(ind,
                    total_valid_loss/(i+1), total_valid_cer*100/total_valid_char))
            log("VALID SET {} LOSS:{:.4f} CER:{:.2f}%".format(ind,
                    total_valid_loss/(len(valid_loader)), total_valid_cer*100/total_valid_char))

        metrics_ = {}
        metrics_["train_loss"] = total_loss / len(train_loader)
        metrics_["valid_loss"] = total_valid_loss / (len(valid_loader))
        metrics_["train_cer"] = total_cer
        metrics_["train_wer"] = total_wer
        metrics_["valid_cer"] = total_valid_cer
        metrics_["valid_wer"] = total_valid_wer
        metrics_["history"] = history
        history.append(metrics_)

        if epoch % constant.args.save_every == 0 and r.lead:
            G["save_model"](model, (epoch+1), opt, metrics_,
                            label2id, id2label, best_model=False)

        # save the best model
        if best_valid_loss > total_valid_loss/len(valid_loader):
            best_valid_loss = total_valid_loss/len(valid_loader)
            if r.lead:
                G["save_model"](model, (epoch+1), opt, metrics_,
                                label2id, id2label, best_model=True)

        if constant.args.shuffle:
            log("SHUFFLE")
            say("SHUFFLE")
            train_sampler.shuffle(epoch)
