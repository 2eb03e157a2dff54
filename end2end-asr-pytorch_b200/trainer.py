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
"""
from __future__ import annotations

import sys

import torch

from .metrics import LabelTable, edit_counts
from .optim import clip_grads


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
        return ref(self, model, train_loader, train_sampler, valid_loader_list, opt, loss_type, start_epoch, num_epochs,
                   label2id, id2label, last_metrics)
    pad = constant.PAD_TOKEN
    p0 = next(iter(model.parameters()), None)
    if p0 is not None and p0.is_cuda:
        table.tensors(p0.device)                         # upload once, outside the loop

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
