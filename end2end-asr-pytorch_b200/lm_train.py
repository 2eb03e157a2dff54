"""Train the LSTM language model that beam-search rescoring uses (`test.py --lm-rescoring --lm-path`) from the ASR
training manifests, on the device, and write the checkpoint the reference's `utils/lstm_utils.LM` and `b200asr.LM` load.

    python -m b200asr.lm_train --train-manifest-list train.csv [...] --valid-manifest-list valid.csv [...] \\
        --labels-path labels.json --save lm_model.pt [--emsize 200] [--nhid 200] [--nlayers 2] [--dropout 0.2] [--tied] \\
        [--lr 20] [--clip 0.25] [--epochs 40] [--batch-size 20] [--bptt 35] [--seed 1111] [--log-interval 200]

Corpus.  Each manifest line is `audio,transcript` (the format SpectrogramDataset reads); only the transcript is read.  Its
text becomes label ids exactly as SpectrogramDataset.parse_transcript makes them (utils/data_loader.py:135-141: SOS + the
lower-cased text without newlines + EOS, characters outside the label set dropped), with label2id built from
--labels-path as train.py builds it.  The words are then those calculate_lm_score asks the LM about
(utils/lstm_utils.py:9-44, restated as modules.lm_string: the special characters dropped, Chinese runs split into one word
per character), plus '<eos>'.  A transcript whose string is empty is skipped: rescoring never queries the LM for one.

Vocabulary.  '<eos>' is 0 and '<oov>' is 1 (LM.seq_to_tensor needs both); then the training words in order of first
appearance, so the same manifests give the same vocabulary.  A validation word outside it counts as '<oov>'.

Loop.  The word-language-model example that RNNModel, batchify, get_batch and repackage_hidden come from: the training
stream batchified into --batch-size columns and walked in --bptt windows with the hidden state carried across windows
(detached); per window zero_grad, RNNModel.forward (dropout included), the cross-entropy loss (ops.XentFn), backward,
clip_grad_norm_(--clip) and the SGD update p += -lr * grad (optim.sgd_step).  Every kernel of a window is this project's;
the host reads nothing back except the losses at a log interval.  After each epoch the validation loss (eval mode,
batch 10) is sum(len(window) * loss) / (len - 1); an improvement saves the checkpoint, otherwise lr /= 4.

Checkpoint.  The dict LM.__init__ reads (utils/lstm_utils.py:48-69): word2idx, idx2word, ntoken, ninp, nhid, nlayers,
dropout, tie_weights, model_state_dict -- CPU tensors and plain Python values only, so it loads under torch.load's default
weights_only=True, which the reference's LM uses.

The CLI needs the built library and an H100; it refuses to run otherwise.
"""
from __future__ import annotations

import argparse
import json
import math
import sys
import time

import torch

from . import _lib as L
from . import ops
from .modules import EOS_CHAR, PAD_CHAR, SOS_CHAR, RNNModel, lm_string
from .optim import clip_grad_norm_, sgd_step

EOS, OOV = "<eos>", "<oov>"
EVAL_BATCH_SIZE = 10


# ------------------------------------------------------------------------------------------------ corpus
def load_labels(labels_path):
    """(label2id, id2label) as train.py:44-57 builds them: PAD, SOS and EOS characters first, then the characters of the
    JSON label list, each at its first occurrence."""
    with open(labels_path) as f:
        labels = PAD_CHAR + SOS_CHAR + EOS_CHAR + str("".join(json.load(f)))
    label2id, id2label = {}, {}
    for ch in labels:
        if ch not in label2id:
            label2id[ch] = len(id2label)
            id2label[len(id2label)] = ch
    return label2id, id2label


def transcript_paths(manifests):
    """The transcript path of every line of the manifests, in order.  Blank lines are skipped; a line without a second
    comma-separated field is an error."""
    paths = []
    for m in manifests:
        with open(m) as f:
            for n, line in enumerate(f.readlines(), 1):
                fields = line.strip().split(",")
                if fields == [""]:
                    continue
                if len(fields) < 2:
                    raise ValueError(f"{m}:{n}: expected 'audio,transcript', got {line.strip()!r}")
                paths.append(fields[1])
    return paths


def parse_transcript(path, label2id):
    """SpectrogramDataset.parse_transcript (utils/data_loader.py:135-141): label ids of SOS + text + EOS, the text lower-cased
    without newlines; characters without a label -- and PAD, id 0 -- are dropped by filter(None, ...)."""
    with open(path, "r", encoding="utf8") as f:
        text = SOS_CHAR + f.read().replace("\n", "").lower() + EOS_CHAR
    return list(filter(None, [label2id.get(ch) for ch in text]))


def transcript_words(path, label2id, id2label):
    """The LM words of one transcript (its rescoring string split, then '<eos>'), or None when the string is empty."""
    s = lm_string(parse_transcript(path, label2id), id2label)
    return None if s == "" else s.split() + [EOS]


class Corpus:
    """word2idx / idx2word and the training and validation word-id streams (int64 CPU tensors)."""

    def __init__(self, train_manifests, valid_manifests, label2id, id2label):
        self.idx2word = [EOS, OOV]
        self.word2idx = {EOS: 0, OOV: 1}
        train = []
        for p in transcript_paths(train_manifests):
            for w in transcript_words(p, label2id, id2label) or ():
                if w not in self.word2idx:
                    self.word2idx[w] = len(self.idx2word)
                    self.idx2word.append(w)
                train.append(self.word2idx[w])
        valid = [self.word2idx.get(w, 1) for p in transcript_paths(valid_manifests)
                 for w in transcript_words(p, label2id, id2label) or ()]
        self.train = torch.tensor(train, dtype=torch.int64)
        self.valid = torch.tensor(valid, dtype=torch.int64)


# ------------------------------------------------------------------------------------------------ batches
def batchify(data, bsz, device=None):
    """The stream cut to a multiple of bsz and laid out as bsz columns: [len // bsz, bsz]."""
    nbatch = data.size(0) // bsz
    data = data.narrow(0, 0, nbatch * bsz).view(bsz, -1).t().contiguous()
    return data if device is None else data.to(device)


def get_batch(source, i, bptt):
    """Window i: inputs source[i : i + n] and the flattened targets source[i + 1 : i + 1 + n], n = min(bptt, len - 1 - i)."""
    seq_len = min(bptt, len(source) - 1 - i)
    return source[i:i + seq_len], source[i + 1:i + 1 + seq_len].view(-1)


def repackage_hidden(h):
    """The hidden state detached from the graph of the previous window."""
    return h.detach() if isinstance(h, torch.Tensor) else tuple(repackage_hidden(v) for v in h)


# ------------------------------------------------------------------------------------------------ loop
def train_epoch(model, data, ntokens, lr, bptt, clip, log_interval=0, epoch=1, log=print):
    """One pass over the batchified training stream `data` [len, B] (on the device).  Returns the windows' losses (0-dim
    device tensors)."""
    model.train()
    hidden = model.init_hidden(data.size(1))
    losses, logged, start = [], 0, time.time()
    n_windows = len(data) // bptt
    for batch, i in enumerate(range(0, data.size(0) - 1, bptt)):
        x, y = get_batch(data, i, bptt)
        model.zero_grad()
        hidden = repackage_hidden(hidden)
        output, hidden = model(x, hidden)
        loss = ops.XentFn.apply(output.view(-1, ntokens), y)
        loss.backward()
        clip_grad_norm_(model.parameters(), clip)
        sgd_step(model.parameters(), lr)
        losses.append(loss.detach())
        if log_interval and batch % log_interval == 0 and batch > 0:
            cur = sum(torch.stack(losses[logged:]).tolist()) / log_interval
            ms = (time.time() - start) * 1000 / log_interval
            log(f"| epoch {epoch:3d} | {batch:5d}/{n_windows:5d} batches | lr {lr:02.2f} | ms/batch {ms:5.2f} | "
                f"loss {cur:5.2f} | ppl {_ppl(cur):8.2f}")
            logged, start = len(losses), time.time()
    return losses


def evaluate(model, data, ntokens, bptt):
    """sum over windows of len(window) * mean loss, over len(data) - 1: the mean per-token loss of the batchified stream
    `data` in eval mode.  One host read, at the end."""
    model.eval()
    hidden = model.init_hidden(data.size(1))
    lens, losses = [], []
    with torch.no_grad():
        for i in range(0, data.size(0) - 1, bptt):
            x, y = get_batch(data, i, bptt)
            output, hidden = model(x, hidden)
            hidden = repackage_hidden(hidden)
            lens.append(len(x))
            losses.append(ops.XentFn.apply(output.view(-1, ntokens), y))
    return sum(n * v for n, v in zip(lens, torch.stack(losses).tolist())) / (len(data) - 1)


def lr_after_epoch(val_loss, best_val_loss, lr):
    """(save, best_val_loss, lr) after an epoch: save on the first epoch and whenever the validation loss improves,
    otherwise keep the best and divide the learning rate by 4."""
    if best_val_loss is None or val_loss < best_val_loss:
        return True, val_loss, lr
    return False, best_val_loss, lr / 4.0


def checkpoint(model, corpus, args):
    """The dict LM.__init__ reads, every tensor on the CPU and every other value a plain Python value."""
    return dict(word2idx=dict(corpus.word2idx), idx2word=list(corpus.idx2word), ntoken=len(corpus.idx2word),
                ninp=int(args.emsize), nhid=int(args.nhid), nlayers=int(args.nlayers), dropout=float(args.dropout),
                tie_weights=bool(args.tied),
                model_state_dict={k: v.detach().cpu() for k, v in model.state_dict().items()})


def _ppl(loss):
    return math.exp(loss) if loss < 700 else math.inf


def parser():
    ap = argparse.ArgumentParser(prog="python -m b200asr.lm_train",
                                 description="Train the LSTM language model for LM rescoring from ASR manifests")
    ap.add_argument("--train-manifest-list", nargs="+", required=True, help="manifests (audio,transcript lines) to train on")
    ap.add_argument("--valid-manifest-list", nargs="+", required=True, help="manifests for the validation loss")
    ap.add_argument("--labels-path", required=True, help="the label JSON of the ASR model (train.py --labels-path)")
    ap.add_argument("--save", default="model.pt", help="checkpoint path (test.py --lm-path)")
    ap.add_argument("--emsize", type=int, default=200, help="size of word embeddings")
    ap.add_argument("--nhid", type=int, default=200, help="number of hidden units per layer")
    ap.add_argument("--nlayers", type=int, default=2, help="number of layers")
    ap.add_argument("--dropout", type=float, default=0.2, help="dropout applied to layers (0 = no dropout)")
    ap.add_argument("--tied", action="store_true", help="tie the word embedding and softmax weights")
    ap.add_argument("--lr", type=float, default=20, help="initial learning rate")
    ap.add_argument("--clip", type=float, default=0.25, help="gradient clipping")
    ap.add_argument("--epochs", type=int, default=40, help="upper epoch limit")
    ap.add_argument("--batch-size", type=int, default=20, help="batch size")
    ap.add_argument("--bptt", type=int, default=35, help="sequence length")
    ap.add_argument("--seed", type=int, default=1111, help="random seed")
    ap.add_argument("--log-interval", type=int, default=200, help="report interval (windows)")
    return ap


def train(args, log=print):
    """Build the corpus, train, save the best checkpoint to args.save.  Returns the best validation loss."""
    L.load(check_device=True)
    if args.tied and args.nhid != args.emsize:
        raise ValueError("When using the tied flag, nhid must be equal to emsize")
    for name in ("batch_size", "bptt", "epochs", "emsize", "nhid", "nlayers"):
        if getattr(args, name) < 1:
            raise ValueError(f"--{name.replace('_', '-')} must be >= 1")
    label2id, id2label = load_labels(args.labels_path)
    corpus = Corpus(args.train_manifest_list, args.valid_manifest_list, label2id, id2label)
    for what, data, bsz in (("training", corpus.train, args.batch_size), ("validation", corpus.valid, EVAL_BATCH_SIZE)):
        if data.numel() < 2 * bsz:
            raise ValueError(f"the {what} corpus has {data.numel()} words; batch size {bsz} needs at least {2 * bsz}")
    ntokens = len(corpus.idx2word)
    log(f"vocabulary {ntokens} words, {corpus.train.numel()} training and {corpus.valid.numel()} validation tokens")
    dev = torch.device("cuda", torch.cuda.current_device())
    torch.manual_seed(args.seed)
    ops.manual_seed(args.seed)
    model = RNNModel("LSTM", ntokens, args.emsize, args.nhid, args.nlayers, args.dropout, args.tied).to(dev)
    train_data = batchify(corpus.train, args.batch_size, dev)
    val_data = batchify(corpus.valid, EVAL_BATCH_SIZE, dev)
    lr, best = args.lr, None
    for epoch in range(1, args.epochs + 1):
        start = time.time()
        train_epoch(model, train_data, ntokens, lr, args.bptt, args.clip, args.log_interval, epoch, log)
        val_loss = evaluate(model, val_data, ntokens, args.bptt)
        log(f"| end of epoch {epoch:3d} | time: {time.time() - start:5.2f}s | valid loss {val_loss:5.2f} | "
            f"valid ppl {_ppl(val_loss):8.2f}")
        save, best, lr = lr_after_epoch(val_loss, best, lr)
        if save:
            torch.save(checkpoint(model, corpus, args), args.save)
            log(f"saved {args.save}")
    return best


def main(argv=None):
    args = parser().parse_args(argv)
    try:
        best = train(args)
    except (RuntimeError, ValueError, OSError) as e:
        print(f"b200asr.lm_train: {e}", file=sys.stderr)
        return 1
    print(f"best validation loss {best:.4f} (ppl {_ppl(best):.2f}); checkpoint: {args.save}")
    return 0


if __name__ == "__main__":
    sys.exit(main())
