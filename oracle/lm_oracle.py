"""CPU oracle for beam search with LM rescoring (models/asr/transformer.py:473-500, utils/lstm_utils.py:9-138).
TEST INFRASTRUCTURE ONLY.

A float64 restatement, pinned by tests/golden/beam_lm.npz (tests/golden/make_beam_lm_golden.py): the LM string of a
hypothesis, its word ids and OOV count, the LSTM language model's summed NLL (torch.nn.LSTM in float64 from a zero state),
lm_score / num_words, and the stable ranking of an utterance's ended hypotheses by final score.
"""
from __future__ import annotations

import math
import unicodedata

import torch
import torch.nn.functional as F

PAD_CHAR, SOS_CHAR, EOS_CHAR = "¶", "§", "¤"      # utils/constant.py:105-107


def _chinese(word):
    for ch in word:
        if unicodedata.category(ch) == "Lo":
            return True
    return False


def lm_string(yseq, id2label) -> str:
    """The string LM.evaluate receives from calculate_lm_score ("" means no LM call)."""
    text = "".join(id2label[int(t)] for t in yseq)
    for ch in (PAD_CHAR, SOS_CHAR, EOS_CHAR):
        text = text.replace(ch, "")
    text = text.replace("  ", " ")
    segments, cur, kind = [], None, None
    for w in text.split(" "):
        k = _chinese(w)
        if cur is None:
            cur, kind = w, k
        elif k != kind:
            segments.append((kind, cur))
            cur, kind = w, k
        else:
            cur = w if cur == "" else cur + " " + w
    segments.append((kind, cur))
    items = []
    for k, seg in segments:
        items.extend(list(seg) if k else [seg])
    res = ""
    for it in items:
        res = it if res == "" else res + " " + it
    for _ in range(2):
        res = res.replace("  ", " ")
    return res


def word_ids(string, word2idx):
    """(ids of string.split() + ['<eos>'], number of OOV words)."""
    words = string.split() + ["<eos>"]
    oov = sum(w not in word2idx for w in words)
    return [word2idx[w] if w in word2idx else word2idx["<oov>"] for w in words], oov


def lstm_nll_sum(P, ids, nlayers):
    """float64 sum over targets ids[1:] of -log p(target | ids[:t+1]) under the LSTM LM with parameters P (the state_dict of
    RNNModel: encoder.weight, rnn.weight_ih_l{k} ..., decoder.weight / bias), zero initial state."""
    x = P["encoder.weight"][torch.tensor(ids[:-1])]
    for l in range(nlayers):
        wi, wh = P[f"rnn.weight_ih_l{l}"], P[f"rnn.weight_hh_l{l}"]
        b = P[f"rnn.bias_ih_l{l}"] + P[f"rnn.bias_hh_l{l}"]
        H = wh.shape[1]
        h = torch.zeros(H, dtype=x.dtype)
        c = torch.zeros(H, dtype=x.dtype)
        outs = []
        for t in range(x.shape[0]):
            gates = wi @ x[t] + wh @ h + b
            i, f, g, o = gates[:H].sigmoid(), gates[H:2 * H].sigmoid(), gates[2 * H:3 * H].tanh(), gates[3 * H:].sigmoid()
            c = f * c + i * g
            h = o * c.tanh()
            outs.append(h)
        x = torch.stack(outs)
    logits = x @ P["decoder.weight"].T + P["decoder.bias"]
    return float(F.cross_entropy(logits, torch.tensor(ids[1:]), reduction="sum"))


def lm_score(yseq, id2label, word2idx, P, nlayers):
    """(lm_score after the OOV penalty, num_words, oov, string) of one ended hypothesis (-999, 0, 0 for an empty string)."""
    s = lm_string(yseq, id2label)
    if s == "":
        return -999.0, 0, 0, s
    ids, oov = word_ids(s, word2idx)
    n = len(ids) - 1
    return -lstm_nll_sum(P, ids, nlayers) / n + 1 - 2 * oov, n + 1, oov, s


def rank(finals, nbest):
    """Indices of the top-nbest final scores, stable (equal scores keep insertion order)."""
    return sorted(range(len(finals)), key=lambda j: finals[j], reverse=True)[:nbest]


def final_score(score, lm, num_words, lm_weight, c_weight):
    return score + lm_weight * lm + math.sqrt(num_words) * c_weight
