#!/usr/bin/env python
"""Generate tests/golden/beam_lm.npz from the UNMODIFIED reference's Decoder.beam_search with lm_rescoring=True
(models/asr/transformer.py:396-517, utils/lstm_utils.py).

Needs the reference checkout (found by oracle/ref_shim.py); runs on CPU:

    python tests/golden/make_beam_lm_golden.py

The other fixtures are not touched.  Shims (none edit the reference): the Q12 shim of oracle/ref_shim.py, --tgt-max-len 301,
and three recorders placed in models.asr.transformer's globals and on the LM object:
  * `calculate_lm_score` is wrapped, so every ended hypothesis is recorded in insertion order with its yseq and the
    (lm_score, num_words, oov) the reference computed;
  * the LM's `evaluate` is wrapped, so the string the LM scored is recorded next to it (none for an empty string);
  * `sorted` records the list beam_search ranks by final_score (:499), which gives each hypothesis's fp32 score and
    final_score and the n-best order.

Model: the 2-layer d = 64 decoder of make_beam_golden.py with its label map (CJK, Latin, " ", multi-character labels).  Two
LSTM LMs from the reference's own RNNModel: 2 layers, ninp 32, nhid 50, untied; and 1 layer, ninp = nhid = 40, tied.  Their
vocabulary holds only some of the label map's words, so OOV words occur.  Cases cover W = 1, 4, 8, lm_weight 0, 0.1 and 5,
c_weight 0 and 1, forced endings (T_e = 6) and hypotheses whose LM string is empty (EOS pushed up).  The script asserts
that these all occur and that the LM changes the n-best against the reference's non-LM ranking in at least one case.
"""
import builtins
import os
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
V = 40
# (W, nbest, lm_weight, c_weight, B, T_e, EOS-row scale, LM index)
CASES = [(1, 1, 0.1, 1.0, 3, 23, -1.0, 0), (4, 4, 0.1, 1.0, 3, 23, -0.9, 0), (4, 2, 5.0, 0.0, 3, 23, -0.9, 1),
         (8, 8, 0.0, 0.0, 2, 23, -1.0, 0), (8, 4, 5.0, 1.0, 2, 30, -1.0, 1), (4, 4, 0.1, 1.0, 3, 6, -2.5, 0)]
LMS = [dict(ninp=32, nhid=50, nlayers=2, tie=False), dict(ninp=40, nhid=40, nlayers=1, tie=True)]
WORDS = ["<eos>", "<oov>", "ab", "c", "d", "e", "f", "ef"] + [chr(0x4E00 + i) for i in range(0, 32, 2)]


def labels(constant):
    chars = [constant.PAD_CHAR, constant.SOS_CHAR, constant.EOS_CHAR, " ", "ab", "c d", " e", "f "]
    chars += [chr(0x4E00 + i) for i in range(V - len(chars))]
    return {c: i for i, c in enumerate(chars)}, {i: c for i, c in enumerate(chars)}


def main():
    sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
    from oracle import ref_shim
    ns = ref_shim.load(["--num-layers", "2", "--num-heads", "2", "--dim-model", "64", "--dim-emb", "64", "--dim-key", "32",
                        "--dim-value", "32", "--dim-inner", "128", "--feat_extractor", "", "--tgt-max-len", "301",
                        "--dropout", "0.0"], q12_shim=True)
    import importlib

    import torch
    lstm_utils = importlib.import_module("utils.lstm_utils")
    l2i, i2l = labels(ns.constant)
    torch.manual_seed(123456)
    model = ns.functions.init_transformer_model(ns.constant.args, l2i, i2l)
    model.eval()
    g = torch.Generator().manual_seed(17)
    with torch.no_grad():
        for n, p in model.named_parameters():
            if p.dim() == 1:
                p.add_(0.1 * torch.randn(p.shape, generator=g))
        model.decoder.output_linear.weight.mul_(4.0)
    w_out = model.decoder.output_linear.weight
    eos_row = w_out[2].detach().clone()

    out = {"meta.cfg": np.array([2, 2, 64, 32, 32, 128, V, 301, 161], dtype=np.int64),
           "meta.labels": np.array([i2l[i] for i in range(V)]), "meta.cases": np.array(CASES, dtype=np.float64),
           "meta.words": np.array(WORDS)}
    for n, p in model.state_dict().items():
        if n.startswith("decoder.") and not n.endswith("positional_encoding.pe"):
            out["param." + n] = p.detach().numpy().copy()

    tmp = tempfile.mkdtemp()
    lms = []
    w2i = {w: i for i, w in enumerate(WORDS)}
    for j, spec in enumerate(LMS):
        torch.manual_seed(1000 + j)
        rnn = lstm_utils.RNNModel("LSTM", len(WORDS), spec["ninp"], spec["nhid"], spec["nlayers"], dropout=0.0,
                                  tie_weights=spec["tie"])
        with torch.no_grad():                      # weights large enough that the LM's scores differ between strings
            for n, p in rnn.named_parameters():
                p.copy_(0.5 * torch.randn(p.shape, generator=g))
        path = os.path.join(tmp, f"lm{j}.pt")
        torch.save(dict(word2idx=w2i, idx2word=WORDS, ntoken=len(WORDS), ninp=spec["ninp"], nhid=spec["nhid"],
                        nlayers=spec["nlayers"], dropout=0.0, tie_weights=spec["tie"], model_state_dict=rnn.state_dict()), path)
        lm = lstm_utils.LM(path)
        lms.append(lm)
        out[f"lm{j}.meta"] = np.array([len(WORDS), spec["ninp"], spec["nhid"], spec["nlayers"], int(spec["tie"])], dtype=np.int64)
        for n, p in lm.model.state_dict().items():
            out[f"lm{j}.p.{n}"] = p.detach().numpy().copy()

    ended, ranked, current = [], [], {}

    def recording_sorted(iterable, key=None, reverse=False):
        res = builtins.sorted(iterable, key=key, reverse=reverse)
        if key is not None and "final_score" in getattr(key, "__code__", compile("0", "", "eval")).co_consts:
            ranked.append([(id(h["yseq"]), float(h["score"]), float(h["final_score"])) for h in res])
        return res

    orig_calc = ns.transformer.calculate_lm_score

    def recording_calc(seq, lm, id2label):
        current.clear()
        lm_score, num_words, oov = orig_calc(seq, lm, id2label)
        ended.append(dict(key=id(seq), yseq=seq[0].tolist(), lm=float(lm_score), nw=int(num_words), oov=int(oov),
                          string=current.get("s", "")))
        return lm_score, num_words, oov

    for lm in lms:
        ev = lm.evaluate

        def recording_evaluate(seq, ev=ev):
            current["s"] = seq
            return ev(seq)

        lm.evaluate = recording_evaluate

    ns.transformer.sorted = recording_sorted
    ns.transformer.calculate_lm_score = recording_calc
    changed = forced = empty = oov_seen = 0
    try:
        for ci, (W, nbest, lw, cw, B, Te, eos_scale, li) in enumerate(CASES):
            W, nbest, B, Te, li = int(W), int(nbest), int(B), int(Te), int(li)
            with torch.no_grad():
                w_out[2] = eos_row * eos_scale
            enc = torch.randn(B, Te, 64, generator=g)
            ut, ids, lens, sc, fin, lmv, nw, oov, strs = [], [], [], [], [], [], [], [], []
            nb = np.full((B, nbest), -1, dtype=np.int64)
            for b in range(B):                      # one utterance per call: the recorders then see one utterance
                ended.clear(); ranked.clear()
                with torch.no_grad():
                    ys, _ = model.decoder.beam_search(enc[b:b + 1], beam_width=W, nbest=nbest, lm_rescoring=True, lm=lms[li],
                                                      lm_weight=lw, c_weight=cw)
                    assert len(ranked) == 2 and len(ranked[0]) == len(ended)
                    ys0, _ = model.decoder.beam_search(enc[b:b + 1], beam_width=W, nbest=nbest, c_weight=cw)
                changed += ys != ys0
                by_key = {k: (s, f) for k, s, f in ranked[0]}
                base = len(ut)
                for h in ended:
                    s, f = by_key[h["key"]]
                    ut.append(b); ids += h["yseq"]; lens.append(len(h["yseq"])); sc.append(s); fin.append(f)
                    lmv.append(h["lm"]); nw.append(h["nw"]); oov.append(h["oov"]); strs.append(h["string"])
                    forced += len(h["yseq"]) == Te + 2
                    empty += h["lm"] == -999
                    oov_seen += h["oov"] > 0
                pos = {h["key"]: base + i for i, h in enumerate(ended)}
                for i, (k, _, _) in enumerate(ranked[0][:nbest]):
                    nb[b, i] = pos[k]
                assert ys == [ended[pos[k] - base]["yseq"] for k, _, _ in ranked[0][:nbest]]
            out[f"c{ci}.enc"] = enc.numpy()
            out[f"c{ci}.eos_row"] = w_out[2].detach().numpy().copy()
            out[f"c{ci}.end_utt"] = np.array(ut, dtype=np.int64)
            out[f"c{ci}.end_ids"] = np.array(ids, dtype=np.int64)
            out[f"c{ci}.end_len"] = np.array(lens, dtype=np.int64)
            out[f"c{ci}.end_score"] = np.array(sc, dtype=np.float32)
            out[f"c{ci}.end_final"] = np.array(fin, dtype=np.float32)
            out[f"c{ci}.end_lm"] = np.array(lmv, dtype=np.float64)
            out[f"c{ci}.end_nw"] = np.array(nw, dtype=np.int64)
            out[f"c{ci}.end_oov"] = np.array(oov, dtype=np.int64)
            out[f"c{ci}.end_str"] = np.array(strs)
            out[f"c{ci}.nbest"] = nb
            print(f"case {ci}: W={W} nbest={nbest} lm_weight={lw} c_weight={cw} T_e={Te} LM {li}: {len(ut)} ended")
    finally:
        del ns.transformer.sorted
        ns.transformer.calculate_lm_score = orig_calc
    print(f"n-best changed by the LM in {changed} utterances; forced {forced}, empty {empty}, with OOV {oov_seen}")
    assert changed and forced and empty and oov_seen
    path = os.path.join(HERE, "beam_lm.npz")
    np.savez_compressed(path, **out)
    print("->", path, "%.1f KB" % (os.path.getsize(path) / 1024))


if __name__ == "__main__":
    main()
