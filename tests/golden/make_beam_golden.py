#!/usr/bin/env python
"""Generate tests/golden/beam.npz from the UNMODIFIED reference's Decoder.beam_search (models/asr/transformer.py:396-517).

Run in the build container only (the GPU box has no reference checkout):

    python tests/golden/make_beam_golden.py

The other fixtures (tests/golden/make_golden.py) are not touched.  Shims (none edit the reference): the Q12 shim of
oracle/ref_shim.py (get_subsequent_mask(...).bool()), --tgt-max-len 301 (the positional table must cover 300 positions),
and a `sorted` placed in models.asr.transformer's globals that records the list beam_search sorts by final_score (:504), so
the fixture holds each returned hypothesis's fp32 score and final_score next to the yseq the reference returns.

Model: 2 layers, d = 64, V = 40, on CPU, in eval mode.  Logits are spread as in the greedy fixture, and the label map has
" ", multi-character labels and labels with inner, leading and trailing spaces, so word counts (and c_weight) matter.
Cases cover W = 1, 4, 8, nbest up to W, c_weight in {0, 0.1, 1}, utterances that end early and ones forced to end at
T_e - 1, and one T_e > 300 batch whose EOS logit is pushed down so that utterances end with no hypothesis.
"""
import builtins
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
V, WIDTH = 40, 302                        # id width: SOS + 300 tokens + EOS
# (W, nbest, c_weight, B, T_e, EOS-row scale).  With this seed the EOS row points away from the decoder states: scaled by
# about -1 EOS competes for the top ranks now and then, scaled by +3 it is the lowest logit at almost every step.
CASES = [(1, 1, 0.1, 3, 23, -1.0), (4, 2, 0.1, 3, 23, -0.9), (4, 4, 1.0, 3, 40, -0.8), (8, 3, 0.0, 3, 23, -0.9),
         (8, 8, 0.1, 2, 30, -1.0), (2, 2, 0.1, 2, 310, 3.0)]


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
    import torch
    l2i, i2l = labels(ns.constant)
    torch.manual_seed(123456)
    model = ns.functions.init_transformer_model(ns.constant.args, l2i, i2l)
    model.eval()
    g = torch.Generator().manual_seed(17)
    with torch.no_grad():
        for n, p in model.named_parameters():
            if p.dim() == 1:
                p.add_(0.1 * torch.randn(p.shape, generator=g))
        model.decoder.output_linear.weight.mul_(4.0)            # spread the logits (fewer near-ties)
    w_out = model.decoder.output_linear.weight
    eos_row = w_out[2].detach().clone()

    calls = []

    def recording_sorted(iterable, key=None, reverse=False):
        out = builtins.sorted(iterable, key=key, reverse=reverse)
        if key is not None and "final_score" in getattr(key, "__code__", compile("0", "", "eval")).co_consts:
            calls.append(out)
        return out

    ns.transformer.sorted = recording_sorted
    out = {"meta.cfg": np.array([2, 2, 64, 32, 32, 128, V, 301, 161], dtype=np.int64),
           "meta.labels": np.array([i2l[i] for i in range(V)]), "meta.cases": np.array(CASES, dtype=np.float64)}
    for n, p in model.state_dict().items():
        if n.startswith("decoder.") and not n.endswith("positional_encoding.pe"):
            out["param." + n] = p.detach().numpy().copy()
    try:
        for ci, (W, nbest, cw, B, Te, eos_scale) in enumerate(CASES):
            with torch.no_grad():
                w_out[2] = eos_row * eos_scale
            enc = torch.randn(B, Te, 64, generator=g)
            calls.clear()
            with torch.no_grad():
                ys, strs = model.decoder.beam_search(enc, beam_width=W, nbest=nbest, c_weight=cw)
            assert len(calls) == 2 * B                          # nbest_hyps and a_nbest_hyps (:504-506) per utterance
            ids = np.full((B, nbest, WIDTH), -1, dtype=np.int64)
            lengths = np.zeros((B, nbest), dtype=np.int64)
            score = np.full((B, nbest), np.nan, dtype=np.float32)
            final = np.full((B, nbest), np.nan, dtype=np.float32)
            k = 0
            for b in range(B):
                for i, h in enumerate(calls[2 * b][:nbest]):
                    y = h["yseq"]
                    assert y == ys[k] and strs[k] == "".join(i2l[t] for t in y[1:])
                    ids[b, i, :len(y)] = y
                    lengths[b, i] = len(y)
                    score[b, i] = float(h["score"])
                    final[b, i] = float(h["final_score"])
                    k += 1
            assert k == len(ys)
            out[f"c{ci}.enc"] = enc.numpy()
            out[f"c{ci}.eos_row"] = w_out[2].detach().numpy().copy()
            out[f"c{ci}.ids"], out[f"c{ci}.lengths"] = ids, lengths
            out[f"c{ci}.score"], out[f"c{ci}.final"] = score, final
            print(f"case {ci}: W={W} nbest={nbest} c_weight={cw} T_e={Te} lengths", lengths.tolist())
    finally:
        del ns.transformer.sorted
    path = os.path.join(HERE, "beam.npz")
    np.savez_compressed(path, **out)
    print("->", path, "%.1f KB" % (os.path.getsize(path) / 1024))


if __name__ == "__main__":
    main()
