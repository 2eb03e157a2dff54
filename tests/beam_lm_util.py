"""tests/golden/beam_lm.npz (tests/golden/make_beam_lm_golden.py): the reference's Decoder.beam_search with
lm_rescoring=True on a small model and two LSTM LMs."""
import os

import numpy as np
import torch

from oracle import asr_oracle as O

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "beam_lm.npz")


def load_beam_lm_golden():
    """(cfg, id2label, word2idx, lms, cases).  lms: dict(ntoken, ninp, nhid, nlayers, tie, P (state_dict tensors)).  Each case:
    dict(W, nbest, lm_weight, c_weight, lm (index), P (decoder parameters with the case's EOS row), enc, ended (list of dicts
    utt, yseq, score, final, lm, nw, oov, string -- every ended hypothesis in insertion order), nbest [B, nbest] (indices into
    ended, -1: none))."""
    z = np.load(GOLDEN)
    c = z["meta.cfg"]
    cfg = O.OracleConfig(num_layers=int(c[0]), num_heads=int(c[1]), dim_model=int(c[2]), dim_key=int(c[3]),
                         dim_value=int(c[4]), dim_inner=int(c[5]), vocab=int(c[6]), tgt_max_len=int(c[7]),
                         freq=int(c[8]), feat_extractor="")
    id2label = {i: str(s) for i, s in enumerate(z["meta.labels"])}
    word2idx = {str(w): i for i, w in enumerate(z["meta.words"])}
    lms = []
    j = 0
    while f"lm{j}.meta" in z.files:
        m = z[f"lm{j}.meta"]
        pre = f"lm{j}.p."
        lms.append(dict(ntoken=int(m[0]), ninp=int(m[1]), nhid=int(m[2]), nlayers=int(m[3]), tie=bool(m[4]),
                        P={k[len(pre):]: torch.from_numpy(z[k]) for k in z.files if k.startswith(pre)}))
        j += 1
    P0 = {k[len("param."):]: torch.from_numpy(z[k]) for k in z.files if k.startswith("param.")}
    cases = []
    for ci, (W, nbest, lw, cw, B, Te, _, li) in enumerate(z["meta.cases"]):
        P = dict(P0)
        w = P0["decoder.output_linear.weight"].clone()
        w[2] = torch.from_numpy(z[f"c{ci}.eos_row"])
        P["decoder.output_linear.weight"] = w
        lens = z[f"c{ci}.end_len"]
        offs = np.concatenate([[0], np.cumsum(lens)])
        ids = z[f"c{ci}.end_ids"]
        ended = [dict(utt=int(z[f"c{ci}.end_utt"][j]), yseq=ids[offs[j]:offs[j + 1]].tolist(), score=float(z[f"c{ci}.end_score"][j]),
                      final=float(z[f"c{ci}.end_final"][j]), lm=float(z[f"c{ci}.end_lm"][j]), nw=int(z[f"c{ci}.end_nw"][j]),
                      oov=int(z[f"c{ci}.end_oov"][j]), string=str(z[f"c{ci}.end_str"][j])) for j in range(len(lens))]
        cases.append(dict(W=int(W), nbest=int(nbest), lm_weight=float(lw), c_weight=float(cw), lm=int(li), P=P,
                          enc=torch.from_numpy(z[f"c{ci}.enc"]), ended=ended, nbest_idx=z[f"c{ci}.nbest"]))
    return cfg, id2label, word2idx, lms, cases
