"""tests/golden/beam.npz (tests/golden/make_beam_golden.py): the reference's Decoder.beam_search on a small model."""
import os

import numpy as np
import torch

from oracle import asr_oracle as O

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "beam.npz")


def load_beam_golden():
    """(cfg, id2label, cases).  Each case: dict(W, nbest, c_weight, P (decoder parameters with that case's EOS row), enc,
    ids [B, nbest, 302] (-1 padded), lengths [B, nbest] (0: no hypothesis), score, final [B, nbest] fp32)."""
    z = np.load(GOLDEN)
    c = z["meta.cfg"]
    cfg = O.OracleConfig(num_layers=int(c[0]), num_heads=int(c[1]), dim_model=int(c[2]), dim_key=int(c[3]),
                         dim_value=int(c[4]), dim_inner=int(c[5]), vocab=int(c[6]), tgt_max_len=int(c[7]),
                         freq=int(c[8]), feat_extractor="")
    id2label = {i: str(s) for i, s in enumerate(z["meta.labels"])}
    P0 = {k[len("param."):]: torch.from_numpy(z[k]) for k in z.files if k.startswith("param.")}
    cases = []
    for ci, (W, nbest, cw, B, Te, _) in enumerate(z["meta.cases"]):
        P = dict(P0)
        w = P0["decoder.output_linear.weight"].clone()
        w[2] = torch.from_numpy(z[f"c{ci}.eos_row"])
        P["decoder.output_linear.weight"] = w
        cases.append(dict(W=int(W), nbest=int(nbest), c_weight=float(cw), P=P, enc=torch.from_numpy(z[f"c{ci}.enc"]),
                          ids=torch.from_numpy(z[f"c{ci}.ids"]), lengths=torch.from_numpy(z[f"c{ci}.lengths"]),
                          score=torch.from_numpy(z[f"c{ci}.score"]), final=torch.from_numpy(z[f"c{ci}.final"])))
    return cfg, id2label, cases


def golden_yseqs(case, b):
    """The reference's n-best yseqs of utterance b (lists including SOS and the final EOS)."""
    return [case["ids"][b, i, :int(n)].tolist() for i, n in enumerate(case["lengths"][b]) if int(n) > 0]
