"""CPU oracle for Decoder.beam_search without LM rescoring (models/asr/transformer.py:396-517).  TEST INFRASTRUCTURE ONLY.

A float64 restatement of the reference's search, pinned by tests/golden/beam.npz (generated from the live reference by
tests/golden/make_beam_golden.py).  It re-decodes every live hypothesis's whole prefix at every step, as the reference does,
but batches an utterance's live hypotheses into one decoder call.  The blocks are those of oracle/asr_oracle.py.
"""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F

from oracle.asr_oracle import EOS, PAD, SOS, OracleConfig, conv_ffn, multi_head_attention, sinusoid_table

PAD_CHAR, SOS_CHAR, EOS_CHAR = "¶", "§", "¤"      # utils/constant.py:105-107


def num_words(yseq, id2label) -> int:
    """transformer.py:490-492: words of the joined labels with the PAD/SOS/EOS characters removed."""
    s = "".join(id2label[t] for t in yseq).replace(PAD_CHAR, "").replace(SOS_CHAR, "").replace(EOS_CHAR, "")
    return len(s.replace("  ", " ").split())


def last_logits(P, cfg: OracleConfig, ys: torch.Tensor, enc: torch.Tensor) -> torch.Tensor:
    """Logits of the last position of every prefix in ys [n, t] (transformer.py:438-454): causal self-attention, no
    cross-attention mask, all-ones non-pad mask, dropout off."""
    n, t = ys.shape
    d = cfg.dim_model
    scale = d ** -0.5 if cfg.emb_trg_sharing else 1.0
    causal = torch.triu(torch.ones(t, t, dtype=torch.uint8), diagonal=1).bool().unsqueeze(0).expand(n, -1, -1)
    x = F.embedding(ys, P["decoder.trg_embedding.weight"], padding_idx=PAD) * scale + sinusoid_table(t, d, enc.dtype).unsqueeze(0)
    e = enc.expand(n, -1, -1)
    for l in range(cfg.num_layers):
        pre = f"decoder.layers.{l}."
        x = multi_head_attention(x, x, x, causal, P, pre + "self_attn.", cfg.num_heads, cfg.dim_key, cfg.dim_value)
        x = multi_head_attention(x, e, e, None, P, pre + "encoder_attn.", cfg.num_heads, cfg.dim_key, cfg.dim_value)
        x = conv_ffn(x, P, pre + "pos_ffn.")
    return F.linear(x[:, -1], P["decoder.output_linear.weight"])


def beam_search(P, cfg: OracleConfig, enc: torch.Tensor, W: int, nbest: int, c_weight: float, id2label, steps: int = 300):
    """The reference's search for every utterance of enc [B, T_e, d] (use float64 parameters and enc).  Per utterance a dict:
      yseqs, scores, finals -- the top-nbest ended hypotheses (yseq with SOS and the final EOS) by final score, stable;
      step_margins       -- per step, the gap between the W-th and (W+1)-th of all (hypothesis, token) scores: the margin of
                            the pruning decision (inf when there are at most W candidates);
      pool_margin        -- the smallest gap between consecutive final scores among the top nbest + 1 ended hypotheses:
                            the margin of the n-best choice and its order (inf with one ended hypothesis or none)."""
    Te = enc.shape[1]
    out = []
    for x in range(enc.shape[0]):
        e = enc[x:x + 1]
        hyps = [(0.0, [SOS])]                                     # (score, yseq), in list order
        ended, step_margins = [], []
        for i in range(steps):
            ys = torch.tensor([h[1] for h in hyps], dtype=torch.long)
            lp = F.log_softmax(last_logits(P, cfg, ys, e), dim=1)
            sc = torch.tensor([h[0] for h in hyps], dtype=lp.dtype).unsqueeze(1) + lp
            allv = sc.flatten().sort(descending=True).values
            step_margins.append(float(allv[W - 1] - allv[W]) if allv.numel() > W else math.inf)
            cand = []
            for j, (s, y) in enumerate(hyps):
                order = torch.sort(-lp[j], stable=True).indices[:W]   # topk, ties to the lower id
                cand += [(float(sc[j, v]), y + [int(v)]) for v in order]
                cand = sorted(cand, key=lambda c: c[0], reverse=True)[:W]
            if i == Te - 1:                                       # :471-473
                cand = [(s, y + [EOS]) for s, y in cand]
            hyps = []
            for s, y in cand:
                if y[-1] == EOS:
                    ended.append((s + math.sqrt(num_words(y, id2label)) * c_weight, s, y))
                else:
                    hyps.append((s, y))
            if not hyps:
                break
        ranked = sorted(ended, key=lambda h: h[0], reverse=True)
        fin = [h[0] for h in ranked[:nbest + 1]]
        gaps = [fin[j] - fin[j + 1] for j in range(len(fin) - 1)]
        out.append(dict(yseqs=[h[2] for h in ranked[:nbest]], scores=[h[1] for h in ranked[:nbest]],
                        finals=[h[0] for h in ranked[:nbest]], step_margins=step_margins,
                        pool_margin=min(gaps) if gaps else math.inf))
    return out
