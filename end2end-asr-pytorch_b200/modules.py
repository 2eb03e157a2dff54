"""Host-side mirror of the reference's model interface for the hot path.

Same class names, constructor arguments, parameter names/shapes (state_dict compatible) and forward
signatures as /root/reference/models/common_layers.py and models/asr/transformer.py -- but every forward is
a composition of libb200asr kernels (ops.py).  The forward bodies are written against attribute names that
exist in BOTH this mirror and the reference classes, so ``install()`` can bind the very same functions onto
the reference's classes (class-level patch, SURVEY.md §8b).

Decoder.beam_search is mirrored (beam_decode: batched, KV-cached, selection on the device), including lm_rescoring=True
with an LSTM language model (RNNModel / LM below, or the reference's utils/lstm_utils.LM); with any other LM object it runs
the reference's own method.  Decoder.greedy_search (greedy_decode_cached) and Transformer.evaluate are mirrored too.
Not mirrored (out of scope, SURVEY.md §2): the Linear-variant FFN (dead code).
"""
from __future__ import annotations

import math
import time
import unicodedata

import numpy as np

import torch
import torch.nn as nn

from . import ops, parallel

PAD_TOKEN, SOS_TOKEN, EOS_TOKEN = 0, 1, 2     # utils/constant.py:102-104


# ------------------------------------------------------------------------------------------------ helpers
def _drop_p(module: nn.Module, dropout: nn.Dropout) -> float:
    return float(dropout.p) if module.training else 0.0


def _as_u8_mask(mask, B, Tq, Tk):
    """Reference-style bool/uint8 (B,Tq,Tk) mask -> contiguous uint8 (compat path only; the model-level forwards
    never build dense masks)."""
    if mask is None:
        return None
    m = mask.expand(B, Tq, Tk)
    return m.to(torch.uint8).contiguous()


def _maps_sink():
    """A list for the attention maps of a forward while ops.attention_maps is on, else None (no map is computed)."""
    return [] if ops.attention_maps_enabled() else None


def _first(maps):
    return maps[0] if maps is not None else None


def _mha_core(self, query, key, value, key_pad=None, dense_mask=None, causal=False, row_scale=None, maps=None):
    """MultiHeadAttention body (models/common_layers.py:170-200) on fused kernels.

    Q/K/V projections write token-major [B,T,H*d]; the attention kernel addresses heads through strides, so
    the permute/contiguous copies of :185-187 and :194-195 do not exist.  `row_scale` (the non-pad mask that the
    layer applies right after, transformer.py:198/536/540) is folded into the LayerNorm epilogue.  `maps`: a list that
    receives the (H*B) x Tq x Tk attention map (ops.attention_probs), or None."""
    B, Tq, _ = query.shape
    Tk = key.shape[1]
    H, dk, dv = self.num_heads, self.dim_key, self.dim_value
    p_attn = _drop_p(self, self.attention.dropout)
    scale = 1.0 / float(self.attention.temperature)
    ql, kl, vl = self.query_linear, self.key_linear, self.value_linear
    link = None
    if key is value:
        link = ops.ResidualLink() if torch.is_grad_enabled() else None
        # projections + attention as one autograd node: Q/K/V (or K/V) run as ONE GEMM when their weights lie back to back
        # in memory (optim.FlatParams), and the attention kernels address the packed output through strides
        o = ops.AttnProjFn.apply(query, key, ql.weight, ql.bias, kl.weight, kl.bias, vl.weight, vl.bias, H, dk, dv,
                                 key_pad, dense_mask, causal, scale, p_attn, link, maps)    # [B,Tq,H*dv], token-major
    else:
        q = ops.LinearFn.apply(query, ql.weight, ql.bias).view(B, Tq, H, dk).permute(0, 2, 1, 3)
        k = ops.LinearFn.apply(key, kl.weight, kl.bias).view(B, Tk, H, dk).permute(0, 2, 1, 3)
        v = ops.LinearFn.apply(value, vl.weight, vl.bias).view(B, Tk, H, dv).permute(0, 2, 1, 3)
        o = ops.SdpaFn.apply(q, k, v, key_pad, dense_mask, causal, scale, p_attn, False, maps)   # (B,H,Tq,dv) view of [B,Tq,H,dv]
        o = o.permute(0, 2, 1, 3).reshape(B, Tq, H * dv)                                  # free: memory is token-major
    o = ops.LinearFn.apply(o, self.output_linear.weight, self.output_linear.bias)
    ln = self.layer_norm
    return ops.AddLNFn.apply(o, query, ln.weight, ln.bias, None, row_scale, ln.eps, _drop_p(self, self.dropout), link)


def _ffn_core(self, x, row_scale=None):
    """PositionwiseFeedForwardWithConv body (models/common_layers.py:135-142)."""
    link = ops.ResidualLink() if torch.is_grad_enabled() else None
    y = ops.FFNFn.apply(x, self.conv_1.weight, self.conv_1.bias, self.conv_2.weight, self.conv_2.bias, link)
    ln = self.layer_norm
    return ops.AddLNFn.apply(y, x, ln.weight, ln.bias, None, row_scale, ln.eps, _drop_p(self, self.dropout), link)


# ------------------------------------------------------------------------------------------------ forwards (bindable)
def sdpa_forward(self, q, k, v, mask=None):
    """ScaledDotProductAttention.forward(q, k, v, mask) -- models/common_layers.py:211-225.
    q,k,v are head-major (H*B) x T x d exactly as the reference passes them and `mask` is the (H*B) x Tq x Tk
    tensor MultiHeadAttention built with mask.repeat(H,1,1); each (h,b) slice is treated as its own batch entry.
    Returns (output, attn): attn is the detached (H*B) x Tq x Tk probability map while ops.attention_maps is on, else None."""
    HB, Tq, dk = q.shape
    Tk, dv = k.shape[1], v.shape[2]
    dense = _as_u8_mask(mask, HB, Tq, Tk)
    as4 = lambda t: t.contiguous().unsqueeze(1)          # (HB,1,T,d): one "head" per batch entry
    p = float(self.dropout.p) if self.training else 0.0
    maps = _maps_sink()
    o = ops.SdpaFn.apply(as4(q), as4(k), as4(v), None, dense, False, 1.0 / float(self.temperature), p, False, maps)
    return o.reshape(HB, Tq, dv), _first(maps)


def mha_forward(self, query, key, value, mask=None):
    """MultiHeadAttention.forward(query, key, value, mask) -> (output, attn) -- common_layers.py:170-200; attn is the
    (H*B) x Tq x Tk map while ops.attention_maps is on, else None."""
    B, Tq, _ = query.shape
    dense = _as_u8_mask(mask, B, Tq, key.shape[1])
    maps = _maps_sink()
    return _mha_core(self, query, key, value, dense_mask=dense, maps=maps), _first(maps)


def ffn_forward(self, x):
    """PositionwiseFeedForwardWithConv.forward(x) -- common_layers.py:135-142."""
    return _ffn_core(self, x)


def encoder_layer_forward(self, enc_input, non_pad_mask=None, self_attn_mask=None):
    """EncoderLayer.forward -- models/asr/transformer.py:195-203 (dense-mask compatible signature) -> (output, self_attn map
    or None)."""
    B, T, _ = enc_input.shape
    rs = non_pad_mask.reshape(-1) if non_pad_mask is not None else None
    maps = _maps_sink()
    x = _mha_core(self.self_attn, enc_input, enc_input, enc_input, dense_mask=_as_u8_mask(self_attn_mask, B, T, T), row_scale=rs,
                  maps=maps)
    return _ffn_core(self.pos_ffn, x, row_scale=rs), _first(maps)


def decoder_layer_forward(self, decoder_input, encoder_output, non_pad_mask=None, self_attn_mask=None, dec_enc_attn_mask=None):
    """DecoderLayer.forward -- models/asr/transformer.py:533-545 (dense-mask compatible signature) -> (output, self_attn,
    enc_attn), the maps None while ops.attention_maps is off."""
    B, T, _ = decoder_input.shape
    Te = encoder_output.shape[1]
    rs = non_pad_mask.reshape(-1) if non_pad_mask is not None else None
    self_maps, cross_maps = _maps_sink(), _maps_sink()
    x = _mha_core(self.self_attn, decoder_input, decoder_input, decoder_input,
                  dense_mask=_as_u8_mask(self_attn_mask, B, T, T), row_scale=rs, maps=self_maps)
    x = _mha_core(self.encoder_attn, x, encoder_output, encoder_output,
                  dense_mask=_as_u8_mask(dec_enc_attn_mask, B, T, Te), row_scale=rs, maps=cross_maps)
    return _ffn_core(self.pos_ffn, x, row_scale=rs), _first(self_maps), _first(cross_maps)


def _encoder_body(self, feats, input_lengths, cf_order=None, maps=None):
    """Encoder.forward body (models/asr/transformer.py:157-180).  `feats` is [B,T,D]; when cf_order=(C,F) its
    feature axis is ordered f*C+c (channels-last conv output) and input_linear's columns are permuted to match.
    Masks are a key-valid byte vector per utterance built from the RAW lengths (quirk Q1 preserved).  `maps`: a list that
    receives each layer's self-attention map, or None."""
    B, T, D = feats.shape
    key_pad, non_pad = ops.length_masks(input_lengths, B, T, feats.device)
    rs = non_pad.view(-1)
    w = self.input_linear.weight
    if cf_order is not None:
        w = ops.PermuteColsFn.apply(w, cf_order[0], cf_order[1])
    x = ops.LinearFn.apply(feats, w, self.input_linear.bias)
    ln = self.layer_norm_input
    pe = self.positional_encoding.pe[0, :T]
    x = ops.AddLNFn.apply(x, None, ln.weight, ln.bias, pe, None, ln.eps, 0.0)
    for layer in self.layers:
        x = _mha_core(layer.self_attn, x, x, x, key_pad=key_pad, row_scale=rs, maps=maps)
        x = _ffn_core(layer.pos_ffn, x, row_scale=rs)
    return x


def encoder_forward(self, padded_input, input_lengths):
    """Encoder.forward(padded_input, input_lengths) -> (output, [self_attn map per layer]); [None]*L while
    ops.attention_maps is off."""
    maps = _maps_sink()
    out = _encoder_body(self, padded_input, input_lengths, maps=maps)
    return out, maps if maps is not None else [None] * len(self.layers)


def decoder_forward(self, padded_input, encoder_padded_outputs, encoder_input_lengths):
    """Decoder.forward -- models/asr/transformer.py:268-305: (pred, gold, [self_attn map per layer], [enc_attn map per
    layer]), [None]*L each while ops.attention_maps is off."""
    self_maps, cross_maps = _maps_sink(), _maps_sink()
    pred, gold = _decoder_body(self, padded_input, encoder_padded_outputs, encoder_input_lengths, self_maps, cross_maps)
    n = len(self.layers)
    return (pred, gold, self_maps if self_maps is not None else [None] * n,
            cross_maps if cross_maps is not None else [None] * n)


def _decoder_body(self, padded_input, encoder_padded_outputs, encoder_input_lengths, self_maps=None, cross_maps=None):
    """Decoder.forward body -> (pred, gold).  Target preprocessing, masks, embedding+PE run on the device without host
    syncs.  self_maps / cross_maps: lists that receive each layer's attention maps, or None."""
    Tt = int(self.trg_max_length)
    seq_in, seq_out, key_pad, non_pad = ops.preprocess_targets(padded_input, Tt)
    B = seq_in.shape[0]
    Te = encoder_padded_outputs.shape[1]
    enc_key_pad, _ = ops.length_masks(encoder_input_lengths, B, Te, encoder_padded_outputs.device)
    rs = non_pad.view(-1)
    pe = self.positional_encoding.pe[0, :Tt]
    x = ops.EmbedFn.apply(seq_in, self.trg_embedding.weight, pe, float(self.x_logit_scale), _drop_p(self, self.dropout), PAD_TOKEN)
    for layer in self.layers:
        x = _mha_core(layer.self_attn, x, x, x, key_pad=key_pad, causal=True, row_scale=rs, maps=self_maps)
        x = _mha_core(layer.encoder_attn, x, encoder_padded_outputs, encoder_padded_outputs, key_pad=enc_key_pad, row_scale=rs,
                      maps=cross_maps)
        x = _ffn_core(layer.pos_ffn, x, row_scale=rs)
    pred = ops.LinearFn.apply(x, self.output_linear.weight, None)
    return pred, seq_out


def greedy_decode_ids(self, encoder_padded_outputs, steps=300):
    """Token ids of Decoder.greedy_search (models/asr/transformer.py:316-394, no LM rescoring) on the fused kernels:
    full-prefix re-decode per step exactly as the reference (causal self-attention, no cross-attention mask, all-ones
    non-pad mask, argmax of the last position).  Returns int64 [B, steps]; string building / EOS cut stay with the caller.
    (The KV-cached incremental decoder is the 'next' row 3 of SURVEY.md §8f.)"""
    B = encoder_padded_outputs.shape[0]
    dev = encoder_padded_outputs.device
    was_training = self.training
    self.eval()
    try:
        with torch.no_grad():
            ys = torch.full((B, 1), SOS_TOKEN, dtype=torch.long, device=dev)
            for _ in range(steps):
                t = ys.shape[1]
                pe = self.positional_encoding.pe[0, :t]
                x = ops.EmbedFn.apply(ys, self.trg_embedding.weight, pe, float(self.x_logit_scale), 0.0, PAD_TOKEN)
                for layer in self.layers:
                    x = _mha_core(layer.self_attn, x, x, x, causal=True)
                    x = _mha_core(layer.encoder_attn, x, encoder_padded_outputs, encoder_padded_outputs)
                    x = _ffn_core(layer.pos_ffn, x)
                last = x[:, -1].contiguous()
                logits = ops.LinearFn.apply(last, self.output_linear.weight, None)
                ys = torch.cat([ys, ops.argmax_rows(logits).view(B, 1)], dim=1)
    finally:
        self.train(was_training)
    return ys[:, 1:]


def greedy_decode_cached(self, encoder_padded_outputs, steps=300, stop_at_eos=False, check_every=8):
    """Incremental greedy decode with self- and cross-attention K/V caches (SURVEY.md §8f row 3): the same token ids as
    greedy_decode_ids / the reference's greedy_search, at O(T) instead of O(T^2) work -- per step only the new position is
    projected, its K/V rows are written by the GEMM into step t of per-layer slab-major caches [steps, B, H*d], and
    single-query attention (ops.decode_attn, split over keys) runs over the cache (self) and over the encoder K/V projected
    once per call (cross, no mask as in transformer.py:347), both read in place through strides.

    stop_at_eos: the EOS cut of transformer.py:385-393 stays on the device -- ids from an utterance's first EOS on are -1
    (the reference drops them when it builds the strings), a device counter tracks finished utterances and the loop ends
    as soon as every utterance has emitted EOS (checked every `check_every` steps: one 4-byte read, no id traffic)
    instead of always running the reference's 300 fixed steps."""
    B, Te, _ = encoder_padded_outputs.shape
    dev = encoder_padded_outputs.device
    was_training = self.training
    self.eval()
    try:
        with torch.no_grad():
            H = self.layers[0].self_attn.num_heads
            dk, dv = self.layers[0].self_attn.dim_key, self.layers[0].self_attn.dim_value
            cross, kc, vc = [], [], []
            for layer in self.layers:
                ca = layer.encoder_attn
                k = ops.LinearFn.apply(encoder_padded_outputs, ca.key_linear.weight, ca.key_linear.bias)        # [B, Te, H*dk]
                v = ops.LinearFn.apply(encoder_padded_outputs, ca.value_linear.weight, ca.value_linear.bias)
                cross.append((k, v))
                kc.append(torch.empty((steps, B, H * dk), device=dev, dtype=torch.float32))
                vc.append(torch.empty((steps, B, H * dv), device=dev, dtype=torch.float32))
            ys = torch.full((B, steps), -1, dtype=torch.long, device=dev) if stop_at_eos else torch.empty((B, steps), dtype=torch.long, device=dev)
            tok = torch.full((B, 1), SOS_TOKEN, dtype=torch.long, device=dev)
            finished = torch.zeros(B + 1, dtype=torch.int32, device=dev) if stop_at_eos else None      # [B] flags + [1] counter
            self_k, self_v = (H * dk, B * H * dk), (H * dv, B * H * dv)               # (row, key) strides of the caches
            cross_k, cross_v = (Te * H * dk, H * dk), (Te * H * dv, H * dv)           # ... and of the encoder projections

            def post(mod, o, x):
                o = ops.LinearFn.apply(o, mod.output_linear.weight, mod.output_linear.bias).view(B, 1, -1)
                return ops.AddLNFn.apply(o, x, mod.layer_norm.weight, mod.layer_norm.bias, None, None, mod.layer_norm.eps, 0.0)

            for t in range(steps):
                pe = self.positional_encoding.pe[0, t:t + 1]
                x = ops.EmbedFn.apply(tok, self.trg_embedding.weight, pe, float(self.x_logit_scale), 0.0, PAD_TOKEN)
                for li, layer in enumerate(self.layers):
                    sa, ca = layer.self_attn, layer.encoder_attn
                    x2 = x.view(B, -1)
                    ops.linear_into(x2, sa.key_linear.weight, sa.key_linear.bias, kc[li][t])
                    ops.linear_into(x2, sa.value_linear.weight, sa.value_linear.bias, vc[li][t])
                    q = ops.LinearFn.apply(x2, sa.query_linear.weight, sa.query_linear.bias)
                    o = ops.decode_attn(q, kc[li], vc[li], H, t + 1, self_k, self_v, dv, 1.0 / float(sa.attention.temperature))
                    x = post(sa, o, x)
                    q = ops.LinearFn.apply(x.view(B, -1), ca.query_linear.weight, ca.query_linear.bias)
                    o = ops.decode_attn(q, cross[li][0], cross[li][1], H, Te, cross_k, cross_v, dv,
                                        1.0 / float(ca.attention.temperature))
                    x = post(ca, o, x)
                    x = _ffn_core(layer.pos_ffn, x)
                logits = ops.LinearFn.apply(x.view(B, -1), self.output_linear.weight, None)
                if stop_at_eos:
                    tok = ops.greedy_step(logits, ys, finished, t)
                    if (t + 1) % check_every == 0 and int(finished[B].item()) == B:
                        break
                else:
                    tok = ops.argmax_rows(logits).view(B, 1)
                    ys[:, t:t + 1] = tok
    finally:
        self.train(was_training)
    return ys


PAD_CHAR, SOS_CHAR, EOS_CHAR = "\u00b6", "\u00a7", "\u00a4"     # utils/constant.py:105-107


def word_records(id2label, V):
    """Per-token word-count record of Decoder.beam_search's num_words (models/asr/transformer.py:490-492): with s the label
    without the PAD/SOS/EOS characters, w = len(s.split()), head / tail = s starts / ends with a non-space character, empty =
    s is "".  A hypothesis carries (words, tail); appending token v gives words += w - (tail and head), and tail = tail_v
    unless s is empty -- exactly len(s.split()) of the joined string.  Returns [V] ints w * 8 + head * 4 + tail * 2 + empty."""
    out = []
    for v in range(V):
        try:
            lab = str(id2label[v])
        except (KeyError, IndexError):
            lab = ""
        s = lab.replace(PAD_CHAR, "").replace(SOS_CHAR, "").replace(EOS_CHAR, "")
        head = bool(s) and not s[0].isspace()
        tail = bool(s) and not s[-1].isspace()
        out.append(len(s.split()) * 8 + head * 4 + tail * 2 + (not s))
    return out


def _word_table(self, V, device):
    """word_records of self.id2label as a device tensor, built once per label map (and device)."""
    cached = self.__dict__.get("_b200_word_table")
    if cached is None or cached[0] is not self.id2label or cached[1] != V or cached[2].device != device:
        tab = torch.tensor(word_records(self.id2label, V), dtype=torch.int32, device=device)
        cached = (self.id2label, V, tab)
        self.__dict__["_b200_word_table"] = cached
    return cached[2]


def _check_beam_positions(self, Te, steps):
    n = min(int(steps), int(Te))
    if int(self.trg_max_length) < n:
        raise ValueError(f"beam search decodes {n} positions (min(steps={steps}, T_e={Te})) but the decoder's positional table "
                         f"covers trg_max_length={self.trg_max_length}: build the model with tgt_max_len >= {n}")


def beam_decode(self, enc, beam_width, nbest=1, c_weight=1.0, steps=300, check_every=8, lm=None, lm_weight=0.1):
    """Batched, KV-cached Decoder.beam_search (models/asr/transformer.py:396-517) on the device.

    All B utterances decode together as B * beam_width rows.  Per step only the new position is projected: its self-attention
    K/V rows are written by the GEMM into step t of per-layer caches [steps, B*W, H*d], and each row attends over its own
    history through an index table that the selection kernel reorders (no K/V moves).  Cross-attention runs over the encoder
    K/V projected once per call (the W queries of an utterance share them).  Selection, the forced EOS at T_e - 1, word counts,
    final scores and the n-best pools stay on the device; the host reads the live-utterance counter every `check_every` steps.

    lm: an LSTM language model (b200asr.LM, or the reference's utils/lstm_utils.LM) rescores every ended hypothesis as
    lm_rescoring=True does (transformer.py:473-481): the selection is unchanged, the device keeps a log of every ended
    hypothesis, and the n-best are ranked by score + lm_weight * lm_score + sqrt(num_words) * c_weight (see lm_rescore).

    Returns device tensors (ids [B, nbest, S + 2] int64: SOS, tokens, EOS, then -1, with S = min(steps, T_e); lengths [B, nbest]
    int64, 0 where an utterance has fewer than nbest ended hypotheses; score and final_score [B, nbest] fp32, NaN there),
    ordered by final_score as the reference's stable sort orders them."""
    B, Te, _ = enc.shape
    _check_beam_positions(self, Te, steps)
    lm_parts = None
    if lm is not None:
        lm_parts = lstm_lm_parts(lm)
        if lm_parts is None:
            raise TypeError("beam_decode: lm must be an LSTM language model (b200asr.LM or utils/lstm_utils.LM)")
    dev = enc.device
    S = min(int(steps), int(Te))
    W = int(beam_width)
    R = B * W
    was_training = self.training
    self.eval()
    try:
        with torch.no_grad():
            tab = _word_table(self, self.output_linear.weight.shape[0], dev)
            H = self.layers[0].self_attn.num_heads
            dk, dv = self.layers[0].self_attn.dim_key, self.layers[0].self_attn.dim_value
            cross, kc, vc = [], [], []
            for layer in self.layers:
                ca = layer.encoder_attn
                k = ops.LinearFn.apply(enc, ca.key_linear.weight, ca.key_linear.bias).view(B, Te, H, dk).permute(0, 2, 1, 3)
                v = ops.LinearFn.apply(enc, ca.value_linear.weight, ca.value_linear.bias).view(B, Te, H, dv).permute(0, 2, 1, 3)
                cross.append((k, v))
                kc.append(torch.empty((S, R, H * dk), device=dev, dtype=torch.float32))
                vc.append(torch.empty((S, R, H * dv), device=dev, dtype=torch.float32))
            buf = ops.BeamBuffers(B, W, int(nbest), S, dev)
            log = ops.EndLog(B, W, S, dev) if lm_parts is not None else None

            def post(mod, o, x):
                o = ops.LinearFn.apply(o, mod.output_linear.weight, mod.output_linear.bias).view(R, 1, -1)
                return ops.AddLNFn.apply(o, x, mod.layer_norm.weight, mod.layer_norm.bias, None, None, mod.layer_norm.eps, 0.0)

            for t in range(S):
                pe = self.positional_encoding.pe[0, t:t + 1]
                x = ops.EmbedFn.apply(buf.next_tok, self.trg_embedding.weight, pe, float(self.x_logit_scale), 0.0, PAD_TOKEN)
                idx = buf.idx[t % 2]
                for li, layer in enumerate(self.layers):
                    sa, ca = layer.self_attn, layer.encoder_attn
                    x2 = x.view(R, -1)
                    ops.linear_into(x2, sa.key_linear.weight, sa.key_linear.bias, kc[li][t])
                    ops.linear_into(x2, sa.value_linear.weight, sa.value_linear.bias, vc[li][t])
                    q = ops.LinearFn.apply(x2, sa.query_linear.weight, sa.query_linear.bias)
                    x = post(sa, ops.beam_self_attn(q, kc[li], vc[li], idx, W, H, t, 1.0 / float(sa.attention.temperature)), x)
                    q = ops.LinearFn.apply(x, ca.query_linear.weight, ca.query_linear.bias).view(B, W, H, dk).permute(0, 2, 1, 3)
                    o = ops.SdpaFn.apply(q, cross[li][0], cross[li][1], None, None, False, 1.0 / float(ca.attention.temperature), 0.0)
                    x = post(ca, o.permute(0, 2, 1, 3).reshape(R, H * dv), x)
                    x = _ffn_core(layer.pos_ffn, x)
                logits = ops.LinearFn.apply(x.view(R, -1), self.output_linear.weight, None)
                if log is None:
                    ops.beam_step(buf, logits, tab, t, Te - 1, c_weight)
                else:
                    ops.beam_step_log(buf, log, logits, tab, t, Te - 1, c_weight)
                if (t + 1) % check_every == 0 and t + 1 < S and int(buf.n_live.item()) == 0:
                    break
            if log is not None:
                return lm_rescore(self, buf, log, lm_parts, lm_weight, c_weight)
            ids, lengths = ops.beam_backtrack(buf)
    finally:
        self.train(was_training)
    return ids, lengths, buf.pool_score, buf.pool_final


def beam_search(self, encoder_padded_outputs, beam_width=2, nbest=5, lm_rescoring=False, lm=None, lm_weight=0.1, c_weight=1,
                prob_weight=1.0):
    """Decoder.beam_search (models/asr/transformer.py:396-517): flat lists of the n-best yseqs (SOS ... EOS, as int lists) and
    their strings ("".join of id2label over yseq[1:]), nbest entries per utterance in batch order, fewer where an utterance
    ends fewer hypotheses (none when it ends none, so Transformer.evaluate falls back to greedy_search).  Decoded by
    beam_decode with 300 steps; the ids come back in one device-to-host copy.  prob_weight is ignored, as by the reference.
    lm_rescoring=True with an LSTM LM (b200asr.LM or utils/lstm_utils.LM) rescores on the device; with any other `lm` it runs
    the reference's own method (kept by install())."""
    if lm_rescoring and lstm_lm_parts(lm) is None:
        from .install import original
        ref = original(type(self), "beam_search")
        if ref is None:
            raise NotImplementedError("beam_search with lm_rescoring=True and a language model other than an LSTM LM runs the "
                                      "reference's own method; call b200asr.install() on the reference's Decoder")
        return ref(self, encoder_padded_outputs, beam_width=beam_width, nbest=nbest, lm_rescoring=lm_rescoring, lm=lm,
                   lm_weight=lm_weight, c_weight=c_weight, prob_weight=prob_weight)
    ids, lengths, _, _ = beam_decode(self, encoder_padded_outputs, beam_width, nbest=nbest, c_weight=c_weight, steps=300,
                                     lm=lm if lm_rescoring else None, lm_weight=lm_weight)
    return beam_strings(torch.cat([lengths.unsqueeze(-1), ids], dim=-1).cpu(), self.id2label)


def beam_strings(both, id2label):
    """The flat yseq and string lists of Decoder.beam_search from host rows `both` [B, nbest, 1 + S + 2] int64: per
    hypothesis its length n (0: none), then its yseq (SOS ... EOS) padded with -1.  The string of a yseq is "".join of
    id2label over yseq[1:]; utterances and their hypotheses in order, none for an empty slot."""
    ys, strs = [], []
    for b in range(both.shape[0]):
        for i in range(both.shape[1]):
            n = int(both[b, i, 0])
            if n == 0:
                continue
            y = both[b, i, 1:1 + n].tolist()
            ys.append(y)
            strs.append("".join(id2label[t] for t in y[1:]))
    return ys, strs


GREEDY_STEPS = 300          # Decoder.greedy_search's fixed step count (transformer.py:332)


def greedy_strings(ids, id2label):
    """The strings of Decoder.greedy_search (models/asr/transformer.py:376 and :385-393) from per-utterance token ids: each id
    maps to id2label[id], except EOS, which maps to EOS_CHAR; the string ends before the first entry EQUAL to EOS_CHAR (a cut
    on the string, so a non-EOS label equal to EOS_CHAR also ends it).  The reference joins the entries of a numpy array
    (np.transpose of the per-step label lists), so every label goes through numpy's str conversion, as here.  An id < 0 ends
    the row as well: greedy_decode_cached(stop_at_eos=True) writes -1 after an utterance's first EOS, where the string has
    already ended."""
    out = []
    for row in ids:
        labels = []
        for i in row:
            if i < 0:
                break
            labels.append(EOS_CHAR if i == EOS_TOKEN else id2label[i])
        st = ""
        for e in np.array(labels, dtype=str):
            if e == EOS_CHAR:
                break
            st += e
        out.append(st)
    return out


def _reference_method(self, name, why):
    from .install import original
    ref = original(type(self), name)
    if ref is None:
        raise NotImplementedError(f"{type(self).__name__}.{name} {why} runs the reference's own method; call b200asr.install() on "
                                  f"the reference's {type(self).__name__}")
    return ref


def greedy_search(self, encoder_padded_outputs, beam_width=2, lm_rescoring=False, lm=None, lm_weight=0.1, c_weight=1):
    """Decoder.greedy_search (models/asr/transformer.py:316-394): the B strings of 300 greedy steps, cut at EOS_CHAR.  Decoded
    by greedy_decode_cached(steps=300, stop_at_eos=True) -- KV-cached, the EOS stop on the device -- with the ids back in one
    device-to-host copy; the strings follow greedy_strings.  lm_rescoring=True (which fails in the reference itself) and a
    decoder in training mode (the reference then applies dropout at every step) run the reference's own method."""
    if lm_rescoring or self.training:
        ref = _reference_method(self, "greedy_search", "with lm_rescoring=True or in training mode")
        return ref(self, encoder_padded_outputs, beam_width=beam_width, lm_rescoring=lm_rescoring, lm=lm, lm_weight=lm_weight,
                   c_weight=c_weight)
    _check_greedy_positions(self)
    ids = greedy_decode_cached(self, encoder_padded_outputs, steps=GREEDY_STEPS, stop_at_eos=True).cpu()
    return greedy_strings(ids.tolist(), self.id2label)


def _check_greedy_positions(self):
    if int(self.trg_max_length) < GREEDY_STEPS:
        raise ValueError(f"greedy search decodes {GREEDY_STEPS} positions but the decoder's positional table covers "
                         f"trg_max_length={self.trg_max_length}: build the model with tgt_max_len >= {GREEDY_STEPS}")


# ------------------------------------------------------------------------------------------------ LM rescoring
def _has_letter_lo(word):
    """data/helper.py:33-54: a word is "Chinese" when one of its characters has Unicode category Lo."""
    return any(unicodedata.category(ch) == "Lo" for ch in word)


def lm_string(yseq, id2label) -> str:
    """The string calculate_lm_score (utils/lstm_utils.py:9-44) scores for a hypothesis: the joined labels without the
    PAD/SOS/EOS characters, "  " -> " " once; the " "-separated pieces grouped into runs of one kind ("Chinese" or not,
    data/helper.py:56-99; the pieces of a run rejoined with " ", empty pieces only after a non-empty one); then every
    character of a Chinese run -- spaces included -- is its own word, a non-Chinese run is one item, items are joined with
    " " (an empty item adds nothing while the result is still empty), and "  " -> " " is applied twice."""
    s = "".join(id2label[t] for t in yseq).replace(PAD_CHAR, "").replace(SOS_CHAR, "").replace(EOS_CHAR, "").replace("  ", " ")
    runs = []                                   # [chinese, text]
    for piece in s.split(" "):
        kind = _has_letter_lo(piece)
        if runs and runs[-1][0] == kind:
            runs[-1][1] = runs[-1][1] + " " + piece if runs[-1][1] else piece
        else:
            runs.append([kind, piece])
    out = ""
    for kind, text in runs:
        for item in (text if kind else (text,)):
            out = out + " " + item if out else item
    return out.replace("  ", " ").replace("  ", " ")


def lm_word_ids(string, word2idx):
    """LM.seq_to_tensor (utils/lstm_utils.py:82-97): ids of string.split() + ['<eos>'] and the number of words mapped to
    '<oov>' (a KeyError if one is needed and the vocabulary has none, as in the reference)."""
    ids, oov = [], 0
    for w in string.split() + ["<eos>"]:
        i = word2idx.get(w)
        if i is None:
            i = word2idx["<oov>"]
            oov += 1
        ids.append(int(i))
    return ids, oov


def lm_final_score(score, nll_sum, n, oov, lm_weight, c_weight):
    """(lm_score, num_words, final_score) of one ended hypothesis in the reference's fp32 operations (transformer.py:478-481,
    lstm_utils.py:36-44, 124-127): total = n * (nll_sum / n); lm_score = -total / n + 1 - 2 * oov; final = score +
    lm_weight * lm_score + sqrt(n + 1) * c_weight.  n is None for an empty string: lm_score -999, num_words 0; n == 0 (a
    string of spaces only) gives NaN, as the reference's mean over no targets does."""
    f = np.float32
    if n is None:
        return -999.0, 0, f(f(score) + f(lm_weight * -999.0)) + f(0.0)
    if n == 0:
        return float("nan"), 1, f("nan")
    total = f(n) * f(f(nll_sum) / f(n))
    lm = f(f(f(-total) / f(n)) + f(1.0)) - f(2 * oov)
    return float(lm), n + 1, f(f(score) + f(lm_weight) * lm) + f(math.sqrt(n + 1) * c_weight)


def lstm_lm_parts(lm):
    """(RNNModel, word2idx) of an LSTM language model object (b200asr.LM or utils/lstm_utils.LM), else None."""
    model, w2i = getattr(lm, "model", None), getattr(lm, "word2idx", None)
    rnn = getattr(model, "rnn", None)
    if not (isinstance(w2i, dict) and isinstance(rnn, nn.LSTM) and isinstance(getattr(model, "encoder", None), nn.Embedding)
            and isinstance(getattr(model, "decoder", None), nn.Linear)):
        return None
    if rnn.bidirectional or rnn.batch_first or getattr(rnn, "proj_size", 0) or rnn.input_size != model.encoder.embedding_dim:
        return None
    return model, w2i


def rank_nbest(finals, nbest):
    """Indices of the nbest largest final scores; equal scores keep insertion order (transformer.py:499: sorted(...,
    reverse=True) is stable)."""
    return sorted(range(len(finals)), key=lambda j: finals[j], reverse=True)[:nbest]


lm_rescore_stats = {}      # timings and counts of the last lm_rescore call (tools/decode_bench.py --lm reports them)


def lm_rescore(self, buf, log, lm_parts, lm_weight, c_weight):
    """n-best of a finished beam search under LM rescoring.  The end log comes to the host in one copy; the yseqs of its
    entries are walked on the device into a packed buffer sized by their lengths and read once; the host builds each LM
    string and its word ids (identical strings are scored once); the word ids go up in one copy and the LSTM LM scores
    every sequence on the device; final scores follow in the reference's fp32 order and each utterance's entries are
    ranked by a stable sort, so equal final scores keep insertion order (transformer.py:499-500)."""
    model, w2i = lm_parts
    dev = buf.score.device
    B, W, nbest, S = buf.B, buf.W, buf.nbest, buf.steps
    t0 = time.perf_counter()
    host = log.buf.cpu().numpy()
    cap = log.cap
    counts = host[:B].astype(np.int64)
    refs = host[B:B + B * cap].astype(np.int64)
    scores = host[B + B * cap:].view(np.float32)
    entries = np.concatenate([b * cap + np.arange(counts[b], dtype=np.int64) for b in range(B)])
    r = refs[entries]
    lens = (r >> 1) // W + 2 + (r & 1)
    offsets = np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.int64)
    packed = ops.beam_backtrack_packed(buf, log, entries, offsets, int(lens.sum())).cpu().numpy()
    seq_of, seqs, item = {}, [], []          # LM string -> index into seqs; per entry (seq index | None, n, oov)
    for j in range(len(entries)):
        st = lm_string(packed[offsets[j]:offsets[j] + lens[j]], self.id2label)
        if st == "":
            item.append((None, None, 0))
            continue
        ids, oov = lm_word_ids(st, w2i)
        n = len(ids) - 1
        if n == 0:
            item.append((None, 0, oov))
            continue
        k = seq_of.setdefault(st, len(seqs))
        if k == len(seqs):
            seqs.append(ids)
        item.append((k, n, oov))
    t1 = time.perf_counter()
    sums = ops.lstm_lm_nll_sums(model, seqs, dev)
    t2 = time.perf_counter()
    ids_out = np.full((B, nbest, S + 2), -1, dtype=np.int64)
    len_out = np.zeros((B, nbest), dtype=np.int64)
    sc_out = np.full((B, nbest), np.nan, dtype=np.float32)
    fin_out = np.full((B, nbest), np.nan, dtype=np.float32)
    j0 = 0
    for b in range(B):
        rows = range(j0, j0 + int(counts[b]))
        j0 += int(counts[b])
        finals = []
        for j in rows:
            k, n, oov = item[j]
            finals.append(lm_final_score(scores[entries[j]], sums[k] if k is not None else 0.0, n, oov, lm_weight, c_weight)[2])
        for i, r in enumerate(rank_nbest(finals, nbest)):
            fs, j = finals[r], rows[r]
            ids_out[b, i, :lens[j]] = packed[offsets[j]:offsets[j] + lens[j]]
            len_out[b, i] = lens[j]
            sc_out[b, i] = scores[entries[j]]
            fin_out[b, i] = fs
    lm_rescore_stats.update(ended=len(entries), sequences=len(seqs), positions=int(sum(len(q) - 1 for q in seqs)),
                            host_s=t1 - t0, lm_s=t2 - t1)
    to = lambda a: torch.from_numpy(a).to(dev)
    return to(ids_out), to(len_out), to(sc_out), to(fin_out)


def _front_end(self, padded_input):
    """CNN front end + flatten of Transformer.forward (models/asr/transformer.py:70-76).
    Returns (feats [B,T',D], cf_order or None)."""
    if self.feat_extractor == "vgg_cnn":
        c = self.conv
        h = ops.VggFrontendFn.apply(padded_input, c[0].weight, c[0].bias, c[2].weight, c[2].bias, c[5].weight, c[5].bias,
                                    c[7].weight, c[7].bias)
        B, T4, F4, C = h.shape
        return h.view(B, T4, F4 * C), (C, F4)
    if self.feat_extractor == "emb_cnn":
        c = self.conv
        # nn.BatchNorm2d state (running_mean, running_var, num_batches_tracked, momentum): updated by the kernel in training
        # mode, used for the normalisation in eval mode -- exactly what the stock module does (transformer.py:34,38)
        def bn_state(m):
            if not m.track_running_stats or m.running_mean is None:
                return None
            return (m.running_mean, m.running_var, m.num_batches_tracked, m.momentum)
        training = self.training or bn_state(c[1]) is None or bn_state(c[4]) is None
        h = ops.EmbFrontendFn.apply(padded_input, c[0].weight, c[0].bias, c[1].weight, c[1].bias, c[3].weight, c[3].bias,
                                    c[4].weight, c[4].bias, float(c[1].eps), training, bn_state(c[1]), bn_state(c[4]))
        return h, None
    return ops.FlattenFn.apply(padded_input), None


def transformer_forward(self, padded_input, input_lengths, padded_target, verbose=False):
    """Transformer.forward -> (pred, gold, hyp_seq, gold_seq) -- models/asr/transformer.py:59-85.  Never computes attention
    maps: the reference discards them here."""
    ops._need_cuda(padded_input, padded_target)
    feats, cf = _front_end(self, padded_input)
    enc = _encoder_body(self.encoder, feats, input_lengths, cf)
    pred, gold = _decoder_body(self.decoder, padded_target, enc, input_lengths)
    hyp_seq = ops.argmax_rows(pred)
    return pred, gold, hyp_seq, gold


def transformer_evaluate(self, padded_input, input_lengths, padded_target, beam_search=False, beam_width=0, beam_nbest=0, lm=None,
                         lm_rescoring=False, lm_weight=0.1, c_weight=1, verbose=False):
    """Transformer.evaluate (models/asr/transformer.py:87-124) -> ([[None] * L, [None] * L], strs_hyps, strs_gold); while
    ops.attention_maps is on, the first value is [decoder self-attention maps, decoder encoder-attention maps] of the
    reference's teacher-forced decoder pass, which then runs (teacher_forced_maps) -- its topk still does not.

    The front end (_front_end: emb_cnn normalises with BatchNorm's running statistics in eval mode) and the encoder run on the
    device, then Decoder.beam_search (nbest=1; greedy_search when fewer than B strings come back, :112-118) or
    Decoder.greedy_search.  The reference's teacher-forced decoder pass and its topk (:107-108) only serve to produce `gold`
    and are skipped: gold comes from ops.preprocess_targets (raising like the reference for a target longer than
    tgt_max_len) in one device-to-host copy, and strs_gold joins id2label over all tgt_max_len entries, PAD included (:110).
    A model in training mode runs the reference's own method.

    In a process that has joined a data-parallel group (parallel.join, as install() does under b200asr.launch) each rank
    decodes its share of the batch and every rank returns the strings of the whole batch (evaluate_sharded); the attention
    maps, when on, are of the whole batch on every rank, without a collective."""
    if self.training:
        ref = _reference_method(self, "evaluate", "in training mode")
        return ref(self, padded_input, input_lengths, padded_target, beam_search=beam_search, beam_width=beam_width,
                   beam_nbest=beam_nbest, lm=lm, lm_rescoring=lm_rescoring, lm_weight=lm_weight, c_weight=c_weight,
                   verbose=verbose)
    ops._need_cuda(padded_input, padded_target)
    dec = self.decoder
    group = parallel.joined()
    n = len(dec.layers)
    maps = [[None] * n, [None] * n]
    if group is not None and not (beam_search and lm_rescoring and lstm_lm_parts(lm) is None):
        strs_hyps, strs_gold = evaluate_sharded(self, group, padded_input, input_lengths, padded_target, beam_search,
                                                beam_width, lm if lm_rescoring else None, lm_weight, c_weight)
        if ops.attention_maps_enabled():
            maps = teacher_forced_maps(self, padded_input, input_lengths, padded_target)
    else:
        strs_hyps, strs_gold, enc = _evaluate_whole(self, padded_input, input_lengths, padded_target, beam_search, beam_width,
                                                    lm, lm_rescoring, lm_weight, c_weight)
        if ops.attention_maps_enabled():
            maps = teacher_forced_maps(self, padded_input, input_lengths, padded_target, enc)
    if verbose:
        print("GOLD", strs_gold)
        print("HYP", strs_hyps)
    return maps, strs_hyps, strs_gold


def teacher_forced_maps(self, padded_input, input_lengths, padded_target, enc=None):
    """[decoder self-attention maps, decoder encoder-attention maps] of Transformer.evaluate's teacher-forced decoder pass
    (models/asr/transformer.py:106: `hyp, gold, *_ = self.decoder(...)` leaves them in `_`), over the whole batch; `enc` is
    the encoder output when the caller has it."""
    with torch.no_grad():
        if enc is None:
            feats, cf = _front_end(self, padded_input)
            enc = _encoder_body(self.encoder, feats, input_lengths, cf)
        self_maps, cross_maps = [], []
        _decoder_body(self.decoder, padded_target, enc, input_lengths, self_maps, cross_maps)
    return [self_maps, cross_maps]


def _gold_strings(self, padded_target):
    _, gold, _, _ = ops.preprocess_targets(padded_target, int(self.decoder.trg_max_length))
    return ["".join([self.id2label[x] for x in g]) for g in gold.cpu().tolist()]


def _evaluate_whole(self, padded_input, input_lengths, padded_target, beam_search, beam_width, lm, lm_rescoring, lm_weight,
                    c_weight):
    """(strs_hyps, strs_gold, encoder output) of the whole batch in this process."""
    dec = self.decoder
    with torch.no_grad():
        feats, cf = _front_end(self, padded_input)
        enc = _encoder_body(self.encoder, feats, input_lengths, cf)
        strs_gold = _gold_strings(self, padded_target)
        B = enc.shape[0]
        if beam_search:
            _, strs_hyps = dec.beam_search(enc, beam_width=beam_width, nbest=1, lm=lm, lm_rescoring=lm_rescoring,
                                           lm_weight=lm_weight, c_weight=c_weight)
            if len(strs_hyps) != B:
                print(">>>>>>> switch to greedy")
                strs_hyps = dec.greedy_search(enc)
        else:
            strs_hyps = dec.greedy_search(enc)
    return strs_hyps, strs_gold, enc


def encoded_frames(self, T: int) -> int:
    """Frames the front end makes of T input frames: the encoder's output length (T_e), from the shapes of the layers in
    self.conv alone (Conv2d / MaxPool2d along the time axis, the last one)."""
    if self.feat_extractor not in ("vgg_cnn", "emb_cnn"):
        return int(T)
    from torch.nn.modules.utils import _pair
    for m in self.conv:
        if isinstance(m, (nn.Conv2d, nn.MaxPool2d)):
            k, s, p, d = (_pair(m.kernel_size)[1], _pair(m.stride)[1], _pair(m.padding)[1], _pair(m.dilation)[1])
            T = (T + 2 * p - d * (k - 1) - 1) // s + 1
    return int(T)


def evaluate_sharded(self, group, padded_input, input_lengths, padded_target, beam_search=False, beam_width=0, lm=None,
                     lm_weight=0.1, c_weight=1):
    """(strs_hyps, strs_gold) of the whole batch, with this rank decoding utterances rank, rank + N, ... of it (group =
    (process group, rank, N) as parallel.joined() returns it).  The batch is sorted by length and a shard decodes until its
    slowest utterance ends, so a strided share gives every rank a similar mix where contiguous chunks would leave rank 0
    the longest utterances.  The front end and the encoder run on the shard at the batch's padded T; the gold strings come
    from the whole padded_target on every rank; the decode and the string assembly are decode_sharded's."""
    _, rank, world = group
    B = padded_input.shape[0]
    with torch.no_grad():
        strs_gold = _gold_strings(self, padded_target)
        enc = None
        if rank < B:
            rows = slice(rank, B, world)
            feats, cf = _front_end(self, padded_input[rows].contiguous())
            enc = _encoder_body(self.encoder, feats, input_lengths[rows].contiguous(), cf)
        Te = encoded_frames(self, padded_input.shape[-1])
        strs_hyps = decode_sharded(self.decoder, enc, B, Te, group, beam_search, beam_width, lm, lm_weight, c_weight)
    return strs_hyps, strs_gold


def decode_sharded(dec, enc, B, Te, group, beam_search=False, beam_width=0, lm=None, lm_weight=0.1, c_weight=1):
    """The strings of Transformer.evaluate's decode (transformer.py:112-118) for a batch of B utterances of which this rank
    holds the encoder outputs of rank, rank + N, ... (`enc`, None for an empty share; T_e frames).  Every rank returns the
    B strings in batch order.

    Greedy: greedy_decode_cached(300 steps, EOS stop on the device) on the share, one all-gather of the ids
    (parallel.gather_rows), greedy_strings.  Beam: beam_decode(nbest=1, LSTM LM rescoring when `lm` is given) on the share,
    one all-gather of [length | yseq] rows; an utterance of any rank that ended no hypothesis makes every rank print
    ">>>>>>> switch to greedy" and take the greedy path on its share, as one process does for the whole batch.  A rank with
    an empty share launches no kernel and joins every collective.  The positional-table checks run on every rank before
    the first collective, so every rank raises alike."""
    pg = group[0]
    if beam_search:
        _check_beam_positions(dec, Te, GREEDY_STEPS)
        S = min(GREEDY_STEPS, int(Te))
        rows = None
        if enc is not None:
            ids, lengths, _, _ = beam_decode(dec, enc, beam_width, nbest=1, c_weight=c_weight, steps=GREEDY_STEPS, lm=lm,
                                             lm_weight=lm_weight)
            rows = torch.cat([lengths.unsqueeze(-1), ids], dim=-1)
        both = parallel.gather_rows(rows, B, (1, S + 3), pg)
        if bool((both[:, 0, 0] > 0).all()):
            return beam_strings(both, dec.id2label)[1]
        print(">>>>>>> switch to greedy")
    _check_greedy_positions(dec)
    ids = greedy_decode_cached(dec, enc, steps=GREEDY_STEPS, stop_at_eos=True) if enc is not None else None
    return greedy_strings(parallel.gather_rows(ids, B, (GREEDY_STEPS,), pg).tolist(), dec.id2label)


# ------------------------------------------------------------------------------------------------ mirror classes
class PositionalEncoding(nn.Module):
    """models/common_layers.py:76-98."""

    def __init__(self, dim_model, max_length=2000):
        super().__init__()
        pe = torch.zeros(max_length, dim_model)
        position = torch.arange(0, max_length).unsqueeze(1).float()
        exp_term = torch.exp(torch.arange(0, dim_model, 2).float() * -(math.log(10000.0) / dim_model))
        pe[:, 0::2] = torch.sin(position * exp_term)
        pe[:, 1::2] = torch.cos(position * exp_term)
        self.register_buffer("pe", pe.unsqueeze(0))

    def forward(self, input):
        return self.pe[:, :input.size(1)]


class ScaledDotProductAttention(nn.Module):
    def __init__(self, temperature, attn_dropout=0.1):
        super().__init__()
        self.temperature = temperature
        self.dropout = nn.Dropout(attn_dropout)
        self.softmax = nn.Softmax(dim=2)

    forward = sdpa_forward


class MultiHeadAttention(nn.Module):
    def __init__(self, num_heads, dim_model, dim_key, dim_value, dropout=0.1):
        super().__init__()
        self.num_heads, self.dim_model, self.dim_key, self.dim_value = num_heads, dim_model, dim_key, dim_value
        self.query_linear = nn.Linear(dim_model, num_heads * dim_key)
        self.key_linear = nn.Linear(dim_model, num_heads * dim_key)
        self.value_linear = nn.Linear(dim_model, num_heads * dim_value)
        self.attention = ScaledDotProductAttention(temperature=float(dim_key) ** 0.5, attn_dropout=dropout)
        self.layer_norm = nn.LayerNorm(dim_model)
        self.output_linear = nn.Linear(num_heads * dim_value, dim_model)
        self.dropout = nn.Dropout(dropout)

    forward = mha_forward


class PositionwiseFeedForwardWithConv(nn.Module):
    def __init__(self, dim_model, dim_hidden, dropout=0.1):
        super().__init__()
        self.conv_1 = nn.Conv1d(dim_model, dim_hidden, 1)
        self.conv_2 = nn.Conv1d(dim_hidden, dim_model, 1)
        self.dropout = nn.Dropout(dropout)
        self.layer_norm = nn.LayerNorm(dim_model)

    forward = ffn_forward


class EncoderLayer(nn.Module):
    def __init__(self, num_heads, dim_model, dim_inner, dim_key, dim_value, dropout=0.1):
        super().__init__()
        self.self_attn = MultiHeadAttention(num_heads, dim_model, dim_key, dim_value, dropout=dropout)
        self.pos_ffn = PositionwiseFeedForwardWithConv(dim_model, dim_inner, dropout=dropout)

    forward = encoder_layer_forward


class Encoder(nn.Module):
    def __init__(self, num_layers, num_heads, dim_model, dim_key, dim_value, dim_input, dim_inner, dropout=0.1,
                 src_max_length=2500):
        super().__init__()
        self.dim_input, self.num_layers, self.num_heads = dim_input, num_layers, num_heads
        self.dim_model, self.dim_key, self.dim_value, self.dim_inner = dim_model, dim_key, dim_value, dim_inner
        self.src_max_length = src_max_length
        self.dropout = nn.Dropout(dropout)
        self.dropout_rate = dropout
        self.input_linear = nn.Linear(dim_input, dim_model)
        self.layer_norm_input = nn.LayerNorm(dim_model)
        self.positional_encoding = PositionalEncoding(dim_model, src_max_length)
        self.layers = nn.ModuleList([EncoderLayer(num_heads, dim_model, dim_inner, dim_key, dim_value, dropout=dropout)
                                     for _ in range(num_layers)])

    forward = encoder_forward


class DecoderLayer(nn.Module):
    def __init__(self, dim_model, dim_inner, num_heads, dim_key, dim_value, dropout=0.1):
        super().__init__()
        self.self_attn = MultiHeadAttention(num_heads, dim_model, dim_key, dim_value, dropout=dropout)
        self.encoder_attn = MultiHeadAttention(num_heads, dim_model, dim_key, dim_value, dropout=dropout)
        self.pos_ffn = PositionwiseFeedForwardWithConv(dim_model, dim_inner, dropout=dropout)

    forward = decoder_layer_forward


class Decoder(nn.Module):
    def __init__(self, id2label, num_src_vocab, num_trg_vocab, num_layers, num_heads, dim_emb, dim_model, dim_inner,
                 dim_key, dim_value, dropout=0.1, trg_max_length=1000, emb_trg_sharing=False):
        super().__init__()
        self.sos_id, self.eos_id = SOS_TOKEN, EOS_TOKEN
        self.id2label = id2label
        self.num_src_vocab, self.num_trg_vocab = num_src_vocab, num_trg_vocab
        self.num_layers, self.num_heads = num_layers, num_heads
        self.dim_emb, self.dim_model, self.dim_inner = dim_emb, dim_model, dim_inner
        self.dim_key, self.dim_value = dim_key, dim_value
        self.dropout_rate = dropout
        self.emb_trg_sharing = emb_trg_sharing
        self.trg_max_length = trg_max_length
        self.trg_embedding = nn.Embedding(num_trg_vocab, dim_emb, padding_idx=PAD_TOKEN)
        self.positional_encoding = PositionalEncoding(dim_model, max_length=trg_max_length)
        self.dropout = nn.Dropout(dropout)
        self.layers = nn.ModuleList([DecoderLayer(dim_model, dim_inner, num_heads, dim_key, dim_value, dropout=dropout)
                                     for _ in range(num_layers)])
        self.output_linear = nn.Linear(dim_model, num_trg_vocab, bias=False)
        if emb_trg_sharing:
            self.output_linear.weight = self.trg_embedding.weight
            self.x_logit_scale = dim_model ** -0.5
        else:
            self.x_logit_scale = 1.0

    forward = decoder_forward
    greedy_decode_ids = greedy_decode_ids
    greedy_decode_cached = greedy_decode_cached
    beam_decode = beam_decode
    beam_search = beam_search
    greedy_search = greedy_search


class Transformer(nn.Module):
    """models/asr/transformer.py:16-124: forward and evaluate."""

    def __init__(self, encoder, decoder, feat_extractor="vgg_cnn"):
        super().__init__()
        self.encoder, self.decoder = encoder, decoder
        self.id2label = decoder.id2label
        self.feat_extractor = feat_extractor
        if feat_extractor == "emb_cnn":
            self.conv = nn.Sequential(
                nn.Conv2d(1, 32, kernel_size=(41, 11), stride=(2, 2), padding=(0, 10)), nn.BatchNorm2d(32),
                nn.Hardtanh(0, 20, inplace=True),
                nn.Conv2d(32, 32, kernel_size=(21, 11), stride=(2, 1)), nn.BatchNorm2d(32),
                nn.Hardtanh(0, 20, inplace=True))
        elif feat_extractor == "vgg_cnn":
            self.conv = nn.Sequential(
                nn.Conv2d(1, 64, 3, stride=1, padding=1), nn.ReLU(), nn.Conv2d(64, 64, 3, stride=1, padding=1), nn.ReLU(),
                nn.MaxPool2d(2, stride=2),
                nn.Conv2d(64, 128, 3, stride=1, padding=1), nn.ReLU(), nn.Conv2d(128, 128, 3, stride=1, padding=1), nn.ReLU(),
                nn.MaxPool2d(2, stride=2))
        for p in self.parameters():      # transformer.py:55-57 (quirk Q4)
            if p.dim() > 1:
                nn.init.xavier_uniform_(p)

    forward = transformer_forward
    evaluate = transformer_evaluate


def rnn_model_forward(self, input, hidden):
    """RNNModel.forward (utils/lstm_utils.py:185-193) -> (decoded [T, B, ntoken], (h_n, c_n)) for rnn_type "LSTM": the
    embedding, the LSTM stack and both dropouts on the device (ops.lstm_stack; dropout only in train mode), the decoder
    through LinearFn.  Other recurrent types and a bidirectional, batch_first or projected LSTM run the reference's own
    forward (install.original)."""
    rnn = self.rnn
    if (getattr(self, "rnn_type", None) != "LSTM" or not isinstance(rnn, nn.LSTM) or rnn.bidirectional or rnn.batch_first
            or getattr(rnn, "proj_size", 0)):
        from .install import original
        ref = original(type(self), "forward")
        if ref is None:
            raise NotImplementedError(f"RNNModel.forward runs on the device for a unidirectional, sequence-first LSTM only "
                                      f"(rnn_type {getattr(self, 'rnn_type', None)!r})")
        return ref(self, input, hidden)
    p_drop = float(self.drop.p) if self.training else 0.0
    p_mid = float(rnn.dropout) if self.training and rnn.num_layers > 1 else 0.0
    out, hidden = ops.lstm_stack(self, input, hidden, p_emb=p_drop, p_mid=p_mid, p_out=p_drop)
    return ops.LinearFn.apply(out, self.decoder.weight, self.decoder.bias), hidden


class RNNModel(nn.Module):
    """utils/lstm_utils.py:138-201 with rnn_type "LSTM" (the only recurrent LM the reference's rescoring loads): the same
    submodules and state_dict names (encoder, rnn, decoder), so the reference's checkpoints load.  Beam-search rescoring
    runs on the device (ops.lstm_lm_nll_sums); forward (rnn_model_forward) trains it on the device."""

    def __init__(self, rnn_type, ntoken, ninp, nhid, nlayers, dropout=0.5, tie_weights=False):
        super().__init__()
        if rnn_type != "LSTM":
            raise ValueError(f"RNNModel: only rnn_type 'LSTM' is supported, got {rnn_type!r}")
        self.drop = nn.Dropout(dropout)
        self.encoder = nn.Embedding(ntoken, ninp)
        self.rnn = nn.LSTM(ninp, nhid, nlayers, dropout=dropout if nlayers > 1 else 0.0)
        self.decoder = nn.Linear(nhid, ntoken)
        if tie_weights:
            if nhid != ninp:
                raise ValueError("When using the tied flag, nhid must be equal to emsize")
            self.decoder.weight = self.encoder.weight
        self.rnn_type, self.nhid, self.nlayers = rnn_type, nhid, nlayers
        with torch.no_grad():
            self.encoder.weight.uniform_(-0.1, 0.1)
            self.decoder.bias.zero_()
            self.decoder.weight.uniform_(-0.1, 0.1)

    forward = rnn_model_forward

    def init_hidden(self, bsz):
        """utils/lstm_utils.py:195-199: the zero state (h0, c0), each [nlayers, bsz, nhid]."""
        weight = next(self.parameters())
        return (weight.new_zeros(self.nlayers, bsz, self.nhid), weight.new_zeros(self.nlayers, bsz, self.nhid))


class LM:
    """utils/lstm_utils.LM: loads the reference's LM checkpoint {word2idx, idx2word, ntoken, ninp, nhid, nlayers, dropout,
    tie_weights, model_state_dict} into an RNNModel.  Pass it as beam_search(..., lm_rescoring=True, lm=LM(path))."""

    def __init__(self, model_path):
        self.model_path = model_path
        ck = torch.load(model_path, map_location="cpu", weights_only=False)
        self.word2idx, self.idx2word = ck["word2idx"], ck["idx2word"]
        self.model = RNNModel("LSTM", ntoken=ck["ntoken"], ninp=ck["ninp"], nhid=ck["nhid"], nlayers=ck["nlayers"],
                              dropout=ck["dropout"], tie_weights=ck["tie_weights"])
        self.model.load_state_dict(ck["model_state_dict"])
        self.model.eval()


def build_model(cfg, id2label=None) -> Transformer:
    """Equivalent of utils/functions.py:116-152 (init_transformer_model) from an ASRConfig."""
    id2label = id2label or {i: str(i) for i in range(cfg.vocab)}
    enc = Encoder(cfg.num_layers, num_heads=cfg.num_heads, dim_model=cfg.dim_model, dim_key=cfg.dim_key,
                  dim_value=cfg.dim_value, dim_input=cfg.dim_input, dim_inner=cfg.dim_inner,
                  src_max_length=cfg.src_max_len, dropout=cfg.dropout)
    dec = Decoder(id2label, num_src_vocab=cfg.vocab, num_trg_vocab=cfg.vocab, num_layers=cfg.num_layers,
                  num_heads=cfg.num_heads, dim_emb=cfg.dim_model, dim_model=cfg.dim_model, dim_inner=cfg.dim_inner,
                  dim_key=cfg.dim_key, dim_value=cfg.dim_value, trg_max_length=cfg.tgt_max_len, dropout=cfg.dropout,
                  emb_trg_sharing=cfg.emb_trg_sharing)
    return Transformer(enc, dec, feat_extractor=cfg.feat_extractor)
