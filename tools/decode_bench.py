#!/usr/bin/env python
"""Beam-search decoding speed at cfg2's model dimensions (4 layers, d = 512, 8 heads of 64, inner 2048, V = 4364,
tgt_max_len = 301): B = 32 utterances of T_e = 200 encoder frames, beam widths 1, 4 and 8.

For Decoder.beam_decode it reports decoded utterances per second, the decode steps run and the kernel launches per step
(CUDA-event timed after one warm-up call).  In the same process, on the same card, it times the reference's own
Decoder.beam_search (one utterance at a time, full-prefix re-decode, the layer forwards on this package's kernels after
install()) on a few utterances of the same batch, checks that both return the same strings there, and prints the card's
name and power limit.  One JSON line per measurement.  Usage:
    python tools/decode_bench.py [--widths 1,4,8] [--ref-utts 2] [--reps 3] [--lm]
--lm decodes with LM rescoring (lm_rescoring=True) under an LSTM LM of ninp = nhid = 650, 2 layers, ntoken = 10 000 (random
weights; its vocabulary holds the label map's words): utt/s, the time split into decode, host segmentation and device LM
scoring, the ended hypotheses and LM positions, the algorithmic TFLOP/s of the LSTM layers (CUDA-event timed over the same
packed sequences), and the reference's own LM-rescored method on --ref-utts utterances with the same strings check.
The reference leg needs the reference checkout staged by oracle/make_ref.py (it is skipped without it)."""
import argparse
import importlib
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import b200asr  # noqa: E402
from oracle import ref_shim  # noqa: E402

ops = importlib.import_module(b200asr.__name__ + ".ops")
modules = importlib.import_module(b200asr.__name__ + ".modules")
FLAGS = ["--num-layers", "4", "--num-heads", "8", "--dim-model", "512", "--dim-emb", "512", "--dim-key", "64", "--dim-value", "64",
         "--dim-inner", "2048", "--feat_extractor", "", "--tgt-max-len", "301", "--dropout", "0.0", "--cuda"]
B, TE, V = 32, 200, 4364


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"device": torch.cuda.get_device_name(), "nvidia_smi": q.stdout.strip().splitlines()[:1]}


def timed(fn, reps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(reps):
        out = fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / 1e3 / reps, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--widths", default="1,4,8")
    ap.add_argument("--ref-utts", type=int, default=2)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--lm", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("decode_bench: no CUDA device (nothing is measured without one)")
    b200asr._lib.load(check_device=True)
    print(json.dumps({"card": card()}), flush=True)
    dev = torch.device("cuda")
    have_ref = ref_shim.available()
    if have_ref:       # the reference's own model class, so that both legs decode the very same weights
        ns = ref_shim.load(FLAGS, q12_shim=True)
        l2i, i2l = ref_shim.labels(V)
        torch.manual_seed(0)
        model = ns.functions.init_transformer_model(ns.constant.args, l2i, i2l)
        ref_beam = ns.transformer.Decoder.beam_search
        b200asr.install()
    else:
        cfg = b200asr.ASRConfig(num_layers=4, num_heads=8, dim_model=512, dim_key=64, dim_value=64, dim_inner=2048, vocab=V,
                                feat_extractor="", tgt_max_len=301, dropout=0.0)
        torch.manual_seed(0)
        model = b200asr.build_model(cfg)
    dec = model.decoder.to(dev).eval()
    g = torch.Generator().manual_seed(1)
    with torch.no_grad():
        dec.output_linear.weight.mul_(4.0)          # a trained model's logits are spread; xavier-init ones barely are
    enc = torch.randn(B, TE, 512, generator=g).to(dev)
    lib = b200asr._lib.load()
    if args.lm:
        return bench_lm(args, dec, enc, ns if have_ref else None)
    for W in [int(w) for w in args.widths.split(",")]:
        n_steps = [0]
        step = ops.beam_step

        def counting(*a, **k):
            n_steps[0] += 1
            return step(*a, **k)

        ops.beam_step = counting
        try:
            with torch.no_grad():
                modules.beam_decode(dec, enc, W, nbest=1, c_weight=0.1)            # warm-up
                n_steps[0] = 0
                l0 = lib.b200asr_launch_count()
                sec, (ids, lengths, _, _) = timed(lambda: modules.beam_decode(dec, enc, W, nbest=1, c_weight=0.1), args.reps)
                launches = (lib.b200asr_launch_count() - l0) / args.reps
        finally:
            ops.beam_step = step
        steps = n_steps[0] / args.reps
        rec = {"impl": "b200asr.beam_decode", "W": W, "B": B, "T_e": TE, "utt_per_s": round(B / sec, 2), "sec_per_call": round(sec, 4),
               "steps": steps, "launches_per_step": round(launches / steps, 1),
               "hyp_lengths_mean": round(float(lengths[:, 0].double().mean()), 1)}
        print(json.dumps(rec), flush=True)
        if have_ref and args.ref_utts > 0:
            n = args.ref_utts
            sub = enc[:n]
            t0 = time.perf_counter()
            with torch.no_grad():
                _, ref_strs = ref_beam(dec, sub, beam_width=W, nbest=1, c_weight=0.1)
            torch.cuda.synchronize()
            ref_sec = time.perf_counter() - t0
            with torch.no_grad():
                _, strs = dec.beam_search(sub, beam_width=W, nbest=1, c_weight=0.1)
            print(json.dumps({"impl": "reference Decoder.beam_search (installed layer forwards)", "W": W, "utterances": n,
                              "T_e": TE, "utt_per_s": round(n / ref_sec, 3), "sec": round(ref_sec, 2),
                              "same_strings_as_beam_search": strs == ref_strs}), flush=True)
    if have_ref:
        b200asr.uninstall()


LM_NINP = LM_NHID = 650
LM_LAYERS, LM_NTOKEN = 2, 10000


class BenchLM:
    """An LSTM LM with the mirror's RNNModel (the reference's LM class reads the same checkpoint)."""

    def __init__(self, labels, dev):
        words = ["<eos>", "<oov>"] + sorted({w for s in labels for w in s.split()})
        words += [f"w{i}" for i in range(LM_NTOKEN - len(words))]
        self.word2idx = {w: i for i, w in enumerate(words[:LM_NTOKEN])}
        self.idx2word = words[:LM_NTOKEN]
        torch.manual_seed(2)
        self.model = b200asr.RNNModel("LSTM", LM_NTOKEN, LM_NINP, LM_NHID, LM_LAYERS, dropout=0.0).to(dev).eval()


def bench_lm(args, dec, enc, ns):
    dev = enc.device
    lm = BenchLM([str(v) for v in dec.id2label.values()], dev)
    ref_lm = None
    if ns is not None and args.ref_utts > 0:
        import tempfile
        lstm_utils = importlib.import_module("utils.lstm_utils")
        path = os.path.join(tempfile.mkdtemp(), "lm.pt")
        torch.save(dict(word2idx=lm.word2idx, idx2word=lm.idx2word, ntoken=LM_NTOKEN, ninp=LM_NINP, nhid=LM_NHID, nlayers=LM_LAYERS,
                        dropout=0.0, tie_weights=False, model_state_dict=lm.model.state_dict()), path)
        ref_lm = lstm_utils.LM(path)
    seen = []
    score_fn = ops.lstm_lm_nll_sums

    def capture(model, seqs, device):
        seen.append(seqs)
        return score_fn(model, seqs, device)

    for W in [int(w) for w in args.widths.split(",")]:
        ops.lstm_lm_nll_sums = capture
        try:
            with torch.no_grad():
                modules.beam_decode(dec, enc, W, nbest=1, c_weight=0.1, lm=lm, lm_weight=0.1)          # warm-up
                tot = host = lm_s = 0.0
                for _ in range(args.reps):
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    modules.beam_decode(dec, enc, W, nbest=1, c_weight=0.1, lm=lm, lm_weight=0.1)
                    torch.cuda.synchronize()
                    tot += time.perf_counter() - t0
                    host += modules.lm_rescore_stats["host_s"]
                    lm_s += modules.lm_rescore_stats["lm_s"]
        finally:
            ops.lstm_lm_nll_sums = score_fn
        st = dict(modules.lm_rescore_stats)
        r = args.reps
        # the LSTM layers alone over the same packed sequences: CUDA events around ops.lstm_lm_layers
        seqs = seen[-1]
        import numpy as np
        lens = np.array([len(q) - 1 for q in seqs])
        order = np.argsort(-lens, kind="stable")
        Mt = np.array([(lens > t).sum() for t in range(int(lens.max()))])
        off = np.concatenate([[0], np.cumsum(Mt)[:-1]])
        inp = np.empty(int(Mt.sum()), dtype=np.int64)
        for j, s in enumerate(order):
            inp[off[:lens[s]] + j] = seqs[s][:-1]
        inp_d = torch.from_numpy(inp).to(dev)
        op = ops.lstm_lm_operands(lm.model, dev)
        ops.lstm_lm_layers(op, inp_d, Mt)
        sec_lstm, _ = timed(lambda: ops.lstm_lm_layers(op, inp_d, Mt), 10)
        P = int(Mt.sum())
        flops = sum(2 * P * 4 * LM_NHID * ((LM_NINP if l == 0 else LM_NHID) + LM_NHID) for l in range(LM_LAYERS))
        print(json.dumps({"impl": "b200asr.beam_decode(lm)", "W": W, "B": B, "T_e": TE, "utt_per_s": round(B * r / tot, 2),
                          "sec_per_call": round(tot / r, 4), "decode_s": round((tot - host - lm_s) / r, 4),
                          "host_segmentation_s": round(host / r, 4), "device_lm_s": round(lm_s / r, 4),
                          "ended_hypotheses": st["ended"], "lm_sequences": st["sequences"], "lm_positions": st["positions"],
                          "lstm_steps": len(Mt), "lstm_layers_s": round(sec_lstm, 5),
                          "lstm_layers_tflops": round(flops / sec_lstm / 1e12, 3)}), flush=True)
        if ref_lm is not None:
            n = args.ref_utts
            sub = enc[:n]
            ref_beam = importlib.import_module(b200asr.__name__ + ".install").original(type(dec), "beam_search")
            t0 = time.perf_counter()
            with torch.no_grad():
                _, ref_strs = ref_beam(dec, sub, beam_width=W, nbest=1, lm_rescoring=True, lm=ref_lm, lm_weight=0.1, c_weight=0.1)
            torch.cuda.synchronize()
            ref_sec = time.perf_counter() - t0
            with torch.no_grad():
                _, strs = dec.beam_search(sub, beam_width=W, nbest=1, lm_rescoring=True, lm=ref_lm, lm_weight=0.1, c_weight=0.1)
            print(json.dumps({"impl": "reference Decoder.beam_search lm_rescoring (installed layer forwards)", "W": W,
                              "utterances": n, "T_e": TE, "utt_per_s": round(n / ref_sec, 4), "sec": round(ref_sec, 2),
                              "same_strings_as_beam_search": strs == ref_strs}), flush=True)
    if ns is not None:
        b200asr.uninstall()


if __name__ == "__main__":
    main()
