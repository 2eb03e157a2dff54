#!/usr/bin/env python
"""Beam-search decoding speed at cfg2's model dimensions (4 layers, d = 512, 8 heads of 64, inner 2048, V = 4364,
tgt_max_len = 301): B = 32 utterances of T_e = 200 encoder frames, beam widths 1, 4 and 8.

For Decoder.beam_decode it reports decoded utterances per second, the decode steps run and the kernel launches per step
(CUDA-event timed after one warm-up call).  In the same process, on the same card, it times the reference's own
Decoder.beam_search (one utterance at a time, full-prefix re-decode, the layer forwards on this package's kernels after
install()) on a few utterances of the same batch, checks that both return the same strings there, and prints the card's
name and power limit.  One JSON line per measurement.  Usage:
    python tools/decode_bench.py [--widths 1,4,8] [--ref-utts 2] [--reps 3]
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


if __name__ == "__main__":
    main()
