#!/usr/bin/env python
"""Beam-search decoding speed at cfg2's model dimensions (4 layers, d = 512, 8 heads of 64, inner 2048, V = 4364,
tgt_max_len = 301): B = 32 utterances of T_e = 200 encoder frames, beam widths 1, 4 and 8.

For Decoder.beam_decode it reports decoded utterances per second, the decode steps run and the kernel launches per step
(CUDA-event timed after one warm-up call).  In the same process, on the same card, it times the reference's own
Decoder.beam_search (one utterance at a time, full-prefix re-decode, the layer forwards on this package's kernels after
install()) on a few utterances of the same batch, checks that both return the same strings there, and prints the card's
name and power limit.  One JSON line per measurement.  Usage:
    python tools/decode_bench.py [--widths 1,4,8] [--ref-utts 2] [--reps 3] [--lm | --greedy | --kernels]
--greedy times Decoder.greedy_search (installed: KV-cached, split-key attention, EOS stop on the device) against the
reference's own greedy_search on --ref-utts utterances (same strings check), then Transformer.evaluate greedy and with beam
width 4, vgg_cnn front end on random spectrograms of 800 frames (T_e = 200), installed against the reference's own evaluate
body; both run install()'s layer forwards and decode methods, so the difference is the reference's cuDNN front end, its
teacher-forced decoder pass, topk and per-element gold syncs.  --kernels times, with torch.profiler (kernel time only), one
single-query attention call of decode_attn, beam_self_attn (W = 1) and the SdpaFn Tq = 1 path at B = 32, H = 8, d = 64 over
T_e in {200, 500} (cross) and t in {16, 128} (self) keys, and the achieved GB/s of the K/V bytes read.
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
    ap.add_argument("--greedy", action="store_true")
    ap.add_argument("--kernels", action="store_true")
    args = ap.parse_args()
    if args.kernels:
        return bench_kernels()
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
    if args.greedy:
        return bench_greedy(args, dec, enc, ns if have_ref else None)
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


def bench_greedy(args, dec, enc, ns):
    lib = b200asr._lib.load()
    n_steps = [0]
    step = ops.greedy_step

    def counting(*a, **k):
        n_steps[0] += 1
        return step(*a, **k)

    ops.greedy_step = counting
    try:
        with torch.no_grad():
            modules.greedy_search(dec, enc)                                 # warm-up
            n_steps[0] = 0
            l0 = lib.b200asr_launch_count()
            sec, strs = timed(lambda: modules.greedy_search(dec, enc), args.reps)
            launches = (lib.b200asr_launch_count() - l0) / args.reps
    finally:
        ops.greedy_step = step
    steps = n_steps[0] / args.reps
    print(json.dumps({"impl": "b200asr Decoder.greedy_search", "B": B, "T_e": TE, "utt_per_s": round(B / sec, 2),
                      "sec_per_call": round(sec, 4), "steps": steps, "launches_per_step": round(launches / steps, 1),
                      "hyp_chars_mean": round(sum(map(len, strs)) / B, 1)}), flush=True)
    install = importlib.import_module(b200asr.__name__ + ".install")
    if ns is not None and args.ref_utts > 0:
        n = args.ref_utts
        sub = enc[:n]
        ref_greedy = install.original(type(dec), "greedy_search")
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        with torch.no_grad():
            ref_strs = ref_greedy(dec, sub)
        torch.cuda.synchronize()
        ref_sec = time.perf_counter() - t0
        with torch.no_grad():
            got = modules.greedy_search(dec, sub)
        print(json.dumps({"impl": "reference Decoder.greedy_search (installed layer forwards)", "utterances": n, "T_e": TE,
                          "utt_per_s": round(n / ref_sec, 3), "sec": round(ref_sec, 2),
                          "same_strings_as_greedy_search": got == ref_strs}), flush=True)

    # Transformer.evaluate with the vgg_cnn front end: 800 frames -> T_e = 200
    T = 4 * TE
    if ns is not None:
        ns_v = ref_shim.load([f if f != "" else "vgg_cnn" for f in FLAGS], q12_shim=True)
        l2i, i2l = ref_shim.labels(V)
        torch.manual_seed(0)
        model = ns_v.functions.init_transformer_model(ns_v.constant.args, l2i, i2l)
    else:
        cfg = b200asr.ASRConfig(num_layers=4, num_heads=8, dim_model=512, dim_key=64, dim_value=64, dim_inner=2048, vocab=V,
                                feat_extractor="vgg_cnn", tgt_max_len=301, dropout=0.0)
        torch.manual_seed(0)
        model = b200asr.build_model(cfg)
    model = model.to(enc.device).eval()
    with torch.no_grad():
        model.decoder.output_linear.weight.mul_(4.0)
    g = torch.Generator().manual_seed(3)
    src = torch.randn(B, 1, 161, T, generator=g).to(enc.device)
    lens = torch.full((B,), T, dtype=torch.int32).to(enc.device)
    tgt = torch.randint(3, V, (B, 40), generator=g).to(enc.device)
    ref_eval = install.original(type(model), "evaluate") if ns is not None else None
    for beam in (False, True):
        kw = dict(beam_search=beam, beam_width=4, beam_nbest=1, c_weight=0.1)
        legs = [("b200asr Transformer.evaluate", lambda: modules.transformer_evaluate(model, src, lens, tgt, **kw))]
        if ref_eval is not None:
            legs.append(("reference Transformer.evaluate (installed layer forwards and decode methods)",
                         lambda: ref_eval(model, src, lens, tgt, **kw)))
        outs = []
        for name, fn in legs:
            with torch.no_grad():
                fn()                                                         # warm-up
                sec, out = timed(fn, args.reps)
            outs.append(out[1:])
            print(json.dumps({"impl": name, "decode": "beam W=4" if beam else "greedy", "feat_extractor": "vgg_cnn", "B": B,
                              "frames": T, "utt_per_s": round(B / sec, 2), "sec_per_call": round(sec, 4)}), flush=True)
        if len(outs) == 2:
            print(json.dumps({"decode": "beam W=4" if beam else "greedy", "same_hyps_and_gold": outs[0] == outs[1]}), flush=True)


def bench_kernels(reps=200):
    """Kernel time per call (torch.profiler, CUDA activity only) of three single-query attention paths."""
    if not torch.cuda.is_available():
        raise SystemExit("decode_bench: no CUDA device (nothing is measured without one)")
    b200asr._lib.load(check_device=True)
    print(json.dumps({"card": card()}), flush=True)
    from torch.profiler import ProfilerActivity, profile
    dev = torch.device("cuda")
    H, d, HBM = 8, 64, 3.35e12
    scale = 1.0 / d ** 0.5
    g = torch.Generator(device=dev).manual_seed(0)
    for kind, Tk in (("cross", 200), ("cross", 500), ("self", 16), ("self", 128)):
        q = torch.randn(B, H * d, generator=g, device=dev)
        kp, vp = (torch.randn(B, Tk, H * d, generator=g, device=dev) for _ in range(2))     # token-major [B, Tk, H*d]
        kc, vc = kp.transpose(0, 1).contiguous(), vp.transpose(0, 1).contiguous()          # slab-major [Tk, B, H*d]
        if kind == "cross":
            da = lambda: ops.decode_attn(q, kp, vp, H, Tk, (Tk * H * d, H * d), (Tk * H * d, H * d), d, scale)
        else:
            da = lambda: ops.decode_attn(q, kc, vc, H, Tk, (H * d, B * H * d), (H * d, B * H * d), d, scale)
        idx = torch.zeros((B, Tk), dtype=torch.int32, device=dev)
        q4 = q.view(B, 1, H, d).permute(0, 2, 1, 3)
        k4, v4 = kp.view(B, Tk, H, d).permute(0, 2, 1, 3), vp.view(B, Tk, H, d).permute(0, 2, 1, 3)
        calls = {"decode_attn": da,
                 "beam_self_attn W=1": lambda: ops.beam_self_attn(q, kc, vc, idx, 1, H, Tk - 1, scale),
                 "SdpaFn Tq=1": lambda: ops.SdpaFn.apply(q4, k4, v4, None, None, False, scale, 0.0)}
        ref = calls["decode_attn"]().view(B, H, d)
        nbytes = 2 * B * Tk * H * d * 4 + 2 * B * H * d * 4          # K, V read once; q read, out written
        for name, fn in calls.items():
            with torch.no_grad():
                o = fn().reshape(B, H, d)
                for _ in range(5):
                    fn()
                torch.cuda.synchronize()
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    for _ in range(reps):
                        fn()
                    torch.cuda.synchronize()
                call_s, _ = timed(fn, reps)
            kern_us = sum(getattr(e, "self_device_time_total", 0.0) for e in prof.key_averages()) / reps
            print(json.dumps({"kernel": name, "attention": kind, "B": B, "H": H, "d": d, "keys": Tk,
                              "kernel_us_per_call": round(kern_us, 2), "call_us_events": round(call_s * 1e6, 2),
                              "GB_per_s": round(nbytes / (kern_us * 1e-6) / 1e9, 1),
                              "share_of_3.35TB_s": round(nbytes / (kern_us * 1e-6) / HBM, 3),
                              "max_abs_diff_vs_decode_attn": float((o - ref).abs().max())}), flush=True)


if __name__ == "__main__":
    main()
