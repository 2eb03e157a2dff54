#!/usr/bin/env python
"""Decoding throughput of the installed Transformer.evaluate, in one process and data-parallel (modules.evaluate_sharded):
greedy, beam width 4 and beam width 4 with an LSTM LM rescoring, at the decoder sizes of tools/decode_bench.py (cfg2: 4
layers, d = 512, 8 heads of 64, inner 2048, V = 4364), B = 32 utterances of T_e = 200 frames (feat_extractor '', random
weights, the EOS row scaled so that utterances end at different steps).

    python tools/dp_decode_time.py [--ranks 2] [--share-gpu] [--reps 3] [--modes greedy,beam4,beam4-lm]

Every arm runs in processes of its own: first 1 process, then --ranks ranks.  The ranks use one GPU each (NCCL) when the
machine has that many, or share GPU 0 over gloo with --share-gpu (or when it has fewer).  Ranks sharing a GPU check the
per-batch protocol and its overhead, not scaling: their kernels compete for one device.  One JSON line per measurement
(utt/s timed with CUDA events around --reps calls after one warm-up call, on rank 0, between two barriers), with the
card's name and power limit."""
import argparse
import json
import os
import socket
import subprocess
import sys
import time
import types

import torch
import torch.distributed as dist
import torch.multiprocessing as mp

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

B, TE, V = 32, 200, 4364
LM_NTOKEN, LM_NINP, LM_NHID, LM_LAYERS = 10000, 650, 650, 2          # tools/decode_bench.py --lm


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return {"device": torch.cuda.get_device_name(), "nvidia_smi": q.stdout.strip().splitlines()[:1]}


def build(dev):
    import b200asr
    labels = {i: c for i, c in enumerate(["¶", "§", "¤"] + [chr(0x4E00 + i) for i in range(V - 3)])}
    cfg = b200asr.ASRConfig(num_layers=4, num_heads=8, dim_model=512, dim_key=64, dim_value=64, dim_inner=2048, vocab=V,
                            feat_extractor="", tgt_max_len=301, dropout=0.0)
    torch.manual_seed(0)
    model = b200asr.build_model(cfg, id2label=labels)
    with torch.no_grad():
        model.decoder.output_linear.weight.mul_(4.0)
        model.decoder.output_linear.weight[2].mul_(1.5)
    words = ["<eos>", "<oov>"] + list(labels.values())[3:]
    words += [f"w{i}" for i in range(LM_NTOKEN - len(words))]
    rnn = b200asr.RNNModel("LSTM", LM_NTOKEN, LM_NINP, LM_NHID, LM_LAYERS, dropout=0.0)
    lm = types.SimpleNamespace(model=rnn.to(dev).eval(), word2idx={w: i for i, w in enumerate(words)})
    g = torch.Generator().manual_seed(1)
    src = torch.randn(B, 1, 161, TE, generator=g).to(dev)
    lens = torch.full((B,), TE, dtype=torch.int32).to(dev)
    tgt = torch.randint(3, V, (B, 20), generator=g).to(dev)
    return model.to(dev).eval(), lm, (src, lens, tgt)


MODES = {"greedy": dict(beam_search=False), "beam4": dict(beam_search=True, beam_width=4),
         "beam4-lm": dict(beam_search=True, beam_width=4, lm_rescoring=True)}


def arm(rank, world, port, backend, modes, reps, out_path):
    import b200asr
    from b200asr import parallel
    if backend == "nccl":
        torch.cuda.set_device(rank)
    dev = torch.device("cuda", torch.cuda.current_device())
    if world > 1:
        os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
        dist.init_process_group(backend, rank=rank, world_size=world)
        parallel.join(dist.group.WORLD)
    model, lm, (src, lens, tgt) = build(dev)
    rows = []
    for mode in modes:
        kw = dict(MODES[mode], beam_nbest=1, c_weight=0.1, lm=lm if mode.endswith("-lm") else None)
        with torch.no_grad():
            _, hyps, _ = model.evaluate(src, lens, tgt, **kw)                  # warm-up
            if world > 1:
                dist.barrier()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            e0.record()
            for _ in range(reps):
                _, hyps, _ = model.evaluate(src, lens, tgt, **kw)
            e1.record()
            torch.cuda.synchronize()
            wall = time.perf_counter() - t0
            if world > 1:
                dist.barrier()
        s = e0.elapsed_time(e1) / 1e3 / reps
        rows.append(dict(mode=mode, ranks=world, backend=backend if world > 1 else None, B=B, T_e=TE, seconds_per_batch=s,
                         utt_per_s=B / s, wall_utt_per_s=B * reps / wall, mean_hyp_len=sum(map(len, hyps)) / len(hyps)))
    parallel.leave()
    if rank == 0:
        torch.save(rows, out_path)
    if world > 1:
        dist.destroy_process_group()


def run(world, backend, modes, reps, tmp):
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    path = os.path.join(tmp, f"rows{world}.pt")
    mp.start_processes(arm, args=(world, port, backend, modes, reps, path), nprocs=world, join=True, start_method="spawn")
    return torch.load(path)


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--ranks", type=int, default=2)
    ap.add_argument("--share-gpu", action="store_true", help="every rank on GPU 0 (gloo)")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--modes", default="greedy,beam4,beam4-lm")
    args = ap.parse_args()
    modes = [m for m in args.modes.split(",") if m]
    shared = args.share_gpu or torch.cuda.device_count() < args.ranks
    backend = "gloo" if shared else "nccl"
    print(json.dumps(dict(card(), gpus=torch.cuda.device_count())), flush=True)
    import tempfile
    with tempfile.TemporaryDirectory() as tmp:
        one = {r["mode"]: r for r in run(1, "nccl", modes, args.reps, tmp)}
        many = {r["mode"]: r for r in run(args.ranks, backend, modes, args.reps, tmp)}
    note = (f"{args.ranks} ranks share one GPU over gloo: this checks the per-batch protocol and its overhead, not scaling"
            if shared else f"{args.ranks} ranks on {args.ranks} GPUs over NCCL")
    for m in modes:
        print(json.dumps(one[m]), flush=True)
        print(json.dumps(dict(many[m], speedup_vs_1_process=many[m]["utt_per_s"] / one[m]["utt_per_s"], note=note)), flush=True)


if __name__ == "__main__":
    main()
