#!/usr/bin/env python
"""Iterations/s and utterances/s of the installed reference Trainer.train at N data-parallel ranks.

    python tools/dp_trainer_time.py [--ranks 1 2 4 8] [--iters 8] [--reps 2] [--batch 32] [--share]

Each N runs as N processes (one per GPU, NCCL; with --share all N on GPU 0 over gloo, which exercises the protocol but
measures no scaling).  Needs the reference staged in oracle/_ref (oracle/make_ref.py).  Model: vgg_cnn, 4 layers,
d_model 512, 8 heads, d_inner 2048, 4364 labels, --label-smoothing 0.1, --clip, dropout 0.  Every rank's loader yields the
same global batches of `batch` utterances (_collate_fn-shaped, T_src = 800 frames of 161 bins, targets of up to 99
labels), of which each rank trains its shard.  Time per iteration: rank 0's host clock between the second and the last
batch its progress bar hands out, first epoch not counted (every iteration ends in a host read of the reduced row, so
the clock follows the device).  utt/s = global batch / time per iteration.  The card, its power limit and SM clock are
read in the same run.
"""
import argparse
import json
import os
import socket
import sys
import tempfile
import time

import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.trainer_time import CFG2, FREQ, T_SRC, VOCAB  # noqa: E402


class Bar:
    marks = []

    def __init__(self, it, leave=True, total=None):
        self.it = it

    def __iter__(self):
        for x in self.it:
            Bar.marks.append(time.perf_counter())
            yield x
        Bar.marks.append(time.perf_counter())

    def set_description(self, s):
        pass


def batch(seed, Lt, B):
    g = torch.Generator().manual_seed(seed)
    src = torch.randn(B, 1, FREQ, T_SRC, generator=g)
    lens = torch.sort((T_SRC * (0.5 + 0.5 * torch.rand(B, generator=g))).long().clamp(1, T_SRC), descending=True).values
    lens[0] = T_SRC
    for i in range(B):
        src[i, :, :, int(lens[i]):] = 0
    tgt = torch.randint(3, VOCAB, (B, Lt), generator=g)
    tl = (Lt * (0.4 + 0.6 * torch.rand(B, generator=g))).long().clamp(1, Lt)
    tl[0] = Lt
    for i in range(B):
        tgt[i, int(tl[i]):] = 0
    return src, tgt, lens.float() / T_SRC, lens.to(torch.int32), tl.to(torch.int32)


def rank_main(rank, world, port, args, out):
    import b200asr
    from oracle import ref_shim
    from tools.features_time import gpu_info
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    if not args.share:
        torch.cuda.set_device(rank)
    if world > 1:
        dist.init_process_group("gloo" if args.share else "nccl", rank=rank, world_size=world,
                                device_id=None if args.share else torch.device("cuda", rank))
    ns = ref_shim.load(CFG2)
    l2i, i2l = ref_shim.labels(VOCAB)
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.manual_seed(0)
    model = ns.functions.init_transformer_model(ns.constant.args, l2i, i2l).cuda()
    opt = ns.functions.init_optimizer(ns.constant.args, model, "noam")
    Lt = ns.constant.args.tgt_max_len - 2
    train = [batch(s, Lt, args.batch) for s in range(args.iters)]
    valid = [batch(1000, Lt, args.batch)]
    times = []
    with tempfile.TemporaryDirectory() as tmp:
        ns.constant.args.save_folder, ns.constant.args.name = tmp, "t"
        ns.trainer.tqdm = Bar
        b200asr.install(process_group=dist.group.WORLD if world > 1 else None)
        try:
            for rep in range(args.reps + 1):
                Bar.marks = []
                tr = [tuple(x.clone() for x in b) for b in train]       # the loop scales src_percentages in place
                va = [[tuple(x.clone() for x in b) for b in valid]]
                ns.trainer.Trainer().train(model, tr, None, va, opt, "ce", 0, 1, l2i, i2l)
                m = Bar.marks[:len(train) + 1]                          # rank 0 draws the bar
                if rep and rank == 0:
                    times.append((m[-1] - m[1]) * 1e3 / (len(m) - 2))
        finally:
            b200asr.uninstall()
    if rank == 0:
        ms = min(times)
        with open(out, "w") as f:
            json.dump({"ranks": world, "share": args.share, "B_global": args.batch, "ms_per_iter": sorted(times),
                       "it_per_s": round(1e3 / ms, 3), "utt_per_s": round(args.batch * 1e3 / ms, 1), "card": gpu_info()}, f)
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ranks", type=int, nargs="+", default=[1, 2, 4, 8])
    ap.add_argument("--iters", type=int, default=8)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--share", action="store_true", help="all ranks on GPU 0 over gloo (protocol check, not scaling)")
    args = ap.parse_args()
    n_gpu = torch.cuda.device_count()
    results = []
    for world in args.ranks:
        if not args.share and world > n_gpu:
            results.append({"ranks": world, "skipped": f"{n_gpu} GPU(s) visible"})
            continue
        with socket.socket() as s:
            s.bind(("127.0.0.1", 0))
            port = s.getsockname()[1]
        with tempfile.TemporaryDirectory() as tmp:
            out = os.path.join(tmp, "r.json")
            mp.start_processes(rank_main, args=(world, port, args, out), nprocs=world, join=True, start_method="spawn")
            with open(out) as f:
                results.append(json.load(f))
        print(json.dumps(results[-1]), flush=True)
    print(json.dumps({"dp_trainer_time": results}))


if __name__ == "__main__":
    main()
