#!/usr/bin/env python
"""Time per iteration and host syncs per iteration of the reference's Trainer.train at cfg2 shapes, installed, with the
reference's own loop and with the bound one (trainer.trainer_train), and b200asr_edit_counts alone.

    python tools/trainer_time.py [--iters 8] [--reps 3]

Needs the reference staged in oracle/_ref (oracle/make_ref.py).  Model: vgg_cnn, 4 layers, d_model 512, 8 heads, d_inner 2048,
4364 labels (one CJK character each), --label-smoothing 0.1, --clip.  Batches: _collate_fn-shaped, B = 32, T_src = 800
frames of 161 bins, targets of up to 99 labels (T_t = 100 with EOS), src and tgt on the device.  The two arms run
alternately in one process, `reps` epochs each, `iters` training batches and one validation batch per epoch.  Time per
iteration: host clock between the second and the last batch the loop takes from its progress bar (every iteration ends in a
host read, so the clock follows the device), first epoch of each arm not counted.  Host syncs per iteration: torch's sync
debug mode, in a separate epoch per arm.  b200asr_edit_counts alone: CUDA events over 200 calls at B = 32, T_t = 100 and
1000.  The card, its power limit and max SM clock are read in the same run.
"""
import argparse
import json
import os
import sys
import tempfile
import time
import warnings

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import b200asr  # noqa: E402
from oracle import ref_shim  # noqa: E402
from tools.features_time import gpu_info, timed  # noqa: E402

CFG2 = ["--num-layers", "4", "--num-heads", "8", "--dim-model", "512", "--dim-emb", "512", "--dim-key", "64", "--dim-value", "64",
        "--dim-inner", "2048", "--feat_extractor", "vgg_cnn", "--tgt-max-len", "101", "--dropout", "0.0",
        "--label-smoothing", "0.1", "--cuda", "--clip", "--max-norm", "400"]
VOCAB, B, T_SRC, FREQ = 4364, 32, 800, 161


class Bar:
    """tqdm stand-in: the host time (and sync count) at which each batch is handed out."""
    marks, syncs = [], None

    def __init__(self, it, leave=True, total=None):
        self.it = it

    def __iter__(self):
        for x in self.it:
            Bar.marks.append((time.perf_counter(), len(Bar.syncs) if Bar.syncs is not None else 0))
            yield x
        Bar.marks.append((time.perf_counter(), len(Bar.syncs) if Bar.syncs is not None else 0))

    def set_description(self, s):
        pass


def batch(seed, Lt):
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
    return src.cuda(), tgt.cuda(), lens.float() / T_SRC, lens.to(torch.int32), tl.to(torch.int32)


def epoch(ns, model, l2i, i2l, opt, train, valid, bound, count_syncs):
    """One epoch of the installed Trainer.train; returns (ms per iteration, syncs per iteration)."""
    Bar.marks = []
    trainer = ns.trainer.Trainer()
    tr = [tuple(x.clone() for x in b) for b in train]                 # the loop scales src_percentages in place
    va = [[tuple(x.clone() for x in b) for b in valid]]
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        if count_syncs:
            Bar.syncs = caught
            torch.cuda.set_sync_debug_mode("warn")
        try:
            if bound:
                trainer.train(model, tr, None, va, opt, "ce", 0, 1, l2i, i2l)
            else:
                b200asr.original(ns.trainer.Trainer, "train")(trainer, model, tr, None, va, opt, "ce", 0, 1, l2i, i2l)
        finally:
            torch.cuda.set_sync_debug_mode("default")
            Bar.syncs = None
    m = Bar.marks[:len(train) + 1]
    ms = (m[-1][0] - m[1][0]) * 1e3 / (len(m) - 2)
    syncs = [b[1] - a[1] for a, b in zip(m[1:], m[2:])]
    return ms, syncs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=8)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    b200asr._lib.load(check_device=True)
    if not ref_shim.available():
        raise SystemExit("the reference is not staged in oracle/_ref (run oracle/make_ref.py)")
    print("card:", gpu_info())
    ns = ref_shim.load(CFG2)
    l2i, i2l = ref_shim.labels(VOCAB)
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.manual_seed(0)
    model = ns.functions.init_transformer_model(ns.constant.args, l2i, i2l).cuda()
    opt = ns.functions.init_optimizer(ns.constant.args, model, "noam")
    Lt = ns.constant.args.tgt_max_len - 2
    train = [batch(s, Lt) for s in range(args.iters)]
    valid = [batch(1000, Lt)]
    result = {"card": gpu_info(), "B": B, "T_src": T_SRC, "T_t": Lt + 1, "iters": args.iters}
    with tempfile.TemporaryDirectory() as tmp:
        ns.constant.args.save_folder, ns.constant.args.name = tmp, "t"
        ns.trainer.tqdm = Bar
        b200asr.install()
        try:
            times = {False: [], True: []}
            for rep in range(args.reps + 1):
                for bound in (False, True):
                    ms, _ = epoch(ns, model, l2i, i2l, opt, train, valid, bound, False)
                    if rep:
                        times[bound].append(ms)
                    print(f"rep {rep} {'bound' if bound else 'reference'} loop: {ms:.1f} ms/iteration", flush=True)
            for bound in (False, True):
                name = "bound" if bound else "reference"
                _, syncs = epoch(ns, model, l2i, i2l, opt, train, valid, bound, True)
                result[f"{name}_ms_per_iter"] = sorted(times[bound])
                result[f"{name}_syncs_per_iter"] = syncs
        finally:
            b200asr.uninstall()
    table = b200asr.LabelTable(i2l, 0, (ns.constant.SOS_CHAR, ns.constant.EOS_CHAR))
    for T in (100, 1000):
        g = torch.Generator().manual_seed(T)
        hyp = torch.randint(3, VOCAB, (B, T), generator=g).cuda()
        gold = torch.randint(3, VOCAB, (B, T), generator=g).cuda()
        gold[:, T - T // 5:] = 0
        result[f"edit_counts_us_T{T}"] = round(1e3 * timed(lambda: b200asr.edit_counts(hyp, gold, table), 200, 20), 1)
    result["card_after"] = gpu_info()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
