#!/usr/bin/env python
"""Time of b200asr_spec_augment on a cfg2-shaped batch of features.

    python tools/spec_augment_time.py [--iters 200] [--warmup 20] [--out FILE]

Batch: B = 32 utterances of 4 to 16 s (seeded) as the front end leaves them at the reference's defaults: F = 161 bins,
T = 1601 frames (16 s at a 10 ms hop), frames past each utterance 0.  Policy: the paper's LD (W 80, two frequency masks of
up to 27 bins, two time masks of up to 100 frames, p 1.0).  Timed with CUDA events around `iters` calls after `warmup`
untimed ones of the raw entry point, each with its own batch counter.  Bytes: the output written once plus the input elements the kernel reads
(frames t < T_b outside every mask, two where the warp interpolates), counted on the host from the draws of the last
call; also printed against the full read + write of the [B,1,F,T] tensor.  The card, its power limit and max SM clock
are read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import b200asr  # noqa: E402
from tests import spec_augment_util as SA  # noqa: E402


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[torch.cuda.current_device()] if q.returncode == 0 else "nvidia-smi unavailable"


def read_bytes(drw, sizes, F, nf, nt):
    """Input bytes the kernel reads for one call with these draws."""
    total = 0
    for b, Tb in enumerate(sizes):
        keep_f = np.ones(F, bool)
        keep_t = np.zeros(Tb, bool) if Tb == 0 else np.ones(Tb, bool)
        for m in range(nf):
            keep_f[drw[b, 3 + 2 * m]:drw[b, 3 + 2 * m] + drw[b, 2 + 2 * m]] = False
        for m in range(nt):
            s = 2 + 2 * nf + 2 * m
            keep_t[drw[b, s + 1]:drw[b, s + 1] + drw[b, s]] = False
        c, w = int(drw[b, 0]), int(drw[b, 1])
        reads = [2 if SA.source_position(t, Tb, c, w) % 1 else 1 for t in range(Tb)]
        total += int(keep_f.sum()) * int(np.dot(keep_t, reads))
    return 4 * total


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--out", default=None, help="also write the JSON result here")
    a = ap.parse_args()
    b200asr._lib.load(check_device=True)
    g = np.random.default_rng(0)
    B, F, hop = 32, 161, 160
    sizes = sorted((1 + g.integers(4 * 16000, 16 * 16000 + 1, B) // hop).tolist(), reverse=True)
    T = 1601
    x = torch.randn(B, 1, F, T, device="cuda")
    for b, n in enumerate(sizes):
        x[b, :, :, n:] = 0
    frames = torch.tensor(sizes, dtype=torch.int32, device="cuda")
    L = b200asr._lib
    lib = L.load()
    out = torch.empty_like(x)
    drw = torch.empty(B, lib.b200asr_spec_augment_draws_ints(2, 2), dtype=torch.int32, device="cuda")
    st = torch.cuda.current_stream().cuda_stream

    def call(counter):      # the raw entry point: SpecAugment.apply's allocations would time the host, not the kernel
        L.check(lib.b200asr_spec_augment(L.ptr(x), L.ptr(out), L.ptr(drw), L.ptr(frames), B, F, T, 80, 27, 2, 100, 1.0, 2, 1,
                                         counter, st), "spec_augment")
    for k in range(a.warmup):
        call(k)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for k in range(a.iters):
        call(a.warmup + k)
    e1.record()
    torch.cuda.synchronize()
    us = e0.elapsed_time(e1) * 1e3 / a.iters
    tensor = x.numel() * 4
    moved = tensor + read_bytes(drw.cpu().numpy(), sizes, F, 2, 2)
    res = dict(what="spec_augment", B=B, F=F, T=T, frames=[min(sizes), max(sizes)], us_per_call=round(us, 2),
               bytes_moved=moved, GBps=round(moved / us / 1e3, 1), full_rw_bytes=2 * tensor,
               full_rw_GBps=round(2 * tensor / us / 1e3, 1), gpu=gpu_info())
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
