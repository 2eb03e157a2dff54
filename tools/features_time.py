#!/usr/bin/env python
"""Time of the device feature front end on a cfg2-shaped batch: `collate_waves` (host packing, upload, features, host
tensors) and its b200asr_stft_features_ex call alone, without and with noise, for every window.

    python tools/features_time.py [--iters 30] [--warmup 5]

Batch: B = 32 utterances of 4 to 16 s at 16 kHz (seeded), n_fft 320, hop 160 (the reference's defaults), src_max_len 4000
(not binding), 3xTF32.  Noise: noise_prob 1 from a bank of four 20 s clips.  Each leg is timed with CUDA events around
`iters` calls after `warmup` untimed ones.  The kernel leg's bytes are what the kernels must move: the waveform read
(+ its second read and the noise segment read for the energies), the padded signal written and read by the GEMM, the
spectrum written and read, the output written, and read and written again by the normalisation.  Also printed: the card,
its power limit and max SM clock, read in the same run.
"""
import argparse
import importlib
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import b200asr  # noqa: E402

F = importlib.import_module(b200asr.__name__ + ".features")


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[torch.cuda.current_device()] if q.returncode == 0 else "nvidia-smi unavailable"


def timed(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def kernel_bytes(lens, noisy, n_fft=320, hop=160):
    B, Lmax = len(lens), max(lens)
    Lp = -(-(Lmax + n_fft) // hop) * hop
    npad = (2 * (n_fft // 2 + 1) + 3) & ~3
    rows = B * Lp // hop
    t_max = 1 + Lmax // hop
    out = B * (n_fft // 2 + 1) * t_max * 4
    wave = sum(lens) * 4
    return {"wave_read": wave, "energy_read": 2 * wave if noisy else 0, "padded_write_read": 2 * (B * Lp + n_fft) * 4,
            "spec_write_read": 2 * rows * npad * 4, "out_write_norm_rw": 3 * out}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    b200asr._lib.load(check_device=True)
    g = np.random.default_rng(0)
    lens = g.integers(4 * 16000, 16 * 16000 + 1, 32).tolist()
    batch = [((0.1 * g.standard_normal(n)).astype(np.float32), g.integers(3, 40, 20).tolist()) for n in lens]
    bank = b200asr.NoiseBank([(0.05 * g.standard_normal(20 * 16000)).astype(np.float32) for _ in range(4)], 16000)
    dev = torch.device("cuda", torch.cuda.current_device())
    order = sorted(range(32), key=lambda i: lens[i], reverse=True)
    host = np.zeros((32, max(lens)), np.float32)
    for r, i in enumerate(order):
        host[r, :lens[i]] = batch[i][0]
    wave = torch.from_numpy(host).to(dev)
    lens_dev = torch.tensor([lens[i] for i in order], dtype=torch.int32, device=dev)
    t_max = 1 + max(lens) // 160
    print("card:", gpu_info())
    rows = []
    for window in F.WINDOWS:
        for noisy in (False, True):
            conf = dict(sample_rate=16000, window_size=0.02, window_stride=0.01, window=window,
                        noise_dir="noise" if noisy else None, noise_prob=1.0, noise_levels=(0.0, 0.5))
            rng = np.random.RandomState(1)
            t_collate = timed(lambda: b200asr.collate_waves(batch, conf, 4000, bank, rng=rng, precision=3), args.iters, args.warmup)
            draws = bank.draw([lens[i] for i in order], 1.0, (0.0, 0.5), np.random.RandomState(2)) if noisy else None
            dn = bank._device_args(draws, [lens[i] for i in order], dev) if noisy else None
            t_kernels = timed(lambda: F._features(wave, lens_dev, t_max, 320, 160, True, True, 3, window, False, dn, 4000),
                              args.iters, args.warmup)
            nbytes = kernel_bytes(lens, noisy)
            total = sum(nbytes.values())
            row = {"window": window, "noise": noisy, "collate_ms": round(t_collate, 3), "kernels_ms": round(t_kernels, 3),
                   "kernel_bytes": nbytes, "kernel_GBps": round(total / t_kernels / 1e6, 1)}
            rows.append(row)
            print(json.dumps(row))
    print("card:", gpu_info())


if __name__ == "__main__":
    main()
