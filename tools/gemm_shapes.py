#!/usr/bin/env python
"""Per-shape timing of the three linear kernels (fwd, dgrad, wgrad) at the cfg2 shapes, through the C ABI.

  python tools/gemm_shapes.py [prec]        # prec: 0 fp32, 1 tf32, 3 3xTF32 (default)

Prints us per call, fp32-equivalent TFLOP/s (2MNK / t) and, for 3xTF32, the fraction of the tensor-pipe roofline
(3 tf32 MMAs per product; peak = MEASURED_PEAKS bf16 dense / 2 if present, else 1100 TF/s).
"""
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import b200asr  # noqa: E402
from b200asr import ops  # noqa: E402

SHAPES = [  # (name, M, N, K)
    ("enc qkv/o", 6400, 512, 512), ("enc ffn1", 6400, 2048, 512), ("enc ffn2", 6400, 512, 2048),
    ("dec qkv/o", 3200, 512, 512), ("dec ffn1", 3200, 2048, 512), ("dec ffn2", 3200, 512, 2048),
    ("enc in", 6400, 512, 5248), ("dec out", 3200, 4000, 512), ("fused qkv", 6400, 1536, 512),
]


def timeit(fn, iters=20):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters * 1e3


def overheads(prec):
    """fixed cost vs per-k-block cost of the persistent engine: one (or two) 128x128 tiles per SM, K swept"""
    dev = torch.device("cuda:0")
    for N in (128, 256):
        for K in (32, 256, 512, 2048, 8192):
            M = 128 * 132
            x = torch.randn(M, K, device=dev)
            w = torch.randn(N, K, device=dev) * 0.05
            b = torch.randn(N, device=dev)
            ws = ops.split_weight(w, prec)
            t = timeit(lambda: ops.linear_fwd(x, w, b, False, prec, ws))
            print("tiles/SM %d  K=%5d (%3d k-blocks)  fwd %7.1f us  -> %6.1f ns per k-block per tile" % (N // 128, K, K // 32, t, t * 1e3 / (K // 32) / (N // 128)))


def main():
    prec = int(sys.argv[1]) if len(sys.argv) > 1 else 3
    if "--overheads" in sys.argv:
        return overheads(prec)
    peak = 1100.0
    try:
        peak = json.load(open(os.path.join(os.path.dirname(__file__), "..", "MEASURED_PEAKS.json")))["bf16_tflops"] / 2   # burst figure: each kernel is timed alone
    except Exception:
        pass
    dev = torch.device("cuda:0")
    print("prec", prec, "tf32 peak", peak)
    for name, M, N, K in SHAPES:
        x = torch.randn(M, K, device=dev)
        w = torch.randn(N, K, device=dev) * 0.05
        b = torch.randn(N, device=dev)
        dy = torch.randn(M, N, device=dev)
        dw = torch.zeros(N, K, device=dev)
        db = torch.zeros(N, device=dev)
        ws = ops.split_weight(w, prec)
        t_f = timeit(lambda: ops.linear_fwd(x, w, b, False, prec, ws))
        t_d = timeit(lambda: ops.linear_bwd_data(dy, w, None, prec, ws))
        t_w = timeit(lambda: ops.linear_bwd_weight(dy, x, True, prec, dw, db))
        fl = 2.0 * M * N * K
        mult = 3 if prec == 3 else 1
        print("%-10s M=%5d N=%5d K=%5d | fwd %7.1f us %6.1f TF (%.2f) | dgrad %7.1f us %6.1f TF (%.2f) | wgrad %7.1f us %6.1f TF (%.2f)" % (
            name, M, N, K, t_f, fl / t_f / 1e6, mult * fl / t_f / 1e6 / peak, t_d, fl / t_d / 1e6, mult * fl / t_d / 1e6 / peak,
            t_w, fl / t_w / 1e6, mult * fl / t_w / 1e6 / peak))


if __name__ == "__main__":
    main()
