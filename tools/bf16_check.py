#!/usr/bin/env python
"""GPU check of the bf16 GEMM modes (precision 2 = bf16, 6 = bf16x3) against float64: y = x w^T + b and dx = dy w for
shapes with M / N / K tails.  Prints max|err| / max|ref| per (shape, precision); 3xTF32 (3) and TF32 (1) for comparison."""
import importlib
import sys

import torch

sys.path.insert(0, ".")
import b200asr  # noqa: E402

ops = importlib.import_module(b200asr.__name__ + ".ops")
L = importlib.import_module(b200asr.__name__ + "._lib")
torch.manual_seed(0)
for (M, N, K) in [(128, 128, 32), (128, 128, 64), (300, 512, 512), (6400, 1536, 512), (130, 4364, 512), (257, 136, 2048), (3200, 512, 2048)]:
    x = torch.randn(M, K, device="cuda")
    w = torch.randn(N, K, device="cuda") * 0.1
    b = torch.randn(N, device="cuda")
    dy = torch.randn(M, N, device="cuda")
    y64 = (x.double() @ w.double().t() + b.double())
    dx64 = dy.double() @ w.double()
    line = f"M={M:5d} N={N:5d} K={K:5d} |"
    for prec in (1, 3, 2, 6):
        ws = ops.split_weight(w, prec)
        try:
            y = ops.linear_fwd(x, w, b, False, prec, ws)
            dx = ops.linear_bwd_data(dy, w, None, prec, ws)
            torch.cuda.synchronize()
            ey = float((y.double() - y64).abs().max() / y64.abs().max())
            ex = float((dx.double() - dx64).abs().max() / dx64.abs().max())
            line += f" p{prec}: fwd {ey:.1e} dgrad {ex:.1e} |"
        except RuntimeError as e:
            line += f" p{prec}: ERROR {str(e)[:80]} |"
    print(line, flush=True)
