#!/usr/bin/env python
"""CUDA-event timing of the 3x3 convolutions of the VGG front end at the cfg2 shapes (B = 32), through the C ABI.
usage: conv_time.py [precision]    (B200ASR_LIB selects an A/B build of the library)

Per layer: the plain forward and unmasked data gradient, the calls the training step makes (the forward with the fused
2 x 2 max-pool on conv2 / conv4, the data gradient with the ReLU mask of the layer's input on conv2 / conv4), and the
weight gradient.  The last line adds up the halo-kernel calls one step makes."""
import sys

import torch

sys.path.insert(0, ".")
import b200asr  # noqa: E402

L = b200asr._lib
lib = L.load(check_device=True)
prec = int(sys.argv[1]) if len(sys.argv) > 1 else 6
st = torch.cuda.current_stream().cuda_stream
B = 32
step_ms = 0.0
# (T, F, Cin, Cout, the step pools the output and masks the data gradient)
for (T, F, Ci, Co, pooled) in [(800, 161, 64, 64, True), (400, 80, 64, 128, False), (400, 80, 128, 128, True)]:
    x = torch.randn(B, T, F, Ci, device="cuda")
    relu_x = torch.relu(x)
    w = torch.randn(Co, Ci, 3, 3, device="cuda") * (9 * Ci) ** -0.5
    b = torch.randn(Co, device="cuda")
    y = torch.empty(B, T, F, Co, device="cuda")
    pool = torch.empty(B, T // 2, F // 2, Co, device="cuda")
    dx = torch.empty(B, T, F, Ci, device="cuda")
    dw, db = torch.empty_like(w), torch.empty_like(b)
    ws = torch.empty(lib.b200asr_conv3x3_ws_bytes(Ci, Co) // 4, device="cuda")
    gf = 2 * 9 * B * T * F * Ci * Co / 1e9
    ops = {"fwd": lambda: lib.b200asr_conv3x3_fwd(L.ptr(x), L.ptr(w), L.ptr(b), L.ptr(y), L.ptr(ws), B, T, F, Ci, Co, 1, prec, st),
           "fwd_pool": lambda: lib.b200asr_conv3x3_fwd_pool(L.ptr(x), L.ptr(w), L.ptr(b), L.ptr(y), L.ptr(pool), None, L.ptr(ws),
                                                            B, T, F, Ci, Co, 1, prec, st),
           "dgrad": lambda: lib.b200asr_conv3x3_bwd_data(L.ptr(y), L.ptr(w), None, L.ptr(dx), None, L.ptr(ws), B, T, F, Ci, Co, prec, st),
           "dgrad_mask": lambda: lib.b200asr_conv3x3_bwd_data(L.ptr(y), L.ptr(w), L.ptr(relu_x), L.ptr(dx), None, L.ptr(ws),
                                                              B, T, F, Ci, Co, prec, st),
           "wgrad": lambda: lib.b200asr_conv3x3_bwd_weight(L.ptr(y), None, L.ptr(x), L.ptr(dw), L.ptr(db), L.ptr(ws), B, T, F, Ci, Co, 3, st)}
    out = []
    for name, f in ops.items():
        for _ in range(3):
            rc = f()
        assert rc == 0, (name, L.last_error())
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(10):
            f()
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / 10
        if name == ("fwd_pool" if pooled else "fwd") or name == ("dgrad_mask" if pooled else "dgrad"):
            step_ms += ms
        out.append("%s %.3f ms %.0f TF/s" % (name, ms, gf / ms))
    print("T=%d F=%d %d->%d p%d | " % (T, F, Ci, Co, prec) + " | ".join(out), flush=True)
print("halo calls of one step (conv2 fwd_pool + dgrad_mask, conv3 fwd + dgrad, conv4 fwd_pool + dgrad_mask): %.3f ms" % step_ms)
