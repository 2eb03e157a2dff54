#!/usr/bin/env python
"""CUDA-event timing of the 3x3 convolutions of the VGG front end at the cfg2 shapes (B = 32), through the C ABI.
usage: conv_time.py [precision]    (B200ASR_LIB selects an A/B build of the library)

Per layer: the plain forward and unmasked data gradient, the calls the training step makes (the forward with the fused
2 x 2 max-pool on conv2 / conv4, the forward that also writes its ReLU bits on conv3, the data gradient with the ReLU mask of
the layer's input on conv2 / conv4 -- as fp32 activations (dgrad_mask) and as the packed bits the step uses (dgrad_bits)),
and the weight gradient; on conv2 / conv4 also the forward that writes the pooling codes with and without y (fwd_pool_codes,
fwd_pool_codes_noy) and the pooling backward from y and from the codes (pool_bwd, pool_bwd_codes).  The last line adds up the
calls of these kinds one step makes."""
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
    # relu_x > 0 packed as the forward writes it: bit c % 32 of int32 word c / 32 (disjoint bits: the wrapping sum is the OR)
    x_bits = ((relu_x > 0).view(B, T, F, Ci // 32, 32).int() << torch.arange(32, device="cuda", dtype=torch.int32)).sum(-1, dtype=torch.int32)
    y_bits = torch.empty(B, T, F, Co // 32, dtype=torch.int32, device="cuda")
    w = torch.randn(Co, Ci, 3, 3, device="cuda") * (9 * Ci) ** -0.5
    b = torch.randn(Co, device="cuda")
    y = torch.empty(B, T, F, Co, device="cuda")
    pool = torch.empty(B, T // 2, F // 2, Co, device="cuda")
    codes = torch.empty(B, T // 2, F // 2, Co // 8, dtype=torch.int32, device="cuda")
    dpool = torch.randn(B, T // 2, F // 2, Co, device="cuda")
    dy_pool = torch.empty(B, T, F, Co, device="cuda")
    dx = torch.empty(B, T, F, Ci, device="cuda")
    dw, db = torch.empty_like(w), torch.empty_like(b)
    ws = torch.empty(lib.b200asr_conv3x3_ws_bytes(Ci, Co) // 4, device="cuda")
    gf = 2 * 9 * B * T * F * Ci * Co / 1e9
    ops = {"fwd": lambda: lib.b200asr_conv3x3_fwd(L.ptr(x), L.ptr(w), L.ptr(b), L.ptr(y), L.ptr(ws), B, T, F, Ci, Co, 1, prec, st),
           "fwd_pool": lambda: lib.b200asr_conv3x3_fwd_pool(L.ptr(x), L.ptr(w), L.ptr(b), L.ptr(y), L.ptr(pool), None, L.ptr(ws),
                                                            B, T, F, Ci, Co, 1, prec, st),
           "fwd_bits": lambda: lib.b200asr_conv3x3_fwd_bits(L.ptr(x), L.ptr(w), L.ptr(b), L.ptr(y), L.ptr(ws), B, T, F, Ci, Co, 1, prec,
                                                            L.ptr(y_bits), st),
           "dgrad": lambda: lib.b200asr_conv3x3_bwd_data(L.ptr(y), L.ptr(w), None, L.ptr(dx), None, L.ptr(ws), B, T, F, Ci, Co, prec, st),
           "dgrad_mask": lambda: lib.b200asr_conv3x3_bwd_data(L.ptr(y), L.ptr(w), L.ptr(relu_x), L.ptr(dx), None, L.ptr(ws),
                                                              B, T, F, Ci, Co, prec, st),
           "dgrad_bits": lambda: lib.b200asr_conv3x3_bwd_data_bits(L.ptr(y), L.ptr(w), L.ptr(x_bits), L.ptr(dx), None, L.ptr(ws),
                                                                   B, T, F, Ci, Co, prec, st),
           **({"fwd_pool_codes": lambda: lib.b200asr_conv3x3_fwd_pool_codes(L.ptr(x), L.ptr(w), L.ptr(b), L.ptr(y), L.ptr(pool), L.ptr(codes),
                                                                        L.ptr(ws), B, T, F, Ci, Co, 1, prec, st),
               **({} if prec not in (2, 6) else {"fwd_pool_codes_noy": lambda: lib.b200asr_conv3x3_fwd_pool_codes(L.ptr(x), L.ptr(w), L.ptr(b), None, L.ptr(pool),
                                                                            L.ptr(codes), L.ptr(ws), B, T, F, Ci, Co, 1, prec, st)}),
               "pool_bwd": lambda: lib.b200asr_maxpool2x2_bwd(L.ptr(dpool), L.ptr(y), L.ptr(dy_pool), None, B, T, F, Co, 1, st),
               "pool_bwd_codes": lambda: lib.b200asr_maxpool2x2_bwd_codes(L.ptr(dpool), L.ptr(codes), L.ptr(dy_pool), None, B, T, F, Co,
                                                                          1, st)} if pooled else {}),
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
        fwd_pool = "fwd_pool_codes_noy" if prec in (2, 6) else "fwd_pool_codes"     # y = NULL needs the pooling epilogue
        if name in ((fwd_pool, "dgrad_bits", "pool_bwd_codes") if pooled else ("fwd_bits", "dgrad")):
            step_ms += ms
        out.append("%s %.3f ms %.0f TF/s" % (name, ms, gf / ms))
    print("T=%d F=%d %d->%d p%d | " % (T, F, Ci, Co, prec) + " | ".join(out), flush=True)
print("calls of one step (conv2 / conv4 fwd_pool_codes_noy + dgrad_bits + pool_bwd_codes, conv3 fwd_bits + dgrad): %.3f ms" % step_ms)
