#!/usr/bin/env python
"""Cost of b200asr.attention_maps: the eval-mode encoder + decoder forward at cfg2 shapes with the switch off and on, per
attention mode, and b200asr_sdpa_probs alone.

    python tools/attn_maps_time.py [--iters 20] [--warmup 5] [--out FILE]

Model: cfg2 (4 + 4 layers, 8 heads, d_model 512, dk = dv = 64), batch 32, encoder T_e = 200 frames (ragged lengths), decoder
T_d = 40 target positions.  Each (mode, switch) leg runs `warmup` untimed forwards, then `iters` timed ones between CUDA
events; the two switch states alternate over three rounds and the median round is reported.  The kernel alone runs at the
encoder self-attention shape (B = 32, H = 8, Tq = Tk = 200, dk = 64) for each precision it serves, timed with CUDA events
over `iters` launches; its traffic is the map it writes (B*H*Tq*Tk floats) plus Q, K, the key-pad bytes and the LSE it
reads, and GB/s is that over the kernel time.  The card, its power limit and max SM clock are read in the same run.
"""
import argparse
import importlib
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import b200asr  # noqa: E402

ops = importlib.import_module(b200asr.__name__ + ".ops")
L = b200asr._lib


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[torch.cuda.current_device()] if q.returncode == 0 else "nvidia-smi unavailable"


def timed(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def model_forward_ms(mode, iters, warmup):
    cfg = b200asr.ASRConfig(tgt_max_len=40)
    torch.manual_seed(0)
    model = b200asr.build_model(cfg).cuda().eval()
    B, Te, Td = 32, 200, 39
    g = torch.Generator().manual_seed(1)
    feats = torch.randn(B, Te, model.encoder.dim_input, generator=g).cuda()
    lens = torch.randint(Te // 2, Te + 1, (B,), generator=g, dtype=torch.int32)
    lens[0] = Te
    lens = lens.cuda()
    tgt = torch.randint(3, cfg.vocab, (B, Td), generator=g).cuda()
    saved = ops.config.attn
    if mode != "default":
        ops.config.attn = ops._PREC_NAMES[mode]

    def step():
        with torch.no_grad():
            enc, _ = model.encoder(feats, lens)
            model.decoder(tgt, enc, lens)
    try:
        rounds = []
        for _ in range(3):
            r = {}
            for on in (False, True):
                with b200asr.attention_maps(on):
                    r[on] = timed(step, iters, warmup)
            rounds.append(r)
    finally:
        ops.config.attn = saved
    off = sorted(r[False] for r in rounds)[1]
    on = sorted(r[True] for r in rounds)[1]
    return off, on


def kernel_ms(prec, iters, warmup):
    B, H, T, d = 32, 8, 200, 64
    g = torch.Generator(device="cuda").manual_seed(2)
    q = torch.randn(B, T, H, d, device="cuda", generator=g).permute(0, 2, 1, 3)
    k = torch.randn(B, T, H, d, device="cuda", generator=g).permute(0, 2, 1, 3)
    v = torch.randn(B, T, H, d, device="cuda", generator=g).permute(0, 2, 1, 3)
    lens = torch.randint(T // 2, T + 1, (B,), device="cuda")
    key_pad = (torch.arange(T, device="cuda")[None] >= lens[:, None]).to(torch.uint8)
    out = torch.empty(B, T, H, d, device="cuda").permute(0, 2, 1, 3)
    lse = torch.empty(B, H, T, device="cuda")
    lib, st = L.load(), torch.cuda.current_stream().cuda_stream
    args = [L.ptr(q), L.ptr(k), L.ptr(v), *q.stride()[:3], *k.stride()[:3], *v.stride()[:3], L.ptr(key_pad), None, 0,
            L.ptr(out), *out.stride()[:3], L.ptr(lse)]
    if prec == L.PREC_BF16X3:
        ws = torch.empty(lib.b200asr_sdpa_fused_ws_bytes(B, H, T, T), device="cuda", dtype=torch.uint8)
        L.check(lib.b200asr_sdpa_fused_fwd(*args, L.ptr(ws), B, H, T, T, d, d, 0.125, 0.0, 0, 0, st), "fused_fwd")
    else:
        L.check(lib.b200asr_sdpa_fwd(*args, B, H, T, T, d, d, 0.125, 0.0, 0, 0, prec, st), "sdpa_fwd")
    shape, strides = ops.maps_layout(B, H, T, T)
    P = torch.empty(shape, device="cuda")

    def call():
        L.check(lib.b200asr_sdpa_probs(L.ptr(q), L.ptr(k), *q.stride()[:3], *k.stride()[:3], L.ptr(key_pad), None, 0, L.ptr(lse),
                                       L.ptr(P), *strides, B, H, T, T, d, 0.125, 0.0, 0, 0, prec, st), "sdpa_probs")
    ms = timed(call, iters * 5, warmup)
    nbytes = 4 * B * H * T * T + 2 * 4 * B * H * T * d + B * T + 4 * B * H * T
    return ms, nbytes / (ms * 1e-3) / 1e9


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    L.load(check_device=True)
    res = {"gpu": gpu_info(), "forward_ms": {}, "probs_kernel": {}}
    for mode in ("default", "bf16x3", "tf32", "fp32"):
        off, on = model_forward_ms(mode, a.iters, a.warmup)
        res["forward_ms"][mode] = {"maps_off": round(off, 3), "maps_on": round(on, 3), "extra_pct": round(100 * (on / off - 1), 1)}
        print(mode, res["forward_ms"][mode], flush=True)
    for name, prec in (("fp32", L.PREC_FP32), ("tf32", L.PREC_TF32), ("bf16x3", L.PREC_BF16X3)):
        ms, gbs = kernel_ms(prec, a.iters, a.warmup)
        res["probs_kernel"][name] = {"us": round(1e3 * ms, 1), "GB_per_s": round(gbs, 1)}
        print(name, res["probs_kernel"][name], flush=True)
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
