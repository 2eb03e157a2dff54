#!/usr/bin/env python
"""One training step (zero_grad + fwd + CE + bwd + Adam) at every BASELINE.json configuration's per-GPU shape: checks that each
shape is supported end to end (finite loss, no shape/alignment rejection) and prints one JSON line per configuration
(CUDA-event timed, 10 warm-up + 20 timed steps).  Usage:
    python tools/run_configs.py [cfg1 cfg2 ...] [--batch N] [--mode default|bf16|tf32x3|fp32]
Modes: default = package default (bf16x3 linear/conv fwd+dgrad, tf32x3 conv wgrad + attention); bf16 = BASELINE cfg5's
"bf16" (one bf16 MMA per product everywhere, TF32 flash attention); tf32x3 = 3xTF32 everywhere; fp32 = CUDA cores."""
import importlib
import json
import sys

import torch

sys.path.insert(0, ".")
import b200asr  # noqa: E402

ops = importlib.import_module(b200asr.__name__ + ".ops")
names = [a for a in sys.argv[1:] if a.startswith("cfg")] or list(b200asr.BASELINE_CONFIGS)
batch_override = int(sys.argv[sys.argv.index("--batch") + 1]) if "--batch" in sys.argv else 0
mode = sys.argv[sys.argv.index("--mode") + 1] if "--mode" in sys.argv else "default"
MODES = {"default": {}, "bf16": dict(linear="bf16", conv="bf16", conv_wgrad="bf16", attn="tf32", attn_bwd="tf32"),
         "tf32x3": dict(linear="tf32x3", conv="tf32x3", conv_wgrad="tf32x3", attn="tf32x3"),
         "fp32": dict(linear="fp32", conv="fp32", conv_wgrad="fp32", attn="fp32", attn_bwd="fp32")}
ops.config.set(**MODES[mode])
dev = torch.device("cuda")
for name in names:
    spec = b200asr.BASELINE_CONFIGS[name]
    cfg, B, T = spec["cfg"], batch_override or spec["batch"], spec["t_src"]
    torch.manual_seed(0)
    model = b200asr.build_model(cfg).to(dev).train()
    dp = b200asr.DataParallelStep(model, model_size=cfg.dim_input, smoothing=cfg.label_smoothing)
    src = torch.randn(B, 1, cfg.freq, T, device=dev)
    lens = torch.full((B,), T, dtype=torch.int32)
    tgt = torch.randint(3, cfg.vocab, (B, cfg.tgt_max_len - 1), device=dev)
    try:
        for _ in range(10):                      # long enough for the SM clocks to ramp up from idle in a fresh process
            dp.step(src, lens, tgt)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(20):
            dp.step(src, lens, tgt)
        e1.record()
        torch.cuda.synchronize()
        loss = float(dp.global_loss())
        ms = e0.elapsed_time(e1) / 20
        print(json.dumps({"config": name, "mode": mode, "per_gpu_batch": B, "t_src": T, "t_enc": cfg.t_enc(T), "t_tgt": cfg.tgt_max_len,
                          "layers": cfg.num_layers, "d_model": cfg.dim_model, "feat": cfg.feat_extractor or "none",
                          "params_M": round(sum(p.numel() for p in model.parameters()) / 1e6, 1), "ms_per_step": round(ms, 2),
                          "utt_per_s": round(B / ms * 1e3, 1), "loss": round(loss, 4),
                          "peak_mem_GiB": round(torch.cuda.max_memory_allocated() / 2 ** 30, 1), "dropout": cfg.dropout,
                          "step": "zero_grad+fwd+CE+bwd+adam, 20 timed steps after 10 warm-up, CUDA events"}), flush=True)
        assert loss == loss and abs(loss) < 1e4
    except Exception as e:  # noqa: BLE001
        print(json.dumps({"config": name, "mode": mode, "error": f"{type(e).__name__}: {str(e)[:300]}"}), flush=True)
    del model, dp
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
