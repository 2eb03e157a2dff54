"""Time one training window of the LSTM LM loop end to end -- zero_grad, forward, loss, backward, gradient clip, SGD update
-- as `python -m b200asr.lm_train` runs it (b200asr.RNNModel, ops.XentFn, b200asr.clip_grad_norm_, optim.sgd_step) and as
the word-language-model example runs it on the reference's RNNModel (cuDNN, nn.CrossEntropyLoss, torch's clip,
p.data.add_), fp32-strict (no TF32) and with torch's default flags; then the loss forward + backward and the SGD step
alone against torch's.  Shapes: ntoken 10 000, ninp = nhid, 2 layers, B = 20, bptt = 35, dropout 0, clip 0.25, lr 20;
the hidden state is carried (detached) from window to window.

    python tools/lm_fit_time.py [--iters 20] [--warmup 5] [--shapes 650,1500]

Prints the card and its power limit, then per shape the mean window time of each path (CUDA events), and for the loss and
the SGD step their call times (CUDA events around the calls, host work included), their device times (the durations of
their kernels, memsets and copies under torch.profiler, a separate pass), the bytes they must move and the rate over device
time.  Needs a GPU and the reference staged in oracle/_ref (oracle/make_ref.py).
"""
import argparse
import importlib
import json
import os
import subprocess
import sys

import torch
import torch.nn as nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import b200asr  # noqa: E402
from oracle import ref_shim  # noqa: E402

ops = importlib.import_module(b200asr.__name__ + ".ops")
optim = importlib.import_module(b200asr.__name__ + ".optim")
LT = b200asr.lm_train
NTOKEN, NLAYERS, B, BPTT, CLIP, LR = 10000, 2, 20, 35, 0.25, 20.0


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name()


def new_window(model, x, y, state):
    model.zero_grad()
    state[0] = LT.repackage_hidden(state[0])
    out, state[0] = model(x, state[0])
    loss = ops.XentFn.apply(out.view(-1, NTOKEN), y)
    loss.backward()
    b200asr.clip_grad_norm_(model.parameters(), CLIP)
    optim.sgd_step(model.parameters(), LR)


def example_window(model, x, y, state):
    model.zero_grad()
    state[0] = LT.repackage_hidden(state[0])
    out, state[0] = model(x, state[0])
    loss = nn.CrossEntropyLoss()(out.view(-1, NTOKEN), y)
    loss.backward()
    torch.nn.utils.clip_grad_norm_(model.parameters(), CLIP)
    for p in model.parameters():
        p.data.add_(p.grad, alpha=-LR)


def timed(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def kernel_ms(fn, iters, warmup):
    """Device time of fn's kernels, memsets and copies per call (torch.profiler, a separate pass)."""
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            fn()
        torch.cuda.synchronize()
    ns = sum(e.duration_ns() for e in prof.profiler.kineto_results.events()
             if e.device_type() == torch.autograd.DeviceType.CUDA)
    return ns / 1e6 / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--shapes", default="650,1500")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("lm_fit_time: no CUDA device (the timings are GPU timings; there is no CPU mode)")
    ref_shim.load([])
    lu = importlib.import_module("utils.lstm_utils")
    print(f"card: {card()}")
    results = []
    for nhid in (int(s) for s in a.shapes.split(",")):
        torch.manual_seed(0)
        mine = b200asr.RNNModel("LSTM", NTOKEN, nhid, nhid, NLAYERS, dropout=0.0).cuda()
        ref = lu.RNNModel("LSTM", NTOKEN, nhid, nhid, NLAYERS, dropout=0.0).cuda()
        ref.load_state_dict(mine.state_dict())
        g = torch.Generator().manual_seed(1)
        x = torch.randint(0, NTOKEN, (BPTT, B), generator=g).cuda()
        y = torch.randint(0, NTOKEN, (BPTT * B,), generator=g).cuda()
        row = dict(nhid=nhid)
        mine.train()
        st = [mine.init_hidden(B)]
        row["window_ms.installed"] = timed(lambda: new_window(mine, x, y, st), a.iters, a.warmup)
        for name, tf32 in (("cudnn_fp32", False), ("cudnn_default", None)):
            saved = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
            if tf32 is not None:
                torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = tf32
            ref.train()
            st = [ref.init_hidden(B)]
            row[f"window_ms.{name}"] = timed(lambda: example_window(ref, x, y, st), a.iters, a.warmup)
            torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = saved
        # the loss alone: forward + backward over the window's [bptt * B, ntoken] logits
        logits = torch.randn(BPTT * B, NTOKEN, generator=g).cuda().requires_grad_(True)
        loss_bytes = 3 * logits.numel() * 4                 # logits read by the forward and the backward, dlogits written

        def xent():
            logits.grad = None
            ops.XentFn.apply(logits, y).backward()

        def torch_xent():
            logits.grad = None
            nn.CrossEntropyLoss()(logits, y).backward()
        for name, fn in (("b200asr", xent), ("torch", torch_xent)):
            row[f"loss_fwd_bwd_ms.{name}"] = timed(fn, 10 * a.iters, a.warmup)
            ms = kernel_ms(fn, 10 * a.iters, a.warmup)
            row[f"loss_fwd_bwd_device_ms.{name}"] = ms
            row[f"loss_fwd_bwd_GBps.{name}"] = loss_bytes / ms / 1e6
        # the SGD step alone over the model's parameters (gradients from one window)
        new_window(mine, x, y, [mine.init_hidden(B)])
        params = list(mine.parameters())
        sgd_bytes = 3 * 4 * sum(p.numel() for p in params)   # param read and written, gradient read

        def torch_sgd():
            for p in params:
                p.data.add_(p.grad, alpha=-1e-6)
        for name, fn in (("b200asr", lambda: optim.sgd_step(params, 1e-6)), ("torch", torch_sgd)):
            row[f"sgd_ms.{name}"] = timed(fn, 10 * a.iters, a.warmup)
            ms = kernel_ms(fn, 10 * a.iters, a.warmup)
            row[f"sgd_device_ms.{name}"] = ms
            row[f"sgd_GBps.{name}"] = sgd_bytes / ms / 1e6
        row["loss_MB"], row["sgd_MB"] = loss_bytes / 1e6, sgd_bytes / 1e6
        row = {k: round(v, 4) if isinstance(v, float) else v for k, v in row.items()}
        results.append(row)
        print(json.dumps(row))
    return results


if __name__ == "__main__":
    main()
