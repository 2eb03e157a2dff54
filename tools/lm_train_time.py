"""Time one BPTT window of LSTM LM training -- forward, torch's cross-entropy, backward -- on the installed kernels
(b200asr.RNNModel, whose forward is modules.rnn_model_forward) and on the reference's RNNModel (cuDNN), fp32-strict
(no TF32) and with torch's default flags, at the word-language-model "medium" (650) and "large" (1500) shapes:
ntoken 10 000, ninp = nhid, 2 layers, B = 20, bptt = 35, dropout 0.

    python tools/lm_train_time.py [--iters 20] [--warmup 5] [--shapes 650,1500]

Prints the card and its power limit, per path the mean window time (CUDA events), the installed path's split by C-ABI
entry point group (ops.profiler, a separate pass) and torch's loss, and each path's max error against float64 on one
window (max-norm, relative to the largest reference entry, over the logits and every parameter gradient).  Needs a GPU
and the reference staged in oracle/_ref (oracle/make_ref.py).
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
NTOKEN, NLAYERS, B, BPTT = 10000, 2, 20, 35
GROUPS = {"recurrence fwd": ("lstm_layer_train_fwd",), "recurrence bwd": ("lstm_layer_train_bwd",),
          "GEMMs": ("linear_fwd", "linear_bwd_data", "linear_bwd_weight"), "operand preparation": ("lstm_prepare", "split_bf16")}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name()


def window(model, x, y, hidden):
    model.zero_grad(set_to_none=True)
    out, _ = model(x, hidden)
    loss = nn.functional.cross_entropy(out.view(-1, NTOKEN), y)
    loss.backward()
    return out, loss


def time_path(model, x, y, hidden, iters, warmup):
    for _ in range(warmup):
        window(model, x, y, hidden)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(iters):
        window(model, x, y, hidden)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def float64_window(sd, x, y, hidden):
    """logits and parameter gradients of one window in float64 on the CPU (eager torch, dropout 0)."""
    P = {k: v.detach().double().cpu().requires_grad_(True) for k, v in sd.items() if not k.startswith("rnn.")}
    nhid = sd["rnn.weight_hh_l0"].shape[1]
    lstm = nn.LSTM(P["encoder.weight"].shape[1], nhid, NLAYERS).double()
    lstm.load_state_dict({k[4:]: v.double().cpu() for k, v in sd.items() if k.startswith("rnn.")})
    emb = P["encoder.weight"][x.cpu()]
    out, _ = lstm(emb, tuple(h.double().cpu() for h in hidden))
    logits = out @ P["decoder.weight"].t() + P["decoder.bias"]
    nn.functional.cross_entropy(logits.view(-1, NTOKEN), y.cpu()).backward()
    grads = {k: v.grad for k, v in P.items()}
    grads.update({"rnn." + k: v.grad for k, v in lstm.named_parameters()})
    return logits.detach(), grads


def max_err(logits, model, ref_logits, ref_grads):
    rel = lambda a, b: float((a.detach().double().cpu() - b).abs().max() / b.abs().max())
    e = rel(logits, ref_logits)
    for k, p in model.named_parameters():
        e = max(e, rel(p.grad, ref_grads[k]))
    return e


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--shapes", default="650,1500")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("lm_train_time: no CUDA device (the timings are GPU timings; there is no CPU mode)")
    ref_shim.load([])
    lu = importlib.import_module("utils.lstm_utils")
    print(f"card: {card()}")
    results = []
    for nhid in (int(s) for s in a.shapes.split(",")):
        torch.manual_seed(0)
        mine = b200asr.RNNModel("LSTM", NTOKEN, nhid, nhid, NLAYERS, dropout=0.0).cuda().train()
        ref = lu.RNNModel("LSTM", NTOKEN, nhid, nhid, NLAYERS, dropout=0.0).cuda().train()
        ref.load_state_dict(mine.state_dict())
        g = torch.Generator().manual_seed(1)
        x = torch.randint(0, NTOKEN, (BPTT, B), generator=g).cuda()
        y = torch.randint(0, NTOKEN, (BPTT * B,), generator=g).cuda()
        hidden = tuple(0.1 * torch.randn(NLAYERS, B, nhid, generator=g).cuda() for _ in range(2))
        ref_logits, ref_grads = float64_window(mine.state_dict(), x, y, hidden)
        row = dict(nhid=nhid)
        out, _ = window(mine, x, y, hidden)
        row["installed_err"] = max_err(out, mine, ref_logits, ref_grads)
        row["installed_ms"] = time_path(mine, x, y, hidden, a.iters, a.warmup)
        for name, tf32 in (("cudnn_fp32", False), ("cudnn_default", None)):
            saved = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
            if tf32 is not None:
                torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = tf32
            out, _ = window(ref, x, y, hidden)
            row[name + "_err"] = max_err(out, ref, ref_logits, ref_grads)
            row[name + "_ms"] = time_path(ref, x, y, hidden, a.iters, a.warmup)
            torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = saved
        # split of the installed window by entry point group (events around every C-ABI call), and torch's loss alone
        ops.profiler.start()
        window(mine, x, y, hidden)
        ops.profiler.stop()
        rep = ops.profiler.report()
        split = {grp: sum(ms for nm in names for _, ms in rep.get(nm, [])) for grp, names in GROUPS.items()}
        split["other entry points"] = sum(ms for nm, lst in rep.items() if not any(nm in v for v in GROUPS.values()) for _, ms in lst)
        logits = out.detach().view(-1, NTOKEN).clone().requires_grad_(True)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        for i in range(a.warmup + a.iters):
            if i == a.warmup:
                e0.record()
            nn.functional.cross_entropy(logits, y).backward()
        e1.record()
        torch.cuda.synchronize()
        split["torch loss fwd+bwd"] = e0.elapsed_time(e1) / a.iters
        row["installed_split_ms"] = {k: round(v, 4) for k, v in split.items()}
        results.append(row)
        print(json.dumps(row))
    return results


if __name__ == "__main__":
    main()
