#!/usr/bin/env python
"""Time of one optimizer step over the cfg2 parameter list (182 fp32 tensors, 36.8 M elements): torch.optim.Adam(foreach=True)
against the device step (optim.adam_step), each without and with the gradient clip (torch.nn.utils.clip_grad_norm_ /
optim.clip_grad_norm_) in front of it, as the reference's Trainer.train runs them with --clip.

    python tools/optim_time.py [--steps 200] [--reps 5]

Each arm has its own parameters, gradients and Adam state.  The four arms run alternately in one process, `reps` rounds of
`steps` steps each after a warm-up round; a round's time is CUDA events around its steps (the host enqueues every step, so the
events also catch a host-bound step), the figure is the median over rounds.  The byte floor counts one pass that reads p, g, m,
v and writes p, m, v (28 bytes per element; the clip adds a read of g and a read + write of g, 12 more) at 3.35 TB/s.  The
card, its power limit and max SM clock are read in the same run.
"""
import argparse
import importlib
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import b200asr  # noqa: E402
from tools.features_time import gpu_info  # noqa: E402

OP = importlib.import_module(b200asr.__name__ + ".optim")


def make_arm(shapes, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    ps = [torch.nn.Parameter(torch.randn(s, device="cuda", generator=g) * 0.05) for s in shapes]
    for p in ps:
        p.grad = torch.randn(p.shape, device="cuda", generator=g) * 1e-3
    return ps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    b200asr._lib.load(check_device=True)
    shapes = [tuple(p.shape) for p in b200asr.build_model(b200asr.BASELINE_CONFIGS["cfg2"]["cfg"]).parameters()]
    n = sum(torch.Size(s).numel() for s in shapes)
    max_norm = 1e-3                                   # below the gradients' norm: the clip scales every step

    arms = {}
    for name in ("torch", "torch+clip", "device", "device+clip"):
        ps = make_arm(shapes, 0)
        opt = torch.optim.Adam(ps, lr=1e-4, betas=(0.9, 0.98), eps=1e-9, foreach=True)
        if name.startswith("torch"):
            step = opt.step
            clip = (lambda ps=ps: torch.nn.utils.clip_grad_norm_(ps, max_norm)) if "clip" in name else None
        else:
            step = (lambda opt=opt: OP.adam_step(opt))
            clip = (lambda ps=ps: OP.clip_grad_norm_(ps, max_norm)) if "clip" in name else None

        def one(step=step, clip=clip):
            if clip is not None:
                clip()
            step()
        arms[name] = one

    times = {k: [] for k in arms}
    for rep in range(a.reps + 1):
        for name, fn in arms.items():
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.steps):
                fn()
            e1.record()
            torch.cuda.synchronize()
            if rep:                                   # round 0 warms up (state creation, scratch, module loading)
                times[name].append(e0.elapsed_time(e1) / a.steps)
    floor = {"": 28 * n / 3.35e12 * 1e3, "+clip": 40 * n / 3.35e12 * 1e3}
    res = {"gpu": gpu_info(), "tensors": len(shapes), "elements": n, "steps_per_round": a.steps, "rounds": a.reps}
    for name, ts in times.items():
        res[name + "_ms"] = round(statistics.median(ts), 4)
        res[name + "_spread_ms"] = [round(min(ts), 4), round(max(ts), 4)]
    res["byte_floor_ms"] = round(floor[""], 4)
    res["byte_floor_clip_ms"] = round(floor["+clip"], 4)
    res["speedup"] = round(res["torch_ms"] / res["device_ms"], 2)
    res["speedup_clip"] = round(res["torch+clip_ms"] / res["device+clip_ms"], 2)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
