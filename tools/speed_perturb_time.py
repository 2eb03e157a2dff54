#!/usr/bin/env python
"""Time of b200asr_resample_packed on a training-shaped batch, of the installed loader's per-batch device step with and
without speed perturbation, and of scipy.signal.resample_poly on one CPU core for comparison.

    python tools/speed_perturb_time.py [--iters 100] [--warmup 10] [--out FILE]

Batch: B = 32 utterances of 15 s at 16 kHz (seeded, on the 16-bit grid, as load_audio reads 16-bit files), factors drawn
by SpeedPerturb() from {0.9, 1.0, 1.1}.  The kernel alone: CUDA events around `iters` launches of the raw entry point
after `warmup` untimed ones.  `PackedLoader.batch` (uploads, the resampling when the batch carries it, the features): a
host clock around `iters` calls, each followed by a device synchronise, with and without the policy, alternating.  The
CPU comparison: resample_poly per utterance in float64 on one thread, once over the batch.  The timed kernel output is
checked against resample_poly within tests/resample_util.py's fp32 bound.  The card, its power limit and max SM clock are
read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys
import time
import types

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import b200asr  # noqa: E402
from b200asr import features as F  # noqa: E402
from b200asr import loader  # noqa: E402
from tests import resample_util as RU  # noqa: E402
from tests.tempo_gain_util import grid16  # noqa: E402


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[torch.cuda.current_device()] if q.returncode == 0 else "nvidia-smi unavailable"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--out", default=None, help="also write the JSON result here")
    a = ap.parse_args()
    b200asr._lib.load(check_device=True)
    sr, B, n = 16000, 32, 15 * 16000
    g = np.random.default_rng(0)
    xs = [grid16(0.3 * np.sin(2 * np.pi * (120 + 300 * g.random()) * np.arange(n) / sr) + 0.1 * g.standard_normal(n))
          for _ in range(B)]
    policy, rs = b200asr.SpeedPerturb(), np.random.RandomState(0)
    ratios = [policy.ratio(policy.draw_one(rs)) for _ in range(B)]
    out_lens = np.array([F.resample_out_length(n, u, d) for u, d in ratios], np.int64)
    in_off = np.arange(B, dtype=np.int64) * n
    wave = torch.from_numpy(np.concatenate(xs)).cuda()
    out = torch.empty(int(out_lens.sum()), device="cuda")
    out_off = np.concatenate([[0], np.cumsum(out_lens)[:-1]]).astype(np.int64)
    items = np.zeros(B, F._RESAMPLE_ITEM)
    for b, (u, d) in enumerate(ratios):
        items[b] = (in_off[b], out_off[b], 0 if u == d == 1 else F._device_taps(u, d, wave.device).data_ptr(), n, u, d, 0)
    items_d = torch.from_numpy(items.view(np.uint8).copy()).cuda()
    L = b200asr._lib
    lib = L.load()
    st = torch.cuda.current_stream().cuda_stream

    def call():             # the raw entry point: resample's uploads would time the host, not the kernel
        L.check(lib.b200asr_resample_packed(L.ptr(wave), wave.numel(), L.ptr(out), out.numel(), items.ctypes.data,
                                            L.ptr(items_d), B, 0, st), "resample_packed")
    for _ in range(a.warmup):
        call()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(a.iters):
        call()
    e1.record()
    torch.cuda.synchronize()
    us = e0.elapsed_time(e1) * 1e3 / a.iters
    o = out.cpu().numpy()

    import scipy.signal
    try:
        from threadpoolctl import threadpool_limits
        limit = threadpool_limits(1)
    except ImportError:
        limit = None
    t0 = time.perf_counter()
    ref = [scipy.signal.resample_poly(x.astype(np.float64), u, d) for x, (u, d) in zip(xs, ratios)]
    cpu_ms = (time.perf_counter() - t0) * 1e3
    del limit
    agree = all(bool((np.abs(o[out_off[b]:out_off[b] + out_lens[b]] - ref[b]) <= RU.fp32_bound(xs[b], *ratios[b]) + 1e-30).all())
                for b in range(B))

    # PackedLoader.batch on the same utterances; the dataset is a stand-in with the reference's defaults (no noise,
    # Hamming), so the reference checkout is not needed here
    loader._data_loader = lambda: None
    loader._window_name = lambda ds, DL: "hamming"
    ds = types.SimpleNamespace(sample_rate=sr, window_size=0.02, window_stride=0.01, normalize=True, noiseInjector=None)
    packed = loader.PackedLoader.__new__(loader.PackedLoader)
    packed.items, packed.bank = types.SimpleNamespace(dataset=ds), None
    pin = lambda t: t.pin_memory()  # noqa: E731

    def packed_batch(speed):
        m = out_lens if speed else np.full(B, n)
        order = sorted(range(B), key=lambda i: m[i], reverse=True)
        frames = [1 + int(m[i]) // 160 for i in order]
        kw = {}
        if speed:
            kw = dict(up=torch.tensor([ratios[i][0] for i in order], dtype=torch.int32),
                      down=torch.tensor([ratios[i][1] for i in order], dtype=torch.int32),
                      speed_lengths=torch.tensor(out_lens[order], dtype=torch.int32))
        return loader.PackedBatch(
            wave=pin(torch.from_numpy(np.concatenate([xs[i] for i in order]))),
            offsets=pin(torch.from_numpy(in_off.copy())), lengths=pin(torch.full((B,), n, dtype=torch.int32)),
            noise_clip=torch.full((B,), -1), noise_start=pin(torch.full((B,), -1)),
            noise_level=pin(torch.full((B,), float("nan"))), targets=torch.zeros(B, 1, dtype=torch.int64),
            input_percentages=torch.tensor([f / frames[0] for f in frames]), input_sizes=torch.tensor(frames, dtype=torch.int32),
            target_sizes=torch.ones(B, dtype=torch.int32), src_max_len=10 ** 9, **kw)
    batches = {True: packed_batch(True), False: packed_batch(False)}
    for s in (True, False):
        for _ in range(a.warmup):
            packed.batch(batches[s])
    torch.cuda.synchronize()
    ms = {True: [], False: []}
    for _ in range(a.iters):
        for s in (True, False):
            t0 = time.perf_counter()
            packed.batch(batches[s])
            torch.cuda.synchronize()
            ms[s].append((time.perf_counter() - t0) * 1e3)
    med = {s: float(np.median(v)) for s, v in ms.items()}
    res = dict(what="resample_packed", B=B, seconds=n / sr, ratios=sorted(set(ratios)), outputs=int(out_lens.sum()),
               kernel_us=round(us, 1), batch_ms_with=round(med[True], 3), batch_ms_without=round(med[False], 3),
               cpu_resample_poly_ms=round(cpu_ms, 1), matches_resample_poly=agree, gpu=gpu_info())
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")
    if not agree:
        sys.exit("the timed output is outside the fp32 bound of resample_poly")


if __name__ == "__main__":
    main()
