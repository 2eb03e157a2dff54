#!/usr/bin/env python
"""Time of b200asr_tempo_gain on a training-shaped batch, and of the installed loader's per-batch device step with and
without it.

    python tools/tempo_gain_time.py [--iters 100] [--warmup 10] [--out FILE]

Batch: B = 32 utterances of 4 to 16 s at 16 kHz (seeded, on the 16-bit grid, as load_audio reads 16-bit files), tempos
and gains drawn by TempoGain() from the reference's ranges ([0.85, 1.15], [-6, 8] dB).  The kernel alone: CUDA events
around `iters` calls of the raw entry point after `warmup` untimed ones.  `PackedLoader.batch` (uploads, the stretch when
the batch carries one, the features): a host clock around `iters` calls, each followed by a device synchronise, with and
without the stretch, alternating.  The output of the timed kernel call is compared with tests/tempo_gain_util.py's
restatement, bit for bit, picks included.  The card, its power limit and max SM clock are read in the same run.
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
from b200asr import loader  # noqa: E402
from tests import tempo_gain_util as TG  # noqa: E402


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
    sr, B = 16000, 32
    g = np.random.default_rng(0)
    lens = g.integers(4 * sr, 16 * sr + 1, B)
    xs = [TG.grid16(0.3 * np.sin(2 * np.pi * (120 + 300 * g.random()) * np.arange(n) / sr) + 0.1 * g.standard_normal(n))
          for n in lens]
    rs = np.random.RandomState(0)
    draws = [b200asr.TempoGain().draw_one(rs) for _ in range(B)]
    tempo = np.array([t for t, _ in draws], np.float64)
    gain = np.array([TG.linear_gain(d) for _, d in draws], np.float32)
    out_lens = np.array([TG.out_length(n, t) for n, t in zip(lens, tempo)], np.int32)
    segment, search, overlap = TG.geometry(sr)
    step = segment - overlap
    K = -(-out_lens.astype(np.int64) // step)
    dev = lambda v, dt: torch.tensor(np.asarray(v), dtype=dt, device="cuda")  # noqa: E731
    wave = dev(np.concatenate(xs), torch.float32)
    in_off = dev(np.concatenate([[0], np.cumsum(lens)[:-1]]), torch.int64)
    out_off_np = np.concatenate([[0], np.cumsum(out_lens)[:-1]]).astype(np.int64)
    pk_off_np = np.concatenate([[0], np.cumsum(K)[:-1]]).astype(np.int64)
    args = [in_off, dev(lens, torch.int32), dev(tempo, torch.float64), dev(gain, torch.float32)]
    out = torch.empty(int(out_lens.sum()), device="cuda")
    picks = torch.empty(int(K.sum()), dtype=torch.int32, device="cuda")
    o_args = [dev(out_off_np, torch.int64), dev(out_lens, torch.int32), picks, dev(pk_off_np, torch.int64)]
    L = b200asr._lib
    lib = L.load()
    st = torch.cuda.current_stream().cuda_stream

    def call():             # the raw entry point: tempo_gain's uploads would time the host, not the kernel
        L.check(lib.b200asr_tempo_gain(L.ptr(wave), *[L.ptr(t) for t in args], L.ptr(out), *[L.ptr(t) for t in o_args], B,
                                       segment, search, overlap, st), "tempo_gain")
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
    o, p = out.cpu().numpy(), picks.cpu().numpy()
    agree = True
    for b in range(B):
        want, wp, _ = TG.stretch(xs[b], tempo[b], gain[b], (segment, search, overlap))
        agree &= bool(np.array_equal(o[out_off_np[b]:out_off_np[b] + out_lens[b]], want) and
                      np.array_equal(p[pk_off_np[b]:pk_off_np[b] + K[b]], wp))

    # PackedLoader.batch on the same utterances, sorted as collate_items sorts them; the dataset is a stand-in with the
    # reference's defaults (no noise, Hamming), so the reference checkout is not needed here
    loader._data_loader = lambda: None
    loader._window_name = lambda ds, DL: "hamming"
    ds = types.SimpleNamespace(sample_rate=sr, window_size=0.02, window_stride=0.01, normalize=True, noiseInjector=None)
    packed = loader.PackedLoader.__new__(loader.PackedLoader)
    packed.items, packed.bank = types.SimpleNamespace(dataset=ds), None
    pin = lambda t: t.pin_memory()  # noqa: E731

    def packed_batch(stretch):
        n = out_lens if stretch else lens
        order = sorted(range(B), key=lambda i: n[i], reverse=True)
        slens = np.array([lens[i] for i in order], np.int32)
        frames = [1 + int(n[i]) // 160 for i in order]
        kw = {}
        if stretch:
            kw = dict(tempo=pin(torch.tensor(tempo[order])), g=pin(torch.tensor(gain[order])),
                      out_lengths=pin(torch.tensor(out_lens[order])))
        return loader.PackedBatch(
            wave=pin(torch.from_numpy(np.concatenate([xs[i] for i in order]))),
            offsets=pin(torch.from_numpy(np.concatenate([[0], np.cumsum(slens, dtype=np.int64)[:-1]]))),
            lengths=pin(torch.from_numpy(slens)), noise_clip=torch.full((B,), -1), noise_start=pin(torch.full((B,), -1)),
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
    res = dict(what="tempo_gain", B=B, seconds=[round(int(lens.min()) / sr, 2), round(int(lens.max()) / sr, 2)],
               segments_max=int(K.max()), segments_total=int(K.sum()), kernel_us=round(us, 1),
               us_per_segment_chain=round(us / int(K.max()), 2), batch_ms_with=round(med[True], 3),
               batch_ms_without=round(med[False], 3), matches_restatement=agree, gpu=gpu_info())
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")
    if not agree:
        sys.exit("the timed output differs from the restatement")


if __name__ == "__main__":
    main()
