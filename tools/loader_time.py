#!/usr/bin/env python
"""Does the installed AudioDataLoader keep up with the bound training iteration?  Times, at cfg2's shape:

  * batches/s of the installed loader over one epoch (workers read audio and draw, the main process uploads the packed
    batch and runs one b200asr_stft_features_packed call), and the main-process host time per batch (the time spent
    in the loader's device step, PackedLoader.batch);
  * ms per iteration of the reference's Trainer.train (bound, cfg2 architecture, CE) over one epoch fed by the installed
    loader, against the same loop over the same batches pre-built on the device: the time from the first training
    iteration's optimizer step to the last one's over the iterations between them, so the first iteration (warm-up),
    the validation pass and the checkpoint (save_model is a no-op here) are not in it.

    python tools/loader_time.py [--batches 24] [--workers 4]

B = 32 utterances of 4 to 16 s at 16 kHz (seeded), src_max_len 4000 (not binding), noise off and on (noise_prob 0.5 from
four 20 s clips); audio is served from memory by tests/test_loader_host.py's stubs of the reference's audio helpers, so
the workers' time is the reference's own Python around them, not file decoding.  The loader's batches/s are over a
whole epoch, worker start-up included (the reference's loader starts its workers every epoch too).  The reference's own
loader (librosa on the workers) is timed only where librosa imports; otherwise it is
reported as not measured.  Also printed: the card, its power limit and max SM clock, read in the same run.
"""
import argparse
import importlib.util
import copy
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import b200asr  # noqa: E402
from oracle import ref_shim  # noqa: E402

CFG2 = ["--num-layers", "4", "--num-heads", "8", "--dim-model", "512", "--dim-emb", "512", "--dim-key", "64", "--dim-value", "64",
        "--dim-inner", "2048", "--feat_extractor", "vgg_cnn", "--tgt-max-len", "40", "--dropout", "0.1", "--cuda",
        "--label-smoothing", "0.1", "--src-max-len", "4000"]


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[torch.cuda.current_device()] if q.returncode == 0 else "nvidia-smi unavailable"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, default=24)
    ap.add_argument("--workers", type=int, default=4)
    a = ap.parse_args()
    librosa = importlib.import_module("librosa") if importlib.util.find_spec("librosa") else None    # before the stubs
    from tests.test_loader_host import Env
    from b200asr import loader as LD
    mp = pytest.MonkeyPatch()
    env = Env(mp)
    env.clips = {f"noise_{i}.wav": (0.2 * np.random.default_rng(90 + i).standard_normal(320000)).astype(np.float32)
                 for i in range(4)}
    DL = env.DL
    B = 32
    lengths = np.random.default_rng(0).integers(64000, 256001, B * a.batches).tolist()
    host_ms = []
    orig_batch = LD.PackedLoader.batch

    def timed_batch(self, pb):
        t = time.perf_counter()
        out = orig_batch(self, pb)
        host_ms.append(1e3 * (time.perf_counter() - t))
        return out

    mp.setattr(LD.PackedLoader, "batch", timed_batch)
    mp.setattr(env.ns.trainer, "save_model", lambda *args, **kwargs: None)        # no checkpoint in the timed epochs
    results = {"gpu": gpu_info(), "command": " ".join([os.path.basename(sys.argv[0])] + sys.argv[1:]), "B": B,
               "batches": a.batches, "workers": a.workers}
    with tempfile.TemporaryDirectory() as tmp:
        for noise in (False, True):
            tag = "noise" if noise else "plain"
            ns = ref_shim.load(CFG2)
            ds = env.dataset(__import__("pathlib").Path(tmp), lengths, prob=0.5 if noise else None, manifests=1)
            b200asr.install()
            try:
                mk = lambda: DL.AudioDataLoader(ds, num_workers=a.workers, batch_sampler=DL.BucketingSampler(ds, batch_size=B))  # noqa: E731
                list(mk())                                                          # warm-up: workers, kernels, the bank
                torch.cuda.synchronize()
                host_ms.clear()
                t = time.perf_counter()
                batches = [tuple(x.clone() if x.is_cuda else x for x in bt) for bt in mk()]
                torch.cuda.synchronize()
                dt = time.perf_counter() - t
                results[f"{tag}.loader_batches_per_s"] = round(a.batches / dt, 2)
                results[f"{tag}.main_host_ms_per_batch"] = round(float(np.median(host_ms)), 3)
                l2i = env.label2id
                i2l = {i: c for c, i in l2i.items()}
                valid = [[copy.deepcopy(batches[0])]]
                arms = {}
                for arm in ("prebuilt", "loader", "prebuilt", "loader"):
                    torch.manual_seed(1)
                    model = ns.functions.init_transformer_model(ns.constant.args, l2i, i2l).cuda()
                    ns.constant.args.save_folder, ns.constant.args.name = tmp, f"{tag}_{arm}"
                    opt = ns.functions.init_optimizer(ns.constant.args, model, "noam")
                    stamps, step = [], opt.step

                    def stamped_step(step=step, stamps=stamps):      # the loop reads the loss every iteration, so a
                        stamps.append(time.perf_counter())          # host stamp here follows the device closely
                        return step()

                    opt.step = stamped_step
                    train = mk() if arm == "loader" else copy.deepcopy(batches)
                    ns.trainer.Trainer().train(model, train, None, copy.deepcopy(valid), opt, "ce", 0, 1, l2i, i2l)
                    assert len(stamps) == a.batches
                    arms.setdefault(arm, []).append(1e3 * (stamps[-1] - stamps[0]) / (a.batches - 1))
                for arm, v in arms.items():
                    results[f"{tag}.trainer_ms_per_iter.{arm}"] = [round(x, 2) for x in v]
            finally:
                b200asr.uninstall()
            if librosa is None:
                results[f"{tag}.reference_loader"] = "not measured (librosa is not installed)"
            else:                                                   # the unmodified loader with the real librosa.stft
                mp.setattr(DL, "librosa", librosa)
                list(mk())
                t = time.perf_counter()
                list(mk())
                results[f"{tag}.reference_loader_batches_per_s"] = round(a.batches / (time.perf_counter() - t), 2)
    mp.undo()
    print(json.dumps(results))


if __name__ == "__main__":
    main()
