#!/usr/bin/env python
"""Data-parallel parity on real GPUs/NCCL (run under torchrun, N >= 2):
N ranks x (B/N utterances) with ONE all-reduce of the flat gradient buffer  ==  1 rank x B utterances.
Checks loss, every gradient (after the 1/global-token normalisation) and the parameters after one Adam step."""
import importlib
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import b200asr  # noqa: E402
from tests.helpers import rel_err  # noqa: E402

rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
torch.cuda.set_device(local)
dev = torch.device("cuda", local)
dist.init_process_group("nccl", device_id=dev)
cfg = b200asr.ASRConfig(num_layers=2, num_heads=4, dim_model=256, dim_key=64, dim_value=64, dim_inner=512, vocab=500,
                        feat_extractor="vgg_cnn", tgt_max_len=24, dropout=0.0, label_smoothing=0.1)
B, T = 4 * world, 96
g = torch.Generator().manual_seed(0)
src = torch.randn(B, 1, cfg.freq, T, generator=g)
lens = torch.full((B,), T, dtype=torch.int32)
tgt = torch.randint(3, cfg.vocab, (B, cfg.tgt_max_len - 1), generator=g)
for i in range(B):
    tgt[i, 5 + (7 * i) % 15:] = 0                      # ranks see different token counts


def make(group=None, seed=123456):
    torch.manual_seed(seed)
    m = b200asr.build_model(cfg).to(dev)
    m.train()
    return b200asr.DataParallelStep(m, model_size=cfg.dim_input, warmup=10, k_lr=1.0, min_lr=1e-6, smoothing=0.1, process_group=group)


solo = dist.new_group([0])                               # rank 0 alone: the single-rank reference step (collective call: all ranks)
dp = make(seed=123456 + rank)                            # ranks build different replicas; the constructor broadcasts rank 0's
s, l, t = b200asr.shard_batch(src, lens, tgt, rank, world)
dp.step(s.to(dev), l, t.to(dev))
loss_dp = float(dp.global_loss())
g_dp = (dp.flat.flat_grad[:dp.flat.numel] * dp._scale[0]).clone()
p_dp = dp.flat.flat.clone()
if rank == 0:
    ref = make(group=solo)                              # single-rank step on the whole batch: no collective
    assert ref.world == 1
    ref.step(src.to(dev), lens, tgt.to(dev))
    g_ref = ref.flat.flat_grad[:ref.flat.numel] * ref._scale[0]
    print("world %d: loss dp %.6f vs single %.6f | grad rel err %.2e | params-after-step rel err %.2e | n_tokens %d" % (
        world, loss_dp, float(ref.global_loss()), rel_err(g_dp, g_ref), rel_err(p_dp, ref.flat.flat), int(dp.flat.extras[1])))
    assert abs(loss_dp - float(ref.global_loss())) < 1e-4 * abs(loss_dp)
    # parameters: the first Adam step is lr * g / (|g| + 1e-9), i.e. sign-like; entries whose gradient is rounding noise
    # (mathematically zero, e.g. key biases) may step in either direction, so the bound is a few learning rates, not 1e-4
    assert rel_err(g_dp, g_ref) < 1e-3 and rel_err(p_dp, ref.flat.flat) < 1e-2
    print("DP PARITY OK (gradient all-reduce overlapped with the front-end backward: %s)" % (dp.flat.tail_offset < dp.flat.numel))
dist.barrier()
dist.destroy_process_group()
