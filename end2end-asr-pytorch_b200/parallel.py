"""Data-parallel training step: one process per GPU, replicated parameters, ONE all-reduce per step.

Mirrors the reference's `--parallel` nn.DataParallel path (utils/functions.py:154-160, SURVEY.md §3.4) with the
strategy of SURVEY.md §5.8: each rank runs forward/backward on its shard of the utterance batch with the
UN-normalised token-loss sum, the flat gradient buffer (+ [sum-loss, n_tokens]) is all-reduced once over
NCCL/NVLink, and the optimizer divides by the GLOBAL token count -- exactly the reference's normalisation over the
gathered global batch (trainer.py:84 + metrics.py:127-130).
"""
from __future__ import annotations

import os

import torch
import torch.distributed as dist

from . import _lib as L
from . import metrics, ops
from .optim import FlatParams, FusedAdam, NoamOpt


def shard_batch(src, lengths, tgt, rank: int, world: int):
    """Rank r takes utterances [r*B/N, (r+1)*B/N) of the (length-sorted) batch, as DataParallel.scatter would."""
    B = src.shape[0]
    if B % world:
        raise ValueError("the batch has to be divisible by the number of GPUs (reference README.md:73)")
    n = B // world
    sl = slice(rank * n, (rank + 1) * n)
    return src[sl], lengths[sl], tgt[sl]


class HostBatchPrefetcher:
    """Pinned host batches -> device on a side stream, one batch ahead of the step that consumes them (what a DataLoader with
    pin_memory does for the reference's `src.cuda()` / `tgt.cuda()`, trainer/asr/trainer.py:66-68, minus the stall: the copy of
    batch i+1 runs under the kernels of batch i).

        pf = HostBatchPrefetcher(device)
        pf.submit(src_h, tgt_h)                 # before the loop
        for ...:
            src, tgt = pf.take()                # the compute stream waits for that copy only
            pf.submit(next_src_h, next_tgt_h)   # starts copying now
            dp.step(src, lengths, tgt)
    """

    def __init__(self, device):
        self.device = torch.device(device)
        self.stream = torch.cuda.Stream(device=self.device)
        self.pending = None

    def submit(self, *host_tensors):
        with torch.cuda.stream(self.stream):
            dev = tuple(t.to(self.device, non_blocking=True) for t in host_tensors)
            ev = torch.cuda.Event()
            ev.record(self.stream)
        self.pending = (dev, ev)

    def take(self):
        if self.pending is None:
            raise RuntimeError("HostBatchPrefetcher.take() without a submitted batch")
        (dev, ev), self.pending = self.pending, None
        cur = torch.cuda.current_stream(self.device)
        cur.wait_event(ev)
        for t in dev:
            t.record_stream(cur)                # allocated on the side stream, consumed on the compute stream
        return dev


class DataParallelStep:
    """zero_grad -> forward -> CE(sum) -> backward -> single all-reduce -> Adam(1/global_tokens)."""

    def __init__(self, model, model_size, warmup=4000, k_lr=1.0, min_lr=1e-5, smoothing=0.0, process_group=None,
                 clip_max_norm=None, loss_fn=None, adam_factory=None):
        """loss_fn(pred, gold, smoothing, reduction='sum') -> (loss_sum, stats[sum, n_tokens, ...]) and
        adam_factory(flat) default to the CUDA kernels; the gloo/CPU tests of the host protocol inject stand-ins."""
        self.model = model
        self.flat = FlatParams(model, extra=2)
        self.loss_fn = loss_fn or metrics.loss_and_stats
        self.adam = (adam_factory or (lambda f: FusedAdam(f, betas=(0.9, 0.98), eps=1e-9)))(self.flat)
        self.opt = NoamOpt(model_size, k_lr, warmup, self.adam, min_lr=min_lr)
        self.smoothing = smoothing
        self.pg = process_group
        self.world = dist.get_world_size(process_group) if dist.is_available() and dist.is_initialized() else 1
        self.clip = clip_max_norm
        # all-reduce the transformer's gradients under the CNN front end's backward / dense-layer weight gradients on a second
        # stream (ops._WgradStream); the environment switches exist for A/B measurements
        self.overlap = os.environ.get("B200ASR_DP_OVERLAP", "1") != "0"
        self.async_wgrad = os.environ.get("B200ASR_ASYNC_WGRAD", "0") != "0"    # measured and rejected, see ops._WgradStream
        self._early = None
        self._scale = torch.zeros(4, device=self.flat.flat.device, dtype=torch.float32)    # [scale, grad norm, scratch, -]
        self._host_tail = loss_fn is not None or adam_factory is not None                  # CPU stand-ins (gloo tests)
        if self.world > 1:
            # replicas start identical (nn.DataParallel re-replicates from device 0 every step, utils/functions.py:158-160;
            # here once is enough because every rank applies the identical update) ...
            dist.broadcast(self.flat.flat, src=dist.get_global_rank(process_group, 0) if process_group is not None else 0,
                           group=process_group)
            # ... but draw DIFFERENT dropout masks for their shards (the kernels' counter-based generator is seeded per process)
            ops.rng.seed = (ops.rng.seed ^ (0x9E3779B97F4A7C15 * (dist.get_rank(process_group) + 1))) & 0xFFFFFFFFFFFFFFFF

    def _reduce_head_early(self):
        """Runs at the start of the CNN front end's backward (ops.frontend_backward_hook): every gradient before
        flat.tail_offset is final, so their all-reduce is issued now, on NCCL's own stream, under the convolution backward."""
        if self.world > 1 and self._early is None and 0 < self.flat.tail_offset < self.flat.numel:
            ops.wgrad_stream.sync()          # the dense layers' weight gradients queued on the side stream
            self._early = dist.all_reduce(self.flat.flat_grad[:self.flat.tail_offset], op=dist.ReduceOp.SUM, group=self.pg, async_op=True)

    def forward_backward(self, src, lengths, tgt):
        """Local shard fwd+bwd with the un-normalised loss; gradients land in the flat buffer."""
        self.flat.zero_grad()
        pred, gold, hyp, _ = self.model(src, lengths, tgt)
        loss_sum, stats = self.loss_fn(pred, gold, self.smoothing, reduction="sum")
        self._early = None
        prev, ops.frontend_backward_hook = ops.frontend_backward_hook, (self._reduce_head_early if self.overlap else None)
        ops.wgrad_stream.enabled = self.async_wgrad and not self._host_tail
        try:
            loss_sum.backward()
        finally:
            ops.frontend_backward_hook = prev
            ops.wgrad_stream.enabled = False
            ops.wgrad_stream.sync()
        self.flat.ensure_grad_views()
        self.flat.extras.copy_(stats[0:2])            # [sum-loss, n_tokens] ride with the gradients
        return pred, hyp, stats

    def all_reduce(self):
        """ONE logical all-reduce(SUM) of [flat grads | sum-loss | n_tokens] per step (the reference's --parallel reduce,
        utils/functions.py:154-160): issued as a head part that overlaps the front end's backward (when forward_backward
        could launch it) and the remaining tail (front-end gradients + the two scalars), or in one piece otherwise."""
        if self.world <= 1:
            return
        if self._early is not None:
            dist.all_reduce(self.flat.flat_grad[self.flat.tail_offset:], op=dist.ReduceOp.SUM, group=self.pg)
            self._early.wait()
            self._early = None
        else:
            dist.all_reduce(self.flat.flat_grad, op=dist.ReduceOp.SUM, group=self.pg)

    def optimizer_step(self):
        """Adam with the gradient read as g * (1 / global n_tokens) * clip coefficient -- both computed on the device
        (b200asr_grad_scale): no host round trip between the all-reduce and the update (trainer.py:108-111)."""
        if self._host_tail:                                                # protocol tests on CPU / gloo
            inv = 1.0 / float(self.flat.extras[1])
            scale = 1.0
            if self.clip is not None:
                norm = float(self.flat.flat_grad[:self.flat.numel].norm()) * inv
                scale = min(1.0, self.clip / (norm + 1e-6))
            self._scale[0] = inv * scale
        else:
            f = self.flat
            L.check(L.load().b200asr_grad_scale(L.ptr(f.flat_grad), f.numel, f.extras[1:2].data_ptr(),
                                                float(self.clip) if self.clip is not None else 0.0, self._scale[2:3].data_ptr(),
                                                L.ptr(self._scale), torch.cuda.current_stream().cuda_stream), "grad_scale")
        self.opt.step(grad_scale=1.0, grad_scale_dev=self._scale[0:1])

    def grad_norm(self) -> torch.Tensor:
        """Norm of the token-normalised global gradient of the last step (device scalar; 0 when clipping is off)."""
        return self._scale[1]

    def step(self, src, lengths, tgt):
        pred, hyp, stats = self.forward_backward(src, lengths, tgt)
        self.all_reduce()
        self.optimizer_step()
        return pred, hyp, stats

    def global_loss(self) -> torch.Tensor:
        """Mean loss over the global batch (device tensor): all-reduced sum / all-reduced token count."""
        e = self.flat.extras
        return e[0] / e[1]
