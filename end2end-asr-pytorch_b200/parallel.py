"""Data-parallel training step: one process per GPU, replicated parameters, ONE all-reduce per step.

Mirrors the reference's `--parallel` nn.DataParallel path (utils/functions.py:154-160, SURVEY.md §3.4) with the
strategy of SURVEY.md §5.8: each rank runs forward/backward on its shard of the utterance batch with the
UN-normalised token-loss sum, the flat gradient buffer (+ [sum-loss, n_tokens]) is all-reduced once over
NCCL/NVLink, and the optimizer divides by the GLOBAL token count -- exactly the reference's normalisation over the
gathered global batch (trainer.py:84 + metrics.py:127-130).

Evaluation shards the same way by utterance, strided instead of chunked: each rank decodes utterances r, r + N, ... of
the batch and one all-gather of fixed-shape id rows (gather_rows) gives every rank the whole batch's result
(modules.evaluate_sharded).
"""
from __future__ import annotations

import os
import random

import numpy as np
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


BACKEND_ENV = "B200ASR_DIST_BACKEND"      # set by b200asr.launch: "nccl", or "gloo" when two ranks share a GPU
_group = None                             # (process group, rank, world size) the bound Trainer.train and evaluate run across


def join(process_group=None):
    """Make the bound Trainer.train data-parallel across `process_group` (a torch.distributed group, or None for the default
    group).  Without a group: join the one the launcher's environment describes (WORLD_SIZE > 1, RANK, MASTER_ADDR,
    MASTER_PORT, B200ASR_DIST_BACKEND), initialising torch.distributed if needed.  Returns (group, rank, world) or None when
    there is nothing to join."""
    global _group
    if process_group is None:
        if int(os.environ.get("WORLD_SIZE", "1")) <= 1:
            return _group
        if not dist.is_initialized():
            dist.init_process_group(os.environ.get(BACKEND_ENV, "nccl"), init_method="env://")
        process_group = dist.group.WORLD
    world = dist.get_world_size(process_group)
    _group = (process_group, dist.get_rank(process_group), world) if world > 1 else None
    return _group


def leave():
    """Forget the group join() recorded (the process group itself stays as it is)."""
    global _group
    _group = None


def joined():
    """(group, rank, world) the bound Trainer.train trains across and the bound Transformer.evaluate decodes across, or None."""
    return _group


def shard_range(B: int, rank: int, world: int):
    """[start, stop) of rank's utterances in a batch of B: chunk `rank` of `torch.arange(B).chunk(world)`, which is how
    nn.DataParallel.scatter splits a batch (chunks of ceil(B / world); the ranks past the last chunk get an empty range)."""
    if world < 1 or not 0 <= rank < world:
        raise ValueError(f"shard_range: rank {rank} of world {world}")
    n = -(-B // world)
    return min(B, rank * n), min(B, (rank + 1) * n)


def _collective_device(process_group=None):
    """Where a collective's tensors live: the current GPU under NCCL, the host under gloo."""
    if dist.get_backend(process_group) == "nccl":
        return torch.device("cuda", torch.cuda.current_device())
    return torch.device("cpu")


def gather_rows(rows, B: int, shape, process_group=None):
    """Every rank's rows of a batch of B utterances, in batch order, as one host tensor [B, *shape] int64.

    Rank r holds the rows of utterances r, r + N, r + 2N, ... (`rows` [len(range(r, B, N)), *shape] int64 on any device, or
    None when it holds none).  ONE all-gather of a fixed block [ceil(B / N), *shape] per rank, padded with -1: on the device
    under NCCL, on the host under gloo.  Row j of rank r's block is utterance j * N + r, so the gathered blocks interleave
    into batch order."""
    world = dist.get_world_size(process_group)
    rank = dist.get_rank(process_group)
    n = -(-B // world)
    dev = _collective_device(process_group)
    block = torch.full((n,) + tuple(shape), -1, dtype=torch.int64, device=dev)
    mine = len(range(rank, B, world))
    if mine:
        if rows is None or tuple(rows.shape) != (mine,) + tuple(shape):
            raise ValueError(f"gather_rows: rank {rank} of {world} holds {mine} of {B} rows of shape {tuple(shape)}, "
                             f"got {None if rows is None else tuple(rows.shape)}")
        block[:mine] = rows.to(device=dev, dtype=torch.int64)
    parts = [torch.empty_like(block) for _ in range(world)]
    dist.all_gather(parts, block, group=process_group)
    return torch.stack(parts, dim=1).reshape((n * world,) + tuple(shape))[:B].cpu()


def broadcast_params(flat, process_group=None):
    """Replicas start identical: rank 0's flat parameter buffer is broadcast to every rank.  nn.DataParallel re-replicates
    from device 0 every step (utils/functions.py:154-160); once is enough here because every rank applies the same update."""
    src = dist.get_global_rank(process_group, 0) if process_group is not None else 0
    dist.broadcast(flat.flat, src=src, group=process_group)


def broadcast_module_state(module, flat, process_group=None):
    """Rank 0's copy of everything in `module` that the flat buffer does not hold -- frozen parameters and buffers
    (BatchNorm running statistics, num_batches_tracked, the positional table) -- broadcast to every rank, so that
    replicas built or loaded differently start identical."""
    src = dist.get_global_rank(process_group, 0) if process_group is not None else 0
    held = {id(p) for p in flat.params}
    for t in [p for p in module.parameters() if id(p) not in held] + list(module.buffers()):
        if t.data.is_contiguous():
            dist.broadcast(t.data, src=src, group=process_group)
        else:
            c = t.data.contiguous()
            dist.broadcast(c, src=src, group=process_group)
            t.data.copy_(c)


def seed_host_rngs(process_group=None):
    """Seed Python's `random`, numpy's global generator and torch's CPU generator identically on every rank, from a seed
    rank 0 draws from its own `random` and broadcasts.  The reference's data order comes from these generators:
    BucketingSampler shuffles its bins (`shuffle(epoch)`) and the ids inside each bin with np.random, SpectrogramDataset
    picks a manifest with random.randint, and the DataLoader draws its workers' base seed from torch's CPU generator.  With
    the same seed every rank's loader yields the same global batches, of which each rank then trains its own chunk.
    Returns the seed."""
    src = dist.get_global_rank(process_group, 0) if process_group is not None else 0
    seed = torch.tensor([random.getrandbits(62)], dtype=torch.int64, device=_collective_device(process_group))
    dist.broadcast(seed, src=src, group=process_group)
    s = int(seed.item())
    random.seed(s)
    np.random.seed(s % 2 ** 32)
    torch.manual_seed(s)
    return s


def fold_rank_into_dropout(rank: int):
    """Ranks draw DIFFERENT dropout masks for their shards: the kernels' counter-based generator is seeded per process."""
    ops.rng.seed = (ops.rng.seed ^ (0x9E3779B97F4A7C15 * (rank + 1))) & 0xFFFFFFFFFFFFFFFF


class GradAllReduce:
    """ONE logical all-reduce(SUM) of a FlatParams gradient buffer (with its extras) per step.  When the CNN front end's
    parameters sit at the tail of the buffer (0 < flat.tail_offset < numel) it goes out in two pieces: the head -- every
    gradient before tail_offset, final once the front end's backward starts -- is issued from ops.frontend_backward_hook on
    the process group's own stream and runs under the convolution backward; the tail follows after backward.  A rank whose
    backward did not reach the hook (an empty shard) issues the head itself, so every rank issues the same collectives."""

    def __init__(self, flat, process_group=None):
        self.flat = flat
        self.pg = process_group
        self.world = dist.get_world_size(process_group) if dist.is_available() and dist.is_initialized() else 1
        self._early = None

    def _split(self) -> bool:
        return 0 < self.flat.tail_offset < self.flat.numel

    def _reduce_head_early(self):
        if self.world > 1 and self._early is None and self._split():
            self._early = dist.all_reduce(self.flat.flat_grad[:self.flat.tail_offset], op=dist.ReduceOp.SUM, group=self.pg,
                                          async_op=True)

    def backward(self, loss):
        """loss.backward() with the head of the all-reduce issued under the front end's backward."""
        self._early = None
        prev, ops.frontend_backward_hook = ops.frontend_backward_hook, self._reduce_head_early
        try:
            loss.backward()
        finally:
            ops.frontend_backward_hook = prev

    def finish(self):
        """The rest of the all-reduce; on return the whole buffer holds the sums over the ranks."""
        if self.world <= 1:
            return
        g = self.flat.flat_grad
        if self._split():
            if self._early is None:
                self._reduce_head_early()
            dist.all_reduce(g[self.flat.tail_offset:], op=dist.ReduceOp.SUM, group=self.pg)
            self._early.wait()
            self._early = None
        else:
            dist.all_reduce(g, op=dist.ReduceOp.SUM, group=self.pg)


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
        self.reducer = GradAllReduce(self.flat, process_group)
        self.world = self.reducer.world
        self.clip = clip_max_norm
        self._scale = torch.zeros(4, device=self.flat.flat.device, dtype=torch.float32)    # [scale, grad norm, scratch, -]
        self._host_tail = loss_fn is not None or adam_factory is not None                  # CPU stand-ins (gloo tests)
        if self.world > 1:
            broadcast_params(self.flat, process_group)
            fold_rank_into_dropout(dist.get_rank(process_group))

    def forward_backward(self, src, lengths, tgt):
        """Local shard fwd+bwd with the un-normalised loss; gradients land in the flat buffer."""
        self.flat.zero_grad()
        pred, gold, hyp, _ = self.model(src, lengths, tgt)
        loss_sum, stats = self.loss_fn(pred, gold, self.smoothing, reduction="sum")
        self.reducer.backward(loss_sum)
        self.flat.ensure_grad_views()
        self.flat.extras.copy_(stats[0:2])            # [sum-loss, n_tokens] ride with the gradients
        return pred, hyp, stats

    def all_reduce(self):
        """ONE logical all-reduce(SUM) of [flat grads | sum-loss | n_tokens] per step (the reference's --parallel reduce,
        utils/functions.py:154-160): issued as a head part that overlaps the front end's backward (when forward_backward
        could launch it) and the remaining tail (front-end gradients + the two scalars), or in one piece when the model has no
        front end at the tail of the buffer (GradAllReduce)."""
        self.reducer.finish()

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
