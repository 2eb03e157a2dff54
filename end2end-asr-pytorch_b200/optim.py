"""Step tail (SURVEY.md §8f rank 1): flat parameter/gradient buffers, fused Adam, Noam schedule; and the reference's own
NoamOpt + torch.optim.Adam step and gradient clip on the device.

FlatParams re-homes every parameter of a module into ONE contiguous fp32 buffer (and its gradient into another),
so the data-parallel step is a single NCCL all-reduce and the optimizer a single kernel launch.  adam_step / noam_step /
clip_grad_norm_ (end of the file) work over the separate tensors a stock torch.optim.Adam holds.
"""
from __future__ import annotations

import math

import torch
from torch.optim import optimizer as torch_optimizer

from . import _lib as L
from . import ops


class FlatParams:
    """Views of all trainable parameters (and their .grad) into two flat fp32 buffers.

    The gradient buffer carries `extra` trailing floats (used for [sum-loss, n_tokens]) so that they ride in
    the same all-reduce as the gradients (SURVEY.md §5.8)."""

    def __init__(self, module: torch.nn.Module, extra: int = 2, tail=("conv",)):
        """tail: names of submodules whose parameters go to the END of the buffers (default: the CNN front end `conv`).  Their
        gradients are the last ones backward produces, so everything before `tail_offset` can be all-reduced while the front
        end's backward is still running (parallel.DataParallelStep)."""
        seen, params = set(), []
        tail_ids = set()
        for name in tail:
            sub = getattr(module, name, None)
            if isinstance(sub, torch.nn.Module):
                tail_ids.update(id(p) for p in sub.parameters())

        def take(p, tail_pass=False):
            if p is not None and p.requires_grad and id(p) not in seen and (tail_pass or id(p) not in tail_ids):
                seen.add(id(p))
                params.append(p)

        # Q/K/V projection weights (then their biases) of every attention block go back to back, so that the block can run
        # them -- and their gradients -- as one stacked GEMM operand (ops.AttnProjFn); everything else in module order
        for m in module.modules():
            lin = [getattr(m, n, None) for n in ("query_linear", "key_linear", "value_linear")]
            if all(isinstance(l, torch.nn.Linear) for l in lin):
                for l in lin:
                    take(l.weight)
                for l in lin:
                    take(l.bias)
        for p in module.parameters():
            take(p)
        n_head = len(params)
        for p in module.parameters():
            take(p, tail_pass=True)
        self.params = params
        dev = params[0].device
        sizes = [p.numel() for p in params]
        # 16-byte aligned slots so every view keeps vector-load alignment
        self.offsets, off = [], 0
        for n in sizes:
            self.offsets.append(off)
            off += (n + 3) // 4 * 4
        self.numel = off
        self.tail_offset = self.offsets[n_head] if n_head < len(params) else off      # first element of the tail parameters
        self.extra = extra
        self.flat = torch.zeros(off, device=dev, dtype=torch.float32)
        self.flat_grad = torch.zeros(off + extra, device=dev, dtype=torch.float32)
        with torch.no_grad():
            for p, o, n in zip(params, self.offsets, sizes):
                self.flat[o:o + n].copy_(p.detach().reshape(-1))
                p.data = self.flat[o:o + n].view(p.shape)
                p.grad = self.flat_grad[o:o + n].view(p.shape)
                p._b200_flat_grad = True      # opt-in for ops._grad_sink: backward kernels may accumulate straight into .grad
        if dev.type == "cuda":
            ops.weight_cache = ops.WeightOperandCache(self)     # bf16 operands of all weights: one conversion launch per step

    @property
    def extras(self) -> torch.Tensor:
        return self.flat_grad[self.numel:]

    def zero_grad(self):
        self.flat_grad.zero_()

    def ensure_grad_views(self):
        """Re-attach .grad views if something (e.g. zero_grad(set_to_none=True)) dropped them."""
        for p, o in zip(self.params, self.offsets):
            n = p.numel()
            view = self.flat_grad[o:o + n].view(p.shape)
            if p.grad is None:
                p.grad = view
            elif p.grad.data_ptr() != view.data_ptr():
                view.copy_(p.grad)
                p.grad = view


class FusedAdam:
    """torch.optim.Adam(betas, eps) semantics (utils/functions.py:107) as one kernel over FlatParams."""

    def __init__(self, flat: FlatParams, lr=1e-3, betas=(0.9, 0.98), eps=1e-9):
        self.flat = flat
        self.param_groups = [dict(lr=lr, betas=betas, eps=eps, params=flat.params)]
        self.m = torch.zeros_like(flat.flat)
        self.v = torch.zeros_like(flat.flat)
        self.t = 0

    def zero_grad(self, set_to_none: bool = False):
        self.flat.zero_grad()

    def step(self, grad_scale: float = 1.0, grad_scale_dev: torch.Tensor = None):
        g = self.param_groups[0]
        self.t += 1
        f = self.flat
        L.check(L.load().b200asr_adam_step(L.ptr(f.flat), L.ptr(f.flat_grad), L.ptr(self.m), L.ptr(self.v), f.numel,
                                           float(g["lr"]), float(g["betas"][0]), float(g["betas"][1]), float(g["eps"]),
                                           self.t, float(grad_scale), L.ptr(grad_scale_dev),
                                           torch.cuda.current_stream().cuda_stream), "adam_step")
        if ops.weight_cache is not None and ops.weight_cache.flat is f:
            ops.weight_cache.after_optimizer_step()

    def grad_sumsq(self) -> torch.Tensor:
        out = torch.zeros(1, device=self.flat.flat.device, dtype=torch.float32)
        L.check(L.load().b200asr_sumsq(L.ptr(self.flat.flat_grad), self.flat.numel, L.ptr(out),
                                       torch.cuda.current_stream().cuda_stream), "sumsq")
        return out

    def state_dict(self):
        return dict(m=self.m, v=self.v, t=self.t, param_groups=[{k: v for k, v in self.param_groups[0].items() if k != "params"}])

    def load_state_dict(self, sd):
        self.m.copy_(sd["m"]); self.v.copy_(sd["v"]); self.t = int(sd["t"])


class NoamOpt:
    """utils/optimizer.py:3-32 -- same attributes and methods; `optimizer` may be FusedAdam or any torch optimizer."""

    def __init__(self, model_size, factor, warmup, optimizer, min_lr=1e-5):
        self.optimizer = optimizer
        self._step = 0
        self.warmup = warmup
        self.factor = factor
        self.model_size = model_size
        self._rate = 0
        self.min_lr = min_lr

    def step(self, **kw):
        self._step += 1
        rate = self.rate()
        for g in self.optimizer.param_groups:
            g["lr"] = rate
        self._rate = rate
        self.optimizer.step(**kw)

    def zero_grad(self):
        self.optimizer.zero_grad()

    def rate(self, step=None):
        step = self._step
        return max(self.min_lr, self.factor * (self.model_size ** (-0.5) * min(step ** (-0.5), step * self.warmup ** (-1.5))))


# ---------------------------------------------------------------- the reference's own optimizer on the device
# NoamOpt (utils/optimizer.py:15-22) steps a stock torch.optim.Adam (utils/functions.py:107) that holds every parameter as a
# separate tensor.  adam_step runs that Adam's step as b200asr_adam_multi launches over the optimizer's OWN state tensors, with
# torch's foreach arithmetic bit for bit, so state_dict() / load_state_dict() -- save_model, load_model, --continue-from --
# keep working in both directions with stock torch.  clip_grad_norm_ is torch.nn.utils.clip_grad_norm_ (norm_type 2) with the
# norm and the coefficient on the device.

_DEVICE = "cuda"             # the device type the kernels run on
_ADAM_DEFAULTS = (("amsgrad", False), ("weight_decay", 0), ("maximize", False), ("capturable", False),
                  ("differentiable", False), ("decoupled_weight_decay", False))


def _plain_cuda_fp32(t, device) -> bool:
    """A dense fp32 tensor on `device` whose elements are one contiguous run of memory."""
    return (torch.is_tensor(t) and t.dtype == torch.float32 and t.layout == torch.strided and t.device == device and
            t.is_contiguous())


def adam_eligible(opt) -> bool:
    """True iff adam_step computes what opt.step() would: a torch.optim.Adam (not a subclass) with one param group, default
    flags (foreach None or True), no step hooks, float hyper-parameters, and every parameter, gradient and state tensor a
    dense contiguous fp32 tensor on one CUDA device."""
    if type(opt) is not torch.optim.Adam or len(opt.param_groups) != 1:
        return False
    if opt._optimizer_step_pre_hooks or opt._optimizer_step_post_hooks:
        return False
    if torch_optimizer._global_optimizer_pre_hooks or torch_optimizer._global_optimizer_post_hooks:
        return False
    g = opt.param_groups[0]
    if any(g.get(k, d) != d for k, d in _ADAM_DEFAULTS) or g.get("fused") or g.get("foreach") is False:
        return False
    betas = g.get("betas")
    if not all(isinstance(x, (int, float)) and not isinstance(x, bool) for x in (g.get("lr"), g.get("eps"), *betas)):
        return False
    params = g["params"]
    if not params or params[0].device.type != _DEVICE:
        return False
    dev = params[0].device
    for p in params:
        if not _plain_cuda_fp32(p, dev):
            return False
        if p.grad is not None and not (_plain_cuda_fp32(p.grad, dev) and p.grad.shape == p.shape):
            return False
        st = opt.state.get(p)
        if st:
            step = st.get("step")
            if set(st) != {"step", "exp_avg", "exp_avg_sq"} or not (torch.is_tensor(step) and step.device.type == "cpu" and
                                                                   step.numel() == 1 and step.is_floating_point()):
                return False
            if not all(_plain_cuda_fp32(st[k], dev) and st[k].shape == p.shape for k in ("exp_avg", "exp_avg_sq")):
                return False
    return True


def _tables(n):
    """[start, end) of each launch over a list of n tensors."""
    cap = L.load().b200asr_optim_table_capacity()
    return [(i, min(n, i + cap)) for i in range(0, n, cap)]


def adam_step(opt) -> None:
    """opt.step() of an Adam that adam_eligible accepts, on the device.  Mirrors Adam._init_group: a parameter without a
    gradient is skipped (no state, its step does not advance); state is created lazily as torch creates it (`step` a CPU
    scalar tensor, exp_avg / exp_avg_sq zeros_like(p, preserve_format)); the steps advance by one as torch's foreach path
    advances them; step_size = -lr / (1 - beta1**step) and bias_correction2_sqrt = (1 - beta2**step) ** 0.5 are formed in
    Python doubles per distinct step value."""
    import numpy as np
    g = opt.param_groups[0]
    lr, (beta1, beta2), eps = g["lr"], g["betas"], g["eps"]
    params, grads, exp_avgs, exp_avg_sqs, steps = [], [], [], [], []
    for p in g["params"]:
        if p.grad is None:
            continue
        state = opt.state[p]
        if len(state) == 0:
            state["step"] = torch.tensor(0.0, dtype=torch_optimizer._get_scalar_dtype())
            state["exp_avg"] = torch.zeros_like(p, memory_format=torch.preserve_format)
            state["exp_avg_sq"] = torch.zeros_like(p, memory_format=torch.preserve_format)
        params.append(p)
        grads.append(p.grad)
        exp_avgs.append(state["exp_avg"])
        exp_avg_sqs.append(state["exp_avg_sq"])
        steps.append(state["step"])
    if not params:
        return
    torch._foreach_add_(steps, torch.tensor(1.0, device="cpu"), alpha=1.0)
    values = [s.item() for s in steps]                  # torch's _get_value
    scalars = {}
    for s in values:
        if s not in scalars:
            bc1, bc2 = 1 - beta1 ** s, 1 - beta2 ** s
            scalars[s] = ((lr / bc1) * -1, bc2 ** 0.5)
    per = [scalars[s] for s in values]
    ptrs = np.array([[t.data_ptr() for t in row] for row in zip(params, grads, exp_avgs, exp_avg_sqs)], dtype=np.uint64)
    numel = np.array([p.numel() for p in params], dtype=np.int64)
    step_size = np.array([a for a, _ in per], dtype=np.float32)
    bc2_sqrt = np.array([b for _, b in per], dtype=np.float32)
    dev = params[0].device
    lib = L.load()
    with torch.cuda.device(dev):
        stream = torch.cuda.current_stream(dev).cuda_stream
        for i, j in _tables(len(params)):
            L.check(lib.b200asr_adam_multi(ptrs[i:j].ctypes.data, numel[i:j].ctypes.data, step_size[i:j].ctypes.data,
                                           bc2_sqrt[i:j].ctypes.data, j - i, 1 - beta1, beta2, 1 - beta2, eps, stream),
                    "adam_multi")
    torch._C._increment_version(params + exp_avgs + exp_avg_sqs)


def noam_step(self):
    """utils.optimizer.NoamOpt.step, bound by install(): the same _step / _rate / lr bookkeeping, then adam_step.  An
    optimizer adam_eligible refuses runs the reference's own NoamOpt.step unchanged."""
    if not adam_eligible(self.optimizer):
        from .install import original
        ref = original(type(self), "step")
        if ref is None:
            raise RuntimeError("b200asr noam_step: NoamOpt.step is not installed (b200asr.install())")
        return ref(self)
    self._step += 1
    rate = self.rate()
    for p in self.optimizer.param_groups:
        p["lr"] = rate
    self._rate = rate
    adam_step(self.optimizer)


def clip_eligible(grads) -> bool:
    """True iff clip_grad_norm_ takes these gradients: at least one, each a dense contiguous fp32 CUDA tensor, one device."""
    return bool(grads) and grads[0].device.type == _DEVICE and all(_plain_cuda_fp32(g, grads[0].device) for g in grads)


def clip_grad_norm_(parameters, max_norm, norm_type=2.0, error_if_nonfinite=False, foreach=None) -> torch.Tensor:
    """torch.nn.utils.clip_grad_norm_ for norm_type=2 and error_if_nonfinite=False on the device: per-tensor norms, the norm
    of those norms, coef = min(1, max_norm / (total + 1e-6)) and grad *= coef, without a host synchronisation.  Returns the
    total norm as a 0-dim device tensor.  The sums run in a fixed order, so repeated calls give the same bits; they may
    differ from torch's in the last bits.  Gradients clip_eligible refuses, another norm type or error_if_nonfinite raise
    ValueError (call torch's for those)."""
    import numpy as np
    if torch.is_tensor(parameters):
        parameters = [parameters]
    grads = [p.grad for p in parameters if p.grad is not None]
    if float(norm_type) != 2.0 or error_if_nonfinite:
        raise ValueError("b200asr.clip_grad_norm_ computes norm_type=2 with error_if_nonfinite=False only")
    if not grads:
        return torch.tensor(0.0)
    if not clip_eligible(grads):
        raise ValueError("b200asr.clip_grad_norm_: every gradient must be a dense contiguous fp32 tensor on one CUDA device")
    dev = grads[0].device
    ptrs = np.array([t.data_ptr() for t in grads], dtype=np.uint64)
    numel = np.array([t.numel() for t in grads], dtype=np.int64)
    lib = L.load()
    with torch.cuda.device(dev):
        stream = torch.cuda.current_stream(dev).cuda_stream
        norms = torch.empty(len(grads), device=dev, dtype=torch.float32)
        out = torch.empty(2, device=dev, dtype=torch.float32)       # total norm, clip coefficient
        tables = _tables(len(grads))
        for i, j in tables:
            L.check(lib.b200asr_norm_multi(ptrs[i:j].ctypes.data, numel[i:j].ctypes.data, j - i, norms[i:].data_ptr(),
                                           stream), "norm_multi")
        L.check(lib.b200asr_clip_coef(norms.data_ptr(), len(grads), float(max_norm), out.data_ptr(), stream), "clip_coef")
        for i, j in tables:
            L.check(lib.b200asr_scale_multi(ptrs[i:j].ctypes.data, numel[i:j].ctypes.data, j - i, out[1:].data_ptr(), stream),
                    "scale_multi")
    torch._C._increment_version(grads)
    return out[0]


def sgd_step(parameters, lr) -> None:
    """`for p in parameters: p.data.add_(p.grad, alpha=-lr)`, the update of the word-language-model loop that trains the LSTM
    LM, as b200asr_sgd_multi launches (one per table of tensors): bit-identical to ATen's add_, no copy, no allocation, no
    host synchronisation.  Parameters without a gradient are skipped.  Every parameter and gradient must be a dense
    contiguous fp32 tensor on one CUDA device (ValueError otherwise).  The parameters' version counters advance, as an
    in-place update of the parameter itself would advance them, so caches keyed on them see the new weights."""
    import numpy as np
    params = [parameters] if torch.is_tensor(parameters) else list(parameters)
    params = [p for p in params if p.grad is not None]
    if not params:
        return
    dev = params[0].device
    if dev.type != _DEVICE or not all(_plain_cuda_fp32(p, dev) and _plain_cuda_fp32(p.grad, dev) and p.grad.shape == p.shape
                                      for p in params):
        raise ValueError("b200asr.sgd_step: every parameter and gradient must be a dense contiguous fp32 tensor on one CUDA device")
    ptrs = np.array([[p.data_ptr(), p.grad.data_ptr()] for p in params], dtype=np.uint64)
    numel = np.array([p.numel() for p in params], dtype=np.int64)
    lib = L.load()
    with torch.cuda.device(dev):
        stream = torch.cuda.current_stream(dev).cuda_stream
        for i, j in _tables(len(params)):
            L.check(lib.b200asr_sgd_multi(ptrs[i:j].ctypes.data, numel[i:j].ctypes.data, j - i, -float(lr), stream), "sgd_multi")
    torch._C._increment_version(params)


def clip_grads(parameters, max_norm):
    """clip_grad_norm_ on the device where clip_eligible takes the gradients, torch.nn.utils.clip_grad_norm_ otherwise."""
    parameters = [parameters] if torch.is_tensor(parameters) else list(parameters)
    if clip_eligible([p.grad for p in parameters if p.grad is not None]):
        return clip_grad_norm_(parameters, max_norm)
    return torch.nn.utils.clip_grad_norm_(parameters, max_norm)
