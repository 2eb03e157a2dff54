"""Host side of the device Adam step and gradient clip (no GPU needed; the library is replaced by a recorder):

  * optim.adam_eligible / clip_eligible: which optimizers and gradients take the device path;
  * optim.adam_step: lazy state exactly as torch.optim.Adam creates it, parameters without a gradient skipped, steps advanced,
    the per-tensor scalars torch forms, and the list split into tables of b200asr_optim_table_capacity() tensors;
  * optim.clip_grad_norm_: its launches per table;
  * install() binds utils.optimizer.NoamOpt.step and uninstall() restores it.
"""
import contextlib
import importlib
import types

import numpy as np
import pytest
import torch

import b200asr

OP = importlib.import_module(b200asr.__name__ + ".optim")
from oracle import ref_shim


class RecordingLib:
    """Stands in for libb200asr: records each call's host arrays."""

    def __init__(self, capacity=4):
        self.capacity = capacity
        self.calls = []

    def b200asr_optim_table_capacity(self):
        return self.capacity

    @staticmethod
    def _arr(addr, n, dtype, width=1):
        return np.ctypeslib.as_array((np.ctypeslib.as_ctypes_type(dtype) * (n * width)).from_address(addr)).copy()

    def b200asr_adam_multi(self, tensors, numel, step_size, bc2_sqrt, count, w, b2, omb2, eps, stream):
        self.calls.append(("adam", self._arr(tensors, count, np.uint64, 4).reshape(count, 4), self._arr(numel, count, np.int64),
                           self._arr(step_size, count, np.float32), self._arr(bc2_sqrt, count, np.float32), w, b2, omb2, eps))
        return 0

    def b200asr_norm_multi(self, tensors, numel, count, norms, stream):
        self.calls.append(("norm", self._arr(tensors, count, np.uint64), self._arr(numel, count, np.int64), norms))
        return 0

    def b200asr_clip_coef(self, norms, count, max_norm, out, stream):
        self.calls.append(("coef", count, max_norm))
        return 0

    def b200asr_scale_multi(self, tensors, numel, count, coef, stream):
        self.calls.append(("scale", self._arr(tensors, count, np.uint64), self._arr(numel, count, np.int64)))
        return 0


@pytest.fixture
def host(monkeypatch):
    """CPU tensors stand for device tensors; the library records instead of launching."""
    lib = RecordingLib()
    monkeypatch.setattr(OP, "_DEVICE", "cpu")
    monkeypatch.setattr(OP.L, "load", lambda *a, **k: lib)
    monkeypatch.setattr(torch.cuda, "device", lambda d: contextlib.nullcontext())
    monkeypatch.setattr(torch.cuda, "current_stream", lambda d=None: types.SimpleNamespace(cuda_stream=0))
    return lib


def params(sizes, seed=0):
    g = torch.Generator().manual_seed(seed)
    return [torch.nn.Parameter(torch.randn(n, generator=g)) for n in sizes]


def with_grads(ps, none=()):
    for i, p in enumerate(ps):
        p.grad = None if i in none else torch.randn(p.shape, dtype=p.dtype)
    return ps


def test_eligibility_rules(host):
    ps = with_grads(params([3, 4]))
    assert OP.adam_eligible(torch.optim.Adam(ps, betas=(0.9, 0.98), eps=1e-9))
    assert OP.adam_eligible(torch.optim.Adam(ps, foreach=True))
    for kw in (dict(amsgrad=True), dict(weight_decay=0.1), dict(maximize=True), dict(foreach=False), dict(fused=True),
               dict(capturable=True), dict(differentiable=True), dict(decoupled_weight_decay=True)):
        try:
            opt = torch.optim.Adam(ps, **kw)
        except (RuntimeError, ValueError):
            continue
        assert not OP.adam_eligible(opt), kw
    assert not OP.adam_eligible(torch.optim.Adam([{"params": ps[:1]}, {"params": ps[1:]}]))
    assert not OP.adam_eligible(torch.optim.AdamW(ps))
    assert not OP.adam_eligible(torch.optim.SGD(ps, lr=0.1))
    assert not OP.adam_eligible(torch.optim.Adam(ps, lr=torch.tensor(0.01), foreach=False))
    assert not OP.adam_eligible(torch.optim.Adam(with_grads([torch.nn.Parameter(torch.zeros(3, dtype=torch.float16))])))
    assert not OP.adam_eligible(torch.optim.Adam(with_grads([torch.nn.Parameter(torch.zeros(4, 3).t())])))
    p = torch.nn.Parameter(torch.zeros(4))
    p.grad = torch.zeros(8)[::2]                                    # a strided gradient
    assert not OP.adam_eligible(torch.optim.Adam([p]))
    opt = torch.optim.Adam(ps)
    h = opt.register_step_pre_hook(lambda *a: None)
    assert not OP.adam_eligible(opt)
    h.remove()
    assert OP.adam_eligible(opt)
    # CPU tensors are not the kernels' device
    OP._DEVICE = "cuda"
    assert not OP.adam_eligible(torch.optim.Adam(ps))
    assert not OP.clip_eligible([p.grad for p in ps])
    OP._DEVICE = "cpu"
    assert OP.clip_eligible([p.grad for p in ps])
    assert not OP.clip_eligible([])
    assert not OP.clip_eligible([torch.zeros(3, dtype=torch.float16)])
    assert not OP.clip_eligible([torch.zeros(4, 3).t()])


def test_lazy_state_skips_parameters_without_a_gradient(host):
    ps = with_grads(params([5, 7, 9]), none={1})
    opt = torch.optim.Adam(ps, betas=(0.9, 0.98), eps=1e-9)
    ref = torch.optim.Adam([torch.nn.Parameter(p.detach().clone()) for p in ps], betas=(0.9, 0.98), eps=1e-9)
    for q, p in zip(ref.param_groups[0]["params"], ps):
        q.grad = None if p.grad is None else p.grad.clone()
    ref.step()
    OP.adam_step(opt)
    assert ps[1] not in opt.state and len(opt.state) == 2
    for p, q in zip(ps, ref.param_groups[0]["params"]):
        if p.grad is None:
            continue
        s, r = opt.state[p], ref.state[q]
        assert set(s) == set(r) == {"step", "exp_avg", "exp_avg_sq"}
        assert s["step"].device.type == "cpu" and s["step"].dtype == r["step"].dtype and s["step"].dim() == 0
        assert float(s["step"]) == float(r["step"]) == 1.0
        for k in ("exp_avg", "exp_avg_sq"):
            assert s[k].shape == p.shape and s[k].dtype == p.dtype and s[k].is_contiguous()
    # the state tensors are the ones handed to the kernel, and the ones state_dict() saves
    (_, ptrs, numel, *_), = host.calls
    assert [int(x) for x in ptrs[:, 0]] == [ps[0].data_ptr(), ps[2].data_ptr()]
    assert [int(x) for x in ptrs[:, 2]] == [opt.state[ps[0]]["exp_avg"].data_ptr(), opt.state[ps[2]]["exp_avg"].data_ptr()]
    assert [int(x) for x in ptrs[:, 3]] == [opt.state[ps[0]]["exp_avg_sq"].data_ptr(), opt.state[ps[2]]["exp_avg_sq"].data_ptr()]
    assert list(numel) == [5, 9]
    sd = opt.state_dict()
    assert sd["state"][0]["exp_avg"] is opt.state[ps[0]]["exp_avg"]


def test_scalars_per_distinct_step_and_versions(host):
    ps = with_grads(params([4, 4, 4]))
    opt = torch.optim.Adam(ps, lr=0.003, betas=(0.8, 0.95), eps=1e-7)
    OP.adam_step(opt)
    ps[1].grad = None
    OP.adam_step(opt)
    ps[1].grad = torch.randn(4)
    v0 = [p._version for p in ps]
    OP.adam_step(opt)
    assert [float(opt.state[p]["step"]) for p in ps] == [3.0, 2.0, 3.0]
    assert all(p._version > v for p, v in zip(ps, v0))          # the kernel's in-place update is visible to version checks
    _, _, _, ss, bc, w, b2, omb2, eps = host.calls[-1]
    for k, s in enumerate([3.0, 2.0, 3.0]):
        assert ss[k] == np.float32((0.003 / (1 - 0.8 ** s)) * -1)
        assert bc[k] == np.float32((1 - 0.95 ** s) ** 0.5)
    assert (w, b2, omb2, eps) == (1 - 0.8, 0.95, 1 - 0.95, 1e-7)


def test_long_lists_are_split_into_tables(host):
    ps = with_grads(params([1 + i for i in range(10)]), none={4})
    OP.adam_step(torch.optim.Adam(ps))
    assert [len(c[2]) for c in host.calls] == [4, 4, 1]
    assert [int(n) for c in host.calls for n in c[2]] == [1, 2, 3, 4, 6, 7, 8, 9, 10]
    host.calls.clear()
    total = OP.clip_grad_norm_(ps, 1.0)
    kinds = [c[0] for c in host.calls]
    assert kinds == ["norm"] * 3 + ["coef"] + ["scale"] * 3
    assert [len(c[1]) for c in host.calls if c[0] == "norm"] == [4, 4, 1]
    norm_calls = [c for c in host.calls if c[0] == "norm"]
    assert norm_calls[1][3] - norm_calls[0][3] == 4 * 4             # each table writes its own slice of the norms
    assert host.calls[3][1:] == (9, 1.0)
    assert total.dim() == 0


def test_clip_rejects_what_it_does_not_compute(host):
    ps = with_grads(params([3]))
    with pytest.raises(ValueError):
        OP.clip_grad_norm_(ps, 1.0, norm_type=1)
    with pytest.raises(ValueError):
        OP.clip_grad_norm_(ps, 1.0, error_if_nonfinite=True)
    assert float(OP.clip_grad_norm_(params([3]), 1.0)) == 0.0        # no gradients: torch's 0
    q = torch.nn.Parameter(torch.zeros(3, dtype=torch.float16))
    q.grad = torch.zeros(3, dtype=torch.float16)
    with pytest.raises(ValueError):
        OP.clip_grad_norm_([q], 1.0)
    host.calls.clear()
    OP.clip_grads([q], 1.0)                                         # the trainer's helper hands it to torch
    assert host.calls == []


@pytest.mark.skipif(not ref_shim.available(), reason="reference checkout not staged (oracle/make_ref.py)")
def test_install_binds_and_uninstall_restores_noam_step():
    ref_shim.load([])
    import utils.optimizer as uo
    before = uo.NoamOpt.step
    b200asr.install()
    try:
        assert uo.NoamOpt.step is OP.noam_step
        assert b200asr.original(uo.NoamOpt, "step") is before
    finally:
        b200asr.uninstall()
    assert uo.NoamOpt.step is before


@pytest.mark.skipif(not ref_shim.available(), reason="reference checkout not staged (oracle/make_ref.py)")
def test_noam_step_keeps_the_schedule_and_falls_back(host):
    ref_shim.load([])
    import utils.optimizer as uo
    b200asr.install()
    try:
        ps = with_grads(params([4, 4]))
        opt = uo.NoamOpt(512, 1.0, 4, torch.optim.Adam(ps, betas=(0.9, 0.98), eps=1e-9), min_lr=1e-5)
        opt.step()
        opt.step()
        assert opt._step == 2 and opt._rate == opt.rate() and opt.optimizer.param_groups[0]["lr"] == opt._rate
        assert [c[0] for c in host.calls] == ["adam", "adam"]
        host.calls.clear()
        sgd = uo.NoamOpt(512, 1.0, 4, torch.optim.Adam(ps, amsgrad=True), min_lr=1e-5)
        sgd.step()                                                  # the reference's own step, torch's Adam
        assert host.calls == [] and sgd._step == 1 and float(sgd.optimizer.state[ps[0]]["step"]) == 1.0
    finally:
        b200asr.uninstall()
