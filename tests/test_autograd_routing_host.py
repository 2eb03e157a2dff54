"""The rule that lets the backward kernels of ops.py add weight gradients straight into a parameter's .grad (ops._grad_sink),
checked on CPU tensors with a toy autograd Function that routes its weight gradient exactly as LinearFn does: into .grad when
the rule allows, else back to autograd.  The rule must give PyTorch's own semantics in every way a caller can ask for
gradients -- plain backward, backward(inputs=...), autograd.grad, frozen parameters, tensor hooks -- because the sink
bypasses the engine.  It rests on torch._C._will_engine_execute_node, a private API of the pinned torch; these tests are what
notices if its behaviour changes.  Also: the backwards refuse create_graph=True, and every autograd Function of ops.py is
in the sweep table of tests/test_gpu_autograd_routing.py (no GPU needed)."""
import importlib
import inspect

import pytest
import torch

import b200asr

ops = importlib.import_module(b200asr.__name__ + ".ops")


class ToyLinearFn(torch.autograd.Function):
    """y = x * w (elementwise); dw = dy * x goes into w.grad when ops' sink rule allows (recorded in `sunk`)."""
    sunk = []

    @staticmethod
    def forward(ctx, x, w):
        ctx.save_for_backward(x, w)
        ctx.w = w
        return x * w

    @staticmethod
    @ops._backward
    def backward(ctx, dy):
        x, w = ctx.saved_tensors
        dw = dy * x if ctx.needs_input_grad[1] else None
        sink = ops._sink_candidate(ctx.w, ctx.next_functions[1][0]) if dw is not None else None
        ToyLinearFn.sunk.append(sink is not None)
        if sink is not None:
            sink.add_(dw)
            dw = None
        return (dy * w if ctx.needs_input_grad[0] else None), dw


def _setup(flat=True):
    """x, w with w re-homed as optim.FlatParams does: data and .grad views of flat buffers, .grad pre-filled with R."""
    g = torch.Generator().manual_seed(0)
    x = torch.randn(6, generator=g).requires_grad_(True)
    w = torch.randn(6, generator=g).requires_grad_(True)
    if flat:
        buf = torch.zeros(10)
        w.grad = buf[2:8]
        w.grad.copy_(torch.randn(6, generator=g))
        w._b200_flat_grad = True
    dy = torch.randn(6, generator=g)
    ToyLinearFn.sunk = []
    return x, w, dy


def _run(x, w, dy, how, **kw):
    y = ToyLinearFn.apply(x, w)
    if how == "backward":
        y.backward(dy, **kw)
        return None
    return torch.autograd.grad(y, kw["inputs"], dy)


def test_plain_backward_sinks_into_the_flat_grad():
    x, w, dy = _setup()
    r, view = w.grad.clone(), w.grad
    _run(x, w, dy, "backward")
    assert ToyLinearFn.sunk == [True]
    assert w.grad is view and torch.equal(w.grad, r + dy * x.detach())
    assert torch.equal(x.grad, dy * w.detach())


def test_backward_inputs_with_the_parameter_sinks():
    x, w, dy = _setup()
    r = w.grad.clone()
    _run(x, w, dy, "backward", inputs=[w])
    assert ToyLinearFn.sunk == [True]
    assert torch.equal(w.grad, r + dy * x.detach()) and x.grad is None


def test_backward_inputs_without_the_parameter_leaves_its_grad():
    x, w, dy = _setup()
    r = w.grad.clone()
    _run(x, w, dy, "backward", inputs=[x])
    assert ToyLinearFn.sunk == [False]
    assert torch.equal(w.grad, r)
    assert torch.equal(x.grad, dy * w.detach())


@pytest.mark.parametrize("wrt", ["w", "x", "both"])
def test_autograd_grad_never_touches_grad(wrt):
    x, w, dy = _setup()
    r = w.grad.clone()
    inputs = {"w": [w], "x": [x], "both": [x, w]}[wrt]
    got = _run(x, w, dy, "grad", inputs=inputs)
    assert ToyLinearFn.sunk == [False]
    assert torch.equal(w.grad, r) and x.grad is None
    want = {"w": [dy * x.detach()], "x": [dy * w.detach()], "both": [dy * w.detach(), dy * x.detach()]}[wrt]
    assert len(got) == len(want) and all(torch.equal(a, b) for a, b in zip(got, want))


def test_frozen_parameter_is_not_sunk():
    """Frozen between forward and backward: the node still asks for the gradient (needs_input_grad is fixed at the forward),
    the rule reads requires_grad itself, and autograd's AccumulateGrad skips a parameter that no longer requires grad."""
    x, w, dy = _setup()
    r = w.grad.clone()
    y = ToyLinearFn.apply(x, w)
    w.requires_grad_(False)
    y.backward(dy)
    assert ToyLinearFn.sunk == [False]
    assert torch.equal(w.grad, r) and torch.equal(x.grad, dy * w)


def test_tensor_hook_sees_the_gradient():
    x, w, dy = _setup()
    r = w.grad.clone()
    w.register_hook(lambda g: 2 * g)
    _run(x, w, dy, "backward")
    assert ToyLinearFn.sunk == [False]
    assert torch.equal(w.grad, r + 2 * (dy * x.detach()))


def test_post_accumulate_hook_fires_once_after_the_add():
    x, w, dy = _setup()
    r = w.grad.clone()
    seen = []
    w.register_post_accumulate_grad_hook(lambda p: seen.append(p.grad.clone()))
    _run(x, w, dy, "backward")
    assert ToyLinearFn.sunk == [False]
    assert len(seen) == 1 and torch.equal(seen[0], r + dy * x.detach()) and torch.equal(w.grad, seen[0])


def test_parameters_without_flat_grad_are_never_sunk():
    x, w, dy = _setup(flat=False)
    _run(x, w, dy, "backward")
    assert ToyLinearFn.sunk == [False] and torch.equal(w.grad, dy * x.detach())


def test_outside_a_backward_the_engine_does_not_accumulate():
    _, w, _ = _setup()
    assert not ops._engine_accumulates(w, torch.autograd.graph.get_gradient_edge(w).node)


def test_private_engine_query_behaves_as_the_gate_assumes():
    """torch._C._will_engine_execute_node: True for an AccumulateGrad node the running backward executes, False for one it
    skips, RuntimeError for a leaf among autograd.grad's inputs."""
    x = torch.randn(3, requires_grad=True)
    w = torch.randn(3, requires_grad=True)
    seen = {}

    class Probe(torch.autograd.Function):
        @staticmethod
        def forward(ctx, a, b):
            return a * b

        @staticmethod
        def backward(ctx, g):
            for name, t in (("x", x), ("w", w)):
                try:
                    seen[name] = torch._C._will_engine_execute_node(torch.autograd.graph.get_gradient_edge(t).node)
                except RuntimeError:
                    seen[name] = "raise"
            return g, g

    Probe.apply(x, w).sum().backward()
    assert seen == {"x": True, "w": True}
    Probe.apply(x, w).sum().backward(inputs=[x])
    assert seen == {"x": True, "w": False}
    torch.autograd.grad(Probe.apply(x, w).sum(), [w])
    assert seen == {"x": False, "w": "raise"}


def test_retained_graph_backward_twice_then_error():
    x, w, dy = _setup()
    r = w.grad.clone()
    y = ToyLinearFn.apply(x, w)
    y.backward(dy, retain_graph=True)
    y.backward(dy)
    assert torch.equal(w.grad, r + dy * x.detach() + dy * x.detach())
    with pytest.raises(RuntimeError, match="backward through the graph a second time"):
        y.backward(dy)


@pytest.mark.filterwarnings("ignore:Using backward\\(\\) with create_graph=True")
def test_create_graph_is_refused():
    x, w, dy = _setup(flat=False)
    with pytest.raises(RuntimeError, match="create_graph=True is not supported"):
        torch.autograd.grad(ToyLinearFn.apply(x, w), [x], dy, create_graph=True)
    with pytest.raises(RuntimeError, match="create_graph=True is not supported"):
        ToyLinearFn.apply(x, w).backward(dy, create_graph=True)


def test_every_autograd_function_is_in_the_gpu_sweep():
    """tests/test_gpu_autograd_routing.py runs retained-graph, third-backward and create_graph checks over SWEEP; a Function
    added to ops.py without an entry there fails here.  Every backward also carries ops._backward."""
    from tests import test_gpu_autograd_routing as R
    fns = {name for name, obj in vars(ops).items()
           if inspect.isclass(obj) and issubclass(obj, torch.autograd.Function) and obj.__module__ == ops.__name__}
    assert fns == set(R.SWEEP), (sorted(fns - set(R.SWEEP)), sorted(set(R.SWEEP) - fns))
    wrapper_code = ops._backward(lambda ctx, g: g).__code__
    for name in fns:
        assert inspect.getattr_static(getattr(ops, name), "backward").__func__.__code__ is wrapper_code, name
