"""The device Adam step (optim.adam_step, NoamOpt.step after install()) and gradient clip (optim.clip_grad_norm_) on the GPU.

  * Adam, bit for bit: the device step and torch.optim.Adam(foreach=True) on identical parameter lists, gradients and NoamOpt
    learning rates give identical parameters, exp_avg, exp_avg_sq and step after 1, 2, 10 and 1000 steps, for betas / eps
    (0.9, 0.98, 1e-9), torch's defaults and (0.3, 0.9, 1e-6) (ATen's other lerp branch).  The list has sizes 1, 3, 5, 7 and
    4k+1, views at float offsets 1-3 into larger storages, tensors across the kernel's chunk boundaries, more tensors than
    one parameter table holds, parameters that never get a gradient and ones that get one every other step (different step
    counts in one launch), and state tensors at a nonzero 16-byte phase; and, separately, the cfg2 model's parameter list.
  * Clip: the total norm against float64; grads == g * coef bit for bit; unchanged below max_norm; reproducible; the
    coefficient against torch.nn.utils.clip_grad_norm_'s.
  * No host synchronisation (torch sync debug mode "error") and a fixed number of launches per table, no memcpy.
  * Checkpoints: save_model after installed steps -> load_model uninstalled -> stock steps, and the reverse, both bit-identical
    to the run that never switched.
  * Optimizers the device step does not take run the reference's own NoamOpt.step: bit-identical to the uninstalled run.
"""
import importlib
import math
import os
import tempfile

import numpy as np
import pytest
import torch

import b200asr
from oracle import ref_shim

pytestmark = pytest.mark.gpu

OP = importlib.import_module(b200asr.__name__ + ".optim")
L = b200asr._lib
DEV = torch.device("cuda", 0)
CHUNK = 4096                       # OPT_CHUNK of csrc/optim.cu


def noam_rate(step, model_size=512, factor=1.0, warmup=25, min_lr=1e-5):
    """utils/optimizer.py:25-30"""
    return max(min_lr, factor * (model_size ** (-0.5) * min(step ** (-0.5), step * warmup ** (-1.5))))


def mixed_specs():
    """(shape, float offset of the view into its storage, gradient mode, state phase) per parameter."""
    specs = [((n,), 0, "always", 0) for n in (1, 3, 5, 7, 4 * 1024 + 1, 4 * 2047 + 1)]
    specs += [((n,), off, "always", 0) for n, off in ((5, 1), (4099, 2), (10001, 3), (3 * CHUNK + 2, 1))]
    specs += [((n,), 0, "always", 0) for n in (CHUNK - 1, CHUNK, CHUNK + 1, 3 * CHUNK + 5, (1 << 20) + 3)]
    specs += [((64, 33), 0, "always", 0), ((7, 5), 2, "always", 0)]
    specs += [((100,), 0, "never", 0), ((4101,), 1, "never", 0)]
    specs += [((300,), 0, "even", 0), ((CHUNK + 7,), 3, "even", 0)]
    specs += [((4101,), 1, "always", 1), ((9000,), 2, "always", 2)]          # state views at the parameter's phase
    g = np.random.default_rng(5)
    specs += [((int(n),), int(o), "always", 0) for n, o in zip(g.integers(1, 300, 560), g.integers(0, 4, 560))]
    return specs


def cfg2_specs():
    model = b200asr.build_model(b200asr.BASELINE_CONFIGS["cfg2"]["cfg"])
    return [(tuple(p.shape), 0, "always", 0) for p in model.parameters()]


class Arm:
    """One copy of a parameter list: parameters and gradients are views into two flat storages, so that one copy per step
    gives every arm the same gradients."""

    def __init__(self, specs, seed=0):
        self.specs = specs
        self.offsets, off = [], 0
        for shape, o, _, _ in specs:
            self.offsets.append(off + o)
            off += (math.prod(shape) + o + 3) // 4 * 4 + 4
        self.total = off
        gen = torch.Generator(device=DEV).manual_seed(seed)
        self.pstore = torch.randn(off, device=DEV, generator=gen)
        self.gstore = torch.zeros(off, device=DEV)
        self.sstore = torch.zeros(2, off, device=DEV)
        self.params = [torch.nn.Parameter(self.pstore[o:o + math.prod(s)].view(s)) for (s, _, _, _), o in zip(specs, self.offsets)]

    def grads(self, step, scale=1e-2):
        gen = torch.Generator(device=DEV).manual_seed(1000 + step)
        self.gstore.copy_(torch.randn(self.total, device=DEV, generator=gen) * scale)
        self.gstore[::7] = 0
        for p, (s, _, mode, _), o in zip(self.params, self.specs, self.offsets):
            on = mode == "always" or (mode == "even" and step % 2 == 0)
            p.grad = self.gstore[o:o + math.prod(s)].view(s) if on else None

    def seed_state(self, opt):
        """Pre-made state (as load_state_dict would leave it) for the entries with a state phase: views of sstore at the
        parameter's 16-byte phase, so that the kernel's head / float4 / tail path runs with a nonzero phase."""
        for p, (s, _, _, ph), o in zip(self.params, self.specs, self.offsets):
            if ph:
                n = math.prod(s)
                opt.state[p] = {"step": torch.tensor(0.0), "exp_avg": self.sstore[0, o:o + n].view(s),
                                "exp_avg_sq": self.sstore[1, o:o + n].view(s)}


def assert_same_adam(a, b, oa, ob, what):
    for k, (p, q) in enumerate(zip(a.params, b.params)):
        assert torch.equal(p, q), (what, k, a.specs[k])
        assert (p in oa.state) == (q in ob.state), (what, k)
        if p in oa.state:
            sa, sb = oa.state[p], ob.state[q]
            assert torch.equal(sa["exp_avg"], sb["exp_avg"]), (what, k, "exp_avg")
            assert torch.equal(sa["exp_avg_sq"], sb["exp_avg_sq"]), (what, k, "exp_avg_sq")
            assert sa["step"].dtype == sb["step"].dtype and float(sa["step"]) == float(sb["step"]), (what, k, "step")


def run_pair(specs, betas, eps, checks):
    ref, dev = Arm(specs), Arm(specs)
    o_ref = torch.optim.Adam(ref.params, betas=betas, eps=eps, foreach=True)
    o_dev = torch.optim.Adam(dev.params, betas=betas, eps=eps)
    ref.seed_state(o_ref)
    dev.seed_state(o_dev)
    for step in range(1, max(checks) + 1):
        lr = noam_rate(step)
        ref.grads(step)
        dev.grads(step)
        assert OP.adam_eligible(o_dev)
        o_ref.param_groups[0]["lr"] = o_dev.param_groups[0]["lr"] = lr
        o_ref.step()
        OP.adam_step(o_dev)
        if step in checks:
            assert_same_adam(ref, dev, o_ref, o_dev, f"step {step}")
    return ref, dev, o_ref, o_dev


@pytest.mark.parametrize("betas,eps", [((0.9, 0.98), 1e-9), ((0.9, 0.999), 1e-8), ((0.3, 0.9), 1e-6)])
def test_adam_matches_torch_foreach_bit_for_bit(betas, eps):
    specs = mixed_specs()
    assert len(specs) > L.load().b200asr_optim_table_capacity()
    ref, dev, o_ref, o_dev = run_pair(specs, betas, eps, (1, 2, 10, 1000))
    never = [p for p, s in zip(dev.params, specs) if s[2] == "never"]
    assert never and all(p not in o_dev.state for p in never)
    even = [p for p, s in zip(dev.params, specs) if s[2] == "even"]
    assert all(float(o_dev.state[p]["step"]) == 500.0 for p in even)
    assert float(o_dev.state[dev.params[0]]["step"]) == 1000.0


def test_adam_matches_torch_foreach_on_the_cfg2_parameter_list():
    specs = cfg2_specs()
    assert len(specs) > 100 and sum(math.prod(s) for s, *_ in specs) > 30_000_000
    run_pair(specs, (0.9, 0.98), 1e-9, (1, 2, 10))


def fp32_coef(total, max_norm):
    """clip_coef_kernel's arithmetic on the host: clamp(reciprocal(total + 1e-6) * max_norm, max=1) in fp32."""
    t = np.float32(total) + np.float32(1e-6)
    c = (np.float32(1) / np.float32(t)) * np.float32(max_norm)
    return np.float32(min(c, np.float32(1)))


@pytest.mark.parametrize("which", ["mixed", "cfg2"])
def test_clip_grad_norm(which):
    specs = mixed_specs() if which == "mixed" else cfg2_specs()
    arm = Arm(specs)
    arm.grads(3, scale=1.0)
    grads = [p.grad for p in arm.params if p.grad is not None]
    before = [g.clone() for g in grads]
    norm64 = math.sqrt(sum(float(g.double().pow(2).sum()) for g in before))
    max_norm = norm64 / 3
    total = b200asr.clip_grad_norm_(arm.params, max_norm)
    assert total.is_cuda and total.dim() == 0 and total.dtype == torch.float32
    t = float(total)
    assert abs(t - norm64) <= 1e-6 * norm64, (t, norm64)
    coef = fp32_coef(t, max_norm)
    assert coef < 1
    for g, g0 in zip(grads, before):
        assert torch.equal(g, g0 * torch.tensor(coef, device=DEV)), "grads == g * coef"
    # the same call again on the same input: the same bits
    arm2 = Arm(specs)
    arm2.grads(3, scale=1.0)
    total2 = b200asr.clip_grad_norm_(arm2.params, max_norm)
    assert torch.equal(total, total2) and torch.equal(arm.gstore, arm2.gstore)
    # below max_norm: coefficient 1, gradients unchanged
    arm3 = Arm(specs)
    arm3.grads(3, scale=1.0)
    keep = arm3.gstore.clone()
    b200asr.clip_grad_norm_(arm3.params, 2 * norm64)
    assert torch.equal(arm3.gstore, keep)
    # torch's clip on the same gradients: the sums run in another order, so the coefficients may differ in the last bits;
    # observed on the H100: 0 ulp on both lists
    arm4 = Arm(specs)
    arm4.grads(3, scale=1.0)
    t_torch = torch.nn.utils.clip_grad_norm_(arm4.params, max_norm)
    c_torch = torch.clamp(max_norm / (t_torch + 1e-6), max=1.0)
    ulp = abs(int(np.float32(coef).view(np.int32)) - int(np.float32(c_torch.item()).view(np.int32)))
    print(f"[{which}] total {t!r} float64 {norm64!r} torch {t_torch.item()!r}; coefficient differs from torch's by {ulp} ulp")
    assert ulp <= 1


def count_cuda(prof):
    """(kernel names, copy names) the profiler saw on the device after the marker kernel (torch.cuda._sleep), each event once:
    a profiler session can also report work that finished before it began."""
    evs = {(e.start_ns(), e.name()) for e in prof.profiler.kineto_results.events()
           if e.device_type() == torch.autograd.DeviceType.CUDA}
    mark = max(t for t, n in evs if "spin" in n.lower())
    evs = sorted((t, n) for t, n in evs if t > mark)
    copies = [n for _, n in evs if "memcpy" in n.lower()]
    kernels = [n for _, n in evs if "memcpy" not in n.lower() and "memset" not in n.lower()]
    return kernels, copies


@pytest.mark.parametrize("clip", [False, True])
def test_step_needs_no_sync_and_few_launches(clip):
    specs = mixed_specs()
    cap = L.load().b200asr_optim_table_capacity()
    arm = Arm(specs)
    opt = torch.optim.Adam(arm.params, betas=(0.9, 0.98), eps=1e-9)
    arm.grads(2)                                               # every parameter that ever gets a gradient has one
    OP.adam_step(opt)                                          # creates the state (a zeros_like launch per state tensor)
    OP.clip_grad_norm_(arm.params, 1.0)                        # sizes the library's scratch
    arm.grads(4)
    n_grads = sum(p.grad is not None for p in arm.params)
    tables = -(-n_grads // cap)
    torch.cuda.synchronize()
    launches0 = L.load().b200asr_launch_count()
    # a warm-up step whose events are discarded first: kernels launched while CUPTI starts tracing can go unrecorded
    seen = []
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA],
                                schedule=torch.profiler.schedule(wait=0, warmup=1, active=1, repeat=1),
                                on_trace_ready=lambda p: seen.append(count_cuda(p))) as prof:
        torch.cuda._sleep(1000)
        torch.cuda.synchronize()
        prof.step()
        torch.cuda._sleep(1000)                                 # marks where the step's work begins
        torch.cuda.set_sync_debug_mode("error")
        try:
            if clip:
                OP.clip_grad_norm_(arm.params, 1.0)
            opt.param_groups[0]["lr"] = noam_rate(4)
            OP.adam_step(opt)
        finally:
            torch.cuda.set_sync_debug_mode(0)
        torch.cuda.synchronize()
        prof.step()
    assert len(seen) == 1
    kernels, copies = seen[0]
    # per table: Adam 1 launch; clip 3 (sum of squares, per-tensor norms, scale); plus the clip coefficient once
    want = tables * (4 if clip else 1) + (1 if clip else 0)
    print(f"clip={clip}: {n_grads} tensors, {tables} tables, {len(kernels)} kernels, {len(copies)} copies")
    assert tables == 2
    assert L.load().b200asr_launch_count() - launches0 == want
    assert len(kernels) == want, [k.split("(")[0][-40:] for k in kernels]
    assert not copies, copies


# ---------------------------------------------------------------- the reference's NoamOpt, checkpoints and fallbacks

SMALL_VGG = ["--num-layers", "2", "--num-heads", "2", "--dim-model", "64", "--dim-emb", "64", "--dim-key", "32", "--dim-value", "32",
             "--dim-inner", "128", "--feat_extractor", "vgg_cnn", "--sample-rate", "4000", "--tgt-max-len", "12", "--cuda",
             "--warmup", "4", "--k-lr", "0.02", "--min-lr", "1e-6"]
needs_ref = pytest.mark.skipif(not ref_shim.available(), reason="reference checkout not staged (oracle/make_ref.py)")


def ref_model(ns, l2i, i2l):
    torch.manual_seed(123456)
    return ns.functions.init_transformer_model(ns.constant.args, l2i, i2l).cuda()


def set_grads(model, step):
    g = torch.Generator(device=DEV).manual_seed(77 + step)
    for p in model.parameters():
        p.grad = torch.randn(p.shape, device=DEV, generator=g) * 1e-2


def steps(model, opt, first, last):
    for s in range(first, last):
        set_grads(model, s)
        opt.step()


def snapshot(model, opt):
    params = [p.detach().clone() for p in model.parameters()]
    st = [{k: v.clone() for k, v in opt.optimizer.state[p].items()} for p in model.parameters()]
    return params, st, opt._step, opt._rate


def assert_same_snapshot(a, b, what):
    for k, (x, y) in enumerate(zip(a[0], b[0])):
        assert torch.equal(x, y), (what, "param", k)
    for k, (x, y) in enumerate(zip(a[1], b[1])):
        assert x.keys() == y.keys(), (what, k)
        for key in x:
            assert torch.equal(x[key], y[key]), (what, k, key)
    assert a[2:] == b[2:], what


@needs_ref
def test_checkpoint_round_trip_with_stock_torch(monkeypatch):
    monkeypatch.setenv("TORCH_FORCE_NO_WEIGHTS_ONLY_LOAD", "1")     # the reference's checkpoint holds argparse.Namespace
    ns = ref_shim.load(SMALL_VGG)
    l2i, i2l = ref_shim.labels(40)
    with tempfile.TemporaryDirectory() as tmp:
        ns.constant.args.save_folder = tmp
        # never switched: stock torch all the way
        model = ref_model(ns, l2i, i2l)
        opt = ns.functions.init_optimizer(ns.constant.args, model, "noam")
        steps(model, opt, 0, 8)
        stock = snapshot(model, opt)
        # never switched, installed all the way (the device step alone)
        model = ref_model(ns, l2i, i2l)
        opt = ns.functions.init_optimizer(ns.constant.args, model, "noam")
        b200asr.install()
        try:
            steps(model, opt, 0, 8)
        finally:
            b200asr.uninstall()
        assert_same_snapshot(snapshot(model, opt), stock, "installed throughout")
        for first_installed in (True, False):
            ns.constant.args.name = f"rt_{first_installed}"
            model = ref_model(ns, l2i, i2l)
            opt = ns.functions.init_optimizer(ns.constant.args, model, "noam")
            if first_installed:
                b200asr.install()
            try:
                steps(model, opt, 0, 4)
                ns.functions.save_model(model, 1, opt, {}, l2i, i2l, best_model=False)
            finally:
                b200asr.uninstall()
            if not first_installed:
                b200asr.install()
            try:
                model2, opt2, *_ = ns.functions.load_model(os.path.join(tmp, ns.constant.args.name, "epoch_1.th"))
                assert next(model2.parameters()).is_cuda and opt2._step == 4
                steps(model2, opt2, 4, 8)
            finally:
                b200asr.uninstall()
            assert_same_snapshot(snapshot(model2, opt2), stock, f"first_installed={first_installed}")


FALLBACKS = {
    "amsgrad": lambda ps: torch.optim.Adam(ps, betas=(0.9, 0.98), eps=1e-9, amsgrad=True),
    "weight_decay": lambda ps: torch.optim.Adam(ps, betas=(0.9, 0.98), eps=1e-9, weight_decay=0.01),
    "fused": lambda ps: torch.optim.Adam(ps, betas=(0.9, 0.98), eps=1e-9, fused=True),
    "cpu": lambda ps: torch.optim.Adam(ps, betas=(0.9, 0.98), eps=1e-9),
    "fp16": lambda ps: torch.optim.Adam(ps, betas=(0.9, 0.98), eps=1e-4),
    "two_groups": lambda ps: torch.optim.Adam([{"params": ps[:2]}, {"params": ps[2:]}], betas=(0.9, 0.98), eps=1e-9),
}


@needs_ref
@pytest.mark.parametrize("case", sorted(FALLBACKS))
def test_other_optimizers_run_the_reference_step(case):
    ns = ref_shim.load(SMALL_VGG)
    dev = torch.device("cpu") if case == "cpu" else DEV
    dtype = torch.float16 if case == "fp16" else torch.float32
    results = {}
    for installed in (False, True):
        g = torch.Generator().manual_seed(3)
        ps = [torch.nn.Parameter(torch.randn(n, generator=g).to(dev, dtype)) for n in (5, 64, 4097)]
        opt = ns.optimizer.NoamOpt(64, 0.02, 4, FALLBACKS[case](ps), min_lr=1e-6)
        if installed:
            b200asr.install()
        launches0 = L.load().b200asr_launch_count()
        try:
            for s in range(3):
                gg = torch.Generator().manual_seed(10 + s)
                for p in ps:
                    p.grad = torch.randn(p.shape, generator=gg).to(dev, dtype)
                opt.step()
        finally:
            if installed:
                b200asr.uninstall()
        assert L.load().b200asr_launch_count() == launches0
        results[installed] = [p.detach().clone() for p in ps], opt._step, opt._rate
    (a, sa, ra), (b, sb, rb) = results[False], results[True]
    assert sa == sb == 3 and ra == rb
    assert all(torch.equal(x, y) for x, y in zip(a, b))
