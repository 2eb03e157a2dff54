"""The UNMODIFIED reference on the GPU, with and without `b200asr.install()` (SURVEY.md 8b: the drop-in boundary on hardware).

The reference checkout travels to the GPU box as oracle/_ref (staged by oracle/make_ref.py, git-ignored).  Here
  * `init_transformer_model` (utils/functions.py:116-152) builds the reference's own `Transformer`;
  * the SAME weights run (i) on the CPU, uninstalled -- the reference's own PyTorch forward/backward, (ii) on the GPU,
    uninstalled -- the reference eager on the GPU (fp32 flags), (iii) on the GPU after `install()` -- our kernels bound onto
    the reference's classes; pred / loss / num_correct / every gradient are compared;
  * the reference's `Trainer.train` loop (trainer/asr/trainer.py:20-211) is driven unchanged for an epoch (train iterations
    with `opt.step()` of the reference's NoamOpt + torch Adam, the eval-mode validation loop, the checkpoint save) with
    synthetic `_collate_fn`-shaped batches, once on the reference eager and once installed: losses, updated parameters and
    BatchNorm buffers must agree.
"""
import copy
import os
import importlib
import tempfile

import pytest
import torch

from oracle import ref_shim
from tests.helpers import grads_rel_err, rel_err

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not ref_shim.available(), reason="reference checkout not staged (oracle/make_ref.py)")]

TOL = 1e-3

SMALL_VGG = ["--num-layers", "2", "--num-heads", "2", "--dim-model", "64", "--dim-emb", "64", "--dim-key", "32", "--dim-value", "32",
             "--dim-inner", "128", "--feat_extractor", "vgg_cnn", "--sample-rate", "4000", "--tgt-max-len", "12"]
SMALL_EMB = ["--num-layers", "1", "--num-heads", "2", "--dim-model", "64", "--dim-emb", "64", "--dim-key", "32", "--dim-value", "32",
             "--dim-inner", "128", "--feat_extractor", "emb_cnn", "--tgt-max-len", "10"]
CFG2_ARCH = ["--num-layers", "4", "--num-heads", "8", "--dim-model", "512", "--dim-emb", "512", "--dim-key", "64", "--dim-value", "64",
             "--dim-inner", "2048", "--feat_extractor", "vgg_cnn", "--tgt-max-len", "40"]


def _fp32_flags():
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    # the reference eager on ATen's native convolution: cuDNN's transform-based algorithms return rounding noise where a
    # weight gradient is exactly zero, and Adam turns that noise into full-size steps (two cuDNN algorithm choices alone
    # then differ by more than the trainer test's bound)
    torch.backends.cudnn.enabled = False


def _build(flags, vocab, extra=()):
    ns = ref_shim.load(list(flags) + ["--dropout", "0.0", "--label-smoothing", "0.1"] + list(extra))
    l2i, i2l = ref_shim.labels(vocab)
    torch.manual_seed(123456)
    model = ns.functions.init_transformer_model(ns.constant.args, l2i, i2l)
    g = torch.Generator().manual_seed(7)
    with torch.no_grad():
        for p in model.parameters():
            if p.dim() == 1:
                p.add_(0.1 * torch.randn(p.shape, generator=g))
    return ns, model, l2i, i2l


def _batch(B, freq, T, vocab, Lt, seed=0, ragged=True):
    g = torch.Generator().manual_seed(seed)
    src = torch.randn(B, 1, freq, T, generator=g)
    lens = (T * (0.5 + 0.5 * torch.rand(B, generator=g))).long().clamp(1, T) if ragged else torch.full((B,), T)
    lens[0] = T
    lens = torch.sort(lens, descending=True).values
    for i in range(B):
        src[i, :, :, int(lens[i]):] = 0
    tgt = torch.randint(3, vocab, (B, Lt), generator=g)
    tl = (Lt * (0.4 + 0.6 * torch.rand(B, generator=g))).long().clamp(1, Lt)
    tl[0] = Lt
    for i in range(B):
        tgt[i, int(tl[i]):] = 0
    return src, lens.to(torch.int32), tgt, tl.to(torch.int32)


def _region(kind, t):
    """The branch every unit took: ReLU 0 / 1 (from the post-activation value), Hardtanh(0, 20) 0 / 1 / 2."""
    t = t.detach().float().cpu()
    return (t > 0).to(torch.int8) + ((t >= 20).to(torch.int8) if kind == "hardtanh" else 0)


class _RefDecisions:
    """Forward hooks on the UNMODIFIED reference: the branch taken by every Hardtanh / ReLU unit of the CNN front end and by
    every ReLU of the position-wise FFNs (F.relu there: hooked through conv_1's output), in execution order -- the order in
    which ops.decision_capture lists the same units of our path (its max-pool entries have no counterpart here)."""

    def __init__(self, model):
        self.out, self.handles = [], []
        for m in model.modules():
            if isinstance(m, torch.nn.Hardtanh):
                self.handles.append(m.register_forward_hook(lambda _m, _i, o: self.out.append(_region("hardtanh", o))))
            elif isinstance(m, torch.nn.ReLU):
                self.handles.append(m.register_forward_hook(lambda _m, _i, o: self.out.append(_region("relu", o))))
            elif type(m).__name__ == "PositionwiseFeedForwardWithConv":      # conv_1 output is [B, d_inner, T]
                self.handles.append(m.conv_1.register_forward_hook(lambda _m, _i, o: self.out.append(_region("relu", o.transpose(1, 2)))))

    def close(self):
        for h in self.handles:
            h.remove()
        return self.out


def _count_flips(ref, ours):
    """(# units whose branch differs, # units); None if the two lists do not describe the same units."""
    ours = [_region(k, t) for k, t in ours if k != "pool"]
    if len(ours) != len(ref) or any(a.shape != b.shape for a, b in zip(ours, ref)):
        return None
    return sum(int((a != b).sum()) for a, b in zip(ours, ref)), sum(a.numel() for a in ref)


def _step(ns, model, src, lens, tgt, dev, decisions=None):
    """One forward / loss / backward through the reference's own code.  decisions: "hooks" records the branch decisions of the
    (uninstalled) reference, "capture" those of our kernels; they are returned as the seventh element."""
    import b200asr
    ops = importlib.import_module(b200asr.__name__ + ".ops")
    model.zero_grad(set_to_none=True)
    rec = _RefDecisions(model) if decisions == "hooks" else None
    if decisions == "capture":
        ops.decision_capture = []
    try:
        pred, gold, hyp, _ = model(src.to(dev), lens, tgt.to(dev), verbose=False)
    finally:
        dec = rec.close() if rec else ops.decision_capture
        ops.decision_capture = None
    loss, n_correct = ns.metrics.calculate_metrics(pred, gold, smoothing=0.1, loss_type="ce")
    loss.backward()
    grads = {n: p.grad.detach().float().cpu() for n, p in model.named_parameters()}
    return pred.detach().float().cpu(), gold.cpu(), hyp.cpu(), float(loss.item()), int(n_correct), grads, dec


@pytest.mark.parametrize("case", ["small_vgg", "small_emb", "cfg2_arch"])
def test_install_on_unmodified_reference_matches_reference_forward_backward(case):
    import b200asr
    flags, vocab, freq, B, T = {"small_vgg": (SMALL_VGG, 40, 41, 3, 32), "small_emb": (SMALL_EMB, 40, 161, 3, 48),
                                "cfg2_arch": (CFG2_ARCH, 4364, 161, 2, 200)}[case]
    ns, model, _, _ = _build(flags, vocab)
    src, lens, tgt, _ = _batch(B, freq, T, vocab, ns.constant.args.tgt_max_len - 1)
    keys = list(model.state_dict().keys())
    model.train()
    _fp32_flags()
    cpu = _step(ns, model, src, lens, tgt, "cpu", "hooks")              # (i) the reference's own CPU forward/backward
    model = model.cuda()
    eager = _step(ns, model, src, lens, tgt, "cuda", "hooks")           # (ii) the reference eager on the GPU
    orig_forward = ns.transformer.Transformer.forward
    b200asr.install()
    try:
        assert ns.transformer.Transformer.forward is not orig_forward
        launches0 = b200asr._lib.load().b200asr_launch_count()
        ours = _step(ns, model, src, lens, tgt, "cuda", "capture")      # (iii) our kernels behind the reference's classes
        assert b200asr._lib.load().b200asr_launch_count() > launches0   # ... and they did launch
    finally:
        b200asr.uninstall()
    assert ns.transformer.Transformer.forward is orig_forward
    assert list(model.state_dict().keys()) == keys                      # module tree / parameter names untouched
    for name, other in (("cpu", cpu), ("eager-gpu", eager)):
        assert torch.equal(ours[1], other[1]), name                     # gold
        e_pred = rel_err(ours[0], other[0])
        errs = grads_rel_err(ours[5], other[5])
        worst = max(errs, key=errs.get)
        real = other[1].ne(0)
        flips = int((ours[2][real] != other[2][real]).sum())
        print(f"[{case}] installed vs {name}: pred {e_pred:.2e} loss {abs(ours[3] - other[3]) / abs(other[3]):.2e} "
              f"grads max {errs[worst]:.2e} ({worst}) argmax flips {flips}/{int(real.sum())} num_correct {ours[4]} vs {other[4]}")
        assert e_pred < TOL
        assert abs(ours[3] - other[3]) < TOL * abs(other[3])
        # 1e5 .. 1e7 ReLU / max-pool units: a handful sit within rounding of their threshold and decide differently under two
        # correct arithmetics (the reference's CPU and GPU runs differ from each other the same way), which moves single
        # rows of the token-sparse decoder FFN gradients by O(1/sqrt(tokens)).  The strict max-norm check of EVERY gradient
        # at the path's own decisions lives in tests/test_gpu_fullsize_parity.py (the oracle there is pinned bit-exactly to
        # this reference, where decisions can be frozen); here: the median tensor in the max norm, every tensor in the
        # relative L2 norm.
        med = sorted(errs.values())[len(errs) // 2]
        unit_flips = _count_flips(other[6], ours[6])
        print(f"[{case}] installed vs {name}: ReLU / Hardtanh units that took another branch: {unit_flips}")
        assert unit_flips is not None, "decision lists of the reference hooks and of ops.decision_capture do not line up"
        # every unit on the same branch: tight bounds.  Otherwise (k of ~1e5 .. 1e7 units within rounding of their threshold):
        # a flipped FFN unit adds / removes one token's term in ITS row of that layer's weight gradient (relative L2 of the
        # tensor up to ~1/sqrt(d_inner)) and moves the gradients below it by O(1 / (tokens sqrt(d_inner))): bounded, not exact.
        same = unit_flips[0] == 0
        assert unit_flips[0] <= 2 + unit_flips[1] // 100000, (name, unit_flips)
        assert med < ((5 if case == "cfg2_arch" else 1) * TOL if same else 10 * TOL), (name, med, unit_flips)
        for k, r in other[5].items():
            denom = max(float(r.norm()), 1e-3 * max(float(v.abs().max()) for v in other[5].values()) * r.numel() ** 0.5)
            assert float((ours[5][k] - r).norm()) / denom < (10 * TOL if same else 0.2), (name, k, unit_flips)
        assert flips <= max(1, int(real.sum()) // 100)                  # near-ties at random init
        assert abs(ours[4] - other[4]) <= max(1, int(real.sum()) // 100)


def _loaders(freq, T, vocab, Lt, n_train, B):
    def one(seed):
        src, lens, tgt, tl = _batch(B, freq, T, vocab, Lt, seed=seed)
        return (src, tgt, lens.float() / float(T), lens, tl)            # _collate_fn order, utils/data_loader.py:213
    return [one(s) for s in range(n_train)], [[one(100)]]


def _run_trainer(ns, model, l2i, i2l, train, valid, installed, tmp):
    """Drive the reference's Trainer.train unchanged for one epoch; returns (per-iteration losses, state_dict)."""
    import b200asr
    ns.constant.args.save_folder, ns.constant.args.name = tmp, "b200" if installed else "eager"
    opt = ns.functions.init_optimizer(ns.constant.args, model, "noam")
    losses = []
    if installed:
        b200asr.install()
    cur = ns.trainer.calculate_metrics

    def recording(*a, **k):
        out = cur(*a, **k)
        losses.append(float(out[0].item()))
        return out

    ns.trainer.calculate_metrics = recording
    try:
        tr = copy.deepcopy(train), copy.deepcopy(valid)                 # the loop scales src_percentages in place (trainer.py:82)
        ns.trainer.Trainer().train(model, tr[0], None, tr[1], opt, "ce", 0, 1, l2i, i2l)
    finally:
        ns.trainer.calculate_metrics = cur
        if installed:
            b200asr.uninstall()
    assert os.path.exists(os.path.join(tmp, ns.constant.args.name, "best_model.th"))      # save_model ran (functions.py:10-57)
    return losses, {k: v.detach().float().cpu().clone() for k, v in model.state_dict().items()}


@pytest.mark.parametrize("case", ["small_vgg", "small_emb"])
def test_reference_trainer_loop_runs_on_installed_kernels(case):
    """trainer/asr/trainer.py:47-118 (train) and :123-190 (eval-mode validation) -- unchanged code, our kernels underneath.
    small_emb also checks the BatchNorm buffers (running_mean / running_var / num_batches_tracked) and the eval-mode
    forward that uses them."""
    flags, vocab, freq, B, T = {"small_vgg": (SMALL_VGG, 40, 41, 4, 32), "small_emb": (SMALL_EMB, 40, 161, 4, 48)}[case]
    _fp32_flags()
    results = {}
    with tempfile.TemporaryDirectory() as tmp:
        for installed in (False, True):
            ns, model, l2i, i2l = _build(flags, vocab, extra=["--cuda", "--warmup", "4", "--k-lr", "0.02", "--min-lr", "1e-6", "--clip", "--max-norm", "400"])
            init = {k: v.detach().float().clone() for k, v in model.state_dict().items()}
            if case == "small_emb":
                # a conv bias in front of BatchNorm is a gauge freedom: its true gradient is zero, Adam turns the rounding noise
                # into +-lr steps, and running_mean absorbs the resulting random walk.  Freeze it so the buffers are comparable.
                model.conv[0].bias.requires_grad_(False)
                model.conv[3].bias.requires_grad_(False)
            model = model.cuda()
            train, valid = _loaders(freq, T, vocab, ns.constant.args.tgt_max_len - 1, 3, B)
            results[installed] = _run_trainer(ns, model, l2i, i2l, train, valid, installed, tmp)
    (l_e, sd_e), (l_b, sd_b) = results[False], results[True]
    print(f"[{case}] losses eager {l_e}\n[{case}] losses b200  {l_b}")
    assert len(l_e) == len(l_b) == 4                                    # 3 train iterations + 1 validation batch
    for a, b in zip(l_e, l_b):
        assert abs(a - b) < TOL * abs(a), (l_e, l_b)
    for k in sd_e:
        if "num_batches_tracked" in k:
            assert sd_e[k].item() == sd_b[k].item() == 3, k
            continue
        if "running_" in k:
            assert rel_err(sd_b[k], sd_e[k]) < TOL, k
            continue
        if k.endswith("positional_encoding.pe"):
            continue
        d_e, d_b = sd_e[k] - init[k], sd_b[k] - init[k]
        if d_e.numel() < 256:
            continue                                                    # tiny tensors: Adam's sign-like first steps on noise-level gradients
        # Adam normalises the step, so an element whose gradient is rounding noise moves by +-lr either way: compare in L2
        assert float((d_e - d_b).norm() / d_e.norm().clamp_min(1e-30)) < (0.05 if d_e.numel() >= 16384 else 0.15), k
