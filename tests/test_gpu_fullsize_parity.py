"""Oracle parity at the TRUE BASELINE.json shapes (driver-run, -m gpu): the CUDA path against the CPU oracle in fp64 (the
"truth") and fp32 (the reference's own arithmetic) on the same seeded, ragged inputs, at the real dims of

  cfg2  4L/8H/d512/d_ff 2048/vgg_cnn/V=4364, T_src=800, T_tgt=100     (B=4 of the 32)
  cfg3  6L/8H/d512 dk=dv=32/emb_cnn/V=4364, T_src=400, T_tgt=100      (B=4 of the 64; BatchNorm statistics over this batch)
  cfg4  6L/8H/d512/vgg_cnn/V=4364, T_src=1000, T_tgt=150              (B=2 of the 32 per GPU)
  cfg5  12L/8H/d768/d_ff 3072/vgg_cnn/V=32, T_src=1600, T_tgt=150     (B=1 of the 16 per GPU)

Batch is the only reduced quantity (utterances are independent, SURVEY.md 8e): every kernel sees its real row lengths, head
dims, tile counts along T/F/d and the real vocabulary.  Bars (north_star: "within 1e-3 relative fp32"): pred max-norm,
loss, argmax ids bit-exact wherever the fp64 top-2 margin exceeds twice the measured logit error (ties at random init are
not decidable by any fp32 implementation, the reference included), and EVERY gradient tensor in the MAX norm
(tests/helpers.py::grads_rel_err, floor for mathematically-zero tensors).

Gradients and the model's discontinuities.  The path has ~1.3e8 ReLU units and max-pool windows at these sizes; a unit
whose pre-activation is within rounding (1e-6 .. 1e-5 of the layer's scale) of its threshold decides differently under two
correct arithmetics, and then its whole O(1) gradient contribution moves (measured at cfg2, B=4: ~150 such units, 2e-3
median / 3e-2 max gradient difference -- the fp32 oracle against the fp64 one shows the same effect at its own noise
level).  The test therefore (1) reads the CUDA path's own decisions (active ReLU / Hardtanh units, pooling winners) from
the activations its kernels produced, (2) counts the decisions that differ from the fp64 oracle's and checks that every
one of them is a threshold case (|fp64 pre-activation| < 1e-4 of the layer's largest) and that they are a < 1e-5 minority,
and (3) compares the gradients in the max norm with the fp64 oracle evaluated AT THOSE DECISIONS (oracle.Decisions), where
the function is smooth: measured 5e-5 (3xTF32) / 7e-5 (bf16x3) / 4e-5 (fp32 kernels) against the 1e-3 bar.
"""
import time

import pytest
import torch

from oracle import asr_oracle as O
from tests.helpers import grads_rel_err, rel_err

pytestmark = pytest.mark.gpu

TOL = 1e-3

CASES = {
    # name: (BASELINE config key, batch, oracle fp64 too)
    "cfg2": ("cfg2", 4),
    "cfg3": ("cfg3", 4),
    "cfg4": ("cfg4", 2),
    "cfg5": ("cfg5", 1),
}


def _oracle_cfg(c):
    return O.OracleConfig(num_layers=c.num_layers, num_heads=c.num_heads, dim_model=c.dim_model, dim_key=c.dim_key,
                          dim_value=c.dim_value, dim_inner=c.dim_inner, vocab=c.vocab, feat_extractor=c.feat_extractor,
                          tgt_max_len=c.tgt_max_len, freq=c.freq)


_cache = {}


def _truth(name):
    """fp64 and fp32 oracle results for a case (computed once per session; ~10 s of CPU work each)."""
    if name in _cache:
        return _cache[name]
    import b200asr
    key, B = CASES[name]
    spec = b200asr.BASELINE_CONFIGS[key]
    ocfg = _oracle_cfg(spec["cfg"])
    P = O.init_params(ocfg, seed=123456)
    g = torch.Generator().manual_seed(5)
    for k, v in P.items():            # norm / bias parameters away from (1, 0) so that their use and gradients are exercised
        if v.dim() == 1:
            v.add_(0.1 * torch.randn(v.shape, generator=g))
    src, lens, tgt = O.synthetic_batch(ocfg, B, spec["t_src"], seed=0, ragged=True)
    torch.set_num_threads(max(torch.get_num_threads(), 16))
    t0 = time.time()
    rec = O.Decisions()
    r64 = O.forward_backward({k: v.double() for k, v in P.items()}, ocfg, src.double(), lens, tgt, 0.1, dec=rec)
    r32 = O.forward_backward(P, ocfg, src, lens, tgt, 0.1)
    print(f"[{name}] oracle fp64+fp32 on the host: {time.time() - t0:.1f} s")
    _cache[name] = (ocfg, P, src, lens, tgt, r64, r32, rec)
    return _cache[name]


def _check(name, precision=None, tol=TOL, tol_grad=TOL, fp32_grade=True):
    import importlib
    import b200asr
    from tests.gpu_util import cuda_model, cuda_step_with_decisions
    ops = importlib.import_module(b200asr.__name__ + ".ops")
    ocfg, P, src, lens, tgt, r64, r32, rec = _truth(name)
    pred64, gold, hyp64, loss64, n_word, grads64 = r64
    pred32, _, hyp32, loss32, _, grads32 = r32
    g64 = {k: v.float() for k, v in grads64.items()}
    old = (ops.config.linear, ops.config.conv, ops.config.attn, ops.config.conv_wgrad, ops.config.attn_bwd)
    try:
        if precision is not None:
            ops.config.set(**precision)
        model = cuda_model(ocfg, P)
        (pred, gold_g, hyp, loss, stats, grads), masks = cuda_step_with_decisions(model, src, lens, tgt, 0.1)
    finally:
        ops.config.linear, ops.config.conv, ops.config.attn, ops.config.conv_wgrad, ops.config.attn_bwd = old
    assert torch.equal(gold_g, gold)
    e_pred = rel_err(pred, pred64)
    e_loss = abs(loss.item() - loss64.item()) / abs(loss64.item())
    # (2) decisions that differ from the fp64 oracle's own: count them, and check each one is a threshold case
    assert set(masks) == set(rec.masks), (sorted(masks), sorted(rec.masks))
    n_flip = n_units = 0
    worst_band = 0.0
    for site in masks:
        diff = masks[site] != rec.masks[site]
        n_units += diff.numel()
        nd = int(diff.sum())
        if nd:
            n_flip += nd
            worst_band = max(worst_band, float(rec.pre[site][diff].abs().max() / rec.pre[site].abs().max()))
    # (3) the fp64 oracle evaluated at the path's own decisions: smooth in the inputs, so the max norm is meaningful
    t0 = time.time()
    r64f = O.forward_backward({k: v.double() for k, v in P.items()}, ocfg, src.double(), lens, tgt, 0.1, dec=O.Decisions(frozen=masks))
    g64f = {k: v.float() for k, v in r64f[5].items()}
    errs = grads_rel_err(grads, g64f)
    # structurally zero gradients (a conv bias in front of BatchNorm, the key biases: the loss does not depend on them) are
    # sums of O(1e6) cancelling terms -- pure rounding noise in ANY arithmetic (fp32 oracle: 2.5e-3 of the 1e-3 * gmax floor);
    # bound them absolutely, at 1e-5 of the largest gradient in the model, instead of relative to the floor
    gmax = max(float(v.abs().max()) for v in g64f.values())
    for k, r in g64f.items():
        if float(r.abs().max()) < 1e-6 * gmax:
            assert float((grads[k].double() - r.double()).abs().max()) < 1e-5 * gmax, k
            errs[k] = 0.0
    worst = max(errs, key=errs.get)
    med = sorted(errs.values())[len(errs) // 2]
    errs_unfrozen = grads_rel_err(grads, g64)
    ref_errs = grads_rel_err(grads32, g64)            # what the reference's own fp32 arithmetic does against fp64 (its own flips included)
    ref_worst = max(ref_errs, key=ref_errs.get)
    real = gold.ne(O.PAD)
    # argmax: decidable positions = fp64 top-2 margin > 2 x the measured absolute logit error
    top2 = pred64.topk(2, dim=2).values
    margin = (top2[..., 0] - top2[..., 1])
    abs_err = (pred.double() - pred64).abs().max().item()
    decidable = real & (margin > 2 * abs_err)
    flips_all = int((hyp[real] != hyp64[real]).sum())
    flips_dec = int((hyp[decidable] != hyp64[decidable]).sum())
    print(f"[{name}] pred {e_pred:.2e} (fp32 oracle {rel_err(pred32, pred64):.2e})  loss {e_loss:.2e}  "
          f"argmax flips {flips_all}/{int(real.sum())} (decidable {flips_dec}/{int(decidable.sum())})  n_word {n_word}\n"
          f"[{name}] decisions: {n_flip} of {n_units} differ from the fp64 oracle's (largest |pre-activation| / layer max among them {worst_band:.1e})\n"
          f"[{name}] grads vs fp64 oracle AT THE PATH'S DECISIONS: max {errs[worst]:.2e} ({worst}) median {med:.2e}   "
          f"[unfrozen: max {max(errs_unfrozen.values()):.2e} median {sorted(errs_unfrozen.values())[len(errs) // 2]:.2e}; "
          f"fp32 oracle vs fp64, unfrozen: max {ref_errs[ref_worst]:.2e}]  (frozen oracle run {time.time() - t0:.1f} s)")
    assert int(stats[1]) == n_word
    assert e_pred < tol, e_pred
    assert e_loss < tol, e_loss
    assert flips_dec == 0
    if fp32_grade:
        assert float(decidable.float().sum() / real.float().sum()) > 0.97   # the tie band stays a small minority
        assert n_flip <= 1e-5 * n_units, (n_flip, n_units)                  # differing decisions: a vanishing minority ...
        assert worst_band < 1e-4, worst_band                                # ... and every one a unit sitting on its threshold
    assert errs[worst] < tol_grad, (worst, errs[worst])                     # every gradient tensor, max norm
    return e_pred, errs


@pytest.mark.parametrize("name", ["cfg2", "cfg3", "cfg4", "cfg5"])
def test_oracle_parity_at_true_baseline_dims(name):
    _check(name)


@pytest.mark.parametrize("name", ["cfg2", "cfg4"])
def test_oracle_parity_3xtf32_everywhere(name):
    """The 3xTF32 split for every contraction (the package default uses the bf16x3 split for the linear
    and convolution forward / data gradient)."""
    _check(name, dict(linear="tf32x3", conv="tf32x3", conv_wgrad="tf32x3", attn="tf32x3"))


def test_cfg5_in_bf16_as_baseline_json_asks():
    """BASELINE.json configs[4] is quoted in bf16: one bf16 MMA per product (bf16 operands, fp32 accumulate, fp32 master
    weights and activations in HBM) for every linear / convolution GEMM incl. the weight gradients, single-pass TF32 flash
    attention.  Tolerance stated separately, as SURVEY.md 8d asks -- bf16 cannot meet 1e-3: bars 3e-2 (logits) / 3e-2
    (loss) / 6e-2 (gradients, max norm, at the path's own decisions)."""
    _check("cfg5", dict(linear="bf16", conv="bf16", conv_wgrad="bf16", attn="tf32", attn_bwd="tf32"), tol=3e-2, tol_grad=6e-2,
           fp32_grade=False)


def test_oracle_parity_cfg2_exact_fp32_kernels():
    """The CUDA-core fp32 build of the same path (precision 0 everywhere): the reference's own arithmetic grade."""
    _check("cfg2", dict(linear="fp32", conv="fp32", attn="fp32", conv_wgrad="fp32", attn_bwd="fp32"))
