"""The LSTM LM's training loop on the device (end2end-asr-pytorch_b200/lm_train.py, `python -m b200asr.lm_train`).

  * b200asr_xent_fwd / _bwd (ops.XentFn, nn.CrossEntropyLoss's defaults) against float64 for rows 1, 7, 700, 4097 and
    V 1, 2, 33, 10 000, 50 000, each with a row pitch equal to V and, with logits shifted by +200, wider than V; outputs
    start NaN.  The row losses carry the bits of b200asr_lm_nll; out-of-range targets give NaN; repeated calls give the same
    bits; no host synchronisation; rejected calls launch nothing.
  * b200asr_sgd_multi (optim.sgd_step) bit-identical to `p.data.add_(p.grad, alpha=-lr)` over a list longer than one table
    (two launches), odd sizes and views at float offsets 1-3, compared over the whole shared storage.
  * The write extent of the three entry points (guard bands of tests/test_gpu_write_extent.py).
  * Five windows and the validation loss of the loop (dropout 0) against the same loop in float64 on the CPU, held to 50x
    the distance of the reference's RNNModel on cuDNN (fp32, no TF32) from it.  Training windows (dropout on) make no
    host synchronisation.
  * The CLI on a tiny synthetic corpus for 2 epochs: the checkpoint loads into the reference's LM and b200asr.LM,
    LM.evaluate agrees installed and on cuDNN, and the reference's beam search with LM rescoring returns the same strings
    installed and uninstalled.
Bars state the error measured on one H100 80GB HBM3 (700 W power limit).
"""
import importlib
import json
import runpy
import sys

import numpy as np
import pytest
import torch
import torch.nn as nn

import b200asr
from oracle import ref_shim
from tests import test_gpu_write_extent as _write_extent
from tests.test_gpu_optimizer_step import Arm, mixed_specs

# register the guard-band checks below with the ABI-wide sweep of tests/test_gpu_write_extent.py, which requires every
# pointer entry point to be covered or exempted
for _name in ("b200asr_xent_fwd", "b200asr_xent_bwd"):
    _write_extent.EXEMPT.setdefault(_name, "tests/test_gpu_lm_train.py: NaN-poisoned outputs with guard bands and guarded gap "
                                           "columns of a row pitch wider than V (test_xent_write_extent)")
_write_extent.EXEMPT.setdefault("b200asr_sgd_multi", "tests/test_gpu_lm_train.py: guard bands around every parameter, gradients "
                                                     "unchanged (test_sgd_multi_write_extent)")

pytestmark = pytest.mark.gpu

ops = importlib.import_module(b200asr.__name__ + ".ops")
OP = importlib.import_module(b200asr.__name__ + ".optim")
LT = b200asr.lm_train
L = b200asr._lib
Arena = _write_extent.Arena
DEV = "cuda"
NLL_RTOL = 2.5e-5       # row losses and the mean vs float64, relative to max(1, |value|): the lm_nll bar (measured 7.7e-6 max)
DX_TOL = 2e-6           # dlogits vs float64, relative to the largest possible entry g / rows (measured 6.1e-7 max)


def _lib():
    return L.load()


def _st():
    return torch.cuda.current_stream().cuda_stream


def _xent(xbuf, V, tg, dloss):
    """b200asr_xent_fwd then _bwd over logits xbuf[:, :V] (row pitch xbuf.stride(0)); outputs start NaN."""
    rows, ld = xbuf.shape
    nll, stats, loss = (torch.full(s, float("nan"), device=DEV) for s in ((rows,), (rows, 2), (1,)))
    dx = torch.full((rows, ld), float("nan"), device=DEV)
    P = L.ptr
    assert _lib().b200asr_xent_fwd(P(xbuf), ld, P(tg), P(nll), P(stats), P(loss), rows, V, _st()) == 0, L.last_error()
    assert _lib().b200asr_xent_bwd(P(xbuf), ld, P(tg), P(stats), P(dloss), P(dx), rows, V, _st()) == 0, L.last_error()
    return nll, stats, loss, dx


def _xent64(x, tg, g):
    """float64 nn.CrossEntropyLoss: (row losses, mean, dlogits) of fp32 logits x [rows, V]."""
    x64 = x.double()
    lse = torch.logsumexp(x64, 1)
    nll = lse - x64.gather(1, tg[:, None])[:, 0]
    d = torch.softmax(x64, 1)
    d[torch.arange(len(tg)), tg] -= 1.0
    return nll, nll.mean(), d * (g / len(tg))


@pytest.mark.parametrize("V", [1, 2, 33, 10000, 50000])
@pytest.mark.parametrize("rows", [1, 7, 700, 4097])
def test_xent_matches_float64(rows, V):
    gen = torch.Generator(device=DEV).manual_seed(rows * 7 + V)
    tg = torch.randint(0, V, (rows,), device=DEV, generator=gen)
    g = 0.75
    dloss = torch.tensor([g], device=DEV)
    errs = {}
    for pad, shift in ((0, 0.0), (5, 200.0)):
        ld = V + pad
        xbuf = torch.full((rows, ld), float("nan"), device=DEV)
        xbuf[:, :V] = 3.0 * torch.randn(rows, V, device=DEV, generator=gen) + shift
        x = xbuf[:, :V]
        nll, stats, loss, dx = _xent(xbuf, V, tg, dloss)
        n64, l64, d64 = _xent64(x, tg, g)
        e_nll = float(((nll.double() - n64).abs() / n64.abs().clamp_min(1.0)).max())
        e_loss = abs(float(loss) - float(l64)) / max(1.0, abs(float(l64)))
        e_dx = float((dx[:, :V].double() - d64).abs().max()) / (g / rows)
        errs[shift] = (e_nll, e_loss, e_dx)
        assert e_nll <= NLL_RTOL and e_loss <= NLL_RTOL and e_dx <= DX_TOL, (shift, e_nll, e_loss, e_dx)
        assert torch.isnan(dx[:, V:]).all()                                # the gap columns are not written
        assert torch.equal(nll, ops.lm_nll(x, tg))                         # the row code of lm_nll, bit for bit
        again = _xent(xbuf, V, tg, dloss)
        for a, b in zip((nll, stats, loss, dx), again):
            assert torch.equal(a.nan_to_num(), b.nan_to_num()) and torch.equal(a.isnan(), b.isnan())
    print(f"xent rows={rows} V={V}: (nll, loss, dlogits) errors {errs[0.0]} at shift 0, {errs[200.0]} at +200")


def test_xent_out_of_range_targets_give_nan():
    rows, V = 6, 33
    x = torch.randn(rows, V, device=DEV, generator=torch.Generator(device=DEV).manual_seed(3))
    tg = torch.tensor([0, -1, 5, 32, 33, 7], device=DEV)
    nll, _, loss, dx = _xent(x, V, tg, torch.ones(1, device=DEV))
    bad = torch.tensor([False, True, False, False, True, False], device=DEV)
    assert torch.isnan(nll[bad]).all() and torch.isfinite(nll[~bad]).all() and torch.isnan(loss).all()
    assert torch.isnan(dx[bad]).all() and torch.isfinite(dx[~bad]).all()
    assert torch.equal(nll.nan_to_num(), ops.lm_nll(x, tg).nan_to_num())


def test_xent_fn_matches_cross_entropy_without_host_sync():
    rows, V = 700, 10000
    gen = torch.Generator(device=DEV).manual_seed(5)
    x = (2.0 * torch.randn(rows, V, device=DEV, generator=gen)).requires_grad_(True)
    tg = torch.randint(0, V, (rows,), device=DEV, generator=gen)
    ops.XentFn.apply(x, tg).backward()                      # warm
    x.grad = None
    torch.cuda.synchronize()
    lib = _lib()
    n0 = lib.b200asr_launch_count()
    torch.cuda.set_sync_debug_mode("error")
    try:
        loss = ops.XentFn.apply(x, tg)
        n1 = lib.b200asr_launch_count()
        (2.0 * loss).backward()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert n1 - n0 == 2 and lib.b200asr_launch_count() - n1 == 1
    x64 = x.detach().double().requires_grad_(True)
    l64 = nn.CrossEntropyLoss()(x64, tg)
    (2.0 * l64).backward()
    assert abs(float(loss) - float(l64)) <= NLL_RTOL * float(l64)
    assert float((x.grad.double() - x64.grad).abs().max()) <= DX_TOL * 2.0 / rows
    for bad in (x.detach().double(), x.detach().cpu(), x.detach()[:, :0], x.detach().t()):
        with pytest.raises(ValueError):
            ops.XentFn.apply(bad, tg if bad.shape[0] == rows else tg[:bad.shape[0]])
    with pytest.raises(ValueError):
        ops.XentFn.apply(x, tg.int())


def test_xent_rejections_launch_nothing():
    lib, P = _lib(), L.ptr
    x = torch.randn(4, 5, device=DEV)
    tg = torch.zeros(4, dtype=torch.int64, device=DEV)
    outs = [torch.full(s, float("nan"), device=DEV) for s in ((4,), (4, 2), (1,), (4, 5), (1,))]
    nll, stats, loss, dx, dl = outs
    n0 = lib.b200asr_launch_count()
    for args, rc in (((P(x), 5, None, P(nll), P(stats), P(loss), 4, 5), -5), ((P(x), 5, P(tg), P(nll), P(stats), None, 4, 5), -5),
                     ((P(x), 4, P(tg), P(nll), P(stats), P(loss), 4, 5), -1), ((P(x), 5, P(tg), P(nll), P(stats), P(loss), 4, 0), -1),
                     ((P(x), 5, P(tg), P(nll), P(stats), P(loss), 0, 5), -1)):
        assert lib.b200asr_xent_fwd(*args, None) == rc and L.last_error().startswith("xent_fwd:")
    for args, rc in (((P(x), 5, P(tg), P(stats), None, P(dx), 4, 5), -5), ((P(x), 5, P(tg), P(stats), P(dl), P(dx), -1, 5), -1),
                     ((P(x), 3, P(tg), P(stats), P(dl), P(dx), 4, 5), -1)):
        assert lib.b200asr_xent_bwd(*args, None) == rc and L.last_error().startswith("xent_bwd:")
    ptrs, numel = np.zeros((1, 2), dtype=np.uint64), np.ones(1, dtype=np.int64)
    assert lib.b200asr_sgd_multi(ptrs.ctypes.data, numel.ctypes.data, 1, -1.0, None) == -5
    assert lib.b200asr_sgd_multi(ptrs.ctypes.data, numel.ctypes.data, 0, -1.0, None) == -1
    assert lib.b200asr_sgd_multi(None, None, 1, -1.0, None) == -5
    assert lib.b200asr_launch_count() == n0
    torch.cuda.synchronize()
    assert all(torch.isnan(t).all() for t in outs)


# ------------------------------------------------------------------------------------------ SGD
@pytest.mark.parametrize("lr", [20.0, 0.3, 1e-3 / 3])
def test_sgd_multi_matches_torch_add_bit_for_bit(lr):
    specs = mixed_specs()
    assert len(specs) > _lib().b200asr_optim_table_capacity()
    ref, dev = Arm(specs), Arm(specs)
    for step in range(1, 4):
        ref.grads(step, scale=1.0)
        dev.grads(step, scale=1.0)
        for p in ref.params:
            if p.grad is not None:
                p.data.add_(p.grad, alpha=-lr)
        OP.sgd_step(dev.params, lr)
        assert torch.equal(ref.pstore, dev.pstore), step          # the whole storage: views and the gaps between them
        assert torch.equal(ref.gstore, dev.gstore)


def test_sgd_step_needs_no_sync_and_one_launch_per_table():
    specs = mixed_specs()
    cap = _lib().b200asr_optim_table_capacity()
    arm = Arm(specs)
    arm.grads(2)
    OP.sgd_step(arm.params, 1.0)
    n_grads = sum(p.grad is not None for p in arm.params)
    tables = -(-n_grads // cap)
    v0 = [p._version for p in arm.params]
    torch.cuda.synchronize()
    launches0 = _lib().b200asr_launch_count()
    torch.cuda.set_sync_debug_mode("error")
    try:
        OP.sgd_step(arm.params, 0.5)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert tables == 2
    assert _lib().b200asr_launch_count() - launches0 == tables
    assert all(p._version > v for p, v in zip(arm.params, v0) if p.grad is not None)
    bad = [torch.nn.Parameter(torch.zeros(3, device=DEV, dtype=torch.float64))]
    bad[0].grad = torch.zeros_like(bad[0])
    with pytest.raises(ValueError):
        OP.sgd_step(bad, 1.0)


# ------------------------------------------------------------------------------------------ write extent
@pytest.mark.parametrize("shift", [0, 16])
@pytest.mark.parametrize("rows,V", [(1, 1), (1, 1000), (257, 33), (257, 1000)])
def test_xent_write_extent(rows, V, shift):
    lib = _lib()
    gen = torch.Generator().manual_seed(rows + V)
    X = (2.0 * torch.randn(rows, V, generator=gen)).cuda()
    T = torch.randint(0, V, (rows,), generator=gen).cuda()
    ld = V + 3
    a = Arena(lib, shift)
    x, tg = a.inp("logits", X, pitch=ld), a.inp("targets", T)
    nll, stats, loss = a.out("nll", (rows,)), a.out("stats", (rows, 2)), a.out("loss", (1,))
    a.call("xent_fwd", x, ld, tg, nll, stats, loss, rows, V)
    b = Arena(lib, shift)
    x2, tg2 = b.inp("logits", X, pitch=ld), b.inp("targets", T)
    st2, dl2 = b.inp("stats", stats.t.clone()), b.inp("dloss", torch.tensor([0.5], device=DEV))
    dx = b.out("dlogits", (rows, V), pitch=ld)
    b.call("xent_bwd", x2, ld, tg2, st2, dl2, dx, rows, V)
    n64, l64, d64 = _xent64(X, T, 0.5)
    assert float(((nll.t.double() - n64).abs() / n64.abs().clamp_min(1.0)).max()) <= NLL_RTOL
    assert abs(float(loss.t) - float(l64)) <= NLL_RTOL * max(1.0, abs(float(l64)))
    assert float((dx.t.double() - d64).abs().max()) <= DX_TOL * 0.5 / rows


@pytest.mark.parametrize("shift", [0, 16])
def test_sgd_multi_write_extent(shift):
    lib = _lib()
    sizes = [1, 3, 5, 4097, 3 * 4096 + 5]
    gen = torch.Generator().manual_seed(shift)
    a = Arena(lib, shift)
    Ps = [torch.randn(n, generator=gen).cuda() for n in sizes]
    Gs = [torch.randn(n, generator=gen).cuda() for n in sizes]
    ps = [a.inout(f"p{k}", P) for k, P in enumerate(Ps)]
    gs = [a.inp(f"g{k}", G) for k, G in enumerate(Gs)]
    ptrs = np.array([[p.ptr, g.ptr] for p, g in zip(ps, gs)], dtype=np.uint64)
    numel = np.array(sizes, dtype=np.int64)
    a.call("sgd_multi", ptrs.ctypes.data, numel.ctypes.data, len(sizes), -0.7)
    for p, P, G in zip(ps, Ps, Gs):
        assert torch.equal(p.t, P.clone().add_(G, alpha=-0.7))


# ------------------------------------------------------------------------------------------ the loop
FLAGS = ["--num-layers", "2", "--num-heads", "2", "--dim-model", "64", "--dim-emb", "64", "--dim-key", "32", "--dim-value", "32",
         "--dim-inner", "128", "--feat_extractor", "", "--tgt-max-len", "301", "--dropout", "0.0", "--cuda"]


def _reference():
    ref_shim.load(FLAGS, q12_shim=True)
    return importlib.import_module("utils.lstm_utils")


def _err(got, ref):
    ref = ref.detach().double().cpu()
    return float((got.detach().double().cpu() - ref).abs().max() / ref.abs().max().clamp_min(1e-30))


def _example_loop(model, train, val, ntoken, bptt, lr, clip):
    """The word-language-model example's epoch and evaluation on torch's own loss, clip and update."""
    model.train()
    hidden = model.init_hidden(train.size(1))
    crit = nn.CrossEntropyLoss()
    losses = []
    for i in range(0, train.size(0) - 1, bptt):
        x, y = LT.get_batch(train, i, bptt)
        model.zero_grad()
        hidden = LT.repackage_hidden(hidden)
        out, hidden = model(x, hidden)
        loss = crit(out.view(-1, ntoken), y)
        loss.backward()
        torch.nn.utils.clip_grad_norm_(model.parameters(), clip)
        for p in model.parameters():
            p.data.add_(p.grad, alpha=-lr)
        losses.append(loss.item())
    model.eval()
    hidden, total = model.init_hidden(val.size(1)), 0.0
    with torch.no_grad():
        for i in range(0, val.size(0) - 1, bptt):
            x, y = LT.get_batch(val, i, bptt)
            out, hidden = model(x, hidden)
            hidden = LT.repackage_hidden(hidden)
            total += len(x) * crit(out.view(-1, ntoken), y).item()
    return losses, {k: v.detach().cpu().double() for k, v in model.state_dict().items()}, total / (len(val) - 1)


@pytest.mark.skipif(not ref_shim.available(), reason="reference checkout not staged (oracle/make_ref.py)")
def test_five_windows_and_validation_within_cudnn_distance_of_float64():
    """Five windows (B = 20, bptt = 35, clip 0.25, SGD lr 20, dropout 0) and the validation loss (batch 10): lm_train's
    train_epoch / evaluate, the example's loop on the reference's RNNModel on cuDNN (fp32, no TF32), and that loop in
    float64 on the CPU, all from the same initial weights."""
    lu = _reference()
    ntoken, emsize, nhid, nl, B, bptt, lr, clip = 100, 48, 64, 2, 20, 35, 20.0, 0.25
    g = torch.Generator().manual_seed(5)
    train = LT.batchify(torch.randint(0, ntoken, (B * bptt * 5 + B,), generator=g), B)
    val = LT.batchify(torch.randint(0, ntoken, (10 * 50,), generator=g), LT.EVAL_BATCH_SIZE)
    torch.manual_seed(11)
    mine = b200asr.RNNModel("LSTM", ntoken, emsize, nhid, nl, dropout=0.0).to(DEV)
    init = {k: v.detach().cpu().clone() for k, v in mine.state_dict().items()}
    losses = LT.train_epoch(mine, train.to(DEV), ntoken, lr, bptt, clip)
    assert len(losses) == 5
    v_mine = LT.evaluate(mine, val.to(DEV), ntoken, bptt)
    mine_run = ([float(l) for l in losses], {k: v.detach().cpu().double() for k, v in mine.state_dict().items()}, v_mine)
    saved = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    try:
        cudnn = lu.RNNModel("LSTM", ntoken, emsize, nhid, nl, dropout=0.0)
        cudnn.load_state_dict(init)
        cudnn_run = _example_loop(cudnn.to(DEV), train.to(DEV), val.to(DEV), ntoken, bptt, lr, clip)
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = saved
    f64 = lu.RNNModel("LSTM", ntoken, emsize, nhid, nl, dropout=0.0)
    f64.load_state_dict(init)
    f64_run = _example_loop(f64.double(), train, val, ntoken, bptt, lr, clip)

    def dist(r):
        return (max(abs(a - b) / abs(b) for a, b in zip(r[0], f64_run[0])), max(_err(r[1][k], f64_run[1][k]) for k in f64_run[1]),
                abs(r[2] - f64_run[2]) / abs(f64_run[2]))
    (le1, pe1, ve1), (le0, pe0, ve0) = dist(mine_run), dist(cudnn_run)
    print(f"lm_train loop vs float64: losses max rel {le1:.1e} installed, {le0:.1e} cuDNN; final parameters max rel {pe1:.1e} "
          f"installed, {pe0:.1e} cuDNN; validation loss rel {ve1:.1e} installed, {ve0:.1e} cuDNN")
    # as the word-LM test of tests/test_gpu_lstm_train.py: SGD at lr 20 moves the parameters by 5 per window, so rounding
    # differences grow along the trajectory; the installed loop is held within 50x cuDNN's own distance from float64
    assert le1 <= 50 * le0 + 1e-5 and pe1 <= 50 * pe0 + 1e-4 and ve1 <= 50 * ve0 + 1e-5, (le1, le0, pe1, pe0, ve1, ve0)


def test_training_windows_need_no_host_sync():
    ntoken, B, bptt = 300, 8, 10
    data = LT.batchify(torch.randint(0, ntoken, (B * bptt * 4 + B,), generator=torch.Generator().manual_seed(2)), B, DEV)
    torch.manual_seed(1)
    model = b200asr.RNNModel("LSTM", ntoken, 32, 48, 2, dropout=0.2).to(DEV)
    LT.train_epoch(model, data, ntoken, 20.0, bptt, 0.25)               # warm: kernels attributed, scratch sized
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        losses = LT.train_epoch(model, data, ntoken, 20.0, bptt, 0.25)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert len(losses) == 4 and all(torch.isfinite(l) for l in losses)


# ------------------------------------------------------------------------------------------ the CLI end to end
def _synthetic_corpus(tmp_path, chars, n_train, n_valid, seed):
    """Manifests of random transcripts over `chars` (one word per character once segmented) and the label file."""
    rng = np.random.default_rng(seed)
    out = {}
    for tag, n in (("train", n_train), ("valid", n_valid)):
        lines = []
        for i in range(n):
            k = int(rng.integers(3, 13))
            text = "".join(chars[int(j)] for j in rng.integers(0, len(chars) // 2, k))
            p = tmp_path / f"{tag}{i}.txt"
            p.write_text(text + "\n", encoding="utf8")
            lines.append(f"{tmp_path}/{tag}{i}.wav,{p}")
        (tmp_path / f"{tag}.csv").write_text("\n".join(lines) + "\n")
        out[tag] = str(tmp_path / f"{tag}.csv")
    (tmp_path / "labels.json").write_text(json.dumps(chars, ensure_ascii=False))
    return out["train"], out["valid"], str(tmp_path / "labels.json")


@pytest.mark.skipif(not ref_shim.available(), reason="reference checkout not staged (oracle/make_ref.py)")
def test_cli_checkpoint_loads_and_rescores_as_the_reference(tmp_path, monkeypatch, capsys):
    lu = _reference()
    ns = ref_shim.load(FLAGS, q12_shim=True)
    V = 40
    l2i, i2l = ref_shim.labels(V)
    chars = [i2l[i] for i in range(3, V)]
    train, valid, labels = _synthetic_corpus(tmp_path, chars, 60, 12, seed=4)
    path = tmp_path / "lm.pt"
    # `python -m b200asr.lm_train ...`, run in this process (runpy is what -m uses)
    monkeypatch.setattr(sys, "argv", ["lm_train", "--train-manifest-list", train, "--valid-manifest-list", valid, "--labels-path",
                                      labels, "--save", str(path), "--epochs", "2", "--emsize", "32", "--nhid", "48", "--batch-size",
                                      "4", "--bptt", "8", "--log-interval", "5", "--dropout", "0.1"])
    with pytest.raises(SystemExit) as done:
        runpy.run_module("b200asr.lm_train", run_name="__main__")
    out = capsys.readouterr()
    print(out.out[-1500:])
    assert done.value.code == 0, out.err[-3000:]
    assert "end of epoch   2" in out.out and path.exists()
    assert LT.load_labels(labels) == (l2i, i2l)

    lm = lu.LM(str(path))                                   # torch.load(path): weights_only=True
    mine = b200asr.LM(str(path))
    assert mine.word2idx == lm.word2idx and mine.idx2word == lm.idx2word and lm.word2idx["<eos>"] == 0
    for k, v in lm.model.state_dict().items():
        assert torch.equal(mine.model.state_dict()[k], v.cpu()), k
    corpus = LT.Corpus([train], [valid], l2i, i2l)
    sentence = " ".join(LT.transcript_words(open(valid).readline().strip().split(",")[1], l2i, i2l)[:-1])

    torch.manual_seed(123456)
    model = ns.functions.init_transformer_model(ns.constant.args, l2i, i2l)
    g = torch.Generator().manual_seed(7)
    with torch.no_grad():
        for p in model.parameters():
            if p.dim() == 1:
                p.add_(0.1 * torch.randn(p.shape, generator=g))
        model.decoder.output_linear.weight.mul_(4.0)
        model.decoder.output_linear.weight[2] *= -1.0
    model = model.cuda().eval()
    src = torch.randn(2, 1, 161, 24, generator=g).cuda()
    lens = torch.full((2,), 24, dtype=torch.int32).cuda()
    tgt = torch.randint(3, V, (2, 6), generator=g).cuda()
    saved = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    scores, strings = {}, {}
    try:
        for installed in (False, True):
            if installed:
                b200asr.install()
            scores[installed] = float(lm.evaluate(sentence)[0])
            with torch.no_grad():
                _, strs, _ = model.evaluate(src, lens, tgt, beam_search=True, beam_width=4, beam_nbest=1, lm_rescoring=True, lm=lm,
                                            lm_weight=2.0, c_weight=0.1)
            strings[installed] = list(strs)
    finally:
        b200asr.uninstall()
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = saved
    e = abs(scores[True] - scores[False]) / abs(scores[False])
    print(f"LM.evaluate({sentence!r}): {scores[True]!r} installed, {scores[False]!r} cuDNN (rel {e:.1e}); "
          f"vocabulary {len(corpus.idx2word)}; beam strings {strings[True]}")
    assert e <= 1e-4, (scores, e)
    assert strings[True] == strings[False], strings
