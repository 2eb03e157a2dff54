"""The bound Trainer.train in data-parallel mode, on one GPU: two gloo ranks sharing it against one process on the whole
batch, both through the UNMODIFIED reference's Trainer.train after install() (cfg1-sized vgg_cnn / emb_cnn models,
dropout 0).  Every arm runs in a process of its own.

vgg_cnn has no batch statistics, so two ranks compute what one process computes on the gathered batch:

  * CER / WER / char / word totals (the checkpoint's metrics), log lines and progress texts are identical;
  * per-iteration losses agree to fp32 summation-order noise;
  * the first iteration's scaled gradient agrees with the single process's in the max norm (bound GRAD_TOL below);
  * parameters and Adam state after 3 iterations stay within the bounds of test_gpu_reference's trainer test;
  * rank 1 logs, draws and prints nothing and writes no checkpoint; rank 0's checkpoint loads into a single-GPU model and
    into a stock torch Adam;
  * an id missing from id2label, or an infeasible CTC utterance, in rank 1's shard alone makes both ranks skip exactly as
    the single process does; an uneven last batch and a batch smaller than the world run;
  * host synchronisations per training iteration are counted (rank 0).
emb_cnn's BatchNorm normalises in training mode with the statistics of the shard each rank sees, as it does on every
replica of nn.DataParallel (no SyncBatchNorm in the reference), so its losses differ from one process on the whole batch
by more than rounding: there the ranks must hold identical parameters and Adam state, rank 0's own running statistics
must be the ones saved, and the checkpoint must load.
"""
import contextlib
import copy
import io
import logging
import os
import socket
import tempfile
import warnings

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from oracle import ref_shim

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not ref_shim.available(), reason="reference checkout not staged (oracle/make_ref.py)")]

GRAD_TOL = 1e-4          # max |g_2ranks - g_1process| over every element, relative to max |g_1process|
LOSS_TOL = 1e-5          # relative, per iteration


class _Records(logging.Handler):
    def __init__(self):
        super().__init__(logging.INFO)
        self.msgs = []

    def emit(self, record):
        if record.name == "root":
            self.msgs.append(record.getMessage())


def _batches(case, ns, vocab):
    from tests.test_gpu_ctc import _trainer_batches
    from tests.test_gpu_reference import _batch, _loaders
    arch, loss_type = case.split("-")[:2]
    freq, B, T = {"small_vgg": (41, 4, 32), "small_emb": (161, 4, 48)}[arch]
    Lt = ns.constant.args.tgt_max_len - 1
    if loss_type == "ctc":
        return _trainer_batches(ns, freq, T, vocab, Lt, B)           # the infeasible utterance is the last of its batch
    train, valid = _loaders(freq, T, vocab - 1, Lt, 3, B)
    if case.endswith("skip"):
        train[1][1][3, 0] = vocab - 1                                  # a gold id id2label lacks, in rank 1's shard only

        def one(seed, b):
            src, lens, tgt, tl = _batch(b, freq, T, vocab - 1, Lt, seed=seed)
            return (src, tgt, lens.float() / float(T), lens, tl)
        train += [one(20, 3), one(21, 1)]                              # uneven last batches: 2 + 1 and 1 + 0 utterances
        valid[0] += [one(22, 3), one(23, 1)]
    return train, valid


def _arm(rank, world, port, case, tmp):
    """One rank (or the single process, world 1): one epoch of the installed reference Trainer.train."""
    import b200asr
    from tests.edit_util import label_set
    from tests.test_gpu_edit_counts import _FakeTqdm
    from tests.test_gpu_reference import SMALL_EMB, SMALL_VGG, _build, _fp32_flags
    if world > 1:
        os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
        dist.init_process_group("gloo", rank=rank, world_size=world)
    arch, loss_type = case.split("-")[:2]
    flags, vocab = {"small_vgg": (SMALL_VGG, 40), "small_emb": (SMALL_EMB, 40)}[arch]
    _fp32_flags()
    ns, model, l2i, _ = _build(flags, vocab, extra=["--cuda", "--warmup", "4", "--k-lr", "0.02", "--min-lr", "1e-6", "--clip",
                                                     "--max-norm", "400", "--loss", loss_type])
    i2l = label_set(vocab, missing=(vocab - 1,) if case.endswith("skip") else ())
    if arch == "small_emb":                      # see test_gpu_reference: a conv bias in front of BatchNorm is a gauge freedom
        model.conv[0].bias.requires_grad_(False)
        model.conv[3].bias.requires_grad_(False)
    model = model.cuda()
    if case.endswith("skip"):
        with torch.no_grad():                    # logit 0 for the missing id: argmax hardly ever picks it
            model.decoder.output_linear.weight[vocab - 1].zero_()
    init = {k: v.detach().cpu().clone() for k, v in model.state_dict().items()}
    train, valid = _batches(case, ns, vocab)
    save = os.path.join(tmp, f"rank{rank}" if world > 1 else "single")
    ns.constant.args.save_folder, ns.constant.args.name = save, "run"
    opt = ns.functions.init_optimizer(ns.constant.args, model, "noam")
    if loss_type == "ctc":
        opt.lr, opt.lr_anneal = 0.0, 0.0
    grads0, losses = [], []
    step = opt.step

    def recording_step():
        if not grads0:
            grads0.append({n: p.grad.detach().cpu().clone() for n, p in model.named_parameters() if p.grad is not None})
        step()
    opt.step = recording_step

    trainer = ns.trainer.Trainer()               # its constructor logs on every rank: train.py calls it on every rank
    records = _Records()
    logging.getLogger().addHandler(records)
    logging.getLogger().setLevel(logging.INFO)
    out = io.StringIO()
    _FakeTqdm.texts, _FakeTqdm.marks = [], []
    b200asr.install(process_group=dist.group.WORLD if world > 1 else None)
    tmod = __import__(b200asr.__name__ + ".trainer", fromlist=["loss_value"])
    cur_metrics, cur_tqdm, cur_value = ns.trainer.calculate_metrics, ns.trainer.tqdm, tmod.loss_value

    def recording_metrics(*a, **k):
        o = cur_metrics(*a, **k)
        losses.append(float(o[0].item()))
        return o

    def recording_value(row):
        v = cur_value(row)
        losses.append(v)
        return v
    ns.trainer.calculate_metrics, ns.trainer.tqdm, tmod.loss_value = recording_metrics, _FakeTqdm, recording_value
    try:
        with warnings.catch_warnings(record=True) as caught, contextlib.redirect_stdout(out):
            warnings.simplefilter("always")
            _FakeTqdm.sync_log = caught
            torch.cuda.set_sync_debug_mode("warn")
            try:
                trainer.train(model, copy.deepcopy(train), None, copy.deepcopy(valid), opt, loss_type, 0, 1, l2i, i2l)
            finally:
                torch.cuda.set_sync_debug_mode("default")
                _FakeTqdm.sync_log = None
    finally:
        ns.trainer.calculate_metrics, ns.trainer.tqdm, tmod.loss_value = cur_metrics, cur_tqdm, cur_value
        b200asr.uninstall()
        logging.getLogger().removeHandler(records)
    marks = _FakeTqdm.marks[:len(train) + 1]
    files = sorted(os.listdir(os.path.join(save, "run"))) if os.path.isdir(os.path.join(save, "run")) else []
    res = dict(losses=losses, logs=records.msgs, texts=list(_FakeTqdm.texts), out=out.getvalue().replace(save, "<save>"),
               step=opt._step, files=files,
               syncs=[b - a for a, b in zip(marks, marks[1:])], init=init, grads0=grads0[0] if grads0 else None,
               sd={k: v.detach().cpu().clone() for k, v in model.state_dict().items()},
               adam={i: {k: (v.cpu().clone() if torch.is_tensor(v) else v) for k, v in s.items()}
                     for i, s in opt.optimizer.state_dict()["state"].items()},
               names=[n for n, _ in model.named_parameters()])
    torch.save(res, os.path.join(tmp, f"result{rank}-{world}.pt"))
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()


def _spawn(world, case, tmp):
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    mp.start_processes(_arm, args=(world, port, case, tmp), nprocs=world, join=True, start_method="spawn")
    return [torch.load(os.path.join(tmp, f"result{r}-{world}.pt"), weights_only=False) for r in range(world)]


def _close(a, b, tol):
    return all(abs(x - y) <= tol * max(abs(x), abs(y), 1e-30) for x, y in zip(a, b)) and len(a) == len(b)


def _strip_loss(texts):
    """Progress texts with the LOSS field cut out (compared numerically instead: fp32 noise can move its 4th decimal)."""
    import re
    return [re.sub(r"LOSS:[-0-9.naif]+", "LOSS:", t) for t in texts]


def _losses_in(texts):
    import re
    return [float(m) for t in texts for m in re.findall(r"LOSS:([-0-9.]+)", t)]


@pytest.mark.parametrize("case", ["small_vgg-ce", "small_emb-ce", "small_vgg-ce-skip", "small_vgg-ctc"])
def test_two_ranks_on_one_gpu_match_one_process(case):
    with tempfile.TemporaryDirectory() as tmp:
        (one,) = _spawn(1, case, tmp)
        r0, r1 = _spawn(2, case, tmp)
        ck_path = os.path.join(tmp, "rank0", "run", "best_model.th")
        ck = torch.load(ck_path, weights_only=False) if os.path.exists(ck_path) else None
        ck1 = torch.load(os.path.join(tmp, "single", "run", "best_model.th"), weights_only=False)
    print(f"[{case}] losses 1 process {one['losses']}\n[{case}] losses 2 ranks   {r0['losses']}")
    print(f"[{case}] host syncs per training iteration: 1 process {one['syncs']}, 2 ranks (rank 0) {r0['syncs']}")
    print(f"[{case}] logs {one['logs']}")
    # rank 1: silent, no checkpoint
    assert r1["logs"] == [] and r1["texts"] == [] and r1["out"] == "" and r1["files"] == []
    assert r0["files"] == one["files"] and "best_model.th" in r0["files"]
    assert r0["out"] == one["out"] and r0["step"] == one["step"] == r1["step"]
    assert r0["names"] == one["names"] and list(r0["sd"]) == list(one["sd"])
    if case.startswith("small_emb"):
        assert len(r0["logs"]) == len(one["logs"]) and len(r0["texts"]) == len(one["texts"]) and r0["step"] == 3
        for k in one["sd"]:
            if "running_" in k:
                assert not torch.equal(r0["sd"][k], r1["sd"][k]), k       # per-rank statistics ...
                assert torch.equal(ck["model_state_dict"][k].cpu(), r0["sd"][k]), k    # ... rank 0's saved
            elif "num_batches_tracked" not in k:
                assert torch.equal(r0["sd"][k], r1["sd"][k]), k
        for i, s in r0["adam"].items():
            assert all(torch.equal(s[key], r1["adam"][i][key]) for key in ("exp_avg", "exp_avg_sq")), i
        _check_checkpoint(case, ck, r0)
        return
    # what the user sees: identical apart from fp32 noise in the loss
    assert r0["logs"] == one["logs"] or (_strip_loss(r0["logs"]) == _strip_loss(one["logs"]) and
                                         _close(_losses_in(r0["logs"]), _losses_in(one["logs"]), 1e-3))
    assert _strip_loss(r0["texts"]) == _strip_loss(one["texts"])
    assert _close(_losses_in(r0["texts"]), _losses_in(one["texts"]), 1e-3)
    m0 = {k: v for k, v in ck["metrics"].items() if k != "history"}
    m1 = {k: v for k, v in ck1["metrics"].items() if k != "history"}
    for k in ("train_cer", "train_wer", "valid_cer", "valid_wer"):
        assert m0[k] == m1[k], k
    assert abs(m0["train_loss"] - m1["train_loss"]) <= LOSS_TOL * abs(m1["train_loss"])
    if case.endswith("skip"):
        assert one["logs"].count("NaN predictions") == 1 and "39\n" in one["out"]
        assert r0["losses"] and one["step"] == 4                    # 5 batches, the one with the missing id skipped
        return
    if case.endswith("ctc"):
        assert "Found infinity loss, masking" in one["logs"]
        assert _close([x for x in r0["losses"] if x != float("inf")], [x for x in one["losses"] if x != float("inf")], LOSS_TOL)
        return
    assert _close(r0["losses"], one["losses"], LOSS_TOL), (r0["losses"], one["losses"])
    # the first iteration's global gradient, scaled by 1 / global tokens
    g_max = max(float(g.abs().max()) for g in one["grads0"].values())
    err = max(float((r0["grads0"][k] - g).abs().max()) for k, g in one["grads0"].items())
    print(f"[{case}] first-iteration gradient: max |diff| {err:.3e} (max |g| {g_max:.3e}, ratio {err / g_max:.2e})")
    assert set(r0["grads0"]) == set(one["grads0"]) and err <= GRAD_TOL * g_max
    # both ranks hold the same parameters
    for k in one["sd"]:
        if "running_" in k or "num_batches_tracked" in k:
            continue
        assert torch.equal(r0["sd"][k], r1["sd"][k]), k
    # after 3 iterations: the bounds of test_gpu_reference.test_reference_trainer_loop_runs_on_installed_kernels
    init = one["init"]
    for k in one["sd"]:
        if "num_batches_tracked" in k or "running_" in k or k.endswith("positional_encoding.pe"):
            continue
        d1, d0 = one["sd"][k].float() - init[k].float(), r0["sd"][k].float() - init[k].float()
        if d1.numel() < 256:
            continue
        assert float((d1 - d0).norm() / d1.norm().clamp_min(1e-30)) < (0.05 if d1.numel() >= 16384 else 0.15), k
    assert set(r0["adam"]) == set(one["adam"])
    for i, s in one["adam"].items():
        assert float(s["step"]) == float(r0["adam"][i]["step"]) == 3.0
        for key in ("exp_avg", "exp_avg_sq"):
            a, b = s[key], r0["adam"][i][key]
            if a.numel() < 256:
                continue
            assert float((a - b).norm() / a.norm().clamp_min(1e-30)) < (0.05 if a.numel() >= 16384 else 0.15), (i, key)
    _check_checkpoint(case, ck, r0)
    steps = [s for s in r0["syncs"][1:len(r0["syncs"]) - 1]]
    assert steps and max(steps) <= 3, r0["syncs"]                  # the read of the reduced row, DESIGN.md §5


def _check_checkpoint(case, ck, r0):
    """Rank 0's checkpoint: a plain single-GPU state_dict and a stock torch Adam state."""
    assert not any(k.startswith("module.") for k in ck["model_state_dict"])
    from tests.test_gpu_reference import SMALL_EMB, SMALL_VGG, _build
    flags = SMALL_VGG if case.startswith("small_vgg") else SMALL_EMB
    ns, model, _, _ = _build(flags, 40, extra=["--cuda"])
    model = model.cuda()
    model.load_state_dict(ck["model_state_dict"])
    adam = torch.optim.Adam(model.parameters(), betas=(0.9, 0.98), eps=1e-9)
    adam.load_state_dict(ck["optimizer_state_dict"])
    assert len(adam.state) == len(r0["adam"])
