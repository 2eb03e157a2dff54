"""The training loop's CER / WER counts on the device (csrc/edit_distance.cu, metrics.edit_counts, trainer.trainer_train).

  * b200asr_edit_counts against tests/edit_util.kernel_counts (itself checked against the reference's string path on the
    CPU), exactly: B in {1, 3, 32, 129}, T in {1, 63, 64, 65, 100, 1000, 4097} with T_h != T_g and PAD cuts everywhere, empty
    strings, PAD at position 0, identical strings, whitespace runs, SOS / EOS joining words, multi-code-point labels, int32 /
    int64 ids and strided views, invalid ids (first-invalid rule), strings longer than shared memory (workspace path).
    Outputs and workspace are poisoned first; repeated calls give identical bits; no host synchronisation; a call launches
    exactly 2 kernels and a rejected one none.
  * With the reference staged (oracle/_ref): the reference's Trainer.train, installed, once through original(...) and once
    through the bound loop: losses, state_dict, checkpoint metrics, logging lines, progress-bar texts and prints are
    identical, including the infinite-loss and missing-id skips; the bound loop's host synchronisations per iteration are
    bounded and do not grow with B * T_t.
"""
import copy
import logging
import os
import tempfile
import warnings

import numpy as np
import pytest
import torch

import b200asr
from oracle import ref_shim
from tests.edit_util import EOS, SOS, kernel_counts, label_set

pytestmark = pytest.mark.gpu

L = b200asr._lib
DEV = "cuda"
SENT = -(2 ** 62) + 12345


def _lib():
    return L.load()


def _table(id2label, pad=0):
    return b200asr.LabelTable(id2label, pad, (SOS, EOS))


def _raw(hyp, gold, table, max_label_len=None):
    """The C ABI with sentinel-filled outputs and workspace: (per_utt, totals, launches, ws)."""
    mll = table.max_label_len if max_label_len is None else max_label_len
    B, T_h, T_g = hyp.shape[0], hyp.shape[1], gold.shape[1]
    off, length, cps, flags, valid = table.tensors(DEV)
    nws = _lib().b200asr_edit_counts_ws_bytes(B, T_h, T_g, mll)
    assert nws >= 16 * B
    ws = torch.full((nws,), 0xAB, dtype=torch.uint8, device=DEV)
    per = torch.full((B + 1, 4), SENT, dtype=torch.int64, device=DEV)          # one sentinel row past the end
    tot = torch.full((6,), SENT, dtype=torch.int64, device=DEV)
    n0 = _lib().b200asr_launch_count()
    rc = _lib().b200asr_edit_counts(L.ptr(hyp), int(hyp.dtype == torch.int64), hyp.stride(0), T_h, L.ptr(gold),
                                    int(gold.dtype == torch.int64), gold.stride(0), T_g, B, L.ptr(off), L.ptr(length),
                                    L.ptr(cps), L.ptr(flags), L.ptr(valid), table.V, mll, table.pad_id, L.ptr(per), L.ptr(tot),
                                    L.ptr(ws), torch.cuda.current_stream().cuda_stream)
    L.check(rc, "edit_counts")
    launches = _lib().b200asr_launch_count() - n0
    per, tot = per.cpu(), tot.cpu()
    assert per[B].tolist() == [SENT] * 4 and tot[5].item() == SENT
    return per[:B].numpy(), tot[:5].numpy(), launches, ws


def _check(hyp, gold, table, **kw):
    per, tot, launches, _ = _raw(hyp, gold, table, **kw)
    ref_per, ref_tot = kernel_counts(hyp.cpu().numpy(), gold.cpu().numpy(), table)
    assert launches == 2
    np.testing.assert_array_equal(per, ref_per)
    np.testing.assert_array_equal(tot, ref_tot)
    return per, tot


def _ids(g, B, T, V, low=1):
    """Random ids in [low, V) with each row cut by PAD at a random position (some rows uncut)."""
    ids = torch.randint(low, V, (B, T), generator=g)
    cut = torch.randint(0, T + 2, (B,), generator=g)
    for b in range(B):
        ids[b, int(cut[b]):] = 0
    return ids


@pytest.mark.parametrize("B,T_h,T_g", [(1, 1, 63), (3, 63, 64), (32, 64, 65), (129, 100, 63), (32, 100, 1), (3, 1000, 65),
                                       (1, 4097, 1000), (3, 65, 4097), (129, 65, 100)])
def test_edit_counts_match_definition(B, T_h, T_g):
    g = torch.Generator().manual_seed(B * 10007 + T_h * 31 + T_g)
    id2label = label_set(40)
    table = _table(id2label)
    hyp, gold = _ids(g, B, T_h, 40).to(DEV), _ids(g, B, T_g, 40).to(DEV)
    if T_h == T_g:
        hyp[0] = gold[0]
    _check(hyp, gold, table)


def test_edit_counts_every_length_across_64_boundaries():
    """One utterance per gold length 0 .. 200 of single-code-point labels (every multiple of 64 crossed), hyp a perturbed
    copy of the gold."""
    g = torch.Generator().manual_seed(3)
    id2label = {0: "¶", 1: SOS, 2: EOS, 3: " ", **{i: chr(ord("a") + i - 4) for i in range(4, 30)}}
    table = _table(id2label)
    B, T = 201, 200
    gold = torch.randint(3, 30, (B, T), generator=g)
    for b in range(B):
        gold[b, b:] = 0
    hyp = gold.clone()
    flip = torch.rand(B, T, generator=g) < 0.1
    hyp[flip] = torch.randint(3, 30, (int(flip.sum()),), generator=g)
    hyp = torch.cat([hyp, torch.randint(3, 30, (B, 7), generator=g)], 1)
    _check(hyp.to(DEV), gold.to(DEV), table)


def test_edit_counts_edge_strings():
    id2label = label_set(40)
    table = _table(id2label)
    sp, tab, a, b, a_sos, eos_b, sos_sp_eos = 3, 8, 4, 5, 13, 14, 15
    rows = [  # (hyp, gold)
        ([0, a, b], [a, b, 0]),                      # empty hyp (PAD at position 0)
        ([a, b], [0, 0, 0]),                         # empty gold: gold_words = 1, gold_chars = 0
        ([0], [0]),
        ([a, b, 6, sp, 7], [a, b, 6, sp, 7]),        # identical
        ([sp, sp, sp], [sp, sp]),                    # all spaces
        ([sp, a, sp, sp, b, sp], [a, sp, b]),        # leading, repeated and trailing whitespace
        ([a, a_sos, b], [a, eos_b]),                 # § / ¤ between two words joins them
        ([a, sos_sp_eos, b], [a, sp, b]),
        ([a, tab, b, 9, 10, 11, b], [a, sp, b, 26, b]),  # \t, ideographic space, nbsp, \x1c, \n split words
        ([12, 12], [6, 18, 20, 21]),                 # multi-code-point labels
    ]
    T = 8
    hyp = torch.zeros(len(rows), T, dtype=torch.int64)
    gold = torch.zeros(len(rows), T, dtype=torch.int64)
    for r, (h, gd) in enumerate(rows):
        hyp[r, :len(h)] = torch.tensor(h)
        gold[r, :len(gd)] = torch.tensor(gd)
    per, _ = _check(hyp.to(DEV), gold.to(DEV), table)
    assert per[1].tolist() == [2, 1, 0, 1] and per[3].tolist()[:2] == [0, 0]


def test_edit_counts_dtypes_and_strided_views():
    g = torch.Generator().manual_seed(5)
    table = _table(label_set(40))
    wide_h = _ids(g, 6, 150, 40).to(DEV)
    wide_g = _ids(g, 6, 90, 40).to(DEV)
    hyp, gold = wide_h[::2, 10:110], wide_g[1::2, :77]                        # row strides 300 / 180
    ref = _check(hyp, gold, table)
    for hd, gd in [(torch.int32, torch.int32), (torch.int32, torch.int64), (torch.int64, torch.int32)]:
        h32, g32 = wide_h.to(hd)[::2, 10:110], wide_g.to(gd)[1::2, :77]
        got = _check(h32, g32, table)
        np.testing.assert_array_equal(got[0], ref[0])
    per, tot = b200asr.edit_counts(wide_h[:, ::2], gold.repeat(2, 1), table)  # element stride 2: copied first
    ref_per, ref_tot = kernel_counts(wide_h[:, ::2].cpu().numpy(), gold.repeat(2, 1).cpu().numpy(), table)
    np.testing.assert_array_equal(per.cpu().numpy(), ref_per)
    np.testing.assert_array_equal(tot.cpu().numpy(), ref_tot)


def test_edit_counts_invalid_ids_first_in_reference_order():
    id2label = label_set(40, missing=(9, 21))
    table = _table(id2label)
    g = torch.Generator().manual_seed(11)
    ok = torch.tensor(sorted(set(id2label) - {0}))
    hyp = ok[torch.randint(0, len(ok), (4, 20), generator=g)]
    gold = ok[torch.randint(0, len(ok), (4, 12), generator=g)]
    _, tot = _check(hyp.to(DEV), gold.to(DEV), table)
    assert tot[4] == -1
    h, gd = hyp.clone(), gold.clone()
    h[0, 3] = 40                                     # beyond V, hyp row 0
    gd[2, 5] = 21                                    # missing, gold row 2: gold rows come first
    gd[3, 1] = -7
    _, tot = _check(h.to(DEV), gd.to(DEV), table)
    assert tot[4] == 21
    gd[2, 5], gd[3, 1] = 4, 4
    gd[2, 3] = 0                                     # an invalid id after the first PAD is never looked up
    gd[2, 7] = 9
    _, tot = _check(h.to(DEV), gd.to(DEV), table)
    assert tot[4] == 40
    _, tot = _check(h.to(DEV, torch.int32), gd.to(DEV, torch.int32), table)
    assert tot[4] == 40


def test_edit_counts_workspace_path():
    """Labels of 300 code points: strings of up to 1000 * 300 code points, far beyond shared memory; with a generous
    max_label_len and short strings the utterances stay in shared memory while the workspace is reserved."""
    g = torch.Generator().manual_seed(13)
    id2label = {0: "¶", 1: SOS, 2: EOS}
    for i in range(3, 20):
        id2label[i] = "".join(np.random.default_rng(i).choice(list("ab c"), 300))
    id2label[20] = "a"
    table = _table(id2label)
    hyp, gold = _ids(g, 3, 40, 20).to(DEV), _ids(g, 3, 25, 20).to(DEV)
    per, tot, _, ws = _raw(hyp, gold, table)
    assert ws.numel() > 16 * 3 + 46 * 1024
    np.testing.assert_array_equal(per, kernel_counts(hyp.cpu().numpy(), gold.cpu().numpy(), table)[0])
    short_h, short_g = torch.full((2, 30), 20, device=DEV), torch.full((2, 9), 20, device=DEV)
    short_g[1, 4:] = 0
    _check(short_h, short_g, table)
    _check(short_h, short_g, table, max_label_len=4000)
    # a label longer than the promised max_label_len: that utterance reports -1s, nothing else is touched
    per, _, _, _ = _raw(hyp[:1], gold[:1], table, max_label_len=2)
    assert per.tolist() == [[-1, -1, -1, -1]]


def test_edit_counts_repeatable_and_sync_free():
    g = torch.Generator().manual_seed(17)
    table = _table(label_set(40))
    hyp, gold = _ids(g, 32, 100, 40).to(DEV), _ids(g, 32, 100, 40).to(DEV)
    first = b200asr.edit_counts(hyp, gold, table)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        outs = [b200asr.edit_counts(hyp, gold, table) for _ in range(3)]
    finally:
        torch.cuda.set_sync_debug_mode("default")
    for per, tot in outs:
        assert torch.equal(per, first[0]) and torch.equal(tot, first[1])


def test_edit_counts_rejections_launch_nothing():
    table = _table(label_set(40))
    off, length, cps, flags, valid = table.tensors(DEV)
    ids = torch.zeros(4, 8, dtype=torch.int64, device=DEV)
    out = torch.full((4, 4), SENT, dtype=torch.int64, device=DEV)
    tot = torch.full((5,), SENT, dtype=torch.int64, device=DEV)
    ws = torch.zeros(4096, dtype=torch.uint8, device=DEV)
    P, st = L.ptr, torch.cuda.current_stream().cuda_stream

    def call(hyp=ids, h64=1, hs=8, T_h=8, gold=ids, g64=1, gs=8, T_g=8, B=4, V=table.V, mll=table.max_label_len, o=out,
             t=tot, w=ws, table_ptr=P(off)):
        return _lib().b200asr_edit_counts(P(hyp) if hyp is not None else None, h64, hs, T_h,
                                          P(gold) if gold is not None else None, g64, gs, T_g, B, table_ptr, P(length),
                                          P(cps), P(flags), P(valid), V, mll, 0, P(o) if o is not None else None, P(t),
                                          P(w) if w is not None else None, st)
    n0 = _lib().b200asr_launch_count()
    assert call(hyp=None) == -5 and call(w=None) == -5 and call(o=None) == -5 and call(table_ptr=None) == -5
    assert call(h64=2) == -5 and call(g64=-1) == -5
    assert call(B=0) == -1 and call(T_h=-1) == -1 and call(V=0) == -1 and call(mll=-1) == -1
    assert call(hs=7) == -1 and call(gs=3) == -1
    assert call(T_h=1 << 20, hs=1 << 20, mll=1 << 10) == -1                    # per-utterance buffer beyond 2^30 ints
    off4 = lambda t: t.view(torch.int32).view(-1)[1:]                           # 4 bytes past an 8-byte boundary
    assert call(o=off4(out)) == -2 and call(w=ws[4:]) == -2 and call(hyp=off4(ids)) == -2 and call(t=off4(tot)) == -2
    assert _lib().b200asr_launch_count() == n0
    assert torch.all(out == SENT) and torch.all(tot == SENT)
    assert call() == 0 and _lib().b200asr_launch_count() == n0 + 2
    assert _lib().b200asr_edit_counts_ws_bytes(4, 8, 8, 0) == 64 and _lib().b200asr_edit_counts_ws_bytes(0, 8, 8, 1) == 0
    with pytest.raises(ValueError):
        b200asr.edit_counts(ids, ids[:3], table)
    with pytest.raises(ValueError):
        b200asr.edit_counts(ids.float(), ids, table)


# ------------------------------------------------------------------------------------- the reference's Trainer.train
needs_ref = pytest.mark.skipif(not ref_shim.available(), reason="reference checkout not staged (oracle/make_ref.py)")


class _FakeTqdm:
    """Stands in for tqdm in the trainer module: records every set_description text, and the number of host syncs the
    caller has seen when each batch is handed out (sync_log, when set)."""
    texts, marks, sync_log = [], [], None

    def __init__(self, it, leave=True, total=None):
        self.it = it

    def __iter__(self):
        for x in self.it:
            _FakeTqdm.marks.append(len(_FakeTqdm.sync_log) if _FakeTqdm.sync_log is not None else 0)
            yield x
        _FakeTqdm.marks.append(len(_FakeTqdm.sync_log) if _FakeTqdm.sync_log is not None else 0)

    def set_description(self, s):
        _FakeTqdm.texts.append(s)


def _run_arm(ns, model, l2i, i2l, train, valid, loss_type, tmp, bound, caplog, capsys, record_losses=True):
    """One epoch of the installed reference Trainer.train, through the bound loop (bound) or the reference's own.  Returns
    everything it makes observable."""
    ns.constant.args.save_folder, ns.constant.args.name = tmp, "run"
    opt = ns.functions.init_optimizer(ns.constant.args, model, "noam")
    if loss_type == "ctc":
        opt.lr, opt.lr_anneal = 0.0, 0.0
    losses = []
    b200asr.install()
    cur_metrics, cur_tqdm = ns.trainer.calculate_metrics, ns.trainer.tqdm

    def recording(*a, **k):
        out = cur_metrics(*a, **k)
        losses.append(float(out[0].item()))
        return out

    if record_losses:
        ns.trainer.calculate_metrics = recording
    ns.trainer.tqdm = _FakeTqdm
    _FakeTqdm.texts, _FakeTqdm.marks = [], []
    caplog.clear()
    capsys.readouterr()
    err = None
    try:
        tr = copy.deepcopy(train), copy.deepcopy(valid)
        trainer = ns.trainer.Trainer()
        if bound:
            assert ns.trainer.Trainer.train is not b200asr.original(ns.trainer.Trainer, "train")
            trainer.train(model, tr[0], None, tr[1], opt, loss_type, 0, 1, l2i, i2l)
        else:
            b200asr.original(ns.trainer.Trainer, "train")(trainer, model, tr[0], None, tr[1], opt, loss_type, 0, 1, l2i, i2l)
    except Exception as e:                            # both arms must fail the same way
        err = f"{type(e).__name__}: {e}"
    finally:
        ns.trainer.calculate_metrics, ns.trainer.tqdm = cur_metrics, cur_tqdm
        b200asr.uninstall()
    logs = [r.getMessage() for r in caplog.records if r.name == "root"]
    out = capsys.readouterr().out
    ck = os.path.join(tmp, "run", "best_model.th")
    metrics = None
    if os.path.exists(ck):
        m = torch.load(ck, weights_only=False)["metrics"]
        metrics = {k: v for k, v in m.items() if k != "history"}
        os.remove(ck)
    sd = {k: v.detach().cpu().clone() for k, v in model.state_dict().items()}
    return dict(losses=losses, sd=sd, metrics=metrics, logs=logs, texts=list(_FakeTqdm.texts), out=out, err=err,
                step=opt._step)


def _cuda_batches(batches):
    return [(s.cuda(), t.cuda(), p, l, tl) for s, t, p, l, tl in batches]


@needs_ref
@pytest.mark.parametrize("case", ["small_vgg-ce", "small_emb-ce", "small_vgg-ctc", "small_vgg-ce-missing-id"])
def test_bound_trainer_loop_matches_reference_loop(case, caplog, capsys):
    from tests.test_gpu_ctc import _trainer_batches
    from tests.test_gpu_reference import SMALL_EMB, SMALL_VGG, _build, _fp32_flags, _loaders
    arch, loss_type = case.split("-")[:2]
    flags, vocab, freq, B, T = {"small_vgg": (SMALL_VGG, 40, 41, 4, 32), "small_emb": (SMALL_EMB, 40, 161, 4, 48)}[arch]
    caplog.set_level(logging.INFO)
    _fp32_flags()
    i2l = label_set(vocab, missing=(vocab - 1,) if case.endswith("missing-id") else ())
    res = {}
    with tempfile.TemporaryDirectory() as tmp:
        for bound in (False, True):
            ns, model, l2i, _ = _build(flags, vocab, extra=["--cuda", "--warmup", "4", "--k-lr", "0.02", "--min-lr", "1e-6",
                                                             "--clip", "--max-norm", "400", "--loss", loss_type])
            model = model.cuda()
            if case.endswith("missing-id"):
                with torch.no_grad():                        # logit 0 for the missing id: argmax hardly ever picks it
                    model.decoder.output_linear.weight[vocab - 1].zero_()
            if loss_type == "ctc":
                train, valid = _trainer_batches(ns, freq, T, vocab, ns.constant.args.tgt_max_len - 1, B)
            else:
                train, valid = _loaders(freq, T, vocab - 1, ns.constant.args.tgt_max_len - 1, 4, B)
                if case.endswith("missing-id"):
                    train[1][1][2, 0] = vocab - 1            # a gold id id2label lacks: that batch is skipped
                    valid[0].append(copy.deepcopy(train[1]))
            res[bound] = _run_arm(ns, model, l2i, i2l, train, valid, loss_type, tmp, bound, caplog, capsys)
    ref, got = res[False], res[True]
    print(f"[{case}] losses {ref['losses']}\n[{case}] logs {ref['logs']}\n[{case}] metrics {ref['metrics']}")
    assert ref["err"] is None, ref["err"]
    for k in ("losses", "metrics", "logs", "texts", "out", "err", "step"):
        assert got[k] == ref[k], k
    for k in ref["sd"]:
        assert torch.equal(got["sd"][k], ref["sd"][k]), k
    assert ref["metrics"]["train_cer"] > 0 and ref["metrics"]["valid_wer"] > 0
    if loss_type == "ctc":
        assert "Found infinity loss, masking" in ref["logs"]
    if case.endswith("missing-id"):
        assert ref["logs"].count("NaN predictions") >= 2 and f"{vocab - 1}\n" in ref["out"]


@needs_ref
def test_bound_trainer_loop_syncs_per_iteration(caplog, capsys):
    """Host syncs per training iteration (torch's sync debug mode), at two batch shapes.  The reference's loop reads two ids
    per token; the bound loop reads the totals row, calculate_metrics's num_correct and the loss."""
    from tests.test_gpu_reference import SMALL_VGG, _batch, _build, _fp32_flags
    _fp32_flags()
    counts = {}
    with tempfile.TemporaryDirectory() as tmp:
        for B, T in ((4, 32), (16, 64)):
            for bound in (False, True):
                ns, model, l2i, i2l = _build(SMALL_VGG, 40, extra=["--cuda", "--warmup", "4", "--clip"])
                model = model.cuda()
                Lt = ns.constant.args.tgt_max_len - 1

                def one(seed):
                    src, lens, tgt, tl = _batch(B, 41, T, 40, Lt, seed=seed)
                    return (src, tgt, lens.float() / float(T), lens, tl)
                train, valid = _cuda_batches([one(s) for s in range(4)]), [_cuda_batches([one(100)])]
                with warnings.catch_warnings(record=True) as caught:
                    warnings.simplefilter("always")
                    _FakeTqdm.sync_log = caught               # _FakeTqdm reads its length at every batch
                    torch.cuda.set_sync_debug_mode("warn")
                    try:
                        r = _run_arm(ns, model, l2i, i2l, train, valid, "ce", tmp, bound, caplog, capsys,
                                     record_losses=False)
                    finally:
                        torch.cuda.set_sync_debug_mode("default")
                        _FakeTqdm.sync_log = None
                assert r["err"] is None, r["err"]
                marks = _FakeTqdm.marks[:5]                  # the 4 training batches handed out, then the end of the loop
                counts[(B, T, bound)] = [b - a for a, b in zip(marks, marks[1:])]
    for (B, T, bound), per_it in sorted(counts.items()):
        print(f"B={B} T_t<={T}: {'bound' if bound else 'reference'} loop host syncs per training iteration {per_it}")
    small, large = counts[(4, 32, True)], counts[(16, 64, True)]
    assert small[1:] == large[1:] and max(small[1:]) <= 3, (small, large)
    assert min(counts[(16, 64, False)]) > 10 * max(large)
