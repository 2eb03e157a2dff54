"""The bound Transformer.evaluate in data-parallel mode, on one GPU: two gloo ranks sharing it against one process, every
arm in a process of its own (the unmodified reference's models and test.py, cfg1-sized vgg_cnn / emb_cnn, tgt_max_len 300).

  * Per shard, bit for bit: for greedy, beam W = 1 and 4 and beam W = 4 with an LSTM LM, at B in {1, 2, 5, 8}, both ranks
    return the same (strs_hyps, strs_gold), and strs_hyps equals, position by position, what one process's installed
    evaluate returns for each rank's sub-batch (utterances r, r + 2, ...; the same padded T) decoded alone.  B = 1 leaves
    rank 1 an empty share.
  * The decode's bits can depend on the number of rows (split-K choices and decode_attn's key chunking follow it), so the
    comparisons with one process on the WHOLE batch are made only where every decision is safe: the fixtures
    (tests/golden/greedy.npz, beam.npz) are compared with the reference's ids for the utterances whose float64 top-2
    margins exceed the bars of the single-process fixture tests, and the fallback batch below is built so that every
    decision's margin is hundreds of logits wide.
  * Fallback: a batch in which only rank 1's utterance ends no beam hypothesis makes both ranks print
    ">>>>>>> switch to greedy" once and return the greedy strings of every utterance, as one process does.
  * test.py's evaluate, loaded from its file, over the installed loader: every rank's final TEST CER / WER / CER_EN /
    CER_ZH text equals the single process's.
  * Counts per batch: greedy 1 collective, beam 1 (the gathered lengths decide the fallback), + 1 on fallback; rank 0's
    host synchronisations are at most one process's on the whole batch plus the collectives.
"""
import contextlib
import io
import os
import pathlib
import re
import socket
import tempfile
import types
import warnings

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from oracle import ref_shim

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not ref_shim.available(), reason="reference checkout not staged (oracle/make_ref.py)")]

BATCHES = (1, 2, 5, 8)
MODES = {"greedy": dict(beam_search=False), "beam1": dict(beam_search=True, beam_width=1),
         "beam4": dict(beam_search=True, beam_width=4), "beam4-lm": dict(beam_search=True, beam_width=4, lm_rescoring=True)}
FALLBACK = "switch to greedy"


def _spawn(fn, world, tmp):
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    mp.start_processes(_arm, args=(fn, world, port, tmp), nprocs=world, join=True, start_method="spawn")
    return [torch.load(os.path.join(tmp, f"{fn}{r}-{world}.pt"), weights_only=False) for r in range(world)]


def _arm(rank, fn, world, port, tmp):
    import b200asr
    if world > 1:
        os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
        dist.init_process_group("gloo", rank=rank, world_size=world)
    group = (dist.group.WORLD, rank, world) if world > 1 else None
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    try:
        res = globals()[fn](b200asr, group)
    finally:
        b200asr.uninstall()
    torch.save(res, os.path.join(tmp, f"{fn}{rank}-{world}.pt"))
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()


class _Counted:
    """Counts the collectives torch.distributed issues and the host synchronisations of the current device."""

    def __init__(self):
        self.collectives = 0

    @contextlib.contextmanager
    def __call__(self, out):
        wrapped = {}
        for name in ("all_gather", "all_reduce", "broadcast", "all_gather_into_tensor"):
            f = getattr(dist, name)

            def counting(*a, _f=f, **k):
                self.collectives += 1
                return _f(*a, **k)
            wrapped[name] = f
            setattr(dist, name, counting)
        self.collectives = 0
        with warnings.catch_warnings(record=True) as caught, contextlib.redirect_stdout(out):
            warnings.simplefilter("always")
            torch.cuda.set_sync_debug_mode("warn")
            try:
                yield self
            finally:
                torch.cuda.set_sync_debug_mode("default")
                for name, f in wrapped.items():
                    setattr(dist, name, f)
        self.syncs = sum("synchroniz" in str(w.message) for w in caught)


# ------------------------------------------------------------------------------------------ 1 + 5: shards and counts
def _lm(labels, device):
    from b200asr import modules as M
    words = ["<eos>", "<oov>"] + sorted(set(labels.values()))[3:23]
    torch.manual_seed(3)
    model = M.RNNModel("LSTM", len(words), 24, 40, 2, dropout=0.0)
    with torch.no_grad():
        for p in model.parameters():
            p.copy_(0.5 * torch.randn(p.shape))
    return types.SimpleNamespace(model=model.to(device).eval(), word2idx={w: i for i, w in enumerate(words)})


def _shard_model(feat):
    from tests.test_gpu_reference import SMALL_EMB, SMALL_VGG, _build
    flags = SMALL_VGG if feat == "vgg_cnn" else SMALL_EMB
    ns, model, _, i2l = _build(flags, 40, extra=["--cuda", "--tgt-max-len", "300"])
    g = torch.Generator().manual_seed(11)
    with torch.no_grad():
        model.decoder.output_linear.weight.mul_(4.0)                     # spread the logits
        model.decoder.output_linear.weight[2].mul_(2.2 if feat == "vgg_cnn" else 1.0)   # the EOS row of test_gpu_greedy_evaluate
        if feat == "emb_cnn":
            for bn in (model.conv[1], model.conv[4]):
                bn.running_mean.copy_(0.2 * torch.randn(bn.running_mean.shape, generator=g))
                bn.running_var.copy_(0.5 + torch.rand(bn.running_var.shape, generator=g))
                bn.num_batches_tracked.fill_(10)
    return model.cuda().eval(), i2l


def _shard_batch(feat, B, seed):
    from tests.test_gpu_reference import _batch
    freq, T = (41, 96) if feat == "vgg_cnn" else (161, 48)
    src, lens, tgt, _ = _batch(B, freq, T, 40, 6, seed=seed)
    return src.cuda(), lens.cuda(), tgt.cuda()


def shards(b200asr, group):
    out = {}
    count = _Counted()
    for feat in ("vgg_cnn", "emb_cnn"):
        model, i2l = _shard_model(feat)
        lm = _lm(i2l, "cuda")
        b200asr.install(process_group=group[0] if group else None)
        for mode, kw in MODES.items():
            kw = dict(kw, beam_nbest=1, c_weight=0.1, lm=lm if kw.get("lm_rescoring") else None)
            for B in BATCHES:
                src, lens, tgt = _shard_batch(feat, B, seed=B)
                text = io.StringIO()
                with torch.no_grad(), count(text):
                    rest, hyps, gold = model.evaluate(src, lens, tgt, **kw)
                r = dict(hyps=hyps, gold=gold, rest=rest, out=text.getvalue(), syncs=count.syncs, collectives=count.collectives)
                if group is None:              # each rank's sub-batch decoded alone
                    r["sub"] = {k: model.evaluate(src[k::2].contiguous(), lens[k::2].contiguous(), tgt[k::2].contiguous(), **kw)[1]
                                for k in range(min(B, 2))}
                out[(feat, mode, B)] = r
        b200asr.uninstall()
    return out


def test_each_rank_decodes_its_share_bit_for_bit():
    with tempfile.TemporaryDirectory() as tmp:
        (one,) = _spawn("shards", 1, tmp)
        r0, r1 = _spawn("shards", 2, tmp)
    assert set(one) == set(r0) == set(r1)
    for key, s in one.items():
        feat, mode, B = key
        a, b = r0[key], r1[key]
        assert (a["hyps"], a["gold"]) == (b["hyps"], b["gold"]), key
        assert a["gold"] == s["gold"] and a["rest"] == s["rest"], key
        assert FALLBACK not in s["out"] and FALLBACK not in a["out"], key        # this batch ends every utterance
        want = [None] * B
        for k, sub in s["sub"].items():
            want[k::2] = sub
        assert a["hyps"] == want, (key, a["hyps"], want)
        beam = mode != "greedy"
        assert a["collectives"] == b["collectives"] == 1, key
        assert a["syncs"] <= s["syncs"] + a["collectives"], (key, a["syncs"], s["syncs"])
        if B == 8:
            print(f"{feat} {mode} B=8: host syncs 1 process {s['syncs']}, 2 ranks (rank 0) {a['syncs']}; "
                  f"collectives {a['collectives']}; hypothesis lengths {[len(h) for h in a['hyps']]}; beam {beam}")


# ------------------------------------------------------------------------------------------ 2: the fixtures
def fixtures(b200asr, group):
    from b200asr import modules as M
    from tests.beam_util import load_beam_golden
    from tests.gpu_util import cuda_model
    from tests.helpers import load_greedy_golden
    from tests.test_gpu_greedy_evaluate import golden_labels
    from oracle import asr_oracle as O

    def decoder(cfg, P, id2label):
        full = dict(O.init_params(cfg, seed=1))
        full.update(P)
        dec = cuda_model(cfg, full, train=False).decoder
        dec.id2label = id2label
        return dec

    def run(dec, enc, beam, W=0, cw=1.0):
        enc = enc.cuda()
        text = io.StringIO()
        with torch.no_grad(), contextlib.redirect_stdout(text):
            if group is not None:
                rank, world = group[1], group[2]
                mine = enc[rank::world].contiguous() if rank < enc.shape[0] else None
                strs = M.decode_sharded(dec, mine, enc.shape[0], enc.shape[1], group, beam, W, None, 0.1, cw)
            elif beam:                         # what one process's evaluate does (transformer.py:112-118)
                strs = dec.beam_search(enc, beam_width=W, nbest=1, c_weight=cw)[1]
                if len(strs) != enc.shape[0]:
                    print(">>>>>>> switch to greedy")
                    strs = dec.greedy_search(enc)
            else:
                strs = dec.greedy_search(enc)
        return strs, text.getvalue()

    cfg, P, enc, _, _ = load_greedy_golden()
    out = {"greedy": run(decoder(cfg, P, golden_labels(cfg.vocab)), enc, False)}
    cfg, id2label, cases = load_beam_golden()
    for ci, c in enumerate(cases):
        out[ci] = run(decoder(cfg, c["P"], id2label), c["enc"], True, c["W"], c["c_weight"])
    return out


def test_fixture_ids_under_two_ranks():
    from oracle import asr_oracle as O
    from oracle import beam_oracle as BO
    from tests.beam_util import load_beam_golden
    from tests.helpers import load_greedy_golden
    from tests.test_gpu_beam_search import MARGIN_BAR
    from tests.test_gpu_greedy_evaluate import golden_labels
    with tempfile.TemporaryDirectory() as tmp:
        (one,) = _spawn("fixtures", 1, tmp)
        r0, r1 = _spawn("fixtures", 2, tmp)
    assert r0 == r1
    # greedy: the band and the comparison of test_gpu_greedy_evaluate.test_greedy_search_returns_the_reference_strings
    cfg, P, enc, ref_ids, ref_len = load_greedy_golden()
    full = dict(O.init_params(cfg, seed=1))
    full.update(P)
    _, margins = O.greedy_decode(full, cfg, enc, steps=300)
    band = 1e-4 * float(margins.abs().max())
    lab = golden_labels(cfg.vocab)
    n_full = 0
    for b in range(enc.shape[0]):
        n = int(ref_len[b])
        want = "".join(lab[int(i)] for i in ref_ids[b, :n])
        safe = int((margins[b] > band).long().cumprod(0).sum())
        m = min(n, safe)
        assert r0["greedy"][0][b][:m] == one["greedy"][0][b][:m] == want[:m], b
        if safe >= n:
            assert r0["greedy"][0][b] == one["greedy"][0][b] == want, b
            n_full += 1
    print(f"greedy fixture: {n_full}/{enc.shape[0]} utterances compared whole, the rest up to their first near-tie")
    # beam: the utterances whose float64 decision margins (nbest = 1) all exceed the bar of test_gpu_beam_search
    cfg, id2label, cases = load_beam_golden()
    n_ok = n_all = 0
    for ci, c in enumerate(cases):
        strs, text = r0[ci]
        assert (FALLBACK in text) == (FALLBACK in one[ci][1]) and text.count(FALLBACK) <= 1, ci
        if FALLBACK in text:
            assert len(strs) == c["enc"].shape[0]
            continue
        Pd = {k: v.double() for k, v in c["P"].items()}
        oracle = BO.beam_search(Pd, cfg, c["enc"].double(), c["W"], 1, c["c_weight"], id2label)
        for b in range(c["enc"].shape[0]):
            n_all += 1
            margin = min(oracle[b]["step_margins"] + [oracle[b]["pool_margin"]])
            if margin <= MARGIN_BAR:
                continue
            y = [int(t) for t in c["ids"][b, 0, :int(c["lengths"][b, 0])]]
            assert strs[b] == one[ci][0][b] == "".join(id2label[t] for t in y[1:]), (ci, b)
            n_ok += 1
    print(f"beam fixture: {n_ok}/{n_all} utterances compared")
    assert n_ok * 2 >= n_all


# ------------------------------------------------------------------------------------------ 3: fallback
def _fallback_decoder(b200asr):
    """A decoder whose every decision depends on one encoder vector: with an encoder output constant in time (e or -e)
    cross-attention returns W_o W_v e whatever the weights, scaled 100x it dominates the residual, the FFN adds nothing,
    and the EOS row is 10 LN(W_o W_v e).  An utterance with e picks EOS at once by a margin of ~600 logits, one with -e
    never picks it; T_e = 310 > 300 steps, so no EOS is forced and that utterance ends no beam hypothesis."""
    from tests.test_gpu_greedy_evaluate import golden_labels
    cfg = b200asr.ASRConfig(num_layers=1, num_heads=2, dim_model=64, dim_key=32, dim_value=32, dim_inner=128, vocab=40,
                            feat_extractor="", tgt_max_len=301, dropout=0.0)
    torch.manual_seed(5)
    model = b200asr.build_model(cfg, id2label=golden_labels(40))
    dec = model.decoder
    e = torch.randn(64, generator=torch.Generator().manual_seed(6))
    with torch.no_grad():
        for layer in dec.layers:
            ca = layer.encoder_attn
            ca.value_linear.bias.zero_()
            ca.output_linear.bias.zero_()
            ca.output_linear.weight.mul_(100.0)
            layer.pos_ffn.conv_2.weight.zero_()
            layer.pos_ffn.conv_2.bias.zero_()
        o = ca.output_linear.weight @ (ca.value_linear.weight @ e)
        dec.output_linear.weight[2] = 10.0 * (o - o.mean()) / o.std(unbiased=False)
    return model.cuda().eval().decoder, e


def fallback(b200asr, group):
    from b200asr import modules as M
    dec, e = _fallback_decoder(b200asr)
    out = {}
    for signs in ((1, -1), (1, -1, 1)):              # rank 1 holds utterance 1, the only one that ends no hypothesis
        enc = torch.stack([s * e for s in signs]).view(len(signs), 1, 64).expand(len(signs), 310, 64).contiguous().cuda()
        text = io.StringIO()
        count = _Counted()
        with torch.no_grad(), count(text):
            if group is not None:
                rank = group[1]
                strs = M.decode_sharded(dec, enc[rank::2].contiguous(), enc.shape[0], 310, group, True, 4, None, 0.1, 0.1)
            else:
                strs = dec.beam_search(enc, beam_width=4, nbest=1, c_weight=0.1)[1]
                n_beam = len(strs)
                if n_beam != enc.shape[0]:
                    print(">>>>>>> switch to greedy")
                    strs = dec.greedy_search(enc)
                out[("beam", signs)] = n_beam
        out[signs] = (strs, text.getvalue(), count.collectives)
        if group is not None:
            lengths = M.beam_decode(dec, enc[group[1]::2].contiguous(), 4, nbest=1, c_weight=0.1)[1].cpu()
            out[("lengths", signs)] = lengths.view(-1).tolist()
    return out


def test_fallback_when_only_rank_1_ends_no_hypothesis():
    with tempfile.TemporaryDirectory() as tmp:
        (one,) = _spawn("fallback", 1, tmp)
        r0, r1 = _spawn("fallback", 2, tmp)
    for signs in ((1, -1), (1, -1, 1)):
        assert all(n > 0 for n in r0[("lengths", signs)]) and r1[("lengths", signs)] == [0]     # only rank 1's share fails
        assert one[("beam", signs)] == len(signs) - 1
        strs, text, _ = one[signs]
        assert text == ">>>>>>> switch to greedy\n"
        assert [len(s) for s in strs] == [0 if s > 0 else 300 for s in signs]
        for r in (r0, r1):
            assert r[signs][0] == strs and r[signs][1] == text, signs
            assert r[signs][2] == 2, signs                  # the beam gather, then the greedy one


# ------------------------------------------------------------------------------------------ 4: test.py end to end
def script_arm(b200asr, group):
    import importlib.util
    import numpy as np
    from tests.test_gpu_loader import _model
    from tests.test_loader_host import Env
    with pytest.MonkeyPatch.context() as monkeypatch, tempfile.TemporaryDirectory() as tmp:
        env = Env(monkeypatch)
        ns, model, _ = _model(env, ["--tgt-max-len", "300"])
        spec = importlib.util.spec_from_file_location("reference_test_script", os.path.join(ns.root, "test.py"))
        script = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(script)
        ds = env.dataset(pathlib.Path(tmp), [16000, 8000, 12000, 4000, 9000, 7000, 15000], prob=0.5, src_max_len=90, window="hamming")
        texts = {}
        for beam in (False, True):
            ns.constant.args.src_max_len = 90
            ns.constant.args.beam_search, ns.constant.args.beam_width, ns.constant.args.beam_nbest = beam, 4, 1
            b200asr.install(process_group=group[0] if group else None)
            try:
                np.random.seed(2), torch.manual_seed(2), __import__("random").seed(2)
                loader = env.DL.AudioDataLoader(ds, num_workers=0, batch_sampler=env.DL.BucketingSampler(ds, batch_size=3))
                err, out = io.StringIO(), io.StringIO()
                with contextlib.redirect_stderr(err), contextlib.redirect_stdout(out):
                    script.evaluate(model, loader)
            finally:
                b200asr.uninstall()
            texts[beam] = (re.findall(r"TEST CER:[\d.]+% WER:[\d.]+% CER_EN:[\d.]+% CER_ZH:[\d.]+%", err.getvalue())[-1],
                           out.getvalue())
    return texts


def test_test_py_evaluate_under_two_ranks():
    with tempfile.TemporaryDirectory() as tmp:
        (one,) = _spawn("script_arm", 1, tmp)
        r0, r1 = _spawn("script_arm", 2, tmp)
    print("test.py:", one)
    assert r0 == r1 == one
