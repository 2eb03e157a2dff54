"""SpecAugment on the device (b200asr_spec_augment, features.SpecAugment, the installed loader's opt-in).

* The draws output equals the host restatement of the counter generator (tests/spec_augment_util.py) exactly.
* The output equals a float64 restatement of warp + masks from those draws: bit for bit where no interpolation happens,
  within 2^-22 (|x[i0]| + |x[i0 + 1]|) where the warp interpolates (one rounding each of the weight, the difference and
  the fma); masked and padding elements are exactly 0.  F = 161 and odd F, T_b of 1, 2, 2W + 1, 2W + 2 and long, every
  degenerate warp segment and overlapping masks.
* NaN-poisoned outputs between sentinel bands, NaN input padding that must not be read, the input left untouched.
* Repeated calls give identical bits; another counter other draws.  Rejections launch and write nothing; a call is one
  launch.
* spectrogram_batch / collate_waves with spec_augment=None are the calls without it; the installed loader with a
  dataset's spec_augment equals collate_waves + SpecAugment.apply; one Trainer.train iteration trains with it; two gloo
  ranks on one GPU see the same augmented batches."""
import os
import tempfile

import numpy as np
import pytest
import torch

from oracle import ref_shim
from tests import spec_augment_util as SA
from tests import test_gpu_write_extent as _write_extent
from tests.test_gpu_linear_precisions import Banded, _waves

pytestmark = pytest.mark.gpu

# b200asr_spec_augment's write extent is guarded here (_call, test_rejections_launch_and_write_nothing): register it with the
# ABI-wide sweep of tests/test_gpu_write_extent.py, which requires every pointer entry point to be covered or exempted
_write_extent.EXEMPT.setdefault("b200asr_spec_augment", "tests/test_gpu_spec_augment.py: NaN-poisoned output between "
                                "sentinel bands (also off the 16-byte grid), draws between sentinel guards, NaN input "
                                "padding that must not be read and the input compared bit for bit, on every call")

NAN = float("nan")
OK, BAD_SHAPE, BAD_ALIGN, BAD_ARG = 0, -1, -2, -5
SENT = -777
needs_ref = pytest.mark.skipif(not ref_shim.available(), reason="reference checkout not staged (oracle/make_ref.py)")


@pytest.fixture(scope="module")
def L():
    import b200asr
    b200asr._lib.load(check_device=True)
    return b200asr._lib


def _input(sizes, F, T, seed):
    """[B,1,F,T] normalised-looking features, NaN past each utterance's frames (the kernel must not read them)."""
    g = np.random.default_rng(seed)
    x = g.standard_normal((len(sizes), 1, F, T)).astype(np.float32) * 2.0 + 0.25
    for b, n in enumerate(sizes):
        x[b, :, :, min(max(n, 0), T):] = NAN
    return x


def _call(L, x, sizes, W, Fp, nf, Tp, p, nt, seed, counter, shift=0):
    """One raw call: output between sentinel bands (NaN inside), draws inside a sentinel-filled int buffer.  Returns
    (rc, out, draws, launches); checks the bands, the draws buffer's guards and that the input is untouched."""
    lib = L.load()
    B, _, F, T = x.shape
    xin = torch.from_numpy(x).cuda()
    keep = xin.clone()
    frames = torch.tensor(sizes, dtype=torch.int32, device="cuda")
    out = Banded((B, 1, F, T), shift=shift)
    nd = lib.b200asr_spec_augment_draws_ints(nf, nt) or 1
    dbuf = torch.full((B * nd + 64,), SENT, dtype=torch.int32, device="cuda")
    draws = dbuf[32:32 + B * nd].view(B, nd)
    n0 = lib.b200asr_launch_count()
    rc = lib.b200asr_spec_augment(L.ptr(xin), L.ptr(out.t), L.ptr(draws), L.ptr(frames), B, F, T, W, Fp, nf, Tp, p, nt, seed, counter,
                                  torch.cuda.current_stream().cuda_stream)
    n = lib.b200asr_launch_count() - n0
    torch.cuda.synchronize()
    assert out.bands_intact() and bool((dbuf[:32] == SENT).all()) and bool((dbuf[32 + B * nd:] == SENT).all())
    assert torch.equal(xin.nan_to_num(7.0), keep.nan_to_num(7.0))
    return rc, out.t.cpu().numpy(), draws.cpu().numpy(), n


def _check(L, sizes, F, T, W, Fp, nf, Tp, p, nt, seed, counter, shift=0):
    x = _input(sizes, F, T, seed * 1000 + counter)
    rc, out, drw, n = _call(L, x, sizes, W, Fp, nf, Tp, p, nt, seed, counter, shift)
    assert rc == OK and n == 1, L.last_error()
    want = SA.draws(sizes, F, T, W, Fp, nf, Tp, p, nt, seed, counter)
    assert np.array_equal(drw, want)
    ref, zero, bound = SA.reference(np.nan_to_num(x, nan=0.0), drw, sizes, nf, nt)
    assert (out[zero] == 0).all()
    exact = ~zero & (bound == 0)
    assert np.array_equal(out[exact], ref[exact].astype(np.float32))
    interp = ~zero & (bound > 0)
    assert (np.abs(out[interp].astype(np.float64) - ref[interp]) <= bound[interp]).all()
    return drw, out, x


W = 4


def _segments(drw, sizes):
    """Kinds of warp met: 'none', 'shift', 'd=0', 'd=T_b-1'."""
    kinds = set()
    for b, Tb in enumerate(sizes):
        c, w = int(drw[b, 0]), int(drw[b, 1])
        if w == 0:
            kinds.add("none")
        else:
            kinds.add("d=0" if c + w == 0 else "d=T_b-1" if c + w == Tb - 1 else "shift")
    return kinds


@pytest.mark.parametrize("F", [161, 7])
def test_draws_and_output_match_the_float64_restatement(L, F):
    """T_b of 1, 2, 2W + 1, 2W + 2, 2W + 3, long and 0 (an empty utterance), over 40 counters: every warp segment kind
    (both degenerate ones included, which the short utterances meet often) and overlapping masks are met."""
    sizes = [1, 2, 2 * W + 1, 2 * W + 2, 2 * W + 3, 2 * W + 2, 1601, 777, 0, 2 * W + 2]
    T = 1601
    kinds, overlap = set(), False
    for counter in range(40):
        drw, _, _ = _check(L, sizes, F, T, W, min(F, 27), 3, 40, 1.0, 3, seed=5, counter=counter)
        kinds |= _segments(drw, sizes)
        for b in range(len(sizes)):
            fm = [(drw[b, 2 + 2 * m + 1], drw[b, 2 + 2 * m]) for m in range(3)]
            overlap |= any(a0 < b0 + bw and b0 < a0 + aw and aw and bw for i, (a0, aw) in enumerate(fm) for (b0, bw) in fm[i + 1:])
    assert kinds == {"none", "shift", "d=0", "d=T_b-1"}, kinds
    assert overlap


@pytest.mark.parametrize("case", ["no-masks", "p0", "full-masks", "W0", "unaligned", "sizes-past-T"])
def test_policy_edges(L, case):
    F, T = 161, 300
    sizes = [300, 150, 9, 1]
    kw = dict(W=5, Fp=27, nf=2, Tp=50, p=0.5, nt=2)
    shift = 0
    if case == "no-masks":
        kw.update(nf=0, nt=0)
    elif case == "p0":
        kw.update(p=0.0)
    elif case == "full-masks":
        kw.update(Fp=F, Tp=T, p=1.0, nf=64, nt=64)
    elif case == "W0":
        kw.update(W=0)
    elif case == "unaligned":
        shift = 1
    else:
        sizes = [400, -3, 300, 2]                    # frames are clamped to [0, T]
    drw, out, _ = _check(L, sizes, F, T, seed=9, counter=3, shift=shift, **kw)
    if case == "p0":
        assert not drw[:, 2 + 2 * kw["nf"]::2].any()
    if case == "W0":
        assert not drw[:, 1].any()
    if case == "full-masks":
        assert (out == 0).mean() > 0.5


def test_repeated_calls_are_bit_identical_and_counters_differ(L):
    sizes, F, T = [1000, 640, 333, 57], 161, 1000
    x = _input(sizes, F, T, 3)
    a = _call(L, x, sizes, 40, 27, 2, 100, 1.0, 2, 11, 7)
    b = _call(L, x, sizes, 40, 27, 2, 100, 1.0, 2, 11, 7)
    c = _call(L, x, sizes, 40, 27, 2, 100, 1.0, 2, 11, 8)
    d = _call(L, x, sizes, 40, 27, 2, 100, 1.0, 2, 12, 7)
    assert np.array_equal(a[1].view(np.int32), b[1].view(np.int32)) and np.array_equal(a[2], b[2])
    assert not np.array_equal(a[2], c[2]) and not np.array_equal(a[2], d[2])
    assert not np.array_equal(a[1], c[1])


def test_rejections_launch_and_write_nothing(L):
    lib = L.load()
    B, F, T = 2, 9, 16
    xin = torch.randn(B, 1, F, T, device="cuda")
    frames = torch.tensor([16, 10], dtype=torch.int32, device="cuda")
    out = Banded((B, 1, F, T))
    draws = torch.full((B * 6 + 2,), SENT, dtype=torch.int32, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    base = dict(i=L.ptr(xin), o=L.ptr(out.t), d=L.ptr(draws), f=L.ptr(frames), B=B, F=F, T=T, W=2, Fp=3, nf=1, Tp=4, p=1.0, nt=1)

    def call(**kw):
        a = dict(base, **kw)
        n0 = lib.b200asr_launch_count()
        rc = lib.b200asr_spec_augment(a["i"], a["o"], a["d"], a["f"], a["B"], a["F"], a["T"], a["W"], a["Fp"], a["nf"],
                                      a["Tp"], a["p"], a["nt"], 1, 0, st)
        return rc, lib.b200asr_launch_count() - n0

    cases = [(dict(i=None), BAD_ARG), (dict(o=None), BAD_ARG), (dict(d=None), BAD_ARG), (dict(f=None), BAD_ARG),
             (dict(i=base["i"] + 2), BAD_ALIGN), (dict(o=base["o"] + 2), BAD_ALIGN), (dict(d=base["d"] + 1), BAD_ALIGN),
             (dict(f=base["f"] + 2), BAD_ALIGN), (dict(B=0), BAD_SHAPE), (dict(F=0), BAD_SHAPE), (dict(T=0), BAD_SHAPE),
             (dict(B=70000), BAD_SHAPE), (dict(W=-1), BAD_ARG), (dict(Fp=10), BAD_ARG), (dict(Fp=-1), BAD_ARG),
             (dict(Tp=-1), BAD_ARG), (dict(p=-0.01), BAD_ARG), (dict(p=1.5), BAD_ARG), (dict(p=NAN), BAD_ARG),
             (dict(nf=-1), BAD_ARG), (dict(nf=65), BAD_ARG), (dict(nt=-2), BAD_ARG), (dict(nt=65), BAD_ARG),
             (dict(o=base["i"]), BAD_ARG), (dict(o=base["i"] + 4 * 5), BAD_ARG), (dict(i=base["o"] + 4 * 100), BAD_ARG)]
    for kw, code in cases:
        assert call(**kw) == (code, 0), kw
    torch.cuda.synchronize()
    assert bool(out.t.isnan().all()) and out.bands_intact() and bool((draws == SENT).all())
    assert call() == (OK, 1)
    torch.cuda.synchronize()
    assert not bool(out.t.isnan().any()) and out.bands_intact() and bool((draws[12:] == SENT).all())


# ------------------------------------------------------------------------------------------------------- host layer

def test_policy_apply_matches_the_entry_point_and_advances_its_counter(L):
    import b200asr
    sizes, F, T = [500, 321, 40], 161, 500
    x = np.nan_to_num(_input(sizes, F, T, 4), nan=0.0)
    aug = b200asr.SpecAugment(20, 27, 2, 60, 0.4, 2, seed=99)
    aug.counter = 5
    got, drw = aug.apply(torch.from_numpy(x).cuda(), torch.tensor(sizes, dtype=torch.int32))      # host sizes
    assert aug.counter == 6
    rc, out, want, _ = _call(L, x, sizes, 20, 27, 2, 60, 0.4, 2, 99, 5)
    assert rc == OK and np.array_equal(drw.cpu().numpy(), want) and np.array_equal(got.cpu().numpy().view(np.int32), out.view(np.int32))
    got2, _ = aug.apply(torch.from_numpy(x).cuda(), torch.tensor(sizes, dtype=torch.int32, device="cuda"))
    assert aug.counter == 7 and not torch.equal(got, got2)
    with pytest.raises(ValueError, match="Fp"):
        b200asr.SpecAugment(2, 27, 1, 5, 1.0, 1, seed=0).apply(torch.zeros(1, 1, 9, 8, device="cuda"), torch.tensor([8]))


def test_helpers_without_a_policy_are_unchanged(L):
    import b200asr
    waves = [torch.from_numpy(w).cuda() for w in _waves([16000, 9000, 4001], seed=5)]
    a = b200asr.spectrogram_batch(waves, max_frames=90)
    b = b200asr.spectrogram_batch(waves, max_frames=90, spec_augment=None)
    assert all(torch.equal(u, v) for u, v in zip(a, b))
    aug = b200asr.SpecAugment(10, 27, 2, 30, 1.0, 2, seed=4)
    c = b200asr.spectrogram_batch(waves, max_frames=90, spec_augment=aug)
    assert aug.counter == 1 and torch.equal(c[1], a[1]) and torch.equal(c[2], a[2])
    aug.counter = 0
    assert torch.equal(c[0], aug.apply(a[0], a[2])[0])
    conf = dict(sample_rate=16000, window_size=0.02, window_stride=0.01, window="hamming")
    batch = [(w.cpu().numpy(), [1, 4, 5]) for w in waves]
    a = b200asr.collate_waves(batch, conf, 120)
    b = b200asr.collate_waves(batch, conf, 120, spec_augment=None)
    assert all(torch.equal(u, v) for u, v in zip(a, b))
    aug.counter = 3
    c = b200asr.collate_waves(batch, conf, 120, spec_augment=aug)
    aug.counter = 3
    assert all(torch.equal(u, v) for u, v in zip(c[1:], a[1:])) and torch.equal(c[0], aug.apply(a[0], a[3])[0])


# ----------------------------------------------------------------------------------------------- the installed loader

@pytest.fixture
def env(monkeypatch):
    from tests.test_loader_host import Env
    return Env(monkeypatch)


LENGTHS = [16000, 8000, 12000, 4000, 9000, 15000, 3000, 11000]


def _policy(seed=21):
    import b200asr
    return b200asr.SpecAugment(12, 27, 2, 30, 0.5, 2, seed=seed)


@needs_ref
def test_installed_loader_applies_the_datasets_policy(env, tmp_path, monkeypatch):
    """With the attribute: collate_waves + SpecAugment.apply on the items the loader made, bit for bit, and the counter
    restarted at 0 by the loader and advanced once per batch.  Without it: collate_waves alone, bit for bit."""
    import b200asr
    from b200asr import loader
    ds = env.dataset(tmp_path, LENGTHS, prob=None, src_max_len=90)
    items = []
    collate = loader.collate_items
    monkeypatch.setattr(loader, "collate_items", lambda its: (items.append([(it.wave, it.ids) for it in its]), collate(its))[1])
    conf = dict(sample_rate=16000, window_size=0.02, window_stride=0.01, window="hamming")
    for attr in (True, False):
        if attr:
            ds.spec_augment = _policy()
            ds.spec_augment.counter = 41                        # building the loader restarts it
        else:
            del ds.spec_augment
        items.clear()
        b200asr.install()
        try:
            np.random.seed(1), torch.manual_seed(1), __import__("random").seed(1)
            got = [tuple(t.clone() for t in b) for b in
                   env.DL.AudioDataLoader(ds, num_workers=0, batch_sampler=env.DL.BucketingSampler(ds, batch_size=3))]
        finally:
            b200asr.uninstall()
        assert len(got) == len(items) == 3
        ref = _policy() if attr else None
        for g, its in zip(got, items):
            want = b200asr.collate_waves(its, conf, 90, spec_augment=ref)
            assert all(torch.equal(u.cpu(), v.cpu()) for u, v in zip(g, want))
        if attr:
            assert ds.spec_augment.counter == ref.counter == 3


@needs_ref
def test_trainer_iteration_trains_with_augmentation(env, tmp_path):
    """One Trainer.train iteration of the bound reference loop over an installed loader whose dataset carries a policy:
    finite loss, every parameter with a nonzero gradient moved, one batch augmented."""
    import b200asr
    from tests.test_gpu_loader import _model
    ds = env.dataset(tmp_path, LENGTHS[:3], prob=None, src_max_len=90)
    ds.spec_augment = _policy()
    valid = [b200asr.collate_waves([(w, [1, 4, 5, 2]) for w in _waves([7000, 5000], seed=3)],
                                   dict(sample_rate=16000, window_size=0.02, window_stride=0.01, window="hamming"), 90)]
    ns, model, i2l = _model(env)
    ns.constant.args.src_max_len, ns.constant.args.save_folder, ns.constant.args.name = 90, str(tmp_path), "aug"
    opt = ns.functions.init_optimizer(ns.constant.args, model, "noam")
    before = {k: v.detach().clone() for k, v in model.named_parameters()}
    losses = []
    b200asr.install()
    cur = ns.trainer.calculate_metrics
    ns.trainer.calculate_metrics = lambda *a, **k: (lambda out: (losses.append(float(out[0].item())), out)[1])(cur(*a, **k))
    try:
        train = env.DL.AudioDataLoader(ds, num_workers=0, batch_sampler=env.DL.BucketingSampler(ds, batch_size=3))
        ns.trainer.Trainer().train(model, train, None, [valid], opt, "ce", 0, 1, env.label2id, i2l)
    finally:
        ns.trainer.calculate_metrics = cur
        b200asr.uninstall()
    assert ds.spec_augment.counter == 1 and len(losses) == 2 and all(np.isfinite(losses)), losses
    graded = [k for k, v in model.named_parameters() if v.grad is not None and bool(v.grad.abs().sum() > 0)]
    assert graded and all(not torch.equal(dict(model.named_parameters())[k], before[k]) for k in graded)


def _rank(rank, world, port, tmp):
    import torch.distributed as dist
    import b200asr
    from b200asr import parallel
    from tests.test_loader_host import Env
    import pathlib
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    mp = pytest.MonkeyPatch()
    try:
        env = Env(mp)
        d = pathlib.Path(tmp) / f"r{rank}"
        d.mkdir()
        ds = env.dataset(d, LENGTHS + [7000, 6000, 14000, 5000], prob=None, src_max_len=90)
        ds.spec_augment = _policy(seed=5)
        __import__("random").seed(100 + rank)                 # different until the ranks agree on a seed
        b200asr.install(process_group=dist.group.WORLD)
        try:
            parallel.seed_host_rngs(dist.group.WORLD)          # what the bound Trainer.train does before its epochs
            loader = env.DL.AudioDataLoader(ds, num_workers=0, batch_sampler=env.DL.BucketingSampler(ds, batch_size=4))
            got = [[t.cpu().clone() for t in b] for _ in range(2) for b in loader]      # two epochs
        finally:
            b200asr.uninstall()
        torch.save(dict(batches=got, counter=ds.spec_augment.counter), os.path.join(tmp, f"rank{rank}.pt"))
    finally:
        mp.undo()
        dist.barrier()
        dist.destroy_process_group()


@needs_ref
def test_two_gloo_ranks_see_the_same_augmented_batches():
    import socket
    import torch.multiprocessing as mp
    with tempfile.TemporaryDirectory() as tmp:
        s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
        mp.start_processes(_rank, args=(2, port, tmp), nprocs=2, join=True, start_method="spawn")
        r0, r1 = (torch.load(os.path.join(tmp, f"rank{r}.pt"), weights_only=False) for r in range(2))
    assert r0["counter"] == r1["counter"] == len(r0["batches"]) == 6
    for a, b in zip(r0["batches"], r1["batches"]):
        assert all(torch.equal(u, v) for u, v in zip(a, b))
    assert not torch.equal(r0["batches"][0][0], r0["batches"][3][0])      # epoch 2 draws anew
