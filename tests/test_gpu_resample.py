"""Polyphase resampling on the device (b200asr_resample_packed, features.resample / SpeedPerturb, the installed loader's
speed perturbation and its noise clips at other sample rates).

* Against scipy.signal.resample_poly in float64 at 10/9, 10/11, 2/1, 1/2, 160/441, 147/160 and 1/1, lengths 0, 1, 2,
  shorter than the filter and 10^5: within the fp32 bound of tests/resample_util.py; 1/1 bit for bit.
* quantize16: exactly the 16-bit rounding of the unquantised output.  A mixed-ratio batch equals each utterance run alone
  and a second launch, bit for bit.  NaN-poisoned gaps around every output and between the inputs; the input compared
  bit for bit; one launch per call; rejections launch and write nothing.
* The installed loader with a dataset's speed_perturb against collate_waves(speed_perturb=...) replaying its draws, also
  with TempoGain and SpecAugment; noise clips at 8 and 44.1 kHz served by the device path and equal to the host
  restatement (resample, quantise, cut); no host synchronisation; one Trainer.train iteration; two gloo ranks."""
import os
import tempfile

import numpy as np
import pytest
import scipy.signal
import torch

from oracle import ref_shim
from tests import resample_util as RU
from tests import test_gpu_write_extent as _write_extent

pytestmark = pytest.mark.gpu

# b200asr_resample_packed's write extent is guarded here (_call, test_rejections_launch_and_write_nothing): register it
# with the ABI-wide sweep of tests/test_gpu_write_extent.py, which requires every pointer entry point to be covered or exempted
_write_extent.EXEMPT.setdefault("b200asr_resample_packed", "tests/test_gpu_resample.py: NaN-poisoned gaps and bands around "
                                "every output, NaN between the inputs that must not be read and the input compared bit for "
                                "bit, on every call")

NAN = float("nan")
OK, BAD_SHAPE, BAD_ALIGN, BAD_ARG = 0, -1, -2, -5
GAP = 37
needs_ref = pytest.mark.skipif(not ref_shim.available(), reason="reference checkout not staged (oracle/make_ref.py)")


@pytest.fixture(scope="module")
def L():
    import b200asr
    b200asr._lib.load(check_device=True)
    return b200asr._lib


def _call(L, xs, ratios, quantize16=False, order=None):
    """One raw call: inputs back to back in `order` with NaN gaps, outputs in reverse order in a NaN buffer with NaN gaps
    (checked untouched after the call).  Returns (rc, outputs per utterance, launches)."""
    from b200asr import features as F
    lib = L.load()
    B = len(xs)
    order = list(range(B)) if order is None else order
    offs, pos = [0] * B, GAP
    for b in order:
        offs[b] = pos
        pos += len(xs[b]) + GAP
    buf = np.full(pos, np.nan, np.float32)
    for b in range(B):
        buf[offs[b]:offs[b] + len(xs[b])] = xs[b]
    xin = torch.from_numpy(buf).cuda()
    keep = xin.clone()
    olens = [F.resample_out_length(len(x), u, d) for x, (u, d) in zip(xs, ratios)]
    oo, pos = [0] * B, GAP
    for b in reversed(order):
        oo[b] = pos
        pos += olens[b] + GAP
    out = torch.full((pos,), NAN, device="cuda")
    items = np.zeros(B, F._RESAMPLE_ITEM)
    for b, (u, d) in enumerate(ratios):
        items[b] = (offs[b], oo[b], 0 if u == d == 1 else F._device_taps(u, d, xin.device).data_ptr(), len(xs[b]), u, d, 0)
    items_d = torch.from_numpy(items.view(np.uint8).copy()).cuda()
    n0 = lib.b200asr_launch_count()
    rc = lib.b200asr_resample_packed(L.ptr(xin), xin.numel(), L.ptr(out), out.numel(), items.ctypes.data, L.ptr(items_d), B,
                                     int(quantize16), torch.cuda.current_stream().cuda_stream)
    n = lib.b200asr_launch_count() - n0
    torch.cuda.synchronize()
    assert torch.equal(xin.nan_to_num(7.0), keep.nan_to_num(7.0))
    o = out.cpu().numpy()
    written = np.zeros(len(o), bool)
    for b in range(B):
        written[oo[b]:oo[b] + olens[b]] = True
    assert np.isnan(o[~written]).all(), "a write outside the outputs"
    return rc, [o[oo[b]:oo[b] + olens[b]] for b in range(B)], n


def _lengths(up, down):
    filt = 2 * 10 * max(up, down) + 1
    return [0, 1, 2, filt // 3, filt - 1, 100000]


@pytest.mark.parametrize("up, down", RU.RATIOS)
def test_matches_resample_poly_within_the_fp32_bound(L, up, down):
    g = np.random.default_rng(up * 7 + down)
    xs = [g.uniform(-1, 1, n).astype(np.float32) for n in _lengths(up, down)]
    rc, outs, n = _call(L, xs, [(up, down)] * len(xs), order=g.permutation(len(xs)).tolist())
    assert rc == OK and n == 1, L.last_error()
    for x, y in zip(xs, outs):
        want = scipy.signal.resample_poly(x.astype(np.float64), up, down)
        assert len(y) == len(want)
        if up == down == 1:
            assert np.array_equal(y.view(np.int32), x.view(np.int32))
        else:
            err = np.abs(y.astype(np.float64) - want)
            assert (err <= RU.fp32_bound(x, up, down) + 1e-30).all(), (len(x), err.max())


@pytest.mark.parametrize("up, down", [(10, 9), (10, 11), (160, 441), (2, 1)])
def test_quantize16_is_the_16_bit_rounding(L, up, down):
    g = np.random.default_rng(3)
    xs = [(1.02 * np.sin(np.arange(n) * 0.01) + 0.02 * g.standard_normal(n)).astype(np.float32) for n in (5000, 777, 1)]
    rc, plain, _ = _call(L, xs, [(up, down)] * 3)
    rc2, q, _ = _call(L, xs, [(up, down)] * 3, quantize16=True)
    assert rc == rc2 == OK
    for p, v in zip(plain, q):
        assert np.array_equal(v.view(np.int32), RU.quantize16(p).view(np.int32))
        k = v.astype(np.float64) * 32768
        assert np.array_equal(k, np.rint(k)) and k.min(initial=0) >= -32768 and k.max(initial=0) <= 32767
    assert max(v.max() for v in q) == np.float32(32767 / 32768) and min(v.min() for v in q) == -1.0     # clipped


def test_mixed_batch_equals_each_alone_and_repeats(L):
    g = np.random.default_rng(9)
    ratios = [(10, 9), (1, 1), (10, 11), (160, 441), (2, 1), (1, 2), (147, 160), (10, 11)]
    xs = [g.uniform(-1, 1, int(n)).astype(np.float32) for n in g.integers(0, 60000, len(ratios))]
    rc, batch, n = _call(L, xs, ratios, order=g.permutation(len(xs)).tolist())
    assert rc == OK and n == 1
    rc, again, _ = _call(L, xs, ratios)
    for b, x in enumerate(xs):
        _, alone, _ = _call(L, [x], [ratios[b]])
        assert np.array_equal(batch[b].view(np.int32), alone[0].view(np.int32)), b
        assert np.array_equal(batch[b].view(np.int32), again[b].view(np.int32)), b


def test_rejections_launch_and_write_nothing(L):
    from b200asr import features as F
    lib = L.load()
    x = torch.rand(3000, device="cuda")
    out = torch.full((4000,), NAN, device="cuda")
    taps = F._device_taps(10, 11, x.device)
    st = torch.cuda.current_stream().cuda_stream

    def call(io=0, oo=0, n=3000, up=10, down=11, o=None, n_out=4000):
        items = np.zeros(1, F._RESAMPLE_ITEM)
        items[0] = (io, oo, taps.data_ptr(), n, up, down, 0)
        d = torch.from_numpy(items.view(np.uint8).copy()).cuda()
        n0 = lib.b200asr_launch_count()
        rc = lib.b200asr_resample_packed(L.ptr(x), x.numel(), L.ptr(out) if o is None else o, n_out, items.ctypes.data,
                                         L.ptr(d), 1, 0, st)
        return rc, lib.b200asr_launch_count() - n0

    cases = [(dict(up=20, down=22), BAD_SHAPE), (dict(up=0), BAD_SHAPE), (dict(down=1001), BAD_SHAPE),
             (dict(io=1), BAD_SHAPE), (dict(oo=1300), BAD_SHAPE), (dict(n_out=2000), BAD_SHAPE),
             (dict(o=L.ptr(x) + 400), BAD_ARG), (dict(o=L.ptr(out) + 2), BAD_ALIGN)]
    for kw, code in cases:
        assert call(**kw) == (code, 0), kw
    torch.cuda.synchronize()
    assert bool(out.isnan().all())
    assert call(oo=5) == (OK, 1)
    torch.cuda.synchronize()
    assert not bool(out[5:2733].isnan().any()) and bool(out[:5].isnan().all()) and bool(out[2733:].isnan().all())


# ------------------------------------------------------------------------------------------------------- host layer

def test_host_call_is_the_entry_point(L):
    import b200asr
    g = np.random.default_rng(4)
    xs = [g.uniform(-1, 1, n).astype(np.float32) for n in (16000, 0, 7001, 30000)]
    ups, downs = [10, 7, 20, 2000], [11, 7, 18, 1000]                # reduced on the host: 10/11, 1/1, 10/9, 2/1
    wave = torch.from_numpy(np.concatenate(xs)).cuda()
    offs = np.concatenate([[0], np.cumsum([len(x) for x in xs])[:-1]])
    n0 = L.load().b200asr_launch_count()
    out, oo, ol = b200asr.resample(wave, offs, [len(x) for x in xs], ups, downs)
    assert L.load().b200asr_launch_count() - n0 == 1
    o, oo, ol = out.cpu().numpy(), oo.cpu().numpy(), ol.cpu().numpy()
    _, want, _ = _call(L, xs, [(10, 11), (1, 1), (10, 9), (2, 1)])
    for b in range(4):
        assert ol[b] == len(want[b]) and np.array_equal(o[oo[b]:oo[b] + ol[b]], want[b])
    for bad in (dict(up=[0, 1, 1, 1]), dict(up=[1009, 1, 1, 1]), dict(up=[1, 1, 1])):    # 1009/11: beyond 1000
        with pytest.raises(ValueError):
            b200asr.resample(wave, offs, [len(x) for x in xs], bad.get("up", ups), downs)
    with pytest.raises(ValueError):
        b200asr.resample(wave, torch.tensor(offs).cuda(), [len(x) for x in xs], ups, downs)


def test_collate_waves_without_a_policy_is_unchanged(L):
    import b200asr
    from tests.test_gpu_tempo_gain import _grid_waves
    conf = dict(sample_rate=16000, window_size=0.02, window_stride=0.01, window="hamming")
    batch = [(w, [1, 4, 5]) for w in _grid_waves([16000, 9000, 4001], 5)]
    a = b200asr.collate_waves(batch, conf, 120)
    b = b200asr.collate_waves(batch, conf, 120, speed_perturb=None)
    assert all(torch.equal(u, v) for u, v in zip(a, b))


# ----------------------------------------------------------------------------------------------- the installed loader

@pytest.fixture
def env(monkeypatch):
    from tests.test_loader_host import Env
    return Env(monkeypatch)


LENGTHS = [16000, 8000, 12000, 4000, 9000, 15000, 3000, 11000, 161, 32000, 2560]


class _Replay:
    """An rng that gives back recorded draws: choice() the speed factors' indices, uniform() the tempo and gain values."""

    def __init__(self, picks, uniforms=()):
        self.picks, self.uniforms = list(picks), list(uniforms)

    def choice(self, n):
        return self.picks.pop(0)

    def uniform(self, low, high):
        return self.uniforms.pop(0)


def _record(monkeypatch):
    """Records the factor index and the tempo / gain values every SpeedPerturb / TempoGain draw makes."""
    from b200asr import features as F
    picks, uniforms = [], []
    sp, tg = F.SpeedPerturb.draw_one, F.TempoGain.draw_one
    monkeypatch.setattr(F.SpeedPerturb, "draw_one", lambda s, rng=np.random: (lambda f: (picks.append(s.factors.index(f)), f)[1])(sp(s, rng)))
    monkeypatch.setattr(F.TempoGain, "draw_one", lambda s, rng=np.random: (lambda d: (uniforms.extend(d), d)[1])(tg(s, rng)))
    return picks, uniforms


@needs_ref
@pytest.mark.parametrize("tempo", [False, True])
@pytest.mark.parametrize("spec", [False, True])
def test_installed_loader_is_collate_waves_with_the_policy(env, tmp_path, monkeypatch, tempo, spec):
    """The installed loader's batches equal collate_waves(speed_perturb=...) over the items its workers made, replaying
    their draws, bit for bit, also with TempoGain and SpecAugment; one launch more per batch than without the policy."""
    import b200asr
    from b200asr import loader
    from tests.tempo_gain_util import grid16
    ds = env.dataset(tmp_path, LENGTHS[:8], prob=None, augment=tempo, src_max_len=90)
    for w in list(env.utts):
        env.utts[w] = grid16(env.utts[w])
    ds.speed_perturb = b200asr.SpeedPerturb()
    if tempo:
        ds.tempo_gain = b200asr.TempoGain()
    if spec:
        ds.spec_augment = b200asr.SpecAugment(W=5, Fp=10, n_freq_masks=1, Tp=10, p=1.0, n_time_masks=1, seed=7)
    items = []
    collate = loader.collate_items
    monkeypatch.setattr(loader, "collate_items", lambda its: (items.append([(it.wave, it.ids) for it in its]), collate(its))[1])
    picks, uniforms = _record(monkeypatch)
    b200asr.install()
    try:
        np.random.seed(1), torch.manual_seed(1), __import__("random").seed(1)
        got = [tuple(t.clone() for t in b)
               for b in env.DL.AudioDataLoader(ds, num_workers=0, batch_sampler=env.DL.BucketingSampler(ds, batch_size=3))]
    finally:
        b200asr.uninstall()
    assert len(got) == len(items) == 3 and len(picks) == 8 and len(set(picks)) > 1
    conf = dict(sample_rate=16000, window_size=0.02, window_stride=0.01, window="hamming")
    ref_aug = b200asr.SpecAugment(W=5, Fp=10, n_freq_masks=1, Tp=10, p=1.0, n_time_masks=1, seed=7) if spec else None
    k, launches = 0, []
    for g, its in zip(got, items):
        rng = _Replay(picks[k:k + len(its)], uniforms[2 * k:2 * (k + len(its))])
        n0 = b200asr._lib.load().b200asr_launch_count()
        want = b200asr.collate_waves(its, conf, 90, rng=rng, speed_perturb=b200asr.SpeedPerturb(), spec_augment=ref_aug,
                                     tempo_gain=b200asr.TempoGain() if tempo else None)
        launches.append(b200asr._lib.load().b200asr_launch_count() - n0)
        k += len(its)
        assert all(torch.equal(u.cpu(), v.cpu()) for u, v in zip(g, want))
    n0 = b200asr._lib.load().b200asr_launch_count()
    b200asr.collate_waves(items[0], conf, 90, rng=_Replay([], uniforms[:6]), tempo_gain=b200asr.TempoGain() if tempo else None,
                          spec_augment=b200asr.SpecAugment(W=5, Fp=10, n_freq_masks=1, Tp=10, p=1.0, n_time_masks=1, seed=7) if spec else None)
    assert launches == [b200asr._lib.load().b200asr_launch_count() - n0 + 1] * 3


def _noise_env(env, rates):
    """Clips 0 and 2 recorded at other rates: their samples are the clip at that rate (len / rate seconds)."""
    from tests.tempo_gain_util import grid16
    names = sorted(env.clips)
    for name, r in zip(names, rates):
        if r != 16000:
            env.clips[name] = grid16(0.3 * np.sin(np.arange(int(len(env.clips[name]) * r / 16000)) * 0.013 * 16000 / r))
            env.rates[name] = r
    return names


@needs_ref
@pytest.mark.parametrize("speed", [False, True])
def test_noise_clips_at_other_rates_use_the_device_path(env, tmp_path, monkeypatch, speed):
    """Clips at 8 and 44.1 kHz on a dataset with resample_noise = True: the installed loader keeps its own path (no reference iterator, no sox); its bank holds
    each such clip resampled to 16 kHz and quantised (the host restatement, within one step of the 16-bit grid where fp32
    and float64 round a half step apart), the draws use each clip's own duration, and its batches equal collate_waves
    over the same draws (the workers' numpy state replayed), with SpeedPerturb and TempoGain too."""
    import b200asr
    from b200asr import loader
    rates = [8000, 16000, 44100]
    names = _noise_env(env, rates)
    ds = env.dataset(tmp_path, LENGTHS[:6], prob=1.0, augment=speed, src_max_len=90)
    ds.resample_noise = True
    if speed:
        ds.speed_perturb, ds.tempo_gain = b200asr.SpeedPerturb(), b200asr.TempoGain()
    monkeypatch.setattr(env.DL, "audio_with_sox", _raise)
    monkeypatch.setattr(env.audio, "augment_audio_with_sox", _raise)
    items, states = [], []
    collate, getitem = loader.collate_items, loader.PackedItems.__getitem__
    monkeypatch.setattr(loader, "collate_items", lambda its: (items.append(list(its)), collate(its))[1])
    monkeypatch.setattr(loader.PackedItems, "__getitem__", lambda s, i: (states.append(np.random.get_state()), getitem(s, i))[1])
    b200asr.install()
    try:
        np.random.seed(2), torch.manual_seed(2), __import__("random").seed(2)
        dl = env.DL.AudioDataLoader(ds, num_workers=0, batch_sampler=env.DL.BucketingSampler(ds, batch_size=3))
        got = [tuple(t.clone() for t in b) for b in dl]
        packed = dl._b200asr_packed
    finally:
        b200asr.uninstall()
    assert not packed.reference and len(got) == 2
    bank = packed.bank
    for c, (name, r) in enumerate(zip(names, rates)):
        x = env.clips[name]
        up, down = b200asr.features.resample_ratio(16000, r)
        want = x if r == 16000 else RU.quantize16(scipy.signal.resample_poly(x.astype(np.float64), up, down))
        clip = bank.bank[bank.offsets[c]:bank.offsets[c] + bank.lengths[c]].cpu().numpy()
        assert len(clip) == len(want) and np.abs(clip - want).max() <= 1 / 32768, r
        assert r == 16000 or np.array_equal(clip, RU.quantize16(clip))
        assert bank.clips.durations[c] == len(x) / r
    assert {it.noise_clip for its in items for it in its} & {0, 2}
    conf = dict(sample_rate=16000, window_size=0.02, window_stride=0.01, window="hamming", noise_dir=str(tmp_path),
                noise_prob=1.0, noise_levels=(0.0, 0.5))
    k = 0
    for g, its in zip(got, items):
        rng = np.random.RandomState()
        rng.set_state(states[k])
        want = b200asr.collate_waves([(it.wave, it.ids) for it in its], conf, 90, noise_bank=bank, rng=rng,
                                     speed_perturb=ds.speed_perturb if speed else None,
                                     tempo_gain=ds.tempo_gain if speed else None)
        k += len(its)
        assert all(torch.equal(u.cpu(), v.cpu()) for u, v in zip(g, want))


def _raise(*a, **k):
    raise AssertionError("sox was called")


@needs_ref
@pytest.mark.parametrize("workers", [0, 2])
def test_installed_loader_makes_no_host_sync(env, tmp_path, monkeypatch, workers):
    import b200asr
    _noise_env(env, [8000, 16000, 44100])
    ds = env.dataset(tmp_path, [16000, 8000, 12000, 4000] * 4, prob=0.5, augment=True)
    ds.speed_perturb, ds.tempo_gain, ds.resample_noise = b200asr.SpeedPerturb(), b200asr.TempoGain(), True
    b200asr.install()
    try:
        it = iter(env.DL.AudioDataLoader(ds, num_workers=workers, batch_size=4))
        next(it)
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            for _ in range(3):
                next(it)
        finally:
            torch.cuda.set_sync_debug_mode("default")
    finally:
        b200asr.uninstall()


@needs_ref
def test_trainer_iteration_trains_with_speed_perturbation(env, tmp_path):
    """One Trainer.train iteration of the bound reference loop over an installed loader whose dataset carries the policy
    and takes noise from clips at 8 and 44.1 kHz: finite losses, every parameter with a gradient moved."""
    import b200asr
    from tests.test_gpu_linear_precisions import _waves
    from tests.test_gpu_loader import _model
    _noise_env(env, [8000, 16000, 44100])
    ds = env.dataset(tmp_path, LENGTHS[:3], prob=0.5, src_max_len=90)
    ds.speed_perturb, ds.resample_noise = b200asr.SpeedPerturb(), True
    valid = [b200asr.collate_waves([(w, [1, 4, 5, 2]) for w in _waves([7000, 5000], seed=3)],
                                   dict(sample_rate=16000, window_size=0.02, window_stride=0.01, window="hamming"), 90)]
    ns, model, i2l = _model(env)
    ns.constant.args.src_max_len, ns.constant.args.save_folder, ns.constant.args.name = 90, str(tmp_path), "speed"
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
    assert len(losses) == 2 and all(np.isfinite(losses)), losses
    graded = [k for k, v in model.named_parameters() if v.grad is not None and bool(v.grad.abs().sum() > 0)]
    assert graded and all(not torch.equal(dict(model.named_parameters())[k], before[k]) for k in graded)


def _rank(rank, world, port, tmp):
    import pathlib
    import torch.distributed as dist
    import b200asr
    from b200asr import parallel
    from tests.test_loader_host import Env
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    mp = pytest.MonkeyPatch()
    try:
        env = Env(mp)
        _noise_env(env, [8000, 16000, 44100])
        d = pathlib.Path(tmp) / f"r{rank}"
        d.mkdir()
        ds = env.dataset(d, LENGTHS + [7000, 6000, 14000, 5000], prob=0.5, src_max_len=90)
        ds.speed_perturb, ds.resample_noise = b200asr.SpeedPerturb(), True
        __import__("random").seed(100 + rank)                 # different until the ranks agree on a seed
        np.random.seed(100 + rank)
        b200asr.install(process_group=dist.group.WORLD)
        try:
            parallel.seed_host_rngs(dist.group.WORLD)          # what the bound Trainer.train does before its epochs
            loader = env.DL.AudioDataLoader(ds, num_workers=0, batch_sampler=env.DL.BucketingSampler(ds, batch_size=4))
            got = [[t.cpu().clone() for t in b] for _ in range(2) for b in loader]      # two epochs
        finally:
            b200asr.uninstall()
        torch.save(dict(batches=got), os.path.join(tmp, f"rank{rank}.pt"))
    finally:
        mp.undo()
        dist.barrier()
        dist.destroy_process_group()


@needs_ref
def test_two_gloo_ranks_see_the_same_perturbed_batches():
    import socket
    import torch.multiprocessing as mp
    with tempfile.TemporaryDirectory() as tmp:
        s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
        mp.start_processes(_rank, args=(2, port, tmp), nprocs=2, join=True, start_method="spawn")
        r0, r1 = (torch.load(os.path.join(tmp, f"rank{r}.pt"), weights_only=False) for r in range(2))
    assert len(r0["batches"]) == len(r1["batches"]) == 8
    for a, b in zip(r0["batches"], r1["batches"]):
        assert all(torch.equal(u, v) for u, v in zip(a, b))
    assert not torch.equal(r0["batches"][0][0], r0["batches"][4][0])      # epoch 2 draws anew
