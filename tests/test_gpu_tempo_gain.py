"""Tempo and gain perturbation on the device (b200asr_tempo_gain, features.tempo_gain / TempoGain, the installed loader's
opt-in for augment=True datasets).

* On 16-bit-grid inputs the picks and the output equal the numpy restatement (tests/tempo_gain_util.py) bit for bit: at
  8, 16 and 48 kHz, tempos 0.85, 1.0, 1.15 and random draws, gains -6 to +8 dB (clipping included), lengths 0, 1, below
  a segment, around multiples of the step and 16 s, in batches whose offsets lie in another order than the utterances.
* On off-grid fp32 inputs every pick's float64 D is within 1e-12 (D_min + sum prev^2) of the restatement's minimum given
  the kernel's previous pick, and the output is the restatement replayed on the kernel's picks, bit for bit.
* NaN-poisoned gaps between the outputs and sentinel-guarded picks; NaN between the inputs, which must not be read; one
  launch per call; identical bits on a second call; rejections launch and write nothing; a bad device tempo or offset
  gives NaN.
* The installed loader with a dataset's tempo_gain against the reference's own loader with sox restated, against
  collate_waves(tempo_gain=...), without host synchronisation, through one Trainer.train iteration with sox raising; a
  dataset without the policy yields the bits and launches of collate_waves without it."""
import numpy as np
import pytest
import torch

from oracle import ref_shim
from tests import tempo_gain_util as TG
from tests import test_gpu_write_extent as _write_extent
from tests.helpers import rel_err

pytestmark = pytest.mark.gpu

# b200asr_tempo_gain's write extent is guarded here (_call, test_rejections_launch_and_write_nothing): register it with the
# ABI-wide sweep of tests/test_gpu_write_extent.py, which requires every pointer entry point to be covered or exempted
_write_extent.EXEMPT.setdefault("b200asr_tempo_gain", "tests/test_gpu_tempo_gain.py: NaN-poisoned gaps and bands around "
                                "every output, sentinel-guarded picks, NaN between the inputs that must not be read and "
                                "the input compared bit for bit, on every call")

NAN = float("nan")
OK, BAD_SHAPE, BAD_ALIGN, BAD_ARG = 0, -1, -2, -5
SENT = -777
GAP = 37                                     # NaN floats around and between the inputs and outputs
BAR = 5e-5                                   # tests/test_gpu_loader.py's bar for the installed loader
needs_ref = pytest.mark.skipif(not ref_shim.available(), reason="reference checkout not staged (oracle/make_ref.py)")


@pytest.fixture(scope="module")
def L():
    import b200asr
    b200asr._lib.load(check_device=True)
    return b200asr._lib


def _call(L, xs, tempos, gains, sr, order=None, in_offsets=None, out_offsets=None, geom=None):
    """One raw call: inputs back to back in `order` with NaN gaps, outputs at their offsets in a NaN buffer with NaN gaps
    (checked untouched after the call), picks in a sentinel-filled buffer with guards.  Returns (rc, outputs, picks,
    launches), outputs and picks per utterance."""
    lib = L.load()
    B = len(xs)
    geom = TG.geometry(sr) if geom is None else geom
    step = geom[0] - geom[2]
    order = list(range(B)) if order is None else order
    lens = [len(x) for x in xs]
    offs, pos = [0] * B, GAP
    for b in order:
        offs[b] = pos
        pos += lens[b] + GAP
    buf = np.full(pos, np.nan, np.float32)
    for b in range(B):
        buf[offs[b]:offs[b] + lens[b]] = xs[b]
    xin = torch.from_numpy(buf).cuda()
    keep = xin.clone()
    olens = [TG.out_length(n, t) if np.isfinite(t) and t > 0 else n for n, t in zip(lens, tempos)]
    oo, pos = [0] * B, GAP
    for b in reversed(order):
        oo[b] = pos
        pos += olens[b] + GAP
    out = torch.full((pos,), NAN, device="cuda")
    K = [-(-m // step) for m in olens]
    po = np.concatenate([[32], 32 + np.cumsum(K)[:-1]]).astype(np.int64)
    pk = torch.full((sum(K) + 64,), SENT, dtype=torch.int32, device="cuda")
    dev = lambda a, dt: torch.tensor(a, dtype=dt, device="cuda")  # noqa: E731
    args = [dev(offs if in_offsets is None else in_offsets, torch.int64), dev(lens, torch.int32),
            dev(tempos, torch.float64), dev([TG.linear_gain(g) for g in gains], torch.float32)]
    o_args = [dev(oo if out_offsets is None else out_offsets, torch.int64), dev(olens, torch.int32), pk, dev(po, torch.int64)]
    n0 = lib.b200asr_launch_count()
    rc = lib.b200asr_tempo_gain(L.ptr(xin), *[L.ptr(a) for a in args], L.ptr(out), *[L.ptr(a) for a in o_args], B, *geom,
                                torch.cuda.current_stream().cuda_stream)
    n = lib.b200asr_launch_count() - n0
    torch.cuda.synchronize()
    assert torch.equal(xin.nan_to_num(7.0), keep.nan_to_num(7.0))
    o = out.cpu().numpy()
    written = np.zeros(len(o), bool)
    for b in range(B):
        written[oo[b]:oo[b] + olens[b]] = True
    assert np.isnan(o[~written]).all(), "a write outside the outputs"
    p = pk.cpu().numpy()
    assert (p[:32] == SENT).all() and (p[32 + sum(K):] == SENT).all()
    return rc, [o[oo[b]:oo[b] + olens[b]] for b in range(B)], [p[po[b]:po[b] + K[b]] for b in range(B)], n


def _grid_waves(lengths, seed, loud=0.9):
    g = np.random.default_rng(seed)
    out = []
    for i, n in enumerate(lengths):
        t = np.arange(n) / 16000.0
        y = 0.4 * np.sin(2 * np.pi * (150 + 400 * g.random()) * t) + 0.15 * g.standard_normal(n)
        if i % 3 == 1:
            y = y * (loud / max(1e-9, np.abs(y).max()) if n else 1)          # loud: +8 dB clips it
        out.append(TG.grid16(y))
    return out


@pytest.mark.parametrize("sr", [8000, 16000, 48000])
def test_picks_and_output_match_the_restatement_on_the_16_bit_grid(L, sr):
    segment, search, overlap = TG.geometry(sr)
    step = segment - overlap
    g = np.random.default_rng(sr)
    lengths = [0, 1, segment - 1, 3 * step - 1, 3 * step, 3 * step + 1, 16 * sr, int(g.integers(2, 5 * sr)), 7 * step + 5]
    tempos = [0.85, 1.0, 1.15] + [float(f"{g.uniform(0.85, 1.15):.3f}") for _ in range(len(lengths) - 3)]
    gains = [-6.0, 8.0, 0.0] + [float(f"{g.uniform(-6, 8):.3f}") for _ in range(len(lengths) - 3)]
    gains[4] = 8.0                                          # a loud utterance (_grid_waves) at +8 dB: it clips
    xs = _grid_waves(lengths, sr)
    for rot in range(3):                                    # every tempo on every length class
        t = tempos[rot:] + tempos[:rot]
        order = g.permutation(len(xs)).tolist()
        rc, outs, picks, n = _call(L, xs, t, gains, sr, order=order)
        assert rc == OK and n == 1, L.last_error()
        for b, x in enumerate(xs):
            want, wpicks, _ = TG.stretch(x, t[b], TG.linear_gain(gains[b]), (segment, search, overlap))
            assert np.array_equal(picks[b], wpicks), (sr, rot, b)
            assert np.array_equal(outs[b].view(np.int32), want.view(np.int32)), (sr, rot, b)
        assert np.abs(outs[4]).max() >= 32767 / 32768


def test_off_grid_picks_are_minimal_and_the_output_replays_them(L):
    sr = 16000
    g = np.random.default_rng(5)
    lengths = [16 * sr, 5 * sr + 3, 12345]
    xs = [(0.3 * g.standard_normal(n)).astype(np.float32) for n in lengths]
    tempos, gains = [0.85, 1.15, 1.0], [3.25, -6.0, 8.0]
    rc, outs, picks, _ = _call(L, xs, tempos, gains, sr, order=[2, 0, 1])
    assert rc == OK
    geom = TG.geometry(sr)
    for b, x in enumerate(xs):
        want, used, Ds = TG.stretch(x, tempos[b], TG.linear_gain(gains[b]), geom, picks=picks[b])
        assert np.array_equal(used, picks[b]) and picks[b][0] == geom[1] // 2
        step = geom[0] - geom[2]
        S = TG.starts(tempos[b], len(picks[b]), step)
        xt = np.zeros(S[-1] + geom[0] + geom[1] + len(x), np.float32)
        xt[:len(x)] = x
        for k in range(1, len(picks[b])):
            p = S[k - 1] + picks[b][k - 1] + step
            prev = xt[p:p + geom[2]].astype(np.float64)
            D = Ds[k - 1]
            assert D[picks[b][k]] - D.min() <= 1e-12 * (D.min() + (prev ** 2).sum()), (b, k)
        assert np.array_equal(outs[b].view(np.int32), want.view(np.int32)), b


def test_repeated_calls_are_bit_identical(L):
    xs = _grid_waves([40000, 9000, 77777], 3)
    a = _call(L, xs, [0.9, 1.1, 0.85], [1.0, -2.0, 7.5], 16000)
    b = _call(L, xs, [0.9, 1.1, 0.85], [1.0, -2.0, 7.5], 16000, order=[1, 2, 0])
    assert a[0] == b[0] == OK and a[3] == b[3] == 1
    assert all(np.array_equal(u.view(np.int32), v.view(np.int32)) for u, v in zip(a[1], b[1]))
    assert all(np.array_equal(u, v) for u, v in zip(a[2], b[2]))


def test_bad_device_data_gives_nan(L):
    """A non-finite or non-positive tempo, or a negative input offset: NaN output and -1 picks; a negative output offset:
    nothing written; the other utterances as usual."""
    xs = _grid_waves([5000] * 6, 8)
    tempos = [1.0, 0.0, -1.0, float("inf"), NAN, 1.05]
    rc, outs, picks, _ = _call(L, xs, tempos, [0.0] * 6, 16000)
    assert rc == OK
    assert np.array_equal(outs[0], TG.stretch(xs[0], 1.0, 1.0, TG.geometry(16000))[0])
    for b in range(1, 5):
        assert np.isnan(outs[b]).all() and (picks[b] == -1).all(), b
    assert np.array_equal(outs[5], TG.stretch(xs[5], 1.05, 1.0, TG.geometry(16000))[0])
    rc, outs, picks, _ = _call(L, xs[:2], [1.0, 1.0], [0.0, 0.0], 16000, in_offsets=[-100, GAP + 5000 + GAP])
    assert rc == OK and np.isnan(outs[0]).all() and (picks[0] == -1).all() and not np.isnan(outs[1]).any()
    rc, outs, picks, _ = _call(L, xs[:2], [1.0, 1.0], [0.0, 0.0], 16000, out_offsets=[-1, GAP])   # GAP: utterance 1's own
    assert rc == OK and np.isnan(outs[0]).all() and (picks[0] == SENT).all() and not np.isnan(outs[1]).any()


def test_rejections_launch_and_write_nothing(L):
    lib = L.load()
    x = torch.from_numpy(_grid_waves([3000], 1)[0]).cuda()
    dev = lambda a, dt: torch.tensor(a, dtype=dt, device="cuda")  # noqa: E731
    io, il, t, g = dev([0], torch.int64), dev([3000], torch.int32), dev([1.0], torch.float64), dev([1.0], torch.float32)
    out = torch.full((3100,), NAN, device="cuda")
    oo, ol = dev([8], torch.int64), dev([3000], torch.int32)
    pk, po = torch.full((16,), SENT, dtype=torch.int32, device="cuda"), dev([2], torch.int64)
    st = torch.cuda.current_stream().cuda_stream
    base = dict(i=L.ptr(x), io=L.ptr(io), il=L.ptr(il), t=L.ptr(t), g=L.ptr(g), o=L.ptr(out), oo=L.ptr(oo), ol=L.ptr(ol),
                p=L.ptr(pk), po=L.ptr(po), B=1, seg=1312, sea=235, ov=192)

    def call(**kw):
        a = dict(base, **kw)
        n0 = lib.b200asr_launch_count()
        rc = lib.b200asr_tempo_gain(a["i"], a["io"], a["il"], a["t"], a["g"], a["o"], a["oo"], a["ol"], a["p"], a["po"],
                                    a["B"], a["seg"], a["sea"], a["ov"], st)
        return rc, lib.b200asr_launch_count() - n0

    cases = [(dict(i=None), BAD_ARG), (dict(t=None), BAD_ARG), (dict(o=None), BAD_ARG), (dict(ol=None), BAD_ARG),
             (dict(p=None), BAD_ARG), (dict(po=None), BAD_ARG), (dict(i=base["i"] + 2), BAD_ALIGN),
             (dict(t=base["t"] + 4), BAD_ALIGN), (dict(o=base["o"] + 1), BAD_ALIGN), (dict(oo=base["oo"] + 4), BAD_ALIGN),
             (dict(B=0), BAD_SHAPE), (dict(ov=4, seg=64), BAD_SHAPE), (dict(ov=200, seg=399), BAD_SHAPE),
             (dict(sea=0), BAD_SHAPE), (dict(seg=40000), BAD_SHAPE)]
    for kw, code in cases:
        assert call(**kw) == (code, 0), kw
    torch.cuda.synchronize()
    assert bool(out.isnan().all()) and bool((pk == SENT).all())
    assert call() == (OK, 1)
    torch.cuda.synchronize()
    assert not bool(out[8:3008].isnan().any()) and bool(out[:8].isnan().all()) and bool(out[3008:].isnan().all())
    assert pk[2:5].tolist() == [117, 117, 117] and bool((pk[5:] == SENT).all())


# ------------------------------------------------------------------------------------------------------- host layer

def test_host_call_is_the_entry_point(L):
    import b200asr
    xs = _grid_waves([16000, 0, 7001, 30000], 4)
    tempos, gains = [0.87, 1.0, 1.149, 0.85], [0.5, 0.0, -6.0, 8.0]
    wave = torch.from_numpy(np.concatenate(xs)).cuda()
    offs = np.concatenate([[0], np.cumsum([len(x) for x in xs])[:-1]])
    n0 = L.load().b200asr_launch_count()
    out, oo, ol, pk, po = b200asr.tempo_gain(wave, offs, [len(x) for x in xs], tempos, gains, 16000, picks=True)
    assert L.load().b200asr_launch_count() - n0 == 1
    o, oo, ol, pk = out.cpu().numpy(), oo.cpu().numpy(), ol.cpu().numpy(), pk.cpu().numpy()
    for b, x in enumerate(xs):
        want, wp, _ = TG.stretch(x, tempos[b], TG.linear_gain(gains[b]), TG.geometry(16000))
        assert ol[b] == len(want) and np.array_equal(o[oo[b]:oo[b] + ol[b]], want)
        assert np.array_equal(pk[po[b]:po[b] + len(wp)], wp)
    with pytest.raises(ValueError):
        b200asr.tempo_gain(wave, offs, [len(x) for x in xs], [1.0, 0.0, 1.0, 1.0], gains, 16000)
    with pytest.raises(ValueError):
        b200asr.tempo_gain(wave, offs, torch.tensor([len(x) for x in xs]).cuda(), tempos, gains, 16000)


def test_collate_waves_without_a_policy_is_unchanged(L):
    import b200asr
    conf = dict(sample_rate=16000, window_size=0.02, window_stride=0.01, window="hamming")
    batch = [(w, [1, 4, 5]) for w in _grid_waves([16000, 9000, 4001], 5)]
    a = b200asr.collate_waves(batch, conf, 120)
    b = b200asr.collate_waves(batch, conf, 120, tempo_gain=None)
    assert all(torch.equal(u, v) for u, v in zip(a, b))


# ----------------------------------------------------------------------------------------------- the installed loader

@pytest.fixture
def env(monkeypatch):
    from tests.test_loader_host import Env
    return Env(monkeypatch)


LENGTHS = [16000, 8000, 12000, 4000, 9000, 15000, 3000, 11000, 161, 32000, 2560]


def _dataset(env, tmp_path, lengths, prob, policy=True, **kw):
    import b200asr
    ds = env.dataset(tmp_path, lengths, prob=prob, augment=True, **kw)
    for w in list(env.utts):
        env.utts[w] = TG.grid16(env.utts[w])
    if policy:
        ds.tempo_gain = b200asr.TempoGain()
    return ds


def _restated_sox(env):
    def augment(path, sample_rate, tempo, gain):
        t, g = float(f"{tempo:.3f}"), float(f"{gain:.3f}")
        return TG.stretch(env._load(path), t, TG.linear_gain(g), TG.geometry(sample_rate))[0]
    return augment


def _materialise(batches):
    return [tuple(t.clone() if t.is_cuda else t for t in b) for b in batches]


@needs_ref
@pytest.mark.parametrize("workers", [0, 2])
@pytest.mark.parametrize("prob", [None, 0.5])
def test_installed_loader_matches_the_reference_loader(env, tmp_path, monkeypatch, workers, prob):
    """The reference's own loader with augment=True and sox restated, against the installed loader with the dataset's
    tempo_gain on the same seeds: the same order, sizes and targets; inputs within the loader's bar."""
    import b200asr
    DL = env.DL
    ds = _dataset(env, tmp_path, LENGTHS, prob, window="hann")
    monkeypatch.setattr(env.audio, "augment_audio_with_sox", _restated_sox(env))
    _run = lambda: list(DL.AudioDataLoader(ds, num_workers=workers, batch_sampler=DL.BucketingSampler(ds, batch_size=4)))  # noqa: E731
    torch.manual_seed(3), np.random.seed(3), __import__("random").seed(3)
    want = _run()
    b200asr.install()
    try:
        torch.manual_seed(3), np.random.seed(3), __import__("random").seed(3)
        got = _materialise(_run())
    finally:
        b200asr.uninstall()
    assert len(got) == len(want) == 3
    for g, w in zip(got, want):
        assert g[0].is_cuda and not any(t.is_cuda for t in g[1:])
        for a, b in zip(g[1:], w[1:]):
            assert a.dtype == b.dtype and torch.equal(a, b)
        assert g[0].shape == w[0].shape and rel_err(g[0].cpu(), w[0]) < BAR


class _Replay:
    """An rng that gives TempoGain.draw_one recorded (tempo, gain_db) pairs back, one uniform() call each."""

    def __init__(self, pairs):
        self.values = [v for p in pairs for v in p]

    def uniform(self, low, high):
        return self.values.pop(0)


@needs_ref
def test_installed_loader_is_collate_waves_with_the_policy(env, tmp_path, monkeypatch):
    """The installed loader's batches equal collate_waves(tempo_gain=...) over the items its workers made, replaying their
    draws, bit for bit; one launch more per batch than without the policy."""
    import b200asr
    from b200asr import features, loader
    ds = _dataset(env, tmp_path, LENGTHS[:8], None, src_max_len=90)
    monkeypatch.setattr(env.audio, "augment_audio_with_sox", _raise)
    items, draws = [], []
    collate, draw = loader.collate_items, features.TempoGain.draw_one
    monkeypatch.setattr(loader, "collate_items", lambda its: (items.append([(it.wave, it.ids) for it in its]), collate(its))[1])
    monkeypatch.setattr(features.TempoGain, "draw_one", lambda s, rng=np.random: (lambda d: (draws.append(d), d)[1])(draw(s, rng)))
    launches = []
    b200asr.install()
    try:
        np.random.seed(1), torch.manual_seed(1), __import__("random").seed(1)
        got = []
        for b in env.DL.AudioDataLoader(ds, num_workers=0, batch_sampler=env.DL.BucketingSampler(ds, batch_size=3)):
            got.append(tuple(t.clone() for t in b))
    finally:
        b200asr.uninstall()
    assert len(got) == len(items) == 3 and len(draws) == 8
    conf = dict(sample_rate=16000, window_size=0.02, window_stride=0.01, window="hamming")
    k = 0
    for g, its in zip(got, items):
        lib0 = b200asr._lib.load().b200asr_launch_count()
        want = b200asr.collate_waves(its, conf, 90, rng=_Replay(draws[k:k + len(its)]), tempo_gain=b200asr.TempoGain())
        launches.append(b200asr._lib.load().b200asr_launch_count() - lib0)
        k += len(its)
        assert all(torch.equal(u.cpu(), v.cpu()) for u, v in zip(g, want))
    plain = b200asr._lib.load().b200asr_launch_count()
    b200asr.collate_waves(items[0], conf, 90)
    assert launches == [b200asr._lib.load().b200asr_launch_count() - plain + 1] * 3


def _raise(*a, **k):
    raise AssertionError("sox was called")


@needs_ref
@pytest.mark.parametrize("workers", [0, 2])
def test_installed_loader_makes_no_host_sync(env, tmp_path, monkeypatch, workers):
    import b200asr
    ds = _dataset(env, tmp_path, [16000, 8000, 12000, 4000] * 4, 0.5)
    monkeypatch.setattr(env.audio, "augment_audio_with_sox", _raise)
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
def test_dataset_without_the_policy_is_unchanged(env, tmp_path):
    """augment=False, no attribute: the installed loader's batches and launches are collate_waves' without a policy."""
    import b200asr
    from b200asr import loader
    ds = env.dataset(tmp_path, LENGTHS[:6], prob=None, src_max_len=90)
    items = []
    collate = loader.collate_items
    loader.collate_items = lambda its: (items.append([(it.wave, it.ids) for it in its]), collate(its))[1]
    lib = b200asr._lib.load()
    b200asr.install()
    try:
        np.random.seed(1), torch.manual_seed(1), __import__("random").seed(1)
        it = iter(env.DL.AudioDataLoader(ds, num_workers=0, batch_sampler=env.DL.BucketingSampler(ds, batch_size=3)))
        got, counts = [], []
        while True:
            n0 = lib.b200asr_launch_count()
            try:
                b = next(it)
            except StopIteration:
                break
            counts.append(lib.b200asr_launch_count() - n0)
            got.append(tuple(t.clone() for t in b))
    finally:
        loader.collate_items = collate
        b200asr.uninstall()
    conf = dict(sample_rate=16000, window_size=0.02, window_stride=0.01, window="hamming")
    for g, its, c in zip(got, items, counts):
        n0 = lib.b200asr_launch_count()
        want = b200asr.collate_waves(its, conf, 90)
        assert c == lib.b200asr_launch_count() - n0
        assert all(torch.equal(u.cpu(), v.cpu()) for u, v in zip(g, want))


@needs_ref
def test_trainer_iteration_trains_without_sox(env, tmp_path, monkeypatch):
    """One Trainer.train iteration of the bound reference loop over an installed loader whose augment=True dataset carries
    the policy, with utils.audio.augment_audio_with_sox raising: finite losses, every parameter with a gradient moved."""
    import b200asr
    from tests.test_gpu_linear_precisions import _waves
    from tests.test_gpu_loader import _model
    ds = _dataset(env, tmp_path, LENGTHS[:3], None, src_max_len=90)
    monkeypatch.setattr(env.audio, "augment_audio_with_sox", _raise)
    valid = [b200asr.collate_waves([(w, [1, 4, 5, 2]) for w in _waves([7000, 5000], seed=3)],
                                   dict(sample_rate=16000, window_size=0.02, window_stride=0.01, window="hamming"), 90)]
    ns, model, i2l = _model(env)
    ns.constant.args.src_max_len, ns.constant.args.save_folder, ns.constant.args.name = 90, str(tmp_path), "tempo"
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
