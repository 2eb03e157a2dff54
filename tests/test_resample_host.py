"""CPU checks of the polyphase resampler and speed perturbation (features.resample / SpeedPerturb, b200asr_resample_packed,
the installed loader's opt-in and its noise clips at other rates): the numpy taps against scipy.signal.firwin, the
phase-split restatement (tests/resample_util.py) against scipy.signal.resample_poly, output lengths, the policy's
validation, ratios, draws and pickling, the worker items' draw order, frame counts and sort with and without the policy,
the noise clips' rate inference and the fallback for clips the device path cannot serve, the entry point's rejections, which need no GPU, and the kernel's build
(no spills, no local memory)."""
import pickle
import random

import numpy as np
import pytest
import scipy.signal
import torch

import b200asr
from b200asr import features as F
from oracle import ref_shim
from tests import resample_util as RU

L = b200asr._lib
needs_ref = pytest.mark.skipif(not ref_shim.available(), reason="reference checkout not staged (oracle/make_ref.py)")


@pytest.fixture(scope="module")
def lib():
    import os
    import __graft_entry__
    if not os.path.exists(L.LIB_PATH):
        __graft_entry__.build()
    return L.load()


@pytest.fixture
def env(monkeypatch):
    from tests.test_loader_host import Env
    return Env(monkeypatch)


@pytest.mark.parametrize("up, down", RU.RATIOS)
def test_taps_are_firwins(up, down):
    """resample_filter / up equals firwin(2 half + 1, 1 / max, ('kaiser', 5.0)) in float64 (np.i0 against
    scipy.special.i0: a few units in the last place), and the phase split is taps[p, m] = fp32(h[p + m up])."""
    if up == down == 1:
        x = np.arange(5.0)
        y = scipy.signal.resample_poly(x, 1, 1)
        assert np.array_equal(y, x) and y is not x and np.array_equal(RU.polyphase(x, 1, 1), x)
        return
    mr = max(up, down)
    want = scipy.signal.firwin(2 * 10 * mr + 1, 1.0 / mr, window=("kaiser", 5.0))
    h = F.resample_filter(up, down)
    assert h.dtype == np.float64 and len(h) == len(want)
    assert np.abs(h / up - want).max() <= 1e-15 * np.abs(want).max()
    taps = F.resample_taps(up, down)
    K = -(-len(h) // up)
    assert taps.dtype == np.float32 and taps.shape == (up, K)
    for p in range(up):
        m = np.arange(K)
        k = p + m * up
        assert np.array_equal(taps[p], np.where(k < len(h), h[np.minimum(k, len(h) - 1)], 0).astype(np.float32))


@pytest.mark.parametrize("up, down", RU.RATIOS)
def test_polyphase_sum_is_resample_poly(up, down):
    g = np.random.default_rng(up * 1000 + down)
    filt = 2 * 10 * max(up, down) + 1
    for n in (0, 1, 2, filt // 3, filt - 1, 100000):
        x = g.uniform(-1, 1, n)
        want = scipy.signal.resample_poly(x, up, down)
        got = RU.polyphase(x, up, down)
        assert len(got) == len(want) == F.resample_out_length(n, up, down), (n, len(want))
        assert np.abs(got - want).max(initial=0) <= 1e-12, n


def test_out_length_and_ratio():
    ol = F.resample_out_length
    assert ol(0, 10, 11) == 0 and ol(1, 10, 11) == 1 and ol(11, 10, 11) == 10 and ol(12, 10, 11) == 11
    assert ol(240000, 10, 9) == 266667 and ol(240000, 10, 11) == 218182 and ol(7, 2, 1) == 14 and ol(7, 1, 2) == 4
    for n in (0, 1, 5, 441, 16001):
        for up, down in RU.RATIOS:
            assert ol(n, up, down) == len(scipy.signal.resample_poly(np.zeros(n), up, down))
    assert F.resample_ratio(16000, 44100) == (160, 441) and F.resample_ratio(2000, 1000) == (2, 1)
    assert F.resample_ratio(np.int64(6), 4) == (3, 2)
    for up, down in ((0, 1), (1, 0), (-2, 1), (1001, 1), (1, 1001), (1.5, 1), (True, 1), (1001, 999)):
        with pytest.raises(ValueError):
            F.resample_ratio(up, down)


def test_speed_perturb_policy():
    sp = b200asr.SpeedPerturb()
    assert sp.factors == (0.9, 1.0, 1.1) and "0.9" in repr(sp)
    assert [sp.ratio(f) for f in sp.factors] == [(10, 9), (1, 1), (10, 11)]
    assert sp.ratio(1) == (1, 1) and sp.ratio(0.95) == (20, 19) and sp.ratio(2) == (1, 2)
    assert sp.out_length(11, 1.1) == 10 and sp.out_length(9, 0.9) == 10 and sp.out_length(16000, 1.0) == 16000
    for bad in ((), (0.0,), (-1.1,), (float("nan"),), (float("inf"),), ("1.1",), (True,), (0.0001,), (1.0013,), 1.1):
        with pytest.raises(ValueError):
            b200asr.SpeedPerturb(bad)
    b200asr.SpeedPerturb((0.001, 1000))                       # 1000/1 and 1/1000: the largest ratios taken
    q = pickle.loads(pickle.dumps(b200asr.SpeedPerturb((0.8, 1.2))))
    assert q.factors == (0.8, 1.2) and repr(q) == "SpeedPerturb(factors=(0.8, 1.2))"


def test_speed_perturb_draws_are_one_choice():
    """draw_one is one rng.choice over the factors: the generator ends where choice over a list of that length ends."""
    sp = b200asr.SpeedPerturb()
    for seed in range(10):
        np.random.seed(seed)
        got = [sp.draw_one(np.random) for _ in range(5)]
        st = np.random.get_state()
        np.random.seed(seed)
        want = [np.random.choice([0.9, 1.0, 1.1]) for _ in range(5)]
        assert got == [float(w) for w in want]
        assert np.array_equal(st[1], np.random.get_state()[1])
    rs = np.random.RandomState(0)
    assert {b200asr.SpeedPerturb().draw_one(rs) for _ in range(60)} == {0.9, 1.0, 1.1}


def test_resample_needs_cuda_and_host_geometry():
    with pytest.raises(RuntimeError, match="CUDA"):
        b200asr.resample(torch.zeros(8), [0], [8], [10], [11])


class _Recorder:
    """Records, per item, the order of the policy, speed and noise draws and the length each noise draw was made for."""

    def __init__(self, monkeypatch):
        self.log = []
        for cls, name in ((F.TempoGain, "tempo"), (F.SpeedPerturb, "speed")):
            orig = cls.draw_one
            monkeypatch.setattr(cls, "draw_one", lambda s, rng=np.random, _o=orig, _n=name: (self.log.append(_n), _o(s, rng))[1])
        orig = F.NoiseClips.draw_one
        monkeypatch.setattr(F.NoiseClips, "draw_one",
                            lambda s, n, *a, _o=orig: (self.log.append(("noise", int(n))), _o(s, n, *a))[1])


@needs_ref
@pytest.mark.parametrize("tempo", [False, True])
@pytest.mark.parametrize("prob", [None, 1.0])
def test_items_draw_speed_after_augment_and_before_noise(env, tmp_path, monkeypatch, tempo, prob):
    """Per item: tempo and gain (with a TempoGain), then the speed factor, then noise for the resampled length; the item's
    ratio, lengths and frames follow from those draws; collate_items sorts by the perturbed frames."""
    from b200asr import loader
    lengths = [8000, 12345, 3200, 161, 30000, 16000]
    ds = env.dataset(tmp_path, lengths, prob=prob, augment=tempo, src_max_len=150)
    if tempo:
        ds.tempo_gain = b200asr.TempoGain()
    ds.speed_perturb = b200asr.SpeedPerturb()
    rec = _Recorder(monkeypatch)
    items = loader.PackedItems(ds, env.clip_set() if prob is not None else None)
    random.seed(3), np.random.seed(3)
    got = []
    for i in range(len(lengths)):
        rec.log.clear()
        it = items[i]
        got.append(it)
        n = it.out_length if tempo else len(it.wave)
        assert it.speed_length == F.resample_out_length(n, it.up, it.down)
        assert (it.up, it.down) in ((10, 9), (1, 1), (10, 11))
        assert it.frames == min(1 + it.speed_length // 160, 150)
        want = (["tempo"] if tempo else []) + ["speed"] + ([("noise", it.speed_length)] if prob is not None else [])
        assert rec.log == want, (i, rec.log)
    assert len({(it.up, it.down) for it in got}) > 1
    pb = loader.collate_items(got)
    order = sorted(range(len(got)), key=lambda i: got[i].frames, reverse=True)
    assert pb.input_sizes.tolist() == [got[i].frames for i in order]
    assert pb.speed_lengths.dtype == torch.int32 and pb.speed_lengths.tolist() == [got[i].speed_length for i in order]
    assert pb.up.tolist() == [got[i].up for i in order] and pb.down.tolist() == [got[i].down for i in order]
    assert (pb.out_lengths is not None) == tempo
    with pytest.raises(ValueError, match="mixes resampled"):
        loader.collate_items([got[0], loader.Item(*got[1][:9])])


@needs_ref
def test_items_without_the_policy_are_unchanged(env, tmp_path):
    """No speed_perturb attribute: the items, their draws and the generator states are those of the parent's items."""
    from b200asr import loader
    ds = env.dataset(tmp_path, [4000, 2000, 9000], prob=0.5)
    items = loader.PackedItems(ds, env.clip_set())
    random.seed(1), np.random.seed(1)
    its = [items[i] for i in range(3)]
    assert all(type(it) is loader.Item for it in its)
    assert loader.collate_items(its).speed_lengths is None
    ds.speed_perturb = b200asr.SpeedPerturb((1.0,))
    random.seed(1), np.random.seed(1)
    with_one = [items[i] for i in range(3)]
    assert any(a.noise_clip != b.noise_clip or a.noise_level != b.noise_level for a, b in zip(its, with_one)) or \
        all(it.noise_clip < 0 for it in its)                  # the extra draw shifts the noise draws that follow it
    assert all(it[9:] == (1, 1, len(it.wave)) for it in with_one)


def test_clip_rate_inference():
    clip_rate = b200asr.loader.clip_rate
    assert clip_rate(16000, 1.0, 16000) == 16000
    assert clip_rate(36000, 36000 / 8000, 16000) == 8000
    assert clip_rate(44100 * 3 + 7, (44100 * 3 + 7) / 44100, 16000) == 44100
    assert clip_rate(16000, 1.00002, 16000) == 16000            # round(duration * sr) == n: the dataset's rate
    assert clip_rate(36000, 4.5001, 16000) is None              # round(36000 / 4.5001) = 8000, round(4.5001 * 8000) != 36000
    assert clip_rate(10, 0.0, 16000) is None and clip_rate(10, -1.0, 16000) is None
    assert clip_rate(10, float("nan"), 16000) is None and clip_rate(10, float("inf"), 16000) is None
    assert clip_rate(0, 0.0, 16000) == 16000


def _same_batches(a, b):
    return len(a) == len(b) and all(all(torch.equal(x, y) for x, y in zip(p, q)) for p, q in zip(a, b))


@needs_ref
@pytest.mark.parametrize("rate, resample", [(8000, False), (36000 / 4.5001, True), (16001, True)])
def test_noise_clips_the_device_cannot_serve_run_the_reference_loader(env, tmp_path, rate, resample):
    """A noise clip at 8 kHz on a dataset without resample_noise, or, with resample_noise = True, a clip whose rate
    cannot be inferred from its duration (36000 samples in 4.5001 s) or whose ratio to 16 kHz is beyond the resampler's
    (16000/16001): the installed loader runs the reference's own iterator and yields its batches; a dataset that also
    carries speed_perturb raises instead of dropping it, and names resample_noise."""
    DL = env.DL
    ds = env.dataset(tmp_path, [4000, 2000, 3000, 2500], prob=0.5)
    if resample:
        ds.resample_noise = True
    env.rates[sorted(env.clips)[1]] = rate
    random.seed(1), np.random.seed(1)
    want = list(DL.AudioDataLoader(ds, batch_size=2))
    b200asr.install()
    try:
        other = DL.AudioDataLoader(ds, batch_size=2)
        random.seed(1), np.random.seed(1)
        got = list(other)
        assert other._b200asr_packed.reference and _same_batches(got, want)
        ds.speed_perturb = b200asr.SpeedPerturb()
        with pytest.raises(RuntimeError, match="speed_perturb.*resample_noise"):
            iter(DL.AudioDataLoader(ds, batch_size=2))
    finally:
        b200asr.uninstall()


def test_entry_point_rejections_need_no_device(lib):
    """Argument checks run on the host before any launch: device pointers that are never dereferenced."""
    IN, OUT, TAPS, DEV = 1 << 24, 1 << 30, 1 << 34, 1 << 36
    BAD_SHAPE, BAD_ALIGN, BAD_ARG = -1, -2, -5

    def items(rows):
        a = np.zeros(len(rows), F._RESAMPLE_ITEM)
        for k, (io, oo, n, up, down) in enumerate(rows):
            a[k] = (io, oo, 0 if up == down == 1 else TAPS, n, up, down, 0)
        return a

    good = [(0, 0, 1100, 10, 11), (1100, 1000, 900, 10, 9), (2000, 2000, 50, 1, 1)]

    def call(rows=good, i=IN, n_in=2050, o=OUT, n_out=2050, it=True, dev=DEV, q=0, B=None, taps=None):
        a = items(rows)
        if taps is not None:
            a["taps"] = taps
        B = len(a) if B is None else B
        return lib.b200asr_resample_packed(i, n_in, o, n_out, a.ctypes.data if it else None, dev, B, q, None)

    assert call(i=None) == BAD_ARG and call(o=None) == BAD_ARG and call(it=False) == BAD_ARG and call(dev=None) == BAD_ARG
    assert call(q=2) == BAD_ARG and call(o=IN + 4 * 2000) == BAD_ARG and call(taps=0) == BAD_ARG
    assert call(taps=TAPS + 2) == BAD_ARG
    assert call(i=IN + 2) == BAD_ALIGN and call(o=OUT + 1) == BAD_ALIGN and call(dev=DEV + 4) == BAD_ALIGN
    assert call(B=0) == BAD_SHAPE and call(n_in=-1) == BAD_SHAPE and call(n_out=-1) == BAD_SHAPE
    for up, down in ((0, 1), (1, 0), (1001, 1), (1, 1001), (20, 22)):
        assert call(rows=[(0, 0, 10, up, down)]) == BAD_SHAPE, (up, down)
    assert call(n_in=2049) == BAD_SHAPE and call(rows=[(-1, 0, 10, 2, 1)]) == BAD_SHAPE
    assert call(rows=[(0, 0, -1, 2, 1)]) == BAD_SHAPE
    assert call(n_out=2049) == BAD_SHAPE and call(rows=[(0, -1, 10, 2, 1)]) == BAD_SHAPE
    assert call(rows=[(0, 0, 100, 1, 1), (100, 99, 10, 1, 1)]) == BAD_SHAPE          # overlapping outputs
    assert call(rows=[(0, 5, 0, 10, 11), (0, 5, 0, 1, 1)]) == 0                         # empty outputs: nothing to launch
    assert "resample_packed" in L.last_error()


def test_kernel_compiles_without_spills_or_local_memory(tmp_path):
    """resample.cu recompiled with build.sh's flags and -Xptxas -v: no stack frame and no spill stores; and in the built
    library, STACK:0 LOCAL:0 (cuobjdump -res-usage)."""
    import os
    import re
    import subprocess
    from tests.test_engine_build import CSRC, CUOBJDUMP, LIB, NVCC, ROOT, _build_flags, _need
    _need(NVCC)
    log = subprocess.run([NVCC, *_build_flags(), "-Xptxas", "-v,-warn-spills", "-c", os.path.join(CSRC, "resample.cu"),
                          "-o", str(tmp_path / "resample.o")], capture_output=True, text=True, cwd=ROOT, check=True).stderr
    props = re.findall(r"Function properties for (\S*resample_kernel\S*)\s*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores",
                       log)
    assert len(props) == 1 and props[0][1:] == ("0", "0"), log[-2000:]
    _need(CUOBJDUMP, LIB)
    out = subprocess.run([CUOBJDUMP, "-res-usage", LIB], check=True, capture_output=True, text=True).stdout
    usage = [u for n, u in re.findall(r"Function (\S+):\s*\n\s*(REG:.*)", out) if "resample_kernel" in n]
    assert len(usage) == 1 and re.search(r"\bSTACK:0\b", usage[0]) and re.search(r"\bLOCAL:0\b", usage[0]), usage
