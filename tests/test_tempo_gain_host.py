"""CPU checks of the tempo and gain perturbation (features.TempoGain, b200asr_tempo_gain, the installed loader's opt-in):
the draws against the reference's load_randomly_augmented_audio, the geometry and output length, the numpy restatement
(tests/tempo_gain_util.py) on tones and at tempo 1, the policy's validation and pickling, the worker items against the
reference's __getitem__ with sox replaced by the restatement, the C entry point's rejections, which need no GPU, and the
kernel's build (no spills, no local memory)."""
import pickle
import random

import numpy as np
import pytest
import torch

import b200asr
from oracle import ref_shim
from tests import tempo_gain_util as TG

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


def _rng_state():
    st = np.random.get_state()
    return st[1].tobytes(), st[2:]


@needs_ref
def test_draws_are_the_references(env):
    """load_randomly_augmented_audio with augment_audio_with_sox recording its arguments: the sox command line's "{:.3f}"
    of its tempo and gain equals TempoGain.draw_one's, and numpy's global state ends identical."""
    seen = []
    env.audio.augment_audio_with_sox = lambda path, sample_rate, tempo, gain: seen.append((tempo, gain)) or np.zeros(1)
    policy = b200asr.TempoGain()
    for seed in range(20):
        np.random.seed(seed)
        env.audio.load_randomly_augmented_audio("u.wav", 16000)
        want = _rng_state()
        np.random.seed(seed)
        tempo, gain = policy.draw_one(np.random)
        assert _rng_state() == want
        assert (f"{tempo:.3f}", f"{gain:.3f}") == tuple(f"{v:.3f}" for v in seen[-1])
        assert 0.85 <= tempo <= 1.15 and -6 <= gain <= 8
    rs = np.random.RandomState(3)
    assert b200asr.TempoGain((0.5, 0.5), (2, 2)).draw_one(rs) == (0.5, 2.0)


@pytest.mark.parametrize("sr, want", [(8000, (656, 117, 96)), (16000, (1312, 235, 192)), (22050, (1808, 324, 264)),
                                      (44100, (3616, 647, 528)), (48000, (3936, 704, 576))])
def test_geometry(sr, want):
    assert b200asr.TempoGain.geometry(sr) == TG.geometry(sr) == want


def test_geometry_rejects_rates_without_one():
    for sr in (0, 100, float("nan"), -16000):
        with pytest.raises(ValueError):
            b200asr.TempoGain.geometry(sr)


def test_out_length():
    ol = b200asr.TempoGain.out_length
    assert ol(0, 0.85) == 0 and ol(1, 1.15) == 1 and ol(16000, 1.0) == 16000
    assert ol(256000, 0.85) == 301176 and ol(256000, 1.15) == 222609
    assert ol(3, 2.0) == 2 and ol(1, 2.0) == 1 and ol(1, 4.0) == 0           # floor(n / tempo + 0.5)
    for n in (1, 17, 1311, 1312, 16000, 255999):
        for t in (0.85, 0.999, 1.0, 1.001, 1.15):
            assert ol(n, t) == TG.out_length(n, t) == int(np.floor(n / t + 0.5))


@pytest.mark.parametrize("tempo", [0.85, 1.0, 1.15])
def test_restatement_keeps_a_tones_pitch(tempo):
    """A 440 Hz tone (16-bit grid) stays at 440 Hz within one FFT bin, and the output has round(n / tempo) samples."""
    sr, n = 16000, 48000
    x = TG.grid16(0.5 * np.sin(2 * np.pi * 440 * np.arange(n) / sr))
    y, picks, _ = TG.stretch(x, tempo, np.float32(1), TG.geometry(sr))
    assert len(y) == round(n / tempo) and len(picks) == -(-len(y) // (1312 - 192))
    spec = np.abs(np.fft.rfft(y * np.hanning(len(y))))
    assert abs(np.argmax(spec) * sr / len(y) - 440) <= sr / len(y)


@pytest.mark.parametrize("sr", [8000, 16000, 48000])
def test_restatement_at_tempo_one_is_a_shift(sr):
    """Tempo 1.000 and gain 0 dB on 16-bit white noise: x[p_0 : p_0 + n] zero-extended, bit for bit."""
    geom = TG.geometry(sr)
    x = TG.grid16(np.random.default_rng(sr).uniform(-0.9, 0.9, 3 * sr + 17))
    y, picks, _ = TG.stretch(x, 1.0, TG.linear_gain(0.0), geom)
    p0 = geom[1] // 2
    want = np.zeros(len(x), np.float32)
    want[:len(x) - p0] = x[p0:]
    assert TG.linear_gain(0.0) == 1 and np.array_equal(y, want) and set(picks.tolist()) == {p0}


def test_restatement_gain_clips():
    x = TG.grid16(np.full(3000, 0.9))
    y, _, _ = TG.stretch(x, 1.0, TG.linear_gain(8.0), TG.geometry(16000))
    assert y.max() == np.float32(32767 / 32768) and TG.linear_gain(8.0) == np.float32(10 ** 0.4)


@pytest.mark.parametrize("kw", [dict(tempo_range=(0.2, 1.0)), dict(tempo_range=(1.0, 4.5)), dict(tempo_range=(1.2, 1.1)),
                                dict(tempo_range=(0.0, 1.0)), dict(tempo_range=(float("nan"), 1.0)),
                                dict(tempo_range=(1.0, float("inf"))), dict(tempo_range=(1.0,)), dict(tempo_range=1.0),
                                dict(tempo_range=("0.9", 1.1)), dict(tempo_range=(True, 1.1)), dict(gain_range=(3, -3)),
                                dict(gain_range=(0, float("inf"))), dict(gain_range=(float("nan"), 0))])
def test_policy_rejects_bad_ranges(kw):
    with pytest.raises(ValueError):
        b200asr.TempoGain(**kw)


def test_policy_defaults_and_pickles():
    a = b200asr.TempoGain()
    assert a.tempo_range == (0.85, 1.15) and a.gain_range == (-6.0, 8.0)
    b = pickle.loads(pickle.dumps(b200asr.TempoGain((0.25, 4), (-1.5, 0))))
    assert b.tempo_range == (0.25, 4.0) and b.gain_range == (-1.5, 0.0) and "tempo_range" in repr(b)
    np.random.seed(9)
    u = b.draw_one(np.random)
    np.random.seed(9)
    assert b200asr.TempoGain((0.25, 4), (-1.5, 0)).draw_one(np.random) == u


def test_tempo_gain_needs_cuda_tensors():
    with pytest.raises(RuntimeError, match="CUDA"):
        b200asr.tempo_gain(torch.zeros(8), [0], [8], [1.0], [0.0], 16000)


def sox_restated(env, records):
    """augment_audio_with_sox replaced by the restatement: the audio stretched with the command line's rounded values."""
    def augment(path, sample_rate, tempo, gain):
        t, g = float(f"{tempo:.3f}"), float(f"{gain:.3f}")
        records.append((t, g))
        return TG.stretch(env._load(path), t, TG.linear_gain(g), TG.geometry(sample_rate))[0]
    return augment


@needs_ref
@pytest.mark.parametrize("prob", [None, 0.0, 0.5, 1.0])
def test_items_make_the_reference_calls_with_the_policy(env, tmp_path, prob):
    """PackedItems over an augment=True dataset with a tempo_gain: the reference's __getitem__, with sox restated, makes the
    same draws (equal generator states after every item); each item's tempo, gain and stretched length are the ones the
    reference used, its frames the reference's, its noise draw made for the stretched length, and the restatement of its
    waveform is what the reference handed to librosa.stft when no noise was added."""
    from b200asr import loader
    lengths = [8000, 12345, 3200, 161, 30000, 16000]
    ds = env.dataset(tmp_path, lengths, prob=prob, augment=True)
    for w in list(env.utts):
        env.utts[w] = TG.grid16(env.utts[w])
    records = []
    env.audio.augment_audio_with_sox = sox_restated(env, records)
    ds.tempo_gain = b200asr.TempoGain()
    items = loader.PackedItems(ds, env.clip_set() if prob is not None else None)
    for seed in (1, 2):
        random.seed(seed), np.random.seed(seed)
        env.stft_calls.clear(), env.sox.clear(), records.clear()
        ref, states = [], []
        for i in range(len(lengths)):
            ref.append(ds[i])
            states.append((random.getstate(), _rng_state()))
        mixes, trims = list(env.stft_calls), list(env.sox)
        random.seed(seed), np.random.seed(seed)
        got = []
        for i in range(len(lengths)):
            got.append(items[i])
            assert (random.getstate(), _rng_state()) == states[i], (seed, i)
        assert len(records) == len(lengths) and (prob != 1.0 or len(trims) == len(lengths))
        for it, (spect, ids), (t, g), mix in zip(got, ref, records, mixes):
            assert it.ids == ids and it.frames == spect.shape[1] and it.tempo == t and it.g == TG.linear_gain(g)
            assert it.out_length == len(mix) == TG.out_length(len(it.wave), t)
            if it.noise_clip >= 0:                      # the segment the reference cut for the stretched length
                path, start = trims.pop(0)
                clip_len = len(env.clips[path])
                s0 = min(max(int(round(start * 16000)), 0), clip_len - it.out_length)
                assert it.noise_start == env.clip_set().offsets[sorted(env.clips).index(path)] + s0
            if it.noise_clip < 0:
                y = TG.stretch(it.wave, it.tempo, np.float32(it.g), TG.geometry(16000))[0]
                assert np.array_equal(y, mix)
        pb = loader.collate_items(got)
        order = sorted(range(len(got)), key=lambda i: got[i].frames, reverse=True)
        assert pb.tempo.dtype == torch.float64 and pb.g.dtype == torch.float32 and pb.out_lengths.dtype == torch.int32
        assert pb.out_lengths.tolist() == [got[i].out_length for i in order]
        assert pb.tempo.tolist() == [got[i].tempo for i in order]


@needs_ref
def test_items_without_the_policy_are_unchanged(env, tmp_path):
    """augment=True without the attribute keeps the reference's sox path; the items carry the defaults and the batch None."""
    from b200asr import loader
    ds = env.dataset(tmp_path, [4000, 2000], prob=None, augment=True)
    items = loader.PackedItems(ds)
    np.random.seed(0)
    its = [items[i] for i in range(2)]
    assert len(env.augments) == 2 and all(it[6:] == (1.0, 1.0, -1) for it in its)
    pb = loader.collate_items(its)
    assert pb.tempo is None and pb.g is None and pb.out_lengths is None
    mixed = [its[0], its[1]._replace(out_length=5)]
    with pytest.raises(ValueError, match="mixes"):
        loader.collate_items(mixed)


@needs_ref
def test_loader_refuses_a_policy_without_augment_or_on_the_reference_iterator(env, tmp_path):
    ds = env.dataset(tmp_path, [4000, 3000], prob=None, augment=False)
    ds.tempo_gain = b200asr.TempoGain()
    b200asr.install()
    try:
        with pytest.raises(ValueError, match="augment=False"):
            env.DL.AudioDataLoader(ds, batch_size=2)
        ds.augment = True
        loader = env.DL.AudioDataLoader(ds, batch_size=2, collate_fn=lambda items: items)
        with pytest.raises(RuntimeError, match="tempo_gain"):
            iter(loader)
    finally:
        b200asr.uninstall()


def test_entry_point_rejections_need_no_device(lib):
    """Argument checks run on the host before any launch: pointers that are never dereferenced."""
    base = dict(i=1 << 20, io=1 << 21, il=1 << 22, t=1 << 23, g=1 << 24, o=1 << 25, oo=1 << 26, ol=1 << 27, p=None, po=None,
                B=2, seg=1312, sea=235, ov=192)

    def call(**kw):
        a = dict(base, **kw)
        return lib.b200asr_tempo_gain(a["i"], a["io"], a["il"], a["t"], a["g"], a["o"], a["oo"], a["ol"], a["p"], a["po"],
                                      a["B"], a["seg"], a["sea"], a["ov"], None)
    BAD_SHAPE, BAD_ALIGN, BAD_ARG = -1, -2, -5
    for k in ("i", "io", "il", "t", "g", "o", "oo", "ol"):
        assert call(**{k: None}) == BAD_ARG, k
    assert call(p=1 << 28) == BAD_ARG and call(po=1 << 28) == BAD_ARG
    for k in ("i", "il", "g", "o", "ol"):
        assert call(**{k: base[k] + 2}) == BAD_ALIGN, k
    for k in ("io", "t", "oo"):
        assert call(**{k: base[k] + 4}) == BAD_ALIGN, k
    assert call(p=(1 << 28) + 2, po=1 << 29) == BAD_ALIGN and call(p=1 << 28, po=(1 << 29) + 4) == BAD_ALIGN
    assert call(B=0) == BAD_SHAPE and call(ov=7, seg=14) == BAD_SHAPE and call(ov=8, seg=15) == BAD_SHAPE
    assert call(sea=0) == BAD_SHAPE and call(ov=-8) == BAD_SHAPE
    assert call(seg=3936 * 8, sea=704, ov=576) == BAD_SHAPE                # 254 KB of shared memory
    assert "tempo_gain" in L.last_error()


def test_kernel_compiles_without_spills_or_local_memory(tmp_path):
    """tempo_gain.cu recompiled with build.sh's flags and -Xptxas -v: no stack frame and no spill stores; and in the built
    library, STACK:0 LOCAL:0 (cuobjdump -res-usage)."""
    import os
    import re
    import subprocess
    from tests.test_engine_build import CSRC, CUOBJDUMP, LIB, NVCC, ROOT, _build_flags, _need
    _need(NVCC)
    log = subprocess.run([NVCC, *_build_flags(), "-Xptxas", "-v,-warn-spills", "-c", os.path.join(CSRC, "tempo_gain.cu"),
                          "-o", str(tmp_path / "tempo_gain.o")], capture_output=True, text=True, cwd=ROOT, check=True).stderr
    props = re.findall(r"Function properties for (\S*tempo_gain_kernel\S*)\s*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores",
                       log)
    assert len(props) == 1 and props[0][1:] == ("0", "0"), log[-2000:]
    _need(CUOBJDUMP, LIB)
    out = subprocess.run([CUOBJDUMP, "-res-usage", LIB], check=True, capture_output=True, text=True).stdout
    usage = [u for n, u in re.findall(r"Function (\S+):\s*\n\s*(REG:.*)", out) if "tempo_gain_kernel" in n]
    assert len(usage) == 1 and re.search(r"\bSTACK:0\b", usage[0]) and re.search(r"\bLOCAL:0\b", usage[0]), usage
