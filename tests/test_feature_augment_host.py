"""CPU checks of the loader options of the feature front end: the windows of tests/augment_oracle.py against scipy, and the
oracle, `NoiseBank.draw` and `collate_waves`' host side against tests/golden/noise.npz, which the unmodified reference's
SpectrogramDataset / NoiseInjection / _collate_fn wrote (tests/golden/make_noise_golden.py)."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import ref_shim
from tests import augment_oracle as AO

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "noise.npz")


def _golden():
    return dict(np.load(GOLDEN))


def _cases(G):
    n = 0
    while f"c{n}.cfg" in G:
        n += 1
    return range(n)


def _split(flat, lengths):
    return np.split(flat, np.cumsum(lengths)[:-1])


def _bank(G):
    import b200asr
    return b200asr.NoiseBank(_split(G["meta.clips"], G["meta.clip_lengths"]), int(G["meta.cfg"][0]), device="cpu")


@pytest.mark.parametrize("n_fft", [320, 31, 161, 256, 33])
@pytest.mark.parametrize("name", AO.WINDOWS)
def test_oracle_windows_are_scipys(name, n_fft):
    from scipy.signal import windows
    for sym in (True, False):
        assert np.allclose(AO.window(name, n_fft, periodic=not sym), getattr(windows, name)(n_fft, sym=sym), rtol=0, atol=1e-15)
    assert np.array_equal(AO.window("kaiser", n_fft), AO.window("hamming", n_fft))       # data_loader.py:52 falls back


def test_fixture_windows_are_the_oracles():
    G = _golden()
    for c in _cases(G):
        name = str(G[f"c{c}.window"])
        assert np.allclose(G[f"c{c}.win"], AO.window(name, 320), rtol=0, atol=1e-15), name


def test_noise_draws_match_the_reference():
    """NoiseBank.draw makes the reference's numpy calls in its order: add, clip, level exact; the segment position in
    seconds bit for bit; the start sample as the fixture's trim restatement."""
    G = _golden()
    bank = _bank(G)
    sr = bank.sample_rate
    for c in _cases(G):
        prob = float(G[f"c{c}.cfg"][0])
        lengths = G[f"c{c}.lengths"]
        np.random.seed(4321 + c)
        d = bank.draw(lengths, prob, tuple(G["meta.noise_levels"]), np.random)
        assert np.array_equal(d.add, G[f"c{c}.add"]) and np.array_equal(d.clip, G[f"c{c}.clip"]), c
        noisy = d.add == 1
        assert np.array_equal(d.level[noisy], G[f"c{c}.level"][noisy]) and np.isnan(d.level[~noisy]).all()
        for b in np.flatnonzero(noisy):
            clip_len, n = int(bank.lengths[d.clip[b]]), int(lengths[b])
            secs = d.rand[b] * (clip_len / sr - n / sr)
            assert secs == G[f"c{c}.noise_start"][b]
            s = min(max(int(round(secs * sr)), 0), clip_len - n)
            assert d.start[b] == bank.offsets[d.clip[b]] + s
        assert (d.start[~noisy] == -1).all()


def test_oracle_mix_and_cut_spectrograms_match_the_reference():
    """The float64 mix agrees with the waveform the reference handed to librosa.stft within 1e-5 of the noise term; the
    normalised, cut spectrograms within 1e-5."""
    G = _golden()
    bank = _bank(G)
    for c in _cases(G):
        lengths = G[f"c{c}.lengths"]
        waves, mixed = _split(G[f"c{c}.waves"], lengths), _split(G[f"c{c}.mixed"], lengths)
        frames = G[f"c{c}.frames"]
        specs = _split(G[f"c{c}.spect"], 161 * frames)
        src_max_len = int(G[f"c{c}.cfg"][1])
        np.random.seed(4321 + c)
        d = bank.draw(lengths, float(G[f"c{c}.cfg"][0]), tuple(G["meta.noise_levels"]), np.random)
        for b, n in enumerate(lengths):
            y = waves[b].astype(np.float64)
            if d.add[b]:
                seg = bank.bank.numpy()[d.start[b]:d.start[b] + n]
                y = AO.mix(y, seg, d.level[b])
                term = np.abs(y - waves[b]).max()
                assert np.abs(y - mixed[b]).max() <= 1e-5 * term, (c, b)
            else:
                assert np.array_equal(mixed[b], waves[b])
            want = specs[b].reshape(161, frames[b])
            got = AO.log_spectrogram(y, window_name=str(G[f"c{c}.window"]), max_frames=src_max_len)
            assert got.shape == want.shape and frames[b] == min(1 + n // 160, src_max_len)
            assert np.abs(got - want).max() <= 1e-5 * np.abs(want).max(), (c, b)


def test_oracle_collate_matches_the_reference():
    G = _golden()
    for c in _cases(G):
        frames = G[f"c{c}.frames"]
        specs = [s.reshape(161, f) for s, f in zip(_split(G[f"c{c}.spect"], 161 * frames), frames)]
        ids = _split(G[f"c{c}.ids"], G[f"c{c}.id_lengths"])
        order, inputs, tgt, pct, sizes, tsizes = AO.collate(specs, ids)
        assert np.array_equal(inputs, G[f"c{c}.inputs"]) and np.array_equal(tgt, G[f"c{c}.targets"])
        assert np.array_equal(pct, G[f"c{c}.pct"]) and np.array_equal(sizes, G[f"c{c}.sizes"])
        assert np.array_equal(tsizes, G[f"c{c}.tsizes"])
        assert G[f"c{c}.targets"].dtype == np.int64 and G[f"c{c}.sizes"].dtype == np.int32
        assert G[f"c{c}.pct"].dtype == np.float32 and G[f"c{c}.tsizes"].dtype == np.int32


def test_draw_rejects_a_clip_shorter_than_the_utterance():
    import b200asr
    bank = b200asr.NoiseBank([np.ones(100, np.float32)], 16000, device="cpu")
    with pytest.raises(ValueError, match="fewer than"):
        bank.draw([101], 1.0, (0.0, 0.5), np.random.RandomState(0))
    d = bank.draw([100], 1.0, (0.0, 0.5), np.random.RandomState(0))          # a segment that is the whole clip
    assert d.start.tolist() == [0]


def test_collate_waves_needs_a_bank_when_the_config_has_noise():
    import b200asr
    conf = dict(sample_rate=16000, window_size=0.02, window_stride=0.01, window="hamming", noise_dir="noise", noise_prob=0.4,
                noise_levels=(0.0, 0.5))
    with pytest.raises(ValueError, match="noise_bank"):
        b200asr.collate_waves([(np.zeros(1600, np.float32), [1, 5, 2])], conf, 4000)


@pytest.mark.skipif(not ref_shim.available(), reason="reference checkout not staged (oracle/make_ref.py)")
def test_make_noise_golden_reproduces_the_fixture(tmp_path):
    out = tmp_path / "noise.npz"
    r = subprocess.run([sys.executable, "-W", "ignore", os.path.join(HERE, "golden", "make_noise_golden.py"), "--out", str(out)],
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    assert out.read_bytes() == open(GOLDEN, "rb").read()
