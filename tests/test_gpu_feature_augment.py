"""The device front end's loader options (b200asr_stft_features_ex, spectrogram_batch's window / noise / max_frames,
NoiseBank, collate_waves) against tests/augment_oracle.py and the reference's fixture tests/golden/noise.npz.

Raw-ABI calls get a NaN workspace of exactly the stated size followed by a NaN guard, and an output between sentinel bands
(tests/test_gpu_linear_precisions.py's Banded).  Launch counts: b200asr_stft_features_ex enqueues what
b200asr_stft_features does (pad, basis, GEMM, magnitudes, + statistics and normalisation), and 2 more with noise (the
energies and their reduction)."""
import os

import numpy as np
import pytest
import torch

from oracle import ref_shim
from tests import augment_oracle as AO
from tests.helpers import rel_err
from tests.test_gpu_linear_precisions import Banded, _waves

pytestmark = pytest.mark.gpu

NAN = float("nan")
OK, BAD_SHAPE, BAD_ARG = 0, -1, -5
GUARD = 1024
NO_CUT = 2 ** 31 - 1
BARS = {0: 2e-5, 3: 5e-5, 1: 5e-3}               # tests/test_features.py's
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "noise.npz")
CONF = dict(sample_rate=16000, window_size=0.02, window_stride=0.01, window="hamming", noise_dir=None, noise_prob=0.4,
            noise_levels=(0.0, 0.5))


@pytest.fixture(scope="module")
def L():
    import b200asr
    b200asr._lib.load(check_device=True)
    return b200asr._lib


def _launches(L):
    return L.load().b200asr_launch_count()


def _batch(waves, Lmax=None):
    lens = [len(w) for w in waves]
    Lmax = Lmax or max(1, max(lens))
    wave = torch.full((len(waves), Lmax), NAN)                       # samples past each length must not be read
    for i, w in enumerate(waves):
        wave[i, :len(w)] = torch.from_numpy(np.asarray(w, np.float32))
    return wave.cuda(), torch.tensor(lens, dtype=torch.int32, device="cuda")


def _ex(L, wave, lens, Tmax, window=0, noise=None, max_frames=NO_CUT, prec=3, reflect=1, normalize=1, periodic=0, ex=True):
    """One raw call (the extended entry point, or b200asr_stft_features with ex=False): (rc, out, frames, launches)."""
    lib = L.load()
    B, Lmax = wave.shape
    nws = (lib.b200asr_stft_features_ex_ws_bytes if ex else lib.b200asr_stft_ws_bytes)(B, Lmax, 320, 160) // 4
    buf = torch.full((nws + GUARD,), NAN, device="cuda")
    out = Banded((B, 1, 161, Tmax))
    frames = torch.full((B,), -1, dtype=torch.int32, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    n0 = _launches(L)
    if ex:
        bank, bank_len, start, level = noise if noise is not None else (None, 0, None, None)
        rc = lib.b200asr_stft_features_ex(L.ptr(wave), L.ptr(lens), L.ptr(out.t), L.ptr(frames), L.ptr(buf), B, Lmax, Tmax, 320, 160,
                                          reflect, normalize, window, periodic, L.ptr(bank), bank_len, L.ptr(start), L.ptr(level),
                                          max_frames, prec, st)
    else:
        rc = lib.b200asr_stft_features(L.ptr(wave), L.ptr(lens), L.ptr(out.t), L.ptr(frames), L.ptr(buf), B, Lmax, Tmax, 320, 160,
                                       reflect, normalize, periodic, prec, st)
    n = _launches(L) - n0
    torch.cuda.synchronize()
    assert bool(buf[nws:].isnan().all()) and out.bands_intact()
    return rc, out.t, frames, n


def _noise_args(bank, starts, levels):
    return (bank, bank.numel(), torch.tensor(starts, dtype=torch.int64, device="cuda"),
            torch.tensor(levels, dtype=torch.float32, device="cuda"))


def _oracle(waves, Tmax, window="hamming", reflect=True, normalize=True, periodic=False, max_frames=None):
    out = np.zeros((len(waves), 1, 161, Tmax), dtype=np.float32)
    for b, y in enumerate(waves):
        if len(y) == 0:
            continue                                                   # one frame of zeros
        s = AO.log_spectrogram(np.asarray(y, np.float64), window_name=window, periodic=periodic, reflect=reflect,
                               normalize=normalize, max_frames=max_frames)
        out[b, 0, :, :s.shape[1]] = s[:, :Tmax]
    return torch.from_numpy(out)


@pytest.mark.parametrize("prec", [0, 1, 3])
@pytest.mark.parametrize("reflect", [True, False])
@pytest.mark.parametrize("window", ["hamming", "hann", "blackman", "bartlett", "kaiser"])
def test_windows_match_oracle(window, reflect, prec):
    import b200asr
    waves = _waves([16000, 12345, 8000, 700, 160], seed=3)
    for periodic in (False, True):
        want = _oracle(waves, 101, window, reflect, periodic=periodic)
        got, pct, sizes = b200asr.spectrogram_batch([torch.from_numpy(w).cuda() for w in waves], reflect=reflect, precision=prec,
                                                    window_periodic=periodic, window=window)
        assert got.shape == want.shape and sizes.tolist() == [101, 78, 51, 5, 2]
        assert rel_err(got, want) < BARS[prec], (window, periodic)


def test_ex_defaults_are_the_plain_call_bit_for_bit(L):
    """Hamming, no noise, no cut: the bits of b200asr_stft_features, also with Lmax past the longest utterance, Tmax past
    every utterance's frames, and without normalisation; the same launches."""
    lens = [16000, 12345, 700, 1, 159, 161]
    waves = _waves(lens, seed=8)
    for Lmax, Tmax, normalize, prec in ((16000, 101, 1, 3), (17777, 112, 1, 0), (16000, 101, 0, 1), (16000, 101, 1, 1)):
        wave, lt = _batch(waves, Lmax)
        a = _ex(L, wave, lt, Tmax, prec=prec, normalize=normalize, ex=False)
        b = _ex(L, wave, lt, Tmax, prec=prec, normalize=normalize)
        assert a[0] == b[0] == OK and a[3] == b[3] == (6 if normalize else 4)
        assert torch.equal(a[1], b[1]) and torch.equal(a[2], b[2]), (Lmax, Tmax, normalize, prec)


def test_cut_normalises_over_the_whole_utterance(L):
    """max_frames cuts after whole-utterance statistics (the oracle's order); a cut no utterance reaches is bit-identical
    to no cut; frames_out reports the kept count."""
    lens = [48000, 16000, 6400, 1600, 300]
    waves = _waves(lens, seed=11)
    wave, lt = _batch(waves)
    full = _ex(L, wave, lt, 301)
    for cut in (301, 302, 5000):
        same = _ex(L, wave, lt, 301, max_frames=cut)
        assert torch.equal(same[1], full[1]) and torch.equal(same[2], full[2]), cut
    for cut, Tmax in ((40, 40), (100, 100), (1, 1), (40, 301)):
        rc, out, frames, _ = _ex(L, wave, lt, Tmax, max_frames=cut)
        assert rc == OK and frames.tolist() == [min(1 + n // 160, cut, Tmax) for n in lens]
        assert rel_err(out, _oracle(waves, Tmax, max_frames=cut)) < BARS[3], cut
    got, pct, sizes = __import__("b200asr").spectrogram_batch([torch.from_numpy(w).cuda() for w in waves], max_frames=40)
    assert got.shape[3] == 40 and sizes.tolist() == [40, 40, 40, 11, 2]
    assert rel_err(got, _oracle(waves, 40, max_frames=40)) < BARS[3]


def _mixed(waves, bank_np, starts, levels):
    out = []
    for y, s, lv in zip(waves, starts, levels):
        out.append(AO.mix(y, bank_np[s:s + len(y)], lv) if s >= 0 and len(y) else np.asarray(y, np.float64))
    return out


def test_noise_edges(L):
    """Lengths 0, 1, hop - 1, hop, hop + 1 and longer ones with noise against the oracle; a segment that ends exactly at
    the end of the bank; a silent segment turns its utterance into NaN (0/0, as numpy); a silent utterance is unchanged;
    an utterance without noise in a noisy batch is bit-identical to the same batch without noise."""
    g = np.random.default_rng(5)
    lens = [0, 1, 159, 160, 161, 4000, 12345, 3000]
    waves = _waves(lens, seed=6)
    bank_np = (0.3 * g.standard_normal(40000)).astype(np.float32)
    bank = torch.from_numpy(bank_np).cuda()
    starts = [0, 17, 100, 2000, 5000, 9000, 40000 - 12345, -1]
    levels = [0.3, 0.2, 0.45, 0.1, 0.33, 0.25, 0.4, 0.5]
    wave, lt = _batch(waves)
    Tmax = 1 + max(lens) // 160
    rc, out, frames, n_noise = _ex(L, wave, lt, Tmax, noise=_noise_args(bank, starts, levels))
    _, plain, _, n_plain = _ex(L, wave, lt, Tmax)
    assert rc == OK and n_noise == n_plain + 2 and frames.tolist() == [1 + n // 160 for n in lens]
    assert bool(torch.isfinite(out).all())
    assert rel_err(out, _oracle(_mixed(waves, bank_np, starts, levels), Tmax)) < BARS[3]
    assert torch.equal(out[7], plain[7]) and float(out[0].abs().max()) == 0.0
    # silent segment -> NaN; silent utterance -> unchanged (its features are those of silence)
    silent_bank = bank.clone()
    silent_bank[1000:1000 + 4000] = 0
    waves2 = [waves[5], np.zeros(3000, np.float32), waves[6]]
    wave2, lt2 = _batch(waves2)
    T2 = 1 + 12345 // 160
    rc, out2, _, _ = _ex(L, wave2, lt2, T2, noise=_noise_args(silent_bank, [1000, 5000, -1], [0.3, 0.3, 0.3]))
    _, plain2, _, _ = _ex(L, wave2, lt2, T2)
    assert rc == OK and bool(out2[0, :, :, :26].isnan().all())
    assert torch.equal(out2[1], plain2[1]) and torch.equal(out2[2], plain2[2])


def test_segment_past_the_bank_is_nan_not_read(L):
    """The starts are device data: an utterance whose segment leaves the bank comes back NaN, the others are unaffected."""
    waves = _waves([4000, 4000], seed=9)
    bank = torch.randn(5000, device="cuda")
    wave, lt = _batch(waves)
    rc, out, _, _ = _ex(L, wave, lt, 26, noise=_noise_args(bank, [1001, 1000], [0.2, 0.2]))
    assert rc == OK and bool(out[0].isnan().all()) and bool(torch.isfinite(out[1]).all())


def test_rejections_launch_and_write_nothing(L):
    waves = _waves([4000, 2500], seed=1)
    wave, lt = _batch(waves)
    bank = torch.randn(5000, device="cuda")
    good = _noise_args(bank, [0, 10], [0.1, 0.1])
    cases = [("window 4", dict(window=4), BAD_ARG), ("window -1", dict(window=-1), BAD_ARG),
             ("bank without starts", dict(noise=(bank, 5000, None, good[3])), BAD_ARG),
             ("starts without bank", dict(noise=(None, 5000, good[2], good[3])), BAD_ARG),
             ("empty bank", dict(noise=(bank, 0, good[2], good[3])), BAD_SHAPE),
             ("max_frames 0", dict(max_frames=0), BAD_SHAPE), ("Tmax", dict(Tmax=27), BAD_SHAPE), ("prec 2", dict(prec=2), BAD_ARG)]
    for what, kw, code in cases:
        Tmax = kw.pop("Tmax", 26)
        rc, out, frames, n = _ex(L, wave, lt, Tmax, **kw)
        assert rc == code and n == 0, what
        assert bool(out.isnan().all()) and frames.tolist() == [-1, -1], what


def _golden():
    return dict(np.load(GOLDEN))


def _split(flat, lengths):
    return np.split(flat, np.cumsum(lengths)[:-1])


def _fixture_case(G, c):
    lengths = G[f"c{c}.lengths"]
    waves = _split(G[f"c{c}.waves"], lengths)
    ids = [t.tolist() for t in _split(G[f"c{c}.ids"], G[f"c{c}.id_lengths"])]
    conf = dict(CONF, window=str(G[f"c{c}.window"]), noise_dir="noise", noise_prob=float(G[f"c{c}.cfg"][0]),
                noise_levels=tuple(G["meta.noise_levels"]))
    return list(zip(waves, ids)), conf, int(G[f"c{c}.cfg"][1])


@pytest.mark.parametrize("case", range(5))
def test_collate_waves_matches_the_reference_loader(case):
    """Noise, window, normalisation, cut and collation against the reference's _collate_fn output: devices, dtypes,
    order, sizes, percentages and targets exact; inputs to the 3xTF32 bar."""
    import b200asr
    G = _golden()
    bank = b200asr.NoiseBank(_split(G["meta.clips"], G["meta.clip_lengths"]), 16000)
    batch, conf, src_max_len = _fixture_case(G, case)
    np.random.seed(4321 + case)
    inputs, targets, pct, sizes, tsizes = b200asr.collate_waves(batch, conf, src_max_len, bank, precision=3)
    assert inputs.is_cuda and not any(t.is_cuda for t in (targets, pct, sizes, tsizes))
    assert (inputs.dtype, targets.dtype, pct.dtype, sizes.dtype, tsizes.dtype) == (torch.float32, torch.int64, torch.float32,
                                                                                    torch.int32, torch.int32)
    assert torch.equal(targets, torch.from_numpy(G[f"c{case}.targets"])) and torch.equal(pct, torch.from_numpy(G[f"c{case}.pct"]))
    assert torch.equal(sizes, torch.from_numpy(G[f"c{case}.sizes"])) and torch.equal(tsizes, torch.from_numpy(G[f"c{case}.tsizes"]))
    want = torch.from_numpy(G[f"c{case}.inputs"])
    assert inputs.shape == want.shape and rel_err(inputs, want) < BARS[3]
    pad = torch.arange(want.shape[3])[None, :] >= sizes[:, None].long()
    assert bool((inputs.cpu()[pad[:, None, None, :].expand_as(inputs)] == 0).all())                     # zero padded


def test_collate_waves_noise_prob_zero_repeats_and_syncs(L):
    """noise_prob 0 gives the bits of a configuration without noise; repeated calls with noise give identical bits; a
    call makes no host synchronisation and enqueues the stated launches."""
    import b200asr
    G = _golden()
    bank = b200asr.NoiseBank(_split(G["meta.clips"], G["meta.clip_lengths"]), 16000)
    batch, conf, _ = _fixture_case(G, 1)
    quiet = b200asr.collate_waves(batch, dict(conf, noise_prob=0.0), 4000, bank)
    plain = b200asr.collate_waves(batch, dict(conf, noise_dir=None), 4000)
    assert all(torch.equal(a, b) for a, b in zip(quiet, plain))
    rng = lambda: np.random.RandomState(3)                              # noqa: E731
    conf1 = dict(conf, noise_prob=1.0)
    first = b200asr.collate_waves(batch, conf1, 4000, bank, rng=rng())
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        n0 = _launches(L)
        again = b200asr.collate_waves(batch, conf1, 4000, bank, rng=rng())
        n_noise = _launches(L) - n0
        n0 = _launches(L)
        b200asr.collate_waves(batch, dict(conf, noise_dir=None), 4000)
        n_plain = _launches(L) - n0
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert all(torch.equal(a, b) for a, b in zip(first, again))
    assert n_noise == n_plain + 2 and n_plain == 6
    assert not torch.equal(first[0], plain[0])


def test_collate_waves_too_short_clip_raises_before_any_launch(L):
    import b200asr
    bank = b200asr.NoiseBank([np.ones(1000, np.float32)], 16000)
    n0 = _launches(L)
    with pytest.raises(ValueError):
        b200asr.collate_waves([(np.ones(1600, np.float32), [1, 4, 2])], dict(CONF, noise_dir="n", noise_prob=1.0), 4000, bank)
    assert _launches(L) == n0


@pytest.mark.skipif(not ref_shim.available(), reason="reference checkout not staged (oracle/make_ref.py)")
def test_collate_waves_batch_trains_the_installed_reference():
    """A collate_waves batch through the reference's Transformer.forward and calculate_metrics, as trainer.py:58-85 runs
    them, with b200asr installed: a finite loss."""
    import b200asr
    ns = ref_shim.load(["--num-layers", "1", "--num-heads", "2", "--dim-model", "64", "--dim-emb", "64", "--dim-key", "32",
                        "--dim-value", "32", "--dim-inner", "128", "--feat_extractor", "vgg_cnn", "--tgt-max-len", "20",
                        "--dropout", "0.0"])
    l2i, i2l = ref_shim.labels(40)
    torch.manual_seed(1)
    model = ns.functions.init_transformer_model(ns.constant.args, l2i, i2l).cuda()
    model.train()
    g = np.random.default_rng(2)
    batch = [(w, [1] + g.integers(3, 40, 3 + b).tolist() + [2]) for b, w in enumerate(_waves([8000, 16000, 4000, 11111], seed=4))]
    bank = b200asr.NoiseBank(_waves([20000, 30000], seed=5), 16000)
    src, tgt, pct, lens, tlens = b200asr.collate_waves(batch, dict(CONF, noise_dir="n", noise_prob=0.5), 4000, bank,
                                                       rng=np.random.RandomState(0))
    b200asr.install()
    try:
        pred, gold, hyp, gold_seq = model(src, lens, tgt.cuda(), verbose=False)
        sizes = pct.mul_(int(pred.size(1))).int()
        loss, n_correct = ns.metrics.calculate_metrics(pred, gold, input_lengths=sizes, target_lengths=tlens, smoothing=0.1,
                                                       loss_type="ce")
        loss.backward()
    finally:
        b200asr.uninstall()
    assert bool(torch.isfinite(loss.detach())) and float(loss.detach()) > 0
