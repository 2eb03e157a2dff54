"""CPU checks of the installed AudioDataLoader's host side (end2end-asr-pytorch_b200/loader.py) against the UNMODIFIED
reference loader (utils/data_loader.py): the worker-side items make the reference's random draws, collate_items gives
_collate_fn's host tensors, workers draw as the reference's workers do, and install() binds and restores the class.

What is not installed is stubbed as tests/golden/make_noise_golden.py stubs it: `librosa` (find_files lists the clips,
stft records the waveform it is handed and returns tests/augment_oracle.stft), `torchaudio`, and the audio helpers
data_loader.py imported (load_audio, get_audio_length, audio_with_sox with the trim restated), with clips and utterances
served from memory; utils.audio.augment_audio_with_sox records the tempo and gain it gets."""
import importlib
import pickle
import random
import sys
import types

import numpy as np
import pytest
import torch

from oracle import ref_shim
from tests import augment_oracle as AO

pytestmark = pytest.mark.skipif(not ref_shim.available(), reason="reference checkout not staged (oracle/make_ref.py)")

SR = 16000
VOCAB = "abcdefgh "
CLIP_LENGTHS = [40000, 36000, 52000]


def _signals(seed, lengths, scale):
    g = np.random.default_rng(seed)
    return [(scale * np.sin(2 * np.pi * (150 + 300 * g.random()) * np.arange(n) / SR) + 0.05 * g.standard_normal(n))
            .astype(np.float32) for n in lengths]


class Env:
    """The reference's data_loader with its I/O served from memory; records what the reference computes."""

    def __init__(self, mp):
        import scipy.signal
        for name in ("hamming", "hann", "blackman", "bartlett"):
            if not hasattr(scipy.signal, name):
                mp.setattr(scipy.signal, name, getattr(scipy.signal.windows, name), raising=False)
        for name in ("librosa", "torchaudio"):
            if name not in sys.modules:
                try:
                    importlib.import_module(name)
                except ImportError:
                    mp.setitem(sys.modules, name, types.ModuleType(name))
        if torch.utils.data.Sampler.__init__ is object.__init__:   # torch >= 2.2 dropped Sampler(data_source)
            mp.setattr(torch.utils.data.Sampler, "__init__", lambda self, data_source=None: None)
        self.ns = ref_shim.load(["--src-max-len", "4000"])
        self.DL = importlib.import_module("utils.data_loader")
        self.audio = importlib.import_module("utils.audio")
        self.clips = {f"noise_{i}.wav": w for i, w in enumerate(_signals(99, CLIP_LENGTHS, 0.2))}
        self.rates = {}
        self.utts = {}
        self.stft_calls, self.sox, self.loads, self.augments = [], [], [], []
        lib = types.SimpleNamespace(util=types.SimpleNamespace(find_files=lambda path: sorted(self.clips)),
                                    stft=self._stft,
                                    magphase=lambda D: (np.abs(D), D / np.where(np.abs(D) == 0, 1, np.abs(D))))
        mp.setattr(self.DL, "librosa", lib)
        mp.setattr(self.DL, "load_audio", self._load)
        mp.setattr(self.DL, "get_audio_length", lambda p: len(self.clips[p]) / self.rates.get(p, SR))
        mp.setattr(self.DL, "audio_with_sox", self._sox)
        mp.setattr(self.audio, "augment_audio_with_sox", self._augment)
        l2i = {c: i for i, c in enumerate([self.ns.constant.PAD_CHAR, self.ns.constant.SOS_CHAR, self.ns.constant.EOS_CHAR] + list(VOCAB))}
        self.label2id = l2i

    def _stft(self, y, n_fft, hop_length, win_length, window):
        win = np.asarray(window(n_fft), dtype=np.float64)
        self.stft_calls.append(np.array(y, copy=True))
        return AO.stft(y, n_fft, hop_length, win)

    def _load(self, path):
        self.loads.append(path)
        return (self.utts[path] if path in self.utts else self.clips[path]).copy()

    def _sox(self, path, sample_rate, start_time, end_time):
        clip = self.clips[path]
        n = int(round((end_time - start_time) * SR))
        s = min(max(int(round(start_time * SR)), 0), len(clip) - n)
        self.sox.append((path, start_time))
        return clip[s:s + n].copy()

    def _augment(self, path, sample_rate, tempo, gain):
        self.augments.append((tempo, gain))
        return self._load(path)

    def dataset(self, tmp, lengths, prob=0.5, window="hamming", augment=False, manifests=2, seed=0, src_max_len=4000):
        """SpectrogramDataset over `manifests` manifests of utterances of `lengths` samples, with noise at `prob`
        (None: no noise_dir)."""
        self.ns.constant.args.src_max_len = src_max_len
        waves = _signals(1000 + seed, lengths, 0.5)
        files = []
        for m in range(manifests):
            path = tmp / f"m{seed}_{m}.csv"
            with open(path, "w") as f:
                for b, w in enumerate(waves):
                    wav, txt = str(tmp / f"u{seed}_{m}_{b}.wav"), tmp / f"u{seed}_{m}_{b}.txt"
                    self.utts[wav] = w if m == 0 else (0.5 * w)
                    txt.write_text("".join(VOCAB[(m + 3 * b + k) % len(VOCAB)] for k in range(2 + (5 * b + m) % 7)))
                    f.write(f"{wav},{txt}\n")
            files.append(str(path))
        conf = dict(sample_rate=SR, window_size=0.02, window_stride=0.01, window=window, noise_dir=str(tmp) if prob is not None else None,
                    noise_prob=prob, noise_levels=(0.0, 0.5))
        return self.DL.SpectrogramDataset(conf, files, self.label2id, normalize=True, augment=augment)

    def clip_set(self):
        import b200asr
        return b200asr.NoiseClips([len(self.clips[p]) for p in sorted(self.clips)], SR)

    def bank_np(self):
        return np.concatenate([self.clips[p] for p in sorted(self.clips)])


@pytest.fixture
def env(monkeypatch):
    return Env(monkeypatch)


def _seed(s):
    random.seed(s)
    np.random.seed(s)


def _rng_state():
    st = np.random.get_state()
    return random.getstate(), st[1].tobytes(), st[2:]


@pytest.mark.parametrize("augment", [False, True])
@pytest.mark.parametrize("prob", [0.0, 0.5, 1.0])
def test_items_make_the_reference_draws(env, tmp_path, prob, augment):
    """Manifest choice, the augment draws, binomial, choice, uniform and rand: the same calls with the same outcomes as the
    unmodified __getitem__ on the same seeds (equal generator states after every item); the float64 mix of the item's
    draws matches the waveform the reference handed to librosa.stft."""
    from b200asr import loader
    lengths = [8000, 12345, 3200, 161, 30000, 16000]
    ds = env.dataset(tmp_path, lengths, prob=prob, augment=augment)
    items = loader.PackedItems(ds, env.clip_set())
    names, bank = sorted(env.clips), env.bank_np()
    offsets = np.concatenate([[0], np.cumsum(CLIP_LENGTHS)[:-1]])
    for seed in (1, 2):
        _seed(seed)
        env.stft_calls.clear(), env.sox.clear(), env.loads.clear(), env.augments.clear()
        ref, ref_states = [], []
        levels = []
        orig_inject = env.DL.NoiseInjection.inject_noise_sample
        env.DL.NoiseInjection.inject_noise_sample = lambda self, d, p, lv: (levels.append((p, lv)), orig_inject(self, d, p, lv))[1]
        try:
            for i in range(len(lengths)):
                ref.append(ds[i])
                ref_states.append(_rng_state())
        finally:
            env.DL.NoiseInjection.inject_noise_sample = orig_inject
        ref_loads, ref_aug, ref_sox, mixes = list(env.loads), list(env.augments), list(env.sox), list(env.stft_calls)
        _seed(seed)
        env.loads.clear(), env.augments.clear()
        got = []
        for i in range(len(lengths)):
            got.append(items[i])
            assert _rng_state() == ref_states[i], (seed, i)
        assert env.loads == ref_loads and env.augments == ref_aug and len(env.augments) == (len(lengths) if augment else 0)
        k = 0
        for i, (it, (spect, ids)) in enumerate(zip(got, ref)):
            assert it.ids == ids and it.frames == spect.shape[1] and it.wave.dtype == np.float32
            if it.noise_clip < 0:
                assert it.noise_start == -1 and np.isnan(it.noise_level)
                assert np.array_equal(mixes[i], it.wave)
                continue
            path, level = levels[k]
            assert ref_sox[k][0] == path == names[it.noise_clip] and it.noise_level == level
            n = len(it.wave)
            want = min(max(int(round(ref_sox[k][1] * SR)), 0), CLIP_LENGTHS[it.noise_clip] - n)
            assert it.noise_start == offsets[it.noise_clip] + want
            y = AO.mix(it.wave, bank[it.noise_start:it.noise_start + n], it.noise_level)
            term = np.abs(y - it.wave).max()
            assert np.abs(y - mixes[i]).max() <= 1e-5 * term, (seed, i)
            k += 1
        assert k == len(levels) and (prob != 1.0 or k == len(lengths)) and (prob != 0.0 or k == 0)


def test_items_replay_the_golden_fixture(env, tmp_path):
    """tests/golden/noise.npz, which the unmodified reference wrote, replays through PackedItems: draws, ids, frames."""
    from b200asr import loader
    import b200asr
    G = dict(np.load(str(__import__("os").path.join(__import__("os").path.dirname(__file__), "golden", "noise.npz"))))
    clip_lengths = G["meta.clip_lengths"]
    clips = np.split(G["meta.clips"], np.cumsum(clip_lengths)[:-1])
    env.clips = {f"noise_{i}.wav": c for i, c in enumerate(clips)}
    nclips = b200asr.NoiseClips(clip_lengths, SR)
    c = 0
    while f"c{c}.cfg" in G:
        lengths = G[f"c{c}.lengths"]
        waves = np.split(G[f"c{c}.waves"], np.cumsum(lengths)[:-1])
        ids = np.split(G[f"c{c}.ids"], np.cumsum(G[f"c{c}.id_lengths"])[:-1])
        prob, src_max_len = float(G[f"c{c}.cfg"][0]), int(G[f"c{c}.cfg"][1])
        ds = env.dataset(tmp_path, lengths, prob=prob, window=str(G[f"c{c}.window"]), manifests=1, seed=50 + c,
                         src_max_len=src_max_len)
        for b, w in enumerate(waves):
            env.utts[ds.ids_list[0][b][0]] = w
            with open(ds.ids_list[0][b][1], "w") as f:
                f.write("".join(VOCAB[(c + 3 * b + k) % len(VOCAB)] for k in range(2 + (5 * b + c) % 7)))
        items = loader.PackedItems(ds, nclips)
        np.random.seed(4321 + c)
        got = [items[b] for b in range(len(lengths))]
        assert [it.noise_clip for it in got] == G[f"c{c}.clip"].tolist()
        assert [int(it.noise_clip >= 0) for it in got] == G[f"c{c}.add"].tolist()
        for b, it in enumerate(got):
            assert it.ids == ids[b].tolist() and it.frames == G[f"c{c}.frames"][b]
            if it.noise_clip >= 0:
                assert it.noise_level == G[f"c{c}.level"][b]
                n = len(it.wave)
                s = min(max(int(round(G[f"c{c}.noise_start"][b] * SR)), 0), int(clip_lengths[it.noise_clip]) - n)
                assert it.noise_start == nclips.offsets[it.noise_clip] + s
        pb = loader.collate_items(got)
        assert torch.equal(pb.targets, torch.from_numpy(G[f"c{c}.targets"])) and torch.equal(pb.input_percentages, torch.from_numpy(G[f"c{c}.pct"]))
        assert torch.equal(pb.input_sizes, torch.from_numpy(G[f"c{c}.sizes"])) and torch.equal(pb.target_sizes, torch.from_numpy(G[f"c{c}.tsizes"]))
        c += 1
    assert c == 5


@pytest.mark.parametrize("src_max_len", [4000, 11, 1])
def test_collate_matches_collate_fn(env, tmp_path, src_max_len):
    """Order, targets, sizes and percentages equal _collate_fn's exactly (values and dtypes), with ties in frame count
    (equal lengths, lengths in the same frame, and the cut); the waveforms are packed in that order."""
    from b200asr import loader
    lengths = [1600, 1600, 1700, 1500, 1650, 161, 1759, 3000, 1600, 159]
    ds = env.dataset(tmp_path, lengths, prob=0.5, src_max_len=src_max_len, manifests=1)
    items = loader.PackedItems(ds, env.clip_set())
    for perm in (list(range(10)), [9, 3, 0, 8, 1, 4, 2, 6, 5, 7]):
        np.random.seed(5)
        ref = [ds[i] for i in perm]
        np.random.seed(5)
        got = [items[i] for i in perm]
        want = env.DL._collate_fn(ref)
        pb = loader.collate_items(got)
        for a, b in zip((pb.targets, pb.input_percentages, pb.input_sizes, pb.target_sizes), want[1:]):
            assert a.dtype == b.dtype and torch.equal(a, b)
        assert pb.src_max_len == src_max_len and pb.offsets.dtype == torch.int64 and pb.lengths.dtype == torch.int32
        order = sorted(range(len(got)), key=lambda i: got[i].frames, reverse=True)
        for r, i in enumerate(order):
            o, n = int(pb.offsets[r]), int(pb.lengths[r])
            assert n == len(got[i].wave) and np.array_equal(pb.wave[o:o + n].numpy(), got[i].wave)
            assert int(pb.noise_start[r]) == got[i].noise_start and int(pb.noise_clip[r]) == got[i].noise_clip
        assert pb.wave.numel() == sum(lengths)


def test_items_and_batches_pickle(env, tmp_path):
    """The adapter, its items and batches pickle (spawn / forkserver workers); the unpickled adapter draws the same."""
    from b200asr import loader
    ds = env.dataset(tmp_path, [4000, 2000], prob=0.5)
    items = loader.PackedItems(ds, env.clip_set())
    again = pickle.loads(pickle.dumps(items))
    _seed(3)
    a = [items[i] for i in range(2)]
    _seed(3)
    b = [again[i] for i in range(2)]
    for x, y in zip(a, b):
        assert np.array_equal(x.wave, y.wave) and pickle.dumps(x[1:]) == pickle.dumps(y[1:])
    pb = pickle.loads(pickle.dumps(loader.collate_items(a)))
    assert torch.equal(pb.wave, loader.collate_items(a).wave)


def _oracle_inputs(pb, bank, window="hamming"):
    """_collate_fn's inputs restated in float64 from a PackedBatch's waveforms and noise draws."""
    specs = []
    for r in range(len(pb.lengths)):
        o, n = int(pb.offsets[r]), int(pb.lengths[r])
        y = pb.wave[o:o + n].numpy().astype(np.float64)
        s = int(pb.noise_start[r])
        if s >= 0:
            y = AO.mix(y, bank[s:s + n], float(pb.noise_level[r]))
        specs.append(AO.log_spectrogram(y, window_name=window, max_frames=pb.src_max_len))
    out = np.zeros((len(specs), 1, 161, int(pb.input_sizes[0])), np.float32)
    for r, s in enumerate(specs):
        out[r, 0, :, :s.shape[1]] = s
    return torch.from_numpy(out)


@pytest.mark.parametrize("prob", [None, 0.5])
def test_workers_draw_as_the_reference_workers(env, tmp_path, prob):
    """At num_workers=2 the installed loader's workers make the draws the unmodified loader's workers make: equal host
    tensors, and the reference's inputs within 1e-5 of the float64 restatement of the workers' waveforms and draws."""
    from b200asr import loader
    lengths = [4000, 4800, 3200, 6400, 1600, 2560, 5000, 3999, 4100]
    ds = env.dataset(tmp_path, lengths, prob=prob)
    items = loader.PackedItems(ds, env.clip_set() if prob is not None else None)
    bank = env.bank_np()
    for seed in (7, 8):
        _seed(seed), torch.manual_seed(seed)                  # BucketingSampler shuffles its bins in place: one each
        want = list(env.DL.AudioDataLoader(ds, num_workers=2, batch_sampler=env.DL.BucketingSampler(ds, batch_size=3)))
        _seed(seed), torch.manual_seed(seed)
        got = list(torch.utils.data.DataLoader(items, num_workers=2, batch_sampler=env.DL.BucketingSampler(ds, batch_size=3),
                                               collate_fn=loader.collate_items))
        assert len(got) == len(want) == 3
        for pb, w in zip(got, want):
            for a, b in zip((pb.targets, pb.input_percentages, pb.input_sizes, pb.target_sizes), w[1:]):
                assert torch.equal(a, b)
            o = _oracle_inputs(pb, bank)
            assert o.shape == w[0].shape and float((o - w[0]).abs().max()) <= 1e-5 * float(w[0].abs().max())
        if prob is not None:
            assert any(bool((pb.noise_start >= 0).any()) for pb in got)


def test_install_binds_and_restores_the_loader(env, tmp_path):
    import b200asr
    from b200asr import loader
    DL = env.DL
    init = DL.AudioDataLoader.__init__
    assert "__iter__" not in vars(DL.AudioDataLoader)
    ds = env.dataset(tmp_path, [4000, 2000, 3000], prob=None)
    before = DL.AudioDataLoader(ds, batch_size=2)
    b200asr.install()
    try:
        assert DL.AudioDataLoader.__init__ is loader.audio_loader_init and DL.AudioDataLoader.__iter__ is loader.audio_loader_iter
        assert b200asr.original(DL.AudioDataLoader, "__init__") is init
        sampler = DL.BucketingSampler(ds, batch_size=2)
        dl = DL.AudioDataLoader(ds, num_workers=0, batch_sampler=sampler)
        packed = dl._b200asr_packed
        assert dl.dataset is ds and dl.batch_sampler is sampler and len(dl) == len(sampler) == 2
        assert packed.inner.batch_sampler is sampler and packed.inner.pin_memory and packed.inner.collate_fn is loader.collate_items
        assert isinstance(packed.inner.dataset, loader.PackedItems) and packed.inner.dataset.dataset is ds
        assert not DL.AudioDataLoader(ds, batch_size=2, pin_memory=False)._b200asr_packed.inner.pin_memory
        assert before.__dict__.get("_b200asr_packed") is None            # built before install(): the reference's path
        spect, ids = ds[0]                                                # direct indexing is the reference's
        assert isinstance(spect, torch.Tensor) and spect.shape == (161, 26) and isinstance(ids, list)
    finally:
        b200asr.uninstall()
    assert DL.AudioDataLoader.__init__ is init and "__iter__" not in vars(DL.AudioDataLoader)


def test_noise_dir_without_clips_runs_the_reference_loader(env, tmp_path):
    """A noise_dir with no audio: the reference fails only on a draw that adds noise, so at noise_prob 0 its loader
    works; the installed loader then runs the reference's path and yields its batches."""
    import b200asr
    DL = env.DL
    env.clips = {}
    ds = env.dataset(tmp_path, [4000, 2000, 3000, 2500], prob=0.0)
    assert ds.noiseInjector.paths == []
    _seed(4)
    want = list(DL.AudioDataLoader(ds, batch_size=2))
    b200asr.install()
    try:
        dl = DL.AudioDataLoader(ds, batch_size=2)
        _seed(4)
        got = list(dl)
        assert dl._b200asr_packed.reference and _same_batches(got, want)
    finally:
        b200asr.uninstall()


class _Pairs(torch.utils.data.Dataset):
    def __len__(self):
        return 4

    def __getitem__(self, i):
        return torch.full((161, 3 + i), float(i)), [1, 3 + i, 2]


def _same_batches(a, b):
    return len(a) == len(b) and all(all(torch.equal(x, y) for x, y in zip(p, q)) for p, q in zip(a, b))


def test_fallbacks_run_the_reference_loader(env, tmp_path):
    """Not a SpectrogramDataset, the caller's collate_fn, or a noise clip at another sample rate: the reference's own
    iterator, with the reference's batches."""
    import b200asr
    DL = env.DL
    ds = env.dataset(tmp_path, [4000, 2000, 3000, 2500], prob=0.5)
    env.rates[sorted(env.clips)[1]] = 8000                                # sox would resample this clip
    _seed(1)
    want = list(DL.AudioDataLoader(ds, batch_size=2))
    want_pairs = list(DL.AudioDataLoader(_Pairs(), batch_size=2))
    b200asr.install()
    try:
        pairs = DL.AudioDataLoader(_Pairs(), batch_size=2)
        assert pairs._b200asr_packed is None and _same_batches(list(pairs), want_pairs)
        own = DL.AudioDataLoader(ds, batch_size=2, collate_fn=DL._collate_fn)
        assert own._b200asr_packed is None
        _seed(1)
        assert _same_batches(list(own), want)
        other = DL.AudioDataLoader(ds, batch_size=2)
        assert other._b200asr_packed is not None
        _seed(1)
        got = list(other)
        assert other._b200asr_packed.reference and _same_batches(got, want)
    finally:
        b200asr.uninstall()
