"""The reference's AudioDataLoader (utils/data_loader.py:217-220) fed from the device feature front end.

After install(), an AudioDataLoader over a SpectrogramDataset yields `_collate_fn`'s 5-tuple `(inputs, targets,
input_percentages, input_sizes, target_sizes)` with `inputs` computed on the current CUDA device by one
`b200asr_stft_features_packed` call per batch, and the other four host tensors equal to `_collate_fn`'s.

Worker side (host, pickles): `PackedItems[i]` makes `SpectrogramDataset.__getitem__`'s calls in its order -- the manifest
draw, the reference's own `load_audio` / `load_randomly_augmented_audio`, the noise draws, `parse_transcript` -- but
returns the waveform and the draws instead of a spectrogram; `collate_items` sorts as `_collate_fn` does and packs the
waveforms back to back.  Main side: `audio_loader_init` / `audio_loader_iter` (bound onto AudioDataLoader by install())
read the noise clips once into a NoiseBank, then upload each batch without a host synchronisation and compute its
features.

SpecAugment is opt-in per dataset: a SpectrogramDataset with a `spec_augment` attribute (a features.SpecAugment) has it
applied to every batch after the features, on the device.  Building the loader restarts the policy's batch counter at
0; the counter then advances once per batch, across epochs.  A dataset without the attribute yields exactly what it
yields without this feature, and the reference's random draws are untouched either way.

Tempo and gain perturbation is opt-in per dataset too: a SpectrogramDataset with `augment=True` and a `tempo_gain`
attribute (a features.TempoGain) has its workers read the audio with the reference's `load_audio` and make
`load_randomly_augmented_audio`'s two draws with `TempoGain.draw_one`, instead of running sox; the noise draw and the
frame count use the stretched length, and each batch is stretched on the device (one `b200asr_tempo_gain` launch) before
its features.  An `augment=True` dataset without the attribute keeps the reference's sox path; the attribute on an
`augment=False` dataset is a ValueError when the loader is built.

Speed perturbation is opt-in per dataset as well, with or without `augment`: a SpectrogramDataset with a `speed_perturb`
attribute (a features.SpeedPerturb) has its workers draw each utterance's factor from np.random after the item's own
`--augment` draws and before its noise draws (an extra draw the reference does not make, so every later draw of that
worker shifts); the noise draw and the frame count use the resampled length, and each batch is resampled on the device
(one `b200asr_resample_packed` launch) after its tempo and gain and before its features.

Resampling noise clips on the device is opt-in per dataset: a noise clip at another sample rate than the dataset's
makes the installed loader run the reference's own loader (which resamples the segment it cuts with sox, in the worker,
per utterance), unless the SpectrogramDataset has `resample_noise = True`.  Then every such clip is resampled once, when
the clips are read, on the device (16-bit output, as sox's `-r sr -b 16` writes it), and the device path serves the
dataset; only a clip whose rate cannot be inferred from its duration and sample count, or whose ratio to the dataset's
rate the resampler does not take, still runs the reference's loader.
"""
from __future__ import annotations

import importlib
import inspect
import random
from math import gcd
from typing import NamedTuple

import numpy as np
import torch
from torch.utils.data import DataLoader, Dataset

from . import features


class Item(NamedTuple):
    """One utterance as a worker returns it: the waveform (fp32), the noise draw as (clip index, first sample in the
    bank, level) -- (-1, -1, NaN) without noise --, the transcript ids and the frame count after the src_max_len cut.
    With a dataset's tempo_gain: the tempo, the linear gain fp32(10^(gain_db / 20)) and the stretched length `out_length`
    that `wave` (the unstretched audio) becomes on the device; out_length -1 (the default) when nothing is stretched."""
    wave: np.ndarray
    noise_clip: int
    noise_start: int
    noise_level: float
    ids: list
    frames: int
    tempo: float = 1.0
    g: float = 1.0
    out_length: int = -1


# An Item of a dataset with speed_perturb: the Item's fields, then the ratio (up, down) of the factor drawn and the length
# `speed_length` the (stretched) waveform is resampled to on the device.
ResampledItem = NamedTuple("ResampledItem", list(Item.__annotations__.items()) + [("up", int), ("down", int),
                                                                                   ("speed_length", int)])


class PackedBatch(NamedTuple):
    """A batch as the workers collate it, sorted as `_collate_fn` sorts (frames, longest first, stable): the waveforms
    back to back (`wave`, at least one sample) at int64 `offsets` with int32 `lengths`; per utterance the noise clip,
    start (int64, -1 without noise) and level (fp32); `_collate_fn`'s four host tensors; the src_max_len of the cut.
    With a dataset's tempo_gain: per utterance the tempo (float64), linear gain (fp32) and stretched length (int32) the
    waveforms are stretched with before their features; None (the default) when nothing is stretched.  With a dataset's
    speed_perturb: per utterance the ratio (up, down, int32) and the resampled length (int32); None when nothing is
    resampled."""
    wave: torch.Tensor
    offsets: torch.Tensor
    lengths: torch.Tensor
    noise_clip: torch.Tensor
    noise_start: torch.Tensor
    noise_level: torch.Tensor
    targets: torch.Tensor
    input_percentages: torch.Tensor
    input_sizes: torch.Tensor
    target_sizes: torch.Tensor
    src_max_len: int
    tempo: torch.Tensor | None = None
    g: torch.Tensor | None = None
    out_lengths: torch.Tensor | None = None
    up: torch.Tensor | None = None
    down: torch.Tensor | None = None
    speed_lengths: torch.Tensor | None = None


def _data_loader():
    return importlib.import_module("utils.data_loader")


class PackedItems(Dataset):
    """The worker side of a SpectrogramDataset: waveforms and the reference's random draws, no spectrogram.  `clips` (a
    features.NoiseClips) is set by the loader before its workers start when the dataset injects noise."""

    def __init__(self, dataset, clips: features.NoiseClips | None = None):
        self.dataset = dataset
        self.clips = clips
        self.hop = int(dataset.sample_rate * dataset.window_stride)

    def __len__(self):
        return len(self.dataset)

    def __getitem__(self, index) -> Item:
        ds, DL = self.dataset, _data_loader()
        ids = ds.ids_list[random.randint(0, len(ds.ids_list) - 1)]            # __getitem__ (:127-130)
        audio_path, transcript_path = ids[index % len(ids)][:2]
        policy = getattr(ds, "tempo_gain", None) if ds.augment else None
        stretch = ()
        if policy is not None:                                                # the stretch is made on the device
            y = DL.load_audio(audio_path)
            tempo, gain_db = policy.draw_one(np.random)                      # load_randomly_augmented_audio's draws
        elif ds.augment:                                                      # parse_audio (:61-70)
            y = DL.load_randomly_augmented_audio(audio_path, ds.sample_rate)
        else:
            y = DL.load_audio(audio_path)
        y = np.ascontiguousarray(y, dtype=np.float32).reshape(-1)
        n = len(y)
        if policy is not None:
            n = policy.out_length(n, tempo)
            stretch = (tempo, float(policy.linear_gain(gain_db)), n)
        speed = getattr(ds, "speed_perturb", None)
        if speed is not None:                                                 # resampled on the device
            up, down = speed.ratio(speed.draw_one(np.random))
            n = features.resample_out_length(n, up, down)
            stretch = (stretch or tuple(Item._field_defaults.values())) + (up, down, n)     # no stretch: its defaults
        clip, start, level = -1, -1, float("nan")
        if ds.noiseInjector:
            if self.clips is None:
                raise RuntimeError("PackedItems: the dataset injects noise but no noise clips were given")
            _, clip, level, _, start = self.clips.draw_one(n, ds.noise_prob, ds.noiseInjector.noise_levels, np.random)
        transcript = ds.parse_transcript(transcript_path)
        src_max_len = importlib.import_module("utils.constant").args.src_max_len      # read at call time, as :131
        return (Item if speed is None else ResampledItem)(y, clip, start, level, transcript, min(1 + n // self.hop, src_max_len),
                                                           *stretch)


def collate_items(items) -> PackedBatch:
    """`_collate_fn` (:182-214) over Items, without the spectrograms: the same order and the same targets, percentages,
    sizes and target sizes (values and dtypes), the waveforms packed in that order."""
    order = sorted(range(len(items)), key=lambda i: items[i].frames, reverse=True)   # sorted(..., reverse=True) is stable
    items = [items[i] for i in order]
    B, t_max = len(items), items[0].frames
    lengths = np.array([len(it.wave) for it in items], dtype=np.int64)
    wave = np.concatenate([it.wave for it in items] + ([np.zeros(1, np.float32)] if lengths.sum() == 0 else []))
    max_tgt = max(len(it.ids) for it in items)
    targets = torch.zeros(B, max_tgt, dtype=torch.int64)
    for r, it in enumerate(items):
        targets[r, :len(it.ids)] = torch.tensor(list(it.ids), dtype=torch.int32)
    stretched = [it.out_length >= 0 for it in items]
    if any(stretched) and not all(stretched):
        raise ValueError("collate_items: a batch mixes stretched and unstretched utterances")
    resampled = [isinstance(it, ResampledItem) for it in items]
    if any(resampled) and not all(resampled):
        raise ValueError("collate_items: a batch mixes resampled and unresampled utterances")
    stretch = {}
    if all(stretched):
        stretch = dict(tempo=torch.tensor([it.tempo for it in items], dtype=torch.float64),
                       g=torch.tensor([it.g for it in items], dtype=torch.float32),
                       out_lengths=torch.tensor([it.out_length for it in items], dtype=torch.int32))
    if all(resampled):
        stretch.update(up=torch.tensor([it.up for it in items], dtype=torch.int32),
                       down=torch.tensor([it.down for it in items], dtype=torch.int32),
                       speed_lengths=torch.tensor([it.speed_length for it in items], dtype=torch.int32))
    return PackedBatch(
        wave=torch.from_numpy(wave),
        offsets=torch.from_numpy(np.concatenate([[0], np.cumsum(lengths)[:-1]]).astype(np.int64)),
        lengths=torch.from_numpy(lengths.astype(np.int32)),
        noise_clip=torch.tensor([it.noise_clip for it in items], dtype=torch.int64),
        noise_start=torch.tensor([it.noise_start for it in items], dtype=torch.int64),
        noise_level=torch.tensor([it.noise_level for it in items], dtype=torch.float32),
        targets=targets,
        input_percentages=torch.tensor([it.frames / float(t_max) for it in items], dtype=torch.float32),
        input_sizes=torch.tensor([it.frames for it in items], dtype=torch.int32),
        target_sizes=torch.tensor([len(it.ids) for it in items], dtype=torch.int32),
        src_max_len=int(importlib.import_module("utils.constant").args.src_max_len), **stretch)


def clip_rate(n: int, duration: float, sample_rate: int) -> int | None:
    """A noise clip's integer sample rate from its sample count `n` and its duration in seconds (get_audio_length):
    `sample_rate` when round(duration * sample_rate) == n, else r = round(n / duration) when round(duration * r) == n;
    None when neither holds (or the duration is not a positive finite number)."""
    if not np.isfinite(duration):
        return None
    if round(duration * sample_rate) == n:
        return int(sample_rate)
    if duration <= 0:
        return None
    r = int(round(n / duration))
    return r if r >= 1 and round(duration * r) == n else None


def _window_name(ds, DL) -> str:
    """The audio_conf['window'] name SpectrogramParser resolved (:52): the key of DL.windows holding ds.window."""
    return next((k for k, v in DL.windows.items() if v is ds.window), "hamming")


class PackedLoader:
    """What an installed AudioDataLoader keeps: a DataLoader over PackedItems with collate_items (the caller's sampler,
    batch sampler, workers and other arguments), the noise bank once read, and the per-batch device step."""

    def __init__(self, outer, arguments: dict):
        ds = outer.dataset
        self.items = PackedItems(ds)
        kwargs = dict(arguments, dataset=self.items, collate_fn=collate_items)
        kwargs.setdefault("pin_memory", True)
        self.inner = DataLoader(**kwargs)
        self.bank = None
        self.reference = False                  # set when the noise clips need the reference's own path (prepare)
        augment = getattr(ds, "spec_augment", None)
        if augment is not None:
            augment.counter = 0

    def prepare(self) -> bool:
        """Read the noise clips into a NoiseBank on the current device, once, before any worker starts.  False when the
        reference's loader has to run: noise_dir holds no clips (the reference then fails only on a draw that adds
        noise, never at noise_prob 0), or a clip's duration (get_audio_length) does not give its sample count at the
        dataset's sample rate, so that sox would resample it -- unless the dataset has `resample_noise = True`: then a clip
        at another rate (clip_rate) is resampled to the dataset's rate on the device, and only a clip whose rate cannot
        be inferred, or whose ratio to the dataset's rate is beyond the resampler's, runs the reference's loader."""
        ds = self.items.dataset
        if self.reference or not ds.noiseInjector:
            return not self.reference
        if self.bank is None:
            if not ds.noiseInjector.paths:              # no clips: the reference fails only on a draw that adds noise
                self.reference = True
                return False
            DL, sr = _data_loader(), ds.sample_rate
            resample = getattr(ds, "resample_noise", False)
            clips, rates = [], []
            for path in ds.noiseInjector.paths:
                y = np.asarray(DL.load_audio(path), dtype=np.float32).reshape(-1)
                r = clip_rate(len(y), DL.get_audio_length(path), sr)
                if r is None or (r != sr and not resample) or max(sr, r) // gcd(int(sr), r) > features.RESAMPLE_MAX_RATE:
                    self.reference = True
                    return False
                clips.append(y)
                rates.append(r)
            self.bank = features.NoiseBank(clips, sr, rates=rates)
            self.items.clips = self.bank.clips
        device = torch.device("cuda", torch.cuda.current_device())
        if self.bank.bank.device != device:
            self.bank.bank = self.bank.bank.to(device)
        return True

    def batch(self, pb: PackedBatch):
        """`_collate_fn`'s 5-tuple of one PackedBatch: the uploads and one feature call on the current stream."""
        ds = self.items.dataset
        device = torch.device("cuda", torch.cuda.current_device())
        up = lambda t: t.to(device, non_blocking=True)          # noqa: E731
        sr = ds.sample_rate
        wave, offsets, lengths_d = up(pb.wave), up(pb.offsets), up(pb.lengths)
        lengths = pb.lengths.numpy()
        offsets_h = pb.offsets.numpy()
        if pb.out_lengths is not None:                          # the stretched waveforms replace the read ones
            wave, offsets, lengths_d, _, _ = features._tempo_gain(wave, offsets, lengths_d, pb.tempo, pb.g, pb.out_lengths, sr)
            lengths = pb.out_lengths.numpy()
            offsets_h = np.concatenate([[0], np.cumsum(lengths, dtype=np.int64)[:-1]])
        if pb.speed_lengths is not None:                        # then the resampled ones replace those
            wave, offsets_h, lengths = features._resample(wave, offsets_h, lengths, pb.up.numpy(), pb.down.numpy(), False)
            offsets, lengths_d = features._pinned_to(offsets_h, device), features._pinned_to(lengths.astype(np.int32), device)
        noise = None
        if self.bank is not None:
            noise = self.bank.device_args(pb.noise_clip.numpy(), pb.noise_start, pb.noise_level, lengths, device)
        inputs, _ = features.stft_features_packed(
            wave, offsets, lengths_d, max(1, int(lengths.max())), int(pb.input_sizes[0]), sr,
            ds.window_size, ds.window_stride, normalize=ds.normalize, window=_window_name(ds, _data_loader()), noise=noise,
            max_frames=pb.src_max_len)
        augment = getattr(ds, "spec_augment", None)
        if augment is not None:
            inputs, _ = augment.apply(inputs, pb.input_sizes)
        return inputs, pb.targets, pb.input_percentages, pb.input_sizes, pb.target_sizes


class _Batches:
    """Iterator over an installed loader's batches; the DataLoader iterator underneath is made at once, as iter() of the
    reference's loader makes it (its workers' base seed is drawn then)."""

    def __init__(self, packed: PackedLoader):
        self.packed = packed
        self.it = iter(packed.inner)

    def __iter__(self):
        return self

    def __len__(self):
        return len(self.it)

    def __next__(self):
        return self.packed.batch(next(self.it))


def _check_tempo_gain(ds):
    if getattr(ds, "tempo_gain", None) is not None and not getattr(ds, "augment", False):
        raise ValueError("the dataset carries tempo_gain but was built with augment=False: the reference would not "
                         "perturb its tempo and gain")


def audio_loader_init(self, *args, **kwargs):
    """AudioDataLoader.__init__ after install(): the reference's own construction (so `dataset`, `sampler`, `len()` are
    its), plus a PackedLoader unless the dataset is not a SpectrogramDataset or the caller passed a collate_fn."""
    from .install import original
    original(type(self), "__init__")(self, *args, **kwargs)
    arguments = inspect.signature(DataLoader.__init__).bind(self, *args, **kwargs).arguments
    arguments.pop("self")
    _check_tempo_gain(self.dataset)
    eligible = isinstance(self.dataset, _data_loader().SpectrogramDataset) and arguments.get("collate_fn") is None
    self._b200asr_packed = PackedLoader(self, dict(arguments)) if eligible else None


def audio_loader_iter(self):
    """AudioDataLoader.__iter__ after install(): device batches from the PackedLoader, or the reference's iterator
    (original(AudioDataLoader, "__iter__")) for a loader without one, without noise clips or with a clip at another rate
    that the dataset does not resample on the device (PackedLoader.prepare)."""
    packed = self.__dict__.get("_b200asr_packed")
    if packed is None or not packed.prepare():
        for attr in ("spec_augment", "tempo_gain", "speed_perturb"):     # the reference's iterator would drop it silently
            if getattr(self.dataset, attr, None) is not None:
                raise RuntimeError(f"the dataset carries {attr}, which only the device front end applies; this loader "
                                   "runs the reference's own iterator (a collate_fn was given, or a noise clip is at "
                                   "another sample rate: set the dataset's resample_noise = True to resample it on the "
                                   "device)")
        from .install import original
        return original(type(self), "__iter__")(self)
    return _Batches(packed)
