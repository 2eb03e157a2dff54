"""GPU feature front end: waveforms -> the batches of the reference's loader.

Mirrors `SpectrogramParser.parse_audio` (utils/data_loader.py:60-91), `SpectrogramDataset.__getitem__` (:126-133) and
`_collate_fn` (:182-214): optional noise injection (`NoiseInjection`, :147-179), STFT (n_fft = sample_rate * window_size,
hop = sample_rate * window_stride, the symmetric window -- the reference passes the callable scipy.signal.<window>, which
librosa evaluates as window(n_fft), i.e. sym=True --, centred frames), magnitude, log1p, per-utterance mean /
unbiased-std normalisation, the src_max_len cut, zero padding to the longest utterance.  One C-ABI call
(`b200asr_stft_features_ex`, or `b200asr_stft_features_packed` over utterances packed back to back): the STFT of the
whole batch is a single 3xTF32 tensor-core GEMM over overlapping frame rows.

`spectrogram_batch` returns the device triple `(inputs, input_percentages, input_sizes)`; `collate_waves` returns
`_collate_fn`'s 5-tuple, sorted, with everything but `inputs` on the host.  `NoiseClips` holds the noise clips' lengths
and makes the reference's random draws (host data: DataLoader workers draw with it); `NoiseBank` adds the clips on the
device.  `SpecAugment` is an opt-in augmentation policy both helpers (and loader.py) apply to their output on the device;
`TempoGain` (with `tempo_gain`) is the reference's tempo and gain perturbation, which collate_waves (and loader.py) apply to
the waveforms before the features.  `SpeedPerturb` (with `resample`, a polyphase resampler restating
scipy.signal.resample_poly) is speed perturbation, applied after the tempo and gain; `NoiseBank` resamples noise clips
at other rates with the same kernel (loader.py does so for a dataset with `resample_noise = True`).  loader.py feeds the reference's AudioDataLoader from here.
"""
from __future__ import annotations

from dataclasses import dataclass
from fractions import Fraction
from math import gcd
from typing import Sequence

import numpy as np
import torch

from . import _lib as L
from . import ops


# utils/data_loader.py:20-21; any other name falls back to Hamming (:52)
WINDOWS = {"hamming": 0, "hann": 1, "blackman": 2, "bartlett": 3}
NO_CUT = 2 ** 31 - 1


def _pinned_to(a: np.ndarray, device) -> torch.Tensor:
    """Host array -> device tensor without a host synchronisation (a pinned staging copy, then an async upload)."""
    return torch.from_numpy(np.ascontiguousarray(a)).pin_memory().to(device, non_blocking=True)


@dataclass
class NoiseDraws:
    """The reference's noise draws for a batch, per utterance in batch order: `add` (binomial outcome), `clip` (index into
    the bank's clips, -1 without noise), `level` (uniform), `rand` (the segment position draw), `start` (first sample of
    the segment in the bank, -1 without noise)."""
    bank: "NoiseBank"
    add: np.ndarray
    clip: np.ndarray
    level: np.ndarray
    rand: np.ndarray
    start: np.ndarray

    def take(self, order) -> "NoiseDraws":
        order = np.asarray(order, dtype=np.int64)
        return NoiseDraws(self.bank, self.add[order], self.clip[order], self.level[order], self.rand[order], self.start[order])


class NoiseClips:
    """Where the noise clips of `NoiseInjection` (utils/data_loader.py:147-179) lie in a `NoiseBank`: their lengths in
    samples, their offsets when back to back, and their sample rate; and each clip's own duration in seconds, which the
    draws use as the reference uses get_audio_length (lengths / sample_rate unless a clip was resampled).  Host data that
    pickles, so DataLoader workers make the reference's draws with it (loader.py) while the samples stay on the device."""

    def __init__(self, lengths, sample_rate: int, durations=None):
        self.lengths = np.asarray(lengths, dtype=np.int64).reshape(-1)
        if len(self.lengths) == 0:
            raise ValueError("NoiseBank needs at least one clip")
        self.offsets = np.concatenate([[0], np.cumsum(self.lengths)[:-1]]).astype(np.int64)
        self.sample_rate = int(sample_rate)
        self.durations = self.lengths / self.sample_rate if durations is None else \
            np.asarray(durations, dtype=np.float64).reshape(-1)
        if len(self.durations) != len(self.lengths):
            raise ValueError(f"{len(self.durations)} durations for {len(self.lengths)} clips")

    def __len__(self):
        return len(self.lengths)

    def draw_one(self, n: int, noise_prob: float, noise_levels, rng=np.random):
        """The reference's draws for one utterance of `n` samples, with its numpy calls in its order (data_loader.py:68-69,
        164-165, 171): binomial(1, noise_prob), and only for a 1: choice over the clips, uniform(*noise_levels), rand().
        `rng` is np.random (the reference's global state) or a RandomState.  Returns (add, clip, level, rand, start): clip
        -1, level and rand NaN, start -1 without noise.

        The segment start is noise_start = rand * (duration - n / sr) seconds, in float64 as :169-172.  The reference
        then cuts the segment with sox `trim` (utils/audio.py:21-32); that cut is not pinned here but restated as the
        sample round(noise_start * sr), clamped so that the n samples fit in the clip; `start` is that sample's index in
        the bank.  A clip shorter than the utterance, where the reference fails its assert (:175), raises ValueError."""
        n = int(n)
        if not rng.binomial(1, noise_prob):
            return 0, -1, float("nan"), float("nan"), -1
        c = int(rng.choice(len(self)))                # np.random.choice(paths): one randint(0, len(paths)) draw
        level = rng.uniform(*noise_levels)
        rand = rng.rand()
        clip_len = int(self.lengths[c])
        if clip_len < n:
            raise ValueError(f"noise clip {c} has {clip_len} samples, fewer than an utterance's {n}")
        noise_start = rand * (float(self.durations[c]) - n / self.sample_rate)
        return 1, c, level, rand, int(self.offsets[c]) + min(max(round(noise_start * self.sample_rate), 0), clip_len - n)

    def check(self, clip, start, lengths):
        """ValueError unless every segment with start >= 0 lies inside its clip."""
        clip, start, lengths = (np.asarray(a, dtype=np.int64) for a in (clip, start, lengths))
        if not (len(clip) == len(start) == len(lengths)):
            raise ValueError(f"{len(start)} noise draws for {len(lengths)} utterances")
        noisy = start >= 0
        c = clip[noisy]
        if ((c < 0) | (c >= len(self))).any() or (start[noisy] < self.offsets[c]).any() or \
                (start[noisy] + lengths[noisy] > self.offsets[c] + self.lengths[c]).any():
            raise ValueError("a noise segment does not lie inside its clip")


class NoiseBank:
    """Noise clips for `NoiseInjection` (utils/data_loader.py:147-179), back to back in one device buffer.

    `clips` are 1-D fp32 waveforms, in the order `librosa.util.find_files(noise_dir)` lists them (sorted paths): `draw`
    picks clips by index, so that order is what makes its choices the reference's.  `rates` gives each clip's integer
    sample rate (None: all at `sample_rate`).  Clips at another rate are resampled to `sample_rate` on the device, all in
    one `resample` launch with quantize16 -- the reference's `sox ... -r sr -b 16` -- and keep their own duration
    (samples / rate) for the draws; ValueError for a rate whose ratio to `sample_rate` exceeds RESAMPLE_MAX_RATE in
    lowest terms.  `clips` (a NoiseClips) is the host side the draws need."""

    def __init__(self, clips, sample_rate: int, device=None, rates=None):
        arrays = [np.asarray(c.detach().cpu() if isinstance(c, torch.Tensor) else c, dtype=np.float32).reshape(-1) for c in clips]
        sr = int(sample_rate)
        rates = [sr] * len(arrays) if rates is None else [int(r) for r in rates]
        if len(rates) != len(arrays) or min(rates, default=1) < 1:
            raise ValueError(f"NoiseBank: rates {rates!r} for {len(arrays)} clips")
        other = [i for i, r in enumerate(rates) if r != sr]
        ratios = {i: resample_ratio(sr, rates[i]) for i in other}
        lengths = [resample_out_length(len(a), *ratios[i]) if i in ratios else len(a) for i, a in enumerate(arrays)]
        self.clips = NoiseClips(lengths, sr, [len(a) / r for a, r in zip(arrays, rates)])
        device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        host = np.zeros(sum(lengths), np.float32)
        for i, a in enumerate(arrays):
            if i not in ratios:
                host[self.clips.offsets[i]:self.clips.offsets[i] + len(a)] = a
        self.bank = torch.from_numpy(host).to(device)
        if any(lengths[i] for i in other):         # written in place into their slots of the bank
            src = [arrays[i] for i in other]
            src_off = np.concatenate([[0], np.cumsum([len(a) for a in src])[:-1]]).astype(np.int64)
            _resample(torch.from_numpy(np.concatenate(src + [np.zeros(1, np.float32)])).to(device), src_off,
                      [len(a) for a in src], [ratios[i][0] for i in other], [ratios[i][1] for i in other], True,
                      out=self.bank, out_offsets=self.clips.offsets[other])

    sample_rate = property(lambda self: self.clips.sample_rate)
    lengths = property(lambda self: self.clips.lengths)
    offsets = property(lambda self: self.clips.offsets)

    def __len__(self):
        return len(self.clips)

    def draw(self, lengths, noise_prob: float, noise_levels, rng=np.random) -> NoiseDraws:
        """NoiseClips.draw_one for utterances of `lengths` samples, in batch order."""
        return self._draws([self.clips.draw_one(n, noise_prob, noise_levels, rng) for n in lengths])

    def _draws(self, rows) -> NoiseDraws:
        """NoiseDraws from NoiseClips.draw_one's rows, in batch order."""
        add, clip, level, rand, start = (np.array(col, dtype=dt).reshape(-1) for col, dt in
                                         zip(zip(*rows) if rows else ((),) * 5,
                                             (np.int64, np.int64, np.float64, np.float64, np.int64)))
        return NoiseDraws(self, add, clip, level, rand, start)

    def device_args(self, clip, start, level, lengths, device):
        """(bank, bank_len, start, level) for the feature calls, or None when no utterance takes noise.  clip, start and
        lengths are host arrays (NoiseClips.check's); start and level are uploaded without a host synchronisation (pinned
        CPU tensors, e.g. from a DataLoader's pin-memory thread, go as they are)."""
        start_np = start.numpy() if isinstance(start, torch.Tensor) else np.asarray(start)
        self.clips.check(clip, start_np, lengths)
        if not (start_np >= 0).any():
            return None
        if self.bank.device != torch.device(device):
            raise ValueError(f"the noise bank is on {self.bank.device}, the batch on {device}")
        up = lambda a, dt: a.to(device, non_blocking=True) if isinstance(a, torch.Tensor) else _pinned_to(np.asarray(a, dt), device)  # noqa: E731
        return self.bank, self.bank.numel(), up(start, np.int64), up(level, np.float32)

    def _device_args(self, draws: NoiseDraws, lengths, device):
        """(bank, bank_len, start, level) for b200asr_stft_features_ex, or None when no utterance takes noise."""
        if draws.bank is not self:
            raise ValueError("the draws were made by another NoiseBank")
        return self.device_args(draws.clip, draws.start, draws.level, lengths, device)


class SpecAugment:
    """SpecAugment (Park et al. 2019) for the device front end's batches: a time warp of parameter `W` frames,
    `n_freq_masks` frequency masks of up to `Fp` bins and `n_time_masks` time masks of up to min(`Tp`, floor(`p` * T_b))
    frames, applied in that order by one `b200asr_spec_augment` launch per batch (include/b200asr.h states the draws and
    the fp32 formulas).  Masked bins and frames become 0, the utterance mean of normalised features.

    The paper's policies for LibriSpeech are LB (W=80, Fp=27, n_freq_masks=1, Tp=100, p=1.0, n_time_masks=1) and LD (the
    same with two masks of each kind); its Switchboard ones are SM (W=40, Fp=15, 2, Tp=70, p=0.2, 2) and SS (W=40, Fp=27, 2,
    Tp=70, p=0.2, 2).  They were tuned on 80 mel bins every 10 ms; the reference's features are n_fft/2 + 1 = 161
    linear bins at the same frame rate, so Fp is worth scaling.  Nothing here has a default.

    The draws come from the counter-based generator of dropout keyed by (`seed`, batch counter, utterance, slot): no host
    draw, no host synchronisation, nothing taken from numpy's, `random`'s or torch's generators.  `counter` counts the
    batches `apply` has augmented; the same (seed, counter) gives the same augmentation on any device and any rank.  A
    SpecAugment holds plain numbers, so it pickles (DataLoader workers receive it with the dataset it is attached to)."""

    MAX_MASKS = 64

    def __init__(self, W: int, Fp: int, n_freq_masks: int, Tp: int, p: float, n_time_masks: int, seed: int):
        ints = dict(W=W, Fp=Fp, n_freq_masks=n_freq_masks, Tp=Tp, n_time_masks=n_time_masks)
        for name, v in ints.items():
            if isinstance(v, bool) or not isinstance(v, (int, np.integer)) or v < 0 or v > 2 ** 31 - 1:
                raise ValueError(f"SpecAugment: {name}={v!r} must be an integer in [0, 2^31 - 1]")
        for name in ("n_freq_masks", "n_time_masks"):
            if ints[name] > self.MAX_MASKS:
                raise ValueError(f"SpecAugment: {name}={ints[name]} exceeds {self.MAX_MASKS}")
        if isinstance(p, bool) or not isinstance(p, (int, float, np.floating, np.integer)) or not 0.0 <= float(np.float32(p)) <= 1.0:
            raise ValueError(f"SpecAugment: p={p!r} must lie in [0, 1]")
        if isinstance(seed, bool) or not isinstance(seed, (int, np.integer)) or not 0 <= seed < 2 ** 64:
            raise ValueError(f"SpecAugment: seed={seed!r} must be an integer in [0, 2^64)")
        self.W, self.Fp, self.n_freq_masks, self.Tp, self.n_time_masks = (int(ints[k]) for k in ints)
        self.p = float(p)
        self.seed = int(seed)
        self.counter = 0

    def __repr__(self):
        return (f"SpecAugment(W={self.W}, Fp={self.Fp}, n_freq_masks={self.n_freq_masks}, Tp={self.Tp}, p={self.p}, "
                f"n_time_masks={self.n_time_masks}, seed={self.seed})")

    @property
    def draws_per_utterance(self) -> int:
        """c, w, then (f, f0) per frequency mask and (t, t0) per time mask."""
        return 2 + 2 * self.n_freq_masks + 2 * self.n_time_masks

    def apply(self, inputs: torch.Tensor, input_sizes: torch.Tensor):
        """Augment `inputs` [B,1,F,T] (CUDA fp32, the front end's layout) whose utterance b has `input_sizes[b]` frames
        (int, on the host or the device; a host tensor is uploaded without a host synchronisation) with batch counter
        `self.counter`, which then advances by one.  Returns (augmented [B,1,F,T], draws [B, draws_per_utterance]
        int32), both new device tensors; `inputs` is left as it is."""
        ops._need_cuda(inputs)
        if inputs.dim() != 4 or inputs.shape[1] != 1:
            raise ValueError(f"SpecAugment.apply: inputs of shape {tuple(inputs.shape)}, not [B, 1, F, T]")
        B, _, F, T = inputs.shape
        if self.Fp > F:
            raise ValueError(f"SpecAugment: Fp={self.Fp} exceeds the {F} frequency bins")
        if input_sizes.numel() != B:
            raise ValueError(f"SpecAugment.apply: {input_sizes.numel()} sizes for {B} utterances")
        x = ops._f32c(inputs)
        if input_sizes.is_cuda:
            frames = input_sizes.to(device=x.device, dtype=torch.int32).contiguous()
        else:
            frames = _pinned_to(input_sizes.numpy().astype(np.int32), x.device)
        out = torch.empty_like(x)
        draws = torch.empty((B, self.draws_per_utterance), device=x.device, dtype=torch.int32)
        counter, self.counter = self.counter, self.counter + 1
        L.check(ops._lib().b200asr_spec_augment(L.ptr(x), L.ptr(out), L.ptr(draws), L.ptr(frames), B, F, T, self.W, self.Fp,
                                                self.n_freq_masks, self.Tp, self.p, self.n_time_masks, self.seed,
                                                int(counter) & (2 ** 64 - 1), ops._stream()), "spec_augment")
        return out, draws


class TempoGain:
    """The reference's `--augment` (`load_randomly_augmented_audio`, utils/audio.py:50-61) on the device: per utterance a
    tempo uniform in `tempo_range` and a gain uniform in `gain_range` dB, applied by `tempo_gain` (WSOLA modelled on sox's
    `tempo` effect, then `gain` and a 16-bit output; include/b200asr.h states the algorithm).  The defaults are the
    reference's ranges.  Parity with sox itself is not pinned: the restated algorithm is the contract.

    A TempoGain holds plain numbers, so it pickles (DataLoader workers receive it with the dataset it is attached to)."""

    TEMPO_LIMITS = (0.25, 4.0)

    def __init__(self, tempo_range=(0.85, 1.15), gain_range=(-6, 8)):
        self.tempo_range = self._range("tempo_range", tempo_range)
        self.gain_range = self._range("gain_range", gain_range)
        lo, hi = self.TEMPO_LIMITS
        if not (lo <= self.tempo_range[0] and self.tempo_range[1] <= hi):
            raise ValueError(f"TempoGain: tempo_range={tempo_range!r} must lie in [{lo}, {hi}]")

    @staticmethod
    def _range(name, r):
        try:
            a, b = r
        except (TypeError, ValueError):
            raise ValueError(f"TempoGain: {name}={r!r} is not a (low, high) pair") from None
        for v in (a, b):
            if isinstance(v, bool) or not isinstance(v, (int, float, np.integer, np.floating)) or not np.isfinite(v):
                raise ValueError(f"TempoGain: {name}={r!r} needs two finite numbers")
        if a > b:
            raise ValueError(f"TempoGain: {name}={r!r} has low > high")
        return float(a), float(b)

    def __repr__(self):
        return f"TempoGain(tempo_range={self.tempo_range}, gain_range={self.gain_range})"

    def draw_one(self, rng=np.random):
        """load_randomly_augmented_audio's draws for one utterance, with its numpy calls in its order: uniform over the
        tempo range, then over the gain range; each rounded as the sox command line writes it ("{:.3f}").  `rng` is
        np.random (the reference's global state) or a RandomState.  Returns (tempo, gain_db)."""
        tempo = rng.uniform(low=self.tempo_range[0], high=self.tempo_range[1])
        gain = rng.uniform(low=self.gain_range[0], high=self.gain_range[1])
        return float(f"{tempo:.3f}"), float(f"{gain:.3f}")

    @staticmethod
    def geometry(sample_rate) -> tuple[int, int, int]:
        """(segment, search, overlap) in samples of sox's default tempo profile at `sample_rate`, in float64: (1312, 235,
        192) at 16 kHz.  ValueError for a rate too low to give a valid geometry."""
        sr = float(sample_rate)
        segment = int(np.floor(sr * 82 / 1000 + 0.5))
        search = int(np.floor(sr * (82 / 5.587) / 1000 + 0.5))
        overlap = int(np.floor(max(sr * (82 / 6.833) / 1000 + 4.5, 16)))
        overlap -= overlap % 8
        if 2 * overlap > segment:
            overlap -= 8
        if not (np.isfinite(sr) and search >= 1 and overlap >= 8 and 2 * overlap <= segment):
            raise ValueError(f"TempoGain: sample_rate={sample_rate!r} gives no valid geometry ({segment}, {search}, {overlap})")
        return segment, search, overlap

    @staticmethod
    def out_length(n: int, tempo: float) -> int:
        """Samples of the output for `n` input samples: floor(n / tempo + 0.5) in float64."""
        return int(np.floor(int(n) / float(tempo) + 0.5))

    @staticmethod
    def linear_gain(gain_db: float) -> np.float32:
        """fp32(10^(gain_db / 20)), computed in float64."""
        return np.float32(10.0 ** (float(gain_db) / 20.0))


def _tempo_gain(wave, offsets, lengths, tempo, g, out_lengths, sample_rate, picks=False):
    """One b200asr_tempo_gain launch.  wave, offsets, lengths on the device; tempo (float64), g (fp32) and out_lengths
    (int) host arrays, or pinned CPU tensors; the outputs back to back in batch order."""
    segment, search, overlap = TempoGain.geometry(sample_rate)
    device = wave.device
    up = lambda a, dt: a.to(device, non_blocking=True) if isinstance(a, torch.Tensor) else _pinned_to(np.asarray(a, dt), device)  # noqa: E731
    out_np = np.asarray(out_lengths.numpy() if isinstance(out_lengths, torch.Tensor) else out_lengths, dtype=np.int64).reshape(-1)
    B = len(out_np)
    out_offsets = np.concatenate([[0], np.cumsum(out_np)[:-1]]).astype(np.int64)
    out = torch.empty(max(1, int(out_np.sum())), device=device, dtype=torch.float32)
    out_off_d, out_len_d = _pinned_to(out_offsets, device), up(out_lengths, np.int32)
    pk = pk_off = pk_off_d = None
    if picks:
        K = -(-out_np // (segment - overlap))
        pk_off = np.concatenate([[0], np.cumsum(K)[:-1]]).astype(np.int64)
        pk = torch.empty(max(1, int(K.sum())), device=device, dtype=torch.int32)
        pk_off_d = _pinned_to(pk_off, device)
    tempo_d, g_d = up(tempo, np.float64), up(g, np.float32)      # held until the launch: a freed block would be reused
    L.check(ops._lib().b200asr_tempo_gain(
        L.ptr(wave), L.ptr(offsets), L.ptr(lengths), L.ptr(tempo_d), L.ptr(g_d), L.ptr(out), L.ptr(out_off_d),
        L.ptr(out_len_d), L.ptr(pk), L.ptr(pk_off_d), B, segment, search, overlap, ops._stream()), "tempo_gain")
    return out, out_off_d, out_len_d, pk, pk_off


def tempo_gain(wave: torch.Tensor, offsets, lengths, tempo, gain_db, sample_rate: int, picks: bool = False):
    """Tempo and gain perturbation of a packed batch (`TempoGain`'s algorithm, include/b200asr.h): utterance b is the
    lengths[b] samples of the 1-D CUDA fp32 `wave` from offsets[b] on (int64; a CUDA tensor, or host data uploaded).
    `lengths` (int32), `tempo` and `gain_db` (one per utterance) are host data: the output lengths are computed from them
    on the host, so there is no host synchronisation; they are uploaded through pinned memory.  One launch.

    Per utterance: out_length = floor(n / tempo + 0.5) samples of WSOLA at sox's default geometry for `sample_rate`
    (TempoGain.geometry), scaled by fp32(10^(gain_db / 20)) and quantised to 16 bits (clamp(rint(32768 v), -32768,
    32767) / 32768, so gains above 0 dB clip loud utterances).  Segment k starts at input sample floor(tempo * k * step +
    0.5) plus its pick p_k, the smallest offset in [0, search) minimising the float64 sum of squared differences to the
    overlap that follows the previous segment (p_0 = search // 2); segments crossfade linearly over `overlap` samples.

    Returns (out, out_offsets, out_lengths): the outputs back to back in batch order (a 1-D CUDA fp32 tensor, at least
    one element), their int64 offsets and int32 lengths on the device.  With picks=True also (picks, pick_offsets): every
    utterance's ceil(out_length / step) picks (int32, device) from its host int64 offset on."""
    ops._need_cuda(wave)
    if isinstance(lengths, torch.Tensor) and lengths.is_cuda:
        raise ValueError("tempo_gain: lengths must be host data (the output lengths are computed on the host)")
    lens = np.asarray(lengths.numpy() if isinstance(lengths, torch.Tensor) else lengths, dtype=np.int64).reshape(-1)
    tempo = np.asarray(tempo, dtype=np.float64).reshape(-1)
    gain_db = np.asarray(gain_db, dtype=np.float64).reshape(-1)
    B = len(lens)
    if not B or len(tempo) != B or len(gain_db) != B:
        raise ValueError(f"tempo_gain: {B} lengths, {len(tempo)} tempos and {len(gain_db)} gains")
    if not (np.isfinite(tempo).all() and (tempo > 0).all()):
        raise ValueError("tempo_gain: every tempo must be finite and positive")
    device = wave.device
    offs = offsets.to(device, torch.int64, non_blocking=True) if isinstance(offsets, torch.Tensor) else \
        _pinned_to(np.asarray(offsets, np.int64), device)
    if offs.numel() != B:
        raise ValueError(f"tempo_gain: {offs.numel()} offsets for {B} utterances")
    out_lengths = np.array([TempoGain.out_length(n, t) for n, t in zip(lens, tempo)], dtype=np.int32)
    g = np.array([TempoGain.linear_gain(d) for d in gain_db], dtype=np.float32)
    out, out_off, out_len, pk, pk_off = _tempo_gain(ops._f32c(wave), offs, _pinned_to(lens.astype(np.int32), device), tempo,
                                                    g, out_lengths, sample_rate, picks)
    return (out, out_off, out_len, pk, pk_off) if picks else (out, out_off, out_len)


RESAMPLE_MAX_RATE = 1000


def resample_ratio(up, down) -> tuple[int, int]:
    """(up, down) in lowest terms; ValueError unless both are integers >= 1 and the larger is at most RESAMPLE_MAX_RATE."""
    for v in (up, down):
        if isinstance(v, bool) or not isinstance(v, (int, np.integer)) or v < 1:
            raise ValueError(f"resample: up={up!r}, down={down!r} must be integers >= 1")
    g = gcd(int(up), int(down))
    up, down = int(up) // g, int(down) // g
    if max(up, down) > RESAMPLE_MAX_RATE:
        raise ValueError(f"resample: {up}/{down} exceeds {RESAMPLE_MAX_RATE} in lowest terms")
    return up, down


def resample_out_length(n: int, up: int, down: int) -> int:
    """ceil(n * up / down): resample_poly's output length for a reduced ratio."""
    return -(-int(n) * int(up) // int(down))


def resample_filter(up: int, down: int) -> np.ndarray:
    """resample_poly's default filter for a reduced ratio, in float64: firwin(2 half + 1, 1 / max(up, down),
    window=('kaiser', 5.0)) * up, half = 10 max(up, down), restated with numpy (np.i0 for the Bessel function, which can
    differ from scipy.special.i0 in the last bit)."""
    mr = max(up, down)
    numtaps, fc = 2 * 10 * mr + 1, 1.0 / mr
    m = np.arange(numtaps, dtype=np.float64) - 0.5 * (numtaps - 1)
    h = fc * np.sinc(fc * m)
    n = np.arange(numtaps, dtype=np.float64)
    alpha = (numtaps - 1) / 2.0
    h *= np.i0(5.0 * np.sqrt(1 - ((n - alpha) / alpha) ** 2.0)) / np.i0(np.float64(5.0))
    h /= np.sum(h)
    return h * up


def resample_taps(up: int, down: int) -> np.ndarray:
    """The kernel's taps for a reduced ratio (up / down != 1): resample_filter split per phase, [up, K] fp32 with
    taps[p, m] = h[p + m up] and zeros past the filter, K = ceil((2 half + 1) / up)."""
    h = resample_filter(up, down)
    K = -(-len(h) // up)
    return np.pad(h, (0, up * K - len(h))).reshape(K, up).T.astype(np.float32)


_TAPS: dict = {}            # (device, up, down) -> the ratio's taps on that device, uploaded once


def _device_taps(up: int, down: int, device) -> torch.Tensor:
    key = (str(device), up, down)
    if key not in _TAPS:
        _TAPS[key] = torch.from_numpy(np.ascontiguousarray(resample_taps(up, down))).to(device)
    return _TAPS[key]


_RESAMPLE_ITEM = np.dtype([("in_offset", "<i8"), ("out_offset", "<i8"), ("taps", "<u8"), ("in_length", "<i4"),
                           ("up", "<i4"), ("down", "<i4"), ("reserved", "<i4")])     # b200asr_resample_item


def _resample(wave, offsets, lengths, ups, downs, quantize16, out=None, out_offsets=None):
    """One b200asr_resample_packed launch.  wave on the device; offsets, lengths and the reduced ratios host data.  The
    outputs go back to back in batch order into a new buffer, or into `out` at the host `out_offsets`.  Returns (out,
    out_offsets, out_lengths), the last two int64 host arrays."""
    device = wave.device
    host = lambda a: np.asarray(a.numpy() if isinstance(a, torch.Tensor) else a, dtype=np.int64).reshape(-1)  # noqa: E731
    offsets, lengths, ups, downs = host(offsets), host(lengths), host(ups), host(downs)
    B = len(lengths)
    out_lengths = np.array([resample_out_length(n, u, d) for n, u, d in zip(lengths, ups, downs)], dtype=np.int64)
    if out is None:
        out_offsets = np.concatenate([[0], np.cumsum(out_lengths)[:-1]]).astype(np.int64)
        out = torch.empty(max(1, int(out_lengths.sum())), device=device, dtype=torch.float32)
    items = np.zeros(B, _RESAMPLE_ITEM)
    items["in_offset"], items["out_offset"], items["in_length"] = offsets, host(out_offsets), lengths
    items["up"], items["down"] = ups, downs
    items["taps"] = [0 if u == d == 1 else _device_taps(int(u), int(d), device).data_ptr() for u, d in zip(ups, downs)]
    items_d = _pinned_to(items.view(np.uint8), device)      # held until the launch: a freed block would be reused
    L.check(ops._lib().b200asr_resample_packed(L.ptr(wave), wave.numel(), L.ptr(out), out.numel(), items.ctypes.data,
                                               L.ptr(items_d), B, int(bool(quantize16)), ops._stream()), "resample_packed")
    return out, host(out_offsets), out_lengths


def resample(wave: torch.Tensor, offsets, lengths, up, down, quantize16: bool = False):
    """scipy.signal.resample_poly(x, up[b], down[b]) with its defaults for every utterance of a packed batch, in fp32 (the
    algorithm and the summation order: include/b200asr.h).  Utterance b is the lengths[b] samples of the 1-D CUDA fp32
    `wave` from offsets[b] on; offsets, lengths and the per-utterance `up` and `down` (reduced here; at most
    RESAMPLE_MAX_RATE in lowest terms) are host data, uploaded through pinned memory, so there is no host
    synchronisation.  A ratio of 1 copies.  quantize16=True rounds the outputs to the 16-bit grid as `sox -b 16` writes
    them (round to nearest, clamped, no dither).  One launch.

    Returns (out, out_offsets, out_lengths): the ceil(n up / down) outputs of every utterance back to back in batch order
    (a 1-D CUDA fp32 tensor, at least one element), their int64 offsets and int32 lengths on the device."""
    ops._need_cuda(wave)
    for name, a in (("offsets", offsets), ("lengths", lengths)):
        if isinstance(a, torch.Tensor) and a.is_cuda:
            raise ValueError(f"resample: {name} must be host data (the launch is checked on the host)")
    lens = np.asarray(lengths.numpy() if isinstance(lengths, torch.Tensor) else lengths, dtype=np.int64).reshape(-1)
    offs = np.asarray(offsets.numpy() if isinstance(offsets, torch.Tensor) else offsets, dtype=np.int64).reshape(-1)
    up, down = np.asarray(up).reshape(-1), np.asarray(down).reshape(-1)
    B = len(lens)
    if not B or len(offs) != B or len(up) != B or len(down) != B:
        raise ValueError(f"resample: {B} lengths, {len(offs)} offsets, {len(up)} ups and {len(down)} downs")
    ratios = [resample_ratio(u.item(), d.item()) for u, d in zip(up, down)]
    out, out_off, out_len = _resample(ops._f32c(wave), offs, lens, [r[0] for r in ratios], [r[1] for r in ratios], quantize16)
    device = wave.device
    return out, _pinned_to(out_off, device), _pinned_to(out_len.astype(np.int32), device)


class SpeedPerturb:
    """Speed perturbation (Ko et al. 2015, "Audio augmentation for speech recognition"): per utterance a factor drawn
    uniformly from `factors` resamples the waveform by up / down = 1 / factor, which changes its tempo and pitch together
    (a factor 1.1 plays 10 % faster: 10 / 11 as many samples).  The resampling is `resample` (scipy.signal.resample_poly
    restated, include/b200asr.h); a factor of 1 copies.  Each factor is taken as the exact decimal Fraction(str(f)).

    A SpeedPerturb holds plain numbers, so it pickles (DataLoader workers receive it with the dataset it is attached to)."""

    def __init__(self, factors=(0.9, 1.0, 1.1)):
        try:
            fs = list(factors)
        except TypeError:
            raise ValueError(f"SpeedPerturb: factors={factors!r} is not a sequence") from None
        if not fs:
            raise ValueError("SpeedPerturb: no factors")
        for f in fs:
            if isinstance(f, bool) or not isinstance(f, (int, float, np.integer, np.floating)) or not np.isfinite(f) or f <= 0:
                raise ValueError(f"SpeedPerturb: factor {f!r} must be a finite number > 0")
            up, down = self.ratio(f)
            if max(up, down) > RESAMPLE_MAX_RATE:
                raise ValueError(f"SpeedPerturb: factor {f!r} gives the ratio {up}/{down}, beyond {RESAMPLE_MAX_RATE} in "
                                 "lowest terms")
        self.factors = tuple(float(f) for f in fs)

    def __repr__(self):
        return f"SpeedPerturb(factors={self.factors})"

    def draw_one(self, rng=np.random) -> float:
        """One rng.choice over the factors (`rng` is np.random, the worker's global state, or a RandomState); returns the
        factor drawn."""
        return self.factors[int(rng.choice(len(self.factors)))]

    @staticmethod
    def ratio(f) -> tuple[int, int]:
        """(up, down) = 1 / Fraction(str(f)) in lowest terms: (10, 11) for 1.1, (10, 9) for 0.9, (1, 1) for 1.0."""
        r = 1 / Fraction(str(f))
        return r.numerator, r.denominator

    @staticmethod
    def out_length(n: int, f) -> int:
        """Samples of an utterance of `n` samples at factor f: ceil(n up / down)."""
        return resample_out_length(n, *SpeedPerturb.ratio(f))


def _geometry(sample_rate, window_size, window_stride):
    return int(sample_rate * window_size), int(sample_rate * window_stride)


def _features(wave, lens, t_max, n_fft, hop, normalize, reflect, precision, window, window_periodic, noise, max_frames,
              offsets=None, Lmax=None):
    """One b200asr_stft_features_ex call on a [B, Lmax] device batch, or with `offsets` one b200asr_stft_features_packed
    call on `wave` holding the utterances back to back (utterance b at offsets[b], Lmax >= every length):
    (inputs [B,1,F,t_max], frames [B] int32)."""
    if offsets is None:
        B, Lmax = wave.shape
    else:
        B = offsets.numel()
    nb = n_fft // 2 + 1
    lib = ops._lib()
    ws = torch.empty(lib.b200asr_stft_features_ex_ws_bytes(B, Lmax, n_fft, hop) // 4, device=wave.device, dtype=torch.float32)
    out = torch.empty((B, 1, nb, t_max), device=wave.device, dtype=torch.float32)
    frames = torch.empty(B, device=wave.device, dtype=torch.int32)
    prec = ops.config.linear if precision is None else precision
    prec = {L.PREC_BF16X3: L.PREC_TF32X3, L.PREC_BF16: L.PREC_TF32}.get(prec, prec)      # the DFT basis is an fp32 operand: tf32 grades
    bank, bank_len, start, level = noise if noise is not None else (None, 0, None, None)
    args = (L.ptr(lens), L.ptr(out), L.ptr(frames), L.ptr(ws), B, Lmax, t_max, n_fft, hop, int(reflect), int(normalize),
            WINDOWS.get(window, 0), int(window_periodic), L.ptr(bank), bank_len, L.ptr(start), L.ptr(level),
            NO_CUT if max_frames is None else max_frames, prec, ops._stream())
    if offsets is None:
        L.check(lib.b200asr_stft_features_ex(L.ptr(wave), *args), "stft_features_ex")
    else:
        L.check(lib.b200asr_stft_features_packed(L.ptr(wave), L.ptr(offsets), *args), "stft_features_packed")
    return out, frames


def stft_features_packed(wave: torch.Tensor, offsets: torch.Tensor, lengths: torch.Tensor, Lmax: int, t_max: int,
                         sample_rate: int = 16000, window_size: float = 0.02, window_stride: float = 0.01, normalize: bool = True,
                         reflect: bool = True, precision: int | None = None, window_periodic: bool = False,
                         window: str = "hamming", noise=None, max_frames: int | None = None):
    """The features of a packed batch: utterance b is the lengths[b] samples of the 1-D CUDA fp32 `wave` from offsets[b]
    (int64) on.  `Lmax` >= every length and `t_max` are host ints (no host read of the device arrays); `noise` is
    NoiseBank.device_args' tuple or None.  Equal bit for bit to spectrogram_batch on the same utterances zero-padded to
    [B, Lmax].  Returns (inputs [B,1,F,t_max] fp32, input_sizes [B] int32) on the device."""
    n_fft, hop = _geometry(sample_rate, window_size, window_stride)
    ops._need_cuda(wave, offsets, lengths)
    return _features(ops._f32c(wave), lengths.to(torch.int32), t_max, n_fft, hop, normalize, reflect, precision, window,
                     window_periodic, noise, max_frames, offsets=offsets.to(torch.int64), Lmax=int(Lmax))


def spectrogram_batch(waves: Sequence[torch.Tensor] | torch.Tensor, lengths: torch.Tensor | None = None, sample_rate: int = 16000,
                      window_size: float = 0.02, window_stride: float = 0.01, normalize: bool = True, reflect: bool = True,
                      precision: int | None = None, window_periodic: bool = False, window: str = "hamming",
                      noise: NoiseDraws | None = None, max_frames: int | None = None, spec_augment: SpecAugment | None = None):
    """waves: list of 1-D CUDA float tensors, or a zero-padded [B, L_max] CUDA tensor with `lengths` (int32 samples).
    `window`: "hamming", "hann", "blackman" or "bartlett" (any other name: Hamming, as the reference).  `noise`: draws of
    `NoiseBank.draw` for these utterances, in this order.  `max_frames`: keep at most this many frames of each utterance
    after normalising over all of them (the reference's src_max_len cut).  `spec_augment`: a SpecAugment applied to the
    batch after the cut (SpecAugment.apply, which advances its counter); None leaves the features as they are.
    Returns (inputs [B,1,F,T_max] fp32, input_percentages [B] fp32, input_sizes [B] int32), all on the device."""
    n_fft, hop = _geometry(sample_rate, window_size, window_stride)
    if isinstance(waves, torch.Tensor):
        if lengths is None:
            raise ValueError("a padded batch needs `lengths`")
        wave = waves
        lens = lengths.to(device=wave.device, dtype=torch.int32)
    else:
        dev = waves[0].device
        lens = torch.tensor([int(w.numel()) for w in waves], dtype=torch.int32, device=dev)
        wave = torch.zeros((len(waves), int(lens.max().item())), device=dev, dtype=torch.float32)
        for b, w in enumerate(waves):
            wave[b, : w.numel()] = w
    ops._need_cuda(wave, lens)
    wave = ops._f32c(wave)
    if max_frames is not None and max_frames < 1:
        raise ValueError(f"max_frames={max_frames}")
    t_max = 1 + int(lens.max().item()) // hop
    if max_frames is not None:
        t_max = min(t_max, max_frames)
    dev_noise = None if noise is None else noise.bank._device_args(noise, lens.cpu().numpy(), wave.device)
    out, frames = _features(wave, lens, t_max, n_fft, hop, normalize, reflect, precision, window, window_periodic, dev_noise,
                            max_frames)
    if spec_augment is not None:
        out, _ = spec_augment.apply(out, frames)
    return out, frames.float() / float(t_max), frames


def collate_waves(batch, audio_conf: dict, src_max_len: int, noise_bank: NoiseBank | None = None, normalize: bool = True,
                  rng=np.random, precision: int | None = None, reflect: bool = True, spec_augment: SpecAugment | None = None,
                  tempo_gain: TempoGain | None = None, speed_perturb: SpeedPerturb | None = None):
    """`_collate_fn` (utils/data_loader.py:182-214) over waveforms: what a DataLoader over the reference's
    `SpectrogramDataset` yields, computed on the device.

    batch: list of (waveform, transcript ids); waveforms are 1-D fp32 host arrays (numpy or CPU tensors).  audio_conf: the
    dict train.py builds (sample_rate, window_size, window_stride, window, noise_dir, noise_prob, noise_levels).  With
    audio_conf["noise_dir"] set, noise is drawn from `noise_bank` (ValueError without one) in batch order, before
    sorting, as `__getitem__` draws it.  Each spectrogram is normalised over the whole utterance, then cut to
    `src_max_len` frames (:131).  `spec_augment`: a SpecAugment applied to the sorted batch after the cut
    (SpecAugment.apply, which advances its counter); None leaves the features as they are.  `tempo_gain`: a TempoGain
    (the reference's `augment=True`): each utterance draws its tempo and gain, then its noise for the stretched length,
    in batch order as `__getitem__` draws them, and the batch is stretched on the device (one `tempo_gain` launch)
    before the features; the frame counts are those of the stretched utterances.  None: no stretch and no such draw.
    `speed_perturb`: a SpeedPerturb: each utterance draws its factor after its tempo and gain and before its noise, the
    noise is drawn for the resampled length, and the batch is resampled on the device (one `resample` launch) after the
    stretch and before the features.  None: no resampling and no such draw.

    Returns (inputs [B,1,F,T] fp32 on the current CUDA device, targets [B,max_tgt] int64, input_percentages [B] fp32,
    input_sizes [B] int32, target_sizes [B] int32), the last four on the host, sorted by frame count, longest first
    (stable).  It launches CUDA work and does not synchronise with the host, so it belongs in the main process rather than
    in DataLoader workers: let the workers return (waveform, ids) lists and call this on each batch."""
    sr = audio_conf["sample_rate"]
    n_fft, hop = _geometry(sr, audio_conf["window_size"], audio_conf["window_stride"])
    if src_max_len < 1:
        raise ValueError(f"src_max_len={src_max_len}")
    waves = [np.asarray(w.detach().cpu() if isinstance(w, torch.Tensor) else w, dtype=np.float32).reshape(-1) for w, _ in batch]
    lens = [len(w) for w in waves]
    noisy = audio_conf.get("noise_dir") is not None
    if noisy and noise_bank is None:
        raise ValueError("audio_conf['noise_dir'] is set but no noise_bank was given")
    if tempo_gain is not None:
        TempoGain.geometry(sr)                        # a rate without a valid geometry fails before any draw
    stretch, speed, rows, out_lens = [], [], [], []
    for n in lens:                                    # per utterance: tempo and gain, speed, then the noise of the final length
        if tempo_gain is not None:
            t, gain_db = tempo_gain.draw_one(rng)
            n = TempoGain.out_length(n, t)
            stretch.append((t, TempoGain.linear_gain(gain_db), n))
        if speed_perturb is not None:
            up, down = speed_perturb.ratio(speed_perturb.draw_one(rng))
            n = resample_out_length(n, up, down)
            speed.append((up, down))
        out_lens.append(n)
        if noisy:
            rows.append(noise_bank.clips.draw_one(n, audio_conf["noise_prob"], audio_conf["noise_levels"], rng))
    draws = noise_bank._draws(rows) if noisy else None
    frames = [min(1 + n // hop, src_max_len) for n in out_lens]
    order = sorted(range(len(batch)), key=frames.__getitem__, reverse=True)          # sorted(..., reverse=True) is stable
    B, Lmax = len(batch), max(1, max(out_lens))
    slens = np.array([lens[i] for i in order], dtype=np.int32)
    offsets = np.concatenate([[0], np.cumsum(slens, dtype=np.int64)[:-1]])
    host = torch.empty(max(1, int(slens.sum())), dtype=torch.float32, pin_memory=True)   # back to back, uploaded without a sync
    h = host.numpy()
    for r, i in enumerate(order):
        h[offsets[r]:offsets[r] + lens[i]] = waves[i]
    device = torch.device("cuda", torch.cuda.current_device())
    wave, wave_offsets, wave_lens = host.to(device, non_blocking=True), _pinned_to(offsets, device), _pinned_to(slens, device)
    if tempo_gain is not None:
        tlens = np.array([stretch[i][2] for i in order], np.int32)
        wave, wave_offsets, wave_lens, _, _ = _tempo_gain(
            wave, wave_offsets, wave_lens, np.array([stretch[i][0] for i in order], np.float64),
            np.array([stretch[i][1] for i in order], np.float32), tlens, sr)
        offsets, slens = np.concatenate([[0], np.cumsum(tlens, dtype=np.int64)[:-1]]), tlens
    if speed_perturb is not None:
        wave, offsets, slens = _resample(wave, offsets, slens, [speed[i][0] for i in order], [speed[i][1] for i in order],
                                         False)
        wave_offsets, wave_lens = _pinned_to(offsets, device), _pinned_to(slens.astype(np.int32), device)
    sout = np.array([out_lens[i] for i in order], dtype=np.int64)
    dev_noise = None if draws is None else noise_bank._device_args(draws.take(order), sout, device)
    t_max = frames[order[0]]
    inputs, _ = _features(wave, wave_lens, t_max, n_fft, hop, normalize, reflect, precision, audio_conf.get("window", "hamming"),
                          False, dev_noise, src_max_len, offsets=wave_offsets, Lmax=Lmax)
    targets_list = [batch[i][1] for i in order]
    max_tgt = max(len(t) for t in targets_list)
    targets = torch.zeros(B, max_tgt, dtype=torch.int64)
    for r, t in enumerate(targets_list):
        targets[r, :len(t)] = torch.tensor(list(t), dtype=torch.int32)
    input_sizes = torch.tensor([frames[i] for i in order], dtype=torch.int32)
    if spec_augment is not None:
        inputs, _ = spec_augment.apply(inputs, input_sizes)
    input_percentages = torch.tensor([frames[i] / float(t_max) for i in order], dtype=torch.float32)
    target_sizes = torch.tensor([len(t) for t in targets_list], dtype=torch.int32)
    return inputs, targets, input_percentages, input_sizes, target_sizes
