#!/usr/bin/env python
"""Generate tests/golden/noise.npz from the UNMODIFIED reference loader: SpectrogramDataset.__getitem__,
SpectrogramParser.parse_audio, NoiseInjection and _collate_fn (utils/data_loader.py:40-214).

Run where the reference checkout is readable (oracle/ref_shim.py finds it):

    python tests/golden/make_noise_golden.py [--out PATH]

What is not installed is stubbed; the reference itself is not edited:
  * `librosa`: util.find_files returns the noise clips' names; stft records the waveform and the window it is given and
    returns tests/augment_oracle.stft of them; magphase is |D| and D / |D|.
  * scipy.signal.{hamming, hann, blackman, bartlett} are scipy.signal.windows.* (scipy >= 1.13 dropped the old names).
  * `torchaudio` (imported by utils/audio.py, never called here) is an empty module when absent.
  * load_audio, get_audio_length and audio_with_sox, as data_loader.py imported them, are lookups in the clips and
    utterances below.  audio_with_sox's sox `trim` is restated: the segment starts at sample round(start * sr), clamped
    so that its round((end - start) * sr) samples fit in the clip -- the rule b200asr.NoiseBank.draw documents.

Cases cover noise_prob 0, 0.5 and 1, every window name plus an unknown one (which falls back to Hamming), and a
src_max_len that cuts and one that does not.  np.random is seeded per case.  The npz is written with fixed zip
timestamps, so a rerun reproduces it byte for byte.
"""
import argparse
import io
import os
import sys
import tempfile
import types
import zipfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
SR, WINDOW_SIZE, WINDOW_STRIDE = 16000, 0.02, 0.01
# (noise_prob, window, src_max_len, utterance lengths in samples)
CASES = [(0.0, "hamming", 4000, [1600, 2399, 800, 2400, 161]),
         (0.5, "hann", 9, [2000, 1440, 3000, 1279, 2500, 960]),
         (1.0, "blackman", 4000, [3200, 1000, 2560, 159, 2100]),
         (1.0, "bartlett", 12, [2880, 1920, 1920, 640, 3100]),
         (0.5, "kaiser", 4000, [1200, 2720, 480, 2240, 1760, 320])]
CLIP_LENGTHS = [4000, 3200, 6400, 3300]            # every clip at least as long as every utterance
NOISE_LEVELS = (0.0, 0.5)
VOCAB = "abcdefgh "


def _signals(seed, lengths, scale):
    g = np.random.default_rng(seed)
    out = []
    for n in lengths:
        t = np.arange(n) / SR
        y = scale * np.sin(2 * np.pi * (150 + 300 * g.random()) * t) + 0.05 * g.standard_normal(n)
        out.append(y.astype(np.float32))
    return out


def _write_npz(path, arrays):
    with zipfile.ZipFile(path, "w", compression=zipfile.ZIP_DEFLATED) as z:
        for k in sorted(arrays):
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.asarray(arrays[k]), allow_pickle=False)
            info = zipfile.ZipInfo(k + ".npy", date_time=(1980, 1, 1, 0, 0, 0))
            info.compress_type = zipfile.ZIP_DEFLATED
            info.external_attr = 0o600 << 16
            z.writestr(info, buf.getvalue())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(HERE, "noise.npz"))
    out_path = ap.parse_args().out
    sys.path.insert(0, ROOT)
    from oracle import ref_shim
    from tests import augment_oracle as AO
    import scipy.signal
    from scipy.signal import windows as W
    for name in ("hamming", "hann", "blackman", "bartlett"):
        if not hasattr(scipy.signal, name):
            setattr(scipy.signal, name, getattr(W, name))
    clips = {f"noise_{i}.wav": w for i, w in enumerate(_signals(99, CLIP_LENGTHS, 0.2))}
    names = sorted(clips)
    calls = []                                          # what the stubbed librosa.stft was handed
    lib = types.ModuleType("librosa")
    lib.util = types.SimpleNamespace(find_files=lambda path: list(names))

    def stft(y, n_fft, hop_length, win_length, window):
        assert win_length == n_fft and callable(window)
        win = np.asarray(window(n_fft), dtype=np.float64)
        calls.append((np.array(y, copy=True), win))
        return AO.stft(y, n_fft, hop_length, win)

    lib.stft = stft
    lib.magphase = lambda D: (np.abs(D), D / np.where(np.abs(D) == 0, 1, np.abs(D)))
    sys.modules["librosa"] = lib
    try:
        import torchaudio  # noqa: F401
    except ImportError:
        sys.modules["torchaudio"] = types.ModuleType("torchaudio")
    ns = ref_shim.load([])
    import importlib
    import torch
    DL = importlib.import_module("utils.data_loader")
    const = ns.constant
    label2id = {c: i for i, c in enumerate([const.PAD_CHAR, const.SOS_CHAR, const.EOS_CHAR] + list(VOCAB))}

    utts = {}
    sox = []                                            # (clip name, start seconds, end seconds) per audio_with_sox call
    levels = []                                         # (clip name, level) per inject_noise_sample call

    def load_audio(path):
        return utts[path].copy()

    def get_audio_length(path):
        return len(clips[path]) / SR

    def audio_with_sox(path, sample_rate, start_time, end_time):
        assert sample_rate == SR
        clip = clips[path]
        n = int(round((end_time - start_time) * SR))
        s = min(max(int(round(start_time * SR)), 0), len(clip) - n)
        sox.append((path, start_time, end_time))
        return clip[s:s + n].copy()

    DL.load_audio, DL.get_audio_length, DL.audio_with_sox = load_audio, get_audio_length, audio_with_sox
    inject = DL.NoiseInjection.inject_noise_sample

    def recording_inject(self, data, noise_path, noise_level):
        levels.append((noise_path, noise_level))
        return inject(self, data, noise_path, noise_level)

    DL.NoiseInjection.inject_noise_sample = recording_inject
    out = {"meta.clips": np.concatenate([clips[n] for n in names]),
           "meta.clip_lengths": np.array([len(clips[n]) for n in names], dtype=np.int64),
           "meta.cfg": np.array([SR, int(SR * WINDOW_SIZE), int(SR * WINDOW_STRIDE)], dtype=np.int64),
           "meta.noise_levels": np.array(NOISE_LEVELS)}
    with tempfile.TemporaryDirectory() as tmp:
        for ci, (prob, window, src_max_len, lengths) in enumerate(CASES):
            waves = _signals(1000 + ci, lengths, 0.5)
            texts = ["".join(VOCAB[(ci + 3 * b + k) % len(VOCAB)] for k in range(2 + (5 * b + ci) % 7)) for b in range(len(waves))]
            manifest = os.path.join(tmp, f"m{ci}.csv")
            with open(manifest, "w") as f:
                for b, (w, t) in enumerate(zip(waves, texts)):
                    wav, txt = os.path.join(tmp, f"c{ci}_{b}.wav"), os.path.join(tmp, f"c{ci}_{b}.txt")
                    utts[wav] = w
                    with open(txt, "w") as g:
                        g.write(t)
                    f.write(f"{wav},{txt}\n")
            ns = ref_shim.load(["--src-max-len", str(src_max_len)])
            conf = dict(sample_rate=SR, window_size=WINDOW_SIZE, window_stride=WINDOW_STRIDE, window=window, noise_dir=tmp,
                        noise_prob=prob, noise_levels=NOISE_LEVELS)
            ds = DL.SpectrogramDataset(conf, [manifest], label2id, normalize=True)
            calls.clear(), sox.clear(), levels.clear()
            np.random.seed(4321 + ci)
            items, noisy = [], []
            for b in range(len(waves)):
                n0 = len(levels)
                items.append(ds[b])
                noisy.append(len(levels) > n0)
            inputs, targets, pct, sizes, tsizes = DL._collate_fn(items)
            assert len(calls) == len(waves) and len(sox) == len(levels)
            B = len(waves)
            clip, level, start_s = np.full(B, -1, np.int64), np.full(B, np.nan), np.full(B, np.nan)
            k = 0
            for b in range(B):
                if noisy[b]:
                    path, lev = levels[k]
                    assert sox[k][0] == path
                    clip[b], level[b], start_s[b] = names.index(path), lev, sox[k][1]
                    k += 1
            assert k == len(levels)
            p = f"c{ci}."
            out[p + "cfg"] = np.array([prob, src_max_len], dtype=np.float64)
            out[p + "window"] = np.array(window)
            out[p + "lengths"] = np.array(lengths, dtype=np.int64)
            out[p + "waves"] = np.concatenate(waves)
            out[p + "mixed"] = np.concatenate([c[0] for c in calls]).astype(np.float32)
            out[p + "win"] = calls[0][1]
            out[p + "ids"] = np.concatenate([np.array(t, dtype=np.int64) for _, t in items])
            out[p + "id_lengths"] = np.array([len(t) for _, t in items], dtype=np.int64)
            out[p + "add"] = np.array(noisy, dtype=np.int64)
            out[p + "clip"], out[p + "level"], out[p + "noise_start"] = clip, level, start_s
            out[p + "spect"] = np.concatenate([s.numpy().reshape(-1) for s, _ in items])
            out[p + "frames"] = np.array([s.shape[1] for s, _ in items], dtype=np.int64)
            out[p + "inputs"], out[p + "targets"], out[p + "pct"] = inputs.numpy(), targets.numpy(), pct.numpy()
            out[p + "sizes"], out[p + "tsizes"] = sizes.numpy(), tsizes.numpy()
            print(f"case {ci}: p={prob} window={window} src_max_len={src_max_len} noisy={noisy} frames={out[p + 'frames'].tolist()}")
    assert torch.is_tensor(inputs)
    _write_npz(out_path, out)
    print("->", out_path, "%.1f KB" % (os.path.getsize(out_path) / 1024))


if __name__ == "__main__":
    main()
