"""CPU restatement of the reference's loader options the device front end adds to oracle/features_oracle.py: every window
of utils/data_loader.py:20-21, noise injection (:163-179) and the src_max_len cut after normalisation (:131).

Windows are scipy's (scipy.signal.windows.*): the reference hands librosa the callable, which librosa evaluates as
window(n_fft), so sym=True; periodic (sym=False) is the window of the first n_fft points of an (n_fft + 1)-point one.
Everything is float64; tests/test_feature_augment_host.py pins it to scipy and to tests/golden/noise.npz, which the
unmodified reference wrote (tests/golden/make_noise_golden.py)."""
import numpy as np

WINDOWS = ("hamming", "hann", "blackman", "bartlett")


def window(name: str, n_fft: int, periodic: bool = False) -> np.ndarray:
    """The reference's window for `name`; any other name is Hamming, as windows.get(name, hamming) (:52)."""
    n = np.arange(n_fft, dtype=np.float64)
    x = 2.0 * n / (n_fft if periodic else n_fft - 1)           # 2 n / (N - 1), or 2 n / N when periodic
    if name == "hann":
        return 0.5 - 0.5 * np.cos(np.pi * x)
    if name == "blackman":
        return 0.42 - 0.5 * np.cos(np.pi * x) + 0.08 * np.cos(2.0 * np.pi * x)
    if name == "bartlett":
        return 1.0 - np.abs(x - 1.0)
    return 0.54 - 0.46 * np.cos(np.pi * x)


def mix(x: np.ndarray, n: np.ndarray, level: float) -> np.ndarray:
    """NoiseInjection.inject_noise_sample (:176-178): x + level * n * e_x / e_n with e = sqrt(mean of squares)."""
    x, n = np.asarray(x, np.float64), np.asarray(n, np.float64)
    ex, en = np.sqrt(x.dot(x) / x.size), np.sqrt(n.dot(n) / n.size)
    with np.errstate(invalid="ignore", divide="ignore"):
        return x + level * n * ex / en


def stft(y: np.ndarray, n_fft: int, hop: int, win: np.ndarray, reflect: bool = True) -> np.ndarray:
    """librosa.stft(y, n_fft, hop, win_length=n_fft, window) with centred frames: complex [n_fft // 2 + 1, 1 + len // hop]."""
    y = np.asarray(y, dtype=np.float64)
    half = n_fft // 2
    yp = np.pad(y, (half, half), mode="reflect" if reflect else "constant")
    n_frames = 1 + len(y) // hop
    idx = np.arange(n_fft)[None, :] + hop * np.arange(n_frames)[:, None]
    return np.fft.rfft(yp[idx] * win[None, :], axis=1).T


def log_spectrogram(y, n_fft=320, hop=160, window_name="hamming", periodic=False, reflect=True, normalize=True,
                    max_frames=None) -> np.ndarray:
    """parse_audio (:72-91) then the cut of __getitem__ (:131): float32 [bins, min(frames, max_frames)], normalised over
    ALL frames of the utterance before the cut."""
    s = np.log1p(np.abs(stft(y, n_fft, hop, window(window_name, n_fft, periodic), reflect)))
    if normalize:
        s = (s - s.mean()) / s.std(ddof=1)                                   # torch.Tensor.std is unbiased
    return s[:, :max_frames].astype(np.float32)


def collate(specs, targets):
    """_collate_fn (:182-214) on (spectrogram, ids) pairs: sorted by frame count, longest first (stable)."""
    order = sorted(range(len(specs)), key=lambda i: specs[i].shape[1], reverse=True)
    t_max = specs[order[0]].shape[1]
    max_tgt = max(len(t) for t in targets)
    inputs = np.zeros((len(specs), 1, specs[0].shape[0], t_max), dtype=np.float32)
    tgt = np.zeros((len(specs), max_tgt), dtype=np.int64)
    for r, i in enumerate(order):
        inputs[r, 0, :, :specs[i].shape[1]] = specs[i]
        tgt[r, :len(targets[i])] = targets[i]
    sizes = np.array([specs[i].shape[1] for i in order], dtype=np.int32)
    pct = np.array([s / float(t_max) for s in sizes], dtype=np.float32)
    return order, inputs, tgt, pct, sizes, np.array([len(targets[i]) for i in order], dtype=np.int32)
