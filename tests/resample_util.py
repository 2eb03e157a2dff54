"""numpy restatement of the polyphase resampler (b200asr_resample_packed, features.resample; include/b200asr.h states the
algorithm): resample_poly's output as the phase-split sum, in float64, and the fp32 error bound of the kernel's sum."""
import numpy as np

from b200asr import features as F

RATIOS = [(10, 9), (10, 11), (2, 1), (1, 2), (160, 441), (147, 160), (1, 1)]


def _terms(x, up, down, taps):
    """(taps of each output's phase [n_out, K], the inputs they multiply [n_out, K]) in float64, zeros past the ends."""
    x = np.asarray(x, np.float64)
    half = 10 * max(up, down)
    n_out = F.resample_out_length(len(x), up, down)
    K = taps.shape[1]
    c = np.arange(n_out, dtype=np.int64) * down + half
    j = c[:, None] // up - np.arange(K)[None, :]
    xt = np.zeros(len(x) + 2 * K + (n_out * down) // up + 2, np.float64)
    xt[K:K + len(x)] = x
    return np.asarray(taps, np.float64)[c % up], xt[np.clip(j + K, 0, len(xt) - 1)]


def polyphase(x, up, down):
    """resample_poly(x, up, down) for a reduced ratio, as the phase-split sum over the float64 filter."""
    if up == down == 1:
        return np.asarray(x, np.float64).copy()
    h = F.resample_filter(up, down)
    K = -(-len(h) // up)
    taps = np.pad(h, (0, up * K - len(h))).reshape(K, up).T
    t, X = _terms(x, up, down, taps)
    return (t * X).sum(axis=1)


def fp32_bound(x, up, down):
    """Per output, a bound on |kernel - resample_poly in float64|: the taps rounded to fp32 (2^-24 each) and K fp32 FMAs
    (2^-24 per step) over sum |h x|, doubled."""
    if up == down == 1:
        return np.zeros(len(x))
    taps = F.resample_taps(up, down)
    t, X = _terms(x, up, down, taps)
    return 2.0 ** -23 * (taps.shape[1] + 2) * (np.abs(t) * np.abs(X)).sum(axis=1)


def quantize16(v):
    """clamp(rint(v * 32768), -32768, 32767) / 32768 in fp32, half to even."""
    v = np.asarray(v, np.float32)
    return (np.clip(np.rint(v * np.float32(32768)), -32768, 32767) / np.float32(32768)).astype(np.float32)
