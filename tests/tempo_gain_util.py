"""numpy restatement of the tempo and gain perturbation (b200asr_tempo_gain, features.TempoGain; include/b200asr.h states
the algorithm): WSOLA at sox's default tempo geometry, then the gain and the 16-bit output.  float64 for the search,
fp32 for every output operation, each rounded on its own (numpy does not contract into FMAs)."""
import numpy as np


def geometry(sr):
    """(segment, search, overlap) of sox's default tempo profile at `sr`, in float64."""
    segment = int(np.floor(sr * 82 / 1000 + 0.5))
    search = int(np.floor(sr * (82 / 5.587) / 1000 + 0.5))
    overlap = int(np.floor(max(sr * (82 / 6.833) / 1000 + 4.5, 16)))
    overlap -= overlap % 8
    if 2 * overlap > segment:
        overlap -= 8
    return segment, search, overlap


def out_length(n, tempo):
    return int(np.floor(n / tempo + 0.5))


def linear_gain(gain_db):
    return np.float32(10.0 ** (gain_db / 20.0))


def starts(tempo, K, step):
    return [int(np.floor(tempo * float(k * step) + 0.5)) for k in range(K)]


def distances(xt, S, prev, search, overlap):
    """D(i) = sum_j (x~[S + i + j] - prev_j)^2 in float64 for i < search; NaN counts as +inf."""
    w = np.lib.stride_tricks.sliding_window_view(xt[S:S + search + overlap - 1].astype(np.float64), overlap)
    D = ((w - prev.astype(np.float64)) ** 2).sum(axis=1)
    return np.where(np.isnan(D), np.inf, D)


def stretch(x, tempo, g, geom, picks=None):
    """The output (fp32, out_length(len(x), tempo) samples) and the picks of one utterance.  With `picks` given, segment k
    uses picks[k] instead of searching (the replay of another implementation's choices); D of every segment k >= 1 is
    returned as well, computed against the previous segment's pick actually used."""
    segment, search, overlap = geom
    step = segment - overlap
    x = np.asarray(x, dtype=np.float32)
    n = len(x)
    olen = out_length(n, tempo)
    K = -(-olen // step)
    S = starts(tempo, K, step)
    xt = np.zeros(max([n] + [s + search + segment for s in S]), np.float32)
    xt[:n] = x
    rcp = np.float32(1) / np.float32(overlap)
    f = np.arange(overlap, dtype=np.float32) * rcp
    one_minus = np.float32(1) - f
    y = np.empty(K * step, np.float32)
    got, Ds = [], []
    prev = None
    for k in range(K):
        if k == 0:
            p = search // 2
        else:
            D = distances(xt, S[k], prev, search, overlap)
            Ds.append(D)
            p = int(np.argmin(D)) if picks is None else int(picks[k])
        seg = xt[S[k] + p:S[k] + p + step].copy()
        if k > 0:
            seg[:overlap] = (prev * one_minus) + (seg[:overlap] * f)
        y[k * step:(k + 1) * step] = seg
        prev = xt[S[k] + p + step:S[k] + p + step + overlap].copy()
        got.append(p)
    v = y[:olen] * np.float32(g)
    q = np.clip(np.rint(v * np.float32(32768)), -32768, 32767) / np.float32(32768)
    return q.astype(np.float32), np.array(got, np.int32), Ds


def grid16(x):
    """x on the 16-bit grid, as load_audio returns a 16-bit file: round(32768 x) / 32768 clamped to [-1, 32767 / 32768]."""
    return (np.clip(np.rint(np.asarray(x, np.float64) * 32768), -32768, 32767) / 32768).astype(np.float32)
