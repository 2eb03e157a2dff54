"""Host restatement of b200asr_spec_augment (include/b200asr.h): its counter-based draws, exactly, and the warp and masks
in float64 from a given set of draws."""
import math

import numpy as np

M64 = 2 ** 64 - 1
GOLDEN = 0x9E3779B97F4A7C15


def splitmix64(z: int) -> int:
    z = (z + GOLDEN) & M64
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M64
    return z ^ (z >> 31)


def key(seed: int, counter: int) -> int:
    """dropout_key(seed, counter) of common.cuh."""
    return splitmix64(seed ^ ((counter * 0xD1342543DE82EF95 + 0x2545F4914F6CDD1D) & M64))


def uniform(k: int, b: int, slot: int, lo: int, hi: int) -> int:
    r = splitmix64((k + ((b << 16) | slot) * GOLDEN) & M64)
    return lo + (((r >> 32) * (hi - lo + 1)) >> 32)


def draws(sizes, F: int, T: int, W: int, Fp: int, nf: int, Tp: int, p: float, nt: int, seed: int, counter: int):
    """[B, 2 + 2 nf + 2 nt] int32: c, w, (f, f0) per frequency mask, (t, t0) per time mask of every utterance."""
    k = key(seed, counter)
    p32 = float(np.float32(p))                     # the kernel takes p as a float
    rows = []
    for b, n in enumerate(sizes):
        Tb = min(max(int(n), 0), T)
        row = [0, 0]
        if Tb > 2 * W + 1:
            row = [uniform(k, b, 0, W, Tb - W - 1), uniform(k, b, 1, -W, W)]
        for m in range(nf):
            f = uniform(k, b, 2 + 2 * m, 0, Fp)
            row += [f, uniform(k, b, 3 + 2 * m, 0, F - f)]
        cap = min(Tp, math.floor(p32 * Tb))
        for m in range(nt):
            s = 2 + 2 * nf + 2 * m
            t = uniform(k, b, s, 0, cap)
            row += [t, uniform(k, b, s + 1, 0, Tb - t)]
        rows.append(row)
    return np.array(rows, dtype=np.int32).reshape(len(sizes), 2 + 2 * nf + 2 * nt)


def source_position(t: int, Tb: int, c: int, w: int) -> float:
    """The warp's source frame for output frame t < Tb, exact: 0 -> 0, c + w -> c, Tb - 1 -> Tb - 1, linear between; the
    end frames read themselves also when c + w is one of them."""
    d = c + w
    if w == 0 or t == 0 or t == Tb - 1:
        return float(t)
    if t <= d:
        return t * c / d
    return c + (t - d) * (Tb - 1 - c) / (Tb - 1 - d)


def reference(x: np.ndarray, drw: np.ndarray, sizes, nf: int, nt: int):
    """float64 SpecAugment of x [B,1,F,T] with the given draws.  Returns (out, zero, bound): zero marks the elements that
    must be exactly 0 (masks and padding), bound the fp32 error allowed per element (0 where the fp32 result must be x's
    own bits): 2^-22 (|x[i0]| + |x[i0 + 1]|) where the warp interpolates."""
    x = np.asarray(x, dtype=np.float64)
    B, _, F, T = x.shape
    out = np.zeros_like(x)
    zero = np.zeros(x.shape, dtype=bool)
    bound = np.zeros_like(x)
    for b in range(B):
        Tb = min(max(int(sizes[b]), 0), T)
        c, w = int(drw[b, 0]), int(drw[b, 1])
        for t in range(Tb):
            s = source_position(t, Tb, c, w)
            i0 = int(math.floor(s))
            a = s - i0
            if a == 0.0:
                out[b, 0, :, t] = x[b, 0, :, i0]
            else:
                out[b, 0, :, t] = x[b, 0, :, i0] + a * (x[b, 0, :, i0 + 1] - x[b, 0, :, i0])
                bound[b, 0, :, t] = 2.0 ** -22 * (np.abs(x[b, 0, :, i0]) + np.abs(x[b, 0, :, i0 + 1]))
        zero[b, 0, :, Tb:] = True
        for m in range(nf):
            f, f0 = int(drw[b, 2 + 2 * m]), int(drw[b, 3 + 2 * m])
            zero[b, 0, f0:f0 + f, :] = True
        for m in range(nt):
            t, t0 = int(drw[b, 2 + 2 * nf + 2 * m]), int(drw[b, 3 + 2 * nf + 2 * m])
            zero[b, 0, :, t0:t0 + t] = True
    out[zero] = 0.0
    bound[zero] = 0.0
    return out, zero, bound
