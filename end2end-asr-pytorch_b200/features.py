"""GPU feature front end: waveforms -> the `(inputs, input_percentages, input_sizes)` triple of the reference's loader.

Mirrors `SpectrogramParser.parse_audio` (utils/data_loader.py:60-91) + the padded batch of `_collate_fn` (:182-214):
STFT (n_fft = sample_rate * window_size, hop = sample_rate * window_stride, symmetric Hamming window -- the reference
passes the callable scipy.signal.hamming, which librosa evaluates as window(n_fft), i.e. sym=True --, centred frames),
magnitude, log1p, per-utterance mean / unbiased-std normalisation, zero padding to the longest utterance.  One C-ABI call
(`b200asr_stft_features`): the STFT of the whole batch is a single 3xTF32 tensor-core GEMM over overlapping frame rows.
"""
from __future__ import annotations

from typing import Sequence

import torch

from . import _lib as L
from . import ops


def spectrogram_batch(waves: Sequence[torch.Tensor] | torch.Tensor, lengths: torch.Tensor | None = None, sample_rate: int = 16000,
                      window_size: float = 0.02, window_stride: float = 0.01, normalize: bool = True, reflect: bool = True,
                      precision: int | None = None, window_periodic: bool = False):
    """waves: list of 1-D CUDA float tensors, or a zero-padded [B, L_max] CUDA tensor with `lengths` (int32 samples).
    Returns (inputs [B,1,F,T_max] fp32, input_percentages [B] fp32, input_sizes [B] int32), all on the device."""
    n_fft, hop = int(sample_rate * window_size), int(sample_rate * window_stride)
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
    B, Lmax = wave.shape
    t_max = 1 + int(lens.max().item()) // hop
    nb = n_fft // 2 + 1
    lib = ops._lib()
    ws = torch.empty(lib.b200asr_stft_ws_bytes(B, Lmax, n_fft, hop) // 4, device=wave.device, dtype=torch.float32)
    out = torch.empty((B, 1, nb, t_max), device=wave.device, dtype=torch.float32)
    frames = torch.empty(B, device=wave.device, dtype=torch.int32)
    prec = ops.config.linear if precision is None else precision
    prec = {L.PREC_BF16X3: L.PREC_TF32X3, L.PREC_BF16: L.PREC_TF32}.get(prec, prec)      # the DFT basis is an fp32 operand: tf32 grades
    L.check(lib.b200asr_stft_features(L.ptr(wave), L.ptr(lens), L.ptr(out), L.ptr(frames), L.ptr(ws), B, Lmax, t_max, n_fft, hop,
                                      int(reflect), int(normalize), int(window_periodic), prec, ops._stream()), "stft_features")
    return out, frames.float() / float(t_max), frames
