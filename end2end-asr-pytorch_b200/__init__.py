"""b200asr -- H100-native hot path of gentaiscool/end2end-asr-pytorch (teacher-forced Transformer-ASR fwd+bwd).

Everything computes in hand-written sm_90a CUDA kernels behind the C ABI of include/b200asr.h
(libb200asr.so, built in-tree).  There is no CPU or stock-PyTorch fallback: importing is fine anywhere, running
needs the built library and an H100.
"""
from . import _lib
from .config import ASRConfig, BASELINE_CONFIGS
from .features import spectrogram_batch
from .install import install, uninstall
from .metrics import calculate_loss, calculate_metrics, loss_and_stats
from .modules import (Decoder, DecoderLayer, Encoder, EncoderLayer, MultiHeadAttention, PositionalEncoding,
                      PositionwiseFeedForwardWithConv, ScaledDotProductAttention, Transformer, build_model)
from .ops import config as precision, manual_seed
from .optim import FlatParams, FusedAdam, NoamOpt
from .parallel import DataParallelStep, HostBatchPrefetcher, shard_batch

__all__ = ["ASRConfig", "BASELINE_CONFIGS", "install", "uninstall", "calculate_loss", "calculate_metrics",
           "loss_and_stats", "Transformer", "Encoder", "Decoder", "EncoderLayer", "DecoderLayer", "MultiHeadAttention",
           "ScaledDotProductAttention", "PositionwiseFeedForwardWithConv", "PositionalEncoding", "build_model",
           "precision", "manual_seed", "spectrogram_batch", "FlatParams", "FusedAdam", "NoamOpt", "DataParallelStep", "HostBatchPrefetcher", "shard_batch"]
