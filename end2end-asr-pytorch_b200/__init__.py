"""b200asr -- H100-native hot path of gentaiscool/end2end-asr-pytorch (teacher-forced Transformer-ASR fwd+bwd).

Everything computes in hand-written sm_90a CUDA kernels behind the C ABI of include/b200asr.h
(libb200asr.so, built in-tree).  There is no CPU or stock-PyTorch fallback: importing is fine anywhere, running
needs the built library and an H100.
"""
from . import _lib, lm_train
from .config import ASRConfig, BASELINE_CONFIGS
from .features import NoiseBank, NoiseClips, collate_waves, spectrogram_batch, stft_features_packed
from .install import install, original, uninstall
from .metrics import LabelTable, calculate_loss, calculate_metrics, edit_counts, loss_and_stats
from .modules import (LM, Decoder, DecoderLayer, Encoder, EncoderLayer, MultiHeadAttention, PositionalEncoding,
                      PositionwiseFeedForwardWithConv, RNNModel, ScaledDotProductAttention, Transformer, build_model)
from .ops import attention_maps, config as precision, manual_seed
from .optim import FlatParams, FusedAdam, NoamOpt, adam_step, clip_grad_norm_
from .parallel import DataParallelStep, HostBatchPrefetcher, shard_batch

__all__ = ["ASRConfig", "BASELINE_CONFIGS", "install", "uninstall", "original", "calculate_loss", "calculate_metrics",
           "loss_and_stats", "LabelTable", "edit_counts","Transformer", "Encoder", "Decoder", "EncoderLayer", "DecoderLayer", "MultiHeadAttention",
           "ScaledDotProductAttention", "PositionwiseFeedForwardWithConv", "PositionalEncoding", "build_model", "RNNModel", "LM",
           "precision", "manual_seed", "attention_maps", "spectrogram_batch", "NoiseBank", "NoiseClips", "collate_waves", "stft_features_packed","FlatParams", "FusedAdam", "NoamOpt", "adam_step", "clip_grad_norm_", "DataParallelStep", "HostBatchPrefetcher", "shard_batch", "lm_train"]
