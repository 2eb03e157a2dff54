/* libb200asr -- C ABI of the H100-native (sm_90a) speech-Transformer training hot path.
 *
 * The reference (gentaiscool/end2end-asr-pytorch) is pure Python on PyTorch and has NO FFI / operator
 * plugin interface (SURVEY.md §8b): its seams are nn.Module.forward methods and two free functions.  Each
 * entry point below therefore cites the reference *call site* whose ATen dispatches it replaces; the
 * host-side binding a maintainer would add is the ctypes stub shown in INTEGRATION.md.
 *
 * Conventions
 *   - plain pointers and sizes only; every pointer is a DEVICE pointer unless stated; fp32 data,
 *     int64 token ids (torch.long), uint8 masks (1 = masked / padded).
 *   - the caller owns all memory it passes (including workspaces); the library keeps one scratch buffer per
 *     (device, stream) of its own, for the partial results of reductions summed in a fixed order, so that the same
 *     inputs give the same bits every run (the fp32 CUDA-core GEMM / convolution / attention backward variants and
 *     the im2col convolution path still accumulate with atomics).
 *   - every function enqueues work on `stream` (a cudaStream_t passed as void*) and returns without
 *     synchronising.  Return value: 0 on success, <0 on error (B200ASR_* below);
 *     b200asr_last_error() gives a thread-local message.  No C++ exception crosses the ABI.
 *   - `precision`: 0 = fp32 FMA on CUDA cores (exact-order fp32 accumulate); 1 = TF32 tensor cores,
 *     one pass; 3 = 3xTF32 split (fp32-grade).  An unsupported (shape, precision) pair is an
 *     error -- there is no silent fallback of any kind (and no CPU path).
 *   - dropout: `p_drop` in [0,1); decisions come from a counter-based generator keyed by
 *     (seed, offset, element index), so *_bwd regenerates the mask of the matching *_fwd call when it is
 *     given the same (seed, offset).
 */
#ifndef B200ASR_H_
#define B200ASR_H_
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200ASR_OK 0
#define B200ASR_BAD_SHAPE -1
#define B200ASR_BAD_ALIGN -2
#define B200ASR_UNSUPPORTED_ARCH -3
#define B200ASR_CUDA_ERROR -4
#define B200ASR_BAD_ARG -5

#define B200ASR_PREC_FP32 0
#define B200ASR_PREC_TF32 1
#define B200ASR_PREC_TF32X3 3
/* bf16 tensor-core modes (fp32 in HBM, operands converted on the way into the tensor core, fp32 accumulate):
 * BF16 = one bf16 MMA per product (BASELINE.json cfg5 asks for bf16); BF16X3 = 2-term bf16 split x ~ hi + lo (16 significant
 * bits) with hi*hi + hi*lo + lo*hi -- three MMAs at twice the TF32 rate, product error ~2^-17 (between TF32 and 3xTF32). */
#define B200ASR_PREC_BF16 2
#define B200ASR_PREC_BF16X3 6

typedef void* b200asr_stream_t; /* cudaStream_t */

int b200asr_version(void);
const char* b200asr_last_error(void);
/* 0 iff the current device is an sm_90 part (H100).  Called by the loader; everything else assumes it. */
int b200asr_device_check(void);
/* Number of CUDA kernels this library has launched in the process so far (bench.py reports the per-step delta). */
unsigned long long b200asr_launch_count(void);

/* ------------------------------------------------------------------------------------------------
 * Dense layers.  Replaces nn.Linear / nn.Conv1d(k=1) dispatches:
 *   encoder input_linear            models/asr/transformer.py:172
 *   Q/K/V/output projections        models/common_layers.py:181-183,197
 *   position-wise FFN conv_1/conv_2 models/common_layers.py:138   (weights (out,in,1) == (out,in))
 *   decoder output_linear (logits)  models/asr/transformer.py:302
 * y[M,N] = act(x[M,K] * w[N,K]^T + bias[N]);  bias may be NULL; relu != 0 applies max(0, .)
 */
int b200asr_linear_fwd(const float* x, const float* w, const float* bias, float* y, int M, int N, int K,
                       int relu, int precision, const void* w_split, b200asr_stream_t stream);
/* dx[M,K] (+)= (dy[M,N] * w[N,K]) .* (relu_out[M,K] > 0 if relu_out != NULL) */
int b200asr_linear_bwd_data(const float* dy, const float* w, const float* relu_out, float* dx, int M, int N,
                            int K, int accumulate, int precision, const void* w_split, b200asr_stream_t stream);
/* w_split, precision 3 (optional): the weight pre-split for the 3xTF32 path by b200asr_split_tf32 --
 * [2][N][K] fp32 = hi = rn_tf32(w) followed by lo = w - hi.  Passing it removes the per-tile weight split from the GEMM
 * (the forward's split is reused by the backward); NULL keeps the split inside the kernel.
 * w_split, precisions 2 / 6 (REQUIRED): the weight converted to bf16 by b200asr_split_bf16 -- linear_fwd takes `dst`
 * ([terms][N][K], needs K % 8 == 0), linear_bwd_data takes the transposed `dst_t` ([terms][K][N8], N8 = N rounded up to 8). */
int b200asr_split_tf32(const float* src, float* dst_hi_lo, long long n, b200asr_stream_t stream);
/* w [N,K] fp32 -> bf16 operands of the bf16 GEMMs: terms = 1: hi = bf16(w); terms = 2: hi followed by lo = bf16(w - hi).
 * dst [terms][N][K] (K-major for y = x w^T) and/or dst_t [terms][K][N8] (K-major for dx = dy w; zero padded columns);
 * either may be NULL. */
int b200asr_split_bf16(const float* w, void* dst, void* dst_t, int N, int K, int terms, b200asr_stream_t stream);
/* The same conversion for MANY matrices of one flat parameter buffer in a single launch (once per optimizer step):
 * desc [ndesc][6] int64 on the device = {src offset, N, K, terms, dst offset, dst_t offset} in elements (src relative to
 * `base`, dst / dst_t relative to `out`, both orientations are written); tile_prefix [ndesc] int32 = number of 32x32 tiles
 * (ceil(K/32) * ceil(N8/32) each) of the matrices before d; total_tiles = their sum. */
int b200asr_split_bf16_batched(const float* base, void* out, const long long* desc, const int* tile_prefix, int ndesc,
                               int total_tiles, b200asr_stream_t stream);
/* dw[N,K] (+)= dy[M,N]^T * x[M,K];  dbias[N] (+)= column sums of dy (dbias may be NULL) */
int b200asr_linear_bwd_weight(const float* dy, const float* x, float* dw, float* dbias, int M, int N, int K,
                              int accumulate, int precision, b200asr_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * Residual + LayerNorm (+ positional encoding, + non-pad row mask).  Replaces
 *   dropout -> add residual -> LayerNorm   models/common_layers.py:197-198 (MHA), :140-141 (FFN)
 *   `out *= non_pad_mask`                   models/asr/transformer.py:198,201,536,540,543
 *   LayerNorm(Linear(x)) + PE               models/asr/transformer.py:172-173
 * z = dropout(x) + residual ; y = (LN(z)*gamma + beta + post_add[row % post_period]) * row_scale[row]
 * residual, post_add, row_scale, z may be NULL (z NULL: LN input is not saved; valid only when it
 * equals x, i.e. residual == NULL and p_drop == 0).  mean/rstd are [rows].  d % 4 == 0, d <= 1024.
 */
int b200asr_add_ln_fwd(const float* x, const float* residual, const float* gamma, const float* beta,
                       const float* post_add, int post_period, const float* row_scale, float* y, float* z,
                       float* mean, float* rstd, int rows, int d, float eps, float p_drop, uint64_t seed,
                       uint64_t offset, b200asr_stream_t stream);
/* dz = grad wrt LN input (== grad wrt residual); dx = grad wrt x (dz through the dropout mask; pass
 * dx == dz when p_drop == 0).  dgamma/dbeta are overwritten, or added to when accumulate != 0 (the host passes the
 * parameters' existing .grad views of the flat gradient buffer).  partial_ws: b200asr_add_ln_bwd_ws_bytes. */
int b200asr_add_ln_bwd(const float* dy, const float* z, const float* gamma, const float* mean,
                       const float* rstd, const float* row_scale, float* dz, float* dx, float* dgamma,
                       float* dbeta, void* partial_ws, int rows, int d, float p_drop, uint64_t seed,
                       uint64_t offset, int accumulate, b200asr_stream_t stream);
size_t b200asr_add_ln_bwd_ws_bytes(int rows, int d);

/* ------------------------------------------------------------------------------------------------
 * Scaled dot-product attention, fused (scores never reach HBM).  Replaces
 *   bmm -> /temperature -> masked_fill(-inf) -> softmax(dim=2) -> dropout -> bmm
 *   models/common_layers.py:215-223, and the head split/merge copies at :185-187,:194-195 through strides.
 * Element (b,h,t,c) of q lives at q[b*q_bs + h*q_hs + t*q_rs + c] (likewise k, v, out, and their grads).
 * key_pad   [B,Tk]     1 = key is padding for every query of that utterance (NULL = none)
 * dense_mask[B,Tq,Tk]  1 = masked (the reference's generic mask, broadcast over heads; NULL = none)
 * causal != 0 masks k > q (models/common_layers.py:66-74).  lse is [B,H,Tq] (log-sum-exp of the scaled,
 * masked scores).  A fully-masked row yields NaN exactly like the reference's softmax.
 * dk, dv in {16,32,64,128}.
 */
int b200asr_sdpa_fwd(const float* q, const float* k, const float* v, long long q_bs, long long q_hs,
                     long long q_rs, long long k_bs, long long k_hs, long long k_rs, long long v_bs,
                     long long v_hs, long long v_rs, const uint8_t* key_pad, const uint8_t* dense_mask,
                     int causal, float* out, long long o_bs, long long o_hs, long long o_rs, float* lse, int B,
                     int H, int Tq, int Tk, int dk, int dv, float scale, float p_drop, uint64_t seed,
                     uint64_t offset, int precision, b200asr_stream_t stream);
/* dq/dk/dv use the strides of q/k/v; they are overwritten.  delta_ws: [B,H,Tq] floats of scratch. */
int b200asr_sdpa_bwd(const float* dout, const float* q, const float* k, const float* v, const float* out,
                     const float* lse, long long q_bs, long long q_hs, long long q_rs, long long k_bs,
                     long long k_hs, long long k_rs, long long v_bs, long long v_hs, long long v_rs,
                     long long o_bs, long long o_hs, long long o_rs, const uint8_t* key_pad,
                     const uint8_t* dense_mask, int causal, float* dq, float* dk_out, float* dv_out,
                     float* delta_ws, int B, int H, int Tq, int Tk, int dk, int dv, float scale, float p_drop,
                     uint64_t seed, uint64_t offset, int precision, b200asr_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * Fused attention at fp32 grade (opt-in): ScaledDotProductAttention.forward, models/common_layers.py:211-225,
 * as ONE forward kernel (QK^T and PV on the tensor cores with the 2-term bf16 split, masks + softmax + dropout on the
 * score fragments in registers) and TWO backward kernels that recompute the probabilities from Q, K and the forward's
 * log-sum-exp.  Same view / mask / dropout conventions as b200asr_sdpa_fwd.  Needs dk = dv = 64 and (forward) Tk <= 448.
 * ws16: b200asr_sdpa_fused_ws_bytes(B,H,Tq,Tk) bytes of workspace the caller keeps from the forward to the backward (the
 * current kernels split the fp32 operands as they load them and leave it unused).  ws_bwd:
 * b200asr_sdpa_fused_bwd_ws_bytes(B,H,Tq) bytes of scratch.
 */
size_t b200asr_sdpa_fused_ws_bytes(int B, int H, int Tq, int Tk);
size_t b200asr_sdpa_fused_bwd_ws_bytes(int B, int H, int Tq);
int b200asr_sdpa_fused_fwd(const float* q, const float* k, const float* v, long long q_bs, long long q_hs, long long q_rs,
                           long long k_bs, long long k_hs, long long k_rs, long long v_bs, long long v_hs, long long v_rs,
                           const uint8_t* key_pad, const uint8_t* dense_mask, int causal, float* out, long long o_bs,
                           long long o_hs, long long o_rs, float* lse, void* ws16, int B, int H, int Tq, int Tk, int dk,
                           int dv, float scale, float p_drop, uint64_t seed, uint64_t offset, b200asr_stream_t stream);
int b200asr_sdpa_fused_bwd(const float* dout, const float* q, const float* k, const float* v, const float* out,
                           const float* lse, long long q_bs, long long q_hs, long long q_rs, long long k_bs,
                           long long k_hs, long long k_rs, long long v_bs, long long v_hs, long long v_rs, long long o_bs,
                           long long o_hs, long long o_rs, const uint8_t* key_pad, const uint8_t* dense_mask, int causal,
                           float* dq, float* dk_out, float* dv_out, const void* ws16, void* ws_bwd, int B, int H, int Tq,
                           int Tk, int dk, int dv, float scale, float p_drop, uint64_t seed, uint64_t offset,
                           b200asr_stream_t stream);

/* Materialised attention (precision 1 = TF32, 3 = 3xTF32): the same contract as b200asr_sdpa_fwd/_bwd
 * (models/common_layers.py:211-225; head views addressed by strides; dropout drawn from the same counter stream, so
 * both paths produce identical masks), computed op for op like the reference -- bmm, masked softmax, dropout, bmm --
 * with the bmm's as batched tensor-core GEMMs and the softmax (and its backward) as exact fp32 row kernels.
 * probs / probs_drop / dp_ws: caller-owned [B,H,Tq,round_up(Tk,4)] float buffers of b200asr_sdpa_mat_ws_bytes bytes;
 * probs (softmax output) and, when p_drop > 0, probs_drop (after dropout) must be kept for the backward call;
 * probs_drop may be NULL when p_drop == 0.  dk, dv multiples of 32; Tk <= 2048. */
size_t b200asr_sdpa_mat_ws_bytes(int B, int H, int Tq, int Tk);
int b200asr_sdpa_mat_fwd(const float* q, const float* k, const float* v, long long q_bs, long long q_hs,
                         long long q_rs, long long k_bs, long long k_hs, long long k_rs, long long v_bs,
                         long long v_hs, long long v_rs, const uint8_t* key_pad, const uint8_t* dense_mask,
                         int causal, float* out, long long o_bs, long long o_hs, long long o_rs, float* probs,
                         float* probs_drop, int B, int H, int Tq, int Tk, int dk, int dv, float scale,
                         float p_drop, uint64_t seed, uint64_t offset, int precision, b200asr_stream_t stream);
/* dq/dk/dv use the strides of q/k/v and are overwritten; dout uses the strides of out */
int b200asr_sdpa_mat_bwd(const float* dout, const float* q, const float* k, const float* v, long long q_bs,
                         long long q_hs, long long q_rs, long long k_bs, long long k_hs, long long k_rs,
                         long long v_bs, long long v_hs, long long v_rs, long long o_bs, long long o_hs,
                         long long o_rs, const float* probs, const float* probs_drop, float* dq, float* dk_out,
                         float* dv_out, float* dp_ws, int B, int H, int Tq, int Tk, int dk, int dv, float scale,
                         float p_drop, uint64_t seed, uint64_t offset, int precision, b200asr_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * VGG front end (models/asr/transformer.py:42-53).  Activations are kept channels-last with time as the
 * outer spatial axis, [B,T,F,C], so the flatten/transpose of :74-76 becomes a free view [B*T, F*C]
 * (feature index f*C+c; the host permutes input_linear's columns once per step instead).
 * Weights keep the reference layout [Co,Ci,3(freq),3(time)].
 */
/* x [B,F,T] (the reference's (B,1,F,T) input as is) -> y [B,T,F,Co], bias + optional ReLU fused */
int b200asr_conv3x3_c1_fwd(const float* x, const float* w, const float* bias, float* y, int B, int F, int T,
                           int Co, int relu, b200asr_stream_t stream);
/* dw[Co,1,3,3], dbias[Co] overwritten; dy is [B,T,F,Co] (already masked by the ReLU derivative) */
int b200asr_conv3x3_c1_bwd_weight(const float* x, const float* dy, float* dw, float* dbias, int B, int F,
                                  int T, int Co, b200asr_stream_t stream);
/* x [B,T,F,Ci] -> y [B,T,F,Co]; ws: b200asr_conv3x3_ws_bytes(Ci,Co) */
int b200asr_conv3x3_fwd(const float* x, const float* w, const float* bias, float* y, void* ws, int B, int T,
                        int F, int Ci, int Co, int relu, int precision, b200asr_stream_t stream);
/* The same convolution followed by MaxPool2d(2, stride 2) (models/asr/transformer.py:44-52: conv, ReLU, pool): y as above AND
 * pooled [B,T/2,F/2,Co] (floor mode).  In the bf16 modes the 2x2 maximum is taken in the convolution's epilogue (four
 * lanes of a warp hold a window), so the activation is not read back; other precisions run the two kernels.
 * pool_idx (optional) [B,T/2,F/2,Co] bytes: which element of each window holds the maximum (ATen's scan order, first maximum;
 * bit 2 set when the maximum is not positive) -- what b200asr_maxpool2x2_bwd_idx routes the gradient by; asking for it runs
 * the stand-alone pooling kernel after the convolution (computing the bytes in the epilogue was measured to cost more than the
 * index-based backward saves). */
int b200asr_conv3x3_fwd_pool(const float* x, const float* w, const float* bias, float* y, float* pooled,
                             unsigned char* pool_idx, void* ws, int B, int T, int F, int Ci, int Co, int relu, int precision,
                             b200asr_stream_t stream);
/* dx[B,T,F,Ci] = conv_transpose(dy) .* (relu_out > 0 if relu_out != NULL).
 * dx16 (optional, precisions 6 / 2 only): the same gradient additionally as bf16 hi | lo "pairs" [2][B,T,F,Ci] (hi = bf16(v),
 * lo = bf16(v - hi)) -- what b200asr_conv3x3_bwd_weight of the layer below takes as dy16. */
int b200asr_conv3x3_bwd_data(const float* dy, const float* w, const float* relu_out, float* dx, void* dx16, void* ws,
                             int B, int T, int F, int Ci, int Co, int precision, b200asr_stream_t stream);
/* dw[Co,Ci,3,3], dbias[Co] overwritten.  dy16 (optional, precisions 6 / 2): dy as bf16 pairs [2][B,T,F,Co] written by its
 * producer (b200asr_maxpool2x2_bwd / b200asr_conv3x3_bwd_data): the kernel then takes its B tiles straight from there by TMA
 * instead of converting the fp32 dy tile (the in-kernel conversion is what bounds the bf16 weight gradient). */
int b200asr_conv3x3_bwd_weight(const float* dy, const void* dy16, const float* x, float* dw, float* dbias, void* ws,
                               int B, int T, int F, int Ci, int Co, int precision, b200asr_stream_t stream);
size_t b200asr_conv3x3_ws_bytes(int Ci, int Co);
/* MaxPool2d(2, stride 2), floor mode: [B,T,F,C] -> [B,T/2,F/2,C] */
int b200asr_maxpool2x2_fwd(const float* x, float* y, int B, int T, int F, int C, b200asr_stream_t stream);
/* the same pooling, additionally writing the index bytes described at b200asr_conv3x3_fwd_pool */
int b200asr_maxpool2x2_fwd_idx(const float* x, float* y, unsigned char* idx, int B, int T, int F, int C,
                               b200asr_stream_t stream);
/* dx[B,T,F,C] = route dy to the first maximum of each window (scan order freq-major, as ATen), then
 * .* (x > 0) when relu_mask != 0 (x is the post-ReLU pool input). */
int b200asr_maxpool2x2_bwd(const float* dy, const float* x, float* dx, void* dx16 /* optional bf16 pairs [2][B,T,F,C] */, int B, int T, int F, int C,
                           int relu_mask, b200asr_stream_t stream);
/* b200asr_maxpool2x2_bwd from the forward's index bytes instead of the activation (reads 1 byte instead of 16 per pooled
 * element): identical result.  relu_mask != 0: a window whose maximum is not positive passes no gradient. */
int b200asr_maxpool2x2_bwd_idx(const float* dy, const unsigned char* idx, float* dx, void* dx16, int B, int T, int F, int C,
                               int relu_mask, b200asr_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * emb_cnn front end (models/asr/transformer.py:33-40): generic strided NCHW convolution, BatchNorm2d
 * (train: batch statistics + running-state update; eval: running statistics) fused with Hardtanh(lo,hi), and the (B,C,F,T)->(B,T,C*F)
 * flatten of :74-76.
 */
int b200asr_conv2d_fwd(const float* x, const float* w, const float* bias, float* y, int B, int Ci, int H,
                       int W, int Co, int KH, int KW, int SH, int SW, int PH, int PW, b200asr_stream_t stream);
int b200asr_conv2d_bwd_data(const float* dy, const float* w, float* dx, int B, int Ci, int H, int W, int Co,
                            int KH, int KW, int SH, int SW, int PH, int PW, b200asr_stream_t stream);
int b200asr_conv2d_bwd_weight(const float* dy, const float* x, float* dw, float* dbias, int B, int Ci, int H,
                              int W, int Co, int KH, int KW, int SH, int SW, int PH, int PW,
                              b200asr_stream_t stream);
/* y = clamp(BN(x), lo, hi); x,y [B,C,H,W] with a row pitch each (floats, >= W; dense tensors pass W); mean/invstd [C] are
 * outputs (the statistics used: saved for backward).
 * training != 0: batch statistics (biased variance, as ATen) and, if the buffers are given, the nn.BatchNorm2d state
 * update running_mean/var <- (1-momentum) old + momentum new (unbiased variance), num_batches_tracked (int64) += 1.
 * training == 0 (model.eval(), trainer.py:123): normalise with running_mean / running_var.
 * Each call is two launches over a (splits x C) grid -- per-block partial statistics, then merge + apply --; ws holds the
 * partials: b200asr_bn_ws_bytes(C) bytes. */
size_t b200asr_bn_ws_bytes(int C);
int b200asr_bn_clamp_fwd(const float* x, const float* gamma, const float* beta, float* y, float* mean,
                         float* invstd, float* running_mean, float* running_var, long long* num_batches_tracked,
                         float* ws, int B, int C, int H, int W, int x_pitch, int y_pitch, float eps, float momentum,
                         int training, float lo, float hi, b200asr_stream_t stream);
int b200asr_bn_clamp_bwd(const float* dy, const float* x, const float* y, const float* gamma,
                         const float* mean, const float* invstd, float* dx, float* dgamma, float* dbeta, float* ws,
                         int B, int C, int H, int W, int dy_pitch, int x_pitch, int y_pitch, int dx_pitch, int training,
                         float lo, float hi, b200asr_stream_t stream);
/* The second emb_cnn convolution (models/asr/transformer.py:37, Conv2d(32, 32, (KH, KW), stride (SH, 1)), no padding) as
 * implicit GEMMs on the tensor cores -- no im2col matrix.  x / dx [B,32,H,W] with row pitch x_pitch, y / dy [B,32,OH,OW] with row
 * pitch y_pitch (floats, multiples of 4: TMA); w [32,32,KH,KW].  precision 6 (bf16x3), 3 (3xTF32) or 2 (bf16) for forward
 * and data gradient; the weight gradient runs 3xTF32, one partial per row split, summed in split order.
 * ws: b200asr_conv2d_tc_ws_bytes(B, H, W, KH, KW) bytes -- the repacked weight slices, and four copies of the tensor whose
 * windows slide (x, or dy for the data gradient) shifted by 0..3 floats, because a TMA box must start on a 16-byte
 * boundary; each call rebuilds what it needs (one HBM-bound pass), so the same buffer may serve all three. */
size_t b200asr_conv2d_tc_ws_bytes(int B, int H, int W, int KH, int KW);
int b200asr_conv2d_tc_fwd(const float* x, const float* w, const float* bias, float* y, void* ws, int B, int Ci, int H,
                          int W, int Co, int KH, int KW, int SH, int x_pitch, int y_pitch, int precision,
                          b200asr_stream_t stream);
int b200asr_conv2d_tc_bwd_data(const float* dy, const float* w, float* dx, void* ws, int B, int Ci, int H, int W, int Co,
                               int KH, int KW, int SH, int x_pitch, int y_pitch, int precision,
                               b200asr_stream_t stream);
int b200asr_conv2d_tc_bwd_weight(const float* dy, const float* x, float* dw, float* dbias, void* ws, int B, int Ci, int H,
                                 int W, int Co, int KH, int KW, int SH, int x_pitch, int y_pitch,
                                 b200asr_stream_t stream);
/* The FIRST emb_cnn convolution (models/asr/transformer.py:33, Conv2d(1, 32, (KH, KW), stride (2, 2), padding (0, PW))) on the
 * same engine: the KH taps along H play the role of input channels (an overlapping tensor-map view of the activation), the
 * stride along W is removed by de-interleaving x into parity copies (x 4 alignments, see above).  x [B,1,H,W] dense;
 * y / dy [B,32,OH,OW] with row pitch y_pitch (any value >= OW for the forward, a multiple of 4 for the weight gradient: TMA).
 * No data gradient (the input is data).  ws: b200asr_conv2d_c1_tc_ws_bytes(B, H, W, KH, KW) bytes. */
size_t b200asr_conv2d_c1_tc_ws_bytes(int B, int H, int W, int KH, int KW);
int b200asr_conv2d_c1_tc_fwd(const float* x, const float* w, const float* bias, float* y, void* ws, int B, int H, int W,
                             int Co, int KH, int KW, int PW, int y_pitch, int precision, b200asr_stream_t stream);
int b200asr_conv2d_c1_tc_bwd_weight(const float* dy, const float* x, float* dw, float* dbias, void* ws, int B, int H,
                                    int W, int Co, int KH, int KW, int PW, int y_pitch, b200asr_stream_t stream);
/* x [B,C,F,T] -> y [B,T,C*F] and its inverse (gradient) */
int b200asr_flatten_bcft_fwd(const float* x, float* y, int B, int C, int F, int T, b200asr_stream_t stream);
int b200asr_flatten_bcft_bwd(const float* dy, float* dx, int B, int C, int F, int T, b200asr_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * Decoder input side.
 *   Decoder.preprocess + pad_list          models/asr/transformer.py:254-266, common_layers.py:14-22
 *   non-pad / key-pad masks (== EOS)       models/asr/transformer.py:282-285
 *   dropout(Embedding(seq_in)*scale + PE)  models/asr/transformer.py:292-293
 * padded_target [B,L] (0-padded).  Outputs, all [B,Tt]: seq_in (SOS,y..,EOS pad), seq_out (y..,EOS,PAD
 * pad), key_pad (seq_in == EOS), non_pad (float 1/0).  status[0] (device int) is set to 1 if some
 * utterance needs more than Tt positions (the reference raises in pad_list).
 */
int b200asr_preprocess_targets(const int64_t* padded_target, int L, int64_t* seq_in, int64_t* seq_out,
                               uint8_t* key_pad, float* non_pad, int* status, int B, int Tt,
                               b200asr_stream_t stream);
int b200asr_embed_fwd(const int64_t* tokens, const float* table, const float* pe, float* out, int rows, int T,
                      int d, int V, float scale, float p_drop, uint64_t seed, uint64_t offset,
                      b200asr_stream_t stream);
/* dtable[V,d] += scatter(dout) (caller zeroes dtable); rows with token == pad_idx contribute nothing */
int b200asr_embed_bwd(const int64_t* tokens, const float* dout, float* dtable, int rows, int d, int V,
                      float scale, float p_drop, uint64_t seed, uint64_t offset, int pad_idx,
                      b200asr_stream_t stream);
/* length masks of models/common_layers.py:28-44,57-64: key_pad[b,t] = (t >= lengths[b]), non_pad = 1-that */
int b200asr_length_masks(const int32_t* lengths, uint8_t* key_pad, float* non_pad, int B, int T,
                         b200asr_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * Output side.
 *   topk(pred,1)                       models/asr/transformer.py:80-82
 *   label-smoothed CE / CE / num_correct   utils/metrics.py:115-132, 88-94
 * stats (device, 5 floats; [3],[4] filled by b200asr_ce_finalize): [0] = sum over non-PAD rows of the row loss, [1] = number of non-PAD rows,
 * [2] = number of correct argmax among them.  stats[0..2] are overwritten.  row_lse is [rows].
 */
int b200asr_argmax_rows(const float* logits, int64_t* out, int rows, int V, b200asr_stream_t stream);
/* One step of Decoder.greedy_search (models/asr/transformer.py:375-382) with the EOS cut of :385-393 kept on the device:
 * next_tok[b] = argmax(logits[b,:]) (first max); ys[b*steps+t] = that id, or -1 from the utterance's first EOS on;
 * finished[b] / *n_finished (int32, zero-initialised by the caller) record which utterances have emitted EOS so the host
 * loop can stop early (SURVEY.md 8f row 3: on-device EOS stop). */
int b200asr_greedy_step(const float* logits, int64_t* next_tok, int64_t* ys, int* finished, int* n_finished, int B, int V,
                        int t, int steps, b200asr_stream_t stream);
int b200asr_ce_fwd(const float* logits, const int64_t* gold, float* row_lse, float* stats, int rows, int V,
                   float smoothing, b200asr_stream_t stream);
/* stats[3] = stats[0] / stats[1] (the reference's mean loss), stats[4] = 1 / stats[1];
 * loss_out[0] = mean ? stats[3] : stats[0].  stats therefore holds 5 floats. */
int b200asr_ce_finalize(float* stats, float* loss_out, int mean, b200asr_stream_t stream);
/* dlogits = gscale * (*gscale_dev) * (*gscale_dev2) * d(sum of row losses)/dlogits (NULL factors = 1);
 * PAD rows get 0 */
int b200asr_ce_bwd(const float* logits, const int64_t* gold, const float* row_lse, float* dlogits, int rows,
                   int V, float smoothing, float gscale, const float* gscale_dev, const float* gscale_dev2,
                   b200asr_stream_t stream);

/* GEMM formulation of the emb_cnn convolutions (default for precision != 0): col[(b,oh,ow)][(ci,kh,kw)] with row pitch Kp
 * (>= Ci*KH*KW, zero padded; multiple of 4 for the tensor-core GEMM), so that conv = b200asr_linear_fwd(col, w[Co][K]),
 * weight gradient = b200asr_linear_bwd_weight, data gradient = b200asr_linear_bwd_data followed by col2im (the adjoint
 * scatter; dx is zeroed inside).  transpose_cp converts [B][C][P] <-> [B][P][C] (to_pc != 0: C-major -> pixel-major). */
int b200asr_im2col(const float* x, float* col, int B, int Ci, int H, int W, int KH, int KW, int SH, int SW, int PH,
                   int PW, int Kp, b200asr_stream_t stream);
int b200asr_col2im(const float* dcol, float* dx, int B, int Ci, int H, int W, int KH, int KW, int SH, int SW, int PH,
                   int PW, int Kp, b200asr_stream_t stream);
int b200asr_transpose_cp(const float* src, float* dst, int B, int C, int P, int to_pc, b200asr_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * Step tail ("next" row of SURVEY.md §8f): Adam(betas, eps) with the learning rate supplied by the host
 * (NoamOpt, utils/optimizer.py:15-32; torch.optim.Adam at utils/functions.py:107) over a flat buffer.
 * g is read as g * gscale * (*gscale_dev if non-NULL) -- e.g. 1/global num_word and the clip coefficient.
 */
int b200asr_adam_step(float* p, const float* g, float* m, float* v, long long n, float lr, float beta1,
                      float beta2, float eps, int step, float gscale, const float* gscale_dev,
                      b200asr_stream_t stream);
/* out[0] += sum(g^2) (caller zeroes out) */
int b200asr_sumsq(const float* g, long long n, float* out, b200asr_stream_t stream);
/* Device-side gradient scale of the step tail: out[0] = (1 / *n_tokens) * clip, where clip = 1 if max_norm <= 0, else
 * min(1, max_norm / (||g||_2 / *n_tokens + 1e-6)) -- torch.nn.utils.clip_grad_norm_ (trainer/asr/trainer.py:108-109) on the
 * token-normalised gradient; out[1] = that norm (0 without clipping).  scratch: 1 float.  No host synchronisation. */
int b200asr_grad_scale(const float* g, long long n, const float* n_tokens, float max_norm, float* scratch, float* out,
                       b200asr_stream_t stream);
/* dst = src permuted: dst[r, f*C + c] = src[r, c*F + f] (input_linear column order, see VGG note);
 * inverse != 0 applies the inverse permutation. */
int b200asr_permute_cols_cf(const float* src, float* dst, int rows, int C, int F, int inverse,
                            b200asr_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * Feature front end ("next" row 4 of SURVEY.md §8f): SpectrogramParser.parse_audio (utils/data_loader.py:60-91)
 * + the padded batch layout of _collate_fn (:182-214).  wave [B,Lmax] fp32 zero padded, lens [B] samples.
 * STFT with n_fft-sample Hamming frames (symmetric window, as the reference's callable scipy.signal.hamming gives
 * through librosa; window_periodic != 0 selects the periodic variant) every hop samples, centred (n_fft/2 padding on both sides,
 * reflected when pad_reflect != 0, zeros otherwise), magnitude, log1p, optional per-utterance mean / unbiased-std
 * normalisation -> out [B,1,n_fft/2+1,Tmax] zero padded; frames_out[b] = 1 + lens[b]/hop (may be NULL).
 * The STFT of the whole batch is ONE GEMM over overlapping frame rows (precision as for b200asr_linear_fwd).
 * ws: b200asr_stft_ws_bytes(B, Lmax, n_fft, hop) bytes.  n_fft % 32 == 0, hop % 4 == 0. */
size_t b200asr_stft_ws_bytes(int B, int Lmax, int n_fft, int hop);
int b200asr_stft_features(const float* wave, const int* lens, float* out, int* frames_out, void* ws, int B,
                          int Lmax, int Tmax, int n_fft, int hop, int pad_reflect, int normalize, int window_periodic,
                          int precision, b200asr_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* B200ASR_H_ */
