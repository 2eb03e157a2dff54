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
 *     inputs give the same bits every run (the fp32 CUDA-core GEMM / convolution / attention backward variants still
 *     accumulate with atomics).
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
 *
 * All three entry points take M >= 0, N > 0, K > 0 and non-NULL x / dy / w / y / dx / dw (bias, relu_out and dbias may be
 * NULL); otherwise, or for a precision other than 0, 1, 3, 2, 6, they return B200ASR_BAD_ARG.
 *   precision 0 (fp32 CUDA cores): any N and K, any 4-byte aligned pointers (16-byte alignment and dimensions that are
 *     multiples of 4 only select vector loads).  Its split-K weight gradient (contraction M >= 1024 and fewer output tiles
 *     than SMs) adds the splits with atomics, so the bits of dw may differ from call to call there.
 *   precisions 1, 3 (TF32 / 3xTF32 tensor cores): the operands the GEMM reads by TMA must be 16-byte aligned with row
 *     pitches that are multiples of 4 floats -- x, w and K for the forward; dy, w, N and K for the data gradient; dy, x, N
 *     and K for the weight gradient -- otherwise B200ASR_BAD_SHAPE.  The forward's N, bias, relu_out and the outputs
 *     have no such rule (they take a scalar epilogue).
 *   precisions 2, 6 (bf16 / bf16x3): w_split is required (see below), otherwise B200ASR_BAD_SHAPE; the weight gradient
 *     has the rules of precision 3.
 * A rejected call launches nothing and writes nothing.
 * M = 0 (an empty batch, pointers still valid): the forward and the data gradient write nothing; the weight gradient sets
 * dw and dbias to 0, or leaves them unchanged when accumulating.  Same at every precision; nothing is launched.
 * Kernel launches per call (b200asr_launch_count): forward and data gradient 1; at precisions 1 and 3, 2 when the
 * contraction is split (no ReLU and no mask, K >= 1024, at most half as many 128 x 128 output tiles as SMs): the GEMM and
 * the reduction of its partial tiles, which adds the bias.  Weight gradient: precision 0: 1, + 2 with dbias (column sums
 * and their reduction); precision 1: 1 or 2 split, + 2 with dbias; precisions 3, 2, 6: 1 unsplit, 2 split, + 1 with dbias
 * when split (the bias gradient is fused into the GEMM; its split partials need a reduction).
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
 * masked scores).  A fully-masked row yields NaN exactly like the reference's softmax: that row of out and lse
 * are NaN; in the backward its dq row is 0, dk stays finite and dv is NaN for every key of that (b, h).
 * dk, dv in {16,32,64,128} (precision 0: every pair, forward and backward).
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

/* Attention probabilities of a flash forward (b200asr_sdpa_fwd at precision 0 or 1, b200asr_sdpa_fused_fwd = precision 6),
 * which keeps only the log-sum-exp: ScaledDotProductAttention.forward's `attn` (models/common_layers.py:217-221).  From the
 * forward's q, k, masks, lse, scale and (p_drop, seed, offset), recomputes the scores at that forward's precision and writes
 * P[b,h,t,j] = exp(scale * S - lse[b,h,t]), times the forward's dropout keep / (1 - p) when p_drop > 0, to
 * probs[b*p_bs + h*p_hs + t*p_rs + j] for j < Tk (any strides; nothing else is written).  Masked keys are 0 and a fully
 * masked row (lse NaN) is NaN.  Shapes: precision 0 dk in {16,32,64,128}, any Tk; precision 1 dk in {32,64}, Tk <= 448;
 * precision 6 dk = 64, Tk <= 448.  Any other (shape, precision) pair returns B200ASR_BAD_SHAPE and launches nothing.
 * q / k strides and alignment as b200asr_sdpa_fwd; probs 4-byte aligned. */
int b200asr_sdpa_probs(const float* q, const float* k, long long q_bs, long long q_hs, long long q_rs, long long k_bs,
                       long long k_hs, long long k_rs, const uint8_t* key_pad, const uint8_t* dense_mask, int causal,
                       const float* lse, float* probs, long long p_bs, long long p_hs, long long p_rs, int B, int H, int Tq,
                       int Tk, int dk, float scale, float p_drop, uint64_t seed, uint64_t offset, int precision,
                       b200asr_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * VGG front end (models/asr/transformer.py:42-53).  Activations are kept channels-last with time as the
 * outer spatial axis, [B,T,F,C], so the flatten/transpose of :74-76 becomes a free view [B*T, F*C]
 * (feature index f*C+c; the host permutes input_linear's columns once per step instead).
 * Weights keep the reference layout [Co,Ci,3(freq),3(time)].
 * Alignment: a pointer the kernels move in vectors must be aligned to the vector -- 16 bytes for the float tensors named
 * below, 4 bytes for pooling index bytes, 8 bytes for bf16 pairs; otherwise the call returns B200ASR_BAD_ALIGN and writes
 * nothing.  Fresh allocations always qualify; a view offset by a few floats may not.
 */
/* x [B,F,T] (the reference's (B,1,F,T) input as is) -> y [B,T,F,Co], bias + optional ReLU fused.  Co % 4 == 0, Co <= 1024,
 * 256 % (Co/4) == 0.  y 16-byte aligned. */
int b200asr_conv3x3_c1_fwd(const float* x, const float* w, const float* bias, float* y, int B, int F, int T,
                           int Co, int relu, b200asr_stream_t stream);
/* dw[Co,1,3,3], dbias[Co] overwritten; dy is [B,T,F,Co] (already masked by the ReLU derivative), 16-byte aligned */
int b200asr_conv3x3_c1_bwd_weight(const float* x, const float* dy, float* dw, float* dbias, int B, int F,
                                  int T, int Co, b200asr_stream_t stream);
/* x [B,T,F,Ci] -> y [B,T,F,Co]; ws: b200asr_conv3x3_ws_bytes(Ci,Co).  Precision 0: x, y and ws 16-byte aligned. */
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
 * lo = bf16(v - hi)) -- what b200asr_conv3x3_bwd_weight of the layer below takes as dy16.
 * Precision 0: dy, relu_out, dx and ws 16-byte aligned. */
int b200asr_conv3x3_bwd_data(const float* dy, const float* w, const float* relu_out, float* dx, void* dx16, void* ws,
                             int B, int T, int F, int Ci, int Co, int precision, b200asr_stream_t stream);
/* ReLU decisions as packed bits (models/asr/transformer.py:44-52: the ReLUs after conv1 and conv3, whose outputs the backward
 * needs only as "> 0" to mask the data gradient of the next convolution): uint32 [B,T,F,C/32], bit c % 32 of word c / 32 =
 * (y > 0) for channel c -- exactly the test the data gradient applies to relu_out (-0.0 and NaN give 0).  1/32 of the bytes of
 * the fp32 activation.  Pointers to bits need 4-byte alignment; otherwise B200ASR_BAD_ALIGN.
 * b200asr_conv3x3_c1_fwd / b200asr_conv3x3_fwd that additionally write y_bits (required; Co % 32 == 0): the epilogue gathers
 * them at every precision but 0, where one more kernel packs them from y. */
int b200asr_conv3x3_c1_fwd_bits(const float* x, const float* w, const float* bias, float* y, int B, int F, int T, int Co,
                                int relu, uint32_t* y_bits, b200asr_stream_t stream);
int b200asr_conv3x3_fwd_bits(const float* x, const float* w, const float* bias, float* y, void* ws, int B, int T, int F, int Ci,
                             int Co, int relu, int precision, uint32_t* y_bits, b200asr_stream_t stream);
/* b200asr_conv3x3_bwd_data with the mask given as relu_bits [B,T,F,Ci/32] (required) instead of relu_out: the same bits of dx
 * and dx16 at every precision, reading 1 bit instead of 4 bytes per element. */
int b200asr_conv3x3_bwd_data_bits(const float* dy, const float* w, const uint32_t* relu_bits, float* dx, void* dx16, void* ws,
                                  int B, int T, int F, int Ci, int Co, int precision, b200asr_stream_t stream);
/* dw[Co,Ci,3,3], dbias[Co] overwritten.  dy16 (optional, precisions 6 / 2): dy as bf16 pairs [2][B,T,F,Co] written by its
 * producer (b200asr_maxpool2x2_bwd / b200asr_conv3x3_bwd_data): the kernel then takes its B tiles straight from there by TMA
 * instead of converting the fp32 dy tile (the in-kernel conversion is what bounds the bf16 weight gradient).
 * Precision 0: dy and x 16-byte aligned. */
int b200asr_conv3x3_bwd_weight(const float* dy, const void* dy16, const float* x, float* dw, float* dbias, void* ws,
                               int B, int T, int F, int Ci, int Co, int precision, b200asr_stream_t stream);
size_t b200asr_conv3x3_ws_bytes(int Ci, int Co);
/* MaxPool2d(2, stride 2), floor mode: [B,T,F,C] -> [B,T/2,F/2,C].  C % 4 == 0; every float tensor of the four pooling
 * entry points 16-byte aligned, idx 4-byte aligned, dx16 8-byte aligned. */
int b200asr_maxpool2x2_fwd(const float* x, float* y, int B, int T, int F, int C, b200asr_stream_t stream);
/* the same pooling, additionally writing the index bytes described at b200asr_conv3x3_fwd_pool */
int b200asr_maxpool2x2_fwd_idx(const float* x, float* y, unsigned char* idx, int B, int T, int F, int C,
                               b200asr_stream_t stream);
/* dx[B,T,F,C] = route dy to the first maximum of each window (scan order freq-major, as ATen), then
 * .* (x > 0) when relu_mask != 0 (x is the post-ReLU pool input).  Rows / columns no window covers (odd T or F) get 0. */
int b200asr_maxpool2x2_bwd(const float* dy, const float* x, float* dx, void* dx16 /* optional bf16 pairs [2][B,T,F,C] */, int B, int T, int F, int C,
                           int relu_mask, b200asr_stream_t stream);
/* b200asr_maxpool2x2_bwd from the forward's index bytes instead of the activation (reads 1 byte instead of 16 per pooled
 * element): identical result.  relu_mask != 0: a window whose maximum is not positive passes no gradient. */
int b200asr_maxpool2x2_bwd_idx(const float* dy, const unsigned char* idx, float* dx, void* dx16, int B, int T, int F, int C,
                               int relu_mask, b200asr_stream_t stream);
/* Pooling decisions as packed codes (models/asr/transformer.py:44-52, the two MaxPool2d(2, 2) after a ReLU, whose input the
 * backward needs only to route the gradient): uint32 [B,T/2,F/2,C/8], nibble c % 8 of word c / 8 = the window position of the
 * first maximum in ATen's scan order (0..3, as the index bytes) | 4 when that maximum is not positive.  1/32 of the bytes of the
 * fp32 pool input.  Needs C % 8 == 0 and pool_codes 4-byte aligned.
 * b200asr_conv3x3_fwd_pool that writes pool_codes (required) next to pooled.  In the bf16 modes the codes come from the
 * convolution's epilogue, and y may be NULL: the full-resolution output is then not written at all.  Other precisions run the
 * stand-alone pooling kernel on y, which must be given. */
int b200asr_conv3x3_fwd_pool_codes(const float* x, const float* w, const float* bias, float* y, float* pooled, uint32_t* pool_codes,
                                   void* ws, int B, int T, int F, int Ci, int Co, int relu, int precision, b200asr_stream_t stream);
/* b200asr_maxpool2x2_bwd from those codes instead of the activation: with relu_mask != 0 the same dx and dx16 bits as
 * b200asr_maxpool2x2_bwd(dy, x, ..., relu_mask = 1) for the pool input x the codes were taken from. */
int b200asr_maxpool2x2_bwd_codes(const float* dy, const uint32_t* codes, float* dx, void* dx16, int B, int T, int F, int C,
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
 * boundary; each call rebuilds what it needs (one HBM-bound pass), so the same buffer may serve all three.
 * Returns B200ASR_BAD_SHAPE for Ci or Co != 32, H < KH, W < KW, a non-positive B / KH / KW / SH, or a row pitch that is not
 * a multiple of 4 or smaller than its row (W, OW); B200ASR_BAD_ARG for a NULL x / dy / w / y / dx / dw / ws (bias and dbias
 * may be NULL) or a precision other than 3, 6 or 2; B200ASR_BAD_ALIGN when a tensor read by TMA (x for the forward, dy for
 * the data gradient, both for the weight gradient) or ws is not 16-byte aligned.  A rejected call launches nothing.
 * Launches: forward and data gradient 3 (weight repack, shifted copies, engine); weight gradient 3 (shifted copies, engine,
 * split reduction), 5 with dbias (+ bias partials, their reduction). */
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
 * No data gradient (the input is data).  ws: b200asr_conv2d_c1_tc_ws_bytes(B, H, W, KH, KW) bytes.
 * Returns B200ASR_BAD_SHAPE for Co != 32, KH outside 1..64, H < KH, W + 2 PW < KW, a non-positive B / KW, a negative PW, or
 * a y_pitch smaller than OW (or, for the weight gradient, not a multiple of 4); B200ASR_BAD_ARG for a NULL x / dy / w / y /
 * dw / ws (bias and dbias may be NULL) or a precision other than 3, 6 or 2; B200ASR_BAD_ALIGN when ws, or dy for the weight
 * gradient, is not 16-byte aligned.  A rejected call launches nothing.  Launches: forward 3 (weight repack, de-interleaved
 * copies, engine); weight gradient 3 (copies, engine, split reduction), 5 with dbias. */
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
/* Beam search (Decoder.beam_search without LM rescoring, models/asr/transformer.py:396-517) for B utterances of W slots each;
 * row r = b * W + s.  Replaces, per step t: the log_softmax + topk of every hypothesis (:454-455), the scoring and the
 * stable sorted(...)[:W] pruning (:458-466), the forced EOS at t == T_e - 1 (:471-473), the EOS test, word count and
 * final_score (:476-495) and the ended_hyps list with its final sort (:504-506).
 *   logits [B*W, V] fp32.  word_tab [V]: w * 8 + head * 4 + tail * 2 + empty per token (w = words of the label with the
 *   PAD/SOS/EOS characters removed, head/tail = it starts/ends with a non-space character, empty = nothing is left).
 *   score [B*W] fp32 and state [B*W][4] int32 (live, words, tail, kept index of the slot at the previous step, -1 before
 *   step 0) are read and rewritten: survivors are compacted into slots 0..n-1 in kept order, dead slots get live = 0,
 *   score = -inf.  next_tok [B*W] int64: the next input token (PAD for dead slots).
 *   idx_cur / idx_nxt [B*W][idx_stride] int32 (idx_stride >= t + 2): entry p of a row is the slot of the utterance whose
 *   K/V cache row at step p holds position p of that hypothesis.  idx_nxt rows get the parent's entries 0..t and their own
 *   slot at t + 1; dead rows point at themselves.
 *   hist_tok / hist_par [steps][B*W] int32: row b*W + k of step t holds the k-th kept candidate's token and its parent's kept
 *   index at step t - 1.  pool_score / pool_final [B][nbest] fp32, pool_ref [B][nbest] int32 ((t * W + k) * 2 + forced) and
 *   pool_n [B] (zero-initialised): the top-nbest ended hypotheses by final_score, stable (a later entry never displaces an
 *   equal one).  *n_live (initialised to B) counts the utterances that still have live hypotheses.
 * Scores are fp32 like the reference's; final_score = score + (float)(sqrt(words) * c_weight).  Ties: topk to the lower
 * token id, the merge to the earlier parent, then the better rank.  1 <= W <= 32, W <= V, 1 <= nbest <= 32; otherwise
 * B200ASR_BAD_SHAPE and nothing is written. */
int b200asr_beam_step(const float* logits, const int32_t* word_tab, int B, int W, int V, int t, int t_eos, int steps, int nbest,
                      double c_weight, float* score, int32_t* state, int64_t* next_tok, const int32_t* idx_cur,
                      int32_t* idx_nxt, int idx_stride, int32_t* hist_tok, int32_t* hist_par, float* pool_score,
                      float* pool_final, int32_t* pool_ref, int32_t* pool_n, int32_t* n_live, b200asr_stream_t stream);
/* Single-query self-attention of beam row r over positions 0..t (the reference re-decodes the whole prefix under a causal
 * mask, :444-452; its last position sees every earlier one, so no mask).  q [R, H*dk], out [R, H*dv]; k_cache / v_cache
 * [steps][R][H*dk | H*dv]: position p of row r is read from step p, row (r - r % W) + idx[r * idx_stride + p].  Exact fp32.
 * dk, dv in {16, 32, 64, 128}; t < 8192. */
int b200asr_beam_self_attn(const float* q, const float* k_cache, const float* v_cache, const int32_t* idx, float* out, int R,
                           int H, int W, int dk, int dv, int t, int idx_stride, float scale, b200asr_stream_t stream);
/* Single-query attention of a decode step (csrc/decode.cu): out[r][h*dv ..] = softmax(scale * q_rh . K_rh^T) . V_rh over Tk
 * keys, no mask, exact fp32.  q [R][H*dk] and out [R][H*dv] are contiguous; key j of row r starts at
 * k + r * k_row_stride + j * k_key_stride (elements), head h at column h * dk; V likewise with dv.  So one kernel reads a
 * slab-major K/V cache [steps][B][H*d] (row stride H*d, key stride B*H*d) and a token-major projection [B*T][H*d] (row
 * stride T*H*d, key stride H*d) in place.  The keys of each (row, head) are split into chunks of a length that depends on
 * (R, H, Tk) only; each chunk's partial (max, sum, o) goes to `ws` and a second kernel merges them in chunk order, so
 * repeated calls give identical bits.  ws: b200asr_decode_attn_ws_bytes(R, H, Tk, dv) bytes (0 = one chunk: ws may be
 * NULL, one launch).  dk, dv in {16, 32, 64, 128}; 1 <= Tk <= 65536; strides >= 0 (B200ASR_BAD_SHAPE); k, v 16-byte
 * aligned and every stride a multiple of 4 (B200ASR_BAD_ALIGN).  A rejected call launches nothing. */
size_t b200asr_decode_attn_ws_bytes(int R, int H, int Tk, int dv);
int b200asr_decode_attn(const float* q, const float* k, const float* v, float* out, float* ws, int R, int H, int dk, int dv,
                        int Tk, long long k_row_stride, long long k_key_stride, long long v_row_stride,
                        long long v_key_stride, float scale, b200asr_stream_t stream);
/* The n-best yseqs (:500-515): ids [B][nbest][steps + 2] int64 = SOS, the tokens along hist_par from each pool entry, EOS if
 * it was forced, then -1; lengths [B][nbest] int64 (0: no hypothesis). */
int b200asr_beam_backtrack(const int32_t* hist_tok, const int32_t* hist_par, const int32_t* pool_ref, const int32_t* pool_n,
                           int64_t* ids, int64_t* lengths, int B, int W, int nbest, int steps, b200asr_stream_t stream);
/* Beam search with LM rescoring (lm_rescoring=True, :473-481): b200asr_beam_step plus an end log of EVERY ended hypothesis,
 * since the LM may promote one that the non-LM n-best pool drops.  Per utterance b, in insertion order (step, then kept rank):
 * end_ref[b * end_cap + e] = (t * W + k) * 2 + forced, end_score[...] = its fp32 score; end_n [B] (zero-initialised) counts
 * them.  end_cap >= W * steps.  Everything else is exactly b200asr_beam_step (which is this call without the log). */
int b200asr_beam_step_log(const float* logits, const int32_t* word_tab, int B, int W, int V, int t, int t_eos, int steps,
                          int nbest, double c_weight, float* score, int32_t* state, int64_t* next_tok, const int32_t* idx_cur,
                          int32_t* idx_nxt, int idx_stride, int32_t* hist_tok, int32_t* hist_par, float* pool_score,
                          float* pool_final, int32_t* pool_ref, int32_t* pool_n, int32_t* n_live, int32_t* end_ref,
                          float* end_score, int32_t* end_n, int end_cap, b200asr_stream_t stream);
/* The yseqs of n end-log entries, packed: entry j = entries[j] (= b * end_cap + e) gets its t + 2 ids (SOS, tokens), plus the
 * EOS if forced, at ids + offsets[j]; the length follows from the entry's ref alone, so the caller sizes ids exactly. */
int b200asr_beam_backtrack_packed(const int32_t* hist_tok, const int32_t* hist_par, const int32_t* end_ref, const int32_t* end_n,
                                  int end_cap, const int64_t* entries, const int64_t* offsets, int n, int64_t* ids, int B, int W,
                                  int steps, b200asr_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * LSTM language model of the LM rescoring (utils/lstm_utils.py: LM.evaluate :105-127 -> RNNModel.forward :185-193 ->
 * nn.LSTM(ninp, nhid, nlayers) + nn.Linear(nhid, ntoken) + CrossEntropyLoss).  H = nhid and I = ninp rounded up to multiples
 * of 8; prepared matrices are gate-interleaved (row 4u + g = gate g of unit u, gate order i, f, g, o) with zero padding.
 *   lstm_prepare: w_ih [4*nhid][ninp], w_hh [4*nhid][nhid], b_ih / b_hh [4*nhid] (NULL = 0) of one layer (nn.LSTM's
 *     weight_ih_l{k} ...) -> w_ih_p [4H][I], w_hh_p [4H][H], bias_p [4H] = b_ih + b_hh.  The bf16x3 operands are then
 *     b200asr_split_bf16(w_*_p, dst, NULL, 4H, K, 2).
 *   lstm_layer_fwd: sequences packed t-major, longest first: batch_sizes (HOST array [T]) = M_t sequences live at step t,
 *     non-increasing, >= 1; position off[t] + s, off[t] = M_0 + .. + M_{t-1}.  xproj [P][4H] = layer input x w_ih_p^T +
 *     bias_p (b200asr_linear_fwd); h [P][H] gets the layer output, c [M_0][H] is workspace.  Step 0 is the zero-state cell;
 *     each later step is one tensor-core launch (bf16x3 h_{t-1} W_hh^T, w_hh_split = its bf16 [2][4H][H] operand) whose
 *     epilogue adds xproj and applies the fp32 cell (1/(1+expf(-x)), tanhf).  H % 8 == 0.
 *   lm_nll: nll[r] = logsumexp(logits[r, :V]) - logits[r, targets[r]] in exact fp32 (row pitch ld); NaN for a target outside
 *     [0, V).  lm_seq_sum: sums[s] = sum over t < lengths[s] of nll[offsets[t] + s], in t order (reproducible). */
int b200asr_lstm_prepare(const float* w_ih, const float* w_hh, const float* b_ih, const float* b_hh, int ninp, int nhid,
                         float* w_ih_p, float* w_hh_p, float* bias_p, b200asr_stream_t stream);
int b200asr_lstm_layer_fwd(const float* xproj, const void* w_hh_split, const int32_t* batch_sizes, int T, int H, float* c, float* h,
                           b200asr_stream_t stream);
/* LSTM LM training: RNNModel("LSTM").forward (utils/lstm_utils.py:185-193) and its backward through time, replacing the
 * nn.LSTM of :147 (cuDNN).  One layer over a fixed batch of B sequences and T steps, rows t-major (row t * B + b).
 *   lstm_layer_train_fwd: xproj [T*B][4H] as for lstm_layer_fwd; h [(T+1)*B][H] with slot 0 (rows 0 .. B-1) = h0 -- read
 *     when has_state (then c0 [B][H] is read too), written as 0 otherwise -- and slot t + 1 = h_t, so that rows 0 .. T*B-1
 *     are h_{t-1} for every t; c [T*B][H] = c_t of every step; gates [T*B][4H] = the activated gates i, f, g, o of every step
 *     (gate-interleaved).  Step 0 is one tensor-core launch of h0 W_hh^T with a state, the zero-state cell without.  The
 *     same recurrence loop as lstm_layer_fwd, whose results it leaves bit-identical.
 *   lstm_layer_train_bwd: from the saved gates, c and c0 (NULL: zero state) and dh_out [T*B][H] (the gradient of every
 *     h_t from above), dh_n / dc_n [B][H] (the gradients of the final state; NULL = 0): dgates [T*B][4H] = the gradients of
 *     the gate pre-activations (interleaved), dc0 [B][H] = the gradient of c0 (NULL: not wanted), dc [B][H] workspace.
 *     Step T - 1 is an elementwise kernel; every earlier step one tensor-core launch of dgates_{t+1} W_hh_p (bf16x3,
 *     w_hh_split_t = the transposed operand dst_t [2][H][4H] of b200asr_split_bf16(w_hh_p, .., 4H, H, 2)) whose epilogue is
 *     the exact-fp32 cell backward.  The parameter gradients are then b200asr_linear_bwd_weight(dgates, x | h rows
 *     0 .. T*B-1), dh0 = b200asr_linear_bwd_data(dgates rows 0 .. B-1, w_hh_p) and dx = b200asr_linear_bwd_data(dgates,
 *     w_ih_p).  H % 8 == 0.
 *   lstm_dropout: y[i] = x[i] / (1 - p) or 0, kept by the counter-based generator keyed by (seed, offset) at element index
 *     i (the generator of b200asr_embed_fwd); applied to a gradient with the same key it is the backward.  n % 4 == 0.
 *   lstm_grad_unprepare: the inverse of lstm_prepare for gradients: dw_ih_p [4H][I], dw_hh_p [4H][H], db_p [4H] ->
 *     dw_ih [4*nhid][ninp], dw_hh [4*nhid][nhid] and db_ih = db_hh [4*nhid] (each output may be NULL), padding dropped. */
int b200asr_lstm_layer_train_fwd(const float* xproj, const void* w_hh_split, int T, int B, int H, int has_state, const float* c0,
                                 float* h, float* c, float* gates, b200asr_stream_t stream);
int b200asr_lstm_layer_train_bwd(const float* gates, const float* c, const float* c0, const float* dh_out, const float* dh_n,
                                 const float* dc_n, const void* w_hh_split_t, int T, int B, int H, float* dc, float* dgates, float* dc0,
                                 b200asr_stream_t stream);
int b200asr_lstm_dropout(const float* x, float* y, long long n, float p, uint64_t seed, uint64_t offset, b200asr_stream_t stream);
int b200asr_lstm_grad_unprepare(const float* dw_ih_p, const float* dw_hh_p, const float* db_p, int ninp, int nhid, float* dw_ih,
                                float* dw_hh, float* db_ih, float* db_hh, b200asr_stream_t stream);
int b200asr_lm_nll(const float* logits, long long ld, const int64_t* targets, float* nll, int rows, int V, b200asr_stream_t stream);
int b200asr_lm_seq_sum(const float* nll, const int64_t* offsets, const int64_t* lengths, int nseq, float* sums,
                       b200asr_stream_t stream);
/* LSTM LM training loss: nn.CrossEntropyLoss() with its defaults (mean over rows, nothing ignored), the criterion of
 * LM.__init__ (utils/lstm_utils.py:69) and of the word-language-model loop that trains RNNModel.  b200asr_ce_* cannot
 * serve: they drop every row whose target is 0 (PAD), and in an LM vocabulary 0 is '<eos>'.
 *   xent_fwd: nll [rows] = the row code of lm_nll (the same bits: logsumexp(logits[r, :V]) - logits[r, targets[r]] in exact
 *     fp32, row pitch ld, NaN for a target outside [0, V)); stats [rows][2] = (row max, logf(sum of exp(x - max))), read by
 *     xent_bwd; loss [1] = (sum of nll) / rows, summed in a fixed order by one CTA.  Two launches.
 *   xent_bwd: dlogits[r, v] = (exp(logits[r, v] - lse_r) - [v == targets[r]]) * (*dloss) / rows, formed as
 *     expf((x - max) - log-sum) from stats; dlogits has the row pitch ld too (columns V .. ld-1 untouched); a row whose
 *     target is outside [0, V) gets NaN.  dloss is a device scalar (the upstream gradient).  One launch.
 * rows >= 1, V >= 1, ld >= V (B200ASR_BAD_SHAPE), no NULL pointer (B200ASR_BAD_ARG); a rejected call launches nothing.  No
 * host synchronisation, no atomics: repeated calls give identical bits. */
int b200asr_xent_fwd(const float* logits, long long ld, const int64_t* targets, float* nll, float* stats, float* loss, int rows, int V,
                     b200asr_stream_t stream);
int b200asr_xent_bwd(const float* logits, long long ld, const int64_t* targets, const float* stats, const float* dloss, float* dlogits,
                     int rows, int V, b200asr_stream_t stream);
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

/* ------------------------------------------------------------------------------------------------
 * CTC loss, the ctc branch of calculate_loss (utils/metrics.py:133-154, trainer/asr/trainer.py:81-85):
 *   F.ctc_loss(log_softmax(logits.transpose(0, 1), dim=2), targets, input_lengths, target_lengths, blank=0,
 *              reduction="mean", zero_infinity=False)
 * computed from the logits in place, exact fp32, in log space.
 *   logits [B][T][V] fp32 contiguous; targets [B][S] int64, row b read at 0 .. target_lengths[b] - 1 only, labels in [0, V)
 *   (label 0 is the blank and allowed: the standard extended-label lattice); input_lengths / target_lengths [B] int32 (device).
 *   max_target_len >= every target_lengths[b], <= S and <= 4095; lengths must satisfy 0 <= input_lengths[b] <= T and
 *   0 <= target_lengths[b] <= max_target_len (the caller validates them; an utterance that breaks this gets NaN).
 *   ws: b200asr_ctc_ws_bytes(B, T, max_target_len) bytes, caller-owned, written by ctc_fwd and read by ctc_bwd (row
 *   log-sum-exps, the extended-label log-probabilities, the scaled alpha and beta lattices, label chains).
 * ctc_fwd: nll [B] = -log P(target_b | logits_b) (+inf if no alignment fits in input_lengths[b] frames; 0 when both lengths
 *   are 0); loss [1] = (sum over b in order of nll[b] / max(target_lengths[b], 1)) / B.
 * ctc_bwd: dlogits [B][T][V] = d(*dloss * loss) / d logits, with nll from ctc_fwd: rows t >= input_lengths[b] get 0, every
 *   row t < input_lengths[b] of an utterance with infinite nll gets NaN (as torch's backward).  No host synchronisation;
 *   reductions in a fixed order, so repeated calls give identical bits. */
size_t b200asr_ctc_ws_bytes(int B, int T, int max_target_len);
int b200asr_ctc_fwd(const float* logits, const int64_t* targets, const int32_t* input_lengths, const int32_t* target_lengths,
                    float* nll, float* loss, void* ws, int B, int T, int V, int S, int max_target_len, b200asr_stream_t stream);
int b200asr_ctc_bwd(const float* logits, const int64_t* targets, const int32_t* input_lengths, const int32_t* target_lengths,
                    const float* nll, const float* dloss, float* dlogits, void* ws, int B, int T, int V, int S, int max_target_len,
                    b200asr_stream_t stream);

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
/* ------------------------------------------------------------------------------------------------
 * Step tail over a list of separate tensors, as torch.optim.Adam holds them: NoamOpt.step (utils/optimizer.py:15-22) around
 * torch.optim.Adam (utils/functions.py:107) and torch.nn.utils.clip_grad_norm_ (trainer/asr/trainer.py:108-109).
 * `tensors` and the other per-tensor arrays are HOST arrays; each entry of `tensors` is a device address.  A call takes
 * 1 .. b200asr_optim_table_capacity() tensors (a longer list is split by the caller, one call per table); every address must
 * be non-NULL and 4-byte aligned (BAD_ARG / BAD_ALIGN), numel >= 0 (0 = nothing to do).  The table travels in the kernel
 * parameters: no host-to-device copy, no allocation, no host synchronisation.  Each call is one launch, except norm_multi
 * (two). */
int b200asr_optim_table_capacity(void);
/* tensors [count][4]: param, grad, exp_avg, exp_avg_sq, numel[count] elements each.  Per element, torch 2.11's foreach Adam
 * (torch/optim/adam.py, _multi_tensor_adam, non-capturable) op by op with the same fp32 roundings:
 *   m = lerp(m, g, lerp_weight); v = v * beta2; v = v + one_minus_beta2 * (g * g);
 *   d = sqrt(v) / bc2_sqrt[k] + eps; p = p + step_size[k] * (m / d)
 * with step_size[k] = -lr / (1 - beta1^step) and bc2_sqrt[k] = (1 - beta2^step)^0.5 of tensor k (lerp_weight = 1 - beta1 and
 * one_minus_beta2 = 1 - beta2 as the host rounds them).  Bit-identical to torch on the same inputs. */
int b200asr_adam_multi(const uint64_t* tensors, const long long* numel, const float* step_size, const float* bc2_sqrt, int count,
                       float lerp_weight, float beta2, float one_minus_beta2, float eps, b200asr_stream_t stream);
/* norms[k] (device, [count]) = ||tensors[k]||_2 (fp32, fixed-order sums: the same bits on every call). */
int b200asr_norm_multi(const uint64_t* tensors, const long long* numel, int count, float* norms, b200asr_stream_t stream);
/* out[0] (device) = sqrt(sum of norms[k]^2), out[1] = min(1, max_norm / (out[0] + 1e-6)) formed as clip_grad_norm_ forms it:
 * reciprocal(out[0] + 1e-6) * max_norm, then clamp(max=1) (NaN stays NaN).  One CTA. */
int b200asr_clip_coef(const float* norms, int count, float max_norm, float* out, b200asr_stream_t stream);
/* tensors[k] *= *coef (device scalar) for every element, in place. */
int b200asr_scale_multi(const uint64_t* tensors, const long long* numel, int count, const float* coef, b200asr_stream_t stream);
/* The word-language-model loop's update `for p in model.parameters(): p.data.add_(p.grad, alpha=-lr)` (the loop that trains
 * utils/lstm_utils.RNNModel): tensors [count][2] = param, grad; param = fma(alpha, grad, param) per element with
 * alpha = (float)(-lr), which is what ATen's add_ computes -- bit-identical to it on the same device. */
int b200asr_sgd_multi(const uint64_t* tensors, const long long* numel, int count, float alpha, b200asr_stream_t stream);

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
 * ws: b200asr_stft_ws_bytes(B, Lmax, n_fft, hop) bytes.  n_fft % 32 == 0, hop % 4 == 0, hop <= n_fft, 1 <= Tmax <=
 * 1 + Lmax/hop (B200ASR_BAD_SHAPE); ws and out 16-byte aligned (B200ASR_BAD_ALIGN); precision 0, 1 or 3, else
 * B200ASR_BAD_ARG.  A rejected call launches nothing. */
size_t b200asr_stft_ws_bytes(int B, int Lmax, int n_fft, int hop);
int b200asr_stft_features(const float* wave, const int* lens, float* out, int* frames_out, void* ws, int B,
                          int Lmax, int Tmax, int n_fft, int hop, int pad_reflect, int normalize, int window_periodic,
                          int precision, b200asr_stream_t stream);
/* The same front end with the rest of the reference's loader options (utils/data_loader.py:20-21,52,126-179):
 *   window: 0 Hamming, 1 Hann, 2 Blackman, 3 Bartlett (scipy's definitions; symmetric unless window_periodic), else
 *     B200ASR_BAD_ARG.
 *   Noise injection (NoiseInjection.inject_noise_sample, :168-179): noise_bank [noise_bank_len] fp32 holds the noise clips
 *     back to back; per utterance noise_start[b] (int64) is the first sample of its segment in the bank, < 0 for no noise,
 *     and noise_level[b] its level.  A noisy utterance of len samples becomes, before framing,
 *       x + ((level * n) * e_x) / e_n   (fp32, in numpy's order),  n = bank[start : start + len],
 *     with e_x, e_n = sqrt(sum of squares / len) of x and n, the sums in double with a fixed reduction order.  A silent
 *     segment gives NaN features (0/0, as in the reference); a silent utterance is unchanged.  All three pointers are
 *     device arrays, NULL together (no noise; otherwise B200ASR_BAD_ARG), and noise_bank_len > 0 with a bank
 *     (B200ASR_BAD_SHAPE).  The caller guarantees start + lens[b] <= noise_bank_len: the starts are device data, which the
 *     library does not read on the host; an utterance whose segment leaves the bank comes back NaN, nothing outside the
 *     bank is read.
 *   max_frames >= 1 (else B200ASR_BAD_SHAPE): the src_max_len cut (:131).  The statistics cover all 1 + lens[b]/hop
 *     frames of each utterance; frames t < min(1 + lens[b]/hop, max_frames, Tmax) are stored and frames_out[b] reports
 *     that count.  A max_frames no utterance reaches gives the bits of an uncut call.
 * With window 0, no noise and Tmax >= every utterance's 1 + lens[b]/hop frames, the output equals b200asr_stft_features's
 * bit for bit.  Other arguments and rejections as b200asr_stft_features; ws: b200asr_stft_features_ex_ws_bytes(B, Lmax,
 * n_fft, hop) bytes.  Launches: as b200asr_stft_features, + 2 with noise (energies, their reduction).  A rejected call
 * launches nothing. */
size_t b200asr_stft_features_ex_ws_bytes(int B, int Lmax, int n_fft, int hop);
int b200asr_stft_features_ex(const float* wave, const int* lens, float* out, int* frames_out, void* ws, int B, int Lmax,
                             int Tmax, int n_fft, int hop, int pad_reflect, int normalize, int window, int window_periodic,
                             const float* noise_bank, long long noise_bank_len, const long long* noise_start,
                             const float* noise_level, int max_frames, int precision, b200asr_stream_t stream);
/* b200asr_stft_features_ex over a packed batch: utterance b is the lens[b] samples at wave + offsets[b] (offsets: B device
 * int64, in any order, overlapping or not), so the caller uploads only the real samples instead of a zero-padded [B, Lmax]
 * rectangle.  Lmax >= every lens[b] sizes the workspace (b200asr_stft_features_ex_ws_bytes(B, Lmax, n_fft, hop)) and
 * bounds Tmax as in b200asr_stft_features_ex.  The output equals b200asr_stft_features_ex's on the same utterances laid out
 * at b * Lmax, bit for bit, with every option.  offsets NULL: B200ASR_BAD_ARG; offsets not 8-byte or wave not 4-byte
 * aligned: B200ASR_BAD_ALIGN.  The offsets are device data, which the library does not read on the host: an utterance
 * with a negative offset comes back NaN, nothing before wave is read.  Other arguments, rejections and launches as
 * b200asr_stft_features_ex. */
int b200asr_stft_features_packed(const float* wave, const long long* offsets, const int* lens, float* out, int* frames_out,
                                 void* ws, int B, int Lmax, int Tmax, int n_fft, int hop, int pad_reflect, int normalize,
                                 int window, int window_periodic, const float* noise_bank, long long noise_bank_len,
                                 const long long* noise_start, const float* noise_level, int max_frames, int precision,
                                 b200asr_stream_t stream);

/* Tempo and gain perturbation of a packed batch of waveforms: WSOLA (waveform-similarity overlap-add), modelled on sox's
 * `tempo` effect with its default profile (linear search; 82 ms segment, 82/5.587 ms search, 82/6.833 ms overlap), then
 * `gain` and the 16-bit output of the reference's `sox ... -b 16 -e si ... tempo T gain G` (utils/audio.py:35-47).  Parity
 * with sox itself is not claimed (sox may add TPDF dither when it writes 16 bits); the algorithm below is the contract.
 *
 * Utterance b: x = the in_lengths[b] fp32 samples at in + in_offsets[b], read as x~, x extended to the right with zeros
 * (nothing outside [in_offsets[b], in_offsets[b] + in_lengths[b]) is read); tempo[b] (float64) and the linear gain g[b]
 * (fp32, the caller's fp32(10^(gain_db / 20)) computed in float64); its output is the out_lengths[b] samples at
 * out + out_offsets[b].  The geometry is the caller's (the host layer computes it from the sample rate sr in float64:
 * segment = floor(sr * 82 / 1000 + 0.5), search = floor(sr * (82 / 5.587) / 1000 + 0.5), overlap = floor(max(sr *
 * (82 / 6.833) / 1000 + 4.5, 16)) rounded down to a multiple of 8, minus 8 if 2 * overlap > segment; at 16 kHz (1312, 235,
 * 192)).  step = segment - overlap; the caller's out_lengths[b] = floor(n / tempo + 0.5) and K_b = ceil(out_lengths[b] /
 * step) segments.
 *   Segment k: input start S_k = floor(tempo * (k * step) + 0.5) in float64 (k * step an exact integer), independent of any
 *   pick.  Pick p_0 = floor(search / 2); for k >= 1, with prev_j = x~[S_{k-1} + p_{k-1} + step + j] (j < overlap), p_k is the
 *   smallest i in [0, search) minimising D(i) = sum_j (x~[S_k + i + j] - prev_j)^2 computed in float64 (a NaN D counts as
 *   +inf).  On inputs from 16-bit files (k / 32768) every term and partial sum of D is exact, so the picks do not depend
 *   on the summation order.  Segment k writes y[k * step + j] for j < step: x~[S_k + p_k + j], except for k >= 1 and
 *   j < overlap the crossfade fp32(fp32(prev_j * fp32(1 - f_j)) + fp32(x~[S_k + p_k + j] * f_j)), f_j = fp32(j * fp32(1 /
 *   overlap)), every operation rounded on its own (no FMA).
 *   Output: v = fp32(y * g), written as clamp(rint(v * 32768), -32768, 32767) / 32768 (half to even; NaN stays NaN) --
 *   what load_audio returns for a 16-bit file; gains above 0 dB clip loud utterances.  Samples k * step + j >=
 *   out_lengths[b] are not written.
 * picks, pick_offsets: NULL together, or p_k written to picks[pick_offsets[b] + k] for k < K_b (int32 / int64 device arrays).
 *
 * One launch, one CTA per utterance walking its K_b segments in order (the next window prefetched while one is searched).
 * Rejections, which launch and write nothing: a NULL pointer other than picks / pick_offsets, or exactly one of those
 * two NULL (B200ASR_BAD_ARG); in, in_lengths, g, out, out_lengths or picks not 4-byte, in_offsets, tempo, out_offsets or
 * pick_offsets not 8-byte aligned (B200ASR_BAD_ALIGN); B < 1, overlap < 8, 2 * overlap > segment, search < 1, or a
 * geometry whose 8 (3 overlap + search - 1) + 8 (search + segment - 1) bytes of shared memory exceed 226 KB
 * (B200ASR_BAD_SHAPE).  The per-utterance arrays are device data, which the library does not read on the host: an
 * utterance with a non-finite or non-positive tempo, a negative in_offsets or a negative in_lengths gets NaN for its
 * out_lengths[b] samples and -1 for its picks; one with a negative out_offsets or out_lengths[b] <= 0 writes nothing (nor
 * does a negative pick_offsets write picks).  out must not overlap in. */
int b200asr_tempo_gain(const float* in, const long long* in_offsets, const int* in_lengths, const double* tempo,
                       const float* g, float* out, const long long* out_offsets, const int* out_lengths, int* picks,
                       const long long* pick_offsets, int B, int segment, int search, int overlap,
                       b200asr_stream_t stream);

/* One utterance of b200asr_resample_packed: its in_length samples start at in + in_offset, its outputs at out + out_offset;
 * up / down is its ratio in lowest terms; taps is a device array of the ratio's phase-split filter (below), NULL allowed
 * for up == down == 1.  40 bytes, 8-byte aligned. */
typedef struct {
  long long in_offset;
  long long out_offset;
  const float* taps;
  int in_length;
  int up;
  int down;
  int reserved;
} b200asr_resample_item;

/* Polyphase resampling of a packed batch of waveforms: utterance b becomes scipy.signal.resample_poly(x, up, down) with
 * its defaults, computed in fp32.  That function is the contract, restated here:
 *   up / down in lowest terms (the caller reduces by the gcd).  up == down == 1: y = x, copied, not filtered.  Otherwise
 *   half = 10 max(up, down) and h = firwin(2 half + 1, 1 / max(up, down), window=('kaiser', 5.0)) * up: the windowed
 *   sinc h_k = w_k sin(pi f (k - half)) / (pi (k - half)) (f for k = half), w the symmetric Kaiser window of beta 5,
 *   scaled to unit sum, then times up, designed in float64 and rounded once to fp32.  x is zero outside [0, n) (scipy's
 *   padtype='constant'), and with scipy's delay compensation the n_out = ceil(n up / down) outputs are
 *     y[i] = sum_j h[i down + half - j up] x[j]    over 0 <= i down + half - j up <= 2 half.
 *   taps, phase-split: with K = ceil((2 half + 1) / up), taps[p K + m] = fp32(h[p + m up]) for p < up, m < K (0 past
 *   2 half).  Output i, with c = i down + half, p = c mod up and j0 = floor(c / up), is the fp32 sum
 *   s = fma(taps[p K + m], x[j0 - m], s) over m = 0, 1, ... while p + m up <= 2 half, from s = 0, in that order: the
 *   bits do not depend on the batch, the launch or the run.
 *   quantize16 = 1 writes clamp(rint(y * 32768), -32768, 32767) / 32768 instead (half to even, no dither; NaN stays
 *   NaN), the grid `sox ... -b 16 -e si` writes; 0 writes y.
 * items: B host descriptors, read and checked before launch; items_dev: a device copy of the same B descriptors, which the
 * kernel reads (the library does not compare them).  in_size / out_size: floats in the in / out buffers.
 *
 * One launch: CTA (chunk, utterance) stages the input window of up to 2048 consecutive outputs in shared memory.
 * Rejections, which launch and write nothing: a NULL in, out, items or items_dev, a quantize16 other than 0 or 1, out
 * overlapping in, or a NULL or misaligned taps where up / down != 1 (B200ASR_BAD_ARG); in or out not 4-byte, items_dev
 * not 8-byte aligned (B200ASR_BAD_ALIGN); B < 1, a negative in_size or out_size, up or down outside [1, 1000] or not
 * coprime, an input outside [0, in_size), an output outside [0, out_size), or two outputs that overlap
 * (B200ASR_BAD_SHAPE).  A batch whose outputs are all empty launches nothing. */
int b200asr_resample_packed(const float* in, long long in_size, float* out, long long out_size,
                            const b200asr_resample_item* items, const b200asr_resample_item* items_dev, int B,
                            int quantize16, b200asr_stream_t stream);

/* SpecAugment (Park et al. 2019, "SpecAugment: A Simple Data Augmentation Method for Automatic Speech Recognition") over a
 * batch of the front end's output: in, out [B,1,F,T] fp32 (the layout above), frames [B] int32 (device) = each
 * utterance's frame count after the src_max_len cut (input_sizes), read as T_b = min(max(frames[b], 0), T).  Applied in
 * this order over frames [0, T_b) of each utterance; frames t >= T_b of out are 0.
 *
 * Draws.  Integer j of utterance b is uniform in [lo, hi]:  lo + ((r >> 32) * (hi - lo + 1)) >> 32  with
 * r = splitmix64(key + (b << 16 | j) * 0x9E3779B97F4A7C15) and key = splitmix64(seed ^ (counter * 0xD1342543DE82EF95 +
 * 0x2545F4914F6CDD1D)) -- the counter stream of dropout (common.cuh: dropout_key, dropout_bits4), 64-bit unsigned
 * arithmetic throughout.  No host draw and no host synchronisation.  draws [B][n] int32 (n =
 * b200asr_spec_augment_draws_ints(n_freq_masks, n_time_masks) = 2 + 2 n_freq_masks + 2 n_time_masks) receives the
 * integers used, at their slot j: c, w, then (f, f0) per frequency mask, then (t, t0) per time mask.
 *
 * Time warp.  If T_b > 2W + 1: c uniform in [W, T_b - W - 1] (slot 0), w uniform in [-W, W] (slot 1); otherwise no draw
 *   is made, c = w = 0 and the utterance is not warped (nor is it when w = 0).  With d = c + w, output frame t reads the
 *   source position s(t) = num / den of the piecewise linear map 0 -> 0, d -> c, T_b - 1 -> T_b - 1 (integers):
 *     t = 0 or t = T_b - 1:  s = t (the end frames stay put)
 *     0 < t <= d:            num = t * c,                   den = d,              i0 = num / den
 *     d < t < T_b - 1:       num = (t - d) * (T_b - 1 - c), den = T_b - 1 - d,    i0 = c + num / den
 *   rem = num % den; out = x[i0] when rem == 0, else fmaf((float)rem / (float)den, x[i0 + 1] - x[i0], x[i0]) in fp32 --
 *   linear interpolation between the two neighbouring source frames, x[i0 + 1] read only then (i0 + 1 <= T_b - 1).
 *   Degenerate segments: with d = 0 (c = W, w = -W) frame 0 still reads frame 0 and frames 1 .. T_b - 2 the second piece,
 *   which starts from c; with d = T_b - 1 (c = T_b - W - 1, w = W) frame T_b - 1 still reads itself and frames 1 .. T_b - 2
 *   the first piece, which ends at c.  Integer parts and remainders are exact; the weight is exact for T_b < 2^24.
 * Frequency masks.  For each of n_freq_masks: f uniform in [0, Fp], f0 uniform in [0, F - f]; bins [f0, f0 + f) become 0.
 * Time masks.  For each of n_time_masks: t uniform in [0, min(Tp, floor(p * T_b))] (p * T_b in double), t0 uniform in
 *   [0, T_b - t]; frames [t0, t0 + t) become 0.
 * 0 is the utterance mean of normalised features.  Masked elements and padding are written as exact zeros.
 *
 * One launch; each element is read once (twice where the warp interpolates) and written once.  Rejections, which launch and
 * write nothing: a NULL pointer (B200ASR_BAD_ARG); a pointer that is not 4-byte aligned (B200ASR_BAD_ALIGN); B, F or T < 1,
 * B > 65535, F > 1048560 or F * T > 2^31 - 1 (B200ASR_BAD_SHAPE); W < 0, Fp < 0, Fp > F, Tp < 0, p outside [0, 1] or NaN, a mask
 * count outside [0, 64], or out overlapping in (the warp reads other frames than it writes) (B200ASR_BAD_ARG).
 * b200asr_spec_augment_draws_ints returns 0 for a mask count outside [0, 64]. */
size_t b200asr_spec_augment_draws_ints(int n_freq_masks, int n_time_masks);
int b200asr_spec_augment(const float* in, float* out, int* draws, const int* frames, int B, int F, int T, int W, int Fp,
                         int n_freq_masks, int Tp, float p, int n_time_masks, unsigned long long seed,
                         unsigned long long counter, b200asr_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * Edit counts of the training loop's CER / WER (trainer/asr/trainer.py:60-79, 96-104 and 153-182), with no host read per
 * token.  Per utterance b the strings h (from hyp row b) and g (from gold row b) are built as the trainer builds them: the
 * ids in order up to the first pad_id, the labels of the ids joined.  Then
 *   per_utt[b][0] = cer_edits  = Levenshtein(h without ' ', g without ' ') over code points   (calculate_cer)
 *   per_utt[b][1] = wer_edits  = Levenshtein over words, a word being a maximal run of code points that are not
 *                                str.isspace(); two words are equal when their code points are      (calculate_wer)
 *   per_utt[b][2] = gold_chars = number of code points of g other than ' '
 *   per_utt[b][3] = gold_words = (number of ' ' in g) + 1                                          (len(g.split(" ")))
 *   totals[0..3]  = the sums of the four columns over b = 0 .. B-1 in order; totals[4] = the first invalid id met in the
 *                   trainer's order -- every gold row before any hyp row, tokens in order within a row, each row up to its
 *                   first pad_id -- or -1 when every such id is valid (an id of -1 itself is therefore not told apart).
 *   An invalid id contributes no code points.
 * hyp [B][T_h] and gold [B][T_g]: ids, int64 (*_int64 = 1) or int32 (0), row b at hyp + b * hyp_row_stride (elements);
 *   row strides >= T.  T_h, T_g >= 0, B >= 1.
 * The label table (CSR, device arrays): for id in [0, V), label_valid[id] != 0 marks a valid id, whose label is the
 *   label_len[id] code points code_points[label_off[id] ..] (int32, 0 .. 0x10FFFF); per code point, cp_flags bit 0 = the
 *   code point is ' ' (U+0020) and bit 1 = str.isspace().  Ids < 0 or >= V are invalid.  Every label_len[id] <=
 *   max_label_len: an utterance whose strings outgrow what that bound allows gets -1 in its four counts.  The trainer's
 *   SOS / EOS removal is the table builder's: it drops those code points from every label.
 * ws: b200asr_edit_counts_ws_bytes(B, T_h, T_g, max_label_len) bytes, 16-byte aligned, caller-owned: 16 * B bytes for the
 *   first invalid position of every row, plus, when the longest strings the shapes allow would not fit in 46 KB of shared
 *   memory, a buffer per utterance that utterances too long for shared memory expand into.  Its size grows as
 *   B * (T_h + T_g) * max_label_len; 0 for shapes whose per-utterance buffer would pass 2^30 int32 entries (about
 *   (T_h + T_g) * max_label_len > 2^28; the call rejects those shapes).
 * Return: B200ASR_BAD_ARG for a NULL pointer or an *_int64 other than 0 / 1, B200ASR_BAD_SHAPE for the shapes above,
 *   B200ASR_BAD_ALIGN for ids / table / outputs not aligned to their element or ws not to 16 bytes.  A rejected call launches
 *   nothing.  Launches: 2 (one CTA per utterance, then one for the totals).  No host synchronisation and no atomics: repeated
 *   calls give identical bits.  Exact anti-diagonal DP, O(|h| |g|) work and |h| + |g| barriers per utterance. */
size_t b200asr_edit_counts_ws_bytes(int B, int T_h, int T_g, int max_label_len);
int b200asr_edit_counts(const void* hyp, int hyp_int64, long long hyp_row_stride, int T_h, const void* gold, int gold_int64,
                        long long gold_row_stride, int T_g, int B, const int* label_off, const int* label_len,
                        const int* code_points, const uint8_t* cp_flags, const uint8_t* label_valid, int V, int max_label_len,
                        long long pad_id, int64_t* per_utt, int64_t* totals, void* ws, b200asr_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* B200ASR_H_ */
