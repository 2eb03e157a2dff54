// Decoder input side (target preprocessing, embedding + PE), output side (argmax, label-smoothed CE) and the
// step tail (Adam, grad-norm).  All HBM-bound: 128-bit accesses, one warp or CTA per row.
#include <math.h>

#include "../../include/b200asr.h"
#include "common.cuh"

namespace b200asr {

constexpr int64_t TOK_PAD = 0, TOK_SOS = 1, TOK_EOS = 2;

__global__ void preprocess_targets_kernel(const int64_t* __restrict__ tgt, int L, int64_t* __restrict__ seq_in,
                                          int64_t* __restrict__ seq_out, uint8_t* __restrict__ key_pad,
                                          float* __restrict__ non_pad, int* __restrict__ status, int B, int Tt) {
  int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const int64_t* y = tgt + (size_t)b * L;
  int64_t* si = seq_in + (size_t)b * Tt;
  int64_t* so = seq_out + (size_t)b * Tt;
  int n = 0;
  si[0] = TOK_SOS;
  for (int i = 0; i < L; i++) {
    int64_t t = y[i];
    if (t == TOK_PAD) continue;
    if (n + 1 < Tt) { si[n + 1] = t; so[n] = t; }
    n++;
  }
  if (n + 1 > Tt) { if (status) atomicExch(status, 1); n = Tt - 1; }
  so[n] = TOK_EOS;
  for (int i = n + 1; i < Tt; i++) { si[i] = TOK_EOS; so[i] = TOK_PAD; }
  for (int i = 0; i < Tt; i++) {
    bool pad = si[i] == TOK_EOS;
    key_pad[(size_t)b * Tt + i] = pad ? 1 : 0;
    non_pad[(size_t)b * Tt + i] = pad ? 0.f : 1.f;
  }
}

__global__ void length_masks_kernel(const int32_t* __restrict__ lengths, uint8_t* __restrict__ key_pad,
                                    float* __restrict__ non_pad, int B, int T) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * T) return;
  int b = i / T, t = i - b * T;
  bool pad = t >= lengths[b];
  if (key_pad) key_pad[i] = pad ? 1 : 0;
  if (non_pad) non_pad[i] = pad ? 0.f : 1.f;
}

__global__ void embed_fwd_kernel(const int64_t* __restrict__ tokens, const float* __restrict__ table,
                                 const float* __restrict__ pe, float* __restrict__ out, int rows, int T, int d, int V,
                                 float scale, uint32_t thresh, float inv_keep, uint64_t key) {
  int row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (row >= rows) return;
  int64_t tok = tokens[row];
  tok = tok < 0 ? 0 : (tok >= V ? V - 1 : tok);
  const float* e = table + (size_t)tok * d;
  const float* p = pe + (size_t)(row % T) * d;
  const size_t base = (size_t)row * d;
  for (int c = lane * 4; c < d; c += 128) {
    float4 a = *reinterpret_cast<const float4*>(e + c);
    float4 q = *reinterpret_cast<const float4*>(p + c);
    a.x = a.x * scale + q.x; a.y = a.y * scale + q.y; a.z = a.z * scale + q.z; a.w = a.w * scale + q.w;
    if (thresh) {
      uint64_t r = dropout_bits4(key, (base + c) >> 2);
      a.x = ((uint32_t)(r) & 0xFFFFu) >= thresh ? a.x * inv_keep : 0.f;
      a.y = ((uint32_t)(r >> 16) & 0xFFFFu) >= thresh ? a.y * inv_keep : 0.f;
      a.z = ((uint32_t)(r >> 32) & 0xFFFFu) >= thresh ? a.z * inv_keep : 0.f;
      a.w = ((uint32_t)(r >> 48) & 0xFFFFu) >= thresh ? a.w * inv_keep : 0.f;
    }
    *reinterpret_cast<float4*>(out + base + c) = a;
  }
}

// One block per row; the FIRST row holding a token adds, in row order, the gradients of every row holding it into that
// token's table row -- no atomics, so a token that occurs many times gets the same sum in every run.
__global__ void embed_bwd_kernel(const int64_t* __restrict__ tokens, const float* __restrict__ dout,
                                 float* __restrict__ dtable, int rows, int d, int V, float scale, uint32_t thresh,
                                 float inv_keep, uint64_t key, int pad_idx) {
  const int row = blockIdx.x;
  const int64_t tok = tokens[row];
  if (tok == pad_idx || tok < 0 || tok >= V) return;
  __shared__ int earlier;
  if (threadIdx.x == 0) earlier = 0;
  __syncthreads();
  for (int j = threadIdx.x; j < row; j += blockDim.x)
    if (tokens[j] == tok) earlier = 1;
  __syncthreads();
  if (earlier) return;
  for (int c = threadIdx.x * 4; c < d; c += blockDim.x * 4) {
    float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int j = row; j < rows; j++) {
      if (__ldg(tokens + j) != tok) continue;
      const size_t base = (size_t)j * d;
      const float4 a = *reinterpret_cast<const float4*>(dout + base + c);
      float k0 = scale, k1 = scale, k2 = scale, k3 = scale;
      if (thresh) {
        uint64_t r = dropout_bits4(key, (base + c) >> 2);
        k0 = ((uint32_t)(r) & 0xFFFFu) >= thresh ? scale * inv_keep : 0.f;
        k1 = ((uint32_t)(r >> 16) & 0xFFFFu) >= thresh ? scale * inv_keep : 0.f;
        k2 = ((uint32_t)(r >> 32) & 0xFFFFu) >= thresh ? scale * inv_keep : 0.f;
        k3 = ((uint32_t)(r >> 48) & 0xFFFFu) >= thresh ? scale * inv_keep : 0.f;
      }
      s.x += a.x * k0; s.y += a.y * k1; s.z += a.z * k2; s.w += a.w * k3;
    }
    float4* g = reinterpret_cast<float4*>(dtable + (size_t)tok * d + c);
    const float4 o = *g;
    *g = make_float4(o.x + s.x, o.y + s.y, o.z + s.z, o.w + s.w);
  }
}

__global__ void argmax_rows_kernel(const float* __restrict__ x, int64_t* __restrict__ out, int rows, int V) {
  int row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (row >= rows) return;
  const float* r = x + (size_t)row * V;
  float bv = -INFINITY; int bi = 0x7fffffff;
  for (int c = lane; c < V; c += 32) { float v = r[c]; if (v > bv) { bv = v; bi = c; } }
  if (bi == 0x7fffffff) bi = lane < V ? lane : 0;     // all -inf / NaN lanes
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    float ov = __shfl_xor_sync(0xffffffffu, bv, o);
    int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    argmax_combine(bv, bi, ov, oi);
  }
  if (lane == 0) out[row] = bi;
}

// One greedy-decoding step (models/asr/transformer.py:375-382 + the EOS cut of :385-393) on the device: argmax of every
// utterance's last-position logits (first max, as torch.max), next input token, the emitted id (-1 once the utterance has
// produced EOS: the reference drops everything from the first EOS on when it builds the strings) and the EOS bookkeeping
// that lets the host stop the loop without reading the ids back (finished[b], *n_finished).
__global__ void greedy_step_kernel(const float* __restrict__ logits, int64_t* __restrict__ next_tok, int64_t* __restrict__ ys,
                                   int* __restrict__ finished, int* __restrict__ n_finished, int B, int V, int t, int steps) {
  int row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (row >= B) return;
  const float* r = logits + (size_t)row * V;
  float bv = -INFINITY; int bi = 0x7fffffff;
  for (int c = lane; c < V; c += 32) { float v = r[c]; if (v > bv) { bv = v; bi = c; } }
  if (bi == 0x7fffffff) bi = lane < V ? lane : 0;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    float ov = __shfl_xor_sync(0xffffffffu, bv, o);
    int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    argmax_combine(bv, bi, ov, oi);
  }
  if (lane == 0) {
    next_tok[row] = bi;
    const int fin = finished[row];
    ys[(size_t)row * steps + t] = (fin || bi == TOK_EOS) ? -1 : bi;
    if (!fin && bi == TOK_EOS) { finished[row] = 1; atomicAdd(n_finished, 1); }
  }
}

constexpr int CE_THREADS = 256;

__global__ void __launch_bounds__(CE_THREADS) ce_fwd_kernel(const float* __restrict__ logits,
                                                            const int64_t* __restrict__ gold, float* __restrict__ row_lse,
                                                            float* __restrict__ part, int rows, int V, float eps) {
  const int row = blockIdx.x;
  const float* x = logits + (size_t)row * V;
  // sum of exp and the sum of the logits, both relative to the row maximum: the loss below is then a combination of
  // terms of the size of the loss itself, whatever offset the logits share (lse - x_g with both ~ 200 would lose 8 bits)
  const RowLse st = block_row_lse<CE_THREADS, true>(x, V);
  const float mx = st.mx, sumd = st.sumdiff;
  const int amax = st.amax;
  if (threadIdx.x == 0) {
    const float lt = logf(st.sumexp);              // lse - mx
    row_lse[row] = mx + lt;
    const int64_t g = gold[row];
    float* pr = part + (size_t)row * 3;            // (loss, 1, correct) of this row; zeros for PAD rows
    pr[0] = pr[1] = pr[2] = 0.f;
    if (g != TOK_PAD) {
      const float xg = x[g] - mx;
      float loss;
      if (eps > 0.f) {
        const float off = eps / (float)V;
        const float wsum = (1.f - eps) + off * (float)(V - 1);
        loss = wsum * lt - (off * (sumd - xg) + (1.f - eps) * xg);
      } else {
        loss = lt - xg;
      }
      pr[0] = loss;
      pr[1] = 1.f;
      pr[2] = (int64_t)amax == g ? 1.f : 0.f;
    }
  }
}

__global__ void __launch_bounds__(CE_THREADS) ce_bwd_kernel(const float* __restrict__ logits,
                                                            const int64_t* __restrict__ gold,
                                                            const float* __restrict__ row_lse, float* __restrict__ dlogits,
                                                            int rows, int V, float eps, float gscale,
                                                            const float* __restrict__ gscale_dev,
                                                            const float* __restrict__ gscale_dev2) {
  const int row = blockIdx.x, tid = threadIdx.x;
  const float* x = logits + (size_t)row * V;
  float* dx = dlogits + (size_t)row * V;
  const int64_t g = gold[row];
  if (g == TOK_PAD) {
    for (int c = tid; c < V; c += CE_THREADS) dx[c] = 0.f;
    return;
  }
  const float gs = gscale * (gscale_dev ? *gscale_dev : 1.f) * (gscale_dev2 ? *gscale_dev2 : 1.f);
  const float lse = row_lse[row];
  const float off = eps > 0.f ? eps / (float)V : 0.f;
  const float on = eps > 0.f ? 1.f - eps : 1.f;
  const float wsum = on + off * (float)(V - 1);
  for (int c = tid; c < V; c += CE_THREADS) {
    float p = expf(x[c] - lse);
    float w = (c == (int)g) ? on : off;
    dx[c] = gs * (p * wsum - w);
  }
}

__global__ void ce_finalize_kernel(float* __restrict__ stats, float* __restrict__ loss_out, int mean) {
  const float s = stats[0], n = stats[1];
  stats[3] = s / n;
  stats[4] = 1.f / n;
  if (loss_out) loss_out[0] = mean ? s / n : s;
}

__global__ void adam_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m, float* __restrict__ v,
                            long long n, float lr, float b1, float b2, float eps, float bc1, float bc2_sqrt, float gscale,
                            const float* __restrict__ gscale_dev) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float gs = gscale * (gscale_dev ? *gscale_dev : 1.f);
  float gi = g[i] * gs;
  float mi = b1 * m[i] + (1.f - b1) * gi;
  float vi = b2 * v[i] + (1.f - b2) * gi * gi;
  m[i] = mi; v[i] = vi;
  // torch.optim.Adam: denom = sqrt(v)/sqrt(bias_correction2) + eps ; p -= lr/bias_correction1 * m / denom
  float denom = sqrtf(vi) / bc2_sqrt + eps;
  p[i] -= (lr / bc1) * mi / denom;
}

// part[block] = the block's sum of squares (reduce_parts adds the blocks in order)
__global__ void sumsq_kernel(const float* __restrict__ g, long long n, float* __restrict__ part) {
  __shared__ float red[8];
  float s = 0.f;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    float v = g[i];
    s += v * v;
  }
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int w = 0; w < (int)(blockDim.x >> 5); w++) t += red[w];
    part[blockIdx.x] = t;
  }
}

// out[0] = (1 / n_tokens) * min(1, max_norm / (||g|| / n_tokens + 1e-6)): the normalisation by the global token count
// (utils/metrics.py:127-130) times the coefficient of torch.nn.utils.clip_grad_norm_ (trainer/asr/trainer.py:108-109),
// computed on the device so that the optimizer step needs no host round trip.
__global__ void grad_scale_kernel(const float* __restrict__ n_tokens, const float* __restrict__ sumsq, float max_norm,
                                  float* __restrict__ out) {
  const float inv = 1.f / n_tokens[0];
  float clip = 1.f;
  if (sumsq) {
    const float norm = sqrtf(sumsq[0]) * inv;
    clip = fminf(1.f, max_norm / (norm + 1e-6f));
  }
  out[0] = inv * clip;
  out[1] = sumsq ? sqrtf(sumsq[0]) * inv : 0.f;      // the gradient norm, for logging
}

__global__ void permute_cols_kernel(const float* __restrict__ src, float* __restrict__ dst, int rows, int C, int F, int inverse) {
  long long n = (long long)rows * C * F;
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  int K = C * F;
  long long r = i / K;
  int j = (int)(i - r * K);
  int sj;
  if (!inverse) { int f = j / C, c = j - f * C; sj = c * F + f; }   // dst col f*C+c <- src col c*F+f
  else { int c = j / F, f = j - c * F; sj = f * C + c; }            // dst col c*F+f <- src col f*C+c
  dst[i] = src[r * K + sj];
}

}  // namespace b200asr

using namespace b200asr;

extern "C" {

int b200asr_preprocess_targets(const int64_t* padded_target, int L, int64_t* seq_in, int64_t* seq_out, uint8_t* key_pad,
                               float* non_pad, int* status, int B, int Tt, b200asr_stream_t stream) {
  B200_REQUIRE(padded_target && seq_in && seq_out && key_pad && non_pad, B200ASR_BAD_ARG, "preprocess_targets: null pointer");
  B200_REQUIRE(B > 0 && Tt >= 2 && L >= 0, B200ASR_BAD_SHAPE, "preprocess_targets: B=%d Tt=%d L=%d", B, Tt, L);
  preprocess_targets_kernel<<<ceil_div(B, 64), 64, 0, (cudaStream_t)stream>>>(padded_target, L, seq_in, seq_out, key_pad, non_pad, status, B, Tt);
  return check_launch("preprocess_targets");
}

int b200asr_length_masks(const int32_t* lengths, uint8_t* key_pad, float* non_pad, int B, int T, b200asr_stream_t stream) {
  B200_REQUIRE(lengths && (key_pad || non_pad) && B > 0 && T > 0, B200ASR_BAD_ARG, "length_masks: bad arguments");
  length_masks_kernel<<<ceil_div(B * T, 256), 256, 0, (cudaStream_t)stream>>>(lengths, key_pad, non_pad, B, T);
  return check_launch("length_masks");
}

int b200asr_embed_fwd(const int64_t* tokens, const float* table, const float* pe, float* out, int rows, int T, int d, int V,
                      float scale, float p_drop, uint64_t seed, uint64_t offset, b200asr_stream_t stream) {
  B200_REQUIRE(tokens && table && pe && out, B200ASR_BAD_ARG, "embed_fwd: null pointer");
  B200_REQUIRE(d % 4 == 0 && T > 0 && V > 0, B200ASR_BAD_SHAPE, "embed_fwd: d=%d T=%d V=%d", d, T, V);
  B200_REQUIRE(aligned16(table) && aligned16(pe) && aligned16(out), B200ASR_BAD_ALIGN, "embed_fwd: alignment");
  if (rows <= 0) return B200ASR_OK;
  embed_fwd_kernel<<<ceil_div(rows, 8), 256, 0, (cudaStream_t)stream>>>(tokens, table, pe, out, rows, T, d, V, scale,
                                                                        p_drop > 0.f ? dropout_thresh16(p_drop) : 0u,
                                                                        dropout_inv_keep(p_drop), dropout_key(seed, offset));
  return check_launch("embed_fwd");
}

int b200asr_embed_bwd(const int64_t* tokens, const float* dout, float* dtable, int rows, int d, int V, float scale,
                      float p_drop, uint64_t seed, uint64_t offset, int pad_idx, b200asr_stream_t stream) {
  B200_REQUIRE(tokens && dout && dtable, B200ASR_BAD_ARG, "embed_bwd: null pointer");
  B200_REQUIRE(d % 4 == 0, B200ASR_BAD_SHAPE, "embed_bwd: d=%d", d);
  if (rows <= 0) return B200ASR_OK;
  embed_bwd_kernel<<<rows, 128, 0, (cudaStream_t)stream>>>(tokens, dout, dtable, rows, d, V, scale,
                                                                        p_drop > 0.f ? dropout_thresh16(p_drop) : 0u,
                                                                        dropout_inv_keep(p_drop), dropout_key(seed, offset), pad_idx);
  return check_launch("embed_bwd");
}

int b200asr_greedy_step(const float* logits, int64_t* next_tok, int64_t* ys, int* finished, int* n_finished, int B, int V, int t,
                        int steps, b200asr_stream_t stream) {
  B200_REQUIRE(logits && next_tok && ys && finished && n_finished && B > 0 && V > 0 && t >= 0 && t < steps, B200ASR_BAD_ARG,
               "greedy_step: bad arguments");
  greedy_step_kernel<<<ceil_div(B * 32, 128), 128, 0, (cudaStream_t)stream>>>(logits, next_tok, ys, finished, n_finished, B, V, t, steps);
  return check_launch("greedy_step");
}

int b200asr_argmax_rows(const float* logits, int64_t* out, int rows, int V, b200asr_stream_t stream) {
  B200_REQUIRE(logits && out && V > 0, B200ASR_BAD_ARG, "argmax_rows: bad arguments");
  if (rows <= 0) return B200ASR_OK;
  argmax_rows_kernel<<<ceil_div(rows, 8), 256, 0, (cudaStream_t)stream>>>(logits, out, rows, V);
  return check_launch("argmax_rows");
}

int b200asr_ce_fwd(const float* logits, const int64_t* gold, float* row_lse, float* stats, int rows, int V, float smoothing,
                   b200asr_stream_t stream) {
  B200_REQUIRE(logits && gold && row_lse && stats && V > 0, B200ASR_BAD_ARG, "ce_fwd: bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  if (rows <= 0) {
    cudaMemsetAsync(stats, 0, 3 * sizeof(float), st);
    return B200ASR_OK;
  }
  float* part = (float*)stream_scratch(sizeof(float) * 3 * (size_t)rows, st);
  if (!part) return B200ASR_CUDA_ERROR;
  ce_fwd_kernel<<<rows, CE_THREADS, 0, st>>>(logits, gold, row_lse, part, rows, V, smoothing);
  int rc = check_launch("ce_fwd");
  return rc ? rc : reduce_parts(part, rows, 3, 3, stats, 0, st);
}

int b200asr_ce_finalize(float* stats, float* loss_out, int mean, b200asr_stream_t stream) {
  B200_REQUIRE(stats, B200ASR_BAD_ARG, "ce_finalize: null pointer");
  ce_finalize_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(stats, loss_out, mean);
  return check_launch("ce_finalize");
}

int b200asr_ce_bwd(const float* logits, const int64_t* gold, const float* row_lse, float* dlogits, int rows, int V,
                   float smoothing, float gscale, const float* gscale_dev, const float* gscale_dev2,
                   b200asr_stream_t stream) {
  B200_REQUIRE(logits && gold && row_lse && dlogits && V > 0, B200ASR_BAD_ARG, "ce_bwd: bad arguments");
  if (rows <= 0) return B200ASR_OK;
  ce_bwd_kernel<<<rows, CE_THREADS, 0, (cudaStream_t)stream>>>(logits, gold, row_lse, dlogits, rows, V, smoothing, gscale, gscale_dev, gscale_dev2);
  return check_launch("ce_bwd");
}

int b200asr_adam_step(float* p, const float* g, float* m, float* v, long long n, float lr, float beta1, float beta2,
                      float eps, int step, float gscale, const float* gscale_dev, b200asr_stream_t stream) {
  B200_REQUIRE(p && g && m && v && step >= 1, B200ASR_BAD_ARG, "adam_step: bad arguments");
  if (n <= 0) return B200ASR_OK;
  float bc1 = 1.f - powf(beta1, (float)step);
  float bc2 = 1.f - powf(beta2, (float)step);
  adam_kernel<<<(unsigned)ceil_div_ll(n, 256), 256, 0, (cudaStream_t)stream>>>(p, g, m, v, n, lr, beta1, beta2, eps, bc1, sqrtf(bc2), gscale, gscale_dev);
  return check_launch("adam_step");
}

int b200asr_sumsq(const float* g, long long n, float* out, b200asr_stream_t stream) {
  B200_REQUIRE(g && out, B200ASR_BAD_ARG, "sumsq: null pointer");
  if (n <= 0) return B200ASR_OK;
  long long blocks = ceil_div_ll(n, 256 * 8);
  int cap = device_sm_count() * 8;
  const int nb = (int)(blocks < cap ? blocks : cap);
  cudaStream_t st = (cudaStream_t)stream;
  float* part = (float*)stream_scratch(sizeof(float) * nb, st);
  if (!part) return B200ASR_CUDA_ERROR;
  sumsq_kernel<<<nb, 256, 0, st>>>(g, n, part);
  int rc = check_launch("sumsq");
  return rc ? rc : reduce_parts(part, nb, 1, 1, out, 1, st);
}

int b200asr_grad_scale(const float* g, long long n, const float* n_tokens, float max_norm, float* scratch, float* out,
                       b200asr_stream_t stream) {
  B200_REQUIRE(n_tokens && out && (max_norm <= 0.f || (g && scratch)), B200ASR_BAD_ARG, "grad_scale: null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  if (max_norm > 0.f) {
    cudaMemsetAsync(scratch, 0, sizeof(float), st);
    if (int rc = b200asr_sumsq(g, n, scratch, stream)) return rc;
  }
  grad_scale_kernel<<<1, 1, 0, st>>>(n_tokens, max_norm > 0.f ? scratch : nullptr, max_norm, out);
  return check_launch("grad_scale");
}

int b200asr_permute_cols_cf(const float* src, float* dst, int rows, int C, int F, int inverse, b200asr_stream_t stream) {
  B200_REQUIRE(src && dst && src != dst, B200ASR_BAD_ARG, "permute_cols_cf: bad arguments");
  long long n = (long long)rows * C * F;
  if (n <= 0) return B200ASR_OK;
  permute_cols_kernel<<<(unsigned)ceil_div_ll(n, 256), 256, 0, (cudaStream_t)stream>>>(src, dst, rows, C, F, inverse);
  return check_launch("permute_cols_cf");
}

}  // extern "C"
