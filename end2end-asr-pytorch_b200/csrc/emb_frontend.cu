// emb_cnn front end (models/asr/transformer.py:33-40): generic strided NCHW convolution (direct form),
// BatchNorm2d with batch statistics fused with the Hardtanh clamp, and the (B,C,F,T)->(B,T,C*F) flatten.
// This path only serves the emb_cnn configuration (BASELINE cfg3).  The convolutions here are the direct kernels coalesced
// along W (precision 0, exact fp32); the tensor-core modes run them as implicit GEMMs (tc_emb.cu).  The BatchNorm / clamp
// and flatten kernels serve both.
#include "../../include/b200asr.h"
#include "common.cuh"

namespace b200asr {

struct ConvG { int B, Ci, H, W, Co, KH, KW, SH, SW, PH, PW, OH, OW; };

__global__ void conv2d_fwd_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ bias,
                                  float* __restrict__ y, ConvG g) {
  long long n = (long long)g.B * g.Co * g.OH * g.OW;
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  int ow = (int)(i % g.OW); long long r = i / g.OW;
  int oh = (int)(r % g.OH); r /= g.OH;
  int co = (int)(r % g.Co); int b = (int)(r / g.Co);
  float acc = bias ? bias[co] : 0.f;
  for (int ci = 0; ci < g.Ci; ci++) {
    const float* xp = x + ((size_t)b * g.Ci + ci) * g.H * g.W;
    const float* wp = w + ((size_t)co * g.Ci + ci) * g.KH * g.KW;
    for (int kh = 0; kh < g.KH; kh++) {
      int ih = oh * g.SH - g.PH + kh;
      if (ih < 0 || ih >= g.H) continue;
      for (int kw = 0; kw < g.KW; kw++) {
        int iw = ow * g.SW - g.PW + kw;
        if (iw < 0 || iw >= g.W) continue;
        acc = fmaf(xp[(size_t)ih * g.W + iw], wp[kh * g.KW + kw], acc);
      }
    }
  }
  y[i] = acc;
}

__global__ void conv2d_bwd_data_kernel(const float* __restrict__ dy, const float* __restrict__ w, float* __restrict__ dx, ConvG g) {
  long long n = (long long)g.B * g.Ci * g.H * g.W;
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  int iw = (int)(i % g.W); long long r = i / g.W;
  int ih = (int)(r % g.H); r /= g.H;
  int ci = (int)(r % g.Ci); int b = (int)(r / g.Ci);
  float acc = 0.f;
  for (int kh = 0; kh < g.KH; kh++) {
    int th = ih + g.PH - kh;
    if (th < 0 || th % g.SH) continue;
    int oh = th / g.SH;
    if (oh >= g.OH) continue;
    for (int kw = 0; kw < g.KW; kw++) {
      int tw = iw + g.PW - kw;
      if (tw < 0 || tw % g.SW) continue;
      int ow = tw / g.SW;
      if (ow >= g.OW) continue;
      for (int co = 0; co < g.Co; co++)
        acc = fmaf(dy[(((size_t)b * g.Co + co) * g.OH + oh) * g.OW + ow], w[(((size_t)co * g.Ci + ci) * g.KH + kh) * g.KW + kw], acc);
    }
  }
  dx[i] = acc;
}

// one CTA per (co, ci, kh): threads run along ow (coalesced dy / x reads), each keeps the KW partial sums of its columns in
// registers while looping over (b, oh); block reduction at the end.  KW <= 16.
__global__ void __launch_bounds__(128) conv2d_bwd_weight_kernel(const float* __restrict__ dy, const float* __restrict__ x,
                                                                float* __restrict__ dw, ConvG g) {
  __shared__ float red[4][16];
  int i = blockIdx.x;
  const int kh = i % g.KH; i /= g.KH;
  const int ci = i % g.Ci; const int co = i / g.Ci;
  float acc[16];
#pragma unroll
  for (int k = 0; k < 16; k++) acc[k] = 0.f;
  for (int b = 0; b < g.B; b++) {
    const float* dyb = dy + ((size_t)b * g.Co + co) * g.OH * g.OW;
    const float* xb = x + ((size_t)b * g.Ci + ci) * g.H * g.W;
    for (int oh = 0; oh < g.OH; oh++) {
      const int ih = oh * g.SH - g.PH + kh;
      if (ih < 0 || ih >= g.H) continue;
      const float* xrow = xb + (size_t)ih * g.W;
      for (int ow = threadIdx.x; ow < g.OW; ow += blockDim.x) {
        const float gv = dyb[(size_t)oh * g.OW + ow];
        const int iw0 = ow * g.SW - g.PW;
#pragma unroll
        for (int k = 0; k < 16; k++) {
          const int iw = iw0 + k;
          if (k < g.KW && iw >= 0 && iw < g.W) acc[k] = fmaf(gv, xrow[iw], acc[k]);
        }
      }
    }
  }
#pragma unroll
  for (int k = 0; k < 16; k++) {
    float v = warp_sum(acc[k]);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5][k] = v;
  }
  __syncthreads();
  if (threadIdx.x < g.KW)
    dw[(((size_t)co * g.Ci + ci) * g.KH + kh) * g.KW + threadIdx.x] = red[0][threadIdx.x] + red[1][threadIdx.x] + red[2][threadIdx.x] + red[3][threadIdx.x];
}

// one CTA per output channel: dbias[co] = sum dy
__global__ void __launch_bounds__(256) conv2d_bias_grad_kernel(const float* __restrict__ dy, float* __restrict__ dbias, int B, int Co, int HW) {
  __shared__ float red[8];
  int co = blockIdx.x;
  float s = 0.f;
  for (long long j = threadIdx.x; j < (long long)B * HW; j += blockDim.x) {
    int b = (int)(j / HW); int k = (int)(j % HW);
    s += dy[((size_t)b * Co + co) * HW + k];
  }
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) { float t = 0.f; for (int w = 0; w < 8; w++) t += red[w]; dbias[co] = t; }
}

__device__ __forceinline__ float block_sum256(float v, float* red) {
  v = warp_sum(v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float t = 0.f;
#pragma unroll
  for (int w = 0; w < 8; w++) t += red[w];
  return t;
}

// BatchNorm2d + Hardtanh (models/asr/transformer.py:34-35,38-39).  training != 0: batch statistics (biased variance for the
// normalisation, as ATen), and -- when the running buffers are given -- the nn.BatchNorm2d state update
//   running_mean <- (1-m) running_mean + m mean,   running_var <- (1-m) running_var + m var * n/(n-1),   num_batches_tracked += 1.
// training == 0 (model.eval(), the reference's validation loop trainer.py:123): normalise with the running statistics.
// Tensors are [B, C, H, W] with a ROW PITCH per tensor (>= W; the implicit-GEMM convolutions need pitches that are
// multiples of 4 floats); a warp walks one row, the block's warps stride over the B*H rows of channel c.
struct BnIdx {
  int B, C, H, W;
  __device__ __forceinline__ size_t at(int row, int w, int c, int pitch) const {      // row = b * H + h
    return (((size_t)(row / H) * C + c) * H + (row % H)) * pitch + w;
  }
};

// Grid = (BN_SPLITS x C): the B*H rows of a channel are cut into BN_SPLITS contiguous ranges, one block each (32 channels
// alone would leave all but 32 SMs idle).  Pass 1 writes one partial per block -- (count, mean, M2) of its range, each
// from a two-pass sum inside the block; pass 2 merges the partials of its channel (Chan et al.'s pairwise update, fixed
// order => deterministic), and applies.  ws: [C][BN_SPLITS][4] floats.
constexpr int BN_SPLITS = 32;

struct BnRange { int r0, r1; };
__device__ __forceinline__ BnRange bn_range(int rows) {
  const int per = (rows + BN_SPLITS - 1) / BN_SPLITS;
  const int r0 = min(rows, (int)blockIdx.x * per);
  return BnRange{r0, min(rows, r0 + per)};
}

__global__ void __launch_bounds__(256) bn_stats_kernel(const float* __restrict__ x, float* __restrict__ ws, BnIdx g, int xp) {
  __shared__ float red[8];
  const int c = blockIdx.y, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const BnRange rr = bn_range(g.B * g.H);
  const float cnt = (float)(rr.r1 - rr.r0) * (float)g.W;
  float s = 0.f;
  for (int r = rr.r0 + warp; r < rr.r1; r += 8)
    for (int w = lane; w < g.W; w += 32) s += x[g.at(r, w, c, xp)];
  const float mean = cnt > 0.f ? block_sum256(s, red) / cnt : 0.f;
  float q = 0.f;
  for (int r = rr.r0 + warp; r < rr.r1; r += 8)                   // the block's range was just read: L1 / L2 hits
    for (int w = lane; w < g.W; w += 32) { const float d = x[g.at(r, w, c, xp)] - mean; q += d * d; }
  q = block_sum256(q, red);
  if (threadIdx.x == 0) {
    float* o = ws + ((size_t)c * BN_SPLITS + blockIdx.x) * 4;
    o[0] = cnt; o[1] = mean; o[2] = q;
  }
}

// merge the BN_SPLITS partials of channel c (every thread computes the same values)
__device__ __forceinline__ void bn_merge(const float* __restrict__ ws, int c, float& mean, float& var) {
  float n = 0.f, m = 0.f, M2 = 0.f;
  for (int s = 0; s < BN_SPLITS; s++) {
    const float* o = ws + ((size_t)c * BN_SPLITS + s) * 4;
    const float nb = o[0];
    if (nb <= 0.f) continue;
    const float d = o[1] - m, nn = n + nb;
    m += d * (nb / nn);
    M2 += o[2] + d * d * (n * nb / nn);
    n = nn;
  }
  mean = m;
  var = n > 0.f ? M2 / n : 0.f;
}

__global__ void __launch_bounds__(256) bn_clamp_fwd_kernel(const float* __restrict__ x, const float* __restrict__ gamma,
                                                           const float* __restrict__ beta, float* __restrict__ y,
                                                           float* __restrict__ mean_out, float* __restrict__ invstd_out,
                                                           float* __restrict__ running_mean, float* __restrict__ running_var,
                                                           long long* __restrict__ num_batches, const float* __restrict__ ws, BnIdx g,
                                                           int xp, int yp, float eps, float momentum, int training, float lo, float hi) {
  const int c = blockIdx.y, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int rows = g.B * g.H;
  const long long n = (long long)rows * g.W;
  float mean, invstd;
  if (training) {
    float var;
    bn_merge(ws, c, mean, var);
    invstd = rsqrtf(var + eps);
    if (blockIdx.x == 0 && threadIdx.x == 0 && running_mean && running_var) {
      running_mean[c] = (1.f - momentum) * running_mean[c] + momentum * mean;
      const float unbiased = n > 1 ? var * ((float)n / (float)(n - 1)) : var;
      running_var[c] = (1.f - momentum) * running_var[c] + momentum * unbiased;
      if (c == 0 && num_batches) *num_batches += 1;
    }
  } else {
    mean = running_mean[c];
    invstd = rsqrtf(running_var[c] + eps);
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) { mean_out[c] = mean; invstd_out[c] = invstd; }
  const float ga = gamma[c], be = beta[c];
  const BnRange rr = bn_range(rows);
  for (int r = rr.r0 + warp; r < rr.r1; r += 8)
    for (int w = lane; w < g.W; w += 32) {
      const float v = (x[g.at(r, w, c, xp)] - mean) * invstd * ga + be;
      y[g.at(r, w, c, yp)] = fminf(fmaxf(v, lo), hi);
    }
}

// backward pass 1: per-block partial sums of g = dy * [lo < y < hi] and g * xhat
__global__ void __launch_bounds__(256) bn_bwd_sums_kernel(const float* __restrict__ dy, const float* __restrict__ x,
                                                          const float* __restrict__ y, const float* __restrict__ mean_in,
                                                          const float* __restrict__ invstd_in, float* __restrict__ ws, BnIdx g, int dyp,
                                                          int xp, int yp, float lo, float hi) {
  __shared__ float red[8];
  const int c = blockIdx.y, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const float mean = mean_in[c], invstd = invstd_in[c];
  const BnRange rr = bn_range(g.B * g.H);
  float s1 = 0.f, s2 = 0.f;
  for (int r = rr.r0 + warp; r < rr.r1; r += 8)
    for (int w = lane; w < g.W; w += 32) {
      const float yv = y[g.at(r, w, c, yp)];
      const float gg = (yv > lo && yv < hi) ? dy[g.at(r, w, c, dyp)] : 0.f;
      const float xh = (x[g.at(r, w, c, xp)] - mean) * invstd;
      s1 += gg; s2 += gg * xh;
    }
  s1 = block_sum256(s1, red);
  s2 = block_sum256(s2, red);
  if (threadIdx.x == 0) {
    float* o = ws + ((size_t)c * BN_SPLITS + blockIdx.x) * 4;
    o[0] = s1; o[1] = s2;
  }
}

__global__ void __launch_bounds__(256) bn_clamp_bwd_kernel(const float* __restrict__ dy, const float* __restrict__ x,
                                                           const float* __restrict__ y, const float* __restrict__ gamma,
                                                           const float* __restrict__ mean_in, const float* __restrict__ invstd_in,
                                                           float* __restrict__ dx, float* __restrict__ dgamma, float* __restrict__ dbeta,
                                                           const float* __restrict__ ws, BnIdx g, int dyp, int xp, int yp, int dxp,
                                                           int training, float lo, float hi) {
  const int c = blockIdx.y, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int rows = g.B * g.H;
  const long long n = (long long)rows * g.W;
  const float mean = mean_in[c], invstd = invstd_in[c], ga = gamma[c];
  float s1 = 0.f, s2 = 0.f;
  for (int s = 0; s < BN_SPLITS; s++) {                          // fixed order: deterministic
    const float* o = ws + ((size_t)c * BN_SPLITS + s) * 4;
    s1 += o[0]; s2 += o[1];
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) { dbeta[c] = s1; dgamma[c] = s2; }
  const float inv_n = training ? 1.f / (float)n : 0.f;      // eval mode: the statistics are constants of the graph
  const BnRange rr = bn_range(rows);
  for (int r = rr.r0 + warp; r < rr.r1; r += 8)
    for (int w = lane; w < g.W; w += 32) {
      const float yv = y[g.at(r, w, c, yp)];
      const float gg = (yv > lo && yv < hi) ? dy[g.at(r, w, c, dyp)] : 0.f;
      const float xh = (x[g.at(r, w, c, xp)] - mean) * invstd;
      dx[g.at(r, w, c, dxp)] = ga * invstd * (gg - s1 * inv_n - xh * s2 * inv_n);
    }
}

// y[b][t][c*F+f] = x[b][c][f][t]  (32x32 smem transpose over (cf, t))
__global__ void flatten_bcft_kernel(const float* __restrict__ src, float* __restrict__ dst, int CF, int T, int to_btk) {
  __shared__ float tile[32][33];
  const int b = blockIdx.z;
  const int k0 = blockIdx.y * 32, t0 = blockIdx.x * 32;
  const float* s = src + (size_t)b * CF * T;
  float* d = dst + (size_t)b * CF * T;
  if (to_btk) {          // src [CF][T] -> dst [T][CF]
    for (int i = threadIdx.y; i < 32; i += 8) {
      int k = k0 + i, t = t0 + threadIdx.x;
      tile[i][threadIdx.x] = (k < CF && t < T) ? s[(size_t)k * T + t] : 0.f;
    }
    __syncthreads();
    for (int i = threadIdx.y; i < 32; i += 8) {
      int t = t0 + i, k = k0 + threadIdx.x;
      if (t < T && k < CF) d[(size_t)t * CF + k] = tile[threadIdx.x][i];
    }
  } else {               // src [T][CF] -> dst [CF][T]
    for (int i = threadIdx.y; i < 32; i += 8) {
      int t = t0 + i, k = k0 + threadIdx.x;
      tile[i][threadIdx.x] = (t < T && k < CF) ? s[(size_t)t * CF + k] : 0.f;
    }
    __syncthreads();
    for (int i = threadIdx.y; i < 32; i += 8) {
      int k = k0 + i, t = t0 + threadIdx.x;
      if (k < CF && t < T) d[(size_t)k * T + t] = tile[threadIdx.x][i];
    }
  }
}

static int make_geom(ConvG& g, int B, int Ci, int H, int W, int Co, int KH, int KW, int SH, int SW, int PH, int PW) {
  B200_REQUIRE(B > 0 && Ci > 0 && Co > 0 && KH > 0 && KW > 0 && SH > 0 && SW > 0 && PH >= 0 && PW >= 0, B200ASR_BAD_SHAPE, "conv2d: bad geometry");
  g = ConvG{B, Ci, H, W, Co, KH, KW, SH, SW, PH, PW, (H + 2 * PH - KH) / SH + 1, (W + 2 * PW - KW) / SW + 1};
  B200_REQUIRE(g.OH > 0 && g.OW > 0, B200ASR_BAD_SHAPE, "conv2d: empty output (H=%d W=%d)", H, W);
  return B200ASR_OK;
}

}  // namespace b200asr

using namespace b200asr;

extern "C" {

int b200asr_conv2d_fwd(const float* x, const float* w, const float* bias, float* y, int B, int Ci, int H, int W, int Co,
                       int KH, int KW, int SH, int SW, int PH, int PW, b200asr_stream_t stream) {
  B200_REQUIRE(x && w && y, B200ASR_BAD_ARG, "conv2d_fwd: null pointer");
  ConvG g; int rc = make_geom(g, B, Ci, H, W, Co, KH, KW, SH, SW, PH, PW); if (rc) return rc;
  long long n = (long long)B * Co * g.OH * g.OW;
  conv2d_fwd_kernel<<<(unsigned)ceil_div_ll(n, 256), 256, 0, (cudaStream_t)stream>>>(x, w, bias, y, g);
  return check_launch("conv2d_fwd");
}

int b200asr_conv2d_bwd_data(const float* dy, const float* w, float* dx, int B, int Ci, int H, int W, int Co, int KH, int KW,
                            int SH, int SW, int PH, int PW, b200asr_stream_t stream) {
  B200_REQUIRE(dy && w && dx, B200ASR_BAD_ARG, "conv2d_bwd_data: null pointer");
  ConvG g; int rc = make_geom(g, B, Ci, H, W, Co, KH, KW, SH, SW, PH, PW); if (rc) return rc;
  long long n = (long long)B * Ci * H * W;
  conv2d_bwd_data_kernel<<<(unsigned)ceil_div_ll(n, 256), 256, 0, (cudaStream_t)stream>>>(dy, w, dx, g);
  return check_launch("conv2d_bwd_data");
}

int b200asr_conv2d_bwd_weight(const float* dy, const float* x, float* dw, float* dbias, int B, int Ci, int H, int W, int Co,
                              int KH, int KW, int SH, int SW, int PH, int PW, b200asr_stream_t stream) {
  B200_REQUIRE(dy && x && dw, B200ASR_BAD_ARG, "conv2d_bwd_weight: null pointer");
  ConvG g; int rc = make_geom(g, B, Ci, H, W, Co, KH, KW, SH, SW, PH, PW); if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  B200_REQUIRE(KW <= 16, B200ASR_BAD_SHAPE, "conv2d_bwd_weight: KW=%d > 16", KW);
  conv2d_bwd_weight_kernel<<<Co * Ci * KH, 128, 0, st>>>(dy, x, dw, g);
  rc = check_launch("conv2d_bwd_weight"); if (rc) return rc;
  if (dbias) { conv2d_bias_grad_kernel<<<Co, 256, 0, st>>>(dy, dbias, B, Co, g.OH * g.OW); return check_launch("conv2d_bias_grad"); }
  return B200ASR_OK;
}

size_t b200asr_bn_ws_bytes(int C) { return C > 0 ? sizeof(float) * 4 * BN_SPLITS * (size_t)C : 0; }

int b200asr_bn_clamp_fwd(const float* x, const float* gamma, const float* beta, float* y, float* mean, float* invstd,
                         float* running_mean, float* running_var, long long* num_batches_tracked, float* ws, int B, int C, int H,
                         int W, int x_pitch, int y_pitch, float eps, float momentum, int training, float lo, float hi,
                         b200asr_stream_t stream) {
  B200_REQUIRE(x && gamma && beta && y && mean && invstd && ws && B > 0 && C > 0 && H > 0 && W > 0 && x_pitch >= W && y_pitch >= W,
               B200ASR_BAD_ARG, "bn_clamp_fwd: bad arguments");
  B200_REQUIRE(C <= 65535, B200ASR_BAD_SHAPE, "bn_clamp_fwd: at most 65535 channels");
  B200_REQUIRE(training || (running_mean && running_var), B200ASR_BAD_ARG, "bn_clamp_fwd: eval mode needs the running statistics");
  cudaStream_t st = (cudaStream_t)stream;
  const dim3 grid(BN_SPLITS, C);
  if (training) {
    bn_stats_kernel<<<grid, 256, 0, st>>>(x, ws, BnIdx{B, C, H, W}, x_pitch);
    note_launch(1);
  }
  bn_clamp_fwd_kernel<<<grid, 256, 0, st>>>(x, gamma, beta, y, mean, invstd, running_mean, running_var, num_batches_tracked, ws,
                                            BnIdx{B, C, H, W}, x_pitch, y_pitch, eps, momentum, training, lo, hi);
  return check_launch("bn_clamp_fwd");
}

int b200asr_bn_clamp_bwd(const float* dy, const float* x, const float* y, const float* gamma, const float* mean,
                         const float* invstd, float* dx, float* dgamma, float* dbeta, float* ws, int B, int C, int H, int W,
                         int dy_pitch, int x_pitch, int y_pitch, int dx_pitch, int training, float lo, float hi,
                         b200asr_stream_t stream) {
  B200_REQUIRE(dy && x && y && gamma && mean && invstd && dx && dgamma && dbeta && ws, B200ASR_BAD_ARG, "bn_clamp_bwd: null pointer");
  B200_REQUIRE(dy_pitch >= W && x_pitch >= W && y_pitch >= W && dx_pitch >= W, B200ASR_BAD_ARG, "bn_clamp_bwd: row pitches must cover W");
  B200_REQUIRE(C <= 65535, B200ASR_BAD_SHAPE, "bn_clamp_bwd: at most 65535 channels");
  cudaStream_t st = (cudaStream_t)stream;
  const dim3 grid(BN_SPLITS, C);
  bn_bwd_sums_kernel<<<grid, 256, 0, st>>>(dy, x, y, mean, invstd, ws, BnIdx{B, C, H, W}, dy_pitch, x_pitch, y_pitch, lo, hi);
  note_launch(1);
  bn_clamp_bwd_kernel<<<grid, 256, 0, st>>>(dy, x, y, gamma, mean, invstd, dx, dgamma, dbeta, ws, BnIdx{B, C, H, W}, dy_pitch, x_pitch,
                                            y_pitch, dx_pitch, training, lo, hi);
  return check_launch("bn_clamp_bwd");
}

int b200asr_flatten_bcft_fwd(const float* x, float* y, int B, int C, int F, int T, b200asr_stream_t stream) {
  B200_REQUIRE(x && y && B > 0, B200ASR_BAD_ARG, "flatten_bcft_fwd: bad arguments");
  dim3 grid(ceil_div(T, 32), ceil_div(C * F, 32), B);
  flatten_bcft_kernel<<<grid, dim3(32, 8), 0, (cudaStream_t)stream>>>(x, y, C * F, T, 1);
  return check_launch("flatten_bcft_fwd");
}

int b200asr_flatten_bcft_bwd(const float* dy, float* dx, int B, int C, int F, int T, b200asr_stream_t stream) {
  B200_REQUIRE(dy && dx && B > 0, B200ASR_BAD_ARG, "flatten_bcft_bwd: bad arguments");
  dim3 grid(ceil_div(T, 32), ceil_div(C * F, 32), B);
  flatten_bcft_kernel<<<grid, dim3(32, 8), 0, (cudaStream_t)stream>>>(dy, dx, C * F, T, 0);
  return check_launch("flatten_bcft_bwd");
}

}  // extern "C"
