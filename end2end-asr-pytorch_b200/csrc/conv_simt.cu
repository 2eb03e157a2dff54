// VGG front end on CUDA cores (precision 0), channels-last [B,T,F,C] activations.
//   conv3x3_c1_*    : first layer (C_in = 1) -- store-bound; one thread = one pixel x 4 output channels,
//                     a warp writes 512 contiguous bytes.
//   conv3x3_igemm   : implicit GEMM (pixels x Cout x 9*Cin), 128-pixel tiles, shared by forward and dgrad
//                     (dgrad = same kernel on dy with flipped/transposed weights).
//   conv3x3_wgrad   : per-tap [Cin x P] * [P x Cout] with the pixel axis split over CTAs (atomics).
//   maxpool2x2      : floor-mode pooling and its gradient (first-max routing, optional ReLU mask).
#include "../../include/b200asr.h"
#include "common.cuh"
#include "kernels.h"

namespace b200asr {

// ------------------------------------------------------------------------------------------------ conv1
// x [B,F,T] -> y [B,T,F,Co]; weights w[Co][1][3(f)][3(t)].  A CTA owns a 32 (time) x 8 (freq) pixel tile: the input patch
// with halo (10 x 34 floats) is staged in shared memory with loads coalesced along time, and each thread owns one channel
// quad, so a warp stores 2 pixels x 256 B = 512 contiguous bytes.  Store-bound by design (1.06 GB at cfg2).
constexpr int C1_TT = 32, C1_TF = 8;

__global__ void __launch_bounds__(256) conv3x3_c1_fwd_kernel(const float* __restrict__ x, const float* __restrict__ w,
                                                             const float* __restrict__ bias, float* __restrict__ y,
                                                             int B, int F, int T, int Co, int relu) {
  __shared__ float patch[C1_TF + 2][C1_TT + 2 + 1];
  const int cqs = Co >> 2;
  const int cq = threadIdx.x % cqs;
  const int slot = threadIdx.x / cqs;
  const int slots = blockDim.x / cqs;
  const int t0 = blockIdx.x * C1_TT, f0 = blockIdx.y * C1_TF, b = blockIdx.z;
  const float* xb = x + (size_t)b * F * T;
  for (int i = threadIdx.x; i < (C1_TF + 2) * (C1_TT + 2); i += blockDim.x) {
    const int pf = i / (C1_TT + 2), pt = i - pf * (C1_TT + 2);
    const int ff = f0 + pf - 1, tt = t0 + pt - 1;
    patch[pf][pt] = (ff >= 0 && ff < F && tt >= 0 && tt < T) ? xb[(size_t)ff * T + tt] : 0.f;
  }
  float wr[4][9], br[4];
#pragma unroll
  for (int c = 0; c < 4; c++) {
    br[c] = bias ? bias[cq * 4 + c] : 0.f;
#pragma unroll
    for (int t = 0; t < 9; t++) wr[c][t] = w[(cq * 4 + c) * 9 + t];
  }
  __syncthreads();
  for (int px = slot; px < C1_TT * C1_TF; px += slots) {      // pixel order: freq fastest -> contiguous output
    const int tl = px / C1_TF, fl = px - tl * C1_TF;
    const int t = t0 + tl, f = f0 + fl;
    if (t >= T || f >= F) continue;
    float o[4] = {br[0], br[1], br[2], br[3]};
#pragma unroll
    for (int df = 0; df < 3; df++)
#pragma unroll
      for (int dt = 0; dt < 3; dt++) {
        const float v = patch[fl + df][tl + dt];
#pragma unroll
        for (int c = 0; c < 4; c++) o[c] = fmaf(v, wr[c][df * 3 + dt], o[c]);
      }
    if (relu) { o[0] = fmaxf(o[0], 0.f); o[1] = fmaxf(o[1], 0.f); o[2] = fmaxf(o[2], 0.f); o[3] = fmaxf(o[3], 0.f); }
    *reinterpret_cast<float4*>(y + (((size_t)b * T + t) * F + f) * Co + cq * 4) = make_float4(o[0], o[1], o[2], o[3]);
  }
}

// dw[Co][9] += sum_p dy[p][co] * x[p + tap]; dbias[co] += sum_p dy[p][co]; same tiling, grid-stride over tiles
// part[block][10 * Co]: this block's [9 * Co] weight-gradient sums (co * 9 + tap) followed by its [Co] bias sums
__global__ void __launch_bounds__(256) conv3x3_c1_wgrad_kernel(const float* __restrict__ x, const float* __restrict__ dy,
                                                               float* __restrict__ part, int B, int F, int T, int Co) {
  extern __shared__ float red[];   // [slots][Co*10] (also reused for nothing else)
  __shared__ float patch[C1_TF + 2][C1_TT + 2 + 1];
  const int cqs = Co >> 2;
  const int cq = threadIdx.x % cqs;
  const int slot = threadIdx.x / cqs;
  const int slots = blockDim.x / cqs;
  float acc[4][10];
#pragma unroll
  for (int c = 0; c < 4; c++)
#pragma unroll
    for (int k = 0; k < 10; k++) acc[c][k] = 0.f;
  const int ntt = (T + C1_TT - 1) / C1_TT, nft = (F + C1_TF - 1) / C1_TF;
  const int ntiles = ntt * nft * B;
  for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int ft = tile % nft, r = tile / nft;
    const int tti = r % ntt, b = r / ntt;
    const int t0 = tti * C1_TT, f0 = ft * C1_TF;
    const float* xb = x + (size_t)b * F * T;
    __syncthreads();
    for (int i = threadIdx.x; i < (C1_TF + 2) * (C1_TT + 2); i += blockDim.x) {
      const int pf = i / (C1_TT + 2), pt = i - pf * (C1_TT + 2);
      const int ff = f0 + pf - 1, tt = t0 + pt - 1;
      patch[pf][pt] = (ff >= 0 && ff < F && tt >= 0 && tt < T) ? xb[(size_t)ff * T + tt] : 0.f;
    }
    __syncthreads();
    // four pixels per trip with all four dy loads issued first: one 16-byte load in flight per thread kept only ~2.4 MB
    // outstanding chip-wide and the kernel ran at 1.6 TB/s of its 1 GB dy stream (latency-bound, not bandwidth-bound)
    for (int px0 = slot; px0 < C1_TT * C1_TF; px0 += 4 * slots) {
      float4 g[4];
      int tl[4], fl[4];
#pragma unroll
      for (int u = 0; u < 4; u++) {
        const int px = px0 + u * slots;
        tl[u] = px / C1_TF; fl[u] = px - tl[u] * C1_TF;
        const int t = t0 + tl[u], f = f0 + fl[u];
        const bool ok = px < C1_TT * C1_TF && t < T && f < F;
        g[u] = ok ? __ldg(reinterpret_cast<const float4*>(dy + (((size_t)b * T + t) * F + f) * Co + cq * 4))
                  : make_float4(0.f, 0.f, 0.f, 0.f);
        if (!ok) { tl[u] = 0; fl[u] = 0; }
      }
#pragma unroll
      for (int u = 0; u < 4; u++) {
        const float gv[4] = {g[u].x, g[u].y, g[u].z, g[u].w};
#pragma unroll
        for (int df = 0; df < 3; df++)
#pragma unroll
          for (int dt = 0; dt < 3; dt++) {
            const float v = patch[fl[u] + df][tl[u] + dt];
#pragma unroll
            for (int c = 0; c < 4; c++) acc[c][df * 3 + dt] = fmaf(gv[c], v, acc[c][df * 3 + dt]);
          }
#pragma unroll
        for (int c = 0; c < 4; c++) acc[c][9] += gv[c];
      }
    }
  }
#pragma unroll
  for (int c = 0; c < 4; c++)
#pragma unroll
    for (int k = 0; k < 10; k++) red[(size_t)slot * Co * 10 + (cq * 4 + c) * 10 + k] = acc[c][k];
  __syncthreads();
  for (int i = threadIdx.x; i < Co * 10; i += blockDim.x) {
    float s = 0.f;
    for (int sl = 0; sl < slots; sl++) s += red[(size_t)sl * Co * 10 + i];
    int co = i / 10, k = i % 10;
    part[(size_t)blockIdx.x * Co * 10 + (k < 9 ? co * 9 + k : 9 * Co + co)] = s;
  }
}

// ------------------------------------------------------------------------------------------------ weight repacks
// fwd:   wr[tap][ci][co] = w[co][ci][tap]
// dgrad: wr[tap'][co][ci] = w[co][ci][8 - tap']   (tap' = flipped tap; rows = contraction channel)
__global__ void conv_repack_kernel(const float* __restrict__ w, float* __restrict__ wr, int Ci, int Co, int dgrad) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  int total = 9 * Ci * Co;
  if (i >= total) return;
  if (!dgrad) {
    int co = i % Co, ci = (i / Co) % Ci, tap = i / (Co * Ci);
    wr[i] = w[((size_t)co * Ci + ci) * 9 + tap];
  } else {
    int ci = i % Ci, co = (i / Ci) % Co, tap = i / (Co * Ci);
    wr[i] = w[((size_t)co * Ci + ci) * 9 + (8 - tap)];
  }
}
// K-major repacks for the tensor-core path (contraction channel contiguous):
// fwd:   wk[tap][co][ci] = w[co][ci][tap]
// dgrad: wk[tap'][ci][co] = w[co][ci][8 - tap']
// split != 0 additionally writes the 3xTF32 halves: wk[i] = rna_tf32(w), wk[total + i] = rna_tf32(w - hi)
__global__ void conv_repack_k_kernel(const float* __restrict__ w, float* __restrict__ wk, int Ci, int Co, int dgrad, int split) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  int total = 9 * Ci * Co;
  if (i >= total) return;
  float v;
  if (!dgrad) {
    int ci = i % Ci, co = (i / Ci) % Co, tap = i / (Co * Ci);
    v = w[((size_t)co * Ci + ci) * 9 + tap];
  } else {
    int co = i % Co, ci = (i / Co) % Ci, tap = i / (Co * Ci);
    v = w[((size_t)co * Ci + ci) * 9 + (8 - tap)];
  }
  if (split) {
    uint32_t u;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(u) : "f"(v));
    float hi = __uint_as_float(u);
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(u) : "f"(v - hi));
    wk[i] = hi;
    wk[total + i] = __uint_as_float(u);
  } else {
    wk[i] = v;
  }
}
// dw[co][ci][tap] = dwr[tap][ci][co]
__global__ void conv_unpack_wgrad_kernel(const float* __restrict__ dwr, float* __restrict__ dw, int Ci, int Co) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  int total = 9 * Ci * Co;
  if (i >= total) return;
  int tap = i % 9, ci = (i / 9) % Ci, co = i / (9 * Ci);
  dw[i] = dwr[((size_t)tap * Ci + ci) * Co + co];
}

// ------------------------------------------------------------------------------------------------ implicit GEMM
constexpr int CBM = 128, CBK = 16, CLD = 132;

// out[p][n] = act( sum_{tap,c} in[p + off(tap)][c] * wr[tap][c][n] + bias[n] ) (.* mask>0)
// in: [P, Cin] pixels (b,t,f order), wr: [9][Cin][Cout]
template <int BN>
__global__ void __launch_bounds__(256) conv3x3_igemm_kernel(const float* __restrict__ in, const float* __restrict__ wr,
                                                            const float* __restrict__ bias,
                                                            const float* __restrict__ mask, float* __restrict__ out,
                                                            int B, int T, int F, int Cin, int Cout, int relu) {
  __shared__ __align__(16) float As[2][CBK][CLD];
  __shared__ __align__(16) float Bs[2][CBK][BN + 4];
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const long long P = (long long)B * T * F;
  const long long p0 = (long long)blockIdx.y * CBM;
  const int n0 = blockIdx.x * BN;
  // this thread's two A rows (pixels) for the loads
  int rf[2], rt[2];
  bool rok[2];
  const int lrow[2] = {tid >> 2, (tid + 256) >> 2};
  const int kq = (tid & 3) * 4;
#pragma unroll
  for (int i = 0; i < 2; i++) {
    long long p = p0 + lrow[i];
    rok[i] = p < P;
    long long pp = rok[i] ? p : 0;
    rf[i] = (int)(pp % F);
    rt[i] = (int)((pp / F) % T);
  }
  constexpr int NJ = BN / 16;
  float acc[8][NJ];
#pragma unroll
  for (int i = 0; i < 8; i++)
#pragma unroll
    for (int j = 0; j < NJ; j++) acc[i][j] = 0.f;

  const int cchunks = Cin / CBK;
  const int nk = 9 * cchunks;
  float4 ra[2], rb[BN / 64];
  auto gload = [&](int kt) {
    const int tap = kt / cchunks, c0 = (kt - tap * cchunks) * CBK;
    const int df = tap / 3 - 1, dt = tap % 3 - 1;     // tap = kf*3 + kt, as in w[Co][Ci][kf(freq)][kt(time)]
#pragma unroll
    for (int i = 0; i < 2; i++) {
      float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
      int tt = rt[i] + dt, ff = rf[i] + df;
      if (rok[i] && tt >= 0 && tt < T && ff >= 0 && ff < F)
        z = *reinterpret_cast<const float4*>(in + (size_t)(p0 + lrow[i] + (long long)dt * F + df) * Cin + c0 + kq);
      ra[i] = z;
    }
    const float* wb = wr + ((size_t)tap * Cin + c0) * Cout + n0;
#pragma unroll
    for (int i = 0; i < BN / 64; i++) {
      int idx = tid + i * 256;
      int kk = idx / (BN / 4), nq = (idx % (BN / 4)) * 4;
      rb[i] = *reinterpret_cast<const float4*>(wb + (size_t)kk * Cout + nq);
    }
  };
  auto sstore = [&](int buf) {
#pragma unroll
    for (int i = 0; i < 2; i++) {
      As[buf][kq + 0][lrow[i]] = ra[i].x; As[buf][kq + 1][lrow[i]] = ra[i].y;
      As[buf][kq + 2][lrow[i]] = ra[i].z; As[buf][kq + 3][lrow[i]] = ra[i].w;
    }
#pragma unroll
    for (int i = 0; i < BN / 64; i++) {
      int idx = tid + i * 256;
      int kk = idx / (BN / 4), nq = (idx % (BN / 4)) * 4;
      *reinterpret_cast<float4*>(&Bs[buf][kk][nq]) = rb[i];
    }
  };
  gload(0);
  sstore(0);
  __syncthreads();
  for (int kt = 0; kt < nk; kt++) {
    const int cur = kt & 1;
    if (kt + 1 < nk) gload(kt + 1);
#pragma unroll
    for (int k = 0; k < CBK; k++) {
      float4 a0 = *reinterpret_cast<const float4*>(&As[cur][k][ty * 4]);
      float4 a1 = *reinterpret_cast<const float4*>(&As[cur][k][64 + ty * 4]);
      float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
      float b[NJ];
      float4 b0 = *reinterpret_cast<const float4*>(&Bs[cur][k][tx * 4]);
      b[0] = b0.x; b[1] = b0.y; b[2] = b0.z; b[3] = b0.w;
      if (NJ == 8) {
        float4 b1 = *reinterpret_cast<const float4*>(&Bs[cur][k][(BN / 2) + tx * 4]);
        b[NJ - 4] = b1.x; b[NJ - 3] = b1.y; b[NJ - 2] = b1.z; b[NJ - 1] = b1.w;
      }
#pragma unroll
      for (int i = 0; i < 8; i++)
#pragma unroll
        for (int j = 0; j < NJ; j++) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    if (kt + 1 < nk) sstore(cur ^ 1);
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 8; i++) {
    long long p = p0 + (i < 4 ? ty * 4 + i : 64 + ty * 4 + (i - 4));
    if (p >= P) continue;
#pragma unroll
    for (int jg = 0; jg < NJ / 4; jg++) {
      int col = n0 + (jg ? BN / 2 : 0) + tx * 4;
      float v[4];
#pragma unroll
      for (int j = 0; j < 4; j++) {
        float t = acc[i][jg * 4 + j];
        if (bias) t += bias[col + j];
        if (relu) t = fmaxf(t, 0.f);
        v[j] = t;
      }
      size_t off = (size_t)p * Cout + col;
      if (mask) {
        float4 m = *reinterpret_cast<const float4*>(mask + off);
        v[0] = m.x > 0.f ? v[0] : 0.f; v[1] = m.y > 0.f ? v[1] : 0.f;
        v[2] = m.z > 0.f ? v[2] : 0.f; v[3] = m.w > 0.f ? v[3] : 0.f;
      }
      *reinterpret_cast<float4*>(out + off) = make_float4(v[0], v[1], v[2], v[3]);
    }
  }
}

// dwr[tap][ci][co] += sum_{p in chunk} x[p + off(tap)][ci] * dy[p][co]
template <int BMC, int BNC>
__global__ void __launch_bounds__(256) conv3x3_wgrad_kernel(const float* __restrict__ x, const float* __restrict__ dy,
                                                            float* __restrict__ dwr, int B, int T, int F, int Ci,
                                                            int Co, int chunk) {
  __shared__ __align__(16) float As[2][CBK][BMC + 4];
  __shared__ __align__(16) float Bs[2][CBK][BNC + 4];
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int tap = blockIdx.z;
  const int df = tap / 3 - 1, dt = tap % 3 - 1;   // tap = kf*3 + kt
  const int tiles_n = Co / BNC;
  const int m0 = (blockIdx.x / tiles_n) * BMC, n0 = (blockIdx.x % tiles_n) * BNC;
  const long long P = (long long)B * T * F;
  const long long pbeg = (long long)blockIdx.y * chunk;
  const long long pend = min(P, pbeg + chunk);
  constexpr int NI = BMC / 16, NJ = BNC / 16;
  float acc[NI][NJ];
#pragma unroll
  for (int i = 0; i < NI; i++)
#pragma unroll
    for (int j = 0; j < NJ; j++) acc[i][j] = 0.f;
  constexpr int AV = BMC / 64, BV = BNC / 64;     // float4 per thread per tile (16 rows x BMC/4 quads / 256)
  float4 ra[AV], rb[BV];
  auto gload = [&](long long pk) {
#pragma unroll
    for (int i = 0; i < AV; i++) {
      int idx = tid + i * 256;
      int kk = idx / (BMC / 4), mq = (idx % (BMC / 4)) * 4;
      long long p = pk + kk;
      float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
      if (p < pend) {
        int f = (int)(p % F), t = (int)((p / F) % T);
        int tt = t + dt, ff = f + df;
        if (tt >= 0 && tt < T && ff >= 0 && ff < F)
          z = *reinterpret_cast<const float4*>(x + (size_t)(p + (long long)dt * F + df) * Ci + m0 + mq);
      }
      ra[i] = z;
    }
#pragma unroll
    for (int i = 0; i < BV; i++) {
      int idx = tid + i * 256;
      int kk = idx / (BNC / 4), nq = (idx % (BNC / 4)) * 4;
      long long p = pk + kk;
      rb[i] = (p < pend) ? *reinterpret_cast<const float4*>(dy + (size_t)p * Co + n0 + nq) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
  };
  auto sstore = [&](int buf) {
#pragma unroll
    for (int i = 0; i < AV; i++) {
      int idx = tid + i * 256;
      *reinterpret_cast<float4*>(&As[buf][idx / (BMC / 4)][(idx % (BMC / 4)) * 4]) = ra[i];
    }
#pragma unroll
    for (int i = 0; i < BV; i++) {
      int idx = tid + i * 256;
      *reinterpret_cast<float4*>(&Bs[buf][idx / (BNC / 4)][(idx % (BNC / 4)) * 4]) = rb[i];
    }
  };
  const int nk = (int)((pend - pbeg + CBK - 1) / CBK);
  if (nk > 0) { gload(pbeg); sstore(0); }
  __syncthreads();
  for (int kt = 0; kt < nk; kt++) {
    const int cur = kt & 1;
    if (kt + 1 < nk) gload(pbeg + (long long)(kt + 1) * CBK);
#pragma unroll
    for (int k = 0; k < CBK; k++) {
      float a[NI], b[NJ];
#pragma unroll
      for (int g = 0; g < NI / 4; g++) {
        float4 v = *reinterpret_cast<const float4*>(&As[cur][k][g * 64 + ty * 4]);
        a[g * 4 + 0] = v.x; a[g * 4 + 1] = v.y; a[g * 4 + 2] = v.z; a[g * 4 + 3] = v.w;
      }
#pragma unroll
      for (int g = 0; g < NJ / 4; g++) {
        float4 v = *reinterpret_cast<const float4*>(&Bs[cur][k][g * 64 + tx * 4]);
        b[g * 4 + 0] = v.x; b[g * 4 + 1] = v.y; b[g * 4 + 2] = v.z; b[g * 4 + 3] = v.w;
      }
#pragma unroll
      for (int i = 0; i < NI; i++)
#pragma unroll
        for (int j = 0; j < NJ; j++) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    if (kt + 1 < nk) sstore(cur ^ 1);
    __syncthreads();
  }
  float* o = dwr + (size_t)tap * Ci * Co;
#pragma unroll
  for (int i = 0; i < NI; i++) {
    int row = m0 + (i / 4) * 64 + ty * 4 + (i % 4);
#pragma unroll
    for (int j = 0; j < NJ; j++) {
      int col = n0 + (j / 4) * 64 + tx * 4 + (j % 4);
      atomicAdd(o + (size_t)row * Co + col, acc[i][j]);
    }
  }
}

// ------------------------------------------------------------------------------------------------ pooling
// which element of the 2x2 window carries the gradient: ATen scans the window freq-major -- (f, t), (f, t+1), (f+1, t),
// (f+1, t+1) = codes 0..3 -- and keeps the FIRST maximum; bit 2 is set when that maximum is not positive (a ReLU in front of
// the pooling then passes no gradient at all).  One byte per pooled element, written by the forward, read by the backward
// instead of the full-resolution activation.
__device__ __forceinline__ uint32_t pool_code(float a0, float a1, float a2, float a3) {
  int best = 0; float m = a0;
  if (a1 > m) { m = a1; best = 1; }
  if (a2 > m) { m = a2; best = 2; }
  if (a3 > m) { m = a3; best = 3; }
  return (uint32_t)best | (m > 0.f ? 0u : 4u);
}

__global__ void maxpool2x2_fwd_kernel(const float* __restrict__ x, float* __restrict__ y, uint8_t* __restrict__ idx, int B, int T, int F, int C) {
  const int T2 = T / 2, F2 = F / 2, C4 = C / 4;
  long long n = (long long)B * T2 * F2 * C4;
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  int c = (int)(i % C4) * 4;
  long long r = i / C4;
  int f2 = (int)(r % F2); r /= F2;
  int t2 = (int)(r % T2);
  int b = (int)(r / T2);
  const float* p = x + (((size_t)b * T + 2 * t2) * F + 2 * f2) * C + c;
  float4 a = *reinterpret_cast<const float4*>(p);
  float4 bq = *reinterpret_cast<const float4*>(p + C);
  float4 cq = *reinterpret_cast<const float4*>(p + (size_t)F * C);
  float4 d = *reinterpret_cast<const float4*>(p + (size_t)F * C + C);
  float4 o;
  o.x = fmaxf(fmaxf(a.x, bq.x), fmaxf(cq.x, d.x));
  o.y = fmaxf(fmaxf(a.y, bq.y), fmaxf(cq.y, d.y));
  o.z = fmaxf(fmaxf(a.z, bq.z), fmaxf(cq.z, d.z));
  o.w = fmaxf(fmaxf(a.w, bq.w), fmaxf(cq.w, d.w));
  const size_t po = (((size_t)b * T2 + t2) * F2 + f2) * C + c;
  *reinterpret_cast<float4*>(y + po) = o;
  if (idx)      // scan order: (f, t) = a, (f, t+1) = cq, (f+1, t) = bq, (f+1, t+1) = d
    *reinterpret_cast<uint32_t*>(idx + po) = pool_code(a.x, cq.x, bq.x, d.x) | (pool_code(a.y, cq.y, bq.y, d.y) << 8) |
                                             (pool_code(a.z, cq.z, bq.z, d.z) << 16) | (pool_code(a.w, cq.w, bq.w, d.w) << 24);
}

// one thread = one 2x2 window x 4 channels; writes all four dx positions (and zeroes are written for the odd tails
// by the tail kernel below).  ATen scans the window freq-major (h = freq outer, w = time inner) and keeps the first max.
// fp32 value -> (bf16 hi, bf16 lo) with hi + lo ~ x to 16 significant bits (the operand split of the bf16 kernels)
__device__ __forceinline__ void pair_of(float x, uint16_t& h, uint16_t& l) {
  const uint32_t r = __float_as_uint(x) + 0x8000u;
  h = (uint16_t)(r >> 16);
  const float lo = x - __uint_as_float(r & 0xFFFF0000u);
  l = (uint16_t)((__float_as_uint(lo) + 0x8000u) >> 16);
}
__device__ __forceinline__ void store_pairs4(uint16_t* __restrict__ hi, size_t lo_off, size_t idx, const float4& v) {
  uint16_t h[4], l[4];
  pair_of(v.x, h[0], l[0]); pair_of(v.y, h[1], l[1]); pair_of(v.z, h[2], l[2]); pair_of(v.w, h[3], l[3]);
  *reinterpret_cast<uint2*>(hi + idx) = make_uint2((uint32_t)h[0] | ((uint32_t)h[1] << 16), (uint32_t)h[2] | ((uint32_t)h[3] << 16));
  *reinterpret_cast<uint2*>(hi + lo_off + idx) = make_uint2((uint32_t)l[0] | ((uint32_t)l[1] << 16), (uint32_t)l[2] | ((uint32_t)l[3] << 16));
}

// dx16 (optional): the same gradient additionally as bf16 hi | lo pairs [2][B,T,F,C] -- the B operand of the convolution
// weight gradient in the bf16 modes arrives from there by TMA (tc_conv.cu WgradPairPolicy)
__global__ void maxpool2x2_bwd_kernel(const float* __restrict__ dy, const float* __restrict__ x, float* __restrict__ dx,
                                      uint16_t* __restrict__ dx16, int B, int T, int F, int C, int relu_mask) {
  const int T2 = T / 2, F2 = F / 2, C4 = C / 4;
  long long n = (long long)B * T2 * F2 * C4;
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  int c = (int)(i % C4) * 4;
  long long r = i / C4;
  int f2 = (int)(r % F2); r /= F2;
  int t2 = (int)(r % T2);
  int b = (int)(r / T2);
  const size_t base = (((size_t)b * T + 2 * t2) * F + 2 * f2) * C + c;
  const size_t o_f = C, o_t = (size_t)F * C;     // +1 in freq, +1 in time
  // scan order: (f0,t0), (f0,t1), (f1,t0), (f1,t1)
  const size_t offs[4] = {0, o_t, o_f, o_f + o_t};
  float4 v[4];
#pragma unroll
  for (int k = 0; k < 4; k++) v[k] = *reinterpret_cast<const float4*>(x + base + offs[k]);
  const float4 g = *reinterpret_cast<const float4*>(dy + (((size_t)b * T2 + t2) * F2 + f2) * C + c);
  float4 out[4];
  auto route = [&](float a0, float a1, float a2, float a3, float gg, float& o0, float& o1, float& o2, float& o3) {
    int best = 0; float m = a0;
    if (a1 > m) { m = a1; best = 1; }
    if (a2 > m) { m = a2; best = 2; }
    if (a3 > m) { m = a3; best = 3; }
    float keep = (!relu_mask || m > 0.f) ? gg : 0.f;
    o0 = best == 0 ? keep : 0.f; o1 = best == 1 ? keep : 0.f; o2 = best == 2 ? keep : 0.f; o3 = best == 3 ? keep : 0.f;
  };
  route(v[0].x, v[1].x, v[2].x, v[3].x, g.x, out[0].x, out[1].x, out[2].x, out[3].x);
  route(v[0].y, v[1].y, v[2].y, v[3].y, g.y, out[0].y, out[1].y, out[2].y, out[3].y);
  route(v[0].z, v[1].z, v[2].z, v[3].z, g.z, out[0].z, out[1].z, out[2].z, out[3].z);
  route(v[0].w, v[1].w, v[2].w, v[3].w, g.w, out[0].w, out[1].w, out[2].w, out[3].w);
#pragma unroll
  for (int k = 0; k < 4; k++) *reinterpret_cast<float4*>(dx + base + offs[k]) = out[k];
  if (dx16) {
    const size_t lo_off = (size_t)B * T * F * C;
#pragma unroll
    for (int k = 0; k < 4; k++) store_pairs4(dx16, lo_off, base + offs[k], out[k]);
  }
}
// the same routing from the forward's index bytes: reads dy and one byte per pooled element instead of the activation
__global__ void maxpool2x2_bwd_idx_kernel(const float* __restrict__ dy, const uint8_t* __restrict__ idx, float* __restrict__ dx,
                                          uint16_t* __restrict__ dx16, int B, int T, int F, int C, int relu_mask) {
  const int T2 = T / 2, F2 = F / 2, C4 = C / 4;
  long long n = (long long)B * T2 * F2 * C4;
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  int c = (int)(i % C4) * 4;
  long long r = i / C4;
  int f2 = (int)(r % F2); r /= F2;
  int t2 = (int)(r % T2);
  int b = (int)(r / T2);
  const size_t po = (((size_t)b * T2 + t2) * F2 + f2) * C + c;
  const float4 g = *reinterpret_cast<const float4*>(dy + po);
  const uint32_t codes = *reinterpret_cast<const uint32_t*>(idx + po);
  const size_t base = (((size_t)b * T + 2 * t2) * F + 2 * f2) * C + c;
  const size_t o_f = C, o_t = (size_t)F * C;
  const size_t offs[4] = {0, o_t, o_f, o_f + o_t};         // scan order, as in maxpool2x2_bwd_kernel
  const uint32_t dead = relu_mask ? 4u : 8u;                // bit 2 = "maximum not positive" counts only behind a ReLU
  const uint32_t c0 = codes & 7u, c1 = (codes >> 8) & 7u, c2 = (codes >> 16) & 7u, c3 = (codes >> 24) & 7u;
  float4 out[4];
#pragma unroll
  for (int k = 0; k < 4; k++) {
    out[k].x = (!(c0 & dead) && (c0 & 3u) == (uint32_t)k) ? g.x : 0.f;
    out[k].y = (!(c1 & dead) && (c1 & 3u) == (uint32_t)k) ? g.y : 0.f;
    out[k].z = (!(c2 & dead) && (c2 & 3u) == (uint32_t)k) ? g.z : 0.f;
    out[k].w = (!(c3 & dead) && (c3 & 3u) == (uint32_t)k) ? g.w : 0.f;
    *reinterpret_cast<float4*>(dx + base + offs[k]) = out[k];
  }
  if (dx16) {
    const size_t lo_off = (size_t)B * T * F * C;
#pragma unroll
    for (int k = 0; k < 4; k++) store_pairs4(dx16, lo_off, base + offs[k], out[k]);
  }
}
// zero the rows/cols that floor-mode pooling never reads (odd T or F): only those positions are visited
__global__ void maxpool2x2_bwd_tail_kernel(float* __restrict__ dx, uint16_t* __restrict__ dx16, int B, int T, int F, int C) {
  const int C4 = C / 4;
  const int odd_f = F & 1, odd_t = T & 1;
  const int Te = (T / 2) * 2;                                    // rows with t < Te only need the odd freq column
  const long long n_col = odd_f ? (long long)B * Te * C4 : 0;    // (b, t < Te, f = F-1)
  const long long n_row = odd_t ? (long long)B * F * C4 : 0;     // (b, t = T-1, all f)
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_col + n_row) return;
  int b, t, f, c;
  if (i < n_col) {
    c = (int)(i % C4) * 4; long long r = i / C4;
    t = (int)(r % Te); b = (int)(r / Te); f = F - 1;
  } else {
    i -= n_col;
    c = (int)(i % C4) * 4; long long r = i / C4;
    f = (int)(r % F); b = (int)(r / F); t = T - 1;
  }
  const size_t idx = (((size_t)b * T + t) * F + f) * C + c;
  *reinterpret_cast<float4*>(dx + idx) = make_float4(0.f, 0.f, 0.f, 0.f);
  if (dx16) {
    *reinterpret_cast<uint2*>(dx16 + idx) = make_uint2(0u, 0u);
    *reinterpret_cast<uint2*>(dx16 + (size_t)B * T * F * C + idx) = make_uint2(0u, 0u);
  }
}

__global__ void relu_bwd_kernel(const float* __restrict__ dy, const float* __restrict__ y, float* __restrict__ dx, long long n4) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n4) return;
  float4 g = reinterpret_cast<const float4*>(dy)[i];
  float4 v = reinterpret_cast<const float4*>(y)[i];
  g.x = v.x > 0.f ? g.x : 0.f; g.y = v.y > 0.f ? g.y : 0.f; g.z = v.z > 0.f ? g.z : 0.f; g.w = v.w > 0.f ? g.w : 0.f;
  reinterpret_cast<float4*>(dx)[i] = g;
}

// host-side launchers used by the API and (for precision 0) nothing else
int conv3x3_simt(const float* in, const float* wr, const float* bias, const float* mask, float* out, int B, int T, int F,
                 int Cin, int Cout, int relu, cudaStream_t st) {
  long long P = (long long)B * T * F;
  if (Cout % 128 == 0) {
    dim3 grid(Cout / 128, (unsigned)ceil_div_ll(P, CBM));
    conv3x3_igemm_kernel<128><<<grid, 256, 0, st>>>(in, wr, bias, mask, out, B, T, F, Cin, Cout, relu);
  } else {
    dim3 grid(Cout / 64, (unsigned)ceil_div_ll(P, CBM));
    conv3x3_igemm_kernel<64><<<grid, 256, 0, st>>>(in, wr, bias, mask, out, B, T, F, Cin, Cout, relu);
  }
  return check_launch("conv3x3_igemm");
}

int conv3x3_wgrad_simt(const float* x, const float* dy, float* dwr, int B, int T, int F, int Ci, int Co, cudaStream_t st) {
  long long P = (long long)B * T * F;
  int bm = (Ci % 128 == 0) ? 128 : 64, bn = (Co % 128 == 0) ? 128 : 64;
  int tiles = (Ci / bm) * (Co / bn);
  int sms = device_sm_count();
  long long want = ceil_div_ll(4LL * sms, 9LL * tiles);
  long long chunk = ceil_div_ll(ceil_div_ll(P, want < 1 ? 1 : want), CBK) * CBK;
  if (chunk < 1024) chunk = 1024;
  dim3 grid(tiles, (unsigned)ceil_div_ll(P, chunk), 9);
  if (bm == 128 && bn == 128) conv3x3_wgrad_kernel<128, 128><<<grid, 256, 0, st>>>(x, dy, dwr, B, T, F, Ci, Co, (int)chunk);
  else if (bm == 64 && bn == 128) conv3x3_wgrad_kernel<64, 128><<<grid, 256, 0, st>>>(x, dy, dwr, B, T, F, Ci, Co, (int)chunk);
  else if (bm == 128 && bn == 64) conv3x3_wgrad_kernel<128, 64><<<grid, 256, 0, st>>>(x, dy, dwr, B, T, F, Ci, Co, (int)chunk);
  else conv3x3_wgrad_kernel<64, 64><<<grid, 256, 0, st>>>(x, dy, dwr, B, T, F, Ci, Co, (int)chunk);
  return check_launch("conv3x3_wgrad");
}

}  // namespace b200asr

using namespace b200asr;

extern "C" {

size_t b200asr_conv3x3_ws_bytes(int Ci, int Co) { return sizeof(float) * 2 * 9 * (size_t)Ci * Co; }   // [hi | lo] weight halves

int b200asr_conv3x3_c1_fwd(const float* x, const float* w, const float* bias, float* y, int B, int F, int T, int Co,
                           int relu, b200asr_stream_t stream) {
  B200_REQUIRE(x && w && y, B200ASR_BAD_ARG, "conv3x3_c1_fwd: null pointer");
  B200_REQUIRE(Co % 4 == 0 && Co <= 1024 && 256 % (Co / 4) == 0, B200ASR_BAD_SHAPE, "conv3x3_c1_fwd: Co=%d unsupported", Co);
  B200_REQUIRE(aligned16(y), B200ASR_BAD_ALIGN, "conv3x3_c1_fwd: y alignment");
  long long P = (long long)B * T * F;
  if (P <= 0) return B200ASR_OK;
  B200_REQUIRE(B <= 65535 && ceil_div(F, C1_TF) <= 65535, B200ASR_BAD_SHAPE, "conv3x3_c1_fwd: grid too large");
  dim3 grid(ceil_div(T, C1_TT), ceil_div(F, C1_TF), B);
  conv3x3_c1_fwd_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(x, w, bias, y, B, F, T, Co, relu);
  return check_launch("conv3x3_c1_fwd");
}

int b200asr_conv3x3_c1_bwd_weight(const float* x, const float* dy, float* dw, float* dbias, int B, int F, int T, int Co,
                                  b200asr_stream_t stream) {
  B200_REQUIRE(x && dy && dw && dbias, B200ASR_BAD_ARG, "conv3x3_c1_bwd_weight: null pointer");
  B200_REQUIRE(Co % 4 == 0 && 256 % (Co / 4) == 0, B200ASR_BAD_SHAPE, "conv3x3_c1_bwd_weight: Co=%d unsupported", Co);
  cudaStream_t st = (cudaStream_t)stream;
  long long P = (long long)B * T * F;
  if (P <= 0) {
    cudaMemsetAsync(dw, 0, sizeof(float) * 9 * (size_t)Co, st);
    cudaMemsetAsync(dbias, 0, sizeof(float) * (size_t)Co, st);
    return B200ASR_OK;
  }
  int slots = 256 / (Co / 4);
  size_t smem = sizeof(float) * (size_t)slots * Co * 10;
  B200_REQUIRE(smem <= 44 * 1024, B200ASR_BAD_SHAPE, "conv3x3_c1_bwd_weight: Co=%d too large", Co);
  int blocks = device_sm_count() * 4;
  float* part = (float*)stream_scratch(sizeof(float) * (size_t)blocks * 10 * Co, st);
  if (!part) return B200ASR_CUDA_ERROR;
  conv3x3_c1_wgrad_kernel<<<blocks, 256, smem, st>>>(x, dy, part, B, F, T, Co);
  int rc = check_launch("conv3x3_c1_wgrad");
  if (rc || (rc = reduce_parts(part, blocks, 10LL * Co, 9LL * Co, dw, 0, st))) return rc;
  return reduce_parts(part + 9 * Co, blocks, 10LL * Co, Co, dbias, 0, st);
}

// bf16 variant of conv_repack_k_kernel for the bf16 modes: wk16[i] = bf16(w), and (terms == 2) wk16[total + i] =
// bf16(w - hi); same K-major [tap][n][c] order (fwd) / flipped taps (dgrad)
__global__ void conv_repack_k_bf16_kernel(const float* __restrict__ w, uint16_t* __restrict__ wk, int Ci, int Co, int dgrad, int terms) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  int total = 9 * Ci * Co;
  if (i >= total) return;
  float v;
  if (!dgrad) {
    int ci = i % Ci, co = (i / Ci) % Co, tap = i / (Co * Ci);
    v = w[((size_t)co * Ci + ci) * 9 + tap];
  } else {
    int co = i % Co, ci = (i / Co) % Ci, tap = i / (Co * Ci);
    v = w[((size_t)co * Ci + ci) * 9 + (8 - tap)];
  }
  const uint32_t r = __float_as_uint(v) + 0x8000u;
  wk[i] = (uint16_t)(r >> 16);
  if (terms == 2) {
    const float lo = v - __uint_as_float(r & 0xFFFF0000u);
    wk[total + i] = (uint16_t)((__float_as_uint(lo) + 0x8000u) >> 16);
  }
}

static bool conv_is_bf16(int precision) { return precision == B200ASR_PREC_BF16 || precision == B200ASR_PREC_BF16X3; }

static int conv_shape_ok(const char* who, int Ci, int Co) {
  B200_REQUIRE(Ci % 16 == 0 && Co % 64 == 0, B200ASR_BAD_SHAPE, "%s: need Ci %% 16 == 0 and Co %% 64 == 0 (Ci=%d Co=%d)", who, Ci, Co);
  return B200ASR_OK;
}

int b200asr_conv3x3_fwd(const float* x, const float* w, const float* bias, float* y, void* ws, int B, int T, int F,
                        int Ci, int Co, int relu, int precision, b200asr_stream_t stream) {
  B200_REQUIRE(x && w && y && ws, B200ASR_BAD_ARG, "conv3x3_fwd: null pointer");
  int rc = conv_shape_ok("conv3x3_fwd", Ci, Co);
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  int total = 9 * Ci * Co;
  note_launch(1);
  if (precision == B200ASR_PREC_FP32) {
    conv_repack_kernel<<<ceil_div(total, 256), 256, 0, st>>>(w, (float*)ws, Ci, Co, 0);
    return conv3x3_simt(x, (const float*)ws, bias, nullptr, y, B, T, F, Ci, Co, relu, st);
  }
  if (conv_is_bf16(precision)) {
    B200_REQUIRE(Ci % 32 == 0 && (Co == 64 || Co == 128), B200ASR_BAD_SHAPE, "conv3x3_fwd (bf16): needs Ci %% 32 == 0 and Co in {64,128}");
    conv_repack_k_bf16_kernel<<<ceil_div(total, 256), 256, 0, st>>>(w, (uint16_t*)ws, Ci, Co, 0, precision == B200ASR_PREC_BF16X3 ? 2 : 1);
    return conv3x3_tc_halo(x, ws, bias, nullptr, y, B, T, F, Ci, Co, relu, precision, st);
  }
  conv_repack_k_kernel<<<ceil_div(total, 256), 256, 0, st>>>(w, (float*)ws, Ci, Co, 0, precision == B200ASR_PREC_TF32X3);
  return conv3x3_tc(x, (const float*)ws, bias, nullptr, y, B, T, F, Ci, Co, relu, precision, st);
}

int b200asr_conv3x3_fwd_pool(const float* x, const float* w, const float* bias, float* y, float* pooled, unsigned char* pool_idx, void* ws,
                             int B, int T, int F, int Ci, int Co, int relu, int precision, b200asr_stream_t stream) {
  B200_REQUIRE(x && w && y && pooled && ws, B200ASR_BAD_ARG, "conv3x3_fwd_pool: null pointer");
  // the pooling rides in the convolution's epilogue (tc_conv_halo.cu) -- unless the arg-max bytes are wanted as well: computing
  // them there was measured to lengthen the epilogue (the critical path of the Cout = 64 kernel) by more than the index-based
  // pooling backward saves, so that request runs the stand-alone pooling kernel
  if (conv_is_bf16(precision) && !pool_idx) {
    int rc = conv_shape_ok("conv3x3_fwd_pool", Ci, Co);
    if (rc) return rc;
    B200_REQUIRE(Ci % 32 == 0 && (Co == 64 || Co == 128), B200ASR_BAD_SHAPE, "conv3x3_fwd_pool (bf16): needs Ci %% 32 == 0 and Co in {64,128}");
    B200_REQUIRE(aligned16(pooled), B200ASR_BAD_ALIGN, "conv3x3_fwd_pool: alignment");
    cudaStream_t st = (cudaStream_t)stream;
    note_launch(1);
    conv_repack_k_bf16_kernel<<<ceil_div(9 * Ci * Co, 256), 256, 0, st>>>(w, (uint16_t*)ws, Ci, Co, 0, precision == B200ASR_PREC_BF16X3 ? 2 : 1);
    return conv3x3_tc_halo(x, ws, bias, nullptr, y, B, T, F, Ci, Co, relu, precision, st, nullptr, pooled);
  }
  if (int rc = b200asr_conv3x3_fwd(x, w, bias, y, ws, B, T, F, Ci, Co, relu, precision, stream)) return rc;
  return pool_idx ? b200asr_maxpool2x2_fwd_idx(y, pooled, pool_idx, B, T, F, Co, stream) : b200asr_maxpool2x2_fwd(y, pooled, B, T, F, Co, stream);
}

int b200asr_conv3x3_bwd_data(const float* dy, const float* w, const float* relu_out, float* dx, void* dx16, void* ws, int B, int T,
                             int F, int Ci, int Co, int precision, b200asr_stream_t stream) {
  B200_REQUIRE(dy && w && dx && ws, B200ASR_BAD_ARG, "conv3x3_bwd_data: null pointer");
  int rc = conv_shape_ok("conv3x3_bwd_data", Co, Ci);   // roles swap: contraction over Co, output channels Ci
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  int total = 9 * Ci * Co;
  note_launch(1);
  if (precision == B200ASR_PREC_FP32) {
    conv_repack_kernel<<<ceil_div(total, 256), 256, 0, st>>>(w, (float*)ws, Ci, Co, 1);
    return conv3x3_simt(dy, (const float*)ws, nullptr, relu_out, dx, B, T, F, Co, Ci, 0, st);
  }
  if (conv_is_bf16(precision)) {
    B200_REQUIRE(Co % 32 == 0 && (Ci == 64 || Ci == 128), B200ASR_BAD_SHAPE, "conv3x3_bwd_data (bf16): needs Co %% 32 == 0 and Ci in {64,128}");
    conv_repack_k_bf16_kernel<<<ceil_div(total, 256), 256, 0, st>>>(w, (uint16_t*)ws, Ci, Co, 1, precision == B200ASR_PREC_BF16X3 ? 2 : 1);
    return conv3x3_tc_halo(dy, ws, nullptr, relu_out, dx, B, T, F, Co, Ci, 0, precision, st, dx16);
  }
  B200_REQUIRE(!dx16, B200ASR_BAD_ARG, "conv3x3_bwd_data: the bf16 pair output exists in the bf16 modes only");
  conv_repack_k_kernel<<<ceil_div(total, 256), 256, 0, st>>>(w, (float*)ws, Ci, Co, 1, precision == B200ASR_PREC_TF32X3);
  return conv3x3_tc(dy, (const float*)ws, nullptr, relu_out, dx, B, T, F, Co, Ci, 0, precision, st);
}

int b200asr_conv3x3_bwd_weight(const float* dy, const void* dy16, const float* x, float* dw, float* dbias, void* ws, int B, int T,
                               int F, int Ci, int Co, int precision, b200asr_stream_t stream) {
  B200_REQUIRE(dy && x && dw && ws, B200ASR_BAD_ARG, "conv3x3_bwd_weight: null pointer");
  B200_REQUIRE(Ci % 64 == 0 && Co % 64 == 0, B200ASR_BAD_SHAPE, "conv3x3_bwd_weight: Ci=%d Co=%d must be multiples of 64", Ci, Co);
  cudaStream_t st = (cudaStream_t)stream;
  cudaMemsetAsync(ws, 0, sizeof(float) * 9 * (size_t)Ci * Co, st);
  int rc;
  int bias_done = 0;
  if (precision == B200ASR_PREC_FP32) rc = conv3x3_wgrad_simt(x, dy, (float*)ws, B, T, F, Ci, Co, st);
  else rc = conv3x3_wgrad_tc(x, dy, (float*)ws, B, T, F, Ci, Co, precision, st, dbias, &bias_done, dy16);
  if (rc) return rc;
  int total = 9 * Ci * Co;
  conv_unpack_wgrad_kernel<<<ceil_div(total, 256), 256, 0, st>>>((const float*)ws, dw, Ci, Co);
  rc = check_launch("conv_unpack_wgrad");
  if (rc) return rc;
  if (dbias && !bias_done) {
    long long P = (long long)B * T * F;
    B200_REQUIRE(P < (1LL << 31), B200ASR_BAD_SHAPE, "conv3x3_bwd_weight: too many pixels");
    return launch_colsum(dy, dbias, (int)P, Co, 0, st);
  }
  return B200ASR_OK;
}

int b200asr_maxpool2x2_fwd(const float* x, float* y, int B, int T, int F, int C, b200asr_stream_t stream) {
  B200_REQUIRE(x && y && C % 4 == 0, B200ASR_BAD_ARG, "maxpool2x2_fwd: bad arguments");
  long long n = (long long)B * (T / 2) * (F / 2) * (C / 4);
  if (n <= 0) return B200ASR_OK;
  maxpool2x2_fwd_kernel<<<(unsigned)ceil_div_ll(n, 256), 256, 0, (cudaStream_t)stream>>>(x, y, nullptr, B, T, F, C);
  return check_launch("maxpool2x2_fwd");
}

int b200asr_maxpool2x2_fwd_idx(const float* x, float* y, unsigned char* idx, int B, int T, int F, int C, b200asr_stream_t stream) {
  B200_REQUIRE(x && y && idx && C % 4 == 0, B200ASR_BAD_ARG, "maxpool2x2_fwd_idx: bad arguments");
  long long n = (long long)B * (T / 2) * (F / 2) * (C / 4);
  if (n <= 0) return B200ASR_OK;
  maxpool2x2_fwd_kernel<<<(unsigned)ceil_div_ll(n, 256), 256, 0, (cudaStream_t)stream>>>(x, y, idx, B, T, F, C);
  return check_launch("maxpool2x2_fwd_idx");
}

int b200asr_maxpool2x2_bwd_idx(const float* dy, const unsigned char* idx, float* dx, void* dx16, int B, int T, int F, int C,
                               int relu_mask, b200asr_stream_t stream) {
  B200_REQUIRE(dy && idx && dx && C % 4 == 0, B200ASR_BAD_ARG, "maxpool2x2_bwd_idx: bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  long long n = (long long)B * (T / 2) * (F / 2) * (C / 4);
  if (n > 0) maxpool2x2_bwd_idx_kernel<<<(unsigned)ceil_div_ll(n, 256), 256, 0, st>>>(dy, idx, dx, (uint16_t*)dx16, B, T, F, C, relu_mask);
  if ((T & 1) || (F & 1)) {
    long long tot = ((F & 1) ? (long long)B * (T / 2) * 2 * (C / 4) : 0) + ((T & 1) ? (long long)B * F * (C / 4) : 0);
    maxpool2x2_bwd_tail_kernel<<<(unsigned)ceil_div_ll(tot, 256), 256, 0, st>>>(dx, (uint16_t*)dx16, B, T, F, C);
    note_launch(1);
  }
  return check_launch("maxpool2x2_bwd_idx");
}

int b200asr_maxpool2x2_bwd(const float* dy, const float* x, float* dx, void* dx16, int B, int T, int F, int C, int relu_mask,
                           b200asr_stream_t stream) {
  B200_REQUIRE(dy && x && dx && C % 4 == 0, B200ASR_BAD_ARG, "maxpool2x2_bwd: bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  long long n = (long long)B * (T / 2) * (F / 2) * (C / 4);
  if (n > 0) maxpool2x2_bwd_kernel<<<(unsigned)ceil_div_ll(n, 256), 256, 0, st>>>(dy, x, dx, (uint16_t*)dx16, B, T, F, C, relu_mask);
  if ((T & 1) || (F & 1)) {
    long long tot = ((F & 1) ? (long long)B * (T / 2) * 2 * (C / 4) : 0) + ((T & 1) ? (long long)B * F * (C / 4) : 0);
    maxpool2x2_bwd_tail_kernel<<<(unsigned)ceil_div_ll(tot, 256), 256, 0, st>>>(dx, (uint16_t*)dx16, B, T, F, C);
    note_launch(1);
  }
  return check_launch("maxpool2x2_bwd");
}

}  // extern "C"
