// Fused scaled-dot-product attention on CUDA cores (precision 0): flash-style online softmax, scores never
// leave the SM.  64x64 (query x key) tiles, 256 threads, each thread owns a 4x4 strided micro-tile
// (rows ty+16i, cols tx+16j) so that shared-memory reads are conflict free with 128-bit accesses.
// This is the exact-fp32 path and the on-device cross-check of the tensor-core attention kernels.
#include <math.h>

#include "../../include/b200asr.h"
#include "attention.h"
#include "common.cuh"

namespace b200asr {

constexpr int TQ = 64, TKT = 64, LP = 68;

__device__ __forceinline__ float half_warp_max(float v) {
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 8));
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 4));
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
  return v;
}
__device__ __forceinline__ float half_warp_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 8);
  v += __shfl_xor_sync(0xffffffffu, v, 4);
  v += __shfl_xor_sync(0xffffffffu, v, 2);
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  return v;
}

// rows x cols tile (cols % 4 == 0) from global (row stride rs) into smem (row stride ld), zero-filled past nrows
__device__ __forceinline__ void load_tile(float* __restrict__ S, int ld, const float* __restrict__ G, long long rs,
                                          int row0, int nrows_total, int cols, int tid) {
  const int vec = cols >> 2;
  for (int idx = tid; idx < 64 * vec; idx += 256) {
    int r = idx / vec, c = (idx - r * vec) * 4;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (row0 + r < nrows_total) v = *reinterpret_cast<const float4*>(G + (long long)(row0 + r) * rs + c);
    *reinterpret_cast<float4*>(S + r * ld + c) = v;
  }
}

__device__ __forceinline__ bool is_masked(const AttnP& p, int b, int q, int key) {
  if (key >= p.Tk) return true;
  if (p.causal && key > q) return true;
  if (p.key_pad && p.key_pad[(size_t)b * p.Tk + key]) return true;
  if (p.dense && q < p.Tq && p.dense[((size_t)b * p.Tq + q) * p.Tk + key]) return true;
  return false;
}

// unscaled scores of a 64x64 tile: s[i][j] = Q row ty+16i . K row tx+16j over dk columns (the forward's and
// sdpa_probs_simt_kernel's arithmetic, so the probabilities rebuilt from the log-sum-exp match the forward's)
__device__ __forceinline__ void score_tile(const float* __restrict__ Qs, const float* __restrict__ Ks, int LQ, int dk, int tx,
                                           int ty, float (&s)[4][4]) {
#pragma unroll
  for (int i = 0; i < 4; i++)
#pragma unroll
    for (int j = 0; j < 4; j++) s[i][j] = 0.f;
  for (int kk = 0; kk < dk; kk += 4) {
    float4 a[4], bb[4];
#pragma unroll
    for (int i = 0; i < 4; i++) a[i] = *reinterpret_cast<const float4*>(Qs + (ty + 16 * i) * LQ + kk);
#pragma unroll
    for (int j = 0; j < 4; j++) bb[j] = *reinterpret_cast<const float4*>(Ks + (tx + 16 * j) * LQ + kk);
#pragma unroll
    for (int i = 0; i < 4; i++)
#pragma unroll
      for (int j = 0; j < 4; j++)
        s[i][j] += a[i].x * bb[j].x + a[i].y * bb[j].y + a[i].z * bb[j].z + a[i].w * bb[j].w;
  }
}

template <int DV>
__global__ void __launch_bounds__(256) sdpa_fwd_simt_kernel(AttnP p) {
  extern __shared__ __align__(16) float smem[];
  const int dk = p.dk, LQ = dk + 4, LV = DV + 4;
  float* Qs = smem;
  float* Ks = Qs + 64 * LQ;
  float* Vs = Ks + 64 * LQ;
  float* Ps = Vs + 64 * LV;
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int q0 = blockIdx.x * TQ, h = blockIdx.y, b = blockIdx.z;
  const float* qg = p.q + b * p.q_bs + h * p.q_hs;
  const float* kg = p.k + b * p.k_bs + h * p.k_hs;
  const float* vg = p.v + b * p.v_bs + h * p.v_hs;
  load_tile(Qs, LQ, qg, p.q_rs, q0, p.Tq, dk, tid);

  float m[4], l[4], o[4][DV / 16];
#pragma unroll
  for (int i = 0; i < 4; i++) {
    m[i] = -INFINITY; l[i] = 0.f;
#pragma unroll
    for (int jj = 0; jj < DV / 16; jj++) o[i][jj] = 0.f;
  }
  const size_t drop_base = ((size_t)b * p.H + h) * p.Tq;

  for (int k0 = 0; k0 < p.Tk; k0 += TKT) {
    if (p.causal && k0 > q0 + TQ - 1) break;
    __syncthreads();
    load_tile(Ks, LQ, kg, p.k_rs, k0, p.Tk, dk, tid);
    load_tile(Vs, LV, vg, p.v_rs, k0, p.Tk, DV, tid);
    __syncthreads();
    float s[4][4];
    score_tile(Qs, Ks, LQ, dk, tx, ty, s);
#pragma unroll
    for (int i = 0; i < 4; i++) {
      const int q = q0 + ty + 16 * i;
      float mx = -INFINITY;
#pragma unroll
      for (int j = 0; j < 4; j++) {
        const int key = k0 + tx + 16 * j;
        s[i][j] = is_masked(p, b, q, key) ? -INFINITY : s[i][j] * p.scale;
        mx = fmaxf(mx, s[i][j]);
      }
      mx = half_warp_max(mx);
      const float m_new = fmaxf(m[i], mx);
      const float m_safe = (m_new == -INFINITY) ? 0.f : m_new;
      const float corr = expf(m[i] - m_safe);
      float rs = 0.f;
#pragma unroll
      for (int j = 0; j < 4; j++) {
        float pe = expf(s[i][j] - m_safe);
        rs += pe;
        if (p.thresh) {
          const int key = k0 + tx + 16 * j;
          pe = dropout_keep(p.key, (drop_base + q) * p.Tk + key, p.thresh) ? pe * p.inv_keep : 0.f;
        }
        Ps[(ty + 16 * i) * LP + tx + 16 * j] = pe;
      }
      rs = half_warp_sum(rs);
      l[i] = l[i] * corr + rs;
      m[i] = m_new;
#pragma unroll
      for (int jj = 0; jj < DV / 16; jj++) o[i][jj] *= corr;
    }
    __syncthreads();
    for (int key = 0; key < TKT; key += 4) {
      float4 pp[4];
#pragma unroll
      for (int i = 0; i < 4; i++) pp[i] = *reinterpret_cast<const float4*>(Ps + (ty + 16 * i) * LP + key);
#pragma unroll
      for (int jj = 0; jj < DV / 16; jj++) {
        const float v0 = Vs[(key + 0) * LV + tx + 16 * jj], v1 = Vs[(key + 1) * LV + tx + 16 * jj];
        const float v2 = Vs[(key + 2) * LV + tx + 16 * jj], v3 = Vs[(key + 3) * LV + tx + 16 * jj];
#pragma unroll
        for (int i = 0; i < 4; i++) o[i][jj] += pp[i].x * v0 + pp[i].y * v1 + pp[i].z * v2 + pp[i].w * v3;
      }
    }
  }
  float* og = p.o + b * p.o_bs + h * p.o_hs;
#pragma unroll
  for (int i = 0; i < 4; i++) {
    const int q = q0 + ty + 16 * i;
    if (q >= p.Tq) continue;
    const float inv = 1.f / l[i];   // l == 0 (fully masked row) -> inf * 0 = NaN, as the reference's softmax
#pragma unroll
    for (int jj = 0; jj < DV / 16; jj++) og[(long long)q * p.o_rs + tx + 16 * jj] = o[i][jj] * inv;
    // a fully masked row's log-sum-exp is NaN, as the tensor-core kernels write it; the backward reads it as "dead row"
    if (tx == 0 && p.lse) p.lse[((size_t)b * p.H + h) * p.Tq + q] = m[i] == -INFINITY ? NAN : m[i] + logf(l[i]);
  }
}

// The probabilities the forward multiplied into V, rebuilt from Q, K and its log-sum-exp: P = expf(scale * S - lse) with
// the masks and the forward's dropout mask (times inv_keep) applied; masked keys are 0, a fully masked row (lse NaN) is
// NaN.  Written through p.o with the strides p.o_bs / o_hs / o_rs (any row stride), staged in shared memory per 64x64
// tile so that the stores go out as whole rows.
__global__ void __launch_bounds__(256) sdpa_probs_simt_kernel(AttnP p) {
  griddep_launch();      // programmatic dependent launch (common.cuh)
  griddep_wait();
  extern __shared__ __align__(16) float smem[];
  const int dk = p.dk, LQ = dk + 4;
  float* Qs = smem;
  float* Ks = Qs + 64 * LQ;
  float* Ps = Ks + 64 * LQ;
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int q0 = blockIdx.x * TQ, h = blockIdx.y, b = blockIdx.z;
  const float* kg = p.k + b * p.k_bs + h * p.k_hs;
  float* og = p.o + b * p.o_bs + h * p.o_hs;
  load_tile(Qs, LQ, p.q + b * p.q_bs + h * p.q_hs, p.q_rs, q0, p.Tq, dk, tid);
  const size_t row_base = ((size_t)b * p.H + h) * p.Tq;
  float lse[4];
#pragma unroll
  for (int i = 0; i < 4; i++) lse[i] = q0 + ty + 16 * i < p.Tq ? p.lse[row_base + q0 + ty + 16 * i] : 0.f;

  for (int k0 = 0; k0 < p.Tk; k0 += TKT) {
    const bool past = p.causal && k0 > q0 + TQ - 1;      // every key of the tile is masked for every query
    __syncthreads();
    if (!past) load_tile(Ks, LQ, kg, p.k_rs, k0, p.Tk, dk, tid);
    __syncthreads();
    float s[4][4];
    if (!past) score_tile(Qs, Ks, LQ, dk, tx, ty, s);
#pragma unroll
    for (int i = 0; i < 4; i++) {
      const int q = q0 + ty + 16 * i;
#pragma unroll
      for (int j = 0; j < 4; j++) {
        const int key = k0 + tx + 16 * j;
        float pr = 0.f;
        if (isnan(lse[i])) {
          pr = NAN;
        } else if (!past && !is_masked(p, b, q, key)) {
          pr = expf(s[i][j] * p.scale - lse[i]);
          if (p.thresh) pr = dropout_keep(p.key, (row_base + q) * p.Tk + key, p.thresh) ? pr * p.inv_keep : 0.f;
        }
        Ps[(ty + 16 * i) * LP + tx + 16 * j] = pr;
      }
    }
    __syncthreads();
    const int nk = min(TKT, p.Tk - k0);
    for (int idx = tid; idx < TQ * TKT; idx += 256) {
      const int r = idx / TKT, c = idx % TKT;
      if (q0 + r < p.Tq && c < nk) og[(long long)(q0 + r) * p.o_rs + k0 + c] = Ps[r * LP + c];
    }
  }
}

int sdpa_probs_simt(const AttnP& p, cudaStream_t st) {
  B200_REQUIRE(p.dk == 16 || p.dk == 32 || p.dk == 64 || p.dk == 128, B200ASR_BAD_SHAPE, "sdpa_probs (fp32): dk=%d unsupported (16/32/64/128)", p.dk);
  constexpr int smem_max = (int)sizeof(float) * (64 * (128 + 4) * 2 + 64 * LP);      // dk = 128
  const int smem = (int)sizeof(float) * (64 * (p.dk + 4) * 2 + 64 * LP);
  static bool attr_set[kMaxDevices] = {};
  if (int rc = ensure_dynamic_smem((const void*)sdpa_probs_simt_kernel, smem_max, attr_set, "sdpa_probs_simt")) return rc;
  launch_pdl(sdpa_probs_simt_kernel, dim3(ceil_div(p.Tq, TQ), p.H, p.B), dim3(256), (size_t)smem, st, p);
  return check_launch("sdpa_probs_simt");
}

// delta[b,h,q] = sum_c dO*O ; also zero dq (strided) for the atomics of the main backward kernel
template <int DV>
__global__ void sdpa_bwd_prep_kernel(AttnP p, const float* __restrict__ dout, float* __restrict__ dq,
                                     float* __restrict__ delta) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  const int total = p.B * p.H * p.Tq;
  if (warp >= total) return;
  const int q = warp % p.Tq, bh = warp / p.Tq, h = bh % p.H, b = bh / p.H;
  const float* og = p.o + b * p.o_bs + h * p.o_hs + (long long)q * p.o_rs;
  const float* dg = dout + b * p.o_bs + h * p.o_hs + (long long)q * p.o_rs;
  float s = 0.f;
  for (int c = lane; c < DV; c += 32) s += og[c] * dg[c];
  s = warp_sum(s);
  if (lane == 0) delta[warp] = s;
  float* dqg = dq + b * p.q_bs + h * p.q_hs + (long long)q * p.q_rs;
  for (int c = lane; c < p.dk; c += 32) dqg[c] = 0.f;
}

template <int DK, int DV>
__global__ void __launch_bounds__(256) sdpa_bwd_simt_kernel(AttnP p, const float* __restrict__ dout,
                                                            float* __restrict__ dq, float* __restrict__ dkout,
                                                            float* __restrict__ dvout, const float* __restrict__ delta) {
  extern __shared__ __align__(16) float smem[];
  constexpr int LQ = DK + 4, LV = DV + 4;
  float* Ks = smem;
  float* Vs = Ks + 64 * LQ;
  float* Qs = Vs + 64 * LV;
  float* Os = Qs + 64 * LQ;   // dO tile
  float* Ps = Os + 64 * LV;   // dropped probabilities
  float* Ds = Ps + 64 * LP;   // dS
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int k0 = blockIdx.x * TKT, h = blockIdx.y, b = blockIdx.z;
  const float* qg = p.q + b * p.q_bs + h * p.q_hs;
  const float* kg = p.k + b * p.k_bs + h * p.k_hs;
  const float* vg = p.v + b * p.v_bs + h * p.v_hs;
  const float* dog = dout + b * p.o_bs + h * p.o_hs;
  load_tile(Ks, LQ, kg, p.k_rs, k0, p.Tk, DK, tid);
  load_tile(Vs, LV, vg, p.v_rs, k0, p.Tk, DV, tid);

  float dka[4][DK / 16], dva[4][DV / 16];
#pragma unroll
  for (int i = 0; i < 4; i++) {
#pragma unroll
    for (int jj = 0; jj < DK / 16; jj++) dka[i][jj] = 0.f;
#pragma unroll
    for (int jj = 0; jj < DV / 16; jj++) dva[i][jj] = 0.f;
  }
  const size_t row_base = ((size_t)b * p.H + h) * p.Tq;
  const int q_start = p.causal ? (k0 / TQ) * TQ : 0;   // queries before the key tile see none of it
  // a fully masked query row (lse NaN) has a NaN row of P in the reference's masked_fill -> softmax, so dV = P^T dO is NaN
  // for every key of the head, skipped query tiles included; masked_fill passes its scores no gradient, so dS stays 0
  bool dead = false;
  for (int i = tid; i < p.Tq; i += 256) dead |= isnan(p.lse[row_base + i]);
  dead = __syncthreads_or(dead);

  for (int q0 = q_start; q0 < p.Tq; q0 += TQ) {
    __syncthreads();
    load_tile(Qs, LQ, qg, p.q_rs, q0, p.Tq, DK, tid);
    load_tile(Os, LV, dog, p.o_rs, q0, p.Tq, DV, tid);
    __syncthreads();
    float s[4][4], dp[4][4];
#pragma unroll
    for (int i = 0; i < 4; i++)
#pragma unroll
      for (int j = 0; j < 4; j++) { s[i][j] = 0.f; dp[i][j] = 0.f; }
#pragma unroll 4
    for (int kk = 0; kk < DK; kk += 4) {
      float4 a[4], bb[4];
#pragma unroll
      for (int i = 0; i < 4; i++) a[i] = *reinterpret_cast<const float4*>(Qs + (ty + 16 * i) * LQ + kk);
#pragma unroll
      for (int j = 0; j < 4; j++) bb[j] = *reinterpret_cast<const float4*>(Ks + (tx + 16 * j) * LQ + kk);
#pragma unroll
      for (int i = 0; i < 4; i++)
#pragma unroll
        for (int j = 0; j < 4; j++)
          s[i][j] += a[i].x * bb[j].x + a[i].y * bb[j].y + a[i].z * bb[j].z + a[i].w * bb[j].w;
    }
#pragma unroll 4
    for (int kk = 0; kk < DV; kk += 4) {
      float4 a[4], bb[4];
#pragma unroll
      for (int i = 0; i < 4; i++) a[i] = *reinterpret_cast<const float4*>(Os + (ty + 16 * i) * LV + kk);
#pragma unroll
      for (int j = 0; j < 4; j++) bb[j] = *reinterpret_cast<const float4*>(Vs + (tx + 16 * j) * LV + kk);
#pragma unroll
      for (int i = 0; i < 4; i++)
#pragma unroll
        for (int j = 0; j < 4; j++)
          dp[i][j] += a[i].x * bb[j].x + a[i].y * bb[j].y + a[i].z * bb[j].z + a[i].w * bb[j].w;
    }
#pragma unroll
    for (int i = 0; i < 4; i++) {
      const int q = q0 + ty + 16 * i;
      const bool qok = q < p.Tq;
      const float lse = qok ? p.lse[row_base + q] : 0.f;
      const float dl = qok ? delta[row_base + q] : 0.f;
#pragma unroll
      for (int j = 0; j < 4; j++) {
        const int key = k0 + tx + 16 * j;
        float pr = 0.f, pd = 0.f, ds = 0.f;
        if (qok && !is_masked(p, b, q, key)) {
          pr = expf(s[i][j] * p.scale - lse);
          float keep = 1.f;
          if (p.thresh) keep = dropout_keep(p.key, (row_base + q) * p.Tk + key, p.thresh) ? p.inv_keep : 0.f;
          pd = pr * keep;
          ds = pr * (dp[i][j] * keep - dl) * p.scale;
        }
        Ps[(ty + 16 * i) * LP + tx + 16 * j] = pd;
        Ds[(ty + 16 * i) * LP + tx + 16 * j] = ds;
      }
    }
    __syncthreads();
    // dV[key][c] += sum_q Pd[q][key] dO[q][c] ; dK[key][c] += sum_q dS[q][key] Q[q][c]   (key = ty+16i)
    for (int q = 0; q < TQ; q++) {
      float pv[4], dsv[4];
#pragma unroll
      for (int i = 0; i < 4; i++) { pv[i] = Ps[q * LP + ty + 16 * i]; dsv[i] = Ds[q * LP + ty + 16 * i]; }
#pragma unroll
      for (int jj = 0; jj < DV / 16; jj++) {
        const float x = Os[q * LV + tx + 16 * jj];
#pragma unroll
        for (int i = 0; i < 4; i++) dva[i][jj] += pv[i] * x;
      }
#pragma unroll
      for (int jj = 0; jj < DK / 16; jj++) {
        const float x = Qs[q * LQ + tx + 16 * jj];
#pragma unroll
        for (int i = 0; i < 4; i++) dka[i][jj] += dsv[i] * x;
      }
    }
    // dQ[q][c] += sum_key dS[q][key] K[key][c]   (q = ty+16i)
    float dqa[4][DK / 16];
#pragma unroll
    for (int i = 0; i < 4; i++)
#pragma unroll
      for (int jj = 0; jj < DK / 16; jj++) dqa[i][jj] = 0.f;
    for (int key = 0; key < TKT; key += 4) {
      float4 dd[4];
#pragma unroll
      for (int i = 0; i < 4; i++) dd[i] = *reinterpret_cast<const float4*>(Ds + (ty + 16 * i) * LP + key);
#pragma unroll
      for (int jj = 0; jj < DK / 16; jj++) {
        const float x0 = Ks[(key + 0) * LQ + tx + 16 * jj], x1 = Ks[(key + 1) * LQ + tx + 16 * jj];
        const float x2 = Ks[(key + 2) * LQ + tx + 16 * jj], x3 = Ks[(key + 3) * LQ + tx + 16 * jj];
#pragma unroll
        for (int i = 0; i < 4; i++) dqa[i][jj] += dd[i].x * x0 + dd[i].y * x1 + dd[i].z * x2 + dd[i].w * x3;
      }
    }
    float* dqg = dq + b * p.q_bs + h * p.q_hs;
#pragma unroll
    for (int i = 0; i < 4; i++) {
      const int q = q0 + ty + 16 * i;
      if (q >= p.Tq) continue;
#pragma unroll
      for (int jj = 0; jj < DK / 16; jj++) atomicAdd(dqg + (long long)q * p.q_rs + tx + 16 * jj, dqa[i][jj]);
    }
  }
  float* dkg = dkout + b * p.k_bs + h * p.k_hs;
  float* dvg = dvout + b * p.v_bs + h * p.v_hs;
#pragma unroll
  for (int i = 0; i < 4; i++) {
    const int key = k0 + ty + 16 * i;
    if (key >= p.Tk) continue;
#pragma unroll
    for (int jj = 0; jj < DK / 16; jj++) dkg[(long long)key * p.k_rs + tx + 16 * jj] = dka[i][jj];
#pragma unroll
    for (int jj = 0; jj < DV / 16; jj++) dvg[(long long)key * p.v_rs + tx + 16 * jj] = dead ? NAN : dva[i][jj];
  }
}

template <int DV>
static int launch_fwd(const AttnP& p, cudaStream_t st) {
  size_t smem = sizeof(float) * (size_t)(64 * (p.dk + 4) * 2 + 64 * (DV + 4) + 64 * LP);
  cudaFuncSetAttribute(sdpa_fwd_simt_kernel<DV>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  dim3 grid(ceil_div(p.Tq, TQ), p.H, p.B);
  sdpa_fwd_simt_kernel<DV><<<grid, 256, smem, st>>>(p);
  return check_launch("sdpa_fwd_simt");
}

int sdpa_fwd_simt(const AttnP& p, cudaStream_t st) {
  switch (p.dv) {
    case 16: return launch_fwd<16>(p, st);
    case 32: return launch_fwd<32>(p, st);
    case 64: return launch_fwd<64>(p, st);
    case 128: return launch_fwd<128>(p, st);
  }
  set_error("sdpa_fwd: dv=%d unsupported (16/32/64/128)", p.dv);
  return B200ASR_BAD_SHAPE;
}

template <int DK, int DV>
static int launch_bwd(const AttnP& p, const float* dout, float* dq, float* dk, float* dv, float* delta,
                      cudaStream_t st) {
  int total = p.B * p.H * p.Tq;
  sdpa_bwd_prep_kernel<DV><<<ceil_div(total, 8), 256, 0, st>>>(p, dout, dq, delta);
  int rc = check_launch("sdpa_bwd_prep");
  if (rc) return rc;
  size_t smem = sizeof(float) * (size_t)(64 * (DK + 4) * 2 + 64 * (DV + 4) * 2 + 64 * LP * 2);
  cudaFuncSetAttribute(sdpa_bwd_simt_kernel<DK, DV>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  dim3 grid(ceil_div(p.Tk, TKT), p.H, p.B);
  sdpa_bwd_simt_kernel<DK, DV><<<grid, 256, smem, st>>>(p, dout, dq, dk, dv, delta);
  return check_launch("sdpa_bwd_simt");
}

int sdpa_bwd_simt(const AttnP& p, const float* dout, float* dq, float* dk, float* dv, float* delta, cudaStream_t st) {
#define CASE(a, b) if (p.dk == a && p.dv == b) return launch_bwd<a, b>(p, dout, dq, dk, dv, delta, st)
  CASE(16, 16); CASE(16, 32); CASE(16, 64); CASE(16, 128); CASE(32, 16); CASE(32, 32); CASE(32, 64); CASE(32, 128);
  CASE(64, 16); CASE(64, 32); CASE(64, 64); CASE(64, 128); CASE(128, 16); CASE(128, 32); CASE(128, 64); CASE(128, 128);
#undef CASE
  set_error("sdpa_bwd: (dk=%d, dv=%d) unsupported", p.dk, p.dv);
  return B200ASR_BAD_SHAPE;
}

}  // namespace b200asr
