// Fused attention on the tensor cores with warp-level MMAs (mma.sync): the TF32 kernels (precision 1, b200asr_sdpa_fwd/_bwd)
// and the opt-in bf16x3 kernels (b200asr_sdpa_fused_*) of ScaledDotProductAttention.forward, models/common_layers.py:211-225.
//
//   forward  : CTA = (64-query tile, head, utterance), a warp owns 16 queries; loops over 64-key blocks:
//              S = Q K^T -> scale, masks, online softmax (running max / sum per row, O rescaled) -> dropout -> O += P V.
//              Scores and probabilities stay in registers.
//   backward : recomputes the probabilities from Q, K and the forward's log-sum-exp (nothing of size Tq x Tk is stored):
//     dkdv   : CTA = 64-key block, a warp owns 16 keys; loops over 64-query tiles: S^T = K Q^T, dP^T = V dO^T,
//              Pd^T = P^T o keep, dS^T = P^T o (dP^T o keep - delta) * scale, dV += Pd^T dO, dK += dS^T Q.
//     dq     : CTA = 64-query tile; loops over 64-key blocks: S = Q K^T, dP = dO V^T, dS, dQ += dS K.
// Operand tiles are staged in shared memory as fp32 rows (pitch D + 4: conflict-free fragment loads) and rounded (MODE 1,
// TF32, m16n8k8) or split (MODE 6, bf16x3: lo*hi + hi*lo + hi*hi, m16n8k16) as the register fragments are built.  The C
// layout of S is the A layout of P for bf16 (pairs 2q, 2q + 1); for tf32 the k order inside each 8-key step is permuted
// (k q <-> key 2q, k q + 4 <-> key 2q + 1) and B is read with the same permutation -- the sum over k does not change.
#include <math.h>

#include "../../include/b200asr.h"
#include "attention.h"
#include "common.cuh"
#include "tc_common.cuh"

namespace b200asr {
namespace tc {

constexpr int FL_ROWS = 64;            // rows per CTA (4 warps x 16)
constexpr int FL_THREADS = 128;

__device__ __forceinline__ void mma_tf32_16x8x8(float (&c)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
  asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}
__device__ __forceinline__ void mma_bf16_16x8x16(float (&c)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}

template <int MODE> struct Fl {
  static constexpr int KS = MODE == 1 ? 8 : 16;                  // contraction per MMA
  struct A { uint32_t h[4], l[4]; };
  struct B { uint32_t h[2], l[2]; };
  static __device__ __forceinline__ uint32_t tf(float x) { return __float_as_uint(tf32_rn(x)); }
  static __device__ __forceinline__ void pair(float x0, float x1, uint32_t& h, uint32_t& l) { split_bf16_pair(x0, x1, h, l); }

  // A rows r0 .. r0 + 15 of a [rows][pitch] fp32 tile, contraction = columns d0 .. d0 + KS - 1
  static __device__ __forceinline__ A a_feat(const float* t, int pitch, int r0, int d0, int g, int q) {
    A a;
    const float* p0 = t + (r0 + g) * pitch + d0;
    const float* p1 = p0 + 8 * pitch;
    if constexpr (MODE == 1) {
      a.h[0] = tf(p0[q]); a.h[1] = tf(p1[q]); a.h[2] = tf(p0[q + 4]); a.h[3] = tf(p1[q + 4]);
    } else {
      pair(p0[2 * q], p0[2 * q + 1], a.h[0], a.l[0]);
      pair(p1[2 * q], p1[2 * q + 1], a.h[1], a.l[1]);
      pair(p0[2 * q + 8], p0[2 * q + 9], a.h[2], a.l[2]);
      pair(p1[2 * q + 8], p1[2 * q + 9], a.h[3], a.l[3]);
    }
    return a;
  }
  // B with n = tile rows n0 .. n0 + 7, contraction = columns d0 .. d0 + KS - 1 (B[k][n] = t[n][k])
  static __device__ __forceinline__ B b_feat(const float* t, int pitch, int n0, int d0, int g, int q) {
    B b;
    const float* p = t + (n0 + g) * pitch + d0;
    if constexpr (MODE == 1) {
      b.h[0] = tf(p[q]); b.h[1] = tf(p[q + 4]);
    } else {
      pair(p[2 * q], p[2 * q + 1], b.h[0], b.l[0]);
      pair(p[2 * q + 8], p[2 * q + 9], b.h[1], b.l[1]);
    }
    return b;
  }
  // B with contraction = tile rows k0 .. k0 + KS - 1, n = columns n0 .. n0 + 7 (B[k][n] = t[k][n]); tf32: permuted k order
  static __device__ __forceinline__ B b_row(const float* t, int pitch, int k0, int n0, int g, int q) {
    B b;
    const float* p = t + k0 * pitch + n0 + g;
    if constexpr (MODE == 1) {
      b.h[0] = tf(p[(2 * q) * pitch]); b.h[1] = tf(p[(2 * q + 1) * pitch]);
    } else {
      pair(p[(2 * q) * pitch], p[(2 * q + 1) * pitch], b.h[0], b.l[0]);
      pair(p[(2 * q + 8) * pitch], p[(2 * q + 9) * pitch], b.h[1], b.l[1]);
    }
    return b;
  }
  // A from accumulator blocks (C layout, 8 columns each): k-step ks covers blocks ks (tf32, permuted) or 2ks, 2ks + 1 (bf16)
  template <int NB> static __device__ __forceinline__ A a_from_c(const float (&c)[NB][4], int ks) {
    A a;
    if constexpr (MODE == 1) {
      a.h[0] = tf(c[ks][0]); a.h[1] = tf(c[ks][2]); a.h[2] = tf(c[ks][1]); a.h[3] = tf(c[ks][3]);
    } else {
      pair(c[2 * ks][0], c[2 * ks][1], a.h[0], a.l[0]);
      pair(c[2 * ks][2], c[2 * ks][3], a.h[1], a.l[1]);
      pair(c[2 * ks + 1][0], c[2 * ks + 1][1], a.h[2], a.l[2]);
      pair(c[2 * ks + 1][2], c[2 * ks + 1][3], a.h[3], a.l[3]);
    }
    return a;
  }
  static __device__ __forceinline__ void mma(float (&c)[4], const A& a, const B& b) {
    if constexpr (MODE == 1) {
      mma_tf32_16x8x8(c, a.h, b.h);
    } else {                                      // small products first
      mma_bf16_16x8x16(c, a.l, b.h);
      mma_bf16_16x8x16(c, a.h, b.l);
      mma_bf16_16x8x16(c, a.h, b.h);
    }
  }
};

// rows [t0, t0 + 64) of a (B,H,T,D) view -> smem [64][D + 4] fp32, zeros beyond T
template <int D>
__device__ __forceinline__ void fl_load_tile(float* dst, const float* base, long long bs, long long hs, long long rs, int b, int h,
                                             int t0, int T) {
  constexpr int P = D + 4, C4 = D / 4;
  for (int i = threadIdx.x; i < FL_ROWS * C4; i += FL_THREADS) {
    const int r = i / C4, c = (i % C4) * 4;
    const int t = t0 + r;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (t < T) v = *reinterpret_cast<const float4*>(base + b * bs + h * hs + (long long)t * rs + c);
    *reinterpret_cast<float4*>(dst + r * P + c) = v;
  }
}

// store a warp's 16 x D accumulator rows (row g / g + 8 of the warp) to a (B,H,T,D) view, scaled by s0 / s1
template <int D>
__device__ __forceinline__ void fl_store_rows(const float (&acc)[D / 8][4], float* base, long long bs, long long hs, long long rs, int b,
                                              int h, int t_lo, int T, int g, int q, float s0, float s1) {
  const int t0 = t_lo + g, t1 = t0 + 8;
  float* o0 = base + b * bs + h * hs + (long long)t0 * rs;
  float* o1 = base + b * bs + h * hs + (long long)t1 * rs;
#pragma unroll
  for (int nb = 0; nb < D / 8; nb++) {
    const int c = nb * 8 + 2 * q;
    if (t0 < T) *reinterpret_cast<float2*>(o0 + c) = make_float2(acc[nb][0] * s0, acc[nb][1] * s0);
    if (t1 < T) *reinterpret_cast<float2*>(o1 + c) = make_float2(acc[nb][2] * s1, acc[nb][3] * s1);
  }
}

__device__ __forceinline__ bool fl_masked(const AttnP& p, const uint8_t* pad, int b, int qi, int key, int key_local) {
  if (pad[key_local] || (p.causal && key > qi)) return true;
  return p.dense && p.dense[((size_t)b * p.Tq + qi) * p.Tk + key] != 0;
}

// ---------------------------------------------------------------------------------------------------------------------
template <int MODE, int DK, int DV>
__global__ void __launch_bounds__(FL_THREADS)
flash_fwd_kernel(const AttnP p) {
  using F = Fl<MODE>;
  constexpr int PK = DK + 4, PV = DV + 4, KS = F::KS;
  extern __shared__ float fl_smem[];
  float* sQ = fl_smem;
  float* sK = sQ + FL_ROWS * PK;
  float* sV = sK + FL_ROWS * PK;
  uint8_t* pad = reinterpret_cast<uint8_t*>(sV + FL_ROWS * PV);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, q = lane & 3;
  const int q0 = blockIdx.x * FL_ROWS, h = blockIdx.y, b = blockIdx.z;
  const int qa = q0 + warp * 16 + g, qb = qa + 8;           // this thread's two query rows
  const size_t bh = (size_t)b * p.H + h;

  fl_load_tile<DK>(sQ, p.q, p.q_bs, p.q_hs, p.q_rs, b, h, q0, p.Tq);
  __syncthreads();
  typename F::A qf[DK / KS];
#pragma unroll
  for (int ks = 0; ks < DK / KS; ks++) qf[ks] = F::a_feat(sQ, PK, warp * 16, ks * KS, g, q);

  float o[DV / 8][4];
#pragma unroll
  for (int i = 0; i < DV / 8; i++) o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f;
  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;

  for (int k0 = 0; k0 < p.Tk; k0 += FL_ROWS) {
    __syncthreads();                                       // previous block's readers are done
    fl_load_tile<DK>(sK, p.k, p.k_bs, p.k_hs, p.k_rs, b, h, k0, p.Tk);
    fl_load_tile<DV>(sV, p.v, p.v_bs, p.v_hs, p.v_rs, b, h, k0, p.Tk);
    if (threadIdx.x < FL_ROWS) {
      const int key = k0 + threadIdx.x;
      pad[threadIdx.x] = (key >= p.Tk || (p.key_pad && p.key_pad[(size_t)b * p.Tk + key])) ? 1 : 0;
    }
    __syncthreads();
    float s[8][4];
#pragma unroll
    for (int nb = 0; nb < 8; nb++) s[nb][0] = s[nb][1] = s[nb][2] = s[nb][3] = 0.f;
#pragma unroll
    for (int ks = 0; ks < DK / KS; ks++)
#pragma unroll
      for (int nb = 0; nb < 8; nb++) F::mma(s[nb], qf[ks], F::b_feat(sK, PK, nb * 8, ks * KS, g, q));
    // scale + masks, block row max
    float bm0 = -INFINITY, bm1 = -INFINITY;
#pragma unroll
    for (int nb = 0; nb < 8; nb++)
#pragma unroll
      for (int e = 0; e < 4; e++) {
        const int kl = nb * 8 + 2 * q + (e & 1), key = k0 + kl, qi = (e & 2) ? qb : qa;
        const bool masked = qi >= p.Tq || fl_masked(p, pad, b, qi, key, kl);
        s[nb][e] = masked ? -INFINITY : s[nb][e] * p.scale;
        if (e & 2) bm1 = fmaxf(bm1, s[nb][e]); else bm0 = fmaxf(bm0, s[nb][e]);
      }
    bm0 = fmaxf(bm0, __shfl_xor_sync(0xffffffffu, bm0, 1)); bm0 = fmaxf(bm0, __shfl_xor_sync(0xffffffffu, bm0, 2));
    bm1 = fmaxf(bm1, __shfl_xor_sync(0xffffffffu, bm1, 1)); bm1 = fmaxf(bm1, __shfl_xor_sync(0xffffffffu, bm1, 2));
    const float mn0 = fmaxf(m0, bm0), mn1 = fmaxf(m1, bm1);
    const float al0 = mn0 == -INFINITY ? 1.f : __expf(m0 - mn0), al1 = mn1 == -INFINITY ? 1.f : __expf(m1 - mn1);
    m0 = mn0; m1 = mn1;
    l0 *= al0; l1 *= al1;
#pragma unroll
    for (int i = 0; i < DV / 8; i++) { o[i][0] *= al0; o[i][1] *= al0; o[i][2] *= al1; o[i][3] *= al1; }
    // p = exp(s - m) (TF32 mode: rounded as the MMA will see it), row sums, dropout
#pragma unroll
    for (int nb = 0; nb < 8; nb++)
#pragma unroll
      for (int e = 0; e < 4; e++) {
        const bool r1 = (e & 2) != 0;
        const float mm = r1 ? m1 : m0;
        float pe = s[nb][e] == -INFINITY ? 0.f : __expf(s[nb][e] - mm);
        if constexpr (MODE == 1) pe = tf32_rn(pe);
        if (r1) l1 += pe; else l0 += pe;
        const int key = k0 + nb * 8 + 2 * q + (e & 1), qi = r1 ? qb : qa;
        if (p.thresh && key < p.Tk && qi < p.Tq)
          pe = dropout_keep(p.key, (bh * p.Tq + qi) * (size_t)p.Tk + key, p.thresh) ? pe * p.inv_keep : 0.f;
        s[nb][e] = pe;
      }
    // O += P V
#pragma unroll
    for (int ks = 0; ks < FL_ROWS / KS; ks++) {
      const typename F::A pa = F::a_from_c(s, ks);
#pragma unroll
      for (int nb = 0; nb < DV / 8; nb++) F::mma(o[nb], pa, F::b_row(sV, PV, ks * KS, nb * 8, g, q));
    }
  }
  l0 += __shfl_xor_sync(0xffffffffu, l0, 1); l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 1); l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
  // a fully masked row has m = -inf: its output and log-sum-exp are NaN, as the reference's softmax gives
  const float inv0 = m0 == -INFINITY ? NAN : 1.f / l0, inv1 = m1 == -INFINITY ? NAN : 1.f / l1;
  fl_store_rows<DV>(o, p.o, p.o_bs, p.o_hs, p.o_rs, b, h, q0 + warp * 16, p.Tq, g, q, inv0, inv1);
  if (p.lse && q == 0) {
    if (qa < p.Tq) p.lse[bh * p.Tq + qa] = m0 == -INFINITY ? NAN : m0 + logf(l0);
    if (qb < p.Tq) p.lse[bh * p.Tq + qb] = m1 == -INFINITY ? NAN : m1 + logf(l1);
  }
}

// ---------------------------------------------------------------------------------------------------------------------
template <int MODE, int DK, int DV>
__global__ void __launch_bounds__(FL_THREADS)
flash_bwd_dkdv_kernel(const AttnP p, const float* __restrict__ dout, const float* __restrict__ delta, float* __restrict__ dk_out,
                      float* __restrict__ dv_out) {
  using F = Fl<MODE>;
  constexpr int PK = DK + 4, PV = DV + 4, KS = F::KS;
  extern __shared__ float fl_smem[];
  float* sK = fl_smem;
  float* sV = sK + FL_ROWS * PK;
  float* sQ = sV + FL_ROWS * PV;
  float* sO = sQ + FL_ROWS * PK;
  float* vec = sO + FL_ROWS * PV;                          // lse[64], delta[64]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, q = lane & 3;
  const int k0 = blockIdx.x * FL_ROWS, h = blockIdx.y, b = blockIdx.z;
  const int ka = k0 + warp * 16 + g, kb = ka + 8;           // this thread's two key rows
  const size_t bh = (size_t)b * p.H + h;
  const bool kpad_a = ka >= p.Tk || (p.key_pad && p.key_pad[(size_t)b * p.Tk + ka]);
  const bool kpad_b = kb >= p.Tk || (p.key_pad && p.key_pad[(size_t)b * p.Tk + kb]);

  fl_load_tile<DK>(sK, p.k, p.k_bs, p.k_hs, p.k_rs, b, h, k0, p.Tk);
  fl_load_tile<DV>(sV, p.v, p.v_bs, p.v_hs, p.v_rs, b, h, k0, p.Tk);
  float dk[DK / 8][4], dv[DV / 8][4];
#pragma unroll
  for (int i = 0; i < DK / 8; i++) dk[i][0] = dk[i][1] = dk[i][2] = dk[i][3] = 0.f;
#pragma unroll
  for (int i = 0; i < DV / 8; i++) dv[i][0] = dv[i][1] = dv[i][2] = dv[i][3] = 0.f;
  const int qstart = p.causal ? k0 : 0;                     // with a causal mask, queries before the key block see none of it

  for (int qt = qstart; qt < p.Tq; qt += FL_ROWS) {
    __syncthreads();
    fl_load_tile<DK>(sQ, p.q, p.q_bs, p.q_hs, p.q_rs, b, h, qt, p.Tq);
    fl_load_tile<DV>(sO, dout, p.o_bs, p.o_hs, p.o_rs, b, h, qt, p.Tq);
    if (threadIdx.x < FL_ROWS) {
      const int qi = qt + threadIdx.x;
      vec[threadIdx.x] = qi < p.Tq ? p.lse[bh * p.Tq + qi] : 0.f;
      vec[FL_ROWS + threadIdx.x] = qi < p.Tq ? delta[bh * p.Tq + qi] : 0.f;
    }
    __syncthreads();
    float s[8][4], dp[8][4];
#pragma unroll
    for (int nb = 0; nb < 8; nb++) s[nb][0] = s[nb][1] = s[nb][2] = s[nb][3] = dp[nb][0] = dp[nb][1] = dp[nb][2] = dp[nb][3] = 0.f;
#pragma unroll
    for (int ks = 0; ks < DK / KS; ks++) {
      const typename F::A a = F::a_feat(sK, PK, warp * 16, ks * KS, g, q);
#pragma unroll
      for (int nb = 0; nb < 8; nb++) F::mma(s[nb], a, F::b_feat(sQ, PK, nb * 8, ks * KS, g, q));     // S^T [keys x queries]
    }
#pragma unroll
    for (int ks = 0; ks < DV / KS; ks++) {
      const typename F::A a = F::a_feat(sV, PV, warp * 16, ks * KS, g, q);
#pragma unroll
      for (int nb = 0; nb < 8; nb++) F::mma(dp[nb], a, F::b_feat(sO, PV, nb * 8, ks * KS, g, q));    // dP^T
    }
#pragma unroll
    for (int nb = 0; nb < 8; nb++)
#pragma unroll
      for (int e = 0; e < 4; e++) {
        const int ql = nb * 8 + 2 * q + (e & 1), qi = qt + ql;
        const int key = (e & 2) ? kb : ka;
        bool masked = ((e & 2) ? kpad_b : kpad_a) || qi >= p.Tq || (p.causal && key > qi);
        if (!masked && p.dense) masked = p.dense[((size_t)b * p.Tq + qi) * p.Tk + key] != 0;
        float pr = 0.f, ds = 0.f;
        if (!masked) {
          const float pe = __expf(s[nb][e] * p.scale - vec[ql]);
          float keep = 1.f;
          if (p.thresh) keep = dropout_keep(p.key, (bh * p.Tq + qi) * (size_t)p.Tk + key, p.thresh) ? p.inv_keep : 0.f;
          pr = pe * keep;
          ds = pe * (dp[nb][e] * keep - vec[FL_ROWS + ql]) * p.scale;
        }
        s[nb][e] = pr;
        dp[nb][e] = ds;
      }
#pragma unroll
    for (int ks = 0; ks < FL_ROWS / KS; ks++) {
      const typename F::A pa = F::a_from_c(s, ks), da = F::a_from_c(dp, ks);
#pragma unroll
      for (int nb = 0; nb < DV / 8; nb++) F::mma(dv[nb], pa, F::b_row(sO, PV, ks * KS, nb * 8, g, q));     // dV += Pd^T dO
#pragma unroll
      for (int nb = 0; nb < DK / 8; nb++) F::mma(dk[nb], da, F::b_row(sQ, PK, ks * KS, nb * 8, g, q));     // dK += dS^T Q
    }
  }
  fl_store_rows<DK>(dk, dk_out, p.k_bs, p.k_hs, p.k_rs, b, h, k0 + warp * 16, p.Tk, g, q, 1.f, 1.f);
  fl_store_rows<DV>(dv, dv_out, p.v_bs, p.v_hs, p.v_rs, b, h, k0 + warp * 16, p.Tk, g, q, 1.f, 1.f);
}

template <int MODE, int DK, int DV>
__global__ void __launch_bounds__(FL_THREADS)
flash_bwd_dq_kernel(const AttnP p, const float* __restrict__ dout, const float* __restrict__ delta, float* __restrict__ dq_out) {
  using F = Fl<MODE>;
  constexpr int PK = DK + 4, PV = DV + 4, KS = F::KS;
  extern __shared__ float fl_smem[];
  float* sQ = fl_smem;
  float* sO = sQ + FL_ROWS * PK;
  float* sK = sO + FL_ROWS * PV;
  float* sV = sK + FL_ROWS * PK;
  uint8_t* pad = reinterpret_cast<uint8_t*>(sV + FL_ROWS * PV);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, q = lane & 3;
  const int q0 = blockIdx.x * FL_ROWS, h = blockIdx.y, b = blockIdx.z;
  const int qa = q0 + warp * 16 + g, qb = qa + 8;
  const size_t bh = (size_t)b * p.H + h;
  const float lse_a = qa < p.Tq ? p.lse[bh * p.Tq + qa] : 0.f, lse_b = qb < p.Tq ? p.lse[bh * p.Tq + qb] : 0.f;
  const float dl_a = qa < p.Tq ? delta[bh * p.Tq + qa] : 0.f, dl_b = qb < p.Tq ? delta[bh * p.Tq + qb] : 0.f;

  fl_load_tile<DK>(sQ, p.q, p.q_bs, p.q_hs, p.q_rs, b, h, q0, p.Tq);
  fl_load_tile<DV>(sO, dout, p.o_bs, p.o_hs, p.o_rs, b, h, q0, p.Tq);
  float dq[DK / 8][4];
#pragma unroll
  for (int i = 0; i < DK / 8; i++) dq[i][0] = dq[i][1] = dq[i][2] = dq[i][3] = 0.f;
  const int kend = p.causal ? min(p.Tk, q0 + FL_ROWS) : p.Tk;     // with a causal mask, keys beyond the tile's last query see nothing

  for (int k0 = 0; k0 < kend; k0 += FL_ROWS) {
    __syncthreads();
    fl_load_tile<DK>(sK, p.k, p.k_bs, p.k_hs, p.k_rs, b, h, k0, p.Tk);
    fl_load_tile<DV>(sV, p.v, p.v_bs, p.v_hs, p.v_rs, b, h, k0, p.Tk);
    if (threadIdx.x < FL_ROWS) {
      const int key = k0 + threadIdx.x;
      pad[threadIdx.x] = (key >= p.Tk || (p.key_pad && p.key_pad[(size_t)b * p.Tk + key])) ? 1 : 0;
    }
    __syncthreads();
    float s[8][4], dp[8][4];
#pragma unroll
    for (int nb = 0; nb < 8; nb++) s[nb][0] = s[nb][1] = s[nb][2] = s[nb][3] = dp[nb][0] = dp[nb][1] = dp[nb][2] = dp[nb][3] = 0.f;
#pragma unroll
    for (int ks = 0; ks < DK / KS; ks++) {
      const typename F::A a = F::a_feat(sQ, PK, warp * 16, ks * KS, g, q);
#pragma unroll
      for (int nb = 0; nb < 8; nb++) F::mma(s[nb], a, F::b_feat(sK, PK, nb * 8, ks * KS, g, q));      // S
    }
#pragma unroll
    for (int ks = 0; ks < DV / KS; ks++) {
      const typename F::A a = F::a_feat(sO, PV, warp * 16, ks * KS, g, q);
#pragma unroll
      for (int nb = 0; nb < 8; nb++) F::mma(dp[nb], a, F::b_feat(sV, PV, nb * 8, ks * KS, g, q));     // dP
    }
#pragma unroll
    for (int nb = 0; nb < 8; nb++)
#pragma unroll
      for (int e = 0; e < 4; e++) {
        const int kl = nb * 8 + 2 * q + (e & 1), key = k0 + kl;
        const bool r1 = (e & 2) != 0;
        const int qi = r1 ? qb : qa;
        const bool masked = qi >= p.Tq || fl_masked(p, pad, b, qi, key, kl);
        float ds = 0.f;
        if (!masked) {
          const float pe = __expf(s[nb][e] * p.scale - (r1 ? lse_b : lse_a));
          float keep = 1.f;
          if (p.thresh) keep = dropout_keep(p.key, (bh * p.Tq + qi) * (size_t)p.Tk + key, p.thresh) ? p.inv_keep : 0.f;
          ds = pe * (dp[nb][e] * keep - (r1 ? dl_b : dl_a)) * p.scale;
        }
        dp[nb][e] = ds;
      }
#pragma unroll
    for (int ks = 0; ks < FL_ROWS / KS; ks++) {
      const typename F::A da = F::a_from_c(dp, ks);
#pragma unroll
      for (int nb = 0; nb < DK / 8; nb++) F::mma(dq[nb], da, F::b_row(sK, PK, ks * KS, nb * 8, g, q));    // dQ += dS K
    }
  }
  fl_store_rows<DK>(dq, dq_out, p.q_bs, p.q_hs, p.q_rs, b, h, q0 + warp * 16, p.Tq, g, q, 1.f, 1.f);
}

// delta[b,h,q] = sum_c dO * O   (one warp per row)
static __global__ void flash_delta_kernel(AttnP p, const float* __restrict__ dout, float* __restrict__ delta) {
  const int w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  const int total = p.B * p.H * p.Tq;
  if (w >= total) return;
  const int q = w % p.Tq, bh = w / p.Tq, h = bh % p.H, b = bh / p.H;
  const float* og = p.o + b * p.o_bs + h * p.o_hs + (long long)q * p.o_rs;
  const float* dg = dout + b * p.o_bs + h * p.o_hs + (long long)q * p.o_rs;
  float s = 0.f;
  for (int c = lane; c < p.dv; c += 32) s += og[c] * dg[c];
  s = warp_sum(s);
  if (lane == 0) delta[w] = s;
}

template <int DK, int DV> constexpr int flash_fwd_smem() { return 4 * FL_ROWS * (2 * (DK + 4) + (DV + 4)) + FL_ROWS; }
template <int DK, int DV> constexpr int flash_bwd_smem() { return 4 * FL_ROWS * (2 * (DK + 4) + 2 * (DV + 4)) + 4 * 2 * FL_ROWS; }

template <int MODE, int DK, int DV>
int flash_fwd(const AttnP& p, cudaStream_t st, const char* what) {
  auto* kern = flash_fwd_kernel<MODE, DK, DV>;
  static bool attr_set[kMaxDevices] = {};
  if (int rc = ensure_dynamic_smem((const void*)kern, flash_fwd_smem<DK, DV>(), attr_set, what)) return rc;
  kern<<<dim3(ceil_div(p.Tq, FL_ROWS), p.H, p.B), FL_THREADS, flash_fwd_smem<DK, DV>(), st>>>(p);
  return check_launch(what);
}

// delta (B*H*Tq floats) is scratch
template <int MODE, int DK, int DV>
int flash_bwd(const AttnP& p, const float* dout, float* dq, float* dk, float* dv, float* delta, cudaStream_t st, const char* what) {
  const int total = p.B * p.H * p.Tq;
  flash_delta_kernel<<<ceil_div(total, 8), 256, 0, st>>>(p, dout, delta);
  if (int rc = check_launch(what)) return rc;
  auto* ka = flash_bwd_dkdv_kernel<MODE, DK, DV>;
  auto* kb = flash_bwd_dq_kernel<MODE, DK, DV>;
  static bool attr_a[kMaxDevices] = {}, attr_b[kMaxDevices] = {};
  if (int rc = ensure_dynamic_smem((const void*)ka, flash_bwd_smem<DK, DV>(), attr_a, what)) return rc;
  if (int rc = ensure_dynamic_smem((const void*)kb, flash_bwd_smem<DK, DV>(), attr_b, what)) return rc;
  ka<<<dim3(ceil_div(p.Tk, FL_ROWS), p.H, p.B), FL_THREADS, flash_bwd_smem<DK, DV>(), st>>>(p, dout, delta, dk, dv);
  if (int rc = check_launch(what)) return rc;
  kb<<<dim3(ceil_div(p.Tq, FL_ROWS), p.H, p.B), FL_THREADS, flash_bwd_smem<DK, DV>(), st>>>(p, dout, delta, dq);
  return check_launch(what);
}

}  // namespace tc

// precision 1: operands rounded to TF32 (nearest) -- letting the tensor core truncate fp32 operands instead biases every
// product toward zero, which acts like a 0.1% temperature error on the softmax.  dk, dv in {32, 64}; Tk <= 448 (the ABI's bound)
constexpr int ATT_MAX_TK = 448;

int sdpa_fwd_tc(const AttnP& p, cudaStream_t st) {
  using namespace tc;
  B200_REQUIRE(p.Tk <= ATT_MAX_TK, B200ASR_BAD_SHAPE, "sdpa_fwd (tensor cores): Tk=%d exceeds %d keys; use precision 0", p.Tk, ATT_MAX_TK);
  B200_REQUIRE(p.H <= 65535 && p.B <= 65535, B200ASR_BAD_SHAPE, "sdpa_fwd (tensor cores): grid too large");
  if (p.dk == 64 && p.dv == 64) return flash_fwd<1, 64, 64>(p, st, "tc_sdpa_fwd");
  if (p.dk == 32 && p.dv == 32) return flash_fwd<1, 32, 32>(p, st, "tc_sdpa_fwd");
  if (p.dk == 64 && p.dv == 32) return flash_fwd<1, 64, 32>(p, st, "tc_sdpa_fwd");
  if (p.dk == 32 && p.dv == 64) return flash_fwd<1, 32, 64>(p, st, "tc_sdpa_fwd");
  set_error("sdpa_fwd (tensor cores): (dk=%d, dv=%d) unsupported, needs dk, dv in {32, 64}; use precision 0", p.dk, p.dv);
  return B200ASR_BAD_SHAPE;
}

int sdpa_bwd_tc(const AttnP& p, const float* dout, float* dq, float* dk, float* dv, float* delta, cudaStream_t st) {
  using namespace tc;
  B200_REQUIRE(p.H <= 65535 && p.B <= 65535, B200ASR_BAD_SHAPE, "sdpa_bwd (tensor cores): grid too large");
  if (p.dk == 64 && p.dv == 64) return flash_bwd<1, 64, 64>(p, dout, dq, dk, dv, delta, st, "tc_sdpa_bwd");
  if (p.dk == 32 && p.dv == 32) return flash_bwd<1, 32, 32>(p, dout, dq, dk, dv, delta, st, "tc_sdpa_bwd");
  if (p.dk == 64 && p.dv == 32) return flash_bwd<1, 64, 32>(p, dout, dq, dk, dv, delta, st, "tc_sdpa_bwd");
  if (p.dk == 32 && p.dv == 64) return flash_bwd<1, 32, 64>(p, dout, dq, dk, dv, delta, st, "tc_sdpa_bwd");
  set_error("sdpa_bwd (tensor cores): (dk=%d, dv=%d) unsupported, needs dk, dv in {32, 64}; use precision 0", p.dk, p.dv);
  return B200ASR_BAD_SHAPE;
}

// bf16x3 (every product hi*hi + hi*lo + lo*hi over x ~ bf16 hi + bf16 lo): dk = dv = 64, Tk <= 448 in the forward
int sdpa_fused_fwd_tc(const AttnP& p, cudaStream_t st) {
  B200_REQUIRE(p.dk == 64 && p.dv == 64, B200ASR_BAD_SHAPE, "sdpa_fused: needs dk = dv = 64 (dk=%d dv=%d); use the materialised path", p.dk, p.dv);
  B200_REQUIRE(p.H <= 65535 && p.B <= 65535, B200ASR_BAD_SHAPE, "sdpa_fused: grid too large");
  B200_REQUIRE(p.Tk <= ATT_MAX_TK, B200ASR_BAD_SHAPE, "sdpa_fused_fwd: Tk=%d exceeds %d keys; use the materialised path", p.Tk, ATT_MAX_TK);
  return tc::flash_fwd<6, 64, 64>(p, st, "sdpa_fused_fwd");
}

int sdpa_fused_bwd_tc(const AttnP& p, const float* dout, float* dq, float* dk, float* dv, float* delta, cudaStream_t st) {
  B200_REQUIRE(p.dk == 64 && p.dv == 64, B200ASR_BAD_SHAPE, "sdpa_fused: needs dk = dv = 64 (dk=%d dv=%d); use the materialised path", p.dk, p.dv);
  B200_REQUIRE(p.H <= 65535 && p.B <= 65535, B200ASR_BAD_SHAPE, "sdpa_fused: grid too large");
  return tc::flash_bwd<6, 64, 64>(p, dout, dq, dk, dv, delta, st, "sdpa_fused_bwd");
}

}  // namespace b200asr
