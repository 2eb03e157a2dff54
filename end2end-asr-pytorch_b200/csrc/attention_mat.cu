// "Materialised" scaled-dot-product attention (precision 3 = 3xTF32, precision 1 = TF32): the contractions run as batched
// tensor-core GEMMs (tc_bgemm.cu) and the masked softmax / dropout and its backward are exact fp32 row kernels in between.
//
//   fwd:  S = Q K^T                  (bgemm, per head, written into `probs`)
//         P = softmax(mask(S * scale)); Pd = dropout(P)      (softmax_fwd_kernel; P kept for backward, Pd only if p > 0)
//         O = Pd V                   (bgemm, written straight into the token-major output)
//   bwd:  dV = Pd^T dO ; dPd = dO V^T (bgemm) ; dS = scale * P (.) (keep*dPd/(1-p) - rowsum(...))  (softmax_bwd_kernel)
//         dQ = dS K ; dK = dS^T Q    (bgemm)
//
// This is what models/common_layers.py:211-225 does op for op (bmm, masked_fill, softmax, dropout, bmm), so the
// score tensor does hit HBM -- at T_e = 200 that is 41 MB per layer, ~25 us of traffic -- but every product is
// fp32-grade (3xTF32) and the dP - delta subtraction of the softmax backward happens in fp32 on fp32-grade inputs,
// which is exactly what the single-pass TF32 flash kernel (tc_attention*.cu) cannot offer (DESIGN.md section 4).
// Dropout uses the same counter-based stream and indexing as attention_simt.cu, so both paths draw identical masks.
#include <math.h>

#include "../../include/b200asr.h"
#include "attention.h"
#include "common.cuh"
#include "kernels.h"

namespace b200asr {

struct SoftP {
  const uint8_t* key_pad;  // [B,Tk] or nullptr
  const uint8_t* dense;    // [B,Tq,Tk] or nullptr
  int causal, H, Tq, Tk, ldp;
  long long rows;          // B * H * Tq
  float scale, inv_keep;
  uint32_t thresh;
  uint64_t key;
};

__device__ __forceinline__ void keep4(const SoftP& p, long long row, int col, bool (&kp)[4]) {
  const uint64_t idx = (uint64_t)row * (uint64_t)p.Tk + (uint64_t)col;
  if ((p.Tk & 3) == 0) {          // the 4 columns share one 64-bit draw (16 bits each)
    const uint64_t r = dropout_bits4(p.key, idx >> 2);
#pragma unroll
    for (int j = 0; j < 4; j++) kp[j] = ((uint32_t)(r >> (16 * j)) & 0xFFFFu) >= p.thresh;
  } else {
#pragma unroll
    for (int j = 0; j < 4; j++) kp[j] = dropout_keep(p.key, idx + j, p.thresh);
  }
}

// one warp per (b, h, q) row; the row (<= 128 * NV floats) lives in registers between the passes
template <int NV>
__global__ void __launch_bounds__(256) softmax_fwd_kernel(SoftP p, float* __restrict__ probs, float* __restrict__ probs_drop) {
  griddep_launch();      // programmatic dependent launch (common.cuh)
  griddep_wait();
  const int lane = threadIdx.x & 31;
  const long long row = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (row >= p.rows) return;
  const int q = (int)(row % p.Tq);
  const int b = (int)(row / ((long long)p.Tq * p.H));
  float* prow = probs + row * p.ldp;
  const uint8_t* kp_row = p.key_pad ? p.key_pad + (size_t)b * p.Tk : nullptr;
  const uint8_t* dn_row = p.dense ? p.dense + ((size_t)b * p.Tq + q) * p.Tk : nullptr;
  float4 x[NV];
  float mx = -INFINITY;
#pragma unroll
  for (int i = 0; i < NV; i++) {
    const int col = 4 * (lane + 32 * i);
    float4 v = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
    if (col < p.ldp) {
      v = *reinterpret_cast<const float4*>(prow + col);
      float* e = reinterpret_cast<float*>(&v);
#pragma unroll
      for (int j = 0; j < 4; j++) {
        const int key = col + j;
        bool masked = key >= p.Tk || (p.causal && key > q);
        if (!masked && kp_row) masked = kp_row[key] != 0;
        if (!masked && dn_row) masked = dn_row[key] != 0;
        e[j] = masked ? -INFINITY : e[j] * p.scale;
        mx = fmaxf(mx, e[j]);
      }
    }
    x[i] = v;
  }
  mx = warp_max(mx);
  const float m_safe = (mx == -INFINITY) ? 0.f : mx;
  float sum = 0.f;
#pragma unroll
  for (int i = 0; i < NV; i++) {
    float* e = reinterpret_cast<float*>(&x[i]);
#pragma unroll
    for (int j = 0; j < 4; j++) { e[j] = expf(e[j] - m_safe); sum += e[j]; }
  }
  sum = warp_sum(sum);
  const float inv = 1.f / sum;     // fully masked row: 0 * inf = NaN, like softmax over all -inf in the reference (and attention_simt.cu)
#pragma unroll
  for (int i = 0; i < NV; i++) {
    const int col = 4 * (lane + 32 * i);
    if (col >= p.ldp) continue;
    float4 v = x[i];
    v.x *= inv; v.y *= inv; v.z *= inv; v.w *= inv;
    *reinterpret_cast<float4*>(prow + col) = v;
    if (probs_drop) {
      bool kp[4];
      keep4(p, row, col, kp);
      float4 d = make_float4(kp[0] ? v.x * p.inv_keep : 0.f, kp[1] ? v.y * p.inv_keep : 0.f,
                             kp[2] ? v.z * p.inv_keep : 0.f, kp[3] ? v.w * p.inv_keep : 0.f);
      *reinterpret_cast<float4*>(probs_drop + row * p.ldp + col) = d;
    }
  }
}

// dS = scale * P (.) (dP - sum_j dP_j P_j),  dP = keep ? dPd / (1 - p) : 0   (in place over dPd)
template <int NV>
__global__ void __launch_bounds__(256) softmax_bwd_kernel(SoftP p, const float* __restrict__ probs, float* __restrict__ dpd) {
  griddep_launch();      // programmatic dependent launch (common.cuh)
  griddep_wait();
  const int lane = threadIdx.x & 31;
  const long long row = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (row >= p.rows) return;
  const float* prow = probs + row * p.ldp;
  float* drow = dpd + row * p.ldp;
  float4 pv[NV], dv[NV];
  float delta = 0.f;
#pragma unroll
  for (int i = 0; i < NV; i++) {
    const int col = 4 * (lane + 32 * i);
    pv[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    dv[i] = pv[i];
    if (col < p.ldp) {
      pv[i] = *reinterpret_cast<const float4*>(prow + col);
      float4 d = *reinterpret_cast<const float4*>(drow + col);
      if (p.thresh) {
        bool kp[4];
        keep4(p, row, col, kp);
        d.x = kp[0] ? d.x * p.inv_keep : 0.f; d.y = kp[1] ? d.y * p.inv_keep : 0.f;
        d.z = kp[2] ? d.z * p.inv_keep : 0.f; d.w = kp[3] ? d.w * p.inv_keep : 0.f;
      }
      dv[i] = d;
      delta += d.x * pv[i].x + d.y * pv[i].y + d.z * pv[i].z + d.w * pv[i].w;   // P = 0 at masked / padding columns
    }
  }
  delta = warp_sum(delta);
#pragma unroll
  for (int i = 0; i < NV; i++) {
    const int col = 4 * (lane + 32 * i);
    if (col >= p.ldp) continue;
    const float4 d = dv[i], q = pv[i];
    *reinterpret_cast<float4*>(drow + col) = make_float4(p.scale * q.x * (d.x - delta), p.scale * q.y * (d.y - delta),
                                                         p.scale * q.z * (d.z - delta), p.scale * q.w * (d.w - delta));
  }
}

template <bool FWD>
static int launch_softmax(const SoftP& p, float* a, float* b, cudaStream_t st) {
  const int nv = ceil_div(p.ldp, 128);
  const unsigned grid = (unsigned)((p.rows + 7) / 8);
#define CASE(NVv)                                                                                   \
  if (nv <= NVv) {                                                                                  \
    if constexpr (FWD) launch_pdl(softmax_fwd_kernel<NVv>, dim3(grid), dim3(256), 0, st, p, a, (float*)b);          \
    else launch_pdl(softmax_bwd_kernel<NVv>, dim3(grid), dim3(256), 0, st, p, (const float*)a, b);   \
    return check_launch(FWD ? "softmax_fwd" : "softmax_bwd");                                       \
  }
  CASE(1) CASE(2) CASE(4) CASE(8) CASE(16)
#undef CASE
  set_error("sdpa_mat: Tk=%d > 2048 is not supported by the materialised path (use precision 0)", p.Tk);
  return B200ASR_BAD_SHAPE;
}

static int nsplit_of(int precision) { return precision == B200ASR_PREC_TF32X3 ? 3 : (precision == B200ASR_PREC_TF32 ? 1 : 0); }

static int check_common(int B, int H, int Tq, int Tk, int dk, int dv, float p_drop, int precision, const void* probs,
                        const void* probs_drop) {
  B200_REQUIRE(B > 0 && H > 0 && Tq > 0 && Tk > 0, B200ASR_BAD_SHAPE, "sdpa_mat: empty problem");
  B200_REQUIRE(dk % 32 == 0 && dv % 32 == 0 && dk <= 256 && dv <= 256, B200ASR_BAD_SHAPE,
               "sdpa_mat: dk=%d dv=%d must be multiples of 32 (<= 256)", dk, dv);
  B200_REQUIRE(nsplit_of(precision) != 0, B200ASR_BAD_ARG, "sdpa_mat: precision %d unsupported (1 = TF32, 3 = 3xTF32)", precision);
  B200_REQUIRE(p_drop >= 0.f && p_drop < 1.f, B200ASR_BAD_ARG, "sdpa_mat: p_drop=%f", p_drop);
  B200_REQUIRE(probs && aligned16(probs) && (p_drop == 0.f || (probs_drop && aligned16(probs_drop))), B200ASR_BAD_ARG,
               "sdpa_mat: probability buffers missing or misaligned");
  return B200ASR_OK;
}

}  // namespace b200asr

using namespace b200asr;

extern "C" {

size_t b200asr_sdpa_mat_ws_bytes(int B, int H, int Tq, int Tk) {
  return sizeof(float) * (size_t)B * H * Tq * (size_t)((Tk + 3) & ~3);
}

int b200asr_sdpa_mat_fwd(const float* q, const float* k, const float* v, long long q_bs, long long q_hs, long long q_rs,
                         long long k_bs, long long k_hs, long long k_rs, long long v_bs, long long v_hs, long long v_rs,
                         const uint8_t* key_pad, const uint8_t* dense_mask, int causal, float* out, long long o_bs,
                         long long o_hs, long long o_rs, float* probs, float* probs_drop, int B, int H, int Tq, int Tk,
                         int dk, int dv, float scale, float p_drop, uint64_t seed, uint64_t offset, int precision,
                         b200asr_stream_t stream) {
  B200_REQUIRE(q && k && v && out, B200ASR_BAD_ARG, "sdpa_mat_fwd: null pointer");
  int rc = check_common(B, H, Tq, Tk, dk, dv, p_drop, precision, probs, probs_drop);
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  const int ns = nsplit_of(precision), ldp = (Tk + 3) & ~3;
  const long long z_stride = (long long)Tq * ldp;
  BOperand Q{q, q_bs, q_hs, q_rs, 1, Tq, dk}, K{k, k_bs, k_hs, k_rs, 1, Tk, dk}, V{v, v_bs, v_hs, v_rs, 1, Tk, dv};
  rc = bgemm_tc(Q, true, K, true, probs, z_stride * H, z_stride, ldp, Tq, Tk, dk, B, H, 1.f, ns, st);
  if (rc) return rc;
  SoftP sp{key_pad, dense_mask, causal, H, Tq, Tk, ldp, (long long)B * H * Tq, scale, dropout_inv_keep(p_drop),
           p_drop > 0.f ? dropout_thresh16(p_drop) : 0u, dropout_key(seed, offset)};
  float* pd = sp.thresh ? probs_drop : nullptr;
  rc = launch_softmax<true>(sp, probs, pd, st);
  if (rc) return rc;
  BOperand P{pd ? pd : probs, z_stride, 0, ldp, 0, Tq, Tk};
  return bgemm_tc(P, true, V, false, out, o_bs, o_hs, (int)o_rs, Tq, dv, Tk, B, H, 1.f, ns, st);
}

int b200asr_sdpa_mat_bwd(const float* dout, const float* q, const float* k, const float* v, long long q_bs, long long q_hs,
                         long long q_rs, long long k_bs, long long k_hs, long long k_rs, long long v_bs, long long v_hs,
                         long long v_rs, long long o_bs, long long o_hs, long long o_rs, const float* probs,
                         const float* probs_drop, float* dq, float* dk_out, float* dv_out, float* dp_ws, int B, int H,
                         int Tq, int Tk, int dk, int dv, float scale, float p_drop, uint64_t seed, uint64_t offset,
                         int precision, b200asr_stream_t stream) {
  B200_REQUIRE(dout && q && k && v && dq && dk_out && dv_out && dp_ws, B200ASR_BAD_ARG, "sdpa_mat_bwd: null pointer");
  int rc = check_common(B, H, Tq, Tk, dk, dv, p_drop, precision, probs, probs_drop);
  if (rc) return rc;
  B200_REQUIRE(aligned16(dp_ws), B200ASR_BAD_ALIGN, "sdpa_mat_bwd: workspace alignment");
  cudaStream_t st = (cudaStream_t)stream;
  const int ns = nsplit_of(precision), ldp = (Tk + 3) & ~3;
  const long long z_stride = (long long)Tq * ldp;
  const float* pd = p_drop > 0.f ? probs_drop : probs;
  BOperand Q{q, q_bs, q_hs, q_rs, 1, Tq, dk}, K{k, k_bs, k_hs, k_rs, 1, Tk, dk}, V{v, v_bs, v_hs, v_rs, 1, Tk, dv};
  BOperand dO{dout, o_bs, o_hs, o_rs, 1, Tq, dv}, Pd{pd, z_stride, 0, ldp, 0, Tq, Tk}, dS{dp_ws, z_stride, 0, ldp, 0, Tq, Tk};
  // dV[Tk,dv] = Pd^T dO          (contraction over Tq: both operands MN-major)
  rc = bgemm_tc(Pd, false, dO, false, dv_out, v_bs, v_hs, (int)v_rs, Tk, dv, Tq, B, H, 1.f, ns, st);
  if (rc) return rc;
  // dPd[Tq,Tk] = dO V^T          (contraction over dv: both K-major)
  rc = bgemm_tc(dO, true, V, true, dp_ws, z_stride * H, z_stride, ldp, Tq, Tk, dv, B, H, 1.f, ns, st);
  if (rc) return rc;
  SoftP sp{nullptr, nullptr, 0, H, Tq, Tk, ldp, (long long)B * H * Tq, scale, dropout_inv_keep(p_drop),
           p_drop > 0.f ? dropout_thresh16(p_drop) : 0u, dropout_key(seed, offset)};
  rc = launch_softmax<false>(sp, const_cast<float*>(probs), dp_ws, st);
  if (rc) return rc;
  // dQ[Tq,dk] = dS K             (A K-major over Tk, B MN-major)
  rc = bgemm_tc(dS, true, K, false, dq, q_bs, q_hs, (int)q_rs, Tq, dk, Tk, B, H, 1.f, ns, st);
  if (rc) return rc;
  // dK[Tk,dk] = dS^T Q           (contraction over Tq: both MN-major)
  return bgemm_tc(dS, false, Q, false, dk_out, k_bs, k_hs, (int)k_rs, Tk, dk, Tq, B, H, 1.f, ns, st);
}

}  // extern "C"
