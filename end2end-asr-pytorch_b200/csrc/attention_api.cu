// b200asr_sdpa_fwd / _bwd and b200asr_sdpa_fused_fwd / _bwd: argument checking and precision dispatch.
#include "../../include/b200asr.h"
#include "attention.h"
#include "common.cuh"

using namespace b200asr;

static int fill(AttnP& p, const float* q, const float* k, const float* v, float* out, float* lse, long long q_bs,
                long long q_hs, long long q_rs, long long k_bs, long long k_hs, long long k_rs, long long v_bs,
                long long v_hs, long long v_rs, long long o_bs, long long o_hs, long long o_rs, const uint8_t* key_pad,
                const uint8_t* dense_mask, int causal, int B, int H, int Tq, int Tk, int dk, int dv, float scale,
                float p_drop, uint64_t seed, uint64_t offset) {
  B200_REQUIRE(q && k && v && out && lse, B200ASR_BAD_ARG, "sdpa: null pointer");
  B200_REQUIRE(B > 0 && H > 0 && Tq > 0 && Tk > 0, B200ASR_BAD_SHAPE, "sdpa: empty problem B=%d H=%d Tq=%d Tk=%d", B, H, Tq, Tk);
  B200_REQUIRE((dk == 16 || dk == 32 || dk == 64 || dk == 128) && (dv == 16 || dv == 32 || dv == 64 || dv == 128),
               B200ASR_BAD_SHAPE, "sdpa: dk=%d dv=%d must be in {16,32,64,128}", dk, dv);
  B200_REQUIRE(q_rs % 4 == 0 && k_rs % 4 == 0 && v_rs % 4 == 0 && o_rs % 4 == 0 && q_bs % 4 == 0 && q_hs % 4 == 0 &&
                   k_bs % 4 == 0 && k_hs % 4 == 0 && v_bs % 4 == 0 && v_hs % 4 == 0 && o_bs % 4 == 0 && o_hs % 4 == 0,
               B200ASR_BAD_ALIGN, "sdpa: strides must be multiples of 4 elements");
  B200_REQUIRE(aligned16(q) && aligned16(k) && aligned16(v) && aligned16(out), B200ASR_BAD_ALIGN, "sdpa: pointers must be 16-byte aligned");
  B200_REQUIRE(p_drop >= 0.f && p_drop < 1.f, B200ASR_BAD_ARG, "sdpa: p_drop=%f", p_drop);
  p.q = q; p.k = k; p.v = v; p.o = out; p.lse = lse;
  p.q_bs = q_bs; p.q_hs = q_hs; p.q_rs = q_rs; p.k_bs = k_bs; p.k_hs = k_hs; p.k_rs = k_rs;
  p.v_bs = v_bs; p.v_hs = v_hs; p.v_rs = v_rs; p.o_bs = o_bs; p.o_hs = o_hs; p.o_rs = o_rs;
  p.key_pad = key_pad; p.dense = dense_mask; p.causal = causal;
  p.B = B; p.H = H; p.Tq = Tq; p.Tk = Tk; p.dk = dk; p.dv = dv; p.scale = scale;
  p.thresh = p_drop > 0.f ? dropout_thresh16(p_drop) : 0u;
  p.inv_keep = dropout_inv_keep(p_drop);
  p.key = dropout_key(seed, offset);
  return B200ASR_OK;
}

extern "C" {

int b200asr_sdpa_fwd(const float* q, const float* k, const float* v, long long q_bs, long long q_hs, long long q_rs,
                     long long k_bs, long long k_hs, long long k_rs, long long v_bs, long long v_hs, long long v_rs,
                     const uint8_t* key_pad, const uint8_t* dense_mask, int causal, float* out, long long o_bs,
                     long long o_hs, long long o_rs, float* lse, int B, int H, int Tq, int Tk, int dk, int dv, float scale,
                     float p_drop, uint64_t seed, uint64_t offset, int precision, b200asr_stream_t stream) {
  AttnP p;
  int rc = fill(p, q, k, v, out, lse, q_bs, q_hs, q_rs, k_bs, k_hs, k_rs, v_bs, v_hs, v_rs, o_bs, o_hs, o_rs, key_pad,
                dense_mask, causal, B, H, Tq, Tk, dk, dv, scale, p_drop, seed, offset);
  if (rc) return rc;
  if (precision == B200ASR_PREC_FP32) return sdpa_fwd_simt(p, (cudaStream_t)stream);
  if (precision == B200ASR_PREC_TF32) return sdpa_fwd_tc(p, (cudaStream_t)stream);
  set_error("sdpa_fwd: precision %d unsupported (0 = fp32 CUDA cores, 1 = TF32 tensor cores)", precision);
  return B200ASR_BAD_ARG;
}

int b200asr_sdpa_bwd(const float* dout, const float* q, const float* k, const float* v, const float* out,
                     const float* lse, long long q_bs, long long q_hs, long long q_rs, long long k_bs, long long k_hs,
                     long long k_rs, long long v_bs, long long v_hs, long long v_rs, long long o_bs, long long o_hs,
                     long long o_rs, const uint8_t* key_pad, const uint8_t* dense_mask, int causal, float* dq,
                     float* dk_out, float* dv_out, float* delta_ws, int B, int H, int Tq, int Tk, int dk, int dv,
                     float scale, float p_drop, uint64_t seed, uint64_t offset, int precision, b200asr_stream_t stream) {
  B200_REQUIRE(dout && dq && dk_out && dv_out && delta_ws, B200ASR_BAD_ARG, "sdpa_bwd: null pointer");
  B200_REQUIRE(aligned16(dout) && aligned16(dq) && aligned16(dk_out) && aligned16(dv_out), B200ASR_BAD_ALIGN, "sdpa_bwd: alignment");
  AttnP p;
  int rc = fill(p, q, k, v, const_cast<float*>(out), const_cast<float*>(lse), q_bs, q_hs, q_rs, k_bs, k_hs, k_rs, v_bs,
                v_hs, v_rs, o_bs, o_hs, o_rs, key_pad, dense_mask, causal, B, H, Tq, Tk, dk, dv, scale, p_drop, seed, offset);
  if (rc) return rc;
  if (precision == B200ASR_PREC_FP32) return sdpa_bwd_simt(p, dout, dq, dk_out, dv_out, delta_ws, (cudaStream_t)stream);
  if (precision == B200ASR_PREC_TF32) return sdpa_bwd_tc(p, dout, dq, dk_out, dv_out, delta_ws, (cudaStream_t)stream);
  set_error("sdpa_bwd: precision %d unsupported", precision);
  return B200ASR_BAD_ARG;
}

// the fused workspaces keep their sizes: ws16 is reserved, ws_bwd = [2][B*H*Tq*64 rounded up to 64] bf16 slots, then delta
static size_t ws16_elems(int B, int H, int T) { return ((size_t)B * H * T * 64 + 63) / 64 * 64; }

size_t b200asr_sdpa_fused_ws_bytes(int B, int H, int Tq, int Tk) {
  return 2 * (2 * ws16_elems(B, H, Tq) + 4 * ws16_elems(B, H, Tk));
}

size_t b200asr_sdpa_fused_bwd_ws_bytes(int B, int H, int Tq) {
  return 2 * 2 * ws16_elems(B, H, Tq) + sizeof(float) * (((size_t)B * H * Tq + 3) / 4 * 4);
}

int b200asr_sdpa_fused_fwd(const float* q, const float* k, const float* v, long long q_bs, long long q_hs, long long q_rs,
                           long long k_bs, long long k_hs, long long k_rs, long long v_bs, long long v_hs, long long v_rs,
                           const uint8_t* key_pad, const uint8_t* dense_mask, int causal, float* out, long long o_bs,
                           long long o_hs, long long o_rs, float* lse, void* ws16, int B, int H, int Tq, int Tk, int dk, int dv,
                           float scale, float p_drop, uint64_t seed, uint64_t offset, b200asr_stream_t stream) {
  B200_REQUIRE(ws16 && aligned16(ws16), B200ASR_BAD_ARG, "sdpa_fused_fwd: workspace");
  AttnP p;
  int rc = fill(p, q, k, v, out, lse, q_bs, q_hs, q_rs, k_bs, k_hs, k_rs, v_bs, v_hs, v_rs, o_bs, o_hs, o_rs, key_pad,
                dense_mask, causal, B, H, Tq, Tk, dk, dv, scale, p_drop, seed, offset);
  return rc ? rc : sdpa_fused_fwd_tc(p, (cudaStream_t)stream);
}

int b200asr_sdpa_fused_bwd(const float* dout, const float* q, const float* k, const float* v, const float* out, const float* lse,
                           long long q_bs, long long q_hs, long long q_rs, long long k_bs, long long k_hs, long long k_rs,
                           long long v_bs, long long v_hs, long long v_rs, long long o_bs, long long o_hs, long long o_rs,
                           const uint8_t* key_pad, const uint8_t* dense_mask, int causal, float* dq, float* dk_out, float* dv_out,
                           const void* ws16, void* ws_bwd, int B, int H, int Tq, int Tk, int dk, int dv, float scale, float p_drop,
                           uint64_t seed, uint64_t offset, b200asr_stream_t stream) {
  B200_REQUIRE(dout && dq && dk_out && dv_out && ws16 && ws_bwd, B200ASR_BAD_ARG, "sdpa_fused_bwd: null pointer");
  B200_REQUIRE(aligned16(dout) && aligned16(dq) && aligned16(dk_out) && aligned16(dv_out) && aligned16(ws_bwd), B200ASR_BAD_ALIGN, "sdpa_fused_bwd: alignment");
  AttnP p;
  int rc = fill(p, q, k, v, const_cast<float*>(out), const_cast<float*>(lse), q_bs, q_hs, q_rs, k_bs, k_hs, k_rs, v_bs,
                v_hs, v_rs, o_bs, o_hs, o_rs, key_pad, dense_mask, causal, B, H, Tq, Tk, dk, dv, scale, p_drop, seed, offset);
  if (rc) return rc;
  float* delta = (float*)((uint16_t*)ws_bwd + 2 * ws16_elems(B, H, Tq));
  return sdpa_fused_bwd_tc(p, dout, dq, dk_out, dv_out, delta, (cudaStream_t)stream);
}

}  // extern "C"
