// Attention parameter block shared by the CUDA-core and tensor-core kernels.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace b200asr {

struct AttnP {
  const float *q, *k, *v;
  float* o;
  float* lse;
  long long q_bs, q_hs, q_rs, k_bs, k_hs, k_rs, v_bs, v_hs, v_rs, o_bs, o_hs, o_rs;
  const uint8_t* key_pad;  // [B,Tk] or nullptr
  const uint8_t* dense;    // [B,Tq,Tk] or nullptr
  int causal, B, H, Tq, Tk, dk, dv;
  float scale;
  uint32_t thresh;   // 16-bit dropout threshold, 0 = no dropout
  float inv_keep;
  uint64_t key;      // dropout key derived from (seed, offset)
};

int sdpa_fwd_simt(const AttnP& p, cudaStream_t st);
int sdpa_bwd_simt(const AttnP& p, const float* dout, float* dq, float* dk, float* dv, float* delta, cudaStream_t st);
// tensor-core kernels (tc_flash.cu): TF32 and the bf16x3 "fused" variant
int sdpa_fwd_tc(const AttnP& p, cudaStream_t st);
int sdpa_bwd_tc(const AttnP& p, const float* dout, float* dq, float* dk, float* dv, float* delta, cudaStream_t st);
int sdpa_fused_fwd_tc(const AttnP& p, cudaStream_t st);
int sdpa_fused_bwd_tc(const AttnP& p, const float* dout, float* dq, float* dk, float* dv, float* delta, cudaStream_t st);
// attention probabilities from the forward's log-sum-exp (p.lse), written through p.o / o_bs / o_hs / o_rs
int sdpa_probs_simt(const AttnP& p, cudaStream_t st);
int sdpa_probs_tc(const AttnP& p, int mode, cudaStream_t st);    // mode 1 = TF32, 6 = bf16x3

}  // namespace b200asr
