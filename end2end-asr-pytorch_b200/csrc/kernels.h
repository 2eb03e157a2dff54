// Internal launcher declarations shared between translation units of libb200asr.
#pragma once
#include <cuda_runtime.h>

namespace b200asr {

// fp32 CUDA-core GEMM: C[m,n] = sum_k A(m,k) B(k,n); *_kmaj: contraction index contiguous.
int gemm_simt(const float* A, bool a_kmaj, int lda, const float* B, bool b_kmaj, int ldb, float* C, int ldc, int M,
              int N, int K, const float* bias, int relu, const float* relu_mask, int accumulate, bool allow_split,
              cudaStream_t st);
int launch_colsum(const float* X, float* out, int M, int N, int accumulate, cudaStream_t st);

// Tensor-core GEMM (tc_gemm.cu).  nsplit = 1 (TF32) or 3 (3xTF32).  Returns B200ASR_BAD_SHAPE when the
// shape/alignment cannot be expressed as TMA tiles (callers turn that into an error, never a fallback).
int gemm_tc(const float* A, bool a_kmaj, int lda, const float* B, bool b_kmaj, int ldb, float* C, int ldc, int M,
            int N, int K, const float* bias, int relu, const float* relu_mask, int accumulate, int nsplit,
            cudaStream_t st, const void* b_split = nullptr, int b_rows = 0, float* rowsum = nullptr);
// nsplit = 2 (bf16) / 6 (bf16x3): A must be K-major fp32; B is ignored and b_split is REQUIRED: the K-major bf16 operand
// [1 or 2][b_rows][ldb] (ldb % 8 == 0) written by b200asr_split_bf16.
// rowsum: optional [M] += sum_k A(m,k), fused into the kernel when both operands are MN-major and nsplit == 3 (the
// bias gradient of the weight-gradient GEMM); gemm_tc_fuses_rowsum() tells the caller whether it will be.
bool gemm_tc_fuses_rowsum(bool a_kmaj, bool b_kmaj, int nsplit);
// b_split: B operand pre-split as [2][b_rows][ldb] (hi | lo), 3xTF32 only -- the kernel then skips its own B split.

// Batched tensor-core GEMM (tc_bgemm.cu): C_z[M,N] = alpha * A_z B_z for z = (batch, head), operands addressed in place.
// An operand is a logical [rows x cols] matrix per z, contiguous along cols; element (b, h, r, c) lives at
// p + b*bs + h*hs + r*rs + c when heads != 0, and at p + z*bs + r*rs + c (z = b*H + h) when heads == 0.
// K-major use: cols = contraction; MN-major use: rows = contraction.
struct BOperand { const float* p; long long bs, hs, rs; int heads, rows, cols; };
int bgemm_tc(const BOperand& A, bool a_kmaj, const BOperand& B, bool b_kmaj, float* C, long long c_bs, long long c_hs, int ldc,
             int M, int N, int K, int Bsz, int H, float alpha, int nsplit, cudaStream_t st);

// Tensor-core implicit-GEMM convolution (tc_conv.cu); takes K-major repacked weights wk[9][Cout][Cin]
// (conv_repack_k_kernel); the weight-gradient variant takes/produces dwr[9][Ci][Co].
int conv3x3_tc(const float* in, const float* wr, const float* bias, const float* mask, float* out, int B, int T, int F,
               int Cin, int Cout, int relu, int precision, cudaStream_t st);
// 3xTF32 forward / data gradient with the input patch (incl. halo) fetched once per 32-channel slice (tc_conv_halo.cu);
// conv3x3_tc dispatches to it for precision 3 (B200ASR_CONV_HALO=0 selects the tap-shifted engine policy instead).
// mode 3 = 3xTF32 (fp32 hi | lo weights), 6 = bf16x3 / 2 = bf16 (bf16 weights from conv_repack_k_bf16)
int conv3x3_tc_halo(const float* in, const void* wk, const float* bias, const float* mask, float* out, int B, int T, int F,
                    int Cin, int Cout, int relu, int mode, cudaStream_t st, void* out16 = nullptr, float* pool = nullptr);
// out16: optional bf16 hi | lo pairs [2][B,T,F,Cout] of the output, written by the epilogue next to `out`
int conv3x3_wgrad_tc(const float* x, const float* dy, float* dwr, int B, int T, int F, int Ci, int Co, int precision,
                     cudaStream_t st, float* dbias = nullptr, int* dbias_done = nullptr, const void* dy16 = nullptr);
// dy16 (bf16 modes only): dy as bf16 hi | lo pairs [2][B,T,F,Co] written by its producer -> B tiles arrive by TMA
// dbias: optional [Co] bias gradient; *dbias_done = 1 when the kernel produced it (3xTF32), else the caller must

}  // namespace b200asr
