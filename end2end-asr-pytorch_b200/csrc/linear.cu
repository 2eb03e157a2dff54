// Dense-layer entry points (forward, data gradient, weight gradient) -- see include/b200asr.h.
#include "../../include/b200asr.h"
#include "common.cuh"
#include "kernels.h"

using namespace b200asr;

static int gemm_dispatch(const float* A, bool ak, int lda, const float* B, bool bk, int ldb, float* C, int ldc, int M,
                         int N, int K, const float* bias, int relu, const float* mask, int accumulate, bool allow_split,
                         int precision, cudaStream_t st, const void* b_split = nullptr, int b_rows = 0, float* rowsum = nullptr) {
  if (precision == B200ASR_PREC_FP32)
    return gemm_simt(A, ak, lda, B, bk, ldb, C, ldc, M, N, K, bias, relu, mask, accumulate, allow_split, st);
  if (precision == B200ASR_PREC_TF32 || precision == B200ASR_PREC_TF32X3)
    return gemm_tc(A, ak, lda, B, bk, ldb, C, ldc, M, N, K, bias, relu, mask, accumulate, precision, st,
                   precision == B200ASR_PREC_TF32X3 ? b_split : nullptr, b_rows, rowsum);
  // weight gradients (both operands MN-major fp32 activations): both tiles are converted to bf16 inside the kernel
  if (precision == B200ASR_PREC_BF16X3 || precision == B200ASR_PREC_BF16) {
    B200_REQUIRE(!ak && !bk, B200ASR_BAD_ARG, "bf16 GEMM without a pre-converted weight operand needs MN-major operands (weight gradient)");
    return gemm_tc(A, ak, lda, B, bk, ldb, C, ldc, M, N, K, bias, relu, mask, accumulate, precision, st, nullptr, 0, rowsum);
  }
  set_error("unknown precision %d", precision);
  return B200ASR_BAD_ARG;
}

extern "C" {

static bool is_bf16_prec(int precision) { return precision == B200ASR_PREC_BF16 || precision == B200ASR_PREC_BF16X3; }

int b200asr_linear_fwd(const float* x, const float* w, const float* bias, float* y, int M, int N, int K, int relu,
                       int precision, const void* w_split, b200asr_stream_t stream) {
  B200_REQUIRE(x && w && y && M >= 0 && N > 0 && K > 0, B200ASR_BAD_ARG, "linear_fwd: bad arguments");
  if (is_bf16_prec(precision)) {
    B200_REQUIRE(w_split && K % 8 == 0, B200ASR_BAD_SHAPE, "linear_fwd (bf16): needs w_split = b200asr_split_bf16(...).dst and K %% 8 == 0 (K=%d)", K);
    return gemm_tc(x, true, K, nullptr, true, K, y, N, M, N, K, bias, relu, nullptr, 0, precision, (cudaStream_t)stream, w_split, N);
  }
  return gemm_dispatch(x, true, K, w, true, K, y, N, M, N, K, bias, relu, nullptr, 0, false, precision,
                       (cudaStream_t)stream, w_split, N);
}

int b200asr_linear_bwd_data(const float* dy, const float* w, const float* relu_out, float* dx, int M, int N, int K,
                            int accumulate, int precision, const void* w_split, b200asr_stream_t stream) {
  B200_REQUIRE(dy && w && dx && M >= 0 && N > 0 && K > 0, B200ASR_BAD_ARG, "linear_bwd_data: bad arguments");
  if (is_bf16_prec(precision)) {
    // dx[m,k] = sum_n dy[m,n] w^T[k,n]: the transposed bf16 copy [terms][K][N8] makes B K-major (contraction n contiguous)
    B200_REQUIRE(w_split && N % 4 == 0, B200ASR_BAD_SHAPE, "linear_bwd_data (bf16): needs w_split = b200asr_split_bf16(...).dst_t and N %% 4 == 0 (N=%d)", N);
    return gemm_tc(dy, true, N, nullptr, true, (N + 7) / 8 * 8, dx, K, M, K, N, nullptr, 0, relu_out, accumulate, precision,
                   (cudaStream_t)stream, w_split, K);
  }
  // dx[m,k] = sum_n dy[m,n] w[n,k]: contraction over n; A = dy (n contiguous), B(n,k) = w[n*K + k] (k contiguous)
  return gemm_dispatch(dy, true, N, w, false, K, dx, K, M, K, N, nullptr, 0, relu_out, accumulate, false, precision,
                       (cudaStream_t)stream, w_split, N);
}

int b200asr_linear_bwd_weight(const float* dy, const float* x, float* dw, float* dbias, int M, int N, int K,
                              int accumulate, int precision, b200asr_stream_t stream) {
  B200_REQUIRE(dy && x && dw && M >= 0 && N > 0 && K > 0, B200ASR_BAD_ARG, "linear_bwd_weight: bad arguments");
  B200_REQUIRE(precision == B200ASR_PREC_FP32 || precision == B200ASR_PREC_TF32 || precision == B200ASR_PREC_TF32X3 ||
               is_bf16_prec(precision), B200ASR_BAD_ARG, "linear_bwd_weight: unknown precision %d", precision);
  cudaStream_t st = (cudaStream_t)stream;
  if (M == 0) {
    // empty batch: the sums over no rows are 0 at every precision (the tensor-core GEMM cannot describe a contraction of
    // length 0 to TMA, so nothing is dispatched)
    if (!accumulate) {
      cudaMemsetAsync(dw, 0, sizeof(float) * (size_t)N * K, st);
      if (dbias) cudaMemsetAsync(dbias, 0, sizeof(float) * (size_t)N, st);
    }
    return B200ASR_OK;
  }
  // dw[n,k] = sum_m dy[m,n] x[m,k]: contraction over m; A(n,m) = dy[m*N + n], B(m,k) = x[m*K + k]
  // db[n] = sum_m dy[m,n] = row sums of A: the 3xTF32 kernel produces them from the tiles it stages (one launch and one
  // HBM pass over dy less); other precisions run the column-sum kernel
  const bool fuse = dbias && precision != B200ASR_PREC_FP32 && gemm_tc_fuses_rowsum(false, false, precision);
  // the fused row sums accumulate into dbias, which is cleared first: reject what gemm_tc rejects before clearing it
  if (fuse)
    B200_REQUIRE(aligned16(dy) && aligned16(x) && N % 4 == 0 && K % 4 == 0, B200ASR_BAD_SHAPE,
                 "linear_bwd_weight: TMA needs 16-byte aligned dy and x, and N=%d and K=%d multiples of 4; use precision 0 for this shape",
                 N, K);
  if (fuse && !accumulate) cudaMemsetAsync(dbias, 0, sizeof(float) * (size_t)N, st);
  int rc = gemm_dispatch(dy, false, N, x, false, K, dw, K, N, K, M, nullptr, 0, nullptr, accumulate, true, precision, st,
                         nullptr, 0, fuse ? dbias : nullptr);
  if (rc) return rc;
  if (dbias && !fuse) return launch_colsum(dy, dbias, M, N, accumulate, st);
  return B200ASR_OK;
}

__global__ void split_tf32_kernel(const float* __restrict__ src, float* __restrict__ dst, long long n) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float x = src[i];
  const float hi = __uint_as_float((__float_as_uint(x) + 0x1000u) & 0xFFFFE000u);
  dst[i] = hi;
  dst[n + i] = x - hi;
}

// w [N,K] fp32 -> bf16 hi (| lo) in both orientations; 32 x 32 tiles through shared memory so that both stores are coalesced
__global__ void __launch_bounds__(256) split_bf16_kernel(const float* __restrict__ w, uint16_t* __restrict__ dst,
                                                         uint16_t* __restrict__ dst_t, int N, int K, int N8, int terms) {
  __shared__ uint16_t th[32][33], tl[32][33];
  const int k0 = blockIdx.x * 32, n0 = blockIdx.y * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  for (int i = ty; i < 32; i += 8) {
    const int n = n0 + i, k = k0 + tx;
    uint16_t h = 0, l = 0;
    if (n < N && k < K) {
      const float x = w[(size_t)n * K + k];
      const uint32_t r = __float_as_uint(x) + 0x8000u;
      h = (uint16_t)(r >> 16);
      const float lo = x - __uint_as_float(r & 0xFFFF0000u);
      l = (uint16_t)((__float_as_uint(lo) + 0x8000u) >> 16);
      if (dst) {
        dst[(size_t)n * K + k] = h;
        if (terms == 2) dst[(size_t)N * K + (size_t)n * K + k] = l;
      }
    }
    th[i][tx] = h; tl[i][tx] = l;
  }
  if (!dst_t) return;
  __syncthreads();
  for (int i = ty; i < 32; i += 8) {
    const int k = k0 + i, n = n0 + tx;
    if (k < K && n < N8) {                       // columns N..N8-1 are written as zeros (their tile entries are 0)
      dst_t[(size_t)k * N8 + n] = th[tx][i];
      if (terms == 2) dst_t[(size_t)K * N8 + (size_t)k * N8 + n] = tl[tx][i];
    }
  }
}

// All weight matrices of a flat parameter buffer in ONE launch: desc[d] = {src offset, N, K, terms, dst offset, dst_t offset}
// (elements; dst / dst_t relative to `out`), tile_prefix[d] = number of 32 x 32 tiles of matrices 0 .. d-1.
__global__ void __launch_bounds__(256) split_bf16_batched_kernel(const float* __restrict__ base, uint16_t* __restrict__ out,
                                                                 const long long* __restrict__ desc, const int* __restrict__ tile_prefix,
                                                                 int ndesc) {
  __shared__ uint16_t th[32][33], tl[32][33];
  int lo = 0, hi = ndesc - 1;                                  // last d with tile_prefix[d] <= blockIdx.x
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (tile_prefix[mid] <= (int)blockIdx.x) lo = mid; else hi = mid - 1;
  }
  const long long* d = desc + 6 * lo;
  const float* w = base + d[0];
  const int N = (int)d[1], K = (int)d[2], terms = (int)d[3];
  uint16_t* dst = out + d[4];
  uint16_t* dst_t = out + d[5];
  const int N8 = (N + 7) / 8 * 8;
  const int local = (int)blockIdx.x - tile_prefix[lo], kt = (K + 31) / 32;
  const int k0 = (local % kt) * 32, n0 = (local / kt) * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  for (int i = ty; i < 32; i += 8) {
    const int n = n0 + i, k = k0 + tx;
    uint16_t h = 0, l = 0;
    if (n < N && k < K) {
      const float x = w[(size_t)n * K + k];
      const uint32_t r = __float_as_uint(x) + 0x8000u;
      h = (uint16_t)(r >> 16);
      const float lo_f = x - __uint_as_float(r & 0xFFFF0000u);
      l = (uint16_t)((__float_as_uint(lo_f) + 0x8000u) >> 16);
      dst[(size_t)n * K + k] = h;
      if (terms == 2) dst[(size_t)N * K + (size_t)n * K + k] = l;
    }
    th[i][tx] = h; tl[i][tx] = l;
  }
  __syncthreads();
  for (int i = ty; i < 32; i += 8) {
    const int k = k0 + i, n = n0 + tx;
    if (k < K && n < N8) {
      dst_t[(size_t)k * N8 + n] = th[tx][i];
      if (terms == 2) dst_t[(size_t)K * N8 + (size_t)k * N8 + n] = tl[tx][i];
    }
  }
}

int b200asr_split_bf16_batched(const float* base, void* out, const long long* desc, const int* tile_prefix, int ndesc,
                               int total_tiles, b200asr_stream_t stream) {
  B200_REQUIRE(base && out && desc && tile_prefix && ndesc > 0 && total_tiles > 0, B200ASR_BAD_ARG, "split_bf16_batched: bad arguments");
  split_bf16_batched_kernel<<<total_tiles, 256, 0, (cudaStream_t)stream>>>(base, (uint16_t*)out, desc, tile_prefix, ndesc);
  return check_launch("split_bf16_batched");
}

int b200asr_split_bf16(const float* w, void* dst, void* dst_t, int N, int K, int terms, b200asr_stream_t stream) {
  B200_REQUIRE(w && (dst || dst_t) && N > 0 && K > 0 && (terms == 1 || terms == 2), B200ASR_BAD_ARG, "split_bf16: bad arguments");
  const int N8 = (N + 7) / 8 * 8;
  dim3 grid(ceil_div(K, 32), ceil_div(N8, 32));
  split_bf16_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(w, (uint16_t*)dst, (uint16_t*)dst_t, N, K, N8, terms);
  return check_launch("split_bf16");
}

int b200asr_split_tf32(const float* src, float* dst_hi_lo, long long n, b200asr_stream_t stream) {
  B200_REQUIRE(src && dst_hi_lo && n >= 0, B200ASR_BAD_ARG, "split_tf32: bad arguments");
  if (n == 0) return B200ASR_OK;
  split_tf32_kernel<<<(unsigned)ceil_div_ll(n, 256), 256, 0, (cudaStream_t)stream>>>(src, dst_hi_lo, n);
  return check_launch("split_tf32");
}

}  // extern "C"
