// fp32 CUDA-core GEMM (precision 0): 128x128x16 tiles, 8x8 register micro-tiles, double-buffered smem,
// 128-bit coalesced global loads on whichever axis is contiguous.  C[m,n] = sum_k A(m,k) * B(k,n).
// This is the exact-fp32 path and the on-device cross-check for the tensor-core kernels.
#include "../../include/b200asr.h"
#include "common.cuh"
#include "kernels.h"

namespace b200asr {

constexpr int BM = 128, BN = 128, BK = 16, LDS = 132;

struct GemmP {
  const float* A; const float* B; float* C;
  int M, N, K, lda, ldb, ldc;
  const float* bias;       // [N] or nullptr
  const float* relu_mask;  // same indexing as C, or nullptr
  int relu, accumulate, klen, splits;
};

// Operand tile loader.  KMAJ: element (r, k) at P[r*ld + k]; otherwise at P[k*ld + r].
template <bool KMAJ, bool VEC>
struct TileLoader {
  float4 v[VEC ? 2 : 1];
  float s[VEC ? 1 : 8];
  __device__ __forceinline__ void load(const float* __restrict__ P, int ld, int R, int r0, int k0, int kend, int tid) {
    if (VEC) {
#pragma unroll
      for (int i = 0; i < 2; i++) {
        int idx = tid + i * 256;
        float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
        if (KMAJ) {
          int row = idx >> 2, kq = (idx & 3) * 4;
          if (r0 + row < R && k0 + kq < kend) z = *reinterpret_cast<const float4*>(P + (size_t)(r0 + row) * ld + k0 + kq);
        } else {
          int kk = idx >> 5, rq = (idx & 31) * 4;
          if (k0 + kk < kend && r0 + rq < R) z = *reinterpret_cast<const float4*>(P + (size_t)(k0 + kk) * ld + r0 + rq);
        }
        v[i] = z;
      }
    } else {
#pragma unroll
      for (int i = 0; i < 8; i++) {
        int idx = tid + i * 256;
        float z = 0.f;
        if (KMAJ) {
          int row = idx >> 4, kk = idx & 15;
          if (r0 + row < R && k0 + kk < kend) z = P[(size_t)(r0 + row) * ld + k0 + kk];
        } else {
          int kk = idx >> 7, rr = idx & 127;
          if (k0 + kk < kend && r0 + rr < R) z = P[(size_t)(k0 + kk) * ld + r0 + rr];
        }
        s[i] = z;
      }
    }
  }
  __device__ __forceinline__ void store(float (*S)[LDS], int tid) const {
    if (VEC) {
#pragma unroll
      for (int i = 0; i < 2; i++) {
        int idx = tid + i * 256;
        if (KMAJ) {
          int row = idx >> 2, kq = (idx & 3) * 4;
          S[kq + 0][row] = v[i].x; S[kq + 1][row] = v[i].y; S[kq + 2][row] = v[i].z; S[kq + 3][row] = v[i].w;
        } else {
          int kk = idx >> 5, rq = (idx & 31) * 4;
          *reinterpret_cast<float4*>(&S[kk][rq]) = v[i];
        }
      }
    } else {
#pragma unroll
      for (int i = 0; i < 8; i++) {
        int idx = tid + i * 256;
        if (KMAJ) { S[idx & 15][idx >> 4] = s[i]; } else { S[idx >> 7][idx & 127] = s[i]; }
      }
    }
  }
};

template <bool AK, bool BKM, bool VEC>
__global__ void __launch_bounds__(256) gemm_simt_kernel(GemmP p) {
  __shared__ __align__(16) float As[2][BK][LDS];
  __shared__ __align__(16) float Bs[2][BK][LDS];
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int m0 = blockIdx.y * BM, n0 = blockIdx.x * BN;
  const int kbeg = blockIdx.z * p.klen;
  const int kend = min(p.K, kbeg + p.klen);
  const int nk = (kend - kbeg + BK - 1) / BK;

  float acc[8][8];
#pragma unroll
  for (int i = 0; i < 8; i++)
#pragma unroll
    for (int j = 0; j < 8; j++) acc[i][j] = 0.f;

  TileLoader<AK, VEC> la;
  TileLoader<BKM, VEC> lb;
  if (nk > 0) {
    la.load(p.A, p.lda, p.M, m0, kbeg, kend, tid);
    lb.load(p.B, p.ldb, p.N, n0, kbeg, kend, tid);
    la.store(As[0], tid);
    lb.store(Bs[0], tid);
  }
  __syncthreads();
  for (int kt = 0; kt < nk; kt++) {
    const int cur = kt & 1;
    if (kt + 1 < nk) {
      la.load(p.A, p.lda, p.M, m0, kbeg + (kt + 1) * BK, kend, tid);
      lb.load(p.B, p.ldb, p.N, n0, kbeg + (kt + 1) * BK, kend, tid);
    }
#pragma unroll
    for (int k = 0; k < BK; k++) {
      float4 a0 = *reinterpret_cast<const float4*>(&As[cur][k][ty * 4]);
      float4 a1 = *reinterpret_cast<const float4*>(&As[cur][k][64 + ty * 4]);
      float4 b0 = *reinterpret_cast<const float4*>(&Bs[cur][k][tx * 4]);
      float4 b1 = *reinterpret_cast<const float4*>(&Bs[cur][k][64 + tx * 4]);
      float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
      float b[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
      for (int i = 0; i < 8; i++)
#pragma unroll
        for (int j = 0; j < 8; j++) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    if (kt + 1 < nk) {
      la.store(As[cur ^ 1], tid);
      lb.store(Bs[cur ^ 1], tid);
    }
    __syncthreads();
  }

  const bool first_split = (blockIdx.z == 0);
  const bool atomic = p.splits > 1;
#pragma unroll
  for (int i = 0; i < 8; i++) {
    int row = m0 + (i < 4 ? ty * 4 + i : 64 + ty * 4 + (i - 4));
    if (row >= p.M) continue;
#pragma unroll
    for (int j = 0; j < 8; j++) {
      int col = n0 + (j < 4 ? tx * 4 + j : 64 + tx * 4 + (j - 4));
      if (col >= p.N) continue;
      float v = acc[i][j];
      size_t off = (size_t)row * p.ldc + col;
      if (atomic) {
        if (p.bias && first_split) v += p.bias[col];
        atomicAdd(p.C + off, v);   // relu / mask are never combined with split-K (enforced by the host)
      } else {
        if (p.bias) v += p.bias[col];
        if (p.relu) v = fmaxf(v, 0.f);
        if (p.relu_mask) v = (p.relu_mask[off] > 0.f) ? v : 0.f;
        if (p.accumulate) v += p.C[off];
        p.C[off] = v;
      }
    }
  }
}

// column sums: part[row slice][n] = sum over the slice's rows of X[m, n] (reduce_parts adds the slices in order)
__global__ void colsum_kernel(const float* __restrict__ X, float* __restrict__ part, int M, int N, int rows_per_cta) {
  __shared__ float red[8][33];
  int c = blockIdx.x * 32 + (threadIdx.x & 31);
  int rl = threadIdx.x >> 5;
  int r0 = blockIdx.y * rows_per_cta, r1 = min(M, r0 + rows_per_cta);
  float s = 0.f;
  if (c < N)
    for (int r = r0 + rl; r < r1; r += 8) s += X[(size_t)r * N + c];
  red[rl][threadIdx.x & 31] = s;
  __syncthreads();
  if (rl == 0 && c < N) {
    float t = 0.f;
#pragma unroll
    for (int i = 0; i < 8; i++) t += red[i][threadIdx.x & 31];
    part[(size_t)blockIdx.y * N + c] = t;
  }
}

int launch_colsum(const float* X, float* out, int M, int N, int accumulate, cudaStream_t st) {
  if (M <= 0) {
    if (!accumulate) cudaMemsetAsync(out, 0, sizeof(float) * (size_t)N, st);
    return B200ASR_OK;
  }
  // enough CTAs to hide the load latency of a skinny reduction; one partial row per slice of rows
  int rows_per_cta = M >= (1 << 20) ? 2048 : 128;
  dim3 grid(ceil_div(N, 32), ceil_div(M, rows_per_cta));
  float* part = (float*)stream_scratch(sizeof(float) * (size_t)grid.y * N, st);
  if (!part) return B200ASR_CUDA_ERROR;
  colsum_kernel<<<grid, 256, 0, st>>>(X, part, M, N, rows_per_cta);
  int rc = check_launch("colsum");
  return rc ? rc : reduce_parts(part, (int)grid.y, N, N, out, accumulate, st);
}

// Generic entry: C[M,N] = A(m,k) B(k,n) with per-operand major flags.
int gemm_simt(const float* A, bool a_kmaj, int lda, const float* B, bool b_kmaj, int ldb, float* C, int ldc, int M,
              int N, int K, const float* bias, int relu, const float* relu_mask, int accumulate, bool allow_split,
              cudaStream_t st) {
  if (M <= 0 || N <= 0) return B200ASR_OK;
  GemmP p{A, B, C, M, N, K, lda, ldb, ldc, bias, relu_mask, relu, accumulate, K, 1};
  int tiles = ceil_div(M, BM) * ceil_div(N, BN);
  int splits = 1;
  if (allow_split && !relu && !relu_mask && K >= 1024) {
    int sms = device_sm_count();
    if (tiles < sms) {
      splits = min(min(ceil_div(2 * sms, tiles), K / 256), 32);
      if (splits < 1) splits = 1;
    }
  }
  if (splits > 1) {
    int klen = ceil_div(ceil_div(K, splits), BK) * BK;
    splits = ceil_div(K, klen);
    p.klen = klen;
    p.splits = splits;
    if (splits > 1 && !accumulate) cudaMemsetAsync(C, 0, sizeof(float) * (size_t)M * ldc, st);  // ldc == N for all callers that split
  }
  bool vec = aligned16(A) && aligned16(B) && (lda % 4 == 0) && (ldb % 4 == 0) &&
             (a_kmaj ? (K % 4 == 0) : (M % 4 == 0)) && (b_kmaj ? (K % 4 == 0) : (N % 4 == 0)) && (p.klen % 4 == 0);
  dim3 grid(ceil_div(N, BN), ceil_div(M, BM), p.splits);
#define LAUNCH(AKv, BKv, Vv) gemm_simt_kernel<AKv, BKv, Vv><<<grid, 256, 0, st>>>(p)
  if (vec) {
    if (a_kmaj && b_kmaj) LAUNCH(true, true, true);
    else if (a_kmaj && !b_kmaj) LAUNCH(true, false, true);
    else if (!a_kmaj && b_kmaj) LAUNCH(false, true, true);
    else LAUNCH(false, false, true);
  } else {
    if (a_kmaj && b_kmaj) LAUNCH(true, true, false);
    else if (a_kmaj && !b_kmaj) LAUNCH(true, false, false);
    else if (!a_kmaj && b_kmaj) LAUNCH(false, true, false);
    else LAUNCH(false, false, false);
  }
#undef LAUNCH
  return check_launch("gemm_simt");
}

}  // namespace b200asr
