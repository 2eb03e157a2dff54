// Batched tensor-core GEMM on the persistent engine: C_z[M,N] = alpha * sum_k A_z(m,k) B_z(k,n) for z = (batch, head).
//
// This is the contraction engine of the "materialised" attention path (attention_mat.cu): Q K^T, P V and the four
// backward products are small per-head GEMMs (T x T x d), and at 3xTF32 the tensor cores run them ~10x faster than the
// fp32 CUDA-core flash kernel while keeping fp32-grade products.  Operands are addressed IN PLACE through 4-D tensor maps
// (column, head, row, batch), so the token-major [B,T,H,d] projections and the [B*H,Tq,Tk] probability buffers need no
// repacking; either operand may be K-major or MN-major exactly as in tc_gemm.cu.
#include "../../include/b200asr.h"
#include "common.cuh"
#include "kernels.h"
#include "tc_common.cuh"
#include "tc_engine.cuh"

namespace b200asr {
namespace tc {

template <bool A_MN, bool B_MN, int BN_>
struct BGemmPolicy {
  static constexpr int BN = BN_, kABytes = 128 * 128, kBBytes = BN_ * 128;
  static constexpr bool kSplitA = true, kSplitB = true, kAMN = A_MN, kBMN = B_MN;
  static constexpr bool kSumA = false, kSumB = false;
  struct Params {
    float* C;
    long long c_bs, c_hs;     // element offsets of (batch, head) in C
    int ldc, M, N, Nst, K, H; // Nst: columns that may be stored (N rounded up to the row pitch's float4 granularity)
    int tiles_m, tiles_n, Z;  // Z = B * H
    int a_heads, b_heads;     // operand addressed as (head, batch) = (z % H, z / H) [1] or as (0, z) [0]
    float alpha;
  };
  static __device__ __forceinline__ int num_tiles(const Params& p) { return p.tiles_m * p.tiles_n * p.Z; }
  static __device__ __forceinline__ int num_kb(const Params& p, int) { return (p.K + 31) / 32; }
  struct Tile { int m0, n0, z, k0, ah, ab, bh, bb; };
  static __device__ __forceinline__ Tile tile(const Params& p, int tile) {
    Tile t;
    const int n = tile % p.tiles_n, r = tile / p.tiles_n;
    t.m0 = (r % p.tiles_m) * 128; t.n0 = n * BN; t.z = r / p.tiles_m; t.k0 = 0;
    const int h = t.z % p.H, b = t.z / p.H;
    t.ah = p.a_heads ? h : 0; t.ab = p.a_heads ? b : t.z;
    t.bh = p.b_heads ? h : 0; t.bb = p.b_heads ? b : t.z;
    return t;
  }
  static __device__ __forceinline__ void load(const Params&, Tile& t, const CUtensorMap* mapA, const CUtensorMap* mapB,
                                              uint32_t sa, uint32_t sb, uint32_t, uint32_t bar, bool leader) {
    const int k0 = t.k0;
    t.k0 += 32;
    if (!leader) return;
    if (!A_MN) tma_load_4d(sa, mapA, bar, k0, t.ah, t.m0, t.ab);
    else
#pragma unroll
      for (int c = 0; c < 4; c++) tma_load_4d(sa + c * 4096, mapA, bar, t.m0 + 32 * c, t.ah, k0, t.ab);
    if (!B_MN) tma_load_4d(sb, mapB, bar, k0, t.bh, t.n0, t.bb);
    else
#pragma unroll
      for (int c = 0; c < BN / 32; c++) tma_load_4d(sb + c * 4096, mapB, bar, t.n0 + 32 * c, t.bh, k0, t.bb);
  }
  static __device__ __forceinline__ void store(const Params& p, const Tile& t, int r, int c0, const float (&v)[32]) {
    const int row = t.m0 + r;
    if (row >= p.M) return;
    float* crow = p.C + (long long)(t.z / p.H) * p.c_bs + (long long)(t.z % p.H) * p.c_hs + (long long)row * p.ldc;
#pragma unroll
    for (int j4 = 0; j4 < 8; j4++) {
      const int col = t.n0 + c0 + j4 * 4;
      if (col < p.Nst)
        *reinterpret_cast<float4*>(crow + col) =
            make_float4(v[j4 * 4] * p.alpha, v[j4 * 4 + 1] * p.alpha, v[j4 * 4 + 2] * p.alpha, v[j4 * 4 + 3] * p.alpha);
    }
  }
};

static int make_operand_map(CUtensorMap* map, const BOperand& x, bool kmaj, int mn_box, int Bsz, int H, bool tf32_dtype) {
  B200_REQUIRE(aligned16(x.p) && x.rs % 4 == 0 && x.bs % 4 == 0 && (!x.heads || x.hs % 4 == 0), B200ASR_BAD_ALIGN,
               "bgemm_tc: operand base must be 16-byte aligned and strides multiples of 4 elements");
  uint64_t dims[4] = {(uint64_t)x.cols, (uint64_t)(x.heads ? H : 1), (uint64_t)x.rows, (uint64_t)(x.heads ? Bsz : Bsz * H)};
  uint64_t strides[3] = {(uint64_t)(x.heads ? x.hs : x.rs), (uint64_t)x.rs, (uint64_t)x.bs};
  uint32_t box[4] = {32u, 1u, kmaj ? (uint32_t)mn_box : 32u, 1u};
  return make_tensor_map_f32(map, x.p, 4, dims, strides, box, tf32_dtype);
}

template <bool A_MN, bool B_MN, int BN, int NSPLIT>
static int launch_bgemm(const CUtensorMap& ma, const CUtensorMap& mb, const typename BGemmPolicy<A_MN, B_MN, BN>::Params& p,
                        cudaStream_t st) {
  return launch_engine<BGemmPolicy<A_MN, B_MN, BN>, NSPLIT>(ma, mb, p, p.tiles_m * p.tiles_n * p.Z, st, "tc_bgemm");
}

}  // namespace tc

int bgemm_tc(const BOperand& A, bool a_kmaj, const BOperand& B, bool b_kmaj, float* C, long long c_bs, long long c_hs, int ldc,
             int M, int N, int K, int Bsz, int H, float alpha, int nsplit, cudaStream_t st) {
  using namespace tc;
  if (M <= 0 || N <= 0 || Bsz <= 0 || H <= 0) return B200ASR_OK;
  B200_REQUIRE(nsplit == 1 || nsplit == 3, B200ASR_BAD_ARG, "bgemm_tc: nsplit must be 1 or 3");
  B200_REQUIRE(aligned16(C) && ldc % 4 == 0 && c_bs % 4 == 0 && c_hs % 4 == 0, B200ASR_BAD_ALIGN, "bgemm_tc: output alignment");
  const int nst = min(ldc, (N + 3) & ~3);
  B200_REQUIRE(nst >= N, B200ASR_BAD_SHAPE, "bgemm_tc: ldc=%d < N=%d", ldc, N);
  const int bn = N <= 64 ? 64 : 128;
  CUtensorMap ma, mb;
  int rc = make_operand_map(&ma, A, a_kmaj, 128, Bsz, H, nsplit == 1);
  if (rc) return rc;
  rc = make_operand_map(&mb, B, b_kmaj, bn, Bsz, H, nsplit == 1);
  if (rc) return rc;
  const bool a_mn = !a_kmaj, b_mn = !b_kmaj;
#define GO2(AM, BM_, BNv)                                                                                              \
  do {                                                                                                                 \
    typename BGemmPolicy<AM, BM_, BNv>::Params p{C, c_bs, c_hs, ldc, M, N, nst, K, H, ceil_div(M, 128), ceil_div(N, BNv),  \
                                                  Bsz * H, A.heads, B.heads, alpha};                                    \
    return nsplit == 3 ? launch_bgemm<AM, BM_, BNv, 3>(ma, mb, p, st) : launch_bgemm<AM, BM_, BNv, 1>(ma, mb, p, st);    \
  } while (0)
#define GO(AM, BM_) do { if (bn == 64) GO2(AM, BM_, 64); else GO2(AM, BM_, 128); } while (0)
  if (!a_mn && !b_mn) GO(false, false);
  if (!a_mn && b_mn) GO(false, true);
  if (a_mn && !b_mn) GO(true, false);
  GO(true, true);
#undef GO
#undef GO2
}

}  // namespace b200asr
