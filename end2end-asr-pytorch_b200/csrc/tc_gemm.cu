// Tensor-core GEMM for sm_90a: C[M,N] = sum_k A(m,k) B(k,n), fp32 in HBM, TF32 / bf16 tensor-core math, fp32 accumulators.
// A policy of the persistent tile engine (tc_engine.cuh):
//
//   * operands arrive by TMA (cp.async.bulk.tensor, 128B swizzle) straight from the fp32 row-major tensors; either operand
//     may be K-major (contraction contiguous) or MN-major (rows contiguous) -- forward, data-gradient and weight-gradient
//     GEMMs all run without a transpose pass in HBM;
//   * 128x128 output tiles, 32-deep k-blocks; tile = (m-tile, n-tile, k-split), n fastest so that the CTAs that run
//     concurrently share the same A rows through L2;
//   * NSPLIT = 1: tf32 once; the tensor maps use the TFLOAT32 data type, so the copy engine rounds fp32 -> tf32
//     to nearest in flight (measured: 4-5x lower error than letting the tensor core truncate the fp32 operands);
//     NSPLIT = 3: "3xTF32" -- hi = rn_tf32(x), lo = x - hi, and lo*hi + hi*lo + hi*hi per k-step, which recovers
//     fp32-grade products (error ~2^-21 relative) at three MMAs per step; weights can arrive pre-split (PRESPLIT);
//   * epilogue: 32-column row pieces (tc_engine.cuh) -> bias / ReLU / ReLU-mask / accumulate -> global;
//     split-K for the skinny weight-gradient shapes (each split writes its partial tile, gemm_splitk_reduce sums them in
//     split order); the weight-gradient instantiation (both operands
//     MN-major) also produces the bias gradient = row sums of its A operand dy^T from the tiles it stages anyway.
#include "../../include/b200asr.h"
#include "common.cuh"
#include "kernels.h"
#include <stdlib.h>

#include "tc_common.cuh"
#include "tc_engine.cuh"

namespace b200asr {
namespace tc {

EncodeTiledFn get_encode_tiled() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = (EncodeTiledFn)p;
  }
  return fn;
}

int make_tensor_map_f32(CUtensorMap* map, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_elems,
                        const uint32_t* box, bool tf32_dtype) {
  EncodeTiledFn enc = get_encode_tiled();
  if (!enc) { set_error("cuTensorMapEncodeTiled is not available from the driver"); return B200ASR_CUDA_ERROR; }
  cuuint64_t gdim[5], gstride[4];
  cuuint32_t bdim[5], estr[5];
  for (int i = 0; i < rank; i++) { gdim[i] = dims[i]; bdim[i] = box[i]; estr[i] = 1; }
  for (int i = 1; i < rank; i++) gstride[i - 1] = strides_elems[i - 1] * sizeof(float);
  // the driver entry point needs the primary context current on THIS thread (autograd runs backward on its own threads,
  // and a thread that has only launched through the runtime so far may not have it bound yet): cudaFree(0) binds it
  static thread_local bool ctx_bound = false;
  if (!ctx_bound) { cudaFree(nullptr); ctx_bound = true; }
  CUresult r = enc(map, tf32_dtype ? CU_TENSOR_MAP_DATA_TYPE_TFLOAT32 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, (cuuint32_t)rank, const_cast<void*>(base), gdim, gstride, bdim, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled failed with CUresult %d", (int)r); return B200ASR_CUDA_ERROR; }
  return B200ASR_OK;
}

int make_tensor_map_bf16(CUtensorMap* map, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_elems,
                         const uint32_t* box) {
  EncodeTiledFn enc = get_encode_tiled();
  if (!enc) { set_error("cuTensorMapEncodeTiled is not available from the driver"); return B200ASR_CUDA_ERROR; }
  cuuint64_t gdim[5], gstride[4];
  cuuint32_t bdim[5], estr[5];
  for (int i = 0; i < rank; i++) { gdim[i] = dims[i]; bdim[i] = box[i]; estr[i] = 1; }
  for (int i = 1; i < rank; i++) gstride[i - 1] = strides_elems[i - 1] * 2;
  static thread_local bool ctx_bound = false;
  if (!ctx_bound) { cudaFree(nullptr); ctx_bound = true; }
  const CUtensorMapSwizzle sw = box[0] * 2 == 64 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_128B;
  CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, (cuuint32_t)rank, const_cast<void*>(base), gdim, gstride, bdim, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, sw, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled (bf16) failed with CUresult %d", (int)r); return B200ASR_CUDA_ERROR; }
  return B200ASR_OK;
}

constexpr int GBM = 128, GBN = 128, GBK = 32;            // tile; k-block in fp32 elements (= 128 bytes)
constexpr int TILE_BYTES = GBM * GBK * 4;                // 16 KB per operand per stage

struct EpiP {
  float* C;
  int ldc, M, N, K;
  const float* bias;
  const float* relu_mask;
  int relu, accumulate, splits, klen;
  float* rowsum;           // [M] += sum_k A(m,k) (bias gradient of the weight-gradient GEMM), or nullptr
  float* part;             // splits > 1: partial tiles [splits][M][N] (scratch), summed by gemm_splitk_reduce
  float* rowpart;          // splits > 1 with rowsum: partial row sums [splits][M]
};

// ---------------------------------------------------------------------------------------------------------------------
// GEMM policy for the persistent engine (tc_engine.cuh): tile = (m-tile, n-tile, k-split), n fastest so that the CTAs that
// run concurrently share the same A rows through L2.
template <bool A_MN, bool B_MN, bool PRESPLIT = false>
struct GemmPolicy {
  static constexpr int BN = GBN, kABytes = TILE_BYTES, kBBytes = TILE_BYTES;
  static constexpr bool kSplitA = true, kSplitB = !PRESPLIT, kAMN = A_MN, kBMN = B_MN;
  static constexpr bool kSumA = A_MN && B_MN && !PRESPLIT, kSumB = false;
  struct Params { EpiP e; int tiles_m, tiles_n, b_rows; };
  static __device__ __forceinline__ int num_tiles(const Params& p) { return p.tiles_m * p.tiles_n * p.e.splits; }
  struct Tile { int m0, n0, z, k0; };                    // tile origin, split-K slice, k cursor
  static __device__ __forceinline__ Tile tile(const Params& p, int tile) {
    Tile t;
    const int n = tile % p.tiles_n, r = tile / p.tiles_n;
    t.m0 = (r % p.tiles_m) * GBM; t.n0 = n * GBN; t.z = r / p.tiles_m;
    t.k0 = t.z * p.e.klen;
    return t;
  }
  static __device__ __forceinline__ int num_kb(const Params& p, int tile) {
    const int z = tile / (p.tiles_n * p.tiles_m);
    const int kbeg = z * p.e.klen, kend = min(p.e.K, kbeg + p.e.klen);
    return (kend - kbeg + GBK - 1) / GBK;
  }
  static __device__ __forceinline__ void load(const Params& p, Tile& t, const CUtensorMap* mapA, const CUtensorMap* mapB,
                                              uint32_t sa, uint32_t sb, uint32_t sb_lo, uint32_t bar, bool leader) {
    const int k0 = t.k0, m0 = t.m0, n0 = t.n0;
    t.k0 += GBK;
    if (!leader) return;
    if (!A_MN) tma_load_2d(sa, mapA, bar, k0, m0);
    else
#pragma unroll
      for (int c = 0; c < 4; c++) tma_load_2d(sa + c * 4096, mapA, bar, m0 + 32 * c, k0);
    // pre-split B: the lo half is the second [b_rows x ld] matrix of the same buffer -> same map, row offset b_rows
#pragma unroll
    for (int half = 0; half < (PRESPLIT ? 2 : 1); half++) {
      const uint32_t dst = half ? sb_lo : sb;
      const int roff = half ? p.b_rows : 0;
      if (!B_MN) tma_load_2d(dst, mapB, bar, k0, n0 + roff);
      else
#pragma unroll
        for (int c = 0; c < 4; c++) tma_load_2d(dst + c * 4096, mapB, bar, n0 + 32 * c, k0 + roff);
    }
  }
  // bf16 modes (engine NSPLIT 2 / 6): fp32 K-major A tile + pre-converted K-major bf16 B tile(s), 64-byte rows (SWIZZLE_64B)
  static __device__ __forceinline__ void load16(const Params& p, Tile& t, const CUtensorMap* mapA, const CUtensorMap* mapB,
                                                uint32_t sa, uint32_t sb, uint32_t sb_lo, uint32_t bar, bool leader, int halves) {
    const int k0 = t.k0, m0 = t.m0, n0 = t.n0;
    t.k0 += GBK;
    if (!leader) return;
    tma_load_2d(sa, mapA, bar, k0, m0);
    tma_load_2d(sb, mapB, bar, k0, n0);
    if (halves == 2) tma_load_2d(sb_lo, mapB, bar, k0, n0 + p.b_rows);
  }
  // every (row, k) of A is staged once by the n-tile-0 tiles (over all k-splits)
  static __device__ __forceinline__ bool want_sums(const Params& p, const Tile& t) { return p.e.rowsum != nullptr && t.n0 == 0; }
  static __device__ __forceinline__ void sum_a_store(const Params& p, const Tile& t, int r, float v) {
    if (t.m0 + r >= p.e.M) return;
    if (p.e.splits > 1) p.e.rowpart[(size_t)t.z * p.e.M + t.m0 + r] = v;
    else p.e.rowsum[t.m0 + r] += v;                      // one tile per row when K is not split
  }
  // Coalesced epilogue (tc_engine.cuh: epilogue_vec4) for the launches whose store takes the fast path below; the same
  // arithmetic per element (bias 0, mask 1, old C 0 where absent), so the results are those of store.
  static constexpr bool kStoreVec4 = true;
  struct Epi4 { float4 b, m, c; };
  static __device__ __forceinline__ bool vec4_ok(const Params& p) {
    const EpiP& e = p.e;
    if ((e.N & 3) != 0) return false;
    if (e.splits > 1) return true;
    return (e.ldc & 3) == 0 && (reinterpret_cast<uintptr_t>(e.C) & 15) == 0 && (reinterpret_cast<uintptr_t>(e.bias) & 15) == 0 &&
           (reinterpret_cast<uintptr_t>(e.relu_mask) & 15) == 0;
  }
  static __device__ __forceinline__ Epi4 load4(const Params& p, const Tile& t, int r, int c) {
    const EpiP& e = p.e;
    Epi4 x{make_float4(0.f, 0.f, 0.f, 0.f), make_float4(1.f, 1.f, 1.f, 1.f), make_float4(0.f, 0.f, 0.f, 0.f)};
    const int row = t.m0 + r, col = t.n0 + c;
    if (e.splits > 1 || row >= e.M || col >= e.N) return x;
    if (e.bias) x.b = __ldg(reinterpret_cast<const float4*>(e.bias + col));
    if (e.relu_mask) x.m = __ldg(reinterpret_cast<const float4*>(e.relu_mask + (size_t)row * e.ldc + col));
    if (e.accumulate) x.c = *reinterpret_cast<const float4*>(e.C + (size_t)row * e.ldc + col);
    return x;
  }
  static __device__ __forceinline__ void store4(const Params& p, const Tile& t, int r, int c, float4 v, const Epi4& x) {
    const EpiP& e = p.e;
    const int row = t.m0 + r, col = t.n0 + c;
    if (row >= e.M || col >= e.N) return;
    if (e.splits > 1) {                                   // this split's partial tile
      *reinterpret_cast<float4*>(e.part + ((size_t)t.z * e.M + row) * e.N + col) = v;
      return;
    }
    float o[4] = {v.x + x.b.x, v.y + x.b.y, v.z + x.b.z, v.w + x.b.w};
    if (e.relu) { o[0] = fmaxf(o[0], 0.f); o[1] = fmaxf(o[1], 0.f); o[2] = fmaxf(o[2], 0.f); o[3] = fmaxf(o[3], 0.f); }
    o[0] = x.m.x > 0.f ? o[0] : 0.f; o[1] = x.m.y > 0.f ? o[1] : 0.f;
    o[2] = x.m.z > 0.f ? o[2] : 0.f; o[3] = x.m.w > 0.f ? o[3] : 0.f;
    *reinterpret_cast<float4*>(e.C + (size_t)row * e.ldc + col) = make_float4(o[0] + x.c.x, o[1] + x.c.y, o[2] + x.c.z, o[3] + x.c.w);
  }
  static __device__ __forceinline__ void store(const Params& p, const Tile& t, int r, int c0, const float (&v)[32]) {
    const EpiP& e = p.e;
    const int m0 = t.m0, n0 = t.n0, z = t.z;
    const int row = m0 + r;
    if (row >= e.M) return;
    const int col0 = n0 + c0;
    float* crow = e.C + (size_t)row * e.ldc;
    const float* mrow = e.relu_mask ? e.relu_mask + (size_t)row * e.ldc : nullptr;
    if (e.splits > 1) {                                   // this split's partial tile
      float* prow = e.part + ((size_t)z * e.M + row) * e.N;
      if ((e.N & 3) == 0 && col0 + 32 <= e.N) {
#pragma unroll
        for (int j = 0; j < 32; j += 4) *reinterpret_cast<float4*>(prow + col0 + j) = make_float4(v[j], v[j + 1], v[j + 2], v[j + 3]);
        return;
      }
#pragma unroll
      for (int j = 0; j < 32; j++)
        if (col0 + j < e.N) prow[col0 + j] = v[j];
      return;
    }
    const bool vec_ok = ((e.ldc & 3) == 0) && ((reinterpret_cast<uintptr_t>(e.C) & 15) == 0);
    if (vec_ok && (e.N & 3) == 0 && (reinterpret_cast<uintptr_t>(e.bias) & 15) == 0 && (reinterpret_cast<uintptr_t>(e.relu_mask) & 15) == 0) {
      // Fast path: ALL the global loads of a 16-column half (bias, ReLU mask, old C) are issued before the first store, so
      // the one epilogue warp of this SM sub-partition pays the load latency twice per chunk instead of once per float4
      // (loads cannot be hoisted above stores through possibly-aliasing pointers; with K = 512 the interleaved version
      // made the epilogue, ~20k clk per 128x128 tile, longer than the 12k clk mainloop).
#pragma unroll
      for (int half = 0; half < 2; half++) {
        float4 bb[4], mm[4], cc[4];
#pragma unroll
        for (int q = 0; q < 4; q++) {
          const int col = col0 + half * 16 + q * 4;
          const bool ok = col < e.N;
          bb[q] = (e.bias && ok) ? __ldg(reinterpret_cast<const float4*>(e.bias + col)) : make_float4(0.f, 0.f, 0.f, 0.f);
          mm[q] = (mrow && ok) ? __ldg(reinterpret_cast<const float4*>(mrow + col)) : make_float4(1.f, 1.f, 1.f, 1.f);
          cc[q] = (e.accumulate && ok) ? *reinterpret_cast<const float4*>(crow + col) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
#pragma unroll
        for (int q = 0; q < 4; q++) {
          const int col = col0 + half * 16 + q * 4;
          if (col >= e.N) break;
          const int j = half * 16 + q * 4;
          float o[4] = {v[j] + bb[q].x, v[j + 1] + bb[q].y, v[j + 2] + bb[q].z, v[j + 3] + bb[q].w};
          if (e.relu) { o[0] = fmaxf(o[0], 0.f); o[1] = fmaxf(o[1], 0.f); o[2] = fmaxf(o[2], 0.f); o[3] = fmaxf(o[3], 0.f); }
          o[0] = mm[q].x > 0.f ? o[0] : 0.f; o[1] = mm[q].y > 0.f ? o[1] : 0.f;
          o[2] = mm[q].z > 0.f ? o[2] : 0.f; o[3] = mm[q].w > 0.f ? o[3] : 0.f;
          *reinterpret_cast<float4*>(crow + col) = make_float4(o[0] + cc[q].x, o[1] + cc[q].y, o[2] + cc[q].z, o[3] + cc[q].w);
        }
      }
      return;
    }
#pragma unroll
    for (int j4 = 0; j4 < 8; j4++) {
      const int col = col0 + j4 * 4;
      if (col >= e.N) break;
      float o[4] = {v[j4 * 4 + 0], v[j4 * 4 + 1], v[j4 * 4 + 2], v[j4 * 4 + 3]};
#pragma unroll
      for (int j = 0; j < 4; j++) {
        if (col + j < e.N) {
          if (e.bias) o[j] += e.bias[col + j];
          if (e.relu) o[j] = fmaxf(o[j], 0.f);
          if (mrow) o[j] = mrow[col + j] > 0.f ? o[j] : 0.f;
          if (e.accumulate) o[j] += crow[col + j];
        }
      }
      if (vec_ok && col + 3 < e.N) *reinterpret_cast<float4*>(crow + col) = make_float4(o[0], o[1], o[2], o[3]);
      else
#pragma unroll
        for (int j = 0; j < 4; j++)
          if (col + j < e.N) crow[col + j] = o[j];
    }
  }
};

// C = (accumulate ? C : 0) + bias + sum of the split partials in split order (split-K never carries ReLU or a mask)
__global__ void gemm_splitk_reduce_kernel(const float* __restrict__ part, int splits, int M, int N, float* __restrict__ C, int ldc,
                                          const float* __restrict__ bias, int accumulate) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)M * N) return;
  const int row = (int)(i / N), col = (int)(i - (long long)row * N);
  float s = 0.f;
  for (int z = 0; z < splits; z++) s += part[(size_t)z * M * N + i];
  float* c = C + (size_t)row * ldc + col;
  *c = (accumulate ? *c : 0.f) + (bias ? bias[col] : 0.f) + s;
}

template <bool A_MN, bool B_MN, int NSPLIT, bool PRESPLIT = false>
static int launch_persistent(const CUtensorMap& ma, const CUtensorMap& mb, const EpiP& e, cudaStream_t st, int b_rows = 0) {
  using Pol = GemmPolicy<A_MN, B_MN, PRESPLIT>;
  typename Pol::Params p{e, ceil_div(e.M, GBM), ceil_div(e.N, GBN), b_rows};
  return launch_engine<Pol, NSPLIT>(ma, mb, p, p.tiles_m * p.tiles_n * e.splits, st, "tc_gemm");
}

}  // namespace tc

static int launch_gemm(const CUtensorMap& ma, const CUtensorMap& mb, const tc::EpiP& e, cudaStream_t st, bool a_kmaj,
                       bool b_kmaj, int nsplit);

bool gemm_tc_fuses_rowsum(bool a_kmaj, bool b_kmaj, int nsplit) { return !a_kmaj && !b_kmaj && (nsplit == 3 || nsplit == 6 || nsplit == 2); }

int gemm_tc(const float* A, bool a_kmaj, int lda, const float* B, bool b_kmaj, int ldb, float* C, int ldc, int M, int N,
            int K, const float* bias, int relu, const float* relu_mask, int accumulate, int nsplit, cudaStream_t st,
            const void* b_split, int b_rows, float* rowsum) {
  using namespace tc;
  if (M <= 0 || N <= 0) return B200ASR_OK;
  if (eng_is_bf16(nsplit) && !(!a_kmaj && !b_kmaj)) {
    // bf16 modes: fp32 K-major A converted in the kernel, pre-converted K-major bf16 B
    B200_REQUIRE(a_kmaj && b_split && b_rows >= N, B200ASR_BAD_ARG, "gemm_tc (bf16): needs a K-major A and the bf16 operand from b200asr_split_bf16");
    B200_REQUIRE(aligned16(A) && aligned16(b_split) && lda % 4 == 0 && ldb % 8 == 0, B200ASR_BAD_SHAPE,
                 "gemm_tc (bf16): TMA needs 16-byte row pitches (lda=%d must be a multiple of 4, ldb=%d of 8)", lda, ldb);
    B200_REQUIRE(!rowsum, B200ASR_BAD_ARG, "gemm_tc (bf16): no fused row sums");
    CUtensorMap ma, mb;
    {
      uint64_t dims[2] = {(uint64_t)K, (uint64_t)M}, strides[1] = {(uint64_t)lda};
      uint32_t box[2] = {GBK, GBM};
      if (int rc = make_tensor_map_f32(&ma, A, 2, dims, strides, box, false)) return rc;
    }
    {
      uint64_t dims[2] = {(uint64_t)K, (uint64_t)(nsplit == 6 ? 2 : 1) * b_rows}, strides[1] = {(uint64_t)ldb};
      uint32_t box[2] = {GBK, GBN};
      if (int rc = make_tensor_map_bf16(&mb, b_split, 2, dims, strides, box)) return rc;
    }
    EpiP e{C, ldc, M, N, K, bias, relu_mask, relu, accumulate, 1, ceil_div(K, GBK) * GBK, nullptr};
    if (nsplit == 6) return launch_persistent<false, false, 6, true>(ma, mb, e, st, b_rows);
    return launch_persistent<false, false, 2, true>(ma, mb, e, st, b_rows);
  }
  const bool presplit = b_split != nullptr && nsplit == 3 && a_kmaj;   // fwd (B K-major) and dgrad (B MN-major)
  if (presplit) B = (const float*)b_split;
  // (bf16 modes with both operands MN-major -- weight gradients -- take the fp32 maps below: both tiles are converted in the kernel)
  B200_REQUIRE(nsplit == 1 || nsplit == 3 || nsplit == 2 || nsplit == 6, B200ASR_BAD_ARG, "gemm_tc: nsplit must be 1, 3 (tf32) or 2, 6 (bf16)");
  B200_REQUIRE(aligned16(A) && aligned16(B) && lda % 4 == 0 && ldb % 4 == 0, B200ASR_BAD_SHAPE,
               "gemm_tc: TMA needs 16-byte aligned operands and leading dimensions that are multiples of 4 (lda=%d ldb=%d); "
               "use precision 0 for this shape", lda, ldb);
  CUtensorMap ma, mb;
  int rc;
  {
    uint64_t dims[2], strides[1] = {(uint64_t)lda};
    uint32_t box[2];
    if (a_kmaj) { dims[0] = (uint64_t)K; dims[1] = (uint64_t)M; box[0] = GBK; box[1] = GBM; }
    else        { dims[0] = (uint64_t)M; dims[1] = (uint64_t)K; box[0] = 32;  box[1] = GBK; }
    rc = make_tensor_map_f32(&ma, A, 2, dims, strides, box, nsplit == 1);
    if (rc) return rc;
  }
  {
    uint64_t dims[2], strides[1] = {(uint64_t)ldb};
    uint32_t box[2];
    // pre-split B = [hi | lo] stacked along the row axis of the weight matrix (b_rows rows each)
    if (b_kmaj) { dims[0] = (uint64_t)K; dims[1] = (uint64_t)(presplit ? 2 * b_rows : N); box[0] = GBK; box[1] = GBN; }
    else        { dims[0] = (uint64_t)N; dims[1] = (uint64_t)(presplit ? 2 * b_rows : K); box[0] = 32;  box[1] = GBK; }
    rc = make_tensor_map_f32(&mb, B, 2, dims, strides, box, nsplit == 1);
    if (rc) return rc;
  }
  B200_REQUIRE(!rowsum || gemm_tc_fuses_rowsum(a_kmaj, b_kmaj, nsplit), B200ASR_BAD_ARG, "gemm_tc: row sums are fused only into the MN/MN 3xTF32 kernel");
  EpiP e{C, ldc, M, N, K, bias, relu_mask, relu, accumulate, 1, ceil_div(K, GBK) * GBK, rowsum};
  const int tiles = ceil_div(M, GBM) * ceil_div(N, GBN);
  if (!relu && !relu_mask && K >= 1024 && tiles * 2 <= device_sm_count()) {
    // Split-K only for skinny outputs (weight gradients: few tiles, long contraction).  A general "split against wave
    // quantisation" rule does not pay: writing and re-reading the partial tiles costs more than the idle SMs of the last
    // round.
    const int sms = device_sm_count();
    int splits = min(min(sms / tiles, K / 256), 16);
    if (splits > 1) {
      e.klen = ceil_div(ceil_div(K, splits), GBK) * GBK;
      e.splits = ceil_div(K, e.klen);
    }
  }
  if (e.splits > 1) {
    const size_t n = (size_t)e.splits * M * N + (rowsum ? (size_t)e.splits * M : 0);
    e.part = (float*)stream_scratch(sizeof(float) * n, st);
    if (!e.part) return B200ASR_CUDA_ERROR;
    e.rowpart = rowsum ? e.part + (size_t)e.splits * M * N : nullptr;
    rc = presplit ? (b_kmaj ? launch_persistent<false, false, 3, true>(ma, mb, e, st, b_rows)
                            : launch_persistent<false, true, 3, true>(ma, mb, e, st, b_rows))
                  : launch_gemm(ma, mb, e, st, a_kmaj, b_kmaj, nsplit);
    if (rc) return rc;
    gemm_splitk_reduce_kernel<<<(unsigned)ceil_div_ll((long long)M * N, 256), 256, 0, st>>>(e.part, e.splits, M, N, C, ldc, bias, accumulate);
    if ((rc = check_launch("gemm_splitk_reduce"))) return rc;
    return rowsum ? reduce_parts(e.rowpart, e.splits, M, M, rowsum, 1, st) : B200ASR_OK;
  }
  if (presplit) return b_kmaj ? launch_persistent<false, false, 3, true>(ma, mb, e, st, b_rows)
                              : launch_persistent<false, true, 3, true>(ma, mb, e, st, b_rows);
  return launch_gemm(ma, mb, e, st, a_kmaj, b_kmaj, nsplit);
}

// the non-presplit fp32-map instantiations, by operand majors and arithmetic
static int launch_gemm(const CUtensorMap& ma, const CUtensorMap& mb, const tc::EpiP& e, cudaStream_t st, bool a_kmaj,
                       bool b_kmaj, int nsplit) {
  using namespace tc;
#define GO(AM, BM_, NS) return launch_persistent<AM, BM_, NS>(ma, mb, e, st)
  const bool a_mn = !a_kmaj, b_mn = !b_kmaj;
  if (nsplit == 6) GO(true, true, 6);
  if (nsplit == 2) GO(true, true, 2);
  if (nsplit == 1) {
    if (!a_mn && !b_mn) GO(false, false, 1);
    if (!a_mn && b_mn) GO(false, true, 1);
    if (a_mn && !b_mn) GO(true, false, 1);
    GO(true, true, 1);
  } else {
    if (!a_mn && !b_mn) GO(false, false, 3);
    if (!a_mn && b_mn) GO(false, true, 3);
    if (a_mn && !b_mn) GO(true, false, 3);
    GO(true, true, 3);
  }
#undef GO
}

}  // namespace b200asr
