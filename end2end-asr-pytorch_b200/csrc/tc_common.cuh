// sm_90a building blocks shared by the tensor-core kernels: mbarrier, TMA (cp.async.bulk.tensor), wgmma (warpgroup MMA with
// the A operand in registers and B described in shared memory), Hopper shared-memory matrix descriptors, operand splits,
// host-side tensor-map encoding.  Bit layouts follow the PTX ISA "asynchronous warpgroup level matrix shared memory layout"
// tables; everything here is written from those tables.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace b200asr {
namespace tc {

// ---------------------------------------------------------------------------------------------- small PTX wrappers
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
// generic-proxy writes to shared memory (threads) made visible to the async proxy (wgmma operand reads, TMA writes)
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
      "selp.u32 %0, 1, 0, p;\n"
      "}\n"
      : "=r"(ok)
      : "r"(bar), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded wait: a protocol bug becomes a trap (CUDA error reported to the caller) instead of a hung GPU.  It prints no
// message on purpose: printf is a function call, and ptxas serializes every wgmma of a kernel that contains a call ANYWHERE
// (C7510, "wgmma pipeline crossing function boundary") -- a message on the producer warp's path alone, where no wgmma is
// ever in flight, is enough to make each MMA of the consumers wait for the previous one.  Every kernel that issues wgmma
// must therefore stay call-free, including its policies' load / store code.  (A call-free record of block, thread and
// barrier, stored into host-mapped memory before the trap, was tried: with it the cfg2 linear weight gradient took 4.93
// instead of 4.52 ms per step on an H100, so the wait stays this small.)
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  while (!mbar_try_wait(bar, parity))
    if (clock64() - t0 > 4000000000LL) __trap();
}
// named barrier over `count` threads (a multiple of 32); id 0 is __syncthreads
__device__ __forceinline__ void named_bar_sync(int id, int count) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory");
}
// arrive on a named barrier without waiting (the threads that wait call named_bar_sync with the same count)
__device__ __forceinline__ void named_bar_arrive(int id, int count) {
  asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(count) : "memory");
}

__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(m) : "memory");
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(dst),
      "l"(map), "r"(bar), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];" ::"r"(dst),
      "l"(map), "r"(bar), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];" ::"r"(dst),
      "l"(map), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}

// one lane of a CONVERGED warp (elect.sync): the issuing warp stays convergent and predicates only the TMA instructions on it
__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile("{\n\t.reg .pred p;\n\telect.sync _|p, 0xffffffff;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(pred));
  return pred != 0;
}

// ---------------------------------------------------------------------------------------------- operand splits
// 3xTF32 operand split: hi <- x rounded to TF32 (nearest, ties away -- the same value cvt.rna.tf32.f32 gives, computed with
// two integer ops on the ALU pipe), lo <- x - hi (exact in fp32, |lo| <= 2^-12 |x|; the tensor core truncates it to TF32,
// an error of <= 2^-22 |x|).
__device__ __forceinline__ float tf32_rn(float x) { return __uint_as_float((__float_as_uint(x) + 0x1000u) & 0xFFFFE000u); }

// 2-term bf16 split ("bf16x3"): x ~ hi + lo with hi = bf16(x), lo = bf16(x - hi) -- 16 significant bits, |x - hi - lo| <=
// 2^-18 |x| -- and hi*hi + hi*lo + lo*hi per product: three bf16 MMAs at TWICE the tf32 rate.  Error per product ~2^-17
// (dropped lo*lo and the representation error), i.e. ~100x below single-pass TF32 and ~30x above 3xTF32.
// pack2(a, b): 32-bit word with bf16(a) in the low half (element k) and bf16(b) in the high half (element k + 1) -- the
// order in which an MMA register fragment holds two consecutive-k elements of a 16-bit operand.
__device__ __forceinline__ uint32_t cvt_bf16x2(float lo_elem, float hi_elem) {     // one F2FP: {hi_elem, lo_elem} -> packed bf16x2 (RN)
  uint32_t d;
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(d) : "f"(hi_elem), "f"(lo_elem));
  return d;
}
__device__ __forceinline__ void split_bf16_pair(float x0, float x1, uint32_t& hi, uint32_t& lo) {
  hi = cvt_bf16x2(x0, x1);
  lo = cvt_bf16x2(x0 - __uint_as_float(hi << 16), x1 - __uint_as_float(hi & 0xFFFF0000u));
}
__device__ __forceinline__ uint32_t pack_bf16_pair(float x0, float x1) {
  return __byte_perm(__float_as_uint(x0) + 0x8000u, __float_as_uint(x1) + 0x8000u, 0x7632);
}

// ---------------------------------------------------------------------------------------------- wgmma
// Every B operand the kernels hand to wgmma is K-major (contraction contiguous) in one of two canonical swizzled layouts:
//   * 128-byte rows (32 fp32 / tf32 k-values), SWIZZLE_128B: 16-byte chunk c of row r stored at chunk c ^ (r & 7), 8-row
//     groups 1024 B apart (SBO = 1024); a k-step of 8 tf32 advances the start address by 32 B;
//   * 64-byte rows (32 bf16 k-values), SWIZZLE_64B: chunk c of row r stored at c ^ ((r >> 1) & 3), 8-row groups 512 B apart
//     (SBO = 512); a k-step of 16 bf16 advances the start address by 32 B.
// Tiles start on 1024-byte boundaries, so the descriptor's base offset is 0; LBO is unused by swizzled K-major layouts.
// The A operand always comes from registers: the kernels read the fp32 tile from shared memory, round or split it, and build
// the fragment (for tf32 k8: a0 = (row g, k q), a1 = (row g + 8, k q), a2 = (g, q + 4), a3 = (g + 8, q + 4) with g = lane / 4,
// q = lane % 4, rows relative to 16 * (warp % 4); for bf16 k16 the pairs (k 2q, 2q + 1) and (k 8 + 2q, 9 + 2q)).
// Accumulator fragment (m64nN, f32): d[4j + {0,1}] = (row g, col 8j + 2q + {0,1}), d[4j + {2,3}] = (row g + 8, same cols).
constexpr uint32_t kLayoutSW128 = 1, kLayoutSW64 = 2;
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t saddr, uint32_t sbo_bytes, uint32_t layout_type) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr & 0x3FFFFu) >> 4);
  d |= (uint64_t)1 << 16;                                    // LBO (unused for swizzled K-major layouts)
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFFu) << 32;
  d |= (uint64_t)layout_type << 62;
  return d;
}
__device__ __forceinline__ uint64_t kmajor_desc_tf32(uint32_t saddr) { return make_smem_desc(saddr, 1024, kLayoutSW128); }
__device__ __forceinline__ uint64_t kmajor_desc_bf16(uint32_t saddr) { return make_smem_desc(saddr, 512, kLayoutSW64); }

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N> __device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// accumulator registers must not be touched by other code between a wgmma and the wait that retires it
template <int N> __device__ __forceinline__ void acc_fence(float (&d)[N]) {
#pragma unroll
  for (int i = 0; i < N; i++) asm volatile("" : "+f"(d[i])::"memory");
}

// register-A fragments of wgmma still in flight: a use here keeps the compiler from reusing their registers before the
// wait that retires those MMAs (call it right after that wait)
__device__ __forceinline__ void keep_live(const uint32_t (&a)[4]) {
  asm volatile("" ::"r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]) : "memory");
}

// D[64 x N] += A[64 x k] (registers) * B[k x N] (shared memory, K-major), fp32 accumulate; k = 8 (tf32) or 16 (bf16).
// The operand lists: N / 2 accumulator registers, the four A registers, the B descriptor, scale-d = scale-a = scale-b = 1
// (and, for bf16, B not transposed).
#define WG_R32 "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, {%16, %17, %18, %19}, %20, 1, 1, 1"
#define WG_R64 "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, {%32, %33, %34, %35}, %36, 1, 1, 1"
#define WG_R128 "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, {%64, %65, %66, %67}, %68, 1, 1, 1"
#define WG_O4(i) "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3])
#define WG_O16(i) WG_O4(i), WG_O4(i + 4), WG_O4(i + 8), WG_O4(i + 12)
#define WG_IN "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc)
#define WG_MMA(N, ...)                                                                                                            \
  if constexpr (BF16) asm volatile("wgmma.mma_async.sync.aligned.m64n" #N "k16.f32.bf16.bf16 " WG_R##N ", 0;" : __VA_ARGS__ : WG_IN); \
  else asm volatile("wgmma.mma_async.sync.aligned.m64n" #N "k8.f32.tf32.tf32 " WG_R##N ";" : __VA_ARGS__ : WG_IN)
template <int N, bool BF16> __device__ __forceinline__ void wgmma_rs(float (&d)[N / 2], const uint32_t (&a)[4], uint64_t bdesc) {
  static_assert(N == 32 || N == 64 || N == 128, "wgmma N");
  if constexpr (N == 32) { WG_MMA(32, WG_O16(0)); }
  else if constexpr (N == 64) { WG_MMA(64, WG_O16(0), WG_O16(16)); }
  else { WG_MMA(128, WG_O16(0), WG_O16(16), WG_O16(32), WG_O16(48)); }
}
template <int N> __device__ __forceinline__ void wgmma_tf32(float (&d)[N / 2], const uint32_t (&a)[4], uint64_t b) { wgmma_rs<N, false>(d, a, b); }
template <int N> __device__ __forceinline__ void wgmma_bf16(float (&d)[N / 2], const uint32_t (&a)[4], uint64_t b) { wgmma_rs<N, true>(d, a, b); }

// ---------------------------------------------------------------------------------------------- host: tensor maps
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn get_encode_tiled();
// fp32 tensor, `rank` dims (innermost first), strides in ELEMENTS for dims 1..rank-1 (dim 0 is contiguous), box[0] = 32
// (128-byte rows, SWIZZLE_128B), out-of-bounds elements read as zero.  tf32_dtype selects CU_TENSOR_MAP_DATA_TYPE_TFLOAT32
// (the copy engine rounds fp32 -> tf32 to nearest in flight) instead of FLOAT32.  Returns 0 on success.
int make_tensor_map_f32(CUtensorMap* map, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_elems,
                        const uint32_t* box, bool tf32_dtype = false);

// bf16 tensor (2 bytes / element), `rank` dims, strides in ELEMENTS; box[0] * 2 bytes = 64 -> SWIZZLE_64B, = 128 -> SWIZZLE_128B.
int make_tensor_map_bf16(CUtensorMap* map, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_elems,
                         const uint32_t* box);

}  // namespace tc
}  // namespace b200asr
