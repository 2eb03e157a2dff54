// Persistent wgmma tile engine shared by the GEMM and the implicit-GEMM convolutions (sm_90a).
//
// One CTA per SM loops over 128 x BN output tiles (static round-robin).  Roles (384 threads):
//   warp 0               TMA producer -- runs ahead across tiles through a ring of shared-memory stages
//   warps 1-3            B converters for B_T16_FROM32 without column sums (EngineCfg::kBByProducer): per stage they
//                        transpose the fp32 B tile into bf16 hi | lo and arrive on the stage's "ready" mbarrier; otherwise
//                        idle (they complete the producer warpgroup, so that the consumers are whole warpgroups)
//   warpgroups 1 and 2   consumers, rows 0-63 and 64-127 of the tile.  Per k-block (32 deep) they
//                          * read their rows of the raw fp32 A tile from the stage and round / split them into wgmma
//                            register fragments (A never needs a tensor-core layout, so either major works);
//                          * make B the K-major operand wgmma reads from shared memory when it did not arrive that way
//                            and warps 1-3 do not convert it (MN-major tiles are transposed, fp32 operands split into
//                            hi | lo or converted to bf16);
//                          * issue the MMAs;
//                        pipelined (mma_pipeline): k-block kb + 1 is prepared -- B made ready, A fragments built into a
//                        second register buffer -- while kb's MMAs run, and kb's stage is released one k-block late;
//                        after the last k-block they stage the accumulators through shared memory and hand 32-column row
//                        pieces to Policy::store, a warp covering 32 consecutive rows -- or, where the policy offers it
//                        (Policy::kStoreVec4), 4-column groups to Policy::load4 / store4, a warp covering whole rows.
// The producer warpgroup gives registers to the consumers (setmaxnreg: 40 / 232 per thread).  The kernel must contain no
// function call anywhere (no printf, no 64-bit division helper in a Policy): ptxas then serializes every wgmma (C7510).
//
// A Policy supplies the problem-specific parts:
//   static constexpr int  BN, kABytes, kBBytes;  static constexpr bool kSplitA, kSplitB (operand needs the in-kernel split);
//   static constexpr bool kAMN, kBMN (operand majors);  struct Params;
//   static __device__ int  num_tiles(const Params&);          static __device__ int num_kb(const Params&, int tile);
//   struct Tile;  static __device__ Tile tile(p, tile);       // tile coordinates, decoded ONCE per tile (integer divisions)
//   static __device__ void load(p, Tile&, mapA, mapB, sa, sb, sb_lo, bar, leader);   // TMA for the next k-block of the tile
//                              // (fixed tx bytes, issued by the leader lane only); every lane advances the k cursor in Tile
//   static __device__ void load16(..., halves);               // the same for the bf16 modes with a pre-converted B
//   static __device__ void store(p, const Tile&, row, col0, const float (&v)[32]);     // 32 accumulator columns of one row
//   static constexpr bool kStoreVec4 (optional);  struct Epi4;  bool vec4_ok(p);  Epi4 load4(p, Tile, row, col);
//       void store4(p, Tile, row, col, float4 v, const Epi4&);     // coalesced epilogue (epilogue_vec4), 4 columns of one row
//   static constexpr bool kSumA, kSumB;   // fused reductions over the contraction index, taken from the fp32 operand tiles
//       the consumers read anyway: kSumA = row sums of A, kSumB = column sums of an MN-major B tile (bias gradients of the
//       weight-gradient GEMMs -- a separate column-sum pass would re-read the operand from HBM)
//   static __device__ bool want_sums(p, Tile);  void sum_a_store(p, Tile, row, v);  void sum_b_store1(p, Tile, col, v);
//       each called once per row / column and tile, with sums taken in a fixed order (no atomics: run-to-run reproducible)
// The producer is ONE thread: anything it does per k-block is on the critical path of the whole SM, so tile coordinates are
// decoded once per tile and k-blocks advance a cursor.
//
// Shared-memory tile layouts (TMA, 128-byte swizzle):
//   K-major fp32 tile (rows x 32 k): row r = 128 B, 16-byte chunk c stored at chunk c ^ (r & 7)
//   MN-major fp32 tile: chunks of 32 rows (4 KB) of 32 k-lines x 128 B; within a k-line, chunk c ^ (k & 7)
//   MN-major bf16 tile ("pairs"): chunks of 64 rows (4 KB) of 32 k-lines x 128 B; within a k-line, chunk c ^ (k & 7)
//   K-major bf16 tile (rows x 32 k): row r = 64 B, chunk c stored at c ^ ((r >> 1) & 3) (64-byte swizzle)
#pragma once
#include <type_traits>

#include "common.cuh"
#include "tc_common.cuh"

namespace b200asr {
namespace tc {

// NSPLIT selects the arithmetic: 1 = TF32, 3 = 3xTF32 (hi*hi + hi*lo + lo*hi over x = hi + lo), 2 = bf16 and
// 6 = bf16x3 (2-term bf16 split, three MMAs at twice the tf32 rate).  In the bf16 modes B is
//   * either a PRE-CONVERTED K-major bf16 operand ([hi] or [hi | lo], 64-byte rows, SWIZZLE_64B; Policy::load16) -- weights,
//   * or (Policy::kSplitB, both operands MN-major: the weight-gradient GEMMs, whose operands are activations) the raw fp32
//     MN-major tile, which the consumers convert into K-major bf16 tiles in a second shared-memory region of the stage,
//   * or (Policy::kBMN without kSplitB) MN-major bf16 hi | lo tiles that the PRODUCER of the activation already wrote next to
//     the fp32 tensor ("pairs"): loaded by TMA like the weights and transposed in place.
__host__ __device__ constexpr bool eng_is_bf16(int nsplit) { return nsplit == 2 || nsplit == 6; }

constexpr int ENG_THREADS = 384;
constexpr int ENG_CONSUMERS = 256;
constexpr int ENG_BAR = 1;                 // named barrier of the consumer threads
constexpr int ENG_SMEM_CAP = 227 * 1024;   // dynamic shared memory per block on sm_90

enum EngBMode { B_READY, B_SPLIT_K, B_T32, B_T16_FROM32, B_T16 };
// accumulator staging buffer of the epilogue: 128 rows of min(BN, 64) + 4 floats (+4: conflict-free row reads)
constexpr int epilogue_bytes(int BN) { return 128 * ((BN < 64 ? BN : 64) + 4) * 4; }

template <class Policy, int NSPLIT> struct EngineCfg {
  static constexpr bool kBf16 = eng_is_bf16(NSPLIT);
  static constexpr int BN = Policy::BN;
  static constexpr int kBHalves = (NSPLIT == 3 || NSPLIT == 6) ? 2 : 1;                     // B tiles per stage (hi | lo)
  static constexpr int kBTile = kBf16 ? BN * 64 : Policy::kBBytes;                           // bf16: 32 k x 2 B = 64-byte rows
  static constexpr int kBRaw = (kBf16 && Policy::kSplitB) ? Policy::kBBytes : 0;             // bf16 + in-kernel B conversion: raw fp32 tile
  static constexpr int kStageBytes = Policy::kABytes + kBRaw + kBHalves * kBTile;
  static constexpr int kOffBraw = Policy::kABytes;
  static constexpr int kOffBhi = Policy::kABytes + kBRaw;
  static constexpr int kOffBlo = kOffBhi + kBTile;
  static constexpr int kBMode = kBf16 ? (Policy::kSplitB ? B_T16_FROM32 : (Policy::kBMN ? B_T16 : B_READY))
                                      : (Policy::kBMN ? B_T32 : ((NSPLIT == 3 && Policy::kSplitB) ? B_SPLIT_K : B_READY));
  static constexpr bool kBSplit = NSPLIT == 3 && Policy::kSplitB;     // B_T32: fp32 B split into hi | lo while transposed
  // B_T16_FROM32 without column sums: warps 1-3 convert B (engine_convert_b16) and signal the consumers per stage.
  // (B_T32 transposes in place, which needs the whole tile in registers first; B_SPLIT_K on warps 1-3 measured no faster.)
  static constexpr bool kBByProducer = kBMode == B_T16_FROM32 && !Policy::kSumB;
  static constexpr int kTxBytes = kBf16 ? Policy::kABytes + (Policy::kSplitB ? Policy::kBBytes : kBHalves * kBTile)
                                        : Policy::kABytes + Policy::kBBytes +
                                          (NSPLIT == 3 && !Policy::kSplitB ? Policy::kBBytes : 0);   // pre-split B arrives as hi+lo
  static constexpr int kEpiBytes = epilogue_bytes(BN);
  static constexpr int kBySmem = (ENG_SMEM_CAP - 1024 - kEpiBytes - 256) / kStageBytes;
  static constexpr int kStages = kBySmem > 8 ? 8 : kBySmem;
  static constexpr int kOffEpi = kStages * kStageBytes;
  static constexpr int kBarOff = kOffEpi + kEpiBytes;
  static constexpr int kSmemBytes = kBarOff + 256 + 1024;
  static_assert(!kBf16 || !Policy::kSplitB || (Policy::kAMN && Policy::kBMN),
                "bf16 modes: a pre-converted bf16 B (K-major weights, or MN-major activation pairs), or both operands MN-major fp32 "
                "with B converted in the kernel");
  static_assert(!Policy::kSumB || Policy::kBMN, "column sums need an MN-major B tile");
  static_assert(BN == 32 || BN == 64 || BN == 128, "BN");
  static_assert(kStages >= 2, "stage too large");
  static_assert(3 * 8 * kStages <= 256, "barriers (full, empty, ready per stage)");
  static_assert(kSmemBytes <= ENG_SMEM_CAP, "shared memory");
};

// byte offset of fp32 element (row r, k) of an A tile
template <bool MN> __device__ __forceinline__ uint32_t a_off(int r, int k) {
  if constexpr (!MN) return r * 128 + (((k >> 2) ^ (r & 7)) << 4) + (k & 3) * 4;
  else return (r >> 5) * 4096 + k * 128 + ((((r & 31) >> 2) ^ (k & 7)) << 4) + (r & 3) * 4;
}
// K-major targets: fp32 (row n, k) in 128-byte rows, bf16 (row n, k) in 64-byte rows
__device__ __forceinline__ uint32_t kmaj32_off(int n, int k) { return n * 128 + (((k >> 2) ^ (n & 7)) << 4) + (k & 3) * 4; }
__device__ __forceinline__ uint32_t kmaj16_off(int n, int k) { return n * 64 + (((k >> 3) ^ ((n >> 1) & 3)) << 4) + (k & 7) * 2; }

// Register split of the 384 threads (setmaxnreg): the producer warpgroup drops to kProducerRegs, the two consumer warpgroups
// rise to kConsumerRegs -- 128 * 40 + 256 * 232 = 64,512, the 168 per thread that __launch_bounds__(384, 1) allots.  The
// consumers need the room for a second set of A fragments (the pipelined k-loop below) next to the accumulators.
constexpr int kProducerRegs = 40, kConsumerRegs = 232;
static_assert(128 * kProducerRegs + 256 * kConsumerRegs <= 384 * 168, "register split");
template <int N> __device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }
template <int N> __device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }

// wgmma register-A fragments of one 32-deep k-block of this thread's rows r0 / r1: hi (and, for the split modes, lo) per
// k-step -- four tf32 k8 steps or two bf16 k16 steps
template <int NSPLIT> struct AFrag {
  static constexpr int KS = eng_is_bf16(NSPLIT) ? 2 : 4;
  uint32_t h[KS][4], l[KS][4];
};
template <int NSPLIT> __device__ __forceinline__ void keep_live(const AFrag<NSPLIT>& f) {
#pragma unroll
  for (int ks = 0; ks < AFrag<NSPLIT>::KS; ks++) {
    keep_live(f.h[ks]);
    if constexpr (NSPLIT == 3 || NSPLIT == 6) keep_live(f.l[ks]);
  }
}

// The A fragments of one k-block: this thread's A rows r0 / r1 (fp32 in shared memory at a_ptr(r, k)) rounded or split per
// NSPLIT.  KPAIR: elements (r, k) and (r, k + 1) are adjacent (8-byte loads).  SUMS: asum0 / asum1 += the fp32 A values of
// rows r0 / r1 this thread read (a quarter of each row; the caller reduces).
template <int NSPLIT, bool KPAIR, bool SUMS, class APtr>
__device__ __forceinline__ void build_afrag(AFrag<NSPLIT>& f, APtr a_ptr, int r0, int r1, int q, float& asum0, float& asum1) {
  if constexpr (!eng_is_bf16(NSPLIT)) {
#pragma unroll
    for (int ks = 0; ks < 4; ks++) {
      const int k0 = ks * 8 + q, k1 = k0 + 4;
      const float x[4] = {*a_ptr(r0, k0), *a_ptr(r1, k0), *a_ptr(r0, k1), *a_ptr(r1, k1)};
      if constexpr (SUMS) { asum0 += x[0] + x[2]; asum1 += x[1] + x[3]; }
#pragma unroll
      for (int i = 0; i < 4; i++) {
        const float h = tf32_rn(x[i]);
        f.h[ks][i] = __float_as_uint(h);
        f.l[ks][i] = __float_as_uint(x[i] - h);
      }
    }
  } else {
#pragma unroll
    for (int ks = 0; ks < 2; ks++) {
#pragma unroll
      for (int i = 0; i < 4; i++) {
        const int r = (i & 1) ? r1 : r0, k = ks * 16 + (i >> 1) * 8 + 2 * q;
        float x0, x1;
        if constexpr (KPAIR) {
          const float2 v = *reinterpret_cast<const float2*>(a_ptr(r, k));
          x0 = v.x; x1 = v.y;
        } else {
          x0 = *a_ptr(r, k);
          x1 = *a_ptr(r, k + 1);
        }
        if constexpr (SUMS) { if (i & 1) asum1 += x0 + x1; else asum0 += x0 + x1; }
        if constexpr (NSPLIT == 6) split_bf16_pair(x0, x1, f.h[ks][i], f.l[ks][i]);
        else f.h[ks][i] = pack_bf16_pair(x0, x1);
      }
    }
  }
}

// The MMAs of one k-block, committed as one group: acc += A (fragments f) * B (K-major tile(s) at bhi | blo).
template <int NSPLIT, int BN>
__device__ __forceinline__ void issue_kblock(float (&acc)[BN / 2], const AFrag<NSPLIT>& f, uint32_t bhi, uint32_t blo) {
  wgmma_fence();
#pragma unroll
  for (int ks = 0; ks < AFrag<NSPLIT>::KS; ks++) {
    if constexpr (!eng_is_bf16(NSPLIT)) {
      if constexpr (NSPLIT == 3) {            // small products first: lo*hi + hi*lo + hi*hi
        wgmma_tf32<BN>(acc, f.l[ks], kmajor_desc_tf32(bhi + ks * 32));
        wgmma_tf32<BN>(acc, f.h[ks], kmajor_desc_tf32(blo + ks * 32));
      }
      wgmma_tf32<BN>(acc, f.h[ks], kmajor_desc_tf32(bhi + ks * 32));
    } else {
      if constexpr (NSPLIT == 6) {
        wgmma_bf16<BN>(acc, f.l[ks], kmajor_desc_bf16(bhi + ks * 32));
        wgmma_bf16<BN>(acc, f.h[ks], kmajor_desc_bf16(blo + ks * 32));
      }
      wgmma_bf16<BN>(acc, f.h[ks], kmajor_desc_bf16(bhi + ks * 32));
    }
  }
  wgmma_commit();
}

// Pipelined k-loop over the nkb k-blocks of one tile: the MMAs of k-block kb run while the fragments of kb + 1 are built
// into the other of two fragment buffers, and k-block kb's stage is released one k-block late, once the wait that leaves
// only kb + 1's group in flight has retired its MMAs.  Each accumulator still receives the same MMAs in the same order.
//   prep(kb, f, bhi, blo): wait for k-block kb's data, make its B operand ready, build its fragments into f and return the
//                          shared-memory addresses of its B tile(s) -- called once per k-block, in order;
//   release(kb):           k-block kb's MMAs have completed (its stage may be refilled) -- called once per k-block, in order.
// Returns with every MMA complete.  The loop runs two k-blocks per trip so that the buffer index is a compile-time constant.
template <int NSPLIT, int BN, class Prep, class Release>
__device__ __forceinline__ void mma_pipeline(float (&acc)[BN / 2], int nkb, Prep&& prep, Release&& release) {
  if (nkb <= 0) return;
  AFrag<NSPLIT> f[2];
  uint32_t bhi[2], blo[2];
  prep(0, f[0], bhi[0], blo[0]);
  auto step = [&](auto u_, int kb) {
    constexpr int U = decltype(u_)::value;
    issue_kblock<NSPLIT, BN>(acc, f[U], bhi[U], blo[U]);
    if (kb > 0) {
      wgmma_wait<1>();                     // k-block kb - 1 is done: its fragment buffer and its stage are free
      keep_live(f[U ^ 1]);                 // (until here the compiler must not reuse those registers)
      release(kb - 1);
    }
    if (kb + 1 < nkb) prep(kb + 1, f[U ^ 1], bhi[U ^ 1], blo[U ^ 1]);
  };
  for (int kb = 0; kb < nkb; kb += 2) {
    step(std::integral_constant<int, 0>(), kb);
    if (kb + 1 < nkb) step(std::integral_constant<int, 1>(), kb + 1);
  }
  wgmma_wait<0>();
  keep_live(f[0]);
  keep_live(f[1]);
  acc_fence(acc);
  release(nkb - 1);
}

// Accumulators of a 128 x BN tile (this thread: rows r0 / r1) staged through shared memory `epi` (128 rows of EC + 4 floats)
// and handed out as 32-column row pieces: out(row, col0, v[32]) with row = ctid % 128, so a warp covers 32 consecutive rows.
// All ENG_CONSUMERS threads call it.
template <int BN, class Out>
__device__ __forceinline__ void epilogue_rows(const float (&acc)[BN / 2], float* epi, int ctid, int r0, int r1, int q, Out out) {
  constexpr int EC = BN < 64 ? BN : 64, EP = EC + 4;
#pragma unroll
  for (int cc = 0; cc < BN / EC; cc++) {
    named_bar_sync(ENG_BAR, ENG_CONSUMERS);           // the previous chunk's readers are done with the buffer
#pragma unroll
    for (int j = 0; j < EC / 8; j++) {
      const int jj = cc * (EC / 8) + j, col = j * 8 + 2 * q;
      *reinterpret_cast<float2*>(epi + r0 * EP + col) = make_float2(acc[4 * jj], acc[4 * jj + 1]);
      *reinterpret_cast<float2*>(epi + r1 * EP + col) = make_float2(acc[4 * jj + 2], acc[4 * jj + 3]);
    }
    named_bar_sync(ENG_BAR, ENG_CONSUMERS);
    const int row = ctid & 127, piece = ctid >> 7;
    if (piece < EC / 32) {
      float v[32];
#pragma unroll
      for (int j = 0; j < 8; j++) {
        const float4 t = *reinterpret_cast<const float4*>(epi + row * EP + piece * 32 + j * 4);
        v[4 * j] = t.x; v[4 * j + 1] = t.y; v[4 * j + 2] = t.z; v[4 * j + 3] = t.w;
      }
      out(row, cc * EC + piece * 32, v);
    }
  }
}

// Policy::kStoreVec4 (optional, default false): the policy also offers a coalesced epilogue -- vec4_ok(p) says whether a
// launch may use it, load4 / store4 handle 4 consecutive columns of one row (loads first, so that a thread's loads of
// several groups are in flight together)
template <class P, class = void> struct policy_store_vec4 : std::false_type {};
template <class P> struct policy_store_vec4<P, std::void_t<decltype(P::kStoreVec4)>> : std::bool_constant<P::kStoreVec4> {};

// The accumulators staged as in epilogue_rows, but handed out as 4-column groups: EC / 4 consecutive lanes cover one row
// of the chunk, so every global access of a warp is a contiguous run of its rows (a 32-column row piece per thread puts
// each of a warp's 16-byte accesses in a different cache line).  All ENG_CONSUMERS threads call it.
template <class Policy, int BN>
__device__ __forceinline__ void epilogue_vec4(const typename Policy::Params& p, const typename Policy::Tile& tc,
                                              const float (&acc)[BN / 2], float* epi, int ctid, int r0, int r1, int q) {
  constexpr int EC = BN < 64 ? BN : 64, EP = EC + 4;
  constexpr int LPR = EC / 4, RPP = ENG_CONSUMERS / LPR, NIT = 128 / RPP, U = 2;   // lanes per row, rows per pass, passes
  static_assert(NIT % U == 0, "passes");
  const int cl = ctid % LPR, rl = ctid / LPR;
#pragma unroll
  for (int cc = 0; cc < BN / EC; cc++) {
    named_bar_sync(ENG_BAR, ENG_CONSUMERS);           // the previous chunk's readers are done with the buffer
#pragma unroll
    for (int j = 0; j < EC / 8; j++) {
      const int jj = cc * (EC / 8) + j, col = j * 8 + 2 * q;
      *reinterpret_cast<float2*>(epi + r0 * EP + col) = make_float2(acc[4 * jj], acc[4 * jj + 1]);
      *reinterpret_cast<float2*>(epi + r1 * EP + col) = make_float2(acc[4 * jj + 2], acc[4 * jj + 3]);
    }
    named_bar_sync(ENG_BAR, ENG_CONSUMERS);
    const int col = cc * EC + cl * 4;
#pragma unroll
    for (int i0 = 0; i0 < NIT; i0 += U) {
      float4 v[U];
      typename Policy::Epi4 x[U];
#pragma unroll
      for (int u = 0; u < U; u++) {
        const int row = (i0 + u) * RPP + rl;
        v[u] = *reinterpret_cast<const float4*>(epi + row * EP + cl * 4);
        x[u] = Policy::load4(p, tc, row, col);
      }
#pragma unroll
      for (int u = 0; u < U; u++) Policy::store4(p, tc, (i0 + u) * RPP + rl, col, v[u], x[u]);
    }
  }
}

constexpr int ENG_CONVERTERS = 3;          // warps 1-3 (Cfg::kBByProducer)

// fp32 MN-major B tile (BN columns x 32 k, at src) -> K-major bf16 hi (| lo) tiles at dh / dl, by one of the ENG_CONVERTERS
// warps (cw): a work item is 32 consecutive columns (lane = column) x 8 consecutive k, read down 8 k-lines and stored as one
// 16-byte row piece per half.  The same split_bf16_pair / pack_bf16_pair of the same (k, k + 1) pairs as the consumers' path.
template <int NSPLIT, int BN>
__device__ __forceinline__ void engine_convert_b16(const uint8_t* src, uint8_t* dh, uint8_t* dl, int cw, int lane) {
  for (int it = cw; it < (BN / 32) * 4; it += ENG_CONVERTERS) {
    const int n = (it >> 2) * 32 + lane, kg = it & 3;
    const uint8_t* col = src + (it >> 2) * 4096 + (lane & 3) * 4;
    float x[8];
#pragma unroll
    for (int j = 0; j < 8; j++) {
      const int k = kg * 8 + j;
      x[j] = *reinterpret_cast<const float*>(col + k * 128 + ((((lane & 31) >> 2) ^ (k & 7)) << 4));
    }
    uint32_t hi[4], lo[4];
#pragma unroll
    for (int j = 0; j < 4; j++) {
      if constexpr (NSPLIT == 6) split_bf16_pair(x[2 * j], x[2 * j + 1], hi[j], lo[j]);
      else hi[j] = pack_bf16_pair(x[2 * j], x[2 * j + 1]);
    }
    *reinterpret_cast<uint4*>(dh + kmaj16_off(n, kg * 8)) = make_uint4(hi[0], hi[1], hi[2], hi[3]);
    if constexpr (NSPLIT == 6) *reinterpret_cast<uint4*>(dl + kmaj16_off(n, kg * 8)) = make_uint4(lo[0], lo[1], lo[2], lo[3]);
  }
}

template <class Policy, int NSPLIT>
__global__ void __launch_bounds__(ENG_THREADS, 1)
tc_engine_kernel(const __grid_constant__ CUtensorMap mapA, const __grid_constant__ CUtensorMap mapB,
                 const typename Policy::Params p) {
  using Cfg = EngineCfg<Policy, NSPLIT>;
  constexpr int S = Cfg::kStages;
  constexpr int BN = Policy::BN;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* gen_base = smem_raw + (smem_base - smem_u32(smem_raw));
  const uint32_t bar_base = smem_base + Cfg::kBarOff;
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (S + s); };
  auto ready_bar = [&](int s) { return bar_base + 8u * (2 * S + s); };   // Cfg::kBByProducer: B of stage s converted

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int ntiles = Policy::num_tiles(p);

  if (threadIdx.x == 0) {
    for (int s = 0; s < S; s++) { mbar_init(full_bar(s), 1); mbar_init(empty_bar(s), ENG_CONSUMERS / 32); }
    if constexpr (Cfg::kBByProducer)
      for (int s = 0; s < S; s++) mbar_init(ready_bar(s), ENG_CONVERTERS);
    fence_barrier_init();
    tma_prefetch_desc(&mapA);
    tma_prefetch_desc(&mapB);
  }
  __syncthreads();
  griddep_launch();      // the next kernel in the stream may start its own prologue as our CTAs retire ...
  griddep_wait();        // ... and ours ran under the predecessor's tail: from here on its results are visible (common.cuh)

  if (warp < 4) {
    setmaxnreg_dec<kProducerRegs>();   // the whole producer warpgroup, so that the consumers can take the registers
    if (warp != 0) {
      if constexpr (Cfg::kBByProducer) {
        // ---------------------------------------------------------------- B conversion (warps 1-3), in k-block order
        uint32_t s = 0, ph = 0;
        for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
          const int nkb = Policy::num_kb(p, tile);
          for (int kb = 0; kb < nkb; kb++) {
            mbar_wait(full_bar(s), ph);
            uint8_t* stage = gen_base + s * Cfg::kStageBytes;
            engine_convert_b16<NSPLIT, BN>(stage + Cfg::kOffBraw, stage + Cfg::kOffBhi, stage + Cfg::kOffBlo, warp - 1, lane);
            fence_proxy_async_smem();        // the consumers' wgmma read these tiles through the async proxy
            __syncwarp();
            if (lane == 0) mbar_arrive(ready_bar(s));
            if (++s == S) { s = 0; ph ^= 1; }
          }
        }
      }
      return;
    }
    // ------------------------------------------------------------------ TMA producer (whole warp loops, one lane issues)
    const bool leader = elect_one();
    uint32_t kbg = 0;
    for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
      const int nkb = Policy::num_kb(p, tile);
      typename Policy::Tile tc = Policy::tile(p, tile);
      for (int kb = 0; kb < nkb; kb++, kbg++) {
        const int s = kbg % S;
        mbar_wait(empty_bar(s), ((kbg / S) & 1) ^ 1);
        const uint32_t sa = smem_base + s * Cfg::kStageBytes;
        if (leader) mbar_expect_tx(full_bar(s), Cfg::kTxBytes);
        if constexpr (Cfg::kBf16 && !Policy::kSplitB) Policy::load16(p, tc, &mapA, &mapB, sa, sa + Cfg::kOffBhi, sa + Cfg::kOffBlo, full_bar(s), leader, Cfg::kBHalves);
        else if constexpr (Cfg::kBf16) Policy::load(p, tc, &mapA, &mapB, sa, sa + Cfg::kOffBraw, 0u, full_bar(s), leader);     // raw fp32 A and B tiles
        else Policy::load(p, tc, &mapA, &mapB, sa, sa + Cfg::kOffBhi, sa + Cfg::kOffBlo, full_bar(s), leader);
        __syncwarp();
      }
    }
    return;
  }
  setmaxnreg_inc<kConsumerRegs>();

  // -------------------------------------------------------------------- consumers
  const int ctid = threadIdx.x - 128;                 // 0 .. 255
  const int wg = ctid >> 7, cw = (ctid >> 5) & 3;
  const int g = lane >> 2, q = lane & 3;
  const int r0 = wg * 64 + cw * 16 + g, r1 = r0 + 8;  // the two A / accumulator rows of this thread
  // B conversion: thread owns 4 consecutive columns n0..n0+3 and KR consecutive k from kk0
  constexpr int NG = BN / 4, KSPL = ENG_CONSUMERS / NG, KR = 32 / KSPL;
  const int n0 = (ctid % NG) * 4, kk0 = (ctid / NG) * KR;
  float* epi = reinterpret_cast<float*>(gen_base + Cfg::kOffEpi);

  uint32_t s = 0, ph = 0, rs = 0;                     // ring position / phase of the next k-block, ring position of the next release
  for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int nkb = Policy::num_kb(p, tile);
    const typename Policy::Tile tc = Policy::tile(p, tile);
    constexpr bool kSums = Policy::kSumA || Policy::kSumB;
    bool want = false;
    if constexpr (kSums) want = Policy::want_sums(p, tc);
    float asum0 = 0.f, asum1 = 0.f;
    float4 bsum = make_float4(0.f, 0.f, 0.f, 0.f);
    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; i++) acc[i] = 0.f;

    auto prep = [&](int, AFrag<NSPLIT>& f, uint32_t& bhi, uint32_t& blo) {
      mbar_wait(full_bar(s), ph);
      if constexpr (Cfg::kBByProducer) mbar_wait(ready_bar(s), ph);
      uint8_t* stage = gen_base + s * Cfg::kStageBytes;
      const uint32_t stage_s = smem_base + s * Cfg::kStageBytes;

      // ---- B as the K-major operand
      if constexpr (Cfg::kBMode == B_SPLIT_K) {
        // elementwise, so the (swizzled) layout does not matter: hi in place, lo into the lo tile
        float4* bh = reinterpret_cast<float4*>(stage + Cfg::kOffBhi);
        float4* bl = reinterpret_cast<float4*>(stage + Cfg::kOffBlo);
#pragma unroll 4
        for (int i = ctid; i < Policy::kBBytes / 16; i += ENG_CONSUMERS) {
          const float4 x = bh[i];
          float4 h, l;
          h.x = tf32_rn(x.x); l.x = x.x - h.x;
          h.y = tf32_rn(x.y); l.y = x.y - h.y;
          h.z = tf32_rn(x.z); l.z = x.z - h.z;
          h.w = tf32_rn(x.w); l.w = x.w - h.w;
          bh[i] = h;
          bl[i] = l;
        }
        fence_proxy_async_smem();
        named_bar_sync(ENG_BAR, ENG_CONSUMERS);
      } else if constexpr (Cfg::kBMode == B_T32 || (Cfg::kBMode == B_T16_FROM32 && !Cfg::kBByProducer)) {
        // fp32 MN-major tile -> K-major (tf32: as is, or hi | lo; bf16: hi (| lo)); thread: 4 columns x KR k-lines
        const uint8_t* src = stage + (Cfg::kBMode == B_T32 ? Cfg::kOffBhi : Cfg::kOffBraw);
        constexpr int NH = (Cfg::kBMode == B_T32 && !Cfg::kBSplit) ? Cfg::kBHalves : 1;    // pre-split halves transposed as they are
        float x[NH][KR][4];
#pragma unroll
        for (int hf = 0; hf < NH; hf++)
#pragma unroll
          for (int i = 0; i < KR; i++) {
            const int k = kk0 + i;
            const float4 v = *reinterpret_cast<const float4*>(src + hf * Cfg::kBTile + (n0 >> 5) * 4096 + k * 128 +
                                                              ((((n0 & 31) >> 2) ^ (k & 7)) << 4));
            x[hf][i][0] = v.x; x[hf][i][1] = v.y; x[hf][i][2] = v.z; x[hf][i][3] = v.w;
            if (hf == 0) { bsum.x += v.x; bsum.y += v.y; bsum.z += v.z; bsum.w += v.w; }
          }
        if constexpr (Cfg::kBMode == B_T32) named_bar_sync(ENG_BAR, ENG_CONSUMERS);     // in place: every thread has read the tile
#pragma unroll
        for (int c = 0; c < 4; c++) {
          const int n = n0 + c;
          if constexpr (Cfg::kBMode == B_T32) {
#pragma unroll
            for (int hf = 0; hf < (Cfg::kBSplit ? 2 : NH); hf++) {
              float o[KR];
#pragma unroll
              for (int i = 0; i < KR; i++) {
                const float v = x[Cfg::kBSplit ? 0 : hf][i][c];
                o[i] = Cfg::kBSplit ? (hf == 0 ? tf32_rn(v) : v - tf32_rn(v)) : v;
              }
              uint8_t* dst = stage + Cfg::kOffBhi + hf * Cfg::kBTile + kmaj32_off(n, kk0);
              if constexpr (KR == 4) *reinterpret_cast<float4*>(dst) = make_float4(o[0], o[1], o[2], o[3]);
              else if constexpr (KR == 2) *reinterpret_cast<float2*>(dst) = make_float2(o[0], o[1]);
              else *reinterpret_cast<float*>(dst) = o[0];
            }
          } else {
            uint32_t hi[(KR + 1) / 2], lo[(KR + 1) / 2];
#pragma unroll
            for (int i = 0; i < KR; i += 2) {
              const float v0 = x[0][i][c], v1 = KR > 1 ? x[0][i + 1 < KR ? i + 1 : i][c] : 0.f;
              if constexpr (NSPLIT == 6) split_bf16_pair(v0, v1, hi[i / 2], lo[i / 2]);
              else hi[i / 2] = pack_bf16_pair(v0, v1);
            }
            uint8_t* dh = stage + Cfg::kOffBhi + kmaj16_off(n, kk0);
            uint8_t* dl = stage + Cfg::kOffBlo + kmaj16_off(n, kk0);
            if constexpr (KR == 4) {
              *reinterpret_cast<uint2*>(dh) = make_uint2(hi[0], hi[1]);
              if constexpr (NSPLIT == 6) *reinterpret_cast<uint2*>(dl) = make_uint2(lo[0], lo[1]);
            } else if constexpr (KR == 2) {
              *reinterpret_cast<uint32_t*>(dh) = hi[0];
              if constexpr (NSPLIT == 6) *reinterpret_cast<uint32_t*>(dl) = lo[0];
            } else {
              *reinterpret_cast<uint16_t*>(dh) = (uint16_t)hi[0];
              if constexpr (NSPLIT == 6) *reinterpret_cast<uint16_t*>(dl) = (uint16_t)lo[0];
            }
          }
        }
        fence_proxy_async_smem();
        named_bar_sync(ENG_BAR, ENG_CONSUMERS);
      } else if constexpr (Cfg::kBMode == B_T16) {
        // bf16 MN-major hi | lo tiles (64-column chunks) -> K-major bf16 tiles, in place; column sums of hi + lo
        uint32_t hv[KR][2], lv[KR][2];
#pragma unroll
        for (int i = 0; i < KR; i++) {
          const int k = kk0 + i;
          const uint32_t off = (n0 >> 6) * 4096 + k * 128 + ((((n0 & 63) >> 3) ^ (k & 7)) << 4) + (n0 & 7) * 2;
          const uint2 h = *reinterpret_cast<const uint2*>(stage + Cfg::kOffBhi + off);
          uint2 l = make_uint2(0u, 0u);
          if constexpr (NSPLIT == 6) l = *reinterpret_cast<const uint2*>(stage + Cfg::kOffBlo + off);
          hv[i][0] = h.x; hv[i][1] = h.y; lv[i][0] = l.x; lv[i][1] = l.y;
          bsum.x += __uint_as_float(h.x << 16) + __uint_as_float(l.x << 16);
          bsum.y += __uint_as_float(h.x & 0xFFFF0000u) + __uint_as_float(l.x & 0xFFFF0000u);
          bsum.z += __uint_as_float(h.y << 16) + __uint_as_float(l.y << 16);
          bsum.w += __uint_as_float(h.y & 0xFFFF0000u) + __uint_as_float(l.y & 0xFFFF0000u);
        }
        named_bar_sync(ENG_BAR, ENG_CONSUMERS);
#pragma unroll
        for (int c = 0; c < 4; c++) {
          const int n = n0 + c;
#pragma unroll
          for (int hf = 0; hf < (NSPLIT == 6 ? 2 : 1); hf++) {
            uint8_t* dst = stage + (hf ? Cfg::kOffBlo : Cfg::kOffBhi) + kmaj16_off(n, kk0);
            uint32_t e[KR];     // column c of the 4: 16-bit half (c & 1) of word (c >> 1)
#pragma unroll
            for (int i = 0; i < KR; i++) e[i] = ((hf ? lv[i][c >> 1] : hv[i][c >> 1]) >> ((c & 1) * 16)) & 0xFFFFu;
            if constexpr (KR == 4) *reinterpret_cast<uint2*>(dst) = make_uint2(e[0] | (e[1] << 16), e[2] | (e[3] << 16));
            else if constexpr (KR == 2) *reinterpret_cast<uint32_t*>(dst) = e[0] | (e[1] << 16);
            else *reinterpret_cast<uint16_t*>(dst) = (uint16_t)e[0];
          }
        }
        fence_proxy_async_smem();
        named_bar_sync(ENG_BAR, ENG_CONSUMERS);
      }

      // ---- A fragments
      const uint8_t* araw = stage;
      build_afrag<NSPLIT, !Policy::kAMN, Policy::kSumA>(
          f, [&](int r, int k) { return reinterpret_cast<const float*>(araw + a_off<Policy::kAMN>(r, k)); }, r0, r1, q, asum0, asum1);
      bhi = stage_s + Cfg::kOffBhi;
      blo = stage_s + Cfg::kOffBlo;
      if (++s == S) { s = 0; ph ^= 1; }
    };
    mma_pipeline<NSPLIT, BN>(acc, nkb, prep, [&](int) {
      __syncwarp();
      if (lane == 0) mbar_arrive(empty_bar(rs));
      if (++rs == S) rs = 0;
    });

    // ---- fused reductions
    if constexpr (kSums) {
      if (want) {
        if constexpr (Policy::kSumA) {
          asum0 += __shfl_xor_sync(0xffffffffu, asum0, 1);
          asum0 += __shfl_xor_sync(0xffffffffu, asum0, 2);
          asum1 += __shfl_xor_sync(0xffffffffu, asum1, 1);
          asum1 += __shfl_xor_sync(0xffffffffu, asum1, 2);
          if (q == 0) { Policy::sum_a_store(p, tc, r0, asum0); Policy::sum_a_store(p, tc, r1, asum1); }
        }
        if constexpr (Policy::kSumB) {
          // the KSPL threads of a column group hold sums over their k-lines: add them in a fixed order
          named_bar_sync(ENG_BAR, ENG_CONSUMERS);         // the previous tile's epilogue is done with the buffer
          *reinterpret_cast<float4*>(epi + (ctid / NG) * BN + n0) = bsum;
          named_bar_sync(ENG_BAR, ENG_CONSUMERS);
          if (ctid < BN) {
            float s = 0.f;
            for (int j = 0; j < KSPL; j++) s += epi[j * BN + ctid];
            Policy::sum_b_store1(p, tc, ctid, s);
          }
        }
      }
    }

    // ---- epilogue
    // (not with B_T32: its consumers hold the transposed B tile and are close to kConsumerRegs already)
    constexpr bool kVec4 = policy_store_vec4<Policy>::value && Cfg::kBMode != B_T32;
    bool vec4 = false;
    if constexpr (kVec4) vec4 = Policy::vec4_ok(p);
    if constexpr (kVec4) {
      if (vec4) epilogue_vec4<Policy, BN>(p, tc, acc, epi, ctid, r0, r1, q);
    }
    if (!vec4)
      epilogue_rows<BN>(acc, epi, ctid, r0, r1, q, [&](int row, int col0, const float (&v)[32]) { Policy::store(p, tc, row, col0, v); });
  }
}

template <class Policy, int NSPLIT>
int launch_engine(const CUtensorMap& ma, const CUtensorMap& mb, const typename Policy::Params& p, int ntiles, cudaStream_t st,
                  const char* what) {
  using Cfg = EngineCfg<Policy, NSPLIT>;
  auto* kern = tc_engine_kernel<Policy, NSPLIT>;
  static bool attr_set[kMaxDevices] = {};
  if (int rc = ensure_dynamic_smem((const void*)kern, Cfg::kSmemBytes, attr_set, what)) return rc;
  if (ntiles <= 0) return B200ASR_OK;
  const int grid = min(ntiles, device_sm_count());
  launch_pdl(kern, dim3(grid), dim3(ENG_THREADS), Cfg::kSmemBytes, st, ma, mb, p);
  return check_launch(what);
}

}  // namespace tc
}  // namespace b200asr
