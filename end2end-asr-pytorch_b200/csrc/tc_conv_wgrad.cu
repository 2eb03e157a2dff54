// 3x3 convolution weight gradient, "halo" variant: all nine taps of a 64-input-channel slice from ONE x patch per pixel
// block, 3xTF32 or TF32 (wgmma, register A).
//
//   dwr[tap][ci][co] = sum_p x[p + off(tap)][ci] * dy[p][co]        (pixels p are the contraction axis)
//
// Why: the tap-shifted weight gradient (tc_conv.cu, WgradPolicy) covers 128 rows of (tap, ci) per tile, so a pixel block's
// dy tile is fetched, transposed and split once per tap group (5 or 9 times) and its x data once per tap.  Here a tile is
// 9 taps x 64 input channels (M = 576, nine m64 row blocks) x 64 output channels: per pixel block of 4 (time) x 8 (freq)
// the CTA loads the x patch including its one-pixel halo -- 6 x 10 pixels x 64 channels, TMA zero fill = padding -- and
// the dy tile once, converts dy once for all nine taps, and the taps are nine shifted row mappings of the patch, exactly
// as in the halo forward convolution (tc_conv_halo.cu).
//
// Roles (384 threads, 1 CTA / SM, one tile per CTA):
//   warpgroup 0            producer: warp 0 issues the TMA of the x patch + dy tile of each pixel block into a ring of
//                          stages; warps 0-3 convert dy -- raw MN-major tile -> K-major hi | lo in the same stage, once for
//                          all nine taps, with the bias-gradient column sums on the way -- and signal the consumers through
//                          an mbarrier.
//   warpgroups 1, 2        consumers: warpgroup 1 owns taps 0-4, warpgroup 2 taps 5-8 (tap = 3 (df + 1) + dt + 1), i.e. five
//                          / four m64n64 accumulator blocks.  A pipeline unit is one (tap, 8-pixel k-step); there are two
//                          fragment buffers.  While unit u's MMAs run, a thread reads unit u + 1's four patch elements,
//                          waits for unit u - 1 (wgmma.wait_group 1), splits the elements into the freed buffer's tf32
//                          hi | lo and issues unit u + 1.  A stage is released one unit late: once the wait in its
//                          successor's first unit has retired the MMAs of its last unit.
// Registers (setmaxnreg): the producer warpgroup drops to 40 per thread and the consumers rise to 232, room for 160
// accumulators, two fragment buffers and the next unit's patch elements.  ptxas (CUDA 12.9) grants the consumers those
// registers only with one code path for both consumer warpgroups, a warp index it knows to be warp-uniform and a branch
// between setmaxnreg.inc and the accumulators' zeroing (see the consumer code); then it spills nothing and serializes no
// wgmma (no C7512, which the 512-thread form with three consumer warpgroups at 152 registers reported).
//
// Contraction order inside a k-step: MMA k position j of step ks is pixel (time ks, freq 2j) for j < 4 and (ks, 2j - 7)
// for j >= 4, so the four lanes q of a quad read patch columns 2q (+1): distinct 128-byte swizzle phases, no bank conflicts.
// The dy conversion writes B in the same order.
//
// Each tile reduces one contiguous range of pixel blocks (its split) and writes its 576 x 64 partial to the split's slot of
// [splits][9][Ci][Co]; reduce_parts sums the splits in a fixed order (no floating-point atomics: bit-reproducible).
#include "../../include/b200asr.h"
#include "common.cuh"
#include "kernels.h"
#include "tc_common.cuh"
#include "tc_engine.cuh"

namespace b200asr {
namespace tc {

constexpr int WH_T = 4, WH_F = 8;                        // pixel block = one 32-deep k-block
constexpr int WH_PT = WH_T + 2, WH_PF = WH_F + 2;        // x patch incl. halo: 6 x 10 pixels
constexpr int WH_PATCH_BOX = WH_PT * WH_PF * 128;        // 7,680 B per 32-channel box
constexpr int WH_PATCH_CHUNK = 8192;                     // boxes on 1024-byte boundaries (128B swizzle phase = row & 7)
constexpr int WH_N = 64;                                 // output channels per tile
constexpr int WH_PRODUCER = 128;                         // warpgroup 0: TMA (warp 0) and dy conversion (warps 0-3)
constexpr int WH_CONSUMERS = 256;                        // warpgroups 1, 2
constexpr int WH_THREADS = WH_PRODUCER + WH_CONSUMERS;
constexpr int WH_CONVERTERS = WH_PRODUCER / 32;
constexpr int WH_TAPS0 = 5;                              // accumulator blocks per consumer (warpgroup 2 uses four)
// Register split (setmaxnreg): __launch_bounds__(384, 1) allots 168 per thread; 128 * 40 + 256 * 232 = 384 * 168.  The
// busier consumer holds five m64n64 accumulator blocks (160) next to two hi | lo fragment buffers (16) and the next unit's
// patch elements.
constexpr int WH_PRODUCER_REGS = 40, WH_CONSUMER_REGS = 232;
static_assert(WH_PRODUCER * WH_PRODUCER_REGS + WH_CONSUMERS * WH_CONSUMER_REGS <= WH_THREADS * 168, "register split");
constexpr int WH_BAR_CONV = 1;                           // named barrier of the producer warpgroup (bias partials)

struct WgHaloP {
  float* part;         // [splits][9][Ci][Co] partial weight gradients
  float* bpart;        // [splits][Co] partial bias gradients, or nullptr
  int Ci, Co, ncs, ncn, nft, ntt, blocks_per_cta, total_blocks;
};

// stage: x patch (two 32-channel boxes) | raw dy tile (two 32-channel chunks, MN-major) | dy hi (| lo) K-major 64 x 32
template <int NSPLIT> struct WgHaloCfg {
  static constexpr int kOffRaw = 2 * WH_PATCH_CHUNK;
  static constexpr int kOffHi = kOffRaw + (WH_N / 32) * 4096;
  static constexpr int kOffLo = kOffHi + WH_N * 128;
  static constexpr int kStageBytes = kOffHi + (NSPLIT == 3 ? 2 : 1) * WH_N * 128;
  static constexpr int kTxBytes = 2 * WH_PATCH_BOX + (WH_N / 32) * 4096;
  static constexpr int kBySmem = (ENG_SMEM_CAP - 1024 - 512) / kStageBytes;
  static constexpr int kStages = kBySmem > 8 ? 8 : kBySmem;
  static constexpr int kBarOff = kStages * kStageBytes;
  static constexpr int kBiasOff = kBarOff + 256;          // bias partials of converter warps 2, 3 (WH_N floats)
  static constexpr int kSmemBytes = kBiasOff + 256 + 1024;
  static_assert(kStages >= 3, "stage too large");
  static_assert(3 * 8 * kStages <= 256, "barriers");
  static_assert(WH_N * 4 <= 256, "bias partials");
  static_assert(kSmemBytes <= ENG_SMEM_CAP, "shared memory");
};

template <int NSPLIT>
__global__ void __launch_bounds__(WH_THREADS, 1)
tc_conv3x3_wgrad_kernel(const __grid_constant__ CUtensorMap mapX, const __grid_constant__ CUtensorMap mapDy, const WgHaloP p) {
  using Cfg = WgHaloCfg<NSPLIT>;
  constexpr int S = Cfg::kStages;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* gen_base = smem_raw + (smem_base - smem_u32(smem_raw));
  const uint32_t bar_base = smem_base + Cfg::kBarOff;
  auto full_bar = [&](int s) { return bar_base + 8u * s; };              // x patch and raw dy of stage s landed
  auto ready_bar = [&](int s) { return bar_base + 8u * (S + s); };       // dy hi | lo of stage s written
  auto empty_bar = [&](int s) { return bar_base + 8u * (2 * S + s); };   // the MMAs of stage s completed

  // the warp index through a shuffle, so that ptxas knows the role branches are warp-uniform (with threadIdx.x >> 5 it
  // spills in the consumers)
  const int warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0), lane = threadIdx.x & 31;
  // tile = split z, then (input-channel slice, output-channel slice): the tiles of one split are adjacent CTAs (shared L2).
  // Each role computes these after setmaxnreg, so that nothing is live across it.
  struct Tile { int z, ci0, co0, blk0, nkb; };
  auto tile_of = [&]() {
    const int groups = p.ncs * p.ncn;
    const int z = blockIdx.x / groups, grp = blockIdx.x % groups;
    const int blk0 = z * p.blocks_per_cta;
    return Tile{z, (grp / p.ncn) * 64, (grp % p.ncn) * WH_N, blk0, max(0, min(p.blocks_per_cta, p.total_blocks - blk0))};
  };

  if (threadIdx.x == 0) {
    for (int s = 0; s < S; s++) {
      mbar_init(full_bar(s), 1);
      mbar_init(ready_bar(s), WH_CONVERTERS);
      mbar_init(empty_bar(s), WH_CONSUMERS / 32);
    }
    fence_barrier_init();
    tma_prefetch_desc(&mapX);
    tma_prefetch_desc(&mapDy);
  }
  __syncthreads();
  griddep_launch();      // programmatic dependent launch, see common.cuh
  griddep_wait();

  if (warp < WH_CONVERTERS) {
    // ------------------------------------------------------------------ producer: TMA (warp 0) + dy conversion (warps 0-3)
    setmaxnreg_dec<WH_PRODUCER_REGS>();
    const Tile t = tile_of();
    const int z = t.z, ci0 = t.ci0, co0 = t.co0, blk0 = t.blk0, nkb = t.nkb;
    // The loads run S - 1 pixel blocks ahead of warp 0's conversion.  (Not S: the stage of block kb + S is free only once
    // the consumers have moved on to block kb + 1, which waits for this warpgroup's conversion of it.)
    const bool leader = elect_one() && warp == 0;
    int ft = blk0 % p.nft, tt = (blk0 / p.nft) % p.ntt, b = blk0 / (p.nft * p.ntt);   // pixel-block cursor, ft fastest
    uint32_t ls = 0, lph = 0;                          // ring position / phase of the next load
    int loaded = 0;
    auto load_next = [&]() {
      mbar_wait(empty_bar(ls), lph ^ 1);
      if (leader) {
        const uint32_t sa = smem_base + ls * Cfg::kStageBytes;
        const int f0 = ft * WH_F, t0 = tt * WH_T;
        mbar_expect_tx(full_bar(ls), Cfg::kTxBytes);
#pragma unroll
        for (int c = 0; c < 2; c++) tma_load_4d(sa + c * WH_PATCH_CHUNK, &mapX, full_bar(ls), ci0 + c * 32, f0 - 1, t0 - 1, b);
#pragma unroll
        for (int c = 0; c < WH_N / 32; c++) tma_load_4d(sa + Cfg::kOffRaw + c * 4096, &mapDy, full_bar(ls), co0 + c * 32, f0, t0, b);
      }
      __syncwarp();
      if (++ft == p.nft) {
        ft = 0;
        if (++tt == p.ntt) { tt = 0; b++; }
      }
      if (++ls == S) { ls = 0; lph ^= 1; }
      loaded++;
    };
    if (warp == 0)
      while (loaded < nkb && loaded < S - 1) load_next();
    // dy conversion: warp w converts output channel n = (w & 1) * 32 + lane at k = 16 (w >> 1) .. + 15 (time rows 2 (w >> 1)
    // and + 1); bias-gradient column sums on the way
    const int c = warp & 1, kg0 = (warp >> 1) * 4, n = c * 32 + lane;
    float bs[4] = {0.f, 0.f, 0.f, 0.f};
    uint32_t s = 0, ph = 0;
    for (int kb = 0; kb < nkb; kb++) {
      mbar_wait(full_bar(s), ph);
      uint8_t* stage = gen_base + s * Cfg::kStageBytes;
      const uint8_t* raw = stage + Cfg::kOffRaw + c * 4096 + (lane & 3) * 4;
#pragma unroll
      for (int kk = 0; kk < 4; kk++) {            // K-major k = 4 kg .. 4 kg + 3 (see the contraction order above)
        const int kg = kg0 + kk;
        float x[4], h[4], l[4];
#pragma unroll
        for (int i = 0; i < 4; i++) {
          const int pix = (kg >> 1) * WH_F + 2 * i + (kg & 1);
          x[i] = *reinterpret_cast<const float*>(raw + pix * 128 + (((lane >> 2) ^ (pix & 7)) << 4));
          bs[i] += x[i];
          h[i] = NSPLIT == 3 ? tf32_rn(x[i]) : x[i];
          l[i] = x[i] - h[i];
        }
        *reinterpret_cast<float4*>(stage + Cfg::kOffHi + kmaj32_off(n, 4 * kg)) = make_float4(h[0], h[1], h[2], h[3]);
        if constexpr (NSPLIT == 3)
          *reinterpret_cast<float4*>(stage + Cfg::kOffLo + kmaj32_off(n, 4 * kg)) = make_float4(l[0], l[1], l[2], l[3]);
      }
      fence_proxy_async_smem();
      __syncwarp();
      if (lane == 0) mbar_arrive(ready_bar(s));
      if (++s == S) { s = 0; ph ^= 1; }
      if (warp == 0 && loaded < nkb) load_next();
    }
    // every pixel block is visited once by the input-channel-slice-0 tiles (over all splits); channel n's sum is warp
    // (n / 32)'s time rows 0-1 plus warp (n / 32 + 2)'s rows 2-3, added in that order
    if (p.bpart && ci0 == 0) {
      float* bx = reinterpret_cast<float*>(gen_base + Cfg::kBiasOff);
      const float v = (bs[0] + bs[1]) + (bs[2] + bs[3]);
      if (warp >= 2) bx[n] = v;
      named_bar_sync(WH_BAR_CONV, WH_PRODUCER);
      if (warp < 2) p.bpart[(size_t)z * p.Co + co0 + n] = v + bx[n];
    }
    return;
  }
  setmaxnreg_inc<WH_CONSUMER_REGS>();

  // -------------------------------------------------------------------- consumers
  // Every tile the host launches has at least one pixel block.  This check also starts a basic block after
  // setmaxnreg.inc: with the accumulators zeroed in the block of the setmaxnreg itself, ptxas (CUDA 12.9) spills them and
  // serializes the wgmma.
  const Tile t = tile_of();
  if (t.nkb <= 0) return;
  // Taps and slots.  Tap (dt, df) reads patch row R = (ks + dt + 1) * WH_PF + df + 1 + 2q + h for pixel (ks, 2q + h) of
  // k-step ks.  Both warpgroups run one code path (a second inlined path for the second tap set also makes ptxas serialize
  // and spill).  Relative to patch column 2 wg (wg = 0 / 1: warpgroup 1 / 2), slots 0-2 are rows + 0, 10, 20 (taps 0-2, or
  // 6-8 for wg = 1), slot 3 is + X with X = 1 (tap 3) or 19 (tap 5), and slot 4, wg = 0 only, + 11 (tap 4).  Slot j
  // accumulates into block j.
  const int wg = (warp - WH_CONVERTERS) >> 2, cw = warp & 3, g = lane >> 2, q = lane & 3;
  // A rows of this thread in each tap block: input channels cw * 16 + g and + 8 (same 32-channel box, swizzle chunks cch
  // and cch + 2).  A row's 128B swizzle term depends on (R + pcol) & 7; byte m of sw[m / 4] holds it for R & 7 = m, so that
  // with R known at compile time a load is a byte extract, an xor and an immediate offset.  Slot 3 reads through its own
  // base (X rows further) and table.
  const int cch = ((cw * 16 + g) & 31) >> 2;
  const int pcol = 2 * wg + 2 * q, x3 = wg ? 19 : 1;
  const int aoff = (cw >> 1) * WH_PATCH_CHUNK + (g & 3) * 4 + pcol * 128;
  uint32_t sw[2] = {0u, 0u}, sw3[2] = {0u, 0u};
#pragma unroll
  for (int m = 0; m < 8; m++) {
    sw[m >> 2] |= ((cch ^ ((m + pcol) & 7)) << 4) << (8 * (m & 3));
    sw3[m >> 2] |= ((cch ^ ((m + pcol + x3) & 7)) << 4) << (8 * (m & 3));
  }
  float acc[WH_TAPS0][WH_N / 2];
#pragma unroll
  for (int j = 0; j < WH_TAPS0; j++)
#pragma unroll
    for (int i = 0; i < WH_N / 2; i++) acc[j][i] = 0.f;
  uint32_t ah[2][4], al[2][4];                         // fragment buffer ks % 2 holds k-step ks of a slot
  uint32_t s = 0, ph = 0;
  const uint8_t* patch = gen_base;
  uint32_t bhi = 0;
  auto enter = [&]() {                                 // wait for stage s: x patch landed, dy hi | lo written
    mbar_wait(full_bar(s), ph);
    mbar_wait(ready_bar(s), ph);
    patch = gen_base + s * Cfg::kStageBytes + aoff;
    bhi = smem_base + s * Cfg::kStageBytes + Cfg::kOffHi;
    asm volatile("" : "+r"(sw[0]), "+r"(sw[1]), "+r"(sw3[0]), "+r"(sw3[1]));   // keeps the extracts in the loop (see sw)
  };
  // fragment of (slot sl, k-step ks): a0 = (row g, pixel 2q), a1 = (g + 8, 2q), a2 = (g, 2q + 1), a3 = (g + 8, 2q + 1) of
  // time row ks
  auto load = [&](int sl, int ks, float (&x)[4]) {
    const int r = ks * WH_PF + (sl < 3 ? sl * WH_PF : sl == 4 ? WH_PF + 1 : 0);
    const uint8_t* base = sl == 3 ? patch + x3 * 128 : patch;
    const uint32_t* tab = sl == 3 ? sw3 : sw;
    auto ld = [&](int rr, int c2) {
      const uint32_t sx = (tab[(rr >> 2) & 1] >> (8 * (rr & 3))) & 0xFFu;
      return *reinterpret_cast<const float*>(base + rr * 128 + (sx ^ (c2 ? 32 : 0)));
    };
    x[0] = ld(r, 0);
    x[1] = ld(r, 1);
    x[2] = ld(r + 1, 0);
    x[3] = ld(r + 1, 1);
  };
  auto split = [&](int b, const float (&x)[4]) {
#pragma unroll
    for (int i = 0; i < 4; i++) {
      const float h = tf32_rn(x[i]);
      ah[b][i] = __float_as_uint(h);
      if constexpr (NSPLIT == 3) al[b][i] = __float_as_uint(x[i] - h);
    }
  };
  {
    enter();
    float x[4];
    load(0, 0, x);
    split(0, x);
  }
  // Pipeline unit = (slot, k-step), in order slot 0 .. 3 (.. 4), k-steps 0-3 within a slot.  While unit u's MMAs run, unit
  // u + 1's patch elements are read; the wait then leaves only u in flight, so u - 1's fragment buffer takes u + 1's split.
  // A stage is released one unit late: the wait in the next pixel block's first unit retires the MMAs of its last unit.
  int kb = 0;
  auto unit = [&](int sl, int ks, float (&a)[WH_N / 2], uint32_t bh) {
    const int b = ks & 1;
    const uint32_t bl = bh + (Cfg::kOffLo - Cfg::kOffHi);
    wgmma_fence();
    if constexpr (NSPLIT == 3) {                       // small products first: lo*hi + hi*lo + hi*hi
      wgmma_tf32<WH_N>(a, al[b], kmajor_desc_tf32(bh + ks * 32));
      wgmma_tf32<WH_N>(a, ah[b], kmajor_desc_tf32(bl + ks * 32));
    }
    wgmma_tf32<WH_N>(a, ah[b], kmajor_desc_tf32(bh + ks * 32));
    wgmma_commit();
    const bool last = ks == 3 && (sl == 4 || (sl == 3 && wg != 0));   // the pixel block's last unit
    const bool next = !last || kb + 1 < t.nkb;
    float x[4];
    if (ks < 3) {
      load(sl, ks + 1, x);
    } else if (!last) {
      load(sl + 1, 0, x);
    } else if (next) {                                 // the next pixel block's first unit, once its stage is ready
      if (++s == S) { s = 0; ph ^= 1; }
      enter();
      load(0, 0, x);
    }
    wgmma_wait<1>();                                   // unit u - 1 is done: its fragment buffer is free
    keep_live(ah[b ^ 1]);                              // (so far: the compiler must not reuse those registers while it runs)
    if constexpr (NSPLIT == 3) keep_live(al[b ^ 1]);
    if (sl == 0 && ks == 0 && kb > 0) {                // ... and it was the last unit of the previous stage
      __syncwarp();
      if (lane == 0) mbar_arrive(empty_bar(s == 0 ? S - 1 : s - 1));
    }
    if (next) split(b ^ 1, x);
  };
  for (; kb < t.nkb; kb++) {
    const uint32_t bh = bhi;
#pragma unroll
    for (int sl = 0; sl < 4; sl++)
#pragma unroll
      for (int ks = 0; ks < 4; ks++) unit(sl, ks, acc[sl], bh);
    if (wg == 0) {
#pragma unroll
      for (int ks = 0; ks < 4; ks++) unit(4, ks, acc[4], bh);
    }
  }
  wgmma_wait<0>();
  keep_live(ah[0]);
  keep_live(ah[1]);
  if constexpr (NSPLIT == 3) {
    keep_live(al[0]);
    keep_live(al[1]);
  }
#pragma unroll
  for (int j = 0; j < WH_TAPS0; j++) acc_fence(acc[j]);

  // ---- partials: accumulator (row g (+8), col 8 jj + 2q (+1)) -> [z][tap][ci][co]; a warp stores full 32-byte sectors
#pragma unroll
  for (int j = 0; j < WH_TAPS0; j++) {
    if (j == 4 && wg != 0) continue;
    const int tap = wg == 0 ? j : j < 3 ? 6 + j : 5;
    float* o = p.part + (((size_t)t.z * 9 + tap) * p.Ci + t.ci0 + cw * 16 + g) * p.Co + t.co0 + 2 * q;
#pragma unroll
    for (int jj = 0; jj < WH_N / 8; jj++) {
      *reinterpret_cast<float2*>(o + 8 * jj) = make_float2(acc[j][4 * jj], acc[j][4 * jj + 1]);
      *reinterpret_cast<float2*>(o + 8 * (size_t)p.Co + 8 * jj) = make_float2(acc[j][4 * jj + 2], acc[j][4 * jj + 3]);
    }
  }
}

template <int NSPLIT>
static int launch_wgrad_halo(const CUtensorMap& mx, const CUtensorMap& mdy, const WgHaloP& p, int tiles, cudaStream_t st) {
  using Cfg = WgHaloCfg<NSPLIT>;
  auto* kern = tc_conv3x3_wgrad_kernel<NSPLIT>;
  static bool attr_set[kMaxDevices] = {};
  if (int rc = ensure_dynamic_smem((const void*)kern, Cfg::kSmemBytes, attr_set, "tc_conv3x3_wgrad")) return rc;
  if (tiles <= 0) return B200ASR_OK;
  launch_pdl(kern, dim3(tiles), dim3(WH_THREADS), Cfg::kSmemBytes, st, mx, mdy, p);
  return check_launch("tc_conv3x3_wgrad");
}

}  // namespace tc

// precision 3 (3xTF32) or 1 (TF32, operands rounded by the TMA copy); dwr: [9][Ci][Co]; dbias (3xTF32 only, may be null)
int conv3x3_wgrad_tc_halo(const float* x, const float* dy, float* dwr, int B, int T, int F, int Ci, int Co, int precision,
                          cudaStream_t st, float* dbias, int* dbias_done) {
  using namespace tc;
  if (dbias_done) *dbias_done = 0;
  B200_REQUIRE(precision == 1 || precision == 3, B200ASR_BAD_ARG, "conv3x3_wgrad_tc_halo: precision must be 1 or 3");
  B200_REQUIRE((Ci == 64 || Ci == 128) && (Co == 64 || Co == 128), B200ASR_BAD_SHAPE,
               "conv3x3_wgrad_tc_halo: needs Ci, Co in {64,128} (Ci=%d Co=%d)", Ci, Co);
  B200_REQUIRE(aligned16(x) && aligned16(dy) && aligned16(dwr), B200ASR_BAD_ALIGN, "conv3x3_wgrad_tc_halo: alignment");
  const bool tf32 = precision == 1;
  CUtensorMap mx, mdy;
  {
    uint64_t dims[4] = {(uint64_t)Ci, (uint64_t)F, (uint64_t)T, (uint64_t)B};
    uint64_t strides[3] = {(uint64_t)Ci, (uint64_t)F * Ci, (uint64_t)T * F * Ci};
    uint32_t box[4] = {32, WH_PF, WH_PT, 1};
    if (int rc = make_tensor_map_f32(&mx, x, 4, dims, strides, box, tf32)) return rc;
  }
  {
    uint64_t dims[4] = {(uint64_t)Co, (uint64_t)F, (uint64_t)T, (uint64_t)B};
    uint64_t strides[3] = {(uint64_t)Co, (uint64_t)F * Co, (uint64_t)T * F * Co};
    uint32_t box[4] = {32, WH_F, WH_T, 1};
    if (int rc = make_tensor_map_f32(&mdy, dy, 4, dims, strides, box, tf32)) return rc;
  }
  const bool fuse_bias = dbias != nullptr && !tf32;
  WgHaloP p{nullptr, nullptr, Ci, Co, Ci / 64, Co / WH_N, ceil_div(F, WH_F), ceil_div(T, WH_T), 0, 0};
  const long long total = (long long)B * p.nft * p.ntt;
  B200_REQUIRE(total < (1LL << 31), B200ASR_BAD_SHAPE, "conv3x3_wgrad_tc_halo: too many pixel blocks");
  p.total_blocks = (int)total;
  // one wave: about one tile per SM over the (Ci / 64) x (Co / 64) channel groups, at least 32 pixel blocks per tile
  const int groups = p.ncs * p.ncn;
  p.blocks_per_cta = max(32, ceil_div(p.total_blocks, max(1, device_sm_count() / groups)));
  const int splits = ceil_div(p.total_blocks, p.blocks_per_cta);
  const long long wn = 9LL * Ci * Co;
  p.part = (float*)stream_scratch(sizeof(float) * (size_t)splits * (wn + (fuse_bias ? Co : 0)), st);
  if (!p.part) return B200ASR_CUDA_ERROR;
  p.bpart = fuse_bias ? p.part + (size_t)splits * wn : nullptr;
  int rc = tf32 ? launch_wgrad_halo<1>(mx, mdy, p, groups * splits, st) : launch_wgrad_halo<3>(mx, mdy, p, groups * splits, st);
  if (rc) return rc;
  if ((rc = reduce_parts(p.part, splits, wn, wn, dwr, 0, st))) return rc;
  if (!fuse_bias) return B200ASR_OK;
  if (dbias_done) *dbias_done = 1;
  return reduce_parts(p.bpart, splits, Co, Co, dbias, 0, st);
}

}  // namespace b200asr
