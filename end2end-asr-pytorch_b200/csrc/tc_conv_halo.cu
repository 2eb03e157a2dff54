// 3x3 convolution (forward / data gradient), "halo" variant of the persistent wgmma kernel: 3xTF32, bf16x3 or bf16.
//
// Why: the tap-shifted implicit GEMM (tc_conv.cu) fetches the activation tile nine times per 32-channel slice (once per tap,
// 16 KB each).  Here the 16 x 8 output tile's input patch INCLUDING its one-pixel halo -- 18 x 10 pixels x 32 channels =
// 22.5 KB -- is fetched ONCE per slice, and the nine taps are nine shifted row mappings of that patch: 6.4x less activation
// traffic (weights are unchanged).
//
// This is possible because the A operand never reaches the tensor core from shared memory: it is issued from registers
// (register-A wgmma), so the patch needs no MMA-legal layout -- a thread simply reads patch row (tt + dt) * 10 + (ff + df)
// for its output pixel (tt, ff) and tap (dt, df).  In the bf16 modes the patch is split into bf16 hi (| lo) ONCE per slice,
// by warps 1-3, into a converted ring whose rows the consumers load with ldmatrix for each of the nine taps; in 3xTF32 the
// consumers split the fp32 patch themselves (build_afrag).
//
// Roles (384 threads, 1 CTA / SM, persistent over tiles):
//   warp 0               TMA (fp32 patch ring, one slice ahead; weight ring of S)
//   warps 1-3            bf16 modes: patch converters (fp32 slot -> converted slot, "ready" mbarrier per slot)
//   warpgroups 1 and 2   consumers in ping-pong: each owns whole tiles (both m64 row blocks of its tiles), the two take the
//                        CTA's tiles in turn, and an ordered pair of named barriers hands the mainloop from one to the
//                        other, so that one warpgroup's epilogue runs under the other's MMAs.
#include <stdlib.h>

#include "../../include/b200asr.h"
#include "common.cuh"
#include "kernels.h"
#include "tc_common.cuh"
#include "tc_engine.cuh"

namespace b200asr {
namespace tc {

constexpr int HT = 16, HF = 8;                         // output tile: 16 time steps x 8 freq bins = 128 MMA rows
constexpr int HPT = HT + 2, HPF = HF + 2;              // input patch incl. halo
constexpr int HPROWS = HPT * HPF;                      // 180 patch rows (pixels)
constexpr int HPATCH_BYTES = HPROWS * 128;             // 23,040 B per 32-channel slice
constexpr int HPATCH_STAGE = (HPATCH_BYTES + 1023) / 1024 * 1024;
constexpr int HALO_ORDER_BAR = 2;                      // named barriers 2 / 3: "consumer warpgroup 0 / 1 may start a mainloop"

struct HaloP {
  uint16_t* out16;       // optional bf16 hi | lo pairs of the output, [2][pixels][Cout] (lo at + npix * Cout), or nullptr
  float* pool;           // optional MaxPool2d(2, 2) of the output, [B, T/2, F/2, Cout] (floor mode), or nullptr
  // optional pooling decisions next to `pool`: a nibble per pooled element, window index in ATen's scan order | 4 when the
  // maximum is not positive; byte (element / 2), low nibble = even channel, or nullptr
  uint8_t* pool_codes;
  float* out;            // the convolution's output, or nullptr (only the pooled output and its codes are wanted)
  const float* bias;
  const float* mask;
  const uint32_t* mask_bits;   // optional ReLU decisions instead of `mask`: [pixels][Cout / 32] words, bit c % 32 = (relu_out > 0)
  uint32_t* out_bits;          // optional bits of (out > 0) in the same layout, or nullptr
  int relu, B, T, F, Cin, Cout, nft, ntt, cch;
};

// MODE: 3 = 3xTF32 (fp32 weight tiles hi | lo, 128-byte rows), 6 = bf16x3 (bf16 weight tiles hi | lo, 64-byte rows, three
// bf16 MMAs per product at twice the tf32 rate), 2 = bf16 (one bf16 weight tile, one MMA).
template <int BN, int MODE> struct HaloCfg {
  static constexpr bool kBf16 = MODE != 3;
  static constexpr int kHalves = MODE == 2 ? 1 : 2;
  static constexpr int kBBytes = BN * (kBf16 ? 64 : 128);
  static constexpr int kStageBytes = kHalves * kBBytes;                         // weights hi | lo of one (tap, slice)
  // fp32 patch ring: the bf16 modes free a slot as soon as it is converted, 3xTF32 after the slice's last tap
  static constexpr int kPSlots = kBf16 ? 2 : 3;
  // converted ring (bf16 modes): a patch row is [hi 64 B | lo 64 B] + 16 B, an odd number of 16-byte chunks, so the 8
  // consecutive patch rows of an ldmatrix phase fall in 8 different bank groups for every tap shift
  static constexpr int kCSlots = kBf16 ? 3 : 0;
  static constexpr int kPitch = kHalves * 64 + 16;
  static constexpr int kCBytes = HPROWS * kPitch;
  static constexpr int kCOff = kPSlots * HPATCH_STAGE;
  static constexpr int kRingOff = (kCOff + kCSlots * kCBytes + 1023) / 1024 * 1024;
  static constexpr int kBySmem = (ENG_SMEM_CAP - 1024 - kRingOff - 256) / kStageBytes;
  static constexpr int kStages = kBySmem > 8 ? 8 : kBySmem;
  static constexpr int kBarOff = kRingOff + kStages * kStageBytes;
  static constexpr int kSmemBytes = kBarOff + 256 + 1024;
  static_assert(kStages >= 2, "stage too large");
  static_assert(16 * (kStages + kPSlots + kCSlots) <= 256, "barriers");
  static_assert(kSmemBytes <= ENG_SMEM_CAP, "shared memory");
};

__device__ __forceinline__ void ldmatrix_x4(uint32_t (&d)[4], uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(d[0]), "=r"(d[1]), "=r"(d[2]), "=r"(d[3])
               : "r"(addr)
               : "memory");
}

// fp32 patch slot (128-byte swizzled rows) -> converted slot (kPitch-byte rows of bf16 [hi | lo]), by converter warp cw: an
// item is 8 channels of one patch row, consecutive lanes take consecutive rows.  The same split_bf16_pair /
// pack_bf16_pair of the same (k, k + 1) pairs as build_afrag.
template <int MODE, int kPitch>
__device__ __forceinline__ void halo_convert(const uint8_t* src, uint8_t* dst, int cw, int lane) {
  for (int it = cw * 32 + lane; it < HPROWS * 4; it += ENG_CONVERTERS * 32) {
    const int pr = it % HPROWS, kg = it / HPROWS;
    const float4 a = *reinterpret_cast<const float4*>(src + pr * 128 + (((2 * kg) ^ (pr & 7)) << 4));
    const float4 b = *reinterpret_cast<const float4*>(src + pr * 128 + (((2 * kg + 1) ^ (pr & 7)) << 4));
    uint4 h, l;
    if constexpr (MODE == 6) {
      split_bf16_pair(a.x, a.y, h.x, l.x);
      split_bf16_pair(a.z, a.w, h.y, l.y);
      split_bf16_pair(b.x, b.y, h.z, l.z);
      split_bf16_pair(b.z, b.w, h.w, l.w);
      *reinterpret_cast<uint4*>(dst + pr * kPitch + 64 + kg * 16) = l;
    } else {
      h = make_uint4(pack_bf16_pair(a.x, a.y), pack_bf16_pair(a.z, a.w), pack_bf16_pair(b.x, b.y), pack_bf16_pair(b.z, b.w));
    }
    *reinterpret_cast<uint4*>(dst + pr * kPitch + kg * 16) = h;
  }
}

// The MMAs of one row block (m64) for one k-block, committed as one group: lo*hi, hi*lo, hi*hi per k-step, as issue_kblock.
template <int MODE, int BN>
__device__ __forceinline__ void halo_issue(float (&acc)[BN / 2], const AFrag<MODE>& f, uint32_t bhi, uint32_t blo) {
  wgmma_fence();
#pragma unroll
  for (int ks = 0; ks < AFrag<MODE>::KS; ks++) {
    if constexpr (MODE == 3) {
      wgmma_tf32<BN>(acc, f.l[ks], kmajor_desc_tf32(bhi + ks * 32));
      wgmma_tf32<BN>(acc, f.h[ks], kmajor_desc_tf32(blo + ks * 32));
      wgmma_tf32<BN>(acc, f.h[ks], kmajor_desc_tf32(bhi + ks * 32));
    } else {
      if constexpr (MODE == 6) {
        wgmma_bf16<BN>(acc, f.l[ks], kmajor_desc_bf16(bhi + ks * 32));
        wgmma_bf16<BN>(acc, f.h[ks], kmajor_desc_bf16(blo + ks * 32));
      }
      wgmma_bf16<BN>(acc, f.h[ks], kmajor_desc_bf16(bhi + ks * 32));
    }
  }
  wgmma_commit();
}

// ring cursor: advance by n positions of a ring of R slots, flipping the phase once per wrap
template <int R> __device__ __forceinline__ void ring_advance(uint32_t& slot, uint32_t& phase, uint32_t n) {
  const uint32_t t = slot + n;
  slot = t % R;
  phase ^= (t / R) & 1u;
}

template <int BN, int MODE>
__global__ void __launch_bounds__(ENG_THREADS, 1)
tc_conv3x3_halo_kernel(const __grid_constant__ CUtensorMap mapA, const __grid_constant__ CUtensorMap mapB, const HaloP p) {
  using Cfg = HaloCfg<BN, MODE>;
  constexpr int S = Cfg::kStages, PS = Cfg::kPSlots, CS = Cfg::kCSlots;
  constexpr bool kConv = Cfg::kBf16;                       // warps 1-3 convert the patch
  constexpr int RS = kConv ? CS : PS;                      // slots of the patch ring the consumers read
  constexpr int kWgWarps = 4;                              // a stage / slot is released by the warps of ONE warpgroup
  // register split (tc_engine.cuh): 3xTF32 has no converters, and its two fragment buffers of 32 registers next to 128
  // accumulators at BN = 128 need 8 more registers per consumer thread than 232
  constexpr int kProdRegs = MODE == 3 ? 24 : kProducerRegs, kConsRegs = MODE == 3 ? 240 : kConsumerRegs;
  static_assert(128 * kProdRegs + 256 * kConsRegs <= 384 * 168, "register split");
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* gen_base = smem_raw + (smem_base - smem_u32(smem_raw));
  const uint32_t bar_base = smem_base + Cfg::kBarOff;
  auto full_bar = [&](int s) { return bar_base + 8u * s; };              // weights of stage s landed
  auto empty_bar = [&](int s) { return bar_base + 8u * (S + s); };       // the MMAs of stage s completed
  auto pfull_bar = [&](int b) { return bar_base + 8u * (2 * S + b); };   // fp32 patch landed / slot free
  auto pempty_bar = [&](int b) { return bar_base + 8u * (2 * S + PS + b); };
  auto cready_bar = [&](int b) { return bar_base + 8u * (2 * S + 2 * PS + b); };   // converted patch written / slot free
  auto cempty_bar = [&](int b) { return bar_base + 8u * (2 * S + 2 * PS + CS + b); };

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int ntiles = p.nft * p.ntt * p.B;

  if (threadIdx.x == 0) {
    for (int s = 0; s < S; s++) { mbar_init(full_bar(s), 1); mbar_init(empty_bar(s), kWgWarps); }
    for (int b = 0; b < PS; b++) { mbar_init(pfull_bar(b), 1); mbar_init(pempty_bar(b), kConv ? ENG_CONVERTERS : kWgWarps); }
    for (int b = 0; b < CS; b++) { mbar_init(cready_bar(b), ENG_CONVERTERS); mbar_init(cempty_bar(b), kWgWarps); }
    fence_barrier_init();
    tma_prefetch_desc(&mapA);
    tma_prefetch_desc(&mapB);
  }
  __syncthreads();
  griddep_launch();      // programmatic dependent launch, see common.cuh
  griddep_wait();

  auto decode = [&](int tile, int& f0, int& t0, int& b) {
    f0 = (tile % p.nft) * HF;
    const int r = tile / p.nft;
    t0 = (r % p.ntt) * HT;
    b = r / p.ntt;
  };

  if (warp < 4) {
    setmaxnreg_dec<kProdRegs>();       // the whole producer warpgroup
    if (warp != 0) {
      if constexpr (kConv) {
        // ---------------------------------------------------------------- patch conversion (warps 1-3), slice order
        const int nsl = (blockIdx.x < ntiles ? (ntiles - 1 - (int)blockIdx.x) / (int)gridDim.x + 1 : 0) * p.cch;
        uint32_t ps = 0, pph = 0, cs = 0, cph = 0;
        for (int i = 0; i < nsl; i++) {
          mbar_wait(pfull_bar(ps), pph);
          mbar_wait(cempty_bar(cs), cph ^ 1);
          halo_convert<MODE, Cfg::kPitch>(gen_base + ps * HPATCH_STAGE, gen_base + Cfg::kCOff + cs * Cfg::kCBytes, warp - 1, lane);
          __syncwarp();
          if (lane == 0) { mbar_arrive(pempty_bar(ps)); mbar_arrive(cready_bar(cs)); }
          ring_advance<PS>(ps, pph, 1);
          ring_advance<CS>(cs, cph, 1);
        }
      }
      return;
    }
    // ------------------------------------------------------------------ TMA producer
    // Patches run ONE SLICE AHEAD of the weights: a patch is first-touch data from HBM while the consumers want it as soon
    // as its slice starts, so it is requested a whole slice (9 k-blocks) early.
    const bool leader = elect_one();
    uint32_t s = 0, ph = 0;
    uint32_t pslot = 0, pph = 0;                     // ring position / phase of the NEXT patch to request
    auto request_patch = [&](int tile, int sl) {
      int f0, t0, b;
      decode(tile, f0, t0, b);
      mbar_wait(pempty_bar(pslot), pph ^ 1);
      if (leader) {
        mbar_expect_tx(pfull_bar(pslot), HPATCH_BYTES);
        tma_load_4d(smem_base + pslot * HPATCH_STAGE, &mapA, pfull_bar(pslot), sl * 32, f0 - 1, t0 - 1, b);   // halo / border = zero fill
      }
      ring_advance<PS>(pslot, pph, 1);
    };
    int tile = blockIdx.x, sl = 0;
    if (tile < ntiles) request_patch(tile, 0);
    while (tile < ntiles) {
      int ntile = tile, nsl = sl + 1;
      if (nsl == p.cch) { nsl = 0; ntile = tile + gridDim.x; }
      if (ntile < ntiles) request_patch(ntile, nsl);
      for (int tap = 0; tap < 9; tap++) {
        mbar_wait(empty_bar(s), ph ^ 1);
        if (leader) {
          const uint32_t sb = smem_base + Cfg::kRingOff + s * Cfg::kStageBytes;
          mbar_expect_tx(full_bar(s), Cfg::kHalves * Cfg::kBBytes);
          tma_load_2d(sb, &mapB, full_bar(s), sl * 32, tap * BN);
          if (Cfg::kHalves == 2) tma_load_2d(sb + Cfg::kBBytes, &mapB, full_bar(s), sl * 32, (9 + tap) * BN);
        }
        __syncwarp();
        ring_advance<S>(s, ph, 1);
      }
      tile = ntile; sl = nsl;
    }
    return;
  }
  setmaxnreg_inc<kConsRegs>();

  // -------------------------------------------------------------------- consumers
  const int ctid = threadIdx.x - 128;
  const int wg = ctid >> 7, cw = (ctid >> 5) & 3;
  const int g = lane >> 2, q = lane & 3;
  const int nkb = p.cch * 9;                           // k-block = (slice, tap), taps fastest
  // A rows of this thread in row block mb (tile rows mb * 64 + cw * 16 + g and + 8 = output pixels (row / 8, row % 8)):
  // patch row for tap (0, 0) = prow + mb * 8 * HPF (and + HPF for the second row)
  const int prow = cw * 2 * HPF + g;
  // ldmatrix (bf16 modes): lane -> row (lane & 7) of matrix lane / 8 = (rows + 8 if odd, k + 8 if >= 2) of the warp's 16 x 16
  const int lm_row = (cw * 2 + ((lane >> 3) & 1)) * HPF + (lane & 7);
  const uint32_t lm_k = (lane >> 4) * 16;
  float dummy0 = 0.f, dummy1 = 0.f;
  uint32_t s = 0, ph = 0;                              // weight ring: next k-block, its phase
  uint32_t cs = 0, cph = 0;                            // patch ring the consumers read (converted / fp32): the same
  auto skip_tile = [&]() {                             // the other warpgroup's tile
    ring_advance<S>(s, ph, nkb);
    ring_advance<RS>(cs, cph, p.cch);
  };
  if (wg == 1) skip_tile();
  for (int tile = blockIdx.x + wg * gridDim.x; tile < ntiles; tile += 2 * gridDim.x) {
    float acc[2][BN / 2];
#pragma unroll
    for (int mb = 0; mb < 2; mb++)
#pragma unroll
      for (int i = 0; i < BN / 2; i++) acc[mb][i] = 0.f;
    // mainloop in tile order: wait until the other warpgroup has waited for the last data of the previous tile (a ring
    // position is reused every S k-blocks, so a waiter that ran ahead by more than one phase would pass on a stale parity)
    if (tile != (int)blockIdx.x) named_bar_sync(HALO_ORDER_BAR + wg, 2 * 128);

    // Pipeline unit = (k-block, row block); the fragments of unit u + 1 are built while u's MMAs run (fragment buffer =
    // row block), and a k-block's stage is released once the MMAs of both its row blocks have completed.
    AFrag<MODE> f[2];
    uint32_t sb = 0, pbase = 0;
    int shift = 0, tap = 0;
    auto build = [&](auto mb_) {
      constexpr int mb = decltype(mb_)::value;
      if constexpr (kConv) {
        const uint32_t a = pbase + (lm_row + mb * 8 * HPF + shift) * Cfg::kPitch + lm_k;
#pragma unroll
        for (int ks = 0; ks < 2; ks++) {
          ldmatrix_x4(f[mb].h[ks], a + ks * 32);
          if constexpr (MODE == 6) ldmatrix_x4(f[mb].l[ks], a + 64 + ks * 32);
        }
      } else {
        const uint8_t* patch = gen_base + (pbase - smem_base);
        const int pr0 = prow + mb * 8 * HPF + shift, pr1 = pr0 + HPF;
        const int r0 = mb * 64 + cw * 16 + g;
        // A element (pixel row r, channel k): patch row pr, 128B swizzle of the TMA box
        build_afrag<MODE, true, false>(
            f[mb],
            [&](int r, int k) {
              const int pr = r == r0 ? pr0 : pr1;
              return reinterpret_cast<const float*>(patch + pr * 128 + (((k >> 2) ^ (pr & 7)) << 4) + (k & 3) * 4);
            },
            r0, r0 + 8, q, dummy0, dummy1);
      }
    };
    auto prep = [&]() {                                // the next k-block's data, and its row block 0 fragments
      if (tap == 0) mbar_wait(kConv ? cready_bar(cs) : pfull_bar(cs), cph);
      mbar_wait(full_bar(s), ph);
      sb = smem_base + Cfg::kRingOff + s * Cfg::kStageBytes;
      pbase = smem_base + (kConv ? Cfg::kCOff + cs * Cfg::kCBytes : cs * HPATCH_STAGE);
      shift = (tap % 3) * HPF + tap / 3;               // tap = 3 * (df + 1) + (dt + 1)
      ring_advance<S>(s, ph, 1);
      if (++tap == 9) { tap = 0; ring_advance<RS>(cs, cph, 1); }
      build(std::integral_constant<int, 0>());
    };
    // the MMAs of the k-block `lag` positions behind the weight cursor have completed; last_tap: it is its slice's last tap,
    // so this warp has read the slice's patch (one position behind the patch cursor) for the last time
    auto release = [&](uint32_t lag, bool last_tap) {
      __syncwarp();
      if (lane == 0) mbar_arrive(empty_bar((s + S - lag) % S));
      if (last_tap && lane == 0) mbar_arrive(kConv ? cempty_bar((cs + RS - 1) % RS) : pempty_bar((cs + RS - 1) % RS));
    };
    prep();
    for (int kb = 0; kb < nkb; kb++) {
      halo_issue<MODE, BN>(acc[0], f[0], sb, sb + Cfg::kBBytes);
      if (kb > 0) {
        wgmma_wait<1>();                               // (kb - 1, row block 1) done: k-block kb - 1 and buffer 1 are free
        keep_live(f[1]);
        release(2, tap == 1);                          // the cursors have passed k-block kb as well
      }
      build(std::integral_constant<int, 1>());
      halo_issue<MODE, BN>(acc[1], f[1], sb, sb + Cfg::kBBytes);
      wgmma_wait<1>();                                 // (kb, row block 0) done: buffer 0 is free
      keep_live(f[0]);
      if (kb + 1 < nkb) prep();
    }
    // every wait of this tile is behind us: the other warpgroup may start its mainloop (if it has a next tile)
    if (tile + (int)gridDim.x < ntiles) named_bar_arrive(HALO_ORDER_BAR + (wg ^ 1), 2 * 128);
    wgmma_wait<0>();
    keep_live(f[0]);
    keep_live(f[1]);
    acc_fence(acc[0]);
    acc_fence(acc[1]);
    release(1, true);

    // ---- epilogue straight from the accumulator layout: bias, ReLU, mask, optional bf16 pairs and fused 2 x 2 max-pool.
    // In row block mb this thread holds time steps tt / tt + 1 (rows r0 / r0 + 8) of freq bin ff, columns 8 j + 2 q, + 1;
    // bin ff + 1 is in lane + 4, so a 2 x 2 window is one register pair here and one in lane ^ 4 (the even-g lane stores).
    // A 32-channel word of the ReLU bits is j = 4 w .. 4 w + 3 of the four lanes of a quad (q = 0..3): bit 8 (j % 4) + 2 q, + 1.
    int f0, t0, b;
    decode(tile, f0, t0, b);
    const int ff = f0 + g;
    const size_t lo_off = (size_t)p.B * p.T * p.F * p.Cout;
    const int wpp = p.Cout >> 5;                         // bit words per pixel
#pragma unroll
    for (int mb = 0; mb < 2; mb++) {
      const int tt = t0 + mb * 8 + cw * 2;
      const bool valid[2] = {tt < p.T && ff < p.F, tt + 1 < p.T && ff < p.F};
      const size_t pix = ((size_t)b * p.T + tt) * p.F + ff;
      const bool pool_st = p.pool && (g & 1) == 0 && tt + 1 < p.T && ff + 1 < p.F;
      float* prow_out = pool_st ? p.pool + (((size_t)b * (p.T >> 1) + (tt >> 1)) * (p.F >> 1) + (ff >> 1)) * p.Cout : nullptr;
      uint32_t mw[2] = {0u, 0u}, ob[2] = {0u, 0u};     // mask word in use / output bits gathered, per time row
#pragma unroll
      for (int j = 0; j < BN / 8; j++) {
        const int col = j * 8 + 2 * q, sh = col & 31;
        const float2 bb = p.bias ? __ldg(reinterpret_cast<const float2*>(p.bias + col)) : make_float2(0.f, 0.f);
        if (p.mask_bits && (j & 3) == 0) {
#pragma unroll
          for (int h = 0; h < 2; h++) mw[h] = valid[h] ? __ldg(p.mask_bits + (pix + (size_t)h * p.F) * wpp + (j >> 2)) : 0u;
        }
        float2 o[2];
#pragma unroll
        for (int h = 0; h < 2; h++) {
          const size_t off = (pix + (size_t)h * p.F) * p.Cout + col;
          const float2 mm = (p.mask && valid[h]) ? __ldg(reinterpret_cast<const float2*>(p.mask + off)) : make_float2(1.f, 1.f);
          o[h] = make_float2(acc[mb][4 * j + 2 * h] + bb.x, acc[mb][4 * j + 2 * h + 1] + bb.y);
          if (p.relu) { o[h].x = fmaxf(o[h].x, 0.f); o[h].y = fmaxf(o[h].y, 0.f); }
          o[h].x = mm.x > 0.f ? o[h].x : 0.f;
          o[h].y = mm.y > 0.f ? o[h].y : 0.f;
          if (p.mask_bits) {
            o[h].x = (mw[h] >> sh) & 1u ? o[h].x : 0.f;
            o[h].y = (mw[h] >> (sh + 1)) & 1u ? o[h].y : 0.f;
          }
          if (p.out_bits) ob[h] |= (o[h].x > 0.f ? 1u << sh : 0u) | (o[h].y > 0.f ? 2u << sh : 0u);
          if (p.out && valid[h]) *reinterpret_cast<float2*>(p.out + off) = o[h];
          if (p.out16 && valid[h]) {   // the same values as bf16 pairs: the weight-gradient kernel's B operand (WgradPairPolicy)
            uint32_t hi, lo;
            split_bf16_pair(o[h].x, o[h].y, hi, lo);
            *reinterpret_cast<uint32_t*>(p.out16 + off) = hi;
            *reinterpret_cast<uint32_t*>(p.out16 + lo_off + off) = lo;
          }
        }
        if (p.pool) {                  // every lane takes part in the shuffles
          const float lx = fmaxf(o[0].x, o[1].x), ly = fmaxf(o[0].y, o[1].y);
          const float rx = __shfl_xor_sync(0xffffffffu, lx, 4), ry = __shfl_xor_sync(0xffffffffu, ly, 4);
          const float mx = fmaxf(lx, rx), my = fmaxf(ly, ry);
          if (pool_st) *reinterpret_cast<float2*>(prow_out + col) = make_float2(mx, my);
          if (p.pool_codes) {
            // window positions in ATen's scan order: this lane's (ff, tt) / (ff, tt + 1) = 0 / 1, lane ^ 4's bin ff + 1 = 2 / 3.
            // The first maximum of each pair, then the later pair only if strictly larger: the same position as the
            // sequential scan of maxpool2x2_bwd for every non-NaN window (post-ReLU values are never NaN)
            const uint32_t sel = (o[1].x > o[0].x ? 1u : 0u) | (o[1].y > o[0].y ? 2u : 0u);
            const uint32_t rsel = __shfl_xor_sync(0xffffffffu, sel, 4);
            const uint32_t cx = (rx > lx ? 2u | (rsel & 1u) : (sel & 1u)) | (mx > 0.f ? 0u : 4u);
            const uint32_t cy = (ry > ly ? 2u | (rsel >> 1) : (sel >> 1)) | (my > 0.f ? 0u : 4u);
            if (pool_st) p.pool_codes[(prow_out - p.pool + col) >> 1] = (uint8_t)(cx | (cy << 4));
          }
        }
        if (p.out_bits && (j & 3) == 3) {   // the quad's word is complete: OR it over the quad, lane q = h stores row h
#pragma unroll
          for (int h = 0; h < 2; h++) {
            ob[h] |= __shfl_xor_sync(0xffffffffu, ob[h], 1);
            ob[h] |= __shfl_xor_sync(0xffffffffu, ob[h], 2);
            if (q == h && valid[h]) p.out_bits[(pix + (size_t)h * p.F) * wpp + (j >> 2)] = ob[h];
            ob[h] = 0u;
          }
        }
      }
    }
    skip_tile();
  }
}

template <int BN, int MODE>
static int launch_halo(const CUtensorMap& ma, const CUtensorMap& mb, const HaloP& p, cudaStream_t st) {
  using Cfg = HaloCfg<BN, MODE>;
  auto* kern = tc_conv3x3_halo_kernel<BN, MODE>;
  static bool attr_set[kMaxDevices] = {};
  if (int rc = ensure_dynamic_smem((const void*)kern, Cfg::kSmemBytes, attr_set, "tc_conv3x3_halo")) return rc;
  const long long tiles = (long long)p.nft * p.ntt * p.B;
  if (tiles <= 0) return B200ASR_OK;
  if (tiles >= (1LL << 30)) { set_error("tc_conv3x3_halo: too many tiles"); return B200ASR_BAD_SHAPE; }   // tile + 2 * grid fits an int
  const int grid = (int)min(tiles, (long long)device_sm_count());
  launch_pdl(kern, dim3(grid), dim3(ENG_THREADS), Cfg::kSmemBytes, st, ma, mb, p);
  return check_launch("tc_conv3x3_halo");
}

}  // namespace tc

// wk: mode 3: [2][9][Cout][Cin] fp32 pre-split K-major weights (hi | lo), as for conv3x3_tc with precision 3;
//     mode 6 / 2: [2 or 1][9][Cout][Cin] bf16 (conv_repack_k_bf16_kernel)
int conv3x3_tc_halo(const float* in, const void* wk, const float* bias, const float* mask, float* out, int B, int T, int F,
                    int Cin, int Cout, int relu, int mode, cudaStream_t st, void* out16, float* pool,
                    const uint32_t* mask_bits, uint32_t* out_bits, uint8_t* pool_codes) {
  using namespace tc;
  B200_REQUIRE(mode == 3 || mode == 6 || mode == 2, B200ASR_BAD_ARG, "conv3x3_tc_halo: mode must be 3 (3xTF32), 6 (bf16x3) or 2 (bf16)");
  B200_REQUIRE(Cin % 32 == 0 && (Cout == 64 || Cout == 128), B200ASR_BAD_SHAPE,
               "conv3x3_tc_halo: needs Cin %% 32 == 0 and Cout in {64,128} (Cin=%d Cout=%d)", Cin, Cout);
  B200_REQUIRE((out || pool) && (!pool_codes || pool), B200ASR_BAD_ARG, "conv3x3_tc_halo: nothing to write");
  B200_REQUIRE(aligned16(in) && aligned16(wk) && aligned16(out) && (!bias || aligned16(bias)) && (!mask || aligned16(mask)),
               B200ASR_BAD_ALIGN, "conv3x3_tc_halo: pointers must be 16-byte aligned");
  B200_REQUIRE(!(mask && mask_bits), B200ASR_BAD_ARG, "conv3x3_tc_halo: pass the ReLU mask as floats or as bits, not both");
  CUtensorMap ma, mb;
  {
    uint64_t dims[4] = {(uint64_t)Cin, (uint64_t)F, (uint64_t)T, (uint64_t)B};
    uint64_t strides[3] = {(uint64_t)Cin, (uint64_t)F * Cin, (uint64_t)T * F * Cin};
    uint32_t box[4] = {32, HPF, HPT, 1};
    int rc = make_tensor_map_f32(&ma, in, 4, dims, strides, box, false);
    if (rc) return rc;
  }
  {
    uint64_t dims[2] = {(uint64_t)Cin, (uint64_t)(mode == 2 ? 9 : 18) * Cout};
    uint64_t strides[1] = {(uint64_t)Cin};
    uint32_t box[2] = {32, (uint32_t)Cout};
    int rc = mode == 3 ? make_tensor_map_f32(&mb, wk, 2, dims, strides, box, false) : make_tensor_map_bf16(&mb, wk, 2, dims, strides, box);
    if (rc) return rc;
  }
  HaloP p{(uint16_t*)out16, pool, pool_codes, out, bias, mask, mask_bits, out_bits, relu, B, T, F, Cin, Cout, ceil_div(F, HF), ceil_div(T, HT), Cin / 32};
  if (mode == 3) return Cout == 64 ? launch_halo<64, 3>(ma, mb, p, st) : launch_halo<128, 3>(ma, mb, p, st);
  if (mode == 6) return Cout == 64 ? launch_halo<64, 6>(ma, mb, p, st) : launch_halo<128, 6>(ma, mb, p, st);
  return Cout == 64 ? launch_halo<64, 2>(ma, mb, p, st) : launch_halo<128, 2>(ma, mb, p, st);
}

}  // namespace b200asr
