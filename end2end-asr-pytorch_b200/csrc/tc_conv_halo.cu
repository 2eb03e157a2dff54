// 3x3 convolution (forward / data gradient), "halo" variant of the persistent wgmma kernel: 3xTF32, bf16x3 or bf16.
//
// Why: the tap-shifted implicit GEMM (tc_conv.cu) fetches the activation tile nine times per 32-channel slice (once per tap,
// 16 KB each).  Here the 16 x 8 output tile's input patch INCLUDING its one-pixel halo -- 18 x 10 pixels x 32 channels =
// 22.5 KB -- is fetched ONCE per slice, and the nine taps are nine shifted row mappings of that patch: 6.4x less activation
// traffic (weights are unchanged).
//
// This is possible because the A operand never reaches the tensor core from shared memory: the consumer threads read the
// fp32 patch, round / split it in registers and issue register-A wgmma (tc_engine.cuh, mma_kblock).  So the patch needs no
// MMA-legal layout -- a thread simply reads patch row (tt + dt) * 10 + (ff + df) for its output pixel (tt, ff) and tap (dt, df).
//
// Roles (384 threads, 1 CTA / SM, persistent over tiles): warp 0 TMA (patch ring of 3, one slice ahead; weight ring of S),
// warpgroups 1 and 2 consumers (output pixels 0-63 / 64-127 of the tile: MMAs, then the epilogue).
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
constexpr int HPATCH_BYTES = HPT * HPF * 128;          // 23,040 B per 32-channel slice
constexpr int HPATCH_STAGE = (HPATCH_BYTES + 1023) / 1024 * 1024;
constexpr int HPATCH_SLOTS = 3;                        // the patch of slice i+1 is requested before the weights of slice i

struct HaloP {
  uint16_t* out16;       // optional bf16 hi | lo pairs of the output, [2][pixels][Cout] (lo at + npix * Cout), or nullptr
  float* pool;           // optional MaxPool2d(2, 2) of the output, [B, T/2, F/2, Cout] (floor mode), or nullptr
  float* out;
  const float* bias;
  const float* mask;
  int relu, B, T, F, Cin, Cout, nft, ntt, cch;
};

// MODE: 3 = 3xTF32 (fp32 weight tiles hi | lo, 128-byte rows), 6 = bf16x3 (bf16 weight tiles hi | lo, 64-byte rows, three
// bf16 MMAs per product at twice the tf32 rate), 2 = bf16 (one bf16 weight tile, one MMA).
template <int BN, int MODE> struct HaloCfg {
  static constexpr bool kBf16 = MODE != 3;
  static constexpr int kHalves = MODE == 2 ? 1 : 2;
  static constexpr int kBBytes = BN * (kBf16 ? 64 : 128);
  static constexpr int kStageBytes = kHalves * kBBytes;                         // weights hi | lo of one (tap, slice)
  static constexpr int kRingOff = HPATCH_SLOTS * HPATCH_STAGE;
  static constexpr int kBySmem = (ENG_SMEM_CAP - 1024 - kRingOff - epilogue_bytes(BN) - 256) / kStageBytes;
  static constexpr int kStages = kBySmem > 8 ? 8 : kBySmem;
  static constexpr int kOffEpi = kRingOff + kStages * kStageBytes;
  static constexpr int kBarOff = kOffEpi + epilogue_bytes(BN);
  static constexpr int kSmemBytes = kBarOff + 256 + 1024;
  static_assert(kStages >= 2, "stage too large");
  static_assert(kSmemBytes <= ENG_SMEM_CAP, "shared memory");
};

template <int BN, int MODE>
__global__ void __launch_bounds__(ENG_THREADS, 1)
tc_conv3x3_halo_kernel(const __grid_constant__ CUtensorMap mapA, const __grid_constant__ CUtensorMap mapB, const HaloP p) {
  using Cfg = HaloCfg<BN, MODE>;
  constexpr int S = Cfg::kStages;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* gen_base = smem_raw + (smem_base - smem_u32(smem_raw));
  const uint32_t bar_base = smem_base + Cfg::kBarOff;
  auto full_bar = [&](int s) { return bar_base + 8u * s; };              // weights of stage s landed
  auto empty_bar = [&](int s) { return bar_base + 8u * (S + s); };       // the MMAs of stage s completed
  auto pfull_bar = [&](int b) { return bar_base + 8u * (2 * S + b); };
  auto pempty_bar = [&](int b) { return bar_base + 8u * (2 * S + HPATCH_SLOTS + b); };

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int ntiles = p.nft * p.ntt * p.B;

  if (threadIdx.x == 0) {
    for (int s = 0; s < S; s++) { mbar_init(full_bar(s), 1); mbar_init(empty_bar(s), ENG_CONSUMERS / 32); }
    for (int b = 0; b < HPATCH_SLOTS; b++) { mbar_init(pfull_bar(b), 1); mbar_init(pempty_bar(b), ENG_CONSUMERS / 32); }
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

  if (warp == 0) {
    // ------------------------------------------------------------------ TMA producer
    // Patches run ONE SLICE AHEAD of the weights: a patch is first-touch data from HBM while the consumers want it as soon
    // as its slice starts, so it is requested a whole slice (9 k-blocks) early into a ring of three.
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
      if (++pslot == HPATCH_SLOTS) { pslot = 0; pph ^= 1; }
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
        if (++s == S) { s = 0; ph ^= 1; }
      }
      tile = ntile; sl = nsl;
    }
    return;
  }
  if (warp < 4) return;

  // -------------------------------------------------------------------- consumers
  const int ctid = threadIdx.x - 128;
  const int wg = ctid >> 7, cw = (ctid >> 5) & 3;
  const int g = lane >> 2, q = lane & 3;
  const int r0 = wg * 64 + cw * 16 + g, r1 = r0 + 8;             // output pixels (row / 8, row % 8) of the tile
  const int prow0 = (r0 >> 3) * HPF + (r0 & 7), prow1 = (r1 >> 3) * HPF + (r1 & 7);   // their patch rows for tap (0, 0)
  float* epi = reinterpret_cast<float*>(gen_base + Cfg::kOffEpi);
  float dummy0 = 0.f, dummy1 = 0.f;
  uint32_t s = 0, ph = 0, ps = 0, pph = 0;
  for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; i++) acc[i] = 0.f;
    for (int sl = 0; sl < p.cch; sl++) {
      const uint8_t* patch = gen_base + ps * HPATCH_STAGE;
      mbar_wait(pfull_bar(ps), pph);
      for (int tap = 0; tap < 9; tap++) {
        mbar_wait(full_bar(s), ph);
        const int shift = (tap % 3) * HPF + tap / 3;                // tap = 3 * (df + 1) + (dt + 1)
        const int pr0 = prow0 + shift, pr1 = prow1 + shift;
        const uint32_t sb = smem_base + Cfg::kRingOff + s * Cfg::kStageBytes;
        // A element (pixel row r, channel k): patch row pr, 128B swizzle of the TMA box
        mma_kblock<MODE, BN, true, false>(
            acc,
            [&](int r, int k) {
              const int pr = r == r0 ? pr0 : pr1;
              return reinterpret_cast<const float*>(patch + pr * 128 + (((k >> 2) ^ (pr & 7)) << 4) + (k & 3) * 4);
            },
            r0, r1, q, sb, sb + Cfg::kBBytes, dummy0, dummy1);
        __syncwarp();
        if (lane == 0) mbar_arrive(empty_bar(s));
        if (++s == S) { s = 0; ph ^= 1; }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(pempty_bar(ps));      // this warp has read the patch for the last time
      if (++ps == HPATCH_SLOTS) { ps = 0; pph ^= 1; }
    }

    // ---- epilogue: bias, ReLU, mask, optional bf16 pairs and fused 2 x 2 max-pool; a warp covers 4 time rows x 8 freq bins
    int f0, t0, b;
    decode(tile, f0, t0, b);
    epilogue_rows<BN>(acc, epi, ctid, r0, r1, q, [&](int r, int c0, const float (&v)[32]) {
      const int tt = t0 + (r >> 3), ff = f0 + (r & 7);
      const bool valid = tt < p.T && ff < p.F;
      if (!valid && !p.pool) return;                  // (with pooling every lane takes part in the shuffles below)
      const size_t pix = ((size_t)b * p.T + tt) * p.F + ff;
      float* orow = p.out + pix * p.Cout;
      uint16_t* orow16 = p.out16 ? p.out16 + pix * p.Cout : nullptr;
      const size_t lo_off = (size_t)p.B * p.T * p.F * p.Cout;
      const float* mrow = p.mask ? p.mask + pix * p.Cout : nullptr;
#pragma unroll
      for (int half = 0; half < 2; half++) {     // all loads of a 16-channel half before its first store
        float4 bb[4], mm[4];
#pragma unroll
        for (int qq = 0; qq < 4; qq++) {
          const int col = c0 + half * 16 + qq * 4;
          bb[qq] = (p.bias && valid) ? __ldg(reinterpret_cast<const float4*>(p.bias + col)) : make_float4(0.f, 0.f, 0.f, 0.f);
          mm[qq] = (mrow && valid) ? __ldg(reinterpret_cast<const float4*>(mrow + col)) : make_float4(1.f, 1.f, 1.f, 1.f);
        }
#pragma unroll
        for (int qq = 0; qq < 4; qq++) {
          const int col = c0 + half * 16 + qq * 4, j = half * 16 + qq * 4;
          float o[4] = {v[j] + bb[qq].x, v[j + 1] + bb[qq].y, v[j + 2] + bb[qq].z, v[j + 3] + bb[qq].w};
          if (p.relu) { o[0] = fmaxf(o[0], 0.f); o[1] = fmaxf(o[1], 0.f); o[2] = fmaxf(o[2], 0.f); o[3] = fmaxf(o[3], 0.f); }
          o[0] = mm[qq].x > 0.f ? o[0] : 0.f; o[1] = mm[qq].y > 0.f ? o[1] : 0.f;
          o[2] = mm[qq].z > 0.f ? o[2] : 0.f; o[3] = mm[qq].w > 0.f ? o[3] : 0.f;
          if (valid) *reinterpret_cast<float4*>(orow + col) = make_float4(o[0], o[1], o[2], o[3]);
          if (orow16 && valid) {       // the same values as bf16 pairs: the weight-gradient kernel's B operand (WgradPairPolicy)
            uint2 h, l;
            split_bf16_pair(o[0], o[1], h.x, l.x);
            split_bf16_pair(o[2], o[3], h.y, l.y);
            *reinterpret_cast<uint2*>(orow16 + col) = h;
            *reinterpret_cast<uint2*>(orow16 + lo_off + col) = l;
          }
          if (p.pool) {
            // fused MaxPool2d(2, 2): a warp holds 4 time rows x 8 freq bins of the tile (lane = 8 * row + bin, tile origin
            // even in both), so the 2 x 2 window of lane l is {l, l ^ 1, l ^ 8, l ^ 9}; the even / even lane stores it
#pragma unroll
            for (int e = 0; e < 4; e++) {
              o[e] = fmaxf(o[e], __shfl_xor_sync(0xffffffffu, o[e], 1));
              o[e] = fmaxf(o[e], __shfl_xor_sync(0xffffffffu, o[e], 8));
            }
            if ((lane & 9) == 0 && tt + 1 < p.T && ff + 1 < p.F)
              *reinterpret_cast<float4*>(p.pool + ((((size_t)b * (p.T >> 1) + (tt >> 1)) * (p.F >> 1) + (ff >> 1)) * p.Cout + col)) =
                  make_float4(o[0], o[1], o[2], o[3]);
          }
        }
      }
    });
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
  if (tiles >= (1LL << 31)) { set_error("tc_conv3x3_halo: too many tiles"); return B200ASR_BAD_SHAPE; }
  const int grid = (int)min(tiles, (long long)device_sm_count());
  launch_pdl(kern, dim3(grid), dim3(ENG_THREADS), Cfg::kSmemBytes, st, ma, mb, p);
  return check_launch("tc_conv3x3_halo");
}

}  // namespace tc

// wk: mode 3: [2][9][Cout][Cin] fp32 pre-split K-major weights (hi | lo), as for conv3x3_tc with precision 3;
//     mode 6 / 2: [2 or 1][9][Cout][Cin] bf16 (conv_repack_k_bf16_kernel)
int conv3x3_tc_halo(const float* in, const void* wk, const float* bias, const float* mask, float* out, int B, int T, int F,
                    int Cin, int Cout, int relu, int mode, cudaStream_t st, void* out16, float* pool) {
  using namespace tc;
  B200_REQUIRE(mode == 3 || mode == 6 || mode == 2, B200ASR_BAD_ARG, "conv3x3_tc_halo: mode must be 3 (3xTF32), 6 (bf16x3) or 2 (bf16)");
  B200_REQUIRE(Cin % 32 == 0 && (Cout == 64 || Cout == 128), B200ASR_BAD_SHAPE,
               "conv3x3_tc_halo: needs Cin %% 32 == 0 and Cout in {64,128} (Cin=%d Cout=%d)", Cin, Cout);
  B200_REQUIRE(aligned16(in) && aligned16(wk) && aligned16(out) && (!bias || aligned16(bias)) && (!mask || aligned16(mask)),
               B200ASR_BAD_ALIGN, "conv3x3_tc_halo: pointers must be 16-byte aligned");
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
  HaloP p{(uint16_t*)out16, pool, out, bias, mask, relu, B, T, F, Cin, Cout, ceil_div(F, HF), ceil_div(T, HT), Cin / 32};
  if (mode == 3) return Cout == 64 ? launch_halo<64, 3>(ma, mb, p, st) : launch_halo<128, 3>(ma, mb, p, st);
  if (mode == 6) return Cout == 64 ? launch_halo<64, 6>(ma, mb, p, st) : launch_halo<128, 6>(ma, mb, p, st);
  return Cout == 64 ? launch_halo<64, 2>(ma, mb, p, st) : launch_halo<128, 2>(ma, mb, p, st);
}

}  // namespace b200asr
