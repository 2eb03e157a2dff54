// Tensor-core implicit-GEMM 3x3 convolution on channels-last [B,T,F,C] activations: forward / data gradient and weight
// gradient, as policies of the persistent tile engine (tc_engine.cuh).
//
// Forward / data gradient (TF32; the 3xTF32 and bf16 modes run on the halo kernel, tc_conv_halo.cu):
//   out[p][n] = act( sum_{tap} sum_c in[p + off(tap)][c] * wk[tap][n][c] + bias[n] ) (.* mask > 0)
//
// One tile = an 8 (time) x 16 (freq) patch = 128 output pixels x BN output channels.  The A operand of k-block
// (tap, 32-channel slice) is ONE 4-D TMA box {32 ch, 16 freq, 8 time, 1 utt} fetched at the tap-shifted coordinate:
// the zero padding of the convolution is TMA's out-of-bounds fill, so there is no im2col buffer and no halo logic.
// The box lands in shared memory as 128 rows x 128 B (K-major, 128B swizzle).
// The B operand is the repacked weight wk[tap][n][c] (K-major, one 2-D box).
//
// Weight gradient (bf16 modes; tf32 / 3xTF32 run on the halo weight-gradient kernel, tc_conv_wgrad.cu):
//   dwr[tap][ci][co] += sum_p x[p + off(tap)][ci] * dy[p][co]
// GEMM with the PIXEL axis as the contraction: both operands are MN-major (channels contiguous, pixels strided), i.e.
// exactly the channels-last activations as they lie in HBM -- no transpose.  One k-block = a 2 (time) x 16 (freq) patch
// of 32 pixels; the A tile is four 32-channel chunks {32 ch, 16, 2, 1} fetched at the tap-shifted coordinate (zero fill
// = padding), the B tile Co/32 chunks of dy at the unshifted coordinate.  M = 128 rows: one tap when Cin = 128, a PAIR of
// taps when Cin = 64 (rows 0-63 tap a, 64-127 tap b; they share the dy tile).  Each tile reduces a contiguous range of
// pixel blocks (its split) and writes its 128 x Co partial to the split's slot; reduce_parts sums the splits in order.  The
// bias gradient (column sums of dy over all pixels) is taken by the tap-group-0 tiles while the dy tile is in shared memory,
// instead of a separate pass that re-reads dy from HBM, and summed over the splits the same way.
#include "../../include/b200asr.h"
#include "common.cuh"
#include "kernels.h"
#include "tc_common.cuh"
#include "tc_engine.cuh"

namespace b200asr {
namespace tc {

constexpr int CT_T = 8, CT_F = 16;                    // forward pixel patch: 8 x 16 = 128 rows of the MMA
constexpr int A_TILE = 128 * 128;                     // bytes per A k-block
constexpr int WG_PF = 16, WG_PT = 2;                  // weight-gradient pixel patch of one k-block (32 pixels)

struct ConvEpi {
  float* out;
  const float* bias;
  const float* mask;
  const uint32_t* mask_bits;   // see conv3x3_tc in kernels.h
  uint32_t* out_bits;
  int relu, B, T, F, Cin, Cout;
};

struct WgP {
  float* part;         // [splits][9][Ci][Co] partial weight gradients
  float* bpart;        // [splits][Co] partial bias gradients, or nullptr
  int B, T, F, Ci, Co, nft, ntt, blocks_per_cta, total_blocks;
};

template <int BN_>
struct ConvPolicy {
  static constexpr int BN = BN_, kABytes = A_TILE, kBBytes = BN_ * 128;
  static constexpr bool kSplitA = true, kSplitB = false, kAMN = false, kBMN = false;     // weights arrive K-major
  static constexpr bool kSumA = false, kSumB = false;
  struct Params { ConvEpi e; int nft, ntt, cch; };
  static __device__ __forceinline__ int num_tiles(const Params& p) { return p.nft * p.ntt * p.e.B; }
  static __device__ __forceinline__ int num_kb(const Params& p, int) { return 9 * p.cch; }
  struct Tile { int f0, t0, b, tap, df, dt, cb; };      // tile origin + k cursor (tap, 32-channel block)
  static __device__ __forceinline__ Tile tile(const Params& p, int tile) {
    Tile t;
    t.f0 = (tile % p.nft) * CT_F;
    const int r = tile / p.nft;
    t.t0 = (r % p.ntt) * CT_T;
    t.b = r / p.ntt;
    t.tap = 0; t.df = -1; t.dt = -1; t.cb = 0;
    return t;
  }
  // k order: tap-major (tap = 3 * (df + 1) + (dt + 1)), 32-channel blocks inside a tap
  static __device__ __forceinline__ void load(const Params& p, Tile& t, const CUtensorMap* mapA, const CUtensorMap* mapB,
                                              uint32_t sa, uint32_t sb, uint32_t, uint32_t bar, bool leader) {
    const int c0 = t.cb * 32;
    if (leader) {
      tma_load_4d(sa, mapA, bar, c0, t.f0 + t.df, t.t0 + t.dt, t.b);
      tma_load_2d(sb, mapB, bar, c0, t.tap * BN);
    }
    if (++t.cb == p.cch) {
      t.cb = 0; t.tap++;
      if (++t.dt == 2) { t.dt = -1; t.df++; }
    }
  }
  static __device__ __forceinline__ void store(const Params& p, const Tile& t, int r, int c0, const float (&v)[32]) {
    const ConvEpi& e = p.e;
    const int tt = t.t0 + r / CT_F, ff = t.f0 + r % CT_F;
    if (tt >= e.T || ff >= e.F) return;
    const size_t pix = ((size_t)t.b * e.T + tt) * e.F + ff;
    float* orow = e.out + pix * e.Cout;
    const float* mrow = e.mask ? e.mask + pix * e.Cout : nullptr;
    // c0 is a multiple of 32: the piece is exactly one word of the ReLU bits
    const size_t word = pix * (e.Cout >> 5) + (c0 >> 5);
    const uint32_t mbits = e.mask_bits ? __ldg(e.mask_bits + word) : ~0u;
    uint32_t obits = 0u;
    // all loads of a 16-channel half before its first store (see GemmPolicy::store)
#pragma unroll
    for (int half = 0; half < 2; half++) {
      float4 bb[4], mm[4];
#pragma unroll
      for (int q = 0; q < 4; q++) {
        const int col = c0 + half * 16 + q * 4;
        bb[q] = e.bias ? __ldg(reinterpret_cast<const float4*>(e.bias + col)) : make_float4(0.f, 0.f, 0.f, 0.f);
        mm[q] = mrow ? __ldg(reinterpret_cast<const float4*>(mrow + col)) : make_float4(1.f, 1.f, 1.f, 1.f);
      }
#pragma unroll
      for (int q = 0; q < 4; q++) {
        const int col = c0 + half * 16 + q * 4, j = half * 16 + q * 4;
        float o[4] = {v[j] + bb[q].x, v[j + 1] + bb[q].y, v[j + 2] + bb[q].z, v[j + 3] + bb[q].w};
        if (e.relu) { o[0] = fmaxf(o[0], 0.f); o[1] = fmaxf(o[1], 0.f); o[2] = fmaxf(o[2], 0.f); o[3] = fmaxf(o[3], 0.f); }
        o[0] = mm[q].x > 0.f ? o[0] : 0.f; o[1] = mm[q].y > 0.f ? o[1] : 0.f;
        o[2] = mm[q].z > 0.f ? o[2] : 0.f; o[3] = mm[q].w > 0.f ? o[3] : 0.f;
        if (e.mask_bits) {
#pragma unroll
          for (int k = 0; k < 4; k++) o[k] = (mbits >> (j + k)) & 1u ? o[k] : 0.f;
        }
        if (e.out_bits) {
#pragma unroll
          for (int k = 0; k < 4; k++) obits |= o[k] > 0.f ? 1u << (j + k) : 0u;
        }
        *reinterpret_cast<float4*>(orow + col) = make_float4(o[0], o[1], o[2], o[3]);
      }
    }
    if (e.out_bits) e.out_bits[word] = obits;
  }
};

template <int CI, int BN_>
struct WgradPolicy {
  static constexpr int BN = BN_, kABytes = 4 * 4096, kBBytes = (BN_ / 32) * 4096;
  static constexpr bool kSplitA = true, kSplitB = true, kAMN = true, kBMN = true;
  static constexpr bool kSumA = false, kSumB = true;       // bias gradient = column sums of the dy tiles
  static constexpr int kGroups = CI == 64 ? 5 : 9;
  struct Params { WgP e; int splits; };
  static __device__ __forceinline__ int num_tiles(const Params& p) { return kGroups * p.splits; }
  static __device__ __forceinline__ int num_kb(const Params& p, int tile) {
    const int blk0 = (tile / kGroups) * p.e.blocks_per_cta;
    return max(0, min(p.e.blocks_per_cta, p.e.total_blocks - blk0));
  }
  static __device__ __forceinline__ void taps(int tile, int& tap_a, int& tap_b) {
    tap_a = (tile % kGroups) * (128 / CI);
    tap_b = (CI == 64 && tap_a + 1 < 9) ? tap_a + 1 : tap_a;
  }
  struct Tile { int tap_a, tap_b, z, ft, tt, b, nkb; };  // tap pair, split + pixel-block cursor (ft fastest, then tt, then b)
  static __device__ __forceinline__ Tile tile(const Params& p, int tile) {
    Tile t;
    taps(tile, t.tap_a, t.tap_b);
    t.z = tile / kGroups;
    const int blk = (tile / kGroups) * p.e.blocks_per_cta;
    t.ft = blk % p.e.nft; t.tt = (blk / p.e.nft) % p.e.ntt; t.b = blk / (p.e.nft * p.e.ntt);
    t.nkb = num_kb(p, tile);
    return t;
  }
  static __device__ __forceinline__ void load(const Params& p, Tile& t, const CUtensorMap* mapX, const CUtensorMap* mapDy,
                                              uint32_t sa, uint32_t sb, uint32_t, uint32_t bar, bool leader) {
    const int f0 = t.ft * WG_PF, t0 = t.tt * WG_PT;
    if (leader) {
#pragma unroll
      for (int c = 0; c < 4; c++) {
        const int tap = (c * 32) / CI == 0 ? t.tap_a : t.tap_b;
        tma_load_4d(sa + c * 4096, mapX, bar, (c * 32) % CI, f0 + tap / 3 - 1, t0 + tap % 3 - 1, t.b);
      }
#pragma unroll
      for (int c = 0; c < BN / 32; c++) tma_load_4d(sb + c * 4096, mapDy, bar, c * 32, f0, t0, t.b);
    }
    if (++t.ft == p.e.nft) {
      t.ft = 0;
      if (++t.tt == p.e.ntt) { t.tt = 0; t.b++; }
    }
  }
  // every pixel block is visited once by the tap-group-0 tiles (over all splits)
  static __device__ __forceinline__ bool want_sums(const Params& p, const Tile& t) { return p.e.bpart != nullptr && t.tap_a == 0; }
  static __device__ __forceinline__ void sum_b_store1(const Params& p, const Tile& t, int col, float v) { p.e.bpart[(size_t)t.z * p.e.Co + col] = v; }
  static __device__ __forceinline__ void store(const Params& p, const Tile& t, int r, int c0, const float (&v)[32]) {
    const int slot = r / CI, ci = r % CI;
    if (slot == 1 && t.tap_b == t.tap_a) return;
    float* orow = p.e.part + (((size_t)t.z * 9 + (slot == 0 ? t.tap_a : t.tap_b)) * p.e.Ci + ci) * p.e.Co + c0;
#pragma unroll
    for (int j = 0; j < 32; j += 4) *reinterpret_cast<float4*>(orow + j) = make_float4(v[j], v[j + 1], v[j + 2], v[j + 3]);
  }
};

// The same weight gradient with the dy operand arriving as bf16 hi | lo "pairs" that its producer (max-pool backward, the
// convolution data gradient) wrote next to the fp32 tensor: [2][B,T,F,Co] bf16, hi first.  The tile is the bf16 MN-major
// image the tensor core reads (64-channel chunks of 4 KB, one 128-byte k-line per pixel, 128B swizzle) straight from TMA
// -- no conversion of B in the kernel, which is what bound the bf16 variant of WgradPolicy (tc_engine.cuh).
template <int CI, int BN_>
struct WgradPairPolicy : WgradPolicy<CI, BN_> {
  using Base = WgradPolicy<CI, BN_>;
  using typename Base::Params;
  using typename Base::Tile;
  static constexpr bool kSplitB = false, kSumB = true;
  static __device__ __forceinline__ void load16(const Params& p, Tile& t, const CUtensorMap* mapX, const CUtensorMap* mapDy16,
                                                uint32_t sa, uint32_t sb, uint32_t sb_lo, uint32_t bar, bool leader, int halves) {
    const int f0 = t.ft * WG_PF, t0 = t.tt * WG_PT;
    if (leader) {
#pragma unroll
      for (int c = 0; c < 4; c++) {
        const int tap = (c * 32) / CI == 0 ? t.tap_a : t.tap_b;
        tma_load_4d(sa + c * 4096, mapX, bar, (c * 32) % CI, f0 + tap / 3 - 1, t0 + tap % 3 - 1, t.b);
      }
#pragma unroll
      for (int c = 0; c < BN_ / 64; c++) {
        tma_load_4d(sb + c * 4096, mapDy16, bar, c * 64, f0, t0, t.b);
        if (halves == 2) tma_load_4d(sb_lo + c * 4096, mapDy16, bar, c * 64, f0, t0, t.b + p.e.B);     // lo = second half of the batch axis
      }
    }
    if (++t.ft == p.e.nft) {
      t.ft = 0;
      if (++t.tt == p.e.ntt) { t.tt = 0; t.b++; }
    }
  }
};

template <int BN>
static int launch_conv_persistent(const CUtensorMap& ma, const CUtensorMap& mb, const ConvEpi& e, cudaStream_t st) {
  typename ConvPolicy<BN>::Params p{e, ceil_div(e.F, CT_F), ceil_div(e.T, CT_T), e.Cin / 32};
  const long long tiles = (long long)p.nft * p.ntt * e.B;
  if (tiles >= (1LL << 31)) { set_error("conv3x3_tc: too many tiles"); return B200ASR_BAD_SHAPE; }
  return launch_engine<ConvPolicy<BN>, 1>(ma, mb, p, (int)tiles, st, "tc_conv3x3");
}

// pixel blocks per split and number of splits: about two tiles per SM over the tap groups, at least 64 blocks per tile
static int wgrad_splits(int Ci, int total_blocks, int& blocks_per_cta) {
  const int groups = Ci == 64 ? 5 : 9;
  const int splits = max(1, (2 * device_sm_count()) / groups);
  blocks_per_cta = max(64, ceil_div(total_blocks, splits));
  return ceil_div(total_blocks, blocks_per_cta);
}

template <int CI, int BN, int NSPLIT, class Pol = WgradPolicy<CI, BN>>
static int launch_wgrad(const CUtensorMap& mx, const CUtensorMap& mdy, const WgP& e, int splits, cudaStream_t st) {
  typename Pol::Params p{e, splits};
  return launch_engine<Pol, NSPLIT>(mx, mdy, p, Pol::kGroups * splits, st, "tc_conv3x3_wgrad");
}

}  // namespace tc

// wk: [9][Cout][Cin] K-major weights (conv_repack_k_kernel).
int conv3x3_tc(const float* in, const float* wk, const float* bias, const float* mask, float* out, int B, int T, int F,
               int Cin, int Cout, int relu, int precision, cudaStream_t st, const uint32_t* mask_bits, uint32_t* out_bits) {
  using namespace tc;
  B200_REQUIRE(precision == 1, B200ASR_BAD_ARG, "conv3x3_tc: precision must be 1");
  B200_REQUIRE(!(mask && mask_bits), B200ASR_BAD_ARG, "conv3x3_tc: pass the ReLU mask as floats or as bits, not both");
  B200_REQUIRE(Cin % 32 == 0 && (Cout == 64 || Cout == 128), B200ASR_BAD_SHAPE,
               "conv3x3_tc: needs Cin %% 32 == 0 and Cout in {64,128} (Cin=%d Cout=%d)", Cin, Cout);
  B200_REQUIRE(aligned16(in) && aligned16(wk) && aligned16(out) && (!bias || aligned16(bias)) && (!mask || aligned16(mask)),
               B200ASR_BAD_ALIGN, "conv3x3_tc: pointers must be 16-byte aligned");
  CUtensorMap ma, mb;
  {
    uint64_t dims[4] = {(uint64_t)Cin, (uint64_t)F, (uint64_t)T, (uint64_t)B};
    uint64_t strides[3] = {(uint64_t)Cin, (uint64_t)F * Cin, (uint64_t)T * F * Cin};
    uint32_t box[4] = {32, CT_F, CT_T, 1};
    int rc = make_tensor_map_f32(&ma, in, 4, dims, strides, box, true);
    if (rc) return rc;
  }
  {
    uint64_t dims[2] = {(uint64_t)Cin, (uint64_t)9 * Cout};
    uint64_t strides[1] = {(uint64_t)Cin};
    uint32_t box[2] = {32, (uint32_t)Cout};
    int rc = make_tensor_map_f32(&mb, wk, 2, dims, strides, box, true);
    if (rc) return rc;
  }
  ConvEpi e{out, bias, mask, mask_bits, out_bits, relu, B, T, F, Cin, Cout};
  return Cout == 64 ? launch_conv_persistent<64>(ma, mb, e, st) : launch_conv_persistent<128>(ma, mb, e, st);
}

// dbias (optional, not at precision 1): [Co], produced by the kernel; returns with *dbias_done = 1 when the
// kernel took care of it (the caller runs the separate column-sum pass otherwise)
int conv3x3_wgrad_tc(const float* x, const float* dy, float* dwr, int B, int T, int F, int Ci, int Co, int precision,
                     cudaStream_t st, float* dbias, int* dbias_done, const void* dy16) {
  using namespace tc;
  if (dbias_done) *dbias_done = 0;
  // dy as bf16 pairs [2][B,T,F,Co] written by its producer (bf16 modes): B tiles by TMA, no conversion in the kernel
  const bool pairs = dy16 && (precision == 6 || precision == 2);
  B200_REQUIRE(precision == 1 || precision == 3 || precision == 2 || precision == 6, B200ASR_BAD_ARG, "conv3x3_wgrad_tc: precision must be 1, 3 (tf32) or 2, 6 (bf16)");
  B200_REQUIRE((Ci == 64 || Ci == 128) && (Co == 64 || Co == 128), B200ASR_BAD_SHAPE,
               "conv3x3_wgrad_tc: needs Ci, Co in {64,128} (Ci=%d Co=%d)", Ci, Co);
  B200_REQUIRE(aligned16(x) && aligned16(pairs ? dy16 : (const void*)dy) && aligned16(dwr), B200ASR_BAD_ALIGN, "conv3x3_wgrad_tc: alignment");
  // tf32 / 3xTF32: all nine taps per x patch (tc_conv_wgrad.cu); the tap-shifted policies below serve the bf16 modes
  if (precision == 1 || precision == 3) return conv3x3_wgrad_tc_halo(x, dy, dwr, B, T, F, Ci, Co, precision, st, dbias, dbias_done);
  CUtensorMap mx, mdy;
  {
    uint64_t dims[4] = {(uint64_t)Ci, (uint64_t)F, (uint64_t)T, (uint64_t)B};
    uint64_t strides[3] = {(uint64_t)Ci, (uint64_t)F * Ci, (uint64_t)T * F * Ci};
    uint32_t box[4] = {32, WG_PF, WG_PT, 1};
    if (int rc = make_tensor_map_f32(&mx, x, 4, dims, strides, box)) return rc;
  }
  if (pairs) {
    uint64_t dims[4] = {(uint64_t)Co, (uint64_t)F, (uint64_t)T, (uint64_t)2 * B};
    uint64_t strides[3] = {(uint64_t)Co, (uint64_t)F * Co, (uint64_t)T * F * Co};
    uint32_t box[4] = {64, WG_PF, WG_PT, 1};
    if (int rc = make_tensor_map_bf16(&mdy, dy16, 4, dims, strides, box)) return rc;
  } else {
    uint64_t dims[4] = {(uint64_t)Co, (uint64_t)F, (uint64_t)T, (uint64_t)B};
    uint64_t strides[3] = {(uint64_t)Co, (uint64_t)F * Co, (uint64_t)T * F * Co};
    uint32_t box[4] = {32, WG_PF, WG_PT, 1};
    if (int rc = make_tensor_map_f32(&mdy, dy, 4, dims, strides, box)) return rc;
  }
  const bool fuse_bias = dbias != nullptr;
  WgP e{nullptr, nullptr, B, T, F, Ci, Co, ceil_div(F, WG_PF), ceil_div(T, WG_PT), 0, 0};
  const long long total = (long long)B * e.nft * e.ntt;
  B200_REQUIRE(total < (1LL << 31), B200ASR_BAD_SHAPE, "conv3x3_wgrad_tc: too many pixel blocks");
  e.total_blocks = (int)total;
  const int splits = wgrad_splits(Ci, e.total_blocks, e.blocks_per_cta);
  const long long wn = 9LL * Ci * Co;
  e.part = (float*)stream_scratch(sizeof(float) * (size_t)splits * (wn + (fuse_bias ? Co : 0)), st);
  if (!e.part) return B200ASR_CUDA_ERROR;
  e.bpart = fuse_bias ? e.part + (size_t)splits * wn : nullptr;
  int rc;
#define WGP(CIv, BNv)                                                                                                  \
  if (pairs) rc = precision == 6 ? launch_wgrad<CIv, BNv, 6, WgradPairPolicy<CIv, BNv>>(mx, mdy, e, splits, st)        \
                                 : launch_wgrad<CIv, BNv, 2, WgradPairPolicy<CIv, BNv>>(mx, mdy, e, splits, st);       \
  else if (precision == 6) rc = launch_wgrad<CIv, BNv, 6>(mx, mdy, e, splits, st);                                     \
  else rc = launch_wgrad<CIv, BNv, 2>(mx, mdy, e, splits, st);
  if (Ci == 64 && Co == 64) { WGP(64, 64) }
  else if (Ci == 64 && Co == 128) { WGP(64, 128) }
  else if (Ci == 128 && Co == 64) { WGP(128, 64) }
  else { WGP(128, 128) }
#undef WGP
  if (rc) return rc;
  if ((rc = reduce_parts(e.part, splits, wn, wn, dwr, 0, st))) return rc;
  if (!fuse_bias) return B200ASR_OK;
  if (dbias_done) *dbias_done = 1;
  return reduce_parts(e.bpart, splits, Co, Co, dbias, 0, st);
}

}  // namespace b200asr
