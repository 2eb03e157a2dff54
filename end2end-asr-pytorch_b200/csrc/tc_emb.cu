// emb_cnn front end, second convolution (models/asr/transformer.py:37: Conv2d(32, 32, kernel (21, 11), stride (2, 1)) on the
// NCHW activation) as IMPLICIT GEMMs on the persistent wgmma engine -- no im2col matrix, no col2im scatter.
//
// Geometry: x [B, 32, H, W], w [32, 32, KH, KW], y [B, 32, OH, OW] with OH = (H - KH) / SH + 1, OW = W - KW + 1 (stride 1
// along W, no padding).  Because the stride along W is 1, the GEMM row index can be the output column:
//
//   forward        y[b, :, oh, ow0 + m]  = sum_{kh, kw} sum_ci  x[b, ci, SH*oh + kh, ow0 + m + kw] * w[:, ci, kh, kw]
//     one k-block = one (kh, kw): the A tile (128 m x 32 ci, MN-major) is ONE strided window of the activation -- 4 TMA
//     boxes {32 w, 32 c} of the (w, c, h, b) view at (ow0 + kw, 0, SH*oh + kh) -- and the B tile the 32 x 32 weight slice of that tap (K-major,
//     pre-converted: bf16 hi | lo for the bf16 modes, tf32 hi | lo for 3xTF32).
//   data gradient  dx[b, :, h, w0 + m]   = sum_{kh == h (mod SH), kw} sum_co  dy[b, co, (h - kh) / SH, w0 + m - kw] * w[co, :, kh, kw]
//     the same kernel: a gather over the taps whose row parity matches h; boxes that reach outside dy are zero-filled by TMA.
//   weight gradient dw[:, ci, kh, kw]    = sum_{b, oh, ow} dy[b, :, oh, ow] * x[b, ci, SH*oh + kh, ow + kw]
//     GEMM rows = (kw, ci) -- four taps x 32 channels per 128-row tile --, columns = co, contraction = output pixels along ow:
//     both operands K-major fp32 windows (3xTF32, B split in the kernel), one partial per row split, summed in split order.
//
// MMA N = 32 (the layer has 32 output channels); the engine's consumers turn the fp32 A tile into register operands exactly
// as for the other policies.  TMA needs 16-byte row pitches, so the NCHW tensors these kernels touch are
// PITCHED: rows of `pitch` floats (a multiple of 4) of which the first W are valid (W = 205 / 195 at cfg3).
//
// TMA also needs the INNERMOST start coordinate of a box to be 16-byte aligned (UTMALDG raises an illegal-instruction
// fault otherwise -- measured), and the windows above start at ow0 + kw for every kw.  So the tensor whose windows slide
// (x for forward / weight gradient, dy for the data gradient) is first written as FOUR copies shifted right by s = 0..3
// floats (copy_s[w'] = src[w' - s], zeros outside: one HBM-bound pass, 5x the activation, against the 231x of an im2col
// matrix); the window that starts at column v is then the box at v + s of copy s = (-v) mod 4, an aligned coordinate.
#include "../../include/b200asr.h"
#include "common.cuh"
#include "kernels.h"
#include "tc_common.cuh"
#include "tc_engine.cuh"

namespace b200asr {
namespace tc {

constexpr int EC = 32;                     // channels in and out

struct EmbG {
  int B, H, W, OH, OW, KH, KW, SH;
  int xp, yp;            // row pitch (floats) of the [B,32,H,W] tensor (x / dx) and of the [B,32,OH,OW] tensor (y / dy)
};

struct EmbConvP {
  float* out;            // forward: y [B, 32, OH, OW]; data gradient: dx [B, 32, H, W]
  const float* bias;     // forward only (may be null)
  EmbG g;
  int rows, width, pitch, tiles_w;      // output rows per image (OH / H), output width (OW / W) and row pitch, 128-wide tiles per row
  int b_rows;                    // rows of one half (hi or lo) of the repacked weight matrix = KH * KW * 32
};

// forward (DGRAD = false) and data gradient (DGRAD = true)
template <bool DGRAD>
struct EmbConvPolicy {
  static constexpr int BN = EC, kABytes = 4 * 4096, kBBytes = EC * 128;
  static constexpr bool kSplitA = true, kSplitB = false, kAMN = true, kBMN = false, kSumA = false, kSumB = false;
  struct Params { EmbConvP e; };
  static __device__ __forceinline__ int num_tiles(const Params& p) { return p.e.g.B * p.e.rows * p.e.tiles_w; }
  struct Tile { int w0, r, b, kh, kw, nkh, kh0; };
  // taps along H that reach output row r: forward all KH; data gradient kh == h (mod SH) with 0 <= (h - kh) / SH < OH
  static __device__ __forceinline__ void kh_range(const EmbG& g, int r, int& kh0, int& nkh) {
    if (!DGRAD) { kh0 = 0; nkh = g.KH; return; }
    int lo = max(0, r - g.SH * (g.OH - 1));
    lo += ((r - lo) % g.SH + g.SH) % g.SH;                 // first kh >= lo with (r - kh) % SH == 0
    const int hi = min(g.KH - 1, r);
    kh0 = lo;
    nkh = hi >= lo ? (hi - lo) / g.SH + 1 : 0;
  }
  static __device__ __forceinline__ Tile tile(const Params& p, int tile) {
    Tile t;
    t.w0 = (tile % p.e.tiles_w) * 128;
    const int q = tile / p.e.tiles_w;
    t.r = q % p.e.rows; t.b = q / p.e.rows;
    kh_range(p.e.g, t.r, t.kh0, t.nkh);
    t.kh = t.kh0; t.kw = 0;
    return t;
  }
  static __device__ __forceinline__ int num_kb(const Params& p, int tile) {
    int kh0, nkh;
    kh_range(p.e.g, (tile / p.e.tiles_w) % p.e.rows, kh0, nkh);
    return nkh * p.e.g.KW;
  }
  static __device__ __forceinline__ void load_a(const Params& p, const Tile& t, const CUtensorMap* mapA, uint32_t sa, uint32_t bar) {
    const int w = DGRAD ? t.w0 - t.kw : t.w0 + t.kw;                   // window start; copy s = (-w) mod 4 holds it at w + s
    const int s = (-w) & 3;
    const int h = DGRAD ? (t.r - t.kh) / p.e.g.SH : t.r * p.e.g.SH + t.kh;
#pragma unroll
    for (int c = 0; c < 4; c++) tma_load_4d(sa + c * 4096, mapA, bar, w + s + 32 * c, 0, h, s * p.e.g.B + t.b);
  }
  static __device__ __forceinline__ void advance(const Params& p, Tile& t) {
    if (++t.kw == p.e.g.KW) { t.kw = 0; t.kh += DGRAD ? p.e.g.SH : 1; }
  }
  // 3xTF32: fp32 hi | lo weight slices (128-byte rows)
  static __device__ __forceinline__ void load(const Params& p, Tile& t, const CUtensorMap* mapA, const CUtensorMap* mapB,
                                              uint32_t sa, uint32_t sb, uint32_t sb_lo, uint32_t bar, bool leader) {
    if (leader) {
      load_a(p, t, mapA, sa, bar);
      const int row = (t.kh * p.e.g.KW + t.kw) * EC;
      tma_load_2d(sb, mapB, bar, 0, row);
      tma_load_2d(sb_lo, mapB, bar, 0, row + p.e.b_rows);
    }
    advance(p, t);
  }
  // bf16 modes: bf16 hi (| lo) weight slices (64-byte rows)
  static __device__ __forceinline__ void load16(const Params& p, Tile& t, const CUtensorMap* mapA, const CUtensorMap* mapB,
                                                uint32_t sa, uint32_t sb, uint32_t sb_lo, uint32_t bar, bool leader, int halves) {
    if (leader) {
      load_a(p, t, mapA, sa, bar);
      const int row = (t.kh * p.e.g.KW + t.kw) * EC;
      tma_load_2d(sb, mapB, bar, 0, row);
      if (halves == 2) tma_load_2d(sb_lo, mapB, bar, 0, row + p.e.b_rows);
    }
    advance(p, t);
  }
  static __device__ __forceinline__ void store(const Params& p, const Tile& t, int r, int c0, const float (&v)[32]) {
    const int w = t.w0 + r;
    if (w >= p.e.width) return;
    // NCHW output: consecutive lanes = consecutive w -> every channel's store is one coalesced 128-byte row segment
    float* o = p.e.out + (((size_t)t.b * EC + c0) * p.e.rows + t.r) * p.e.pitch + w;
    const size_t cs = (size_t)p.e.rows * p.e.pitch;
#pragma unroll
    for (int j = 0; j < 32; j++) o[j * cs] = v[j] + (p.e.bias ? __ldg(p.e.bias + c0 + j) : 0.f);
  }
};

struct EmbWgP {
  float* part;           // [splits][32 co, 32 ci, KH, KW] partial weight gradients
  EmbG g;
  int m_tiles, splits, rows_per_split, owb;      // ceil(KW / 4); splits of the B*OH output rows; 32-wide ow blocks per row
};

struct EmbWgradPolicy {
  static constexpr int BN = EC, kABytes = 4 * 4096, kBBytes = EC * 128;
  static constexpr bool kSplitA = true, kSplitB = true, kAMN = false, kBMN = false, kSumA = false, kSumB = false;
  struct Params { EmbWgP e; };
  static __device__ __forceinline__ int num_tiles(const Params& p) { return p.e.g.KH * p.e.m_tiles * p.e.splits; }
  struct Tile { int kh, mt, z, row, row_end, ob; };       // tap row, kw group, split, (b, oh) row cursor, ow-block cursor
  static __device__ __forceinline__ Tile tile(const Params& p, int tile) {
    Tile t;
    t.kh = tile % p.e.g.KH;
    const int q = tile / p.e.g.KH;
    t.mt = q % p.e.m_tiles;
    const int z = q / p.e.m_tiles;
    t.z = z;
    t.row = z * p.e.rows_per_split;
    t.row_end = min(p.e.g.B * p.e.g.OH, t.row + p.e.rows_per_split);
    t.ob = 0;
    return t;
  }
  static __device__ __forceinline__ int num_kb(const Params& p, int tile) {
    const int z = tile / (p.e.g.KH * p.e.m_tiles);
    const int r0 = z * p.e.rows_per_split, r1 = min(p.e.g.B * p.e.g.OH, r0 + p.e.rows_per_split);
    return max(0, r1 - r0) * p.e.owb;
  }
  static __device__ __forceinline__ void load(const Params& p, Tile& t, const CUtensorMap* mapX, const CUtensorMap* mapDy,
                                              uint32_t sa, uint32_t sb, uint32_t, uint32_t bar, bool leader) {
    if (leader) {
      const int b = t.row / p.e.g.OH, oh = t.row % p.e.g.OH, ow0 = t.ob * 32;
#pragma unroll
      for (int j = 0; j < 4; j++) {
        const int kw = t.mt * 4 + j;
        // taps beyond KW: a box at channel coordinate 32 is entirely out of bounds -> zero rows, same byte count
        const int s = (-kw) & 3;                                        // shifted copy that holds column ow0 + kw at an aligned coordinate
        tma_load_4d(sa + j * 4096, mapX, bar, ow0 + kw + s, kw < p.e.g.KW ? 0 : EC, p.e.g.SH * oh + t.kh, s * p.e.g.B + b);
      }
      tma_load_4d(sb, mapDy, bar, ow0, 0, oh, b);
    }
    if (++t.ob == p.e.owb) { t.ob = 0; t.row++; }
  }
  static __device__ __forceinline__ void store(const Params& p, const Tile& t, int r, int c0, const float (&v)[32]) {
    const int kw = t.mt * 4 + r / EC, ci = r % EC;
    if (kw >= p.e.g.KW) return;
    const size_t cs = (size_t)EC * p.e.g.KH * p.e.g.KW;
    float* o = p.e.part + (size_t)t.z * EC * cs + ((size_t)ci * p.e.g.KH + t.kh) * p.e.g.KW + kw;        // + co * (32 * KH * KW)
#pragma unroll
    for (int j = 0; j < 32; j++) o[(size_t)(c0 + j) * cs] = v[j];
  }
};

// ----------------------------------------------------------------------------------------------------------------------
// First emb_cnn convolution (models/asr/transformer.py:33: Conv2d(1, 32, (41, 11), stride (2, 2), padding (0, 10))) on the
// same engine.  With ONE input channel the contraction index is the tap itself; the 41 taps along H take the role of the
// channels: the activation is read through an OVERLAPPING tensor-map view (w, kh, oh, n) whose kh stride is one input row
// and whose oh stride is two, so a box {32 w, 32 kh} is a 32 x 32 window of "channel" rows for output row oh (rows beyond
// kh = 40 are out of bounds of the view: zero fill).  A k-block = (kw, block of 32 kh): 11 x 2 per tile.  The stride 2 along
// W is taken out by de-interleaving: input column 2 (ow + q) + r with r = (kw - PW) & 1, q = (kw - PW - r) / 2 lives in the
// parity-r copy at column ow + q; each parity copy exists in the four 16-byte alignments (see above): eight half-width copies.
struct Emb1G {
  int B, H, W, OH, OW, KH, KW, PW, pd;      // pd: pitch of the de-interleaved copies
};
__device__ __forceinline__ void emb1_window(int kw, int PW, int w0, int& col, int& copy) {
  const int e = kw - PW, r = e & 1, q = (e - r) >> 1;          // e - r is even: exact for negative values too
  const int v = w0 + q, s = (-v) & 3;
  col = v + s;
  copy = r * 4 + s;
}

struct Emb1ConvP {
  float* out;            // y [B, 32, OH, OW], row pitch `pitch`
  const float* bias;
  Emb1G g;
  int pitch, tiles_w, nkblk;      // 128-wide tiles per output row; 32-deep kh blocks (2 for KH = 41)
};

struct Emb1ConvPolicy {
  static constexpr int BN = EC, kABytes = 4 * 4096, kBBytes = EC * 128;
  static constexpr bool kSplitA = true, kSplitB = false, kAMN = true, kBMN = false, kSumA = false, kSumB = false;
  struct Params { Emb1ConvP e; };
  static __device__ __forceinline__ int num_tiles(const Params& p) { return p.e.g.B * p.e.g.OH * p.e.tiles_w; }
  struct Tile { int w0, oh, b, t; };                     // t: k-block cursor = kw * nkblk + kblk
  static __device__ __forceinline__ Tile tile(const Params& p, int tile) {
    Tile t;
    t.w0 = (tile % p.e.tiles_w) * 128;
    const int q = tile / p.e.tiles_w;
    t.oh = q % p.e.g.OH; t.b = q / p.e.g.OH; t.t = 0;
    return t;
  }
  static __device__ __forceinline__ int num_kb(const Params& p, int) { return p.e.g.KW * p.e.nkblk; }
  static __device__ __forceinline__ void load_a(const Params& p, const Tile& t, const CUtensorMap* mapA, uint32_t sa, uint32_t bar) {
    int col, copy;
    emb1_window(t.t / p.e.nkblk, p.e.g.PW, t.w0, col, copy);
    const int kh0 = (t.t % p.e.nkblk) * 32;
#pragma unroll
    for (int c = 0; c < 4; c++) tma_load_4d(sa + c * 4096, mapA, bar, col + 32 * c, kh0, t.oh, copy * p.e.g.B + t.b);
  }
  static __device__ __forceinline__ void load(const Params& p, Tile& t, const CUtensorMap* mapA, const CUtensorMap* mapB,
                                              uint32_t sa, uint32_t sb, uint32_t sb_lo, uint32_t bar, bool leader) {
    if (leader) {
      load_a(p, t, mapA, sa, bar);
      tma_load_2d(sb, mapB, bar, 0, t.t * EC);
      tma_load_2d(sb_lo, mapB, bar, 0, (p.e.g.KW * p.e.nkblk + t.t) * EC);
    }
    t.t++;
  }
  static __device__ __forceinline__ void load16(const Params& p, Tile& t, const CUtensorMap* mapA, const CUtensorMap* mapB,
                                                uint32_t sa, uint32_t sb, uint32_t sb_lo, uint32_t bar, bool leader, int halves) {
    if (leader) {
      load_a(p, t, mapA, sa, bar);
      tma_load_2d(sb, mapB, bar, 0, t.t * EC);
      if (halves == 2) tma_load_2d(sb_lo, mapB, bar, 0, (p.e.g.KW * p.e.nkblk + t.t) * EC);
    }
    t.t++;
  }
  static __device__ __forceinline__ void store(const Params& p, const Tile& t, int r, int c0, const float (&v)[32]) {
    const int w = t.w0 + r;
    if (w >= p.e.g.OW) return;
    float* o = p.e.out + (((size_t)t.b * EC + c0) * p.e.g.OH + t.oh) * p.e.pitch + w;
    const size_t cs = (size_t)p.e.g.OH * p.e.pitch;
#pragma unroll
    for (int j = 0; j < 32; j++) o[j * cs] = v[j] + (p.e.bias ? __ldg(p.e.bias + c0 + j) : 0.f);
  }
};

// weight gradient of the first convolution: rows = (kw (4 per tile), kh in its 32-block), columns = co, contraction = output
// pixels along ow (32 per k-block); x windows from the de-interleaved copies, dy [B, 32, OH, OW] (row pitch a multiple of 4)
struct Emb1WgP {
  float* part;           // [splits][32 co, 1, KH, KW] partial weight gradients
  Emb1G g;
  int m_tiles, nkblk, splits, rows_per_split, owb;
};

struct Emb1WgradPolicy {
  static constexpr int BN = EC, kABytes = 4 * 4096, kBBytes = EC * 128;
  static constexpr bool kSplitA = true, kSplitB = true, kAMN = false, kBMN = false, kSumA = false, kSumB = false;
  struct Params { Emb1WgP e; };
  static __device__ __forceinline__ int num_tiles(const Params& p) { return p.e.nkblk * p.e.m_tiles * p.e.splits; }
  struct Tile { int kblk, mt, z, row, row_end, ob; };
  static __device__ __forceinline__ Tile tile(const Params& p, int tile) {
    Tile t;
    t.kblk = tile % p.e.nkblk;
    const int q = tile / p.e.nkblk;
    t.mt = q % p.e.m_tiles;
    const int z = q / p.e.m_tiles;
    t.z = z;
    t.row = z * p.e.rows_per_split;
    t.row_end = min(p.e.g.B * p.e.g.OH, t.row + p.e.rows_per_split);
    t.ob = 0;
    return t;
  }
  static __device__ __forceinline__ int num_kb(const Params& p, int tile) {
    const int z = tile / (p.e.nkblk * p.e.m_tiles);
    const int r0 = z * p.e.rows_per_split, r1 = min(p.e.g.B * p.e.g.OH, r0 + p.e.rows_per_split);
    return max(0, r1 - r0) * p.e.owb;
  }
  static __device__ __forceinline__ void load(const Params& p, Tile& t, const CUtensorMap* mapX, const CUtensorMap* mapDy,
                                              uint32_t sa, uint32_t sb, uint32_t, uint32_t bar, bool leader) {
    if (leader) {
      const int b = t.row / p.e.g.OH, oh = t.row % p.e.g.OH, ow0 = t.ob * 32;
#pragma unroll
      for (int j = 0; j < 4; j++) {
        const int kw = t.mt * 4 + j;
        int col, copy;
        emb1_window(min(kw, p.e.g.KW - 1), p.e.g.PW, ow0, col, copy);
        // taps beyond KW: a box at kh coordinate 64 is entirely outside the view -> zero rows, same byte count
        tma_load_4d(sa + j * 4096, mapX, bar, col, kw < p.e.g.KW ? t.kblk * 32 : 64, oh, copy * p.e.g.B + b);
      }
      tma_load_4d(sb, mapDy, bar, ow0, 0, oh, b);
    }
    if (++t.ob == p.e.owb) { t.ob = 0; t.row++; }
  }
  static __device__ __forceinline__ void store(const Params& p, const Tile& t, int r, int c0, const float (&v)[32]) {
    const int kw = t.mt * 4 + r / 32, kh = t.kblk * 32 + r % 32;
    if (kw >= p.e.g.KW || kh >= p.e.g.KH) return;
    const size_t cs = (size_t)p.e.g.KH * p.e.g.KW;
    float* o = p.e.part + (size_t)t.z * EC * cs + (size_t)kh * p.e.g.KW + kw;        // + co * (KH * KW)
#pragma unroll
    for (int j = 0; j < 32; j++) o[(size_t)(c0 + j) * cs] = v[j];
  }
};

// x [B, H, W] -> eight copies [parity r][shift s][B][H][pd]: copy[w'] = x[2 (w' - s) + r], zeros outside
__global__ void emb1_prep_kernel(const float* __restrict__ x, float* __restrict__ dst, long long R, int W, int pd) {
  const int q = pd / 4;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= R * q) return;
  const long long row = i / q;
  const int w0 = (int)(i % q) * 4;
  const float* in = x + row * W;
#pragma unroll
  for (int r = 0; r < 2; r++) {
    float v[7];
#pragma unroll
    for (int j = 0; j < 7; j++) {
      const int c = 2 * (w0 - 3 + j) + r;
      v[j] = (c >= 0 && c < W) ? __ldg(in + c) : 0.f;
    }
#pragma unroll
    for (int s = 0; s < 4; s++)
      *reinterpret_cast<float4*>(dst + ((size_t)(r * 4 + s) * R + row) * pd + w0) = make_float4(v[3 - s], v[4 - s], v[5 - s], v[6 - s]);
  }
}

// w [32 co, 1, KH, KW] -> [(kw, kblk)][co][32 kh] (zero beyond KH); mode 3: fp32 hi | lo, modes 6 / 2: bf16 hi (| lo)
__global__ void emb1_repack_kernel(const float* __restrict__ w, void* __restrict__ out, int KH, int KW, int nkblk, int mode) {
  const int total = KW * nkblk * EC * 32;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int k = i % 32, co = (i / 32) % EC, t = i / (32 * EC);
  const int kh = (t % nkblk) * 32 + k, kw = t / nkblk;
  const float v = kh < KH ? w[((size_t)co * KH + kh) * KW + kw] : 0.f;
  if (mode == 3) {
    float* o = (float*)out;
    const float hi = tf32_rn(v);
    o[i] = hi;
    o[total + i] = v - hi;
  } else {
    uint16_t* o = (uint16_t*)out;
    const uint32_t r = __float_as_uint(v) + 0x8000u;
    o[i] = (uint16_t)(r >> 16);
    if (mode == 6) {
      const float lo = v - __uint_as_float(r & 0xFFFF0000u);
      o[total + i] = (uint16_t)((__float_as_uint(lo) + 0x8000u) >> 16);
    }
  }
}

// w [32 co, 32 ci, KH, KW] -> tap-major 32 x 32 slices: forward [(kh, kw)][co][ci], data gradient [(kh, kw)][ci][co];
// mode 3: fp32 (rn_tf32(w) | w - hi); modes 6 / 2: bf16 (hi | lo) / hi
__global__ void emb_repack_kernel(const float* __restrict__ w, void* __restrict__ out, int KH, int KW, int dgrad, int mode) {
  const int taps = KH * KW, total = taps * EC * EC;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int inner = i % EC, outer = (i / EC) % EC, tap = i / (EC * EC);
  const int co = dgrad ? inner : outer, ci = dgrad ? outer : inner;
  const float v = w[((size_t)co * EC + ci) * taps + tap];
  if (mode == 3) {
    float* o = (float*)out;
    const float hi = tf32_rn(v);
    o[i] = hi;
    o[total + i] = v - hi;
  } else {
    uint16_t* o = (uint16_t*)out;
    const uint32_t r = __float_as_uint(v) + 0x8000u;
    o[i] = (uint16_t)(r >> 16);
    if (mode == 6) {
      const float lo = v - __uint_as_float(r & 0xFFFF0000u);
      o[total + i] = (uint16_t)((__float_as_uint(lo) + 0x8000u) >> 16);
    }
  }
}

// db[c] = sum over (b, h, w) of dy: grid (splits, 32 channels), a warp walks a row; part[split][c] = the block's sum, added
// up in split order by reduce_parts
constexpr int EMB_BIAS_SPLITS = 32;
__global__ void emb_bias_grad_kernel(const float* __restrict__ dy, float* __restrict__ part, int B, int H, int W, int P) {
  __shared__ float red[8];
  const int c = blockIdx.y, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int rows = B * H;
  float s = 0.f;
  for (int r = blockIdx.x * 8 + warp; r < rows; r += gridDim.x * 8) {
    const float* row = dy + (((size_t)(r / H) * EC + c) * H + (r % H)) * P;
    for (int w = lane; w < W; w += 32) s += row[w];
  }
  s = warp_sum(s);
  if (lane == 0) red[warp] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int w = 0; w < 8; w++) t += red[w];
    part[blockIdx.x * EC + c] = t;
  }
}

// rows [R][Ps] (first W valid) -> four copies [4][R][Pd], copy s shifted right by s floats, zeros elsewhere
__global__ void emb_shift4_kernel(const float* __restrict__ src, float* __restrict__ dst, long long R, int W, int Ps, int Pd) {
  const int q = Pd / 4;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= R * q) return;
  const long long row = i / q;
  const int w0 = (int)(i % q) * 4;
  const float* in = src + row * Ps;
  float v[7];
#pragma unroll
  for (int j = 0; j < 7; j++) {
    const int w = w0 - 3 + j;
    v[j] = (w >= 0 && w < W) ? __ldg(in + w) : 0.f;
  }
#pragma unroll
  for (int s = 0; s < 4; s++)
    *reinterpret_cast<float4*>(dst + ((size_t)s * R + row) * Pd + w0) = make_float4(v[3 - s], v[4 - s], v[5 - s], v[6 - s]);
}

static inline int shift_pitch(int W) { return (W + 3 + 3) / 4 * 4; }
static inline size_t shift_floats(int B, int H, int W) { return (size_t)4 * B * EC * H * shift_pitch(W); }
static inline size_t weight_floats(int KH, int KW) { return ((size_t)2 * KH * KW * EC * EC + 255) / 256 * 256; }

static int make_shifted(const float* src, float* dst, int B, int H, int W, int P, cudaStream_t st) {
  const long long R = (long long)B * EC * H, n = R * (shift_pitch(W) / 4);
  emb_shift4_kernel<<<(unsigned)ceil_div_ll(n, 256), 256, 0, st>>>(src, dst, R, W, P, shift_pitch(W));
  return check_launch("conv2d_tc_shift4");
}

// [N, 32, H, .] (row pitch P, W valid columns) seen as the 4-D tensor (w, c, h, n): a box {32 w, 32 c, 1, 1} is one 32 x 32
// window of a row across all channels.  For the shifted copies N = 4 * B (index s * B + b) and every column is valid.
static int nchw_map(CUtensorMap* m, const float* base, int W, int P, int H, int N) {
  uint64_t dims[4] = {(uint64_t)W, (uint64_t)EC, (uint64_t)H, (uint64_t)N};
  uint64_t strides[3] = {(uint64_t)H * P, (uint64_t)P, (uint64_t)EC * H * P};
  uint32_t box[4] = {32, EC, 1, 1};
  return make_tensor_map_f32(m, base, 4, dims, strides, box, false);
}

static inline int emb1_pitch(int W) { return ((W + 1) / 2 + 3 + 3) / 4 * 4; }
static inline size_t emb1_copy_floats(int B, int H, int W) { return (size_t)8 * B * H * emb1_pitch(W); }
static inline size_t emb1_weight_floats(int KH, int KW) { return ((size_t)2 * KW * ((KH + 31) / 32) * EC * 32 + 255) / 256 * 256; }

static int emb1_geom(Emb1G& g, const char* who, int B, int H, int W, int Co, int KH, int KW, int PW) {
  B200_REQUIRE(Co == EC, B200ASR_BAD_SHAPE, "%s: 32 output channels (Co=%d)", who, Co);
  B200_REQUIRE(B > 0 && KH > 0 && KH <= 64 && KW > 0 && PW >= 0 && H >= KH && W + 2 * PW >= KW, B200ASR_BAD_SHAPE, "%s: bad geometry", who);
  g = Emb1G{B, H, W, (H - KH) / 2 + 1, (W + 2 * PW - KW) / 2 + 1, KH, KW, PW, emb1_pitch(W)};
  return B200ASR_OK;
}

// the de-interleaved, shifted copies and the overlapping (w, kh, oh, n) view of them
static int emb1_prepare(CUtensorMap* m, const float* x, float* copies, const Emb1G& g, cudaStream_t st) {
  const long long R = (long long)g.B * g.H, n = R * (g.pd / 4);
  emb1_prep_kernel<<<(unsigned)ceil_div_ll(n, 256), 256, 0, st>>>(x, copies, R, g.W, g.pd);
  if (int rc = check_launch("conv2d_c1_prep")) return rc;
  uint64_t dims[4] = {(uint64_t)g.pd, (uint64_t)g.KH, (uint64_t)g.OH, (uint64_t)8 * g.B};
  uint64_t strides[3] = {(uint64_t)g.pd, (uint64_t)2 * g.pd, (uint64_t)g.H * g.pd};
  uint32_t box[4] = {32, 32, 1, 1};
  return make_tensor_map_f32(m, copies, 4, dims, strides, box, false);
}

template <bool DGRAD>
static int launch_emb_conv(const CUtensorMap& ma, const CUtensorMap& mb, const EmbConvP& e, int mode, cudaStream_t st) {
  using Pol = EmbConvPolicy<DGRAD>;
  typename Pol::Params p{e};
  const long long tiles = (long long)e.g.B * e.rows * e.tiles_w;
  if (tiles >= (1LL << 31)) { set_error("conv2d_tc: too many tiles"); return B200ASR_BAD_SHAPE; }
  if (mode == 3) return launch_engine<Pol, 3>(ma, mb, p, (int)tiles, st, "conv2d_tc");
  if (mode == 6) return launch_engine<Pol, 6>(ma, mb, p, (int)tiles, st, "conv2d_tc");
  return launch_engine<Pol, 2>(ma, mb, p, (int)tiles, st, "conv2d_tc");
}

static int emb_geom(EmbG& g, const char* who, int B, int Ci, int H, int W, int Co, int KH, int KW, int SH, int xp, int yp) {
  B200_REQUIRE(Ci == EC && Co == EC, B200ASR_BAD_SHAPE, "%s: the implicit-GEMM kernels take 32 input and 32 output channels (Ci=%d Co=%d)", who, Ci, Co);
  B200_REQUIRE(B > 0 && KH > 0 && KW > 0 && SH > 0 && H >= KH && W >= KW, B200ASR_BAD_SHAPE, "%s: bad geometry", who);
  g = EmbG{B, H, W, (H - KH) / SH + 1, W - KW + 1, KH, KW, SH, xp, yp};
  B200_REQUIRE(xp >= W && yp >= g.OW && xp % 4 == 0 && yp % 4 == 0, B200ASR_BAD_SHAPE,
               "%s: row pitches must be multiples of 4 floats (TMA) and cover the rows (x pitch %d for W=%d, y pitch %d for OW=%d)", who, xp, W, yp, g.OW);
  return B200ASR_OK;
}

}  // namespace tc
}  // namespace b200asr

using namespace b200asr;
using namespace b200asr::tc;

extern "C" {

size_t b200asr_conv2d_tc_ws_bytes(int B, int H, int W, int KH, int KW) {
  if (B <= 0 || H <= 0 || W <= 0 || KH <= 0 || KW <= 0) return 0;
  return sizeof(float) * (weight_floats(KH, KW) + shift_floats(B, H, W));        // x copies >= dy copies
}

int b200asr_conv2d_tc_fwd(const float* x, const float* w, const float* bias, float* y, void* ws, int B, int Ci, int H, int W, int Co,
                          int KH, int KW, int SH, int x_pitch, int y_pitch, int precision, b200asr_stream_t stream) {
  B200_REQUIRE(x && w && y && ws, B200ASR_BAD_ARG, "conv2d_tc_fwd: null pointer");
  B200_REQUIRE(precision == 3 || precision == 6 || precision == 2, B200ASR_BAD_ARG, "conv2d_tc_fwd: precision must be 3, 6 or 2");
  EmbG g;
  if (int rc = emb_geom(g, "conv2d_tc_fwd", B, Ci, H, W, Co, KH, KW, SH, x_pitch, y_pitch)) return rc;
  B200_REQUIRE(aligned16(x) && aligned16(ws), B200ASR_BAD_ALIGN, "conv2d_tc_fwd: alignment");
  cudaStream_t st = (cudaStream_t)stream;
  const int total = KH * KW * EC * EC;
  emb_repack_kernel<<<ceil_div(total, 256), 256, 0, st>>>(w, ws, KH, KW, 0, precision);
  note_launch(1);
  CUtensorMap ma, mb;
  float* xs = (float*)ws + weight_floats(KH, KW);
  if (int rc = make_shifted(x, xs, B, H, W, x_pitch, st)) return rc;
  if (int rc = nchw_map(&ma, xs, shift_pitch(W), shift_pitch(W), H, 4 * B)) return rc;
  {
    uint64_t dims[2] = {(uint64_t)EC, (uint64_t)(precision == 2 ? 1 : 2) * KH * KW * EC}, strides[1] = {(uint64_t)EC};
    uint32_t box[2] = {EC, EC};
    int rc = precision == 3 ? make_tensor_map_f32(&mb, ws, 2, dims, strides, box, false) : make_tensor_map_bf16(&mb, ws, 2, dims, strides, box);
    if (rc) return rc;
  }
  EmbConvP e{y, bias, g, g.OH, g.OW, y_pitch, ceil_div(g.OW, 128), KH * KW * EC};
  return launch_emb_conv<false>(ma, mb, e, precision, st);
}

int b200asr_conv2d_tc_bwd_data(const float* dy, const float* w, float* dx, void* ws, int B, int Ci, int H, int W, int Co, int KH,
                               int KW, int SH, int x_pitch, int y_pitch, int precision, b200asr_stream_t stream) {
  B200_REQUIRE(dy && w && dx && ws, B200ASR_BAD_ARG, "conv2d_tc_bwd_data: null pointer");
  B200_REQUIRE(precision == 3 || precision == 6 || precision == 2, B200ASR_BAD_ARG, "conv2d_tc_bwd_data: precision must be 3, 6 or 2");
  EmbG g;
  if (int rc = emb_geom(g, "conv2d_tc_bwd_data", B, Ci, H, W, Co, KH, KW, SH, x_pitch, y_pitch)) return rc;
  B200_REQUIRE(aligned16(dy) && aligned16(ws), B200ASR_BAD_ALIGN, "conv2d_tc_bwd_data: alignment");
  cudaStream_t st = (cudaStream_t)stream;
  const int total = KH * KW * EC * EC;
  emb_repack_kernel<<<ceil_div(total, 256), 256, 0, st>>>(w, ws, KH, KW, 1, precision);
  note_launch(1);
  CUtensorMap ma, mb;
  float* dys = (float*)ws + weight_floats(KH, KW);
  if (int rc = make_shifted(dy, dys, B, g.OH, g.OW, y_pitch, st)) return rc;
  if (int rc = nchw_map(&ma, dys, shift_pitch(g.OW), shift_pitch(g.OW), g.OH, 4 * B)) return rc;
  {
    uint64_t dims[2] = {(uint64_t)EC, (uint64_t)(precision == 2 ? 1 : 2) * KH * KW * EC}, strides[1] = {(uint64_t)EC};
    uint32_t box[2] = {EC, EC};
    int rc = precision == 3 ? make_tensor_map_f32(&mb, ws, 2, dims, strides, box, false) : make_tensor_map_bf16(&mb, ws, 2, dims, strides, box);
    if (rc) return rc;
  }
  EmbConvP e{dx, nullptr, g, H, W, x_pitch, ceil_div(W, 128), KH * KW * EC};
  return launch_emb_conv<true>(ma, mb, e, precision, st);
}

int b200asr_conv2d_tc_bwd_weight(const float* dy, const float* x, float* dw, float* dbias, void* ws, int B, int Ci, int H, int W, int Co,
                                 int KH, int KW, int SH, int x_pitch, int y_pitch, b200asr_stream_t stream) {
  B200_REQUIRE(dy && x && dw && ws, B200ASR_BAD_ARG, "conv2d_tc_bwd_weight: null pointer");
  EmbG g;
  if (int rc = emb_geom(g, "conv2d_tc_bwd_weight", B, Ci, H, W, Co, KH, KW, SH, x_pitch, y_pitch)) return rc;
  B200_REQUIRE(aligned16(dy) && aligned16(x) && aligned16(ws), B200ASR_BAD_ALIGN, "conv2d_tc_bwd_weight: alignment");
  cudaStream_t st = (cudaStream_t)stream;
  CUtensorMap mx, mdy;
  float* xs = (float*)ws + weight_floats(KH, KW);
  if (int rc = make_shifted(x, xs, B, H, W, x_pitch, st)) return rc;
  if (int rc = nchw_map(&mx, xs, shift_pitch(W), shift_pitch(W), H, 4 * B)) return rc;
  if (int rc = nchw_map(&mdy, dy, g.OW, y_pitch, g.OH, B)) return rc;
  EmbWgP e{nullptr, g, ceil_div(KW, 4), 1, B * g.OH, ceil_div(g.OW, 32)};
  const int base = KH * e.m_tiles, rows = B * g.OH;
  int splits = max(1, (3 * device_sm_count()) / base);
  e.rows_per_split = max(8, ceil_div(rows, splits));
  e.splits = ceil_div(rows, e.rows_per_split);
  const size_t wn = (size_t)EC * EC * KH * KW;
  e.part = (float*)stream_scratch(sizeof(float) * ((size_t)e.splits * wn + EMB_BIAS_SPLITS * EC), st);
  if (!e.part) return B200ASR_CUDA_ERROR;
  EmbWgradPolicy::Params p{e};
  int rc = launch_engine<EmbWgradPolicy, 3>(mx, mdy, p, base * e.splits, st, "conv2d_tc_wgrad");
  if (rc || (rc = reduce_parts(e.part, e.splits, (long long)wn, (long long)wn, dw, 0, st))) return rc;
  if (dbias) {
    float* bpart = e.part + (size_t)e.splits * wn;
    emb_bias_grad_kernel<<<dim3(EMB_BIAS_SPLITS, EC), 256, 0, st>>>(dy, bpart, B, g.OH, g.OW, y_pitch);
    if ((rc = check_launch("conv2d_tc_bias_grad"))) return rc;
    return reduce_parts(bpart, EMB_BIAS_SPLITS, EC, EC, dbias, 0, st);
  }
  return B200ASR_OK;
}

size_t b200asr_conv2d_c1_tc_ws_bytes(int B, int H, int W, int KH, int KW) {
  if (B <= 0 || H <= 0 || W <= 0 || KH <= 0 || KW <= 0) return 0;
  return sizeof(float) * (emb1_weight_floats(KH, KW) + emb1_copy_floats(B, H, W));
}

int b200asr_conv2d_c1_tc_fwd(const float* x, const float* w, const float* bias, float* y, void* ws, int B, int H, int W, int Co, int KH,
                             int KW, int PW, int y_pitch, int precision, b200asr_stream_t stream) {
  B200_REQUIRE(x && w && y && ws, B200ASR_BAD_ARG, "conv2d_c1_tc_fwd: null pointer");
  B200_REQUIRE(precision == 3 || precision == 6 || precision == 2, B200ASR_BAD_ARG, "conv2d_c1_tc_fwd: precision must be 3, 6 or 2");
  Emb1G g;
  if (int rc = emb1_geom(g, "conv2d_c1_tc_fwd", B, H, W, Co, KH, KW, PW)) return rc;
  B200_REQUIRE(y_pitch >= g.OW, B200ASR_BAD_SHAPE, "conv2d_c1_tc_fwd: y pitch %d does not cover OW=%d", y_pitch, g.OW);
  B200_REQUIRE(aligned16(ws), B200ASR_BAD_ALIGN, "conv2d_c1_tc_fwd: ws needs a 16-byte aligned base");
  cudaStream_t st = (cudaStream_t)stream;
  const int nkblk = ceil_div(KH, 32), rows = KW * nkblk * EC;
  emb1_repack_kernel<<<ceil_div(rows * 32, 256), 256, 0, st>>>(w, ws, KH, KW, nkblk, precision);
  note_launch(1);
  CUtensorMap ma, mb;
  if (int rc = emb1_prepare(&ma, x, (float*)ws + emb1_weight_floats(KH, KW), g, st)) return rc;
  {
    uint64_t dims[2] = {32, (uint64_t)(precision == 2 ? 1 : 2) * rows}, strides[1] = {32};
    uint32_t box[2] = {32, EC};
    int rc = precision == 3 ? make_tensor_map_f32(&mb, ws, 2, dims, strides, box, false) : make_tensor_map_bf16(&mb, ws, 2, dims, strides, box);
    if (rc) return rc;
  }
  Emb1ConvPolicy::Params p{Emb1ConvP{y, bias, g, y_pitch, ceil_div(g.OW, 128), nkblk}};
  const long long tiles = (long long)B * g.OH * p.e.tiles_w;
  if (tiles >= (1LL << 31)) { set_error("conv2d_c1_tc: too many tiles"); return B200ASR_BAD_SHAPE; }
  if (precision == 3) return launch_engine<Emb1ConvPolicy, 3>(ma, mb, p, (int)tiles, st, "conv2d_c1_tc");
  if (precision == 6) return launch_engine<Emb1ConvPolicy, 6>(ma, mb, p, (int)tiles, st, "conv2d_c1_tc");
  return launch_engine<Emb1ConvPolicy, 2>(ma, mb, p, (int)tiles, st, "conv2d_c1_tc");
}

int b200asr_conv2d_c1_tc_bwd_weight(const float* dy, const float* x, float* dw, float* dbias, void* ws, int B, int H, int W, int Co,
                                    int KH, int KW, int PW, int y_pitch, b200asr_stream_t stream) {
  B200_REQUIRE(dy && x && dw && ws, B200ASR_BAD_ARG, "conv2d_c1_tc_bwd_weight: null pointer");
  Emb1G g;
  if (int rc = emb1_geom(g, "conv2d_c1_tc_bwd_weight", B, H, W, Co, KH, KW, PW)) return rc;
  B200_REQUIRE(y_pitch >= g.OW && y_pitch % 4 == 0, B200ASR_BAD_SHAPE,
               "conv2d_c1_tc_bwd_weight: the dy row pitch must be a multiple of 4 floats (TMA) and cover the row (y pitch %d for OW=%d)", y_pitch, g.OW);
  B200_REQUIRE(aligned16(dy) && aligned16(ws), B200ASR_BAD_ALIGN, "conv2d_c1_tc_bwd_weight: dy and ws need 16-byte aligned bases (TMA)");
  cudaStream_t st = (cudaStream_t)stream;
  CUtensorMap mx, mdy;
  if (int rc = emb1_prepare(&mx, x, (float*)ws + emb1_weight_floats(KH, KW), g, st)) return rc;
  if (int rc = nchw_map(&mdy, dy, g.OW, y_pitch, g.OH, B)) return rc;
  Emb1WgP e{nullptr, g, ceil_div(KW, 4), ceil_div(KH, 32), 1, B * g.OH, ceil_div(g.OW, 32)};
  const int base = e.nkblk * e.m_tiles, rows = B * g.OH;
  int splits = max(1, (3 * device_sm_count()) / base);
  e.rows_per_split = max(8, ceil_div(rows, splits));
  e.splits = ceil_div(rows, e.rows_per_split);
  const size_t wn = (size_t)EC * KH * KW;
  e.part = (float*)stream_scratch(sizeof(float) * ((size_t)e.splits * wn + EMB_BIAS_SPLITS * EC), st);
  if (!e.part) return B200ASR_CUDA_ERROR;
  Emb1WgradPolicy::Params p{e};
  int rc = launch_engine<Emb1WgradPolicy, 3>(mx, mdy, p, base * e.splits, st, "conv2d_c1_tc_wgrad");
  if (rc || (rc = reduce_parts(e.part, e.splits, (long long)wn, (long long)wn, dw, 0, st))) return rc;
  if (dbias) {
    float* bpart = e.part + (size_t)e.splits * wn;
    emb_bias_grad_kernel<<<dim3(EMB_BIAS_SPLITS, EC), 256, 0, st>>>(dy, bpart, B, g.OH, g.OW, y_pitch);
    if ((rc = check_launch("conv2d_c1_tc_bias_grad"))) return rc;
    return reduce_parts(bpart, EMB_BIAS_SPLITS, EC, EC, dbias, 0, st);
  }
  return B200ASR_OK;
}

}  // extern "C"
