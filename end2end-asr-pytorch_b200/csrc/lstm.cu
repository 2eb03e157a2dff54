// LSTM language model (utils/lstm_utils.py:105-138, RNNModel("LSTM") :138-201) on sm_90a: the prepared weight layout
// (lstm_prepare) and its inverse for gradients (lstm_grad_unprepare), the recurrence as one tile-engine launch per (layer,
// step) whose epilogue is the LSTM cell (LstmCellPolicyT: rescoring, and training with the gates and cell states saved),
// the backward recurrence with the cell backward in the epilogue (LstmCellBwdPolicy), the dropout between layers
// (lstm_dropout), the exact-fp32 token NLL of the logits rows (lm_nll) and the per-sequence sums (lm_seq_sum).
//
// Layout.  H = nhid and I = ninp rounded up to multiples of 8 (16-byte bf16 row pitches for TMA).  The gate rows of W_ih / W_hh
// are interleaved -- prepared row 4u + g holds gate g (PyTorch order i, f, g, o) of unit u -- so that every 32 consecutive
// output columns of a GEMM against them carry all four gates of 8 units and the cell needs nothing outside its 32-column
// epilogue piece.  Padded rows, columns and bias entries are 0: a padded unit sees i = f = o = 1/2, g = 0, so c and h stay 0.
// Sequences are packed t-major in descending length order: position off[t] + s is step t of sequence s, M_t sequences are
// live at step t (M_t non-increasing), so step t reads rows 0 .. M_t - 1 of step t - 1 and every read is in bounds.
#include <math.h>

#include "../../include/b200asr.h"
#include "common.cuh"
#include "tc_common.cuh"
#include "tc_engine.cuh"

namespace b200asr {

__device__ __forceinline__ float lstm_sigmoid(float x) { return 1.f / (1.f + expf(-x)); }

// Cell of 8 consecutive units u0 .. u0+7 of one row: gates[4q + g] = pre-activation of gate g of unit u0 + q (recurrent
// product, or 0 at t = 0), xp = the row's input projection + bias at the same columns; c_prev read (0 when `first`), c
// written (c == c_prev: in place), h written.  SAVE: the activated gates i, f, g, o go to gsave (the same 32 interleaved
// columns), for the backward recurrence.
template <bool SAVE>
__device__ __forceinline__ void lstm_cell8(const float (&gates)[32], const float* __restrict__ xp, const float* c_prev, float* c,
                                           float* __restrict__ h, float* __restrict__ gsave, bool first) {
  float xv[32];
#pragma unroll
  for (int j = 0; j < 8; j++) {
    const float4 t = *reinterpret_cast<const float4*>(xp + 4 * j);
    xv[4 * j] = t.x; xv[4 * j + 1] = t.y; xv[4 * j + 2] = t.z; xv[4 * j + 3] = t.w;
  }
  float cv[8], hv[8];
  if (first) {
#pragma unroll
    for (int q = 0; q < 8; q++) cv[q] = 0.f;
  } else {
    const float4 a = *reinterpret_cast<const float4*>(c_prev), b = *reinterpret_cast<const float4*>(c_prev + 4);
    cv[0] = a.x; cv[1] = a.y; cv[2] = a.z; cv[3] = a.w; cv[4] = b.x; cv[5] = b.y; cv[6] = b.z; cv[7] = b.w;
  }
#pragma unroll
  for (int q = 0; q < 8; q++) {
    const float gi = lstm_sigmoid(gates[4 * q] + xv[4 * q]);
    const float gf = lstm_sigmoid(gates[4 * q + 1] + xv[4 * q + 1]);
    const float gg = tanhf(gates[4 * q + 2] + xv[4 * q + 2]);
    const float go = lstm_sigmoid(gates[4 * q + 3] + xv[4 * q + 3]);
    cv[q] = gf * cv[q] + gi * gg;
    hv[q] = go * tanhf(cv[q]);
    if constexpr (SAVE) *reinterpret_cast<float4*>(gsave + 4 * q) = make_float4(gi, gf, gg, go);
  }
  *reinterpret_cast<float4*>(c) = make_float4(cv[0], cv[1], cv[2], cv[3]);
  *reinterpret_cast<float4*>(c + 4) = make_float4(cv[4], cv[5], cv[6], cv[7]);
  *reinterpret_cast<float4*>(h) = make_float4(hv[0], hv[1], hv[2], hv[3]);
  *reinterpret_cast<float4*>(h + 4) = make_float4(hv[4], hv[5], hv[6], hv[7]);
}

// Backward of the cell for 8 consecutive units u0 .. u0+7 of one row at step t, on the activations the forward saved:
// g = the 32 saved gates of the units (i, f, g, o interleaved), f_next = the saved gates of step t + 1 at the same columns
// (NULL at t = T - 1), c = c_t, c_prev = c_{t-1} (NULL: zero), dh_out = the gradient of h_t from above, dh_rec = the
// recurrent part dgates_{t+1} W_hh (or the gradient of h_n at t = T - 1).  dc holds dc_{t+1} (the gradient of c_n at T - 1)
// and is overwritten with dc_t; dg gets the pre-activation gradients di, df, dg, do.  Exact fp32.
__device__ __forceinline__ void lstm_cell8_bwd(const float (&dh_rec)[8], const float* __restrict__ g, const float* __restrict__ f_next,
                                               const float* __restrict__ c, const float* __restrict__ c_prev,
                                               const float* __restrict__ dh_out, float* __restrict__ dc, float* __restrict__ dg) {
  float cv[8], cp[8], dho[8], dcv[8];
  {
    const float4 a = *reinterpret_cast<const float4*>(c), b = *reinterpret_cast<const float4*>(c + 4);
    cv[0] = a.x; cv[1] = a.y; cv[2] = a.z; cv[3] = a.w; cv[4] = b.x; cv[5] = b.y; cv[6] = b.z; cv[7] = b.w;
  }
  if (c_prev) {
    const float4 a = *reinterpret_cast<const float4*>(c_prev), b = *reinterpret_cast<const float4*>(c_prev + 4);
    cp[0] = a.x; cp[1] = a.y; cp[2] = a.z; cp[3] = a.w; cp[4] = b.x; cp[5] = b.y; cp[6] = b.z; cp[7] = b.w;
  } else {
#pragma unroll
    for (int q = 0; q < 8; q++) cp[q] = 0.f;
  }
  {
    const float4 a = *reinterpret_cast<const float4*>(dh_out), b = *reinterpret_cast<const float4*>(dh_out + 4);
    dho[0] = a.x; dho[1] = a.y; dho[2] = a.z; dho[3] = a.w; dho[4] = b.x; dho[5] = b.y; dho[6] = b.z; dho[7] = b.w;
  }
  {
    const float4 a = *reinterpret_cast<const float4*>(dc), b = *reinterpret_cast<const float4*>(dc + 4);
    dcv[0] = a.x; dcv[1] = a.y; dcv[2] = a.z; dcv[3] = a.w; dcv[4] = b.x; dcv[5] = b.y; dcv[6] = b.z; dcv[7] = b.w;
  }
#pragma unroll
  for (int q = 0; q < 8; q++) {
    const float4 a = *reinterpret_cast<const float4*>(g + 4 * q);          // i, f, g, o of unit u0 + q
    const float dh = dh_rec[q] + dho[q];
    const float tc = tanhf(cv[q]);
    const float dcn = f_next ? dcv[q] * f_next[4 * q + 1] : dcv[q];
    const float dct = dcn + dh * a.w * (1.f - tc * tc);
    dcv[q] = dct;
    *reinterpret_cast<float4*>(dg + 4 * q) = make_float4(dct * a.z * a.x * (1.f - a.x), dct * cp[q] * a.y * (1.f - a.y),
                                                         dct * a.x * (1.f - a.z * a.z), dh * tc * a.w * (1.f - a.w));
  }
  *reinterpret_cast<float4*>(dc) = make_float4(dcv[0], dcv[1], dcv[2], dcv[3]);
  *reinterpret_cast<float4*>(dc + 4) = make_float4(dcv[4], dcv[5], dcv[6], dcv[7]);
}

namespace tc {

// One step of one layer: gates = h_{t-1}[0:M] W_hh^T (M x 4H, K = H) on the tile engine (bf16x3, W_hh pre-converted),
// the cell applied by the epilogue to each 32-column piece.  No split-K: the cell needs the whole sum.  kSave (training):
// c_t goes to its own buffer (c_prev = c_{t-1}) and the activated gates are saved; without it c is updated in place.
template <bool kSave>
struct LstmCellPolicyT {
  static constexpr int BN = 128, kABytes = 128 * 32 * 4, kBBytes = 128 * 32 * 4;
  static constexpr bool kSplitA = true, kSplitB = false, kAMN = false, kBMN = false, kSumA = false, kSumB = false;
  struct Params {
    const float* xproj;    // [M][4H] rows of step t: input projection + folded bias, gate-interleaved
    const float* c_prev;   // [>= M][H] cell state of step t - 1
    float* c;              // [>= M][H] cell state of step t (== c_prev without kSave)
    float* h;              // [M][H] h_t (rows of step t of the packed output)
    float* gates;          // kSave: [M][4H] activated gates of step t
    int M, H, tiles_n;
  };
  static __device__ __forceinline__ int num_tiles(const Params& p) { return ((p.M + 127) / 128) * p.tiles_n; }
  static __device__ __forceinline__ int num_kb(const Params& p, int) { return (p.H + 31) / 32; }
  struct Tile { int m0, n0, k0; };
  static __device__ __forceinline__ Tile tile(const Params& p, int tile) {
    Tile t;
    t.m0 = (tile / p.tiles_n) * 128; t.n0 = (tile % p.tiles_n) * 128; t.k0 = 0;
    return t;
  }
  static __device__ __forceinline__ void load16(const Params& p, Tile& t, const CUtensorMap* mapA, const CUtensorMap* mapB,
                                                uint32_t sa, uint32_t sb, uint32_t sb_lo, uint32_t bar, bool leader, int halves) {
    const int k0 = t.k0;
    t.k0 += 32;
    if (!leader) return;
    tma_load_2d(sa, mapA, bar, k0, t.m0);
    tma_load_2d(sb, mapB, bar, k0, t.n0);
    if (halves == 2) tma_load_2d(sb_lo, mapB, bar, k0, t.n0 + 4 * p.H);     // lo half: rows 4H .. 8H - 1 of the operand
  }
  static __device__ __forceinline__ void store(const Params& p, const Tile& t, int r, int c0, const float (&v)[32]) {
    const int row = t.m0 + r, col = t.n0 + c0;
    if (row >= p.M || col >= 4 * p.H) return;
    const int u0 = col >> 2;
    lstm_cell8<kSave>(v, p.xproj + (size_t)row * 4 * p.H + col, p.c_prev + (size_t)row * p.H + u0, p.c + (size_t)row * p.H + u0,
                      p.h + (size_t)row * p.H + u0, kSave ? p.gates + (size_t)row * 4 * p.H + col : nullptr, false);
  }
};
using LstmCellPolicy = LstmCellPolicyT<false>;
using LstmCellTrainPolicy = LstmCellPolicyT<true>;

// One step t <= T - 2 of the backward recurrence of one layer: dh_rec = dgates_{t+1}[0:M] W_hh_p (M x H, K = 4H) on the tile
// engine (bf16x3; B = the transposed operand [H][4H] of b200asr_split_bf16), the cell backward in the epilogue.  An
// epilogue piece covers 32 units, whose saved gates are 128 contiguous columns of the interleaved layout; it is handled as
// four groups of 8 units.
struct LstmCellBwdPolicy {
  static constexpr int BN = 128, kABytes = 128 * 32 * 4, kBBytes = 128 * 32 * 4;
  static constexpr bool kSplitA = true, kSplitB = false, kAMN = false, kBMN = false, kSumA = false, kSumB = false;
  struct Params {
    const float* gates;    // [M][4H] saved gates of step t
    const float* f_next;   // [M][4H] saved gates of step t + 1
    const float* c;        // [M][H] c_t
    const float* c_prev;   // [M][H] c_{t-1}, NULL = zero (t = 0 from a zero state)
    const float* dh_out;   // [M][H] gradient of h_t from the layer above / the decoder
    float* dc;             // [M][H] dc_{t+1} in, dc_t out
    float* dgates;         // [M][4H] dgates_t
    int M, H, tiles_n;
  };
  static __device__ __forceinline__ int num_tiles(const Params& p) { return ((p.M + 127) / 128) * p.tiles_n; }
  static __device__ __forceinline__ int num_kb(const Params& p, int) { return p.H / 8; }       // 4H / 32
  struct Tile { int m0, n0, k0; };
  static __device__ __forceinline__ Tile tile(const Params& p, int tile) {
    Tile t;
    t.m0 = (tile / p.tiles_n) * 128; t.n0 = (tile % p.tiles_n) * 128; t.k0 = 0;
    return t;
  }
  static __device__ __forceinline__ void load16(const Params& p, Tile& t, const CUtensorMap* mapA, const CUtensorMap* mapB,
                                                uint32_t sa, uint32_t sb, uint32_t sb_lo, uint32_t bar, bool leader, int halves) {
    const int k0 = t.k0;
    t.k0 += 32;
    if (!leader) return;
    tma_load_2d(sa, mapA, bar, k0, t.m0);
    tma_load_2d(sb, mapB, bar, k0, t.n0);
    if (halves == 2) tma_load_2d(sb_lo, mapB, bar, k0, t.n0 + p.H);         // lo half: rows H .. 2H - 1 of the operand
  }
  static __device__ __forceinline__ void store(const Params& p, const Tile& t, int r, int c0, const float (&v)[32]) {
    const int row = t.m0 + r, col = t.n0 + c0;
    if (row >= p.M) return;
    const size_t rh = (size_t)row * p.H, rg = (size_t)row * 4 * p.H;
#pragma unroll
    for (int j = 0; j < 4; j++) {
      const int u0 = col + 8 * j;
      if (u0 >= p.H) return;
      float d[8];
#pragma unroll
      for (int q = 0; q < 8; q++) d[q] = v[8 * j + q];
      lstm_cell8_bwd(d, p.gates + rg + 4 * u0, p.f_next + rg + 4 * u0, p.c + rh + u0, p.c_prev ? p.c_prev + rh + u0 : nullptr,
                     p.dh_out + rh + u0, p.dc + rh + u0, p.dgates + rg + 4 * u0);
    }
  }
};

}  // namespace tc

// Step 0 of a layer from the zero state (no recurrent product): one thread per (row, group of 8 units).
template <bool SAVE>
__global__ void lstm_cell0_kernel(const float* __restrict__ xproj, float* __restrict__ c, float* __restrict__ h,
                                  float* __restrict__ gsave, int M, int H) {
  const int G = H / 8;
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= (long long)M * G) return;
  const int row = (int)(e / G), u0 = (int)(e - (long long)row * G) * 8;
  float zero[32];
#pragma unroll
  for (int j = 0; j < 32; j++) zero[j] = 0.f;
  lstm_cell8<SAVE>(zero, xproj + (size_t)row * 4 * H + 4 * u0, c + (size_t)row * H + u0, c + (size_t)row * H + u0,
                   h + (size_t)row * H + u0, SAVE ? gsave + (size_t)row * 4 * H + 4 * u0 : nullptr, true);
}

// Step T - 1 of the backward recurrence (no later step): dh_rec = the gradient of h_n (NULL: 0), dc_{t+1} = the gradient
// of c_n (NULL: 0) copied into dc first.  One thread per (row, group of 8 units).
__global__ void lstm_bwd_last_kernel(const float* __restrict__ gates, const float* __restrict__ c, const float* __restrict__ c_prev,
                                     const float* __restrict__ dh_out, const float* __restrict__ dh_n, const float* __restrict__ dc_n,
                                     float* __restrict__ dc, float* __restrict__ dgates, int M, int H) {
  const int G = H / 8;
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= (long long)M * G) return;
  const int row = (int)(e / G), u0 = (int)(e - (long long)row * G) * 8;
  const size_t rh = (size_t)row * H + u0, rg = (size_t)row * 4 * H + 4 * u0;
  float d[8];
#pragma unroll
  for (int q = 0; q < 8; q++) {
    d[q] = dh_n ? dh_n[rh + q] : 0.f;
    dc[rh + q] = dc_n ? dc_n[rh + q] : 0.f;
  }
  lstm_cell8_bwd(d, gates + rg, nullptr, c + rh, c_prev ? c_prev + rh : nullptr, dh_out + rh, dc + rh, dgates + rg);
}

// dc0 = dc_0 * f_0: the gradient of the initial cell state.
__global__ void lstm_dc0_kernel(const float* __restrict__ dc, const float* __restrict__ gates0, float* __restrict__ dc0, int M, int H) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= (long long)M * H) return;
  const long long row = e / H, u = e - row * H;
  dc0[e] = dc[e] * gates0[row * 4 * H + 4 * u + 1];
}

// y = x * mask * 1/(1-p) with the counter-based generator (common.cuh) keyed by (seed, offset), element index i: the same
// call on a gradient applies the forward's mask again.  Four elements per thread.
__global__ void lstm_dropout_kernel(const float* __restrict__ x, float* __restrict__ y, long long n4, uint32_t thresh, float inv_keep,
                                    uint64_t key) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n4) return;
  float4 a = reinterpret_cast<const float4*>(x)[i];
  const uint64_t r = dropout_bits4(key, (uint64_t)i);
  a.x = ((uint32_t)(r) & 0xFFFFu) >= thresh ? a.x * inv_keep : 0.f;
  a.y = ((uint32_t)(r >> 16) & 0xFFFFu) >= thresh ? a.y * inv_keep : 0.f;
  a.z = ((uint32_t)(r >> 32) & 0xFFFFu) >= thresh ? a.z * inv_keep : 0.f;
  a.w = ((uint32_t)(r >> 48) & 0xFFFFu) >= thresh ? a.w * inv_keep : 0.f;
  reinterpret_cast<float4*>(y)[i] = a;
}

// Inverse of lstm_prepare for gradients: block x = PyTorch row g * nhid + u <- prepared row 4u + g, padding dropped.
__global__ void lstm_grad_unprepare_kernel(const float* __restrict__ dw_ih_p, const float* __restrict__ dw_hh_p,
                                           const float* __restrict__ db_p, int ninp, int nhid, int I, int H, float* __restrict__ dw_ih,
                                           float* __restrict__ dw_hh, float* __restrict__ db_ih, float* __restrict__ db_hh) {
  const int r = blockIdx.x, g = r / nhid, u = r - g * nhid;
  const size_t pr = 4 * (size_t)u + g;
  if (dw_ih)
    for (int j = threadIdx.x; j < ninp; j += blockDim.x) dw_ih[(size_t)r * ninp + j] = dw_ih_p[pr * I + j];
  if (dw_hh)
    for (int k = threadIdx.x; k < nhid; k += blockDim.x) dw_hh[(size_t)r * nhid + k] = dw_hh_p[pr * H + k];
  if (threadIdx.x == 0) {
    if (db_ih) db_ih[r] = db_p[pr];
    if (db_hh) db_hh[r] = db_p[pr];
  }
}

// The recurrence of one layer, shared by rescoring (kSave = false: packed ragged batches, c in place, zero state) and
// training (kSave: fixed batch B = batch_sizes[t], c_t and the gates of every step kept).  Step t's rows start at packed row
// offset `cur` of xproj / h (and of c and gates with kSave); h_{t-1} is read from the previous step's rows, which for t = 0
// with a given state is the slot of h0 just before h.
template <bool kSave>
static int lstm_recurrence(const float* xproj, const void* w_hh_split, const int32_t* batch_sizes, int B, int T, int H, bool has_state,
                           const float* c0, float* c, float* h, float* gates, cudaStream_t st) {
  using Policy = tc::LstmCellPolicyT<kSave>;
  const int N = 4 * H;
  CUtensorMap mb;
  {
    uint64_t dims[2] = {(uint64_t)H, (uint64_t)2 * N}, strides[1] = {(uint64_t)H};
    uint32_t box[2] = {32, 128};
    if (int rc = tc::make_tensor_map_bf16(&mb, w_hh_split, 2, dims, strides, box)) return rc;
  }
  long long prev = 0, cur = 0;                       // packed row offsets of steps t - 1 and t
  for (int t = 0; t < T; t++) {
    const int M = batch_sizes ? batch_sizes[t] : B;
    float* c_out = kSave ? c + cur * H : c;
    float* g_out = kSave ? gates + cur * N : nullptr;
    if (t == 0 && !has_state) {
      lstm_cell0_kernel<kSave><<<ceil_div(M * (H / 8), 128), 128, 0, st>>>(xproj, c_out, h, g_out, M, H);
      if (int rc = check_launch("lstm_cell0")) return rc;
    } else {
      const float* a = t == 0 ? h - (long long)M * H : h + prev * H;
      const float* c_prev = !kSave ? c : (t == 0 ? c0 : c + prev * H);
      CUtensorMap ma;
      uint64_t dims[2] = {(uint64_t)H, (uint64_t)M}, strides[1] = {(uint64_t)H};
      uint32_t box[2] = {32, 128};
      if (int rc = tc::make_tensor_map_f32(&ma, a, 2, dims, strides, box, false)) return rc;
      typename Policy::Params p{xproj + cur * N, c_prev, c_out, h + cur * H, g_out, M, H, ceil_div(N, 128)};
      if (int rc = tc::launch_engine<Policy, 6>(ma, mb, p, ceil_div(M, 128) * p.tiles_n, st, "lstm_cell")) return rc;
    }
    prev = cur;
    cur += M;
  }
  return B200ASR_OK;
}

// Prepared operands of one layer: w_ih_p [4H][I], w_hh_p [4H][H] gate-interleaved and zero padded, bias_p [4H] = b_ih + b_hh.
// Block y = prepared row; threads stride over the I + H columns of both matrices.
__global__ void lstm_prepare_kernel(const float* __restrict__ w_ih, const float* __restrict__ w_hh, const float* __restrict__ b_ih,
                                    const float* __restrict__ b_hh, int ninp, int nhid, int I, int H, float* __restrict__ w_ih_p,
                                    float* __restrict__ w_hh_p, float* __restrict__ bias_p) {
  const int pr = blockIdx.x, u = pr >> 2, g = pr & 3;
  const bool real = u < nhid;
  const size_t src = (size_t)g * nhid + u;
  for (int j = threadIdx.x; j < I + H; j += blockDim.x) {
    if (j < I) w_ih_p[(size_t)pr * I + j] = (real && j < ninp) ? w_ih[src * ninp + j] : 0.f;
    else {
      const int k = j - I;
      w_hh_p[(size_t)pr * H + k] = (real && k < nhid) ? w_hh[src * nhid + k] : 0.f;
    }
  }
  if (threadIdx.x == 0) bias_p[pr] = real ? (b_ih ? b_ih[src] : 0.f) + (b_hh ? b_hh[src] : 0.f) : 0.f;
}

// One CTA per row: nll = logsumexp(x) - x[target] in exact fp32 (expf / logf); block reductions in a fixed order.
constexpr int NLL_THREADS = 256;
__global__ void __launch_bounds__(NLL_THREADS) lm_nll_kernel(const float* __restrict__ logits, long long ld,
                                                             const int64_t* __restrict__ targets, float* __restrict__ nll, int V) {
  const int row = blockIdx.x;
  const float* x = logits + (size_t)row * ld;
  const RowLse st = block_row_lse<NLL_THREADS, false>(x, V);
  if (threadIdx.x == 0) {
    const int64_t tg = targets[row];
    nll[row] = (tg >= 0 && tg < V) ? (st.mx + logf(st.sumexp)) - x[tg] : NAN;
  }
}

// sums[s] = sum over t < len[s] of nll[off[t] + s], in t order (one thread per sequence).
__global__ void lm_seq_sum_kernel(const float* __restrict__ nll, const int64_t* __restrict__ off, const int64_t* __restrict__ len,
                                  int nseq, float* __restrict__ sums) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= nseq) return;
  float acc = 0.f;
  for (long long t = 0; t < len[s]; t++) acc += nll[off[t] + s];
  sums[s] = acc;
}

}  // namespace b200asr

using namespace b200asr;

extern "C" {

int b200asr_lstm_prepare(const float* w_ih, const float* w_hh, const float* b_ih, const float* b_hh, int ninp, int nhid,
                         float* w_ih_p, float* w_hh_p, float* bias_p, b200asr_stream_t stream) {
  B200_REQUIRE(w_ih && w_hh && w_ih_p && w_hh_p && bias_p, B200ASR_BAD_ARG, "lstm_prepare: null pointer");
  B200_REQUIRE(ninp >= 1 && nhid >= 1, B200ASR_BAD_SHAPE, "lstm_prepare: ninp=%d nhid=%d must be >= 1", ninp, nhid);
  const int I = (ninp + 7) / 8 * 8, H = (nhid + 7) / 8 * 8;
  lstm_prepare_kernel<<<4 * H, 256, 0, (cudaStream_t)stream>>>(w_ih, w_hh, b_ih, b_hh, ninp, nhid, I, H, w_ih_p, w_hh_p, bias_p);
  return check_launch("lstm_prepare");
}

int b200asr_lstm_layer_fwd(const float* xproj, const void* w_hh_split, const int32_t* batch_sizes, int T, int H, float* c, float* h,
                           b200asr_stream_t stream) {
  B200_REQUIRE(xproj && w_hh_split && batch_sizes && c && h, B200ASR_BAD_ARG, "lstm_layer_fwd: null pointer");
  B200_REQUIRE(H >= 8 && H % 8 == 0, B200ASR_BAD_SHAPE, "lstm_layer_fwd: H=%d must be a positive multiple of 8 (pad nhid)", H);
  B200_REQUIRE(T >= 1, B200ASR_BAD_SHAPE, "lstm_layer_fwd: T=%d must be >= 1", T);
  for (int t = 0; t < T; t++)
    B200_REQUIRE(batch_sizes[t] >= 1 && (t == 0 || batch_sizes[t] <= batch_sizes[t - 1]), B200ASR_BAD_SHAPE,
                 "lstm_layer_fwd: batch_sizes[%d]=%d must be >= 1 and non-increasing (sequences sorted by length, descending)", t,
                 batch_sizes[t]);
  B200_REQUIRE(aligned16(xproj) && aligned16(w_hh_split) && aligned16(c) && aligned16(h), B200ASR_BAD_ALIGN,
               "lstm_layer_fwd: xproj, w_hh_split, c and h must be 16-byte aligned");
  return lstm_recurrence<false>(xproj, w_hh_split, batch_sizes, 0, T, H, false, nullptr, c, h, nullptr, (cudaStream_t)stream);
}

int b200asr_lstm_layer_train_fwd(const float* xproj, const void* w_hh_split, int T, int B, int H, int has_state, const float* c0,
                                 float* h, float* c, float* gates, b200asr_stream_t stream) {
  B200_REQUIRE(xproj && w_hh_split && h && c && gates && (!has_state || c0), B200ASR_BAD_ARG, "lstm_layer_train_fwd: null pointer");
  B200_REQUIRE(H >= 8 && H % 8 == 0, B200ASR_BAD_SHAPE, "lstm_layer_train_fwd: H=%d must be a positive multiple of 8 (pad nhid)", H);
  B200_REQUIRE(T >= 1 && B >= 1, B200ASR_BAD_SHAPE, "lstm_layer_train_fwd: T=%d B=%d must be >= 1", T, B);
  B200_REQUIRE(aligned16(xproj) && aligned16(w_hh_split) && aligned16(h) && aligned16(c) && aligned16(gates) && (!has_state || aligned16(c0)),
               B200ASR_BAD_ALIGN, "lstm_layer_train_fwd: xproj, w_hh_split, h, c, c0 and gates must be 16-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  if (!has_state) cudaMemsetAsync(h, 0, sizeof(float) * (size_t)B * H, st);       // h_{-1} = 0 for the dW_hh operand
  return lstm_recurrence<true>(xproj, w_hh_split, nullptr, B, T, H, has_state != 0, c0, c, h + (size_t)B * H, gates, st);
}

int b200asr_lstm_layer_train_bwd(const float* gates, const float* c, const float* c0, const float* dh_out, const float* dh_n,
                                 const float* dc_n, const void* w_hh_split_t, int T, int B, int H, float* dc, float* dgates, float* dc0,
                                 b200asr_stream_t stream) {
  B200_REQUIRE(gates && c && dh_out && w_hh_split_t && dc && dgates, B200ASR_BAD_ARG, "lstm_layer_train_bwd: null pointer");
  B200_REQUIRE(H >= 8 && H % 8 == 0, B200ASR_BAD_SHAPE, "lstm_layer_train_bwd: H=%d must be a positive multiple of 8 (pad nhid)", H);
  B200_REQUIRE(T >= 1 && B >= 1, B200ASR_BAD_SHAPE, "lstm_layer_train_bwd: T=%d B=%d must be >= 1", T, B);
  B200_REQUIRE(aligned16(gates) && aligned16(c) && aligned16(dh_out) && aligned16(w_hh_split_t) && aligned16(dc) && aligned16(dgates) &&
                   (!c0 || aligned16(c0)),
               B200ASR_BAD_ALIGN, "lstm_layer_train_bwd: gates, c, c0, dh_out, w_hh_split_t, dc and dgates must be 16-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  const int N = 4 * H;
  const size_t sh = (size_t)B * H, sg = (size_t)B * N;
  auto c_prev = [&](int t) { return t == 0 ? c0 : c + (t - 1) * sh; };
  lstm_bwd_last_kernel<<<ceil_div(B * (H / 8), 128), 128, 0, st>>>(gates + (T - 1) * sg, c + (T - 1) * sh, c_prev(T - 1),
                                                                   dh_out + (T - 1) * sh, dh_n, dc_n, dc, dgates + (T - 1) * sg, B, H);
  if (int rc = check_launch("lstm_bwd_last")) return rc;
  if (T > 1) {
    CUtensorMap mb;
    {
      uint64_t dims[2] = {(uint64_t)N, (uint64_t)2 * H}, strides[1] = {(uint64_t)N};
      uint32_t box[2] = {32, 128};
      if (int rc = tc::make_tensor_map_bf16(&mb, w_hh_split_t, 2, dims, strides, box)) return rc;
    }
    for (int t = T - 2; t >= 0; t--) {
      CUtensorMap ma;
      uint64_t dims[2] = {(uint64_t)N, (uint64_t)B}, strides[1] = {(uint64_t)N};
      uint32_t box[2] = {32, 128};
      if (int rc = tc::make_tensor_map_f32(&ma, dgates + (t + 1) * sg, 2, dims, strides, box, false)) return rc;
      tc::LstmCellBwdPolicy::Params p{gates + t * sg, gates + (t + 1) * sg, c + t * sh, c_prev(t), dh_out + t * sh, dc,
                                      dgates + t * sg, B, H, ceil_div(H, 128)};
      if (int rc = tc::launch_engine<tc::LstmCellBwdPolicy, 6>(ma, mb, p, ceil_div(B, 128) * p.tiles_n, st, "lstm_cell_bwd")) return rc;
    }
  }
  if (dc0) {
    lstm_dc0_kernel<<<ceil_div(B * H, 256), 256, 0, st>>>(dc, gates, dc0, B, H);
    return check_launch("lstm_dc0");
  }
  return B200ASR_OK;
}

int b200asr_lstm_dropout(const float* x, float* y, long long n, float p, uint64_t seed, uint64_t offset, b200asr_stream_t stream) {
  B200_REQUIRE(x && y, B200ASR_BAD_ARG, "lstm_dropout: null pointer");
  B200_REQUIRE(n >= 0 && n % 4 == 0 && p >= 0.f && p < 1.f, B200ASR_BAD_SHAPE, "lstm_dropout: n=%lld must be a multiple of 4, p=%g in [0, 1)",
               n, (double)p);
  B200_REQUIRE(aligned16(x) && aligned16(y), B200ASR_BAD_ALIGN, "lstm_dropout: x and y must be 16-byte aligned");
  if (n == 0) return B200ASR_OK;
  lstm_dropout_kernel<<<(unsigned)ceil_div_ll(n / 4, 256), 256, 0, (cudaStream_t)stream>>>(
      x, y, n / 4, p > 0.f ? dropout_thresh16(p) : 0u, dropout_inv_keep(p), dropout_key(seed, offset));
  return check_launch("lstm_dropout");
}

int b200asr_lstm_grad_unprepare(const float* dw_ih_p, const float* dw_hh_p, const float* db_p, int ninp, int nhid, float* dw_ih,
                                float* dw_hh, float* db_ih, float* db_hh, b200asr_stream_t stream) {
  B200_REQUIRE((!dw_ih || dw_ih_p) && (!dw_hh || dw_hh_p) && (!(db_ih || db_hh) || db_p), B200ASR_BAD_ARG,
               "lstm_grad_unprepare: an output without its prepared gradient");
  B200_REQUIRE(ninp >= 1 && nhid >= 1, B200ASR_BAD_SHAPE, "lstm_grad_unprepare: ninp=%d nhid=%d must be >= 1", ninp, nhid);
  const int I = (ninp + 7) / 8 * 8, H = (nhid + 7) / 8 * 8;
  lstm_grad_unprepare_kernel<<<4 * nhid, 256, 0, (cudaStream_t)stream>>>(dw_ih_p, dw_hh_p, db_p, ninp, nhid, I, H, dw_ih, dw_hh, db_ih,
                                                                          db_hh);
  return check_launch("lstm_grad_unprepare");
}

int b200asr_lm_nll(const float* logits, long long ld, const int64_t* targets, float* nll, int rows, int V, b200asr_stream_t stream) {
  B200_REQUIRE(logits && targets && nll, B200ASR_BAD_ARG, "lm_nll: null pointer");
  B200_REQUIRE(V >= 1 && ld >= V && rows >= 0, B200ASR_BAD_SHAPE, "lm_nll: rows=%d V=%d ld=%lld (need V >= 1, ld >= V)", rows, V, ld);
  if (rows == 0) return B200ASR_OK;
  lm_nll_kernel<<<rows, NLL_THREADS, 0, (cudaStream_t)stream>>>(logits, ld, targets, nll, V);
  return check_launch("lm_nll");
}

int b200asr_lm_seq_sum(const float* nll, const int64_t* offsets, const int64_t* lengths, int nseq, float* sums,
                       b200asr_stream_t stream) {
  B200_REQUIRE(nll && offsets && lengths && sums, B200ASR_BAD_ARG, "lm_seq_sum: null pointer");
  B200_REQUIRE(nseq >= 0, B200ASR_BAD_SHAPE, "lm_seq_sum: nseq=%d", nseq);
  if (nseq == 0) return B200ASR_OK;
  lm_seq_sum_kernel<<<ceil_div(nseq, 128), 128, 0, (cudaStream_t)stream>>>(nll, offsets, lengths, nseq, sums);
  return check_launch("lm_seq_sum");
}

}  // extern "C"
