// LSTM language model forward for beam-search rescoring (utils/lstm_utils.py:105-138, RNNModel("LSTM") :138-201) on sm_90a:
// the prepared weight layout (lstm_prepare), the recurrence as one tile-engine launch per (layer, step) whose epilogue is the
// LSTM cell (LstmCellPolicy), the exact-fp32 token NLL of the logits rows (lm_nll) and the per-sequence sums (lm_seq_sum).
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
// product, or 0 at t = 0), xp = the row's input projection + bias at the same columns; c updated in place (c_prev = 0 when
// `first`), h written.
__device__ __forceinline__ void lstm_cell8(const float (&gates)[32], const float* __restrict__ xp, float* __restrict__ c,
                                           float* __restrict__ h, bool first) {
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
    const float4 a = *reinterpret_cast<const float4*>(c), b = *reinterpret_cast<const float4*>(c + 4);
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
  }
  *reinterpret_cast<float4*>(c) = make_float4(cv[0], cv[1], cv[2], cv[3]);
  *reinterpret_cast<float4*>(c + 4) = make_float4(cv[4], cv[5], cv[6], cv[7]);
  *reinterpret_cast<float4*>(h) = make_float4(hv[0], hv[1], hv[2], hv[3]);
  *reinterpret_cast<float4*>(h + 4) = make_float4(hv[4], hv[5], hv[6], hv[7]);
}

namespace tc {

// One step t >= 1 of one layer: gates = h_{t-1}[0:M] W_hh^T (M x 4H, K = H) on the tile engine (bf16x3, W_hh pre-converted),
// the cell applied by the epilogue to each 32-column piece.  No split-K: the cell needs the whole sum.
struct LstmCellPolicy {
  static constexpr int BN = 128, kABytes = 128 * 32 * 4, kBBytes = 128 * 32 * 4;
  static constexpr bool kSplitA = true, kSplitB = false, kAMN = false, kBMN = false, kSumA = false, kSumB = false;
  struct Params {
    const float* xproj;    // [M][4H] rows of step t: input projection + folded bias, gate-interleaved
    float* c;              // [>= M][H] cell state, updated in place
    float* h;              // [M][H] h_t (rows of step t of the packed output)
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
    lstm_cell8(v, p.xproj + (size_t)row * 4 * p.H + col, p.c + (size_t)row * p.H + u0, p.h + (size_t)row * p.H + u0, false);
  }
};

}  // namespace tc

// Step 0 of a layer (zero state, no recurrent product): one thread per (row, group of 8 units).
__global__ void lstm_cell0_kernel(const float* __restrict__ xproj, float* __restrict__ c, float* __restrict__ h, int M, int H) {
  const int G = H / 8;
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= (long long)M * G) return;
  const int row = (int)(e / G), u0 = (int)(e - (long long)row * G) * 8;
  float zero[32];
#pragma unroll
  for (int j = 0; j < 32; j++) zero[j] = 0.f;
  lstm_cell8(zero, xproj + (size_t)row * 4 * H + 4 * u0, c + (size_t)row * H + u0, h + (size_t)row * H + u0, true);
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
  cudaStream_t st = (cudaStream_t)stream;
  const int N = 4 * H;
  lstm_cell0_kernel<<<ceil_div(batch_sizes[0] * (H / 8), 128), 128, 0, st>>>(xproj, c, h, batch_sizes[0], H);
  if (int rc = check_launch("lstm_cell0")) return rc;
  CUtensorMap mb;
  {
    uint64_t dims[2] = {(uint64_t)H, (uint64_t)2 * N}, strides[1] = {(uint64_t)H};
    uint32_t box[2] = {32, 128};
    if (int rc = tc::make_tensor_map_bf16(&mb, w_hh_split, 2, dims, strides, box)) return rc;
  }
  long long prev = 0, cur = batch_sizes[0];          // packed row offsets of steps t - 1 and t
  for (int t = 1; t < T; t++) {
    const int M = batch_sizes[t];
    CUtensorMap ma;
    uint64_t dims[2] = {(uint64_t)H, (uint64_t)M}, strides[1] = {(uint64_t)H};
    uint32_t box[2] = {32, 128};
    if (int rc = tc::make_tensor_map_f32(&ma, h + prev * H, 2, dims, strides, box, false)) return rc;
    tc::LstmCellPolicy::Params p{xproj + cur * N, c, h + cur * H, M, H, ceil_div(N, 128)};
    if (int rc = tc::launch_engine<tc::LstmCellPolicy, 6>(ma, mb, p, ceil_div(M, 128) * p.tiles_n, st, "lstm_cell")) return rc;
    prev = cur;
    cur += M;
  }
  return B200ASR_OK;
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
