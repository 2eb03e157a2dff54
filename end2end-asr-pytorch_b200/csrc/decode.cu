// Single-query attention of a decode step (b200asr_decode_attn): out[r, h] = softmax(scale * q[r,h] . K[r,h]^T) . V[r,h] over
// Tk keys, no mask, exact fp32 on CUDA cores.  The call reads every K/V byte once and does ~2 FLOP per byte, so it is bound
// by HBM / L2 bandwidth: the key range of each (row, head) is split into chunks, one CTA per (row, head, chunk), so that
// even a few hundred (row, head) pairs fill the machine.  Each CTA writes a partial (max, sum, unnormalised o) and a second
// kernel merges the partials in chunk order; with a single chunk the first kernel writes the output itself.
#include <math.h>

#include "../../include/b200asr.h"
#include "common.cuh"

namespace b200asr {

constexpr int DA_THREADS = 128;
constexpr int DA_WARPS = DA_THREADS / 32;
constexpr int DA_KC_MIN = 64;          // keys per chunk, at least
constexpr int DA_KC_MAX = 1024;        // keys per chunk, at most (the chunk's scores live in shared memory)
constexpr int DA_TARGET_CTAS = 1024;   // split until (row, head, chunk) CTAs reach ~8 per SM of an H100 SXM (132 SMs)
constexpr int DA_MAX_TK = 65536;

// Keys per chunk.  A function of (R, H, Tk) only -- never of the device -- so the partials, and hence the bits of the
// merged result, are the same on every call and every card.
static int decode_attn_chunk(int R, int H, int Tk) {
  const long long rh = (long long)R * H;
  const long long want = rh >= DA_TARGET_CTAS ? 1 : DA_TARGET_CTAS / rh;
  long long kc = ((ceil_div_ll(Tk, want) + 31) / 32) * 32;
  if (kc < DA_KC_MIN) kc = DA_KC_MIN;
  if (kc > DA_KC_MAX) kc = DA_KC_MAX;
  return (int)kc;
}

// One CTA per (row r, head h, chunk c) of keys [c * KC, min(Tk, c * KC + KC)).  Scores: DK / 4 lanes per key (one float4
// each), reduced by shuffles; softmax statistics and P.V per CTA in a fixed order.  ws == nullptr: single chunk, the CTA
// writes out = o / sum.  Otherwise it writes ws_m / ws_l [RH][nc] and ws_o [RH][nc][DV].
template <int DK, int DV>
__global__ void __launch_bounds__(DA_THREADS) decode_attn_part_kernel(
    const float* __restrict__ q, const float* __restrict__ k, const float* __restrict__ v, float* __restrict__ out,
    float* __restrict__ ws_m, float* __restrict__ ws_l, float* __restrict__ ws_o, int H, int Tk, int KC, int nc,
    long long k_rs, long long k_ks, long long v_rs, long long v_ks, float scale) {
  __shared__ float sq[DK];
  __shared__ float sp[DA_KC_MAX];
  __shared__ float sred[DA_WARPS];
  __shared__ __align__(16) float so[DA_WARPS][DV];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int g = blockIdx.x / nc, c = blockIdx.x - g * nc;
  const int r = g / H, h = g - r * H;
  const int j0 = c * KC;
  const int n = min(Tk - j0, KC);
  for (int i = tid; i < DK; i += DA_THREADS) sq[i] = q[(size_t)g * DK + i];
  __syncthreads();

  // 1. scores of the chunk's keys into sp
  constexpr int GK = DK / 4, KPW = 32 / GK;            // lanes per key, keys per warp and pass
  const float4 qv = reinterpret_cast<const float4*>(sq)[lane % GK];
  const float* kb = k + r * k_rs + (long long)j0 * k_ks + h * DK + 4 * (lane % GK);
#pragma unroll 4
  for (int base = warp * KPW; base < n; base += DA_WARPS * KPW) {
    const int jj = base + lane / GK;
    float s = 0.f;
    if (jj < n) {
      const float4 kv = *reinterpret_cast<const float4*>(kb + jj * k_ks);
      s = qv.x * kv.x + qv.y * kv.y + qv.z * kv.z + qv.w * kv.w;
    }
#pragma unroll
    for (int o = GK / 2; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (jj < n && lane % GK == 0) sp[jj] = s * scale;
  }
  __syncthreads();

  // 2. max, exp, sum (fixed order: per thread, then lanes, then warps 0..3)
  float mx = -INFINITY;
  for (int j = tid; j < n; j += DA_THREADS) mx = fmaxf(mx, sp[j]);
  mx = warp_max(mx);
  if (lane == 0) sred[warp] = mx;
  __syncthreads();
  mx = sred[0];
#pragma unroll
  for (int w = 1; w < DA_WARPS; w++) mx = fmaxf(mx, sred[w]);
  __syncthreads();
  float sum = 0.f;
  for (int j = tid; j < n; j += DA_THREADS) {
    const float e = expf(sp[j] - mx);
    sp[j] = e;
    sum += e;
  }
  sum = warp_sum(sum);
  if (lane == 0) sred[warp] = sum;
  __syncthreads();
  sum = sred[0];
#pragma unroll
  for (int w = 1; w < DA_WARPS; w++) sum += sred[w];

  // 3. o = sum_j p_j v_j: DV / 4 lanes per key (one float4 each), then the key groups of a warp, then the warps
  constexpr int GV = DV / 4, VPW = 32 / GV;
  const float* vb = v + r * v_rs + (long long)j0 * v_ks + h * DV + 4 * (lane % GV);
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll 4
  for (int jj = warp * VPW + lane / GV; jj < n; jj += DA_WARPS * VPW) {
    const float4 vv = *reinterpret_cast<const float4*>(vb + jj * v_ks);
    const float p = sp[jj];
    acc.x += p * vv.x; acc.y += p * vv.y; acc.z += p * vv.z; acc.w += p * vv.w;
  }
#pragma unroll
  for (int o = GV; o < 32; o <<= 1) {
    acc.x += __shfl_xor_sync(0xffffffffu, acc.x, o);
    acc.y += __shfl_xor_sync(0xffffffffu, acc.y, o);
    acc.z += __shfl_xor_sync(0xffffffffu, acc.z, o);
    acc.w += __shfl_xor_sync(0xffffffffu, acc.w, o);
  }
  if (lane < GV) reinterpret_cast<float4*>(so[warp])[lane] = acc;
  __syncthreads();
  for (int i = tid; i < DV; i += DA_THREADS) {
    float o = so[0][i];
#pragma unroll
    for (int w = 1; w < DA_WARPS; w++) o += so[w][i];
    if (ws_o == nullptr) {
      out[(size_t)g * DV + i] = o / sum;
    } else {
      ws_o[((size_t)g * nc + c) * DV + i] = o;
    }
  }
  if (ws_o != nullptr && tid == 0) {
    ws_m[(size_t)g * nc + c] = mx;
    ws_l[(size_t)g * nc + c] = sum;
  }
}

// One warp per (row, head): out = sum_c e^(m_c - M) o_c / sum_c e^(m_c - M) l_c, M = max_c m_c, summed in chunk order.
template <int DV>
__global__ void __launch_bounds__(DA_THREADS) decode_attn_merge_kernel(const float* __restrict__ ws_m,
                                                                      const float* __restrict__ ws_l,
                                                                      const float* __restrict__ ws_o, float* __restrict__ out,
                                                                      int RH, int nc) {
  const int g = blockIdx.x * DA_WARPS + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (g >= RH) return;
  const float* m = ws_m + (size_t)g * nc;
  const float* l = ws_l + (size_t)g * nc;
  const float* o = ws_o + (size_t)g * nc * DV;
  float M = -INFINITY;
  for (int c = 0; c < nc; c++) M = fmaxf(M, m[c]);
  constexpr int NA = DV >= 32 ? DV / 32 : 1;
  float acc[NA];
#pragma unroll
  for (int a = 0; a < NA; a++) acc[a] = 0.f;
  float den = 0.f;
  for (int c = 0; c < nc; c++) {
    const float w = expf(m[c] - M);
    den += w * l[c];
#pragma unroll
    for (int a = 0; a < NA; a++)
      if (a * 32 + lane < DV) acc[a] += w * o[(size_t)c * DV + a * 32 + lane];
  }
#pragma unroll
  for (int a = 0; a < NA; a++)
    if (a * 32 + lane < DV) out[(size_t)g * DV + a * 32 + lane] = acc[a] / den;
}

template <int DK, int DV>
static int launch_decode_attn(const float* q, const float* k, const float* v, float* out, float* ws, int R, int H, int Tk,
                              long long k_rs, long long k_ks, long long v_rs, long long v_ks, float scale, cudaStream_t st) {
  const int KC = decode_attn_chunk(R, H, Tk);
  const int nc = ceil_div(Tk, KC);
  const int RH = R * H;
  float *ws_m = nullptr, *ws_l = nullptr, *ws_o = nullptr;
  if (nc > 1) {
    ws_m = ws;
    ws_l = ws + (size_t)RH * nc;
    ws_o = ws + (size_t)2 * RH * nc;
  }
  decode_attn_part_kernel<DK, DV><<<RH * nc, DA_THREADS, 0, st>>>(q, k, v, out, ws_m, ws_l, ws_o, H, Tk, KC, nc, k_rs, k_ks,
                                                                  v_rs, v_ks, scale);
  if (int rc = check_launch("decode_attn")) return rc;
  if (nc == 1) return B200ASR_OK;
  decode_attn_merge_kernel<DV><<<ceil_div(RH, DA_WARPS), DA_THREADS, 0, st>>>(ws_m, ws_l, ws_o, out, RH, nc);
  return check_launch("decode_attn_merge");
}

template <int DK>
static int launch_decode_attn_dv(int dv, const float* q, const float* k, const float* v, float* out, float* ws, int R, int H,
                                 int Tk, long long k_rs, long long k_ks, long long v_rs, long long v_ks, float scale,
                                 cudaStream_t st) {
  switch (dv) {
    case 16: return launch_decode_attn<DK, 16>(q, k, v, out, ws, R, H, Tk, k_rs, k_ks, v_rs, v_ks, scale, st);
    case 32: return launch_decode_attn<DK, 32>(q, k, v, out, ws, R, H, Tk, k_rs, k_ks, v_rs, v_ks, scale, st);
    case 64: return launch_decode_attn<DK, 64>(q, k, v, out, ws, R, H, Tk, k_rs, k_ks, v_rs, v_ks, scale, st);
    default: return launch_decode_attn<DK, 128>(q, k, v, out, ws, R, H, Tk, k_rs, k_ks, v_rs, v_ks, scale, st);
  }
}

static bool head_dim_ok(int d) { return d == 16 || d == 32 || d == 64 || d == 128; }

}  // namespace b200asr

using namespace b200asr;

extern "C" {

size_t b200asr_decode_attn_ws_bytes(int R, int H, int Tk, int dv) {
  if (R < 1 || H < 1 || Tk < 1 || Tk > DA_MAX_TK || dv < 1) return 0;
  const int nc = ceil_div(Tk, decode_attn_chunk(R, H, Tk));
  if (nc == 1) return 0;
  return (size_t)R * H * nc * (size_t)(dv + 2) * sizeof(float);
}

int b200asr_decode_attn(const float* q, const float* k, const float* v, float* out, float* ws, int R, int H, int dk, int dv,
                        int Tk, long long k_row_stride, long long k_key_stride, long long v_row_stride,
                        long long v_key_stride, float scale, b200asr_stream_t stream) {
  B200_REQUIRE(q && k && v && out, B200ASR_BAD_ARG, "decode_attn: null pointer");
  B200_REQUIRE(head_dim_ok(dk) && head_dim_ok(dv), B200ASR_BAD_SHAPE,
               "decode_attn: head dims (dk=%d, dv=%d) must each be 16, 32, 64 or 128", dk, dv);
  B200_REQUIRE(R >= 1 && H >= 1 && Tk >= 1 && Tk <= DA_MAX_TK, B200ASR_BAD_SHAPE,
               "decode_attn: R=%d H=%d Tk=%d (need R, H >= 1 and 1 <= Tk <= %d)", R, H, Tk, DA_MAX_TK);
  B200_REQUIRE(k_row_stride >= 0 && k_key_stride >= 0 && v_row_stride >= 0 && v_key_stride >= 0, B200ASR_BAD_SHAPE,
               "decode_attn: strides must be >= 0 (k %lld/%lld, v %lld/%lld)", k_row_stride, k_key_stride, v_row_stride,
               v_key_stride);
  const int nc = ceil_div(Tk, decode_attn_chunk(R, H, Tk));
  B200_REQUIRE((long long)R * H * nc <= 0x7fffffffLL, B200ASR_BAD_SHAPE, "decode_attn: R*H*chunks too large (R=%d H=%d Tk=%d)",
               R, H, Tk);
  B200_REQUIRE(nc == 1 || ws, B200ASR_BAD_ARG, "decode_attn: ws is NULL but %d key chunks need b200asr_decode_attn_ws_bytes", nc);
  B200_REQUIRE(aligned16(k) && aligned16(v) && k_row_stride % 4 == 0 && k_key_stride % 4 == 0 && v_row_stride % 4 == 0 &&
                   v_key_stride % 4 == 0,
               B200ASR_BAD_ALIGN, "decode_attn: K/V must be 16-byte aligned and their strides multiples of 4 floats");
  cudaStream_t st = (cudaStream_t)stream;
  switch (dk) {
    case 16: return launch_decode_attn_dv<16>(dv, q, k, v, out, ws, R, H, Tk, k_row_stride, k_key_stride, v_row_stride, v_key_stride, scale, st);
    case 32: return launch_decode_attn_dv<32>(dv, q, k, v, out, ws, R, H, Tk, k_row_stride, k_key_stride, v_row_stride, v_key_stride, scale, st);
    case 64: return launch_decode_attn_dv<64>(dv, q, k, v, out, ws, R, H, Tk, k_row_stride, k_key_stride, v_row_stride, v_key_stride, scale, st);
    default: return launch_decode_attn_dv<128>(dv, q, k, v, out, ws, R, H, Tk, k_row_stride, k_key_stride, v_row_stride, v_key_stride, scale, st);
  }
}

}  // extern "C"
