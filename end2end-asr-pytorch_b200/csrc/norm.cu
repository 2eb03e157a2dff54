// Residual + LayerNorm (+PE, + non-pad row mask), forward and backward.  HBM-bound: one warp owns a row,
// the row lives in registers (128-bit loads), statistics via warp shuffles.  See include/b200asr.h.
#include "../../include/b200asr.h"
#include "common.cuh"

namespace b200asr {

constexpr int LN_WARPS = 4;
constexpr int LN_MAXV = 8;  // float4 per lane -> d <= 1024 (kernels are instantiated for NV = 1, 2, 4, 6, 8)

static int ln_bwd_blocks(int rows) {
  int b = ceil_div(rows, LN_WARPS);          // one row per warp up to 2368 CTAs: latency-bound otherwise
  return b < 2368 ? (b < 1 ? 1 : b) : 2368;
}

template <int NV>
__global__ void __launch_bounds__(LN_WARPS * 32)
add_ln_fwd_kernel(const float* __restrict__ x, const float* __restrict__ res, const float* __restrict__ gamma,
                  const float* __restrict__ beta, const float* __restrict__ post, int period,
                  const float* __restrict__ rowscale, float* __restrict__ y, float* __restrict__ z,
                  float* __restrict__ mean_out, float* __restrict__ rstd_out, int rows, int d, float eps,
                  uint32_t thresh, float inv_keep, uint64_t key) {
  griddep_launch();      // programmatic dependent launch (common.cuh)
  griddep_wait();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int row = blockIdx.x * LN_WARPS + warp;
  if (row >= rows) return;
  const size_t base = (size_t)row * d;
  float4 v[NV];
  float sum = 0.f;
#pragma unroll
  for (int i = 0; i < NV; i++) {
    int col = (i * 32 + lane) * 4;
    if (col < d) {
      float4 a = *reinterpret_cast<const float4*>(x + base + col);
      if (thresh) {
        uint64_t r = dropout_bits4(key, (base + col) >> 2);
        a.x = ((uint32_t)(r) & 0xFFFFu) >= thresh ? a.x * inv_keep : 0.f;
        a.y = ((uint32_t)(r >> 16) & 0xFFFFu) >= thresh ? a.y * inv_keep : 0.f;
        a.z = ((uint32_t)(r >> 32) & 0xFFFFu) >= thresh ? a.z * inv_keep : 0.f;
        a.w = ((uint32_t)(r >> 48) & 0xFFFFu) >= thresh ? a.w * inv_keep : 0.f;
      }
      if (res) {
        float4 b = *reinterpret_cast<const float4*>(res + base + col);
        a.x += b.x; a.y += b.y; a.z += b.z; a.w += b.w;
      }
      if (z) *reinterpret_cast<float4*>(z + base + col) = a;
      v[i] = a;
      sum += a.x + a.y + a.z + a.w;
    }
  }
  const float mean = warp_sum(sum) / (float)d;
  float sq = 0.f;
#pragma unroll
  for (int i = 0; i < NV; i++) {
    int col = (i * 32 + lane) * 4;
    if (col < d) {
      float a = v[i].x - mean, b = v[i].y - mean, c = v[i].z - mean, e = v[i].w - mean;
      sq += a * a + b * b + c * c + e * e;
    }
  }
  const float rstd = rsqrtf(warp_sum(sq) / (float)d + eps);
  if (lane == 0) { mean_out[row] = mean; rstd_out[row] = rstd; }
  const float rs = rowscale ? rowscale[row] : 1.f;
  const float* prow = post ? post + (size_t)(row % period) * d : nullptr;
#pragma unroll
  for (int i = 0; i < NV; i++) {
    int col = (i * 32 + lane) * 4;
    if (col < d) {
      float4 g = *reinterpret_cast<const float4*>(gamma + col);
      float4 b = *reinterpret_cast<const float4*>(beta + col);
      float4 o;
      o.x = (v[i].x - mean) * rstd * g.x + b.x;
      o.y = (v[i].y - mean) * rstd * g.y + b.y;
      o.z = (v[i].z - mean) * rstd * g.z + b.z;
      o.w = (v[i].w - mean) * rstd * g.w + b.w;
      if (prow) {
        float4 q = *reinterpret_cast<const float4*>(prow + col);
        o.x += q.x; o.y += q.y; o.z += q.z; o.w += q.w;
      }
      o.x *= rs; o.y *= rs; o.z *= rs; o.w *= rs;
      *reinterpret_cast<float4*>(y + base + col) = o;
    }
  }
}

template <int NV>
__global__ void __launch_bounds__(LN_WARPS * 32)
add_ln_bwd_kernel(const float* __restrict__ dy, const float* __restrict__ z, const float* __restrict__ gamma,
                  const float* __restrict__ mean_in, const float* __restrict__ rstd_in,
                  const float* __restrict__ rowscale, float* __restrict__ dz, float* __restrict__ dx,
                  float* __restrict__ partial, int rows, int d, uint32_t thresh, float inv_keep, uint64_t key) {
  __shared__ __align__(16) float sdg[LN_WARPS][NV * 128];
  __shared__ __align__(16) float sdb[LN_WARPS][NV * 128];
  griddep_launch();      // programmatic dependent launch (common.cuh)
  griddep_wait();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float4 dg[NV], db[NV];
#pragma unroll
  for (int i = 0; i < NV; i++) { dg[i] = make_float4(0, 0, 0, 0); db[i] = make_float4(0, 0, 0, 0); }
  const float invd = 1.f / (float)d;
  for (int row = blockIdx.x * LN_WARPS + warp; row < rows; row += gridDim.x * LN_WARPS) {
    const size_t base = (size_t)row * d;
    const float mean = mean_in[row], rstd = rstd_in[row];
    const float rs = rowscale ? rowscale[row] : 1.f;
    float4 xh[NV], gx[NV];
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int i = 0; i < NV; i++) {
      int col = (i * 32 + lane) * 4;
      if (col < d) {
        float4 a = *reinterpret_cast<const float4*>(z + base + col);
        float4 g = *reinterpret_cast<const float4*>(dy + base + col);
        float4 w = *reinterpret_cast<const float4*>(gamma + col);
        a.x = (a.x - mean) * rstd; a.y = (a.y - mean) * rstd; a.z = (a.z - mean) * rstd; a.w = (a.w - mean) * rstd;
        g.x *= rs; g.y *= rs; g.z *= rs; g.w *= rs;
        dg[i].x += g.x * a.x; dg[i].y += g.y * a.y; dg[i].z += g.z * a.z; dg[i].w += g.w * a.w;
        db[i].x += g.x; db[i].y += g.y; db[i].z += g.z; db[i].w += g.w;
        g.x *= w.x; g.y *= w.y; g.z *= w.z; g.w *= w.w;
        s1 += g.x + g.y + g.z + g.w;
        s2 += g.x * a.x + g.y * a.y + g.z * a.z + g.w * a.w;
        xh[i] = a; gx[i] = g;
      }
    }
    s1 = warp_sum(s1) * invd;
    s2 = warp_sum(s2) * invd;
#pragma unroll
    for (int i = 0; i < NV; i++) {
      int col = (i * 32 + lane) * 4;
      if (col < d) {
        float4 o;
        o.x = rstd * (gx[i].x - s1 - xh[i].x * s2);
        o.y = rstd * (gx[i].y - s1 - xh[i].y * s2);
        o.z = rstd * (gx[i].z - s1 - xh[i].z * s2);
        o.w = rstd * (gx[i].w - s1 - xh[i].w * s2);
        if (dz) *reinterpret_cast<float4*>(dz + base + col) = o;
        if (thresh) {
          uint64_t r = dropout_bits4(key, (base + col) >> 2);
          o.x = ((uint32_t)(r) & 0xFFFFu) >= thresh ? o.x * inv_keep : 0.f;
          o.y = ((uint32_t)(r >> 16) & 0xFFFFu) >= thresh ? o.y * inv_keep : 0.f;
          o.z = ((uint32_t)(r >> 32) & 0xFFFFu) >= thresh ? o.z * inv_keep : 0.f;
          o.w = ((uint32_t)(r >> 48) & 0xFFFFu) >= thresh ? o.w * inv_keep : 0.f;
        }
        if (dx && (dx != dz || thresh)) *reinterpret_cast<float4*>(dx + base + col) = o;
      }
    }
  }
#pragma unroll
  for (int i = 0; i < NV; i++) {
    int col = (i * 32 + lane) * 4;
    if (col < d) {
      *reinterpret_cast<float4*>(&sdg[warp][col]) = dg[i];
      *reinterpret_cast<float4*>(&sdb[warp][col]) = db[i];
    }
  }
  __syncthreads();
  float* pg = partial + (size_t)blockIdx.x * 2 * d;
  for (int c = threadIdx.x; c < d; c += blockDim.x) {
    float a = 0.f, b = 0.f;
#pragma unroll
    for (int w = 0; w < LN_WARPS; w++) { a += sdg[w][c]; b += sdb[w][c]; }
    pg[c] = a;
    pg[d + c] = b;
  }
}

// dgamma/dbeta = column sums of the per-CTA partials: grid (d/32, row slices); 32 columns x 8 row lanes per CTA, smem tree,
// one sum per column and slice into `slices` [LN_FIN_SLICES][2d], which reduce_parts adds up in slice order (a single-slice
// version was latency-bound: 16 CTAs walking 1600 partial rows took longer than the main kernel)
constexpr int LN_FIN_SLICES = 16;
__global__ void __launch_bounds__(256) ln_bwd_finalize_kernel(const float* __restrict__ partial, int nblk, int d,
                                                              float* __restrict__ slices) {
  __shared__ float ra[8][33], rb[8][33];
  griddep_launch();      // programmatic dependent launch (common.cuh)
  griddep_wait();
  const int cl = threadIdx.x & 31, rl = threadIdx.x >> 5;
  const int c = blockIdx.x * 32 + cl;
  const int per = (nblk + gridDim.y - 1) / gridDim.y;
  const int r0 = blockIdx.y * per, r1 = min(nblk, r0 + per);
  float a = 0.f, b = 0.f;
  if (c < d)
    for (int i = r0 + rl; i < r1; i += 8) {
      a += partial[(size_t)i * 2 * d + c];
      b += partial[(size_t)i * 2 * d + d + c];
    }
  ra[rl][cl] = a; rb[rl][cl] = b;
  __syncthreads();
  if (rl == 0 && c < d) {
    float sa = 0.f, sb = 0.f;
#pragma unroll
    for (int i = 0; i < 8; i++) { sa += ra[i][cl]; sb += rb[i][cl]; }
    slices[(size_t)blockIdx.y * 2 * d + c] = sa;
    slices[(size_t)blockIdx.y * 2 * d + d + c] = sb;
  }
}

}  // namespace b200asr

using namespace b200asr;

extern "C" {

size_t b200asr_add_ln_bwd_ws_bytes(int rows, int d) { return sizeof(float) * 2 * (size_t)d * ln_bwd_blocks(rows); }

int b200asr_add_ln_fwd(const float* x, const float* residual, const float* gamma, const float* beta,
                       const float* post_add, int post_period, const float* row_scale, float* y, float* z, float* mean,
                       float* rstd, int rows, int d, float eps, float p_drop, uint64_t seed, uint64_t offset,
                       b200asr_stream_t stream) {
  B200_REQUIRE(x && gamma && beta && y && mean && rstd, B200ASR_BAD_ARG, "add_ln_fwd: null pointer");
  B200_REQUIRE(d > 0 && d % 4 == 0 && d <= LN_MAXV * 128, B200ASR_BAD_SHAPE, "add_ln_fwd: d=%d must be a multiple of 4 and <= %d", d, LN_MAXV * 128);
  B200_REQUIRE(p_drop >= 0.f && p_drop < 1.f, B200ASR_BAD_ARG, "add_ln_fwd: p_drop=%f", p_drop);
  B200_REQUIRE(z || (!residual && p_drop == 0.f), B200ASR_BAD_ARG, "add_ln_fwd: z (saved LN input) required with residual or dropout");
  B200_REQUIRE(!post_add || post_period > 0, B200ASR_BAD_ARG, "add_ln_fwd: post_period");
  B200_REQUIRE(aligned16(x) && aligned16(y) && aligned16(gamma) && aligned16(beta) && (!residual || aligned16(residual)) && (!z || aligned16(z)) && (!post_add || aligned16(post_add)),
               B200ASR_BAD_ALIGN, "add_ln_fwd: pointers must be 16-byte aligned");
  if (rows <= 0) return B200ASR_OK;
  uint32_t th = p_drop > 0.f ? dropout_thresh16(p_drop) : 0u;
#define LN_FWD(NVv) launch_pdl(add_ln_fwd_kernel<NVv>, dim3(ceil_div(rows, LN_WARPS)), dim3(LN_WARPS * 32), 0, (cudaStream_t)stream, \
      x, residual, gamma, beta, post_add, post_period, row_scale, y, z, mean, rstd, rows, d, eps, th, \
      dropout_inv_keep(p_drop), dropout_key(seed, offset))
  const int nv = ceil_div(d, 128);
  if (nv <= 1) LN_FWD(1); else if (nv <= 2) LN_FWD(2); else if (nv <= 4) LN_FWD(4); else if (nv <= 6) LN_FWD(6); else LN_FWD(8);
#undef LN_FWD
  return check_launch("add_ln_fwd");
}

int b200asr_add_ln_bwd(const float* dy, const float* z, const float* gamma, const float* mean, const float* rstd,
                       const float* row_scale, float* dz, float* dx, float* dgamma, float* dbeta, void* partial_ws,
                       int rows, int d, float p_drop, uint64_t seed, uint64_t offset, int accumulate,
                       b200asr_stream_t stream) {
  B200_REQUIRE(dy && z && gamma && mean && rstd && dgamma && dbeta && partial_ws && (dz || dx), B200ASR_BAD_ARG, "add_ln_bwd: null pointer");
  B200_REQUIRE(d > 0 && d % 4 == 0 && d <= LN_MAXV * 128, B200ASR_BAD_SHAPE, "add_ln_bwd: d=%d unsupported", d);
  B200_REQUIRE(aligned16(dy) && aligned16(z) && aligned16(gamma) && (!dz || aligned16(dz)) && (!dx || aligned16(dx)), B200ASR_BAD_ALIGN, "add_ln_bwd: alignment");
  cudaStream_t st = (cudaStream_t)stream;
  if (rows <= 0) {
    if (!accumulate) {
      cudaMemsetAsync(dgamma, 0, sizeof(float) * d, st);
      cudaMemsetAsync(dbeta, 0, sizeof(float) * d, st);
    }
    return B200ASR_OK;
  }
  uint32_t th = p_drop > 0.f ? dropout_thresh16(p_drop) : 0u;
  int nblk = ln_bwd_blocks(rows);
#define LN_BWD(NVv) launch_pdl(add_ln_bwd_kernel<NVv>, dim3(nblk), dim3(LN_WARPS * 32), 0, st, dy, z, gamma, mean, rstd, row_scale, dz, dx, \
      (float*)partial_ws, rows, d, th, dropout_inv_keep(p_drop), dropout_key(seed, offset))
  const int nv = ceil_div(d, 128);
  if (nv <= 1) LN_BWD(1); else if (nv <= 2) LN_BWD(2); else if (nv <= 4) LN_BWD(4); else if (nv <= 6) LN_BWD(6); else LN_BWD(8);
#undef LN_BWD
  int rc = check_launch("add_ln_bwd");
  if (rc) return rc;
  float* slices = (float*)stream_scratch(sizeof(float) * 2 * (size_t)d * LN_FIN_SLICES, st);
  if (!slices) return B200ASR_CUDA_ERROR;
  launch_pdl(ln_bwd_finalize_kernel, dim3(ceil_div(d, 32), LN_FIN_SLICES), dim3(256), 0, st, (const float*)partial_ws, nblk, d, slices);
  if ((rc = check_launch("ln_bwd_finalize"))) return rc;
  if ((rc = reduce_parts(slices, LN_FIN_SLICES, 2LL * d, d, dgamma, accumulate, st))) return rc;
  return reduce_parts(slices + d, LN_FIN_SLICES, 2LL * d, d, dbeta, accumulate, st);
}

}  // extern "C"
