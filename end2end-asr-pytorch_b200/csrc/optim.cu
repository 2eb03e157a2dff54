// Step tail over a LIST of separate tensors, the way torch.optim.Adam holds them (no flat buffer): Adam with the arithmetic of
// torch's foreach implementation, and the gradient-norm clip of torch.nn.utils.clip_grad_norm_ (norm_type 2).
//
// Every kernel takes its per-tensor table by value in the kernel parameters (__grid_constant__, up to 32 KB on sm_90), so a
// step needs no host-to-device copy, no allocation and no synchronisation.  A table holds at most OPT_TABLE tensors; a longer
// list is split into several tables, one launch each.  Each tensor is cut into chunks of OPT_CHUNK elements, one CTA per
// chunk; block_end[] (running chunk counts) maps a CTA to its tensor by binary search.  Where a tensor's pointers all share
// one 16-byte phase the chunk runs on float4 with a scalar head (up to 3 elements, first chunk) and tail (last chunk);
// otherwise -- a view at an odd float offset next to freshly allocated optimizer state -- it runs scalar.
#include "../../include/b200asr.h"
#include "common.cuh"

namespace b200asr {
namespace {

constexpr int OPT_TABLE = 512;       // tensors per launch (the Adam table is 28.7 KB of kernel parameters)
constexpr int OPT_THREADS = 256;
constexpr int OPT_CHUNK = 4096;      // elements per CTA: 4 float4 per thread

struct Span {
  long long n;
  int head;     // scalar elements before the first 16-byte aligned one; -1: the pointers differ in phase, all scalar
  int pad;
};

struct AdamTable {
  float* p[OPT_TABLE];
  const float* g[OPT_TABLE];
  float* m[OPT_TABLE];
  float* v[OPT_TABLE];
  Span s[OPT_TABLE];
  float step_size[OPT_TABLE];        // -lr / (1 - beta1^step), as torch passes it to addcdiv
  float bc2_sqrt[OPT_TABLE];         // (1 - beta2^step) ** 0.5
  int block_end[OPT_TABLE];
  int count;
  float lerp_w, beta2, one_minus_beta2, eps;
};

struct GradTable {
  float* g[OPT_TABLE];
  Span s[OPT_TABLE];
  int block_end[OPT_TABLE];
  int count;
};

static_assert(sizeof(AdamTable) <= 32764, "Adam table exceeds the kernel parameter limit");

__device__ __forceinline__ int table_entry(const int* block_end, int count) {
  int lo = 0, hi = count - 1;
  const int b = (int)blockIdx.x;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (block_end[mid] > b) hi = mid; else lo = mid + 1;
  }
  return lo;
}

// Visits the elements of chunk c of a tensor: one(i) for a scalar element, four(i) for the float4 at elements i .. i+3.
template <typename One, typename Four>
__device__ __forceinline__ void visit_chunk(const Span& s, long long c, One&& one, Four&& four) {
  const int tid = threadIdx.x;
  if (s.head < 0) {
    const long long b = c * OPT_CHUNK, e = min(s.n, b + OPT_CHUNK);
    for (long long i = b + tid; i < e; i += OPT_THREADS) one(i);
    return;
  }
  const long long nvec = (s.n - s.head) >> 2;
  const long long b = c * (OPT_CHUNK / 4), e = min(nvec, b + OPT_CHUNK / 4);
  if (c == 0 && tid < s.head) one(tid);
  for (long long i = b + tid; i < e; i += OPT_THREADS) four(s.head + 4 * i);
  const long long tail = s.head + 4 * nvec;
  if (e == nvec && tid < s.n - tail) one(tail + tid);
}

// One element of torch 2.11's _multi_tensor_adam (non-capturable, no amsgrad / weight decay / maximize), op by op, each op
// rounded on its own as the compiled ATen foreach kernels round it (fp32 opmath; a + s * b contracted to one fma):
//   _foreach_lerp_(m, g, w)      ATen lerp: |w| < 0.5 ? m + w * (g - m) : g - (g - m) * (1 - w)
//   _foreach_mul_(v, beta2)
//   _foreach_addcmul_(v, g, g, 1 - beta2)          v + (1 - beta2) * (g * g)
//   d = _foreach_sqrt(v); _foreach_div_(d, bc2_sqrt); _foreach_add_(d, eps)
//   _foreach_addcdiv_(p, m, d, step_size)          p + step_size * (m / d)
__device__ __forceinline__ void adam_elem(float& p, float g, float& m, float& v, float w, float b2, float omb2, float eps,
                                          float step_size, float bc2_sqrt) {
  const float diff = __fsub_rn(g, m);
  m = fabsf(w) < 0.5f ? __fmaf_rn(w, diff, m) : __fmaf_rn(-diff, __fsub_rn(1.f, w), g);
  v = __fmul_rn(v, b2);
  v = __fmaf_rn(omb2, __fmul_rn(g, g), v);
  const float d = __fadd_rn(__fdiv_rn(__fsqrt_rn(v), bc2_sqrt), eps);
  p = __fmaf_rn(step_size, __fdiv_rn(m, d), p);
}

__global__ void __launch_bounds__(OPT_THREADS) adam_multi_kernel(const __grid_constant__ AdamTable t) {
  const int k = table_entry(t.block_end, t.count);
  const long long c = (long long)blockIdx.x - (k ? t.block_end[k - 1] : 0);
  float* __restrict__ p = t.p[k];
  const float* __restrict__ g = t.g[k];
  float* __restrict__ m = t.m[k];
  float* __restrict__ v = t.v[k];
  const float w = t.lerp_w, b2 = t.beta2, omb2 = t.one_minus_beta2, eps = t.eps, ss = t.step_size[k], bc = t.bc2_sqrt[k];
  visit_chunk(
      t.s[k], c,
      [&](long long i) {
        float pi = p[i], mi = m[i], vi = v[i];
        adam_elem(pi, g[i], mi, vi, w, b2, omb2, eps, ss, bc);
        p[i] = pi; m[i] = mi; v[i] = vi;
      },
      [&](long long i) {
        float4 P = *reinterpret_cast<const float4*>(p + i), G = *reinterpret_cast<const float4*>(g + i);
        float4 M = *reinterpret_cast<const float4*>(m + i), V = *reinterpret_cast<const float4*>(v + i);
        adam_elem(P.x, G.x, M.x, V.x, w, b2, omb2, eps, ss, bc);
        adam_elem(P.y, G.y, M.y, V.y, w, b2, omb2, eps, ss, bc);
        adam_elem(P.z, G.z, M.z, V.z, w, b2, omb2, eps, ss, bc);
        adam_elem(P.w, G.w, M.w, V.w, w, b2, omb2, eps, ss, bc);
        *reinterpret_cast<float4*>(p + i) = P; *reinterpret_cast<float4*>(m + i) = M;
        *reinterpret_cast<float4*>(v + i) = V;
      });
}

// part[blockIdx.x] = the chunk's sum of squares: each thread adds its elements in order, then the warps, then the 8 warp sums
// in order -- the same bits on every run
__global__ void __launch_bounds__(OPT_THREADS) sumsq_multi_kernel(const __grid_constant__ GradTable t, float* __restrict__ part) {
  __shared__ float red[OPT_THREADS / 32];
  const int k = table_entry(t.block_end, t.count);
  const long long c = (long long)blockIdx.x - (k ? t.block_end[k - 1] : 0);
  const float* __restrict__ g = t.g[k];
  float s = 0.f;
  visit_chunk(
      t.s[k], c, [&](long long i) { s = __fmaf_rn(g[i], g[i], s); },
      [&](long long i) {
        const float4 G = *reinterpret_cast<const float4*>(g + i);
        s = __fmaf_rn(G.x, G.x, s); s = __fmaf_rn(G.y, G.y, s); s = __fmaf_rn(G.z, G.z, s); s = __fmaf_rn(G.w, G.w, s);
      });
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    float r = 0.f;
#pragma unroll
    for (int w = 0; w < OPT_THREADS / 32; w++) r = __fadd_rn(r, red[w]);
    part[blockIdx.x] = r;
  }
}

// norms[k] = sqrt(sum of tensor k's chunk partials), one warp per tensor: lane l adds partials l, l + 32, ... in order, then
// the fixed xor-shuffle tree adds the lanes
__global__ void tensor_norms_kernel(const __grid_constant__ GradTable t, const float* __restrict__ part, float* __restrict__ norms) {
  const int k = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5), lane = threadIdx.x & 31;
  if (k >= t.count) return;
  float s = 0.f;
  for (int b = (k ? t.block_end[k - 1] : 0) + lane; b < t.block_end[k]; b += 32) s = __fadd_rn(s, part[b]);
  s = warp_sum(s);
  if (lane == 0) norms[k] = __fsqrt_rn(s);
}

// out[0] = sqrt(sum of norms^2) (torch: vector_norm(stack(per-tensor norms))), out[1] = the clip coefficient as
// clip_grad_norm_ forms it: clamp(max_norm / (total + 1e-6), max=1), where max_norm / x is reciprocal(x) * max_norm (a NaN
// total gives a NaN coefficient, as torch.clamp does).  One CTA; fixed-order sums.
__global__ void __launch_bounds__(OPT_THREADS) clip_coef_kernel(const float* __restrict__ norms, int count, float max_norm,
                                                                float* __restrict__ out) {
  __shared__ float red[OPT_THREADS / 32];
  float s = 0.f;
  for (int k = threadIdx.x; k < count; k += OPT_THREADS) s = __fmaf_rn(norms[k], norms[k], s);
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    float r = 0.f;
#pragma unroll
    for (int w = 0; w < OPT_THREADS / 32; w++) r = __fadd_rn(r, red[w]);
    const float total = __fsqrt_rn(r);
    const float coef = __fmul_rn(__frcp_rn(__fadd_rn(total, 1e-6f)), max_norm);
    out[0] = total;
    out[1] = coef > 1.f ? 1.f : coef;
  }
}

// g *= *coef for every element (torch._foreach_mul_(grads, coef))
__global__ void __launch_bounds__(OPT_THREADS) scale_multi_kernel(const __grid_constant__ GradTable t, const float* __restrict__ coef) {
  const int k = table_entry(t.block_end, t.count);
  const long long c = (long long)blockIdx.x - (k ? t.block_end[k - 1] : 0);
  float* __restrict__ g = t.g[k];
  const float a = *coef;
  visit_chunk(
      t.s[k], c, [&](long long i) { g[i] = __fmul_rn(g[i], a); },
      [&](long long i) {
        float4 G = *reinterpret_cast<const float4*>(g + i);
        G.x = __fmul_rn(G.x, a); G.y = __fmul_rn(G.y, a); G.z = __fmul_rn(G.z, a); G.w = __fmul_rn(G.w, a);
        *reinterpret_cast<float4*>(g + i) = G;
      });
}

// Span and chunk count of a tensor whose pointers are ptrs[0 .. nptr-1] (an empty tensor gets no chunk)
static long long plan_span(const uint64_t* ptrs, int nptr, long long n, Span& s) {
  const uint64_t phase = ptrs[0] & 15u;
  bool same = true;
  for (int j = 1; j < nptr; j++) same = same && (ptrs[j] & 15u) == phase;
  s.n = n;
  s.pad = 0;
  if (n == 0) {
    s.head = 0;
    return 0;
  }
  if (!same) {
    s.head = -1;
    return ceil_div_ll(n, OPT_CHUNK);
  }
  const long long h = (long long)((16u - phase) & 15u) / 4;
  s.head = (int)(h < n ? h : n);
  const long long chunks = ceil_div_ll((n - s.head) / 4, OPT_CHUNK / 4);
  return chunks > 0 ? chunks : 1;
}

// Checks the host arrays of one call and fills spans / block_end.  Returns the number of CTAs or a negative error code.
static long long plan_table(const uint64_t* ptrs, int nptr, const long long* numel, int count, Span* spans, int* block_end,
                            const char* what) {
  B200_REQUIRE(ptrs && numel, B200ASR_BAD_ARG, "%s: null table", what);
  B200_REQUIRE(count >= 1 && count <= OPT_TABLE, B200ASR_BAD_SHAPE, "%s: count %d outside [1, %d]", what, count, OPT_TABLE);
  long long blocks = 0;
  for (int k = 0; k < count; k++) {
    const uint64_t* q = ptrs + (size_t)k * nptr;
    B200_REQUIRE(numel[k] >= 0, B200ASR_BAD_SHAPE, "%s: tensor %d has numel %lld", what, k, numel[k]);
    for (int j = 0; j < nptr; j++) {
      B200_REQUIRE(q[j] != 0, B200ASR_BAD_ARG, "%s: tensor %d, pointer %d is NULL", what, k, j);
      B200_REQUIRE((q[j] & 3u) == 0, B200ASR_BAD_ALIGN, "%s: tensor %d, pointer %d is not 4-byte aligned", what, k, j);
    }
    blocks += plan_span(q, nptr, numel[k], spans[k]);
    B200_REQUIRE(blocks < (1LL << 31), B200ASR_BAD_SHAPE, "%s: table too large", what);
    block_end[k] = (int)blocks;
  }
  return blocks;
}

static long long plan_grads(const uint64_t* tensors, const long long* numel, int count, GradTable& t, const char* what) {
  const long long blocks = plan_table(tensors, 1, numel, count, t.s, t.block_end, what);
  if (blocks < 0) return blocks;
  t.count = count;
  for (int k = 0; k < count; k++) t.g[k] = reinterpret_cast<float*>(tensors[k]);
  return blocks;
}

}  // namespace
}  // namespace b200asr

using namespace b200asr;

extern "C" {

int b200asr_optim_table_capacity(void) { return OPT_TABLE; }

int b200asr_adam_multi(const uint64_t* tensors, const long long* numel, const float* step_size, const float* bc2_sqrt, int count,
                       float lerp_weight, float beta2, float one_minus_beta2, float eps, b200asr_stream_t stream) {
  B200_REQUIRE(step_size && bc2_sqrt, B200ASR_BAD_ARG, "adam_multi: null scalars");
  AdamTable t;
  const long long blocks = plan_table(tensors, 4, numel, count, t.s, t.block_end, "adam_multi");
  if (blocks <= 0) return (int)blocks;
  t.count = count;
  for (int k = 0; k < count; k++) {
    const uint64_t* q = tensors + (size_t)k * 4;
    t.p[k] = reinterpret_cast<float*>(q[0]);
    t.g[k] = reinterpret_cast<const float*>(q[1]);
    t.m[k] = reinterpret_cast<float*>(q[2]);
    t.v[k] = reinterpret_cast<float*>(q[3]);
    t.step_size[k] = step_size[k];
    t.bc2_sqrt[k] = bc2_sqrt[k];
  }
  t.lerp_w = lerp_weight; t.beta2 = beta2; t.one_minus_beta2 = one_minus_beta2; t.eps = eps;
  adam_multi_kernel<<<(unsigned)blocks, OPT_THREADS, 0, (cudaStream_t)stream>>>(t);
  return check_launch("adam_multi");
}

int b200asr_norm_multi(const uint64_t* tensors, const long long* numel, int count, float* norms, b200asr_stream_t stream) {
  B200_REQUIRE(norms, B200ASR_BAD_ARG, "norm_multi: null output");
  GradTable t;
  const long long blocks = plan_grads(tensors, numel, count, t, "norm_multi");
  if (blocks < 0) return (int)blocks;
  cudaStream_t st = (cudaStream_t)stream;
  float* part = nullptr;
  if (blocks > 0) {
    part = (float*)stream_scratch(sizeof(float) * (size_t)blocks, st);
    if (!part) return B200ASR_CUDA_ERROR;
    sumsq_multi_kernel<<<(unsigned)blocks, OPT_THREADS, 0, st>>>(t, part);
    if (int rc = check_launch("norm_multi")) return rc;
  }
  tensor_norms_kernel<<<ceil_div(count, 4), 128, 0, st>>>(t, part, norms);
  return check_launch("norm_multi");
}

int b200asr_clip_coef(const float* norms, int count, float max_norm, float* out, b200asr_stream_t stream) {
  B200_REQUIRE(norms && out && count >= 1, B200ASR_BAD_ARG, "clip_coef: bad arguments");
  clip_coef_kernel<<<1, OPT_THREADS, 0, (cudaStream_t)stream>>>(norms, count, max_norm, out);
  return check_launch("clip_coef");
}

int b200asr_scale_multi(const uint64_t* tensors, const long long* numel, int count, const float* coef, b200asr_stream_t stream) {
  B200_REQUIRE(coef, B200ASR_BAD_ARG, "scale_multi: null coefficient");
  GradTable t;
  const long long blocks = plan_grads(tensors, numel, count, t, "scale_multi");
  if (blocks <= 0) return (int)blocks;
  scale_multi_kernel<<<(unsigned)blocks, OPT_THREADS, 0, (cudaStream_t)stream>>>(t, coef);
  return check_launch("scale_multi");
}

}  // extern "C"
