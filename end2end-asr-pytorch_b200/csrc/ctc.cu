// CTC loss of utils/metrics.py:133-154 (F.ctc_loss(log_softmax(pred.transpose(0, 1)), targets, input_lengths,
// target_lengths, blank=0, reduction="mean")) straight from the [B, T, V] logits, exact fp32 on CUDA cores, log space.
//
//   ctc_lp:    one CTA per (b, t) row: the row's log-sum-exp (block_row_lse) and lp'[b, t, s] = z[b, t, l'(s)] - lse over the
//              2 L_b + 1 states of the extended label sequence l' = (blank, l_1, blank, l_2, ..., blank).
//   ctc_rec:   one CTA per utterance: the alpha (forward) or beta (backward) recursion over t, the states of t and t - 1
//              double-buffered in shared memory, one barrier per step.  Each step's states are renormalised by their
//              maximum (Rabiner scaling in log space): the stored alpha-hat / beta-hat stay near 0, where fp32 keeps ~1e-7 of
//              them, and the scales add up (Kahan) into nll_b.  Unscaled log alphas reach -8000 at T = 1000, V = 4364, where
//              one fp32 ulp is 1e-3 and the occupation probabilities exp(alpha + beta - lp' + nll) would carry percent errors.
//   ctc_grad:  one CTA per (b, t) row: gamma_t(s) = exp(w_s) / sum_s exp(w_s), w = alpha-hat + beta-hat - lp' (the sum is
//              P(l | x) times the two scales, so gamma needs no nll), summed per label in a fixed state order, then
//              dz = g_b (softmax(z) - sum of gamma of the label).  No floating-point atomics anywhere.
#include <math.h>

#include "../../include/b200asr.h"
#include "common.cuh"

namespace b200asr {

constexpr int CTC_LP_THREADS = 256;
constexpr int CTC_REC_THREADS = 256;
constexpr int CTC_GRAD_THREADS = 256;
constexpr int CTC_MAX_K = 32;                                  // states per thread of ctc_rec
constexpr int CTC_MAX_STATES = CTC_MAX_K * CTC_REC_THREADS;    // 2 * max_target_len + 1 <= 8192

// Workspace (caller-owned), in this order: row (max, log sum exp(z - max)) [B][T][2] fp32; lp', alpha-hat, beta-hat
// [B][T][Sp] fp32 each (Sp = 2 Lmax + 1); next_same / first [B][Lmax] int32: for target position i, the next position
// j > i with the same label (-1: none) and whether i is the label's first occurrence.
struct CtcWs {
  float *row, *lp, *alpha, *beta;
  int *next_same, *first;
};
static inline CtcWs ctc_ws(void* ws, int B, int T, int Lmax) {
  const size_t Sp = 2 * (size_t)Lmax + 1, rows = (size_t)B * T;
  CtcWs w;
  w.row = (float*)ws;
  w.lp = w.row + 2 * rows;
  w.alpha = w.lp + rows * Sp;
  w.beta = w.alpha + rows * Sp;
  w.next_same = (int*)(w.beta + rows * Sp);
  w.first = w.next_same + (size_t)B * Lmax;
  return w;
}

// An utterance whose lengths break the contract (the host validates them; here they are device data) gets a NaN loss and
// NaN gradient rows instead of out-of-range reads.
__device__ __forceinline__ bool ctc_lengths_ok(int Tb, int Lb, int T, int Lmax) { return Tb >= 0 && Tb <= T && Lb >= 0 && Lb <= Lmax; }

__device__ __forceinline__ float lse3(float a, float b, float c) {
  const float m = fmaxf(a, fmaxf(b, c));
  if (m == -INFINITY) return -INFINITY;
  return m + logf(expf(a - m) + expf(b - m) + expf(c - m));
}

__global__ void __launch_bounds__(CTC_LP_THREADS) ctc_lp_kernel(const float* __restrict__ logits, const int64_t* __restrict__ targets,
                                                                const int32_t* __restrict__ in_len, const int32_t* __restrict__ tgt_len,
                                                                float* __restrict__ row_out, float* __restrict__ lp, int T, int V,
                                                                int S, int Lmax) {
  const int r = blockIdx.x, b = r / T, t = r - b * T;
  const int Tb = in_len[b], Lb = tgt_len[b];
  if (!ctc_lengths_ok(Tb, Lb, T, Lmax) || t >= Tb) return;
  const float* x = logits + (size_t)r * V;
  const RowLse st = block_row_lse<CTC_LP_THREADS, false>(x, V);
  const float lt = logf(st.sumexp);
  if (threadIdx.x == 0) { row_out[2 * (size_t)r] = st.mx; row_out[2 * (size_t)r + 1] = lt; }
  const int Sb = 2 * Lb + 1;
  const size_t Sp = 2 * (size_t)Lmax + 1;
  float* out = lp + (size_t)r * Sp;
  for (int s = threadIdx.x; s < Sb; s += CTC_LP_THREADS) {
    const int64_t l = (s & 1) ? targets[(size_t)b * S + (s >> 1)] : 0;
    out[s] = (l >= 0 && l < V) ? (x[l] - st.mx) - lt : NAN;
  }
}

// The alpha (BACK = false) or beta (BACK = true) recursion of utterance blockIdx.x over t < T_b; thread tid owns states
// s = k * CTC_REC_THREADS + tid, k < K.  u_t(s) = lp'_t(s) + lse(hat_{t-1}(s), hat_{t-1}(s -+ 1), hat_{t-1}(s -+ 2) if the skip
// is allowed); c_t = max_s u_t(s); hat_t = u_t - c_t goes to `out` [T][Sp].  The skip into s (alpha) or out of s (beta)
// exists where l'(s) != l'(s -+ 2), i.e. for odd s whose label differs from the neighbouring label.  The alpha pass also
// writes nll[b] = -(sum_t c_t + log(hat(S_b - 1) + hat(S_b - 2))) and the label chains of the gradient kernel.
template <int K, bool BACK>
__global__ void __launch_bounds__(CTC_REC_THREADS) ctc_rec_kernel(const int64_t* __restrict__ targets, const int32_t* __restrict__ in_len,
                                                                  const int32_t* __restrict__ tgt_len, const float* __restrict__ lp,
                                                                  float* __restrict__ out, float* __restrict__ nll,
                                                                  int* __restrict__ next_same, int* __restrict__ first, int T, int S,
                                                                  int Lmax) {
  extern __shared__ float smem[];
  __shared__ float wmax[2][CTC_REC_THREADS / 32];
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int Sp = 2 * Lmax + 1;
  int* lab = reinterpret_cast<int*>(smem);
  float* buf = smem + Lmax;                                    // [2][Sp]
  const int Tb = in_len[b], Lb = tgt_len[b];
  if (!ctc_lengths_ok(Tb, Lb, T, Lmax)) {
    if (!BACK && tid == 0) nll[b] = NAN;
    return;
  }
  const int Sb = 2 * Lb + 1;
  for (int i = tid; i < Lb; i += CTC_REC_THREADS) {
    const int64_t l = targets[(size_t)b * S + i];
    lab[i] = (l >= 0 && l < 0x7fffffff) ? (int)l : -1;         // out-of-range labels already make lp' NaN
  }
  __syncthreads();
  if (!BACK) {
    for (int i = tid; i < Lb; i += CTC_REC_THREADS) {
      int f = 1, n = -1;
      for (int j = 0; j < i; j++)
        if (lab[j] == lab[i]) { f = 0; break; }
      for (int j = i + 1; j < Lb; j++)
        if (lab[j] == lab[i]) { n = j; break; }
      first[(size_t)b * Lmax + i] = f;
      next_same[(size_t)b * Lmax + i] = n;
    }
    if (Tb == 0) {                                             // no frames: P = 1 for the empty target, 0 otherwise
      if (tid == 0) nll[b] = Lb == 0 ? 0.f : INFINITY;
      return;
    }
  } else if (Tb == 0) {
    return;
  }
  const float* lpb = lp + (size_t)b * T * Sp;
  float* ob = out + (size_t)b * T * Sp;
  uint32_t skip = 0;                                           // bit k: state k * CTC_REC_THREADS + tid has the skip
  float u[K], lpn[K];
#pragma unroll
  for (int k = 0; k < K; k++) {
    const int s = k * CTC_REC_THREADS + tid;
    const bool sk = !BACK ? (s < Sb && (s & 1) && s >= 3 && lab[s >> 1] != lab[(s >> 1) - 1])
                          : (s < Sb && (s & 1) && s + 2 < Sb && lab[(s >> 1) + 1] != lab[s >> 1]);
    skip |= (uint32_t)sk << k;
  }
  // first step: the two states a path can start (alpha) or end (beta) in
  int t = BACK ? Tb - 1 : 0;
  float lm = -INFINITY;
#pragma unroll
  for (int k = 0; k < K; k++) {
    const int s = k * CTC_REC_THREADS + tid;
    const bool start = BACK ? (s >= Sb - 2) : (s < 2);
    u[k] = (s < Sb && start) ? lpb[(size_t)t * Sp + s] : -INFINITY;
    if (s < Sb) buf[s] = u[k];
    lm = fmaxf(lm, u[k]);
  }
  lm = warp_max(lm);
  if (lane == 0) wmax[0][warp] = lm;
  const int step = BACK ? -1 : 1;
#pragma unroll
  for (int k = 0; k < K; k++) {
    const int s = k * CTC_REC_THREADS + tid;
    lpn[k] = (s < Sb && Tb > 1) ? lpb[(size_t)(t + step) * Sp + s] : 0.f;
  }
  __syncthreads();
  float C = 0.f, comp = 0.f;                                   // Kahan sum of the scales c_t
  for (int i = 1; i <= Tb; i++) {
    const int p = (i - 1) & 1;
    float c = wmax[p][0];
#pragma unroll
    for (int w = 1; w < CTC_REC_THREADS / 32; w++) c = fmaxf(c, wmax[p][w]);
    if (c == -INFINITY) c = 0.f;                               // no state reachable: nothing to rescale
    {
      const float y = c - comp, s2 = C + y;
      comp = (s2 - C) - y;
      C = s2;
    }
#pragma unroll
    for (int k = 0; k < K; k++) {
      const int s = k * CTC_REC_THREADS + tid;
      if (s < Sb) ob[(size_t)t * Sp + s] = u[k] - c;
    }
    if (i == Tb) break;
    t += step;
    const float* prev = buf + p * Sp;
    float* cur = buf + (p ^ 1) * Sp;
    lm = -INFINITY;
#pragma unroll
    for (int k = 0; k < K; k++) {
      const int s = k * CTC_REC_THREADS + tid;
      if (s < Sb) {
        const float a0 = prev[s];
        const float a1 = BACK ? (s + 1 < Sb ? prev[s + 1] : -INFINITY) : (s >= 1 ? prev[s - 1] : -INFINITY);
        const float a2 = ((skip >> k) & 1u) ? prev[BACK ? s + 2 : s - 2] : -INFINITY;
        u[k] = lpn[k] + (lse3(a0, a1, a2) - c);
        cur[s] = u[k];
        lm = fmaxf(lm, u[k]);
      }
    }
    const bool more = i + 1 < Tb;
#pragma unroll
    for (int k = 0; k < K; k++) {                              // prefetch lp' of the next step under the barrier
      const int s = k * CTC_REC_THREADS + tid;
      if (s < Sb && more) lpn[k] = lpb[(size_t)(t + step) * Sp + s];
    }
    lm = warp_max(lm);
    if (lane == 0) wmax[p ^ 1][warp] = lm;
    __syncthreads();
  }
  if (!BACK && tid == 0) {
    // buf of the last step holds u_{T_b - 1}; C includes its scale
    const float* last = buf + ((Tb - 1) & 1) * Sp;
    float c = wmax[(Tb - 1) & 1][0];
    for (int w = 1; w < CTC_REC_THREADS / 32; w++) c = fmaxf(c, wmax[(Tb - 1) & 1][w]);
    if (c == -INFINITY) c = 0.f;
    const float e1 = last[Sb - 1] - c, e2 = Sb >= 2 ? last[Sb - 2] - c : -INFINITY;
    const float m = fmaxf(e1, e2);
    const float l = m == -INFINITY ? -INFINITY : m + logf(expf(e1 - m) + expf(e2 - m));
    nll[b] = -(C + (l - comp));
  }
}

// Fixed-order block sum of one value per thread (every thread gets it); red: CTC_GRAD_THREADS / 32 floats of shared memory.
__device__ __forceinline__ float block_sum_fixed(float v, float* red) {
  v = warp_sum(v);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float s = 0.f;
  for (int w = 0; w < CTC_GRAD_THREADS / 32; w++) s += red[w];
  __syncthreads();
  return s;
}
__device__ __forceinline__ float block_max(float v, float* red) {
  v = warp_max(v);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float s = red[0];
  for (int w = 1; w < CTC_GRAD_THREADS / 32; w++) s = fmaxf(s, red[w]);
  __syncthreads();
  return s;
}

__global__ void __launch_bounds__(CTC_GRAD_THREADS) ctc_grad_kernel(const float* __restrict__ logits, const int64_t* __restrict__ targets,
                                                                    const int32_t* __restrict__ in_len, const int32_t* __restrict__ tgt_len,
                                                                    const float* __restrict__ nll, const float* __restrict__ dloss,
                                                                    CtcWs w, float* __restrict__ dlogits, int B, int T, int V, int S,
                                                                    int Lmax) {
  extern __shared__ float gamma[];                             // [Sp]
  __shared__ float red[CTC_GRAD_THREADS / 32];
  const int r = blockIdx.x, b = r / T, t = r - b * T, tid = threadIdx.x;
  const int Tb = in_len[b], Lb = tgt_len[b];
  float* dz = dlogits + (size_t)r * V;
  const bool ok = ctc_lengths_ok(Tb, Lb, T, Lmax);
  if (ok && t >= Tb) {                                         // frames past the utterance do not enter the loss
    for (int v = tid; v < V; v += CTC_GRAD_THREADS) dz[v] = 0.f;
    return;
  }
  const float nb = ok ? nll[b] : NAN;
  if (!(nb < INFINITY)) {                                      // infeasible (+inf) or broken: NaN, as torch's backward gives
    for (int v = tid; v < V; v += CTC_GRAD_THREADS) dz[v] = NAN;
    return;
  }
  const float g = (dloss[0] / (float)B) / (float)(Lb > 1 ? Lb : 1);
  const int Sb = 2 * Lb + 1;
  const size_t Sp = 2 * (size_t)Lmax + 1, o = (size_t)r * Sp;
  float m = -INFINITY;
  for (int s = tid; s < Sb; s += CTC_GRAD_THREADS) {
    const float ws = w.alpha[o + s] + w.beta[o + s] - w.lp[o + s];
    gamma[s] = ws;
    m = fmaxf(m, ws);
  }
  m = block_max(m, red);
  float z = 0.f;
  for (int s = tid; s < Sb; s += CTC_GRAD_THREADS) {
    const float e = expf(gamma[s] - m);
    gamma[s] = e;
    z += e;
  }
  z = block_sum_fixed(z, red);
  const float inv_z = 1.f / z;
  float g0 = 0.f;                                              // the blank's occupation: even states, and odd ones labelled 0
  for (int s = tid; s < Sb; s += CTC_GRAD_THREADS) {
    const float gs = gamma[s] * inv_z;
    gamma[s] = gs;
    if (!(s & 1) || targets[(size_t)b * S + (s >> 1)] == 0) g0 += gs;
  }
  g0 = block_sum_fixed(g0, red);                               // also orders the gamma writes before the chain walks
  const float* x = logits + (size_t)r * V;
  const float mx = w.row[2 * (size_t)r], lt = w.row[2 * (size_t)r + 1];
  for (int v = tid; v < V; v += CTC_GRAD_THREADS) dz[v] = g * expf((x[v] - mx) - lt);
  __syncthreads();
  if (tid == 0) dz[0] = g * (expf((x[0] - mx) - lt) - g0);
  for (int i = tid; i < Lb; i += CTC_GRAD_THREADS) {
    const int64_t l = targets[(size_t)b * S + i];
    if (l <= 0 || l >= V || !w.first[(size_t)b * Lmax + i]) continue;
    float acc = 0.f;                                           // the label's states in increasing order
    for (int j = i; j >= 0; j = w.next_same[(size_t)b * Lmax + j]) acc += gamma[2 * j + 1];
    dz[l] = g * (expf((x[l] - mx) - lt) - acc);
  }
}

// loss = (sum over b, in order, of nll_b / max(L_b, 1)) / B
__global__ void ctc_mean_kernel(const float* __restrict__ nll, const int32_t* __restrict__ tgt_len, float* __restrict__ loss, int B) {
  float s = 0.f;
  for (int b = 0; b < B; b++) {
    const int l = tgt_len[b];
    s += nll[b] / (float)(l > 1 ? l : 1);
  }
  loss[0] = s / (float)B;
}

static int ctc_k(int Lmax) {
  const int states = 2 * Lmax + 1;
  int k = 1;
  while (k * CTC_REC_THREADS < states) k *= 2;
  return k;
}

template <bool BACK>
static int launch_rec(int K, const int64_t* targets, const int32_t* in_len, const int32_t* tgt_len, const float* lp, float* out,
                      float* nll, int* next_same, int* first, int B, int T, int S, int Lmax, cudaStream_t st) {
  const int smem = (int)(sizeof(int) * (size_t)Lmax + sizeof(float) * 2 * (2 * (size_t)Lmax + 1));
  void (*kern)(const int64_t*, const int32_t*, const int32_t*, const float*, float*, float*, int*, int*, int, int, int) = nullptr;
  static bool done[6][kMaxDevices];
  int which = 0;
  switch (K) {
    case 1: kern = ctc_rec_kernel<1, BACK>; which = 0; break;
    case 2: kern = ctc_rec_kernel<2, BACK>; which = 1; break;
    case 4: kern = ctc_rec_kernel<4, BACK>; which = 2; break;
    case 8: kern = ctc_rec_kernel<8, BACK>; which = 3; break;
    case 16: kern = ctc_rec_kernel<16, BACK>; which = 4; break;
    default: kern = ctc_rec_kernel<32, BACK>; which = 5; break;
  }
  // the attribute is set once per device, so to the largest size any call can ask for
  constexpr int kMaxSmem = (int)(sizeof(int) * ((CTC_MAX_STATES - 1) / 2) + sizeof(float) * 2 * (CTC_MAX_STATES - 1));
  if (int rc = ensure_dynamic_smem((const void*)kern, kMaxSmem, done[which], BACK ? "ctc_beta" : "ctc_alpha")) return rc;
  kern<<<B, CTC_REC_THREADS, smem, st>>>(targets, in_len, tgt_len, lp, out, nll, next_same, first, T, S, Lmax);
  return check_launch(BACK ? "ctc_beta" : "ctc_alpha");
}

}  // namespace b200asr

using namespace b200asr;

extern "C" {

size_t b200asr_ctc_ws_bytes(int B, int T, int max_target_len) {
  if (B <= 0 || T <= 0 || max_target_len < 0) return 0;
  const size_t rows = (size_t)B * T, Sp = 2 * (size_t)max_target_len + 1;
  return sizeof(float) * (2 * rows + 3 * rows * Sp) + sizeof(int) * 2 * (size_t)B * max_target_len;
}

#define CTC_CHECK_ARGS(what)                                                                                                     \
  B200_REQUIRE(logits && targets && input_lengths && target_lengths && nll && ws, B200ASR_BAD_ARG, what ": null pointer");      \
  B200_REQUIRE(B >= 1 && T >= 1 && V >= 1 && S >= 0 && max_target_len >= 0 && max_target_len <= S &&                           \
                   2 * max_target_len + 1 <= CTC_MAX_STATES,                                                                    \
               B200ASR_BAD_SHAPE, what ": B=%d T=%d V=%d S=%d max_target_len=%d (need >= 1, max_target_len <= S and <= %d)", B, \
               T, V, S, max_target_len, (CTC_MAX_STATES - 1) / 2)

int b200asr_ctc_fwd(const float* logits, const int64_t* targets, const int32_t* input_lengths, const int32_t* target_lengths,
                    float* nll, float* loss, void* ws, int B, int T, int V, int S, int max_target_len, b200asr_stream_t stream) {
  CTC_CHECK_ARGS("ctc_fwd");
  B200_REQUIRE(loss, B200ASR_BAD_ARG, "ctc_fwd: null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  const CtcWs w = ctc_ws(ws, B, T, max_target_len);
  ctc_lp_kernel<<<B * T, CTC_LP_THREADS, 0, st>>>(logits, targets, input_lengths, target_lengths, w.row, w.lp, T, V, S, max_target_len);
  if (int rc = check_launch("ctc_lp")) return rc;
  if (int rc = launch_rec<false>(ctc_k(max_target_len), targets, input_lengths, target_lengths, w.lp, w.alpha, nll, w.next_same,
                                 w.first, B, T, S, max_target_len, st))
    return rc;
  ctc_mean_kernel<<<1, 1, 0, st>>>(nll, target_lengths, loss, B);
  return check_launch("ctc_mean");
}

int b200asr_ctc_bwd(const float* logits, const int64_t* targets, const int32_t* input_lengths, const int32_t* target_lengths,
                    const float* nll, const float* dloss, float* dlogits, void* ws, int B, int T, int V, int S, int max_target_len,
                    b200asr_stream_t stream) {
  CTC_CHECK_ARGS("ctc_bwd");
  B200_REQUIRE(dloss && dlogits, B200ASR_BAD_ARG, "ctc_bwd: null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  const CtcWs w = ctc_ws(ws, B, T, max_target_len);
  if (int rc = launch_rec<true>(ctc_k(max_target_len), targets, input_lengths, target_lengths, w.lp, w.beta, nullptr, nullptr,
                                nullptr, B, T, S, max_target_len, st))
    return rc;
  const int smem = (int)(sizeof(float) * (2 * (size_t)max_target_len + 1));   // <= 32 KB: no opt-in needed
  ctc_grad_kernel<<<B * T, CTC_GRAD_THREADS, smem, st>>>(logits, targets, input_lengths, target_lengths, nll, dloss, w, dlogits, B, T,
                                                         V, S, max_target_len);
  return check_launch("ctc_grad");
}

}  // extern "C"
