// Batched beam search (Decoder.beam_search, models/asr/transformer.py:396-517) on the device: the per-step selection, EOS
// bookkeeping, word counting and n-best pool (beam_step), single-query self-attention over a shared K/V cache addressed
// through a per-row index table (beam_self_attn) and the final walk along the back-pointers (beam_backtrack).
#include <math.h>

#include "../../include/b200asr.h"
#include "common.cuh"

namespace b200asr {

constexpr int BEAM_MAX = 32;          // beam width and n-best limit
constexpr int BEAM_THREADS = 256;
constexpr int BEAM_MAX_T = 8192;      // longest self-attention history (positions) of beam_self_attn
constexpr int TOK_PAD_ID = 0, TOK_SOS_ID = 1, TOK_EOS_ID = 2;

// (value, index) order of the search: larger value first, then the smaller index
__device__ __forceinline__ bool beam_before(float v, int i, float ov, int oi) { return v > ov || (v == ov && i < oi); }

// Best (value, index) of the warp that comes strictly after (pv, pi) in beam_before order: the k-th call of a loop that
// feeds back its own result yields the k-th element, so a row's top-W needs no sorting and no marks.
__device__ __forceinline__ void warp_best_after(float& bv, int& bi) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (beam_before(ov, oi, bv, bi)) { bv = ov; bi = oi; }
  }
}

// One CTA per utterance b; rows b*W .. b*W+W-1 of `logits` are its beam slots.
__global__ void __launch_bounds__(BEAM_THREADS) beam_step_kernel(
    const float* __restrict__ logits, const int32_t* __restrict__ word_tab, int W, int V, int t, int t_eos, int nbest,
    double c_weight, float* __restrict__ score, int32_t* __restrict__ state, int64_t* __restrict__ next_tok,
    const int32_t* __restrict__ idx_cur, int32_t* __restrict__ idx_nxt, int idx_stride, int32_t* __restrict__ hist_tok,
    int32_t* __restrict__ hist_par, float* __restrict__ pool_score, float* __restrict__ pool_final,
    int32_t* __restrict__ pool_ref, int32_t* __restrict__ pool_n, int32_t* __restrict__ n_live, int BW,
    int32_t* __restrict__ end_ref, float* __restrict__ end_score, int32_t* __restrict__ end_n, int end_cap) {
  __shared__ float c_val[BEAM_MAX * BEAM_MAX];     // candidate scores, index parent * W + rank
  __shared__ int c_tok[BEAM_MAX * BEAM_MAX];
  __shared__ float p_score[BEAM_MAX];
  __shared__ int p_state[BEAM_MAX][4];
  __shared__ int kept[BEAM_MAX];
  __shared__ int src_slot[BEAM_MAX];
  __shared__ int n_kept_s, n_surv_s;
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int row0 = b * W;
  if (tid < W) {
    p_score[tid] = score[row0 + tid];
#pragma unroll
    for (int f = 0; f < 4; f++) p_state[tid][f] = state[(size_t)(row0 + tid) * 4 + f];
  }
  __syncthreads();

  // 1. per live row: fp32 log_softmax of the logits and its top-W (ties to the lower token id), as score + logp
  for (int j = warp; j < W; j += BEAM_THREADS / 32) {
    if (!p_state[j][0]) continue;
    const float* x = logits + (size_t)(row0 + j) * V;
    float mx = -INFINITY;
    for (int c = lane; c < V; c += 32) mx = fmaxf(mx, x[c]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    float s = 0.f;
    for (int c = lane; c < V; c += 32) s += expf(x[c] - mx);
    s = warp_sum(s);
    const float lt = logf(s);
    float pv = INFINITY;
    int pi = -1;
    for (int r = 0; r < W; r++) {
      float bv = -INFINITY;
      int bi = 0x7fffffff;
      for (int c = lane; c < V; c += 32) {
        const float lp = (x[c] - mx) - lt;
        if (beam_before(pv, pi, lp, c) && beam_before(lp, c, bv, bi)) { bv = lp; bi = c; }
      }
      warp_best_after(bv, bi);
      if (bi == 0x7fffffff) bi = 0;           // only non-finite logits left: keep the index valid
      if (lane == 0) { c_val[j * W + r] = p_score[j] + bv; c_tok[j * W + r] = bi; }
      pv = bv; pi = bi;
    }
  }
  __syncthreads();

  // 2. merge to W: global top-W of every (parent, rank) candidate by score, ties to the earlier parent, then rank -- what the
  //    reference's stable sorted(...)[:W] after each parent keeps (transformer.py:466)
  if (warp == 0) {
    float pv = INFINITY;
    int pi = -1, n = 0;
    for (int k = 0; k < W; k++) {
      float bv = -INFINITY;
      int bi = 0x7fffffff;
      for (int c = lane; c < W * W; c += 32) {
        if (!p_state[c / W][0]) continue;
        const float v = c_val[c];
        if (beam_before(pv, pi, v, c) && beam_before(v, c, bv, bi)) { bv = v; bi = c; }
      }
      warp_best_after(bv, bi);
      if (bi == 0x7fffffff) break;             // no live parent
      if (lane == 0) kept[k] = bi;
      pv = bv; pi = bi; n++;
    }
    if (lane == 0) n_kept_s = n;
  }
  __syncthreads();

  // 3. forced EOS, word state, final score, n-best pool and compaction, in kept order (transformer.py:470-497)
  if (tid == 0) {
    const int n_kept = n_kept_s;
    const bool forced = t == t_eos;
    int n = 0, pn = pool_n[b];
    float* ps = pool_score + (size_t)b * nbest;
    float* pf = pool_final + (size_t)b * nbest;
    int32_t* pr = pool_ref + (size_t)b * nbest;
    for (int k = 0; k < n_kept; k++) {
      const int c = kept[k], j = c / W, tok = c_tok[c];
      const float sc = c_val[c];
      const int rec = word_tab[tok];           // w * 8 + head * 4 + tail * 2 + empty
      int words = p_state[j][1], tail = p_state[j][2];
      words += (rec >> 3) - (tail & (rec >> 2) & 1);
      if (!(rec & 1)) tail = (rec >> 1) & 1;
      hist_tok[(size_t)t * BW + row0 + k] = tok;
      hist_par[(size_t)t * BW + row0 + k] = p_state[j][3];
      if (forced || tok == TOK_EOS_ID) {
        const int ref = ((t * W + k) << 1) | (forced ? 1 : 0);
        if (end_ref) {                         // end log: every ended hypothesis, in insertion order
          const int e = end_n[b];
          end_ref[(size_t)b * end_cap + e] = ref;
          end_score[(size_t)b * end_cap + e] = sc;
          end_n[b] = e + 1;
        }
        const float fs = sc + (float)(sqrt((double)words) * c_weight);
        int pos = 0;                           // stable: after every entry with an equal or larger final score
        while (pos < pn && !(fs > pf[pos])) pos++;
        if (pos < nbest) {
          const int last = pn < nbest ? pn : nbest - 1;
          for (int q = last; q > pos; q--) { ps[q] = ps[q - 1]; pf[q] = pf[q - 1]; pr[q] = pr[q - 1]; }
          ps[pos] = sc; pf[pos] = fs; pr[pos] = ref;
          if (pn < nbest) pn++;
        }
      } else {
        const int r = row0 + n;
        score[r] = sc;
        state[(size_t)r * 4 + 0] = 1; state[(size_t)r * 4 + 1] = words;
        state[(size_t)r * 4 + 2] = tail; state[(size_t)r * 4 + 3] = k;
        next_tok[r] = tok;
        src_slot[n++] = j;
      }
    }
    for (int s = n; s < W; s++) {
      const int r = row0 + s;
      score[r] = -INFINITY;
      state[(size_t)r * 4 + 0] = 0; state[(size_t)r * 4 + 1] = 0; state[(size_t)r * 4 + 2] = 0; state[(size_t)r * 4 + 3] = -1;
      next_tok[r] = TOK_PAD_ID;
    }
    pool_n[b] = pn;
    n_surv_s = n;
    if (n_kept > 0 && n == 0) atomicSub(n_live, 1);
  }
  __syncthreads();

  // 4. index table of the next step: a survivor's history is its parent's positions 0..t, then its own slot at t + 1; a dead
  //    slot points at itself everywhere (its outputs are never selected, its reads stay in bounds)
  const int n = n_surv_s;
  for (int e = tid; e < W * (t + 2); e += BEAM_THREADS) {
    const int s = e / (t + 2), p = e - s * (t + 2);
    int v = s;
    if (s < n && p <= t) v = idx_cur[(size_t)(row0 + src_slot[s]) * idx_stride + p];
    idx_nxt[(size_t)(row0 + s) * idx_stride + p] = v;
  }
}

// One warp per (row, head): softmax(q k^T * scale) v over positions 0..t of the row's history, position p read from cache
// step p, slot idx[row][p] of the same utterance.  Exact fp32; the scores live in shared memory.
template <int DK, int DV>
__global__ void __launch_bounds__(128) beam_self_attn_kernel(const float* __restrict__ q, const float* __restrict__ kc,
                                                             const float* __restrict__ vc, const int32_t* __restrict__ idx,
                                                             float* __restrict__ out, int R, int H, int W, int t,
                                                             int idx_stride, float scale) {
  extern __shared__ float smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = blockIdx.x * 4 + warp;
  if (g >= R * H) return;
  const int r = g / H, h = g - r * H, base = r - r % W;
  const int T = t + 1;
  float* sq = smem + warp * (DK + T);
  float* sp = sq + DK;
  const float* qr = q + (size_t)r * H * DK + h * DK;
  for (int c = lane; c < DK; c += 32) sq[c] = qr[c];
  __syncwarp();
  const int32_t* ir = idx + (size_t)r * idx_stride;
  const size_t kstep = (size_t)R * H * DK, vstep = (size_t)R * H * DV;
  float mx = -INFINITY;
  for (int p = lane; p < T; p += 32) {
    const float4* kr = reinterpret_cast<const float4*>(kc + p * kstep + (size_t)(base + ir[p]) * H * DK + h * DK);
    float s = 0.f;
#pragma unroll
    for (int c = 0; c < DK / 4; c++) {
      const float4 kv = kr[c];
      s += sq[4 * c] * kv.x + sq[4 * c + 1] * kv.y + sq[4 * c + 2] * kv.z + sq[4 * c + 3] * kv.w;
    }
    s *= scale;
    sp[p] = s;
    mx = fmaxf(mx, s);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  float sum = 0.f;
  for (int p = lane; p < T; p += 32) {
    const float e = expf(sp[p] - mx);
    sp[p] = e;
    sum += e;
  }
  sum = warp_sum(sum);
  __syncwarp();
  constexpr int NA = DV >= 32 ? DV / 32 : 1;
  float acc[NA];
#pragma unroll
  for (int a = 0; a < NA; a++) acc[a] = 0.f;
  for (int p = 0; p < T; p++) {
    const float* vr = vc + p * vstep + (size_t)(base + ir[p]) * H * DV + h * DV;
    const float w = sp[p];
#pragma unroll
    for (int a = 0; a < NA; a++)
      if (a * 32 + lane < DV) acc[a] += w * vr[a * 32 + lane];
  }
  const float inv = 1.f / sum;
  float* o = out + (size_t)r * H * DV + h * DV;
#pragma unroll
  for (int a = 0; a < NA; a++)
    if (a * 32 + lane < DV) o[a * 32 + lane] = acc[a] * inv;
}

// One thread per ended hypothesis: SOS, the tokens along the back-pointers, the forced EOS if any.  Entry i of utterance b's
// list is refs[b * cap + i] ((t * W + k) * 2 + forced; valid for i < counts[b]).  Fixed-stride output (entries == nullptr):
// thread e = b * cap + i writes row e of ids [B * cap][steps + 2], -1 after the hypothesis, and lengths[e] (0: no entry).
// Packed output: thread j writes the t + 2 (+ 1 if forced) ids of entry entries[j] from ids + off[j].
__global__ void beam_backtrack_kernel(const int32_t* __restrict__ hist_tok, const int32_t* __restrict__ hist_par,
                                      const int32_t* __restrict__ refs, const int32_t* __restrict__ counts, int cap,
                                      const int64_t* __restrict__ entries, const int64_t* __restrict__ off, int n,
                                      int64_t* __restrict__ ids, int64_t* __restrict__ lengths, int B, int W, int steps) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  const int e = entries ? (int)entries[j] : j;
  const int b = e / cap, i = e - b * cap;
  const int L = steps + 2;
  int64_t* y = entries ? ids + off[j] : ids + (size_t)e * L;
  int len = 0;
  if (i < counts[b]) {
    const int ref = refs[e], forced = ref & 1;
    const int t = (ref >> 1) / W;
    int k = (ref >> 1) - t * W;
    len = t + 2 + forced;
    y[0] = TOK_SOS_ID;
    for (int s = t; s >= 0; s--) {
      const size_t hrow = (size_t)s * B * W + (size_t)b * W + k;
      y[s + 1] = hist_tok[hrow];
      k = hist_par[hrow];
    }
    if (forced) y[t + 2] = TOK_EOS_ID;
  }
  if (entries) return;
  for (int p = len; p < L; p++) y[p] = -1;
  lengths[e] = len;
}

template <int DK, int DV>
static int launch_self_attn(const float* q, const float* kc, const float* vc, const int32_t* idx, float* out, int R, int H,
                            int W, int t, int idx_stride, float scale, cudaStream_t st) {
  const int smem = 4 * (DK + t + 1) * (int)sizeof(float);
  static bool done[kMaxDevices] = {};
  if (smem > 48 * 1024) {      // reserved once per device, for the longest history accepted (t < BEAM_MAX_T)
    if (int rc = ensure_dynamic_smem((const void*)beam_self_attn_kernel<DK, DV>, 4 * (DK + BEAM_MAX_T) * (int)sizeof(float),
                                     done, "beam_self_attn"))
      return rc;
  }
  beam_self_attn_kernel<DK, DV><<<ceil_div(R * H, 4), 128, smem, st>>>(q, kc, vc, idx, out, R, H, W, t, idx_stride, scale);
  return check_launch("beam_self_attn");
}

template <int DK>
static int launch_self_attn_dv(int dv, const float* q, const float* kc, const float* vc, const int32_t* idx, float* out, int R,
                               int H, int W, int t, int idx_stride, float scale, cudaStream_t st) {
  switch (dv) {
    case 16: return launch_self_attn<DK, 16>(q, kc, vc, idx, out, R, H, W, t, idx_stride, scale, st);
    case 32: return launch_self_attn<DK, 32>(q, kc, vc, idx, out, R, H, W, t, idx_stride, scale, st);
    case 64: return launch_self_attn<DK, 64>(q, kc, vc, idx, out, R, H, W, t, idx_stride, scale, st);
    default: return launch_self_attn<DK, 128>(q, kc, vc, idx, out, R, H, W, t, idx_stride, scale, st);
  }
}

}  // namespace b200asr

using namespace b200asr;

static int beam_step_impl(const float* logits, const int32_t* word_tab, int B, int W, int V, int t, int t_eos, int steps,
                          int nbest, double c_weight, float* score, int32_t* state, int64_t* next_tok, const int32_t* idx_cur,
                          int32_t* idx_nxt, int idx_stride, int32_t* hist_tok, int32_t* hist_par, float* pool_score,
                          float* pool_final, int32_t* pool_ref, int32_t* pool_n, int32_t* n_live, int32_t* end_ref,
                          float* end_score, int32_t* end_n, int end_cap, b200asr_stream_t stream) {
  B200_REQUIRE(logits && word_tab && score && state && next_tok && idx_cur && idx_nxt && hist_tok && hist_par && pool_score &&
               pool_final && pool_ref && pool_n && n_live, B200ASR_BAD_ARG, "beam_step: null pointer");
  B200_REQUIRE(idx_cur != idx_nxt, B200ASR_BAD_ARG, "beam_step: idx_cur and idx_nxt must be different buffers");
  B200_REQUIRE(W >= 1 && W <= BEAM_MAX && W <= V, B200ASR_BAD_SHAPE, "beam_step: beam width W=%d must satisfy 1 <= W <= %d and W <= V=%d",
               W, BEAM_MAX, V);
  B200_REQUIRE(nbest >= 1 && nbest <= BEAM_MAX, B200ASR_BAD_SHAPE, "beam_step: nbest=%d must satisfy 1 <= nbest <= %d", nbest, BEAM_MAX);
  B200_REQUIRE(B >= 1 && t >= 0 && t < steps && idx_stride >= t + 2, B200ASR_BAD_SHAPE,
               "beam_step: B=%d t=%d steps=%d idx_stride=%d (need B >= 1, 0 <= t < steps, idx_stride >= t + 2)", B, t, steps,
               idx_stride);
  beam_step_kernel<<<B, BEAM_THREADS, 0, (cudaStream_t)stream>>>(logits, word_tab, W, V, t, t_eos, nbest, c_weight, score, state,
                                                                 next_tok, idx_cur, idx_nxt, idx_stride, hist_tok, hist_par,
                                                                 pool_score, pool_final, pool_ref, pool_n, n_live, B * W, end_ref,
                                                                 end_score, end_n, end_cap);
  return check_launch("beam_step");
}

extern "C" {

int b200asr_beam_step(const float* logits, const int32_t* word_tab, int B, int W, int V, int t, int t_eos, int steps, int nbest,
                      double c_weight, float* score, int32_t* state, int64_t* next_tok, const int32_t* idx_cur,
                      int32_t* idx_nxt, int idx_stride, int32_t* hist_tok, int32_t* hist_par, float* pool_score,
                      float* pool_final, int32_t* pool_ref, int32_t* pool_n, int32_t* n_live, b200asr_stream_t stream) {
  return beam_step_impl(logits, word_tab, B, W, V, t, t_eos, steps, nbest, c_weight, score, state, next_tok, idx_cur, idx_nxt,
                        idx_stride, hist_tok, hist_par, pool_score, pool_final, pool_ref, pool_n, n_live, nullptr, nullptr,
                        nullptr, 0, stream);
}

int b200asr_beam_step_log(const float* logits, const int32_t* word_tab, int B, int W, int V, int t, int t_eos, int steps,
                          int nbest, double c_weight, float* score, int32_t* state, int64_t* next_tok, const int32_t* idx_cur,
                          int32_t* idx_nxt, int idx_stride, int32_t* hist_tok, int32_t* hist_par, float* pool_score,
                          float* pool_final, int32_t* pool_ref, int32_t* pool_n, int32_t* n_live, int32_t* end_ref,
                          float* end_score, int32_t* end_n, int end_cap, b200asr_stream_t stream) {
  B200_REQUIRE(end_ref && end_score && end_n, B200ASR_BAD_ARG, "beam_step_log: null pointer");
  B200_REQUIRE(end_cap >= W * steps && W >= 1, B200ASR_BAD_SHAPE, "beam_step_log: end_cap=%d must be >= W * steps = %d", end_cap,
               W * steps);
  return beam_step_impl(logits, word_tab, B, W, V, t, t_eos, steps, nbest, c_weight, score, state, next_tok, idx_cur, idx_nxt,
                        idx_stride, hist_tok, hist_par, pool_score, pool_final, pool_ref, pool_n, n_live, end_ref, end_score,
                        end_n, end_cap, stream);
}

int b200asr_beam_self_attn(const float* q, const float* k_cache, const float* v_cache, const int32_t* idx, float* out, int R,
                           int H, int W, int dk, int dv, int t, int idx_stride, float scale, b200asr_stream_t stream) {
  B200_REQUIRE(q && k_cache && v_cache && idx && out, B200ASR_BAD_ARG, "beam_self_attn: null pointer");
  B200_REQUIRE((dk == 16 || dk == 32 || dk == 64 || dk == 128) && (dv == 16 || dv == 32 || dv == 64 || dv == 128),
               B200ASR_BAD_SHAPE, "beam_self_attn: head dims (dk=%d, dv=%d) must each be 16, 32, 64 or 128", dk, dv);
  B200_REQUIRE(R >= 1 && H >= 1 && W >= 1 && R % W == 0 && t >= 0 && idx_stride >= t + 1 && t < BEAM_MAX_T, B200ASR_BAD_SHAPE,
               "beam_self_attn: R=%d H=%d W=%d t=%d idx_stride=%d (need R a multiple of W, idx_stride > t, t < %d)", R, H, W,
               t, idx_stride, BEAM_MAX_T);
  B200_REQUIRE(aligned16(k_cache) && aligned16(v_cache), B200ASR_BAD_ALIGN, "beam_self_attn: K/V caches must be 16-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  switch (dk) {
    case 16: return launch_self_attn_dv<16>(dv, q, k_cache, v_cache, idx, out, R, H, W, t, idx_stride, scale, st);
    case 32: return launch_self_attn_dv<32>(dv, q, k_cache, v_cache, idx, out, R, H, W, t, idx_stride, scale, st);
    case 64: return launch_self_attn_dv<64>(dv, q, k_cache, v_cache, idx, out, R, H, W, t, idx_stride, scale, st);
    default: return launch_self_attn_dv<128>(dv, q, k_cache, v_cache, idx, out, R, H, W, t, idx_stride, scale, st);
  }
}

int b200asr_beam_backtrack(const int32_t* hist_tok, const int32_t* hist_par, const int32_t* pool_ref, const int32_t* pool_n,
                           int64_t* ids, int64_t* lengths, int B, int W, int nbest, int steps, b200asr_stream_t stream) {
  B200_REQUIRE(hist_tok && hist_par && pool_ref && pool_n && ids && lengths, B200ASR_BAD_ARG, "beam_backtrack: null pointer");
  B200_REQUIRE(B >= 1 && W >= 1 && W <= BEAM_MAX && nbest >= 1 && nbest <= BEAM_MAX && steps >= 1, B200ASR_BAD_SHAPE,
               "beam_backtrack: B=%d W=%d nbest=%d steps=%d", B, W, nbest, steps);
  beam_backtrack_kernel<<<ceil_div(B * nbest, 128), 128, 0, (cudaStream_t)stream>>>(
      hist_tok, hist_par, pool_ref, pool_n, nbest, nullptr, nullptr, B * nbest, ids, lengths, B, W, steps);
  return check_launch("beam_backtrack");
}

int b200asr_beam_backtrack_packed(const int32_t* hist_tok, const int32_t* hist_par, const int32_t* end_ref, const int32_t* end_n,
                                  int end_cap, const int64_t* entries, const int64_t* offsets, int n, int64_t* ids, int B, int W,
                                  int steps, b200asr_stream_t stream) {
  B200_REQUIRE(hist_tok && hist_par && end_ref && end_n && entries && offsets && ids, B200ASR_BAD_ARG,
               "beam_backtrack_packed: null pointer");
  B200_REQUIRE(B >= 1 && W >= 1 && W <= BEAM_MAX && steps >= 1 && end_cap >= 1 && n >= 0, B200ASR_BAD_SHAPE,
               "beam_backtrack_packed: B=%d W=%d steps=%d end_cap=%d n=%d", B, W, steps, end_cap, n);
  if (n == 0) return B200ASR_OK;
  beam_backtrack_kernel<<<ceil_div(n, 128), 128, 0, (cudaStream_t)stream>>>(hist_tok, hist_par, end_ref, end_n, end_cap, entries,
                                                                            offsets, n, ids, nullptr, B, W, steps);
  return check_launch("beam_backtrack_packed");
}

}  // extern "C"
