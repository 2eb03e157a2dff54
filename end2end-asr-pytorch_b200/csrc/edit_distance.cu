// Edit counts of the training loop's CER / WER (b200asr_edit_counts): per utterance, the strings the trainer joins from
// id2label (trainer/asr/trainer.py:60-79, 96-104) are expanded on the device from a label table and compared with an exact
// Levenshtein distance, over code points without ' ' (calculate_cer) and over whitespace-separated words (calculate_wer).
//
// One CTA per utterance.  The CTA expands both strings into one int buffer -- shared memory when it fits, the utterance's
// slice of the workspace otherwise -- packing each code point with its flags, splits them into words, gives every word the
// index of the first word with the same code points (so the word DP compares ints and word equality is exact), and runs two
// anti-diagonal DPs with three rolling diagonals.  A second, single-thread kernel sums the per-utterance counts in utterance
// order and finds the first invalid id.  No atomics: the same inputs give the same bits on every call.
#include <limits.h>

#include "../../include/b200asr.h"
#include "common.cuh"

namespace b200asr {

constexpr int EC_THREADS = 256;
constexpr int EC_WARPS = EC_THREADS / 32;
constexpr int EC_SMEM_BYTES = 46 * 1024;               // + the scans' static arrays: under the 48 KB that need no opt-in
constexpr int EC_SPACE = 1 << 24;                      // packed flag: the code point is ' ' (U+0020)
constexpr int EC_WS = 1 << 25;                         // packed flag: str.isspace()
constexpr int EC_CP = (1 << 24) - 1;
constexpr long long EC_MAX_INTS = 1LL << 30;           // per-utterance buffer limit (int32 entries)

// Int32 entries one utterance needs for hyp / gold strings of Lh / Lg code points: both strings, both without ' ',
// word starts / lengths / ids ((L + 1) / 2 words at most per side) and three diagonals of the shorter DP side + 1.
__host__ __device__ inline long long ec_need(long long Lh, long long Lg) {
  const long long words = (Lh + 1) / 2 + (Lg + 1) / 2;
  return 2 * (Lh + Lg) + 3 * words + 3 * ((Lh < Lg ? Lh : Lg) + 1);
}

static long long ec_cap(int T_h, int T_g, int max_label_len) {
  return ec_need((long long)T_h * max_label_len, (long long)T_g * max_label_len);
}

struct EcTable {
  const int* off;
  const int* len;
  const int* cp;
  const uint8_t* flags;
  const uint8_t* valid;
  int V;
};

__device__ __forceinline__ long long ec_load_id(const void* ids, int i64, long long idx) {
  return i64 ? static_cast<const long long*>(ids)[idx] : (long long)static_cast<const int*>(ids)[idx];
}

__device__ __forceinline__ bool ec_valid(const EcTable& tb, long long id) {
  return id >= 0 && id < tb.V && tb.valid[id] != 0;
}

// Exclusive prefix sum over the CTA's threads, thread order; `total` gets the sum of all.  Ends with a barrier.
template <typename T>
__device__ __forceinline__ T ec_scan(T v, T& total) {
  __shared__ T wsum[EC_WARPS];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  T x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const T y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  if (lane == 31) wsum[warp] = x;
  __syncthreads();
  T before = 0, tot = 0;
#pragma unroll
  for (int w = 0; w < EC_WARPS; w++) {
    if (w < warp) before += wsum[w];
    tot += wsum[w];
  }
  __syncthreads();
  total = tot;
  return before + x - v;
}

__device__ __forceinline__ long long ec_min(long long v) {
  __shared__ long long wmin[EC_WARPS];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = min(v, __shfl_xor_sync(0xffffffffu, v, o));
  if (lane == 0) wmin[warp] = v;
  __syncthreads();
  long long m = wmin[0];
#pragma unroll
  for (int w = 1; w < EC_WARPS; w++) m = min(m, wmin[w]);
  __syncthreads();
  return m;
}

// Tokens before the first PAD (*p), their code-point count (returned) and the position of the first invalid id among them
// (*bad, -1 if none).  Invalid ids contribute no code points.
__device__ long long ec_measure(const void* ids, int i64, long long row, int T, long long pad, const EcTable& tb, int* p,
                                long long* bad) {
  long long first_pad = T;
  for (int t = threadIdx.x; t < T; t += EC_THREADS)
    if (ec_load_id(ids, i64, row + t) == pad) { first_pad = t; break; }
  *p = (int)ec_min(first_pad);
  long long n = 0, b = LLONG_MAX;
  for (int t = threadIdx.x; t < *p; t += EC_THREADS) {
    const long long id = ec_load_id(ids, i64, row + t);
    if (ec_valid(tb, id)) n += tb.len[id];
    else b = min(b, (long long)t);
  }
  long long total;
  ec_scan(n, total);
  b = ec_min(b);
  *bad = b == LLONG_MAX ? -1 : b;
  return total;
}

// Writes the packed code points of tokens [0, p) to s[0 ..).
__device__ void ec_expand(const void* ids, int i64, long long row, int p, const EcTable& tb, int* s) {
  int base = 0;
  for (int t0 = 0; t0 < p; t0 += EC_THREADS) {
    const int t = t0 + threadIdx.x;
    int n = 0, off = 0;
    if (t < p) {
      const long long id = ec_load_id(ids, i64, row + t);
      if (ec_valid(tb, id)) { n = tb.len[id]; off = tb.off[id]; }
    }
    int total;
    const int at = base + ec_scan(n, total);
    for (int k = 0; k < n; k++) s[at + k] = tb.cp[off + k] | ((int)(tb.flags[off + k] & 3) << 24);
    base += total;
  }
  __syncthreads();
}

// Over s[0, L): the code points other than ' ' go to nosp[0 ..) (count in *n_nosp); the words (maximal runs without
// isspace) get their start (index into buf) and length in wstart / wlen (count in *n_words).
__device__ void ec_split(const int* buf, int s0, int L, int* nosp, int* wstart, int* wlen, int* n_nosp, int* n_words) {
  const int* s = buf + s0;
  long long base = 0;                                  // (words << 32) | code points kept so far
  for (int i0 = 0; i0 < L; i0 += EC_THREADS) {
    const int i = i0 + threadIdx.x;
    bool keep = false, start = false;
    int c = 0;
    if (i < L) {
      c = s[i];
      keep = !(c & EC_SPACE);
      start = !(c & EC_WS) && (i == 0 || (s[i - 1] & EC_WS));
    }
    long long total;
    const long long at = base + ec_scan((long long)start << 32 | (long long)keep, total);
    if (keep) nosp[(int)(at & 0xffffffffLL)] = c & EC_CP;
    if (start) {
      int j = i + 1;
      while (j < L && !(s[j] & EC_WS)) j++;
      const int w = (int)(at >> 32);
      wstart[w] = s0 + i;
      wlen[w] = j - i;
    }
    base += total;
  }
  *n_nosp = (int)(base & 0xffffffffLL);
  *n_words = (int)(base >> 32);
}

// Levenshtein distance of a[0, n) and b[0, m) by anti-diagonals; diag holds 3 * (min(n, m) + 1) ints.  Every thread
// returns it.  The caller's writes to a and b must be behind a barrier.
__device__ int ec_levenshtein(const int* a, int n, const int* b, int m, int* diag) {
  if (n > m) {
    const int* t = a; a = b; b = t;
    const int k = n; n = m; m = k;
  }
  if (n == 0) return m;
  int* d0 = diag;                                      // diagonal d - 2, indexed by i
  int* d1 = diag + (n + 1);                            // diagonal d - 1
  int* d2 = diag + 2 * (n + 1);                        // diagonal d
  for (int d = 0; d <= n + m; d++) {
    const int lo = max(0, d - m), hi = min(n, d);
    for (int i = lo + threadIdx.x; i <= hi; i += EC_THREADS) {
      const int j = d - i;
      int v;
      if (i == 0) v = j;
      else if (j == 0) v = i;
      else v = min(min(d1[i - 1], d1[i]) + 1, d0[i - 1] + (a[i - 1] != b[j - 1] ? 1 : 0));
      d2[i] = v;
    }
    __syncthreads();
    int* t = d0; d0 = d1; d1 = d2; d2 = t;
  }
  const int dist = d1[n];
  __syncthreads();                                     // before diag is reused
  return dist;
}

// One CTA per utterance b: out[b] = {cer_edits, wer_edits, gold_chars, gold_words}; bad_pos[b] / bad_pos[B + b] = first invalid
// position in gold row b / hyp row b, or -1.  An utterance whose strings need more than `cap` ints (a label longer than the
// max_label_len the caller promised) gets -1 in all four counts.
__global__ void __launch_bounds__(EC_THREADS) edit_counts_kernel(
    const void* __restrict__ hyp, int hyp_i64, long long hyp_rs, int T_h, const void* __restrict__ gold, int gold_i64,
    long long gold_rs, int T_g, EcTable tb, long long pad, long long* __restrict__ out, long long* __restrict__ bad_pos,
    int* __restrict__ ws_str, long long cap, int smem_ints, int B) {
  extern __shared__ int ec_smem[];
  const int b = blockIdx.x;
  const long long hrow = (long long)b * hyp_rs, grow = (long long)b * gold_rs;
  int ph, pg;
  long long bad_h, bad_g;
  const long long Lh = ec_measure(hyp, hyp_i64, hrow, T_h, pad, tb, &ph, &bad_h);
  const long long Lg = ec_measure(gold, gold_i64, grow, T_g, pad, tb, &pg, &bad_g);
  if (threadIdx.x == 0) {
    bad_pos[b] = bad_g;
    bad_pos[B + b] = bad_h;
  }
  const long long need = ec_need(Lh, Lg);
  if (need > cap) {
    if (threadIdx.x < 4) out[(long long)b * 4 + threadIdx.x] = -1;
    return;
  }
  int* buf = need <= smem_ints ? ec_smem : ws_str + (long long)b * cap;
  const int nh = (int)Lh, ng = (int)Lg;
  const int wcap = (nh + 1) / 2 + (ng + 1) / 2;
  int* nosp = buf + nh + ng;                           // hyp without ' ' at nosp[0 ..), gold at nosp[nh ..)
  int* wstart = nosp + nh + ng;
  int* wlen = wstart + wcap;
  int* wid = wlen + wcap;
  int* diag = wid + wcap;

  ec_expand(hyp, hyp_i64, hrow, ph, tb, buf);
  ec_expand(gold, gold_i64, grow, pg, tb, buf + nh);
  int ch, cg, wh, wg;
  ec_split(buf, 0, nh, nosp, wstart, wlen, &ch, &wh);
  ec_split(buf, nh, ng, nosp + nh, wstart + wh, wlen + wh, &cg, &wg);
  __syncthreads();

  // word ids: the index of the first word (hyp words, then gold words) with the same code points
  for (int w = threadIdx.x; w < wh + wg; w += EC_THREADS) {
    const int* sw = buf + wstart[w];
    const int lw = wlen[w];
    int k = 0;
    for (; k < w; k++) {
      if (wlen[k] != lw) continue;
      const int* sk = buf + wstart[k];
      int e = 0;
      while (e < lw && ((sk[e] ^ sw[e]) & EC_CP) == 0) e++;
      if (e == lw) break;
    }
    wid[w] = k;
  }
  __syncthreads();

  const int cer = ec_levenshtein(nosp, ch, nosp + nh, cg, diag);
  const int wer = ec_levenshtein(wid, wh, wid + wh, wg, diag);
  if (threadIdx.x == 0) {
    long long* o = out + (long long)b * 4;
    o[0] = cer;
    o[1] = wer;
    o[2] = cg;
    o[3] = (long long)(ng - cg) + 1;
  }
}

// totals = {sum cer_edits, sum wer_edits, sum gold_chars, sum gold_words} in utterance order, then the first invalid id in the
// trainer's order (every gold row before any hyp row), or -1.
__global__ void edit_counts_total_kernel(const long long* __restrict__ out, const long long* __restrict__ bad_pos,
                                         const void* __restrict__ hyp, int hyp_i64, long long hyp_rs,
                                         const void* __restrict__ gold, int gold_i64, long long gold_rs, int B,
                                         long long* __restrict__ totals) {
  long long s[4] = {0, 0, 0, 0};
  for (int b = 0; b < B; b++)
    for (int k = 0; k < 4; k++) s[k] += out[(long long)b * 4 + k];
  long long first = -1;
  for (int r = 0; r < 2 * B; r++) {
    const long long pos = bad_pos[r];
    if (pos < 0) continue;
    first = r < B ? ec_load_id(gold, gold_i64, (long long)r * gold_rs + pos)
                  : ec_load_id(hyp, hyp_i64, (long long)(r - B) * hyp_rs + pos);
    break;
  }
  for (int k = 0; k < 4; k++) totals[k] = s[k];
  totals[4] = first;
}

static size_t ec_str_bytes(int B, int T_h, int T_g, int max_label_len) {
  const long long cap = ec_cap(T_h, T_g, max_label_len);
  return cap * 4 <= EC_SMEM_BYTES ? 0 : (size_t)B * (size_t)cap * 4;
}

}  // namespace b200asr

using namespace b200asr;

extern "C" {

size_t b200asr_edit_counts_ws_bytes(int B, int T_h, int T_g, int max_label_len) {
  if (B < 1 || T_h < 0 || T_g < 0 || max_label_len < 0 || ec_cap(T_h, T_g, max_label_len) > EC_MAX_INTS) return 0;
  return (size_t)B * 2 * sizeof(long long) + ec_str_bytes(B, T_h, T_g, max_label_len);
}

int b200asr_edit_counts(const void* hyp, int hyp_int64, long long hyp_row_stride, int T_h, const void* gold, int gold_int64,
                        long long gold_row_stride, int T_g, int B, const int* label_off, const int* label_len,
                        const int* code_points, const uint8_t* cp_flags, const uint8_t* label_valid, int V, int max_label_len,
                        long long pad_id, int64_t* per_utt, int64_t* totals, void* ws, b200asr_stream_t stream) {
  B200_REQUIRE(hyp && gold && label_off && label_len && code_points && cp_flags && label_valid && per_utt && totals && ws,
               B200ASR_BAD_ARG, "edit_counts: null pointer");
  B200_REQUIRE((hyp_int64 == 0 || hyp_int64 == 1) && (gold_int64 == 0 || gold_int64 == 1), B200ASR_BAD_ARG,
               "edit_counts: hyp_int64 / gold_int64 must be 0 (int32 ids) or 1 (int64 ids), got %d / %d", hyp_int64,
               gold_int64);
  B200_REQUIRE(B >= 1 && T_h >= 0 && T_g >= 0 && V >= 1 && max_label_len >= 0, B200ASR_BAD_SHAPE,
               "edit_counts: B=%d T_h=%d T_g=%d V=%d max_label_len=%d (need B, V >= 1 and T_h, T_g, max_label_len >= 0)", B,
               T_h, T_g, V, max_label_len);
  B200_REQUIRE(hyp_row_stride >= T_h && gold_row_stride >= T_g && (B == 1 || (hyp_row_stride >= 1 && gold_row_stride >= 1)),
               B200ASR_BAD_SHAPE, "edit_counts: row strides %lld / %lld must be >= T_h=%d / T_g=%d", hyp_row_stride,
               gold_row_stride, T_h, T_g);
  const long long cap = ec_cap(T_h, T_g, max_label_len);
  B200_REQUIRE(cap <= EC_MAX_INTS, B200ASR_BAD_SHAPE,
               "edit_counts: (T_h + T_g) * max_label_len too large (T_h=%d T_g=%d max_label_len=%d)", T_h, T_g,
               max_label_len);
  B200_REQUIRE(((uintptr_t)hyp % (hyp_int64 ? 8 : 4)) == 0 && ((uintptr_t)gold % (gold_int64 ? 8 : 4)) == 0 &&
                   ((uintptr_t)label_off % 4) == 0 && ((uintptr_t)label_len % 4) == 0 && ((uintptr_t)code_points % 4) == 0 &&
                   ((uintptr_t)per_utt % 8) == 0 && ((uintptr_t)totals % 8) == 0 && ((uintptr_t)ws % 16) == 0,
               B200ASR_BAD_ALIGN, "edit_counts: ids, table, outputs or ws not aligned to their element (ws: 16 bytes)");
  cudaStream_t st = (cudaStream_t)stream;
  long long* bad_pos = static_cast<long long*>(ws);
  int* ws_str = ec_str_bytes(B, T_h, T_g, max_label_len) ? reinterpret_cast<int*>(bad_pos + 2 * (size_t)B) : nullptr;
  const int smem_ints = (int)(cap * 4 <= EC_SMEM_BYTES ? cap : EC_SMEM_BYTES / 4);
  const EcTable tb = {label_off, label_len, code_points, cp_flags, label_valid, V};
  edit_counts_kernel<<<B, EC_THREADS, (size_t)smem_ints * 4, st>>>(hyp, hyp_int64, hyp_row_stride, T_h, gold, gold_int64,
                                                                   gold_row_stride, T_g, tb, pad_id, (long long*)per_utt,
                                                                   bad_pos, ws_str, cap, smem_ints, B);
  if (int rc = check_launch("edit_counts")) return rc;
  edit_counts_total_kernel<<<1, 1, 0, st>>>((const long long*)per_utt, bad_pos, hyp, hyp_int64, hyp_row_stride, gold,
                                            gold_int64, gold_row_stride, B, (long long*)totals);
  return check_launch("edit_counts_total");
}

}  // extern "C"
