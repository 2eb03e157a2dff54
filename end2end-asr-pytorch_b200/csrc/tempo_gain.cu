// Tempo and gain perturbation (WSOLA, modelled on sox's `tempo` effect with its default profile, then `gain` and a 16-bit
// output) over a packed batch of waveforms: one CTA per utterance, one launch per batch.  include/b200asr.h states the
// algorithm; the geometry (segment, search, overlap) comes from the caller.
//
// Segment k's input start S_k = floor(tempo * k * step + 0.5) does not depend on any pick, so while segment k is searched
// the window x~[S_{k+1} .. S_{k+1} + search + segment - 2] of the next segment is already on its way into shared memory
// (cp.async, two window buffers).  That window holds every sample segment k+1 reads: its candidates, its output samples and
// the overlap the segment after it is matched against, which is copied out as float64 `prev` once the pick is known.  The
// search gives each thread one candidate at a time and sums (x - prev)^2 over the overlap in float64 from a float64 copy of
// the window; the arg-min goes through warp shuffles and shared memory, ties to the smaller index.  The step samples are
// then written coalesced, crossfaded, scaled by the gain and quantised to 16 bits.
#include <float.h>
#include <limits.h>
#include <math.h>

#include "../../include/b200asr.h"
#include "common.cuh"

namespace b200asr {

constexpr int kTempoThreads = 256;
constexpr int kTempoWarps = kTempoThreads / 32;
constexpr long long kTempoMaxSmem = 226 * 1024;      // sm_90's 227 KB opt-in per CTA, less room for the static part

// dynamic shared memory: prev [2][overlap] and the window's float64 copy [search + overlap - 1] (doubles), then the two
// windows [2][search + segment - 1] (floats)
static long long tempo_smem_bytes(long long segment, long long search, long long overlap) {
  return (2 * overlap + search + overlap - 1) * (long long)sizeof(double) + 2 * (search + segment - 1) * (long long)sizeof(float);
}

__device__ __forceinline__ void cp_async4(float* dst, const float* src) {
  const unsigned s = (unsigned)__cvta_generic_to_shared(dst);
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(s), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_group 0;" ::: "memory"); }

// dst[t] = x~[S_k + t] for t < W: the samples of [0, n) by cp.async, zeros elsewhere (the zero extension is synthesised,
// nothing outside the utterance is read)
__device__ __forceinline__ void tempo_load_window(float* dst, const float* x, long long n, double tempo, long long k, int step,
                                                  int W) {
  const double s = floor(tempo * (double)(k * step) + 0.5);
  const long long s0 = s < (double)n ? (long long)s : n;        // past the end: all zeros, no int64 overflow
  for (int t = threadIdx.x; t < W; t += kTempoThreads) {
    const long long e = s0 + t;
    if (e < n) cp_async4(dst + t, x + e);
    else dst[t] = 0.f;
  }
  cp_async_commit();
}

// clamp(rint(v * 32768), -32768, 32767) / 32768, half to even; NaN stays NaN
__device__ __forceinline__ float tempo_quantise16(float v) {
  float q = rintf(__fmul_rn(v, 32768.f));
  q = q < -32768.f ? -32768.f : (q > 32767.f ? 32767.f : q);
  return __fmul_rn(q, 1.f / 32768.f);
}

__global__ void __launch_bounds__(kTempoThreads) tempo_gain_kernel(
    const float* __restrict__ in, const long long* __restrict__ in_offsets, const int* __restrict__ in_lengths,
    const double* __restrict__ tempo, const float* __restrict__ gain, float* __restrict__ out,
    const long long* __restrict__ out_offsets, const int* __restrict__ out_lengths, int* __restrict__ picks,
    const long long* __restrict__ pick_offsets, int segment, int search, int overlap) {
  extern __shared__ __align__(16) unsigned char tempo_smem[];
  double* prev = reinterpret_cast<double*>(tempo_smem);       // [2][overlap]: slot k & 1 is written by segment k
  double* wd = prev + 2 * overlap;                             // [search + overlap - 1]: the candidates' samples
  float* win = reinterpret_cast<float*>(wd + search + overlap - 1);   // [2][W]: slot k & 1 holds segment k's window
  __shared__ double red_d[kTempoWarps];
  __shared__ int red_i[kTempoWarps];
  __shared__ int pick_s;
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int W = search + segment - 1, step = segment - overlap, nd = search + overlap - 1;
  const long long ooff = out_offsets[b];
  const int olen = out_lengths[b];
  if (ooff < 0 || olen <= 0) return;                           // nowhere to write, or nothing
  const long long K = (olen + step - 1) / step;
  int* pk = nullptr;
  if (picks) {
    const long long po = pick_offsets[b];
    if (po >= 0) pk = picks + po;
  }
  float* o = out + ooff;
  const double t = tempo[b];
  const long long ioff = in_offsets[b];
  const int n = in_lengths[b];
  if (!(t > 0.0 && t <= DBL_MAX) || ioff < 0 || n < 0) {      // device data the host did not check: NaN out
    for (int i = tid; i < olen; i += kTempoThreads) o[i] = __int_as_float(0x7fc00000);
    if (pk)
      for (long long k = tid; k < K; k += kTempoThreads) pk[k] = -1;
    return;
  }
  const float g = gain[b];
  const float* x = in + ioff;
  const float rcp = __fdiv_rn(1.f, (float)overlap);
  int p = search / 2;
  tempo_load_window(win, x, n, t, 0, step, W);
  for (long long k = 0; k < K; k++) {
    const float* buf = win + (k & 1) * W;
    const double* pv = prev + ((k + 1) & 1) * overlap;          // written by segment k - 1
    cp_async_wait_all();
    __syncthreads();                                            // window k landed; segment k - 1 is done with its slots
    if (k + 1 < K) tempo_load_window(win + ((k + 1) & 1) * W, x, n, t, k + 1, step, W);
    if (k > 0) {
      for (int i = tid; i < nd; i += kTempoThreads) wd[i] = (double)buf[i];
      __syncthreads();
      double bd = INFINITY;
      int bi = INT_MAX;
      for (int i = tid; i < search; i += kTempoThreads) {       // increasing i: a strict < keeps the smaller index
        double d0 = 0.0, d1 = 0.0;
        int j = 0;
        for (; j + 1 < overlap; j += 2) {
          const double e0 = wd[i + j] - pv[j], e1 = wd[i + j + 1] - pv[j + 1];
          d0 = fma(e0, e0, d0);
          d1 = fma(e1, e1, d1);
        }
        if (j < overlap) {
          const double e0 = wd[i + j] - pv[j];
          d0 = fma(e0, e0, d0);
        }
        double d = d0 + d1;
        if (isnan(d)) d = INFINITY;
        if (d < bd || bi == INT_MAX) { bd = d; bi = i; }
      }
#pragma unroll
      for (int s = 16; s > 0; s >>= 1) {
        const double od = __shfl_xor_sync(0xffffffffu, bd, s);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, s);
        if (od < bd || (od == bd && oi < bi)) { bd = od; bi = oi; }
      }
      if (lane == 0) { red_d[warp] = bd; red_i[warp] = bi; }
      __syncthreads();
      if (warp == 0) {
        bd = lane < kTempoWarps ? red_d[lane] : INFINITY;
        bi = lane < kTempoWarps ? red_i[lane] : INT_MAX;
#pragma unroll
        for (int s = 16; s > 0; s >>= 1) {
          const double od = __shfl_xor_sync(0xffffffffu, bd, s);
          const int oi = __shfl_xor_sync(0xffffffffu, bi, s);
          if (od < bd || (od == bd && oi < bi)) { bd = od; bi = oi; }
        }
        if (lane == 0) pick_s = bi;
      }
      __syncthreads();
      p = pick_s;
    }
    const long long base = k * step;
    for (int j = tid; j < step && base + j < olen; j += kTempoThreads) {
      float y = buf[p + j];
      if (k > 0 && j < overlap) {                               // crossfade, no contraction into FMAs
        const float f = __fmul_rn((float)j, rcp);
        y = __fadd_rn(__fmul_rn((float)pv[j], __fsub_rn(1.f, f)), __fmul_rn(y, f));
      }
      o[base + j] = tempo_quantise16(__fmul_rn(y, g));
    }
    double* nv = prev + (k & 1) * overlap;
    for (int j = tid; j < overlap; j += kTempoThreads) nv[j] = (double)buf[p + step + j];
    if (pk && tid == 0) pk[k] = p;
  }
}

}  // namespace b200asr

using namespace b200asr;

extern "C" {

int b200asr_tempo_gain(const float* in, const long long* in_offsets, const int* in_lengths, const double* tempo,
                       const float* g, float* out, const long long* out_offsets, const int* out_lengths, int* picks,
                       const long long* pick_offsets, int B, int segment, int search, int overlap,
                       b200asr_stream_t stream) {
  B200_REQUIRE(in && in_offsets && in_lengths && tempo && g && out && out_offsets && out_lengths, B200ASR_BAD_ARG,
               "tempo_gain: null pointer");
  B200_REQUIRE((picks == nullptr) == (pick_offsets == nullptr), B200ASR_BAD_ARG,
               "tempo_gain: picks and pick_offsets must be both NULL or both set");
  const auto a4 = [](const void* p) { return ((uintptr_t)p & 3) == 0; };
  const auto a8 = [](const void* p) { return ((uintptr_t)p & 7) == 0; };
  B200_REQUIRE(a4(in) && a4(in_lengths) && a4(g) && a4(out) && a4(out_lengths) && a4(picks) && a8(in_offsets) && a8(tempo) &&
                   a8(out_offsets) && a8(pick_offsets),
               B200ASR_BAD_ALIGN, "tempo_gain: float and int arrays must be 4-byte, int64 and double arrays 8-byte aligned");
  B200_REQUIRE(B > 0, B200ASR_BAD_SHAPE, "tempo_gain: B=%d", B);
  B200_REQUIRE(overlap >= 8 && search >= 1 && 2LL * overlap <= (long long)segment, B200ASR_BAD_SHAPE,
               "tempo_gain: segment=%d, search=%d, overlap=%d (overlap >= 8, 2 * overlap <= segment, search >= 1)", segment,
               search, overlap);
  const long long smem = tempo_smem_bytes(segment, search, overlap);
  B200_REQUIRE(smem <= kTempoMaxSmem, B200ASR_BAD_SHAPE,
               "tempo_gain: segment=%d, search=%d, overlap=%d need %lld bytes of shared memory (at most %lld)", segment,
               search, overlap, smem, kTempoMaxSmem);
  static bool smem_done[kMaxDevices] = {};
  const int rc = ensure_dynamic_smem((const void*)tempo_gain_kernel, (int)kTempoMaxSmem, smem_done, "tempo_gain");
  if (rc != B200ASR_OK) return rc;
  tempo_gain_kernel<<<B, kTempoThreads, (size_t)smem, (cudaStream_t)stream>>>(
      in, in_offsets, in_lengths, tempo, g, out, out_offsets, out_lengths, picks, pick_offsets, segment, search, overlap);
  return check_launch("tempo_gain");
}

}  // extern "C"
