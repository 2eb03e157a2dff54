// Polyphase resampling of a packed batch of waveforms (scipy.signal.resample_poly with its defaults, restated in
// include/b200asr.h): one launch per batch, each utterance at its own ratio up / down.
//
// CTA (chunk, utterance) computes `chunk` consecutive outputs of one utterance.  It stages the input window those outputs
// read -- zeros outside the utterance, so the zero padding costs no branch -- in shared memory, then each thread computes
// outputs tid, tid + 256, ... of the chunk: output i sits at c = i * down + half on the upsampled grid, reads phase
// c mod up of the ratio's taps (from the read-only cache; a ratio's taps are a few KB shared by every CTA) against
// x[c / up - m], m = 0, 1, ..., summed with fp32 FMAs in increasing m.  That order does not depend on the chunking or on
// the other utterances of the batch, so the bits repeat and a batch equals each of its utterances run alone.
#include <algorithm>
#include <limits.h>
#include <vector>

#include "../../include/b200asr.h"
#include "common.cuh"

namespace b200asr {

constexpr int kResampleThreads = 256;
constexpr int kResampleChunk = 8 * kResampleThreads;           // outputs per CTA, at most
constexpr int kResampleWindow = 24576;                          // input floats staged per CTA, at most (96 KB)
constexpr int kResampleMaxRate = 1000;
constexpr int kResampleMaxGridY = 65535;

struct ResampleGeom {
  long long half, K, chunk, window;                             // half length, taps per phase, outputs and inputs per CTA
};

// The geometry of a reduced ratio; up == down == 1 is a copy (half 0, one "tap").
__host__ __device__ __forceinline__ ResampleGeom resample_geom(int up, int down) {
  ResampleGeom g;
  const bool copy = up == 1 && down == 1;
  g.half = copy ? 0 : 10LL * (up > down ? up : down);
  g.K = (2 * g.half + up) / up;                                 // ceil((2 half + 1) / up)
  const long long fit = (kResampleWindow - g.K) * up / down + 1;
  g.chunk = fit < kResampleChunk ? fit : kResampleChunk;
  g.window = ((g.chunk - 1) * down + up - 1) / up + g.K;       // >= the inputs any chunk reads
  return g;
}

__host__ __device__ __forceinline__ long long resample_out_length(long long n, int up, int down) {
  return (n * up + down - 1) / down;
}

// clamp(rint(v * 32768), -32768, 32767) / 32768, half to even; NaN stays NaN
__device__ __forceinline__ float resample_quantise16(float v) {
  float q = rintf(__fmul_rn(v, 32768.f));
  q = q < -32768.f ? -32768.f : (q > 32767.f ? 32767.f : q);
  return __fmul_rn(q, 1.f / 32768.f);
}

__global__ void __launch_bounds__(kResampleThreads) resample_kernel(const float* __restrict__ in, float* __restrict__ out,
                                                                    const b200asr_resample_item* __restrict__ items, int B,
                                                                    int quantize16) {
  extern __shared__ float xs[];
  for (int b = blockIdx.y; b < B; b += gridDim.y) {
    const b200asr_resample_item it = items[b];
    const ResampleGeom g = resample_geom(it.up, it.down);
    const long long n = it.in_length, n_out = resample_out_length(n, it.up, it.down);
    const long long i0 = (long long)blockIdx.x * g.chunk;
    if (i0 >= n_out) continue;                                   // uniform per CTA
    const int cnt = (int)(n_out - i0 < g.chunk ? n_out - i0 : g.chunk);
    const long long jlo = (i0 * it.down + g.half) / it.up - (g.K - 1);
    const long long jhi = ((i0 + cnt - 1) * it.down + g.half) / it.up;
    const int W = (int)(jhi - jlo + 1);
    const float* x = in + it.in_offset;
    __syncthreads();                                             // the previous utterance is done with xs
    for (int t = threadIdx.x; t < W; t += kResampleThreads) {
      const long long j = jlo + t;
      xs[t] = (j >= 0 && j < n) ? __ldg(x + j) : 0.f;
    }
    __syncthreads();
    float* o = out + it.out_offset;
    for (int r = threadIdx.x; r < cnt; r += kResampleThreads) {
      const long long i = i0 + r, c = i * it.down + g.half, j0 = c / it.up;
      const int ph = (int)(c - j0 * it.up);
      const float* xp = xs + (j0 - jlo);
      float s;
      if (g.half == 0) {
        s = xp[0];
      } else {
        const float* h = it.taps + (long long)ph * g.K;
        const int kp = (int)((2 * g.half - ph) / it.up) + 1;     // taps of this phase: ph + m * up <= 2 half
        s = 0.f;
        for (int m = 0; m < kp; m++) s = __fmaf_rn(__ldg(h + m), xp[-m], s);
      }
      o[i] = quantize16 ? resample_quantise16(s) : s;
    }
  }
}

static long long gcd_ll(long long a, long long b) {
  while (b) {
    const long long t = a % b;
    a = b;
    b = t;
  }
  return a;
}

}  // namespace b200asr

using namespace b200asr;

extern "C" {

int b200asr_resample_packed(const float* in, long long in_size, float* out, long long out_size,
                            const b200asr_resample_item* items, const b200asr_resample_item* items_dev, int B,
                            int quantize16, b200asr_stream_t stream) {
  B200_REQUIRE(in && out && items && items_dev, B200ASR_BAD_ARG, "resample_packed: null pointer");
  B200_REQUIRE(((uintptr_t)in & 3) == 0 && ((uintptr_t)out & 3) == 0 && ((uintptr_t)items_dev & 7) == 0, B200ASR_BAD_ALIGN,
               "resample_packed: in and out must be 4-byte, items_dev 8-byte aligned");
  B200_REQUIRE(B > 0 && in_size >= 0 && out_size >= 0, B200ASR_BAD_SHAPE, "resample_packed: B=%d, in_size=%lld, out_size=%lld",
               B, in_size, out_size);
  B200_REQUIRE(quantize16 == 0 || quantize16 == 1, B200ASR_BAD_ARG, "resample_packed: quantize16=%d", quantize16);
  const uintptr_t ib = (uintptr_t)in, ie = ib + 4 * (uintptr_t)in_size, ob = (uintptr_t)out, oe = ob + 4 * (uintptr_t)out_size;
  B200_REQUIRE(oe <= ib || ie <= ob, B200ASR_BAD_ARG, "resample_packed: out overlaps in");
  std::vector<std::pair<long long, long long>> spans;           // (first, end) of every non-empty output
  long long chunks = 0, smem = 0;
  for (int b = 0; b < B; b++) {
    const b200asr_resample_item& it = items[b];
    B200_REQUIRE(it.up >= 1 && it.down >= 1 && it.up <= kResampleMaxRate && it.down <= kResampleMaxRate &&
                     gcd_ll(it.up, it.down) == 1,
                 B200ASR_BAD_SHAPE, "resample_packed: utterance %d has up=%d, down=%d (coprime, each in [1, %d])", b, it.up,
                 it.down, kResampleMaxRate);
    const bool copy = it.up == 1 && it.down == 1;
    B200_REQUIRE(copy || (it.taps && ((uintptr_t)it.taps & 3) == 0), B200ASR_BAD_ARG,
                 "resample_packed: utterance %d needs 4-byte aligned taps", b);
    B200_REQUIRE(it.in_offset >= 0 && it.in_length >= 0 && it.in_offset <= in_size - it.in_length, B200ASR_BAD_SHAPE,
                 "resample_packed: utterance %d reads [%lld, %lld + %d) of %lld input samples", b, it.in_offset,
                 it.in_offset, it.in_length, in_size);
    const long long n_out = resample_out_length(it.in_length, it.up, it.down);
    B200_REQUIRE(it.out_offset >= 0 && it.out_offset <= out_size - n_out, B200ASR_BAD_SHAPE,
                 "resample_packed: utterance %d writes [%lld, %lld + %lld) of %lld output samples", b, it.out_offset,
                 it.out_offset, n_out, out_size);
    if (n_out == 0) continue;
    spans.emplace_back(it.out_offset, it.out_offset + n_out);
    const ResampleGeom g = resample_geom(it.up, it.down);
    chunks = std::max(chunks, (n_out + g.chunk - 1) / g.chunk);
    smem = std::max(smem, g.window * (long long)sizeof(float));
  }
  std::sort(spans.begin(), spans.end());
  for (size_t k = 1; k < spans.size(); k++)
    B200_REQUIRE(spans[k - 1].second <= spans[k].first, B200ASR_BAD_SHAPE,
                 "resample_packed: outputs [%lld, %lld) and [%lld, %lld) overlap", spans[k - 1].first, spans[k - 1].second,
                 spans[k].first, spans[k].second);
  B200_REQUIRE(chunks <= INT_MAX, B200ASR_BAD_SHAPE, "resample_packed: %lld chunks of outputs", chunks);
  if (chunks == 0) return B200ASR_OK;                           // nothing to write
  static bool smem_done[kMaxDevices] = {};
  const int rc = ensure_dynamic_smem((const void*)resample_kernel, kResampleWindow * (int)sizeof(float), smem_done,
                                     "resample_packed");
  if (rc != B200ASR_OK) return rc;
  const dim3 grid((unsigned)chunks, (unsigned)std::min(B, kResampleMaxGridY));
  resample_kernel<<<grid, kResampleThreads, (size_t)smem, (cudaStream_t)stream>>>(in, out, items_dev, B, quantize16);
  return check_launch("resample_packed");
}

}  // extern "C"
