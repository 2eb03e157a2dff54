// SpecAugment (Park et al. 2019) over a batch of spectrograms in _collate_fn's layout: time warp, frequency masks and
// time masks, one launch per batch, draws made on the device from the counter-based generator of dropout (common.cuh).
//
// Block (x, y, b) covers 128 consecutive frames x 16 bins of utterance b.  Its first threads make the utterance's draws
// into shared memory -- one thread per (c, w) pair or per mask, each pair two generator calls, so every block of b computes
// the same integers -- and block (0, 0, b) writes them out.  Each thread then owns one frame: it resolves the time masks
// and the warp's source once, then runs down the 16 bins, so every element is read once (two frames where the warp
// interpolates) and written once: 0 inside a mask or past the utterance's frames, the warped value elsewhere.  The warp's
// source position is an exact rational num / den of integers: the integer part picks the frame, the remainder the weight.
#include <limits.h>
#include <math.h>

#include "../../include/b200asr.h"
#include "common.cuh"

namespace b200asr {

constexpr int kSpecAugMaxMasks = 64;                 // per kind: 2 + 4 * 64 ints of draws per utterance
constexpr int kSpecAugThreads = 128;                 // consecutive frames of one utterance, one per thread
constexpr int kSpecAugRows = 16;                     // frequency bins per block: a block covers 16 x 128 elements

// uniform integer in [lo, hi] (hi >= lo) from draw `slot` of utterance b: the high 32 bits of splitmix64(key + (b << 16 |
// slot) * golden), scaled by the range size with a 64-bit multiply
__device__ __forceinline__ int spec_aug_uniform(uint64_t key, int b, int slot, int lo, int hi) {
  const uint64_t r = dropout_bits4(key, ((uint64_t)b << 16) | (uint64_t)slot);
  return lo + (int)(((r >> 32) * (uint64_t)((long long)hi - lo + 1)) >> 32);
}

__global__ void __launch_bounds__(kSpecAugThreads) spec_augment_kernel(
    const float* __restrict__ in, float* __restrict__ out, int* __restrict__ draws, const int* __restrict__ frames, int F,
    int T, int W, int Fp, int nf, int Tp, float p, int nt, uint64_t key) {
  __shared__ int d[2 + 4 * kSpecAugMaxMasks];
  const int b = blockIdx.z, nd = 2 + 2 * nf + 2 * nt;
  const int Tb = min(max(frames[b], 0), T);
  const bool warps = (long long)Tb > 2LL * W + 1;      // 64-bit: 2W + 1 may pass INT_MAX
  const int tid = threadIdx.x;
  for (int j = tid; j <= nf + nt; j += kSpecAugThreads) {
    if (j == 0) {
      d[0] = warps ? spec_aug_uniform(key, b, 0, W, Tb - W - 1) : 0;
      d[1] = warps ? spec_aug_uniform(key, b, 1, -W, W) : 0;
    } else if (j <= nf) {
      const int s = 2 * j;                            // frequency mask j - 1: slots 2 + 2m, 3 + 2m
      const int fw = spec_aug_uniform(key, b, s, 0, Fp);
      d[s] = fw;
      d[s + 1] = spec_aug_uniform(key, b, s + 1, 0, F - fw);
    } else {
      const int s = 2 * j;                            // time mask j - 1 - nf: slots 2 + 2 nf + 2m, + 1
      const int tw = spec_aug_uniform(key, b, s, 0, min(Tp, (int)floor((double)p * (double)Tb)));
      d[s] = tw;
      d[s + 1] = spec_aug_uniform(key, b, s + 1, 0, Tb - tw);
    }
  }
  __syncthreads();
  if (blockIdx.x == 0 && blockIdx.y == 0)
    for (int j = tid; j < nd; j += kSpecAugThreads) draws[(size_t)b * nd + j] = d[j];
  const int t = blockIdx.x * kSpecAugThreads + tid;
  if (t >= T) return;
  // per frame: masked or padding, else the source frame i0 and the weight of frame i0 + 1 (interp: rem != 0)
  bool tzero = t >= Tb;
  for (int m = 0; m < nt && !tzero; m++) {
    const int s = 2 + 2 * nf + 2 * m;
    tzero = t >= d[s + 1] && t < d[s + 1] + d[s];
  }
  const int c = d[0], dc = d[0] + d[1];               // source frame c lands on frame dc = c + w
  int i0 = t;
  float wt = 0.f;
  bool interp = false;
  if (!tzero && warps && dc != c && t > 0 && t < Tb - 1) {     // frames 0 and T_b - 1 read themselves
    long long num, den;
    int lo;
    if (t <= dc) { num = (long long)t * c; den = dc; lo = 0; }
    else { num = (long long)(t - dc) * (Tb - 1 - c); den = Tb - 1 - dc; lo = c; }
    i0 = lo + (int)(num / den);
    const long long rem = num % den;
    interp = rem != 0;
    wt = (float)rem / (float)den;
  }
  const int f0 = blockIdx.y * kSpecAugRows;
  const size_t plane = (size_t)F * T;
  const float* src = in + (size_t)b * plane + (size_t)f0 * T;
  float* dst = out + (size_t)b * plane + (size_t)f0 * T + t;
#pragma unroll
  for (int r = 0; r < kSpecAugRows; r++) {
    const int f = f0 + r;
    if (f >= F) break;
    bool zero = tzero;
    for (int m = 0; m < nf && !zero; m++) zero = f >= d[3 + 2 * m] && f < d[3 + 2 * m] + d[2 + 2 * m];
    float v = 0.f;
    if (!zero) {
      const float* row = src + (size_t)r * T;
      const float x0 = row[i0];
      v = interp ? fmaf(wt, row[i0 + 1] - x0, x0) : x0;
    }
    dst[(size_t)r * T] = v;
  }
}

}  // namespace b200asr

using namespace b200asr;

extern "C" {

size_t b200asr_spec_augment_draws_ints(int n_freq_masks, int n_time_masks) {
  if (n_freq_masks < 0 || n_freq_masks > kSpecAugMaxMasks || n_time_masks < 0 || n_time_masks > kSpecAugMaxMasks) return 0;
  return 2 + 2 * (size_t)n_freq_masks + 2 * (size_t)n_time_masks;
}

int b200asr_spec_augment(const float* in, float* out, int* draws, const int* frames, int B, int F, int T, int W, int Fp,
                         int n_freq_masks, int Tp, float p, int n_time_masks, unsigned long long seed,
                         unsigned long long counter, b200asr_stream_t stream) {
  B200_REQUIRE(in && out && draws && frames, B200ASR_BAD_ARG, "spec_augment: null pointer");
  B200_REQUIRE(((uintptr_t)in & 3) == 0 && ((uintptr_t)out & 3) == 0 && ((uintptr_t)draws & 3) == 0 &&
                   ((uintptr_t)frames & 3) == 0,
               B200ASR_BAD_ALIGN, "spec_augment: in, out, draws and frames must be 4-byte aligned");
  B200_REQUIRE(B > 0 && F > 0 && T > 0, B200ASR_BAD_SHAPE, "spec_augment: B=%d F=%d T=%d", B, F, T);
  B200_REQUIRE(B <= 65535, B200ASR_BAD_SHAPE, "spec_augment: B=%d exceeds 65535", B);
  const size_t plane = (size_t)F * T, n = (size_t)B * plane;
  B200_REQUIRE(plane <= INT_MAX && ceil_div(F, kSpecAugRows) <= 65535, B200ASR_BAD_SHAPE,
               "spec_augment: F=%d, T=%d (F * T <= 2^31 - 1, F <= %d)", F, T, 65535 * kSpecAugRows);
  B200_REQUIRE(W >= 0 && Fp >= 0 && Fp <= F && Tp >= 0, B200ASR_BAD_ARG,
               "spec_augment: W=%d, Fp=%d (0 .. F=%d) and Tp=%d must not be negative", W, Fp, F, Tp);
  B200_REQUIRE(p >= 0.f && p <= 1.f, B200ASR_BAD_ARG, "spec_augment: p=%g outside [0, 1]", (double)p);
  B200_REQUIRE(n_freq_masks >= 0 && n_freq_masks <= kSpecAugMaxMasks && n_time_masks >= 0 && n_time_masks <= kSpecAugMaxMasks,
               B200ASR_BAD_ARG, "spec_augment: mask counts %d, %d (0 .. %d each)", n_freq_masks, n_time_masks, kSpecAugMaxMasks);
  // the warp reads frames other than the one it writes: the output may not overlap the input
  const uintptr_t a = (uintptr_t)in, o = (uintptr_t)out, bytes = (uintptr_t)(n * sizeof(float));
  B200_REQUIRE(a + bytes <= o || o + bytes <= a, B200ASR_BAD_ARG, "spec_augment: out overlaps in");
  const uint64_t key = dropout_key(seed, counter);
  const dim3 grid((unsigned)ceil_div(T, kSpecAugThreads), (unsigned)ceil_div(F, kSpecAugRows), (unsigned)B);
  spec_augment_kernel<<<grid, kSpecAugThreads, 0, (cudaStream_t)stream>>>(
      in, out, draws, frames, F, T, W, Fp, n_freq_masks, Tp, p, n_time_masks, key);
  return check_launch("spec_augment");
}

}  // extern "C"
