// Feature front end ("next" row 4 of SURVEY.md section 8f): waveform -> normalised log-magnitude spectrogram in the layout
// the training path consumes, i.e. what utils/data_loader.py:60-91 (parse_audio: librosa.stft n_fft = sr*0.02, hop = sr*0.01,
// Hamming window, centred frames; magnitude; log1p; per-utterance mean / unbiased-std normalisation) followed by the
// zero-padded batch tensor of _collate_fn (:182-214) produce on the CPU.
//
// The STFT is a GEMM: frame t of an utterance is the n_fft samples starting at t*hop of its reflect-padded signal, so with
// every padded signal placed at a multiple of `hop` in one buffer ALL frames of the batch are the rows of one matrix with
// row stride hop (rows overlap; TMA only needs a 16-byte-multiple stride), multiplied by the windowed DFT basis
// [2*(n_fft/2+1) x n_fft] (cos rows, then -sin rows).  It runs on the 3xTF32 tensor-core GEMM of the training path (or the
// fp32 CUDA-core GEMM), then two bandwidth-bound kernels do |.|, log1p, the statistics and the transposed, zero-padded
// store.  Rows that straddle two utterances are computed and ignored.
#include <math.h>

#include "../../include/b200asr.h"
#include "common.cuh"
#include "kernels.h"

namespace b200asr {

struct FeatWs {               // carve-up of the caller's workspace (all offsets in floats, 16-byte aligned)
  size_t padded, basis, spec, stats, total;
  int Lp, rows_per_utt, npad;
};

static FeatWs feat_ws(int B, int Lmax, int n_fft, int hop) {
  FeatWs w;
  w.Lp = ceil_div(Lmax + n_fft, hop) * hop;                 // padded signal pitch: a multiple of hop
  w.rows_per_utt = w.Lp / hop;
  w.npad = (2 * (n_fft / 2 + 1) + 3) & ~3;                  // GEMM N: cos + sin rows, padded to a multiple of 4
  auto al = [](size_t x) { return (x + 3) & ~(size_t)3; };
  w.padded = 0;
  w.basis = al((size_t)B * w.Lp + n_fft);                    // + n_fft: the last (ignored) rows still read in bounds
  w.spec = w.basis + al((size_t)w.npad * n_fft);
  w.stats = w.spec + al((size_t)B * w.rows_per_utt * w.npad);
  w.total = w.stats + al((size_t)4 * B);                     // two doubles per utterance
  return w;
}

// centred framing: n_fft/2 samples of padding on both sides; mode 1 = reflect (librosa's default when the reference was
// written), mode 0 = zeros (librosa >= 0.10 default)
__global__ void feat_pad_kernel(const float* __restrict__ wave, const int* __restrict__ lens, float* __restrict__ padded,
                                int B, int Lmax, int Lp, int half, int reflect, size_t total) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int b = (int)(i / Lp), j = (int)(i % Lp);
  float v = 0.f;
  if (b < B) {
    const int len = lens[b];
    int src = j - half;
    if (j < len + 2 * half && len > 0) {
      if (src < 0 || src >= len) {
        if (!reflect) src = -1;
        else if (len == 1) src = 0;
        else {                                    // numpy 'reflect' for any pad width: period 2 (len - 1), no edge repeat
          const int period = 2 * (len - 1);
          int m = src % period;
          if (m < 0) m += period;
          src = m < len ? m : period - m;
        }
      }
      if (src >= 0) v = wave[(size_t)b * Lmax + src];
    }
  }
  padded[i] = v;
}

// basis[r][n]: r < nb: w[n] cos(2 pi r n / N); nb <= r < 2 nb: -w[n] sin(2 pi (r-nb) n / N); zero rows after.
// w = Hamming window over wden points: wden = N - 1 is the SYMMETRIC window -- what the reference computes: it hands the
// callable scipy.signal.hamming to librosa.stft (utils/data_loader.py:20,52,77-78) and librosa.filters.get_window calls a
// callable as window(N), i.e. sym=True --; wden = N is the periodic window of window='hamming' strings.
__global__ void feat_basis_kernel(float* __restrict__ basis, int n_fft, int nb, int npad, int wden) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= npad * n_fft) return;
  const int r = i / n_fft, n = i % n_fft;
  float v = 0.f;
  if (r < 2 * nb) {
    const int k = r < nb ? r : r - nb;
    const int m = (int)(((long long)k * n) % n_fft);                 // exact phase reduction
    float s, c;
    sincospif(2.0f * (float)m / (float)n_fft, &s, &c);
    const float w = 0.54f - 0.46f * cospif(2.0f * (float)n / (float)wden);
    v = r < nb ? w * c : -w * s;
  }
  basis[i] = v;
}

// spec [B*R, npad] (re | im) -> out [B, nb, Tmax] = log1p(|X|) for t < frames[b] (0 beyond), plus per-utterance sum / sum
// of squares in double.  32 x 32 (frame x bin) tiles through shared memory so that both sides are coalesced.
__global__ void feat_mag_kernel(const float* __restrict__ spec, const int* __restrict__ lens, float* __restrict__ out,
                                double* __restrict__ stats, int* __restrict__ frames_out, int R, int npad, int nb, int Tmax,
                                int hop) {
  __shared__ float tile[32][33];
  __shared__ double red[2][8];
  const int b = blockIdx.z, t0 = blockIdx.x * 32, k0 = blockIdx.y * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;            // 256 threads: 32 x 8
  const int nfr = min(1 + lens[b] / hop, Tmax);
  if (blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0 && frames_out) frames_out[b] = nfr;
  double s1 = 0.0, s2 = 0.0;
  for (int i = ty; i < 32; i += 8) {                                  // read: consecutive threads = consecutive bins
    const int t = t0 + i, k = k0 + tx;
    float v = 0.f;
    if (t < nfr && k < nb) {
      const float* row = spec + ((size_t)b * R + t) * npad;
      const float re = row[k], im = row[nb + k];
      v = log1pf(sqrtf(re * re + im * im));
      s1 += v; s2 += (double)v * v;
    }
    tile[i][tx] = v;
  }
  __syncthreads();
  for (int i = ty; i < 32; i += 8) {                                  // write: consecutive threads = consecutive frames
    const int k = k0 + i, t = t0 + tx;
    if (k < nb && t < Tmax) out[((size_t)b * nb + k) * Tmax + t] = tile[tx][i];
  }
  for (int o = 16; o > 0; o >>= 1) { s1 += __shfl_xor_sync(0xffffffffu, s1, o); s2 += __shfl_xor_sync(0xffffffffu, s2, o); }
  if (tx == 0) { red[0][ty] = s1; red[1][ty] = s2; }
  __syncthreads();
  if (threadIdx.x == 0) {
    double a = 0.0, c = 0.0;
    for (int i = 0; i < 8; i++) { a += red[0][i]; c += red[1][i]; }
    atomicAdd(stats + 2 * b, a);
    atomicAdd(stats + 2 * b + 1, c);
  }
}

// spect.add_(-mean); spect.div_(std) with torch's unbiased std (utils/data_loader.py:85-89), valid frames only
__global__ void feat_norm_kernel(float* __restrict__ out, const double* __restrict__ stats, const int* __restrict__ lens,
                                 int nb, int Tmax, int hop) {
  const int b = blockIdx.y;
  const int nfr = min(1 + lens[b] / hop, Tmax);
  const double n = (double)nfr * nb;
  const double mean = stats[2 * b] / n;
  const double var = n > 1.0 ? (stats[2 * b + 1] - n * mean * mean) / (n - 1.0) : 0.0;
  const float m = (float)mean, inv = (float)(1.0 / sqrt(var > 0.0 ? var : 1.0));
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nb * Tmax) return;
  const int t = i % Tmax;
  if (t < nfr) {
    float* p = out + (size_t)b * nb * Tmax + i;
    *p = (*p - m) * inv;
  }
}

}  // namespace b200asr

using namespace b200asr;

extern "C" {

size_t b200asr_stft_ws_bytes(int B, int Lmax, int n_fft, int hop) {
  if (B <= 0 || Lmax <= 0 || n_fft <= 0 || hop <= 0) return 0;
  return feat_ws(B, Lmax, n_fft, hop).total * sizeof(float);
}

int b200asr_stft_features(const float* wave, const int* lens, float* out, int* frames_out, void* ws, int B, int Lmax,
                          int Tmax, int n_fft, int hop, int pad_reflect, int normalize, int window_periodic, int precision,
                          b200asr_stream_t stream) {
  B200_REQUIRE(wave && lens && out && ws, B200ASR_BAD_ARG, "stft_features: null pointer");
  B200_REQUIRE(B > 0 && Lmax > 0 && Tmax > 0, B200ASR_BAD_SHAPE, "stft_features: empty problem");
  B200_REQUIRE(n_fft % 32 == 0 && hop % 4 == 0 && hop > 0 && hop <= n_fft, B200ASR_BAD_SHAPE,
               "stft_features: n_fft=%d must be a multiple of 32 and hop=%d a multiple of 4 (<= n_fft)", n_fft, hop);
  B200_REQUIRE(aligned16(ws) && aligned16(out), B200ASR_BAD_ALIGN, "stft_features: alignment");
  cudaStream_t st = (cudaStream_t)stream;
  const FeatWs w = feat_ws(B, Lmax, n_fft, hop);
  const int nb = n_fft / 2 + 1;
  B200_REQUIRE(Tmax <= w.rows_per_utt, B200ASR_BAD_SHAPE, "stft_features: Tmax=%d exceeds 1 + Lmax/hop", Tmax);
  float* base = (float*)ws;
  float* padded = base + w.padded;
  float* basis = base + w.basis;
  float* spec = base + w.spec;
  double* stats = (double*)(base + w.stats);
  const size_t total = (size_t)B * w.Lp + n_fft;
  feat_pad_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(wave, lens, padded, B, Lmax, w.Lp, n_fft / 2, pad_reflect, total);
  int rc = check_launch("feat_pad");
  if (rc) return rc;
  feat_basis_kernel<<<ceil_div(w.npad * n_fft, 256), 256, 0, st>>>(basis, n_fft, nb, w.npad, window_periodic ? n_fft : n_fft - 1);
  rc = check_launch("feat_basis");
  if (rc) return rc;
  const int M = B * w.rows_per_utt;
  if (precision == B200ASR_PREC_FP32)
    rc = gemm_simt(padded, true, hop, basis, true, n_fft, spec, w.npad, M, w.npad, n_fft, nullptr, 0, nullptr, 0, false, st);
  else if (precision == B200ASR_PREC_TF32 || precision == B200ASR_PREC_TF32X3)
    rc = gemm_tc(padded, true, hop, basis, true, n_fft, spec, w.npad, M, w.npad, n_fft, nullptr, 0, nullptr, 0, precision, st);
  else { set_error("stft_features: unknown precision %d", precision); return B200ASR_BAD_ARG; }
  if (rc) return rc;
  cudaMemsetAsync(stats, 0, sizeof(double) * 2 * (size_t)B, st);
  dim3 grid(ceil_div(Tmax, 32), ceil_div(nb, 32), B);
  feat_mag_kernel<<<grid, 256, 0, st>>>(spec, lens, out, stats, frames_out, w.rows_per_utt, w.npad, nb, Tmax, hop);
  rc = check_launch("feat_mag");
  if (rc) return rc;
  if (normalize) {
    dim3 g2(ceil_div(nb * Tmax, 256), B);
    feat_norm_kernel<<<g2, 256, 0, st>>>(out, stats, lens, nb, Tmax, hop);
    rc = check_launch("feat_norm");
  }
  return rc;
}

}  // extern "C"
