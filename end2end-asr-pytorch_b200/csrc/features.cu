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
#include <limits.h>
#include <math.h>

#include "../../include/b200asr.h"
#include "common.cuh"
#include "kernels.h"

namespace b200asr {

struct FeatWs {               // carve-up of the caller's workspace (all offsets in floats, 16-byte aligned)
  size_t padded, basis, spec, stats, parts, total;
  int Lp, rows_per_utt, npad, max_tiles;
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
  w.parts = w.stats + al((size_t)4 * B);                     // two doubles per utterance
  w.max_tiles = ceil_div(w.rows_per_utt, 32) * ceil_div(n_fft / 2 + 1, 32);   // feat_mag tiles per utterance at Tmax's bound
  w.total = w.parts + al((size_t)4 * B * w.max_tiles);       // two doubles per tile
  return w;
}

// centred framing: n_fft/2 samples of padding on both sides; mode 1 = reflect (librosa's default when the reference was
// written), mode 0 = zeros (librosa >= 0.10 default).  With kNoise, the sample at source index s of a noisy utterance
// (nstart[b] >= 0) is the reference's NoiseInjection mix (utils/data_loader.py:176-178), in numpy's fp32 order:
//   x[s] + ((level * n[s]) * e_x) / e_n,   n = bank[nstart[b] : nstart[b] + len],   e = sqrt(sum of squares / len)
// with the sums of squares from feat_energy_kernel + feat_stats_kernel.  A silent segment gives 0/0 = NaN, a silent
// utterance x + 0, as numpy does.  A segment that leaves the bank makes the whole utterance NaN instead of being read.
// Utterance b starts at wave + utt_base(b): offsets[b] in a packed batch, b * Lmax in a [B, Lmax] one (offsets NULL); a
// negative offset makes the utterance NaN instead of being read.
__device__ __forceinline__ long long utt_base(const long long* __restrict__ offsets, int b, int Lmax) {
  return offsets ? offsets[b] : (long long)b * Lmax;
}

template <bool kNoise>
__global__ void feat_pad_kernel(const float* __restrict__ wave, const long long* __restrict__ offsets,
                                const int* __restrict__ lens, float* __restrict__ padded, int B, int Lmax, int Lp, int half,
                                int reflect, size_t total, const float* __restrict__ bank, long long bank_len,
                                const long long* __restrict__ nstart, const float* __restrict__ nlevel,
                                const double* __restrict__ estats) {
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
      const long long base = utt_base(offsets, b, Lmax);
      if (base < 0) src = -1, v = __int_as_float(0x7fc00000);
      if (src >= 0) v = wave[base + src];
      if (kNoise && src >= 0) {
        const long long st = nstart[b];
        if (st >= 0) {
          if (st > bank_len - len) v = __int_as_float(0x7fc00000);
          else {
            const float ex = (float)sqrt(estats[2 * b] / len), en = (float)sqrt(estats[2 * b + 1] / len);
            v = v + ((nlevel[b] * bank[st + src]) * ex) / en;
          }
        }
      }
    }
  }
  padded[i] = v;
}

// Sums of squares of a noisy utterance and of its noise segment, in double: block (c, b) takes samples [c, c + 1) *
// kEnergyChunk of utterance b, thread i every 256th of them from i on, then a fixed tree; its pair goes to its own slot
// parts[b][c][2] for feat_stats_kernel to add up in chunk order (no atomics: the same bits every call).
constexpr int kEnergyChunk = 4096;

__global__ void feat_energy_kernel(const float* __restrict__ wave, const long long* __restrict__ offsets,
                                   const int* __restrict__ lens, const float* __restrict__ bank, long long bank_len,
                                   const long long* __restrict__ nstart, double* __restrict__ parts, int Lmax) {
  __shared__ double red[2][8];
  const int b = blockIdx.y, c = blockIdx.x;
  const int len = lens[b];
  const long long st = nstart[b], base = utt_base(offsets, b, Lmax);
  double sx = 0.0, sn = 0.0;
  if (st >= 0 && st <= bank_len - len && base >= 0) {
    const int hi = min(len, (c + 1) * kEnergyChunk);
    for (int i = c * kEnergyChunk + (int)threadIdx.x; i < hi; i += 256) {
      const double x = wave[base + i], n = bank[st + i];
      sx += x * x;
      sn += n * n;
    }
  }
  for (int o = 16; o > 0; o >>= 1) { sx += __shfl_xor_sync(0xffffffffu, sx, o); sn += __shfl_xor_sync(0xffffffffu, sn, o); }
  if ((threadIdx.x & 31) == 0) { red[0][threadIdx.x >> 5] = sx; red[1][threadIdx.x >> 5] = sn; }
  __syncthreads();
  if (threadIdx.x == 0) {
    double a = 0.0, e = 0.0;
    for (int w = 0; w < 8; w++) { a += red[0][w]; e += red[1][w]; }
    double* o = parts + ((size_t)b * gridDim.x + c) * 2;
    o[0] = a;
    o[1] = e;
  }
}

// basis[r][n]: r < nb: w[n] cos(2 pi r n / N); nb <= r < 2 nb: -w[n] sin(2 pi (r-nb) n / N); zero rows after.
// w = scipy's window over wden points: wden = N - 1 is the SYMMETRIC window -- what the reference computes: it hands the
// callable scipy.signal.<window> to librosa.stft (utils/data_loader.py:20,52,77-78) and librosa.filters.get_window calls a
// callable as window(N), i.e. sym=True --; wden = N is the periodic window of window='hamming' strings.
// window: 0 Hamming 0.54 - 0.46 cos(2 pi n / wden), 1 Hann 0.5 - 0.5 cos(.), 2 Blackman 0.42 - 0.5 cos(.) + 0.08 cos(2 .),
// 3 Bartlett 1 - |2 n / wden - 1| (zero end points when symmetric).
__global__ void feat_basis_kernel(float* __restrict__ basis, int n_fft, int nb, int npad, int wden, int window) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= npad * n_fft) return;
  const int r = i / n_fft, n = i % n_fft;
  float v = 0.f;
  if (r < 2 * nb) {
    const int k = r < nb ? r : r - nb;
    const int m = (int)(((long long)k * n) % n_fft);                 // exact phase reduction
    float s, c;
    sincospif(2.0f * (float)m / (float)n_fft, &s, &c);
    const float x = 2.0f * (float)n / (float)wden;
    float w;
    switch (window) {
      case 1: w = 0.5f - 0.5f * cospif(x); break;
      case 2: w = 0.42f - 0.5f * cospif(x) + 0.08f * cospif(2.0f * x); break;
      case 3: w = 1.0f - fabsf(x - 1.0f); break;
      default: w = 0.54f - 0.46f * cospif(2.0f * (float)n / (float)wden);
    }
    v = r < nb ? w * c : -w * s;
  }
  basis[i] = v;
}

// spec [B*R, npad] (re | im) -> out [B, nb, Tmax] = log1p(|X|) for t < keep = min(frames[b], keep_cap) (0 beyond), plus
// the tile's sum / sum of squares over t < min(frames[b], stat_cap) in double, written to its own slot parts[b][tile][2]
// (feat_stats_kernel adds them up in tile order, so the normalisation does not depend on the order in which tiles finish).
// Tiles x < gx_main (the ones that store) take slots y * gx_main + x; tiles past them only add statistics and take the
// slots after those.  32 x 32 (frame x bin) tiles through shared memory so that both sides are coalesced.
__global__ void feat_mag_kernel(const float* __restrict__ spec, const int* __restrict__ lens, float* __restrict__ out,
                                double* __restrict__ parts, int* __restrict__ frames_out, int R, int npad, int nb, int Tmax,
                                int hop, int stat_cap, int keep_cap, int gx_main) {
  __shared__ float tile[32][33];
  __shared__ double red[2][8];
  const int b = blockIdx.z, t0 = blockIdx.x * 32, k0 = blockIdx.y * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;            // 256 threads: 32 x 8
  const int nfr = 1 + lens[b] / hop, nst = min(nfr, stat_cap), nkeep = min(nfr, keep_cap);
  if (blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0 && frames_out) frames_out[b] = nkeep;
  double s1 = 0.0, s2 = 0.0;
  for (int i = ty; i < 32; i += 8) {                                  // read: consecutive threads = consecutive bins
    const int t = t0 + i, k = k0 + tx;
    float v = 0.f;
    if (t < nst && k < nb) {
      const float* row = spec + ((size_t)b * R + t) * npad;
      const float re = row[k], im = row[nb + k];
      v = log1pf(sqrtf(re * re + im * im));
      s1 += v; s2 += (double)v * v;
    }
    tile[i][tx] = t < nkeep ? v : 0.f;
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
    const int gy = gridDim.y, x = blockIdx.x, y = blockIdx.y;
    const size_t slot = x < gx_main ? (size_t)y * gx_main + x : (size_t)gx_main * gy + (size_t)y * (gridDim.x - gx_main) + (x - gx_main);
    double* o = parts + ((size_t)b * gridDim.x * gy + slot) * 2;
    o[0] = a;
    o[1] = c;
  }
}

// stats[b] = (sum, sum of squares) of utterance b: one warp per utterance, lane l takes slots l, l + 32, ... of the first
// `nmain` in order, then a fixed shuffle tree -- the same bits every run; slots nmain .. tiles - 1 are summed the same way
// and added last (a batch whose extra slots are all zero gets the bits of the first `nmain` alone)
__global__ void feat_stats_kernel(const double* __restrict__ parts, double* __restrict__ stats, int nmain, int tiles) {
  const int b = blockIdx.x, lane = threadIdx.x;
  const double* p = parts + (size_t)b * tiles * 2;
  double a = 0.0, c = 0.0;
  for (int i = lane; i < nmain; i += 32) { a += p[2 * i]; c += p[2 * i + 1]; }
  for (int o = 16; o > 0; o >>= 1) { a += __shfl_xor_sync(0xffffffffu, a, o); c += __shfl_xor_sync(0xffffffffu, c, o); }
  if (nmain < tiles) {
    double a2 = 0.0, c2 = 0.0;
    for (int i = nmain + lane; i < tiles; i += 32) { a2 += p[2 * i]; c2 += p[2 * i + 1]; }
    for (int o = 16; o > 0; o >>= 1) { a2 += __shfl_xor_sync(0xffffffffu, a2, o); c2 += __shfl_xor_sync(0xffffffffu, c2, o); }
    a += a2;
    c += c2;
  }
  if (lane == 0) { stats[2 * b] = a; stats[2 * b + 1] = c; }
}

// spect.add_(-mean); spect.div_(std) with torch's unbiased std (utils/data_loader.py:85-89) over the min(frames, stat_cap)
// frames the statistics cover, applied to the min(frames, keep_cap) frames stored
__global__ void feat_norm_kernel(float* __restrict__ out, const double* __restrict__ stats, const int* __restrict__ lens,
                                 int nb, int Tmax, int hop, int stat_cap, int keep_cap) {
  const int b = blockIdx.y;
  const int nfr = min(1 + lens[b] / hop, stat_cap), nkeep = min(1 + lens[b] / hop, keep_cap);
  const double n = (double)nfr * nb;
  const double mean = stats[2 * b] / n;
  const double var = n > 1.0 ? (stats[2 * b + 1] - n * mean * mean) / (n - 1.0) : 0.0;
  const float m = (float)mean, inv = (float)(1.0 / sqrt(var > 0.0 ? var : 1.0));
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nb * Tmax) return;
  const int t = i % Tmax;
  if (t < nkeep) {
    float* p = out + (size_t)b * nb * Tmax + i;
    *p = (*p - m) * inv;
  }
}

struct FeatNoise {             // NoiseInjection's inputs: bank [bank_len] fp32, per utterance a start (< 0: none) and level
  const float* bank;
  long long bank_len;
  const long long* start;
  const float* level;
};

static size_t feat_energy_chunks(int Lmax) { return (size_t)ceil_div(Lmax, kEnergyChunk); }

// the checks both entry points share; the caller has checked its own arguments first
static int feat_check(const float* wave, const int* lens, const float* out, const void* ws, int B, int Lmax, int Tmax, int n_fft,
                      int hop, int precision) {
  B200_REQUIRE(wave && lens && out && ws, B200ASR_BAD_ARG, "stft_features: null pointer");
  B200_REQUIRE(B > 0 && Lmax > 0 && Tmax > 0, B200ASR_BAD_SHAPE, "stft_features: empty problem");
  B200_REQUIRE(n_fft % 32 == 0 && hop % 4 == 0 && hop > 0 && hop <= n_fft, B200ASR_BAD_SHAPE,
               "stft_features: n_fft=%d must be a multiple of 32 and hop=%d a multiple of 4 (<= n_fft)", n_fft, hop);
  B200_REQUIRE(aligned16(ws) && aligned16(out), B200ASR_BAD_ALIGN, "stft_features: alignment");
  B200_REQUIRE(precision == B200ASR_PREC_FP32 || precision == B200ASR_PREC_TF32 || precision == B200ASR_PREC_TF32X3,
               B200ASR_BAD_ARG, "stft_features: precision %d (0, 1 or 3: the DFT basis is an fp32 operand)", precision);
  // the longest utterance that fits in Lmax samples has 1 + Lmax/hop frames
  B200_REQUIRE(Tmax <= 1 + Lmax / hop, B200ASR_BAD_SHAPE, "stft_features: Tmax=%d exceeds 1 + Lmax/hop = %d", Tmax, 1 + Lmax / hop);
  return B200ASR_OK;
}

// Enqueues the front end on checked arguments.  Statistics cover min(frames, stat_cap) frames of each utterance, with
// gx_stat >= ceil(Tmax / 32) frame tiles; min(frames, keep_cap) frames are stored.
static int feat_run(const float* wave, const long long* offsets, const int* lens, float* out, int* frames_out, void* ws, int B, int Lmax, int Tmax,
                    int n_fft, int hop, int pad_reflect, int normalize, int window, int window_periodic, const FeatNoise* noise,
                    int stat_cap, int keep_cap, int gx_stat, int precision, cudaStream_t st) {
  const FeatWs w = feat_ws(B, Lmax, n_fft, hop);
  const int nb = n_fft / 2 + 1;
  float* base = (float*)ws;
  float* padded = base + w.padded;
  float* basis = base + w.basis;
  float* spec = base + w.spec;
  double* stats = (double*)(base + w.stats);
  double* parts = (double*)(base + w.parts);
  const size_t total = (size_t)B * w.Lp + n_fft;
  const unsigned pad_blocks = (unsigned)((total + 255) / 256);
  int rc;
  if (noise) {
    // energies: partials in the workspace past the front end's own part, then (sum x^2, sum n^2) per utterance
    double* eparts = (double*)(base + w.total);
    double* estats = eparts + 2 * (size_t)B * feat_energy_chunks(Lmax);
    feat_energy_kernel<<<dim3((unsigned)feat_energy_chunks(Lmax), B), 256, 0, st>>>(wave, offsets, lens, noise->bank,
                                                                                   noise->bank_len, noise->start, eparts, Lmax);
    rc = check_launch("feat_energy");
    if (rc) return rc;
    feat_stats_kernel<<<B, 32, 0, st>>>(eparts, estats, (int)feat_energy_chunks(Lmax), (int)feat_energy_chunks(Lmax));
    rc = check_launch("feat_energy_stats");
    if (rc) return rc;
    feat_pad_kernel<true><<<pad_blocks, 256, 0, st>>>(wave, offsets, lens, padded, B, Lmax, w.Lp, n_fft / 2, pad_reflect, total,
                                                       noise->bank, noise->bank_len, noise->start, noise->level, estats);
  } else {
    feat_pad_kernel<false><<<pad_blocks, 256, 0, st>>>(wave, offsets, lens, padded, B, Lmax, w.Lp, n_fft / 2, pad_reflect, total,
                                                        nullptr, 0, nullptr, nullptr, nullptr);
  }
  rc = check_launch("feat_pad");
  if (rc) return rc;
  feat_basis_kernel<<<ceil_div(w.npad * n_fft, 256), 256, 0, st>>>(basis, n_fft, nb, w.npad, window_periodic ? n_fft : n_fft - 1,
                                                                   window);
  rc = check_launch("feat_basis");
  if (rc) return rc;
  const int M = B * w.rows_per_utt;
  if (precision == B200ASR_PREC_FP32)
    rc = gemm_simt(padded, true, hop, basis, true, n_fft, spec, w.npad, M, w.npad, n_fft, nullptr, 0, nullptr, 0, false, st);
  else
    rc = gemm_tc(padded, true, hop, basis, true, n_fft, spec, w.npad, M, w.npad, n_fft, nullptr, 0, nullptr, 0, precision, st);
  if (rc) return rc;
  const int gx_main = ceil_div(Tmax, 32);
  dim3 grid(gx_stat, ceil_div(nb, 32), B);
  feat_mag_kernel<<<grid, 256, 0, st>>>(spec, lens, out, parts, frames_out, w.rows_per_utt, w.npad, nb, Tmax, hop, stat_cap,
                                        keep_cap, gx_main);
  rc = check_launch("feat_mag");
  if (rc) return rc;
  if (normalize) {
    feat_stats_kernel<<<B, 32, 0, st>>>(parts, stats, (int)(gx_main * grid.y), (int)(grid.x * grid.y));
    rc = check_launch("feat_stats");
    if (rc) return rc;
    dim3 g2(ceil_div(nb * Tmax, 256), B);
    feat_norm_kernel<<<g2, 256, 0, st>>>(out, stats, lens, nb, Tmax, hop, stat_cap, keep_cap);
    rc = check_launch("feat_norm");
  }
  return rc;
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
  const int rc = feat_check(wave, lens, out, ws, B, Lmax, Tmax, n_fft, hop, precision);
  if (rc) return rc;
  return feat_run(wave, nullptr, lens, out, frames_out, ws, B, Lmax, Tmax, n_fft, hop, pad_reflect, normalize, 0, window_periodic, nullptr,
                  Tmax, Tmax, ceil_div(Tmax, 32), precision, (cudaStream_t)stream);
}

size_t b200asr_stft_features_ex_ws_bytes(int B, int Lmax, int n_fft, int hop) {
  if (B <= 0 || Lmax <= 0 || n_fft <= 0 || hop <= 0) return 0;
  // + the energy partials (two doubles per utterance and chunk) and sums (two doubles per utterance)
  return (feat_ws(B, Lmax, n_fft, hop).total + 4 * (size_t)B * (feat_energy_chunks(Lmax) + 1)) * sizeof(float);
}

}  // extern "C"

// b200asr_stft_features_ex (offsets NULL: utterance b at wave + b * Lmax) and b200asr_stft_features_packed (at
// wave + offsets[b]): one path
static int feat_ex(const char* what, const float* wave, const long long* offsets, const int* lens, float* out, int* frames_out,
                   void* ws, int B, int Lmax, int Tmax, int n_fft, int hop, int pad_reflect, int normalize, int window,
                   int window_periodic, const float* noise_bank, long long noise_bank_len, const long long* noise_start,
                   const float* noise_level, int max_frames, int precision, cudaStream_t stream) {
  B200_REQUIRE(window >= 0 && window <= 3, B200ASR_BAD_ARG, "%s: window %d (0 Hamming, 1 Hann, 2 Blackman, 3 Bartlett)", what,
               window);
  B200_REQUIRE((noise_bank == nullptr) == (noise_start == nullptr) && (noise_bank == nullptr) == (noise_level == nullptr),
               B200ASR_BAD_ARG, "%s: noise_bank, noise_start and noise_level go together", what);
  B200_REQUIRE(noise_bank == nullptr || noise_bank_len > 0, B200ASR_BAD_SHAPE, "%s: noise_bank_len=%lld", what, noise_bank_len);
  B200_REQUIRE(max_frames > 0, B200ASR_BAD_SHAPE, "%s: max_frames=%d", what, max_frames);
  const int rc = feat_check(wave, lens, out, ws, B, Lmax, Tmax, n_fft, hop, precision);
  if (rc) return rc;
  const FeatNoise noise = {noise_bank, noise_bank_len, noise_start, noise_level};
  // statistics over every frame an utterance of at most Lmax samples can have, whatever is stored
  return feat_run(wave, offsets, lens, out, frames_out, ws, B, Lmax, Tmax, n_fft, hop, pad_reflect, normalize, window,
                  window_periodic, noise_bank ? &noise : nullptr, INT_MAX, min(max_frames, Tmax), ceil_div(1 + Lmax / hop, 32),
                  precision, stream);
}

extern "C" {

int b200asr_stft_features_ex(const float* wave, const int* lens, float* out, int* frames_out, void* ws, int B, int Lmax,
                             int Tmax, int n_fft, int hop, int pad_reflect, int normalize, int window, int window_periodic,
                             const float* noise_bank, long long noise_bank_len, const long long* noise_start,
                             const float* noise_level, int max_frames, int precision, b200asr_stream_t stream) {
  return feat_ex("stft_features_ex", wave, nullptr, lens, out, frames_out, ws, B, Lmax, Tmax, n_fft, hop, pad_reflect, normalize, window,
                 window_periodic, noise_bank, noise_bank_len, noise_start, noise_level, max_frames, precision,
                 (cudaStream_t)stream);
}

int b200asr_stft_features_packed(const float* wave, const long long* offsets, const int* lens, float* out, int* frames_out,
                                 void* ws, int B, int Lmax, int Tmax, int n_fft, int hop, int pad_reflect, int normalize,
                                 int window, int window_periodic, const float* noise_bank, long long noise_bank_len,
                                 const long long* noise_start, const float* noise_level, int max_frames, int precision,
                                 b200asr_stream_t stream) {
  B200_REQUIRE(offsets, B200ASR_BAD_ARG, "stft_features_packed: null offsets");
  B200_REQUIRE(((uintptr_t)offsets & 7) == 0 && ((uintptr_t)wave & 3) == 0, B200ASR_BAD_ALIGN,
               "stft_features_packed: offsets must be 8-byte and wave 4-byte aligned");
  return feat_ex("stft_features_packed", wave, offsets, lens, out, frames_out, ws, B, Lmax, Tmax, n_fft, hop, pad_reflect, normalize, window,
                 window_periodic, noise_bank, noise_bank_len, noise_start, noise_level, max_frames, precision,
                 (cudaStream_t)stream);
}

}  // extern "C"
