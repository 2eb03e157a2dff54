// Shared device/host helpers for libb200asr (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#define B200ASR_OK 0
#define B200ASR_BAD_SHAPE -1
#define B200ASR_BAD_ALIGN -2
#define B200ASR_UNSUPPORTED_ARCH -3
#define B200ASR_CUDA_ERROR -4
#define B200ASR_BAD_ARG -5

namespace b200asr {

void set_error(const char* fmt, ...);
int check_launch(const char* what);   // cudaGetLastError -> error code (+message); counts one kernel launch
void note_launch(int n);              // additional kernel launches not followed by their own check_launch
int device_sm_count();
// cudaFuncSetAttribute(MaxDynamicSharedMemorySize) once per (kernel, device): function attributes are per device, and the
// reference's nn.DataParallel drives several devices from one process.  `done` is the caller's per-kernel flag array.
constexpr int kMaxDevices = 64;
int ensure_dynamic_smem(const void* kernel, int bytes, bool (&done)[kMaxDevices], const char* what);
int ensure_sm90();                    // B200ASR_OK iff current device is compute capability 9.0

// Fixed-order reductions.  Where many CTAs contribute to the same outputs they write partial results to separate slots and
// reduce_parts() sums the slots in a fixed order: floating-point atomics would make the rounding of every such sum -- and
// so the whole training step -- change from run to run.  stream_scratch() is the library's own device buffer for those
// partials, one per (device, stream), valid for work enqueued on `st`; a larger request reallocates it (cudaFree
// synchronises the device, so that happens during the first steps only).  nullptr (with the error set) on failure.
void* stream_scratch(size_t bytes, cudaStream_t st);
// out[i] = (accumulate ? out[i] : 0) + sum over z = 0 .. parts-1 of part[z * stride + i], for i < n
int reduce_parts(const float* part, int parts, long long stride, long long n, float* out, int accumulate, cudaStream_t st);

#define B200_REQUIRE(cond, code, ...)            \
  do {                                           \
    if (!(cond)) {                               \
      b200asr::set_error(__VA_ARGS__);           \
      return (code);                             \
    }                                            \
  } while (0)

// Programmatic dependent launch.  A kernel launched through launch_pdl() may begin while its predecessor in the stream is
// still draining (the predecessor calls griddep_launch() early; the hardware starts the dependent grid once every CTA of the
// predecessor has done so or exited): its prologue -- barrier init, descriptor prefetch -- and the launch
// latency then overlap the predecessor's tail.  Contract: EVERY kernel launched this way executes griddep_wait() before its
// first global-memory access; griddep_wait() returns when the predecessor grid has completed and its writes are visible, so
// ordering stays transitive along the stream.  Kernels launched the ordinary way are unaffected (both instructions are no-ops
// for them).  B200ASR_PDL=0 turns the attribute off.
bool pdl_enabled();
#ifdef __CUDACC__
__device__ __forceinline__ void griddep_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void griddep_launch() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
template <typename... KArgs, typename... Args>
static inline void launch_pdl(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl_enabled() ? 1 : 0;
  cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);       // errors surface in check_launch()
}
#endif

static inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }
static inline int ceil_div(int a, int b) { return (a + b - 1) / b; }
static inline long long ceil_div_ll(long long a, long long b) { return (a + b - 1) / b; }

// ---------------------------------------------------------------- counter-based dropout RNG
// keep(seed, stream, idx): 16-bit uniform from splitmix64 over (seed, stream, idx/4); four decisions
// per 64-bit draw.  The same (seed, stream, idx) always yields the same decision, so backward kernels
// regenerate the forward mask instead of storing it.
__host__ __device__ __forceinline__ uint64_t splitmix64(uint64_t z) {
  z += 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}
__host__ __device__ __forceinline__ uint64_t dropout_key(uint64_t seed, uint64_t stream) {
  return splitmix64(seed ^ (stream * 0xD1342543DE82EF95ull + 0x2545F4914F6CDD1Dull));
}
// 4 x 16-bit lanes for elements [4*group, 4*group+3]
__host__ __device__ __forceinline__ uint64_t dropout_bits4(uint64_t key, uint64_t group) {
  return splitmix64(key + group * 0x9E3779B97F4A7C15ull);
}
__host__ __device__ __forceinline__ bool dropout_keep(uint64_t key, uint64_t idx, uint32_t thresh16) {
  uint64_t r = dropout_bits4(key, idx >> 2);
  uint32_t bits = (uint32_t)(r >> (16 * (idx & 3))) & 0xFFFFu;
  return bits >= thresh16;
}
static inline uint32_t dropout_thresh16(float p) {
  float t = p * 65536.0f + 0.5f;
  if (t < 0.f) t = 0.f;
  if (t > 65535.f) t = 65535.f;
  return (uint32_t)t;
}
// effective drop probability implied by the 16-bit threshold (used for the 1/(1-p) scale so E[x] is exact)
static inline float dropout_inv_keep(float p) {
  if (p <= 0.f) return 1.f;
  return 1.0f / (1.0f - (float)dropout_thresh16(p) / 65536.0f);
}

// ---------------------------------------------------------------- warp helpers
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

}  // namespace b200asr
