#include <stdlib.h>
// Error plumbing, device checks, version, scratch and fixed-order reductions.
#include <stdarg.h>

#include <map>
#include <mutex>
#include <utility>

#include "../../include/b200asr.h"
#include "common.cuh"

namespace b200asr {

static thread_local char g_err[512] = "";

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

static unsigned long long g_launches = 0;   // kernels launched by this library (process-wide, approximate under threads)
void note_launch(int n) { g_launches += (unsigned long long)n; }

int check_launch(const char* what) {
  g_launches += 1;
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_error("%s: CUDA error %d (%s)", what, (int)e, cudaGetErrorString(e));
    return B200ASR_CUDA_ERROR;
  }
  return B200ASR_OK;
}

int ensure_dynamic_smem(const void* kernel, int bytes, bool (&done)[kMaxDevices], const char* what) {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= kMaxDevices) { set_error("%s: cannot query the current device", what); return B200ASR_CUDA_ERROR; }
  if (done[dev]) return B200ASR_OK;
  cudaError_t r = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
  if (r != cudaSuccess) { set_error("%s: cannot reserve %d bytes of shared memory: %s", what, bytes, cudaGetErrorString(r)); return B200ASR_CUDA_ERROR; }
  done[dev] = true;
  return B200ASR_OK;
}

bool pdl_enabled() {
  static const bool on = [] { const char* e = getenv("B200ASR_PDL"); return !(e && e[0] == '0'); }();
  return on;
}

int device_sm_count() {
  static thread_local int cached_dev = -1, cached = 0;
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return 132;
  if (dev != cached_dev) {
    cudaDeviceProp p;
    if (cudaGetDeviceProperties(&p, dev) != cudaSuccess) return 132;
    cached = p.multiProcessorCount;
    cached_dev = dev;
  }
  return cached;
}

int ensure_sm90() {
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) {
    set_error("no CUDA device: %s", cudaGetErrorString(e));
    return B200ASR_UNSUPPORTED_ARCH;
  }
  int major = 0, minor = 0;
  cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev);
  cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev);
  if (major != 9 || minor != 0) {
    set_error("libb200asr is built for sm_90a (H100) only; device %d is sm_%d%d", dev, major, minor);
    return B200ASR_UNSUPPORTED_ARCH;
  }
  return B200ASR_OK;
}

void* stream_scratch(size_t bytes, cudaStream_t st) {
  static std::mutex mu;
  static std::map<std::pair<int, cudaStream_t>, std::pair<void*, size_t>> pools;
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) { set_error("stream_scratch: cannot query the current device"); return nullptr; }
  std::lock_guard<std::mutex> lock(mu);
  auto& slot = pools[std::make_pair(dev, st)];
  if (slot.second < bytes) {
    if (slot.first) cudaFree(slot.first);
    slot.first = nullptr;
    slot.second = 0;
    const size_t want = (bytes + (1u << 20) - 1) & ~(size_t)((1u << 20) - 1);
    if (cudaMalloc(&slot.first, want) != cudaSuccess) {
      cudaGetLastError();
      slot.first = nullptr;
      set_error("stream_scratch: cannot allocate %zu bytes", want);
      return nullptr;
    }
    slot.second = want;
  }
  return slot.first;
}

// 32 outputs x 8 part lanes per CTA: lane l sums parts l, l + 8, ... in order, then the 8 lane sums are added in order
__global__ void reduce_parts_kernel(const float* __restrict__ part, int parts, long long stride, long long n,
                                    float* __restrict__ out, int accumulate) {
  __shared__ float red[8][33];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const long long i = (long long)blockIdx.x * 32 + tx;
  float s = 0.f;
  if (i < n)
    for (int z = ty; z < parts; z += 8) s += part[(long long)z * stride + i];
  red[ty][tx] = s;
  __syncthreads();
  if (ty == 0 && i < n) {
    float t = 0.f;
#pragma unroll
    for (int w = 0; w < 8; w++) t += red[w][tx];
    out[i] = (accumulate ? out[i] : 0.f) + t;
  }
}

int reduce_parts(const float* part, int parts, long long stride, long long n, float* out, int accumulate, cudaStream_t st) {
  if (n <= 0) return B200ASR_OK;
  reduce_parts_kernel<<<(unsigned)ceil_div_ll(n, 32), 256, 0, st>>>(part, parts, stride, n, out, accumulate);
  return check_launch("reduce_parts");
}

}  // namespace b200asr

extern "C" {
int b200asr_version(void) { return 100; }
const char* b200asr_last_error(void) { return b200asr::g_err; }
int b200asr_device_check(void) { return b200asr::ensure_sm90(); }
unsigned long long b200asr_launch_count(void) { return b200asr::g_launches; }
}
