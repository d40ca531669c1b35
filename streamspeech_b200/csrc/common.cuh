// Shared device helpers for the sm_90a kernels.
#pragma once
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include <mutex>
#include <set>
#include <unordered_set>
#include <utility>

namespace ss {

// Programmatic dependent launch: allow the next kernel in the stream (if it was launched with the PDL attribute, see
// kernels_skinny.cu) to begin its independent prologue while this grid is still running.  A no-op otherwise.
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
// ... and the matching wait: everything the previous kernels of the stream wrote is visible after it.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// set while a stream capture is recording the launches (CUDA-graph replay of a stage): programmatic launches are recorded
// as plain launches unless the engine option graph_pdl asks otherwise
extern thread_local int g_pdl_off;

// Shared-memory carve-out: the wgmma kernels need > 100 KB of shared memory per CTA, the SIMT kernels a few KB.  An SM
// holds ONE carve-out at a time, so kernels that ask for different ones cannot share an SM and every change drains it
// -- which is what the vocoder's three concurrent streams of alternating conv / reduce kernels would do.  With the option on
// (default) every kernel of the library asks for the maximum shared-memory carve-out, once per kernel function.
extern int g_prefer_shared;

// Function attributes (cudaFuncSetAttribute) belong to the CURRENT DEVICE: a process that holds handles on several devices
// must configure every kernel once per device, not once per process.  true the first time (device, key) is seen.
inline bool first_time_on_device(const void* key) {
  static std::mutex mu;
  static std::set<std::pair<int, const void*>> seen;
  int dev = 0;
  cudaGetDevice(&dev);
  std::lock_guard<std::mutex> g(mu);
  return seen.insert({dev, key}).second;
}
// SM count of the current device (cached per device)
inline int current_device_sms() {
  static std::mutex mu;
  static int sms[64] = {0};
  int dev = 0;
  cudaGetDevice(&dev);
  std::lock_guard<std::mutex> g(mu);
  if (dev < 0 || dev >= 64) return 0;
  if (sms[dev] == 0) cudaDeviceGetAttribute(&sms[dev], cudaDevAttrMultiProcessorCount, dev);
  return sms[dev];
}

inline void prefer_shared_once(const void* fn) {
  if (!g_prefer_shared) return;
  // (key fn + 1: a key space distinct from the max-shared-memory configuration of the same function)
  if (first_time_on_device((const char*)fn + 1)) cudaFuncSetAttribute(fn, cudaFuncAttributePreferredSharedMemoryCarveout, 100);
}

// launch with programmatic stream serialization: the grid may be scheduled while its predecessor is still running; every
// kernel launched this way calls pdl_wait() before it touches memory (so semantics equal a normal launch, minus the
// launch / scheduling latency that now overlaps the predecessor)
template <typename... KArgs, typename... Args>
inline void launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args... args) {
  prefer_shared_once((const void*)kernel);
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  // only small grids launch early: CTAs of a large dependent grid would sit on shared memory / registers that the
  // (multi-wave) predecessor still needs
  const unsigned long long ctas = (unsigned long long)grid.x * grid.y * grid.z;
  attr[0].val.programmaticStreamSerializationAllowed = (ctas <= 296 && !g_pdl_off) ? 1 : 0;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

// same, unconditionally (kernels that do real work before pdl_wait(): the skinny GEMM's weight prefetch)
template <typename... KArgs, typename... Args>
inline void launch_pdl_always(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args... args) {
  prefer_shared_once((const void*)kernel);
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = g_pdl_off ? 0 : 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

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

// block-wide sum for blockDim.x <= 1024 (multiple of 32); `red` is >= 32 floats of shared memory
__device__ __forceinline__ float block_sum(float v, float* red) {
  int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  v = warp_sum(v);
  __syncthreads();
  if (lane == 0) red[w] = v;
  __syncthreads();
  int nw = (blockDim.x + 31) >> 5;
  float t = (threadIdx.x < nw) ? red[threadIdx.x] : 0.f;
  if (w == 0) {
    t = warp_sum(t);
    if (lane == 0) red[0] = t;
  }
  __syncthreads();
  return red[0];
}

}  // namespace ss
