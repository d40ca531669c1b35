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

// launch with programmatic stream serialization: the grid may be scheduled while its predecessor is still running; every
// kernel launched this way calls pdl_wait() before it touches memory (so semantics equal a normal launch, minus the
// launch / scheduling latency that now overlaps the predecessor)
template <typename... KArgs, typename... Args>
inline void launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args... args) {
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
  attr[0].val.programmaticStreamSerializationAllowed = ctas <= 296 ? 1 : 0;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

// same, unconditionally (kernels that do real work before pdl_wait(): the skinny GEMM's weight prefetch)
template <typename... KArgs, typename... Args>
inline void launch_pdl_always(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
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

// arg-max of log_softmax(x[0 .. V)) with the columns masked[0 .. n_masked) excluded, first index wins on ties, for a block of 256
// threads (CTCDecoder.generate, agent/ctc_decoder.py:53-62; F.log_softmax = (x - max) - log(sum(exp(x - max)))).  Every row of
// every caller goes through this one reduction order, so all arg-maxes agree bit for bit.  The index is valid in thread 0.
__device__ __forceinline__ int block_masked_argmax256(const float* __restrict__ x, int V, const int* __restrict__ masked, int n_masked) {
  __shared__ float red[32];
  __shared__ float sval[8];
  __shared__ int sidx[8];
  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  float mx = -INFINITY;
  for (int c = tid; c < V; c += 256) mx = fmaxf(mx, x[c]);
  mx = warp_max(mx);
  if (lane == 0) red[w] = mx;
  __syncthreads();
  mx = red[0];
  for (int i = 1; i < 8; ++i) mx = fmaxf(mx, red[i]);
  __syncthreads();
  float s = 0.f;
  for (int c = tid; c < V; c += 256) s += expf(x[c] - mx);
  s = block_sum(s, red);
  const float lse = logf(s);
  float best = -INFINITY;
  int bi = 0x7fffffff;
  for (int c = tid; c < V; c += 256) {
    bool m = false;
    for (int q = 0; q < n_masked; ++q) m |= (masked[q] == c);
    const float lp = m ? -INFINITY : (x[c] - mx) - lse;
    if (lp > best || (lp == best && c < bi)) {
      best = lp;
      bi = c;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ob = __shfl_xor_sync(0xffffffffu, best, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (ob > best || (ob == best && oi < bi)) {
      best = ob;
      bi = oi;
    }
  }
  __syncthreads();
  if (lane == 0) {
    sval[w] = best;
    sidx[w] = bi;
  }
  __syncthreads();
  if (tid == 0) {
    for (int i = 1; i < 8; ++i)  // per-warp winners in warp order
      if (sval[i] > best || (sval[i] == best && sidx[i] < bi)) {
        best = sval[i];
        bi = sidx[i];
      }
  }
  return bi;
}

// CTC collapse (CTCDecoder.generate, agent/ctc_decoder.py:64-111) of one arg-max sequence am[i * stride], i < n: repeats, then
// blank and pad, are dropped; the kept tokens go to toks[0 .. count), their positions to index (optional), the count to *count.
// Any block size that is a multiple of 32 up to 1024: thread t owns the contiguous slice [t * per, (t + 1) * per) and a block-wide
// exclusive scan of the keep counts places its outputs.  The loads bypass L1 (__ldcg), so the arg-max may have been written by
// other CTAs of the same grid.  `wsum` is 32 ints of shared memory; a caller that collapses twice synchronises in between.
__device__ __forceinline__ void block_ctc_collapse(const int64_t* am, int64_t stride, int n, int blank, int pad, int64_t* __restrict__ toks,
                                                   int* __restrict__ index, int* __restrict__ count, int* wsum) {
  const int t = threadIdx.x, lane = t & 31, w = t >> 5, nw = blockDim.x >> 5;
  const int per = (n + (int)blockDim.x - 1) / (int)blockDim.x;
  const int lo = min(n, t * per), hi = min(n, lo + per);
  int c = 0;
  int64_t prev = lo > 0 ? __ldcg(am + (int64_t)(lo - 1) * stride) : -1;
  for (int i = lo; i < hi; ++i) {
    const int64_t v = __ldcg(am + (int64_t)i * stride);
    if ((i == 0 || v != prev) && v != blank && v != pad) ++c;
    prev = v;
  }
  int inc = c;  // inclusive scan inside the warp, then over the warp totals
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int y = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += y;
  }
  if (lane == 31) wsum[w] = inc;
  __syncthreads();
  if (w == 0) {
    int s = lane < nw ? wsum[lane] : 0;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int y = __shfl_up_sync(0xffffffffu, s, o);
      if (lane >= o) s += y;
    }
    wsum[lane] = s;  // wsum[31] = the total
  }
  __syncthreads();
  int base = (w > 0 ? wsum[w - 1] : 0) + inc - c;
  prev = lo > 0 ? __ldcg(am + (int64_t)(lo - 1) * stride) : -1;
  for (int i = lo; i < hi; ++i) {
    const int64_t v = __ldcg(am + (int64_t)i * stride);
    if ((i == 0 || v != prev) && v != blank && v != pad) {
      toks[base] = v;
      if (index) index[base] = i;
      ++base;
    }
    prev = v;
  }
  if (t == 0) *count = wsum[31];
}

}  // namespace ss
