// Device helpers shared by the MT decoder's single-token kernel (kernels_persist_mt.cu) and its batched form
// (kernels_persist_mtb.cu).  Both kernels build every row from these functions, which is what makes a row of the batched search
// bit-identical to the single-token search of the same sample.  Internal to those two translation units.
#pragma once
#include "common.cuh"
#include "kernels.h"
#include "kernels_persist.h"

namespace ss {
namespace {

constexpr int MW = 8;
constexpr int MTT = MW * 32;
constexpr int MHD = 64;

__device__ __forceinline__ float4 ldw(const float* p) {
  float4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p));
  return r;
}

struct MtSmem {
  float x[512];     // residual stream of the token (model dim <= 512)
  float v[2048];    // GEMV input vector (LN(x), attention output or FFN hidden)
  float S[1024];    // attention scores
  float qh[MHD];
  float pv[16][MHD];
  float red[MW];
  float rbest[MW];
  int ridx[MW];
  int tok;
};

__device__ __forceinline__ float block_reduce_sum(MtSmem& sm, float v) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  v = warp_sum(v);
  __syncthreads();
  if (lane == 0) sm.red[w] = v;
  __syncthreads();
  float t = sm.red[0];
#pragma unroll
  for (int i = 1; i < MW; ++i) t += sm.red[i];
  return t;
}
__device__ __forceinline__ float block_reduce_max(MtSmem& sm, float v) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  v = warp_max(v);
  __syncthreads();
  if (lane == 0) sm.red[w] = v;
  __syncthreads();
  float t = sm.red[0];
#pragma unroll
  for (int i = 1; i < MW; ++i) t = fmaxf(t, sm.red[i]);
  return t;
}

// sm.v[0..dim) = LayerNorm(sm.x[0..dim)) (two-pass, as layer_norm_kernel); dim == 512: two values per thread
__device__ __forceinline__ void ln_to_v(MtSmem& sm, const float* __restrict__ g, const float* __restrict__ b, int dim) {
  const int t = threadIdx.x;
  float a0 = sm.x[t], a1 = sm.x[t + MTT];
  float mean = block_reduce_sum(sm, a0 + a1) / (float)dim;
  float d0 = a0 - mean, d1 = a1 - mean;
  float var = block_reduce_sum(sm, fmaf(d0, d0, d1 * d1)) / (float)dim;
  float rstd = 1.0f / sqrtf(var + 1e-5f);
  sm.v[t] = d0 * rstd * g[t] + b[t];
  sm.v[t + MTT] = d1 * rstd * g[t + MTT] + b[t + MTT];
  __syncthreads();
}

// LayerNorm parameters of this thread's two columns, loaded ahead of use (the loads fly while the phase's input arrives)
struct LnP {
  float g0, g1, b0, b1;
};
__device__ __forceinline__ LnP ln_load(const float* __restrict__ g, const float* __restrict__ b) {
  const int t = threadIdx.x;
  return LnP{__ldg(g + t), __ldg(g + t + MTT), __ldg(b + t), __ldg(b + t + MTT)};
}
__device__ __forceinline__ void ln_to_v(MtSmem& sm, const LnP& p, int dim) {
  const int t = threadIdx.x;
  float a0 = sm.x[t], a1 = sm.x[t + MTT];
  float mean = block_reduce_sum(sm, a0 + a1) / (float)dim;
  float d0 = a0 - mean, d1 = a1 - mean;
  float var = block_reduce_sum(sm, fmaf(d0, d0, d1 * d1)) / (float)dim;
  float rstd = 1.0f / sqrtf(var + 1e-5f);
  sm.v[t] = d0 * rstd * p.g0 + p.b0;
  sm.v[t + MTT] = d1 * rstd * p.g1 + p.b1;
  __syncthreads();
}

// coherent copy global -> shared (activations written by other CTAs before the last barrier)
__device__ __forceinline__ void load_vec(float* dst, const float* src, int n) {
  for (int i = threadIdx.x * 4; i < n; i += MTT * 4) *reinterpret_cast<float4*>(dst + i) = *reinterpret_cast<const float4*>(src + i);
  __syncthreads();
}

// y[col] = epi(col, W[col][:] . xs) for col in [0, N): warp gw owns columns gw, gw + nw, ... (at most MAXC: every phase is
// sized so that one round covers N).  Split in two so that the weight loads are in flight while the CTA stages the input
// vector (global -> shared, LayerNorm): gemv_issue() before the staging, gemv_finish() after it.
template <int K, int MAXC>
struct GemvW {
  float4 w[MAXC][K / 128];
  float bias[MAXC];  // (filled by gemv_issue_b: the epilogue of gemv_finish_b receives acc + bias)
};
template <int K, int MAXC>
__device__ __forceinline__ void gemv_issue(GemvW<K, MAXC>& r, const float* __restrict__ W, int N) {
  const int lane = threadIdx.x & 31;
  const int gw = blockIdx.x * MW + (threadIdx.x >> 5), nw = gridDim.x * MW;
#pragma unroll
  for (int c = 0; c < MAXC; ++c) {
    const int col = gw + c * nw;
#pragma unroll
    for (int it = 0; it < K / 128; ++it)
      r.w[c][it] = col < N ? ldw(W + (int64_t)col * K + it * 128 + lane * 4) : make_float4(0.f, 0.f, 0.f, 0.f);
  }
}
// variant with the bias of each column loaded together with its weights (no global load left in the epilogue)
template <int K, int MAXC>
__device__ __forceinline__ void gemv_issue_b(GemvW<K, MAXC>& r, const float* __restrict__ W, int N, const float* __restrict__ bias) {
  gemv_issue(r, W, N);
  const int gw = blockIdx.x * MW + (threadIdx.x >> 5), nw = gridDim.x * MW;
#pragma unroll
  for (int c = 0; c < MAXC; ++c) {
    const int col = gw + c * nw;
    r.bias[c] = (bias != nullptr && col < N) ? __ldg(bias + col) : 0.f;
  }
}
template <int K, int MAXC, typename F>
__device__ __forceinline__ void gemv_finish_b(const GemvW<K, MAXC>& r, const float* xs, int N, F&& epi) {
  constexpr int NIT = K / 128;
  const int lane = threadIdx.x & 31;
  const int gw = blockIdx.x * MW + (threadIdx.x >> 5), nw = gridDim.x * MW;
  float4 xv[NIT];
#pragma unroll
  for (int it = 0; it < NIT; ++it) xv[it] = *reinterpret_cast<const float4*>(xs + it * 128 + lane * 4);
#pragma unroll
  for (int c = 0; c < MAXC; ++c) {
    float acc = 0.f;
#pragma unroll
    for (int it = 0; it < NIT; ++it) {
      acc = fmaf(xv[it].x, r.w[c][it].x, acc);
      acc = fmaf(xv[it].y, r.w[c][it].y, acc);
      acc = fmaf(xv[it].z, r.w[c][it].z, acc);
      acc = fmaf(xv[it].w, r.w[c][it].w, acc);
    }
    acc = warp_sum(acc);
    const int col = gw + c * nw;
    if (lane == 0 && col < N) epi(col, acc + r.bias[c]);
  }
}
template <int K, int MAXC, typename F>
__device__ __forceinline__ void gemv_finish(const GemvW<K, MAXC>& r, const float* xs, int N, F&& epi) {
  constexpr int NIT = K / 128;
  const int lane = threadIdx.x & 31;
  const int gw = blockIdx.x * MW + (threadIdx.x >> 5), nw = gridDim.x * MW;
  float4 xv[NIT];
#pragma unroll
  for (int it = 0; it < NIT; ++it) xv[it] = *reinterpret_cast<const float4*>(xs + it * 128 + lane * 4);
#pragma unroll
  for (int c = 0; c < MAXC; ++c) {
    float acc = 0.f;
#pragma unroll
    for (int it = 0; it < NIT; ++it) {
      acc = fmaf(xv[it].x, r.w[c][it].x, acc);
      acc = fmaf(xv[it].y, r.w[c][it].y, acc);
      acc = fmaf(xv[it].z, r.w[c][it].z, acc);
      acc = fmaf(xv[it].w, r.w[c][it].w, acc);
    }
    acc = warp_sum(acc);
    const int col = gw + c * nw;
    if (lane == 0 && col < N) epi(col, acc);
  }
}

// arg-max of log_softmax(x[0 .. vocab)) with pad always masked and eos masked while s < 1 (min_len), first index wins on ties
// (argmax_rows_kernel); the whole CTA computes it, every thread gets the index
__device__ __forceinline__ int masked_argmax(MtSmem& sm, const float* x, int vocab, int pad, int eos, int s) {
  const int tid = threadIdx.x;
  float mx = -INFINITY;
  for (int c = tid; c < vocab; c += MTT) mx = fmaxf(mx, x[c]);
  mx = block_reduce_max(sm, mx);
  float su = 0.f;
  for (int c = tid; c < vocab; c += MTT) su += expf(x[c] - mx);
  su = block_reduce_sum(sm, su);
  const float lse = logf(su);
  float best = -INFINITY;
  int bi = 0x7fffffff;
  for (int c = tid; c < vocab; c += MTT) {
    const bool masked = (c == pad) || (s < 1 && c == eos);
    float lp = masked ? -INFINITY : (x[c] - mx) - lse;
    if (lp > best || (lp == best && c < bi)) {
      best = lp;
      bi = c;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    float ob = __shfl_xor_sync(0xffffffffu, best, o);
    int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (ob > best || (ob == best && oi < bi)) {
      best = ob;
      bi = oi;
    }
  }
  __syncthreads();
  if ((tid & 31) == 0) {
    sm.rbest[tid >> 5] = best;
    sm.ridx[tid >> 5] = bi;
  }
  __syncthreads();
  if (tid == 0) {
    for (int i = 1; i < MW; ++i)
      if (sm.rbest[i] > best || (sm.rbest[i] == best && sm.ridx[i] < bi)) {
        best = sm.rbest[i];
        bi = sm.ridx[i];
      }
    sm.tok = bi;
  }
  __syncthreads();
  return sm.tok;
}

// one output column of a head's out-projection partial: a = the head's attention output (a0 = a[lane], a1 = a[lane + 32]),
// w0 / w1 = the column's weights at the same inputs; every lane gets the sum
__device__ __forceinline__ float head_col_partial(float a0, float a1, float w0, float w1) { return warp_sum(fmaf(a0, w0, a1 * w1)); }

// out-projection of a head (v2's per-head partials): columns are split over the CTAs of a head group
constexpr int GRP = 16;                 // CTAs per head group (8 heads x 16 = 128 CTAs)
constexpr int PCOLS = 512 / GRP;        // out-projection columns per CTA of a group
constexpr int PCOLS_PER_WARP = PCOLS / MW;

// attend_head with every independent load issued up front: the key row of this thread, the first 8 value rows of its part and the
// query are all in flight together (one L2 round trip instead of three dependent ones); n <= 256 keys take a single pass
__device__ void attend_head_early(MtSmem& sm, const float* q, const float* kbase, const float* vbase, int ld, int n, float* out) {
  const int tid = threadIdx.x;
  const int q4 = (tid & 15) * 4, part = tid >> 4;
  float4 kk[MHD / 4];
  {
    const bool ok = tid < n;
    const float* kr = kbase + (int64_t)(ok ? tid : 0) * ld;
#pragma unroll
    for (int d = 0; d < MHD / 4; ++d) kk[d] = ok ? *reinterpret_cast<const float4*>(kr + 4 * d) : make_float4(0.f, 0.f, 0.f, 0.f);
  }
  float4 vv0[8];
#pragma unroll
  for (int u = 0; u < 8; ++u) {
    const int j = part + 16 * u;
    vv0[u] = j < n ? *reinterpret_cast<const float4*>(vbase + (int64_t)j * ld + q4) : make_float4(0.f, 0.f, 0.f, 0.f);
  }
  __syncthreads();
  if (tid < MHD) sm.qh[tid] = q[tid] * 0.125f;
  __syncthreads();
  float mx = -INFINITY;
  for (int j = tid; j < n; j += MTT) {
    if (j != tid) {
      const float* kr = kbase + (int64_t)j * ld;
#pragma unroll
      for (int d = 0; d < MHD / 4; ++d) kk[d] = *reinterpret_cast<const float4*>(kr + 4 * d);
    }
    float s = 0.f;
#pragma unroll
    for (int d = 0; d < MHD / 4; ++d) {
      s = fmaf(sm.qh[4 * d], kk[d].x, s);
      s = fmaf(sm.qh[4 * d + 1], kk[d].y, s);
      s = fmaf(sm.qh[4 * d + 2], kk[d].z, s);
      s = fmaf(sm.qh[4 * d + 3], kk[d].w, s);
    }
    sm.S[j] = s;
    mx = fmaxf(mx, s);
  }
  mx = block_reduce_max(sm, mx);
  float sum = 0.f;
  for (int j = tid; j < n; j += MTT) {
    float e = expf(sm.S[j] - mx);
    sm.S[j] = e;
    sum += e;
  }
  sum = block_reduce_sum(sm, sum);
  float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll 1
  for (int j0 = part; j0 < n; j0 += 16 * 8) {
    float4 vv[8];
    float pp[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      const int j = j0 + 16 * u;
      const bool ok = j < n;
      vv[u] = j0 == part ? vv0[u] : (ok ? *reinterpret_cast<const float4*>(vbase + (int64_t)j * ld + q4) : make_float4(0.f, 0.f, 0.f, 0.f));
      pp[u] = ok ? sm.S[j] : 0.f;
    }
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      a.x = fmaf(pp[u], vv[u].x, a.x);
      a.y = fmaf(pp[u], vv[u].y, a.y);
      a.z = fmaf(pp[u], vv[u].z, a.z);
      a.w = fmaf(pp[u], vv[u].w, a.w);
    }
  }
  *reinterpret_cast<float4*>(&sm.pv[part][q4]) = a;
  __syncthreads();
  if (tid < MHD) {
    float t = 0.f;
#pragma unroll
    for (int x = 0; x < 16; ++x) t += sm.pv[x][tid];
    out[tid] = t / sum;
  }
}

// x[c] += sum_h part[h][c] + bias[c]   (every CTA, identical order); x is a 512-float residual row in shared memory,
// part is [8][512] in global memory
__device__ __forceinline__ void add_head_partials(float* x, const float* part, const float* __restrict__ bias) {
  for (int c = threadIdx.x; c < 512; c += MTT) {
    float t = part[c];
#pragma unroll
    for (int h = 1; h < 8; ++h) t += part[h * 512 + c];
    x[c] = x[c] + (t + (bias ? bias[c] : 0.f));
  }
  __syncthreads();
}

// L2 prefetch of the weight rows this warp's gemv phase will read (same column assignment as gemv_issue): one layer ahead, so that the
// register loads of the phase hit L2 instead of HBM (the first pass over a layer's 14.7 MB otherwise costs a DRAM latency per phase)
template <int K, int MAXC>
__device__ __forceinline__ void gemv_prefetch(const float* __restrict__ W, int N) {
  const int lane = threadIdx.x & 31;
  const int gw = blockIdx.x * MW + (threadIdx.x >> 5), nw = gridDim.x * MW;
  constexpr int LINES = K * 4 / 128;  // 128-byte lines per weight row
#pragma unroll
  for (int c = 0; c < MAXC; ++c) {
    const int col = gw + c * nw;
    if (col < N) {
#pragma unroll
      for (int l0 = 0; l0 < LINES; l0 += 32)
        if (l0 + lane < LINES) asm volatile("prefetch.global.L2 [%0];" ::"l"(W + (int64_t)col * K + (l0 + lane) * 32));
    }
  }
}
// ... and of the 32 x 64 out-projection block of (head h, column group j): 2 lines per column
__device__ __forceinline__ void hp_prefetch(const float* __restrict__ W, int h, int j) {
  const int t = threadIdx.x;
  if (t < PCOLS * 2) asm volatile("prefetch.global.L2 [%0];" ::"l"(W + (int64_t)(j * PCOLS + (t >> 1)) * 512 + h * MHD + (t & 1) * 32));
}
__device__ __forceinline__ void layer_prefetch(const MtLayerP& L, bool in_group, int grp_h, int grp_j) {
  gemv_prefetch<512, 2>(L.wqkv, 3 * 512);
  gemv_prefetch<512, 1>(L.wcq, 512);
  gemv_prefetch<512, 2>(L.w1, 2048);
  gemv_prefetch<2048, 1>(L.w2, 512);
  if (in_group) {
    hp_prefetch(L.wo, grp_h, grp_j);
    hp_prefetch(L.wco, grp_h, grp_j);
  }
}

}  // namespace
}  // namespace ss
