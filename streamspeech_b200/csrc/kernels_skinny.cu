// Skinny GEMM for the streaming regime (M <= 64 rows: cached encoder step M = 16, MT decode step M = 1):
//   out[m][n] = epilogue( sum_k A[m][k] * W[n][k] ),  A row-major [M][K], W row-major [N][K].
// These GEMMs are weight-streaming problems (2 MB of W for 16 rows), so the kernel is organised around memory-level
// parallelism instead of tiles:
//   * one warp per (group of CPT output columns, K-slice); lanes stride K with 128-bit loads, so CPT whole slices of
//     W rows are in flight per warp at once; W is read exactly once (streaming, L1 no-allocate), the A rows
//     (<= 128 KB) are re-read through L1/L2 once per column group;
//   * the KS K-slices of a column group live in one CTA and are combined through shared memory in a fixed order
//     (deterministic results); the epilogue (bias / ReLU / SiLU / GLU / residual / Q|K|V routing) runs one row per lane;
//   * optional fused LayerNorm of A (row statistics per CTA, normalisation applied while loading A);
//   * programmatic dependent launch: the first W slices are fetched BEFORE griddepcontrol.wait, i.e. while the previous
//     kernel of the stream is still running (weights never depend on it).
// HBM/L2-bound by construction: algorithmic bytes = N*K*4 (weights) + M*K*4 + M*N*4.
#include "common.cuh"
#include "kernels.h"

namespace ss {
namespace {

constexpr int SK_WARPS = 8;
constexpr int SK_PF = 2;  // prefetched 128-bit W loads per column and lane

__device__ __forceinline__ float sk_act(float x, int act) {
  switch (act) {
    case ACT_RELU: return x > 0.f ? x : 0.f;
    case ACT_SILU: return x / (1.0f + expf(-x));
    case ACT_TANH: return tanhf(x);
    default: return x;
  }
}

__device__ __forceinline__ float4 ld_stream(const float* p) {
  float4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p));
  return r;
}

// MR = rows per pass (accumulators per lane and column), KS = K-slices per column group, CPT = columns per task
// (GLU: CPT = 2 = one (value, gate) pair)
template <int MR, int KS, int CPT, bool GLU>
__global__ void __launch_bounds__(SK_WARPS * 32) skinny_gemm_kernel(const float* __restrict__ A, int lda, const float* __restrict__ W,
                                                                    int M, int N, int K, Epilogue ep) {
  constexpr int TASKS_PER_CTA = SK_WARPS / KS;
  __shared__ float part[SK_WARPS][CPT][MR];
  __shared__ float ln_mean[64], ln_rstd[64];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const bool fuse_ln = ep.ln_gamma != nullptr;
  const int slice = warp % KS, tslot = warp / KS;
  const int ntasks = N / CPT;
  const int kslice = K / KS;  // multiple of 128 (checked by the host)
  const int k_lo = slice * kslice, k_hi = k_lo + kslice;
  const int first_task = blockIdx.x * TASKS_PER_CTA + tslot;

  pdl_trigger();
  float4 wpre[CPT][SK_PF];
#pragma unroll
  for (int c = 0; c < CPT; ++c)
#pragma unroll
    for (int i = 0; i < SK_PF; ++i) {
      int k = k_lo + lane * 4 + i * 128;
      wpre[c][i] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (first_task < ntasks && k < k_hi) wpre[c][i] = ld_stream(W + ((int64_t)first_task * CPT + c) * K + k);
    }
  pdl_wait();

  if (fuse_ln) {
    // row statistics with the same operation order as layer_norm_kernel (two-pass, lane-strided, shuffle tree)
    for (int m = warp; m < M; m += SK_WARPS) {
      const float* xr = A + (int64_t)m * lda;
      float s = 0.f;
      for (int c = lane; c < K; c += 32) s += xr[c];
      float mean = warp_sum(s) / (float)K;
      float ss_ = 0.f;
      for (int c = lane; c < K; c += 32) {
        float d = xr[c] - mean;
        ss_ = fmaf(d, d, ss_);
      }
      float var = warp_sum(ss_) / (float)K;
      if (lane == 0) {
        ln_mean[m] = mean;
        ln_rstd[m] = 1.0f / sqrtf(var + 1e-5f);
      }
    }
    __syncthreads();
  }

  for (int tbase = blockIdx.x * TASKS_PER_CTA; tbase < ntasks; tbase += gridDim.x * TASKS_PER_CTA) {
    const int task = tbase + tslot;
    const bool active = task < ntasks;
    const int n0 = task * CPT;
    for (int mb = 0; mb < M; mb += MR) {
      float acc[CPT][MR];
#pragma unroll
      for (int c = 0; c < CPT; ++c)
#pragma unroll
        for (int r = 0; r < MR; ++r) acc[c][r] = 0.f;
      if (active) {
        const float* w0 = W + (int64_t)n0 * K;
        const bool first = (task == first_task) && mb == 0;
        auto step = [&](int k, const float4* wv) {
          float4 g4 = make_float4(1.f, 1.f, 1.f, 1.f), b4 = make_float4(0.f, 0.f, 0.f, 0.f);
          if (fuse_ln) {
            g4 = *reinterpret_cast<const float4*>(ep.ln_gamma + k);
            b4 = *reinterpret_cast<const float4*>(ep.ln_beta + k);
          }
#pragma unroll
          for (int r = 0; r < MR; ++r) {
            if (mb + r < M) {
              float4 x = *reinterpret_cast<const float4*>(A + (int64_t)(mb + r) * lda + k);
              if (fuse_ln) {
                const float mu = ln_mean[mb + r], rs = ln_rstd[mb + r];
                x.x = (x.x - mu) * rs * g4.x + b4.x;
                x.y = (x.y - mu) * rs * g4.y + b4.y;
                x.z = (x.z - mu) * rs * g4.z + b4.z;
                x.w = (x.w - mu) * rs * g4.w + b4.w;
              }
#pragma unroll
              for (int c = 0; c < CPT; ++c) {
                acc[c][r] = fmaf(x.x, wv[c].x, acc[c][r]);
                acc[c][r] = fmaf(x.y, wv[c].y, acc[c][r]);
                acc[c][r] = fmaf(x.z, wv[c].z, acc[c][r]);
                acc[c][r] = fmaf(x.w, wv[c].w, acc[c][r]);
              }
            }
          }
        };
        int k = k_lo + lane * 4;
#pragma unroll
        for (int i = 0; i < SK_PF; ++i, k += 128) {
          if (k < k_hi) {
            float4 wv[CPT];
#pragma unroll
            for (int c = 0; c < CPT; ++c) wv[c] = first ? wpre[c][i] : ld_stream(w0 + (int64_t)c * K + k);
            step(k, wv);
          }
        }
#pragma unroll 2
        for (; k < k_hi; k += 128) {
          float4 wv[CPT];
#pragma unroll
          for (int c = 0; c < CPT; ++c) wv[c] = ld_stream(w0 + (int64_t)c * K + k);
          step(k, wv);
        }
      }
      // lane r ends up holding the warp totals of row r
      float mine[CPT];
#pragma unroll
      for (int c = 0; c < CPT; ++c) {
        mine[c] = 0.f;
#pragma unroll
        for (int r = 0; r < MR; ++r) {
          float t = warp_sum(acc[c][r]);
          if (lane == r) mine[c] = t;
        }
      }
      if (KS > 1) {
        if (lane < MR) {
#pragma unroll
          for (int c = 0; c < CPT; ++c) part[warp][c][lane] = mine[c];
        }
        __syncthreads();
        if (slice == 0 && lane < MR) {
#pragma unroll
          for (int c = 0; c < CPT; ++c) {
            float t = part[warp][c][lane];
#pragma unroll
            for (int s = 1; s < KS; ++s) t += part[warp + s][c][lane];
            mine[c] = t;
          }
        }
      }
      const int m = mb + lane;
      if (active && slice == 0 && lane < MR && m < M) {
#pragma unroll
        for (int c = 0; c < (GLU ? 1 : CPT); ++c) {
          float y;
          int oc;
          if (GLU) {
            float av = mine[0] + (ep.bias ? ep.bias[n0] : 0.f);
            float gv = mine[CPT - 1] + (ep.bias ? ep.bias[n0 + 1] : 0.f);
            y = ep.alpha * (av * (1.0f / (1.0f + expf(-gv))));
            oc = n0 >> 1;
          } else {
            y = ep.alpha * sk_act(mine[c] + (ep.bias ? ep.bias[n0 + c] : 0.f), ep.act);
            oc = n0 + c;
          }
          float* obase = ep.out;
          int ld = ep.ldo;
          if (ep.split_n > 0) {  // fused Q|K|V: route the column block to its own buffer
            int p = oc / ep.split_n;
            oc -= p * ep.split_n;
            if (p == 1) { obase = ep.out2; ld = ep.ldo2; }
            else if (p == 2) { obase = ep.out3; ld = ep.ldo3; }
          }
          int64_t o = (int64_t)m * ld + oc;
          if (ep.residual) y += ep.res_scale * ep.residual[o];
          if (ep.accumulate) y += obase[o];
          obase[o] = y;
        }
      }
      if (KS > 1) __syncthreads();  // `part` is reused by the next pass / task
    }
  }
}

template <int MR, int KS, int CPT, bool GLU>
void launch_skinny(const float* A, int lda, const float* W, int M, int N, int K, const Epilogue& ep, cudaStream_t st) {
  const int ntasks = N / CPT;
  const int per_cta = SK_WARPS / KS;
  int grid = (ntasks + per_cta - 1) / per_cta;
  // with a fused LayerNorm every CTA recomputes the row statistics: keep the grid at two CTAs per SM and loop over tasks
  const int sms = std::max(1, current_device_sms());
  const int cap = ep.ln_gamma ? sms * 2 : sms * 8;
  if (grid > cap) grid = cap;
  launch_pdl_always(skinny_gemm_kernel<MR, KS, CPT, GLU>, dim3(grid), dim3(SK_WARPS * 32), 0, st, A, lda, W, M, N, K, ep);
}

template <int MR, int CPT, bool GLU>
void dispatch_ks(int ks, const float* A, int lda, const float* W, int M, int N, int K, const Epilogue& ep, cudaStream_t st) {
  switch (ks) {
    case 1: launch_skinny<MR, 1, CPT, GLU>(A, lda, W, M, N, K, ep, st); break;
    case 2: launch_skinny<MR, 2, CPT, GLU>(A, lda, W, M, N, K, ep, st); break;
    case 4: launch_skinny<MR, 4, CPT, GLU>(A, lda, W, M, N, K, ep, st); break;
    default: launch_skinny<MR, 8, CPT, GLU>(A, lda, W, M, N, K, ep, st); break;
  }
}

}  // namespace

bool skinny_gemm_supported(int M, int N, int K, const Epilogue& ep) {
  if (M < 1 || M > 64 || (K & 127) != 0 || ep.out_L > 0) return false;
  if (ep.ln_gamma && K > 1024) return false;
  if (ep.glu && (N & 1)) return false;
  return true;
}

void skinny_gemm(const float* A, int lda, const float* W, int M, int N, int K, const Epilogue& ep, cudaStream_t st) {
  ++g_launches;
  // columns per warp-task: 4 independent W rows in flight per lane and one A load shared by 4 columns
  const int cpt = ep.glu ? 2 : ((N & 3) == 0 && (ep.split_n == 0 || (ep.split_n & 3) == 0) ? 4 : 1);
  const int ntasks = N / cpt;
  // K-slices per column group: enough warp-tasks to cover the SMs, every slice a multiple of 128 columns
  int ks = 1;
  while (ks < 8 && (long)ntasks * ks < 1184 && K % (ks * 2 * 128) == 0) ks *= 2;
  if (M == 1) {
    if (ep.glu) dispatch_ks<1, 2, true>(ks, A, lda, W, M, N, K, ep, st);
    else if (cpt == 4) dispatch_ks<1, 4, false>(ks, A, lda, W, M, N, K, ep, st);
    else dispatch_ks<1, 1, false>(ks, A, lda, W, M, N, K, ep, st);
  } else if (M <= 8) {
    if (ep.glu) dispatch_ks<8, 2, true>(ks, A, lda, W, M, N, K, ep, st);
    else if (cpt == 4) dispatch_ks<8, 4, false>(ks, A, lda, W, M, N, K, ep, st);
    else dispatch_ks<8, 1, false>(ks, A, lda, W, M, N, K, ep, st);
  } else {
    if (ep.glu) dispatch_ks<16, 2, true>(ks, A, lda, W, M, N, K, ep, st);
    else if (cpt == 4) dispatch_ks<16, 4, false>(ks, A, lda, W, M, N, K, ep, st);
    else dispatch_ks<16, 1, false>(ks, A, lda, W, M, N, K, ep, st);
  }
}

}  // namespace ss
