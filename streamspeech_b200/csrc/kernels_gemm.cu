// fp32 SIMT GEMM with an implicit-im2col A operand (conv-as-GEMM over channels-last activations)
// and fused epilogues (bias, activation, GLU, residual, strided row scatter for transposed convs).
//
// Why fp32 CUDA cores here: the parity bar is bit-exact arg-max tokens against the reference's fp32
// CPU path (BASELINE.json north_star); every GEMM on the path feeds an arg-max within a few layers.
// This kernel is the exact-precision baseline; the wgmma path (kernels_umma2.cu) takes the large-M GEMMs.
#include <algorithm>

#include "common.cuh"
#include "kernels.h"

namespace ss {

namespace {

constexpr int BK = 16;
constexpr int NT = 256;

template <bool CONV>
__device__ __forceinline__ float4 load_a4(const ConvA& a, int m, int kk, int M, int K) {
  float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
  if (m >= M || kk >= K) return v;
  const float* p;
  if (CONV) {
    int b = m / a.L_rows;
    int t = m - b * a.L_rows + a.t_offset;
    int tap = kk / a.C_in;
    int ci = kk - tap * a.C_in;
    int center = t * a.stride;
    int pos = center + tap * a.dil - a.pad_left;
    if (pos < 0 || pos >= a.L_in) return v;
    if (a.chunk > 0 && pos >= (center / a.chunk + 1) * a.chunk) return v;
    if (a.lengths != nullptr && pos >= a.lengths[b]) return v;
    int xr = a.x_rows > 0 ? a.x_rows : a.L_in;
    int pr = pos - a.x_row0;
    if (pr < 0 || pr >= xr) return v;
    p = a.x + ((int64_t)b * xr + pr) * a.ldx + ci;
  } else {
    p = a.x + (int64_t)m * a.ldx + kk;
  }
  v = *reinterpret_cast<const float4*>(p);
  if (a.pre_lrelu != 1.0f) {
    v.x = v.x > 0.f ? v.x : v.x * a.pre_lrelu;
    v.y = v.y > 0.f ? v.y : v.y * a.pre_lrelu;
    v.z = v.z > 0.f ? v.z : v.z * a.pre_lrelu;
    v.w = v.w > 0.f ? v.w : v.w * a.pre_lrelu;
  }
  return v;
}

__device__ __forceinline__ float apply_act(float x, int act) {
  switch (act) {
    case ACT_RELU: return x > 0.f ? x : 0.f;
    case ACT_SILU: return x / (1.0f + expf(-x));
    case ACT_TANH: return tanhf(x);
    case ACT_GELU: return 0.5f * x * (1.0f + erff(x * 0.70710678118654752f));
    default: return x;
  }
}

// gridDim.z > 1: split-K.  Slice z accumulates k-tiles [z*tiles_per_split, (z+1)*tiles_per_split) and stores the raw
// partial sums to ws[z][M][N]; splitk_epilogue_kernel then reduces the slices in a fixed order and applies the epilogue.
// The plain 128 x 16 tile is picked for M >= 128 x #SMs rows: it is held to 64 registers (4 CTAs per SM), which ptxas does not
// choose for it unasked.
template <int BM, int BN, bool CONV>
__global__ void __launch_bounds__(NT, (BM == 128 && BN == 16 && !CONV) ? 4 : 0) gemm_kernel(ConvA a, const float* __restrict__ W, int M, int N, int K, Epilogue ep,
                                                  int tiles_per_split, float* __restrict__ ws) {
  pdl_trigger();
  pdl_wait();
  constexpr int TM = BM / 16;
  constexpr int TN = BN / 16;
  constexpr int A_F4 = BM * BK / 4;  // float4 loads per A tile
  constexpr int B_F4 = BN * BK / 4;
  constexpr int A_PER = (A_F4 + NT - 1) / NT;
  constexpr int B_PER = (B_F4 + NT - 1) / NT;
  __shared__ __align__(16) float As[2][BK][BM + 4];
  __shared__ __align__(16) float Bs[2][BK][BN + 4];

  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;
  const int m0 = blockIdx.y * BM, n0 = blockIdx.x * BN;

  float acc[TM][TN];
#pragma unroll
  for (int i = 0; i < TM; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

  // Global -> register -> shared staging with a register prefetch distance of PF k-tiles: the loads of tile kt + PF are in
  // flight while tile kt is computed, so one DRAM / L2 round trip (~1 us) is covered by PF iterations of FMAs even at one
  // CTA per SM (the streaming vocoder / decoder GEMMs launch 100-300 CTAs).  The im2col predicates and the pre-activation
  // stay on the register path (cp.async could not apply them).
  constexpr int PF = 3;
  float4 ra[PF][A_PER], rb[PF][B_PER];
  auto gload = [&](int k0, float4* qa, float4* qb) {
#pragma unroll
    for (int i = 0; i < A_PER; ++i) {
      int idx = tid + i * NT;
      if (idx < A_F4) qa[i] = load_a4<CONV>(a, m0 + (idx >> 2), k0 + ((idx & 3) << 2), M, K);
    }
#pragma unroll
    for (int i = 0; i < B_PER; ++i) {
      int idx = tid + i * NT;
      if (idx < B_F4) {
        int n = n0 + (idx >> 2), kk = k0 + ((idx & 3) << 2);
        qb[i] = (n < N && kk < K) ? *reinterpret_cast<const float4*>(W + (int64_t)n * K + kk) : make_float4(0.f, 0.f, 0.f, 0.f);
      }
    }
  };
  auto sstore = [&](int buf, const float4* qa, const float4* qb) {
#pragma unroll
    for (int i = 0; i < A_PER; ++i) {
      int idx = tid + i * NT;
      if (idx < A_F4) {
        int r = idx >> 2, kq = (idx & 3) << 2;
        As[buf][kq + 0][r] = qa[i].x;
        As[buf][kq + 1][r] = qa[i].y;
        As[buf][kq + 2][r] = qa[i].z;
        As[buf][kq + 3][r] = qa[i].w;
      }
    }
#pragma unroll
    for (int i = 0; i < B_PER; ++i) {
      int idx = tid + i * NT;
      if (idx < B_F4) {
        int r = idx >> 2, kq = (idx & 3) << 2;
        Bs[buf][kq + 0][r] = qb[i].x;
        Bs[buf][kq + 1][r] = qb[i].y;
        Bs[buf][kq + 2][r] = qb[i].z;
        Bs[buf][kq + 3][r] = qb[i].w;
      }
    }
  };

  const int nk_all = (K + BK - 1) / BK;
  const int kt0 = blockIdx.z * tiles_per_split;
  const int nk = min(nk_all, kt0 + tiles_per_split) - kt0;
#pragma unroll
  for (int d = 0; d < PF; ++d)
    if (d < nk) gload((kt0 + d) * BK, ra[d], rb[d]);
  // iteration kt: registers of tile kt -> smem[kt & 1]; barrier; refill that register set with tile kt + PF; compute.
  // (a warp that runs ahead stores tile kt + 1 into the other buffer, and reaches tile kt + 2's store only after the
  // barrier of iteration kt + 1, i.e. after every warp has finished computing on smem[kt & 1])
  for (int ktb = 0; ktb < nk; ktb += PF) {
#pragma unroll
    for (int d = 0; d < PF; ++d) {
      const int kt = ktb + d;
      if (kt < nk) {
        const int buf = kt & 1;
        sstore(buf, ra[d], rb[d]);
        __syncthreads();
        if (kt + PF < nk) gload((kt0 + kt + PF) * BK, ra[d], rb[d]);
#pragma unroll
        for (int k = 0; k < BK; ++k) {
          float av[TM], bv[TN];
#pragma unroll
          for (int i = 0; i < TM; ++i) av[i] = As[buf][k][ty * TM + i];
#pragma unroll
          for (int j = 0; j < TN; ++j) bv[j] = Bs[buf][k][tx * TN + j];
#pragma unroll
          for (int i = 0; i < TM; ++i)
#pragma unroll
            for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
        }
      }
    }
  }

  if (ws != nullptr) {  // split-K: raw partial sums
    float* wz = ws + (int64_t)blockIdx.z * M * N;
#pragma unroll
    for (int i = 0; i < TM; ++i) {
      int m = m0 + ty * TM + i;
      if (m >= M) continue;
#pragma unroll
      for (int j = 0; j < TN; ++j) {
        int n = n0 + tx * TN + j;
        if (n < N) wz[(int64_t)m * N + n] = acc[i][j];
      }
    }
    return;
  }
  // ---- epilogue
#pragma unroll
  for (int i = 0; i < TM; ++i) {
    int m = m0 + ty * TM + i;
    if (m >= M) continue;
    int64_t orow = m;
    if (ep.out_L > 0) {
      int b = m / a.L_rows;
      int t = m - b * a.L_rows;
      orow = (int64_t)b * ep.out_L + (int64_t)t * ep.out_row_stride + ep.out_row_offset;
    }
    float* orow_p = ep.out + orow * ep.ldo;
    const float* rrow_p = ep.residual ? ep.residual + orow * ep.ldo : nullptr;
    if (ep.glu) {
      if (TN >= 2) {
#pragma unroll
        for (int j = 0; j + 1 < TN; j += 2) {
          int n = n0 + tx * TN + j;
          if (n >= N) continue;
          float av_ = acc[i][j] + (ep.bias ? ep.bias[n] : 0.f);
          float gv = acc[i][j + 1] + (ep.bias ? ep.bias[n + 1] : 0.f);
          float y = ep.alpha * (av_ * (1.0f / (1.0f + expf(-gv))));
          int oc = n >> 1;
          if (rrow_p) y += ep.res_scale * rrow_p[oc];
          if (ep.accumulate) y += orow_p[oc];
          orow_p[oc] = y;
        }
      }
    } else {
#pragma unroll
      for (int j = 0; j < TN; ++j) {
        int n = n0 + tx * TN + j;
        if (n >= N) continue;
        float y = acc[i][j] + (ep.bias ? ep.bias[n] : 0.f);
        y = ep.alpha * apply_act(y, ep.act);
        if (rrow_p) y += ep.res_scale * rrow_p[n];
        if (ep.accumulate) y += orow_p[n];
        orow_p[n] = y;
      }
    }
  }
}

__global__ void splitk_epilogue_kernel(const float* __restrict__ ws, int splits, int M, int N, int L_rows, Epilogue ep) {
  pdl_trigger();
  pdl_wait();
  const int ncols = ep.glu ? N / 2 : N;
  int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= M * ncols) return;
  int m = idx / ncols, oc = idx - m * ncols;
  int64_t orow = m;
  if (ep.out_L > 0) {
    int b = m / L_rows;
    int t = m - b * L_rows;
    orow = (int64_t)b * ep.out_L + (int64_t)t * ep.out_row_stride + ep.out_row_offset;
  }
  float y;
  if (ep.glu) {
    int n = 2 * oc;
    float av_ = 0.f, gv = 0.f;
    for (int z = 0; z < splits; ++z) {
      const float* p = ws + ((int64_t)z * M + m) * N + n;
      av_ += p[0];
      gv += p[1];
    }
    if (ep.bias) {
      av_ += ep.bias[n];
      gv += ep.bias[n + 1];
    }
    y = ep.alpha * (av_ * (1.0f / (1.0f + expf(-gv))));
  } else {
    float acc = 0.f;
    for (int z = 0; z < splits; ++z) acc += ws[((int64_t)z * M + m) * N + oc];
    if (ep.bias) acc += ep.bias[oc];
    y = ep.alpha * apply_act(acc, ep.act);
  }
  float* op = ep.out + orow * ep.ldo + oc;
  if (ep.residual) y += ep.res_scale * ep.residual[orow * ep.ldo + oc];
  if (ep.accumulate) y += *op;
  *op = y;
}

constexpr size_t SPLITK_WS_BYTES = 32u << 20;

}  // namespace

float* splitk_workspace(float** splitk, size_t bytes) {
  if (!splitk || bytes > SPLITK_WS_BYTES) return nullptr;
  if (!*splitk && cudaMalloc((void**)splitk, SPLITK_WS_BYTES) != cudaSuccess) {
    *splitk = nullptr;
    cudaGetLastError();
  }
  return *splitk;
}

size_t splitk_workspace_bytes() { return SPLITK_WS_BYTES; }

void splitk_epilogue(const float* ws, int splits, int M, int N, int L_rows, const Epilogue& ep, cudaStream_t st) {
  ++g_launches;
  int total = M * (ep.glu ? N / 2 : N);
  launch_pdl(splitk_epilogue_kernel, dim3((total + 255) / 256), dim3(256), 0, st, ws, splits, M, N, L_rows, ep);
}

namespace {

template <int BM, int BN>
void launch(const ConvA& a, const float* W, int M, int N, int K, const Epilogue& ep, GemmPlan plan, float** splitk, cudaStream_t st) {
  dim3 grid((N + BN - 1) / BN, (M + BM - 1) / BM);
  float* ws = nullptr;
  if (plan.splits > 1) {
    ws = splitk_workspace(splitk, (size_t)plan.splits * M * N * sizeof(float));
    if (!ws) {
      plan.splits = 1;
      plan.tiles_per_split = (K + BK - 1) / BK;
    }
  }
  grid.z = plan.splits;
  if (plan.conv)
    gemm_kernel<BM, BN, true><<<grid, NT, 0, st>>>(a, W, M, N, K, ep, plan.tiles_per_split, ws);  // tile GEMMs never launch early (see launch_pdl)
  else
    gemm_kernel<BM, BN, false><<<grid, NT, 0, st>>>(a, W, M, N, K, ep, plan.tiles_per_split, ws);
  if (plan.splits > 1) {
    ++g_launches;
    int total = M * (ep.glu ? N / 2 : N);
    launch_pdl(splitk_epilogue_kernel, dim3((total + 255) / 256), dim3(256), 0, st, ws, plan.splits, M, N, a.L_rows, ep);
  }
}

}  // namespace

bool gemm_conv_supported(const ConvA& a, const float* W, int N, const Epilogue& ep) {
  if (!a.x || !W || a.C_in < 1 || a.ldx < a.C_in || (a.C_in & 3) || (a.ldx & 3) || a.ksize < 1 || N < 1) return false;
  if ((reinterpret_cast<uintptr_t>(a.x) & 15) || (reinterpret_cast<uintptr_t>(W) & 15)) return false;
  if (ep.ln_gamma || ep.ln_beta || ep.split_n || (ep.glu && (N & 1))) return false;
  return true;
}

GemmPlan gemm_conv_plan(const ConvA& a, int N, const Epilogue& ep, bool have_scratch) {
  const int M = a.B * a.L_rows;
  const int K = a.ksize * a.C_in;
  GemmPlan p;
  p.conv = !(a.ksize == 1 && a.stride == 1 && a.pad_left == 0 && a.chunk == 0 && a.lengths == nullptr && a.L_in == a.L_rows &&
             a.t_offset == 0 && a.x_row0 == 0 && a.x_rows == 0);
  // ---- tile
  auto ctas = [&](int bm, int bn) { return (long)((M + bm - 1) / bm) * ((N + bn - 1) / bn); };
  const long target = std::max(1, current_device_sms());  // one wave of SMs
  const int nk = (K + BK - 1) / BK;
  if (N <= 16 && !ep.glu) {
    p.BN = 16;
    p.BM = ctas(128, 16) >= target ? 128 : 32;
  } else if (N <= 32) {
    p.BN = 32;
    p.BM = ctas(64, 32) >= target ? 64 : 32;
  } else {
    // Prefer the largest tile that still fills the GPU once split-K (slices of >= 8 k-tiles, at most 8 slices) is counted:
    // a long K walked by few small CTAs is latency-bound.
    const long max_splits = std::max(1, std::min(8, nk / 8));
    if (ctas(128, 64) >= 2 * target) p.BM = 128, p.BN = 64;
    else if (ctas(64, 64) * max_splits >= target) p.BM = 64, p.BN = 64;
    else if (ctas(32, 64) * max_splits >= target) p.BM = 32, p.BN = 64;
    else p.BM = 32, p.BN = 32;
  }
  // ---- split-K
  int splits = 1;
  const long tile_ctas = ctas(p.BM, p.BN);
  if (a.k_tiles_per_split > 0) {
    splits = (nk + a.k_tiles_per_split - 1) / a.k_tiles_per_split;
    if ((size_t)splits * M * N * sizeof(float) > SPLITK_WS_BYTES) splits = 1;
  } else if (tile_ctas < target && nk >= 8) {
    splits = (int)std::min<long>((target + tile_ctas - 1) / tile_ctas, nk / 4);  // >= 4 k-tiles (64 columns) per slice
    if ((size_t)splits * M * N * sizeof(float) > SPLITK_WS_BYTES) splits = 1;
  }
  if (!have_scratch) splits = 1;
  p.tiles_per_split = nk;
  if (splits > 1) {
    p.tiles_per_split = (nk + splits - 1) / splits;
    splits = (nk + p.tiles_per_split - 1) / p.tiles_per_split;
  }
  p.splits = splits;
  return p;
}

void gemm_conv(const ConvA& a, const float* W, int N, const Epilogue& ep, float** splitk, cudaStream_t st) {
  ++g_launches;
  const int M = a.B * a.L_rows;
  const int K = a.ksize * a.C_in;
  if (M <= 0 || N <= 0) return;
  const GemmPlan p = gemm_conv_plan(a, N, ep, splitk != nullptr);
  switch (p.BM * 1000 + p.BN) {
    case 128016: launch<128, 16>(a, W, M, N, K, ep, p, splitk, st); break;
    case 32016: launch<32, 16>(a, W, M, N, K, ep, p, splitk, st); break;
    case 64032: launch<64, 32>(a, W, M, N, K, ep, p, splitk, st); break;
    case 128064: launch<128, 64>(a, W, M, N, K, ep, p, splitk, st); break;
    case 64064: launch<64, 64>(a, W, M, N, K, ep, p, splitk, st); break;
    case 32064: launch<32, 64>(a, W, M, N, K, ep, p, splitk, st); break;
    default: launch<32, 32>(a, W, M, N, K, ep, p, splitk, st); break;
  }
}

}  // namespace ss
