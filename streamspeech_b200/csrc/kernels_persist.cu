// Persistent cooperative kernel for one streaming step of the chunk-Conformer encoder stack.
//
// At batch 1 a 320 ms step touches <= 16 active rows and ~11 MB of fp32 weights per layer; run as separate kernels it is
// bounded by kernel boundaries (137 dependent launches), not by HBM or FLOPs.  This kernel keeps
// one CTA per SM resident for ALL layers and replaces the kernel boundaries by grid-wide barriers, 9 per layer:
//   [LN + W1 + SiLU] | [W2 + 0.5 res] | [LN + QKV -> q, K-cache, V-cache] | [rel-pos attention] | [out + res] |
//   [LN + PW1 + GLU -> conv cache, depthwise k31 + BN + SiLU] | [PW2 + res] | [LN + W1 + SiLU] | [W2 + 0.5 res]
// The layer's final LayerNorm is not a phase of its own: the next layer's first phase applies it while staging its input,
// and the first residual add after it applies it to the residual it reads (one explicit LN phase closes the last layer).
//
// GEMM phases (M <= 16 rows): the CTA stages the (layer-normed) activations once in shared memory, each warp owns CPT
// output columns x one K-slice, streams its weight rows with 128-bit non-coherent loads issued BEFORE the staging (so the
// HBM latency overlaps the LayerNorm), reduces the 16 row sums with a halving shuffle tree and a fixed-order K-slice sum.
// Same arithmetic as the per-kernel path of ss_encoder_stream_step, which remains the fallback for shapes this kernel
// does not cover (nA > 16, D != 256, ...).
#include <cooperative_groups.h>

#include "common.cuh"
#include "kernels.h"
#include "kernels_persist.h"

namespace cg = cooperative_groups;

namespace ss {
namespace {

constexpr int PW = 8;          // warps per CTA
constexpr int PT = PW * 32;    // threads per CTA
constexpr int PMR = 16;        // max active rows
constexpr int PHD = 64;        // head dim
constexpr int PD = 256;        // model dim

__device__ __forceinline__ unsigned long long globaltimer_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
  return t;
}

__device__ __forceinline__ float4 ldw(const float* p) {
  float4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p));
  return r;
}

// L2 prefetch of a weight matrix, spread over the whole grid (one 128-byte line per request)
__device__ __forceinline__ void prefetch_l2(const float* p, int n_floats) {
  const int lines = n_floats >> 5;
  for (int i = blockIdx.x * PT + threadIdx.x; i < lines; i += gridDim.x * PT)
    asm volatile("prefetch.global.L2 [%0];" ::"l"(p + (size_t)i * 32));
}

// All GEMM weights of one layer (~10 MB): issued one layer ahead, so the phases of the next layer stream their weights from
// L2 instead of paying an HBM round trip right after every grid barrier.
__device__ __forceinline__ void prefetch_layer(const PersistLayer& L, int D, int FFN) {
  prefetch_l2(L.ffn1_w1, D * FFN);
  prefetch_l2(L.ffn1_w2, D * FFN);
  prefetch_l2(L.wqkv, 3 * D * D);
  prefetch_l2(L.wo, D * D);
  prefetch_l2(L.pw1, 2 * D * D);
  prefetch_l2(L.pw2, D * D);
  prefetch_l2(L.ffn2_w1, D * FFN);
  prefetch_l2(L.ffn2_w2, D * FFN);
}

struct GemmEpi {
  const float* bias = nullptr;
  int act = ACT_NONE;       // ignored when GLU
  float alpha = 1.f;
  float* out = nullptr;     // column block 0
  int ldo = 0;
  bool residual = false;    // out += (in place)
  const float* res_ln_g = nullptr;  // residual read is LN(out) with the stats in Smem::fin_* (deferred final LayerNorm)
  const float* res_ln_b = nullptr;
  int split_n = 0;          // > 0: route column blocks of this width to out / out2 / out3
  float* out2 = nullptr;
  float* out3 = nullptr;
  int ldo2 = 0, ldo3 = 0;
};

struct DwFuse {  // depthwise conv + BN + SiLU on the GLU outputs (conv module), fused into the PW1 phase
  const float* gc;   // conv cache of this layer [Tpos][D] (GLU outputs of all rows so far)
  const float* w;    // [k][D]
  const float* scale;
  const float* shift;
  float* dw;         // [nA][D]
  int a0, T, k, chunk;
};

struct Smem {
  float As[PMR * PD];        // staged (layer-normed) activations, row stride PD
  float part[PW][4][PMR];
  float fin_mean[PMR], fin_rstd[PMR];
  float S[1024];
  float qa[PHD], qb[PHD];
  float pv[PW][PHD];
  float strip[PW][48];
  float wstrip[PW][32];
  float red[PW];
  float hs[PMR][16];          // fused FFN: this CTA's 16 hidden units for the 16 rows
  float rsum[PW][32];         // fused FFN reduce: per-warp partial sums of 32 outputs
  unsigned long long* fine;  // profile mode, CTA 0, layer 1: (tag, clock64) stamps inside the phases
  int nfine;
};

__device__ __forceinline__ void fine_stamp(Smem& sm, int tag) {
  if (threadIdx.x == 0 && sm.fine != nullptr && sm.nfine < 120) {
    sm.fine[2 * sm.nfine] = (unsigned long long)tag;
    sm.fine[2 * sm.nfine + 1] = (unsigned long long)clock64();
    ++sm.nfine;
  }
}

// As[m][:] = LN_b(LN_a(x[m][:])) for m < M (zeros above); LN_a (the previous layer's deferred final LayerNorm) is optional
// and leaves its row statistics in sm.fin_*.  Warp w owns rows w and w + 8; 8 values per lane per row.  No barrier inside.
__device__ __forceinline__ void stage_ln(Smem& sm, const float* x, int M, const float* __restrict__ ga, const float* __restrict__ ba,
                                         const float* __restrict__ gb, const float* __restrict__ bb) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float v[2][8];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int m = warp + h * PW;
#pragma unroll
    for (int i = 0; i < 8; ++i) v[h][i] = m < M ? x[(int64_t)m * PD + lane + (i << 5)] : 0.f;
  }
  float g[8], b[8];
  if (ga != nullptr) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      g[i] = ga[lane + (i << 5)];
      b[i] = ba[lane + (i << 5)];
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int m = warp + h * PW;
      float s = 0.f;
#pragma unroll
      for (int i = 0; i < 8; ++i) s += v[h][i];
      const float mean = warp_sum(s) / (float)PD;
      float q = 0.f;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        float d = v[h][i] - mean;
        q = fmaf(d, d, q);
      }
      const float rstd = 1.0f / sqrtf(warp_sum(q) / (float)PD + 1e-5f);
      if (lane == 0) {
        sm.fin_mean[m] = mean;
        sm.fin_rstd[m] = rstd;
      }
#pragma unroll
      for (int i = 0; i < 8; ++i) v[h][i] = (v[h][i] - mean) * rstd * g[i] + b[i];
    }
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    g[i] = gb[lane + (i << 5)];
    b[i] = bb[lane + (i << 5)];
  }
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int m = warp + h * PW;
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) s += v[h][i];
    const float mean = warp_sum(s) / (float)PD;
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      float d = v[h][i] - mean;
      q = fmaf(d, d, q);
    }
    const float rstd = 1.0f / sqrtf(warp_sum(q) / (float)PD + 1e-5f);
#pragma unroll
    for (int i = 0; i < 8; ++i) sm.As[m * PD + lane + (i << 5)] = m < M ? (v[h][i] - mean) * rstd * g[i] + b[i] : 0.f;
  }
}

// As[m][:] = a[m][:] (K == PD), zeros for m >= M
__device__ __forceinline__ void stage_copy(Smem& sm, const float* a, int M) {
#pragma unroll
  for (int i = 0; i < (PMR * PD / 4) / PT; ++i) {
    const int idx = threadIdx.x + i * PT;  // float4 index
    const int m = idx / (PD / 4);
    float4 val = make_float4(0.f, 0.f, 0.f, 0.f);
    if (m < M) val = *reinterpret_cast<const float4*>(a + (int64_t)idx * 4);
    *reinterpret_cast<float4*>(sm.As + idx * 4) = val;
  }
}

enum { STAGE_LN = 0, STAGE_COPY = 1, STAGE_NONE = 2 };

// out[M][N'] = epi( A[M][K] @ W[N][K]^T ), M <= 16.  All CTAs of the grid take part.  STAGE_LN / STAGE_COPY: K == PD and A
// goes through shared memory (LN: As = LN(LN_pre?(A))); STAGE_NONE: every warp reads its K-slice of A from global memory.
// Activations are written by other CTAs between barriers: they are read with plain (coherent) loads, never through
// __restrict__ / ld.global.nc; only weights take the non-coherent streaming path.
template <int CPT, bool GLU, int KS, int K, int STAGE>
__device__ void phase_gemm(Smem& sm, const float* A, const float* __restrict__ pre_g, const float* __restrict__ pre_b,
                           const float* __restrict__ ln_g, const float* __restrict__ ln_b, const float* __restrict__ W, int M, int N,
                           const GemmEpi& ep, const DwFuse* dwf, int tag) {
  constexpr int KSLICE = K / KS;
  constexpr int NIT = KSLICE / 128;
  static_assert(KSLICE % 128 == 0, "K slice must be a multiple of 128");
  static_assert(STAGE == STAGE_NONE || K == PD, "staged GEMMs have K == PD");
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  constexpr int TPC = PW / KS;
  const int slice = warp % KS, tslot = warp / KS;
  const int ntasks = N / CPT;
  const int k_lo = slice * KSLICE;
  const int m = lane >> 1;  // row owned in the epilogue (even lanes)
  const bool owner = (lane & 1) == 0;
  fine_stamp(sm, tag);
  bool first = true;
  for (int tbase = blockIdx.x * TPC; tbase < ntasks; tbase += gridDim.x * TPC) {
    const int task = tbase + tslot;
    const bool active = task < ntasks;
    const int n0 = task * CPT;
    // ---- issue the weight loads of the whole task first: their HBM latency overlaps the staging below
    float4 wv[NIT][CPT];
#pragma unroll
    for (int it = 0; it < NIT; ++it)
#pragma unroll
      for (int c = 0; c < CPT; ++c)
        wv[it][c] = active ? ldw(W + (int64_t)(n0 + c) * K + k_lo + it * 128 + lane * 4) : make_float4(0.f, 0.f, 0.f, 0.f);
    // epilogue operands that do not depend on the GEMM: bias, residual, depthwise taps / cached rows
    float bias_v[CPT], res_v[CPT];
    float dw_old = 0.f, dw_tap = 0.f;
    const bool epi_lane = active && slice == 0 && owner && m < M;
#pragma unroll
    for (int c = 0; c < CPT; ++c) {
      bias_v[c] = (ep.bias != nullptr && active) ? ep.bias[n0 + c] : 0.f;
      res_v[c] = 0.f;
    }
    if (!GLU && ep.residual && epi_lane) {
#pragma unroll
      for (int c = 0; c < CPT; ++c) res_v[c] = ep.out[(int64_t)m * ep.ldo + n0 + c];
    }
    if (GLU && dwf != nullptr && active && slice == 0) {
      const int half = (dwf->k - 1) >> 1, oc = n0 >> 1;
      const int p = dwf->a0 - half + lane;
      if (lane < half && p >= 0) dw_old = dwf->gc[(int64_t)p * PD + oc];
      if (lane < dwf->k) dw_tap = dwf->w[lane * PD + oc];
    }
    if (first) {
      if (STAGE == STAGE_LN) stage_ln(sm, A, M, pre_g, pre_b, ln_g, ln_b);
      if (STAGE == STAGE_COPY) stage_copy(sm, A, M);
      if (STAGE != STAGE_NONE) __syncthreads();
      first = false;
      fine_stamp(sm, tag + 1);
    }
    float acc[CPT][PMR];
#pragma unroll
    for (int c = 0; c < CPT; ++c)
#pragma unroll
      for (int r = 0; r < PMR; ++r) acc[c][r] = 0.f;
#pragma unroll
    for (int it = 0; it < NIT; ++it) {
      const int k = k_lo + it * 128 + lane * 4;
#pragma unroll
      for (int r = 0; r < PMR; ++r) {
        float4 x;
        if (STAGE == STAGE_NONE) {
          x = (r < M) ? *reinterpret_cast<const float4*>(A + (int64_t)r * K + k) : make_float4(0.f, 0.f, 0.f, 0.f);
        } else {
          x = *reinterpret_cast<const float4*>(sm.As + r * PD + k);
        }
#pragma unroll
        for (int c = 0; c < CPT; ++c) {
          acc[c][r] = fmaf(x.x, wv[it][c].x, acc[c][r]);
          acc[c][r] = fmaf(x.y, wv[it][c].y, acc[c][r]);
          acc[c][r] = fmaf(x.z, wv[it][c].z, acc[c][r]);
          acc[c][r] = fmaf(x.w, wv[it][c].w, acc[c][r]);
        }
      }
    }
    fine_stamp(sm, tag + 2);
    // 16 row sums per column across the warp: recursive halving (16 shuffles per column instead of 16 x 5); even lane
    // 2m ends up with the sum of row m.  Fixed order -> deterministic.
    float mine[CPT];
#pragma unroll
    for (int c = 0; c < CPT; ++c) {
      const bool b4 = lane & 16, b3 = lane & 8, b2 = lane & 4, b1 = lane & 2;
      float w8[8], w4[4], w2[2];
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        float send = b4 ? acc[c][i] : acc[c][i + 8];
        float keep = b4 ? acc[c][i + 8] : acc[c][i];
        w8[i] = keep + __shfl_xor_sync(0xffffffffu, send, 16);
      }
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        float send = b3 ? w8[i] : w8[i + 4];
        float keep = b3 ? w8[i + 4] : w8[i];
        w4[i] = keep + __shfl_xor_sync(0xffffffffu, send, 8);
      }
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        float send = b2 ? w4[i] : w4[i + 2];
        float keep = b2 ? w4[i + 2] : w4[i];
        w2[i] = keep + __shfl_xor_sync(0xffffffffu, send, 4);
      }
      float send = b1 ? w2[0] : w2[1];
      float keep = b1 ? w2[1] : w2[0];
      float w1 = keep + __shfl_xor_sync(0xffffffffu, send, 2);
      mine[c] = w1 + __shfl_xor_sync(0xffffffffu, w1, 1);
    }
    if (KS > 1) {
      if (owner) {
#pragma unroll
        for (int c = 0; c < CPT; ++c) sm.part[warp][c][m] = mine[c];
      }
      __syncthreads();
      if (slice == 0 && owner) {
#pragma unroll
        for (int c = 0; c < CPT; ++c) {
          float t = sm.part[warp][c][m];
#pragma unroll
          for (int s = 1; s < KS; ++s) t += sm.part[warp + s][c][m];
          mine[c] = t;
        }
      }
    }
    fine_stamp(sm, tag + 3);
    if (GLU) {
      float y = 0.f;
      const int oc = n0 >> 1;
      if (epi_lane) {
        float av = mine[0] + bias_v[0];
        float gv = mine[CPT - 1] + bias_v[CPT - 1];
        y = ep.alpha * (av * (1.0f / (1.0f + expf(-gv))));
        ep.out[(int64_t)m * ep.ldo + oc] = y;
      }
      if (dwf != nullptr && active && slice == 0) {
        // depthwise conv over time for channel oc: strip = [half cached rows | the M new rows | zeros]
        const int half = (dwf->k - 1) >> 1;
        float* strip = sm.strip[warp];
        float* wst = sm.wstrip[warp];
        if (lane < half) strip[lane] = dw_old;
        if (half + M + lane < 48) strip[half + M + lane] = 0.f;  // (rows past the last new one are masked by `lim` anyway)
        wst[lane] = dw_tap;
        __syncwarp();
        if (epi_lane) strip[half + m] = y;
        __syncwarp();
        if (lane < M) {
          const int t = dwf->a0 + lane;
          const int lim = dwf->chunk > 0 ? min(dwf->T, (t / dwf->chunk + 1) * dwf->chunk) : dwf->T;
          float a = 0.f;
          for (int j = 0; j < dwf->k; ++j) {
            const int p = t - half + j;
            if (p >= 0 && p < lim) a = fmaf(wst[j], strip[lane + j], a);
          }
          float v = a * dwf->scale[oc] + dwf->shift[oc];
          dwf->dw[(int64_t)lane * PD + oc] = v / (1.0f + expf(-v));
        }
        __syncwarp();
      }
    } else if (epi_lane) {
#pragma unroll
      for (int c = 0; c < CPT; ++c) {
        float v = mine[c] + bias_v[c];
        if (ep.act == ACT_SILU) v = v / (1.0f + expf(-v));
        float y = ep.alpha * v;
        int oc = n0 + c;
        float* obase = ep.out;
        int ld = ep.ldo;
        if (ep.split_n > 0) {
          int p = oc / ep.split_n;
          oc -= p * ep.split_n;
          if (p == 1) { obase = ep.out2; ld = ep.ldo2; }
          else if (p == 2) { obase = ep.out3; ld = ep.ldo3; }
        }
        if (ep.residual) {
          float r = res_v[c];
          if (ep.res_ln_g != nullptr) r = (r - sm.fin_mean[m]) * sm.fin_rstd[m] * ep.res_ln_g[oc] + ep.res_ln_b[oc];
          y += r;
        }
        obase[(int64_t)m * ld + oc] = y;
      }
    }
    if (KS > 1) __syncthreads();
    fine_stamp(sm, tag + 4);
  }
  if (STAGE == STAGE_LN && first && pre_g != nullptr) {  // CTA without a task: the next phase still needs sm.fin_*
    stage_ln(sm, A, M, pre_g, pre_b, ln_g, ln_b);
    __syncthreads();
  }
}

// ---- fused FFN (x += alpha * W2 act(W1 LN(x))) in TWO light phases instead of a W1 phase and a W2 phase that makes every CTA
// read the whole 16 x 2048 hidden from L2 (16 MB per phase):
//   phase A : CTA j < FFN/16 owns hidden units [16j, 16j+16): hid = SiLU(LN(x) W1[16 rows]^T + b1) stays in shared memory, then the
//             rank-16 update  P[j][m][n] = sum_u hid[m][u] * W2T[16j+u][n]  (W2T = W2 transposed, one coalesced 1 KB row per unit)
//             goes to a global scratch (16 KB per CTA);
//   phase A': CTA c owns 32 consecutive outputs (m, n): sums the FFN/16 partials in a fixed order (deterministic), adds bias,
//             alpha and the residual.
constexpr int FFN_UNITS = 16;   // hidden units per CTA

template <int FFN>
__device__ void phase_ffn_partial(Smem& sm, const float* x, const float* __restrict__ pre_g, const float* __restrict__ pre_b,
                                  const float* __restrict__ ln_g, const float* __restrict__ ln_b, const float* __restrict__ W1,
                                  const float* __restrict__ b1, const float* __restrict__ W2T, float* P, int M, int tag) {
  constexpr int NJ = FFN / FFN_UNITS;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int j = blockIdx.x;
  fine_stamp(sm, tag);
  if (j >= NJ) return;  // (the reduce phase reads sm.fin_* only in CTAs < 8 M <= NJ, which all stage below)
  // weight loads first: 2 hidden units per warp (2 x 2 float4 per lane), 16 W2T values per thread
  const int u0 = warp * 2;
  float4 wv[2][2];
#pragma unroll
  for (int c = 0; c < 2; ++c)
#pragma unroll
    for (int it = 0; it < 2; ++it) wv[c][it] = ldw(W1 + (int64_t)(j * FFN_UNITS + u0 + c) * PD + it * 128 + lane * 4);
  float w2[FFN_UNITS];
#pragma unroll
  for (int u = 0; u < FFN_UNITS; ++u) w2[u] = __ldg(W2T + (int64_t)(j * FFN_UNITS + u) * PD + threadIdx.x);
  const float bias0 = b1[j * FFN_UNITS + u0], bias1 = b1[j * FFN_UNITS + u0 + 1];
  stage_ln(sm, x, M, pre_g, pre_b, ln_g, ln_b);
  __syncthreads();
  fine_stamp(sm, tag + 1);
  float acc[2][PMR];
#pragma unroll
  for (int c = 0; c < 2; ++c)
#pragma unroll
    for (int r = 0; r < PMR; ++r) acc[c][r] = 0.f;
#pragma unroll
  for (int it = 0; it < 2; ++it) {
    const int k = it * 128 + lane * 4;
#pragma unroll
    for (int r = 0; r < PMR; ++r) {
      const float4 xv = *reinterpret_cast<const float4*>(sm.As + r * PD + k);
#pragma unroll
      for (int c = 0; c < 2; ++c) {
        acc[c][r] = fmaf(xv.x, wv[c][it].x, acc[c][r]);
        acc[c][r] = fmaf(xv.y, wv[c][it].y, acc[c][r]);
        acc[c][r] = fmaf(xv.z, wv[c][it].z, acc[c][r]);
        acc[c][r] = fmaf(xv.w, wv[c][it].w, acc[c][r]);
      }
    }
  }
  // 16 row sums per unit across the warp (same halving tree as phase_gemm): even lane 2m ends with row m
#pragma unroll
  for (int c = 0; c < 2; ++c) {
    const bool b4 = lane & 16, b3 = lane & 8, b2 = lane & 4, b1_ = lane & 2;
    float w8[8], w4[4], w2r[2];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      float send = b4 ? acc[c][i] : acc[c][i + 8];
      float keep = b4 ? acc[c][i + 8] : acc[c][i];
      w8[i] = keep + __shfl_xor_sync(0xffffffffu, send, 16);
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      float send = b3 ? w8[i] : w8[i + 4];
      float keep = b3 ? w8[i + 4] : w8[i];
      w4[i] = keep + __shfl_xor_sync(0xffffffffu, send, 8);
    }
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      float send = b2 ? w4[i] : w4[i + 2];
      float keep = b2 ? w4[i + 2] : w4[i];
      w2r[i] = keep + __shfl_xor_sync(0xffffffffu, send, 4);
    }
    float send = b1_ ? w2r[0] : w2r[1];
    float keep = b1_ ? w2r[1] : w2r[0];
    float w1 = keep + __shfl_xor_sync(0xffffffffu, send, 2);
    float v = w1 + __shfl_xor_sync(0xffffffffu, w1, 1);
    if ((lane & 1) == 0) {
      v += c ? bias1 : bias0;
      sm.hs[lane >> 1][u0 + c] = v / (1.0f + expf(-v));  // SiLU
    }
  }
  __syncthreads();
  fine_stamp(sm, tag + 2);
  // rank-16 update: thread n owns output column n for all rows
  float* Pj = P + (int64_t)j * PMR * PD;
  for (int m = 0; m < M; ++m) {
    float a = 0.f;
#pragma unroll
    for (int u4 = 0; u4 < FFN_UNITS / 4; ++u4) {
      const float4 hv = *reinterpret_cast<const float4*>(&sm.hs[m][u4 * 4]);
      a = fmaf(hv.x, w2[u4 * 4], a);
      a = fmaf(hv.y, w2[u4 * 4 + 1], a);
      a = fmaf(hv.z, w2[u4 * 4 + 2], a);
      a = fmaf(hv.w, w2[u4 * 4 + 3], a);
    }
    Pj[m * PD + threadIdx.x] = a;
  }
  fine_stamp(sm, tag + 3);
}

// x[m][n] = res(x[m][n]) + alpha * (sum_j P[j][m][n] + b2[n]); res = LN_pre when pre_g != nullptr (row statistics in sm.fin_*
// from this CTA's own staging in phase A).  CTA c owns the 32 consecutive outputs starting at 32 c.
template <int FFN>
__device__ void phase_ffn_reduce(Smem& sm, float* x, const float* P, const float* __restrict__ b2, float alpha,
                                 const float* __restrict__ pre_g, const float* __restrict__ pre_b, int M, int tag) {
  constexpr int NJ = FFN / FFN_UNITS;
  static_assert(NJ % PW == 0, "partials split evenly over the warps");
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  fine_stamp(sm, tag);
  const int o = blockIdx.x * 32 + lane;
  if (blockIdx.x * 32 >= M * PD) return;   // (CTA-uniform)
  float s = 0.f;
  float v[NJ / PW];
#pragma unroll
  for (int i = 0; i < NJ / PW; ++i) v[i] = P[(int64_t)(warp + i * PW) * PMR * PD + o];  // plain loads: written by other CTAs before the barrier
#pragma unroll
  for (int i = 0; i < NJ / PW; ++i) s += v[i];
  sm.rsum[warp][lane] = s;
  __syncthreads();
  if (warp == 0) {
    float t = sm.rsum[0][lane];
#pragma unroll
    for (int w = 1; w < PW; ++w) t += sm.rsum[w][lane];
    const int m = o / PD, n = o - m * PD;
    float r = x[o];
    if (pre_g != nullptr) r = (r - sm.fin_mean[m]) * sm.fin_rstd[m] * pre_g[n] + pre_b[n];
    x[o] = alpha * (t + b2[n]) + r;
  }
  fine_stamp(sm, tag + 1);
}

// rel-pos attention for the active rows: one CTA per (row, head) task
__device__ void phase_attention(Smem& sm, const float* q, const float* kc, const float* vc, const float* __restrict__ pos, int Tpos,
                                const float* __restrict__ bias_u, const float* __restrict__ bias_v, float* out, int nA, int a0, int T, int D,
                                int H, int chunk) {
  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  for (int task = blockIdx.x; task < nA * H; task += gridDim.x) {
    const int r = task / H, h = task - r * H;
    const int i = a0 + r;
    const int lim = chunk > 0 ? min((i / chunk + 1) * chunk, T) : T;
    const int n = max(1, lim);
    __syncthreads();  // smem reuse across tasks
    if (tid < PHD) {
      float val = q[(int64_t)r * D + h * PHD + tid];
      sm.qa[tid] = val + bias_u[h * PHD + tid];
      sm.qb[tid] = val + bias_v[h * PHD + tid];
    }
    __syncthreads();
    const float* kb = kc + h * PHD;
    const float* vb = vc + h * PHD;
    const float* pb = pos + h * PHD;
    float mx = -INFINITY;
    for (int j = tid; j < n; j += PT) {
      const float* kr = kb + (int64_t)j * D;
      const float* pr = pb + (int64_t)(i - j + Tpos - 1) * D;
      float4 kk[PHD / 4], pp[PHD / 4];
#pragma unroll
      for (int d = 0; d < PHD / 4; ++d) {
        kk[d] = *reinterpret_cast<const float4*>(kr + 4 * d);
        pp[d] = *reinterpret_cast<const float4*>(pr + 4 * d);
      }
      float ac = 0.f, bd = 0.f;
#pragma unroll
      for (int d = 0; d < PHD / 4; ++d) {
        ac = fmaf(sm.qa[4 * d], kk[d].x, ac); ac = fmaf(sm.qa[4 * d + 1], kk[d].y, ac);
        ac = fmaf(sm.qa[4 * d + 2], kk[d].z, ac); ac = fmaf(sm.qa[4 * d + 3], kk[d].w, ac);
        bd = fmaf(sm.qb[4 * d], pp[d].x, bd); bd = fmaf(sm.qb[4 * d + 1], pp[d].y, bd);
        bd = fmaf(sm.qb[4 * d + 2], pp[d].z, bd); bd = fmaf(sm.qb[4 * d + 3], pp[d].w, bd);
      }
      float s = (ac + bd) * 0.125f;
      sm.S[j] = s;
      mx = fmaxf(mx, s);
    }
    mx = warp_max(mx);
    if (lane == 0) sm.red[w] = mx;
    __syncthreads();
    mx = sm.red[0];
#pragma unroll
    for (int x = 1; x < PW; ++x) mx = fmaxf(mx, sm.red[x]);
    __syncthreads();
    float sum = 0.f;
    for (int j = tid; j < n; j += PT) {
      float e = expf(sm.S[j] - mx);
      sm.S[j] = e;
      sum += e;
    }
    sum = warp_sum(sum);
    if (lane == 0) sm.red[w] = sum;
    __syncthreads();
    sum = sm.red[0];
#pragma unroll
    for (int x = 1; x < PW; ++x) sum += sm.red[x];
    // out[d] = sum_j p_j V[j][d]: warp w takes keys j = w (mod 8), 8 keys in flight; lane owns dims 2*lane, 2*lane+1
    float a0_ = 0.f, a1_ = 0.f;
    for (int j0 = w; j0 < n; j0 += PW * 16) {  // 16 keys (independent 8-byte loads) in flight per lane: 2 rounds at T = 250
      float2 vv[16];
      float p[16];
#pragma unroll
      for (int u = 0; u < 16; ++u) {
        const int j = j0 + u * PW;
        const bool ok = j < n;
        vv[u] = ok ? *reinterpret_cast<const float2*>(vb + (int64_t)j * D + 2 * lane) : make_float2(0.f, 0.f);
        p[u] = ok ? sm.S[j] : 0.f;
      }
#pragma unroll
      for (int u = 0; u < 16; ++u) {
        a0_ = fmaf(p[u], vv[u].x, a0_);
        a1_ = fmaf(p[u], vv[u].y, a1_);
      }
    }
    sm.pv[w][2 * lane] = a0_;
    sm.pv[w][2 * lane + 1] = a1_;
    __syncthreads();
    if (tid < PHD) {
      float t = 0.f;
#pragma unroll
      for (int x = 0; x < PW; ++x) t += sm.pv[x][tid];
      out[(int64_t)r * D + h * PHD + tid] = t / sum;
    }
  }
}

__device__ void phase_layer_norm(float* x, const float* __restrict__ g, const float* __restrict__ b, int M, int D) {
  const int lane = threadIdx.x & 31;
  const int gw = blockIdx.x * PW + (threadIdx.x >> 5);
  if (gw >= M) return;
  float* xr = x + (int64_t)gw * D;
  float v[8];  // D == 256
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    v[i] = xr[lane + (i << 5)];
    s += v[i];
  }
  float mean = warp_sum(s) / (float)D;
  float ss_ = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    float d = v[i] - mean;
    ss_ = fmaf(d, d, ss_);
  }
  float rstd = 1.0f / sqrtf(warp_sum(ss_) / (float)D + 1e-5f);
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    int c = lane + (i << 5);
    xr[c] = (v[i] - mean) * rstd * g[c] + b[c];
  }
}

template <int FFN>
__global__ void __launch_bounds__(PT, 1) encoder_layers_persistent_kernel(const PersistLayer* __restrict__ layers, int n_layers, float* x,
                                                                          float* hid, float* qb, float* att, float* dw, float* kc_all,
                                                                          float* vc_all, float* gc_all, int nA, int a0, int T, int H, int Tpos,
                                                                          int chunk, int conv_chunk, int dw_k, unsigned long long* ts,
                                                                          unsigned* bar_ctr, unsigned bar_target, int prefetch,
                                                                          float* ffn_scratch) {
  constexpr int D = PD;
  cg::grid_group grid = cg::this_grid();
  __shared__ __align__(16) Smem sm;
  int nts = 0;
  const bool stamp = ts != nullptr && blockIdx.x == 0 && threadIdx.x == 0;
  if (threadIdx.x == 0) {
    sm.fine = nullptr;
    sm.nfine = 0;
  }
#define GRID_SYNC()                                       \
  if (bar_ctr != nullptr) grid_barrier(bar_ctr, bar_target); \
  else grid.sync();
  if (ts != nullptr) {  // profile mode: two back-to-back barriers first (pure barrier cost)
    if (stamp) ts[nts++] = globaltimer_ns();
    GRID_SYNC();
    if (stamp) ts[nts++] = globaltimer_ns();
    GRID_SYNC();
    if (stamp) ts[nts++] = globaltimer_ns();
  }
  // profile mode: every CTA also records when it ARRIVES at each barrier of layer 1 (ts[512 + cta * 16 + phase])
#define PHASE_END(tag)                                                                                          \
  fine_stamp(sm, tag);                                                                                          \
  if (ts != nullptr && li == 1 && threadIdx.x == 0) ts[512 + blockIdx.x * 16 + (tag) / 10 - 1] = globaltimer_ns(); \
  GRID_SYNC();                                                                                                  \
  if (stamp) ts[nts++] = globaltimer_ns();
  for (int li = 0; li < n_layers; ++li) {
    if (threadIdx.x == 0) sm.fine = (ts != nullptr && blockIdx.x == 0 && li == 1) ? ts + 256 : nullptr;
    const PersistLayer L = layers[li];
    if (prefetch) {
      if (li == 0 && prefetch > 1) prefetch_layer(L, D, FFN);
      if (li + 1 < n_layers) prefetch_layer(layers[li + 1], D, FFN);
    }
    // the previous layer's final LayerNorm is still pending on x (applied on the fly in the first two phases)
    const float* pre_g = li > 0 ? layers[li - 1].fin_g : nullptr;
    const float* pre_b = li > 0 ? layers[li - 1].fin_b : nullptr;
    float* kc = kc_all + (size_t)li * Tpos * D;
    float* vc = vc_all + (size_t)li * Tpos * D;
    float* gc = gc_all + (size_t)li * Tpos * D;
    GemmEpi e;
    // x = x + 0.5 * W2(SiLU(W1 LN(x)))
    if (ffn_scratch != nullptr) {
      phase_ffn_partial<FFN>(sm, x, pre_g, pre_b, L.ffn1_g, L.ffn1_b, L.ffn1_w1, L.ffn1_b1, L.ffn1_w2t, ffn_scratch, nA, 10);
      PHASE_END(15);
      phase_ffn_reduce<FFN>(sm, x, ffn_scratch, L.ffn1_b2, 0.5f, pre_g, pre_b, nA, 20);
      PHASE_END(25);
    } else {
    e = GemmEpi(); e.bias = L.ffn1_b1; e.act = ACT_SILU; e.out = hid; e.ldo = FFN;
    phase_gemm<4, false, 2, D, STAGE_LN>(sm, x, pre_g, pre_b, L.ffn1_g, L.ffn1_b, L.ffn1_w1, nA, FFN, e, nullptr, 10);
    PHASE_END(15);
    e = GemmEpi(); e.bias = L.ffn1_b2; e.alpha = 0.5f; e.out = x; e.ldo = D; e.residual = true; e.res_ln_g = pre_g; e.res_ln_b = pre_b;
    phase_gemm<2, false, 8, FFN, STAGE_NONE>(sm, hid, nullptr, nullptr, nullptr, nullptr, L.ffn1_w2, nA, D, e, nullptr, 20);
    PHASE_END(25);
    }
    // q -> qb, k / v -> cache rows a0..
    e = GemmEpi(); e.bias = L.bqkv; e.out = qb; e.ldo = D; e.split_n = D; e.out2 = kc + (size_t)a0 * D; e.ldo2 = D; e.out3 = vc + (size_t)a0 * D; e.ldo3 = D;
    phase_gemm<2, false, 2, D, STAGE_LN>(sm, x, nullptr, nullptr, L.attn_g, L.attn_b, L.wqkv, nA, 3 * D, e, nullptr, 30);
    PHASE_END(35);
    fine_stamp(sm, 40);
    phase_attention(sm, qb, kc, vc, L.pos_proj, Tpos, L.pos_u, L.pos_v, att, nA, a0, T, D, H, chunk);
    PHASE_END(45);
    e = GemmEpi(); e.bias = L.bo; e.out = x; e.ldo = D; e.residual = true;
    phase_gemm<1, false, 2, D, STAGE_COPY>(sm, att, nullptr, nullptr, nullptr, nullptr, L.wo, nA, D, e, nullptr, 50);
    PHASE_END(55);
    // conv module: LN + PW1 + GLU (-> conv cache) + depthwise + BN + SiLU
    e = GemmEpi(); e.bias = L.pw1_b; e.out = gc + (size_t)a0 * D; e.ldo = D;
    DwFuse dwf{gc, L.dw_w, L.bn_scale, L.bn_shift, dw, a0, T, dw_k, conv_chunk};
    phase_gemm<2, true, 2, D, STAGE_LN>(sm, x, nullptr, nullptr, L.conv_g, L.conv_b, L.pw1, nA, 2 * D, e, &dwf, 60);
    PHASE_END(65);
    e = GemmEpi(); e.bias = L.pw2_b; e.out = x; e.ldo = D; e.residual = true;
    phase_gemm<1, false, 2, D, STAGE_COPY>(sm, dw, nullptr, nullptr, nullptr, nullptr, L.pw2, nA, D, e, nullptr, 70);
    PHASE_END(75);
    if (ffn_scratch != nullptr) {
      phase_ffn_partial<FFN>(sm, x, nullptr, nullptr, L.ffn2_g, L.ffn2_b, L.ffn2_w1, L.ffn2_b1, L.ffn2_w2t, ffn_scratch, nA, 80);
      PHASE_END(85);
      phase_ffn_reduce<FFN>(sm, x, ffn_scratch, L.ffn2_b2, 0.5f, nullptr, nullptr, nA, 90);
      PHASE_END(95);
    } else {
    e = GemmEpi(); e.bias = L.ffn2_b1; e.act = ACT_SILU; e.out = hid; e.ldo = FFN;
    phase_gemm<4, false, 2, D, STAGE_LN>(sm, x, nullptr, nullptr, L.ffn2_g, L.ffn2_b, L.ffn2_w1, nA, FFN, e, nullptr, 80);
    PHASE_END(85);
    e = GemmEpi(); e.bias = L.ffn2_b2; e.alpha = 0.5f; e.out = x; e.ldo = D; e.residual = true;
    phase_gemm<2, false, 8, FFN, STAGE_NONE>(sm, hid, nullptr, nullptr, nullptr, nullptr, L.ffn2_w2, nA, D, e, nullptr, 90);
    PHASE_END(95);
    }
  }
#undef PHASE_END
#undef GRID_SYNC
  phase_layer_norm(x, layers[n_layers - 1].fin_g, layers[n_layers - 1].fin_b, nA, D);
}

}  // namespace

bool encoder_layers_persistent_supported(int nA, int D, int FFN, int H, int T, int dw_k) {
  return nA >= 1 && nA <= PMR && D == PD && FFN == 2048 && H * PHD == D && T <= 1024 && (dw_k & 1) == 1 && dw_k <= 31;
}

int encoder_layers_persistent(const PersistLayer* layers_dev, int n_layers, float* x, float* hid, float* qb, float* att, float* dw, float* kc,
                              float* vc, float* gc, int nA, int a0, int T, int D, int FFN, int H, int Tpos, int chunk, int conv_chunk, int dw_k,
                              unsigned long long* ts, unsigned* bar_ctr, unsigned* bar_target_host, int prefetch, float* ffn_scratch,
                              cudaStream_t st) {
  ++g_launches;
  (void)D;
  (void)FFN;
  auto kernel = encoder_layers_persistent_kernel<2048>;
  int occ = 0;
  if (first_time_on_device((const void*)kernel)) {  // cooperative launch needs one resident CTA per SM on this device
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kernel, PT, 0);
    if (occ < 1) return -1;
  }
  const int grid = current_device_sms();
  if (grid <= 0) return -1;
  unsigned bar_target = bar_target_host ? *bar_target_host : 0u;
  if (grid < 2048 / FFN_UNITS) ffn_scratch = nullptr;  // the fused FFN phases give every hidden-unit group its own CTA
  void* args[] = {(void*)&layers_dev, (void*)&n_layers, (void*)&x, (void*)&hid, (void*)&qb, (void*)&att, (void*)&dw, (void*)&kc, (void*)&vc,
                  (void*)&gc, (void*)&nA, (void*)&a0, (void*)&T, (void*)&H, (void*)&Tpos, (void*)&chunk, (void*)&conv_chunk, (void*)&dw_k,
                  (void*)&ts, (void*)&bar_ctr, (void*)&bar_target, (void*)&prefetch, (void*)&ffn_scratch};
  cudaError_t e = cudaLaunchCooperativeKernel((void*)kernel, dim3(grid), dim3(PT), args, 0, st);
  if (e != cudaSuccess) return -2;
  if (bar_ctr != nullptr && bar_target_host != nullptr) *bar_target_host += (unsigned)grid * (unsigned)(9 * n_layers + (ts != nullptr ? 2 : 0));
  return 0;
}

}  // namespace ss
