// Persistent cooperative kernel for the MT decoder's PREFIX pass: all 4 pre-LN layers over the M <= 64 forced-prefix tokens
// [eos, t1 .. t_{M-1}] of one generate_decoder call (agent/sequence_generator.py:165-582 re-runs the decoder on the whole prefix
// at every policy() call, agent:179) in ONE launch.  It fills the self-attention K / V cache rows 0 .. M-1 and the final-LN
// feature rows; the single-token kernel (kernels_persist_mt.cu) then continues at position M.  As separate kernels the pass was
// 38 dependent launches; here it is 33 grid-barrier phases:
//   per layer: [LN + QKV -> q, K/V cache] | [causal self-attention] | [out + res] | [LN + Q] | [cross-attention] | [out + res] |
//              [LN + FC1 + ReLU] | [FC2 + res]       then: final LN -> feature rows
// GEMM phases are the M <= 16 scheme of kernels_persist.cu extended to row blocks of 16 with the weights of a task held in
// registers across the blocks (W is read once per CTA-task); activations with K = 512 are staged (layer-normed) in shared
// memory, the K = 2048 FFN hidden is read per K-slice from L2.  Attention: one CTA per (head, block of 8 query rows), one warp
// per row, so the 8 warps of a CTA share the K / V rows of their head through L1.
#include "common.cuh"
#include "kernels.h"
#include "kernels_persist.h"

namespace ss {
namespace {

constexpr int QW = 8;            // warps per CTA
constexpr int QT = QW * 32;
constexpr int QRB = 16;          // rows per block (accumulators per lane and column)
constexpr int QMAXM = 64;        // max prefix rows
constexpr int QD = 512;          // model dim
constexpr int QFFN = 2048;
constexpr int QHD = 64;
constexpr int QMAXT = 1024;      // max encoder rows (cross-attention keys)

__device__ __forceinline__ float4 ldw(const float* p) {
  float4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p));
  return r;
}

struct QSmem {                    // static part; As (staged activations [QMAXM][QD]) and S (scores [QW][QMAXT]) are dynamic
  float part[QW][4][QRB];
  float qs[QW][QHD];
};

// As[m][:] = LN(x[m][:]) for m < M; rows [M, Mpad) are zero.  Warp w takes rows w, w + 8, ...; 16 values per lane.
// `src_tok` != nullptr: x is built here from the token embeddings (first layer) and CTA 0 also writes it to xg.
__device__ __forceinline__ void stage_ln512(float* As, const float* x, int M, int Mpad, const float* __restrict__ g, const float* __restrict__ b,
                                            const int64_t* src_tok, const float* __restrict__ emb, const float* __restrict__ pos, int pad,
                                            float emb_scale, float* xg) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  // the LayerNorm parameters of this lane's 16 columns and the rows of 2 row slots are all in flight before the first reduction
  // (one row at a time meant two dependent L2 round trips per row)
  float gv[16], bv[16];
#pragma unroll
  for (int i = 0; i < 16; ++i) {
    gv[i] = __ldg(g + lane + (i << 5));
    bv[i] = __ldg(b + lane + (i << 5));
  }
  for (int m0 = warp; m0 < Mpad; m0 += 2 * QW) {
    float v[2][16];
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      const int m = m0 + u * QW;
      if (m < M) {
        if (src_tok != nullptr) {
          const int64_t tok = src_tok[m];
          const int p = (tok == pad) ? pad : pad + 1 + m;
#pragma unroll
          for (int i = 0; i < 16; ++i) {
            const int c = lane + (i << 5);
            v[u][i] = emb_scale * emb[tok * QD + c] + pos[(int64_t)p * QD + c];
          }
          if (blockIdx.x == 0) {
#pragma unroll
            for (int i = 0; i < 16; ++i) xg[(int64_t)m * QD + lane + (i << 5)] = v[u][i];
          }
        } else {
#pragma unroll
          for (int i = 0; i < 16; ++i) v[u][i] = x[(int64_t)m * QD + lane + (i << 5)];
        }
      } else {
#pragma unroll
        for (int i = 0; i < 16; ++i) v[u][i] = 0.f;
      }
    }
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      const int m = m0 + u * QW;
      if (m >= Mpad) continue;
      if (m < M) {
        float s = 0.f;
#pragma unroll
        for (int i = 0; i < 16; ++i) s += v[u][i];
        const float mean = warp_sum(s) / (float)QD;
        float q = 0.f;
#pragma unroll
        for (int i = 0; i < 16; ++i) {
          const float d = v[u][i] - mean;
          q = fmaf(d, d, q);
        }
        const float rstd = 1.0f / sqrtf(warp_sum(q) / (float)QD + 1e-5f);
#pragma unroll
        for (int i = 0; i < 16; ++i) As[m * QD + lane + (i << 5)] = (v[u][i] - mean) * rstd * gv[i] + bv[i];
      } else {
#pragma unroll
        for (int i = 0; i < 16; ++i) As[m * QD + lane + (i << 5)] = 0.f;
      }
    }
  }
}

// As[m][:] = a[m][:] (K = 512), zeros for M <= m < Mpad
__device__ __forceinline__ void stage_copy512(float* As, const float* a, int M, int Mpad) {
  for (int idx = threadIdx.x; idx < Mpad * (QD / 4); idx += QT) {
    const int m = idx / (QD / 4);
    float4 val = make_float4(0.f, 0.f, 0.f, 0.f);
    if (m < M) val = *reinterpret_cast<const float4*>(a + (int64_t)idx * 4);
    *reinterpret_cast<float4*>(As + idx * 4) = val;
  }
}

// epi(m, col, value) for every m < M, col < N of  A[M][K] @ W[N][K]^T.  STAGED: A = As in shared memory (K == QD);
// otherwise every warp reads its K-slice of A from global memory (coherent loads: written by other CTAs before the barrier).
// `stage` (staging of As + CTA barrier, or nothing) runs after the weight loads of the CTA's first task have been issued, so the
// weights fly while the activations are staged; CTAs without a task skip it.
template <int CPT, int KS, int K, bool STAGED, typename Stage, typename Epi>
__device__ __forceinline__ void pgemm(QSmem& sm, const float* As, const float* A, const float* __restrict__ W, int M, int N, Stage&& stage, Epi&& epi) {
  constexpr int KSLICE = K / KS;
  constexpr int NIT = KSLICE / 128;
  static_assert(KSLICE % 128 == 0, "K slice must be a multiple of 128");
  static_assert(CPT <= 4, "part[] holds 4 columns");
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  constexpr int TPC = QW / KS;
  const int slice = warp % KS, tslot = warp / KS;
  const int ntasks = N / CPT;
  const int k_lo = slice * KSLICE;
  const int mrow = lane >> 1;
  const bool owner = (lane & 1) == 0;
  for (int tbase = blockIdx.x * TPC; tbase < ntasks; tbase += gridDim.x * TPC) {
    const int task = tbase + tslot;
    const bool active = task < ntasks;
    const int n0 = task * CPT;
    float4 wv[NIT][CPT];
#pragma unroll
    for (int it = 0; it < NIT; ++it)
#pragma unroll
      for (int c = 0; c < CPT; ++c)
        wv[it][c] = active ? ldw(W + (int64_t)(n0 + c) * K + k_lo + it * 128 + lane * 4) : make_float4(0.f, 0.f, 0.f, 0.f);
    if (tbase == (int)blockIdx.x * TPC) stage();
    for (int mb = 0; mb < M; mb += QRB) {
      float acc[CPT][QRB];
#pragma unroll
      for (int c = 0; c < CPT; ++c)
#pragma unroll
        for (int r = 0; r < QRB; ++r) acc[c][r] = 0.f;
#pragma unroll
      for (int it = 0; it < NIT; ++it) {
        const int k = k_lo + it * 128 + lane * 4;
#pragma unroll
        for (int r = 0; r < QRB; ++r) {
          float4 x;
          if (STAGED) {
            x = *reinterpret_cast<const float4*>(As + (mb + r) * K + k);
          } else {
            x = (mb + r < M) ? *reinterpret_cast<const float4*>(A + (int64_t)(mb + r) * K + k) : make_float4(0.f, 0.f, 0.f, 0.f);
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
      // 16 row sums per column across the warp (recursive halving, fixed order): even lane 2m ends with row m
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
          for (int c = 0; c < CPT; ++c) sm.part[warp][c][mrow] = mine[c];
        }
        __syncthreads();
        if (slice == 0 && owner) {
#pragma unroll
          for (int c = 0; c < CPT; ++c) {
            float t = sm.part[warp][c][mrow];
#pragma unroll
            for (int s = 1; s < KS; ++s) t += sm.part[warp + s][c][mrow];
            mine[c] = t;
          }
        }
      }
      if (active && slice == 0 && owner && mb + mrow < M) {
#pragma unroll
        for (int c = 0; c < CPT; ++c) epi(mb + mrow, n0 + c, mine[c]);
      }
      if (KS > 1) __syncthreads();
    }
  }
}

// softmax(q K^T / 8) V for query rows [r0, r0 + 8) of head h: one warp per row.  causal: keys 0 .. row, else keys 0 .. nk-1.
// K / V rows at kbase / vbase + j * ld.  S = this warp's score buffer (>= nk floats).
__device__ __forceinline__ void attend_rows(QSmem& sm, float* S, const float* q, const float* kbase, const float* vbase, int ld, int row, int M,
                                            int nk, float* out) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (row >= M) return;
  __syncwarp();
  sm.qs[warp][lane] = q[lane] * 0.125f;
  sm.qs[warp][lane + 32] = q[lane + 32] * 0.125f;
  __syncwarp();
  float mx = -INFINITY;
  for (int j = lane; j < nk; j += 32) {
    const float* kr = kbase + (int64_t)j * ld;
    float s = 0.f;
#pragma unroll
    for (int d = 0; d < QHD / 4; ++d) {
      const float4 kk = *reinterpret_cast<const float4*>(kr + 4 * d);
      s = fmaf(sm.qs[warp][4 * d], kk.x, s);
      s = fmaf(sm.qs[warp][4 * d + 1], kk.y, s);
      s = fmaf(sm.qs[warp][4 * d + 2], kk.z, s);
      s = fmaf(sm.qs[warp][4 * d + 3], kk.w, s);
    }
    S[j] = s;
    mx = fmaxf(mx, s);
  }
  mx = warp_max(mx);
  float sum = 0.f;
  for (int j = lane; j < nk; j += 32) {
    const float e = expf(S[j] - mx);
    S[j] = e;
    sum += e;
  }
  sum = warp_sum(sum);
  __syncwarp();
  float a0 = 0.f, a1 = 0.f;  // dims lane, lane + 32
  // 32 keys per round: 64 independent coalesced loads in flight per lane (the loop used to be 4 keys per L2 round trip:
  // 40 dependent round trips for 160 cross-attention keys per prefix row and layer)
#pragma unroll 1
  for (int j0 = 0; j0 < nk; j0 += 32) {
    float v0[32], v1[32];
#pragma unroll
    for (int u = 0; u < 32; ++u) {
      const bool ok = j0 + u < nk;
      const float* vr = vbase + (int64_t)(ok ? j0 + u : 0) * ld;
      v0[u] = ok ? vr[lane] : 0.f;
      v1[u] = ok ? vr[lane + 32] : 0.f;
    }
#pragma unroll
    for (int u = 0; u < 32; ++u) {
      const float p = (j0 + u < nk) ? S[j0 + u] : 0.f;
      a0 = fmaf(p, v0[u], a0);
      a1 = fmaf(p, v1[u], a1);
    }
  }
  out[lane] = a0 / sum;
  out[lane + 32] = a1 / sum;
}

__global__ void __launch_bounds__(QT, 1) mt_prefix_persistent_kernel(MtDecodeParams P, const MtLayerP* __restrict__ layers, int M, int T,
                                                                     unsigned* bar_ctr, unsigned bar_target) {
  extern __shared__ __align__(16) float dyn[];
  __shared__ QSmem sm;
  float* As = dyn;                               // [Mpad][QD]
  const int Mpad = (M + QRB - 1) / QRB * QRB;
  float* Sall = dyn + (size_t)QMAXM * QD;        // [QW][QMAXT]
  const int warp = threadIdx.x >> 5;
  float* S = Sall + warp * QMAXT;
  const float emb_scale = sqrtf((float)QD);
  float* x = P.x;        // [M][QD] residual stream (global)
  float* qb = P.q;       // [M][QD]
  float* att = P.attn;   // [M][QD]
  float* hid = P.hid;    // [M][QFFN]
#define BAR() grid_barrier(bar_ctr, bar_target)
  for (int l = 0; l < P.n_layers; ++l) {
    const MtLayerP L = layers[l];
    float* kc = P.self_k + (size_t)l * P.max_pos * QD;
    float* vc = P.self_v + (size_t)l * P.max_pos * QD;
    // (1) q | k | v = LN(x) Wqkv^T  (layer 0 builds x from the embeddings while staging)
    pgemm<4, 2, QD, true>(sm, As, nullptr, L.wqkv, M, 3 * QD, [&]() {
      stage_ln512(As, x, M, Mpad, L.self_g, L.self_b, l == 0 ? P.tok : nullptr, P.emb, P.pos, P.pad, emb_scale, x);
      __syncthreads();
    }, [&](int m, int col, float acc) {
      const float y = acc + (L.bqkv ? L.bqkv[col] : 0.f);
      if (col < QD) qb[(int64_t)m * QD + col] = y;
      else if (col < 2 * QD) kc[(int64_t)m * QD + col - QD] = y;
      else vc[(int64_t)m * QD + col - 2 * QD] = y;
    });
    BAR();
    // (2) causal self-attention: CTA = (head, 8 rows)
    for (int task = blockIdx.x; task < P.heads * ((M + QW - 1) / QW); task += gridDim.x) {
      const int h = task % P.heads, r0 = (task / P.heads) * QW;
      const int row = r0 + warp;
      attend_rows(sm, S, qb + (int64_t)row * QD + h * QHD, kc + h * QHD, vc + h * QHD, QD, row, M, row + 1, att + (int64_t)row * QD + h * QHD);
    }
    BAR();
    // (3) x += attn Wo^T
    pgemm<2, 2, QD, true>(sm, As, nullptr, L.wo, M, QD, [&]() {
      stage_copy512(As, att, M, Mpad);
      __syncthreads();
    }, [&](int m, int col, float acc) {
      x[(int64_t)m * QD + col] = (acc + (L.bo ? L.bo[col] : 0.f)) + x[(int64_t)m * QD + col];
    });
    BAR();
    // (4) q = LN(x) Wcq^T
    pgemm<2, 2, QD, true>(sm, As, nullptr, L.wcq, M, QD, [&]() {
      stage_ln512(As, x, M, Mpad, L.cross_g, L.cross_b, nullptr, nullptr, nullptr, 0, 0.f, nullptr);
      __syncthreads();
    }, [&](int m, int col, float acc) { qb[(int64_t)m * QD + col] = acc + (L.bcq ? L.bcq[col] : 0.f); });
    BAR();
    // (5) cross-attention over the T encoder rows (K | V rows projected before the launch)
    {
      const float* cross = P.cross_kv + (size_t)l * P.cross_cap * 2 * QD;
      for (int task = blockIdx.x; task < P.heads * ((M + QW - 1) / QW); task += gridDim.x) {
        const int h = task % P.heads, r0 = (task / P.heads) * QW;
        const int row = r0 + warp;
        attend_rows(sm, S, qb + (int64_t)row * QD + h * QHD, cross + h * QHD, cross + QD + h * QHD, 2 * QD, row, M, T, att + (int64_t)row * QD + h * QHD);
      }
    }
    BAR();
    // (6) x += attn Wco^T
    pgemm<2, 2, QD, true>(sm, As, nullptr, L.wco, M, QD, [&]() {
      stage_copy512(As, att, M, Mpad);
      __syncthreads();
    }, [&](int m, int col, float acc) {
      x[(int64_t)m * QD + col] = (acc + (L.bco ? L.bco[col] : 0.f)) + x[(int64_t)m * QD + col];
    });
    BAR();
    // (7) hid = relu(LN(x) W1^T)
    pgemm<4, 2, QD, true>(sm, As, nullptr, L.w1, M, QFFN, [&]() {
      stage_ln512(As, x, M, Mpad, L.fin_g, L.fin_b, nullptr, nullptr, nullptr, 0, 0.f, nullptr);
      __syncthreads();
    }, [&](int m, int col, float acc) {
      const float y = acc + (L.b1 ? L.b1[col] : 0.f);
      hid[(int64_t)m * QFFN + col] = y > 0.f ? y : 0.f;
    });
    BAR();
    // (8) x += hid W2^T
    pgemm<4, 8, QFFN, false>(sm, nullptr, hid, L.w2, M, QD, [&]() {}, [&](int m, int col, float acc) {
      x[(int64_t)m * QD + col] = (acc + (L.b2 ? L.b2[col] : 0.f)) + x[(int64_t)m * QD + col];
    });
    BAR();
  }
#undef BAR
  // final LayerNorm -> feature rows (one warp per row, same arithmetic as stage_ln512)
  {
    const int lane = threadIdx.x & 31;
    for (int m = blockIdx.x * QW + warp; m < M; m += gridDim.x * QW) {
      float v[16];
#pragma unroll
      for (int i = 0; i < 16; ++i) v[i] = x[(int64_t)m * QD + lane + (i << 5)];
      float s = 0.f;
#pragma unroll
      for (int i = 0; i < 16; ++i) s += v[i];
      const float mean = warp_sum(s) / (float)QD;
      float q = 0.f;
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        const float d = v[i] - mean;
        q = fmaf(d, d, q);
      }
      const float rstd = 1.0f / sqrtf(warp_sum(q) / (float)QD + 1e-5f);
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        const int c = lane + (i << 5);
        P.feats[(int64_t)m * QD + c] = (v[i] - mean) * rstd * P.out_g[c] + P.out_b[c];
      }
    }
  }
}

}  // namespace

bool mt_prefix_persistent_supported(int dim, int ffn, int heads, int M, int T) {
  return dim == QD && ffn == QFFN && heads * QHD == dim && M >= 1 && M <= QMAXM && T >= 1 && T <= QMAXT;
}

int mt_prefix_persistent(const MtDecodeParams& P, const MtLayerP* layers_dev, int M, int T, unsigned* bar_ctr, unsigned* bar_target_host,
                         cudaStream_t st) {
  ++g_launches;
  const size_t smem = ((size_t)QMAXM * QD + (size_t)QW * QMAXT) * sizeof(float);
  if (first_time_on_device((const void*)mt_prefix_persistent_kernel)) {
    if (cudaFuncSetAttribute(mt_prefix_persistent_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) return -1;
  }
  const int grid = current_device_sms();
  if (grid <= 0) return -1;
  MtDecodeParams p = P;
  unsigned bar_target = *bar_target_host;
  void* args[] = {(void*)&p, (void*)&layers_dev, (void*)&M, (void*)&T, (void*)&bar_ctr, (void*)&bar_target};
  cudaError_t e = cudaLaunchCooperativeKernel((void*)mt_prefix_persistent_kernel, dim3(grid), dim3(QT), args, smem, st);
  if (e != cudaSuccess) return -2;
  *bar_target_host += (unsigned)grid * (unsigned)(P.n_layers * 8);
  return 0;
}

}  // namespace ss
