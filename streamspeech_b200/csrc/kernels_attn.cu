// Attention kernels (fp32, head_dim 64).
//   relpos_attention: RelPositionMultiHeadedAttention.forward with the rel_shift folded into the index
//                     bd[i][j] = (q_i + v) . P[i - j]   (uni_unity/modules/espnet_multihead_attention.py:133-209)
//   mha_attention   : fairseq MultiheadAttention slow path (ctc_unity/modules/multihead_attention.py:555-784)
// Two kernel shapes per op:
//   * tile kernel: one CTA per (16 queries, head, batch); K / V (/ P) tiles of 64 keys are staged in shared memory with
//     coalesced 128-bit loads and consumed with an online softmax (running max / sum), so K and V are read once per
//     query tile and nothing of size T x T ever exists;
//   * row kernel: one CTA per (query, head, batch) for streaming steps with a handful of queries, keys split over the
//     CTA's threads so that many loads are in flight.
#include "common.cuh"
#include "kernels.h"

namespace ss {
namespace {

constexpr int QT = 16;      // queries per CTA (tile kernel)
constexpr int KT = 64;      // keys per shared-memory tile
constexpr int ATT_NT = 128;
constexpr int HD = 64;      // head dim
constexpr int LDK = HD + 4; // padded row stride of the K/V/P tiles (bank-conflict-free 128-bit reads)

__device__ __forceinline__ float dot64(const float* __restrict__ a, const float* __restrict__ b) {
  float acc = 0.f;
#pragma unroll
  for (int d = 0; d < HD; d += 4) {
    float4 x = *reinterpret_cast<const float4*>(a + d);
    float4 y = *reinterpret_cast<const float4*>(b + d);
    acc = fmaf(x.x, y.x, acc);
    acc = fmaf(x.y, y.y, acc);
    acc = fmaf(x.z, y.z, acc);
    acc = fmaf(x.w, y.w, acc);
  }
  return acc;
}

// cooperative copy of `rows` rows of 64 floats (global row stride ld) into a padded smem tile; rows >= valid are zero
__device__ __forceinline__ void load_tile(float* dst, const float* __restrict__ src, int64_t ld, int rows, int valid) {
  for (int e = threadIdx.x; e < rows * (HD / 4); e += ATT_NT) {
    int r = e >> 4, c = (e & 15) << 2;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (r < valid) v = *reinterpret_cast<const float4*>(src + (int64_t)r * ld + c);
    *reinterpret_cast<float4*>(dst + r * LDK + c) = v;
  }
}

// Tile kernel.  RELPOS: queries carry two biased copies (q+u for content, q+v for position) and the score adds
// (q+v).P[i-j]; otherwise plain scaled dot product.  nvis(i) = number of visible keys of query i (a prefix).
template <bool RELPOS>
__global__ void __launch_bounds__(ATT_NT) attn_tile_kernel(const float* __restrict__ q, int ldq, const float* __restrict__ k, int ldk,
                                                           const float* __restrict__ v, int ldv, const float* __restrict__ pos, int Tpos,
                                                           int ldp, const float* __restrict__ bias_u, const float* __restrict__ bias_v,
                                                           float* __restrict__ out, int ldo, int nQ, int q_offset, int T, float scale,
                                                           int chunk, int causal, int causal_offset, const int* __restrict__ lengths) {
  pdl_trigger();
  pdl_wait();
  extern __shared__ __align__(16) float smem[];
  float* Qa = smem;                          // [QT][LDK]  (q+u) or scaled q
  float* Qb = Qa + QT * LDK;                 // [QT][LDK]  (q+v)           (RELPOS only)
  float* Ks = Qb + (RELPOS ? QT * LDK : 0);  // [KT][LDK]
  float* Vs = Ks + KT * LDK;                 // [KT][LDK]
  float* Ps = Vs + KT * LDK;                 // [KT+QT-1][LDK]             (RELPOS only)
  float* Sc = Ps + (RELPOS ? (KT + QT - 1) * LDK : 0);  // [QT][KT+1] probabilities of the current tile
  __shared__ int nvis[QT];
  const int b = blockIdx.z, h = blockIdx.y, r0 = blockIdx.x * QT;
  const int nq = min(QT, nQ - r0);
  const int len = lengths ? min(lengths[b], T) : T;
  const float* qb = q + ((int64_t)b * nQ) * ldq + h * HD;
  const float* kb = k + ((int64_t)b * T) * ldk + h * HD;
  const float* vb = v + ((int64_t)b * T) * ldv + h * HD;
  for (int e = threadIdx.x; e < QT * HD; e += ATT_NT) {
    int qq = e >> 6, d = e & 63;
    float val = (qq < nq) ? qb[(int64_t)(r0 + qq) * ldq + d] : 0.f;
    if (RELPOS) {
      Qa[qq * LDK + d] = val + bias_u[h * HD + d];
      Qb[qq * LDK + d] = val + bias_v[h * HD + d];
    } else {
      Qa[qq * LDK + d] = val * scale;  // q *= scaling (multihead_attention.py:573)
    }
  }
  if (threadIdx.x < QT) {
    int i = q_offset + r0 + threadIdx.x;  // absolute query position
    int lim;
    if (RELPOS) lim = chunk > 0 ? min((i / chunk + 1) * chunk, T) : T;  // chunk mask (s2t_conformer.py:195-213)
    else lim = causal ? min(i + causal_offset + 1, T) : T;
    nvis[threadIdx.x] = threadIdx.x < nq ? max(1, min(lim, len)) : 0;
  }
  __syncthreads();
  int kmax = 0;
  for (int qq = 0; qq < nq; ++qq) kmax = max(kmax, nvis[qq]);
  const int tq = threadIdx.x >> 3;        // query owned by this thread (8 threads per query)
  const int tg = threadIdx.x & 7;         // key phase / dim group
  const int my_nvis = nvis[tq];
  const int i_abs = q_offset + r0 + tq;
  float m_run = -INFINITY, l_run = 0.f;
  float acc[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) acc[e] = 0.f;
  // plain attention: the query row of this thread lives in registers, so a score costs 16 shared-memory reads (the key) instead
  // of 32 (the unit decoder's 25 S x 25 S self-attention is bound by shared-memory bandwidth)
  float4 qreg[RELPOS ? 1 : HD / 4];
  if (!RELPOS) {
#pragma unroll
    for (int d = 0; d < HD / 4; ++d) qreg[d] = *reinterpret_cast<const float4*>(Qa + tq * LDK + 4 * d);
  }
  for (int j0 = 0; j0 < kmax; j0 += KT) {
    const int nk = min(KT, kmax - j0);
    __syncthreads();  // previous tile fully consumed
    load_tile(Ks, kb + (int64_t)j0 * ldk, ldk, KT, nk);
    load_tile(Vs, vb + (int64_t)j0 * ldv, ldv, KT, nk);
    const int rel_lo = (q_offset + r0) - (j0 + KT - 1);  // smallest relative position (i - j) touched by this tile
    if (RELPOS) {
      const float* pb = pos + h * HD;
      for (int e = threadIdx.x; e < (KT + QT - 1) * (HD / 4); e += ATT_NT) {
        int r = e >> 4, c = (e & 15) << 2;
        int rel = rel_lo + r;
        float4 pv = make_float4(0.f, 0.f, 0.f, 0.f);
        if (rel > -Tpos && rel < Tpos) pv = *reinterpret_cast<const float4*>(pb + (int64_t)(rel + Tpos - 1) * ldp + c);
        *reinterpret_cast<float4*>(Ps + r * LDK + c) = pv;
      }
    }
    __syncthreads();
    // scores of this thread: keys jj = tg + 8*i
    float sc[8];
    float tmax = -INFINITY;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      int jj = tg + 8 * i;
      int j = j0 + jj;
      float s = -INFINITY;
      if (j < my_nvis) {
        if (RELPOS) {
          s = dot64(Qa + tq * LDK, Ks + jj * LDK);
          s = (s + dot64(Qb + tq * LDK, Ps + ((i_abs - j) - rel_lo) * LDK)) * 0.125f;  // / sqrt(d_k), d_k = 64
        } else {
          const float* kr = Ks + jj * LDK;
          float a = 0.f;  // same accumulation order as dot64
#pragma unroll
          for (int d = 0; d < HD / 4; ++d) {
            const float4 y = *reinterpret_cast<const float4*>(kr + 4 * d);
            a = fmaf(qreg[d].x, y.x, a);
            a = fmaf(qreg[d].y, y.y, a);
            a = fmaf(qreg[d].z, y.z, a);
            a = fmaf(qreg[d].w, y.w, a);
          }
          s = a;
        }
      }
      sc[i] = s;
      tmax = fmaxf(tmax, s);
    }
    // row max / sum across the 8 threads of the query (they are 8 consecutive lanes of one warp)
#pragma unroll
    for (int o = 1; o < 8; o <<= 1) tmax = fmaxf(tmax, __shfl_xor_sync(0xffffffffu, tmax, o));
    const float m_new = fmaxf(m_run, tmax);
    const float corr = (m_new == -INFINITY) ? 1.f : expf(m_run - m_new);
    float tsum = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      float p = (sc[i] == -INFINITY) ? 0.f : expf(sc[i] - m_new);
      Sc[tq * (KT + 1) + tg + 8 * i] = p;
      tsum += p;
    }
#pragma unroll
    for (int o = 1; o < 8; o <<= 1) tsum += __shfl_xor_sync(0xffffffffu, tsum, o);
    l_run = l_run * corr + tsum;
    m_run = m_new;
    __syncwarp();  // the Sc row of a query is written and read by lanes of the same warp
    const int d0 = tg * 4;  // this thread owns dims [d0, d0+4) and [32+d0, 32+d0+4): conflict-free 128-bit reads of V
#pragma unroll
    for (int e = 0; e < 8; ++e) acc[e] *= corr;
    const float* prow = Sc + tq * (KT + 1);
#pragma unroll 4
    for (int jj = 0; jj < nk; ++jj) {
      float p = prow[jj];
      float4 a = *reinterpret_cast<const float4*>(Vs + jj * LDK + d0);
      float4 c4 = *reinterpret_cast<const float4*>(Vs + jj * LDK + 32 + d0);
      acc[0] = fmaf(p, a.x, acc[0]);
      acc[1] = fmaf(p, a.y, acc[1]);
      acc[2] = fmaf(p, a.z, acc[2]);
      acc[3] = fmaf(p, a.w, acc[3]);
      acc[4] = fmaf(p, c4.x, acc[4]);
      acc[5] = fmaf(p, c4.y, acc[5]);
      acc[6] = fmaf(p, c4.z, acc[6]);
      acc[7] = fmaf(p, c4.w, acc[7]);
    }
  }
  if (tq < nq) {
    float inv = 1.0f / l_run;
    float* op = out + ((int64_t)b * nQ + r0 + tq) * ldo + h * HD + tg * 4;
    *reinterpret_cast<float4*>(op) = make_float4(acc[0] * inv, acc[1] * inv, acc[2] * inv, acc[3] * inv);
    *reinterpret_cast<float4*>(op + 32) = make_float4(acc[4] * inv, acc[5] * inv, acc[6] * inv, acc[7] * inv);
  }
}

// ---- row kernel: one CTA per (query row, head, batch)
__device__ __forceinline__ float block_max128(float v, float* red) {
  v = warp_max(v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  return fmaxf(fmaxf(red[0], red[1]), fmaxf(red[2], red[3]));
}
__device__ __forceinline__ float block_sum128(float v, float* red) {
  v = warp_sum(v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  return (red[0] + red[1]) + (red[2] + red[3]);
}

template <bool RELPOS>
__global__ void __launch_bounds__(ATT_NT) attn_row_kernel(const float* __restrict__ q, int ldq, const float* __restrict__ k, int ldk,
                                                          const float* __restrict__ v, int ldv, const float* __restrict__ pos, int Tpos,
                                                          int ldp, const float* __restrict__ bias_u, const float* __restrict__ bias_v,
                                                          float* __restrict__ out, int ldo, int nQ, int q_offset, int T, float scale,
                                                          int chunk, int causal, int causal_offset, const int* __restrict__ lengths) {
  pdl_trigger();
  pdl_wait();
  extern __shared__ __align__(16) float smem[];
  float* S = smem;  // [T]
  __shared__ __align__(16) float qa[HD], qb2[HD];
  __shared__ __align__(16) float part[4][HD];
  __shared__ float red[4];
  const int r = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const int i = q_offset + r;
  const int len = lengths ? min(lengths[b], T) : T;
  int lim;
  if (RELPOS) lim = chunk > 0 ? min((i / chunk + 1) * chunk, T) : T;
  else lim = causal ? min(r + causal_offset + 1, T) : T;
  const int n = max(1, min(lim, len));
  const float* qp = q + ((int64_t)b * nQ + r) * ldq + h * HD;
  const float* kb = k + ((int64_t)b * T) * ldk + h * HD;
  const float* vb = v + ((int64_t)b * T) * ldv + h * HD;
  if (threadIdx.x < HD) {
    float val = qp[threadIdx.x];
    if (RELPOS) {
      qa[threadIdx.x] = val + bias_u[h * HD + threadIdx.x];
      qb2[threadIdx.x] = val + bias_v[h * HD + threadIdx.x];
    } else {
      qa[threadIdx.x] = val * scale;
    }
  }
  __syncthreads();
  float mx = -INFINITY;
  for (int j = threadIdx.x; j < n; j += ATT_NT) {
    float s = dot64(qa, kb + (int64_t)j * ldk);
    if (RELPOS) s = (s + dot64(qb2, pos + (int64_t)(i - j + Tpos - 1) * ldp + h * HD)) * 0.125f;
    S[j] = s;
    mx = fmaxf(mx, s);
  }
  mx = block_max128(mx, red);
  float sum = 0.f;
  for (int j = threadIdx.x; j < n; j += ATT_NT) {
    float e = expf(S[j] - mx);
    S[j] = e;
    sum += e;
  }
  sum = block_sum128(sum, red);
  __syncthreads();
  // out[d] = sum_j p_j V[j][d]: warp w takes keys j = w (mod 4); lane owns dims 2*lane, 2*lane+1 (coalesced 256 B rows)
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float a0 = 0.f, a1 = 0.f;
#pragma unroll 4
  for (int j = w; j < n; j += 4) {
    float p = S[j];
    float2 vv = *reinterpret_cast<const float2*>(vb + (int64_t)j * ldv + 2 * lane);
    a0 = fmaf(p, vv.x, a0);
    a1 = fmaf(p, vv.y, a1);
  }
  part[w][2 * lane] = a0;
  part[w][2 * lane + 1] = a1;
  __syncthreads();
  if (threadIdx.x < HD) {
    float t = (part[0][threadIdx.x] + part[1][threadIdx.x]) + (part[2][threadIdx.x] + part[3][threadIdx.x]);
    out[((int64_t)b * nQ + r) * ldo + h * HD + threadIdx.x] = t / sum;
  }
}

// Causal self-attention over a sequence in which every key / value / query row is repeated R times in a row (the first layer
// of the CTC unit decoder: each T2U state is upsampled x25 and, because the reference's positional embedding indexes the
// batch axis there (SURVEY.md N1), all R copies of a token carry identical inputs, hence identical q, k, v).  For the copy
// r of group g the softmax over the R*g + r + 1 visible positions collapses to a softmax over g + 1 distinct keys with
// multiplicities R (earlier groups) and r + 1 (own group):
//     out[g, r] = (R * A_g + c * e_g * v_g) / (R * a_g + c * e_g),   A_g = sum_{j < g'} e_j v_j,  a_g = sum_{j < g'} e_j,
// e_j = exp(s_j - max), g' = min(g, n_valid), c = r + 1 if g < n_valid else 0 (keys of padded groups are masked).
// One CTA per (group, head, sample); q / k / v of sample b are its S group rows b*S .. b*S + S-1, out gets its rows b*S*R ..
// (S*R rows per sample) and kv_len[b] is its valid group count.  A sample's arithmetic does not depend on the batch.
__global__ void __launch_bounds__(ATT_NT) grouped_causal_attn_kernel(const float* __restrict__ q, int ldq, const float* __restrict__ k, int ldk,
                                                                      const float* __restrict__ v, int ldv, float* __restrict__ out, int ldo,
                                                                      int S, int R, float scale, const int* __restrict__ kv_len) {
  pdl_trigger();
  pdl_wait();
  extern __shared__ __align__(16) float smem[];  // [S] scores
  __shared__ __align__(16) float qs[HD];
  __shared__ float red[4];
  __shared__ float part[2][HD];
  const int g = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  q += (int64_t)b * S * ldq;
  k += (int64_t)b * S * ldk;
  v += (int64_t)b * S * ldv;
  out += (int64_t)b * S * R * ldo;
  const int n_valid = kv_len ? min(kv_len[b], S) : S;
  const int n_prev = min(g, n_valid);           // earlier groups, every one of their R copies is visible
  const bool own = g < n_valid;
  const int n = n_prev + (own ? 1 : 0);         // distinct visible keys (own group last)
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x < HD) qs[threadIdx.x] = q[(int64_t)g * ldq + h * HD + threadIdx.x] * scale;
  __syncthreads();
  float mx = -INFINITY;
  for (int j = threadIdx.x; j < n; j += ATT_NT) {
    const int key = (j < n_prev) ? j : g;
    float sc = dot64(qs, k + (int64_t)key * ldk + h * HD);
    smem[j] = sc;
    mx = fmaxf(mx, sc);
  }
  mx = block_max128(mx, red);
  float sum = 0.f;
  for (int j = threadIdx.x; j < n; j += ATT_NT) {
    float e = expf(smem[j] - mx);
    smem[j] = e;
    if (j < n_prev) sum += e;
  }
  sum = block_sum128(sum, red);  // a_g
  __syncthreads();
  // A_g[d]: two halves of the earlier keys per dimension
  {
    const int d = threadIdx.x & (HD - 1), half = threadIdx.x >> 6;
    float a = 0.f;
    for (int j = half; j < n_prev; j += 2) a = fmaf(smem[j], v[(int64_t)j * ldv + h * HD + d], a);
    part[half][d] = a;
  }
  __syncthreads();
  const float e_own = own ? smem[n_prev] : 0.f;
  for (int idx = threadIdx.x; idx < R * HD; idx += ATT_NT) {
    const int r = idx >> 6, d = idx & (HD - 1);
    const float c = own ? (float)(r + 1) : 0.f;
    const float num = (float)R * (part[0][d] + part[1][d]) + c * e_own * (own ? v[(int64_t)g * ldv + h * HD + d] : 0.f);
    const float den = (float)R * sum + c * e_own;
    out[((int64_t)g * R + r) * ldo + h * HD + d] = num / den;
  }
}

template <bool RELPOS>
void launch_attn(const float* q, int ldq, const float* k, int ldk, const float* v, int ldv, const float* pos, int Tpos, int ldp,
                 const float* bias_u, const float* bias_v, float* out, int ldo, int B, int nQ, int q_offset, int T, int H, float scale,
                 int chunk, int causal, int causal_offset, const int* lengths, int B_choice, int kernel, cudaStream_t st) {
  // row or tile kernel, chosen from B_choice samples of this shape (1: from one sample, so that batching never switches a
  // sample's arithmetic to the other kernel); kernel = 1 / 2 forces the row / tile kernel (parity tests; the caller checks that
  // T fits the row kernel's shared memory)
  const long tiles = (long)((nQ + QT - 1) / QT) * H * B_choice;
  if (kernel == 1 || (kernel == 0 && tiles < 96 && (size_t)T * sizeof(float) <= 160 * 1024)) {
    size_t smem_row = (size_t)((T + 3) & ~3) * sizeof(float);
    if (smem_row > 40 * 1024 && first_time_on_device((const void*)attn_row_kernel<RELPOS>))
      cudaFuncSetAttribute(attn_row_kernel<RELPOS>, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024);
    launch_pdl(attn_row_kernel<RELPOS>, dim3(dim3(nQ, H, B)), dim3(ATT_NT), smem_row, st, q, ldq, k, ldk, v, ldv, pos, Tpos, ldp, bias_u, bias_v, out, ldo, nQ,
                                                                      q_offset, T, scale, chunk, causal, causal_offset, lengths);
    return;
  }
  size_t smem = (size_t)((RELPOS ? 2 : 1) * QT * LDK + 2 * KT * LDK + (RELPOS ? (KT + QT - 1) * LDK : 0) + QT * (KT + 1)) * sizeof(float);
  if (first_time_on_device((const void*)attn_tile_kernel<RELPOS>))
    cudaFuncSetAttribute(attn_tile_kernel<RELPOS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  launch_pdl(attn_tile_kernel<RELPOS>, dim3(dim3((nQ + QT - 1) / QT, H, B)), dim3(ATT_NT), smem, st, q, ldq, k, ldk, v, ldv, pos, Tpos, ldp, bias_u, bias_v, out, ldo,
                                                                                 nQ, q_offset, T, scale, chunk, causal, causal_offset, lengths);
}

}  // namespace

void relpos_attention(const float* q, int ldq, const float* k, int ldk, const float* v, int ldv, const float* pos, int Tpos,
                      const float* bias_u, const float* bias_v, float* out, int B, int nQ, int q_offset, int T, int H, int D,
                      int chunk, const int* lengths_dev, cudaStream_t st, int kernel) {
  ++g_launches;
  if (B <= 0 || T <= 0 || nQ <= 0) return;
  launch_attn<true>(q, ldq, k, ldk, v, ldv, pos, Tpos, D, bias_u, bias_v, out, D, B, nQ, q_offset, T, H, 0.125f, chunk, 0, 0, lengths_dev, B, kernel,
                    st);
}

void grouped_causal_attention(const float* q, int ldq, const float* k, int ldk, const float* v, int ldv, float* out, int ldo, int S, int R,
                              int H, float scale, const int* kv_len_dev, int B, cudaStream_t st) {
  ++g_launches;
  if (S <= 0 || R <= 0 || B <= 0) return;
  launch_pdl(grouped_causal_attn_kernel, dim3(S, H, B), dim3(ATT_NT), (size_t)((S + 3) & ~3) * sizeof(float), st, q, ldq, k, ldk, v, ldv, out, ldo, S,
             R, scale, kv_len_dev);
}

void mha_attention(const float* q, int ldq, const float* k, int ldk, const float* v, int ldv, float* out, int ldo, int B,
                   int Tq, int Tk, int H, float scale, int causal, int causal_offset, const int* kv_len_dev,
                   cudaStream_t st, int kernel) {
  ++g_launches;
  if (B <= 0 || Tq <= 0 || Tk <= 0) return;
  launch_attn<false>(q, ldq, k, ldk, v, ldv, nullptr, 0, 0, nullptr, nullptr, out, ldo, B, Tq, 0, Tk, H, scale, 0, causal, causal_offset,
                     kv_len_dev, 1, kernel, st);
}

}  // namespace ss
