// Streaming / scan kernels of the path: LayerNorm, depthwise chunk-causal conv + BN + SiLU, embedding
// gathers, arg-max over the vocabulary, CTC collapse, duration rounding, frame expansion, conv_post.
// All HBM-bound: coalesced row-major accesses, warp-shuffle reductions, no re-reads.
#include <algorithm>

#include "common.cuh"
#include "kernels.h"

namespace ss {
unsigned long long g_launches = 0;
thread_local int g_pdl_off = 0;
int g_prefer_shared = 0;  // option prefer_shared (see common.cuh)
namespace {

// one warp per row; two-pass (mean, then centred sum of squares) like ATen's RowwiseMoments result
template <int N>  // N = C / 32
__global__ void layer_norm_kernel(const float* __restrict__ x, int ldx, float* __restrict__ y, int ldy,
                                  const float* __restrict__ gamma, const float* __restrict__ beta, int rows) {
  pdl_trigger();
  pdl_wait();
  constexpr int C = N * 32;
  int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  int lane = threadIdx.x & 31;
  if (row >= rows) return;
  const float* xr = x + (int64_t)row * ldx;
  float v[N];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < N; ++i) {
    v[i] = xr[lane + (i << 5)];
    s += v[i];
  }
  float mean = warp_sum(s) / (float)C;
  float ss_ = 0.f;
#pragma unroll
  for (int i = 0; i < N; ++i) {
    float d = v[i] - mean;
    ss_ = fmaf(d, d, ss_);
  }
  float var = warp_sum(ss_) / (float)C;
  float rstd = 1.0f / sqrtf(var + 1e-5f);
  float* yr = y + (int64_t)row * ldy;
#pragma unroll
  for (int i = 0; i < N; ++i) {
    int c = lane + (i << 5);
    yr[c] = (v[i] - mean) * rstd * gamma[c] + beta[c];
  }
}

__global__ void depthwise_bn_silu_kernel(const float* __restrict__ x, int ldx, const float* __restrict__ w,
                                         const float* __restrict__ scale, const float* __restrict__ shift,
                                         float* __restrict__ y, int ldy, int T, int t0, int n, int C, int k, int chunk) {
  pdl_trigger();
  pdl_wait();
  int row = blockIdx.x;  // b*n + r
  int b = row / n, t = t0 + (row - b * n);
  int half = (k - 1) >> 1;
  int lim = T;
  if (chunk > 0) lim = min(T, (t / chunk + 1) * chunk);  // future beyond the chunk end is zero (chunk_causal_conv1d.py:40-62)
  // NB: the reference convolves over padded frames too (padding is only masked in attention)
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float acc = 0.f;
    // taps in groups of 8: the loads of a group are independent and all in flight before the FMA chain consumes them
    for (int j0 = 0; j0 < k; j0 += 8) {
      float xv[8], wv[8];
#pragma unroll
      for (int jj = 0; jj < 8; ++jj) {
        int j = j0 + jj, p = t - half + j;
        bool ok = j < k && p >= 0 && p < lim;
        xv[jj] = ok ? x[((int64_t)b * T + p) * ldx + c] : 0.f;
        wv[jj] = ok ? w[j * C + c] : 0.f;
      }
#pragma unroll
      for (int jj = 0; jj < 8; ++jj) acc = fmaf(wv[jj], xv[jj], acc);
    }
    float v = acc * scale[c] + shift[c];
    y[(int64_t)row * ldy + c] = v / (1.0f + expf(-v));
  }
}

__global__ void scale_kernel(float* x, int64_t n, float s) {
  pdl_trigger();
  pdl_wait();
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) x[i] *= s;
}

__global__ void add3_kernel(const float4* __restrict__ a, const float4* __restrict__ b, const float4* __restrict__ c, float4* __restrict__ out,
                            int64_t n4) {
  pdl_trigger();
  pdl_wait();
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n4) return;
  float4 x = a[i], y = b[i], z = c[i], r;
  r.x = z.x + (y.x + x.x);
  r.y = z.y + (y.y + x.y);
  r.z = z.z + (y.z + x.z);
  r.w = z.w + (y.w + x.w);
  out[i] = r;
}

__global__ void copy_kernel(const float* __restrict__ s, float* __restrict__ d, int64_t n) {
  pdl_trigger();
  pdl_wait();
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) d[i] = s[i];
}

__global__ void embed_tokens_pos_kernel(const int64_t* __restrict__ tokens, const int* __restrict__ positions, int pos_offset,
                                        const float* __restrict__ emb, const float* __restrict__ pos_table, float scale,
                                        float* __restrict__ out, int rows, int C, int pad_idx) {
  pdl_trigger();
  pdl_wait();
  int r = blockIdx.x;
  int64_t tok = tokens[r];
  // make_positions (fairseq/utils.py:256-266) for sequences whose pads are trailing:
  // non-pad token at index i gets pad_idx + 1 + i, pad gets pad_idx (a zero row)
  int p = positions ? positions[r] : (tok == pad_idx ? pad_idx : pad_idx + 1 + pos_offset + r);
  for (int c = threadIdx.x; c < C; c += blockDim.x)
    out[(int64_t)r * C + c] = scale * emb[tok * C + c] + pos_table[(int64_t)p * C + c];
}

__global__ void repeat_rows_add_kernel(const float* __restrict__ x, int S, int R, int C, const float* __restrict__ addvec,
                                       float* __restrict__ out) {
  pdl_trigger();
  pdl_wait();
  int r = blockIdx.x;  // output row s*R + rr
  int s = r / R;
  const float* xr = x + (int64_t)s * C;
  // N1 quirk: position index comes from the VALUE x[t, b, 0]: != 1.0 -> pad+1 (addvec), == 1.0 -> pad (zero row)
  bool add = addvec != nullptr && xr[0] != 1.0f;
  for (int c = threadIdx.x; c < C; c += blockDim.x) out[(int64_t)r * C + c] = xr[c] + (add ? addvec[c] : 0.f);
}

// arg-max of log_softmax(logits) with masked columns, first index wins on ties
// (CTCDecoder.generate, agent/ctc_decoder.py:53-62; F.log_softmax = (x - max) - log(sum(exp(x - max))))
__global__ void argmax_rows_kernel(const float* __restrict__ logits, int ld, int V, const int* __restrict__ masked, int n_masked,
                                   int64_t* __restrict__ out_idx, float* __restrict__ out_lprob) {
  pdl_trigger();
  pdl_wait();
  __shared__ float red[32];
  __shared__ float sval[32];
  __shared__ int sidx[32];
  int row = blockIdx.x;
  const float* x = logits + (int64_t)row * ld;
  float mx = -INFINITY;
  for (int c = threadIdx.x; c < V; c += blockDim.x) mx = fmaxf(mx, x[c]);
  mx = warp_max(mx);
  int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = blockDim.x >> 5;
  if (lane == 0) red[w] = mx;
  __syncthreads();
  mx = red[0];
  for (int i = 1; i < nw; ++i) mx = fmaxf(mx, red[i]);
  __syncthreads();
  float s = 0.f;
  for (int c = threadIdx.x; c < V; c += blockDim.x) s += expf(x[c] - mx);
  s = block_sum(s, red);
  float lse = logf(s);
  float best = -INFINITY;
  int bi = 0x7fffffff;
  for (int c = threadIdx.x; c < V; c += blockDim.x) {
    bool m = false;
    for (int q = 0; q < n_masked; ++q) m |= (masked[q] == c);
    float lp = m ? -INFINITY : (x[c] - mx) - lse;
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
  if (lane == 0) {
    sval[w] = best;
    sidx[w] = bi;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int i = 1; i < nw; ++i)
      if (sval[i] > best || (sval[i] == best && sidx[i] < bi)) {
        best = sval[i];
        bi = sidx[i];
      }
    out_idx[row] = bi;
    if (out_lprob) out_lprob[row] = best;
  }
}

__global__ void ctc_collapse_kernel(const int64_t* __restrict__ am, int n, int blank, int pad, int64_t* __restrict__ toks,
                                    int* __restrict__ index, int* __restrict__ count) {
  pdl_trigger();
  pdl_wait();
  // one CTA of 1024 threads; thread t owns the contiguous slice [t*per, (t+1)*per); block-wide exclusive scan of the keep counts
  __shared__ int wsum[32];
  const int t = threadIdx.x, lane = t & 31, w = t >> 5;
  const int per = (n + 1023) / 1024;
  const int lo = min(n, t * per), hi = min(n, lo + per);
  int c = 0;
  for (int i = lo; i < hi; ++i) {
    int64_t v = am[i];
    c += ((i == 0 || v != am[i - 1]) && v != blank && v != pad) ? 1 : 0;
  }
  int inc = c;  // inclusive scan inside the warp
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    int y = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += y;
  }
  if (lane == 31) wsum[w] = inc;
  __syncthreads();
  if (w == 0) {
    int s = wsum[lane];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      int y = __shfl_up_sync(0xffffffffu, s, o);
      if (lane >= o) s += y;
    }
    wsum[lane] = s;
  }
  __syncthreads();
  int base = (w > 0 ? wsum[w - 1] : 0) + inc - c;
  for (int i = lo; i < hi; ++i) {
    int64_t v = am[i];
    if ((i == 0 || v != am[i - 1]) && v != blank && v != pad) {
      toks[base] = v;
      if (index) index[base] = i;
      ++base;
    }
  }
  if (t == 1023) *count = wsum[31];
}

// Both CTC heads of one policy() call after the fused [rows][2V] projection: block b = (head, new row) computes the arg-max of
// log_softmax with masks exactly like argmax_rows_kernel; the LAST block to finish (ticket) then collapses both arg-max
// sequences (CTCDecoder.generate, agent/ctc_decoder.py:64-111) into the packed outputs
//   out[head] = [count (int32 in the first int64) | tokens[n_rows] int64 | index[n_rows] int32], stride out_stride int64 words.
__global__ void __launch_bounds__(256) ctc_argmax_collapse_pair_kernel(const float* __restrict__ logits, int ld, int V, int n_new, int row0,
                                                                      int n_rows, const int* __restrict__ masked, int n_masked, int blank,
                                                                      int pad, int64_t* am0, int64_t* am1, int64_t* out, int out_stride,
                                                                      unsigned* ticket) {
  pdl_trigger();
  pdl_wait();
  __shared__ float red[32];
  __shared__ float sval[8];
  __shared__ int sidx[8];
  __shared__ int scount[256];
  __shared__ unsigned s_last;
  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  if ((int)blockIdx.x < 2 * n_new) {
    const int head = blockIdx.x / n_new, r = blockIdx.x - head * n_new;
    const float* x = logits + (int64_t)r * ld + head * V;
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
      float lp = m ? -INFINITY : (x[c] - mx) - lse;
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
    if (lane == 0) {
      sval[w] = best;
      sidx[w] = bi;
    }
    __syncthreads();
    if (tid == 0) {
      for (int i = 1; i < 8; ++i)
        if (sval[i] > best || (sval[i] == best && sidx[i] < bi)) {
          best = sval[i];
          bi = sidx[i];
        }
      (head ? am1 : am0)[row0 + r] = bi;
    }
  }
  // ---- ticket: the last block collapses both sequences
  __syncthreads();
  if (tid == 0) {
    __threadfence();
    s_last = atomicAdd(ticket, 1u) == gridDim.x - 1 ? 1u : 0u;
  }
  __syncthreads();
  if (!s_last) return;
  if (tid == 0) *ticket = 0u;
  __threadfence();
  const int per = (n_rows + 255) / 256;
  for (int head = 0; head < 2; ++head) {
    const int64_t* am = head ? am1 : am0;
    int64_t* o = out + (int64_t)head * out_stride;
    int64_t* toks = o + 1;
    int* index = reinterpret_cast<int*>(o + 1 + n_rows);
    const int lo = min(tid * per, n_rows), hi = min(lo + per, n_rows);
    int c = 0;
    int64_t prev = lo > 0 ? __ldcg(am + lo - 1) : -1;
    for (int i = lo; i < hi; ++i) {
      int64_t v = __ldcg(am + i);
      if ((i == 0 || v != prev) && v != blank && v != pad) ++c;
      prev = v;
    }
    scount[tid] = c;
    __syncthreads();
    // inclusive scan over 256 counts (Hillis-Steele)
    for (int off = 1; off < 256; off <<= 1) {
      int add = tid >= off ? scount[tid - off] : 0;
      __syncthreads();
      scount[tid] += add;
      __syncthreads();
    }
    int base = scount[tid] - c;
    prev = lo > 0 ? __ldcg(am + lo - 1) : -1;
    for (int i = lo; i < hi; ++i) {
      int64_t v = __ldcg(am + i);
      if ((i == 0 || v != prev) && v != blank && v != pad) {
        toks[base] = v;
        index[base] = i;
        ++base;
      }
      prev = v;
    }
    if (tid == 255) *reinterpret_cast<int*>(o) = scount[255];
    __syncthreads();
  }
}

__global__ void gather_rows_kernel(const int64_t* __restrict__ idx, int idx_offset, const float* __restrict__ table, int C,
                                   float* __restrict__ out) {
  pdl_trigger();
  pdl_wait();
  int r = blockIdx.x;
  int64_t t = idx[r] + idx_offset;
  for (int c = threadIdx.x; c < C; c += blockDim.x) out[(int64_t)r * C + c] = table[t * C + c];
}

__global__ void duration_kernel(const float* __restrict__ logdur, int n, int64_t* __restrict__ dur, int* __restrict__ cumsum) {
  pdl_trigger();
  pdl_wait();
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  int acc = 0;
  cumsum[0] = 0;
  for (int i = 0; i < n; ++i) {
    // torch.clamp(torch.round(torch.exp(x) - 1).long(), min=1)  (agent/tts/codehifigan.py:63-65); round = half-to-even
    float d = rintf(expf(logdur[i]) - 1.0f);
    long long di = (long long)d;
    if (di < 1) di = 1;
    if (di > 100000) di = 100000;
    dur[i] = di;
    acc += (int)di;
    cumsum[i + 1] = acc;
  }
}

__global__ void expand_frames_kernel(const float* __restrict__ emb, const int* __restrict__ cumsum, int U, int f0, int C,
                                     float* __restrict__ out) {
  pdl_trigger();
  pdl_wait();
  int f = f0 + blockIdx.x;
  int lo = 0, hi = U;  // find u with cumsum[u] <= f < cumsum[u+1]
  while (hi - lo > 1) {
    int mid = (lo + hi) >> 1;
    if (cumsum[mid] <= f) lo = mid; else hi = mid;
  }
  for (int c = threadIdx.x; c < C; c += blockDim.x) out[(int64_t)blockIdx.x * C + c] = emb[(int64_t)lo * C + c];
}

__global__ void conv_post_tanh_kernel(const float* __restrict__ x, int L, int C, const float* __restrict__ w, float bias, int k,
                                      float pre_slope, float* __restrict__ out) {
  pdl_trigger();
  pdl_wait();
  int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= L) return;
  int half = (k - 1) >> 1;
  float acc = bias;
  for (int j = 0; j < k; ++j) {
    int p = t - half + j;
    if (p < 0 || p >= L) continue;
    const float* xr = x + (int64_t)p * C;
    for (int c = 0; c < C; ++c) {
      float v = xr[c];
      v = v > 0.f ? v : v * pre_slope;
      acc = fmaf(w[j * C + c], v, acc);
    }
  }
  out[t] = tanhf(acc);
}

}  // namespace

void layer_norm(const float* x, int ldx, float* y, int ldy, const float* gamma, const float* beta, int rows, int C,
                cudaStream_t st) {
  ++g_launches;
  if (rows <= 0) return;
  const int wpb = 8;
  dim3 grid((rows + wpb - 1) / wpb);
  switch (C) {
    case 128: launch_pdl(layer_norm_kernel<4>, dim3(grid), dim3(wpb * 32), 0, st, x, ldx, y, ldy, gamma, beta, rows); break;
    case 256: launch_pdl(layer_norm_kernel<8>, dim3(grid), dim3(wpb * 32), 0, st, x, ldx, y, ldy, gamma, beta, rows); break;
    case 512: launch_pdl(layer_norm_kernel<16>, dim3(grid), dim3(wpb * 32), 0, st, x, ldx, y, ldy, gamma, beta, rows); break;
    case 1024: launch_pdl(layer_norm_kernel<32>, dim3(grid), dim3(wpb * 32), 0, st, x, ldx, y, ldy, gamma, beta, rows); break;
    default: break;  // engine validates C at finalize
  }
}

void depthwise_bn_silu(const float* x, int ldx, const float* w, const float* scale, const float* shift, float* y, int ldy,
                       int B, int T, int t0, int n, int C, int k, int chunk, cudaStream_t st) {
  ++g_launches;
  if (B * n <= 0) return;
  launch_pdl(depthwise_bn_silu_kernel, dim3(B * n), dim3(256), 0, st, x, ldx, w, scale, shift, y, ldy, T, t0, n, C, k, chunk);
}

void scale_rows(float* x, int64_t n, float s, cudaStream_t st) {
  ++g_launches;
  if (n <= 0) return;
  launch_pdl(scale_kernel, dim3((unsigned)((n + 255) / 256)), dim3(256), 0, st, x, n, s);
}

void add3_f32(const float* a, const float* b, const float* c, float* out, int64_t n, cudaStream_t st) {
  ++g_launches;
  if (n <= 0) return;
  const int64_t n4 = n / 4;
  launch_pdl(add3_kernel, dim3((unsigned)((n4 + 255) / 256)), dim3(256), 0, st, (const float4*)a, (const float4*)b, (const float4*)c, (float4*)out, n4);
}

void copy_f32(const float* src, float* dst, int64_t n, cudaStream_t st) {
  ++g_launches;
  if (n <= 0) return;
  launch_pdl(copy_kernel, dim3((unsigned)((n + 255) / 256)), dim3(256), 0, st, src, dst, n);
}

void embed_tokens_pos(const int64_t* tokens, const int* positions_or_null, int pos_offset, const float* emb,
                      const float* pos_table, float scale, float* out, int rows, int C, int pad_idx, cudaStream_t st) {
  ++g_launches;
  if (rows <= 0) return;
  launch_pdl(embed_tokens_pos_kernel, dim3(rows), dim3(128), 0, st, tokens, positions_or_null, pos_offset, emb, pos_table, scale, out, rows, C, pad_idx);
}

void repeat_rows_add(const float* x, int S, int R, int C, const float* addvec_or_null, float* out, cudaStream_t st) {
  ++g_launches;
  if (S * R <= 0) return;
  launch_pdl(repeat_rows_add_kernel, dim3(S * R), dim3(128), 0, st, x, S, R, C, addvec_or_null, out);
}

void argmax_rows(const float* logits, int ld, int rows, int V, const int* masked_cols, int n_masked, int64_t* out_idx,
                 float* out_lprob_or_null, cudaStream_t st) {
  ++g_launches;
  if (rows <= 0) return;
  launch_pdl(argmax_rows_kernel, dim3(rows), dim3(256), 0, st, logits, ld, V, masked_cols, n_masked, out_idx, out_lprob_or_null);
}

void ctc_collapse(const int64_t* argmax, int n, int blank, int pad, int64_t* out_tokens, int* out_index, int* out_count,
                  cudaStream_t st) {
  ++g_launches;
  launch_pdl(ctc_collapse_kernel, dim3(1), dim3(1024), 0, st, argmax, n, blank, pad, out_tokens, out_index, out_count);
}

void ctc_argmax_collapse_pair(const float* logits, int ld, int V, int n_new, int row0, int n_rows, const int* masked, int n_masked, int blank,
                              int pad, int64_t* am0, int64_t* am1, int64_t* out, int out_stride, unsigned* ticket, cudaStream_t st) {
  ++g_launches;
  launch_pdl(ctc_argmax_collapse_pair_kernel, dim3(std::max(1, 2 * n_new)), dim3(256), 0, st, logits, ld, V, n_new, row0, n_rows, masked, n_masked,
             blank, pad, am0, am1, out, out_stride, ticket);
}

// out[i] = sum_k h[k] * x[3 i + k - width], i in [i0, i0 + n): 48 kHz -> 16 kHz windowed-sinc decimation (x zero outside [0, n_in))
__global__ void __launch_bounds__(256) resample_3to1_kernel(const float* __restrict__ x, int64_t n_in, const float* __restrict__ h, int taps,
                                                           int width, int64_t i0, int n, float* __restrict__ out) {
  pdl_trigger();
  pdl_wait();
  __shared__ float hs[64];
  __shared__ float xs[3 * 256 + 64];
  const int tid = threadIdx.x;
  if (tid < taps) hs[tid] = h[tid];
  const int64_t ib = i0 + (int64_t)blockIdx.x * 256;       // first output of this block
  const int64_t base = 3 * ib - width;                      // first input sample the block touches
  const int span = 3 * 255 + taps;                          // inputs touched by 256 outputs
  for (int j = tid; j < span; j += 256) {
    const int64_t p = base + j;
    xs[j] = (p >= 0 && p < n_in) ? x[p] : 0.f;
  }
  __syncthreads();
  const int64_t i = ib + tid;
  if (i >= i0 + n) return;
  float acc = 0.f;
  for (int k = 0; k < taps; ++k) acc = fmaf(hs[k], xs[3 * tid + k], acc);
  out[i] = acc;
}

void resample_3to1(const float* x, int64_t n_in, const float* h, int taps, int width, int64_t i0, int n, float* out, cudaStream_t st) {
  ++g_launches;
  if (n <= 0) return;
  launch_pdl(resample_3to1_kernel, dim3((n + 255) / 256), dim3(256), 0, st, x, n_in, h, taps, width, i0, n, out);
}

void gather_rows(const int64_t* idx, int n, int idx_offset, const float* table, int C, float* out, cudaStream_t st) {
  ++g_launches;
  if (n <= 0) return;
  launch_pdl(gather_rows_kernel, dim3(n), dim3(128), 0, st, idx, idx_offset, table, C, out);
}

void duration_from_log(const float* logdur, int n, int64_t* dur, int* cumsum, cudaStream_t st) {
  ++g_launches;
  launch_pdl(duration_kernel, dim3(1), dim3(32), 0, st, logdur, n, dur, cumsum);
}

void expand_frames(const float* emb, const int* cumsum, int U, int f0, int nf, int C, float* out, cudaStream_t st) {
  ++g_launches;
  if (nf <= 0) return;
  launch_pdl(expand_frames_kernel, dim3(nf), dim3(128), 0, st, emb, cumsum, U, f0, C, out);
}

void conv_post_tanh(const float* x, int L, int C, const float* w, float bias, int k, float pre_slope, float* out,
                    cudaStream_t st) {
  ++g_launches;
  if (L <= 0) return;
  launch_pdl(conv_post_tanh_kernel, dim3((L + 127) / 128), dim3(128), 0, st, x, L, C, w, bias, k, pre_slope, out);
}

}  // namespace ss
