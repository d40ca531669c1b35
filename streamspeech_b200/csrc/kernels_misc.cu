// Streaming / scan kernels of the path: LayerNorm, depthwise chunk-causal conv + BN + SiLU, embedding
// gathers, arg-max over the vocabulary, CTC collapse, duration rounding, frame expansion, conv_post.
// All HBM-bound: coalesced row-major accesses, warp-shuffle reductions, no re-reads.
#include <algorithm>

#include "common.cuh"
#include "kernels.h"

namespace ss {
unsigned long long g_launches = 0;
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
  int r = blockIdx.x;  // output row (b*S + s)*R + rr
  int s = r / R;
  const float* xr = x + (int64_t)s * C;
  if (addvec) addvec += (int64_t)(r / (S * R)) * C;  // sample b's row
  // N1 quirk: position index comes from the VALUE x[t, b, 0]: != 1.0 -> pad+1+b (addvec), == 1.0 -> pad (zero row)
  bool add = addvec != nullptr && xr[0] != 1.0f;
  for (int c = threadIdx.x; c < C; c += blockDim.x) out[(int64_t)r * C + c] = xr[c] + (add ? addvec[c] : 0.f);
}

// arg-max rows (block_masked_argmax256), one CTA of 256 threads per row
__global__ void argmax_rows_kernel(const float* __restrict__ logits, int ld, int V, const int* __restrict__ masked, int n_masked,
                                   int64_t* __restrict__ out_idx) {
  pdl_trigger();
  pdl_wait();
  const int bi = block_masked_argmax256(logits + (int64_t)blockIdx.x * ld, V, masked, n_masked);
  if (threadIdx.x == 0) out_idx[blockIdx.x] = bi;
}

// argmax_rows_kernel plus the winner's log-probability over all V columns (the offline unit decoder's positional scores,
// ctc_generator.py:54-61): the same reduction, so the index equals argmax_rows_kernel's bit for bit, and the same bytes read
__global__ void argmax_lprob_rows_kernel(const float* __restrict__ logits, int ld, int V, const int* __restrict__ masked, int n_masked,
                                         int64_t* __restrict__ out_idx, float* __restrict__ out_lprob) {
  pdl_trigger();
  pdl_wait();
  float lp;
  const int bi = block_masked_argmax_lprob256(logits + (int64_t)blockIdx.x * ld, V, masked, n_masked, lp);
  if (threadIdx.x == 0) {
    out_idx[blockIdx.x] = bi;
    out_lprob[blockIdx.x] = lp;
  }
}

// CTC collapse (block_ctc_collapse), one CTA of 1024 threads per sequence s = blockIdx.x: entries am[((s / inner) * n + i) * inner +
// s % inner] for i < n (or < n_seq[s / inner]), outputs at s * seg_stride int64 words
__global__ void ctc_collapse_kernel(const int64_t* __restrict__ am, int n, const int* __restrict__ n_seq, int inner, int blank, int pad,
                                    int64_t* __restrict__ toks, int* __restrict__ index, int* __restrict__ count, int64_t seg_stride) {
  pdl_trigger();
  pdl_wait();
  __shared__ int wsum[32];
  const int s = blockIdx.x;
  block_ctc_collapse(am + (int64_t)(s / inner) * n * inner + s % inner, inner, n_seq ? n_seq[s / inner] : n, blank, pad, toks + s * seg_stride,
                     index ? index + 2 * s * seg_stride : nullptr, count + 2 * s * seg_stride, wsum);
}

// Both CTC heads of one policy() call after the fused [rows][2V] projection: block b = (head, new row) computes the arg-max; the
// LAST block to finish (ticket) then collapses both arg-max sequences into the packed outputs
//   out[head] = [count (int32 in the first int64) | tokens[n_rows] int64 | index[n_rows] int32], stride out_stride int64 words.
__global__ void __launch_bounds__(256) ctc_argmax_collapse_pair_kernel(const float* __restrict__ logits, int ld, int V, int n_new, int row0,
                                                                      int n_rows, const int* __restrict__ masked, int n_masked, int blank,
                                                                      int pad, int64_t* am0, int64_t* am1, int64_t* out, int out_stride,
                                                                      unsigned* ticket) {
  pdl_trigger();
  pdl_wait();
  __shared__ int wsum[32];
  __shared__ unsigned s_last;
  const int tid = threadIdx.x;
  if ((int)blockIdx.x < 2 * n_new) {
    const int head = blockIdx.x / n_new, r = blockIdx.x - head * n_new;
    const int bi = block_masked_argmax256(logits + (int64_t)r * ld + head * V, V, masked, n_masked);
    if (tid == 0) (head ? am1 : am0)[row0 + r] = bi;
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
  for (int head = 0; head < 2; ++head) {
    int64_t* o = out + (int64_t)head * out_stride;
    block_ctc_collapse(head ? am1 : am0, 1, n_rows, blank, pad, o + 1, reinterpret_cast<int*>(o + 1 + n_rows), reinterpret_cast<int*>(o), wsum);
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

__global__ void gather_codes_ragged_kernel(const int64_t* __restrict__ codes, VocSeqs q, int rows_per_seq, const float* __restrict__ table,
                                           int C, float* __restrict__ emb) {
  pdl_trigger();
  pdl_wait();
  const int s = blockIdx.y, i = blockIdx.x;
  const bool valid = i < q.s[s].U;
  const int64_t t = valid ? codes[q.s[s].c0 - s + i] : 0;
  float* o = emb + (int64_t)(q.s[s].u0 + i) * C;
  for (int c = threadIdx.x; c < C; c += blockDim.x) o[c] = valid ? table[t * C + c] : 0.f;
}

__global__ void zero_pad_rows_kernel(float* __restrict__ x, VocSeqs q, int rows_per_seq, int C) {
  pdl_trigger();
  pdl_wait();
  const int s = blockIdx.y, i = blockIdx.x;
  if (i < q.s[s].U) return;
  float* o = x + (int64_t)(q.s[s].u0 + i) * C;
  for (int c = threadIdx.x; c < C; c += blockDim.x) o[c] = 0.f;
}

__global__ void duration_ragged_kernel(const float* __restrict__ logdur, VocSeqs q, int64_t* __restrict__ dur, int* __restrict__ cumsum) {
  pdl_trigger();
  pdl_wait();
  if (threadIdx.x != 0) return;
  const int s = blockIdx.x;
  const int n = q.s[s].U;
  const float* ld = logdur ? logdur + q.s[s].u0 : nullptr;
  int64_t* d = dur + (q.s[s].c0 - s);
  int* cs = cumsum + q.s[s].c0;
  int acc = 0;
  cs[0] = 0;
  for (int i = 0; i < n; ++i) {
    // torch.clamp(torch.round(torch.exp(x) - 1).long(), min=1)  (agent/tts/codehifigan.py:63-65); round = half-to-even
    long long di = 1;
    if (ld) {
      float f = rintf(expf(ld[i]) - 1.0f);
      di = (long long)f;
      if (di < 1) di = 1;
      if (di > 100000) di = 100000;
    }
    d[i] = di;
    acc += (int)di;
    cs[i + 1] = acc;
  }
}

__global__ void expand_frames_ragged_kernel(const float* __restrict__ emb, const int* __restrict__ cumsum, VocSeqs q, int C,
                                            float* __restrict__ out) {
  pdl_trigger();
  pdl_wait();
  const int r = blockIdx.x;  // output row
  int s = 0;
  while (s + 1 < q.n && r >= q.s[s + 1].row0) ++s;
  const int* cs = cumsum + q.s[s].c0;
  const int f = q.s[s].f_lo + (r - q.s[s].row0);
  int lo = 0, hi = q.s[s].U;  // find u with cumsum[u] <= f < cumsum[u+1]
  while (hi - lo > 1) {
    int mid = (lo + hi) >> 1;
    if (cs[mid] <= f) lo = mid; else hi = mid;
  }
  const float* e = emb + (int64_t)(q.s[s].u0 + lo) * C;
  for (int c = threadIdx.x; c < C; c += blockDim.x) out[(int64_t)r * C + c] = e[c];
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

namespace {

// layer_norm_kernel<n> for n in [1, N]: C = 32 n
template <int N>
bool launch_layer_norm(int n, dim3 grid, dim3 block, cudaStream_t st, const float* x, int ldx, float* y, int ldy, const float* gamma,
                       const float* beta, int rows) {
  if (n == N) {
    launch_pdl(layer_norm_kernel<N>, grid, block, 0, st, x, ldx, y, ldy, gamma, beta, rows);
    return true;
  }
  if constexpr (N > 1) return launch_layer_norm<N - 1>(n, grid, block, st, x, ldx, y, ldy, gamma, beta, rows);
  return false;
}

}  // namespace

bool layer_norm_supported(int C) { return C >= 32 && C <= 1024 && C % 32 == 0; }

bool layer_norm(const float* x, int ldx, float* y, int ldy, const float* gamma, const float* beta, int rows, int C,
                cudaStream_t st) {
  if (!layer_norm_supported(C)) return false;
  ++g_launches;
  if (rows <= 0) return true;
  const int wpb = 8;
  return launch_layer_norm<32>(C / 32, dim3((rows + wpb - 1) / wpb), dim3(wpb * 32), st, x, ldx, y, ldy, gamma, beta, rows);
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

void repeat_rows_add(const float* x, int S, int R, int C, const float* addvec_or_null, float* out, int B, cudaStream_t st) {
  ++g_launches;
  if (S * R <= 0 || B <= 0) return;
  launch_pdl(repeat_rows_add_kernel, dim3(B * S * R), dim3(128), 0, st, x, S, R, C, addvec_or_null, out);
}

void argmax_rows(const float* logits, int ld, int rows, int V, const int* masked_cols, int n_masked, int64_t* out_idx, cudaStream_t st) {
  ++g_launches;
  if (rows <= 0) return;
  launch_pdl(argmax_rows_kernel, dim3(rows), dim3(256), 0, st, logits, ld, V, masked_cols, n_masked, out_idx);
}

void argmax_lprob_rows(const float* logits, int ld, int rows, int V, const int* masked_cols, int n_masked, int64_t* out_idx, float* out_lprob,
                       cudaStream_t st) {
  ++g_launches;
  if (rows <= 0) return;
  launch_pdl(argmax_lprob_rows_kernel, dim3(rows), dim3(256), 0, st, logits, ld, V, masked_cols, n_masked, out_idx, out_lprob);
}

void ctc_collapse_segments(const int64_t* argmax, int n, int inner, int n_seg, int blank, int pad, int64_t* out_tokens, int* out_index,
                           int* out_count, int64_t seg_stride, cudaStream_t st, const int* n_seq_dev) {
  ++g_launches;
  if (n_seg <= 0) return;
  launch_pdl(ctc_collapse_kernel, dim3(n_seg), dim3(1024), 0, st, argmax, n, n_seq_dev, inner, blank, pad, out_tokens, out_index, out_count,
             seg_stride);
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

void gather_codes_ragged(const int64_t* codes, const VocSeqs& q, int rows_per_seq, const float* table, int C, float* emb, cudaStream_t st) {
  ++g_launches;
  if (q.n <= 0 || rows_per_seq <= 0) return;
  launch_pdl(gather_codes_ragged_kernel, dim3(rows_per_seq, q.n), dim3(128), 0, st, codes, q, rows_per_seq, table, C, emb);
}

void zero_pad_rows(float* x, const VocSeqs& q, int rows_per_seq, int C, cudaStream_t st) {
  ++g_launches;
  if (q.n <= 0 || rows_per_seq <= 0) return;
  launch_pdl(zero_pad_rows_kernel, dim3(rows_per_seq, q.n), dim3(128), 0, st, x, q, rows_per_seq, C);
}

void duration_from_log_ragged(const float* logdur, const VocSeqs& q, int64_t* dur, int* cumsum, cudaStream_t st) {
  ++g_launches;
  if (q.n <= 0) return;
  launch_pdl(duration_ragged_kernel, dim3(q.n), dim3(32), 0, st, logdur, q, dur, cumsum);
}

void expand_frames_ragged(const float* emb, const int* cumsum, const VocSeqs& q, int total_rows, int C, float* out, cudaStream_t st) {
  ++g_launches;
  if (q.n <= 0 || total_rows <= 0) return;
  launch_pdl(expand_frames_ragged_kernel, dim3(total_rows), dim3(128), 0, st, emb, cumsum, q, C, out);
}

void conv_post_tanh(const float* x, int L, int C, const float* w, float bias, int k, float pre_slope, float* out,
                    cudaStream_t st) {
  ++g_launches;
  if (L <= 0) return;
  launch_pdl(conv_post_tanh_kernel, dim3((L + 127) / 128), dim3(128), 0, st, x, L, C, w, bias, k, pre_slope, out);
}

}  // namespace ss
