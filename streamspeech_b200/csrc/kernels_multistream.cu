// Kernels of the multi-stream (batched streaming) path: n concurrent utterances share ONE pass over the encoder weights.
//
// Every stream owns a slot of the handle's stream pool (engine_pool.cu): audio, fbank frames, per-layer K / V / conv-input
// caches, encoder output rows and CTC arg-max rows, all at a fixed per-slot stride.  A batched step concatenates the active
// rows of ALL its streams into dense [sum nA][C] activations (stream b at rows row0 .. row0 + nA - 1 of its descriptor; streams
// may differ in nA and in their chunk sizes), so every GEMM of the step is the ordinary linear() over sum nA rows; the kernels here are the
// per-stream (ragged) parts: windows gathered from / rows scattered to the slots, relative-position attention of each stream's
// rows over ITS OWN key / value cache, the chunk-causal depthwise conv over ITS OWN conv-input cache, the 48 -> 16 kHz decimation
// and fbank of each stream's new samples / frames, and the CTC arg-max / collapse per stream.  Arithmetic is that of the
// single-stream kernels (kernels_attn.cu attn_row_kernel, kernels_misc.cu depthwise_bn_silu_kernel / resample_3to1_kernel,
// kernels_fbank.cu); the CTC kernels call the same block_masked_argmax256 / block_ctc_collapse (common.cuh).
#include <algorithm>

#include "common.cuh"
#include "kernels.h"
#include "kernels_multistream.h"

namespace ss {
namespace {

constexpr int HD = 64;
constexpr int MS_NT = 128;

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

// dst[b][r][:] = src_base[slot[b] * slot_stride + (row0[b] + r) * C + :]   (rows gathered from a slot buffer; rows below 0 or at /
// beyond limit[b] read as zero)
__global__ void ms_gather_rows_kernel(const float* __restrict__ src_base, int64_t slot_stride, const MsStream* __restrict__ S, int which_row0,
                                      int rows, int C, float* __restrict__ dst) {
  pdl_trigger();
  pdl_wait();
  const int b = blockIdx.y, r = blockIdx.x;
  const MsStream s = S[b];
  const int p = (which_row0 == 0 ? s.f_lo : s.a0) + r;
  const int lim = which_row0 == 0 ? s.F : s.T;
  const float* src = src_base + (int64_t)s.slot * slot_stride + (int64_t)p * C;
  float* d = dst + ((int64_t)b * rows + r) * C;
  const bool ok = p >= 0 && p < lim;
  for (int c = threadIdx.x * 4; c < C; c += blockDim.x * 4)
    *reinterpret_cast<float4*>(d + c) = ok ? *reinterpret_cast<const float4*>(src + c) : make_float4(0.f, 0.f, 0.f, 0.f);
}

// dst_base[slot[b] * slot_stride + (a0[b] + r) * C + :] = src[row0[b] + r][:], r < nA[b]   (up to three sources -> three slot
// buffers in one launch)
__global__ void ms_scatter_rows_kernel(const float* __restrict__ s0, const float* __restrict__ s1, const float* __restrict__ s2, int lds,
                                       float* __restrict__ d0, float* __restrict__ d1, float* __restrict__ d2, int64_t slot_stride,
                                       const MsStream* __restrict__ S, int C) {
  pdl_trigger();
  pdl_wait();
  const int b = blockIdx.y, r = blockIdx.x;
  const MsStream s = S[b];
  if (r >= s.nA) return;
  const int64_t so = ((int64_t)s.row0 + r) * lds;
  const int64_t dof = (int64_t)s.slot * slot_stride + (int64_t)(s.a0 + r) * C;
  for (int c = threadIdx.x * 4; c < C; c += blockDim.x * 4) {
    *reinterpret_cast<float4*>(d0 + dof + c) = *reinterpret_cast<const float4*>(s0 + so + c);
    if (s1 != nullptr) *reinterpret_cast<float4*>(d1 + dof + c) = *reinterpret_cast<const float4*>(s1 + so + c);
    if (s2 != nullptr) *reinterpret_cast<float4*>(d2 + dof + c) = *reinterpret_cast<const float4*>(s2 + so + c);
  }
}

// Relative-position attention (attn_row_kernel<RELPOS> of kernels_attn.cu): CTA = (active row r, head h, stream b); keys 0 .. lim-1
// of stream b's cache at kc / vc + slot * slot_stride (this layer's [Tcap][D] block), lim = end of the query's attention chunk
// (the stream's own chunk size).  Query / output row row0[b] + r; CTAs with r >= nA[b] exit before any barrier.
__global__ void __launch_bounds__(MS_NT) ms_relpos_attn_kernel(const float* __restrict__ q, int ldq, const float* __restrict__ kc,
                                                               const float* __restrict__ vc, int64_t slot_stride, int D,
                                                               const float* __restrict__ pos, int Tpos, const float* __restrict__ bias_u,
                                                               const float* __restrict__ bias_v, float* __restrict__ out, int ldo,
                                                               const MsStream* __restrict__ S) {
  pdl_trigger();
  pdl_wait();
  extern __shared__ __align__(16) float smem[];
  float* Sc = smem;  // [T]
  __shared__ __align__(16) float qa[HD], qb2[HD];
  __shared__ __align__(16) float part[4][HD];
  __shared__ float red[4];
  const int r = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const MsStream s = S[b];
  if (r >= s.nA) return;
  const int chunk = s.attn_chunk;
  const int i = s.a0 + r;
  const int lim = chunk > 0 ? min((i / chunk + 1) * chunk, s.T) : s.T;
  const int n = max(1, lim);
  const int64_t row = (int64_t)s.row0 + r;
  const float* qp = q + row * ldq + h * HD;
  const float* kb = kc + (int64_t)s.slot * slot_stride + h * HD;
  const float* vb = vc + (int64_t)s.slot * slot_stride + h * HD;
  if (threadIdx.x < HD) {
    const float val = qp[threadIdx.x];
    qa[threadIdx.x] = val + bias_u[h * HD + threadIdx.x];
    qb2[threadIdx.x] = val + bias_v[h * HD + threadIdx.x];
  }
  __syncthreads();
  float mx = -INFINITY;
  for (int j = threadIdx.x; j < n; j += MS_NT) {
    float sc = dot64(qa, kb + (int64_t)j * D);
    sc = (sc + dot64(qb2, pos + (int64_t)(i - j + Tpos - 1) * D + h * HD)) * 0.125f;
    Sc[j] = sc;
    mx = fmaxf(mx, sc);
  }
  mx = block_max128(mx, red);
  float sum = 0.f;
  for (int j = threadIdx.x; j < n; j += MS_NT) {
    const float e = expf(Sc[j] - mx);
    Sc[j] = e;
    sum += e;
  }
  sum = block_sum128(sum, red);
  __syncthreads();
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float a0 = 0.f, a1 = 0.f;
#pragma unroll 4
  for (int j = w; j < n; j += 4) {
    const float p = Sc[j];
    const float2 vv = *reinterpret_cast<const float2*>(vb + (int64_t)j * D + 2 * lane);
    a0 = fmaf(p, vv.x, a0);
    a1 = fmaf(p, vv.y, a1);
  }
  part[w][2 * lane] = a0;
  part[w][2 * lane + 1] = a1;
  __syncthreads();
  if (threadIdx.x < HD) {
    const float t = (part[0][threadIdx.x] + part[1][threadIdx.x]) + (part[2][threadIdx.x] + part[3][threadIdx.x]);
    out[row * ldo + h * HD + threadIdx.x] = t / sum;
  }
}

// depthwise chunk-causal conv + BN + SiLU over stream b's conv-input cache (depthwise_bn_silu_kernel of kernels_misc.cu), with the
// stream's own conv chunk; output row row0[b] + r
__global__ void ms_depthwise_kernel(const float* __restrict__ gc, int64_t slot_stride, const float* __restrict__ w, const float* __restrict__ scale,
                                    const float* __restrict__ shift, float* __restrict__ y, int ldy, const MsStream* __restrict__ S, int C, int k) {
  pdl_trigger();
  pdl_wait();
  const int b = blockIdx.y, r = blockIdx.x;
  const MsStream s = S[b];
  if (r >= s.nA) return;
  const int chunk = s.conv_chunk;
  const int t = s.a0 + r;
  const int half = (k - 1) >> 1;
  const int lim = chunk > 0 ? min(s.T, (t / chunk + 1) * chunk) : s.T;
  const float* x = gc + (int64_t)s.slot * slot_stride;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float acc = 0.f;
    for (int j0 = 0; j0 < k; j0 += 8) {
      float xv[8], wv[8];
#pragma unroll
      for (int jj = 0; jj < 8; ++jj) {
        const int j = j0 + jj, p = t - half + j;
        const bool ok = j < k && p >= 0 && p < lim;
        xv[jj] = ok ? x[(int64_t)p * C + c] : 0.f;
        wv[jj] = ok ? w[j * C + c] : 0.f;
      }
#pragma unroll
      for (int jj = 0; jj < 8; ++jj) acc = fmaf(wv[jj], xv[jj], acc);
    }
    const float v = acc * scale[c] + shift[c];
    y[((int64_t)s.row0 + r) * ldy + c] = v / (1.0f + expf(-v));
  }
}

// ---- fbank of the new frames of every stream (fbank_kernel of kernels_fbank.cu with a per-stream descriptor and the mel bank
// transposed to [257][80], so that the 80 mel threads read coalesced rows).  The 400 samples of a frame arrive in shared memory by
// ONE bulk-async copy (cp.async.bulk, the TMA 1-D path: 1600 contiguous bytes at a 640-byte-aligned offset) signalled on an mbarrier.
constexpr int FRAME = 400, SHIFT = 160, NFFT = 512, NBIN = 257, NMEL = 80;

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__global__ void __launch_bounds__(256) ms_fbank_kernel(const float* __restrict__ audio_base, int64_t audio_stride, float* __restrict__ feat_base,
                                                       int64_t feat_stride, const MsStream* __restrict__ S, const float* __restrict__ melT,
                                                       const float* __restrict__ window, const float* __restrict__ cmvn_mean,
                                                       const float* __restrict__ cmvn_std) {
  pdl_trigger();
  pdl_wait();
  __shared__ float re[NFFT], im[NFFT];
  __shared__ float twc[NFFT / 2], tws[NFFT / 2];
  __shared__ __align__(128) float frame[FRAME];
  __shared__ float red[32];
  __shared__ __align__(8) unsigned long long mbar;
  const int tid = threadIdx.x;
  const MsStream s = S[blockIdx.y];
  if ((int)blockIdx.x >= s.n_new_frames) return;
  const int f = s.frame0 + blockIdx.x;
  const float* src = audio_base + (int64_t)s.slot * audio_stride + (int64_t)f * SHIFT;
  if (tid == 0) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(smem_u32(&mbar)));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (tid == 0) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(&mbar)), "r"(FRAME * 4) : "memory");
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(frame)), "l"(src),
                 "r"(FRAME * 4), "r"(smem_u32(&mbar))
                 : "memory");
  }
  {
    float sn, cs;
    sincospif(-(float)tid / 256.0f, &sn, &cs);  // exp(-2*pi*i*tid/512), overlaps the copy
    twc[tid] = cs;
    tws[tid] = sn;
  }
  {  // wait for the bulk copy (phase 0)
    uint32_t done = 0;
    while (!done) {
      asm volatile(
          "{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], 0;\n\tselp.u32 %0, 1, 0, p;\n\t}"
          : "=r"(done)
          : "r"(smem_u32(&mbar))
          : "memory");
    }
  }
  float sum = 0.f;
  for (int j = tid; j < FRAME; j += 256) {
    const float v = frame[j] * 32768.0f;
    sum += v;
  }
  const float mean = block_sum(sum, red) / (float)FRAME;
  for (int j = tid; j < NFFT; j += 256) {
    float v = 0.f;
    if (j < FRAME) {
      const float x0 = frame[j] * 32768.0f - mean;
      const float xm = frame[j > 0 ? j - 1 : 0] * 32768.0f - mean;
      v = (x0 - 0.97f * xm) * window[j];
    }
    const int r = __brev((unsigned)j) >> (32 - 9);
    re[r] = v;
    im[r] = 0.f;
  }
  __syncthreads();
#pragma unroll
  for (int stage = 0; stage < 9; ++stage) {
    const int half = 1 << stage;
    const int grp = tid >> stage, pos = tid & (half - 1);
    const int i = (grp << (stage + 1)) + pos, j = i + half;
    const int tw = pos << (8 - stage);
    const float wr = twc[tw], wi = tws[tw];
    const float xr = re[j], xi = im[j];
    const float tr = wr * xr - wi * xi, ti = wr * xi + wi * xr;
    const float ur = re[i], ui = im[i];
    re[i] = ur + tr;
    im[i] = ui + ti;
    re[j] = ur - tr;
    im[j] = ui - ti;
    __syncthreads();
  }
  for (int k = tid; k < NBIN; k += 256) {
    const float a = sqrtf(re[k] * re[k] + im[k] * im[k]);
    frame[k] = a * a;
  }
  __syncthreads();
  if (tid < NMEL) {
    float acc = 0.f;
    for (int k = 0; k < NBIN; ++k) acc = fmaf(frame[k], melT[k * NMEL + tid], acc);
    float v = logf(fmaxf(acc, 1.1920928955078125e-07f));
    if (cmvn_mean) v = (v - cmvn_mean[tid]) / cmvn_std[tid];
    feat_base[(int64_t)s.slot * feat_stride + (int64_t)f * NMEL + tid] = v;
  }
}

// ---- 48 -> 16 kHz decimation of the new samples of every stream (resample_3to1_kernel of kernels_misc.cu with a per-stream
// descriptor): block = (256 outputs, stream b).  Same taps, same shared-memory window, same fmaf order over k and zeros outside
// [0, n48), so every 16 kHz sample equals, bit for bit, what ss_resample_48k_to_16k produces from the same 48 kHz prefix.
__global__ void __launch_bounds__(256) ms_resample_3to1_kernel(const float* __restrict__ a48_base, int64_t a48_stride, float* __restrict__ a16_base,
                                                              int64_t a16_stride, const MsStream* __restrict__ S, const float* __restrict__ h,
                                                              int taps, int width) {
  pdl_trigger();
  pdl_wait();
  __shared__ float hs[64];
  __shared__ float xs[3 * 256 + 64];
  const int tid = threadIdx.x;
  const MsStream s = S[blockIdx.y];
  if ((int)blockIdx.x * 256 >= s.n16_new) return;
  if (tid < taps) hs[tid] = h[tid];
  const float* x = a48_base + (int64_t)s.slot * a48_stride;
  const int64_t ib = s.n16_done + (int64_t)blockIdx.x * 256;  // first output of this block
  const int64_t base = 3 * ib - width;                         // first input sample the block touches
  const int span = 3 * 255 + taps;                             // inputs touched by 256 outputs
  for (int j = tid; j < span; j += 256) {
    const int64_t p = base + j;
    xs[j] = (p >= 0 && p < s.n48) ? x[p] : 0.f;
  }
  __syncthreads();
  const int64_t i = ib + tid;
  if (i >= s.n16_done + s.n16_new) return;
  float acc = 0.f;
  for (int k = 0; k < taps; ++k) acc = fmaf(hs[k], xs[3 * tid + k], acc);
  a16_base[(int64_t)s.slot * a16_stride + i] = acc;
}

// arg-max (block_masked_argmax256) of the new rows of every stream: block = (row r, stream b, head), logits row = (row0 + r),
// r < nA, columns [head * V, head * V + V); result -> am_base[(slot * 2 + head) * am_stride + a0 + r]
__global__ void __launch_bounds__(256) ms_ctc_argmax_kernel(const float* __restrict__ logits, int ld, int V, const int* __restrict__ masked,
                                                            int n_masked, int64_t* __restrict__ am_base, int64_t am_stride,
                                                            const MsStream* __restrict__ S) {
  pdl_trigger();
  pdl_wait();
  const int r = blockIdx.x, b = blockIdx.y, head = blockIdx.z;
  const MsStream s = S[b];
  if (r >= s.nA) return;
  const int bi = block_masked_argmax256(logits + ((int64_t)s.row0 + r) * ld + head * V, V, masked, n_masked);
  if (threadIdx.x == 0) am_base[((int64_t)s.slot * 2 + head) * am_stride + s.a0 + r] = bi;
}

// CTC collapse (block_ctc_collapse) of stream b / head over rows 0 .. T-1 of its arg-max rows -> out + S[b].out_off + head * (2 T + 2):
// [count (int32) | tokens[T] int64 | index[T] int32]
__global__ void __launch_bounds__(256) ms_ctc_collapse_kernel(const int64_t* __restrict__ am_base, int64_t am_stride, const MsStream* __restrict__ S,
                                                              int blank, int pad, int64_t* __restrict__ out) {
  pdl_trigger();
  pdl_wait();
  __shared__ int wsum[32];
  const int head = blockIdx.y;
  const MsStream s = S[blockIdx.x];
  const int n = s.T;
  int64_t* o = out + s.out_off + (int64_t)head * (2 * n + 2);
  block_ctc_collapse(am_base + ((int64_t)s.slot * 2 + head) * am_stride, 1, n, blank, pad, o + 1, reinterpret_cast<int*>(o + 1 + n),
                     reinterpret_cast<int*>(o), wsum);
}

}  // namespace

void ms_gather_rows(const float* src_base, int64_t slot_stride, const MsStream* S, int n, int which, int rows, int C, float* dst, cudaStream_t st) {
  ++g_launches;
  if (n * rows <= 0) return;
  launch_pdl(ms_gather_rows_kernel, dim3(rows, n), dim3(64), 0, st, src_base, slot_stride, S, which, rows, C, dst);
}

void ms_scatter_rows(const float* s0, const float* s1, const float* s2, int lds, float* d0, float* d1, float* d2, int64_t slot_stride, const MsStream* S,
                     int n, int max_nA, int C, cudaStream_t st) {
  ++g_launches;
  if (n * max_nA <= 0) return;
  launch_pdl(ms_scatter_rows_kernel, dim3(max_nA, n), dim3(64), 0, st, s0, s1, s2, lds, d0, d1, d2, slot_stride, S, C);
}

void ms_relpos_attention(const float* q, int ldq, const float* kc, const float* vc, int64_t slot_stride, int D, const float* pos, int Tpos,
                         const float* bias_u, const float* bias_v, float* out, int ldo, const MsStream* S, int n, int max_nA, int H, int Tmax,
                         cudaStream_t st) {
  ++g_launches;
  if (n * max_nA <= 0) return;
  const size_t smem = (size_t)((Tmax + 3) & ~3) * sizeof(float);
  if (smem > 40 * 1024 && first_time_on_device((const void*)ms_relpos_attn_kernel))
    cudaFuncSetAttribute(ms_relpos_attn_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024);
  launch_pdl(ms_relpos_attn_kernel, dim3(max_nA, H, n), dim3(MS_NT), smem, st, q, ldq, kc, vc, slot_stride, D, pos, Tpos, bias_u, bias_v, out, ldo, S);
}

void ms_depthwise(const float* gc, int64_t slot_stride, const float* w, const float* scale, const float* shift, float* y, int ldy, const MsStream* S, int n,
                  int max_nA, int C, int k, cudaStream_t st) {
  ++g_launches;
  if (n * max_nA <= 0) return;
  launch_pdl(ms_depthwise_kernel, dim3(max_nA, n), dim3(256), 0, st, gc, slot_stride, w, scale, shift, y, ldy, S, C, k);
}

void ms_fbank(const float* audio_base, int64_t audio_stride, float* feat_base, int64_t feat_stride, const MsStream* S, int n, int max_new_frames,
              const float* melT, const float* window, const float* cmvn_mean, const float* cmvn_std, cudaStream_t st) {
  ++g_launches;
  if (n <= 0 || max_new_frames <= 0) return;
  launch_pdl(ms_fbank_kernel, dim3(max_new_frames, n), dim3(256), 0, st, audio_base, audio_stride, feat_base, feat_stride, S, melT, window, cmvn_mean,
             cmvn_std);
}

void ms_resample_3to1(const float* a48_base, int64_t a48_stride, float* a16_base, int64_t a16_stride, const MsStream* S, int n, int max_new,
                      const float* h, int taps, int width, cudaStream_t st) {
  ++g_launches;
  if (n <= 0 || max_new <= 0) return;
  launch_pdl(ms_resample_3to1_kernel, dim3((max_new + 255) / 256, n), dim3(256), 0, st, a48_base, a48_stride, a16_base, a16_stride, S, h, taps, width);
}

void ms_ctc_argmax(const float* logits, int ld, int V, const int* masked, int n_masked, int64_t* am_base, int64_t am_stride, const MsStream* S, int n,
                   int max_nA, int heads, cudaStream_t st) {
  ++g_launches;
  if (n * max_nA <= 0) return;
  launch_pdl(ms_ctc_argmax_kernel, dim3(max_nA, n, heads), dim3(256), 0, st, logits, ld, V, masked, n_masked, am_base, am_stride, S);
}

void ms_ctc_collapse(const int64_t* am_base, int64_t am_stride, const MsStream* S, int n, int heads, int blank, int pad, int64_t* out, cudaStream_t st) {
  ++g_launches;
  if (n <= 0) return;
  launch_pdl(ms_ctc_collapse_kernel, dim3(n, heads), dim3(256), 0, st, am_base, am_stride, S, blank, pad, out);
}

}  // namespace ss
