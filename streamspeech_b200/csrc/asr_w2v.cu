// The ASR-BLEU transcriber (include/streamspeech_b200.h, ss_asr_*): fairseq's Wav2VecCtc forward pass
// (fairseq/models/wav2vec/wav2vec2.py, wav2vec2_asr.py) and the beam-1 CTC rule of asr_bleu/utils.py, on its own handle.
//   extractor layer 0 (C_in = 1)      : asr_conv0_kernel, direct conv + bias + LayerNorm over channels + GELU in one CTA per frame
//   extractor layers 1 ..             : strided implicit GEMM (gemm_conv, fp32 FMA) + asr_ln_gelu_kernel
//   feature LayerNorm + projection    : layer_norm + wgmma linear (bf16x3)
//   grouped positional conv           : one implicit GEMM per group (gemm_conv, frames >= the sample's length read as zero) with
//                                       the GELU and the residual add in its epilogue
//   pre-LN transformer layers         : layer_norm + wgmma linears (fused Q|K|V, GELU FFN, residual epilogues) + mha_attention
//                                       (tile kernel, per-sample key lengths, no length limit)
//   final LayerNorm + proj            : layer_norm + wgmma linear, then asr_argmax_collapse_kernel (one CTA per utterance)
// Batch invariance: the utterances of a group are padded to its longest; no GEMM splits K (each output's sum runs over K in one
// order whatever the row count), the attention always takes the tile kernel and every other kernel is per row, so an utterance's
// emissions do not depend on what shares the call.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <string>

#include "common.cuh"
#include "engine.h"

using namespace ss;

namespace {

constexpr int kBlank = 0;  // "<s>": tokens[0] of the letter dictionary (utils.py:202, blank_token = tokens[0])
constexpr int kUnk = 3;    // "<unk>": never emitted (unk_score = -inf)
constexpr float kLnEps = 1e-5f;

__device__ __forceinline__ float gelu_erf(float x) { return 0.5f * x * (1.0f + erff(x * 0.70710678118654752f)); }

// LayerNorm over the C values one per thread (C = blockDim.x), then GELU; mean first, then the mean of squared deviations (F.layer_norm)
__device__ __forceinline__ float block_ln_gelu(float v, float g, float b, int C, float* red) {
  const float mean = block_sum(v, red) / (float)C;
  const float d = v - mean;
  const float var = block_sum(d * d, red) / (float)C;
  return gelu_erf(d * rsqrtf(var + kLnEps) * g + b);
}

// F.layer_norm(wav, wav.shape): one CTA per utterance; sums in double, so the statistics do not depend on the reduction order
__global__ void __launch_bounds__(1024) asr_wave_norm_kernel(const float* __restrict__ x, const int64_t* __restrict__ off, float* __restrict__ y) {
  pdl_trigger();
  pdl_wait();
  __shared__ double red[32];
  const int64_t o = off[blockIdx.x], n = off[blockIdx.x + 1] - o;
  auto bsum = [&](double v) {
    for (int s = 16; s > 0; s >>= 1) v += __shfl_xor_sync(0xffffffffu, v, s);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    double t = 0.0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t += red[w];
    return t;
  };
  double s = 0.0;
  for (int64_t i = threadIdx.x; i < n; i += blockDim.x) s += x[o + i];
  const double mean = bsum(s) / (double)n;
  double q = 0.0;
  for (int64_t i = threadIdx.x; i < n; i += blockDim.x) {
    const double d = x[o + i] - mean;
    q += d * d;
  }
  const double var = bsum(q) / (double)n;
  const float m = (float)mean, r = (float)(1.0 / sqrt(var + (double)kLnEps));
  for (int64_t i = threadIdx.x; i < n; i += blockDim.x) y[o + i] = (x[o + i] - m) * r;
}

// extractor layer 0: out[b][t][c] = GELU(LN_c(bias[c] + sum_j w[c][j] * x_b[t * stride + j])); grid (Lmax, B), C threads
__global__ void __launch_bounds__(1024) asr_conv0_kernel(const float* __restrict__ x, const int64_t* __restrict__ off, const int* __restrict__ L_out,
                                                         const float* __restrict__ w, const float* __restrict__ bias, const float* __restrict__ g,
                                                         const float* __restrict__ beta, int k, int stride, int Lmax, float* __restrict__ out) {
  pdl_trigger();
  pdl_wait();
  __shared__ float red[32];
  extern __shared__ float xs[];
  const int b = blockIdx.y, t = blockIdx.x, C = blockDim.x, c = threadIdx.x;
  if (t >= L_out[b]) return;
  const float* xb = x + off[b] + (int64_t)t * stride;
  for (int j = c; j < k; j += C) xs[j] = xb[j];
  __syncthreads();
  float acc = 0.f;
  for (int j = 0; j < k; ++j) acc = fmaf(w[c * k + j], xs[j], acc);
  acc += bias[c];
  out[((int64_t)b * Lmax + t) * C + c] = block_ln_gelu(acc, g[c], beta[c], C, red);
}

// in place: x[r] = GELU(LN(x[r])) over rows of C = blockDim.x channels
__global__ void __launch_bounds__(1024) asr_ln_gelu_kernel(float* __restrict__ x, const float* __restrict__ g, const float* __restrict__ beta) {
  pdl_trigger();
  pdl_wait();
  __shared__ float red[32];
  const int C = blockDim.x, c = threadIdx.x;
  float* row = x + (int64_t)blockIdx.x * C;
  row[c] = block_ln_gelu(row[c], g[c], beta[c], C, red);
}

// per utterance b (one CTA of 1024 threads): arg-max of its T_b rows of logits [Tmax][V] with <unk> excluded, first index on ties, into
// am[b][Tmax]; then the CTC collapse into packed[b * stride] = [count | tokens]
__global__ void __launch_bounds__(1024) asr_argmax_collapse_kernel(const float* __restrict__ logits, int V, int Tmax, const int* __restrict__ T,
                                                                   int64_t* am, int64_t* __restrict__ packed, int64_t stride) {
  pdl_trigger();
  pdl_wait();
  __shared__ int wsum[32];
  const int b = blockIdx.x, lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int n = T[b];
  int64_t* amb = am + (int64_t)b * Tmax;
  for (int r = w; r < n; r += 32) {
    const float* row = logits + ((int64_t)b * Tmax + r) * V;
    float best = -INFINITY;
    int bi = 0x7fffffff;
    for (int c = lane; c < V; c += 32) {
      const float v = row[c];
      if (c != kUnk && (v > best || (v == best && c < bi))) {
        best = v;
        bi = c;
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, best, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (ov > best || (ov == best && oi < bi)) {
        best = ov;
        bi = oi;
      }
    }
    if (lane == 0) amb[r] = bi;
  }
  __threadfence_block();
  __syncthreads();
  int64_t* out = packed + (int64_t)b * stride;
  block_ctc_collapse(amb, 1, n, kBlank, kBlank, out + 1, nullptr, reinterpret_cast<int*>(out), wsum);
}

}  // namespace

struct ss_asr {
  int device = 0;
  ss_asr_config cfg{};
  std::string err;
  bool finalized = false;
  std::map<std::string, HostTensor> host;
  std::vector<void*> dev_allocs;
  // sizes (from the shapes)
  int n_conv = 0, C = 0, D = 0, F = 0, H = 0, V = 0, pos_k = 0, pos_groups = 0, max_frames = 0;
  int conv_k[SS_ASR_MAX_CONV] = {0};
  // weights
  float* conv_w[SS_ASR_MAX_CONV] = {nullptr};  // layer 0 [C][k]; layers >= 1 tap-major [C][k * C]
  float* conv_b[SS_ASR_MAX_CONV] = {nullptr};
  LNorm conv_ln[SS_ASR_MAX_CONV];
  LNorm feat_ln, enc_ln;
  Linear post_proj, proj;
  std::vector<Linear> pos_conv;  // per group: [cg][k * cg] tap-major (weight norm folded), bias slice
  struct Layer {
    LNorm ln1, ln2;
    Linear qkv, out, fc1, fc2;
  };
  std::vector<Layer> layers;
  Umma2Cache* umma = nullptr;
  Arena ws;
  cudaEvent_t ev[5] = {nullptr, nullptr, nullptr, nullptr, nullptr};
  double stage_ms[4] = {0, 0, 0, 0};
  int fail(int code, const std::string& m) {
    err = m;
    return code;
  }
};

namespace {

thread_local std::string g_asr_create_err = "null handle";
const char* kPre = "w2v_encoder.w2v_model.";

const HostTensor* find(ss_asr* h, const std::string& key) {
  auto it = h->host.find(key);
  return it == h->host.end() ? nullptr : &it->second;
}

float* upload(ss_asr* h, const float* src, size_t n) {
  float* d = nullptr;
  if (cudaMalloc((void**)&d, std::max<size_t>(n, 1) * sizeof(float)) != cudaSuccess) return nullptr;
  h->dev_allocs.push_back(d);
  cudaMemcpy(d, src, n * sizeof(float), cudaMemcpyHostToDevice);
  return d;
}

// out[m][N] = epilogue(x[m][K] @ W^T) on the wgmma kernel with 3 bf16 pieces and no split-K (gemm_conv where wgmma does not take the shape)
void asr_linear(ss_asr* h, const float* x, int M, const Linear& l, Epilogue ep, cudaStream_t st) {
  ConvA a;
  a.x = x; a.B = 1; a.L_in = M; a.L_rows = M; a.C_in = l.K; a.ldx = l.K;
  ep.bias = l.b;
  if (umma2_supported(a, l.N, ep)) umma2_conv(h->umma, a, l.w, l.N, ep, 3, nullptr, st);
  else gemm_conv(a, l.w, l.N, ep, nullptr, st);
}

Epilogue ep_to(float* out, int ldo, int act = ACT_NONE, const float* residual = nullptr) {
  Epilogue e;
  e.out = out; e.ldo = ldo; e.act = act; e.residual = residual;
  return e;
}

int64_t frames_of(const ss_asr* h, int64_t n, int layers) {
  int64_t L = n;
  for (int i = 0; i < layers; ++i) L = L >= h->conv_k[i] ? (L - h->conv_k[i]) / h->cfg.conv_stride[i] + 1 : 0;
  return L;
}

// checks every utterance before anything is launched; T[b] = its encoder frames
int check_batch(ss_asr* h, const float* audio, const int64_t* off, int B, std::vector<int>& T, const char* where) {
  if (!h->finalized) return h->fail(SS_ERR_STATE, std::string(where) + ": call ss_asr_finalize first");
  if (B <= 0 || !audio || !off) return h->fail(SS_ERR_INVALID, std::string(where) + ": B <= 0 or a null pointer");
  T.assign(B, 0);
  for (int b = 0; b < B; ++b) {
    if (off[b] < 0 || off[b + 1] < off[b]) return h->fail(SS_ERR_INVALID, std::string(where) + ": offsets must be non-negative and non-decreasing");
    const int64_t t = frames_of(h, off[b + 1] - off[b], h->n_conv);
    if (t <= 0)
      return h->fail(SS_ERR_INVALID, std::string(where) + ": utterance " + std::to_string(b) + " has " + std::to_string(off[b + 1] - off[b]) +
                                         " samples, fewer than one encoder frame needs");
    if (t > h->max_frames)
      return h->fail(SS_ERR_CAPACITY, std::string(where) + ": utterance " + std::to_string(b) + " has " + std::to_string(t) +
                                          " encoder frames; max_frames is " + std::to_string(h->max_frames));
    T[b] = (int)t;
  }
  return SS_OK;
}

// groups of consecutive utterances whose padded rows fit SS_ASR_BATCH_ROWS (an utterance longer than that is a group of its own)
std::vector<std::pair<int, int>> groups_of(const std::vector<int>& T) {
  std::vector<std::pair<int, int>> g;
  int b0 = 0, tmax = 0;
  for (int b = 0; b < (int)T.size(); ++b) {
    const int t = std::max(tmax, T[b]);
    if (b > b0 && (int64_t)t * (b - b0 + 1) > SS_ASR_BATCH_ROWS) {
      g.push_back({b0, b});
      b0 = b;
      tmax = T[b];
    } else {
      tmax = t;
    }
  }
  g.push_back({b0, (int)T.size()});
  return g;
}

int check_launch_asr(ss_asr* h) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return h->fail(SS_ERR_CUDA, std::string("ss_asr: ") + cudaGetErrorString(e));
  return SS_OK;
}

void rec(ss_asr* h, int i, cudaStream_t st) {
  if (h->cfg.time_stages) cudaEventRecord(h->ev[i], st);
}

// The forward pass of utterances [b0, b1).  stop < 0: the whole call (packed tokens, optional arg-max / emissions); otherwise the
// activations after stage `stop` (ss_asr_debug_stage) to stage_out.  row0: the group's first output row among all utterances.
int forward_group(ss_asr* h, cudaStream_t st, const float* audio, const int64_t* off, int b0, int b1, const std::vector<int>& T, int64_t row0,
                  int stop, float* stage_out, int64_t* packed, int64_t packed_stride, int64_t* argmax_out, float* emis_out) {
  const int B = b1 - b0, C = h->C, D = h->D, Lc = h->n_conv;
  // per-layer lengths of the group's utterances
  std::vector<int> lens((size_t)(Lc + 1) * B);
  std::vector<int> Lmax(Lc + 1, 0);
  std::vector<int64_t> offs(B + 1);
  for (int i = 0; i < B; ++i) offs[i] = off[b0 + i] - off[b0];
  offs[B] = off[b1] - off[b0];
  for (int l = 0; l <= Lc; ++l)
    for (int i = 0; i < B; ++i) {
      const int v = (int)frames_of(h, offs[i + 1] - offs[i], l);
      lens[(size_t)l * B + i] = v;
      Lmax[l] = std::max(Lmax[l], v);
    }
  const int Tm = Lmax[Lc];
  const int64_t R = (int64_t)B * Tm;
  int64_t ext_a = 0, ext_b = 0;  // ping-pong extractor buffers: the outputs of conv layers 0, 2, 4, .. go to a, of 1, 3, .. to b
  for (int m = 1; m <= Lc; ++m) {
    int64_t& e = (m % 2 == 1) ? ext_a : ext_b;
    e = std::max(e, (int64_t)B * Lmax[m] * C);
  }
  const int64_t n_audio = offs[B];
  size_t bytes = 0;
  auto add = [&](int64_t n) { bytes += ((size_t)n * 4 + 255) & ~(size_t)255; };
  add(h->cfg.normalize ? n_audio : 0); add(ext_a); add(ext_b);
  add(R * D); add(R * D); add(R * 3 * D); add(R * D); add(R * h->F); add(R * h->V); add(R * 2);
  add((int64_t)(Lc + 1) * B + 2 * (B + 1));
  h->ws.reset();
  if (!h->ws.ensure(bytes + 4096)) return h->fail(SS_ERR_CUDA, "ss_asr_transcribe: out of device memory for the workspace");
  float* wav = h->cfg.normalize ? h->ws.f32(n_audio) : nullptr;
  float* ea = h->ws.f32(ext_a);
  float* eb = h->ws.f32(ext_b);
  float* x = h->ws.f32(R * D);
  float* y = h->ws.f32(R * D);
  float* qkv = h->ws.f32(R * 3 * D);
  float* att = h->ws.f32(R * D);
  float* ffn = h->ws.f32(R * h->F);
  float* logits = h->ws.f32(R * h->V);
  int64_t* am = (int64_t*)h->ws.raw(R * 8);
  int* lens_dev = (int*)h->ws.raw((size_t)(Lc + 1) * B * 4);
  int64_t* offs_dev = (int64_t*)h->ws.raw((size_t)(B + 1) * 8);
  if (cudaMemcpyAsync(lens_dev, lens.data(), lens.size() * 4, cudaMemcpyHostToDevice, st) != cudaSuccess ||
      cudaMemcpyAsync(offs_dev, offs.data(), offs.size() * 8, cudaMemcpyHostToDevice, st) != cudaSuccess ||
      cudaStreamSynchronize(st) != cudaSuccess)
    return h->fail(SS_ERR_CUDA, "ss_asr_transcribe: upload of the lengths failed");
  const int* T_dev = lens_dev + (size_t)Lc * B;
  const float* src = audio + off[b0];
  // copy out rows of the padded [B][Tm][width] activations, utterances in order
  auto copy_rows = [&](const float* act, int width, float* dst) {
    int64_t r = row0;
    for (int i = 0; i < B; ++i) {
      cudaMemcpyAsync(dst + r * width, act + (int64_t)i * Tm * width, (size_t)T[b0 + i] * width * 4, cudaMemcpyDeviceToDevice, st);
      r += T[b0 + i];
    }
  };

  // ---- extractor
  rec(h, 0, st);
  if (wav) {
    ++g_launches;
    launch_pdl(asr_wave_norm_kernel, dim3(B), dim3(1024), 0, st, src, (const int64_t*)offs_dev, wav);
    src = wav;
  }
  ++g_launches;
  launch_pdl(asr_conv0_kernel, dim3(Lmax[1], B), dim3(C), (size_t)h->conv_k[0] * 4, st, src, (const int64_t*)offs_dev, (const int*)(lens_dev + B),
             (const float*)h->conv_w[0], (const float*)h->conv_b[0], (const float*)h->conv_ln[0].g, (const float*)h->conv_ln[0].b, h->conv_k[0],
             h->cfg.conv_stride[0], Lmax[1], ea);
  float* cur = ea;
  for (int l = 1; l < Lc; ++l) {
    float* nxt = (l % 2 == 1) ? eb : ea;
    ConvA a;
    a.x = cur; a.B = B; a.L_in = Lmax[l]; a.L_rows = Lmax[l + 1]; a.C_in = C; a.ldx = C;
    a.ksize = h->conv_k[l]; a.stride = h->cfg.conv_stride[l]; a.lengths = lens_dev + (size_t)l * B;
    Epilogue e = ep_to(nxt, C);
    e.bias = h->conv_b[l];
    gemm_conv(a, h->conv_w[l], C, e, nullptr, st);
    ++g_launches;
    launch_pdl(asr_ln_gelu_kernel, dim3((unsigned)((int64_t)B * Lmax[l + 1])), dim3(C), 0, st, nxt, (const float*)h->conv_ln[l].g,
               (const float*)h->conv_ln[l].b);
    cur = nxt;
  }
  rec(h, 1, st);
  if (stop == 0) {
    copy_rows(cur, C, stage_out);
    return check_launch_asr(h);
  }
  // ---- feature LayerNorm + post_extract_proj
  layer_norm(cur, C, y, C, h->feat_ln.g, h->feat_ln.b, (int)R, C, st);
  asr_linear(h, y, (int)R, h->post_proj, ep_to(x, D), st);
  if (stop == 1) {
    copy_rows(x, D, stage_out);
    return check_launch_asr(h);
  }
  // ---- positional conv: y = x + GELU(conv(x) + bias), one implicit GEMM per group, frames >= T_b zero
  const int cg = D / h->pos_groups;
  for (int g = 0; g < h->pos_groups; ++g) {
    ConvA a;
    a.x = x + g * cg; a.B = B; a.L_in = Tm; a.L_rows = Tm; a.C_in = cg; a.ldx = D;
    a.ksize = h->pos_k; a.pad_left = h->pos_k / 2; a.lengths = T_dev;
    Epilogue e = ep_to(y + g * cg, D, ACT_GELU, x + g * cg);
    e.bias = h->pos_conv[g].b;
    gemm_conv(a, h->pos_conv[g].w, cg, e, nullptr, st);
  }
  std::swap(x, y);
  rec(h, 2, st);
  if (stop == 2) {
    copy_rows(x, D, stage_out);
    return check_launch_asr(h);
  }
  // ---- transformer layers (pre-LN)
  for (size_t li = 0; li < h->layers.size(); ++li) {
    const auto& L = h->layers[li];
    layer_norm(x, D, y, D, L.ln1.g, L.ln1.b, (int)R, D, st);
    asr_linear(h, y, (int)R, L.qkv, ep_to(qkv, 3 * D), st);
    mha_attention(qkv, 3 * D, qkv + D, 3 * D, qkv + 2 * D, 3 * D, att, D, B, Tm, Tm, h->H, 0.125f, 0, 0, T_dev, st, 2);
    asr_linear(h, att, (int)R, L.out, ep_to(x, D, ACT_NONE, x), st);
    layer_norm(x, D, y, D, L.ln2.g, L.ln2.b, (int)R, D, st);
    asr_linear(h, y, (int)R, L.fc1, ep_to(ffn, h->F, ACT_GELU), st);
    asr_linear(h, ffn, (int)R, L.fc2, ep_to(x, D, ACT_NONE, x), st);
    if (stop == 3 + (int)li) {
      copy_rows(x, D, stage_out);
      return check_launch_asr(h);
    }
  }
  rec(h, 3, st);
  // ---- final LayerNorm + proj + arg-max + collapse
  const int nl = (int)h->layers.size();
  layer_norm(x, D, y, D, h->enc_ln.g, h->enc_ln.b, (int)R, D, st);
  if (stop == 3 + nl) {
    copy_rows(y, D, stage_out);
    return check_launch_asr(h);
  }
  asr_linear(h, y, (int)R, h->proj, ep_to(logits, h->V), st);
  if (stop == 4 + nl) {
    copy_rows(logits, h->V, stage_out);
    return check_launch_asr(h);
  }
  ++g_launches;
  launch_pdl(asr_argmax_collapse_kernel, dim3(B), dim3(1024), 0, st, (const float*)logits, h->V, Tm, T_dev, am, packed + (int64_t)b0 * packed_stride,
             packed_stride);
  if (emis_out) copy_rows(logits, h->V, emis_out);
  if (argmax_out) {
    int64_t r = row0;
    for (int i = 0; i < B; ++i) {
      cudaMemcpyAsync(argmax_out + r, am + (int64_t)i * Tm, (size_t)T[b0 + i] * 8, cudaMemcpyDeviceToDevice, st);
      r += T[b0 + i];
    }
  }
  rec(h, 4, st);
  if (h->cfg.time_stages) {
    cudaEventSynchronize(h->ev[4]);
    for (int i = 0; i < 4; ++i) {
      float ms = 0.f;
      cudaEventElapsedTime(&ms, h->ev[i], h->ev[i + 1]);
      h->stage_ms[i] += ms;
    }
  }
  return check_launch_asr(h);
}

}  // namespace

int ss_asr_create(ss_asr** out, int device, const ss_asr_config* cfg) {
  if (!out || !cfg) return SS_ERR_INVALID;
  *out = nullptr;
  g_asr_create_err = "null handle";
  auto refuse = [](const std::string& m) {
    g_asr_create_err = "ss_asr_create: " + m;
    return SS_ERR_INVALID;
  };
  if (cfg->n_conv < 1 || cfg->n_conv > SS_ASR_MAX_CONV) return refuse("n_conv = " + std::to_string(cfg->n_conv) + " is outside [1, 8]");
  for (int i = 0; i < cfg->n_conv; ++i)
    if (cfg->conv_stride[i] < 1) return refuse("conv_feature_layers: stride " + std::to_string(cfg->conv_stride[i]) + " of layer " + std::to_string(i));
  if (cfg->extractor_layer_norm != 1) return refuse("extractor_mode \"default\" (group norm) is not supported; only \"layer_norm\"");
  if (cfg->layer_norm_first != 1) return refuse("layer_norm_first = False (post-LN layers) is not supported");
  if (cfg->pos_conv_depth != 1) return refuse("pos_conv_depth = " + std::to_string(cfg->pos_conv_depth) + " is not supported; only 1");
  if (cfg->conformer != 0) return refuse("layer_type \"conformer\" is not supported; only \"transformer\"");
  if (cfg->max_frames < 0) return refuse("max_frames < 0");
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess || n <= 0 || device < 0 || device >= n) return SS_ERR_CUDA;
  if (cudaSetDevice(device) != cudaSuccess) return SS_ERR_CUDA;
  ss_asr* h = new ss_asr();
  h->device = device;
  h->cfg = *cfg;
  h->max_frames = cfg->max_frames > 0 ? cfg->max_frames : 4096;
  h->umma = new Umma2Cache();
  for (auto& e : h->ev) cudaEventCreate(&e);
  *out = h;
  return SS_OK;
}

int ss_asr_destroy(ss_asr* h) {
  if (!h) return SS_ERR_INVALID;
  cudaSetDevice(h->device);
  cudaDeviceSynchronize();
  umma2_cache_destroy(h->umma);
  for (void* p : h->dev_allocs) cudaFree(p);
  if (h->ws.base) cudaFree(h->ws.base);
  for (auto& e : h->ev) cudaEventDestroy(e);
  delete h;
  return SS_OK;
}

const char* ss_asr_last_error(const ss_asr* h) { return h ? h->err.c_str() : g_asr_create_err.c_str(); }

int ss_asr_load_tensor(ss_asr* h, const char* key, const float* data, int ndim, const int64_t* shape) {
  if (!h || !key || ndim < 0 || ndim > 8 || (ndim > 0 && (!shape || !data))) return SS_ERR_INVALID;
  if (h->finalized) return h->fail(SS_ERR_STATE, "ss_asr_load_tensor: the handle is finalized");
  const std::string k(key);
  const bool used = k.rfind("w2v_encoder.proj.", 0) == 0 ||
                    (k.rfind(kPre, 0) == 0 && (k.find("feature_extractor.") != std::string::npos || k.find(".layer_norm.") != std::string::npos ||
                                               k.find("post_extract_proj.") != std::string::npos || k.find(".encoder.") != std::string::npos));
  if (!used) return SS_OK;
  if (k.find(".encoder.pos_conv.1.") != std::string::npos || k.find(".encoder.pos_conv.2.") != std::string::npos)
    return h->fail(SS_ERR_INVALID, "ss_asr_load_tensor: " + k + ": pos_conv_depth > 1 is not supported");
  HostTensor t;
  t.shape.assign(shape, shape + ndim);
  for (auto s : t.shape)
    if (s < 0) return h->fail(SS_ERR_INVALID, "ss_asr_load_tensor: negative dimension in " + k);
  t.data.assign(data, data + t.numel());
  h->host[k] = std::move(t);
  return SS_OK;
}

int64_t ss_asr_num_frames(const ss_asr* h, int64_t n) {
  if (!h || !h->finalized) return -1;
  return frames_of(h, n, h->n_conv);
}

int ss_asr_finalize(ss_asr* h) {
  if (!h) return SS_ERR_INVALID;
  if (h->finalized) return SS_OK;
  cudaSetDevice(h->device);
  const std::string P(kPre);
  auto need = [&](const std::string& k, std::vector<int64_t> shape, const HostTensor** out) -> int {
    const HostTensor* t = find(h, k);
    if (!t) return h->fail(SS_ERR_MISSING, "ss_asr_finalize: missing " + k);
    if (!shape.empty() && t->shape != shape) {
      std::string s;
      for (auto v : t->shape) s += std::to_string(v) + ",";
      return h->fail(SS_ERR_INVALID, "ss_asr_finalize: " + k + " has shape [" + s + "], not the one the model's other tensors imply");
    }
    *out = t;
    return SS_OK;
  };
  int rc;
  const HostTensor *t, *t2;
  // ---- extractor
  int nc = 0;
  while (find(h, P + "feature_extractor.conv_layers." + std::to_string(nc) + ".0.weight")) ++nc;
  if (nc != h->cfg.n_conv)
    return h->fail(SS_ERR_INVALID, "ss_asr_finalize: the state dict has " + std::to_string(nc) + " conv layers, the config " + std::to_string(h->cfg.n_conv));
  h->n_conv = nc;
  for (int i = 0; i < nc; ++i) {
    const std::string pre = P + "feature_extractor.conv_layers." + std::to_string(i);
    const HostTensor* w = find(h, pre + ".0.weight");
    if (w->shape.size() != 3) return h->fail(SS_ERR_INVALID, "ss_asr_finalize: " + pre + ".0.weight is not 3-D");
    const int cout = (int)w->shape[0], cin = (int)w->shape[1], k = (int)w->shape[2];
    if (i == 0) {
      h->C = cout;
      if (cin != 1) return h->fail(SS_ERR_INVALID, "ss_asr_finalize: conv layer 0 must have one input channel");
      if (cout < 32 || cout > 1024 || cout % 32) return h->fail(SS_ERR_INVALID, "ss_asr_finalize: extractor width must be a multiple of 32 in [32, 1024]");
    } else if (cout != h->C || cin != h->C) {
      return h->fail(SS_ERR_INVALID, "ss_asr_finalize: conv layers of different widths are not supported");
    }
    h->conv_k[i] = k;
    std::vector<float> wr((size_t)cout * k * cin);
    for (int o = 0; o < cout; ++o)
      for (int c = 0; c < cin; ++c)
        for (int j = 0; j < k; ++j) wr[((size_t)o * k + j) * cin + c] = w->data[((size_t)o * cin + c) * k + j];
    h->conv_w[i] = upload(h, wr.data(), wr.size());
    const HostTensor* b = find(h, pre + ".0.bias");  // conv_bias = False: no key
    std::vector<float> zb(cout, 0.f);
    h->conv_b[i] = upload(h, b ? b->data.data() : zb.data(), cout);
    if ((rc = need(pre + ".2.1.weight", {cout}, &t)) || (rc = need(pre + ".2.1.bias", {cout}, &t2))) return rc;
    h->conv_ln[i] = LNorm{upload(h, t->data.data(), cout), upload(h, t2->data.data(), cout), cout};
  }
  const int C = h->C;
  if (!layer_norm_supported(C)) return h->fail(SS_ERR_INVALID, "ss_asr_finalize: the feature LayerNorm cannot take width " + std::to_string(C));
  if ((rc = need(P + "layer_norm.weight", {C}, &t)) || (rc = need(P + "layer_norm.bias", {C}, &t2))) return rc;
  h->feat_ln = LNorm{upload(h, t->data.data(), C), upload(h, t2->data.data(), C), C};
  const HostTensor* pw = find(h, P + "post_extract_proj.weight");
  if (!pw || pw->shape.size() != 2 || pw->shape[1] != C) return h->fail(SS_ERR_MISSING, "ss_asr_finalize: missing " + P + "post_extract_proj.weight [D][C]");
  const int D = (int)pw->shape[0];
  h->D = D;
  if (D % 64 || D > 1024 || !layer_norm_supported(D))
    return h->fail(SS_ERR_INVALID, "ss_asr_finalize: model dim " + std::to_string(D) + " must be a multiple of 64 up to 1024");
  h->H = h->cfg.heads > 0 ? h->cfg.heads : D / 64;
  if (D != h->H * 64)
    return h->fail(SS_ERR_INVALID, "ss_asr_finalize: encoder_attention_heads = " + std::to_string(h->H) + " gives head dim " + std::to_string(D / h->H) +
                                       "; only 64 is supported");
  if ((rc = need(P + "post_extract_proj.bias", {D}, &t2)) != SS_OK) return rc;
  h->post_proj = Linear{upload(h, pw->data.data(), pw->data.size()), upload(h, t2->data.data(), D), D, C};
  // ---- positional conv (weight norm over dims 0 and 1 folded: w = g[j] * v / ||v[:, :, j]||)
  const HostTensor* pb;
  if ((rc = need(P + "encoder.pos_conv.0.bias", {D}, &pb)) != SS_OK) return rc;
  std::vector<float> wpos;
  int cg = 0, kp = 0;
  if (const HostTensor* wf = find(h, P + "encoder.pos_conv.0.weight")) {
    if (wf->shape.size() != 3 || wf->shape[0] != D) return h->fail(SS_ERR_INVALID, "ss_asr_finalize: encoder.pos_conv.0.weight must be [D][D / groups][k]");
    cg = (int)wf->shape[1]; kp = (int)wf->shape[2];
    wpos = wf->data;
  } else {
    const HostTensor *g, *v;
    if ((rc = need(P + "encoder.pos_conv.0.weight_v", {}, &v)) != SS_OK) return rc;
    if (v->shape.size() != 3 || v->shape[0] != D) return h->fail(SS_ERR_INVALID, "ss_asr_finalize: encoder.pos_conv.0.weight_v must be [D][D / groups][k]");
    cg = (int)v->shape[1]; kp = (int)v->shape[2];
    if ((rc = need(P + "encoder.pos_conv.0.weight_g", {1, 1, kp}, &g)) != SS_OK) return rc;
    wpos.resize(v->data.size());
    for (int j = 0; j < kp; ++j) {
      double ss = 0.0;
      for (int64_t oi = 0; oi < (int64_t)D * cg; ++oi) ss += (double)v->data[oi * kp + j] * v->data[oi * kp + j];
      const double s = g->data[j] / std::sqrt(ss);
      for (int64_t oi = 0; oi < (int64_t)D * cg; ++oi) wpos[oi * kp + j] = (float)(v->data[oi * kp + j] * s);
    }
  }
  if (cg <= 0 || D % cg || cg % 4) return h->fail(SS_ERR_INVALID, "ss_asr_finalize: positional-conv groups must have a multiple of 4 channels");
  h->pos_k = kp;
  h->pos_groups = D / cg;
  for (int g = 0; g < h->pos_groups; ++g) {
    std::vector<float> wr((size_t)cg * kp * cg);
    for (int o = 0; o < cg; ++o)
      for (int c = 0; c < cg; ++c)
        for (int j = 0; j < kp; ++j) wr[((size_t)o * kp + j) * cg + c] = wpos[(((size_t)(g * cg + o)) * cg + c) * kp + j];
    h->pos_conv.push_back(Linear{upload(h, wr.data(), wr.size()), upload(h, pb->data.data() + g * cg, cg), cg, kp * cg});
  }
  // ---- layers
  if (find(h, P + "encoder.layers.0.conv_module.depthwise_conv.weight")) return h->fail(SS_ERR_INVALID, "ss_asr_finalize: conformer layers are not supported");
  int nl = 0;
  while (find(h, P + "encoder.layers." + std::to_string(nl) + ".self_attn.q_proj.weight")) ++nl;
  if (nl == 0) return h->fail(SS_ERR_MISSING, "ss_asr_finalize: missing " + P + "encoder.layers.0.self_attn.q_proj.weight");
  const HostTensor* f1 = find(h, P + "encoder.layers.0.fc1.weight");
  if (!f1 || f1->shape.size() != 2) return h->fail(SS_ERR_MISSING, "ss_asr_finalize: missing " + P + "encoder.layers.0.fc1.weight");
  const int F = (int)f1->shape[0];
  h->F = F;
  if (F % 16) return h->fail(SS_ERR_INVALID, "ss_asr_finalize: FFN width must be a multiple of 16");
  for (int l = 0; l < nl; ++l) {
    const std::string pre = P + "encoder.layers." + std::to_string(l) + ".";
    ss_asr::Layer L;
    std::vector<float> wqkv, bqkv;
    for (const char* nm : {"q_proj", "k_proj", "v_proj"}) {
      if ((rc = need(pre + "self_attn." + nm + ".weight", {D, D}, &t)) || (rc = need(pre + "self_attn." + nm + ".bias", {D}, &t2))) return rc;
      wqkv.insert(wqkv.end(), t->data.begin(), t->data.end());
      bqkv.insert(bqkv.end(), t2->data.begin(), t2->data.end());
    }
    L.qkv = Linear{upload(h, wqkv.data(), wqkv.size()), upload(h, bqkv.data(), bqkv.size()), 3 * D, D};
    auto lin = [&](const std::string& nm, int N, int K, Linear* o) -> int {
      if ((rc = need(pre + nm + ".weight", {N, K}, &t)) || (rc = need(pre + nm + ".bias", {N}, &t2))) return rc;
      *o = Linear{upload(h, t->data.data(), t->data.size()), upload(h, t2->data.data(), N), N, K};
      return SS_OK;
    };
    auto ln = [&](const std::string& nm, LNorm* o) -> int {
      if ((rc = need(pre + nm + ".weight", {D}, &t)) || (rc = need(pre + nm + ".bias", {D}, &t2))) return rc;
      *o = LNorm{upload(h, t->data.data(), D), upload(h, t2->data.data(), D), D};
      return SS_OK;
    };
    if ((rc = lin("self_attn.out_proj", D, D, &L.out)) || (rc = lin("fc1", F, D, &L.fc1)) || (rc = lin("fc2", D, F, &L.fc2)) ||
        (rc = ln("self_attn_layer_norm", &L.ln1)) || (rc = ln("final_layer_norm", &L.ln2)))
      return rc;
    h->layers.push_back(L);
  }
  if ((rc = need(P + "encoder.layer_norm.weight", {D}, &t)) || (rc = need(P + "encoder.layer_norm.bias", {D}, &t2))) return rc;
  h->enc_ln = LNorm{upload(h, t->data.data(), D), upload(h, t2->data.data(), D), D};
  const HostTensor* pj = find(h, "w2v_encoder.proj.weight");
  if (!pj || pj->shape.size() != 2 || pj->shape[1] != D) return h->fail(SS_ERR_MISSING, "ss_asr_finalize: missing w2v_encoder.proj.weight [V][D]");
  h->V = (int)pj->shape[0];
  if (h->V <= kUnk || h->V % 4) return h->fail(SS_ERR_INVALID, "ss_asr_finalize: the vocabulary must hold the 4 specials and be a multiple of 4");
  if ((rc = need("w2v_encoder.proj.bias", {h->V}, &t2)) != SS_OK) return rc;
  h->proj = Linear{upload(h, pj->data.data(), pj->data.size()), upload(h, t2->data.data(), h->V), h->V, D};
  for (void* p : h->dev_allocs)
    if (!p) return h->fail(SS_ERR_CUDA, "ss_asr_finalize: out of device memory for the weights");
  if (cudaDeviceSynchronize() != cudaSuccess) return h->fail(SS_ERR_CUDA, "ss_asr_finalize: upload failed");
  h->host.clear();
  h->finalized = true;
  return SS_OK;
}

static int asr_run(ss_asr* h, void* stream, const float* audio, const int64_t* off, int B, int stop, float* stage_out, int64_t* packed,
                   int64_t packed_stride, int64_t* argmax_out, float* emis_out, const char* where) {
  if (!h) return SS_ERR_INVALID;
  cudaSetDevice(h->device);
  std::vector<int> T;
  int rc = check_batch(h, audio, off, B, T, where);
  if (rc) return rc;
  if (stop < 0) {
    if (!packed) return h->fail(SS_ERR_INVALID, std::string(where) + ": packed_out_dev is null");
    for (int b = 0; b < B; ++b)
      if (packed_stride < (int64_t)T[b] + 1)
        return h->fail(SS_ERR_INVALID, std::string(where) + ": packed_stride " + std::to_string(packed_stride) + " < T + 1 = " + std::to_string(T[b] + 1));
  } else if (stop > 4 + (int)h->layers.size() || !stage_out) {
    return h->fail(SS_ERR_INVALID, std::string(where) + ": stage outside [0, 4 + layers] or a null output");
  }
  int64_t row0 = 0;
  for (auto [b0, b1] : groups_of(T)) {
    if ((rc = forward_group(h, (cudaStream_t)stream, audio, off, b0, b1, T, row0, stop, stage_out, packed, packed_stride, argmax_out, emis_out))) return rc;
    for (int b = b0; b < b1; ++b) row0 += T[b];
  }
  return SS_OK;
}

int ss_asr_transcribe(ss_asr* h, void* stream, const float* audio_dev, const int64_t* offsets_host, int B, int64_t* packed_out_dev,
                      int64_t packed_stride, int64_t* argmax_dev, float* emissions_dev) {
  return asr_run(h, stream, audio_dev, offsets_host, B, -1, nullptr, packed_out_dev, packed_stride, argmax_dev, emissions_dev, "ss_asr_transcribe");
}

int ss_asr_debug_stage(ss_asr* h, void* stream, const float* audio_dev, const int64_t* offsets_host, int B, int stage, float* out_dev) {
  if (h && stage < 0) return h->fail(SS_ERR_INVALID, "ss_asr_debug_stage: stage < 0");
  return asr_run(h, stream, audio_dev, offsets_host, B, stage, out_dev, nullptr, 0, nullptr, nullptr, "ss_asr_debug_stage");
}

int ss_asr_stage_ms(ss_asr* h, double* ms) {
  if (!h || !ms) return SS_ERR_INVALID;
  for (int i = 0; i < 4; ++i) {
    ms[i] = h->stage_ms[i];
    h->stage_ms[i] = 0.0;
  }
  return SS_OK;
}
