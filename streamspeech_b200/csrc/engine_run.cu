// The per-block entry points of the C-ABI: each one enqueues the kernels of one reference call site.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <stdexcept>
#include <tuple>

#include "engine.h"

using namespace ss;

namespace {

inline cudaStream_t S(void* s) { return (cudaStream_t)s; }

int check_launch(ss_engine* h, const char* where) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return h->fail(SS_ERR_CUDA, std::string(where) + ": " + cudaGetErrorString(e));
  return SS_OK;
}

// tensor-core routing of the current entry point (set from the handle at the top of each entry point)
thread_local int g_umma_linear = 0;
thread_local int g_umma_conv = 0;
thread_local int g_umma_min_rows = 128;
thread_local int g_umma_min_channels = 16;
thread_local Umma2Cache* g_umma2_cache = nullptr;

void route_from(ss_engine* h) {
  g_umma_linear = h->umma_linear;
  g_umma_min_rows = h->umma_min_rows;
  g_umma_min_channels = h->umma_min_channels;
  if (!h->umma2_cache) h->umma2_cache = umma2_cache_create();
  g_umma2_cache = h->umma2_cache;
}

// conv-as-GEMM dispatch: the wgmma split-bf16 kernel (kernels_umma2.cu; mode 12 / 13 = 2 / 3 bf16 pieces per operand) when enabled and
// the shape fits, the fp32 CUDA-core kernel otherwise
void conv_gemm(const ConvA& a, const float* W, int N, const Epilogue& ep, cudaStream_t st) {
  const int rows = a.B * a.L_rows;
  if (g_umma_conv >= 12 && g_umma2_cache && rows >= g_umma_min_rows && a.C_in >= g_umma_min_channels && umma2_supported(a, N, ep))
    umma2_conv(g_umma2_cache, a, W, N, ep, g_umma_conv - 10, st);
  else
    gemm_conv(a, W, N, ep, st);
}

// plain linear: out[M][N] = epilogue(x[M][K] @ W^T)
void linear(const float* x, int ldx, int M, const Linear& l, Epilogue ep, cudaStream_t st) {
  ConvA a;
  a.x = x; a.B = 1; a.L_in = M; a.L_rows = M; a.C_in = l.K; a.ldx = ldx;
  ep.bias = l.b;
  if (skinny_gemm_supported(M, l.N, l.K, ep) && (ldx & 3) == 0)
    skinny_gemm(x, ldx, l.w, M, l.N, l.K, ep, st);
  else if (g_umma_linear >= 12 && g_umma2_cache && M >= g_umma_min_rows && umma2_supported(a, l.N, ep))
    umma2_conv(g_umma2_cache, a, l.w, l.N, ep, g_umma_linear - 10, st);
  else
    gemm_conv(a, l.w, l.N, ep, st);
}
// out = epilogue(LayerNorm(x) @ W^T).  The LN is fused into the skinny kernel's A load when the shape allows it,
// otherwise it is a separate launch into `scratch` [M][K].
void ln_linear(const float* x, int ldx, int M, const LNorm& ln, const Linear& l, Epilogue ep, float* scratch, cudaStream_t st) {
  ep.bias = l.b;
  Epilogue fused = ep;
  fused.ln_gamma = ln.g;
  fused.ln_beta = ln.b;
  if (ln.C == l.K && (ldx & 3) == 0 && skinny_gemm_supported(M, l.N, l.K, fused)) {
    skinny_gemm(x, ldx, l.w, M, l.N, l.K, fused, st);
    return;
  }
  layer_norm(x, ldx, scratch, l.K, ln.g, ln.b, M, l.K, st);
  linear(scratch, l.K, M, l, ep, st);
}

// q | k | v = LayerNorm(x) @ Wqkv^T with the three column blocks routed to their own buffers (query scratch, K cache
// rows, V cache rows).  One launch on the skinny path; LN + three GEMMs otherwise.
void ln_qkv_routed(const float* x, int ldx, int M, const LNorm& ln, const Linear& qkv, int dim, float* q, int ldq, float* k, int ldk,
                   float* v, int ldv, float* scratch, cudaStream_t st) {
  Epilogue ep;
  ep.out = q; ep.ldo = ldq; ep.out2 = k; ep.ldo2 = ldk; ep.out3 = v; ep.ldo3 = ldv; ep.split_n = dim;
  ep.bias = qkv.b; ep.ln_gamma = ln.g; ep.ln_beta = ln.b;
  if (ln.C == qkv.K && (ldx & 3) == 0 && skinny_gemm_supported(M, qkv.N, qkv.K, ep)) {
    skinny_gemm(x, ldx, qkv.w, M, qkv.N, qkv.K, ep, st);
    return;
  }
  layer_norm(x, ldx, scratch, qkv.K, ln.g, ln.b, M, qkv.K, st);
  Linear part = qkv;
  part.N = dim;
  float* outs[3] = {q, k, v};
  int lds[3] = {ldq, ldk, ldv};
  for (int p = 0; p < 3; ++p) {
    part.w = qkv.w + (size_t)p * dim * qkv.K;
    part.b = qkv.b + p * dim;
    Epilogue e;
    e.out = outs[p]; e.ldo = lds[p];
    linear(scratch, qkv.K, M, part, e, st);
  }
}

Epilogue ep_out(float* out, int ldo, int act = ACT_NONE) {
  Epilogue e;
  e.out = out; e.ldo = ldo; e.act = act;
  return e;
}
Epilogue ep_residual(float* inout, int ldo, float alpha = 1.0f) {  // inout = inout + alpha * y
  Epilogue e;
  e.out = inout; e.ldo = ldo; e.alpha = alpha; e.residual = inout; e.res_scale = 1.0f;
  return e;
}

// A persistent kernel whose grid barrier timed out raised persist_bar[SS_BAR_ERR_WORD].  `flag` = its host copy (taken after a
// synchronisation).  Re-arms the barrier (counter and host target back in step) and reports the failure.
int report_async_error(ss_engine* h, unsigned flag, const char* where) {
  if (!flag) return SS_OK;
  cudaDeviceSynchronize();
  if (h->persist_bar) cudaMemset(h->persist_bar, 0, 64 * sizeof(unsigned));
  h->persist_bar_target = 0;
  return h->fail(SS_ERR_CUDA, std::string(where) + ": a grid barrier of a persistent kernel timed out; the results of the calls since the "
                                                   "last check are invalid (barrier re-armed)");
}

void clear_graphs(ss_engine* h) {
  cudaDeviceSynchronize();
  for (auto& kv : h->voc_graphs) cudaGraphExecDestroy(kv.second.first);
  h->voc_graphs.clear();
  h->voc_fused.clear();  // (their packed weight pointers may be gone too)
}

bool ws_begin(ss_engine* h, size_t bytes) {
  h->ws.reset();
  return h->ws.ensure(bytes);
}

// Frame counts up to this run the vocoder generator as one persistent kernel.  It was measured faster than the multi-launch path
// at 52 (the streaming agent's calls: new frames plus the receptive field), 180 and 750 frames (the offline leg); longer sequences,
// which were not measured, keep the multi-launch path.
constexpr int kVocFusedMaxFrames = 1024;

// Job / phase tables of the fused generator for N input frames with the arena's buffers (built once per (N, arena) and kept on
// the device).  nullptr when a shape is outside what the kernel supports or memory runs out.
VocFusedParams* vocoder_fused_table(ss_engine* h, int N, const float* frames, float* bufX, float* bufY, const std::vector<float*>& rbA,
                                                    const std::vector<float*>& rbB, const std::vector<float*>& rbT, const std::vector<float*>& rbO,
                                                    cudaStream_t st) {
  const auto key = std::make_pair(N, (uintptr_t)h->ws.base);
  auto it = h->voc_fused.find(key);
  if (it != h->voc_fused.end()) return &it->second;
  const ss_config& c = h->cfg;
  const int grid = vocoder_fused_grid();
  if (grid <= 0) return nullptr;
  std::vector<VocJob> jobs;
  std::vector<VocPhase> phases;
  int a_stride = 0, b_stride = 0;
  bool ok = true;
  auto job = [&](const float* x0, const float* x1, const float* x2, int L_in, int M, int C_in, int k, int dil, int pad_left, float slope,
                 const float* W, const float* bias, float* out, int Nout, int stride, int offset, const float* residual, float alpha, float res_scale) {
    VocJob j{};
    j.x0 = x0; j.x1 = x1; j.x2 = x2; j.L_in = L_in; j.M = M; j.C_in = C_in; j.ksize = k; j.dil = dil; j.pad_left = pad_left; j.slope = slope;
    j.wp = reinterpret_cast<const unsigned char*>(W);  // replaced by the packed copy once the phase's tile width is known
    j.bias = bias; j.out = out; j.N = Nout; j.out_row_stride = stride; j.out_row_offset = offset; j.residual = residual; j.alpha = alpha;
    j.res_scale = res_scale;
    j.CK = (C_in % 32 == 0) ? 32 : 16;
    j.m_tiles = (M + VOC_FUSED_BM - 1) / VOC_FUSED_BM;
    if (C_in % 16 != 0 || Nout % 16 != 0 || k < 1 || (k - 1) * dil > 50 || bias == nullptr) ok = false;
    jobs.push_back(j);
  };
  // closes the phase of jobs [first, end): tile width, packed weights, longest jobs first
  auto phase = [&](int first) {
    const int n_jobs = (int)jobs.size() - first;
    int items32 = 0;
    for (int i = first; i < (int)jobs.size(); ++i) items32 += jobs[i].N % 32 == 0 ? jobs[i].m_tiles * (jobs[i].N / 32) : 0;
    const bool bn32 = items32 >= grid;  // 16-column tiles when 32-column ones would leave SMs idle
    VocPhase p{first, n_jobs, 0};
    for (int i = first; i < (int)jobs.size(); ++i) {
      VocJob& j = jobs[i];
      j.BN = (bn32 && j.N % 32 == 0) ? 32 : 16;
      j.n_tiles = j.N / j.BN;
      j.wp = umma2_packed_weights(h->umma2_cache, reinterpret_cast<const float*>(j.wp), j.N, j.C_in, j.ksize, j.BN, j.CK, 2, st);
      if (j.wp == nullptr) ok = false;
      const int rs_pad = ((VOC_FUSED_BM + (j.ksize - 1) * j.dil + 7) & ~7) + 4;
      a_stride = std::max(a_stride, 2 * (j.CK / 8) * rs_pad * 16);
      b_stride = std::max(b_stride, j.ksize * 2 * j.BN * j.CK * 2);
      p.n_items += j.m_tiles * j.n_tiles;
    }
    std::stable_sort(jobs.begin() + first, jobs.end(), [](const VocJob& a, const VocJob& b) { return a.ksize > b.ksize; });
    phases.push_back(p);
  };
  jobs.reserve(1 + c.voc_n_ups * (8 + 2 * c.voc_n_rb * c.voc_rb_ndil));
  job(frames, nullptr, nullptr, N, N, c.voc_in_dim, 7, 1, 3, 1.0f, h->conv_pre.lin.w, h->conv_pre.lin.b, bufX, c.voc_init_channels, 1, 0, nullptr,
      1.0f, 1.0f);
  phase(0);
  const int nrb = c.voc_n_rb, nd = c.voc_rb_ndil;
  int L = N;
  for (int i = 0; i < c.voc_n_ups; ++i) {
    const UpsampleW& U = h->ups[i];
    const int Lout = L * U.u;
    // stage input: conv_pre's output, or the previous stage's three resblock outputs summed while loading
    const float* x0 = i == 0 ? bufX : rbO[0];
    const float* x1 = i == 0 ? nullptr : rbO[1];
    const float* x2 = i == 0 ? nullptr : rbO[2];
    int first = (int)jobs.size();
    for (int phi = 0; phi < U.u; ++phi) {
      const int J = U.phase_J[phi], q0 = U.phase_q0[phi];
      const int nrows = (Lout - 1 - phi + U.pad) / U.u - q0 + 1;
      if (nrows <= 0) continue;
      job(x0, x1, x2, L, nrows, U.cin, J, 1, (J - 1) - q0, 0.1f, U.phase_w[phi].w, U.bias, bufY, U.cout, U.u, q0 * U.u + phi - U.pad, nullptr,
          1.0f, 1.0f);
    }
    phase(first);
    L = Lout;
    const int ch = U.cout;
    for (int m = 0; m < nd; ++m) {
      first = (int)jobs.size();
      for (int j = 0; j < nrb; ++j) {
        const ConvW& w1 = h->rb1[i][j][m];
        const float* cur = m == 0 ? bufY : (m == 1 ? rbA[j] : rbB[j]);
        job(cur, nullptr, nullptr, L, L, ch, w1.ksize, w1.dil, (w1.ksize * w1.dil - w1.dil) / 2, 0.1f, w1.lin.w, w1.lin.b, rbT[j], ch, 1, 0,
            nullptr, 1.0f, 1.0f);
      }
      phase(first);
      first = (int)jobs.size();
      for (int j = 0; j < nrb; ++j) {
        const ConvW& w2 = h->rb2[i][j][m];
        const float* cur = m == 0 ? bufY : (m == 1 ? rbA[j] : rbB[j]);
        float* out = m + 1 < nd ? (m == 0 ? rbA[j] : rbB[j]) : rbO[j];
        const float s = m + 1 < nd ? 1.0f : 1.0f / nrb;  // last pair of the block: (xt + x) / num_kernels
        job(rbT[j], nullptr, nullptr, L, L, ch, w2.ksize, 1, (w2.ksize - 1) / 2, 0.1f, w2.lin.w, w2.lin.b, out, ch, 1, 0, cur, s, s);
      }
      phase(first);
    }
  }
  if (!ok || jobs.size() > VOC_MAX_JOBS || phases.size() > VOC_MAX_PHASES || vocoder_fused_smem(a_stride, b_stride) > 200 * 1024) return nullptr;
  if (h->voc_fused.size() >= 64) h->voc_fused.clear();
  VocFusedParams& p = h->voc_fused[key];
  std::copy(jobs.begin(), jobs.end(), p.jobs);
  std::copy(phases.begin(), phases.end(), p.phases);
  p.n_phases = (int)phases.size();
  p.a_stride = a_stride;
  p.b_stride = b_stride;
  return &p;
}

struct DecScratch {
  float *y, *q, *kv, *attn, *hid, *qkv;
};

// pre-LN transformer layer over x[n][dim] (TransformerDecoderLayerBase.forward / TransformerEncoderLayerBase.forward,
// ctc_unity/modules/transformer_layer.py:165-230,388-551).  Self-attention keys/values come either from the
// layer's own fused qkv (full sequence, cache == nullptr) or from an external KV cache that already holds `past` rows.
void dec_layer(const DecLayerW& L, float* x, int n, int dim, int ffn, int heads, bool causal, int self_kv_len_limit,
               const int* self_kv_len_dev, float* cache_k, float* cache_v, int past, const float* cross_kv, int Tk,
               const int* cross_len_dev, DecScratch& s, cudaStream_t st, int group_R = 0, const int* group_len_dev = nullptr) {
  const float scale = 0.125f;  // head_dim ** -0.5, head_dim = 64
  if (group_R > 1 && !cache_k && causal && n % group_R == 0) {
    // rows come in groups of group_R identical consecutive rows (unit decoder layer 1): project the n / group_R distinct
    // rows only and collapse the causal softmax over the copies analytically (grouped_causal_attn_kernel)
    const int S = n / group_R;
    ln_linear(x, dim * group_R, S, L.self_ln, L.qkv, ep_out(s.qkv, 3 * dim), s.y, st);
    grouped_causal_attention(s.qkv, 3 * dim, s.qkv + dim, 3 * dim, s.qkv + 2 * dim, 3 * dim, s.attn, dim, S, group_R, heads, scale, group_len_dev, st);
  } else if (cache_k) {
    ln_qkv_routed(x, dim, n, L.self_ln, L.qkv, dim, s.q, dim, cache_k + (size_t)past * dim, dim, cache_v + (size_t)past * dim, dim, s.y, st);
    mha_attention(s.q, dim, cache_k, dim, cache_v, dim, s.attn, dim, 1, n, past + n, heads, scale, 1, past, self_kv_len_dev, st);
  } else {
    ln_linear(x, dim, n, L.self_ln, L.qkv, ep_out(s.qkv, 3 * dim), s.y, st);
    mha_attention(s.qkv, 3 * dim, s.qkv + dim, 3 * dim, s.qkv + 2 * dim, 3 * dim, s.attn, dim, 1, n, n, heads, scale,
                  causal ? 1 : 0, 0, self_kv_len_dev, st);
  }
  (void)self_kv_len_limit;
  linear(s.attn, dim, n, L.out, ep_residual(x, dim), st);
  if (L.has_cross) {
    ln_linear(x, dim, n, L.cross_ln, L.cq, ep_out(s.q, dim), s.y, st);
    mha_attention(s.q, dim, cross_kv, 2 * dim, cross_kv + dim, 2 * dim, s.attn, dim, 1, n, Tk, heads, scale, 0, 0, cross_len_dev, st);
    linear(s.attn, dim, n, L.cout, ep_residual(x, dim), st);
  }
  ln_linear(x, dim, n, L.final_ln, L.fc1, ep_out(s.hid, ffn, ACT_RELU), s.y, st);
  linear(s.hid, ffn, n, L.fc2, ep_residual(x, dim), st);
}

// keep_rows > 0: rows [0, keep_rows) of every layer survive a reallocation (incremental-state decoding keeps cross K / V across calls)
int ensure_mt_cross(ss_engine* h, int T, int keep_rows = 0) {
  if (T <= h->mt_cross_cap) return SS_OK;
  const int cap = std::max(T + T / 2, 512);
  const size_t row = (size_t)2 * h->cfg.mt_dim;
  float* fresh = nullptr;
  if (cudaMalloc((void**)&fresh, (size_t)h->cfg.mt_layers * cap * row * sizeof(float)) != cudaSuccess) return h->fail(SS_ERR_CUDA, "cudaMalloc(mt cross kv) failed");
  if (h->mt_cross_kv) {
    cudaDeviceSynchronize();  // earlier launches may still read the old buffer
    if (keep_rows > 0)
      for (int l = 0; l < h->cfg.mt_layers; ++l)
        cudaMemcpy(fresh + (size_t)l * cap * row, h->mt_cross_kv + (size_t)l * h->mt_cross_cap * row, (size_t)keep_rows * row * sizeof(float), cudaMemcpyDeviceToDevice);
    cudaFree(h->mt_cross_kv);
  }
  h->mt_cross_kv = fresh;
  h->mt_cross_final = 0;
  h->mt_cross_cap = cap;
  return SS_OK;
}

// run the MT decoder on n tokens (already on the device at h->mt_tok_dev[past .. past+n)) with the KV cache holding `past` rows;
// writes final-LN features to feats[n][dim]
void mt_forward(ss_engine* h, int past, int n, int T, const int* self_kv_len_dev, float* feats, DecScratch& s, float* x, cudaStream_t st) {
  const ss_config& c = h->cfg;
  const int dim = c.mt_dim;
  embed_tokens_pos(h->mt_tok_dev + past, nullptr, past, h->mt_emb, h->mt_pos, sqrtf((float)dim), x, n, dim, c.pad, st);
  for (int l = 0; l < c.mt_layers; ++l) {
    float* ck = h->mt_self_k + (size_t)l * c.max_mt_positions * dim;
    float* cv = h->mt_self_v + (size_t)l * c.max_mt_positions * dim;
    const float* cross = h->mt_cross_kv + (size_t)l * h->mt_cross_cap * 2 * dim;
    dec_layer(h->mt[l], x, n, dim, c.mt_ffn, c.mt_heads, true, 0, self_kv_len_dev, ck, cv, past, cross, T, nullptr, s, st);
  }
  layer_norm(x, dim, feats, dim, h->mt_ln.g, h->mt_ln.b, n, dim, st);
}

// cross-attention K | V of the encoder rows.  Rows the caller declared final (ss_mt_stable_rows) at the previous call were
// projected then and are not touched again; everything above is (re)computed.
void mt_begin(ss_engine* h, const float* enc_dev, int T, cudaStream_t st) {
  const ss_config& c = h->cfg;
  int from = (h->mt_cross_enc == enc_dev) ? std::min(h->mt_cross_final, T) : 0;
  if (from < 0) from = 0;
  if (T > from) {
    for (int l = 0; l < c.mt_layers; ++l) {
      float* cross = h->mt_cross_kv + (size_t)l * h->mt_cross_cap * 2 * c.mt_dim;
      linear(enc_dev + (size_t)from * c.enc_dim, c.enc_dim, T - from, h->mt[l].ckv, ep_out(cross + (size_t)from * 2 * c.mt_dim, 2 * c.mt_dim), st);
    }
  }
  h->mt_cross_final = std::min(h->mt_stable_hint, T);
  h->mt_stable_hint = 0;
  h->mt_cross_enc = enc_dev;
}

DecScratch dec_scratch(ss_engine* h, int n, int dim, int ffn) {
  DecScratch s;
  s.y = h->ws.f32((size_t)n * dim);
  s.q = h->ws.f32((size_t)n * dim);
  s.attn = h->ws.f32((size_t)n * dim);
  s.hid = h->ws.f32((size_t)n * ffn);
  s.qkv = h->ws.f32((size_t)n * 3 * dim);
  s.kv = nullptr;
  return s;
}

// device buffers of the batched greedy search, grown on demand: self K / V for tok_ld positions, cross K / V for Tmax rows per sample
int ensure_mt_batch(ss_engine* h, int tok_ld, int Tmax) {
  const ss_config& c = h->cfg;
  const size_t R = MT_BATCH_MAX_ROWS;
  if (tok_ld > h->mtb_tok_ld || Tmax > h->mtb_cross_cap) cudaDeviceSynchronize();  // earlier launches may still read the old buffers
  if (tok_ld > h->mtb_tok_ld) {
    if (h->mtb_self_kv) cudaFree(h->mtb_self_kv);
    h->mtb_self_kv = nullptr;
    h->mtb_tok_ld = 0;
    if (cudaMalloc((void**)&h->mtb_self_kv, (size_t)2 * c.mt_layers * R * tok_ld * c.mt_dim * sizeof(float)) != cudaSuccess) {
      h->mtb_self_kv = nullptr;
      return h->fail(SS_ERR_CUDA, "cudaMalloc(batched mt self kv) failed");
    }
    h->mtb_tok_ld = tok_ld;
  }
  if (Tmax > h->mtb_cross_cap) {
    const int cap = std::max(Tmax + Tmax / 2, 512);
    if (h->mtb_cross_kv) cudaFree(h->mtb_cross_kv);
    h->mtb_cross_kv = nullptr;
    h->mtb_cross_cap = 0;
    if (cudaMalloc((void**)&h->mtb_cross_kv, (size_t)c.mt_layers * R * cap * 2 * c.mt_dim * sizeof(float)) != cudaSuccess) {
      h->mtb_cross_kv = nullptr;
      return h->fail(SS_ERR_CUDA, "cudaMalloc(batched mt cross kv) failed");
    }
    h->mtb_cross_cap = cap;
  }
  if (!h->mtb_tok_pinned && cudaHostAlloc((void**)&h->mtb_tok_pinned, R * 16 * sizeof(int64_t), cudaHostAllocDefault) != cudaSuccess) {
    h->mtb_tok_pinned = nullptr;
    return h->fail(SS_ERR_CUDA, "cudaHostAlloc(batched mt tokens) failed");
  }
  return SS_OK;
}

// Greedy search of samples g0 .. g0 + Bg - 1 (Bg <= MT_BATCH_MAX_ROWS) on mt_decode_batch_kernel.  Returns SS_OK, an error code
// (reported), or -1 when the first cooperative launch was refused (nothing written to the outputs yet: the caller falls back).
int mt_batch_group(ss_engine* h, cudaStream_t st, const float* enc_dev, int g0, int Bg, int T_stride, const int32_t* T_host, int max_len,
                   int64_t* tokens_out_host, int max_out, int32_t* n_out_host) {
  const ss_config& c = h->cfg;
  const int dim = c.mt_dim;
  const size_t R = MT_BATCH_MAX_ROWS;
  int Tmax = 0;
  for (int b = 0; b < Bg; ++b) Tmax = std::max(Tmax, (int)T_host[g0 + b]);
  int rc = ensure_mt_batch(h, max_len + 2, Tmax);
  if (rc) return rc;
  const int ld = h->mtb_tok_ld;
  // cross K / V: the same projection call as mt_begin with the sample's own row count (the GEMM routing depends on M)
  for (int b = 0; b < Bg; ++b)
    for (int l = 0; l < c.mt_layers; ++l)
      linear(enc_dev + (size_t)(g0 + b) * T_stride * c.enc_dim, c.enc_dim, T_host[g0 + b], h->mt[l].ckv,
             ep_out(h->mtb_cross_kv + ((size_t)l * R + b) * h->mtb_cross_cap * 2 * dim, 2 * dim), st);
  const size_t floats = (size_t)Bg * (dim * 11 + c.mt_ffn + c.tgt_vocab);
  if (!ws_begin(h, floats * sizeof(float) + (size_t)Bg * ld * sizeof(int64_t) + (size_t)Bg * 2 * sizeof(int) + 16 * 256))
    return h->fail(SS_ERR_CUDA, "workspace allocation failed");
  MtBatchParams P;
  P.n_layers = c.mt_layers; P.vocab = c.tgt_vocab; P.pad = c.pad; P.eos = c.eos;
  P.rows = Bg; P.tok_ld = ld; P.cross_cap = h->mtb_cross_cap;
  P.emb = h->mt_emb; P.pos = h->mt_pos; P.out_g = h->mt_ln.g; P.out_b = h->mt_ln.b;
  P.self_k = h->mtb_self_kv; P.self_v = h->mtb_self_kv + (size_t)c.mt_layers * R * ld * dim; P.cross_kv = h->mtb_cross_kv;
  P.q = h->ws.f32((size_t)Bg * dim); P.part = h->ws.f32((size_t)Bg * 8 * dim); P.delta = h->ws.f32((size_t)Bg * dim);
  P.hid = h->ws.f32((size_t)Bg * c.mt_ffn); P.logits = h->ws.f32((size_t)Bg * c.tgt_vocab);
  P.tok = (int64_t*)h->ws.raw((size_t)Bg * ld * sizeof(int64_t));
  int* ints = (int*)h->ws.raw((size_t)Bg * 2 * sizeof(int));  // [fin | cross_len]
  if (!P.q || !P.part || !P.delta || !P.hid || !P.logits || !P.tok || !ints) return h->fail(SS_ERR_CUDA, "workspace too small");
  P.fin = ints;
  P.cross_len = ints + Bg;
  std::vector<int64_t> tok0((size_t)Bg * ld, c.eos);  // column 0 = eos (the decoder's bos); the kernel writes the rest
  std::vector<int> ints0(2 * Bg, 0);
  for (int b = 0; b < Bg; ++b) ints0[Bg + b] = T_host[g0 + b];
  cudaMemcpyAsync(P.tok, tok0.data(), tok0.size() * sizeof(int64_t), cudaMemcpyHostToDevice, st);
  cudaMemcpyAsync(ints, ints0.data(), ints0.size() * sizeof(int), cudaMemcpyHostToDevice, st);
  cudaStreamSynchronize(st);  // (host vectors)
  for (int b = 0; b < Bg; ++b) n_out_host[g0 + b] = 0;
  std::vector<char> done(Bg, 0);
  int active = Bg;
  constexpr int kBurst = 16;  // steps per launch, as ss_mt_greedy; the host reads the tokens back once per burst
  for (int step = 0; step < max_len && active > 0; step += kBurst) {  // step max_len is the forced eos: no work
    const int cnt = std::min(kBurst, max_len - step);
    if (mt_decode_batch(P, h->mt_persist_layers, step, cnt, h->persist_bar, &h->persist_bar_target, st) != 0) {
      cudaGetLastError();
      if (step == 0) return -1;
      return h->fail(SS_ERR_CUDA, "cooperative launch of the batched MT kernel was refused");
    }
    cudaMemcpy2DAsync(h->mtb_tok_pinned, cnt * sizeof(int64_t), P.tok + step + 1, ld * sizeof(int64_t), cnt * sizeof(int64_t), Bg,
                      cudaMemcpyDeviceToHost, st);
    if (h->async_err_pinned) cudaMemcpyAsync(h->async_err_pinned, h->persist_bar + SS_BAR_ERR_WORD, sizeof(unsigned), cudaMemcpyDeviceToHost, st);
    if (cudaStreamSynchronize(st) != cudaSuccess) return h->fail(SS_ERR_CUDA, std::string("ss_mt_greedy_batch: ") + cudaGetErrorString(cudaGetLastError()));
    if (h->async_err_pinned && *h->async_err_pinned) {
      const unsigned f = *h->async_err_pinned;
      *h->async_err_pinned = 0;
      return report_async_error(h, f, "ss_mt_greedy_batch");
    }
    for (int b = 0; b < Bg; ++b) {
      for (int i = 0; i < cnt && !done[b]; ++i) {
        const int64_t next = h->mtb_tok_pinned[(size_t)b * cnt + i];
        if (next == c.eos) {
          done[b] = 1;
          --active;
        } else {
          tokens_out_host[(size_t)(g0 + b) * max_out + n_out_host[g0 + b]++] = next;
        }
      }
    }
  }
  return SS_OK;
}

}  // namespace

extern "C" {

int64_t ss_launch_count(const ss_engine*) { return (int64_t)ss::g_launches; }

int ss_async_error(ss_engine* h) {
  if (!h) return SS_ERR_INVALID;
  if (!h->persist_bar) return SS_OK;
  unsigned f = 0;
  if (cudaMemcpy(&f, h->persist_bar + SS_BAR_ERR_WORD, sizeof(unsigned), cudaMemcpyDeviceToHost) != cudaSuccess)
    return h->fail(SS_ERR_CUDA, std::string("ss_async_error: ") + cudaGetErrorString(cudaGetLastError()));
  return report_async_error(h, f, "ss_async_error");
}

int64_t ss_fbank_num_frames(int64_t n) {
  if (n < 240) return 0;
  int64_t f = (n - 240) / 160;
  return f < 0 ? 0 : f;
}

int64_t ss_encoder_out_frames(int64_t F) {
  if (F <= 0) return 0;
  int64_t t = (F - 1) / 2 + 1;
  return (t - 1) / 2 + 1;
}

int ss_fbank(ss_engine* h, void* stream, const float* samples_dev, int64_t n_samples, int64_t frame0, int64_t n_frames,
             float* out_dev) {
  if (!h || !h->finalized) return h ? h->fail(SS_ERR_STATE, "engine not finalized") : SS_ERR_INVALID;
  if (n_frames <= 0) return SS_OK;
  if (frame0 < 0 || (frame0 + n_frames - 1) * 160 + 400 > n_samples) return h->fail(SS_ERR_INVALID, "fbank frame range exceeds samples");
  if (h->fbank_tma && ((uintptr_t)samples_dev & 15) == 0)  // frames are complete (checked above): the bulk copy never leaves the buffer
    fbank_cmvn_tma(samples_dev, (int)frame0, (int)n_frames, h->melT, h->window, h->cmvn_mean, h->cmvn_std, out_dev, S(stream));
  else
    fbank_cmvn(samples_dev, n_samples, (int)frame0, (int)n_frames, h->mel_bank, h->window, h->cmvn_mean, nullptr, h->cmvn_std, out_dev, S(stream));
  return check_launch(h, "ss_fbank");
}

int64_t ss_resample_out_len(int64_t n_in_48k, int finished) {
  if (n_in_48k <= 0) return 0;
  if (finished) return (n_in_48k + 2) / 3;                 // ceil(n / 3): the whole-signal length of torchaudio.functional.resample
  const int64_t last = (n_in_48k - 22) / 3;                // outputs whose 41-tap support [3i - 19, 3i + 21] is complete
  return n_in_48k >= 22 ? last + 1 : 0;
}

int ss_resample_48k_to_16k(ss_engine* h, void* stream, const float* in_dev, int64_t n_in, int64_t out0, int64_t n_out, float* out_dev) {
  if (!h || !h->finalized) return h ? h->fail(SS_ERR_STATE, "engine not finalized") : SS_ERR_INVALID;
  if (!h->resample_h) return h->fail(SS_ERR_MISSING, "__const__.resample_3to1 was not loaded");
  if (n_out <= 0) return SS_OK;
  if (out0 < 0 || n_in < 0 || out0 + n_out > (n_in + 2) / 3) return h->fail(SS_ERR_INVALID, "resample output range exceeds ceil(n_in / 3)");
  resample_3to1(in_dev, n_in, h->resample_h, h->resample_taps, h->resample_width, out0, (int)n_out, out_dev, S(stream));
  return check_launch(h, "ss_resample_48k_to_16k");
}

int ss_encoder_forward(ss_engine* h, void* stream, const float* feats_dev, const int32_t* lengths_host, int B, int F, float* out_dev) {
  if (h) route_from(h);
  if (!h || !h->finalized) return h ? h->fail(SS_ERR_STATE, "engine not finalized") : SS_ERR_INVALID;
  if (B <= 0 || F <= 0) return h->fail(SS_ERR_INVALID, "empty encoder input");
  const ss_config& c = h->cfg;
  cudaStream_t st = S(stream);
  const int D = c.enc_dim;
  const int T1 = (F - 1) / 2 + 1, T = (T1 - 1) / 2 + 1;
  if (T > h->Tpos) return h->fail(SS_ERR_CAPACITY, "encoder sequence longer than max_enc_frames");
  const size_t rows = (size_t)B * T;
  size_t need = ((size_t)B * T1 * (c.conv_channels / 2) + rows * (size_t)(D * 6 + c.enc_ffn + 3 * D) + 4096) * sizeof(float) + 16 * 256;
  if (!ws_begin(h, need)) return h->fail(SS_ERR_CUDA, "workspace allocation failed");
  float* c1 = h->ws.f32((size_t)B * T1 * (c.conv_channels / 2));
  float* x = out_dev;  // the residual stream lives in the caller's output buffer
  float* y = h->ws.f32(rows * D);
  float* hid = h->ws.f32(rows * c.enc_ffn);
  float* qkv = h->ws.f32(rows * 3 * D);
  float* att = h->ws.f32(rows * D);
  float* glu = h->ws.f32(rows * D);
  float* dw = h->ws.f32(rows * D);
  float* x0 = h->ws.f32(rows * D);
  if (!c1 || !y || !hid || !qkv || !att || !glu || !dw || !x0) return h->fail(SS_ERR_CUDA, "workspace too small");
  // per-sample encoder lengths (Conv1dSubsampler.get_out_seq_lens_tensor, convolution.py:75-79)
  const int* len_dev = nullptr;
  if (lengths_host) {
    bool all_full = true;
    std::vector<int> lens(B);
    for (int b = 0; b < B; ++b) {
      int l = lengths_host[b];
      if (l < 1 || l > F) return h->fail(SS_ERR_INVALID, "bad src_lengths");
      l = (l - 1) / 2 + 1;
      l = (l - 1) / 2 + 1;
      lens[b] = l;
      all_full &= (l == T);
    }
    if (!all_full) {
      if (B > h->lengths_cap) {
        if (h->lengths_dev) cudaFree(h->lengths_dev);
        h->lengths_dev = nullptr;
        h->lengths_cap = 0;
        if (cudaMalloc((void**)&h->lengths_dev, (size_t)B * 2 * sizeof(int)) != cudaSuccess) return h->fail(SS_ERR_CUDA, "cudaMalloc(lengths) failed");
        h->lengths_cap = B * 2;
      }
      if (cudaMemcpyAsync(h->lengths_dev, lens.data(), B * sizeof(int), cudaMemcpyHostToDevice, st) != cudaSuccess ||
          cudaStreamSynchronize(st) != cudaSuccess)  // `lens` is a stack vector
        return h->fail(SS_ERR_CUDA, "copy of src_lengths failed");
      len_dev = h->lengths_dev;
    }
  }
  const int cc = h->conv_chunk;
  // E1: two chunk-causal stride-2 convs + GLU (convolution.py:81-89).  conv_chunk == 0: plain Conv1d(padding=k//2)
  {
    ConvA a;
    a.x = feats_dev; a.B = B; a.L_in = F; a.L_rows = T1; a.C_in = c.feat_dim; a.ldx = c.feat_dim;
    a.ksize = c.conv_kernel; a.stride = 2; a.pad_left = c.conv_kernel / 2; a.chunk = cc;
    Epilogue ep = ep_out(c1, c.conv_channels / 2);
    ep.bias = h->sub_conv[0].b; ep.glu = 1;
    gemm_conv(a, h->sub_conv[0].w, h->sub_conv[0].N, ep, st);
    ConvA a2;
    a2.x = c1; a2.B = B; a2.L_in = T1; a2.L_rows = T; a2.C_in = c.conv_channels / 2; a2.ldx = c.conv_channels / 2;
    a2.ksize = c.conv_kernel; a2.stride = 2; a2.pad_left = c.conv_kernel / 2; a2.chunk = cc;
    Epilogue ep2 = ep_out(x0, D);
    ep2.bias = h->sub_conv[1].b; ep2.glu = 1; ep2.alpha = sqrtf((float)D);  // x = embed_scale * x (s2t_conformer.py:127)
    gemm_conv(a2, h->sub_conv[1].w, h->sub_conv[1].N, ep2, st);
  }
  linear(x0, D, (int)rows, h->enc_linear, ep_out(x, D), st);  // s2t_conformer.py:139
  for (int i = 0; i < c.enc_layers; ++i) {
    const ConformerLayerW& L = h->enc[i];
    // x = x + 0.5 * ffn1(x)
    layer_norm(x, D, y, D, L.ffn1_ln.g, L.ffn1_ln.b, (int)rows, D, st);
    linear(y, D, (int)rows, L.ffn1_w1, ep_out(hid, c.enc_ffn, ACT_SILU), st);
    linear(hid, c.enc_ffn, (int)rows, L.ffn1_w2, ep_residual(x, D, 0.5f), st);
    // x = x + self_attn(LN(x))
    layer_norm(x, D, y, D, L.attn_ln.g, L.attn_ln.b, (int)rows, D, st);
    linear(y, D, (int)rows, L.qkv, ep_out(qkv, 3 * D), st);
    relpos_attention(qkv, 3 * D, qkv + D, 3 * D, qkv + 2 * D, 3 * D, L.pos_proj, h->Tpos, L.pos_u, L.pos_v, att, B, T, 0, T, c.enc_heads, D,
                     h->attn_chunk, len_dev, st);
    linear(att, D, (int)rows, L.attn_out, ep_residual(x, D), st);
    // x = x + conv_module(x)
    layer_norm(x, D, y, D, L.conv_ln.g, L.conv_ln.b, (int)rows, D, st);
    {
      Epilogue ep = ep_out(glu, D);
      ep.glu = 1;
      linear(y, D, (int)rows, L.pw1, ep, st);
    }
    depthwise_bn_silu(glu, D, L.dw_w, L.bn_scale, L.bn_shift, dw, D, B, T, 0, T, D, c.dw_kernel, cc, st);
    linear(dw, D, (int)rows, L.pw2, ep_residual(x, D), st);
    // x = LN(x + 0.5 * ffn2(x))
    layer_norm(x, D, y, D, L.ffn2_ln.g, L.ffn2_ln.b, (int)rows, D, st);
    linear(y, D, (int)rows, L.ffn2_w1, ep_out(hid, c.enc_ffn, ACT_SILU), st);
    linear(hid, c.enc_ffn, (int)rows, L.ffn2_w2, ep_residual(x, D, 0.5f), st);
    layer_norm(x, D, x, D, L.final_ln.g, L.final_ln.b, (int)rows, D, st);
  }
  return check_launch(h, "ss_encoder_forward");
}

int ss_encoder_stream_reset(ss_engine* h) {
  if (!h) return SS_ERR_INVALID;
  h->st_T_final = 0;
  h->mt_cross_final = 0;
  h->mt_stable_hint = 0;
  return SS_OK;
}

int ss_mt_stable_rows(ss_engine* h, int rows) {
  if (!h) return SS_ERR_INVALID;
  h->mt_stable_hint = rows > 0 ? rows : 0;
  return SS_OK;
}

int ss_encoder_stream_step(ss_engine* h, void* stream, const float* feats_dev, int F, float* enc_out_dev, int32_t* T_out, int32_t* T_final_out) {
  if (h) route_from(h);
  if (!h || !h->finalized) return h ? h->fail(SS_ERR_STATE, "engine not finalized") : SS_ERR_INVALID;
  if (h->attn_chunk <= 0 || h->conv_chunk <= 0) return h->fail(SS_ERR_STATE, "streaming encoder needs a chunked model (ss_set_chunk)");
  const ss_config& c = h->cfg;
  cudaStream_t st = S(stream);
  const int D = c.enc_dim;
  if (F <= 0) {
    if (T_out) *T_out = 0;
    if (T_final_out) *T_final_out = h->st_T_final;
    return SS_OK;
  }
  const int T1 = (F - 1) / 2 + 1, T = (T1 - 1) / 2 + 1;
  if (T > h->Tpos) return h->fail(SS_ERR_CAPACITY, "encoder sequence longer than max_enc_frames");
  // Rows of a group [iG, (i+1)G) are final once 4*G*(i+1) fbank frames exist, where G must be a common multiple of the
  // attention chunk and the conv chunk (every chunk grid has a boundary at the group's end): G = lcm.  For nested settings
  // (4/8, 8/8, 16/16) that is the larger one; for 12/8, 24/16, 40/16 ... it is not.
  int G;
  {
    int a = h->attn_chunk, b = h->conv_chunk;
    while (b) { int t = a % b; a = b; b = t; }
    G = h->attn_chunk / a * h->conv_chunk;
  }
  const int a0 = std::min(h->st_T_final, T);
  const int nA = T - a0;
  if (T_out) *T_out = T;
  const int cc = h->conv_chunk;
  if (nA > 0) {
    const int t1_lo = std::max(0, 2 * a0 - (c.conv_kernel / 2));
    const int n1 = T1 - t1_lo;
    size_t need = ((size_t)n1 * (c.conv_channels / 2) + (size_t)nA * (size_t)(6 * D + c.enc_ffn) + 4096) * sizeof(float) + 16 * 256;
    if (!ws_begin(h, need)) return h->fail(SS_ERR_CUDA, "workspace allocation failed");
    float* c1 = h->ws.f32((size_t)n1 * (c.conv_channels / 2));
    float* x0 = h->ws.f32((size_t)nA * D);
    float* y = h->ws.f32((size_t)nA * D);
    float* hid = h->ws.f32((size_t)nA * c.enc_ffn);
    float* qb = h->ws.f32((size_t)nA * D);
    float* att = h->ws.f32((size_t)nA * D);
    float* dw = h->ws.f32((size_t)nA * D);
    if (!c1 || !x0 || !y || !hid || !qb || !att || !dw) return h->fail(SS_ERR_CUDA, "workspace too small");
    float* x = enc_out_dev + (size_t)a0 * D;
    {
      ConvA a;
      a.x = feats_dev; a.B = 1; a.L_in = F; a.L_rows = n1; a.C_in = c.feat_dim; a.ldx = c.feat_dim;
      a.ksize = c.conv_kernel; a.stride = 2; a.pad_left = c.conv_kernel / 2; a.chunk = cc; a.t_offset = t1_lo;
      Epilogue ep = ep_out(c1, c.conv_channels / 2);
      ep.bias = h->sub_conv[0].b; ep.glu = 1;
      gemm_conv(a, h->sub_conv[0].w, h->sub_conv[0].N, ep, st);
      ConvA a2;
      a2.x = c1; a2.B = 1; a2.L_in = T1; a2.L_rows = nA; a2.C_in = c.conv_channels / 2; a2.ldx = c.conv_channels / 2;
      a2.ksize = c.conv_kernel; a2.stride = 2; a2.pad_left = c.conv_kernel / 2; a2.chunk = cc;
      a2.t_offset = a0; a2.x_row0 = t1_lo; a2.x_rows = n1;
      Epilogue ep2 = ep_out(x0, D);
      ep2.bias = h->sub_conv[1].b; ep2.glu = 1; ep2.alpha = sqrtf((float)D);
      gemm_conv(a2, h->sub_conv[1].w, h->sub_conv[1].N, ep2, st);
    }
    linear(x0, D, nA, h->enc_linear, ep_out(x, D), st);
    bool persistent = h->persistent_encoder && encoder_layers_persistent_supported(nA, D, c.enc_ffn, c.enc_heads, T, c.dw_kernel);
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    if (persistent && h->persistent_time) {  // bench: CUDA events on the launching stream around the dominant kernel
      if (h->time_events.size() < 4096 && cudaEventCreate(&ev0) == cudaSuccess && cudaEventCreate(&ev1) == cudaSuccess) {
        cudaEventRecord(ev0, st);
      } else {
        ev0 = ev1 = nullptr;
      }
    }
    bool cluster_done = false;
    if (persistent && h->persistent_encoder_cluster && h->cl_blobs && h->persist_bar &&
        encoder_layers_cluster_supported(nA, D, c.enc_ffn, c.enc_heads, T, c.dw_kernel)) {
      const float* pos_tabs[16];
      for (int i = 0; i < 16; ++i) pos_tabs[i] = i < c.enc_layers ? h->enc[i].pos_proj : nullptr;
      cluster_done = c.enc_layers <= 16 && encoder_layers_cluster(h->persist_layers, h->cl_blobs, c.enc_layers, x, h->st_k, h->st_v, h->st_glu, nA, a0, T, h->Tpos, h->attn_chunk, cc,
                                            c.dw_kernel, h->persist_bar, &h->persist_bar_target, h->persistent_profile ? h->persist_ts : nullptr, pos_tabs, h->cluster_cooperative, st) == 0;
      if (cluster_done) ++h->cl_steps;
      if (!cluster_done) cudaGetLastError();  // refused launch: the one-CTA-per-SM kernel below takes the step
    }
    if (persistent && !cluster_done)
      persistent = encoder_layers_persistent(h->persistent_alias ? h->persist_alias : h->persist_layers, c.enc_layers, x, hid, qb, att, dw, h->st_k, h->st_v, h->st_glu, nA, a0, T, D,
                                             c.enc_ffn, c.enc_heads, h->Tpos, h->attn_chunk, cc, c.dw_kernel,
                                             h->persistent_profile ? h->persist_ts : nullptr,
                                             h->persistent_barrier ? h->persist_bar : nullptr, &h->persist_bar_target,
                                             h->persistent_prefetch, h->persistent_ffn_fused ? h->persist_ffn_scratch : nullptr, st) == 0;
    if (ev0 && ev1) {
      cudaEventRecord(ev1, st);
      // algorithmic bytes of this launch: every GEMM weight once + the K / V caches and relative-position rows the attention reads
      const double wbytes = (double)c.enc_layers * (4.0 * D * c.enc_ffn + 7.0 * D * D) * 4.0;
      const double kvbytes = (double)c.enc_layers * (2.0 * T + (T + nA)) * D * 4.0;
      h->time_events.push_back({ev0, ev1, wbytes + kvbytes});
    }
    if (!persistent) cudaGetLastError();  // a refused cooperative launch falls back to the per-kernel path
    for (int i = 0; i < c.enc_layers && !persistent; ++i) {
      const ConformerLayerW& L = h->enc[i];
      float* kc = h->st_k + (size_t)i * h->Tpos * D;
      float* vc = h->st_v + (size_t)i * h->Tpos * D;
      float* gc = h->st_glu + (size_t)i * h->Tpos * D;
      ln_linear(x, D, nA, L.ffn1_ln, L.ffn1_w1, ep_out(hid, c.enc_ffn, ACT_SILU), y, st);
      linear(hid, c.enc_ffn, nA, L.ffn1_w2, ep_residual(x, D, 0.5f), st);
      // q -> scratch, k / v -> cache rows a0.. (provisional tail rows are overwritten next call)
      ln_qkv_routed(x, D, nA, L.attn_ln, L.qkv, D, qb, D, kc + (size_t)a0 * D, D, vc + (size_t)a0 * D, D, y, st);
      relpos_attention(qb, D, kc, D, vc, D, L.pos_proj, h->Tpos, L.pos_u, L.pos_v, att, 1, nA, a0, T, c.enc_heads, D, h->attn_chunk, nullptr, st);
      linear(att, D, nA, L.attn_out, ep_residual(x, D), st);
      {
        Epilogue ep = ep_out(gc + (size_t)a0 * D, D);
        ep.glu = 1;
        ln_linear(x, D, nA, L.conv_ln, L.pw1, ep, y, st);
      }
      depthwise_bn_silu(gc, D, L.dw_w, L.bn_scale, L.bn_shift, dw, D, 1, T, a0, nA, D, c.dw_kernel, cc, st);
      linear(dw, D, nA, L.pw2, ep_residual(x, D), st);
      ln_linear(x, D, nA, L.ffn2_ln, L.ffn2_w1, ep_out(hid, c.enc_ffn, ACT_SILU), y, st);
      linear(hid, c.enc_ffn, nA, L.ffn2_w2, ep_residual(x, D, 0.5f), st);
      layer_norm(x, D, x, D, L.final_ln.g, L.final_ln.b, nA, D, st);
    }
  }
  h->st_T_final = std::max(h->st_T_final, std::min(T, (F / (4 * G)) * G));
  if (T_final_out) *T_final_out = h->st_T_final;
  return check_launch(h, "ss_encoder_stream_step");
}

int ss_ctc_greedy_rows(ss_engine* h, void* stream, int head, const float* enc_dev, int rows, int row0, int64_t* argmax_dev,
                       int64_t* tokens_dev, int32_t* index_dev, int32_t* count_dev) {
  if (h) route_from(h);
  if (!h || !h->finalized) return h ? h->fail(SS_ERR_STATE, "engine not finalized") : SS_ERR_INVALID;
  if (head < 0 || head > 1 || rows <= 0 || row0 < 0 || row0 > rows) return h->fail(SS_ERR_INVALID, "bad ctc head / rows");
  const Linear& l = h->ctc_head[head];
  cudaStream_t st = S(stream);
  const int nr = rows - row0;  // rows below row0 keep the arg-max the caller cached from an earlier call
  if (nr > 0) {
    if (!ws_begin(h, (size_t)nr * l.N * sizeof(float) + 4096)) return h->fail(SS_ERR_CUDA, "workspace allocation failed");
    float* logits = h->ws.f32((size_t)nr * l.N);
    linear(enc_dev + (size_t)row0 * h->cfg.enc_dim, h->cfg.enc_dim, nr, l, ep_out(logits, l.N), st);
    argmax_rows(logits, l.N, nr, l.N, h->mask_pad_unk, 2, argmax_dev + row0, nullptr, st);  // never select pad, unk
  }
  ctc_collapse(argmax_dev, rows, 0 /* <s> is the CTC blank (agent/ctc_decoder.py:72-76) */, h->cfg.pad, tokens_dev, index_dev, count_dev, st);
  return check_launch(h, "ss_ctc_greedy");
}

int ss_ctc_greedy_pair(ss_engine* h, void* stream, const float* enc_dev, int rows, int row0, int64_t* argmax0_dev, int64_t* argmax1_dev,
                       int64_t* packed_out_dev) {
  if (h) route_from(h);
  if (!h || !h->finalized) return h ? h->fail(SS_ERR_STATE, "engine not finalized") : SS_ERR_INVALID;
  if (rows <= 0 || row0 < 0 || row0 > rows) return h->fail(SS_ERR_INVALID, "bad ctc rows");
  cudaStream_t st = S(stream);
  const int V = h->cfg.src_vocab;
  const int nr = rows - row0;
  const int W = 2 * rows + 2;
  if (h->ctc_pair.N != 2 * V || h->cfg.tgt_vocab != V) {  // different vocabularies: two single-head calls into the same packing
    for (int hd = 0; hd < 2; ++hd) {
      int64_t* o = packed_out_dev + (size_t)hd * W;
      int rc = ss_ctc_greedy_rows(h, stream, hd, enc_dev, rows, row0, hd ? argmax1_dev : argmax0_dev, o + 1, reinterpret_cast<int32_t*>(o + 1 + rows),
                                  reinterpret_cast<int32_t*>(o));
      if (rc) return rc;
    }
    return SS_OK;
  }
  float* logits = nullptr;
  if (nr > 0) {
    if (!ws_begin(h, (size_t)nr * 2 * V * sizeof(float) + 4096)) return h->fail(SS_ERR_CUDA, "workspace allocation failed");
    logits = h->ws.f32((size_t)nr * 2 * V);
    linear(enc_dev + (size_t)row0 * h->cfg.enc_dim, h->cfg.enc_dim, nr, h->ctc_pair, ep_out(logits, 2 * V), st);
  }
  ctc_argmax_collapse_pair(logits, 2 * V, V, nr, row0, rows, h->mask_pad_unk, 2, 0 /* <s> = CTC blank */, h->cfg.pad, argmax0_dev, argmax1_dev,
                           packed_out_dev, W, h->ctc_ticket, st);
  return check_launch(h, "ss_ctc_greedy_pair");
}

int ss_ctc_greedy(ss_engine* h, void* stream, int head, const float* enc_dev, int rows, int64_t* argmax_dev, int64_t* tokens_dev,
                  int32_t* index_dev, int32_t* count_dev) {
  return ss_ctc_greedy_rows(h, stream, head, enc_dev, rows, 0, argmax_dev, tokens_dev, index_dev, count_dev);
}

int ss_mt_features(ss_engine* h, void* stream, const float* enc_dev, int T, const int64_t* tokens_host, int n, float* feats_out_dev,
                   float* logits_last_dev) {
  if (h) route_from(h);
  if (!h || !h->finalized) return h ? h->fail(SS_ERR_STATE, "engine not finalized") : SS_ERR_INVALID;
  const ss_config& c = h->cfg;
  if (n <= 0 || n > c.max_mt_positions || T <= 0) return h->fail(SS_ERR_INVALID, "bad MT sequence length");
  cudaStream_t st = S(stream);
  int rc = ensure_mt_cross(h, T);
  if (rc) return rc;
  int n_valid = n;  // trailing pads (whole_word path, agent:576-591) are masked as keys
  while (n_valid > 0 && tokens_host[n_valid - 1] == c.pad) --n_valid;
  for (int i = 0; i < n_valid; ++i)
    if (tokens_host[i] == c.pad) return h->fail(SS_ERR_INVALID, "pads are only supported as a tail");
  const int dim = c.mt_dim;
  if (!ws_begin(h, ((size_t)n * (dim * 7 + c.mt_ffn) + 4096) * sizeof(float))) return h->fail(SS_ERR_CUDA, "workspace allocation failed");
  DecScratch s = dec_scratch(h, n, dim, c.mt_ffn);
  float* x = h->ws.f32((size_t)n * dim);
  int* kvlen = nullptr;
  cudaMemcpyAsync(h->mt_tok_dev, tokens_host, n * sizeof(int64_t), cudaMemcpyHostToDevice, st);
  if (n_valid < n) {
    kvlen = (int*)h->ws.raw(sizeof(int));
    cudaMemcpyAsync(kvlen, &n_valid, sizeof(int), cudaMemcpyHostToDevice, st);
  }
  cudaStreamSynchronize(st);  // tokens_host / n_valid are caller / stack memory
  mt_begin(h, enc_dev, T, st);
  mt_forward(h, 0, n, T, kvlen, feats_out_dev, s, x, st);
  if (logits_last_dev) {
    Linear out;
    out.w = h->mt_emb; out.b = nullptr; out.N = c.tgt_vocab; out.K = dim;
    linear(feats_out_dev + (size_t)(n - 1) * dim, dim, 1, out, ep_out(logits_last_dev, c.tgt_vocab), st);
  }
  return check_launch(h, "ss_mt_features");
}

int ss_mt_greedy(ss_engine* h, void* stream, const float* enc_dev, int T, const int64_t* prefix_host, int n_prefix, int max_new_tokens,
                 int max_len_b, int64_t* tokens_out_host, int max_out, int* n_out, float* feats_out_dev) {
  if (h) route_from(h);
  if (!h || !h->finalized) return h ? h->fail(SS_ERR_STATE, "engine not finalized") : SS_ERR_INVALID;
  const ss_config& c = h->cfg;
  cudaStream_t st = S(stream);
  if (T <= 0 || n_prefix < 0 || !n_out) return h->fail(SS_ERR_INVALID, "bad arguments to ss_mt_greedy");
  const int start = n_prefix;
  int max_len = (max_new_tokens == -1) ? std::min(max_len_b, c.max_mt_positions - 1) : start + max_new_tokens;
  if (max_len < 1) return h->fail(SS_ERR_INVALID, "min_len cannot be larger than max_len");
  if (start > max_len) return h->fail(SS_ERR_INVALID, "prefix longer than max_len");
  if (max_len + 2 > c.max_mt_positions || max_len > max_out) return h->fail(SS_ERR_CAPACITY, "MT hypothesis longer than capacity");
  int rc = ensure_mt_cross(h, T);
  if (rc) return rc;
  const int dim = c.mt_dim;
  const int nmax = std::max(start + 1, 1);
  const size_t feat_floats = feats_out_dev ? 0 : (size_t)(max_len + 2) * dim;  // no caller buffer: features go to scratch
  if (!ws_begin(h, ((size_t)nmax * (dim * 7 + c.mt_ffn) + c.tgt_vocab + feat_floats + 4096) * sizeof(float))) return h->fail(SS_ERR_CUDA, "workspace allocation failed");
  DecScratch s = dec_scratch(h, nmax, dim, c.mt_ffn);
  float* x = h->ws.f32((size_t)nmax * dim);
  float* logits = h->ws.f32(c.tgt_vocab);
  if (!feats_out_dev) feats_out_dev = h->ws.f32(feat_floats);
  Linear outp;
  outp.w = h->mt_emb; outp.b = nullptr; outp.N = c.tgt_vocab; outp.K = dim;
  // tokens buffer = [eos, prefix...]
  std::vector<int64_t> toks(start + 1);
  toks[0] = c.eos;
  for (int i = 0; i < start; ++i) toks[i + 1] = prefix_host[i];
  cudaMemcpyAsync(h->mt_tok_dev, toks.data(), toks.size() * sizeof(int64_t), cudaMemcpyHostToDevice, st);
  cudaStreamSynchronize(st);
  mt_begin(h, enc_dev, T, st);
  int fed = 0;  // rows in the KV cache
  int n_tok = start;  // hypothesis length so far (without eos)
  for (int i = 0; i < start; ++i) tokens_out_host[i] = prefix_host[i];
  // The arg-max of step s is written straight into the device token buffer at s+1, so consecutive steps need no host
  // round trip.  Steps are enqueued in bursts; the host reads the burst's tokens back once and stops at the first eos
  // (steps enqueued past an eos only produce rows that are never read).
  const int burst = (max_new_tokens >= 0) ? std::max(1, max_new_tokens) : 16;
  const bool persistent_mt = h->persistent_mt && mt_decode_persistent_supported(dim, c.mt_ffn, c.mt_heads, c.tgt_vocab, c.max_mt_positions, T);
  int step = start;
  bool done = false;
  if (persistent_mt && h->persistent_mt_prefix && h->persist_bar && start >= 1 && mt_prefix_persistent_supported(dim, c.mt_ffn, c.mt_heads, start, T)) {
    // rows 0 .. start-1 ([eos, p1 .. p_{start-1}]) in one cooperative launch; the single-token kernel continues at position `start`
    MtDecodeParams P;
    P.n_layers = c.mt_layers; P.heads = c.mt_heads; P.vocab = c.tgt_vocab; P.pad = c.pad; P.eos = c.eos;
    P.max_pos = c.max_mt_positions; P.cross_cap = h->mt_cross_cap;
    P.emb = h->mt_emb; P.pos = h->mt_pos; P.out_g = h->mt_ln.g; P.out_b = h->mt_ln.b;
    P.self_k = h->mt_self_k; P.self_v = h->mt_self_v; P.cross_kv = h->mt_cross_kv;
    P.tok = h->mt_tok_dev; P.feats = feats_out_dev; P.x = x; P.q = s.q; P.attn = s.attn; P.hid = s.hid; P.logits = logits;
        if (h->persistent_mt_v2 && h->mt_part) { P.part = h->mt_part; P.delta = h->mt_part + (size_t)8 * c.mt_dim; }
        if (h->persistent_profile) P.ts = h->persist_ts;
    if (mt_prefix_persistent(P, h->mt_persist_layers, start, T, h->persist_bar, &h->persist_bar_target, st) == 0)
      fed = start;
    else
      cudaGetLastError();  // refused launch: per-kernel path
  }
  while (!done) {
    const int burst_first = step;
    int enq = 0;
    for (; step <= max_len && enq < burst; ++step, ++enq) {
      // feed tokens[fed .. step]  (first iteration: the whole prefix; afterwards one token)
      int n = step + 1 - fed;
      if (n == 1 && persistent_mt && h->persist_bar) {
        // the rest of the burst as ONE cooperative launch (it stops by itself at eos / max_len)
        const int cnt = std::min(max_len - step + 1, burst - enq);
        MtDecodeParams P;
        P.n_layers = c.mt_layers; P.heads = c.mt_heads; P.vocab = c.tgt_vocab; P.pad = c.pad; P.eos = c.eos;
        P.max_pos = c.max_mt_positions; P.cross_cap = h->mt_cross_cap;
        P.emb = h->mt_emb; P.pos = h->mt_pos; P.out_g = h->mt_ln.g; P.out_b = h->mt_ln.b;
        P.self_k = h->mt_self_k; P.self_v = h->mt_self_v; P.cross_kv = h->mt_cross_kv;
        P.tok = h->mt_tok_dev; P.feats = feats_out_dev; P.x = x; P.q = s.q; P.attn = s.attn; P.hid = s.hid; P.logits = logits;
        if (h->persistent_mt_v2 && h->mt_part) { P.part = h->mt_part; P.delta = h->mt_part + (size_t)8 * c.mt_dim; }
        if (h->persistent_profile) P.ts = h->persist_ts;
        cudaEvent_t ev0 = nullptr, ev1 = nullptr;
        if (h->persistent_time && h->mt_time_events.size() < 4096 && cudaEventCreate(&ev0) == cudaSuccess && cudaEventCreate(&ev1) == cudaSuccess)
          cudaEventRecord(ev0, st);
        else
          ev0 = ev1 = nullptr;
        const int rc_launch = mt_decode_persistent(P, h->mt_persist_layers, step, cnt, max_len, T, h->persist_bar, &h->persist_bar_target, st);
        if (ev0 && ev1) {
          cudaEventRecord(ev1, st);
          h->mt_time_events.push_back({ev0, ev1, -1.0});  // steps executed: filled in below once the tokens are read
        }
        if (rc_launch == 0) {
          fed = step + cnt;
          if (step + cnt - 1 >= max_len) done = true;
          step += cnt;
          enq += cnt;
          break;
        }
        cudaGetLastError();  // refused launch: per-kernel path below
      }
      mt_forward(h, fed, n, T, nullptr, feats_out_dev + (size_t)fed * dim, s, x, st);
      fed = step + 1;
      if (step >= max_len) {  // eos is forced here (sequence_generator.py:362-364): no need for the logits
        done = true;
        ++step;
        break;
      }
      linear(feats_out_dev + (size_t)step * dim, dim, 1, outp, ep_out(logits, c.tgt_vocab), st);
      // lprobs[pad] = -inf; eos banned while step < min_len (=1)
      if (step < 1)
        argmax_rows(logits, c.tgt_vocab, 1, c.tgt_vocab, h->mask_pad_eos, 2, h->mt_tok_dev + step + 1, nullptr, st);
      else
        argmax_rows(logits, c.tgt_vocab, 1, c.tgt_vocab, h->mask_pad_unk, 1, h->mt_tok_dev + step + 1, nullptr, st);
    }
    // tokens produced by this burst live at mt_tok_dev[burst_first+1 .. ]; the forced-eos step produced none
    int produced = step - burst_first - (done ? 1 : 0);
    if (produced > 0) {
      cudaMemcpyAsync(h->mt_next_pinned, h->mt_tok_dev + burst_first + 1, produced * sizeof(int64_t), cudaMemcpyDeviceToHost, st);
      if (h->persist_bar && h->async_err_pinned)
        cudaMemcpyAsync(h->async_err_pinned, h->persist_bar + SS_BAR_ERR_WORD, sizeof(unsigned), cudaMemcpyDeviceToHost, st);
      if (cudaStreamSynchronize(st) != cudaSuccess)
        return h->fail(SS_ERR_CUDA, std::string("ss_mt_greedy: ") + cudaGetErrorString(cudaGetLastError()));
      if (h->async_err_pinned && *h->async_err_pinned) {
        const unsigned f = *h->async_err_pinned;
        *h->async_err_pinned = 0;
        return report_async_error(h, f, "ss_mt_greedy");
      }
      int steps_run = produced;
      for (int i = 0; i < produced; ++i) {
        int64_t next = h->mt_next_pinned[i];
        if (next == c.eos) {
          done = true;
          steps_run = i + 1;  // (the kernel stops after the step that produced eos)
          break;
        }
        tokens_out_host[n_tok++] = next;
      }
      if (!h->mt_time_events.empty() && h->mt_time_events.back().bytes < 0.0) h->mt_time_events.back().bytes = (double)steps_run;
    }
    if (step > max_len) done = true;
  }
  *n_out = n_tok;
  return check_launch(h, "ss_mt_greedy");
}

int ss_mt_greedy_batch(ss_engine* h, void* stream, const float* enc_dev, int B, int T_stride, const int32_t* T_host, int max_len_b,
                       int64_t* tokens_out_host, int max_out, int32_t* n_out_host) {
  if (h) route_from(h);
  if (!h || !h->finalized) return h ? h->fail(SS_ERR_STATE, "engine not finalized") : SS_ERR_INVALID;
  const ss_config& c = h->cfg;
  if (B <= 0 || T_stride <= 0 || !enc_dev || !T_host || !tokens_out_host || !n_out_host)
    return h->fail(SS_ERR_INVALID, "bad arguments to ss_mt_greedy_batch");
  int Tmax = 0;
  for (int b = 0; b < B; ++b) {
    if (T_host[b] < 1 || T_host[b] > T_stride) return h->fail(SS_ERR_INVALID, "ss_mt_greedy_batch: sample length outside [1, T_stride]");
    Tmax = std::max(Tmax, (int)T_host[b]);
  }
  const int max_len = std::min(max_len_b, c.max_mt_positions - 1);
  if (max_len < 1) return h->fail(SS_ERR_INVALID, "min_len cannot be larger than max_len");
  if (max_len + 2 > c.max_mt_positions || max_len > max_out) return h->fail(SS_ERR_CAPACITY, "MT hypothesis longer than capacity");
  cudaStream_t st = S(stream);
  // the batched kernel reproduces the rows of the 6-barrier single-token kernel: it runs where ss_mt_greedy would run that one
  const bool batched = h->persistent_mt && h->persistent_mt_v2 && h->mt_part && h->persist_bar && c.mt_heads == 8 &&
                       mt_decode_persistent_supported(c.mt_dim, c.mt_ffn, c.mt_heads, c.tgt_vocab, c.max_mt_positions, Tmax);
  for (int g0 = 0; g0 < B; g0 += MT_BATCH_MAX_ROWS) {
    const int Bg = std::min(MT_BATCH_MAX_ROWS, B - g0);
    if (batched && Bg >= h->mt_batch_min_rows) {
      const int rc = mt_batch_group(h, st, enc_dev, g0, Bg, T_stride, T_host, max_len, tokens_out_host, max_out, n_out_host);
      if (rc != -1) {
        if (rc) return rc;
        continue;
      }
    }
    // sample by sample on ss_mt_greedy's path.  It uses the single-stream MT buffers, so their cross K / V cache is marked
    // invalid afterwards (a streaming call on this handle then projects every row again) and a pending stable-rows hint is kept.
    const int hint = h->mt_stable_hint;
    h->mt_stable_hint = 0;
    int rc = SS_OK;
    for (int b = g0; b < g0 + Bg && rc == SS_OK; ++b) {
      int n = 0;
      rc = ss_mt_greedy(h, stream, enc_dev + (size_t)b * T_stride * c.enc_dim, T_host[b], nullptr, 0, -1, max_len_b,
                        tokens_out_host + (size_t)b * max_out, max_out, &n, nullptr);
      n_out_host[b] = n;
    }
    h->mt_cross_enc = nullptr;
    h->mt_cross_final = 0;
    h->mt_stable_hint = hint;
    if (rc) return rc;
  }
  return check_launch(h, "ss_mt_greedy_batch");
}

int ss_mt_incremental_reset(ss_engine* h) {
  if (!h) return SS_ERR_INVALID;
  h->mt_inc_self_len = 0;
  h->mt_inc_cross_rows = 0;
  return SS_OK;
}

int ss_mt_greedy_incremental(ss_engine* h, void* stream, const float* enc_dev, int T, const int64_t* prefix_host, int n_prefix,
                             int max_new_tokens, int max_len_b, int64_t* tokens_out_host, int max_out, int* n_out) {
  if (h) route_from(h);
  if (!h || !h->finalized) return h ? h->fail(SS_ERR_STATE, "engine not finalized") : SS_ERR_INVALID;
  const ss_config& c = h->cfg;
  cudaStream_t st = S(stream);
  if (T <= 0 || n_prefix < 0 || !n_out) return h->fail(SS_ERR_INVALID, "bad arguments to ss_mt_greedy_incremental");
  const int start = n_prefix;
  const int max_len = (max_new_tokens == -1) ? max_len_b : start + max_new_tokens;
  if (max_len < 1) return h->fail(SS_ERR_INVALID, "min_len cannot be larger than max_len");
  if (start > max_len) return h->fail(SS_ERR_INVALID, "prefix longer than max_len");
  // slot of the token at position s = s + kv_off; the first call starts with an empty cache (kv_off = 0), every later call
  // re-feeds the last prefix token on top of the entry the previous call's final step left (kv_off grows by one per call)
  const int kv_off = h->mt_inc_self_len - start;
  if (kv_off < 0) return h->fail(SS_ERR_STATE, "incremental MT state is shorter than the prefix (reset missing, or a prefix that this state did not produce)");
  if (max_len + kv_off + 2 > c.max_mt_positions || max_len > max_out) return h->fail(SS_ERR_CAPACITY, "MT hypothesis longer than capacity");
  if (!h->persistent_mt || !h->persist_bar || !mt_decode_persistent_supported(c.mt_dim, c.mt_ffn, c.mt_heads, c.tgt_vocab, c.max_mt_positions, std::max(T, h->mt_inc_cross_rows)))
    return h->fail(SS_ERR_STATE, "incremental MT decoding runs on the persistent MT kernel, which is off or does not support this shape");
  int rc = ensure_mt_cross(h, std::max(T, h->mt_inc_cross_rows), h->mt_inc_cross_rows);
  if (rc) return rc;
  const int dim = c.mt_dim;
  if (!ws_begin(h, ((size_t)(dim * 8 + c.mt_ffn) + c.tgt_vocab + (size_t)c.max_mt_positions * dim + 4096) * sizeof(float))) return h->fail(SS_ERR_CUDA, "workspace allocation failed");
  DecScratch s = dec_scratch(h, 1, dim, c.mt_ffn);
  float* x = h->ws.f32(dim);
  float* logits = h->ws.f32(c.tgt_vocab);
  float* feats = h->ws.f32((size_t)c.max_mt_positions * dim);
  if (!x || !logits || !feats) return h->fail(SS_ERR_CUDA, "workspace too small");
  // cross K / V: only the encoder rows that were not there at the previous call are projected and appended; older rows keep
  // the projections of the (then provisional) encoder output of the call that first saw them (N12)
  if (h->mt_inc_cross_rows == 0) {  // a fresh state must not inherit rows of an earlier utterance
    h->mt_cross_final = 0;
    h->mt_cross_enc = nullptr;
  }
  if (T > h->mt_inc_cross_rows) {
    const int from = h->mt_inc_cross_rows;
    for (int l = 0; l < c.mt_layers; ++l) {
      float* cross = h->mt_cross_kv + (size_t)l * h->mt_cross_cap * 2 * dim;
      linear(enc_dev + (size_t)from * c.enc_dim, c.enc_dim, T - from, h->mt[l].ckv, ep_out(cross + (size_t)from * 2 * dim, 2 * dim), st);
    }
    h->mt_inc_cross_rows = T;
  }
  const int Tk = h->mt_inc_cross_rows;
  std::vector<int64_t> toks(start + 1);
  toks[0] = c.eos;
  for (int i = 0; i < start; ++i) toks[i + 1] = prefix_host[i];
  cudaMemcpyAsync(h->mt_tok_dev, toks.data(), toks.size() * sizeof(int64_t), cudaMemcpyHostToDevice, st);
  cudaStreamSynchronize(st);
  int n_tok = start;
  for (int i = 0; i < start; ++i) tokens_out_host[i] = prefix_host[i];
  const int burst = (max_new_tokens >= 0) ? std::max(1, max_new_tokens + 1) : 32;
  int step = start;
  bool done = false;
  while (!done) {
    const int cnt = std::min(max_len - step + 1, burst);
    MtDecodeParams P;
    P.n_layers = c.mt_layers; P.heads = c.mt_heads; P.vocab = c.tgt_vocab; P.pad = c.pad; P.eos = c.eos;
    P.max_pos = c.max_mt_positions; P.cross_cap = h->mt_cross_cap; P.kv_off = kv_off;
    P.emb = h->mt_emb; P.pos = h->mt_pos; P.out_g = h->mt_ln.g; P.out_b = h->mt_ln.b;
    P.self_k = h->mt_self_k; P.self_v = h->mt_self_v; P.cross_kv = h->mt_cross_kv;
    P.tok = h->mt_tok_dev; P.feats = feats; P.x = x; P.q = s.q; P.attn = s.attn; P.hid = s.hid; P.logits = logits;
        if (h->persistent_mt_v2 && h->mt_part) { P.part = h->mt_part; P.delta = h->mt_part + (size_t)8 * c.mt_dim; }
        if (h->persistent_profile) P.ts = h->persist_ts;
    if (mt_decode_persistent(P, h->mt_persist_layers, step, cnt, max_len, Tk, h->persist_bar, &h->persist_bar_target, st) != 0) {
      cudaGetLastError();
      return h->fail(SS_ERR_CUDA, "cooperative launch of the persistent MT kernel was refused");
    }
    const int readable = std::min(cnt, max_len - step);  // the forced-eos step writes no token
    if (readable > 0) cudaMemcpyAsync(h->mt_next_pinned, h->mt_tok_dev + step + 1, readable * sizeof(int64_t), cudaMemcpyDeviceToHost, st);
    if (h->async_err_pinned) cudaMemcpyAsync(h->async_err_pinned, h->persist_bar + SS_BAR_ERR_WORD, sizeof(unsigned), cudaMemcpyDeviceToHost, st);
    if (cudaStreamSynchronize(st) != cudaSuccess) return h->fail(SS_ERR_CUDA, std::string("ss_mt_greedy_incremental: ") + cudaGetErrorString(cudaGetLastError()));
    if (h->async_err_pinned && *h->async_err_pinned) {
      const unsigned f = *h->async_err_pinned;
      *h->async_err_pinned = 0;
      return report_async_error(h, f, "ss_mt_greedy_incremental");
    }
    for (int i = 0; i < cnt && !done; ++i) {
      const int sidx = step + i;            // this step fed the token at position sidx (one more cache entry)
      h->mt_inc_self_len = sidx + kv_off + 1;
      if (sidx >= max_len) { done = true; break; }   // eos forced (sequence_generator.py:362-364)
      const int64_t next = h->mt_next_pinned[i];
      if (next == c.eos) { done = true; break; }
      tokens_out_host[n_tok++] = next;
    }
    step += cnt;
    if (step > max_len) done = true;
  }
  *n_out = n_tok;
  return check_launch(h, "ss_mt_greedy_incremental");
}

int ss_t2u_unit_decode(ss_engine* h, void* stream, const float* mt_feats_dev, int Slen, int n_pad_tail, int mask_eos, int64_t* argmax_dev,
                       int64_t* units_dev, int32_t* count_dev, float* t2u_out_dev, float* logits_dev) {
  if (h) route_from(h);
  if (!h || !h->finalized) return h ? h->fail(SS_ERR_STATE, "engine not finalized") : SS_ERR_INVALID;
  const ss_config& c = h->cfg;
  cudaStream_t st = S(stream);
  if (Slen <= 0 || n_pad_tail < 0 || n_pad_tail >= Slen) return h->fail(SS_ERR_INVALID, "bad T2U sequence length");
  const int dim = c.unit_dim, R = c.ctc_upsample_rate, L = Slen * R;
  size_t need = ((size_t)L * (dim * 8 + c.unit_ffn + c.unit_vocab) + (size_t)Slen * dim * 12 + (size_t)Slen * c.unit_ffn + 8192) * sizeof(float);
  if (!ws_begin(h, need)) return h->fail(SS_ERR_CUDA, "workspace allocation failed");
  // ---- T1: UniTransformerEncoderNoEmb.forward
  DecScratch s1 = dec_scratch(h, Slen, dim, c.unit_ffn);
  float* x = h->ws.f32((size_t)Slen * dim);
  float* t2u = t2u_out_dev ? t2u_out_dev : h->ws.f32((size_t)Slen * dim);
  int* kvlen = nullptr;
  int* kvlen_up = nullptr;
  if (n_pad_tail > 0) {  // encoder_padding_mask on the trailing pad positions
    int v[2] = {Slen - n_pad_tail, (Slen - n_pad_tail) * R};
    kvlen = (int*)h->ws.raw(2 * sizeof(int));
    kvlen_up = kvlen + 1;
    cudaMemcpyAsync(kvlen, v, sizeof(v), cudaMemcpyHostToDevice, st);
    cudaStreamSynchronize(st);
  }
  copy_f32(mt_feats_dev, x, (int64_t)Slen * dim, st);
  for (int l = 0; l < c.t2u_layers; ++l)
    dec_layer(h->t2u[l], x, Slen, dim, c.unit_ffn, c.unit_heads, c.uni_encoder != 0, 0, kvlen, nullptr, nullptr, 0, nullptr, 0, nullptr, s1, st);
  layer_norm(x, dim, t2u, dim, h->t2u_ln.g, h->t2u_ln.b, Slen, dim, st);
  // ---- U1: CTCTransformerUnitDecoder: x25 upsample + (quirky) positional embedding, 2 layers, out-proj
  DecScratch s2 = dec_scratch(h, L, dim, c.unit_ffn);
  float* xu = h->ws.f32((size_t)L * dim);
  float* ckv = h->ws.f32((size_t)Slen * 2 * dim);
  float* logits = logits_dev ? logits_dev : h->ws.f32((size_t)L * c.unit_vocab);
  if (!xu || !ckv || !logits) return h->fail(SS_ERR_CUDA, "workspace too small");
  repeat_rows_add(t2u, Slen, R, dim, h->unit_pos_row, xu, st);
  for (int l = 0; l < c.unit_layers; ++l) {
    linear(t2u, dim, Slen, h->unit[l].ckv, ep_out(ckv, 2 * dim), st);
    // layer 0 sees R identical copies of every T2U state (same positional row for every step, N1): grouped self-attention
    const int gR = (l == 0 && h->unit_grouped) ? R : 0;
    dec_layer(h->unit[l], xu, L, dim, c.unit_ffn, c.unit_heads, true, 0, kvlen_up, nullptr, nullptr, 0, ckv, Slen, kvlen, s2, st, gR, kvlen);
  }
  layer_norm(xu, dim, xu, dim, h->unit_ln.g, h->unit_ln.b, L, dim, st);
  Linear outp;
  outp.w = h->unit_emb; outp.b = nullptr; outp.N = c.unit_vocab; outp.K = dim;
  linear(xu, dim, L, outp, ep_out(logits, c.unit_vocab), st);
  // ---- U2: never select pad, unk (agent version) [+ eos: offline version]
  argmax_rows(logits, c.unit_vocab, L, c.unit_vocab, h->mask_pad_unk, mask_eos ? 3 : 2, argmax_dev, nullptr, st);
  ctc_collapse(argmax_dev, L, c.unit_vocab - 1, c.pad, units_dev, nullptr, count_dev, st);
  return check_launch(h, "ss_t2u_unit_decode");
}

int ss_unit_position_row(ss_engine* h, const float* row_host) {
  if (!h || !h->finalized || !row_host) return h ? h->fail(SS_ERR_STATE, "engine not finalized / null row") : SS_ERR_INVALID;
  cudaDeviceSynchronize();  // earlier unit-decoder launches may still read the old row
  if (cudaMemcpy(h->unit_pos_row, row_host, (size_t)h->cfg.unit_dim * sizeof(float), cudaMemcpyHostToDevice) != cudaSuccess)
    return h->fail(SS_ERR_CUDA, "cudaMemcpy(unit positional row) failed");
  return SS_OK;
}

int ss_vocoder_durations(ss_engine* h, void* stream, const int64_t* codes_dev, int U, int dur_prediction, int64_t* dur_out_dev,
                         int32_t* cumsum_out_dev) {
  if (!h || !h->finalized) return h ? h->fail(SS_ERR_STATE, "engine not finalized") : SS_ERR_INVALID;
  if (!h->has_vocoder) return h->fail(SS_ERR_STATE, "no vocoder weights were loaded");
  if (U <= 0) return h->fail(SS_ERR_INVALID, "empty code sequence");
  const ss_config& c = h->cfg;
  cudaStream_t st = S(stream);
  const int E = c.voc_embedding_dim, Hd = c.voc_dur_hidden;
  if (U > h->voc_ucap) {
    if (h->voc_unit_emb) cudaFree(h->voc_unit_emb);
    if (h->voc_cumsum) cudaFree(h->voc_cumsum);
    h->voc_unit_emb = nullptr;
    h->voc_cumsum = nullptr;
    h->voc_ucap = 0;
    const int cap = std::max(2 * U, 1024);
    if (cudaMalloc((void**)&h->voc_unit_emb, (size_t)cap * E * sizeof(float)) != cudaSuccess ||
        cudaMalloc((void**)&h->voc_cumsum, (size_t)(cap + 1) * sizeof(int)) != cudaSuccess)
      return h->fail(SS_ERR_CUDA, "cudaMalloc(vocoder unit cache) failed");
    h->voc_ucap = cap;
  }
  h->voc_U = U;
  if (!ws_begin(h, ((size_t)U * (2 * Hd + 2) + 4096) * sizeof(float))) return h->fail(SS_ERR_CUDA, "workspace allocation failed");
  gather_rows(codes_dev, U, 0, h->voc_dict, E, h->voc_unit_emb, st);
  float* a = h->ws.f32((size_t)U * Hd);
  float* b = h->ws.f32((size_t)U * Hd);
  float* ld = h->ws.f32(U);
  if (dur_prediction) {
    // VariancePredictor.forward (fairseq/models/text_to_speech/fastspeech2.py:144-151)
    ConvA c1;
    c1.x = h->voc_unit_emb; c1.B = 1; c1.L_in = U; c1.L_rows = U; c1.C_in = E; c1.ldx = E;
    c1.ksize = h->dur_conv1.ksize; c1.pad_left = (h->dur_conv1.ksize - 1) / 2;
    Epilogue e1 = ep_out(a, Hd, ACT_RELU);
    e1.bias = h->dur_conv1.lin.b;
    gemm_conv(c1, h->dur_conv1.lin.w, Hd, e1, st);
    layer_norm(a, Hd, a, Hd, h->dur_ln1.g, h->dur_ln1.b, U, Hd, st);
    ConvA c2;
    c2.x = a; c2.B = 1; c2.L_in = U; c2.L_rows = U; c2.C_in = Hd; c2.ldx = Hd;
    c2.ksize = h->dur_conv2.ksize; c2.pad_left = 1;  // padding=1 is hard-coded for conv2 (fastspeech2.py:137)
    Epilogue e2 = ep_out(b, Hd, ACT_RELU);
    e2.bias = h->dur_conv2.lin.b;
    gemm_conv(c2, h->dur_conv2.lin.w, Hd, e2, st);
    layer_norm(b, Hd, b, Hd, h->dur_ln2.g, h->dur_ln2.b, U, Hd, st);
    linear(b, Hd, U, h->dur_proj, ep_out(ld, 1), st);
  } else {
    // no duration prediction: every code is one frame; log(2) rounds to dur 1
    std::vector<float> v(U, 0.6931472f);
    cudaMemcpyAsync(ld, v.data(), U * sizeof(float), cudaMemcpyHostToDevice, st);
    cudaStreamSynchronize(st);
  }
  duration_from_log(ld, U, dur_out_dev, h->voc_cumsum, st);
  if (cumsum_out_dev) cudaMemcpyAsync(cumsum_out_dev, h->voc_cumsum, (U + 1) * sizeof(int), cudaMemcpyDeviceToDevice, st);
  return check_launch(h, "ss_vocoder_durations");
}

int ss_vocoder_generate(ss_engine* h, void* stream, int total_frames, int frame0, int n_frames, int left_context, float* wav_out_dev) {
  if (!h || !h->finalized) return h ? h->fail(SS_ERR_STATE, "engine not finalized") : SS_ERR_INVALID;
  if (!h->has_vocoder || h->voc_U <= 0) return h->fail(SS_ERR_STATE, "ss_vocoder_durations must run first");
  if (n_frames <= 0 || frame0 < 0 || frame0 + n_frames != total_frames) return h->fail(SS_ERR_INVALID, "vocoder frame range must be the tail of the sequence");
  const ss_config& c = h->cfg;
  cudaStream_t st = S(stream);
  route_from(h);
  g_umma_conv = h->umma_vocoder;
  int ctx = left_context < 0 ? h->receptive_field : left_context;
  ctx = std::min(ctx, frame0);
  const int f_lo = frame0 - ctx;
  const int N = n_frames + ctx;
  // workspace: input frames + per-stage buffers
  size_t maxbuf = 0;
  {
    int ch = c.voc_init_channels;
    size_t L = N;
    maxbuf = L * ch;
    for (int i = 0; i < c.voc_n_ups; ++i) {
      L *= c.voc_up_rates[i];
      ch /= 2;
      maxbuf = std::max(maxbuf, L * ch);
    }
  }
  const int nrb = c.voc_n_rb;
  size_t total = ((size_t)N * c.voc_in_dim + (size_t)(2 + 4 * nrb) * maxbuf + (size_t)N * h->hop + 8192) * sizeof(float) + 64 * 256;
  if (!ws_begin(h, total)) return h->fail(SS_ERR_CUDA, "workspace allocation failed");
  float* frames = h->ws.f32((size_t)N * c.voc_in_dim);
  float* bufX = h->ws.f32(maxbuf);   // stage input / output
  float* bufY = h->ws.f32(maxbuf);   // upsampled stage activation
  // per resblock (they run concurrently): ping-pong pair, conv1 output, block output
  std::vector<float*> rbA(nrb), rbB(nrb), rbT(nrb), rbO(nrb);
  bool ok = frames && bufX && bufY;
  for (int j = 0; j < nrb; ++j) {
    rbA[j] = h->ws.f32(maxbuf); rbB[j] = h->ws.f32(maxbuf); rbT[j] = h->ws.f32(maxbuf); rbO[j] = h->ws.f32(maxbuf);
    ok = ok && rbA[j] && rbB[j] && rbT[j] && rbO[j];
  }
  float* wav = h->ws.f32((size_t)N * h->hop);
  if (!ok || !wav) return h->fail(SS_ERR_CUDA, "workspace too small");
  // The resblocks of a stage are independent until their outputs are averaged (hifigan.py:158-165).  Each one is a chain of
  // small latency-bound convs, so they run on separate streams (block 0 on the caller's) and overlap on the GPU.
  const bool fan_out = h->vocoder_streams && nrb == 3 && (g_umma_conv == 0 || g_umma_conv >= 12);
  if (fan_out && !h->fork_event) {
    bool made = cudaEventCreateWithFlags(&h->fork_event, cudaEventDisableTiming) == cudaSuccess;
    for (int i = 0; i < 2 && made; ++i)
      made = cudaStreamCreateWithFlags(&h->aux_stream[i], cudaStreamNonBlocking) == cudaSuccess &&
             cudaEventCreateWithFlags(&h->join_event[i], cudaEventDisableTiming) == cudaSuccess;
    if (!made) return h->fail(SS_ERR_CUDA, "cannot create the vocoder's auxiliary streams");
  }
  // V1 tail: repeat_interleave(x, dur) for the frame window (agent/tts/codehifigan.py:66)
  expand_frames(h->voc_unit_emb, h->voc_cumsum, h->voc_U, f_lo, N, c.voc_embedding_dim, frames, st);
  // Short sequences (the streaming calls): conv_pre .. conv_post as one persistent kernel whose phases are separated by grid
  // barriers.  A shape it does not support or a refused cooperative launch falls through to the multi-launch path below.
  const bool fused = h->vocoder_fused != 0 && (h->vocoder_fused == 1 || N <= kVocFusedMaxFrames) && g_umma_conv == 12 && nrb == 3 &&
                     h->persist_bar != nullptr;
  if (fused) {
    VocFusedParams* P = vocoder_fused_table(h, N, frames, bufX, bufY, rbA, rbB, rbT, rbO, st);
    if (P) {
      VocPost& post = P->post;
      post.x0 = rbO[0]; post.x1 = rbO[1]; post.x2 = rbO[2];
      post.w = h->conv_post_w; post.bias = h->conv_post_b; post.slope = 0.01f;  // leaky_relu(x) [slope 0.01, hifigan.py:166]
      post.L = N * h->hop; post.C = h->conv_post_c; post.k = h->conv_post_k; post.t0 = ctx * h->hop;
      post.out = wav_out_dev;
      if (vocoder_fused(*P, h->persist_bar, &h->persist_bar_target, st) == 0) return check_launch(h, "ss_vocoder_generate");
    }
  }
  // Everything from conv_pre to conv_post depends on the call only through N (buffer addresses are arena offsets): ~190
  // launches on three streams whose host enqueue time exceeds their GPU time.  With option vocoder_graph the sequence is
  // recorded once per (N, arena, routing) by stream capture and replayed as one CUDA graph afterwards.
  auto generator_body = [&](cudaStream_t st) {
  // conv_pre
  {
    ConvA a;
    a.x = frames; a.B = 1; a.L_in = N; a.L_rows = N; a.C_in = c.voc_in_dim; a.ldx = c.voc_in_dim; a.ksize = 7; a.pad_left = 3;
    Epilogue e = ep_out(bufX, c.voc_init_channels);
    e.bias = h->conv_pre.lin.b;
    conv_gemm(a, h->conv_pre.lin.w, c.voc_init_channels, e, st);
  }
  int L = N, ch = c.voc_init_channels;
  for (int i = 0; i < c.voc_n_ups; ++i) {
    const UpsampleW& U = h->ups[i];
    const int Lout = L * U.u;
    // x = ups[i](leaky_relu(x, 0.1)): one GEMM per output phase, rows scattered with stride u.  The phases are independent
    // (disjoint output rows): they are spread over the same three streams as the resblocks below.
    const bool fan_up = fan_out && U.u > 1;
    if (fan_up) {
      cudaEventRecord(h->fork_event, st);
      for (int q = 0; q < 2; ++q) cudaStreamWaitEvent(h->aux_stream[q], h->fork_event, 0);
    }
    for (int phi = 0; phi < U.u; ++phi) {
      int J = U.phase_J[phi], q0 = U.phase_q0[phi];
      int qmax = (Lout - 1 - phi + U.pad) / U.u;
      int nrows = qmax - q0 + 1;
      if (nrows <= 0) continue;
      const int lane = fan_up ? phi % 3 : 0;
      cudaStream_t sp = lane > 0 ? h->aux_stream[lane - 1] : st;
      set_splitk_slot(lane);
      ConvA a;
      a.x = bufX; a.B = 1; a.L_in = L; a.L_rows = nrows; a.C_in = U.cin; a.ldx = U.cin; a.ksize = J; a.pad_left = (J - 1) - q0;
      a.pre_lrelu = 0.1f;
      Epilogue e = ep_out(bufY, U.cout);
      e.bias = U.bias;
      e.out_L = Lout; e.out_row_stride = U.u; e.out_row_offset = q0 * U.u + phi - U.pad;
      conv_gemm(a, U.phase_w[phi].w, U.cout, e, sp);
    }
    set_splitk_slot(0);
    if (fan_up)
      for (int q = 0; q < 2; ++q) {
        cudaEventRecord(h->join_event[q], h->aux_stream[q]);
        cudaStreamWaitEvent(st, h->join_event[q], 0);
      }
    L = Lout;
    ch = U.cout;
    // xs = sum_j resblock_j(x) / num_kernels  (hifigan.py:158-165); ResBlock.forward :95-102
    if (fan_out) {
      cudaEventRecord(h->fork_event, st);
      for (int q = 0; q < 2; ++q) cudaStreamWaitEvent(h->aux_stream[q], h->fork_event, 0);
    }
    for (int j = 0; j < nrb; ++j) {
      cudaStream_t sj = (fan_out && j > 0) ? h->aux_stream[j - 1] : st;
      set_splitk_slot(fan_out ? j : 0);
      const float* cur = bufY;
      float* pingpong[2] = {rbA[j], rbB[j]};
      int nd = c.voc_rb_ndil;
      for (int m = 0; m < nd; ++m) {
        const ConvW& w1 = h->rb1[i][j][m];
        const ConvW& w2 = h->rb2[i][j][m];
        ConvA a1;
        a1.x = cur; a1.B = 1; a1.L_in = L; a1.L_rows = L; a1.C_in = ch; a1.ldx = ch; a1.ksize = w1.ksize; a1.dil = w1.dil;
        a1.pad_left = (w1.ksize * w1.dil - w1.dil) / 2; a1.pre_lrelu = 0.1f;
        Epilogue e1 = ep_out(rbT[j], ch);
        e1.bias = w1.lin.b;
        conv_gemm(a1, w1.lin.w, ch, e1, sj);
        ConvA a2;
        a2.x = rbT[j]; a2.B = 1; a2.L_in = L; a2.L_rows = L; a2.C_in = ch; a2.ldx = ch; a2.ksize = w2.ksize; a2.dil = 1;
        a2.pad_left = (w2.ksize - 1) / 2; a2.pre_lrelu = 0.1f;
        Epilogue e2;
        e2.bias = w2.lin.b;
        e2.ldo = ch;
        e2.residual = cur;  // x = xt + x
        if (m + 1 < nd) {
          e2.out = pingpong[m & 1];
          e2.res_scale = 1.0f;
        } else {
          // last pair of the block: (xt + x) / num_kernels, summed over the blocks below
          e2.out = nrb == 3 ? rbO[j] : bufX;
          e2.alpha = 1.0f / nrb;
          e2.res_scale = 1.0f / nrb;
          e2.accumulate = nrb != 3 && j > 0;  // (other block counts: accumulate in place, single stream)
        }
        conv_gemm(a2, w2.lin.w, ch, e2, sj);
        cur = e2.out;
      }
      if (fan_out && j > 0) cudaEventRecord(h->join_event[j - 1], sj);
    }
    set_splitk_slot(0);
    if (fan_out)
      for (int q = 0; q < 2; ++q) cudaStreamWaitEvent(st, h->join_event[q], 0);
    // stage output in the reference's summation order: block 0, then + block 1, then + block 2
    if (nrb == 3) add3_f32(rbO[0], rbO[1], rbO[2], bufX, (int64_t)L * ch, st);
  }
  // x = leaky_relu(x) [slope 0.01, hifigan.py:166]; conv_post; tanh
  conv_post_tanh(bufX, L, ch, h->conv_post_w, h->conv_post_b, h->conv_post_k, 0.01f, wav, st);
  };
  bool replayed = false;
  if (h->vocoder_graph) {
    const auto key = std::make_tuple(N, (uintptr_t)h->ws.base, g_umma_conv, g_umma_min_rows * 4096 + g_umma_min_channels, h->vocoder_streams);
    auto it = h->voc_graphs.find(key);
    if (it != h->voc_graphs.end()) {
      if (cudaGraphLaunch(it->second.first, st) == cudaSuccess) {
        g_launches += it->second.second;
        replayed = true;
      } else {
        cudaGetLastError();
      }
    } else {
      // first sight of this key: run eagerly now (that also performs every lazy initialisation: packed weights, split
      // scratch, function attributes), then record the same sequence for the next call.  The capture runs on an
      // engine-owned stream because the caller's stream may be the legacy default stream, which cannot be captured.
      generator_body(st);
      replayed = true;
      if (!h->capture_stream) cudaStreamCreateWithFlags(&h->capture_stream, cudaStreamNonBlocking);
      const unsigned long long before = g_launches;
      if (h->capture_stream && cudaStreamBeginCapture(h->capture_stream, cudaStreamCaptureModeRelaxed) == cudaSuccess) {
        g_pdl_off = h->graph_pdl ? 0 : 1;
        generator_body(h->capture_stream);
        g_pdl_off = 0;
        cudaGraph_t graph = nullptr;
        cudaGraphExec_t exec = nullptr;
        if (cudaStreamEndCapture(h->capture_stream, &graph) == cudaSuccess && graph != nullptr &&
            cudaGraphInstantiate(&exec, graph, 0) == cudaSuccess) {
          h->voc_graphs[key] = std::make_pair(exec, (int)(g_launches - before));
        } else {
          cudaGetLastError();
          h->vocoder_graph = 0;  // capture is not possible here: stay on the eager path
        }
        if (graph) cudaGraphDestroy(graph);
      } else {
        cudaGetLastError();
        h->vocoder_graph = 0;
      }
      g_launches = before;
    }
  }
  if (!replayed) generator_body(st);
  copy_f32(wav + (size_t)ctx * h->hop, wav_out_dev, (int64_t)n_frames * h->hop, st);
  return check_launch(h, "ss_vocoder_generate");
}

int ss_set_option(ss_engine* h, const char* name, int value) {
  if (!h || !name) return SS_ERR_INVALID;
  std::string n(name);
  if (n == "umma_vocoder") h->umma_vocoder = value;
  else if (n == "umma_linear") h->umma_linear = value;
  else if (n == "umma_min_rows") h->umma_min_rows = value;
  else if (n == "umma_min_channels") h->umma_min_channels = value;
  else if (n == "umma2_cache_clear") {  // debug tools that reuse a weight address
    umma2_cache_clear(h->umma2_cache);
    clear_graphs(h);
  }
  else if (n == "umma2_split_below") { g_umma2_split_below = value; clear_graphs(h); }
  else if (n == "umma2_min_units") { g_umma2_min_units = value; clear_graphs(h); }
  else if (n == "umma2_debug") {
    if (value && !g_umma2_dbg) {
      if (cudaMalloc(&g_umma2_dbg, 16 * sizeof(unsigned long long)) != cudaSuccess) return h->fail(SS_ERR_CUDA, "cudaMalloc failed");
      cudaMemset(g_umma2_dbg, 0, 16 * sizeof(unsigned long long));
    }
    if (!value && g_umma2_dbg) {
      cudaDeviceSynchronize();
      cudaFree(g_umma2_dbg);
      g_umma2_dbg = nullptr;
    }
  }
  else if (n == "prefer_shared") g_prefer_shared = value;  // takes effect for kernels that have not been launched yet
  else if (n == "unit_grouped") h->unit_grouped = value;
  else if (n == "vocoder_graph") h->vocoder_graph = value;
  else if (n == "vocoder_fused") h->vocoder_fused = value;
  else if (n == "graph_pdl") h->graph_pdl = value;
  else if (n == "fbank_tma") h->fbank_tma = value;
  else if (n == "umma2_fused_reduce") g_umma2_fused_reduce = value;
  else if (n == "persistent_encoder") h->persistent_encoder = value;
  else if (n == "persistent_ffn_fused") h->persistent_ffn_fused = value;
  else if (n == "cluster_cooperative") h->cluster_cooperative = value;  // 0: plain cluster launch (ncu cannot replay cooperative cluster launches)
  else if (n == "persistent_encoder_cluster") {  // kernels_persist_cl.cu: weights repacked once into per-(layer, rank) blobs
    if (value && !h->cl_blobs) {
      if (!h->persist_layers || !h->persist_bar) return h->fail(SS_ERR_STATE, "persistent_encoder_cluster needs a finalized engine");
      const size_t n_f = encoder_layers_cluster_blob_floats(h->cfg.enc_layers);
      if (h->cfg.enc_dim != 256 || h->cfg.enc_ffn != 2048) return h->fail(SS_ERR_INVALID, "persistent_encoder_cluster: encoder must be 256 / 2048");
      if (cudaMalloc(&h->cl_blobs, n_f * sizeof(float)) != cudaSuccess) return h->fail(SS_ERR_CUDA, "cudaMalloc failed");
      h->dev_allocs.push_back(h->cl_blobs);
      encoder_layers_cluster_pack(h->persist_layers, h->cfg.enc_layers, h->cfg.dw_kernel, h->cl_blobs, 0);
      if (cudaDeviceSynchronize() != cudaSuccess) return h->fail(SS_ERR_CUDA, "packing the cluster weight blobs failed");
    }
    h->persistent_encoder_cluster = value;
  }
  else if (n == "vocoder_streams") h->vocoder_streams = value;
  else if (n == "persistent_mt") h->persistent_mt = value;
  else if (n == "persistent_mt_prefix") h->persistent_mt_prefix = value;
  else if (n == "persistent_mt_v2") h->persistent_mt_v2 = value;
  else if (n == "mt_batch_min_rows") h->mt_batch_min_rows = value;
  else if (n == "persistent_prefetch") h->persistent_prefetch = value;
  else if (n == "persistent_time") h->persistent_time = value;
  else if (n == "persistent_barrier") {
    if (value && !h->persist_bar) {
      if (cudaMalloc(&h->persist_bar, 256) != cudaSuccess) return h->fail(SS_ERR_CUDA, "cudaMalloc failed");
      h->dev_allocs.push_back(h->persist_bar);
      cudaMemset(h->persist_bar, 0, 256);
      h->persist_bar_target = 0;
    }
    h->persistent_barrier = value;
  }
  else if (n == "persistent_alias") {  // timing experiment: all layers read layer 0's weights (results are wrong)
    if (value && !h->persist_alias) {
      const int L = h->cfg.enc_layers;
      if (cudaMalloc(&h->persist_alias, L * sizeof(PersistLayer)) != cudaSuccess) return h->fail(SS_ERR_CUDA, "cudaMalloc failed");
      h->dev_allocs.push_back(h->persist_alias);
      for (int i = 0; i < L; ++i) cudaMemcpy(h->persist_alias + i, h->persist_layers, sizeof(PersistLayer), cudaMemcpyDeviceToDevice);
    }
    h->persistent_alias = value;
  }
  else if (n == "persistent_profile") {
    if (value && !h->persist_ts) {
      if (cudaMalloc(&h->persist_ts, 4096 * sizeof(unsigned long long)) != cudaSuccess) return h->fail(SS_ERR_CUDA, "cudaMalloc failed");
      h->dev_allocs.push_back(h->persist_ts);
    }
    h->persistent_profile = value;
  }
  else return h->fail(SS_ERR_INVALID, "unknown option " + n);
  return SS_OK;
}

int ss_debug_copy(ss_engine* h, const char* what, void* host_dst, size_t bytes) {
  if (!h || !what || !host_dst) return SS_ERR_INVALID;
  std::string n(what);
  if (n == "persist_ts") {
    if (!h->persist_ts || bytes > 4096 * sizeof(unsigned long long)) return h->fail(SS_ERR_STATE, "no phase timestamps (set option persistent_profile)");
    if (cudaMemcpy(host_dst, h->persist_ts, bytes, cudaMemcpyDeviceToHost) != cudaSuccess) return h->fail(SS_ERR_CUDA, "cudaMemcpy failed");
    return SS_OK;
  }
  if (n == "umma2_ts") {
    if (!g_umma2_dbg || bytes > 16 * sizeof(unsigned long long)) return h->fail(SS_ERR_STATE, "no stamps (set option umma2_debug)");
    if (cudaMemcpy(host_dst, g_umma2_dbg, bytes, cudaMemcpyDeviceToHost) != cudaSuccess) return h->fail(SS_ERR_CUDA, "cudaMemcpy failed");
    return SS_OK;
  }
  if (n == "cluster_steps") {  // long long: encoder steps taken by the cluster kernel so far
    if (bytes < sizeof(long long)) return h->fail(SS_ERR_INVALID, "cluster_steps needs a long long");
    *(long long*)host_dst = h->cl_steps;
    return SS_OK;
  }
  if (n == "mt_time") {  // double[3] = {summed ms, launches, summed steps} of the single-token MT kernel since the last query
    if (bytes < 3 * sizeof(double)) return h->fail(SS_ERR_INVALID, "mt_time needs 3 doubles");
    cudaDeviceSynchronize();
    double* out = (double*)host_dst;
    out[0] = out[1] = out[2] = 0.0;
    for (auto& e : h->mt_time_events) {
      float ms = 0.f;
      if (e.bytes >= 0.0 && cudaEventElapsedTime(&ms, e.e0, e.e1) == cudaSuccess) {
        out[0] += ms;
        out[1] += 1.0;
        out[2] += e.bytes;
      }
      cudaEventDestroy(e.e0);
      cudaEventDestroy(e.e1);
    }
    cudaGetLastError();
    h->mt_time_events.clear();
    return SS_OK;
  }
  // double[3] = {summed ms, launches, summed algorithmic bytes} since the last query, of the persistent encoder kernel
  // ("persist_time") or of the stream pool's resample kernel ("pool_resample_time")
  if (n == "persist_time" || n == "pool_resample_time") {
    if (bytes < 3 * sizeof(double)) return h->fail(SS_ERR_INVALID, n + " needs 3 doubles");
    std::vector<ss_engine::TimedLaunch>& events = n == "persist_time" ? h->time_events : h->pool.resample_events;
    cudaDeviceSynchronize();
    double* out = (double*)host_dst;
    out[0] = out[1] = out[2] = 0.0;
    for (auto& e : events) {
      float ms = 0.f;
      if (cudaEventElapsedTime(&ms, e.e0, e.e1) == cudaSuccess) {
        out[0] += ms;
        out[1] += 1.0;
        out[2] += e.bytes;
      }
      cudaEventDestroy(e.e0);
      cudaEventDestroy(e.e1);
    }
    cudaGetLastError();
    events.clear();
    return SS_OK;
  }
  return h->fail(SS_ERR_INVALID, "unknown debug buffer " + n);
}

int ss_op_linear_umma(ss_engine* h, void* stream, const float* x_dev, int M, int K, const float* w_dev, const float* bias_dev, int N, int act,
                      int pieces, float* out_dev) {
  if (!h) return SS_ERR_INVALID;
  route_from(h);
  if (pieces != 2 && pieces != 3) return h->fail(SS_ERR_INVALID, "pieces must be 2 (bf16x3) or 3 (bf16x6)");
  ConvA a;
  a.x = x_dev; a.B = 1; a.L_in = M; a.L_rows = M; a.C_in = K; a.ldx = K;
  Epilogue ep = ep_out(out_dev, N, act);
  ep.bias = bias_dev;
  if (!umma2_supported(a, N, ep)) return h->fail(SS_ERR_INVALID, "shape not supported by the wgmma kernel");
  umma2_conv(h->umma2_cache, a, w_dev, N, ep, pieces, S(stream));
  return check_launch(h, "ss_op_linear_umma");
}

int ss_op_conv1d(ss_engine* h, void* stream, const float* x_dev, int L, int C_in, const float* w_dev, const float* bias_dev, int N, int ksize,
                 int dil, int pad_left, float pre_lrelu, int mode, float* out_dev) {
  if (!h) return SS_ERR_INVALID;
  route_from(h);
  ConvA a;
  a.x = x_dev; a.B = 1; a.L_in = L; a.L_rows = L; a.C_in = C_in; a.ldx = C_in; a.ksize = ksize; a.dil = dil; a.pad_left = pad_left;
  a.pre_lrelu = pre_lrelu;
  Epilogue ep = ep_out(out_dev, N);
  ep.bias = bias_dev;
  if (mode >= 12) {
    if (!umma2_supported(a, N, ep)) return h->fail(SS_ERR_INVALID, "shape not supported by the wgmma conv kernel");
    umma2_conv(h->umma2_cache, a, w_dev, N, ep, mode - 10, S(stream));
  } else if (mode >= 2) {
    return h->fail(SS_ERR_INVALID, "modes 2 / 3 (first-generation tensor-core kernel) were removed: use 12 / 13");
  } else {
    gemm_conv(a, w_dev, N, ep, S(stream));
  }
  return check_launch(h, "ss_op_conv1d");
}

int ss_op_linear(ss_engine* h, void* stream, const float* x_dev, int M, int K, const float* w_dev, const float* bias_dev, int N, int act,
                 float* out_dev) {
  if (!h) return SS_ERR_INVALID;
  Linear l;
  l.w = const_cast<float*>(w_dev); l.b = const_cast<float*>(bias_dev); l.N = N; l.K = K;
  linear(x_dev, K, M, l, ep_out(out_dev, N, act), S(stream));
  return check_launch(h, "ss_op_linear");
}

int ss_op_layer_norm(ss_engine* h, void* stream, const float* x_dev, int rows, int C, const float* g_dev, const float* b_dev, float* out_dev) {
  if (!h) return SS_ERR_INVALID;
  layer_norm(x_dev, C, out_dev, C, g_dev, b_dev, rows, C, S(stream));
  return check_launch(h, "ss_op_layer_norm");
}

}  // extern "C"

#include "engine_pool.inc"
