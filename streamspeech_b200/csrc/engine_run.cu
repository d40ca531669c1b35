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

// entries that project encoder rows through the CTC heads, which a UnitY checkpoint does not have: SS_ERR_STATE before anything is read
int refuse_without_ctc(ss_engine* h, const char* where) {
  return h->fail(SS_ERR_STATE, std::string(where) + ": this model has no CTC heads (source_unigram_decoder.proj and "
                               "ctc_target_unigram_decoder.proj were not loaded: a UnitY checkpoint)");
}

int check_launch(ss_engine* h, const char* where) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return h->fail(SS_ERR_CUDA, std::string(where) + ": " + cudaGetErrorString(e));
  return SS_OK;
}

// The GEMM kernels behind linear() / conv_gemm(), numbered as ss_op_gemm_args.kernel: 1 = gemm_conv, 2 = skinny_gemm, 3 / 4 = umma2_conv
// with 2 / 3 bf16 pieces per operand.
enum GemmKernel : int { GK_GEMM_CONV = 1, GK_SKINNY = 2, GK_UMMA2 = 3, GK_UMMA3 = 4 };
int umma_kernel(int option) { return option - 10 >= 3 ? GK_UMMA3 : GK_UMMA2; }  // option 12 / 13 (umma_vocoder, umma_linear)

// conv-as-GEMM routing of the vocoder: the wgmma split-bf16 kernel (kernels_umma2.cu; umma_vocoder 12 / 13 = 2 / 3 bf16 pieces per
// operand) when enabled and the shape fits, the fp32 CUDA-core kernel otherwise
int conv_gemm_kernel(const ss_engine* h, const ConvA& a, int N, const Epilogue& ep) {
  const int rows = a.B * a.L_rows;
  if (h->umma_vocoder >= 12 && rows >= h->umma_min_rows && a.C_in >= h->umma_min_channels && umma2_supported(a, N, ep))
    return umma_kernel(h->umma_vocoder);
  return GK_GEMM_CONV;
}

// lane: the split-K region of the launching stream
void conv_gemm(ss_engine* h, const ConvA& a, const float* W, int N, const Epilogue& ep, int lane, cudaStream_t st) {
  if (conv_gemm_kernel(h, a, N, ep) != GK_GEMM_CONV)
    umma2_conv(h->umma2_cache, a, W, N, ep, h->umma_vocoder - 10, &h->splitk[lane], st);
  else
    gemm_conv(a, W, N, ep, &h->splitk[lane], st);
}

// routing of a plain linear (a: x as B = 1, L_in = L_rows = M, C_in = K, ldx).  samples > 1: x stacks that many samples of equal row
// counts.  The tensor-core routing is decided from one sample's rows (M / samples), so that a sample's GEMMs take the same class of
// kernel (fp32 or wgmma) as in the single-sample call: the batch then reproduces the single-sample rounding instead of adding the
// split-bf16 error.
int linear_kernel(const ss_engine* h, const ConvA& a, int N, const Epilogue& ep, int samples) {
  const int M = a.L_rows;
  if (skinny_gemm_supported(M, N, a.C_in, ep) && (a.ldx & 3) == 0) return GK_SKINNY;
  if (h->umma_linear >= 12 && M / samples >= h->umma_min_rows && umma2_supported(a, N, ep)) return umma_kernel(h->umma_linear);
  return GK_GEMM_CONV;
}

// plain linear: out[M][N] = epilogue(x[M][K] @ W^T)
void linear(ss_engine* h, const float* x, int ldx, int M, const Linear& l, Epilogue ep, cudaStream_t st, int samples = 1) {
  ConvA a;
  a.x = x; a.B = 1; a.L_in = M; a.L_rows = M; a.C_in = l.K; a.ldx = ldx;
  ep.bias = l.b;
  switch (linear_kernel(h, a, l.N, ep, samples)) {
    case GK_SKINNY: skinny_gemm(x, ldx, l.w, M, l.N, l.K, ep, st); break;
    case GK_GEMM_CONV: gemm_conv(a, l.w, l.N, ep, &h->splitk[0], st); break;
    default: umma2_conv(h->umma2_cache, a, l.w, l.N, ep, h->umma_linear - 10, &h->splitk[0], st); break;
  }
}
// out = epilogue(LayerNorm(x) @ W^T).  The LN is fused into the skinny kernel's A load when the shape allows it,
// otherwise it is a separate launch into `scratch` [M][K].
void ln_linear(ss_engine* h, const float* x, int ldx, int M, const LNorm& ln, const Linear& l, Epilogue ep, float* scratch, cudaStream_t st,
               int samples = 1) {
  ep.bias = l.b;
  Epilogue fused = ep;
  fused.ln_gamma = ln.g;
  fused.ln_beta = ln.b;
  if (ln.C == l.K && (ldx & 3) == 0 && skinny_gemm_supported(M, l.N, l.K, fused)) {
    skinny_gemm(x, ldx, l.w, M, l.N, l.K, fused, st);
    return;
  }
  layer_norm(x, ldx, scratch, l.K, ln.g, ln.b, M, l.K, st);
  linear(h, scratch, l.K, M, l, ep, st, samples);
}

// q | k | v = LayerNorm(x) @ Wqkv^T with the three column blocks routed to their own buffers (query scratch, K cache
// rows, V cache rows).  One launch on the skinny path; LN + three GEMMs otherwise.
void ln_qkv_routed(ss_engine* h, const float* x, int ldx, int M, const LNorm& ln, const Linear& qkv, int dim, float* q, int ldq, float* k, int ldk,
                   float* v, int ldv, float* scratch, cudaStream_t st, int samples = 1) {
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
    linear(h, scratch, qkv.K, M, part, e, st, samples);
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

// Read-back of a burst of MT steps: `rows` rows of `width` tokens at a device pitch of `pitch` tokens (width 0: nothing to read)
// into dst_pinned [rows][width], and the barrier error word; then one synchronisation.  A timed-out grid barrier is reported.
int sync_burst(ss_engine* h, cudaStream_t st, int64_t* dst_pinned, const int64_t* src_dev, int width, int pitch, int rows, const char* where) {
  if (width > 0)
    cudaMemcpy2DAsync(dst_pinned, width * sizeof(int64_t), src_dev, pitch * sizeof(int64_t), width * sizeof(int64_t), rows, cudaMemcpyDeviceToHost, st);
  if (h->async_err_pinned) cudaMemcpyAsync(h->async_err_pinned, h->persist_bar + SS_BAR_ERR_WORD, sizeof(unsigned), cudaMemcpyDeviceToHost, st);
  if (cudaStreamSynchronize(st) != cudaSuccess) return h->fail(SS_ERR_CUDA, std::string(where) + ": " + cudaGetErrorString(cudaGetLastError()));
  if (h->async_err_pinned && *h->async_err_pinned) {
    const unsigned f = *h->async_err_pinned;
    *h->async_err_pinned = 0;
    return report_async_error(h, f, where);
  }
  return SS_OK;
}

void clear_voc_fused(ss_engine* h) {
  cudaDeviceSynchronize();
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
// Frames of one ragged generate group: its sequences share the workspace buffers (~14 x 20 KB per frame at the default
// generator), so a group of 3072 frames holds four 750-frame utterances in 0.9 GB (one 750-frame call alone: 0.2 GB).
constexpr int kVocGroupFrames = 3072;
// k-tiles (16 columns each) per split-K slice of the duration predictor's GEMMs: fixed, so that a row's sums do not depend on the
// call's row count
constexpr int kVocDurTilesPerSplit = 4;

// Job / phase templates of the fused generator over `cap` frames of the arena's buffers (built once per (cap, arena) and kept on
// the handle).  nullptr when a shape is outside what the kernel supports.
VocFusedParams* vocoder_fused_table(ss_engine* h, int cap, const float* frames, float* bufX, float* bufY, const std::vector<float*>& rbA,
                                    const std::vector<float*>& rbB, const std::vector<float*>& rbT, const std::vector<float*>& rbO) {
  const auto key = std::make_pair(cap, (uintptr_t)h->ws.base);
  auto it = h->voc_fused.find(key);
  if (it != h->voc_fused.end()) return &it->second;
  const ss_config& c = h->cfg;
  std::vector<VocJob> jobs;
  std::vector<VocPhase> phases;
  int a_stride = 0;
  bool ok = true;
  auto job = [&](const float* x0, const float* x1, const float* x2, int in_mult, int C_in, int k, int dil, int pad_left, float slope,
                 const float* W, const float* bias, float* out, int Nout, int stride, int offset, int m_adj, const float* residual,
                 float alpha, float res_scale) {
    VocJob j{};
    j.x0 = x0; j.x1 = x1; j.x2 = x2; j.in_mult = in_mult; j.C_in = C_in; j.ksize = k; j.dil = dil; j.pad_left = pad_left; j.slope = slope;
    j.wp = reinterpret_cast<const unsigned char*>(W);  // the fp32 weights: packed per tile width by the calls (vocoder_fused_fill)
    j.bias = bias; j.out = out; j.N = Nout; j.out_row_stride = stride; j.out_row_offset = offset; j.m_adj = m_adj;
    j.residual = residual; j.alpha = alpha; j.res_scale = res_scale;
    j.CK = (C_in % 32 == 0) ? 32 : 16;
    if (C_in % 16 != 0 || Nout % 16 != 0 || k < 1 || (k - 1) * dil > 50 || bias == nullptr) ok = false;
    const int rs_pad = ((VOC_FUSED_BM + (k - 1) * dil + 7) & ~7) + 4;
    a_stride = std::max(a_stride, 2 * (j.CK / 8) * rs_pad * 16);
    jobs.push_back(j);
  };
  // closes the phase of jobs [first, end): longest jobs first
  auto phase = [&](int first) {
    std::stable_sort(jobs.begin() + first, jobs.end(), [](const VocJob& a, const VocJob& b) { return a.ksize > b.ksize; });
    phases.push_back(VocPhase{first, (int)jobs.size() - first, 0});
  };
  jobs.reserve(1 + c.voc_n_ups * (8 + 2 * c.voc_n_rb * c.voc_rb_ndil));
  job(frames, nullptr, nullptr, 1, c.voc_in_dim, 7, 1, 3, 1.0f, h->conv_pre.lin.w, h->conv_pre.lin.b, bufX, c.voc_init_channels, 1, 0, 0,
      nullptr, 1.0f, 1.0f);
  phase(0);
  const int nrb = c.voc_n_rb, nd = c.voc_rb_ndil;
  int mult = 1;  // rows per frame of the stage input
  for (int i = 0; i < c.voc_n_ups; ++i) {
    const UpsampleW& U = h->ups[i];
    // stage input: conv_pre's output, or the previous stage's three resblock outputs summed while loading
    const float* x0 = i == 0 ? bufX : rbO[0];
    const float* x1 = i == 0 ? nullptr : rbO[1];
    const float* x2 = i == 0 ? nullptr : rbO[2];
    int first = (int)jobs.size();
    // output phase phi owns rows q0 .. (L * u - 1 - phi + pad) / u of its phase: M = L + floor((pad - 1 - phi) / u) - (q0 - 1)
    for (int phi = 0; phi < U.u; ++phi) {
      const int J = U.phase_J[phi], q0 = U.phase_q0[phi], a = U.pad - 1 - phi;
      const int m_adj = (a >= 0 ? a / U.u : -((-a + U.u - 1) / U.u)) - (q0 - 1);
      job(x0, x1, x2, mult, U.cin, J, 1, (J - 1) - q0, 0.1f, U.phase_w[phi].w, U.bias, bufY, U.cout, U.u, q0 * U.u + phi - U.pad, m_adj, nullptr,
          1.0f, 1.0f);
    }
    phase(first);
    mult *= U.u;
    const int ch = U.cout;
    for (int m = 0; m < nd; ++m) {
      first = (int)jobs.size();
      for (int j = 0; j < nrb; ++j) {
        const ConvW& w1 = h->rb1[i][j][m];
        const float* cur = m == 0 ? bufY : (m == 1 ? rbA[j] : rbB[j]);
        job(cur, nullptr, nullptr, mult, ch, w1.ksize, w1.dil, (w1.ksize * w1.dil - w1.dil) / 2, 0.1f, w1.lin.w, w1.lin.b, rbT[j], ch, 1, 0, 0,
            nullptr, 1.0f, 1.0f);
      }
      phase(first);
      first = (int)jobs.size();
      for (int j = 0; j < nrb; ++j) {
        const ConvW& w2 = h->rb2[i][j][m];
        const float* cur = m == 0 ? bufY : (m == 1 ? rbA[j] : rbB[j]);
        float* out = m + 1 < nd ? (m == 0 ? rbA[j] : rbB[j]) : rbO[j];
        const float s = m + 1 < nd ? 1.0f : 1.0f / nrb;  // last pair of the block: (xt + x) / num_kernels
        job(rbT[j], nullptr, nullptr, mult, ch, w2.ksize, 1, (w2.ksize - 1) / 2, 0.1f, w2.lin.w, w2.lin.b, out, ch, 1, 0, 0, cur, s, s);
      }
      phase(first);
    }
  }
  if (!ok || jobs.size() > VOC_MAX_JOBS || phases.size() > VOC_MAX_PHASES) return nullptr;
  if (h->voc_fused.size() >= 64) h->voc_fused.clear();
  VocFusedParams& p = h->voc_fused[key];
  std::copy(jobs.begin(), jobs.end(), p.jobs);
  std::copy(phases.begin(), phases.end(), p.phases);
  p.n_phases = (int)phases.size();
  p.a_stride = a_stride;
  p.post.x0 = rbO[0]; p.post.x1 = rbO[1]; p.post.x2 = rbO[2];
  p.post.w = h->conv_post_w; p.post.bias = h->conv_post_b; p.post.slope = 0.01f;  // leaky_relu(x) [slope 0.01, hifigan.py:166]
  p.post.hop = h->hop; p.post.C = h->conv_post_c; p.post.k = h->conv_post_k;
  return &p;
}

// One fused-kernel sequence of a ragged generate call: N frames at row0 of the group's frame buffer, the new samples from frame
// ctx on, written to wav_out + dst.
struct VocFusedSeq {
  int N, row0, ctx, dst;
};

// Fills h->voc_call from template T for the sequences `seqs`.  Each sequence gets the tile widths and tiles a call with that
// sequence alone takes: the 32-column width in a phase when its own 32-column items would fill the grid.  False when the packed
// weights cannot be made or shared memory would exceed what the kernel is set up for.
bool vocoder_fused_fill(ss_engine* h, VocFusedParams& T, const std::vector<VocFusedSeq>& seqs, float* wav_out, cudaStream_t st) {
  const int grid = vocoder_fused_grid();
  if (grid <= 0 || seqs.empty() || (int)seqs.size() > VOC_MAX_STREAMS) return false;
  VocFusedParams& p = h->voc_call;
  std::copy(T.jobs, T.jobs + VOC_MAX_JOBS, p.jobs);
  std::copy(T.phases, T.phases + VOC_MAX_PHASES, p.phases);
  p.n_phases = T.n_phases;
  p.a_stride = T.a_stride;
  p.post = T.post;
  p.post.out = wav_out;
  p.n_streams = (int)seqs.size();
  int out0 = 0;
  for (size_t s = 0; s < seqs.size(); ++s) {
    VocStreamGeo& G = p.streams[s];
    G.bn32 = 0;
    G.N = seqs[s].N; G.row0 = seqs[s].row0; G.t0 = seqs[s].ctx * h->hop; G.out0 = out0; G.dst = seqs[s].dst;
    out0 += (G.N - seqs[s].ctx) * h->hop;
  }
  p.post.total = out0;
  auto m_tiles = [](const VocJob& J, int N) {
    const int M = N * J.in_mult + J.m_adj;
    return M > 0 ? (M + VOC_FUSED_BM - 1) / VOC_FUSED_BM : 0;
  };
  int b_stride = 0;
  for (int ph = 0; ph < p.n_phases; ++ph) {
    const VocPhase& P = p.phases[ph];
    int items = 0;
    bool use16[VOC_MAX_JOBS] = {}, use32[VOC_MAX_JOBS] = {};
    for (size_t s = 0; s < seqs.size(); ++s) {
      VocStreamGeo& G = p.streams[s];
      int items32 = 0;
      for (int jb = P.first_job; jb < P.first_job + P.n_jobs; ++jb)
        items32 += p.jobs[jb].N % 32 == 0 ? m_tiles(p.jobs[jb], G.N) * (p.jobs[jb].N / 32) : 0;
      const bool bn32 = items32 >= grid;  // 16-column tiles when 32-column ones would leave SMs idle
      if (bn32) G.bn32 |= 1ull << ph;
      p.item0[ph][s] = items;
      for (int jb = P.first_job; jb < P.first_job + P.n_jobs; ++jb) {
        const VocJob& J = p.jobs[jb];
        const int mt = m_tiles(J, G.N);
        if (mt == 0) continue;
        const int BN = (bn32 && J.N % 32 == 0) ? 32 : 16;
        (BN == 32 ? use32 : use16)[jb] = true;
        items += mt * (J.N / BN);
      }
    }
    p.phases[ph].n_items = items;
    for (int jb = P.first_job; jb < P.first_job + P.n_jobs; ++jb) {
      VocJob& J = T.jobs[jb];
      const float* W = reinterpret_cast<const float*>(J.wp);
      for (int BN : {16, 32}) {
        if (!(BN == 32 ? use32 : use16)[jb]) continue;
        const unsigned char*& wp = BN == 32 ? J.wp32 : J.wp16;
        if (!wp) wp = umma2_packed_weights(h->umma2_cache, W, J.N, J.C_in, J.ksize, BN, J.CK, 2, st);
        if (!wp) return false;
        (BN == 32 ? p.jobs[jb].wp32 : p.jobs[jb].wp16) = wp;
        b_stride = std::max(b_stride, J.ksize * 2 * BN * J.CK * 2);
      }
    }
  }
  p.b_stride = b_stride;
  return vocoder_fused_smem(p.a_stride, p.b_stride) <= 200 * 1024;
}

struct DecScratch {
  float *y, *q, *kv, *attn, *hid, *qkv;
};

// pre-LN transformer layer over x[n][dim] (TransformerDecoderLayerBase.forward / TransformerEncoderLayerBase.forward,
// ctc_unity/modules/transformer_layer.py:165-230,388-551).  Self-attention keys/values come either from the
// layer's own fused qkv (full sequence, cache == nullptr) or from an external KV cache that already holds `past` rows.
// nb > 1 (no cache): x holds nb samples of n / nb rows each; sample b attends to its own rows, cross_kv rows b*Tk .., the
// key-length arrays are indexed by sample, and the GEMMs are routed by one sample's rows (linear's `samples`).
void dec_layer(ss_engine* h, const DecLayerW& L, float* x, int n, int dim, int ffn, int heads, bool causal, const int* self_kv_len_dev, float* cache_k, float* cache_v, int past, const float* cross_kv, int Tk,
               const int* cross_len_dev, DecScratch& s, cudaStream_t st, int group_R = 0, const int* group_len_dev = nullptr, int nb = 1) {
  const float scale = 0.125f;  // head_dim ** -0.5, head_dim = 64
  const int rows = n / nb;       // per sample
  if (group_R > 1 && !cache_k && causal && rows % group_R == 0) {
    // rows come in groups of group_R identical consecutive rows (unit decoder layer 1): project the n / group_R distinct
    // rows only and collapse the causal softmax over the copies analytically (grouped_causal_attn_kernel)
    const int S = n / group_R;
    ln_linear(h, x, dim * group_R, S, L.self_ln, L.qkv, ep_out(s.qkv, 3 * dim), s.y, st, nb);
    grouped_causal_attention(s.qkv, 3 * dim, s.qkv + dim, 3 * dim, s.qkv + 2 * dim, 3 * dim, s.attn, dim, S / nb, group_R, heads, scale,
                             group_len_dev, nb, st);
  } else if (cache_k) {
    ln_qkv_routed(h, x, dim, n, L.self_ln, L.qkv, dim, s.q, dim, cache_k + (size_t)past * dim, dim, cache_v + (size_t)past * dim, dim, s.y, st, nb);
    mha_attention(s.q, dim, cache_k, dim, cache_v, dim, s.attn, dim, 1, n, past + n, heads, scale, 1, past, self_kv_len_dev, st);
  } else {
    ln_linear(h, x, dim, n, L.self_ln, L.qkv, ep_out(s.qkv, 3 * dim), s.y, st, nb);
    mha_attention(s.qkv, 3 * dim, s.qkv + dim, 3 * dim, s.qkv + 2 * dim, 3 * dim, s.attn, dim, nb, rows, rows, heads, scale,
                  causal ? 1 : 0, 0, self_kv_len_dev, st);
  }
  linear(h, s.attn, dim, n, L.out, ep_residual(x, dim), st, nb);
  if (L.has_cross) {
    ln_linear(h, x, dim, n, L.cross_ln, L.cq, ep_out(s.q, dim), s.y, st, nb);
    mha_attention(s.q, dim, cross_kv, 2 * dim, cross_kv + dim, 2 * dim, s.attn, dim, nb, rows, Tk, heads, scale, 0, 0, cross_len_dev, st);
    linear(h, s.attn, dim, n, L.cout, ep_residual(x, dim), st, nb);
  }
  ln_linear(h, x, dim, n, L.final_ln, L.fc1, ep_out(s.hid, ffn, ACT_RELU), s.y, st, nb);
  linear(h, s.hid, ffn, n, L.fc2, ep_residual(x, dim), st, nb);
}

// keep_rows > 0: rows [0, keep_rows) of every layer survive a reallocation (incremental-state decoding keeps cross K / V across calls)
int ensure_mt_cross(ss_engine* h, int T, int keep_rows = 0) {
  if (T <= h->mt_cross_cap) return SS_OK;
  if (keep_rows < h->mt_inc_cross_rows) h->mt_inc_overwritten = true;  // (as mt_begin: the rows of the incremental state are lost)
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
    dec_layer(h, h->mt[l], x, n, dim, c.mt_ffn, c.mt_heads, true, self_kv_len_dev, ck, cv, past, cross, T, nullptr, s, st);
  }
  layer_norm(x, dim, feats, dim, h->mt_ln.g, h->mt_ln.b, n, dim, st);
}

// cross-attention K | V of encoder rows [from, T) of enc into rows [from, T) of a cache whose layers are layer_rows rows apart: one
// linear per MT layer over the T - from rows (the GEMM routing depends on that M)
void project_cross(ss_engine* h, const std::vector<DecLayerW>& layers, int in_dim, const float* enc, int from, int T, float* cache, size_t layer_rows,
                   cudaStream_t st) {
  if (T <= from) return;
  for (size_t l = 0; l < layers.size(); ++l)
    linear(h, enc + (size_t)from * in_dim, in_dim, T - from, layers[l].ckv, ep_out(cache + (l * layer_rows + from) * 2 * layers[l].cq.N, 2 * layers[l].cq.N), st);
}
void mt_project_cross(ss_engine* h, const float* enc, int from, int T, float* cache, size_t layer_rows, cudaStream_t st) {
  project_cross(h, h->mt, h->cfg.enc_dim, enc, from, T, cache, layer_rows, st);
}

// cross-attention K | V of the encoder rows.  Rows the caller declared final (ss_mt_stable_rows) at the previous call were
// projected then and are not touched again; everything above is (re)computed.  The search that follows writes the self-attention
// cache from entry 0: both are the buffers of the handle's incremental state, which is then no longer the one its calls left.
void mt_begin(ss_engine* h, const float* enc_dev, int T, cudaStream_t st) {
  if (h->mt_inc_self_len > 0 || h->mt_inc_cross_rows > 0) h->mt_inc_overwritten = true;
  int from = (h->mt_cross_enc == enc_dev) ? std::min(h->mt_cross_final, T) : 0;
  if (from < 0) from = 0;
  mt_project_cross(h, enc_dev, from, T, h->mt_cross_kv, h->mt_cross_cap, st);
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

// parameters of the persistent MT kernels over the handle's single-stream buffers (mt_begin's caches, mt_tok_dev)
MtDecodeParams mt_decode_params(ss_engine* h, const DecScratch& s, float* x, float* logits, float* feats, int kv_off) {
  const ss_config& c = h->cfg;
  MtDecodeParams P;
  P.n_layers = c.mt_layers; P.heads = c.mt_heads; P.vocab = c.tgt_vocab; P.pad = c.pad; P.eos = c.eos;
  P.max_pos = c.max_mt_positions; P.cross_cap = h->mt_cross_cap; P.kv_off = kv_off;
  P.emb = h->mt_emb; P.pos = h->mt_pos; P.out_g = h->mt_ln.g; P.out_b = h->mt_ln.b;
  P.self_k = h->mt_self_k; P.self_v = h->mt_self_v; P.cross_kv = h->mt_cross_kv;
  P.tok = h->mt_tok_dev; P.feats = feats; P.x = x; P.q = s.q; P.attn = s.attn; P.hid = s.hid; P.logits = logits;
  P.part = h->mt_part; P.delta = h->mt_part + (size_t)8 * c.mt_dim;
  if (h->persistent_profile) P.ts = h->persist_ts;
  return P;
}

// the single-token MT kernel runs a search over Tk cross rows on this handle (the batched kernel reproduces its rows: it runs there too)
bool mt_single_token_runs(const ss_engine* h, int Tk) {
  const ss_config& c = h->cfg;
  return h->persistent_mt && mt_decode_persistent_supported(c.mt_dim, c.mt_ffn, c.mt_heads, c.tgt_vocab, c.max_mt_positions, Tk);
}

// caller tokens index the embedding table: every one of tok[0 .. n) must be in [0, tgt_vocab)
bool mt_tokens_in_vocab(const ss_engine* h, const int64_t* tok, int n) {
  for (int i = 0; i < n; ++i)
    if (tok[i] < 0 || tok[i] >= h->cfg.tgt_vocab) return false;
  return true;
}

// max_len of a greedy search over a forced prefix of `start` tokens: max_len_b (capped by the positions) for max_new_tokens == -1,
// else start + max_new_tokens.  The hypothesis must fit max_out tokens and, with feats_ld > 0, max_len + 1 feature rows.
int mt_search_len(ss_engine* h, int start, int max_new_tokens, int max_len_b, int max_out, int feats_ld, int* max_len) {
  const int P = h->cfg.max_mt_positions;
  const int ml = (max_new_tokens == -1) ? std::min(max_len_b, P - 1) : start + max_new_tokens;
  if (ml < 1) return h->fail(SS_ERR_INVALID, "min_len cannot be larger than max_len");
  if (start > ml) return h->fail(SS_ERR_INVALID, "prefix longer than max_len");
  if (ml + 2 > P || ml > max_out || (feats_ld > 0 && ml + 1 > feats_ld)) return h->fail(SS_ERR_CAPACITY, "MT hypothesis longer than capacity");
  *max_len = ml;
  return SS_OK;
}

// max_len and kv_off of an incremental search (ss_mt_greedy_incremental, or pool slot `slot` >= 0) whose state holds self_len
// self-attention entries.  The slot of the token at position s is s + kv_off: the first call starts with an empty cache (kv_off = 0),
// every later call re-feeds the last prefix token on top of the entry the previous call's final step left (kv_off grows by one per
// call).  kernel_runs: mt_single_token_runs over the state's cross rows.
int mt_incremental_len(ss_engine* h, int slot, int start, int max_new_tokens, int max_len_b, int self_len, int max_out, bool kernel_runs,
                       int* max_len, int* kv_off) {
  const int P = h->cfg.max_mt_positions;
  const int ml = (max_new_tokens == -1) ? max_len_b : start + max_new_tokens;
  if (ml < 1) return h->fail(SS_ERR_INVALID, "min_len cannot be larger than max_len");
  if (start > ml) return h->fail(SS_ERR_INVALID, "prefix longer than max_len");
  if (slot < 0 && h->mt_inc_overwritten)
    return h->fail(SS_ERR_STATE, "ss_mt_greedy or ss_mt_features ran on this handle after the last incremental call and overwrote the incremental "
                                 "MT state (they share its caches): call ss_mt_incremental_reset before the next ss_mt_greedy_incremental");
  const int off = self_len - start;
  if (off < 0)
    return h->fail(SS_ERR_STATE, slot < 0 ? "incremental MT state is shorter than the prefix (reset missing, or a prefix that this state did not produce)"
                                          : "the slot's incremental MT state is shorter than the prefix (a prefix that this state did not produce)");
  if (ml + off + 2 > P) {
    const std::string need = "MT hypothesis longer than capacity: the incremental search needs " + std::to_string(ml + off + 2) +
                             " self-attention entries (max_len " + std::to_string(ml) + " + " + std::to_string(off) +
                             " kept from earlier calls + 2), max_mt_positions = " + std::to_string(P);
    return h->fail(SS_ERR_CAPACITY, slot < 0 ? need : "slot " + std::to_string(slot) + ": " + need);
  }
  if (ml > max_out) return h->fail(SS_ERR_CAPACITY, "MT hypothesis longer than capacity");
  if (!kernel_runs) return h->fail(SS_ERR_STATE, "incremental MT decoding runs on the persistent MT kernel, which is off or does not support this shape");
  *max_len = ml;
  *kv_off = off;
  return SS_OK;
}

// the token buffer of a single-stream search, [eos, prefix...] (eos is the decoder's bos), and the prefix as the first tokens of the
// hypothesis
void mt_put_prefix(ss_engine* h, cudaStream_t st, const int64_t* prefix_host, int start, int64_t* tokens_out_host) {
  std::vector<int64_t> toks(start + 1);
  toks[0] = h->cfg.eos;
  for (int i = 0; i < start; ++i) toks[i + 1] = prefix_host[i];
  cudaMemcpyAsync(h->mt_tok_dev, toks.data(), toks.size() * sizeof(int64_t), cudaMemcpyHostToDevice, st);
  cudaStreamSynchronize(st);  // (host vector)
  for (int i = 0; i < start; ++i) tokens_out_host[i] = prefix_host[i];
}

// Burst loop of the single-token kernel.  P holds the search's state (self_k / self_v / cross_kv, kv_off) and P.tok the tokens of
// positions <= *step; positions *step .. max_len run over Tk cross rows.  Tokens of positions *first + 1 .. *step were enqueued by the
// caller and not read yet: they are read back with the first launch's, which runs `burst` minus those steps (every launch and its
// read-back covers `burst` steps).  The kernel stops by itself at eos and at the forced eos of position max_len.  New tokens up to eos
// go to tokens_out_host[*n_tok ...]; *self_len (optional) follows the entries the self-attention cache holds.  Returns SS_OK once the
// search ended, an error code (reported), or -1 when a launch was refused: *first / *step then give the unread tokens and the position
// of the refused launch, and nothing from it on was enqueued.
int mt_single_token_bursts(ss_engine* h, cudaStream_t st, const MtDecodeParams& P, int* first, int* step, int max_len, int Tk, int burst,
                           int64_t* tokens_out_host, int* n_tok, int* self_len, const char* where) {
  bool done = false;
  while (!done) {
    const int f = *first, s = *step;
    const int cnt = std::min(max_len - s + 1, burst - (s - f));
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    const bool timed = h->persistent_time && h->mt_time_events.size() < 4096 && cudaEventCreate(&ev0) == cudaSuccess && cudaEventCreate(&ev1) == cudaSuccess;
    if (timed) cudaEventRecord(ev0, st);
    const int rc_launch = mt_decode_persistent(P, h->mt_persist_layers, s, cnt, max_len, Tk, h->persist_bar, &h->persist_bar_target, st);
    if (timed) {
      cudaEventRecord(ev1, st);
      h->mt_time_events.push_back({ev0, ev1, -1.0});  // steps executed: filled in below once the tokens are read
    }
    if (rc_launch != 0) {
      cudaGetLastError();
      return -1;
    }
    done = s + cnt > max_len;      // eos forced at max_len (sequence_generator.py:362-364): that step writes no token
    int last = s + cnt - 1;        // the last position fed
    const int produced = std::min(s + cnt, max_len) - f;
    int steps_run = produced;
    // an incremental search also waits for a launch that only ran the forced-eos step: a barrier timeout there is reported by the
    // call that left the state's last entry
    if (produced > 0 || self_len) {
      const int rc = sync_burst(h, st, h->mt_next_pinned, P.tok + f + 1, produced, produced, 1, where);
      if (rc) return rc;
      for (int i = 0; i < produced; ++i) {
        const int64_t next = h->mt_next_pinned[i];
        if (next == h->cfg.eos) {
          done = true;
          steps_run = i + 1;  // (the kernel stops after the step that produced eos)
          last = f + i;
          break;
        }
        tokens_out_host[(*n_tok)++] = next;
      }
    }
    if (timed && steps_run > 0) h->mt_time_events.back().bytes = (double)steps_run;  // (mt_time counts launches that produced a token)
    if (self_len) *self_len = last + P.kv_off + 1;
    *first = *step = s + cnt;
  }
  return SS_OK;
}

// Burst loop of the batched kernel: steps 0 .. steps - 1 of the P.rows rows, 16 per launch and host read-back; row b's tokens up to its
// eos are appended at tokens_out_host[b * max_out + n_out_host[b]].  Returns SS_OK, an error code (reported), or -1 when the first
// launch was refused (nothing written to the outputs yet: the caller decodes per sample).
int mt_batch_bursts(ss_engine* h, cudaStream_t st, const MtBatchParams& P, int steps, int64_t* tokens_out_host, int max_out, int32_t* n_out_host,
                    const char* where) {
  std::vector<char> done(P.rows, 0);
  int active = P.rows;
  constexpr int kBurst = 16;  // the rows of h->mtb_tok_pinned
  for (int step = 0; step < steps && active > 0; step += kBurst) {
    const int cnt = std::min(kBurst, steps - step);
    if (mt_decode_batch(P, h->mt_persist_layers, step, cnt, h->persist_bar, &h->persist_bar_target, st) != 0) {
      cudaGetLastError();
      if (step == 0) return -1;
      return h->fail(SS_ERR_CUDA, "cooperative launch of the batched MT kernel was refused");
    }
    const int rc = sync_burst(h, st, h->mtb_tok_pinned, P.tok + step + 1, cnt, P.tok_ld, P.rows, where);
    if (rc) return rc;
    for (int b = 0; b < P.rows; ++b) {
      for (int i = 0; i < cnt && !done[b]; ++i) {
        const int64_t next = h->mtb_tok_pinned[(size_t)b * cnt + i];
        if (next == P.eos) {
          done[b] = 1;
          --active;
        } else {
          tokens_out_host[(size_t)b * max_out + n_out_host[b]++] = next;
        }
      }
    }
  }
  return SS_OK;
}

// device buffers of the batched searches, grown on demand: self K / V for tok_ld positions (second_self_kv: a second such buffer,
// the beam search's reorder target), cross K / V for Tmax rows per sample
int ensure_mt_batch(ss_engine* h, int tok_ld, int Tmax, bool second_self_kv = false) {
  const ss_config& c = h->cfg;
  const size_t R = MT_BATCH_MAX_ROWS;
  if (tok_ld > h->mtb_tok_ld || Tmax > h->mtb_cross_cap) cudaDeviceSynchronize();  // earlier launches may still read the old buffers
  const size_t NL = std::max(c.mt_layers, c.unit_layers);  // (the unit search runs on these buffers too)
  if (tok_ld > h->mtb_tok_ld) {
    if (h->mtb_self_kv) cudaFree(h->mtb_self_kv);
    if (h->mtb_self_kv2) cudaFree(h->mtb_self_kv2);
    h->mtb_self_kv = h->mtb_self_kv2 = nullptr;
    h->mtb_tok_ld = 0;
    if (cudaMalloc((void**)&h->mtb_self_kv, (size_t)2 * NL * R * tok_ld * c.mt_dim * sizeof(float)) != cudaSuccess) {
      h->mtb_self_kv = nullptr;
      return h->fail(SS_ERR_CUDA, "cudaMalloc(batched mt self kv) failed");
    }
    h->mtb_tok_ld = tok_ld;
  }
  if (second_self_kv && !h->mtb_self_kv2 &&
      cudaMalloc((void**)&h->mtb_self_kv2, (size_t)2 * NL * R * h->mtb_tok_ld * c.mt_dim * sizeof(float)) != cudaSuccess) {
    h->mtb_self_kv2 = nullptr;
    return h->fail(SS_ERR_CUDA, "cudaMalloc(batched mt self kv, second buffer) failed");
  }
  if (Tmax > h->mtb_cross_cap) {
    const int cap = std::max(Tmax + Tmax / 2, 512);
    if (h->mtb_cross_kv) cudaFree(h->mtb_cross_kv);
    h->mtb_cross_kv = nullptr;
    h->mtb_cross_cap = 0;
    if (cudaMalloc((void**)&h->mtb_cross_kv, (size_t)NL * R * cap * 2 * c.mt_dim * sizeof(float)) != cudaSuccess) {
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
  // cross K / V: the same projection as mt_begin with the sample's own row count (the GEMM routing depends on M)
  for (int b = 0; b < Bg; ++b)
    mt_project_cross(h, enc_dev + (size_t)(g0 + b) * T_stride * c.enc_dim, 0, T_host[g0 + b], h->mtb_cross_kv + (size_t)b * h->mtb_cross_cap * 2 * dim,
                     R * h->mtb_cross_cap, st);
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
  // step max_len is the forced eos: no work
  return mt_batch_bursts(h, st, P, max_len, tokens_out_host + (size_t)g0 * max_out, max_out, n_out_host + g0, "ss_mt_greedy_batch");
}

// The decoder a beam search runs on the batched decoder kernel: the MT decoder (ss_mt_beam_batch) or UnitY's unit decoder at beam 1
// (ss_unit_search_batch).  Both are 512 wide with 2048-wide FFNs; cross-attention reads rows of in_dim floats projected by the layers.
struct SearchDecoder {
  int n_layers, ffn, vocab, in_dim;
  const float *emb, *pos, *out_g, *out_b;
  const MtLayerP* layers_dev;
  const std::vector<DecLayerW>* layers;
  const char* where;
};

SearchDecoder mt_search_decoder(const ss_engine* h) {
  const ss_config& c = h->cfg;
  return {c.mt_layers, c.mt_ffn, c.tgt_vocab, c.enc_dim, h->mt_emb, h->mt_pos, h->mt_ln.g, h->mt_ln.b, h->mt_persist_layers, &h->mt, "ss_mt_beam_batch"};
}

// Beam search of samples g0 .. g0 + Sg - 1 (Sg * beam <= MT_BATCH_MAX_ROWS rows) on mt_decode_batch_kernel's beam instantiation.
// The steps run in bursts of 16 per launch; after each burst the host reads one done flag per sample and stops once all are set.
// The search ends with K finalized hypotheses per sample, read once at the end and sorted by score (stable: on equal scores the
// earlier finalized first).  Returns SS_OK or an error code (reported).
int mt_beam_group(ss_engine* h, cudaStream_t st, const SearchDecoder& D, const float* enc_dev, int g0, int Sg, int beam, int T_stride, const int32_t* T_host,
                  int max_len, float len_penalty, int64_t* tokens_out_host, int max_out, int32_t* n_out_host, float* scores_out_host,
                  float* pos_scores_out_host) {
  const ss_config& c = h->cfg;
  const int dim = c.mt_dim, K = beam, rows = Sg * K, nh = Sg * K;
  const size_t R = MT_BATCH_MAX_ROWS;
  int Tmax = 0;
  for (int b = 0; b < Sg; ++b) Tmax = std::max(Tmax, (int)T_host[g0 + b]);
  int rc = ensure_mt_batch(h, max_len + 2, Tmax, K > 1);  // (beam 1 keeps its self-attention cache in place)
  if (rc) return rc;
  const int ld = h->mtb_tok_ld;
  // cross K / V once per sample (its K beams read the same block), as ss_mt_greedy_batch projects it
  for (int b = 0; b < Sg; ++b)
    project_cross(h, *D.layers, D.in_dim, enc_dev + (size_t)(g0 + b) * T_stride * D.in_dim, 0, T_host[g0 + b],
                  h->mtb_cross_kv + (size_t)b * h->mtb_cross_cap * 2 * dim, R * h->mtb_cross_cap, st);
  const size_t floats = (size_t)rows * (dim * 11 + D.ffn + D.vocab + 2 * ld + 2 * K) + (size_t)nh * (ld + 1);
  const size_t i64s = (size_t)2 * rows * ld + (size_t)nh * ld;
  const size_t ints = (size_t)rows * (4 + 2 * K) + (size_t)Sg * 2 + nh;
  if (!ws_begin(h, floats * sizeof(float) + i64s * sizeof(int64_t) + ints * sizeof(int) + 32 * 256)) return h->fail(SS_ERR_CUDA, "workspace allocation failed");
  MtBatchParams P;
  P.n_layers = D.n_layers; P.vocab = D.vocab; P.pad = c.pad; P.eos = c.eos;
  P.rows = rows; P.tok_ld = ld; P.cross_cap = h->mtb_cross_cap;
  P.emb = D.emb; P.pos = D.pos; P.out_g = D.out_g; P.out_b = D.out_b;
  P.self_k = h->mtb_self_kv; P.self_v = h->mtb_self_kv + (size_t)D.n_layers * R * ld * dim; P.cross_kv = h->mtb_cross_kv;
  P.q = h->ws.f32((size_t)rows * dim); P.part = h->ws.f32((size_t)rows * 8 * dim); P.delta = h->ws.f32((size_t)rows * dim);
  P.hid = h->ws.f32((size_t)rows * D.ffn); P.logits = h->ws.f32((size_t)rows * D.vocab);
  P.tok = (int64_t*)h->ws.raw((size_t)rows * ld * sizeof(int64_t));
  MtBeamParams Bm;
  Bm.beam = K; Bm.max_len = max_len; Bm.len_penalty = len_penalty;
  Bm.tok2 = (int64_t*)h->ws.raw((size_t)rows * ld * sizeof(int64_t));
  if (K > 1) Bm.self_k2 = h->mtb_self_kv2, Bm.self_v2 = h->mtb_self_kv2 + (size_t)D.n_layers * R * ld * dim;
  Bm.cum = h->ws.f32((size_t)2 * rows * ld); Bm.cand = h->ws.f32((size_t)rows * 2 * K);
  Bm.cand_tok = (int*)h->ws.raw((size_t)rows * 2 * K * sizeof(int)); Bm.parent = (int*)h->ws.raw((size_t)rows * sizeof(int));
  Bm.hyp_tok = (int64_t*)h->ws.raw((size_t)nh * ld * sizeof(int64_t)); Bm.hyp_pos = h->ws.f32((size_t)nh * ld);
  Bm.hyp_score = h->ws.f32(nh); Bm.hyp_len = (int*)h->ws.raw((size_t)nh * sizeof(int));
  int* init = (int*)h->ws.raw(((size_t)2 * rows + 2 * Sg) * sizeof(int));  // [fin | cross_len | n_fin | done]
  if (!P.q || !P.part || !P.delta || !P.hid || !P.logits || !P.tok || !Bm.tok2 || !Bm.cum || !Bm.cand || !Bm.cand_tok || !Bm.parent ||
      !Bm.hyp_tok || !Bm.hyp_pos || !Bm.hyp_score || !Bm.hyp_len || !init)
    return h->fail(SS_ERR_CUDA, "workspace too small");
  P.fin = init;
  P.cross_len = init + rows;
  Bm.n_fin = init + 2 * rows;
  Bm.done = Bm.n_fin + Sg;
  std::vector<int64_t> tok0((size_t)rows * ld, c.eos);  // column 0 = eos (the decoder's bos)
  std::vector<int> init0(2 * rows + 2 * Sg, 0);
  for (int r = 0; r < rows; ++r) {
    init0[r] = r % K != 0;  // step 0 runs beam 0 only (lprobs[:, ::beam_size]); its selection starts every beam
    init0[rows + r] = T_host[g0 + r / K];
  }
  // (no synchronisation here: tok0 / init0 outlive every burst of this function, whose first read-back synchronises the stream)
  cudaMemcpyAsync(P.tok, tok0.data(), tok0.size() * sizeof(int64_t), cudaMemcpyHostToDevice, st);
  cudaMemcpyAsync(init, init0.data(), init0.size() * sizeof(int), cudaMemcpyHostToDevice, st);
  int* done_pinned = reinterpret_cast<int*>(h->mtb_tok_pinned);  // (MT_BATCH_MAX_ROWS * 16 int64 words)
  constexpr int kBurst = 16;
  for (int step = 0; step <= max_len; step += kBurst) {  // step max_len forces eos: it still scores and finalizes every beam
    const int cnt = std::min(kBurst, max_len + 1 - step);
    if (mt_decode_batch(P, D.layers_dev, step, cnt, h->persist_bar, &h->persist_bar_target, st, &Bm) != 0) {
      cudaGetLastError();
      return h->fail(SS_ERR_CUDA, std::string(D.where) + ": the cooperative launch of the batched decoder kernel's beam search was refused");
    }
    cudaMemcpyAsync(done_pinned, Bm.done, Sg * sizeof(int), cudaMemcpyDeviceToHost, st);
    rc = sync_burst(h, st, nullptr, nullptr, 0, 0, 0, D.where);
    if (rc) return rc;
    if (std::all_of(done_pinned, done_pinned + Sg, [](int d) { return d != 0; })) break;
  }
  std::vector<int64_t> toks((size_t)nh * ld);
  std::vector<float> pos((size_t)nh * ld), score(nh);
  std::vector<int> len(nh), nfin(Sg);
  cudaMemcpyAsync(toks.data(), Bm.hyp_tok, toks.size() * sizeof(int64_t), cudaMemcpyDeviceToHost, st);
  cudaMemcpyAsync(pos.data(), Bm.hyp_pos, pos.size() * sizeof(float), cudaMemcpyDeviceToHost, st);
  cudaMemcpyAsync(score.data(), Bm.hyp_score, nh * sizeof(float), cudaMemcpyDeviceToHost, st);
  cudaMemcpyAsync(len.data(), Bm.hyp_len, nh * sizeof(int), cudaMemcpyDeviceToHost, st);
  cudaMemcpyAsync(nfin.data(), Bm.n_fin, Sg * sizeof(int), cudaMemcpyDeviceToHost, st);
  if (cudaStreamSynchronize(st) != cudaSuccess) return h->fail(SS_ERR_CUDA, std::string(D.where) + ": " + cudaGetErrorString(cudaGetLastError()));
  for (int j = 0; j < Sg; ++j) {
    if (nfin[j] != K) return h->fail(SS_ERR_CUDA, std::string(D.where) + ": a sample ended with fewer than beam finalized hypotheses");
    std::vector<int> order(K);
    for (int i = 0; i < K; ++i) order[i] = i;
    std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return score[(size_t)j * K + a] > score[(size_t)j * K + b]; });
    for (int i = 0; i < K; ++i) {
      const size_t src = (size_t)j * K + order[i], dst = (size_t)(g0 + j) * K + i;
      const int n = len[src];  // eos included
      std::copy(toks.begin() + src * ld, toks.begin() + src * ld + n - 1, tokens_out_host + dst * max_out);
      std::copy(pos.begin() + src * ld, pos.begin() + src * ld + n, pos_scores_out_host + dst * (max_out + 1));
      n_out_host[dst] = n - 1;
      scores_out_host[dst] = score[src];
    }
  }
  return SS_OK;
}

// Streams i0 .. i0 + n - 1 of a batched search one by one through ss_mt_greedy: stream i decodes encoder block enc_block[i] (nullptr:
// block i) of enc, enc_ld floats apart, over its T[i] rows, after its n_prefix[i] tokens pfx[i] (nullptr: none) with max_new_tokens[i]
// (nullptr: -1); its features (feats_out_dev non-null) go to rows i * feats_ld.  ss_mt_greedy uses the single-stream MT buffers, so
// their cross K / V cache is marked invalid afterwards (a streaming call on this handle then projects every row again) and a pending
// stable-rows hint is kept.
int mt_greedy_per_stream(ss_engine* h, void* stream, int i0, int n, const float* enc, size_t enc_ld, const int32_t* enc_block, const int32_t* T,
                         const int64_t* const* pfx, const int32_t* n_prefix, const int32_t* max_new_tokens, int max_len_b, int64_t* tokens_out_host,
                         int max_out, int32_t* n_out_host, float* feats_out_dev, int feats_ld) {
  const int hint = h->mt_stable_hint;
  h->mt_stable_hint = 0;
  int rc = SS_OK;
  for (int i = i0; i < i0 + n && rc == SS_OK; ++i) {
    int n_tok = 0;
    rc = ss_mt_greedy(h, stream, enc + (enc_block ? enc_block[i] : i) * enc_ld, T[i], pfx ? pfx[i] : nullptr, n_prefix ? n_prefix[i] : 0,
                      max_new_tokens ? max_new_tokens[i] : -1, max_len_b, tokens_out_host + (size_t)i * max_out, max_out, &n_tok,
                      feats_out_dev ? feats_out_dev + (size_t)i * feats_ld * h->cfg.mt_dim : nullptr);
    n_out_host[i] = n_tok;
  }
  h->mt_cross_enc = nullptr;
  h->mt_cross_final = 0;
  h->mt_stable_hint = hint;
  return rc;
}

// T2U encoder -> unit decoder -> unit CTC of B samples of Slen positions (mt_feats [B][Slen][dim]); sample b adds positional row
// pos_rows[b] (N1), has S_host[b] positions (nullptr: every sample has Slen; positions >= S_b are neither keys nor decoded into
// units) and n_pad_tail_host[b] trailing pad positions among them.  Its arg-max goes to argmax_dev + b * Slen * R, its units
// to units_dev + b * seg_stride and its count to count_dev + 2 * b * seg_stride (int64 words, as ctc_collapse_segments).  Key
// lengths are uploaded (one synchronisation) only when some sample has a pad tail or fewer than Slen positions; otherwise every
// attention runs at full length.
// t2u_out_dev / logits_dev (optional, B = 1): the T2U encoder output and the unit logits are written there.
// lprob_dev (optional, [B][Slen * R]): each row's arg-max log-probability (argmax_lprob_rows instead of argmax_rows).
int t2u_unit_decode(ss_engine* h, cudaStream_t st, const float* mt_feats_dev, int B, int Slen, const int32_t* S_host, const int32_t* n_pad_tail_host,
                    const float* pos_rows_dev, int mask_eos, int64_t* argmax_dev, int64_t* units_dev, int32_t* count_dev, int64_t seg_stride,
                    float* t2u_out_dev, float* logits_dev, float* lprob_dev, const char* where) {
  const ss_config& c = h->cfg;
  const int dim = c.unit_dim, R = c.ctc_upsample_rate, L = Slen * R;
  std::vector<int> lens(3 * (size_t)B);  // [valid T2U positions B | valid upsampled rows B | decoded upsampled rows B]
  bool padded = false, ragged = false;
  for (int b = 0; b < B; ++b) {
    const int Sb = S_host ? S_host[b] : Slen, np = n_pad_tail_host[b];
    if (Sb < 1 || Sb > Slen) return h->fail(SS_ERR_INVALID, std::string(where) + ": sample length outside [1, S_stride]");
    if (np < 0 || np >= Sb) return h->fail(SS_ERR_INVALID, std::string(where) + ": n_pad_tail outside [0, S)");
    lens[b] = Sb - np;
    lens[B + b] = (Sb - np) * R;
    lens[2 * B + b] = Sb * R;
    padded |= np > 0 || Sb < Slen;
    ragged |= Sb < Slen;
  }
  const int G = std::max(1, SS_UNIT_BATCH_ROWS / L);
  const int Bg_max = std::min(G, B);
  const size_t n_max = (size_t)Bg_max * Slen, rows_max = (size_t)Bg_max * L;
  const size_t need = (rows_max * (dim * 8 + c.unit_ffn + c.unit_vocab) + n_max * (dim * 11 + c.unit_ffn)) * sizeof(float) + lens.size() * sizeof(int) +
                      16 * 256;
  if (!ws_begin(h, need)) return h->fail(SS_ERR_CUDA, "workspace allocation failed");
  int* lens_dev = padded ? (int*)h->ws.raw(lens.size() * sizeof(int)) : nullptr;
  DecScratch s1 = dec_scratch(h, (int)n_max, dim, c.unit_ffn);
  float* x = h->ws.f32(n_max * dim);
  float* t2u = t2u_out_dev ? t2u_out_dev : h->ws.f32(n_max * dim);
  float* ckv = h->ws.f32(n_max * 2 * dim);
  DecScratch s2 = dec_scratch(h, (int)rows_max, dim, c.unit_ffn);
  float* xu = h->ws.f32(rows_max * dim);
  float* logits = logits_dev ? logits_dev : h->ws.f32(rows_max * c.unit_vocab);
  if ((padded && !lens_dev) || !s1.qkv || !x || !t2u || !ckv || !s2.qkv || !xu || !logits) return h->fail(SS_ERR_CUDA, "workspace too small");
  if (padded) {  // the encoder_padding_mask of each sample's pad tail
    cudaMemcpyAsync(lens_dev, lens.data(), lens.size() * sizeof(int), cudaMemcpyHostToDevice, st);
    if (cudaStreamSynchronize(st) != cudaSuccess)  // (host vector)
      return h->fail(SS_ERR_CUDA, std::string(where) + ": " + cudaGetErrorString(cudaGetLastError()));
  }
  Linear outp;
  outp.w = h->unit_emb; outp.b = nullptr; outp.N = c.unit_vocab; outp.K = dim;
  for (int g0 = 0; g0 < B; g0 += G) {
    const int Bg = std::min(G, B - g0);
    const int n = Bg * Slen, rows = Bg * L;
    const int* s_len = padded ? lens_dev + g0 : nullptr;       // T2U key lengths, unit cross-attention key lengths, valid groups of layer 1
    const int* up_len = padded ? lens_dev + B + g0 : nullptr;  // unit self-attention key lengths
    const int* dec_len = ragged ? lens_dev + 2 * B + g0 : nullptr;  // upsampled rows collapsed into units
    // ---- T1: UniTransformerEncoderNoEmb.forward on the group's samples
    copy_f32(mt_feats_dev + (size_t)g0 * Slen * dim, x, (int64_t)n * dim, st);
    for (int l = 0; l < c.t2u_layers; ++l)
      dec_layer(h, h->t2u[l], x, n, dim, c.unit_ffn, c.unit_heads, c.uni_encoder != 0, s_len, nullptr, nullptr, 0, nullptr, 0, nullptr, s1, st, 0,
                nullptr, Bg);
    layer_norm(x, dim, t2u, dim, h->t2u_ln.g, h->t2u_ln.b, n, dim, st);
    // ---- U1: CTCTransformerUnitDecoder: x R upsample + (quirky) positional row of each sample (N1), 2 layers, out-proj
    repeat_rows_add(t2u, Slen, R, dim, pos_rows_dev + (size_t)g0 * dim, xu, Bg, st);
    for (int l = 0; l < c.unit_layers; ++l) {
      linear(h, t2u, dim, n, h->unit[l].ckv, ep_out(ckv, 2 * dim), st, Bg);
      // layer 0 sees R identical copies of every T2U state (same positional row for every step, N1): grouped self-attention
      const int gR = (l == 0 && h->unit_grouped) ? R : 0;
      dec_layer(h, h->unit[l], xu, rows, dim, c.unit_ffn, c.unit_heads, true, up_len, nullptr, nullptr, 0, ckv, Slen, s_len, s2, st, gR, s_len, Bg);
    }
    layer_norm(xu, dim, xu, dim, h->unit_ln.g, h->unit_ln.b, rows, dim, st);
    linear(h, xu, dim, rows, outp, ep_out(logits, c.unit_vocab), st, Bg);
    // ---- U2: never select pad, unk (agent version) [+ eos: offline version], then each sample's collapse
    int64_t* am = argmax_dev + (size_t)g0 * L;
    if (lprob_dev)
      argmax_lprob_rows(logits, c.unit_vocab, rows, c.unit_vocab, h->mask_pad_unk, mask_eos ? 3 : 2, am, lprob_dev + (size_t)g0 * L, st);
    else
      argmax_rows(logits, c.unit_vocab, rows, c.unit_vocab, h->mask_pad_unk, mask_eos ? 3 : 2, am, st);
    ctc_collapse_segments(am, L, 1, Bg, c.unit_vocab - 1, c.pad, units_dev + g0 * seg_stride, nullptr, count_dev + 2 * g0 * seg_stride, seg_stride,
                          st, dec_len);
  }
  return check_launch(h, where);
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
    gemm_conv(a, h->sub_conv[0].w, h->sub_conv[0].N, ep, &h->splitk[0], st);
    ConvA a2;
    a2.x = c1; a2.B = B; a2.L_in = T1; a2.L_rows = T; a2.C_in = c.conv_channels / 2; a2.ldx = c.conv_channels / 2;
    a2.ksize = c.conv_kernel; a2.stride = 2; a2.pad_left = c.conv_kernel / 2; a2.chunk = cc;
    Epilogue ep2 = ep_out(x0, D);
    ep2.bias = h->sub_conv[1].b; ep2.glu = 1; ep2.alpha = sqrtf((float)D);  // x = embed_scale * x (s2t_conformer.py:127)
    gemm_conv(a2, h->sub_conv[1].w, h->sub_conv[1].N, ep2, &h->splitk[0], st);
  }
  linear(h, x0, D, (int)rows, h->enc_linear, ep_out(x, D), st);  // s2t_conformer.py:139
  for (int i = 0; i < c.enc_layers; ++i) {
    const ConformerLayerW& L = h->enc[i];
    // x = x + 0.5 * ffn1(x)
    layer_norm(x, D, y, D, L.ffn1_ln.g, L.ffn1_ln.b, (int)rows, D, st);
    linear(h, y, D, (int)rows, L.ffn1_w1, ep_out(hid, c.enc_ffn, ACT_SILU), st);
    linear(h, hid, c.enc_ffn, (int)rows, L.ffn1_w2, ep_residual(x, D, 0.5f), st);
    // x = x + self_attn(LN(x))
    layer_norm(x, D, y, D, L.attn_ln.g, L.attn_ln.b, (int)rows, D, st);
    linear(h, y, D, (int)rows, L.qkv, ep_out(qkv, 3 * D), st);
    relpos_attention(qkv, 3 * D, qkv + D, 3 * D, qkv + 2 * D, 3 * D, L.pos_proj, h->Tpos, L.pos_u, L.pos_v, att, B, T, 0, T, c.enc_heads, D,
                     h->attn_chunk, len_dev, st);
    linear(h, att, D, (int)rows, L.attn_out, ep_residual(x, D), st);
    // x = x + conv_module(x)
    layer_norm(x, D, y, D, L.conv_ln.g, L.conv_ln.b, (int)rows, D, st);
    {
      Epilogue ep = ep_out(glu, D);
      ep.glu = 1;
      linear(h, y, D, (int)rows, L.pw1, ep, st);
    }
    depthwise_bn_silu(glu, D, L.dw_w, L.bn_scale, L.bn_shift, dw, D, B, T, 0, T, D, c.dw_kernel, cc, st);
    linear(h, dw, D, (int)rows, L.pw2, ep_residual(x, D), st);
    // x = LN(x + 0.5 * ffn2(x))
    layer_norm(x, D, y, D, L.ffn2_ln.g, L.ffn2_ln.b, (int)rows, D, st);
    linear(h, y, D, (int)rows, L.ffn2_w1, ep_out(hid, c.enc_ffn, ACT_SILU), st);
    linear(h, hid, c.enc_ffn, (int)rows, L.ffn2_w2, ep_residual(x, D, 0.5f), st);
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
      gemm_conv(a, h->sub_conv[0].w, h->sub_conv[0].N, ep, &h->splitk[0], st);
      ConvA a2;
      a2.x = c1; a2.B = 1; a2.L_in = T1; a2.L_rows = nA; a2.C_in = c.conv_channels / 2; a2.ldx = c.conv_channels / 2;
      a2.ksize = c.conv_kernel; a2.stride = 2; a2.pad_left = c.conv_kernel / 2; a2.chunk = cc;
      a2.t_offset = a0; a2.x_row0 = t1_lo; a2.x_rows = n1;
      Epilogue ep2 = ep_out(x0, D);
      ep2.bias = h->sub_conv[1].b; ep2.glu = 1; ep2.alpha = sqrtf((float)D);
      gemm_conv(a2, h->sub_conv[1].w, h->sub_conv[1].N, ep2, &h->splitk[0], st);
    }
    linear(h, x0, D, nA, h->enc_linear, ep_out(x, D), st);
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
    if (persistent && h->persistent_encoder_cluster && h->cl_blobs &&
        encoder_layers_cluster_supported(nA, D, c.enc_ffn, c.enc_heads, T, c.dw_kernel)) {
      const float* pos_tabs[16];
      for (int i = 0; i < 16; ++i) pos_tabs[i] = i < c.enc_layers ? h->enc[i].pos_proj : nullptr;
      cluster_done = c.enc_layers <= 16 && encoder_layers_cluster(h->persist_layers, h->cl_blobs, c.enc_layers, x, h->st_k, h->st_v, h->st_glu, nA, a0, T, h->Tpos, h->attn_chunk, cc,
                                            c.dw_kernel, h->persist_bar, &h->persist_bar_target, h->persistent_profile ? h->persist_ts : nullptr, pos_tabs, h->cluster_cooperative, st) == 0;
      if (cluster_done) ++h->cl_steps;
      if (!cluster_done) cudaGetLastError();  // refused launch: the one-CTA-per-SM kernel below takes the step
    }
    if (persistent && !cluster_done)
      persistent = encoder_layers_persistent(h->persist_layers, c.enc_layers, x, hid, qb, att, dw, h->st_k, h->st_v, h->st_glu, nA, a0, T, D,
                                             c.enc_ffn, c.enc_heads, h->Tpos, h->attn_chunk, cc, c.dw_kernel,
                                             h->persistent_profile ? h->persist_ts : nullptr, h->persist_bar, &h->persist_bar_target,
                                             h->persistent_ffn_fused ? h->persist_ffn_scratch : nullptr, st) == 0;
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
      ln_linear(h, x, D, nA, L.ffn1_ln, L.ffn1_w1, ep_out(hid, c.enc_ffn, ACT_SILU), y, st);
      linear(h, hid, c.enc_ffn, nA, L.ffn1_w2, ep_residual(x, D, 0.5f), st);
      // q -> scratch, k / v -> cache rows a0.. (provisional tail rows are overwritten next call)
      ln_qkv_routed(h, x, D, nA, L.attn_ln, L.qkv, D, qb, D, kc + (size_t)a0 * D, D, vc + (size_t)a0 * D, D, y, st);
      relpos_attention(qb, D, kc, D, vc, D, L.pos_proj, h->Tpos, L.pos_u, L.pos_v, att, 1, nA, a0, T, c.enc_heads, D, h->attn_chunk, nullptr, st);
      linear(h, att, D, nA, L.attn_out, ep_residual(x, D), st);
      {
        Epilogue ep = ep_out(gc + (size_t)a0 * D, D);
        ep.glu = 1;
        ln_linear(h, x, D, nA, L.conv_ln, L.pw1, ep, y, st);
      }
      depthwise_bn_silu(gc, D, L.dw_w, L.bn_scale, L.bn_shift, dw, D, 1, T, a0, nA, D, c.dw_kernel, cc, st);
      linear(h, dw, D, nA, L.pw2, ep_residual(x, D), st);
      ln_linear(h, x, D, nA, L.ffn2_ln, L.ffn2_w1, ep_out(hid, c.enc_ffn, ACT_SILU), y, st);
      linear(h, hid, c.enc_ffn, nA, L.ffn2_w2, ep_residual(x, D, 0.5f), st);
      layer_norm(x, D, x, D, L.final_ln.g, L.final_ln.b, nA, D, st);
    }
  }
  h->st_T_final = std::max(h->st_T_final, std::min(T, (F / (4 * G)) * G));
  if (T_final_out) *T_final_out = h->st_T_final;
  return check_launch(h, "ss_encoder_stream_step");
}

int ss_ctc_greedy_rows(ss_engine* h, void* stream, int head, const float* enc_dev, int rows, int row0, int64_t* argmax_dev,
                       int64_t* tokens_dev, int32_t* index_dev, int32_t* count_dev) {
  if (!h || !h->finalized) return h ? h->fail(SS_ERR_STATE, "engine not finalized") : SS_ERR_INVALID;
  if (!h->has_ctc) return refuse_without_ctc(h, "ss_ctc_greedy");
  if (head < 0 || head > 1 || rows <= 0 || row0 < 0 || row0 > rows) return h->fail(SS_ERR_INVALID, "bad ctc head / rows");
  const Linear& l = h->ctc_head[head];
  cudaStream_t st = S(stream);
  const int nr = rows - row0;  // rows below row0 keep the arg-max the caller cached from an earlier call
  if (nr > 0) {
    if (!ws_begin(h, (size_t)nr * l.N * sizeof(float) + 4096)) return h->fail(SS_ERR_CUDA, "workspace allocation failed");
    float* logits = h->ws.f32((size_t)nr * l.N);
    linear(h, enc_dev + (size_t)row0 * h->cfg.enc_dim, h->cfg.enc_dim, nr, l, ep_out(logits, l.N), st);
    argmax_rows(logits, l.N, nr, l.N, h->mask_pad_unk, 2, argmax_dev + row0, st);  // never select pad, unk
  }
  // <s> is the CTC blank (agent/ctc_decoder.py:72-76)
  ctc_collapse_segments(argmax_dev, rows, 1, 1, 0, h->cfg.pad, tokens_dev, index_dev, count_dev, 0, st);
  return check_launch(h, "ss_ctc_greedy");
}

int ss_ctc_greedy_pair(ss_engine* h, void* stream, const float* enc_dev, int rows, int row0, int64_t* argmax0_dev, int64_t* argmax1_dev,
                       int64_t* packed_out_dev) {
  if (!h || !h->finalized) return h ? h->fail(SS_ERR_STATE, "engine not finalized") : SS_ERR_INVALID;
  if (!h->has_ctc) return refuse_without_ctc(h, "ss_ctc_greedy_pair");
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
    linear(h, enc_dev + (size_t)row0 * h->cfg.enc_dim, h->cfg.enc_dim, nr, h->ctc_pair, ep_out(logits, 2 * V), st);
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
  if (!h || !h->finalized) return h ? h->fail(SS_ERR_STATE, "engine not finalized") : SS_ERR_INVALID;
  const ss_config& c = h->cfg;
  if (n <= 0 || n > c.max_mt_positions || T <= 0) return h->fail(SS_ERR_INVALID, "bad MT sequence length");
  if (!mt_tokens_in_vocab(h, tokens_host, n)) return h->fail(SS_ERR_INVALID, "ss_mt_features: token outside the vocabulary");
  cudaStream_t st = S(stream);
  int n_valid = n;  // trailing pads (whole_word path, agent:576-591) are masked as keys
  while (n_valid > 0 && tokens_host[n_valid - 1] == c.pad) --n_valid;
  for (int i = 0; i < n_valid; ++i)
    if (tokens_host[i] == c.pad) return h->fail(SS_ERR_INVALID, "pads are only supported as a tail");
  int rc = ensure_mt_cross(h, T);
  if (rc) return rc;
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
    linear(h, feats_out_dev + (size_t)(n - 1) * dim, dim, 1, out, ep_out(logits_last_dev, c.tgt_vocab), st);
  }
  return check_launch(h, "ss_mt_features");
}

int ss_mt_greedy(ss_engine* h, void* stream, const float* enc_dev, int T, const int64_t* prefix_host, int n_prefix, int max_new_tokens,
                 int max_len_b, int64_t* tokens_out_host, int max_out, int* n_out, float* feats_out_dev) {
  if (!h || !h->finalized) return h ? h->fail(SS_ERR_STATE, "engine not finalized") : SS_ERR_INVALID;
  const ss_config& c = h->cfg;
  cudaStream_t st = S(stream);
  if (T <= 0 || n_prefix < 0 || !n_out) return h->fail(SS_ERR_INVALID, "bad arguments to ss_mt_greedy");
  const int start = n_prefix;
  if (!mt_tokens_in_vocab(h, prefix_host, start)) return h->fail(SS_ERR_INVALID, "ss_mt_greedy: prefix token outside the vocabulary");
  int max_len = 0;
  int rc = mt_search_len(h, start, max_new_tokens, max_len_b, max_out, 0, &max_len);
  if (rc) return rc;
  rc = ensure_mt_cross(h, T);
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
  mt_put_prefix(h, st, prefix_host, start, tokens_out_host);
  mt_begin(h, enc_dev, T, st);
  int fed = 0;  // rows in the KV cache
  int n_tok = start;  // hypothesis length so far (without eos)
  // The arg-max of step s is written straight into the device token buffer at s+1, so consecutive steps need no host
  // round trip.  Steps are enqueued in bursts; the host reads the burst's tokens back once and stops at the first eos
  // (steps enqueued past an eos only produce rows that are never read).
  const int burst = (max_new_tokens >= 0) ? std::max(1, max_new_tokens) : 16;
  bool single = mt_single_token_runs(h, T);
  const MtDecodeParams P = mt_decode_params(h, s, x, logits, feats_out_dev, 0);
  if (single && h->persistent_mt_prefix && start >= 1 && mt_prefix_persistent_supported(dim, c.mt_ffn, c.mt_heads, start, T)) {
    // rows 0 .. start-1 ([eos, p1 .. p_{start-1}]) in one cooperative launch; the single-token kernel continues at position `start`
    if (mt_prefix_persistent(P, h->mt_persist_layers, start, T, h->persist_bar, &h->persist_bar_target, st) == 0)
      fed = start;
    else
      cudaGetLastError();  // refused launch: per-kernel path
  }
  int step = start;
  bool done = false;
  while (!done) {
    int burst_first = step;  // tokens of positions burst_first + 1 .. step are not read yet
    for (; step <= max_len && step - burst_first < burst; ++step) {
      if (single && step == fed) {
        // the rest of the search on the single-token kernel, the rest of this burst in its first launch
        rc = mt_single_token_bursts(h, st, P, &burst_first, &step, max_len, T, burst, tokens_out_host, &n_tok, nullptr, "ss_mt_greedy");
        if (rc != -1) {
          if (rc) return rc;
          *n_out = n_tok;
          return check_launch(h, "ss_mt_greedy");
        }
        single = false;  // refused launch: the per-kernel path below finishes the search from this step
        fed = step;
      }
      // feed tokens[fed .. step]  (first iteration: the whole prefix; afterwards one token)
      mt_forward(h, fed, step + 1 - fed, T, nullptr, feats_out_dev + (size_t)fed * dim, s, x, st);
      fed = step + 1;
      if (step >= max_len) {  // eos is forced here (sequence_generator.py:362-364): no need for the logits
        done = true;
        ++step;
        break;
      }
      linear(h, feats_out_dev + (size_t)step * dim, dim, 1, outp, ep_out(logits, c.tgt_vocab), st);
      // lprobs[pad] = -inf; eos banned while step < min_len (=1)
      if (step < 1)
        argmax_rows(logits, c.tgt_vocab, 1, c.tgt_vocab, h->mask_pad_eos, 2, h->mt_tok_dev + step + 1, st);
      else
        argmax_rows(logits, c.tgt_vocab, 1, c.tgt_vocab, h->mask_pad_unk, 1, h->mt_tok_dev + step + 1, st);
    }
    // tokens produced by this burst live at mt_tok_dev[burst_first+1 .. ]; the forced-eos step produced none
    const int produced = step - burst_first - (done ? 1 : 0);
    if (produced > 0) {
      rc = sync_burst(h, st, h->mt_next_pinned, h->mt_tok_dev + burst_first + 1, produced, produced, 1, "ss_mt_greedy");
      if (rc) return rc;
      for (int i = 0; i < produced; ++i) {
        const int64_t next = h->mt_next_pinned[i];
        if (next == c.eos) {
          done = true;
          break;
        }
        tokens_out_host[n_tok++] = next;
      }
    }
    if (step > max_len) done = true;
  }
  *n_out = n_tok;
  return check_launch(h, "ss_mt_greedy");
}

int ss_mt_greedy_batch(ss_engine* h, void* stream, const float* enc_dev, int B, int T_stride, const int32_t* T_host, int max_len_b,
                       int64_t* tokens_out_host, int max_out, int32_t* n_out_host) {
  if (!h || !h->finalized) return h ? h->fail(SS_ERR_STATE, "engine not finalized") : SS_ERR_INVALID;
  const ss_config& c = h->cfg;
  if (B <= 0 || T_stride <= 0 || !enc_dev || !T_host || !tokens_out_host || !n_out_host)
    return h->fail(SS_ERR_INVALID, "bad arguments to ss_mt_greedy_batch");
  int Tmax = 0;
  for (int b = 0; b < B; ++b) {
    if (T_host[b] < 1 || T_host[b] > T_stride) return h->fail(SS_ERR_INVALID, "ss_mt_greedy_batch: sample length outside [1, T_stride]");
    Tmax = std::max(Tmax, (int)T_host[b]);
  }
  int max_len = 0;
  int rc = mt_search_len(h, 0, -1, max_len_b, max_out, 0, &max_len);
  if (rc) return rc;
  cudaStream_t st = S(stream);
  const bool batched = mt_single_token_runs(h, Tmax);
  for (int g0 = 0; g0 < B; g0 += MT_BATCH_MAX_ROWS) {
    const int Bg = std::min(MT_BATCH_MAX_ROWS, B - g0);
    rc = batched && Bg >= h->mt_batch_min_rows ? mt_batch_group(h, st, enc_dev, g0, Bg, T_stride, T_host, max_len, tokens_out_host, max_out, n_out_host) : -1;
    if (rc == -1)  // sample by sample on ss_mt_greedy's path
      rc = mt_greedy_per_stream(h, stream, g0, Bg, enc_dev, (size_t)T_stride * c.enc_dim, nullptr, T_host, nullptr, nullptr, nullptr, max_len_b,
                                tokens_out_host, max_out, n_out_host, nullptr, 0);
    if (rc) return rc;
  }
  return check_launch(h, "ss_mt_greedy_batch");
}

int ss_mt_beam_batch(ss_engine* h, void* stream, const float* enc_dev, int B, int T_stride, const int32_t* T_host, int beam, int max_len_b,
                     float len_penalty, int64_t* tokens_out_host, int max_out, int32_t* n_out_host, float* scores_out_host,
                     float* pos_scores_out_host) {
  if (!h || !h->finalized) return h ? h->fail(SS_ERR_STATE, "engine not finalized") : SS_ERR_INVALID;
  const ss_config& c = h->cfg;
  if (B <= 0 || T_stride <= 0 || !enc_dev || !T_host || !tokens_out_host || !n_out_host || !scores_out_host || !pos_scores_out_host)
    return h->fail(SS_ERR_INVALID, "bad arguments to ss_mt_beam_batch");
  if (beam < 2 || beam > MT_BATCH_MAX_ROWS || 2 * beam > c.tgt_vocab)
    return h->fail(SS_ERR_INVALID, "ss_mt_beam_batch: beam outside [2, 32] (beam 1 is ss_mt_greedy_batch)");
  if (!std::isfinite(len_penalty)) return h->fail(SS_ERR_INVALID, "ss_mt_beam_batch: len_penalty is not finite");
  int Tmax = 0;
  for (int b = 0; b < B; ++b) {
    if (T_host[b] < 1 || T_host[b] > T_stride) return h->fail(SS_ERR_INVALID, "ss_mt_beam_batch: sample length outside [1, T_stride]");
    Tmax = std::max(Tmax, (int)T_host[b]);
  }
  int max_len = 0;
  int rc = mt_search_len(h, 0, -1, max_len_b, max_out, 0, &max_len);
  if (rc) return rc;
  if (!mt_single_token_runs(h, Tmax))
    return h->fail(SS_ERR_CUDA, "ss_mt_beam_batch: the beam search runs on the persistent MT kernels, which are off (option persistent_mt) "
                                "or do not support this shape");
  cudaStream_t st = S(stream);
  const int S_launch = MT_BATCH_MAX_ROWS / beam;  // samples per launch
  for (int g0 = 0; g0 < B; g0 += S_launch) {
    rc = mt_beam_group(h, st, mt_search_decoder(h), enc_dev, g0, std::min(S_launch, B - g0), beam, T_stride, T_host, max_len, len_penalty,
                       tokens_out_host, max_out, n_out_host, scores_out_host, pos_scores_out_host);
    if (rc) return rc;
  }
  return check_launch(h, "ss_mt_beam_batch");
}

int ss_t2u_encode_batch(ss_engine* h, void* stream, const float* mt_feats_dev, int B, int S_stride, const int32_t* S_host, float* out_dev) {
  if (!h || !h->finalized) return h ? h->fail(SS_ERR_STATE, "engine not finalized") : SS_ERR_INVALID;
  const ss_config& c = h->cfg;
  if (B <= 0 || S_stride <= 0 || !mt_feats_dev || !S_host || !out_dev) return h->fail(SS_ERR_INVALID, "bad arguments to ss_t2u_encode_batch");
  if (S_stride > c.max_mt_positions) return h->fail(SS_ERR_INVALID, "ss_t2u_encode_batch: S_stride > max_mt_positions");
  bool ragged = false;
  for (int b = 0; b < B; ++b) {
    if (S_host[b] < 1 || S_host[b] > S_stride) return h->fail(SS_ERR_INVALID, "ss_t2u_encode_batch: sample length outside [1, S_stride]");
    ragged |= S_host[b] < S_stride;
  }
  const int dim = c.unit_dim;
  const int G = std::max(1, SS_UNIT_BATCH_ROWS / S_stride);
  const size_t n_max = (size_t)std::min(G, B) * S_stride;
  if (!ws_begin(h, n_max * (dim * 8 + c.unit_ffn) * sizeof(float) + (size_t)B * sizeof(int) + 8 * 256)) return h->fail(SS_ERR_CUDA, "workspace allocation failed");
  int* lens_dev = ragged ? (int*)h->ws.raw((size_t)B * sizeof(int)) : nullptr;
  DecScratch sc = dec_scratch(h, (int)n_max, dim, c.unit_ffn);
  float* x = h->ws.f32(n_max * dim);
  if ((ragged && !lens_dev) || !sc.qkv || !x) return h->fail(SS_ERR_CUDA, "workspace too small");
  cudaStream_t st = S(stream);
  if (ragged) {  // the padding mask of prev_output_tokens_mt: keys at or beyond S_b
    cudaMemcpyAsync(lens_dev, S_host, (size_t)B * sizeof(int), cudaMemcpyHostToDevice, st);
    if (cudaStreamSynchronize(st) != cudaSuccess) return h->fail(SS_ERR_CUDA, std::string("ss_t2u_encode_batch: ") + cudaGetErrorString(cudaGetLastError()));
  }
  for (int g0 = 0; g0 < B; g0 += G) {
    const int Bg = std::min(G, B - g0), n = Bg * S_stride;
    copy_f32(mt_feats_dev + (size_t)g0 * S_stride * dim, x, (int64_t)n * dim, st);
    for (int l = 0; l < c.t2u_layers; ++l)
      dec_layer(h, h->t2u[l], x, n, dim, c.unit_ffn, c.unit_heads, c.uni_encoder != 0, ragged ? lens_dev + g0 : nullptr, nullptr, nullptr, 0, nullptr,
                0, nullptr, sc, st, 0, nullptr, Bg);
    layer_norm(x, dim, out_dev + (size_t)g0 * S_stride * dim, dim, h->t2u_ln.g, h->t2u_ln.b, n, dim, st);
  }
  return check_launch(h, "ss_t2u_encode_batch");
}

int ss_unit_search_batch(ss_engine* h, void* stream, const float* t2u_dev, int B, int S_stride, const int32_t* S_host, int max_len, float len_penalty,
                         int64_t* tokens_out_host, int max_out, int32_t* n_out_host, float* scores_out_host, float* pos_scores_out_host) {
  if (!h || !h->finalized) return h ? h->fail(SS_ERR_STATE, "engine not finalized") : SS_ERR_INVALID;
  const ss_config& c = h->cfg;
  if (B <= 0 || S_stride <= 0 || !t2u_dev || !S_host || !tokens_out_host || !n_out_host || !scores_out_host || !pos_scores_out_host)
    return h->fail(SS_ERR_INVALID, "bad arguments to ss_unit_search_batch");
  if (!h->unit_pos)
    return h->fail(SS_ERR_STATE, "ss_unit_search_batch: the handle has no autoregressive unit decoder (a StreamSpeech checkpoint; "
                                 "UnitY loads __const__.unit_pos_table)");
  if (max_len < 1) return h->fail(SS_ERR_INVALID, "ss_unit_search_batch: min_len cannot be larger than max_len");
  if (!std::isfinite(len_penalty)) return h->fail(SS_ERR_INVALID, "ss_unit_search_batch: len_penalty is not finite");
  int Smax = 0;
  for (int b = 0; b < B; ++b) {
    if (S_host[b] < 1 || S_host[b] > S_stride) return h->fail(SS_ERR_INVALID, "ss_unit_search_batch: sample length outside [1, S_stride]");
    Smax = std::max(Smax, (int)S_host[b]);
  }
  if (max_len > max_out) return h->fail(SS_ERR_CAPACITY, "ss_unit_search_batch: max_len > max_out");
  if (max_len + c.pad + 2 > h->unit_pos_rows)
    return h->fail(SS_ERR_CAPACITY, "ss_unit_search_batch: max_len " + std::to_string(max_len) + " needs " + std::to_string(max_len + c.pad + 2) +
                                        " rows of the unit position table, which has " + std::to_string(h->unit_pos_rows) + " (max_target_positions + pad + 1)");
  if (!h->persistent_mt || !mt_decode_persistent_supported(c.unit_dim, c.unit_ffn, c.unit_heads, c.unit_vocab, max_len + 2, Smax))
    return h->fail(Smax > 1024 ? SS_ERR_CAPACITY : SS_ERR_CUDA,
                   "ss_unit_search_batch: the unit search runs on the batched decoder kernel, which is off (option persistent_mt) or does not "
                   "support this shape (T2U states per sample <= 1024)");
  const SearchDecoder D{c.unit_layers, c.unit_ffn, c.unit_vocab, c.unit_dim, h->unit_emb, h->unit_pos, h->unit_ln.g, h->unit_ln.b,
                        h->unit_persist_layers, &h->unit, "ss_unit_search_batch"};
  cudaStream_t st = S(stream);
  for (int g0 = 0; g0 < B; g0 += MT_BATCH_MAX_ROWS) {
    const int rc = mt_beam_group(h, st, D, t2u_dev, g0, std::min(MT_BATCH_MAX_ROWS, B - g0), 1, S_stride, S_host, max_len, len_penalty, tokens_out_host,
                                 max_out, n_out_host, scores_out_host, pos_scores_out_host);
    if (rc) return rc;
  }
  return check_launch(h, "ss_unit_search_batch");
}

int ss_mt_incremental_reset(ss_engine* h) {
  if (!h) return SS_ERR_INVALID;
  h->mt_inc_self_len = 0;
  h->mt_inc_cross_rows = 0;
  h->mt_inc_overwritten = false;
  return SS_OK;
}

int ss_mt_greedy_incremental(ss_engine* h, void* stream, const float* enc_dev, int T, const int64_t* prefix_host, int n_prefix,
                             int max_new_tokens, int max_len_b, int64_t* tokens_out_host, int max_out, int* n_out) {
  if (!h || !h->finalized) return h ? h->fail(SS_ERR_STATE, "engine not finalized") : SS_ERR_INVALID;
  const ss_config& c = h->cfg;
  cudaStream_t st = S(stream);
  if (T <= 0 || n_prefix < 0 || !n_out) return h->fail(SS_ERR_INVALID, "bad arguments to ss_mt_greedy_incremental");
  const int start = n_prefix;
  if (!mt_tokens_in_vocab(h, prefix_host, start)) return h->fail(SS_ERR_INVALID, "ss_mt_greedy_incremental: prefix token outside the vocabulary");
  const int Tk = std::max(T, h->mt_inc_cross_rows);
  int max_len = 0, kv_off = 0;
  int rc = mt_incremental_len(h, -1, start, max_new_tokens, max_len_b, h->mt_inc_self_len, max_out, mt_single_token_runs(h, Tk), &max_len, &kv_off);
  if (rc) return rc;
  rc = ensure_mt_cross(h, Tk, h->mt_inc_cross_rows);
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
  mt_project_cross(h, enc_dev, h->mt_inc_cross_rows, T, h->mt_cross_kv, h->mt_cross_cap, st);
  h->mt_inc_cross_rows = Tk;
  mt_put_prefix(h, st, prefix_host, start, tokens_out_host);
  int n_tok = start, first = start, step = start;
  const int burst = (max_new_tokens >= 0) ? std::max(1, max_new_tokens + 1) : 32;
  const MtDecodeParams P = mt_decode_params(h, s, x, logits, feats, kv_off);
  rc = mt_single_token_bursts(h, st, P, &first, &step, max_len, Tk, burst, tokens_out_host, &n_tok, &h->mt_inc_self_len, "ss_mt_greedy_incremental");
  if (rc == -1) return h->fail(SS_ERR_CUDA, "ss_mt_greedy_incremental: cooperative launch of the persistent MT kernel was refused");
  if (rc) return rc;
  *n_out = n_tok;
  return check_launch(h, "ss_mt_greedy_incremental");
}

int ss_t2u_unit_decode(ss_engine* h, void* stream, const float* mt_feats_dev, int Slen, int n_pad_tail, int mask_eos, int64_t* argmax_dev,
                       int64_t* units_dev, int32_t* count_dev, float* t2u_out_dev, float* logits_dev) {
  if (!h || !h->finalized) return h ? h->fail(SS_ERR_STATE, "engine not finalized") : SS_ERR_INVALID;
  if (Slen <= 0 || n_pad_tail < 0 || n_pad_tail >= Slen) return h->fail(SS_ERR_INVALID, "bad T2U sequence length");
  const int32_t np = n_pad_tail;
  return t2u_unit_decode(h, S(stream), mt_feats_dev, 1, Slen, nullptr, &np, h->unit_pos_row, mask_eos, argmax_dev, units_dev, count_dev, 0, t2u_out_dev,
                         logits_dev, nullptr, "ss_t2u_unit_decode");
}

int ss_unit_position_row(ss_engine* h, const float* row_host) {
  if (!h || !h->finalized || !row_host) return h ? h->fail(SS_ERR_STATE, "engine not finalized / null row") : SS_ERR_INVALID;
  cudaDeviceSynchronize();  // earlier unit-decoder launches may still read the old row
  if (cudaMemcpy(h->unit_pos_row, row_host, (size_t)h->cfg.unit_dim * sizeof(float), cudaMemcpyHostToDevice) != cudaSuccess)
    return h->fail(SS_ERR_CUDA, "cudaMemcpy(unit positional row) failed");
  return SS_OK;
}

int ss_ctc_greedy_batch(ss_engine* h, void* stream, const float* enc_dev, int B, int T, int64_t* packed_out_dev) {
  if (!h || !h->finalized) return h ? h->fail(SS_ERR_STATE, "engine not finalized") : SS_ERR_INVALID;
  if (!h->has_ctc) return refuse_without_ctc(h, "ss_ctc_greedy_batch");
  if (B <= 0 || T <= 0 || !enc_dev || !packed_out_dev) return h->fail(SS_ERR_INVALID, "bad arguments to ss_ctc_greedy_batch");
  const ss_config& c = h->cfg;
  cudaStream_t st = S(stream);
  const bool pair = h->ctc_pair.N == 2 * c.src_vocab && c.tgt_vocab == c.src_vocab;
  const int Vmax = std::max(c.src_vocab, c.tgt_vocab);
  const int64_t W = 2 * (int64_t)T + 2;  // one head's packed output
  const int G = std::max(1, SS_CTC_BATCH_ROWS / T);
  for (int g0 = 0; g0 < B; g0 += G) {
    const int Bg = std::min(G, B - g0);
    const int rows = Bg * T;
    if (!ws_begin(h, (size_t)rows * 2 * Vmax * sizeof(float) + (size_t)rows * 2 * sizeof(int64_t) + 4 * 256))
      return h->fail(SS_ERR_CUDA, "workspace allocation failed");
    float* logits = h->ws.f32((size_t)rows * 2 * Vmax);
    int64_t* am = (int64_t*)h->ws.raw((size_t)rows * 2 * sizeof(int64_t));
    if (!logits || !am) return h->fail(SS_ERR_CUDA, "workspace too small");
    const float* x = enc_dev + (size_t)g0 * T * c.enc_dim;
    int64_t* out = packed_out_dev + (size_t)g0 * 2 * W;
    if (pair) {
      // [rows][2V] logits = 2 * rows arg-max rows of V (head-minor); sequence s = 2 b + head is sample b's head, at out + s * W
      linear(h, x, c.enc_dim, rows, h->ctc_pair, ep_out(logits, 2 * c.src_vocab), st, Bg);
      argmax_rows(logits, c.src_vocab, 2 * rows, c.src_vocab, h->mask_pad_unk, 2, am, st);  // never select pad, unk
      ctc_collapse_segments(am, T, 2, 2 * Bg, 0 /* <s> = CTC blank */, c.pad, out + 1, reinterpret_cast<int*>(out + 1 + T),
                            reinterpret_cast<int*>(out), W, st);
    } else {
      for (int hd = 0; hd < 2; ++hd) {
        const Linear& l = h->ctc_head[hd];
        linear(h, x, c.enc_dim, rows, l, ep_out(logits, l.N), st, Bg);
        argmax_rows(logits, l.N, rows, l.N, h->mask_pad_unk, 2, am, st);
        int64_t* o = out + hd * W;
        ctc_collapse_segments(am, T, 1, Bg, 0, c.pad, o + 1, reinterpret_cast<int*>(o + 1 + T), reinterpret_cast<int*>(o), 2 * W, st);
      }
    }
  }
  return check_launch(h, "ss_ctc_greedy_batch");
}

int ss_mt_features_batch(ss_engine* h, void* stream, const float* enc_dev, int B, int T_stride, const int32_t* T_host, const int64_t* tokens_host,
                         int Slen, float* feats_out_dev) {
  if (!h || !h->finalized) return h ? h->fail(SS_ERR_STATE, "engine not finalized") : SS_ERR_INVALID;
  const ss_config& c = h->cfg;
  if (B <= 0 || T_stride <= 0 || Slen <= 0 || Slen > c.max_mt_positions || !enc_dev || !T_host || !tokens_host || !feats_out_dev)
    return h->fail(SS_ERR_INVALID, "bad arguments to ss_mt_features_batch");
  // host side: [tokens int64 B*S | positions B*S | self key lengths B | cross key lengths B], one upload
  std::vector<int64_t> toks(tokens_host, tokens_host + (size_t)B * Slen);
  std::vector<int> ints((size_t)B * Slen + 2 * B);
  int* pos = ints.data();
  int* self_len = pos + (size_t)B * Slen;
  int* cross_len = self_len + B;
  for (int b = 0; b < B; ++b) {
    if (T_host[b] < 1 || T_host[b] > T_stride) return h->fail(SS_ERR_INVALID, "ss_mt_features_batch: sample length outside [1, T_stride]");
    const int64_t* t = tokens_host + (size_t)b * Slen;
    if (!mt_tokens_in_vocab(h, t, Slen)) return h->fail(SS_ERR_INVALID, "ss_mt_features_batch: token outside the vocabulary");
    int n_valid = Slen;  // trailing pads are masked as keys (ss_mt_features)
    while (n_valid > 0 && t[n_valid - 1] == c.pad) --n_valid;
    for (int i = 0; i < Slen; ++i) {
      if (i < n_valid && t[i] == c.pad) return h->fail(SS_ERR_INVALID, "pads are only supported as a tail");
      pos[(size_t)b * Slen + i] = t[i] == c.pad ? c.pad : c.pad + 1 + i;  // make_positions, restarting for every sample
    }
    self_len[b] = n_valid;
    cross_len[b] = T_host[b];
  }
  cudaStream_t st = S(stream);
  const int dim = c.mt_dim;
  const int G = std::max(1, SS_UNIT_BATCH_ROWS / (Slen * c.ctc_upsample_rate));
  const int Bg_max = std::min(G, B);
  const size_t n_max = (size_t)Bg_max * Slen;
  const size_t int_bytes = toks.size() * sizeof(int64_t) + ints.size() * sizeof(int);
  if (!ws_begin(h, (n_max * (dim * 8 + c.mt_ffn) + (size_t)Bg_max * T_stride * 2 * dim) * sizeof(float) + int_bytes + 16 * 256))
    return h->fail(SS_ERR_CUDA, "workspace allocation failed");
  int64_t* tok_dev = (int64_t*)h->ws.raw(toks.size() * sizeof(int64_t));
  int* ints_dev = (int*)h->ws.raw(ints.size() * sizeof(int));
  DecScratch s = dec_scratch(h, (int)n_max, dim, c.mt_ffn);
  float* x = h->ws.f32(n_max * dim);
  float* ckv = h->ws.f32((size_t)Bg_max * T_stride * 2 * dim);
  if (!tok_dev || !ints_dev || !s.hid || !s.qkv || !x || !ckv) return h->fail(SS_ERR_CUDA, "workspace too small");
  cudaMemcpyAsync(tok_dev, toks.data(), toks.size() * sizeof(int64_t), cudaMemcpyHostToDevice, st);
  cudaMemcpyAsync(ints_dev, ints.data(), ints.size() * sizeof(int), cudaMemcpyHostToDevice, st);
  if (cudaStreamSynchronize(st) != cudaSuccess)  // (host vectors)
    return h->fail(SS_ERR_CUDA, std::string("ss_mt_features_batch: ") + cudaGetErrorString(cudaGetLastError()));
  const int* pos_dev = ints_dev;
  const int* self_len_dev = pos_dev + (size_t)B * Slen;
  const int* cross_len_dev = self_len_dev + B;
  for (int g0 = 0; g0 < B; g0 += G) {
    const int Bg = std::min(G, B - g0);
    const int n = Bg * Slen;
    embed_tokens_pos(tok_dev + (size_t)g0 * Slen, pos_dev + (size_t)g0 * Slen, 0, h->mt_emb, h->mt_pos, sqrtf((float)dim), x, n, dim, c.pad, st);
    for (int l = 0; l < c.mt_layers; ++l) {
      // this layer's cross K / V of every row of the group's samples (rows past T_b are masked by cross_len)
      linear(h, enc_dev + (size_t)g0 * T_stride * c.enc_dim, c.enc_dim, Bg * T_stride, h->mt[l].ckv, ep_out(ckv, 2 * dim), st, Bg);
      dec_layer(h, h->mt[l], x, n, dim, c.mt_ffn, c.mt_heads, true, self_len_dev + g0, nullptr, nullptr, 0, ckv, T_stride, cross_len_dev + g0, s, st, 0,
                nullptr, Bg);
    }
    layer_norm(x, dim, feats_out_dev + (size_t)g0 * Slen * dim, dim, h->mt_ln.g, h->mt_ln.b, n, dim, st);
  }
  return check_launch(h, "ss_mt_features_batch");
}

// the checks and packed-output layout of ss_t2u_unit_decode_ragged / _batch_scored
static int t2u_unit_decode_packed(ss_engine* h, void* stream, const float* mt_feats_dev, int B, int S_stride, const int32_t* S_host,
                                  const int32_t* n_pad_tail_host, const float* pos_rows_dev, int mask_eos, int64_t* argmax_dev,
                                  int64_t* packed_units_dev, float* lprob_dev, const char* where) {
  if (!h || !h->finalized) return h ? h->fail(SS_ERR_STATE, "engine not finalized") : SS_ERR_INVALID;
  const ss_config& c = h->cfg;
  if (B <= 0 || S_stride <= 0 || S_stride > c.max_mt_positions || !mt_feats_dev || !n_pad_tail_host || !pos_rows_dev || !argmax_dev ||
      !packed_units_dev)
    return h->fail(SS_ERR_INVALID, std::string("bad arguments to ") + where);
  // sample b's [count | units] row of packed_units_dev: L + 1 int64 words
  const int64_t W = (int64_t)S_stride * c.ctc_upsample_rate + 1;
  return t2u_unit_decode(h, S(stream), mt_feats_dev, B, S_stride, S_host, n_pad_tail_host, pos_rows_dev, mask_eos, argmax_dev, packed_units_dev + 1,
                         reinterpret_cast<int32_t*>(packed_units_dev), W, nullptr, nullptr, lprob_dev, where);
}

int ss_t2u_unit_decode_ragged(ss_engine* h, void* stream, const float* mt_feats_dev, int B, int S_stride, const int32_t* S_host,
                              const int32_t* n_pad_tail_host, const float* pos_rows_dev, int mask_eos, int64_t* argmax_dev, int64_t* packed_units_dev) {
  return t2u_unit_decode_packed(h, stream, mt_feats_dev, B, S_stride, S_host, n_pad_tail_host, pos_rows_dev, mask_eos, argmax_dev, packed_units_dev,
                                nullptr, "ss_t2u_unit_decode_ragged");
}

int ss_t2u_unit_decode_batch_scored(ss_engine* h, void* stream, const float* mt_feats_dev, int B, int Slen, const int32_t* n_pad_tail_host,
                                    const float* pos_rows_dev, int mask_eos, int64_t* argmax_dev, int64_t* packed_units_dev, float* lprob_dev) {
  if (h && !lprob_dev) return h->fail(SS_ERR_INVALID, "bad arguments to ss_t2u_unit_decode_batch_scored");
  return t2u_unit_decode_packed(h, stream, mt_feats_dev, B, Slen, nullptr, n_pad_tail_host, pos_rows_dev, mask_eos, argmax_dev, packed_units_dev,
                                lprob_dev, "ss_t2u_unit_decode_batch_scored");
}

int ss_t2u_unit_decode_batch(ss_engine* h, void* stream, const float* mt_feats_dev, int B, int Slen, const int32_t* n_pad_tail_host, const float* pos_rows_dev,
                             int mask_eos, int64_t* argmax_dev, int64_t* packed_units_dev) {
  return ss_t2u_unit_decode_ragged(h, stream, mt_feats_dev, B, Slen, nullptr, n_pad_tail_host, pos_rows_dev, mask_eos, argmax_dev, packed_units_dev);
}

// The generator of one sequence as one launch per convolution (the reference path for the fused kernel, and the path of
// sequences it does not take): frames [N][in_dim] -> the n = N - ctx new frames' samples at out.
static void vocoder_multi_launch(ss_engine* h, cudaStream_t st, const float* frames, int N, int ctx, float* bufX, float* bufY, const std::vector<float*>& rbA,
                          const std::vector<float*>& rbB, const std::vector<float*>& rbT, const std::vector<float*>& rbO, float* wav, bool fan_out,
                          float* out) {
  const ss_config& c = h->cfg;
  const int nrb = c.voc_n_rb;
  // conv_pre
  {
    ConvA a;
    a.x = frames; a.B = 1; a.L_in = N; a.L_rows = N; a.C_in = c.voc_in_dim; a.ldx = c.voc_in_dim; a.ksize = 7; a.pad_left = 3;
    Epilogue e = ep_out(bufX, c.voc_init_channels);
    e.bias = h->conv_pre.lin.b;
    conv_gemm(h, a, h->conv_pre.lin.w, c.voc_init_channels, e, 0, st);
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
      ConvA a;
      a.x = bufX; a.B = 1; a.L_in = L; a.L_rows = nrows; a.C_in = U.cin; a.ldx = U.cin; a.ksize = J; a.pad_left = (J - 1) - q0;
      a.pre_lrelu = 0.1f;
      Epilogue e = ep_out(bufY, U.cout);
      e.bias = U.bias;
      e.out_L = Lout; e.out_row_stride = U.u; e.out_row_offset = q0 * U.u + phi - U.pad;
      conv_gemm(h, a, U.phase_w[phi].w, U.cout, e, lane, sp);
    }
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
      const int lane = fan_out ? j : 0;
      cudaStream_t sj = lane > 0 ? h->aux_stream[lane - 1] : st;
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
        conv_gemm(h, a1, w1.lin.w, ch, e1, lane, sj);
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
        conv_gemm(h, a2, w2.lin.w, ch, e2, lane, sj);
        cur = e2.out;
      }
      if (lane > 0) cudaEventRecord(h->join_event[lane - 1], sj);
    }
    if (fan_out)
      for (int q = 0; q < 2; ++q) cudaStreamWaitEvent(st, h->join_event[q], 0);
    // stage output in the reference's summation order: block 0, then + block 1, then + block 2
    if (nrb == 3) add3_f32(rbO[0], rbO[1], rbO[2], bufX, (int64_t)L * ch, st);
  }
  // x = leaky_relu(x) [slope 0.01, hifigan.py:166]; conv_post; tanh
  conv_post_tanh(bufX, L, ch, h->conv_post_w, h->conv_post_b, h->conv_post_k, 0.01f, wav, st);
  copy_f32(wav + (size_t)ctx * h->hop, out, (int64_t)(N - ctx) * h->hop, st);
}

int ss_vocoder_durations_ragged(ss_engine* h, void* stream, int n, const int64_t* codes_dev, const int32_t* U_host, int dur_prediction,
                                int64_t* dur_out_dev, int32_t* cumsum_out_dev) {
  if (!h || !h->finalized) return h ? h->fail(SS_ERR_STATE, "engine not finalized") : SS_ERR_INVALID;
  if (!h->has_vocoder) return h->fail(SS_ERR_STATE, "no vocoder weights were loaded");
  if (n <= 0 || !codes_dev || !U_host || !dur_out_dev) return h->fail(SS_ERR_INVALID, "bad arguments to ss_vocoder_durations_ragged");
  for (int s = 0; s < n; ++s)
    if (U_host[s] <= 0) return h->fail(SS_ERR_INVALID, "empty code sequence");
  const ss_config& c = h->cfg;
  cudaStream_t st = S(stream);
  const int E = c.voc_embedding_dim, Hd = c.voc_dur_hidden;
  // Padded rows of one group: the split-K partial sums of its GEMMs (conv1, conv2: Hd columns; projection: 1) must fit the split-K
  // scratch, or the GEMM would run unsplit and the group's rows would not equal those of a call of their own.  A sequence longer than
  // this runs alone, as in a call of its own.
  auto slices = [](int K) { return ((K + 15) / 16 + kVocDurTilesPerSplit - 1) / kVocDurTilesPerSplit; };
  const size_t per_row = (size_t)std::max({slices(h->dur_conv1.ksize * E) * Hd, slices(h->dur_conv2.ksize * Hd) * Hd, slices(Hd)}) * sizeof(float);
  const size_t dur_rows = splitk_workspace_bytes() / per_row;
  // groups of consecutive sequences, each padded to its longest one: [count][Umax] rows
  struct Group { int s0, count, Umax, row0; };
  std::vector<Group> groups;
  int rows = 0, max_rows = 0, n_cum = 0;
  for (int s = 0; s < n; ++s) {
    const int U = U_host[s];
    n_cum += U + 1;
    if (!groups.empty()) {
      Group& g = groups.back();
      const int um = std::max(g.Umax, U);
      if (g.count < VOC_MAX_STREAMS && (size_t)(g.count + 1) * um <= dur_rows) {
        ++g.count;
        g.Umax = um;
        continue;
      }
      rows += g.count * g.Umax;
      max_rows = std::max(max_rows, g.count * g.Umax);
    }
    groups.push_back(Group{s, 1, U, rows});
  }
  rows += groups.back().count * groups.back().Umax;
  max_rows = std::max(max_rows, groups.back().count * groups.back().Umax);
  if (rows > h->voc_ucap || n_cum > h->voc_ccap) {
    if (h->voc_unit_emb) cudaFree(h->voc_unit_emb);
    if (h->voc_cumsum) cudaFree(h->voc_cumsum);
    h->voc_unit_emb = nullptr;
    h->voc_cumsum = nullptr;
    h->voc_ucap = h->voc_ccap = 0;
    h->voc_seqs.clear();
    const int ucap = std::max(2 * rows, 1024), ccap = std::max(2 * n_cum, 1024);
    if (cudaMalloc((void**)&h->voc_unit_emb, (size_t)ucap * E * sizeof(float)) != cudaSuccess ||
        cudaMalloc((void**)&h->voc_cumsum, (size_t)ccap * sizeof(int)) != cudaSuccess)
      return h->fail(SS_ERR_CUDA, "cudaMalloc(vocoder unit cache) failed");
    h->voc_ucap = ucap;
    h->voc_ccap = ccap;
  }
  if (!ws_begin(h, ((size_t)max_rows * (2 * Hd + 1) + 4096) * sizeof(float))) return h->fail(SS_ERR_CUDA, "workspace allocation failed");
  float* a = h->ws.f32((size_t)max_rows * Hd);
  float* b = h->ws.f32((size_t)max_rows * Hd);
  float* ld = h->ws.f32(max_rows);
  if (!a || !b || !ld) return h->fail(SS_ERR_CUDA, "workspace too small");
  h->voc_seqs.assign(n, ss_engine::VocSeq{});
  int packed = 0;  // units of the sequences before the group
  for (const Group& g : groups) {
    // group-local geometry: unit rows of the padded [count][Umax] block, packed codes / durations / cumsums from the group's first
    VocSeqs q{};
    q.n = g.count;
    int pu = 0;
    for (int i = 0; i < g.count; ++i) {
      const int s = g.s0 + i;
      q.s[i].u0 = i * g.Umax;
      q.s[i].U = U_host[s];
      q.s[i].c0 = pu + i;
      h->voc_seqs[s] = ss_engine::VocSeq{g.row0 + i * g.Umax, U_host[s], packed + pu + g.s0 + i};
      pu += U_host[s];
    }
    const int M = g.count * g.Umax;
    float* emb = h->voc_unit_emb + (size_t)g.row0 * E;
    gather_codes_ragged(codes_dev + packed, q, g.Umax, h->voc_dict, E, emb, st);
    if (dur_prediction) {
      // VariancePredictor.forward (fairseq/models/text_to_speech/fastspeech2.py:144-151) on every sequence of the group.  Each
      // sequence sees zeros past its end, as alone: its pad rows are zero in the embeddings and re-zeroed after LayerNorm 1.
      // The split-K slices are fixed, so that a row's sums do not depend on the group's row count.
      ConvA c1;
      c1.x = emb; c1.B = g.count; c1.L_in = g.Umax; c1.L_rows = g.Umax; c1.C_in = E; c1.ldx = E;
      c1.ksize = h->dur_conv1.ksize; c1.pad_left = (h->dur_conv1.ksize - 1) / 2; c1.k_tiles_per_split = kVocDurTilesPerSplit;
      Epilogue e1 = ep_out(a, Hd, ACT_RELU);
      e1.bias = h->dur_conv1.lin.b;
      gemm_conv(c1, h->dur_conv1.lin.w, Hd, e1, &h->splitk[0], st);
      layer_norm(a, Hd, a, Hd, h->dur_ln1.g, h->dur_ln1.b, M, Hd, st);
      if (g.count > 1) zero_pad_rows(a, q, g.Umax, Hd, st);
      ConvA c2;
      c2.x = a; c2.B = g.count; c2.L_in = g.Umax; c2.L_rows = g.Umax; c2.C_in = Hd; c2.ldx = Hd;
      c2.ksize = h->dur_conv2.ksize; c2.pad_left = 1;  // padding=1 is hard-coded for conv2 (fastspeech2.py:137)
      c2.k_tiles_per_split = kVocDurTilesPerSplit;
      Epilogue e2 = ep_out(b, Hd, ACT_RELU);
      e2.bias = h->dur_conv2.lin.b;
      gemm_conv(c2, h->dur_conv2.lin.w, Hd, e2, &h->splitk[0], st);
      layer_norm(b, Hd, b, Hd, h->dur_ln2.g, h->dur_ln2.b, M, Hd, st);
      ConvA pr;
      pr.x = b; pr.L_in = M; pr.L_rows = M; pr.C_in = Hd; pr.ldx = Hd; pr.k_tiles_per_split = kVocDurTilesPerSplit;
      Epilogue e3 = ep_out(ld, 1);
      e3.bias = h->dur_proj.b;
      gemm_conv(pr, h->dur_proj.w, 1, e3, &h->splitk[0], st);
    }
    // no duration prediction: every code is one frame
    duration_from_log_ragged(dur_prediction ? ld : nullptr, q, dur_out_dev + packed, h->voc_cumsum + packed + g.s0, st);
    packed += pu;
  }
  if (cumsum_out_dev) cudaMemcpyAsync(cumsum_out_dev, h->voc_cumsum, (size_t)n_cum * sizeof(int), cudaMemcpyDeviceToDevice, st);
  return check_launch(h, "ss_vocoder_durations_ragged");
}

int ss_vocoder_durations(ss_engine* h, void* stream, const int64_t* codes_dev, int U, int dur_prediction, int64_t* dur_out_dev,
                         int32_t* cumsum_out_dev) {
  const int32_t U_host = U;
  return ss_vocoder_durations_ragged(h, stream, 1, codes_dev, &U_host, dur_prediction, dur_out_dev, cumsum_out_dev);
}

int ss_vocoder_generate_ragged(ss_engine* h, void* stream, int n, const int32_t* total_frames_host, const int32_t* frame0_host,
                               const int32_t* n_frames_host, const int32_t* left_context_host, float* wav_out_dev) {
  if (!h || !h->finalized) return h ? h->fail(SS_ERR_STATE, "engine not finalized") : SS_ERR_INVALID;
  if (!h->has_vocoder) return h->fail(SS_ERR_STATE, "no vocoder weights were loaded");
  if (n <= 0 || !total_frames_host || !frame0_host || !n_frames_host || !left_context_host || !wav_out_dev)
    return h->fail(SS_ERR_INVALID, "bad arguments to ss_vocoder_generate_ragged");
  if ((size_t)n != h->voc_seqs.size())
    return h->fail(SS_ERR_STATE, "ss_vocoder_generate_ragged needs an ss_vocoder_durations_ragged call with the same n first");
  for (int s = 0; s < n; ++s)
    if (n_frames_host[s] <= 0 || frame0_host[s] < 0 || frame0_host[s] + n_frames_host[s] != total_frames_host[s])
      return h->fail(SS_ERR_INVALID, "vocoder frame range must be the tail of the sequence");
  const ss_config& c = h->cfg;
  cudaStream_t st = S(stream);
  const int nrb = c.voc_n_rb;
  std::vector<int> ctx(n), N(n), dst(n);
  int n_out = 0;
  for (int s = 0; s < n; ++s) {
    ctx[s] = std::min(left_context_host[s] < 0 ? h->receptive_field : (int)left_context_host[s], (int)frame0_host[s]);
    N[s] = n_frames_host[s] + ctx[s];
    dst[s] = n_out;
    n_out += n_frames_host[s] * h->hop;
  }
  // groups of consecutive sequences that share the workspace buffers, sequence s at frame row row0[s] of its group
  std::vector<int> g_first, row0(n);
  int cap = 0, rows = 0;
  for (int s = 0; s < n; ++s) {
    if (s == 0 || s - g_first.back() >= VOC_MAX_STREAMS || rows + N[s] > kVocGroupFrames) {
      g_first.push_back(s);
      rows = 0;
    }
    row0[s] = rows;
    rows += N[s];
    cap = std::max(cap, rows);
  }
  g_first.push_back(n);
  cap = (cap + 63) & ~63;  // (a stable capacity keeps the fused kernel's templates cached across calls)
  // workspace: the group's frames + per-stage buffers; per frame each buffer holds max over stages of rows x channels
  size_t per_frame = c.voc_init_channels;
  {
    size_t L = 1, ch = c.voc_init_channels;
    for (int i = 0; i < c.voc_n_ups; ++i) {
      L *= c.voc_up_rates[i];
      ch /= 2;
      per_frame = std::max(per_frame, L * ch);
    }
  }
  const size_t maxbuf = (size_t)cap * per_frame;
  size_t total = ((size_t)cap * c.voc_in_dim + (size_t)(2 + 4 * nrb) * maxbuf + (size_t)cap * h->hop + 8192) * sizeof(float) + 64 * 256;
  if (!ws_begin(h, total)) return h->fail(SS_ERR_CUDA, "workspace allocation failed");
  float* frames = h->ws.f32((size_t)cap * c.voc_in_dim);
  float* bufX = h->ws.f32(maxbuf);   // stage input / output
  float* bufY = h->ws.f32(maxbuf);   // upsampled stage activation
  // per resblock (they run concurrently): ping-pong pair, conv1 output, block output
  std::vector<float*> rbA(nrb), rbB(nrb), rbT(nrb), rbO(nrb);
  bool ok = frames && bufX && bufY;
  for (int j = 0; j < nrb; ++j) {
    rbA[j] = h->ws.f32(maxbuf); rbB[j] = h->ws.f32(maxbuf); rbT[j] = h->ws.f32(maxbuf); rbO[j] = h->ws.f32(maxbuf);
    ok = ok && rbA[j] && rbB[j] && rbT[j] && rbO[j];
  }
  float* wav = h->ws.f32((size_t)cap * h->hop);
  if (!ok || !wav) return h->fail(SS_ERR_CUDA, "workspace too small");
  // The resblocks of a stage are independent until their outputs are averaged (hifigan.py:158-165).  Each one is a chain of
  // small latency-bound convs, so the multi-launch path runs them on separate streams (block 0 on the caller's) and they overlap.
  const bool fan_out = h->vocoder_streams && nrb == 3 && (h->umma_vocoder == 0 || h->umma_vocoder >= 12);
  if (fan_out && !h->fork_event) {
    bool made = cudaEventCreateWithFlags(&h->fork_event, cudaEventDisableTiming) == cudaSuccess;
    for (int i = 0; i < 2 && made; ++i)
      made = cudaStreamCreateWithFlags(&h->aux_stream[i], cudaStreamNonBlocking) == cudaSuccess &&
             cudaEventCreateWithFlags(&h->join_event[i], cudaEventDisableTiming) == cudaSuccess;
    if (!made) return h->fail(SS_ERR_CUDA, "cannot create the vocoder's auxiliary streams");
  }
  const bool fused_on = h->vocoder_fused != 0 && h->umma_vocoder == 12 && nrb == 3;
  for (size_t g = 0; g + 1 < g_first.size(); ++g) {
    const int s0 = g_first[g], s1 = g_first[g + 1];
    // V1 tail: repeat_interleave(x, dur) for each sequence's frame window (agent/tts/codehifigan.py:66), one launch
    VocSeqs q{};
    q.n = s1 - s0;
    for (int s = s0; s < s1; ++s) {
      const ss_engine::VocSeq& v = h->voc_seqs[s];
      q.s[s - s0] = {v.u0, v.U, v.c0, frame0_host[s] - ctx[s], N[s], row0[s]};
    }
    expand_frames_ragged(h->voc_unit_emb, h->voc_cumsum, q, row0[s1 - 1] + N[s1 - 1], c.voc_in_dim, frames, st);
    // Sequences of up to kVocFusedMaxFrames frames: conv_pre .. conv_post as one persistent kernel whose phases are separated by
    // grid barriers.  Longer ones, a shape the kernel does not support or a refused cooperative launch take the multi-launch path.
    std::vector<VocFusedSeq> fs;
    std::vector<char> in_fused(s1 - s0, 0);
    for (int s = s0; s < s1; ++s) {
      in_fused[s - s0] = fused_on && (h->vocoder_fused == 1 || N[s] <= kVocFusedMaxFrames);
      if (in_fused[s - s0]) fs.push_back(VocFusedSeq{N[s], row0[s], ctx[s], dst[s]});
    }
    bool launched = false;
    if (!fs.empty()) {
      VocFusedParams* T = vocoder_fused_table(h, cap, frames, bufX, bufY, rbA, rbB, rbT, rbO);
      launched = T && vocoder_fused_fill(h, *T, fs, wav_out_dev, st) && vocoder_fused(h->voc_call, h->persist_bar, &h->persist_bar_target, st) == 0;
    }
    for (int s = s0; s < s1; ++s)
      if (!(launched && in_fused[s - s0]))
        vocoder_multi_launch(h, st, frames + (size_t)row0[s] * c.voc_in_dim, N[s], ctx[s], bufX, bufY, rbA, rbB, rbT, rbO, wav, fan_out,
                             wav_out_dev + dst[s]);
  }
  return check_launch(h, "ss_vocoder_generate_ragged");
}

int ss_vocoder_generate(ss_engine* h, void* stream, int total_frames, int frame0, int n_frames, int left_context, float* wav_out_dev) {
  const int32_t t = total_frames, f0 = frame0, nf = n_frames, lc = left_context;
  return ss_vocoder_generate_ragged(h, stream, 1, &t, &f0, &nf, &lc, wav_out_dev);
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
    clear_voc_fused(h);
  }
  else if (n == "umma2_debug") {
    unsigned long long*& dbg = h->umma2_cache->dbg;
    if (value && !dbg) {
      if (cudaMalloc(&dbg, 16 * sizeof(unsigned long long)) != cudaSuccess) return h->fail(SS_ERR_CUDA, "cudaMalloc failed");
      cudaMemset(dbg, 0, 16 * sizeof(unsigned long long));
    }
    if (!value && dbg) {
      cudaDeviceSynchronize();
      cudaFree(dbg);
      dbg = nullptr;
    }
  }
  else if (n == "unit_grouped") h->unit_grouped = value;
  else if (n == "vocoder_fused") h->vocoder_fused = value;
  else if (n == "fbank_tma") h->fbank_tma = value;
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
  else if (n == "mt_batch_min_rows") h->mt_batch_min_rows = value;
  else if (n == "persistent_time") h->persistent_time = value;
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
    const unsigned long long* dbg = h->umma2_cache->dbg;
    if (!dbg || bytes > 16 * sizeof(unsigned long long)) return h->fail(SS_ERR_STATE, "no stamps (set option umma2_debug)");
    if (cudaMemcpy(host_dst, dbg, bytes, cudaMemcpyDeviceToHost) != cudaSuccess) return h->fail(SS_ERR_CUDA, "cudaMemcpy failed");
    return SS_OK;
  }
  if (n == "cluster_steps") {  // long long: encoder steps taken by the cluster kernel so far
    if (bytes < sizeof(long long)) return h->fail(SS_ERR_INVALID, "cluster_steps needs a long long");
    *(long long*)host_dst = h->cl_steps;
    return SS_OK;
  }
  // the incremental MT state of the handle or of one pool slot: {entries, cross_rows} (int32), self K, self V [mt_layers][entries][mt_dim],
  // cross K | V [mt_layers][cross_rows][2 * mt_dim]; bytes == 8 copies the two counts alone
  if (n == "mt_inc_state" || n.rfind("pool_mt_inc_state:", 0) == 0) {
    const ss_config& c = h->cfg;
    const size_t D = c.mt_dim, NL = c.mt_layers;
    int entries = h->mt_inc_self_len, rows = h->mt_inc_cross_rows;
    const float *sk = h->mt_self_k, *sv = h->mt_self_v, *ckv = h->mt_cross_kv;
    size_t cross_cap = h->mt_cross_cap;
    if (n[0] == 'p') {
      ss_engine::StreamPool& P = h->pool;
      char* end = nullptr;
      const long slot = std::strtol(n.c_str() + 18, &end, 10);
      if (!P.n_slots || end == n.c_str() + 18 || *end || slot < 0 || slot >= P.n_slots) return h->fail(SS_ERR_INVALID, "bad pool slot in " + n);
      entries = P.mt_inc_self_len[slot];
      rows = P.mt_inc_cross_rows[slot];
      const size_t self_slot = NL * c.max_mt_positions * D;
      sk = P.mt_self_kv ? P.mt_self_kv + slot * self_slot : nullptr;
      sv = P.mt_self_kv ? P.mt_self_kv + (P.n_slots + slot) * self_slot : nullptr;
      ckv = P.mt_cross ? P.mt_cross + slot * NL * P.Tcap * 2 * D : nullptr;
      cross_cap = P.Tcap;
    }
    int32_t* counts = (int32_t*)host_dst;
    const size_t need = 2 * sizeof(int32_t) + (2 * NL * entries * D + NL * rows * 2 * D) * sizeof(float);
    if (bytes == 2 * sizeof(int32_t)) {
      counts[0] = entries;
      counts[1] = rows;
      return SS_OK;
    }
    if (bytes < need) return h->fail(SS_ERR_INVALID, n + " needs " + std::to_string(need) + " bytes");
    counts[0] = entries;
    counts[1] = rows;
    float* out = (float*)(counts + 2);
    cudaDeviceSynchronize();
    for (size_t l = 0; l < NL && entries > 0; ++l)
      if (cudaMemcpy(out + l * entries * D, sk + l * c.max_mt_positions * D, entries * D * sizeof(float), cudaMemcpyDeviceToHost) != cudaSuccess ||
          cudaMemcpy(out + (NL + l) * entries * D, sv + l * c.max_mt_positions * D, entries * D * sizeof(float), cudaMemcpyDeviceToHost) != cudaSuccess)
        return h->fail(SS_ERR_CUDA, "cudaMemcpy failed");
    out += 2 * NL * entries * D;
    for (size_t l = 0; l < NL && rows > 0; ++l)
      if (cudaMemcpy(out + l * rows * 2 * D, ckv + l * cross_cap * 2 * D, rows * 2 * D * sizeof(float), cudaMemcpyDeviceToHost) != cudaSuccess)
        return h->fail(SS_ERR_CUDA, "cudaMemcpy failed");
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
  if (pieces != 2 && pieces != 3) return h->fail(SS_ERR_INVALID, "pieces must be 2 (bf16x3) or 3 (bf16x6)");
  ConvA a;
  a.x = x_dev; a.B = 1; a.L_in = M; a.L_rows = M; a.C_in = K; a.ldx = K;
  Epilogue ep = ep_out(out_dev, N, act);
  ep.bias = bias_dev;
  if (!umma2_supported(a, N, ep)) return h->fail(SS_ERR_INVALID, "shape not supported by the wgmma kernel");
  umma2_conv(h->umma2_cache, a, w_dev, N, ep, pieces, &h->splitk[0], S(stream));
  return check_launch(h, "ss_op_linear_umma");
}

int ss_op_conv1d(ss_engine* h, void* stream, const float* x_dev, int L, int C_in, const float* w_dev, const float* bias_dev, int N, int ksize,
                 int dil, int pad_left, float pre_lrelu, int mode, float* out_dev) {
  if (!h) return SS_ERR_INVALID;
  ConvA a;
  a.x = x_dev; a.B = 1; a.L_in = L; a.L_rows = L; a.C_in = C_in; a.ldx = C_in; a.ksize = ksize; a.dil = dil; a.pad_left = pad_left;
  a.pre_lrelu = pre_lrelu;
  Epilogue ep = ep_out(out_dev, N);
  ep.bias = bias_dev;
  if (mode >= 12) {
    if (!umma2_supported(a, N, ep)) return h->fail(SS_ERR_INVALID, "shape not supported by the wgmma conv kernel");
    umma2_conv(h->umma2_cache, a, w_dev, N, ep, mode - 10, &h->splitk[0], S(stream));
  } else if (mode >= 2) {
    return h->fail(SS_ERR_INVALID, "modes 2 / 3 (first-generation tensor-core kernel) were removed: use 12 / 13");
  } else {
    if (!gemm_conv_supported(a, w_dev, N, ep))
      return h->fail(SS_ERR_INVALID, "ss_op_conv1d: gemm_conv needs C_in % 4 == 0 and 16-byte aligned x and w");
    gemm_conv(a, w_dev, N, ep, &h->splitk[0], S(stream));
  }
  return check_launch(h, "ss_op_conv1d");
}

int ss_op_linear(ss_engine* h, void* stream, const float* x_dev, int M, int K, const float* w_dev, const float* bias_dev, int N, int act,
                 float* out_dev) {
  if (!h) return SS_ERR_INVALID;
  // the plain linear: skinny / fp32 CUDA-core kernels whatever the handle's routing (ss_op_linear_umma is the wgmma hook)
  Epilogue ep = ep_out(out_dev, N, act);
  ep.bias = bias_dev;
  ConvA a;
  a.x = x_dev; a.B = 1; a.L_in = M; a.L_rows = M; a.C_in = K; a.ldx = K;
  // both kernels read x and w as float4: 16-byte alignment and K % 4 == 0
  if (!gemm_conv_supported(a, w_dev, N, ep)) return h->fail(SS_ERR_INVALID, "ss_op_linear: needs K % 4 == 0 and 16-byte aligned x and w");
  if (skinny_gemm_supported(M, N, K, ep)) skinny_gemm(x_dev, K, w_dev, M, N, K, ep, S(stream));
  else gemm_conv(a, w_dev, N, ep, &h->splitk[0], S(stream));
  return check_launch(h, "ss_op_linear");
}

int ss_op_layer_norm(ss_engine* h, void* stream, const float* x_dev, int ldx, int rows, int C, const float* g_dev, const float* b_dev, float* out_dev,
                     int ldy) {
  if (!h) return SS_ERR_INVALID;
  if (!x_dev || !g_dev || !b_dev || !out_dev || rows < 0 || ldx < C || ldy < C)
    return h->fail(SS_ERR_INVALID, "ss_op_layer_norm: a null pointer, rows < 0 or a row stride below C");
  if (!layer_norm_supported(C)) return h->fail(SS_ERR_INVALID, "ss_op_layer_norm: C = " + std::to_string(C) + " is not a multiple of 32 in [32, 1024]");
  layer_norm(x_dev, ldx, out_dev, ldy, g_dev, b_dev, rows, C, S(stream));
  return check_launch(h, "ss_op_layer_norm");
}

int ss_op_gemm(ss_engine* h, void* stream, ss_op_gemm_args* g) {
  if (!h) return SS_ERR_INVALID;
  if (!g) return h->fail(SS_ERR_INVALID, "ss_op_gemm: null arguments");
  auto refuse = [&](const std::string& why) { return h->fail(SS_ERR_INVALID, "ss_op_gemm: " + why); };
  ConvA a;
  a.x = g->x; a.B = g->B; a.L_in = g->L_in; a.L_rows = g->L_rows; a.C_in = g->C_in; a.ldx = g->ldx; a.ksize = g->ksize; a.stride = g->stride;
  a.dil = g->dil; a.pad_left = g->pad_left; a.chunk = g->chunk; a.pre_lrelu = g->pre_lrelu; a.lengths = g->lengths; a.t_offset = g->t_offset;
  a.x_row0 = g->x_row0; a.x_rows = g->x_rows; a.k_tiles_per_split = g->k_tiles_per_split;
  Epilogue ep;
  ep.bias = g->bias; ep.act = g->act; ep.glu = g->glu; ep.alpha = g->alpha; ep.residual = g->residual; ep.res_scale = g->res_scale;
  ep.accumulate = g->accumulate; ep.out = g->out; ep.ldo = g->ldo; ep.out_L = g->out_L; ep.out_row_stride = g->out_row_stride;
  ep.out_row_offset = g->out_row_offset; ep.ln_gamma = g->ln_gamma; ep.ln_beta = g->ln_beta; ep.split_n = g->split_n; ep.out2 = g->out2;
  ep.out3 = g->out3; ep.ldo2 = g->ldo2; ep.ldo3 = g->ldo3;
  const int N = g->N, M = a.B * a.L_rows, K = a.ksize * a.C_in;
  if (!a.x || !g->w || !ep.out) return refuse("null x, w or out");
  if (a.B < 1 || a.L_in < 1 || a.L_rows < 1 || a.C_in < 1 || a.ldx < a.C_in || a.ksize < 1 || a.stride < 1 || a.dil < 1 || a.pad_left < 0 ||
      a.chunk < 0 || a.t_offset < 0 || a.x_row0 < 0 || a.x_rows < 0 || a.k_tiles_per_split < 0 || N < 1)
    return refuse("bad A shape or N");
  if (ep.act < ACT_NONE || ep.act > ACT_GELU || (ep.glu != 0 && ep.glu != 1) || (ep.accumulate != 0 && ep.accumulate != 1) || ep.out_L < 0 ||
      ep.ldo < 1 || (ep.ln_gamma == nullptr) != (ep.ln_beta == nullptr) || ep.split_n < 0 ||
      (ep.split_n > 0 && (!ep.out2 || !ep.out3 || (ep.glu ? N / 2 : N) > 3 * ep.split_n)))
    return refuse("bad epilogue");
  if (g->kernel < 0 || g->kernel > GK_UMMA3) return refuse("kernel must be in [0, 4]");
  if (g->splitk != 0 && g->splitk != 1) return refuse("splitk must be 0 or 1");
  const bool plain = a.B == 1 && a.ksize == 1 && a.stride == 1 && a.pad_left == 0 && a.chunk == 0 && !a.lengths && a.L_in == a.L_rows &&
                     a.t_offset == 0 && a.x_row0 == 0 && a.x_rows == 0;
  int kernel = g->kernel;
  if (kernel == 0) {
    kernel = plain ? linear_kernel(h, a, N, ep, 1) : conv_gemm_kernel(h, a, N, ep);
    // the engine fuses the LayerNorm and the Q|K|V routing only on the skinny kernel (ln_linear, ln_qkv_routed)
    if ((ep.ln_gamma || ep.split_n) && kernel != GK_SKINNY) return refuse("the fused LayerNorm and split_n routing exist only on skinny_gemm");
  }
  float** splitk = g->splitk ? &h->splitk[0] : nullptr;
  g->route_kernel = kernel;
  g->route_bm = g->route_bn = g->route_mr = g->route_ks = g->route_cpt = g->route_grid = g->route_u_bn = g->route_u_ck = g->route_u_upt =
      g->route_u_sb = 0;
  g->route_splits = 1;
  const uintptr_t misaligned = (reinterpret_cast<uintptr_t>(a.x) | reinterpret_cast<uintptr_t>(g->w)) & 15;
  if (kernel == GK_GEMM_CONV) {
    if (!gemm_conv_supported(a, g->w, N, ep))
      return refuse("gemm_conv needs C_in and ldx multiples of 4, 16-byte aligned x and w, an even N with glu, and no ln_gamma / split_n");
    const GemmPlan p = gemm_conv_plan(a, N, ep, splitk != nullptr);
    g->route_bm = p.BM; g->route_bn = p.BN; g->route_splits = p.splits;
    gemm_conv(a, g->w, N, ep, splitk, S(stream));
  } else if (kernel == GK_SKINNY) {
    if (!plain || !skinny_gemm_supported(M, N, K, ep) || (a.ldx & 3) || misaligned ||
        (ep.ln_gamma && ((reinterpret_cast<uintptr_t>(ep.ln_gamma) | reinterpret_cast<uintptr_t>(ep.ln_beta)) & 15)))
      return refuse("skinny_gemm needs a plain matrix with M <= 64, K % 128 == 0, ldx % 4 == 0, 16-byte aligned x, w (and LN vectors), "
                    "K <= 1024 with LayerNorm, an even N with glu, no out_L and act in [0, 4]");
    const SkinnyPlan p = skinny_gemm_plan(M, N, K, ep);
    g->route_mr = p.MR; g->route_ks = p.KS; g->route_cpt = p.CPT; g->route_grid = p.grid;
    skinny_gemm(a.x, a.ldx, g->w, M, N, K, ep, S(stream));
  } else {
    if (!umma2_supported(a, N, ep)) return refuse("shape not supported by the wgmma kernel");
    const int pieces = kernel == GK_UMMA3 ? 3 : 2;
    const Umma2Plan p = umma2_plan(a, N, pieces, splitk != nullptr);
    g->route_splits = p.splits; g->route_u_bn = p.BN; g->route_u_ck = p.CK; g->route_u_upt = p.UPT; g->route_u_sb = p.SB;
    umma2_conv(h->umma2_cache, a, g->w, N, ep, pieces, splitk, S(stream));
  }
  return check_launch(h, "ss_op_gemm");
}

int ss_op_argmax_rows(ss_engine* h, void* stream, const float* logits_dev, int rows, int V, int ld, int n_masked, int64_t* idx_dev, float* lprob_dev) {
  if (!h || rows < 0 || V <= 0 || ld < V || n_masked < 0 || n_masked > 3 || !logits_dev || !idx_dev) return h ? h->fail(SS_ERR_INVALID, "bad arguments to ss_op_argmax_rows") : SS_ERR_INVALID;
  if (lprob_dev)
    argmax_lprob_rows(logits_dev, ld, rows, V, h->mask_pad_unk, n_masked, idx_dev, lprob_dev, S(stream));
  else
    argmax_rows(logits_dev, ld, rows, V, h->mask_pad_unk, n_masked, idx_dev, S(stream));
  return check_launch(h, "ss_op_argmax_rows");
}

}  // extern "C"

namespace {

// Host arrays of one parity-test launch, copied to device memory that lives until the launch has finished.
struct OpUploads {
  std::vector<void*> ptrs;
  template <class T>
  const T* put(const T* host, size_t n) {
    if (!host || n == 0) return nullptr;
    void* d = nullptr;
    if (cudaMalloc(&d, n * sizeof(T)) != cudaSuccess) throw std::runtime_error("cudaMalloc failed");
    ptrs.push_back(d);
    if (cudaMemcpy(d, host, n * sizeof(T), cudaMemcpyHostToDevice) != cudaSuccess) throw std::runtime_error("cudaMemcpy failed");
    return static_cast<const T*>(d);
  }
  // checks the launch, waits for it and frees the copies
  int finish(ss_engine* h, cudaStream_t st, const char* where) {
    const int rc = check_launch(h, where);
    if (rc != SS_OK) return rc;
    const cudaError_t e = cudaStreamSynchronize(st);
    return e == cudaSuccess ? SS_OK : h->fail(SS_ERR_CUDA, std::string(where) + ": " + cudaGetErrorString(e));
  }
  ~OpUploads() {
    for (void* p : ptrs) cudaFree(p);
  }
};

bool row_stride_ok(int ld, int D) { return ld >= D && ld % 4 == 0; }

// every length in [1, T]
bool lengths_ok(const int32_t* len, int B, int T) {
  for (int b = 0; len && b < B; ++b)
    if (len[b] < 1 || len[b] > T) return false;
  return true;
}

constexpr size_t ROW_KERNEL_SMEM = 160 * 1024;  // kernels_attn.cu: the row kernel keeps T scores in shared memory

}  // namespace

extern "C" {

int ss_op_relpos_attention(ss_engine* h, void* stream, const float* q_dev, int ldq, const float* k_dev, int ldk, const float* v_dev, int ldv,
                           const float* pos_dev, int Tpos, const float* bias_u_dev, const float* bias_v_dev, float* out_dev, int B, int nQ,
                           int q_offset, int T, int H, int D, int chunk, const int32_t* lengths_host, int kernel) {
  if (!h) return SS_ERR_INVALID;
  if (!q_dev || !k_dev || !v_dev || !pos_dev || !bias_u_dev || !bias_v_dev || !out_dev) return h->fail(SS_ERR_INVALID, "ss_op_relpos_attention: null pointer");
  if (B < 1 || nQ < 1 || T < 1 || H < 1 || D != H * 64 || T > Tpos || q_offset < 0 || q_offset + nQ > T || chunk < 0 || kernel < 0 || kernel > 2 ||
      !row_stride_ok(ldq, D) || !row_stride_ok(ldk, D) || !row_stride_ok(ldv, D))
    return h->fail(SS_ERR_INVALID, "ss_op_relpos_attention: bad shape");
  if (!lengths_ok(lengths_host, B, T)) return h->fail(SS_ERR_INVALID, "ss_op_relpos_attention: a length outside [1, T]");
  if (kernel == 1 && (size_t)T * sizeof(float) > ROW_KERNEL_SMEM) return h->fail(SS_ERR_INVALID, "ss_op_relpos_attention: T too long for the row kernel");
  try {
    OpUploads up;
    relpos_attention(q_dev, ldq, k_dev, ldk, v_dev, ldv, pos_dev, Tpos, bias_u_dev, bias_v_dev, out_dev, B, nQ, q_offset, T, H, D, chunk,
                     up.put(lengths_host, B), S(stream), kernel);
    return up.finish(h, S(stream), "ss_op_relpos_attention");
  } catch (const std::exception& e) {
    return h->fail(SS_ERR_CUDA, e.what());
  }
}

int ss_op_mha_attention(ss_engine* h, void* stream, const float* q_dev, int ldq, const float* k_dev, int ldk, const float* v_dev, int ldv, float* out_dev,
                        int ldo, int B, int Tq, int Tk, int H, float scale, int causal, int causal_offset, const int32_t* kv_len_host, int kernel) {
  if (!h) return SS_ERR_INVALID;
  if (!q_dev || !k_dev || !v_dev || !out_dev) return h->fail(SS_ERR_INVALID, "ss_op_mha_attention: null pointer");
  const int D = H * 64;
  if (B < 1 || Tq < 1 || Tk < 1 || H < 1 || causal < 0 || causal > 1 || causal_offset < 0 || kernel < 0 || kernel > 2 || !row_stride_ok(ldq, D) ||
      !row_stride_ok(ldk, D) || !row_stride_ok(ldv, D) || !row_stride_ok(ldo, D))
    return h->fail(SS_ERR_INVALID, "ss_op_mha_attention: bad shape");
  if (!lengths_ok(kv_len_host, B, Tk)) return h->fail(SS_ERR_INVALID, "ss_op_mha_attention: a key length outside [1, Tk]");
  if (kernel == 1 && (size_t)Tk * sizeof(float) > ROW_KERNEL_SMEM) return h->fail(SS_ERR_INVALID, "ss_op_mha_attention: Tk too long for the row kernel");
  try {
    OpUploads up;
    mha_attention(q_dev, ldq, k_dev, ldk, v_dev, ldv, out_dev, ldo, B, Tq, Tk, H, scale, causal, causal_offset, up.put(kv_len_host, B), S(stream),
                  kernel);
    return up.finish(h, S(stream), "ss_op_mha_attention");
  } catch (const std::exception& e) {
    return h->fail(SS_ERR_CUDA, e.what());
  }
}

int ss_op_grouped_causal_attention(ss_engine* h, void* stream, const float* q_dev, int ldq, const float* k_dev, int ldk, const float* v_dev, int ldv,
                                   float* out_dev, int ldo, int S_, int R, int H, float scale, int B, const int32_t* kv_len_host) {
  if (!h) return SS_ERR_INVALID;
  if (!q_dev || !k_dev || !v_dev || !out_dev) return h->fail(SS_ERR_INVALID, "ss_op_grouped_causal_attention: null pointer");
  const int D = H * 64;
  // the kernel keeps S scores in the default 48 KB of dynamic shared memory
  if (B < 1 || S_ < 1 || S_ > 12 * 1024 || R < 1 || H < 1 || !row_stride_ok(ldq, D) || !row_stride_ok(ldk, D) || !row_stride_ok(ldv, D) ||
      ldo < D)
    return h->fail(SS_ERR_INVALID, "ss_op_grouped_causal_attention: bad shape");
  if (!lengths_ok(kv_len_host, B, S_)) return h->fail(SS_ERR_INVALID, "ss_op_grouped_causal_attention: a key length outside [1, S]");
  try {
    OpUploads up;
    grouped_causal_attention(q_dev, ldq, k_dev, ldk, v_dev, ldv, out_dev, ldo, S_, R, H, scale, up.put(kv_len_host, B), B, S(stream));
    return up.finish(h, S(stream), "ss_op_grouped_causal_attention");
  } catch (const std::exception& e) {
    return h->fail(SS_ERR_CUDA, e.what());
  }
}

int ss_op_depthwise_bn_silu(ss_engine* h, void* stream, const float* x_dev, int ldx, const float* w_dev, const float* scale_dev, const float* shift_dev,
                            float* y_dev, int ldy, int B, int T, int t0, int n, int C, int k, int chunk) {
  if (!h) return SS_ERR_INVALID;
  if (!x_dev || !w_dev || !scale_dev || !shift_dev || !y_dev) return h->fail(SS_ERR_INVALID, "ss_op_depthwise_bn_silu: null pointer");
  if (B < 1 || T < 1 || t0 < 0 || n < 1 || t0 + n > T || C < 1 || ldx < C || ldy < C || k < 1 || k % 2 == 0 || chunk < 0)
    return h->fail(SS_ERR_INVALID, "ss_op_depthwise_bn_silu: bad shape");
  depthwise_bn_silu(x_dev, ldx, w_dev, scale_dev, shift_dev, y_dev, ldy, B, T, t0, n, C, k, chunk, S(stream));
  return check_launch(h, "ss_op_depthwise_bn_silu");
}

}  // extern "C"

namespace {

// MsStream descriptors of a multi-stream parity-test launch; false when a stream is out of range: a slot outside [0, n_slots), T outside
// [1, T_cap], a0 < 0, nA outside [0, T - a0], a chunk < 0, or output rows outside [0, rows)
bool ms_streams(int n, const int32_t* slot, const int32_t* a0, const int32_t* nA, const int32_t* T, const int32_t* chunk, const int32_t* row0,
                int n_slots, int T_cap, int rows, bool conv, std::vector<MsStream>& out, int& max_nA, int& Tmax) {
  out.assign(n, MsStream{});
  max_nA = 0;
  Tmax = 0;
  for (int b = 0; b < n; ++b) {
    MsStream& s = out[b];
    s.slot = slot[b]; s.a0 = a0[b]; s.nA = nA[b]; s.T = T[b]; s.row0 = row0[b];
    (conv ? s.conv_chunk : s.attn_chunk) = chunk[b];
    if (s.slot < 0 || s.slot >= n_slots || s.T < 1 || s.T > T_cap || s.a0 < 0 || s.nA < 0 || s.nA > s.T - s.a0 || chunk[b] < 0 || s.row0 < 0 ||
        s.row0 + s.nA > rows)
      return false;
    max_nA = std::max(max_nA, s.nA);
    Tmax = std::max(Tmax, s.T);
  }
  return true;
}

}  // namespace

extern "C" {

int ss_op_ms_relpos_attention(ss_engine* h, void* stream, const float* q_dev, int ldq, const float* kc_dev, const float* vc_dev, int64_t slot_stride,
                              int n_slots, const float* pos_dev, int Tpos, const float* bias_u_dev, const float* bias_v_dev, float* out_dev, int ldo,
                              int rows, int H, int n, const int32_t* slot_host, const int32_t* a0_host, const int32_t* nA_host, const int32_t* T_host,
                              const int32_t* attn_chunk_host, const int32_t* row0_host) {
  if (!h) return SS_ERR_INVALID;
  if (!q_dev || !kc_dev || !vc_dev || !pos_dev || !bias_u_dev || !bias_v_dev || !out_dev || !slot_host || !a0_host || !nA_host || !T_host ||
      !attn_chunk_host || !row0_host)
    return h->fail(SS_ERR_INVALID, "ss_op_ms_relpos_attention: null pointer");
  const int D = H * 64;
  if (n < 1 || H < 1 || n_slots < 1 || rows < 1 || Tpos < 1 || slot_stride < (int64_t)D || !row_stride_ok(ldq, D) || !row_stride_ok(ldo, D))
    return h->fail(SS_ERR_INVALID, "ss_op_ms_relpos_attention: bad shape");
  // keys of a stream: T rows of D floats inside its slot; the row kernel keeps T scores in shared memory
  const int T_cap = (int)std::min<int64_t>({(int64_t)Tpos, slot_stride / D, (int64_t)(ROW_KERNEL_SMEM / sizeof(float))});
  std::vector<MsStream> st_host;
  int max_nA = 0, Tmax = 0;
  if (!ms_streams(n, slot_host, a0_host, nA_host, T_host, attn_chunk_host, row0_host, n_slots, T_cap, rows, false, st_host, max_nA, Tmax))
    return h->fail(SS_ERR_INVALID, "ss_op_ms_relpos_attention: a stream's slot, rows or chunk is out of range");
  try {
    OpUploads up;
    ms_relpos_attention(q_dev, ldq, kc_dev, vc_dev, slot_stride, D, pos_dev, Tpos, bias_u_dev, bias_v_dev, out_dev, ldo, up.put(st_host.data(), n), n,
                        max_nA, H, Tmax, S(stream));
    return up.finish(h, S(stream), "ss_op_ms_relpos_attention");
  } catch (const std::exception& e) {
    return h->fail(SS_ERR_CUDA, e.what());
  }
}

int ss_op_ms_depthwise(ss_engine* h, void* stream, const float* x_dev, int64_t slot_stride, int n_slots, const float* w_dev, const float* scale_dev,
                       const float* shift_dev, float* y_dev, int ldy, int rows, int C, int k, int n, const int32_t* slot_host, const int32_t* a0_host,
                       const int32_t* nA_host, const int32_t* T_host, const int32_t* conv_chunk_host, const int32_t* row0_host) {
  if (!h) return SS_ERR_INVALID;
  if (!x_dev || !w_dev || !scale_dev || !shift_dev || !y_dev || !slot_host || !a0_host || !nA_host || !T_host || !conv_chunk_host || !row0_host)
    return h->fail(SS_ERR_INVALID, "ss_op_ms_depthwise: null pointer");
  if (n < 1 || C < 1 || k < 1 || k % 2 == 0 || n_slots < 1 || rows < 1 || slot_stride < (int64_t)C || ldy < C)
    return h->fail(SS_ERR_INVALID, "ss_op_ms_depthwise: bad shape");
  std::vector<MsStream> st_host;
  int max_nA = 0, Tmax = 0;
  const int T_cap = (int)std::min<int64_t>(slot_stride / C, 1 << 30);
  if (!ms_streams(n, slot_host, a0_host, nA_host, T_host, conv_chunk_host, row0_host, n_slots, T_cap, rows, true, st_host, max_nA, Tmax))
    return h->fail(SS_ERR_INVALID, "ss_op_ms_depthwise: a stream's slot, rows or chunk is out of range");
  try {
    OpUploads up;
    ms_depthwise(x_dev, slot_stride, w_dev, scale_dev, shift_dev, y_dev, ldy, up.put(st_host.data(), n), n, max_nA, C, k, S(stream));
    return up.finish(h, S(stream), "ss_op_ms_depthwise");
  } catch (const std::exception& e) {
    return h->fail(SS_ERR_CUDA, e.what());
  }
}

}  // extern "C"

#include "engine_pool.inc"
