// Handle lifecycle, tensor loading and the one-time repack to kernel layouts (ss_finalize).
#include <cstdio>
#include <cstring>
#include <cmath>
#include <stdexcept>

#include "engine.h"

using namespace ss;

namespace ss {

void* Arena::raw(size_t bytes) {
  size_t a = (off + 255) & ~(size_t)255;
  if (a + bytes > cap) return nullptr;
  off = a + bytes;
  return base + a;
}

bool Arena::ensure(size_t bytes) {
  if (bytes <= cap) return true;
  if (base) cudaFree(base);
  base = nullptr;
  cap = 0;
  size_t want = bytes + (bytes >> 2) + (1 << 20);
  if (cudaMalloc((void**)&base, want) != cudaSuccess) return false;
  cap = want;
  return true;
}

}  // namespace ss

namespace {

struct MissingKey : std::runtime_error {
  using std::runtime_error::runtime_error;
};

const HostTensor& get(ss_engine* h, const std::string& key) {
  auto it = h->host.find(key);
  if (it == h->host.end()) throw MissingKey(key);
  return it->second;
}

float* upload(ss_engine* h, const float* src, size_t n) {
  float* d = nullptr;
  if (cudaMalloc((void**)&d, std::max<size_t>(n, 1) * sizeof(float)) != cudaSuccess) throw std::runtime_error("cudaMalloc failed");
  h->dev_allocs.push_back(d);
  if (n) cudaMemcpy(d, src, n * sizeof(float), cudaMemcpyHostToDevice);
  return d;
}
float* upload(ss_engine* h, const std::vector<float>& v) { return upload(h, v.data(), v.size()); }

template <typename T>
T* dev_alloc(ss_engine* h, size_t n) {
  T* d = nullptr;
  if (cudaMalloc((void**)&d, std::max<size_t>(n, 1) * sizeof(T)) != cudaSuccess) throw std::runtime_error("cudaMalloc failed");
  h->dev_allocs.push_back(d);
  return d;
}

void expect_shape(const HostTensor& t, const std::string& key, std::initializer_list<int64_t> shape) {
  std::vector<int64_t> s(shape);
  if (t.shape != s) {
    std::string m = "shape mismatch for " + key + ": got [";
    for (auto v : t.shape) m += std::to_string(v) + ",";
    m += "] expected [";
    for (auto v : s) m += std::to_string(v) + ",";
    throw std::runtime_error(m + "]");
  }
}

Linear make_linear(ss_engine* h, const std::string& prefix, int N, int K, bool bias = true) {
  const HostTensor& w = get(h, prefix + ".weight");
  if (w.numel() != (int64_t)N * K) throw std::runtime_error("size mismatch for " + prefix + ".weight");
  Linear l;
  l.N = N;
  l.K = K;
  l.w = upload(h, w.data);
  if (bias) {
    const HostTensor& b = get(h, prefix + ".bias");
    if (b.numel() != N) throw std::runtime_error("size mismatch for " + prefix + ".bias");
    l.b = upload(h, b.data);
  }
  return l;
}

// rows of several [Ni][K] linears concatenated
Linear make_fused(ss_engine* h, const std::vector<std::string>& prefixes, int Neach, int K) {
  std::vector<float> w, b;
  for (auto& p : prefixes) {
    const HostTensor& wi = get(h, p + ".weight");
    const HostTensor& bi = get(h, p + ".bias");
    if (wi.numel() != (int64_t)Neach * K || bi.numel() != Neach) throw std::runtime_error("size mismatch for " + p);
    w.insert(w.end(), wi.data.begin(), wi.data.end());
    b.insert(b.end(), bi.data.begin(), bi.data.end());
  }
  Linear l;
  l.N = Neach * (int)prefixes.size();
  l.K = K;
  l.w = upload(h, w);
  l.b = upload(h, b);
  return l;
}

LNorm make_ln(ss_engine* h, const std::string& prefix, int C) {
  const HostTensor& g = get(h, prefix + ".weight");
  const HostTensor& b = get(h, prefix + ".bias");
  if (g.numel() != C || b.numel() != C) throw std::runtime_error("size mismatch for " + prefix);
  if (C != 128 && C != 256 && C != 512 && C != 1024) throw std::runtime_error("LayerNorm width must be 128/256/512/1024: " + prefix);
  LNorm l;
  l.C = C;
  l.g = upload(h, g.data);
  l.b = upload(h, b.data);
  return l;
}

// torch Conv1d weight [Cout][Cin][k] -> [Cout'][k*Cin] (tap-major), optional GLU row interleave
ConvW make_conv(ss_engine* h, const std::string& prefix, int cout, int cin, int k, int dil, bool glu_interleave, bool bias = true) {
  const HostTensor& w = get(h, prefix + ".weight");
  if (w.numel() != (int64_t)cout * cin * k) throw std::runtime_error("size mismatch for " + prefix + ".weight");
  std::vector<float> p((size_t)cout * cin * k);
  std::vector<float> pb(cout, 0.f);
  const HostTensor* b = bias ? &get(h, prefix + ".bias") : nullptr;
  if (b && b->numel() != cout) throw std::runtime_error("size mismatch for " + prefix + ".bias");
  for (int co = 0; co < cout; ++co) {
    int row = co;
    if (glu_interleave) row = (co < cout / 2) ? 2 * co : 2 * (co - cout / 2) + 1;
    for (int ci = 0; ci < cin; ++ci)
      for (int t = 0; t < k; ++t) p[(size_t)row * k * cin + (size_t)t * cin + ci] = w.data[((size_t)co * cin + ci) * k + t];
    if (b) pb[row] = b->data[co];
  }
  ConvW c;
  c.ksize = k;
  c.cin = cin;
  c.cout = cout;
  c.dil = dil;
  c.lin.N = cout;
  c.lin.K = k * cin;
  c.lin.w = upload(h, p);
  c.lin.b = bias ? upload(h, pb) : nullptr;
  return c;
}

DecLayerW make_dec_layer(ss_engine* h, const std::string& p, int dim, int ffn, int kdim, bool cross) {
  DecLayerW L;
  L.self_ln = make_ln(h, p + ".self_attn_layer_norm", dim);
  L.q = make_linear(h, p + ".self_attn.q_proj", dim, dim);
  L.k = make_linear(h, p + ".self_attn.k_proj", dim, dim);
  L.v = make_linear(h, p + ".self_attn.v_proj", dim, dim);
  L.qkv = make_fused(h, {p + ".self_attn.q_proj", p + ".self_attn.k_proj", p + ".self_attn.v_proj"}, dim, dim);
  L.out = make_linear(h, p + ".self_attn.out_proj", dim, dim);
  L.has_cross = cross;
  if (cross) {
    L.cross_ln = make_ln(h, p + ".encoder_attn_layer_norm", dim);
    L.cq = make_linear(h, p + ".encoder_attn.q_proj", dim, dim);
    L.ckv = make_fused(h, {p + ".encoder_attn.k_proj", p + ".encoder_attn.v_proj"}, dim, kdim);
    L.cout = make_linear(h, p + ".encoder_attn.out_proj", dim, dim);
  }
  L.final_ln = make_ln(h, p + ".final_layer_norm", dim);
  L.fc1 = make_linear(h, p + ".fc1", ffn, dim);
  L.fc2 = make_linear(h, p + ".fc2", dim, ffn);
  return L;
}

void finalize_impl(ss_engine* h) {
  const ss_config& c = h->cfg;
  const int D = c.enc_dim;
  if (D != c.enc_heads * 64 || c.mt_dim != c.mt_heads * 64 || c.unit_dim != c.unit_heads * 64)
    throw std::runtime_error("attention kernels require head_dim == 64");
  // ---- front-end constants
  {
    const HostTensor& mb = get(h, "__const__.mel_bank");
    expect_shape(mb, "__const__.mel_bank", {80, 257});
    h->mel_bank = upload(h, mb.data);
    {
      std::vector<float> t((size_t)257 * 80);
      for (int m = 0; m < 80; ++m)
        for (int k = 0; k < 257; ++k) t[(size_t)k * 80 + m] = mb.data[(size_t)m * 257 + k];
      h->melT = upload(h, t);
    }
    const HostTensor& w = get(h, "__const__.window");
    expect_shape(w, "__const__.window", {400});
    h->window = upload(h, w.data);
    if (h->host.count("__const__.gcmvn_mean")) {
      h->cmvn_mean = upload(h, get(h, "__const__.gcmvn_mean").data);
      h->cmvn_std = upload(h, get(h, "__const__.gcmvn_std").data);
    }
    if (h->host.count("__const__.resample_3to1")) {
      const HostTensor& r = get(h, "__const__.resample_3to1");
      if (r.numel() < 4 || r.numel() > 64 || (r.numel() - 3) % 2 != 0) throw std::runtime_error("bad __const__.resample_3to1");
      h->resample_h = upload(h, r.data);
      h->resample_taps = (int)r.numel();
      h->resample_width = ((int)r.numel() - 3) / 2;
    }
    int m[3] = {c.pad, c.unk, c.eos};
    h->mask_pad_unk = dev_alloc<int>(h, 3);
    cudaMemcpy(h->mask_pad_unk, m, sizeof(m), cudaMemcpyHostToDevice);
    int m2[2] = {c.pad, c.eos};
    h->mask_pad_eos = dev_alloc<int>(h, 2);
    cudaMemcpy(h->mask_pad_eos, m2, sizeof(m2), cudaMemcpyHostToDevice);
  }
  // ---- subsampler (GLU-interleaved conv-as-GEMM weights)
  {
    ConvW c0 = make_conv(h, "encoder.subsample.conv_layers.0", c.conv_channels, c.feat_dim, c.conv_kernel, 1, true);
    ConvW c1 = make_conv(h, "encoder.subsample.conv_layers.1", 2 * D, c.conv_channels / 2, c.conv_kernel, 1, true);
    h->sub_conv[0] = c0.lin;
    h->sub_conv[1] = c1.lin;
    h->enc_linear = make_linear(h, "encoder.linear", D, D);
  }
  // ---- rel-pos table rows: pe(r) for r = Tpos-1 ... -(Tpos-1) as the reference builds it; we want row index r + Tpos - 1
  const HostTensor& pe = get(h, "__const__.enc_pe");  // [2*Tpos-1][D], row k <-> relative position (Tpos-1-k)
  h->Tpos = c.max_enc_frames;
  expect_shape(pe, "__const__.enc_pe", {2 * (int64_t)h->Tpos - 1, D});
  std::vector<float> pe_flipped(pe.data.size());
  const int P = 2 * h->Tpos - 1;
  for (int k = 0; k < P; ++k) memcpy(&pe_flipped[(size_t)(P - 1 - k) * D], &pe.data[(size_t)k * D], D * sizeof(float));
  float* pe_dev = upload(h, pe_flipped);
  h->enc.resize(c.enc_layers);
  for (int i = 0; i < c.enc_layers; ++i) {
    ConformerLayerW& L = h->enc[i];
    std::string p = "encoder.conformer_layers." + std::to_string(i);
    L.ffn1_ln = make_ln(h, p + ".ffn1.layer_norm", D);
    L.ffn1_w1 = make_linear(h, p + ".ffn1.w_1", c.enc_ffn, D);
    L.ffn1_w2 = make_linear(h, p + ".ffn1.w_2", D, c.enc_ffn);
    L.ffn2_ln = make_ln(h, p + ".ffn2.layer_norm", D);
    L.ffn2_w1 = make_linear(h, p + ".ffn2.w_1", c.enc_ffn, D);
    L.ffn2_w2 = make_linear(h, p + ".ffn2.w_2", D, c.enc_ffn);
    L.attn_ln = make_ln(h, p + ".self_attn_layer_norm", D);
    L.qkv = make_fused(h, {p + ".self_attn.linear_q", p + ".self_attn.linear_k", p + ".self_attn.linear_v"}, D, D);
    L.attn_out = make_linear(h, p + ".self_attn.linear_out", D, D);
    L.pos_u = upload(h, get(h, p + ".self_attn.pos_bias_u").data);
    L.pos_v = upload(h, get(h, p + ".self_attn.pos_bias_v").data);
    // P_l = pe @ linear_pos^T, computed on the device with the same GEMM kernel
    Linear lp = make_linear(h, p + ".self_attn.linear_pos", D, D, false);
    L.pos_proj = dev_alloc<float>(h, (size_t)P * D);
    ConvA a;
    a.x = pe_dev; a.B = 1; a.L_in = P; a.L_rows = P; a.C_in = D; a.ldx = D;
    Epilogue ep;
    ep.out = L.pos_proj; ep.ldo = D;
    gemm_conv(a, lp.w, D, ep, &h->splitk[0], 0);
    L.conv_ln = make_ln(h, p + ".conv_module.layer_norm", D);
    ConvW pw1 = make_conv(h, p + ".conv_module.pointwise_conv1", 2 * D, D, 1, 1, true, false);
    L.pw1 = pw1.lin;
    {
      const HostTensor& dw = get(h, p + ".conv_module.depthwise_conv.weight");
      expect_shape(dw, p + ".conv_module.depthwise_conv.weight", {D, 1, c.dw_kernel});
      std::vector<float> t((size_t)c.dw_kernel * D);
      for (int ch = 0; ch < D; ++ch)
        for (int k = 0; k < c.dw_kernel; ++k) t[(size_t)k * D + ch] = dw.data[(size_t)ch * c.dw_kernel + k];
      L.dw_w = upload(h, t);
      const auto& g = get(h, p + ".conv_module.batch_norm.weight").data;
      const auto& b = get(h, p + ".conv_module.batch_norm.bias").data;
      const auto& rm = get(h, p + ".conv_module.batch_norm.running_mean").data;
      const auto& rv = get(h, p + ".conv_module.batch_norm.running_var").data;
      std::vector<float> sc(D), sh(D);
      for (int ch = 0; ch < D; ++ch) {  // eval-mode BatchNorm1d folded: y = (x - mean) / sqrt(var + eps) * g + b
        float inv = 1.0f / std::sqrt(rv[ch] + 1e-5f);
        sc[ch] = g[ch] * inv;
        sh[ch] = b[ch] - rm[ch] * g[ch] * inv;
      }
      L.bn_scale = upload(h, sc);
      L.bn_shift = upload(h, sh);
    }
    ConvW pw2 = make_conv(h, p + ".conv_module.pointwise_conv2", D, D, 1, 1, false, false);
    L.pw2 = pw2.lin;
    L.final_ln = make_ln(h, p + ".final_layer_norm", D);
  }
  {
    size_t n = (size_t)c.enc_layers * h->Tpos * D;
    h->st_k = dev_alloc<float>(h, n);
    h->st_v = dev_alloc<float>(h, n);
    h->st_glu = dev_alloc<float>(h, n);
    std::vector<PersistLayer> pl(c.enc_layers);
    for (int i = 0; i < c.enc_layers; ++i) {
      const ConformerLayerW& L = h->enc[i];
      PersistLayer& q = pl[i];
      q.ffn1_g = L.ffn1_ln.g; q.ffn1_b = L.ffn1_ln.b; q.ffn1_w1 = L.ffn1_w1.w; q.ffn1_b1 = L.ffn1_w1.b; q.ffn1_w2 = L.ffn1_w2.w; q.ffn1_b2 = L.ffn1_w2.b;
      q.attn_g = L.attn_ln.g; q.attn_b = L.attn_ln.b; q.wqkv = L.qkv.w; q.bqkv = L.qkv.b; q.wo = L.attn_out.w; q.bo = L.attn_out.b;
      q.pos_u = L.pos_u; q.pos_v = L.pos_v; q.pos_proj = L.pos_proj;
      q.conv_g = L.conv_ln.g; q.conv_b = L.conv_ln.b; q.pw1 = L.pw1.w; q.pw1_b = L.pw1.b; q.dw_w = L.dw_w; q.bn_scale = L.bn_scale;
      q.bn_shift = L.bn_shift; q.pw2 = L.pw2.w; q.pw2_b = L.pw2.b;
      q.ffn2_g = L.ffn2_ln.g; q.ffn2_b = L.ffn2_ln.b; q.ffn2_w1 = L.ffn2_w1.w; q.ffn2_b1 = L.ffn2_w1.b; q.ffn2_w2 = L.ffn2_w2.w; q.ffn2_b2 = L.ffn2_w2.b;
      q.fin_g = L.final_ln.g; q.fin_b = L.final_ln.b;
      // W2 transposed [FFN][D]: the fused FFN phases read one coalesced 1 KB row per hidden unit
      for (int which = 0; which < 2; ++which) {
        const HostTensor& w2 = get(h, "encoder.conformer_layers." + std::to_string(&q - pl.data()) + (which ? ".ffn2.w_2.weight" : ".ffn1.w_2.weight"));
        std::vector<float> t((size_t)c.enc_ffn * D);
        for (int n = 0; n < D; ++n)
          for (int u = 0; u < c.enc_ffn; ++u) t[(size_t)u * D + n] = w2.data[(size_t)n * c.enc_ffn + u];
        (which ? q.ffn2_w2t : q.ffn1_w2t) = upload(h, t);
      }
    }
    h->persist_ffn_scratch = dev_alloc<float>(h, (size_t)(c.enc_ffn / 16) * 16 * D);
    h->persist_layers = dev_alloc<PersistLayer>(h, pl.size());
    cudaMemcpy(h->persist_layers, pl.data(), pl.size() * sizeof(PersistLayer), cudaMemcpyHostToDevice);
    h->persist_bar = dev_alloc<unsigned>(h, 64);
    cudaMemset(h->persist_bar, 0, 64 * sizeof(unsigned));
    h->persist_bar_target = 0;
    if (!h->async_err_pinned && cudaHostAlloc((void**)&h->async_err_pinned, sizeof(unsigned), cudaHostAllocDefault) == cudaSuccess)
      *h->async_err_pinned = 0;
  }
  // ---- CTC heads (optional: a UnitY checkpoint has neither; a StreamSpeech one needs both)
  h->has_ctc = h->host.count("source_unigram_decoder.proj.weight") || h->host.count("ctc_target_unigram_decoder.proj.weight");
  if (!h->has_ctc) {
  } else if (c.src_vocab == c.tgt_vocab) {
    // one [2V][D] matrix: both heads of a policy() call are ONE GEMM (ss_ctc_greedy_pair); the single heads are views of it
    h->ctc_pair = make_fused(h, {"source_unigram_decoder.proj", "ctc_target_unigram_decoder.proj"}, c.src_vocab, D);
    h->ctc_head[0] = h->ctc_pair;
    h->ctc_head[0].N = c.src_vocab;
    h->ctc_head[1] = h->ctc_pair;
    h->ctc_head[1].N = c.tgt_vocab;
    h->ctc_head[1].w = h->ctc_pair.w + (size_t)c.src_vocab * D;
    h->ctc_head[1].b = h->ctc_pair.b + c.src_vocab;
  } else {
    h->ctc_head[0] = make_linear(h, "source_unigram_decoder.proj", c.src_vocab, D);
    h->ctc_head[1] = make_linear(h, "ctc_target_unigram_decoder.proj", c.tgt_vocab, D);
  }
  h->ctc_ticket = dev_alloc<unsigned>(h, 8);
  cudaMemset(h->ctc_ticket, 0, 8 * sizeof(unsigned));
  // ---- MT decoder
  {
    const HostTensor& e = get(h, "target_unigram_decoder.embed_tokens.weight");
    expect_shape(e, "target_unigram_decoder.embed_tokens.weight", {c.tgt_vocab, c.mt_dim});
    h->mt_emb = upload(h, e.data);
    const HostTensor& pt = get(h, "__const__.mt_pos_table");
    if (pt.shape.size() != 2 || pt.shape[1] != c.mt_dim || pt.shape[0] < (int64_t)c.max_mt_positions + c.pad + 2)
      throw std::runtime_error("bad __const__.mt_pos_table (needs max_mt_positions + pad + 2 rows of mt_dim)");
    h->mt_pos_rows = (int)pt.shape[0];
    h->mt_pos = upload(h, pt.data);
    for (int i = 0; i < c.mt_layers; ++i)
      h->mt.push_back(make_dec_layer(h, "target_unigram_decoder.layers." + std::to_string(i), c.mt_dim, c.mt_ffn, D, true));
    h->mt_ln = make_ln(h, "target_unigram_decoder.layer_norm", c.mt_dim);
    size_t cache = (size_t)c.mt_layers * c.max_mt_positions * c.mt_dim;
    h->mt_self_k = dev_alloc<float>(h, cache);
    h->mt_self_v = dev_alloc<float>(h, cache);
    h->mt_tok_dev = dev_alloc<int64_t>(h, c.max_mt_positions + 8);
    h->mt_part = dev_alloc<float>(h, (size_t)9 * c.mt_dim);
    cudaMallocHost((void**)&h->mt_next_pinned, (size_t)(c.max_mt_positions + 8) * sizeof(int64_t));
    std::vector<MtLayerP> ml(c.mt_layers);
    for (int i = 0; i < c.mt_layers; ++i) {
      const DecLayerW& L = h->mt[i];
      MtLayerP& q = ml[i];
      q.self_g = L.self_ln.g; q.self_b = L.self_ln.b; q.wqkv = L.qkv.w; q.bqkv = L.qkv.b; q.wo = L.out.w; q.bo = L.out.b;
      q.cross_g = L.cross_ln.g; q.cross_b = L.cross_ln.b; q.wcq = L.cq.w; q.bcq = L.cq.b; q.wco = L.cout.w; q.bco = L.cout.b;
      q.fin_g = L.final_ln.g; q.fin_b = L.final_ln.b; q.w1 = L.fc1.w; q.b1 = L.fc1.b; q.w2 = L.fc2.w; q.b2 = L.fc2.b;
    }
    h->mt_persist_layers = dev_alloc<MtLayerP>(h, ml.size());
    cudaMemcpy(h->mt_persist_layers, ml.data(), ml.size() * sizeof(MtLayerP), cudaMemcpyHostToDevice);
  }
  // ---- T2U encoder + unit decoder
  for (int i = 0; i < c.t2u_layers; ++i)
    h->t2u.push_back(make_dec_layer(h, "synthesizer_encoder.layers." + std::to_string(i), c.unit_dim, c.unit_ffn, c.unit_dim, false));
  h->t2u_ln = make_ln(h, "synthesizer_encoder.layer_norm", c.unit_dim);
  for (int i = 0; i < c.unit_layers; ++i)
    h->unit.push_back(make_dec_layer(h, "decoder.layers." + std::to_string(i), c.unit_dim, c.unit_ffn, c.unit_dim, true));
  h->unit_ln = make_ln(h, "decoder.layer_norm", c.unit_dim);
  {
    const HostTensor& e = get(h, "decoder.embed_tokens.weight");
    expect_shape(e, "decoder.embed_tokens.weight", {c.unit_vocab, c.unit_dim});
    h->unit_emb = upload(h, e.data);
    const HostTensor& pr = get(h, "__const__.unit_pos_row");
    expect_shape(pr, "__const__.unit_pos_row", {c.unit_dim});
    h->unit_pos_row = upload(h, pr.data);
    // the output projection is the embedding (share_decoder_input_output_embed): a stored copy must be that tensor
    auto op = h->host.find("decoder.output_projection.weight");
    if (op != h->host.end() && (op->second.shape != e.shape || op->second.data != e.data))
      throw std::runtime_error("decoder.output_projection.weight differs from decoder.embed_tokens.weight: the unit decoder's output "
                               "projection must be tied to its embedding");
  }
  // ---- UnitY: the autoregressive unit decoder searched on the batched decoder kernel (ss_unit_search_batch)
  if (h->host.count("__const__.unit_pos_table")) {
    if (!mt_decode_persistent_supported(c.unit_dim, c.unit_ffn, c.unit_heads, c.unit_vocab, 1, 1))
      throw std::runtime_error("unit decoder of " + std::to_string(c.unit_dim) + " / " + std::to_string(c.unit_ffn) + " / " +
                               std::to_string(c.unit_heads) + " (dim / ffn / heads): the autoregressive unit search's kernel takes 512 / 2048 / 8");
    const HostTensor& pt = get(h, "__const__.unit_pos_table");
    if (pt.shape.size() != 2 || pt.shape[1] != c.unit_dim || pt.shape[0] < (int64_t)c.pad + 3)
      throw std::runtime_error("bad __const__.unit_pos_table (needs max_target_positions + pad + 1 rows of unit_dim)");
    h->unit_pos_rows = (int)pt.shape[0];
    h->unit_pos = upload(h, pt.data);
    std::vector<MtLayerP> ul(c.unit_layers);
    for (int i = 0; i < c.unit_layers; ++i) {
      const DecLayerW& L = h->unit[i];
      MtLayerP& q = ul[i];
      q.self_g = L.self_ln.g; q.self_b = L.self_ln.b; q.wqkv = L.qkv.w; q.bqkv = L.qkv.b; q.wo = L.out.w; q.bo = L.out.b;
      q.cross_g = L.cross_ln.g; q.cross_b = L.cross_ln.b; q.wcq = L.cq.w; q.bcq = L.cq.b; q.wco = L.cout.w; q.bco = L.cout.b;
      q.fin_g = L.final_ln.g; q.fin_b = L.final_ln.b; q.w1 = L.fc1.w; q.b1 = L.fc1.b; q.w2 = L.fc2.w; q.b2 = L.fc2.b;
    }
    h->unit_persist_layers = dev_alloc<MtLayerP>(h, ul.size());
    cudaMemcpy(h->unit_persist_layers, ul.data(), ul.size() * sizeof(MtLayerP), cudaMemcpyHostToDevice);
  }
  // ---- vocoder (optional: the ASR / S2TT agents do not load one)
  h->has_vocoder = h->host.count("vocoder.dict.weight") > 0;
  if (h->has_vocoder) {
    const int E = c.voc_embedding_dim;
    const HostTensor& dict = get(h, "vocoder.dict.weight");
    expect_shape(dict, "vocoder.dict.weight", {c.voc_num_embeddings, E});
    h->voc_dict = upload(h, dict.data);
    h->dur_conv1 = make_conv(h, "vocoder.dur_predictor.conv1.0", c.voc_dur_hidden, E, c.voc_dur_kernel, 1, false);
    h->dur_ln1 = make_ln(h, "vocoder.dur_predictor.ln1", c.voc_dur_hidden);
    h->dur_conv2 = make_conv(h, "vocoder.dur_predictor.conv2.0", c.voc_dur_hidden, c.voc_dur_hidden, c.voc_dur_kernel, 1, false);
    h->dur_ln2 = make_ln(h, "vocoder.dur_predictor.ln2", c.voc_dur_hidden);
    h->dur_proj = make_linear(h, "vocoder.dur_predictor.proj", 1, c.voc_dur_hidden);
    h->conv_pre = make_conv(h, "vocoder.conv_pre", c.voc_init_channels, c.voc_in_dim, 7, 1, false);
    int ch = c.voc_init_channels;
    h->hop = 1;
    h->rb1.resize(c.voc_n_ups);
    h->rb2.resize(c.voc_n_ups);
    for (int i = 0; i < c.voc_n_ups; ++i) {
      UpsampleW U;
      U.u = c.voc_up_rates[i];
      U.k = c.voc_up_kernels[i];
      U.pad = (U.k - U.u) / 2;
      U.cin = ch;
      U.cout = ch / 2;
      if ((U.k - U.u) % 2 != 0 || U.pad >= U.u + U.k) throw std::runtime_error("unsupported upsample geometry");
      h->hop *= U.u;
      const std::string p = "vocoder.ups." + std::to_string(i);
      const HostTensor& w = get(h, p + ".weight");  // ConvTranspose1d: [Cin][Cout][k]
      expect_shape(w, p + ".weight", {U.cin, U.cout, U.k});
      U.bias = upload(h, get(h, p + ".bias").data);
      // polyphase split: out[q*u + phi - pad] = sum_j x[q - j] * W[:, :, phi + j*u]
      for (int phi = 0; phi < U.u; ++phi) {
        int J = (U.k - phi + U.u - 1) / U.u;
        std::vector<float> pw((size_t)U.cout * J * U.cin);
        for (int co = 0; co < U.cout; ++co)
          for (int jp = 0; jp < J; ++jp) {        // tap jp reads input q - (J-1) + jp  <->  j = J-1-jp
            int kk = phi + (J - 1 - jp) * U.u;
            for (int ci = 0; ci < U.cin; ++ci)
              pw[((size_t)co * J + jp) * U.cin + ci] = w.data[((size_t)ci * U.cout + co) * U.k + kk];
          }
        Linear l;
        l.N = U.cout;
        l.K = J * U.cin;
        l.w = upload(h, pw);
        l.b = U.bias;
        U.phase_w.push_back(l);
        U.phase_J.push_back(J);
        U.phase_q0.push_back(phi < U.pad ? (U.pad - phi + U.u - 1) / U.u : 0);
      }
      h->ups.push_back(U);
      ch = U.cout;
      h->rb1[i].resize(c.voc_n_rb);
      h->rb2[i].resize(c.voc_n_rb);
      for (int j = 0; j < c.voc_n_rb; ++j) {
        int rb = i * c.voc_n_rb + j;
        int rk = c.voc_rb_kernels[j];
        for (int m = 0; m < c.voc_rb_ndil; ++m) {
          std::string q = "vocoder.resblocks." + std::to_string(rb);
          h->rb1[i][j].push_back(make_conv(h, q + ".convs1." + std::to_string(m), ch, ch, rk, c.voc_rb_dils[j][m], false));
          h->rb2[i][j].push_back(make_conv(h, q + ".convs2." + std::to_string(m), ch, ch, rk, 1, false));
        }
      }
    }
    {
      const HostTensor& w = get(h, "vocoder.conv_post.weight");  // [1][ch][7]
      expect_shape(w, "vocoder.conv_post.weight", {1, ch, 7});
      std::vector<float> t((size_t)7 * ch);
      for (int ci = 0; ci < ch; ++ci)
        for (int k = 0; k < 7; ++k) t[(size_t)k * ch + ci] = w.data[(size_t)ci * 7 + k];
      h->conv_post_w = upload(h, t);
      h->conv_post_b = get(h, "vocoder.conv_post.bias").data[0];
      h->conv_post_c = ch;
      h->conv_post_k = 7;
    }
    // receptive field of the generator in input frames (left side), over-approximated
    int maxk = 0, sumd = 0;
    for (int j = 0; j < c.voc_n_rb; ++j) {
      int s = 0;
      for (int m = 0; m < c.voc_rb_ndil; ++m) s += c.voc_rb_dils[j][m] + 1;
      int r = (c.voc_rb_kernels[j] - 1) / 2 * s;
      if (r > maxk) maxk = r;
      (void)sumd;
    }
    int r = 3;
    for (int i = c.voc_n_ups - 1; i >= 0; --i) {
      r += maxk;
      r = (r + c.voc_up_kernels[i] + c.voc_up_rates[i] - 1) / c.voc_up_rates[i] + 1;
    }
    h->receptive_field = r + 3;
  }
  if (cudaDeviceSynchronize() != cudaSuccess) throw std::runtime_error(std::string("CUDA error during finalize: ") + cudaGetErrorString(cudaGetLastError()));
  h->host.clear();
  h->finalized = true;
}

}  // namespace

// what ss_last_error(NULL) returns: the reason of this thread's last refused ss_create (which leaves no handle to ask)
static thread_local std::string g_create_err = "null handle";

extern "C" {

const char* ss_version(void) { return "streamspeech_b200 0.1 (sm_90a)"; }

int ss_create(ss_engine** out, int device, const ss_config* cfg) {
  if (!out || !cfg) return SS_ERR_INVALID;
  *out = nullptr;
  g_create_err = "null handle";
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess || n <= 0 || device >= n) return SS_ERR_CUDA;
  if (cudaSetDevice(device) != cudaSuccess) return SS_ERR_CUDA;
  if (cfg->max_mt_positions < 3 || cfg->max_mt_positions > SS_MAX_MT_POSITIONS) {  // (max_len >= 1 needs max_len + 2 entries)
    g_create_err = "ss_create: max_mt_positions = " + std::to_string(cfg->max_mt_positions) + " is outside [3, " + std::to_string(SS_MAX_MT_POSITIONS) + "]";
    return SS_ERR_INVALID;
  }
  ss_engine* h = new ss_engine();
  h->device = device;
  h->cfg = *cfg;
  if (h->cfg.voc_n_ups > SS_MAX_UPS || h->cfg.voc_n_rb > SS_MAX_RB || h->cfg.voc_rb_ndil > SS_MAX_DIL) {
    delete h;
    return SS_ERR_INVALID;
  }
  h->umma2_cache = new ss::Umma2Cache();
  *out = h;
  return SS_OK;
}

int ss_destroy(ss_engine* h) {
  if (!h) return SS_OK;
  cudaSetDevice(h->device);
  cudaDeviceSynchronize();
  for (void* p : h->dev_allocs) cudaFree(p);
  ss::umma2_cache_destroy(h->umma2_cache);
  for (float* p : h->splitk)
    if (p) cudaFree(p);
  if (h->ws.base) cudaFree(h->ws.base);
  if (h->mt_cross_kv) cudaFree(h->mt_cross_kv);
  if (h->mtb_self_kv) cudaFree(h->mtb_self_kv);
  if (h->mtb_self_kv2) cudaFree(h->mtb_self_kv2);
  if (h->mtb_cross_kv) cudaFree(h->mtb_cross_kv);
  if (h->mtb_tok_pinned) cudaFreeHost(h->mtb_tok_pinned);
  if (h->mt_next_pinned) cudaFreeHost(h->mt_next_pinned);
  if (h->async_err_pinned) cudaFreeHost(h->async_err_pinned);
  if (h->pool.desc_pinned) cudaFreeHost(h->pool.desc_pinned);
  if (h->pool.desc_pinned2) cudaFreeHost(h->pool.desc_pinned2);
  for (auto& e : h->pool.resample_events) {
    cudaEventDestroy(e.e0);
    cudaEventDestroy(e.e1);
  }
  if (h->voc_unit_emb) cudaFree(h->voc_unit_emb);
  if (h->voc_cumsum) cudaFree(h->voc_cumsum);
  if (h->lengths_dev) cudaFree(h->lengths_dev);
  for (int i = 0; i < 2; ++i) {
    if (h->aux_stream[i]) cudaStreamDestroy(h->aux_stream[i]);
    if (h->join_event[i]) cudaEventDestroy(h->join_event[i]);
  }
  if (h->fork_event) cudaEventDestroy(h->fork_event);
  delete h;
  return SS_OK;
}

const char* ss_last_error(const ss_engine* h) { return h ? h->err.c_str() : g_create_err.c_str(); }

int ss_load_tensor(ss_engine* h, const char* key, const float* data_host, int ndim, const int64_t* shape) {
  if (!h || !key || !data_host || ndim < 0 || ndim > 8) return SS_ERR_INVALID;
  if (h->finalized) return h->fail(SS_ERR_STATE, "ss_load_tensor after ss_finalize");
  HostTensor t;
  int64_t n = 1;
  for (int i = 0; i < ndim; ++i) {
    t.shape.push_back(shape[i]);
    n *= shape[i];
  }
  t.data.assign(data_host, data_host + n);
  h->host[key] = std::move(t);
  return SS_OK;
}

int ss_finalize(ss_engine* h) {
  if (!h) return SS_ERR_INVALID;
  if (h->finalized) return SS_OK;
  cudaSetDevice(h->device);
  try {
    finalize_impl(h);
  } catch (const MissingKey& e) {
    return h->fail(SS_ERR_MISSING, std::string("missing state-dict key: ") + e.what());
  } catch (const std::exception& e) {
    return h->fail(SS_ERR_INVALID, e.what());
  }
  return SS_OK;
}

int ss_set_chunk(ss_engine* h, int attn_chunk, int conv_chunk) {
  if (!h || attn_chunk < 0 || conv_chunk < 0) return SS_ERR_INVALID;
  if (conv_chunk % 2 != 0) return h->fail(SS_ERR_INVALID, "conv chunk must be even (stride-2 subsampler)");
  h->attn_chunk = attn_chunk;
  h->conv_chunk = conv_chunk;
  return SS_OK;
}

int ss_vocoder_hop(const ss_engine* h) { return h ? h->hop : 0; }
int ss_vocoder_receptive_field(const ss_engine* h) { return h ? h->receptive_field : 0; }

}  // extern "C"
