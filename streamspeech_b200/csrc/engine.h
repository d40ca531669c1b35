// Engine state behind the C-ABI handle: host copies of the loaded tensors, repacked device weights,
// a bump-allocated workspace and the per-call scratch of the decoders.
#pragma once
#include <cuda_runtime.h>

#include <map>
#include <utility>
#include <string>
#include <vector>

#include "../../include/streamspeech_b200.h"
#include "kernels.h"
#include "kernels_persist.h"
#include "kernels_multistream.h"

namespace ss {

struct HostTensor {
  std::vector<float> data;
  std::vector<int64_t> shape;
  int64_t numel() const {
    int64_t n = 1;
    for (auto s : shape) n *= s;
    return n;
  }
};

struct Linear {
  float* w = nullptr;  // [N][K]
  float* b = nullptr;  // [N] or null
  int N = 0, K = 0;
};
struct LNorm {
  float* g = nullptr;
  float* b = nullptr;
  int C = 0;
};

struct ConformerLayerW {
  LNorm ffn1_ln, ffn2_ln, attn_ln, conv_ln, final_ln;
  Linear ffn1_w1, ffn1_w2, ffn2_w1, ffn2_w2;
  Linear qkv, attn_out;
  float* pos_u = nullptr;
  float* pos_v = nullptr;
  float* pos_proj = nullptr;  // [2*Tpos-1][D]: linear_pos(pe(r)), row r + Tpos - 1
  Linear pw1;                 // GLU-interleaved rows
  float* dw_w = nullptr;      // [k][C]
  float* bn_scale = nullptr;
  float* bn_shift = nullptr;
  Linear pw2;
};

struct DecLayerW {  // transformer layer (self-attn [+ cross-attn] + FFN), pre-LN
  LNorm self_ln, cross_ln, final_ln;
  Linear q, k, v, qkv, out;      // self attention (qkv = fused rows q|k|v)
  Linear cq, ckv, cout;          // cross attention (ckv = fused k|v)
  Linear fc1, fc2;
  bool has_cross = false;
};

struct ConvW {  // conv-as-GEMM weight [Cout][ksize*Cin]
  Linear lin;
  int ksize = 1, cin = 0, cout = 0, dil = 1;
};

struct UpsampleW {
  int u = 1, k = 1, pad = 0, cin = 0, cout = 0;
  std::vector<Linear> phase_w;  // per output phase: [Cout][J*Cin]
  std::vector<int> phase_J, phase_q0;
  float* bias = nullptr;
};

struct Arena {
  char* base = nullptr;
  size_t cap = 0, off = 0;
  float* f32(size_t n) { return (float*)raw(n * 4); }
  void* raw(size_t bytes);
  void reset() { off = 0; }
  bool ensure(size_t bytes);  // (re)allocate when empty; must be called when off == 0
};

}  // namespace ss

struct ss_engine {
  int device = 0;
  ss_config cfg{};
  std::string err;
  bool finalized = false;
  int attn_chunk = 8, conv_chunk = 8;
  int umma_vocoder = 0;   // 0 = fp32 CUDA-core convs, 2 / 3 = wgmma with that many bf16 pieces per operand
  int umma_linear = 0;    // same for large-M linears (unit decoder, T2U, MT prefill, full-prefix encoder)
                          // 12 / 13: second-generation kernel (kernels_umma2.cu) with 2 / 3 pieces
  int unit_grouped = 1;         // unit decoder layer 1: self-attention over the S distinct rows instead of the 25*S copies
  int umma_min_rows = 128;      // GEMMs with fewer rows stay on the fp32 CUDA-core kernels
  int umma_min_channels = 16;   // convs with fewer input channels stay on the fp32 CUDA-core kernel
  ss::Umma2Cache* umma2_cache = nullptr;  // packed bf16-split weights of kernels_umma2.cu (created by ss_create)
  // split-K scratch regions of the GEMMs (ss::splitk_workspace, allocated by the first split into each): region 0 serves every GEMM
  // on the caller's stream, regions 1 / 2 the vocoder's auxiliary streams
  float* splitk[3] = {nullptr, nullptr, nullptr};
  int vocoder_streams = 1;     // 1: the parallel resblocks of a vocoder stage run on three streams, 0: one stream
  cudaStream_t aux_stream[2] = {nullptr, nullptr};
  cudaEvent_t fork_event = nullptr, join_event[2] = {nullptr, nullptr};
  // whole generator as one persistent kernel (kernels_umma2.cu vocoder_fused): -1 = when the frame count is at most
  // voc_fused_max_frames, 0 = never (multi-launch path), 1 = whenever the shapes allow it
  int vocoder_fused = -1;
  // job / phase templates of the fused kernel per (frame capacity, arena): the packed-weight pointers of each tile width are filled
  // in by the first call that uses them
  std::map<std::pair<int, uintptr_t>, ss::VocFusedParams> voc_fused;
  ss::VocFusedParams voc_call{};  // the templates with one call's sequences filled in
  float* persist_ffn_scratch = nullptr;  // [enc_ffn / 16][16][enc_dim] partial sums of the fused FFN phases
  float* cl_blobs = nullptr;             // [enc_layers][16][624][256] weight blobs of the cluster encoder kernel (allocated when the option is set)
  int cluster_cooperative = 1;           // cooperative launch attribute of the cluster kernel (0 only under a serialising profiler)
  long long cl_steps = 0;                // steps the cluster kernel has taken (ss_debug_copy "cluster_steps")
  int persistent_encoder_cluster = 0;    // kernels_persist_cl.cu instead of kernels_persist.cu for steps with <= 16 active rows
  int persistent_ffn_fused = 1;          // fused FFN phases in the persistent encoder kernel (0: separate W1 / W2 phases)
  int fbank_tma = 1;           // fbank frames staged by cp.async.bulk + transposed mel bank (0: plain loads, [80][257] mel bank)
  int persistent_encoder = 1;  // streaming encoder step as ONE cooperative kernel (kernels_persist.cu) when the shape fits
  std::map<std::string, ss::HostTensor> host;  // loaded tensors by key
  std::vector<void*> dev_allocs;

  // ---- packed weights
  ss::Linear sub_conv[2];
  ss::Linear enc_linear;
  std::vector<ss::ConformerLayerW> enc;
  int Tpos = 0;
  bool has_ctc = true;              // the CTC heads were loaded (StreamSpeech); a UnitY checkpoint has none
  ss::Linear ctc_head[2];
  ss::Linear ctc_pair;              // both heads as one [2V][D] linear (N == 0 when the vocabularies differ)
  unsigned* ctc_ticket = nullptr;   // "last block done" ticket of ctc_argmax_collapse_pair_kernel
  float* mt_emb = nullptr;
  float* mt_pos = nullptr;  // sinusoid table [max_mt_positions + pad + 2][mt_dim]
  int mt_pos_rows = 0;
  std::vector<ss::DecLayerW> mt;
  ss::LNorm mt_ln;
  std::vector<ss::DecLayerW> t2u;
  ss::LNorm t2u_ln;
  std::vector<ss::DecLayerW> unit;
  ss::LNorm unit_ln;
  float* unit_emb = nullptr;
  float* unit_pos_row = nullptr;  // sinusoid row pad+1 (N1 quirk)
  // UnitY's autoregressive unit decoder (ss_unit_search_batch), loaded when "__const__.unit_pos_table" is
  float* unit_pos = nullptr;                   // sinusoid table [max_target_positions + pad + 1][unit_dim]
  int unit_pos_rows = 0;
  ss::MtLayerP* unit_persist_layers = nullptr;  // [unit_layers] device pointer table for the batched decoder kernel
  float* mel_bank = nullptr;
  float* melT = nullptr;            // mel bank transposed [257][80] (TMA-staged fbank kernels)
  float* window = nullptr;
  float* cmvn_mean = nullptr;
  float* cmvn_std = nullptr;
  float* resample_h = nullptr;      // 48 kHz -> 16 kHz decimation filter ("__const__.resample_3to1"), taps / half width below
  int resample_taps = 0, resample_width = 0;
  int* mask_pad_unk = nullptr;      // device [3] = {pad, unk, eos}
  int* mask_pad_eos = nullptr;      // device [2] = {pad, eos}
  // vocoder
  bool has_vocoder = false;
  float* voc_dict = nullptr;
  ss::ConvW dur_conv1, dur_conv2;
  ss::LNorm dur_ln1, dur_ln2;
  ss::Linear dur_proj;
  ss::ConvW conv_pre;
  std::vector<ss::UpsampleW> ups;
  std::vector<std::vector<std::vector<ss::ConvW>>> rb1, rb2;  // [stage][resblock][dil idx]
  float* conv_post_w = nullptr;  // [k][C]
  float conv_post_b = 0.f;
  int conv_post_k = 7, conv_post_c = 0;
  int hop = 1, receptive_field = 0;

  // ---- workspaces
  ss::Arena ws;        // per-call scratch
  // MT decoder per-call caches
  float* mt_self_k = nullptr;  // [layers][max_pos][mt_dim]
  float* mt_self_v = nullptr;
  float* mt_cross_kv = nullptr;  // [layers][Tcap][2*mt_dim]
  int mt_cross_cap = 0;
  int mt_cross_final = 0;            // rows of mt_cross_kv that were projected from final encoder rows (ss_mt_stable_rows)
  int mt_stable_hint = 0;            // hint for the next MT call, consumed by it
  const float* mt_cross_enc = nullptr;  // encoder buffer those rows came from
  // incremental-state decoding across calls (ss_mt_greedy_incremental: the S2TT / ASR agents' use_incremental_states=True)
  int mt_inc_self_len = 0;           // entries in the self-attention cache (can exceed the hypothesis length: call boundaries
                                     // feed the last prefix token again, speech_to_text.s2tt agent + sequence_generator.py:338-346)
  int mt_inc_cross_rows = 0;         // encoder rows whose cross K / V were appended (never refreshed, transformer_layer.py:492-505)
  bool mt_inc_overwritten = false;   // ss_mt_greedy / ss_mt_features (mt_begin) wrote over a non-empty incremental state: refused until reset
  int64_t* mt_tok_dev = nullptr;  // [max_pos]
  int64_t* mt_next_pinned = nullptr;
  // vocoder: the unit sequences of the last ss_vocoder_durations_ragged call, cached for ss_vocoder_generate_ragged
  float* voc_unit_emb = nullptr;  // [voc_ucap][emb]: sequence s at rows u0 .. u0 + U - 1
  int* voc_cumsum = nullptr;      // [voc_ccap]: sequence s's U + 1 frame offsets at c0 (packed in sequence order)
  int voc_ucap = 0, voc_ccap = 0;
  struct VocSeq { int u0, U, c0; };
  std::vector<VocSeq> voc_seqs;
  // streaming encoder state (one utterance per handle)
  int st_T_final = 0;
  float* st_k = nullptr;    // [enc_layers][Tpos][enc_dim]
  float* st_v = nullptr;
  float* st_glu = nullptr;  // conv-module GLU outputs (depthwise-conv inputs)
  unsigned long long* persist_ts = nullptr;    // [4096] phase timestamps when option persistent_profile is set
  int persistent_profile = 0;
  int persistent_time = 0;           // record CUDA events around the persistent encoder kernel (bench roofline)
  struct TimedLaunch { cudaEvent_t e0, e1; double bytes; };
  std::vector<TimedLaunch> time_events;
  std::vector<TimedLaunch> mt_time_events;  // the single-token MT kernel's launches (bytes field = steps executed)
  unsigned* persist_bar = nullptr;   // arrival counter of the persistent kernels' grid barrier (allocated by ss_finalize)
  unsigned persist_bar_target = 0;
  unsigned* async_err_pinned = nullptr;  // host copy of persist_bar[SS_BAR_ERR_WORD] (read back at synchronisation points)
  ss::MtLayerP* mt_persist_layers = nullptr;   // [mt_layers] device pointer table for kernels_persist_mt.cu
  int persistent_mt = 1;                       // single-token MT decode steps as one cooperative kernel per burst
  float* mt_part = nullptr;                    // [9][mt_dim] scratch of that kernel (per-head partials + FFN delta)
  int persistent_mt_prefix = 1;                // ... and the forced-prefix pass (M <= 64 rows) as one cooperative kernel
  // batched greedy search (ss_mt_greedy_batch): caches of its own, so that a streaming agent's MT state on the handle survives it
  float* mtb_self_kv = nullptr;                // K then V: 2 x [max(mt_layers, unit_layers)][MT_BATCH_MAX_ROWS][mtb_tok_ld][mt_dim]
  float* mtb_self_kv2 = nullptr;               // the beam search's second buffer of the same shape (ss_mt_beam_batch)
  int mtb_tok_ld = 0;
  float* mtb_cross_kv = nullptr;               // [max(mt_layers, unit_layers)][MT_BATCH_MAX_ROWS][mtb_cross_cap][2 * mt_dim]
  int mtb_cross_cap = 0;
  int64_t* mtb_tok_pinned = nullptr;           // [MT_BATCH_MAX_ROWS][16] tokens of one burst
  int mt_batch_min_rows = 2;                   // groups with fewer rows decode per sample on the single-token kernel (faster at B = 1)
  ss::PersistLayer* persist_layers = nullptr;  // [enc_layers] device copy of the per-layer pointer table
  int* lengths_dev = nullptr;     // [Bcap]
  int lengths_cap = 0;

  // ---- multi-stream pool (engine_pool.inc): per-slot streaming state at fixed strides
  struct StreamPool {
    int n_slots = 0, Tcap = 0, Fcap = 0;
    int rate = 16000;                                  // source sample rate: 16000, or 48000 (resampled per slot inside ss_pool_step)
    int64_t audio_cap = 0, audio48_cap = 0;
    float *audio = nullptr, *feats = nullptr, *k = nullptr, *v = nullptr, *glu = nullptr, *enc_out = nullptr, *melT = nullptr;
    float* audio48 = nullptr;                          // 48 kHz pools: [slot][audio48_cap] pushed samples; `audio` holds their 16 kHz signal
    int64_t* ctc_am = nullptr;                         // [slot][2][Tcap]
    ss::MsStream *desc_dev = nullptr, *desc_pinned = nullptr, *desc_dev2 = nullptr, *desc_pinned2 = nullptr;
    std::vector<int> T_final, n_feat;
    std::vector<int64_t> n_audio;                      // 16 kHz samples in `audio` (the fbank's input)
    std::vector<int64_t> n48;                          // 48 kHz pools: samples in `audio48`
    std::vector<char> finished;                        // ss_pool_finish: the slot's source is closed
    std::vector<int> attn_chunk, conv_chunk;           // ss_pool_set_chunk: the slot's own chunk sizes (0, 0 = the handle's ss_set_chunk)
    std::vector<TimedLaunch> resample_events;          // option persistent_time: CUDA events around ms_resample_3to1 (bytes = 16 per output)
    std::vector<int> T_rows;                           // encoder rows of the slot after its last step (0: none yet)
    // ss_pool_mt_greedy: cross-attention K / V of every slot [slot][mt_layers][Tcap][2 * mt_dim] (allocated by its first call); rows
    // [0, mt_cross_rows[slot]) were projected from final encoder rows and are not projected again until ss_pool_reset
    float* mt_cross = nullptr;
    std::vector<int> mt_cross_rows;
    // ss_pool_mt_greedy_incremental: the reference's incremental MT decoder state per slot, as the handle keeps it for one stream
    // (mt_inc_self_len / mt_inc_cross_rows).  Self-attention K then V, each [slot][mt_layers][max_mt_positions][mt_dim] (allocated
    // by its first call): a slot's block is MtDecodeParams' self_k / self_v, and its block of mt_cross is cross_kv with cross_cap = Tcap.
    float* mt_self_kv = nullptr;
    std::vector<int> mt_inc_self_len, mt_inc_cross_rows;
    // which search owns the slot's block of mt_cross since its last reset: ss_pool_mt_greedy re-projects rows at or above T_final,
    // the incremental search keeps every row it projected, so a slot serves one of them until ss_pool_reset
    enum MtOwner : char { kMtNone, kMtGreedy, kMtIncremental };
    std::vector<char> mt_owner;
  } pool;

  int fail(int code, const std::string& msg) {
    err = msg;
    return code;
  }
};
