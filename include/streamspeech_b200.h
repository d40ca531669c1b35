/* C-ABI of libstreamspeech_b200.so — the drop-in boundary under the SimulEval agent / fairseq model surface.
 *
 * The reference (ictnlp/StreamSpeech) has no FFI: its hot path is Python objects calling PyTorch
 * (SURVEY.md §8b).  Each entry point below replaces one reference call site; the citation names the
 * reference function whose arithmetic it reproduces (paths relative to the reference tree).
 *
 * Conventions
 *  - every function returns 0 on success, a negative ss_status otherwise; nothing throws across the ABI;
 *    ss_last_error(h) returns a message for the last failure on that handle;
 *  - pointers named *_dev are CUDA device pointers on the handle's device, *_host are host pointers;
 *  - the caller allocates all inputs/outputs (torch tensors -> data_ptr()); the library owns weights,
 *    workspaces and per-stream caches only;
 *  - `stream` is a cudaStream_t (as void*).  Work is enqueued on it; functions documented as
 *    "enqueue only" never synchronise, the others synchronise that stream where stated;
 *  - one handle may be used from one host thread at a time; distinct handles share no device state (weights, caches,
 *    workspaces, split-K scratch, barrier counters, options are per handle).  Process-wide are only the launch counter
 *    (ss_launch_count) and the per-device kernel attribute cache.
 */
#ifndef STREAMSPEECH_B200_H_
#define STREAMSPEECH_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct ss_engine ss_engine;

enum ss_status {
  SS_OK = 0,
  SS_ERR_INVALID = -1,   /* bad argument / shape */
  SS_ERR_MISSING = -2,   /* a required state-dict key was not loaded */
  SS_ERR_CUDA = -3,      /* CUDA runtime error */
  SS_ERR_STATE = -4,     /* call order (e.g. run before finalize) */
  SS_ERR_CAPACITY = -5   /* sequence longer than the configured maximum */
};

#define SS_MAX_UPS 8
#define SS_MAX_RB 4
#define SS_MAX_DIL 4

/* Model dimensions: fairseq cfg of the checkpoint + vocoder config.json
 * (researches/ctc_unity/models/streamspeech_model.py:418-430, agent/tts/codehifigan.py:9-33). */
typedef struct ss_config {
  int32_t feat_dim, enc_dim, enc_ffn, enc_heads, enc_layers, dw_kernel, conv_channels, conv_kernel;
  int32_t src_vocab, tgt_vocab;
  int32_t mt_dim, mt_ffn, mt_heads, mt_layers;
  int32_t t2u_layers, unit_dim, unit_ffn, unit_heads, unit_layers, unit_vocab, ctc_upsample_rate;
  int32_t bos, pad, eos, unk, uni_encoder;
  int32_t max_enc_frames;   /* longest encoder sequence (40 ms frames) the rel-pos tables cover */
  int32_t max_mt_positions; /* entries of every MT self-attention cache, 3 .. SS_MAX_MT_POSITIONS (see below) */
  /* CodeHiFiGAN */
  int32_t voc_n_ups, voc_up_rates[SS_MAX_UPS], voc_up_kernels[SS_MAX_UPS], voc_init_channels;
  int32_t voc_n_rb, voc_rb_kernels[SS_MAX_RB], voc_rb_ndil, voc_rb_dils[SS_MAX_RB][SS_MAX_DIL];
  int32_t voc_num_embeddings, voc_embedding_dim, voc_in_dim, voc_dur_hidden, voc_dur_kernel;
} ss_config;

/* max_mt_positions sizes everything the MT searches index by position: the handle's self-attention K / V caches
 * [mt_layers][max_mt_positions][mt_dim], its token and feature buffers, the position table the host loads as "__const__.mt_pos_table"
 * (max_mt_positions + pad + 2 rows) and, per stream-pool slot, the incremental search's K / V caches (2 x mt_layers x max_mt_positions
 * x mt_dim floats, allocated for every slot by the first ss_pool_mt_greedy_incremental: with mt_layers = 4 and mt_dim = 512, 16 MB
 * per slot at 1024 and 32 MB at 2048, so 1 GB for 32 slots at 2048).  A search needs max_len + 2 entries and is refused with
 * SS_ERR_CAPACITY before any launch otherwise.  The incremental searches keep one more entry per call of the utterance (max_len +
 * kv_off + 2), so the S2TT agents, whose generator allows max_decoder_positions - 1 tokens once the source is finished, need
 * max_decoder_positions + (MT calls of the utterance) + 2: 2048 covers every utterance that max_enc_frames = 1024 admits (1200
 * positions; a 41 s utterance in 160 ms segments makes 256 calls).  The self-attention of the persistent MT kernels takes any number
 * of entries; ss_create refuses a value outside [3, SS_MAX_MT_POSITIONS] with SS_ERR_INVALID. */
#define SS_MAX_MT_POSITIONS 8192

/* ---- lifecycle --------------------------------------------------------------------------------------- */
int ss_create(ss_engine** out, int device, const ss_config* cfg);
int ss_destroy(ss_engine* h);
const char* ss_last_error(const ss_engine* h); /* h == NULL: why this thread's last ss_create was refused */
const char* ss_version(void);

/* Load one fp32 tensor of the checkpoint by its fairseq state-dict key (host memory, row-major).
 * Replaces load_state_dict: fairseq/checkpoint_utils.py load_model_ensemble -> agent:355-393;
 * vocoder keys are prefixed "vocoder." (agent/tts/vocoder.py:37-45, weight_norm already removed).
 * Constants the reference computes at construction (sinusoid tables, mel bank, Povey window, gcmvn)
 * are passed the same way under "__const__." keys by the Python host. */
int ss_load_tensor(ss_engine* h, const char* key, const float* data_host, int ndim, const int64_t* shape);
/* Repack to kernel layouts (GLU interleave, conv im2col order, BN fold, rel-pos projections,
 * transposed-conv polyphase split) and upload.  Fails with SS_ERR_MISSING naming the first missing key. */
int ss_finalize(ss_engine* h);

/* encoder.chunk_size / conv chunk (agent:395-413; ASR agent :361-375).  0 = offline model (N10). */
int ss_set_chunk(ss_engine* h, int attn_chunk, int conv_chunk);

/* ---- F1/F2: OnlineFeatureExtractor.__call__ + transform (agent:66-98) --------------------------------- */
/* number of fbank frames for n 16 kHz samples: floor((n - 240) / 160), >= 0 */
int64_t ss_fbank_num_frames(int64_t n_samples);
/* frames [frame0, frame0+n_frames) of the utterance `samples_dev` (fp32, NOT scaled) -> out_dev[n_frames][80]. enqueue only */
int ss_fbank(ss_engine* h, void* stream, const float* samples_dev, int64_t n_samples, int64_t frame0, int64_t n_frames,
             float* out_dev);

/* ---- F1, wire format: convert_waveform(..., to_sample_rate=16000) (fairseq/fairseq/data/audio/audio_utils.py:53-62), called by
 * OnlineFeatureExtractor with sr = 48000 (agent:32-35,66).  The reference resamples with sox `rate` through torchaudio.sox_effects
 * (third party, not in this image); here: windowed-sinc decimation by 3 with the filter of torchaudio.functional.resample
 * (Hann-windowed sinc, lowpass_filter_width 6, rolloff 0.99, 41 taps), loaded as "__const__.resample_3to1".
 * out_dev[i] for i in [out0, out0 + n_out) (absolute 16 kHz sample index) from in_dev[0 .. n_in) at 48 kHz.
 * ss_resample_out_len: 16 kHz samples that are FINAL given n 48 kHz samples so far (filter support complete), or the whole-signal
 * length ceil(n / 3) once the source is finished -- the streaming agent only consumes final samples. enqueue only */
int64_t ss_resample_out_len(int64_t n_in_48k, int finished);
int ss_resample_48k_to_16k(ss_engine* h, void* stream, const float* in_dev, int64_t n_in, int64_t out0, int64_t n_out, float* out_dev);

/* ---- E1-E6: ChunkS2SConformerEncoder.forward (chunk_unity/models/s2t_conformer.py:111-163) -------------- */
/* encoder frames for F fbank frames: two stride-2 convs (chunk_unity/modules/convolution.py:75-79) */
int64_t ss_encoder_out_frames(int64_t n_fbank_frames);
/* feats_dev [B][F][80] (zero padded), lengths_host[B] (or NULL = all F) -> out_dev [B][T][enc_dim], T = ss_encoder_out_frames(F).
 * Full recompute of the prefix, like the reference.  enqueue only. */
int ss_encoder_forward(ss_engine* h, void* stream, const float* feats_dev, const int32_t* lengths_host, int B, int F,
                       float* out_dev);

/* Streaming form of the same encoder for ONE utterance per handle (what the reference agent recomputes from sample 0
 * on every policy() call, agent:433): frames of completed chunk groups are final (SURVEY.md §7.2), so only the rows
 * [T_final_prev, T) are computed; per-layer K/V and conv-module inputs of the final rows are cached in the handle.
 * feats_dev [F][feat_dim] = ALL fbank frames so far; enc_out_dev = caller-owned persistent buffer [>= T][enc_dim]
 * whose rows < T_final_prev are left untouched.  *T_out = ss_encoder_out_frames(F); *T_final_out = rows now final.
 * Requires attn_chunk > 0.  enqueue only */
int ss_encoder_stream_reset(ss_engine* h);
int ss_encoder_stream_step(ss_engine* h, void* stream, const float* feats_dev, int F, float* enc_out_dev, int32_t* T_out,
                           int32_t* T_final_out);

/* ---- C1: CTCDecoder.generate (agent/ctc_decoder.py:40-111): Linear -> log_softmax -> mask pad,unk -> argmax -> collapse.
 * head 0 = source_unigram (ASR), 1 = ctc_target_unigram (ST).  enc_dev [rows][enc_dim] of ONE utterance.
 * argmax_dev[rows] int64; tokens_dev[rows] int64 / index_dev[rows] int32 hold *count_dev collapsed entries. enqueue only */
int ss_ctc_greedy(ss_engine* h, void* stream, int head, const float* enc_dev, int rows, int64_t* argmax_dev,
                  int64_t* tokens_dev, int32_t* index_dev, int32_t* count_dev);
/* Same, for a caller that keeps `argmax_dev` across calls on a growing sequence: only rows [row0, rows) are projected and
 * arg-maxed (rows below row0 keep their cached arg-max, valid when those encoder rows have not changed, i.e. they are
 * below the T_final of the previous ss_encoder_stream_step); the collapse runs over all `rows`. */
int ss_ctc_greedy_rows(ss_engine* h, void* stream, int head, const float* enc_dev, int rows, int row0, int64_t* argmax_dev,
                       int64_t* tokens_dev, int32_t* index_dev, int32_t* count_dev);

/* Both heads of one policy() call (agent:437 and :461) in two launches: one [rows - row0][2V] projection over the concatenated
 * head weights and one kernel that takes the arg-max of every new row and then (last block) collapses both sequences.
 * argmax{0,1}_dev as in ss_ctc_greedy_rows (caller-kept, rows below row0 valid).  packed_out_dev holds, per head h, at int64
 * offset h * (2 * rows + 2): [count (int32) | tokens[rows] int64 | index[rows] int32] -- one device->host copy reads everything.
 * Heads with different vocabularies fall back to two ss_ctc_greedy_rows calls with the same packing.  enqueue only */
int ss_ctc_greedy_pair(ss_engine* h, void* stream, const float* enc_dev, int rows, int row0, int64_t* argmax0_dev, int64_t* argmax1_dev,
                       int64_t* packed_out_dev);

/* Samples per launch group of ss_ctc_greedy_batch: at most max(1, SS_CTC_BATCH_ROWS / T) samples (their logits, 2 x vocab floats per
 * row, live in the workspace together). */
#define SS_CTC_BATCH_ROWS 8192
/* Both CTC heads over every row of B padded utterances (the offline generator's prints, ctc_decoder.py:40-111 on the padded
 * encoder output: padded rows are NOT trimmed).  enc_dev [B][T][enc_dim].  Per launch group: one [rows][2V] projection over the
 * concatenated head weights (one projection per head when the two vocabularies differ), one arg-max launch over every row of both
 * heads and one collapse launch with one CTA per (sample, head).  packed_out_dev holds, for sample b at int64 offset
 * b * 2 * (2T + 2), ss_ctc_greedy_pair's packing of its two heads: head h at + h * (2T + 2) = [count (int32) | tokens[T] int64 |
 * index[T] int32], so one device->host copy reads the whole batch.  Sample b's output equals ss_ctc_greedy_rows(head, enc_b, T, 0)
 * (the projection may take another GEMM kernel at a different row count).  Keeps no state.
 * Errors: SS_ERR_INVALID for B <= 0, T <= 0 or a null pointer.  enqueue only */
int ss_ctc_greedy_batch(ss_engine* h, void* stream, const float* enc_dev, int B, int T, int64_t* packed_out_dev);

/* ---- M1/M2: SequenceGenerator.generate_decoder, beam 1 (agent/sequence_generator.py:165-582) + the extra
 * mt_decoder(prev_output_tokens, features_only=True) forward (agent:638-642).
 * prefix_host[n_prefix] = tgt_subwords_indices; max_new_tokens as in the agent (-1 = source finished:
 * max_len = min(max_len_b, max_positions-1)).  Writes the finalized hypothesis WITHOUT the trailing eos to
 * tokens_out_host (capacity max_out) and the decoder features of [eos, tokens...] to feats_out_dev[(n_out+1)][mt_dim].
 * Synchronises `stream` once per generated token (the arg-max is needed on the host for the stop test).
 * Errors: SS_ERR_INVALID for a prefix token outside [0, tgt_vocab), before anything is launched or the handle's state changes. */
int ss_mt_greedy(ss_engine* h, void* stream, const float* enc_dev, int T, const int64_t* prefix_host, int n_prefix,
                 int max_new_tokens, int max_len_b, int64_t* tokens_out_host, int max_out, int* n_out,
                 float* feats_out_dev);
/* Greedy MT search (beam 1, no prefix, max_len = min(max_len_b, max_mt_positions - 1)) for B independent samples.
 * enc_dev: [B][T_stride][enc_dim] (e.g. ss_encoder_forward's padded output); T_host[b]: sample b's unpadded rows, 1 <= T_b <= T_stride.
 * tokens_out_host: [B][max_out], hypothesis without eos; n_out_host[b]: its length.  Each row equals ss_mt_greedy on enc_b[:T_b].
 * Up to 32 samples are decoded together in one persistent kernel (larger B: consecutive groups of 32), reading the MT weights
 * once per step for all of them, with its own caches: the single-stream MT state of the handle is not touched.  Where that
 * kernel cannot run (option persistent_mt = 0, an unsupported shape, a refused cooperative launch) and for groups of fewer
 * than 2 samples (option mt_batch_min_rows), samples are decoded one by one through ss_mt_greedy; that path leaves the
 * single-stream cross K / V cache invalid, so the next streaming call projects all its rows again.
 * Errors: SS_ERR_INVALID for B <= 0, a T_b outside [1, T_stride] or a null pointer; SS_ERR_CAPACITY when max_len > max_out. */
int ss_mt_greedy_batch(ss_engine* h, void* stream, const float* enc_dev, int B, int T_stride, const int32_t* T_host, int max_len_b,
                       int64_t* tokens_out_host, int max_out, int32_t* n_out_host);
/* MT beam search of width `beam` (SequenceGenerator.generate_decoder with BeamSearch, beam_size = beam, min_len 1,
 * normalize_scores, no prefix; the offline generator's --beam-mt K --lenpen len_penalty) for B independent samples.  enc_dev,
 * T_stride, T_host and max_len_b as ss_mt_greedy_batch.  For sample b, hypothesis i < beam (sorted by score, highest first; on
 * equal scores the one finalized first) is written to tokens_out_host[(b * beam + i) * max_out ...] without eos, its length to
 * n_out_host[b * beam + i], its score (sum of log-probabilities, eos included, over (length + 1) ** len_penalty) to
 * scores_out_host[b * beam + i], and its per-token scores, eos's last, to pos_scores_out_host[(b * beam + i) * (max_out + 1) ...].
 * The candidates of a step are ranked by score; on exactly equal scores the lower index beam * tgt_vocab + token ranks first.
 * Each launch of the batched MT kernel holds floor(32 / beam) samples of beam rows each, whose beams share one cross K / V
 * projection; the search keeps all its state on the device and the host reads one done flag per sample per burst of 16 steps.
 * Like ss_mt_greedy_batch it does not touch the handle's single-stream MT state.
 * Errors, all before anything is launched: SS_ERR_INVALID for B <= 0, beam outside [2, 32] (beam 1 is ss_mt_greedy_batch), a
 * non-finite len_penalty, a T_b outside [1, T_stride] or a null pointer; SS_ERR_CAPACITY when max_len > max_out; SS_ERR_CUDA
 * when the persistent MT kernels are off (option persistent_mt) or do not support the shape.  A refused cooperative launch is
 * SS_ERR_CUDA too (there is no other implementation of the beam search). */
int ss_mt_beam_batch(ss_engine* h, void* stream, const float* enc_dev, int B, int T_stride, const int32_t* T_host, int beam, int max_len_b,
                     float len_penalty, int64_t* tokens_out_host, int max_out, int32_t* n_out_host, float* scores_out_host,
                     float* pos_scores_out_host);
/* Streaming hint for the NEXT ss_mt_greedy / ss_mt_features call: rows [0, rows) of the encoder output passed to it are
 * final, i.e. bit-identical in every later call with the same buffer until ss_encoder_stream_reset (ss_encoder_stream_step
 * reports that count as T_final).  Their cross-attention keys / values are then projected once instead of on every call.
 * Without the hint every call projects all rows (the reference recomputes everything, agent:520-538). */
int ss_mt_stable_rows(ss_engine* h, int rows);
/* teacher-forced features for tokens_host[n] (pads allowed only as a tail): TransformerDecoderBase.extract_features_scriptable
 * (ctc_unity/modules/transformer_decoder.py:257-403).  feats_out_dev [n][mt_dim]; logits_last_dev (optional) [tgt_vocab]. enqueue only.
 * Errors: SS_ERR_INVALID for a token outside [0, tgt_vocab), before anything is launched or the handle's state changes. */
int ss_mt_features(ss_engine* h, void* stream, const float* enc_dev, int T, const int64_t* tokens_host, int n,
                   float* feats_out_dev, float* logits_last_dev);
/* Samples per launch group of ss_mt_features_batch and ss_t2u_unit_decode_batch: at most max(1, SS_UNIT_BATCH_ROWS / (S * rate))
 * samples, i.e. the unit decoder's upsampled rows of a group stay within this budget (about 28 KB of workspace per row with the
 * StreamSpeech sizes); larger batches run as consecutive groups. */
#define SS_UNIT_BATCH_ROWS 32768
/* ss_mt_features for B samples of one padded batch (the offline generator's mt_decoder(prev_output_tokens_mt, features_only),
 * sequence_generator_multi_decoder_ctc.py:287-291).  enc_dev [B][T_stride][enc_dim]; sample b's cross-attention keys are its
 * first T_host[b] rows, 1 <= T_b <= T_stride.  tokens_host [B][S] = [eos, hyp_b..., pad...] (pads only as a tail; positions
 * restart for every sample and pads get the padding position); self-attention is causal over sample b's S_b non-pad tokens.
 * feats_out_dev [B][S][mt_dim].  The cross K / V are projected into the call's workspace, one layer at a time: the handle's
 * single-stream MT state (cross K / V cache, stable-rows hint, incremental caches, token buffer) is neither read nor written.
 * Sample b's rows equal ss_mt_features(enc_b[:T_b], tokens_b) within float tolerance (the GEMMs may take another kernel at
 * B * S rows; the attention arithmetic of a sample is the same).  Synchronises `stream` once (upload of the tokens and lengths).
 * Errors: SS_ERR_INVALID for B <= 0, S <= 0 or S > max_mt_positions, T_stride <= 0, a T_b outside [1, T_stride], a token outside
 * the vocabulary, a pad before a non-pad token, or a null pointer. */
int ss_mt_features_batch(ss_engine* h, void* stream, const float* enc_dev, int B, int T_stride, const int32_t* T_host, const int64_t* tokens_host,
                         int S, float* feats_out_dev);

/* ---- M1 with the reference's incremental states (use_incremental_states=True: speech_to_text.s2tt.streamspeech.agent.py:136,178;
 * SURVEY.md N12).  The decoder state lives in the handle ACROSS calls until ss_mt_incremental_reset (the agent's reset()):
 *  - self-attention K / V of every token fed so far are kept; each call feeds only tokens it has not fed -- except that its first
 *    step feeds the last prefix token again (fairseq slices prev_output_tokens[:, -1:], ctc_unity/modules/transformer_decoder.py:
 *    305-308, and the previous call's final, eos-forcing step had already fed it), which leaves a duplicate cache entry per call;
 *  - cross-attention K / V are projected only for encoder rows beyond those cached by earlier calls (transformer_layer.py:
 *    492-505) and never refreshed, i.e. early rows keep the projections of the then-provisional encoder output.
 * Both quirks change the hypothesis and are reproduced.  The state shares the handle's MT caches with ss_mt_greedy and ss_mt_features,
 * which write them from row 0: once either has run on a handle whose state is not empty, ss_mt_greedy_incremental returns SS_ERR_STATE
 * before any launch until ss_mt_incremental_reset (the batched, beam and pool entry points leave the state alone unless they fall back
 * to ss_mt_greedy, see there).  ss_debug_copy "mt_inc_state" reads the state back.  max_len_b = the caller's max_len for max_new_tokens == -1
 * (min(int(max_len_a * src_len + max_len_b), max_decoder_positions - 1), sequence_generator.py:205-215).  Requires the
 * persistent MT kernel (option persistent_mt = 1).  Synchronises `stream` once per burst.  A prefix token outside [0, tgt_vocab)
 * is SS_ERR_INVALID, refused before anything is launched or the state changes. */
int ss_mt_incremental_reset(ss_engine* h);
int ss_mt_greedy_incremental(ss_engine* h, void* stream, const float* enc_dev, int T, const int64_t* prefix_host, int n_prefix,
                             int max_new_tokens, int max_len_b, int64_t* tokens_out_host, int max_out, int* n_out);

/* ---- T1/U1/U2: synthesizer_encoder -> CTCTransformerUnitDecoder -> CTCSequenceGenerator.generate
 * (ctc_unity/modules/transformer_encoder.py:32-77, ctc_transformer_unit_decoder.py:53-260, agent/ctc_generator.py:41-123).
 * mt_feats_dev [S][mt_dim]; n_pad_tail = number of trailing <pad> positions of prev_output_tokens_mt (whole_word).
 * argmax_dev [S*rate] int64, units_dev [S*rate] int64 (dictionary indices, blank/pad removed), count_dev. mask_eos = offline generator (N3).
 * t2u_out_dev / logits_dev optional (NULL) debug outputs [S][unit_dim], [S*rate][unit_vocab].  enqueue only */
int ss_t2u_unit_decode(ss_engine* h, void* stream, const float* mt_feats_dev, int S, int n_pad_tail, int mask_eos,
                       int64_t* argmax_dev, int64_t* units_dev, int32_t* count_dev, float* t2u_out_dev, float* logits_dev);
/* ss_t2u_unit_decode for B samples of one padded batch (sequence_generator_multi_decoder_ctc.py:293-330): T2U encoder with each
 * sample's padding mask -> LayerNorm -> x rate upsample plus sample b's positional row pos_rows_dev[b] (N1: the row the reference
 * gives batch element b, i.e. sinusoidal row pad + 1 + b of the WHOLE batch, even when the batch runs in several groups) -> the
 * unit decoder layers -> LayerNorm -> out-projection -> arg-max (pad, unk masked, + eos when mask_eos: N3) -> CTC collapse of each
 * sample.  mt_feats_dev [B][S][mt_dim]; n_pad_tail_host[b] in [0, S): trailing pad positions of sample b, whose rows are decoded
 * too (N2); pos_rows_dev [B][unit_dim].  argmax_dev [B][S * rate]; packed_units_dev [B][S * rate + 1], row b = [count (int32 in the
 * first int64) | units], so that one device->host copy reads every sample.  Sample b equals ss_t2u_unit_decode(mt_feats_b,
 * n_pad_tail_b) with the positional row set to pos_rows_dev[b] (within float tolerance for the activations; the GEMMs may take
 * another kernel at more rows).  Neither reads nor writes the handle's positional row (ss_unit_position_row) and does not
 * synchronise the device (unless the workspace has to grow); synchronises `stream` once (upload of the key lengths) when some
 * sample has a pad tail, not at all otherwise.  ss_t2u_unit_decode is the same code with B = 1.
 * Errors: SS_ERR_INVALID for B <= 0, S <= 0 or S > max_mt_positions, an n_pad_tail outside [0, S), or a null pointer. */
int ss_t2u_unit_decode_batch(ss_engine* h, void* stream, const float* mt_feats_dev, int B, int S, const int32_t* n_pad_tail_host, const float* pos_rows_dev,
                             int mask_eos, int64_t* argmax_dev, int64_t* packed_units_dev);
/* ss_t2u_unit_decode_batch plus the unit hypothesis' positional scores (CTCSequenceGenerator.generate, ctc_generator.py:54-61):
 * lprob_dev [B][S * rate] fp32, row r of sample b = log_softmax(logits[b][r])[argmax[b][r]] over all unit_vocab columns (the masked
 * pad / unk / eos columns stay in the normaliser, as the reference masks after log_softmax), pad-tail rows included.  argmax_dev and
 * packed_units_dev are bit-identical to ss_t2u_unit_decode_batch's.  Same synchronisation and groups as ss_t2u_unit_decode_batch.
 * Errors: those of ss_t2u_unit_decode_batch, and SS_ERR_INVALID for a null lprob_dev. */
int ss_t2u_unit_decode_batch_scored(ss_engine* h, void* stream, const float* mt_feats_dev, int B, int S, const int32_t* n_pad_tail_host,
                                    const float* pos_rows_dev, int mask_eos, int64_t* argmax_dev, int64_t* packed_units_dev, float* lprob_dev);
/* ss_t2u_unit_decode_batch over ragged lengths (the stream pool's S2ST agents: every writing stream has its own number of MT
 * positions).  mt_feats_dev [B][S_stride][mt_dim]; sample b has S_host[b] positions, 1 <= S_b <= S_stride (S_host NULL: all S_stride),
 * of which the last n_pad_tail_host[b] (in [0, S_b)) are N2 pad positions that are decoded; positions >= S_b are neither keys nor
 * decoded into units.  argmax_dev [B][S_stride * rate] (rows >= S_b * rate unspecified) and packed_units_dev [B][S_stride * rate + 1]
 * as ss_t2u_unit_decode_batch, whose call this is with every S_b = S_stride.  Sample b equals ss_t2u_unit_decode(mt_feats_b[:S_b],
 * n_pad_tail_b) with positional row pos_rows_dev[b] (within float tolerance; the GEMMs may take another kernel at more rows).
 * Synchronises `stream` once (upload of the key lengths) when some sample has a pad tail or S_b < S_stride, not at all otherwise.
 * Errors: SS_ERR_INVALID for B <= 0, S_stride <= 0 or S_stride > max_mt_positions, an S_b outside [1, S_stride], an n_pad_tail
 * outside [0, S_b), or a null pointer. */
int ss_t2u_unit_decode_ragged(ss_engine* h, void* stream, const float* mt_feats_dev, int B, int S_stride, const int32_t* S_host,
                              const int32_t* n_pad_tail_host, const float* pos_rows_dev, int mask_eos, int64_t* argmax_dev, int64_t* packed_units_dev);

/* ---- UnitY (researches/translatotron, `fairseq-generate --task speech_to_speech_modified`): the T2U encoder on its own, then the
 * autoregressive unit decoder searched token by token (examples/speech_to_speech/unity/sequence_generator.py, driven by
 * sequence_generator_multi_decoder.py:259-268).  A UnitY checkpoint has no CTC heads: ss_finalize then records that, and ss_ctc_greedy,
 * ss_ctc_greedy_rows, ss_ctc_greedy_pair, ss_ctc_greedy_batch and ss_pool_step return SS_ERR_STATE naming the missing heads.  The unit
 * search needs "__const__.unit_pos_table" (the sinusoidal table of max_target_positions + pad + 1 rows of unit_dim); with it ss_finalize
 * refuses a unit decoder that is not 512 wide with 2048-wide FFNs and 8 heads (SS_ERR_INVALID), and a stored
 * decoder.output_projection.weight that is not the embedding.
 *
 * synthesizer_encoder(x, padding_mask) (TransformerEncoderNoEmb) of B samples: mt_feats_dev [B][S_stride][unit_dim] (ss_mt_features_batch's
 * output), sample b's positions >= S_host[b] are masked keys (prev_output_tokens_mt's pads); causal when the config's uni_encoder is set
 * (UnitY: bidirectional); no positions are added.  out_dev [B][S_stride][unit_dim] after the final LayerNorm (rows >= S_b computed too).
 * Samples run in groups of at most max(1, SS_UNIT_BATCH_ROWS / S_stride).  Synchronises `stream` once (upload of the key lengths) when
 * some S_b < S_stride, not at all otherwise.
 * Errors: SS_ERR_INVALID for B <= 0, S_stride <= 0 or > max_mt_positions, an S_b outside [1, S_stride] or a null pointer. */
int ss_t2u_encode_batch(ss_engine* h, void* stream, const float* mt_feats_dev, int B, int S_stride, const int32_t* S_host, float* out_dev);
/* The unit search at beam 1 (SequenceGenerator.generate_decoder with BeamSearch, beam_size 1, min_len 1, normalize_scores, unk penalty 0,
 * temperature 1) for B samples: sample b cross-attends to its first S_host[b] rows of t2u_dev [B][S_stride][unit_dim] (ss_t2u_encode_batch's
 * output), projected once per call into cross K / V of every unit layer.  Step s takes log_softmax over all unit_vocab columns, then pad is
 * -inf, eos is -inf at step 0 and everything but eos at step max_len; the best token continues the row, eos ends it.  max_len is the
 * caller's min(int(max_len_a * src_tokens.size(1) + max_len_b), max_decoder_positions - 1): the BATCH's padded source length, so one
 * max_len for every sample.  Writes sample b's tokens without eos to tokens_out_host[b * max_out ...], their count to n_out_host[b], its
 * positional scores (the log-probability of every chosen token, eos last) to pos_scores_out_host[b * (max_out + 1) ...] and its score
 * (their sum over (n_out + 1) ** len_penalty) to scores_out_host[b].  Runs on the batched decoder kernel's beam instantiation at beam 1
 * (the reference's own search; each row's self-attention cache stays in place, any number of entries), 32 samples per launch group, steps
 * in bursts of 16 per launch; the host reads one done flag per sample per burst (one synchronisation) and stops once all are set.  Shares
 * the batched MT searches' device buffers, not the handle's single-stream MT state.
 * Errors, all before anything is launched: SS_ERR_INVALID for B <= 0, S_stride <= 0, an S_b outside [1, S_stride], max_len < 1, a
 * non-finite len_penalty or a null pointer; SS_ERR_STATE on a handle without "__const__.unit_pos_table" (a StreamSpeech checkpoint);
 * SS_ERR_CAPACITY when max_len > max_out, max_len + pad + 2 exceeds the position table's rows, or an S_b > 1024; SS_ERR_CUDA when option
 * persistent_mt is 0.  A refused cooperative launch is SS_ERR_CUDA (there is no other implementation). */
int ss_unit_search_batch(ss_engine* h, void* stream, const float* t2u_dev, int B, int S_stride, const int32_t* S_host, int max_len, float len_penalty,
                         int64_t* tokens_out_host, int max_out, int32_t* n_out_host, float* scores_out_host, float* pos_scores_out_host);

/* Positional-embedding row (unit_dim floats, host memory) the CTC unit decoder adds to every upsampled T2U state.  The
 * reference computes positions from x[:, :, 0] viewed as [bsz, seq] (ctc_transformer_unit_decoder.py:176-181, SURVEY.md N1), so
 * every time step of batch element b gets the sinusoidal row pad + 1 + b.  The engine is created with the row of b = 0 (the
 * streaming agents); a per-sample reproduction of a batch sets the row of each sample before decoding it (the offline generator
 * passes every sample's row to ss_t2u_unit_decode_batch instead).  Synchronises the device. */
int ss_unit_position_row(ss_engine* h, const float* row_host);
/* ---- V1: CodeGenerator.forward front half (agent/tts/codehifigan.py:56-66): embedding + duration predictor.
 * codes_dev[U] int64 unit ids (0..num_embeddings-1); dur_out_dev[U] int64; cumsum_out_dev[U+1] int32 (frame offsets).
 * dur_prediction=0 -> every duration is 1.  The expanded frame sequence stays cached in the handle for ss_vocoder_generate. enqueue only */
int ss_vocoder_durations(ss_engine* h, void* stream, const int64_t* codes_dev, int U, int dur_prediction, int64_t* dur_out_dev,
                         int32_t* cumsum_out_dev);
/* ---- V2: HiFi-GAN Generator.forward (fairseq/models/text_to_speech/hifigan.py:154-170) on frames
 * [frame0 - ctx, frame0 + n_frames) of the cached sequence of total_frames frames (ctx = min(left_context, frame0);
 * left_context < 0 = the generator's full receptive field, which makes the result equal to a full-sequence pass);
 * writes n_frames*hop samples for frames [frame0, frame0+n_frames) to wav_out_dev.  frame0 + n_frames must equal total_frames
 * (the agent always emits the tail).  enqueue only */
int ss_vocoder_generate(ss_engine* h, void* stream, int total_frames, int frame0, int n_frames, int left_context,
                        float* wav_out_dev);
/* ---- V1 + V2 of n sequences at once (ss_vocoder_durations / ss_vocoder_generate are these calls with n = 1).
 * Durations: codes_dev holds the n code sequences concatenated (U_host[n] units each); dur_out_dev receives the durations
 * packed the same way, and cumsum_out_dev (optional) one cumsum of U_s + 1 frame offsets per sequence, packed in sequence order.
 * The duration predictor runs over groups of up to 32 sequences (and as many padded rows as its split-K scratch holds) in a fixed
 * number of launches per group, each sequence seeing its own zero padding; every sequence's durations and cumsum equal those of a
 * call with that sequence alone.  The expanded sequences stay
 * cached in the handle for ss_vocoder_generate_ragged.
 * Generate: sequence s does what ss_vocoder_generate(total_frames_host[s], frame0_host[s], n_frames_host[s],
 * left_context_host[s]) does, bit for bit, and its n_frames_s * hop samples are written packed in sequence order to wav_out_dev.
 * n must equal the last durations call's n.  Sequences of up to 1024 frames (after the left context) run together in one
 * cooperative launch of the fused generator kernel per group (up to 32 sequences and 3072 frames), after one frame-expansion
 * launch; longer ones, and every sequence when the cooperative launch is refused or option vocoder_fused = 0, take the
 * multi-launch path.  Errors: SS_ERR_INVALID for n <= 0, a U_s <= 0, a frame range that is not the tail or a null pointer;
 * SS_ERR_STATE without vocoder weights, or for a generate call without a durations call of the same n.  enqueue only */
int ss_vocoder_durations_ragged(ss_engine* h, void* stream, int n, const int64_t* codes_dev, const int32_t* U_host, int dur_prediction,
                                int64_t* dur_out_dev, int32_t* cumsum_out_dev);
int ss_vocoder_generate_ragged(ss_engine* h, void* stream, int n, const int32_t* total_frames_host, const int32_t* frame0_host,
                               const int32_t* n_frames_host, const int32_t* left_context_host, float* wav_out_dev);
int ss_vocoder_hop(const ss_engine* h);
int ss_vocoder_receptive_field(const ss_engine* h);

/* ---- multi-stream pool: n concurrent utterances per handle, ONE batched streaming step (SURVEY.md §8 f2; BASELINE configs[3] = 256
 * concurrent ASR streams, 32 per GPU).  The reference is one utterance per agent process (agent/speech_to_text.asr.streamspeech.
 * agent.py:385-433).  Each stream owns a slot: device audio, fbank frames, per-layer K / V / conv-input caches, encoder rows and CTC
 * arg-max rows.  Results of every stream equal the single-stream entry points' (same arithmetic per stream; GEMMs see the rows of
 * all n streams). */
int ss_pool_create(ss_engine* h, int n_slots, int max_seconds);  /* 16 kHz sources: ss_pool_create_rate(h, n_slots, max_seconds, 16000) */
/* Pool whose sources arrive at sample_rate = 16000 or 48000 Hz (anything else: SS_ERR_INVALID).  A 48 kHz pool keeps the pushed
 * samples in a second per-slot row of max_seconds * 48000 + 1200 samples; every ss_pool_step first extends each listed slot's 16 kHz
 * row on the device (one launch for all slots) with the samples that are final, as the single-stream 48 kHz agent does:
 * [produced so far, ss_resample_out_len(n48, finished)), each bit-identical to ss_resample_48k_to_16k on the same 48 kHz prefix. */
int ss_pool_create_rate(ss_engine* h, int n_slots, int max_seconds, int sample_rate);
int ss_pool_reset(ss_engine* h, int slot);                       /* new utterance on this slot (clears the finished flag) */
/* The slot's own latency: attention chunk and conv chunk of its streaming encoder, as ss_set_chunk sets them for the handle
 * (attn_chunk > 0, conv_chunk > 0 and even; otherwise SS_ERR_INVALID).  (0, 0) = follow the handle's ss_set_chunk at step time,
 * the default.  Slots of different latencies share every batched step and its one pass over the encoder weights.  SS_ERR_STATE
 * while the slot holds samples (a stream keeps its latency for the whole utterance); the setting survives ss_pool_reset. */
int ss_pool_set_chunk(ss_engine* h, int slot, int attn_chunk, int conv_chunk);
/* append n samples at the pool's rate (host memory) to the slot's device audio: enqueue of one host->device copy.  The capacity
 * check counts samples at that rate.  SS_ERR_STATE after ss_pool_finish until ss_pool_reset */
int ss_pool_push_audio(ss_engine* h, void* stream, int slot, const float* samples_host, int n);
/* The slot's source is closed: in a 48 kHz pool the next step produces the 16 kHz tail up to ceil(n48 / 3) (ss_resample_out_len
 * with finished = 1).  In a 16 kHz pool it only sets the flag, so callers need not branch on the rate. */
int ss_pool_finish(ss_engine* h, int slot);
/* state of a slot: 16 kHz samples available to fbank (in a 48 kHz pool: those produced by the steps so far), fbank frames held,
 * final encoder rows, device pointers of its encoder rows [Tcap][enc_dim] and fbank frames [Fcap][feat_dim] (any out pointer may
 * be NULL) */
int ss_pool_info(ss_engine* h, int slot, int64_t* n_audio, int32_t* n_feat, int32_t* T_final, float** enc_out_dev, float** feats_dev);
/* One streaming step of the n listed slots over all the audio pushed so far: OnlineFeatureExtractor (new frames only) ->
 * forward_encoder (rows not yet final, ss_encoder_stream_step semantics) -> CTCDecoder.generate for ctc_heads heads (0: none, 1: ASR,
 * 2: ASR + ST).  Per stream i, packed_out_dev + out_off_host[i] holds per head [count (int32) | tokens[T_i] int64 | index[T_i] int32]
 * (head h at + h * (2 T_i + 2) int64 words).  T_out_host / T_final_out_host / out_off_host: n entries each (host, written before
 * return).  Synchronises `stream` once at entry (descriptor staging); everything else is enqueue only. */
int ss_pool_step(ss_engine* h, void* stream, int n, const int32_t* slots_host, int ctc_heads, int64_t* packed_out_dev, int64_t packed_capacity,
                 int32_t* T_out_host, int32_t* T_final_out_host, int64_t* out_off_host);
/* Greedy MT search (M1) of n pool streams at once, each continuing its own forced prefix: stream i (slot slots_host[i]) gets what
 * ss_mt_greedy(enc, prefix_i, n_prefix_host[i], max_new_tokens_host[i], max_len_b) gives on the slot's encoder rows [0, T_i) of its
 * last ss_pool_step: max_len = n_prefix + max_new_tokens, or min(max_len_b, max_mt_positions - 1) for -1 (source finished); eos banned
 * at position 0 and forced at max_len.  prefix_host holds the n prefixes concatenated.  tokens_out_host [n][max_out]: the hypothesis
 * without eos (prefix included), n_out_host[i] its length; feats_out_dev [n][feats_ld][mt_dim]: the decoder features of [eos, tokens...]
 * (rows 0 .. n_out_host[i]).  Up to 32 streams are decoded together on the batched MT kernel after one teacher-forced pass over all
 * their prefixes; larger n run as consecutive groups.  The cross-attention K / V of every slot are cached in the pool ([slot][mt_layers]
 * [Tcap][2 * mt_dim], allocated by the first call): rows below the slot's T_final are projected once, as ss_mt_stable_rows does for one
 * stream, until ss_pool_reset.  Groups of fewer than mt_batch_min_rows streams and refused cooperative launches decode stream by stream
 * through ss_mt_greedy (which leaves the single-stream cross K / V cache invalid, as ss_mt_greedy_batch's fallback does); otherwise the
 * handle's single-stream MT state (cross K / V cache, stable-rows hint, incremental state, token buffer) is neither read nor written.
 * Tokens equal ss_mt_greedy's; features within float tolerance (the prefix rows are computed by the per-operation kernels).
 * Synchronises `stream` once per group for the uploads and once per burst of 16 steps.
 * Errors: SS_ERR_INVALID for a bad or repeated slot, a slot without encoder rows, a prefix longer than max_len, a prefix token outside
 * the vocabulary or a null pointer; SS_ERR_CAPACITY when max_len + 2 > max_mt_positions, max_len > max_out or max_len >= feats_ld. */
int ss_pool_mt_greedy(ss_engine* h, void* stream, int n, const int32_t* slots_host, const int64_t* prefix_host, const int32_t* n_prefix_host,
                      const int32_t* max_new_tokens_host, int max_len_b, int64_t* tokens_out_host, int max_out, int32_t* n_out_host,
                      float* feats_out_dev, int feats_ld);
/* ss_mt_greedy_incremental (the S2TT agent's MT search with the reference's incremental states, N12) for n pool streams at once,
 * each on its slot's own state: stream i (slot slots_host[i]) gets exactly what ss_mt_greedy_incremental(enc, T_i, prefix_i,
 * n_prefix_host[i], max_new_tokens_host[i], max_len_host[i]) gives on a handle holding that slot's state, with enc the slot's
 * encoder rows [0, T_i) of its last ss_pool_step.  max_len_host[i] is the stream's max_len for max_new_tokens == -1.  The state
 * lives in the pool until ss_pool_reset: per slot a self-attention cache [mt_layers][max_mt_positions][mt_dim] (K and V; allocated by
 * the first call for every slot) with its entry count, and the cross-attention K / V of the encoder rows seen so far.  As in the
 * single-stream call, each call re-feeds the last prefix token (one duplicate self-attention entry per call: the prefix's entry of
 * position p is p + kv_off with kv_off = entries - n_prefix) and projects only encoder rows that earlier calls had not seen; those are
 * never refreshed.  Prefix tokens are not fed again (their K / V are in the cache).  prefix_host holds the n prefixes concatenated;
 * tokens_out_host [n][max_out] gets each hypothesis without eos (prefix included), n_out_host[i] its length.
 * Up to 32 streams form a group: the new encoder rows of the whole group are projected at once, then groups of at least
 * mt_batch_min_rows streams decode together on the batched MT kernel and smaller ones stream by stream on the single-token kernel,
 * both over the same slot state.  The handle's single-stream MT state is neither read nor written.  A slot's cross K / V serve either
 * this call or ss_pool_mt_greedy (which re-projects rows above T_final) between resets: the other one returns SS_ERR_STATE.
 * Synchronises `stream` once per group for the uploads and once per burst of 16 steps.
 * Errors, all before any launch or state change: SS_ERR_INVALID for a bad or repeated slot, a slot without encoder rows, a null
 * pointer, a prefix token outside the vocabulary, max_len < 1 or a prefix longer than max_len; SS_ERR_STATE when kv_off < 0 (a prefix
 * the state did not produce), the persistent MT kernel is off or does not support the shape, or ss_pool_mt_greedy owns the slot;
 * SS_ERR_CAPACITY when max_len + kv_off + 2 > max_mt_positions or max_len > max_out.  A refused cooperative launch is SS_ERR_CUDA. */
int ss_pool_mt_greedy_incremental(ss_engine* h, void* stream, int n, const int32_t* slots_host, const int64_t* prefix_host,
                                  const int32_t* n_prefix_host, const int32_t* max_new_tokens_host, const int32_t* max_len_host,
                                  int64_t* tokens_out_host, int max_out, int32_t* n_out_host);

/* ---- single ops exported for the parity tests (same kernels the entry points above launch) ------------- */
int ss_op_linear(ss_engine* h, void* stream, const float* x_dev, int M, int K, const float* w_dev, const float* bias_dev, int N,
                 int act, float* out_dev);
/* same GEMM on the wgmma tensor-core kernel (kernels_umma2.cu, bf16 operand splitting, pieces = 2: 3 MMAs, 3: 6 MMAs per product);
 * parity-test / roofline hook */
int ss_op_linear_umma(ss_engine* h, void* stream, const float* x_dev, int M, int K, const float* w_dev, const float* bias_dev, int N,
                      int act, int pieces, float* out_dev);
/* out[L][N] = conv1d(pre_lrelu(x[L][C_in]), w[N][ksize*C_in] (tap-major), stride 1, dilation dil, left padding pad_left) + bias on
 * the kernel selected by mode: 0 = fp32 CUDA cores, 12 / 13 = wgmma tap-shift kernel with pre-packed weights (kernels_umma2.cu,
 * 2 / 3 bf16 pieces per operand); parity-test hook */
int ss_op_conv1d(ss_engine* h, void* stream, const float* x_dev, int L, int C_in, const float* w_dev, const float* bias_dev, int N,
                 int ksize, int dil, int pad_left, float pre_lrelu, int mode, float* out_dev);
/* engine options: "umma_vocoder" / "umma_linear" = 0 (fp32 CUDA cores), 12 or 13 (wgmma kernel, 2 or 3 bf16 pieces per operand); "umma_min_rows" / "umma_min_channels": smaller GEMMs / convs stay on
 * the fp32 kernels; "umma2_cache_clear": drop the packed weight copies;
 * "persistent_encoder" = 1 (default): ss_encoder_stream_step runs the layer stack as one cooperative kernel when the
 * shape fits, 0: one kernel per op; "vocoder_streams" = 1 (default): the three parallel resblocks of a vocoder stage run
 * on the caller's stream plus two engine-owned streams (joined before the call returns control of the stream);
 * "persistent_encoder_cluster" = 1 (0 on a fresh handle; the Python engine switches it on): steps with <= 16 active rows run on
 * the cluster kernel (4 thread-block clusters x 16 CTAs, activations in distributed shared memory; allocates 123 MB of repacked
 * weights the first time); larger steps and refused launches take the one-CTA-per-SM kernel; "cluster_cooperative" = 1 (default; 0 only
 * under a profiler that serialises kernels and cannot replay cooperative cluster launches);
 * "persistent_ffn_fused", "persistent_mt", "persistent_mt_prefix", "fbank_tma" = 1 (default): kernel variants of
 * round 2, each tested against the path it replaces;
 * "persistent_profile" = 1: the persistent kernels record %globaltimer stamps per phase; "persistent_time" = 1: CUDA events around
 * the encoder-stack kernel, every launch of the single-token MT kernel (ss_mt_greedy and the incremental searches) and the stream
 * pool's resample kernel (read with ss_debug_copy "persist_time" / "mt_time" / "pool_resample_time") */
int ss_set_option(ss_engine* h, const char* name, int value);
/* synchronous copy of a diagnostic buffer to the host: "persist_ts" = uint64 ns stamps of the last persistent step;
 * "persist_time" / "mt_time" / "pool_resample_time" = double[3] {summed ms, launches, summed algorithmic bytes / executed steps /
 * algorithmic bytes} since the last query;
 * "cluster_steps" = long long, encoder steps taken by the cluster kernel;
 * "mt_inc_state" / "pool_mt_inc_state:<slot>" = the incremental MT state of the handle (ss_mt_greedy_incremental) or of one pool slot
 * (ss_pool_mt_greedy_incremental): {entries, cross_rows} as int32, then fp32 self-attention K and V, each [mt_layers][entries][mt_dim]
 * (entry p + kv_off holds position p), then cross-attention K | V [mt_layers][cross_rows][2 * mt_dim].  bytes == 8 copies the two counts
 * alone; any other size below the whole state is SS_ERR_INVALID.  Synchronises the device. */
int ss_debug_copy(ss_engine* h, const char* what, void* host_dst, size_t bytes);
/* out rows r * ldy = LayerNorm(x rows r * ldx) * g + b over C columns (eps 1e-5) for r < rows.  Errors: SS_ERR_INVALID, before any
 * launch, for C outside {32, 64, .., 1024}, ldx or ldy < C, rows < 0 or a null pointer. */
int ss_op_layer_norm(ss_engine* h, void* stream, const float* x_dev, int ldx, int rows, int C, const float* g_dev, const float* b_dev,
                     float* out_dev, int ldy);
/* One GEMM of the engine's kernel layer with every field of its launch contract (kernels.h: ConvA, Epilogue), for the parity tests:
 *   A[m][tap * C_in + ci] = pre_lrelu(x[b][p - x_row0][ci]) with m = b * L_rows + t and p = (t + t_offset) * stride + tap * dil - pad_left,
 *   zero when p < 0, p >= L_in, p >= lengths[b], p outside [x_row0, x_row0 + x_rows) or (chunk > 0) p at or past the end of the chunk that
 *   holds (t + t_offset) * stride; x holds x_rows rows (0: L_in) of ldx floats per batch element;
 *   y = alpha * act(A W^T + bias) (glu: columns are (value, gate) pairs -> value * sigmoid(gate), N / 2 outputs), then
 *   + res_scale * residual[o] and + out[o] (accumulate), at o = row * ldo + column with row = b * out_L + t * out_row_stride +
 *   out_row_offset (out_L > 0) or m.  skinny_gemm only: A := LayerNorm(A) (ln_gamma / ln_beta, K = C_in), and split_n > 0 routes output
 *   column c to out / out2 / out3 by c / split_n (strides ldo / ldo2 / ldo3).
 * kernel: 0 = the engine's own choice for the shape (its linear routing for a plain B = 1 matrix, its conv routing otherwise, with the
 * handle's options), 1 = gemm_conv, 2 = skinny_gemm, 3 / 4 = umma2_conv with 2 / 3 bf16 pieces.  splitk: 0 = no split-K scratch (the
 * call never splits K), 1 = the handle's scratch.  lengths is a device array.  The route_* fields are written: the kernel taken,
 * gemm_conv's BM x BN tile, the split-K slices (1 = none), skinny's MR / KS / CPT / grid CTAs, umma2's BN / CK / UPT / SB.
 * Errors, before any launch: SS_ERR_INVALID for a shape or epilogue the chosen kernel cannot take (its *_supported rule, or for
 * gemm_conv: C_in, ldx not multiples of 4 or x, w not 16-byte aligned), a null pointer, or a kernel outside [0, 4].  enqueue only */
typedef struct ss_op_gemm_args {
  const float* x;
  const int32_t* lengths;
  int32_t B, L_in, L_rows, C_in, ldx, ksize, stride, dil, pad_left, chunk;
  float pre_lrelu;
  int32_t t_offset, x_row0, x_rows, k_tiles_per_split;
  const float* w;
  int32_t N;
  const float* bias;
  int32_t act, glu;
  float alpha;
  const float* residual;
  float res_scale;
  int32_t accumulate;
  float* out;
  int32_t ldo, out_L, out_row_stride, out_row_offset;
  const float* ln_gamma;
  const float* ln_beta;
  int32_t split_n;
  float* out2;
  float* out3;
  int32_t ldo2, ldo3;
  int32_t kernel, splitk;
  int32_t route_kernel, route_bm, route_bn, route_splits, route_mr, route_ks, route_cpt, route_grid, route_u_bn, route_u_ck, route_u_upt,
      route_u_sb;
} ss_op_gemm_args;
int ss_op_gemm(ss_engine* h, void* stream, ss_op_gemm_args* args);
/* The unit arg-max hook: logits_dev [rows][ld] -> idx_dev [rows] with the first n_masked (<= 3) of pad, unk, eos never selected,
 * through argmax_rows (lprob_dev NULL) or argmax_lprob_rows (lprob_dev [rows]: each winner's log_softmax over all V columns). */
int ss_op_argmax_rows(ss_engine* h, void* stream, const float* logits_dev, int rows, int V, int ld, int n_masked, int64_t* idx_dev, float* lprob_dev);
/* Attention and depthwise-conv hooks: each launches the launch function the engine uses (kernels.h) on `stream`; the hooks that take host arrays
 * copy them to the device and synchronise `stream`.  head_dim is 64 and D = H * 64; row strides are in floats, >= D and multiples
 * of 4.  kernel: 0 = the row / tile kernel the engine would choose for this shape, 1 = row kernel, 2 = tile kernel.
 * Errors: SS_ERR_INVALID for a null pointer or any shape outside what the kernels take; the handle stays usable. */
/* rel-pos self-attention: q rows b * nQ + r (absolute positions q_offset + r), k / v rows b * T + j, pos [2 * Tpos - 1][D] (row
 * (i - j) + Tpos - 1), out [B * nQ][D].  Needs T <= Tpos, q_offset + nQ <= T, chunk >= 0 (0 = full), lengths_host (optional) in
 * [1, T], and for kernel = 1, T * 4 bytes <= 160 KB. */
int ss_op_relpos_attention(ss_engine* h, void* stream, const float* q_dev, int ldq, const float* k_dev, int ldk, const float* v_dev, int ldv,
                           const float* pos_dev, int Tpos, const float* bias_u_dev, const float* bias_v_dev, float* out_dev, int B, int nQ,
                           int q_offset, int T, int H, int D, int chunk, const int32_t* lengths_host, int kernel);
/* multi-head attention: q rows b * Tq + t, k / v rows b * Tk + j; causal: key j visible to query t iff j <= t + causal_offset;
 * kv_len_host (optional) in [1, Tk]; for kernel = 1, Tk * 4 bytes <= 160 KB */
int ss_op_mha_attention(ss_engine* h, void* stream, const float* q_dev, int ldq, const float* k_dev, int ldk, const float* v_dev, int ldv, float* out_dev,
                        int ldo, int B, int Tq, int Tk, int H, float scale, int causal, int causal_offset, const int32_t* kv_len_host, int kernel);
/* causal self-attention over S groups of R identical rows (the unit decoder's first layer): q / k / v rows b * S + g, out rows
 * (b * S + g) * R + r; kv_len_host (optional) = valid groups per sample, in [1, S]; S <= 12288 */
int ss_op_grouped_causal_attention(ss_engine* h, void* stream, const float* q_dev, int ldq, const float* k_dev, int ldk, const float* v_dev, int ldv,
                                   float* out_dev, int ldo, int S, int R, int H, float scale, int B, const int32_t* kv_len_host);
/* chunk-causal depthwise conv (w [k][C], odd k) + folded BatchNorm (scale, shift [C]) + SiLU over x [B * T][ldx] at positions t0 .. t0 + n - 1
 * (t0 + n <= T) -> y rows b * n + r; chunk >= 0 (0 = no chunk) */
int ss_op_depthwise_bn_silu(ss_engine* h, void* stream, const float* x_dev, int ldx, const float* w_dev, const float* scale_dev, const float* shift_dev,
                            float* y_dev, int ldy, int B, int T, int t0, int n, int C, int k, int chunk);
/* the stream pool's ragged kernels over n streams: stream b uses slot slot_host[b] in [0, n_slots) of the slot buffers (slot_stride floats
 * apart; keys / conv inputs are rows of D / C floats), computes its rows a0 .. a0 + nA - 1 (0 <= nA <= T - a0) with its own chunk, and
 * reads / writes rows row0 .. row0 + nA - 1 of q / out / y (row0 + nA <= rows).  Relative-position attention needs T <= Tpos and
 * T * 4 bytes <= 160 KB. */
int ss_op_ms_relpos_attention(ss_engine* h, void* stream, const float* q_dev, int ldq, const float* kc_dev, const float* vc_dev, int64_t slot_stride,
                              int n_slots, const float* pos_dev, int Tpos, const float* bias_u_dev, const float* bias_v_dev, float* out_dev, int ldo,
                              int rows, int H, int n, const int32_t* slot_host, const int32_t* a0_host, const int32_t* nA_host, const int32_t* T_host,
                              const int32_t* attn_chunk_host, const int32_t* row0_host);
int ss_op_ms_depthwise(ss_engine* h, void* stream, const float* x_dev, int64_t slot_stride, int n_slots, const float* w_dev, const float* scale_dev,
                       const float* shift_dev, float* y_dev, int ldy, int rows, int C, int k, int n, const int32_t* slot_host, const int32_t* a0_host,
                       const int32_t* nA_host, const int32_t* T_host, const int32_t* conv_chunk_host, const int32_t* row0_host);

/* ---- ASR-BLEU transcriber: fairseq's Wav2VecCtc (wav2vec 2.0 + CTC letter projection), the `en` model of asr_bleu/asr_model_cfgs.json,
 * as asr_bleu/utils.py:247-288 runs it: model.w2v_encoder(audio, padding_mask)["encoder_out"], then torchaudio's ctc_decoder at
 * beam 1 without lexicon or LM.  A handle of its own: nothing is shared with an ss_engine.  Same conventions as above (caller-owned
 * device buffers, work on the caller's stream, negative codes + ss_asr_last_error, all state per handle).
 * Settings the state dict's shapes do not carry come from the checkpoint's stored cfg (or fairseq's defaults) through ss_asr_config;
 * everything outside the `en` model's family is refused at ss_asr_create with a message naming the setting. */
typedef struct ss_asr ss_asr;
#define SS_ASR_MAX_CONV 8
typedef struct ss_asr_config {
  int32_t n_conv;                        /* feature-extractor conv layers (conv_feature_layers), 1 .. SS_ASR_MAX_CONV */
  int32_t conv_stride[SS_ASR_MAX_CONV];  /* their strides (kernel sizes and widths come from the weights) */
  int32_t extractor_layer_norm;          /* extractor_mode: 1 = "layer_norm"; 0 = "default" (group norm) is refused */
  int32_t layer_norm_first;              /* 1 = pre-LN layers; 0 (post-LN) is refused */
  int32_t pos_conv_depth;                /* 1; deeper positional convs are refused */
  int32_t conformer;                     /* layer_type: 0 = "transformer"; 1 ("conformer") is refused */
  int32_t heads;                         /* encoder_attention_heads, 0 = dim / 64; a head dim other than 64 is refused */
  int32_t normalize;                     /* task.normalize: 1 = layer_norm over each whole waveform (eps 1e-5) before the extractor */
  int32_t max_frames;                    /* longest utterance in encoder frames (20 ms), 0 = 4096 (81.9 s at 16 kHz) */
  int32_t time_stages;                   /* 1: CUDA events around each stage (ss_asr_stage_ms); the call then synchronises per group */
} ss_asr_config;
/* Encoder frames are counted in launch groups of at most this many padded rows (B_group x longest T of the group); a longer single
 * utterance forms a group of its own.  The handle's workspace for a full group is about 2 GB at the Large shapes: the extractor's two
 * ping-pong buffers (conv layer 0 gives ~64 rows of C floats per encoder frame: ~1.07 GB + 0.54 GB at C = 512) and ~45 KB per encoder row. */
#define SS_ASR_BATCH_ROWS 8192
int ss_asr_create(ss_asr** out, int device, const ss_asr_config* cfg);
int ss_asr_destroy(ss_asr* h);
const char* ss_asr_last_error(const ss_asr* h); /* h == NULL: why this thread's last ss_asr_create was refused */
/* One fp32 tensor by its fairseq key as stored: "w2v_encoder.w2v_model.*" and "w2v_encoder.proj.*".  Keys the forward pass does not
 * read (mask_emb, quantizer, ...) are ignored.  pos_conv may come weight-normed (weight_g / weight_v, norm over dims 0 and 1) or folded. */
int ss_asr_load_tensor(ss_asr* h, const char* key, const float* data_host, int ndim, const int64_t* shape);
/* Takes every size from the shapes (conv kernels and widths, model dim, FFN, layers, positional-conv kernel and groups, vocabulary),
 * folds the weight norm, repacks and uploads.  SS_ERR_MISSING names the first missing key; SS_ERR_INVALID a shape the kernels do not take. */
int ss_asr_finalize(ss_asr* h);
/* encoder frames of an utterance of n samples: floor((L - k) / s) + 1 per conv layer (0 when some layer gets fewer than k frames);
 * -1 before ss_asr_finalize */
int64_t ss_asr_num_frames(const ss_asr* h, int64_t n_samples);
/* Transcribe B utterances: sample b is audio_dev[offsets_host[b] .. offsets_host[b + 1]) (fp32, 16-bit PCM scaled by 1/32768, at the
 * model's rate).  Per utterance: emissions = proj(encoder(extractor(audio))) [T_b][V]; arg-max of every row over the raw emissions with
 * <unk> (index 3) excluded, first index on ties (flashlight's lexicon-free beam-1 step with unk_score = -inf and no LM); then repeats
 * collapsed and blanks (index 0, "<s>") dropped (torchaudio CTCDecoder._get_tokens).
 * packed_out_dev: row b at b * packed_stride int64 words = [count (int32 in the first word) | tokens[count]]; packed_stride >= T_b + 1.
 * argmax_dev (optional) [sum T_b] int64 and emissions_dev (optional) [sum T_b][V] fp32: rows of the utterances in order.
 * Utterances run in launch groups (SS_ASR_BATCH_ROWS), padded to the group's longest; no GEMM splits K and the attention takes one
 * kernel for every shape, so an utterance's emissions are bit-identical to a call with that utterance alone.
 * Errors, before any launch: SS_ERR_STATE before finalize; SS_ERR_INVALID for B <= 0, a null pointer, decreasing offsets, an utterance
 * too short for one frame or a packed_stride below T_b + 1; SS_ERR_CAPACITY for T_b > max_frames.  Synchronises `stream` once per
 * launch group (upload of the lengths), and per stage when time_stages is set. */
int ss_asr_transcribe(ss_asr* h, void* stream, const float* audio_dev, const int64_t* offsets_host, int B, int64_t* packed_out_dev,
                      int64_t packed_stride, int64_t* argmax_dev, float* emissions_dev);
/* The activations after one stage of the same forward pass, rows of the utterances in order (test hook): stage 0 = extractor output
 * [sum T_b][C] (after the last conv block's GELU), 1 = feature LayerNorm + post_extract_proj [.][D], 2 = + positional conv [.][D],
 * 3 + l = after transformer layer l [.][D], 3 + layers = final LayerNorm [.][D], 4 + layers = emissions [.][V].  Errors as ss_asr_transcribe,
 * and SS_ERR_INVALID for a stage outside [0, 4 + layers]. */
int ss_asr_debug_stage(ss_asr* h, void* stream, const float* audio_dev, const int64_t* offsets_host, int B, int stage, float* out_dev);
/* {extractor, positional conv, transformer layers, final LayerNorm + proj + arg-max + collapse} device ms summed over the calls since
 * the last query (time_stages = 1; zeros otherwise), and resets them. */
int ss_asr_stage_ms(ss_asr* h, double* ms_out4);

/* number of kernels this library has launched in this process (bench.py reports the difference over the timed region as
 * gpu_launches; the counter is process-wide, not per handle) */
int64_t ss_launch_count(const ss_engine* h);
/* The persistent cooperative kernels (encoder layer stack, MT decode steps) separate their phases with a counter-based grid
 * barrier.  A barrier that times out (lost arrival, pre-empted CTA) raises a device flag instead of hanging or passing
 * silently; this call synchronises the device, returns SS_ERR_CUDA if the flag was raised since the last check (results of
 * the enqueue-only calls since then are invalid) and re-arms the barrier.  ss_mt_greedy performs the same check at its own
 * synchronisation point. */
int ss_async_error(ss_engine* h);

#ifdef __cplusplus
}
#endif
#endif /* STREAMSPEECH_B200_H_ */
