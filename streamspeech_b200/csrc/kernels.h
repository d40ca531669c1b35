// Internal C++ launch API of the sm_90a kernels (streamspeech_b200/csrc/kernels_*.cu).
// Everything enqueues on the given stream and never synchronises.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <map>
#include <tuple>
#include <vector>

namespace ss {

extern unsigned long long g_launches;  // kernels launched by this library (process-wide)

enum Act : int { ACT_NONE = 0, ACT_RELU = 1, ACT_SILU = 2, ACT_TANH = 3 };

// A-operand of a GEMM viewed as a 1-D convolution over a channels-last activation
// x[B][L_in][C_in]:  A[m][tap*C_in + ci] = pre(x[b][t*stride + tap*dil - pad_left][ci]),
// m = b*L_rows + t, zero outside [0, L_in) and (chunk-causal) at or beyond the end of the
// chunk that holds t*stride.  A plain row-major matrix is ksize=1, stride=1, pad_left=0.
struct ConvA {
  const float* x = nullptr;
  int B = 1;         // batch
  int L_in = 0;      // rows per batch element in x
  int L_rows = 0;    // GEMM rows per batch element (M = B * L_rows)
  int C_in = 0;      // channels (row length of x is ldx)
  int ldx = 0;       // row stride of x in floats (>= C_in)
  int ksize = 1;
  int stride = 1;
  int dil = 1;
  int pad_left = 0;
  int chunk = 0;           // >0: chunk-causal masking (ChunkCausalConv1d semantics)
  float pre_lrelu = 1.0f;  // leaky-relu slope applied while loading A (1 = identity)
  const int* lengths = nullptr;  // optional per-batch valid length of x rows (rows >= length read as zero)
  // windowed (streaming) use: GEMM row 0 is logical output position t_offset, and buffer row 0 of x is logical
  // input position x_row0 (x holds x_rows rows per batch element; 0 = L_in).  Masks use logical positions.
  int t_offset = 0;
  int x_row0 = 0;
  int x_rows = 0;
  // > 0 (gemm_conv): split-K slices of this many k-tiles whatever M is, so that a row's sum does not depend on how many rows the
  // call has (0: the slice count is chosen to fill the GPU)
  int k_tiles_per_split = 0;
};

struct Epilogue {
  const float* bias = nullptr;      // [N]
  int act = ACT_NONE;
  int glu = 0;                      // 1: columns are interleaved (a, gate) pairs -> N/2 outputs a*sigmoid(gate)
  float alpha = 1.0f;               // y = alpha * act(acc + bias)
  const float* residual = nullptr;  // y += res_scale * residual[out index]
  float res_scale = 1.0f;
  int accumulate = 0;               // y += previous out value
  float* out = nullptr;
  int ldo = 0;                      // row stride of out in floats
  // output row of GEMM row m = b*L_rows + t is  b*out_L + t*out_row_stride + out_row_offset
  int out_L = 0;
  int out_row_stride = 1;
  int out_row_offset = 0;
  // ---- skinny-GEMM-only fusions (engine checks skinny_gemm_supported before setting them)
  // A := LayerNorm(A) over the K columns (eps 1e-5) applied while loading A; K must be the full row width
  const float* ln_gamma = nullptr;
  const float* ln_beta = nullptr;
  // column routing: columns [p*split_n, (p+1)*split_n) go to out / out2 / out3 (fused Q|K|V projections writing
  // straight into the query buffer and the K / V caches)
  int split_n = 0;
  float* out2 = nullptr;
  float* out3 = nullptr;
  int ldo2 = 0, ldo3 = 0;
};

// C[M,N] = epilogue( A[M,K] * W[N,K]^T ), K = ksize*C_in, W row-major with K contiguous.
// splitk: the caller's split-K scratch region (nullptr: never split), see splitk_workspace.
void gemm_conv(const ConvA& a, const float* W, int N, const Epilogue& ep, float** splitk, cudaStream_t st);

// Split-K scratch: *splitk is a region of splitk_workspace_bytes() that the first GEMM splitting into it allocates and its owner
// frees; the launches that share a region must be stream-ordered.  Returns the region when `bytes` fit it (nullptr: no region,
// request too large or out of memory).
float* splitk_workspace(float** splitk, size_t bytes);
size_t splitk_workspace_bytes();  // capacity of one split-K scratch region
// fixed-order reduce of the split-K partial sums + epilogue
void splitk_epilogue(const float* ws, int splits, int M, int N, int L_rows, const Epilogue& ep, cudaStream_t st);

// wgmma path (kernels_umma2.cu): stride-1 convolutions / linears over one sequence (B = 1) with
// pre-packed bf16-split weights streamed by cp.async.bulk and activations converted once per channel chunk (taps are
// descriptor row shifts).  The cache owns the packed weight copies (keyed by weight pointer and tiling).
struct Umma2Cache {
  std::map<std::tuple<const float*, int, int, int, int, int, int>, unsigned char*> packed;
  std::vector<void*> allocs;
  unsigned long long* dbg = nullptr;  // optional device buffer of 16 %globaltimer stamps of CTA (0,0,0) (freed by umma2_cache_destroy)
};
void umma2_cache_clear(Umma2Cache* c);  // frees the packed weights
void umma2_cache_destroy(Umma2Cache* c);
bool umma2_supported(const ConvA& a, int N, const Epilogue& ep);
void umma2_conv(Umma2Cache* cache, const ConvA& a, const float* W, int N, const Epilogue& ep, int pieces, float** splitk, cudaStream_t st);
// packed copy of W[N][ksize*C_in] in the kernels' tiling (made once per weight matrix and tiling; nullptr when out of memory)
const unsigned char* umma2_packed_weights(Umma2Cache* cache, const float* W, int N, int C_in, int ksize, int BN, int CK, int NP, cudaStream_t st);

// ---- the vocoder generator of up to VOC_MAX_STREAMS sequences as one persistent cooperative wgmma kernel (kernels_umma2.cu, bf16x3)
// One job = one stride-1 convolution of the generator, tiled per sequence into 128-row x BN-column work items:
//   out[m * out_row_stride + out_row_offset][n] = alpha * (sum_{j, ci} pre(x[m + j*dil - pad_left][ci]) * W[n][j][ci] + bias[n])
//                                                + res_scale * residual[same index]
// with x = x0, or x2 + (x1 + x0) when x1 != nullptr (the sum of a stage's three resblock outputs), pre = leaky_relu(slope).
// The job table holds each convolution once.  Sequence s of N_s frames owns rows [row0_s * in_mult, (row0_s + N_s) * in_mult) of
// the job's input buffer and the matching rows (x out_row_stride) of its output: the kernel resolves L_in, M, the row bases and the
// tile width of (job, sequence) from the sequence's VocStreamGeo, so every sequence gets the tiles a call of its own would run.
struct VocJob {
  const float *x0, *x1, *x2;
  int C_in, ksize, dil, pad_left;
  float slope;
  const unsigned char* wp;              // the fp32 weights W (the host packs them per tile width into wp16 / wp32 when first used)
  const unsigned char *wp16, *wp32;     // umma2_packed_weights(W, N, C_in, ksize, BN = 16 / 32, CK, 2) (nullptr when unused)
  const float* bias;
  float* out;
  int N, out_row_stride, out_row_offset;
  const float* residual;
  float alpha, res_scale;
  int CK;
  // per sequence: L_in = N_s * in_mult, M = L_in + m_adj (upsample phases skip the rows their output phase does not own); output
  // rows start at row0_s * in_mult * out_row_stride
  int in_mult, m_adj;
};
struct VocPhase {  // jobs [first_job, first_job + n_jobs) are independent; items of the phase = sum over sequences of m_tiles * n_tiles
  int first_job, n_jobs, n_items;
};
// per sequence: N frames at row0 of the packed frame buffer; conv_post computes samples [t0, N * hop), numbered from out0 among
// all sequences' samples, into out[dst ..); bit ph of bn32 = the 32-column tile width in phase ph (the choice a call with this
// sequence alone makes)
struct VocStreamGeo {
  unsigned long long bn32;
  int N, row0, t0, out0, dst;
};
// last phase, per sequence: out[t - t0] = tanh(bias + sum_{j, c} w[j][c] * leaky_relu(x2 + (x1 + x0))[t + j - (k-1)/2][c])
// for t in [t0, L = N * hop), with x rows counted from row0 * hop
struct VocPost {
  const float *x0, *x1, *x2;
  const float* w;  // [k][C]
  float bias, slope;
  int hop, C, k, total;  // total = samples written by all sequences
  float* out;
};
constexpr int VOC_FUSED_BM = 128;
constexpr int VOC_MAX_JOBS = 128, VOC_MAX_PHASES = 40, VOC_MAX_STREAMS = 32;
struct VocFusedParams {  // passed by value in the kernel's parameter space (< 32 KB): no per-call upload
  VocJob jobs[VOC_MAX_JOBS];
  VocPhase phases[VOC_MAX_PHASES];
  int n_phases, n_streams;
  int a_stride, b_stride;  // shared-memory bytes of one A stage (rows x channels x pieces) / one B stage (all taps of a chunk)
  VocPost post;
  VocStreamGeo streams[VOC_MAX_STREAMS];
  int item0[VOC_MAX_PHASES][VOC_MAX_STREAMS];  // first work item of sequence s in phase ph
};
static_assert(VOC_MAX_PHASES <= 64, "VocStreamGeo::bn32 has one bit per phase");
static_assert(sizeof(VocFusedParams) <= 32000, "the fused vocoder parameters must fit the 32 KB kernel parameter space");
// CTAs of the cooperative launch on the current device (0: the kernel cannot be made resident)
int vocoder_fused_grid();
size_t vocoder_fused_smem(int a_stride, int b_stride);
// returns 0 (enqueued; the barrier target advanced by grid x n_phases) or < 0 (launch refused)
int vocoder_fused(const VocFusedParams& p, unsigned* bar_ctr, unsigned* bar_target_host, cudaStream_t st);

// Per-sequence geometry of the vocoder's ragged front end (kernels_misc.cu), passed by value.
struct VocSeqs {
  int n;
  struct {
    int u0;     // first unit row of the sequence in the unit-embedding / log-duration buffers
    int U;      // units
    int c0;     // first entry of its cumsum [U + 1] in the packed cumsum buffer (durations: also dur_out[c0 - s ..])
    int f_lo;   // expand: first frame
    int N;      // expand: frames
    int row0;   // expand: first output row
  } s[VOC_MAX_STREAMS];
};
// emb rows u0_s + [0, U_max) = table[codes[packed offset of s + i]] for i < U_s, zero rows for i in [U_s, rows_per_seq)
void gather_codes_ragged(const int64_t* codes, const VocSeqs& q, int rows_per_seq, const float* table, int C, float* emb, cudaStream_t st);
// zero rows [U_s, rows_per_seq) of sequence s (rows u0_s ..) of x [.][C]
void zero_pad_rows(float* x, const VocSeqs& q, int rows_per_seq, int C, cudaStream_t st);
// per sequence: dur = clamp(round(exp(logdur) - 1), min 1) (round half to even like torch.round; logdur == nullptr: every
// duration is 1) into dur[c0_s - s ..], and its inclusive prefix sum into cumsum[c0_s .. c0_s + U_s] (one CTA per sequence)
void duration_from_log_ragged(const float* logdur, const VocSeqs& q, int64_t* dur, int* cumsum, cudaStream_t st);
// out rows row0_s + i = emb[u0_s + unit of frame f_lo_s + i] for i < N_s (repeat_interleave via the cumsum at c0_s)
void expand_frames_ragged(const float* emb, const int* cumsum, const VocSeqs& q, int total_rows, int C, float* out, cudaStream_t st);

// Weight-streaming GEMM for M <= 64 rows (plain row-major A): one warp per output column, see kernels_skinny.cu.
bool skinny_gemm_supported(int M, int N, int K, const Epilogue& ep);
void skinny_gemm(const float* A, int lda, const float* W, int M, int N, int K, const Epilogue& ep, cudaStream_t st);

// y[r] = LayerNorm(x[r]) * gamma + beta, rows of length C (C <= 1024, multiple of 32)
void layer_norm(const float* x, int ldx, float* y, int ldy, const float* gamma, const float* beta, int rows, int C,
                cudaStream_t st);

// Kaldi fbank + global CMVN for frames [f0, f0+nf) of a 16 kHz signal (already on device, NOT scaled by 2^15).
void fbank_cmvn(const float* samples, int64_t n_samples, int f0, int nf, const float* mel_bank /*[80][257]*/,
                const float* window /*[400]*/, const float* cmvn_mean, const float* cmvn_inv_std_or_null,
                const float* cmvn_std, float* out /*[nf][80]*/, cudaStream_t st);

// the same frames with the sample window staged by cp.async.bulk (TMA 1-D) and the mel bank transposed to [257][80]; `samples`
// must be 16-byte aligned and hold every requested frame completely
void fbank_cmvn_tma(const float* samples, int f0, int nf, const float* melT, const float* window, const float* cmvn_mean, const float* cmvn_std,
                    float* out, cudaStream_t st);

// Relative-position self-attention of the chunk-Conformer (espnet_multihead_attention.py:154-209).
// q: [B*nQ][ldq] rows for absolute query positions q_offset .. q_offset+nQ-1; k, v: [B*T][ld] rows for absolute
// key positions 0..T-1; pos: [2*Tpos-1][D] rows indexed by (i-j) + Tpos-1; out: [B*nQ][D].
// Full recompute: q = qkv, k = qkv + D, v = qkv + 2D, ld* = 3D, q_offset = 0, nQ = T.
// kernel: 0 = row or tile kernel by the shape rule of kernels_attn.cu; 1 = row kernel (T * 4 bytes <= 160 KB), 2 = tile kernel
// (the forced choices exist for the parity tests)
void relpos_attention(const float* q, int ldq, const float* k, int ldk, const float* v, int ldv, const float* pos, int Tpos,
                      const float* bias_u, const float* bias_v, float* out, int B, int nQ, int q_offset, int T, int H, int D,
                      int chunk /*0 = full*/, const int* lengths_dev, cudaStream_t st, int kernel = 0);

// Standard multi-head attention, head_dim 64.  q rows = b*Tq + t, k / v rows = b*Tk + j.  kv_len[b] (device, optional) masks
// keys >= len.  causal: key j visible to query i iff j <= i + causal_offset.  Each sample gets the same kernel and arithmetic
// as a call with B = 1.  kernel: as relpos_attention's.
void mha_attention(const float* q, int ldq, const float* k, int ldk, const float* v, int ldv, float* out, int ldo, int B,
                   int Tq, int Tk, int H, float scale, int causal, int causal_offset, const int* kv_len_dev,
                   cudaStream_t st, int kernel = 0);

// Causal self-attention over S groups of R identical consecutive rows (unit decoder layer 1, see kernels_attn.cu), for B samples:
// q / k / v hold each sample's S distinct rows (rows b*S + g), out gets S*R rows per sample (rows (b*S + g)*R + r).
// kv_len[b] (device, optional) = number of valid (non-pad) groups of sample b.
void grouped_causal_attention(const float* q, int ldq, const float* k, int ldk, const float* v, int ldv, float* out, int ldo, int S, int R,
                              int H, float scale, const int* kv_len_dev, int B, cudaStream_t st);

// depthwise chunk-causal conv (k taps, left context (k-1)/2) + folded BatchNorm + SiLU, channels-last.
// x: [B*T][C] (absolute positions 0..T-1); computes positions t0..t0+n-1 into y rows 0..n-1 per batch element.
void depthwise_bn_silu(const float* x, int ldx, const float* w /*[k][C]*/, const float* scale, const float* shift,
                       float* y, int ldy, int B, int T, int t0, int n, int C, int k, int chunk, cudaStream_t st);

// misc elementwise / gather kernels
void scale_rows(float* x, int64_t n, float s, cudaStream_t st);
void embed_tokens_pos(const int64_t* tokens, const int* positions_or_null, int pos_offset, const float* emb,
                      const float* pos_table, float scale, float* out, int rows, int C, int pad_idx, cudaStream_t st);
// x [B*S][C] -> out [B*S*R][C]: every row repeated R times, plus row b of addvec [B][C] for sample b (N1 quirk, see the kernel)
void repeat_rows_add(const float* x, int S, int R, int C, const float* addvec_or_null, float* out, int B, cudaStream_t st);
// arg-max of log_softmax over V columns of every row, masked columns excluded, first index wins on ties
void argmax_rows(const float* logits, int ld, int rows, int V, const int* masked_cols, int n_masked, int64_t* out_idx, cudaStream_t st);
// CTC collapse (dedup consecutive, drop blank/pad) of n_seg sequences of n entries, one CTA each.  Sequence s reads
// argmax[((s / inner) * n + i) * inner + s % inner] (inner = 2: the arg-max rows of two heads interleaved) and writes
// out_tokens + s * seg_stride, and out_index (optional) / out_count + 2 * s * seg_stride (seg_stride in int64 words, so that one
// packed buffer holds every sequence's output; a single sequence passes n_seg = 1, inner = 1).  n_seq_dev (device, optional): sample
// s / inner has only its first n_seq_dev[s / inner] entries (ragged lengths at a common stride n).
void ctc_collapse_segments(const int64_t* argmax, int n, int inner, int n_seg, int blank, int pad, int64_t* out_tokens, int* out_index,
                           int* out_count, int64_t seg_stride, cudaStream_t st, const int* n_seq_dev = nullptr);
// both CTC heads: arg-max of the new rows [row0, row0 + n_new) from logits [n_new][ld] (head h at columns h*V..), then collapse
// of all n_rows rows of both arg-max arrays into out[head] = [count | tokens[n_rows] | index[n_rows] (int32)]
void ctc_argmax_collapse_pair(const float* logits, int ld, int V, int n_new, int row0, int n_rows, const int* masked, int n_masked, int blank,
                              int pad, int64_t* am0, int64_t* am1, int64_t* out, int out_stride, unsigned* ticket, cudaStream_t st);
void gather_rows(const int64_t* idx, int n, int idx_offset, const float* table, int C, float* out, cudaStream_t st);
// conv_post (C_in -> 1, k taps, "same" padding) + leaky_relu(slope) on the input + tanh
void conv_post_tanh(const float* x, int L, int C, const float* w /*[k][C]*/, float bias, int k, float pre_slope, float* out,
                    cudaStream_t st);
void copy_f32(const float* src, float* dst, int64_t n, cudaStream_t st);
// 48 kHz -> 16 kHz: out[i] = sum_k h[k] * x[3 i + k - width] for i in [i0, i0 + n) (taps <= 64); out is indexed by absolute i
void resample_3to1(const float* x, int64_t n_in, const float* h, int taps, int width, int64_t i0, int n, float* out, cudaStream_t st);
// out = c + (b + a), elementwise (n % 4 == 0): joins the vocoder's three resblock streams in the reference's summation order
void add3_f32(const float* a, const float* b, const float* c, float* out, int64_t n, cudaStream_t st);

}  // namespace ss
