// Persistent cooperative encoder-stack kernel (kernels_persist.cu): one launch per streaming step for all layers.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace ss {

// word of the barrier buffer (unsigned[64]: [0] = arrival counter) that a timed-out grid barrier raises
#define SS_BAR_ERR_WORD 32

#ifdef __CUDACC__
// Grid barrier of the persistent cooperative kernels, on a monotonic arrival counter (one red.release per CTA, relaxed polling,
// one acquire fence at the end).  `target` is the counter value that marks "every CTA has arrived at this barrier"; the host
// carries it across launches.
__device__ __forceinline__ void grid_barrier(unsigned* ctr, unsigned& target) {
  __syncthreads();
  target += gridDim.x;
  if (threadIdx.x == 0) {
    asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(ctr) : "memory");
    unsigned v, spins = 0;
    do {  // (bounded: a counter out of step with the host's target must not hang the device)
      asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(ctr) : "memory");
    } while ((int)(v - target) < 0 && ++spins < (1u << 20));
    // A counter that never reaches the target (lost arrival, counter out of step with the host's target) must neither hang
    // the device nor pass silently: the word ctr[SS_BAR_ERR_WORD] is raised and the host reports it at its next
    // synchronisation point (ss_async_error / ss_mt_greedy), after which results of this launch are invalid.
    if ((int)(v - target) < 0) atomicExch(ctr + SS_BAR_ERR_WORD, 1u);
    asm volatile("fence.acq_rel.gpu;" ::: "memory");
  }
  __syncthreads();
}
// split form of the grid barrier: arrive publishes this CTA's writes; everything issued between arrive and wait (the next phase's
// weight, bias and LayerNorm-parameter loads: they do not depend on the phase that just ended) flies while the other CTAs arrive
__device__ __forceinline__ void grid_arrive(unsigned* ctr, unsigned& target) {
  __syncthreads();
  target += gridDim.x;
  if (threadIdx.x == 0) asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(ctr) : "memory");
}
__device__ __forceinline__ void grid_wait(unsigned* ctr, unsigned target) {
  if (threadIdx.x == 0) {
    unsigned v, spins = 0;
    do {
      asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(ctr) : "memory");
    } while ((int)(v - target) < 0 && ++spins < (1u << 20));
    if ((int)(v - target) < 0) atomicExch(ctr + SS_BAR_ERR_WORD, 1u);
    asm volatile("fence.acq_rel.gpu;" ::: "memory");
  }
  __syncthreads();
}
#endif

struct PersistLayer {  // device pointers of one Conformer layer (fp32, layouts as in engine.h ConformerLayerW)
  const float *ffn1_g, *ffn1_b, *ffn1_w1, *ffn1_b1, *ffn1_w2, *ffn1_b2;
  const float *attn_g, *attn_b, *wqkv, *bqkv, *wo, *bo, *pos_u, *pos_v, *pos_proj;
  const float *conv_g, *conv_b, *pw1, *pw1_b, *dw_w, *bn_scale, *bn_shift, *pw2, *pw2_b;
  const float *ffn2_g, *ffn2_b, *ffn2_w1, *ffn2_b1, *ffn2_w2, *ffn2_b2;
  const float *fin_g, *fin_b;
  const float *ffn1_w2t, *ffn2_w2t;   // W2 transposed [FFN][D] (fused FFN phases of kernels_persist.cu)
};

bool encoder_layers_persistent_supported(int nA, int D, int FFN, int H, int T, int dw_k);
// returns 0 on success (kernel enqueued on `st`), < 0 if the cooperative launch was refused
int encoder_layers_persistent(const PersistLayer* layers_dev, int n_layers, float* x, float* hid, float* qb, float* att, float* dw, float* kc,
                              float* vc, float* gc, int nA, int a0, int T, int D, int FFN, int H, int Tpos, int chunk, int conv_chunk, int dw_k,
                              unsigned long long* timestamps_or_null, unsigned* barrier_counter_dev_or_null,
                              unsigned* barrier_target_host, int prefetch /*0 off, 1 next layer, 2 also layer 0*/,
                              float* ffn_scratch_or_null /* [FFN/16][16][D]: fused FFN phases; nullptr = W1 / W2 phases */, cudaStream_t st);

// ---- cluster version of the encoder step (kernels_persist_cl.cu): 4 clusters x 16 CTAs, activations in distributed shared memory,
// weights streamed from per-(layer, rank) blobs.  nA <= 16 rows.
size_t encoder_layers_cluster_blob_floats(int n_layers);
void encoder_layers_cluster_pack(const PersistLayer* layers_dev, int n_layers, int dw_k, float* blobs_dev, cudaStream_t st);
bool encoder_layers_cluster_supported(int nA, int D, int FFN, int H, int T, int dw_k);
int encoder_layers_cluster(const PersistLayer* layers_dev, const float* blobs_dev, int n_layers, float* x, float* kc, float* vc, float* gc, int nA,
                           int a0, int T, int Tpos, int chunk, int conv_chunk, int dw_k, unsigned* bar_ctr, unsigned* bar_target_host,
                           unsigned long long* ts_or_null, const float* const* pos_proj_host /* n_layers (<= 16) device pointers */, int cooperative /* 1; 0 only under a profiler that cannot replay cooperative cluster launches */,
                           cudaStream_t st);

// ---- MT decoder, single-token greedy steps (kernels_persist_mt.cu)
struct MtLayerP {  // device pointers of one pre-LN decoder layer (fp32, [N][K] weights)
  const float *self_g, *self_b, *wqkv, *bqkv, *wo, *bo;
  const float *cross_g, *cross_b, *wcq, *bcq, *wco, *bco;
  const float *fin_g, *fin_b, *w1, *b1, *w2, *b2;
};
struct MtDecodeParams {
  int n_layers, heads, vocab, pad, eos, max_pos, cross_cap;
  int kv_off = 0;                           // self-attention cache slot of the token at position s is s + kv_off (> 0 only in the
                                            // reference's incremental-state mode, where call boundaries duplicate an entry)
  const float *emb, *pos, *out_g, *out_b;   // tied embedding / output projection [vocab][dim], sinusoidal table, final LN
  float *self_k, *self_v;                   // [layers][max_pos][dim]
  const float* cross_kv;                    // [layers][cross_cap][2 * dim] (K | V per row)
  int64_t* tok;                             // device token buffer: tok[s] is fed at step s, the arg-max goes to tok[s + 1]
  float* feats;                             // [.][dim] final-LN features, row s
  float *x, *q, *attn, *hid, *logits;       // scratch: dim, dim, dim, ffn, vocab floats
  unsigned long long* ts = nullptr;         // profiling (option persistent_profile): ns stamps of CTA 0 for the 2nd step's layer 1
  float *part = nullptr, *delta = nullptr;  // version-2 step (6 barriers per layer): per-head out-projection partials [8][dim], FFN delta [dim];
                                            // nullptr selects the 8-barrier kernel
};
bool mt_decode_persistent_supported(int dim, int ffn, int heads, int vocab, int max_pos, int T);
// enqueue `nsteps` greedy steps starting with the token at position step0; returns 0, or < 0 if the launch was refused
int mt_decode_persistent(const MtDecodeParams& P, const MtLayerP* layers_dev, int step0, int nsteps, int max_len, int T,
                         unsigned* barrier_counter_dev, unsigned* barrier_target_host, cudaStream_t st);

// ---- MT decoder, greedy search of up to MT_BATCH_MAX_ROWS independent samples per launch (kernels_persist_mtb.cu)
#define MT_BATCH_MAX_ROWS 32
struct MtBatchParams {
  int n_layers, vocab, pad, eos;
  int rows;                                 // rows of this launch (<= MT_BATCH_MAX_ROWS)
  int tok_ld;                               // row stride of tok and of the self-attention cache (> the last step fed)
  int cross_cap;                            // rows per sample in cross_kv
  const float *emb, *pos, *out_g, *out_b;   // as MtDecodeParams
  float *self_k, *self_v;                   // [layers][MT_BATCH_MAX_ROWS][tok_ld][dim]
  const float* cross_kv;                    // [layers][MT_BATCH_MAX_ROWS][cross_cap][2 * dim] (K | V per encoder row)
  const int* cross_len;                     // [rows] encoder rows of each sample
  int64_t* tok;                             // [rows][tok_ld]: tok[b][s] is fed at step s, the arg-max goes to tok[b][s + 1]
  int* fin;                                 // [rows]: set once the row produced eos; finished rows are skipped
  float *q, *part, *delta, *hid, *logits;   // scratch per row: dim, 8 x dim, dim, ffn, vocab floats
};
// enqueue steps step0 .. step0 + nsteps - 1 (all < max_len: the forced-eos step needs no work) for every unfinished row;
// returns 0, or < 0 if the launch was refused
int mt_decode_batch(const MtBatchParams& P, const MtLayerP* layers_dev, int step0, int nsteps, unsigned* barrier_counter_dev,
                    unsigned* barrier_target_host, cudaStream_t st);

// ---- MT decoder, prefix pass over M <= 64 rows (kernels_persist_mtp.cu): fills self-attention cache rows 0 .. M-1 and feature
// rows 0 .. M-1 from P.tok[0 .. M-1]; P.x / P.q / P.attn hold M x dim floats, P.hid M x ffn
bool mt_prefix_persistent_supported(int dim, int ffn, int heads, int M, int T);
int mt_prefix_persistent(const MtDecodeParams& P, const MtLayerP* layers_dev, int M, int T, unsigned* barrier_counter_dev,
                         unsigned* barrier_target_host, cudaStream_t st);

}  // namespace ss
