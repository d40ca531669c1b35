// Multi-stream (batched streaming) kernels, see kernels_multistream.cu.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace ss {

// One stream of a batched step (device array, one entry per batch element).
struct MsStream {
  int slot;          // pool slot: every per-stream buffer is base + slot * stride
  int a0;            // first active (not yet final) encoder row = rows final before this step
  int T;             // encoder rows after this step (keys 0 .. T-1)
  int F;             // fbank frames after this step
  int f_lo;          // first fbank frame the subsampler window of this step reads
  int frame0;        // fbank: first new frame
  int n_new_frames;  // fbank: number of new frames
  int n16_new;       // 48 kHz pools: 16 kHz samples the resampler produces in this step (0 in 16 kHz pools)
  int row0;          // encoder stack: first row of this stream in the step's concatenated active rows
  int nA;            // encoder stack: active rows of this stream (T - a0; 0 = nothing to encode)
  int attn_chunk;    // this stream's attention chunk (encoder rows)
  int conv_chunk;    // this stream's conv chunk (depthwise conv and subsampler)
  int64_t out_off;  // CTC collapse: int64 offset of this stream's packed output
  int64_t n48;       // 48 kHz pools: 48 kHz samples pushed to the slot so far
  int64_t n16_done;  // 48 kHz pools: first 16 kHz sample of this step (samples below it were produced by earlier steps)
};

void ms_gather_rows(const float* src_base, int64_t slot_stride, const MsStream* S, int n, int which /*0: rows from f_lo (limit F), 1: rows from a0 (limit T)*/,
                    int rows, int C, float* dst, cudaStream_t st);
// Ragged encoder-stack kernels: stream b's rows are rows S[b].row0 .. S[b].row0 + S[b].nA - 1 of the dense activations, and its
// chunk sizes come from S[b].  max_nA = the largest S[b].nA: the grid covers it and blocks past a stream's own nA exit at once.
void ms_scatter_rows(const float* s0, const float* s1, const float* s2, int lds, float* d0, float* d1, float* d2, int64_t slot_stride, const MsStream* S,
                     int n, int max_nA, int C, cudaStream_t st);
void ms_relpos_attention(const float* q, int ldq, const float* kc, const float* vc, int64_t slot_stride, int D, const float* pos, int Tpos,
                         const float* bias_u, const float* bias_v, float* out, int ldo, const MsStream* S, int n, int max_nA, int H, int Tmax,
                         cudaStream_t st);
void ms_depthwise(const float* gc, int64_t slot_stride, const float* w, const float* scale, const float* shift, float* y, int ldy, const MsStream* S, int n,
                  int max_nA, int C, int k, cudaStream_t st);
void ms_fbank(const float* audio_base, int64_t audio_stride, float* feat_base, int64_t feat_stride, const MsStream* S, int n, int max_new_frames,
              const float* melT /*[257][80]*/, const float* window, const float* cmvn_mean, const float* cmvn_std, cudaStream_t st);
// 48 -> 16 kHz decimation of every stream's new samples: a16_base[slot * a16_stride + i] for i in [n16_done, n16_done + n16_new) from
// a48_base[slot * a48_stride + 0 .. n48) (resample_3to1 of kernels.h per stream; max_new = largest n16_new)
void ms_resample_3to1(const float* a48_base, int64_t a48_stride, float* a16_base, int64_t a16_stride, const MsStream* S, int n, int max_new,
                      const float* h, int taps, int width, cudaStream_t st);
void ms_ctc_argmax(const float* logits, int ld, int V, const int* masked, int n_masked, int64_t* am_base, int64_t am_stride, const MsStream* S, int n,
                   int max_nA, int heads, cudaStream_t st);
void ms_ctc_collapse(const int64_t* am_base, int64_t am_stride, const MsStream* S, int n, int heads, int blank, int pad, int64_t* out, cudaStream_t st);

}  // namespace ss
