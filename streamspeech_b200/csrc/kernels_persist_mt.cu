// Persistent cooperative kernel for the single-token steps of the MT decoder's greedy search (beam 1).
//
// One decode step is a chain of ~37 dependent M = 1 operations (4 pre-LN layers of self-attention, cross-attention and
// FFN, the tied output projection over 6000 entries and the arg-max); as separate kernels its time per token is
// nearly all kernel boundaries.  This kernel keeps one CTA per SM resident for a whole burst
// of steps and separates the phases with the counter barrier of kernels_persist.h, 6 per layer (25 per token):
//   per layer: [LN + QKV] | [self-attn + Wo partials] | [x += sum, LN + Wcq] | [cross-attn + Wco partials] |
//              [x += sum, LN + FC1 + ReLU] | [FC2 -> delta]          (next layer / final LN: x += delta)
//   then:      [final LN -> features row, logits = E @ feat] | arg-max of log_softmax (every CTA redundantly) + embedding
// Attention and its out-projection share a phase: the 16 CTAs of a head group each compute the (tiny, M = 1) attention of
// their head redundantly and then the PARTIAL out-projection of their 32 output columns over that head's 64 inputs; the 8
// per-head partial vectors are summed (fixed order) by every CTA while it stages the next phase, together with bias and
// residual, so the residual stream x lives in shared memory of every CTA and is never exchanged.  Same for the
// cross-attention block; the FFN output is handed over the same way (one 512-vector).  The "v2" in the kernel's
// name stands for this 6-barrier design.
// GEMV phases give each warp up to MAXC output columns and issue all weight loads before the reduction.
// Semantics follow ss_mt_greedy's per-kernel path (sequence_generator.py:generate_decoder with beam 1): pad is always
// masked, eos only while step < min_len (= 1), eos is forced at max_len (no logits are computed for that step).
#include "kernels_persist_mt.cuh"

namespace ss {
namespace {

// the out-projection weights head_partial_proj multiplies with, loaded before the attention they follow
struct HpW {
  float w0[PCOLS_PER_WARP], w1[PCOLS_PER_WARP];
};

// partial[h][32 j + c] = sum_{i < 64} a[i] * W[(32 j + c)][64 h + i]   (W row-major [512][512]); a = this CTA's attention output;
// the weights are loaded (hp_load) before the attention they follow
__device__ __forceinline__ HpW hp_load(const float* __restrict__ W, int h, int j) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  HpW r;
#pragma unroll
  for (int c = 0; c < PCOLS_PER_WARP; ++c) {
    const float* w = W + (int64_t)(j * PCOLS + warp * PCOLS_PER_WARP + c) * 512 + h * MHD;
    r.w0[c] = __ldg(w + lane);
    r.w1[c] = __ldg(w + lane + 32);
  }
  return r;
}
__device__ __forceinline__ void head_partial_proj_w(const float* a, const HpW& hw, int j, float* part_h) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const float a0 = a[lane], a1 = a[lane + 32];
#pragma unroll
  for (int c = 0; c < PCOLS_PER_WARP; ++c) {
    const float acc = head_col_partial(a0, a1, hw.w0[c], hw.w1[c]);
    if (lane == 0) part_h[j * PCOLS + warp * PCOLS_PER_WARP + c] = acc;
  }
}

__global__ void __launch_bounds__(MTT, 1) mt_decode_persistent_kernel_v2(MtDecodeParams P, const MtLayerP* __restrict__ layers, int step0,
                                                                         int nsteps, int max_len, int T, unsigned* bar_ctr,
                                                                         unsigned bar_target) {
  __shared__ __align__(16) MtSmem sm;
  __shared__ __align__(16) float att_h[MHD];
  constexpr int DIM = 512, FFN = 2048;
  const int tid = threadIdx.x;
  const int barriers_per_step = P.n_layers * 6 + 1;
  int done_barriers = 0;
  const float emb_scale = sqrtf((float)DIM);
  const int grp_h = blockIdx.x / GRP, grp_j = blockIdx.x % GRP;
  const bool in_group = blockIdx.x < 8 * GRP;
  float* part = P.part;    // [8][512]
  float* delta = P.delta;  // [512]
#define BAR()                          \
  grid_barrier(bar_ctr, bar_target);   \
  ++done_barriers;
#define ARRIVE()                       \
  grid_arrive(bar_ctr, bar_target);    \
  ++done_barriers;
#define WAIT() grid_wait(bar_ctr, bar_target)
  int nts = 0;
  bool stamping = false;
#define STAMP(id)                                          \
  if (stamping && tid == 0) {                              \
    unsigned long long t_;                                 \
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t_)); \
    P.ts[1 + 2 * nts] = (id);                              \
    P.ts[2 + 2 * nts] = t_;                                \
    ++nts;                                                 \
    P.ts[0] = nts;                                         \
  }
  for (int si = 0; si < nsteps; ++si) {
    const int s = step0 + si;
    {
      const int64_t tok = (si == 0) ? P.tok[s] : (int64_t)sm.tok;
      const int p = (tok == P.pad) ? P.pad : P.pad + 1 + s;
      for (int c = tid; c < DIM; c += MTT) sm.x[c] = emb_scale * P.emb[tok * DIM + c] + P.pos[(int64_t)p * DIM + c];
      __syncthreads();
    }
    GemvW<DIM, 2> w_qkv;  // weights of phase (1): issued at the start of the step (layer 0) or before the previous layer's last wait
    LnP ln_self;
    {
      const MtLayerP L0 = layers[0];
      gemv_issue_b(w_qkv, L0.wqkv, 3 * DIM, L0.bqkv);
      ln_self = ln_load(L0.self_g, L0.self_b);
    }
    for (int l = 0; l < P.n_layers; ++l) {
      const MtLayerP L = layers[l];
      stamping = P.ts != nullptr && blockIdx.x == 0 && si == 1 && l == 1;
      STAMP(0);
      if (l + 1 < P.n_layers) layer_prefetch(layers[l + 1], in_group, grp_h, grp_j);
      else {
        gemv_prefetch<DIM, 6>(P.emb, P.vocab);                           // the tied output projection of this step
        if (si + 1 < nsteps) layer_prefetch(layers[0], in_group, grp_h, grp_j);  // and layer 0 of the next one
      }
      float* kc = P.self_k + ((size_t)l * P.max_pos + s + P.kv_off) * DIM;
      float* vc = P.self_v + ((size_t)l * P.max_pos + s + P.kv_off) * DIM;
      // (1) x += FFN delta of the previous layer; q | k | v = LN(x) Wqkv^T
      if (l > 0) {
        for (int c = tid; c < DIM; c += MTT) sm.x[c] = sm.x[c] + delta[c];
        __syncthreads();
      }
      ln_to_v(sm, ln_self, DIM);
      gemv_finish_b(w_qkv, sm.v, 3 * DIM, [&](int col, float y) {
        if (col < DIM) P.q[col] = y;
        else if (col < 2 * DIM) kc[col - DIM] = y;
        else vc[col - 2 * DIM] = y;
      });
      STAMP(1);
      ARRIVE();
      HpW hw;
      if (in_group) hw = hp_load(L.wo, grp_h, grp_j);
      WAIT();
      STAMP(2);
      // (2) self-attention of head grp_h (every CTA of the group) + partial out-projection of this CTA's 32 columns
      if (in_group) {
        attend_head_self(sm, P.q + grp_h * MHD, P.self_k + (size_t)l * P.max_pos * DIM + grp_h * MHD, P.self_v + (size_t)l * P.max_pos * DIM + grp_h * MHD,
                          DIM, s + P.kv_off + 1, att_h);
        __syncthreads();
        head_partial_proj_w(att_h, hw, grp_j, part + grp_h * DIM);
      }
      STAMP(3);
      ARRIVE();
      GemvW<DIM, 1> w_cq;
      gemv_issue_b(w_cq, L.wcq, DIM, L.bcq);
      const LnP ln_cross = ln_load(L.cross_g, L.cross_b);
      WAIT();
      STAMP(4);
      // (3) x += sum_h partials + bo; q = LN(x) Wcq^T
      add_head_partials(sm.x, part, L.bo);
      ln_to_v(sm, ln_cross, DIM);
      gemv_finish_b(w_cq, sm.v, DIM, [&](int col, float y) { P.q[col] = y; });
      STAMP(5);
      ARRIVE();
      if (in_group) hw = hp_load(L.wco, grp_h, grp_j);
      WAIT();
      STAMP(6);
      // (4) cross-attention of head grp_h + partial out-projection
      if (in_group) {
        const float* cross = P.cross_kv + (size_t)l * P.cross_cap * 2 * DIM;
        attend_head_early(sm, P.q + grp_h * MHD, cross + grp_h * MHD, cross + DIM + grp_h * MHD, 2 * DIM, T, att_h);
        __syncthreads();
        head_partial_proj_w(att_h, hw, grp_j, part + grp_h * DIM);
      }
      STAMP(7);
      ARRIVE();
      GemvW<DIM, 2> w_1;
      gemv_issue_b(w_1, L.w1, FFN, L.b1);
      const LnP ln_fin = ln_load(L.fin_g, L.fin_b);
      WAIT();
      STAMP(8);
      // (5) x += sum_h partials + bco; hid = relu(LN(x) W1^T)
      add_head_partials(sm.x, part, L.bco);
      ln_to_v(sm, ln_fin, DIM);
      gemv_finish_b(w_1, sm.v, FFN, [&](int col, float y) { P.hid[col] = y > 0.f ? y : 0.f; });
      STAMP(9);
      ARRIVE();
      GemvW<FFN, 1> w_2;
      gemv_issue_b(w_2, L.w2, DIM, L.b2);
      WAIT();
      STAMP(10);
      // (6) delta = hid W2^T + b2
      load_vec(sm.v, P.hid, FFN);
      gemv_finish_b(w_2, sm.v, DIM, [&](int col, float y) { delta[col] = y; });
      STAMP(11);
      ARRIVE();
      if (l + 1 < P.n_layers) {
        const MtLayerP Ln = layers[l + 1];
        gemv_issue_b(w_qkv, Ln.wqkv, 3 * DIM, Ln.bqkv);
        ln_self = ln_load(Ln.self_g, Ln.self_b);
      }
      WAIT();
      STAMP(12);
    }
    const bool forced_eos = s >= max_len;
    GemvW<DIM, 6> w_out;
    if (!forced_eos) gemv_issue(w_out, P.emb, P.vocab);
    const LnP ln_out = ln_load(P.out_g, P.out_b);
    for (int c = tid; c < DIM; c += MTT) sm.x[c] = sm.x[c] + delta[c];
    __syncthreads();
    ln_to_v(sm, ln_out, DIM);
    if (blockIdx.x == 0)
      for (int c = tid; c < DIM; c += MTT) P.feats[(size_t)s * DIM + c] = sm.v[c];
    if (!forced_eos) gemv_finish(w_out, sm.v, P.vocab, [&](int col, float acc) { P.logits[col] = acc; });
    BAR();
    if (forced_eos) break;
    {
      const int tk = masked_argmax(sm, P.logits, P.vocab, P.pad, P.eos, s);
      if (tid == 0 && blockIdx.x == 0) P.tok[s + 1] = tk;
      if (tk == P.eos) break;
    }
  }
#undef BAR
#undef ARRIVE
#undef WAIT
#undef STAMP
  const int planned = nsteps * barriers_per_step;
  if (threadIdx.x == 0 && done_barriers < planned) atomicAdd(bar_ctr, (unsigned)(planned - done_barriers));
}

}  // namespace

bool mt_decode_persistent_supported(int dim, int ffn, int heads, int vocab, int max_pos, int T) {
  // (one round of columns per phase: vocab <= 6 columns x 8 warps x #SMs, checked against the smallest supported grid; the
  // self-attention cache may hold any number of entries, the cross-attention of T encoder rows keeps its scores in MtSmem::S)
  return vocab <= 6 * MW * 132 && dim == 512 && ffn == 2048 && heads * MHD == dim && vocab >= 1 && max_pos >= 1 && T >= 1 && T <= MSC;
}

int mt_decode_persistent(const MtDecodeParams& P, const MtLayerP* layers_dev, int step0, int nsteps, int max_len, int T, unsigned* bar_ctr,
                         unsigned* bar_target_host, cudaStream_t st) {
  ++g_launches;
  int occ = 0;
  if (first_time_on_device((const void*)mt_decode_persistent_kernel_v2)) {  // cooperative launch needs one resident CTA per SM on this device
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, mt_decode_persistent_kernel_v2, MTT, 0);
    if (occ < 1) return -1;
  }
  const int grid = current_device_sms();
  if (grid <= 0) return -1;
  if (grid < 8 * GRP || P.vocab > 6 * MW * grid) return -1;  // head groups; one round of columns per GEMV phase (see gemv_issue)
  MtDecodeParams p = P;
  unsigned bar_target = *bar_target_host;
  void* args[] = {(void*)&p, (void*)&layers_dev, (void*)&step0, (void*)&nsteps, (void*)&max_len, (void*)&T, (void*)&bar_ctr, (void*)&bar_target};
  cudaError_t e = cudaLaunchCooperativeKernel((void*)mt_decode_persistent_kernel_v2, dim3(grid), dim3(MTT), args, 0, st);
  if (e != cudaSuccess) return -2;
  *bar_target_host += (unsigned)grid * (unsigned)(nsteps * (P.n_layers * 6 + 1));
  return 0;
}

}  // namespace ss
