// Persistent cooperative kernel for the single-token steps of the MT decoder's greedy search (beam 1).
//
// One decode step is a chain of ~37 dependent M = 1 operations (4 pre-LN layers of self-attention, cross-attention and
// FFN, the tied output projection over 6000 entries and the arg-max); as separate kernels its time per token is
// nearly all kernel boundaries.  This kernel keeps one CTA per SM resident for a whole burst
// of steps and separates the phases with the counter barrier of kernels_persist.cu (33 barriers per token):
//   per layer: [LN + QKV -> q, K/V cache row] | [self-attention, CTA per head] | [out + res] | [LN + Q] |
//              [cross-attention over the encoder states, CTA per head] | [out + res] | [LN + FC1 + ReLU] | [FC2 + res]
//   then:      [final LN -> features row, logits = E @ feat] | arg-max of log_softmax (every CTA redundantly) + embedding
// The 512-float residual stream lives in global memory and is re-read into shared memory by every CTA after each phase
// that updates it; GEMV phases give each warp up to MAXC output columns and issue all weight loads before the reduction.
// Semantics follow ss_mt_greedy's per-kernel path (sequence_generator.py:generate_decoder with beam 1): pad is always
// masked, eos only while step < min_len (= 1), eos is forced at max_len (no logits are computed for that step).
#include "kernels_persist_mt.cuh"

namespace ss {
namespace {

// softmax(q . K^T * scale) V for one head by one CTA: q[64], K/V rows at kbase/vbase + j * ld, n keys; out[64]
__device__ void attend_head(MtSmem& sm, const float* q, const float* kbase, const float* vbase, int ld, int n, float* out) {
  const int tid = threadIdx.x;
  __syncthreads();
  if (tid < MHD) sm.qh[tid] = q[tid] * 0.125f;
  __syncthreads();
  float mx = -INFINITY;
  for (int j = tid; j < n; j += MTT) {
    const float* kr = kbase + (int64_t)j * ld;
    float4 kk[MHD / 4];
#pragma unroll
    for (int d = 0; d < MHD / 4; ++d) kk[d] = *reinterpret_cast<const float4*>(kr + 4 * d);
    float s = 0.f;
#pragma unroll
    for (int d = 0; d < MHD / 4; ++d) {
      s = fmaf(sm.qh[4 * d], kk[d].x, s);
      s = fmaf(sm.qh[4 * d + 1], kk[d].y, s);
      s = fmaf(sm.qh[4 * d + 2], kk[d].z, s);
      s = fmaf(sm.qh[4 * d + 3], kk[d].w, s);
    }
    sm.S[j] = s;
    mx = fmaxf(mx, s);
  }
  mx = block_reduce_max(sm, mx);
  float sum = 0.f;
  for (int j = tid; j < n; j += MTT) {
    float e = expf(sm.S[j] - mx);
    sm.S[j] = e;
    sum += e;
  }
  sum = block_reduce_sum(sm, sum);
  // thread (part, q): keys j = part (mod 16), dims [4q, 4q + 4); 8 keys (8 independent 16-byte loads) in flight per thread.
  // (4 key phases x 1 float used to mean 40 dependent L2 round trips for 160 encoder rows)
  const int q4 = (tid & 15) * 4, part = tid >> 4;
  float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll 1
  for (int j0 = part; j0 < n; j0 += 16 * 8) {
    float4 vv[8];
    float pp[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      const int j = j0 + 16 * u;
      const bool ok = j < n;
      vv[u] = ok ? *reinterpret_cast<const float4*>(vbase + (int64_t)j * ld + q4) : make_float4(0.f, 0.f, 0.f, 0.f);
      pp[u] = ok ? sm.S[j] : 0.f;
    }
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      a.x = fmaf(pp[u], vv[u].x, a.x);
      a.y = fmaf(pp[u], vv[u].y, a.y);
      a.z = fmaf(pp[u], vv[u].z, a.z);
      a.w = fmaf(pp[u], vv[u].w, a.w);
    }
  }
  *reinterpret_cast<float4*>(&sm.pv[part][q4]) = a;
  __syncthreads();
  if (tid < MHD) {
    float t = 0.f;
#pragma unroll
    for (int x = 0; x < 16; ++x) t += sm.pv[x][tid];
    out[tid] = t / sum;
  }
}

__global__ void __launch_bounds__(MTT, 1) mt_decode_persistent_kernel(MtDecodeParams P, const MtLayerP* __restrict__ layers, int step0,
                                                                      int nsteps, int max_len, int T, unsigned* bar_ctr,
                                                                      unsigned bar_target) {
  __shared__ __align__(16) MtSmem sm;
  constexpr int DIM = 512, FFN = 2048;
  const int tid = threadIdx.x;
  const int barriers_per_step = P.n_layers * 8 + 1;
  int done_barriers = 0;
  const float emb_scale = sqrtf((float)DIM);
#define BAR()                          \
  grid_barrier(bar_ctr, bar_target);   \
  ++done_barriers;
  for (int si = 0; si < nsteps; ++si) {
    const int s = step0 + si;  // position of the token fed in this step = its row in the self-attention cache
    // ---- embedding (every CTA; the token was written by the previous step's arg-max or by the host)
    {
      const int64_t tok = (si == 0) ? P.tok[s] : (int64_t)sm.tok;  // later tokens: this CTA's own arg-max (no barrier needed)
      const int p = (tok == P.pad) ? P.pad : P.pad + 1 + s;
      for (int c = tid; c < DIM; c += MTT) sm.x[c] = emb_scale * P.emb[tok * DIM + c] + P.pos[(int64_t)p * DIM + c];
      __syncthreads();
    }
    for (int l = 0; l < P.n_layers; ++l) {
      const MtLayerP L = layers[l];
      float* kc = P.self_k + ((size_t)l * P.max_pos + s + P.kv_off) * DIM;
      float* vc = P.self_v + ((size_t)l * P.max_pos + s + P.kv_off) * DIM;
      // (1) q | k | v = LN(x) Wqkv^T
      GemvW<DIM, 2> w_qkv;
      gemv_issue(w_qkv, L.wqkv, 3 * DIM);
      if (l > 0) load_vec(sm.x, P.x, DIM);
      ln_to_v(sm, L.self_g, L.self_b, DIM);
      gemv_finish(w_qkv, sm.v, 3 * DIM, [&](int col, float acc) {
        float y = acc + (L.bqkv ? L.bqkv[col] : 0.f);
        if (col < DIM) P.q[col] = y;
        else if (col < 2 * DIM) kc[col - DIM] = y;
        else vc[col - 2 * DIM] = y;
      });
      BAR();
      // (2) causal self-attention over rows 0..s (+ kv_off) of the cache
      if (blockIdx.x < P.heads) {
        const int h = blockIdx.x;
        attend_head(sm, P.q + h * MHD, P.self_k + (size_t)l * P.max_pos * DIM + h * MHD, P.self_v + (size_t)l * P.max_pos * DIM + h * MHD, DIM,
                    s + P.kv_off + 1, P.attn + h * MHD);
      }
      BAR();
      // (3) x += attn Wo^T
      GemvW<DIM, 1> w_o;
      gemv_issue(w_o, L.wo, DIM);
      load_vec(sm.v, P.attn, DIM);
      gemv_finish(w_o, sm.v, DIM, [&](int col, float acc) { P.x[col] = (acc + (L.bo ? L.bo[col] : 0.f)) + sm.x[col]; });
      BAR();
      // (4) q = LN(x) Wcq^T
      GemvW<DIM, 1> w_cq;
      gemv_issue(w_cq, L.wcq, DIM);
      load_vec(sm.x, P.x, DIM);
      ln_to_v(sm, L.cross_g, L.cross_b, DIM);
      gemv_finish(w_cq, sm.v, DIM, [&](int col, float acc) { P.q[col] = acc + (L.bcq ? L.bcq[col] : 0.f); });
      BAR();
      // (5) cross-attention over the T encoder states (K | V rows precomputed by mt_begin)
      if (blockIdx.x < P.heads) {
        const int h = blockIdx.x;
        const float* cross = P.cross_kv + (size_t)l * P.cross_cap * 2 * DIM;
        attend_head(sm, P.q + h * MHD, cross + h * MHD, cross + DIM + h * MHD, 2 * DIM, T, P.attn + h * MHD);
      }
      BAR();
      // (6) x += attn Wco^T
      GemvW<DIM, 1> w_co;
      gemv_issue(w_co, L.wco, DIM);
      load_vec(sm.v, P.attn, DIM);
      gemv_finish(w_co, sm.v, DIM, [&](int col, float acc) { P.x[col] = (acc + (L.bco ? L.bco[col] : 0.f)) + sm.x[col]; });
      BAR();
      // (7) hid = relu(LN(x) W1^T)
      GemvW<DIM, 2> w_1;
      gemv_issue(w_1, L.w1, FFN);
      load_vec(sm.x, P.x, DIM);
      ln_to_v(sm, L.fin_g, L.fin_b, DIM);
      gemv_finish(w_1, sm.v, FFN, [&](int col, float acc) {
        float y = acc + (L.b1 ? L.b1[col] : 0.f);
        P.hid[col] = y > 0.f ? y : 0.f;
      });
      BAR();
      // (8) x += hid W2^T
      GemvW<FFN, 1> w_2;
      gemv_issue(w_2, L.w2, DIM);
      load_vec(sm.v, P.hid, FFN);
      gemv_finish(w_2, sm.v, DIM, [&](int col, float acc) { P.x[col] = (acc + (L.b2 ? L.b2[col] : 0.f)) + sm.x[col]; });
      BAR();
    }
    // ---- final LN -> feature row; logits over the tied embedding unless eos is forced at this step
    const bool forced_eos = s >= max_len;
    GemvW<DIM, 6> w_out;
    if (!forced_eos) gemv_issue(w_out, P.emb, P.vocab);
    load_vec(sm.x, P.x, DIM);
    ln_to_v(sm, P.out_g, P.out_b, DIM);
    if (blockIdx.x == 0)
      for (int c = tid; c < DIM; c += MTT) P.feats[(size_t)s * DIM + c] = sm.v[c];
    if (!forced_eos) gemv_finish(w_out, sm.v, P.vocab, [&](int col, float acc) { P.logits[col] = acc; });
    BAR();
    if (forced_eos) break;
    // ---- arg-max of log_softmax(logits) with masks, first index wins on ties (argmax_rows_kernel); every CTA
    {
      const float* x = P.logits;
      float mx = -INFINITY;
      for (int c = tid; c < P.vocab; c += MTT) mx = fmaxf(mx, x[c]);
      mx = block_reduce_max(sm, mx);
      float su = 0.f;
      for (int c = tid; c < P.vocab; c += MTT) su += expf(x[c] - mx);
      su = block_reduce_sum(sm, su);
      const float lse = logf(su);
      float best = -INFINITY;
      int bi = 0x7fffffff;
      for (int c = tid; c < P.vocab; c += MTT) {
        const bool masked = (c == P.pad) || (s < 1 && c == P.eos);
        float lp = masked ? -INFINITY : (x[c] - mx) - lse;
        if (lp > best || (lp == best && c < bi)) {
          best = lp;
          bi = c;
        }
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        float ob = __shfl_xor_sync(0xffffffffu, best, o);
        int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (ob > best || (ob == best && oi < bi)) {
          best = ob;
          bi = oi;
        }
      }
      __syncthreads();
      if ((tid & 31) == 0) {
        sm.rbest[tid >> 5] = best;
        sm.ridx[tid >> 5] = bi;
      }
      __syncthreads();
      if (tid == 0) {
        for (int i = 1; i < MW; ++i)
          if (sm.rbest[i] > best || (sm.rbest[i] == best && sm.ridx[i] < bi)) {
            best = sm.rbest[i];
            bi = sm.ridx[i];
          }
        sm.tok = bi;
        if (blockIdx.x == 0) P.tok[s + 1] = bi;
      }
      __syncthreads();
      if (sm.tok == P.eos) break;  // the host stops at the first eos; later steps would never be read
    }
  }
#undef BAR
  // leave the barrier counter where the host expects it after a full burst
  const int planned = nsteps * barriers_per_step;
  if (threadIdx.x == 0 && done_barriers < planned) atomicAdd(bar_ctr, (unsigned)(planned - done_barriers));
}

// ---- version 2 of the single-token step: 6 grid barriers per layer instead of 8.
// The two phases [attention of head h on ONE CTA] | barrier | [out-projection over all CTAs] become one: the 16 CTAs of a head
// group each compute the (tiny, M = 1) attention of their head redundantly and then the PARTIAL out-projection of their 32
// output columns over that head's 64 inputs; the 8 per-head partial vectors are summed (fixed order) by every CTA while it stages
// the next phase, together with bias and residual, so the residual stream x lives in shared memory of every CTA and is never
// exchanged.  Same for the cross-attention block; the FFN output is handed over the same way (one 512-vector).
//   per layer: [LN + QKV] | [self-attn + Wo partials] | [x += sum, LN + Wcq] | [cross-attn + Wco partials] |
//              [x += sum, LN + FC1 + ReLU] | [FC2 -> delta]          (next layer / final LN: x += delta)

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
        attend_head_early(sm, P.q + grp_h * MHD, P.self_k + (size_t)l * P.max_pos * DIM + grp_h * MHD, P.self_v + (size_t)l * P.max_pos * DIM + grp_h * MHD,
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
  // (one round of columns per phase: vocab <= 6 columns x 8 warps x #SMs, checked against the smallest supported grid)
  return vocab <= 6 * MW * 132 && dim == 512 && ffn == 2048 && heads * MHD == dim && vocab >= 1 && max_pos <= 1024 && T >= 1 && T <= 1024;
}

int mt_decode_persistent(const MtDecodeParams& P, const MtLayerP* layers_dev, int step0, int nsteps, int max_len, int T, unsigned* bar_ctr,
                         unsigned* bar_target_host, cudaStream_t st) {
  ++g_launches;
  int occ = 0;
  if (first_time_on_device((const void*)mt_decode_persistent_kernel)) {  // cooperative launch needs one resident CTA per SM on this device
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, mt_decode_persistent_kernel, MTT, 0);
    if (occ < 1) return -1;
  }
  const int grid = current_device_sms();
  if (grid <= 0) return -1;
  if (grid < 128 || P.vocab > 6 * MW * grid) return -1;  // one round of columns per GEMV phase (see gemv_issue)
  MtDecodeParams p = P;
  unsigned bar_target = *bar_target_host;
  void* args[] = {(void*)&p, (void*)&layers_dev, (void*)&step0, (void*)&nsteps, (void*)&max_len, (void*)&T, (void*)&bar_ctr, (void*)&bar_target};
  const bool v2 = P.part != nullptr && P.delta != nullptr && P.heads == 8 && grid >= 8 * GRP;
  cudaError_t e = cudaLaunchCooperativeKernel(v2 ? (void*)mt_decode_persistent_kernel_v2 : (void*)mt_decode_persistent_kernel, dim3(grid), dim3(MTT), args,
                                              0, st);
  if (e != cudaSuccess) return -2;
  *bar_target_host += (unsigned)grid * (unsigned)(nsteps * (P.n_layers * (v2 ? 6 : 8) + 1));
  return 0;
}

}  // namespace ss
