// Greedy MT search (beam 1, no prefix) for up to MT_BATCH_MAX_ROWS independent samples in one persistent cooperative kernel:
// the offline generator's batch decoded together.  The phases are those of mt_decode_persistent_kernel_v2 (6 split barriers
// per layer), and each phase's weights are loaded into registers ONCE per step and applied to every unfinished row:
//   per layer: [LN + QKV] | [self-attn + Wo partials] | [x += sum, LN + Wcq] | [cross-attn + Wco partials] |
//              [x += sum, LN + FC1 + ReLU] | [FC2 -> delta]
//   then:      [x += delta, final LN, logits = E @ feat] | [arg-max of log_softmax, row i on CTA i]
// The stream pool's search (ss_pool_mt_greedy) continues each row after a forced prefix: with MtBatchParams' per-row fields a row
// feeds position start + step (position embedding, cache row, self-attention length and the position-0 eos ban follow), stops at
// its own max_len with eos forced, reads its slot's cross K / V and writes its final-LN rows as features.
// The incremental search (ss_pool_mt_greedy_incremental) runs a third instantiation on the same per-row fields plus two more: row r
// keeps its self-attention cache in a block of its own that lives across calls (self_row[r], [layers][self_ld][dim] as
// MtDecodeParams' self_k / self_v), and the position-p entry of that cache is p + kv_off[r] (the single-token kernel's kv_off).
// The offline beam search (ss_mt_beam_batch) is a fourth instantiation (MtBeamParams): the same layer phases and logits, then
// candidates (row i on CTA i) and selection (sample j on CTA j) in place of the arg-max, one more grid barrier per step, and the
// reorder of the rows' self-attention caches into a second buffer at the start of the next step.  At beam 1 (UnitY's unit search,
// ss_unit_search_batch, on the unit decoder's 2 layers) every row is its own parent: the caches stay in place and are not reordered.
// Every CTA keeps the residual rows of all samples in shared memory (32 x 2 KB); the LayerNorm outputs share a second
// 64 KB buffer with the FFN hidden rows, which do not fit at once (8 KB each) and are staged 8 rows at a time.
//
// Exactness: a row is computed with v2's arithmetic (same lane partition and warp_sum tree per GEMV column, same two-pass
// LayerNorm sums, same attention split, head partials summed in head order, same embedding), so each row is bit-identical to
// ss_mt_greedy on that sample alone and the tokens are equal by construction.  Three things are distributed differently, with
// unchanged arithmetic:
//  - attention: v2 has all 16 CTAs of a head group compute the head's attention redundantly and each project 32 columns;
//    here unfinished row i goes to CTA (i mod 16) of the group, which projects all 512 columns of that row.  Redundancy would
//    cost B attentions per CTA and phase; the split costs each CTA the head's 512 x 64 out-projection block from L2.
//  - arg-max: v2 runs it redundantly in every CTA.  With B rows that would be B full-vocabulary passes (three block-wide
//    reductions each) per CTA and step; spreading the rows over CTAs costs one more grid barrier instead (6 * layers + 2 per step).
//  - LayerNorm: one warp per row; it forms the same 8 per-warp sums (warp_sum over the same 32 elements) and adds them in
//    the same order as ln_to_v, without the block-wide __syncthreads per row.
#include "kernels_persist_mt.cuh"

namespace ss {
namespace {

constexpr int MAXR = MT_BATCH_MAX_ROWS;
constexpr int ROWS_PER_CTA = MAXR / GRP;  // attention rows per CTA of a head group
constexpr int DIM = 512, FFN = 2048;
constexpr int HID_TILE = MAXR * DIM / FFN;  // FFN hidden rows staged at once in the LayerNorm buffer
static_assert(MAXR % GRP == 0 && HID_TILE >= 1, "row split");

struct MtbSmem {
  int act[MAXR];  // unfinished rows, in row order
  int nact;
  float att[ROWS_PER_CTA][MHD];
};

constexpr size_t kDynSmem = (size_t)2 * MAXR * DIM * sizeof(float);  // residual rows + LayerNorm rows / hidden tile

// vb[r] = LayerNorm(xs[r]) for every unfinished row r; bit-identical to ln_to_v(sm, LnP, 512) (see the file comment)
__device__ __forceinline__ void ln_rows(const MtbSmem& sb, const float* xs, float* vb, const float* __restrict__ g, const float* __restrict__ b) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int i = warp; i < sb.nact; i += MW) {
    const int r = sb.act[i];
    const float* x = xs + r * DIM;
    float* v = vb + r * DIM;
    float a0[MW], a1[MW];
    float mean = 0.f;
#pragma unroll
    for (int w = 0; w < MW; ++w) {
      a0[w] = x[w * 32 + lane];
      a1[w] = x[w * 32 + lane + MTT];
      const float s = warp_sum(a0[w] + a1[w]);
      mean = (w == 0) ? s : mean + s;
    }
    mean = mean / (float)DIM;
    float var = 0.f;
#pragma unroll
    for (int w = 0; w < MW; ++w) {
      a0[w] = a0[w] - mean;
      a1[w] = a1[w] - mean;
      const float s = warp_sum(fmaf(a0[w], a0[w], a1[w] * a1[w]));
      var = (w == 0) ? s : var + s;
    }
    var = var / (float)DIM;
    const float rstd = 1.0f / sqrtf(var + 1e-5f);
#pragma unroll
    for (int w = 0; w < MW; ++w) {
      const int t = w * 32 + lane;
      v[t] = a0[w] * rstd * __ldg(g + t) + __ldg(b + t);
      v[t + MTT] = a1[w] * rstd * __ldg(g + t + MTT) + __ldg(b + t + MTT);
    }
  }
  __syncthreads();
}

// xs[r] += sum_h part[r][h] + bias for every unfinished row (add_head_partials per row)
__device__ __forceinline__ void add_partials_rows(const MtbSmem& sb, float* xs, const float* part, const float* __restrict__ bias) {
#pragma unroll 4
  for (int e = threadIdx.x; e < sb.nact * DIM; e += MTT) {
    const int r = sb.act[e / DIM], c = e % DIM;
    const float* pr = part + (size_t)r * 8 * DIM;
    float t = pr[c];
#pragma unroll
    for (int h = 1; h < 8; ++h) t += pr[h * DIM + c];
    xs[r * DIM + c] = xs[r * DIM + c] + (t + (bias ? bias[c] : 0.f));
  }
  __syncthreads();
}

// xs[r] += delta[r] for every unfinished row
__device__ __forceinline__ void add_delta_rows(const MtbSmem& sb, float* xs, const float* delta) {
  for (int e = threadIdx.x; e < sb.nact * DIM; e += MTT) {
    const int r = sb.act[e / DIM], c = e % DIM;
    xs[r * DIM + c] = xs[r * DIM + c] + delta[(size_t)r * DIM + c];
  }
  __syncthreads();
}

// attention of head h for this CTA's rows (unfinished rows i = j, j + 16, ...) and their partial out-projections over all 512
// columns: part[r][h][col] = sum_{i < 64} a[i] * W[col][64 h + i], warp w owning columns [64 w, 64 w + 64).  kSelf: the rows' key
// counts are cache lengths, which may exceed MSC (attend_head_self, as the single-token kernel); cross-attention has at most MSC keys
template <bool kSelf, typename KV>
__device__ __forceinline__ void attend_rows(MtSmem& sm, MtbSmem& sb, const float* q, KV&& kv, const float* __restrict__ W, int h, int j,
                                            float* part) {
  int nloc = 0;
  for (int i = j; i < sb.nact; i += GRP, ++nloc) {
    const int r = sb.act[i];
    const float* kb;
    const float* vbase;
    int ld, n;
    kv(r, kb, vbase, ld, n);
    if constexpr (kSelf) attend_head_self(sm, q + (size_t)r * DIM + h * MHD, kb + h * MHD, vbase + h * MHD, ld, n, sb.att[nloc]);
    else attend_head_early(sm, q + (size_t)r * DIM + h * MHD, kb + h * MHD, vbase + h * MHD, ld, n, sb.att[nloc]);
  }
  __syncthreads();
  if (nloc == 0) return;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float a0[ROWS_PER_CTA], a1[ROWS_PER_CTA];
#pragma unroll
  for (int k = 0; k < ROWS_PER_CTA; ++k) {
    a0[k] = sb.att[k][lane];
    a1[k] = sb.att[k][lane + 32];
  }
  constexpr int CU = 16;  // columns whose weights are in flight together
#pragma unroll 1
  for (int c0 = 0; c0 < 64; c0 += CU) {
    float w0[CU], w1[CU];
#pragma unroll
    for (int u = 0; u < CU; ++u) {
      const float* w = W + (int64_t)(warp * 64 + c0 + u) * DIM + h * MHD;
      w0[u] = __ldg(w + lane);
      w1[u] = __ldg(w + lane + 32);
    }
#pragma unroll
    for (int k = 0; k < ROWS_PER_CTA; ++k) {
      if (k < nloc) {
        float* pr = part + ((size_t)sb.act[j + k * GRP] * 8 + h) * DIM + warp * 64 + c0;
#pragma unroll
        for (int u = 0; u < CU; ++u) {
          const float acc = head_col_partial(a0[k], a1[k], w0[u], w1[u]);
          if (lane == 0) pr[u] = acc;
        }
      }
    }
  }
}

// the four searches: offline (no per-row fields), a forced prefix continued (start / max_len / cross_row / feats), the
// incremental search on slot-resident self-attention caches (those fields plus self_row / kv_off, feats optional), and the
// offline beam search (MtBeamParams)
enum MtbMode { kMtbOffline, kMtbPrefix, kMtbIncremental, kMtbBeam };

// position row r feeds at step s
template <int kMode>
__device__ __forceinline__ int row_pos(const MtBatchParams& P, int r, int s) {
  return kMode == kMtbPrefix || kMode == kMtbIncremental ? P.start[r] + s : s;
}

// kMtbIncremental: offset of row r's layer-l block in the slot-resident self-attention cache (K and V alike)
__device__ __forceinline__ size_t self_block(const MtBatchParams& P, int r, int l) {
  return ((size_t)P.self_row[r] * P.n_layers + l) * P.self_ld * DIM;
}

__device__ __forceinline__ void load_active(MtbSmem& sb, const int* fin, int rows) {
  if (threadIdx.x == 0) {
    int n = 0;
    for (int r = 0; r < rows; ++r)
      if (*(volatile const int*)(fin + r) == 0) sb.act[n++] = r;
    sb.nact = n;
  }
  __syncthreads();
}

// ---- beam search (kMtbBeam).  Order of candidates: higher score first; on exactly equal scores the lower flat index
// (beam * vocab + token, fairseq's view(bsz, -1) of the sample's candidates) first.

__device__ __forceinline__ bool cand_before(float v, int k, float bv, int bk) { return v > bv || (v == bv && k < bk); }

// The k best of the n entries vals[0 .. n) (shared memory, n >= k) in cand_before order of (vals[e], key(e)); the whole CTA takes
// part and thread 0 writes out_v[i] / out_k[i] for i < k.  Entry e belongs to thread e mod MTT, which keeps its best untaken
// entry: a round reduces those, the winner's entry becomes NaN (never selected again) and only its thread scans again.
// red: 6 x MW words of scratch (two rounds' worth: one __syncthreads per round).
template <typename Key>
__device__ __forceinline__ void block_top_k(float* vals, int n, Key key, int k, float* red, float* out_v, int* out_k) {
  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  float bv;
  int bk, be;
  auto scan = [&]() {
    bv = -INFINITY, bk = 0x7fffffff, be = -1;
    for (int e = tid; e < n; e += MTT) {
      const float v = vals[e];
      const int kk = key(e);
      if (cand_before(v, kk, bv, bk)) bv = v, bk = kk, be = e;
    }
  };
  scan();
  for (int i = 0; i < k; ++i) {
    float v = bv;
    int kk = bk, e = be;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, v, o);
      const int ok = __shfl_xor_sync(0xffffffffu, kk, o), oe = __shfl_xor_sync(0xffffffffu, e, o);
      if (cand_before(ov, ok, v, kk)) v = ov, kk = ok, e = oe;
    }
    float* rv = red + (i & 1) * 3 * MW;
    int* rk = reinterpret_cast<int*>(rv + MW);
    int* re = rk + MW;
    if (lane == 0) rv[w] = v, rk[w] = kk, re[w] = e;
    __syncthreads();
    v = rv[0], kk = rk[0], e = re[0];
#pragma unroll
    for (int x = 1; x < MW; ++x)
      if (cand_before(rv[x], rk[x], v, kk)) v = rv[x], kk = rk[x], e = re[x];
    if (tid == 0) out_v[i] = v, out_k[i] = kk;
    if (e >= 0 && tid == e % MTT) {
      vals[e] = NAN;
      scan();
    }
  }
  __syncthreads();
}

// step s > 0: the self-attention cache rows 0 .. s - 1 of every live row r (all layers, K and V) from row parent[r] of the previous
// step's buffer; the whole grid takes part, one float4 per thread and round.  Step s's QKV phase writes only row s.
__device__ __forceinline__ void beam_gather_kv(const MtBatchParams& P, const MtBeamParams& B, const MtbSmem& sb, int s, float* kd, float* vd, const float* ks,
                                               const float* vs) {
  constexpr int Q = DIM / 4;
  const size_t layer = (size_t)MAXR * P.tok_ld * DIM;
  const int64_t total = (int64_t)sb.nact * P.n_layers * s * 2 * Q;
  for (int64_t g = (int64_t)blockIdx.x * MTT + threadIdx.x; g < total; g += (int64_t)gridDim.x * MTT) {
    const int q = (int)(g % Q);
    int64_t u = g / Q;
    const int kv = (int)(u & 1);
    u >>= 1;
    const int p = (int)(u % s);
    u /= s;
    const int l = (int)(u % P.n_layers), r = sb.act[u / P.n_layers];
    const size_t dst = l * layer + ((size_t)r * P.tok_ld + p) * DIM, src = l * layer + ((size_t)B.parent[r] * P.tok_ld + p) * DIM;
    *reinterpret_cast<float4*>((kv ? vd : kd) + dst + 4 * q) = *reinterpret_cast<const float4*>((kv ? vs : ks) + src + 4 * q);
  }
}

// candidates of row r at step s: log_softmax of its logits (masked_argmax's max / sum-exp / logf), pad masked, eos masked at
// step 0 (min_len 1), everything but eos masked from step max_len on, plus the row's cumulative score (BeamSearch.step); the
// 2 K best (score, token) go to B.cand / B.cand_tok.  lp: the vocabulary's scores (shared memory).
__device__ __forceinline__ void beam_row_candidates(MtSmem& sm, const MtBatchParams& P, const MtBeamParams& B, int r, int s, const float* cum, float* lp,
                                                    float* red) {
  const int K2 = 2 * B.beam;
  const float* x = P.logits + (size_t)r * P.vocab;
  float mx, lse;
  row_log_softmax_terms(sm, x, P.vocab, mx, lse);
  const float prev = s > 0 ? cum[(size_t)r * P.tok_ld + s - 1] : 0.f;
  for (int c = threadIdx.x; c < P.vocab; c += MTT) {
    float v = (x[c] - mx) - lse;
    if (v != v || c == P.pad || (s >= B.max_len ? c != P.eos : (s < 1 && c == P.eos))) v = -INFINITY;
    lp[c] = s > 0 ? v + prev : v;  // (step 0: lprobs[:, ::beam_size], no score yet)
  }
  __syncthreads();
  block_top_k(lp, P.vocab, [](int e) { return e; }, K2, red, B.cand + (size_t)r * K2, B.cand_tok + (size_t)r * K2);
}

// the selection of sample j at step s (generate_decoder's bookkeeping around BeamSearch.step): the 2 K best of its beams'
// candidates (at step 0 those of beam 0 only); eos among the first K, in rank order, finalized while the sample holds fewer than
// K hypotheses (finalize_hypos); the sample is done with K of them or at step max_len; otherwise the first K candidates that are
// not a finite eos become the new beams: token and score histories reordered into the next buffers, parents recorded for the
// self-attention gather of the next step.  buf: shared memory for 8 K^2 + 4 K floats; red: block_top_k's scratch.
__device__ __forceinline__ void beam_select(const MtBatchParams& P, const MtBeamParams& B, int j, int s, const int64_t* tok, int64_t* tok_nx, const float* cum,
                                            float* cum_nx, float* buf, float* red) {
  const int K = B.beam, K2 = 2 * K, V = P.vocab, tid = threadIdx.x, ld = P.tok_ld;
  const int nb = s == 0 ? 1 : K, n = nb * K2;
  float* cv = buf;
  int* ck = reinterpret_cast<int*>(cv + n);
  float* sel_v = reinterpret_cast<float*>(ck + n);
  int* sel_k = reinterpret_cast<int*>(sel_v + K2);
  int* par = sel_k + K2;  // [K] parent rows: finalized hypotheses first, then the new beams
  int* nxt = par + K;     // [K] the new beams' tokens
  float* sc = reinterpret_cast<float*>(nxt + K);  // [K] their scores / the finalized eos scores
  int* meta = reinterpret_cast<int*>(sc + K);     // finalized before this step, finalized now, done
  for (int e = tid; e < n; e += MTT) {
    const size_t c = (size_t)(j * K + e / K2) * K2 + e % K2;
    cv[e] = B.cand[c];
    ck[e] = (e / K2) * V + B.cand_tok[c];
  }
  __syncthreads();
  block_top_k(cv, n, [&](int e) { return ck[e]; }, K2, red, sel_v, sel_k);
  if (tid == 0) {
    const int nf0 = B.n_fin[j];
    int nf = nf0, m = 0;
    for (int k = 0; k < K; ++k)
      if (sel_k[k] % V == P.eos && sel_v[k] != -INFINITY && nf < K) {
        par[m] = j * K + sel_k[k] / V;
        sc[m++] = sel_v[k];
        ++nf;
      }
    const int done = nf == K || s >= B.max_len;
    meta[0] = nf0, meta[1] = m, meta[2] = done;
    B.n_fin[j] = nf;
    B.done[j] = done;
  }
  __syncthreads();
  const int nf0 = meta[0], nfz = meta[1], done = meta[2];
  const float norm = (float)pow((double)(s + 1), (double)B.len_penalty);
  for (int f = 0; f < nfz; ++f) {
    const int pr = par[f];
    const size_t h = (size_t)j * K + nf0 + f;
    for (int t = tid; t <= s; t += MTT) {
      B.hyp_tok[h * ld + t] = t < s ? tok[(size_t)pr * ld + t + 1] : P.eos;
      const float c1 = t < s ? cum[(size_t)pr * ld + t] : sc[f];
      B.hyp_pos[h * ld + t] = t == 0 ? c1 : c1 - cum[(size_t)pr * ld + t - 1];
    }
    if (tid == 0) {
      B.hyp_score[h] = sc[f] / norm;
      B.hyp_len[h] = s + 1;
    }
  }
  __syncthreads();
  if (done) {
    for (int b = tid; b < K; b += MTT) P.fin[j * K + b] = 1;
    return;
  }
  if (tid == 0)
    for (int k = 0, m = 0; k < K2 && m < K; ++k)
      if (!(sel_k[k] % V == P.eos && sel_v[k] != -INFINITY)) {
        par[m] = j * K + sel_k[k] / V;
        nxt[m] = sel_k[k] % V;
        sc[m++] = sel_v[k];
      }
  __syncthreads();
  for (int e = tid; e < K * (s + 2); e += MTT) {
    const int b = e / (s + 2), t = e % (s + 2), r = j * K + b;
    tok_nx[(size_t)r * ld + t] = t <= s ? tok[(size_t)par[b] * ld + t] : nxt[b];
    if (t <= s) cum_nx[(size_t)r * ld + t] = t < s ? cum[(size_t)par[b] * ld + t] : sc[b];
  }
  for (int b = tid; b < K; b += MTT) {
    B.parent[j * K + b] = par[b];
    P.fin[j * K + b] = 0;
  }
}

// kMtbOffline: the per-row fields are null and compiled out (the offline generator's search as before they existed)
template <int kMode>
__global__ void __launch_bounds__(MTT, 1) mt_decode_batch_kernel(MtBatchParams P, const MtLayerP* __restrict__ layers, int step0, int nsteps,
                                                                 unsigned* bar_ctr, unsigned bar_target, MtBeamParams B) {
  __shared__ __align__(16) MtSmem sm;
  __shared__ MtbSmem sb;
  extern __shared__ __align__(16) float dyn[];
  float* xs = dyn;               // [MAXR][DIM] residual rows
  float* vb = dyn + MAXR * DIM;  // [MAXR][DIM] LayerNorm rows, or [HID_TILE][FFN] hidden rows
  const int tid = threadIdx.x;
  const int barriers_per_step = P.n_layers * 6 + (kMode == kMtbBeam ? 3 : 2);  // (the beam's selection: one more)
  int done_barriers = 0;
  const float emb_scale = sqrtf((float)DIM);
  const int grp_h = blockIdx.x / GRP, grp_j = blockIdx.x % GRP;
  const bool in_group = blockIdx.x < 8 * GRP;
#define BAR()                          \
  grid_barrier(bar_ctr, bar_target);   \
  ++done_barriers;
#define ARRIVE()                       \
  grid_arrive(bar_ctr, bar_target);    \
  ++done_barriers;
#define WAIT() grid_wait(bar_ctr, bar_target)
  load_active(sb, P.fin, P.rows);
  for (int si = 0; si < nsteps && sb.nact > 0; ++si) {
    const int s = step0 + si;
    // beam search: the rows' tokens, scores and self-attention caches alternate between two buffers (step s reads buffer s & 1)
    const bool alt = kMode == kMtbBeam && (s & 1);
    // beam 1 (the unit search): every row continues itself (parent[r] = r), so its cache stays in one buffer and is not gathered
    const bool alt_kv = alt && B.beam > 1;
    if constexpr (kMode == kMtbBeam)
      if (s > 0 && B.beam > 1) beam_gather_kv(P, B, sb, s, alt ? B.self_k2 : P.self_k, alt ? B.self_v2 : P.self_v, alt ? P.self_k : B.self_k2, alt ? P.self_v : B.self_v2);
    for (int e = tid; e < sb.nact * DIM; e += MTT) {
      const int r = sb.act[e / DIM], c = e % DIM;
      const int64_t tok = (alt ? B.tok2 : P.tok)[(size_t)r * P.tok_ld + s];
      const int p = (tok == P.pad) ? P.pad : P.pad + 1 + row_pos<kMode>(P, r, s);
      xs[r * DIM + c] = emb_scale * P.emb[tok * DIM + c] + P.pos[(int64_t)p * DIM + c];
    }
    __syncthreads();
    GemvW<DIM, 2> w_qkv;
    {
      const MtLayerP L0 = layers[0];
      gemv_issue_b(w_qkv, L0.wqkv, 3 * DIM, L0.bqkv);
    }
    for (int l = 0; l < P.n_layers; ++l) {
      const MtLayerP L = layers[l];
      if (l + 1 < P.n_layers) layer_prefetch(layers[l + 1], in_group, grp_h, grp_j);
      else {
        gemv_prefetch<DIM, 6>(P.emb, P.vocab);
        if (si + 1 < nsteps) layer_prefetch(layers[0], in_group, grp_h, grp_j);
      }
      float* kl = (alt_kv ? B.self_k2 : P.self_k) + (size_t)l * MAXR * P.tok_ld * DIM;
      float* vl = (alt_kv ? B.self_v2 : P.self_v) + (size_t)l * MAXR * P.tok_ld * DIM;
      // (1) x += FFN delta of the previous layer; q | k | v = LN(x) Wqkv^T
      if (l > 0) add_delta_rows(sb, xs, P.delta);
      ln_rows(sb, xs, vb, L.self_g, L.self_b);
      for (int i = 0; i < sb.nact; ++i) {
        const int r = sb.act[i];
        const int pos = row_pos<kMode>(P, r, s);
        float* kc = kl + ((size_t)r * P.tok_ld + pos) * DIM;
        float* vc = vl + ((size_t)r * P.tok_ld + pos) * DIM;
        if constexpr (kMode == kMtbIncremental) {
          const size_t e = self_block(P, r, l) + (size_t)(pos + P.kv_off[r]) * DIM;
          kc = P.self_k + e;
          vc = P.self_v + e;
        }
        gemv_finish_b(w_qkv, vb + r * DIM, 3 * DIM, [&](int col, float y) {
          if (col < DIM) P.q[(size_t)r * DIM + col] = y;
          else if (col < 2 * DIM) kc[col - DIM] = y;
          else vc[col - 2 * DIM] = y;
        });
      }
      ARRIVE();
      WAIT();
      // (2) self-attention over positions 0..s of each row's cache + partial out-projections
      if (in_group)
        attend_rows<true>(sm, sb, P.q, [&](int r, const float*& kb, const float*& vbs, int& ld, int& n) {
          ld = DIM;
          if constexpr (kMode == kMtbIncremental) {
            const size_t b = self_block(P, r, l);
            kb = P.self_k + b;
            vbs = P.self_v + b;
            n = row_pos<kMode>(P, r, s) + P.kv_off[r] + 1;
          } else {
            kb = kl + (size_t)r * P.tok_ld * DIM;
            vbs = vl + (size_t)r * P.tok_ld * DIM;
            n = row_pos<kMode>(P, r, s) + 1;
          }
        }, L.wo, grp_h, grp_j, P.part);
      ARRIVE();
      GemvW<DIM, 1> w_cq;
      gemv_issue_b(w_cq, L.wcq, DIM, L.bcq);
      WAIT();
      // (3) x += sum_h partials + bo; q = LN(x) Wcq^T
      add_partials_rows(sb, xs, P.part, L.bo);
      ln_rows(sb, xs, vb, L.cross_g, L.cross_b);
      for (int i = 0; i < sb.nact; ++i) {
        const int r = sb.act[i];
        gemv_finish_b(w_cq, vb + r * DIM, DIM, [&](int col, float y) { P.q[(size_t)r * DIM + col] = y; });
      }
      ARRIVE();
      WAIT();
      // (4) cross-attention over the first cross_len[r] encoder rows of each sample + partial out-projections
      if (in_group)
        attend_rows<false>(sm, sb, P.q, [&](int r, const float*& kb, const float*& vbs, int& ld, int& n) {
          const size_t blk = kMode == kMtbPrefix || kMode == kMtbIncremental ? (size_t)P.cross_row[r] * P.n_layers + l
                             : (size_t)l * MAXR + (kMode == kMtbBeam ? r / B.beam : r);
          kb = P.cross_kv + blk * P.cross_cap * 2 * DIM;
          vbs = kb + DIM;
          ld = 2 * DIM;
          n = P.cross_len[r];
        }, L.wco, grp_h, grp_j, P.part);
      ARRIVE();
      GemvW<DIM, 2> w_1;
      gemv_issue_b(w_1, L.w1, FFN, L.b1);
      WAIT();
      // (5) x += sum_h partials + bco; hid = relu(LN(x) W1^T)
      add_partials_rows(sb, xs, P.part, L.bco);
      ln_rows(sb, xs, vb, L.fin_g, L.fin_b);
      for (int i = 0; i < sb.nact; ++i) {
        const int r = sb.act[i];
        gemv_finish_b(w_1, vb + r * DIM, FFN, [&](int col, float y) { P.hid[(size_t)r * FFN + col] = y > 0.f ? y : 0.f; });
      }
      ARRIVE();
      GemvW<FFN, 1> w_2;
      gemv_issue_b(w_2, L.w2, DIM, L.b2);
      WAIT();
      // (6) delta = hid W2^T + b2, the hidden rows staged HID_TILE at a time
      for (int i0 = 0; i0 < sb.nact; i0 += HID_TILE) {
        const int n = min(HID_TILE, sb.nact - i0);
        for (int e = tid * 4; e < n * FFN; e += MTT * 4)
          *reinterpret_cast<float4*>(vb + e) = *reinterpret_cast<const float4*>(P.hid + (size_t)sb.act[i0 + e / FFN] * FFN + e % FFN);
        __syncthreads();
        for (int k = 0; k < n; ++k) {
          const int r = sb.act[i0 + k];
          gemv_finish_b(w_2, vb + k * FFN, DIM, [&](int col, float y) { P.delta[(size_t)r * DIM + col] = y; });
        }
        __syncthreads();
      }
      ARRIVE();
      if (l + 1 < P.n_layers) {
        const MtLayerP Ln = layers[l + 1];
        gemv_issue_b(w_qkv, Ln.wqkv, 3 * DIM, Ln.bqkv);
      }
      WAIT();
    }
    // ---- final LN and logits over the tied embedding for every unfinished row
    GemvW<DIM, 6> w_out;
    gemv_issue(w_out, P.emb, P.vocab);
    add_delta_rows(sb, xs, P.delta);
    ln_rows(sb, xs, vb, P.out_g, P.out_b);
    if ((kMode == kMtbPrefix || (kMode == kMtbIncremental && P.feats)) && blockIdx.x == 0)
      for (int e = tid; e < sb.nact * DIM; e += MTT) {
        const int r = sb.act[e / DIM], c = e % DIM;
        P.feats[((size_t)r * P.feats_ld + row_pos<kMode>(P, r, s)) * DIM + c] = vb[r * DIM + c];
      }
    for (int i = 0; i < sb.nact; ++i) {
      const int r = sb.act[i];
      gemv_finish(w_out, vb + r * DIM, P.vocab, [&](int col, float acc) { P.logits[(size_t)r * P.vocab + col] = acc; });
    }
    BAR();
    if constexpr (kMode == kMtbBeam) {
      // ---- candidates: live row i on CTA i; then the selection: sample j on CTA j (xs is free until the next step's embedding)
      const int64_t* tok_s = alt ? B.tok2 : P.tok;
      int64_t* const tok_nx = alt ? P.tok : B.tok2;
      const float* cum = B.cum + (alt ? (size_t)P.rows * P.tok_ld : 0);
      float* cum_nx = B.cum + (alt ? 0 : (size_t)P.rows * P.tok_ld);
      for (int i = blockIdx.x; i < sb.nact; i += gridDim.x) beam_row_candidates(sm, P, B, sb.act[i], s, cum, vb, xs);
      BAR();
      for (int j = blockIdx.x; j < P.rows / B.beam; j += gridDim.x)
        if (!B.done[j]) beam_select(P, B, j, s, tok_s, tok_nx, cum, cum_nx, vb, xs);
    } else {
      // ---- arg-max: unfinished row i on CTA i (eos forced at the row's max_len)
      for (int i = blockIdx.x; i < sb.nact; i += gridDim.x) {
        const int r = sb.act[i];
        const int pos = row_pos<kMode>(P, r, s);
        const int tk = (kMode != kMtbOffline && pos >= P.max_len[r]) ? P.eos : masked_argmax(sm, P.logits + (size_t)r * P.vocab, P.vocab, P.pad, P.eos, pos);
        if (tid == 0) {
          P.tok[(size_t)r * P.tok_ld + s + 1] = tk;
          if (tk == P.eos) P.fin[r] = 1;
        }
      }
    }
    BAR();
    load_active(sb, P.fin, P.rows);
  }
#undef BAR
#undef ARRIVE
#undef WAIT
  // leave the barrier counter where the host expects it after a full burst
  const int planned = nsteps * barriers_per_step;
  if (threadIdx.x == 0 && done_barriers < planned) atomicAdd(bar_ctr, (unsigned)(planned - done_barriers));
}

}  // namespace

int mt_decode_batch(const MtBatchParams& P, const MtLayerP* layers_dev, int step0, int nsteps, unsigned* bar_ctr, unsigned* bar_target_host,
                    cudaStream_t st, const MtBeamParams* beam_p) {
  ++g_launches;
  if (P.rows < 1 || P.rows > MAXR) return -1;
  const bool rows = P.start != nullptr, inc = P.self_row != nullptr, beam = beam_p != nullptr;
  if (rows && (!P.max_len || !P.cross_row || (!P.feats && !inc))) return -1;  // the per-row fields come together
  if (inc && (!rows || !P.kv_off || P.self_ld < 1)) return -1;
  const MtBeamParams B = beam ? *beam_p : MtBeamParams{};
  if (beam && (rows || B.beam < 1 || B.beam > MAXR || P.rows % B.beam != 0 || 2 * B.beam > P.vocab || B.max_len + 2 > P.tok_ld ||
               (B.beam > 1 && (!B.self_k2 || !B.self_v2))))
    return -1;
  const void* kernel = beam   ? (const void*)mt_decode_batch_kernel<kMtbBeam>
                       : inc  ? (const void*)mt_decode_batch_kernel<kMtbIncremental>
                       : rows ? (const void*)mt_decode_batch_kernel<kMtbPrefix>
                              : (const void*)mt_decode_batch_kernel<kMtbOffline>;
  if (first_time_on_device(kernel)) {  // cooperative launch needs one resident CTA per SM
    cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kDynSmem);
    int occ = 0;
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kernel, MTT, kDynSmem);
    if (occ < 1) return -1;
  }
  const int grid = current_device_sms();
  if (grid < 8 * GRP || grid < MAXR || P.vocab > 6 * MW * grid) return -1;  // head groups; one round of columns per GEMV phase
  MtBatchParams p = P;
  unsigned bar_target = *bar_target_host;
  MtBeamParams b = B;
  void* args[] = {(void*)&p, (void*)&layers_dev, (void*)&step0, (void*)&nsteps, (void*)&bar_ctr, (void*)&bar_target, (void*)&b};
  if (cudaLaunchCooperativeKernel(kernel, dim3(grid), dim3(MTT), args, kDynSmem, st) != cudaSuccess) return -2;
  *bar_target_host += (unsigned)grid * (unsigned)(nsteps * (P.n_layers * 6 + (beam ? 3 : 2)));
  return 0;
}

}  // namespace ss
