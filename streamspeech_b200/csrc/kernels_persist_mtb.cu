// Greedy MT search (beam 1, no prefix) for up to MT_BATCH_MAX_ROWS independent samples in one persistent cooperative kernel:
// the offline generator's batch decoded together.  The phases are those of mt_decode_persistent_kernel_v2 (6 split barriers
// per layer), and each phase's weights are loaded into registers ONCE per step and applied to every unfinished row:
//   per layer: [LN + QKV] | [self-attn + Wo partials] | [x += sum, LN + Wcq] | [cross-attn + Wco partials] |
//              [x += sum, LN + FC1 + ReLU] | [FC2 -> delta]
//   then:      [x += delta, final LN, logits = E @ feat] | [arg-max of log_softmax, row i on CTA i]
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
// columns: part[r][h][col] = sum_{i < 64} a[i] * W[col][64 h + i], warp w owning columns [64 w, 64 w + 64)
template <typename KV>
__device__ __forceinline__ void attend_rows(MtSmem& sm, MtbSmem& sb, const float* q, KV&& kv, const float* __restrict__ W, int h, int j,
                                            float* part) {
  int nloc = 0;
  for (int i = j; i < sb.nact; i += GRP, ++nloc) {
    const int r = sb.act[i];
    const float* kb;
    const float* vbase;
    int ld, n;
    kv(r, kb, vbase, ld, n);
    attend_head_early(sm, q + (size_t)r * DIM + h * MHD, kb + h * MHD, vbase + h * MHD, ld, n, sb.att[nloc]);
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

__device__ __forceinline__ void load_active(MtbSmem& sb, const int* fin, int rows) {
  if (threadIdx.x == 0) {
    int n = 0;
    for (int r = 0; r < rows; ++r)
      if (*(volatile const int*)(fin + r) == 0) sb.act[n++] = r;
    sb.nact = n;
  }
  __syncthreads();
}

__global__ void __launch_bounds__(MTT, 1) mt_decode_batch_kernel(MtBatchParams P, const MtLayerP* __restrict__ layers, int step0, int nsteps,
                                                                 unsigned* bar_ctr, unsigned bar_target) {
  __shared__ __align__(16) MtSmem sm;
  __shared__ MtbSmem sb;
  extern __shared__ __align__(16) float dyn[];
  float* xs = dyn;               // [MAXR][DIM] residual rows
  float* vb = dyn + MAXR * DIM;  // [MAXR][DIM] LayerNorm rows, or [HID_TILE][FFN] hidden rows
  const int tid = threadIdx.x;
  const int barriers_per_step = P.n_layers * 6 + 2;
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
    for (int e = tid; e < sb.nact * DIM; e += MTT) {
      const int r = sb.act[e / DIM], c = e % DIM;
      const int64_t tok = P.tok[(size_t)r * P.tok_ld + s];
      const int p = (tok == P.pad) ? P.pad : P.pad + 1 + s;
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
      float* kl = P.self_k + (size_t)l * MAXR * P.tok_ld * DIM;
      float* vl = P.self_v + (size_t)l * MAXR * P.tok_ld * DIM;
      const float* cl = P.cross_kv + (size_t)l * MAXR * P.cross_cap * 2 * DIM;
      // (1) x += FFN delta of the previous layer; q | k | v = LN(x) Wqkv^T
      if (l > 0) add_delta_rows(sb, xs, P.delta);
      ln_rows(sb, xs, vb, L.self_g, L.self_b);
      for (int i = 0; i < sb.nact; ++i) {
        const int r = sb.act[i];
        float* kc = kl + ((size_t)r * P.tok_ld + s) * DIM;
        float* vc = vl + ((size_t)r * P.tok_ld + s) * DIM;
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
        attend_rows(sm, sb, P.q, [&](int r, const float*& kb, const float*& vbs, int& ld, int& n) {
          kb = kl + (size_t)r * P.tok_ld * DIM;
          vbs = vl + (size_t)r * P.tok_ld * DIM;
          ld = DIM;
          n = s + 1;
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
        attend_rows(sm, sb, P.q, [&](int r, const float*& kb, const float*& vbs, int& ld, int& n) {
          kb = cl + (size_t)r * P.cross_cap * 2 * DIM;
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
    for (int i = 0; i < sb.nact; ++i) {
      const int r = sb.act[i];
      gemv_finish(w_out, vb + r * DIM, P.vocab, [&](int col, float acc) { P.logits[(size_t)r * P.vocab + col] = acc; });
    }
    BAR();
    // ---- arg-max: unfinished row i on CTA i
    for (int i = blockIdx.x; i < sb.nact; i += gridDim.x) {
      const int r = sb.act[i];
      const int tk = masked_argmax(sm, P.logits + (size_t)r * P.vocab, P.vocab, P.pad, P.eos, s);
      if (tid == 0) {
        P.tok[(size_t)r * P.tok_ld + s + 1] = tk;
        if (tk == P.eos) P.fin[r] = 1;
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
                    cudaStream_t st) {
  ++g_launches;
  if (P.rows < 1 || P.rows > MAXR) return -1;
  if (first_time_on_device((const void*)mt_decode_batch_kernel)) {  // cooperative launch needs one resident CTA per SM
    cudaFuncSetAttribute(mt_decode_batch_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kDynSmem);
    int occ = 0;
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, mt_decode_batch_kernel, MTT, kDynSmem);
    if (occ < 1) return -1;
  }
  const int grid = current_device_sms();
  if (grid < 8 * GRP || grid < MAXR || P.vocab > 6 * MW * grid) return -1;  // head groups; one round of columns per GEMV phase
  MtBatchParams p = P;
  unsigned bar_target = *bar_target_host;
  void* args[] = {(void*)&p, (void*)&layers_dev, (void*)&step0, (void*)&nsteps, (void*)&bar_ctr, (void*)&bar_target};
  if (cudaLaunchCooperativeKernel((void*)mt_decode_batch_kernel, dim3(grid), dim3(MTT), args, kDynSmem, st) != cudaSuccess) return -2;
  *bar_target_host += (unsigned)grid * (unsigned)(nsteps * (P.n_layers * 6 + 2));
  return 0;
}

}  // namespace ss
