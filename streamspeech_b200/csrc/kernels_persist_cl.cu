// Cluster version of the streaming encoder step (option persistent_encoder_cluster): the <= 16 active rows are split over 4
// thread-block clusters of 16 CTAs (4 rows per cluster), and inside a cluster the activations NEVER leave the chip: every CTA keeps
// the cluster's residual rows in shared memory and GEMM outputs are exchanged through distributed shared memory instead of global
// memory + a grid barrier over one CTA per SM (every phase of kernels_persist.cu).  Only two steps per layer
// involve the other clusters -- the K / V rows and the conv-module GLU rows of the step are published to the per-layer caches in
// global memory -- and keep a (split) grid barrier over the 64 CTAs.
//
//   per layer and cluster (CTA rank c of 16):
//     FFN  : LN (local) -> W1 rows [128c, 128c+128) -> SiLU -> rank-128 update with W2^T rows [128c, ..) -> partial [4][256]
//            -> reduce-scatter (rank d sums the 16 partials of columns [16d, 16d+16) in rank order) -> bias, 0.5, residual
//            -> all-gather of the new residual columns
//     MHA  : LN -> q | k | v columns [16c, 16c+16) -> k, v to the global cache, q to the 4 CTAs of its head -> grid arrive ->
//            CTA (head c / 4, key part c % 4): scores of all 4 rows against its keys of earlier steps -> grid wait -> keys of this step ->
//            partial softmax / PV -> all-gather of (acc[64], max, sum) -> every CTA combines -> Wo columns [16c, ..) + residual -> all-gather
//     conv : LN -> PW1 GLU channels [16c, ..) -> GLU rows to the global conv cache -> grid barrier -> depthwise k31 + BN + SiLU on those
//            channels -> all-gather -> PW2 columns + residual -> all-gather
//     FFN, final LayerNorm (local: every CTA holds complete rows)
//   exchanges: st.async into the receiver's buffer, counted in bytes on the receiver's mbarrier (no cluster barriers: their release
//   fence is a MEMBAR.ALL.GPU).
//   weights: each (layer, rank) owns one contiguous blob in consumption order (a 15 KB parameter block + 21 chunks of <= 32 KB, packed
//   once); a producer warp streams it with cp.async.bulk (TMA) into a 5-slot ring of shared memory, ahead of the 8 compute warps and
//   independent of every exchange.  Each cluster reads all weights (4 x 123 MB through L2, 1 x from HBM: ncu 136 MB per launch).
// fp32 CUDA-core arithmetic as in kernels_persist.cu (different summation order: ~2e-6 on the encoder output).
// Design notes and measurements: DESIGN.md 5a.
#include <cooperative_groups.h>

#include "common.cuh"
#include "kernels.h"
#include "kernels_persist.h"

namespace cg = cooperative_groups;

namespace ss {
namespace {

constexpr int CT = 256;              // compute threads (8 warps); warp 8 is the weight-copy producer
constexpr int CWP = CT / 32;
constexpr int CT_ALL = CT + 32;
constexpr int CS = 16;               // cluster size
constexpr int CR = 4;                // rows per cluster
constexpr int NCL = 4;               // clusters
constexpr int CD = 256;              // model dim
constexpr int CHD = 64;
constexpr int NSLOT = 5;
constexpr int SLOT_FLOATS = 32 * CD; // 32 KB
constexpr int CHUNKS_PER_LAYER = 21;

// rows (of 256 floats) of chunk j of a layer blob: W1 4 x 32 | W2T 4 x 32 | q+k 32 | v 16 | wo 16 | pw1 32 | pw2 16 | W1 4 x 32 | W2T 4 x 32
__host__ __device__ constexpr int chunk_rows(int j) { return (j == 9 || j == 10 || j == 12) ? 16 : 32; }
__host__ __device__ constexpr int chunk_row0(int j) {
  int r = 0;
  for (int i = 0; i < j; ++i) r += chunk_rows(i);
  return r;
}
constexpr int BLOB_ROWS = chunk_row0(CHUNKS_PER_LAYER);  // 624
// small per-layer vectors of a rank (LayerNorm parameters, the rank's bias slices, its head's pos biases, its 16 depthwise channels):
// one 15 KB block in front of the weight rows, double-buffered in shared memory so no phase waits on a global load
constexpr int PO_FFN1_G = 0, PO_FFN1_B = 256, PO_ATTN_G = 512, PO_ATTN_B = 768, PO_CONV_G = 1024, PO_CONV_B = 1280, PO_FFN2_G = 1536,
              PO_FFN2_B = 1792, PO_FIN_G = 2048, PO_FIN_B = 2304, PO_FFN1_B1 = 2560, PO_FFN2_B1 = 2688, PO_FFN1_B2 = 2816, PO_FFN2_B2 = 2832,
              PO_BQKV = 2848, PO_BO = 2896, PO_PW1B = 2912, PO_PW2B = 2944, PO_BN_S = 2960, PO_BN_H = 2976, PO_POSU = 2992, PO_POSV = 3056,
              PO_DW = 3120, PO_END = PO_DW + 31 * 16;
constexpr int PAR_FLOATS = 15 * CD;  // 3840 >= PO_END (3616)
static_assert(PO_END <= PAR_FLOATS, "parameter block");
constexpr size_t BLOB_STRIDE = (size_t)PAR_FLOATS + (size_t)BLOB_ROWS * CD;  // floats per (layer, rank)

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// Exchange channels: a receive buffer in every CTA's shared memory plus an mbarrier that counts the bytes landing in it.  Senders
// store with st.async (remote write + complete_tx on the receiver's mbarrier); the receiver arms the expected byte count and waits
// for the phase -- no cluster barrier and no cluster-scope release fence (which is a MEMBAR.ALL.GPU).
// A buffer is reused only after an all-to-all exchange on another channel, which a sender cannot pass before every receiver has
// finished reading (it needs the receiver's own contribution, sent after those reads), so no flow control is needed.
enum { CH_RED = 0, CH_XS = 1, CH_QS = 2, CH_ATTP = 3, CH_AS = 4, N_CH = 5 };

__device__ __forceinline__ uint32_t mapa_u32(uint32_t local, int rank) {
  uint32_t remote;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(remote) : "r"(local), "r"(rank));
  return remote;
}
// value -> `local`'s address in CTA `rank`, counted on that CTA's mbarrier `bar_local` (both given as this CTA's addresses)
__device__ __forceinline__ void st_peer(const float* local, int rank, float v, const unsigned long long* bar_local) {
  asm volatile("st.async.weak.shared::cluster.mbarrier::complete_tx::bytes.b32 [%0], %1, [%2];" ::"r"(mapa_u32(smem_u32(local), rank)),
               "r"(__float_as_uint(v)), "r"(mapa_u32(smem_u32(bar_local), rank))
               : "memory");
}

__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  uint32_t done = 0;
  while (!done) {
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                 : "=r"(done)
                 : "r"(bar), "r"(parity)
                 : "memory");
  }
}

__device__ __forceinline__ unsigned long long globaltimer_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

// cluster barrier with release / acquire ordering of the distributed-shared-memory stores (all 288 threads of all 16 CTAs)
__device__ __forceinline__ void cluster_sync() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}

// CTA barrier of the 8 compute warps (the producer warp never joins it)
__device__ __forceinline__ void csync() { asm volatile("bar.sync 1, 256;" ::: "memory"); }

// split form: arrive publishes this CTA's global writes, wait returns when all CTAs have arrived
__device__ __forceinline__ void grid_arrive(unsigned* ctr, unsigned& target) {
  csync();
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
  csync();
}

struct ClSmem {
  float xs[CR][CD];          // residual rows of the cluster (replicated in every CTA)
  float As[CR][CD];          // staged GEMM input: LayerNorm output, gathered attention rows or gathered depthwise rows
  union {                    // FFN phases | attention phase (both receive buffers are written by peers only inside their phase)
    struct {
      float hs[CR][128];       // this CTA's 128 hidden units
      float red[CS][CR][16];   // reduce-scatter receive buffer: red[src][row][col of this CTA's 16-column slice]
    } f;
    float attp[CS][CR][CHD + 2];  // attention partials of every CTA of the cluster: acc[64], max, sum of exponentials
  } u;
  struct {
    float S[CR][256];          // scores / exponentials of this CTA's key slots (0 where the row may not attend the key)
    float ml[CR][2];
    float pv[4][CR][CHD];      // per key group partial outputs
  } att;
  float qs[CR][CHD];         // queries of this CTA's head (4 rows), gathered from the 4 column owners
  float qa[CR][CHD], qb[CR][CHD];
  float outc[CR][48];        // raw outputs of a column-split GEMM (q | k | v, or 32 GLU inputs, or 16 columns)
  float par[2][PAR_FLOATS];  // parameter block of layer li in par[li & 1]
  unsigned long long full[NSLOT];
  unsigned long long empty[NSLOT];  // one arrival per warp when it has finished reading the slot
  unsigned long long parfull[2];
  unsigned long long parfree[2];    // the compute warps are done with the parameter buffer (one arrival per layer)
  unsigned long long xbar[N_CH];    // exchange channels (bytes landed in the receive buffers)
};

// As[r][:] = LN(xs[r][:]) * g + b (warp r; rows are complete in every CTA); ends with a CTA barrier
__device__ __noinline__ void stage_ln(ClSmem& sm, const float* g, const float* b) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (warp < CR) {
    float v[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) v[i] = sm.xs[warp][lane + (i << 5)];
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) s += v[i];
    const float mean = warp_sum(s) / (float)CD;
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float d = v[i] - mean;
      q = fmaf(d, d, q);
    }
    const float rstd = 1.0f / sqrtf(warp_sum(q) / (float)CD + 1e-5f);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int c = lane + (i << 5);
      sm.As[warp][c] = (v[i] - mean) * rstd * g[c] + b[c];
    }
  }
  csync();
}

// Column-split GEMM of one ring chunk (row-major weight rows of 256 floats, `rows` = 32 or 16 of them) against the 4 staged rows As.
// Lane l holds x[r][4 l .. 4 l + 4) and x[r][128 + 4 l ..) of the 4 rows in registers for the whole phase (load_x) and reads its 32 B
// of each weight row (every lane a distinct 16 B: full-rate 128-bit shared-memory loads, each weight byte read once); the 16 (weight
// row j = warp + 8 s, activation row r) partial sums of a warp are reduced over the 32 lanes with a halving tree (16 shuffles);
// even lane 2 v ends with the sum v = s * 4 + r.  (A (k group, row) lane mapping needs 4 shuffles but 4 x the shared-memory
// wavefronts -- lanes sharing a 16 B address still cost a quarter-warp phase each.)
struct XRegs {
  float4 v[CR][2];
};
__device__ __forceinline__ void load_x(const ClSmem& sm, XRegs& x) {
  const int lane = threadIdx.x & 31;
#pragma unroll
  for (int r = 0; r < CR; ++r) {
    x.v[r][0] = *reinterpret_cast<const float4*>(&sm.As[r][lane * 4]);
    x.v[r][1] = *reinterpret_cast<const float4*>(&sm.As[r][128 + lane * 4]);
  }
}

template <int rows>
__device__ __forceinline__ void chunk_fma(const XRegs& x, const float* wchunk, float (&acc)[16]) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int s = 0; s < 4; ++s) {
    if (s * CWP >= rows) {  // (compile time: a 16-row chunk has two weight rows per warp)
#pragma unroll
      for (int r = 0; r < CR; ++r) acc[s * 4 + r] = 0.f;
      continue;
    }
    const float4 w0 = *reinterpret_cast<const float4*>(wchunk + (warp + s * CWP) * CD + lane * 4);
    const float4 w1 = *reinterpret_cast<const float4*>(wchunk + (warp + s * CWP) * CD + 128 + lane * 4);
#pragma unroll
    for (int r = 0; r < CR; ++r) {
      float a = x.v[r][0].x * w0.x;
      a = fmaf(x.v[r][0].y, w0.y, a);
      a = fmaf(x.v[r][0].z, w0.z, a);
      a = fmaf(x.v[r][0].w, w0.w, a);
      a = fmaf(x.v[r][1].x, w1.x, a);
      a = fmaf(x.v[r][1].y, w1.y, a);
      a = fmaf(x.v[r][1].z, w1.z, a);
      a = fmaf(x.v[r][1].w, w1.w, a);
      acc[s * 4 + r] = a;
    }
  }
}

template <int rows>
__device__ __forceinline__ float chunk_tree(const float (&acc)[16]) {
  const int lane = threadIdx.x & 31;
  const bool b4 = lane & 16, b3 = lane & 8, b2 = lane & 4, b1 = lane & 2;
  float w4[4], w2[2];
  if (rows > 16) {
    float w8[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) w8[i] = (b4 ? acc[i + 8] : acc[i]) + __shfl_xor_sync(0xffffffffu, b4 ? acc[i] : acc[i + 8], 16);
#pragma unroll
    for (int i = 0; i < 4; ++i) w4[i] = (b3 ? w8[i + 4] : w8[i]) + __shfl_xor_sync(0xffffffffu, b3 ? w8[i] : w8[i + 4], 8);
  } else {
    // slots 0, 1 only: 8 sums; bit 4 is summed in full, bit 3 selects the slot
    float w8[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) w8[i] = acc[i] + __shfl_xor_sync(0xffffffffu, acc[i], 16);
#pragma unroll
    for (int i = 0; i < 4; ++i) w4[i] = (b3 ? w8[i + 4] : w8[i]) + __shfl_xor_sync(0xffffffffu, b3 ? w8[i] : w8[i + 4], 8);
  }
#pragma unroll
  for (int i = 0; i < 2; ++i) w2[i] = (b2 ? w4[i + 2] : w4[i]) + __shfl_xor_sync(0xffffffffu, b2 ? w4[i] : w4[i + 2], 4);
  float v = (b1 ? w2[1] : w2[0]) + __shfl_xor_sync(0xffffffffu, b1 ? w2[0] : w2[1], 2);
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  return v;
}

// out(j, r, value) on the lane that owns (weight row j of the chunk, activation row r).  rows = 32: lane bits (4, 3) = s, bits (2, 1)
// = r; rows = 16: bit 3 = s (bit 4 lanes hold copies), bits (2, 1) = r
template <int rows, typename F>
__device__ __forceinline__ void chunk_epi(float v, F&& out) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const bool owner = rows > 16 ? (lane & 1) == 0 : (lane & 17) == 0;
  if (owner) {
    const int s = rows > 16 ? (lane >> 3) : ((lane >> 3) & 1);
    out(warp + s * CWP, (lane >> 1) & 3, v);
  }
}

template <int rows, typename F>
__device__ __forceinline__ void chunk_gemm(const XRegs& x, const float* wchunk, F&& out) {
  float acc[16];
  chunk_fma<rows>(x, wchunk, acc);
  chunk_epi<rows>(chunk_tree<rows>(acc), out);
}

// Two 32-row chunks through ONE tree: 32 partial sums (index = chunk * 16 + s * 4 + r) -> every lane ends with one complete sum
// (lane bit 4 = chunk, bits (3, 2) = s, bits (1, 0) = r): 31 shuffles for two chunks in 5 dependent levels instead of 2 x 5
__device__ __forceinline__ float pair_tree(const float (&a0)[16], const float (&a1)[16]) {
  const int lane = threadIdx.x & 31;
  const bool b4 = lane & 16, b3 = lane & 8, b2 = lane & 4, b1 = lane & 2, b0 = lane & 1;
  float w16[16], w8[8], w4[4], w2[2];
#pragma unroll
  for (int i = 0; i < 16; ++i) w16[i] = (b4 ? a1[i] : a0[i]) + __shfl_xor_sync(0xffffffffu, b4 ? a0[i] : a1[i], 16);
#pragma unroll
  for (int i = 0; i < 8; ++i) w8[i] = (b3 ? w16[i + 8] : w16[i]) + __shfl_xor_sync(0xffffffffu, b3 ? w16[i] : w16[i + 8], 8);
#pragma unroll
  for (int i = 0; i < 4; ++i) w4[i] = (b2 ? w8[i + 4] : w8[i]) + __shfl_xor_sync(0xffffffffu, b2 ? w8[i] : w8[i + 4], 4);
#pragma unroll
  for (int i = 0; i < 2; ++i) w2[i] = (b1 ? w4[i + 2] : w4[i]) + __shfl_xor_sync(0xffffffffu, b1 ? w4[i] : w4[i + 2], 2);
  return (b0 ? w2[1] : w2[0]) + __shfl_xor_sync(0xffffffffu, b0 ? w2[0] : w2[1], 1);
}

struct ClParams {
  const PersistLayer* layers;  // (not read by the kernel: every weight and parameter comes from the blobs; the pack kernels read it)
  const float* blobs;          // [n_layers][CS][BLOB_STRIDE]: per (layer, rank) the parameter block, then 624 weight rows of 256 floats
  int n_layers;
  float* x;                    // [nA][256] active rows (in: encoder.linear output, out: layer-stack output)
  float *kc, *vc, *gc;         // per-layer caches [n_layers][Tpos][256]
  int nA, a0, T, Tpos, chunk, conv_chunk, dw_k;
  unsigned* bar_ctr;
  unsigned bar_target;
  const float* pos_proj[16];   // per layer: projected relative-position table [2 * Tpos - 1][256]
  unsigned long long* ts;      // profiling (option persistent_profile): ts[0] = number of stamps, then (id, ns) pairs of CTA 0, layer 1
};

// one ring chunk (`rows` = 32 or 16 weight rows) against the staged rows: sm.outc[r][off + j] = sum_k As[r][k] w[j][k] + bias[off + j].
// NOT inlined: the five single-chunk GEMMs of a layer share one copy of the code (the kernel's instruction footprint decides how
// much of every phase is instruction-fetch latency: the L1.5 instruction cache holds 32 KB and each layer runs its code once).
__device__ __noinline__ void gemm_chunk(ClSmem* smp, const float* wchunk, int rows, int off, const float* bias) {
  ClSmem& sm = *smp;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  XRegs x;
  load_x(sm, x);
  float acc[16];
  chunk_fma<32>(x, wchunk, acc);  // (a 16-row chunk: slots 2, 3 read stale rows of the ring slot; their sums are dropped below)
  const float v = chunk_tree<32>(acc);
  if ((lane & 1) == 0) {
    const int j = warp + (lane >> 3) * CWP;
    if (j < rows) sm.outc[(lane >> 1) & 3][off + j] = v + bias[off + j];
  }
}

__global__ void __launch_bounds__(CT_ALL, 1) encoder_layers_cluster_kernel(ClParams P) {  // (9 warps are allocated like 12: 168 registers)
  extern __shared__ __align__(128) unsigned char dyn[];
  ClSmem& sm = *reinterpret_cast<ClSmem*>(dyn);
  float* ring = reinterpret_cast<float*>(dyn + ((sizeof(ClSmem) + 127) & ~(size_t)127));
  cg::cluster_group cluster = cg::this_cluster();
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int c = (int)cluster.block_rank();           // rank in the cluster
  const int g = blockIdx.x / CS;                     // cluster index = row group
  const int r_lo = g * CR;
  const int nr = max(0, min(CR, P.nA - r_lo));       // valid rows of this cluster
  unsigned bar_target = P.bar_target;
  const int total_chunks = P.n_layers * CHUNKS_PER_LAYER;

  if (tid == 0) {
    for (int i = 0; i < NSLOT; ++i) asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(smem_u32(&sm.full[i])));
    for (int i = 0; i < NSLOT; ++i) asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(&sm.empty[i])), "r"(CWP));
    for (int i = 0; i < 2; ++i) asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(smem_u32(&sm.parfull[i])));
    for (int i = 0; i < 2; ++i) asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(smem_u32(&sm.parfree[i])));
    for (int i = 0; i < N_CH; ++i) asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(smem_u32(&sm.xbar[i])));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  // residual rows of the cluster (zero rows where the cluster has fewer than 4)
  for (int i = tid; i < CR * CD; i += CT_ALL) {
    const int r = i / CD;
    sm.xs[r][i - r * CD] = r < nr ? P.x[(int64_t)(r_lo + r) * CD + (i - r * CD)] : 0.f;
  }
  __syncthreads();

  if (warp == CWP) {
    // ---- producer warp.  Chunk qi of this rank's stream goes to ring slot qi % NSLOT; lane 0 refills a slot when all 8 compute warps
    // have released it.  The warp joins every cluster barrier (all threads of the cluster must), so it services the releases that
    // precede each one; per layer the compute warps release   FFN 8 | 0 | q k v 2 | attention 0 | Wo 1 | PW1 1 | PW2 1 | FFN 8 | 0
    // chunks before the 9 barriers.  The refills behind the q / k / v and PW1 chunks are deferred past the attention / depthwise phases
    // (their global loads would queue behind 32 KB weight copies on the SM's memory port; nothing needs those slots that early).
    auto issue = [&](int qi) {
      const int slot = qi % NSLOT;
      const int li = qi / CHUNKS_PER_LAYER, j = qi - li * CHUNKS_PER_LAYER;
      const int row0 = 32 * j - 16 * ((j > 9) + (j > 10) + (j > 12));  // = chunk_row0(j): chunks 9, 10, 12 have 16 rows
      const uint32_t bytes = (uint32_t)chunk_rows(j) * CD * 4u;
      const float* src = P.blobs + (size_t)(li * CS + c) * BLOB_STRIDE + PAR_FLOATS + (size_t)row0 * CD;
      // (WAR on the slot: the readers' mbarrier arrivals, observed by this thread, order their reads before the copy)
      asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(&sm.full[slot])), "r"(bytes) : "memory");
      asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(ring + (size_t)slot * SLOT_FLOATS)),
                   "l"(src), "r"(bytes), "r"(smem_u32(&sm.full[slot]))
                   : "memory");
    };
    auto issue_par = [&](int li) {
      if (li >= P.n_layers) return;
      const uint32_t bytes = PAR_FLOATS * 4u;
      const uint32_t bar = smem_u32(&sm.parfull[li & 1]);
      asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
      asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(&sm.par[li & 1][0])),
                   "l"(P.blobs + (size_t)(li * CS + c) * BLOB_STRIDE), "r"(bytes), "r"(bar)
                   : "memory");
    };
    // L2 prefetch of what this CTA's attention of layer `pl` will read from earlier steps' rows (the weight stream of a step evicts them)
    auto prefetch_attn = [&](int pl) {
      const int h = c >> 2, p = c & 3;
      if (pl < P.n_layers && nr > 0) {
        const int i0 = P.a0 + r_lo, il = i0 + nr - 1;
        const int lim = min(P.chunk > 0 ? min((il / P.chunk + 1) * P.chunk, P.T) : P.T, P.a0);
        const char* kb = reinterpret_cast<const char*>(P.kc + (size_t)pl * P.Tpos * CD + h * CHD);
        const char* vb = reinterpret_cast<const char*>(P.vc + (size_t)pl * P.Tpos * CD + h * CHD);
        const char* pb = reinterpret_cast<const char*>(P.pos_proj[pl] + h * CHD);
        const int ns = lim > p ? (lim - p + 3) >> 2 : 0;  // this CTA's keys j = 4 slot + p
#pragma unroll 1
        for (int x = lane; x < 2 * ns; x += 32) {
          const int j = 4 * (x >> 1) + p;
          const size_t half = (x & 1) * 128;
          asm volatile("prefetch.global.L2 [%0];" ::"l"(kb + (size_t)j * CD * 4 + half));
          asm volatile("prefetch.global.L2 [%0];" ::"l"(vb + (size_t)j * CD * 4 + half));
#pragma unroll
          for (int r = 0; r < CR; ++r) asm volatile("prefetch.global.L2 [%0];" ::"l"(pb + (size_t)(i0 + r - j + P.Tpos - 1) * CD * 4 + half));
        }
      }
    };
    if (lane == 0) {
      issue_par(0);
      issue_par(1);
    }
    prefetch_attn(0);
    cluster_sync();  // (start-up barrier)
#pragma unroll 1
    for (int issued = 0; issued < total_chunks; ++issued) {
      const int li = issued / CHUNKS_PER_LAYER, j = issued - li * CHUNKS_PER_LAYER;
      if (lane == 0) {
        if (issued >= NSLOT) mbar_wait(smem_u32(&sm.empty[issued % NSLOT]), (uint32_t)(((issued - NSLOT) / NSLOT) & 1));
        issue(issued);
      }
      __syncwarp();
      if (j == 8) {
        // the compute warps are past chunk 3 of layer li, so layer li - 1 is done: its parameter buffer takes layer li + 1
        const int L = li + 1;
        if (L >= 2 && L < P.n_layers && lane == 0) {
          mbar_wait(smem_u32(&sm.parfree[L & 1]), (uint32_t)(((L - 2) >> 1) & 1));
          issue_par(L);
        }
        prefetch_attn(L);
      }
    }
    cluster_sync();  // (exit barrier)
    return;
  }

  cluster_sync();  // every CTA of the cluster runs and has initialised its shared memory before any DSMEM traffic
  int q = 0;       // chunk counter
  auto acquire = [&]() -> const float* {
    mbar_wait(smem_u32(&sm.full[q % NSLOT]), (uint32_t)((q / NSLOT) & 1));
    return ring + (size_t)(q % NSLOT) * SLOT_FLOATS;
  };
  auto release = [&]() {  // this warp has finished reading the slot
    __syncwarp();
    if (lane == 0) asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(&sm.empty[q % NSLOT])) : "memory");
    ++q;
  };
  unsigned xph = 0;  // phase parity per exchange channel
  auto xwait = [&](int ch, uint32_t bytes) {
    const uint32_t bar = smem_u32(&sm.xbar[ch]);
    if (tid == 0) asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
    mbar_wait(bar, (xph >> ch) & 1u);
    xph ^= 1u << ch;
  };
  int nts = 0;
  bool stamping = false;
  auto stamp = [&](int id) {
    if (stamping && tid == 0) {
      P.ts[1 + 2 * nts] = (unsigned long long)id;
      P.ts[2 + 2 * nts] = globaltimer_ns();
      ++nts;
    }
  };
  // xs[:, 16 c .. 16 c + 16) += outc[:, 0 .. 16) + bias, all-gathered over the cluster (epilogue of a column-split GEMM)
  auto residual_gather = [&](const float* bias) {
    csync();
    if (tid < CR * 16) {
      const int r = tid >> 4, j = tid & 15;
      const float y = sm.xs[r][c * 16 + j] + (sm.outc[r][j] + bias[j]);
#pragma unroll 1
      for (int d = 0; d < CS; ++d) st_peer(&sm.xs[r][c * 16 + j], d, y, &sm.xbar[CH_XS]);
    }
    xwait(CH_XS, CS * CR * 16 * 4);
  };
  const int h = c >> 2, p = c & 3;  // attention: head and key part of this CTA
  // keys row r may attend: [0, lim_of(r)); rows past the cluster's last valid one attend nothing
  auto lim_of = [&](int r) {
    const int i = P.a0 + r_lo + r;
    return r < nr ? (P.chunk > 0 ? min((i / P.chunk + 1) * P.chunk, P.T) : P.T) : 0;
  };
  const int lim_max = nr > 0 ? lim_of(nr - 1) : 0;  // (non-decreasing in r)
  const int ns_all = lim_max > p ? (lim_max - p + 3) >> 2 : 0;  // this CTA's key slots: j = 4 slot + p < lim_max
  const int ns_old = min(ns_all, (P.a0 - p + 3) >> 2);          // ... of which written by earlier steps (j < a0)

#pragma unroll 1
  for (int li = 0; li < P.n_layers; ++li) {
    const float* pos_proj = P.pos_proj[li];
    mbar_wait(smem_u32(&sm.parfull[li & 1]), (uint32_t)((li >> 1) & 1));
    const float* par = sm.par[li & 1];
    stamping = P.ts != nullptr && blockIdx.x == 0 && li == 1;
    stamp(0);
    float* kc = P.kc + (size_t)li * P.Tpos * CD;
    float* vc = P.vc + (size_t)li * P.Tpos * CD;
    float* gc = P.gc + (size_t)li * P.Tpos * CD;
#pragma unroll 1
    for (int half = 0; half < 2; ++half) {
      // ================= FFN: xs += 0.5 * (W2 silu(W1 LN(xs) + b1) + b2), 8 chunks =================
      {
        const float* b1 = par + (half ? PO_FFN2_B1 : PO_FFN1_B1);
        const float* b2 = par + (half ? PO_FFN2_B2 : PO_FFN1_B2);
        stage_ln(sm, par + (half ? PO_FFN2_G : PO_FFN1_G), par + (half ? PO_FFN2_B : PO_FFN1_B));
        {
          XRegs x;
          load_x(sm, x);
#pragma unroll 1
          for (int pair = 0; pair < 2; ++pair) {
            float a0[16], a1[16];
            chunk_fma<32>(x, acquire(), a0);
            release();
            chunk_fma<32>(x, acquire(), a1);
            release();
            const float v = pair_tree(a0, a1);
            // lane = chunk * 16 + s * 4 + r  ->  hidden unit (of this rank's 128) = (2 pair + chunk) * 32 + warp + 8 s
            const int u = (2 * pair + (lane >> 4)) * 32 + warp + ((lane >> 2) & 3) * CWP;
            const float y = v + b1[u];
            sm.u.f.hs[lane & 3][u] = __fdividef(y, 1.0f + expf(-y));
          }
        }
        csync();  // hs complete
        // rank-128 update: thread = (column pair cp = tid % 128, half kh = tid / 128 of each chunk's 32 hidden units): one 8-byte weight
        // load and four broadcast loads per 8 FMAs; the two halves are added through shared memory
        float acc[CR][2] = {};
        {
          const int cp = tid & 127, kh = tid >> 7;
#pragma unroll 1
          for (int part = 0; part < 4; ++part) {
            const float* w = acquire() + (kh * 16) * CD + 2 * cp;
            const float* hb = &sm.u.f.hs[0][part * 32 + kh * 16];
#pragma unroll
            for (int u = 0; u < 16; u += 4) {
              float2 wv[4];
              float4 hv[CR];
#pragma unroll
              for (int x = 0; x < 4; ++x) wv[x] = *reinterpret_cast<const float2*>(w + (u + x) * CD);
#pragma unroll
              for (int r = 0; r < CR; ++r) hv[r] = *reinterpret_cast<const float4*>(hb + r * 128 + u);
#pragma unroll
              for (int r = 0; r < CR; ++r) {
                acc[r][0] = fmaf(hv[r].x, wv[0].x, acc[r][0]); acc[r][1] = fmaf(hv[r].x, wv[0].y, acc[r][1]);
                acc[r][0] = fmaf(hv[r].y, wv[1].x, acc[r][0]); acc[r][1] = fmaf(hv[r].y, wv[1].y, acc[r][1]);
                acc[r][0] = fmaf(hv[r].z, wv[2].x, acc[r][0]); acc[r][1] = fmaf(hv[r].z, wv[2].y, acc[r][1]);
                acc[r][0] = fmaf(hv[r].w, wv[3].x, acc[r][0]); acc[r][1] = fmaf(hv[r].w, wv[3].y, acc[r][1]);
              }
            }
            release();
          }
          // halves: kh = 1 hands its sums to kh = 0 through As (free until the next LayerNorm staging)
          if (kh == 1) {
#pragma unroll
            for (int r = 0; r < CR; ++r) *reinterpret_cast<float2*>(&sm.As[r][2 * cp]) = make_float2(acc[r][0], acc[r][1]);
          }
          csync();
          if (kh == 0) {
#pragma unroll
            for (int r = 0; r < CR; ++r) {
              const float2 o = *reinterpret_cast<const float2*>(&sm.As[r][2 * cp]);
              // reduce-scatter: column n belongs to rank n / 16
              st_peer(&sm.u.f.red[c][r][(2 * cp) & 15], (2 * cp) >> 4, acc[r][0] + o.x, &sm.xbar[CH_RED]);
              st_peer(&sm.u.f.red[c][r][(2 * cp + 1) & 15], (2 * cp + 1) >> 4, acc[r][1] + o.y, &sm.xbar[CH_RED]);
            }
          }
        }
        xwait(CH_RED, CS * CR * 16 * 4);
        if (tid < CR * 16) {
          const int r = tid >> 4, j = tid & 15;
          float t = sm.u.f.red[0][r][j];
#pragma unroll
          for (int s = 1; s < CS; ++s) t += sm.u.f.red[s][r][j];
          const float y = sm.xs[r][c * 16 + j] + 0.5f * (t + b2[j]);
#pragma unroll 1
          for (int d = 0; d < CS; ++d) st_peer(&sm.xs[r][c * 16 + j], d, y, &sm.xbar[CH_XS]);
        }
        xwait(CH_XS, CS * CR * 16 * 4);
      }
      stamp(half ? 11 : 1);
      if (half == 1) {
        // final LayerNorm of the layer, in place (every CTA holds the complete rows: no exchange)
        if (warp < CR) {
          float v[8];
#pragma unroll
          for (int i = 0; i < 8; ++i) v[i] = sm.xs[warp][lane + (i << 5)];
          float s = 0.f;
#pragma unroll
          for (int i = 0; i < 8; ++i) s += v[i];
          const float mean = warp_sum(s) / (float)CD;
          float qv = 0.f;
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            const float d = v[i] - mean;
            qv = fmaf(d, d, qv);
          }
          const float rstd = 1.0f / sqrtf(warp_sum(qv) / (float)CD + 1e-5f);
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            const int cc = lane + (i << 5);
            sm.xs[warp][cc] = (v[i] - mean) * rstd * par[PO_FIN_G + cc] + par[PO_FIN_B + cc];
          }
        }
        csync();
        if (tid == 0) asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(&sm.parfree[li & 1])) : "memory");
        stamp(12);
        if (stamping && tid == 0) P.ts[0] = (unsigned long long)nts;
        break;
      }
      // ================= attention block =================
      // CTA c = (head h = c / 4, key part p = c % 4): it attends ALL 4 rows of the cluster over the keys j = 4 slot + p of head h and
      // all-gathers the un-normalised partial (acc[64], max, sum) per row; every CTA then combines the 16 partials into the 4 complete
      // attention rows (one cluster barrier, each CTA reads a quarter of K / V / pos instead of all of it).
      stage_ln(sm, par + PO_ATTN_G, par + PO_ATTN_B);
      gemm_chunk(&sm, acquire(), 32, 0, par + PO_BQKV);   // q -> outc[:, 0..16), k -> outc[:, 16..32)
      release();
      gemm_chunk(&sm, acquire(), 16, 32, par + PO_BQKV);  // v -> outc[:, 32..48)
      release();
      csync();
      if (tid < CR * 16) {
        const int r = tid >> 4, j = tid & 15;
        if (r < nr) {
          kc[(int64_t)(P.a0 + r_lo + r) * CD + c * 16 + j] = sm.outc[r][16 + j];
          vc[(int64_t)(P.a0 + r_lo + r) * CD + c * 16 + j] = sm.outc[r][32 + j];
        }
        // q columns [16 c, 16 c + 16) = dims [16 p, 16 p + 16) of head h: to the 4 CTAs of the head
#pragma unroll 1
        for (int pp = 0; pp < 4; ++pp) st_peer(&sm.qs[r][p * 16 + j], (c & ~3) + pp, sm.outc[r][j], &sm.xbar[CH_QS]);
      }
      grid_arrive(P.bar_ctr, bar_target);  // K / V rows of this CTA are published; the wait comes after the work on older keys
      xwait(CH_QS, 4 * CR * 16 * 4);       // q gathered
      stamp(2);
      {
        const int r = tid >> 6, d = tid & 63;
        const float qv = sm.qs[r][d];
        sm.qa[r][d] = qv + par[PO_POSU + d];
        sm.qb[r][d] = qv + par[PO_POSV + d];
      }
      csync();
      {
        // scores: half a warp per key (lane l16 holds dims [4 l16, 4 l16 + 4) of q + u, q + v of the 4 rows and loads 16 B of the key row
        // and of the 4 relative-position rows), 2 keys per half-warp in flight; first the keys of earlier steps, then -- after the
        // grid barrier -- the keys of this step
        const float* kb = kc + h * CHD;
        const float* pb = pos_proj + h * CHD;
        const int hw = tid >> 4, l16 = tid & 15;
        float4 qa4[CR], qb4[CR];
#pragma unroll
        for (int r = 0; r < CR; ++r) {
          qa4[r] = *reinterpret_cast<const float4*>(&sm.qa[r][4 * l16]);
          qb4[r] = *reinterpret_cast<const float4*>(&sm.qb[r][4 * l16]);
        }
        const int i0 = P.a0 + r_lo;  // position of row 0
        const bool b3 = l16 & 8, b2 = l16 & 4;
        const int rown = (b3 ? 2 : 0) + (b2 ? 1 : 0);  // the row whose score this lane ends up with
        const int lim_own = lim_of(rown);
#pragma unroll 1
        for (int ph = 0; ph < 2; ++ph) {
          if (ph == 1) {
            stamp(3);
            grid_wait(P.bar_ctr, bar_target);  // K / V rows of all clusters are in the cache
            stamp(4);
          }
          const int s1 = ph ? ns_all : ns_old;
#pragma unroll 1
          for (int sb = ph ? ns_old : 0; sb < s1; sb += 32) {
            float4 kk[2], pp4[2][CR];
#pragma unroll
            for (int u = 0; u < 2; ++u) {
              const int slot = sb + u * 16 + hw, j = 4 * slot + p;
              const bool ok = slot < s1;
              kk[u] = ok ? *reinterpret_cast<const float4*>(kb + (int64_t)j * CD + 4 * l16) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
              for (int r = 0; r < CR; ++r)
                pp4[u][r] = ok ? *reinterpret_cast<const float4*>(pb + (int64_t)(i0 + r - j + P.Tpos - 1) * CD + 4 * l16) : make_float4(0.f, 0.f, 0.f, 0.f);
            }
#pragma unroll
            for (int u = 0; u < 2; ++u) {
              const int slot = sb + u * 16 + hw, j = 4 * slot + p;
              float sc[CR];
#pragma unroll
              for (int r = 0; r < CR; ++r) {
                float t = qa4[r].x * kk[u].x;
                t = fmaf(qa4[r].y, kk[u].y, t); t = fmaf(qa4[r].z, kk[u].z, t); t = fmaf(qa4[r].w, kk[u].w, t);
                t = fmaf(qb4[r].x, pp4[u][r].x, t); t = fmaf(qb4[r].y, pp4[u][r].y, t);
                t = fmaf(qb4[r].z, pp4[u][r].z, t); t = fmaf(qb4[r].w, pp4[u][r].w, t);
                sc[r] = t;
              }
              // 4 sums over 16 lanes: halving on lane bits 3, 2, then full sums over bits 1, 0
              const float t0 = (b3 ? sc[2] : sc[0]) + __shfl_xor_sync(0xffffffffu, b3 ? sc[0] : sc[2], 8);
              const float t1 = (b3 ? sc[3] : sc[1]) + __shfl_xor_sync(0xffffffffu, b3 ? sc[1] : sc[3], 8);
              float v = (b2 ? t1 : t0) + __shfl_xor_sync(0xffffffffu, b2 ? t0 : t1, 4);
              v += __shfl_xor_sync(0xffffffffu, v, 2);
              v += __shfl_xor_sync(0xffffffffu, v, 1);
              if ((l16 & 3) == 0 && slot < s1) sm.att.S[rown][slot] = j < lim_own ? v * 0.125f : -INFINITY;
            }
          }
        }
      }
      csync();
      // per row: max and sum of my keys' exponentials (warp r); keys the row may not attend get weight 0
      if (warp < CR) {
        const int lw = lim_of(warp);
        const int ns = lw > p ? (lw - p + 3) >> 2 : 0;
        float mx = -INFINITY;
#pragma unroll 1
        for (int sl = lane; sl < ns; sl += 32) mx = fmaxf(mx, sm.att.S[warp][sl]);
        mx = warp_max(mx);
        float sum = 0.f;
#pragma unroll 1
        for (int sl = lane; sl < ns_all; sl += 32) {
          const float e = sl < ns ? expf(sm.att.S[warp][sl] - mx) : 0.f;
          sm.att.S[warp][sl] = e;
          sum += e;
        }
        sum = warp_sum(sum);
        if (lane == 0) {
          sm.att.ml[warp][0] = mx;
          sm.att.ml[warp][1] = sum;
        }
      }
      csync();
      {
        // un-normalised outputs over my keys: thread = (dim d, key group kg of 4): each V element is loaded once and used for the 4
        // rows; all loads of a thread (<= 16 at T <= 256) in flight at once; the 4 key groups are summed through shared memory
        const int kg = tid >> 6, d = tid & 63;
        const float* vb = vc + h * CHD + d;
        float acc[CR] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll 1
        for (int sb = kg; sb < ns_all; sb += 64) {
          float vv[16];
#pragma unroll
          for (int u = 0; u < 16; ++u) vv[u] = sb + 4 * u < ns_all ? vb[(int64_t)(4 * (sb + 4 * u) + p) * CD] : 0.f;
#pragma unroll
          for (int u = 0; u < 16; ++u) {
            const bool ok = sb + 4 * u < ns_all;  // (S past the last slot was never written: select, do not multiply by 0)
#pragma unroll
            for (int r = 0; r < CR; ++r) acc[r] = fmaf(ok ? sm.att.S[r][min(sb + 4 * u, 255)] : 0.f, vv[u], acc[r]);
          }
        }
#pragma unroll
        for (int r = 0; r < CR; ++r) sm.att.pv[kg][r][d] = acc[r];
        csync();
        const int r = tid >> 6;
        const float tot = sm.att.pv[0][r][d] + sm.att.pv[1][r][d] + sm.att.pv[2][r][d] + sm.att.pv[3][r][d];
        const float mv = sm.att.ml[r][d & 1];
#pragma unroll 1
        for (int dst = 0; dst < CS; ++dst) {
          st_peer(&sm.u.attp[c][r][d], dst, tot, &sm.xbar[CH_ATTP]);
          if (d < 2) st_peer(&sm.u.attp[c][r][CHD + d], dst, mv, &sm.xbar[CH_ATTP]);
        }
      }
      stamp(5);
      xwait(CH_ATTP, CS * CR * (CHD + 2) * 4);
      {
        // combine: As[r][hh * 64 + d] = sum_p e^(m_p - M) acc_p[d] / sum_p e^(m_p - M) l_p over the 4 key parts of head hh
        const int r = tid >> 6, d = tid & 63;
#pragma unroll 1
        for (int hh = 0; hh < 4; ++hh) {
          float m[4], M = -INFINITY;
#pragma unroll
          for (int pp = 0; pp < 4; ++pp) {
            m[pp] = sm.u.attp[hh * 4 + pp][r][CHD];
            M = fmaxf(M, m[pp]);
          }
          float num = 0.f, den = 0.f;
#pragma unroll
          for (int pp = 0; pp < 4; ++pp) {
            const float l = sm.u.attp[hh * 4 + pp][r][CHD + 1];
            const float wgt = l > 0.f ? expf(m[pp] - M) : 0.f;
            num = fmaf(wgt, sm.u.attp[hh * 4 + pp][r][d], num);
            den = fmaf(wgt, l, den);
          }
          sm.As[r][hh * CHD + d] = den > 0.f ? num / den : 0.f;
        }
      }
      csync();
      stamp(6);
      gemm_chunk(&sm, acquire(), 16, 0, par + PO_END);  // Wo rows [16 c, 16 c + 16) (bias added with the residual; par[PO_END..] is 0)
      release();
      residual_gather(par + PO_BO);
      stamp(7);
      // ================= conv module =================
      stage_ln(sm, par + PO_CONV_G, par + PO_CONV_B);
      gemm_chunk(&sm, acquire(), 32, 0, par + PO_PW1B);  // PW1: interleaved (value, gate) rows of channels [16 c, 16 c + 16)
      release();
      csync();
      if (tid < CR * 16) {
        const int r = tid >> 4, ch = tid & 15;
        if (r < nr) {
          const float a = sm.outc[r][2 * ch], gate = sm.outc[r][2 * ch + 1];
          gc[(int64_t)(P.a0 + r_lo + r) * CD + c * 16 + ch] = a * (1.0f / (1.0f + expf(-gate)));
        }
      }
      grid_arrive(P.bar_ctr, bar_target);
      stamp(8);
      grid_wait(P.bar_ctr, bar_target);  // GLU rows of all clusters are in the conv cache
      {
        // depthwise conv + BatchNorm + SiLU of (row r, channel ch): 4 lanes take 8 taps each (all loads in flight), summed by shuffle
        const int r = tid >> 6, ch = (tid >> 2) & 15, tg = tid & 3, oc = c * 16 + ch;
        const int t = P.a0 + r_lo + r, half_k = (P.dw_k - 1) >> 1;
        const int lim = r < nr ? (P.conv_chunk > 0 ? min(P.T, (t / P.conv_chunk + 1) * P.conv_chunk) : P.T) : 0;
        float gv[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) {  // (rows outside the sequence / chunk and taps >= dw_k contribute 0)
          const int tap = tg * 8 + j, pz = t - half_k + tap;
          gv[j] = (tap < P.dw_k && pz >= 0 && pz < lim) ? gc[(int64_t)pz * CD + oc] : 0.f;
        }
        float a = 0.f;
#pragma unroll
        for (int j = 0; j < 8; ++j) a = fmaf(tg * 8 + j < 31 ? par[PO_DW + (tg * 8 + j) * 16 + ch] : 0.f, gv[j], a);
        a += __shfl_xor_sync(0xffffffffu, a, 1);
        a += __shfl_xor_sync(0xffffffffu, a, 2);
        const float v = a * par[PO_BN_S + ch] + par[PO_BN_H + ch];
        const float y = r < nr ? v / (1.0f + expf(-v)) : 0.f;
        // all-gather of the depthwise rows: lane tg stores to ranks tg, tg + 4, ...
#pragma unroll 1
        for (int d = tg; d < CS; d += 4) st_peer(&sm.As[r][oc], d, y, &sm.xbar[CH_AS]);
      }
      stamp(9);
      xwait(CH_AS, CS * CR * 16 * 4);
      gemm_chunk(&sm, acquire(), 16, 0, par + PO_END);  // PW2 rows [16 c, 16 c + 16)
      release();
      residual_gather(par + PO_PW2B);
      stamp(10);
    }
  }
  if (c == 0) {
    for (int i = tid; i < nr * CD; i += CT) P.x[(int64_t)r_lo * CD + i] = sm.xs[i / CD][i % CD];
  }
  cluster_sync();  // no CTA exits while a peer may still address its shared memory
}

// weight row `row` of (layer li, rank c): see the chunk table above.  One thread per float4.
__global__ void cluster_pack_kernel(const PersistLayer* __restrict__ layers, int n_layers, float* __restrict__ blobs) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;  // float4 index
  const int64_t total = (int64_t)n_layers * CS * BLOB_ROWS * (CD / 4);
  if (idx >= total) return;
  const int k4 = (int)(idx % (CD / 4));
  int64_t t = idx / (CD / 4);
  const int row = (int)(t % BLOB_ROWS);
  t /= BLOB_ROWS;
  const int c = (int)(t % CS), li = (int)(t / CS);
  const PersistLayer& L = layers[li];
  const float* src;
  if (row < 128) src = L.ffn1_w1 + (int64_t)(c * 128 + row) * CD;
  else if (row < 256) src = L.ffn1_w2t + (int64_t)(c * 128 + row - 128) * CD;
  else if (row < 272) src = L.wqkv + (int64_t)(c * 16 + row - 256) * CD;
  else if (row < 288) src = L.wqkv + (int64_t)(CD + c * 16 + row - 272) * CD;
  else if (row < 304) src = L.wqkv + (int64_t)(2 * CD + c * 16 + row - 288) * CD;
  else if (row < 320) src = L.wo + (int64_t)(c * 16 + row - 304) * CD;
  else if (row < 352) src = L.pw1 + (int64_t)(c * 32 + row - 320) * CD;
  else if (row < 368) src = L.pw2 + (int64_t)(c * 16 + row - 352) * CD;
  else if (row < 496) src = L.ffn2_w1 + (int64_t)(c * 128 + row - 368) * CD;
  else src = L.ffn2_w2t + (int64_t)(c * 128 + row - 496) * CD;
  float* dst = blobs + (size_t)(li * CS + c) * BLOB_STRIDE + PAR_FLOATS + (size_t)row * CD;
  reinterpret_cast<float4*>(dst)[k4] = reinterpret_cast<const float4*>(src)[k4];
}

// parameter block of (layer li, rank c): one thread per float
__global__ void cluster_pack_params_kernel(const PersistLayer* __restrict__ layers, int n_layers, int dw_k, float* __restrict__ blobs) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n_layers * CS * PAR_FLOATS) return;
  const int o = idx % PAR_FLOATS, c = (idx / PAR_FLOATS) % CS, li = idx / (PAR_FLOATS * CS);
  const PersistLayer& L = layers[li];
  float v = 0.f;
  if (o < PO_FFN1_B1) {
    const float* tab[10] = {L.ffn1_g, L.ffn1_b, L.attn_g, L.attn_b, L.conv_g, L.conv_b, L.ffn2_g, L.ffn2_b, L.fin_g, L.fin_b};
    v = tab[o >> 8][o & 255];
  } else if (o < PO_FFN2_B1) v = L.ffn1_b1[c * 128 + o - PO_FFN1_B1];
  else if (o < PO_FFN1_B2) v = L.ffn2_b1[c * 128 + o - PO_FFN2_B1];
  else if (o < PO_FFN2_B2) v = L.ffn1_b2[c * 16 + o - PO_FFN1_B2];
  else if (o < PO_BQKV) v = L.ffn2_b2[c * 16 + o - PO_FFN2_B2];
  else if (o < PO_BO) v = L.bqkv[((o - PO_BQKV) >> 4) * CD + c * 16 + ((o - PO_BQKV) & 15)];
  else if (o < PO_PW1B) v = L.bo[c * 16 + o - PO_BO];
  else if (o < PO_PW2B) v = L.pw1_b ? L.pw1_b[c * 32 + o - PO_PW1B] : 0.f;
  else if (o < PO_BN_S) v = L.pw2_b ? L.pw2_b[c * 16 + o - PO_PW2B] : 0.f;
  else if (o < PO_BN_H) v = L.bn_scale[c * 16 + o - PO_BN_S];
  else if (o < PO_POSU) v = L.bn_shift[c * 16 + o - PO_BN_H];
  else if (o < PO_POSV) v = L.pos_u[(c >> 2) * CHD + o - PO_POSU];
  else if (o < PO_DW) v = L.pos_v[(c >> 2) * CHD + o - PO_POSV];
  else if (o < PO_END) {
    const int tap = (o - PO_DW) >> 4, ch = (o - PO_DW) & 15;
    v = tap < dw_k ? L.dw_w[tap * CD + c * 16 + ch] : 0.f;
  }
  blobs[(size_t)(li * CS + c) * BLOB_STRIDE + o] = v;
}

}  // namespace

size_t encoder_layers_cluster_blob_floats(int n_layers) { return (size_t)n_layers * CS * BLOB_STRIDE; }

void encoder_layers_cluster_pack(const PersistLayer* layers_dev, int n_layers, int dw_k, float* blobs_dev, cudaStream_t st) {
  const int64_t total = (int64_t)n_layers * CS * BLOB_ROWS * (CD / 4);
  cluster_pack_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(layers_dev, n_layers, blobs_dev);
  const int np = n_layers * CS * PAR_FLOATS;
  cluster_pack_params_kernel<<<(np + 255) / 256, 256, 0, st>>>(layers_dev, n_layers, dw_k, blobs_dev);
}

bool encoder_layers_cluster_supported(int nA, int D, int FFN, int H, int T, int dw_k) {
  return nA >= 1 && nA <= NCL * CR && D == CD && FFN == 2048 && H * CHD == D && T <= 1024 && (dw_k & 1) == 1 && dw_k <= 31;
}

int encoder_layers_cluster(const PersistLayer* layers_dev, const float* blobs_dev, int n_layers, float* x, float* kc, float* vc, float* gc, int nA,
                           int a0, int T, int Tpos, int chunk, int conv_chunk, int dw_k, unsigned* bar_ctr, unsigned* bar_target_host,
                           unsigned long long* ts_or_null, const float* const* pos_proj_host, int cooperative, cudaStream_t st) {
  if (n_layers > 16) return -1;
  ++g_launches;
  const size_t smem = ((sizeof(ClSmem) + 127) & ~(size_t)127) + (size_t)NSLOT * SLOT_FLOATS * sizeof(float);
  if (first_time_on_device((const void*)encoder_layers_cluster_kernel)) {
    if (cudaFuncSetAttribute(encoder_layers_cluster_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) return -1;
    if (cudaFuncSetAttribute(encoder_layers_cluster_kernel, cudaFuncAttributeNonPortableClusterSizeAllowed, 1) != cudaSuccess) return -1;
  }
  ClParams P;
  P.layers = layers_dev; P.blobs = blobs_dev; P.n_layers = n_layers; P.x = x; P.kc = kc; P.vc = vc; P.gc = gc;
  P.nA = nA; P.a0 = a0; P.T = T; P.Tpos = Tpos; P.chunk = chunk; P.conv_chunk = conv_chunk; P.dw_k = dw_k;
  P.bar_ctr = bar_ctr; P.bar_target = *bar_target_host; P.ts = ts_or_null;
  for (int i = 0; i < 16; ++i) P.pos_proj[i] = i < n_layers ? pos_proj_host[i] : nullptr;
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(NCL * CS);
  cfg.blockDim = dim3(CT_ALL);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[2];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = CS;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  attr[1].id = cudaLaunchAttributeCooperative;  // all 4 clusters co-resident (they meet in a grid barrier)
  attr[1].val.cooperative = 1;
  cfg.attrs = attr;
  cfg.numAttrs = cooperative ? 2 : 1;  // (without the attribute co-residency is not guaranteed: only under a profiler that serialises kernels)
  int max_clusters = 0;
  if (cudaOccupancyMaxActiveClusters(&max_clusters, encoder_layers_cluster_kernel, &cfg) != cudaSuccess || max_clusters < NCL) {
    cudaGetLastError();
    return -1;  // the 64 CTAs could not be co-resident: their grid barrier would time out
  }
  if (cudaLaunchKernelEx(&cfg, encoder_layers_cluster_kernel, P) != cudaSuccess) return -2;
  *bar_target_host += (unsigned)(NCL * CS) * (unsigned)(2 * n_layers);
  return 0;
}

}  // namespace ss
