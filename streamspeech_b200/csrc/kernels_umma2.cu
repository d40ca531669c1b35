// wgmma implicit-GEMM convolution / linear kernel (warp-specialised, weights pre-packed).
//
//   out[t][n] = epilogue( sum_{tap j, channel ci}  pre(x[t + j*dil - pad_left][ci]) * W[n][j*C_in + ci] )
//
// for stride-1 convolutions over one channels-last sequence (B = 1; a plain linear layer is ksize = 1).  fp32 operands are
// split into NP bf16 pieces (x = x0 + x1 [+ x2]) and the product is accumulated in fp32 registers as 3 (NP = 2, ~2^-16
// relative) or 6 (NP = 3, ~fp32) bf16 wgmma products.  Structure:
//
//   * weights are split and laid out ONCE (umma2_pack_kernel, cached per weight matrix) as ready-made shared-memory tiles
//     [n-tile][channel chunk][tap][piece][BN x CK bf16, canonical no-swizzle K-major core matrices]; a producer thread
//     streams them with cp.async.bulk (the TMA engine's 1-D bulk copy) into a ring of SB stages, completion on mbarriers;
//   * the activation rows of an output tile are converted ONCE per channel chunk, halo included: rows
//     [m0 - pad_left, m0 + 128 + (k-1)*dil - pad_left) x CK channels.  In the no-swizzle layout a plane of 8 channels is a
//     linear array of rows at a 16-byte pitch, so tap j is the same staged data with the descriptor's start address moved
//     by j*dil rows: a k-tap convolution costs k MMAs per staged chunk instead of k im2col conversions;
//   * roles: warps 0-7 are two warpgroups that convert (global fp32 -> registers, one chunk ahead -> bf16 pieces in smem)
//     and issue the wgmma of their 64 rows of the 128-row tile; warp 8 runs the weight ring.  The MMAs of a (chunk, tap)
//     unit run asynchronously while the next unit is issued and the next chunk is converted; a unit's weight stage (and,
//     after its last tap, the activation stage) is released once the following unit has been issued and it has completed.
//     The accumulators go through a padded shared-memory tile so the fused epilogue writes whole rows.
//   * split over (chunk, tap) units on gridDim.z when the tile grid alone cannot fill the GPU; partial sums are reduced
//     in a fixed order by splitk_epilogue_kernel (kernels_gemm.cu).
#include <cuda_bf16.h>

#include <algorithm>
#include <map>
#include <tuple>
#include <vector>

#include "common.cuh"
#include "kernels.h"
#include "kernels_persist.h"

namespace ss {

namespace {

constexpr int U2_BM = 128;
constexpr int U2_CONVERTERS = 256;  // warps 0-7 (two warpgroups of 64 output rows each)
constexpr int U2_THREADS = 288;     // + weight-ring warp
constexpr int U2_MAX_UNITS = 6;     // float4 units per converter thread and chunk: rows * CK/4 <= 6 * 256
constexpr int U2_MAX_SB = 4;
constexpr int U2_MAX_HALO = 64;

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ float u2_act(float x, int act) {
  switch (act) {
    case ACT_RELU: return x > 0.f ? x : 0.f;
    case ACT_SILU: return x / (1.0f + expf(-x));
    case ACT_TANH: return tanhf(x);
    case ACT_GELU: return 0.5f * x * (1.0f + erff(x * 0.70710678118654752f));
    default: return x;
  }
}

// K-major, no-swizzle wgmma shared-memory matrix descriptor
__device__ __forceinline__ uint64_t u2_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr >> 4) & 0x3FFF);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;  // next 8-column plane along K
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;  // next 8-row group along M / N
  return d;
}

// D[64 x BN] += A[64 x 16] * B[BN x 16]^T, bf16 operands in shared memory, fp32 accumulators in registers.  Register 4 i + r of
// thread t of the warpgroup holds row 16 (t / 32) + (t % 32) / 4 + 8 (r / 2), column 8 i + 2 (t % 4) + r % 2.
template <int BN>
__device__ __forceinline__ void u2_wgmma(float (&d)[BN / 2], uint64_t a, uint64_t b);
template <>
__device__ __forceinline__ void u2_wgmma<16>(float (&d)[8], uint64_t a, uint64_t b) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
      : "l"(a), "l"(b), "r"(1));
}
template <>
__device__ __forceinline__ void u2_wgmma<32>(float (&d)[16], uint64_t a, uint64_t b) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(a), "l"(b), "r"(1));
}
template <>
__device__ __forceinline__ void u2_wgmma<64>(float (&d)[32], uint64_t a, uint64_t b) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(a), "l"(b), "r"(1));
}
template <>
__device__ __forceinline__ void u2_wgmma<128>(float (&d)[64], uint64_t a, uint64_t b) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(a), "l"(b), "r"(1));
}

template <int NACC>
__device__ __forceinline__ void u2_fence_acc(float (&d)[NACC]) {
#pragma unroll
  for (int i = 0; i < NACC; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

__device__ __forceinline__ void u2_wait(uint32_t bar, uint32_t parity) {
  uint32_t done = 0;
  while (!done) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done)
        : "r"(bar), "r"(parity)
        : "memory");
  }
}

__device__ __forceinline__ void u2_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}

struct U2Params {
  ConvA a;
  Epilogue ep;
  const unsigned char* wp;  // packed weight tiles
  int M, N;
  int CK;                   // channels per chunk (16 or 32)
  int ksize, dil;
  int rs;                   // staged rows per chunk = 128 + (ksize - 1) * dil
  int rs_pad;               // row capacity of a staged 8-channel plane (plane = rs_pad * 16 bytes)
  int units_total;          // (C_in / CK) * ksize
  int units_per_split;
  int SB;                   // weight ring stages
  float* ws;                // split partial sums [gridDim.z][M][N] or null
  unsigned long long* dbg;  // optional: %globaltimer stamps of CTA (0,0,0) at the hand-off points (option umma2_debug)
};

__device__ __forceinline__ void u2_stamp(const U2Params& p, int slot) {
  if (p.dbg != nullptr && blockIdx.x == 0 && blockIdx.y == 0 && blockIdx.z == 0) {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    p.dbg[slot] = t;
  }
}

template <int NP>
__device__ __forceinline__ void u2_split_store(float4 v, unsigned char* stage, uint32_t piece_bytes, uint32_t off) {
#pragma unroll
  for (int p = 0; p < NP; ++p) {
    __nv_bfloat162 h01 = __floats2bfloat162_rn(v.x, v.y);
    __nv_bfloat162 h23 = __floats2bfloat162_rn(v.z, v.w);
    uint2 packed;
    packed.x = *reinterpret_cast<uint32_t*>(&h01);
    packed.y = *reinterpret_cast<uint32_t*>(&h23);
    *reinterpret_cast<uint2*>(stage + p * piece_bytes + off) = packed;
    if (p + 1 < NP) {
      v.x -= __low2float(h01);
      v.y -= __high2float(h01);
      v.z -= __low2float(h23);
      v.w -= __high2float(h23);
    }
  }
}

template <int BN, int NP, int UPT, int SETS>
__global__ void __launch_bounds__(U2_THREADS, 1) umma2_kernel(const __grid_constant__ U2Params p) {
  constexpr int NACC = BN / 2;
  constexpr int TP = BN + 8;  // pitch (floats) of the output tile: conflict-free 8-byte fragment stores
  extern __shared__ __align__(128) unsigned char smem[];
  __shared__ __align__(8) uint64_t bars[4 + 2 * U2_MAX_SB];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int m0 = blockIdx.y * U2_BM, nt = blockIdx.x, n0 = nt * BN;
  const int CK = p.CK, k = p.ksize, SB = p.SB;
  const uint32_t a_plane = (uint32_t)p.rs_pad * 16u;
  const uint32_t a_piece = (uint32_t)(CK >> 3) * a_plane;
  const uint32_t a_stage = NP * a_piece;
  const uint32_t b_piece = (uint32_t)BN * CK * 2u;
  const uint32_t b_unit = NP * b_piece;
  unsigned char* a_smem = smem + ((128u - (smem_u32(smem) & 127u)) & 127u);  // 128-byte aligned whatever the static layout is
  unsigned char* b_smem = a_smem + ((2 * a_stage + 127u) & ~127u);
  const uint32_t a_full = smem_u32(&bars[0]), a_empty = smem_u32(&bars[2]), b_full = smem_u32(&bars[4]);
  const uint32_t b_empty = smem_u32(&bars[4 + U2_MAX_SB]);

  const int u0 = blockIdx.z * p.units_per_split;
  const int u1 = min(p.units_total, u0 + p.units_per_split);
  const int n_units = u1 - u0;
  const int c_first = u0 / k, c_last = (u1 - 1) / k;
  const int n_local = c_last - c_first + 1;

  if (tid == 0) u2_stamp(p, 0);
  // ---- converter set-up (every warp computes the addresses; only warps 0-7 load)
  const int upr_shift = (CK == 32) ? 3 : 2;  // float4 units per row = CK / 4
  const int upr = 1 << upr_shift;
  const int n_a = p.rs * upr;
  int64_t goff[UPT];
  uint32_t soff[UPT];
#pragma unroll
  for (int i = 0; i < UPT; ++i) {
    const int idx = tid + i * U2_CONVERTERS;
    const int r = idx >> upr_shift, q = idx & (upr - 1);
    const int pos = m0 + r - p.a.pad_left;
    const bool inb = idx < n_a && pos >= 0 && pos < p.a.L_in;
    goff[i] = inb ? (int64_t)pos * p.a.ldx + q * 4 : (int64_t)-1;
    soff[i] = (uint32_t)(q >> 1) * a_plane + (uint32_t)r * 16u + (uint32_t)(q & 1) * 8u;
  }
  const float slope = p.a.pre_lrelu;
  // register ring of SETS chunk loads: while chunk cl is converted, the loads of chunks cl+1 .. cl+SETS-1 are in flight
  // (UPT = 6, SETS = 2 for convolutions with a halo; UPT = 4, SETS = 3 for linears, whose chunks carry few MMAs)
  float4 pf[SETS][UPT];
  auto issue = [&](int c, float4* dst) {
    const float* xc = p.a.x + (int64_t)c * CK;
#pragma unroll
    for (int i = 0; i < UPT; ++i)
      dst[i] = goff[i] >= 0 ? __ldg(reinterpret_cast<const float4*>(xc + goff[i])) : make_float4(0.f, 0.f, 0.f, 0.f);
  };
  if (warp < 8) {  // the first chunk loads do not depend on the barriers: they fly while the mbarriers are set up
#pragma unroll
    for (int d = 0; d < SETS - 1; ++d)
      if (d < n_local) issue(c_first + d, pf[d]);
  }

  if (tid == 0) {
    for (int i = 0; i < 2; ++i) {
      asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(a_full + 8 * i), "r"(U2_CONVERTERS / 32) : "memory");
      asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(a_empty + 8 * i), "r"(2) : "memory");  // one per warpgroup
    }
    for (int i = 0; i < U2_MAX_SB; ++i) {
      asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(b_full + 8 * i), "r"(1) : "memory");
      asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(b_empty + 8 * i), "r"(2) : "memory");
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (tid == 0) u2_stamp(p, 1);

  if (warp < 8) {
    // ---------------- converters + MMA issue: activation rows -> bf16 pieces, one channel chunk per stage
    const int wg = warp >> 2;  // warpgroup: output rows [64 wg, 64 wg + 64) of the tile
    const bool wg_leader = (tid & 127) == 0;
    float acc[NACC];
#pragma unroll
    for (int i = 0; i < NACC; ++i) acc[i] = 0.f;
    uint32_t uc = 0;
    int prev_sb = -1, prev_sa = -1;  // stages of the unit still in flight (prev_sa >= 0: it was the last tap of its chunk)
    for (int clb = 0; clb < n_local; clb += SETS) {
#pragma unroll
      for (int d = 0; d < SETS; ++d) {
        const int cl = clb + d;
        if (cl < n_local) {
          const int sa = cl & 1, ua = cl >> 1;
          if (cl + SETS - 1 < n_local) issue(c_first + cl + SETS - 1, pf[(d + SETS - 1) % SETS]);
          if (ua >= 1) u2_wait(a_empty + 8 * sa, (uint32_t)((ua - 1) & 1));  // the MMAs of chunk cl-2 have read this stage
          unsigned char* stage = a_smem + (size_t)sa * a_stage;
#pragma unroll
          for (int i = 0; i < UPT; ++i) {
            if (tid + i * U2_CONVERTERS < n_a) {
              float4 v = pf[d][i];
              if (slope != 1.0f) {
                v.x = v.x > 0.f ? v.x : v.x * slope;
                v.y = v.y > 0.f ? v.y : v.y * slope;
                v.z = v.z > 0.f ? v.z : v.z * slope;
                v.w = v.w > 0.f ? v.w : v.w * slope;
              }
              u2_split_store<NP>(v, stage, a_piece, soff[i]);
            }
          }
          // every lane publishes its own generic-proxy writes to the async proxy, then one lane per warp arrives
          asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
          __syncwarp();
          if (lane == 0) u2_arrive(a_full + 8 * sa);
          if (tid == 0 && cl == 0) u2_stamp(p, 2);
          u2_wait(a_full + 8 * sa, (uint32_t)(ua & 1));  // both warpgroups' rows are staged
          if (tid == 0 && cl == 0) u2_stamp(p, 3);
          const int c = c_first + cl;
          const int j_lo = (cl == 0) ? u0 - c * k : 0;
          const int j_hi = (cl == n_local - 1) ? (u1 - 1) - c * k : k - 1;
          const uint32_t a_base = smem_u32(a_smem + (size_t)sa * a_stage) + (uint32_t)wg * 64u * 16u;
          const uint32_t b_plane = (uint32_t)BN * 16u;
          for (int j = j_lo; j <= j_hi; ++j, ++uc) {
            const uint32_t sb = uc % (uint32_t)SB, ub = uc / (uint32_t)SB;
            u2_wait(b_full + 8 * sb, ub & 1u);
            if (tid == 0 && uc == 0) u2_stamp(p, 4);
            const uint32_t a_tap = a_base + (uint32_t)(j * p.dil) * 16u;
            const uint32_t b_base = smem_u32(b_smem + (size_t)sb * b_unit);
            u2_fence_acc<NACC>(acc);
            asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
            for (int ks = 0; ks < (CK >> 4); ++ks) {
              uint64_t ad[NP], bd[NP];
#pragma unroll
              for (int q = 0; q < NP; ++q) {
                ad[q] = u2_desc(a_tap + q * a_piece + ks * 2 * a_plane, a_plane, 128);
                bd[q] = u2_desc(b_base + q * b_piece + ks * 2 * b_plane, b_plane, 128);
              }
              u2_wgmma<BN>(acc, ad[0], bd[0]);
              u2_wgmma<BN>(acc, ad[0], bd[1]);
              u2_wgmma<BN>(acc, ad[1], bd[0]);
              if (NP == 3) {
                u2_wgmma<BN>(acc, ad[1], bd[1]);
                u2_wgmma<BN>(acc, ad[0], bd[NP - 1]);
                u2_wgmma<BN>(acc, ad[NP - 1], bd[0]);
              }
            }
            asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
            asm volatile("wgmma.wait_group.sync.aligned 1;" ::: "memory");  // the previous unit has completed
            u2_fence_acc<NACC>(acc);
            if (wg_leader && prev_sb >= 0) {
              u2_arrive(b_empty + 8 * prev_sb);
              if (prev_sa >= 0) u2_arrive(a_empty + 8 * prev_sa);
            }
            prev_sb = (int)sb;
            prev_sa = (j == j_hi) ? sa : -1;
          }
        }
      }
    }
    asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");
    u2_fence_acc<NACC>(acc);
    if (tid == 0) u2_stamp(p, 5);

    // ---------------- epilogue: accumulators -> padded shared-memory tile (the operand stages are free once both warpgroups'
    // MMAs have completed) -> rows written with lanes on consecutive columns: full 128-byte segments, bias / residual reads
    // coalesced too.  The mode (split partial sums / GLU / plain) is decided outside the loops.
    asm volatile("bar.sync 1, %0;" ::"n"(U2_CONVERTERS) : "memory");
    float* tile = reinterpret_cast<float*>(a_smem);
    {
      const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);
      const int c0 = 2 * (lane & 3);
#pragma unroll
      for (int i = 0; i < BN / 8; ++i) {
        *reinterpret_cast<float2*>(tile + r0 * TP + 8 * i + c0) = make_float2(acc[4 * i], acc[4 * i + 1]);
        *reinterpret_cast<float2*>(tile + (r0 + 8) * TP + 8 * i + c0) = make_float2(acc[4 * i + 2], acc[4 * i + 3]);
      }
    }
    asm volatile("bar.sync 1, %0;" ::"n"(U2_CONVERTERS) : "memory");
    if (tid == 0) u2_stamp(p, 7);
    const Epilogue& ep = p.ep;
    const int M = p.M, N = p.N;
    const int rows = min(U2_BM, M - m0);
    const int cols = min(BN, N - n0);
    if (p.ws != nullptr) {  // split: raw partial sums
      for (int idx = tid; idx < rows * BN; idx += U2_CONVERTERS) {
        const int r = idx / BN, c = idx - r * BN;
        if (c < cols) p.ws[((int64_t)blockIdx.z * M + m0 + r) * N + n0 + c] = tile[r * TP + c];
      }
    } else if (ep.glu) {  // columns are interleaved (a, gate) pairs
      constexpr int HB = BN / 2;
      for (int idx = tid; idx < rows * HB; idx += U2_CONVERTERS) {
        const int r = idx / HB, c = idx - r * HB;
        const int n = n0 + 2 * c;
        if (2 * c < cols) {
          const int m = m0 + r;
          const int64_t o = (ep.out_L > 0 ? (int64_t)m * ep.out_row_stride + ep.out_row_offset : (int64_t)m) * ep.ldo + (n >> 1);  // B == 1
          float v = tile[r * TP + 2 * c], gate = tile[r * TP + 2 * c + 1];
          if (ep.bias != nullptr) {
            v += ep.bias[n];
            gate += ep.bias[n + 1];
          }
          float res = 0.f;
          if (ep.residual) res = ep.res_scale * ep.residual[o];
          if (ep.accumulate) res += ep.out[o];
          ep.out[o] = ep.alpha * (v * (1.0f / (1.0f + expf(-gate)))) + res;
        }
      }
    } else {
      const int act = ep.act;
      for (int idx = tid; idx < rows * BN; idx += U2_CONVERTERS) {
        const int r = idx / BN, c = idx - r * BN;
        if (c < cols) {
          const int m = m0 + r, n = n0 + c;
          const int64_t o = (ep.out_L > 0 ? (int64_t)m * ep.out_row_stride + ep.out_row_offset : (int64_t)m) * ep.ldo + n;  // B == 1
          const float v = tile[r * TP + c] + (ep.bias != nullptr ? ep.bias[n] : 0.f);
          float res = 0.f;
          if (ep.residual) res = ep.res_scale * ep.residual[o];
          if (ep.accumulate) res += ep.out[o];
          ep.out[o] = ep.alpha * u2_act(v, act) + res;
        }
      }
    }
  } else if (warp == 8) {
    // ---------------- weight ring: one bulk copy per (chunk, tap) unit, all pieces
    if (lane == 0) {
      const unsigned char* src = p.wp + ((size_t)nt * p.units_total + u0) * b_unit;
      for (uint32_t uc = 0; uc < (uint32_t)n_units; ++uc) {
        const uint32_t sb = uc % (uint32_t)SB, ub = uc / (uint32_t)SB;
        if (ub >= 1) u2_wait(b_empty + 8 * sb, (ub - 1) & 1u);
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(b_full + 8 * sb), "r"(b_unit) : "memory");
        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                     ::"r"(smem_u32(b_smem + (size_t)sb * b_unit)), "l"(src + (size_t)uc * b_unit), "r"(b_unit), "r"(b_full + 8 * sb)
                     : "memory");
      }
    }
  }
  if (tid == 0) u2_stamp(p, 8);
}

// W[N][ksize*C_in] fp32 (tap-major columns) -> [n-tile][chunk][tap][piece][plane (8 channels)][row (BN)][8 bf16]
template <int NP>
__global__ void umma2_pack_kernel(const float* __restrict__ W, int N, int C_in, int ksize, int BN, int CK, int n_tiles,
                                  unsigned char* __restrict__ out) {
  const int planes = CK >> 3;
  const int n_chunks = C_in / CK;
  const int64_t total = (int64_t)n_tiles * n_chunks * ksize * planes * BN;  // one thread per (tile row, plane) = 8 channels
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  int r = (int)(idx % BN);
  int64_t t = idx / BN;
  int pl = (int)(t % planes); t /= planes;
  int j = (int)(t % ksize); t /= ksize;
  int c = (int)(t % n_chunks);
  int nt = (int)(t / n_chunks);
  const int n = nt * BN + r;
  float v[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) v[e] = n < N ? W[(int64_t)n * ksize * C_in + (int64_t)j * C_in + c * CK + pl * 8 + e] : 0.f;
  const size_t piece_bytes = (size_t)BN * CK * 2;
  unsigned char* unit = out + (((size_t)nt * n_chunks + c) * ksize + j) * NP * piece_bytes;
#pragma unroll
  for (int pc = 0; pc < NP; ++pc) {
    uint32_t w4[4];
#pragma unroll
    for (int e = 0; e < 8; e += 2) {
      __nv_bfloat162 h = __floats2bfloat162_rn(v[e], v[e + 1]);
      w4[e >> 1] = *reinterpret_cast<uint32_t*>(&h);
      v[e] -= __low2float(h);
      v[e + 1] -= __high2float(h);
    }
    *reinterpret_cast<uint4*>(unit + pc * piece_bytes + (size_t)pl * BN * 16 + (size_t)r * 16) = make_uint4(w4[0], w4[1], w4[2], w4[3]);
  }
}

constexpr int U2_SPLIT_BELOW = 60;  // tile grids smaller than this are split over (chunk, tap) units (below one wave, the extra
                                    // reduce launch can cost more than the idle SMs)
constexpr int U2_MIN_UNITS = 4;     // ... into slices of at least this many units

int u2_bn(int N) { return N >= 128 ? 128 : N > 32 ? 64 : N > 16 ? 32 : 16; }

template <int BN, int NP, int UPT, int SETS>
void u2_launch_v(const U2Params& p, dim3 grid, size_t smem, cudaStream_t st) {
  if (first_time_on_device((const void*)umma2_kernel<BN, NP, UPT, SETS>))
    cudaFuncSetAttribute(umma2_kernel<BN, NP, UPT, SETS>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
  umma2_kernel<BN, NP, UPT, SETS><<<grid, U2_THREADS, smem, st>>>(p);
}

template <int BN, int NP>
void u2_launch(const U2Params& p, int upt, dim3 grid, size_t smem, cudaStream_t st) {
  if (upt == 4) u2_launch_v<BN, NP, 4, 3>(p, grid, smem, st);
  else u2_launch_v<BN, NP, U2_MAX_UNITS, 2>(p, grid, smem, st);
}

}  // namespace

void umma2_cache_clear(Umma2Cache* c) {
  if (!c) return;
  cudaDeviceSynchronize();
  for (void* p : c->allocs) cudaFree(p);
  c->allocs.clear();
  c->packed.clear();
}

void umma2_cache_destroy(Umma2Cache* c) {
  if (!c) return;
  umma2_cache_clear(c);
  if (c->dbg) cudaFree(c->dbg);
  delete c;
}

bool umma2_supported(const ConvA& a, int N, const Epilogue& ep) {
  if (a.B != 1 || a.stride != 1 || a.chunk != 0 || a.lengths != nullptr) return false;
  if (a.t_offset != 0 || a.x_row0 != 0 || a.x_rows != 0) return false;
  if ((a.C_in & 15) != 0 || (a.ldx & 3) != 0 || a.C_in > a.ldx) return false;
  if ((reinterpret_cast<uintptr_t>(a.x) & 15) != 0) return false;
  if ((a.ksize - 1) * a.dil > U2_MAX_HALO || a.ksize < 1 || a.dil < 1) return false;
  if (N < 16 || (ep.glu && (N & 1))) return false;
  if (ep.ln_gamma != nullptr || ep.split_n > 0) return false;
  if (ep.out_L > 0 && a.L_rows <= 0) return false;
  return true;
}

const unsigned char* umma2_packed_weights(Umma2Cache* cache, const float* W, int N, int C_in, int k, int BN, int CK, int NP, cudaStream_t st) {
  auto key = std::make_tuple(W, N, C_in, k, BN, NP, CK);
  auto it = cache->packed.find(key);
  if (it != cache->packed.end()) return it->second;
  const int n_chunks = C_in / CK;
  const int n_tiles = (N + BN - 1) / BN;
  unsigned char* wp = nullptr;
  const size_t bytes = (size_t)n_tiles * n_chunks * k * NP * BN * CK * 2;
  if (cudaMalloc((void**)&wp, bytes) != cudaSuccess) {
    cudaGetLastError();
    return nullptr;
  }
  cache->allocs.push_back(wp);
  cache->packed[key] = wp;
  const int64_t total = (int64_t)n_tiles * n_chunks * k * (CK >> 3) * BN;
  const int blocks = (int)((total + 255) / 256);
  if (NP == 3)
    umma2_pack_kernel<3><<<blocks, 256, 0, st>>>(W, N, C_in, k, BN, CK, n_tiles, wp);
  else
    umma2_pack_kernel<2><<<blocks, 256, 0, st>>>(W, N, C_in, k, BN, CK, n_tiles, wp);
  return wp;
}

Umma2Plan umma2_plan(const ConvA& a, int N, int pieces, bool have_scratch) {
  Umma2Plan q;
  const int M = a.L_rows;
  q.NP = pieces >= 3 ? 3 : 2;
  q.BN = u2_bn(N);
  q.CK = (a.C_in % 32 == 0) ? 32 : 16;
  const int k = a.ksize;
  const int rs = U2_BM + (k - 1) * a.dil;  // staged rows per chunk
  const int rs_pad = ((rs + 7) & ~7) + 4;
  const int n_a = rs * (q.CK / 4);  // float4 units per staged chunk
  q.UPT = n_a <= 4 * U2_CONVERTERS ? 4 : U2_MAX_UNITS;
  q.SETS = q.UPT == 4 ? 3 : 2;
  const size_t a_bytes = (size_t)2 * q.NP * (q.CK >> 3) * rs_pad * 16;
  const size_t b_unit = (size_t)q.NP * q.BN * q.CK * 2;
  q.SB = (((a_bytes + 127) & ~(size_t)127) + 4 * b_unit <= 110 * 1024) ? 4 : 3;
  // ---- split over (chunk, tap) units when the tile grid cannot fill the GPU
  const int units_total = (a.C_in / q.CK) * k;
  const int m_tiles = (M + U2_BM - 1) / U2_BM;
  const long base = (long)m_tiles * ((N + q.BN - 1) / q.BN);
  int splits = 1;
  if (base < U2_SPLIT_BELOW && units_total >= 2 * U2_MIN_UNITS) {
    const long sms = std::max(1, current_device_sms());
    splits = (int)std::min<long>((sms + base - 1) / base, units_total / U2_MIN_UNITS);
    while (splits > 1 && (size_t)splits * M * N * sizeof(float) > (32u << 20)) --splits;
  }
  if (!have_scratch) splits = 1;
  q.units_per_split = (units_total + splits - 1) / splits;
  q.splits = (units_total + q.units_per_split - 1) / q.units_per_split;
  return q;
}

void umma2_conv(Umma2Cache* cache, const ConvA& a, const float* W, int N, const Epilogue& ep, int pieces, float** splitk, cudaStream_t st) {
  const int M = a.L_rows;
  if (M <= 0) {
    ++g_launches;
    return;
  }
  const Umma2Plan q = umma2_plan(a, N, pieces, splitk != nullptr);
  const int NP = q.NP, BN = q.BN, CK = q.CK;
  const int k = a.ksize;
  // ---- packed weights (once per weight matrix and tiling)
  const unsigned char* wp = umma2_packed_weights(cache, W, N, a.C_in, k, BN, CK, NP, st);
  if (wp == nullptr) {
    gemm_conv(a, W, N, ep, splitk, st);  // out of memory for the packed copy: exact fp32 path
    return;
  }
  ++g_launches;
  const int n_tiles = (N + BN - 1) / BN;
  U2Params p;
  p.a = a;
  p.ep = ep;
  p.wp = wp;
  p.M = M;
  p.N = N;
  p.CK = CK;
  p.ksize = k;
  p.dil = a.dil;
  p.rs = U2_BM + (k - 1) * a.dil;
  p.rs_pad = ((p.rs + 7) & ~7) + 4;  // planes 64 bytes out of phase: halves the bank conflicts of the 8-byte piece stores
  p.units_total = (a.C_in / CK) * k;
  const int m_tiles = (M + U2_BM - 1) / U2_BM;
  int splits = q.splits, ups = q.units_per_split;
  float* ws = nullptr;
  if (splits > 1) {
    ws = splitk_workspace(splitk, (size_t)splits * M * N * sizeof(float));
    if (!ws) {
      splits = 1;
      ups = p.units_total;
    }
  }
  p.units_per_split = ups;
  p.ws = ws;
  p.dbg = cache->dbg;
  p.SB = q.SB;
  const size_t a_bytes = (size_t)2 * NP * (CK >> 3) * p.rs_pad * 16;
  const size_t b_unit = (size_t)NP * BN * CK * 2;
  const size_t smem = std::max<size_t>(((a_bytes + 127) & ~(size_t)127) + p.SB * b_unit, (size_t)U2_BM * (BN + 8) * sizeof(float)) + 256;  // >= the epilogue's output tile
  dim3 grid(n_tiles, m_tiles, splits);
  if (NP == 3) {
    switch (BN) {
      case 128: u2_launch<128, 3>(p, q.UPT, grid, smem, st); break;
      case 64: u2_launch<64, 3>(p, q.UPT, grid, smem, st); break;
      case 32: u2_launch<32, 3>(p, q.UPT, grid, smem, st); break;
      default: u2_launch<16, 3>(p, q.UPT, grid, smem, st); break;
    }
  } else {
    switch (BN) {
      case 128: u2_launch<128, 2>(p, q.UPT, grid, smem, st); break;
      case 64: u2_launch<64, 2>(p, q.UPT, grid, smem, st); break;
      case 32: u2_launch<32, 2>(p, q.UPT, grid, smem, st); break;
      default: u2_launch<16, 2>(p, q.UPT, grid, smem, st); break;
    }
  }
  if (splits > 1) splitk_epilogue(ws, splits, M, N, a.L_rows, ep, st);
}

// ------------------------------------------------------------------------------------------------ fused vocoder generator
// One CTA per SM runs the phases of the generator (conv_pre | per stage: upsample phases, then 6 resblock depths with the three
// resblocks' convs as independent jobs | conv_post + tanh) and meets the other CTAs in a grid barrier after each phase.  Work item
// i of a phase goes to CTA i % gridDim.x; the host orders a phase's jobs by decreasing kernel size so the long items start first.
// An item is a whole 128-row x BN output tile (two warpgroups of 64 rows), so a row's sum does not depend on the schedule.
// Per channel chunk the item stages the activation rows (halo included, taps are descriptor row shifts as in umma2_kernel) and
// all taps of the chunk's packed weights; both are double-buffered so the loads of chunk c+1 fly while the MMAs of chunk c run.
namespace {

constexpr int VF_THREADS = 256;
constexpr int VF_UPT = 6;  // float4 units per thread and chunk: (128 + max halo 50) rows x 8 units <= 6 x 256

__device__ __forceinline__ void vf_cp_async16(uint32_t dst, const void* src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
}

// a job template resolved for one sequence: its rows, the packed weights of its tile width and its row bases (in floats)
struct VocSeqJob {
  int L_in, M, m_tiles, n_tiles, BN;
  const unsigned char* wp;
  int64_t in_off, out_off;
};

template <int BN, bool ADD3>
__device__ __forceinline__ void vf_item(const VocJob& J, const VocSeqJob& Q, int mt, int nt, unsigned char* a_smem, unsigned char* b_smem,
                                        float* tile, uint32_t a_stride, uint32_t b_stride) {
  constexpr int NACC = BN / 2;
  constexpr int TP = BN + 8;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = warp >> 2;
  const int m0 = mt * VOC_FUSED_BM, n0 = nt * BN;
  const int CK = J.CK, k = J.ksize, dil = J.dil, C_in = J.C_in;
  const int n_chunks = C_in / CK;
  const int rs = VOC_FUSED_BM + (k - 1) * dil;
  const uint32_t a_plane = (uint32_t)(((rs + 7) & ~7) + 4) * 16u;
  const uint32_t a_piece = (uint32_t)(CK >> 3) * a_plane;
  const uint32_t b_plane = (uint32_t)BN * 16u;
  const uint32_t b_piece = (uint32_t)BN * CK * 2u;
  const uint32_t b_unit = 2u * b_piece;
  const uint32_t b_chunk = (uint32_t)k * b_unit;
  const unsigned char* wsrc = Q.wp + (size_t)nt * n_chunks * b_chunk;

  const int upr_shift = (CK == 32) ? 3 : 2;
  const int upr = 1 << upr_shift;
  const int n_a = rs * upr;
  int64_t goff[VF_UPT];
  uint32_t soff[VF_UPT];
#pragma unroll
  for (int i = 0; i < VF_UPT; ++i) {
    const int idx = tid + i * VF_THREADS;
    const int r = idx >> upr_shift, q = idx & (upr - 1);
    const int pos = m0 + r - J.pad_left;
    const bool inb = idx < n_a && pos >= 0 && pos < Q.L_in;
    goff[i] = inb ? Q.in_off + (int64_t)pos * C_in + q * 4 : (int64_t)-1;
    soff[i] = (uint32_t)(q >> 1) * a_plane + (uint32_t)r * 16u + (uint32_t)(q & 1) * 8u;
  }
  // activations are written by earlier phases of this kernel: L2 loads (.cg), never the non-coherent read-only path
  float4 pf[ADD3 ? 3 : 1][VF_UPT];
  auto load_a = [&](int c) {
#pragma unroll
    for (int i = 0; i < VF_UPT; ++i) {
      const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
      const int64_t o = goff[i] + (int64_t)c * CK;
      pf[0][i] = goff[i] >= 0 ? __ldcg(reinterpret_cast<const float4*>(J.x0 + o)) : z;
      if (ADD3) {
        pf[ADD3 ? 1 : 0][i] = goff[i] >= 0 ? __ldcg(reinterpret_cast<const float4*>(J.x1 + o)) : z;
        pf[ADD3 ? 2 : 0][i] = goff[i] >= 0 ? __ldcg(reinterpret_cast<const float4*>(J.x2 + o)) : z;
      }
    }
  };
  auto load_b = [&](int c, int s) {
    const unsigned char* src = wsrc + (size_t)c * b_chunk;
    const uint32_t dst = smem_u32(b_smem + (size_t)s * b_stride);
    for (uint32_t i = tid; i < (b_chunk >> 4); i += VF_THREADS) vf_cp_async16(dst + 16u * i, src + 16u * i);
    asm volatile("cp.async.commit_group;" ::: "memory");
  };

  float acc[NACC];
#pragma unroll
  for (int i = 0; i < NACC; ++i) acc[i] = 0.f;
  load_b(0, 0);
  load_a(0);
  const float slope = J.slope;
  for (int c = 0; c < n_chunks; ++c) {
    const int s = c & 1;
    unsigned char* stage = a_smem + (size_t)s * a_stride;
#pragma unroll
    for (int i = 0; i < VF_UPT; ++i) {
      if (tid + i * VF_THREADS < n_a) {
        float4 v = pf[0][i];
        if (ADD3) {  // the stage's resblock outputs in the reference's order: (b0 + b1) + b2
          const float4 b1 = pf[ADD3 ? 1 : 0][i], b2 = pf[ADD3 ? 2 : 0][i];
          v = make_float4(b2.x + (b1.x + v.x), b2.y + (b1.y + v.y), b2.z + (b1.z + v.z), b2.w + (b1.w + v.w));
        }
        if (slope != 1.0f) {
          v.x = v.x > 0.f ? v.x : v.x * slope;
          v.y = v.y > 0.f ? v.y : v.y * slope;
          v.z = v.z > 0.f ? v.z : v.z * slope;
          v.w = v.w > 0.f ? v.w : v.w * slope;
        }
        u2_split_store<2>(v, stage, a_piece, soff[i]);
      }
    }
    asm volatile("cp.async.wait_group 0;" ::: "memory");
    // this thread's generic-proxy writes (staged rows, copied weights) become visible to the async proxy (wgmma)
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();
    if (c + 1 < n_chunks) {  // the stages of chunk c-1 are free: every warp waited for its MMAs before the barrier above
      load_b(c + 1, s ^ 1);
      load_a(c + 1);
    }
    const uint32_t a_base = smem_u32(stage) + (uint32_t)wg * 64u * 16u;
    const uint32_t b_base0 = smem_u32(b_smem + (size_t)s * b_stride);
    u2_fence_acc<NACC>(acc);
    asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
    for (int j = 0; j < k; ++j) {
      const uint32_t a_tap = a_base + (uint32_t)(j * dil) * 16u;
      const uint32_t b_base = b_base0 + (uint32_t)j * b_unit;
      for (int ks = 0; ks < (CK >> 4); ++ks) {
        const uint64_t a0 = u2_desc(a_tap + ks * 2 * a_plane, a_plane, 128), a1 = u2_desc(a_tap + a_piece + ks * 2 * a_plane, a_plane, 128);
        const uint64_t b0 = u2_desc(b_base + ks * 2 * b_plane, b_plane, 128), b1 = u2_desc(b_base + b_piece + ks * 2 * b_plane, b_plane, 128);
        u2_wgmma<BN>(acc, a0, b0);
        u2_wgmma<BN>(acc, a0, b1);
        u2_wgmma<BN>(acc, a1, b0);
      }
    }
    asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
    asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");
    u2_fence_acc<NACC>(acc);
  }
  // epilogue through the padded tile: whole rows per warp, bias / residual reads coalesced
  {
    const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);
    const int c0 = 2 * (lane & 3);
#pragma unroll
    for (int i = 0; i < BN / 8; ++i) {
      *reinterpret_cast<float2*>(tile + r0 * TP + 8 * i + c0) = make_float2(acc[4 * i], acc[4 * i + 1]);
      *reinterpret_cast<float2*>(tile + (r0 + 8) * TP + 8 * i + c0) = make_float2(acc[4 * i + 2], acc[4 * i + 3]);
    }
  }
  __syncthreads();
  const int rows = min(VOC_FUSED_BM, Q.M - m0);
  for (int idx = tid; idx < rows * BN; idx += VF_THREADS) {
    const int r = idx / BN, cc = idx - r * BN;
    const int n = n0 + cc;
    const int64_t o = Q.out_off + ((int64_t)(m0 + r) * J.out_row_stride + J.out_row_offset) * J.N + n;
    const float v = tile[r * TP + cc] + J.bias[n];
    const float res = J.residual != nullptr ? J.res_scale * __ldcg(J.residual + o) : 0.f;
    J.out[o] = J.alpha * v + res;
  }
  __syncthreads();  // the tile and the operand stages are reused by the next item
}

// job template T resolved for one sequence (see VocJob)
__device__ __forceinline__ VocSeqJob vf_resolve(const VocJob& T, const VocStreamGeo& G, bool bn32) {
  VocSeqJob Q;
  Q.L_in = G.N * T.in_mult;
  Q.M = Q.L_in + T.m_adj;
  Q.m_tiles = Q.M > 0 ? (Q.M + VOC_FUSED_BM - 1) / VOC_FUSED_BM : 0;
  const bool w32 = bn32 && (T.N & 31) == 0;
  Q.BN = w32 ? 32 : 16;
  Q.wp = w32 ? T.wp32 : T.wp16;
  Q.n_tiles = w32 ? T.N >> 5 : T.N >> 4;
  Q.in_off = (int64_t)G.row0 * T.in_mult * T.C_in;
  Q.out_off = (int64_t)G.row0 * T.in_mult * T.out_row_stride * T.N;
  return Q;
}

__global__ void __launch_bounds__(VF_THREADS, 1)
    vocoder_fused_kernel(const __grid_constant__ VocFusedParams p, unsigned* bar_ctr, unsigned bar_target) {
  extern __shared__ __align__(128) unsigned char smem[];
  const uint32_t a_stride = (uint32_t)p.a_stride, b_stride = (uint32_t)p.b_stride;
  unsigned char* a_smem = smem + ((128u - (smem_u32(smem) & 127u)) & 127u);
  unsigned char* b_smem = a_smem + 2 * (size_t)a_stride;
  float* tile = reinterpret_cast<float*>(b_smem + 2 * (size_t)b_stride);
  const VocJob* jobs = p.jobs;
  const VocPost& post = p.post;
  // Items are numbered sequence by sequence, job by job, and this CTA's i only grows: (s, jb) is a cursor that moves forward,
  // with the items of (s, jb) from `base` on, so a job is resolved once per CTA and sequence, not once per item.  The cursor of a
  // phase is set up before the grid barrier that precedes it, so its parameter loads overlap the wait.
  int s = 0, jb = 0, base = 0;
  VocSeqJob Q = vf_resolve(jobs[p.phases[0].first_job], p.streams[0], p.streams[0].bn32 & 1ull);
  for (int ph = 0; ph < p.n_phases; ++ph) {
    const VocPhase P = p.phases[ph];
    s = 0;
    jb = P.first_job;
    base = 0;
    for (int i = blockIdx.x; i < P.n_items; i += gridDim.x) {
      if (s + 1 < p.n_streams && i >= p.item0[ph][s + 1]) {
        do ++s; while (s + 1 < p.n_streams && i >= p.item0[ph][s + 1]);
        jb = P.first_job;
        base = p.item0[ph][s];
        Q = vf_resolve(jobs[jb], p.streams[s], (p.streams[s].bn32 >> ph) & 1ull);
      }
      while (i - base >= Q.m_tiles * Q.n_tiles) {
        base += Q.m_tiles * Q.n_tiles;
        Q = vf_resolve(jobs[++jb], p.streams[s], (p.streams[s].bn32 >> ph) & 1ull);
      }
      const VocJob& J = jobs[jb];
      const int rest = i - base;
      const int nt = rest % Q.n_tiles, mt = rest / Q.n_tiles;  // neighbouring CTAs share activation rows
      const bool add3 = J.x1 != nullptr;
      if (Q.BN == 32) {
        if (add3) vf_item<32, true>(J, Q, mt, nt, a_smem, b_smem, tile, a_stride, b_stride);
        else vf_item<32, false>(J, Q, mt, nt, a_smem, b_smem, tile, a_stride, b_stride);
      } else {
        if (add3) vf_item<16, true>(J, Q, mt, nt, a_smem, b_smem, tile, a_stride, b_stride);
        else vf_item<16, false>(J, Q, mt, nt, a_smem, b_smem, tile, a_stride, b_stride);
      }
    }
    if (ph + 1 < p.n_phases) Q = vf_resolve(jobs[p.phases[ph + 1].first_job], p.streams[0], (p.streams[0].bn32 >> (ph + 1)) & 1ull);
    grid_barrier(bar_ctr, bar_target);
  }
  // conv_post + tanh on each sequence's new samples only, straight into the caller's buffer (same arithmetic order as
  // conv_post_tanh_kernel); sample o of the output belongs to the sequence whose [out0, out0 + (N * hop - t0)) holds it
  const int half = (post.k - 1) >> 1;
  s = 0;
  for (int o = blockIdx.x * VF_THREADS + threadIdx.x; o < post.total; o += gridDim.x * VF_THREADS) {
    while (s + 1 < p.n_streams && o >= p.streams[s + 1].out0) ++s;
    const VocStreamGeo& G = p.streams[s];
    const int L = G.N * post.hop, t = o - G.out0 + G.t0;
    const float* x0 = post.x0 + (int64_t)G.row0 * post.hop * post.C;
    const float* x1 = post.x1 + (int64_t)G.row0 * post.hop * post.C;
    const float* x2 = post.x2 + (int64_t)G.row0 * post.hop * post.C;
    float acc = post.bias;
    for (int j = 0; j < post.k; ++j) {
      const int p = t - half + j;
      if (p < 0 || p >= L) continue;
      const int64_t row = (int64_t)p * post.C;
      for (int c = 0; c < post.C; ++c) {
        float v = __ldcg(x2 + row + c) + (__ldcg(x1 + row + c) + __ldcg(x0 + row + c));
        v = v > 0.f ? v : v * post.slope;
        acc = fmaf(post.w[j * post.C + c], v, acc);
      }
    }
    post.out[G.dst + (o - G.out0)] = tanhf(acc);
  }
}

}  // namespace

size_t vocoder_fused_smem(int a_stride, int b_stride) {
  return 2 * (size_t)a_stride + 2 * (size_t)b_stride + (size_t)VOC_FUSED_BM * (32 + 8) * sizeof(float) + 128;
}

int vocoder_fused_grid() {
  // the largest shared-memory footprint the engine asks for (stage-0 resblock k = 11, dil 5, 32 channels per chunk, BN = 32)
  static const size_t smem_max = 200 * 1024;
  if (first_time_on_device((const void*)vocoder_fused_kernel))
    cudaFuncSetAttribute(vocoder_fused_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_max);
  int occ = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, vocoder_fused_kernel, VF_THREADS, smem_max) != cudaSuccess) {
    cudaGetLastError();
    return 0;
  }
  return occ >= 1 ? current_device_sms() : 0;
}

int vocoder_fused(const VocFusedParams& p, unsigned* bar_ctr, unsigned* bar_target_host, cudaStream_t st) {
  const int grid = vocoder_fused_grid();
  const size_t smem = vocoder_fused_smem(p.a_stride, p.b_stride);
  if (grid <= 0 || smem > 200 * 1024) return -1;
  unsigned bar_target = *bar_target_host;
  void* args[] = {(void*)&p, (void*)&bar_ctr, (void*)&bar_target};
  if (cudaLaunchCooperativeKernel((void*)vocoder_fused_kernel, dim3(grid), dim3(VF_THREADS), args, smem, st) != cudaSuccess) {
    cudaGetLastError();
    return -2;
  }
  ++g_launches;
  *bar_target_host += (unsigned)grid * (unsigned)p.n_phases;
  return 0;
}

}  // namespace ss
