// Kaldi-compatible log-mel filterbank + global CMVN, one CTA per 25 ms frame.
// Arithmetic follows torchaudio.compliance.kaldi.fbank with the arguments the reference passes
// (fairseq/fairseq/data/audio/audio_utils.py:241-247; SURVEY.md Appendix B): x*2^15, per-frame DC removal,
// pre-emphasis 0.97 (replicate pad), Povey window, zero-pad 400 -> 512, |rfft|^2, 80 mel bins, log(max(., eps)),
// then (x - mean) / std (agent/speech_to_speech.streamspeech.agent.py:89-98).
// The 400 samples of a frame are staged in shared memory once (1.6 KB in, 320 B out per frame): HBM-bound.
#include "common.cuh"
#include "kernels.h"

namespace ss {
namespace {

constexpr int FRAME = 400, SHIFT = 160, NFFT = 512, NBIN = 257, NMEL = 80;

__global__ void __launch_bounds__(256) fbank_kernel(const float* __restrict__ samples, int64_t n_samples, int f0,
                                                    const float* __restrict__ mel_bank, const float* __restrict__ window,
                                                    const float* __restrict__ cmvn_mean, const float* __restrict__ cmvn_std,
                                                    float* __restrict__ out) {
  pdl_trigger();
  pdl_wait();
  __shared__ float re[NFFT], im[NFFT];
  __shared__ float twc[NFFT / 2], tws[NFFT / 2];
  __shared__ float frame[FRAME];
  __shared__ float red[32];
  const int tid = threadIdx.x;
  const int f = f0 + blockIdx.x;
  const int64_t base = (int64_t)f * SHIFT;
  float s = 0.f;
  for (int j = tid; j < FRAME; j += 256) {
    float v = (base + j < n_samples) ? samples[base + j] * 32768.0f : 0.f;
    frame[j] = v;
    s += v;
  }
  {
    float sn, cs;
    sincospif(-(float)tid / 256.0f, &sn, &cs);  // exp(-2*pi*i*tid/512)
    twc[tid] = cs;
    tws[tid] = sn;
  }
  float mean = block_sum(s, red) / (float)FRAME;
  // bit-reversed load of the windowed, pre-emphasised frame (zero padded to 512)
  for (int j = tid; j < NFFT; j += 256) {
    float v = 0.f;
    if (j < FRAME) {
      float x0 = frame[j] - mean;
      float xm = frame[j > 0 ? j - 1 : 0] - mean;
      v = (x0 - 0.97f * xm) * window[j];
    }
    int r = __brev((unsigned)j) >> (32 - 9);
    re[r] = v;
    im[r] = 0.f;
  }
  __syncthreads();
#pragma unroll
  for (int stage = 0; stage < 9; ++stage) {
    int half = 1 << stage;
    int grp = tid >> stage, pos = tid & (half - 1);
    int i = (grp << (stage + 1)) + pos, j = i + half;
    int tw = pos << (8 - stage);
    float wr = twc[tw], wi = tws[tw];
    float xr = re[j], xi = im[j];
    float tr = wr * xr - wi * xi, ti = wr * xi + wi * xr;
    float ur = re[i], ui = im[i];
    re[i] = ur + tr;
    im[i] = ui + ti;
    re[j] = ur - tr;
    im[j] = ui - ti;
    __syncthreads();
  }
  // power spectrum: spectrum.abs().pow(2)
  for (int k = tid; k < NBIN; k += 256) {
    float a = sqrtf(re[k] * re[k] + im[k] * im[k]);
    frame[k] = a * a;  // reuse (257 <= 400)
  }
  __syncthreads();
  if (tid < NMEL) {
    const float* wrow = mel_bank + tid * NBIN;
    float acc = 0.f;
    for (int k = 0; k < NBIN; ++k) acc = fmaf(frame[k], wrow[k], acc);
    float v = logf(fmaxf(acc, 1.1920928955078125e-07f));
    if (cmvn_mean) v = (v - cmvn_mean[tid]) / cmvn_std[tid];
    out[(int64_t)blockIdx.x * NMEL + tid] = v;
  }
}

// Same arithmetic, TMA staging: the 400 samples of the frame (1600 contiguous bytes, 640-byte aligned offsets) arrive in shared
// memory by ONE bulk-async copy (cp.async.bulk = the TMA engine's 1-D path, UBLKCP in SASS) completing on an mbarrier while the
// twiddle table is being computed; the mel bank is read TRANSPOSED ([257][80]) so that the 80 mel threads read coalesced rows
// (the [80][257] layout made every lane walk its own 1 KB row: 80 uncoalesced streams per frame).
__device__ __forceinline__ uint32_t fb_smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__global__ void __launch_bounds__(256) fbank_tma_kernel(const float* __restrict__ samples, int f0, const float* __restrict__ melT,
                                                        const float* __restrict__ window, const float* __restrict__ cmvn_mean,
                                                        const float* __restrict__ cmvn_std, float* __restrict__ out) {
  pdl_trigger();
  pdl_wait();
  __shared__ float re[NFFT], im[NFFT];
  __shared__ float twc[NFFT / 2], tws[NFFT / 2];
  __shared__ __align__(128) float frame[FRAME];
  __shared__ float red[32];
  __shared__ __align__(8) unsigned long long mbar;
  const int tid = threadIdx.x;
  const int f = f0 + blockIdx.x;
  const float* src = samples + (int64_t)f * SHIFT;
  if (tid == 0) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(fb_smem_u32(&mbar)));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (tid == 0) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(fb_smem_u32(&mbar)), "r"(FRAME * 4) : "memory");
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(fb_smem_u32(frame)), "l"(src),
                 "r"(FRAME * 4), "r"(fb_smem_u32(&mbar))
                 : "memory");
  }
  {
    float sn, cs;
    sincospif(-(float)tid / 256.0f, &sn, &cs);  // exp(-2*pi*i*tid/512), overlaps the copy
    twc[tid] = cs;
    tws[tid] = sn;
  }
  {
    uint32_t done = 0;
    while (!done) {
      asm volatile(
          "{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], 0;\n\tselp.u32 %0, 1, 0, p;\n\t}"
          : "=r"(done)
          : "r"(fb_smem_u32(&mbar))
          : "memory");
    }
  }
  float s = 0.f;
  for (int j = tid; j < FRAME; j += 256) s += frame[j] * 32768.0f;
  const float mean = block_sum(s, red) / (float)FRAME;
  for (int j = tid; j < NFFT; j += 256) {
    float v = 0.f;
    if (j < FRAME) {
      const float x0 = frame[j] * 32768.0f - mean;
      const float xm = frame[j > 0 ? j - 1 : 0] * 32768.0f - mean;
      v = (x0 - 0.97f * xm) * window[j];
    }
    const int r = __brev((unsigned)j) >> (32 - 9);
    re[r] = v;
    im[r] = 0.f;
  }
  __syncthreads();
#pragma unroll
  for (int stage = 0; stage < 9; ++stage) {
    const int half = 1 << stage;
    const int grp = tid >> stage, pos = tid & (half - 1);
    const int i = (grp << (stage + 1)) + pos, j = i + half;
    const int tw = pos << (8 - stage);
    const float wr = twc[tw], wi = tws[tw];
    const float xr = re[j], xi = im[j];
    const float tr = wr * xr - wi * xi, ti = wr * xi + wi * xr;
    const float ur = re[i], ui = im[i];
    re[i] = ur + tr;
    im[i] = ui + ti;
    re[j] = ur - tr;
    im[j] = ui - ti;
    __syncthreads();
  }
  for (int k = tid; k < NBIN; k += 256) {
    const float a = sqrtf(re[k] * re[k] + im[k] * im[k]);
    frame[k] = a * a;
  }
  __syncthreads();
  if (tid < NMEL) {
    float acc = 0.f;
    for (int k = 0; k < NBIN; ++k) acc = fmaf(frame[k], melT[k * NMEL + tid], acc);
    float v = logf(fmaxf(acc, 1.1920928955078125e-07f));
    if (cmvn_mean) v = (v - cmvn_mean[tid]) / cmvn_std[tid];
    out[(int64_t)blockIdx.x * NMEL + tid] = v;
  }
}

}  // namespace

// TMA-staged variant (melT = mel bank transposed to [257][80]); requires 16-byte aligned `samples` and every frame inside the buffer
void fbank_cmvn_tma(const float* samples, int f0, int nf, const float* melT, const float* window, const float* cmvn_mean, const float* cmvn_std,
                    float* out, cudaStream_t st) {
  ++g_launches;
  if (nf <= 0) return;
  launch_pdl(fbank_tma_kernel, dim3(nf), dim3(256), 0, st, samples, f0, melT, window, cmvn_mean, cmvn_std, out);
}

void fbank_cmvn(const float* samples, int64_t n_samples, int f0, int nf, const float* mel_bank, const float* window,
                const float* cmvn_mean, const float* /*unused*/, const float* cmvn_std, float* out, cudaStream_t st) {
  ++g_launches;
  if (nf <= 0) return;
  launch_pdl(fbank_kernel, dim3(nf), dim3(256), 0, st, samples, n_samples, f0, mel_bank, window, cmvn_mean, cmvn_std, out);
}

}  // namespace ss
