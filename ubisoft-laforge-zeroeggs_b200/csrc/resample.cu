// Rate conversion of raw WAV PCM to 16 kHz on the device: what the reference's read_wavfile(..., desired_fs=16000) gets from
// SoX (audio_files.py:52-78, 115-146: `rate -h 16000`, `channels 1`, 32-bit output).  One launch decodes the interleaved PCM
// (int16 x/2^15, int32 x/2^31, uint8 (u-128)/128, float32 clipped to [-1, 1]), averages the channels, runs the polyphase FIR of
// the prototype zeggs_b200.audio.design_resampler builds and clamps the result to [-1, 1].
//
// Output j sits at time j / fs_out.  With t = j M + delay (delay = the prototype's centre tap), it is
//   y[j] = sum_q taps[p][q] * x[t / L - q],   p = t mod L,   taps[p][q] = h[p + q L],   x = 0 outside [0, n_in).
// Outputs j, j + L, j + 2L, ... share the phase p, and their newest inputs lie M apart.  A warp task is the 32 outputs
// j0 + lane * L of one phase: the tap loads are warp-uniform (one broadcast float4 per 4 taps), and the lanes read shared
// memory at stride M, free of bank conflicts for odd M (3 at 48 kHz, 441 at 44.1 / 22.05 / 11.025 kHz).  Tasks are numbered
// tau = row * L + column, row r holding outputs [32 L r, 32 L (r + 1)).  A CTA owns `nt` consecutive tasks, where nt is a
// multiple of L (L <= 32: whole rows, i.e. 32 nt consecutive outputs) or a divisor of L (L > 32: part of one row); it stages
// the decoded, mixed input span those outputs need in shared memory once.  Four partial sums per output, fp32.
#include "common.cuh"
#include "../../include/zeggs_b200.h"

namespace zeggs {
void count_launch();

namespace {

constexpr int RS_THREADS = 256;
constexpr int RS_WARPS = RS_THREADS / 32;

template <int DT> __device__ __forceinline__ float pcm_sample(const void* p, long long i);
template <> __device__ __forceinline__ float pcm_sample<ZEGGS_PCM_I16>(const void* p, long long i) {
  return (float)__ldg((const short*)p + i) * (1.0f / 32768.0f);
}
template <> __device__ __forceinline__ float pcm_sample<ZEGGS_PCM_I32>(const void* p, long long i) {
  return (float)__ldg((const int*)p + i) * (1.0f / 2147483648.0f);
}
template <> __device__ __forceinline__ float pcm_sample<ZEGGS_PCM_U8>(const void* p, long long i) {
  return ((float)__ldg((const unsigned char*)p + i) - 128.0f) * (1.0f / 128.0f);
}
template <> __device__ __forceinline__ float pcm_sample<ZEGGS_PCM_F32>(const void* p, long long i) {
  return fminf(fmaxf(__ldg((const float*)p + i), -1.0f), 1.0f);      // SoX clips float input when it converts it
}

// first output of task tau (lane 0)
__host__ __device__ __forceinline__ long long task_j0(long long tau, int L) { return (tau / L) * 32LL * L + tau % L; }

template <int DT>
__global__ void __launch_bounds__(RS_THREADS) resample_kernel(const void* __restrict__ pcm, long long n_in, int C, float inv_c,
                                                              const float* __restrict__ taps, int L, int M, int K4, long long delay,
                                                              long long n_out, int nt, float* __restrict__ out) {
  extern __shared__ float xs[];
  const long long tau0 = (long long)blockIdx.x * nt;
  const long long jmin = task_j0(tau0, L);
  const long long jmax = task_j0(tau0 + nt - 1, L) + 31LL * L;
  // xs[e] = x[lo + e]; the K4 - K zero taps at the end of each phase read up to 3 samples below the oldest real tap
  const long long lo = (jmin * M + delay) / L - K4 + 1;
  const int span = (int)((jmax * M + delay) / L - lo + 1);
  for (int e = threadIdx.x; e < span; e += RS_THREADS) {
    const long long m = lo + e;
    float v = 0.0f;
    if (m >= 0 && m < n_in) {
      const long long base = m * C;
      float s = pcm_sample<DT>(pcm, base);
      for (int c = 1; c < C; ++c) s += pcm_sample<DT>(pcm, base + c);
      v = s * inv_c;
    }
    xs[e] = v;
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int k = warp; k < nt; k += RS_WARPS) {
    const long long j = task_j0(tau0 + k, L) + (long long)lane * L;
    const long long t = j * M + delay;
    const float4* h = reinterpret_cast<const float4*>(taps + (size_t)(t % L) * K4);
    const float* x = xs + (t / L - lo);
    float a0 = 0.0f, a1 = 0.0f, a2 = 0.0f, a3 = 0.0f;
#pragma unroll 4
    for (int q = 0; q < K4; q += 4) {
      const float4 w = __ldg(h + (q >> 2));
      a0 = fmaf(w.x, x[-q], a0);
      a1 = fmaf(w.y, x[-q - 1], a1);
      a2 = fmaf(w.z, x[-q - 2], a2);
      a3 = fmaf(w.w, x[-q - 3], a3);
    }
    if (j < n_out) out[j] = fminf(fmaxf((a0 + a1) + (a2 + a3), -1.0f), 1.0f);
  }
}

template <int DT>
int launch(const zeggs_resample_args& a, int nt, long long n_blocks, size_t smem, cudaStream_t s) {
  auto kern = resample_kernel<DT>;
  if (smem > 48 * 1024) ZCHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  kern<<<(unsigned)n_blocks, RS_THREADS, smem, s>>>(a.pcm, a.n_in, a.channels, 1.0f / (float)a.channels, a.taps, a.L, a.M, a.K4,
                                                    a.delay, a.n_out, nt, a.out);
  count_launch();
  ZCHECK_LAUNCH();
  return ZEGGS_OK;
}

}  // namespace

extern "C" int zeggs_resample(const zeggs_resample_args* ap, void* stream_) {
  ZCHECK_ARG(ap, "resample: null args");
  const zeggs_resample_args& a = *ap;
  ZCHECK_ARG(a.n_in >= 0 && a.n_out >= 0 && a.channels >= 1, "resample: bad shape (n_in %lld, n_out %lld, channels %d)", a.n_in, a.n_out,
             a.channels);
  ZCHECK_ARG(a.L >= 1 && a.L <= 1024 && a.M >= 1 && a.K4 >= 4 && a.K4 % 4 == 0 && a.delay >= 0, "resample: bad filter geometry");
  ZCHECK_ARG(a.dtype >= ZEGGS_PCM_I16 && a.dtype <= ZEGGS_PCM_F32, "resample: unknown PCM dtype %d", a.dtype);
  ZCHECK_ARG(a.taps && (a.out || a.n_out == 0) && (a.pcm || a.n_in == 0), "resample: null pointer");
  ZCHECK_ARG(((uintptr_t)a.taps & 15) == 0, "resample: taps must be 16-byte aligned");
  if (a.n_out == 0) return ZEGGS_OK;
  cudaStream_t s = (cudaStream_t)stream_;
  int nt = 1;
  if (a.L <= 32) nt = (32 / a.L) * a.L;
  else for (int d = 32; d >= 1; --d) if (a.L % d == 0) { nt = d; break; }
  const long long rows = (a.n_out + 32LL * a.L - 1) / (32LL * a.L);
  const long long n_blocks = (rows * a.L + nt - 1) / nt;
  // every CTA's output range spans task_j0(nt - 1) + 31 L outputs (tau0 is aligned to nt, so no CTA crosses a row unevenly)
  const long long diff = task_j0(nt - 1, a.L) + 31LL * a.L;
  const long long span = diff * a.M / a.L + 2 + a.K4;
  int dev = 0, smem_max = 0;
  ZCHECK_CUDA(cudaGetDevice(&dev));
  ZCHECK_CUDA(cudaDeviceGetAttribute(&smem_max, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
  const size_t smem = (size_t)span * sizeof(float);
  ZCHECK_SUPPORTED(smem <= (size_t)smem_max, "resample: L/M = %d/%d needs %zu bytes of shared memory per CTA (at most %d)", a.L, a.M, smem,
                   smem_max);
  ZCHECK_SUPPORTED(n_blocks < (1LL << 31), "resample: %lld output samples is too many", a.n_out);
  switch (a.dtype) {
    case ZEGGS_PCM_I16: return launch<ZEGGS_PCM_I16>(a, nt, n_blocks, smem, s);
    case ZEGGS_PCM_I32: return launch<ZEGGS_PCM_I32>(a, nt, n_blocks, smem, s);
    case ZEGGS_PCM_U8: return launch<ZEGGS_PCM_U8>(a, nt, n_blocks, smem, s);
    default: return launch<ZEGGS_PCM_F32>(a, nt, n_blocks, smem, s);
  }
}

}  // namespace zeggs
