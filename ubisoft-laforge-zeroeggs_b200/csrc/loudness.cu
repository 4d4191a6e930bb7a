// BS.1770 integrated loudness + gain to a target LUFS, per clip, on the device (SURVEY.md 8f row 4).
// Replaces the pyloudnorm calls of ZEGGS/data_pipeline.py:34-39 (Meter.integrated_loudness + normalize.loudness): K-weighting
// (high shelf then high pass biquads, float64 recursion, rounded to float32 after each stage like the package's in-place
// float32 channel buffer), 0.4 s gating blocks with 75 % overlap, absolute (-70 LUFS) and relative (-10 LU) gates.
//
// Parallel form of the recursive filters: the gating-block boundaries cut every clip into SEGMENTS (1600 samples at 16 kHz);
// one thread owns one (clip, segment), starts `warm` samples earlier from a zero state (K-weighting's slowest pole pair, the
// 38 Hz double pole, decays as n r^n with r = 0.985: 4800 samples reduce the start-up transient below 1e-28) and accumulates
// the energy of its segment; a second kernel, one CTA per clip, applies the two gates.  Each gating pass recomputes every block
// energy z_j from the handful of segment energies the block covers (4 at 16 kHz), in a fixed order, so the meter keeps no
// per-block array and takes clips of any length; the result is deterministic.  Samples may be float32
// or int16 PCM (x / 32768, audio_files.py:211-236).  The gain is applied by the mel kernel at load (mel.cu), not here:
// the waveform is never rewritten in HBM.
#include "library.cuh"

namespace zeggs {

struct Biquads { double b0[2], b1[2], b2[2], a1[2], a2[2]; };

template <typename TIn>
__device__ __forceinline__ float load_sample(const TIn* p, size_t i);
template <> __device__ __forceinline__ float load_sample<float>(const float* p, size_t i) { return __ldg(p + i); }
template <> __device__ __forceinline__ float load_sample<short>(const short* p, size_t i) { return (float)__ldg(p + i) * (1.0f / 32768.0f); }

template <typename TIn>
__global__ void __launch_bounds__(128) kweight_segment_energy_kernel(const TIn* __restrict__ wav, int n_clips, int n_samples, Biquads q,
                                                                     const int* __restrict__ seg_bounds, int n_seg, int warm,
                                                                     double* __restrict__ seg_energy) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n_clips * n_seg) return;
  // consecutive threads take consecutive CLIPS of the same segment: every thread of a warp runs the same trip counts
  const int seg = idx / n_clips, clip = idx % n_clips;
  const int s0 = seg_bounds[seg], s1 = seg_bounds[seg + 1];
  int start = s0 - warm;
  if (start < 0) start = 0;
  const TIn* x = wav + (size_t)clip * n_samples;
  double z1a = 0.0, z2a = 0.0, z1b = 0.0, z2b = 0.0, e = 0.0;
  for (int n = start; n < s1; ++n) {
    const double xv = (double)load_sample<TIn>(x, (size_t)n);
    // direct form II transposed (scipy.signal.lfilter), stage 0 = high shelf, stage 1 = high pass
    const double ya = fma(q.b0[0], xv, z1a);
    z1a = fma(-q.a1[0], ya, fma(q.b1[0], xv, z2a));
    z2a = fma(-q.a2[0], ya, q.b2[0] * xv);
    const double xb = (double)(float)ya;                      // the package stores each stage back into the float32 buffer
    const double yb = fma(q.b0[1], xb, z1b);
    z1b = fma(-q.a1[1], yb, fma(q.b1[1], xb, z2b));
    z2b = fma(-q.a2[1], yb, q.b2[1] * xb);
    if (n >= s0) { const double yf = (double)(float)yb; e = fma(yf, yf, e); }
  }
  seg_energy[(size_t)clip * n_seg + seg] = e;
}

// one CTA per clip: block energies from the segment sums, the two gates, integrated loudness, gain
__global__ void __launch_bounds__(128) loudness_gate_kernel(const double* __restrict__ seg_energy, int n_seg, const int* __restrict__ blk_lo,
                                                            const int* __restrict__ blk_hi, int n_blocks, double inv_block_len, double target,
                                                            float* __restrict__ gain_out, float* __restrict__ lufs_out) {
  __shared__ double red[128];
  __shared__ int redn[128];
  const int clip = blockIdx.x, tid = threadIdx.x;
  const double* se = seg_energy + (size_t)clip * n_seg;
  auto block_energy = [&](int j) -> double {                  // z_j = (sum of its segments' energies) / (0.4 s * rate)
    double s = 0.0;
    for (int k = __ldg(blk_lo + j); k < __ldg(blk_hi + j); ++k) s += se[k];
    return s * inv_block_len;
  };
  auto gated_mean = [&](double thr, bool strict) -> double {     // mean of z_j over blocks with l_j (>= | >) thr; NaN if none
    double s = 0.0; int c = 0;
    for (int j = tid; j < n_blocks; j += blockDim.x) {
      const double z = block_energy(j);
      const double l = -0.691 + 10.0 * log10(z);
      const bool in = strict ? (l > thr && l > -70.0) : (l >= thr);
      if (in) { s += z; ++c; }
    }
    red[tid] = s; redn[tid] = c;
    __syncthreads();
    for (int o = 64; o > 0; o >>= 1) { if (tid < o) { red[tid] += red[tid + o]; redn[tid] += redn[tid + o]; } __syncthreads(); }
    const double m = redn[0] > 0 ? red[0] / (double)redn[0] : nan("");
    __syncthreads();
    return m;
  };
  const double za = gated_mean(-70.0, false);                               // absolute gate
  const double gamma_r = -0.691 + 10.0 * log10(za) - 10.0;                  // NaN when nothing passed: every comparison below is false
  double zr = gated_mean(gamma_r, true);
  if (isnan(zr)) zr = 0.0;                                                   // np.nan_to_num
  const double lufs = -0.691 + 10.0 * log10(zr);
  if (tid == 0) {
    gain_out[clip] = (float)pow(10.0, (target - lufs) / 20.0);
    if (lufs_out) lufs_out[clip] = (float)lufs;
  }
}

extern "C" size_t zeggs_loudness_workspace_bytes(int n_clips, int n_seg) {
  return (n_clips < 1 || n_seg < 1) ? 0 : (size_t)n_clips * n_seg * sizeof(double);
}

extern "C" int zeggs_loudness_gain(const zeggs_loudness_args* ap, void* stream_) {
  ZCHECK_ARG(ap, "loudness: null args");
  const zeggs_loudness_args& a = *ap;
  cudaStream_t s = (cudaStream_t)stream_;
  ZCHECK_ARG(a.n_clips >= 0 && a.n_samples >= 1 && a.n_seg >= 1 && a.n_blocks >= 1, "loudness: bad shape");
  ZCHECK_ARG((long long)a.n_clips * a.n_seg + 127 <= INT_MAX, "loudness: too many (clip, segment) pairs for one grid");   // int thread index
  ZCHECK_ARG((a.wav != nullptr) != (a.wav_i16 != nullptr), "loudness: exactly one of wav / wav_i16");
  ZCHECK_ARG(a.seg_bounds && a.blk_seg_lo && a.blk_seg_hi && a.gain_out && a.workspace, "loudness: null table/output pointer");
  ZCHECK_ARG(a.workspace_bytes >= zeggs_loudness_workspace_bytes(a.n_clips, a.n_seg), "loudness: workspace too small");
  if (a.n_clips == 0) return ZEGGS_OK;
  Biquads q;
  for (int i = 0; i < 2; ++i) { q.b0[i] = a.coef[5 * i]; q.b1[i] = a.coef[5 * i + 1]; q.b2[i] = a.coef[5 * i + 2]; q.a1[i] = a.coef[5 * i + 3]; q.a2[i] = a.coef[5 * i + 4]; }
  double* se = (double*)a.workspace;
  const int total = a.n_clips * a.n_seg;
  if (a.wav) kweight_segment_energy_kernel<float><<<ceil_div(total, 128), 128, 0, s>>>(a.wav, a.n_clips, a.n_samples, q, a.seg_bounds, a.n_seg, a.warm, se);
  else kweight_segment_energy_kernel<short><<<ceil_div(total, 128), 128, 0, s>>>(a.wav_i16, a.n_clips, a.n_samples, q, a.seg_bounds, a.n_seg, a.warm, se);
  count_launch();
  loudness_gate_kernel<<<a.n_clips, 128, 0, s>>>(se, a.n_seg, a.blk_seg_lo, a.blk_seg_hi, a.n_blocks, a.inv_block_len, a.target_lufs,
                                                 a.gain_out, a.lufs_out);
  count_launch();
  ZCHECK_LAUNCH();
  return ZEGGS_OK;
}

}  // namespace zeggs
