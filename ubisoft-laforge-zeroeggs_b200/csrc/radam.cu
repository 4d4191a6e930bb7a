// Fused multi-tensor RAdam (ZEGGS/optimizers.py:31-99) over one flat fp32 parameter buffer:
// weight_decay = 0, degenerated_to_sgd = True (the configuration train.py:160 uses).  The step count and the
// hyper-parameters live in device memory, so a captured CUDA graph can replay the step.  The hyper-parameters are the host's
// doubles: the reference forms 1 - beta and the rectification terms in Python floats and torch rounds each scalar to fp32 once,
// so forming 1.0f - (float)beta2 instead would scale every v term by 1 - 1.3e-5 at beta2 = 0.999.  The rectification terms
// depend only on the step count; one thread evaluates them in double and the main kernel reads them back.  `grad_scale` folds
// the 1/world_size of the data-parallel all-reduce into the same pass.
#include <math.h>
#include "library.cuh"

namespace zeggs {

__global__ void radam_prep_kernel(double* __restrict__ hyper, int* __restrict__ step_count) {
  const int step = *step_count + 1;
  *step_count = step;
  const double lr = hyper[0], beta1 = hyper[1], beta2 = hyper[2];
  const double b2t = pow(beta2, (double)step);
  const double n_max = 2.0 / (1.0 - beta2) - 1.0;
  const double n_sma = n_max - 2.0 * step * b2t / (1.0 - b2t);            // optimizers.py:66-68
  double step_size, adaptive;
  if (n_sma >= 5.0) {
    step_size = sqrt((1.0 - b2t) * (n_sma - 4.0) / (n_max - 4.0) * (n_sma - 2.0) / n_sma * n_max / (n_max - 2.0)) /
                (1.0 - pow(beta1, (double)step));                         // :72-76
    adaptive = 1.0;
  } else {
    step_size = 1.0 / (1.0 - pow(beta1, (double)step));                   // :77-78
    adaptive = 0.0;
  }
  hyper[5] = step_size * lr;
  hyper[6] = adaptive;
}
__global__ void radam_dev_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m, float* __restrict__ v,
                                 size_t n, const double* __restrict__ hyper) {
  // each scalar rounded to fp32 once, as torch rounds the Python scalars of optimizers.py:58-59, :89, :94
  const float beta1 = (float)hyper[1], beta2 = (float)hyper[2], one_m_beta1 = (float)(1.0 - hyper[1]),
              one_m_beta2 = (float)(1.0 - hyper[2]), eps = (float)hyper[3], grad_scale = (float)hyper[4], step_lr = (float)hyper[5];
  const bool adaptive = hyper[6] != 0.0;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const float gi = g[i] * grad_scale;
    const float vi = v[i] * beta2 + one_m_beta2 * gi * gi;        // optimizers.py:58
    const float mi = m[i] * beta1 + one_m_beta1 * gi;             // :59
    v[i] = vi; m[i] = mi;
    if (adaptive) p[i] = p[i] - step_lr * mi / (sqrtf(vi) + eps); // :88-89
    else p[i] = p[i] - step_lr * mi;                              // :94
  }
}
extern "C" int zeggs_radam_step_dev(float* p, const float* g, float* m, float* v, size_t n, double* hyper, int* step_count, void* stream) {
  ZCHECK_ARG(p && g && m && v && hyper && step_count, "radam (device scalars): bad arguments");
  if (n == 0) return ZEGGS_OK;
  ScopedTimer tm("optimizer", (cudaStream_t)stream);
  radam_prep_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(hyper, step_count);
  count_launch();
  const size_t blocks = (n + 1023) / 1024;
  radam_dev_kernel<<<(unsigned)(blocks > 1184 ? 1184 : blocks), 256, 0, (cudaStream_t)stream>>>(p, g, m, v, n, hyper);
  count_launch();
  ZCHECK_LAUNCH();
  return ZEGGS_OK;
}

}  // namespace zeggs

// ---------------------------------------------------------------------------------------------- dropout masks
// mask[i] = (u_i >= p) / (1 - p), u_i ~ U[0,1) from a counter-based generator (the Bernoulli draw + rescale of
// nn.Dropout / F.dropout, modules.py:263-270, :383-388, :551, :606) in ONE pass instead of rand / compare / cast / scale.
// splitmix64 of (seed, index): independent of the launch shape, reproducible for a given seed.
namespace zeggs {
__device__ __forceinline__ uint32_t mix_u32(uint64_t seed, uint64_t i) {
  uint64_t z = seed + 0x9E3779B97F4A7C15ULL * (i + 1);
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ULL;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBULL;
  z = z ^ (z >> 31);
  return (uint32_t)(z >> 32);
}
__global__ void dropout_mask_kernel(float* __restrict__ out, size_t n, float p, float keep_scale, uint64_t seed) {
  const uint32_t thr = (uint32_t)fminf(4294967040.0f, p * 4294967296.0f);     // P(u32 < thr) = p
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    out[i] = mix_u32(seed, i) >= thr ? keep_scale : 0.0f;
}
__global__ void dropout_mask_dev_kernel(float* __restrict__ out, size_t n, float p, float keep_scale,
                                        const unsigned long long* __restrict__ seed_dev, unsigned long long salt) {
  // effective seed: splitmix-style hash of (device seed, salt)
  uint64_t z = *seed_dev * 0xD1342543DE82EF95ULL + (salt + 1) * 0x9E3779B97F4A7C15ULL;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ULL;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBULL;
  const uint64_t seed = z ^ (z >> 31);
  const uint32_t thr = (uint32_t)fminf(4294967040.0f, p * 4294967296.0f);
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    out[i] = mix_u32(seed, i) >= thr ? keep_scale : 0.0f;
}
extern "C" int zeggs_dropout_mask_dev(float* out, size_t n, float p, const unsigned long long* seed_dev, unsigned long long salt, void* stream) {
  ZCHECK_ARG(out && seed_dev && p >= 0.0f && p < 1.0f, "dropout mask (device seed): bad arguments");
  if (n == 0) return ZEGGS_OK;
  const size_t blocks = (n + 1023) / 1024;
  dropout_mask_dev_kernel<<<(unsigned)(blocks > 2368 ? 2368 : blocks), 256, 0, (cudaStream_t)stream>>>(out, n, p, 1.0f / (1.0f - p), seed_dev, salt);
  count_launch();
  ZCHECK_LAUNCH();
  return ZEGGS_OK;
}
// N(0,1) draws from the same counter-based generator (Box-Muller on two 32-bit words per pair): the VAE noise of
// modules.py:299 (torch.randn_like) without torch's generator, so a captured graph draws fresh noise on every replay
__global__ void randn_dev_kernel(float* __restrict__ out, size_t n, const unsigned long long* __restrict__ seed_dev, unsigned long long salt) {
  uint64_t z = *seed_dev * 0xD1342543DE82EF95ULL + (salt + 1) * 0x9E3779B97F4A7C15ULL;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ULL;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBULL;
  const uint64_t seed = z ^ (z >> 31);
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; 2 * i < n; i += (size_t)gridDim.x * blockDim.x) {
    const float u1 = ((float)mix_u32(seed, 2 * i) + 1.0f) * (1.0f / 4294967296.0f);        // (0, 1]
    const float u2 = (float)mix_u32(seed, 2 * i + 1) * (1.0f / 4294967296.0f);
    const float r = sqrtf(-2.0f * logf(u1));
    float sn, cs;
    sincosf(6.283185307179586f * u2, &sn, &cs);
    out[2 * i] = r * cs;
    if (2 * i + 1 < n) out[2 * i + 1] = r * sn;
  }
}
extern "C" int zeggs_randn_dev(float* out, size_t n, const unsigned long long* seed_dev, unsigned long long salt, void* stream) {
  ZCHECK_ARG(out && seed_dev, "randn (device seed): bad arguments");
  if (n == 0) return ZEGGS_OK;
  const size_t blocks = (n / 2 + 256) / 256;
  randn_dev_kernel<<<(unsigned)(blocks > 1184 ? 1184 : blocks), 256, 0, (cudaStream_t)stream>>>(out, n, seed_dev, salt);
  count_launch();
  ZCHECK_LAUNCH();
  return ZEGGS_OK;
}
extern "C" int zeggs_dropout_mask(float* out, size_t n, float p, unsigned long long seed, void* stream) {
  ZCHECK_ARG(out && p >= 0.0f && p < 1.0f, "dropout mask: bad arguments");
  if (n == 0) return ZEGGS_OK;
  const size_t blocks = (n + 1023) / 1024;
  dropout_mask_kernel<<<(unsigned)(blocks > 2368 ? 2368 : blocks), 256, 0, (cudaStream_t)stream>>>(out, n, p, 1.0f / (1.0f - p), seed);
  count_launch();
  ZCHECK_LAUNCH();
  return ZEGGS_OK;
}
}  // namespace zeggs
