// zeggs_b200 -- shared device/host helpers for the sm_90a kernels.
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

namespace zeggs {

// ------------------------------------------------------------------ error plumbing (never throw across the ABI)
void set_error(const char* fmt, ...);
const char* get_error();

#define ZEGGS_OK 0
#define ZEGGS_ERR_ARG (-1)
#define ZEGGS_ERR_CUDA (-2)
#define ZEGGS_ERR_UNSUPPORTED (-3)
#define ZEGGS_ERR_TIMEOUT (-4)

#define ZCHECK_ARG(cond, ...)                      \
  do {                                             \
    if (!(cond)) {                                 \
      zeggs::set_error(__VA_ARGS__);               \
      return ZEGGS_ERR_ARG;                        \
    }                                              \
  } while (0)

#define ZCHECK_SUPPORTED(cond, ...)                \
  do {                                             \
    if (!(cond)) {                                 \
      zeggs::set_error(__VA_ARGS__);               \
      return ZEGGS_ERR_UNSUPPORTED;                \
    }                                              \
  } while (0)

#define ZCHECK_CUDA(expr)                                                                 \
  do {                                                                                    \
    cudaError_t _e = (expr);                                                              \
    if (_e != cudaSuccess) {                                                              \
      zeggs::set_error("%s:%d CUDA error %s: %s", __FILE__, __LINE__, #expr,              \
                       cudaGetErrorString(_e));                                           \
      return ZEGGS_ERR_CUDA;                                                              \
    }                                                                                     \
  } while (0)

#define ZCHECK_LAUNCH() ZCHECK_CUDA(cudaGetLastError())

// ------------------------------------------------------------------ pose layout (modules.py:699-710, 731-736)
constexpr int NJ = 75;
constexpr int P_OUT = 6 + NJ * 15;  // 1131
constexpr int P_IN = P_OUT + 3;     // 1134
constexpr int OFF_LPOS = 6;
constexpr int OFF_LTXY = 6 + NJ * 3;
constexpr int OFF_LVEL = 6 + NJ * 9;
constexpr int OFF_LVRT = 6 + NJ * 12;

__host__ __device__ inline int ceil_div(int a, int b) { return (a + b - 1) / b; }
__host__ __device__ inline int round_up(int a, int b) { return ceil_div(a, b) * b; }

// ------------------------------------------------------------------ small math (w-first quaternions, tquat.py)
struct V3 { float x, y, z; };
struct Q4 { float w, x, y, z; };

__host__ __device__ inline V3 v3(float x, float y, float z) { V3 r; r.x = x; r.y = y; r.z = z; return r; }
__host__ __device__ inline V3 operator+(V3 a, V3 b) { return v3(a.x + b.x, a.y + b.y, a.z + b.z); }
__host__ __device__ inline V3 operator-(V3 a, V3 b) { return v3(a.x - b.x, a.y - b.y, a.z - b.z); }
__host__ __device__ inline V3 operator*(float s, V3 a) { return v3(s * a.x, s * a.y, s * a.z); }
__host__ __device__ inline V3 cross(V3 a, V3 b) {
  return v3(a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x);
}
__host__ __device__ inline float dot(V3 a, V3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }

// tquat.py:17-20  quat_mul_vec:  t = 2*cross(q.xyz, v);  v + w*t + cross(q.xyz, t)
__host__ __device__ inline V3 quat_mul_vec(Q4 q, V3 v) {
  V3 u = v3(q.x, q.y, q.z);
  V3 t = 2.0f * cross(u, v);
  return v + q.w * t + cross(u, t);
}
__host__ __device__ inline Q4 quat_inv(Q4 q) { Q4 r; r.w = q.w; r.x = -q.x; r.y = -q.y; r.z = -q.z; return r; }
// tquat.py:5-15  quat_mul(x, y)
__host__ __device__ inline Q4 quat_mul(Q4 x, Q4 y) {
  Q4 r;
  r.w = y.w * x.w - y.x * x.x - y.y * x.y - y.z * x.z;
  r.x = y.w * x.x + y.x * x.w - y.y * x.z + y.z * x.y;
  r.y = y.w * x.y + y.x * x.z + y.y * x.w - y.z * x.x;
  r.z = y.w * x.z - y.x * x.y + y.y * x.x + y.z * x.w;
  return r;
}
// tquat.py:93-106  quat_from_helical(v) = quat_exp(v/2), eps = 1e-5
__host__ __device__ inline Q4 quat_from_helical(V3 h) {
  V3 x = 0.5f * h;
  float ha = sqrtf(dot(x, x));
  Q4 r;
  if (ha < 1e-5f) {
    float n = sqrtf(1.0f + dot(x, x)) + 1e-5f;  // quat_normalize(cat[1, x]), eps 1e-5 (tquat.py:49-51)
    r.w = 1.0f / n; r.x = x.x / n; r.y = x.y / n; r.z = x.z / n;
  } else {
    float s = sinf(ha) / ha;  // x * sinc(ha/pi) = x * sin(ha)/ha
    r.w = cosf(ha); r.x = x.x * s; r.y = x.y * s; r.z = x.z * s;
  }
  return r;
}

// ---- backward helpers (BPTT through the root integration, modules.py:696, 739-740)
// f = quat_mul_vec(q, v); given df returns dq, dv
__host__ __device__ inline void quat_mul_vec_bwd(Q4 q, V3 v, V3 df, Q4& dq, V3& dv) {
  V3 u = v3(q.x, q.y, q.z);
  V3 t = 2.0f * cross(u, v);
  V3 dt = q.w * df + cross(df, u);
  V3 du = cross(t, df) + 2.0f * cross(v, dt);
  dv = df + 2.0f * cross(dt, u);
  dq.w = dot(df, t); dq.x = du.x; dq.y = du.y; dq.z = du.z;
}
// r = quat_mul(x, y); given dr returns dx, dy
__host__ __device__ inline void quat_mul_bwd(Q4 x, Q4 y, Q4 d, Q4& dx, Q4& dy) {
  dx.w = d.w * y.w + d.x * y.x + d.y * y.y + d.z * y.z;
  dx.x = -d.w * y.x + d.x * y.w - d.y * y.z + d.z * y.y;
  dx.y = -d.w * y.y + d.x * y.z + d.y * y.w - d.z * y.x;
  dx.z = -d.w * y.z - d.x * y.y + d.y * y.x + d.z * y.w;
  dy.w = d.w * x.w + d.x * x.x + d.y * x.y + d.z * x.z;
  dy.x = -d.w * x.x + d.x * x.w + d.y * x.z - d.z * x.y;
  dy.y = -d.w * x.y - d.x * x.z + d.y * x.w + d.z * x.x;
  dy.z = -d.w * x.z + d.x * x.y - d.y * x.x + d.z * x.w;
}
// E = quat_from_helical(h) = quat_exp(h/2); given dE returns dh
__host__ __device__ inline V3 quat_from_helical_bwd(V3 h, Q4 dE) {
  V3 x = 0.5f * h;
  float a2 = dot(x, x);
  float a = sqrtf(a2);
  V3 dEv = v3(dE.x, dE.y, dE.z);
  V3 dx;
  if (a < 1e-5f) {
    float rn = sqrtf(1.0f + a2);
    float n = rn + 1e-5f;
    float proj = dE.w + dot(dEv, x);            // dE . [1, x]
    dx = (1.0f / n) * dEv - (proj / (n * n * rn)) * x;
  } else {
    float sn = sinf(a), cs = cosf(a);
    float s = sn / a;
    float dsda = (a * cs - sn) / a2;
    float coef = (-dE.w * sn + dot(dEv, x) * dsda) / a;
    dx = s * dEv + coef * x;
  }
  return 0.5f * dx;
}

__device__ __forceinline__ float elu_f(float x) { return x > 0.0f ? x : expm1f(x); }
__device__ __forceinline__ float elu_grad_from_pre(float pre) { return pre > 0.0f ? 1.0f : expf(pre); }
__device__ __forceinline__ float sigmoid_f(float x) { return 1.0f / (1.0f + expf(-x)); }

// ------------------------------------------------------------------ async copy / cache-controlled access
__device__ __forceinline__ void cp_async16(void* smem, const void* gmem) {
  unsigned s = (unsigned)__cvta_generic_to_shared(smem);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(s), "l"(gmem));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N)); }

__device__ __forceinline__ float ld_cg(const float* p) { return __ldcg(p); }
__device__ __forceinline__ float4 ld_cg4(const float4* p) { return __ldcg(p); }

// ------------------------------------------------------------------ grid-wide barrier for persistent kernels
// All CTAs of a cooperative launch call grid_sync() the same number of times.  `bar` points at two
// zero-initialised unsigned ints in global memory: [0] arrival counter (monotone), [1] error flag.
// A bounded spin (~2 s) turns a would-be hang into an error flag + early exit.
struct GridBarrier {
  unsigned* counter;
  unsigned* error;
  unsigned epoch;
  unsigned nblocks;
};

__device__ __forceinline__ unsigned ld_acquire_u32(const unsigned* p) {
  unsigned v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];\n" : "=r"(v) : "l"(p) : "memory");
  return v;
}

// returns false on timeout / peer error (caller must unwind: every CTA sees the flag)
__device__ __forceinline__ bool grid_sync(GridBarrier& gb) {
  __shared__ int s_ok;
  __syncthreads();
  gb.epoch += 1;
  if (threadIdx.x == 0) {
    int ok = 1;
    __threadfence();
    atomicAdd(gb.counter, 1u);
    const unsigned target = gb.epoch * gb.nblocks;
    long long t0 = clock64();
    unsigned it = 0;
    while (ld_acquire_u32(gb.counter) < target) {
      if ((++it & 1023u) == 0) {
        if (ld_acquire_u32(gb.error) != 0u) { ok = 0; break; }
        if (clock64() - t0 > 4000000000LL) { atomicExch(gb.error, 1u); ok = 0; break; }
      }
    }
    s_ok = ok;
  }
  __syncthreads();
  return s_ok != 0;
}

}  // namespace zeggs
