// The library's internal host API: launch bookkeeping, per-device launch limits, the persistent-kernel launcher, workspace
// carving, the GEMM front end and the launchers one source offers the others.
#pragma once
#include <type_traits>
#include <utility>
#include "common.cuh"
#include "../../include/zeggs_b200.h"

namespace zeggs {

void count_launch();
int timer_id(const char* name);
void* timer_begin(int id, cudaStream_t s);
void timer_end(void* h, cudaStream_t s);
struct ScopedTimer {
  void* h; cudaStream_t s;
  ScopedTimer(const char* name, cudaStream_t st) : h(timer_begin(timer_id(name), st)), s(st) {}
  ~ScopedTimer() { timer_end(h, s); }
};

#define LAUNCH_OK() do { count_launch(); ZCHECK_LAUNCH(); } while (0)
#define RC(x) do { int _rc = (x); if (_rc) return _rc; } while (0)

// ------------------------------------------------------------------ launch limits (abi.cu)
// Queried once per device ordinal: a process may drive several GPUs, and function attributes are per device context.
struct DeviceLimits { int sms; size_t smem_optin; };   // SMs, opt-in dynamic shared memory of one block
int device_limits(DeviceLimits* lim);                   // of the current device
// raises the kernel's dynamic shared-memory limit on the current device to at least `smem` bytes (the CUDA call only when it grows)
int set_max_dynamic_smem(const void* kernel, size_t smem);
template <typename... P>
int set_max_dynamic_smem(void (*kernel)(P...), size_t smem) { return set_max_dynamic_smem((const void*)kernel, smem); }
// CTAs of `block` threads and `smem` bytes that can be resident at once on the current device, in clusters of `cluster` (1 or 2)
int persistent_capacity(const void* kernel, int block, size_t smem, int cluster, int* ctas);

// Persistent kernels spin on grid-wide barriers, so every CTA must be resident at once: the grid is checked against what fits
// (once per kernel, device and shared-memory size) and launched cooperatively, as clusters of `cluster` CTAs.
template <typename... P, typename... A>
int launch_persistent(void (*kernel)(P...), int grid, int block, size_t smem, int cluster, cudaStream_t stream, A&&... args) {
  int fits = 0;
  RC(persistent_capacity((const void*)kernel, block, smem, cluster, &fits));
  ZCHECK_ARG(grid <= fits, "persistent kernel: cooperative grid of %d CTAs (clusters of %d, %zu bytes of shared memory each) does not fit: "
             "%d resident", grid, cluster, smem, fits);
  cudaLaunchAttribute attr[2];
  attr[0].id = cudaLaunchAttributeCooperative;
  attr[0].val.cooperative = 1;
  attr[1].id = cudaLaunchAttributeClusterDimension;
  attr[1].val.clusterDim.x = cluster; attr[1].val.clusterDim.y = 1; attr[1].val.clusterDim.z = 1;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(grid); cfg.blockDim = dim3(block); cfg.dynamicSmemBytes = smem; cfg.stream = stream;
  cfg.attrs = attr; cfg.numAttrs = cluster > 1 ? 2 : 1;
  ZCHECK_CUDA(cudaLaunchKernelEx(&cfg, kernel, std::forward<A>(args)...));
  count_launch();
  return ZEGGS_OK;
}

// ------------------------------------------------------------------ the fp32 recurrences' partition (decoder and GRU style encoder)
// units per CTA: CTA c owns hidden units c*U .. c*U+U-1, and the grid G = H/U must fit one CTA per SM (132 on the H100 SXM).  4 up to
// H = 528, 8 up to 1056, 16 up to 2112; -1 = H unsupported.
inline int units_per_cta(int H) {
  if (H % 4 == 0 && H / 4 <= 132) return 4;
  if (H % 8 == 0 && H / 8 <= 132) return 8;
  if (H % 16 == 0 && H / 16 <= 132) return 16;
  return -1;
}

// calls f(std::integral_constant<int, U>{}) for the units per CTA units_per_cta chose (4, 8 or 16): the one place a run-time U becomes
// the template argument of the fp32 kernels
template <class F>
auto dispatch_units(int U, F&& f) {
  if (U == 4) return f(std::integral_constant<int, 4>{});
  if (U == 8) return f(std::integral_constant<int, 8>{});
  return f(std::integral_constant<int, 16>{});
}

// the largest number of 32-sample batch tiles whose dynamic shared memory smem_of(nbt) (growing with nbt) fits `cap` bytes
template <typename F>
int max_batch_tiles(F smem_of, size_t cap) {
  int nbt = 0;
  while (smem_of(nbt + 1) <= cap) ++nbt;
  return nbt;
}

// ------------------------------------------------------------------ workspace carving
// Cuts one caller-provided buffer into consecutive pieces.  Each piece's size is rounded up to `round` bytes; with base == nullptr
// only the offsets are computed, so one function gives both a workspace's size and its carve-up.
struct Arena {
  char* base;
  size_t off = 0;
  size_t round = 256;
  char* bytes(size_t n) { char* p = here(); off += (n + round - 1) / round * round; return p; }
  float* take(size_t nfloats) { return (float*)bytes(nfloats * sizeof(float)); }
  // the next piece starts at an address that is a multiple of a (a power of two)
  Arena& align(size_t a) { off = (((uintptr_t)base + off + a - 1) & ~(uintptr_t)(a - 1)) - (uintptr_t)base; return *this; }
  char* here() const { return base ? base + off : nullptr; }
  size_t rest(size_t cap) const { return off < cap ? cap - off : 0; }   // bytes left of a `cap`-byte buffer
};

// ------------------------------------------------------------------ GEMM front end (gemm.cu, tc_gemm.cu)
int sgemm_launch(int trans_a, int M, int N, int K, const float* A, int lda, const float* B, int ldb,
                 const float* bias, float* C, int ldc, int act, int accumulate, cudaStream_t stream);
int sgemm_batched_launch(int mode, int M, int N, int K, const float* A, int lda, const float* B, int ldb,
                         const float* bias, float* C, int ldc, int act, int accumulate, int batch,
                         long long sA, long long sB, long long sC, cudaStream_t stream);
int gemm_f32_auto(int mode, int M, int N, int K, const float* A, int lda, const float* B, int ldb, const float* bias,
                  float* C, int ldc, int act, int accumulate, cudaStream_t stream);
const zeggs_ctx* swap_ctx(const zeggs_ctx* c);
// RAII: the caller's context is the active one for the duration of one extern "C" entry point on this host thread
struct CtxScope {
  const zeggs_ctx* old; bool active;
  explicit CtxScope(const zeggs_ctx* c) : old(nullptr), active(c != nullptr) { if (active) old = swap_ctx(c); }
  ~CtxScope() { if (active) swap_ctx(old); }
};
int gemm_mode();
char* scratch_base();
size_t scratch_bytes();
int split_hist_launch(const float* x, long long slot_stride, int S, int R, __nv_bfloat16* hi, __nv_bfloat16* lo, cudaStream_t stream,
                      float* rowsum = nullptr, int s_begin = 0);
int transpose_bf16_launch(const __nv_bfloat16* in, int R, int Ncols, size_t ld_in, __nv_bfloat16* out, size_t ld_out, cudaStream_t stream);
int split_t_launch(const float* x, int rows, int cols, int ld_in, __nv_bfloat16* hi, __nv_bfloat16* lo, int ld_out, cudaStream_t stream);
// convolution-as-GEMM on the tensor cores with the operand produced straight from x (tc_gemm.cu); ZEGGS_CONV_NOT_TAKEN = use the im2col path
constexpr int ZEGGS_CONV_NOT_TAKEN = -1000;
int conv_gemm_fwd(const float* x, int B, int T, int C, int k, int pad, int replicate, const float* W, const float* bias, float* y, int N,
                  int act, cudaStream_t stream);
int conv_gemm_wgrad(const float* dpre, int N, const float* x, int B, int T, int C, int k, int pad, int replicate, float* dW, cudaStream_t stream);
int tc_gemm_launch(int M, int N, int K, const __nv_bfloat16* A_hi, const __nv_bfloat16* A_lo, int lda,
                   const __nv_bfloat16* B_hi, const __nv_bfloat16* B_lo, int ldb, const float* bias,
                   float* C, int ldc, int act, int accumulate, cudaStream_t stream, float* splitk_ws = nullptr,
                   size_t splitk_ws_bytes = 0);
int sgemm_batched2_launch(int mode, int M, int N, int K, const float* A, int lda, const float* B, int ldb,
                          const float* bias, float* C, int ldc, int act, int accumulate, int batch,
                          long long sA, long long sB, long long sC, int inner, long long iA, long long iB, long long iC,
                          float alpha, cudaStream_t stream);
// StyleEncoderGRU recurrences (style_gru.cu)
int style_gru_max_batch(int H);
int style_gru_fwd_launch(int B, int T, int H, const float* Whh, const float* bhh, const float* GI, float* Hs, float* Gs, float* hcat,
                         unsigned* bar, cudaStream_t s);
int style_gru_bwd_launch(int B, int T, int H, const float* Whh, const float* Hs, const float* Gs, const float* dhf, int ld_dhf,
                         float* dGih, float* dGhh, unsigned* bar, cudaStream_t s);
int style_gru_rev_cell_fwd(int B, int H, const float* GIr, const float* bhh, float* hcat, cudaStream_t s);
int style_gru_rev_cell_bwd(int B, int H, const float* GIr, const float* bhh, const float* dhcat, float* dGIr, float* dGHr, cudaStream_t s);

}  // namespace zeggs
