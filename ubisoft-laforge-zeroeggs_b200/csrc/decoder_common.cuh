// Geometry, workspace layout and the weight-stationary "skinny GEMM" building block shared by the
// decoder forward and backward persistent kernels.
#pragma once
#include "common.cuh"
#include "../../include/zeggs_b200.h"

namespace zeggs {

constexpr int K1P = 1136;  // P_IN (1134) rounded up to the 16-row k-chunk

void count_launch();
int timer_id(const char* name);
void* timer_begin(int id, cudaStream_t s);
void timer_end(void* h, cudaStream_t s);
struct ScopedTimer {
  void* h; cudaStream_t s;
  ScopedTimer(const char* name, cudaStream_t st) : h(timer_begin(timer_id(name), st)), s(st) {}
  ~ScopedTimer() { timer_end(h, s); }
};
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
int set_fast_wgrad_internal(int on);   // returns the previous setting
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
int style_gru_units(int H);
int style_gru_fwd_launch(int B, int T, int H, const float* Whh, const float* bhh, const float* GI, float* Hs, float* Gs, float* hcat,
                         unsigned* bar, cudaStream_t s);
int style_gru_bwd_launch(int B, int T, int H, const float* Whh, const float* Hs, const float* Gs, const float* dhf, int ld_dhf,
                         float* dGih, float* dGhh, unsigned* bar, cudaStream_t s);
int style_gru_rev_cell_fwd(int B, int H, const float* GIr, const float* bhh, float* hcat, cudaStream_t s);
int style_gru_rev_cell_bwd(int B, int H, const float* GIr, const float* bhh, const float* dhcat, float* dGIr, float* dGHr, cudaStream_t s);

// units per CTA: the grid G = H/U must fit one CTA per SM (132 on the H100 SXM)
inline int pick_U(int H) {
  if (H % 4 == 0 && H / 4 <= 132) return 4;
  if (H % 8 == 0 && H / 8 <= 132) return 8;
  return -1;
}

// hidden sizes the tensor-core recurrence (engine 1: forward and BPTT kernels) covers; every tc size / pack / run entry point
// applies this one rule (the BPTT kernel pairs 64-wide k-blocks, and below 384 nothing has been validated)
inline bool tc_hidden_ok(int H) { return H % 128 == 0 && H >= 384 && H <= 1024; }

struct DecGeom {
  int B, H, S, Z, A;   // A = 1134 + S + Z
  int U, G;            // units per CTA, CTAs
  int nbt;             // 32-sample batch tiles
  int rpc, n4t;        // layer2 rows per CTA, 16-row tiles per CTA
  __host__ __device__ size_t off_p2() const { return (size_t)G * K1P * 4 * U; }
  __host__ __device__ size_t off_p3() const { return off_p2() + (size_t)G * H * 6 * U; }
  __host__ __device__ size_t off_p4() const { return off_p3() + (size_t)G * H * 6 * U; }
  __host__ __device__ size_t packed_floats() const { return off_p4() + (size_t)G * n4t * H * 16; }
  // backward (transposed) packing, see decoder_bwd.cu
};

inline DecGeom make_geom(int B, int H, int S, int Z) {
  DecGeom g;
  g.B = B; g.H = H; g.S = S; g.Z = Z; g.A = P_IN + S + Z;
  g.U = pick_U(H); g.G = H / g.U;
  g.nbt = ceil_div(B, 32);
  g.rpc = ceil_div(P_OUT, g.G);
  g.n4t = ceil_div(g.rpc, 16);
  return g;
}

// Workspace carve-up.  All recurrent activation buffers are k-major per 32-sample batch tile:
// buf[slot][bt][k][32]  (slot = t when saving for backward, t&1 otherwise).
struct DecWs {
  unsigned* bar;
  float *cse_in, *cse_h1, *cse_h2, *cse_out;
  float *S01;  // [T][nbt][4H][32]   hoisted speech/style contributions (+ b0 / b_ih0); tc engine: [T][32][4H]
  float *CONDR;  // [T][nbt*32][S+Z]  cond rows (tc engine: A operand of the hoisted GEMM)
  float *XP;   // [TS][nbt][K1P][32] normalised pose input of step t
  float *A;    // [TS][nbt][H][32]   ELU(layer0)
  float *H0, *H1;  // [TS][nbt][H][32]  GRU states (slot 0 = CellStateEncoder output)
  float *G0, *G1;  // [T][nbt][4][H][32] r,z,n,(W_hn h + b_hn)   (save only)
  // tc engine (layer2 folded into the next step's layer0/GRU0 input GEMM, see decoder_fwd_tc.cu)
  void* H1B;       // bf16 [T*32][H]     row-major history of h1(t): A operand of the batched layer2 GEMM
  float* YC;       // [T*32][1131]       raw layer2 outputs of the batched GEMM (rows (t,b))
  float* Y6;       // [T][32][8]         de-normalised root velocity channels the in-kernel root integration used
  float* GZ;       // [T][32][4]         normalised gaze direction fed to step t
  int TS, save;
  size_t bytes;
};

inline DecWs make_ws(void* base, const DecGeom& g, int T, int save) {
  DecWs w;
  size_t off = 0;
  auto take = [&](size_t nfloats) {
    float* p = base ? (float*)((char*)base + off) : nullptr;
    off += ((nfloats * sizeof(float) + 255) / 256) * (size_t)256;
    return p;
  };
  w.save = save ? 1 : 0;
  w.TS = save ? T : 2;
  w.bar = (unsigned*)take(64);
  w.cse_in = take((size_t)g.B * (P_IN + g.Z));
  w.cse_h1 = take((size_t)g.B * g.H);
  w.cse_h2 = take((size_t)g.B * g.H);
  w.cse_out = take((size_t)g.B * 2 * g.H);
  w.S01 = take((size_t)T * g.nbt * 4 * g.H * 32);
  w.XP = take((size_t)(w.TS + 1) * g.nbt * K1P * 32);   // +1: step T-1 never writes slot T, keep the index math simple
  w.A = take((size_t)w.TS * g.nbt * g.H * 32);
  w.H0 = take((size_t)w.TS * g.nbt * g.H * 32);
  w.H1 = take((size_t)w.TS * g.nbt * g.H * 32);
  w.G0 = take(save ? (size_t)T * g.nbt * 4 * g.H * 32 : 64);
  w.G1 = take(save ? (size_t)T * g.nbt * 4 * g.H * 32 : 64);
  w.CONDR = take((size_t)T * g.nbt * 32 * (g.S + g.Z));
  w.H1B = (void*)take((size_t)T * 32 * g.H / 2);
  w.YC = take((size_t)T * 32 * P_OUT);
  w.Y6 = take((size_t)T * 32 * 8);
  w.GZ = take((size_t)T * 32 * 4);
  w.bytes = off;
  return w;
}

const float* decoder_tc_mfold(const zeggs_decoder_fwd_args& a);   // fp32 [4H][H] fold matrix inside packed_tc
int decoder_fwd_tc_run(const zeggs_decoder_fwd_args& a, const DecGeom& g, const DecWs& w, cudaStream_t stream);

// ------------------------------------------------------------------ skinny GEMM
// One CTA (8 warps) computes out[r][b] = sum_k Wt[k][r] * x[k][b] for a tile of R = 4*RT rows and 32
// batch columns.  Wt is the CTA's pre-packed k-major slice [K][R]; x is a k-major activation vector
// [K][32] (x_a feeds row groups ng 0,1; x_b feeds ng 2,3 when DUAL).  The K range is cut into 16-row
// chunks dealt round-robin to the 8 warps; each warp runs its own double-buffered cp.async pipeline
// (no block-wide barrier inside the K loop) and keeps a [RT][4] register tile per lane
// (lane = bg + 8*ng: batch quad bg, row group ng).  Partial sums of the 8 warps are combined through
// shared memory by reduce_store()/red_sum().
template <int RT>
struct SkinnyCfg {
  static constexpr int R = 4 * RT;
  static constexpr int WCH = 16 * R;        // floats of W per chunk
  static constexpr int STG = WCH + 1024;    // + two x chunks of 16x32
};

template <int RT, bool DUAL>
__device__ __forceinline__ void skinny_gemm(float (&acc)[RT][4], const float* __restrict__ Wt,
                                            const float* __restrict__ xa, const float* __restrict__ xb,
                                            int nchunks, float* wbuf) {
  constexpr int R = 4 * RT, WCH = 16 * R, STG = WCH + 1024;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int bg = lane & 7, ng = lane >> 3;
#pragma unroll
  for (int i = 0; i < RT; ++i) { acc[i][0] = 0.f; acc[i][1] = 0.f; acc[i][2] = 0.f; acc[i][3] = 0.f; }
  auto issue = [&](int chunk, int s) {
    float* dst = wbuf + s * STG;
    const float* src = Wt + (size_t)chunk * WCH;
#pragma unroll
    for (int i = 0; i < WCH / 128; ++i) cp_async16(dst + 4 * (lane + 32 * i), src + 4 * (lane + 32 * i));
    const float* sa = xa + (size_t)chunk * 512;
#pragma unroll
    for (int i = 0; i < 4; ++i) cp_async16(dst + WCH + 4 * (lane + 32 * i), sa + 4 * (lane + 32 * i));
    if (DUAL) {
      const float* sb = xb + (size_t)chunk * 512;
#pragma unroll
      for (int i = 0; i < 4; ++i) cp_async16(dst + WCH + 512 + 4 * (lane + 32 * i), sb + 4 * (lane + 32 * i));
    }
    cp_async_commit();
  };
  int s = 0;
  if (warp < nchunks) issue(warp, 0);
  for (int ch = warp; ch < nchunks; ch += 8) {
    if (ch + 8 < nchunks) { issue(ch + 8, s ^ 1); cp_async_wait<1>(); } else { cp_async_wait<0>(); }
    __syncwarp();
    const float* W = wbuf + s * STG + ng * RT;
    const float* X = wbuf + s * STG + WCH + ((DUAL && ng >= 2) ? 512 : 0) + bg * 4;
#pragma unroll
    for (int k = 0; k < 16; ++k) {
      const float4 xv = *reinterpret_cast<const float4*>(X + k * 32);
      float wv[RT];
#pragma unroll
      for (int i = 0; i < RT / 2; ++i) {
        const float2 t2 = *reinterpret_cast<const float2*>(W + k * R + 2 * i);
        wv[2 * i] = t2.x; wv[2 * i + 1] = t2.y;
      }
#pragma unroll
      for (int i = 0; i < RT; ++i) {
        acc[i][0] = fmaf(wv[i], xv.x, acc[i][0]);
        acc[i][1] = fmaf(wv[i], xv.y, acc[i][1]);
        acc[i][2] = fmaf(wv[i], xv.z, acc[i][2]);
        acc[i][3] = fmaf(wv[i], xv.w, acc[i][3]);
      }
    }
    __syncwarp();
    s ^= 1;
  }
}

// red[warp][row][32]; row = ng*RT + i
template <int RT>
__device__ __forceinline__ void reduce_store(const float (&acc)[RT][4], float* red) {
  constexpr int R = 4 * RT;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int bg = lane & 7, ng = lane >> 3;
#pragma unroll
  for (int i = 0; i < RT; ++i)
    *reinterpret_cast<float4*>(red + ((size_t)(warp * R + ng * RT + i)) * 32 + bg * 4) =
        make_float4(acc[i][0], acc[i][1], acc[i][2], acc[i][3]);
}

template <int R>
__device__ __forceinline__ float red_sum(const float* red, int row, int b) {
  float s = 0.f;
#pragma unroll
  for (int w = 0; w < 8; ++w) s += red[((size_t)(w * R + row)) * 32 + b];
  return s;
}

}  // namespace zeggs
