// Geometry, workspace layout and the weight-stationary "skinny GEMM" building block shared by the
// decoder forward and backward persistent kernels.
#pragma once
#include <type_traits>
#include "library.cuh"

namespace zeggs {

constexpr int K1P = 1136;  // P_IN (1134) rounded up to the 16-row k-chunk

// units per CTA: the grid G = H/U must fit one CTA per SM (132 on the H100 SXM).  At U = 16 the fp32 recurrences run each stage as
// two passes of 8 units (pass_units), so the register tiles and shared-memory stages stay those of U = 8.
inline int pick_U(int H) {
  if (H % 4 == 0 && H / 4 <= 132) return 4;
  if (H % 8 == 0 && H / 8 <= 132) return 8;
  if (H % 16 == 0 && H / 16 <= 132) return 16;
  return -1;
}

// calls f(std::integral_constant<int, U>{}) for the units per CTA pick_U chose (4, 8 or 16): the one place a run-time U becomes the
// template argument of the fp32 kernels
template <class F>
auto dispatch_units(int U, F&& f) {
  if (U == 4) return f(std::integral_constant<int, 4>{});
  if (U == 8) return f(std::integral_constant<int, 8>{});
  return f(std::integral_constant<int, 16>{});
}

// units of one pass of the fp32 recurrences: a CTA's U units are U / pass_units(U) passes, each with its own contiguous weight slice
__host__ __device__ constexpr int pass_units(int U) { return U < 8 ? U : 8; }

// hidden sizes the tensor-core recurrence (engine 1: forward and BPTT kernels) covers; every tc size / pack / run entry point
// applies this one rule (the BPTT kernel pairs 64-wide k-blocks, and below 384 nothing has been validated)
inline bool tc_hidden_ok(int H) { return H % 128 == 0 && H >= 384 && H <= 1024; }
// hidden sizes the fp32 recurrences (engine 0, normal and FiLM) cover: every fp32 size / pack / run entry point applies this rule
inline bool fp32_hidden_ok(int H) { return H % 16 == 0 && pick_U(H) > 0; }

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
  Arena a{(char*)base};
  w.save = save ? 1 : 0;
  w.TS = save ? T : 2;
  w.bar = (unsigned*)a.take(64);
  w.cse_in = a.take((size_t)g.B * (P_IN + g.Z));
  w.cse_h1 = a.take((size_t)g.B * g.H);
  w.cse_h2 = a.take((size_t)g.B * g.H);
  w.cse_out = a.take((size_t)g.B * 2 * g.H);
  w.S01 = a.take((size_t)T * g.nbt * 4 * g.H * 32);
  w.XP = a.take((size_t)(w.TS + 1) * g.nbt * K1P * 32);   // +1: step T-1 never writes slot T, keep the index math simple
  w.A = a.take((size_t)w.TS * g.nbt * g.H * 32);
  w.H0 = a.take((size_t)w.TS * g.nbt * g.H * 32);
  w.H1 = a.take((size_t)w.TS * g.nbt * g.H * 32);
  w.G0 = a.take(save ? (size_t)T * g.nbt * 4 * g.H * 32 : 64);
  w.G1 = a.take(save ? (size_t)T * g.nbt * 4 * g.H * 32 : 64);
  w.CONDR = a.take((size_t)T * g.nbt * 32 * (g.S + g.Z));
  w.H1B = (void*)a.take((size_t)T * 32 * g.H / 2);
  w.YC = a.take((size_t)T * 32 * P_OUT);
  w.Y6 = a.take((size_t)T * 32 * 8);
  w.GZ = a.take((size_t)T * 32 * 4);
  w.bytes = a.off;
  return w;
}

// FiLM decoder (rnn_cond "film"): what the fp32 recurrences read and write beyond the normal decoder's workspace.  The normal
// decoder's kernels take a zeroed one.  GB / DGB rows are (b*T + t): [g-1 (2H) | be (2H)] and their gradients (rows t = 0 stay 0).
struct FilmDev {
  const float* GB;   // [B*T][4H]  predictor outputs: layer-0 half then layer-2 half of gamma - 1, then of beta
  const float* bm;   // [H]        layer2 bias
  float *E0, *E2;    // [TS][nbt][H][32]  ELU outputs of layer0 / layer2 before the modulation (save only)
  float* C2;         // [TS][nbt][H][32]  modulated layer-2 output: the input of layer3
  float* DGB;        // backward: [B*T][4H]
  float* DP2;        // backward: [T][nbt][H][32]  d pre-activation of layer2
};

// rows of the layer-2 FiLM tile (per-CTA units padded to the 8-row minimum of the skinny GEMM)
__host__ __device__ constexpr int film_rows(int U) { return U < 8 ? 8 : U; }

// FiLM forward workspace: the normal decoder's carve-up followed by GB, E0, E2, C2; bytes = the whole workspace
inline FilmDev make_film_ws(void* base, const DecWs& w, const DecGeom& g, int T, size_t* bytes) {
  FilmDev f = {};
  Arena a{(char*)base, w.bytes};
  f.GB = a.take((size_t)g.B * T * 4 * g.H);
  f.E0 = a.take(w.save ? (size_t)T * g.nbt * g.H * 32 : 64);
  f.E2 = a.take(w.save ? (size_t)T * g.nbt * g.H * 32 : 64);
  f.C2 = a.take((size_t)w.TS * g.nbt * g.H * 32);
  *bytes = a.off;
  return f;
}

// the recurrence's geometry of a FiLM decoder: style does not enter layer0 or the GRU, so their input width is 1134 + S
inline DecGeom make_film_geom(int B, int H, int S, int Z) {
  DecGeom g = make_geom(B, H, S, Z);
  g.A = P_IN + S;
  return g;
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
