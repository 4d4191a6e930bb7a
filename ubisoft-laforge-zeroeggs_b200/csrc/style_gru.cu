// Bidirectional GRU of StyleEncoderGRU (ZEGGS/modules.py:307-343): the recurrences behind zeggs_style_enc_gru_fwd / _bwd (encoders.cu
// runs the convolutions, the input projections, the projection layer and the VAE sample around them with the shared GEMM front end).
//
// Only output[:, -1] is consumed (:342), so
//   - the forward direction is a true T-step recurrence: ONE persistent cooperative launch (gru_fwd_kernel);
//   - the reverse direction at position T-1 has seen x[T-1] alone, from h = 0: one GRU cell (rev_cell_*), whose W_hh never
//     contributes (its gradient is exactly zero) while b_hh does.
// The input terms x W_ih^T + b_ih of all steps are one batched GEMM issued before the recurrence, so each step's dependent work is
// [B,H] x [H,3H] plus the gate math.  fp32 throughout (FFMA, fp32 state): one engine.
//
// Partitioning (both recurrence kernels): G = H/U CTAs, CTA c owns hidden units j in [c*U, (c+1)*U).
//   forward: CTA c keeps the W_hh rows of its units (3U x H, k-major) resident in shared memory, reads the whole h(t-1) (exchanged
//            through global memory, one grid barrier per step) and writes h(t) of its units.
//   BPTT:    CTA c keeps the W_hh COLUMNS of its units (3H x U) resident.  Phase A (local) turns dh(t) of its units into the gate
//            gradients dG_ih(t), dG_hh(t) of its units; grid barrier; phase B reads the whole dG_hh(t) and forms
//            dh(t-1) = dh(t) * z + dG_hh(t) W_hh for its own units -- which is exactly what phase A of step t-1 needs: one barrier per
//            step again.
//   U = 16 (1056 < H <= 2112): W_hh is 3H^2 fp32 (53.5 MB at H = 2112) against ~30 MB of shared memory on all SMs together, so
//            neither kernel keeps it resident: each K chunk's slice of the CTA's rows (forward) or columns (BPTT) is read from global
//            memory (through L2) into shared memory next to the staged operand chunk, every step.  Same products, same order.
// The K dimension of each per-step product is staged through shared memory in 512-row chunks ([k][33] fp32, conflict-free for
// 32 batch lanes; every thread has 8 global loads in flight per round, since the step is bound by the latency of this exchange);
// batches larger than 32 loop over 32-sample tiles.
#include "library.cuh"

namespace zeggs {

constexpr int GRU_KC = 512;          // rows of the staged operand chunk (the whole h at H = 512)
constexpr int GRU_THREADS = 256;     // 8 warps; warp w takes an eighth of the chunk's rows

// dst[kk][bl] (row stride 33) = src[(b0 + bl) * ld + k0 + kk] for kk < kc, bl < 32; zero for samples b >= B.  Read through L2 (__ldcg):
// the rows were written by other CTAs of the same launch.
__device__ __forceinline__ void gru_stage(float* __restrict__ dst, const float* src, size_t ld, int B, int b0, int k0, int kc) {
  const int n = kc * 32;
  for (int i0 = threadIdx.x; i0 < n; i0 += GRU_THREADS * 8) {
    float v[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const int i = i0 + e * GRU_THREADS, kk = i % kc, b = b0 + i / kc;
      v[e] = (i < n && b < B) ? __ldcg(src + (size_t)b * ld + k0 + kk) : 0.f;
    }
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const int i = i0 + e * GRU_THREADS;
      if (i < n) dst[(i % kc) * 33 + i / kc] = v[e];
    }
  }
}

// U = 16: row stride of the forward's streamed W_hh chunk [KC][GRU_WS], 3U = 48 padded to 52 so that a warp's staging stores
// (16 rows x 2 float4 columns) land in 32 distinct banks, and rows stay 16-byte aligned for the float4 reads of the product
constexpr int GRU_WS = 52;

// W_hh may sit at any 4-byte offset (TrainStep packs all parameters into one flat buffer), so global reads are scalar; a thread reads
// 4 consecutive floats of a row per item and keeps 8 items (32 loads) in flight.
__device__ __forceinline__ float4 ldg4_any(const float* p) { return make_float4(__ldg(p), __ldg(p + 1), __ldg(p + 2), __ldg(p + 3)); }

// Ws[kk][g*16 + u] (row stride GRU_WS) = W_hh[g*H + j0 + u][k0 + kk] for the 48 rows of the CTA's 16 units, kk < kc (kc % 16 == 0).
// Lane bits: 1 for the 4 floats along k, 4 for the row, so a warp reads 16 rows x 32 bytes.
__device__ __forceinline__ void gru_stage_rows16(float* __restrict__ dst, const float* __restrict__ W, int H, int j0, int k0, int kc) {
  const int n = 12 * kc;                   // items of 4 floats: 48 rows x kc/4
  for (int i0 = threadIdx.x; i0 < n; i0 += GRU_THREADS * 8) {
    float4 v[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const int i = i0 + e * GRU_THREADS, rest = i >> 5, g = rest % 3, u = (i >> 1) & 15, k = 4 * (2 * (rest / 3) + (i & 1));
      v[e] = i < n ? ldg4_any(W + (size_t)(g * H + j0 + u) * H + k0 + k) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const int i = i0 + e * GRU_THREADS, rest = i >> 5, g = rest % 3, u = (i >> 1) & 15, k = 4 * (2 * (rest / 3) + (i & 1));
      if (i < n) {
        float* d = dst + k * GRU_WS + g * 16 + u;
        d[0] = v[e].x; d[GRU_WS] = v[e].y; d[2 * GRU_WS] = v[e].z; d[3 * GRU_WS] = v[e].w;
      }
    }
  }
}

// Wc[kk][u] = W_hh[r0 + kk][j0 + u] for the CTA's 16 columns, kk < kc: 64 contiguous bytes per row, stored as they are read
__device__ __forceinline__ void gru_stage_cols16(float* __restrict__ dst, const float* __restrict__ W, int H, int j0, int r0, int kc) {
  const int n = 4 * kc;
  for (int i0 = threadIdx.x; i0 < n; i0 += GRU_THREADS * 8) {
    float4 v[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const int i = i0 + e * GRU_THREADS;
      v[e] = i < n ? ldg4_any(W + (size_t)(r0 + (i >> 2)) * H + j0 + 4 * (i & 3)) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const int i = i0 + e * GRU_THREADS;
      if (i < n) reinterpret_cast<float4*>(dst)[i] = v[e];
    }
  }
}

// units per CTA: 4 while the grid fits one CTA per SM of the H100 (H <= 528), else 8 (H <= 1056), else 16 (H <= 2112); 0 = unsupported
int style_gru_units(int H) {
  if (H % 4 == 0 && H / 4 <= 132) return 4;
  if (H % 8 == 0 && H / 8 <= 132) return 8;
  if (H % 16 == 0 && H / 16 <= 132) return 16;
  return 0;
}

// dynamic shared memory per CTA: the forward kernel's with nbt = 0, the BPTT kernel's with its nbt 32-sample tiles of carry.
// U = 16 keeps no weights resident: the forward holds one [KC][GRU_WS] chunk of W_hh rows, the BPTT one [KC][U] chunk of columns.
template <int U>
static size_t gru_smem_bytes(int H, int nbt) {
  if (U == 16)
    return (size_t)(nbt == 0 ? GRU_KC * GRU_WS + GRU_KC * 33 + 8 * 3 * U * 32
                             : GRU_KC * U + GRU_KC * 33 + 8 * U * 32 + nbt * U * 32) * sizeof(float);
  return (size_t)(3 * U * H + GRU_KC * 33 + 8 * 3 * U * 32 + nbt * U * 32) * sizeof(float);
}

// The opt-in shared memory of one block on sm_90 (227 KB).  A constant rather than a device query, so the workspace query and
// both entry points refuse a batch the backward cannot run before the forward has run.
constexpr size_t GRU_SMEM_LIMIT = 232448;

// the largest batch one call takes at hidden size H (0 = H unsupported): the BPTT kernel's carry grows by U*32 floats per tile
int style_gru_max_batch(int H) {
  const int U = style_gru_units(H);
  if (U == 0) return 0;
  auto bytes = [&](int nbt) { return U == 4 ? gru_smem_bytes<4>(H, nbt) : U == 8 ? gru_smem_bytes<8>(H, nbt) : gru_smem_bytes<16>(H, nbt); };
  int nbt = 0;
  while (bytes(nbt + 1) <= GRU_SMEM_LIMIT) ++nbt;
  return 32 * nbt;
}

// ------------------------------------------------------------------ forward recurrence (modules.py:341, nn.GRU gate order r, z, n)
// GI [B*T][3H] = x W_ih^T + b_ih (rows b*T + t);  Hs [T+1][B][H]: slot 0 = h(-1) = 0 (zeroed by the caller), slot t+1 = h(t);
// Gs [T][B][4H] = r, z, n, W_hn h + b_hn (what BPTT needs);  hcat [B][2H]: h(T-1) into columns [0, H).
template <int U>
__global__ void __launch_bounds__(GRU_THREADS, 1) gru_fwd_kernel(int B, int T, int H, const float* __restrict__ Whh,
                                                                 const float* __restrict__ bhh, const float* __restrict__ GI,
                                                                 float* Hs, float* __restrict__ Gs, float* __restrict__ hcat,
                                                                 unsigned* bar) {
  constexpr int R = 3 * U;
  constexpr bool STREAM = U == 16;        // W_hh read per K chunk (see the top of the file)
  constexpr int WS = STREAM ? GRU_WS : R;
  extern __shared__ __align__(16) float sm[];
  float* Ws = sm;                         // [H][R]: Ws[k*R + g*U + u] = W_hh[g*H + c*U + u][k]; streamed: rows k0 .. k0+kc-1, stride WS
  float* hs = Ws + (STREAM ? (size_t)GRU_KC * WS : (size_t)R * H);   // [KC][33]
  float* red = hs + GRU_KC * 33;          // [8][R][32]
  const int c = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if constexpr (!STREAM)
    for (int i = tid; i < R * H; i += GRU_THREADS) {
      const int r = i / H, k = i - r * H, g = r / U, u = r - g * U;
      Ws[(size_t)k * R + r] = Whh[(size_t)(g * H + c * U + u) * H + k];
    }
  GridBarrier gb; gb.counter = bar; gb.error = bar + 1; gb.epoch = 0; gb.nblocks = gridDim.x;
  const int H3 = 3 * H;
  for (int t = 0; t < T; ++t) {
    const float* hprev = Hs + (size_t)t * B * H;
    for (int b0 = 0; b0 < B; b0 += 32) {
      float acc[R];
#pragma unroll
      for (int r = 0; r < R; ++r) acc[r] = 0.f;
      for (int k0 = 0; k0 < H; k0 += GRU_KC) {
        const int kc = min(GRU_KC, H - k0);
        __syncthreads();
        gru_stage(hs, hprev, H, B, b0, k0, kc);
        if constexpr (STREAM) gru_stage_rows16(Ws, Whh, H, c * U, k0, kc);
        __syncthreads();
        const int kw = (kc + 7) / 8, kend = min(kc, warp * kw + kw);
        for (int kk = warp * kw; kk < kend; ++kk) {
          const float hv = hs[kk * 33 + lane];
          const float4* w4 = reinterpret_cast<const float4*>(Ws + (size_t)((STREAM ? 0 : k0) + kk) * WS);
#pragma unroll
          for (int q = 0; q < R / 4; ++q) {
            const float4 w = w4[q];
            acc[4 * q + 0] = fmaf(w.x, hv, acc[4 * q + 0]);
            acc[4 * q + 1] = fmaf(w.y, hv, acc[4 * q + 1]);
            acc[4 * q + 2] = fmaf(w.z, hv, acc[4 * q + 2]);
            acc[4 * q + 3] = fmaf(w.w, hv, acc[4 * q + 3]);
          }
        }
      }
#pragma unroll
      for (int r = 0; r < R; ++r) red[(warp * R + r) * 32 + lane] = acc[r];
      __syncthreads();
      for (int i = tid; i < U * 32; i += GRU_THREADS) {
        const int u = i >> 5, bl = i & 31, b = b0 + bl, j = c * U + u;
        if (b >= B) continue;
        float gh[3];
#pragma unroll
        for (int g = 0; g < 3; ++g) {
          float s = 0.f;
#pragma unroll
          for (int w = 0; w < 8; ++w) s += red[(w * R + g * U + u) * 32 + bl];
          gh[g] = s + bhh[g * H + j];
        }
        const float* gi = GI + ((size_t)b * T + t) * H3;
        const float r = sigmoid_f(gi[j] + gh[0]), z = sigmoid_f(gi[H + j] + gh[1]);
        const float n = tanhf(gi[2 * H + j] + r * gh[2]);
        const float hp = __ldcg(hprev + (size_t)b * H + j);
        const float h = (1.f - z) * n + z * hp;
        Hs[((size_t)(t + 1) * B + b) * H + j] = h;
        float* G = Gs + ((size_t)t * B + b) * 4 * H;
        G[j] = r; G[H + j] = z; G[2 * H + j] = n; G[3 * H + j] = gh[2];
        if (t == T - 1) hcat[(size_t)b * 2 * H + j] = h;
      }
    }
    if (t + 1 < T) { if (!grid_sync(gb)) return; }
  }
}

// ------------------------------------------------------------------ BPTT of the forward direction
// dhf [B] rows of stride ld_dhf: dL/dh(T-1).  Writes dGih [B*T][3H] (rows b*T + t; gradient of the input pre-activations x W_ih^T + b_ih)
// and dGhh [T][B][3H] (gradient of W_hh h + b_hh).  Weight / bias / input gradients follow as GEMMs and column sums on the host side.
template <int U>
__global__ void __launch_bounds__(GRU_THREADS, 1) gru_bwd_kernel(int B, int T, int H, const float* __restrict__ Whh,
                                                                 const float* __restrict__ Hs, const float* __restrict__ Gs,
                                                                 const float* __restrict__ dhf, int ld_dhf, float* __restrict__ dGih,
                                                                 float* dGhh, unsigned* bar) {
  extern __shared__ __align__(16) float sm[];
  constexpr bool STREAM = U == 16;         // W_hh read per K chunk (see the top of the file)
  const int H3 = 3 * H, nbt = (B + 31) / 32;
  float* Wc = sm;                          // [3H][U]: Wc[row*U + u] = W_hh[row][c*U + u]; streamed: rows r0 .. r0+kc-1
  float* ds = Wc + (size_t)(STREAM ? GRU_KC : H3) * U;       // [KC][33]
  float* red = ds + GRU_KC * 33;           // [8][U][32]  (room for 3U reserved by gru_smem_bytes below U = 16)
  float* carry = red + 8 * (STREAM ? 1 : 3) * U * 32;        // [nbt][U][32]: dh of the own units
  const int c = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if constexpr (!STREAM)
    for (int i = tid; i < H3 * U; i += GRU_THREADS) {
      const int row = i / U, u = i - row * U;
      Wc[i] = Whh[(size_t)row * H + c * U + u];
    }
  for (int i = tid; i < nbt * U * 32; i += GRU_THREADS) {
    const int bt = i / (U * 32), u = (i >> 5) % U, bl = i & 31, b = bt * 32 + bl;
    carry[i] = b < B ? dhf[(size_t)b * ld_dhf + c * U + u] : 0.f;
  }
  __syncthreads();
  GridBarrier gb; gb.counter = bar; gb.error = bar + 1; gb.epoch = 0; gb.nblocks = gridDim.x;
  for (int t = T - 1; t >= 0; --t) {
    // phase A: gate gradients of the own units (h(t) = (1-z) n + z h(t-1))
    for (int i = tid; i < nbt * U * 32; i += GRU_THREADS) {
      const int bt = i / (U * 32), u = (i >> 5) % U, bl = i & 31, b = bt * 32 + bl, j = c * U + u;
      if (b >= B) continue;
      const float dh = carry[i];
      const float* G = Gs + ((size_t)t * B + b) * 4 * H;
      const float r = G[j], z = G[H + j], n = G[2 * H + j], ghn = G[3 * H + j];
      const float hp = Hs[((size_t)t * B + b) * H + j];
      const float dpn = dh * (1.f - z) * (1.f - n * n);
      const float dpr = dpn * ghn * r * (1.f - r);
      const float dpz = dh * (hp - n) * z * (1.f - z);
      float* gi = dGih + ((size_t)b * T + t) * H3;
      gi[j] = dpr; gi[H + j] = dpz; gi[2 * H + j] = dpn;
      float* gh = dGhh + ((size_t)t * B + b) * H3;
      gh[j] = dpr; gh[H + j] = dpz; gh[2 * H + j] = dpn * r;
      carry[i] = dh * z;
    }
    if (t == 0) break;                     // h(-1) = 0 is a constant: no dh(-1)
    if (!grid_sync(gb)) return;
    // phase B: dh(t-1)[own units] += dG_hh(t) W_hh[:, own units]
    const float* dg = dGhh + (size_t)t * B * H3;
    for (int bt = 0; bt < nbt; ++bt) {
      const int b0 = bt * 32;
      float acc[U];
#pragma unroll
      for (int u = 0; u < U; ++u) acc[u] = 0.f;
      for (int r0 = 0; r0 < H3; r0 += GRU_KC) {
        const int kc = min(GRU_KC, H3 - r0);
        __syncthreads();
        gru_stage(ds, dg, H3, B, b0, r0, kc);
        if constexpr (STREAM) gru_stage_cols16(Wc, Whh, H, c * U, r0, kc);
        __syncthreads();
        const int kw = (kc + 7) / 8, kend = min(kc, warp * kw + kw);
        for (int kk = warp * kw; kk < kend; ++kk) {
          const float dv = ds[kk * 33 + lane];
          const float4* w4 = reinterpret_cast<const float4*>(Wc + (size_t)((STREAM ? 0 : r0) + kk) * U);
#pragma unroll
          for (int q = 0; q < U / 4; ++q) {
            const float4 w = w4[q];
            acc[4 * q + 0] = fmaf(w.x, dv, acc[4 * q + 0]);
            acc[4 * q + 1] = fmaf(w.y, dv, acc[4 * q + 1]);
            acc[4 * q + 2] = fmaf(w.z, dv, acc[4 * q + 2]);
            acc[4 * q + 3] = fmaf(w.w, dv, acc[4 * q + 3]);
          }
        }
      }
#pragma unroll
      for (int u = 0; u < U; ++u) red[(warp * U + u) * 32 + lane] = acc[u];
      __syncthreads();
      for (int i = tid; i < U * 32; i += GRU_THREADS) {
        const int u = i >> 5, bl = i & 31;
        float s = 0.f;
#pragma unroll
        for (int w = 0; w < 8; ++w) s += red[(w * U + u) * 32 + bl];
        carry[bt * U * 32 + i] += s;
      }
    }
    __syncthreads();
  }
}

// ------------------------------------------------------------------ the reverse direction: one GRU cell from h = 0
// GIr [B][3H] = x[:, T-1] W_ih_r^T + b_ih_r;  W_hh_r h = 0, so the hidden-side pre-activations are b_hh_r.  h_r -> hcat[:, H:2H].
__global__ void rev_cell_fwd_kernel(int B, int H, const float* __restrict__ GIr, const float* __restrict__ bhh, float* __restrict__ hcat) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * H) return;
  const int b = i / H, j = i - b * H;
  const float* gi = GIr + (size_t)b * 3 * H;
  const float r = sigmoid_f(gi[j] + bhh[j]), z = sigmoid_f(gi[H + j] + bhh[H + j]);
  const float n = tanhf(gi[2 * H + j] + r * bhh[2 * H + j]);
  hcat[(size_t)b * 2 * H + H + j] = (1.f - z) * n;
}
// dh_r = dhcat[:, H:2H] -> dGIr (input-side pre-activations) and dGHr (hidden-side: b_hh_r's gradient rows)
__global__ void rev_cell_bwd_kernel(int B, int H, const float* __restrict__ GIr, const float* __restrict__ bhh, const float* __restrict__ dhcat,
                                    float* __restrict__ dGIr, float* __restrict__ dGHr) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * H) return;
  const int b = i / H, j = i - b * H;
  const float* gi = GIr + (size_t)b * 3 * H;
  const float r = sigmoid_f(gi[j] + bhh[j]), z = sigmoid_f(gi[H + j] + bhh[H + j]);
  const float n = tanhf(gi[2 * H + j] + r * bhh[2 * H + j]);
  const float dh = dhcat[(size_t)b * 2 * H + H + j];
  const float dpn = dh * (1.f - z) * (1.f - n * n);
  const float dpr = dpn * bhh[2 * H + j] * r * (1.f - r);
  const float dpz = -dh * n * z * (1.f - z);
  float* a = dGIr + (size_t)b * 3 * H;
  float* h = dGHr + (size_t)b * 3 * H;
  a[j] = dpr; a[H + j] = dpz; a[2 * H + j] = dpn;
  h[j] = dpr; h[H + j] = dpz; h[2 * H + j] = dpn * r;
}

// ------------------------------------------------------------------ host side
int style_gru_fwd_launch(int B, int T, int H, const float* Whh, const float* bhh, const float* GI, float* Hs, float* Gs, float* hcat,
                         unsigned* bar, cudaStream_t s) {
  const int U = style_gru_units(H);
  ZCHECK_ARG(U > 0 && B >= 1 && T >= 1, "style GRU: hidden size %d unsupported (need H %% 4 == 0, H <= 528, H %% 8 == 0, H <= 1056, "
             "or H %% 16 == 0, H <= 2112)", H);
  ZCHECK_CUDA(cudaMemsetAsync(bar, 0, 2 * sizeof(unsigned), s));
  ZCHECK_CUDA(cudaMemsetAsync(Hs, 0, (size_t)B * H * sizeof(float), s));     // h(-1) = 0
  if (U == 4) return launch_persistent(gru_fwd_kernel<4>, H / 4, GRU_THREADS, gru_smem_bytes<4>(H, 0), 1, s, B, T, H, Whh, bhh, GI, Hs, Gs, hcat, bar);
  if (U == 8) return launch_persistent(gru_fwd_kernel<8>, H / 8, GRU_THREADS, gru_smem_bytes<8>(H, 0), 1, s, B, T, H, Whh, bhh, GI, Hs, Gs, hcat, bar);
  return launch_persistent(gru_fwd_kernel<16>, H / 16, GRU_THREADS, gru_smem_bytes<16>(H, 0), 1, s, B, T, H, Whh, bhh, GI, Hs, Gs, hcat, bar);
}

int style_gru_bwd_launch(int B, int T, int H, const float* Whh, const float* Hs, const float* Gs, const float* dhf, int ld_dhf,
                         float* dGih, float* dGhh, unsigned* bar, cudaStream_t s) {
  const int U = style_gru_units(H);
  ZCHECK_ARG(U > 0 && B >= 1 && T >= 1, "style GRU: hidden size %d unsupported", H);
  ZCHECK_ARG(B <= style_gru_max_batch(H), "style GRU bwd: batch %d above the %d samples the shared memory holds at hidden size %d", B,
             style_gru_max_batch(H), H);
  ZCHECK_CUDA(cudaMemsetAsync(bar, 0, 2 * sizeof(unsigned), s));
  const int nbt = (B + 31) / 32;
  if (U == 4)
    return launch_persistent(gru_bwd_kernel<4>, H / 4, GRU_THREADS, gru_smem_bytes<4>(H, nbt), 1, s, B, T, H, Whh, Hs, Gs, dhf, ld_dhf, dGih, dGhh, bar);
  if (U == 8)
    return launch_persistent(gru_bwd_kernel<8>, H / 8, GRU_THREADS, gru_smem_bytes<8>(H, nbt), 1, s, B, T, H, Whh, Hs, Gs, dhf, ld_dhf, dGih, dGhh, bar);
  return launch_persistent(gru_bwd_kernel<16>, H / 16, GRU_THREADS, gru_smem_bytes<16>(H, nbt), 1, s, B, T, H, Whh, Hs, Gs, dhf, ld_dhf, dGih, dGhh, bar);
}

int style_gru_rev_cell_fwd(int B, int H, const float* GIr, const float* bhh, float* hcat, cudaStream_t s) {
  rev_cell_fwd_kernel<<<ceil_div(B * H, 256), 256, 0, s>>>(B, H, GIr, bhh, hcat);
  count_launch(); ZCHECK_LAUNCH(); return ZEGGS_OK;
}

int style_gru_rev_cell_bwd(int B, int H, const float* GIr, const float* bhh, const float* dhcat, float* dGIr, float* dGHr, cudaStream_t s) {
  rev_cell_bwd_kernel<<<ceil_div(B * H, 256), 256, 0, s>>>(B, H, GIr, bhh, dhcat, dGIr, dGHr);
  count_launch(); ZCHECK_LAUNCH(); return ZEGGS_OK;
}

}  // namespace zeggs
