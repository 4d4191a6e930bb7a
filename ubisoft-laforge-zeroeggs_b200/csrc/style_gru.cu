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
  const int U = units_per_cta(H);
  if (U < 0) return 0;
  auto smem_of = [U, H](int nbt) { return dispatch_units(U, [H, nbt](auto u) { return gru_smem_bytes<u>(H, nbt); }); };
  return 32 * max_batch_tiles(smem_of, GRU_SMEM_LIMIT);
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
  GridBarrier gb(bar);
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
        float r, z, n;
        const float h = gru_gate_fwd(gi[j], gi[H + j], gi[2 * H + j], gh[0], gh[1], gh[2], __ldcg(hprev + (size_t)b * H + j), r, z, n);
        Hs[((size_t)(t + 1) * B + b) * H + j] = h;
        float* G = Gs + ((size_t)t * B + b) * 4 * H;
        G[j] = r; G[H + j] = z; G[2 * H + j] = n; G[3 * H + j] = gh[2];
        if (t == T - 1) hcat[(size_t)b * 2 * H + j] = h;
      }
    }
    if (t + 1 < T) grid_sync(gb);
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
  GridBarrier gb(bar);
  for (int t = T - 1; t >= 0; --t) {
    // phase A: gate gradients of the own units (h(t) = (1-z) n + z h(t-1))
    for (int i = tid; i < nbt * U * 32; i += GRU_THREADS) {
      const int bt = i / (U * 32), u = (i >> 5) % U, bl = i & 31, b = bt * 32 + bl, j = c * U + u;
      if (b >= B) continue;
      const float* G = Gs + ((size_t)t * B + b) * 4 * H;
      float dgi[3], dgh[3], dhz;
      gru_gate_bwd(carry[i], G[j], G[H + j], G[2 * H + j], G[3 * H + j], Hs[((size_t)t * B + b) * H + j], dgi, dgh, dhz);
      float* gi = dGih + ((size_t)b * T + t) * H3;
      gi[j] = dgi[0]; gi[H + j] = dgi[1]; gi[2 * H + j] = dgi[2];
      float* gh = dGhh + ((size_t)t * B + b) * H3;
      gh[j] = dgh[0]; gh[H + j] = dgh[1]; gh[2 * H + j] = dgh[2];
      carry[i] = dhz;
    }
    if (t == 0) break;                     // h(-1) = 0 is a constant: no dh(-1)
    grid_sync(gb);
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
// Both kernels pass h_prev = -0, not +0: x + (-0) is x and -0 - n is -n for every x and n, signs of zero included, so the cell's
// (1 - z) n + z h_prev and its dh (h_prev - n) are exactly (1 - z) n and -dh n.
__global__ void rev_cell_fwd_kernel(int B, int H, const float* __restrict__ GIr, const float* __restrict__ bhh, float* __restrict__ hcat) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * H) return;
  const int b = i / H, j = i - b * H;
  const float* gi = GIr + (size_t)b * 3 * H;
  float r, z, n;
  hcat[(size_t)b * 2 * H + H + j] = gru_gate_fwd(gi[j], gi[H + j], gi[2 * H + j], bhh[j], bhh[H + j], bhh[2 * H + j], -0.f, r, z, n);
}
// dh_r = dhcat[:, H:2H] -> dGIr (input-side pre-activations) and dGHr (hidden-side: b_hh_r's gradient rows)
__global__ void rev_cell_bwd_kernel(int B, int H, const float* __restrict__ GIr, const float* __restrict__ bhh, const float* __restrict__ dhcat,
                                    float* __restrict__ dGIr, float* __restrict__ dGHr) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * H) return;
  const int b = i / H, j = i - b * H;
  const float* gi = GIr + (size_t)b * 3 * H;
  float r, z, n, dgi[3], dgh[3], dhz;
  gru_gate_fwd(gi[j], gi[H + j], gi[2 * H + j], bhh[j], bhh[H + j], bhh[2 * H + j], -0.f, r, z, n);
  gru_gate_bwd(dhcat[(size_t)b * 2 * H + H + j], r, z, n, bhh[2 * H + j], -0.f, dgi, dgh, dhz);
  float* a = dGIr + (size_t)b * 3 * H;
  float* h = dGHr + (size_t)b * 3 * H;
  a[j] = dgi[0]; a[H + j] = dgi[1]; a[2 * H + j] = dgi[2];
  h[j] = dgh[0]; h[H + j] = dgh[1]; h[2 * H + j] = dgh[2];
}

// ------------------------------------------------------------------ host side
int style_gru_fwd_launch(int B, int T, int H, const float* Whh, const float* bhh, const float* GI, float* Hs, float* Gs, float* hcat,
                         unsigned* bar, cudaStream_t s) {
  const int U = units_per_cta(H);
  ZCHECK_ARG(U > 0 && B >= 1 && T >= 1, "style GRU: hidden size %d unsupported (need H %% 4 == 0, H <= 528, H %% 8 == 0, H <= 1056, "
             "or H %% 16 == 0, H <= 2112)", H);
  ZCHECK_CUDA(cudaMemsetAsync(bar, 0, 2 * sizeof(unsigned), s));
  ZCHECK_CUDA(cudaMemsetAsync(Hs, 0, (size_t)B * H * sizeof(float), s));     // h(-1) = 0
  return dispatch_units(U, [&](auto u) {
    return launch_persistent(gru_fwd_kernel<u>, H / u, GRU_THREADS, gru_smem_bytes<u>(H, 0), 1, s, B, T, H, Whh, bhh, GI, Hs, Gs, hcat, bar);
  });
}

int style_gru_bwd_launch(int B, int T, int H, const float* Whh, const float* Hs, const float* Gs, const float* dhf, int ld_dhf,
                         float* dGih, float* dGhh, unsigned* bar, cudaStream_t s) {
  const int U = units_per_cta(H);
  ZCHECK_ARG(U > 0 && B >= 1 && T >= 1, "style GRU: hidden size %d unsupported", H);
  ZCHECK_ARG(B <= style_gru_max_batch(H), "style GRU bwd: batch %d above the %d samples the shared memory holds at hidden size %d", B,
             style_gru_max_batch(H), H);
  ZCHECK_CUDA(cudaMemsetAsync(bar, 0, 2 * sizeof(unsigned), s));
  const int nbt = (B + 31) / 32;
  return dispatch_units(U, [&](auto u) {
    return launch_persistent(gru_bwd_kernel<u>, H / u, GRU_THREADS, gru_smem_bytes<u>(H, nbt), 1, s, B, T, H, Whh, Hs, Gs, dhf, ld_dhf, dGih,
                             dGhh, bar);
  });
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
