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
// The K dimension of each per-step product is staged through shared memory in 512-row chunks ([k][33] fp32, conflict-free for
// 32 batch lanes; every thread has 8 global loads in flight per round, since the step is bound by the latency of this exchange);
// batches larger than 32 loop over 32-sample tiles.
#include "decoder_common.cuh"

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

// units per CTA: 4 while the grid fits one CTA per SM of the H100 (H <= 528), else 8 (H <= 1056); 0 = unsupported
int style_gru_units(int H) {
  if (H % 4 == 0 && H / 4 <= 132) return 4;
  if (H % 8 == 0 && H / 8 <= 132) return 8;
  return 0;
}

template <int U>
static size_t gru_smem_bytes(int H, int nbt) {
  return (size_t)(3 * U * H + GRU_KC * 33 + 8 * 3 * U * 32 + nbt * U * 32) * sizeof(float);
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
  extern __shared__ __align__(16) float sm[];
  float* Ws = sm;                         // [H][R]: Ws[k*R + g*U + u] = W_hh[g*H + c*U + u][k]
  float* hs = Ws + (size_t)R * H;         // [KC][33]
  float* red = hs + GRU_KC * 33;          // [8][R][32]
  const int c = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
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
        __syncthreads();
        const int kw = (kc + 7) / 8, kend = min(kc, warp * kw + kw);
        for (int kk = warp * kw; kk < kend; ++kk) {
          const float hv = hs[kk * 33 + lane];
          const float4* w4 = reinterpret_cast<const float4*>(Ws + (size_t)(k0 + kk) * R);
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
  const int H3 = 3 * H, nbt = (B + 31) / 32;
  float* Wc = sm;                          // [3H][U]: Wc[row*U + u] = W_hh[row][c*U + u]
  float* ds = Wc + (size_t)H3 * U;         // [KC][33]
  float* red = ds + GRU_KC * 33;           // [8][U][32]  (room for 3U reserved by gru_smem_bytes)
  float* carry = red + 8 * 3 * U * 32;     // [nbt][U][32]: dh of the own units
  const int c = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
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
        __syncthreads();
        const int kw = (kc + 7) / 8, kend = min(kc, warp * kw + kw);
        for (int kk = warp * kw; kk < kend; ++kk) {
          const float dv = ds[kk * 33 + lane];
          const float4* w4 = reinterpret_cast<const float4*>(Wc + (size_t)(r0 + kk) * U);
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
template <typename K>
static int launch_coop(K kern, int G, size_t smem, void** args, cudaStream_t s) {
  ZCHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  int dev = 0, nsm = 0, occ = 0;
  ZCHECK_CUDA(cudaGetDevice(&dev));
  ZCHECK_CUDA(cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, dev));
  ZCHECK_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, GRU_THREADS, smem));
  ZCHECK_ARG(occ * nsm >= G, "style GRU: cooperative grid of %d CTAs does not fit (%d SMs x %d)", G, nsm, occ);
  ZCHECK_CUDA(cudaLaunchCooperativeKernel((void*)kern, dim3(G), dim3(GRU_THREADS), args, smem, s));
  count_launch();
  return ZEGGS_OK;
}

int style_gru_fwd_launch(int B, int T, int H, const float* Whh, const float* bhh, const float* GI, float* Hs, float* Gs, float* hcat,
                         unsigned* bar, cudaStream_t s) {
  const int U = style_gru_units(H);
  ZCHECK_ARG(U > 0 && B >= 1 && T >= 1, "style GRU: hidden size %d unsupported (need H %% 4 == 0, H <= 528, or H %% 8 == 0, H <= 1056)", H);
  ZCHECK_CUDA(cudaMemsetAsync(bar, 0, 2 * sizeof(unsigned), s));
  ZCHECK_CUDA(cudaMemsetAsync(Hs, 0, (size_t)B * H * sizeof(float), s));     // h(-1) = 0
  void* args[] = {(void*)&B, (void*)&T, (void*)&H, (void*)&Whh, (void*)&bhh, (void*)&GI, (void*)&Hs, (void*)&Gs, (void*)&hcat, (void*)&bar};
  if (U == 4) return launch_coop(gru_fwd_kernel<4>, H / 4, gru_smem_bytes<4>(H, 0), args, s);
  return launch_coop(gru_fwd_kernel<8>, H / 8, gru_smem_bytes<8>(H, 0), args, s);
}

int style_gru_bwd_launch(int B, int T, int H, const float* Whh, const float* Hs, const float* Gs, const float* dhf, int ld_dhf,
                         float* dGih, float* dGhh, unsigned* bar, cudaStream_t s) {
  const int U = style_gru_units(H);
  ZCHECK_ARG(U > 0 && B >= 1 && T >= 1, "style GRU: hidden size %d unsupported", H);
  ZCHECK_CUDA(cudaMemsetAsync(bar, 0, 2 * sizeof(unsigned), s));
  const int nbt = (B + 31) / 32;
  void* args[] = {(void*)&B, (void*)&T, (void*)&H, (void*)&Whh, (void*)&Hs, (void*)&Gs, (void*)&dhf, (void*)&ld_dhf, (void*)&dGih,
                  (void*)&dGhh, (void*)&bar};
  if (U == 4) return launch_coop(gru_bwd_kernel<4>, H / 4, gru_smem_bytes<4>(H, nbt), args, s);
  return launch_coop(gru_bwd_kernel<8>, H / 8, gru_smem_bytes<8>(H, nbt), args, s);
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
