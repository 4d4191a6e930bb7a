// Decoder window backward (full BPTT, no detach anywhere -- modules.py:100-151 under autograd):
// one persistent cooperative kernel walks t = T-1 .. 1 with four transposed skinny-GEMM stages per step,
// then batched kernels produce the weight gradients from the saved per-step activations / gate gradients.
//
//   R(t)  dY_acc[t] = dY_ext[t] + d x_pose(t+1)/sigma_in  (+ root-integration backward on channels 0..5)
//   B1    dh1 = dh1_acc + W2^T (dY_acc*sigma_out)           -> GRU1 gate backward -> dgi1, dgh1
//   B2    dh0 = dh0_acc + W_ih1^T dgi1 -> GRU0 gate backward -> dgi0, dgh0 ;  dh1_acc = dh1*z1 + W_hh1^T dgh1
//   B3    da = W_ih0[:, :H]^T dgi0 -> dpre_a = da*ELU'(a)   ;  dh0_acc = dh0*z0 + W_hh0^T dgh0 ;
//         dxp1 = W_ih0[:, pose]^T dgi0
//   B4    dxp = dxp1 + W0[:, pose]^T dpre_a  -> R(t-1)
// Row ownership of the x_pose gradient uses the permuted order [vel 3, vrt 3, gaze 3, rest] so that CTA 0
// holds everything the per-sample root / gaze backward (modules.py:696, 739-740) needs.
#include "decoder_common.cuh"
#include "decoder_bwd_common.cuh"

namespace zeggs {

// PB1[c][k<1136][R1]      W2[k][cU+r]                       (x = dy, k = output channel)
// PB2[c][k<3H][2U]        r<U: W_ih1[k][cU+r]   else W_hh1[k][cU+r-U]
// PB3a[c][k<3H][2U]       r<U: W_ih0[k][cU+r]   else W_hh0[k][cU+r-U]
// PB3b[c][tile][k<3H][16] W_ih0[k][H + perm(c*rpcb + tile*16 + r)]
// PB4[c][tile][k<H][16]   W0[k][perm(c*rpcb + tile*16 + r)]
__global__ void pack_decoder_bwd_kernel(DecGeom g, BwdGeom bg, const float* __restrict__ W0, const float* __restrict__ Wih0,
                                        const float* __restrict__ Whh0, const float* __restrict__ Wih1,
                                        const float* __restrict__ Whh1, const float* __restrict__ W2, float* __restrict__ out) {
  const int H = g.H, U = g.U, A = g.A;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < bg.total; i += (size_t)gridDim.x * blockDim.x) {
    float v = 0.f;
    if (i < bg.off2) {
      size_t e = i;
      int r = e % bg.R1; e /= bg.R1;
      int k = e % K1P; int c = e / K1P;
      if (r < U && k < P_OUT) v = W2[(size_t)k * H + c * U + r];
    } else if (i < bg.off3b) {
      const bool l0 = i >= bg.off3a;
      size_t e = i - (l0 ? bg.off3a : bg.off2);
      int r = e % (2 * U); e /= (2 * U);
      int k = e % (3 * H); int c = e / (3 * H);
      const bool hh = r >= U;
      int j = c * U + (hh ? r - U : r);
      if (!l0) v = hh ? Whh1[(size_t)k * H + j] : Wih1[(size_t)k * H + j];
      else     v = hh ? Whh0[(size_t)k * H + j] : Wih0[(size_t)k * (A + H) + j];
    } else {
      const bool p4 = i >= bg.off4;
      const int KK = p4 ? H : 3 * H;
      size_t e = i - (p4 ? bg.off4 : bg.off3b);
      int r = e % 16; e /= 16;
      int k = e % KK; e /= KK;
      int tile = e % bg.n4b; int c = e / bg.n4b;
      int lr = tile * 16 + r, m = c * bg.rpcb + lr;
      if (lr < bg.rpcb && m < P_IN) {
        int n = xp_perm(m);
        v = p4 ? W0[(size_t)k * A + n] : Wih0[(size_t)k * (A + H) + H + n];
      }
    }
    out[i] = v;
  }
}

template <int U>
__global__ void __launch_bounds__(256, 1)
decoder_bwd_kernel(zeggs_decoder_fwd_args a, DecGeom g, BwdGeom bg, DecWs w, BwdWs bw, BwdArgsDev d) {
  extern __shared__ __align__(16) float smem[];
  constexpr int RT1 = (U < 8 ? 8 : U) / 4;   // B1 tile rows / 4
  constexpr int RT2 = (2 * U) / 4;           // dual tiles
  constexpr int RTM = 4;                     // widest tile used here (16 rows)
  float* stage = smem;                                   // 8 warps x 2 x STG(RTM)
  float* red = smem + 8 * 2 * SkinnyCfg<RTM>::STG;       // [8][16][32]
  float* dhz1 = red + 8 * 16 * 32;                       // [nbt][U][32]   dh1 * z1
  float* dhz0 = dhz1 + g.nbt * U * 32;                   // [nbt][U][32]
  float* dxp1 = dhz0 + g.nbt * U * 32;                   // [nbt][n4b*16][32]
  float* rootg = dxp1 + g.nbt * bg.n4b * 16 * 32;        // [nbt][9][32]  dxp rows vel,vrt,gaze (CTA 0)
  float* dpq = rootg + g.nbt * 9 * 32;                   // [nbt][7][32]  running d root_pos(3) / d root_rot(4) (CTA 0)
  const int c = blockIdx.x, tid = threadIdx.x, warp = tid >> 5;
  const int H = a.H, T = a.T, nbt = g.nbt;
  float* wstage = stage + warp * 2 * SkinnyCfg<RTM>::STG;
  GridBarrier gb; gb.counter = bw.bar; gb.error = bw.bar + 1; gb.epoch = 0; gb.nblocks = gridDim.x;
  const float* PB1 = d.packed + (size_t)c * K1P * bg.R1;
  const float* PB2 = d.packed + bg.off2 + (size_t)c * 3 * H * 2 * U;
  const float* PB3a = d.packed + bg.off3a + (size_t)c * 3 * H * 2 * U;
  const float* PB3b = d.packed + bg.off3b + (size_t)c * bg.n4b * 3 * H * 16;
  const float* PB4 = d.packed + bg.off4 + (size_t)c * bg.n4b * H * 16;
  const size_t actH = (size_t)nbt * H * 32, act3 = (size_t)nbt * 3 * H * 32, actX = (size_t)nbt * K1P * 32, act4 = (size_t)nbt * 4 * H * 32;

  // R(t): finalise dY_acc[t] from dxp (shared `red`-summed values passed through `dxpv`), write DY[t] (scaled by sigma_out).
  // `have_dxp` false for t = T-1.  Executed after B4(t+1) (or as the kernel prologue).
  auto phase_R = [&](int t, int bt, int tile, bool have_dxp) {
    // per-row part: rows of this CTA / tile
    for (int idx = tid; idx < 16 * 32; idx += 256) {
      const int r = idx >> 5, b = idx & 31;
      const int lr = tile * 16 + r, m = c * bg.rpcb + lr;
      if (lr >= bg.rpcb || m >= P_IN) continue;
      const int n = xp_perm(m);
      float dx = 0.f;
      if (have_dxp) dx = (dxp1[(bt * bg.n4b * 16 + lr) * 32 + b] + red_sum<16>(red, r, b)) / a.in_std[n];   // modules.py:713
      if (m < 9) { rootg[(bt * 9 + m) * 32 + b] = dx; continue; }   // CTA 0: handled below with the root terms
      const int bgl = bt * 32 + b;
      float ext = (d.dY && bgl < a.B) ? d.dY[((size_t)bgl * T + t) * P_OUT + n] : 0.f;
      bw.DY[t * actX + ((size_t)bt * K1P + n) * 32 + b] = (ext + dx) * a.out_std[n];                      // modules.py:728
    }
  };
  auto phase_R_root = [&](int t, int bt, bool have_dxp) {
    // CTA 0, one thread per sample: gaze backward of step t+1, root-integration backward of step t.
    if (c != 0) return;
    __syncthreads();
    if (tid < 32) {
      const int b = tid, bgl = bt * 32 + b;
      float* pq = dpq + (bt * 7) * 32;
      if (bgl < a.B) {
        V3 dp; Q4 dq;
        if (!have_dxp) {   // t = T-1: running grads start from the external ones
          dp = d.dRootPos ? v3(d.dRootPos[((size_t)bgl * T + t) * 3 + 0], d.dRootPos[((size_t)bgl * T + t) * 3 + 1], d.dRootPos[((size_t)bgl * T + t) * 3 + 2]) : v3(0, 0, 0);
          if (d.dRootRot) { const float* e = d.dRootRot + ((size_t)bgl * T + t) * 4; dq.w = e[0]; dq.x = e[1]; dq.y = e[2]; dq.z = e[3]; }
          else { dq.w = dq.x = dq.y = dq.z = 0.f; }
        } else {
          dp = v3(pq[0 * 32 + b], pq[1 * 32 + b], pq[2 * 32 + b]);
          dq.w = pq[3 * 32 + b]; dq.x = pq[4 * 32 + b]; dq.y = pq[5 * 32 + b]; dq.z = pq[6 * 32 + b];
        }
        const float* rp = a.root_pos + ((size_t)bgl * T + t) * 3;
        const float* rq = a.root_rot + ((size_t)bgl * T + t) * 4;
        Q4 qt; qt.w = rq[0]; qt.x = rq[1]; qt.y = rq[2]; qt.z = rq[3];
        if (have_dxp) {
          // gaze_dir(t+1) = R(q_t)^-1 (gaze_pos[t+1] - p_t)      modules.py:696
          const float* gp = a.gaze_pos + ((size_t)bgl * T + (t + 1)) * 3;
          V3 u = v3(gp[0] - rp[0], gp[1] - rp[1], gp[2] - rp[2]);
          V3 dgd = v3(rootg[(bt * 9 + 6) * 32 + b], rootg[(bt * 9 + 7) * 32 + b], rootg[(bt * 9 + 8) * 32 + b]);
          Q4 dqc; V3 du;
          quat_mul_vec_bwd(quat_inv(qt), u, dgd, dqc, du);
          dq.w += dqc.w; dq.x -= dqc.x; dq.y -= dqc.y; dq.z -= dqc.z;
          dp = dp - du;
        }
        // root integration of step t (modules.py:739-740): p_t = R(q_{t-1})(vel dt) + p_{t-1};  q_t = exp(R(q_{t-1})(vrt dt)/2) * q_{t-1}
        const float* rq1 = a.root_rot + ((size_t)bgl * T + (t - 1)) * 4;
        Q4 q1; q1.w = rq1[0]; q1.x = rq1[1]; q1.y = rq1[2]; q1.z = rq1[3];
        const float* yt = a.Y + ((size_t)bgl * T + t) * P_OUT;
        V3 a1 = a.dt * v3(yt[0], yt[1], yt[2]);
        V3 a2 = a.dt * v3(yt[3], yt[4], yt[5]);
        Q4 dq_a, dq_b, dq_c, dE; V3 da1, da2;
        quat_mul_vec_bwd(q1, a1, dp, dq_a, da1);
        V3 wv = quat_mul_vec(q1, a2);
        Q4 E = quat_from_helical(wv);
        quat_mul_bwd(E, q1, dq, dE, dq_b);
        V3 dw = quat_from_helical_bwd(wv, dE);
        quat_mul_vec_bwd(q1, a2, dw, dq_c, da2);
        // d vel / d vrt of frame t join the x_pose gradient on channels 0..5
        float dch[6] = {a.dt * da1.x, a.dt * da1.y, a.dt * da1.z, a.dt * da2.x, a.dt * da2.y, a.dt * da2.z};
#pragma unroll
        for (int n = 0; n < 6; ++n) {
          float ext = d.dY ? d.dY[((size_t)bgl * T + t) * P_OUT + n] : 0.f;
          float dx = have_dxp ? rootg[(bt * 9 + n) * 32 + b] : 0.f;
          bw.DY[t * actX + ((size_t)bt * K1P + n) * 32 + b] = (ext + dx + dch[n]) * a.out_std[n];
        }
        // running grads for frame t-1: external + through the integration
        V3 dp1 = dp; Q4 dq1;
        dq1.w = dq_a.w + dq_b.w + dq_c.w; dq1.x = dq_a.x + dq_b.x + dq_c.x; dq1.y = dq_a.y + dq_b.y + dq_c.y; dq1.z = dq_a.z + dq_b.z + dq_c.z;
        if (d.dRootPos) { const float* e = d.dRootPos + ((size_t)bgl * T + (t - 1)) * 3; dp1 = dp1 + v3(e[0], e[1], e[2]); }
        if (d.dRootRot) { const float* e = d.dRootRot + ((size_t)bgl * T + (t - 1)) * 4; dq1.w += e[0]; dq1.x += e[1]; dq1.y += e[2]; dq1.z += e[3]; }
        pq[0 * 32 + b] = dp1.x; pq[1 * 32 + b] = dp1.y; pq[2 * 32 + b] = dp1.z;
        pq[3 * 32 + b] = dq1.w; pq[4 * 32 + b] = dq1.x; pq[5 * 32 + b] = dq1.y; pq[6 * 32 + b] = dq1.z;
      } else {
#pragma unroll
        for (int n = 0; n < 6; ++n) bw.DY[t * actX + ((size_t)bt * K1P + n) * 32 + b] = 0.f;
      }
    }
    __syncthreads();
  };

  // ---- prologue: R(T-1) without a dxp term
  for (int bt = 0; bt < nbt; ++bt) {
    for (int tile = 0; tile < bg.n4b; ++tile) phase_R(T - 1, bt, tile, false);
    phase_R_root(T - 1, bt, false);
  }
  if (!grid_sync(gb)) return;

  for (int t = T - 1; t >= 1; --t) {
    // ------------------------------------------------------------ B1
    for (int bt = 0; bt < nbt; ++bt) {
      float acc[RT1][4];
      const float* x = bw.DY + t * actX + (size_t)bt * K1P * 32;
      skinny_gemm<RT1, false>(acc, PB1, x, x, K1P / 16, wstage);
      reduce_store<RT1>(acc, red);
      __syncthreads();
      for (int idx = tid; idx < U * 32; idx += 256) {
        const int u = idx >> 5, b = idx & 31, j = c * U + u;
        float* acc1 = bw.DH1 + ((size_t)bt * H + j) * 32 + b;
        float dh = red_sum<4 * RT1>(red, u, b) + (t == T - 1 ? 0.f : *acc1);
        const float* G = w.G1 + t * act4 + (size_t)bt * 4 * H * 32;
        float r = G[(size_t)(0 * H + j) * 32 + b], z = G[(size_t)(1 * H + j) * 32 + b];
        float n = G[(size_t)(2 * H + j) * 32 + b], ghn = G[(size_t)(3 * H + j) * 32 + b];
        float hp = w.H1[(t - 1) * actH + ((size_t)bt * H + j) * 32 + b];
        float dgi[3], dgh[3], dhz;
        gru_gate_bwd(dh, r, z, n, ghn, hp, dgi, dgh, dhz);
        dhz1[(bt * U + u) * 32 + b] = dhz;
#pragma unroll
        for (int q = 0; q < 3; ++q) {
          bw.DGI1[t * act3 + ((size_t)bt * 3 * H + q * H + j) * 32 + b] = dgi[q];
          bw.DGH1[t * act3 + ((size_t)bt * 3 * H + q * H + j) * 32 + b] = dgh[q];
        }
      }
      __syncthreads();
    }
    if (!grid_sync(gb)) return;
    // ------------------------------------------------------------ B2
    for (int bt = 0; bt < nbt; ++bt) {
      float acc[RT2][4];
      const float* xa = bw.DGI1 + t * act3 + (size_t)bt * 3 * H * 32;
      const float* xb = bw.DGH1 + t * act3 + (size_t)bt * 3 * H * 32;
      skinny_gemm<RT2, true>(acc, PB2, xa, xb, 3 * H / 16, wstage);
      reduce_store<RT2>(acc, red);
      __syncthreads();
      for (int idx = tid; idx < U * 32; idx += 256) {
        const int u = idx >> 5, b = idx & 31, j = c * U + u;
        float* acc0 = bw.DH0 + ((size_t)bt * H + j) * 32 + b;
        float dh = red_sum<2 * U>(red, u, b) + (t == T - 1 ? 0.f : *acc0);
        const float* G = w.G0 + t * act4 + (size_t)bt * 4 * H * 32;
        float r = G[(size_t)(0 * H + j) * 32 + b], z = G[(size_t)(1 * H + j) * 32 + b];
        float n = G[(size_t)(2 * H + j) * 32 + b], ghn = G[(size_t)(3 * H + j) * 32 + b];
        float hp = w.H0[(t - 1) * actH + ((size_t)bt * H + j) * 32 + b];
        float dgi[3], dgh[3], dhz;
        gru_gate_bwd(dh, r, z, n, ghn, hp, dgi, dgh, dhz);
        dhz0[(bt * U + u) * 32 + b] = dhz;
#pragma unroll
        for (int q = 0; q < 3; ++q) {
          bw.DGI0[t * act3 + ((size_t)bt * 3 * H + q * H + j) * 32 + b] = dgi[q];
          bw.DGH0[t * act3 + ((size_t)bt * 3 * H + q * H + j) * 32 + b] = dgh[q];
        }
        // dh1(t-1) = dh1*z1 + W_hh1^T dgh1
        bw.DH1[((size_t)bt * H + j) * 32 + b] = red_sum<2 * U>(red, U + u, b) + dhz1[(bt * U + u) * 32 + b];
      }
      __syncthreads();
    }
    if (!grid_sync(gb)) return;
    // ------------------------------------------------------------ B3
    for (int bt = 0; bt < nbt; ++bt) {
      {
        float acc[RT2][4];
        const float* xa = bw.DGI0 + t * act3 + (size_t)bt * 3 * H * 32;
        const float* xb = bw.DGH0 + t * act3 + (size_t)bt * 3 * H * 32;
        skinny_gemm<RT2, true>(acc, PB3a, xa, xb, 3 * H / 16, wstage);
        reduce_store<RT2>(acc, red);
        __syncthreads();
        for (int idx = tid; idx < U * 32; idx += 256) {
          const int u = idx >> 5, b = idx & 31, j = c * U + u;
          float av = w.A[t * actH + ((size_t)bt * H + j) * 32 + b];
          float da = red_sum<2 * U>(red, u, b);
          bw.DPA[t * actH + ((size_t)bt * H + j) * 32 + b] = da * (av > 0.f ? 1.f : av + 1.f);   // ELU'(pre) = a+1 for pre<=0
          bw.DH0[((size_t)bt * H + j) * 32 + b] = red_sum<2 * U>(red, U + u, b) + dhz0[(bt * U + u) * 32 + b];
        }
        __syncthreads();
      }
      if (t > 1) {
        const float* x = bw.DGI0 + t * act3 + (size_t)bt * 3 * H * 32;
        for (int tile = 0; tile < bg.n4b; ++tile) {
          float acc[4][4];
          skinny_gemm<4, false>(acc, PB3b + (size_t)tile * 3 * H * 16, x, x, 3 * H / 16, wstage);
          reduce_store<4>(acc, red);
          __syncthreads();
          for (int idx = tid; idx < 16 * 32; idx += 256) {
            const int r = idx >> 5, b = idx & 31;
            dxp1[(bt * bg.n4b * 16 + tile * 16 + r) * 32 + b] = red_sum<16>(red, r, b);
          }
          __syncthreads();
        }
      }
    }
    if (t == 1) break;
    if (!grid_sync(gb)) return;
    // ------------------------------------------------------------ B4 + R(t-1)
    for (int bt = 0; bt < nbt; ++bt) {
      const float* x = bw.DPA + t * actH + (size_t)bt * H * 32;
      for (int tile = 0; tile < bg.n4b; ++tile) {
        float acc[4][4];
        skinny_gemm<4, false>(acc, PB4 + (size_t)tile * H * 16, x, x, H / 16, wstage);
        reduce_store<4>(acc, red);
        __syncthreads();
        phase_R(t - 1, bt, tile, true);
        __syncthreads();
      }
      phase_R_root(t - 1, bt, true);
    }
    if (!grid_sync(gb)) return;
  }
}

// ------------------------------------------------------------------ batched kernels over the k-major histories
// dW[n][k] = sum_{t'<nT} sum_{bt} sum_b GA[t'][bt][n][b] * XB[t'][bt][k][b]      (64 x 64 tile per CTA)
__global__ void __launch_bounds__(256) wgrad_kmajor_kernel(const float* __restrict__ GA, long long gaT, long long gaBT, int N,
                                                           const float* __restrict__ XB, long long xbT, long long xbBT, int K,
                                                           int nT, int nbt, float* __restrict__ dW, int ldw) {
  __shared__ float As[32][64 + 1];
  __shared__ float Bs[32][64 + 1];
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int n0 = blockIdx.y * 64, k0 = blockIdx.x * 64;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  for (int s = 0; s < nT * nbt; ++s) {
    const int tt = s / nbt, bt = s - tt * nbt;
    const float* ga = GA + tt * gaT + bt * gaBT;
    const float* xb = XB + tt * xbT + bt * xbBT;
    for (int i = tid; i < 64 * 32; i += 256) {
      const int r = i >> 5, b = i & 31;
      As[b][r] = (n0 + r < N) ? __ldg(ga + (size_t)(n0 + r) * 32 + b) : 0.f;
      Bs[b][r] = (k0 + r < K) ? __ldg(xb + (size_t)(k0 + r) * 32 + b) : 0.f;
    }
    __syncthreads();
#pragma unroll 8
    for (int b = 0; b < 32; ++b) {
      float av[4], bv[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) { av[i] = As[b][ty * 4 + i]; bv[i] = Bs[b][tx * 4 + i]; }
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int n = n0 + ty * 4 + i;
    if (n >= N) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int k = k0 + tx * 4 + j;
      if (k < K) dW[(size_t)n * ldw + k] = acc[i][j];
    }
  }
}

// db[n] = sum over slots and b of GA[t'][bt][n][b]; one warp per row
__global__ void rowsum_kmajor_kernel(const float* __restrict__ GA, long long gaT, long long gaBT, int N, int nT, int nbt, float* __restrict__ db) {
  const int n = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (n >= N) return;
  float s = 0.f;
  for (int tt = 0; tt < nT; ++tt)
    for (int bt = 0; bt < nbt; ++bt) s += __ldg(GA + tt * gaT + bt * gaBT + (size_t)n * 32 + lane);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) db[n] = s;
}

// COND[t][bt][c][32] = [speech | style][b, t, c]
__global__ void cond_kmajor_kernel(zeggs_decoder_fwd_args a, DecGeom g, float* __restrict__ COND) {
  const int C = a.S + a.Z;
  const size_t total = (size_t)a.T * g.nbt * C * 32;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    int bl = i % 32; size_t e = i / 32;
    int cc = e % C; e /= C;
    int bt = e % g.nbt; int t = e / g.nbt;
    int b = bt * 32 + bl;
    float v = 0.f;
    if (b < a.B) v = cc < a.S ? a.speech[((size_t)b * a.T + t) * a.S + cc] : a.style[((size_t)b * a.T + t) * a.Z + (cc - a.S)];
    COND[i] = v;
  }
}

// dSpeech/dStyle[b][t][c] from DCOND[t][bt][c][32] (t>=1) ; t = 0: zero for speech, CellStateEncoder input grad for style
// rows != 0: DCOND is [(t*32 + b)][c] (tc engine, nbt == 1)
__global__ void dcond_scatter_kernel(zeggs_decoder_fwd_args a, DecGeom g, const float* __restrict__ DCOND, const float* __restrict__ cse_din,
                                     float* __restrict__ dSpeech, float* __restrict__ dStyle, int rows) {
  const int C = a.S + a.Z;
  const size_t total = (size_t)a.B * a.T * C;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    int cc = i % C; size_t e = i / C;
    int t = e % a.T; int b = e / a.T;
    float v = 0.f;
    if (t >= 1) v = rows ? DCOND[((size_t)t * 32 + b) * C + cc] : DCOND[(((size_t)t * g.nbt + b / 32) * C + cc) * 32 + (b % 32)];
    else if (cc >= a.S) v = cse_din[(size_t)b * (P_IN + a.Z) + P_IN + (cc - a.S)];
    if (cc < a.S) { if (dSpeech) dSpeech[((size_t)b * a.T + t) * a.S + cc] = v; }
    else if (dStyle) dStyle[((size_t)b * a.T + t) * a.Z + (cc - a.S)] = v;
  }
}

// cse_dout[b][l*H + j] = DH_l[bt][j][bl]
__global__ void cse_gather_kernel(int B, int H, const float* __restrict__ dh0, const float* __restrict__ dh1, float* __restrict__ dout) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * 2 * H) return;
  int b = i / (2 * H), r = i % (2 * H);
  const float* src = r < H ? dh0 : dh1;
  int j = r % H;
  dout[i] = src[((size_t)(b / 32) * H + j) * 32 + (b % 32)];
}

__global__ void elu_bwd_kernel(float* __restrict__ dx, const float* __restrict__ y, size_t n) {
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i < n) { float v = y[i]; dx[i] *= (v > 0.f ? 1.f : v + 1.f); }
}

__global__ void colsum_kernel(const float* __restrict__ x, int rows, int cols, float* __restrict__ out) {
  int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= cols) return;
  float s = 0.f;
  for (int r = 0; r < rows; ++r) s += x[(size_t)r * cols + c];
  out[c] = s;
}

// tc engine (folded recurrence): rebuild the layer-2 / x_pose gradient history the weight gradients read.
//   DY[t][n][b] = out_std[n] (dY_ext[b][t][n] + DXP[(t+1,b)][n] / in_std[n] + [n < 6] DCH[t][b][n]),  t = 1..T-1
// One CTA per (t, 64-channel chunk); DXP rows (t,b) are transposed through shared memory into the k-major history.
__global__ void __launch_bounds__(256) dy_combine_kernel(zeggs_decoder_fwd_args a, const float* __restrict__ dYext, const float* __restrict__ dxp,
                                                         const float* __restrict__ dch, float* __restrict__ DY) {
  __shared__ float tile[32][65];
  const int t = 1 + blockIdx.x, n0 = blockIdx.y * 64, T = a.T;
  const int tx = threadIdx.x & 63, ty = threadIdx.x >> 6;
  const int n = n0 + tx;
  float os = 0.f, ris = 0.f;
  if (n < P_OUT) { os = a.out_std[n]; ris = 1.0f / a.in_std[n]; }
  for (int b = ty; b < 32; b += 4) {
    float v = 0.f;
    if (n < P_OUT && b < a.B) {
      v = dYext ? dYext[((size_t)b * T + t) * P_OUT + n] : 0.f;
      if (t + 1 < T) v += dxp[((size_t)(t + 1) * 32 + b) * P_OUT + n] * ris;
      if (n < 6) v += dch[((size_t)t * 32 + b) * 8 + n];
      v *= os;
    }
    tile[b][tx] = v;
  }
  __syncthreads();
  float* dst = DY + (size_t)t * K1P * 32;
  const int b = threadIdx.x & 31;
  for (int r = threadIdx.x >> 5; r < 64; r += 8) {
    const int nn = n0 + r;
    if (nn < P_OUT) dst[(size_t)nn * 32 + b] = tile[b][r];
  }
}

// ------------------------------------------------------------------ host
extern "C" size_t zeggs_decoder_packed_bwd_bytes(int H, int S, int Z) {
  if (H % 16 != 0 || pick_U(H) <= 0) return 0;
  DecGeom g = make_geom(1, H, S, Z);
  return make_bgeom(g).total * sizeof(float);
}

extern "C" int zeggs_decoder_pack_weights_bwd(const zeggs_decoder_fwd_args* a, float* packed, void* stream_) {
  CtxScope ctx_scope(a ? a->ctx : nullptr);
  ZCHECK_ARG(a && packed && a->H % 16 == 0 && pick_U(a->H) > 0, "decoder bwd pack: bad arguments");
  DecGeom g = make_geom(a->B, a->H, a->S, a->Z);
  BwdGeom bg = make_bgeom(g);
  pack_decoder_bwd_kernel<<<592, 256, 0, (cudaStream_t)stream_>>>(g, bg, a->W0, a->W_ih0, a->W_hh0, a->W_ih1, a->W_hh1, a->W2, packed);
  count_launch();
  ZCHECK_LAUNCH();
  return ZEGGS_OK;
}

extern "C" size_t zeggs_decoder_bwd_workspace_bytes(int B, int T, int H, int S, int Z) {
  if (H % 16 != 0 || pick_U(H) <= 0 || B < 1 || T < 1) return 0;
  DecGeom g = make_geom(B, H, S, Z);
  return make_bws(nullptr, g, T).bytes;
}

template <int U>
static int launch_bwd(const zeggs_decoder_fwd_args& a, const DecGeom& g, const BwdGeom& bg, const DecWs& w, const BwdWs& bw,
                      const BwdArgsDev& d, cudaStream_t stream) {
  size_t smem = (size_t)(8 * 2 * SkinnyCfg<4>::STG + 8 * 16 * 32 + 2 * g.nbt * U * 32 + g.nbt * bg.n4b * 16 * 32 + g.nbt * 9 * 32 + g.nbt * 7 * 32) * sizeof(float);
  ZCHECK_CUDA(cudaFuncSetAttribute(decoder_bwd_kernel<U>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  int dev = 0, nsm = 0, occ = 0;
  ZCHECK_CUDA(cudaGetDevice(&dev));
  ZCHECK_CUDA(cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, dev));
  ZCHECK_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, decoder_bwd_kernel<U>, 256, smem));
  ZCHECK_ARG(occ * nsm >= g.G, "decoder bwd: cooperative grid of %d CTAs does not fit", g.G);
  void* args[] = {(void*)&a, (void*)&g, (void*)&bg, (void*)&w, (void*)&bw, (void*)&d};
  ZCHECK_CUDA(cudaLaunchCooperativeKernel((void*)decoder_bwd_kernel<U>, dim3(g.G), dim3(256), args, smem, stream));
  count_launch();
  return ZEGGS_OK;
}

static int wgrad(const float* GA, long long gaT, long long gaBT, int N, const float* XB, long long xbT, long long xbBT, int K,
                 int nT, int nbt, float* dW, int ldw, cudaStream_t stream) {
  wgrad_kmajor_kernel<<<dim3(ceil_div(K, 64), ceil_div(N, 64)), 256, 0, stream>>>(GA, gaT, gaBT, N, XB, xbT, xbBT, K, nT, nbt, dW, ldw);
  count_launch();
  ZCHECK_LAUNCH();
  return ZEGGS_OK;
}
static int rowsum(const float* GA, long long gaT, long long gaBT, int N, int nT, int nbt, float* db, cudaStream_t stream) {
  rowsum_kmajor_kernel<<<ceil_div(N, 8), 256, 0, stream>>>(GA, gaT, gaBT, N, nT, nbt, db);
  count_launch();
  ZCHECK_LAUNCH();
  return ZEGGS_OK;
}

extern "C" int zeggs_decoder_window_bwd(const zeggs_decoder_fwd_args* ap, const zeggs_decoder_bwd_args* bp, void* stream_) {
  CtxScope ctx_scope(ap ? ap->ctx : nullptr);
  ZCHECK_ARG(ap && bp, "decoder bwd: null args");
  const zeggs_decoder_fwd_args& a = *ap;
  const zeggs_decoder_bwd_args& b = *bp;
  cudaStream_t stream = (cudaStream_t)stream_;
  ZCHECK_ARG(a.save_for_backward && a.workspace, "decoder bwd: forward must have run with save_for_backward=1");
  ZCHECK_ARG(a.T >= 1 && b.phase >= 0 && b.phase <= 2, "decoder bwd: bad T=%d / phase=%d", a.T, b.phase);
  if (a.T == 1) {
    // a one-frame window outputs the given first pose (modules.py:72-79): no weight and no conditioning input reaches it, so every
    // gradient is zero (the reference's autograd gives the same)
    if (b.phase == 2) return ZEGGS_OK;
    const size_t H = a.H, A = P_IN + a.S + a.Z, Kin = P_IN + a.Z;
    const struct { float* p; size_t n; } zero[] = {
        {b.dW0, H * A}, {b.db0, H}, {b.dW_ih0, 3 * H * (A + H)}, {b.db_ih0, 3 * H}, {b.dW_hh0, 3 * H * H}, {b.db_hh0, 3 * H},
        {b.dW_ih1, 3 * H * H}, {b.db_ih1, 3 * H}, {b.dW_hh1, 3 * H * H}, {b.db_hh1, 3 * H}, {b.dW2, (size_t)P_OUT * H}, {b.db2, (size_t)P_OUT},
        {b.dWc0, H * Kin}, {b.dbc0, H}, {b.dWc1, H * H}, {b.dbc1, H}, {b.dWc2, 2 * H * H}, {b.dbc2, 2 * H},
        {b.dSpeech, (size_t)a.B * a.S}, {b.dStyle, (size_t)a.B * a.Z}};
    for (const auto& z : zero)
      if (z.p) ZCHECK_CUDA(cudaMemsetAsync(z.p, 0, z.n * sizeof(float), stream));
    return ZEGGS_OK;
  }
  DecGeom g = make_geom(a.B, a.H, a.S, a.Z);
  BwdGeom bg = make_bgeom(g);
  DecWs w = make_ws(a.workspace, g, a.T, 1);
  BwdWs bw = make_bws(b.workspace, g, a.T);
  ZCHECK_ARG(b.workspace && b.workspace_bytes >= bw.bytes, "decoder bwd: workspace too small (%zu < %zu)", b.workspace_bytes, bw.bytes);
  const bool use_tc = a.engine == 1 && b.packed_bwd_tc != nullptr && g.nbt == 1 && bg.n4b == 1;
  ZCHECK_ARG(use_tc || b.packed_bwd, "decoder bwd: packed_bwd missing");
  const int H = a.H, T = a.T, nbt = g.nbt, C = a.S + a.Z, A = g.A;
  // phase 0: the whole backward.  The tensor-core engine can run it in two calls so that the encoders' backward passes (which need only
  // dSpeech / dStyle) overlap the large weight-gradient GEMMs on other streams: phase 1 = BPTT recurrence + CellStateEncoder backward +
  // the conditioning gradients (dSpeech, dStyle); phase 2 = every remaining parameter gradient.  Other engines do all of it in phase 1.
  const int phase = b.phase;
  ZCHECK_ARG(phase >= 0 && phase <= 2, "decoder bwd: phase must be 0, 1 or 2");
  const bool fold = use_tc && nbt == 1 && H % 64 == 0 && gemm_mode() != 0 && scratch_base() != nullptr;
  const bool p1 = phase != 2, p2 = phase != 1 || !fold;
  if (phase == 2 && !fold) return ZEGGS_OK;
  int rc;
  if (p1) {
    ZCHECK_CUDA(cudaMemsetAsync(bw.bar, 0, 256, stream));
    ZCHECK_CUDA(cudaMemsetAsync(bw.DY, 0, (size_t)T * nbt * K1P * 32 * sizeof(float), stream));
    BwdArgsDev d; d.dY = b.dY; d.dRootPos = b.dRootPos; d.dRootRot = b.dRootRot; d.packed = b.packed_bwd;
    ScopedTimer tm("decoder_bwd", stream);
    if (use_tc) rc = decoder_bwd_tc_run(a, b, g, w, bw, stream);
    else rc = (g.U == 4) ? launch_bwd<4>(a, g, bg, w, bw, d, stream) : launch_bwd<8>(a, g, bg, w, bw, d, stream);
    if (rc) return rc;
  }
  ScopedTimer tmw("decoder_wgrad", stream);
  if (p1) {
    cond_kmajor_kernel<<<592, 256, 0, stream>>>(a, g, bw.COND);
    count_launch();
    ZCHECK_LAUNCH();
  }
  const long long sH = (long long)nbt * H * 32, s3 = (long long)nbt * 3 * H * 32, sX = (long long)nbt * K1P * 32, sC = (long long)nbt * C * 32;
  const int nT = T - 1;
  const int Kin = P_IN + a.Z;
  // ---- CellStateEncoder backward (modules.py:238-243).  Its small GEMMs stage operands at the base of the scratch buffer, so on the
  // folded path it runs BEFORE the bf16 history copies are laid out there (cse_tail = false afterwards)
  auto cse_backward = [&]() -> int {
    int r;
    cse_gather_kernel<<<ceil_div(a.B * 2 * H, 256), 256, 0, stream>>>(a.B, H, bw.DH0, bw.DH1, bw.cse_dout);
    count_launch();
    r = sgemm_launch(1, 2 * H, H, a.B, bw.cse_dout, 2 * H, w.cse_h2, H, nullptr, b.dWc2, H, 0, 0, stream); if (r) return r;
    colsum_kernel<<<ceil_div(2 * H, 256), 256, 0, stream>>>(bw.cse_dout, a.B, 2 * H, b.dbc2); count_launch();
    r = gemm_f32_auto(2, a.B, H, 2 * H, bw.cse_dout, 2 * H, a.Wc2, H, nullptr, bw.cse_d2, H, 0, 0, stream); if (r) return r;
    elu_bwd_kernel<<<ceil_div(a.B * H, 256), 256, 0, stream>>>(bw.cse_d2, w.cse_h2, (size_t)a.B * H); count_launch();
    r = sgemm_launch(1, H, H, a.B, bw.cse_d2, H, w.cse_h1, H, nullptr, b.dWc1, H, 0, 0, stream); if (r) return r;
    colsum_kernel<<<ceil_div(H, 256), 256, 0, stream>>>(bw.cse_d2, a.B, H, b.dbc1); count_launch();
    r = gemm_f32_auto(2, a.B, H, H, bw.cse_d2, H, a.Wc1, H, nullptr, bw.cse_d1, H, 0, 0, stream); if (r) return r;
    elu_bwd_kernel<<<ceil_div(a.B * H, 256), 256, 0, stream>>>(bw.cse_d1, w.cse_h1, (size_t)a.B * H); count_launch();
    r = sgemm_launch(1, H, Kin, a.B, bw.cse_d1, H, w.cse_in, Kin, nullptr, b.dWc0, Kin, 0, 0, stream); if (r) return r;
    colsum_kernel<<<ceil_div(H, 256), 256, 0, stream>>>(bw.cse_d1, a.B, H, b.dbc0); count_launch();
    r = gemm_f32_auto(2, a.B, Kin, H, bw.cse_d1, H, a.Wc0, Kin, nullptr, bw.cse_din, Kin, 0, 0, stream); if (r) return r;
    ZCHECK_LAUNCH();
    return ZEGGS_OK;
  };
  bool cse_tail = true;
  if (fold && p1) { if ((rc = cse_backward())) return rc; }
  if (fold) cse_tail = false;
  // ---- weight gradients (slots t = 1..T-1).  tensor-core path: every history is re-laid out once as bf16 (hi, lo)
  // [rows][(T*nbt)*32] (contraction index contiguous) in the scratch buffer, then each dW is one NT GEMM with
  // K = (T-1)*nbt*32; "previous step" operands are the same buffer shifted by one slot (32*nbt columns).
  bool tc_done = false, dcond_rows = false;
  if (gemm_mode() != 0 && scratch_base() != nullptr) {
    // the tc engine's recurrence already runs on bf16 operands: a single bf16 pass matches its accuracy
    const bool want_lo = gemm_mode() == 1 && !use_tc;
    const int S = T * nbt;                       // slots per history
    const size_t ld = (size_t)S * 32;
    char* p = scratch_base();
    struct Hist { const float* src; long long stride; int rows; __nv_bfloat16 *hi, *lo; float* db; };
    Hist hs[11] = {
      {bw.DY, sX, P_OUT, nullptr, nullptr, b.db2}, {bw.DGI1, s3, 3 * H, nullptr, nullptr, b.db_ih1}, {bw.DGH1, s3, 3 * H, nullptr, nullptr, b.db_hh1},
      {bw.DGI0, s3, 3 * H, nullptr, nullptr, b.db_ih0}, {bw.DGH0, s3, 3 * H, nullptr, nullptr, b.db_hh0}, {bw.DPA, sH, H, nullptr, nullptr, b.db0},
      {w.H0, sH, H, nullptr, nullptr, nullptr}, {w.H1, sH, H, nullptr, nullptr, nullptr}, {w.A, sH, H, nullptr, nullptr, nullptr},
      {w.XP, sX, P_IN, nullptr, nullptr, nullptr}, {bw.COND, sC, C, nullptr, nullptr, nullptr}};
    size_t need = 0;
    for (auto& h : hs) need += (size_t)h.rows * ld * 2 * (want_lo ? 2 : 1);
    // tc engine: the dpre_a / dgi0 histories are also needed transposed ([(t,b)][row], bf16) -- for the hoisted cond terms and
    // for the x_pose gradient of the folded recurrence -- plus the transposed weight blocks and the DXP result
    const size_t extra = fold ? (ld * H * 2 + ld * 3 * H * 2 + (size_t)C * 4 * H * 2 + (size_t)P_OUT * 4 * H * 2 + ld * P_OUT * 4 + 4096) : 0;
    if (need + extra <= scratch_bytes()) {
      // all hi parts first, then all lo parts: (ld * 2) bytes per row, 16 B aligned, so consecutive histories stack into ONE
      // row-contiguous operand ([a | x_pose | cond] is the input of layer0 / GRU0 in the weights' own column order)
      for (auto& h : hs) { h.hi = (__nv_bfloat16*)p; p += (size_t)h.rows * ld * 2; }
      if (want_lo) for (auto& h : hs) { h.lo = (__nv_bfloat16*)p; p += (size_t)h.rows * ld * 2; }
      auto takeq = [&](size_t bytes) { char* r = (char*)(((uintptr_t)p + 255) & ~(uintptr_t)255); p = r + bytes; return r; };
      __nv_bfloat16 *paT = nullptr, *giT = nullptr, *w0T = nullptr, *wiT = nullptr, *w0xT = nullptr, *wixT = nullptr;
      float* dxp = nullptr;
      if (fold) {
        paT = (__nv_bfloat16*)takeq(ld * H * 2); giT = (__nv_bfloat16*)takeq(ld * 3 * H * 2);
        w0T = (__nv_bfloat16*)takeq((size_t)C * H * 2); wiT = (__nv_bfloat16*)takeq((size_t)C * 3 * H * 2);
        w0xT = (__nv_bfloat16*)takeq((size_t)P_OUT * H * 2); wixT = (__nv_bfloat16*)takeq((size_t)P_OUT * 3 * H * 2);
        dxp = (float*)takeq(ld * P_OUT * 4);
      }
      const int cur = nbt * 32;                  // column offset of slot t = 1
      const int Kc = nT * nbt * 32;
      // per-slot stride of the fp32 history is (stride / nbt) floats: slots (t,bt) are contiguous
      // gradient histories: the same pass returns the bias gradient (sum over slots t >= 1, i.e. s >= nbt)
      auto split = [&](Hist& h) { return split_hist_launch(h.src, h.stride / nbt, S, h.rows, h.hi, h.lo, stream, h.db, nbt); };
      if (fold) {
        if (p1) {
          // ---- phase 1: d cond on the tensor cores (single-pass bf16): contract the transposed dpa / dgi0 histories with the transposed
          // cond columns of W0 / W_ih0:  DCOND[(t,b)][c] = dpa^T W0[:, 1134+c] + dgi0^T W_ih0[:, H+1134+c]
          if ((rc = split(hs[3]))) return rc;
          if ((rc = split(hs[5]))) return rc;
          if ((rc = transpose_bf16_launch(hs[5].hi, H, (int)ld, ld, paT, H, stream))) return rc;
          if ((rc = transpose_bf16_launch(hs[3].hi, 3 * H, (int)ld, ld, giT, 3 * H, stream))) return rc;
          if ((rc = split_t_launch(a.W0 + P_IN, H, C, A, w0T, nullptr, H, stream))) return rc;
          if ((rc = split_t_launch(a.W_ih0 + H + P_IN, 3 * H, C, A + H, wiT, nullptr, 3 * H, stream))) return rc;
          float* out = bw.DCOND + (size_t)cur * C;
          if ((rc = tc_gemm_launch(Kc, C, H, paT + (size_t)cur * H, nullptr, H, w0T, nullptr, H, nullptr, out, C, 0, 0, stream))) return rc;
          if ((rc = tc_gemm_launch(Kc, C, 3 * H, giT + (size_t)cur * 3 * H, nullptr, 3 * H, wiT, nullptr, 3 * H, nullptr, out, C, 0, 1, stream))) return rc;
          dcond_scatter_kernel<<<592, 256, 0, stream>>>(a, g, bw.DCOND, bw.cse_din, b.dSpeech, b.dStyle, 1);
          count_launch();
          ZCHECK_LAUNCH();
        }
        dcond_rows = true;
        if (p2) {
          for (int hi_ : {1, 2, 4, 6, 7, 8, 9, 10}) if ((rc = split(hs[hi_]))) return rc;
          // the x_pose gradient of every step at once (transposed dpre_a / dgi0 histories from phase 1):
          //   DXP[(t,b)][n] = dpre_a(t)^T W0[:, n] + dgi0(t)^T W_ih0[:, H + n]      (n < 1131; modules.py:172-175 adjoint)
          // and the layer-2 / x_pose gradient history the weight gradients read (modules.py:713, :728 adjoints):
          //   DY[t][n][b] = out_std[n] (dY_ext[b][t][n] + DXP[(t+1,b)][n] / in_std[n] + [n < 6] dch(t)[b][n])
          if ((rc = split_t_launch(a.W0, H, P_OUT, A, w0xT, nullptr, H, stream))) return rc;
          if ((rc = split_t_launch(a.W_ih0 + H, 3 * H, P_OUT, A + H, wixT, nullptr, 3 * H, stream))) return rc;
          if ((rc = tc_gemm_launch(Kc, P_OUT, H, paT + (size_t)cur * H, nullptr, H, w0xT, nullptr, H, nullptr, dxp + (size_t)cur * P_OUT, P_OUT, 0, 0, stream))) return rc;
          if ((rc = tc_gemm_launch(Kc, P_OUT, 3 * H, giT + (size_t)cur * 3 * H, nullptr, 3 * H, wixT, nullptr, 3 * H, nullptr, dxp + (size_t)cur * P_OUT, P_OUT, 0, 1, stream))) return rc;
          dy_combine_kernel<<<dim3(T - 1, ceil_div(P_OUT, 64)), 256, 0, stream>>>(a, b.dY, dxp, bw.DCH, bw.DY);
          count_launch();
          ZCHECK_LAUNCH();
          if ((rc = split(hs[0]))) return rc;
        }
      } else {
        for (auto& h : hs) if ((rc = split(h))) return rc;
      }
      if (p2) {
        char* ws_p = (char*)(((uintptr_t)p + 255) & ~(uintptr_t)255);             // split-K partials behind the histories
        const size_t ws_bytes = (size_t)(scratch_base() + scratch_bytes() - ws_p);
        auto G = [&](const Hist& ga, int ga_off, int N, const Hist& xb, int xb_off, int K, float* dW, int ldw) {
          return tc_gemm_launch(N, K, Kc, ga.hi + ga_off, want_lo ? ga.lo + ga_off : nullptr, (int)ld,
                                xb.hi + xb_off, want_lo ? xb.lo + xb_off : nullptr, (int)ld, nullptr, dW, ldw, 0, 0, stream,
                                (float*)ws_p, ws_bytes);
        };
        const Hist &hDY = hs[0], &hGI1 = hs[1], &hGH1 = hs[2], &hGI0 = hs[3], &hGH0 = hs[4], &hPA = hs[5], &hH0 = hs[6], &hH1 = hs[7],
                   &hA = hs[8], &hXP = hs[9];
        if ((rc = G(hDY, cur, P_OUT, hH1, cur, H, b.dW2, H))) return rc;
        if ((rc = G(hGI1, cur, 3 * H, hH0, cur, H, b.dW_ih1, H))) return rc;
        if ((rc = G(hGH1, cur, 3 * H, hH1, 0, H, b.dW_hh1, H))) return rc;
        if ((rc = G(hGI0, cur, 3 * H, hA, cur, H + P_IN + C, b.dW_ih0, A + H))) return rc;     // [a | x_pose | cond] stacked
        if ((rc = G(hGH0, cur, 3 * H, hH0, 0, H, b.dW_hh0, H))) return rc;
        if ((rc = G(hPA, cur, H, hXP, cur, P_IN + C, b.dW0, A))) return rc;                    // [x_pose | cond] stacked
      }
      tc_done = true;
    } else {
      ZCHECK_ARG(!use_tc, "decoder bwd tc: scratch buffer too small for the batched gradient GEMMs (%zu bytes needed)", need + extra);
    }
  } else {
    ZCHECK_ARG(!use_tc, "decoder bwd tc: needs the tensor-core GEMM front end (a zeggs_ctx with scratch, gemm mode 1 or 2)");
  }
  if (fold) return ZEGGS_OK;                    // the folded path is complete (CellStateEncoder + scatter ran in phase 1)
#define WG(...) do { if (!tc_done) { rc = wgrad(__VA_ARGS__); if (rc) return rc; } } while (0)
#define RS(...) do { if (!tc_done) { rc = rowsum(__VA_ARGS__); if (rc) return rc; } } while (0)
  // layer2: dW2 = DY . H1[t]^T
  WG(bw.DY + sX, sX, (long long)K1P * 32, P_OUT, w.H1 + sH, sH, (long long)H * 32, H, nT, nbt, b.dW2, H, stream);
  RS(bw.DY + sX, sX, (long long)K1P * 32, P_OUT, nT, nbt, b.db2, stream);
  // GRU layer 1
  WG(bw.DGI1 + s3, s3, (long long)3 * H * 32, 3 * H, w.H0 + sH, sH, (long long)H * 32, H, nT, nbt, b.dW_ih1, H, stream);
  WG(bw.DGH1 + s3, s3, (long long)3 * H * 32, 3 * H, w.H1, sH, (long long)H * 32, H, nT, nbt, b.dW_hh1, H, stream);
  RS(bw.DGI1 + s3, s3, (long long)3 * H * 32, 3 * H, nT, nbt, b.db_ih1, stream);
  RS(bw.DGH1 + s3, s3, (long long)3 * H * 32, 3 * H, nT, nbt, b.db_hh1, stream);
  // GRU layer 0: input = [a | x_pose | cond]
  WG(bw.DGI0 + s3, s3, (long long)3 * H * 32, 3 * H, w.A + sH, sH, (long long)H * 32, H, nT, nbt, b.dW_ih0, A + H, stream);
  WG(bw.DGI0 + s3, s3, (long long)3 * H * 32, 3 * H, w.XP + sX, sX, (long long)K1P * 32, P_IN, nT, nbt, b.dW_ih0 + H, A + H, stream);
  WG(bw.DGI0 + s3, s3, (long long)3 * H * 32, 3 * H, bw.COND + sC, sC, (long long)C * 32, C, nT, nbt, b.dW_ih0 + H + P_IN, A + H, stream);
  WG(bw.DGH0 + s3, s3, (long long)3 * H * 32, 3 * H, w.H0, sH, (long long)H * 32, H, nT, nbt, b.dW_hh0, H, stream);
  RS(bw.DGI0 + s3, s3, (long long)3 * H * 32, 3 * H, nT, nbt, b.db_ih0, stream);
  RS(bw.DGH0 + s3, s3, (long long)3 * H * 32, 3 * H, nT, nbt, b.db_hh0, stream);
  // layer0
  WG(bw.DPA + sH, sH, (long long)H * 32, H, w.XP + sX, sX, (long long)K1P * 32, P_IN, nT, nbt, b.dW0, A, stream);
  WG(bw.DPA + sH, sH, (long long)H * 32, H, bw.COND + sC, sC, (long long)C * 32, C, nT, nbt, b.dW0 + P_IN, A, stream);
  RS(bw.DPA + sH, sH, (long long)H * 32, H, nT, nbt, b.db0, stream);
#undef WG
#undef RS
  // ---- d cond[t] = W0[:, 1134:]^T dpre_a + W_ih0[:, H+1134:]^T dgi0   (batched over slots t >= 1)
  if (!dcond_rows) {
    rc = sgemm_batched_launch(1, C, 32, H, a.W0 + P_IN, A, bw.DPA + sH, 32, nullptr, bw.DCOND + sC, 32, 0, 0, nT * nbt, 0, (long long)H * 32, (long long)C * 32, stream); if (rc) return rc;
    rc = sgemm_batched_launch(1, C, 32, 3 * H, a.W_ih0 + H + P_IN, A + H, bw.DGI0 + s3, 32, nullptr, bw.DCOND + sC, 32, 0, 1, nT * nbt, 0, (long long)3 * H * 32, (long long)C * 32, stream); if (rc) return rc;
  }
  if (cse_tail) { if ((rc = cse_backward())) return rc; }
  dcond_scatter_kernel<<<592, 256, 0, stream>>>(a, g, bw.DCOND, bw.cse_din, b.dSpeech, b.dStyle, dcond_rows ? 1 : 0);
  count_launch();
  ZCHECK_LAUNCH();
  return ZEGGS_OK;
}

}  // namespace zeggs
