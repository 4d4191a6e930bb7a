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

// CTA c's units are passes p of V = pass_units(U) units (one pass below U = 16); j(r) = cU + pV + r, R1P = film_rows(V) = R1 / (U/V):
// PB1[c][p][k<1136][R1P]  W2[k][j(r)]                       (x = dy, k = output channel)
// PB2[c][p][k<3H][2V]     r<V: W_ih1[k][j(r)]   else W_hh1[k][j(r-V)]
// PB3a[c][p][k<3H][2V]    r<V: W_ih0[k][j(r)]   else W_hh0[k][j(r-V)]
// PB3b[c][tile][k<3H][16] W_ih0[k][H + perm(c*rpcb + tile*16 + r)]
// PB4[c][tile][k<H][16]   W0[k][perm(c*rpcb + tile*16 + r)]
__global__ void pack_decoder_bwd_kernel(DecGeom g, BwdGeom bg, const float* __restrict__ W0, const float* __restrict__ Wih0,
                                        const float* __restrict__ Whh0, const float* __restrict__ Wih1,
                                        const float* __restrict__ Whh1, const float* __restrict__ W2, float* __restrict__ out) {
  const int H = g.H, U = g.U, A = g.A, V = pass_units(U), NP = U / V, R1P = bg.R1 / NP;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < bg.total; i += (size_t)gridDim.x * blockDim.x) {
    float v = 0.f;
    if (i < bg.off2) {
      size_t e = i;
      int r = e % R1P; e /= R1P;
      int k = e % K1P; e /= K1P;
      int p = e % NP, c = e / NP;
      if (r < V && k < P_OUT) v = W2[(size_t)k * H + c * U + p * V + r];
    } else if (i < bg.off3b) {
      const bool l0 = i >= bg.off3a;
      size_t e = i - (l0 ? bg.off3a : bg.off2);
      int r = e % (2 * V); e /= (2 * V);
      int k = e % (3 * H); e /= (3 * H);
      int p = e % NP, c = e / NP;
      const bool hh = r >= V;
      int j = c * U + p * V + (hh ? r - V : r);
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

// FILM: the FiLM decoder's BPTT.  B1 splits in two stages: B1a  dc = W3^T (dY_acc*sigma_out) -> d gamma/beta of layer2, dpre2 (DP2);
// B1b  dh1 = dh1_acc + Wm^T dpre2.  B3 takes the layer-0 modulation: d gamma/beta of layer0, dpre_a = da * gamma * ELU'.
// B1 / B1a / B2 / B3a run once per pass of V units, on the pass-major slices PB1 / PBm / PB2 / PB3a.
template <int U, bool FILM>
__global__ void __launch_bounds__(256, 1)
decoder_bwd_kernel(zeggs_decoder_fwd_args a, DecGeom g, BwdGeom bg, DecWs w, BwdWs bw, BwdArgsDev d, FilmDev f) {
  extern __shared__ __align__(16) float smem[];
  constexpr int V = pass_units(U), NP = U / V;
  constexpr int RT1 = film_rows(V) / 4;      // B1 tile rows / 4
  constexpr int RT2 = (2 * V) / 4;           // dual tiles
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
  const float* PB2 = d.packed + bg.off2 + (size_t)c * 3 * H * 2 * U;    // + p * 3H * 2V per pass
  const float* PB3a = d.packed + bg.off3a + (size_t)c * 3 * H * 2 * U;
  const float* PB3b = d.packed + bg.off3b + (size_t)c * bg.n4b * 3 * H * 16;
  const float* PB4 = d.packed + bg.off4 + (size_t)c * bg.n4b * H * 16;
  const float* PBm = d.packed + bg.total + (size_t)c * H * bg.R1;   // FiLM: PBm[c][p][k][r] = Wm[k][c*U + p*V + r]
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
    if constexpr (FILM) {
      // ---------------------------------------------------------- B1a (FiLM: layer3, modulation and ELU of layer2)
      for (int bt = 0; bt < nbt; ++bt)
      for (int p = 0; p < NP; ++p) {
        float acc[RT1][4];
        const float* x = bw.DY + t * actX + (size_t)bt * K1P * 32;
        skinny_gemm<RT1, false>(acc, PB1 + (size_t)p * K1P * 4 * RT1, x, x, K1P / 16, wstage);
        reduce_store<RT1>(acc, red);
        __syncthreads();
        for (int idx = tid; idx < V * 32; idx += 256) {
          const int b = idx & 31, j = c * U + p * V + (idx >> 5), bgl = bt * 32 + b;
          const float dc = red_sum<4 * RT1>(red, idx >> 5, b);
          const float e = f.E2[t * actH + ((size_t)bt * H + j) * 32 + b];
          float gm = 1.f;
          if (bgl < a.B) {
            const size_t row = ((size_t)bgl * T + t) * 4 * H;
            gm += f.GB[row + H + j];
            f.DGB[row + H + j] = dc * e;
            f.DGB[row + 3 * H + j] = dc;
          }
          f.DP2[t * actH + ((size_t)bt * H + j) * 32 + b] = dc * gm * (e > 0.f ? 1.f : e + 1.f);
        }
        __syncthreads();
      }
      if (!grid_sync(gb)) return;
    }
    // ------------------------------------------------------------ B1 (FiLM: B1b)
    for (int bt = 0; bt < nbt; ++bt)
    for (int p = 0; p < NP; ++p) {
      float acc[RT1][4];
      if constexpr (FILM) {
        const float* x = f.DP2 + t * actH + (size_t)bt * H * 32;
        skinny_gemm<RT1, false>(acc, PBm + (size_t)p * H * 4 * RT1, x, x, H / 16, wstage);
      } else {
        const float* x = bw.DY + t * actX + (size_t)bt * K1P * 32;
        skinny_gemm<RT1, false>(acc, PB1 + (size_t)p * K1P * 4 * RT1, x, x, K1P / 16, wstage);
      }
      reduce_store<RT1>(acc, red);
      __syncthreads();
      for (int idx = tid; idx < V * 32; idx += 256) {
        const int u = p * V + (idx >> 5), b = idx & 31, j = c * U + u;
        float* acc1 = bw.DH1 + ((size_t)bt * H + j) * 32 + b;
        float dh = red_sum<4 * RT1>(red, idx >> 5, b) + (t == T - 1 ? 0.f : *acc1);
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
    for (int bt = 0; bt < nbt; ++bt)
    for (int p = 0; p < NP; ++p) {
      float acc[RT2][4];
      const float* xa = bw.DGI1 + t * act3 + (size_t)bt * 3 * H * 32;
      const float* xb = bw.DGH1 + t * act3 + (size_t)bt * 3 * H * 32;
      skinny_gemm<RT2, true>(acc, PB2 + (size_t)p * 3 * H * 2 * V, xa, xb, 3 * H / 16, wstage);
      reduce_store<RT2>(acc, red);
      __syncthreads();
      for (int idx = tid; idx < V * 32; idx += 256) {
        const int u = p * V + (idx >> 5), v = idx >> 5, b = idx & 31, j = c * U + u;
        float* acc0 = bw.DH0 + ((size_t)bt * H + j) * 32 + b;
        float dh = red_sum<2 * V>(red, v, b) + (t == T - 1 ? 0.f : *acc0);
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
        bw.DH1[((size_t)bt * H + j) * 32 + b] = red_sum<2 * V>(red, V + v, b) + dhz1[(bt * U + u) * 32 + b];
      }
      __syncthreads();
    }
    if (!grid_sync(gb)) return;
    // ------------------------------------------------------------ B3
    for (int bt = 0; bt < nbt; ++bt) {
      for (int p = 0; p < NP; ++p) {
        float acc[RT2][4];
        const float* xa = bw.DGI0 + t * act3 + (size_t)bt * 3 * H * 32;
        const float* xb = bw.DGH0 + t * act3 + (size_t)bt * 3 * H * 32;
        skinny_gemm<RT2, true>(acc, PB3a + (size_t)p * 3 * H * 2 * V, xa, xb, 3 * H / 16, wstage);
        reduce_store<RT2>(acc, red);
        __syncthreads();
        for (int idx = tid; idx < V * 32; idx += 256) {
          const int u = p * V + (idx >> 5), v = idx >> 5, b = idx & 31, j = c * U + u;
          if constexpr (FILM) {
            const float da = red_sum<2 * V>(red, v, b);
            const int bgl = bt * 32 + b;
            const float e = f.E0[t * actH + ((size_t)bt * H + j) * 32 + b];
            float gm = 1.f;
            if (bgl < a.B) {
              const size_t row = ((size_t)bgl * T + t) * 4 * H;
              gm += f.GB[row + j];
              f.DGB[row + j] = da * e;
              f.DGB[row + 2 * H + j] = da;
            }
            bw.DPA[t * actH + ((size_t)bt * H + j) * 32 + b] = da * gm * (e > 0.f ? 1.f : e + 1.f);
          } else {
            float av = w.A[t * actH + ((size_t)bt * H + j) * 32 + b];
            float da = red_sum<2 * V>(red, v, b);
            bw.DPA[t * actH + ((size_t)bt * H + j) * 32 + b] = da * (av > 0.f ? 1.f : av + 1.f);   // ELU'(pre) = a+1 for pre<=0
          }
          bw.DH0[((size_t)bt * H + j) * 32 + b] = red_sum<2 * V>(red, V + v, b) + dhz0[(bt * U + u) * 32 + b];
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
  if (!fp32_hidden_ok(H)) return 0;
  DecGeom g = make_geom(1, H, S, Z);
  return make_bgeom(g).total * sizeof(float);
}

// the transposed slices of geometry g: the whole pack of the normal decoder, the front of the FiLM decoder's
static int pack_bwd_slices(const zeggs_decoder_fwd_args& a, const DecGeom& g, float* packed, cudaStream_t stream) {
  pack_decoder_bwd_kernel<<<592, 256, 0, stream>>>(g, make_bgeom(g), a.W0, a.W_ih0, a.W_hh0, a.W_ih1, a.W_hh1, a.W2, packed);
  LAUNCH_OK();
  return ZEGGS_OK;
}

extern "C" int zeggs_decoder_pack_weights_bwd(const zeggs_decoder_fwd_args* a, float* packed, void* stream) {
  CtxScope ctx_scope(a ? a->ctx : nullptr);
  ZCHECK_ARG(a && packed && fp32_hidden_ok(a->H), "decoder bwd pack: bad arguments");
  return pack_bwd_slices(*a, make_geom(a->B, a->H, a->S, a->Z), packed, (cudaStream_t)stream);
}

extern "C" size_t zeggs_decoder_bwd_workspace_bytes(int B, int T, int H, int S, int Z) {
  if (!fp32_hidden_ok(H) || B < 1 || T < 1) return 0;
  DecGeom g = make_geom(B, H, S, Z);
  return make_bws(nullptr, g, T).bytes;
}

// dynamic shared memory per CTA of the BPTT recurrence: it grows with the 32-sample batch tiles, which bounds the batch of one call
static size_t bwd_smem_bytes(const DecGeom& g, const BwdGeom& bg, int nbt) {
  return (size_t)(8 * 2 * SkinnyCfg<4>::STG + 8 * 16 * 32 + 2 * nbt * g.U * 32 + nbt * bg.n4b * 16 * 32 + nbt * 9 * 32 + nbt * 7 * 32) *
         sizeof(float);
}

static int check_bwd_batch(const DecGeom& g, const BwdGeom& bg) {
  DeviceLimits lim;
  RC(device_limits(&lim));
  auto smem_of = [&](int nbt) { return bwd_smem_bytes(g, bg, nbt); };
  ZCHECK_ARG(smem_of(g.nbt) <= lim.smem_optin, "decoder bwd: batch %d needs %zu bytes of shared memory per CTA at hidden size %d (%zu "
             "available): at most %d samples per call", g.B, smem_of(g.nbt), g.H, lim.smem_optin, 32 * max_batch_tiles(smem_of, lim.smem_optin));
  return ZEGGS_OK;
}

// the BPTT recurrence of the fp32 engine, normal and FiLM.  It refuses a batch its shared memory cannot hold before it enqueues anything.
template <bool FILM>
static int bptt_fp32(const zeggs_decoder_fwd_args& a, const zeggs_decoder_bwd_args& b, const DecGeom& g, const DecWs& w, const BwdWs& bw,
                     const FilmDev& f, cudaStream_t stream) {
  const BwdGeom bg = make_bgeom(g);
  RC(check_bwd_batch(g, bg));
  ZCHECK_CUDA(cudaMemsetAsync(bw.bar, 0, 256, stream));
  ZCHECK_CUDA(cudaMemsetAsync(bw.DY, 0, (size_t)a.T * g.nbt * K1P * 32 * sizeof(float), stream));
  // the FiLM recurrence writes the rows t >= 1 of DGB; the rows t = 0 stay zero
  if constexpr (FILM) ZCHECK_CUDA(cudaMemsetAsync(f.DGB, 0, (size_t)a.B * a.T * 4 * a.H * sizeof(float), stream));
  BwdArgsDev d; d.dY = b.dY; d.dRootPos = b.dRootPos; d.dRootRot = b.dRootRot; d.packed = b.packed_bwd;
  ScopedTimer tm("decoder_bwd", stream);
  return dispatch_units(g.U, [&](auto u) {
    return launch_persistent(decoder_bwd_kernel<u, FILM>, g.G, 256, bwd_smem_bytes(g, bg, g.nbt), 1, stream, a, g, bg, w, bw, d, f);
  });
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

WgradHists wgrad_hists(const zeggs_decoder_fwd_args& a, const zeggs_decoder_bwd_args& b, const DecGeom& g, const DecWs& w,
                       const BwdWs& bw, bool want_lo) {
  const int H = a.H, nbt = g.nbt, C = a.S + a.Z;
  const long long sH = (long long)nbt * H * 32, s3 = (long long)nbt * 3 * H * 32, sX = (long long)nbt * K1P * 32, sC = (long long)nbt * C * 32;
  WgradHists hs = {{
      {bw.DY, sX, P_OUT, nullptr, nullptr, b.db2}, {bw.DGI1, s3, 3 * H, nullptr, nullptr, b.db_ih1}, {bw.DGH1, s3, 3 * H, nullptr, nullptr, b.db_hh1},
      {bw.DGI0, s3, 3 * H, nullptr, nullptr, b.db_ih0}, {bw.DGH0, s3, 3 * H, nullptr, nullptr, b.db_hh0}, {bw.DPA, sH, H, nullptr, nullptr, b.db0},
      {w.H0, sH, H, nullptr, nullptr, nullptr}, {w.H1, sH, H, nullptr, nullptr, nullptr}, {w.A, sH, H, nullptr, nullptr, nullptr},
      {w.XP, sX, P_IN, nullptr, nullptr, nullptr}, {bw.COND, sC, C, nullptr, nullptr, nullptr}}};
  hs.slots = a.T * nbt;
  hs.nbt = nbt;
  hs.ld = (size_t)hs.slots * 32;
  Arena sc{scratch_base(), 0, 1};   // rows of (ld * 2) bytes: no rounding between the copies, they stack into one operand
  for (auto& h : hs.h) h.hi = (__nv_bfloat16*)sc.bytes((size_t)h.rows * hs.ld * 2);
  if (want_lo) for (auto& h : hs.h) h.lo = (__nv_bfloat16*)sc.bytes((size_t)h.rows * hs.ld * 2);
  hs.bytes = sc.off;
  return hs;
}

int split_hist(const WgradHists& hs, int i, cudaStream_t stream) {
  // per-slot stride of the fp32 history is (stride / nbt) floats: slots (t,bt) are contiguous.  The bias gradient is the sum over
  // slots t >= 1, i.e. s >= nbt
  const WgradHist& h = hs.h[i];
  return split_hist_launch(h.src, h.stride / hs.nbt, hs.slots, h.rows, h.hi, h.lo, stream, h.db, hs.nbt);
}

int wgrad_gemms(const zeggs_decoder_fwd_args& a, const zeggs_decoder_bwd_args& b, const DecGeom& g, const WgradHists& hs, bool want_lo,
                Arena tail, cudaStream_t stream) {
  const int H = a.H, A = g.A, C = a.S + a.Z;
  const int cur = g.nbt * 32;                       // column offset of slot t = 1
  const int Kc = (a.T - 1) * g.nbt * 32;
  // the histories may end within 255 bytes of the scratch end: the aligned tail then lies past it and there is no split-K room
  float* const ws = (float*)tail.align(256).here();
  const size_t ws_bytes = tail.rest(scratch_bytes());
  auto G = [&](int ga, int ga_off, int N, int xb, int xb_off, int K, float* dW, int ldw) {
    const WgradHist &x = hs.h[ga], &y = hs.h[xb];
    return tc_gemm_launch(N, K, Kc, x.hi + ga_off, want_lo ? x.lo + ga_off : nullptr, (int)hs.ld,
                          y.hi + xb_off, want_lo ? y.lo + xb_off : nullptr, (int)hs.ld, nullptr, dW, ldw, 0, 0, stream,
                          ws, ws_bytes);
  };
  int rc;
  if ((rc = G(HDY, cur, P_OUT, HH1, cur, H, b.dW2, H))) return rc;
  if ((rc = G(HGI1, cur, 3 * H, HH0, cur, H, b.dW_ih1, H))) return rc;
  if ((rc = G(HGH1, cur, 3 * H, HH1, 0, H, b.dW_hh1, H))) return rc;
  if ((rc = G(HGI0, cur, 3 * H, HA, cur, H + P_IN + C, b.dW_ih0, A + H))) return rc;     // [a | x_pose | cond] stacked
  if ((rc = G(HGH0, cur, 3 * H, HH0, 0, H, b.dW_hh0, H))) return rc;
  return G(HPA, cur, H, HXP, cur, P_IN + C, b.dW0, A);                                    // [x_pose | cond] stacked
}

int cond_kmajor(const zeggs_decoder_fwd_args& a, const DecGeom& g, const BwdWs& bw, cudaStream_t stream) {
  cond_kmajor_kernel<<<592, 256, 0, stream>>>(a, g, bw.COND);
  count_launch();
  ZCHECK_LAUNCH();
  return ZEGGS_OK;
}

int cse_backward(const zeggs_decoder_fwd_args& a, const zeggs_decoder_bwd_args& b, const DecWs& w, const BwdWs& bw, cudaStream_t stream) {
  const int H = a.H, Kin = P_IN + a.Z;
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
}

int dy_combine(const zeggs_decoder_fwd_args& a, const zeggs_decoder_bwd_args& b, const float* dxp, const BwdWs& bw, cudaStream_t stream) {
  dy_combine_kernel<<<dim3(a.T - 1, ceil_div(P_OUT, 64)), 256, 0, stream>>>(a, b.dY, dxp, bw.DCH, bw.DY);
  count_launch();
  ZCHECK_LAUNCH();
  return ZEGGS_OK;
}

int dcond_scatter(const zeggs_decoder_fwd_args& a, const zeggs_decoder_bwd_args& b, const DecGeom& g, const BwdWs& bw, int rows,
                  cudaStream_t stream) {
  dcond_scatter_kernel<<<592, 256, 0, stream>>>(a, g, bw.DCOND, bw.cse_din, b.dSpeech, b.dStyle, rows);
  count_launch();
  ZCHECK_LAUNCH();
  return ZEGGS_OK;
}

// SIMT weight gradients over the k-major fp32 histories (slots t >= 1); l2in: the history of the output layer's input (h1, or the FiLM
// decoder's modulated layer-2 output).  The conditioning columns are those of `a` (S + Z, or S alone for the FiLM decoder).
static int wgrad_simt(const zeggs_decoder_fwd_args& a, const zeggs_decoder_bwd_args& b, const DecGeom& g, const DecWs& w, const BwdWs& bw,
                      const float* l2in, cudaStream_t stream) {
  const int H = a.H, nbt = g.nbt, C = a.S + a.Z, A = g.A, nT = a.T - 1;
  const long long sH = (long long)nbt * H * 32, s3 = (long long)nbt * 3 * H * 32, sX = (long long)nbt * K1P * 32, sC = (long long)nbt * C * 32;
  int rc;
  // output layer: dW2 = DY . l2in[t]^T
  if ((rc = wgrad(bw.DY + sX, sX, (long long)K1P * 32, P_OUT, l2in + sH, sH, (long long)H * 32, H, nT, nbt, b.dW2, H, stream))) return rc;
  if ((rc = rowsum(bw.DY + sX, sX, (long long)K1P * 32, P_OUT, nT, nbt, b.db2, stream))) return rc;
  // GRU layer 1
  if ((rc = wgrad(bw.DGI1 + s3, s3, (long long)3 * H * 32, 3 * H, w.H0 + sH, sH, (long long)H * 32, H, nT, nbt, b.dW_ih1, H, stream))) return rc;
  if ((rc = wgrad(bw.DGH1 + s3, s3, (long long)3 * H * 32, 3 * H, w.H1, sH, (long long)H * 32, H, nT, nbt, b.dW_hh1, H, stream))) return rc;
  if ((rc = rowsum(bw.DGI1 + s3, s3, (long long)3 * H * 32, 3 * H, nT, nbt, b.db_ih1, stream))) return rc;
  if ((rc = rowsum(bw.DGH1 + s3, s3, (long long)3 * H * 32, 3 * H, nT, nbt, b.db_hh1, stream))) return rc;
  // GRU layer 0: input = [a | x_pose | cond]
  if ((rc = wgrad(bw.DGI0 + s3, s3, (long long)3 * H * 32, 3 * H, w.A + sH, sH, (long long)H * 32, H, nT, nbt, b.dW_ih0, A + H, stream))) return rc;
  if ((rc = wgrad(bw.DGI0 + s3, s3, (long long)3 * H * 32, 3 * H, w.XP + sX, sX, (long long)K1P * 32, P_IN, nT, nbt, b.dW_ih0 + H, A + H, stream))) return rc;
  if ((rc = wgrad(bw.DGI0 + s3, s3, (long long)3 * H * 32, 3 * H, bw.COND + sC, sC, (long long)C * 32, C, nT, nbt, b.dW_ih0 + H + P_IN, A + H, stream))) return rc;
  if ((rc = wgrad(bw.DGH0 + s3, s3, (long long)3 * H * 32, 3 * H, w.H0, sH, (long long)H * 32, H, nT, nbt, b.dW_hh0, H, stream))) return rc;
  if ((rc = rowsum(bw.DGI0 + s3, s3, (long long)3 * H * 32, 3 * H, nT, nbt, b.db_ih0, stream))) return rc;
  if ((rc = rowsum(bw.DGH0 + s3, s3, (long long)3 * H * 32, 3 * H, nT, nbt, b.db_hh0, stream))) return rc;
  // layer0
  if ((rc = wgrad(bw.DPA + sH, sH, (long long)H * 32, H, w.XP + sX, sX, (long long)K1P * 32, P_IN, nT, nbt, b.dW0, A, stream))) return rc;
  if ((rc = wgrad(bw.DPA + sH, sH, (long long)H * 32, H, bw.COND + sC, sC, (long long)C * 32, C, nT, nbt, b.dW0 + P_IN, A, stream))) return rc;
  if ((rc = rowsum(bw.DPA + sH, sH, (long long)H * 32, H, nT, nbt, b.db0, stream))) return rc;
  return ZEGGS_OK;
}

// d cond[t] = W0[:, 1134:]^T dpre_a + W_ih0[:, H+1134:]^T dgi0   (batched over slots t >= 1)
static int dcond_gemms(const zeggs_decoder_fwd_args& a, const DecGeom& g, const BwdWs& bw, cudaStream_t stream) {
  const int H = a.H, nbt = g.nbt, C = a.S + a.Z, A = g.A, nT = a.T - 1;
  const long long sH = (long long)nbt * H * 32, s3 = (long long)nbt * 3 * H * 32, sC = (long long)nbt * C * 32;
  int rc = sgemm_batched_launch(1, C, 32, H, a.W0 + P_IN, A, bw.DPA + sH, 32, nullptr, bw.DCOND + sC, 32, 0, 0, nT * nbt, 0, (long long)H * 32, (long long)C * 32, stream); if (rc) return rc;
  return sgemm_batched_launch(1, C, 32, 3 * H, a.W_ih0 + H + P_IN, A + H, bw.DGI0 + s3, 32, nullptr, bw.DCOND + sC, 32, 0, 1, nT * nbt, 0, (long long)3 * H * 32, (long long)C * 32, stream);
}

// fp32 engine: the SIMT BPTT recurrence, then the weight gradients, d cond, the CellStateEncoder backward and the dSpeech / dStyle
// scatter.  It does all of it in phase 1 (or 0) and nothing in phase 2.
static int decoder_window_bwd_fp32(const zeggs_decoder_fwd_args& a, const zeggs_decoder_bwd_args& b, const DecGeom& g, const DecWs& w,
                                   const BwdWs& bw, cudaStream_t stream) {
  ZCHECK_ARG(b.packed_bwd, "decoder bwd: packed_bwd missing");
  if (b.phase == 2) return ZEGGS_OK;
  int rc;
  if ((rc = bptt_fp32<false>(a, b, g, w, bw, FilmDev{}, stream))) return rc;
  ScopedTimer tm("decoder_wgrad", stream);
  if ((rc = cond_kmajor(a, g, bw, stream))) return rc;
  // weight gradients: tensor-core GEMMs over split-bf16 copies of the histories when those fit the scratch buffer (a second, lo pass
  // in GEMM mode 1 for ~fp32 accuracy), the SIMT k-major kernels otherwise
  const bool want_lo = gemm_mode() == 1;
  const WgradHists hs = wgrad_hists(a, b, g, w, bw, want_lo);
  if (gemm_mode() == 1 && scratch_base() != nullptr && hs.bytes <= scratch_bytes()) {
    for (int i = 0; i < NHIST; ++i) if ((rc = split_hist(hs, i, stream))) return rc;
    if ((rc = wgrad_gemms(a, b, g, hs, want_lo, Arena{scratch_base(), hs.bytes, 1}, stream))) return rc;
  } else {
    if ((rc = wgrad_simt(a, b, g, w, bw, w.H1, stream))) return rc;
  }
  if ((rc = dcond_gemms(a, g, bw, stream))) return rc;
  if ((rc = cse_backward(a, b, w, bw, stream))) return rc;
  return dcond_scatter(a, b, g, bw, 0, stream);
}

// a one-frame window outputs the given first pose (modules.py:72-79): no weight and no conditioning input reaches it, so every
// gradient is zero (the reference's autograd gives the same).  A: input width of layer0.
static int zero_window_grads(const zeggs_decoder_fwd_args& a, const zeggs_decoder_bwd_args& b, size_t A, cudaStream_t stream) {
  const size_t H = a.H, Kin = P_IN + a.Z;
  const struct { float* p; size_t n; } zero[] = {
      {b.dW0, H * A}, {b.db0, H}, {b.dW_ih0, 3 * H * (A + H)}, {b.db_ih0, 3 * H}, {b.dW_hh0, 3 * H * H}, {b.db_hh0, 3 * H},
      {b.dW_ih1, 3 * H * H}, {b.db_ih1, 3 * H}, {b.dW_hh1, 3 * H * H}, {b.db_hh1, 3 * H}, {b.dW2, (size_t)P_OUT * H}, {b.db2, (size_t)P_OUT},
      {b.dWc0, H * Kin}, {b.dbc0, H}, {b.dWc1, H * H}, {b.dbc1, H}, {b.dWc2, 2 * H * H}, {b.dbc2, 2 * H},
      {b.dSpeech, (size_t)a.B * a.S}, {b.dStyle, (size_t)a.B * a.Z}};
  for (const auto& z : zero)
    if (z.p) ZCHECK_CUDA(cudaMemsetAsync(z.p, 0, z.n * sizeof(float), stream));
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
  if (a.T == 1) return b.phase == 2 ? ZEGGS_OK : zero_window_grads(a, b, P_IN + a.S + a.Z, stream);
  DecGeom g = make_geom(a.B, a.H, a.S, a.Z);
  DecWs w = make_ws(a.workspace, g, a.T, 1);
  BwdWs bw = make_bws(b.workspace, g, a.T);
  ZCHECK_ARG(b.workspace && b.workspace_bytes >= bw.bytes, "decoder bwd: workspace too small (%zu < %zu)", b.workspace_bytes, bw.bytes);
  // a tensor-core forward with no BPTT pack (packed_bwd_tc == NULL) takes the fp32 backward
  if (a.engine == 1 && b.packed_bwd_tc) return decoder_window_bwd_tc(a, b, g, w, bw, stream);
  return decoder_window_bwd_fp32(a, b, g, w, bw, stream);
}


// ------------------------------------------------------------------ FiLM decoder (fp32 engine)
// PBm[c][p][k][r] = Wm[k][c*U + p*V + r] (r < V, zero up to R1P = R1 / (U/V)), behind the normal decoder's transposed slices
__global__ void pack_film_bwd_kernel(DecGeom g, int R1, const float* __restrict__ Wm, float* __restrict__ out) {
  const int H = g.H, U = g.U, V = pass_units(U), R1P = R1 / (U / V);
  const size_t total = (size_t)g.G * H * R1;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int r = i % R1P, k = (i / R1P) % H, cp = i / ((size_t)R1P * H);   // cp = c * (U / V) + p
    out[i] = r < V ? Wm[(size_t)k * H + cp * V + r] : 0.f;
  }
}

// out[c] = sum over rows of x[r][c] (row stride ld)
__global__ void colsum_ld_kernel(const float* __restrict__ x, int rows, int cols, int ld, float* __restrict__ out) {
  int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= cols) return;
  float s = 0.f;
  for (int r = 0; r < rows; ++r) s += x[(size_t)r * ld + c];
  out[c] = s;
}

// dStyle[b][0][:] += the CellStateEncoder's input gradient of the style columns (frame 0 has no FiLM term)
__global__ void film_style0_kernel(int B, int T, int Z, const float* __restrict__ cse_din, float* __restrict__ dStyle) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * Z) return;
  int b = i / Z, z = i % Z;
  dStyle[(size_t)b * T * Z + z] += cse_din[(size_t)b * (P_IN + Z) + P_IN + z];
}

static size_t film_bwd_extra_floats(const DecGeom& g) { return (size_t)g.G * g.H * make_bgeom(g).R1; }

extern "C" size_t zeggs_decoder_packed_bwd_film_bytes(int H, int S, int Z) {
  if (!fp32_hidden_ok(H)) return 0;
  DecGeom g = make_film_geom(1, H, S, Z);
  return (make_bgeom(g).total + film_bwd_extra_floats(g)) * sizeof(float);
}

extern "C" int zeggs_decoder_pack_weights_bwd_film(const zeggs_decoder_film_fwd_args* f, float* packed, void* stream_) {
  CtxScope ctx_scope(f ? f->dec.ctx : nullptr);
  ZCHECK_ARG(f && packed && f->Wm && fp32_hidden_ok(f->dec.H), "film decoder bwd pack: bad arguments");
  const zeggs_decoder_fwd_args& a = f->dec;
  DecGeom g = make_film_geom(a.B, a.H, a.S, a.Z);
  BwdGeom bg = make_bgeom(g);
  cudaStream_t stream = (cudaStream_t)stream_;
  int rc = pack_bwd_slices(a, g, packed, stream); if (rc) return rc;
  pack_film_bwd_kernel<<<264, 256, 0, stream>>>(g, bg.R1, f->Wm, packed + bg.total);
  LAUNCH_OK();
  return ZEGGS_OK;
}

// backward workspace: the normal decoder's carve-up followed by DGB [B*T][4H] and DP2 [T][nbt][H][32]
static size_t film_bwd_ws(void* base, const DecGeom& g, int T, FilmDev& f) {
  Arena a{(char*)base, make_bws(nullptr, g, T).bytes};
  f.DGB = a.take((size_t)g.B * T * 4 * g.H);
  f.DP2 = a.take((size_t)T * g.nbt * g.H * 32);
  return a.off;
}

extern "C" size_t zeggs_decoder_film_bwd_workspace_bytes(int B, int T, int H, int S, int Z) {
  if (!fp32_hidden_ok(H) || B < 1 || T < 1) return 0;
  FilmDev f = {};
  return film_bwd_ws(nullptr, make_film_geom(B, H, S, Z), T, f);
}

extern "C" int zeggs_decoder_film_window_bwd(const zeggs_decoder_film_fwd_args* fp, const zeggs_decoder_film_bwd_args* bp, void* stream_) {
  CtxScope ctx_scope(fp ? fp->dec.ctx : nullptr);
  ZCHECK_ARG(fp && bp, "film decoder bwd: null args");
  const zeggs_decoder_fwd_args& a = fp->dec;
  const zeggs_decoder_bwd_args& b = bp->dec;
  cudaStream_t stream = (cudaStream_t)stream_;
  ZCHECK_ARG(a.save_for_backward && a.workspace, "film decoder bwd: forward must have run with save_for_backward=1");
  ZCHECK_ARG(a.T >= 1 && b.phase >= 0 && b.phase <= 2, "film decoder bwd: bad T=%d / phase=%d", a.T, b.phase);
  ZCHECK_SUPPORTED(a.engine == 0, "film decoder bwd: only the fp32 engine (engine 0)");
  ZCHECK_ARG(b.packed_bwd, "film decoder bwd: packed_bwd missing (call zeggs_decoder_pack_weights_bwd_film)");
  if (b.phase == 2) return ZEGGS_OK;
  const int H = a.H, T = a.T, Z = a.Z;
  if (T == 1) {
    int rc = zero_window_grads(a, b, P_IN + a.S, stream); if (rc) return rc;
    const struct { float* p; size_t n; } zero[] = {{bp->dWm, (size_t)H * H}, {bp->dbm, (size_t)H}, {bp->dWg, (size_t)2 * H * Z},
                                                   {bp->dbg, (size_t)2 * H}, {bp->dWb, (size_t)2 * H * Z}, {bp->dbb, (size_t)2 * H}};
    for (const auto& z : zero)
      if (z.p) ZCHECK_CUDA(cudaMemsetAsync(z.p, 0, z.n * sizeof(float), stream));
    return ZEGGS_OK;
  }
  DecGeom g = make_film_geom(a.B, H, a.S, Z);
  DecWs w = make_ws(a.workspace, g, T, 1);
  size_t fwd_bytes = 0;
  FilmDev f = make_film_ws(a.workspace, w, g, T, &fwd_bytes);
  BwdWs bw = make_bws(b.workspace, g, T);
  const size_t need = film_bwd_ws(b.workspace, g, T, f);
  ZCHECK_ARG(a.workspace_bytes >= fwd_bytes, "film decoder bwd: forward workspace too small (%zu < %zu)", a.workspace_bytes, fwd_bytes);
  ZCHECK_ARG(b.workspace && b.workspace_bytes >= need, "film decoder bwd: workspace too small (%zu < %zu)", b.workspace_bytes, need);
  const int nbt = g.nbt, BT = a.B * T;
  int rc;
  if ((rc = bptt_fp32<true>(a, b, g, w, bw, f, stream))) return rc;
  ScopedTimer tm("decoder_wgrad", stream);
  // the recurrence's conditioning input is the speech alone: the normal decoder's host steps with no style columns
  zeggs_decoder_fwd_args as = a;
  as.Z = 0;
  if ((rc = cond_kmajor(as, g, bw, stream))) return rc;
  if ((rc = wgrad_simt(as, b, g, w, bw, f.C2, stream))) return rc;
  const long long sH = (long long)nbt * H * 32;
  if ((rc = wgrad(f.DP2 + sH, sH, (long long)H * 32, H, w.H1 + sH, sH, (long long)H * 32, H, T - 1, nbt, bp->dWm, H, stream))) return rc;
  if ((rc = rowsum(f.DP2 + sH, sH, (long long)H * 32, H, T - 1, nbt, bp->dbm, stream))) return rc;
  if ((rc = dcond_gemms(as, g, bw, stream))) return rc;
  if ((rc = cse_backward(a, b, w, bw, stream))) return rc;
  if ((rc = dcond_scatter(as, b, g, bw, 0, stream))) return rc;
  // the predictors (modules.py:215-217): dW = dGB^T style, db = column sums, dStyle = dG Wg + dBe Wb (+ the CellStateEncoder's part)
  rc = gemm_f32_auto(1, 2 * H, Z, BT, f.DGB, 4 * H, a.style, Z, nullptr, bp->dWg, Z, 0, 0, stream); if (rc) return rc;
  rc = gemm_f32_auto(1, 2 * H, Z, BT, f.DGB + 2 * H, 4 * H, a.style, Z, nullptr, bp->dWb, Z, 0, 0, stream); if (rc) return rc;
  colsum_ld_kernel<<<ceil_div(2 * H, 256), 256, 0, stream>>>(f.DGB, BT, 2 * H, 4 * H, bp->dbg);
  count_launch();
  colsum_ld_kernel<<<ceil_div(2 * H, 256), 256, 0, stream>>>(f.DGB + 2 * H, BT, 2 * H, 4 * H, bp->dbb);
  count_launch();
  ZCHECK_LAUNCH();
  if (b.dStyle) {
    rc = gemm_f32_auto(2, BT, Z, 2 * H, f.DGB, 4 * H, fp->Wg, Z, nullptr, b.dStyle, Z, 0, 0, stream); if (rc) return rc;
    rc = gemm_f32_auto(2, BT, Z, 2 * H, f.DGB + 2 * H, 4 * H, fp->Wb, Z, nullptr, b.dStyle, Z, 0, 1, stream); if (rc) return rc;
    film_style0_kernel<<<ceil_div(a.B * Z, 256), 256, 0, stream>>>(a.B, T, Z, bw.cse_din, b.dStyle);
    count_launch();
    ZCHECK_LAUNCH();
  }
  return ZEGGS_OK;
}

}  // namespace zeggs
