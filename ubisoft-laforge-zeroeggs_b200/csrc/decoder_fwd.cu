// Decoder window forward: CellStateEncoder + (T-1) autoregressive GRU steps in ONE persistent
// cooperative kernel.  Replaces Decoder.forward (ZEGGS/modules.py:47-162), RecurrentDecoderNormal
// (:165-185), CellStateEncoder (:230-243), vectorize_input (:677-713), devectorize_output (:716-742).
//
// Partitioning: G = H/U CTAs, CTA c owns hidden units [c*U, (c+1)*U) of layer0 / GRU0 / GRU1 and
// ceil(1131/G) rows of layer2.  Every step is 4 weight-stationary "skinny GEMM" stages separated by a
// grid barrier; each CTA streams its own pre-packed k-major weight slice (L2 resident) and the
// k-major activation vector of the previous stage:
//   S1  x_pose(t)            -> a(t) = ELU(W0p x + S0[t]),  gi0p = W_ih0[:,pose] x + S1[t]
//   S2  a(t), h0(t-1)        -> h0(t)   (GRU layer 0; r,z,n with b_hn inside r*(.))
//   S3  h0(t), h1(t-1)       -> h1(t)   (GRU layer 1)
//   S4  h1(t)                -> y(t) = W2 h1 + b2 -> de-normalise -> pose(t), root integration,
//                               x_pose(t+1) = normalise(pose(t), gaze(t+1))
// The speech/style columns of W0 / W_ih0 do not depend on the recurrence and are hoisted out of the
// time loop into one batched pre-pass (S0/S1 above).
#include "decoder_common.cuh"

namespace zeggs {

// ------------------------------------------------------------------ weight packing
// CTA c's units are passes p of V = pass_units(U) units each (one pass below U = 16), unit j = c*U + p*V + r%V:
// P1[c][p][k][r]  r in [0,4V): g=r/V (0: layer0, 1..3: W_ih0 gate g-1), k over pose cols
// P2[c][p][k][r]  r in [0,6V): r<3V: W_ih0[g*H+j][k] (hidden cols), else W_hh0[g*H+j][k]
// P3[c][p][k][r]  same with W_ih1 / W_hh1
// P4[c][tile][k][16]  W2 rows c*rpc + tile*16 + r
__global__ void pack_decoder_kernel(DecGeom g, const float* __restrict__ W0, const float* __restrict__ Wih0,
                                    const float* __restrict__ Whh0, const float* __restrict__ Wih1,
                                    const float* __restrict__ Whh1, const float* __restrict__ W2,
                                    float* __restrict__ out) {
  const size_t total = g.packed_floats();
  const int H = g.H, U = g.U, A = g.A, V = pass_units(U), NP = U / V;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    float v = 0.f;
    if (i < g.off_p2()) {
      size_t e = i;
      int r = e % (4 * V); e /= (4 * V);
      int k = e % K1P; e /= K1P;
      int p = e % NP, c = e / NP;
      int gi = r / V, j = c * U + p * V + r % V;
      if (k < P_IN) v = (gi == 0) ? W0[(size_t)j * A + k] : Wih0[(size_t)((gi - 1) * H + j) * (A + H) + H + k];
    } else if (i < g.off_p4()) {
      const bool l1 = i >= g.off_p3();
      size_t e = i - (l1 ? g.off_p3() : g.off_p2());
      int r = e % (6 * V); e /= (6 * V);
      int k = e % H; e /= H;
      int p = e % NP, c = e / NP;
      const bool hh = r >= 3 * V;
      int rr = hh ? r - 3 * V : r;
      int gi = rr / V, j = c * U + p * V + rr % V;
      if (!l1) v = hh ? Whh0[(size_t)(gi * H + j) * H + k] : Wih0[(size_t)(gi * H + j) * (A + H) + k];
      else     v = hh ? Whh1[(size_t)(gi * H + j) * H + k] : Wih1[(size_t)(gi * H + j) * H + k];
    } else {
      size_t e = i - g.off_p4();
      int r = e % 16; e /= 16;
      int k = e % H; e /= H;
      int tile = e % g.n4t; int c = e / g.n4t;
      int lr = tile * 16 + r;
      int n = c * g.rpc + lr;
      if (lr < g.rpc && n < P_OUT) v = W2[(size_t)n * H + k];
    }
    out[i] = v;
  }
}

// ------------------------------------------------------------------ prologue
// frame 0 of the outputs, CellStateEncoder input [x0 | style[:,0]] and x_pose(1) = vectorize(pose0, gaze[:,1])
__global__ void decoder_prologue_kernel(zeggs_decoder_fwd_args a, DecGeom g, float* cse_in, float* xp1) {
  const int b = blockIdx.x;
  const int Z = a.Z, T = a.T;
  Q4 q; q.w = a.root_rot0[b * 4 + 0]; q.x = a.root_rot0[b * 4 + 1]; q.y = a.root_rot0[b * 4 + 2]; q.z = a.root_rot0[b * 4 + 3];
  V3 p = v3(a.root_pos0[b * 3 + 0], a.root_pos0[b * 3 + 1], a.root_pos0[b * 3 + 2]);
  const int bt = b / 32, bl = b % 32;
  float* xp = xp1 + (size_t)bt * K1P * 32;
  for (int n = threadIdx.x; n < P_IN + Z; n += blockDim.x) {
    if (n < P_OUT) {
      float v = a.pose0[(size_t)b * P_OUT + n];
      a.Y[((size_t)b * T + 0) * P_OUT + n] = v;
      float xn = (v - a.in_mean[n]) / a.in_std[n];
      cse_in[(size_t)b * (P_IN + Z) + n] = xn;
      if (T > 1) xp[(size_t)n * 32 + bl] = xn;
    } else if (n < P_IN) {
      int d = n - P_OUT;
      // gaze_dir = R(root_rot)^-1 (gaze_pos - root_pos)   modules.py:696
      V3 g0 = v3(a.gaze_pos[((size_t)b * T + 0) * 3 + 0], a.gaze_pos[((size_t)b * T + 0) * 3 + 1], a.gaze_pos[((size_t)b * T + 0) * 3 + 2]);
      V3 d0 = quat_mul_vec(quat_inv(q), g0 - p);
      float v0 = d == 0 ? d0.x : (d == 1 ? d0.y : d0.z);
      cse_in[(size_t)b * (P_IN + Z) + n] = (v0 - a.in_mean[n]) / a.in_std[n];
      if (T > 1) {
        V3 g1 = v3(a.gaze_pos[((size_t)b * T + 1) * 3 + 0], a.gaze_pos[((size_t)b * T + 1) * 3 + 1], a.gaze_pos[((size_t)b * T + 1) * 3 + 2]);
        V3 d1 = quat_mul_vec(quat_inv(q), g1 - p);
        float v1 = d == 0 ? d1.x : (d == 1 ? d1.y : d1.z);
        xp[(size_t)n * 32 + bl] = (v1 - a.in_mean[n]) / a.in_std[n];
      }
    } else {
      cse_in[(size_t)b * (P_IN + Z) + n] = a.style[((size_t)b * T + 0) * Z + (n - P_IN)];
    }
  }
  if (threadIdx.x < 3) a.root_pos[((size_t)b * T) * 3 + threadIdx.x] = a.root_pos0[b * 3 + threadIdx.x];
  if (threadIdx.x < 4) a.root_rot[((size_t)b * T) * 4 + threadIdx.x] = a.root_rot0[b * 4 + threadIdx.x];
}

// cse_out[B][2H] -> H0[slot0], H1[slot0] in k-major [bt][H][32]   (modules.py:243)
__global__ void cse_scatter_kernel(int B, int H, const float* __restrict__ cse_out, float* __restrict__ h0, float* __restrict__ h1) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * 2 * H) return;
  int b = i / (2 * H), r = i % (2 * H);
  int l = r / H, j = r % H;
  float* dst = l == 0 ? h0 : h1;
  dst[((size_t)(b / 32) * H + j) * 32 + (b % 32)] = cse_out[i];
}

// S01[t][bt][n][32], n in [0,4H): n<H: b0[n] + W0[n, 1134:] . cond ; else b_ih0[n-H] + W_ih0[n-H, H+1134:] . cond
// cond = [speech[b,t,:] | style[b,t,:]].  One CTA per (t, bt, 64-row tile).
__global__ void __launch_bounds__(256) cond_precompute_kernel(zeggs_decoder_fwd_args a, DecGeom g, float* __restrict__ S01) {
  extern __shared__ float sm[];
  const int C = a.S + a.Z, H = a.H, T = a.T, A = g.A;
  float* cs = sm;              // [C][33]
  float* ws = sm + C * 33;     // [64][C+1]
  const int t = blockIdx.x, bt = blockIdx.y, n0 = blockIdx.z * 64;
  for (int i = threadIdx.x; i < 32 * C; i += blockDim.x) {
    int bl = i / C, cc = i % C;
    int b = bt * 32 + bl;
    float v = 0.f;
    if (b < a.B) v = cc < a.S ? a.speech[((size_t)b * T + t) * a.S + cc] : a.style[((size_t)b * T + t) * a.Z + (cc - a.S)];
    cs[cc * 33 + bl] = v;
  }
  for (int i = threadIdx.x; i < 64 * C; i += blockDim.x) {
    int r = i / C, cc = i % C;
    int n = n0 + r;
    float v = 0.f;
    if (n < 4 * H) v = n < H ? a.W0[(size_t)n * A + P_IN + cc] : a.W_ih0[(size_t)(n - H) * (A + H) + H + P_IN + cc];
    ws[r * (C + 1) + cc] = v;
  }
  __syncthreads();
  const int bl = threadIdx.x & 31, rw = threadIdx.x >> 5;  // 8 warps x 8 rows
  for (int rr = 0; rr < 8; ++rr) {
    int r = rw * 8 + rr, n = n0 + r;
    if (n >= 4 * H) break;
    float acc = n < H ? a.b0[n] : a.b_ih0[n - H];
    for (int cc = 0; cc < C; ++cc) acc = fmaf(ws[r * (C + 1) + cc], cs[cc * 33 + bl], acc);
    S01[(((size_t)t * g.nbt + bt) * 4 * H + n) * 32 + bl] = acc;
  }
}

// ------------------------------------------------------------------ the persistent kernel
// FILM: the FiLM decoder's step (modulated layer0, the extra layer2 stage, layer3 as the output layer; see FilmDev)
// Stages 1-3 (and FiLM 3b) run once per pass of V units: the tiles are those of V units, the weight slices P1-P3 / P5 pass-major.
template <int U, bool FILM>
__global__ void __launch_bounds__(256, 1) decoder_fwd_kernel(zeggs_decoder_fwd_args a, DecGeom g, DecWs w, FilmDev f) {
  extern __shared__ __align__(16) float smem[];
  constexpr int V = pass_units(U), NP = U / V;
  constexpr int RT1 = V, RT2 = (6 * V) / 4;
  float* stage = smem;                                  // 8 warps x 2 x STG_MAX
  float* red = smem + 8 * 2 * SkinnyCfg<RT2>::STG;      // [8][6V][32]
  float* gi0p = red + 8 * 6 * V * 32;                   // [nbt][3][U][32]
  float* rootv = gi0p + g.nbt * 3 * U * 32;             // [6][32]
  const int c = blockIdx.x, tid = threadIdx.x, warp = tid >> 5;
  const int H = a.H, T = a.T, nbt = g.nbt;
  float* wstage = stage + warp * 2 * SkinnyCfg<RT2>::STG;
  GridBarrier gb(w.bar);

  const float* P1 = a.packed + (size_t)c * K1P * 4 * U;
  const float* P2 = a.packed + g.off_p2() + (size_t)c * H * 6 * U;
  const float* P3 = a.packed + g.off_p3() + (size_t)c * H * 6 * U;
  const float* P4 = a.packed + g.off_p4() + (size_t)c * g.n4t * H * 16;
  constexpr int RTM = film_rows(V) / 4;          // FiLM layer2 tile (film_rows(V) rows per pass)
  const float* P5 = a.packed + g.packed_floats() + (size_t)c * NP * H * 4 * RTM;
  const size_t actH = (size_t)nbt * H * 32;      // floats per time slot of an [nbt][H][32] buffer
  const size_t actX = (size_t)nbt * K1P * 32;

  for (int t = 1; t < T; ++t) {
    const int ts = w.save ? t : (t & 1), tp = w.save ? t - 1 : ((t - 1) & 1), tn = w.save ? t + 1 : ((t + 1) & 1);
    // ------------------------------------------------------------ stage 1
    for (int q = 0; q < nbt * NP; ++q) {
      const int bt = q / NP, p = q % NP;
      float acc[RT1][4];
      const float* x = w.XP + ts * actX + (size_t)bt * K1P * 32;
      skinny_gemm<RT1, false>(acc, P1 + (size_t)p * K1P * 4 * V, x, x, K1P / 16, wstage);
      reduce_store<RT1>(acc, red);
      __syncthreads();
      for (int idx = tid; idx < V * 32; idx += 256) {
        const int u = p * V + (idx >> 5), b = idx & 31, j = c * U + u;
        const float* S = w.S01 + (((size_t)t * nbt + bt) * 4 * H) * 32;
        float pre = red_sum<4 * V>(red, idx >> 5, b) + S[(size_t)j * 32 + b];
        if constexpr (FILM) {
          const int bgl = bt * 32 + b;
          const float* gb = f.GB + ((size_t)bgl * T + t) * 4 * H;
          const float e = elu_f(pre);
          w.A[ts * actH + ((size_t)bt * H + j) * 32 + b] = bgl < a.B ? e * (1.f + gb[j]) + gb[2 * H + j] : e;   // modules.py:219-220
          if (w.save) f.E0[ts * actH + ((size_t)bt * H + j) * 32 + b] = e;
        } else {
          w.A[ts * actH + ((size_t)bt * H + j) * 32 + b] = elu_f(pre);
        }
#pragma unroll
        for (int gi = 0; gi < 3; ++gi)
          gi0p[((bt * 3 + gi) * U + u) * 32 + b] = red_sum<4 * V>(red, (1 + gi) * V + (idx >> 5), b) + S[(size_t)(H + gi * H + j) * 32 + b];
      }
      __syncthreads();
    }
    grid_sync(gb);
    // ------------------------------------------------------------ stage 2 (GRU layer 0)
    for (int q = 0; q < nbt * NP; ++q) {
      const int bt = q / NP, p = q % NP;
      float acc[RT2][4];
      const float* xa = w.A + ts * actH + (size_t)bt * H * 32;
      const float* xb = w.H0 + tp * actH + (size_t)bt * H * 32;
      skinny_gemm<RT2, true>(acc, P2 + (size_t)p * H * 6 * V, xa, xb, H / 16, wstage);
      reduce_store<RT2>(acc, red);
      __syncthreads();
      for (int idx = tid; idx < V * 32; idx += 256) {
        const int u = p * V + (idx >> 5), v = idx >> 5, b = idx & 31, j = c * U + u;
        float gir = red_sum<6 * V>(red, 0 * V + v, b) + gi0p[((bt * 3 + 0) * U + u) * 32 + b];
        float giz = red_sum<6 * V>(red, 1 * V + v, b) + gi0p[((bt * 3 + 1) * U + u) * 32 + b];
        float gin = red_sum<6 * V>(red, 2 * V + v, b) + gi0p[((bt * 3 + 2) * U + u) * 32 + b];
        float ghr = red_sum<6 * V>(red, 3 * V + v, b) + a.b_hh0[0 * H + j];
        float ghz = red_sum<6 * V>(red, 4 * V + v, b) + a.b_hh0[1 * H + j];
        float ghn = red_sum<6 * V>(red, 5 * V + v, b) + a.b_hh0[2 * H + j];
        float r, z, n;
        float h = gru_gate_fwd(gir, giz, gin, ghr, ghz, ghn, ld_cg(xb + (size_t)j * 32 + b), r, z, n);
        w.H0[ts * actH + ((size_t)bt * H + j) * 32 + b] = h;
        if (w.save) {
          float* G = w.G0 + ((size_t)t * nbt + bt) * 4 * H * 32;
          G[(size_t)(0 * H + j) * 32 + b] = r; G[(size_t)(1 * H + j) * 32 + b] = z;
          G[(size_t)(2 * H + j) * 32 + b] = n; G[(size_t)(3 * H + j) * 32 + b] = ghn;
        }
      }
      __syncthreads();
    }
    grid_sync(gb);
    // ------------------------------------------------------------ stage 3 (GRU layer 1)
    for (int q = 0; q < nbt * NP; ++q) {
      const int bt = q / NP, p = q % NP;
      float acc[RT2][4];
      const float* xa = w.H0 + ts * actH + (size_t)bt * H * 32;
      const float* xb = w.H1 + tp * actH + (size_t)bt * H * 32;
      skinny_gemm<RT2, true>(acc, P3 + (size_t)p * H * 6 * V, xa, xb, H / 16, wstage);
      reduce_store<RT2>(acc, red);
      __syncthreads();
      for (int idx = tid; idx < V * 32; idx += 256) {
        const int u = p * V + (idx >> 5), v = idx >> 5, b = idx & 31, j = c * U + u;
        float gir = red_sum<6 * V>(red, 0 * V + v, b) + a.b_ih1[0 * H + j];
        float giz = red_sum<6 * V>(red, 1 * V + v, b) + a.b_ih1[1 * H + j];
        float gin = red_sum<6 * V>(red, 2 * V + v, b) + a.b_ih1[2 * H + j];
        float ghr = red_sum<6 * V>(red, 3 * V + v, b) + a.b_hh1[0 * H + j];
        float ghz = red_sum<6 * V>(red, 4 * V + v, b) + a.b_hh1[1 * H + j];
        float ghn = red_sum<6 * V>(red, 5 * V + v, b) + a.b_hh1[2 * H + j];
        float r, z, n;
        float h = gru_gate_fwd(gir, giz, gin, ghr, ghz, ghn, ld_cg(xb + (size_t)j * 32 + b), r, z, n);
        w.H1[ts * actH + ((size_t)bt * H + j) * 32 + b] = h;
        if (w.save) {
          float* G = w.G1 + ((size_t)t * nbt + bt) * 4 * H * 32;
          G[(size_t)(0 * H + j) * 32 + b] = r; G[(size_t)(1 * H + j) * 32 + b] = z;
          G[(size_t)(2 * H + j) * 32 + b] = n; G[(size_t)(3 * H + j) * 32 + b] = ghn;
        }
      }
      __syncthreads();
    }
    grid_sync(gb);
    if constexpr (FILM) {
      // ---------------------------------------------------------- stage 3b (FiLM layer2: c = ELU(Wm h1 + bm) * g[H:] + be[H:])
      for (int q = 0; q < nbt * NP; ++q) {
        const int bt = q / NP, p = q % NP;
        float acc[RTM][4];
        const float* x = w.H1 + ts * actH + (size_t)bt * H * 32;
        skinny_gemm<RTM, false>(acc, P5 + (size_t)p * H * 4 * RTM, x, x, H / 16, wstage);
        reduce_store<RTM>(acc, red);
        __syncthreads();
        for (int idx = tid; idx < V * 32; idx += 256) {
          const int b = idx & 31, j = c * U + p * V + (idx >> 5), bgl = bt * 32 + b;
          const float e = elu_f(red_sum<4 * RTM>(red, idx >> 5, b) + f.bm[j]);
          const float* gbr = f.GB + ((size_t)bgl * T + t) * 4 * H;
          f.C2[ts * actH + ((size_t)bt * H + j) * 32 + b] = bgl < a.B ? e * (1.f + gbr[H + j]) + gbr[3 * H + j] : e;   // modules.py:224-225
          if (w.save) f.E2[ts * actH + ((size_t)bt * H + j) * 32 + b] = e;
        }
        __syncthreads();
      }
      grid_sync(gb);
    }
    // ------------------------------------------------------------ stage 4 (layer2 -- FiLM: layer3 -- + pose integration)
    for (int bt = 0; bt < nbt; ++bt) {
      const float* x = (FILM ? f.C2 : w.H1) + ts * actH + (size_t)bt * H * 32;
      float* xpn = w.XP + tn * actX + (size_t)bt * K1P * 32;
      for (int tile = 0; tile < g.n4t; ++tile) {
        float acc[4][4];
        skinny_gemm<4, false>(acc, P4 + (size_t)tile * H * 16, x, x, H / 16, wstage);
        reduce_store<4>(acc, red);
        __syncthreads();
        for (int idx = tid; idx < 16 * 32; idx += 256) {
          const int r = idx >> 5, b = idx & 31;
          const int lr = tile * 16 + r, n = c * g.rpc + lr;
          if (lr < g.rpc && n < P_OUT) {
            float y = red_sum<16>(red, r, b) + a.b2[n];
            float p = y * a.out_std[n] + a.out_mean[n];        // modules.py:728
            const int bgl = bt * 32 + b;
            if (bgl < a.B) a.Y[((size_t)bgl * T + t) * P_OUT + n] = p;
            if (t + 1 < T) xpn[(size_t)n * 32 + b] = (p - a.in_mean[n]) / a.in_std[n];   // modules.py:713
            if (n < 6) rootv[n * 32 + b] = p;
          }
        }
        __syncthreads();
      }
      if (c == 0 && tid < 32) {
        const int b = tid, bgl = bt * 32 + b;
        if (bgl < a.B) {
          const float* rp = a.root_pos + ((size_t)bgl * T + (t - 1)) * 3;
          const float* rq = a.root_rot + ((size_t)bgl * T + (t - 1)) * 4;
          V3 pos = v3(rp[0], rp[1], rp[2]);
          Q4 q; q.w = rq[0]; q.x = rq[1]; q.y = rq[2]; q.z = rq[3];
          V3 vel = v3(rootv[0 * 32 + b], rootv[1 * 32 + b], rootv[2 * 32 + b]);
          V3 vrt = v3(rootv[3 * 32 + b], rootv[4 * 32 + b], rootv[5 * 32 + b]);
          V3 npos = quat_mul_vec(q, a.dt * vel) + pos;                               // modules.py:739
          Q4 nq = quat_mul(quat_from_helical(quat_mul_vec(q, a.dt * vrt)), q);      // modules.py:740
          float* op = a.root_pos + ((size_t)bgl * T + t) * 3;
          float* oq = a.root_rot + ((size_t)bgl * T + t) * 4;
          op[0] = npos.x; op[1] = npos.y; op[2] = npos.z;
          oq[0] = nq.w; oq[1] = nq.x; oq[2] = nq.y; oq[3] = nq.z;
          if (t + 1 < T) {
            const float* gp = a.gaze_pos + ((size_t)bgl * T + (t + 1)) * 3;
            V3 gd = quat_mul_vec(quat_inv(nq), v3(gp[0], gp[1], gp[2]) - npos);     // modules.py:696
            xpn[(size_t)(P_OUT + 0) * 32 + b] = (gd.x - a.in_mean[P_OUT + 0]) / a.in_std[P_OUT + 0];
            xpn[(size_t)(P_OUT + 1) * 32 + b] = (gd.y - a.in_mean[P_OUT + 1]) / a.in_std[P_OUT + 1];
            xpn[(size_t)(P_OUT + 2) * 32 + b] = (gd.z - a.in_mean[P_OUT + 2]) / a.in_std[P_OUT + 2];
          }
        }
      }
      __syncthreads();
    }
    if (t + 1 < T) grid_sync(gb);
  }
}

// ------------------------------------------------------------------ host side
// dynamic shared memory per CTA of the fp32 recurrence: it grows with the 32-sample batch tiles, which bounds the batch of one call
template <int U>
static size_t fwd_smem_bytes(int nbt) {
  constexpr int V = pass_units(U), RT2 = (6 * V) / 4;
  return (size_t)(8 * 2 * SkinnyCfg<RT2>::STG + 8 * 6 * V * 32 + nbt * 3 * U * 32 + 6 * 32) * sizeof(float);
}

static int check_fwd_args(const zeggs_decoder_fwd_args* a) {
  ZCHECK_ARG(a != nullptr, "decoder: null args");
  ZCHECK_ARG(a->B >= 1 && a->T >= 1, "decoder: bad B=%d T=%d", a->B, a->T);
  ZCHECK_ARG(fp32_hidden_ok(a->H), "decoder: hidden size %d unsupported (need H%%16==0, H<=2112)", a->H);
  ZCHECK_ARG(a->S >= 1 && a->Z >= 1 && a->S + a->Z <= 256, "decoder: bad S=%d Z=%d", a->S, a->Z);
  if (a->engine != 1) {
    const int U = units_per_cta(a->H);
    auto smem_of = [U](int nbt) { return dispatch_units(U, [nbt](auto u) { return fwd_smem_bytes<u>(nbt); }); };
    const int nbt = ceil_div(a->B, 32);
    DeviceLimits lim;
    RC(device_limits(&lim));
    ZCHECK_ARG(smem_of(nbt) <= lim.smem_optin, "decoder: batch %d needs %zu bytes of shared memory per CTA at hidden size %d (%zu available): "
               "at most %d samples per call", a->B, smem_of(nbt), a->H, lim.smem_optin, 32 * max_batch_tiles(smem_of, lim.smem_optin));
  }
  return ZEGGS_OK;
}

extern "C" size_t zeggs_decoder_packed_bytes(int H, int S, int Z) {
  if (!fp32_hidden_ok(H)) return 0;
  DecGeom g = make_geom(1, H, S, Z);
  return g.packed_floats() * sizeof(float);
}

// P1-P4 of geometry g: the whole pack of the normal decoder, the front of the FiLM decoder's
static int pack_fwd_slices(const zeggs_decoder_fwd_args& a, const DecGeom& g, float* packed, cudaStream_t stream) {
  pack_decoder_kernel<<<592, 256, 0, stream>>>(g, a.W0, a.W_ih0, a.W_hh0, a.W_ih1, a.W_hh1, a.W2, packed);
  LAUNCH_OK();
  return ZEGGS_OK;
}

extern "C" int zeggs_decoder_pack_weights(const zeggs_decoder_fwd_args* a, float* packed, void* stream) {
  CtxScope ctx_scope(a ? a->ctx : nullptr);
  int rc = check_fwd_args(a); if (rc) return rc;
  return pack_fwd_slices(*a, make_geom(a->B, a->H, a->S, a->Z), packed, (cudaStream_t)stream);
}

extern "C" size_t zeggs_decoder_workspace_bytes(int B, int T, int H, int S, int Z, int save) {
  if (!fp32_hidden_ok(H) || B < 1 || T < 1) return 0;
  DecGeom g = make_geom(B, H, S, Z);
  return make_ws(nullptr, g, T, save).bytes;
}

// fp32 engine, normal and FiLM: the hoisted conditioning terms of `a` (the FiLM decoder passes Z = 0: its recurrence reads the speech
// alone), then the SIMT recurrence
template <bool FILM>
static int decoder_fwd_fp32_run(const zeggs_decoder_fwd_args& a, const DecGeom& g, const DecWs& w, const FilmDev& f, cudaStream_t stream) {
  const int C = a.S + a.Z;
  const size_t sm = (size_t)(C * 33 + 64 * (C + 1)) * sizeof(float);
  RC(set_max_dynamic_smem(cond_precompute_kernel, sm));
  cond_precompute_kernel<<<dim3(a.T, g.nbt, ceil_div(4 * a.H, 64)), 256, sm, stream>>>(a, g, w.S01);
  count_launch();
  ZCHECK_LAUNCH();
  ScopedTimer tm("decoder_fwd", stream);
  // the shared memory is within the device's limit: check_fwd_args
  return dispatch_units(g.U, [&](auto u) {
    return launch_persistent(decoder_fwd_kernel<u, FILM>, g.G, 256, fwd_smem_bytes<u>(g.nbt), 1, stream, a, g, w, f);
  });
}

// frame 0 and the initial GRU state (modules.py:72-98), shared by both decoders
static int decoder_fwd_prologue(const zeggs_decoder_fwd_args& a, const DecGeom& g, const DecWs& w, cudaStream_t stream) {
  int rc;
  // zero: barrier words, the x_pose slots (k padding rows / batch padding columns) and the h slot 0
  ZCHECK_CUDA(cudaMemsetAsync(w.bar, 0, 256, stream));
  ZCHECK_CUDA(cudaMemsetAsync(w.XP, 0, (size_t)w.TS * g.nbt * K1P * 32 * sizeof(float), stream));
  ZCHECK_CUDA(cudaMemsetAsync(w.H0, 0, (size_t)g.nbt * a.H * 32 * sizeof(float), stream));
  ZCHECK_CUDA(cudaMemsetAsync(w.H1, 0, (size_t)g.nbt * a.H * 32 * sizeof(float), stream));
  decoder_prologue_kernel<<<a.B, 256, 0, stream>>>(a, g, w.cse_in, w.XP + (size_t)g.nbt * K1P * 32);
  count_launch();
  ZCHECK_LAUNCH();
  // CellStateEncoder (modules.py:238-243)
  rc = gemm_f32_auto(0, a.B, a.H, P_IN + a.Z, w.cse_in, P_IN + a.Z, a.Wc0, P_IN + a.Z, a.bc0, w.cse_h1, a.H, 1, 0, stream); if (rc) return rc;
  rc = gemm_f32_auto(0, a.B, a.H, a.H, w.cse_h1, a.H, a.Wc1, a.H, a.bc1, w.cse_h2, a.H, 1, 0, stream); if (rc) return rc;
  rc = gemm_f32_auto(0, a.B, 2 * a.H, a.H, w.cse_h2, a.H, a.Wc2, a.H, a.bc2, w.cse_out, 2 * a.H, 0, 0, stream); if (rc) return rc;
  cse_scatter_kernel<<<ceil_div(a.B * 2 * a.H, 256), 256, 0, stream>>>(a.B, a.H, w.cse_out, w.H0, w.H1);
  count_launch();
  ZCHECK_LAUNCH();
  return ZEGGS_OK;
}

extern "C" int zeggs_decoder_window_fwd(const zeggs_decoder_fwd_args* ap, void* stream_) {
  int rc = check_fwd_args(ap); if (rc) return rc;
  const zeggs_decoder_fwd_args& a = *ap;
  CtxScope ctx_scope(a.ctx);
  cudaStream_t stream = (cudaStream_t)stream_;
  DecGeom g = make_geom(a.B, a.H, a.S, a.Z);
  DecWs w = make_ws(a.workspace, g, a.T, a.save_for_backward);
  ZCHECK_ARG(a.workspace != nullptr && a.workspace_bytes >= w.bytes, "decoder: workspace too small (%zu < %zu)", a.workspace_bytes, w.bytes);
  ZCHECK_ARG(a.engine == 1 || a.packed != nullptr, "decoder: packed weights missing (call zeggs_decoder_pack_weights)");
  ZCHECK_SUPPORTED(a.engine != 1 || tc_hidden_ok(a.H), "decoder tc engine: hidden size %d unsupported (needs H %% 128 == 0, 384 <= H <= 1024)", a.H);
  if ((rc = decoder_fwd_prologue(a, g, w, stream))) return rc;
  if (a.T == 1) return ZEGGS_OK;
  return a.engine == 1 ? decoder_fwd_tc_run(a, g, w, stream) : decoder_fwd_fp32_run<false>(a, g, w, FilmDev{}, stream);
}

// ------------------------------------------------------------------ FiLM decoder (fp32 engine)
// P5[c][p][k][r] = Wm[c*U + p*V + r][k] (r < V; rows up to film_rows(V) are zero), behind the normal decoder's slices
__global__ void pack_film_kernel(DecGeom g, const float* __restrict__ Wm, float* __restrict__ out) {
  const int H = g.H, U = g.U, V = pass_units(U), R = film_rows(V);
  const size_t total = (size_t)g.G * (U / V) * H * R;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int r = i % R, k = (i / R) % H, cp = i / ((size_t)R * H);   // cp = c * (U / V) + p
    out[i] = r < V ? Wm[(size_t)(cp * V + r) * H + k] : 0.f;
  }
}

static int check_film_args(const zeggs_decoder_film_fwd_args* f) {
  ZCHECK_ARG(f != nullptr, "film decoder: null args");
  int rc = check_fwd_args(&f->dec); if (rc) return rc;
  ZCHECK_SUPPORTED(f->dec.engine == 0, "film decoder: only the fp32 engine (engine 0) runs the FiLM recurrence: its layer2 carries an ELU "
                                       "and a modulation, so the tensor-core engine's layer-2 fold does not apply");
  ZCHECK_ARG(f->Wm && f->bm && f->Wg && f->bg && f->Wb && f->bb, "film decoder: layer2 / predictor weights missing");
  return ZEGGS_OK;
}

static size_t film_packed_floats(const DecGeom& g) { return g.packed_floats() + (size_t)g.G * g.H * film_rows(g.U); }

extern "C" size_t zeggs_decoder_packed_film_bytes(int H, int S, int Z) {
  if (!fp32_hidden_ok(H)) return 0;
  return film_packed_floats(make_film_geom(1, H, S, Z)) * sizeof(float);
}

extern "C" int zeggs_decoder_pack_weights_film(const zeggs_decoder_film_fwd_args* f, float* packed, void* stream_) {
  CtxScope ctx_scope(f ? f->dec.ctx : nullptr);
  int rc = check_film_args(f); if (rc) return rc;
  const zeggs_decoder_fwd_args& a = f->dec;
  cudaStream_t stream = (cudaStream_t)stream_;
  DecGeom g = make_film_geom(a.B, a.H, a.S, a.Z);
  if ((rc = pack_fwd_slices(a, g, packed, stream))) return rc;
  pack_film_kernel<<<264, 256, 0, stream>>>(g, f->Wm, packed + g.packed_floats());
  LAUNCH_OK();
  return ZEGGS_OK;
}

extern "C" size_t zeggs_decoder_film_workspace_bytes(int B, int T, int H, int S, int Z, int save) {
  if (!fp32_hidden_ok(H) || B < 1 || T < 1) return 0;
  DecGeom g = make_film_geom(B, H, S, Z);
  size_t bytes = 0;
  make_film_ws(nullptr, make_ws(nullptr, g, T, save), g, T, &bytes);
  return bytes;
}

extern "C" int zeggs_decoder_film_window_fwd(const zeggs_decoder_film_fwd_args* fp, void* stream_) {
  int rc = check_film_args(fp); if (rc) return rc;
  const zeggs_decoder_fwd_args& a = fp->dec;
  CtxScope ctx_scope(a.ctx);
  cudaStream_t stream = (cudaStream_t)stream_;
  DecGeom g = make_film_geom(a.B, a.H, a.S, a.Z);
  DecWs w = make_ws(a.workspace, g, a.T, a.save_for_backward);
  size_t bytes = 0;
  FilmDev f = make_film_ws(a.workspace, w, g, a.T, &bytes);
  f.bm = fp->bm;
  ZCHECK_ARG(a.workspace != nullptr && a.workspace_bytes >= bytes, "film decoder: workspace too small (%zu < %zu)", a.workspace_bytes, bytes);
  ZCHECK_ARG(a.packed != nullptr, "film decoder: packed weights missing (call zeggs_decoder_pack_weights_film)");
  if ((rc = decoder_fwd_prologue(a, g, w, stream))) return rc;
  if (a.T == 1) return ZEGGS_OK;
  // gamma - 1 and beta of every (b, t) as two GEMMs through the front end (modules.py:215-217)
  float* GB = const_cast<float*>(f.GB);
  rc = gemm_f32_auto(0, a.B * a.T, 2 * a.H, a.Z, a.style, a.Z, fp->Wg, a.Z, fp->bg, GB, 4 * a.H, 0, 0, stream); if (rc) return rc;
  rc = gemm_f32_auto(0, a.B * a.T, 2 * a.H, a.Z, a.style, a.Z, fp->Wb, a.Z, fp->bb, GB + 2 * a.H, 4 * a.H, 0, 0, stream); if (rc) return rc;
  // style does not enter layer0 / GRU0: the normal decoder's pre-pass and recurrence with no style columns
  zeggs_decoder_fwd_args as = a;
  as.Z = 0;
  return decoder_fwd_fp32_run<true>(as, g, w, f, stream);
}

}  // namespace zeggs
