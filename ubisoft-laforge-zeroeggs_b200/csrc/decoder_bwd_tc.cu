// Decoder BPTT recurrence on the tensor cores (engine 1).  Three stages per reverse step (B2, B3, B4 + R), a grid barrier
// between stages, every transposed GEMM a wgmma chain.
//
// The gradient w.r.t. a GRU layer's gate pre-activations is four H-vectors per sample: dpr, dpz, dpn (= d gi) and
// dpn*r (the n-block of d gh).  They are stored as ONE bf16 image of 128 rows = 4 blocks x 32 samples, K = H, so
// the 128 rows of two m64 MMAs are fully used and the K = 3H contractions of the SIMT formulation
// (dh_below = W_ih^T dgi, dh_prev = W_hh^T dgh) collapse into a single K = H chain per layer:
//     D[(blk,b)][(w,j)] = sum_k img[(blk,b)][k] * Wt[(w,j)][k]
// and the wanted sums are the block-diagonal entries (pr with *_r, pz with *_z, pn with ih_n, pnr with hh_n), added
// up by the epilogue from the accumulator staged in shared memory.
//
// Layer 2 is FOLDED out of the recurrence exactly as in the forward (decoder_fwd_tc.cu): with
// Mfold = (Wx[:, :1131] diag(os/is)) W2,
//     dh1(t-1) = W2^T (os * dY_ext(t-1))                       -- ONE batched GEMM before the recurrence (PRE)
//              + Mfold^T [dpre_a ; dgi0](t)                    -- extra columns of the B3 / B4 chains (block-diagonal again)
//              + W2[0:6]^T (os * dch(t-1))                     -- root-integration adjoint, run redundantly by every CTA
//              + (GRU1 recurrent terms),
// where the gaze adjoint feeding the root chain needs Wx[:, 1131:1134]^T dS1(t): three more columns per block.
//   B2  A = G1 image [128 x H],   B = [W_ih1^T | W_hh1^T]                       -> dh0 (+GRU0 adjoint -> G0 image), dh1(t-1) part
//   B3  A = G0 image [128 x H],   B = [W_ih0a^T | W_hh0^T | 3 x (Mfold_g^T, Wgz_g^T)] -> d pre_a image, dh0(t-1), fold / gaze parts
//   B4  A = d pre_a image [32 x H], B = [Mfold_a^T | Wgz_a^T]                  -> fold / gaze parts -> R(t-1): root adjoint,
//                                                                                  dh1(t-1) -> GRU1 gate adjoint -> G1 image
// The x_pose / layer-2 gradient history the weight gradients need (DY) is rebuilt after the recurrence by two batched
// GEMMs over the transposed dpre_a / dgi0 histories (decoder_bwd.cu).
// fp32 histories for the weight gradients are written in the same k-major layout as the SIMT kernel, so the batched
// wgrad code is shared.
#include "decoder_bwd_common.cuh"
#include "tc_dec_common.cuh"

namespace zeggs {

constexpr int BT_RING = 3;               // unified operand ring: each slot = 2 k-blocks of (A tile 16 KB | B tile)
constexpr int BT_XPART = 32768;          // bytes of the A part of a slot
constexpr int BT_ACC_LD = 132;           // column stride (floats) of the staged accumulator: 128 rows + 4 (bank spread)

struct BtGeom {
  int N2, N3, N4, P6;
  int kbH;
  int wslot;              // bytes of one weight k-block tile slot (max N * 128, 1 KB aligned)
  int slot_bytes;         // BT_XPART + 2 * wslot
  size_t off[4];          // chains: 0 = B2, 1 = B3, 2 = B4
  size_t cta_bytes;
};

inline BtGeom make_btgeom(const DecGeom& g, const BwdGeom&) {
  BtGeom t;
  t.P6 = round_up(6 * g.U, 16); t.N2 = t.P6; t.N3 = t.P6 + 48; t.N4 = 16;
  t.kbH = ceil_div(g.H, 64);
  t.wslot = round_up(t.N3 * 128, 1024);
  t.slot_bytes = BT_XPART + 2 * t.wslot;
  size_t off = 0;
  t.off[0] = off; off += (size_t)t.kbH * t.N2 * 128;
  t.off[1] = off; off += (size_t)t.kbH * t.N3 * 128;
  t.off[2] = off; off += (size_t)t.kbH * t.N4 * 128;
  t.off[3] = off;
  t.cta_bytes = off;
  return t;
}

// B3's extra 48 rows = three 16-row groups (gates r, z, n of d gi0): rows 0..U-1 = Mfold[(1+g)H + k][j] (this CTA's units j),
// rows 8..10 = W_ih0[gH + k][H + 1131 + d] (gaze columns); B4's 16 rows: the same with the pre_a block / W0.
// One thread per 16-byte image chunk, rows fastest: for a fixed k the 8 units of a row group are contiguous in the source
// (the weights are read transposed), so a warp reads full 32-byte segments.
__global__ void pack_decoder_bwd_tc_kernel(DecGeom g, BtGeom tg, const float* __restrict__ Mfold, const float* __restrict__ W0,
                                           const float* __restrict__ Wih0, const float* __restrict__ Whh0,
                                           const float* __restrict__ Wih1, const float* __restrict__ Whh1, uint8_t* __restrict__ out) {
  const int H = g.H, U = g.U, A = g.A;
  const size_t per = tg.cta_bytes / 16, total = (size_t)g.G * per;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int c = (int)(i / per);
    size_t ci = i % per;                                // chunk index inside the CTA block, re-ordered (kb, logical chunk, row)
    int chain = 2;
    for (int q = 0; q < 2; ++q) if (ci < tg.off[q + 1] / 16) { chain = q; break; }
    ci -= tg.off[chain] / 16;
    const int N = chain == 0 ? tg.N2 : chain == 1 ? tg.N3 : tg.N4;
    const int row = (int)(ci % N), cl = (int)((ci / N) % 8), kb = (int)(ci / ((size_t)8 * N));
    const int k0 = kb * 64 + cl * 8;
    const float* src = nullptr; size_t stride = 0;      // element e of the chunk = src[e * stride]
    if (k0 < H) {
      if (chain <= 1 && row < 6 * U) {                  // gate-row transposes
        const int wsel = row / U, u = row % U, gq = wsel % 3, j = c * U + u;
        const size_t r = (size_t)(gq * H + k0);
        if (chain == 0) { src = (wsel < 3 ? Wih1 : Whh1) + r * H + j; stride = H; }
        else if (wsel < 3) { src = Wih0 + r * (A + H) + j; stride = A + H; }
        else { src = Whh0 + r * H + j; stride = H; }
      } else if (chain == 1 && row >= tg.P6) {
        const int rr = row - tg.P6, gq = rr / 16, lr = rr % 16;
        if (lr < U) { src = Mfold + ((size_t)(1 + gq) * H + k0) * H + c * U + lr; stride = H; }
        else if (lr >= 8 && lr < 11) { src = Wih0 + (size_t)(gq * H + k0) * (A + H) + H + P_OUT + (lr - 8); stride = A + H; }
      } else if (chain == 2) {
        if (row < U) { src = Mfold + (size_t)k0 * H + c * U + row; stride = H; }
        else if (row >= 8 && row < 11) { src = W0 + (size_t)k0 * A + P_OUT + (row - 8); stride = A; }
      }
    }
    __nv_bfloat16 t[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) t[e] = __float2bfloat16_rn(src ? __ldg(src + (size_t)e * stride) : 0.f);
    uint8_t* dst = out + (size_t)c * tg.cta_bytes + tg.off[chain] + (size_t)kb * N * 128 + (size_t)row * 128 + (size_t)((cl ^ (row & 7)) << 4);
    *reinterpret_cast<uint4*>(dst) = *reinterpret_cast<const uint4*>(t);
  }
}

struct BtWs { uint8_t *g1img, *g0img, *dpaimg; const float* pre; float* dch; long long* dbg; size_t bytes; };
long long* tc_debug_buffer();
inline BtWs make_btws(void* base, const DecGeom& g) {
  BtWs w; size_t off = 0;
  auto take = [&](size_t n) { uint8_t* p = base ? (uint8_t*)base + off : nullptr; off += ((n + 1023) / 1024) * 1024; return p; };
  const size_t kbH = ceil_div(g.H, 64);
  w.g1img = take(kbH * 16384); w.g0img = take(kbH * 16384); w.dpaimg = take(kbH * 4096);
  w.pre = nullptr; w.dch = nullptr; w.dbg = nullptr;
  w.bytes = off; return w;
}

#define BTDBG1(ev) do { if (iw.dbg && c == 1 && lane == 0 && (T - 1 - t) < 64) iw.dbg[(T - 1 - t) * 32 + (ev)] = clock64(); } while (0)
#define BTDBG(ev) do { if (iw.dbg && c == 0 && lane == 0 && (T - 1 - t) < 64) iw.dbg[(T - 1 - t) * 32 + (ev)] = clock64(); } while (0)

// store U bf16 values at (row, k = j0..j0+U-1) of an image with `rows`-row tiles
template <int U>
__device__ __forceinline__ void store_img_row(uint8_t* img, int rows, int row, int j0, const float (&h)[U]) {
  __nv_bfloat16 t[U];
#pragma unroll
  for (int i = 0; i < U; ++i) t[i] = __float2bfloat16_rn(h[i]);
  uint8_t* p = img + img_off(rows, row, j0);
  if (U == 8) *reinterpret_cast<uint4*>(p) = *reinterpret_cast<const uint4*>(t);
  else *reinterpret_cast<uint2*>(p) = *reinterpret_cast<const uint2*>(t);
}

// Warp roles (224 threads): warps 0..3 = the MMA warpgroup, warp 4 = epilogue (lane = sample), warp 5 = weight producer (runs
// ahead across barriers), warp 6 = activation loader (grid-barrier waiter; streams the A images through the ring).  A chain's
// accumulator D[128 x N] is two m64 wgmma accumulators in the warpgroup's registers; once the chain has completed they are staged
// in shared memory (column-major, BT_ACC_LD floats per column) and the epilogue adds up the block-diagonal entries from there.
template <int U>
__global__ void __launch_bounds__(224, 1)
decoder_bwd_tc_kernel(zeggs_decoder_fwd_args a, DecGeom g, BwdGeom bg, BtGeom tg, DecWs w, BwdWs bw, BtWs iw, BwdArgsDev d,
                      const uint8_t* __restrict__ packed) {
  constexpr int P6 = (6 * U + 15) / 16 * 16, N2 = P6, N3 = P6 + 48, N4 = 16;
  constexpr int LD = BT_ACC_LD;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* ring = smem;                                         // BT_RING slots: [A kb0 | A kb1 | B kb0 | B kb1]
  uint8_t* tail = ring + (size_t)BT_RING * tg.slot_bytes;
  uint64_t* full = reinterpret_cast<uint64_t*>(tail);           // [BT_RING]  two producers (activations, weights) arrive on each
  uint64_t* empty = full + BT_RING;                             // [BT_RING]  one arrival per MMA warp
  uint64_t* d_full = empty + BT_RING;                           // [3]
  float* accs = reinterpret_cast<float*>(tail + 512);           // [N3][LD]  staged accumulator of the last chain
  float* c_w2r = accs + N3 * LD;                                // [6][U]  W2[n][j] * out_std[n], n < 6, this CTA's units
  float* c_gis = c_w2r + 6 * U;                                 // [4]     1 / in_std of the gaze channels

  // warp index broadcast from lane 0: provably warp-uniform, so the role branches below do not count as divergent code for wgmma
  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0), lane = threadIdx.x & 31;
  const int c = blockIdx.x, H = a.H, T = a.T;
  const int kbH = tg.kbH;
  const uint8_t* pk = packed + (size_t)c * tg.cta_bytes;
  constexpr int W_EPI = 4, W_PROD = 5, W_LOAD = 6;

  if (threadIdx.x == 0) {
    for (int i = 0; i < BT_RING; ++i) { mbar_init(&full[i], 2); mbar_init(&empty[i], 4); }
    for (int i = 0; i < 3; ++i) mbar_init(&d_full[i], 1);
    fence_mbar_init();
  }
  if (threadIdx.x < 6 * U) {
    const int n = threadIdx.x / U, u = threadIdx.x % U;
    c_w2r[threadIdx.x] = a.W2[(size_t)n * H + c * U + u] * a.out_std[n];
  }
  if (threadIdx.x < 3) c_gis[threadIdx.x] = 1.0f / a.in_std[P_OUT + threadIdx.x];
  __syncthreads();
  const size_t actH = (size_t)g.nbt * H * 32, act3 = (size_t)g.nbt * 3 * H * 32, act4 = (size_t)g.nbt * 4 * H * 32;

  if (warp == W_PROD) {
    // ================= weight producer (its half of every slot may be filled before the stage's grid barrier)
    if (lane == 0) {
      uint32_t it = 0;
      auto stream = [&](int chain, int nkb, int N, int kps) {
        const uint8_t* src = pk + tg.off[chain];
        const uint32_t tile = (uint32_t)N * 128;
        for (int kb = 0; kb < nkb; kb += kps, ++it) {
          const uint32_t s = it % BT_RING, ph = (it / BT_RING) & 1;
          const uint32_t bytes = (uint32_t)min(kps, nkb - kb) * tile;
          mbar_wait(&empty[s], ph ^ 1);
          mbar_arrive_expect_tx(&full[s], bytes);
          bulk_g2s(ring + (size_t)s * tg.slot_bytes + BT_XPART, src + (size_t)kb * tile, bytes, &full[s]);
        }
      };
      for (int t = T - 1; t >= 1; --t) {
        stream(0, kbH, tg.N2, 2); stream(1, kbH, tg.N3, 2);
        if (t > 1) stream(2, kbH, tg.N4, 8);
      }
    }
  } else if (warp == W_LOAD) {
    // ================= activation loader
    if (lane == 0) {
      uint32_t it = 0; unsigned epoch = 0;
      int t = T - 1; int sidx = 0;
      auto stream = [&](const uint8_t* img, int nkb, uint32_t tile_bytes) {
        grid_wait(bw.bar, (++epoch) * gridDim.x);
        if (iw.dbg && c == 0 && (T - 1 - t) < 64) iw.dbg[(T - 1 - t) * 32 + 2 * (sidx & 3)] = clock64();
        ++sidx;
        fence_proxy_async();
        const int kps = BT_XPART / (int)tile_bytes;               // 2 k-blocks of a 128-row image, 8 of a 32-row image
        for (int kb = 0; kb < nkb; kb += kps, ++it) {
          const uint32_t s = it % BT_RING, ph = (it / BT_RING) & 1;
          const uint32_t bytes = (uint32_t)min(kps, nkb - kb) * tile_bytes;
          mbar_wait(&empty[s], ph ^ 1);
          mbar_arrive_expect_tx(&full[s], bytes);
          bulk_g2s(ring + (size_t)s * tg.slot_bytes, img + (size_t)kb * tile_bytes, bytes, &full[s]);
        }
      };
      for (t = T - 1; t >= 1; --t) {
        sidx = 0;
        stream(iw.g1img, kbH, 16384); BTDBG(3);
        stream(iw.g0img, kbH, 16384); BTDBG(5);
        if (t > 1) { stream(iw.dpaimg, kbH, 4096); BTDBG(7); }
      }
    }
  } else if (warp < 4) {
    // ================= MMA warpgroup: one wait per slot, one wgmma group per slot, released once the next group is issued
    uint32_t it = 0;
    const uint64_t dR = make_smem_desc_sw128(ring);
    const uint32_t sstep = (uint32_t)(tg.slot_bytes >> 4);
    float d2[2][N2 / 2], d3[2][N3 / 2], d4[2][N4 / 2];
    // rows 64..127 of a 128-row image tile are 8 KB past its base; `two` = both row halves (128-row images) or rows 0..63 only
    auto chain_mma = [&](auto& dd, auto two, int nkb, int kps, uint32_t atile) {
      constexpr int N = 2 * (int)(sizeof(dd[0]) / sizeof(float));
      constexpr bool TWO = decltype(two)::value;
      const uint32_t astep = atile >> 4, wstep = (uint32_t)(N * 128) >> 4;
      uint32_t prev = 0;
      for (int kb = 0; kb < nkb; kb += kps, ++it) {
        const uint32_t s = it % BT_RING, ph = (it / BT_RING) & 1;
        const int nk = min(kps, nkb - kb);
        mbar_wait(&full[s], ph);
        uint64_t da = dR + (uint64_t)s * sstep, db = da + (BT_XPART >> 4);
        wgmma_fence();
        for (int kk = 0; kk < nk; ++kk, da += astep, db += wstep) {
#pragma unroll
          for (int ks = 0; ks < 4; ++ks) {
            const uint32_t acc = (kb + kk + ks) > 0 ? 1u : 0u;
            Wgmma<N>::mma(dd[0], da + 2 * ks, db + 2 * ks, acc);
            if constexpr (TWO) Wgmma<N>::mma(dd[1], da + 512 + 2 * ks, db + 2 * ks, acc);
          }
        }
        wgmma_commit();
        if (kb > 0) {
          wgmma_wait<1>();
          if (lane == 0) mbar_arrive(&empty[prev]);
        }
        prev = s;
      }
      wgmma_wait<0>();
      wgmma_fence_operands(dd[0]);
      if (TWO) wgmma_fence_operands(dd[1]);
      if (lane == 0) mbar_arrive(&empty[prev]);
      stage_acc<N>(dd[0], accs, LD, 0, TWO ? 64 : 32);
      if constexpr (TWO) stage_acc<N>(dd[1], accs, LD, 64, 64);
    };
    auto publish = [&](int i) {
      named_bar(1, 128);
      if (threadIdx.x == 0) mbar_arrive(&d_full[i]);
    };
    for (int t = T - 1; t >= 1; --t) {
      chain_mma(d2, std::true_type(), kbH, 2, 16384); publish(0); BTDBG(9);
      chain_mma(d3, std::true_type(), kbH, 2, 16384); publish(1); BTDBG(10);
      if (t > 1) { chain_mma(d4, std::false_type(), kbH, 8, 4096); publish(2); BTDBG(11); }
    }
  } else if (warp == W_EPI) {
    // ================= epilogue (lane = sample b).  Row 32*blk + b of a staged 128-row accumulator is block blk of sample b:
    // B2 / B3 blocks pr, pz, pn, pnr pair with the weight column groups (ih_r, hh_r), (ih_z, hh_z), (ih_n, -), (-, hh_n).
    const int b = lane;
    const bool live = b < a.B;
    const int j0 = c * U;
    auto A = [&](int col, int blk) { return accs[(size_t)col * LD + 32 * blk + b]; };
    // ---- R(t): adjoint of the root integration of frame t and of the gaze direction of step t+1 (modules.py:696, :739-740),
    // run by EVERY CTA for the 32 samples (lane = sample).  Returns dch[0:6] = d loss / d (de-normalised y(t)[0:6])
    // through the root chain and advances the running d root_pos / d root_rot.
    float dpq[7] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    float rpv[3] = {}, rqv[4] = {}, gpv[3] = {}, rq1v[4] = {}, ytv[6] = {}, e1p[3] = {}, e1q[4] = {}, e0p[3] = {}, e0q[4] = {};
    Q4 r_qinv, r_q1, r_E; V3 r_u, r_a1, r_a2, r_x; float r_k0 = 0.f, r_k1 = 0.f, r_k2 = 0.f;
    auto R_prefetch = [&](int t, bool have_dxp) {
      if (!live) return;
      const size_t bt = (size_t)b * T + t;
#pragma unroll
      for (int i = 0; i < 3; ++i) {
        rpv[i] = a.root_pos[bt * 3 + i];
        gpv[i] = have_dxp ? a.gaze_pos[(bt + 1) * 3 + i] : 0.f;
        e1p[i] = d.dRootPos ? d.dRootPos[(bt - 1) * 3 + i] : 0.f;
        e0p[i] = (!have_dxp && d.dRootPos) ? d.dRootPos[bt * 3 + i] : 0.f;
      }
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        rqv[i] = a.root_rot[bt * 4 + i];
        rq1v[i] = a.root_rot[(bt - 1) * 4 + i];
        e1q[i] = d.dRootRot ? d.dRootRot[(bt - 1) * 4 + i] : 0.f;
        e0q[i] = (!have_dxp && d.dRootRot) ? d.dRootRot[bt * 4 + i] : 0.f;
      }
#pragma unroll
      for (int i = 0; i < 6; ++i) ytv[i] = a.Y[bt * P_OUT + i];
    };
    auto R_precompute = [&]() {               // gradient-independent part (before the wait on the B4 accumulator)
      if (!live) return;
      Q4 qt; qt.w = rqv[0]; qt.x = rqv[1]; qt.y = rqv[2]; qt.z = rqv[3];
      r_qinv = quat_inv(qt);
      r_u = v3(gpv[0] - rpv[0], gpv[1] - rpv[1], gpv[2] - rpv[2]);
      r_q1.w = rq1v[0]; r_q1.x = rq1v[1]; r_q1.y = rq1v[2]; r_q1.z = rq1v[3];
      r_a1 = a.dt * v3(ytv[0], ytv[1], ytv[2]);
      r_a2 = a.dt * v3(ytv[3], ytv[4], ytv[5]);
      const V3 wv = quat_mul_vec(r_q1, r_a2);
      r_E = quat_from_helical(wv);
      // quat_from_helical_bwd is linear in dE: dx = k0 * dEv + (k1 * dE.w + k2 * dot(dEv, x)) * x   (common.cuh)
      r_x = 0.5f * wv;
      const float a2 = dot(r_x, r_x), an = sqrtf(a2);
      if (an < 1e-5f) {
        const float rn = sqrtf(1.0f + a2), n = rn + 1e-5f;
        r_k0 = 1.0f / n; r_k1 = -1.0f / (n * n * rn); r_k2 = r_k1;
      } else {
        const float sn = sinf(an), cs = cosf(an);
        r_k0 = sn / an; r_k1 = -sn / an; r_k2 = (an * cs - sn) / (a2 * an);
      }
    };
    auto R_adjoint = [&](const float (&dgz)[3], bool have_dxp, float (&dch)[6]) {
#pragma unroll
      for (int i = 0; i < 6; ++i) dch[i] = 0.f;
      if (!live) return;
      V3 dp; Q4 dq;
      if (!have_dxp) {
        dp = v3(e0p[0], e0p[1], e0p[2]); dq.w = e0q[0]; dq.x = e0q[1]; dq.y = e0q[2]; dq.z = e0q[3];
      } else {
        dp = v3(dpq[0], dpq[1], dpq[2]); dq.w = dpq[3]; dq.x = dpq[4]; dq.y = dpq[5]; dq.z = dpq[6];
        Q4 dqc; V3 du;                       // gaze_dir(t+1) = R(q_t)^-1 (gaze_pos[t+1] - p_t)
        quat_mul_vec_bwd(r_qinv, r_u, v3(dgz[0], dgz[1], dgz[2]), dqc, du);
        dq.w += dqc.w; dq.x -= dqc.x; dq.y -= dqc.y; dq.z -= dqc.z;
        dp = dp - du;
      }
      Q4 dq_a, dq_b, dq_c, dE; V3 da1, da2;
      quat_mul_vec_bwd(r_q1, r_a1, dp, dq_a, da1);
      quat_mul_bwd(r_E, r_q1, dq, dE, dq_b);
      const V3 dEv = v3(dE.x, dE.y, dE.z);
      const V3 dw = 0.5f * (r_k0 * dEv + (r_k1 * dE.w + r_k2 * dot(dEv, r_x)) * r_x);
      quat_mul_vec_bwd(r_q1, r_a2, dw, dq_c, da2);
      dch[0] = a.dt * da1.x; dch[1] = a.dt * da1.y; dch[2] = a.dt * da1.z; dch[3] = a.dt * da2.x; dch[4] = a.dt * da2.y; dch[5] = a.dt * da2.z;
      dpq[0] = dp.x + e1p[0]; dpq[1] = dp.y + e1p[1]; dpq[2] = dp.z + e1p[2];
      dpq[3] = dq_a.w + dq_b.w + dq_c.w + e1q[0]; dpq[4] = dq_a.x + dq_b.x + dq_c.x + e1q[1];
      dpq[5] = dq_a.y + dq_b.y + dq_c.y + e1q[2]; dpq[6] = dq_a.z + dq_b.z + dq_c.z + e1q[3];
    };
    // ---- GRU layer-1 gate adjoint of frame t from dh1(t): writes the G1 image + histories, keeps dh1*z
    float dhz1[U], dhz0[U], dsum[16];
    float g1r[U], g1z[U], g1n[U], g1hn[U], g1hp[U], g1acc[U], prev[U];
    auto G1_prefetch = [&](int t) {
      const float* G = w.G1 + t * act4;
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int j = j0 + u;
        g1r[u] = G[(size_t)(0 * H + j) * 32 + b]; g1z[u] = G[(size_t)(1 * H + j) * 32 + b];
        g1n[u] = G[(size_t)(2 * H + j) * 32 + b]; g1hn[u] = G[(size_t)(3 * H + j) * 32 + b];
        g1hp[u] = w.H1[(t - 1) * actH + (size_t)j * 32 + b];
        g1acc[u] = t == T - 1 ? 0.f : bw.DH1[(size_t)j * 32 + b];
      }
      const float* P = iw.pre + ((size_t)(live ? b : 0) * T + t) * H + j0;      // W2^T (os * dY_ext(t)) rows (b,t)
#pragma unroll
      for (int u4 = 0; u4 < U; u4 += 4) {
        const float4 v4 = live ? __ldg(reinterpret_cast<const float4*>(P + u4)) : make_float4(0.f, 0.f, 0.f, 0.f);
        prev[u4] = v4.x; prev[u4 + 1] = v4.y; prev[u4 + 2] = v4.z; prev[u4 + 3] = v4.w;
      }
    };
    auto G1_adjoint = [&](int t, const float (&fold)[U], const float (&dch)[6]) {
      float pr[U], pz[U], pn[U], pnr[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        float dh = prev[u] + fold[u] + g1acc[u];
#pragma unroll
        for (int n = 0; n < 6; ++n) dh = fmaf(c_w2r[n * U + u], dch[n], dh);
        float dgi[3], dgh[3];
        gru_gate_bwd(dh, g1r[u], g1z[u], g1n[u], g1hn[u], g1hp[u], dgi, dgh, dhz1[u]);
        pr[u] = dgi[0]; pz[u] = dgi[1]; pn[u] = dgi[2]; pnr[u] = dgh[2];
      }
      store_img_row<U>(iw.g1img, 128, 0 * 32 + b, j0, pr); store_img_row<U>(iw.g1img, 128, 1 * 32 + b, j0, pz);
      store_img_row<U>(iw.g1img, 128, 2 * 32 + b, j0, pn); store_img_row<U>(iw.g1img, 128, 3 * 32 + b, j0, pnr);
      grid_arrive(bw.bar);
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int j = j0 + u;
        bw.DGI1[t * act3 + (size_t)(0 * H + j) * 32 + b] = pr[u]; bw.DGI1[t * act3 + (size_t)(1 * H + j) * 32 + b] = pz[u];
        bw.DGI1[t * act3 + (size_t)(2 * H + j) * 32 + b] = pn[u];
        bw.DGH1[t * act3 + (size_t)(0 * H + j) * 32 + b] = pr[u]; bw.DGH1[t * act3 + (size_t)(1 * H + j) * 32 + b] = pz[u];
        bw.DGH1[t * act3 + (size_t)(2 * H + j) * 32 + b] = pnr[u];
      }
      if (c == 0 && live) {
        float* dc = iw.dch + ((size_t)t * 32 + b) * 8;
#pragma unroll
        for (int n = 0; n < 6; ++n) dc[n] = dch[n];
      }
    };

    {
      // frame T-1: only external gradients reach the root chain and dh1
      const float zero3[3] = {0.f, 0.f, 0.f};
      float zeroU[U], dch[6];
#pragma unroll
      for (int u = 0; u < U; ++u) zeroU[u] = 0.f;
      R_prefetch(T - 1, false); R_precompute(); G1_prefetch(T - 1);
      R_adjoint(zero3, false, dch);
      G1_adjoint(T - 1, zeroU, dch);
    }
    for (int t = T - 1; t >= 1; --t) {
      const uint32_t ph = (uint32_t)((T - 1 - t) & 1);
      // ------------------------------------------------------------ B2 epilogue
      float gr[U], gz[U], gn[U], ghn[U], hp[U], acc[U];
      {
        const float* G = w.G0 + t * act4;
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const int j = j0 + u;
          gr[u] = G[(size_t)(0 * H + j) * 32 + b]; gz[u] = G[(size_t)(1 * H + j) * 32 + b];
          gn[u] = G[(size_t)(2 * H + j) * 32 + b]; ghn[u] = G[(size_t)(3 * H + j) * 32 + b];
          hp[u] = w.H0[(t - 1) * actH + (size_t)j * 32 + b];
          acc[u] = t == T - 1 ? 0.f : bw.DH0[(size_t)j * 32 + b];
        }
      }
      mbar_wait(&d_full[0], ph);
      BTDBG(14);
      {
        float pr[U], pz[U], pn[U], pnr[U], dh1n[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const float oa = (A(0 * U + u, 0) + A(1 * U + u, 1)) + A(2 * U + u, 2);     // W_ih1^T dgi1
          const float ob = (A(3 * U + u, 0) + A(4 * U + u, 1)) + A(5 * U + u, 3);     // W_hh1^T dgh1
          float dgi[3], dgh[3];
          gru_gate_bwd(oa + acc[u], gr[u], gz[u], gn[u], ghn[u], hp[u], dgi, dgh, dhz0[u]);
          pr[u] = dgi[0]; pz[u] = dgi[1]; pn[u] = dgi[2]; pnr[u] = dgh[2];
          dh1n[u] = ob + dhz1[u];                                         // dh1(t-1) = dh1*z1 + W_hh1^T dgh1 (+ fold terms at B4)
        }
        store_img_row<U>(iw.g0img, 128, 0 * 32 + b, j0, pr); store_img_row<U>(iw.g0img, 128, 1 * 32 + b, j0, pz);
        store_img_row<U>(iw.g0img, 128, 2 * 32 + b, j0, pn); store_img_row<U>(iw.g0img, 128, 3 * 32 + b, j0, pnr);
        BTDBG(16);
        grid_arrive(bw.bar);
#pragma unroll
        for (int u = 0; u < U; ++u) bw.DH1[(size_t)(j0 + u) * 32 + b] = dh1n[u];   // private to this thread: no ordering needed
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const int j = j0 + u;
          bw.DGI0[t * act3 + (size_t)(0 * H + j) * 32 + b] = pr[u]; bw.DGI0[t * act3 + (size_t)(1 * H + j) * 32 + b] = pz[u];
          bw.DGI0[t * act3 + (size_t)(2 * H + j) * 32 + b] = pn[u];
          bw.DGH0[t * act3 + (size_t)(0 * H + j) * 32 + b] = pr[u]; bw.DGH0[t * act3 + (size_t)(1 * H + j) * 32 + b] = pz[u];
          bw.DGH0[t * act3 + (size_t)(2 * H + j) * 32 + b] = pnr[u];
        }
      }
      // ------------------------------------------------------------ B3 epilogue
      float av[U];
#pragma unroll
      for (int u = 0; u < U; ++u) av[u] = w.A[t * actH + (size_t)(j0 + u) * 32 + b];
      mbar_wait(&d_full[1], ph);
      BTDBG(17);
      {
        float dpa[U], dh0n[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const float da = (A(0 * U + u, 0) + A(1 * U + u, 1)) + A(2 * U + u, 2);
          const float ob = (A(3 * U + u, 0) + A(4 * U + u, 1)) + A(5 * U + u, 3);
          dpa[u] = da * (av[u] > 0.f ? 1.f : av[u] + 1.f);                 // ELU'(pre) = a + 1 for pre <= 0
          dh0n[u] = ob + dhz0[u];
        }
#pragma unroll
        for (int r = 0; r < 16; ++r)          // gate blocks of Mfold^T dgi0 (cols 0..U-1) and of the gaze adjoint (cols 8..10)
          dsum[r] = (A(P6 + r, 0) + A(P6 + 16 + r, 1)) + A(P6 + 32 + r, 2);
        store_img_row<U>(iw.dpaimg, 32, b, j0, dpa);
        BTDBG(18);
        if (t > 1) grid_arrive(bw.bar);
#pragma unroll
        for (int u = 0; u < U; ++u) { bw.DH0[(size_t)(j0 + u) * 32 + b] = dh0n[u]; bw.DPA[t * actH + (size_t)(j0 + u) * 32 + b] = dpa[u]; }
      }
      if (t == 1) break;
      // ------------------------------------------------------------ B4 epilogue: fold / gaze totals -> R(t-1) -> dh1(t-1) -> G1 image
      R_prefetch(t - 1, true); R_precompute(); G1_prefetch(t - 1);
      mbar_wait(&d_full[2], ph);
      BTDBG(19);
      float tot[16];
#pragma unroll
      for (int r = 0; r < 16; ++r) tot[r] = A(r, 0) + dsum[r];
      float fold[U], dgz[3], dch[6];
#pragma unroll
      for (int u = 0; u < U; ++u) fold[u] = tot[u];
#pragma unroll
      for (int i = 0; i < 3; ++i) dgz[i] = tot[8 + i] * c_gis[i];          // modules.py:713 (x = (gaze_dir - mean) / std)
      R_adjoint(dgz, true, dch);
      BTDBG(20);
      G1_adjoint(t - 1, fold, dch);
    }
  }
}

// ------------------------------------------------------------------ host
// dYs[(b,t)][n] = bf16(out_std[n] * dY[b][t][n]) (zero padded to ld): A operand of PRE = dYs . W2   (modules.py:728 adjoint)
__global__ void dy_scale_bf16_kernel(const float* __restrict__ dY, const float* __restrict__ os, size_t rows, int ld, __nv_bfloat16* __restrict__ out) {
  const size_t total = rows * (size_t)ld;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const size_t r = i / ld; const int n = (int)(i % ld);
    out[i] = __float2bfloat16_rn((dY && n < P_OUT) ? dY[r * P_OUT + n] * os[n] : 0.f);
  }
}

extern "C" size_t zeggs_decoder_packed_bwd_tc_bytes(int H, int S, int Z) {
  // the BPTT kernel pairs k-blocks (H % 128 == 0, part of tc_hidden_ok)
  if (!tc_hidden_ok(H)) return 0;
  DecGeom g = make_geom(1, H, S, Z);
  BtGeom tg = make_btgeom(g, make_bgeom(g));
  return (size_t)g.G * tg.cta_bytes;
}
extern "C" size_t zeggs_decoder_bwd_tc_workspace_bytes(int H, int S, int Z) {
  if (!tc_hidden_ok(H)) return 0;
  return make_btws(nullptr, make_geom(1, H, S, Z)).bytes;
}
extern "C" int zeggs_decoder_pack_weights_bwd_tc(const zeggs_decoder_fwd_args* a, void* packed, void* stream_) {
  CtxScope ctx_scope(a ? a->ctx : nullptr);
  ZCHECK_ARG(a && packed, "decoder bwd tc pack: bad arguments");
  ZCHECK_SUPPORTED(tc_hidden_ok(a->H), "decoder bwd tc pack: hidden size %d unsupported (needs H %% 128 == 0, 384 <= H <= 1024)", a->H);
  const float* mfold = decoder_tc_mfold(*a);
  ZCHECK_ARG(mfold != nullptr, "decoder bwd tc pack: the forward pack (zeggs_decoder_pack_weights_tc -> args.packed_tc) must run first");
  DecGeom g = make_geom(a->B, a->H, a->S, a->Z);
  BwdGeom bg = make_bgeom(g);
  BtGeom tg = make_btgeom(g, bg);
  ZCHECK_ARG(g.U <= 8, "decoder bwd tc: unsupported units per CTA");
  ScopedTimer tm_pack("weight_pack", (cudaStream_t)stream_);
  pack_decoder_bwd_tc_kernel<<<592, 256, 0, (cudaStream_t)stream_>>>(g, tg, mfold, a->W0, a->W_ih0, a->W_hh0, a->W_ih1, a->W_hh1, (uint8_t*)packed);
  count_launch();
  ZCHECK_LAUNCH();
  return ZEGGS_OK;
}

template <int U>
static int launch_bt(const zeggs_decoder_fwd_args& a, const DecGeom& g, const BwdGeom& bg, const BtGeom& tg, const DecWs& w,
                     const BwdWs& bw, const BtWs& iw, const BwdArgsDev& d, const uint8_t* packed, cudaStream_t stream) {
  const size_t smem = 1024 + (size_t)BT_RING * tg.slot_bytes + 512 + (size_t)(tg.N3 * BT_ACC_LD + 6 * U + 16) * sizeof(float);
  static size_t checked_smem = 0;     // attribute + co-residency check once per shared-memory size (one device per process)
  if (checked_smem != smem) {
    ZCHECK_CUDA(cudaFuncSetAttribute(decoder_bwd_tc_kernel<U>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int dev = 0, nsm = 0, occ = 0;
    ZCHECK_CUDA(cudaGetDevice(&dev));
    ZCHECK_CUDA(cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, dev));
    ZCHECK_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, decoder_bwd_tc_kernel<U>, 224, smem));
    ZCHECK_ARG(occ * nsm >= g.G, "decoder bwd tc: cooperative grid of %d CTAs does not fit", g.G);
    checked_smem = smem;
  }
  void* args[] = {(void*)&a, (void*)&g, (void*)&bg, (void*)&tg, (void*)&w, (void*)&bw, (void*)&iw, (void*)&d, (void*)&packed};
  ZCHECK_CUDA(cudaLaunchCooperativeKernel((void*)decoder_bwd_tc_kernel<U>, dim3(g.G), dim3(224), args, smem, stream));
  count_launch();
  return ZEGGS_OK;
}

int decoder_bwd_tc_run(const zeggs_decoder_fwd_args& a, const zeggs_decoder_bwd_args& b, const DecGeom& g, const DecWs& w,
                       const BwdWs& bw, cudaStream_t stream) {
  BwdGeom bg = make_bgeom(g);
  ZCHECK_ARG(g.nbt == 1, "decoder bwd tc engine needs B <= 32 (got B=%d)", a.B);
  ZCHECK_ARG(b.packed_bwd_tc && b.workspace_tc, "decoder bwd tc: packed_bwd_tc / workspace_tc missing");
  BtGeom tg = make_btgeom(g, bg);
  ZCHECK_ARG((tg.kbH % 2) == 0, "decoder bwd tc: unsupported geometry");
  BtWs iw = make_btws(b.workspace_tc, g);
  iw.dbg = tc_debug_buffer();
  iw.dch = bw.DCH;
  // PRE[(b,t)][j] = sum_n W2[n][j] out_std[n] dY[b][t][n]: the layer-2 adjoint of the external gradient for every frame at once
  const int H = a.H, ld = round_up(P_OUT, 8);
  const size_t rows = (size_t)a.B * a.T;
  char* p = scratch_base();
  ZCHECK_ARG(p != nullptr, "decoder bwd tc: scratch buffer missing (zeggs_ctx.scratch)");
  auto take = [&](size_t bytes) { char* r = p; p += (bytes + 255) / 256 * 256; return r; };
  __nv_bfloat16* dys = (__nv_bfloat16*)take(rows * ld * 2);
  __nv_bfloat16* w2t = (__nv_bfloat16*)take((size_t)H * ld * 2);
  float* pre = (float*)take(rows * H * sizeof(float));
  ZCHECK_ARG((size_t)(p - scratch_base()) <= scratch_bytes(), "decoder bwd tc: scratch buffer too small (%zu bytes needed)", (size_t)(p - scratch_base()));
  dy_scale_bf16_kernel<<<1184, 256, 0, stream>>>(b.dY, a.out_std, rows, ld, dys); count_launch();
  int rc = split_t_launch(a.W2, P_OUT, H, H, w2t, nullptr, ld, stream); if (rc) return rc;
  rc = tc_gemm_launch((int)rows, H, ld, dys, nullptr, ld, w2t, nullptr, ld, nullptr, pre, H, 0, 0, stream); if (rc) return rc;
  iw.pre = pre;
  BwdArgsDev d; d.dY = b.dY; d.dRootPos = b.dRootPos; d.dRootRot = b.dRootRot; d.packed = nullptr;
  return g.U == 4 ? launch_bt<4>(a, g, bg, tg, w, bw, iw, d, (const uint8_t*)b.packed_bwd_tc, stream)
                  : launch_bt<8>(a, g, bg, tg, w, bw, iw, d, (const uint8_t*)b.packed_bwd_tc, stream);
}

}  // namespace zeggs
