// Decoder BPTT recurrence on the tensor cores (engine 1).  Three stages per reverse step (B2, B3, B4 + R), a grid barrier
// between stages, every transposed GEMM a wgmma chain.
//
// The gradient w.r.t. a GRU layer's gate pre-activations is four H-vectors per sample: dpr, dpz, dpn (= d gi) and
// dpn*r (the n-block of d gh).  They are stored as ONE bf16 image of 128 rows = 4 blocks x 32 samples in the order
// [pr, pnr | pz, pn], K = H, and the K = 3H contractions of the SIMT formulation (dh_below = W_ih^T dgi,
// dh_prev = W_hh^T dgh) collapse into a single K = H chain per layer:
//     D[(blk,b)][(w,j)] = sum_k img[(blk,b)][k] * Wt[(w,j)][k]
// of which only the block-diagonal entries are wanted (pr with *_r, pz with *_z, pn with ih_n, pnr with hh_n).
//
// The grid runs as clusters of 2 CTAs.  A pair covers the 2U units of CTAs 2p and 2p+1 and splits the image by row
// halves: rank 0 streams rows 0..63 (pr, pnr) of every k-block tile and multiplies them by the columns they pair with
// (ih_r, hh_r, hh_n), rank 1 streams rows 64..127 (pz, pn) against (ih_z, hh_z, ih_n), each over the full K in one
// m64 accumulator.  So each SM receives half the image bytes and no MMA is spent on off-diagonal blocks.  Each rank
// stages its accumulator in its own shared memory, and the epilogue of either rank reads the entries for its own U
// units from both staging buffers (distributed shared memory), adding them in the same order as a single CTA would.
//
// Layer 2 is FOLDED out of the recurrence exactly as in the forward (decoder_fwd_tc.cu): with
// Mfold = (Wx[:, :1131] diag(os/is)) W2,
//     dh1(t-1) = W2^T (os * dY_ext(t-1))                       -- ONE batched GEMM before the recurrence (PRE)
//              + Mfold^T [dpre_a ; dgi0](t)                    -- extra columns of the B3 / B4 chains (block-diagonal again)
//              + W2[0:6]^T (os * dch(t-1))                     -- root-integration adjoint, run redundantly by every CTA
//              + (GRU1 recurrent terms),
// where the gaze adjoint feeding the root chain needs Wx[:, 1131:1134]^T dS1(t): three more columns per block.
//   B2  A = G1 image [64 of 128 x H],  B = 3 of [W_ih1^T | W_hh1^T]             -> dh0 (+GRU0 adjoint -> G0 image), dh1(t-1) part
//   B3  A = G0 image [64 of 128 x H],  B = 3 of [W_ih0a^T | W_hh0^T], 1 or 2 of 3 x (Mfold_g^T, Wgz_g^T)
//                                                                                -> d pre_a image, dh0(t-1), fold / gaze parts
//   B4  A = d pre_a image [32 x H], B = [Mfold_a^T | Wgz_a^T]                  -> fold / gaze parts -> R(t-1): root adjoint,
//                                                                                  dh1(t-1) -> GRU1 gate adjoint -> G1 image
// The x_pose / layer-2 gradient history the weight gradients need (DY) is rebuilt after the recurrence by two batched
// GEMMs over the transposed dpre_a / dgi0 histories (decoder_window_bwd_tc).
// fp32 histories for the weight gradients are written in the same k-major layout as the SIMT kernel, so the batched
// wgrad code is shared.
#include "decoder_bwd_common.cuh"
#include "tc_dec_common.cuh"

namespace zeggs {

constexpr int BT_RING = 4;               // unified operand ring: each slot = 2 k-blocks of (A half tile 8 KB | B tile)
constexpr int BT_XPART = 16384;          // bytes of the A part of a slot
constexpr int BT_ACC_LD = 68;            // column stride (floats) of a staged accumulator: 64 rows + 4 (bank spread)

// Column groups of a pair (2U units: CTA 2p's, then CTA 2p+1's).  B2 / B3 begin with three gate groups of 2U columns:
// rank 0 (image rows pr, pnr) ih_r, hh_r, hh_n; rank 1 (pz, pn) ih_z, hh_z, ih_n.  B3 then has the fold / gaze groups of the
// blocks the rank holds (rank 0: gate r; rank 1: gates z, n), FG columns each: 2U Mfold columns and 3 gaze columns, padded.
// Three fold groups over two ranks make rank 1's B3 chain the wider one (U = 8: 96 vs 72 columns).
struct BtGeom {
  int N2, N3[2], N4, FG;  // chain widths (B3 per cluster rank), fold group width
  int kbH;
  int wslot;              // bytes of one weight k-block tile slot (max N * 128, 1 KB aligned)
  int slot_bytes;         // BT_XPART + 2 * wslot
  size_t off[3];          // chains: 0 = B2, 1 = B3, 2 = B4; B3 last, so that only the block's length depends on the rank
  size_t cta_bytes;       // rank 1's block (the longer one); rank 0's ends with unused bytes
};

inline BtGeom make_btgeom(const DecGeom& g, const BwdGeom&) {
  BtGeom t;
  t.FG = round_up(2 * g.U + 3, 8);
  t.N2 = 6 * g.U; t.N3[0] = t.N2 + t.FG; t.N3[1] = t.N2 + 2 * t.FG; t.N4 = 16;
  t.kbH = ceil_div(g.H, 64);
  t.wslot = round_up(t.N3[1] * 128, 1024);
  t.slot_bytes = BT_XPART + 2 * t.wslot;
  t.off[0] = 0;
  t.off[2] = (size_t)t.kbH * t.N2 * 128;
  t.off[1] = t.off[2] + (size_t)t.kbH * t.N4 * 128;
  t.cta_bytes = t.off[1] + (size_t)t.kbH * t.N3[1] * 128;
  return t;
}

// Weight blocks per (pair p, rank rk) with the column groups above.  Gate group columns: unit p*2U + w of W^T for the group's
// (matrix, gate); fold group of gate gq: columns 0..2U-1 = Mfold[(1+gq)H + k][p*2U + w], 2U..2U+2 = W_ih0[gq H + k][H + 1131 + d]
// (gaze).  B4 is per CTA: rows 0..U-1 = Mfold[k][j] (this CTA's units j), rows 8..10 = W0[k][1131 + d].
// One thread per 16-byte image chunk, rows fastest: for a fixed k the units of a column group are contiguous in the source
// (the weights are read transposed), so a warp reads full 32-byte segments.
__global__ void pack_decoder_bwd_tc_kernel(DecGeom g, BtGeom tg, const float* __restrict__ Mfold, const float* __restrict__ W0,
                                           const float* __restrict__ Wih0, const float* __restrict__ Whh0,
                                           const float* __restrict__ Wih1, const float* __restrict__ Whh1, uint8_t* __restrict__ out) {
  const int H = g.H, U = g.U, A = g.A, N2 = tg.N2, FG = tg.FG;
  const size_t per = tg.cta_bytes / 16, total = (size_t)g.G * per;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int c = (int)(i / per), rk = c & 1, p = c >> 1;
    size_t ci = i % per;                                // chunk index inside the CTA block, re-ordered (kb, logical chunk, row)
    const int chain = ci < tg.off[2] / 16 ? 0 : ci < tg.off[1] / 16 ? 2 : 1;
    ci -= tg.off[chain] / 16;
    const int N = chain == 0 ? N2 : chain == 1 ? tg.N3[rk] : tg.N4;
    if (ci >= (size_t)tg.kbH * 8 * N) continue;        // the unused tail of rank 0's block
    const int row = (int)(ci % N), cl = (int)((ci / N) % 8), kb = (int)(ci / ((size_t)8 * N));
    const int k0 = kb * 64 + cl * 8;
    const float* src = nullptr; size_t stride = 0;      // element e of the chunk = src[e * stride]
    if (k0 < H) {
      if (chain <= 1 && row < N2) {                     // gate-row transposes
        const int grp = row / (2 * U), j = p * 2 * U + row % (2 * U);
        const bool ih = rk == 0 ? grp == 0 : grp != 1;
        const int gq = grp == 2 ? 2 : rk;
        const size_t r = (size_t)(gq * H + k0);
        if (chain == 0) { src = (ih ? Wih1 : Whh1) + r * H + j; stride = H; }
        else if (ih) { src = Wih0 + r * (A + H) + j; stride = A + H; }
        else { src = Whh0 + r * H + j; stride = H; }
      } else if (chain == 1) {
        const int f = (row - N2) / FG, lr = (row - N2) % FG, gq = rk + f;
        if (lr < 2 * U) { src = Mfold + ((size_t)(1 + gq) * H + k0) * H + p * 2 * U + lr; stride = H; }
        else if (lr < 2 * U + 3) { src = Wih0 + (size_t)(gq * H + k0) * (A + H) + H + P_OUT + (lr - 2 * U); stride = A + H; }
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

// trace of CTAs 0 and 1 (both ranks of pair 0): dbg[c][reverse step < 64][event < 32], clock64 of the CTA's SM
#define BTDBG(ev) do { if (iw.dbg && c < 2 && lane == 0 && (T - 1 - t) < 64) iw.dbg[c * 2048 + (T - 1 - t) * 32 + (ev)] = clock64(); } while (0)

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
// ahead across barriers), warp 6 = activation loader (grid-barrier waiter; streams the rank's half of the A images through the
// ring).  A chain's accumulator D[64 x N] is one m64 wgmma accumulator in the warpgroup's registers; once the chain has completed
// it is staged in this stage's buffer in shared memory (column-major, BT_ACC_LD floats per column), the local epilogue and the
// peer's are signalled, and each adds up the block-diagonal entries for its own units from both ranks' buffers.
//
// Reusing a stage buffer across reverse steps is race-free: the buffer of stage s is rewritten at step t-1 only after that
// step's chain s has consumed its image, which the loader streams only after a grid barrier that every CTA's epilogue arrives
// at after its stage-s reads of step t: the G1 image of t-1 (for B2) after the B4 epilogue of t, the G0 image (B3) after the
// B2 epilogue of t-1, the dpa image (B4) after the B3 epilogue of t-1.  The same ordering keeps a rank's remote arrival on
// d_full[s] for step t-1 behind the epilogue's wait on it for step t, so no phase of d_full completes early.
template <int U>
__global__ void __launch_bounds__(224, 1)
decoder_bwd_tc_kernel(zeggs_decoder_fwd_args a, DecGeom g, BwdGeom bg, BtGeom tg, DecWs w, BwdWs bw, BtWs iw, BwdArgsDev d,
                      const uint8_t* __restrict__ packed) {
  constexpr int N2 = 6 * U, FG = (2 * U + 3 + 7) / 8 * 8, N3A = N2 + FG, N3B = N2 + 2 * FG, N4 = 16;
  constexpr int LD = BT_ACC_LD;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* ring = smem;                                         // BT_RING slots: [A kb0 | A kb1 | B kb0 | B kb1]
  uint8_t* tail = ring + (size_t)BT_RING * tg.slot_bytes;
  uint64_t* full = reinterpret_cast<uint64_t*>(tail);           // [BT_RING]  two producers (activations, weights) arrive on each
  uint64_t* empty = full + BT_RING;                             // [BT_RING]  one arrival per MMA warp
  uint64_t* d_full = empty + BT_RING;                           // [3]  B2, B3: this rank's and the peer's publish; B4: this rank's
  float* acc2 = reinterpret_cast<float*>(tail + 512);           // [N2][LD]   staged B2 accumulator (read by both ranks)
  float* acc3 = acc2 + N2 * LD;                                 // [N3B][LD]  staged B3 accumulator (read by both ranks)
  float* acc4 = acc3 + N3B * LD;                                // [N4][LD]   staged B4 accumulator (rows 0..31)
  float* c_w2r = acc4 + N4 * LD;                                // [6][U]  W2[n][j] * out_std[n], n < 6, this CTA's units
  float* c_gis = c_w2r + 6 * U;                                 // [4]     1 / in_std of the gaze channels

  // warp index broadcast from lane 0: provably warp-uniform, so the role branches below do not count as divergent code for wgmma
  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0), lane = threadIdx.x & 31;
  const int c = blockIdx.x, H = a.H, T = a.T;
  const int rk = c & 1, peer = rk ^ 1;                          // rank in the cluster (clusters of 2 along x)
  const int kbH = tg.kbH;
  const uint8_t* pk = packed + (size_t)c * tg.cta_bytes;
  constexpr int W_EPI = 4, W_PROD = 5, W_LOAD = 6;

  if (threadIdx.x == 0) {
    for (int i = 0; i < BT_RING; ++i) { mbar_init(&full[i], 2); mbar_init(&empty[i], 4); }
    mbar_init(&d_full[0], 2); mbar_init(&d_full[1], 2); mbar_init(&d_full[2], 1);
    fence_mbar_init();
  }
  if (threadIdx.x < 6 * U) {
    const int n = threadIdx.x / U, u = threadIdx.x % U;
    c_w2r[threadIdx.x] = a.W2[(size_t)n * H + c * U + u] * a.out_std[n];
  }
  if (threadIdx.x < 3) c_gis[threadIdx.x] = 1.0f / a.in_std[P_OUT + threadIdx.x];
  cluster_sync_all();                                           // both ranks' mbarriers are initialised before any remote arrive
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
        stream(0, kbH, tg.N2, 2); stream(1, kbH, tg.N3[rk], 2);
        if (t > 1) stream(2, kbH, tg.N4, 4);
      }
    }
  } else if (warp == W_LOAD) {
    // ================= activation loader: per k-block, the rank's 64-row half of a 128-row tile (8 KB, contiguous: the SW128
    // swizzle depends on row & 7 only) or a whole 32-row tile
    if (lane == 0) {
      uint32_t it = 0; unsigned epoch = 0;
      int t = T - 1; int sidx = 0;
      auto stream = [&](const uint8_t* img, int nkb, uint32_t tile_bytes, uint32_t part_bytes, uint32_t part_off) {
        grid_wait(bw.bar, (++epoch) * gridDim.x);
        if (iw.dbg && c < 2 && (T - 1 - t) < 64) iw.dbg[c * 2048 + (T - 1 - t) * 32 + 2 * (sidx & 3)] = clock64();
        ++sidx;
        fence_proxy_async();
        const int kps = BT_XPART / (int)part_bytes;               // 2 k-blocks of a 128-row image, 4 of a 32-row image
        for (int kb = 0; kb < nkb; kb += kps, ++it) {
          const uint32_t s = it % BT_RING, ph = (it / BT_RING) & 1;
          const int nk = min(kps, nkb - kb);
          mbar_wait(&empty[s], ph ^ 1);
          mbar_arrive_expect_tx(&full[s], (uint32_t)nk * part_bytes);
          for (int kk = 0; kk < nk; ++kk)
            bulk_g2s(ring + (size_t)s * tg.slot_bytes + (size_t)kk * part_bytes, img + (size_t)(kb + kk) * tile_bytes + part_off,
                     part_bytes, &full[s]);
        }
      };
      for (t = T - 1; t >= 1; --t) {
        sidx = 0;
        stream(iw.g1img, kbH, 16384, 8192, rk * 8192); BTDBG(3);
        stream(iw.g0img, kbH, 16384, 8192, rk * 8192); BTDBG(5);
        if (t > 1) { stream(iw.dpaimg, kbH, 4096, 4096, 0); BTDBG(7); }
      }
    }
  } else if (warp < 4) {
    // ================= MMA warpgroup: one wait per slot, one wgmma group per slot, released once the next group is issued
    uint32_t it = 0;
    const uint64_t dR = make_smem_desc_sw128(ring);
    const uint32_t sstep = (uint32_t)(tg.slot_bytes >> 4);
    float d2[N2 / 2], d3a[N3A / 2], d3b[N3B / 2], d4[N4 / 2];
    // a 32-row B4 tile feeds the m64 MMA rows 32..63 from whatever follows it in the slot: they are never staged
    auto chain_mma = [&](auto& dd, int nkb, int kps, uint32_t atile, float* out, int nrows) {
      constexpr int N = 2 * (int)(sizeof(dd) / sizeof(float));
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
          for (int ks = 0; ks < 4; ++ks) Wgmma<N>::mma(dd, da + 2 * ks, db + 2 * ks, (kb + kk + ks) > 0 ? 1u : 0u);
        }
        wgmma_commit();
        if (kb > 0) {
          wgmma_wait<1>();
          if (lane == 0) mbar_arrive(&empty[prev]);
        }
        prev = s;
      }
      wgmma_wait<0>();
      wgmma_fence_operands(dd);
      if (lane == 0) mbar_arrive(&empty[prev]);
      stage_acc<N>(dd, out, LD, 0, nrows);
    };
    // B2 / B3 buffers are read by both ranks: the peer is signalled with a cluster-scope release after the staging barrier
    auto publish = [&](int i) {
      named_bar(1, 128);
      if (threadIdx.x == 0) {
        mbar_arrive(&d_full[i]);
        if (i < 2) mbar_arrive_cluster(&d_full[i], (uint32_t)peer);
      }
    };
    for (int t = T - 1; t >= 1; --t) {
      chain_mma(d2, kbH, 2, 8192, acc2, 64); publish(0); BTDBG(9);
      if (rk == 0) chain_mma(d3a, kbH, 2, 8192, acc3, 64);
      else chain_mma(d3b, kbH, 2, 8192, acc3, 64);
      publish(1); BTDBG(10);
      if (t > 1) { chain_mma(d4, kbH, 4, 4096, acc4, 32); publish(2); BTDBG(11); }
    }
  } else if (warp == W_EPI) {
    // ================= epilogue (lane = sample b).  Row 32*blk + b of a staged B2 / B3 accumulator is local block blk of sample
    // b: rank 0 holds pr, pnr, rank 1 pz, pn.  Column grp * 2U + wo + u is unit u of this CTA in gate group grp (wo = rk * U).
    const int b = lane;
    const bool live = b < a.B;
    const int j0 = c * U, wo = rk * U;
    // shared::cluster addresses of rank 0's and rank 1's B2 buffer (acc3 = acc2 + N2 * LD in both CTAs)
    const uint32_t a2r0 = cluster_map(acc2, 0u), a2r1 = cluster_map(acc2, 1u);
    auto X = [&](uint32_t s, int col, int blk) { return ld_cluster_f32(s + (uint32_t)(col * LD + 32 * blk + b) * 4u); };
    auto A = [&](const float* s, int col, int blk) { return s[(size_t)col * LD + 32 * blk + b]; };
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
    float dhz1[U], dhz0[U], dsf[U], dsg[3];
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
      store_img_row<U>(iw.g1img, 128, 0 * 32 + b, j0, pr); store_img_row<U>(iw.g1img, 128, 1 * 32 + b, j0, pnr);
      store_img_row<U>(iw.g1img, 128, 2 * 32 + b, j0, pz); store_img_row<U>(iw.g1img, 128, 3 * 32 + b, j0, pn);
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
      mbar_wait_cluster(&d_full[0], ph);
      BTDBG(14);
      {
        float pr[U], pz[U], pn[U], pnr[U], dh1n[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const float oa = (X(a2r0, 0 * 2 * U + wo + u, 0) + X(a2r1, 0 * 2 * U + wo + u, 0)) + X(a2r1, 2 * 2 * U + wo + u, 1);  // W_ih1^T dgi1
          const float ob = (X(a2r0, 1 * 2 * U + wo + u, 0) + X(a2r1, 1 * 2 * U + wo + u, 0)) + X(a2r0, 2 * 2 * U + wo + u, 1);  // W_hh1^T dgh1
          float dgi[3], dgh[3];
          gru_gate_bwd(oa + acc[u], gr[u], gz[u], gn[u], ghn[u], hp[u], dgi, dgh, dhz0[u]);
          pr[u] = dgi[0]; pz[u] = dgi[1]; pn[u] = dgi[2]; pnr[u] = dgh[2];
          dh1n[u] = ob + dhz1[u];                                         // dh1(t-1) = dh1*z1 + W_hh1^T dgh1 (+ fold terms at B4)
        }
        store_img_row<U>(iw.g0img, 128, 0 * 32 + b, j0, pr); store_img_row<U>(iw.g0img, 128, 1 * 32 + b, j0, pnr);
        store_img_row<U>(iw.g0img, 128, 2 * 32 + b, j0, pz); store_img_row<U>(iw.g0img, 128, 3 * 32 + b, j0, pn);
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
      mbar_wait_cluster(&d_full[1], ph);
      BTDBG(17);
      {
        float dpa[U], dh0n[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const float da = (X(a2r0, N2 + 0 * 2 * U + wo + u, 0) + X(a2r1, N2 + 0 * 2 * U + wo + u, 0)) + X(a2r1, N2 + 2 * 2 * U + wo + u, 1);
          const float ob = (X(a2r0, N2 + 1 * 2 * U + wo + u, 0) + X(a2r1, N2 + 1 * 2 * U + wo + u, 0)) + X(a2r0, N2 + 2 * 2 * U + wo + u, 1);
          dpa[u] = da * (av[u] > 0.f ? 1.f : av[u] + 1.f);                 // ELU'(pre) = a + 1 for pre <= 0
          dh0n[u] = ob + dhz0[u];
        }
        // fold groups r (rank 0), z, n (rank 1): Mfold^T dgi0 for this CTA's units, and the gaze adjoint (columns 2U..2U+2)
#pragma unroll
        for (int u = 0; u < U; ++u) dsf[u] = (X(a2r0, N2 + N2 + wo + u, 0) + X(a2r1, N2 + N2 + wo + u, 0)) + X(a2r1, N2 + N2 + FG + wo + u, 1);
#pragma unroll
        for (int i = 0; i < 3; ++i)
          dsg[i] = (X(a2r0, N2 + N2 + 2 * U + i, 0) + X(a2r1, N2 + N2 + 2 * U + i, 0)) + X(a2r1, N2 + N2 + FG + 2 * U + i, 1);
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
      float fold[U], dgz[3], dch[6];
#pragma unroll
      for (int u = 0; u < U; ++u) fold[u] = A(acc4, u, 0) + dsf[u];
#pragma unroll
      for (int i = 0; i < 3; ++i) dgz[i] = (A(acc4, 8 + i, 0) + dsg[i]) * c_gis[i];   // modules.py:713 (x = (gaze_dir - mean) / std)
      R_adjoint(dgz, true, dch);
      BTDBG(20);
      G1_adjoint(t - 1, fold, dch);
    }
  }
  cluster_sync_all();           // a CTA's shared memory must outlive the peer's last reads of its staged accumulators
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
  const size_t smem = 1024 + (size_t)BT_RING * tg.slot_bytes + 512 +
                      (size_t)((tg.N2 + tg.N3[1] + tg.N4) * BT_ACC_LD + 6 * U + 16) * sizeof(float);
  // clusters of 2 CTAs (the pairs sharing an image), launched cooperatively: the kernel spins on a grid barrier, so every
  // CTA must be resident at once
  cudaLaunchAttribute attr[2];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = 2; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
  attr[1].id = cudaLaunchAttributeCooperative;
  attr[1].val.cooperative = 1;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(g.G); cfg.blockDim = dim3(224); cfg.dynamicSmemBytes = smem; cfg.stream = stream;
  cfg.attrs = attr; cfg.numAttrs = 2;
  static size_t checked_smem = 0;     // attribute + co-residency query once per shared-memory size (one device per process)
  static int max_clusters = 0;
  if (checked_smem != smem) {
    ZCHECK_CUDA(cudaFuncSetAttribute(decoder_bwd_tc_kernel<U>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    cudaLaunchConfig_t occ = cfg;
    occ.numAttrs = 1;                 // the cluster shape only
    ZCHECK_CUDA(cudaOccupancyMaxActiveClusters(&max_clusters, decoder_bwd_tc_kernel<U>, &occ));
    checked_smem = smem;
  }
  ZCHECK_ARG(2 * max_clusters >= g.G, "decoder bwd tc: cooperative grid of %d CTAs in clusters of 2 does not fit (%d clusters resident)",
             g.G, max_clusters);
  ZCHECK_CUDA(cudaLaunchKernelEx(&cfg, decoder_bwd_tc_kernel<U>, a, g, bg, tg, w, bw, iw, d, packed));
  count_launch();
  return ZEGGS_OK;
}

// Tensor-core engine backward.  Phase 0 runs all of it.  Phase 1 runs the BPTT recurrence, the CellStateEncoder backward and the
// conditioning gradients (dSpeech, dStyle); phase 2 every remaining parameter gradient.  Split in two calls, the encoders' backward
// passes (which need only dSpeech / dStyle) can overlap the large weight-gradient GEMMs on other streams.  Phase 2 reads the history
// copies phase 1 left in the scratch buffer, which wgrad_hists and the carve-up below place at the same addresses in both calls.
int decoder_window_bwd_tc(const zeggs_decoder_fwd_args& a, const zeggs_decoder_bwd_args& b, const DecGeom& g, const DecWs& w,
                          const BwdWs& bw, cudaStream_t stream) {
  const int H = a.H, T = a.T, C = a.S + a.Z, A = g.A, phase = b.phase;
  const BwdGeom bg = make_bgeom(g);
  const BtGeom tg = make_btgeom(g, bg);
  ZCHECK_SUPPORTED(tc_hidden_ok(H), "decoder bwd tc: hidden size %d unsupported (needs H %% 128 == 0, 384 <= H <= 1024)", H);
  ZCHECK_ARG(g.nbt == 1 && bg.n4b == 1, "decoder bwd tc engine needs B <= 32 (got B=%d)", a.B);
  ZCHECK_ARG(b.workspace_tc, "decoder bwd tc: workspace_tc missing");
  ZCHECK_ARG(gemm_mode() != 0 && scratch_base() != nullptr,
             "decoder bwd tc: needs the tensor-core GEMM front end (a zeggs_ctx with scratch, gemm mode 1 or 2)");
  // PRE[(b,t)][j] = sum_n W2[n][j] out_std[n] dY[b][t][n]: the layer-2 adjoint of the external gradient for every frame at once,
  // operands and result at the scratch base for the duration of the recurrence
  const int ldy = round_up(P_OUT, 8);
  const size_t rows = (size_t)a.B * T;
  char* p = scratch_base();
  auto take = [&](size_t bytes) { char* r = p; p += (bytes + 255) / 256 * 256; return r; };
  __nv_bfloat16* dys = (__nv_bfloat16*)take(rows * ldy * 2);
  __nv_bfloat16* w2t = (__nv_bfloat16*)take((size_t)H * ldy * 2);
  float* pre = (float*)take(rows * H * sizeof(float));
  ZCHECK_ARG((size_t)(p - scratch_base()) <= scratch_bytes(), "decoder bwd tc: scratch buffer too small (%zu bytes needed)", (size_t)(p - scratch_base()));
  // the weight gradients: single-pass bf16 history copies (the recurrence already runs on bf16 operands, so one pass matches its
  // accuracy), and behind them the dpa / dgi0 copies transposed to [(t,b)][row] (A operands of the d cond and x_pose gradient GEMMs),
  // the transposed cond / x_pose columns of W0 / W_ih0 and the DXP result
  const WgradHists hs = wgrad_hists(a, b, g, w, bw, false);
  const size_t ld = hs.ld;
  const size_t extra = ld * H * 2 + ld * 3 * H * 2 + (size_t)C * 4 * H * 2 + (size_t)P_OUT * 4 * H * 2 + ld * P_OUT * 4 + 4096;
  ZCHECK_ARG(hs.bytes + extra <= scratch_bytes(), "decoder bwd tc: scratch buffer too small for the batched gradient GEMMs (%zu bytes needed)",
             hs.bytes + extra);
  char* q = hs.end;
  auto takeq = [&](size_t bytes) { char* r = (char*)(((uintptr_t)q + 255) & ~(uintptr_t)255); q = r + bytes; return r; };
  __nv_bfloat16* paT = (__nv_bfloat16*)takeq(ld * H * 2);
  __nv_bfloat16* giT = (__nv_bfloat16*)takeq(ld * 3 * H * 2);
  __nv_bfloat16* w0T = (__nv_bfloat16*)takeq((size_t)C * H * 2);
  __nv_bfloat16* wiT = (__nv_bfloat16*)takeq((size_t)C * 3 * H * 2);
  __nv_bfloat16* w0xT = (__nv_bfloat16*)takeq((size_t)P_OUT * H * 2);
  __nv_bfloat16* wixT = (__nv_bfloat16*)takeq((size_t)P_OUT * 3 * H * 2);
  float* dxp = (float*)takeq(ld * P_OUT * 4);
  const int cur = 32;                    // row of (t = 1, b = 0) in the transposed copies, column of slot t = 1 in the others
  const int Kc = (T - 1) * 32;
  int rc;
  if (phase != 2) {
    ZCHECK_CUDA(cudaMemsetAsync(bw.bar, 0, 256, stream));
    ZCHECK_CUDA(cudaMemsetAsync(bw.DY, 0, (size_t)T * K1P * 32 * sizeof(float), stream));
    ScopedTimer tm("decoder_bwd", stream);
    dy_scale_bf16_kernel<<<1184, 256, 0, stream>>>(b.dY, a.out_std, rows, ldy, dys); count_launch();
    if ((rc = split_t_launch(a.W2, P_OUT, H, H, w2t, nullptr, ldy, stream))) return rc;
    if ((rc = tc_gemm_launch((int)rows, H, ldy, dys, nullptr, ldy, w2t, nullptr, ldy, nullptr, pre, H, 0, 0, stream))) return rc;
    BtWs iw = make_btws(b.workspace_tc, g);
    iw.dbg = tc_debug_buffer();
    iw.dch = bw.DCH;
    iw.pre = pre;
    BwdArgsDev d; d.dY = b.dY; d.dRootPos = b.dRootPos; d.dRootRot = b.dRootRot; d.packed = nullptr;
    const uint8_t* pk = (const uint8_t*)b.packed_bwd_tc;
    rc = g.U == 4 ? launch_bt<4>(a, g, bg, tg, w, bw, iw, d, pk, stream) : launch_bt<8>(a, g, bg, tg, w, bw, iw, d, pk, stream);
    if (rc) return rc;
  }
  ScopedTimer tm("decoder_wgrad", stream);
  if (phase != 2) {
    if ((rc = cond_kmajor(a, g, bw, stream))) return rc;
    // before the history copies overwrite its staging area at the scratch base
    if ((rc = cse_backward(a, b, w, bw, stream))) return rc;
    // d cond on the tensor cores: DCOND[(t,b)][c] = dpa^T W0[:, 1134+c] + dgi0^T W_ih0[:, H+1134+c]
    if ((rc = split_hist(hs, HGI0, stream))) return rc;
    if ((rc = split_hist(hs, HPA, stream))) return rc;
    if ((rc = transpose_bf16_launch(hs.h[HPA].hi, H, (int)ld, ld, paT, H, stream))) return rc;
    if ((rc = transpose_bf16_launch(hs.h[HGI0].hi, 3 * H, (int)ld, ld, giT, 3 * H, stream))) return rc;
    if ((rc = split_t_launch(a.W0 + P_IN, H, C, A, w0T, nullptr, H, stream))) return rc;
    if ((rc = split_t_launch(a.W_ih0 + H + P_IN, 3 * H, C, A + H, wiT, nullptr, 3 * H, stream))) return rc;
    float* out = bw.DCOND + (size_t)cur * C;
    if ((rc = tc_gemm_launch(Kc, C, H, paT + (size_t)cur * H, nullptr, H, w0T, nullptr, H, nullptr, out, C, 0, 0, stream))) return rc;
    if ((rc = tc_gemm_launch(Kc, C, 3 * H, giT + (size_t)cur * 3 * H, nullptr, 3 * H, wiT, nullptr, 3 * H, nullptr, out, C, 0, 1, stream))) return rc;
    if ((rc = dcond_scatter(a, b, g, bw, 1, stream))) return rc;
  }
  if (phase != 1) {
    for (int i : {HGI1, HGH1, HGH0, HH0, HH1, HA, HXP, HCOND}) if ((rc = split_hist(hs, i, stream))) return rc;
    // the x_pose gradient of every step at once, from the transposed dpre_a / dgi0 copies of phase 1:
    //   DXP[(t,b)][n] = dpre_a(t)^T W0[:, n] + dgi0(t)^T W_ih0[:, H + n]      (n < 1131; modules.py:172-175 adjoint)
    // then the layer-2 / x_pose gradient history the weight gradients read (modules.py:713, :728 adjoints)
    if ((rc = split_t_launch(a.W0, H, P_OUT, A, w0xT, nullptr, H, stream))) return rc;
    if ((rc = split_t_launch(a.W_ih0 + H, 3 * H, P_OUT, A + H, wixT, nullptr, 3 * H, stream))) return rc;
    if ((rc = tc_gemm_launch(Kc, P_OUT, H, paT + (size_t)cur * H, nullptr, H, w0xT, nullptr, H, nullptr, dxp + (size_t)cur * P_OUT, P_OUT, 0, 0, stream))) return rc;
    if ((rc = tc_gemm_launch(Kc, P_OUT, 3 * H, giT + (size_t)cur * 3 * H, nullptr, 3 * H, wixT, nullptr, 3 * H, nullptr, dxp + (size_t)cur * P_OUT, P_OUT, 0, 1, stream))) return rc;
    if ((rc = dy_combine(a, b, dxp, bw, stream))) return rc;
    if ((rc = split_hist(hs, HDY, stream))) return rc;
    if ((rc = wgrad_gemms(a, b, g, hs, false, q, stream))) return rc;
  }
  return ZEGGS_OK;
}

}  // namespace zeggs
