// Decoder window forward on the Hopper tensor cores (engine 1).
//
// Same persistent, weight-stationary partition as decoder_fwd.cu (CTA c owns U hidden units of layer0 / GRU0 / GRU1),
// but (1) every stage GEMM is a wgmma chain and (2) layer2 is FOLDED out of the recurrence:
//
//   x(t+1)[n] = ((W2 h1(t) + b2)[n] * os[n] + om[n] - im[n]) / is[n]          n < 1131     (modules.py:728, :713)
//   [pre_a ; gi0](t+1) = Wx x(t+1) + cond terms,   Wx = [W0[:, :1134] ; W_ih0[:, H:H+1134]]   (modules.py:172-175)
//
// is linear in h1(t) apart from the three gaze columns, so with  Mfold = (Wx[:, :1131] diag(os/is)) W2   [4H x H]
//   [pre_a ; gi0](t+1) = Mfold h1(t) + cfold + Wx[:, 1131:1134] gaze(t+1) + S01[t+1]
// and a step needs only THREE all-to-all exchanges (a, h0, h1) instead of four.  The gaze direction needs the root
// state, i.e. y(t)[0:6] = W2[0:6] h1(t): six extra rows in every CTA's fold chain, and every CTA integrates the root
// trajectory of the 32 samples redundantly (modules.py:739-740, :696).  y(t) itself, the pose outputs and the x_pose
// history for the backward pass are produced AFTER the recurrence by one batched tensor-core GEMM over the bf16 h1 history
// (zeggs tc_gemm) + one elementwise pass.
//
// MMA shape: D[64 x N] (f32, registers of one warpgroup) = X[64 x K] (bf16, smem) * Wslice[N x K]^T (bf16, smem),
// wgmma.m64nNk16: rows 0..31 of the A operand are the 32 samples, rows 32..63 alias the following k-block (their
// accumulator rows are never read).
//
//   * Activations live in global memory as bf16 *shared-memory images* (128-byte rows, 16-byte chunks XOR-swizzled
//     by row&7 = SWIZZLE_128B K-major canonical layout), written by the producing epilogue: one cp.async.bulk per
//     16 KB chunk brings them in -- no tensor maps, no conversion passes.  Each stage loads ONE vector and runs the
//     critical chain plus the next consumer of the same vector from the same shared-memory copy
//     (h1(t-1): fold chain + gh1;  a(t): gi0a;  h0(t): gi1 + gh0 of step t+1).
//   * Weight slices are pre-packed once per optimizer step into the same image format per (CTA, chain, k-block) and
//     streamed through a shared-memory ring by a dedicated producer warp that runs ahead across grid barriers.
//   * Warp roles (256 threads): warps 0,1 = epilogue (lanes 0..15 = samples 0..15 / 16..31: gates / ELU / root
//     integration in fp32, writes next activations as bf16 images + fp32 state/history), warp 2 = weight producer,
//     warp 3 = activation loader (waits on the grid barrier, then bulk-copies X), warps 4..7 = MMA warpgroup.
//   GRU state, gates, pose integration and all saved-for-backward tensors stay fp32; only the MMA operands are bf16.
#include "decoder_common.cuh"
#include "tc_common.cuh"
#include "tc_dec_common.cuh"

namespace zeggs {

constexpr int TC_RING = 4;              // operand ring slots
constexpr int TC_GKB = 4;               // k-blocks per ring slot ("group"): ONE mbarrier wait per 16 MMAs
constexpr int TC_NEPI = 2;              // epilogue warps (grid-barrier arrivals per CTA and stage)
constexpr int TC_ACC_LD = 36;           // column stride (floats) of the staged accumulators: 32 sample rows + 4 (bank spread)

struct TcGeom {
  int NP;          // rows of a gate chain: round_up(3U,8)
  int N1;          // rows of the fold chain: 4U + 8 (6 used: W2[0:6])
  int kbH;         // k-blocks of an H-vector
  int slot_bytes;  // ring slot: TC_GKB k-block tiles of the widest chain
  size_t chain_off[6];   // byte offset of chain c inside one CTA's packed block
  size_t cta_bytes;
  // tail of the packed buffer (after G * cta_bytes)
  size_t off_mfold, off_wxdt, off_cfold, off_bfold, off_w2b, total_bytes;
};

__host__ __device__ inline size_t tc_tile_bytes(int N) { return (size_t)N * 128; }

inline TcGeom make_tcgeom(const DecGeom& g) {
  TcGeom t;
  t.NP = round_up(3 * g.U, 8);      // M = 64 allows N % 8 == 0: no padding rows at U = 8
  t.N1 = 4 * g.U + 8;
  t.kbH = ceil_div(g.H, 64);
  t.slot_bytes = TC_GKB * (int)tc_tile_bytes(t.N1);
  size_t off = 0;
  t.chain_off[0] = off; off += (size_t)t.kbH * tc_tile_bytes(t.N1);     // fold  X = h1(t-1)
  t.chain_off[1] = off; off += (size_t)t.kbH * tc_tile_bytes(t.NP);     // gh0   X = h0(t-1)
  t.chain_off[2] = off; off += (size_t)t.kbH * tc_tile_bytes(t.NP);     // gi0a  X = a(t)
  t.chain_off[3] = off; off += (size_t)t.kbH * tc_tile_bytes(t.NP);     // gh1   X = h1(t-1)
  t.chain_off[4] = off; off += (size_t)t.kbH * tc_tile_bytes(t.NP);     // gi1   X = h0(t)
  t.chain_off[5] = off;
  t.cta_bytes = off;
  auto al = [](size_t x) { return (x + 255) / 256 * 256; };
  size_t o = al((size_t)g.G * t.cta_bytes);
  t.off_mfold = o; o = al(o + (size_t)4 * g.H * g.H * 4);
  t.off_wxdt = o;  o = al(o + (size_t)P_OUT * 4 * g.H * 4);
  t.off_cfold = o; o = al(o + (size_t)4 * g.H * 4);
  t.off_bfold = o; o = al(o + (size_t)4 * g.H * 4);
  t.off_w2b = o;   o = al(o + (size_t)round_up(P_OUT, 128) * g.H * 2);
  t.total_bytes = o;
  return t;
}

// ------------------------------------------------------------------ fold preparation (once per weight version)
// WxDt[n][row] = Wx[row][n] * os[n] / is[n],  n < 1131, row < 4H   (transposed so the fold product is one TN GEMM)
__global__ void fold_wxdt_kernel(int H, int A, const float* __restrict__ W0, const float* __restrict__ Wih0,
                                 const float* __restrict__ os, const float* __restrict__ is, float* __restrict__ out) {
  __shared__ float tile[32][33];
  const int r0 = blockIdx.y * 32, n0 = blockIdx.x * 32;
  for (int i = threadIdx.y; i < 32; i += 8) {
    const int row = r0 + i, n = n0 + threadIdx.x;
    float v = 0.f;
    if (row < 4 * H && n < P_OUT) v = row < H ? W0[(size_t)row * A + n] : Wih0[(size_t)(row - H) * (A + H) + H + n];
    tile[i][threadIdx.x] = v;
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += 8) {
    const int n = n0 + i, row = r0 + threadIdx.x;
    if (n < P_OUT && row < 4 * H) out[(size_t)n * 4 * H + row] = tile[threadIdx.x][i] * os[n] / is[n];
  }
}
// cfold[row] = sum_n Wx[row][n] (b2[n] os[n] + om[n] - im[n]) / is[n];  bfold = [b0 ; b_ih0] + cfold.  One warp per row.
__global__ void fold_const_kernel(int H, int A, const float* __restrict__ W0, const float* __restrict__ Wih0,
                                  const float* __restrict__ b0, const float* __restrict__ bih0, const float* __restrict__ b2,
                                  const float* __restrict__ os, const float* __restrict__ om, const float* __restrict__ im,
                                  const float* __restrict__ is, float* __restrict__ cfold, float* __restrict__ bfold) {
  const int row = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= 4 * H) return;
  const float* wr = row < H ? W0 + (size_t)row * A : Wih0 + (size_t)(row - H) * (A + H) + H;
  float acc = 0.f;
  for (int n = lane; n < P_OUT; n += 32) acc = fmaf(wr[n], (b2[n] * os[n] + om[n] - im[n]) / is[n], acc);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if (lane == 0) { cfold[row] = acc; bfold[row] = acc + (row < H ? b0[row] : bih0[row - H]); }
}
// S01[1][b][row] += Wx[row] . x(1)[:, b] - cfold[row]   (the first step consumes the given pose, not h1(0))
__global__ void fold_first_step_kernel(int H, int A, const float* __restrict__ W0, const float* __restrict__ Wih0,
                                       const float* __restrict__ xp1 /* [K1P][32] */, const float* __restrict__ cfold,
                                       float* __restrict__ S01_t1 /* [32][4H] */) {
  const int row = blockIdx.x * 8 + (threadIdx.x >> 5), b = threadIdx.x & 31;
  if (row >= 4 * H) return;
  const float* wr = row < H ? W0 + (size_t)row * A : Wih0 + (size_t)(row - H) * (A + H) + H;
  float acc = 0.f;
  for (int n = 0; n < P_IN; ++n) acc = fmaf(__ldg(wr + n), xp1[(size_t)n * 32 + b], acc);
  S01_t1[(size_t)b * 4 * H + row] += acc - cfold[row];
}

// ------------------------------------------------------------------ packing (bf16 images of the weight slices)
// One thread per 16-byte image chunk: 8 consecutive k of one weight row (two 16-byte reads, one 16-byte write).
__global__ void pack_decoder_tc_kernel(DecGeom g, TcGeom tg, const float* __restrict__ Mfold, const float* __restrict__ Wih0,
                                       const float* __restrict__ Whh0, const float* __restrict__ Wih1,
                                       const float* __restrict__ Whh1, const float* __restrict__ W2, uint8_t* __restrict__ out) {
  const int H = g.H, U = g.U, A = g.A;
  const size_t per = tg.cta_bytes / 16, total = (size_t)g.G * per;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int c = (int)(i / per);
    size_t b = (i % per) * 16;                          // byte offset inside the CTA block
    int chain = 4;
    for (int q = 0; q < 4; ++q) if (b < tg.chain_off[q + 1]) { chain = q; break; }
    b -= tg.chain_off[chain];
    const int N = chain == 0 ? tg.N1 : tg.NP;
    const int kb = (int)(b / tc_tile_bytes(N));
    const int rb = (int)(b % tc_tile_bytes(N));
    const int row = rb / 128, chunk_phys = (rb % 128) / 16;
    const int k0 = kb * 64 + ((chunk_phys ^ (row & 7)) << 3);
    const float* src = nullptr;
    if (k0 < H) {
      if (chain == 0) {
        if (row < 4 * U) { const int gi = row / U, j = c * U + row % U; src = Mfold + (size_t)(gi * H + j) * H + k0; }
        else if (row < 4 * U + 6) src = W2 + (size_t)(row - 4 * U) * H + k0;
      } else if (row < 3 * U) {
        const int gi = row / U, j = c * U + row % U;
        const size_t r = (size_t)(gi * H + j);
        src = chain == 1 ? Whh0 + r * H + k0 : chain == 2 ? Wih0 + r * (A + H) + k0 : chain == 3 ? Whh1 + r * H + k0 : Wih1 + r * H + k0;
      }
    }
    __nv_bfloat16 t[8];
    if (src && (reinterpret_cast<uintptr_t>(src) & 7) == 0) {
#pragma unroll
      for (int e = 0; e < 8; e += 2) {                  // 8-byte aligned row segment (always for even row strides)
        const float2 v = __ldg(reinterpret_cast<const float2*>(src + e));
        t[e] = __float2bfloat16_rn(v.x); t[e + 1] = __float2bfloat16_rn(v.y);
      }
    } else if (src) {                                   // odd row stride (e.g. W_ih0 with the 9-label style code, A + H = 2231)
#pragma unroll
      for (int e = 0; e < 8; ++e) t[e] = __float2bfloat16_rn(__ldg(src + e));
    } else {
#pragma unroll
      for (int e = 0; e < 8; ++e) t[e] = __float2bfloat16_rn(0.f);
    }
    *reinterpret_cast<uint4*>(out + i * 16) = *reinterpret_cast<const uint4*>(t);
  }
}

// fp32 k-major vector [K][32] -> bf16 image (32 rows); K padded with zeros to kbs*64
__global__ void image_from_kmajor_kernel(const float* __restrict__ src, int K, int kbs, uint8_t* __restrict__ img) {
  const int total = kbs * 64 * 32;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int b = i & 31, k = i >> 5;
    const float v = k < K ? src[(size_t)k * 32 + b] : 0.f;
    *reinterpret_cast<__nv_bfloat16*>(img + img_off(32, b, k)) = __float2bfloat16_rn(v);
  }
}

struct TcWs {
  uint8_t *ab, *h0b[2], *h1b[2];            // bf16 activation images
  long long* dbg;                            // optional per-step phase timestamps of CTA 0 (clock64), [T][32]
  size_t bytes;
};
inline TcWs make_tcws(void* base, const DecGeom& g) {
  TcWs w; size_t off = 0;
  auto take = [&](size_t n) { uint8_t* p = base ? (uint8_t*)base + off : nullptr; off += ((n + 1023) / 1024) * 1024; return p; };
  const size_t hb = (size_t)ceil_div(g.H, 64) * 4096;
  w.ab = take(hb);
  w.h0b[0] = take(hb); w.h0b[1] = take(hb); w.h1b[0] = take(hb); w.h1b[1] = take(hb);
  w.dbg = nullptr;
  w.bytes = off; return w;
}

// per-CTA phase timestamps (development trace): dbg[(cta * 64 + t) * 32 + event], SM-local clock64
#define TCDBG(ev) do { if (tw.dbg && warp_lane0 && t < 64) tw.dbg[((size_t)c * 64 + t) * 32 + (ev)] = clock64(); } while (0)

// Warp roles (256 threads): warps 0,1 = epilogue, warp 2 = weight producer, warp 3 = activation loader, warps 4..7 = the MMA
// warpgroup.  A chain's accumulator D[64 x N] lives in the warpgroup's registers; once its last MMA has completed, rows 0..31 (the
// samples) are staged in shared memory, column-major with a 36-float column stride, for the epilogue.  One accumulator per chain:
// the MMAs of a chain accumulate back to back into the same registers.
template <int U>
__global__ void __launch_bounds__(256, 1)
decoder_fwd_tc_kernel(zeggs_decoder_fwd_args a, DecGeom g, TcGeom tg, DecWs w, TcWs tw, const uint8_t* __restrict__ packed) {
  constexpr int NP = (3 * U + 7) / 8 * 8;        // gate-chain rows (24 for U=8, 16 for U=4)
  constexpr int N1 = 4 * U + 8;                  // fold-chain rows
  constexpr int SLOT = TC_GKB * N1 * 128;
  constexpr int ACC_LD = TC_ACC_LD;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  // layout: X0 | X1 | ring | 4 KB slack | barriers | constants | staged accumulators
  // (operand rows 32..63 of the last k-block alias what follows)
  const int kbH = tg.kbH;
  uint8_t* X0 = smem;
  uint8_t* X1 = X0 + kbH * 4096;
  uint8_t* ring = X1 + kbH * 4096;
  uint8_t* tail = ring + TC_RING * SLOT + 4096;
  uint64_t* bars = reinterpret_cast<uint64_t*>(tail);
  uint64_t* full = bars;                        // [TC_RING]  two arrivals per use: weight producer + activation loader
  uint64_t* empty = bars + TC_RING;             // [TC_RING]  one arrival per MMA warp
  uint64_t* d_full = empty + TC_RING;           // [3]
  float* cst = reinterpret_cast<float*>(tail + 512);   // per-CTA constants
  float* c_bhh0 = cst;            // [3U]
  float* c_bih1 = cst + 3 * U;    // [3U]
  float* c_bhh1 = cst + 6 * U;    // [3U]
  float* c_wgz = cst + 12 * U;    // [4U][4]  gaze columns of Wx for this CTA's fold rows (16-byte rows)
  float* c_y6 = c_wgz + 16 * U;   // b2[0:6], out_std[0:6], out_mean[0:6]
  float* c_gz = c_y6 + 18;        // in_mean[1131:1134], 1 / in_std[1131:1134]
  float* acc_gh0 = c_gz + 8;                    // [NP][ACC_LD]  gh0
  float* acc_gh1 = acc_gh0 + NP * ACC_LD;       // [NP][ACC_LD]  gh1
  float* acc_main = acc_gh1 + NP * ACC_LD;      // [N1][ACC_LD]  fold / gi0a / gi1

  // warp index broadcast from lane 0: provably warp-uniform, so the role branches below do not count as divergent code for wgmma
  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0), lane = threadIdx.x & 31;
  const bool warp_lane0 = lane == 0;
  const int c = blockIdx.x, H = a.H, T = a.T;
  const uint8_t* pk = packed + (size_t)c * tg.cta_bytes;
  constexpr int W_PROD = 2, W_LOAD = 3;

  if (threadIdx.x == 0) {
    for (int i = 0; i < TC_RING; ++i) { mbar_init(&full[i], 2); mbar_init(&empty[i], 4); }
    for (int i = 0; i < 3; ++i) mbar_init(&d_full[i], 1);
    fence_mbar_init();
  }
  for (int i = threadIdx.x; i < 3 * U; i += blockDim.x) {
    const int j = (i / U) * H + c * U + (i % U);
    c_bhh0[i] = a.b_hh0[j]; c_bih1[i] = a.b_ih1[j]; c_bhh1[i] = a.b_hh1[j];
  }
  for (int i = threadIdx.x; i < 16 * U; i += blockDim.x) {
    const int row = i / 4, d = i % 4, gi = row / U, j = c * U + row % U;
    c_wgz[i] = d == 3 ? 0.f : gi == 0 ? a.W0[(size_t)j * g.A + P_OUT + d] : a.W_ih0[(size_t)((gi - 1) * H + j) * (g.A + H) + H + P_OUT + d];
  }
  if (threadIdx.x < 6) {
    c_y6[threadIdx.x] = a.b2[threadIdx.x]; c_y6[6 + threadIdx.x] = a.out_std[threadIdx.x]; c_y6[12 + threadIdx.x] = a.out_mean[threadIdx.x];
  }
  if (threadIdx.x < 3) { c_gz[threadIdx.x] = a.in_mean[P_OUT + threadIdx.x]; c_gz[3 + threadIdx.x] = 1.0f / a.in_std[P_OUT + threadIdx.x]; }
  __syncthreads();
  const size_t actH = (size_t)g.nbt * H * 32;
  const unsigned bar_n = gridDim.x * TC_NEPI;

  const int ng = (kbH + TC_GKB - 1) / TC_GKB;      // ring groups per chain
  auto group_kb = [&](int gi) { return gi * TC_GKB; };
  // Operand ring: slot = the weight tiles of TC_GKB k-blocks.  The X chunk of the same k-blocks lands in the resident X
  // buffer but completes on the SAME mbarrier, so the MMA warpgroup waits once per 16 k-steps.  Chains whose X is already
  // resident (gh1 after the fold chain, gh0 after gi1) get the second arrival from the weight producer.  Chain sequence: q = 0:
  // gh0 of step 1;  step t: q = 1 + 5 (t-1) + {0 fold, 1 gh1, 2 gi0a, 3 gi1, 4 gh0 of t+1};  the last fold chain: q = 5 (T-1).
  if (warp == W_PROD) {
    // ================= weight producer: streams every chain's tiles in the MMA warp's consumption order
    if (lane == 0) {
      uint32_t it = 0;
      auto stream = [&](int chain, bool has_loader) {
        const int N = chain == 0 ? N1 : NP;
        const uint8_t* src = pk + tg.chain_off[chain];
        for (int gi = 0; gi < ng; ++gi, ++it) {
          const int kb = group_kb(gi);
          const uint32_t s = it % TC_RING, ph = (it / TC_RING) & 1;
          const uint32_t bytes = (uint32_t)((kbH - kb >= TC_GKB ? TC_GKB : kbH - kb) * tc_tile_bytes(N));
          mbar_wait(&empty[s], ph ^ 1);
          mbar_arrive_expect_tx(&full[s], bytes);
          bulk_g2s(ring + (size_t)s * SLOT, src + (size_t)kb * tc_tile_bytes(N), bytes, &full[s]);
          if (!has_loader) mbar_arrive(&full[s]);
        }
      };
      stream(1, true);                                 // gh0 of step 1
      for (int t = 1; t < T; ++t) {                    // per step: fold(0), gh1(3), gi0a(2), gi1(4), gh0 of t+1 (1)
        stream(0, true); stream(3, false); stream(2, true); stream(4, true);
        if (t + 1 < T) stream(1, false);
      }
      stream(0, true);                                 // y(T-1)[0:6] for the last root integration
    }
  } else if (warp == W_LOAD) {
    // ================= activation loader.  Load n goes to X buffer n&1.  Re-use of an X buffer needs no handshake: a load
    // is only issued after a grid barrier whose epilogues waited on commits covering every MMA that read the old contents.
    if (lane == 0) {
      auto load = [&](const uint8_t* img, uint32_t q, uint32_t n) {
        uint8_t* X = (n & 1) ? X1 : X0;
        fence_proxy_async();
        uint32_t it = q * (uint32_t)ng;
        for (int gi = 0; gi < ng; ++gi, ++it) {
          const int kb = group_kb(gi);
          const uint32_t s = it % TC_RING, ph = (it / TC_RING) & 1;
          const uint32_t bytes = (uint32_t)((kbH - kb >= TC_GKB ? TC_GKB : kbH - kb) * 4096);
          mbar_wait(&empty[s], ph ^ 1);
          mbar_arrive_expect_tx(&full[s], bytes);
          bulk_g2s(X + (size_t)kb * 4096, img + (size_t)kb * 4096, bytes, &full[s]);
        }
      };
      load(tw.h0b[0], 0, 0);                                        // h0(0) for gh0 of step 1
      for (int t = 1; t < T; ++t) {
        const uint32_t base = 1u + 5u * (uint32_t)(t - 1);
        if (t > 1) grid_wait(w.bar, (unsigned)(3 * (t - 1)) * bar_n);           // C(t-1): h1(t-1) complete
        if (tw.dbg && t < 64) tw.dbg[((size_t)c * 64 + t) * 32 + 0] = clock64();
        load(tw.h1b[(t - 1) & 1], base, (uint32_t)(3 * t - 2));
        grid_wait(w.bar, (unsigned)(3 * (t - 1) + 1) * bar_n);                  // A(t): a(t) complete
        if (tw.dbg && t < 64) tw.dbg[((size_t)c * 64 + t) * 32 + 8] = clock64();
        load(tw.ab, base + 2, (uint32_t)(3 * t - 1));
        grid_wait(w.bar, (unsigned)(3 * (t - 1) + 2) * bar_n);                  // B(t): h0(t) complete
        if (tw.dbg && t < 64) tw.dbg[((size_t)c * 64 + t) * 32 + 14] = clock64();
        load(tw.h0b[t & 1], base + 3, (uint32_t)(3 * t));
      }
      grid_wait(w.bar, (unsigned)(3 * (T - 1)) * bar_n);
      load(tw.h1b[(T - 1) & 1], 5u * (uint32_t)(T - 1), (uint32_t)(3 * T - 2));
    }
  } else if (warp >= 4) {
    // ================= MMA warpgroup.  Group g of a chain is committed as one wgmma group; its ring slot is released once the
    // next group is issued and g has completed (one group in flight behind the issue point).
    uint32_t it = 0, n = 0;
    const uint64_t dX0 = make_smem_desc_sw128(X0), dX1 = make_smem_desc_sw128(X1), dRing = make_smem_desc_sw128(ring);
    float dF[N1 / 2], dG[NP / 2];
    auto chain_mma = [&](auto& d, float* out) {      // reads X buffer n&1, stages the sample rows of D at `out`
      constexpr int N = 2 * (int)(sizeof(d) / sizeof(float));
      const uint64_t dx = (n & 1) ? dX1 : dX0;
      const uint64_t bstep = (uint64_t)(N * 8);            // one k-block tile of the weight slice, in 16-byte units
      uint32_t prev = 0;
      for (int gi = 0; gi < ng; ++gi, ++it) {
        const int kb = group_kb(gi);
        const uint32_t s = it % TC_RING, ph = (it / TC_RING) & 1;
        mbar_wait(&full[s], ph);
        const uint64_t da = dx + (uint64_t)kb * 256, db = dRing + (uint64_t)s * (SLOT >> 4);
        const int nk = kbH - kb >= TC_GKB ? TC_GKB : kbH - kb;
        wgmma_fence();
#pragma unroll
        for (int j = 0; j < TC_GKB; ++j) {
          if (j < nk) {
#pragma unroll
            for (int ks = 0; ks < 4; ++ks)
              Wgmma<N>::mma(d, da + (uint64_t)(j * 256 + 2 * ks), db + (uint64_t)j * bstep + 2 * ks, (gi | j | ks) != 0 ? 1u : 0u);
          }
        }
        wgmma_commit();
        if (gi > 0) {
          wgmma_wait<1>();
          if (warp_lane0) mbar_arrive(&empty[prev]);
        }
        prev = s;
      }
      wgmma_wait<0>();
      wgmma_fence_operands(d);
      if (warp_lane0) mbar_arrive(&empty[prev]);
      stage_acc<N>(d, out, ACC_LD, 0, 32);
    };
    auto publish = [&](int i) {                      // every staged column so far -> epilogue
      named_bar(1, 128);
      if (threadIdx.x == 128) mbar_arrive(&d_full[i]);
    };
    chain_mma(dG, acc_gh0);                                             // gh0 of step 1 from h0(0)
    ++n;
    for (int t = 1; t < T; ++t) {
      chain_mma(dF, acc_main);                                          // fold: [pre_a ; gi0 ; y6] from h1(t-1)
      publish(0);
      TCDBG(4);
      chain_mma(dG, acc_gh1);                                           // gh1 from h1(t-1)
      ++n;
      TCDBG(10);
      chain_mma(dG, acc_main);                                          // gi0a from a(t)
      publish(1);
      ++n;
      TCDBG(11);
      chain_mma(dG, acc_main);                                          // gi1 from h0(t)
      publish(2);
      TCDBG(16);
      if (t + 1 < T) chain_mma(dG, acc_gh0);                            // gh0 of step t+1 from h0(t)
      ++n;
    }
    chain_mma(dF, acc_main);                                            // y(T-1)[0:6]
    publish(0);
  } else {
    const bool act = lane < 16;
    const int b = warp * 16 + (lane & 15);
    const bool live = act && b < a.B;
    const int j0 = c * U;
    const float* m_b = acc_main + b;
    const float* g0_b = acc_gh0 + b;
    const float* g1_b = acc_gh1 + b;
    // root state of sample b (every CTA integrates it redundantly; CTA 0 writes it out)
    V3 pos = v3(0.f, 0.f, 0.f);
    Q4 q; q.w = 1.f; q.x = q.y = q.z = 0.f;
    if (live) {
      pos = v3(a.root_pos0[b * 3 + 0], a.root_pos0[b * 3 + 1], a.root_pos0[b * 3 + 2]);
      q.w = a.root_rot0[b * 4 + 0]; q.x = a.root_rot0[b * 4 + 1]; q.y = a.root_rot0[b * 4 + 2]; q.z = a.root_rot0[b * 4 + 3];
    }
    float gi0p[3 * U];
    for (int t = 1; t <= T; ++t) {
      const uint32_t ph = (t - 1) & 1;
      const int ts = w.save ? t : (t & 1), tp = w.save ? t - 1 : ((t - 1) & 1);
      // ---------------- stage A   (operands that do not depend on the MMA are fetched before the wait)
      float sv[4 * U];
      V3 gzp = v3(0.f, 0.f, 0.f);
      if (t < T) {
        const float* S = w.S01 + ((size_t)t * 32 + (b & 31)) * 4 * H + j0;      // [t][b][4H]: U consecutive floats per gate block
#pragma unroll
        for (int qq = 0; qq < 4; ++qq) {
#pragma unroll
          for (int u4 = 0; u4 < U; u4 += 4) {
            const float4 v4 = __ldg(reinterpret_cast<const float4*>(S + (size_t)qq * H + u4));
            sv[qq * U + u4 + 0] = v4.x; sv[qq * U + u4 + 1] = v4.y; sv[qq * U + u4 + 2] = v4.z; sv[qq * U + u4 + 3] = v4.w;
          }
        }
        if (live) { const float* gp = a.gaze_pos + ((size_t)b * T + t) * 3; gzp = v3(gp[0], gp[1], gp[2]); }
      }
      mbar_wait(&d_full[0], ph);
      TCDBG(5);
      {
        // y6 columns and the fold columns (+ hoisted terms) first; the serial root / gaze chain then overlaps nothing else
        float y8[8];
        acc_ld<8>(m_b + 4 * U * ACC_LD, ACC_LD, y8);
        if (t >= 2 && t < T) {
#pragma unroll
          for (int qq = 0; qq < 4; ++qq) {
            float v[U];
            acc_ld<U>(m_b + qq * U * ACC_LD, ACC_LD, v);
#pragma unroll
            for (int u = 0; u < U; ++u) sv[qq * U + u] += v[u];
          }
        }
        float p6[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f}, gzn[3] = {0.f, 0.f, 0.f};
        if (t >= 2) {
          // y(t-1)[0:6] -> root(t-1)   (modules.py:728, :739-740); SFU sin/cos/rsqrt like the gate math of this engine
#pragma unroll
          for (int i = 0; i < 6; ++i) p6[i] = (y8[i] + c_y6[i]) * c_y6[6 + i] + c_y6[12 + i];
          const V3 npos = quat_mul_vec(q, a.dt * v3(p6[0], p6[1], p6[2])) + pos;
          const V3 hx = (0.5f * a.dt) * quat_mul_vec(q, v3(p6[3], p6[4], p6[5]));
          const float a2 = dot(hx, hx);
          Q4 e;
          if (a2 < 1e-10f) {
            const float rn = __fdividef(1.0f, sqrtf(1.0f + a2) + 1e-5f);
            e.w = rn; e.x = hx.x * rn; e.y = hx.y * rn; e.z = hx.z * rn;
          } else {
            const float ri = rsqrtf(a2), ha = a2 * ri, sc = __sinf(ha) * ri;
            e.w = __cosf(ha); e.x = hx.x * sc; e.y = hx.y * sc; e.z = hx.z * sc;
          }
          const Q4 nq = quat_mul(e, q);
          pos = npos; q = nq;
        }
        if (t == T) {
          if (c == 0 && live) {
            float* op = a.root_pos + ((size_t)b * T + (t - 1)) * 3;
            float* oq = a.root_rot + ((size_t)b * T + (t - 1)) * 4;
            op[0] = pos.x; op[1] = pos.y; op[2] = pos.z;
            oq[0] = q.w; oq[1] = q.x; oq[2] = q.y; oq[3] = q.z;
            float* y6 = w.Y6 + ((size_t)(t - 1) * 32 + b) * 8;
#pragma unroll
            for (int i = 0; i < 6; ++i) y6[i] = p6[i];
          }
          break;
        }
        float av[U];
        if (t >= 2) {
          const V3 gd = quat_mul_vec(quat_inv(q), gzp - pos);          // modules.py:696
          gzn[0] = (gd.x - c_gz[0]) * c_gz[3]; gzn[1] = (gd.y - c_gz[1]) * c_gz[4]; gzn[2] = (gd.z - c_gz[2]) * c_gz[5];
#pragma unroll
          for (int i = 0; i < 4 * U; ++i) {
            const float4 wg = *reinterpret_cast<const float4*>(c_wgz + 4 * i);
            sv[i] += wg.x * gzn[0] + wg.y * gzn[1] + wg.z * gzn[2];
          }
        }
#pragma unroll
        for (int u = 0; u < U; ++u) av[u] = sv[u] > 0.f ? sv[u] : __expf(sv[u]) - 1.0f;   // ELU (modules.py:183)
#pragma unroll
        for (int i = 0; i < 3 * U; ++i) gi0p[i] = sv[U + i];
        if (act) store_img_units<U>(tw.ab, b, j0, av);
        TCDBG(6);
        grid_arrive(w.bar);                     // only the bf16 image feeds other CTAs: publish it first ...
        TCDBG(7);
        if (act) {
#pragma unroll
          for (int u = 0; u < U; ++u) w.A[ts * actH + (size_t)(j0 + u) * 32 + b] = av[u];   // ... fp32 history afterwards
        }
        if (c == 0 && live && t >= 2) {
          float* op = a.root_pos + ((size_t)b * T + (t - 1)) * 3;
          float* oq = a.root_rot + ((size_t)b * T + (t - 1)) * 4;
          op[0] = pos.x; op[1] = pos.y; op[2] = pos.z;
          oq[0] = q.w; oq[1] = q.x; oq[2] = q.y; oq[3] = q.z;
          float* y6 = w.Y6 + ((size_t)(t - 1) * 32 + b) * 8;
#pragma unroll
          for (int i = 0; i < 6; ++i) y6[i] = p6[i];
          float* gz = w.GZ + ((size_t)t * 32 + b) * 4; gz[0] = gzn[0]; gz[1] = gzn[1]; gz[2] = gzn[2];
        }
      }
      // ---------------- stage B (GRU layer 0)
      float hp[U];
#pragma unroll
      for (int u = 0; u < U; ++u) hp[u] = w.H0[tp * actH + (size_t)(j0 + u) * 32 + (b & 31)];
      mbar_wait(&d_full[1], ph);
      TCDBG(12);
      {
        float hv[U], rr[U], zz[U], nn[U], gn[U];
        {
          float gh[U], gi[U];
          acc_ld<U>(g0_b, ACC_LD, gh); acc_ld<U>(m_b, ACC_LD, gi);
#pragma unroll
          for (int u = 0; u < U; ++u) rr[u] = fast_sigmoid(gi[u] + gi0p[u] + gh[u] + c_bhh0[u]);
          acc_ld<U>(g0_b + U * ACC_LD, ACC_LD, gh); acc_ld<U>(m_b + U * ACC_LD, ACC_LD, gi);
#pragma unroll
          for (int u = 0; u < U; ++u) zz[u] = fast_sigmoid(gi[u] + gi0p[U + u] + gh[u] + c_bhh0[U + u]);
          acc_ld<U>(g0_b + 2 * U * ACC_LD, ACC_LD, gh); acc_ld<U>(m_b + 2 * U * ACC_LD, ACC_LD, gi);
#pragma unroll
          for (int u = 0; u < U; ++u) {
            gn[u] = gh[u] + c_bhh0[2 * U + u];
            nn[u] = fast_tanh(gi[u] + gi0p[2 * U + u] + rr[u] * gn[u]);
            hv[u] = (1.f - zz[u]) * nn[u] + zz[u] * hp[u];
          }
        }
        if (act) store_img_units<U>(tw.h0b[t & 1], b, j0, hv);
        TCDBG(13);
        grid_arrive(w.bar);
        if (act) {
#pragma unroll
          for (int u = 0; u < U; ++u) w.H0[ts * actH + (size_t)(j0 + u) * 32 + b] = hv[u];
          if (w.save) {
            float* G = w.G0 + ((size_t)t * g.nbt) * 4 * H * 32;
#pragma unroll
            for (int u = 0; u < U; ++u) {
              const int j = j0 + u;
              G[(size_t)(0 * H + j) * 32 + b] = rr[u]; G[(size_t)(1 * H + j) * 32 + b] = zz[u];
              G[(size_t)(2 * H + j) * 32 + b] = nn[u]; G[(size_t)(3 * H + j) * 32 + b] = gn[u];
            }
          }
        }
      }
      // ---------------- stage C (GRU layer 1)
#pragma unroll
      for (int u = 0; u < U; ++u) hp[u] = w.H1[tp * actH + (size_t)(j0 + u) * 32 + (b & 31)];
      mbar_wait(&d_full[2], ph);
      TCDBG(17);
      {
        float hv[U], rr[U], zz[U], nn[U], gn[U];
        {
          float gh[U], gi[U];
          acc_ld<U>(g1_b, ACC_LD, gh); acc_ld<U>(m_b, ACC_LD, gi);
#pragma unroll
          for (int u = 0; u < U; ++u) rr[u] = fast_sigmoid(gi[u] + c_bih1[u] + gh[u] + c_bhh1[u]);
          acc_ld<U>(g1_b + U * ACC_LD, ACC_LD, gh); acc_ld<U>(m_b + U * ACC_LD, ACC_LD, gi);
#pragma unroll
          for (int u = 0; u < U; ++u) zz[u] = fast_sigmoid(gi[u] + c_bih1[U + u] + gh[u] + c_bhh1[U + u]);
          acc_ld<U>(g1_b + 2 * U * ACC_LD, ACC_LD, gh); acc_ld<U>(m_b + 2 * U * ACC_LD, ACC_LD, gi);
#pragma unroll
          for (int u = 0; u < U; ++u) {
            gn[u] = gh[u] + c_bhh1[2 * U + u];
            nn[u] = fast_tanh(gi[u] + c_bih1[2 * U + u] + rr[u] * gn[u]);
            hv[u] = (1.f - zz[u]) * nn[u] + zz[u] * hp[u];
          }
        }
        if (act) store_img_units<U>(tw.h1b[t & 1], b, j0, hv);
        TCDBG(18);
        grid_arrive(w.bar);
        TCDBG(19);
        if (act) {
          // bf16 row of the h1 history: A operand of the batched layer2 GEMM (rows (t,b))
          __nv_bfloat16 hb[U];
#pragma unroll
          for (int u = 0; u < U; ++u) hb[u] = __float2bfloat16_rn(hv[u]);
          __nv_bfloat16* dst = reinterpret_cast<__nv_bfloat16*>(w.H1B) + ((size_t)t * 32 + b) * H + j0;
          if (U == 8) *reinterpret_cast<uint4*>(dst) = *reinterpret_cast<const uint4*>(hb);
          else *reinterpret_cast<uint2*>(dst) = *reinterpret_cast<const uint2*>(hb);
#pragma unroll
          for (int u = 0; u < U; ++u) w.H1[ts * actH + (size_t)(j0 + u) * 32 + b] = hv[u];
          if (w.save) {
            float* G = w.G1 + ((size_t)t * g.nbt) * 4 * H * 32;
#pragma unroll
            for (int u = 0; u < U; ++u) {
              const int j = j0 + u;
              G[(size_t)(0 * H + j) * 32 + b] = rr[u]; G[(size_t)(1 * H + j) * 32 + b] = zz[u];
              G[(size_t)(2 * H + j) * 32 + b] = nn[u]; G[(size_t)(3 * H + j) * 32 + b] = gn[u];
            }
          }
        }
      }
    }
  }
}

// ------------------------------------------------------------------ after the recurrence: outputs + x_pose history
// YC[(t,b)][n] = W2[n] . h1(t)[b] + b2[n]  (batched GEMM)  ->  Y[b][t][n] = YC * os + om  (modules.py:728; channels 0..5
// take the values the in-kernel root integration used),  XP[t+1][n][b] = (Y - im) / is  (modules.py:713) and the gaze
// rows of XP[t+1] from GZ (saved for the weight gradients).  One CTA per (t, 64-channel chunk).
__global__ void __launch_bounds__(256) fold_finish_kernel(zeggs_decoder_fwd_args a, DecWs w, int nch) {
  __shared__ float tile[32][65];
  const int t = 1 + blockIdx.x, n0 = blockIdx.y * 64, T = a.T;
  const int tx = threadIdx.x & 63, ty = threadIdx.x >> 6;       // 4 rows of 64 channels per pass
  const int n = n0 + tx;
  float os = 0.f, om = 0.f;
  if (n < P_OUT) { os = a.out_std[n]; om = a.out_mean[n]; }
  for (int b = ty; b < 32; b += 4) {
    float p = 0.f;
    if (n < P_OUT) {
      p = w.YC[((size_t)(t - 1) * 32 + b) * P_OUT + n] * os + om;
      if (n < 6) p = w.Y6[((size_t)t * 32 + b) * 8 + n];
      if (b < a.B) a.Y[((size_t)b * T + t) * P_OUT + n] = p;
    }
    tile[b][tx] = p;
  }
  if (!w.save || t + 1 >= T) return;
  __syncthreads();
  float* xp = w.XP + (size_t)(t + 1) * K1P * 32;
  const int b = threadIdx.x & 31;
  for (int r = threadIdx.x >> 5; r < 64; r += 8) {
    const int nn = n0 + r;
    if (nn < P_OUT) xp[(size_t)nn * 32 + b] = (tile[b][r] - a.in_mean[nn]) / a.in_std[nn];
  }
  if (blockIdx.y == nch - 1 && threadIdx.x < 96) {
    const int d = threadIdx.x >> 5;
    xp[(size_t)(P_OUT + d) * 32 + b] = b < a.B ? w.GZ[((size_t)(t + 1) * 32 + b) * 4 + d] : 0.f;
  }
}

// cond rows for the tc engine: R[(t*32 + b)][c] = [speech[b,t,:] | style[b,t,:]] (zero rows for b >= B)
__global__ void cond_rows_kernel(zeggs_decoder_fwd_args a, float* __restrict__ R) {
  const int C = a.S + a.Z, T = a.T;
  const size_t total = (size_t)T * 32 * C;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int cc = (int)(i % C); const size_t e = i / C;
    const int b = (int)(e & 31), t = (int)(e >> 5);
    float v = 0.f;
    if (b < a.B) v = cc < a.S ? a.speech[((size_t)b * T + t) * a.S + cc] : a.style[((size_t)b * T + t) * a.Z + (cc - a.S)];
    R[i] = v;
  }
}

// ------------------------------------------------------------------ host
extern "C" size_t zeggs_decoder_packed_tc_bytes(int H, int S, int Z) {
  if (!tc_hidden_ok(H)) return 0;
  DecGeom g = make_geom(1, H, S, Z);
  return make_tcgeom(g).total_bytes;
}
extern "C" size_t zeggs_decoder_tc_workspace_bytes(int H, int S, int Z) {
  if (!tc_hidden_ok(H)) return 0;
  DecGeom g = make_geom(1, H, S, Z);
  return make_tcws(nullptr, g).bytes;
}
extern "C" int zeggs_decoder_pack_weights_tc(const zeggs_decoder_fwd_args* a, void* packed, void* stream_) {
  CtxScope ctx_scope(a ? a->ctx : nullptr);
  ZCHECK_ARG(a && packed, "decoder tc pack: bad arguments");
  ZCHECK_SUPPORTED(tc_hidden_ok(a->H), "decoder tc pack: hidden size %d unsupported (needs H %% 128 == 0, 384 <= H <= 1024)", a->H);
  ZCHECK_ARG(a->in_mean && a->in_std && a->out_mean && a->out_std, "decoder tc pack: normalisation statistics missing");
  cudaStream_t stream = (cudaStream_t)stream_;
  ScopedTimer tm_pack("weight_pack", stream);
  DecGeom g = make_geom(a->B, a->H, a->S, a->Z);
  TcGeom tg = make_tcgeom(g);
  const int H = a->H;
  uint8_t* base = (uint8_t*)packed;
  float* mfold = (float*)(base + tg.off_mfold);
  float* wxdt = (float*)(base + tg.off_wxdt);
  float* cfold = (float*)(base + tg.off_cfold);
  float* bfold = (float*)(base + tg.off_bfold);
  __nv_bfloat16* w2b = (__nv_bfloat16*)(base + tg.off_w2b);
  fold_wxdt_kernel<<<dim3(ceil_div(P_OUT, 32), ceil_div(4 * H, 32)), dim3(32, 8), 0, stream>>>(H, g.A, a->W0, a->W_ih0, a->out_std, a->in_std, wxdt);
  count_launch();
  fold_const_kernel<<<ceil_div(4 * H, 8), 256, 0, stream>>>(H, g.A, a->W0, a->W_ih0, a->b0, a->b_ih0, a->b2, a->out_std, a->out_mean,
                                                            a->in_mean, a->in_std, cfold, bfold);
  count_launch();
  ZCHECK_LAUNCH();
  // Mfold[4H][H] = WxDt^T [4H x 1131] . W2 [1131 x H]     (fp32-grade: split-bf16 tensor-core GEMM when a scratch buffer is set)
  const int fw = set_fast_wgrad_internal(0);       // the fold matrix is a weight product: always the fp32-grade 3-pass GEMM
  int rc = gemm_f32_auto(1, 4 * H, H, P_OUT, wxdt, 4 * H, a->W2, H, nullptr, mfold, H, 0, 0, stream);
  set_fast_wgrad_internal(fw);
  if (rc) return rc;
  pack_decoder_tc_kernel<<<592, 256, 0, stream>>>(g, tg, mfold, a->W_ih0, a->W_hh0, a->W_ih1, a->W_hh1, a->W2, base);
  count_launch();
  ZCHECK_CUDA(cudaMemsetAsync(w2b, 0, (size_t)round_up(P_OUT, 128) * H * 2, stream));
  rc = zeggs_split_bf16(a->W2, P_OUT, H, H, w2b, nullptr, H, stream_); if (rc) return rc;
  ZCHECK_LAUNCH();
  return ZEGGS_OK;
}

template <int U>
static int launch_tc(const zeggs_decoder_fwd_args& a, const DecGeom& g, const TcGeom& tg, const DecWs& w, const TcWs& tw,
                     const uint8_t* packed, cudaStream_t stream) {
  const size_t smem = 1024 + (size_t)2 * tg.kbH * 4096 + (size_t)TC_RING * tg.slot_bytes + 4096 + 512 +
                      (size_t)(28 * U + 26 + (2 * tg.NP + tg.N1) * TC_ACC_LD) * sizeof(float);
  constexpr int NT = 256;
  static size_t checked_smem = 0;     // attribute + co-residency check once per shared-memory size (one device per process)
  if (checked_smem != smem) {
    ZCHECK_CUDA(cudaFuncSetAttribute(decoder_fwd_tc_kernel<U>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int dev = 0, nsm = 0, occ = 0;
    ZCHECK_CUDA(cudaGetDevice(&dev));
    ZCHECK_CUDA(cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, dev));
    ZCHECK_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, decoder_fwd_tc_kernel<U>, NT, smem));
    ZCHECK_ARG(occ * nsm >= g.G, "decoder tc: cooperative grid of %d CTAs does not fit", g.G);
    checked_smem = smem;
  }
  void* args[] = {(void*)&a, (void*)&g, (void*)&tg, (void*)&w, (void*)&tw, (void*)&packed};
  ZCHECK_CUDA(cudaLaunchCooperativeKernel((void*)decoder_fwd_tc_kernel<U>, dim3(g.G), dim3(NT), args, smem, stream));
  count_launch();
  return ZEGGS_OK;
}

const float* decoder_tc_mfold(const zeggs_decoder_fwd_args& a) {
  if (!a.packed_tc) return nullptr;
  DecGeom g = make_geom(a.B, a.H, a.S, a.Z);
  return reinterpret_cast<const float*>((const uint8_t*)a.packed_tc + make_tcgeom(g).off_mfold);
}

static long long* g_tc_dbg = nullptr;
long long* tc_debug_buffer() { return g_tc_dbg; }
extern "C" void zeggs_debug_set_tc_trace(void* p) { g_tc_dbg = (long long*)p; }

// tc engine after the prologue / CellStateEncoder of zeggs_decoder_window_fwd, which has checked tc_hidden_ok(H): the hoisted speech /
// style terms, the recurrence, then layer 2 of every step at once
int decoder_fwd_tc_run(const zeggs_decoder_fwd_args& a, const DecGeom& g, const DecWs& w, cudaStream_t stream) {
  TcGeom tg = make_tcgeom(g);
  ZCHECK_ARG(g.nbt == 1, "decoder tc engine handles one 32-sample batch tile (B <= 32); got B=%d", a.B);
  ZCHECK_ARG(a.packed_tc && a.workspace_tc, "decoder tc: packed_tc / workspace_tc missing");
  const uint8_t* pk = (const uint8_t*)a.packed_tc;
  const float* cfold = (const float*)(pk + tg.off_cfold);
  const float* bfold = (const float*)(pk + tg.off_bfold);
  const int C = a.S + a.Z, H = a.H;
  // hoisted terms: S01[(t,b)][4H] = cond rows [(t,b)][C] . [W0[:, 1134:] ; W_ih0[:, H+1134:]]^T + bfold, then the first step's pose
  // contribution
  cond_rows_kernel<<<592, 256, 0, stream>>>(a, w.CONDR);
  count_launch();
  ZCHECK_LAUNCH();
  int rc = gemm_f32_auto(0, a.T * 32, H, C, w.CONDR, C, a.W0 + P_IN, g.A, bfold, w.S01, 4 * H, 0, 0, stream); if (rc) return rc;
  rc = gemm_f32_auto(0, a.T * 32, 3 * H, C, w.CONDR, C, a.W_ih0 + H + P_IN, g.A + H, bfold + H, w.S01 + H, 4 * H, 0, 0, stream); if (rc) return rc;
  fold_first_step_kernel<<<ceil_div(4 * H, 8), 256, 0, stream>>>(H, g.A, a.W0, a.W_ih0, w.XP + (size_t)K1P * 32, cfold, w.S01 + (size_t)32 * 4 * H);
  count_launch();
  ZCHECK_LAUNCH();
  TcWs tw = make_tcws(a.workspace_tc, g);
  tw.dbg = g_tc_dbg;
  // images of h0(0), h1(0) from the fp32 k-major buffers the CellStateEncoder wrote
  image_from_kmajor_kernel<<<64, 256, 0, stream>>>(w.H0, a.H, tg.kbH, tw.h0b[0]); count_launch();
  image_from_kmajor_kernel<<<64, 256, 0, stream>>>(w.H1, a.H, tg.kbH, tw.h1b[0]); count_launch();
  ZCHECK_LAUNCH();
  ScopedTimer tm("decoder_fwd", stream);
  rc = g.U == 4 ? launch_tc<4>(a, g, tg, w, tw, pk, stream) : launch_tc<8>(a, g, tg, w, tw, pk, stream);
  if (rc) return rc;
  // layer2 for every step at once: YC[(t,b)][:] = h1(t) W2^T + b2 over the bf16 history (rows t = 1..T-1)
  const __nv_bfloat16* h1b = reinterpret_cast<const __nv_bfloat16*>(w.H1B) + (size_t)32 * a.H;
  const __nv_bfloat16* w2b = reinterpret_cast<const __nv_bfloat16*>(pk + tg.off_w2b);
  rc = tc_gemm_launch((a.T - 1) * 32, P_OUT, a.H, h1b, nullptr, a.H, w2b, nullptr, a.H, a.b2, w.YC, P_OUT, 0, 0, stream); if (rc) return rc;
  const int nch = ceil_div(P_OUT, 64);
  fold_finish_kernel<<<dim3(a.T - 1, nch), 256, 0, stream>>>(a, w, nch);
  count_launch();
  ZCHECK_LAUNCH();
  return ZEGGS_OK;
}

}  // namespace zeggs
