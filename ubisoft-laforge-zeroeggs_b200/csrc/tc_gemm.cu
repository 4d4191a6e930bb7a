// wgmma / TMA GEMM for the batched (non-recurrent) contractions on the path:
//   C[M,N] (f32) = sum over passes p of  A_p[M,K] (bf16, K-major) * B_p[N,K]^T (bf16, K-major)  (+bias, act)
// One 128 x BN output tile per CTA; BLOCK_K = 64 bf16 (one 128-byte swizzle atom row).
// Warp roles (288 threads): warps 0..3 and 4..7 = two consumer warpgroups (rows 0..63 / 64..127 of the tile, accumulators in
// registers, wgmma.m64n128k16 per 128 columns), warp 8 = TMA producer.
// Three passes implement the split-bf16 ("bf16x3") scheme: x = hi + lo with hi = bf16(x),
// lo = bf16(x - hi); passes (A_hi,B_hi), (A_lo,B_hi), (A_hi,B_lo) accumulate into the same accumulator,
// recovering ~fp32 product accuracy at 3x the tensor work.
#include <cuda.h>
#include <mutex>
#include "library.cuh"
#include "tc_common.cuh"

namespace zeggs {

constexpr int TG_BM = 128, TG_BK = 64;
constexpr int TG_A_BYTES = TG_BM * TG_BK * 2;
constexpr int TG_THREADS = 288;

struct TcGemmMaps {
  CUtensorMap a[2];
  CUtensorMap b[2];
};

// One-pass products stage A and B per k-block; BN = 256 (N >= 256) holds A 16 KB + B 32 KB per stage, so each A byte feeds
// twice the columns.  FUSE is the split-bf16 three-pass scheme: A_hi, A_lo, B_hi, B_lo of a k-block are staged ONCE (64 KB) and
// the three products hi*hi, lo*hi, hi*lo issued back to back from that stage.
// Epilogue: the accumulators go through a padded shared-memory tile (the pipeline stages are dead once both warpgroups have
// passed the final wait) so that the global accesses are row-contiguous, read-modify-write of C included.
template <int BN, int STAGES, bool FUSE>
__global__ void __launch_bounds__(TG_THREADS, 1)
tc_gemm_kernel(const __grid_constant__ TcGemmMaps maps, int M, int N, int K,
               const float* __restrict__ bias, float* __restrict__ C, int ldc, int act, int accumulate,
               float* __restrict__ part, int kb_per_split, int mtile0) {
  constexpr int B_BYTES = BN * TG_BK * 2;
  constexpr int NOP = FUSE ? 2 : 1;                 // operand copies per stage (hi [, lo])
  constexpr int STAGE_A = NOP * TG_A_BYTES, STAGE_B = NOP * B_BYTES;
  constexpr int NJ = BN / 128;                      // m64n128 accumulators per consumer thread
  constexpr int TLD = BN + 4;                       // staging-tile row stride (floats)
  static_assert(!(FUSE && BN != 128), "tile variant");
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sA = smem;
  uint8_t* sB = smem + STAGES * STAGE_A;
  uint64_t* full = reinterpret_cast<uint64_t*>(sB + STAGES * STAGE_B);
  uint64_t* empty = full + STAGES;

  // warp index broadcast from lane 0: provably warp-uniform, so the role branches below do not count as divergent code for wgmma
  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0), lane = threadIdx.x & 31;
  const int m0 = (blockIdx.y + mtile0) * TG_BM, n0 = blockIdx.x * BN;
  // split-K: blockIdx.z owns k-blocks [kb0, kb0 + kblocks); its raw fp32 tile goes to part[z][M][N] (reduced afterwards)
  const int kb0 = blockIdx.z * kb_per_split;
  const int kblocks = min(kb_per_split, ceil_div(K, TG_BK) - kb0);

  if (threadIdx.x == 0) {
    for (int i = 0; i < NOP; ++i) { tma_prefetch_desc(&maps.a[i]); tma_prefetch_desc(&maps.b[i]); }
    for (int s = 0; s < STAGES; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 8); }   // empty: one arrival per consumer warp
    fence_mbar_init();
  }
  __syncthreads();

  if (warp == 8) {
    if (lane == 0) {
      for (int it = 0; it < kblocks; ++it) {
        const int s = it % STAGES, ph = (it / STAGES) & 1, kb = kb0 + it;
        mbar_wait(&empty[s], ph ^ 1);
        mbar_arrive_expect_tx(&full[s], STAGE_A + STAGE_B);
        tma_load_2d(sA + s * STAGE_A, &maps.a[0], &full[s], kb * TG_BK, m0);
        tma_load_2d(sB + s * STAGE_B, &maps.b[0], &full[s], kb * TG_BK, n0);
        if (FUSE) {
          tma_load_2d(sA + s * STAGE_A + TG_A_BYTES, &maps.a[1], &full[s], kb * TG_BK, m0);
          tma_load_2d(sB + s * STAGE_B + B_BYTES, &maps.b[1], &full[s], kb * TG_BK, n0);
        }
      }
    }
    return;
  }
  // ---- consumer warpgroup wg: rows [64 wg, 64 wg + 64) of the tile
  const int wg = warp >> 2;
  float d[NJ][64];
  int prev = 0;
  for (int it = 0; it < kblocks; ++it) {
    const int s = it % STAGES, ph = (it / STAGES) & 1;
    mbar_wait(&full[s], ph);
    const uint64_t da = make_smem_desc_sw128(sA + s * STAGE_A + wg * (64 * 128));
    const uint64_t db = make_smem_desc_sw128(sB + s * STAGE_B);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < TG_BK / 16; ++k) {
      const uint32_t acc = (it | k) != 0 ? 1u : 0u;
#pragma unroll
      for (int j = 0; j < NJ; ++j) {
        const uint64_t bj = db + (uint64_t)(j * 128 * 128 / 16) + 2 * k;
        Wgmma<128>::mma(d[j], da + 2 * k, bj, acc);
        if (FUSE) {
          Wgmma<128>::mma(d[j], da + (TG_A_BYTES >> 4) + 2 * k, bj, 1u);            // lo * hi
          Wgmma<128>::mma(d[j], da + 2 * k, bj + (B_BYTES >> 4), 1u);               // hi * lo
        }
      }
    }
    wgmma_commit();
    if (it > 0) {
      wgmma_wait<1>();
      if (lane == 0) mbar_arrive(&empty[prev]);
    }
    prev = s;
  }
  wgmma_wait<0>();
#pragma unroll
  for (int j = 0; j < NJ; ++j) wgmma_fence_operands(d[j]);
  named_bar(1, 256);                                 // both warpgroups are done with every stage: reuse them as the staging tile
  float* tile = reinterpret_cast<float*>(smem) + (size_t)wg * 64 * TLD;
  {
    const int r = 16 * (warp & 3) + (lane >> 2), cc = 2 * (lane & 3);
#pragma unroll
    for (int j = 0; j < NJ; ++j) {
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        const int col = j * 128 + 8 * i + cc;
        *reinterpret_cast<float2*>(tile + (size_t)r * TLD + col) = make_float2(d[j][4 * i], d[j][4 * i + 1]);
        *reinterpret_cast<float2*>(tile + (size_t)(r + 8) * TLD + col) = make_float2(d[j][4 * i + 2], d[j][4 * i + 3]);
      }
    }
  }
  named_bar(2 + wg, 128);
  const int tid = threadIdx.x & 127;
  const int rows = min(64, M - (m0 + wg * 64));
  for (int c0 = 0; c0 < BN; c0 += 128) {
    const int cl = c0 + tid, n = n0 + cl;
    if (n >= N) continue;
    const float bv = (!part && bias) ? bias[n] : 0.f;
    if (part) {
      float* pcol = part + ((size_t)blockIdx.z * M + m0 + wg * 64) * N + n;
      for (int r = 0; r < rows; ++r) pcol[(size_t)r * N] = tile[(size_t)r * TLD + cl];
    } else {
      float* ccol = C + (size_t)(m0 + wg * 64) * ldc + n;
      for (int r0 = 0; r0 < rows; r0 += 8) {
        // read-modify-write: the 8 loads of a row group are issued before its first store (a load after a store to the same array
        // is not hoisted by the compiler)
        float cv[8];
#pragma unroll
        for (int r = 0; r < 8; ++r) cv[r] = (accumulate && r0 + r < rows) ? ccol[(size_t)(r0 + r) * ldc] : 0.f;
#pragma unroll
        for (int r = 0; r < 8; ++r) {
          if (r0 + r < rows) {
            float x = tile[(size_t)(r0 + r) * TLD + cl] + bv;
            if (act == 1) x = elu_f(x); else if (act == 2) x = fmaxf(x, 0.f);
            ccol[(size_t)(r0 + r) * ldc] = x + cv[r];
          }
        }
      }
    }
  }
}

// sum of the split-K partial tiles + the epilogue of the un-split kernel (deterministic order)
__global__ void splitk_reduce_kernel(const float* __restrict__ part, int splits, int M, int N, const float* __restrict__ bias,
                                     float* __restrict__ C, int ldc, int act, int accumulate) {
  const size_t total = (size_t)M * N;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int m = (int)(i / N), n = (int)(i % N);
    float x = 0.f;
    for (int z = 0; z < splits; ++z) x += part[(size_t)z * total + i];
    if (bias) x += bias[n];
    if (act == 1) x = elu_f(x); else if (act == 2) x = fmaxf(x, 0.f);
    float* c = C + (size_t)m * ldc + n;
    *c = accumulate ? *c + x : x;
  }
}

// fp32 -> (hi, lo) bf16 split, row-major, optional zero padding of the row to ld_out
__global__ void split_bf16_kernel(const float* __restrict__ x, int rows, int cols, int ld_in,
                                  __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo, int ld_out) {
  const size_t total = (size_t)rows * ld_out;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int r = (int)(i / ld_out), c = (int)(i % ld_out);
    float v = c < cols ? x[(size_t)r * ld_in + c] : 0.f;
    __nv_bfloat16 h = __float2bfloat16_rn(v);
    hi[i] = h;
    if (lo) lo[i] = __float2bfloat16_rn(v - __bfloat162float(h));
  }
}

// transposing split: x[rows][cols] (ld_in) -> hi/lo [cols][ld_out] (ld_out >= rows, zero padded); 32x32 tiles, blockIdx.y striding
// over the ceil(ld_out / 32) row tiles (launch with split_t_grid)
__global__ void split_bf16_t_kernel(const float* __restrict__ x, int rows, int cols, int ld_in,
                                    __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo, int ld_out) {
  __shared__ float tile[32][33];
  const int c0 = blockIdx.x * 32;
  for (int r0 = blockIdx.y * 32; r0 < ld_out; r0 += gridDim.y * 32) {
    for (int i = threadIdx.y; i < 32; i += 8) {
      const int r = r0 + i, c = c0 + threadIdx.x;
      tile[i][threadIdx.x] = (r < rows && c < cols) ? x[(size_t)r * ld_in + c] : 0.f;
    }
    __syncthreads();
    for (int i = threadIdx.y; i < 32; i += 8) {
      const int c = c0 + i, r = r0 + threadIdx.x;     // output row c, output column r
      if (c < cols && r < ld_out) {
        const float v = tile[threadIdx.x][i];
        const __nv_bfloat16 h = __float2bfloat16_rn(v);
        hi[(size_t)c * ld_out + r] = h;
        if (lo) lo[(size_t)c * ld_out + r] = __float2bfloat16_rn(v - __bfloat162float(h));
      }
    }
    __syncthreads();
  }
}

// grid of split_bf16_t_kernel: one block per 32 x 32 tile up to grid.y's limit of 65535 row tiles (2,097,120 rows), striding beyond
static dim3 split_t_grid(int cols, int ld_out) { return dim3(ceil_div(cols, 32), std::min(ceil_div(ld_out, 32), 65535)); }

// k-major history [S][R_src][32] (slot stride given) -> hi/lo [R][S*32]: out[r][s*32 + b] = in[s][r][b].
// One warp per history row r: lanes = samples b, the warp walks the slots (128 B in, 64 B out per slot, both streams
// sequential) and, when `rowsum` is given, also returns sum over slots s >= s_begin and samples of in[s][r][b] (the bias
// gradient of that row) -- fixed summation order, no atomics.
__global__ void __launch_bounds__(256) split_bf16_hist_kernel(const float* __restrict__ x, long long slot_stride, int S, int R,
                                                              __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo,
                                                              float* __restrict__ rowsum, int s_begin) {
  const int lane = threadIdx.x & 31;
  const size_t ld = (size_t)S * 32;
  for (int r = blockIdx.x * 8 + (threadIdx.x >> 5); r < R; r += gridDim.x * 8) {
    const float* src = x + (size_t)r * 32 + lane;
    __nv_bfloat16* oh = hi + (size_t)r * ld + lane;
    __nv_bfloat16* ol = lo ? lo + (size_t)r * ld + lane : nullptr;
    float acc = 0.f;
    int sidx = 0;
    for (; sidx + 8 <= S; sidx += 8) {
      float v[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) v[i] = __ldg(src + (size_t)(sidx + i) * slot_stride);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const __nv_bfloat16 h = __float2bfloat16_rn(v[i]);
        oh[(size_t)(sidx + i) * 32] = h;
        if (ol) ol[(size_t)(sidx + i) * 32] = __float2bfloat16_rn(v[i] - __bfloat162float(h));
        if (sidx + i >= s_begin) acc += v[i];
      }
    }
    for (; sidx < S; ++sidx) {
      const float v = __ldg(src + (size_t)sidx * slot_stride);
      const __nv_bfloat16 h = __float2bfloat16_rn(v);
      oh[(size_t)sidx * 32] = h;
      if (ol) ol[(size_t)sidx * 32] = __float2bfloat16_rn(v - __bfloat162float(h));
      if (sidx >= s_begin) acc += v;
    }
    if (rowsum) {
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
      if (lane == 0) rowsum[r] = acc;
    }
  }
}

// bf16 transpose: in[R][ld_in] (first Ncols columns) -> out[Ncols][ld_out]; 64x64 tiles, 4-byte accesses both ways
__global__ void __launch_bounds__(256) transpose_bf16_kernel(const uint16_t* __restrict__ in, int R, int Ncols, size_t ld_in,
                                                             uint16_t* __restrict__ out, size_t ld_out) {
  __shared__ uint16_t tile[64][66];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int r0 = blockIdx.y * 64, c0 = blockIdx.x * 64;
  for (int r = ty; r < 64; r += 8) {
    const int rr = r0 + r, cc = c0 + 2 * tx;
    uint32_t v = 0;
    if (rr < R && cc + 1 < Ncols) v = *reinterpret_cast<const uint32_t*>(in + (size_t)rr * ld_in + cc);
    else if (rr < R && cc < Ncols) v = in[(size_t)rr * ld_in + cc];
    tile[r][2 * tx] = (uint16_t)(v & 0xffffu); tile[r][2 * tx + 1] = (uint16_t)(v >> 16);
  }
  __syncthreads();
  for (int c = ty; c < 64; c += 8) {
    const int cc = c0 + c, rr = r0 + 2 * tx;
    if (cc >= Ncols) continue;
    const uint32_t v = (uint32_t)tile[2 * tx][c] | ((uint32_t)tile[2 * tx + 1][c] << 16);
    if (rr + 1 < R) *reinterpret_cast<uint32_t*>(out + (size_t)cc * ld_out + rr) = v;
    else if (rr < R) out[(size_t)cc * ld_out + rr] = (uint16_t)(v & 0xffffu);
  }
}

int transpose_bf16_launch(const __nv_bfloat16* in, int R, int Ncols, size_t ld_in, __nv_bfloat16* out, size_t ld_out, cudaStream_t stream) {
  ZCHECK_ARG((ld_in % 2) == 0 && (ld_out % 2) == 0 && ((uintptr_t)in & 3) == 0 && ((uintptr_t)out & 3) == 0, "transpose_bf16: 4-byte alignment");
  transpose_bf16_kernel<<<dim3(ceil_div(Ncols, 64), ceil_div(R, 64)), 256, 0, stream>>>((const uint16_t*)in, R, Ncols, ld_in, (uint16_t*)out, ld_out);
  count_launch();
  ZCHECK_LAUNCH();
  return ZEGGS_OK;
}

// transposing split of a weight sub-block: x[rows][cols] (ld_in) -> hi [cols][ld_out] bf16
int split_t_launch(const float* x, int rows, int cols, int ld_in, __nv_bfloat16* hi, __nv_bfloat16* lo, int ld_out, cudaStream_t stream);

static int encode_map_uncached(CUtensorMap* m, const void* base, int rows, int K, int ld_elems, int box_rows) {
  PFN_encodeTiled fn = get_encode_fn();
  ZCHECK_ARG(fn != nullptr, "tc_gemm: cuTensorMapEncodeTiled not available from the driver");
  cuuint64_t dims[2] = {(cuuint64_t)K, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)ld_elems * 2};
  cuuint32_t box[2] = {(cuuint32_t)TG_BK, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  ZCHECK_ARG(r == CUDA_SUCCESS, "tc_gemm: cuTensorMapEncodeTiled failed (%d) rows=%d K=%d ld=%d", (int)r, rows, K, ld_elems);
  return ZEGGS_OK;
}

// A tensor map describes geometry only (base, extents, strides, box), and a training step presents the same few hundred
// operand geometries every iteration (caller-owned buffers come back at the same addresses): a small direct-mapped cache
// takes the ~250 driver encodes per step off the launch path.
static int encode_map(CUtensorMap* m, const void* base, int rows, int K, int ld_elems, int box_rows) {
  struct Entry { const void* base; int rows, K, ld, box; bool valid; CUtensorMap map; };
  constexpr int NE = 1024;
  static Entry* cache = nullptr;
  static std::mutex mu;
  std::lock_guard<std::mutex> lock(mu);
  if (!cache) cache = new Entry[NE]();
  uint64_t hsh = (uint64_t)(uintptr_t)base * 0x9E3779B97F4A7C15ULL ^ ((uint64_t)rows << 40) ^ ((uint64_t)K << 20) ^ ((uint64_t)ld_elems << 4) ^ (uint64_t)box_rows;
  Entry& e = cache[(hsh >> 20) % NE];
  if (e.valid && e.base == base && e.rows == rows && e.K == K && e.ld == ld_elems && e.box == box_rows) { *m = e.map; return ZEGGS_OK; }
  int rc = encode_map_uncached(m, base, rows, K, ld_elems, box_rows);
  if (rc) return rc;
  e.base = base; e.rows = rows; e.K = K; e.ld = ld_elems; e.box = box_rows; e.map = *m; e.valid = true;
  return ZEGGS_OK;
}

int tc_gemm_launch(int M, int N, int K, const __nv_bfloat16* A_hi, const __nv_bfloat16* A_lo, int lda,
                   const __nv_bfloat16* B_hi, const __nv_bfloat16* B_lo, int ldb, const float* bias,
                   float* C, int ldc, int act, int accumulate, cudaStream_t stream, float* splitk_ws, size_t splitk_ws_bytes) {
  ZCHECK_ARG(M > 0 && N > 0 && K > 0 && A_hi && B_hi && C, "tc_gemm: bad arguments");
  ZCHECK_ARG(lda % 8 == 0 && ldb % 8 == 0, "tc_gemm: leading dimensions must be multiples of 8 bf16 (16 B)");
  ZCHECK_ARG(((uintptr_t)A_hi & 15) == 0 && ((uintptr_t)B_hi & 15) == 0, "tc_gemm: operands must be 16-byte aligned");
  // tiles: split-bf16 (hi and lo of both operands) -> fused three passes, 128x128, 3 stages; one pass -> 128x256 when N >= 256,
  // 128x128 otherwise, 4 stages
  const bool fused = A_lo && B_lo;
  const int BN = !fused && N >= 256 ? 256 : 128;
  TcGemmMaps maps;
  memset(&maps, 0, sizeof(maps));
  int rc;
  if ((rc = encode_map(&maps.a[0], A_hi, M, K, lda, TG_BM))) return rc;
  if ((rc = encode_map(&maps.b[0], B_hi, N, K, ldb, BN))) return rc;
  if (fused) {
    if ((rc = encode_map(&maps.a[1], A_lo, M, K, lda, TG_BM))) return rc;
    if ((rc = encode_map(&maps.b[1], B_lo, N, K, ldb, BN))) return rc;
  }
  auto smem_of = [](int bm, int bn, int stages, int nop) { return (size_t)1024 + (size_t)stages * nop * (bm * TG_BK * 2 + bn * TG_BK * 2) + (2 * stages + 1) * 8 + 16; };
  const size_t smem = fused ? smem_of(128, 128, 3, 2) : BN == 256 ? smem_of(128, 256, 4, 1) : smem_of(128, 128, 4, 1);
  RC(set_max_dynamic_smem(fused ? tc_gemm_kernel<128, 3, true> : BN == 128 ? tc_gemm_kernel<128, 4, false> : tc_gemm_kernel<256, 4, false>, smem));
  DeviceLimits lim;
  RC(device_limits(&lim));
  // split-K when the output has too few tiles to fill the SMs and the contraction is long: blockIdx.z writes its raw partial tile to
  // splitk_ws, and splitk_reduce_kernel sums them in a fixed order and applies the epilogue
  const int tiles = ceil_div(N, BN) * ceil_div(M, TG_BM), kblocks = ceil_div(K, TG_BK);
  int splits = 1;
  if (splitk_ws && tiles <= lim.sms / 2 && kblocks >= 8) {
    splits = std::min(std::max(1, lim.sms / tiles), kblocks / 2);
    const size_t per = (size_t)M * N * sizeof(float);
    if ((size_t)splits * per > splitk_ws_bytes) splits = (int)(splitk_ws_bytes / per);
    splits = std::max(splits, 1);
  }
  const int kbs = ceil_div(kblocks, splits);
  splits = ceil_div(kblocks, kbs);                        // every z gets at least one k-block
  float* const part = splits > 1 ? splitk_ws : nullptr;
  // with `part` set the kernel stores the raw tile and leaves bias, act and accumulate to the reduction.  grid.y holds at most 65535
  // row tiles: a taller product runs as consecutive slices of row tiles, one launch each, starting at row tile t0
  const int mtiles = ceil_div(M, TG_BM);
  for (int t0 = 0; t0 < mtiles; t0 += 65535) {
    const dim3 grid(ceil_div(N, BN), std::min(mtiles - t0, 65535), splits);
    if (fused) tc_gemm_kernel<128, 3, true><<<grid, TG_THREADS, smem, stream>>>(maps, M, N, K, bias, C, ldc, act, accumulate, part, kbs, t0);
    else if (BN == 256) tc_gemm_kernel<256, 4, false><<<grid, TG_THREADS, smem, stream>>>(maps, M, N, K, bias, C, ldc, act, accumulate, part, kbs, t0);
    else tc_gemm_kernel<128, 4, false><<<grid, TG_THREADS, smem, stream>>>(maps, M, N, K, bias, C, ldc, act, accumulate, part, kbs, t0);
    count_launch();
  }
  if (part) {
    const size_t total = (size_t)M * N;
    splitk_reduce_kernel<<<(int)std::min<size_t>(1184, (total + 255) / 256), 256, 0, stream>>>(part, splits, M, N, bias, C, ldc, act, accumulate);
    count_launch();
  }
  ZCHECK_LAUNCH();
  return ZEGGS_OK;
}

int split_t_launch(const float* x, int rows, int cols, int ld_in, __nv_bfloat16* hi, __nv_bfloat16* lo, int ld_out, cudaStream_t stream) {
  split_bf16_t_kernel<<<split_t_grid(cols, ld_out), dim3(32, 8), 0, stream>>>(x, rows, cols, ld_in, hi, lo, ld_out);
  count_launch();
  ZCHECK_LAUNCH();
  return ZEGGS_OK;
}

// ------------------------------------------------------------------ fp32-in / fp32-out front end
// The context of the entry point currently executing on this host thread (CtxScope in library.cuh): per-call state passed
// by the caller.  Calls that pass none get k_no_ctx: no scratch, so products run on the fp32 SIMT kernel and convolutions take the
// im2col path.
static const zeggs_ctx k_no_ctx = {nullptr, 0, 1, 0};
static thread_local const zeggs_ctx* tl_ctx = &k_no_ctx;
const zeggs_ctx* swap_ctx(const zeggs_ctx* c) { const zeggs_ctx* old = tl_ctx; tl_ctx = c; return old; }
int gemm_mode() { return tl_ctx->gemm_mode; }
char* scratch_base() { return (char*)tl_ctx->scratch; }
size_t scratch_bytes() { return tl_ctx->scratch_bytes; }

int split_hist_launch(const float* x, long long slot_stride, int S, int R, __nv_bfloat16* hi, __nv_bfloat16* lo, cudaStream_t stream,
                      float* rowsum, int s_begin) {
  split_bf16_hist_kernel<<<std::min(ceil_div(R, 8), 1184), 256, 0, stream>>>(x, slot_stride, S, R, hi, lo, rowsum, s_begin);
  count_launch();
  ZCHECK_LAUNCH();
  return ZEGGS_OK;
}

// bf16 operands of one tensor-core product, carved from the scratch buffer in this order: Ah [rows_a][Kp], Bh [rows_b][Kp], then
// (three-pass products only) Al, Bl, each rounded up to 256 bytes.  The split-K partial tiles get the rest of the buffer, so the
// carve fixes the split count and with it the summation order.
struct TcOperands {
  __nv_bfloat16 *Ah, *Bh, *Al, *Bl;   // Al = Bl = nullptr for a one-pass product
  float* ws;
  size_t ws_bytes;
};

// The rule for which arithmetic a product of the front end gets, given the active context.  A product runs on the tensor cores
// when the context is in GEMM mode 1, has scratch, the product has at least 4e6 multiply-adds and its operand copies fit the
// scratch; it is then split-bf16 (three passes, ~fp32 accuracy), or one bf16 pass for a weight gradient when the context sets
// fast_wgrad.  -> ZEGGS_OK with *op carved; ZEGGS_CONV_NOT_TAKEN when the product belongs on the SIMT path; ZEGGS_ERR_ARG for a
// GEMM mode other than 0 or 1.
static int plan_tc_operands(int rows_a, int rows_b, int Kp, double macs, bool wgrad, TcOperands* op) {
  const zeggs_ctx& c = *tl_ctx;
  ZCHECK_ARG(c.gemm_mode == 0 || c.gemm_mode == 1, "zeggs_ctx.gemm_mode must be 0 (fp32 SIMT) or 1 (tensor-core split-bf16), got %d",
             c.gemm_mode);
  if (c.gemm_mode == 0 || c.scratch == nullptr || macs < 4.0e6) return ZEGGS_CONV_NOT_TAKEN;
  const bool lo = !(wgrad && c.fast_wgrad);
  Arena a{(char*)c.scratch};
  op->Ah = (__nv_bfloat16*)a.bytes((size_t)rows_a * Kp * 2);
  op->Bh = (__nv_bfloat16*)a.bytes((size_t)rows_b * Kp * 2);
  op->Al = lo ? (__nv_bfloat16*)a.bytes((size_t)rows_a * Kp * 2) : nullptr;
  op->Bl = lo ? (__nv_bfloat16*)a.bytes((size_t)rows_b * Kp * 2) : nullptr;
  a.align(256);
  if (a.off > c.scratch_bytes) return ZEGGS_CONV_NOT_TAKEN;
  op->ws = (float*)a.here();
  op->ws_bytes = a.rest(c.scratch_bytes);
  return ZEGGS_OK;
}

// mode 0: C = act(A[M,K] B[N,K]^T + bias);  1: C = A[K,M]^T B[K,N];  2: C = A[M,K] B[K,N]   (all fp32, row-major)
// Mode 1 is the layout of the weight gradients.  plan_tc_operands picks the tensor cores or the fp32 SIMT kernel.
int gemm_f32_auto(int mode, int M, int N, int K, const float* A, int lda, const float* B, int ldb, const float* bias,
                  float* C, int ldc, int act, int accumulate, cudaStream_t stream) {
  const int Kp = round_up(K, 8);
  TcOperands op;
  const int rc = plan_tc_operands(M, N, Kp, (double)M * N * K, mode == 1, &op);
  if (rc == ZEGGS_CONV_NOT_TAKEN) return sgemm_launch(mode, M, N, K, A, lda, B, ldb, bias, C, ldc, act, accumulate, stream);
  if (rc) return rc;
  const dim3 tb(32, 8);
  if (mode == 1) split_bf16_t_kernel<<<split_t_grid(M, Kp), tb, 0, stream>>>(A, K, M, lda, op.Ah, op.Al, Kp);
  else split_bf16_kernel<<<592, 256, 0, stream>>>(A, M, K, lda, op.Ah, op.Al, Kp);
  count_launch();
  if (mode == 0) split_bf16_kernel<<<592, 256, 0, stream>>>(B, N, K, ldb, op.Bh, op.Bl, Kp);
  else split_bf16_t_kernel<<<split_t_grid(N, Kp), tb, 0, stream>>>(B, K, N, ldb, op.Bh, op.Bl, Kp);
  count_launch();
  ZCHECK_LAUNCH();
  return tc_gemm_launch(M, N, K, op.Ah, op.Al, Kp, op.Bh, op.Bl, Kp, bias, C, ldc, act, accumulate, stream, op.ws, op.ws_bytes);
}

// ------------------------------------------------------------------ convolution operands without a materialised im2col matrix
// The 1-D convolutions of the encoders are GEMMs over col[(b,t)][c*k + kk] = x[b][t + kk - pad][c].  Writing col in fp32 and splitting
// it to bf16 afterwards moved the k-fold expanded matrix three times (write fp32, read fp32, write bf16); these producers write the bf16
// (hi, lo) operand of the GEMM straight from x -- row-major for the forward product, transposed ([c*k+kk][(b,t)]) for the weight gradient.
__global__ void im2col_split_kernel(const float* __restrict__ x, int B, int T, int C, int k, int pad, int replicate,
                                    __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo, int ld_out) {
  // one output row (b,t) per block iteration, threads over column pairs: 32-bit index arithmetic only (a flat 64-bit index with two
  // divisions per element pair made the first version issue-bound at 1.4 TB/s)
  const int half = ld_out >> 1, K = C * k, M = B * T;
  for (int m = blockIdx.x; m < M; m += gridDim.x) {
    const int b = m / T, t = m - b * T;
    const float* xb = x + (size_t)b * T * C;
    __nv_bfloat16* hrow = hi + (size_t)m * ld_out;
    __nv_bfloat16* lrow = lo ? lo + (size_t)m * ld_out : nullptr;
    for (int j2 = threadIdx.x; j2 < half; j2 += blockDim.x) {
      const int j = 2 * j2;
      float v[2];
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int col = j + e;
        v[e] = 0.f;
        if (col < K) {
          const int c = col / k, kk = col - c * k;
          int sidx = t + kk - pad;
          if (replicate) { sidx = sidx < 0 ? 0 : (sidx >= T ? T - 1 : sidx); v[e] = xb[sidx * C + c]; }
          else if (sidx >= 0 && sidx < T) v[e] = xb[sidx * C + c];
        }
      }
      const __nv_bfloat16 h0 = __float2bfloat16_rn(v[0]), h1 = __float2bfloat16_rn(v[1]);
      __nv_bfloat162 hh; hh.x = h0; hh.y = h1;
      *reinterpret_cast<__nv_bfloat162*>(hrow + j) = hh;
      if (lrow) {
        __nv_bfloat162 ll; ll.x = __float2bfloat16_rn(v[0] - __bfloat162float(h0)); ll.y = __float2bfloat16_rn(v[1] - __bfloat162float(h1));
        *reinterpret_cast<__nv_bfloat162*>(lrow + j) = ll;
      }
    }
  }
}
// transposed: hi/lo[c*k + kk][m] (ld_out >= B*T, zero padded); grid (ceil(C/32), ceil(ld_out/128), k), block (32, 8):
// a block moves 32 channels x 128 rows, so every output row segment is 256 contiguous bytes (the 32 x 32 version wrote 64-byte pieces)
__global__ void im2col_split_t_kernel(const float* __restrict__ x, int B, int T, int C, int k, int pad, int replicate,
                                      __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo, int ld_out) {
  __shared__ float tile[128][33];
  const int kk = blockIdx.z, c0 = blockIdx.x * 32, m0 = blockIdx.y * 128, M = B * T;
  for (int i = threadIdx.y; i < 128; i += 8) {
    const int m = m0 + i, c = c0 + threadIdx.x;
    float v = 0.f;
    if (m < M && c < C) {
      const int b = m / T, t = m - b * T;
      int sidx = t + kk - pad;
      if (replicate) { sidx = sidx < 0 ? 0 : (sidx >= T ? T - 1 : sidx); v = x[((size_t)b * T + sidx) * C + c]; }
      else if (sidx >= 0 && sidx < T) v = x[((size_t)b * T + sidx) * C + c];
    }
    tile[i][threadIdx.x] = v;
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += 8) {
    const int c = c0 + i;
    if (c >= C) continue;
    const size_t o = ((size_t)c * k + kk) * ld_out;
#pragma unroll
    for (int j = 0; j < 2; ++j) {                  // two rows per thread: 4-byte stores, 128 bytes per warp instruction (ld_out % 8 == 0)
      const int mm = j * 64 + 2 * threadIdx.x, m = m0 + mm;
      if (m < ld_out) {
        const float v0 = tile[mm][i], v1 = tile[mm + 1][i];
        __nv_bfloat162 hh; hh.x = __float2bfloat16_rn(v0); hh.y = __float2bfloat16_rn(v1);
        *reinterpret_cast<__nv_bfloat162*>(hi + o + m) = hh;
        if (lo) {
          __nv_bfloat162 ll; ll.x = __float2bfloat16_rn(v0 - __bfloat162float(hh.x)); ll.y = __float2bfloat16_rn(v1 - __bfloat162float(hh.y));
          *reinterpret_cast<__nv_bfloat162*>(lo + o + m) = ll;
        }
      }
    }
  }
}

// y[(b,t)][n] = act(sum_{c,kk} x[b][t+kk-pad][c] W[n][c*k+kk] + bias[n]) on the tensor cores; ZEGGS_CONV_NOT_TAKEN when the tensor-core front end
// does not apply (fp32 SIMT mode, no / too small scratch): the caller then runs im2col + the generic product.
int conv_gemm_fwd(const float* x, int B, int T, int C, int k, int pad, int replicate, const float* W, const float* bias, float* y, int N,
                  int act, cudaStream_t stream) {
  const int M = B * T, K = C * k, Kp = round_up(K, 8);
  TcOperands op;
  const int rc = plan_tc_operands(M, N, Kp, (double)M * N * K, false, &op);
  if (rc) return rc;
  DeviceLimits lim;
  RC(device_limits(&lim));
  im2col_split_kernel<<<std::min(M, lim.sms * 16), 256, 0, stream>>>(x, B, T, C, k, pad, replicate, op.Ah, op.Al, Kp);
  count_launch();
  split_bf16_kernel<<<592, 256, 0, stream>>>(W, N, K, K, op.Bh, op.Bl, Kp);
  count_launch();
  ZCHECK_LAUNCH();
  return tc_gemm_launch(M, N, K, op.Ah, op.Al, Kp, op.Bh, op.Bl, Kp, bias, y, N, act, 0, stream, op.ws, op.ws_bytes);
}

// dW[n][c*k+kk] = sum_{(b,t)} dpre[(b,t)][n] x[b][t+kk-pad][c]
int conv_gemm_wgrad(const float* dpre, int N, const float* x, int B, int T, int C, int k, int pad, int replicate, float* dW, cudaStream_t stream) {
  const int M = B * T, K = C * k, Mp = round_up(M, 8);
  TcOperands op;
  const int rc = plan_tc_operands(N, K, Mp, (double)M * N * K, true, &op);
  if (rc) return rc;
  const dim3 tb(32, 8);
  split_bf16_t_kernel<<<split_t_grid(N, Mp), tb, 0, stream>>>(dpre, M, N, N, op.Ah, op.Al, Mp);
  count_launch();
  im2col_split_t_kernel<<<dim3(ceil_div(C, 32), ceil_div(Mp, 128), k), tb, 0, stream>>>(x, B, T, C, k, pad, replicate, op.Bh, op.Bl, Mp);
  count_launch();
  ZCHECK_LAUNCH();
  return tc_gemm_launch(N, K, M, op.Ah, op.Al, Mp, op.Bh, op.Bl, Mp, nullptr, dW, K, 0, 0, stream, op.ws, op.ws_bytes);
}

extern "C" int zeggs_gemm_f32_ctx(const zeggs_ctx* ctx, int mode, int M, int N, int K, const float* A, int lda, const float* B, int ldb,
                                  const float* bias, float* C, int ldc, int act, int accumulate, void* stream) {
  CtxScope scope(ctx);
  return gemm_f32_auto(mode, M, N, K, A, lda, B, ldb, bias, C, ldc, act, accumulate, (cudaStream_t)stream);
}

extern "C" int zeggs_tc_gemm_bf16(int M, int N, int K, const void* A_hi, const void* A_lo, int lda, const void* B_hi,
                                  const void* B_lo, int ldb, const float* bias, float* C, int ldc, int act,
                                  int accumulate, void* stream) {
  return tc_gemm_launch(M, N, K, (const __nv_bfloat16*)A_hi, (const __nv_bfloat16*)A_lo, lda, (const __nv_bfloat16*)B_hi,
                        (const __nv_bfloat16*)B_lo, ldb, bias, C, ldc, act, accumulate, (cudaStream_t)stream);
}

extern "C" int zeggs_split_bf16(const float* x, int rows, int cols, int ld_in, void* hi, void* lo, int ld_out, void* stream) {
  ZCHECK_ARG(x && hi && rows > 0 && cols > 0 && ld_out >= cols, "split_bf16: bad arguments");
  split_bf16_kernel<<<592, 256, 0, (cudaStream_t)stream>>>(x, rows, cols, ld_in, (__nv_bfloat16*)hi, (__nv_bfloat16*)lo, ld_out);
  count_launch();
  ZCHECK_LAUNCH();
  return ZEGGS_OK;
}

}  // namespace zeggs
