// Style embedding space statistics (include/zeggs_b200.h, zeggs_embedding_moments): float64 mean, covariance and per-group sums of
// N float32 embedding rows, for zeggs_b200.style_space.  Beyond the reference, which has no such statistics.
//
//   pass 1  embed_group_partial_kernel  CTA (slice, 128 columns): per-group column sums of its slice, in row order, in shared memory
//           embed_mean_kernel           group sums = partials in slice order; mean = group sums in group order / N; counts
//   pass 2  embed_cov_partial_kernel    CTA (upper-triangle 64x64 tile, slice): sum over its rows of (x_i - mean_i)(x_j - mean_j)
//           embed_cov_kernel            partials in slice order / (N - 1), written to (i, j) and (j, i) from the same sum
// Every partial goes through the caller's workspace and no atomics are used, so the result does not depend on scheduling.
#include <algorithm>

#include "library.cuh"

namespace zeggs {
namespace {

constexpr int kGroupCols = 128;   // columns of one pass-1 CTA (one thread each)
constexpr int kTile = 64;         // covariance tile edge
constexpr int kRowsPerStage = 16; // rows of centred data staged in shared memory per step of pass 2

struct Slicing {
  long long S, R;  // slices, rows per slice (the last may be shorter)
  int nb, tiles;   // 64-column blocks, upper-triangle tiles
};

Slicing slicing(long long N, int Z) {
  Slicing s;
  s.nb = (Z + kTile - 1) / kTile;
  s.tiles = s.nb * (s.nb + 1) / 2;
  const long long s0 = std::min((N + 255) / 256, (long long)std::max(1, 512 / s.tiles));
  s.R = (N + s0 - 1) / s0;
  s.S = (N + s.R - 1) / s.R;
  return s;
}

struct EmbedWs {
  double* part_sum;      // [S][G][Z]
  long long* part_cnt;   // [S][G]
  double* part_cov;      // [S][tiles][64][64]
  size_t bytes;
};

EmbedWs embed_ws(void* base, const Slicing& sl, int Z, int G) {
  Arena ar{(char*)base};
  EmbedWs w;
  w.part_sum = (double*)ar.bytes(sizeof(double) * (size_t)sl.S * G * Z);
  w.part_cnt = (long long*)ar.bytes(sizeof(long long) * (size_t)sl.S * G);
  w.part_cov = (double*)ar.bytes(sizeof(double) * (size_t)sl.S * sl.tiles * kTile * kTile);
  w.bytes = ar.off;
  return w;
}

// upper-triangle tile t -> (ib, jb), ib <= jb, numbered row by row
__device__ inline void tile_coords(int t, int nb, int& ib, int& jb) {
  ib = 0;
  while (t >= nb - ib) { t -= nb - ib; ++ib; }
  jb = ib + t;
}

__device__ inline int tile_index(int ib, int jb, int nb) { return ib * nb - ib * (ib - 1) / 2 + (jb - ib); }

__global__ void __launch_bounds__(kGroupCols) embed_group_partial_kernel(const float* __restrict__ X, const int* __restrict__ group,
                                                                         long long N, int Z, int G, long long R,
                                                                         double* __restrict__ part_sum, long long* __restrict__ part_cnt) {
  extern __shared__ double acc[];   // [G][kGroupCols]: each thread owns one column of it
  const int tid = threadIdx.x, c = blockIdx.y * kGroupCols + tid;
  const long long s = blockIdx.x, r0 = s * R, r1 = min(N, r0 + R);
  for (int g = 0; g < G; ++g) acc[g * kGroupCols + tid] = 0.0;
  if (c < Z) {
    for (long long r = r0; r < r1; ++r) {
      const int g = __ldg(group + r);
      if ((unsigned)g < (unsigned)G) acc[g * kGroupCols + tid] += (double)__ldg(X + r * Z + c);
    }
    for (int g = 0; g < G; ++g) part_sum[((size_t)s * G + g) * Z + c] = acc[g * kGroupCols + tid];
  }
  if (blockIdx.y == 0) {
    for (int g = tid; g < G; g += kGroupCols) {
      long long n = 0;
      for (long long r = r0; r < r1; ++r) n += __ldg(group + r) == g;
      part_cnt[s * G + g] = n;
    }
  }
}

__global__ void __launch_bounds__(kGroupCols) embed_mean_kernel(long long N, int Z, int G, long long S, const double* __restrict__ part_sum,
                                                                const long long* __restrict__ part_cnt, double* __restrict__ mean,
                                                                double* __restrict__ group_sum, long long* __restrict__ group_count) {
  const int c = blockIdx.x * kGroupCols + threadIdx.x;
  if (c < Z) {
    double tot = 0.0;
    for (int g = 0; g < G; ++g) {
      double sg = 0.0;
      for (long long s = 0; s < S; ++s) sg += part_sum[((size_t)s * G + g) * Z + c];
      group_sum[(size_t)g * Z + c] = sg;
      tot += sg;
    }
    mean[c] = tot / (double)N;
  }
  if (blockIdx.x == 0) {
    for (int g = threadIdx.x; g < G; g += kGroupCols) {
      long long n = 0;
      for (long long s = 0; s < S; ++s) n += part_cnt[s * G + g];
      group_count[g] = n;
    }
  }
}

// 256 threads: thread (ty, tx) = (tid / 16, tid % 16) accumulates rows ty + 16 a and columns tx + 16 b (a, b < 4) of the tile, so the
// 16 threads of a half-warp read 16 consecutive doubles of the staged column block (no bank conflicts) and the i-side is a broadcast.
__global__ void __launch_bounds__(256) embed_cov_partial_kernel(const float* __restrict__ X, long long N, int Z, int nb, long long R,
                                                                const double* __restrict__ mean, double* __restrict__ part_cov) {
  __shared__ double As[kRowsPerStage][kTile], Bs[kRowsPerStage][kTile];
  int ib, jb;
  tile_coords(blockIdx.x, nb, ib, jb);
  const int tid = threadIdx.x, ty = tid >> 4, tx = tid & 15;
  const long long s = blockIdx.y, r0 = s * R, r1 = min(N, r0 + R);
  double acc[4][4] = {};
  for (long long rb = r0; rb < r1; rb += kRowsPerStage) {
    for (int e = tid; e < kRowsPerStage * kTile; e += 256) {
      const int k = e / kTile, col = e % kTile;
      const long long r = rb + k;
      const int ci = ib * kTile + col, cj = jb * kTile + col;
      As[k][col] = (r < r1 && ci < Z) ? (double)__ldg(X + r * Z + ci) - mean[ci] : 0.0;
      Bs[k][col] = (r < r1 && cj < Z) ? (double)__ldg(X + r * Z + cj) - mean[cj] : 0.0;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < kRowsPerStage; ++k) {
      double a[4], b[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) { a[q] = As[k][ty + 16 * q]; b[q] = Bs[k][tx + 16 * q]; }
#pragma unroll
      for (int p = 0; p < 4; ++p)
#pragma unroll
        for (int q = 0; q < 4; ++q) acc[p][q] = fma(a[p], b[q], acc[p][q]);
    }
    __syncthreads();
  }
  double* out = part_cov + ((size_t)s * gridDim.x + blockIdx.x) * kTile * kTile;
#pragma unroll
  for (int p = 0; p < 4; ++p)
#pragma unroll
    for (int q = 0; q < 4; ++q) out[(ty + 16 * p) * kTile + tx + 16 * q] = acc[p][q];
}

__global__ void __launch_bounds__(256) embed_cov_kernel(long long N, int Z, int nb, int tiles, long long S,
                                                        const double* __restrict__ part_cov, double* __restrict__ cov) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= (long long)Z * Z) return;
  const int r = (int)(e / Z), c = (int)(e % Z);
  const int i = min(r, c), j = max(r, c);
  const size_t off = (size_t)tile_index(i / kTile, j / kTile, nb) * kTile * kTile + (i % kTile) * kTile + j % kTile;
  double sum = 0.0;
  for (long long s = 0; s < S; ++s) sum += part_cov[(size_t)s * tiles * kTile * kTile + off];
  cov[e] = sum / (double)(N - 1);
}

}  // namespace
}  // namespace zeggs

using namespace zeggs;

extern "C" size_t zeggs_embedding_moments_workspace_size(long long N, int Z, int G) {
  if (N < 1 || Z < 1 || Z > ZEGGS_EMBED_MAX_Z || G < 1 || G > ZEGGS_EMBED_MAX_GROUPS) return 0;
  return embed_ws(nullptr, slicing(N, Z), Z, G).bytes;
}

extern "C" int zeggs_embedding_moments(const zeggs_embedding_moments_args* ap, void* stream) {
  ZCHECK_ARG(ap, "embedding moments: null args");
  const zeggs_embedding_moments_args& a = *ap;
  ZCHECK_ARG(a.N >= 1, "embedding moments: N = %lld rows, at least 1 is needed", a.N);
  ZCHECK_ARG(a.Z >= 1 && a.Z <= ZEGGS_EMBED_MAX_Z, "embedding moments: Z = %d (1..%d)", a.Z, ZEGGS_EMBED_MAX_Z);
  ZCHECK_ARG(a.G >= 1 && a.G <= ZEGGS_EMBED_MAX_GROUPS, "embedding moments: G = %d groups (1..%d)", a.G, ZEGGS_EMBED_MAX_GROUPS);
  ZCHECK_ARG(a.X && a.group && a.mean && a.cov && a.group_sum && a.group_count && a.workspace, "embedding moments: null pointer");
  const Slicing sl = slicing(a.N, a.Z);
  const EmbedWs w = embed_ws(a.workspace, sl, a.Z, a.G);
  ZCHECK_ARG(a.workspace_bytes >= w.bytes, "embedding moments: workspace %zu < %zu bytes", a.workspace_bytes, w.bytes);
  cudaStream_t s = (cudaStream_t)stream;
  const size_t smem = sizeof(double) * kGroupCols * a.G;
  RC(set_max_dynamic_smem(embed_group_partial_kernel, smem));
  const unsigned col_blocks = (unsigned)ceil_div(a.Z, kGroupCols);
  embed_group_partial_kernel<<<dim3((unsigned)sl.S, col_blocks), kGroupCols, smem, s>>>(a.X, a.group, a.N, a.Z, a.G, sl.R, w.part_sum,
                                                                                        w.part_cnt);
  LAUNCH_OK();
  embed_mean_kernel<<<col_blocks, kGroupCols, 0, s>>>(a.N, a.Z, a.G, sl.S, w.part_sum, w.part_cnt, a.mean, a.group_sum, a.group_count);
  LAUNCH_OK();
  embed_cov_partial_kernel<<<dim3((unsigned)sl.tiles, (unsigned)sl.S), 256, 0, s>>>(a.X, a.N, a.Z, sl.nb, sl.R, a.mean, w.part_cov);
  LAUNCH_OK();
  const long long zz = (long long)a.Z * a.Z;
  embed_cov_kernel<<<(unsigned)((zz + 255) / 256), 256, 0, s>>>(a.N, a.Z, sl.nb, sl.tiles, sl.S, w.part_cov, a.cov);
  LAUNCH_OK();
  return ZEGGS_OK;
}
