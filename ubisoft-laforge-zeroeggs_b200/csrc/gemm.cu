// Generic fp32 SIMT GEMM for the batched (non-recurrent) linear layers and weight gradients.
//   trans_a = 0:  C[M,N] = act(A[M,K] * B[N,K]^T + bias)     (nn.Linear forward / input gradients)
//   trans_a = 1:  C[M,N] = A[K,M]^T * B[K,N] (+ C)           (weight gradients, contraction over rows)
//   trans_a = 2:  C[M,N] = A[M,K]   * B[K,N]                 (input gradients)
// 64x64x16 tiles, 256 threads, 4x4 register tile per thread.
#include "library.cuh"

namespace zeggs {

// MODE 0: A[M,K] B[N,K] (NT)   1: A[K,M] B[K,N] (TN)   2: A[M,K] B[K,N] (NN); blockIdx.z = batch
template <int MODE>
__global__ void __launch_bounds__(256) sgemm_kernel(int M, int N, int K, const float* __restrict__ A, int lda,
                                                    const float* __restrict__ B, int ldb, const float* __restrict__ bias,
                                                    float* __restrict__ C, int ldc, int act, int accumulate,
                                                    long long sA, long long sB, long long sC, int inner,
                                                    long long iA, long long iB, long long iC, float alpha) {
  { const int zo = blockIdx.z / inner, zi = blockIdx.z - zo * inner;
    A += zo * sA + zi * iA; B += zo * sB + zi * iB; C += zo * sC + zi * iC; }
  __shared__ float As[16][64 + 4];
  __shared__ float Bs[16][64 + 4];
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int m0 = blockIdx.y * 64, n0 = blockIdx.x * 64;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  for (int k0 = 0; k0 < K; k0 += 16) {
    if (MODE == 1) {
      // A[k][m], B[k][n]: 16 x 64 each, 4 elements per thread, coalesced along m / n
      for (int i = tid; i < 16 * 64; i += 256) {
        int kk = i >> 6, mm = i & 63;
        int k = k0 + kk;
        As[kk][mm] = (k < K && m0 + mm < M) ? A[(size_t)k * lda + m0 + mm] : 0.f;
        Bs[kk][mm] = (k < K && n0 + mm < N) ? B[(size_t)k * ldb + n0 + mm] : 0.f;
      }
    } else if (MODE == 2) {
      for (int i = tid; i < 16 * 64; i += 256) {
        int mm = i >> 4, kk = i & 15;
        As[kk][mm] = (k0 + kk < K && m0 + mm < M) ? A[(size_t)(m0 + mm) * lda + k0 + kk] : 0.f;
        int kb = i >> 6, nn = i & 63;
        Bs[kb][nn] = (k0 + kb < K && n0 + nn < N) ? B[(size_t)(k0 + kb) * ldb + n0 + nn] : 0.f;
      }
    } else {
      for (int i = tid; i < 16 * 64; i += 256) {
        int mm = i >> 4, kk = i & 15;
        int k = k0 + kk;
        As[kk][mm] = (k < K && m0 + mm < M) ? A[(size_t)(m0 + mm) * lda + k] : 0.f;
        Bs[kk][mm] = (k < K && n0 + mm < N) ? B[(size_t)(n0 + mm) * ldb + k] : 0.f;
      }
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < 16; ++kk) {
      float av[4], bv[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) { av[i] = As[kk][ty * 4 + i]; bv[i] = Bs[kk][tx * 4 + i]; }
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    int m = m0 + ty * 4 + i;
    if (m >= M) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      int n = n0 + tx * 4 + j;
      if (n >= N) continue;
      float v = acc[i][j] * alpha;
      if (bias) v += bias[n];
      if (act == 1) v = elu_f(v); else if (act == 2) v = fmaxf(v, 0.f);
      if (accumulate) v += C[(size_t)m * ldc + n];
      C[(size_t)m * ldc + n] = v;
    }
  }
}

// Narrow-output variant (N <= 32: the attention products P V, P^T dO, dS K, dS^T Q with 32-channel heads): 128 x 32 tile, every thread
// a 4 x 4 block (the 64 x 64 kernel would idle half its threads), 32-deep k chunks, one 128-bit shared load per operand per k.
// MODE 1: A[K,M] B[K,N] (TN)   2: A[M,K] B[K,N] (NN)
template <int MODE>
__global__ void __launch_bounds__(256) sgemm_n32_kernel(int M, int N, int K, const float* __restrict__ A, int lda,
                                                        const float* __restrict__ B, int ldb, const float* __restrict__ bias,
                                                        float* __restrict__ C, int ldc, int act, int accumulate,
                                                        long long sA, long long sB, long long sC, int inner,
                                                        long long iA, long long iB, long long iC, float alpha) {
  { const int zo = blockIdx.z / inner, zi = blockIdx.z - zo * inner;
    A += zo * sA + zi * iA; B += zo * sB + zi * iB; C += zo * sC + zi * iC; }
  __shared__ __align__(16) float As[32][128 + 4];
  __shared__ __align__(16) float Bs[32][32 + 4];
  const int tid = threadIdx.x, tx = tid & 7, ty = tid >> 3;
  const int m0 = blockIdx.y * 128;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  // register-staged software pipeline: the global loads of chunk c+1 are in flight while chunk c is multiplied out of shared memory
  float ra[16], rb[4];
  auto gload = [&](int k0) {
#pragma unroll
    for (int u = 0; u < 16; ++u) {
      const int i = tid + u * 256;
      if (MODE == 1) { const int kk = i >> 7, mm = i & 127, k = k0 + kk; ra[u] = (k < K && m0 + mm < M) ? A[(size_t)k * lda + m0 + mm] : 0.f; }
      else { const int mm = i >> 5, kk = i & 31, k = k0 + kk; ra[u] = (k < K && m0 + mm < M) ? A[(size_t)(m0 + mm) * lda + k] : 0.f; }
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int i = tid + u * 256, kk = i >> 5, nn = i & 31, k = k0 + kk;
      rb[u] = (k < K && nn < N) ? B[(size_t)k * ldb + nn] : 0.f;
    }
  };
  auto sstore = [&]() {
#pragma unroll
    for (int u = 0; u < 16; ++u) {
      const int i = tid + u * 256;
      if (MODE == 1) As[i >> 7][i & 127] = ra[u]; else As[i & 31][i >> 5] = ra[u];
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) { const int i = tid + u * 256; Bs[i >> 5][i & 31] = rb[u]; }
  };
  gload(0);
  for (int k0 = 0; k0 < K; k0 += 32) {
    sstore();
    __syncthreads();
    if (k0 + 32 < K) gload(k0 + 32);
#pragma unroll
    for (int kk = 0; kk < 32; ++kk) {
      const float4 a4 = *reinterpret_cast<const float4*>(&As[kk][ty * 4]);
      const float4 b4 = *reinterpret_cast<const float4*>(&Bs[kk][tx * 4]);
      const float av[4] = {a4.x, a4.y, a4.z, a4.w}, bv[4] = {b4.x, b4.y, b4.z, b4.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int m = m0 + ty * 4 + i;
    if (m >= M) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int n = tx * 4 + j;
      if (n >= N) continue;
      float v = acc[i][j] * alpha;
      if (bias) v += bias[n];
      if (act == 1) v = elu_f(v); else if (act == 2) v = fmaxf(v, 0.f);
      if (accumulate) v += C[(size_t)m * ldc + n];
      C[(size_t)m * ldc + n] = v;
    }
  }
}

// batch index z = zo*inner + zi; operand X is offset by zo*sX + zi*iX (e.g. zo = sample, zi = attention head)
int sgemm_batched2_launch(int mode, int M, int N, int K, const float* A, int lda, const float* B, int ldb,
                          const float* bias, float* C, int ldc, int act, int accumulate, int batch,
                          long long sA, long long sB, long long sC, int inner, long long iA, long long iB, long long iC,
                          float alpha, cudaStream_t stream) {
  ZCHECK_ARG(M > 0 && N > 0 && K > 0 && A && B && C && batch >= 1 && batch <= 65535 && inner >= 1, "sgemm: bad arguments M=%d N=%d K=%d batch=%d", M, N, K, batch);
  const bool n32 = N <= 32 && mode != 0 && M >= 128;
  // grid.y holds at most 65535 row tiles: a taller product runs as consecutive row slices, one launch each (A and C offset by the
  // slice's first row; in mode 1 a row of C is a column of A)
  const int slice = 65535 * (n32 ? 128 : 64);
  for (int m0 = 0; m0 < M; m0 += slice) {
    const int Ms = std::min(slice, M - m0);
    const float* As = A + (mode == 1 ? (size_t)m0 : (size_t)m0 * lda);
    float* Cs = C + (size_t)m0 * ldc;
    if (n32) {
      dim3 gridn(1, ceil_div(Ms, 128), batch);
      if (mode == 1) sgemm_n32_kernel<1><<<gridn, 256, 0, stream>>>(Ms, N, K, As, lda, B, ldb, bias, Cs, ldc, act, accumulate, sA, sB, sC, inner, iA, iB, iC, alpha);
      else sgemm_n32_kernel<2><<<gridn, 256, 0, stream>>>(Ms, N, K, As, lda, B, ldb, bias, Cs, ldc, act, accumulate, sA, sB, sC, inner, iA, iB, iC, alpha);
    } else {
      dim3 grid(ceil_div(N, 64), ceil_div(Ms, 64), batch);
      if (mode == 1) sgemm_kernel<1><<<grid, 256, 0, stream>>>(Ms, N, K, As, lda, B, ldb, bias, Cs, ldc, act, accumulate, sA, sB, sC, inner, iA, iB, iC, alpha);
      else if (mode == 2) sgemm_kernel<2><<<grid, 256, 0, stream>>>(Ms, N, K, As, lda, B, ldb, bias, Cs, ldc, act, accumulate, sA, sB, sC, inner, iA, iB, iC, alpha);
      else sgemm_kernel<0><<<grid, 256, 0, stream>>>(Ms, N, K, As, lda, B, ldb, bias, Cs, ldc, act, accumulate, sA, sB, sC, inner, iA, iB, iC, alpha);
    }
    count_launch();
    ZCHECK_LAUNCH();
  }
  return ZEGGS_OK;
}

int sgemm_batched_launch(int mode, int M, int N, int K, const float* A, int lda, const float* B, int ldb,
                         const float* bias, float* C, int ldc, int act, int accumulate, int batch,
                         long long sA, long long sB, long long sC, cudaStream_t stream) {
  return sgemm_batched2_launch(mode, M, N, K, A, lda, B, ldb, bias, C, ldc, act, accumulate, batch, sA, sB, sC, 1, 0, 0, 0, 1.0f, stream);
}

int sgemm_launch(int trans_a, int M, int N, int K, const float* A, int lda, const float* B, int ldb,
                 const float* bias, float* C, int ldc, int act, int accumulate, cudaStream_t stream) {
  return sgemm_batched_launch(trans_a, M, N, K, A, lda, B, ldb, bias, C, ldc, act, accumulate, 1, 0, 0, 0, stream);
}

extern "C" int zeggs_sgemm(int trans_a, int M, int N, int K, const float* A, int lda, const float* B, int ldb,
                           const float* bias, float* C, int ldc, int act, int accumulate, void* stream) {
  return sgemm_launch(trans_a, M, N, K, A, lda, B, ldb, bias, C, ldc, act, accumulate, (cudaStream_t)stream);
}

}  // namespace zeggs
