// SpeechEncoder (ZEGGS/modules.py:249-272) and StyleEncoder (attn + VAE, modules.py:278-304, 346-420,
// 445-651) forward and backward.  Every convolution is lowered to im2col + GEMM (the GEMM engine is shared
// with the decoder's batched contractions); normalisation, attention softmax, dropout-mask application,
// pooling and the VAE sample are small row-wise kernels.  One C-ABI call per module direction; all
// intermediates live in the caller's workspace (they are the "saved tensors" of the backward).
// Dropout masks are explicit multiplier tensors (0 or 1/(1-p)) supplied by the caller (NULL = eval mode).
#include "library.cuh"

namespace zeggs {

// ------------------------------------------------------------------ small kernels
// col[(b,t)][c*k + kk] = x[b][t + kk - pad][c]  (zero or replicate padding);  x: [B,T,C]
__global__ void im2col_kernel(const float* __restrict__ x, int B, int T, int C, int k, int pad, int replicate, float* __restrict__ col) {
  const size_t total = (size_t)B * T * C * k;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    int kk = i % k; size_t e = i / k;
    int c = e % C; e /= C;
    int t = e % T; int b = e / T;
    int s = t + kk - pad;
    float v = 0.f;
    if (replicate) { s = s < 0 ? 0 : (s >= T ? T - 1 : s); v = x[((size_t)b * T + s) * C + c]; }
    else if (s >= 0 && s < T) v = x[((size_t)b * T + s) * C + c];
    col[i] = v;
  }
}
// adjoint of im2col: dx[b][s][c] = sum over (t,kk) that read x[b][s][c]
__global__ void col2im_kernel(const float* __restrict__ dcol, int B, int T, int C, int k, int pad, int replicate, float* __restrict__ dx) {
  const size_t total = (size_t)B * T * C;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    int c = i % C; size_t e = i / C;
    int s = e % T; int b = e / T;
    float acc = 0.f;
    for (int kk = 0; kk < k; ++kk) {
      int t = s - kk + pad;
      if (t >= 0 && t < T) acc += dcol[((size_t)b * T + t) * C * k + (size_t)c * k + kk];
    }
    if (replicate) {
      if (s == 0) {          // reads with t + kk - pad < 0
        for (int kk = 0; kk < k; ++kk)
          for (int t = 0; t < T && t + kk - pad < 0; ++t) acc += dcol[((size_t)b * T + t) * C * k + (size_t)c * k + kk];
      }
      if (s == T - 1) {      // reads with t + kk - pad > T-1
        for (int kk = 0; kk < k; ++kk)
          for (int t = T - 1; t >= 0 && t + kk - pad > T - 1; --t) acc += dcol[((size_t)b * T + t) * C * k + (size_t)c * k + kk];
      }
    }
    dx[i] = acc;
  }
}
// dst = a * (mask ? mask : 1) * (y ? act'(y) : 1)      actgrad: 1 = ELU' from output, 2 = ReLU' from output
__global__ void ew_mul_kernel(float* __restrict__ dst, const float* __restrict__ a, const float* __restrict__ mask,
                              const float* __restrict__ y, int actgrad, size_t n) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    float v = a[i];
    if (mask) v *= mask[i];
    if (y) { float yy = y[i]; v *= (actgrad == 1) ? (yy > 0.f ? 1.f : yy + 1.f) : (yy > 0.f ? 1.f : 0.f); }
    dst[i] = v;
  }
}
// dst = a + b (b optional broadcast over batch with period `period` elements; period 0 = same shape)
__global__ void ew_add_kernel(float* __restrict__ dst, const float* __restrict__ a, const float* __restrict__ b, size_t n, size_t period) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    dst[i] = a[i] + b[period ? i % period : i];
}
// LayerNorm over the last dim (nn.LayerNorm, eps 1e-5, biased variance).  One warp per row.
// in = a (+ res);  saves xhat and rstd for the backward.
__global__ void layernorm_fwd_kernel(const float* __restrict__ a, const float* __restrict__ res, const float* __restrict__ gamma,
                                     const float* __restrict__ beta, int rows, int D, float* __restrict__ y,
                                     float* __restrict__ xhat, float* __restrict__ rstd) {
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= rows) return;
  const float* pa = a + (size_t)row * D;
  const float* pr = res ? res + (size_t)row * D : nullptr;
  float s = 0.f;
  for (int i = lane; i < D; i += 32) s += pa[i] + (pr ? pr[i] : 0.f);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  const float mean = s / D;
  float v = 0.f;
  for (int i = lane; i < D; i += 32) { float d = pa[i] + (pr ? pr[i] : 0.f) - mean; v += d * d; }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  const float rs = rsqrtf(v / D + 1e-5f);
  for (int i = lane; i < D; i += 32) {
    float xh = (pa[i] + (pr ? pr[i] : 0.f) - mean) * rs;
    xhat[(size_t)row * D + i] = xh;
    y[(size_t)row * D + i] = xh * gamma[i] + beta[i];
  }
  if (lane == 0) rstd[row] = rs;
}
// dx = rstd * (g - mean(g) - xhat*mean(g*xhat)), g = dy*gamma
__global__ void layernorm_bwd_kernel(const float* __restrict__ dy, const float* __restrict__ xhat, const float* __restrict__ rstd,
                                     const float* __restrict__ gamma, int rows, int D, float* __restrict__ dx) {
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= rows) return;
  const float* pd = dy + (size_t)row * D;
  const float* px = xhat + (size_t)row * D;
  float s1 = 0.f, s2 = 0.f;
  for (int i = lane; i < D; i += 32) { float g = pd[i] * gamma[i]; s1 += g; s2 += g * px[i]; }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) { s1 += __shfl_xor_sync(0xffffffffu, s1, o); s2 += __shfl_xor_sync(0xffffffffu, s2, o); }
  const float m1 = s1 / D, m2 = s2 / D, rs = rstd[row];
  for (int i = lane; i < D; i += 32) dx[(size_t)row * D + i] = rs * (pd[i] * gamma[i] - m1 - px[i] * m2);
}
// Column reductions over many rows in ONE launch (deterministic): grid (ceil(D/32), RB), block (32,8); every block writes its
// partial[rb][2][D] sums, the LAST block to arrive for a column group (device counter, reset by that block so the next launch finds
// zeros) adds the RB partials in a fixed order.  mode 0: out0 = sum_r a[r][d];  mode 1: out0 = sum a*b, out1 = sum a.  Rows of a and b
// are ld apart (ld >= D: a slab of a wider matrix).
constexpr int COLRED_RB = 64;
constexpr int COLRED_MAXD = 4096;
__global__ void colred_kernel(const float* __restrict__ a, const float* __restrict__ b, int rows, int D, int ld, float* partial, int* counters,
                              float* __restrict__ out0, float* __restrict__ out1) {
  __shared__ float s0[8][33], s1[8][33];
  __shared__ int last;
  const int d = blockIdx.x * 32 + threadIdx.x;
  const int per = (rows + gridDim.y - 1) / gridDim.y;
  const int r_lo = blockIdx.y * per, r_hi = min(rows, r_lo + per);
  float x = 0.f, y = 0.f;
  if (d < D) {
    // four independent row streams per thread (fixed order of the final adds): the loads of a stripe are in flight together
    float xa[4] = {0.f, 0.f, 0.f, 0.f}, ya[4] = {0.f, 0.f, 0.f, 0.f};
    int r = r_lo + threadIdx.y;
    for (; r + 24 < r_hi; r += 32) {
      float v[4], w[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) { v[u] = a[(size_t)(r + 8 * u) * ld + d]; w[u] = b ? b[(size_t)(r + 8 * u) * ld + d] : 1.f; }
#pragma unroll
      for (int u = 0; u < 4; ++u) { xa[u] += v[u] * w[u]; ya[u] += v[u]; }
    }
    for (; r < r_hi; r += 8) {
      const float v = a[(size_t)r * ld + d];
      xa[0] += b ? v * b[(size_t)r * ld + d] : v; ya[0] += v;
    }
    x = (xa[0] + xa[1]) + (xa[2] + xa[3]); y = (ya[0] + ya[1]) + (ya[2] + ya[3]);
  }
  s0[threadIdx.y][threadIdx.x] = x; s1[threadIdx.y][threadIdx.x] = y;
  __syncthreads();
  if (threadIdx.y == 0 && d < D) {
    for (int r = 1; r < 8; ++r) { x += s0[r][threadIdx.x]; y += s1[r][threadIdx.x]; }
    partial[((size_t)blockIdx.y * 2) * D + d] = x;
    partial[((size_t)blockIdx.y * 2 + 1) * D + d] = y;
    __threadfence();
  }
  __syncthreads();
  if (threadIdx.x == 0 && threadIdx.y == 0) {
    const int t = atomicAdd(&counters[blockIdx.x], 1);
    last = (t == (int)gridDim.y - 1);
    if (last) counters[blockIdx.x] = 0;
  }
  __syncthreads();
  if (!last) return;
  __threadfence();
  x = 0.f; y = 0.f;
  if (d < D)
    for (int rb = threadIdx.y; rb < (int)gridDim.y; rb += 8) {
      x += __ldcg(&partial[((size_t)rb * 2) * D + d]);
      y += __ldcg(&partial[((size_t)rb * 2 + 1) * D + d]);
    }
  s0[threadIdx.y][threadIdx.x] = x; s1[threadIdx.y][threadIdx.x] = y;
  __syncthreads();
  if (threadIdx.y == 0 && d < D) {
    for (int r = 1; r < 8; ++r) { x += s0[r][threadIdx.x]; y += s1[r][threadIdx.x]; }
    out0[d] = x;
    if (out1) out1[d] = y;
  }
}
// row-wise softmax (+ dropout multiplier) over rows of length L:  P = softmax(S);  Pd = P * mask
__global__ void softmax_rows_kernel(const float* __restrict__ S, const float* __restrict__ mask, size_t rows, int L,
                                    float* __restrict__ P, float* __restrict__ Pd) {
  const size_t row = blockIdx.x * (size_t)(blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  const float* s = S + row * L;
  float mx = -INFINITY;
  for (int i = lane; i < L; i += 32) mx = fmaxf(mx, s[i]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  float sum = 0.f;
  for (int i = lane; i < L; i += 32) sum += expf(s[i] - mx);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  const float inv = 1.f / sum;
  for (int i = lane; i < L; i += 32) {
    float p = expf(s[i] - mx) * inv;
    P[row * L + i] = p;
    Pd[row * L + i] = mask ? p * mask[row * L + i] : p;
  }
}
// dS = P * (dP - sum(dP*P)),  dP = dPd * mask      (in place on dPd)
__global__ void softmax_bwd_rows_kernel(float* __restrict__ dPd, const float* __restrict__ P, const float* __restrict__ mask, size_t rows, int L) {
  const size_t row = blockIdx.x * (size_t)(blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  float* d = dPd + row * L;
  const float* p = P + row * L;
  float dotv = 0.f;
  for (int i = lane; i < L; i += 32) { float dp = mask ? d[i] * mask[row * L + i] : d[i]; dotv += dp * p[i]; }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) dotv += __shfl_xor_sync(0xffffffffu, dotv, o);
  for (int i = lane; i < L; i += 32) { float dp = mask ? d[i] * mask[row * L + i] : d[i]; d[i] = p[i] * (dp - dotv); }
}
// pooled[b][e] = sum_t x[b][t][e] / T
__global__ void meanpool_kernel(const float* __restrict__ x, int B, int T, int E, float* __restrict__ out) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * E) return;
  int b = i / E, e = i % E;
  float s = 0.f;
  for (int t = 0; t < T; ++t) s += x[((size_t)b * T + t) * E + e];
  out[i] = s / (float)T;
}
__global__ void meanpool_bwd_kernel(const float* __restrict__ dout, int B, int T, int E, float* __restrict__ dx) {
  const size_t total = (size_t)B * T * E;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    int e = i % E; int b = i / ((size_t)T * E);
    dx[i] = dout[(size_t)b * E + e] / (float)T;
  }
}
// z = mu + eps * exp(0.5 logvar) / temperature      (modules.py:292-302)
__global__ void vae_sample_kernel(const float* __restrict__ pooled, const float* __restrict__ eps, int B, int Z, float inv_temp,
                                  float* __restrict__ z, float* __restrict__ mu, float* __restrict__ logvar) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * Z) return;
  int b = i / Z, j = i % Z;
  float m = pooled[(size_t)b * 2 * Z + j], lv = pooled[(size_t)b * 2 * Z + Z + j];
  mu[i] = m; logvar[i] = lv;
  z[i] = m + (eps ? eps[i] : 0.f) * expf(0.5f * lv) * inv_temp;
}
// dpooled from dz, dmu, dlogvar (any may be null)
__global__ void vae_sample_bwd_kernel(const float* __restrict__ dz, const float* __restrict__ dmu, const float* __restrict__ dlv,
                                      const float* __restrict__ eps, const float* __restrict__ logvar, int B, int Z, float inv_temp,
                                      float* __restrict__ dpooled) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * Z) return;
  int b = i / Z, j = i % Z;
  float gz = dz ? dz[i] : 0.f;
  float gm = gz + (dmu ? dmu[i] : 0.f);
  float gl = (dlv ? dlv[i] : 0.f) + (eps ? gz * eps[i] * 0.5f * expf(0.5f * logvar[i]) * inv_temp : 0.f);
  dpooled[(size_t)b * 2 * Z + j] = gm;
  dpooled[(size_t)b * 2 * Z + Z + j] = gl;
}
// ------------------------------------------------------------------ launch helpers
#define GRID1(n) (unsigned)((((size_t)(n) + 255) / 256) > 4736 ? 4736 : (((size_t)(n) + 255) / 256))

static int im2col(const float* x, int B, int T, int C, int k, int pad, int rep, float* col, cudaStream_t s) {
  im2col_kernel<<<GRID1((size_t)B * T * C * k), 256, 0, s>>>(x, B, T, C, k, pad, rep, col); LAUNCH_OK(); return 0; }
static int col2im(const float* dcol, int B, int T, int C, int k, int pad, int rep, float* dx, cudaStream_t s) {
  col2im_kernel<<<GRID1((size_t)B * T * C), 256, 0, s>>>(dcol, B, T, C, k, pad, rep, dx); LAUNCH_OK(); return 0; }
static int ew_mul(float* dst, const float* a, const float* mask, const float* y, int ag, size_t n, cudaStream_t s) {
  ew_mul_kernel<<<GRID1(n), 256, 0, s>>>(dst, a, mask, y, ag, n); LAUNCH_OK(); return 0; }
static int ew_add(float* dst, const float* a, const float* b, size_t n, size_t period, cudaStream_t s) {
  ew_add_kernel<<<GRID1(n), 256, 0, s>>>(dst, a, b, n, period); LAUNCH_OK(); return 0; }
static int ln_fwd(const float* a, const float* res, const float* g, const float* b, int rows, int D, float* y, float* xh, float* rs, cudaStream_t s) {
  layernorm_fwd_kernel<<<ceil_div(rows, 8), 256, 0, s>>>(a, res, g, b, rows, D, y, xh, rs); LAUNCH_OK(); return 0; }
// red: the column reductions' scratch inside the calling module's workspace, [COLRED_RB][2][4096] partials + arrival counters.
// Wider sums (the GRU's 3H bias columns above H = 1365) run as consecutive slabs of at most 4096 columns through the same scratch:
// stream order keeps a slab's partials until its last block has read them, and that block leaves the counters at zero.
static int colred(const float* a, const float* b, int rows, int D, float* out0, float* out1, float* red, cudaStream_t s) {
  ZCHECK_ARG(red != nullptr, "column reduction: scratch missing");
  const int RB = rows < 8 * COLRED_RB ? ceil_div(rows, 8) : COLRED_RB;
  int* counters = reinterpret_cast<int*>(red + (size_t)COLRED_RB * 2 * COLRED_MAXD);
  for (int d0 = 0; d0 < D; d0 += COLRED_MAXD) {
    const int w = std::min(COLRED_MAXD, D - d0);
    colred_kernel<<<dim3(ceil_div(w, 32), RB), dim3(32, 8), 0, s>>>(a + d0, b ? b + d0 : nullptr, rows, w, D, red, counters, out0 + d0,
                                                                     out1 ? out1 + d0 : nullptr);
    LAUNCH_OK();
  }
  return 0; }
// the arrival counters behind the partials must be zero before the first reduction of a call (the workspace is caller memory)
static int colred_reset(float* red, cudaStream_t s) {
  ZCHECK_CUDA(cudaMemsetAsync(red + (size_t)COLRED_RB * 2 * COLRED_MAXD, 0, (COLRED_MAXD / 32) * sizeof(int), s)); return 0; }
static int ln_bwd(const float* dy, const float* xh, const float* rs, const float* g, int rows, int D, float* dx, float* dg, float* db,
                  float* red, cudaStream_t s) {
  layernorm_bwd_kernel<<<ceil_div(rows, 8), 256, 0, s>>>(dy, xh, rs, g, rows, D, dx); LAUNCH_OK();
  return colred(dy, xh, rows, D, dg, db, red, s); }
static int colsum(const float* x, int rows, int cols, float* out, float* red, cudaStream_t s) {
  return colred(x, nullptr, rows, cols, out, nullptr, red, s); }
// Linear / conv-as-GEMM forward: y[M,N] = act(x[M,K] W[N,K]^T + b)
static int lin_fwd(const float* x, const float* W, const float* b, float* y, int M, int N, int K, int act, cudaStream_t s) {
  return gemm_f32_auto(0, M, N, K, x, K, W, K, b, y, N, act, 0, s); }
// backward of y = x W^T + b given dpre[M,N]:  dW[N,K] = dpre^T x ; db ; dx[M,K] = dpre W (optional)
static int lin_bwd(const float* dpre, const float* x, const float* W, float* dW, float* db, float* dx, int M, int N, int K, float* red,
                   cudaStream_t s) {
  RC(gemm_f32_auto(1, N, K, M, dpre, N, x, K, nullptr, dW, K, 0, 0, s));
  if (db) RC(colsum(dpre, M, N, db, red, s));
  if (dx) RC(gemm_f32_auto(2, M, K, N, dpre, N, W, K, nullptr, dx, K, 0, 0, s));
  return 0;
}

// 1-D convolution (channels-last, 'same' zero or replicate padding) as a GEMM.  Fast path: the bf16 operands are produced straight from
// x (conv_gemm_*, no im2col matrix in HBM); otherwise im2col into `col` + the generic product.
static int conv_fwd(const float* x, int B, int T, int C, int k, int pad, int rep, const float* W, const float* b, float* y, int N, int act,
                    float* col, cudaStream_t s) {
  const int rc = conv_gemm_fwd(x, B, T, C, k, pad, rep, W, b, y, N, act, s);
  if (rc != ZEGGS_CONV_NOT_TAKEN) return rc;
  RC(im2col(x, B, T, C, k, pad, rep, col, s));
  return lin_fwd(col, W, b, y, B * T, N, C * k, act, s);
}
// backward given dpre[(b,t)][N]: dW, db, and (optional) dcol[(b,t)][C*k] = dpre W for col2im
static int conv_bwd(const float* dpre, const float* x, int B, int T, int C, int k, int pad, int rep, const float* W, float* dW, float* db,
                    float* dcol, int N, float* col, float* red, cudaStream_t s) {
  const int M = B * T, K = C * k;
  int rc = conv_gemm_wgrad(dpre, N, x, B, T, C, k, pad, rep, dW, s);
  if (rc == ZEGGS_CONV_NOT_TAKEN) {
    RC(im2col(x, B, T, C, k, pad, rep, col, s));
    rc = gemm_f32_auto(1, N, K, M, dpre, N, col, K, nullptr, dW, K, 0, 0, s);
  }
  if (rc) return rc;
  if (db) RC(colsum(dpre, M, N, db, red, s));
  if (dcol) RC(gemm_f32_auto(2, M, K, N, dpre, N, W, K, nullptr, dcol, K, 0, 0, s));
  return 0;
}

// ================================================================== SpeechEncoder
struct SpeechWs { float *h0, *h0d, *col1, *h1, *h1d, *t0, *t1, *dcol, *red; size_t bytes; };
static SpeechWs speech_ws(void* base, int B, int T, int Cin, int H, int O, int k) {
  Arena a{(char*)base, 0};
  SpeechWs w; const size_t R = (size_t)B * T;
  w.h0 = a.take(R * H); w.h0d = a.take(R * H); w.col1 = a.take(R * H * k); w.h1 = a.take(R * O); w.h1d = a.take(R * O);
  w.t0 = a.take(R * (H > O ? H : O)); w.t1 = a.take(R * (H > O ? H : O)); w.dcol = a.take(R * H * k);
  w.red = a.take((size_t)COLRED_RB * 2 * COLRED_MAXD + COLRED_MAXD / 32);
  w.bytes = a.off; return w;
}
extern "C" size_t zeggs_speech_enc_workspace_bytes(int B, int T, int Cin, int H, int O) {
  if (B < 1 || T < 1) return 0;
  return speech_ws(nullptr, B, T, Cin, H, O, 31).bytes;
}
extern "C" int zeggs_speech_enc_fwd(const zeggs_speech_enc_args* ap, void* stream_) {
  CtxScope ctx_scope(ap ? ap->ctx : nullptr);
  ZCHECK_ARG(ap, "speech_enc: null args");
  const zeggs_speech_enc_args& a = *ap; cudaStream_t s = (cudaStream_t)stream_;
  const int B = a.B, T = a.T, Cin = a.C_in, H = a.H, O = a.O, k = 31, M = B * T;
  ZCHECK_ARG(B >= 1 && T >= 1 && Cin >= 1 && H >= 1 && O >= 1 && a.x && a.y, "speech_enc: bad arguments");
  SpeechWs w = speech_ws(a.workspace, B, T, Cin, H, O, k);
  ZCHECK_ARG(a.workspace && a.workspace_bytes >= w.bytes, "speech_enc: workspace too small");
  ScopedTimer tm("encoders_fwd", s);
  RC(lin_fwd(a.x, a.W0, a.b0, w.h0, M, H, Cin, 1, s));                              // conv k=1 + ELU   (:267)
  RC(ew_mul(w.h0d, w.h0, a.mask0, nullptr, 0, (size_t)M * H, s));                   // drop0
  RC(conv_fwd(w.h0d, B, T, H, k, k / 2, 1, a.W1, a.b1, w.h1, O, 1, w.col1, s));     // conv k=31, replicate 'same' padding, + ELU  (:268)
  RC(ew_mul(w.h1d, w.h1, a.mask1, nullptr, 0, (size_t)M * O, s));                   // drop1
  RC(lin_fwd(w.h1d, a.W2, a.b2, a.y, M, O, O, 1, s));                               // Linear + ELU     (:270)
  return ZEGGS_OK;
}
extern "C" int zeggs_speech_enc_bwd(const zeggs_speech_enc_args* ap, const zeggs_speech_enc_grads* gp, void* stream_) {
  CtxScope ctx_scope(ap ? ap->ctx : nullptr);
  ZCHECK_ARG(ap && gp && gp->dy, "speech_enc bwd: null args");
  const zeggs_speech_enc_args& a = *ap; const zeggs_speech_enc_grads& g = *gp; cudaStream_t s = (cudaStream_t)stream_;
  const int B = a.B, T = a.T, Cin = a.C_in, H = a.H, O = a.O, k = 31, M = B * T;
  SpeechWs w = speech_ws(a.workspace, B, T, Cin, H, O, k);
  RC(colred_reset(w.red, s));
  ScopedTimer tm("encoders_bwd", s);
  RC(ew_mul(w.t0, g.dy, nullptr, a.y, 1, (size_t)M * O, s));                        // dpre2 = dy * ELU'(y)
  RC(lin_bwd(w.t0, w.h1d, a.W2, g.dW2, g.db2, w.t1, M, O, O, w.red, s));            // t1 = d h1d
  RC(ew_mul(w.t0, w.t1, a.mask1, w.h1, 1, (size_t)M * O, s));                       // dpre1
  RC(conv_bwd(w.t0, w.h0d, B, T, H, k, k / 2, 1, a.W1, g.dW1, g.db1, w.dcol, O, w.col1, w.red, s)); // dW1, db1, dcol1
  RC(col2im(w.dcol, B, T, H, k, k / 2, 1, w.t1, s));                                // d h0d
  RC(ew_mul(w.t0, w.t1, a.mask0, w.h0, 1, (size_t)M * H, s));                       // dpre0
  RC(lin_bwd(w.t0, a.x, a.W0, g.dW0, g.db0, nullptr, M, H, Cin, w.red, s));
  return ZEGGS_OK;
}

// ================================================================== StyleEncoder (attn, VAE)
struct StyleWs {
  float *col0, *c1, *l1, *xh1, *rs1, *l1d, *col1, *c2, *l2, *xh2, *rs2, *l2d, *pe, *x0, *qkv, *S, *P, *Pd, *o, *ao, *aod,
        *x1, *xh3, *rs3, *colf, *f1, *colf2, *f2, *f2d, *x2, *xh4, *rs4, *pooled;
  float *g0, *g1, *g2, *gqkv, *gcol, *red;   // backward temporaries
  size_t bytes;
};
static StyleWs style_ws(void* base, int B, int T, int Cin, int Hs, int E, int nh) {
  Arena a{(char*)base, 0};
  StyleWs w; const size_t R = (size_t)B * T;
  w.col0 = a.take(R * Cin * 3); w.c1 = a.take(R * Hs); w.l1 = a.take(R * Hs); w.xh1 = a.take(R * Hs); w.rs1 = a.take(R);
  w.l1d = a.take(R * Hs); w.col1 = a.take(R * Hs * 3); w.c2 = a.take(R * E); w.l2 = a.take(R * E); w.xh2 = a.take(R * E);
  w.rs2 = a.take(R); w.l2d = a.take(R * E); w.pe = a.take((size_t)T * E); w.x0 = a.take(R * E); w.qkv = a.take(R * 3 * E);
  w.S = a.take((size_t)B * nh * T * T); w.P = a.take((size_t)B * nh * T * T); w.Pd = a.take((size_t)B * nh * T * T);
  w.o = a.take(R * E); w.ao = a.take(R * E); w.aod = a.take(R * E); w.x1 = a.take(R * E); w.xh3 = a.take(R * E); w.rs3 = a.take(R);
  w.colf = a.take(R * E * 3); w.f1 = a.take(R * E); w.colf2 = a.take(R * E * 3); w.f2 = a.take(R * E); w.f2d = a.take(R * E);
  w.x2 = a.take(R * E); w.xh4 = a.take(R * E); w.rs4 = a.take(R); w.pooled = a.take((size_t)B * E);
  const size_t big = Hs > 3 * E ? Hs : 3 * E;
  w.g0 = a.take(R * big); w.g1 = a.take(R * big); w.g2 = a.take(R * big); w.gqkv = a.take(R * 3 * E);
  w.gcol = a.take(R * (size_t)(Hs * 3 > E * 3 ? Hs * 3 : E * 3));
  w.red = a.take((size_t)COLRED_RB * 2 * COLRED_MAXD + COLRED_MAXD / 32);
  w.bytes = a.off; return w;
}
extern "C" size_t zeggs_style_enc_workspace_bytes(int B, int T, int Cin, int Hs, int E, int nheads) {
  if (B < 1 || T < 1 || nheads < 1 || E % nheads) return 0;
  return style_ws(nullptr, B, T, Cin, Hs, E, nheads).bytes;
}

extern "C" int zeggs_style_enc_fwd(const zeggs_style_enc_args* ap, void* stream_) {
  CtxScope ctx_scope(ap ? ap->ctx : nullptr);
  ZCHECK_ARG(ap, "style_enc: null args");
  const zeggs_style_enc_args& a = *ap; cudaStream_t s = (cudaStream_t)stream_;
  const int B = a.B, T = a.T, Cin = a.C_in, Hs = a.H, E = a.E, nh = a.nheads, M = B * T, d = E / nh;
  const bool vae = a.mu != nullptr;
  ZCHECK_ARG(B >= 1 && T >= 1 && nh >= 1 && E % nh == 0 && (!vae || E % 2 == 0) && a.x && a.z && (a.logvar != nullptr) == vae,
             "style_enc: bad arguments");
  ZCHECK_ARG((long long)B * nh <= 65535, "style_enc: B*nheads too large for one launch");
  StyleWs w = style_ws(a.workspace, B, T, Cin, Hs, E, nh);
  ZCHECK_ARG(a.workspace && a.workspace_bytes >= w.bytes, "style_enc: workspace too small");
  ScopedTimer tm("encoders_fwd", s);
  // conv stack (modules.py:359-384): conv k3 zero-pad -> ReLU -> LayerNorm -> Dropout, twice
  RC(conv_fwd(a.x, B, T, Cin, 3, 1, 0, a.Wc1, a.bc1, w.c1, Hs, 2, w.col0, s));
  RC(ln_fwd(w.c1, nullptr, a.ln1_g, a.ln1_b, M, Hs, w.l1, w.xh1, w.rs1, s));
  RC(ew_mul(w.l1d, w.l1, a.mask_c1, nullptr, 0, (size_t)M * Hs, s));
  RC(conv_fwd(w.l1d, B, T, Hs, 3, 1, 0, a.Wc2, a.bc2, w.c2, E, 2, w.col1, s));
  RC(ln_fwd(w.c2, nullptr, a.ln2_g, a.ln2_b, M, E, w.l2, w.xh2, w.rs2, s));
  RC(ew_mul(w.l2d, w.l2, a.mask_c2, nullptr, 0, (size_t)M * E, s));
  ZCHECK_ARG(a.pe != nullptr, "style_enc: positional-encoding table missing");
  RC(ew_add(w.x0, w.l2d, a.pe, (size_t)M * E, (size_t)T * E, s));                                    // :410
  // multi-head self-attention (modules.py:529, 544-555)
  RC(lin_fwd(w.x0, a.Win, a.bin, w.qkv, M, 3 * E, E, 0, s));
  const long long TT = (long long)T * T;
  RC(sgemm_batched2_launch(0, T, T, d, w.qkv, 3 * E, w.qkv + E, 3 * E, nullptr, w.S, T, 0, 0, B * nh,
                           (long long)T * 3 * E, (long long)T * 3 * E, nh * TT, nh, d, d, TT, 1.0f / sqrtf((float)d), s));
  softmax_rows_kernel<<<(unsigned)(((size_t)B * nh * T + 7) / 8), 256, 0, s>>>(w.S, a.mask_attn, (size_t)B * nh * T, T, w.P, w.Pd); LAUNCH_OK();
  RC(sgemm_batched2_launch(2, T, d, T, w.Pd, T, w.qkv + 2 * E, 3 * E, nullptr, w.o, E, 0, 0, B * nh,
                           nh * TT, (long long)T * 3 * E, (long long)T * E, nh, TT, d, d, 1.0f, s));
  RC(lin_fwd(w.o, a.Wout, a.bout, w.ao, M, E, E, 0, s));
  RC(ew_mul(w.aod, w.ao, a.mask_ao, nullptr, 0, (size_t)M * E, s));
  RC(ln_fwd(w.aod, w.x0, a.ln3_g, a.ln3_b, M, E, w.x1, w.xh3, w.rs3, s));                            // :555
  // position-wise conv feed-forward (modules.py:571-603)
  RC(conv_fwd(w.x1, B, T, E, 3, 1, 0, a.Wf1, a.bf1, w.f1, E, 2, w.colf, s));
  RC(conv_fwd(w.f1, B, T, E, 3, 1, 0, a.Wf2, a.bf2, w.f2, E, 0, w.colf2, s));
  RC(ew_mul(w.f2d, w.f2, a.mask_ff, nullptr, 0, (size_t)M * E, s));
  RC(ln_fwd(w.f2d, w.x1, a.ln4_g, a.ln4_b, M, E, w.x2, w.xh4, w.rs4, s));                            // :603
  if (!vae) {                                                                                        // use_vae=False: z = pooled (:303-304)
    meanpool_kernel<<<ceil_div(B * E, 256), 256, 0, s>>>(w.x2, B, T, E, a.z); LAUNCH_OK();
    return ZEGGS_OK;
  }
  meanpool_kernel<<<ceil_div(B * E, 256), 256, 0, s>>>(w.x2, B, T, E, w.pooled); LAUNCH_OK();        // :416-418
  vae_sample_kernel<<<ceil_div(B * (E / 2), 256), 256, 0, s>>>(w.pooled, a.eps, B, E / 2, 1.0f / a.temperature, a.z, a.mu, a.logvar); LAUNCH_OK();
  return ZEGGS_OK;
}

extern "C" int zeggs_style_enc_bwd(const zeggs_style_enc_args* ap, const zeggs_style_enc_grads* gp, void* stream_) {
  CtxScope ctx_scope(ap ? ap->ctx : nullptr);
  ZCHECK_ARG(ap && gp, "style_enc bwd: null args");
  const zeggs_style_enc_args& a = *ap; const zeggs_style_enc_grads& g = *gp; cudaStream_t s = (cudaStream_t)stream_;
  const int B = a.B, T = a.T, Cin = a.C_in, Hs = a.H, E = a.E, nh = a.nheads, M = B * T, d = E / nh;
  StyleWs w = style_ws(a.workspace, B, T, Cin, Hs, E, nh);
  const long long TT = (long long)T * T;
  const size_t nE = (size_t)M * E;
  const bool vae = a.mu != nullptr;
  ZCHECK_ARG(vae || (g.dz && !g.dmu && !g.dlogvar), "style_enc bwd: without the VAE (mu == NULL) dz [B,E] is required and dmu / dlogvar must be NULL");
  RC(colred_reset(w.red, s));
  ScopedTimer tm("encoders_bwd", s);
  // VAE sample + mean pool
  if (vae) {
    vae_sample_bwd_kernel<<<ceil_div(B * (E / 2), 256), 256, 0, s>>>(g.dz, g.dmu, g.dlogvar, a.eps, a.logvar, B, E / 2, 1.0f / a.temperature, w.pooled); LAUNCH_OK();
  }
  meanpool_bwd_kernel<<<GRID1(nE), 256, 0, s>>>(vae ? w.pooled : g.dz, B, T, E, w.g0); LAUNCH_OK();  // g0 = d x2
  // x2 = LN4(f2d + x1)
  RC(ln_bwd(w.g0, w.xh4, w.rs4, a.ln4_g, M, E, w.g1, g.dln4_g, g.dln4_b, w.red, s));                 // g1 = d(f2d + x1)
  RC(ew_mul(w.g0, w.g1, a.mask_ff, nullptr, 0, nE, s));                                              // g0 = d f2 (pre-act, linear)
  RC(conv_bwd(w.g0, w.f1, B, T, E, 3, 1, 0, a.Wf2, g.dWf2, g.dbf2, w.gcol, E, w.colf2, w.red, s));
  RC(col2im(w.gcol, B, T, E, 3, 1, 0, w.g0, s));                                                     // g0 = d f1
  RC(ew_mul(w.g0, w.g0, nullptr, w.f1, 2, nE, s));                                                   // ReLU'
  RC(conv_bwd(w.g0, w.x1, B, T, E, 3, 1, 0, a.Wf1, g.dWf1, g.dbf1, w.gcol, E, w.colf, w.red, s));
  RC(col2im(w.gcol, B, T, E, 3, 1, 0, w.g0, s));                                                     // g0 = d x1 via FF
  RC(ew_add(w.g1, w.g1, w.g0, nE, 0, s));                                                            // g1 = total d x1
  // x1 = LN3(aod + x0)
  RC(ln_bwd(w.g1, w.xh3, w.rs3, a.ln3_g, M, E, w.g2, g.dln3_g, g.dln3_b, w.red, s));                 // g2 = d(aod + x0)
  RC(ew_mul(w.g0, w.g2, a.mask_ao, nullptr, 0, nE, s));                                              // g0 = d ao
  RC(lin_bwd(w.g0, w.o, a.Wout, g.dWout, g.dbout, w.g1, M, E, E, w.red, s));                         // g1 = d o
  // attention: o = Pd v ; Pd = softmax(S) * mask ; S = scale q k^T
  float* dPd = w.S;   // S is dead after the forward softmax: reuse for dPd / dS
  RC(sgemm_batched2_launch(0, T, T, d, w.g1, E, w.qkv + 2 * E, 3 * E, nullptr, dPd, T, 0, 0, B * nh,
                           (long long)T * E, (long long)T * 3 * E, nh * TT, nh, d, d, TT, 1.0f, s));   // dPd = do v^T
  RC(sgemm_batched2_launch(1, T, d, T, w.Pd, T, w.g1, E, nullptr, w.gqkv + 2 * E, 3 * E, 0, 0, B * nh,
                           nh * TT, (long long)T * E, (long long)T * 3 * E, nh, TT, d, d, 1.0f, s));   // dv = Pd^T do
  softmax_bwd_rows_kernel<<<(unsigned)(((size_t)B * nh * T + 7) / 8), 256, 0, s>>>(dPd, w.P, a.mask_attn, (size_t)B * nh * T, T); LAUNCH_OK();
  const float sc = 1.0f / sqrtf((float)d);
  RC(sgemm_batched2_launch(2, T, d, T, dPd, T, w.qkv + E, 3 * E, nullptr, w.gqkv, 3 * E, 0, 0, B * nh,
                           nh * TT, (long long)T * 3 * E, (long long)T * 3 * E, nh, TT, d, d, sc, s));  // dq = scale dS k
  RC(sgemm_batched2_launch(1, T, d, T, dPd, T, w.qkv, 3 * E, nullptr, w.gqkv + E, 3 * E, 0, 0, B * nh,
                           nh * TT, (long long)T * 3 * E, (long long)T * 3 * E, nh, TT, d, d, sc, s));  // dk = scale dS^T q
  RC(lin_bwd(w.gqkv, w.x0, a.Win, g.dWin, g.dbin, w.g0, M, 3 * E, E, w.red, s));                      // g0 = d x0 via qkv
  RC(ew_add(w.g2, w.g2, w.g0, nE, 0, s));                                                            // g2 = total d x0 = d l2d
  // conv stack
  RC(ew_mul(w.g0, w.g2, a.mask_c2, nullptr, 0, nE, s));                                              // d l2
  RC(ln_bwd(w.g0, w.xh2, w.rs2, a.ln2_g, M, E, w.g1, g.dln2_g, g.dln2_b, w.red, s));                 // g1 = d c2
  RC(ew_mul(w.g1, w.g1, nullptr, w.c2, 2, nE, s));
  RC(conv_bwd(w.g1, w.l1d, B, T, Hs, 3, 1, 0, a.Wc2, g.dWc2, g.dbc2, w.gcol, E, w.col1, w.red, s));
  RC(col2im(w.gcol, B, T, Hs, 3, 1, 0, w.g0, s));                                                    // g0 = d l1d
  RC(ew_mul(w.g0, w.g0, a.mask_c1, nullptr, 0, (size_t)M * Hs, s));
  RC(ln_bwd(w.g0, w.xh1, w.rs1, a.ln1_g, M, Hs, w.g1, g.dln1_g, g.dln1_b, w.red, s));                // g1 = d c1
  RC(ew_mul(w.g1, w.g1, nullptr, w.c1, 2, (size_t)M * Hs, s));
  RC(conv_bwd(w.g1, a.x, B, T, Cin, 3, 1, 0, a.Wc1, g.dWc1, g.dbc1, nullptr, Hs, w.col0, w.red, s));
  return ZEGGS_OK;
}

// ================================================================== StyleEncoder (gru, with or without the VAE)
// The recurrences are in style_gru.cu; everything around them is the GEMM front end and the small kernels above.
struct StyleGruWs {
  unsigned* bar;
  float *col0, *c1, *col1, *c2, *GI, *Hs, *Gs, *GIr, *hcat, *pooled;
  float *dpooled, *dhcat, *dGIr, *dGHr, *dGih, *dGhh, *dc2, *dc1, *gcol, *red;   // backward temporaries
  size_t bytes;
};
static StyleGruWs style_gru_ws(void* base, int B, int T, int Cin, int H, int E, bool vae) {
  Arena a{(char*)base, 0};
  StyleGruWs w; const size_t R = (size_t)B * T;
  w.bar = (unsigned*)a.take(64);
  w.col0 = a.take(R * Cin * 3); w.c1 = a.take(R * H); w.col1 = a.take(R * H * 3); w.c2 = a.take(R * H);
  w.GI = a.take(R * 3 * H);                    // [B*T][3H] input terms of the forward direction
  w.Hs = a.take((R + B) * H);                  // [T+1][B][H] h(-1) = 0, h(0) .. h(T-1)
  w.Gs = a.take(R * 4 * H);                    // [T][B][4H] r, z, n, W_hn h + b_hn
  w.GIr = a.take((size_t)B * 3 * H); w.hcat = a.take((size_t)B * 2 * H); w.pooled = a.take(vae ? (size_t)B * E : 1);
  w.dpooled = a.take(vae ? (size_t)B * E : 1); w.dhcat = a.take((size_t)B * 2 * H);
  w.dGIr = a.take((size_t)B * 3 * H); w.dGHr = a.take((size_t)B * 3 * H);
  w.dGih = w.GI;                               // GI is dead once the forward recurrence has run: its gradient takes its place
  w.dGhh = a.take(R * 3 * H);                  // [T][B][3H]
  w.dc2 = a.take(R * H); w.dc1 = a.take(R * H); w.gcol = a.take(R * H * 3);
  w.red = a.take((size_t)COLRED_RB * 2 * COLRED_MAXD + COLRED_MAXD / 32);
  w.bytes = a.off; return w;
}
extern "C" size_t zeggs_style_enc_gru_workspace_bytes(int B, int T, int Cin, int H, int E, int use_vae) {
  // style_gru_max_batch is 0 for an unsupported hidden size
  if (B < 1 || T < 1 || Cin < 1 || E < 1 || B > style_gru_max_batch(H) || (use_vae && E % 2)) return 0;
  return style_gru_ws(nullptr, B, T, Cin, H, E, use_vae != 0).bytes;
}

extern "C" int zeggs_style_enc_gru_fwd(const zeggs_style_enc_gru_args* ap, void* stream_) {
  CtxScope ctx_scope(ap ? ap->ctx : nullptr);
  ZCHECK_ARG(ap, "style_enc_gru: null args");
  const zeggs_style_enc_gru_args& a = *ap; cudaStream_t s = (cudaStream_t)stream_;
  const int B = a.B, T = a.T, Cin = a.C_in, H = a.H, E = a.E, M = B * T;
  const bool vae = a.mu != nullptr;
  ZCHECK_ARG(B >= 1 && T >= 1 && Cin >= 1 && E >= 1 && (!vae || E % 2 == 0) && a.x && a.z && (a.logvar != nullptr) == vae,
             "style_enc_gru: bad arguments");
  ZCHECK_ARG(units_per_cta(H) > 0, "style_enc_gru: hidden size %d unsupported (H %% 4 == 0 and H <= 528, H %% 8 == 0 and H <= 1056, "
             "or H %% 16 == 0 and H <= 2112)", H);
  ZCHECK_ARG(B <= style_gru_max_batch(H), "style_enc_gru: batch %d too large: at hidden size %d the backward's shared memory holds at "
             "most %d samples per call", B, H, style_gru_max_batch(H));
  StyleGruWs w = style_gru_ws(a.workspace, B, T, Cin, H, E, vae);
  ZCHECK_ARG(a.workspace && a.workspace_bytes >= w.bytes, "style_enc_gru: workspace too small");
  ScopedTimer tm("encoders_fwd", s);
  // convs (modules.py:311-333): conv k3 zero-pad -> ReLU, twice
  RC(conv_fwd(a.x, B, T, Cin, 3, 1, 0, a.Wc1, a.bc1, w.c1, H, 2, w.col0, s));
  RC(conv_fwd(w.c1, B, T, H, 3, 1, 0, a.Wc2, a.bc2, w.c2, H, 2, w.col1, s));
  // rnn_layer (:334, 341): forward direction over all T steps, reverse direction = one cell at T-1 from h = 0
  RC(lin_fwd(w.c2, a.W_ih, a.b_ih, w.GI, M, 3 * H, H, 0, s));
  RC(style_gru_fwd_launch(B, T, H, a.W_hh, a.b_hh, w.GI, w.Hs, w.Gs, w.hcat, w.bar, s));
  RC(gemm_f32_auto(0, B, 3 * H, H, w.c2 + (size_t)(T - 1) * H, T * H, a.W_ih_r, H, a.b_ih_r, w.GIr, 3 * H, 0, 0, s));
  RC(style_gru_rev_cell_fwd(B, H, w.GIr, a.b_hh_r, w.hcat, s));
  // projection_layer(output[:, -1]) (:342), then the VAE split / sample (:291-302) or z = the projection (:303-304)
  RC(lin_fwd(w.hcat, a.Wp, a.bp, vae ? w.pooled : a.z, B, E, 2 * H, 0, s));
  if (vae) {
    vae_sample_kernel<<<ceil_div(B * (E / 2), 256), 256, 0, s>>>(w.pooled, a.eps, B, E / 2, 1.0f / a.temperature, a.z, a.mu, a.logvar); LAUNCH_OK();
  }
  return ZEGGS_OK;
}

extern "C" int zeggs_style_enc_gru_bwd(const zeggs_style_enc_gru_args* ap, const zeggs_style_enc_gru_grads* gp, void* stream_) {
  CtxScope ctx_scope(ap ? ap->ctx : nullptr);
  ZCHECK_ARG(ap && gp, "style_enc_gru bwd: null args");
  const zeggs_style_enc_gru_args& a = *ap; const zeggs_style_enc_gru_grads& g = *gp; cudaStream_t s = (cudaStream_t)stream_;
  const int B = a.B, T = a.T, Cin = a.C_in, H = a.H, E = a.E, M = B * T;
  const bool vae = a.mu != nullptr;
  ZCHECK_ARG(vae || (g.dz && !g.dmu && !g.dlogvar), "style_enc_gru bwd: without the VAE (mu == NULL) dz [B,E] is required and dmu / dlogvar must be NULL");
  ZCHECK_ARG(units_per_cta(H) > 0, "style_enc_gru bwd: hidden size %d unsupported", H);
  ZCHECK_ARG(B <= style_gru_max_batch(H), "style_enc_gru bwd: batch %d too large: at hidden size %d the shared memory holds at most %d "
             "samples per call", B, H, style_gru_max_batch(H));
  StyleGruWs w = style_gru_ws(a.workspace, B, T, Cin, H, E, vae);
  ZCHECK_ARG(a.workspace && a.workspace_bytes >= w.bytes, "style_enc_gru bwd: workspace too small");
  RC(colred_reset(w.red, s));
  ScopedTimer tm("encoders_bwd", s);
  const float* dproj = g.dz;
  if (vae) {
    vae_sample_bwd_kernel<<<ceil_div(B * (E / 2), 256), 256, 0, s>>>(g.dz, g.dmu, g.dlogvar, a.eps, a.logvar, B, E / 2, 1.0f / a.temperature, w.dpooled); LAUNCH_OK();
    dproj = w.dpooled;
  }
  RC(lin_bwd(dproj, w.hcat, a.Wp, g.dWp, g.dbp, w.dhcat, B, E, 2 * H, w.red, s));                   // dhcat = d output[:, -1]
  // reverse cell at T-1: W_ih_r / b_ih_r / b_hh_r gradients, W_hh_r's is zero (it multiplied h = 0)
  RC(style_gru_rev_cell_bwd(B, H, w.GIr, a.b_hh_r, w.dhcat, w.dGIr, w.dGHr, s));
  RC(gemm_f32_auto(1, 3 * H, H, B, w.dGIr, 3 * H, w.c2 + (size_t)(T - 1) * H, T * H, nullptr, g.dW_ih_r, H, 0, 0, s));
  RC(colsum(w.dGIr, B, 3 * H, g.db_ih_r, w.red, s));
  RC(colsum(w.dGHr, B, 3 * H, g.db_hh_r, w.red, s));
  ZCHECK_CUDA(cudaMemsetAsync(g.dW_hh_r, 0, (size_t)3 * H * H * sizeof(float), s));
  // forward direction: BPTT, then every weight / bias / input gradient as a GEMM or column sum over all (t, b)
  RC(style_gru_bwd_launch(B, T, H, a.W_hh, w.Hs, w.Gs, w.dhcat, 2 * H, w.dGih, w.dGhh, w.bar, s));
  RC(gemm_f32_auto(1, 3 * H, H, M, w.dGhh, 3 * H, w.Hs, H, nullptr, g.dW_hh, H, 0, 0, s));            // sum_t dG_hh(t)^T h(t-1)
  RC(colsum(w.dGhh, M, 3 * H, g.db_hh, w.red, s));
  RC(lin_bwd(w.dGih, w.c2, a.W_ih, g.dW_ih, g.db_ih, w.dc2, M, 3 * H, H, w.red, s));
  RC(gemm_f32_auto(2, B, H, 3 * H, w.dGIr, 3 * H, a.W_ih_r, H, nullptr, w.dc2 + (size_t)(T - 1) * H, T * H, 0, 1, s));   // + reverse cell
  // convs
  RC(ew_mul(w.dc2, w.dc2, nullptr, w.c2, 2, (size_t)M * H, s));
  RC(conv_bwd(w.dc2, w.c1, B, T, H, 3, 1, 0, a.Wc2, g.dWc2, g.dbc2, w.gcol, H, w.col1, w.red, s));
  RC(col2im(w.gcol, B, T, H, 3, 1, 0, w.dc1, s));
  RC(ew_mul(w.dc1, w.dc1, nullptr, w.c1, 2, (size_t)M * H, s));
  RC(conv_bwd(w.dc1, a.x, B, T, Cin, 3, 1, 0, a.Wc1, g.dWc1, g.dbc1, nullptr, H, w.col0, w.red, s));
  return ZEGGS_OK;
}

}  // namespace zeggs
