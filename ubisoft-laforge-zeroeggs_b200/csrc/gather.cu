// Device-resident window supplier (SURVEY.md 8f row 2): replaces the per-sample Python indexing + 11 host->device copies of
// ZEGGS/dataset.py:110-153, 176-204 and ZEGGS/train.py:215-225.  The processed arrays live in HBM; one launch gathers, for every
// sample of the batch, the training window (rows [start, start + T) of every array) and the style-example window
// (rows [ex_start, ex_start + ex_n) of the six pose arrays concatenated to 1134 channels with a zero gaze slot, then -- when the
// example is shorter than L -- its own last L - ex_n rows again, dataset.py:198-203).  Pure row copies: bit-exact, HBM bound
// (every output byte written once, every input byte read once; rows are contiguous so all accesses are coalesced).
#include "library.cuh"

namespace zeggs {

// One warp per output row.  Arrays 0..n_arrays-1: dst[a][(b*T + t)][0:width[a]] = src[a][start[b] + t][0:width[a]].
// The style example uses the arrays listed in ex_src (in order) as column blocks of a 1134-wide row.
__global__ void __launch_bounds__(256) window_gather_kernel(zeggs_gather_args a) {
  const int lane = threadIdx.x & 31;
  const long long warp0 = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const long long nwarps = (long long)gridDim.x * (blockDim.x >> 5);
  const long long win_rows = (long long)a.B * a.T;
  const long long ex_rows = a.ex_out ? (long long)a.B * a.L : 0;
  for (long long r = warp0; r < (win_rows + ex_rows) ; r += nwarps) {
    if (r < win_rows) {
      const int b = (int)(r / a.T), t = (int)(r % a.T);
      const long long srow = (long long)a.start[b] + t;
      for (int k = 0; k < a.n_arrays; ++k) {
        const int w = a.width[k];
        const float* s = a.src[k] + srow * w;
        float* d = a.dst[k] + r * w;
        for (int c = lane; c < w; c += 32) d[c] = __ldg(s + c);
      }
    } else {
      const long long e = r - win_rows;
      const int b = (int)(e / a.L), l = (int)(e % a.L);
      const int n = a.ex_n[b];
      // rows past the example's own length repeat its tail: vec = cat(vec, vec[-L + n:])  (dataset.py:201-203)
      const long long srow = (long long)a.ex_start[b] + (l < n ? l : 2 * n - a.L + (l - n));
      float* d = a.ex_out + e * a.ex_width;
      int off = 0;
      for (int k = 0; k < a.n_ex; ++k) {
        const int w = a.width[a.ex_src[k]];
        const float* s = a.src[a.ex_src[k]] + srow * w;
        for (int c = lane; c < w; c += 32) d[off + c] = __ldg(s + c);
        off += w;
      }
      for (int c = off + lane; c < a.ex_width; c += 32) d[c] = 0.f;      // gaze slot zero before normalisation (dataset.py:194-197)
    }
  }
}

extern "C" int zeggs_window_gather(const zeggs_gather_args* ap, void* stream) {
  ZCHECK_ARG(ap, "gather: null args");
  const zeggs_gather_args& a = *ap;
  ZCHECK_ARG(a.B >= 0 && a.T >= 1 && a.n_arrays >= 1 && a.n_arrays <= ZEGGS_GATHER_MAX && a.start, "gather: bad arguments");
  for (int k = 0; k < a.n_arrays; ++k) ZCHECK_ARG(a.src[k] && a.dst[k] && a.width[k] >= 1, "gather: array %d incomplete", k);
  if (a.ex_out) {
    ZCHECK_ARG(a.L >= 1 && a.ex_start && a.ex_n && a.n_ex >= 1 && a.n_ex <= ZEGGS_GATHER_MAX, "gather: style-example arguments incomplete");
    int tot = 0;
    for (int k = 0; k < a.n_ex; ++k) { ZCHECK_ARG(a.ex_src[k] >= 0 && a.ex_src[k] < a.n_arrays, "gather: bad example source"); tot += a.width[a.ex_src[k]]; }
    ZCHECK_ARG(tot <= a.ex_width, "gather: example row wider than ex_width");
  }
  if (a.B == 0) return ZEGGS_OK;
  const long long rows = (long long)a.B * a.T + (a.ex_out ? (long long)a.B * a.L : 0);
  const long long blocks = (rows + 7) / 8;
  window_gather_kernel<<<(unsigned)(blocks > 132 * 8 ? 132 * 8 : blocks), 256, 0, (cudaStream_t)stream>>>(a);
  count_launch();
  ZCHECK_LAUNCH();
  return ZEGGS_OK;
}

// out[r][c] = (x[r][c] - mean[c]) / std[c]: the reference normalises every network input with two broadcast tensor ops
// (train.py:232-234, 247-249); one pass instead of two here, same arithmetic (fp32 subtract, then IEEE divide).
__global__ void normalize_rows_kernel(const float* __restrict__ x, const float* __restrict__ mean, const float* __restrict__ stdv,
                                      float* __restrict__ out, long long rows, int C) {
  const long long total = rows * C;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    out[i] = __fdiv_rn(__fsub_rn(x[i], mean[c]), stdv[c]);
  }
}
extern "C" int zeggs_normalize_rows(const float* x, const float* mean, const float* stdv, float* out, long long rows, int C, void* stream) {
  ZCHECK_ARG(x && mean && stdv && out && rows >= 0 && C >= 1, "normalize_rows: bad arguments");
  if (rows == 0) return ZEGGS_OK;
  const long long blocks = (rows * C + 255) / 256;
  normalize_rows_kernel<<<(unsigned)(blocks > 132 * 16 ? 132 * 16 : blocks), 256, 0, (cudaStream_t)stream>>>(x, mean, stdv, out, rows, C);
  count_launch();
  ZCHECK_LAUNCH();
  return ZEGGS_OK;
}

}  // namespace zeggs
