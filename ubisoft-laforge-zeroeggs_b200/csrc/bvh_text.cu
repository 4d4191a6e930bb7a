// BVH MOTION block text on the device (include/zeggs_b200.h, "BVH MOTION block text"): the parser behind
// zeggs_b200.animation.load_bvh and the writer behind zeggs_b200.bvhio.save_bvh, both exact (bvh_text.cuh).
//
// Both are "count per chunk, scan the chunk counts, recount and scatter" passes:
//   parse:  line breaks per 4 KB chunk -> scan -> break positions; non-blank lines per 2048 lines -> scan -> row -> line map; one
//           thread per row tokenises and converts its line (a 75-joint row is ~2.3 KB of text).
//   format: "%f " lengths per 1024 values -> scan -> each value written at its offset.
// Grids over lines are sized from n_bytes (the line count is only known on the device); CTAs past the last line return at once.
#include "library.cuh"
#include "bvh_text.cuh"

namespace zeggs {

constexpr int BT_THREADS = 256;
constexpr int BT_BYTES_PER_THREAD = 16;
constexpr int BT_CHUNK = BT_THREADS * BT_BYTES_PER_THREAD;   // text bytes per CTA
constexpr int BT_LINES_PER_THREAD = 8;
constexpr int BT_LINE_CHUNK = BT_THREADS * BT_LINES_PER_THREAD;
constexpr int BT_VALUES_PER_THREAD = 4;
constexpr int BT_VALUE_CHUNK = BT_THREADS * BT_VALUES_PER_THREAD;
constexpr int BT_ROW_THREADS = 128;

// exclusive prefix sum over the CTA (BT_THREADS threads); *total = the CTA's sum
template <typename I>
__device__ I block_exclusive_scan(I v, I* total) {
  __shared__ I warp_sum[BT_THREADS / 32];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  I x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const I y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  if (lane == 31) warp_sum[w] = x;
  __syncthreads();
  if (w == 0) {
    I s = lane < BT_THREADS / 32 ? warp_sum[lane] : I(0);
#pragma unroll
    for (int o = 1; o < BT_THREADS / 32; o <<= 1) {
      const I y = __shfl_up_sync(0xffffffffu, s, o);
      if (lane >= o) s += y;
    }
    if (lane < BT_THREADS / 32) warp_sum[lane] = s;     // inclusive sums of the warps
  }
  __syncthreads();
  *total = warp_sum[BT_THREADS / 32 - 1];
  const I r = x - v + (w ? warp_sum[w - 1] : I(0));
  __syncthreads();                                      // warp_sum is reused by the next call
  return r;
}

// in place: counts[0..m) -> exclusive prefix sums; *total = min(sum, cap).  One CTA walks the array in tiles with a carry.
template <typename I>
__global__ void __launch_bounds__(BT_THREADS) bt_scan_kernel(I* counts, int m, I* total, I cap) {
  I carry = 0;
  for (int base = 0; base < m; base += BT_THREADS) {
    const int i = base + threadIdx.x;
    const I v = i < m ? counts[i] : I(0);
    I tile;
    const I ex = block_exclusive_scan(v, &tile);
    if (i < m) counts[i] = carry + ex;
    carry += tile;
  }
  if (threadIdx.x == 0) *total = carry < cap ? carry : cap;
}

// ------------------------------------------------------------------ parser
// Line breaks as Python's universal newlines see them: "\r", or "\n" not preceded by "\r" (so "\r\n" is one break).  Bit b of the
// result is byte i0 + b of this thread's 16; non-ASCII bytes raise *non_ascii.
__device__ __forceinline__ unsigned bt_breaks16(const unsigned char* text, long long n, long long i0, bool* non_ascii) {
  unsigned char c[BT_BYTES_PER_THREAD];
  if (i0 + BT_BYTES_PER_THREAD <= n) {
    const uint4 w = *reinterpret_cast<const uint4*>(text + i0);       // the text is 16-byte aligned, chunks are multiples of 16
    memcpy(c, &w, 16);
  } else {
#pragma unroll
    for (int b = 0; b < BT_BYTES_PER_THREAD; ++b) c[b] = i0 + b < n ? text[i0 + b] : (unsigned char)' ';
  }
  unsigned prev = i0 > 0 && i0 <= n ? text[i0 - 1] : 0u;
  unsigned mask = 0;
  bool hi = false;
#pragma unroll
  for (int b = 0; b < BT_BYTES_PER_THREAD; ++b) {
    const unsigned x = c[b];
    if (x == '\r' || (x == '\n' && prev != '\r')) mask |= 1u << b;
    hi |= x >= 0x80u;
    prev = x;
  }
  *non_ascii = hi;
  return mask;
}

__global__ void __launch_bounds__(BT_THREADS) bt_break_count_kernel(const unsigned char* text, long long n, int* counts, int* status) {
  const long long i0 = (long long)blockIdx.x * BT_CHUNK + threadIdx.x * BT_BYTES_PER_THREAD;
  bool hi = false;
  const int k = i0 < n ? __popc(bt_breaks16(text, n, i0, &hi)) : 0;
  if (__syncthreads_or(hi) && threadIdx.x == 0) atomicOr(status + 2, 2);
  int tot;
  block_exclusive_scan(k, &tot);
  if (threadIdx.x == 0) counts[blockIdx.x] = tot;
}

__global__ void __launch_bounds__(BT_THREADS) bt_break_scatter_kernel(const unsigned char* text, long long n, const int* offsets,
                                                                        int* breaks) {
  const long long i0 = (long long)blockIdx.x * BT_CHUNK + threadIdx.x * BT_BYTES_PER_THREAD;
  bool hi = false;
  unsigned mask = i0 < n ? bt_breaks16(text, n, i0, &hi) : 0u;
  int tot;
  int o = offsets[blockIdx.x] + block_exclusive_scan(__popc(mask), &tot);
  for (; mask; mask &= mask - 1) breaks[o++] = (int)(i0 + __ffs(mask) - 1);
}

// line l = [start, end): between the breaks l-1 and l (the last line ends at n)
__device__ __forceinline__ void bt_line(const int* breaks, int nbreaks, long long n, int l, long long* s, long long* e) {
  *s = l ? (long long)breaks[l - 1] + 1 : 0;
  *e = l < nbreaks ? (long long)breaks[l] : n;
}

// bit i of the result: line l0 + i is non-blank (holds a byte that strip() keeps)
__device__ __forceinline__ unsigned bt_nonblank8(const unsigned char* text, long long n, const int* breaks, int nbreaks, int l0) {
  unsigned mask = 0;
  for (int i = 0; i < BT_LINES_PER_THREAD; ++i) {
    const int l = l0 + i;
    if (l > nbreaks) break;
    long long s, e;
    bt_line(breaks, nbreaks, n, l, &s, &e);
    while (s < e && bvh_is_space(text[s])) ++s;
    if (s < e) mask |= 1u << i;
  }
  return mask;
}

__global__ void __launch_bounds__(BT_THREADS) bt_row_count_kernel(const unsigned char* text, long long n, const int* breaks,
                                                                    const int* nbreaks_p, int* counts) {
  const int nbreaks = *nbreaks_p;
  if ((long long)blockIdx.x * BT_LINE_CHUNK > nbreaks) { if (threadIdx.x == 0) counts[blockIdx.x] = 0; return; }
  const int l0 = blockIdx.x * BT_LINE_CHUNK + threadIdx.x * BT_LINES_PER_THREAD;
  int tot;
  block_exclusive_scan(__popc(bt_nonblank8(text, n, breaks, nbreaks, l0)), &tot);
  if (threadIdx.x == 0) counts[blockIdx.x] = tot;
}

__global__ void __launch_bounds__(BT_THREADS) bt_row_scatter_kernel(const unsigned char* text, long long n, const int* breaks,
                                                                      const int* nbreaks_p, const int* offsets, int n_frames,
                                                                      int* row_line) {
  const int nbreaks = *nbreaks_p;
  if ((long long)blockIdx.x * BT_LINE_CHUNK > nbreaks || offsets[blockIdx.x] >= n_frames) return;
  const int l0 = blockIdx.x * BT_LINE_CHUNK + threadIdx.x * BT_LINES_PER_THREAD;
  unsigned mask = bt_nonblank8(text, n, breaks, nbreaks, l0);
  int tot;
  int r = offsets[blockIdx.x] + block_exclusive_scan(__popc(mask), &tot);
  for (; mask && r < n_frames; mask &= mask - 1) row_line[r++] = l0 + __ffs(mask) - 1;
}

__global__ void __launch_bounds__(BT_ROW_THREADS) bt_parse_rows_kernel(zeggs_bvh_parse_args a, const int* breaks, const int* nbreaks_p,
                                                                         const int* row_line) {
  const int r = blockIdx.x * BT_ROW_THREADS + threadIdx.x;
  if (r >= a.status[0]) return;
  long long s, e;
  bt_line(breaks, *nbreaks_p, a.n_bytes, row_line[r], &s, &e);
  const unsigned char* t = a.text;
  double* out = a.out + (size_t)r * a.C;
  int col = 0;
  for (;;) {
    while (s < e && bvh_is_space(t[s])) ++s;
    if (s >= e) break;
    long long te = s;
    while (te < e && !bvh_is_space(t[te])) ++te;
    if (col < a.C) {
      double v;
      if (bvh_parse_token(t + s, t + te, &v)) {
        out[col] = v;
      } else {
        const int k = atomicAdd(a.status + 1, 1);
        if (k < a.max_flagged) { a.flagged[2 * (size_t)k] = (long long)r * a.C + col; a.flagged[2 * (size_t)k + 1] = s; }
      }
    }
    ++col;
    s = te;
  }
  if (col != a.C) atomicOr(a.status + 2, 1);
}

struct ParseWs { int *chunk, *nbreaks, *breaks, *line_chunk, *nonblank, *row_line; };
static size_t parse_carve(char* base, long long n, int F, ParseWs* w) {
  const long long nchunks = (n + BT_CHUNK - 1) / BT_CHUNK, nlchunks = (n + 1 + BT_LINE_CHUNK - 1) / BT_LINE_CHUNK;
  Arena ar{base};
  w->chunk = (int*)ar.bytes(sizeof(int) * nchunks);
  w->nbreaks = (int*)ar.bytes(sizeof(int));
  w->nonblank = (int*)ar.bytes(sizeof(int));
  w->breaks = (int*)ar.bytes(sizeof(int) * (size_t)n);
  w->line_chunk = (int*)ar.bytes(sizeof(int) * nlchunks);
  w->row_line = (int*)ar.bytes(sizeof(int) * (size_t)F);
  return ar.off;
}

extern "C" size_t zeggs_bvh_parse_motion_workspace_size(long long n_bytes, int n_frames) {
  if (n_bytes < 0 || n_bytes >= (1ll << 31) || n_frames < 0) return 0;
  ParseWs w;
  return parse_carve(nullptr, n_bytes, n_frames, &w);
}

extern "C" int zeggs_bvh_parse_motion(const zeggs_bvh_parse_args* ap, void* stream) {
  ZCHECK_ARG(ap, "bvh parse: null args");
  const zeggs_bvh_parse_args& a = *ap;
  ZCHECK_ARG(a.n_bytes >= 0 && a.n_bytes < (1ll << 31) && a.n_frames >= 0 && a.C >= 1 && a.max_flagged >= 0,
             "bvh parse: bad sizes (n_bytes %lld, n_frames %d, C %d)", a.n_bytes, a.n_frames, a.C);
  ZCHECK_ARG(a.status && (a.n_bytes == 0 || a.text) && (a.n_frames == 0 || a.out) && (a.max_flagged == 0 || a.flagged),
             "bvh parse: null pointer");
  ZCHECK_ARG(((uintptr_t)a.text & 15) == 0, "bvh parse: text must be 16-byte aligned");
  const size_t need = zeggs_bvh_parse_motion_workspace_size(a.n_bytes, a.n_frames);
  ZCHECK_ARG(a.workspace && a.workspace_bytes >= need, "bvh parse: workspace of %zu bytes, %zu needed", a.workspace_bytes, need);
  cudaStream_t s = (cudaStream_t)stream;
  ZCHECK_CUDA(cudaMemsetAsync(a.status, 0, 3 * sizeof(int), s));
  if (a.n_frames == 0) return ZEGGS_OK;
  ParseWs w;
  parse_carve((char*)a.workspace, a.n_bytes, a.n_frames, &w);
  const int nchunks = (int)((a.n_bytes + BT_CHUNK - 1) / BT_CHUNK);
  const int nlchunks = (int)((a.n_bytes + 1 + BT_LINE_CHUNK - 1) / BT_LINE_CHUNK);
  if (nchunks) {
    bt_break_count_kernel<<<nchunks, BT_THREADS, 0, s>>>(a.text, a.n_bytes, w.chunk, a.status);
    LAUNCH_OK();
  }
  bt_scan_kernel<int><<<1, BT_THREADS, 0, s>>>(w.chunk, nchunks, w.nbreaks, 0x7fffffff);
  LAUNCH_OK();
  if (nchunks) {
    bt_break_scatter_kernel<<<nchunks, BT_THREADS, 0, s>>>(a.text, a.n_bytes, w.chunk, w.breaks);
    LAUNCH_OK();
  }
  bt_row_count_kernel<<<nlchunks, BT_THREADS, 0, s>>>(a.text, a.n_bytes, w.breaks, w.nbreaks, w.line_chunk);
  LAUNCH_OK();
  bt_scan_kernel<int><<<1, BT_THREADS, 0, s>>>(w.line_chunk, nlchunks, a.status, a.n_frames);   // status[0] = rows taken
  LAUNCH_OK();
  bt_row_scatter_kernel<<<nlchunks, BT_THREADS, 0, s>>>(a.text, a.n_bytes, w.breaks, w.nbreaks, w.line_chunk, a.n_frames, w.row_line);
  LAUNCH_OK();
  bt_parse_rows_kernel<<<(a.n_frames + BT_ROW_THREADS - 1) / BT_ROW_THREADS, BT_ROW_THREADS, 0, s>>>(a, w.breaks, w.nbreaks, w.row_line);
  LAUNCH_OK();
  return ZEGGS_OK;
}

// ------------------------------------------------------------------ writer
__device__ __forceinline__ double bt_value(const zeggs_bvh_format_args& a, int C, long long i) {
  const long long t = i / C;
  const int c = (int)(i - t * C);
  const int j = c < 3 ? 0 : a.seq[(c - 3) / 3];
  const long long k = ((t * a.J) + j) * 3 + (c < 3 ? c : (c - 3) % 3);
  const void* src = c < 3 ? a.positions : a.rotations;
  return a.in_f64 ? ((const double*)src)[k] : (double)((const float*)src)[k];
}

// bytes of value i in the text: "%f", the separating space and, after the last column, the newline (0 for a flagged value)
__device__ __forceinline__ int bt_value_len(int n, int C, long long i) {
  return n < 0 ? 0 : n + 1 + ((i % C) == C - 1);
}

__global__ void __launch_bounds__(BT_THREADS) bt_format_count_kernel(zeggs_bvh_format_args a, int C, long long V, long long* counts) {
  const long long i0 = (long long)blockIdx.x * BT_VALUE_CHUNK + threadIdx.x * BT_VALUES_PER_THREAD;
  long long len = 0;
#pragma unroll
  for (int k = 0; k < BT_VALUES_PER_THREAD; ++k)
    if (i0 + k < V) len += bt_value_len(bvh_format_f(bt_value(a, C, i0 + k), nullptr), C, i0 + k);
  long long tot;
  block_exclusive_scan(len, &tot);
  if (threadIdx.x == 0) counts[blockIdx.x] = tot;
}

__global__ void __launch_bounds__(BT_THREADS) bt_format_write_kernel(zeggs_bvh_format_args a, int C, long long V, const long long* offsets) {
  const long long i0 = (long long)blockIdx.x * BT_VALUE_CHUNK + threadIdx.x * BT_VALUES_PER_THREAD;
  double v[BT_VALUES_PER_THREAD];
  int n[BT_VALUES_PER_THREAD];
  long long len = 0;
#pragma unroll
  for (int k = 0; k < BT_VALUES_PER_THREAD; ++k) {
    v[k] = 0.0; n[k] = -1;
    if (i0 + k < V) {
      v[k] = bt_value(a, C, i0 + k);
      n[k] = bvh_format_f(v[k], nullptr);
      len += bt_value_len(n[k], C, i0 + k);
    }
  }
  long long tot;
  long long o = offsets[blockIdx.x] + block_exclusive_scan(len, &tot);
#pragma unroll
  for (int k = 0; k < BT_VALUES_PER_THREAD; ++k) {
    const long long i = i0 + k;
    if (i >= V) break;
    const long long t = i / C;
    const int c = (int)(i - t * C);
    if (c == 0) a.row_start[t] = o;
    if (n[k] < 0) {
      const unsigned long long f = atomicAdd((unsigned long long*)(a.status + 1), 1ull);
      if (f < (unsigned long long)a.max_flagged) a.flagged[f] = i;
    } else {
      bvh_format_f(v[k], a.out + o);
      o += n[k];
      a.out[o++] = ' ';
      if (c == C - 1) a.out[o++] = '\n';
    }
    if (i == V - 1) a.row_start[a.T] = o;
  }
}

static size_t format_carve(char* base, long long V, long long** chunk) {
  Arena ar{base};
  *chunk = (long long*)ar.bytes(sizeof(long long) * (size_t)((V + BT_VALUE_CHUNK - 1) / BT_VALUE_CHUNK));
  return ar.off;
}

extern "C" long long zeggs_bvh_format_motion_max_size(int T, int J) {
  if (T < 0 || J < 1) return 0;
  return (long long)T * (3 + 3ll * J) * (BVH_F_MAX_CHARS + 1) + T;
}

extern "C" size_t zeggs_bvh_format_motion_workspace_size(int T, int J) {
  if (T < 0 || J < 1) return 0;
  long long* c;
  return format_carve(nullptr, (long long)T * (3 + 3ll * J), &c);
}

extern "C" int zeggs_bvh_format_motion(const zeggs_bvh_format_args* ap, void* stream) {
  ZCHECK_ARG(ap, "bvh format: null args");
  const zeggs_bvh_format_args& a = *ap;
  ZCHECK_ARG(a.T >= 0 && a.J >= 1 && a.max_flagged >= 0 && (a.in_f64 == 0 || a.in_f64 == 1), "bvh format: bad sizes (T %d, J %d)",
             a.T, a.J);
  ZCHECK_ARG(a.status && a.row_start && (a.max_flagged == 0 || a.flagged), "bvh format: null pointer");
  ZCHECK_ARG(a.T == 0 || (a.positions && a.rotations && a.seq && a.out), "bvh format: null pointer");
  ZCHECK_ARG(a.out_capacity >= zeggs_bvh_format_motion_max_size(a.T, a.J), "bvh format: output of %lld bytes, %lld needed",
             a.out_capacity, zeggs_bvh_format_motion_max_size(a.T, a.J));
  const size_t need = zeggs_bvh_format_motion_workspace_size(a.T, a.J);
  ZCHECK_ARG(a.workspace && a.workspace_bytes >= need, "bvh format: workspace of %zu bytes, %zu needed", a.workspace_bytes, need);
  cudaStream_t s = (cudaStream_t)stream;
  ZCHECK_CUDA(cudaMemsetAsync(a.status, 0, 2 * sizeof(long long), s));
  if (a.T == 0) {
    ZCHECK_CUDA(cudaMemsetAsync(a.row_start, 0, sizeof(long long), s));
    return ZEGGS_OK;
  }
  const int C = 3 + 3 * a.J;
  const long long V = (long long)a.T * C;
  long long* chunk;
  format_carve((char*)a.workspace, V, &chunk);
  const int nchunks = (int)((V + BT_VALUE_CHUNK - 1) / BT_VALUE_CHUNK);
  bt_format_count_kernel<<<nchunks, BT_THREADS, 0, s>>>(a, C, V, chunk);
  LAUNCH_OK();
  bt_scan_kernel<long long><<<1, BT_THREADS, 0, s>>>(chunk, nchunks, a.status, (long long)1 << 62);   // status[0] = total bytes
  LAUNCH_OK();
  bt_format_write_kernel<<<nchunks, BT_THREADS, 0, s>>>(a, C, V, chunk);
  LAUNCH_OK();
  return ZEGGS_OK;
}

}  // namespace zeggs
