// Geometry / workspace of the decoder backward shared by the fp32 SIMT and the tensor-core recurrences.
#pragma once
#include "decoder_common.cuh"

namespace zeggs {

struct BwdGeom {
  int R1;        // padded rows of the CTA's B1 tiles (>= U, multiple of 8; film_rows(pass_units(U)) per pass)
  int rpcb;      // x_pose-gradient rows per CTA (>= 9)
  int n4b;       // 16-row tiles per CTA for those rows
  size_t off2, off3a, off3b, off4, total;
};

__host__ __device__ inline int xp_perm(int m) {   // permuted row -> natural x_pose row
  if (m < 6) return m;
  if (m < 9) return P_OUT + (m - 6);
  return m - 3;
}

inline BwdGeom make_bgeom(const DecGeom& g) {
  BwdGeom b;
  b.R1 = g.U < 8 ? 8 : g.U;
  b.rpcb = ceil_div(P_IN, g.G) < 9 ? 9 : ceil_div(P_IN, g.G);
  b.n4b = ceil_div(b.rpcb, 16);
  b.off2 = (size_t)g.G * K1P * b.R1;
  b.off3a = b.off2 + (size_t)g.G * 3 * g.H * 2 * g.U;
  b.off3b = b.off3a + (size_t)g.G * 3 * g.H * 2 * g.U;
  b.off4 = b.off3b + (size_t)g.G * b.n4b * 3 * g.H * 16;
  b.total = b.off4 + (size_t)g.G * b.n4b * g.H * 16;
  return b;
}

struct BwdWs {
  unsigned* bar;
  float *DY, *DGI1, *DGH1, *DGI0, *DGH0, *DPA, *DH0, *DH1, *COND, *DCOND;
  float *cse_dout, *cse_d2, *cse_d1, *cse_din;
  float* DCH;   // tc engine: [T][32][8] d loss / d y(t)[0:6] through the root-integration chain
  size_t bytes;
};

inline BwdWs make_bws(void* base, const DecGeom& g, int T) {
  BwdWs w;
  Arena a{(char*)base};
  const size_t S = (size_t)T * g.nbt;
  const int C = g.S + g.Z;
  w.bar = (unsigned*)a.take(64);
  w.DY = a.take(S * K1P * 32);
  w.DGI1 = a.take(S * 3 * g.H * 32); w.DGH1 = a.take(S * 3 * g.H * 32);
  w.DGI0 = a.take(S * 3 * g.H * 32); w.DGH0 = a.take(S * 3 * g.H * 32);
  w.DPA = a.take(S * g.H * 32);
  w.DH0 = a.take((size_t)g.nbt * g.H * 32); w.DH1 = a.take((size_t)g.nbt * g.H * 32);
  w.COND = a.take(S * C * 32); w.DCOND = a.take(S * C * 32);
  w.cse_dout = a.take((size_t)g.B * 2 * g.H); w.cse_d2 = a.take((size_t)g.B * g.H); w.cse_d1 = a.take((size_t)g.B * g.H);
  w.cse_din = a.take((size_t)g.B * (P_IN + g.Z));
  w.DCH = a.take((size_t)T * 32 * 8);
  w.bytes = a.off;
  return w;
}

struct BwdArgsDev {
  const float *dY, *dRootPos, *dRootRot;   // upstream grads (may be null)
  const float* packed;
};

// ------------------------------------------------------------------ host steps shared by the two backward routines
// Weight gradients (slots t = 1..T-1) on the tensor cores: each of the 11 fp32 histories is re-laid out once as bf16 hi (and lo)
// [rows][T*nbt*32] (contraction index contiguous) from the base of the scratch buffer, all hi parts first, then all lo parts.  (ld * 2)
// bytes per row keep every copy 16 B aligned, so consecutive histories stack into ONE row-contiguous operand ([a | x_pose | cond] is
// the input of layer0 / GRU0 in the weights' own column order).  Each dW is one NT GEMM with K = (T-1)*nbt*32; "previous step"
// operands are the same copy shifted by one slot (32*nbt columns).
enum { HDY, HGI1, HGH1, HGI0, HGH0, HPA, HH0, HH1, HA, HXP, HCOND, NHIST };
struct WgradHist { const float* src; long long stride; int rows; __nv_bfloat16 *hi, *lo; float* db; };   // db: bias gradient
struct WgradHists {
  WgradHist h[NHIST];
  int slots, nbt;     // slots per history (T * nbt), batch tiles
  size_t ld, bytes;   // columns of every copy (slots * 32), bytes of all copies (from the scratch base)
};
// The table and the carve-up, host arithmetic only: calls with the same geometry and scratch buffer return the same addresses.
WgradHists wgrad_hists(const zeggs_decoder_fwd_args& a, const zeggs_decoder_bwd_args& b, const DecGeom& g, const DecWs& w,
                       const BwdWs& bw, bool want_lo);
int split_hist(const WgradHists& hs, int i, cudaStream_t stream);
// the six GEMMs; split-K partials go to the rest of the scratch buffer behind `tail` (an arena over it)
int wgrad_gemms(const zeggs_decoder_fwd_args& a, const zeggs_decoder_bwd_args& b, const DecGeom& g, const WgradHists& hs, bool want_lo,
                Arena tail, cudaStream_t stream);
int cond_kmajor(const zeggs_decoder_fwd_args& a, const DecGeom& g, const BwdWs& bw, cudaStream_t stream);
// CellStateEncoder backward (modules.py:238-243); its small GEMMs stage operands at the base of the scratch buffer
int cse_backward(const zeggs_decoder_fwd_args& a, const zeggs_decoder_bwd_args& b, const DecWs& w, const BwdWs& bw, cudaStream_t stream);
int dcond_scatter(const zeggs_decoder_fwd_args& a, const zeggs_decoder_bwd_args& b, const DecGeom& g, const BwdWs& bw, int rows,
                  cudaStream_t stream);
int dy_combine(const zeggs_decoder_fwd_args& a, const zeggs_decoder_bwd_args& b, const float* dxp, const BwdWs& bw, cudaStream_t stream);
int decoder_window_bwd_tc(const zeggs_decoder_fwd_args& a, const zeggs_decoder_bwd_args& b, const DecGeom& g, const DecWs& w,
                          const BwdWs& bw, cudaStream_t stream);

}  // namespace zeggs
