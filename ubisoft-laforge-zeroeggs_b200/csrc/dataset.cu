// Training-set construction on the device (ZEGGS/data_pipeline.py:90-228, 412-432, 562-648):
//   zeggs_anim_features   per-frame animation features of one take (preprocess_animation), float64 arithmetic, float32 out
//   zeggs_spline_resample the time-stretch (griddata(method="cubic") in 1-D = interp1d(kind="cubic"), a not-a-knot cubic spline)
//   zeggs_masked_moments  per-channel means / population stds and pooled group stds over the training rows
// No atomics: every reduction and scan runs in a fixed order, so two runs give bitwise-identical results.
#include <cmath>
#include "common.cuh"
#include "../../include/zeggs_b200.h"

namespace zeggs { void count_launch(); }

namespace zeggs_ds {

struct D3 { double x, y, z; };
struct DQ { double w, x, y, z; };

__device__ __forceinline__ D3 d3(double x, double y, double z) { D3 r; r.x = x; r.y = y; r.z = z; return r; }
__device__ __forceinline__ D3 sub(D3 a, D3 b) { return d3(a.x - b.x, a.y - b.y, a.z - b.z); }
__device__ __forceinline__ D3 scale(D3 a, double s) { return d3(a.x * s, a.y * s, a.z * s); }
__device__ __forceinline__ D3 cross(D3 a, D3 b) { return d3(a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x); }
__device__ __forceinline__ DQ qmul(DQ a, DQ b) {
  DQ r;
  r.w = a.w * b.w - a.x * b.x - a.y * b.y - a.z * b.z;
  r.x = a.w * b.x + a.x * b.w + a.y * b.z - a.z * b.y;
  r.y = a.w * b.y - a.x * b.z + a.y * b.w + a.z * b.x;
  r.z = a.w * b.z + a.x * b.y - a.y * b.x + a.z * b.w;
  return r;
}
__device__ __forceinline__ DQ qinv(DQ q) { q.x = -q.x; q.y = -q.y; q.z = -q.z; return q; }
// quat.py mul_vec: v + w t + u x t with t = 2 u x v
__device__ __forceinline__ D3 qrot(DQ q, D3 v) {
  const D3 u = d3(q.x, q.y, q.z);
  D3 t = cross(u, v);
  t = scale(t, 2.0);
  const D3 c = cross(u, t);
  return d3(v.x + q.w * t.x + c.x, v.y + q.w * t.y + c.y, v.z + q.w * t.z + c.z);
}
// quat.py:49-67: abs (the sign that makes w > 0) then to_helical = 2 log(q), eps 1e-5
__device__ __forceinline__ D3 helical_abs(DQ q) {
  if (!(q.w > 0.0)) { q.w = -q.w; q.x = -q.x; q.y = -q.y; q.z = -q.z; }
  const double len = sqrt(q.x * q.x + q.y * q.y + q.z * q.z);
  const double half = len < 1e-5 ? 1.0 : atan2(len, q.w) / len;
  return d3(2.0 * half * q.x, 2.0 * half * q.y, 2.0 * half * q.z);
}
__device__ __forceinline__ D3 load3(const double* p) { return d3(p[0], p[1], p[2]); }
__device__ __forceinline__ void store3(float* p, D3 v) { p[0] = (float)v.x; p[1] = (float)v.y; p[2] = (float)v.z; }
__device__ __forceinline__ void store4(float* p, DQ q) { p[0] = (float)q.w; p[1] = (float)q.x; p[2] = (float)q.y; p[3] = (float)q.z; }

// quat.py:154-163: from_euler(radians(e), order) = q(order[0]) * (q(order[1]) * q(order[2]))
__device__ __forceinline__ DQ from_euler_deg(const double* e, int a0, int a1, int a2) {
  const int axis[3] = {a0, a1, a2};
  DQ q[3];
  for (int i = 0; i < 3; ++i) {
    const double a = e[i] * (M_PI / 180.0);
    const double c = cos(a / 2.0), s = sin(a / 2.0);
    q[i].w = c; q[i].x = axis[i] == 0 ? s : 0.0; q[i].y = axis[i] == 1 ? s : 0.0; q[i].z = axis[i] == 2 ? s : 0.0;
  }
  return qmul(q[0], qmul(q[1], q[2]));
}

// ================================================================================================ animation features
// unroll (quat.py:130-136) flips frame t when dot(q_t, y_{t-1}) < 0, y the already unrolled sequence.  With s_t the sign given to
// frame t and d_t = dot(raw_t, raw_{t-1}): s_t = s_{t-1} if d_t > 0, -s_{t-1} if d_t < 0, +1 if d_t == 0.  Each frame is thus the
// map s -> a s + b on {-1, +1} (keep (1, 0), negate (-1, 0), reset (0, 1)); composing the maps is an exact prefix scan.
struct SignOp { int a, b; };
__device__ __forceinline__ SignOp compose(SignOp first, SignOp then) { SignOp r; r.a = then.a * first.a; r.b = then.a * first.b + then.b; return r; }
__device__ __forceinline__ SignOp decode(signed char c) { SignOp o; o.a = c == 2 ? 0 : (c == 1 ? -1 : 1); o.b = c == 2 ? 1 : 0; return o; }

__global__ void __launch_bounds__(256) euler_to_quat_kernel(const double* __restrict__ rot, DQ* __restrict__ q, size_t n, int a0, int a1, int a2) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    q[i] = from_euler_deg(rot + i * 3, a0, a1, a2);
}

__global__ void __launch_bounds__(256) sign_op_kernel(const DQ* __restrict__ q, signed char* __restrict__ op, int T, int J) {
  const size_t n = (size_t)T * J;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    if (i < (size_t)J) { op[i] = 2; continue; }           // frame 0 keeps its sign
    const DQ c = q[i], p = q[i - J];
    const double d = c.w * p.w + c.x * p.x + c.y * p.y + c.z * p.z;
    op[i] = d > 0.0 ? 0 : (d < 0.0 ? 1 : 2);
  }
}

// one block per joint: thread k composes frames [k L, (k+1) L), a block scan of the 256 compositions, then each thread applies
__global__ void __launch_bounds__(256) unroll_kernel(DQ* __restrict__ q, const signed char* __restrict__ op, int T, int J) {
  const int j = blockIdx.x;
  const int L = (T + blockDim.x - 1) / blockDim.x;
  const int t0 = min(T, (int)threadIdx.x * L), t1 = min(T, t0 + L);
  SignOp acc; acc.a = 1; acc.b = 0;
  for (int t = t0; t < t1; ++t) acc = compose(acc, decode(op[(size_t)t * J + j]));
  __shared__ SignOp sh[256];
  sh[threadIdx.x] = acc;
  __syncthreads();
  for (int off = 1; off < (int)blockDim.x; off <<= 1) {
    SignOp v = sh[threadIdx.x];
    if ((int)threadIdx.x >= off) v = compose(sh[threadIdx.x - off], v);
    __syncthreads();
    sh[threadIdx.x] = v;
    __syncthreads();
  }
  int s = 1;                                              // any start value: frame 0 resets it
  if (threadIdx.x > 0) { const SignOp p = sh[threadIdx.x - 1]; s = p.a * s + p.b; }
  for (int t = t0; t < t1; ++t) {
    const SignOp o = decode(op[(size_t)t * J + j]);
    s = o.a * s + o.b;
    if (s < 0) { DQ& x = q[(size_t)t * J + j]; x.w = -x.w; x.x = -x.x; x.y = -x.y; x.z = -x.z; }
  }
}

// global transform of joint k from the local ones, walking up its chain (the reference's fk() composes the same products top-down)
__device__ __forceinline__ void chain_fk(const DQ* q, const double* pos, const int* parents, int J, int k, DQ& R, D3& P) {
  R = q[k]; P = load3(pos + (size_t)k * 3);
  for (int p = parents[k]; p >= 0; p = parents[p]) {
    P = qrot(q[p], P); P.x += pos[(size_t)p * 3]; P.y += pos[(size_t)p * 3 + 1]; P.z += pos[(size_t)p * 3 + 2];
    R = qmul(q[p], R);
  }
}

// per frame (data_pipeline.py:99-125): ground-projected Spine2, facing from the Hips' z axis, gaze target 100 units along the Head's
__global__ void __launch_bounds__(128) root_kernel(zeggs_anim_features_args a, const DQ* __restrict__ q, D3* __restrict__ root_pos,
                                                   DQ* __restrict__ root_rot, double* __restrict__ gaze_all) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= a.T) return;
  const DQ* qt = q + (size_t)t * a.J;
  const double* pt = a.positions + (size_t)t * a.J * 3;
  DQ R; D3 P;
  chain_fk(qt, pt, a.parents, a.J, a.spine2, R, P);
  const D3 rp = d3(P.x * 1.0, P.y * 0.0, P.z * 1.0);
  chain_fk(qt, pt, a.parents, a.J, a.hips, R, P);
  D3 f = qrot(R, d3(0.0, 0.0, 1.0));
  f.y = 0.0;
  f = scale(f, 1.0 / sqrt(f.x * f.x + f.y * f.y + f.z * f.z));
  // quat.between([0,0,1], f) then normalize
  const D3 c = cross(d3(0.0, 0.0, 1.0), f);
  DQ rr; rr.w = sqrt(1.0 * (f.x * f.x + f.y * f.y + f.z * f.z)) + f.z; rr.x = c.x; rr.y = c.y; rr.z = c.z;
  const double nr = sqrt(rr.w * rr.w + rr.x * rr.x + rr.y * rr.y + rr.z * rr.z);
  rr.w /= nr; rr.x /= nr; rr.y /= nr; rr.z /= nr;
  chain_fk(qt, pt, a.parents, a.J, a.head, R, P);
  D3 g = qrot(R, d3(0.0, 0.0, 1.0));
  g.y = 0.0;
  g = scale(g, 1.0 / sqrt(g.x * g.x + g.y * g.y + g.z * g.z));
  root_pos[t] = rp;
  root_rot[t] = rr;
  gaze_all[t] = rp.x + 100.0 * g.x;
  gaze_all[(size_t)a.T + t] = rp.y + 100.0 * g.y;
  gaze_all[2 * (size_t)a.T + t] = rp.z + 100.0 * g.z;
}

// exact median per component (np.median: the middle value, or the mean of the two middle values when T is even).  Thread i owns
// value v_i and counts the values below and equal to it; v_i holds every rank in [less, less + equal).  Equal values write equal bits.
__global__ void __launch_bounds__(256) median_select_kernel(const double* __restrict__ v, int T, double* __restrict__ sel) {
  const int comp = blockIdx.y;
  const double* x = v + (size_t)comp * T;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const double xi = i < T ? x[i] : 0.0;
  __shared__ double tile[256];
  int less = 0, equal = 0;
  for (int base = 0; base < T; base += 256) {
    __syncthreads();
    if (base + (int)threadIdx.x < T) tile[threadIdx.x] = x[base + threadIdx.x];
    __syncthreads();
    const int n = min(256, T - base);
    for (int k = 0; k < n; ++k) { const double y = tile[k]; less += y < xi; equal += y == xi; }
  }
  if (i >= T) return;
  const int k_lo = (T - 1) / 2, k_hi = T / 2;
  if (less <= k_lo && k_lo < less + equal) sel[comp * 2] = xi;
  if (less <= k_hi && k_hi < less + equal) sel[comp * 2 + 1] = xi;
}

struct FeatCtx {
  zeggs_anim_features_args a;
  const DQ* q;
  const D3* root_pos;
  const DQ* root_rot;
};

// joint j of frame t made relative to the root (data_pipeline.py:145-147); other joints unchanged
__device__ __forceinline__ D3 rel_pos(const FeatCtx& c, int t, int j) {
  const D3 p = load3(c.a.positions + ((size_t)t * c.a.J + j) * 3);
  return j == 0 ? qrot(qinv(c.root_rot[t]), sub(p, c.root_pos[t])) : p;
}
__device__ __forceinline__ DQ rel_rot(const FeatCtx& c, int t, int j) {
  const DQ r = c.q[(size_t)t * c.a.J + j];
  return j == 0 ? qmul(qinv(c.root_rot[t]), r) : r;
}
// finite differences for t >= 1 (data_pipeline.py:150-156)
__device__ __forceinline__ D3 lvel_at(const FeatCtx& c, int t, int j) { return scale(sub(rel_pos(c, t, j), rel_pos(c, t - 1, j)), 1.0 / c.a.dt); }
__device__ __forceinline__ D3 lvrt_at(const FeatCtx& c, int t, int j) {
  return scale(helical_abs(qmul(rel_rot(c, t, j), qinv(rel_rot(c, t - 1, j)))), 1.0 / c.a.dt);
}
__device__ __forceinline__ D3 rvel_at(const FeatCtx& c, int t) { return scale(sub(c.root_pos[t], c.root_pos[t - 1]), 1.0 / c.a.dt); }
__device__ __forceinline__ D3 rvrt_at(const FeatCtx& c, int t) {
  return scale(helical_abs(qmul(c.root_rot[t], qinv(c.root_rot[t - 1]))), 1.0 / c.a.dt);
}
// frame 0: v1 - (v3 - v2)
__device__ __forceinline__ D3 extrap(D3 v1, D3 v2, D3 v3) { return sub(v1, sub(v3, v2)); }

__global__ void __launch_bounds__(256) joint_feature_kernel(FeatCtx c, const double* __restrict__ sel) {
  const zeggs_anim_features_args& a = c.a;
  const size_t n = (size_t)a.T * a.J;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const int t = (int)(i / a.J), j = (int)(i % a.J);
    store3(a.lpos + i * 3, rel_pos(c, t, j));
    const DQ r = rel_rot(c, t, j);
    store3(a.ltxy + i * 6, qrot(r, d3(1.0, 0.0, 0.0)));
    store3(a.ltxy + i * 6 + 3, qrot(r, d3(0.0, 1.0, 0.0)));
    store3(a.lvel + i * 3, t > 0 ? lvel_at(c, t, j) : extrap(lvel_at(c, 1, j), lvel_at(c, 2, j), lvel_at(c, 3, j)));
    store3(a.lvrt + i * 3, t > 0 ? lvrt_at(c, t, j) : extrap(lvrt_at(c, 1, j), lvrt_at(c, 2, j), lvrt_at(c, 3, j)));
    if (j != 0) continue;
    // per-frame channels (data_pipeline.py:126-169): velocities in the previous frame's root space, frame 0 in its own
    const DQ rr = c.root_rot[t];
    const DQ prev_inv = qinv(c.root_rot[t > 0 ? t - 1 : 0]);
    const D3 rv = t > 0 ? rvel_at(c, t) : extrap(rvel_at(c, 1), rvel_at(c, 2), rvel_at(c, 3));
    const D3 rw = t > 0 ? rvrt_at(c, t) : extrap(rvrt_at(c, 1), rvrt_at(c, 2), rvrt_at(c, 3));
    store3(a.root_vel + (size_t)t * 3, qrot(prev_inv, rv));
    store3(a.root_vrt + (size_t)t * 3, qrot(prev_inv, rw));
    store3(a.root_pos + (size_t)t * 3, c.root_pos[t]);
    store4(a.root_rot + (size_t)t * 4, rr);
    D3 gp;
    if (a.T & 1) gp = d3(sel[0], sel[2], sel[4]);
    else gp = d3((sel[0] + sel[1]) / 2.0, (sel[2] + sel[3]) / 2.0, (sel[4] + sel[5]) / 2.0);
    store3(a.gaze_pos + (size_t)t * 3, gp);
    store3(a.gaze_dir + (size_t)t * 3, qrot(qinv(rr), sub(gp, c.root_pos[t])));
  }
}

struct FeatWs { DQ* q; signed char* op; D3* root_pos; DQ* root_rot; double* gaze; double* sel; size_t bytes; };
static FeatWs feat_ws(void* base, int T, int J) {
  auto up = [](size_t x) { return (x + 255) & ~(size_t)255; };
  FeatWs w;
  char* p = (char*)base;
  size_t o = 0;
  w.q = (DQ*)(p + o); o += up(sizeof(DQ) * (size_t)T * J);
  w.op = (signed char*)(p + o); o += up((size_t)T * J);
  w.root_pos = (D3*)(p + o); o += up(sizeof(D3) * (size_t)T);
  w.root_rot = (DQ*)(p + o); o += up(sizeof(DQ) * (size_t)T);
  w.gaze = (double*)(p + o); o += up(sizeof(double) * 3 * (size_t)T);
  w.sel = (double*)(p + o); o += up(sizeof(double) * 6);
  w.bytes = o;
  return w;
}
static unsigned grid_for(size_t n, int block) { const size_t b = (n + block - 1) / block; return (unsigned)(b > 132 * 32 ? 132 * 32 : (b ? b : 1)); }

// quat.normalize then quat.to_euler (quat.py:92-93, 111-127) then np.degrees: the stretched rotations back to BVH channels
__global__ void __launch_bounds__(256) quat_to_euler_kernel(const double* __restrict__ q, double* __restrict__ e, long long n, int order) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const double* p = q + i * 4;
    const double nrm = sqrt(p[0] * p[0] + p[1] * p[1] + p[2] * p[2] + p[3] * p[3]) + 0.0;
    const double x0 = p[0] / nrm, x1 = p[1] / nrm, x2 = p[2] / nrm, x3 = p[3] / nrm;
    double a, b, c;
    if (order == 0) {          // zyx
      a = atan2(2.0 * (x0 * x3 + x1 * x2), 1.0 - 2.0 * (x2 * x2 + x3 * x3));
      b = asin(fmin(fmax(2.0 * (x0 * x2 - x3 * x1), -1.0), 1.0));
      c = atan2(2.0 * (x0 * x1 + x2 * x3), 1.0 - 2.0 * (x1 * x1 + x2 * x2));
    } else {                   // xzy
      a = atan2(2.0 * (x1 * x0 - x2 * x3), -x1 * x1 + x2 * x2 - x3 * x3 + x0 * x0);
      b = atan2(2.0 * (x2 * x0 - x1 * x3), x1 * x1 - x2 * x2 - x3 * x3 + x0 * x0);
      c = asin(fmin(fmax(2.0 * (x1 * x2 + x3 * x0), -1.0), 1.0));
    }
    const double r2d = 180.0 / M_PI;
    e[i * 3] = a * r2d; e[i * 3 + 1] = b * r2d; e[i * 3 + 2] = c * r2d;
  }
}

// ================================================================================================ not-a-knot cubic spline
// On the uniform grid x_i = i the second derivatives M solve M_{i-1} + 4 M_i + M_{i+1} = 6 d_i (d_i = y_{i-1} - 2 y_i + y_{i+1})
// for i = 1 .. n-2, and not-a-knot (M_0 = 2 M_1 - M_2, M_{n-1} = 2 M_{n-2} - M_{n-3}) reduces rows 1 and n-2 to M_1 = d_1 and
// M_{n-2} = d_{n-2}.  The interior is the Toeplitz system [1 4 1] with known ends.  Its infinite-grid inverse is
// g_k = g0 (-r)^|k| (r = 2 - sqrt 3, g0 = 1 / (2 sqrt 3)), so with the right-hand side restricted to i = 2 .. n-3:
//   M~_i = g0 (P_i + Q_i),  P_i = sum_{k <= i} (-r)^(i-k) rhs_k,  Q_i = sum_{k > i} (-r)^(k-i) rhs_k
// (one causal and one anticausal first-order recursion), and the exact solution adds the two decaying homogeneous solutions
// alpha (-r)^(i-1) + beta (-r)^(n-2-i) that restore M_1 = d_1 and M_{n-2} = d_{n-2}.  A chunk of S values runs both recursions
// from a halo of H samples beyond its ends: the dropped terms weigh r^H < 1e-27 (H = 48), so chunks are independent to fp64
// rounding, and at the true ends (k = 2, n-3) the recursions start exactly.
constexpr double kR = 0.26794919243112270;     // 2 - sqrt(3)
constexpr double kG0 = 0.28867513459481287;    // 1 / (2 sqrt(3))
constexpr int kChunk = 256, kHalo = 48;

template <typename Tin>
__device__ __forceinline__ double rhs_at(const Tin* y, long long n, int C, int c, long long k) {
  if (k < 2 || k > n - 3) return 0.0;
  return 6.0 * (((double)y[(k - 1) * C + c] - 2.0 * (double)y[k * C + c]) + (double)y[(k + 1) * C + c]);
}

template <typename Tin>
__global__ void __launch_bounds__(128) spline_mtilde_kernel(const Tin* __restrict__ y, long long n, int C, double* __restrict__ M) {
  const long long n_chunks = (n + kChunk - 1) / kChunk;
  const long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (idx >= n_chunks * C) return;
  const int c = (int)(idx % C);
  const long long ch = idx / C;
  const long long i0 = ch * kChunk, i1 = min(n, i0 + kChunk);
  double P = 0.0;
  for (long long k = max(1LL, i0 - kHalo); k < i1; ++k) {
    P = rhs_at(y, n, C, c, k) - kR * P;
    if (k >= i0) M[k * C + c] = kG0 * P;
  }
  double Q = 0.0;                                      // Q_k for k = top, truncated
  for (long long k = min(n - 2, i1 - 1 + kHalo); k >= max(1LL, i0); --k) {
    if (k < i1) M[k * C + c] += kG0 * Q;
    Q = -kR * (rhs_at(y, n, C, c, k) + Q);              // -> Q_{k-1}
  }
}

__device__ __forceinline__ double powr(long long e) {   // (-r)^e, 0 once it is below fp64 resolution of the solution
  if (e >= 64) return 0.0;
  double p = 1.0;
  for (long long i = 0; i < e; ++i) p *= -kR;
  return p;
}

template <typename Tin>
__global__ void spline_ab_kernel(const Tin* __restrict__ y, long long n, int C, const double* __restrict__ M, double* __restrict__ ab) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  auto d = [&](long long i) { return ((double)y[(i - 1) * C + c] - 2.0 * (double)y[i * C + c]) + (double)y[(i + 1) * C + c]; };
  const double e1 = d(1) - M[1 * C + c], e2 = d(n - 2) - M[(n - 2) * C + c];
  const double rho = powr(n - 3);
  const double det = 1.0 - rho * rho;
  ab[2 * c] = (e1 - rho * e2) / det;
  ab[2 * c + 1] = (e2 - rho * e1) / det;
}

__global__ void __launch_bounds__(256) spline_fix_kernel(long long n, int C, double* __restrict__ M, const double* __restrict__ ab) {
  const long long total = (n - 2) * C;
  for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    const long long i = 1 + idx / C;
    const int c = (int)(idx % C);
    const long long e1 = i - 1, e2 = n - 2 - i;
    double v = M[i * C + c];
    if (e1 < 64) v += ab[2 * c] * powr(e1);
    if (e2 < 64) v += ab[2 * c + 1] * powr(e2);
    M[i * C + c] = v;
  }
}

template <typename Tin>
__global__ void __launch_bounds__(256) spline_eval_kernel(const Tin* __restrict__ y, long long n, long long m, int C,
                                                          const double* __restrict__ M, double* __restrict__ out) {
  const long long total = m * C;
  const double step = m > 1 ? (double)(n - 1) / (double)(m - 1) : 0.0;          // np.linspace(0, n-1, m)
  for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    const long long k = idx / C;
    const int c = (int)(idx % C);
    const double x = (m > 1 && k == m - 1) ? (double)(n - 1) : (double)k * step;
    long long i = (long long)floor(x);
    if (i > n - 2) i = n - 2;
    if (i < 0) i = 0;
    const double t = x - (double)i, u = 1.0 - t;
    auto Mi = [&](long long j) {
      if (j == 0) return 2.0 * M[1 * C + c] - M[2 * C + c];
      if (j == n - 1) return 2.0 * M[(n - 2) * C + c] - M[(n - 3) * C + c];
      return M[j * C + c];
    };
    const double m0 = Mi(i), m1 = Mi(i + 1);
    const double y0 = (double)y[i * C + c], y1 = (double)y[(i + 1) * C + c];
    out[idx] = u * y0 + t * y1 + ((u * u * u - u) * m0 + (t * t * t - t) * m1) / 6.0;
  }
}

// ================================================================================================ masked moments
constexpr int kRowsPerChunk = 256;

__device__ __forceinline__ int group_of(const zeggs_moments_args& a, int c, int& col) {
  int off = 0;
  for (int g = 0; g < a.n_groups; ++g) {
    if (c < off + a.width[g]) { col = c - off; return g; }
    off += a.width[g];
  }
  col = 0;
  return 0;
}

// pass 0: per-(row chunk, channel) sums of x.  pass 1: sums of (x - mean_c)^2 and (x - mean_group)^2.
template <int PASS>
__global__ void __launch_bounds__(256) moments_partial_kernel(zeggs_moments_args a, int W, double* __restrict__ part0,
                                                              double* __restrict__ part1, const double* __restrict__ gmean) {
  const long long ch = blockIdx.x;
  const long long r0 = ch * kRowsPerChunk, r1 = min(a.n_sel, r0 + kRowsPerChunk);
  for (int c = threadIdx.x; c < W; c += blockDim.x) {
    int col;
    const int g = group_of(a, c, col);
    const float* src = a.src[g];
    const int w = a.width[g];
    double s0 = 0.0, s1 = 0.0;
    const double mc = PASS ? a.mean[c] : 0.0, mg = PASS ? gmean[g] : 0.0;
    for (long long r = r0; r < r1; ++r) {
      const double x = (double)src[(long long)a.rows[r] * w + col];
      if (PASS == 0) {
        s0 += x;
      } else {
        const double d0 = x - mc, d1 = x - mg;
        s0 += d0 * d0; s1 += d1 * d1;
      }
    }
    part0[ch * W + c] = s0;
    if (PASS) part1[ch * W + c] = s1;
  }
}

template <int PASS>
__global__ void __launch_bounds__(256) moments_channel_kernel(zeggs_moments_args a, int W, long long n_chunks, const double* __restrict__ part0,
                                                              const double* __restrict__ part1, double* __restrict__ csum) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= W) return;
  double s0 = 0.0, s1 = 0.0;
  for (long long ch = 0; ch < n_chunks; ++ch) { s0 += part0[ch * W + c]; if (PASS) s1 += part1[ch * W + c]; }
  const double n = (double)a.n_sel;
  if (PASS == 0) { a.mean[c] = s0 / n; csum[c] = s0; }
  else { a.std[c] = sqrt(s0 / n); csum[c] = s1; }
}

// one thread per group, channels in order: pass 0 the group mean, pass 1 the pooled std
template <int PASS>
__global__ void moments_group_kernel(zeggs_moments_args a, const double* __restrict__ csum, double* __restrict__ gmean) {
  const int g = threadIdx.x;
  if (g >= a.n_groups) return;
  int off = 0;
  for (int k = 0; k < g; ++k) off += a.width[k];
  double s = 0.0;
  for (int c = off; c < off + a.width[g]; ++c) s += csum[c];
  const double n = (double)a.n_sel * (double)a.width[g];
  if (PASS == 0) gmean[g] = s / n;
  else a.group_std[g] = sqrt(s / n);
}

}  // namespace zeggs_ds

using namespace zeggs;
using namespace zeggs_ds;

extern "C" size_t zeggs_anim_features_workspace_bytes(int T, int J) {
  if (T < 1 || J < 1) return 0;
  return feat_ws(nullptr, T, J).bytes;
}

extern "C" int zeggs_anim_features(const zeggs_anim_features_args* ap, void* stream) {
  ZCHECK_ARG(ap, "anim features: null args");
  const zeggs_anim_features_args& a = *ap;
  ZCHECK_ARG(a.T >= 4, "anim features: T = %d frames, at least 4 are needed (frame 0's velocities are extrapolated from frames 1..3)", a.T);
  ZCHECK_ARG(a.J >= 1, "anim features: J = %d", a.J);
  for (int i = 0; i < 3; ++i) ZCHECK_ARG(a.order[i] >= 0 && a.order[i] <= 2, "anim features: order[%d] = %d is not an axis (0 x, 1 y, 2 z)", i, a.order[i]);
  ZCHECK_ARG(a.rotations && a.parents && a.workspace, "anim features: null pointer");
  const bool features = a.positions != nullptr;
  ZCHECK_ARG(features || a.quat_out, "anim features: neither positions (features) nor quat_out (unroll) given");
  if (features) {
    ZCHECK_ARG(a.spine2 >= 0 && a.spine2 < a.J && a.hips >= 0 && a.hips < a.J && a.head >= 0 && a.head < a.J, "anim features: joint index out of range");
    ZCHECK_ARG(a.dt > 0.0, "anim features: dt = %g", a.dt);
    ZCHECK_ARG(a.root_pos && a.root_rot && a.root_vel && a.root_vrt && a.lpos && a.ltxy && a.lvel && a.lvrt && a.gaze_pos && a.gaze_dir,
               "anim features: null output");
  }
  const FeatWs w = feat_ws(a.workspace, a.T, a.J);
  ZCHECK_ARG(a.workspace_bytes >= w.bytes, "anim features: workspace %zu < %zu bytes", a.workspace_bytes, w.bytes);
  cudaStream_t s = (cudaStream_t)stream;
  const size_t n = (size_t)a.T * a.J;
  euler_to_quat_kernel<<<grid_for(n, 256), 256, 0, s>>>(a.rotations, w.q, n, a.order[0], a.order[1], a.order[2]);
  count_launch();
  sign_op_kernel<<<grid_for(n, 256), 256, 0, s>>>(w.q, w.op, a.T, a.J);
  count_launch();
  unroll_kernel<<<a.J, 256, 0, s>>>(w.q, w.op, a.T, a.J);
  count_launch();
  ZCHECK_LAUNCH();
  if (a.quat_out) ZCHECK_CUDA(cudaMemcpyAsync(a.quat_out, w.q, sizeof(DQ) * n, cudaMemcpyDeviceToDevice, s));
  if (!features) return ZEGGS_OK;
  root_kernel<<<ceil_div(a.T, 128), 128, 0, s>>>(a, w.q, w.root_pos, w.root_rot, w.gaze);
  count_launch();
  median_select_kernel<<<dim3(ceil_div(a.T, 256), 3), 256, 0, s>>>(w.gaze, a.T, w.sel);
  count_launch();
  FeatCtx c; c.a = a; c.q = w.q; c.root_pos = w.root_pos; c.root_rot = w.root_rot;
  joint_feature_kernel<<<grid_for(n, 256), 256, 0, s>>>(c, w.sel);
  count_launch();
  ZCHECK_LAUNCH();
  return ZEGGS_OK;
}

extern "C" int zeggs_quat_to_euler_deg(const double* q, double* euler_deg, long long n, int order, void* stream) {
  ZCHECK_ARG(n >= 0 && (n == 0 || (q && euler_deg)), "quat to euler: bad arguments");
  ZCHECK_SUPPORTED(order == 0 || order == 1, "quat to euler: order %d (0 = zyx and 1 = xzy are the orders quat.to_euler converts to)", order);
  if (n == 0) return ZEGGS_OK;
  quat_to_euler_kernel<<<grid_for((size_t)n, 256), 256, 0, (cudaStream_t)stream>>>(q, euler_deg, n, order);
  count_launch();
  ZCHECK_LAUNCH();
  return ZEGGS_OK;
}

extern "C" size_t zeggs_spline_resample_workspace_bytes(long long n, int C) {
  if (n < 4 || C < 1) return 0;
  return sizeof(double) * ((size_t)n * C + 2 * (size_t)C);
}

extern "C" int zeggs_spline_resample(const zeggs_spline_args* ap, void* stream) {
  ZCHECK_ARG(ap, "spline: null args");
  const zeggs_spline_args& a = *ap;
  ZCHECK_ARG(a.n >= 4, "spline: n = %lld samples, a cubic spline needs at least 4", a.n);
  ZCHECK_ARG(a.m >= 0 && a.C >= 1, "spline: m = %lld, C = %d", a.m, a.C);
  ZCHECK_ARG(a.x && a.y && a.workspace, "spline: null pointer");
  const size_t need = zeggs_spline_resample_workspace_bytes(a.n, a.C);
  ZCHECK_ARG(a.workspace_bytes >= need, "spline: workspace %zu < %zu bytes", a.workspace_bytes, need);
  if (a.m == 0) return ZEGGS_OK;
  cudaStream_t s = (cudaStream_t)stream;
  double* M = (double*)a.workspace;
  double* ab = M + (size_t)a.n * a.C;
  const long long n_chunks = (a.n + kChunk - 1) / kChunk;
  const unsigned g1 = (unsigned)((n_chunks * a.C + 127) / 128);
  const unsigned gab = (unsigned)ceil_div(a.C, 128);
  if (a.in_f64) {
    const double* x = (const double*)a.x;
    spline_mtilde_kernel<double><<<g1, 128, 0, s>>>(x, a.n, a.C, M);
    spline_ab_kernel<double><<<gab, 128, 0, s>>>(x, a.n, a.C, M, ab);
  } else {
    const float* x = (const float*)a.x;
    spline_mtilde_kernel<float><<<g1, 128, 0, s>>>(x, a.n, a.C, M);
    spline_ab_kernel<float><<<gab, 128, 0, s>>>(x, a.n, a.C, M, ab);
  }
  spline_fix_kernel<<<grid_for((size_t)(a.n - 2) * a.C, 256), 256, 0, s>>>(a.n, a.C, M, ab);
  const unsigned ge = grid_for((size_t)a.m * a.C, 256);
  if (a.in_f64) spline_eval_kernel<double><<<ge, 256, 0, s>>>((const double*)a.x, a.n, a.m, a.C, M, a.y);
  else spline_eval_kernel<float><<<ge, 256, 0, s>>>((const float*)a.x, a.n, a.m, a.C, M, a.y);
  for (int i = 0; i < 4; ++i) count_launch();
  ZCHECK_LAUNCH();
  return ZEGGS_OK;
}

extern "C" size_t zeggs_masked_moments_workspace_bytes(long long n_sel, int total_width) {
  if (n_sel < 1 || total_width < 1) return 0;
  const size_t chunks = (size_t)((n_sel + kRowsPerChunk - 1) / kRowsPerChunk);
  return sizeof(double) * (2 * chunks * total_width + total_width + ZEGGS_MOMENTS_MAX_GROUPS);
}

extern "C" int zeggs_masked_moments(const zeggs_moments_args* ap, void* stream) {
  ZCHECK_ARG(ap, "moments: null args");
  const zeggs_moments_args& a = *ap;
  ZCHECK_ARG(a.n_groups >= 1 && a.n_groups <= ZEGGS_MOMENTS_MAX_GROUPS, "moments: n_groups = %d (1..%d)", a.n_groups, ZEGGS_MOMENTS_MAX_GROUPS);
  ZCHECK_ARG(a.n_sel >= 1, "moments: no selected rows");
  ZCHECK_ARG(a.rows && a.mean && a.std && a.group_std && a.workspace, "moments: null pointer");
  int W = 0;
  for (int g = 0; g < a.n_groups; ++g) {
    ZCHECK_ARG(a.src[g] && a.width[g] >= 1, "moments: group %d has no data", g);
    W += a.width[g];
  }
  const size_t need = zeggs_masked_moments_workspace_bytes(a.n_sel, W);
  ZCHECK_ARG(a.workspace_bytes >= need, "moments: workspace %zu < %zu bytes", a.workspace_bytes, need);
  const long long n_chunks = (a.n_sel + kRowsPerChunk - 1) / kRowsPerChunk;
  double* part0 = (double*)a.workspace;
  double* part1 = part0 + (size_t)n_chunks * W;
  double* csum = part1 + (size_t)n_chunks * W;
  double* gmean = csum + W;
  cudaStream_t s = (cudaStream_t)stream;
  const unsigned gc = (unsigned)ceil_div(W, 256);
  moments_partial_kernel<0><<<(unsigned)n_chunks, 256, 0, s>>>(a, W, part0, part1, gmean);
  moments_channel_kernel<0><<<gc, 256, 0, s>>>(a, W, n_chunks, part0, part1, csum);
  moments_group_kernel<0><<<1, 32, 0, s>>>(a, csum, gmean);
  moments_partial_kernel<1><<<(unsigned)n_chunks, 256, 0, s>>>(a, W, part0, part1, gmean);
  moments_channel_kernel<1><<<gc, 256, 0, s>>>(a, W, n_chunks, part0, part1, csum);
  moments_group_kernel<1><<<1, 32, 0, s>>>(a, csum, gmean);
  for (int i = 0; i < 6; ++i) count_launch();
  ZCHECK_LAUNCH();
  return ZEGGS_OK;
}
