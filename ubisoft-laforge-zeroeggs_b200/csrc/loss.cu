// Training loss, forward + backward in one call (ZEGGS/train.py:277-421): local->world transforms, two
// 75-joint FK passes (output and ground truth, anim/txform.py:10-34), 17 weighted L1 means (4 of them on frame-to-frame
// differences) + the annealed KL term, /18 -- and the gradient of that scalar w.r.t. the decoder outputs.
// One warp per frame, one tree level at a time; the kernels are described above loss_tree_kernel.
#include "library.cuh"

namespace zeggs {

// ------------------------------------------------------------------ per-frame 3x3 / quaternion math and its adjoints
struct M3 { float m[9]; };   // row-major

__host__ __device__ inline V3 mv(const M3& a, V3 v) {
  return v3(a.m[0] * v.x + a.m[1] * v.y + a.m[2] * v.z, a.m[3] * v.x + a.m[4] * v.y + a.m[5] * v.z, a.m[6] * v.x + a.m[7] * v.y + a.m[8] * v.z);
}
__host__ __device__ inline V3 mtv(const M3& a, V3 v) {   // a^T v
  return v3(a.m[0] * v.x + a.m[3] * v.y + a.m[6] * v.z, a.m[1] * v.x + a.m[4] * v.y + a.m[7] * v.z, a.m[2] * v.x + a.m[5] * v.y + a.m[8] * v.z);
}
__host__ __device__ inline M3 mm(const M3& a, const M3& b) {
  M3 r;
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) r.m[i * 3 + j] = a.m[i * 3] * b.m[j] + a.m[i * 3 + 1] * b.m[3 + j] + a.m[i * 3 + 2] * b.m[6 + j];
  return r;
}
__host__ __device__ inline M3 mtm(const M3& a, const M3& b) {  // a^T b
  M3 r;
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) r.m[i * 3 + j] = a.m[i] * b.m[j] + a.m[3 + i] * b.m[3 + j] + a.m[6 + i] * b.m[6 + j];
  return r;
}
__host__ __device__ inline M3 mmt(const M3& a, const M3& b) {  // a b^T
  M3 r;
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) r.m[i * 3 + j] = a.m[i * 3] * b.m[j * 3] + a.m[i * 3 + 1] * b.m[j * 3 + 1] + a.m[i * 3 + 2] * b.m[j * 3 + 2];
  return r;
}
__host__ __device__ inline void add_outer(M3& d, V3 a, V3 b) {   // d += a b^T
  d.m[0] += a.x * b.x; d.m[1] += a.x * b.y; d.m[2] += a.x * b.z;
  d.m[3] += a.y * b.x; d.m[4] += a.y * b.y; d.m[5] += a.y * b.z;
  d.m[6] += a.z * b.x; d.m[7] += a.z * b.y; d.m[8] += a.z * b.z;
}
__host__ __device__ inline M3 quat_to_xform(Q4 q) {  // tquat.py:53-67
  float x2 = q.x + q.x, y2 = q.y + q.y, z2 = q.z + q.z;
  float xx = q.x * x2, yy = q.y * y2, wx = q.w * x2;
  float xy = q.x * y2, yz = q.y * z2, wy = q.w * y2;
  float xz = q.x * z2, zz = q.z * z2, wz = q.w * z2;
  M3 r;
  r.m[0] = 1.0f - (yy + zz); r.m[1] = xy - wz; r.m[2] = xz + wy;
  r.m[3] = xy + wz; r.m[4] = 1.0f - (xx + zz); r.m[5] = yz - wx;
  r.m[6] = xz - wy; r.m[7] = yz + wx; r.m[8] = 1.0f - (xx + yy);
  return r;
}
__host__ __device__ inline Q4 quat_to_xform_bwd(Q4 q, const M3& d) {
  Q4 g;
  g.w = 2.0f * (-q.z * d.m[1] + q.y * d.m[2] + q.z * d.m[3] - q.x * d.m[5] - q.y * d.m[6] + q.x * d.m[7]);
  g.x = 2.0f * (q.y * d.m[1] + q.z * d.m[2] + q.y * d.m[3] - 2.0f * q.x * d.m[4] - q.w * d.m[5] + q.z * d.m[6] + q.w * d.m[7] - 2.0f * q.x * d.m[8]);
  g.y = 2.0f * (-2.0f * q.y * d.m[0] + q.x * d.m[1] + q.w * d.m[2] + q.x * d.m[3] + q.z * d.m[5] - q.w * d.m[6] + q.z * d.m[7] - 2.0f * q.y * d.m[8]);
  g.z = 2.0f * (-2.0f * q.z * d.m[0] - q.w * d.m[1] + q.x * d.m[2] + q.w * d.m[3] - 2.0f * q.z * d.m[4] + q.y * d.m[5] + q.x * d.m[6] + q.y * d.m[7]);
  return g;
}
// u = v / (|v| + eps) and its adjoint
__host__ __device__ inline V3 unit_eps(V3 v, float eps) { float n = sqrtf(dot(v, v)); return (1.0f / (n + eps)) * v; }
__host__ __device__ inline V3 unit_eps_bwd(V3 v, float eps, V3 du) {
  float n = sqrtf(dot(v, v));
  V3 r = (1.0f / (n + eps)) * du;
  if (n > 0.0f) r = r - (dot(du, v) / ((n + eps) * (n + eps) * n)) * v;
  return r;
}
// txform.py:23-34: columns of the result are the normalised x, y = z cross x, z = x cross xy[1] axes
__host__ __device__ inline M3 orthogonalize_xy(V3 x, V3 yv) {
  V3 z = cross(x, yv), y = cross(z, x);
  V3 X = unit_eps(x, 1e-10f), Y = unit_eps(y, 1e-10f), Z = unit_eps(z, 1e-10f);
  M3 r;
  r.m[0] = X.x; r.m[1] = Y.x; r.m[2] = Z.x;
  r.m[3] = X.y; r.m[4] = Y.y; r.m[5] = Z.y;
  r.m[6] = X.z; r.m[7] = Y.z; r.m[8] = Z.z;
  return r;
}
__host__ __device__ inline void orthogonalize_xy_bwd(V3 x, V3 yv, const M3& d, V3& dx, V3& dyv) {
  V3 z = cross(x, yv), y = cross(z, x);
  V3 dX = v3(d.m[0], d.m[3], d.m[6]), dY = v3(d.m[1], d.m[4], d.m[7]), dZ = v3(d.m[2], d.m[5], d.m[8]);
  dx = unit_eps_bwd(x, 1e-10f, dX);
  V3 dy = unit_eps_bwd(y, 1e-10f, dY);
  V3 dz = unit_eps_bwd(z, 1e-10f, dZ);
  // y = z x x
  dz = dz + cross(x, dy);
  dx = dx + cross(dy, z);
  // z = x x yv
  dx = dx + cross(yv, dz);
  dyv = cross(dz, x);
}

// dRootRot[b][t] = own[b][t] + prev[b][t+1]
__global__ void root_rot_combine_kernel(const float* __restrict__ own, const float* __restrict__ prev, int B, int T, float* __restrict__ out) {
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= (size_t)B * T * 4) return;
  size_t f = i / 4; int t = (int)(f % T);
  out[i] = own[i] + (t + 1 < T ? prev[i + 4] : 0.f);
}

// ================================================================================================================
// One warp owns one frame; the joints of one tree level are processed in parallel (the shipped skeleton: 13 levels, at most 12
// joints wide) and every world-space quantity lives in shared memory.  The only global intermediates are the differences D of the
// four channel groups whose frame-to-frame terms need the neighbouring frames (1575 floats per frame), 17 per-frame partial sums,
// the signs of D and the output-side FK results the adjoint re-reads.  Results are bitwise reproducible (fixed shuffle and frame
// orders).
//   K0 loss_tree_kernel    level order and child lists of the skeleton, from `parents`
//   K1 loss_w_fwd_kernel   FK of the output (lanes 0..15) and of the target (lanes 16..31), D, direct |D| sums, D rows of the diff groups
//                          + the signs of D (2 x 33 bits per joint) and the output-side FK rotations / angular velocities for K2
//   K2 loss_w_bwd_kernel   two frames per warp, no forward recompute: builds dLoss/dQ from K1's signs (direct terms) and the
//                          neighbours' D rows (frame-difference terms), runs the adjoint FK level by level (children publish their
//                          contribution, parents gather them in index order), writes the dY row + the root gradients
//                          (forward-only calls run loss_w_diff_kernel instead: the frame-difference sums alone)
//   K3 loss_w_final_kernel deterministic reduction over frames + KL
// The frame-difference residual is evaluated as (D[t+1] - D[t]) / dt with D = Q_out - Q_target (train.py:356-393 computes
// dQ_out/dt - dQ_target/dt: equal up to fp32 rounding).
// ================================================================================================================
struct TreeTables {           // built on the device from `parents` by loss_tree_kernel (one thread; 75 joints)
  int order[NJ];              // joints sorted by level
  int lvl_off[NJ + 1];        // level l = order[lvl_off[l] .. lvl_off[l+1])
  int nlev;
  int child_off[NJ + 1];      // children of joint i = child_idx[child_off[i] .. child_off[i+1]) in index order
  int child_idx[NJ];
  int parents[NJ];
};
__global__ void loss_tree_kernel(const int* __restrict__ parents, TreeTables* __restrict__ tt) {
  // one thread per joint (blockDim >= NJ): level by walking up the parent chain, position inside the level and the child list by one
  // O(NJ) scan each -- the former single-thread construction (O(NJ^2) dependent steps) cost 50 us on the loss's critical path
  __shared__ TreeTables st;
  __shared__ int lvl[NJ], nchild[NJ];
  if (blockIdx.x != 0) return;
  const int i = threadIdx.x;
  if (i < NJ) st.parents[i] = i == 0 ? -1 : parents[i];
  if (i <= NJ) st.lvl_off[i] = 0;
  __syncthreads();
  if (i < NJ) {
    int l = 0;
    for (int p = st.parents[i]; p >= 0 && l < NJ; p = st.parents[p]) ++l;
    lvl[i] = l;
    int nc = 0;
    for (int c = 1; c < NJ; ++c) nc += st.parents[c] == i;
    nchild[i] = nc;
  }
  __syncthreads();
  if (i == 0) {                               // two short prefix sums
    int maxl = 0;
    for (int j = 0; j < NJ; ++j) maxl = lvl[j] > maxl ? lvl[j] : maxl;
    st.nlev = maxl + 1;
    int n = 0;
    for (int l = 0; l <= maxl; ++l) { st.lvl_off[l] = n; for (int j = 0; j < NJ; ++j) n += lvl[j] == l; }
    st.lvl_off[maxl + 1] = n;
    int m = 0;
    for (int j = 0; j < NJ; ++j) { st.child_off[j] = m; m += nchild[j]; }
    st.child_off[NJ] = m;
  }
  if (i < NJ) st.child_idx[i] = 0;
  __syncthreads();
  if (i < NJ) {
    int pos = st.lvl_off[lvl[i]];
    for (int j = 0; j < i; ++j) pos += lvl[j] == lvl[i];
    st.order[pos] = i;
    int m = st.child_off[i];
    for (int c = 1; c < NJ; ++c) if (st.parents[c] == i) st.child_idx[m++] = c;
  }
  __syncthreads();
  const int* src = reinterpret_cast<const int*>(&st);
  int* dst = reinterpret_cast<int*>(tt);
  for (int k = threadIdx.x; k < (int)(sizeof(TreeTables) / sizeof(int)); k += blockDim.x) dst[k] = src[k];
}

constexpr int LW_WARPS = 4;                      // frames per CTA
// per-joint record: the channel groups of one joint in the order the terms consume them
constexpr int R_LPOS = 0, R_LTXY = 3, R_LVEL = 9, R_LVRT = 12, R_GP = 15, R_GR = 18, R_GV = 27, R_GT = 30, LW_REC = 33;
constexpr int LW_Q = NJ * LW_REC;                // 2475 floats per side
constexpr int LW_RT = 24;                        // root block: pos3 R9 velw3 vrtw3 gaze3
constexpr int LW_DD = NJ * 21;                   // 1575: D rows of LPOS (225) | LTXY (450) | CPOS (225) | CMAT (675)
constexpr int LW_FWD_FLOATS = 2 * LW_Q + 2 * LW_RT;
constexpr int LW_NP = 17;                        // partial sums per frame: terms 0..11, gaze, then the 4 frame-difference terms
constexpr int LW_SW = NJ * 4 + 2;                // sign words per frame: joint i -> pos_lo, pos_hi, neg_lo, neg_hi (33 bits each); root pos, neg

struct LossWArgs {
  int B, T; float dt;
  const float *Y[2], *rp[2], *rq[2];            // [0] output, [1] target; Y rows [frame][1131]
  const float* gaze;
  const TreeTables* tt;
  float* Dd;                                     // [frames][LW_DD]
  float* partial;                                // [frames][LW_NP]
  float* F;                                      // [frames][NJ * 12]: output-side FK results the adjoint needs (gr9, gt3 per joint)
  unsigned* S;                                   // [frames][LW_SW]: sign masks of D (per joint 2 x (pos, neg) words; root block last)
  float *dY, *dRootPos, *dq_own, *dq_prev;
};

__device__ __forceinline__ M3 ldm9(const float* p) { M3 r;
#pragma unroll
  for (int i = 0; i < 9; ++i) r.m[i] = p[i];
  return r; }
__device__ __forceinline__ void stm9(float* p, const M3& v) {
#pragma unroll
  for (int i = 0; i < 9; ++i) p[i] = v.m[i]; }
__device__ __forceinline__ V3 ldv(const float* p) { return v3(p[0], p[1], p[2]); }
__device__ __forceinline__ void stv(float* p, V3 v) { p[0] = v.x; p[1] = v.y; p[2] = v.z; }
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float sgnf(float d) { return (float)((d > 0.f) - (d < 0.f)); }
// record element -> direct-term group (4 LPOS, 5 LTXY, 6 LVEL, 7 LVRT, 8 CPOS, 9 CMAT, 10 CVEL, 11 CVRT)
__device__ __forceinline__ int rec_group(int e) { return e < 3 ? 4 : e < 9 ? 5 : e < 12 ? 6 : e < 15 ? 7 : e < 18 ? 8 : e < 27 ? 9 : e < 30 ? 10 : 11; }

// static weights / channel counts of the 13 direct groups in partial order (terms 0..11, then gaze = term 16) and of the four
// frame-difference terms (12..15: LPOS, LTXY, CPOS, CMAT); train.py:340-395
__constant__ float c_lw_w[13] = {0.1f, 10.f, 0.1f, 5.f, 15.f, 15.f, 10.f, 7.f, 0.1f, 3.f, 0.06f, 1.25f, 10.f};
__constant__ float c_lw_n[13] = {3.f, 9.f, 3.f, 3.f, NJ * 3.f, NJ * 6.f, NJ * 3.f, NJ * 3.f, NJ * 3.f, NJ * 9.f, NJ * 3.f, NJ * 3.f, 3.f};
__constant__ float c_lw_dw[4] = {7.f, 8.f, 0.06f, 1.25f};
__constant__ float c_lw_dn[4] = {NJ * 3.f, NJ * 6.f, NJ * 3.f, NJ * 9.f};

// forward of both sides into shared memory (lanes 0..15: output side, 16..31: target side): q[side][joint][33], rt[side][21]
__device__ __forceinline__ void lw_forward(const LossWArgs& a, const TreeTables& tt, size_t frame, int lane, float* const (&q)[2], float* const (&rt)[2]) {
  const int side = lane >> 4, l16 = lane & 15;
  const int t = (int)(frame % a.T);
  const float* y = a.Y[side] + frame * P_OUT;
  float* qs = q[side];
  // local values of every joint: global -> records up front (independent loads: one memory latency instead of one per tree level)
  for (int i = l16; i < NJ; i += 16) {
    float* ci = qs + i * LW_REC;
    stv(ci + R_LPOS, ldv(y + OFF_LPOS + 3 * i)); stv(ci + R_LTXY, ldv(y + OFF_LTXY + 6 * i)); stv(ci + R_LTXY + 3, ldv(y + OFF_LTXY + 6 * i + 3));
    stv(ci + R_LVEL, ldv(y + OFF_LVEL + 3 * i)); stv(ci + R_LVRT, ldv(y + OFF_LVRT + 3 * i));
  }
  __syncwarp();
  if (l16 == 0) {
    const float* q4 = a.rq[side] + frame * 4;
    Q4 qr; qr.w = q4[0]; qr.x = q4[1]; qr.y = q4[2]; qr.z = q4[3];
    Q4 qp = qr;
    if (t > 0) { qp.w = q4[-4]; qp.x = q4[-3]; qp.y = q4[-2]; qp.z = q4[-1]; }
    const V3 pos = ldv(a.rp[side] + frame * 3), gz = ldv(a.gaze + frame * 3);
    const M3 R = quat_to_xform(qr);
    const V3 velw = quat_mul_vec(qp, ldv(y)), vrtw = quat_mul_vec(qp, ldv(y + 3));          // train.py:281-286
    float* r = rt[side];
    stv(r, pos); stm9(r + 3, R); stv(r + 12, velw); stv(r + 15, vrtw);
    stv(r + 18, quat_mul_vec(quat_inv(qr), unit_eps(gz - pos, 1e-8f)));                     // train.py:336-337
    const V3 lp = ldv(qs + R_LPOS), lv = ldv(qs + R_LVEL), lr = ldv(qs + R_LVRT);
    const V3 x = ldv(qs + R_LTXY), yv = ldv(qs + R_LTXY + 3);
    const V3 rp0 = quat_mul_vec(qr, lp);
    const V3 p0 = rp0 + pos, t0 = vrtw + quat_mul_vec(qr, lr), v0 = velw + quat_mul_vec(qr, lv) + cross(vrtw, rp0);
    // joint 0 is compared in world space (train.py:296-305); its raw two-axis rotation stays local
    stv(qs + R_LPOS, p0); stv(qs + R_LVEL, v0); stv(qs + R_LVRT, t0);
    stv(qs + R_GP, p0); stm9(qs + R_GR, mm(R, orthogonalize_xy(x, yv))); stv(qs + R_GV, v0); stv(qs + R_GT, t0);
  }
  __syncwarp();
  for (int l = 1; l < tt.nlev; ++l) {                       // txform.py:10-20, one tree level at a time
    for (int k = tt.lvl_off[l] + l16; k < tt.lvl_off[l + 1]; k += 16) {
      const int i = tt.order[k], p = tt.parents[i];
      const float* cp = qs + p * LW_REC;
      float* ci = qs + i * LW_REC;
      const M3 grp = ldm9(cp + R_GR);
      const V3 gpp = ldv(cp + R_GP), gtp = ldv(cp + R_GT), gvp = ldv(cp + R_GV);
      const V3 lp = ldv(ci + R_LPOS), lv = ldv(ci + R_LVEL), lr = ldv(ci + R_LVRT);
      const V3 x = ldv(ci + R_LTXY), yv = ldv(ci + R_LTXY + 3);
      const V3 rp = mv(grp, lp);
      stv(ci + R_GP, gpp + rp); stm9(ci + R_GR, mm(grp, orthogonalize_xy(x, yv))); stv(ci + R_GV, gvp + mv(grp, lv) + cross(gtp, rp));
      stv(ci + R_GT, gtp + mv(grp, lr));
    }
    __syncwarp();
  }
}

// position of record element (joint i, element e) inside a frame's D row, or -1 when the group has no frame-difference term
__device__ __forceinline__ int dd_index(int i, int e) {
  if (e < 3) return 3 * i + e;                                   // LPOS
  if (e < 9) return NJ * 3 + 6 * i + (e - 3);                    // LTXY
  if (e >= R_GP && e < R_GR) return NJ * 9 + 3 * i + (e - R_GP); // CPOS
  if (e >= R_GR && e < R_GV) return NJ * 12 + 9 * i + (e - R_GR);// CMAT
  return -1;
}

__global__ void __launch_bounds__(LW_WARPS * 32) loss_w_fwd_kernel(LossWArgs a) {
  extern __shared__ float lw_sm[];
  __shared__ TreeTables tt;
  for (int i = threadIdx.x; i < (int)(sizeof(TreeTables) / 4); i += blockDim.x) reinterpret_cast<int*>(&tt)[i] = reinterpret_cast<const int*>(a.tt)[i];
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const size_t frame = (size_t)blockIdx.x * LW_WARPS + warp;
  if (frame >= (size_t)a.B * a.T) return;
  float* base = lw_sm + (size_t)warp * LW_FWD_FLOATS;
  float* const q[2] = {base, base + LW_Q};
  float* const rt[2] = {base + 2 * LW_Q, base + 2 * LW_Q + LW_RT};
  lw_forward(a, tt, frame, lane, q, rt);
  float sum[13];
#pragma unroll
  for (int g = 0; g < 13; ++g) sum[g] = 0.f;
  float* dd = a.Dd + frame * LW_DD;
  unsigned* sg = a.S + frame * LW_SW;
  float* fk = a.F + frame * (NJ * 12);
  for (int i = lane; i < NJ; i += 32) {
    const float* o = q[0] + i * LW_REC; const float* w = q[1] + i * LW_REC;
    unsigned long long pos = 0ull, neg = 0ull;
#pragma unroll
    for (int e = 0; e < LW_REC; ++e) {
      const float D = o[e] - w[e];
      sum[rec_group(e)] += fabsf(D);
      if (D > 0.f) pos |= 1ull << e;
      if (D < 0.f) neg |= 1ull << e;
      const int x = dd_index(i, e);
      if (x >= 0) dd[x] = D;
    }
    sg[4 * i] = (unsigned)pos; sg[4 * i + 1] = (unsigned)(pos >> 32); sg[4 * i + 2] = (unsigned)neg; sg[4 * i + 3] = (unsigned)(neg >> 32);
#pragma unroll
    for (int m = 0; m < 9; ++m) fk[12 * i + m] = o[R_GR + m];
#pragma unroll
    for (int m = 0; m < 3; ++m) fk[12 * i + 9 + m] = o[R_GT + m];
  }
  if (lane == 0) {
    const float* o = rt[0]; const float* w = rt[1];
    unsigned pos = 0u, neg = 0u;
#pragma unroll
    for (int k = 0; k < 21; ++k) {
      const float D = o[k] - w[k];
      sum[k < 3 ? 0 : k < 12 ? 1 : k < 15 ? 2 : k < 18 ? 3 : 12] += fabsf(D);
      if (D > 0.f) pos |= 1u << k;
      if (D < 0.f) neg |= 1u << k;
    }
    sg[NJ * 4] = pos; sg[NJ * 4 + 1] = neg;
  }
#pragma unroll
  for (int g = 0; g < 13; ++g) { const float v = warp_sum(sum[g]); if (lane == 0) a.partial[frame * LW_NP + g] = v; }
}

// K2: two frames per warp (lanes 0..15 / 16..31), no forward recompute: the output-side FK results and the signs of D come from K1.
// Per frame in shared memory: O-records [joint][27] = locals (lpos3 ltxy6 lvel3 lvrt3) + gr9 + gt3 -- a processed joint's record is
// re-used for its hand-over [gr9 gp3 gt3 gv3] -- and G-records [joint][33] = dLoss/d(record), plus the 21 root gradients.
constexpr int LB_WARPS = 3;                      // 6 frames per CTA, 2 CTAs per SM
constexpr int O_LPOS = 0, O_LTXY = 3, O_LVEL = 9, O_LVRT = 12, O_GR = 15, O_GT = 24, LB_OREC = 27;
constexpr int LB_FRAME_FLOATS = NJ * LB_OREC + NJ * LW_REC + LW_RT;     // 4524

__device__ __forceinline__ float half_sum(float v) {          // sum over the 16 lanes of a half warp
#pragma unroll
  for (int o = 8; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__global__ void __launch_bounds__(LB_WARPS * 32) loss_w_bwd_kernel(LossWArgs a) {
  extern __shared__ float lw_sm[];
  __shared__ TreeTables tt;
  for (int i = threadIdx.x; i < (int)(sizeof(TreeTables) / 4); i += blockDim.x) reinterpret_cast<int*>(&tt)[i] = reinterpret_cast<const int*>(a.tt)[i];
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, half = lane >> 4, l16 = lane & 15;
  const size_t nframes = (size_t)a.B * a.T;
  const size_t frame_raw = ((size_t)blockIdx.x * LB_WARPS + warp) * 2 + half;
  const bool live = frame_raw < nframes;
  const size_t frame = live ? frame_raw : nframes - 1;          // a dead half mirrors the last frame (no stores), keeping the warp converged
  const int t = (int)(frame % a.T);
  float* base = lw_sm + ((size_t)warp * 2 + half) * LB_FRAME_FLOATS;
  float* Q = base;                                   // O-records
  float* G = base + NJ * LB_OREC;                    // G-records
  float* gr_ = G + NJ * LW_REC;                      // root gradients (21)
  const float* y = a.Y[0] + frame * P_OUT;
  const float* fk = a.F + frame * (NJ * 12);
  const unsigned* sg = a.S + frame * LW_SW;
  float* gy = a.dY + frame * P_OUT;
  const float BT = (float)a.B * (float)a.T;
  // ---- records: locals from the pose row, FK results and signs from K1; dLoss/dQ of the direct terms
  for (int i = l16; i < NJ; i += 16) {
    float* qi = Q + i * LB_OREC;
    stv(qi + O_LPOS, ldv(y + OFF_LPOS + 3 * i)); stv(qi + O_LTXY, ldv(y + OFF_LTXY + 6 * i)); stv(qi + O_LTXY + 3, ldv(y + OFF_LTXY + 6 * i + 3));
    stv(qi + O_LVEL, ldv(y + OFF_LVEL + 3 * i)); stv(qi + O_LVRT, ldv(y + OFF_LVRT + 3 * i));
#pragma unroll
    for (int m = 0; m < 12; ++m) qi[O_GR + m] = fk[12 * i + m];
    const unsigned long long pos = (unsigned long long)sg[4 * i] | ((unsigned long long)sg[4 * i + 1] << 32);
    const unsigned long long neg = (unsigned long long)sg[4 * i + 2] | ((unsigned long long)sg[4 * i + 3] << 32);
    float* gi = G + i * LW_REC;
#pragma unroll
    for (int e = 0; e < LW_REC; ++e) {
      const int g = rec_group(e);
      const float sc = c_lw_w[g] / (BT * c_lw_n[g]) * (1.0f / 18.0f);
      gi[e] = ((pos >> e) & 1ull) ? sc : ((neg >> e) & 1ull) ? -sc : 0.f;
    }
  }
  if (l16 == 0) {
    const unsigned pos = sg[NJ * 4], neg = sg[NJ * 4 + 1];
#pragma unroll
    for (int k = 0; k < 21; ++k) {
      const int g = k < 3 ? 0 : k < 12 ? 1 : k < 15 ? 2 : k < 18 ? 3 : 12;
      const float sc = c_lw_w[g] / (BT * c_lw_n[g]) * (1.0f / 18.0f);
      gr_[k] = ((pos >> k) & 1u) ? sc : ((neg >> k) & 1u) ? -sc : 0.f;
    }
  }
  __syncwarp();
  // ---- frame-difference terms (train.py:356-393): e_t = (D[t+1] - D[t]) / dt from the neighbouring frames' D rows, per joint
  float dsum[4] = {0.f, 0.f, 0.f, 0.f};
  if (a.T > 1) {
    const float inv_dt = 1.0f / a.dt;
    const float* d0 = a.Dd + frame * LW_DD;
    const bool has_p = t + 1 < a.T, has_m = t > 0;
    const float nd = (float)a.B * (float)(a.T - 1);
    for (int i = l16; i < NJ; i += 16) {
      float* gi = G + i * LW_REC;
      auto run = [&](int x0, int n, int e0, int g) {        // n consecutive D-row entries starting at x0 <-> record elements e0..
        const float sc = c_lw_dw[g] * inv_dt / (nd * c_lw_dn[g]) * (1.0f / 18.0f);
        for (int k = 0; k < n; ++k) {
          const float D = d0[x0 + k];
          float gd = 0.f;
          if (has_p) { const float er = (d0[x0 + k + LW_DD] - D) * inv_dt; dsum[g] += fabsf(er); gd -= sgnf(er); }
          if (has_m) { const float el = (D - d0[x0 + k - LW_DD]) * inv_dt; gd += sgnf(el); }
          gi[e0 + k] += sc * gd;
        }
      };
      run(3 * i, 3, R_LPOS, 0); run(NJ * 3 + 6 * i, 6, R_LTXY, 1); run(NJ * 9 + 3 * i, 3, R_GP, 2); run(NJ * 12 + 9 * i, 9, R_GR, 3);
    }
  }
#pragma unroll
  for (int g = 0; g < 4; ++g) { const float v = half_sum(dsum[g]); if (l16 == 0 && live) a.partial[frame * LW_NP + 13 + g] = v; }
  __syncwarp();
  // ---- adjoint FK, deepest level first: a joint gathers its children's hand-overs, then publishes its own in its (dead) O-record
  for (int l = tt.nlev - 1; l >= 1; --l) {
    for (int k = tt.lvl_off[l] + l16; k < tt.lvl_off[l + 1]; k += 16) {
      const int i = tt.order[k], p = tt.parents[i];
      float* gi = G + i * LW_REC;
      for (int cc = tt.child_off[i]; cc < tt.child_off[i + 1]; ++cc) {
        const float* ps = Q + tt.child_idx[cc] * LB_OREC;
#pragma unroll
        for (int m = 0; m < 9; ++m) gi[R_GR + m] += ps[m];
#pragma unroll
        for (int m = 0; m < 3; ++m) { gi[R_GP + m] += ps[9 + m]; gi[R_GT + m] += ps[12 + m]; gi[R_GV + m] += ps[15 + m]; }
      }
      float* qi = Q + i * LB_OREC; const float* qp = Q + p * LB_OREC;
      const V3 lp = ldv(qi + O_LPOS), lv = ldv(qi + O_LVEL), lr = ldv(qi + O_LVRT), x = ldv(qi + O_LTXY), yv = ldv(qi + O_LTXY + 3);
      const M3 lm = orthogonalize_xy(x, yv);
      const M3 grp = ldm9(qp + O_GR);
      const V3 gtp = ldv(qp + O_GT);
      const V3 rp = mv(grp, lp);
      const V3 dgp = ldv(gi + R_GP), dgt = ldv(gi + R_GT), dgv = ldv(gi + R_GV);
      const M3 dgr = ldm9(gi + R_GR);
      const V3 drp = dgp + cross(dgv, gtp);                 // gp[i] = gp[p] + rp ;  gv[i] += gt[p] x rp
      M3 acc = mmt(dgr, lm);                                // gr[i] = gr[p] lmat
      add_outer(acc, dgv, lv);                              // gv[i] += gr[p] lvel
      add_outer(acc, dgt, lr);                              // gt[i]  = gt[p] + gr[p] lvrt
      add_outer(acc, drp, lp);                              // rp = gr[p] lpos
      stm9(qi, acc); stv(qi + 9, dgp); stv(qi + 12, dgt + cross(rp, dgv)); stv(qi + 15, dgv);
      if (live) {       // local quantities of joint i: direct L1 terms + FK
        stv(gy + OFF_LPOS + 3 * i, ldv(gi + R_LPOS) + mtv(grp, drp));
        stv(gy + OFF_LVEL + 3 * i, ldv(gi + R_LVEL) + mtv(grp, dgv));
        stv(gy + OFF_LVRT + 3 * i, ldv(gi + R_LVRT) + mtv(grp, dgt));
        V3 dx, dyv;
        orthogonalize_xy_bwd(x, yv, mtm(grp, dgr), dx, dyv);
        stv(gy + OFF_LTXY + 6 * i, ldv(gi + R_LTXY) + dx);
        stv(gy + OFF_LTXY + 6 * i + 3, ldv(gi + R_LTXY + 3) + dyv);
      }
    }
    __syncwarp();
  }
  // ---- joint 0 + root terms (one lane per frame; the serial tail of the chain)
  if (l16 == 0 && live) {
    float* g0 = G;
    for (int cc = tt.child_off[0]; cc < tt.child_off[1]; ++cc) {
      const float* ps = Q + tt.child_idx[cc] * LB_OREC;
#pragma unroll
      for (int m = 0; m < 9; ++m) g0[R_GR + m] += ps[m];
#pragma unroll
      for (int m = 0; m < 3; ++m) { g0[R_GP + m] += ps[9 + m]; g0[R_GT + m] += ps[12 + m]; g0[R_GV + m] += ps[15 + m]; }
    }
    const float* q4 = a.rq[0] + frame * 4;
    Q4 qr; qr.w = q4[0]; qr.x = q4[1]; qr.y = q4[2]; qr.z = q4[3];
    Q4 qp = qr;
    if (t > 0) { qp.w = q4[-4]; qp.x = q4[-3]; qp.y = q4[-2]; qp.z = q4[-1]; }
    const V3 pos = ldv(a.rp[0] + frame * 3), gz = ldv(a.gaze + frame * 3);
    const M3 R = quat_to_xform(qr);
    const V3 lp = ldv(Q + O_LPOS), lv = ldv(Q + O_LVEL), lr = ldv(Q + O_LVRT), x = ldv(Q + O_LTXY), yv = ldv(Q + O_LTXY + 3);   // joint 0's raw locals
    const V3 vel = ldv(y), vrt = ldv(y + 3);
    const V3 vrtw = quat_mul_vec(qp, vrt);
    const V3 rp0 = quat_mul_vec(qr, lp);
    // joint 0 receives the local (world-space) and the FK-root gradients
    const V3 dp0 = ldv(g0 + R_LPOS) + ldv(g0 + R_GP);
    const V3 dv0 = ldv(g0 + R_LVEL) + ldv(g0 + R_GV);
    const V3 dt0 = ldv(g0 + R_LVRT) + ldv(g0 + R_GT);
    const M3 dm0 = ldm9(g0 + R_GR);
    M3 dR = ldm9(gr_ + 3);
    V3 dpos = ldv(gr_) + dp0;                                  // p0 = rp0 + pos
    const V3 dvelw = ldv(gr_ + 12) + dv0;                      // v0 = velw + rot(q, lv) + vrtw x rp0
    const V3 dvrtw = ldv(gr_ + 15) + dt0 + cross(rp0, dv0);    // t0 = vrtw + rot(q, lr)
    const V3 drp0 = dp0 + cross(dv0, vrtw);
    Q4 dq; dq.w = dq.x = dq.y = dq.z = 0.f;
    Q4 gq; V3 gv_;
    quat_mul_vec_bwd(qr, lp, drp0, gq, gv_); dq.w += gq.w; dq.x += gq.x; dq.y += gq.y; dq.z += gq.z;
    stv(gy + OFF_LPOS, gv_);
    quat_mul_vec_bwd(qr, lv, dv0, gq, gv_);  dq.w += gq.w; dq.x += gq.x; dq.y += gq.y; dq.z += gq.z;
    stv(gy + OFF_LVEL, gv_);
    quat_mul_vec_bwd(qr, lr, dt0, gq, gv_);  dq.w += gq.w; dq.x += gq.x; dq.y += gq.y; dq.z += gq.z;
    stv(gy + OFF_LVRT, gv_);
    const M3 lm0 = orthogonalize_xy(x, yv);                    // m0 = R lmat0
    const M3 tm = mmt(dm0, lm0);
#pragma unroll
    for (int k = 0; k < 9; ++k) dR.m[k] += tm.m[k];
    V3 dx, dyv;
    orthogonalize_xy_bwd(x, yv, mtm(R, dm0), dx, dyv);
    stv(gy + OFF_LTXY, ldv(g0 + R_LTXY) + dx);
    stv(gy + OFF_LTXY + 3, ldv(g0 + R_LTXY + 3) + dyv);
    gq = quat_to_xform_bwd(qr, dR);          dq.w += gq.w; dq.x += gq.x; dq.y += gq.y; dq.z += gq.z;
    const V3 u = gz - pos;                                     // gaze = rot(q^-1, unit(gaze - pos))
    const V3 un = unit_eps(u, 1e-8f);
    quat_mul_vec_bwd(quat_inv(qr), un, ldv(gr_ + 18), gq, gv_);
    dq.w += gq.w; dq.x -= gq.x; dq.y -= gq.y; dq.z -= gq.z;
    dpos = dpos - unit_eps_bwd(u, 1e-8f, gv_);
    Q4 dqp; dqp.w = dqp.x = dqp.y = dqp.z = 0.f;              // the world root velocities use the PREVIOUS frame's rotation
    quat_mul_vec_bwd(qp, vel, dvelw, gq, gv_); dqp.w += gq.w; dqp.x += gq.x; dqp.y += gq.y; dqp.z += gq.z;
    stv(gy, gv_);
    quat_mul_vec_bwd(qp, vrt, dvrtw, gq, gv_); dqp.w += gq.w; dqp.x += gq.x; dqp.y += gq.y; dqp.z += gq.z;
    stv(gy + 3, gv_);
    if (t == 0) { dq.w += dqp.w; dq.x += dqp.x; dq.y += dqp.y; dq.z += dqp.z; dqp.w = dqp.x = dqp.y = dqp.z = 0.f; }
    stv(a.dRootPos + frame * 3, dpos);
    float* o1 = a.dq_own + frame * 4; o1[0] = dq.w; o1[1] = dq.x; o1[2] = dq.y; o1[3] = dq.z;
    float* o2 = a.dq_prev + frame * 4; o2[0] = dqp.w; o2[1] = dqp.x; o2[2] = dqp.y; o2[3] = dqp.z;
  }
}

// forward-only calls (no gradient requested): the four frame-difference sums from the D rows, one warp per frame
__global__ void __launch_bounds__(256) loss_w_diff_kernel(LossWArgs a) {
  const int lane = threadIdx.x & 31;
  const size_t frame = (size_t)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (frame >= (size_t)a.B * a.T) return;
  const int t = (int)(frame % a.T);
  float dsum[4] = {0.f, 0.f, 0.f, 0.f};
  if (t + 1 < a.T) {
    const float inv_dt = 1.0f / a.dt;
    const float* d0 = a.Dd + frame * LW_DD;
    for (int x = lane; x < LW_DD; x += 32) {
      const int g = x < NJ * 3 ? 0 : x < NJ * 9 ? 1 : x < NJ * 12 ? 2 : 3;
      dsum[g] += fabsf((d0[x + LW_DD] - d0[x]) * inv_dt);
    }
  }
#pragma unroll
  for (int g = 0; g < 4; ++g) { const float v = warp_sum(dsum[g]); if (lane == 0) a.partial[frame * LW_NP + 13 + g] = v; }
}

// deterministic reduction over frames (warp g owns term g: lanes stride the frames, fixed shuffle tree, double) + KL
__global__ void __launch_bounds__(LW_NP * 32) loss_w_final_kernel(const float* __restrict__ partial, int B, int T, const float* __restrict__ mu,
                                                                  const float* __restrict__ logvar, int Z, float kl_weight_host,
                                                                  const float* __restrict__ kl_weight_dev, float* __restrict__ losses,
                                                                  float* __restrict__ dmu, float* __restrict__ dlogvar) {
  const float kl_weight = kl_weight_dev ? *kl_weight_dev : kl_weight_host;
  __shared__ double tsum[LW_NP + 1];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int frames = B * T;
  double s = 0.0;
  for (int f = lane; f < frames; f += 32) s += partial[(size_t)f * LW_NP + warp];
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) {
    const double BT = (double)B * T;
    if (warp < 13) tsum[warp] = s * ((double)c_lw_w[warp] / (BT * c_lw_n[warp]));
    else tsum[warp] = T > 1 ? s * ((double)c_lw_dw[warp - 13] / ((double)B * (T - 1) * c_lw_dn[warp - 13])) : 0.0;
  }
  double kl = 0.0;
  if (mu && logvar) {
    for (int i = threadIdx.x; i < B * Z; i += blockDim.x) {
      float m_ = mu[i], lv = logvar[i];
      kl += -0.5 * (1.0 + lv - (double)m_ * m_ - exp((double)lv));
      const float gscale = kl_weight / ((float)B * (float)Z) / 18.0f;
      if (dmu) dmu[i] = gscale * m_;
      if (dlogvar) dlogvar[i] = gscale * 0.5f * (expf(lv) - 1.0f);
    }
  }
  __shared__ double klw[LW_NP];
  for (int o = 16; o > 0; o >>= 1) kl += __shfl_xor_sync(0xffffffffu, kl, o);
  if (lane == 0) klw[warp] = kl;
  __syncthreads();
  if (threadIdx.x == 0) {
    double klt = 0.0;
    for (int w = 0; w < LW_NP; ++w) klt += klw[w];
    // losses[1..17]: train.py:397-416 order = terms 0..11, the four difference terms (12..15), gaze (16); [18] = weighted KL
    double total = 0.0;
    for (int k = 0; k < 12; ++k) { losses[1 + k] = (float)tsum[k]; total += tsum[k]; }
    for (int k = 0; k < 4; ++k) { losses[13 + k] = (float)tsum[13 + k]; total += tsum[13 + k]; }
    losses[17] = (float)tsum[12]; total += tsum[12];
    const double klterm = (mu && logvar) ? kl_weight * klt / ((double)B * Z) : 0.0;
    losses[18] = (float)klterm; total += klterm;
    losses[0] = (float)(total / 18.0);
  }
}

struct LossWs { float *Dd, *fpartial, *F, *dq_own, *dq_prev; unsigned* S; TreeTables* tt; size_t bytes; };
static LossWs loss_ws(void* base, int B, int T) {
  LossWs w; Arena a{(char*)base};
  const size_t BT = (size_t)B * T;
  w.dq_own = a.take(BT * 4); w.dq_prev = a.take(BT * 4);
  w.Dd = a.take(BT * LW_DD); w.fpartial = a.take(BT * LW_NP); w.tt = (TreeTables*)a.take(sizeof(TreeTables) / 4 + 1);
  w.F = a.take(BT * NJ * 12); w.S = (unsigned*)a.take(BT * LW_SW);
  w.bytes = a.off; return w;
}
extern "C" size_t zeggs_loss_workspace_bytes(int B, int T) { return (B < 1 || T < 1) ? 0 : loss_ws(nullptr, B, T).bytes; }

extern "C" int zeggs_loss_fwd_bwd(const zeggs_loss_args* ap, void* stream_) {
  ZCHECK_ARG(ap, "loss: null args");
  const zeggs_loss_args& a = *ap; cudaStream_t s = (cudaStream_t)stream_;
  ZCHECK_ARG(a.B >= 1 && a.T >= 1 && a.Y && a.root_pos && a.root_rot && a.WY && a.W_root_pos && a.W_root_rot && a.gaze_pos && a.parents && a.losses,
             "loss: bad arguments");
  LossWs w = loss_ws(a.workspace, a.B, a.T);
  ZCHECK_ARG(a.workspace && a.workspace_bytes >= w.bytes, "loss: workspace too small");
  const int BT = a.B * a.T;
  ZCHECK_ARG((long long)a.B * a.T < (1ll << 31), "loss: too many frames");
  ScopedTimer tm("loss", s);
  LossWArgs wa;
  wa.B = a.B; wa.T = a.T; wa.dt = a.dt;
  wa.Y[0] = a.Y; wa.Y[1] = a.WY; wa.rp[0] = a.root_pos; wa.rp[1] = a.W_root_pos; wa.rq[0] = a.root_rot; wa.rq[1] = a.W_root_rot;
  wa.gaze = a.gaze_pos; wa.tt = w.tt; wa.Dd = w.Dd; wa.partial = w.fpartial; wa.F = w.F; wa.S = w.S;
  wa.dY = a.dY; wa.dRootPos = a.dRootPos; wa.dq_own = w.dq_own; wa.dq_prev = w.dq_prev;
  RC(set_max_dynamic_smem(loss_w_fwd_kernel, LW_WARPS * LW_FWD_FLOATS * sizeof(float)));
  RC(set_max_dynamic_smem(loss_w_bwd_kernel, LB_WARPS * 2 * LB_FRAME_FLOATS * sizeof(float)));
  loss_tree_kernel<<<1, 96, 0, s>>>(a.parents, w.tt); count_launch();
  const int nb = ceil_div(BT, LW_WARPS);
  loss_w_fwd_kernel<<<nb, LW_WARPS * 32, LW_WARPS * LW_FWD_FLOATS * sizeof(float), s>>>(wa); count_launch();
  if (a.dY) {
    ZCHECK_ARG(a.dRootPos && a.dRootRot, "loss: gradient outputs missing");
    loss_w_bwd_kernel<<<ceil_div(BT, LB_WARPS * 2), LB_WARPS * 32, LB_WARPS * 2 * LB_FRAME_FLOATS * sizeof(float), s>>>(wa); count_launch();
    root_rot_combine_kernel<<<ceil_div(BT * 4, 256), 256, 0, s>>>(w.dq_own, w.dq_prev, a.B, a.T, a.dRootRot); count_launch();
  } else if (a.T > 1) {
    wa.dY = nullptr;
    loss_w_diff_kernel<<<ceil_div(BT, 8), 256, 0, s>>>(wa); count_launch();
  }
  loss_w_final_kernel<<<1, LW_NP * 32, 0, s>>>(w.fpartial, a.B, a.T, a.mu, a.logvar, a.Z, a.kl_weight, a.kl_weight_dev, a.losses, a.dmu, a.dlogvar);
  count_launch();
  ZCHECK_LAUNCH();
  return ZEGGS_OK;
}

}  // namespace zeggs
