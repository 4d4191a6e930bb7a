// Pose tensors -> BVH channel values on the device (SURVEY.md 8f row 3): replaces the numpy post-step of
// ZEGGS/generate.py:389-406: anim/txform.py:23-34 (xform_orthogonalize_from_xy), anim/quat.py:166-206 (from_xform),
// ZEGGS/utils.py:47-87 (write_bvh: re-base the root on its first frame, apply start_position / start_rotation, fold the
// root transform into joint 0), anim/quat.py:111-119 (to_euler 'zyx') and np.degrees.  One thread per (clip, frame, joint);
// pure streaming: 36 B in, 24 B out per joint (+16 B when the local quaternions are requested).
#include "library.cuh"

namespace zeggs {

__device__ __forceinline__ Q4 quat_from_matrix(const float m[3][3]) {
  // quat.py:166-206, the four-branch form, eps 1e-10
  const float eps = 1e-10f;
  const float t = m[0][0] + m[1][1] + m[2][2];
  Q4 q;
  if (t > 0.f) {
    const float s = 0.5f / sqrtf(fmaxf(t + 1.f, eps));
    q.w = 0.25f / s; q.x = s * (m[2][1] - m[1][2]); q.y = s * (m[0][2] - m[2][0]); q.z = s * (m[1][0] - m[0][1]);
  } else if (m[0][0] > m[1][1] && m[0][0] > m[2][2]) {
    const float s = 2.0f * sqrtf(fmaxf(1.0f + m[0][0] - m[1][1] - m[2][2], eps));
    q.w = (m[2][1] - m[1][2]) / s; q.x = s * 0.25f; q.y = (m[0][1] + m[1][0]) / s; q.z = (m[0][2] + m[2][0]) / s;
  } else if (m[1][1] > m[2][2]) {
    const float s = 2.0f * sqrtf(fmaxf(1.0f + m[1][1] - m[0][0] - m[2][2], eps));
    q.w = (m[0][2] - m[2][0]) / s; q.x = (m[0][1] + m[1][0]) / s; q.y = s * 0.25f; q.z = (m[1][2] + m[2][1]) / s;
  } else {
    const float s = 2.0f * sqrtf(fmaxf(1.0f + m[2][2] - m[0][0] - m[1][1], eps));
    q.w = (m[1][0] - m[0][1]) / s; q.x = (m[0][2] + m[2][0]) / s; q.y = (m[1][2] + m[2][1]) / s; q.z = s * 0.25f;
  }
  return q;
}

// float64 versions of the root composition (quat.py:36-38 computes the cross products in float64)
struct D3 { double x, y, z; };
__device__ __forceinline__ D3 dcross(D3 a, D3 b) { D3 r; r.x = a.y * b.z - a.z * b.y; r.y = a.z * b.x - a.x * b.z; r.z = a.x * b.y - a.y * b.x; return r; }
__device__ __forceinline__ D3 dquat_mul_vec(Q4 q, D3 v) {
  D3 u; u.x = q.x; u.y = q.y; u.z = q.z;
  D3 t = dcross(u, v); t.x *= 2.0; t.y *= 2.0; t.z *= 2.0;
  D3 c = dcross(u, t), r;
  r.x = v.x + (double)q.w * t.x + c.x; r.y = v.y + (double)q.w * t.y + c.y; r.z = v.z + (double)q.w * t.z + c.z;
  return r;
}

__global__ void __launch_bounds__(256) pose_to_bvh_kernel(zeggs_pose_post_args a) {
  const size_t total = (size_t)a.N * a.T * a.J;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int j = (int)(i % a.J);
    const size_t f = i / a.J;                       // frame index n*T + t
    const int n = (int)(f / a.T);
    const float* xy = a.ltxy + i * 6;
    // txform.py:23-34: x, z = x x y, y = z x x, each / (norm + 1e-10); the axes are the COLUMNS of the matrix
    const V3 X = v3(xy[0], xy[1], xy[2]), Yr = v3(xy[3], xy[4], xy[5]);
    const V3 Z = cross(X, Yr), Y = cross(Z, X);
    const float ix = 1.0f / (sqrtf(dot(X, X)) + 1e-10f), iy = 1.0f / (sqrtf(dot(Y, Y)) + 1e-10f), iz = 1.0f / (sqrtf(dot(Z, Z)) + 1e-10f);
    float m[3][3] = {{X.x * ix, Y.x * iy, Z.x * iz}, {X.y * ix, Y.y * iy, Z.y * iz}, {X.z * ix, Y.z * iy, Z.z * iz}};
    Q4 q = quat_from_matrix(m);
    float px = a.lpos[i * 3], py = a.lpos[i * 3 + 1], pz = a.lpos[i * 3 + 2];
    if (j == 0) {
      // utils.py:60-76
      const float* rp = a.root_pos + f * 3;
      const float* rr4 = a.root_rot + f * 4;
      Q4 rr; rr.w = rr4[0]; rr.x = rr4[1]; rr.y = rr4[2]; rr.z = rr4[3];
      D3 rpos; rpos.x = rp[0]; rpos.y = rp[1]; rpos.z = rp[2];
      if (a.rebase) {
        const float* p0 = a.root_pos + (size_t)n * a.T * 3;
        const float* q0 = a.root_rot + (size_t)n * a.T * 4;
        Q4 oi; oi.w = q0[0]; oi.x = -q0[1]; oi.y = -q0[2]; oi.z = -q0[3];
        D3 d; d.x = (double)(rp[0] - p0[0]); d.y = (double)(rp[1] - p0[1]); d.z = (double)(rp[2] - p0[2]);
        rpos = dquat_mul_vec(oi, d);
        rr = quat_mul(oi, rr);
        Q4 sr; sr.w = a.start_rot[0]; sr.x = a.start_rot[1]; sr.y = a.start_rot[2]; sr.z = a.start_rot[3];
        rpos = dquat_mul_vec(sr, rpos);
        rpos.x += a.start_pos[0]; rpos.y += a.start_pos[1]; rpos.z += a.start_pos[2];
        rr = quat_mul(sr, rr);
      }
      D3 lp; lp.x = px; lp.y = py; lp.z = pz;
      const D3 w = dquat_mul_vec(rr, lp);
      px = (float)(w.x + rpos.x); py = (float)(w.y + rpos.y); pz = (float)(w.z + rpos.z);
      q = quat_mul(rr, q);
    }
    a.positions[i * 3] = px; a.positions[i * 3 + 1] = py; a.positions[i * 3 + 2] = pz;
    if (a.lrot) { a.lrot[i * 4] = q.w; a.lrot[i * 4 + 1] = q.x; a.lrot[i * 4 + 2] = q.y; a.lrot[i * 4 + 3] = q.z; }
    // quat.py:111-119 'zyx' then degrees
    const float r2d = 57.29577951308232f;
    const float ez = atan2f(2.0f * (q.w * q.z + q.x * q.y), 1.0f - 2.0f * (q.y * q.y + q.z * q.z));
    const float ey = asinf(fminf(fmaxf(2.0f * (q.w * q.y - q.z * q.x), -1.0f), 1.0f));
    const float ex = atan2f(2.0f * (q.w * q.x + q.y * q.z), 1.0f - 2.0f * (q.x * q.x + q.y * q.y));
    a.euler_deg[i * 3] = ez * r2d; a.euler_deg[i * 3 + 1] = ey * r2d; a.euler_deg[i * 3 + 2] = ex * r2d;
  }
}

extern "C" int zeggs_pose_to_bvh_channels(const zeggs_pose_post_args* ap, void* stream) {
  ZCHECK_ARG(ap, "pose post: null args");
  const zeggs_pose_post_args& a = *ap;
  ZCHECK_ARG(a.N >= 0 && a.T >= 1 && a.J >= 1, "pose post: bad shape");
  ZCHECK_ARG(a.root_pos && a.root_rot && a.lpos && a.ltxy && a.positions && a.euler_deg, "pose post: null pointer");
  if (a.N == 0) return ZEGGS_OK;
  const size_t total = (size_t)a.N * a.T * a.J;
  const size_t blocks = (total + 255) / 256;
  pose_to_bvh_kernel<<<(unsigned)(blocks > 132 * 16 ? 132 * 16 : blocks), 256, 0, (cudaStream_t)stream>>>(a);
  count_launch();
  ZCHECK_LAUNCH();
  return ZEGGS_OK;
}

}  // namespace zeggs
