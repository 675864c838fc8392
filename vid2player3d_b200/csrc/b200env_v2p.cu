// b200env_v2p.cu - kernels + C ABI for the vid2player rows of the hot path (SURVEY.md 8a, a10-a17):
// SMPL-FK targets, ball aerodynamics / reset, state-from-sim, and the high-level env's
// bounce/estimator bookkeeping + reward + observation + reset FSM fused into one launch.
// Reference (paths relative to /root/reference/vid2player):
//   _smpl_to_sim / _forward_kinematics        env/tasks/humanoid_smpl_im_mvae.py:897-946, utils/hybrik.py:597-652
//   rotation_matrix_to_quaternion/_angle_axis utils/konia_transform.py:348-438, 558-655
//   apply_external_force_to_ball              env/tasks/humanoid_smpl_im_mvae.py:711-739 (+ utils/tennis_ball.py:15-37)
//   _reset_balls + offline pool               env/tasks/humanoid_smpl_im_mvae.py:503-524, utils/tennis_ball.py:422-456
//   _update_state_from_sim                    env/tasks/humanoid_smpl_im_mvae.py:799-860
//   controller post_physics_step              env/tasks/physics_mvae_controller.py:271-314,333-360,368-436,481-602
//   TennisBallOutEstimator.estimate           utils/tennis_ball_out_estimator.py:126-205
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/b200env_v2p.h"
#include "counter_rng.cuh"

#define FULL 0xffffffffu
#define V2P_WARPS 4

static thread_local char g_verr[256] = "";
static int vfail(int code, const char* msg) {
  snprintf(g_verr, sizeof(g_verr), "%s", msg);
  return code;
}
#define V_CUDA_OK()                                                        \
  do {                                                                     \
    cudaError_t _e = cudaGetLastError();                                   \
    if (_e != cudaSuccess) return vfail(-10, cudaGetErrorString(_e));      \
  } while (0)

// ------------------------------------------------------------------------------------------ konia conversions
// templated on the scalar type: the float instantiation is what the float launches always ran (the float overloads of sqrt, fmax,
// atan2, ... are sqrtf, fmaxf, atan2f), the double one serves the double instantiation of the backhand fix
template <typename T>
__device__ __forceinline__ T safe_div(T num, T den) {  // safe_zero_division, eps 1e-6
  if (fabs(den) < T(1e-6)) den += T(1e-6);
  return num / den;
}
// rotation matrix (row-major) -> quaternion wxyz  (konia_transform.py:348-438)
template <typename T>
__device__ __forceinline__ void rotmat_to_quat_wxyz(const T* m, T* q) {
  const T m00 = m[0], m01 = m[1], m02 = m[2], m10 = m[3], m11 = m[4], m12 = m[5], m20 = m[6], m21 = m[7], m22 = m[8];
  const T trace = m00 + m11 + m22;
  if (trace > T(0)) {
    T sq = sqrt(fmax(trace + T(1), T(1e-6))) * T(2);
    q[0] = T(0.25) * sq; q[1] = safe_div(m21 - m12, sq); q[2] = safe_div(m02 - m20, sq); q[3] = safe_div(m10 - m01, sq);
  } else if ((m00 > m11) && (m00 > m22)) {
    T sq = sqrt(fmax(T(1) + m00 - m11 - m22, T(1e-6))) * T(2);
    q[0] = safe_div(m21 - m12, sq); q[1] = T(0.25) * sq; q[2] = safe_div(m01 + m10, sq); q[3] = safe_div(m02 + m20, sq);
  } else if (m11 > m22) {
    T sq = sqrt(fmax(T(1) + m11 - m00 - m22, T(1e-6))) * T(2);
    q[0] = safe_div(m02 - m20, sq); q[1] = safe_div(m01 + m10, sq); q[2] = T(0.25) * sq; q[3] = safe_div(m12 + m21, sq);
  } else {
    T sq = sqrt(fmax(T(1) + m22 - m00 - m11, T(1e-6))) * T(2);
    q[0] = safe_div(m10 - m01, sq); q[1] = safe_div(m02 + m20, sq); q[2] = safe_div(m12 + m21, sq); q[3] = T(0.25) * sq;
  }
}
template <typename T>
__device__ __forceinline__ T safe_atan2(T y, T x) {  // torch_safe_atan2 (:41-49)
  if (fabs(y) < T(1e-6) && fabs(x) < T(1e-6)) y += T(1e-6);
  return atan2(y, x);
}
// quaternion wxyz -> rotation vector (konia_transform.py:558-628)
template <typename T>
__device__ __forceinline__ void quat_wxyz_to_angle_axis(const T* q, T* aa) {
  const T c = q[0], q1 = q[1], q2 = q[2], q3 = q[3];
  const T s2 = q1 * q1 + q2 * q2 + q3 * q3;
  const T s = sqrt(fmax(s2, T(1e-6)));
  const T two_theta = T(2) * (c < T(0) ? safe_atan2(-s, -c) : safe_atan2(s, c));
  const T k = s2 > T(0) ? safe_div(two_theta, s) : T(2);
  aa[0] = q1 * k; aa[1] = q2 * k; aa[2] = q3 * k;
}
// quaternion (given in the converter's WXYZ slot order) -> rotation matrix (konia_transform.py:474-555)
__device__ __forceinline__ void quat_wxyz_to_rotmat(const float* qi, float* m) {
  const float n0 = sqrtf(qi[0] * qi[0] + qi[1] * qi[1] + qi[2] * qi[2] + qi[3] * qi[3]);
  const float n = n0 < 1e-12f ? 1e-12f : n0;   // clamp_min that keeps a NaN (fmaxf would drop it): a NaN quaternion gives a NaN matrix
  const float w = qi[0] / n, x = qi[1] / n, y = qi[2] / n, z = qi[3] / n;
  const float tx = 2.0f * x, ty = 2.0f * y, tz = 2.0f * z;
  const float twx = tx * w, twy = ty * w, twz = tz * w, txx = tx * x, txy = ty * x, txz = tz * x, tyy = ty * y, tyz = tz * y, tzz = tz * z;
  m[0] = 1.0f - (tyy + tzz); m[1] = txy - twz; m[2] = txz + twy;
  m[3] = txy + twz; m[4] = 1.0f - (txx + tzz); m[5] = tyz - twx;
  m[6] = txz - twy; m[7] = tyz + twx; m[8] = 1.0f - (txx + tyy);
}
__device__ __forceinline__ void qmul_xyzw(const float* a, const float* b, float* o) {
  const float x1 = a[0], y1 = a[1], z1 = a[2], w1 = a[3], x2 = b[0], y2 = b[1], z2 = b[2], w2 = b[3];
  o[0] = w1 * x2 + x1 * w2 + y1 * z2 - z1 * y2;
  o[1] = w1 * y2 - x1 * z2 + y1 * w2 + z1 * x2;
  o[2] = w1 * z2 + x1 * y2 - y1 * x2 + z1 * w2;
  o[3] = w1 * w2 - x1 * x2 - y1 * y2 - z1 * z2;
}

// ------------------------------------------------------------------------------------------ a13: SMPL FK targets
// one link of the SMPL chain (hybrik.py:597-652): G = G_parent R ; P = G_parent rel + P_parent
template <typename T>
__device__ __forceinline__ void chain_link(const T* pG, const T* pP, const T* R, const T* rel, T* G, T* P) {
#pragma unroll
  for (int r = 0; r < 3; r++) {
#pragma unroll
    for (int c = 0; c < 3; c++) G[r * 3 + c] = pG[r * 3] * R[c] + pG[r * 3 + 1] * R[3 + c] + pG[r * 3 + 2] * R[6 + c];
    P[r] = pG[r * 3] * rel[0] + pG[r * 3 + 1] * rel[1] + pG[r * 3 + 2] * rel[2] + pP[r];
  }
}
__global__ void __launch_bounds__(V2P_WARPS * 32)
smpl_to_sim_kernel(int n, const float* __restrict__ root_pos, const float* __restrict__ rotmat, const float* __restrict__ rest_all,
                   int num_rest, const int32_t* __restrict__ parents, const int32_t* __restrict__ smpl_2_mujoco, float dt,
                   const float* prev_root_pos, const float* __restrict__ prev_rb_rot, float* root_rot, float* dof_pos,
                   float* root_vel, float* root_ang_vel, float* dof_vel, float* rb_pos, float* rb_rot, float* prev_root_pos_update,
                   float* target_root_pos_out, const uint8_t* __restrict__ only_mask) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t e = (int64_t)blockIdx.x * V2P_WARPS + warp;
  if (e >= n) return;
  if (only_mask && !only_mask[e]) return;      // mask-driven reset: FK of the envs being reset only
  const float* rest = rest_all + (e % num_rest) * 72;   // per-shape rest joints: env e has shape e % num_rest (dual: players alternate)
  const bool act = lane < 24;
  const int j = act ? lane : 0;
  const int par = parents[j] < 0 ? 0 : parents[j];
  int mj = 0;  // mujoco index of SMPL joint j (inverse of smpl_2_mujoco)
  for (int k = 0; k < 24; k++)
    if (smpl_2_mujoco[k] == j) mj = k;
  float Rl[9], G[9], P[3], rel[3];
#pragma unroll
  for (int k = 0; k < 9; k++) Rl[k] = rotmat[(e * 24 + j) * 9 + k];
#pragma unroll
  for (int k = 0; k < 3; k++) rel[k] = rest[j * 3 + k] - (j > 0 ? rest[par * 3 + k] : 0.0f);
  // local angle-axis -> dof targets (root excluded), mujoco order
  if (act && mj > 0) {
    float q[4], aa[3];
    rotmat_to_quat_wxyz(Rl, q);
    quat_wxyz_to_angle_axis(q, aa);
#pragma unroll
    for (int k = 0; k < 3; k++) dof_pos[e * 69 + (mj - 1) * 3 + k] = aa[k];
  }
  // FK chain (hybrik.py:597-652): G_j = G_parent R_j ; P_j = G_parent rel_j + P_parent
  bool done = (lane == 0);
#pragma unroll
  for (int k = 0; k < 9; k++) G[k] = Rl[k];
#pragma unroll
  for (int k = 0; k < 3; k++) P[k] = rel[k];
  for (int it = 0; it < 9; it++) {
    float pG[9], pP[3];
#pragma unroll
    for (int k = 0; k < 9; k++) pG[k] = __shfl_sync(FULL, G[k], par);
#pragma unroll
    for (int k = 0; k < 3; k++) pP[k] = __shfl_sync(FULL, P[k], par);
    const bool pdone = __shfl_sync(FULL, (int)done, par) != 0;
    if (act && !done && pdone) {
      chain_link(pG, pP, Rl, rel, G, P);
      done = true;
    }
  }
  float qw[4], q[4];
  rotmat_to_quat_wxyz(G, qw);
  q[0] = qw[1]; q[1] = qw[2]; q[2] = qw[3]; q[3] = qw[0];
  if (act) {
#pragma unroll
    for (int k = 0; k < 3; k++) rb_pos[(e * 24 + mj) * 3 + k] = P[k] - (rest[k] - root_pos[e * 3 + k]);
#pragma unroll
    for (int k = 0; k < 4; k++) rb_rot[(e * 24 + mj) * 4 + k] = q[k];
    if (mj == 0) {
#pragma unroll
      for (int k = 0; k < 4; k++) root_rot[e * 4 + k] = q[k];
    }
    if (prev_root_pos && prev_rb_rot) {
      // diff = quat_normalize(quat_mul(conj(prev), cur)) ; axis*angle/dt   (:909-919)
      const float* pq = prev_rb_rot + (e * 24 + mj) * 4;
      float cj[4] = {-pq[0], -pq[1], -pq[2], pq[3]}, d[4];
      qmul_xyzw(cj, q, d);
      const float sg = d[3] < 0.0f ? -1.0f : 1.0f;  // quat_pos
#pragma unroll
      for (int k = 0; k < 4; k++) d[k] *= sg;
      const float nn = fmaxf(sqrtf(d[0] * d[0] + d[1] * d[1] + d[2] * d[2] + d[3] * d[3]), 1e-9f);
#pragma unroll
      for (int k = 0; k < 4; k++) d[k] /= nn;
      // quat_to_angle_axis (utils/torch_utils.py:82-102)
      float st = sqrtf(__fsub_rn(1.0f, __fmul_rn(d[3], d[3])));
      float ang = 2.0f * acosf(d[3]);
      ang = atan2f(sinf(ang), cosf(ang));
      float ax[3];
      if (fabsf(st) > 1e-5f) { ax[0] = d[0] / st; ax[1] = d[1] / st; ax[2] = d[2] / st; }
      else { ang = 0.0f; ax[0] = 0.0f; ax[1] = 0.0f; ax[2] = 1.0f; }
      float dv[3] = {ax[0] * ang / dt, ax[1] * ang / dt, ax[2] * ang / dt};
      if (mj == 0) {
#pragma unroll
        for (int k = 0; k < 3; k++) {
          root_ang_vel[e * 3 + k] = dv[k] / dt;  // reference quirk: divided by dt twice (:917-919)
          root_vel[e * 3 + k] = (root_pos[e * 3 + k] - prev_root_pos[e * 3 + k]) / dt;
        }
      } else {
#pragma unroll
        for (int k = 0; k < 3; k++) dof_vel[e * 69 + (mj - 1) * 3 + k] = dv[k];
      }
    } else {
      if (mj == 0) {
#pragma unroll
        for (int k = 0; k < 3; k++) { root_ang_vel[e * 3 + k] = 0.0f; root_vel[e * 3 + k] = 0.0f; }
      } else {
#pragma unroll
        for (int k = 0; k < 3; k++) dof_vel[e * 69 + (mj - 1) * 3 + k] = 0.0f;
      }
    }
    // _save_prev_target_motion_state (:741-750) / `self._target_root_pos = root_pos` folded in: the lane that just read the previous
    // root position stores the current one (prev_root_pos_update may alias prev_root_pos)
    if (mj == 0) {
#pragma unroll
      for (int k = 0; k < 3; k++) {
        const float r = root_pos[e * 3 + k];
        if (prev_root_pos_update) prev_root_pos_update[e * 3 + k] = r;
        if (target_root_pos_out) target_root_pos_out[e * 3 + k] = r;
      }
    }
  }
}

// ------------------------------------------------------------------------------------------ a13b: head look-at correction
// angle_axis_to_rotation_matrix (konia_transform.py:250-334)
template <typename T>
__device__ __forceinline__ void aa_to_rotmat(const T* aa, T* m) {
  const T theta2 = aa[0] * aa[0] + aa[1] * aa[1] + aa[2] * aa[2];
  if (theta2 > T(1e-6)) {
    const T theta = sqrt(fmax(theta2, T(1e-6)));
    const T wx = aa[0] / (theta + T(1e-6)), wy = aa[1] / (theta + T(1e-6)), wz = aa[2] / (theta + T(1e-6));
    const T c = cos(theta), s = sin(theta), k = T(1) - c;
    m[0] = c + wx * wx * k; m[1] = wx * wy * k - wz * s; m[2] = wy * s + wx * wz * k;
    m[3] = wz * s + wx * wy * k; m[4] = c + wy * wy * k; m[5] = -wx * s + wy * wz * k;
    m[6] = -wy * s + wx * wz * k; m[7] = wx * s + wy * wz * k; m[8] = c + wz * wz * k;
  } else {
    m[0] = T(1); m[1] = -aa[2]; m[2] = aa[1]; m[3] = aa[2]; m[4] = T(1); m[5] = -aa[0]; m[6] = -aa[1]; m[7] = aa[0]; m[8] = T(1);
  }
}
__global__ void fix_head_kernel(int n, const float* __restrict__ rb_pos, const float* __restrict__ rb_rot, int head_body,
                                const float* __restrict__ ball_pos, const float* __restrict__ root_pos, float* joint_rotmat) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n) return;
  const float* hq = rb_rot + (e * 24 + head_body) * 4;
  const float qw[4] = {hq[3], hq[0], hq[1], hq[2]};
  float m[9];
  quat_wxyz_to_rotmat(qw, m);
  float lx = m[2], ly = m[5];   // head_rotmat @ (0,0,1), xy part
  float ln = fmaxf(sqrtf(lx * lx + ly * ly), 1e-12f);
  lx /= ln; ly /= ln;
  float bx = ball_pos[e * 3] - rb_pos[(e * 24 + head_body) * 3], by = ball_pos[e * 3 + 1] - rb_pos[(e * 24 + head_body) * 3 + 1];
  float bn = fmaxf(sqrtf(bx * bx + by * by), 1e-12f);
  bx /= bn; by /= bn;
  float d = atan2f(by, bx) - atan2f(ly, lx);
  if (d > 3.14159265358979323846f) d -= 6.283185307179586f;
  if (d < -3.14159265358979323846f) d += 6.283185307179586f;
  const bool miss = (ball_pos[e * 3 + 1] < root_pos[e * 3 + 1] - 0.5f) || (fabsf(ball_pos[e * 3]) > 4.0f);
  if (miss) d = 0.0f;
  const int joints[2] = {15, 12};  // SMPLPose.Head, SMPLPose.Neck
#pragma unroll
  for (int j = 0; j < 2; j++) {
    float* R = joint_rotmat + (e * 24 + joints[j]) * 9;
    float Rl[9], q[4], aa[3], o[9];
#pragma unroll
    for (int k = 0; k < 9; k++) Rl[k] = R[k];
    rotmat_to_quat_wxyz(Rl, q);
    quat_wxyz_to_angle_axis(q, aa);
    aa[1] += d / 2.0f;
    aa_to_rotmat(aa, o);
#pragma unroll
    for (int k = 0; k < 9; k++) R[k] = o[k];
  }
}

// ------------------------------------------------------------------------------------------ a10: ball aerodynamics
#define BALL_R 0.032f
#define BALL_KF 0.0019462794807519486f  // rho*pi*R^2/2, rho = 1.21 (tennis_ball.py:17-22)
#define BALL_CD 0.55f
__device__ __forceinline__ void ball_aero_force(const float* vel, const float* angvel, float spin_scale, float* force) {
  float vs = sqrtf(vel[0] * vel[0] + vel[1] * vel[1] + vel[2] * vel[2]);
  if (vs == 0.0f) vs += 1.0f;
  const float vn[3] = {vel[0] / vs, vel[1] / vs, vel[2] / vs};
  // vel_tan = vn x (0,0,-1)
  const float vt[3] = {-vn[1], vn[0], 0.0f};
  const float vspin = sqrtf(angvel[0] * angvel[0] + angvel[1] * angvel[1] + angvel[2] * angvel[2]) / 6.283185307179586f;
  float cl = 1.0f / (2.0f + fabsf(vs / (vspin * spin_scale + 1e-6f)));
  cl = cl * (vspin > 0.0f ? -1.0f : 1.0f);
  // vel_tan x vn
  const float cx = vt[1] * vn[2] - vt[2] * vn[1], cy = vt[2] * vn[0] - vt[0] * vn[2], cz = vt[0] * vn[1] - vt[1] * vn[0];
  const float kd = -BALL_KF * BALL_CD * vs, kl = -BALL_KF * cl * vs * vs;
  force[0] = kd * vel[0] + kl * cx;
  force[1] = kd * vel[1] + kl * cy;
  force[2] = kd * vel[2] + kl * cz;
}
__global__ void ball_aero_kernel(int n, const float* __restrict__ ball_states, int stride, uint8_t* has_bounce, uint8_t* has_bounce_now,
                                 float* bounce_pos, float* force, int substeps, float spin_scale) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n) return;
  const float* b = ball_states + e * stride;
  float f[3];
  ball_aero_force(b + 7, b + 10, spin_scale, f);
  force[e * 3] = f[0]; force[e * 3 + 1] = f[1]; force[e * 3 + 2] = f[2];
  const float thr = substeps > 2 ? BALL_R * 6.0f : BALL_R * 4.0f;
  const bool now = !has_bounce[e] && (b[2] <= thr);
  if (now) {
    has_bounce_now[e] = 1; has_bounce[e] = 1;
    bounce_pos[e * 3] = b[0]; bounce_pos[e * 3 + 1] = b[1]; bounce_pos[e * 3 + 2] = b[2];
  }
}

// ------------------------------------------------------------------------------------------ a17: ball reset from the pool
__global__ void ball_reset_kernel(int n, const int64_t* __restrict__ env_ids, const int64_t* __restrict__ pool_index,
                                  const float* __restrict__ pool, float* ball_states, int stride, float* ball_pos, float* ball_vel,
                                  uint8_t* has_bounce, float* bounce_pos, uint8_t* has_contact, float* traj) {
  const int i = blockIdx.x;
  if (i >= n) return;
  const int64_t e = env_ids[i];
  const float* row = pool + pool_index[i] * 307;
  for (int k = threadIdx.x; k < 300; k += blockDim.x) traj[e * 300 + k] = row[7 + k];
  if (threadIdx.x == 0) {
    float* b = ball_states + e * stride;
    const float v[3] = {row[3], row[4], row[5]};
    // ang vel = vspin * 2pi * normalize(v x (0,0,-1))   (:508-509)
    float c[3] = {-v[1], v[0], 0.0f};
    const float nn = fmaxf(sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(c[0], c[0]), __fmul_rn(c[1], c[1])), __fmul_rn(c[2], c[2]))), 1e-12f);
    const float s = row[6] * 3.141592653589793f * 2.0f;
#pragma unroll
    for (int k = 0; k < 3; k++) { b[k] = row[k]; b[7 + k] = v[k]; b[10 + k] = s * (c[k] / nn); ball_pos[e * 3 + k] = row[k]; ball_vel[e * 3 + k] = v[k]; bounce_pos[e * 3 + k] = 0.0f; }
    has_bounce[e] = 0; has_contact[e] = 0;
  }
}

// ------------------------------------------------------------------------------------------ a11 / a12: state from sim
__global__ void update_state_kernel(b200v2p_state_t s) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= s.n) return;
  if (s.only_mask && !s.only_mask[e]) return;     // reset path: the reference refreshes the state views when humanoids were reset (:186-187)
  const float* rb = s.rigid_body_state + e * s.bodies_per_env * 13;
  const float* ball = s.ball_states + e * s.ball_stride;
  // velocity-jump contact detector (substeps > 2): uses the ball velocity of the previous control step (:800-808)
  const bool now = !s.has_contact[e] && (ball[8] > 0.0f) && ((ball[8] - s.ball_vel[e * 3 + 1]) > 10.0f);
  s.has_contact_now[e] = now ? 1 : 0;
  if (now) s.has_contact[e] = 1;
  const bool second = s.dual && (e & 1);
  const int wrist_body = second ? s.wrist_body2 : s.wrist_body, racket_body = second ? s.racket_body2 : s.racket_body;
  const float* grip = second ? s.grip_normal2 : s.grip_normal;
  const float* wq = rb + wrist_body * 13 + 3;
  const float qw[4] = {wq[3], wq[0], wq[1], wq[2]};
  float m[9];
  quat_wxyz_to_rotmat(qw, m);
#pragma unroll
  for (int k = 0; k < 3; k++) {
    s.root_pos[e * 3 + k] = rb[k];
    s.root_vel[e * 3 + k] = s.root_states[e * s.root_stride + 7 + k];
    s.racket_pos[e * 3 + k] = rb[racket_body * 13 + k];
    s.racket_vel[e * 3 + k] = rb[racket_body * 13 + 7 + k];
    s.racket_normal[e * 3 + k] = m[k * 3] * grip[0] + m[k * 3 + 1] * grip[1] + m[k * 3 + 2] * grip[2];
    s.ball_pos[e * 3 + k] = ball[k];
    s.ball_vel[e * 3 + k] = ball[7 + k];
  }
  s.ball_vspin[e] = sqrtf(ball[10] * ball[10] + ball[11] * ball[11] + ball[12] * ball[12]) / 6.283185307179586f;
}

// ------------------------------------------------------------------------------------------ a14-a16: controller post step
__device__ __forceinline__ bool in_court(float x, float y) { return x > -4.11f && x < 4.11f && y > 0.0f && y < 11.89f; }
__device__ __forceinline__ float est_index(float v, const float* r) {  // clamp + round (:126-162)
  v = fminf(fmaxf(v, r[0]), r[1] - r[2]);
  return rintf((v - r[0]) / r[2]);
}
// AverageMeterUnSync.update (utils/common.py:52-63) of meter m for env e; envs are independent, so no atomics
__device__ __forceinline__ void meter_update(const b200v2p_ctrl_t& c, int m, int64_t e, float v) {
  const int64_t i = (int64_t)m * c.n + e;
  const float s = __fadd_rn(c.meter_sum[i], v);
  const int64_t k = c.meter_count[i] + 1;
  c.meter_sum[i] = s;
  c.meter_count[i] = k;
  c.meter_avg[i] = __fdiv_rn(s, __ll2float_rn(k));   // float32 / int64 promotes to float32
  if (v > c.meter_max[i]) c.meter_max[i] = v;
}
// MVAEControllerVis._compute_reset + _compute_stats (env/tasks/mvae_controller_vis.py:64-93): flags, reset masking, then stats
__device__ __forceinline__ void eval_reset(const b200v2p_ctrl_t& c, int64_t e, const float* rp, const float* bp, bool has_contact) {
  const int64_t ta = c.tar_action[e];
  const bool terminate = c.progress_buf[e] > (int64_t)c.eval_episode_length;
  const bool in_time = c.tar_time[e] >= c.tar_time_total[e];
  bool reaction = (has_contact && ta == 0 && c.has_bounce[e] && in_time) || (!has_contact && in_time);
  bool recovery = ta == 1 && (has_contact || bp[1] < rp[1] - 1.0f || fabsf(c.ball_vel[e * 3 + 1]) < 2.0f);
  if (terminate) { reaction = true; recovery = false; }
  c.terminate_buf[e] = terminate ? 1 : 0;
  c.reset_buf[e] = terminate ? 1 : 0;
  c.reset_reaction[e] = reaction ? 1 : 0;
  c.reset_recovery[e] = recovery ? 1 : 0;
  if (!recovery) return;
  meter_update(c, 0, e, has_contact ? 1.0f : 0.0f);
  meter_update(c, 1, e, c.swing_type_cycle[e] == 1 ? 1.0f : 0.0f);
  const bool bin = c.est_bounce_in[e] != 0;
  meter_update(c, 2, e, bin ? 1.0f : 0.0f);
  if (bin) {
    float d[3];
#pragma unroll
    for (int k = 0; k < 3; k++) d[k] = __fsub_rn(c.est_bounce_pos[e * 3 + k], c.target_bounce_pos[e * 3 + k]);
    meter_update(c, 3, e, sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(d[0], d[0]), __fmul_rn(d[1], d[1])), __fmul_rn(d[2], d[2]))));
  }
}
// min / max that keep a NaN (torch.clamp semantics), as the cast of libb200nn.so does: an env whose observation blew up gets a NaN
// operand, and so NaN actions, instead of plausible clamped ones
__device__ __forceinline__ float clamp_nan(float x, float lo, float hi) {
  float r;
  asm("max.NaN.f32 %0, %1, %2;" : "=f"(r) : "f"(x), "f"(lo));
  asm("min.NaN.f32 %0, %1, %2;" : "=f"(r) : "f"(r), "f"(hi));
  return r;
}
// the high-level policy's bf16 operand row of env e from the observation row `o` the warp has just stored (see b200v2p_ctrl_t.policy_x)
__device__ __forceinline__ void policy_row(const b200v2p_ctrl_t& c, int64_t e, const float* o, int lane) {
  __syncwarp();   // the row's values were stored by the other lanes
  const int p = c.policy_dual ? (int)(e & 1) : 0;
  const int64_t r = c.policy_dual ? p * (int64_t)(c.n >> 1) + (e >> 1) : e;
  __nv_bfloat16* x = reinterpret_cast<__nv_bfloat16*>(c.policy_x) + r * c.policy_ld;
  const float* mean = c.policy_mean ? c.policy_mean + p * c.num_obs : nullptr;
  const float* rstd = c.policy_rstd ? c.policy_rstd + p * c.num_obs : nullptr;
  const float clip = c.policy_clip[p];
  for (int k = lane; k < c.num_obs; k += 32) {
    float v = clamp_nan(o[k], -c.policy_clip_obs, c.policy_clip_obs);
    if (mean) v = (v - __ldg(mean + k)) * __ldg(rstd + k);
    x[k] = __float2bfloat16_rn(clamp_nan(v, -clip, clip));
  }
}

// EVAL: the reset rule of the test-time task replaces the training FSM; the training / dual instantiation is the kernel as it was
template <bool EVAL>
__global__ void __launch_bounds__(V2P_WARPS * 32) controller_post_kernel(b200v2p_ctrl_t c) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t e = (int64_t)blockIdx.x * V2P_WARPS + warp;
  if (e >= c.n) return;
  const bool touched = c.touch_mask && c.touch_mask[e];
  if (c.obs_only && c.touch_mask && !touched && !c.reset_reaction[e] && !c.reset_recovery[e]) return;   // row still current
  const float* rb = c.rigid_body_state + e * c.bodies_per_env * 13;
  if (c.advance && !c.obs_only) {
    // tail of physics_step (:364-366) + head of post_physics_step (:441-444) folded in: the future-trajectory window moves on by one
    // frame (roll(-1), last frame zeroed), the reaction timer and the episode progress count one step.  In place inside the warp.
    float* tr = c.ball_traj + e * 300;
    float tmp[10];
#pragma unroll
    for (int i = 0; i < 10; i++) {
      const int k = lane + 32 * i;
      tmp[i] = k < 297 ? tr[k + 3] : 0.0f;
    }
    __syncwarp();
#pragma unroll
    for (int i = 0; i < 10; i++) {
      const int k = lane + 32 * i;
      if (k < 300) tr[k] = tmp[i];
    }
    if (lane == 0) { c.tar_time[e] += 1; c.progress_buf[e] += 1; }
    __syncwarp();
  }
  const float rp[3] = {c.root_pos[e * 3], c.root_pos[e * 3 + 1], c.root_pos[e * 3 + 2]};
  const float bp[3] = {c.ball_pos[e * 3], c.ball_pos[e * 3 + 1], c.ball_pos[e * 3 + 2]};
  const float kp[3] = {c.racket_pos[e * 3], c.racket_pos[e * 3 + 1], c.racket_pos[e * 3 + 2]};
  const bool has_contact = c.has_contact[e] != 0;
  // ---- _update_state (:271-314): true bounce in court, estimated bounce of the outgoing ball
  if (lane == 0 && !c.obs_only) {
    if (c.tar_action[e] == 0 && c.has_bounce_now[e]) c.bounce_in[e] = in_court(c.bounce_pos[e * 3], c.bounce_pos[e * 3 + 1]) ? 1 : 0;
    if (c.has_contact_now[e] && c.est_x) {
      const float* b = c.ball_states + e * c.ball_stride;
      const float *VX = c.est_params, *VY = c.est_params + 3, *VS = c.est_params + 6, *TX = c.est_params + 9, *TY = c.est_params + 12;
      // x_net, vel_x and vspin round every product like the reference's tensor ops (no fma contraction): one rounding flips the
      // x_net = +-4 validity test or the table row at a cell edge
      bool valid = (b[8] > VX[0]) && (b[9] > VY[0]) && (b[9] < VY[1]) && (b[2] < TY[1]);
      const float x_net = __fadd_rn(b[0], __fmul_rn(b[7], fabsf(b[1] / b[8])));
      valid = valid && (x_net > -4.0f) && (x_net < 4.0f);
      if (valid) {
        const float vel_x = sqrtf(__fadd_rn(__fmul_rn(b[7], b[7]), __fmul_rn(b[8], b[8])));
        const float vspin = sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(b[10], b[10]), __fmul_rn(b[11], b[11])), __fmul_rn(b[12], b[12]))) / 6.283185307179586f;
        const float d1 = (VY[1] - VY[0]) / VY[2], d2 = (VS[1] - VS[0]) / VS[2];
        const int64_t ti = (int64_t)(est_index(vel_x, VX) * d1 * d2 + est_index(b[9], VY) * d2 + est_index(vspin, VS));
        const float* tx = c.est_x + ti * c.est_nx;
        const float* ty = c.est_y + ti * c.est_ny * 2;
        const int hi = (int)est_index(b[2], TY);
        float bx = b[0] + ty[hi * 2] * b[7] / vel_x, by = b[1] + ty[hi * 2] * b[8] / vel_x, bt = ty[hi * 2 + 1];
        const float net_dist = -b[1] / b[8] * vel_x;
        const int ni = (int)est_index(net_dist, TX);
        if (tx[ni] + b[2] < 1.07f) { bx = 0.0f; by = 0.0f; bt = 0.0f; }  // into the net (NET_HEIGHT)
        float mx = tx[0];
        for (int k = 1; k < c.est_nx; k++) mx = fmaxf(mx, tx[k]);
        c.est_bounce_pos[e * 3] = bx; c.est_bounce_pos[e * 3 + 1] = by;
        c.est_bounce_time[e] = bt;
        c.est_max_height[e] = b[2] + mx;
        c.est_bounce_in[e] = in_court(bx, by) ? 1 : 0;
      }
    }
  }
  __syncwarp();
  // ---- reward (:368-406, jit :493-602)
  if (lane == 0 && !c.obs_only) {
    const float phase = c.phase[e];
    float d2 = 0.0f;
#pragma unroll
    for (int k = 0; k < 3; k++) d2 += (bp[k] - kp[k]) * (bp[k] - kp[k]);
    float rew = 0.0f, s0 = 0.0f, s1 = 0.0f;
    const float tp[3] = {c.target_bounce_pos[e * 3], c.target_bounce_pos[e * 3 + 1], c.target_bounce_pos[e * 3 + 2]};
    if (c.reward_type == 0) {  // reach
      const float cp = c.swing_type[e] == -1 ? 3.0f : 3.14159265358979323846f;
      s0 = (c.tar_action[e] == 1 ? 1.0f : 0.0f) * expf(-c.scale_pos * d2) * expf(-c.scale_phase * (phase - cp) * (phase - cp));
      rew = s0 * c.w_pos;
    } else {
      const int64_t st = c.reward_type == 1 ? c.swing_type[e] : c.swing_type_cycle[e];
      const float cp = st >= 2 ? 3.0f : 3.14159265358979323846f;
      s0 = (has_contact ? 0.0f : 1.0f) * expf(-c.scale_pos * d2) * expf(-c.scale_phase * (phase - cp) * (phase - cp)) + (has_contact ? 1.0f : 0.0f);
      if (c.reward_type == 1) {  // return
        float err = 0.0f;
        const float* src = c.has_bounce[e] ? (c.bounce_pos + e * 3) : bp;
#pragma unroll
        for (int k = 0; k < 3; k++) err += (src[k] - tp[k]) * (src[k] - tp[k]);
        const float r = (400.0f - err) / 400.0f;
        s1 = (has_contact ? 1.0f : 0.0f) * (r < 0.0f ? 0.0f : (r > 1.0f ? 1.0f : r));   // torch.clamp keeps a NaN
      } else {  // return_w_estimate
        float err = 0.0f;
#pragma unroll
        for (int k = 0; k < 3; k++) err += (c.est_bounce_pos[e * 3 + k] - tp[k]) * (c.est_bounce_pos[e * 3 + k] - tp[k]);
        s1 = (c.est_bounce_in[e] ? 1.0f : 0.0f) * expf(-c.scale_bounce_pos * err) * expf(-c.scale_bounce_time * c.est_bounce_time[e]);
      }
      rew = c.w_pos * s0 + c.w_ball_pos * s1;
    }
    c.rew_buf[e] = rew;
    c.sub_rewards[e * 2] = s0; c.sub_rewards[e * 2 + 1] = s1;
  }
  // ---- observation (:316-360): actor 225 | ball trajectory 3*L relative to the racket | target - root xy
  float* o = c.obs_buf + e * c.num_obs;
  bool nan = false;
  if (lane < 3) { o[lane] = rp[lane]; o[3 + lane] = c.root_vel[e * 3 + lane]; o[222 + lane] = c.racket_normal[e * 3 + lane]; nan |= isnan(o[lane]) || isnan(o[3 + lane]) || isnan(o[222 + lane]); }
  if (lane < 24) {
    const float* b1 = rb + (lane + 1) * 13;  // bodies 1..24 (23 humanoid + Racket) relative to the root
#pragma unroll
    for (int k = 0; k < 3; k++) { float v = b1[k] - rp[k]; o[6 + lane * 3 + k] = v; nan |= isnan(v); }
    const float* q = rb + lane * 13 + 3;  // xyzw fed to the WXYZ converter as is (reference quirk, :339)
    float m[9];
    quat_wxyz_to_rotmat(q, m);
    float* r6 = o + 78 + lane * 6;  // rotmat_to_rot6d: cat(mat[...,0], mat[...,1]) = first and second COLUMN
    r6[0] = m[0]; r6[1] = m[3]; r6[2] = m[6]; r6[3] = m[1]; r6[4] = m[4]; r6[5] = m[7];
#pragma unroll
    for (int k = 0; k < 6; k++) nan |= isnan(r6[k]);
  }
  const float* rk = rb + c.racket_body * 13;
  const int L3 = c.obs_traj_len * 3;
  if (c.ball_obs) {   // _compute_task_obs :345-346: _ball_obs <- roll(-1) with the current ball position appended (kept in every mode)
    float* hst = c.ball_obs + e * L3;
    const bool touch = !c.obs_only || c.reset_reaction[e] || (!c.dual && c.reset_recovery[e]);   // obs_only: the reference refreshes
    if (touch) {                                                                                // the reset ids only (:200-201; dual :64-66)
      float tmp[10];   // L3 <= 300 -> at most 10 values per lane: read everything, then write (in-place shift inside the warp)
#pragma unroll
      for (int i = 0; i < 10; i++) {
        const int k = lane + 32 * i;
        tmp[i] = k < L3 - 3 ? hst[k + 3] : (k < L3 ? c.ball_pos[e * 3 + k - (L3 - 3)] : 0.0f);
      }
      __syncwarp();
#pragma unroll
      for (int i = 0; i < 10; i++) {
        const int k = lane + 32 * i;
        if (k < L3) hst[k] = tmp[i];
      }
      __syncwarp();
    }
  }
  const float* src = c.use_history ? c.ball_obs + e * L3 : c.ball_traj + e * 300;
  for (int k = lane; k < L3; k += 32) { float v = src[k] - rk[k % 3]; o[225 + k] = v; nan |= isnan(v); }
  if (c.use_target && lane < 2) { float v = c.target_bounce_pos[e * 3 + lane] - rp[lane]; o[225 + c.obs_traj_len * 3 + lane] = v; nan |= isnan(v); }
  const bool has_nan = __any_sync(FULL, nan);
  if (c.policy_x) policy_row(c, e, o, lane);
  // ---- dual reset FSM (physics_mvae_controller_dual.py:92-120): the opponent's flags are recomputed from its inputs (no exchange)
  if (EVAL) {
    if (lane == 0 && !c.obs_only) eval_reset(c, e, rp, bp, has_contact);
    return;
  }
  if (lane == 0 && !c.obs_only && c.dual) {   // the terms below are restated by dual_terms (rally results): change both together
    const int64_t p = e ^ 1;
    bool rec[2], term[2];
    for (int w = 0; w < 2; w++) {
      const int64_t i = w ? p : e;
      const bool ta1 = c.tar_action[i] == 1, ta0 = c.tar_action[i] == 0, hc = c.has_contact[i] != 0, hb = c.has_bounce[i] != 0;
      // bounce_in AFTER this step's _update_state: recomputed when it is being rewritten (by this or the partner's warp)
      const bool bin = (ta0 && c.has_bounce_now[i]) ? in_court(c.bounce_pos[i * 3], c.bounce_pos[i * 3 + 1]) : (c.bounce_in[i] != 0);
      const bool miss_ball = c.ball_pos[i * 3 + 1] < c.root_pos[i * 3 + 1] - 1.0f;
      const bool twice = hb && c.ball_pos[i * 3 + 2] < 0.05f;
      rec[w] = ta1 && (hc || miss_ball || twice);
      term[w] = (rec[w] && !hc) || (ta0 && hb && !bin);
    }
    c.distance[e] += sqrtf(c.root_vel[e * 3] * c.root_vel[e * 3] + c.root_vel[e * 3 + 1] * c.root_vel[e * 3 + 1]);  // _compute_stats
    bool reaction = rec[1], recovery = rec[0];     // "recovery also marks the reaction of their opponent"
    if (term[0] || term[1]) { c.reset_buf[e] = 1; reaction = false; recovery = false; }
    c.reset_reaction[e] = reaction ? 1 : 0;
    c.reset_recovery[e] = recovery ? 1 : 0;
  }
  // ---- reset FSM (:408-436)
  if (lane == 0 && !c.obs_only && !c.dual) {
    const bool out = rp[0] < c.court_min[0] || rp[1] < c.court_min[1] || rp[0] > c.court_max[0] || rp[1] > c.court_max[1];
    bool terminate = out || has_nan;
    int64_t reset = (c.progress_buf[e] >= (int64_t)c.max_episode_length - 1) ? 1 : (terminate ? 1 : 0);
    bool reaction = c.tar_time[e] == c.tar_time_total[e];
    const bool behind = bp[1] < rp[1] - 1.0f;
    bool recovery = (c.tar_action[e] == 1) && (has_contact || behind);
    c.distance[e] += sqrtf(c.root_vel[e * 3] * c.root_vel[e * 3] + c.root_vel[e * 3 + 1] * c.root_vel[e * 3 + 1]);  // _compute_stats
    if (c.early_termination) {
      terminate = terminate || (recovery && !has_contact) || behind;
      if (c.reward_type == 2) terminate = terminate || (has_contact && !c.est_bounce_in[e]);
    }
    if (terminate) { reset = 1; recovery = false; }
    reaction = reaction || (reset != 0);
    c.terminate_buf[e] = terminate ? 1 : 0;
    c.reset_buf[e] = reset;
    c.reset_reaction[e] = reaction ? 1 : 0;
    c.reset_recovery[e] = recovery ? 1 : 0;
  }
  if (lane == 0 && c.obs_only && touched) { c.reset_reaction[e] = 0; c.reset_recovery[e] = 0; }   // tail of _reset_envs (:176-177) for the reset humanoids
}

// ------------------------------------------------------------------------------------------ per-row results of the test set
// b200v2p_eval_ball_stats: one thread per env.  The flagged lanes of a warp are grouped by row (__match_any_sync); a group's counts are
// popcounts of its ballots, its error the sum of its bounce-in lanes' fixed-point values; the group's lowest lane adds them.
// kDraws: the draws form (reset_reaction -> row_served), else the events form (reset_recovery -> buckets)
#define BSTATS_THREADS 256
template <bool kDraws>
__global__ void __launch_bounds__(BSTATS_THREADS) eval_ball_stats_kernel(b200v2p_bstats_t d) {
  const int lane = threadIdx.x & 31;
  const int64_t e = (int64_t)blockIdx.x * BSTATS_THREADS + threadIdx.x;
  const bool ev = e < d.n && (kDraws ? d.reset_reaction[e] : d.reset_recovery[e]) != 0;
  const unsigned evs = __ballot_sync(FULL, ev);
  if (evs == 0) return;                       // warp-uniform
  int64_t row = 0;
  unsigned peers = 0;
  if (ev) {
    row = (d.pool_cursor[e] + d.pool_size - 1) % d.pool_size;
    peers = __match_any_sync(evs, (unsigned long long)row);
  }
  if constexpr (kDraws) {
    if (ev && lane == __ffs(peers) - 1)
      atomicAdd(reinterpret_cast<unsigned long long*>(d.row_served + row), (unsigned long long)__popc(peers));
    return;
  }
  bool hit = false, fh = false, bin = false;
  long long q = 0;
  if (ev) {
    hit = d.has_contact[e] != 0;
    fh = d.swing_type_cycle[e] == 1;
    bin = d.est_bounce_in[e] != 0;
    if (bin) {   // meter 3's value (eval_reset), then fixed point: v * 2^24 is exact in double, one rounding to the integer
      float dd[3];
#pragma unroll
      for (int k = 0; k < 3; k++) dd[k] = __fsub_rn(d.est_bounce_pos[e * 3 + k], d.target_bounce_pos[e * 3 + k]);
      const float v = sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(dd[0], dd[0]), __fmul_rn(dd[1], dd[1])), __fmul_rn(dd[2], dd[2])));
      q = __double2ll_rn((double)v * B200V2P_BSTATS_FIX_SCALE);
    }
  }
  const unsigned hits = __ballot_sync(FULL, hit), fhs = __ballot_sync(FULL, fh), bins = __ballot_sync(FULL, bin);
  long long err = 0;
  for (unsigned m = bins; m; m &= m - 1) {    // warp-uniform: every lane takes part in each shuffle
    const int src = __ffs(m) - 1;
    const long long t = __shfl_sync(FULL, q, src);
    if ((peers >> src) & 1u) err += t;
  }
  if (!ev || lane != __ffs(peers) - 1) return;
  unsigned long long* b = reinterpret_cast<unsigned long long*>(d.buckets + row * B200V2P_BSTATS_COLS);
  atomicAdd(b, (unsigned long long)__popc(peers));
  const unsigned long long c[3] = {(unsigned long long)__popc(peers & hits), (unsigned long long)__popc(peers & fhs),
                                   (unsigned long long)__popc(peers & bins)};
#pragma unroll
  for (int k = 0; k < 3; k++)
    if (c[k]) atomicAdd(b + 1 + k, c[k]);
  if (err) atomicAdd(b + 4, (unsigned long long)err);
}

// ------------------------------------------------------------------------------------------ rally results of the dual test run
// b200v2p_eval_rally_stats: one thread per pair.  The per-pair state is the thread's own; the warp's counts are popcounts of ballots and
// its shot / frame sums a shuffle reduction, added by lane 0; the ending lanes are grouped by histogram bucket (__match_any_sync) and
// each group's lowest lane adds it.  Integer atomics only, so every run gives the same bits whatever the order.
#define RSTATS_THREADS 256
// the terms of the dual reset rule (physics_mvae_controller_dual.py:92-120) for player env i, as the dual block of
// controller_post_kernel computes them.  A copy of those lines rather than a function both kernels call: moving them into a shared
// function changes the post kernel's SASS, which is kept as shipped.  This launch runs after the post launch, so bounce_in[i] already
// holds this step's value, which the post kernel recomputes for the partner's env.  rec: the player meets the ball (to hit, and it
// touched it, is behind or bounced twice); out: a ball it hit bounced out
struct DualTerms { bool rec, hc, twice, out; };
__device__ __forceinline__ DualTerms dual_terms(const b200v2p_rstats_t& d, int64_t i) {
  const bool ta1 = d.tar_action[i] == 1, ta0 = d.tar_action[i] == 0, hc = d.has_contact[i] != 0, hb = d.has_bounce[i] != 0;
  const bool bin = d.bounce_in[i] != 0;
  const bool miss_ball = d.ball_pos[i * 3 + 1] < d.root_pos[i * 3 + 1] - 1.0f;
  const bool twice = hb && d.ball_pos[i * 3 + 2] < 0.05f;
  DualTerms t;
  t.rec = ta1 && (hc || miss_ball || twice);
  t.hc = hc;
  t.twice = twice;
  t.out = ta0 && hb && !bin;
  return t;
}
__device__ __forceinline__ long long warp_sum(long long v) {
#pragma unroll
  for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(FULL, v, o);
  return v;
}
__global__ void __launch_bounds__(RSTATS_THREADS) eval_rally_stats_kernel(b200v2p_rstats_t d) {
  const int lane = threadIdx.x & 31;
  const int64_t k = (int64_t)blockIdx.x * RSTATS_THREADS + threadIdx.x;
  bool faced[2] = {false, false}, hit[2] = {false, false}, fh[2] = {false, false};
  bool cause[2][B200V2P_RSTATS_CAUSES] = {};
  bool end = false;
  long long shots = 0, frames = 0;
  if (k < (d.n >> 1)) {
    const int64_t a = 2 * k;
    const int64_t progress = d.progress_buf[a];
    const bool opening = progress == 1;      // the first post launch after the pair's reset opens its rally
    if (opening || d.pair_open[k]) {
      long long h[2] = {0, 0};
      if (!opening) { h[0] = d.pair_hits[a]; h[1] = d.pair_hits[a + 1]; }
#pragma unroll
      for (int w = 0; w < 2; w++) {
        const int64_t i = a + w;
        const DualTerms t = dual_terms(d, i);
        faced[w] = t.rec;
        hit[w] = t.rec && t.hc;
        fh[w] = hit[w] && d.swing_type_cycle[i] == 1;
        cause[w][0] = t.rec && !t.hc && !t.twice;    // behind
        cause[w][1] = t.rec && !t.hc && t.twice;     // double bounce
        cause[w][2] = t.out;
        h[w] += hit[w] ? 1 : 0;
        end = end || cause[w][0] || cause[w][1] || cause[w][2];
      }
      if (opening || hit[0] || hit[1]) { d.pair_hits[a] = h[0]; d.pair_hits[a + 1] = h[1]; }
      if (end) {
        shots = h[0] + h[1];
        frames = progress;
      }
      if (opening || end) d.pair_open[k] = end ? 0 : 1;    // open until the rally ends (the pair then waits for its reset)
    }
  }
  const unsigned ends = __ballot_sync(FULL, end);
  if (__ballot_sync(FULL, end || faced[0] || faced[1]) == 0) return;   // warp-uniform
  if (end) {
    const long long bucket = shots < B200V2P_RSTATS_HIST - 1 ? shots : B200V2P_RSTATS_HIST - 1;
    const unsigned peers = __match_any_sync(ends, (unsigned long long)bucket);
    if (lane == __ffs(peers) - 1)
      atomicAdd(reinterpret_cast<unsigned long long*>(d.shots_hist + bucket), (unsigned long long)__popc(peers));
  }
  unsigned long long v[15];
  v[0] = __popc(ends);
  v[1] = ends ? (unsigned long long)warp_sum(shots) : 0ull;
  v[2] = ends ? (unsigned long long)warp_sum(frames) : 0ull;
#pragma unroll
  for (int w = 0; w < 2; w++) {
#pragma unroll
    for (int c = 0; c < B200V2P_RSTATS_CAUSES; c++) v[3 + w * B200V2P_RSTATS_CAUSES + c] = __popc(__ballot_sync(FULL, cause[w][c]));
    v[9 + w * 3] = __popc(__ballot_sync(FULL, faced[w]));
    v[10 + w * 3] = __popc(__ballot_sync(FULL, hit[w]));
    v[11 + w * 3] = __popc(__ballot_sync(FULL, fh[w]));
  }
  if (lane != 0) return;
  unsigned long long* const dst[3] = {reinterpret_cast<unsigned long long*>(d.totals), reinterpret_cast<unsigned long long*>(d.ends),
                                      reinterpret_cast<unsigned long long*>(d.player)};
#pragma unroll
  for (int j = 0; j < 15; j++)
    if (v[j]) atomicAdd(j < 3 ? dst[0] + j : (j < 9 ? dst[1] + (j - 3) : dst[2] + (j - 9)), v[j]);
}

// ------------------------------------------------------------------------------------------ test-time rally recorder
// render_vis's per-frame append (mvae_controller_vis.py:140-146, mvae_controller_vis_dual.py:156-162): one warp per env writes the
// env's frame at row *row_counter (single; the last block advances the counter) or progress_buf[e] (dual); rows >= cap are dropped
__global__ void __launch_bounds__(V2P_WARPS * 32) eval_record_kernel(b200v2p_rec_t r) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t e = (int64_t)blockIdx.x * V2P_WARPS + warp;
  if (e < r.n) {
    const int64_t row = r.row_counter ? r.row_counter[0] : r.progress_buf[e];
    if (row >= 0 && row < r.cap) {
      const int64_t o = e * r.cap + row;
      for (int k = lane; k < 72; k += 32) r.rec_joint_rot[o * 72 + k] = r.joint_rot[e * 72 + k];
      if (lane < 3) {
        r.rec_root_pos[o * 3 + lane] = r.root_pos[e * 3 + lane];
        r.rec_ball_pos[o * 3 + lane] = r.ball_pos[e * 3 + lane];
        if (r.rec_target_pos) r.rec_target_pos[o * 3 + lane] = r.target_pos[e * 3 + lane];
      }
      if (lane == 3) r.rec_phase[o] = r.phase[e];
      if (lane == 4) r.rec_swing_type[o] = r.swing_type[e];
      if (lane == 5 && r.rec_tar_action) r.rec_tar_action[o] = r.tar_action[e];
    }
  }
  if (r.row_counter) last_block_advance(r.row_counter, r.done_counter, 1);
}

// ------------------------------------------------------------------------------------------ dual best-episode list
// mvae_controller_vis_dual.py:164-195 on one CTA: first argmax over the flagged pairs, then the insertion rule on the slot order.
// The argmax is torch.argmax's: a NaN ranks above every number and the first NaN wins, so the pair taken is the same whatever the
// thread and shuffle order.  The insertion rule's > is false for a NaN, as in the reference: a NaN pair enters only an empty list,
// and once it is there nothing passes it.
__global__ void __launch_bounds__(1024) eval_best_select_kernel(b200v2p_best_t b) {
  __shared__ float sd[32];
  __shared__ int64_t sk[32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float d = 0.0f;
  int64_t k = -1;   // a thread walks its pairs in increasing order, so a strict rank keeps the first of equal distances or NaNs
  for (int64_t p = threadIdx.x; p < b.n / 2; p += blockDim.x) {
    if (b.reset_buf[2 * p] == 0) continue;
    const float v = __fadd_rn(b.distance[2 * p], b.distance[2 * p + 1]);
    if (k < 0 || (d == d && (v != v || v > d))) { d = v; k = p; }
  }
  // (d, k) beats (od, ok) when it is valid and either the other is not, or its distance ranks higher (NaN above every number), or
  // ranks the same (equal, or both NaN) with a lower pair
  const auto take = [](float od, int64_t ok, float d, int64_t k) {
    const bool onan = od != od, dnan = d != d;
    return ok >= 0 && (k < 0 || (onan && !dnan) || (!dnan && od > d) || ((od == d || (onan && dnan)) && ok < k));
  };
#pragma unroll
  for (int s = 16; s > 0; s >>= 1) {
    const float od = __shfl_down_sync(FULL, d, s);
    const int64_t ok = __shfl_down_sync(FULL, k, s);
    if (take(od, ok, d, k)) { d = od; k = ok; }
  }
  if (lane == 0) { sd[warp] = d; sk[warp] = k; }
  __syncthreads();
  if (threadIdx.x != 0) return;
  for (int w = 1; w < (int)(blockDim.x >> 5); w++)
    if (take(sd[w], sk[w], d, k)) { d = sd[w]; k = sk[w]; }
  b.copy_slot[0] = -1;
  if (k < 0) return;
  const int64_t L = b.list_len[0];
  if (L > 0 && !(d > b.best_distance[b.order[L - 1]])) return;   // the list grows only past its last entry, even while short
  int64_t ins = 0;
  while (ins < L && !(d > b.best_distance[b.order[ins]])) ins++;
  const int64_t slot = L < b.num_eg ? L : b.order[b.num_eg - 1];   // a free slot, or the one of the entry that falls off the end
  const int64_t nl = L < b.num_eg ? L + 1 : L;
  for (int64_t i = nl - 1; i > ins; i--) b.order[i] = b.order[i - 1];
  b.order[ins] = slot;
  b.list_len[0] = nl;
  b.best_distance[slot] = d;
  b.best_env[slot] = 2 * k;
  const int64_t nf = b.progress_buf[2 * k];
  b.best_nframes[slot] = nf < b.cap ? nf : b.cap;
  b.copy_slot[0] = slot;
}
// rows [0, best_nframes) of both envs of the chosen pair -> best_*[slot]: block (row, player), thread = one value of the row
__global__ void __launch_bounds__(96) eval_best_copy_kernel(b200v2p_best_t b) {
  const int64_t slot = b.copy_slot[0];
  if (slot < 0) return;
  const int64_t row = blockIdx.x;
  if (row >= b.best_nframes[slot]) return;
  const int t = threadIdx.x;
  const int64_t s = (b.best_env[slot] + blockIdx.y) * b.cap + row, o = (slot * 2 + blockIdx.y) * b.cap + row;
  if (t < 72) b.best_joint_rot[o * 72 + t] = b.rec_joint_rot[s * 72 + t];
  else if (t < 75) b.best_root_pos[o * 3 + t - 72] = b.rec_root_pos[s * 3 + t - 72];
  else if (t < 78) b.best_ball_pos[o * 3 + t - 75] = b.rec_ball_pos[s * 3 + t - 75];
  else if (t == 78) b.best_phase[o] = b.rec_phase[s];
  else if (t == 79) b.best_swing_type[o] = b.rec_swing_type[s];
  else if (t == 80) b.best_tar_action[o] = b.rec_tar_action[s];
}

// ------------------------------------------------------------------------------------------ two-hand backhand fix
// HumanoidSMPLIMMVAE.optimize_two_hand_backhand (env/tasks/humanoid_smpl_im_mvae.py:948-1031, single=True) with the selection and
// write-back of its callers (mvae_controller_vis.py:181-191, mvae_controller_vis_dual.py:213-231).  One CTA per problem (one player of
// one episode): it compacts its selected frames into a batch of M rows, computes each row's fixed Spine3 (joint 9) transform and
// target once, then runs every Adam step in the kernel: FK of the free arm (collar, shoulder, elbow, wrist, hand), the L1 gradients,
// reverse mode through the chain and the konia exp map, the Adam update.  The delta is double-buffered and one barrier per step
// makes every row read its neighbour's delta of the same step.  Per-row state lives in the caller's scratch (M has no bound).
#define BHFIX_THREADS 256
enum { BH_BASE = 0, BH_G9 = 12, BH_P9 = 21, BH_TGT = 24, BH_M = 27, BH_V = 39, BH_D = 51 };   // BH_D: two 12-word delta buffers
static_assert(BH_D + 24 == B200V2P_BHFIX_FRAME_WORDS, "scratch words per frame");

template <typename T>
__device__ __forceinline__ T l1_sign(T x) { return x > T(0) ? T(1) : (x < T(0) ? T(-1) : T(0)); }   // torch.sgn: 0 at 0 and at NaN

// reverse mode of aa_to_rotmat: dL/daa from dL/dR for the formula as written.  Normal branch: theta = sqrt(theta2),
// w = aa / (theta + 1e-6), R = c I + s [w]x + (1 - c) w w^T; where theta2 <= 1e-6 autograd sees the Taylor branch I + [aa]x alone
template <typename T>
__device__ __forceinline__ void aa_to_rotmat_vjp(const T* aa, const T* dR, T* g) {
  const T v[3] = {dR[7] - dR[5], dR[2] - dR[6], dR[3] - dR[1]};   // <dR, d[w]x / dw>
  const T theta2 = aa[0] * aa[0] + aa[1] * aa[1] + aa[2] * aa[2];
  if (!(theta2 > T(1e-6))) {
    g[0] = v[0]; g[1] = v[1]; g[2] = v[2];
    return;
  }
  const T theta = sqrt(theta2), d = theta + T(1e-6);
  const T w[3] = {aa[0] / d, aa[1] / d, aa[2] / d};
  const T c = cos(theta), s = sin(theta), k = T(1) - c;
  T Sw[3];   // (dR + dR^T) w
#pragma unroll
  for (int r = 0; r < 3; r++) Sw[r] = (dR[r * 3] + dR[r]) * w[0] + (dR[r * 3 + 1] + dR[3 + r]) * w[1] + (dR[r * 3 + 2] + dR[6 + r]) * w[2];
  const T dk = T(0.5) * (w[0] * Sw[0] + w[1] * Sw[1] + w[2] * Sw[2]);
  const T dc = dR[0] + dR[4] + dR[8] - dk;
  const T ds = w[0] * v[0] + w[1] * v[1] + w[2] * v[2];
  T dw[3];
#pragma unroll
  for (int r = 0; r < 3; r++) dw[r] = s * v[r] + k * Sw[r];
  const T dd = -(dw[0] * w[0] + dw[1] * w[1] + dw[2] * w[2]) / d;
  const T dtheta = -s * dc + c * ds + dd;
#pragma unroll
  for (int r = 0; r < 3; r++) g[r] = dw[r] / d + aa[r] * dtheta / theta;
}

template <typename T>
__device__ __forceinline__ void rel_joint(const T* rest, int j, int par, T* rel) {
#pragma unroll
  for (int k = 0; k < 3; k++) rel[k] = rest[j * 3 + k] - rest[par * 3 + k];
}

template <typename T>
__global__ void __launch_bounds__(BHFIX_THREADS) backhand_fix_kernel(const b200v2p_bhprob_t* __restrict__ probs, int32_t* __restrict__ idx_all,
                                                                      T* __restrict__ state_all, int iters, T* __restrict__ losses) {
  __shared__ T rest[72];
  __shared__ int s_warp[BHFIX_THREADS / 32];
  __shared__ int s_count;
  __shared__ T s_red[3][BHFIX_THREADS / 32];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const b200v2p_bhprob_t pr = probs[blockIdx.x];
  int64_t off = 0;   // frames of the problems before this one, each rounded up to a warp's 32
  for (unsigned q = 0; q < blockIdx.x; q++) off += (probs[q].T + 31) / 32 * 32;
  const int64_t Tn = pr.T;
  const T* jr = (const T*)pr.joint_rot;
  const T* ph = (const T*)pr.phase;
  T* out = (T*)pr.out;
  int32_t* idx = idx_all + off;
  T* st = state_all + off * B200V2P_BHFIX_FRAME_WORDS;
  // scratch word w of batch row i: rows grouped by 32, one word of a group's rows contiguous (a warp's access is coalesced and the
  // word offsets are immediates)
  const auto row_of = [&](int i) { return st + (int64_t)(i >> 5) * (B200V2P_BHFIX_FRAME_WORDS * 32) + (i & 31); };
  if (Tn > 0)
    for (int k = tid; k < 72; k += BHFIX_THREADS) rest[k] = ((const T*)pr.rest)[k];
  if (tid == 0) s_count = 0;
  __syncthreads();

  // need_fix = (swing_type == 2) & (phase > 2) & (phase < 5), compacted in frame order; the other rows are copied through
  for (int64_t c0 = 0; c0 < Tn; c0 += BHFIX_THREADS) {
    const int64_t f = c0 + tid;
    bool sel = false;
    if (f < Tn) {
      const T phf = ph[f];
      sel = pr.swing_type[f] == 2 && phf > T(2) && phf < T(5);
      if (!sel && out != jr)
        for (int k = 0; k < 72; k++) out[f * 72 + k] = jr[f * 72 + k];
    }
    const unsigned b = __ballot_sync(FULL, sel);
    if (lane == 0) s_warp[warp] = __popc(b);
    __syncthreads();
    int base = s_count;
    for (int w = 0; w < warp; w++) base += s_warp[w];
    if (sel) idx[base + __popc(b & ((1u << lane) - 1u))] = (int32_t)f;
    __syncthreads();
    if (tid == 0)
      for (int w = 0; w < BHFIX_THREADS / 32; w++) s_count += s_warp[w];
    __syncthreads();
  }
  const int M = s_count;
  // free arm (fitted) and racket arm, from the collar to the hand; delta row k = 3 - chain position (Wrist, Elbow, Shoulder, Collar)
  // SMPL left arm from the collar: 13, 16, 18, 20, 22 (L_Hand); the right arm's joints are one further each
  const int L = pr.righthand ? 0 : 1;
  const auto left_arm = [](int c) { return c ? 14 + 2 * c : 13; };
  const auto fc = [&](int c) { return left_arm(c) + L; };
  const auto rc = [&](int c) { return left_arm(c) + 1 - L; };
  __shared__ T frel[5][3];
  if (tid < 5) rel_joint(rest, fc(tid), tid ? fc(tid - 1) : 9, frel[tid]);
  __syncthreads();

  // per row: Spine3's global transform, the target 2 hand - wrist - root of the racket arm (root_pos = 0: rb = P - rest[0]),
  // the base angle-axis of the fitted joints (rotation_matrix_to_angle_axis of angle_axis_to_rotation_matrix), Adam state
  for (int i = tid; i < M; i += BHFIX_THREADS) {
    const T* a = jr + (int64_t)idx[i] * 72;
    T* row = row_of(i);
    T R[9], G[9], P[3], Gn[9], Pn[3], rel[3];
    aa_to_rotmat(a, G);
#pragma unroll
    for (int k = 0; k < 3; k++) P[k] = rest[k];
    const int spine[3] = {3, 6, 9};
#pragma unroll
    for (int s = 0; s < 3; s++) {
      aa_to_rotmat(a + spine[s] * 3, R);
      rel_joint(rest, spine[s], s ? spine[s - 1] : 0, rel);
      chain_link(G, P, R, rel, Gn, Pn);
#pragma unroll
      for (int k = 0; k < 9; k++) G[k] = Gn[k];
#pragma unroll
      for (int k = 0; k < 3; k++) P[k] = Pn[k];
    }
#pragma unroll
    for (int k = 0; k < 9; k++) row[(BH_G9 + k) * 32] = G[k];
#pragma unroll
    for (int k = 0; k < 3; k++) row[(BH_P9 + k) * 32] = P[k];
#pragma unroll
    for (int c = 0; c < 4; c++) {
      aa_to_rotmat(a + rc(c) * 3, R);
      rel_joint(rest, rc(c), c ? rc(c - 1) : 9, rel);
      chain_link(G, P, R, rel, Gn, Pn);
#pragma unroll
      for (int k = 0; k < 9; k++) G[k] = Gn[k];
#pragma unroll
      for (int k = 0; k < 3; k++) P[k] = Pn[k];
    }
    rel_joint(rest, rc(4), rc(3), rel);
#pragma unroll
    for (int r = 0; r < 3; r++) {
      const T hand = G[r * 3] * rel[0] + G[r * 3 + 1] * rel[1] + G[r * 3 + 2] * rel[2] + P[r];
      const T root = rest[r] - (rest[r] - T(0));
      row[(BH_TGT + r) * 32] = T(2) * (hand - (rest[r] - T(0))) - (P[r] - (rest[r] - T(0))) - root;
    }
#pragma unroll
    for (int c = 0; c < 4; c++) {
      T q[4], aa[3];
      aa_to_rotmat(a + fc(c) * 3, R);
      rotmat_to_quat_wxyz(R, q);
      quat_wxyz_to_angle_axis(q, aa);
#pragma unroll
      for (int k = 0; k < 3; k++) row[(BH_BASE + (3 - c) * 3 + k) * 32] = aa[k];
    }
#pragma unroll
    for (int k = 0; k < 12; k++) { row[(BH_M + k) * 32] = T(0); row[(BH_V + k) * 32] = T(0); row[(BH_D + k) * 32] = T(0); }
  }
  __syncthreads();

  // L1Loss(mean) * weight: d/dx = weight / numel * sgn(x)
  const T w_tgt = T(1) / T(3 * (int64_t)M), w_reg = T(0.2) / T(12 * (int64_t)M), w_smooth = T(0.5) / T(12 * ((int64_t)M - 1));
  T sum_tgt = T(0), sum_reg = T(0), sum_smooth = T(0);
  for (int it = 0; it < iters; it++) {
    // torch.optim.Adam(lr=0.005, betas=(0.9, 0.999), eps=1e-8): bias corrections in double like the Python scalars, then the tensor type
    const double bc1 = 1.0 - pow(0.9, (double)(it + 1)), bc2 = 1.0 - pow(0.999, (double)(it + 1));
    const T step_size = T(0.005 / bc1), bc2_sqrt = T(sqrt(bc2));
    const int dc = BH_D + 12 * (it & 1), dn = BH_D + 12 * ((it + 1) & 1);   // delta words read / written by this step
    const bool last = it == iters - 1;
    for (int i = tid; i < M; i += BHFIX_THREADS) {
      T* row = row_of(i);
      const T* prev = row_of(i - 1);
      // the fitted joint c's angle-axis is re-read where it is needed (scratch, cache-resident) rather than held in registers
      const auto joint_aa = [&](int c, T* a) {
#pragma unroll
        for (int k = 0; k < 3; k++) a[k] = row[(BH_BASE + (3 - c) * 3 + k) * 32] + row[(dc + (3 - c) * 3 + k) * 32];
      };
      T G[4][9], P[3], R[9], a[3];
#pragma unroll
      for (int k = 0; k < 9; k++) G[0][k] = row[(BH_G9 + k) * 32];
#pragma unroll
      for (int k = 0; k < 3; k++) P[k] = row[(BH_P9 + k) * 32];
      // forward: G[c] is the parent transform of chain joint c (G[0] = Spine3); the wrist's transform ends in Gw
      T Gw[9];
#pragma unroll
      for (int c = 0; c < 4; c++) {
        T Pn[3];
        joint_aa(c, a);
        aa_to_rotmat(a, R);
        chain_link(G[c], P, R, frel[c], c < 3 ? G[c + 1] : Gw, Pn);
#pragma unroll
        for (int k = 0; k < 3; k++) P[k] = Pn[k];
      }
      T gh[3], diff[3];
#pragma unroll
      for (int r = 0; r < 3; r++) {
        const T hand = Gw[r * 3] * frel[4][0] + Gw[r * 3 + 1] * frel[4][1] + Gw[r * 3 + 2] * frel[4][2] + P[r];
        diff[r] = (hand - (rest[r] - T(0))) - row[(BH_TGT + r) * 32];
        gh[r] = w_tgt * l1_sign(diff[r]);
      }
      // reverse: dG = dL/d(transform of chain joint c); P_c = G[c] rel_c + P_{c-1} passes gh to every link.  Each joint's three
      // components take their reg and smoothness terms and the Adam update as soon as their FK gradient is known.
      T dG[9], s_reg = T(0), s_smooth = T(0);
#pragma unroll
      for (int r = 0; r < 3; r++)
#pragma unroll
        for (int k = 0; k < 3; k++) dG[r * 3 + k] = gh[r] * frel[4][k];
#pragma unroll
      for (int c = 3; c >= 0; c--) {
        T dR[9], dGp[9], g[3];
        joint_aa(c, a);
        aa_to_rotmat(a, R);
#pragma unroll
        for (int r = 0; r < 3; r++)
#pragma unroll
          for (int k = 0; k < 3; k++) {
            dR[r * 3 + k] = G[c][r] * dG[k] + G[c][3 + r] * dG[3 + k] + G[c][6 + r] * dG[6 + k];
            dGp[r * 3 + k] = dG[r * 3] * R[k * 3] + dG[r * 3 + 1] * R[k * 3 + 1] + dG[r * 3 + 2] * R[k * 3 + 2] + gh[r] * frel[c][k];
          }
        aa_to_rotmat_vjp(a, dR, g);
#pragma unroll
        for (int k = 0; k < 9; k++) dG[k] = dGp[k];
#pragma unroll
        for (int k = 0; k < 3; k++) {
          const int64_t w = (3 - c) * 3 + k;
          const T dl = row[(dc + w) * 32];
          T gk = g[k] + w_reg * l1_sign(dl);
          s_reg += fabs(dl);
          if (i > 0) {
            const T dd = dl - prev[(dc + w) * 32];
            gk += w_smooth * l1_sign(dd);
            s_smooth += fabs(dd);
          }
          T m = row[(BH_M + w) * 32], v = row[(BH_V + w) * 32];
          m = m + T(1.0 - 0.9) * (gk - m);                       // lerp_(grad, 1 - beta1), weight < 0.5 form
          v = v * T(0.999) + T(1.0 - 0.999) * gk * gk;          // mul_(beta2).addcmul_(grad, grad, value=1 - beta2)
          row[(BH_M + w) * 32] = m;
          row[(BH_V + w) * 32] = v;
          row[(dn + w) * 32] = dl - step_size * (m / (sqrt(v) / bc2_sqrt + T(1e-8)));
        }
      }
      if (last) {
        sum_tgt += fabs(diff[0]) + fabs(diff[1]) + fabs(diff[2]);
        sum_reg += s_reg;
        sum_smooth += s_smooth;
      }
    }
    __syncthreads();
  }

  // write-back: all 24 joints of a selected row through rotation_matrix_to_angle_axis, the fitted four from base + delta
  const int df = BH_D + 12 * (iters & 1);
  for (int i = tid; i < M; i += BHFIX_THREADS) {
    const int64_t f = idx[i];
    const T* row = row_of(i);
    for (int j = 0; j < 24; j++) {
      T a[3], R[9], q[4], o[3];
      const int c = j == fc(0) ? 0 : (j == fc(1) ? 1 : (j == fc(2) ? 2 : (j == fc(3) ? 3 : -1)));
#pragma unroll
      for (int k = 0; k < 3; k++)
        a[k] = c < 0 ? jr[f * 72 + j * 3 + k] : row[(BH_BASE + (3 - c) * 3 + k) * 32] + row[(df + (3 - c) * 3 + k) * 32];
      aa_to_rotmat(a, R);
      rotmat_to_quat_wxyz(R, q);
      quat_wxyz_to_angle_axis(q, o);
#pragma unroll
      for (int k = 0; k < 3; k++) out[f * 72 + j * 3 + k] = o[k];
    }
  }
  if (!losses) return;
  T part[3] = {sum_tgt, sum_reg, sum_smooth};
#pragma unroll
  for (int t = 0; t < 3; t++) {
#pragma unroll
    for (int s = 16; s > 0; s >>= 1) part[t] += __shfl_down_sync(FULL, part[t], s);
    if (lane == 0) s_red[t][warp] = part[t];
  }
  __syncthreads();
  if (tid != 0) return;
  T tot[3] = {T(0), T(0), T(0)};
  for (int w = 0; w < BHFIX_THREADS / 32; w++)
    for (int t = 0; t < 3; t++) tot[t] += s_red[t][w];
  // the mean of an empty L1 is NaN: every term at M = 0, the smoothness term at M <= 1; all three when no step was evaluated
  const T nan = T(NAN);
  losses[blockIdx.x * 3] = iters ? tot[0] / T(3 * (int64_t)M) : nan;
  losses[blockIdx.x * 3 + 1] = iters ? tot[1] / T(12 * (int64_t)M) * T(0.2) : nan;
  losses[blockIdx.x * 3 + 2] = iters && M > 1 ? tot[2] / T(12 * ((int64_t)M - 1)) * T(0.5) : nan;
}

// ------------------------------------------------------------------------------------------ dual mode: incoming-ball table
struct InParams { float lo[4], hi_m_step[4], step[4], d1, d2, d3; };   // HEIGHT, VEL_X, VEL_Y, VSPIN
__device__ __forceinline__ float in_round(float v, const InParams& P, int k) {   // clamp, (v - lo) / step, round half-even (:27-45)
  v = fminf(fmaxf(v, P.lo[k]), P.hi_m_step[k]);
  return rintf(__fdiv_rn(__fsub_rn(v, P.lo[k]), P.step[k]));
}
__global__ void __launch_bounds__(V2P_WARPS * 32) ball_in_estimate_kernel(int n, const int64_t* __restrict__ contact_ids,
                                                                          const float* __restrict__ ball_states, int stride,
                                                                          const float* __restrict__ table, int64_t rows, InParams P,
                                                                          float* __restrict__ traj, float* __restrict__ s_in,
                                                                          float* __restrict__ s_out) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t i = (int64_t)blockIdx.x * V2P_WARPS + warp;
  if (i >= n) return;
  const float* b = ball_states + contact_ids[i] * stride;
  const float vel_x = sqrtf(__fadd_rn(__fmul_rn(b[7], b[7]), __fmul_rn(b[8], b[8])));
  const float dx = __fdiv_rn(b[7], vel_x), dy = __fdiv_rn(b[8], vel_x);
  const float vspin = __fdiv_rn(sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(b[10], b[10]), __fmul_rn(b[11], b[11])), __fmul_rn(b[12], b[12]))),
                                6.283185307179586f);
  const float rh = in_round(b[2], P, 0), rx = in_round(vel_x, P, 1), ry = in_round(b[9], P, 2), rs = in_round(vspin, P, 3);
  // float32 index sum, truncated like .long() (:38-41)
  const float fi = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(__fmul_rn(__fmul_rn(rh, P.d1), P.d2), P.d3), __fmul_rn(__fmul_rn(rx, P.d2), P.d3)),
                                       __fmul_rn(ry, P.d3)), rs);
  int64_t row = (int64_t)fi;
  row = row < 0 ? 0 : (row >= rows ? rows - 1 : row);   // the reference would raise on an out-of-range row; clamp instead of faulting
  const float* t = table + row * 100;
  for (int k = lane; k < 50; k += 32) {   // traj_trans (:63-65): distance along the hit direction -> xy, mirrored for the receiver
    const float d = t[k * 2], z = t[k * 2 + 1];
    float* o = traj + (i * 50 + k) * 3;
    o[0] = -__fadd_rn(__fmul_rn(d, dx), b[0]);
    o[1] = -__fadd_rn(__fmul_rn(d, dy), b[1]);
    o[2] = z;
  }
  if (lane == 0) {
    const float height = __fadd_rn(__fmul_rn(rh, P.step[0]), P.lo[0]), vx = __fadd_rn(__fmul_rn(rx, P.step[1]), P.lo[1]);
    const float vy = __fadd_rn(__fmul_rn(ry, P.step[2]), P.lo[2]), vs = __fadd_rn(__fmul_rn(rs, P.step[3]), P.lo[3]);
    float* si = s_in + i * 13;
    float* so = s_out + i * 13;
    const float vin[2] = {__fmul_rn(-vx, dx), __fmul_rn(-vx, dy)};
    const float sp = __fmul_rn(__fmul_rn(vs, 3.141592653589793f), 2.0f);
    // omega = vspin * 2 pi * normalize(v x (0,0,-1)) = (-v_y, v_x, 0) / |.|.  The clamp keeps a NaN like F.normalize's clamp_min:
    // at v_xy = 0 the direction is NaN, and so is every component of omega, z included (0 / NaN)
    const float n0 = sqrtf(__fadd_rn(__fmul_rn(vin[1], vin[1]), __fmul_rn(vin[0], vin[0])));
    const float nn = n0 < 1e-12f ? 1e-12f : n0;
    const float wz = __fmul_rn(sp, __fdiv_rn(0.0f, nn));
    const float wi[3] = {__fmul_rn(sp, __fdiv_rn(-vin[1], nn)), __fmul_rn(sp, __fdiv_rn(vin[0], nn)), wz};
    si[0] = -b[0]; si[1] = -b[1]; si[2] = height;
    so[0] = b[0];  so[1] = b[1];  so[2] = height;
#pragma unroll
    for (int k = 3; k < 7; k++) { si[k] = b[k]; so[k] = b[k]; }
    si[7] = vin[0]; si[8] = vin[1]; si[9] = vy;
    so[7] = -vin[0]; so[8] = -vin[1]; so[9] = vy;
#pragma unroll
    for (int k = 0; k < 3; k++) { si[10 + k] = wi[k]; so[10 + k] = k < 2 ? -wi[k] : wz; }
  }
}

// ------------------------------------------------------------------------------------------ mask-driven task reset
// kSequential: the test-set branch of the offline pool (tennis_ball.py:444-447), row pool_cursor[e], then the cursor moves on
template <bool kSequential>
__global__ void __launch_bounds__(V2P_WARPS * 32) task_reset_kernel(b200v2p_treset_t r) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t e = (int64_t)blockIdx.x * V2P_WARPS + warp;
  if (e >= r.n) return;
  const bool rea = r.reset_reaction[e] != 0, rec = r.reset_recovery[e] != 0;
  if (!rea && !rec) return;
  if (rea) {  // _reset_balls (:503-524) with the offline pool's generate (tennis_ball.py:435-456)
    int64_t idx;
    if constexpr (kSequential) {
      idx = r.pool_cursor[e];     // no start_pos remapping in this branch
    } else {                      // sample_random (:436-444)
      idx = r.pool_rand[e];
      if (r.ball_pos[e * 3 + 1] > 0.0f) {
        idx = (int64_t)((r.ball_pos[e * 3] + 4.0f) / 8.0f * (float)r.pool_size) + r.side_rand[e];
        idx = idx < 0 ? 0 : (idx > r.pool_size - 1 ? r.pool_size - 1 : idx);
      }
    }
    const float* row = r.pool + idx * 307;
    __syncwarp();   // every lane has read the cursor before lane 0 moves it
    if constexpr (kSequential) {
      if (lane == 0) r.pool_cursor[e] = (idx + 1) % r.pool_size;
    }
    if (r.ball_obs) {   // use_history_ball_obs: _ball_traj is left alone (:187-188), _ball_obs <- the launch position repeated (:213-214)
      for (int k = lane; k < r.obs_traj_len * 3; k += 32) r.ball_obs[e * r.obs_traj_len * 3 + k] = row[k % 3];
    } else {
      for (int k = lane; k < 300; k += 32) r.ball_traj[e * 300 + k] = row[7 + k];
    }
    if (lane == 0) {
      float* b = r.ball_states + e * r.ball_stride;
      float* rb = r.rigid_body_state + (e * r.bodies_per_env + r.bodies_per_env - 1) * 13;
      const float v[3] = {row[3], row[4], row[5]};
      const float c[3] = {-v[1], v[0], 0.0f};
      // F.normalize and the target below: every product rounded on its own, like the reference's tensor ops (no fma contraction)
      const float nn = fmaxf(sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(c[0], c[0]), __fmul_rn(c[1], c[1])), __fmul_rn(c[2], c[2]))), 1e-12f);
      const float sp = row[6] * 3.141592653589793f * 2.0f;
#pragma unroll
      for (int k = 0; k < 3; k++) {
        const float w = sp * (c[k] / nn);
        b[k] = row[k]; b[7 + k] = v[k]; b[10 + k] = w;
        rb[k] = row[k]; rb[7 + k] = v[k]; rb[10 + k] = w;
        r.ball_pos[e * 3 + k] = row[k]; r.ball_vel[e * 3 + k] = v[k]; r.bounce_pos[e * 3 + k] = 0.0f;
      }
      r.has_bounce[e] = 0; r.has_contact[e] = 0;
    }
  }
  if (lane != 0) return;
  if (rec) {  // _reset_recovery_tasks (:242-245)
    r.tar_action[e] = 0;
    r.has_bounce[e] = 0;
    r.bounce_pos[e * 3] = 0.0f; r.bounce_pos[e * 3 + 1] = 0.0f; r.bounce_pos[e * 3 + 2] = 0.0f;
  }
  if (rea) {  // _reset_reaction_tasks (:203-240)
    r.tar_time[e] = 0;
    r.tar_action[e] = 1;
    r.num_reset_reaction[e] += 1;
    r.bounce_in[e] = 0;
    r.est_bounce_pos[e * 3] = 0.0f; r.est_bounce_pos[e * 3 + 1] = 0.0f; r.est_bounce_pos[e * 3 + 2] = 0.0f;
    r.est_bounce_time[e] = 0.0f;
    r.est_bounce_in[e] = 0;
    r.est_max_height[e] = 0.0f;
    r.swing_type_cycle[e] = -1;
    r.tar_time_total[e] = (int64_t)r.reaction_nframes + r.frame_rand[e];
    if (r.target_mode == 1) {        // 'continuous': one target shared by the envs reset in this call (:226-229)
#pragma unroll
      for (int k = 0; k < 3; k++)
        r.target_bounce_pos[e * 3 + k] = __fadd_rn(__fmul_rn(r.target_seed[k], r.target_max[k] - r.target_min[k]), r.target_min[k]);
    } else if (r.target_mode == 2) { // left / middle / right (:230-237)
      const float sd = r.target_seed[e];
      r.target_bounce_pos[e * 3] = sd < 0.33f ? -3.0f : (sd > 0.67f ? 3.0f : 0.0f);
      r.target_bounce_pos[e * 3 + 1] = 10.0f; r.target_bounce_pos[e * 3 + 2] = 0.0f;
    }
  }
}

// ------------------------------------------------------------------------------------------ humanoid reset from the FK pose
__global__ void __launch_bounds__(V2P_WARPS * 32) actor_reset_kernel(b200v2p_areset_t r) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int i = blockIdx.x * V2P_WARPS + warp;
  if (i >= r.n) return;
  const int64_t e = r.env_ids[i];
  if (r.mask && !r.mask[e]) return;
  const int nd = r.num_dof;
  float* rb = r.rigid_body_state + e * r.bodies_per_env * 13;
  if (lane < 24) {
    float* row = rb + lane * 13;
    const float* p = r.src_rb_pos + (e * 24 + lane) * 3;
    const float* q = r.src_rb_rot + (e * 24 + lane) * 4;
#pragma unroll
    for (int k = 0; k < 3; k++) { row[k] = p[k]; row[7 + k] = 0.0f; row[10 + k] = 0.0f; }
#pragma unroll
    for (int k = 0; k < 4; k++) { row[3 + k] = q[k]; r.prev_target_rb_rot[(e * 24 + lane) * 4 + k] = q[k]; }
  }
  if (lane == 24 && r.racket_body >= 0) {  // welded racket row = parent pose + rotated offset (first obs is consistent)
    const bool second = r.dual && (e & 1);
    const int rpar = second ? r.racket_parent2 : r.racket_parent;
    const float* pp = r.src_rb_pos + (e * 24 + rpar) * 3;
    const float* q = r.src_rb_rot + (e * 24 + rpar) * 4;
    const float* ro = second ? r.racket_offset2 : r.racket_offset;
    const float o[3] = {ro[0], ro[1], ro[2]};
    float t[3] = {2.0f * (q[1] * o[2] - q[2] * o[1]), 2.0f * (q[2] * o[0] - q[0] * o[2]), 2.0f * (q[0] * o[1] - q[1] * o[0])};
    float u[3] = {q[1] * t[2] - q[2] * t[1], q[2] * t[0] - q[0] * t[2], q[0] * t[1] - q[1] * t[0]};
    float* row = rb + r.racket_body * 13;
#pragma unroll
    for (int k = 0; k < 3; k++) { row[k] = pp[k] + o[k] + q[3] * t[k] + u[k]; row[7 + k] = 0.0f; row[10 + k] = 0.0f; }
#pragma unroll
    for (int k = 0; k < 4; k++) row[3 + k] = q[k];
  }
  for (int k = lane; k < nd; k += 32) {
    const float v = r.src_dof_pos[e * nd + k];
    r.dof_state[(e * nd + k) * 2] = v; r.dof_state[(e * nd + k) * 2 + 1] = 0.0f;
    r.pd_target_dof_pos[e * nd + k] = v;
  }
  if (lane == 0) {
    float* rs = r.root_states + e * r.root_stride;
#pragma unroll
    for (int k = 0; k < 3; k++) {
      const float v = r.src_root_pos[e * 3 + k];
      rs[k] = v; rs[7 + k] = 0.0f; rs[10 + k] = 0.0f;
      r.prev_target_root_pos[e * 3 + k] = v; r.root_pos[e * 3 + k] = v; r.root_vel[e * 3 + k] = 0.0f; r.target_root_pos[e * 3 + k] = v;
    }
#pragma unroll
    for (int k = 0; k < 4; k++) rs[3 + k] = r.src_root_rot[e * 4 + k];
    r.progress_buf[e] = 0; r.reset_buf[e] = 0; r.terminate_buf[e] = 0;
  }
}

// ------------------------------------------------------------------------------------------ controller bookkeeping of a humanoid reset
// PhysicsMVAEController._reset_envs (:176-181) for the envs whose mask is set: the controller's own progress / reset / terminate
// counters and statistics, one launch instead of seven masked fills
__global__ void ctrl_reset_kernel(int n, const uint8_t* __restrict__ mask, int64_t* progress, int64_t* reset_buf, int64_t* terminate,
                                  int64_t* num_reset_reaction, float* distance, int64_t* num_reset) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n || !mask[e]) return;
  progress[e] = 0; reset_buf[e] = 0; terminate[e] = 0; num_reset_reaction[e] = 0; distance[e] = 0.0f; num_reset[e] += 1;
}

// ------------------------------------------------------------------------------------------ high-level pre_physics_step
// PhysicsMVAEController.pre_physics_step (:247-262) before the motion generator runs: the latent part of the action scaled by
// vae_action_scale, replaced by clamp(N(0,1), -5, 5) for the envs in recovery (random_walk_in_recovery), the residual-dof part scaled
// by residual_dof_scale.  The normal deviates come from a counter-based generator (splitmix64 of seed, step counter, element index +
// Box-Muller, counter_rng.cuh) so that the step needs no separate RNG launch; the step counter lives on the device and is advanced
// by the last block to finish, which keeps the launch replayable inside a CUDA graph.
__global__ void pre_step_kernel(b200v2p_prestep_t p) {
  const int W = p.num_latent + p.num_res_dof;
  const int64_t step = p.step_counter[0];
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < (int64_t)p.n * W) {
    const int64_t e = i / W;
    const int k = (int)(i - e * W);
    const float a = p.actions[e * p.num_actions + k];
    if (k < p.num_latent) {
      float v = a * p.vae_action_scale;
      if (p.random_walk_in_recovery && p.tar_action[e] == 0) v = fminf(fmaxf(counter_normal(p.seed, (uint64_t)step, (uint64_t)i), -5.0f), 5.0f);
      p.mvae_actions[e * p.num_latent + k] = v;
    } else {
      p.res_dof_actions[e * p.num_res_dof + (k - p.num_latent)] = a * p.residual_dof_scale;
    }
  }
  last_block_advance(p.step_counter, p.done_counter, 1);
}

// ------------------------------------------------------------------------------------------ resident kinematic target stream
// StreamMotionPlayer (tasks/physics_mvae_controller.py; SURVEY.md 8d "synthetic kinematic target stream"): env e reads frame
// (t + off[e]) % K of the ring kept in HBM into the live buffers the FK kernel and the controller read.  One launch instead of six
// index_selects and the index arithmetic; `advance` = 1 moves the stream clock on by one frame first (step), 0 re-reads (reset).
__global__ void __launch_bounds__(V2P_WARPS * 32) stream_gather_kernel(b200v2p_stream_t s) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t e = (int64_t)blockIdx.x * V2P_WARPS + warp;
  const int64_t t = s.clock[0] + s.advance;
  if (e < s.n && (!s.reseed_mask || s.reseed_mask[e])) {
    if (s.reseed_mask) {          // reset of the masked envs: a fresh offset into the stream (counter-based draw), others untouched
      const uint64_t h = splitmix64(splitmix64(s.seed ^ ((uint64_t)t * 0xD1B54A32D192ED03ull)) + (uint64_t)e);
      if (lane == 0) s.offset[e] = (int64_t)(h % (uint64_t)s.frames);
      __syncwarp();
    }
    int64_t f = (t + s.offset[e]) % s.frames;
    if (f < 0) f += s.frames;
    const int64_t row = f * s.n + e;
    const float4* src = reinterpret_cast<const float4*>(s.ring_rotmat + row * 216);
    float4* dst = reinterpret_cast<float4*>(s.rotmat + e * 216);
    for (int k = lane; k < 54; k += 32) dst[k] = src[k];
    if (lane < 3) { s.root_pos[e * 3 + lane] = s.ring_root_pos[row * 3 + lane]; s.racket_pos[e * 3 + lane] = s.ring_racket_pos[row * 3 + lane]; }
    if (lane == 3) s.phase[e] = s.ring_phase[row];
    if (lane == 4) s.swing_type[e] = s.ring_swing_type[row];
    if (lane == 5) s.swing_type_cycle[e] = s.ring_swing_type_cycle[row];
  }
  if (s.advance) last_block_advance(s.clock, s.done_counter, s.advance);
}

// ------------------------------------------------------------------------------------------ C ABI
extern "C" {

const char* b200v2p_last_error(void) { return g_verr; }

int b200v2p_smpl_to_sim(const b200v2p_smpl_t* d, void* stream) {
  if (!d) return vfail(-1, "b200v2p_smpl_to_sim: bad arguments");
  const int n = d->n;
  if (n == 0) return 0;
  if (n < 0 || !d->root_pos || !d->joint_rotmat || !d->rest || !d->parents || !d->smpl_2_mujoco || !d->root_rot || !d->dof_pos || !d->root_vel ||
      !d->root_ang_vel || !d->dof_vel || !d->rb_pos || !d->rb_rot)
    return vfail(-1, "b200v2p_smpl_to_sim: bad arguments");
  if (!(d->dt > 0)) return vfail(-2, "b200v2p_smpl_to_sim: dt must be positive");
  if (d->num_rest < 1) return vfail(-2, "b200v2p_smpl_to_sim: num_rest must be >= 1");
  smpl_to_sim_kernel<<<(n + V2P_WARPS - 1) / V2P_WARPS, V2P_WARPS * 32, 0, (cudaStream_t)stream>>>(
      n, d->root_pos, d->joint_rotmat, d->rest, d->num_rest, d->parents, d->smpl_2_mujoco, d->dt, d->prev_root_pos, d->prev_rb_rot, d->root_rot,
      d->dof_pos, d->root_vel, d->root_ang_vel, d->dof_vel, d->rb_pos, d->rb_rot, d->prev_root_pos_update, d->target_root_pos_out, d->only_mask);
  V_CUDA_OK();
  return 0;
}

int b200v2p_fix_head(const b200v2p_head_t* d, void* stream) {
  if (!d) return vfail(-1, "b200v2p_fix_head: bad arguments");
  const int n = d->n;
  if (n == 0) return 0;
  if (n < 0 || !d->rb_pos || !d->rb_rot || !d->ball_pos || !d->root_pos || !d->joint_rotmat || d->head_body < 0 || d->head_body > 23)
    return vfail(-1, "b200v2p_fix_head: bad arguments");
  fix_head_kernel<<<(n + 127) / 128, 128, 0, (cudaStream_t)stream>>>(n, d->rb_pos, d->rb_rot, d->head_body, d->ball_pos, d->root_pos,
                                                                     d->joint_rotmat);
  V_CUDA_OK();
  return 0;
}

int b200v2p_ball_aero(const b200v2p_aero_t* d, void* stream) {
  if (!d) return vfail(-1, "b200v2p_ball_aero: bad arguments");
  const int n = d->n;
  if (n == 0) return 0;
  if (n < 0 || !d->ball_states || !d->has_bounce || !d->has_bounce_now || !d->bounce_pos || !d->force || d->stride < 13)
    return vfail(-1, "b200v2p_ball_aero: bad arguments");
  ball_aero_kernel<<<(n + 127) / 128, 128, 0, (cudaStream_t)stream>>>(n, d->ball_states, d->stride, d->has_bounce, d->has_bounce_now,
                                                                     d->bounce_pos, d->force, d->substeps, d->spin_scale);
  V_CUDA_OK();
  return 0;
}

int b200v2p_ball_reset(const b200v2p_breset_t* d, void* stream) {
  if (!d) return vfail(-1, "b200v2p_ball_reset: bad arguments");
  const int n = d->n;
  if (n == 0) return 0;
  if (n < 0 || !d->env_ids || !d->pool_index || !d->pool || !d->ball_states || !d->ball_pos || !d->ball_vel || !d->has_bounce || !d->bounce_pos ||
      !d->has_contact || !d->traj || d->stride < 13)
    return vfail(-1, "b200v2p_ball_reset: bad arguments");
  ball_reset_kernel<<<n, 64, 0, (cudaStream_t)stream>>>(n, d->env_ids, d->pool_index, d->pool, d->ball_states, d->stride, d->ball_pos,
                                                        d->ball_vel, d->has_bounce, d->bounce_pos, d->has_contact, d->traj);
  V_CUDA_OK();
  return 0;
}

int b200v2p_ball_in_estimate(const b200v2p_inest_t* d, void* stream) {
  if (!d) return vfail(-1, "b200v2p_ball_in_estimate: bad arguments");
  const int n = d->n;
  if (n == 0) return 0;
  if (n < 0 || !d->contact_ids || !d->ball_states || !d->table || d->table_rows < 1 || !d->traj || !d->states_in || !d->states_out ||
      d->stride < 13)
    return vfail(-1, "b200v2p_ball_in_estimate: bad arguments");
  const double* params = d->params;
  for (int k = 0; k < 4; k++)
    if (!(params[k * 3 + 2] > 0)) return vfail(-2, "b200v2p_ball_in_estimate: grid steps must be positive");
  InParams P;
  double dim[4];
  for (int k = 0; k < 4; k++) {   // python-double arithmetic of the reference, then the float32 cast torch applies to scalars
    const double lo = params[k * 3], hi = params[k * 3 + 1], st = params[k * 3 + 2];
    P.lo[k] = (float)lo; P.hi_m_step[k] = (float)(hi - st); P.step[k] = (float)st;
    dim[k] = (hi - lo) / st;
  }
  P.d1 = (float)dim[1]; P.d2 = (float)dim[2]; P.d3 = (float)dim[3];
  ball_in_estimate_kernel<<<(n + V2P_WARPS - 1) / V2P_WARPS, V2P_WARPS * 32, 0, (cudaStream_t)stream>>>(
      n, d->contact_ids, d->ball_states, d->stride, d->table, d->table_rows, P, d->traj, d->states_in, d->states_out);
  V_CUDA_OK();
  return 0;
}

int b200v2p_update_state(const b200v2p_state_t* s, void* stream) {
  if (!s) return vfail(-1, "b200v2p_update_state: null");
  if (s->n == 0) return 0;
  const int B = s->bodies_per_env;
  const auto body_ok = [B](int b) { return b >= 0 && b < B; };
  if (s->n < 0 || !s->rigid_body_state || !s->root_states || !s->ball_states || !s->has_contact || !s->has_contact_now || !s->root_pos ||
      !s->root_vel || !s->racket_pos || !s->racket_vel || !s->racket_normal || !s->ball_pos || !s->ball_vel || !s->ball_vspin ||
      s->ball_stride < 13 || s->root_stride < 13)
    return vfail(-1, "b200v2p_update_state: bad arguments");
  if (!body_ok(s->racket_body) || !body_ok(s->wrist_body) || (s->dual && (!body_ok(s->racket_body2) || !body_ok(s->wrist_body2))))
    return vfail(-2, "b200v2p_update_state: racket and wrist bodies must lie in [0, bodies_per_env)");
  update_state_kernel<<<(s->n + 127) / 128, 128, 0, (cudaStream_t)stream>>>(*s);
  V_CUDA_OK();
  return 0;
}

int b200v2p_actor_reset(const b200v2p_areset_t* r, void* stream) {
  if (!r) return vfail(-1, "b200v2p_actor_reset: null");
  if (r->n == 0) return 0;
  if (r->n < 0 || !r->env_ids || !r->src_root_pos || !r->root_states) return vfail(-1, "b200v2p_actor_reset: bad arguments");
  actor_reset_kernel<<<(r->n + V2P_WARPS - 1) / V2P_WARPS, V2P_WARPS * 32, 0, (cudaStream_t)stream>>>(*r);
  V_CUDA_OK();
  return 0;
}

int b200v2p_task_reset(const b200v2p_treset_t* r, void* stream) {
  if (!r) return vfail(-1, "b200v2p_task_reset: null");
  if (r->n == 0) return 0;
  if (r->pool_size < 1 || !r->pool || !r->reset_reaction || !r->reset_recovery) return vfail(-1, "b200v2p_task_reset: bad arguments");
  const unsigned grid = (r->n + V2P_WARPS - 1) / V2P_WARPS;
  if (r->pool_cursor)
    task_reset_kernel<true><<<grid, V2P_WARPS * 32, 0, (cudaStream_t)stream>>>(*r);
  else
    task_reset_kernel<false><<<grid, V2P_WARPS * 32, 0, (cudaStream_t)stream>>>(*r);
  V_CUDA_OK();
  return 0;
}

int32_t b200v2p_task_reset_desc_size(void) { return (int32_t)sizeof(b200v2p_treset_t); }

int b200v2p_eval_ball_stats(const b200v2p_bstats_t* d, void* stream) {
  if (!d) return vfail(-1, "b200v2p_eval_ball_stats: null");
  if (d->n == 0) return 0;
  if (d->n < 0 || d->pool_size < 1 || !d->pool_cursor) return vfail(-1, "b200v2p_eval_ball_stats: bad arguments");
  const bool draws = d->reset_reaction != nullptr;
  if (draws == (d->reset_recovery != nullptr))
    return vfail(-1, "b200v2p_eval_ball_stats: give reset_reaction (draws) or reset_recovery (events), not both or neither");
  if (draws ? !d->row_served
            : (!d->has_contact || !d->swing_type_cycle || !d->est_bounce_in || !d->est_bounce_pos || !d->target_bounce_pos || !d->buckets))
    return vfail(-1, "b200v2p_eval_ball_stats: bad arguments");
  const unsigned grid = (d->n + BSTATS_THREADS - 1) / BSTATS_THREADS;
  if (draws)
    eval_ball_stats_kernel<true><<<grid, BSTATS_THREADS, 0, (cudaStream_t)stream>>>(*d);
  else
    eval_ball_stats_kernel<false><<<grid, BSTATS_THREADS, 0, (cudaStream_t)stream>>>(*d);
  V_CUDA_OK();
  return 0;
}

int32_t b200v2p_eval_ball_stats_desc_size(void) { return (int32_t)sizeof(b200v2p_bstats_t); }

int b200v2p_eval_rally_stats(const b200v2p_rstats_t* d, void* stream) {
  if (!d) return vfail(-1, "b200v2p_eval_rally_stats: null");
  if (d->n < 0 || (d->n & 1)) return vfail(-1, "b200v2p_eval_rally_stats: n must be even and >= 0 (the pairs 2k, 2k+1)");
  const struct { const void* p; const char* name; } fields[] = {
      {d->tar_action, "tar_action"}, {d->has_contact, "has_contact"}, {d->has_bounce, "has_bounce"}, {d->bounce_in, "bounce_in"},
      {d->ball_pos, "ball_pos"}, {d->root_pos, "root_pos"}, {d->swing_type_cycle, "swing_type_cycle"}, {d->progress_buf, "progress_buf"},
      {d->pair_open, "pair_open"}, {d->pair_hits, "pair_hits"}, {d->totals, "totals"}, {d->ends, "ends"}, {d->player, "player"},
      {d->shots_hist, "shots_hist"}};
  for (const auto& f : fields)
    if (!f.p) {
      snprintf(g_verr, sizeof(g_verr), "b200v2p_eval_rally_stats: %s is NULL", f.name);
      return -1;
    }
  if (d->n == 0) return 0;
  const int64_t pairs = d->n >> 1;
  eval_rally_stats_kernel<<<(unsigned)((pairs + RSTATS_THREADS - 1) / RSTATS_THREADS), RSTATS_THREADS, 0, (cudaStream_t)stream>>>(*d);
  V_CUDA_OK();
  return 0;
}

int32_t b200v2p_eval_rally_stats_desc_size(void) { return (int32_t)sizeof(b200v2p_rstats_t); }

int b200v2p_ctrl_reset(const b200v2p_creset_t* d, void* stream) {
  if (!d) return vfail(-1, "b200v2p_ctrl_reset: bad arguments");
  const int n = d->n;
  if (n == 0) return 0;
  if (n < 0 || !d->mask || !d->progress_buf || !d->reset_buf || !d->terminate_buf || !d->num_reset_reaction || !d->distance || !d->num_reset)
    return vfail(-1, "b200v2p_ctrl_reset: bad arguments");
  ctrl_reset_kernel<<<(n + 255) / 256, 256, 0, (cudaStream_t)stream>>>(n, d->mask, d->progress_buf, d->reset_buf, d->terminate_buf,
                                                                      d->num_reset_reaction, d->distance, d->num_reset);
  V_CUDA_OK();
  return 0;
}

int b200v2p_pre_step(const b200v2p_prestep_t* p, void* stream) {
  if (!p) return vfail(-1, "b200v2p_pre_step: null");
  if (p->n == 0) return 0;
  if (p->n < 0 || !p->actions || !p->mvae_actions || !p->step_counter || !p->done_counter || p->num_latent < 1 || p->num_res_dof < 0 ||
      p->num_actions < p->num_latent + p->num_res_dof || (p->num_res_dof > 0 && !p->res_dof_actions) || (p->random_walk_in_recovery && !p->tar_action))
    return vfail(-1, "b200v2p_pre_step: bad arguments");
  const int64_t total = (int64_t)p->n * (p->num_latent + p->num_res_dof);
  pre_step_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(*p);
  V_CUDA_OK();
  return 0;
}

int b200v2p_stream_gather(const b200v2p_stream_t* s, void* stream) {
  if (!s) return vfail(-1, "b200v2p_stream_gather: null");
  if (s->n == 0) return 0;
  if (s->n < 0 || s->frames < 1 || !s->clock || !s->done_counter || !s->offset || !s->ring_rotmat || !s->rotmat || !s->ring_root_pos || !s->root_pos ||
      !s->ring_racket_pos || !s->racket_pos || !s->ring_phase || !s->phase || !s->ring_swing_type || !s->swing_type || !s->ring_swing_type_cycle ||
      !s->swing_type_cycle || s->advance < 0)
    return vfail(-1, "b200v2p_stream_gather: bad arguments");
  if (((uintptr_t)s->ring_rotmat | (uintptr_t)s->rotmat) & 15) return vfail(-2, "b200v2p_stream_gather: rotation matrices must be 16-byte aligned");
  stream_gather_kernel<<<(s->n + V2P_WARPS - 1) / V2P_WARPS, V2P_WARPS * 32, 0, (cudaStream_t)stream>>>(*s);
  V_CUDA_OK();
  return 0;
}

int b200v2p_controller_post(const b200v2p_ctrl_t* c, void* stream) {
  if (!c) return vfail(-1, "b200v2p_controller_post: null");
  if (c->n == 0) return 0;
  if (c->n < 0) return vfail(-1, "b200v2p_controller_post: bad arguments");
  // the NaN test of the reset FSM covers the columns the launch writes: a wider row would carry columns it never checks
  if (c->obs_traj_len < 0 || c->obs_traj_len > 100 || c->num_obs != 225 + 3 * c->obs_traj_len + (c->use_target ? 2 : 0))
    return vfail(-2, "b200v2p_controller_post: observation width / trajectory length mismatch");
  if (c->dual && (c->n & 1)) return vfail(-2, "b200v2p_controller_post: dual mode needs an even number of envs (pairs 2k, 2k+1)");
  if (c->reward_type < 0 || c->reward_type > 2) return vfail(-2, "b200v2p_controller_post: reward_type must be 0 (reach), 1 (return) or 2 (return_w_estimate)");
  if (c->use_history && !c->ball_obs) return vfail(-2, "b200v2p_controller_post: use_history needs the ball_obs buffer");
  if (c->policy_x) {
    if (c->policy_ld < c->num_obs) return vfail(-2, "b200v2p_controller_post: policy_ld is smaller than the observation row");
    if ((c->policy_mean == nullptr) != (c->policy_rstd == nullptr)) return vfail(-2, "b200v2p_controller_post: policy_mean and policy_rstd go together");
    if (c->policy_dual && (c->n & 1)) return vfail(-2, "b200v2p_controller_post: policy_dual needs an even number of envs");
    if (!(c->policy_clip_obs > 0.f) || !(c->policy_clip[0] > 0.f) || (c->policy_dual && !(c->policy_clip[1] > 0.f)))
      return vfail(-2, "b200v2p_controller_post: the policy row's clamps must be positive (inf: none)");
  }
  const unsigned grid = (c->n + V2P_WARPS - 1) / V2P_WARPS;
  if (c->eval && !c->obs_only) {
    if (c->dual) return vfail(-2, "b200v2p_controller_post: the test-time reset rule is single-player (dual keeps its FSM)");
    if (!c->ball_vel || !c->meter_sum || !c->meter_count || !c->meter_avg || !c->meter_max)
      return vfail(-1, "b200v2p_controller_post: eval needs ball_vel and the four meters' arrays");
    controller_post_kernel<true><<<grid, V2P_WARPS * 32, 0, (cudaStream_t)stream>>>(*c);
  } else {
    controller_post_kernel<false><<<grid, V2P_WARPS * 32, 0, (cudaStream_t)stream>>>(*c);
  }
  V_CUDA_OK();
  return 0;
}

int b200v2p_eval_record(const b200v2p_rec_t* r, void* stream) {
  if (!r) return vfail(-1, "b200v2p_eval_record: null");
  if (r->n == 0) return 0;
  if (r->n < 0 || r->cap < 1 || !r->joint_rot || !r->root_pos || !r->ball_pos || !r->phase || !r->swing_type || !r->rec_joint_rot ||
      !r->rec_root_pos || !r->rec_ball_pos || !r->rec_phase || !r->rec_swing_type || (r->rec_target_pos && !r->target_pos) ||
      (r->rec_tar_action && !r->tar_action))
    return vfail(-1, "b200v2p_eval_record: bad arguments");
  if (r->row_counter ? !r->done_counter : !r->progress_buf)
    return vfail(-2, "b200v2p_eval_record: a row counter (with its done counter) or progress_buf is needed");
  eval_record_kernel<<<(r->n + V2P_WARPS - 1) / V2P_WARPS, V2P_WARPS * 32, 0, (cudaStream_t)stream>>>(*r);
  V_CUDA_OK();
  return 0;
}

int b200v2p_eval_best(const b200v2p_best_t* b, void* stream) {
  if (!b) return vfail(-1, "b200v2p_eval_best: null");
  if (b->n == 0) return 0;
  if (b->n < 0 || (b->n & 1)) return vfail(-2, "b200v2p_eval_best: needs an even number of envs (pairs 2k, 2k+1)");
  if (b->cap < 1 || b->num_eg < 1 || !b->reset_buf || !b->progress_buf || !b->distance || !b->list_len || !b->order || !b->best_distance ||
      !b->best_env || !b->best_nframes || !b->copy_slot || !b->rec_joint_rot || !b->rec_root_pos || !b->rec_ball_pos || !b->rec_phase ||
      !b->rec_swing_type || !b->rec_tar_action || !b->best_joint_rot || !b->best_root_pos || !b->best_ball_pos || !b->best_phase ||
      !b->best_swing_type || !b->best_tar_action)
    return vfail(-1, "b200v2p_eval_best: bad arguments");
  eval_best_select_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(*b);
  eval_best_copy_kernel<<<dim3(b->cap, 2), 96, 0, (cudaStream_t)stream>>>(*b);
  V_CUDA_OK();
  return 0;
}

int b200v2p_backhand_fix(const b200v2p_bhfix_t* f, void* stream) {
  if (!f) return vfail(-1, "b200v2p_backhand_fix: null");
  if (f->num_problems < 0 || f->iters < 0) return vfail(-1, "b200v2p_backhand_fix: negative problem count or iters");
  if (f->num_problems == 0) return 0;
  if (!f->problems || !f->scratch) return vfail(-1, "b200v2p_backhand_fix: null problem table or scratch");
  if (f->precision != 0 && f->precision != 1) return vfail(-2, "b200v2p_backhand_fix: precision must be 0 (float32) or 1 (float64)");
  if ((uintptr_t)f->scratch & 15) return vfail(-2, "b200v2p_backhand_fix: scratch must be 16-byte aligned");
  int64_t frames = 0;
  for (int p = 0; p < f->num_problems; p++) {
    const b200v2p_bhprob_t& q = f->problems[p];
    if (q.T < 0 || q.T > INT32_MAX) return vfail(-1, "b200v2p_backhand_fix: T must lie in [0, 2^31)");
    if (q.T > 0 && (!q.joint_rot || !q.phase || !q.swing_type || !q.rest || !q.out))   // an empty episode may come with null arrays
      return vfail(-1, "b200v2p_backhand_fix: null problem array");
    if (q.swing_type_len < q.T) return vfail(-2, "b200v2p_backhand_fix: swing_type row shorter than T");
    frames += (q.T + 31) / 32 * 32;
  }
  const int S = f->precision ? 8 : 4;
  if (f->scratch_bytes < B200V2P_BHFIX_SCRATCH_BYTES(f->num_problems, frames, S)) return vfail(-2, "b200v2p_backhand_fix: scratch too small");
  char* s = (char*)f->scratch;
  const int64_t idx_at = B200V2P_BHFIX_ALIGN((int64_t)f->num_problems * (int64_t)sizeof(b200v2p_bhprob_t));
  const int64_t state_at = idx_at + B200V2P_BHFIX_ALIGN(frames * 4);
  // pageable source: the call returns once the table is staged, so the caller's array may go right away
  if (cudaMemcpyAsync(s, f->problems, f->num_problems * sizeof(b200v2p_bhprob_t), cudaMemcpyHostToDevice, (cudaStream_t)stream) != cudaSuccess)
    return vfail(-10, cudaGetErrorString(cudaGetLastError()));
  const b200v2p_bhprob_t* probs = (const b200v2p_bhprob_t*)s;
  int32_t* idx = (int32_t*)(s + idx_at);
  if (f->precision)
    backhand_fix_kernel<double><<<f->num_problems, BHFIX_THREADS, 0, (cudaStream_t)stream>>>(probs, idx, (double*)(s + state_at), f->iters,
                                                                                              (double*)f->losses);
  else
    backhand_fix_kernel<float><<<f->num_problems, BHFIX_THREADS, 0, (cudaStream_t)stream>>>(probs, idx, (float*)(s + state_at), f->iters,
                                                                                             (float*)f->losses);
  V_CUDA_OK();
  return 0;
}

}  // extern "C"
