// packed.cuh - "4 envs per warp" variant of the articulated control step (included by b200env.cu).
//
// Why: in the lane-per-body kernel the three tree passes run with 2-8 of 32
// lanes active - at most 5 bodies share a tree depth.  Here a warp owns EPW = 4 envs; lane = (env slot g = lane/8, body slot
// s = lane%8) and at every tree level slot s handles the s-th body of that depth (host table DevTree::lvl_*), so the level
// loops run on up to 20 lanes and are executed once for 4 envs.  Bodies change lanes from level to level, therefore the
// per-body quantities live in per-warp shared-memory records instead of registers; parent<->child exchange is a plain
// shared-memory read (no shuffles).  The arithmetic is the same as substep<T>() - same model, same oracle.
#pragma once

#ifndef PK_CONTACT_COMPACT
#define PK_CONTACT_COMPACT 1   // 1: per-vertex ground contact as a compacted phase of its own (pk_contact_phase); bit-identical;
                               // 0 keeps the in-place form for A/B
#endif
#ifndef PK_SYNC_EVERY
#define PK_SYNC_EVERY 1   // CTA barrier every n-th substep (keeps the CTA's warps on the same instruction-cache lines)
#endif
#ifndef PK_WARPS
#define PK_WARPS 8          // split form: 8 warps x 4 envs x 6.7 KB records + the 7.1 KB DevBlob header = 221 KB of shared memory: one CTA per SM
#endif
#ifndef PK_WARPS_FUSED
#define PK_WARPS_FUSED 7    // fused form: its 0.9 KB of prologue scratch per warp leaves room for 7 warps only
#endif
#ifndef PK_SHADOW
#define PK_SHADOW 0         // experiment (b200env.cu): twice the warps, the second half running store-less copies of the first
#endif
#define EPW 4     // envs per warp
#define BALL_SLOT 7   // the ball of env g is carried by lane (g, BALL_SLOT) in registers
#define SLOTS 8   // lanes per env
#define PK_LANES_PER_ENV SLOTS
// Record layout (element offsets).  Records are 16-byte aligned (REC % 4 == 0, ENV_STRIDE % 4 == 0) and the fields that are
// read / written together form runs that start on 4-float boundaries, so that a run moves with LDS.128 / STS.128 instead of one
// 32-bit access per float (ncu r1g: 21 M of the 97 M warp instructions of a launch were scalar LDS / STS).  Body b lives in
// record B.t.rix[b] = its rank in breadth-first order: the bodies of one tree depth are handled by neighbouring lanes at the
// same time, and consecutive records are 17 float4 apart -> 8 different bank groups for the 8 lanes of a quarter-warp phase
// (the SMPL numbering itself puts siblings 4 bodies apart = the same bank group).
// 68 floats hold everything the substep has live at once (71 at peak, minus the PD target, which a lane keeps in registers
// through the control step - pk_pd_take - and no padding): 32 envs of records fit next to the constant block, so one CTA of
// 8 warps carries 32 envs per SM.
enum {
  R_Q = 0, R_P = 4, R_W = 7, R_V = 10, R_WT = 13,          // [0,16)  world pose / velocity of the body origin, joint velocity
  R_QJ = 16,                                               // [16,20) joint rotation
  R_R = 20, R_ZETA = 23, R_U = 29,                         // [20,32) p - p_parent, velocity-product terms, joint-space bias
  R_A = 32, R_BM = 38, R_C = 47, R_BN = 53, R_BF = 56,     // [32,59) articulated inertia + bias (27 contiguous)
  R_CFX = 59,                                              // contact force x
  R_E = 60,                                                // [60,66) E_w, then D^-1
  R_CFY = 66, R_CFZ = 67, REC = 68
};
#define R_AB 27    // length of the run A[6] Bm[9] C[6] bn[3] bf[3] at R_A
#define R_PD R_U   // between control steps a body's PD target is parked in its U slot (dead there; pk_pd_take / pk_pd_park)
#define R_ACC 52   // (alpha, a) of the body after the backward pass: aliases C[5], bn, bf[0..1] (dead by then); v4 + v2
#define B200_MAX_BODIES_PK 25
#define ENV_EXT (B200_MAX_BODIES_PK * REC)  // per-env extras: extF[3] extT[3] reactF[3] reactX[3]
#define ENV_STRIDE (ENV_EXT + 12)
#define RIX(B, b) ((B).t.rix[b])

// run of N record elements starting at the compile-time offset OFF of a 16-byte aligned record: float -> widest aligned accesses
template <int OFF, int N, int K> __device__ __forceinline__ void ldr_f(const float* rec, float* r) {
  if constexpr (K < N) {
    if constexpr ((OFF + K) % 4 == 0 && N - K >= 4) {
      const float4 v = *reinterpret_cast<const float4*>(rec + OFF + K);
      r[K] = v.x; r[K + 1] = v.y; r[K + 2] = v.z; r[K + 3] = v.w;
      ldr_f<OFF, N, K + 4>(rec, r);
    } else if constexpr ((OFF + K) % 2 == 0 && N - K >= 2) {
      const float2 v = *reinterpret_cast<const float2*>(rec + OFF + K);
      r[K] = v.x; r[K + 1] = v.y;
      ldr_f<OFF, N, K + 2>(rec, r);
    } else {
      r[K] = rec[OFF + K];
      ldr_f<OFF, N, K + 1>(rec, r);
    }
  }
}
template <int OFF, int N, int K> __device__ __forceinline__ void str_f(float* rec, const float* r) {
  if constexpr (K < N) {
    if constexpr ((OFF + K) % 4 == 0 && N - K >= 4) {
      *reinterpret_cast<float4*>(rec + OFF + K) = make_float4(r[K], r[K + 1], r[K + 2], r[K + 3]);
      str_f<OFF, N, K + 4>(rec, r);
    } else if constexpr ((OFF + K) % 2 == 0 && N - K >= 2) {
      *reinterpret_cast<float2*>(rec + OFF + K) = make_float2(r[K], r[K + 1]);
      str_f<OFF, N, K + 2>(rec, r);
    } else {
      rec[OFF + K] = r[K];
      str_f<OFF, N, K + 1>(rec, r);
    }
  }
}
template <int OFF, int N> __device__ __forceinline__ void ldr(const float* rec, float* r) { ldr_f<OFF, N, 0>(rec, r); }
#if defined(PK_SHADOW) && PK_SHADOW && defined(__CUDA_ARCH__)
#define PK_IS_SHADOW ((int)threadIdx.x >= (int)blockDim.x / 2)
#else
#define PK_IS_SHADOW false
#endif
template <int OFF, int N> __device__ __forceinline__ void str(float* rec, const float* r) { if (PK_IS_SHADOW) return; str_f<OFF, N, 0>(rec, r); }
template <int OFF, int N> __device__ __forceinline__ void ldr(const double* rec, double* r) {
#pragma unroll
  for (int k = 0; k < N; k++) r[k] = rec[OFF + k];
}
template <int OFF, int N> __device__ __forceinline__ void str(double* rec, const double* r) {
#pragma unroll
  for (int k = 0; k < N; k++) rec[OFF + k] = r[k];
}

// PD targets.  pk_store_state parks a body's target in the U slot of its record (R_PD), which the substep does not use between
// control steps.  At the start of a control step each lane takes the targets of the bodies it runs in the body pass
// (b = rr * LPE + s) into registers, pd[rr % 3]: with LPE = 8 and at most 25 bodies, rr = 3 only occurs for b = 24 on slot 0, whose
// rr = 0 body is the root (no target).  At the end it parks them again (U is dead once the last forward pass has read it), so that
// the records hold them for the next control step of a multi-step launch.
#define PK_PD_SLOTS 3
static_assert(B200_MAX_BODIES_PK <= PK_PD_SLOTS * SLOTS + 1, "pd[rr % 3] needs at most 3 body-pass rounds per lane besides the root");
// the target of the body of round rr (selects, not an indexed access: pd stays in registers)
template <typename T> __device__ __forceinline__ void pk_pd_pick(const T (&pd)[PK_PD_SLOTS][3], int rr, T* out) {
#pragma unroll
  for (int k = 0; k < 3; k++) out[k] = rr == 1 ? pd[1][k] : (rr == 2 ? pd[2][k] : pd[0][k]);
}
template <typename T, int LPE = SLOTS>
__device__ __forceinline__ void pk_pd_take(const DevBlob& B, const T* env, int s, bool valid, T (&pd)[PK_PD_SLOTS][3]) {
  const b200_model_t& M = B.m;
#pragma unroll
  for (int i = 0; i < PK_PD_SLOTS; i++) pd[i][0] = pd[i][1] = pd[i][2] = T(0);
  for (int rr = 0; rr * LPE < M.nb; rr++) {
    const int b = rr * LPE + s;
    if (!valid || b == 0 || b >= M.nb || M.fixed[b]) continue;
    T t[3];
    ldr<R_PD, 3>(env + RIX(B, b) * REC, t);
#pragma unroll
    for (int k = 0; k < 3; k++) {
      if (rr == 1) pd[1][k] = t[k];
      else if (rr == 2) pd[2][k] = t[k];
      else pd[0][k] = t[k];
    }
  }
}
template <typename T, int LPE = SLOTS>
__device__ __forceinline__ void pk_pd_park(const DevBlob& B, T* env, int s, bool valid, const T (&pd)[PK_PD_SLOTS][3]) {
  const b200_model_t& M = B.m;
  for (int rr = 0; rr * LPE < M.nb; rr++) {
    const int b = rr * LPE + s;
    if (!valid || b == 0 || b >= M.nb || M.fixed[b]) continue;
    T t[3];
    pk_pd_pick<T>(pd, rr, t);
    str<R_PD, 3>(env + RIX(B, b) * REC, t);
  }
}

// kinematics of one body from its parent's record.  JOINT_IN_REGS: the caller (forward pass) just produced the body's joint
// rotation / velocity and hands them over in registers (they are already in the record, this only saves the reload).
// B: the topology (tree tables, parent, fixed); MN: the model whose numeric constants (here the joint offset) the body uses - B.m
// itself, or in a batch of mixed assets (step_kernel_packed<true, false, true>) the env's own asset.
template <typename T, bool WITH_ZETA, bool JOINT_IN_REGS = false>
__device__ __forceinline__ void pk_fk(const DevBlob& B, const b200_model_t& MN, T* env, int b, const T* qj_in = nullptr, const T* wt_in = nullptr) {
  const b200_model_t& M = B.m;
  T* rec = env + RIX(B, b) * REC;
  const T* par = env + RIX(B, M.parent[b]) * REC;
  T ps[13];  // parent Q[4] p[3] w[3] v[3]
  ldr<R_Q, 13>(par, ps);
  const T *pQ = ps, *pp = ps + 4, *pw = ps + 7, *pv = ps + 10;
  T off[3] = {T(MN.offset[b][0]), T(MN.offset[b][1]), T(MN.offset[b][2])}, rr[3], wxr[3];
  T o[16];   // own Q[4] p[3] w[3] v[3] wt[3]
  qrot(pQ, off, rr);
  cross3(pw, rr, wxr);
#pragma unroll
  for (int k = 0; k < 3; k++) { o[4 + k] = pp[k] + rr[k]; o[10 + k] = pv[k] + wxr[k]; }
  if (M.fixed[b]) {
#pragma unroll
    for (int k = 0; k < 4; k++) o[k] = pQ[k];
#pragma unroll
    for (int k = 0; k < 3; k++) o[7 + k] = pw[k];
    str<R_Q, 13>(rec, o);
    if (WITH_ZETA) str<R_R, 3>(rec, rr);
  } else {
    T qj[4], wt[3], wj[3];
    if (JOINT_IN_REGS) {
#pragma unroll
      for (int k = 0; k < 4; k++) qj[k] = qj_in[k];
#pragma unroll
      for (int k = 0; k < 3; k++) wt[k] = wt_in[k];
    } else {
      T t4[4];
      ldr<R_QJ, 4>(rec, qj);
      ldr<12, 4>(rec, t4);   // v[2] | wt[3]
      wt[0] = t4[1]; wt[1] = t4[2]; wt[2] = t4[3];
    }
    qmul(pQ, qj, o);
    qnormalize(o);
    qrot(o, wt, wj);
#pragma unroll
    for (int k = 0; k < 3; k++) { o[7 + k] = pw[k] + wj[k]; o[13 + k] = wt[k]; }
    str<R_Q, 16>(rec, o);
    if (WITH_ZETA) {
      T rz[9];
      rz[0] = rr[0]; rz[1] = rr[1]; rz[2] = rr[2];
      cross3(pw, wj, rz + 3); cross3(pw, wxr, rz + 6);
      str<R_R, 9>(rec, rz);
    }
  }
}
template <typename T, bool WITH_ZETA, bool JOINT_IN_REGS = false>
__device__ __forceinline__ void pk_fk(const DevBlob& B, T* env, int b, const T* qj_in = nullptr, const T* wt_in = nullptr) {
  pk_fk<T, WITH_ZETA, JOINT_IN_REGS>(B, B.m, env, b, qj_in, wt_in);
}

// rigid-body inertia + bias + external / contact / joint-drive terms of one dynamic body -> record
// DEFER_CONTACT (PK_CONTACT_COMPACT): only the penetration mask of the hull is computed here and left in the record (in the two
// slots of the contact force y/z - bit patterns, 0 = no contact = a zero force); pk_contact_phase adds the vertices afterwards.
template <typename T> __device__ __forceinline__ T pk_bits_to_slot(uint32_t x);
template <> __device__ __forceinline__ float pk_bits_to_slot<float>(uint32_t x) { float f; memcpy(&f, &x, 4); return f; }
template <> __device__ __forceinline__ double pk_bits_to_slot<double>(uint32_t x) { return (double)x; }
__device__ __forceinline__ uint32_t pk_slot_to_bits(float f) { uint32_t x; memcpy(&x, &f, 4); return x; }
__device__ __forceinline__ uint32_t pk_slot_to_bits(double d) { return (uint32_t)d; }

// pd: the body's PD target (from the lane's registers, pk_pd_pick).  MN / verts: the numeric constants and hull vertices of the
// body's model (see pk_fk); B: the topology.
template <typename T, bool DEFER_CONTACT = false>
__device__ __forceinline__ void pk_body(const DevBlob& B, const b200_model_t& MN, const float* __restrict__ verts, const PhysCfg<T>& c, T* env,
                                        int b, bool ext_on, const T* pd) {
  const b200_model_t& M = B.m;
  T* rec = env + RIX(B, b) * REC;
  T own[16], R[9];   // Q[4] p[3] w[3] v[3] wt[3]
  ldr<R_Q, 16>(rec, own);
  const T *Q = own, *p = own + 4, *w = own + 7, *v = own + 10;
  qmat(Q, R);
  T ab[R_AB];        // A[6] Bm[9] C[6] bn[3] bf[3]: one run of the record
  T *A = ab, *Bm = ab + 6, *C = ab + 15, *bn = ab + 21, *bf = ab + 24, cf[3] = {0, 0, 0};
#pragma unroll
  for (int k = 6; k < 21; k++) ab[k] = T(0);
  const T ms = T(MN.mass[b]);
  T cl[3] = {T(MN.com[b][0]), T(MN.com[b][1]), T(MN.com[b][2])}, cw[3];
  mv3(R, cl, cw);
  {
    T Ib[6], F[9], RF[9];
#pragma unroll
    for (int k = 0; k < 6; k++) Ib[k] = T(MN.inertia[b][k]);
    sym_full(Ib, F);
#pragma unroll
    for (int i = 0; i < 3; i++)
#pragma unroll
      for (int j = 0; j < 3; j++) RF[i * 3 + j] = R[i * 3] * F[j] + R[i * 3 + 1] * F[3 + j] + R[i * 3 + 2] * F[6 + j];
    const T c2 = cw[0] * cw[0] + cw[1] * cw[1] + cw[2] * cw[2];
    A[0] = RF[0] * R[0] + RF[1] * R[1] + RF[2] * R[2] + ms * (c2 - cw[0] * cw[0]);
    A[1] = RF[3] * R[3] + RF[4] * R[4] + RF[5] * R[5] + ms * (c2 - cw[1] * cw[1]);
    A[2] = RF[6] * R[6] + RF[7] * R[7] + RF[8] * R[8] + ms * (c2 - cw[2] * cw[2]);
    A[3] = RF[0] * R[3] + RF[1] * R[4] + RF[2] * R[5] - ms * cw[0] * cw[1];
    A[4] = RF[0] * R[6] + RF[1] * R[7] + RF[2] * R[8] - ms * cw[0] * cw[2];
    A[5] = RF[3] * R[6] + RF[4] * R[7] + RF[5] * R[8] - ms * cw[1] * cw[2];
  }
  Bm[1] = -ms * cw[2]; Bm[2] = ms * cw[1];
  Bm[3] = ms * cw[2]; Bm[5] = -ms * cw[0];
  Bm[6] = -ms * cw[1]; Bm[7] = ms * cw[0];
  C[0] = C[1] = C[2] = ms;
  {
    T Iw[3], t1[3], t2[3];
    sym_mv(A, w, Iw);
    cross3(w, Iw, bn);
    cross3(w, cw, t1);
    cross3(w, t1, t2);
    bn[0] -= ms * cw[1] * c.gz;
    bn[1] += ms * cw[0] * c.gz;
    bf[0] = ms * t2[0]; bf[1] = ms * t2[1]; bf[2] = ms * t2[2] - ms * c.gz;
  }
  const T* ext = env + ENV_EXT;
  if (c.has_ball && c.racket_body >= 0 && b == M.parent[c.racket_body]) {  // reaction of the last racket impact on the wrist
    T rF[3] = {ext[6], ext[7], ext[8]}, dx[3] = {ext[9] - p[0], ext[10] - p[1], ext[11] - p[2]}, t[3];
    cross3(dx, rF, t);
#pragma unroll
    for (int k = 0; k < 3; k++) { bn[k] -= t[k]; bf[k] -= rF[k]; }
  }
  if (b == 0 && ext_on) {
    T eF[3] = {ext[0], ext[1], ext[2]}, cxF[3];
    cross3(cw, eF, cxF);
#pragma unroll
    for (int k = 0; k < 3; k++) { bn[k] -= ext[3 + k] + cxF[k]; bf[k] -= eF[k]; }
  }
  const int nv = ABL == 6 ? 0 : MN.nverts[b];
  if (DEFER_CONTACT) {
    unsigned long long mask = 0ull;
    if (nv > 0 && p[2] - T(MN.radius[b]) < T(0)) mask = contact_mask<T>(verts + (size_t)b * MN.vmax * 3, MN.vmax, nv, R, p);
    cf[1] = pk_bits_to_slot<T>((uint32_t)mask);
    cf[2] = pk_bits_to_slot<T>((uint32_t)(mask >> 32));
  } else if (nv > 0 && p[2] - T(MN.radius[b]) < T(0)) {
    contact_hull<T>(verts + (size_t)b * MN.vmax * 3, MN.vmax, nv, c, R, p, v, w, A, Bm, C, bn, bf, cf);
  }
  str<R_A, R_AB>(rec, ab);
  if (!PK_IS_SHADOW) rec[R_CFX] = cf[0];
  str<R_CFY, 2>(rec, cf + 1);
  if (b > 0) {
    const int d0 = M.dof_of_body[b];
    T qj[4], q[3], tau[3], e[3], u[3], E[6];
    ldr<R_QJ, 4>(rec, qj);
    const T* wt = own + 13;
    qlog(qj, q);
#pragma unroll
    for (int k = 0; k < 3; k++) {
      T kp = T(MN.kp[d0 + k]), kd = T(MN.kd[d0 + k]);
      e[k] = T(MN.armature[d0 + k]) + c.h * kd + c.h * c.h * kp;
      tau[k] = kp * (pd[k] - q[k] - c.h * wt[k]) - kd * wt[k];
      T lo = T(MN.lim_lo[d0 + k]), hi = T(MN.lim_hi[d0 + k]);
      if (q[k] < lo) { tau[k] += c.limk * (lo - q[k] - c.h * wt[k]) - c.limc * wt[k]; e[k] += c.h * c.limc + c.h * c.h * c.limk; }
      else if (q[k] > hi) { tau[k] += c.limk * (hi - q[k] - c.h * wt[k]) - c.limc * wt[k]; e[k] += c.h * c.limc + c.h * c.h * c.limk; }
    }
    mv3(R, tau, u);
    E[0] = R[0] * R[0] * e[0] + R[1] * R[1] * e[1] + R[2] * R[2] * e[2];
    E[1] = R[3] * R[3] * e[0] + R[4] * R[4] * e[1] + R[5] * R[5] * e[2];
    E[2] = R[6] * R[6] * e[0] + R[7] * R[7] * e[1] + R[8] * R[8] * e[2];
    E[3] = R[0] * R[3] * e[0] + R[1] * R[4] * e[1] + R[2] * R[5] * e[2];
    E[4] = R[0] * R[6] * e[0] + R[1] * R[7] * e[1] + R[2] * R[8] * e[2];
    E[5] = R[3] * R[6] * e[0] + R[4] * R[7] * e[1] + R[5] * R[8] * e[2];
    str<R_E, 6>(rec, E); str<R_U, 3>(rec, u);
  }
}
template <typename T, bool DEFER_CONTACT = false>
__device__ __forceinline__ void pk_body(const DevBlob& B, const float* __restrict__ verts, const PhysCfg<T>& c, T* env, int b, bool ext_on,
                                        const T* pd) {
  pk_body<T, DEFER_CONTACT>(B, B.m, verts, c, env, b, ext_on, pd);
}

// backward step of one dynamic non-root body: D^-1, u, articulated inertia/bias shifted to the parent origin -> out[27]
template <typename T>
__device__ __forceinline__ void pk_backward(const DevBlob& B, T* env, int b, T* out) {
  T* rec = env + RIX(B, b) * REC;
  T ab[R_AB], rzu[12], E[6];   // A[6] Bm[9] C[6] bn[3] bf[3] | r[3] zeta[6] u[3]
  ldr<R_A, R_AB>(rec, ab); ldr<R_R, 12>(rec, rzu); ldr<R_E, 6>(rec, E);
  const T *A = ab, *Bm = ab + 6, *C = ab + 15, *bn = ab + 21, *bf = ab + 24, *r = rzu, *zeta = rzu + 3;
  T u[3] = {rzu[9], rzu[10], rzu[11]};
  T D[6], Dinv[6];
#pragma unroll
  for (int k = 0; k < 6; k++) D[k] = A[k] + E[k];
  sym_inv(D, Dinv);
  u[0] -= bn[0]; u[1] -= bn[1]; u[2] -= bn[2];
  str<R_E, 6>(rec, Dinv); str<R_U, 3>(rec, u);
  T Af[9], Df[9];
  sym_full(A, Af);
  sym_full(Dinv, Df);
  T G[9], K[9];
#pragma unroll
  for (int i = 0; i < 3; i++)
#pragma unroll
    for (int j = 0; j < 3; j++) {
      G[i * 3 + j] = Df[i * 3] * Af[j] + Df[i * 3 + 1] * Af[3 + j] + Df[i * 3 + 2] * Af[6 + j];
      K[i * 3 + j] = Df[i * 3] * Bm[j] + Df[i * 3 + 1] * Bm[3 + j] + Df[i * 3 + 2] * Bm[6 + j];
    }
  T aA[6], aB[9], aC[6];
  aA[0] = A[0] - (Af[0] * G[0] + Af[1] * G[3] + Af[2] * G[6]);
  aA[1] = A[1] - (Af[3] * G[1] + Af[4] * G[4] + Af[5] * G[7]);
  aA[2] = A[2] - (Af[6] * G[2] + Af[7] * G[5] + Af[8] * G[8]);
  aA[3] = A[3] - (Af[0] * G[1] + Af[1] * G[4] + Af[2] * G[7]);
  aA[4] = A[4] - (Af[0] * G[2] + Af[1] * G[5] + Af[2] * G[8]);
  aA[5] = A[5] - (Af[3] * G[2] + Af[4] * G[5] + Af[5] * G[8]);
#pragma unroll
  for (int i = 0; i < 3; i++)
#pragma unroll
    for (int j = 0; j < 3; j++) aB[i * 3 + j] = Bm[i * 3 + j] - (Af[i * 3] * K[j] + Af[i * 3 + 1] * K[3 + j] + Af[i * 3 + 2] * K[6 + j]);
  aC[0] = C[0] - (Bm[0] * K[0] + Bm[3] * K[3] + Bm[6] * K[6]);
  aC[1] = C[1] - (Bm[1] * K[1] + Bm[4] * K[4] + Bm[7] * K[7]);
  aC[2] = C[2] - (Bm[2] * K[2] + Bm[5] * K[5] + Bm[8] * K[8]);
  aC[3] = C[3] - (Bm[0] * K[1] + Bm[3] * K[4] + Bm[6] * K[7]);
  aC[4] = C[4] - (Bm[0] * K[2] + Bm[3] * K[5] + Bm[6] * K[8]);
  aC[5] = C[5] - (Bm[1] * K[2] + Bm[4] * K[5] + Bm[7] * K[8]);
  T s[3], an[3], af[3], t1[3], t2[3], As[3], Bts[3];
  sym_mv(Dinv, u, s);
  sym_mv(aA, zeta, t1);
  mv3(aB, zeta + 3, t2);
  sym_mv(A, s, As);
#pragma unroll
  for (int k = 0; k < 3; k++) an[k] = bn[k] + t1[k] + t2[k] + As[k];
  mtv3(aB, zeta, t1);
  sym_mv(aC, zeta + 3, t2);
  mtv3(Bm, s, Bts);
#pragma unroll
  for (int k = 0; k < 3; k++) af[k] = bf[k] + t1[k] + t2[k] + Bts[k];
  T Cf[9], Bp[9];
  sym_full(aC, Cf);
#pragma unroll
  for (int j = 0; j < 3; j++) {
    T col[3] = {Cf[j], Cf[3 + j], Cf[6 + j]}, x[3];
    cross3(r, col, x);
    Bp[j] = aB[j] + x[0]; Bp[3 + j] = aB[3 + j] + x[1]; Bp[6 + j] = aB[6 + j] + x[2];
  }
  T P1[9], P2[9];
#pragma unroll
  for (int j = 0; j < 3; j++) {
    T x[3];
    cross3(r, Bp + 3 * j, x);
    P1[j] = x[0]; P1[3 + j] = x[1]; P1[6 + j] = x[2];
    cross3(r, aB + 3 * j, x);
    P2[j] = x[0]; P2[3 + j] = x[1]; P2[6 + j] = x[2];
  }
  out[0] = aA[0] + P1[0] + P2[0];
  out[1] = aA[1] + P1[4] + P2[4];
  out[2] = aA[2] + P1[8] + P2[8];
  out[3] = aA[3] + P1[1] + P2[3];
  out[4] = aA[4] + P1[2] + P2[6];
  out[5] = aA[5] + P1[5] + P2[7];
#pragma unroll
  for (int k = 0; k < 9; k++) out[6 + k] = Bp[k];
#pragma unroll
  for (int k = 0; k < 6; k++) out[15 + k] = aC[k];
  T rxf[3];
  cross3(r, af, rxf);
#pragma unroll
  for (int k = 0; k < 3; k++) { out[21 + k] = an[k] + rxf[k]; out[24 + k] = af[k]; }
}

template <typename T> __device__ __forceinline__ void pk_root(const PhysCfg<T>& c, T* env) {
  T* rec = env;   // the root is record 0
  T ab[R_AB], acc[6];
  ldr<R_A, R_AB>(rec, ab);
  const T *A = ab, *Bm = ab + 6, *C = ab + 15, *bn = ab + 21, *bf = ab + 24;
  T Ci[6], Cif[9], BC[9], S[6], Si[6], rhs[3], t[3];
  sym_inv(C, Ci);
  sym_full(Ci, Cif);
#pragma unroll
  for (int i = 0; i < 3; i++)
#pragma unroll
    for (int j = 0; j < 3; j++) BC[i * 3 + j] = Bm[i * 3] * Cif[j] + Bm[i * 3 + 1] * Cif[3 + j] + Bm[i * 3 + 2] * Cif[6 + j];
  S[0] = A[0] - (BC[0] * Bm[0] + BC[1] * Bm[1] + BC[2] * Bm[2]);
  S[1] = A[1] - (BC[3] * Bm[3] + BC[4] * Bm[4] + BC[5] * Bm[5]);
  S[2] = A[2] - (BC[6] * Bm[6] + BC[7] * Bm[7] + BC[8] * Bm[8]);
  S[3] = A[3] - (BC[0] * Bm[3] + BC[1] * Bm[4] + BC[2] * Bm[5]);
  S[4] = A[4] - (BC[0] * Bm[6] + BC[1] * Bm[7] + BC[2] * Bm[8]);
  S[5] = A[5] - (BC[3] * Bm[6] + BC[4] * Bm[7] + BC[5] * Bm[8]);
  sym_inv(S, Si);
  mv3(BC, bf, t);
#pragma unroll
  for (int k = 0; k < 3; k++) rhs[k] = -bn[k] + t[k];
  sym_mv(Si, rhs, acc);
  mtv3(Bm, acc, t);
#pragma unroll
  for (int k = 0; k < 3; k++) t[k] = -bf[k] - t[k];
  sym_mv(Ci, t, acc + 3);
  str<R_ACC, 6>(rec, acc);
}

// forward step of one dynamic non-root body: accelerations, integrate the joint state; the new joint rotation / velocity are also
// returned in registers for the kinematics that follow at once (pk_fk<.., JOINT_IN_REGS>).
// SENSOR && stash (last substep of a control step with the DOF force sensor): the joint's exp-map coordinates q at the start of the
// substep and the implicit drive's velocity qd + h qdd (before damping and the clamp) go into the body's E slot, dead once D^-1 has
// been read here, for pk_dof_force.
template <typename T, bool SENSOR = false>
__device__ __forceinline__ void pk_forward(const DevBlob& B, const PhysCfg<T>& c, T* env, int b, T* qn, T* wt, bool stash = false) {
  const b200_model_t& M = B.m;
  T* rec = env + RIX(B, b) * REC;
  const T* par = env + RIX(B, M.parent[b]) * REC;
  T pa[6], abm[16], Dinv[6], rzu[12], Q[4], vw[4], qj[4];   // abm: A[6] Bm[9] (C[0]);  rzu: r[3] zeta[6] u[3];  vw: v[2] wt[3]
  ldr<R_ACC, 6>(par, pa);
  ldr<R_A, 16>(rec, abm); ldr<R_E, 6>(rec, Dinv); ldr<R_R, 12>(rec, rzu);
  ldr<R_Q, 4>(rec, Q); ldr<12, 4>(rec, vw); ldr<R_QJ, 4>(rec, qj);
  const T *A = abm, *Bm = abm + 6, *r = rzu, *zeta = rzu + 3, *u = rzu + 9;
  wt[0] = vw[1]; wt[1] = vw[2]; wt[2] = vw[3];
  T axr[3], Ap[6], t1[3], t2[3], t[3], gam[3], wd[3], acc[6];
  cross3(pa, r, axr);
#pragma unroll
  for (int k = 0; k < 3; k++) { Ap[k] = pa[k] + zeta[k]; Ap[3 + k] = pa[3 + k] + axr[k] + zeta[3 + k]; }
  sym_mv(A, Ap, t1);
  mv3(Bm, Ap + 3, t2);
#pragma unroll
  for (int k = 0; k < 3; k++) t[k] = u[k] - t1[k] - t2[k];
  sym_mv(Dinv, t, gam);
#pragma unroll
  for (int k = 0; k < 3; k++) { acc[k] = Ap[k] + gam[k]; acc[3 + k] = Ap[3 + k]; }
  str<R_ACC, 6>(rec, acc);
  T cq[4] = {-Q[0], -Q[1], -Q[2], Q[3]};
  qrot(cq, gam, wd);  // R^T gam
  if (SENSOR && stash) {
    T st[6];
    qlog(qj, st);
#pragma unroll
    for (int k = 0; k < 3; k++) st[3 + k] = wt[k] + c.h * wd[k];
    str<R_E, 6>(rec, st);
  }
#pragma unroll
  for (int k = 0; k < 3; k++) wt[k] = (wt[k] + c.h * wd[k]) * c.damp;
  T n2 = wt[0] * wt[0] + wt[1] * wt[1] + wt[2] * wt[2];
  if (n2 > c.wmax * c.wmax) { T sc = c.wmax * rsqrt_(n2); wt[0] *= sc; wt[1] *= sc; wt[2] *= sc; }
  T hv[3] = {c.h * wt[0], c.h * wt[1], c.h * wt[2]}, dq[4];
  qexp_small(hv, dq);
  qmul(qj, dq, qn);
  qnormalize(qn);
  vw[1] = wt[0]; vw[2] = wt[1]; vw[3] = wt[2];
  str<12, 4>(rec, vw); str<R_QJ, 4>(rec, qn);
}

template <typename T> __device__ __forceinline__ void pk_root_integrate(const PhysCfg<T>& c, T* env) {
  T* rec = env;
  T acc[6], o[13];   // Q[4] p[3] w[3] v[3]
  ldr<R_ACC, 6>(rec, acc); ldr<R_Q, 13>(rec, o);
  T *Q = o, *p = o + 4, *w = o + 7, *v = o + 10;
#pragma unroll
  for (int k = 0; k < 3; k++) { w[k] = (w[k] + c.h * acc[k]) * c.damp; v[k] += c.h * acc[3 + k]; }
  T n2 = w[0] * w[0] + w[1] * w[1] + w[2] * w[2];
  if (n2 > c.wmax * c.wmax) { T sc = c.wmax * rsqrt_(n2); w[0] *= sc; w[1] *= sc; w[2] *= sc; }
  T hv[3] = {c.h * w[0], c.h * w[1], c.h * w[2]}, dq[4], qn[4];
#pragma unroll
  for (int k = 0; k < 3; k++) p[k] += c.h * v[k];
  qexp_small(hv, dq);
  qmul(dq, Q, qn);
  qnormalize(qn);
#pragma unroll
  for (int k = 0; k < 4; k++) Q[k] = qn[k];
  str<R_Q, 13>(rec, o);
}

// PK_CONTACT_COMPACT: the per-vertex part of the ground contact as its own phase.  In the body pass a lane's bodies sit in three
// rounds and every round costs the warp as many vertex iterations as its busiest lane (tools/contact_imbalance.py: 32 serial
// iterations per substep with 7 % of the lanes busy for fallen humanoids, on 2.8 bodies in contact per env).  Here the bodies whose
// penetration mask is non-zero are compacted per env group (ballot + n-th set bit) and handed to the 8 lanes of the group: all
// bodies in contact of an env go in ONE round (two if there are more than 8).  Each body is still summed by one lane in ascending
// vertex order onto the values the body pass stored, so every result is bit-identical to the in-place form.
__device__ __forceinline__ int pk_nth_set_bit(uint32_t w, int n) {   // position of the n-th (0-based) set bit of w; w has more than n bits set
#if defined(__CUDA_ARCH__)
  return __fns(w, 0, n + 1);
#else
  for (int k = 0; k < 32; k++) if ((w >> k) & 1u) { if (n == 0) return k; n--; }
  return -1;
#endif
}
template <typename T>
__device__ __forceinline__ void pk_contact_phase(const DevBlob& B, const b200_model_t& MN, const float* __restrict__ verts, const PhysCfg<T>& c, T* env,
                                                 int lane, bool valid) {
  const b200_model_t& M = B.m;
  const int g = lane >> 3, s = lane & 7, nb = M.nb;
  // which of my bodies (rounds 0..2 of the body pass) have penetrating vertices
  uint32_t word = 0;   // bit rr*8 + slot over the 8 lanes of my env group
  for (int rr = 0; rr * SLOTS < nb; rr++) {
    const int b = rr * SLOTS + s;
    bool hit = false;
    if (valid && b < nb && !M.fixed[b]) {
      const T* rec = env + RIX(B, b) * REC;
      hit = (pk_slot_to_bits(rec[R_CFY]) | pk_slot_to_bits(rec[R_CFZ])) != 0u;
    }
    const uint32_t bal = __ballot_sync(FULL, hit);
    word |= ((bal >> (g * 8)) & 0xFFu) << (rr * 8);
  }
  int n = 0;
  for (uint32_t w = word; w; w &= w - 1) n++;
  for (int t0 = 0; __any_sync(FULL, t0 < n); t0 += 8) {
    const int idx = t0 + s;
    if (idx < n) {
      const int b = pk_nth_set_bit(word, idx);        // = rr*8 + slot = the body index
      T* rec = env + RIX(B, b) * REC;
      T own[13], R[9], ab[R_AB], cf[3];
      ldr<R_Q, 13>(rec, own);
      ldr<R_A, R_AB>(rec, ab);
      const unsigned long long mask = (unsigned long long)pk_slot_to_bits(rec[R_CFY]) | ((unsigned long long)pk_slot_to_bits(rec[R_CFZ]) << 32);
      cf[0] = rec[R_CFX]; cf[1] = T(0); cf[2] = T(0);
      qmat(own, R);
      contact_apply<T>(verts + (size_t)b * MN.vmax * 3, MN.vmax, mask, c, R, own + 4, own + 10, own + 7, ab, ab + 6, ab + 15, ab + 21, ab + 24, cf);
      str<R_A, R_AB>(rec, ab);
      if (!PK_IS_SHADOW) rec[R_CFX] = cf[0];
      str<R_CFY, 2>(rec, cf + 1);
    }
  }
}

// Optional contacts of the ball with the humanoid's bodies and the racket handle (b200_cfg_t::ball_body_contact; float64 restatement:
// oracle/physics_ref.c::ball_contacts_extra_ref).  Runs on the ball's lane right after ball_substep, against the poses / velocities the
// bodies had at the start of the substep (what the records hold at that point, like the string-bed test).  A body's hull = spheres of
// radius vrho[b] on its vertices, the handle = a capsule; the DEEPEST contact of the substep gets the impulse and the ball is moved out
// of it.  The obstacle is kinematic: no reaction on the humanoid (57 g ball).
template <typename T>
__device__ __forceinline__ void pk_ball_contacts_extra(const DevBlob& B, const float* verts, const PhysCfg<T>& c, const T* env, Ball<T>& ball) {
  const b200_model_t& M = B.m;
  {
    T rp[3];
    ldr<R_P, 3>(env, rp);   // the root is record 0
    const T dx = ball.p[0] - rp[0], dy = ball.p[1] - rp[1], dz = ball.p[2] - rp[2];
    if (dx * dx + dy * dy + dz * dz > T(2.25)) return;   // nothing of the player within 1.5 m of the pelvis
  }
  T best = T(0), bn[3] = {T(0), T(0), T(1)}, bvo[3] = {T(0), T(0), T(0)}, be = c.eb, bmu = c.mub;
  for (int b = 0; b < M.nb; b++) {
    const bool handle = b == c.racket_body && c.hdl[6] > T(0);
    const int nv = M.nverts[b];
    if (nv == 0 && !handle) continue;
    T s[13];   // Q[4] p[3] w[3] v[3]
    ldr<R_Q, 13>(env + RIX(B, b) * REC, s);
    const T *Q = s, *p = s + 4, *w = s + 7, *v = s + 10;
    const T d[3] = {ball.p[0] - p[0], ball.p[1] - p[1], ball.p[2] - p[2]};
    const T d2 = d[0] * d[0] + d[1] * d[1] + d[2] * d[2];
    const int nt = handle ? 0 : B.t.ntris[b];
    const T reach = handle ? T(0.6) : T(M.radius[b]) + (nt > 0 ? T(0) : T(B.t.vrho[b])) + c.bR;
    if (d2 > reach * reach) continue;
    const T cq[4] = {-Q[0], -Q[1], -Q[2], Q[3]};
    T dl[3], pen = T(0), nl[3] = {T(0), T(0), T(1)};
    qrot(cq, d, dl);   // ball centre in the body frame
    if (nt > 0) {
      if (!hull_sphere<T>(verts + (size_t)b * M.vmax * 3, M.vmax, B.t.face_planes + (size_t)b * B.t.face_tmax * 4,
                          B.t.face_tris + (size_t)b * B.t.face_tmax * 4, nt, dl, c.bR, pen, nl))
        continue;
    } else {
      T el[3] = {T(0), T(0), T(0)}, dist = T(0), rad = T(0);
      if (handle) {
        const T a[3] = {c.hdl[3] - c.hdl[0], c.hdl[4] - c.hdl[1], c.hdl[5] - c.hdl[2]};
        const T q0[3] = {dl[0] - c.hdl[0], dl[1] - c.hdl[1], dl[2] - c.hdl[2]};
        T t = (q0[0] * a[0] + q0[1] * a[1] + q0[2] * a[2]) * rcp_(a[0] * a[0] + a[1] * a[1] + a[2] * a[2]);
        t = t < T(0) ? T(0) : (t > T(1) ? T(1) : t);
#pragma unroll
        for (int k = 0; k < 3; k++) el[k] = q0[k] - t * a[k];
        dist = sqrt_(el[0] * el[0] + el[1] * el[1] + el[2] * el[2]);
        rad = c.hdl[6];
      } else {
        const float* vb = verts + (size_t)b * M.vmax * 3;
        T m2 = T(1e30);
        for (int k = 0; k < nv; k++) {
          const T ex = dl[0] - T(vb[k]), ey = dl[1] - T(vb[M.vmax + k]), ez = dl[2] - T(vb[2 * M.vmax + k]);
          const T e2 = ex * ex + ey * ey + ez * ez;
          if (e2 < m2) { m2 = e2; el[0] = ex; el[1] = ey; el[2] = ez; }
        }
        dist = sqrt_(m2);
        rad = T(B.t.vrho[b]);
      }
      pen = c.bR + rad - dist;
      if (!(dist > T(1e-9))) continue;
      const T id = rcp_(dist);
      nl[0] = el[0] * id; nl[1] = el[1] * id; nl[2] = el[2] * id;
    }
    if (pen > best) {
      best = pen;
      qrot(Q, nl, bn);
      // velocity of the obstacle at the contact point x = c - R n
      const T x[3] = {d[0] - c.bR * bn[0], d[1] - c.bR * bn[1], d[2] - c.bR * bn[2]};
      T wxx[3];
      cross3(w, x, wxx);
#pragma unroll
      for (int k = 0; k < 3; k++) bvo[k] = v[k] + wxx[k];
      be = handle ? c.er : c.eb;
      bmu = handle ? c.mur : c.mub;
    }
  }
  if (best > T(0)) {
    T J[3];
    ball_impulse(c, ball, bn, bvo, be, bmu, J);
#pragma unroll
    for (int k = 0; k < 3; k++) ball.p[k] += best * bn[k];
  }
}

// The same contacts on the 8 lanes of the env's group.  Every lane of the warp calls this (the exchanges are warp shuffles).  Two stages:
// (1) lane (g, s) pre-tests bodies s, s + 8, s + 16, (24) of env g against the ball its group's lane BALL_SLOT carries (reach test
// against the bounding sphere); the cheap shapes - the racket handle capsule, bodies of a model without hull faces - are finished
// right there; (2) the bodies with a convex hull that passed the reach test are taken one after the other, in ascending body order, by
// the WHOLE group (hull_sphere_coop: the hull's faces over 8 lanes).  The first version walked a hull's ~100 faces twice on one lane,
// one dependent L2 round trip per face, and that one lane decided when a one-wave launch ended.  The
// deepest contact wins (ties: the lower body index, as in the serial loop of the restatement) and the ball's lane applies it.
template <typename T, int RS = REC>   // RS: record stride (packed_t.cuh has its own record layout; the pose run is the same)
__device__ __forceinline__ void pk_ball_contacts_group(const DevBlob& B, const float* verts, const PhysCfg<T>& c, const T* env, int lane, bool valid,
                                                       Ball<T>& ball) {
  const b200_model_t& M = B.m;
  const int g = lane >> 3, s = lane & 7, src = (lane & ~7) | BALL_SLOT;
  T bp[3];
#pragma unroll
  for (int k = 0; k < 3; k++) bp[k] = __shfl_sync(FULL, ball.p[k], src);
  bool near = valid;
  if (near) {
    T rp[3];
    ldr<R_P, 3>(env, rp);   // the root is record 0
    const T dx = bp[0] - rp[0], dy = bp[1] - rp[1], dz = bp[2] - rp[2];
    near = dx * dx + dy * dy + dz * dz <= T(2.25);       // nothing of the player beyond 1.5 m of the pelvis
  }
  if (!__any_sync(FULL, near)) return;                   // no ball of this warp is near its player (warp-uniform)
  T best = T(0), bn[3] = {T(0), T(0), T(1)}, bvo[3] = {T(0), T(0), T(0)}, be = c.eb, bmu = c.mub;
  int bbody = 1 << 20;
  auto take = [&](int b, bool handle, T pen, const T* nl, const T* st, const T* d) {   // contact of depth pen with body b (pose st): keep the deepest
    if (pen > best || (pen == best && b < bbody)) {
      const T *Q = st, *w = st + 7, *v = st + 10;
      best = pen;
      bbody = b;
      qrot(Q, nl, bn);
      const T x[3] = {d[0] - c.bR * bn[0], d[1] - c.bR * bn[1], d[2] - c.bR * bn[2]};   // contact point relative to the body origin
      T wxx[3];
      cross3(w, x, wxx);
#pragma unroll
      for (int k = 0; k < 3; k++) bvo[k] = v[k] + wxx[k];
      be = handle ? c.er : c.eb;
      bmu = handle ? c.mur : c.mub;
    }
  };
  // ---- stage 1: reach tests; cheap shapes finished; hull bodies in reach -> candidate bits of my env
  uint32_t cand = 0;
  for (int rr = 0; rr * SLOTS < M.nb; rr++) {
    const int b = rr * SLOTS + s;
    bool hull = false;
    if (near && b < M.nb) {
      const bool handle = b == c.racket_body && c.hdl[6] > T(0);
      const int nv = M.nverts[b];
      if (nv > 0 || handle) {
        T st[13];   // Q[4] p[3] w[3] v[3]
        ldr<R_Q, 13>(env + RIX(B, b) * RS, st);
        const T *Q = st, *p = st + 4;
        const T d[3] = {bp[0] - p[0], bp[1] - p[1], bp[2] - p[2]};
        const T d2 = d[0] * d[0] + d[1] * d[1] + d[2] * d[2];
        const int nt = handle ? 0 : B.t.ntris[b];          // > 0: exact test against the body's convex hull
        const T reach = handle ? T(0.6) : T(M.radius[b]) + (nt > 0 ? T(0) : T(B.t.vrho[b])) + c.bR;
        if (!(d2 > reach * reach)) {
          if (nt > 0) {      // second reach test: the hull's own bounding sphere (about its centroid; DevTree::bs)
            const T cl[3] = {T(B.t.bs[b][0]), T(B.t.bs[b][1]), T(B.t.bs[b][2])};
            T cw[3];
            qrot(Q, cl, cw);
            const T e[3] = {d[0] - cw[0], d[1] - cw[1], d[2] - cw[2]}, rr2 = T(B.t.bs[b][3]) + c.bR;
            hull = !(e[0] * e[0] + e[1] * e[1] + e[2] * e[2] > rr2 * rr2);
          } else {
            const T cq[4] = {-Q[0], -Q[1], -Q[2], Q[3]};
            T dl[3], el[3] = {T(0), T(0), T(0)}, dist = T(0), rad = T(0);
            qrot(cq, d, dl);   // ball centre in the body frame
            if (handle) {
              const T a[3] = {c.hdl[3] - c.hdl[0], c.hdl[4] - c.hdl[1], c.hdl[5] - c.hdl[2]};
              const T q0[3] = {dl[0] - c.hdl[0], dl[1] - c.hdl[1], dl[2] - c.hdl[2]};
              T t = (q0[0] * a[0] + q0[1] * a[1] + q0[2] * a[2]) * rcp_(a[0] * a[0] + a[1] * a[1] + a[2] * a[2]);
              t = t < T(0) ? T(0) : (t > T(1) ? T(1) : t);
#pragma unroll
              for (int k = 0; k < 3; k++) el[k] = q0[k] - t * a[k];
              dist = sqrt_(el[0] * el[0] + el[1] * el[1] + el[2] * el[2]);
              rad = c.hdl[6];
            } else {         // a model compiled without hull faces: spheres on the hull vertices stand in for the hull
              const float* vb = verts + (size_t)b * M.vmax * 3;
              T m2 = T(1e30);
              for (int k = 0; k < nv; k++) {
                const T ex = dl[0] - T(vb[k]), ey = dl[1] - T(vb[M.vmax + k]), ez = dl[2] - T(vb[2 * M.vmax + k]);
                const T e2 = ex * ex + ey * ey + ez * ez;
                if (e2 < m2) { m2 = e2; el[0] = ex; el[1] = ey; el[2] = ez; }
              }
              dist = sqrt_(m2);
              rad = T(B.t.vrho[b]);
            }
            const T pen = c.bR + rad - dist;
            if (dist > T(1e-9)) {
              const T id = rcp_(dist);
              const T nl[3] = {el[0] * id, el[1] * id, el[2] * id};
              if (pen > T(0)) take(b, handle, pen, nl, st, d);
            }
          }
        }
      }
    }
    cand |= ((__ballot_sync(FULL, hull) >> (g * 8)) & 0xFFu) << (rr * SLOTS);
  }
  // ---- stage 2: the hull bodies in reach, one at a time, the hull's faces over the 8 lanes of the group
  while (__any_sync(FULL, cand != 0u)) {
    const bool act = cand != 0u;
    int b = 0;
    if (act) {
      b = pk_nth_set_bit(cand, 0);
      cand &= cand - 1u;
    }
    T st[13], d[3] = {T(0), T(0), T(0)}, dl[3] = {T(0), T(0), T(0)}, pen = T(0), nl[3] = {T(0), T(0), T(1)};
    ldr<R_Q, 13>(env + RIX(B, b) * RS, st);       // (lanes without a candidate read body 0: unused)
    if (act) {
      const T *Q = st, *p = st + 4;
      d[0] = bp[0] - p[0]; d[1] = bp[1] - p[1]; d[2] = bp[2] - p[2];
      const T cq[4] = {-Q[0], -Q[1], -Q[2], Q[3]};
      qrot(cq, d, dl);   // ball centre in the body frame
    }
    const int nt = act ? B.t.ntris[b] : 1;
    const bool hit = hull_sphere_coop<T>(verts + (size_t)b * M.vmax * 3, M.vmax, B.t.face_planes + (size_t)b * B.t.face_tmax * 4,
                                         B.t.face_tris + (size_t)b * B.t.face_tmax * 4, nt, dl, c.bR, s, act, pen, nl);
    if (hit && pen > T(0)) take(b, false, pen, nl, st, d);
  }
  // deepest contact of the group (butterfly over the 8 lanes; equal depths: the lower body index, like the serial loop); skipped by
  // the whole warp when no lane found a contact (the common substep)
  if (!__any_sync(FULL, best > T(0))) return;
#pragma unroll
  for (int off = 1; off < SLOTS; off <<= 1) {
    const T opn = __shfl_xor_sync(FULL, best, off);
    const int obd = __shfl_xor_sync(FULL, bbody, off);
    T on[3], ov[3];
#pragma unroll
    for (int k = 0; k < 3; k++) { on[k] = __shfl_xor_sync(FULL, bn[k], off); ov[k] = __shfl_xor_sync(FULL, bvo[k], off); }
    const T oe = __shfl_xor_sync(FULL, be, off), om = __shfl_xor_sync(FULL, bmu, off);
    if (opn > best || (opn == best && obd < bbody)) {
      best = opn; bbody = obd; be = oe; bmu = om;
#pragma unroll
      for (int k = 0; k < 3; k++) { bn[k] = on[k]; bvo[k] = ov[k]; }
    }
  }
  if (valid && s == BALL_SLOT && best > T(0)) {
    T J[3];
    ball_impulse(c, ball, bn, bvo, be, bmu, J);
#pragma unroll
    for (int k = 0; k < 3; k++) ball.p[k] += best * bn[k];
  }
}

// DOF force sensor (b200_buffers_t::dof_force).  out[3j + k] = the generalized force that joint j's drive and its limit spring-damper
// applied in the last substep of the control step, in the joint's child frame (the frame of dof_vel, so out . dof_vel is the drive's
// power).  The drive is implicit, so the force is taken at the end-of-substep velocity qd+ = qd + h qdd, not the start-of-substep one:
//   tau = kp (pd - q - h qd+) - kd qd+  [+ limk (lim - q - h qd+) - limc qd+ while the limit is active]
// i.e. the explicit torque of pk_body minus (h kd + h^2 kp [+ h limc + h^2 limk]) qdd.  Armature is inertia, not a force; contact and
// joint-reaction forces are not part of it.  Run after the last substep by the lane that owns the body's PD target (pk_pd_take), from
// q and qd+ that pk_forward left in the body's E slot; the three values go straight to global memory.
template <typename T, int LPE = SLOTS>
__device__ __forceinline__ void pk_dof_force(const DevBlob& B, const b200_model_t& MN, const PhysCfg<T>& c, const T* env, int s, bool valid,
                                             const T (&pd)[PK_PD_SLOTS][3], T* __restrict__ out) {
  const b200_model_t& M = B.m;
  for (int rr = 0; rr * LPE < M.nb; rr++) {
    const int b = rr * LPE + s;
    if (!valid || b == 0 || b >= M.nb || M.fixed[b]) continue;
    T st[6], p[3];   // q[3] qd+[3]
    ldr<R_E, 6>(env + RIX(B, b) * REC, st);
    pk_pd_pick<T>(pd, rr, p);
    const int d0 = M.dof_of_body[b];
#pragma unroll
    for (int k = 0; k < 3; k++) {
      const T q = st[k], qd = st[3 + k];
      const T kp = T(MN.kp[d0 + k]), kd = T(MN.kd[d0 + k]);
      T tau = kp * (p[k] - q - c.h * qd) - kd * qd;
      const T lo = T(MN.lim_lo[d0 + k]), hi = T(MN.lim_hi[d0 + k]);
      if (q < lo) tau += c.limk * (lo - q - c.h * qd) - c.limc * qd;
      else if (q > hi) tau += c.limk * (hi - q - c.h * qd) - c.limc * qd;
      out[d0 + k] = tau;
    }
  }
}

// One control step for the warp's EPW envs.  wrec: the warp's records; valid: this lane's env exists.
// The ball of env g is carried by lane (g, BALL_SLOT) in registers.
// B: the tree tables and topology every env of the warp shares; MN / verts: the numeric constants and hull vertices of this lane's
// env (B.m and its vertices when the warp's envs are of one asset).  The ball paths read B only: a handle whose envs have different
// assets has no ball (b200env_create_assets).
// DOF_FORCE: the DOF force sensor (pk_dof_force) into dof_force = the [nd] row of this lane's env (null on a lane without an env).
template <typename T, bool DOF_FORCE = false>
__device__ __forceinline__ void control_step_packed(const DevBlob& B, const b200_model_t& MN, const float* verts, const PhysCfg<T>& c, T* wrec,
                                                    int lane, bool valid, Ball<T>& ball, bool cta_sync, T* dof_force = nullptr) {
  const b200_model_t& M = B.m;
  const int g = lane >> 3, s = lane & 7;
  T* env = wrec + g * ENV_STRIDE;
  const int nb = M.nb;
  T pd[PK_PD_SLOTS][3];   // PD targets of my body-pass bodies
  pk_pd_take<T>(B, env, s, valid, pd);
  // kinematics of the start state, root -> leaves; every later FK is fused into the forward pass of the substep before it
  for (int d = 1; d <= M.max_depth; d++) {
    const int b = valid ? B.t.lvl_all[d][s] : -1;
    if (b >= 0) pk_fk<T, true>(B, MN, env, b);
    __syncwarp();
  }
  for (int sim = 0; sim < c.cfi; sim++) {
    if (c.has_ball && valid && s == BALL_SLOT) {
      ball_aero<T>(ball.v, ball.w, c.spin_scale, ball.fa);
      const T thr = c.substeps > 2 ? c.bR * T(6) : c.bR * T(4);
      if (!ball.has_bounce && ball.p[2] <= thr) {
        ball.has_bounce = 1; ball.bounce_now = 1;
        ball.bpos[0] = ball.p[0]; ball.bpos[1] = ball.p[1]; ball.bpos[2] = ball.p[2];
      }
    }
    for (int sub = 0; sub < c.substeps; sub++) {
      if (cta_sync && (PK_SYNC_EVERY == 1 || (sub % PK_SYNC_EVERY) == 0)) __syncthreads();
      // 1. per-body inertia / bias / contacts / joint drive
      for (int rr = 0; rr * SLOTS < (ABL == 8 ? 0 : nb); rr++) {
        const int b = rr * SLOTS + s;
        if (valid && b < nb && !M.fixed[b]) {
          T pdb[3];
          pk_pd_pick<T>(pd, rr, pdb);
          pk_body<T, PK_CONTACT_COMPACT != 0>(B, MN, verts, c, env, b, sim == 0, pdb);
        }
      }
      __syncwarp();
#if PK_CONTACT_COMPACT
      pk_contact_phase<T>(B, MN, verts, c, env, lane, valid);
      __syncwarp();
#endif
      // 2. articulated inertia, leaves -> root
      for (int d = (ABL == 9 ? 0 : M.max_depth); d >= 1; d--) {
        const int b = valid ? B.t.lvl_dyn[d][s] : -1;
        T out[R_AB];
        if (b >= 0) pk_backward<T>(B, env, b, out);
        const int rounds = B.t.maxch[d - 1];
        for (int cr = 0; cr < rounds; cr++) {
          if (b >= 0 && B.t.child_rank[b] == cr) {
            T* pr = env + RIX(B, M.parent[b]) * REC;
            T acc[R_AB];
            ldr<R_A, R_AB>(pr, acc);
#pragma unroll
            for (int k = 0; k < R_AB; k++) acc[k] += out[k];
            str<R_A, R_AB>(pr, acc);
          }
          __syncwarp();
        }
      }
      // 3. root acceleration (lane slot 0) next to the ball (slot 7: uses the racket's start-of-substep pose / velocity, which the
      //    fused pass below is about to overwrite), then the root is integrated
      if (c.has_ball && valid && s == BALL_SLOT) {
        T rQ[4] = {0, 0, 0, 1}, rp[3] = {0, 0, 0}, rv[3] = {0, 0, 0}, rw[3] = {0, 0, 0};
        const bool has_racket = c.racket_body >= 0;
        if (has_racket) {
          const T* rr = env + RIX(B, c.racket_body) * REC;
          T rs[13];
          ldr<R_Q, 13>(rr, rs);
#pragma unroll
          for (int k = 0; k < 4; k++) rQ[k] = rs[k];
#pragma unroll
          for (int k = 0; k < 3; k++) { rp[k] = rs[4 + k]; rw[k] = rs[7 + k]; rv[k] = rs[10 + k]; }
        }
        ball_substep<T>(c, ball, has_racket, rQ, rp, rv, rw);
        T* ext = env + ENV_EXT;
#pragma unroll
        for (int k = 0; k < 3; k++) { if (!PK_IS_SHADOW) { ext[6 + k] = ball.rF[k]; ext[9 + k] = ball.rX[k]; } }
      }
      if (c.ball_body) pk_ball_contacts_group<T>(B, verts, c, env, lane, valid, ball);   // all lanes: the body loop is spread over the group
      if (valid && s == 0) pk_root<T>(c, env);
      if (c.ball_body) __syncwarp();   // the extra ball contacts read the root's pose: integrate it only after every lane is done
      if (valid && s == 0) pk_root_integrate<T>(c, env);
      __syncwarp();
      // 4. root -> leaves: accelerations + joint integration of a body, then at once its kinematics for the next substep
      //    (its parent's new pose is already in place); welded bodies only have the kinematics
      for (int d = 1; d <= (ABL == 10 ? 0 : M.max_depth); d++) {
        const int b = valid ? B.t.lvl_all[d][s] : -1;
        if (b >= 0) {
          if (!M.fixed[b]) {
            T qn[4], wt[3];
            pk_forward<T, DOF_FORCE>(B, c, env, b, qn, wt, DOF_FORCE && sim == c.cfi - 1 && sub == c.substeps - 1);
            pk_fk<T, true, true>(B, MN, env, b, qn, wt);
          } else {
            pk_fk<T, true>(B, MN, env, b);
          }
        }
        __syncwarp();
      }
    }
  }
  if (DOF_FORCE) pk_dof_force<T>(B, MN, c, env, s, valid && dof_force != nullptr, pd, dof_force);
  pk_pd_park<T>(B, env, s, valid, pd);
}
template <typename T>
__device__ __forceinline__ void control_step_packed(const DevBlob& B, const float* verts, const PhysCfg<T>& c, T* wrec, int lane, bool valid,
                                                    Ball<T>& ball, bool cta_sync) {
  control_step_packed<T>(B, B.m, verts, c, wrec, lane, valid, ball, cta_sync);
}

// state of one env between the lane-per-body prologue / epilogue (lane = body) and the records
template <typename T> __device__ __forceinline__ void pk_store_state(T* env, const LaneConst& lc, int lane, const Lane<T>& L, const T* pd,
                                                                     const T* extF, const T* extT) {
  if (lc.active) {
    T* rec = env + lc.rix * REC;
    if (lane == 0) {
      T o[13];
#pragma unroll
      for (int k = 0; k < 4; k++) o[k] = L.Q[k];
#pragma unroll
      for (int k = 0; k < 3; k++) { o[4 + k] = L.p[k]; o[7 + k] = L.w[k]; o[10 + k] = L.v[k]; }
      str<R_Q, 13>(rec, o);
    } else if (lc.dyn) {
      str<R_QJ, 4>(rec, L.qj);
      str<R_PD, 3>(rec, pd);
      str<R_WT, 3>(rec, L.wt);
    }
  }
  if (lane == 0 && !PK_IS_SHADOW) {
    T* ext = env + ENV_EXT;
#pragma unroll
    for (int k = 0; k < 3; k++) { ext[k] = extF[k]; ext[3 + k] = extT[k]; ext[6 + k] = T(0); ext[9 + k] = T(0); }
  }
}
template <typename T> __device__ __forceinline__ void pk_load_state(const T* env, const LaneConst& lc, int lane, Lane<T>& L, T* cf) {
  lane_rest(L);
#pragma unroll
  for (int k = 0; k < 3; k++) cf[k] = 0;
  if (lc.active) {
    const T* rec = env + lc.rix * REC;
    T o[16];
    ldr<R_Q, 16>(rec, o);
#pragma unroll
    for (int k = 0; k < 4; k++) L.Q[k] = o[k];
#pragma unroll
    for (int k = 0; k < 3; k++) { L.p[k] = o[4 + k]; L.w[k] = o[7 + k]; L.v[k] = o[10 + k]; }
    if (lc.dyn) {
      cf[0] = rec[R_CFX];
      ldr<R_CFY, 2>(rec, cf + 1);
      if (lane > 0) {
        ldr<R_QJ, 4>(rec, L.qj);
#pragma unroll
        for (int k = 0; k < 3; k++) L.wt[k] = o[13 + k];
      }
    }
  }
}
// between two control steps of the test kernels the joint rotation crosses as exp-map coordinates (like the state rows do); the
// records of the warp's NE envs eb, eb + 1, .. below n.  Twin of pt_requantize.
template <typename T, int NE = EPW> __device__ __forceinline__ void pk_requantize(T* wrec, const LaneConst& lc, int lane, int64_t eb, int64_t n) {
  for (int k = 0; k < NE; k++) {
    if (eb + k >= n) break;
    if (lc.dyn && lane > 0) {
      T* rec = wrec + k * ENV_STRIDE + lc.rix * REC;
      T qj[4], q[3];
      ldr<R_QJ, 4>(rec, qj);
      qlog(qj, q);
      qexp(q, qj);
      str<R_QJ, 4>(rec, qj);
    }
  }
  __syncwarp();
}
