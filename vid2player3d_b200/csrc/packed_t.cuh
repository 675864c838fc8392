// packed_t.cuh - the "one wave" form of the packed articulated step (included by b200env.cu after packed.cuh).
//
// Why: step_kernel_packed keeps a 68-float record per body in shared memory, 6.7 KB per env, so an SM holds 32 envs (8 warps); the
// launch is latency-bound on one warp's dependent instruction stream.  56 resident envs per SM (14 warps) need <= 3.7 KB per env of
// shared memory, but the fields that lanes hand to each other are already 4.0 KB.  Here
//   * every dynamic body has ONE owner lane for all passes (DevTree::pt_slot: the bodies of a tree depth sit in different slots of
//     the env's 8 lanes), so the fields only the owner touches - joint state, PD target, r / zeta, joint-space bias, E / D^-1 and the
//     C / bn / bf part of the articulated inertia: 40 floats per body - move out of shared memory into a LANE-PRIVATE store: 128
//     values per lane, three 40-value blocks (DevTree::pt_blk); on the GPU a per-thread array in local memory (interleaved by the
//     hardware, so a warp's access to one column is one coalesced transaction, cached in L1 / L2);
//   * child -> parent hand-over of the articulated inertia goes through a small per-env mailbox (one entry per body of a depth)
//     instead of read-modify-write on the parent's record; the parent adds its children in rank order (same order, same bits);
//   * what stays in shared memory per body is the pose / velocity of its origin (13 floats, read by children, the ball, contacts)
//     and A / Bm of the articulated inertia (15; the accelerations alias A after the body's forward step): 28 floats, a stride that
//     keeps the 128-bit accesses of neighbouring lanes conflict-free.  3.6 KB per env with the mailbox, the residual wrench and the ball;
//   * ground contact: masks in the body pass, the bodies in contact of an env compacted into exchange entries carved out of the mailbox
//     (idle between two backward passes) and applied by the env's 8 lanes, 8 bodies per chunk.
// The arithmetic is that of packed.cuh, operation for operation (tests/test_gpu_tmem.py holds the two kernels to exact equality in a
// -fmad=false build; tests/test_emu_packed.py in float32 emulation).  PS is the private store, PrivMem: the thread's local array on
// the GPU (float), one row of a plain array per lane in the CPU lane emulator (double).
#pragma once

enum { PT_Q = 0, PT_P = 4, PT_W = 7, PT_V = 10, PT_A = 13, PT_BM = 19, PT_REC = 28 };
#define PT_ACC PT_A         // (alpha, a) of a body after its forward step: aliases A (dead by then)
enum { PT_SQJ = 13, PT_SPD = 17, PT_SWT = 20 };   // staging of joint rotation / PD target / joint velocity between the lane-per-body prologue / epilogue and the owners
#define PT_MAXREC B200_MAX_BODIES_PK
#define PT_MBOX_MAX 6
#define PT_MB 28
#define PT_BALL_T 24        // the env's ball (Ball<T>) parked in the env's shared memory between its substeps: 24 values of T cover the struct
enum { PT_ENV_MBOX = PT_MAXREC * PT_REC, PT_ENV_EXT = PT_ENV_MBOX + PT_MBOX_MAX * PT_MB, PT_ENV_BALL = PT_ENV_EXT + 12,
       PT_ENV_STRIDE = PT_ENV_BALL + PT_BALL_T };
// private fields of a body: column offsets inside its block (runs start on the boundary of the widest shape that moves them)
enum { TQ_QJ = 0, TQ_WT = 4, TQ_PD = 7, TQ_R = 10, TQ_ZETA = 13, TQ_U = 19, TQ_E = 22, TQ_C = 28, TQ_BN = 34, TQ_BF = 37, PT_COLS = 40 };
#define PT_BLOCKS 3
#ifndef PT_PROF
#define PT_PROF 0   // 1 (tools/pt_prof.sh): per-warp cycle counts of the phases of a control step -> g_pt_prof (which warp ends last, and in what)
#endif
#if PT_PROF && defined(__CUDACC__)
#define PT_PROF_SLOTS 8
__device__ unsigned long long g_pt_prof[4096 * PT_PROF_SLOTS];
#define PT_T0() unsigned long long pt_t_ = clock64()
#define PT_TICK(i) do { const unsigned long long n_ = clock64(); pt_acc_[i] += n_ - pt_t_; pt_t_ = n_; } while (0)
#else
#define PT_T0() do {} while (0)
#define PT_TICK(i) do {} while (0)
#endif
#ifndef PT_SYNC_EVERY
#define PT_SYNC_EVERY 1   // CTA barrier every n-th substep (PT_STEP_SYNC): instruction-cache sharing against waiting for the slowest warp
#endif
#ifndef PT_CONTACT_COMPACT
#define PT_CONTACT_COMPACT 1   // per-vertex ground contact as a compacted phase: the bodies in contact of an env are handed to the env's 8 lanes
#endif                         // (exchange through the hand-over mailbox, idle between two backward passes); 0: in place on the owner's lane
#ifndef PT_CX
#define PT_CX 8                // exchange entries per env (one per lane of the group), carved out of the mailbox: PT_CX * PT_CXS <= PT_MBOX_MAX * PT_MB;
#endif                         // an env with more bodies in contact takes several chunks (their masks wait in the owners' spare columns)
enum { CX_CBB = 0, CX_MASK = 12, PT_CXS = 16 };   // layout of an exchange entry: C bn bf, mask lo / hi, body index (PT_CXS values, 16-byte aligned)
static_assert(PT_CX * PT_CXS <= PT_MBOX_MAX * PT_MB && PT_CX <= 8, "exchange entries must fit the mailbox, one per lane of the group at most");
#ifndef PT_ABL
#define PT_ABL 0   // ablation of the phases (timing / register-pressure experiments only): 1 body pass, 2 backward, 3 forward, 4 root / ball, 5 no ground contact
#endif
#define PT_WARP_COLS 128    // values of one lane's private store
#define PT_XMASK (PT_BLOCKS * PT_COLS)   // columns 120..125 of a lane: penetration masks (2 words per block) of bodies waiting for a later contact chunk

// private store as plain memory: one array of PT_BLOCKS * PT_COLS values per lane
template <typename T> struct PrivMem {
  T* base;
  template <int OFF, int N> __device__ __forceinline__ void ld(int blk, T* r) const {
#pragma unroll
    for (int k = 0; k < N; k++) r[k] = base[blk * PT_COLS + OFF + k];
  }
  template <int OFF, int N> __device__ __forceinline__ void st(int blk, const T* r) const {
#pragma unroll
    for (int k = 0; k < N; k++) base[blk * PT_COLS + OFF + k] = r[k];
  }
  __device__ __forceinline__ void ld2(int col, T* r) const { r[0] = base[col]; r[1] = base[col + 1]; }   // run-time (even) column
  __device__ __forceinline__ void st2(int col, const T* r) const { base[col] = r[0]; base[col + 1] = r[1]; }
  __device__ __forceinline__ void wait_ld() const {}
  __device__ __forceinline__ void wait_st() const {}
};


// the barrier at the top of a substep: the whole CTA, or (PT_SYNC_GROUPS = 2) the even and the odd warps among themselves - half as many
// warps to wait for, two instruction streams in the instruction cache
#ifndef PT_SYNC_GROUPS
#define PT_SYNC_GROUPS 1
#endif
__device__ __forceinline__ void pt_substep_barrier() {
#if defined(__CUDA_ARCH__)
  if (PT_SYNC_GROUPS == 1) { __syncthreads(); return; }
  const unsigned w = threadIdx.x >> 5, nw = blockDim.x >> 5;
  const unsigned grp = w % PT_SYNC_GROUPS, cnt = (nw - grp + PT_SYNC_GROUPS - 1) / PT_SYNC_GROUPS * 32;   // warps grp, grp + G, ...
  asm volatile("bar.sync %0, %1;" ::"r"(grp + 1), "r"(cnt) : "memory");
#else
  __syncthreads();
#endif
}

// kinematics of body b from its parent's pose; the joint rotation / velocity come in registers.  Stores the pose of the body origin;
// a jointed body also returns r = p - p_parent and the velocity-product terms (rz[9], private fields of the owner).
template <typename T>
__device__ __forceinline__ void pt_fk(const DevBlob& B, T* env, int b, const T* qj, const T* wt, T* rz) {
  const b200_model_t& M = B.m;
  T* rec = env + RIX(B, b) * PT_REC;
  const T* par = env + RIX(B, M.parent[b]) * PT_REC;
  T ps[13];  // parent Q[4] p[3] w[3] v[3]
  ldr<PT_Q, 13>(par, ps);
  const T *pQ = ps, *pp = ps + 4, *pw = ps + 7, *pv = ps + 10;
  T off[3] = {T(M.offset[b][0]), T(M.offset[b][1]), T(M.offset[b][2])}, rr[3], wxr[3];
  T o[13];   // own Q[4] p[3] w[3] v[3]
  qrot(pQ, off, rr);
  cross3(pw, rr, wxr);
#pragma unroll
  for (int k = 0; k < 3; k++) { o[4 + k] = pp[k] + rr[k]; o[10 + k] = pv[k] + wxr[k]; }
  if (M.fixed[b]) {
#pragma unroll
    for (int k = 0; k < 4; k++) o[k] = pQ[k];
#pragma unroll
    for (int k = 0; k < 3; k++) o[7 + k] = pw[k];
    str<PT_Q, 13>(rec, o);
  } else {
    T wj[3];
    qmul(pQ, qj, o);
    qnormalize(o);
    qrot(o, wt, wj);
#pragma unroll
    for (int k = 0; k < 3; k++) o[7 + k] = pw[k] + wj[k];
    str<PT_Q, 13>(rec, o);
    rz[0] = rr[0]; rz[1] = rr[1]; rz[2] = rr[2];
    cross3(pw, wj, rz + 3); cross3(pw, wxr, rz + 6);
  }
}

// rigid-body inertia + bias + external / ground-contact terms of one dynamic body: A / Bm go to the body's record, the rest comes back
// in registers for the private store (cbb = C[6] bn[3] bf[3]); cf[3] is the ground-contact force on the body.  The joint drive is a
// section of its own (pt_body_drive) so that the joint state is only fetched from the private store after the contact code is done with
// its registers.
// PT_CONTACT_COMPACT: only the penetration mask of the hull is computed here (returned in mask); pt_contact_phase adds the vertices.
template <typename T>
__device__ __forceinline__ void pt_body_inertia(const DevBlob& B, const float* __restrict__ verts, const PhysCfg<T>& c, T* env, int b, bool ext_on,
                                                T* cbb, T* cf, unsigned long long& mask) {
  const b200_model_t& M = B.m;
  T* rec = env + RIX(B, b) * PT_REC;
  T own[13], R[9];   // Q[4] p[3] w[3] v[3]
  ldr<PT_Q, 13>(rec, own);
  const T *Q = own, *p = own + 4, *w = own + 7, *v = own + 10;
  qmat(Q, R);
  T ab[28];          // A[6] Bm[9] C[6] bn[3] bf[3] pad
  T *A = ab, *Bm = ab + 6, *C = ab + 15, *bn = ab + 21, *bf = ab + 24;
  cf[0] = cf[1] = cf[2] = T(0);
#pragma unroll
  for (int k = 6; k < 21; k++) ab[k] = T(0);
  ab[27] = T(0);
  const T ms = T(M.mass[b]);
  T cl[3] = {T(M.com[b][0]), T(M.com[b][1]), T(M.com[b][2])}, cw[3];
  mv3(R, cl, cw);
  {
    T Ib[6], F[9], RF[9];
#pragma unroll
    for (int k = 0; k < 6; k++) Ib[k] = T(M.inertia[b][k]);
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
  const T* ext = env + PT_ENV_EXT;
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
  const int nv = M.nverts[b];
  mask = 0ull;
  if (PT_ABL != 5 && nv > 0 && p[2] - T(M.radius[b]) < T(0)) {
#if PT_CONTACT_COMPACT
    mask = contact_mask<T>(verts + (size_t)b * M.vmax * 3, M.vmax, nv, R, p);
#else
    contact_hull<T>(verts + (size_t)b * M.vmax * 3, M.vmax, nv, c, R, p, v, w, A, Bm, C, bn, bf, cf);
#endif
  }
  str<PT_A, 15>(rec, ab);
#pragma unroll
  for (int k = 0; k < 12; k++) cbb[k] = ab[15 + k];
}
// implicit PD drive + joint limits of a jointed body: jp = qj[4] wt[3] pd[3] (private) -> E[6] (world-frame diagonal terms), u[3]
template <typename T>
__device__ __forceinline__ void pt_body_drive(const DevBlob& B, const PhysCfg<T>& c, const T* env, int b, const T* jp, T* E, T* u) {
  const b200_model_t& M = B.m;
  T Q[4], R[9];
  ldr<PT_Q, 4>(env + RIX(B, b) * PT_REC, Q);
  qmat(Q, R);
  const int d0 = M.dof_of_body[b];
  T q[3], tau[3], e[3];
  const T *qj = jp, *wt = jp + 4, *pd = jp + 7;
  qlog(qj, q);
#pragma unroll
  for (int k = 0; k < 3; k++) {
    T kp = T(M.kp[d0 + k]), kd = T(M.kd[d0 + k]);
    e[k] = T(M.armature[d0 + k]) + c.h * kd + c.h * c.h * kp;
    tau[k] = kp * (pd[k] - q[k] - c.h * wt[k]) - kd * wt[k];
    T lo = T(M.lim_lo[d0 + k]), hi = T(M.lim_hi[d0 + k]);
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
}

// bit patterns <-> slots of the value type (the mask words and the body index ride in an exchange entry next to the floats)
template <typename T> __device__ __forceinline__ T pt_bits_to_slot(uint32_t x) { return pk_bits_to_slot<T>(x); }
__device__ __forceinline__ int pt_popc(uint32_t x) {
#if defined(__CUDA_ARCH__)
  return __popc(x);
#else
  int n = 0;
  for (; x; x &= x - 1) n++;
  return n;
#endif
}
// PT_CONTACT_COMPACT, the worker side: lane s of the env's group takes exchange entry s (body, penetration mask, C / bn / bf as the body
// pass left them), adds the penetrating vertices in ascending order to A / Bm (the body's record) and C / bn / bf / cf (the entry) - the
// same sums in the same order as the in-place form - and leaves the results in the entry for the owner.
template <typename T>
__device__ __forceinline__ void pt_contact_phase(const DevBlob& B, const float* __restrict__ verts, const PhysCfg<T>& c, T* env, int s, int n,
                                                 T* cf_env, bool last) {
  const b200_model_t& M = B.m;
  if (s < n) {
    T* ent = env + PT_ENV_MBOX + s * PT_CXS;
    T cbb[12], mk[3], own[13], R[9], ab[28], cf[3] = {T(0), T(0), T(0)};
    ldr<CX_CBB, 12>(ent, cbb);
    ldr<CX_MASK, 3>(ent, mk);
    const int b = (int)pk_slot_to_bits(mk[2]);
    const unsigned long long mask = (unsigned long long)pk_slot_to_bits(mk[0]) | ((unsigned long long)pk_slot_to_bits(mk[1]) << 32);
    T* rec = env + RIX(B, b) * PT_REC;
    ldr<PT_Q, 13>(rec, own);
    ldr<PT_A, 15>(rec, ab);
#pragma unroll
    for (int k = 0; k < 12; k++) ab[15 + k] = cbb[k];
    qmat(own, R);
    contact_apply<T>(verts + (size_t)b * M.vmax * 3, M.vmax, mask, c, R, own + 4, own + 10, own + 7, ab, ab + 6, ab + 15, ab + 21, ab + 24, cf);
    str<PT_A, 15>(rec, ab);
    str<CX_CBB, 12>(ent, ab + 15);
    if (last && cf_env) { cf_env[b * 3] = cf[0]; cf_env[b * 3 + 1] = cf[1]; cf_env[b * 3 + 2] = cf[2]; }
  }
}

// backward step of one dynamic non-root body, registers only: ab = A[6] Bm[9] C[6] bn[3] bf[3] (children already added), rzu = r[3]
// zeta[6] u[3], E -> D^-1 (in place), u -> u - bn (in rzu[9..11]); the articulated inertia / bias shifted to the parent origin goes to
// the body's hand-over entry mbox[28]
template <typename T>
__device__ __forceinline__ void pt_backward(const T* ab, T* rzu, T* E, T* mbox) {
  const T *A = ab, *Bm = ab + 6, *C = ab + 15, *bn = ab + 21, *bf = ab + 24, *r = rzu, *zeta = rzu + 3;
  T u[3] = {rzu[9], rzu[10], rzu[11]};
  T D[6], Dinv[6];
#pragma unroll
  for (int k = 0; k < 6; k++) D[k] = A[k] + E[k];
  sym_inv(D, Dinv);
  u[0] -= bn[0]; u[1] -= bn[1]; u[2] -= bn[2];
#pragma unroll
  for (int k = 0; k < 6; k++) E[k] = Dinv[k];
  rzu[9] = u[0]; rzu[10] = u[1]; rzu[11] = u[2];
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
  T out[28];
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
  out[27] = T(0);
  str<0, 28>(mbox, out);
}

// root: 6 x 6 solve by block elimination, registers only (ab: the root's articulated inertia / bias with its children added)
template <typename T> __device__ __forceinline__ void pt_root(const T* ab, T* acc) {
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
}

// forward step of one dynamic non-root body: accelerations (left in the record for the children: PT_ACC aliases A), integration of the
// joint state.  Dinv, rzu (r zeta u) and qj / wt (in: old, out: new) are the owner's private fields, in registers.
template <typename T>
__device__ __forceinline__ void pt_forward(const DevBlob& B, const PhysCfg<T>& c, T* env, int b, const T* Dinv, const T* rzu, T* qj, T* wt) {
  const b200_model_t& M = B.m;
  T* rec = env + RIX(B, b) * PT_REC;
  const T* par = env + RIX(B, M.parent[b]) * PT_REC;
  T pa[6], abm[15], Q[4];
  ldr<PT_ACC, 6>(par, pa);
  ldr<PT_A, 15>(rec, abm);
  ldr<PT_Q, 4>(rec, Q);
  const T *A = abm, *Bm = abm + 6, *r = rzu, *zeta = rzu + 3, *u = rzu + 9;
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
  str<PT_ACC, 6>(rec, acc);
  T cq[4] = {-Q[0], -Q[1], -Q[2], Q[3]};
  qrot(cq, gam, wd);  // R^T gam
#pragma unroll
  for (int k = 0; k < 3; k++) wt[k] = (wt[k] + c.h * wd[k]) * c.damp;
  T n2 = wt[0] * wt[0] + wt[1] * wt[1] + wt[2] * wt[2];
  if (n2 > c.wmax * c.wmax) { T sc = c.wmax * rsqrt_(n2); wt[0] *= sc; wt[1] *= sc; wt[2] *= sc; }
  T hv[3] = {c.h * wt[0], c.h * wt[1], c.h * wt[2]}, dq[4], qn[4];
  qexp_small(hv, dq);
  qmul(qj, dq, qn);
  qnormalize(qn);
#pragma unroll
  for (int k = 0; k < 4; k++) qj[k] = qn[k];
}

template <typename T> __device__ __forceinline__ void pt_root_integrate(const PhysCfg<T>& c, T* env) {
  T* rec = env;   // the root is record 0
  T acc[6], o[13];   // Q[4] p[3] w[3] v[3]
  ldr<PT_ACC, 6>(rec, acc); ldr<PT_Q, 13>(rec, o);
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
  str<PT_Q, 13>(rec, o);
}

// ab (A Bm from the record, C bn bf from the private store) += the hand-over entries of the body's children, in child-rank order
template <typename T> __device__ __forceinline__ int pt_add_children(const DevBlob& B, const T* env, int b, T* ab) {
  int nch = 0;
#pragma unroll 1
  for (int cr = 0; cr < MAX_CHILD; cr++) {
    const int ch = B.t.child[b][cr];
    if (ch < 0) break;
    const T* mb = env + PT_ENV_MBOX + B.t.pt_mbox[ch] * PT_MB;
    T o[28];
    ldr<0, 28>(mb, o);
#pragma unroll
    for (int k = 0; k < 27; k++) ab[k] += o[k];
    nch++;
  }
  return nch;
}

// One control step for the warp's EPW envs.  wrec: the warp's records (PT_ENV_STRIDE per env); valid: this lane's env exists; ps: the
// lane's private store, already holding qj / wt / pd of its bodies (pt_adopt); cf_env: where the ground-contact forces of this lane's
// env go after the last substep ([body][3], may be null).  The ball of env g is carried by lane (g, BALL_SLOT) in registers.
template <typename T, typename PS>
__device__ __forceinline__ void control_step_t(const DevBlob& B, const float* verts, const PhysCfg<T>& c, T* wrec, int lane, bool valid,
                                               Ball<T>& ball, const PS& ps, T* cf_env, bool cta_sync) {
  const b200_model_t& M = B.m;
  const int g = lane >> 3, s = lane & 7;
  T* env = wrec + g * PT_ENV_STRIDE;
  const int rblk = B.t.pt_blk[0], rslot = B.t.pt_slot[0];
  // the ball lives in the env's shared memory during the step (24 registers less in every phase of every lane); the lane that carries
  // it takes it into registers for its own substep only
  static_assert(sizeof(Ball<T>) <= PT_BALL_T * sizeof(T), "Ball<T> must fit its parking slot");
  Ball<T>* sball = reinterpret_cast<Ball<T>*>(env + PT_ENV_BALL);
  const bool ball_lane = c.has_ball && valid && s == BALL_SLOT;
  if (ball_lane) *sball = ball;
  // kinematics of the start state, root -> leaves; every later FK is fused into the forward pass of the substep before it
  for (int d = 1; d <= M.max_depth; d++) {
    const int b = valid ? B.t.pt_lvl[d][s] : -1;
    const int blk = B.t.pt_lblk[d];
    T jq[7], rz[9];   // qj[4] wt[3]
    if (blk >= 0) { ps.wait_st(); ps.template ld<TQ_QJ, 7>(blk, jq); ps.template ld<TQ_R, 9>(blk, rz); ps.wait_ld(); }
    if (b >= 0) pt_fk<T>(B, env, b, jq, jq + 4, rz);
    if (blk >= 0) ps.template st<TQ_R, 9>(blk, rz);
    __syncwarp();
  }
#if PT_PROF && defined(__CUDACC__)
  unsigned long long pt_acc_[PT_PROF_SLOTS] = {0, 0, 0, 0, 0, 0, 0, 0};
#endif
  PT_T0();
  for (int sim = 0; sim < c.cfi; sim++) {
    if (ball_lane) {
      Ball<T>& bl = *sball;
      ball_aero<T>(bl.v, bl.w, c.spin_scale, bl.fa);
      const T thr = c.substeps > 2 ? c.bR * T(6) : c.bR * T(4);
      if (!bl.has_bounce && bl.p[2] <= thr) {
        bl.has_bounce = 1; bl.bounce_now = 1;
        bl.bpos[0] = bl.p[0]; bl.bpos[1] = bl.p[1]; bl.bpos[2] = bl.p[2];
      }
    }
    for (int sub = 0; sub < c.substeps; sub++) {
      PT_TICK(7);
      if (cta_sync && (PT_SYNC_EVERY == 1 || (sim * c.substeps + sub) % PT_SYNC_EVERY == 0)) pt_substep_barrier();
      PT_TICK(0);
      const bool last = sim == c.cfi - 1 && sub == c.substeps - 1;
      // 1. per-body inertia / bias / ground contact / joint drive: the owner's three bodies, one per column block
      ps.wait_st();
      int ncx = 0;            // bodies in contact of my env so far
      uint32_t xmine = 0;     // per block k, 6 bits: bit 6k = my body of that block is in contact, bits 6k+1..6k+5 = its rank among the env's
      for (int k = 0; k < (PT_ABL == 1 ? 0 : PT_BLOCKS); k++) {
        const int b = valid ? B.t.pt_body[k][s] : -1;
        {
          T cbb[12], cf[3];
          unsigned long long mask = 0ull;
          if (b >= 0) pt_body_inertia<T>(B, verts, c, env, b, sim == 0, cbb, cf, mask);
#if PT_CONTACT_COMPACT
          const bool hit = mask != 0ull;
          const uint32_t gb = (__ballot_sync(FULL, hit) >> (g * 8)) & 0xFFu;
          const int idx = ncx + pt_popc(gb & ((1u << s) - 1u));
          ncx += pt_popc(gb);
          T later[2] = {T(0), T(0)};     // mask words of a body that has to wait for a later chunk
          if (hit) {
            xmine |= (1u | ((uint32_t)idx << 1)) << (6 * k);
            if (idx < PT_CX) {       // first chunk: hand the per-vertex part to the env's lanes right away
              T* ent = env + PT_ENV_MBOX + idx * PT_CXS;
              const T mk[3] = {pt_bits_to_slot<T>((uint32_t)mask), pt_bits_to_slot<T>((uint32_t)(mask >> 32)), pt_bits_to_slot<T>((uint32_t)b)};
              str<CX_CBB, 12>(ent, cbb);
              str<CX_MASK, 3>(ent, mk);
            } else {
              later[0] = pt_bits_to_slot<T>((uint32_t)mask); later[1] = pt_bits_to_slot<T>((uint32_t)(mask >> 32));
            }
          }
          ps.st2(PT_XMASK + 2 * k, later);
          if (b >= 0 && !hit && last && cf_env) { cf_env[b * 3] = cf[0]; cf_env[b * 3 + 1] = cf[1]; cf_env[b * 3 + 2] = cf[2]; }
#else
          if (b >= 0 && last && cf_env) { cf_env[b * 3] = cf[0]; cf_env[b * 3 + 1] = cf[1]; cf_env[b * 3 + 2] = cf[2]; }
#endif
          ps.template st<TQ_C, 12>(k, cbb);
        }
        T jp[10], E[6], u[3];   // jp: qj[4] wt[3] pd[3]
        ps.template ld<TQ_QJ, 10>(k, jp);
        ps.wait_ld();
        if (b > 0) pt_body_drive<T>(B, c, env, b, jp, E, u);
        ps.template st<TQ_U, 3>(k, u); ps.template st<TQ_E, 6>(k, E);
      }
      PT_TICK(1);
#if PT_CONTACT_COMPACT
      if (__any_sync(FULL, ncx > 0)) {            // some env of the warp touches the ground (warp-uniform)
        for (int c0 = 0;; c0 += PT_CX) {          // chunks of PT_CX bodies per env: one body per lane of the group
          if (c0 > 0) {                           // owners of the bodies ranked c0 .. c0 + PT_CX - 1 hand them over now
            for (int k = 0; k < PT_BLOCKS; k++) {
              const uint32_t f = xmine >> (6 * k);
              const int idx = (int)((f >> 1) & 31u) - c0;
              const bool mine = (f & 1u) && idx >= 0 && idx < PT_CX;
              if (!__any_sync(FULL, mine)) continue;   // (warp-uniform)
              T cbb[12], mk[3];
              ps.wait_st();
              ps.template ld<TQ_C, 12>(k, cbb); ps.ld2(PT_XMASK + 2 * k, mk);
              ps.wait_ld();
              if (mine) {
                T* ent = env + PT_ENV_MBOX + idx * PT_CXS;
                mk[2] = pt_bits_to_slot<T>((uint32_t)B.t.pt_body[k][s]);
                str<CX_CBB, 12>(ent, cbb);
                str<CX_MASK, 3>(ent, mk);
              }
            }
          }
          __syncwarp();                           // entries and A / Bm records visible to the group
          pt_contact_phase<T>(B, verts, c, env, s, ncx - c0 < PT_CX ? ncx - c0 : PT_CX, cf_env, last);
          __syncwarp();
          for (int k = 0; k < PT_BLOCKS; k++) {   // owners take C / bn / bf of their handed-over bodies back into the private store
            const uint32_t f = xmine >> (6 * k);
            const int idx = (int)((f >> 1) & 31u) - c0;
            const bool mine = (f & 1u) && idx >= 0 && idx < PT_CX;
            if (!__any_sync(FULL, mine)) continue;   // no lane of the warp handed a body of this block over in this chunk (warp-uniform)
            T cbb[12];
            ps.wait_st();
            ps.template ld<TQ_C, 12>(k, cbb);
            ps.wait_ld();
            if (mine) ldr<CX_CBB, 12>(env + PT_ENV_MBOX + idx * PT_CXS, cbb);
            ps.template st<TQ_C, 12>(k, cbb);
          }
          __syncwarp();                           // the entries are free: next chunk, or the hand-over entries of the backward pass
          if (!__any_sync(FULL, ncx > c0 + PT_CX)) break;
        }
      }
#endif
      PT_TICK(2);
      // 2. articulated inertia, leaves -> root
      for (int d = (PT_ABL == 2 ? 0 : M.max_depth); d >= 1; d--) {
        const int blk = B.t.pt_lblk[d];
        if (blk < 0) continue;                    // a depth of welded bodies only (warp-uniform)
        int b = valid ? B.t.pt_lvl[d][s] : -1;
        if (b >= 0 && M.fixed[b]) b = -1;
        T ab[28], rzu[12], E[6];
        ps.wait_st();
        ps.template ld<TQ_C, 12>(blk, ab + 15); ps.template ld<TQ_R, 12>(blk, rzu); ps.template ld<TQ_E, 6>(blk, E);
        ps.wait_ld();
        if (b >= 0) {
          T* rec = env + RIX(B, b) * PT_REC;
          ldr<PT_A, 15>(rec, ab);
          if (pt_add_children<T>(B, env, b, ab) > 0) str<PT_A, 15>(rec, ab);   // the forward step needs A / Bm with the children in
        }
        __syncwarp();                             // every lane has taken the entries of depth d + 1 out of the mailbox
        if (b >= 0) pt_backward<T>(ab, rzu, E, env + PT_ENV_MBOX + B.t.pt_mbox[b] * PT_MB);   // hand-over entry written as it is computed
        ps.template st<TQ_E, 6>(blk, E); ps.template st<TQ_U, 3>(blk, rzu + 9);
        __syncwarp();
      }
      PT_TICK(3);
      // 3. root acceleration (the root's owner lane) next to the ball (slot 7: uses the racket's start-of-substep pose / velocity, which
      //    the fused pass below is about to overwrite), then the root is integrated
      T rab[28];
      ps.wait_st();
      ps.template ld<TQ_C, 12>(rblk, rab + 15);
      ps.wait_ld();
      if (PT_ABL != 4 && c.has_ball) {
        Ball<T>& bl = *sball;   // worked on in place (every lane of the group may read it, only the ball's lane writes)
        if (ball_lane) {
          T rQ[4] = {0, 0, 0, 1}, rp[3] = {0, 0, 0}, rv[3] = {0, 0, 0}, rw[3] = {0, 0, 0};
          const bool has_racket = c.racket_body >= 0;
          if (has_racket) {
            const T* rr = env + RIX(B, c.racket_body) * PT_REC;
            T rs[13];
            ldr<PT_Q, 13>(rr, rs);
#pragma unroll
            for (int k = 0; k < 4; k++) rQ[k] = rs[k];
#pragma unroll
            for (int k = 0; k < 3; k++) { rp[k] = rs[4 + k]; rw[k] = rs[7 + k]; rv[k] = rs[10 + k]; }
          }
          ball_substep<T>(c, bl, has_racket, rQ, rp, rv, rw);
          T* ext = env + PT_ENV_EXT;
#pragma unroll
          for (int k = 0; k < 3; k++) { ext[6 + k] = bl.rF[k]; ext[9 + k] = bl.rX[k]; }
        }
        if (c.ball_body) pk_ball_contacts_group<T, PT_REC>(B, verts, c, env, lane, valid, bl);   // all lanes: the body loop is spread over the group
      }
      if (valid && s == rslot) {
        T acc[6];
        ldr<PT_A, 15>(env, rab);
        pt_add_children<T>(B, env, 0, rab);
        pt_root<T>(rab, acc);
        str<PT_ACC, 6>(env, acc);
      }
      if (c.ball_body) __syncwarp();   // the extra ball contacts read the root's pose: integrate it only after every lane is done
      if (valid && s == rslot) pt_root_integrate<T>(c, env);
      __syncwarp();
      PT_TICK(4);
      // 4. root -> leaves: accelerations + joint integration of a body, then at once its kinematics for the next substep
      //    (its parent's new pose is already in place); welded bodies only have the kinematics
      for (int d = 1; d <= (PT_ABL == 3 ? 0 : M.max_depth); d++) {
        const int b = valid ? B.t.pt_lvl[d][s] : -1;
        const int blk = B.t.pt_lblk[d];
        T Dinv[6], rzu[12], jq[7];
        if (blk >= 0) {
          ps.wait_st();
          ps.template ld<TQ_E, 6>(blk, Dinv); ps.template ld<TQ_R, 12>(blk, rzu); ps.template ld<TQ_QJ, 7>(blk, jq);
          ps.wait_ld();
        }
        if (b >= 0) {
          if (!M.fixed[b]) pt_forward<T>(B, c, env, b, Dinv, rzu, jq, jq + 4);
          pt_fk<T>(B, env, b, jq, jq + 4, rzu);
        }
        if (blk >= 0) { ps.template st<TQ_QJ, 7>(blk, jq); ps.template st<TQ_R, 9>(blk, rzu); }
        __syncwarp();
      }
    }
  }
  PT_TICK(5);
#if PT_PROF && defined(__CUDACC__)
  if (lane == 0) {
    const unsigned wid = (blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5)) & 4095u;
    for (int i = 0; i < PT_PROF_SLOTS; i++) g_pt_prof[wid * PT_PROF_SLOTS + i] = pt_acc_[i];
  }
#endif
  if (ball_lane) ball = *sball;
}

// lane-per-body prologue (lane = body of ONE env) -> records: root pose, and the joint state / PD target of the jointed bodies staged
// in the (not yet used) A / Bm run of their record for pt_adopt
template <typename T> __device__ __forceinline__ void pt_stage_in(T* env, const LaneConst& lc, int lane, const Lane<T>& L, const T* pd,
                                                                  const T* extF, const T* extT) {
  if (lc.active) {
    T* rec = env + lc.rix * PT_REC;
    if (lane == 0) {
      T o[13];
#pragma unroll
      for (int k = 0; k < 4; k++) o[k] = L.Q[k];
#pragma unroll
      for (int k = 0; k < 3; k++) { o[4 + k] = L.p[k]; o[7 + k] = L.w[k]; o[10 + k] = L.v[k]; }
      str<PT_Q, 13>(rec, o);
    } else if (lc.dyn) {
      T o[10];
#pragma unroll
      for (int k = 0; k < 4; k++) o[k] = L.qj[k];
#pragma unroll
      for (int k = 0; k < 3; k++) { o[4 + k] = pd[k]; o[7 + k] = L.wt[k]; }
      str<PT_SQJ, 10>(rec, o);
    }
  }
  if (lane == 0) {
    T* ext = env + PT_ENV_EXT;
#pragma unroll
    for (int k = 0; k < 3; k++) { ext[k] = extF[k]; ext[3 + k] = extT[k]; ext[6 + k] = T(0); ext[9 + k] = T(0); }
  }
}
// owners take the staged joint state / PD target of their bodies into the private store (after a __syncwarp behind pt_stage_in)
template <typename T, typename PS>
__device__ __forceinline__ void pt_adopt(const DevBlob& B, const T* wrec, int lane, bool valid, const PS& ps) {
  const int g = lane >> 3, s = lane & 7;
  const T* env = wrec + g * PT_ENV_STRIDE;
  for (int k = 0; k < PT_BLOCKS; k++) {
    const int b = valid ? B.t.pt_body[k][s] : -1;
    T st[10], jp[10];   // staged: qj[4] pd[3] wt[3]; private: qj[4] wt[3] pd[3]
#pragma unroll
    for (int j = 0; j < 10; j++) st[j] = T(0);
    st[3] = T(1);
    if (b > 0) ldr<PT_SQJ, 10>(env + RIX(B, b) * PT_REC, st);
#pragma unroll
    for (int j = 0; j < 4; j++) jp[j] = st[j];
#pragma unroll
    for (int j = 0; j < 3; j++) { jp[4 + j] = st[7 + j]; jp[7 + j] = st[4 + j]; }
    ps.template st<TQ_QJ, 10>(k, jp);
  }
  ps.wait_st();
}
// owners publish the joint state of their bodies for the lane-per-body epilogue (the A / Bm run is dead after the last forward pass)
template <typename T, typename PS>
__device__ __forceinline__ void pt_publish(const DevBlob& B, T* wrec, int lane, bool valid, const PS& ps) {
  const int g = lane >> 3, s = lane & 7;
  T* env = wrec + g * PT_ENV_STRIDE;
  for (int k = 0; k < PT_BLOCKS; k++) {
    const int b = valid ? B.t.pt_body[k][s] : -1;
    T jq[7];
    ps.wait_st();
    ps.template ld<TQ_QJ, 7>(k, jq);
    ps.wait_ld();
    if (b > 0) {
      T* rec = env + RIX(B, b) * PT_REC;
      str<PT_SQJ, 4>(rec, jq);
      str<PT_SWT, 3>(rec, jq + 4);
    }
  }
}
// between two control steps of the test kernels the joint rotation crosses as exp-map coordinates (like the state rows do)
template <typename T, typename PS>
__device__ __forceinline__ void pt_requantize(const DevBlob& B, int lane, bool valid, const PS& ps) {
  const int s = lane & 7;
  for (int k = 0; k < PT_BLOCKS; k++) {
    const int b = valid ? B.t.pt_body[k][s] : -1;
    T qj[4], q[3];
    ps.wait_st();
    ps.template ld<TQ_QJ, 4>(k, qj);
    ps.wait_ld();
    if (b > 0) { qlog(qj, q); qexp(q, qj); }
    ps.template st<TQ_QJ, 4>(k, qj);
  }
}
template <typename T> __device__ __forceinline__ void pt_load_state(const T* env, const LaneConst& lc, int lane, Lane<T>& L) {
  lane_rest(L);
  if (lc.active) {
    const T* rec = env + lc.rix * PT_REC;
    T o[13];
    ldr<PT_Q, 13>(rec, o);
#pragma unroll
    for (int k = 0; k < 4; k++) L.Q[k] = o[k];
#pragma unroll
    for (int k = 0; k < 3; k++) { L.p[k] = o[4 + k]; L.w[k] = o[7 + k]; L.v[k] = o[10 + k]; }
    if (lc.dyn && lane > 0) {
      ldr<PT_SQJ, 4>(rec, L.qj);
      ldr<PT_SWT, 3>(rec, L.wt);
    }
  }
}
