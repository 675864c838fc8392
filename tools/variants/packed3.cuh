// packed3.cuh - "2 envs per warp, 3 lanes per body in the backward pass" form of the articulated control step.
//
// Why: the 4-envs-per-warp kernel is bound by one warp's dependent instruction stream - 7
// warps per SM keep 38 % of the issue slots busy, and shared memory (then 7.2 KB of records per env) did not allow more envs in flight.
// The same 28 envs per SM could be spread over 14 warps if a warp carries 2 envs, which pays only if the stream per warp gets
// shorter.  Here lane = (env g = lane / 16, body slot s = (lane % 16) / 3, column c = lane % 3), lane 15 of each half-warp carries
// the ball.  The backward step of a body - the longest block of a tree level - is done by its 3 column lanes: each owns one column
// of the 3x3 blocks (G = D^-1 A, K = D^-1 B, the articulated A / B / C, the shifted blocks) and one component of the bias
// vectors; rows that live in other lanes come by warp shuffle (10 per body and level).  Body pass: one lane per body, 16 lanes per
// env (2 rounds for 24 bodies instead of 3 x 8).  Kinematics / root / forward pass: the column-0 lane, code shared with packed.cuh.
// Same records, same model, same oracle; results differ from packed.cuh by rounding only (a symmetric block is assembled from one
// column per lane).
#pragma once
#include "../../vid2player3d_b200/csrc/packed.cuh"

#define EPW3 2        // envs per warp
#define LPE3 16       // lanes per env
#define SLOTS3 5      // body slots per env in the tree passes (a tree depth may hold at most 5 bodies)
#define BALL_SLOT3 15 // lane of the half-warp that carries the ball

template <typename T> __device__ __forceinline__ void symcol(const T* S, int c, T* o) {  // column c of a symmetric 3x3 [xx yy zz xy xz yz]
  o[0] = c == 0 ? S[0] : (c == 1 ? S[3] : S[4]);
  o[1] = c == 0 ? S[3] : (c == 1 ? S[1] : S[5]);
  o[2] = c == 0 ? S[4] : (c == 1 ? S[5] : S[2]);
}
template <typename T> __device__ __forceinline__ T pick3(const T* v, int i) { return i == 0 ? v[0] : (i == 1 ? v[1] : v[2]); }
template <typename T> __device__ __forceinline__ T dot3(const T* a, const T* b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }

// Backward step of dynamic non-root body b, column c of 3 (every lane of the warp calls this - it shuffles - lanes without a body
// pass live = false and work on the root's record, results unused).  l1 / l2: the lanes that hold columns (c+1)%3 and (c+2)%3.
// Outputs, already shifted to the parent's origin: column c of A', B', C', component c of the bias (bn, bf).
template <typename T>
__device__ __forceinline__ void pk_backward3(const DevBlob& B, T* env, int b, bool live, int c, int l1, int l2, T* oA, T* oB, T* oC, T& obn,
                                             T& obf) {
  T* rec = env + RIX(B, b) * REC;
  T ab[R_AB], rzu[12], E[6];   // A[6] Bm[9] C[6] bn[3] bf[3] | r[3] zeta_a[3] zeta_l[3] u[3]
  ldr<R_A, R_AB>(rec, ab); ldr<R_R, 12>(rec, rzu); ldr<R_E, 6>(rec, E);
  const T *A = ab, *Bm = ab + 6, *C = ab + 15, *bn = ab + 21, *bf = ab + 24, *r = rzu, *za = rzu + 3, *zl = rzu + 6;
  T D[6], Dinv[6], ub[3];
#pragma unroll
  for (int k = 0; k < 6; k++) D[k] = A[k] + E[k];
  sym_inv(D, Dinv);
#pragma unroll
  for (int k = 0; k < 3; k++) ub[k] = rzu[9 + k] - bn[k];
  T Ac[3], Bc[3], Cc[3], g3[3], k3[3], t3[3], aA[3], aB[3], aC[3];
  symcol(A, c, Ac);
  Bc[0] = pick3(Bm, c); Bc[1] = pick3(Bm + 3, c); Bc[2] = pick3(Bm + 6, c);
  symcol(C, c, Cc);
  sym_mv(Dinv, Ac, g3);
  sym_mv(Dinv, Bc, k3);
  sym_mv(A, g3, t3);
#pragma unroll
  for (int k = 0; k < 3; k++) aA[k] = Ac[k] - t3[k];
  sym_mv(A, k3, t3);
#pragma unroll
  for (int k = 0; k < 3; k++) aB[k] = Bc[k] - t3[k];
  mtv3(Bm, k3, t3);
#pragma unroll
  for (int k = 0; k < 3; k++) aC[k] = Cc[k] - t3[k];
  // bias: component c of  an = bn + aA za + aB zl + A s,  af = bf + aB^T za + aC zl + Bm^T s   (s = D^-1 (u - bn))
  T s3[3], tz[3], zz[3];
  sym_mv(Dinv, ub, s3);
  mv3(Bm, zl, tz);
  sym_mv(Dinv, tz, zz);
  const T an = pick3(bn, c) + dot3(aA, za) + (pick3(tz, c) - dot3(Ac, zz)) + dot3(Ac, s3);
  const T af = pick3(bf, c) + dot3(aB, za) + dot3(aC, zl) + dot3(Bc, s3);
  // shift to the parent's origin (r = p - p_parent):  B' = aB + [r]x aC,  A' = aA + [r]x B'^T - aB [r]x,  C' = aC
  T rxc[3], Bp[3];
  cross3(r, aC, rxc);
#pragma unroll
  for (int k = 0; k < 3; k++) Bp[k] = aB[k] + rxc[k];
  const int c1 = c == 2 ? 0 : c + 1, c2 = c == 0 ? 2 : c - 1;   // (c+1)%3, (c+2)%3
  // columns c1, c2 of aB (for aB [r]x e_c = aB[:,c1] r[c2] - aB[:,c2] r[c1])
  T x1[3], x2[3];
#pragma unroll
  for (int k = 0; k < 3; k++) { x1[k] = __shfl_sync(FULL, aB[k], l1); x2[k] = __shfl_sync(FULL, aB[k], l2); }
  // row c of B': element c of the columns held by l1 (column c1) and l2 (column c2): at round d a lane offers element (c - d) % 3
  const T off1 = pick3(Bp, c2), off2 = pick3(Bp, c1);          // (c-1)%3 = c2, (c-2)%3 = c1
  const T in1 = __shfl_sync(FULL, off1, l1), in2 = __shfl_sync(FULL, off2, l2);
  T brow[3];
  brow[0] = c == 0 ? Bp[0] : (c1 == 0 ? in1 : in2);
  brow[1] = c == 1 ? Bp[1] : (c1 == 1 ? in1 : in2);
  brow[2] = c == 2 ? Bp[2] : (c1 == 2 ? in1 : in2);
  T rxb[3];
  cross3(r, brow, rxb);
  const T r1 = pick3(r, c1), r2 = pick3(r, c2);
#pragma unroll
  for (int k = 0; k < 3; k++) { oA[k] = aA[k] + rxb[k] - (x1[k] * r2 - x2[k] * r1); oB[k] = Bp[k]; oC[k] = aC[k]; }
  // r x af: components c1, c2 of af from the other two lanes
  const T af1 = __shfl_sync(FULL, af, l1), af2 = __shfl_sync(FULL, af, l2);
  obn = an + (r1 * af2 - r2 * af1);
  obf = af;
  // D^-1 and u - bn are what the forward pass reads.  Stored after the shuffles: every lane of the triple has consumed E and u by then.
  if (live && c == 0) { str<R_E, 6>(rec, Dinv); str<R_U, 3>(rec, ub); }
}

// add column c of a child's shifted blocks to the parent's record (each lane of the triple owns disjoint entries)
template <typename T>
__device__ __forceinline__ void pk_accumulate3(T* pr, int c, const T* oA, const T* oB, const T* oC, T obn, T obf) {
  if (c == 0) {
    pr[R_A + 0] += oA[0]; pr[R_A + 3] += oA[1]; pr[R_A + 4] += oA[2];
    pr[R_C + 0] += oC[0]; pr[R_C + 3] += oC[1]; pr[R_C + 4] += oC[2];
  } else if (c == 1) {
    pr[R_A + 1] += oA[1]; pr[R_A + 5] += oA[2];
    pr[R_C + 1] += oC[1]; pr[R_C + 5] += oC[2];
  } else {
    pr[R_A + 2] += oA[2];
    pr[R_C + 2] += oC[2];
  }
  pr[R_BM + c] += oB[0]; pr[R_BM + 3 + c] += oB[1]; pr[R_BM + 6 + c] += oB[2];
  pr[R_BN + c] += obn;
  pr[R_BF + c] += obf;
}

// One control step for the warp's EPW3 envs.  wrec: the warp's records; valid: this lane's env exists.
template <typename T>
__device__ __forceinline__ void control_step_packed3(const DevBlob& B, const float* verts, const PhysCfg<T>& c, T* wrec, int lane, bool valid,
                                                     Ball<T>& ball, bool /*cta_sync*/) {
  const b200_model_t& M = B.m;
  const int g = lane >> 4, u = lane & 15;
  const int s = u / 3, col = u - 3 * s;
  const bool tree = valid && u < 15;                  // lanes that take part in the tree passes
  const bool lead = tree && col == 0;                 // the lane that runs the single-lane phases of its body slot
  const int base = (lane & 16) + 3 * s;               // first lane of my column triple
  const int l1 = (base + (col == 2 ? 0 : col + 1)) & 31, l2 = (base + (col == 0 ? 2 : col - 1)) & 31;
  T* env = wrec + g * ENV_STRIDE;
  const int nb = M.nb;
  T pd[PK_PD_SLOTS][3];   // PD targets of my body-pass bodies (b = rr * 16 + u, rr = 0, 1)
  pk_pd_take<T, LPE3>(B, env, u, valid, pd);
  for (int d = 1; d <= M.max_depth; d++) {
    const int b = lead ? B.t.lvl_all[d][s] : -1;
    if (b >= 0) pk_fk<T, true>(B, env, b);
    __syncwarp();
  }
  for (int sim = 0; sim < c.cfi; sim++) {
    if (c.has_ball && valid && u == BALL_SLOT3) {
      ball_aero<T>(ball.v, ball.w, c.spin_scale, ball.fa);
      const T thr = c.substeps > 2 ? c.bR * T(6) : c.bR * T(4);
      if (!ball.has_bounce && ball.p[2] <= thr) {
        ball.has_bounce = 1; ball.bounce_now = 1;
        ball.bpos[0] = ball.p[0]; ball.bpos[1] = ball.p[1]; ball.bpos[2] = ball.p[2];
      }
    }
    for (int sub = 0; sub < c.substeps; sub++) {
      // 1. per-body inertia / bias / contacts / joint drive: one lane per body, 16 lanes per env
      for (int rr = 0; rr * LPE3 < nb; rr++) {
        const int b = rr * LPE3 + u;
        if (valid && b < nb && !M.fixed[b]) {
          T pdb[3];
          pk_pd_pick<T>(pd, rr, pdb);
          pk_body<T>(B, verts, c, env, b, sim == 0, pdb);
        }
      }
      __syncwarp();
      // 2. articulated inertia, leaves -> root: 3 lanes per body
      for (int d = M.max_depth; d >= 1; d--) {
        const int b = tree ? B.t.lvl_dyn[d][s] : -1;
        T oA[3], oB[3], oC[3], obn, obf;
        pk_backward3<T>(B, env, b >= 0 ? b : 0, b >= 0, col, l1, l2, oA, oB, oC, obn, obf);
        __syncwarp();   // every triple has read its own record before a sibling's triple adds to the shared parent ... (parents are one level up: no hazard; keeps the phases aligned)
        const int rounds = B.t.maxch[d - 1];
        for (int cr = 0; cr < rounds; cr++) {
          if (b >= 0 && B.t.child_rank[b] == cr) pk_accumulate3<T>(env + RIX(B, M.parent[b]) * REC, col, oA, oB, oC, obn, obf);
          __syncwarp();
        }
      }
      // 3. root acceleration next to the ball, then the root is integrated
      if (c.has_ball && valid && u == BALL_SLOT3) {
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
        if (c.ball_body) pk_ball_contacts_extra<T>(B, verts, c, env, ball);
        T* ext = env + ENV_EXT;
#pragma unroll
        for (int k = 0; k < 3; k++) { ext[6 + k] = ball.rF[k]; ext[9 + k] = ball.rX[k]; }
      }
      if (valid && u == 0) pk_root<T>(c, env);
      if (c.ball_body) __syncwarp();   // the extra ball contacts read the root's pose: integrate it only after the ball lane is done
      if (valid && u == 0) pk_root_integrate<T>(c, env);
      __syncwarp();
      // 4. root -> leaves: accelerations + joint integration of a body, then at once its kinematics for the next substep
      for (int d = 1; d <= M.max_depth; d++) {
        const int b = lead ? B.t.lvl_all[d][s] : -1;
        if (b >= 0) {
          if (!M.fixed[b]) {
            T qn[4], wt[3];
            pk_forward<T>(B, c, env, b, qn, wt);
            pk_fk<T, true, true>(B, env, b, qn, wt);
          } else {
            pk_fk<T, true>(B, env, b);
          }
        }
        __syncwarp();
      }
    }
  }
  pk_pd_park<T, LPE3>(B, env, u, valid, pd);
}
