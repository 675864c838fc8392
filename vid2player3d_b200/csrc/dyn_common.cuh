// dyn_common.cuh - device code shared by every form of the articulated step (b200env.cu: lane-per-body kernel; packed.cuh /
// packed3.cuh: envs packed into a warp) and by the offline ball generators: constant-block layout, small math, per-lane state,
// the tennis-ball model, ground contact of a convex hull.  Plain templated C++ with __device__ qualifiers only - it also compiles
// as host code under tests/emu/cuda_compat.h, which is how the packed kernels are checked lane by lane on the CPU
// (tests/emu/emu_packed.cpp runs one host thread per lane, __syncwarp() = a barrier).
#pragma once
#include <math.h>
#include <stdint.h>
#include <string.h>

#include "../../include/b200env.h"

#ifndef FULL
#define FULL 0xffffffffu
#endif
#define MAX_CHILD 4
#define MAX_LEVELS 16
// ------------------------------------------------------------------------------------------
// device-side constant block: header | tree tables | hull vertices   (all 16-byte multiples)
#define PK_SLOTS 8
struct DevTree {
  int32_t child[B200_MAX_BODIES][MAX_CHILD];  // dynamic (non-welded) children, -1 padded
  int32_t maxch[MAX_LEVELS];                  // max #children over the bodies of each depth
  // packed (4 envs / warp) variant: the s-th body of every tree depth, and each body's rank among its siblings
  int32_t lvl_all[MAX_LEVELS][PK_SLOTS];      // all bodies of the depth (kinematics), -1 padded
  int32_t lvl_dyn[MAX_LEVELS][PK_SLOTS];      // non-welded bodies of the depth (dynamics), -1 padded
  int32_t child_rank[B200_MAX_BODIES];
  int32_t rix[B200_MAX_BODIES];               // record index of a body in the packed kernel's shared-memory layout = breadth-first rank
  float vrho[B200_MAX_BODIES];                // ball-body contact: radius of the sphere every hull vertex of the body stands for (hull_vertex_radius)
  // exact ball / hull contact (b200env_set_hull_faces): faces of every body's convex hull in global memory - planes [nb][face_tmax] float4
  // (outward unit normal, offset), tris [nb][face_tmax] 4 x uint8 (vertex indices, outward winding) - and their number per body (0 = none)
  const float* face_planes;
  const unsigned char* face_tris;
  int32_t face_tmax, face_pad_[3];
  int32_t ntris[B200_MAX_BODIES];
  // packed_t.cuh (one-wave kernel: lane-private fields in thread-local memory): every dynamic body has a fixed owner lane slot and one
  // of three column blocks of its lane's private store; the bodies of one tree depth share a block (one warp-uniform block per level pass)
  int8_t pt_blk[B200_MAX_BODIES];             // column block of a dynamic body, -1: welded
  int8_t pt_slot[B200_MAX_BODIES];            // lane slot of the body in every pass
  int8_t pt_body[3][PK_SLOTS];                // body pass: the dynamic body of (block, slot), -1 padded
  int8_t pt_lvl[MAX_LEVELS][PK_SLOTS];        // level passes: body of that depth at its slot (welded ones included), -1 padded
  int8_t pt_lblk[MAX_LEVELS];                 // block of the depth's dynamic bodies, -1: none
  int8_t pt_mbox[B200_MAX_BODIES];            // mailbox entry of a dynamic body = its rank among the dynamic bodies of its depth
  int32_t pt_ok, pt_nmbox, pt_pad_[4];        // pt_ok: the tree fits (3 blocks x 8 slots); pt_nmbox: mailbox entries per env
  // ball-body contact: bounding sphere of every hull about the centroid of its vertices (body frame: centre xyz, radius) - the reach
  // test in front of the exact hull query.  The sphere about the body ORIGIN (b200_model_t::radius, what the ground contact uses) is
  // up to a limb's length for a hull that starts at its joint; a ball near a lying player passed it for ten bodies at a time.
  // Pruning only: a ball outside this sphere + its radius is outside the hull + its radius.
  float bs[B200_MAX_BODIES][4];
};
struct DevBlob {
  b200_model_t m;
  DevTree t;
  // float verts[nb][3][vmax] follows (SoA per body: x | y | z, see contact_hull)
};
static_assert(sizeof(b200_model_t) % 16 == 0, "model block must be a 16-byte multiple for the bulk copy");
static_assert(sizeof(DevBlob) % 16 == 0, "blob header must be a 16-byte multiple");

// host side: owner slots / column blocks of packed_t.cuh.  The dynamic bodies of every tree depth go into ONE of three blocks of
// PK_SLOTS slots (exhaustive search over the 3^depths assignments, first fit); inside a block slots are handed out in depth order.
// A welded body needs a lane at its depth but no column block: it takes a slot its depth does not use.
static inline void build_pt_tables(const b200_model_t* model, DevTree& t) {
  t.pt_ok = 0; t.pt_nmbox = 0;
  for (int b = 0; b < B200_MAX_BODIES; b++) { t.pt_blk[b] = -1; t.pt_slot[b] = -1; t.pt_mbox[b] = -1; }
  for (int k = 0; k < 3; k++) for (int s = 0; s < PK_SLOTS; s++) t.pt_body[k][s] = -1;
  for (int d = 0; d < MAX_LEVELS; d++) { t.pt_lblk[d] = -1; for (int s = 0; s < PK_SLOTS; s++) t.pt_lvl[d][s] = -1; }
  int ndyn[MAX_LEVELS] = {0}, nall[MAX_LEVELS] = {0}, maxd = 0;
  for (int b = 0; b < model->nb; b++) {
    const int d = model->depth[b];
    if (d < 0 || d >= MAX_LEVELS) return;
    nall[d]++;
    if (!model->fixed[b]) ndyn[d]++;
    if (d > maxd) maxd = d;
  }
  for (int d = 0; d <= maxd; d++) if (nall[d] > PK_SLOTS) return;
  int asg[MAX_LEVELS] = {0}, found = 0;
  long total = 1;
  for (int d = 0; d <= maxd; d++) total *= 3;
  for (long code = 0; code < total && !found; code++) {
    int fill[3] = {0, 0, 0};
    long c = code;
    bool ok = true;
    for (int d = 0; d <= maxd; d++) { asg[d] = (int)(c % 3); c /= 3; fill[asg[d]] += ndyn[d]; if (fill[asg[d]] > PK_SLOTS) { ok = false; break; } }
    if (ok) found = 1;
  }
  if (!found) return;
  int fill[3] = {0, 0, 0};
  for (int d = 0; d <= maxd; d++) {
    unsigned used = 0;
    int nm = 0;
    for (int b = 0; b < model->nb; b++) {
      if (model->depth[b] != d || model->fixed[b]) continue;
      const int k = asg[d], s = fill[k]++;
      t.pt_blk[b] = (int8_t)k; t.pt_slot[b] = (int8_t)s; t.pt_body[k][s] = (int8_t)b; t.pt_lvl[d][s] = (int8_t)b; t.pt_mbox[b] = (int8_t)nm++;
      t.pt_lblk[d] = (int8_t)k;
      used |= 1u << s;
    }
    if (d >= 1 && nm > t.pt_nmbox) t.pt_nmbox = nm;
    for (int b = 0; b < model->nb; b++) {
      if (model->depth[b] != d || !model->fixed[b]) continue;
      int s = 0;
      while (s < PK_SLOTS && ((used >> s) & 1u)) s++;
      if (s == PK_SLOTS) return;
      t.pt_slot[b] = (int8_t)s; t.pt_lvl[d][s] = (int8_t)b;
      used |= 1u << s;
    }
  }
  t.pt_ok = 1;
}

// host side: tree tables of a model (used by b200env_create and by the CPU lane emulator).  Returns 0, -1 (bodies not in
// topological order) or -2 (too many children); *slots_ok = 0 when a tree depth has more bodies than the packed kernels have slots.
static inline int build_dev_blob(const b200_model_t* model, DevBlob& hb, int* slots_ok) {
  memset(&hb, 0, sizeof(hb));
  hb.m = *model;
  *slots_ok = 1;
  for (int b = 0; b < B200_MAX_BODIES; b++)
    for (int c = 0; c < MAX_CHILD; c++) hb.t.child[b][c] = -1;
  int cnt[B200_MAX_BODIES] = {0};
  for (int b = 1; b < model->nb; b++) {
    if (model->fixed[b]) continue;
    int p = model->parent[b];
    if (p < 0 || p >= b) return -1;
    if (cnt[p] >= MAX_CHILD) return -2;
    hb.t.child[p][cnt[p]++] = b;
  }
  for (int b = 0; b < model->nb; b++)
    if (cnt[b] > hb.t.maxch[model->depth[b]]) hb.t.maxch[model->depth[b]] = cnt[b];
  int na[MAX_LEVELS] = {0}, ndy[MAX_LEVELS] = {0}, rk[B200_MAX_BODIES] = {0};
  for (int d = 0; d < MAX_LEVELS; d++)
    for (int k = 0; k < PK_SLOTS; k++) { hb.t.lvl_all[d][k] = -1; hb.t.lvl_dyn[d][k] = -1; }
  for (int b = 0; b < model->nb; b++) {
    const int d = model->depth[b];
    if (na[d] >= PK_SLOTS) { *slots_ok = 0; continue; }
    hb.t.lvl_all[d][na[d]++] = b;
    if (!model->fixed[b]) {
      hb.t.lvl_dyn[d][ndy[d]++] = b;
      if (b > 0) hb.t.child_rank[b] = rk[model->parent[b]]++;
    }
  }
  build_pt_tables(model, hb.t);
  int next = 0;   // breadth-first record order (packed.cuh: neighbouring lanes of a tree depth -> neighbouring records)
  for (int d = 0; d < MAX_LEVELS; d++)
    for (int b = 0; b < model->nb; b++)
      if (model->depth[b] == d) hb.t.rix[b] = next++;
  return 0;
}
// bounding spheres of the hulls about their vertex centroids (DevTree::bs); verts: AoS [nb][vmax][3] as the ABI hands them over
static inline void hull_bounding_spheres(const b200_model_t* model, const float* verts, float (*bs)[4]) {
  for (int b = 0; b < B200_MAX_BODIES; b++) bs[b][0] = bs[b][1] = bs[b][2] = bs[b][3] = 0.0f;
  for (int b = 0; b < model->nb; b++) {
    const int nv = model->nverts[b];
    if (nv < 1) continue;
    const float* v = verts + (size_t)b * model->vmax * 3;
    double c[3] = {0, 0, 0};
    for (int i = 0; i < nv; i++) for (int k = 0; k < 3; k++) c[k] += v[i * 3 + k];
    for (int k = 0; k < 3; k++) c[k] /= nv;
    const float cf[3] = {(float)c[0], (float)c[1], (float)c[2]};
    double r2 = 0;
    for (int i = 0; i < nv; i++) {
      const double dx = (double)v[i * 3] - cf[0], dy = (double)v[i * 3 + 1] - cf[1], dz = (double)v[i * 3 + 2] - cf[2];
      const double d2 = dx * dx + dy * dy + dz * dz;
      if (d2 > r2) r2 = d2;
    }
    bs[b][0] = cf[0]; bs[b][1] = cf[1]; bs[b][2] = cf[2];
    bs[b][3] = (float)(sqrt(r2) * 1.0001 + 1e-6);     // conservative against the float arithmetic of the device-side test
  }
}
// ball-body contact (b200_cfg_t::ball_body_contact): a body's hull is stood in for by spheres on its vertices; radius = half the mean
// distance of a vertex to its nearest neighbour, kept within [5 mm, 5 cm].  Same function (same float arithmetic) in oracle/physics_ref.c.
static inline void hull_vertex_radius(const b200_model_t* model, const float* verts, float* vrho) {
  for (int b = 0; b < B200_MAX_BODIES; b++) vrho[b] = 0.0f;
  for (int b = 0; b < model->nb; b++) {
    const int nv = model->nverts[b];
    if (nv < 2) continue;
    const float* v = verts + (size_t)b * model->vmax * 3;
    double sum = 0.0;
    for (int i = 0; i < nv; i++) {
      double best = 1e30;
      for (int j = 0; j < nv; j++) {
        if (j == i) continue;
        const double dx = (double)v[i * 3] - v[j * 3], dy = (double)v[i * 3 + 1] - v[j * 3 + 1], dz = (double)v[i * 3 + 2] - v[j * 3 + 2];
        const double d2 = dx * dx + dy * dy + dz * dz;
        if (d2 > 1e-12 && d2 < best) best = d2;
      }
      sum += sqrt(best);
    }
    double r = 0.5 * sum / nv;
    r = r < 0.005 ? 0.005 : (r > 0.05 ? 0.05 : r);
    vrho[b] = (float)r;
  }
}
// hull vertices AoS [nb][vmax][3] (ABI) -> SoA [nb][3][vmax] (what contact_hull reads with 128-bit loads); dst zero-initialised
static inline void verts_to_soa(const b200_model_t* model, const float* verts, float* soa) {
  for (int b = 0; b < model->nb; b++)
    for (int k = 0; k < model->nverts[b]; k++)
      for (int a = 0; a < 3; a++) soa[((size_t)b * 3 + a) * model->vmax + k] = verts[((size_t)b * model->vmax + k) * 3 + a];
}

// ------------------------------------------------------------------------------------------
// small math (templated on float / double)
#if defined(__CUDACC__)
__device__ __forceinline__ int emu_lane_id() { return (int)(threadIdx.x & 31); }
#else
static inline int emu_lane_id() { return emu_lane; }   // tests/emu/cuda_compat.h: the lane this host thread plays
#endif
template <typename T> __device__ __forceinline__ T shfl(T v, int src) { return __shfl_sync(FULL, v, src); }
template <typename T> __device__ __forceinline__ T warp_sum(T v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(FULL, v, o);
  return v;
}
// fast reciprocal / rsqrt for the float path (MUFU, ~2 ulp); exact for the double (test) path
__device__ __forceinline__ float rcp_(float x) { return __fdividef(1.0f, x); }
__device__ __forceinline__ double rcp_(double x) { return 1.0 / x; }
__device__ __forceinline__ float rsqrt_(float x) { return rsqrtf(x); }
__device__ __forceinline__ double rsqrt_(double x) { return 1.0 / sqrt(x); }
__device__ __forceinline__ float sqrt_(float x) { return x * rsqrtf(fmaxf(x, 1e-37f)); }
__device__ __forceinline__ double sqrt_(double x) { return sqrt(x); }
template <typename T> __device__ __forceinline__ void cross3(const T* a, const T* b, T* o) {
  T x = a[1] * b[2] - a[2] * b[1], y = a[2] * b[0] - a[0] * b[2], z = a[0] * b[1] - a[1] * b[0];
  o[0] = x; o[1] = y; o[2] = z;
}
template <typename T> __device__ __forceinline__ void qmul(const T* a, const T* b, T* o) {
  T x1 = a[0], y1 = a[1], z1 = a[2], w1 = a[3], x2 = b[0], y2 = b[1], z2 = b[2], w2 = b[3];
  o[0] = w1 * x2 + x1 * w2 + y1 * z2 - z1 * y2;
  o[1] = w1 * y2 - x1 * z2 + y1 * w2 + z1 * x2;
  o[2] = w1 * z2 + x1 * y2 - y1 * x2 + z1 * w2;
  o[3] = w1 * w2 - x1 * x2 - y1 * y2 - z1 * z2;
}
template <typename T> __device__ __forceinline__ void qnormalize(T* q) {
  T n = rsqrt_(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
  q[0] *= n; q[1] *= n; q[2] *= n; q[3] *= n;
}
// rotate v by unit quaternion q:  v + 2 w (qv x v) + 2 qv x (qv x v)
template <typename T> __device__ __forceinline__ void qrot(const T* q, const T* v, T* o) {
  T t[3], u[3];
  cross3(q, v, t);
  t[0] *= T(2); t[1] *= T(2); t[2] *= T(2);
  cross3(q, t, u);
  o[0] = v[0] + q[3] * t[0] + u[0];
  o[1] = v[1] + q[3] * t[1] + u[1];
  o[2] = v[2] + q[3] * t[2] + u[2];
}
template <typename T> __device__ __forceinline__ void qmat(const T* q, T* R) {  // row-major 3x3
  T x = q[0], y = q[1], z = q[2], w = q[3];
  R[0] = 1 - 2 * (y * y + z * z); R[1] = 2 * (x * y - z * w); R[2] = 2 * (x * z + y * w);
  R[3] = 2 * (x * y + z * w); R[4] = 1 - 2 * (x * x + z * z); R[5] = 2 * (y * z - x * w);
  R[6] = 2 * (x * z - y * w); R[7] = 2 * (y * z + x * w); R[8] = 1 - 2 * (x * x + y * y);
}
template <typename T> __device__ __forceinline__ void mv3(const T* R, const T* v, T* o) {
  T a = R[0] * v[0] + R[1] * v[1] + R[2] * v[2];
  T b = R[3] * v[0] + R[4] * v[1] + R[5] * v[2];
  T c = R[6] * v[0] + R[7] * v[1] + R[8] * v[2];
  o[0] = a; o[1] = b; o[2] = c;
}
template <typename T> __device__ __forceinline__ void mtv3(const T* R, const T* v, T* o) {
  T a = R[0] * v[0] + R[3] * v[1] + R[6] * v[2];
  T b = R[1] * v[0] + R[4] * v[1] + R[7] * v[2];
  T c = R[2] * v[0] + R[5] * v[1] + R[8] * v[2];
  o[0] = a; o[1] = b; o[2] = c;
}
// rotation vector -> quaternion (exact exponential)
template <typename T> __device__ __forceinline__ void qexp(const T* v, T* q) {
  T a2 = v[0] * v[0] + v[1] * v[1] + v[2] * v[2];
  T a = sqrt(a2), s;
  if (a < T(1e-6)) s = T(0.5) - a2 / T(48); else s = sin(T(0.5) * a) / a;
  q[0] = s * v[0]; q[1] = s * v[1]; q[2] = s * v[2]; q[3] = cos(T(0.5) * a);
}
// exponential for the per-substep increments (|v| = h*|omega| <= h*max_ang_vel < 1 rad): even-power series,
// truncation error < 2e-9 for |v| <= 2; the double path keeps sin/cos
__device__ __forceinline__ void qexp_small(const float* v, float* q) {
  const float a2 = v[0] * v[0] + v[1] * v[1] + v[2] * v[2];
  if (a2 > 4.0f) { qexp(v, q); return; }
  const float s = 0.5f + a2 * (-1.0f / 48.0f + a2 * (1.0f / 3840.0f + a2 * (-1.0f / 645120.0f + a2 * (1.0f / 185794560.0f))));
  const float c = 1.0f + a2 * (-0.125f + a2 * (1.0f / 384.0f + a2 * (-1.0f / 46080.0f + a2 * (1.0f / 10321920.0f + a2 * (-1.0f / 3715891200.0f)))));
  q[0] = s * v[0]; q[1] = s * v[1]; q[2] = s * v[2]; q[3] = c;
}
__device__ __forceinline__ void qexp_small(const double* v, double* q) { qexp(v, q); }
// quaternion -> rotation vector, angle in [0, pi]
template <typename T> __device__ __forceinline__ void qlog(const T* qi, T* v) {
  T sg = qi[3] < T(0) ? T(-1) : T(1);
  T x = sg * qi[0], y = sg * qi[1], z = sg * qi[2], w = sg * qi[3];
  T s2 = x * x + y * y + z * z;
  T s = sqrt_(s2), f;
  if (s < T(1e-6)) f = T(2) + s2 * T(1.0 / 3.0); else f = T(2) * atan2(s, w) * rcp_(s);
  v[0] = f * x; v[1] = f * y; v[2] = f * z;
}
// symmetric 3x3 stored as [xx, yy, zz, xy, xz, yz]
template <typename T> __device__ __forceinline__ void sym_mv(const T* S, const T* v, T* o) {
  T a = S[0] * v[0] + S[3] * v[1] + S[4] * v[2];
  T b = S[3] * v[0] + S[1] * v[1] + S[5] * v[2];
  T c = S[4] * v[0] + S[5] * v[1] + S[2] * v[2];
  o[0] = a; o[1] = b; o[2] = c;
}
template <typename T> __device__ __forceinline__ void sym_inv(const T* S, T* O) {
  T c00 = S[1] * S[2] - S[5] * S[5];
  T c01 = S[5] * S[4] - S[3] * S[2];
  T c02 = S[3] * S[5] - S[1] * S[4];
  T det = S[0] * c00 + S[3] * c01 + S[4] * c02;
  T id = rcp_(det);
  O[0] = c00 * id;
  O[1] = (S[0] * S[2] - S[4] * S[4]) * id;
  O[2] = (S[0] * S[1] - S[3] * S[3]) * id;
  O[3] = c01 * id;
  O[4] = c02 * id;
  O[5] = (S[3] * S[4] - S[0] * S[5]) * id;
}
// full 3x3 (row-major) from symmetric
template <typename T> __device__ __forceinline__ void sym_full(const T* S, T* F) {
  F[0] = S[0]; F[1] = S[3]; F[2] = S[4];
  F[3] = S[3]; F[4] = S[1]; F[5] = S[5];
  F[6] = S[4]; F[7] = S[5]; F[8] = S[2];
}

// ------------------------------------------------------------------------------------------
// per-lane (per-body) state
template <typename T> struct Lane {
  T Q[4], p[3], w[3], v[3];  // world pose and velocity of the body origin
  T qj[4], wt[3];            // joint rotation (child in parent) and joint velocity (child frame)
};
// the body at rest: zero vectors, identity rotations (what a lane without a body, or without a joint, holds)
template <typename T> __device__ __forceinline__ void lane_rest(Lane<T>& L) {
#pragma unroll
  for (int k = 0; k < 4; k++) { L.Q[k] = 0; L.qj[k] = 0; }
  L.Q[3] = 1; L.qj[3] = 1;
#pragma unroll
  for (int k = 0; k < 3; k++) { L.p[k] = 0; L.w[k] = 0; L.v[k] = 0; L.wt[k] = 0; }
}
struct LaneConst {
  int par, depth, dof0;
  int rix;           // packed kernels: the body's record index (DevTree::rix); set by the kernel after lane_const()
  bool active, dyn;  // dyn: takes part in the dynamics (not welded)
};

template <typename T> struct PhysCfg {
  T h, gz, kn, cn, mu, vs, damp, wmax, limk, limc;
  int substeps, cfi;
  // tennis ball (vid2player): lane BALL_LANE integrates it next to the humanoid
  int has_ball, racket_body, wrist_body;
  T bm, bI, bR, spin_scale, eg, mug, er, mur, vth, hc[3], hh, hr, hq[4];
  int ball_body;        // optional ball contacts with the bodies / the racket handle (b200_cfg_t::ball_body_contact)
  T eb, mub, hdl[7];    // their restitution / friction; handle capsule p0[3] p1[3] radius in the racket frame
};
#ifndef ABL
#define ABL 0   // tools/ablate.sh: 1 no physics, 2 epilogue = state write-back only, 3 no reward block, 4 no MoCap sample / targets, 5 no obs
#endif
#define BALL_LANE 31
// ball state held by lane BALL_LANE (DESIGN.md 3b; float64 restatement: oracle/physics_ref.c::ball_substep)
template <typename T> struct Ball {
  T p[3], v[3], w[3];   // position, linear and angular velocity (world)
  T fa[3];              // aerodynamic force, refreshed once per sim step like the reference (humanoid_smpl_im_mvae.py:752-756)
  T rF[3], rX[3];       // reaction force on the racket from the last impact (applied to the wrist link next substep) and its point
  int hits;             // racket impacts so far
  int has_bounce, bounce_now;
  T bpos[3];
};
template <typename T> __device__ __forceinline__ PhysCfg<T> make_phys_cfg(const b200_cfg_t& c) {
  PhysCfg<T> p;
  p.h = T(c.sim_dt) / T(c.substeps);
  p.gz = T(c.gravity_z); p.kn = T(c.contact_kn); p.cn = T(c.contact_cn); p.mu = T(c.friction_mu);
  p.vs = T(c.friction_vs); p.damp = T(1) - p.h * T(c.ang_damping); p.wmax = T(c.max_ang_vel);
  p.limk = T(c.limit_k); p.limc = T(c.limit_c);
  p.substeps = c.substeps; p.cfi = c.control_freq_inv;
  p.has_ball = c.has_ball; p.racket_body = c.racket_body; p.wrist_body = 0;
  p.bm = T(c.ball_mass); p.bI = T(c.ball_inertia); p.bR = T(c.ball_radius); p.spin_scale = T(c.spin_scale);
  p.eg = T(c.ball_e_ground); p.mug = T(c.ball_mu_ground); p.er = T(c.ball_e_racket); p.mur = T(c.ball_mu_racket);
  p.vth = T(c.bounce_threshold_velocity);
  p.hc[0] = T(c.racket_head_center[0]); p.hc[1] = T(c.racket_head_center[1]); p.hc[2] = T(c.racket_head_center[2]);
  p.hh = T(c.racket_head_halfthick); p.hr = T(c.racket_head_radius);
#pragma unroll
  for (int k = 0; k < 4; k++) p.hq[k] = T(c.racket_head_quat[k]);
  p.ball_body = c.has_ball && c.ball_body_contact;
  p.eb = T(c.ball_e_body); p.mub = T(c.ball_mu_body);
#pragma unroll
  for (int k = 0; k < 7; k++) p.hdl[k] = T(c.racket_handle[k]);
  return p;
}

// forward kinematics, level by level: fills Q,p,w,v (world) of every lane from the root state and
// the joint state.  Optionally returns r = p - p_parent and the velocity-product terms zeta.
#ifndef LEVEL_SYNC
#define LEVEL_SYNC 0  // 1: CTA barrier at every tree level (keeps all warps of the CTA in the same code region: I-cache sharing)
#endif
template <typename T, bool WITH_ZETA>
__device__ __forceinline__ void fk_pass(const b200_model_t& M, const LaneConst& lc, int lane, Lane<T>& L, T* r, T* zeta,
                                        bool lsync = false) {
  for (int d = 1; d <= M.max_depth; d++) {
    if (LEVEL_SYNC && lsync) __syncthreads();
    T pQ[4], pp[3], pw[3], pv[3];
#pragma unroll
    for (int k = 0; k < 4; k++) pQ[k] = shfl(L.Q[k], lc.par);
#pragma unroll
    for (int k = 0; k < 3; k++) { pp[k] = shfl(L.p[k], lc.par); pw[k] = shfl(L.w[k], lc.par); pv[k] = shfl(L.v[k], lc.par); }
    if (lc.active && lc.depth == d) {
      T off[3] = {T(M.offset[lane][0]), T(M.offset[lane][1]), T(M.offset[lane][2])};
      T rr[3], wxr[3];
      qrot(pQ, off, rr);
      cross3(pw, rr, wxr);
#pragma unroll
      for (int k = 0; k < 3; k++) { L.p[k] = pp[k] + rr[k]; L.v[k] = pv[k] + wxr[k]; }
      if (WITH_ZETA) { r[0] = rr[0]; r[1] = rr[1]; r[2] = rr[2]; }
      if (!lc.dyn) {
#pragma unroll
        for (int k = 0; k < 4; k++) L.Q[k] = pQ[k];
#pragma unroll
        for (int k = 0; k < 3; k++) L.w[k] = pw[k];
      } else {
        qmul(pQ, L.qj, L.Q);
        qnormalize(L.Q);
        T wj[3];
        qrot(L.Q, L.wt, wj);
#pragma unroll
        for (int k = 0; k < 3; k++) L.w[k] = pw[k] + wj[k];
        if (WITH_ZETA) { cross3(pw, wj, zeta); cross3(pw, wxr, zeta + 3); }
      }
    }
  }
}


// drag + Magnus lift on the ball (apply_external_force_to_ball, humanoid_smpl_im_mvae.py:711-739; constants tennis_ball.py:15-37)
template <typename T> __device__ __forceinline__ void ball_aero(const T* vel, const T* angvel, T spin_scale, T* force) {
  const T KF = T(0.0019462794807519486), CD = T(0.55);
  T vs = sqrt_(vel[0] * vel[0] + vel[1] * vel[1] + vel[2] * vel[2]);
  if (vs == T(0)) vs += T(1);
  const T iv = rcp_(vs);
  const T vn[3] = {vel[0] * iv, vel[1] * iv, vel[2] * iv};
  const T vt[3] = {-vn[1], vn[0], T(0)};  // vn x (0,0,-1)
  const T vspin = sqrt_(angvel[0] * angvel[0] + angvel[1] * angvel[1] + angvel[2] * angvel[2]) * T(0.15915494309189535);
  T cl = rcp_(T(2) + fabs(vs * rcp_(vspin * spin_scale + T(1e-6))));
  cl = vspin > T(0) ? -cl : cl;
  const T cx = vt[1] * vn[2] - vt[2] * vn[1], cy = vt[2] * vn[0] - vt[0] * vn[2], cz = vt[0] * vn[1] - vt[1] * vn[0];
  const T kd = -KF * CD * vs, kl = -KF * cl * vs * vs;
  force[0] = kd * vel[0] + kl * cx; force[1] = kd * vel[1] + kl * cy; force[2] = kd * vel[2] + kl * cz;
}
// impulse on a sphere at contact normal n (pointing from the obstacle into the ball), obstacle point velocity vo:
// restitution e on the normal part, Coulomb friction mu capped at the sticking impulse (spin coupled through I).
template <typename T>
__device__ __forceinline__ void ball_impulse(const PhysCfg<T>& c, Ball<T>& B, const T* n, const T* vo, T e, T mu, T* J) {
  // contact point on the ball: -R n ; u = v + w x (-R n) - vo
  T rn[3] = {-c.bR * n[0], -c.bR * n[1], -c.bR * n[2]}, wxr[3];
  cross3(B.w, rn, wxr);
  T u[3] = {B.v[0] + wxr[0] - vo[0], B.v[1] + wxr[1] - vo[1], B.v[2] + wxr[2] - vo[2]};
  const T un = u[0] * n[0] + u[1] * n[1] + u[2] * n[2];
  J[0] = J[1] = J[2] = T(0);
  if (!(un < T(0))) return;
  const T jn = (-un > c.vth ? (T(1) + e) : T(1)) * (-un) * c.bm;
  T ut[3] = {u[0] - un * n[0], u[1] - un * n[1], u[2] - un * n[2]};
  const T utn = sqrt_(ut[0] * ut[0] + ut[1] * ut[1] + ut[2] * ut[2]);
  T jt = T(0);
  if (utn > T(1e-9)) {
    const T stick = c.bm * utn * rcp_(T(1) + c.bm * c.bR * c.bR * rcp_(c.bI));
    jt = mu * jn < stick ? mu * jn : stick;
    const T iu = rcp_(utn);
    ut[0] *= iu; ut[1] *= iu; ut[2] *= iu;
  }
#pragma unroll
  for (int k = 0; k < 3; k++) J[k] = jn * n[k] - jt * ut[k];
  T rxJ[3];
  cross3(rn, J, rxJ);
  const T im = rcp_(c.bm), iI = rcp_(c.bI);
#pragma unroll
  for (int k = 0; k < 3; k++) { B.v[k] += J[k] * im; B.w[k] += rxJ[k] * iI; }
}
// one substep of the ball: gravity + aero, swept test against the racket head (a cylinder of half thickness hh and
// radius hr centred at hc in the racket frame; pose/velocity of the racket at the START of the substep), ground bounce.
template <typename T>
__device__ __forceinline__ void ball_substep(const PhysCfg<T>& c, Ball<T>& B, bool has_racket, const T* rQ, const T* rp, const T* rv, const T* rw) {
  const T im = rcp_(c.bm);
  B.v[0] += c.h * B.fa[0] * im; B.v[1] += c.h * B.fa[1] * im; B.v[2] += c.h * (c.gz + B.fa[2] * im);
  B.rF[0] = B.rF[1] = B.rF[2] = T(0);
  T thit = T(-1), nl = T(0);
  if (has_racket) {
    T d[3] = {B.p[0] - rp[0], B.p[1] - rp[1], B.p[2] - rp[2]}, wxd[3];
    cross3(rw, d, wxd);
    T vrel_w[3] = {B.v[0] - rv[0] - wxd[0], B.v[1] - rv[1] - wxd[1], B.v[2] - rv[2] - wxd[2]};
    T hQ[4];
    qmul(rQ, c.hq, hQ);   // head frame in the world (string-bed normal = its +y)
    T cq[4] = {-hQ[0], -hQ[1], -hQ[2], hQ[3]}, d0[3], vr[3];
    qrot(cq, d, d0);
    qrot(cq, vrel_w, vr);
    d0[0] -= c.hc[0]; d0[1] -= c.hc[1]; d0[2] -= c.hc[2];
    const T H = c.hh + c.bR, Rad = c.hr + c.bR;
    if (fabs(d0[1]) < H) {
      if (d0[0] * d0[0] + d0[2] * d0[2] < Rad * Rad) { thit = T(0); nl = d0[1] >= T(0) ? T(1) : T(-1); }
    } else {
      T t = T(-1);
      if (d0[1] >= H && vr[1] < T(0)) t = (d0[1] - H) * rcp_(-vr[1]);
      else if (d0[1] <= -H && vr[1] > T(0)) t = (-H - d0[1]) * rcp_(vr[1]);
      if (t >= T(0) && t <= c.h) {
        const T hx = d0[0] + t * vr[0], hz = d0[2] + t * vr[2];
        if (hx * hx + hz * hz < Rad * Rad) { thit = t; nl = d0[1] >= T(0) ? T(1) : T(-1); }
      }
    }
    if (thit >= T(0)) {
      const T ny[3] = {T(0), nl, T(0)};
      T n[3], J[3], vo[3];
      qrot(hQ, ny, n);
      T xc[3] = {B.p[0] + thit * B.v[0] - c.bR * n[0], B.p[1] + thit * B.v[1] - c.bR * n[1], B.p[2] + thit * B.v[2] - c.bR * n[2]};
      T dx[3] = {xc[0] - rp[0], xc[1] - rp[1], xc[2] - rp[2]}, wxx[3];
      cross3(rw, dx, wxx);
      vo[0] = rv[0] + wxx[0]; vo[1] = rv[1] + wxx[1]; vo[2] = rv[2] + wxx[2];
      const T vb[3] = {B.v[0], B.v[1], B.v[2]};
      ball_impulse(c, B, n, vo, c.er, c.mur, J);
      if (J[0] != T(0) || J[1] != T(0) || J[2] != T(0)) {
        const T ih = rcp_(c.h);
#pragma unroll
        for (int k = 0; k < 3; k++) { B.rF[k] = -J[k] * ih; B.rX[k] = xc[k]; B.p[k] += thit * vb[k] + (c.h - thit) * B.v[k]; }
        B.hits++;
      } else {
        thit = T(-1);
      }
    }
  }
  if (thit < T(0)) {
#pragma unroll
    for (int k = 0; k < 3; k++) B.p[k] += c.h * B.v[k];
  }
  if (B.p[2] < c.bR && B.v[2] < T(0)) {  // ground
    const T n[3] = {T(0), T(0), T(1)}, vo[3] = {T(0), T(0), T(0)};
    T J[3];
    ball_impulse(c, B, n, vo, c.eg, c.mug, J);
    B.p[2] = c.bR;
  }
}

// One substep of length h (DESIGN.md 3; float64 restatement: oracle/physics_ref.c::substep).
// Ground contact of one body's convex-hull vertices against z = 0, implicit in the velocity (DESIGN.md 3).
// vb: the body's vertices in the blob, SoA  x[vmax] | y[vmax] | z[vmax]  (vmax % 4 == 0, 16-byte aligned, padding = 0).
// Pass 1 tests four vertices per iteration (3 LDS.128, independent FMAs) and records the penetrating ones in a bit mask;
// pass 2 visits only those, in ascending vertex order - the accumulation order (and therefore every bit of the result)
// is the same as a plain loop over k.  With most vertices above the ground the serial per-vertex test was ~40 % of the
// physics time of fallen humanoids (tools/ablate.sh).
// pass 1: 64-bit mask of the hull vertices below the ground plane (four vertices per iteration)
template <typename T>
__device__ __forceinline__ unsigned long long contact_mask(const float* __restrict__ vb, int vmax, int nv, const T* R, const T* p) {
  unsigned long long mask = 0ull;
  const T pz = p[2];
  for (int k0 = 0; k0 < nv; k0 += 4) {
    const float4 X = *reinterpret_cast<const float4*>(vb + k0);
    const float4 Y = *reinterpret_cast<const float4*>(vb + vmax + k0);
    const float4 Z = *reinterpret_cast<const float4*>(vb + 2 * vmax + k0);
    const T r0 = R[6] * T(X.x) + R[7] * T(Y.x) + R[8] * T(Z.x);
    const T r1 = R[6] * T(X.y) + R[7] * T(Y.y) + R[8] * T(Z.y);
    const T r2 = R[6] * T(X.z) + R[7] * T(Y.z) + R[8] * T(Z.z);
    const T r3 = R[6] * T(X.w) + R[7] * T(Y.w) + R[8] * T(Z.w);
    const unsigned m = ((-(pz + r0) > T(0)) ? 1u : 0u) | ((-(pz + r1) > T(0)) ? 2u : 0u) | ((-(pz + r2) > T(0)) ? 4u : 0u) |
                       ((-(pz + r3) > T(0)) ? 8u : 0u);
    mask |= (unsigned long long)m << k0;
  }
  if (nv < 64) mask &= (1ull << nv) - 1ull;   // padding vertices (zeros) never count
  return mask;
}
// pass 2: the penetrating vertices, in ascending vertex order, added to the body's inertia / bias / contact force
template <typename T>
__device__ __forceinline__ void contact_apply(const float* __restrict__ vb, int vmax, unsigned long long mask, const PhysCfg<T>& c, const T* R,
                                              const T* p, const T* v, const T* w, T* A, T* Bm, T* C, T* bn, T* bf, T* cf) {
  const T pz = p[2];
  const T kimp = c.h * c.cn + c.h * c.h * c.kn;
  while (mask) {
    const int k = __ffsll((long long)mask) - 1;
    mask &= mask - 1ull;
    const T vl[3] = {T(vb[k]), T(vb[vmax + k]), T(vb[2 * vmax + k])};
    const T rz = R[6] * vl[0] + R[7] * vl[1] + R[8] * vl[2];
    const T pen = -(pz + rz);
    if (!(pen > T(0))) continue;   // (re-tested: the two passes may contract their FMAs differently)
    const T rx = R[0] * vl[0] + R[1] * vl[1] + R[2] * vl[2];
    const T ry = R[3] * vl[0] + R[4] * vl[1] + R[5] * vl[2];
    const T ux = v[0] + w[1] * rz - w[2] * ry;
    const T uy = v[1] + w[2] * rx - w[0] * rz;
    const T uz = v[2] + w[0] * ry - w[1] * rx;
    const T fn0 = c.kn * pen - c.cn * uz;
    if (!(fn0 > T(0))) continue;
    const T ut = sqrt_(ux * ux + uy * uy);
    const T ct = c.mu * fn0 * rcp_(ut > c.vs ? ut : c.vs);
    const T hct = c.h * ct;
    // Jn = [(ry, -rx, 0); (0,0,1)], Jx = [(0, rz, -ry); (1,0,0)], Jy = [(-rz, 0, rx); (0,1,0)]
    A[0] += kimp * ry * ry + hct * rz * rz;
    A[1] += kimp * rx * rx + hct * rz * rz;
    A[2] += hct * (ry * ry + rx * rx);
    A[3] += -kimp * ry * rx;
    A[4] += -hct * rz * rx;
    A[5] += -hct * rz * ry;
    Bm[2] += kimp * ry;   // (Jn_ang)(Jn_lin)^T : column z
    Bm[5] += -kimp * rx;
    Bm[3] += hct * rz;    // Jx: ang (0,rz,-ry) x lin ex -> column x
    Bm[6] += -hct * ry;
    Bm[1] += -hct * rz;   // Jy: ang (-rz,0,rx) x lin ey -> column y
    Bm[7] += hct * rx;
    C[0] += hct; C[1] += hct; C[2] += kimp;
    // wrench W = Jn fn0 - ct (Jx ux + Jy uy);  b -= W
    const T fx = -ct * ux, fy = -ct * uy;
    bn[0] -= ry * fn0 - rz * fy;
    bn[1] -= -rx * fn0 + rz * fx;
    bn[2] -= -ry * fx + rx * fy;
    bf[0] -= fx; bf[1] -= fy; bf[2] -= fn0;
    cf[0] += fx; cf[1] += fy; cf[2] += fn0;
  }
}
template <typename T>
__device__ __forceinline__ void contact_hull(const float* __restrict__ vb, int vmax, int nv, const PhysCfg<T>& c, const T* R, const T* p,
                                             const T* v, const T* w, T* A, T* Bm, T* C, T* bn, T* bf, T* cf) {
  contact_apply<T>(vb, vmax, contact_mask<T>(vb, vmax, nv, R, p), c, R, p, v, w, A, Bm, C, bn, bf, cf);
}

// ---- exact sphere / convex hull query (float64 restatement: oracle/physics_ref.c::hull_sphere_ref).  c: sphere centre in the body frame.
// (1) s = max over the face planes of n.c - d: s > R separates exactly; (2) s <= 0: centre inside the hull, depth R - s along the
// least-penetrated face normal; (3) else the closest point of the hull surface = closest point over its triangles (Ericson 5.1.5).
// vb: the body's hull vertices, SoA [3][vmax] (shared memory); pl / tr: its planes / triangles (global memory, L2-resident).
template <typename T>
__device__ __forceinline__ bool closest_on_triangle(const T* p, const T* a, const T* b, const T* c, T* q) {
  T ab[3], ac[3], ap[3];
#pragma unroll
  for (int k = 0; k < 3; k++) { ab[k] = b[k] - a[k]; ac[k] = c[k] - a[k]; ap[k] = p[k] - a[k]; }
  const T d1 = ab[0] * ap[0] + ab[1] * ap[1] + ab[2] * ap[2], d2 = ac[0] * ap[0] + ac[1] * ap[1] + ac[2] * ap[2];
  if (d1 <= T(0) && d2 <= T(0)) { q[0] = a[0]; q[1] = a[1]; q[2] = a[2]; return false; }
  T bp[3];
#pragma unroll
  for (int k = 0; k < 3; k++) bp[k] = p[k] - b[k];
  const T d3 = ab[0] * bp[0] + ab[1] * bp[1] + ab[2] * bp[2], d4 = ac[0] * bp[0] + ac[1] * bp[1] + ac[2] * bp[2];
  if (d3 >= T(0) && d4 <= d3) { q[0] = b[0]; q[1] = b[1]; q[2] = b[2]; return false; }
  const T vc = d1 * d4 - d3 * d2;
  if (vc <= T(0) && d1 >= T(0) && d3 <= T(0)) {
    const T v = d1 / (d1 - d3);
#pragma unroll
    for (int k = 0; k < 3; k++) q[k] = a[k] + v * ab[k];
    return false;
  }
  T cp[3];
#pragma unroll
  for (int k = 0; k < 3; k++) cp[k] = p[k] - c[k];
  const T d5 = ab[0] * cp[0] + ab[1] * cp[1] + ab[2] * cp[2], d6 = ac[0] * cp[0] + ac[1] * cp[1] + ac[2] * cp[2];
  if (d6 >= T(0) && d5 <= d6) { q[0] = c[0]; q[1] = c[1]; q[2] = c[2]; return false; }
  const T vb2 = d5 * d2 - d1 * d6;
  if (vb2 <= T(0) && d2 >= T(0) && d6 <= T(0)) {
    const T w = d2 / (d2 - d6);
#pragma unroll
    for (int k = 0; k < 3; k++) q[k] = a[k] + w * ac[k];
    return false;
  }
  const T va = d3 * d6 - d5 * d4;
  if (va <= T(0) && (d4 - d3) >= T(0) && (d5 - d6) >= T(0)) {
    const T w = (d4 - d3) / ((d4 - d3) + (d5 - d6));
#pragma unroll
    for (int k = 0; k < 3; k++) q[k] = b[k] + w * (c[k] - b[k]);
    return false;
  }
  const T den = T(1) / (va + vb2 + vc), v = vb2 * den, w = vc * den;
#pragma unroll
  for (int k = 0; k < 3; k++) q[k] = a[k] + ab[k] * v + ac[k] * w;
  return true;   // the projection of p onto the triangle's plane lies inside the triangle
}
// Shortcut of the closest-point pass.  For a point outside a convex hull, the largest plane offset smax (face imax, pass 1) is a lower bound
// of its distance to the hull, attained iff the projection onto that plane lies inside the face - then the other faces need not be
// walked.  Returns whether it applied; best / qb = squared distance / closest point on face imax in that case (untouched otherwise).
template <typename T>
__device__ __forceinline__ bool hull_nearest_on_face(const float* vb, int vmax, const unsigned char* tr, int imax, const T* c, T& best, T* qb) {
  const uint32_t tri = *reinterpret_cast<const uint32_t*>(tr + 4 * imax);
  const int i0 = tri & 0xFFu, i1 = (tri >> 8) & 0xFFu, i2 = (tri >> 16) & 0xFFu;
  const T a[3] = {T(vb[i0]), T(vb[vmax + i0]), T(vb[2 * vmax + i0])};
  const T b[3] = {T(vb[i1]), T(vb[vmax + i1]), T(vb[2 * vmax + i1])};
  const T cc[3] = {T(vb[i2]), T(vb[vmax + i2]), T(vb[2 * vmax + i2])};
  T q[3];
  if (!closest_on_triangle<T>(c, a, b, cc, q)) return false;
  best = (c[0] - q[0]) * (c[0] - q[0]) + (c[1] - q[1]) * (c[1] - q[1]) + (c[2] - q[2]) * (c[2] - q[2]);
  qb[0] = q[0]; qb[1] = q[1]; qb[2] = q[2];
  return true;
}
template <typename T>
__device__ __forceinline__ bool hull_sphere(const float* vb, int vmax, const float* pl, const unsigned char* tr, int nt, const T* c, T R, T& pen,
                                            T* nl) {
  // The planes and triangles live in global memory (L2): four faces per iteration, their loads issued together, so that a lane pays one
  // memory latency per four faces instead of one per face (the face loop of ONE lane decides when a one-wave launch ends).  Faces are still examined in ascending order: same separating test, same maximum, same closest point.
  T smax = T(-1e30);
  int imax = 0;
  for (int t = 0; t < nt; t += 4) {
    float4 P[4];
#pragma unroll
    for (int j = 0; j < 4; j++) P[j] = *reinterpret_cast<const float4*>(pl + 4 * (t + j < nt ? t + j : nt - 1));   // past the end: the last face again
    T sd[4];
#pragma unroll
    for (int j = 0; j < 4; j++) sd[j] = T(P[j].x) * c[0] + T(P[j].y) * c[1] + T(P[j].z) * c[2] - T(P[j].w);
    if (sd[0] > R || sd[1] > R || sd[2] > R || sd[3] > R) return false;   // a separating face plane: the common outcome for a ball that is merely near the body
#pragma unroll
    for (int j = 0; j < 4; j++)
      if (sd[j] > smax) { smax = sd[j]; imax = t + j; }   // (a repeated last face never beats itself)
  }
  if (smax <= T(0)) {
    pen = R - smax;
    nl[0] = T(pl[4 * imax]); nl[1] = T(pl[4 * imax + 1]); nl[2] = T(pl[4 * imax + 2]);
    return true;
  }
  T best = T(1e30), qb[3] = {T(0), T(0), T(0)};
  if (hull_nearest_on_face<T>(vb, vmax, tr, imax, c, best, qb)) nt = 0;   // the projection onto the farthest face plane lies inside that face: done
  for (int t = 0; t < nt; t += 4) {
    // the closest point of a convex hull to an outside point lies on a face the point sees (its offset from that face's plane is
    // positive): the back faces are skipped
    float4 P[4];
    uint32_t tri[4];
#pragma unroll
    for (int j = 0; j < 4; j++) {
      const int tt = t + j < nt ? t + j : nt - 1;
      P[j] = *reinterpret_cast<const float4*>(pl + 4 * tt);
      tri[j] = *reinterpret_cast<const uint32_t*>(tr + 4 * tt);
    }
#pragma unroll
    for (int j = 0; j < 4; j++) {
      if (t + j >= nt) break;
      if (!(T(P[j].x) * c[0] + T(P[j].y) * c[1] + T(P[j].z) * c[2] - T(P[j].w) > T(0))) continue;
      const int i0 = tri[j] & 0xFFu, i1 = (tri[j] >> 8) & 0xFFu, i2 = (tri[j] >> 16) & 0xFFu;
      const T a[3] = {T(vb[i0]), T(vb[vmax + i0]), T(vb[2 * vmax + i0])};
      const T b[3] = {T(vb[i1]), T(vb[vmax + i1]), T(vb[2 * vmax + i1])};
      const T cc[3] = {T(vb[i2]), T(vb[vmax + i2]), T(vb[2 * vmax + i2])};
      T q[3];
      closest_on_triangle<T>(c, a, b, cc, q);
      const T e2 = (c[0] - q[0]) * (c[0] - q[0]) + (c[1] - q[1]) * (c[1] - q[1]) + (c[2] - q[2]) * (c[2] - q[2]);
      if (e2 < best) { best = e2; qb[0] = q[0]; qb[1] = q[1]; qb[2] = q[2]; }
    }
  }
  const T dist = sqrt_(best);
  if (!(dist < R) || dist <= T(1e-9)) return false;
  pen = R - dist;
  const T id = T(1) / dist;
  nl[0] = (c[0] - qb[0]) * id; nl[1] = (c[1] - qb[1]) * id; nl[2] = (c[2] - qb[2]) * id;
  return true;
}


// hull_sphere with the faces of ONE body spread over the 8 lanes of an env's group (lane slot s takes the faces s, s + 8, s + 16, ...,
// four of them per iteration): what bounds a launch is the longest serial face walk of a single lane -
// ~2 x 100 dependent L2 round trips when one lane does a whole hull.  Every lane of the WARP calls this together (the exchanges are
// warp shuffles); act: this lane's group has a body to test (its arguments are the same on the 8 lanes).  The outcome is the serial
// function's bit for bit: the same per-face values, the maximum / the minimum taken with the serial loop's tie rule (the lowest face).
template <typename T>
__device__ __forceinline__ bool hull_sphere_coop(const float* vb, int vmax, const float* pl, const unsigned char* tr, int nt, const T* c, T R, int s,
                                                 bool act, T& pen, T* nl) {
  // ---- pass 1: separating plane / deepest face
  T smax = T(-1e30);
  int imax = 1 << 30;
  bool sep = false, done = !act;
  for (int t0 = 0;; t0 += 32) {
    if (!done) {
      float4 P[4];
      int ti[4];
#pragma unroll
      for (int j = 0; j < 4; j++) { ti[j] = t0 + 8 * j + s; P[j] = *reinterpret_cast<const float4*>(pl + 4 * (ti[j] < nt ? ti[j] : nt - 1)); }
#pragma unroll
      for (int j = 0; j < 4; j++) {
        if (ti[j] >= nt) continue;
        const T sd = T(P[j].x) * c[0] + T(P[j].y) * c[1] + T(P[j].z) * c[2] - T(P[j].w);
        if (sd > R) sep = true;
        if (sd > smax) { smax = sd; imax = ti[j]; }
      }
    }
    // a separating plane anywhere in my group ends the group's walk (the serial loop returns at the first one: no side effects either way)
    const uint32_t gs = (__ballot_sync(FULL, sep) >> ((emu_lane_id() >> 3) * 8)) & 0xFFu;
    if (gs) sep = true;
    if (sep || t0 + 32 >= nt) done = true;
    if (!__any_sync(FULL, !done)) break;
  }
  // deepest face of the group: maximum, ties to the lowest face index (= the serial loop's first maximum)
#pragma unroll
  for (int off = 1; off < 8; off <<= 1) {
    const T os = __shfl_xor_sync(FULL, smax, off);
    const int oi = __shfl_xor_sync(FULL, imax, off);
    if (os > smax || (os == smax && oi < imax)) { smax = os; imax = oi; }
  }
  const bool inside = act && !sep && smax <= T(0);
  if (inside) {
    pen = R - smax;
    nl[0] = T(pl[4 * imax]); nl[1] = T(pl[4 * imax + 1]); nl[2] = T(pl[4 * imax + 2]);
  }
  // ---- pass 2: closest point over the faces the centre sees (groups that are decided idle through it)
  bool need = act && !sep && !inside;
  T best = T(1e30), qb[3] = {T(0), T(0), T(0)};
  int ibest = 1 << 30;
  if (need && hull_nearest_on_face<T>(vb, vmax, tr, imax, c, best, qb)) need = false;   // same on the 8 lanes of the group (same arguments)
  if (__any_sync(FULL, need)) {
    bool fin = !need;
    for (int t0 = 0;; t0 += 32) {
      if (!fin) {
        float4 P[4];
        uint32_t tri[4];
        int ti[4];
#pragma unroll
        for (int j = 0; j < 4; j++) {
          ti[j] = t0 + 8 * j + s;
          const int tt = ti[j] < nt ? ti[j] : nt - 1;
          P[j] = *reinterpret_cast<const float4*>(pl + 4 * tt);
          tri[j] = *reinterpret_cast<const uint32_t*>(tr + 4 * tt);
        }
#pragma unroll
        for (int j = 0; j < 4; j++) {
          if (ti[j] >= nt) continue;
          if (!(T(P[j].x) * c[0] + T(P[j].y) * c[1] + T(P[j].z) * c[2] - T(P[j].w) > T(0))) continue;
          const int i0 = tri[j] & 0xFFu, i1 = (tri[j] >> 8) & 0xFFu, i2 = (tri[j] >> 16) & 0xFFu;
          const T a[3] = {T(vb[i0]), T(vb[vmax + i0]), T(vb[2 * vmax + i0])};
          const T b[3] = {T(vb[i1]), T(vb[vmax + i1]), T(vb[2 * vmax + i1])};
          const T cc[3] = {T(vb[i2]), T(vb[vmax + i2]), T(vb[2 * vmax + i2])};
          T q[3];
          closest_on_triangle<T>(c, a, b, cc, q);
          const T e2 = (c[0] - q[0]) * (c[0] - q[0]) + (c[1] - q[1]) * (c[1] - q[1]) + (c[2] - q[2]) * (c[2] - q[2]);
          if (e2 < best) { best = e2; ibest = ti[j]; qb[0] = q[0]; qb[1] = q[1]; qb[2] = q[2]; }
        }
        if (t0 + 32 >= nt) fin = true;
      }
      if (!__any_sync(FULL, !fin)) break;
    }
    // nearest face of the group: minimum, ties to the lowest face index (= the serial loop's first minimum)
#pragma unroll
    for (int off = 1; off < 8; off <<= 1) {
      const T ob = __shfl_xor_sync(FULL, best, off);
      const int oi = __shfl_xor_sync(FULL, ibest, off);
      const T o0 = __shfl_xor_sync(FULL, qb[0], off), o1 = __shfl_xor_sync(FULL, qb[1], off), o2 = __shfl_xor_sync(FULL, qb[2], off);
      if (ob < best || (ob == best && oi < ibest)) { best = ob; ibest = oi; qb[0] = o0; qb[1] = o1; qb[2] = o2; }
    }
  }
  if (!act || sep) return false;
  if (inside) return true;
  const T dist = sqrt_(best);
  if (!(dist < R) || dist <= T(1e-9)) return false;
  pen = R - dist;
  const T id = T(1) / dist;
  nl[0] = (c[0] - qb[0]) * id; nl[1] = (c[1] - qb[1]) * id; nl[2] = (c[2] - qb[2]) * id;
  return true;
}


template <typename T> __device__ __forceinline__ void ball_clear(Ball<T>& b) {
#pragma unroll
  for (int k = 0; k < 3; k++) { b.p[k] = 0; b.v[k] = 0; b.w[k] = 0; b.fa[k] = 0; b.rF[k] = 0; b.rX[k] = 0; b.bpos[k] = 0; }
  b.hits = 0; b.has_bounce = 0; b.bounce_now = 0;
}

__device__ __forceinline__ LaneConst lane_const(const b200_model_t& M, int lane) {
  LaneConst lc;
  lc.active = lane < M.nb;
  lc.par = lc.active ? (M.parent[lane] < 0 ? 0 : M.parent[lane]) : 0;
  lc.depth = lc.active ? M.depth[lane] : -1;
  lc.dof0 = lc.active ? M.dof_of_body[lane] : -1;
  lc.dyn = lc.active && !M.fixed[lane];
  lc.rix = lane;
  return lc;
}

// ------------------------------------------------------------------------------------------
// state I/O of one env (lane = body)

// Middle launch of the split step: the state rows the pre_kernel left behind for the NE envs of the hand-out positions eb .. eb + NE - 1
// (row(i) = the env row of position i): root row, joint state, PD targets and residual wrench (ext_wrench [N][6]).  Every load of the
// NE envs is issued before the first use (one memory latency instead of NE); positions from end on (a ragged tail) re-read the last env
// and are not unpacked.  gather_state_rows loads, unpack_state_row gives env eb + k as the physics wants it.  The caller keeps the
// loop over k: with the loop and the record store inside one helper the step kernels' SASS is scheduled differently.
template <int NE> struct StateRows {
  float rq[NE][3], rw[NE][3], rp[NE][3];   // joint exp-map coordinates, joint velocity, PD target
  float r1[NE];                            // lane j < 13: root_states[e][j], 13 <= j < 19: the residual wrench
};
template <int NE, typename Row>
__device__ __forceinline__ void gather_state_rows(const b200_buffers_t& bf, const b200_model_t& M, const LaneConst& lc, int lane, int64_t eb,
                                                  int64_t end, const Row& row, const float* __restrict__ ext_wrench, StateRows<NE>& r) {
  const int nd = M.nd;
#pragma unroll
  for (int k = 0; k < NE; k++) {
    const int64_t ek = eb + k < end ? eb + k : end - 1;
    const int64_t e = row(ek);
    if (lc.dyn && lane > 0) {
      const float* ds = bf.dof_state + (e * nd + lc.dof0) * 2;
#pragma unroll
      for (int j = 0; j < 3; j++) { r.rq[k][j] = ds[2 * j]; r.rw[k][j] = ds[2 * j + 1]; r.rp[k][j] = bf.pd_targets[e * nd + lc.dof0 + j]; }
    }
    r.r1[k] = lane < 13 ? bf.root_states[e * bf.actors_per_env * 13 + lane] : (lane < 19 ? ext_wrench[e * 6 + lane - 13] : 0.f);
  }
}
template <int NE>
__device__ __forceinline__ void unpack_state_row(const StateRows<NE>& r, int k, const LaneConst& lc, int lane, Lane<float>& L, float* pdtar,
                                                 float* extF, float* extT) {
  lane_rest(L);
#pragma unroll
  for (int j = 0; j < 3; j++) { pdtar[j] = 0.f; extF[j] = 0.f; extT[j] = 0.f; }
  float rr[19];
#pragma unroll
  for (int j = 0; j < 19; j++) rr[j] = __shfl_sync(FULL, r.r1[k], j);
  if (lane == 0) {
#pragma unroll
    for (int j = 0; j < 3; j++) { L.p[j] = rr[j]; L.v[j] = rr[7 + j]; L.w[j] = rr[10 + j]; extF[j] = rr[13 + j]; extT[j] = rr[16 + j]; }
#pragma unroll
    for (int j = 0; j < 4; j++) L.Q[j] = rr[3 + j];
    qnormalize(L.Q);
  }
  if (lc.dyn && lane > 0) {
#pragma unroll
    for (int j = 0; j < 3; j++) { L.wt[j] = r.rw[k][j]; pdtar[j] = r.rp[k][j]; }
    qexp(r.rq[k], L.qj);
  }
}

// The arrays of the physics-only entry (b200env_physics_only; the CPU lane emulator has the same signature): root [n][13],
// dof_pos / dof_vel / pd_tar [n][nd], ext [n][6], rb_out [n][nb][13], contact_out [n][nb][3], ball [n][13] (p, -, v, w as a root row),
// hits [n], dof_force [n][nd] (the DOF force sensor of the last control step, packed.cuh::pk_dof_force; read by the sensor instantiation
// of physics_kernel_packed only).  ext, contact_out, ball, hits and dof_force may be null.
template <typename T> struct EnvArrays {
  T *root, *dof_pos, *dof_vel;
  const T *pd_tar, *ext;
  T *rb_out, *contact_out, *ball;
  int32_t* hits;
  T* dof_force;
};
template <typename T>
__device__ __forceinline__ void env_arrays_load(const EnvArrays<T>& io, int nd, const LaneConst& lc, int lane, int64_t e, Lane<T>& L, T* pdt,
                                                T* eF, T* eT) {
  lane_rest(L);
#pragma unroll
  for (int j = 0; j < 3; j++) { pdt[j] = 0; eF[j] = 0; eT[j] = 0; }
  if (lane == 0) {
    const T* rs = io.root + e * 13;
#pragma unroll
    for (int j = 0; j < 3; j++) { L.p[j] = rs[j]; L.v[j] = rs[7 + j]; L.w[j] = rs[10 + j]; }
#pragma unroll
    for (int j = 0; j < 4; j++) L.Q[j] = rs[3 + j];
    qnormalize(L.Q);
    if (io.ext) for (int j = 0; j < 3; j++) { eF[j] = io.ext[e * 6 + j]; eT[j] = io.ext[e * 6 + 3 + j]; }
  }
  if (lc.dyn && lane > 0) {
    T q[3];
#pragma unroll
    for (int j = 0; j < 3; j++) { q[j] = io.dof_pos[e * nd + lc.dof0 + j]; L.wt[j] = io.dof_vel[e * nd + lc.dof0 + j]; pdt[j] = io.pd_tar[e * nd + lc.dof0 + j]; }
    qexp(q, L.qj);
  }
}
// cf: the contact force of the lane's body, written for every body.  cf = null: the step wrote the rows of the jointed bodies itself
// (control_step_t), a welded body's row is 0.
template <typename T>
__device__ __forceinline__ void env_arrays_store(const EnvArrays<T>& io, int nb, int nd, const LaneConst& lc, int lane, int64_t e, const Lane<T>& L,
                                                 const T* cf) {
  if (lane == 0) {
    T* rs = io.root + e * 13;
#pragma unroll
    for (int j = 0; j < 3; j++) { rs[j] = L.p[j]; rs[7 + j] = L.v[j]; rs[10 + j] = L.w[j]; }
#pragma unroll
    for (int j = 0; j < 4; j++) rs[3 + j] = L.Q[j];
  }
  if (lc.dyn && lane > 0) {
    T q[3];
    qlog(L.qj, q);
#pragma unroll
    for (int j = 0; j < 3; j++) { io.dof_pos[e * nd + lc.dof0 + j] = q[j]; io.dof_vel[e * nd + lc.dof0 + j] = L.wt[j]; }
  }
  if (lc.active) {
    T* rb = io.rb_out + (e * nb + lane) * 13;
#pragma unroll
    for (int j = 0; j < 3; j++) { rb[j] = L.p[j]; rb[7 + j] = L.v[j]; rb[10 + j] = L.w[j]; }
#pragma unroll
    for (int j = 0; j < 4; j++) rb[3 + j] = L.Q[j];
    if (io.contact_out && (cf || !lc.dyn))
      for (int j = 0; j < 3; j++) io.contact_out[(e * nb + lane) * 3 + j] = cf ? cf[j] : T(0);
  }
}
template <typename T> __device__ __forceinline__ void env_arrays_load_ball(const EnvArrays<T>& io, int64_t e, Ball<T>& ball) {
#pragma unroll
  for (int j = 0; j < 3; j++) { ball.p[j] = io.ball[e * 13 + j]; ball.v[j] = io.ball[e * 13 + 7 + j]; ball.w[j] = io.ball[e * 13 + 10 + j]; }
}
template <typename T> __device__ __forceinline__ void env_arrays_store_ball(const EnvArrays<T>& io, int64_t e, const Ball<T>& ball) {
#pragma unroll
  for (int j = 0; j < 3; j++) { io.ball[e * 13 + j] = ball.p[j]; io.ball[e * 13 + 7 + j] = ball.v[j]; io.ball[e * 13 + 10 + j] = ball.w[j]; }
  if (io.hits) io.hits[e] = ball.hits;
}

