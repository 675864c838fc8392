// ballgen.cuh - offline tennis-ball data generators (include/b200ball.h, SURVEY.md 8f-2).  Included at the end of b200env.cu:
// the balls are integrated by the very ball model of the env step kernel (Ball<T>, ball_substep<T> above), so the pool
// trajectories and the estimator tables are consistent with what the envs simulate.  float64 twin: oracle/ref_port_ballgen.py.
//
// One thread per ball.  A trajectory is a serial chain (a sim step needs the previous one), the balls are independent: the
// launch is sized to fill the machine with resident warps.  Output rows are written by the owning thread as they are produced
// (12 B per 30 Hz frame, or one table column at a time); the rows of a warp are 480-1200 B apart, the sectors are completed in
// L2 by the same thread a few iterations later.
#pragma once
#include "../../include/b200ball.h"

#define BALLGEN_THREADS 128
#define NET_HEIGHT_F 1.07  // tennis_ball.py:20

// forces of simulate() (tennis_ball.py:160-183) / simulate_without_bounce (:58-74): drag + Magnus lift like ball_aero(), but the
// lift direction follows the sign of the LAUNCH spin (vspin := -|w|/2pi for a back-spin launch)
template <typename T>
__device__ __forceinline__ void ball_aero_signed(const T* vel, const T* angvel, T launch_vspin, T spin_scale, T* force) {
  const T KF = T(0.0019462794807519486), CD = T(0.55);
  T vs = sqrt_(vel[0] * vel[0] + vel[1] * vel[1] + vel[2] * vel[2]);
  if (vs == T(0)) vs += T(1);   // a ball at rest: no force (the env's apply_external_force_to_ball has this guard, :715; simulate() divides 0/0)
  const T iv = rcp_(vs);
  const T vn[3] = {vel[0] * iv, vel[1] * iv, vel[2] * iv};
  const T vt[3] = {-vn[1], vn[0], T(0)};  // vn x (0,0,-1)
  T vspin = sqrt_(angvel[0] * angvel[0] + angvel[1] * angvel[1] + angvel[2] * angvel[2]) * T(0.15915494309189535);
  if (!(launch_vspin > T(0))) vspin = -vspin;
  T cl = rcp_(T(2) + fabs(vs * rcp_(vspin * spin_scale + T(1e-6))));
  cl = vspin > T(0) ? -cl : cl;
  const T cx = vt[1] * vn[2] - vt[2] * vn[1], cy = vt[2] * vn[0] - vt[0] * vn[2], cz = vt[0] * vn[1] - vt[1] * vn[0];
  const T kd = -KF * CD * vs, kl = -KF * cl * vs * vs;
  force[0] = kd * vel[0] + kl * cx; force[1] = kd * vel[1] + kl * cy; force[2] = kd * vel[2] + kl * cz;
}

template <typename T> __device__ __forceinline__ PhysCfg<T> ballgen_cfg(const b200ball_sim_t& c) {
  PhysCfg<T> p;
  p.h = T(c.sim_dt) / T(c.substeps);
  p.gz = T(c.gravity_z);
  p.kn = p.cn = p.mu = p.vs = p.damp = p.wmax = p.limk = p.limc = T(0);
  p.substeps = c.substeps; p.cfi = c.control_freq_inv;
  p.has_ball = 1; p.racket_body = -1; p.wrist_body = 0;
  p.bm = T(c.ball_mass); p.bI = T(c.ball_inertia); p.bR = T(c.ball_radius); p.spin_scale = T(c.spin_scale);
  p.eg = T(c.e_ground); p.mug = T(c.mu_ground); p.er = T(0); p.mur = T(0); p.vth = T(c.bounce_threshold_velocity);
  p.hc[0] = p.hc[1] = p.hc[2] = T(0); p.hh = p.hr = T(0);
  p.hq[0] = p.hq[1] = p.hq[2] = T(0); p.hq[3] = T(1);
  p.ball_body = 0; p.eb = p.mub = T(0);
  for (int k = 0; k < 7; k++) p.hdl[k] = T(0);
  return p;
}

// launch state: angular velocity = vspin * 2pi * normalize(v x (0,0,-1))  (tennis_ball.py:134-139)
template <typename T> __device__ __forceinline__ void ballgen_launch(Ball<T>& B, const T* p, const T* v, T vspin) {
  ball_clear(B);
  const T c[3] = {-v[1], v[0], T(0)};
  T nn = sqrt_(c[0] * c[0] + c[1] * c[1]);
  nn = nn > T(1e-12) ? nn : T(1e-12);
  const T s = vspin * T(6.283185307179586) / nn;
#pragma unroll
  for (int k = 0; k < 3; k++) { B.p[k] = p[k]; B.v[k] = v[k]; B.w[k] = s * c[k]; }
}

// ------------------------------------------------------------------------------------------ simulate()  (tennis_ball.py:113-218)
// The samples of a row are produced 12 B at a time, the rows of a warp are F*12 B apart: written straight from the loop every
// store instruction touches 32 different sectors (ncu r1h: the kernel waits on its own stores, 11 stall cycles per issue).
// So the block stages BALLGEN_CHUNK frames per ball in shared memory and writes them out together: consecutive lanes write
// consecutive floats of a row segment (BALLGEN_CHUNK * nc * 4 = 96 B contiguous).
#define BALLGEN_CHUNK 8
template <typename T>
__global__ void __launch_bounds__(BALLGEN_THREADS)
ball_simulate_kernel(b200ball_sim_t c, int64_t n, const T* __restrict__ lp, const T* __restrict__ lv, const T* __restrict__ ls,
                     T* __restrict__ traj, T* __restrict__ bounce_pos, int64_t* __restrict__ bounce_idx, uint8_t* __restrict__ pass_net) {
  constexpr int TS = BALLGEN_CHUNK * 3 + 1;   // tile row stride (odd: the threads of a warp hit different banks)
  __shared__ T tile[BALLGEN_THREADS * TS];
  const int64_t row0 = (int64_t)blockIdx.x * blockDim.x;
  const int64_t i = row0 + threadIdx.x;
  const bool active = i < n;
  const int64_t ii = active ? i : n - 1;      // idle threads of the last block shadow the last ball (never stored)
  const PhysCfg<T> pc = ballgen_cfg<T>(c);
  Ball<T> B;
  const T p0[3] = {lp[ii * 3], lp[ii * 3 + 1], lp[ii * 3 + 2]}, v0[3] = {lv[ii * 3], lv[ii * 3 + 1], lv[ii * 3 + 2]};
  T lvs = ls[ii];
  ballgen_launch(B, p0, v0, lvs);
  const T thr = c.substeps > 2 ? pc.bR * T(6) : pc.bR * T(4);
  const int F = c.num_frames, nc = 3 - c.first_comp;
  bool has_bounce = false, has_pass = false, pass_ok = false;
  int64_t bidx = F - 1;
  T bp[3] = {T(0), T(0), T(0)};
  T* mine = tile + threadIdx.x * TS;
  const int rows_here = (int)((n - row0) < (int64_t)blockDim.x ? (n - row0) : (int64_t)blockDim.x);
  for (int t0 = 0; t0 < F; t0 += BALLGEN_CHUNK) {
    const int nf = F - t0 < BALLGEN_CHUNK ? F - t0 : BALLGEN_CHUNK;
    for (int tt = 0; tt < nf; tt++) {
      const int t = t0 + tt;
#pragma unroll
      for (int k = 0; k < 3; k++)
        if (k >= c.first_comp) mine[tt * nc + k - c.first_comp] = B.p[k];
      for (int s = 0; s < c.control_freq_inv; s++) {
        ball_aero_signed<T>(B.v, B.w, lvs, pc.spin_scale, B.fa);
        if (!has_pass && B.p[1] < T(0)) { pass_ok = !has_bounce && B.p[2] > T(NET_HEIGHT_F); has_pass = true; }     // :168-170
        if (!has_bounce && B.p[2] <= thr) {                                                                         // :185-199
          bp[0] = B.p[0]; bp[1] = B.p[1]; bp[2] = B.p[2];
          bidx = t; has_bounce = true;
          if (!(lvs > T(0))) lvs = -lvs;   // "backspin ball changes to topspin after bounce"
        }
        for (int sub = 0; sub < c.substeps; sub++) ball_substep<T>(pc, B, false, nullptr, nullptr, nullptr, nullptr);
      }
    }
    __syncthreads();
    const int seg = nf * nc;                       // floats per row in this chunk
    for (int idx = threadIdx.x; idx < rows_here * seg; idx += blockDim.x) {
      const int r = idx / seg, k = idx - r * seg;
      traj[((row0 + r) * F + t0) * nc + k] = tile[r * TS + k];
    }
    __syncthreads();
  }
  if (!active) return;
  bounce_pos[i * 3] = bp[0]; bounce_pos[i * 3 + 1] = bp[1]; bounce_pos[i * 3 + 2] = bp[2];
  bounce_idx[i] = bidx;
  pass_net[i] = pass_ok ? 1 : 0;
}

// ------------------------------------------------------------------------- simulate_without_bounce()  (tennis_ball_out_estimator.py:21-121)
// The reference stores the whole 60 Hz trajectory and then walks it once per grid value with a monotone sample pointer
// (:90-110).  Both walks only ever look at two consecutive samples, so here a row is resampled while it is integrated:
// at sample t every pending grid value whose stop condition holds (`!(t < T-1 && y_t < x)` resp. `!(t < T-1 && -z_t < y)`) is
// emitted from samples (t-1, t).  t = 0 pairs sample 0 with sample "-1" = the LAST sample (Python index wrap, reachable only
// by grid values <= 0): those columns are emitted after the loop.
template <typename T>
__global__ void __launch_bounds__(BALLGEN_THREADS)
ball_out_rows_kernel(b200ball_sim_t c, int64_t n, const T* __restrict__ vel_h, const T* __restrict__ vel_v, const T* __restrict__ vspin,
                     const float* __restrict__ gx, const int32_t* __restrict__ cx, int ngx, int nx, const float* __restrict__ gy,
                     const int32_t* __restrict__ cy, int ngy, int ny, T* __restrict__ out_x, T* __restrict__ out_y) {
  extern __shared__ unsigned char bg_smem[];
  float* sgx = reinterpret_cast<float*>(bg_smem);
  float* sgy = sgx + ngx;
  int32_t* scx = reinterpret_cast<int32_t*>(sgy + ngy);
  int32_t* scy = scx + ngx;
  for (int k = threadIdx.x; k < ngx; k += blockDim.x) { sgx[k] = gx[k]; scx[k] = cx[k]; }
  for (int k = threadIdx.x; k < ngy; k += blockDim.x) { sgy[k] = gy[k]; scy[k] = cy[k]; }
  __syncthreads();
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const T h = T(c.sim_dt) / T(c.substeps), gz = T(c.gravity_z), im = rcp_(T(c.ball_mass));
  Ball<T> B;
  const T p0[3] = {T(0), T(0), T(0)}, v0[3] = {T(0), vel_h[i], vel_v[i]};
  const T lvs = vspin[i];
  ballgen_launch(B, p0, v0, lvs);
  const int Tn = (c.num_frames + 1) * c.control_freq_inv;
  const T tscale = T(c.control_freq_inv * 30);
  T* ox = out_x + i * nx;
  T* oy = out_y + i * ny * 2;
  int jx = 0, jy = 0, n0x = 0, n0y = 0;
  T y1 = T(0), z1 = T(0);  // previous sample
  // Both walks emit their columns in ascending order, a few samples apart.  Written one float at a time, every store of a warp
  // hits 32 different sectors and every sector is written 8 times (ncu r1h: 8.8 GB of DRAM traffic for 4.06 GB of tables).  So a
  // thread collects the current group of 8 floats (8 columns of out_x, 4 (distance, time) pairs of out_y) in shared memory and
  // writes it with two 128-bit stores = one full sector; incomplete or out-of-order groups, and tables whose base address is not
  // 16-byte aligned, fall back to scalar stores.
  T* bxs = reinterpret_cast<T*>(bg_smem + (((size_t)(ngx + ngy) * 8 + 15) & ~(size_t)15));   // [8][threads] x group, then y group
  T* bys = bxs + 8 * BALLGEN_THREADS;
  const int tid = threadIdx.x;
  const bool vec_ok = sizeof(T) == 4 && (nx & 3) == 0 && ((ny * 2) & 3) == 0 &&
                      ((reinterpret_cast<uintptr_t>(out_x) | reinterpret_cast<uintptr_t>(out_y)) & 15) == 0;
  int gxb = -1, gyb = -1;
  unsigned mx = 0u, my = 0u;
  auto flush = [&](T* dst, const T* buf, int g, unsigned& m) {       // group g of a row: 8 floats at dst + 8 g
    if (m == 0xFFu && vec_ok) {
      float4 lo = make_float4(float(buf[0 * BALLGEN_THREADS + tid]), float(buf[1 * BALLGEN_THREADS + tid]), float(buf[2 * BALLGEN_THREADS + tid]),
                              float(buf[3 * BALLGEN_THREADS + tid]));
      float4 hi = make_float4(float(buf[4 * BALLGEN_THREADS + tid]), float(buf[5 * BALLGEN_THREADS + tid]), float(buf[6 * BALLGEN_THREADS + tid]),
                              float(buf[7 * BALLGEN_THREADS + tid]));
      float4* d4 = reinterpret_cast<float4*>(dst + 8 * g);
      d4[0] = lo; d4[1] = hi;
    } else {
      for (int k = 0; k < 8; k++)
        if ((m >> k) & 1u) dst[8 * g + k] = buf[k * BALLGEN_THREADS + tid];
    }
    m = 0u;
  };
  auto put_x = [&](int col, T val) {
    if ((unsigned)col >= (unsigned)nx) return;   // a column outside the row is never stored
    const int g = col >> 3;
    if (g != gxb) { if (mx) flush(ox, bxs, gxb, mx); gxb = g; }
    bxs[(col & 7) * BALLGEN_THREADS + tid] = val;
    mx |= 1u << (col & 7);
    if (mx == 0xFFu) flush(ox, bxs, gxb, mx);
  };
  auto put_y = [&](int col, T d, T tm) {
    if ((unsigned)col >= (unsigned)ny) return;
    const int g = col >> 2, k = (col & 3) * 2;
    if (g != gyb) { if (my) flush(oy, bys, gyb, my); gyb = g; }
    bys[k * BALLGEN_THREADS + tid] = d;
    bys[(k + 1) * BALLGEN_THREADS + tid] = tm;
    my |= 3u << k;
    if (my == 0xFFu) flush(oy, bys, gyb, my);
  };
  auto val_x = [&](int j, T ya, T za, T yb, T zb) -> T {
    const T x = T(sgx[j]);
    const T w = (x - ya) / (yb - ya);
    return za * (T(1) - w) + zb * w;
  };
  auto val_y = [&](int j, T ya, T za, T yb, T zb, int t, T& d, T& tm) {
    const T y = T(sgy[j]);
    const T w = (-y - za) / (zb - za);
    d = ya * (T(1) - w) + yb * w;
    tm = (T(t - 1) * (T(1) - w) + T(t) * w) / tscale;
  };
  auto emit_x = [&](int j, T ya, T za, T yb, T zb) { put_x(scx[j], val_x(j, ya, za, yb, zb)); };
  auto emit_y = [&](int j, T ya, T za, T yb, T zb, int t) {
    T d, tm;
    val_y(j, ya, za, yb, zb, t, d, tm);
    put_y(scy[j], d, tm);
  };
  // free flight: the angular velocity never changes, so the signed spin term of the lift is a per-row constant, and the
  // `substeps` substeps of a sim step under a constant force have the closed form  v += n h a,  p += n h v + h^2 a n(n+1)/2
  // (what the loop `v += h a; p += h v` sums to) - the oracle's loop and this agree to rounding.
  T vspin_c = sqrt_(B.w[0] * B.w[0] + B.w[1] * B.w[1] + B.w[2] * B.w[2]) * T(0.15915494309189535);
  if (!(lvs > T(0))) vspin_c = -vspin_c;
  const T spin_rc = rcp_(vspin_c * T(c.spin_scale) + T(1e-6));
  const T cl_sign = vspin_c > T(0) ? T(-1) : T(1);
  const T KF = T(0.0019462794807519486), CD = T(0.55);
  const T nh = T(c.substeps) * h, hh = h * h * T(c.substeps * (c.substeps + 1) / 2);
  const T INF = T(1e30);
  T thx = ngx > 0 ? T(sgx[0]) : INF, thy = ngy > 0 ? T(sgy[0]) : INF;   // next pending grid value of each walk
  for (int t = 0; t < Tn; t++) {
    const T y2 = B.p[1], z2 = B.p[2];
    const bool last = t == Tn - 1;
    while (jx < ngx && (last || !(y2 < thx))) {
      if (t == 0) { put_x(scx[jx], T(0)); n0x++; } else emit_x(jx, y1, z1, y2, z2);
      jx++;
      thx = jx < ngx ? T(sgx[jx]) : INF;
    }
    while (jy < ngy && (last || !(-z2 < thy))) {
      if (t == 0) { put_y(scy[jy], T(0), T(0)); n0y++; } else emit_y(jy, y1, z1, y2, z2, t);
      jy++;
      thy = jy < ngy ? T(sgy[jy]) : INF;
    }
    y1 = y2; z1 = z2;
    if (last) break;
    const T vs2 = B.v[0] * B.v[0] + B.v[1] * B.v[1] + B.v[2] * B.v[2];
    const T ivs = rsqrt_(vs2), vs = vs2 * ivs;
    const T n0 = B.v[0] * ivs, n1 = B.v[1] * ivs, n2 = B.v[2] * ivs;
    const T cl = cl_sign * rcp_(T(2) + fabs(vs * spin_rc));
    const T kd = -KF * CD * vs, kl = -KF * cl * vs2;
    const T a0 = (kd * B.v[0] + kl * (n0 * n2)) * im, a1 = (kd * B.v[1] + kl * (n1 * n2)) * im,
            a2 = (kd * B.v[2] - kl * (n0 * n0 + n1 * n1)) * im + gz;
    B.p[0] += nh * B.v[0] + hh * a0; B.p[1] += nh * B.v[1] + hh * a1; B.p[2] += nh * B.v[2] + hh * a2;
    B.v[0] += nh * a0; B.v[1] += nh * a1; B.v[2] += nh * a2;
  }
  if (mx) flush(ox, bxs, gxb, mx);
  if (my) flush(oy, bys, gyb, my);
  // Grid values reached at sample 0 pair sample 0 with sample "-1" = the last one.  For the value 0 (the only one the shipped
  // grids have there) the interpolation weight is (0 - a)/(0 - a) = 1 and the result 0 - already written - unless the last
  // sample is degenerate; anything else is recomputed the reference's way and stored over the placeholder.  The reference writes
  // the columns in grid order, so an entry whose column a later grid value also maps to is left to that later value.
  const bool plain = y1 != T(0) && z1 != T(0) && fabs(y1) < T(1e30) && fabs(z1) < T(1e30);
  auto kept = [](const int32_t* col, int j, int ng, int ncol) {
    if ((unsigned)col[j] >= (unsigned)ncol) return false;
    for (int k = j + 1; k < ng; k++)
      if (col[k] == col[j]) return false;
    return true;
  };
  for (int j = 0; j < n0x; j++)
    if (!(plain && sgx[j] == 0.f) && kept(scx, j, ngx, nx)) ox[scx[j]] = val_x(j, y1, z1, T(0), T(0));
  for (int j = 0; j < n0y; j++)
    if (!(plain && sgy[j] == 0.f) && kept(scy, j, ngy, ny)) {
      T d, tm;
      val_y(j, y1, z1, T(0), T(0), 0, d, tm);
      oy[scy[j] * 2] = d; oy[scy[j] * 2 + 1] = tm;
    }
}

extern "C" {

static int ballgen_check(const b200ball_sim_t* c, int64_t n, int32_t prec, const char* who) {
  if (!c) return fail(-1, "%s: null cfg", who);
  if (n < 0 || prec < 0 || prec > 1) return fail(-2, "%s: n >= 0 and prec in {0,1} required", who);
  if (c->num_frames < 1 || c->control_freq_inv < 1 || c->substeps < 1 || c->first_comp < 0 || c->first_comp > 2 || !(c->sim_dt > 0.f) ||
      !(c->ball_mass > 0.f) || !(c->ball_inertia > 0.f) || !(c->ball_radius > 0.f))
    return fail(-2, "%s: bad simulation parameters", who);
  return 0;
}

int b200ball_simulate(const b200ball_sim_t* cfg, int64_t n, int32_t prec, const void* launch_pos, const void* launch_vel,
                      const void* launch_vspin, void* traj, void* bounce_pos, int64_t* bounce_idx, uint8_t* pass_net, void* stream) {
  if (int rc = ballgen_check(cfg, n, prec, "b200ball_simulate")) return rc;
  if (n == 0) return 0;
  if (!launch_pos || !launch_vel || !launch_vspin || !traj || !bounce_pos || !bounce_idx || !pass_net)
    return fail(-1, "b200ball_simulate: null argument%s");
  const unsigned grid = (unsigned)((n + BALLGEN_THREADS - 1) / BALLGEN_THREADS);
  if (prec == 0)
    ball_simulate_kernel<float><<<grid, BALLGEN_THREADS, 0, (cudaStream_t)stream>>>(*cfg, n, (const float*)launch_pos, (const float*)launch_vel,
                                                                                   (const float*)launch_vspin, (float*)traj, (float*)bounce_pos,
                                                                                   bounce_idx, pass_net);
  else
    ball_simulate_kernel<double><<<grid, BALLGEN_THREADS, 0, (cudaStream_t)stream>>>(*cfg, n, (const double*)launch_pos, (const double*)launch_vel,
                                                                                    (const double*)launch_vspin, (double*)traj, (double*)bounce_pos,
                                                                                    bounce_idx, pass_net);
  CUDA_OK(cudaGetLastError());
  return 0;
}

int b200ball_out_rows(const b200ball_sim_t* cfg, int64_t n, int32_t prec, const void* vel_h, const void* vel_v, const void* vspin,
                      const float* grid_x, const int32_t* col_x, int32_t ngx, int32_t nx, const float* grid_y, const int32_t* col_y,
                      int32_t ngy, int32_t ny, void* out_x, void* out_y, void* stream) {
  if (int rc = ballgen_check(cfg, n, prec, "b200ball_out_rows")) return rc;
  if (n == 0) return 0;
  if (!vel_h || !vel_v || !vspin || !grid_x || !col_x || !grid_y || !col_y || !out_x || !out_y) return fail(-1, "b200ball_out_rows: null argument%s");
  if (ngx < 0 || ngy < 0 || nx < 1 || ny < 1 || ngx > 4096 || ngy > 4096) return fail(-2, "b200ball_out_rows: grid sizes out of range%s");
  const unsigned grid = (unsigned)((n + BALLGEN_THREADS - 1) / BALLGEN_THREADS);
  const size_t smem = (((size_t)(ngx + ngy) * (sizeof(float) + sizeof(int32_t)) + 15) & ~(size_t)15) +
                      (size_t)16 * BALLGEN_THREADS * (prec == 0 ? sizeof(float) : sizeof(double));   // grids + the two 8-float groups per thread
  if (smem > 48 * 1024)   // grids of thousands of values: opt in to more than the default 48 KB of dynamic shared memory (at most 80 KB)
    CUDA_OK(prec == 0 ? cudaFuncSetAttribute(ball_out_rows_kernel<float>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)
                      : cudaFuncSetAttribute(ball_out_rows_kernel<double>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  if (prec == 0)
    ball_out_rows_kernel<float><<<grid, BALLGEN_THREADS, smem, (cudaStream_t)stream>>>(*cfg, n, (const float*)vel_h, (const float*)vel_v,
                                                                                      (const float*)vspin, grid_x, col_x, ngx, nx, grid_y, col_y, ngy,
                                                                                      ny, (float*)out_x, (float*)out_y);
  else
    ball_out_rows_kernel<double><<<grid, BALLGEN_THREADS, smem, (cudaStream_t)stream>>>(*cfg, n, (const double*)vel_h, (const double*)vel_v,
                                                                                       (const double*)vspin, grid_x, col_x, ngx, nx, grid_y, col_y,
                                                                                       ngy, ny, (double*)out_x, (double*)out_y);
  CUDA_OK(cudaGetLastError());
  return 0;
}

}  // extern "C"
