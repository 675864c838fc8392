// emu_mixed.cpp - TEST INFRASTRUCTURE: the packed articulated step on the CPU (emu_packed.cpp: one host thread per lane) with envs of
// different assets of one topology in one warp, as step_kernel_packed<true, false, true> runs them: the tree tables of asset 0, the
// numeric constants and hull vertices of each env's own asset (control_step_packed's MN / verts per lane).  Built by
// tests/test_assets_mixed.py with the flags of tests/emu/build.py.
#include "emu_packed.cpp"

namespace {
template <typename T> struct MixedJob {
  const DevBlob* topo;            // asset 0: the tree tables every env shares
  const DevBlob* const* env_blob; // [n] the header of env e's asset
  const float* const* env_verts;  // [n] its SoA hull vertices
  const b200_cfg_t* cfg;
  int n, n_steps;
  T *root, *dof_pos, *dof_vel;
  const T *pd_tar, *ext;
  T *rb_out, *contact_out;
};

// lane_main (emu_packed.cpp) without the ball, each lane on its env's model
template <typename T> void lane_main_mixed(EmuWarp* w, int lane, const MixedJob<T>* J, int64_t eb, T* wrec) {
  emu_warp = w;
  emu_lane = lane;
  const DevBlob& B = *J->topo;
  const b200_model_t& M = B.m;
  const int n = J->n, nb = M.nb, nd = M.nd;
  LaneConst lc = lane_const(M, lane);
  if (lc.active) lc.rix = B.t.rix[lane];
  const PhysCfg<T> pc = make_phys_cfg<T>(*J->cfg);
  const int g = lane / SLOTS;
  for (int k = 0; k < EPW; k++) {
    const int64_t e = eb + k;
    if (e >= n) break;
    Lane<T> L;
    for (int j = 0; j < 4; j++) { L.Q[j] = 0; L.qj[j] = 0; }
    L.Q[3] = 1; L.qj[3] = 1;
    for (int j = 0; j < 3; j++) { L.p[j] = 0; L.w[j] = 0; L.v[j] = 0; L.wt[j] = 0; }
    T pdt[3] = {0, 0, 0}, eF[3] = {0, 0, 0}, eT[3] = {0, 0, 0};
    if (lane == 0) {
      const T* rs = J->root + e * 13;
      for (int j = 0; j < 3; j++) { L.p[j] = rs[j]; L.v[j] = rs[7 + j]; L.w[j] = rs[10 + j]; }
      for (int j = 0; j < 4; j++) L.Q[j] = rs[3 + j];
      qnormalize(L.Q);
      if (J->ext) for (int j = 0; j < 3; j++) { eF[j] = J->ext[e * 6 + j]; eT[j] = J->ext[e * 6 + 3 + j]; }
    }
    if (lc.dyn && lane > 0) {
      T q[3];
      for (int j = 0; j < 3; j++) { q[j] = J->dof_pos[e * nd + lc.dof0 + j]; L.wt[j] = J->dof_vel[e * nd + lc.dof0 + j]; pdt[j] = J->pd_tar[e * nd + lc.dof0 + j]; }
      qexp(q, L.qj);
    }
    pk_store_state<T>(wrec + k * ENV_STRIDE, lc, lane, L, pdt, eF, eT);
  }
  __syncwarp();
  const bool valid = eb + g < n;
  const int64_t me = valid ? eb + g : eb;   // a lane without an env takes the warp's first env's model, as the kernel does
  Ball<T> ball;
  ball_clear(ball);
  for (int st_ = 0; st_ < J->n_steps; st_++) {
    control_step_packed<T>(B, J->env_blob[me]->m, J->env_verts[me], pc, wrec, lane, valid, ball, false);
    if (st_ + 1 < J->n_steps) {
      for (int k = 0; k < EPW; k++) {
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
  }
  for (int k = 0; k < EPW; k++) {
    const int64_t e = eb + k;
    if (e >= n) break;
    Lane<T> L;
    T cf[3];
    pk_load_state<T>(wrec + k * ENV_STRIDE, lc, lane, L, cf);
    if (lane == 0) {
      T* rs = J->root + e * 13;
      for (int j = 0; j < 3; j++) { rs[j] = L.p[j]; rs[7 + j] = L.v[j]; rs[10 + j] = L.w[j]; }
      for (int j = 0; j < 4; j++) rs[3 + j] = L.Q[j];
    }
    if (lc.dyn && lane > 0) {
      T q[3];
      qlog(L.qj, q);
      for (int j = 0; j < 3; j++) { J->dof_pos[e * nd + lc.dof0 + j] = q[j]; J->dof_vel[e * nd + lc.dof0 + j] = L.wt[j]; }
    }
    if (lc.active) {
      T* rb = J->rb_out + (e * nb + lane) * 13;
      for (int j = 0; j < 3; j++) { rb[j] = L.p[j]; rb[7 + j] = L.v[j]; rb[10 + j] = L.w[j]; }
      for (int j = 0; j < 4; j++) rb[3 + j] = L.Q[j];
      if (J->contact_out) for (int j = 0; j < 3; j++) J->contact_out[(e * nb + lane) * 3 + j] = cf[j];
    }
  }
}
}  // namespace

template <typename T>
static int run_mixed(const b200_model_t* models, const float* const* verts, int num_assets, const int32_t* env_asset, const b200_cfg_t* cfg, int n,
                     int n_steps, T* root, T* dof_pos, T* dof_vel, const T* pd_tar, const T* ext, T* rb_out, T* contact_out) {
  std::vector<DevBlob> hb(num_assets);
  std::vector<std::vector<float>> soa(num_assets);
  std::vector<const float*> sv(num_assets);
  for (int a = 0; a < num_assets; a++) {
    int slots_ok = 1;
    if (build_dev_blob(&models[a], hb[a], &slots_ok) != 0 || !slots_ok || models[a].nb > B200_MAX_BODIES_PK) return -1;
    if (models[a].nb != models[0].nb || models[a].nd != models[0].nd) return -2;
    soa[a].assign((size_t)models[a].nb * models[a].vmax * 3 + 16, 0.0f);
    float* p = soa[a].data();
    while ((uintptr_t)p % 16) p++;
    verts_to_soa(&models[a], verts[a], p);
    sv[a] = p;
  }
  std::vector<const DevBlob*> eblob(n);
  std::vector<const float*> everts(n);
  for (int e = 0; e < n; e++) {
    if (env_asset[e] < 0 || env_asset[e] >= num_assets) return -3;
    eblob[e] = &hb[env_asset[e]];
    everts[e] = sv[env_asset[e]];
  }
  MixedJob<T> J{&hb[0], eblob.data(), everts.data(), cfg, n, n_steps, root, dof_pos, dof_vel, pd_tar, ext, rb_out, contact_out};
  std::vector<T> rec((size_t)EPW * ENV_STRIDE + 8, T(0));
  T* wrec = rec.data();
  while ((uintptr_t)wrec % 16) wrec++;
  for (int64_t eb = 0; eb < n; eb += EPW) {
    EmuWarp w;
    std::vector<std::thread> th;
    for (int lane = 0; lane < 32; lane++) th.emplace_back(lane_main_mixed<T>, &w, lane, &J, eb, wrec);
    for (auto& t : th) t.join();
  }
  return 0;
}

// models [num_assets], verts [num_assets] (AoS [nb][vmax][3] each), env_asset [n]; the other arguments as emu_packed_physics (no ball)
extern "C" int emu_mixed_physics(const b200_model_t* models, const float* const* verts, int num_assets, const int32_t* env_asset, const b200_cfg_t* cfg,
                                 int n, int n_steps, double* root, double* dof_pos, double* dof_vel, const double* pd_tar, const double* ext,
                                 double* rb_out, double* contact_out) {
  return run_mixed<double>(models, verts, num_assets, env_asset, cfg, n, n_steps, root, dof_pos, dof_vel, pd_tar, ext, rb_out, contact_out);
}
extern "C" int emu_mixed_physics_f32(const b200_model_t* models, const float* const* verts, int num_assets, const int32_t* env_asset,
                                     const b200_cfg_t* cfg, int n, int n_steps, float* root, float* dof_pos, float* dof_vel, const float* pd_tar,
                                     const float* ext, float* rb_out, float* contact_out) {
  return run_mixed<float>(models, verts, num_assets, env_asset, cfg, n, n_steps, root, dof_pos, dof_vel, pd_tar, ext, rb_out, contact_out);
}
