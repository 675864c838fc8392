// emu_mixed.cpp - TEST INFRASTRUCTURE: the packed articulated step on the CPU (emu_packed.cpp: one host thread per lane) with envs of
// different assets of one topology in one warp, as step_kernel_packed<true, false, true> runs them: the tree tables of asset 0, the
// numeric constants and hull vertices of each env's own asset (control_step_packed's MN / verts per lane).  Built by
// tests/test_assets_mixed.py with the flags of tests/emu/build.py.
#include "emu_packed.cpp"

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
  return run_warps(Job<T>{&hb[0], sv[0], eblob.data(), everts.data(), cfg, n, n_steps,
                          {root, dof_pos, dof_vel, pd_tar, ext, rb_out, contact_out, nullptr, nullptr}});
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
