// emu_dof_force.cpp - TEST INFRASTRUCTURE: the DOF force sensor instantiation of the packed articulated step
// (control_step_packed<T, true>, csrc/packed.cuh::pk_dof_force) on the CPU lane emulator of emu_packed.cpp (one host thread per lane),
// as physics_kernel_packed<T, WARPS, true> runs it.  emu_dof_force_physics takes the arguments of emu_packed_physics plus
// dof_force [n][nd]; the library also exports emu_packed_physics itself, so that one build runs the step with the sensor and without.
// Built by tests/test_dof_force.py with the flags of tests/emu/build.py.
#include "emu_packed.cpp"

#if defined(EMU_PACKED3) || defined(EMU_PACKEDT)
#error "the DOF force sensor is built into the packed form only"
#endif

namespace {
// lane_main of emu_packed.cpp with the sensor: the lanes of env eb + g write its dof_force row after every control step
template <typename T> void lane_main_dof_force(EmuWarp* w, int lane, const Job<T>* J, int64_t eb, T* wrec) {
  emu_warp = w;
  emu_lane = lane;
  const DevBlob& B = *J->B;
  const b200_model_t& M = B.m;
  const int n = J->n, nb = M.nb, nd = M.nd;
  LaneConst lc = lane_const(M, lane);
  if (lc.active) lc.rix = B.t.rix[lane];
  PhysCfg<T> pc = make_phys_cfg<T>(*J->cfg);
  const bool with_ball = pc.has_ball && J->io.ball != nullptr;
  pc.has_ball = with_ball;
  const int g = lane / EMU_LPE, s = lane % EMU_LPE;
  for (int k = 0; k < EMU_EPW; k++) {
    const int64_t e = eb + k;
    if (e >= n) break;
    Lane<T> L;
    T pdt[3], eF[3], eT[3];
    env_arrays_load<T>(J->io, nd, lc, lane, e, L, pdt, eF, eT);
    pk_store_state<T>(wrec + k * ENV_STRIDE, lc, lane, L, pdt, eF, eT);
  }
  __syncwarp();
  const bool valid = g < EMU_EPW && eb + g < n;
  Ball<T> ball;
  ball_clear(ball);
  if (with_ball && valid && s == EMU_BALL_SLOT) env_arrays_load_ball<T>(J->io, eb + g, ball);
  T* const dof_force = valid ? J->io.dof_force + (eb + g) * nd : nullptr;
  for (int st_ = 0; st_ < J->n_steps; st_++) {
    control_step_packed<T, true>(B, M, J->verts, pc, wrec, lane, valid, ball, false, dof_force);
    if (st_ + 1 < J->n_steps) pk_requantize<T, EMU_EPW>(wrec, lc, lane, eb, n);
  }
  for (int k = 0; k < EMU_EPW; k++) {
    const int64_t e = eb + k;
    if (e >= n) break;
    Lane<T> L;
    T cf[3];
    pk_load_state<T>(wrec + k * ENV_STRIDE, lc, lane, L, cf);
    env_arrays_store<T>(J->io, nb, nd, lc, lane, e, L, cf);
  }
  if (with_ball && valid && s == EMU_BALL_SLOT) env_arrays_store_ball<T>(J->io, eb + g, ball);
}

template <typename T>
int run_dof_force(const b200_model_t* model, const float* verts, const b200_cfg_t* cfg, int n, int n_steps, T* root, T* dof_pos, T* dof_vel,
                  const T* pd_tar, const T* ext, T* rb_out, T* contact_out, T* ballio, int32_t* hits, T* dof_force) {
  DevBlob hb;
  int slots_ok = 1;
  if (!dof_force || build_dev_blob(model, hb, &slots_ok) != 0 || !slots_ok || model->nb > B200_MAX_BODIES_PK) return -1;
  hull_vertex_radius(model, verts, hb.t.vrho);
  hull_bounding_spheres(model, verts, hb.t.bs);
  if (g_face_planes) {
    hb.t.face_planes = g_face_planes;
    hb.t.face_tris = g_face_tris;
    hb.t.face_tmax = g_face_tmax;
    for (int b = 0; b < model->nb; b++) hb.t.ntris[b] = g_face_ntris[b];
  }
  std::vector<float> soa((size_t)model->nb * model->vmax * 3 + 16, 0.0f);
  float* sv = soa.data();
  while ((uintptr_t)sv % 16) sv++;
  verts_to_soa(model, verts, sv);
  const Job<T> J{&hb, sv, nullptr, nullptr, cfg, n, n_steps, {root, dof_pos, dof_vel, pd_tar, ext, rb_out, contact_out, ballio, hits, dof_force}};
  std::vector<T> rec((size_t)EMU_EPW * ENV_STRIDE + 8, T(0));
  T* wrec = rec.data();
  while ((uintptr_t)wrec % 16) wrec++;
  for (int64_t eb = 0; eb < n; eb += EMU_EPW) {
    EmuWarp w;
    std::vector<std::thread> th;
    for (int lane = 0; lane < 32; lane++) th.emplace_back(lane_main_dof_force<T>, &w, lane, &J, eb, wrec);
    for (auto& t : th) t.join();
  }
  return 0;
}
}  // namespace

extern "C" int emu_dof_force_physics(const b200_model_t* model, const float* verts, const b200_cfg_t* cfg, int n, int n_steps, double* root,
                                     double* dof_pos, double* dof_vel, const double* pd_tar, const double* ext, double* rb_out,
                                     double* contact_out, double* ballio, int32_t* hits, double* dof_force) {
  return run_dof_force<double>(model, verts, cfg, n, n_steps, root, dof_pos, dof_vel, pd_tar, ext, rb_out, contact_out, ballio, hits, dof_force);
}
extern "C" int emu_dof_force_physics_f32(const b200_model_t* model, const float* verts, const b200_cfg_t* cfg, int n, int n_steps, float* root,
                                         float* dof_pos, float* dof_vel, const float* pd_tar, const float* ext, float* rb_out,
                                         float* contact_out, float* ballio, int32_t* hits, float* dof_force) {
  return run_dof_force<float>(model, verts, cfg, n, n_steps, root, dof_pos, dof_vel, pd_tar, ext, rb_out, contact_out, ballio, hits, dof_force);
}
