// emu_packed.cpp - TEST INFRASTRUCTURE: the packed articulated step (csrc/packed*.cuh) executed on the CPU, one host thread per
// lane, in float64, behind the same signature as b200env_physics_only.  Lets a new lane mapping of the kernel be checked against
// the float64 restatement (oracle/physics_ref.c) without a GPU.  Built by tests/emu/build.py (g++ -O1 -pthread -shared).
#include "cuda_compat.h"

thread_local EmuWarp* emu_warp = nullptr;
thread_local int emu_lane = 0;

#include "../../vid2player3d_b200/csrc/dyn_common.cuh"
#ifdef EMU_PACKED3
#include "../../tools/variants/packed3.cuh"
#define EMU_EPW EPW3
#define EMU_LPE LPE3
#define EMU_BALL_SLOT BALL_SLOT3
#define EMU_STEP(B, MN, ...) control_step_packed3<T>(B, __VA_ARGS__)   // one asset: MN is B.m
#else
#include "../../vid2player3d_b200/csrc/packed.cuh"
#ifdef EMU_PACKEDT
#include "../../vid2player3d_b200/csrc/packed_t.cuh"   // one-wave form: private fields in a per-lane array here (PrivMem), a thread-local array on the GPU
#endif
#define EMU_EPW EPW
#define EMU_LPE PK_LANES_PER_ENV
#define EMU_BALL_SLOT BALL_SLOT
#define EMU_STEP(B, MN, ...) control_step_packed<T>(B, MN, __VA_ARGS__)
#endif

#include <vector>

namespace {
template <typename T> struct Job {
  const DevBlob* B;                 // the model; envs of several assets (emu_mixed.cpp): asset 0's, whose tree tables they share
  const float* verts;
  const DevBlob* const* env_blob;   // several assets: [n] the header of env e's asset (its numeric constants), else null
  const float* const* env_verts;    // several assets: [n] its SoA hull vertices, else null
  const b200_cfg_t* cfg;
  int n, n_steps;
  EnvArrays<T> io;
};

// one warp = the body of physics_kernel_packed<double> (b200env.cu) for envs eb .. eb + EPW - 1; with several assets each lane steps
// with its env's model, as step_kernel_packed<true, false, true> does
template <typename T> void lane_main(EmuWarp* w, int lane, const Job<T>* J, int64_t eb, T* wrec) {
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
  const int64_t me = valid ? eb + g : eb;   // a lane without an env takes the warp's first env's model, as the kernel does
  const b200_model_t& MN = J->env_blob ? J->env_blob[me]->m : M;
  const float* verts = J->env_verts ? J->env_verts[me] : J->verts;
  Ball<T> ball;
  ball_clear(ball);
  if (with_ball && valid && s == EMU_BALL_SLOT) env_arrays_load_ball<T>(J->io, eb + g, ball);
  for (int st_ = 0; st_ < J->n_steps; st_++) {
    EMU_STEP(B, MN, verts, pc, wrec, lane, valid, ball, false);
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

#ifdef EMU_PACKEDT
// one warp = the body of physics_kernel_tmem (b200env.cu) for envs eb .. eb + EPW - 1, private store = priv (one array per lane)
template <typename T> void lane_main_t(EmuWarp* w, int lane, const Job<T>* J, int64_t eb, T* wrec, T* priv) {
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
  PrivMem<T> ps{priv + (size_t)lane * PT_WARP_COLS};
  for (int k = 0; k < EMU_EPW; k++) {
    const int64_t e = eb + k;
    if (e >= n) break;
    Lane<T> L;
    T pdt[3], eF[3], eT[3];
    env_arrays_load<T>(J->io, nd, lc, lane, e, L, pdt, eF, eT);
    pt_stage_in<T>(wrec + k * PT_ENV_STRIDE, lc, lane, L, pdt, eF, eT);
  }
  __syncwarp();
  const bool valid = g < EMU_EPW && eb + g < n;
  pt_adopt<T>(B, wrec, lane, valid, ps);
  Ball<T> ball;
  ball_clear(ball);
  if (with_ball && valid && s == EMU_BALL_SLOT) env_arrays_load_ball<T>(J->io, eb + g, ball);
  T* cf_env = (valid && J->io.contact_out) ? J->io.contact_out + (eb + g) * nb * 3 : nullptr;
  for (int st_ = 0; st_ < J->n_steps; st_++) {
    control_step_t<T>(B, J->verts, pc, wrec, lane, valid, ball, ps, cf_env, false);
    if (st_ + 1 < J->n_steps) pt_requantize<T>(B, lane, valid, ps);
  }
  pt_publish<T>(B, wrec, lane, valid, ps);
  __syncwarp();
  for (int k = 0; k < EMU_EPW; k++) {
    const int64_t e = eb + k;
    if (e >= n) break;
    Lane<T> L;
    pt_load_state<T>(wrec + k * PT_ENV_STRIDE, lc, lane, L);
    env_arrays_store<T>(J->io, nb, nd, lc, lane, e, L, nullptr);
  }
  if (with_ball && valid && s == EMU_BALL_SLOT) env_arrays_store_ball<T>(J->io, eb + g, ball);
}
#endif

// the warps of J, one after the other (each warp: 32 host threads)
template <typename T> int run_warps(const Job<T>& J) {
#ifdef EMU_PACKEDT
  if (!J.B->t.pt_ok) return -2;
  std::vector<T> rec((size_t)EMU_EPW * PT_ENV_STRIDE + 8, T(0)), priv((size_t)32 * PT_WARP_COLS, T(0));
#else
  std::vector<T> rec((size_t)EMU_EPW * ENV_STRIDE + 8, T(0));
#endif
  T* wrec = rec.data();
  while ((uintptr_t)wrec % 16) wrec++;   // the records are read with 128-bit accesses on the float path
  for (int64_t eb = 0; eb < J.n; eb += EMU_EPW) {
    EmuWarp w;
    std::vector<std::thread> th;
#ifdef EMU_PACKEDT
    for (int lane = 0; lane < 32; lane++) th.emplace_back(lane_main_t<T>, &w, lane, &J, eb, wrec, priv.data());
#else
    for (int lane = 0; lane < 32; lane++) th.emplace_back(lane_main<T>, &w, lane, &J, eb, wrec);
#endif
    for (auto& t : th) t.join();
  }
  return 0;
}
}  // namespace

// hull faces of the exact ball / hull query (b200env_set_hull_faces on the product side): host arrays kept by the caller
static const float* g_face_planes = nullptr;
static const unsigned char* g_face_tris = nullptr;
static const int32_t* g_face_ntris = nullptr;
static int g_face_tmax = 0;
extern "C" void emu_set_hull_faces(const float* planes, const unsigned char* tris, const int32_t* ntris, int tmax) {
  g_face_planes = planes; g_face_tris = tris; g_face_ntris = ntris; g_face_tmax = tmax;
}

template <typename T>
static int run(const b200_model_t* model, const float* verts, const b200_cfg_t* cfg, int n, int n_steps, T* root, T* dof_pos, T* dof_vel,
               const T* pd_tar, const T* ext, T* rb_out, T* contact_out, T* ballio, int32_t* hits) {
  DevBlob hb;
  int slots_ok = 1;
  if (build_dev_blob(model, hb, &slots_ok) != 0 || !slots_ok || model->nb > B200_MAX_BODIES_PK) return -1;
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
  while ((uintptr_t)sv % 16) sv++;   // contact_hull reads the vertices with 128-bit loads
  verts_to_soa(model, verts, sv);
  return run_warps(Job<T>{&hb, sv, nullptr, nullptr, cfg, n, n_steps, {root, dof_pos, dof_vel, pd_tar, ext, rb_out, contact_out, ballio, hits}});
}

// float64: the parity instantiation (vs oracle/physics_ref.c to round-off); float32: the arithmetic the product kernel runs
// (host libm instead of the MUFU approximations of rcp_ / rsqrt_)
extern "C" int emu_packed_physics(const b200_model_t* model, const float* verts, const b200_cfg_t* cfg, int n, int n_steps, double* root,
                                  double* dof_pos, double* dof_vel, const double* pd_tar, const double* ext, double* rb_out,
                                  double* contact_out, double* ballio, int32_t* hits) {
  return run<double>(model, verts, cfg, n, n_steps, root, dof_pos, dof_vel, pd_tar, ext, rb_out, contact_out, ballio, hits);
}
extern "C" int emu_packed_physics_f32(const b200_model_t* model, const float* verts, const b200_cfg_t* cfg, int n, int n_steps, float* root,
                                      float* dof_pos, float* dof_vel, const float* pd_tar, const float* ext, float* rb_out,
                                      float* contact_out, float* ballio, int32_t* hits) {
  return run<float>(model, verts, cfg, n, n_steps, root, dof_pos, dof_vel, pd_tar, ext, rb_out, contact_out, ballio, hits);
}

// owner-slot tables of the one-wave form (DevTree::pt_*, csrc/dyn_common.cuh::build_pt_tables) for a model: tests/test_emu_packed.py checks
// their invariants on the shipped assets and on a tree that does not fit
extern "C" int emu_pt_tables(const b200_model_t* model, int8_t* blk, int8_t* slot, int8_t* body, int8_t* lvl, int8_t* lblk, int8_t* mbox,
                             int32_t* nmbox) {
  static DevBlob hb;
  int slots_ok = 1;
  if (build_dev_blob(model, hb, &slots_ok) != 0) return -1;
  memcpy(blk, hb.t.pt_blk, sizeof(hb.t.pt_blk)); memcpy(slot, hb.t.pt_slot, sizeof(hb.t.pt_slot));
  memcpy(body, hb.t.pt_body, sizeof(hb.t.pt_body)); memcpy(lvl, hb.t.pt_lvl, sizeof(hb.t.pt_lvl));
  memcpy(lblk, hb.t.pt_lblk, sizeof(hb.t.pt_lblk)); memcpy(mbox, hb.t.pt_mbox, sizeof(hb.t.pt_mbox));
  *nmbox = hb.t.pt_nmbox;
  return hb.t.pt_ok;
}

// The exact ball / convex-hull query on its own: form 0 = hull_sphere (one lane walks the hull), form 1 = hull_sphere_coop (the hull's faces
// over the 8 lanes of a group; 4 groups = 4 query points per emulated warp).  Float64.  centres [n][3] in the body frame of `body`;
// out_hit [n], out_pen [n], out_nl [n][3].  Faces from emu_set_hull_faces.
namespace {
struct HsJob { const float* sv; int vmax; const float* pl; const unsigned char* tr; int nt; const double* c; double R; int n, form; int32_t* hit; double* pen; double* nl; };
void hs_lane(EmuWarp* w, int lane, const HsJob* J, int q0) {
  emu_warp = w;
  emu_lane = lane;
  const int g = lane >> 3, s = lane & 7, q = q0 + g;
  const bool act = q < J->n;
  double c[3] = {0, 0, 0}, pen = 0, nl[3] = {0, 0, 1};
  if (act) for (int k = 0; k < 3; k++) c[k] = J->c[q * 3 + k];
  bool hit;
  if (J->form == 1) hit = hull_sphere_coop<double>(J->sv, J->vmax, J->pl, J->tr, J->nt, c, J->R, s, act, pen, nl);
  else hit = act && s == 0 && hull_sphere<double>(J->sv, J->vmax, J->pl, J->tr, J->nt, c, J->R, pen, nl);
  if (act && s == (J->form == 1 ? 5 : 0)) {       // any lane of the group holds the cooperative result: take lane 5's
    J->hit[q] = hit ? 1 : 0; J->pen[q] = pen;
    for (int k = 0; k < 3; k++) J->nl[q * 3 + k] = nl[k];
  }
}
}  // namespace
extern "C" int emu_hull_sphere(const b200_model_t* model, const float* verts, int body, int form, int n, const double* centres, double R,
                               int32_t* out_hit, double* out_pen, double* out_nl) {
  if (!g_face_planes || g_face_ntris[body] <= 0) return -1;
  std::vector<float> soa((size_t)model->nb * model->vmax * 3 + 16, 0.0f);
  float* sv = soa.data();
  while ((uintptr_t)sv % 16) sv++;
  verts_to_soa(model, verts, sv);
  HsJob J{sv + (size_t)body * model->vmax * 3, model->vmax, g_face_planes + (size_t)body * g_face_tmax * 4, g_face_tris + (size_t)body * g_face_tmax * 4,
          g_face_ntris[body], centres, R, n, form, out_hit, out_pen, out_nl};
  for (int q0 = 0; q0 < n; q0 += 4) {
    EmuWarp w;
    std::vector<std::thread> th;
    for (int lane = 0; lane < 32; lane++) th.emplace_back(hs_lane, &w, lane, &J, q0);
    for (auto& t : th) t.join();
  }
  return 0;
}
