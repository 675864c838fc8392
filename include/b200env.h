/* b200env.h - C ABI of the H100-native vectorised humanoid(+ball) environment step.
 *
 * This is the drop-in boundary under the reference's Task surface (SURVEY.md 8b, "Level A").
 * The reference has no C ABI of its own: its tasks talk to Isaac Gym through pybind
 * (`gym.simulate`, `gym.set_dof_position_target_tensor`, `gym.apply_rigid_body_force_tensors`,
 * `gym.refresh_*_tensor`, `gym.set_*_tensor_indexed`, zero-copy `gymtorch.wrap_tensor` views).
 * Each entry point below names the reference interface it replaces (paths relative to
 * /root/reference).  The Python mirror of the Task classes (vid2player3d_b200/tasks) binds
 * these with ctypes; INTEGRATION.md shows the stub a reference maintainer would add.
 *
 * Conventions: plain pointers + sizes, no torch types.  All `float*` / `int64_t*` buffers are
 * DEVICE pointers owned by the caller (PyTorch storages), laid out exactly like the Isaac Gym
 * tensors the reference wraps, so the reference's view/slice code keeps working.  Quaternions
 * are xyzw, world is z-up.  Every call is asynchronous on `stream` (a cudaStream_t passed as
 * void*), allocates nothing, and never synchronises the host.  Return 0 = ok; otherwise a
 * negative code and b200env_last_error() describes it.
 */
#ifndef B200ENV_H
#define B200ENV_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200_MAX_BODIES 32
#define B200_MAX_DOF 96
#define B200_MAX_KEY 8
#define B200_ABI_VERSION 6

/* Per-asset constant block produced by vid2player3d_b200/model_compiler.py from the MJCF/STL
 * assets (replaces gym.load_asset + create_actor + set_actor_dof_properties:
 * embodied_pose/env/tasks/humanoid_smpl_im.py:273-300,356-389).  Followed in memory by
 * `float verts[nb][vmax][3]` (convex-hull vertices in the body frame). */
typedef struct b200_model {
  int32_t nb;        /* rigid bodies incl. welded ones (24, or 25 with Racket) */
  int32_t nd;        /* actuated dof = 3 * spherical joints (69) */
  int32_t vmax;      /* vertex stride per body */
  int32_t max_depth; /* tree depth of the deepest body (root = 0) */
  int32_t parent[B200_MAX_BODIES];
  int32_t depth[B200_MAX_BODIES];
  int32_t dof_of_body[B200_MAX_BODIES]; /* first dof index of the body's spherical joint, -1 = root / welded */
  int32_t fixed[B200_MAX_BODIES];       /* 1 = welded to its parent (no joint) */
  int32_t nverts[B200_MAX_BODIES];
  float offset[B200_MAX_BODIES][3];  /* joint position in the parent frame */
  float mass[B200_MAX_BODIES];       /* dynamics mass (welded children folded into parent, 0 for welded) */
  float com[B200_MAX_BODIES][3];
  float inertia[B200_MAX_BODIES][6]; /* about COM, body frame: xx yy zz xy xz yz */
  float radius[B200_MAX_BODIES];     /* bounding radius of the hull about the body origin */
  float kp[B200_MAX_DOF];            /* PD stiffness per dof, already scaled by mass/90*kp_scale */
  float kd[B200_MAX_DOF];
  float armature[B200_MAX_DOF];
  float lim_lo[B200_MAX_DOF];
  float lim_hi[B200_MAX_DOF];
} b200_model_t;

/* Simulation + task constants (replaces gymapi.SimParams / the yaml `sim:` block,
 * embodied_pose/utils/config.py:198-231, cfg/amass_im.yaml:37-52, and the env: block entries
 * read by humanoid_smpl_im.py:54-117). */
typedef struct b200_cfg {
  float sim_dt;             /* 1/60 */
  int32_t substeps;         /* 2 */
  int32_t control_freq_inv; /* 2 */
  float gravity_z;          /* -9.81 */
  float contact_kn, contact_cn, friction_mu, friction_vs; /* ground contact model (DESIGN.md) */
  float ang_damping, max_ang_vel;                         /* AssetOptions: 0.01, 100 */
  float limit_k, limit_c;                                 /* joint-limit spring/damper */
  float pd_tar_lim;                                       /* 0.5*pi (humanoid_smpl_im.py:73) */
  float res_force_scale, res_torque_scale;                /* 31.85 (cfg/amass_im.yaml:24) */
  int32_t max_episode_length;                             /* episodeLength */
  int32_t enable_early_termination;
  float termination_height[B200_MAX_BODIES];              /* humanoid_smpl_im.py:217-224 */
  int32_t contact_body[B200_MAX_BODIES];                  /* 1 = excluded from the fall test (contactBodies) */
  float body_pos_weight[B200_MAX_BODIES];                 /* humanoid_smpl_im.py:110-115 */
  float k_dof, k_vel, k_pos, k_rot, w_dof, w_vel, w_pos, w_rot; /* reward_specs :682 */
  int32_t num_key;
  int32_t key_body[B200_MAX_KEY];                         /* keyBodies */
  int32_t shape_dim;                                      /* motion_bodies width (11) */
  float ground_tolerance;
  /* --- vid2player physics player env (vid2player/env/tasks/humanoid_smpl_im_mvae.py) --- */
  int32_t task_mode;   /* 0: HumanoidSMPLIM (MoCap target + obs + reward + reset fused in the step)
                          1: HumanoidSMPLIMMVAE player step (:663-797): physics + ball, no task logic in the step */
  int32_t pd_mode;     /* 0: clamp(action, q +- lim) (embodied_pose :391-396); 1: clamp(target_dof + action, q +- lim) (:693-709) */
  int32_t has_ball;    /* 1: actor 1 of every env is the tennis ball (tennis_ball.urdf: r 0.032, m 0.057, I 4e-5) */
  int32_t racket_body; /* body index of the welded Racket (24), -1 = none */
  float ball_mass, ball_inertia, ball_radius, spin_scale;
  float ball_e_ground, ball_mu_ground, ball_e_racket, ball_mu_racket, bounce_threshold_velocity;
  float racket_head_center[3]; /* HEAD frame (see racket_head_quat): cylinder fromto="0 0 0 0 0.0425 0" size 0.15 (federer.xml:190) */
  float racket_head_halfthick, racket_head_radius;
  float racket_head_quat[4]; /* xyzw, racket frame -> head frame whose +y is the string-bed normal: identity for the right-handed
                                assets, 45 deg about x for nadal.xml's cylinder fromto="0 -.015 -.015 0 .015 .015" */
  /* --- optional: the other contacts of the ball (in the reference the ball collides with every shape of the env: collision filter 0,
   * humanoid_smpl_im_mvae.py:436-442).  Default off.  Bodies: exact sphere / convex-hull query against the faces installed with
   * b200env_set_hull_faces (a body without faces: every hull vertex is a sphere of half the mean vertex spacing); handle: the cylinder fromto="0.5 0 0 0.15 0 0" size 0.016 of the Racket body as a capsule.  The deepest contact of
   * a substep gets the impulse (restitution / Coulomb friction like the string bed); the obstacle is kinematic (no reaction on it). */
  int32_t ball_body_contact;
  float ball_e_body, ball_mu_body; /* PhysX "average" of the ball (0.9 / 0.2) and a default shape (0 / 1): 0.45, 0.6 */
  float racket_handle[7];          /* racket frame: p0[3], p1[3], radius; radius 0 = no handle */
} b200_cfg_t;

/* Reference MoCap buffer (embodied_pose/utils/motion_lib.py:68-93): flat device arrays. */
typedef struct b200_motion_lib {
  const float* gts;   /* [F,nb24,3] global translations */
  const float* grs;   /* [F,nb24,4] global rotations */
  const float* lrs;   /* [F,nb24,4] local rotations */
  const float* grvs;  /* [F,3] */
  const float* gravs; /* [F,3] */
  const float* dvs;   /* [F,nd] */
  const float* motion_lengths;  /* [M] */
  const int64_t* num_frames;    /* [M] */
  const float* motion_dt;       /* [M] */
  const int64_t* length_starts; /* [M] */
  const float* min_verts_h;     /* [M] */
  int32_t num_motions;
  int32_t num_lib_bodies; /* bodies per MoCap frame (24) */
  int64_t total_frames;
} b200_motion_lib_t;

/* Torch-owned state / output tensors.  Layouts mirror the Isaac Gym tensors the reference
 * wraps in _setup_tensors (embodied_pose/env/tasks/humanoid_smpl.py:66-113). */
typedef struct b200_buffers {
  float* root_states;      /* [N, actors_per_env, 13]  (humanoid = actor 0) */
  int32_t actors_per_env;
  float* dof_state;        /* [N, nd, 2] (pos, vel) */
  float* rigid_body_state; /* [N, bodies_per_env, 13] */
  float* contact_forces;   /* [N, bodies_per_env, 3] */
  int32_t bodies_per_env;  /* >= nb (ball appended in vid2player) */
  float* obs_buf;          /* [N, num_obs] */
  int32_t num_obs;
  float* rew_buf;          /* [N] */
  float* sub_rewards;      /* [N,4] */
  int64_t* reset_buf;      /* [N] */
  int64_t* progress_buf;   /* [N] */
  int64_t* terminate_buf;  /* [N] */
  const int64_t* motion_ids; /* [N] _reset_ref_motion_ids */
  float* ref_motion_times;   /* [N] _cur_ref_motion_times */
  const float* motion_bodies;/* [N, shape_dim] _reset_ref_motion_bodies */
  /* current targets (humanoid_smpl_im.py:594-624) */
  float *t_root_pos, *t_root_rot, *t_dof_pos, *t_root_vel, *t_root_ang_vel, *t_dof_vel, *t_key_pos, *t_rb_pos, *t_rb_rot;
  /* previous targets used by the reward (:626-636, :677-680) */
  float *p_dof_pos, *p_dof_vel, *p_rb_pos, *p_rb_rot;
  float* pd_targets;       /* [N, nd] last PD targets (set_dof_position_target_tensor argument) */
  float* actions_used;     /* [N, num_actions] actions after zeroing reset envs (self.actions) */
  int32_t num_actions;     /* row width of `actions` / `actions_used`: nd + 6 with a residual root wrench (res_force_scale > 0,
                              humanoid_smpl_im.py:111-112), nd without (the 6 residual columns are then neither read nor written) */
  /* vid2player player env only (may be NULL when cfg.has_ball == 0); bool tensors, 1 byte each */
  uint8_t* has_bounce;       /* [N] _has_bounce */
  uint8_t* has_bounce_now;   /* [N] _has_bounce_now (cleared at the start of every step, :688) */
  float* bounce_pos;         /* [N,3] _bounce_pos */
  uint8_t* racket_hit_now;   /* [N] exact racket-ball impact during this step (contact-force sensor path, :771-779) */
} b200_buffers_t;

typedef struct b200env* b200env_handle;

int b200env_abi_version(void);
const char* b200env_last_error(void);

/* replaces BaseTask.create_sim + gym.prepare_sim (base_task.py:48-49): builds nothing per env,
 * uploads the constant block once.  `model` and `verts` are HOST pointers. */
int b200env_create(const b200_model_t* model, const float* verts, const b200_cfg_t* cfg, int32_t num_envs,
                   int32_t device, b200env_handle* out);
int b200env_destroy(b200env_handle h);
/* replaces gym.acquire_*_tensor + gymtorch.wrap_tensor (humanoid_smpl.py:66-113) */
int b200env_bind(b200env_handle h, const b200_buffers_t* bufs);
/* replaces torch.load(motion_lib) residency (humanoid_smpl_im.py:420-440) */
int b200env_set_motion_lib(b200env_handle h, const b200_motion_lib_t* ml);

/* replaces BaseTask.step = pre_physics_step + _physics_step + post_physics_step
 * (base_task.py:147-165; humanoid_smpl_im.py:125-157,398-418): ONE fused launch.
 * actions: [N, b200_buffers_t::num_actions] device. */
int b200env_step(b200env_handle h, const float* actions, void* stream);

/* replaces HumanoidSMPLIM._reset_envs for ref-state init (humanoid_smpl_im.py:442-450,489-528,
 * 741-755; humanoid_smpl.py:153-173): env_ids [n] int64 device, motion_times [n] float device
 * (sampled by the host like MotionLib.sample_time). */
int b200env_reset(b200env_handle h, const int64_t* env_ids, const float* motion_times, int32_t n, void* stream);

/* replaces MotionLib.get_motion_state(..., return_rigid_body=True, adjust_height=True)
 * (motion_lib.py:164-266) for arbitrary (id, time) pairs, e.g. _init_context
 * (humanoid_smpl_im.py:530-563).  Any output pointer may be NULL. */
int b200env_motion_state(b200env_handle h, const int64_t* motion_ids, const float* motion_times, int32_t n,
                         float* root_pos, float* root_rot, float* dof_pos, float* root_vel, float* root_ang_vel,
                         float* dof_vel, float* key_pos, float* rb_pos, float* rb_rot, void* stream);

/* replaces compute_humanoid_observations_imitation (humanoid_smpl_im.py:773-850 ==
 * models/im_network_builder.py:262-338): obs [n,1+..=734 for 24 bodies].  Bit 1 of `local_root_obs` selects the
 * 'joint_pos' variant compute_humanoid_observations_imitation_jpos (:853-915, 513 wide). */
int b200env_obs_imitation(b200env_handle h, int32_t n, const float* body_pos, const float* body_rot,
                          const float* target_pos, const float* target_rot, const float* dof_pos, const float* dof_vel,
                          const float* target_dof_pos, const float* body_vel, const float* body_ang_vel,
                          const float* motion_bodies, int32_t local_root_obs, int32_t root_height_obs, float* obs,
                          void* stream);

/* The same observation computed straight from the Isaac-layout state rows the env owns - rigid_body_state [n, bodies_per_env, 13]
 * (pos 0:3, rot 3:7, vel 7:10, ang vel 10:13; the first `humanoid bodies` rows of every env are used) and dof_state [n, nd, 2] -
 * instead of six contiguous gathers of them (what the reference's slicing + cat amounts to, humanoid_smpl_im_mvae.py:862-895).
 * obs_bf16 (may be NULL): additionally writes the policy's first-layer operand row, bf16(clamp((obs - mean) * rstd, -clamp, clamp)),
 * [n, ld_bf16] (RunningMeanStd + the +-5 clamp of ImitatorPlayer.run_one_step, vid2player/players/im_player.py:187-190; mean /
 * rstd NULL = no normalisation), so that the network forward (include/b200nn.h) starts without a cast launch. */
int b200env_obs_imitation_rows(b200env_handle h, int32_t n, const float* rigid_body_state, int32_t bodies_per_env, const float* dof_state,
                               const float* target_pos, const float* target_rot, const float* target_dof_pos, const float* motion_bodies,
                               int32_t local_root_obs, int32_t root_height_obs, float* obs, void* obs_bf16, int32_t ld_bf16, const float* mean,
                               const float* rstd, float clamp, void* stream);

/* Physics-only control step on caller-provided arrays, float (prec=0) or double (prec=1): a separate test launch
 * (physics_kernel_packed; physics_kernel_tmem / physics_kernel for the other forms) that shares the control step
 * (control_step_packed) with b200env_step's physics launch, but not that launch's persistent hand-out of env batches,
 * its state-row loads and stores or its shared-memory layout.  Exposed so tests can compare the control step with the
 * float64 CPU restatement (oracle/physics_ref.c).  root [n,13], dof_pos/dof_vel/pd_tar [n,nd],
 * ext_wrench [n,6] (force, torque on body 0, world frame, first sim step only),
 * rb_out [n,nb,13], contact_out [n,nb,3].  n_steps control steps are run back to back.
 * ball: in/out [n,13] (pos, quat unused, lin vel, ang vel) or NULL; ball_hits [n] counts racket impacts (or NULL). */
int b200env_physics_only(b200env_handle h, int32_t prec, int32_t n, int32_t n_steps, void* root, void* dof_pos,
                         void* dof_vel, const void* pd_tar, const void* ext_wrench, void* rb_out, void* contact_out,
                         void* ball, int32_t* ball_hits, void* stream);

/* replaces HumanoidSMPLIM._init_context (embodied_pose/env/tasks/humanoid_smpl_im.py:530-563): for listed env i and frame
 * j in [0, num_frames): t = motion_times[i] + dt + (first_frame + j) * dt; writes
 * context_feat[row, j, :] = rb_pos | rb_rot | dof_pos | rb_pos | dof_pos  ([N, num_frames, 2*(3B+D)+4B] row-major) and
 * context_mask[row, j] = t <= motion_length + 2 dt, with row = env_ids[i] (or i when env_ids is NULL). */
int b200env_motion_context(b200env_handle h, const int64_t* env_ids, const int64_t* motion_ids, const float* motion_times, int32_t n,
                           int32_t num_frames, int32_t first_frame, float dt, float* context_feat, uint8_t* context_mask, void* stream);

/* Heterogeneous assets per env (dual mode: env 2k = player 0's asset, env 2k+1 = player 1's,
 * vid2player/env/tasks/humanoid_smpl_im_mvae.py:270-275 `motion_ids[1::2] = 1`): one handle per asset, all bound to the SAME
 * tensors; handle-local env i of b200env_step is row env_first + env_stride * i.  num_envs at create = envs of the slice. */
int b200env_set_env_slice(b200env_handle h, int32_t env_first, int32_t env_stride);

/* Faces of every body's convex hull, for the exact sphere / convex-hull query of the ball against the humanoid's bodies
 * (cfg.ball_body_contact; PhysX collides the ball's sphere shape with the convex meshes of the asset the reference loads with
 * default AssetOptions - one convex hull per mesh, vid2player/env/tasks/humanoid_smpl.py:277-283).  planes [nb, tmax, 4] float (outward unit normal n, offset d: n.x <= d
 * inside), tris [nb, tmax, 4] uint8 (three vertex indices into the body's hull vertices, outward winding, one pad byte),
 * ntris [nb] int32 (0: body keeps the sphere-per-vertex approximation).  HOST pointers; copied.  Without this call every body
 * uses the approximation. */
int b200env_set_hull_faces(b200env_handle h, const float* planes, const uint8_t* tris, const int32_t* ntris, int32_t tmax);

/* Which form of the physics launch this handle uses: 0 lane-per-body kernel, 1 step_kernel_packed (32 envs per SM in the split form:
 * two rounds for 8192 envs on 132 SMs), 2 packed3 (A/B builds only), 3 step_kernel_tmem (56 envs per SM, lane-private fields in thread-local memory).  Chosen at
 * b200env_create from the model's tree and the environment variable B200ENV_KERNEL (lane | packed | tmem; default: see DESIGN.md 5). */
int32_t b200env_kernel_form(b200env_handle h);

/* Shape of b200env_step's physics launch for this handle: *envs_per_batch = envs a CTA takes per ticket (32 for the split
 * step_kernel_packed, 28 for the fused form, 56 for step_kernel_tmem, 8 for the lane-per-body kernel), *grid = resident CTA slots
 * of the persistent launch (CTAs per SM x SMs).  A step of n envs runs min(*grid, ceil(n / *envs_per_batch)) CTAs, so batch b of
 * the env order runs in round b / *grid.  Computed from the same expressions b200env_step uses; needs the device, not a bind. */
int b200env_physics_launch_shape(b200env_handle h, int32_t* envs_per_batch, int32_t* grid);

/* Several assets of one topology in one handle (replaces the per-env actors of HumanoidSMPLIM._create_envs, each built from its
 * motion's body: embodied_pose/env/tasks/humanoid_smpl_im.py:231-351, PD gains scaled by that actor's mass :356-389).  models [num_assets]
 * and verts [num_assets] (verts[a]: [nb][models[a].vmax][3]) are HOST arrays; env e is simulated with asset env_asset[e] for the
 * handle's lifetime.  Every asset must have asset 0's topology (nb, nd, max_depth, parent, depth, fixed, dof_of_body); vmax, the
 * vertices and every numeric field may differ.  The physics launch hands out the batches of b200env_plan_assets (at most 32 envs of
 * one asset each) and re-stages the asset's header in shared memory when a CTA moves to a batch of another asset; every other launch
 * reads the topology only.  Not supported with several assets (refused with an error): cfg.has_ball, the non-default kernel forms
 * (B200ENV_KERNEL=lane|tmem|packed3, B200ENV_SPLIT=0, B200ENV_SORT=1), b200env_set_env_slice, b200env_set_hull_faces and
 * b200env_physics_only. */
int b200env_create_assets(const b200_model_t* models, const float* const* verts, int32_t num_assets, const int32_t* env_asset,
                          const b200_cfg_t* cfg, int32_t num_envs, int32_t device, b200env_handle* out);

/* The batch plan of b200env_create_assets, host only (no device needed): rows [num_envs] = the envs grouped by asset (ascending env
 * index inside an asset), then one batch per up to envs_per_batch consecutive rows of one asset: batch i covers rows
 * [batch_first[i], batch_first[i] + batch_count[i]) of asset batch_asset[i].  Asset a gets ceil(n_a / envs_per_batch) batches (none
 * when n_a = 0), in ascending asset order.  The batch arrays need room for num_envs entries; *num_batches receives their number. */
int b200env_plan_assets(const int32_t* env_asset, int32_t num_envs, int32_t num_assets, int32_t envs_per_batch, int32_t* rows,
                        int32_t* batch_asset, int32_t* batch_first, int32_t* batch_count, int32_t* num_batches);

/* The plan a handle of b200env_create_assets runs (batch b runs in round b / grid of b200env_physics_launch_shape).  Array
 * arguments may be NULL (query the sizes first: rows has num_envs entries, the batch arrays *num_batches).  Fails on a handle of
 * b200env_create. */
int b200env_asset_plan(b200env_handle h, int32_t* num_assets, int32_t* num_batches, int32_t* rows, int32_t* batch_asset,
                       int32_t* batch_first, int32_t* batch_count);

/* number of kernels launched by this handle so far (bench.py "gpu_launches") */
int64_t b200env_launch_count(b200env_handle h);

/* Measurement aid (bench.py `roofline.kernel_ms`): with timing on, b200env_step records a CUDA event pair around the physics launch
 * (step_kernel_packed / step_kernel_packed3 / the fused kernel) on the launching stream.  b200env_kernel_ms synchronises the recorded
 * events, returns the mean duration in ms of the launches since the last call (or since timing was switched on) in *mean_ms and their
 * number in *count, and clears the record.  At most 4096 launches are kept between two reads; not for use inside a CUDA graph capture. */
int b200env_set_kernel_timing(b200env_handle h, int32_t on);
int b200env_kernel_ms(b200env_handle h, double* mean_ms, int32_t* count);

#ifdef __cplusplus
}
#endif
#endif /* B200ENV_H */
