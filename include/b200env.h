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
#define B200_ABI_VERSION 11

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
  int32_t shape_dim;                                      /* motion_bodies width (11); create refuses it outside [0, 32] */
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
  /* DOF force sensors (enable_actor_dof_force_sensors + acquire_dof_force_tensor, embodied_pose/env/tasks/humanoid_smpl_im.py:369,
   * humanoid_smpl.py:77-78), NULL = none.  [N, nd]: dof_force[e, 3j + k] = the generalized force joint j's PD drive and its limit
   * spring-damper applied during the LAST substep of the step, in the joint's child frame (the frame of the dof velocities), taken at
   * the end-of-substep velocity qd+ = qd + h qdd of the implicit drive: kp (pd - q - h qd+) - kd qd+ [+ limk (lim - q - h qd+) - limc qd+
   * while a limit is active].  Armature (inertia), contact and joint-reaction forces are not part of it.  Written by the physics
   * launch of b200env_step (rows of the handle's env slice only); b200env_bind refuses it for the A/B kernel forms
   * (B200ENV_KERNEL=lane|tmem|packed3, B200ENV_SPLIT=0). */
  float* dof_force;
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

/* HumanoidSMPLIM._reset_actors + _init_context (humanoid_smpl_im.py:470-563) for every env e < num_envs with mask[e] != 0, driven by
 * the device mask instead of an id list: no host synchronisation, two launches, replayable inside a CUDA graph.
 * Draws: u_k = (bits(seed, *counter, 2e + k) >> 40) * 2^-24 with bits = splitmix64(splitmix64(seed ^ counter * 0xD1B54A32D192ED03) + idx).
 * u_1 < ref_prob: ref-state init at t = 0 (sample_time 0) or t = u_0 * max(motion_length - truncate, 0) in float32 (sample_time 1,
 * MotionLib.sample_time); the rows are written exactly as b200env_reset writes them at (e, t), reset_times[e] = t, and the
 * context window exactly as b200env_motion_context writes it for (e, motion_ids[e], t, num_frames, first_frame, dt).
 * Otherwise default init (_reset_default :482-487): root row = init_root[e] ([N,13]), dof pos / vel = init_dof_pos[e] /
 * init_dof_vel[e] ([N,nd]), progress / reset / terminate = 0, raw obs from the new dofs and the rigid-body rows as they stand;
 * init_* may be NULL when ref_prob >= 1.  Rows whose mask is clear are not touched.
 * counter: [1] int64 device, advanced by 1 by every call; work: [num_envs + 2] int32 device, zero before the first call (each call
 * leaves its counters zero).
 * The xf_* fields and feat_width are the transform program of the window (B200_XF_* below, as b200env_motion_context applies it);
 * both launches read the same *counter, so its draws are those b200env_motion_context makes for (e, frame, body) at that counter. */
typedef struct b200_reset_masked {
  int32_t sample_time;     /* 0: ref-state init at t = 0, 1: at a drawn time */
  float truncate, ref_prob;
  int32_t num_frames, first_frame;
  float dt;
  uint64_t seed;
  const uint8_t* mask;     /* [num_envs] */
  int64_t* counter;        /* [1] */
  const float *init_root, *init_dof_pos, *init_dof_vel; /* NULL when ref_prob >= 1 */
  float* reset_times;      /* [num_envs] */
  float* context_feat;     /* [num_envs, num_frames, W] */
  uint8_t* context_mask;   /* [num_envs, num_frames] */
  int32_t* work;           /* [num_envs + 2] */
  /* transform program, appended within ABI version 11; all zero = no transforms, rows W wide */
  int32_t xf_ops[3];
  uint32_t xf_joint_mask;
  float xf_noisy_prob, xf_noise_std, xf_conf_std, xf_min_conf, xf_random_prob;
  int32_t feat_width;
  /* window offset of a game restarted mid-run (b200env_im_motion_queue), appended within ABI version 11; step NULL = the window above.
   * With step set, s = step[0] % context_length and the window of env e is the one b200env_motion_context writes for (e, motion_ids[e],
   * reset_times[e], num_frames, first_frame - s, dt): frame j at t = reset_times[e] + dt + (first_frame - s + j) dt.  The policy reads
   * slot context_padding + step % context_length (b200env_im_policy_rows), so the restarted game's next step reads the frame at
   * reset_times[e] + dt, bit for bit the frame a game the full reset started reads at step 0.  Frames before time 0 clamp to frame 0. */
  const int64_t* step;     /* [1] b200_play_stats_t::step, or NULL */
  int32_t context_length;  /* >= 1 when step is set */
  int32_t pad_;
} b200_reset_masked_t;
int b200env_reset_masked(b200env_handle h, const b200_reset_masked_t* d, void* stream);

/* replaces MotionLib.get_motion_state(..., return_rigid_body=True, adjust_height=True)
 * (motion_lib.py:164-266) for arbitrary (id, time) pairs, e.g. _init_context
 * (humanoid_smpl_im.py:530-563).  Any output pointer may be NULL. */
typedef struct b200_motion_state {
  int32_t n, pad_;
  const int64_t* motion_ids;   /* [n] */
  const float* motion_times;   /* [n] */
  float *root_pos, *root_rot, *dof_pos, *root_vel, *root_ang_vel, *dof_vel, *key_pos, *rb_pos, *rb_rot;
} b200_motion_state_t;
int b200env_motion_state(b200env_handle h, const b200_motion_state_t* d, void* stream);

/* replaces compute_humanoid_observations_imitation (humanoid_smpl_im.py:773-850 ==
 * models/im_network_builder.py:262-338): obs [n,1+..=734 for 24 bodies].  jpos != 0 selects the 'joint_pos' variant
 * compute_humanoid_observations_imitation_jpos (:853-915, 513 wide).  Returns -2 before any launch when the row is wider than 768
 * columns or the humanoid has more than 32 bodies (one lane per body). */
typedef struct b200_obs_imitation {
  int32_t n, local_root_obs, root_height_obs, jpos;
  const float *body_pos, *body_rot, *target_pos, *target_rot, *dof_pos, *dof_vel, *target_dof_pos, *body_vel, *body_ang_vel;
  const float* motion_bodies;
  float* obs;
} b200_obs_imitation_t;
int b200env_obs_imitation(b200env_handle h, const b200_obs_imitation_t* d, void* stream);

/* The same observation computed straight from the Isaac-layout state rows the env owns - rigid_body_state [n, bodies_per_env, 13]
 * (pos 0:3, rot 3:7, vel 7:10, ang vel 10:13; the first `humanoid bodies` rows of every env are used) and dof_state [n, nd, 2] -
 * instead of six contiguous gathers of them (what the reference's slicing + cat amounts to, humanoid_smpl_im_mvae.py:862-895).
 * obs_bf16 (may be NULL): additionally writes the policy's first-layer operand row, bf16(clamp((obs - mean) * rstd, -clamp, clamp)),
 * [n, ld_bf16] (RunningMeanStd + the +-5 clamp of ImitatorPlayer.run_one_step, vid2player/players/im_player.py:187-190; mean /
 * rstd NULL = no normalisation), so that the network forward (include/b200nn.h) starts without a cast launch.  jpos selects the
 * 'joint_pos' variant, as above.  Returns -2 before any launch on the refusals of b200env_obs_imitation, and when obs_bf16 is given
 * with ld_bf16 smaller than the row width, an odd ld_bf16 or an address that is not 4-byte aligned (the row is stored as bf16 pairs). */
typedef struct b200_obs_rows {
  int32_t n, bodies_per_env, local_root_obs, root_height_obs, jpos, ld_bf16;
  float clamp;
  float clamp1;                   /* b200env_obs_imitation_rows_dual: player 1's clamp (clamp is player 0's); ignored otherwise */
  const float *rigid_body_state, *dof_state, *target_pos, *target_rot, *target_dof_pos, *motion_bodies;
  float* obs;
  void* obs_bf16;                 /* NULL: no operand row */
  const float *mean, *rstd;       /* NULL: no normalisation */
} b200_obs_rows_t;
int b200env_obs_imitation_rows(b200env_handle h, const b200_obs_rows_t* d, void* stream);
/* The same launch for the two players of a rally (envs 2k and 2k+1), each with its own trained low-level policy
 * (ImitatorBuilderDual.Network.eval_actor, vid2player/models/im_network_builder_dual.py:37-45): env e's operand row is
 * (e & 1) * n/2 + (e >> 1), so each player's rows are one block, and player e & 1 uses row e & 1 of mean / rstd ([2, row width]) and
 * clamp (player 0) or clamp1 (player 1); the float row stays in env order.  A clamp may be inf (RunningNorm at n == 0: no clamp).
 * Returns -2 before any launch on the refusals of b200env_obs_imitation_rows, on an odd n and on a clamp or clamp1 that is not
 * positive. */
int b200env_obs_imitation_rows_dual(b200env_handle h, const b200_obs_rows_t* d, void* stream);

/* The imitation policy's first-layer operand at test time (ImitatorBuilder.Network.preprocess_input, non-training branch, + running_obs,
 * embodied_pose/models/im_network_builder.py:117-189): the 734-wide observation of compute_humanoid_observations_imitation with
 * local_root_obs = root_height_obs = 1, built from
 *   - obs_buf [n, num_obs], the raw observation the step writes, split as obs_names / obs_dims (body_pos | body_rot | dof_pos | dof_vel |
 *     body_vel | body_ang_vel | motion_bodies, humanoid_smpl_im.py:198-211); every value is clamped to +-clip_obs as it is loaded (the
 *     wrapper's torch.clamp(obs_buf, -clip_obs, clip_obs); inf = no clamp);
 *   - the target body_pos | body_rot | dof_pos of frame context_padding + (step[0] % context_length) of context_feat [n, num_frames,
 *     feat_width] (the window b200env_motion_context writes; forward_context(flatten=False) + obtain_cur_context(t) :117-145).
 * Writes x [n, ld] bf16 = clamp((obs - mean) * rstd, -clip, clip) (RunningNorm / RunningMeanStd; mean / rstd NULL: the row as it is, no
 * clamp) and resid [n, nd] = the slot's target dof_pos (the residual action of eval_actor :226-228, added by the last GEMM layer's
 * epilogue, include/b200nn.h).  `step` is a device counter (b200env_play_stats advances it), so one capture replays every step. */
typedef struct b200_im_policy {
  int32_t n;               /* envs: rows 0 .. n-1 of every array */
  int32_t num_obs;         /* row stride of obs_buf (>= the 7 named blocks) */
  int32_t num_frames;      /* frames of a context window (context_length + 2 context_padding) */
  int32_t feat_width;      /* floats of a context frame (>= 7 bodies + dofs: body_pos | body_rot | dof_pos | ...) */
  int32_t context_padding;
  int32_t context_length;
  int32_t ld;              /* bf16 elements per row of x: even, >= the observation width */
  float clip_obs;          /* clamp of the raw observation; inf = none */
  float clip;              /* the normaliser's clamp (with mean / rstd only) */
  int32_t pad_;
  const float* obs_buf;
  const float* context_feat;
  const int64_t* step;     /* [1] */
  const float* mean;       /* [734] or NULL */
  const float* rstd;       /* [734] or NULL */
  void* x;                 /* bf16, 4-byte aligned */
  float* resid;            /* [n, nd] */
} b200_im_policy_t;

/* One launch (the observation launch's per-env warp code, obs_imitation_kernel).  Returns -2 before any launch on the refusals of
 * b200env_obs_imitation, an ld smaller than the row, odd or an x that is not 4-byte aligned, an obs_buf row narrower than the named
 * blocks, a context frame narrower than its three target blocks, a slot outside the window (context_padding < 0, context_length < 1 or
 * context_padding + context_length > num_frames), mean without rstd or a normaliser clamp that is not positive.  A handle of several
 * assets is served: the launch reads only the topology they share. */
int b200env_im_policy_rows(b200env_handle h, const b200_im_policy_t* d, void* stream);

/* ImitatorPlayer.run's bookkeeping of one step (embodied_pose/players/im_player.py:226-304, num_agents = 1), one CTA in a fixed
 * summation order (replays give the same sums).  Per env: done = reset_buf != 0, cr += rew, steps += 1, step_done = done (1 - prev_done).
 * When any step_done is set: totals += (sum cr, sum steps) over them (double), games[0] += their count, cr *= 1 - done,
 * steps *= 1 - done, and (count, sum cr, sum steps) is appended to log [max_log, 3] at row games[2] (games[2] += 1; a full log keeps
 * counting but writes nothing).  The float sums are summed in float32, like the reference's cr[done].sum().  Then prev_done = done,
 * games[1] (stop) = games[0] >= n_games or done of env 0, and step[0] += 1.  While games[1] is set the call changes nothing.
 * Queue form (queue_games > 0, b200env_im_motion_queue): games[1] = games[0] >= queue_games instead; env 0's done does not stop the
 * run, since a finished env takes the next queued game. */
typedef struct b200_play_stats {
  int32_t n;
  int32_t max_log;
  int64_t n_games;         /* games_num * n_game_life */
  const float* rew;        /* [n] */
  const int64_t* reset_buf;/* [n] */
  float* cr;               /* [n] */
  float* steps;            /* [n] */
  float* prev_dones;       /* [n] */
  double* totals;          /* [2]: sum_rewards, sum_steps */
  double* log;             /* [max_log, 3] */
  int64_t* games;          /* [3]: games_played, stop, log rows */
  int64_t* step;           /* [1] */
  int64_t queue_games;     /* appended within ABI version 11: 0 = the rule above, else the queued games of the run (R M) */
} b200_play_stats_t;

int b200env_play_stats(const b200_play_stats_t* d, void* stream);
/* sizeof(b200_play_stats_t) as the library was built; the binding refuses a library whose size differs from its own */
int32_t b200env_play_stats_desc_size(void);

/* The motion queue of an imitation test run over a library larger than the env count (HumanoidSMPLIMVis with
 * cfg.env.b200_motion_queue; an addition, the reference's ImitatorPlayer.run never resets an env mid-game).  The queue holds the
 * entries q = r M + m (r < R rounds, m < M motions) in that order; entries below *cursor are taken.  One CTA walks the envs in env
 * order, in chunks of its threads: the k-th env (k = 0, 1, ...) whose reset_buf is set and whose idle byte is clear gets entry
 * q = *cursor + k when q < queue_len, and then
 *   motion_ids[e] = q % M, entry[e] = q, motion_bodies[e] = lib_motion_bodies[q % M], game_env[q] = e, game_start_step[q] = step[0]
 *   (the step counter b200env_play_stats advanced: the index of the new game's first step), mask[e] = 1, and the done memory of
 *   the new game is cleared, prev_dones[e] = 0 (b200_play_stats_t) and env_flags[e, 0] = 0 (b200_im_motion_stats_t, when given),
 *   as the host clears them before a full reset, so a game that ends on its first step is counted too;
 * otherwise (the queue is empty) idle[e] = 1: the env is never reset again and its reset_buf stays set (the step keeps a done env
 * done), so the bookkeeping counts its last game once.  mask[e] = 0 for every other env, and *cursor advances once, by the entries
 * taken.  No atomics: the same flags give the same assignment.  The caller then resets the masked envs (b200env_reset_masked with
 * its step field, so each restarted window is aligned with the policy's slot).  games: b200_play_stats_t::games or NULL; while
 * games[1] (stop) is set the launch clears the mask and changes nothing else.  Returns -1 on a NULL pointer but games and env_flags,
 * -2 before
 * any launch when n, num_motions or queue_len is not positive, or shape_dim is outside [0, 32].
 * Bodies (motion_asset and env_asset, appended within ABI version 11; both NULL = the launch above): an env that takes entry q also
 * gets env_asset[e] = motion_asset[q % M], the asset of its next motion; an idle env and a stopped run change nothing.  The caller
 * then re-points the handle's asset table (b200env_set_env_assets) before the masked reset, so the next physics launch steps each
 * restarted env with its new motion's body.  -1 when only one of the two is set. */
typedef struct b200_im_motion_queue {
  int32_t n;                       /* envs */
  int32_t num_motions;             /* M */
  int64_t queue_len;               /* R M */
  int32_t shape_dim;               /* columns of motion_bodies */
  int32_t pad_;
  const int64_t* reset_buf;        /* [n] */
  const float* lib_motion_bodies;  /* [M, shape_dim] */
  int64_t* motion_ids;             /* [n] */
  float* motion_bodies;            /* [n, shape_dim] */
  int64_t* entry;                  /* [n]: the entry each env plays */
  uint8_t* mask;                   /* [n]: the envs to reset */
  uint8_t* idle;                   /* [n] */
  int64_t* cursor;                 /* [1] */
  int64_t* game_env;               /* [queue_len] */
  int64_t* game_start_step;        /* [queue_len] */
  const int64_t* step;             /* [1] b200_play_stats_t::step */
  const int64_t* games;            /* [3] or NULL */
  float* prev_dones;               /* [n] b200_play_stats_t::prev_dones */
  int32_t* env_flags;              /* [n, 2] b200_im_motion_stats_t::env_flags, or NULL */
  const int32_t* motion_asset;     /* [M]: the asset of each motion, or NULL */
  int32_t* env_asset;              /* [n]: the asset each env is simulated with, or NULL */
} b200_im_motion_queue_t;
int b200env_im_motion_queue(const b200_im_motion_queue_t* d, void* stream);
/* sizeof(b200_im_motion_queue_t) as the library was built; the binding refuses a library whose size differs from its own */
int32_t b200env_im_motion_queue_desc_size(void);

/* The training resample of HumanoidSMPLIM (cfg.env.b200_resample_motions; an addition, the reference draws each env's motion once):
 * before a reset, every env e < n with mask[e] != 0 and progress_buf[e] > 0 (it played at least one step) draws a new motion from the
 * distribution whose running sum is cdf [M] (b200env_motion_weights writes it; it need not end at 1):
 *   u = (bits(seed', c, e) >> 11) * 2^-53, with bits = splitmix64(splitmix64(seed' ^ c * 0xD1B54A32D192ED03) + e) as in
 *   b200env_reset_masked, c = *counter, and seed' = splitmix64(seed ^ 0x6D6F74696F6E6964) (seed is the caller's seed, the one the
 *   masked reset takes; the constant is "motionid" in ASCII), so the draw shares no key with the masked reset's or the transforms';
 *   the new motion m is the smallest with cdf[m] > u * cdf[M - 1], clamped to M - 1 (a motion with no weight is not drawn);
 *   motion_ids[e] = m, motion_bodies[e] = lib_motion_bodies[m], and env_asset[e] = motion_asset[m] when both are given.
 * Counts (tries and fails, both or neither): before the draw, tries[old] += 1 and fails[old] += (terminate_buf[e] != 0) for the motion
 * old = motion_ids[e] the env just finished; integer atomics, so the counts do not depend on the order.  Every other env is untouched.
 * One thread per env; the last CTA advances *counter by 1 and re-arms the done ticket ([1], zero before the first call).  The caller
 * then re-points the handle's assets (b200env_set_env_assets) and resets the masked envs.  Returns -1 on a NULL required pointer or
 * one pointer of a pair, -2 before any launch when n or num_motions is not positive or shape_dim lies outside [0, 32]. */
typedef struct b200_resample_motions {
  int32_t n;                       /* envs */
  int32_t num_motions;             /* M */
  int32_t shape_dim;               /* columns of motion_bodies */
  int32_t pad_;
  uint64_t seed;
  const uint8_t* mask;             /* [n] */
  const int64_t* progress_buf;     /* [n] */
  const int64_t* terminate_buf;    /* [n] */
  const double* cdf;               /* [M] */
  const float* lib_motion_bodies;  /* [M, shape_dim] */
  int64_t* motion_ids;             /* [n] */
  float* motion_bodies;            /* [n, shape_dim] */
  int64_t* counter;                /* [1] */
  uint32_t* done;                  /* [1] */
  int64_t* tries;                  /* [M] or NULL */
  int64_t* fails;                  /* [M] or NULL */
  const int32_t* motion_asset;     /* [M] or NULL */
  int32_t* env_asset;              /* [n] or NULL */
} b200_resample_motions_t;
int b200env_resample_motions(const b200_resample_motions_t* d, void* stream);
/* sizeof(b200_resample_motions_t) as the library was built; the binding refuses a library whose size differs from its own */
int32_t b200env_resample_motions_desc_size(void);

/* The motion distribution of the training resample, rebuilt from the failure counts (cfg.env.b200_hard_motion_share = h), in one CTA
 * with no host synchronisation.  b_m = base[m] (double), or 1 when base is NULL.  With h > 0: for every motion with tries[m] > 0,
 * rate[m] = fails[m] / tries[m] (double); the others keep theirs; then tries and fails are zeroed.  Then
 *   p_m = (1 - h) b_m / S_b + h b_m rate[m] / S_br, with S_b = sum b, S_br = sum b rate, or p_m = b_m / S_b when S_br = 0 or h = 0,
 * and cdf[m] = p_0 + ... + p_m, written in place.  The sums and the scan run in double in a fixed order (each thread a run of
 * consecutive motions, then a tree over the threads), so every call on the same inputs writes the same bits.  tries, fails and rate
 * may be NULL when h = 0 (the base distribution).  Returns -1 on a NULL cdf, or a NULL count or rate with h > 0; -2 before any
 * launch when num_motions is not positive or h is not a finite number in [0, 1]. */
typedef struct b200_motion_weights {
  int32_t num_motions;             /* M */
  int32_t pad_;
  double h;
  const float* base;               /* [M] or NULL (uniform) */
  int64_t* tries;                  /* [M] */
  int64_t* fails;                  /* [M] */
  double* rate;                    /* [M] */
  double* cdf;                     /* [M] */
} b200_motion_weights_t;
int b200env_motion_weights(const b200_motion_weights_t* d, void* stream);
/* sizeof(b200_motion_weights_t) as the library was built; the binding refuses a library whose size differs from its own */
int32_t b200env_motion_weights_desc_size(void);

/* One recorded frame of HumanoidSMPLIMVis._sync_ref_motion (embodied_pose/env/tasks/humanoid_smpl_im_vis.py:128-152) for every listed
 * env: the qpos the reference's MuJoCo viewer shows, without the viewer.  One warp per recorded env i (row env_ids[i]); frame
 * f = *frame.  With nq = 7 + nd and J = nd / 3, row (i, f) of qpos [n_rec, cap, 2, nq] gets
 *   copy 0: rigid_body_state[e, 0] pos, its quaternion xyzw as wxyz, then the euler angles of dof_pos[e] (the dof_state column);
 *   copy 1: init = 0: the root row of p_rb_pos / p_rb_rot and the euler angles of p_dof_pos[e]; init = 1: copy 0; then x += 1.
 * The viewer's third copy (copy 0 with z += 1000) is left to the host.  The euler angles of a joint's rotation vector a are konia's
 * angle_axis_to_quaternion (theta = sqrt(max(|a|^2, 1e-6)), k = sin(theta / 2) / theta, w = cos(theta / 2); |a| = 0: (1, 0, 0, 0))
 * and ypr_euler_from_quat (atan2 with 1e-6 added to y when |y| and |x| are both below 1e-6, asin of the argument clamped to
 * +-(1 - 1e-6)), computed in double from the float32 state and stored yaw, pitch, roll (the [2, 1, 0] reorder of its roll, pitch, yaw).  rec_motion_ids / rec_reset [n_rec, cap] get motion_ids[e] and reset_buf[e] (0 with init).
 * The last CTA advances *frame by one (the ticket `done` is re-armed), so one CUDA graph capture replays every frame.
 * games: b200_play_stats_t::games or NULL.  While games[1] (stop) is set, or *frame >= cap, the launch writes nothing and does not
 * advance; the launch that writes frame cap - 1 sets games[1], so the bookkeeping of the same step changes nothing.  NULL: no stop flag.
 * Returns -2 before any launch when n_rec, cap or num_envs is not positive, nd is not a positive multiple of 3, or num_bodies or
 * num_lib_bodies is below 1.  env_ids must lie in [0, num_envs): the launch does not check them. */
typedef struct b200_im_record {
  int32_t n_rec;           /* recorded envs E */
  int32_t num_envs;        /* rows of the state arrays */
  int32_t num_bodies;      /* bodies per env of rigid_body_state */
  int32_t num_lib_bodies;  /* bodies per env of p_rb_pos / p_rb_rot */
  int32_t nd;              /* dofs: 3 per joint */
  int32_t cap;             /* frames of the record buffers */
  int32_t init;            /* 1: render_vis(init=True) */
  int32_t pad_;
  const int64_t* env_ids;          /* [n_rec] */
  const float* rigid_body_state;   /* [num_envs, num_bodies, 13] */
  const float* dof_state;          /* [num_envs, nd, 2] */
  const float* p_dof_pos;          /* [num_envs, nd] */
  const float* p_rb_pos;           /* [num_envs, num_lib_bodies, 3] */
  const float* p_rb_rot;           /* [num_envs, num_lib_bodies, 4] */
  const int64_t* reset_buf;        /* [num_envs] */
  const int64_t* motion_ids;       /* [num_envs] */
  float* qpos;                     /* [n_rec, cap, 2, 7 + nd] */
  int64_t* rec_motion_ids;         /* [n_rec, cap] */
  int64_t* rec_reset;              /* [n_rec, cap] */
  int64_t* frame;                  /* [1] */
  uint32_t* done;                  /* [1] ticket, 0 between launches */
  int64_t* games;                  /* [3] or NULL */
} b200_im_record_t;
int b200env_im_record(const b200_im_record_t* d, void* stream);
/* sizeof(b200_im_record_t) as the library was built; the binding refuses a library whose size differs from its own */
int32_t b200env_im_record_desc_size(void);

/* Per-motion meters of one test step (HumanoidSMPLIMVis.run_test with cfg.env.b200_motion_stats): the step's reward, its four
 * sub-rewards (compute_humanoid_reward, embodied_pose/env/tasks/humanoid_smpl_im.py:919-955) and the body-position error, summed per
 * game and folded, when the game ends, into the bucket of the env's motion.  Two launches in a fixed order, no float atomics, so a
 * replay gives the same bits:
 *   accumulate, one warp per env e: env_sums[e] += (rew, 1, sub_rewards[e, 0..3], err) in double, where err is the mean over the
 *     num_lib_bodies bodies b of |rigid_body_state[e, b, 0:3] - target_rb_pos[e, b]| (metres, computed in double); then, with
 *     done = reset_buf[e] != 0 (b200env_play_stats' rule), env_flags[e] = (done, ended), ended = done (1 - prev_done) ? 1 +
 *     (terminate_buf[e] != 0) : 0;
 *   fold, one CTA per motion m: over motion_envs[motion_start[m] .. motion_start[m + 1]), in that order, every env with ended != 0
 *     adds (1, ended == 2) to counts[m] (games, falls) and env_sums[e] to sums[m], then its env_sums row and ended are zeroed.
 * The caller zeroes env_sums and env_flags when a game starts, as b200env_play_stats' cr / steps / prev_dones.  games:
 * b200_play_stats_t::games or NULL; while games[1] (stop) is set neither launch changes anything.  Each env must appear exactly once
 * in motion_envs: the launch does not check the lists.  Returns -2 before any launch when n or num_motions is not positive or
 * num_lib_bodies is not in [1, num_bodies].
 *
 * Pose metrics (cfg.env.b200_pose_metrics; all five pose pointers set, or all NULL for the meters alone): with p_b the simulated and
 * r_b the target position of body b < num_lib_bodies (body 0 the root), the accumulate launch also adds, per frame, the means over
 * the bodies of
 *   l   = |(p_b - p_0) - (r_b - r_0)|                                          root-relative MPJPE
 *   pa  = |s R (p_b - mean p) + mean r - r_b|                                  PA-MPJPE: s, R the similarity of HMR/SPIN's
 *         compute_similarity_transform (proper rotation), s = 0 when the simulated bodies have no spread (var1 = 0)
 *   vel = |(p_t - p_t-1) - (r_t - r_t-1)|                                      from the game's second frame on
 *   acc = |(p_t - 2 p_t-1 + p_t-2) - (r_t - 2 r_t-1 + r_t-2)|                  from the game's third frame on
 * in double to env_pose[e] (with the frame counts of vel and acc), and keeps in env_pose[e, 6] the game's largest err (the
 * body-position error above), NaN once a frame has a non-finite error.  The previous two frames are kept in pose_hist (float, as
 * the positions arrive) with pose_fill frames valid; a game's end (ended != 0) empties it.  The fold adds the env_pose sums of the
 * finished games to pose_sums[m], takes the largest of their maxima into pose_sums[m, 6] (NaN if one is NaN), counts in success[m]
 * the games whose maximum is <= success_threshold (so not NaN), and zeroes the env's row.  The caller zeroes env_pose and pose_fill
 * when a game starts.  One warp per env with lane b on body b: returns -2 when num_lib_bodies > 32 or success_threshold is not a
 * finite positive number, and -1 when only some pose pointers are NULL, all after the checks above. */
#define B200_IM_MOTION_METERS_FIELDS                                                                                              \
  int32_t n;                       /* envs */                                                                                       \
  int32_t num_motions;             /* M */                                                                                          \
  int32_t num_bodies;              /* bodies per env of rigid_body_state */                                                         \
  int32_t num_lib_bodies;          /* bodies compared: rows per env of target_rb_pos */                                             \
  const float* rew;                /* [n] */                                                                                        \
  const float* sub_rewards;        /* [n, 4]: dof, vel, body_pos, body_rot */                                                       \
  const int64_t* reset_buf;        /* [n] */                                                                                        \
  const int64_t* terminate_buf;    /* [n]: 1 = the episode ended in a fall */                                                       \
  const float* rigid_body_state;   /* [n, num_bodies, 13] */                                                                        \
  const float* target_rb_pos;      /* [n, num_lib_bodies, 3]: the targets the step's reward compared against (p_rb_pos) */          \
  const int64_t* motion_start;     /* [M + 1] */                                                                                    \
  const int64_t* motion_envs;      /* [n]: the envs of each motion, grouped by motion, in env order within one */                   \
  double* env_sums;                /* [n, 7]: rew, steps, sub_rewards[4], err of the game so far */                                 \
  int32_t* env_flags;              /* [n, 2]: prev_done, ended */                                                                   \
  int64_t* counts;                 /* [M, 2]: games, falls */                                                                       \
  double* sums;                    /* [M, 7]: the env_sums columns of the finished games */                                         \
  const int64_t* games;            /* [3] or NULL */
/* the meters' fields alone: the parameter of the meters' kernels.  A by-value kernel parameter over 128 bytes is read through its
 * address instead of being loaded up front, so the meters' kernels take these 120 bytes and not the whole descriptor. */
typedef struct b200_im_motion_stats {
  B200_IM_MOTION_METERS_FIELDS
} b200_im_motion_meters_t;
typedef struct b200_im_motion_stats_desc {
  B200_IM_MOTION_METERS_FIELDS
  double* env_pose;                /* [n, 7] or NULL: l, pa, vel, acc sums, vel frames, acc frames, largest err of the game so far */
  float* pose_hist;                /* [n, 2, 2, num_lib_bodies, 3] or NULL: frames t-1, t-2 of (simulated, target) positions */
  int32_t* pose_fill;              /* [n] or NULL: frames of pose_hist that hold this game's positions, 0..2 */
  double* pose_sums;               /* [M, 7] or NULL: the env_pose columns of the finished games, column 6 their largest err */
  int64_t* success;                /* [M] or NULL: finished games whose largest err is <= success_threshold */
  double success_threshold;        /* metres */
} b200_im_motion_stats_t;
int b200env_im_motion_stats(const b200_im_motion_stats_t* d, void* stream);
/* sizeof(b200_im_motion_stats_t) as the library was built; the binding refuses a library whose size differs from its own */
int32_t b200env_im_motion_stats_desc_size(void);

/* The same meters with the motion queue (b200env_im_motion_queue): the rows of counts, sums, pose_sums and success are the queue's
 * entries (meters.num_motions = R M rows) and meters.motion_start / motion_envs are not read (may be NULL).  The accumulate launch is
 * the one above; the fold, one thread per env, adds each game that ended in this step to row env_entry[e], which must lie in
 * [0, R M), with the column rules above.  Every entry is played once, so every row has one writer and needs no atomics.  Refusals of
 * b200env_im_motion_stats, and -1 when env_entry is NULL. */
typedef struct b200_im_motion_queue_stats {
  b200_im_motion_stats_t meters;
  const int64_t* env_entry;        /* [n]: the entry each env plays */
} b200_im_motion_queue_stats_t;
int b200env_im_motion_queue_stats(const b200_im_motion_queue_stats_t* d, void* stream);
/* sizeof(b200_im_motion_queue_stats_t) as the library was built; the binding refuses a library whose size differs from its own */
int32_t b200env_im_motion_queue_stats_desc_size(void);

/* Physics-only control step on caller-provided arrays, float (prec=0) or double (prec=1): a separate test launch
 * (physics_kernel_packed; physics_kernel_tmem / physics_kernel for the other forms) that shares the control step
 * (control_step_packed) with b200env_step's physics launch, but not that launch's persistent hand-out of env batches,
 * its state-row loads and stores or its shared-memory layout.  Exposed so tests can compare the control step with the
 * float64 CPU restatement (oracle/physics_ref.c).  root [n,13], dof_pos/dof_vel/pd_tar [n,nd],
 * ext_wrench [n,6] (force, torque on body 0, world frame, first sim step only),
 * rb_out [n,nb,13], contact_out [n,nb,3].  n_steps control steps are run back to back.
 * ball: in/out [n,13] (pos, quat unused, lin vel, ang vel) or NULL; ball_hits [n] counts racket impacts (or NULL).
 * dof_force_out: [n,nd] in the precision of prec, the DOF force sensor of the last control step (b200_buffers_t::dof_force), or NULL;
 * refused like the sensor at b200env_bind on a handle of an A/B kernel form. */
int b200env_physics_only(b200env_handle h, int32_t prec, int32_t n, int32_t n_steps, void* root, void* dof_pos,
                         void* dof_vel, const void* pd_tar, const void* ext_wrench, void* rb_out, void* contact_out,
                         void* ball, int32_t* ball_hits, void* stream, void* dof_force_out);

/* replaces HumanoidSMPLIM._init_context (embodied_pose/env/tasks/humanoid_smpl_im.py:530-563): for listed env i and frame
 * j in [0, num_frames): t = motion_times[i] + dt + (first_frame + j) * dt; writes
 * context_feat[row, j, :] = rb_pos | rb_rot | dof_pos | rb_pos | dof_pos  ([N, num_frames, 2*(3B+D)+4B] row-major) and
 * context_mask[row, j] = t <= motion_length + 2 dt, with row = env_ids[i] (or i when env_ids is NULL).
 *
 * Transform program (HumanoidSMPLIM._transform_target, humanoid_smpl_im.py:565-592, cfg.env.transform_specs): xf_ops[0..2] lists up
 * to three of B200_XF_MASK_JOINTS / B200_XF_NOISY_JOINTS / B200_XF_MASK_RANDOM_JOINTS in the cfg's order, each at most once, ended by
 * 0.  feat_width is the row width of context_feat: 0 or W = 2 (3 nb + nd) + 4 nb without a program, W + nb (the joint_conf block
 * appended) with one.  Lane b of frame j of row e starts from pos = body_pos[b], conf = local = 1 and applies the ops in order:
 *   MASK_JOINTS:   bit b of xf_joint_mask set: local = 0, and conf = 0 while no NOISY_JOINTS ran before; then pos *= local
 *                  (the reference zeroes and multiplies by its local joint_conf tensor, which NOISY_JOINTS stops aliasing);
 *   NOISY_JOINTS:  noise = z * (u0 < xf_noisy_prob ? xf_noise_std : 0), z = three N(0, 1) draws; pos += noise;
 *                  conf = erfc(|noise| / (sqrt 3 xf_conf_std) / sqrt 2); conf < xf_min_conf: conf = 0, pos = 0;
 *   MASK_RANDOM_JOINTS: b > 0 and u4 < xf_random_prob: conf = 0 (and local, while aliased), pos = 0.
 * The row is body_pos (transformed) | body_rot | dof_pos | body_pos_gt | dof_pos_gt | conf; every frame is transformed whatever its
 * mask.  Draws: bits(seed, *counter, 2 num_envs + ((e P + j) nb + b) 5 + k), u_k = (bits >> 40) 2^-24 for k = 0, 4 and z = the
 * Box-Muller normal of counter_rng.cuh for k = 1..3; the offset 2 num_envs keeps them clear of b200env_reset_masked's 2e + k.  This
 * launch reads *counter and does not advance it.  Returns -2 before any launch on a repeated or unknown op, an op after a 0, a prob
 * outside [0, 1], xf_conf_std <= 0 or xf_noise_std < 0 with NOISY_JOINTS, a feat_width other than W or W + nb (W + nb with ops),
 * and counter NULL with NOISY_JOINTS or MASK_RANDOM_JOINTS.  A zeroed program is the window without transforms. */
#define B200_XF_MASK_JOINTS 1
#define B200_XF_NOISY_JOINTS 2
#define B200_XF_MASK_RANDOM_JOINTS 3
typedef struct b200_motion_context {
  int32_t n, num_frames, first_frame;
  float dt;
  const int64_t* env_ids;      /* [n] or NULL */
  const int64_t* motion_ids;   /* [n] */
  const float* motion_times;   /* [n] */
  float* context_feat;
  uint8_t* context_mask;
  /* transform program, appended within ABI version 11; all zero = no transforms, rows W wide */
  int32_t xf_ops[3];
  uint32_t xf_joint_mask;
  float xf_noisy_prob, xf_noise_std, xf_conf_std, xf_min_conf, xf_random_prob;
  int32_t feat_width;
  uint64_t seed;
  const int64_t* counter;      /* [1], or NULL without draws */
} b200_motion_context_t;
int b200env_motion_context(b200env_handle h, const b200_motion_context_t* d, void* stream);

/* sizeof(b200_reset_masked_t) and sizeof(b200_motion_context_t) as the library was built: both grew by appended fields within ABI
 * version 11, and the binding refuses a library whose sizes differ from its own. */
int32_t b200env_reset_masked_desc_size(void);
int32_t b200env_motion_context_desc_size(void);

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
 * and verts [num_assets] (verts[a]: [nb][models[a].vmax][3]) are HOST arrays; env e is simulated with asset env_asset[e], for the
 * handle's lifetime unless the handle is fixed to the mixed plan (b200env_fix_mixed_plan), whose b200env_set_env_assets moves envs to
 * other assets of the handle on the device.  Every asset must have asset 0's topology (nb, nd, max_depth, parent, depth, fixed, dof_of_body); vmax, the
 * vertices and every numeric field may differ.  The physics launch runs one of two plans:
 *  - grouped (b200env_plan_assets): batches of at most 32 envs of one asset each; a CTA re-stages the asset's header in shared memory
 *    when it moves to a batch of another asset;
 *  - mixed (b200env_plan_assets_mixed): batches of 32 consecutive envs whatever their assets; each env's lanes read the numeric
 *    constants and hull vertices of its own asset from global memory.
 * The mixed plan runs exactly when it takes fewer rounds of the persistent grid (b200env_choose_asset_plan with the grid of
 * b200env_physics_launch_shape); the environment variable B200ENV_ASSET_PLAN=grouped|mixed overrides that rule for A/B measurements
 * and tests.  The results of both plans are bit-identical.  Every other launch reads the topology only.  Not supported with several assets (refused with an error): cfg.has_ball, the non-default kernel forms
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

/* The mixed batch plan of b200env_create_assets, host only, same arguments and outputs as b200env_plan_assets: rows = 0 .. num_envs-1
 * (ascending env index, whatever the asset), batch i covers rows [i * envs_per_batch, ...) up to envs_per_batch of them;
 * batch_asset[i] = the asset of its envs when they all have one, else -1.  ceil(num_envs / envs_per_batch) batches. */
int b200env_plan_assets_mixed(const int32_t* env_asset, int32_t num_envs, int32_t num_assets, int32_t envs_per_batch, int32_t* rows,
                              int32_t* batch_asset, int32_t* batch_first, int32_t* batch_count, int32_t* num_batches);

/* The plan rule of b200env_create_assets, host only: *mixed = 1 when ceil(ceil(num_envs / B) / grid) < ceil(sum_a ceil(n_a / B) / grid),
 * i.e. when the mixed plan takes fewer rounds of a persistent grid of `grid` CTAs than the grouped plan (B = 32 envs per batch in
 * both, n_a = envs of asset a), else 0. */
int b200env_choose_asset_plan(const int32_t* env_asset, int32_t num_envs, int32_t num_assets, int32_t grid, int32_t* mixed);

/* The plan a handle of b200env_create_assets runs (batch b runs in round b / grid of b200env_physics_launch_shape); *mixed = 1 for
 * the mixed plan, 0 for the grouped one.  Array arguments and mixed may be NULL (query the sizes first: rows has num_envs entries,
 * the batch arrays *num_batches).  Fails on a handle of b200env_create.  batch_asset describes the env_asset of b200env_create_assets:
 * after b200env_set_env_assets a mixed batch's envs may run other assets. */
int b200env_asset_plan(b200env_handle h, int32_t* num_assets, int32_t* num_batches, int32_t* rows, int32_t* batch_asset,
                       int32_t* batch_first, int32_t* batch_count, int32_t* mixed);

/* Setup call on a handle of b200env_create_assets, before its first step: the handle runs the mixed plan for its lifetime, whatever
 * the rule (or B200ENV_ASSET_PLAN) chose, so that b200env_set_env_assets may re-point its envs' assets on the device (the mixed plan's
 * batches do not depend on the assignment; the grouped plan's do).  Host work and one device allocation, like create: the env ->
 * asset-header table of the mixed plan when the grouped plan had been chosen.  Both plans give bit-identical results.  Afterwards
 * b200env_asset_plan reports mixed = 1 and the mixed batches of the creation-time assignment.  Returns -2 on a handle of
 * b200env_create (one asset); calling it twice is allowed. */
int b200env_fix_mixed_plan(b200env_handle h);

/* Re-point the assets of the envs of a handle fixed to the mixed plan, on the device: one thread per env sets env e's entry of the
 * asset-header table to asset env_asset[e] (an index into the models of b200env_create_assets), read by every physics launch from the
 * next one on.  An index outside [0, num_assets) leaves that env's asset as it was and, when *error is 0, sets *error = e + 1 (the
 * first such env the launch met; the word keeps it until the caller clears it).  No allocation, no host synchronisation: graph-safe.
 * Returns -1 on a NULL pointer, -2 before any launch on a handle not fixed to the mixed plan or when n is not the handle's env count. */
typedef struct b200_set_env_assets {
  int32_t n;                       /* envs: the handle's num_envs */
  int32_t pad_;
  const int32_t* env_asset;        /* [n] */
  int32_t* error;                  /* [1] */
} b200_set_env_assets_t;
int b200env_set_env_assets(b200env_handle h, const b200_set_env_assets_t* d, void* stream);
/* sizeof(b200_set_env_assets_t) as the library was built; the binding refuses a library whose size differs from its own */
int32_t b200env_set_env_assets_desc_size(void);

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
