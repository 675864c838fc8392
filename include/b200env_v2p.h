/* b200env_v2p.h - C ABI of the vid2player rows of the rollout hot path (SURVEY.md 8a, a10-a17).
 * Stateless entry points: plain device pointers + sizes, asynchronous on `stream`, no allocation, no host sync.
 * Bool tensors are 1 byte per element (torch.bool storage).  Paths below are relative to /root/reference/vid2player. */
#ifndef B200ENV_V2P_H
#define B200ENV_V2P_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

const char* b200v2p_last_error(void);

/* replaces HumanoidSMPLIMMVAE._smpl_to_sim + _forward_kinematics (env/tasks/humanoid_smpl_im_mvae.py:897-946, utils/hybrik.py:597-652):
 * joint_rotmat [n,24,3,3] and rest [num_rest,24,3] in SMPL joint order (env e uses shape e % num_rest: 1 = one player,
 * 2 = dual mode's alternating players, n = a shape per env); outputs in MuJoCo body order (smpl_2_mujoco);
 * prev_* NULL -> zero velocities.  prev_root_pos_update / target_root_pos_out (either may be NULL): after the finite difference the
 * root position of this call is stored there - `_save_prev_target_motion_state` (:741-750) and `self._target_root_pos = root_pos`
 * (:655) folded into the launch; prev_root_pos_update may be the same buffer as prev_root_pos.  only_mask (may be NULL): bool [n], the
 * envs whose entry is 0 are skipped (mask-driven reset: FK of the envs being reset only). */
typedef struct b200v2p_smpl {
  int32_t n, num_rest;
  float dt;
  int32_t pad_;
  const float *root_pos, *joint_rotmat, *rest; /* [n,3], [n,24,3,3], [num_rest,24,3] */
  const int32_t *parents, *smpl_2_mujoco;      /* [24] */
  const float *prev_root_pos, *prev_rb_rot;    /* NULL: zero velocities */
  float *root_rot, *dof_pos, *root_vel, *root_ang_vel, *dof_vel, *rb_pos, *rb_rot;
  float *prev_root_pos_update, *target_root_pos_out; /* NULL: not stored */
  const uint8_t* only_mask;                    /* NULL: every env */
} b200v2p_smpl_t;
int b200v2p_smpl_to_sim(const b200v2p_smpl_t* d, void* stream);

/* replaces the fix_head_orientation block of _set_target_motion_state (env/tasks/humanoid_smpl_im_mvae.py:605-634):
 * rb_pos/rb_rot [n,24,*] = FK of the uncorrected pose (MuJoCo order, head_body = 13); joint_rotmat [n,24,3,3] (SMPL order) is
 * corrected in place at SMPL joints Head (15) and Neck (12). */
typedef struct b200v2p_head {
  int32_t n, head_body;
  const float *rb_pos, *rb_rot, *ball_pos, *root_pos;
  float* joint_rotmat;
} b200v2p_head_t;
int b200v2p_fix_head(const b200v2p_head_t* d, void* stream);

/* replaces apply_external_force_to_ball (env/tasks/humanoid_smpl_im_mvae.py:711-739): drag + Magnus lift, bounce flag */
typedef struct b200v2p_aero {
  int32_t n, stride, substeps; /* stride: floats between consecutive envs' ball rows, >= 13 */
  float spin_scale;
  const float* ball_states;
  uint8_t *has_bounce, *has_bounce_now;
  float *bounce_pos, *force;
} b200v2p_aero_t;
int b200v2p_ball_aero(const b200v2p_aero_t* d, void* stream);

/* replaces _reset_balls + TennisBallGeneratorOffline.generate (:503-524, utils/tennis_ball.py:435-456): pool [P,307] */
typedef struct b200v2p_breset {
  int32_t n, stride;           /* stride: floats between consecutive envs' ball rows, >= 13 */
  const int64_t *env_ids, *pool_index;
  const float* pool;
  float *ball_states, *ball_pos, *ball_vel;
  uint8_t* has_bounce;
  float* bounce_pos;
  uint8_t* has_contact;
  float* traj;
} b200v2p_breset_t;
int b200v2p_ball_reset(const b200v2p_breset_t* d, void* stream);

/* replaces _update_state_from_sim (:799-860), substeps > 2 contact detector */
typedef struct b200v2p_state {
  int32_t n, bodies_per_env, ball_stride, root_stride, racket_body, wrist_body;
  float grip_normal[3];
  /* dual_mode 'different' (:839-842, :79-84): odd envs use the second player's grip / racket bodies when dual != 0 */
  int32_t dual, racket_body2, wrist_body2;
  float grip_normal2[3];
  const float* rigid_body_state; /* [n, bodies_per_env, 13] */
  const float* root_states;      /* humanoid root row per env, stride root_stride floats */
  const float* ball_states;      /* ball root row per env, stride ball_stride floats */
  uint8_t *has_contact, *has_contact_now;
  float *root_pos, *root_vel, *racket_pos, *racket_vel, *racket_normal, *ball_pos, *ball_vel, *ball_vspin;
  const uint8_t* only_mask;      /* NULL, or bool [n]: refresh the envs whose entry is set only (reset path) */
} b200v2p_state_t;
int b200v2p_update_state(const b200v2p_state_t* s, void* stream);

/* replaces PhysicsMVAEController.post_physics_step's device work (env/tasks/physics_mvae_controller.py:441-452):
 * _update_state (:271-314, incl. TennisBallOutEstimator.estimate utils/tennis_ball_out_estimator.py:164-205),
 * _compute_reward (:368-406, jit :493-602), _compute_observations (:316-360), _compute_reset (:408-436). */
typedef struct b200v2p_ctrl {
  int32_t n, bodies_per_env, ball_stride, racket_body, num_obs, obs_traj_len, use_target, reward_type, early_termination,
      max_episode_length, est_nx, est_ny;
  int32_t obs_only; /* 1: refresh obs_buf only (the _compute_observations call of _reset_envs :200-201), touch nothing else */
  int32_t dual;     /* 1: reset FSM of PhysicsMVAEControllerDual._compute_reset (env/tasks/physics_mvae_controller_dual.py:92-120):
                       envs (2k, 2k+1) are opponents, so n must be even; reset_buf is only ever SET, terminate_buf is not written.
                       num_obs must equal 225 + 3 * obs_traj_len (+ 2 with use_target): the NaN test sees exactly these columns */
  int32_t use_history; /* cfg use_history_ball_obs (:348-351): the task observation is the HISTORY of ball positions (ball_obs)
                          instead of the future trajectory window (ball_traj) */
  int32_t advance;     /* 1 (ignored with obs_only): first do the tail of physics_step and the head of post_physics_step (:364-366,
                          :441-444) - ball_traj <- roll(-1) with a zero last frame, tar_time += 1, progress_buf += 1 - then the rest */
  float scale_pos, scale_phase, scale_bounce_pos, scale_bounce_time, w_pos, w_ball_pos;
  float court_min[2], court_max[2];
  float est_params[15]; /* VEL_X, VEL_Y, VSPIN, TRAJ_X, TRAJ_Y ranges (lo, hi, step) */
  const float* rigid_body_state;
  const float* ball_states;
  const float *root_pos, *root_vel, *racket_pos, *racket_normal, *ball_pos;
  const uint8_t *has_contact, *has_contact_now, *has_bounce, *has_bounce_now;
  const float* bounce_pos;
  float* ball_traj; /* [n,100,3]; written only with advance = 1 */
  const float* target_bounce_pos;
  const float* phase;
  const int64_t *swing_type, *swing_type_cycle, *tar_action;
  int64_t* tar_time;            /* written only with advance = 1 */
  const int64_t* tar_time_total;
  int64_t* progress_buf;        /* written only with advance = 1 */
  const float *est_x, *est_y; /* estimator tables [rows, est_nx], [rows, est_ny, 2]; NULL = no estimator (dual mode) */
  uint8_t *bounce_in, *est_bounce_in, *reset_reaction, *reset_recovery;
  float *est_bounce_pos, *est_bounce_time, *est_max_height, *distance;
  float *obs_buf, *rew_buf, *sub_rewards; /* sub_rewards [n,2] */
  int64_t *reset_buf, *terminate_buf;
  float* ball_obs; /* [n, obs_traj_len, 3] _ball_obs (:65): rolled by one and appended with ball_pos at every observation (:345-346);
                      in obs_only mode only for the envs whose reset masks are set (the reference refreshes those ids only).
                      NULL = not kept (then use_history must be 0) */
  const uint8_t* touch_mask; /* NULL, or bool [n] with obs_only: the humanoids just reset.  Rows of envs that are neither in it nor flagged
                                reset_reaction / reset_recovery are still current and skipped; the task flags of the envs in it are cleared
                                at the end (tail of _reset_envs, :176-177) */
  /* test-time reset rule of MVAEControllerVis._compute_reset / _compute_stats (env/tasks/mvae_controller_vis.py:64-93), used when
   * eval = 1 (not with dual; ignored with obs_only) instead of the training FSM: terminate = reset = progress > eval_episode_length;
   * in_time = tar_time >= tar_time_total; reaction = (contact & tar_action == 0 & has_bounce & in_time) | (!contact & in_time);
   * recovery = tar_action == 1 & (contact | ball_y < root_y - 1 | |ball_vel_y| < 2); a reset sets reaction and clears recovery.  No
   * NaN / court / early termination, distance not advanced.  The envs in recovery then update the four AverageMeterUnSync meters
   * (utils/common.py:40-63) in place, meter m of env e at [m * n + e]: 0 hit_rate (contact), 1 fh_ratio (swing_type_cycle == 1),
   * 2 bounce_in_rate (est_bounce_in), 3 bounce_in_pos_error (|est_bounce_pos - target_bounce_pos|, envs with est_bounce_in only):
   * sum += v, count += 1, avg = sum / count, max = v > max ? v : max. */
  int32_t eval, eval_episode_length;
  const float* ball_vel;           /* [n,3]; eval only */
  float *meter_sum, *meter_avg, *meter_max; /* [4,n]; eval only */
  int64_t* meter_count;            /* [4,n]; eval only */
  /* the high-level policy's first-layer operand (V2PPlayer.get_action, players/v2p_player.py:113-131), written from the same values as
   * every observation row this launch writes, obs_only included (rows it skips are left alone): column k < num_obs of env e's row is
   * bf16(clamp((clamp(obs[e,k], -policy_clip_obs, policy_clip_obs) - mean[k]) * rstd[k], -clip, clip)), i.e. the wrapper's observation
   * clamp, then the normaliser (rl_games RunningMeanStd or RunningNorm with rstd precomputed, the clamp c).  policy_x NULL: not written.
   * policy_dual: env e's row is (e & 1) * n/2 + (e >> 1), so each player's rows are one block (n even), and player e & 1 uses row e & 1
   * of mean / rstd ([2, num_obs]) and clip = policy_clip[e & 1]; otherwise row e, mean / rstd [num_obs], policy_clip[0].
   * mean / rstd NULL: no normalisation (clamps still applied).  Columns [num_obs, policy_ld) are not written. */
  void* policy_x;                  /* bf16 [rows, policy_ld] */
  const float *policy_mean, *policy_rstd;
  int32_t policy_ld, policy_dual;
  float policy_clip_obs, policy_clip[2];
  int32_t pad_;
} b200v2p_ctrl_t;
int b200v2p_controller_post(const b200v2p_ctrl_t* c, void* stream);

/* replaces the action handling of PhysicsMVAEController.pre_physics_step (env/tasks/physics_mvae_controller.py:247-262) that precedes
 * the motion generator: mvae_actions = actions[:, :num_latent] * vae_action_scale, replaced by clamp(N(0,1), -5, 5) where
 * tar_action == 0 when random_walk_in_recovery; res_dof_actions = actions[:, num_latent : num_latent + num_res_dof] *
 * residual_dof_scale.  The normal deviates are counter-based (seed, *step_counter, element), *step_counter is advanced by the launch
 * (done_counter: one zero-initialised uint32 of scratch), so that a captured step replays with fresh numbers. */
typedef struct b200v2p_prestep {
  int32_t n, num_actions, num_latent, num_res_dof, random_walk_in_recovery;
  float vae_action_scale, residual_dof_scale;
  uint64_t seed;
  const float* actions;        /* [n, num_actions] */
  const int64_t* tar_action;   /* [n] */
  int64_t* step_counter;       /* [1] */
  uint32_t* done_counter;      /* [1] scratch, zero between launches */
  float* mvae_actions;         /* [n, num_latent] */
  float* res_dof_actions;      /* [n, num_res_dof] or NULL */
} b200v2p_prestep_t;
int b200v2p_pre_step(const b200v2p_prestep_t* p, void* stream);

/* the controller's own bookkeeping of a humanoid reset (env/tasks/physics_mvae_controller.py:176-181, 203-210) for the envs whose mask
 * is set: progress / reset / terminate / num_reset_reaction <- 0, distance <- 0, num_reset += 1 */
typedef struct b200v2p_creset {
  int32_t n, pad_;
  const uint8_t* mask;
  int64_t *progress_buf, *reset_buf, *terminate_buf, *num_reset_reaction;
  float* distance;
  int64_t* num_reset;
} b200v2p_creset_t;
int b200v2p_ctrl_reset(const b200v2p_creset_t* d, void* stream);

/* The resident kinematic target stream that stands in for the unreleased MVAE motion generator (SURVEY.md 8d, config 3): `frames`
 * frames of every field for all n envs are kept in HBM ([frames * n, ...], frame-major); env e reads frame (clock + advance +
 * offset[e]) % frames into the live buffers MVAEPlayer exposes (players/mvae_player.py: _joint_rotmat [n,24,3,3], _root_pos,
 * _racket_pos [n,3], _phase_pred [n], _swing_type, _swing_type_cycle [n] int64).  advance = 1: a step (the clock moves on), 0: re-read
 * after a reset changed offsets. */
typedef struct b200v2p_stream {
  int32_t n, frames, advance, pad_;
  int64_t* clock;              /* [1] */
  uint32_t* done_counter;      /* [1] scratch, zero between launches */
  int64_t* offset;             /* [n] */
  const uint8_t* reseed_mask;  /* NULL, or bool [n] (reset): the envs whose entry is set draw a new offset (counter-based: seed, clock, env)
                                  and re-read their frame; the others are left alone */
  uint64_t seed;
  const float* ring_rotmat;    float* rotmat;
  const float* ring_root_pos;  float* root_pos;
  const float* ring_racket_pos; float* racket_pos;
  const float* ring_phase;     float* phase;
  const int64_t* ring_swing_type; int64_t* swing_type;
  const int64_t* ring_swing_type_cycle; int64_t* swing_type_cycle;
} b200v2p_stream_t;
int b200v2p_stream_gather(const b200v2p_stream_t* s, void* stream);

/* replaces TennisBallInEstimator.estimate (utils/tennis_ball_in_estimator.py:22-81), the table lookup of
 * HumanoidSMPLIMMVAEDual._reset_balls (env/tasks/humanoid_smpl_im_mvae_dual.py:63-72): for query i the ball row
 * ball_states + contact_ids[i]*stride (the ball the opponent just hit) is snapped to the table grid; outputs the incoming
 * trajectory in the receiver's frame traj[n,50,3] and the snapped in / out ball states [n,13].  The caller scatters them
 * (states[ball_ids] = in, then states[contact_ids] = out).  table [rows,50,2]; params = HEIGHT, VEL_X, VEL_Y, VSPIN (lo,hi,step). */
typedef struct b200v2p_inest {
  int32_t n, stride;
  int64_t table_rows;
  double params[12];
  const int64_t* contact_ids;
  const float *ball_states, *table;
  float *traj, *states_in, *states_out;
} b200v2p_inest_t;
int b200v2p_ball_in_estimate(const b200v2p_inest_t* d, void* stream);

/* replaces the per-step task part of PhysicsMVAEController._reset_envs when no humanoid needs a reset
 * (env/tasks/physics_mvae_controller.py:173-201: _reset_balls for the reaction envs :503-524, _reset_recovery_tasks :242-245,
 * _reset_reaction_tasks :203-240), driven by the device-side masks instead of nonzero() id lists: no host sync.
 * Random draws come in as device tensors (torch RNG): pool_rand[n] in [0,P), side_rand[n] in [-1000,1000), frame_rand[n] in [-5,5),
 * target_seed: 3 floats (continuous mode) or n floats (discrete mode).
 * pool_cursor: NULL, or int64 [n] for the fixed test set (TennisBallGeneratorOffline with sample_random False, tennis_ball.py:444-447):
 * a reaction env takes pool row pool_cursor[e] and moves its cursor to (pool_cursor[e] + 1) % pool_size; the ball's side is not looked
 * at and pool_rand / side_rand are not read.  The cursor is only written here, so a graph replay advances it with no host work. */
typedef struct b200v2p_treset {
  int32_t n, pool_size, ball_stride, bodies_per_env, reaction_nframes, target_mode; /* 0 none, 1 continuous, 2 discrete */
  float target_min[3], target_max[3];
  const uint8_t *reset_reaction, *reset_recovery;
  const int64_t *pool_rand, *side_rand, *frame_rand;
  const float* target_seed;
  const float* pool;          /* [P,307] */
  float* ball_states;         /* first ball root row, stride ball_stride */
  float* rigid_body_state;    /* ball = last body row of each env */
  float *ball_pos, *ball_vel, *bounce_pos, *ball_traj, *est_bounce_pos, *est_bounce_time, *est_max_height, *target_bounce_pos;
  uint8_t *has_bounce, *has_contact, *bounce_in, *est_bounce_in;
  int64_t *tar_time, *tar_time_total, *tar_action, *num_reset_reaction, *swing_type_cycle;
  float* ball_obs;       /* use_history_ball_obs (:213-214): rows of the reaction envs <- the new ball position repeated; NULL = off */
  int32_t obs_traj_len, pad_;
  int64_t* pool_cursor;  /* appended field: a descriptor zeroed past obs_traj_len / pad_ keeps the random draw */
} b200v2p_treset_t;
int b200v2p_task_reset(const b200v2p_treset_t* r, void* stream);
/* sizeof(b200v2p_treset_t) of the library, so that a binding refuses a library built before pool_cursor */
int32_t b200v2p_task_reset_desc_size(void);

/* Per-row results of the fixed test set (MVAEControllerVis with cfg.env.b200_ball_stats).  No reference counterpart: the reference's
 * _compute_stats (env/tasks/mvae_controller_vis.py:80-93) keeps per-env meters only.  Every flagged env adds to the bucket of the pool
 * row r = (pool_cursor[e] + pool_size - 1) % pool_size, one behind its cursor: the cursor moves by one (mod pool_size) at each draw
 * only, so r is the row of the env's last draw.  One launch, in one of two forms (exactly one of reset_reaction / reset_recovery):
 *   draws   (reset_reaction, row_served), right after b200v2p_task_reset with pool_cursor: each env that just drew (reset_reaction set)
 *           adds 1 to row_served[r], the row it took;
 *   events  (reset_recovery and the fields after it), right after the eval post launch (b200v2p_controller_post with eval set),
 *           before the next task reset: each recovery event (the events at which the meters update) adds (1, has_contact,
 *           swing_type_cycle == 1, est_bounce_in, est_bounce_in ? q(|est_bounce_pos - target_bounce_pos|) : 0) to buckets[r], the
 *           distance in float32 as meter 3 takes it.  A recovery needs tar_action 1, which only a reaction reset (a draw) sets, so r
 *           is the row of the ball the env plays.
 * Lanes of a warp that share a row are folded with __match_any_sync, and each row's leader adds the warp's totals with integer
 * atomics, so the counts are the same bits on every run whatever the order.  q(v) = rint(v * 2^24): fixed point in units of 2^-24 m,
 * exact for v >= 0.5 m (a float there has no bits below 2^-24), off by at most 2^-25 m below; a bounce-in error lies inside the court
 * and target box (under 64 m = 2^30 units), so a row holds 2^33 events before the int64 can overflow.  The caller divides column 4 by
 * 2^24 to get metres.  pool_cursor must lie in [0, pool_size), as the task reset leaves it. */
#define B200V2P_BSTATS_COLS 5                 /* recoveries, hits, forehands, bounce_in, bounce-in error in 2^-24 m */
#define B200V2P_BSTATS_FIX_SCALE 16777216.0   /* 2^24 */
typedef struct b200v2p_bstats {
  int32_t n, pool_size;
  const int64_t* pool_cursor;        /* [n] */
  const uint8_t* reset_reaction;     /* [n]: draws form, else NULL */
  int64_t* row_served;               /* [pool_size]: draws form, else NULL */
  const uint8_t* reset_recovery;     /* [n]: events form, else NULL; the events form needs every field below */
  const uint8_t* has_contact;        /* [n] */
  const int64_t* swing_type_cycle;   /* [n] */
  const uint8_t* est_bounce_in;      /* [n] */
  const float* est_bounce_pos;       /* [n, 3] */
  const float* target_bounce_pos;    /* [n, 3] */
  int64_t* buckets;                  /* [pool_size, B200V2P_BSTATS_COLS] */
} b200v2p_bstats_t;
int b200v2p_eval_ball_stats(const b200v2p_bstats_t* d, void* stream);
/* sizeof(b200v2p_bstats_t) as the library was built; the binding refuses a library whose size differs from its own */
int32_t b200v2p_eval_ball_stats_desc_size(void);

/* Rally results of the dual test run (MVAEControllerVisDual with cfg.env.b200_rally_stats).  No reference counterpart: the reference's
 * MVAEControllerVisDual keeps no meters (env/tasks/mvae_controller_vis_dual.py:164-195 only sums _distance to choose what to render).
 * Launched right after each full dual post launch (b200v2p_controller_post with dual, advance, not obs_only), one thread per pair k of
 * the envs a = 2k (player 0) and b = 2k + 1 (player 1).  For player w on env i it takes the terms of the dual reset rule
 * (physics_mvae_controller_dual.py:92-120) as the post launch computes them (a copy of its lines, which keeps the post kernel's SASS):
 *   ta1, ta0 = tar_action[i] is 1 (to hit) / 0 (recovering); hc = has_contact[i]; hb = has_bounce[i]; bin = bounce_in[i] (as the post
 *   launch has just updated it); behind = ball_y < root_y - 1; twice = hb && ball_z < 0.05;
 *   rec[w] = ta1 && (hc || behind || twice)   the player meets a ball;
 *   out[w] = ta0 && hb && !bin                 a ball the player hit bounced out.
 * Counting, while the pair is open:
 *   faced[w] += rec[w]; a rec is a hit when hc (a forehand when also swing_type_cycle[i] == 1), else a miss, caused by double_bounce
 *   when twice, else behind.  The rally ends at the step where any player misses or has out, which is when the FSM sets reset_buf on the
 *   pair: rallies += 1, ends[w][cause] += 1 for each player that caused it (causes behind, double_bounce, out; both players can count at
 *   the same step), then this step's hits are added, the rally's hit total h (both players) goes to shots_hist[min(h, 64)] and
 *   shots_sum, progress_buf[a] to frames_sum, and the pair closes.
 *   A pair opens at the first post launch after its humanoids were reset (progress_buf[a] == 1), which zeroes its running hits
 *   pair_hits[k]; events count only while it is open, so a host loop that steps a finished pair without resetting it counts its
 *   ending once, and every reset path (masked, id list, the first reset) opens the rally without a hook of its own.  The serve is no
 *   hit: a served ball that bounces out ends the rally as the server's out with 0 shots, as the FSM does.
 * Invariants: faced[w] == hits[w] + misses[w]; hits[0] + hits[1] == shots_sum + the open pairs' running hits while pairs are reset
 * only after their rally ended (as the test loop resets them, from reset_buf); sum(shots_hist) == rallies.  Per-warp aggregation (ballots and popcounts, __match_any_sync on the histogram bucket) and integer atomics only, so
 * every run gives the same bits whatever the order.  n must be even; every pointer is required. */
#define B200V2P_RSTATS_HIST 65      /* shots per rally 0..63, then 64 = 64 or more */
#define B200V2P_RSTATS_CAUSES 3     /* behind, double_bounce, out */
typedef struct b200v2p_rstats {
  int32_t n, pad_;
  const int64_t* tar_action;         /* [n] */
  const uint8_t* has_contact;        /* [n] */
  const uint8_t* has_bounce;         /* [n] */
  const uint8_t* bounce_in;          /* [n] */
  const float* ball_pos;             /* [n, 3] */
  const float* root_pos;             /* [n, 3] */
  const int64_t* swing_type_cycle;   /* [n] */
  const int64_t* progress_buf;       /* [n] */
  uint8_t* pair_open;                /* [n/2] state: the pair is in a rally */
  int64_t* pair_hits;                /* [n/2, 2] state: the hits of each player in the pair's current (or last) rally */
  int64_t* totals;                   /* [3] rallies, shots_sum, frames_sum */
  int64_t* ends;                     /* [2, B200V2P_RSTATS_CAUSES] rallies ended by each player, by cause */
  int64_t* player;                   /* [2, 3] faced, hits, forehands */
  int64_t* shots_hist;               /* [B200V2P_RSTATS_HIST] */
} b200v2p_rstats_t;
int b200v2p_eval_rally_stats(const b200v2p_rstats_t* d, void* stream);
/* sizeof(b200v2p_rstats_t) as the library was built; the binding refuses a library whose size differs from its own */
int32_t b200v2p_eval_rally_stats_desc_size(void);

/* replaces HumanoidSMPLIMMVAE._reset_actors + _set_env_state + _reset_env_tensors for an id list
 * (env/tasks/humanoid_smpl_im_mvae.py:463-501, 562-581): the FK of the motion generator's pose (b200v2p_smpl_to_sim over all
 * envs, prev = NULL) is scattered into the simulation state of the listed envs; velocities zero. */
typedef struct b200v2p_areset {
  int32_t n, num_dof, bodies_per_env, root_stride, racket_body, racket_parent;
  float racket_offset[3];
  int32_t dual;             /* 1: odd envs use racket_offset2 / racket_parent2 (second player's asset) */
  float racket_offset2[3];
  int32_t racket_parent2, pad_;
  const int64_t* env_ids;
  const float *src_root_pos, *src_root_rot, *src_dof_pos, *src_rb_pos, *src_rb_rot; /* [N,...] FK results */
  float *root_states, *dof_state, *rigid_body_state;
  float *prev_target_root_pos, *prev_target_rb_rot, *root_pos, *root_vel, *pd_target_dof_pos, *target_root_pos;
  int64_t *progress_buf, *reset_buf, *terminate_buf;
  const uint8_t* mask;      /* optional [N]: row env_ids[i] is reset only when mask[env_ids[i]] != 0 (mask-driven form: env_ids =
                               0..N-1, n = N; no id list has to be built on the host, the launch can live in a CUDA graph) */
} b200v2p_areset_t;
int b200v2p_actor_reset(const b200v2p_areset_t* r, void* stream);

/* Rally recorder of the test-time tasks: the frame MVAEControllerVis.render_vis (env/tasks/mvae_controller_vis.py:140-146) and
 * MVAEControllerVisDual.render_vis (mvae_controller_vis_dual.py:156-162) append on every call, written for all n envs into
 * device-resident buffers [n, cap, ...] at row r: r = *row_counter (single; the launch advances the counter by one) or
 * r = progress_buf[e] (dual, row_counter NULL).  Rows at or past cap are not written (the reference's 1800-row buffer would raise).
 * rec_target_pos (single) and rec_tar_action (dual) may be NULL. */
typedef struct b200v2p_rec {
  int32_t n, cap;
  int64_t* row_counter;        /* [1] or NULL */
  uint32_t* done_counter;      /* [1] scratch, zero between launches (with row_counter) */
  const int64_t* progress_buf; /* [n] (dual) */
  const float *joint_rot, *root_pos, *ball_pos, *target_pos, *phase; /* [n,24,3], [n,3] x3, [n] */
  const int64_t *swing_type, *tar_action;                            /* [n] */
  float *rec_joint_rot, *rec_root_pos, *rec_ball_pos, *rec_target_pos, *rec_phase;
  int64_t *rec_swing_type, *rec_tar_action;
} b200v2p_rec_t;
int b200v2p_eval_record(const b200v2p_rec_t* r, void* stream);

/* Best-episode list of MVAEControllerVisDual.render_vis (mvae_controller_vis_dual.py:164-195), on the device.  Does nothing when
 * no reset_buf is set.  Otherwise the flagged pairs (2k, 2k+1; the dual reset FSM flags both players) are reduced to the first
 * argmax of distance[2k] + distance[2k+1]; it enters the list when the list is empty or it beats the list's last distance, in
 * front of the first entry it beats; the list keeps num_eg entries.  The list is order[i] = slot of the i-th best, with
 * best_distance / best_env (the pair's even env) / best_nframes (min(progress_buf, cap)) by slot, so an insertion moves slot
 * indices.  A second launch copies rows [0, nframes) of both envs of the chosen pair from the recording (b200v2p_eval_record's
 * rec_* buffers [n, cap, ...]) into best_* [num_eg, 2, cap, ...] at the chosen slot; copy_slot [1] holds that slot, or -1. */
typedef struct b200v2p_best {
  int32_t n, cap, num_eg, pad_;
  const int64_t *reset_buf, *progress_buf;
  const float* distance;
  int64_t* list_len;     /* [1] */
  int64_t* order;        /* [num_eg] */
  float* best_distance;  /* [num_eg] */
  int64_t *best_env, *best_nframes, *copy_slot;
  const float *rec_joint_rot, *rec_root_pos, *rec_ball_pos, *rec_phase;
  const int64_t *rec_swing_type, *rec_tar_action;
  float *best_joint_rot, *best_root_pos, *best_ball_pos, *best_phase;
  int64_t *best_swing_type, *best_tar_action;
} b200v2p_best_t;
int b200v2p_eval_best(const b200v2p_best_t* b, void* stream);

/* Two-hand backhand fix of an exported episode (cfg vid2player.fix_two_hand_backhand_post): HumanoidSMPLIMMVAE.optimize_two_hand_backhand
 * with single=True (env/tasks/humanoid_smpl_im_mvae.py:948-1031) and the frame selection and write-back of its callers
 * (mvae_controller_vis.py:181-191, mvae_controller_vis_dual.py:213-231), one CTA per problem, all problems in one launch.
 * A problem is one player of one episode: the frames with swing_type == 2 and 2 < phase < 5 are taken in frame order as one batch
 * (neighbouring batch rows are coupled by the smoothness term even across segments); the free arm's Wrist, Elbow, Shoulder and
 * Collar angle-axis get a delta that `iters` Adam steps (lr 0.005) fit so that the free hand reaches 2 hand - wrist of the racket
 * arm (L1 target + 0.2 L1 delta + 0.5 L1 smoothness).  out: the selected rows are all 24 joints round-tripped through
 * angle_axis_to_rotation_matrix / rotation_matrix_to_angle_axis with the fitted arm; every other row is joint_rot's, bit for bit.
 * The FK uses the problem's own rest joints for every frame (the reference reads envs 0..M-1's) and rb_pos is the 7th output of
 * _smpl_to_sim (the reference unpacks nine of eight values).  Float arrays are float or double as `precision` says. */
typedef struct b200v2p_bhprob {
  const void* joint_rot;       /* [T,24,3] axis-angle rows (SMPL joint order) */
  const void* phase;           /* [T] */
  const int64_t* swing_type;   /* [swing_type_len], swing_type_len >= T */
  const void* rest;            /* [24,3] rest joints of the player, SMPL order */
  void* out;                   /* [T,24,3]; may be joint_rot itself */
  int64_t T, swing_type_len;   /* the arrays may be NULL when T is 0 */
  int32_t righthand, pad_;     /* 1: the racket is in the right hand, the left arm is fitted */
} b200v2p_bhprob_t;

/* the scratch a launch needs: the problem table, then one int32 frame index and B200V2P_BHFIX_FRAME_WORDS scalars of the precision per
 * frame, each part 256-byte aligned; F = the sum over the problems of T rounded up to a multiple of 32 */
#define B200V2P_BHFIX_FRAME_WORDS 75
#define B200V2P_BHFIX_ALIGN(x) ((((int64_t)(x)) + 255) / 256 * 256)
#define B200V2P_BHFIX_SCRATCH_BYTES(P, F, S) (B200V2P_BHFIX_ALIGN((int64_t)(P) * (int64_t)sizeof(b200v2p_bhprob_t)) + B200V2P_BHFIX_ALIGN((int64_t)(F) * 4) + (int64_t)(F) * B200V2P_BHFIX_FRAME_WORDS * (S))

typedef struct b200v2p_bhfix {
  int32_t num_problems;
  int32_t iters;                      /* Adam steps: 500 in the reference */
  const b200v2p_bhprob_t* problems;   /* host array [num_problems], copied into the scratch on the stream (the one entry point here
                                         that copies from the host: from pageable memory the copy first waits for the stream) */
  void* scratch;                      /* device, 16-byte aligned, scratch_bytes >= B200V2P_BHFIX_SCRATCH_BYTES(num_problems, F, 4 or 8) */
  int64_t scratch_bytes;
  void* losses;                       /* optional [num_problems,3]: target, reg, smooth terms of the last evaluated step (NaN: none) */
  int32_t precision, pad_;            /* 0 float32, 1 float64 */
} b200v2p_bhfix_t;
int b200v2p_backhand_fix(const b200v2p_bhfix_t* f, void* stream);

#ifdef __cplusplus
}
#endif
#endif
