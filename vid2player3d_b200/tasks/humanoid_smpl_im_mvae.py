"""HumanoidSMPLIMMVAE mirror - the vid2player physics-player env
(vid2player/env/tasks/humanoid_smpl_im_mvae.py): humanoid (+ welded racket) + tennis ball per env, targets from a
kinematic motion generator (the MVAE player in the reference), 734-d imitation obs computed IN the env, and a `step`
that runs PD actuation + articulated dynamics + ball flight / bounce / racket impact as one fused CUDA launch.

Same attribute surface as the reference class for what the high-level controller reads
(physics_mvae_controller.py:271-301,336-357): `_root_pos _root_vel _racket_pos _racket_vel _racket_normal _ball_pos
_ball_vel _ball_vspin _ball_root_states _rigid_body_pos _rigid_body_rot _has_bounce _has_bounce_now _bounce_pos
_has_racket_ball_contact(_now)`, methods `reset(h_ids, b_ids) -> traj`, `post_mvae_step()`, `step(actions)`.
"""
import os
from types import SimpleNamespace

import numpy as np
import torch

from .. import abi, ball as ball_data, model_compiler, native, native_v2p
from ..torch_ops import quaternion_wxyz_to_angle_axis
from .base_task import BaseTask

SMPL_NAMES = ["Pelvis", "L_Hip", "R_Hip", "Torso", "L_Knee", "R_Knee", "Spine", "L_Ankle", "R_Ankle", "Chest", "L_Toe", "R_Toe",
              "Neck", "L_Thorax", "R_Thorax", "Head", "L_Shoulder", "R_Shoulder", "L_Elbow", "R_Elbow", "L_Wrist", "R_Wrist",
              "L_Hand", "R_Hand"]
SMPL_PARENTS = [-1, 0, 0, 0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 9, 9, 12, 13, 14, 16, 17, 18, 19, 20, 21]
TEST_MODES = ('random', 'single_cycle', 'multiple_cycle')


def resolve_ball_pool(cfg_v2p, is_train):
    """The incoming-ball pool of the single-player task and how it is drawn (:121-130): (pool [P, 307] float32 or None, sequential).

    Training, or test_mode 'random' (the default): `ball_pool`, else the file `ball_traj_file`, else a synthetic pool; rows are drawn
    at random.  At test time with test_mode 'single_cycle' or 'multiple_cycle' (set from env.ball_traj_file_test by
    PhysicsMVAEController): `ball_pool_test`, else the file `ball_traj_file_test`; every env walks the rows in order (sequential).  A
    missing test set is refused, since a random pool in its place would measure something else.  Dual mode builds no pool (None, False):
    its incoming balls come from the in-estimator table, so the test-set keys are ignored there, as in the reference."""
    if cfg_v2p.get('dual_mode', False):
        return None, False
    mode = cfg_v2p.get('test_mode', 'random')
    if mode not in TEST_MODES:
        raise ValueError(f"vid2player.test_mode {mode!r}: must be one of {', '.join(TEST_MODES)}")
    if is_train or mode == 'random':
        pool = cfg_v2p.get("ball_pool", None)
        if pool is None:
            path = cfg_v2p.get("ball_traj_file")
            pool = np.load(path) if path and os.path.exists(path) else ball_data.synthetic_pool(2048, seed=10, spin_scale=cfg_v2p.get("spin_scale", 1.0))
        return np.asarray(pool, np.float32), False
    pool = cfg_v2p.get("ball_pool_test", None)
    if pool is None:
        path = cfg_v2p.get("ball_traj_file_test")
        if not path:
            raise ValueError(f"vid2player.test_mode {mode!r} evaluates on a fixed test set, but neither ball_traj_file_test nor "
                             "ball_pool_test is given")
        if not os.path.exists(path):
            raise ValueError(f"vid2player.ball_traj_file_test {path!r} does not exist: the test set cannot be evaluated")
        pool = np.load(path)
    pool = np.asarray(pool, np.float32)
    if pool.ndim != 2 or pool.shape[0] < 1 or pool.shape[1] != 307:
        raise ValueError(f"the ball test set must be [P >= 1, 307] (launch pos, vel, vspin, 100 x 3 trajectory), got {list(pool.shape)}")
    return pool, True


class HumanoidSMPLIMMVAE(BaseTask):
    def __init__(self, cfg, sim_params, physics_engine, device_type, device_id, headless):
        self.cfg = cfg
        env = cfg["env"]
        self.cfg_v2p = env["vid2player"]
        self._is_train = env.get("is_train", True)
        self.sim_dt = float(getattr(sim_params, "dt", 1.0 / 60.0) if not isinstance(sim_params, dict) else sim_params.get("dt", 1.0 / 60.0))
        self.sim_substeps = int(cfg.get("sim", {}).get("substeps", 2))
        self.residual_force_scale = env.get("residual_force_scale", 0.0)
        self.residual_torque_scale = env.get("residual_torque_scale", self.residual_force_scale)
        self.kp_scale = env.get("kp_scale", 1.0)
        self.kd_scale = env.get("kd_scale", self.kp_scale)
        self.no_scale_action = env.get("no_scale_action", True)
        self.max_episode_length = env["episodeLength"]
        self._local_root_obs = env.get("localRootObs", True)
        self._root_height_obs = env.get("rootHeightObs", True)
        self._num_humanoid_bodies = 24
        self._racket_body_id = self._racket_body_id_true = 24
        self._racket_hand_body_id, self._racket_wrist_body_id, self._free_hand_body_id, self._head_body_id = 23, 22, 18, 13
        cfg["device_type"], cfg["device_id"], cfg["headless"] = device_type, device_id, True
        self.device = "cuda:" + str(device_id)

        # one asset, or one per player in dual_mode 'different' (:260-275: env 2k -> asset 0, env 2k+1 -> asset 1)
        files = env["asset"]["assetFileName"]
        files = list(files) if isinstance(files, (list, tuple)) else [files]
        # left-handed assets are brought into the right-handed body order (Racket last), see model_compiler.canonical_racket_last
        self._models = [model_compiler.canonical_racket_last(model_compiler.load_compiled(os.path.splitext(os.path.basename(f))[0]))
                        for f in files]
        self._model = self._models[0]
        self.body_names = [str(x) for x in self._model["body_names"]]
        self.num_bodies = len(self.body_names)          # 25 = humanoid + Racket (the ball is a separate actor)
        for m in self._models:
            if [str(x) for x in m["body_names"]] != self.body_names or self.num_bodies != 25 or self.body_names[-1] != "Racket":
                raise ValueError("vid2player assets must be the 24-body SMPL humanoid + a welded Racket")
        # per-player racket wrist (:68-84): R_Wrist 22, or L_Wrist 17 for a left-handed player; the racket's parent in the asset
        self._racket_parents = [int(m["parent"][24]) for m in self._models]
        rh = self.cfg_v2p.get('righthand', True)
        rh = list(rh) if isinstance(rh, (list, tuple)) else [rh] * len(self._models)
        for k, (r, par) in enumerate(zip(rh, self._racket_parents)):
            if par != (22 if r else 17):
                raise ValueError(f"asset {files[k]} has its racket on body {par}, which contradicts righthand={r}")
        self._racket_wrist_body_id = self._racket_parents[0] if len(set(self._racket_parents)) == 1 else list(self._racket_parents)
        if env["numEnvs"] % len(self._models):
            raise ValueError("numEnvs must be a multiple of the number of assets")
        self.num_dof = self._num_dof = len(self._model["kp"])
        self._num_actions = self.num_dof + (6 if self.residual_force_scale > 0 else 0)
        self._dof_offsets = list(range(0, self.num_dof + 1, 3))
        self._dof_obs_size = 23 * 6
        self._num_obs = 1 + 23 * 3 + 24 * 6 + 24 * 6 + self.num_dof + 11 + self.num_dof + 24 * 9 + 11   # 734 (:1046-1132)
        env["numObservations"], env["numActions"] = self._num_obs, self._num_actions
        self._build_mujoco_smpl_transform()
        super().__init__(cfg=cfg)
        self.dt = self.control_freq_inv * self.sim_dt
        self._terminate_buf = torch.ones(self.num_envs, device=self.device, dtype=torch.long)
        self._mvae_player = None
        self._controller = None
        self._obs_operand = None
        self._fast_targets = not self.cfg_v2p.get('fix_head_orientation') and not self.cfg_v2p.get('add_residual_root')
        self._setup_tensors()

    def _build_mujoco_smpl_transform(self):
        """:218-237"""
        mj = self.body_names[:24]
        self._smpl_2_mujoco = [SMPL_NAMES.index(q) for q in mj]
        self._mujoco_2_smpl = [mj.index(q) for q in SMPL_NAMES]

    def get_obs_size(self):
        return self._num_obs

    def get_action_size(self):
        return self._num_actions

    def create_sim(self):
        env = self.cfg["env"]
        v2p = self.cfg_v2p
        ball = dict(spin_scale=v2p.get("spin_scale", 1.0))
        rest = v2p.get("restitution", 0.9)
        plane_rest = env.get("plane", {}).get("restitution", 0.0)
        ball["ball_e_racket"] = rest                                            # racket & ball share `restitution` (:414,436)
        ball["ball_e_ground"] = 0.5 * (rest + plane_rest)                        # PhysX average combine
        ball["ball_mu_racket"] = 0.5 * (v2p.get("racket_friction", 0.8) + v2p.get("ball_friction", 0.2))
        ball["ball_mu_ground"] = 0.5 * (env.get("plane", {}).get("dynamicFriction", 1.0) + v2p.get("ball_friction", 0.2))
        # the ball also collides with the humanoid's bodies and the racket handle, as it does in the reference's PhysX scene (ball
        # collision filter 0, :436-442); include/b200env.h `ball_body_contact`, exact against the bodies' convex hulls
        # (b200env_set_hull_faces).  On by default (the body loop runs on the 8 lanes of the env's group);
        # vid2player.ball_body_contact: False switches it off
        if v2p.get("ball_body_contact", True):
            ball["ball_body_contact"] = 1
            ball["ball_e_body"] = 0.5 * rest                                      # body shapes: default material (restitution 0, friction 1)
            ball["ball_mu_body"] = 0.5 * (1.0 + v2p.get("ball_friction", 0.2))
        mk_cfg = lambda model: abi.make_cfg(  # noqa: E731
            model, sim_dt=self.sim_dt, substeps=self.sim_substeps, control_freq_inv=env.get("controlFrequencyInv", 2),
            pd_tar_lim=0.5 * np.pi, res_force_scale=self.residual_force_scale, res_torque_scale=self.residual_torque_scale,
            max_episode_length=self.max_episode_length, enable_early_termination=False, contact_bodies=tuple(env.get("contactBodies", ())),
            key_bodies=tuple(env.get("keyBodies", ())), friction_mu=env.get("plane", {}).get("dynamicFriction", 1.0),
            task_mode=1, pd_mode=1, ball=ball, **self.cfg.get("b200_physics", {}))
        self._cfg_struct = mk_cfg(self._model)
        # one handle per asset; handle k steps rows k, k+K, ... of the shared tensors (b200env_set_env_slice)
        self._envs, K = [], len(self._models)
        for k, m in enumerate(self._models):
            pd_scale = float(m["mass"].sum()) / env.get("default_humanoid_mass", 90.0)      # :381-389 kp, kd *= mass / 90
            ms, verts = abi.pack_model(m, pd_scale * self.kp_scale, pd_scale * self.kd_scale)
            if k == 0:
                self._model_struct, self._verts = ms, verts
            h = native.Env(ms, verts, mk_cfg(m), self.num_envs // K, self.device_id)      # racket head geometry is per asset
            if K > 1:
                h.set_env_slice(k, K)
            if ball.get("ball_body_contact"):
                # exact sphere / convex-hull query against the hull faces the model compiler stored (model_compiler.hull_faces)
                h.set_hull_faces(*abi.pack_faces(m, verts))
            self._envs.append(h)
        self._env = self._envs[0]

    def _setup_tensors(self):
        """:135-189 - Isaac layouts: 2 actors / env (humanoid, ball), 26 rigid bodies / env (25 + ball)"""
        N, dev, D = self.num_envs, self.device, self.num_dof
        f = lambda *s: torch.zeros(*s, device=dev, dtype=torch.float)  # noqa: E731
        b = lambda *s: torch.zeros(*s, device=dev, dtype=torch.bool)   # noqa: E731
        self._root_states = f(N * 2, 13)
        self._root_states[:, 6] = 1.0
        rs = self._root_states.view(N, 2, 13)
        self._humanoid_root_states, self._ball_root_states = rs[:, 0], rs[:, 1]
        self._humanoid_root_states[:, 2] = 0.89
        self._dof_state = f(N * D, 2)
        self._dof_pos, self._dof_vel = self._dof_state.view(N, D, 2)[..., 0], self._dof_state.view(N, D, 2)[..., 1]
        self._rigid_body_state = f(N * 26, 13)
        self._rigid_body_state[:, 6] = 1.0
        rbs = self._rigid_body_state.view(N, 26, 13)
        self._rigid_body_pos, self._rigid_body_rot = rbs[:, :25, 0:3], rbs[:, :25, 3:7]
        if not self._is_train:   # :113-116 test-time export of the simulated pose (SMPL joint order)
            self._joint_rot = torch.zeros((self.num_envs, 24, 3), device=self.device, dtype=torch.float32)
            # device index tensors: a Python-list index is a host-to-device copy, which a CUDA graph capture of the step refuses
            self._xyzw_to_wxyz_t = torch.tensor([3, 0, 1, 2], device=self.device)
            self._mujoco_2_smpl_t = torch.tensor(self._mujoco_2_smpl, device=self.device)
        self._rigid_body_vel, self._rigid_body_ang_vel = rbs[:, :25, 7:10], rbs[:, :25, 10:13]
        self._contact_force_tensor = f(N * 26, 3)
        self._contact_forces = self._contact_force_tensor.view(N, 26, 3)
        for k in ("_root_pos", "_root_vel", "_racket_pos", "_racket_vel", "_racket_normal", "_ball_pos", "_ball_vel", "_bounce_pos",
                  "_target_root_pos", "_prev_target_root_pos", "_target_root_vel", "_target_root_ang_vel"):
            setattr(self, k, f(N, 3))
        self._ball_vspin = f(N)
        for k in ("_has_bounce", "_has_bounce_now", "_has_racket_ball_contact", "_has_racket_ball_contact_now", "_racket_hit_now"):
            setattr(self, k, b(N))
        self._target_root_rot = f(N, 4)
        self._target_dof_pos, self._target_dof_vel = f(N, D), f(N, D)
        self._target_rb_pos, self._target_rb_rot = f(N, 24, 3), f(N, 24, 4)
        self._target_rb_rot[..., 3] = 1.0
        self._prev_target_dof_pos, self._prev_target_dof_vel = f(N, D), f(N, D)
        self._prev_target_rb_pos, self._prev_target_rb_rot = f(N, 24, 3), f(N, 24, 4)
        self._prev_target_rb_rot[..., 3] = 1.0
        self._pd_target_dof_pos = f(N, D)
        # DOF force sensors (:381, refreshed after every step :588; include/b200env.h b200_buffers_t::dof_force): written by the physics
        # launch of every step with cfg.env.dof_force_sensors (each handle of dual mode its own rows), else zeros
        self.dof_force_tensor = f(N, D)
        self.actions = f(N, self._num_actions)
        self._reset_ref_motion_bodies = f(N, 11)
        self._reset_ref_motion_bodies[:, 0] = 1          # gender male (:254-260)
        beta = self.cfg_v2p.get('smpl_beta')
        if beta is not None:
            if self.cfg_v2p.get('dual_mode') == 'different':
                self._reset_ref_motion_bodies[::2, 1:11] = torch.tensor(beta[0], device=dev, dtype=torch.float)
                self._reset_ref_motion_bodies[1::2, 1:11] = torch.tensor(beta[1], device=dev, dtype=torch.float)
            else:
                self._reset_ref_motion_bodies[:, 1:11] = torch.tensor(beta, device=dev, dtype=torch.float).view(-1)[:10]
        self._sub_rewards4, self._key_dummy = f(N, 4), f(N, max(1, self._cfg_struct.num_key), 3)
        self._zero_ids = torch.zeros(N, device=dev, dtype=torch.long)
        self._zero_t = f(N)
        t = dict(root_states=self._root_states, dof_state=self._dof_state, rigid_body_state=self._rigid_body_state,
                 contact_forces=self._contact_force_tensor, obs_buf=self.obs_buf, rew_buf=self.rew_buf, sub_rewards=self._sub_rewards4,
                 reset_buf=self.reset_buf, progress_buf=self.progress_buf, terminate_buf=self._terminate_buf, motion_ids=self._zero_ids,
                 ref_motion_times=self._zero_t, motion_bodies=self._reset_ref_motion_bodies, t_root_pos=self._target_root_pos,
                 t_root_rot=self._target_root_rot, t_dof_pos=self._target_dof_pos, t_root_vel=self._target_root_vel,
                 t_root_ang_vel=self._target_root_ang_vel, t_dof_vel=self._target_dof_vel, t_key_pos=self._key_dummy,
                 t_rb_pos=self._target_rb_pos, t_rb_rot=self._target_rb_rot, p_dof_pos=self._prev_target_dof_pos,
                 p_dof_vel=self._prev_target_dof_vel, p_rb_pos=self._prev_target_rb_pos, p_rb_rot=self._prev_target_rb_rot,
                 pd_targets=self._pd_target_dof_pos, actions_used=self.actions, has_bounce=self._has_bounce,
                 has_bounce_now=self._has_bounce_now, bounce_pos=self._bounce_pos, racket_hit_now=self._racket_hit_now)
        if self.cfg["env"].get("dof_force_sensors", False):
            t["dof_force"] = self.dof_force_tensor
        for h in self._envs:
            h.bind(t, actors_per_env=2, bodies_per_env=26, num_obs=self.num_obs)
        # SMPL kinematic constants for the FK targets (rest joints of the shipped skeletons, SMPL joint order), one per asset
        rests = []
        for m in self._models:
            pos = np.zeros((24, 3))
            for i in range(24):
                pos[i] = m["offset"][i] + (pos[m["parent"][i]] if m["parent"][i] >= 0 else 0)
            rests.append(np.stack([pos[self.body_names.index(n)] for n in SMPL_NAMES]).astype(np.float32))
        K = len(rests)
        self._rest_t = torch.tensor(np.stack(rests), device=dev).contiguous()            # [K,24,3]: env e uses shape e % K
        self._smpl = SimpleNamespace(joint_pos_bind=self._rest_t.repeat(N // K, 1, 1), parents=torch.tensor(SMPL_PARENTS, device=dev))
        self._parents_t = torch.tensor(SMPL_PARENTS, device=dev, dtype=torch.int32)
        self._s2m_t = torch.tensor(self._smpl_2_mujoco, device=dev, dtype=torch.int32)
        self._tmp = dict(root_rot=f(N, 4), dof_pos=f(N, D), root_vel=f(N, 3), root_ang_vel=f(N, 3), dof_vel=f(N, D), rb_pos=f(N, 24, 3),
                         rb_rot=f(N, 24, 4))
        # incoming-ball pool (TennisBallGeneratorOffline, utils/tennis_ball.py:422-456); dual mode has the in-estimator instead (:126-130)
        pool, sequential = resolve_ball_pool(self.cfg_v2p, self._is_train)
        if pool is not None:
            self._ball_pool = torch.tensor(pool, device=dev).contiguous()
        # the test set's per-env cursor (sample_idx, :433): only the ball resets move it, so it carries over humanoid resets
        self._ball_pool_cursor = torch.zeros(N, device=dev, dtype=torch.long) if sequential else None
        self._ball_row_served = None    # int64 [P] set by MVAEControllerVis (b200_ball_stats): every draw counts its row
        self._ball_traj_buf = f(N, 100, 3)
        self.extras["terminate"] = self._terminate_buf

    # ------------------------------------------------------------------ targets + obs (post_mvae_step :593-598)
    def _smpl_to_sim_into(self, root_pos, joint_rotmat, out, prev_root_pos=None, prev_rb_rot=None):
        native_v2p.smpl_to_sim(root_pos.contiguous(), joint_rotmat.contiguous(), self._rest_t, self._parents_t, self._s2m_t, self.dt, out,
                               prev_root_pos=prev_root_pos, prev_rb_rot=prev_rb_rot)

    def _set_target_motion_state(self):
        """:600-661 (fix_head_orientation off): targets = FK of the motion generator's pose, velocities by finite difference
        against the previous targets."""
        out = dict(root_rot=self._target_root_rot, dof_pos=self._target_dof_pos, root_vel=self._target_root_vel,
                   root_ang_vel=self._target_root_ang_vel, dof_vel=self._target_dof_vel, rb_pos=self._target_rb_pos, rb_rot=self._target_rb_rot)
        if self._fast_targets:
            # ONE launch: FK + finite differences against the previous targets (p_rb_rot is a buffer of its own, so no clone), and the
            # kernel itself stores this call's root position as the new "previous" / target root position
            native_v2p.smpl_to_sim(self._mvae_player._root_pos, self._mvae_player._joint_rotmat, self._rest_t, self._parents_t, self._s2m_t,
                                   self.dt, out, prev_root_pos=self._prev_target_root_pos, prev_rb_rot=self._prev_target_rb_rot,
                                   prev_root_pos_update=self._prev_target_root_pos, target_root_pos_out=self._target_root_pos)
            return
        root = self._mvae_player._root_pos.clone()
        if self.cfg_v2p.get('add_residual_root') and self._controller is not None:
            root += self._controller._res_root_actions
        if self.cfg_v2p.get('fix_head_orientation'):    # :605-634: FK of the raw pose, yaw Head/Neck towards the ball (in place)
            self._smpl_to_sim_into(root, self._mvae_player._joint_rotmat, self._tmp)
            native_v2p.fix_head(self._tmp["rb_pos"], self._tmp["rb_rot"], self._ball_pos, self._root_pos, self._mvae_player._joint_rotmat,
                                head_body=self._head_body_id)
        prev_rot = self._prev_target_rb_rot.clone()     # the kernel overwrites rb_rot rows it also reads as "previous"
        self._smpl_to_sim_into(root, self._mvae_player._joint_rotmat, out, self._prev_target_root_pos, prev_rot)
        self._target_root_pos.copy_(root)

    def _compute_observations(self):
        """:862-895 -> compute_humanoid_observations_imitation (:1046-1132) into obs_buf"""
        # (bf16 operand buffer, mean, rstd, clamp, dual, player 1's clamp) of a wgmma low-level policy, or None
        op = self._obs_operand
        self._env.obs_imitation_rows(self.num_envs, self._rigid_body_state, 26, self._dof_state, self._target_rb_pos, self._target_rb_rot,
                                     self._target_dof_pos, self._reset_ref_motion_bodies, self._local_root_obs, self._root_height_obs, self.obs_buf,
                                     obs_bf16=op[0] if op else None, mean=op[1] if op else None, rstd=op[2] if op else None,
                                     clamp=op[3] if op else 5.0, dual=op[4] if op else False, clamp1=op[5] if op else None)

    def post_mvae_step(self):
        self._set_target_motion_state()
        self._compute_observations()

    # ------------------------------------------------------------------ step (BaseTask.step :147-165 with :663-797)
    def step(self, actions):
        if not self._fast_targets:
            self._prev_target_root_pos.copy_(self._target_root_pos)      # _save_prev_target_motion_state (:741-750); else inside smpl_to_sim
        # pre_physics_step :689 zeroes _has_racket_ball_contact_now here; _update_state_from_sim below rewrites every row of it
        actions = actions.to(self.device, dtype=torch.float).contiguous()
        for h in self._envs:          # one launch per asset (dual: even envs, then odd envs)
            h.step(actions)
        self._update_state_from_sim()

    def _update_state_from_sim(self, only_mask=None):
        """:799-860; only_mask (bool [N], reset path): refresh the masked envs only"""
        t = dict(has_contact=self._has_racket_ball_contact, has_contact_now=self._has_racket_ball_contact_now, root_pos=self._root_pos,
                 root_vel=self._root_vel, racket_pos=self._racket_pos, racket_vel=self._racket_vel, racket_normal=self._racket_normal,
                 ball_pos=self._ball_pos, ball_vel=self._ball_vel, ball_vspin=self._ball_vspin)
        if self.sim_substeps <= 2:
            # contact-force sensor path (:771-779): the step kernel reports the exact racket impact
            now = self._racket_hit_now & ~self._has_racket_ball_contact
            self._has_racket_ball_contact |= now
            keep = self._has_racket_ball_contact.clone()
            native_v2p.update_state(self.num_envs, 26, self._rigid_body_state, self._root_states, 26, self._root_states[1:], 26, t,
                                    grip=self._grip(), wrist_body=self._racket_wrist_body_id)
            self._has_racket_ball_contact.copy_(keep)
            self._has_racket_ball_contact_now.copy_(now)
        else:
            native_v2p.update_state(self.num_envs, 26, self._rigid_body_state, self._root_states, 26, self._root_states[1:], 26, t,
                                    grip=self._grip(), wrist_body=self._racket_wrist_body_id, only_mask=only_mask)
        if not self._is_train:
            # :814-820 test-time export of the simulated pose as SMPL joint rotations (root angle-axis | dof_pos, SMPL joint order)
            root_rot = quaternion_wxyz_to_angle_axis(self._rigid_body_rot[:, 0][..., self._xyzw_to_wxyz_t])
            self._joint_rot[:] = torch.cat((root_rot.reshape(self.num_envs, 1, 3), self._dof_pos.reshape(self.num_envs, -1, 3)),
                                           dim=1)[:, self._mujoco_2_smpl_t]

    def _grip(self):
        g = self.cfg_v2p.get('grip', 'eastern')            # a pair in dual_mode 'different' (:839-842)
        return list(g) if isinstance(g, (list, tuple)) else g

    # ------------------------------------------------------------------ reset (:447-524, 562-581)
    def reset(self, reset_humanoid_env_ids, reset_ball_env_ids):
        traj = None
        if len(reset_humanoid_env_ids) > 0:
            self._reset_actors(reset_humanoid_env_ids)
        if len(reset_ball_env_ids) > 0:
            traj = self._reset_balls(reset_ball_env_ids)
        return traj

    def _reset_actors(self, env_ids):
        """:463-501 + :562-581: sim state <- FK of the motion generator's initial pose (zero velocities); 2 launches"""
        self._smpl_to_sim_into(self._mvae_player._root_pos.contiguous(), self._mvae_player._joint_rotmat, self._tmp)
        cfg = dict(n=len(env_ids), num_dof=self.num_dof, bodies_per_env=26, root_stride=26, racket_body=24,
                   racket_parent=self._racket_parents[0], racket_offset=self._model["offset"][24],
                   racket_offset2=self._models[1]["offset"][24] if len(self._models) == 2 else None,
                   racket_parent2=self._racket_parents[-1])
        native_v2p.actor_reset(cfg, dict(
            env_ids=env_ids.contiguous(), src_root_pos=self._mvae_player._root_pos.contiguous(), src_root_rot=self._tmp["root_rot"],
            src_dof_pos=self._tmp["dof_pos"], src_rb_pos=self._tmp["rb_pos"], src_rb_rot=self._tmp["rb_rot"], root_states=self._root_states,
            dof_state=self._dof_state, rigid_body_state=self._rigid_body_state, prev_target_root_pos=self._prev_target_root_pos,
            prev_target_rb_rot=self._prev_target_rb_rot, root_pos=self._root_pos, root_vel=self._root_vel,
            pd_target_dof_pos=self._pd_target_dof_pos, target_root_pos=self._target_root_pos, progress_buf=self.progress_buf,
            reset_buf=self.reset_buf, terminate_buf=self._terminate_buf))

    def _reset_actors_masked(self, mask):
        """_reset_actors for the envs whose mask is set: same two launches over all rows, no id list (CUDA-graph safe)"""
        if not hasattr(self, "_all_ids"):
            self._all_ids = torch.arange(self.num_envs, device=self.device, dtype=torch.long)
        native_v2p.smpl_to_sim(self._mvae_player._root_pos.contiguous(), self._mvae_player._joint_rotmat.contiguous(), self._rest_t, self._parents_t,
                               self._s2m_t, self.dt, self._tmp, only_mask=mask)
        cfg = dict(n=self.num_envs, num_dof=self.num_dof, bodies_per_env=26, root_stride=26, racket_body=24,
                   racket_parent=self._racket_parents[0], racket_offset=self._model["offset"][24],
                   racket_offset2=self._models[1]["offset"][24] if len(self._models) == 2 else None,
                   racket_parent2=self._racket_parents[-1])
        native_v2p.actor_reset(cfg, dict(
            env_ids=self._all_ids, mask=mask, src_root_pos=self._mvae_player._root_pos.contiguous(), src_root_rot=self._tmp["root_rot"],
            src_dof_pos=self._tmp["dof_pos"], src_rb_pos=self._tmp["rb_pos"], src_rb_rot=self._tmp["rb_rot"], root_states=self._root_states,
            dof_state=self._dof_state, rigid_body_state=self._rigid_body_state, prev_target_root_pos=self._prev_target_root_pos,
            prev_target_rb_rot=self._prev_target_rb_rot, root_pos=self._root_pos, root_vel=self._root_vel,
            pd_target_dof_pos=self._pd_target_dof_pos, target_root_pos=self._target_root_pos, progress_buf=self.progress_buf,
            reset_buf=self.reset_buf, terminate_buf=self._terminate_buf))

    def _reset_balls(self, env_ids):
        """:503-524 with TennisBallGeneratorOffline.generate (tennis_ball.py:435-456): the random branch (:436-444), or on a test set
        the env's next row in order (:444-447)"""
        P = self._ball_pool.shape[0]
        if self._ball_pool_cursor is not None:
            idx = self._ball_pool_cursor[env_ids]
            self._ball_pool_cursor[env_ids] = (idx + 1) % P
            if self._ball_row_served is not None:
                self._ball_row_served.index_add_(0, idx, torch.ones_like(idx))
        else:
            idx = torch.randint(0, P, (len(env_ids),), device=self.device)
            other = self._ball_pos[env_ids, 1] > 0
            if other.any():
                j = ((self._ball_pos[env_ids, 0] + 4) / 8 * P).long() + torch.randint(-1000, 1000, (len(env_ids),), device=self.device)
                idx = torch.where(other, torch.clamp(j, 0, P - 1), idx)
        native_v2p.ball_reset(env_ids.contiguous(), idx.contiguous(), self._ball_pool, self._root_states[1:], self._ball_pos, self._ball_vel,
                              self._has_bounce, self._bounce_pos, self._has_racket_ball_contact, self._ball_traj_buf, stride=26)
        rbs = self._rigid_body_state.view(self.num_envs, 26, 13)
        rbs[env_ids, 25, 0:3] = self._ball_root_states[env_ids, 0:3]
        rbs[env_ids, 25, 7:13] = self._ball_root_states[env_ids, 7:13]
        return self._ball_traj_buf[env_ids]

    def render_vis(self, init=False):
        return


class HumanoidSMPLIMMVAEDual(HumanoidSMPLIMMVAE):
    """vid2player/env/tasks/humanoid_smpl_im_mvae_dual.py: envs (2k, 2k+1) are the two players of one rally, each in its own
    court frame; a ball hit in one env re-enters the partner env mirrored, snapped to the incoming-ball table."""

    def __init__(self, cfg, sim_params, physics_engine, device_type, device_id, headless):
        super().__init__(cfg=cfg, sim_params=sim_params, physics_engine=physics_engine, device_type=device_type, device_id=device_id,
                         headless=headless)
        if self.num_envs % 2:
            raise ValueError("dual mode needs an even number of envs (opponents are envs 2k and 2k+1)")
        tab = self.cfg_v2p.get('ball_in_table', None)          # (table [rows,50,2], params [4,3]); utils/tennis_ball_in_estimator.py
        if tab is None:
            path = self.cfg_v2p.get('ball_traj_file')
            if path and os.path.exists(path):
                tab = (np.load(path), np.array([ball_data.IN_PARAMS[k] for k in ("HEIGHT", "VEL_X", "VEL_Y", "VSPIN")], np.float64))
            else:
                tab = ball_data.synthetic_in_table(spin_scale=self.cfg_v2p.get('spin_scale', 1.0))
        self._in_table = torch.tensor(np.asarray(tab[0], np.float32), device=self.device).contiguous()
        self._in_params = np.asarray(tab[1], np.float64)

    def reset(self, reset_actor_reaction_env_ids, reset_ball_env_ids):
        return self._reset_envs(reset_actor_reaction_env_ids, reset_ball_env_ids)

    def _reset_envs(self, reset_actor_reaction_env_ids, reset_ball_env_ids):
        """:34-50"""
        from ..torch_ops import get_opponent_env_ids
        reset_actor_recovery_env_ids = get_opponent_env_ids(reset_actor_reaction_env_ids)
        reset_actor_env_ids = torch.cat([reset_actor_reaction_env_ids, reset_actor_recovery_env_ids])
        traj = None
        if len(reset_actor_env_ids) > 0:
            self._reset_actors(reset_actor_env_ids)
        if len(reset_ball_env_ids) > 0:
            traj = self._reset_balls(reset_actor_recovery_env_ids, reset_ball_env_ids)
        return traj

    def _reset_balls_masked(self, serve_mask, recv_mask, opp):
        """_reset_balls (:52-80) with masks instead of id lists (CUDA-graph safe): `serve_mask` = the recovery actors (servers),
        `recv_mask` = the envs that receive a new incoming ball, `opp` = arange(N) ^ 1.  Same order of effects as the id-list form."""
        bs, dev, N = self._ball_root_states, self.device, self.num_envs
        m = serve_mask[:, None]
        bs[:, 0:3] = torch.where(m, self._mvae_player._racket_pos, bs[:, 0:3])
        if not hasattr(self, "_serve_spin"):
            self._serve_spin = torch.tensor([-40.0, 0.0, 0.0], device=dev)    # created outside any graph capture (first, eager call)
        bs[:, 10:13] = torch.where(m, self._serve_spin, bs[:, 10:13])
        v = torch.stack([torch.rand(N, device=dev) * 4 + -2, torch.rand(N, device=dev) * 4 + 28, torch.rand(N, device=dev) * 3 + 5], -1)
        bs[:, 7:10] = torch.where(m, v, bs[:, 7:10])
        if not hasattr(self, "_in_buf"):
            self._in_buf = (torch.empty(N, 50, 3, device=dev), torch.empty(N, 13, device=dev), torch.empty(N, 13, device=dev))
        traj, s_in, s_out = self._in_buf
        # every env as a receiver of the ball of its opponent; only the rows of recv_mask are used
        native_v2p.ball_in_estimate(opp, self._root_states[1:], 26, self._in_table, self._in_params, traj, s_in, s_out)
        r = recv_mask[:, None]
        hit = recv_mask[opp][:, None]                      # envs whose ball was just handed over (contact_env_ids)
        new = torch.where(r, s_in, bs)
        new = torch.where(hit, s_out[opp], new)            # the hitter's own ball, snapped to the same grid point (written second)
        bs.copy_(new)
        self._has_bounce.masked_fill_(recv_mask, False)
        self._bounce_pos.masked_fill_(r, 0.0)
        self._has_racket_ball_contact.masked_fill_(recv_mask, False)
        self._ball_pos.copy_(torch.where(r, bs[:, 0:3], self._ball_pos))
        self._ball_vel.copy_(torch.where(r, bs[:, 7:10], self._ball_vel))
        both = r | hit
        rbs = self._rigid_body_state.view(N, 26, 13)
        rbs[:, 25, 0:3] = torch.where(both, bs[:, 0:3], rbs[:, 25, 0:3])
        rbs[:, 25, 7:13] = torch.where(both, bs[:, 7:13], rbs[:, 25, 7:13])
        return traj

    def _reset_balls(self, reset_actor_recovery_env_ids, reset_ball_env_ids):
        """:52-80: serve = the ball at the server's racket with a random velocity; then every env in `reset_ball_env_ids` receives
        the ball its opponent just hit (b200v2p_ball_in_estimate), and the opponent's own ball is snapped to the same grid point."""
        from ..torch_ops import get_opponent_env_ids
        bs, dev = self._ball_root_states, self.device
        if len(reset_actor_recovery_env_ids) > 0:
            ids, n = reset_actor_recovery_env_ids, len(reset_actor_recovery_env_ids)
            bs[ids, :3] = self._mvae_player._racket_pos[ids]
            bs[ids, 10:13] = torch.tensor([-40.0, 0.0, 0.0], device=dev)
            bs[ids, 7] = torch.rand(n, device=dev) * 4 + -2
            bs[ids, 8] = torch.rand(n, device=dev) * 4 + 28
            bs[ids, 9] = torch.rand(n, device=dev) * 3 + 5
        contact_env_ids = get_opponent_env_ids(reset_ball_env_ids)
        n = len(reset_ball_env_ids)
        traj = torch.empty(n, 50, 3, device=dev)
        s_in, s_out = torch.empty(n, 13, device=dev), torch.empty(n, 13, device=dev)
        native_v2p.ball_in_estimate(contact_env_ids.contiguous(), self._root_states[1:], 26, self._in_table, self._in_params, traj, s_in, s_out)
        bs[reset_ball_env_ids] = s_in
        bs[contact_env_ids] = s_out
        self._has_bounce[reset_ball_env_ids] = False
        self._bounce_pos[reset_ball_env_ids] = 0
        self._has_racket_ball_contact[reset_ball_env_ids] = False
        self._ball_pos[reset_ball_env_ids] = bs[reset_ball_env_ids, 0:3]
        self._ball_vel[reset_ball_env_ids] = bs[reset_ball_env_ids, 7:10]
        # the simulator-side copy of the ball rows (_reset_env_tensors :562-572 pushes the root states of both ball actors)
        both = torch.cat([contact_env_ids, reset_ball_env_ids])
        rbs = self._rigid_body_state.view(self.num_envs, 26, 13)
        rbs[both, 25, 0:3] = bs[both, 0:3]
        rbs[both, 25, 7:13] = bs[both, 7:13]
        return traj
