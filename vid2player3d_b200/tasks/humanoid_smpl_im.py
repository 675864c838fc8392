"""HumanoidSMPLIM mirror - the low-level imitation env of the reference
(embodied_pose/env/tasks/humanoid_smpl_im.py + humanoid_smpl.py), same constructor, attributes
and semantics, with the whole `step` running as ONE fused CUDA launch (csrc/b200env.cu) and
`reset` as one more.

Tensor layouts are the Isaac Gym ones the reference wraps in `_setup_tensors`
(humanoid_smpl.py:66-113), so `_rigid_body_pos`, `_dof_pos`, `_humanoid_root_states`, ... are the
same views a reference user expects, and the kernels write straight into them.
"""
import os

import numpy as np
import torch

from .. import abi, model_compiler, native
from ..motion_lib import FlatMotionLib
from .base_task import BaseTask


def _sim_param(sim_params, name, default):
    if sim_params is None:
        return default
    if isinstance(sim_params, dict):
        return sim_params.get(name, default)
    return getattr(sim_params, name, default)


class HumanoidSMPLIM(BaseTask):
    def __init__(self, cfg, sim_params, physics_engine, device_type, device_id, headless):
        self.cfg = cfg
        self.args = cfg.get('args', None)
        env = cfg["env"]
        self.sim_params = sim_params
        self.physics_engine = physics_engine
        self.sim_dt = float(_sim_param(sim_params, "dt", 1.0 / 60.0))
        self.sim_substeps = int(_sim_param(sim_params, "substeps", cfg.get("sim", {}).get("substeps", 2)))

        self.has_shape_obs = env.get("has_shape_obs", False)
        self.residual_force_scale = env.get("residual_force_scale", 0.0)
        self.residual_torque_scale = env.get("residual_torque_scale", self.residual_force_scale)
        self.kp_scale = env.get("kp_scale", 1.0)
        self.kd_scale = env.get("kd_scale", self.kp_scale)
        self.context_length = env.get('context_length', 32)
        self.context_padding = env.get('context_padding', 8)
        self.truncate_time = env.get('truncate_time', True)
        self.pd_tar_lim = env.get('pd_tar_lim', 0.5) * np.pi
        control_freq_inv = env["controlFrequencyInv"]
        self._motion_sync_dt = control_freq_inv * self.sim_dt
        if self.args is not None and getattr(self.args, "test", False):
            env["stateInit"] = 'Start'
        self._state_init = env.get("stateInit", "Hybrid")
        self._hybrid_init_prob = env.get("hybridInitProb", 1.0)
        self._pd_control = env.get("pdControl", True)
        if not self._pd_control:
            raise NotImplementedError("torque control (pdControl: False) is not on the hot path")
        self.max_episode_length = env["episodeLength"]
        self._local_root_obs = env.get("localRootObs", True)
        self._root_height_obs = env.get("rootHeightObs", True)
        self._enable_early_termination = env["enableEarlyTermination"]
        self.ground_tolerance = env.get('ground_tolerance', 0.0)
        self.model = None
        self._sub_rewards_names = 'dof_reward,vel_reward,body_pos_reward,body_rot_reward'

        cfg["device_type"], cfg["device_id"], cfg["headless"] = device_type, device_id, headless
        self.device = "cuda:" + str(device_id)
        self._load_motion(env['motion_file'] if 'motion_file' in env else env['motion_lib'])
        self._load_asset()
        self._setup_character_props(env["keyBodies"])
        super().__init__(cfg=cfg)
        self.dt = self.control_freq_inv * self.sim_dt

        body_weights = env.get('body_pos_weights', dict())
        self.body_pos_weights = torch.ones(self.num_bodies, device=self.device)
        for val, bodies in body_weights.items():
            for body in bodies:
                self.body_pos_weights[self.body_names.index(body)] = val
        self._terminate_buf = torch.ones(self.num_envs, device=self.device, dtype=torch.long)
        self._sub_rewards = torch.zeros(self.num_envs, 4, device=self.device)
        self._bind()

    # ------------------------------------------------------------------ construction
    def _load_motion(self, motion_file):
        """humanoid_smpl_im.py:420-440.  Accepts a FlatMotionLib, a path - `.b200ml` flat file, `.npz`, a reference
        `torch.save(motion_lib)` `.pth`, or a directory of them sliced by cfg.env.motion_file_range and merged - or a loaded
        reference MotionLib object."""
        if isinstance(motion_file, FlatMotionLib):
            flat = motion_file
        elif isinstance(motion_file, (str, os.PathLike)):
            flat = FlatMotionLib.load_any(motion_file, self.cfg["env"].get("motion_file_range", None))
        elif all(hasattr(motion_file, k) for k in ("gts", "grs", "lrs", "_motion_lengths")):
            flat = FlatMotionLib.from_reference(motion_file)
        else:
            raise TypeError(f"motion_lib / motion_file: expected a FlatMotionLib, a path or a reference MotionLib, got {type(motion_file)}")
        self._motion_lib = flat
        dev = self.device
        self._ml_t = {k: torch.from_numpy(getattr(flat, k)).to(dev).contiguous() for k in FlatMotionLib.FIELDS}

    def _load_asset(self):
        name = os.path.splitext(os.path.basename(self.cfg["env"]["asset"]["assetFileName"]))[0]
        self._model = model_compiler.load_compiled(name)
        self.body_names = [str(x) for x in self._model["body_names"]]
        self.dof_names = [str(x) for x in self._model["dof_names"]]
        self.num_bodies = len(self.body_names)
        self.num_dof = len(self.dof_names)
        self.humanoid_mass = float(self._model["mass"].sum())
        self.humanoid_masses = np.full(self.cfg["env"]["numEnvs"], self.humanoid_mass)

    def _setup_character_props(self, key_bodies):
        """humanoid_smpl_im.py:159-215"""
        self._dof_body_ids = [int(x) for x in self._model["dof_body_ids"]]
        self._dof_offsets = list(range(0, self.num_dof + 1, 3))
        self._dof_obs_size = len(self._dof_body_ids) * 6
        self._num_actions = self._num_dof = self.num_dof
        if self.residual_force_scale > 0:
            self._num_actions += 6
        nb = self._num_lib_bodies = self._motion_lib.gts.shape[1]
        shape_dim = self._motion_lib.motion_bodies.shape[-1]
        shape_dict = {'body_pos': (nb, 3), 'body_pos_gt': (nb, 3), 'body_rot': (nb, 4), 'dof_pos': (self._num_dof,),
                      'dof_pos_gt': (self._num_dof,), 'dof_vel': (self._num_dof,), 'body_vel': (nb, 3),
                      'body_ang_vel': (nb, 3), 'motion_bodies': (shape_dim,), 'joint_conf': (nb,)}
        self.obs_names = ['body_pos', 'body_rot', 'dof_pos', 'dof_vel', 'body_vel', 'body_ang_vel', 'motion_bodies']
        self.obs_shapes = [shape_dict[x] for x in self.obs_names]
        self.obs_dims = [int(np.prod(x)) for x in self.obs_shapes]
        self.context_names = ['body_pos', 'body_rot', 'dof_pos', 'body_pos_gt', 'dof_pos_gt']
        self._transform_specs = self.cfg['env'].get('transform_specs', None)
        if 'transform_specs' in self.cfg['env']:             # :202-204
            self.context_names.append('joint_conf')
        self.context_shapes = [shape_dict[x] for x in self.context_names]
        self.context_dims = [int(np.prod(x)) for x in self.context_shapes]
        self.is_env_dim_setup = False
        self._num_obs = sum(self.obs_dims)
        self.cfg["env"]["numObservations"] = self.get_obs_size()
        self.cfg["env"]["numActions"] = self.get_action_size()
        self._key_body_names = list(key_bodies)

    def get_obs_size(self):
        return self._num_obs

    def get_action_size(self):
        return self._num_actions

    def _pack(self, model):
        """pack_model with the PD gains scaled by the model's own mass (:376-383)"""
        pd_scale = float(model["mass"].sum()) / self.cfg["env"].get('default_humanoid_mass', 90.0)
        return abi.pack_model(model, pd_scale * self.kp_scale, pd_scale * self.kd_scale)

    def _motion_asset_models(self):
        """cfg.env.motion_assets: one entry per motion of the library - an asset file name (resolved like asset.assetFileName) or a
        compiled model dict - as (compiled models of the distinct assets, asset index of every motion).  Identical compiled assets
        (same packed constants and vertices) are one asset."""
        entries = self.cfg["env"]["motion_assets"]
        if len(entries) != self._motion_lib.num_motions():
            raise ValueError(f"motion_assets has {len(entries)} entries for {self._motion_lib.num_motions()} motions")
        models, keys, of_motion = [], {}, []
        for entry in entries:
            if isinstance(entry, (str, os.PathLike)):
                entry = model_compiler.load_compiled(os.path.splitext(os.path.basename(str(entry)))[0])
            ms, verts = self._pack(entry)
            key = bytes(ms) + verts.tobytes()
            if key not in keys:
                keys[key] = len(models)
                models.append(entry)
            of_motion.append(keys[key])
        return models, np.asarray(of_motion, np.int64)

    def create_sim(self):
        """Stub of BaseTask.create_sim/_create_envs (humanoid_smpl_im.py:231-351): all N envs are instances of one compiled model -
        O(1) host work, no per-env Python loop.  With cfg.env.motion_assets, env e is simulated with the asset of its motion
        _reset_ref_motion_ids[e] (one handle of several assets: the motion ids are sampled here, before the handle exists)."""
        env = self.cfg["env"]
        self._model_struct, self._verts = self._pack(self._model)
        structs = None
        if "motion_assets" in env:
            self._reset_ref_motion_ids = self._sample_motion_ids()
            models, of_motion = self._motion_asset_models()
            self._env_asset = of_motion[self._reset_ref_motion_ids.cpu().numpy()]
            self._asset_models = models
            packed = [self._pack(m) for m in models]
            structs, verts = [p[0] for p in packed], [p[1] for p in packed]
            self.humanoid_masses = np.array([float(m["mass"].sum()) for m in models])[self._env_asset]     # :370-371
            self._model_struct, self._verts = structs[self._env_asset[-1]], verts[self._env_asset[-1]]  # the last env's, as the loop leaves them
            lim = models[self._env_asset[0]]["limits"]                                                    # env 0's (:340-349)
        else:
            lim = self._model["limits"]
        self.stiffness = torch.tensor(list(self._model_struct.kp)[:self.num_dof], device=self.device)
        self.damping = torch.tensor(list(self._model_struct.kd)[:self.num_dof], device=self.device)
        self.dof_limits_lower = torch.tensor(np.minimum(lim[:, 0], lim[:, 1]), device=self.device, dtype=torch.float)
        self.dof_limits_upper = torch.tensor(np.maximum(lim[:, 0], lim[:, 1]), device=self.device, dtype=torch.float)
        physx = self.cfg.get("b200_physics", {})
        self._cfg_struct = abi.make_cfg(
            self._model, sim_dt=self.sim_dt, substeps=self.sim_substeps, control_freq_inv=env["controlFrequencyInv"],
            pd_tar_lim=self.pd_tar_lim, res_force_scale=self.residual_force_scale,
            res_torque_scale=self.residual_torque_scale, max_episode_length=self.max_episode_length,
            enable_early_termination=self._enable_early_termination,
            termination_body_height=env.get("terminationBodyHeight", env.get("terminationHeight", -0.5)),
            termination_head_height=env.get("terminationHeadHeight", 0.3), contact_bodies=tuple(env["contactBodies"]),
            key_bodies=tuple(env["keyBodies"]), body_pos_weights=env.get('body_pos_weights', None),
            reward_specs=env.get('reward_specs', None), shape_dim=self._motion_lib.motion_bodies.shape[-1],
            ground_tolerance=self.ground_tolerance, friction_mu=env["plane"]["dynamicFriction"], **physx)
        if structs is None:
            self._env = native.Env(self._model_struct, self._verts, self._cfg_struct, self.num_envs, self.device_id)
        else:
            self._env = native.Env(structs, verts, self._cfg_struct, self.num_envs, self.device_id, env_asset=self._env_asset)
        self._key_body_ids = torch.tensor(list(self._cfg_struct.key_body)[:self._cfg_struct.num_key], device=self.device)
        self._contact_body_ids = torch.tensor([i for i in range(self.num_bodies) if self._cfg_struct.contact_body[i]],
                                              device=self.device)
        self._termination_heights = torch.tensor(list(self._cfg_struct.termination_height)[:self.num_bodies], device=self.device)

    def _bind(self):
        """_setup_tensors (humanoid_smpl.py:66-113): same shapes / views, torch-owned storage."""
        N, dev = self.num_envs, self.device
        B, D, nbl = self.num_bodies, self.num_dof, self._num_lib_bodies
        f = lambda *s: torch.zeros(*s, device=dev, dtype=torch.float)  # noqa: E731
        self._root_states = f(N, 13)
        self._root_states[:, 2] = 0.89  # start pose (:362-365)
        self._root_states[:, 6] = 1.0
        self._humanoid_root_states = self._root_states.view(N, 1, 13)[..., 0, :]
        self._initial_humanoid_root_states = self._humanoid_root_states.clone()
        self._dof_state = f(N * D, 2)
        self._dof_pos = self._dof_state.view(N, D, 2)[..., 0]
        self._dof_vel = self._dof_state.view(N, D, 2)[..., 1]
        self._initial_dof_pos, self._initial_dof_vel = f(N, D), f(N, D)
        self._rigid_body_state = f(N * B, 13)
        self._rigid_body_state[:, 6] = 1.0
        rbs = self._rigid_body_state.view(N, B, 13)
        self._rigid_body_pos, self._rigid_body_rot = rbs[..., 0:3], rbs[..., 3:7]
        self._rigid_body_vel, self._rigid_body_ang_vel = rbs[..., 7:10], rbs[..., 10:13]
        self._contact_force_tensor = f(N * B, 3)
        self._contact_forces = self._contact_force_tensor.view(N, B, 3)
        self.dof_force_tensor = f(N, D)
        K, S = self._cfg_struct.num_key, self._cfg_struct.shape_dim
        if "motion_assets" not in self.cfg["env"]:   # with motion_assets create_sim sampled them
            self._reset_ref_motion_ids = self._sample_motion_ids()
        self._reset_ref_motion_bodies = self._ml_t["motion_bodies"][self._reset_ref_motion_ids].contiguous()
        self._cur_ref_motion_times = f(N)
        self._reset_ref_motion_times = f(N)
        self._target_root_pos, self._target_root_rot = f(N, 3), f(N, 4)
        self._target_dof_pos, self._target_dof_vel = f(N, D), f(N, D)
        self._target_root_vel, self._target_root_ang_vel = f(N, 3), f(N, 3)
        self._target_key_pos, self._target_rb_pos, self._target_rb_rot = f(N, K, 3), f(N, nbl, 3), f(N, nbl, 4)
        self._prev_target_dof_pos, self._prev_target_dof_vel = f(N, D), f(N, D)
        self._prev_target_rb_pos, self._prev_target_rb_rot = f(N, nbl, 3), f(N, nbl, 4)
        self._pd_target_dof_pos = f(N, D)
        self.actions = f(N, self._num_actions)
        t = dict(root_states=self._root_states, dof_state=self._dof_state, rigid_body_state=self._rigid_body_state,
                 contact_forces=self._contact_force_tensor, obs_buf=self.obs_buf, rew_buf=self.rew_buf,
                 sub_rewards=self._sub_rewards, reset_buf=self.reset_buf, progress_buf=self.progress_buf,
                 terminate_buf=self._terminate_buf, motion_ids=self._reset_ref_motion_ids,
                 ref_motion_times=self._cur_ref_motion_times, motion_bodies=self._reset_ref_motion_bodies,
                 t_root_pos=self._target_root_pos, t_root_rot=self._target_root_rot, t_dof_pos=self._target_dof_pos,
                 t_root_vel=self._target_root_vel, t_root_ang_vel=self._target_root_ang_vel,
                 t_dof_vel=self._target_dof_vel, t_key_pos=self._target_key_pos, t_rb_pos=self._target_rb_pos,
                 t_rb_rot=self._target_rb_rot, p_dof_pos=self._prev_target_dof_pos, p_dof_vel=self._prev_target_dof_vel,
                 p_rb_pos=self._prev_target_rb_pos, p_rb_rot=self._prev_target_rb_rot,
                 pd_targets=self._pd_target_dof_pos, actions_used=self.actions)
        self._env.bind(t, actors_per_env=1, bodies_per_env=B, num_obs=self.num_obs)
        self._env.set_motion_lib(self._ml_t, nbl)
        self.extras["terminate"] = self._terminate_buf
        self.extras["sub_rewards"] = self._sub_rewards
        self.extras["sub_rewards_names"] = self._sub_rewards_names
        # SMPL kinematic constants the agent/network reads (humanoid_smpl_im.py:325-327)
        self.smpl_parents = torch.tensor(self._model["parent"][:nbl].astype(np.int64), device=dev)
        self.smpl_rest_joints = None  # needs the licensed SMPL model files (out of scope, SURVEY.md 2 row 17)

    def _sample_motion_ids(self):
        """humanoid_smpl_im.py:247-254"""
        env, M = self.cfg['env'], self._motion_lib.num_motions()
        if env.get('sample_first_motions', False):
            ids = torch.arange(self.num_envs, device=self.device) % M
        else:
            lens = self._ml_t["motion_lengths"]
            w = lens / lens.sum() if env.get('motion_weights_from_length', False) else torch.full_like(lens, 1.0 / M)
            ids = torch.multinomial(w, num_samples=self.num_envs, replacement=True)
        if 'motion_id' in env:
            ids[:] = env['motion_id']
        return ids.contiguous()

    # ------------------------------------------------------------------ Task surface
    def register_model(self, model):
        self.model = model

    def pre_epoch(self, epoch):
        return

    def step(self, actions):
        """BaseTask.step (base_task.py:147-165) = pre_physics_step + _physics_step + post_physics_step,
        fused into one launch; results are visible in the task buffers on return (same stream)."""
        a = actions.to(self.device, dtype=torch.float).contiguous()
        self._env.step(a)

    def reset(self, env_ids=None):
        """humanoid_smpl.py:136-140 -> _reset_envs (:153-159)"""
        if env_ids is None:
            env_ids = torch.arange(self.num_envs, device=self.device, dtype=torch.long)
        if len(env_ids) > 0:
            self._reset_actors(env_ids.to(self.device, dtype=torch.long).contiguous())

    def _reset_actors(self, env_ids):
        """:470-480, :638-651"""
        if self._state_init in ("Start", "Random"):
            self._reset_ref_state_init(env_ids)
        elif self._state_init == "Hybrid":
            if self._hybrid_init_prob >= 1.0:
                self._reset_ref_state_init(env_ids)
            else:
                mask = torch.bernoulli(torch.full((len(env_ids),), float(self._hybrid_init_prob), device=self.device)) == 1.0
                if mask.any():
                    self._reset_ref_state_init(env_ids[mask].contiguous())
                if (~mask).any():
                    self._reset_default(env_ids[~mask].contiguous())
        elif self._state_init == "Default":
            self._reset_default(env_ids)
        else:
            raise ValueError(f"Unsupported state initialization strategy: {self._state_init}")

    def _reset_default(self, env_ids):
        """:482-487 + humanoid_smpl.py:161-173; cold path, plain torch."""
        self._humanoid_root_states[env_ids] = self._initial_humanoid_root_states[env_ids]
        self._dof_pos[env_ids] = self._initial_dof_pos[env_ids]
        self._dof_vel[env_ids] = self._initial_dof_vel[env_ids]
        self.progress_buf[env_ids] = 0
        self.reset_buf[env_ids] = 0
        self._terminate_buf[env_ids] = 0
        obs = torch.cat([x[env_ids].reshape(len(env_ids), -1) for x in (
            self._rigid_body_pos[:, :self._num_lib_bodies], self._rigid_body_rot[:, :self._num_lib_bodies], self._dof_pos,
            self._dof_vel, self._rigid_body_vel[:, :self._num_lib_bodies], self._rigid_body_ang_vel[:, :self._num_lib_bodies],
            self._reset_ref_motion_bodies)], dim=-1)
        self.obs_buf[env_ids] = obs

    def sample_time(self, motion_ids, truncate_time=None):
        """MotionLib.sample_time (motion_lib.py:138-159)"""
        phase = torch.rand(motion_ids.shape, device=self.device)
        motion_len = self._ml_t["motion_lengths"][motion_ids]
        if truncate_time is not None:
            motion_len = torch.clamp_min(motion_len - truncate_time, 0)
        return phase * motion_len

    def _reset_ref_state_init(self, env_ids):
        """:489-528 (state write + targets + obs in one launch), then _init_context (:530-563)"""
        motion_ids = self._reset_ref_motion_ids[env_ids]
        if self._state_init in ("Random", "Hybrid"):
            truncate_time = self.context_length * self.dt if self.truncate_time else None
            motion_times = self.sample_time(motion_ids, truncate_time).contiguous()
        else:
            motion_times = torch.zeros(len(env_ids), device=self.device)
        self._env.reset(env_ids, motion_times)
        self._reset_ref_motion_times[env_ids] = motion_times
        self._reset_ref_env_ids = env_ids
        self._init_context(env_ids, motion_ids, motion_times)

    def _init_context(self, env_ids, motion_ids, motion_times):
        """:530-563: 48-frame MoCap window per env -> context_feat / context_mask (one launch)."""
        n = len(env_ids)
        P = self.context_length + self.context_padding * 2
        nbl, D = self._num_lib_bodies, self.num_dof
        W = 2 * (3 * nbl + D) + 4 * nbl
        with_conf = 'joint_conf' in self.context_names
        if not hasattr(self, "context_feat"):
            self.context_feat = torch.zeros(self.num_envs, P, W + (nbl if with_conf else 0), device=self.device)
            self.context_mask = torch.zeros(self.num_envs, P, device=self.device, dtype=torch.bool)
            self._context_raw = torch.zeros(self.num_envs, P, W, device=self.device) if with_conf else self.context_feat
        env_ids = env_ids.to(self.device, dtype=torch.long).contiguous()
        self._env.motion_context(env_ids, motion_ids.contiguous(), motion_times.contiguous(),
                                 P, -self.context_padding, self.dt, self._context_raw, self.context_mask)
        if with_conf:
            self.context_feat[env_ids] = self._transform_target(self._context_raw[env_ids])
        if self.model is not None:
            if not self.is_env_dim_setup:
                self.model.a2c_network.setup_env_named_dims(self.obs_names, self.obs_shapes, self.obs_dims,
                                                            self.context_names, self.context_shapes, self.context_dims)
                self.is_env_dim_setup = True
            with torch.no_grad():
                self.model.a2c_network.forward_context(self.context_feat, self.context_mask)

    def _transform_target(self, raw):
        """:565-592 on the rows of the window the kernel just wrote ([n, P, body_pos | body_rot | dof_pos | body_pos_gt | dof_pos_gt]):
        `mask_joints` / `noisy_joints` / `mask_random_joints` edit body_pos and produce joint_conf, appended as the last nbl columns.
        Reset-time only (cold path), plain torch on the device; the normal CDF is 0.5 erfc(-x / sqrt 2) instead of the reference's
        round trip through scipy on the CPU."""
        nbl = self._num_lib_bodies
        n, P, _ = raw.shape
        body_pos = raw[..., :3 * nbl].reshape(n, P, nbl, 3).clone()
        conf = torch.ones(n, P, nbl, device=raw.device)
        for transform, specs in (self._transform_specs or {}).items():
            if transform == 'mask_joints':
                idx = [self.body_names.index(j) for j in specs['joints']]
                conf[..., idx] = 0.0
                body_pos = body_pos * conf.unsqueeze(-1)
            elif transform == 'noisy_joints':
                noise_std = torch.full_like(conf, float(specs['noise_std']))
                noise_std[torch.bernoulli(torch.full_like(conf, float(specs['prob']))) == 0.0] = 0.0
                noise = torch.randn_like(body_pos) * noise_std.unsqueeze(-1)
                noise_norm = noise.norm(dim=-1) / (np.sqrt(3) * specs['conf_std'])
                conf = torch.erfc(noise_norm / np.sqrt(2.0))            # (1 - cdf(x)) * 2
                body_pos = body_pos + noise
                occluded = conf < specs['min_conf']
                conf[occluded] = 0.0
                body_pos[occluded] = 0.0
            elif transform == 'mask_random_joints':
                drop = torch.bernoulli(torch.full_like(conf, float(specs['prob']))) == 1.0
                drop[..., 0] = False
                conf[drop] = 0.0
                body_pos[drop] = 0.0
            else:
                raise NotImplementedError(f"transform_specs: unknown transform {transform!r}")
        return torch.cat([body_pos.reshape(n, P, -1), raw[..., 3 * nbl:], conf], dim=-1)

    def _init_context_torch(self, env_ids, motion_ids, motion_times):
        """the same window composed with torch ops from b200env_motion_state outputs (written like the reference, :530-563);
        kept as the executable specification b200env_motion_context is tested against"""
        n = len(env_ids)
        P = self.context_length + self.context_padding * 2
        steps = self.dt * torch.arange(-self.context_padding, self.context_length + self.context_padding, device=self.device)
        all_times = ((motion_times + self.dt).unsqueeze(-1) + steps).contiguous()
        all_ids = motion_ids.unsqueeze(-1).expand(n, P).contiguous()
        nbl, D = self._num_lib_bodies, self.num_dof
        f = lambda *s: torch.empty(*s, device=self.device, dtype=torch.float)  # noqa: E731
        rb_pos, rb_rot, dof_pos = f(n * P, nbl, 3), f(n * P, nbl, 4), f(n * P, D)
        self._env.motion_state(all_ids.view(-1), all_times.view(-1), dict(rb_pos=rb_pos, rb_rot=rb_rot, dof_pos=dof_pos))
        feat = torch.cat([rb_pos.view(n * P, -1), rb_rot.view(n * P, -1), dof_pos, rb_pos.view(n * P, -1), dof_pos], dim=-1)
        mask = all_times <= (self._ml_t["motion_lengths"][motion_ids] + 2 * self.dt).unsqueeze(-1)
        return feat.view(n, P, -1), mask

    def compute_imitation_obs(self, body_pos, body_rot, target_pos, target_rot, dof_pos, dof_vel, target_dof_pos,
                              body_vel, body_ang_vel, motion_bodies, local_root_obs=True, root_height_obs=True,
                              obs_type='full'):
        """compute_humanoid_observations_imitation (:773-850 == models/im_network_builder.py:262-338) as one
        kernel; what the embodied_pose network calls on the raw 461-d obs + context.  obs_type 'joint_pos' is
        compute_humanoid_observations_imitation_jpos (:853-915)."""
        n, nb = body_pos.shape[0], body_pos.shape[1]
        c = lambda x: x.contiguous().float()  # noqa: E731
        jpos = obs_type == 'joint_pos'
        width = 1 + (nb - 1) * 3 + nb * 6 + nb * 6 + self.num_dof + motion_bodies.shape[-1]
        width += (3 + nb * 3) if jpos else (11 + self.num_dof + nb * 9)
        obs = torch.empty(n, width, device=self.device)
        self._env.obs_imitation(c(body_pos), c(body_rot), c(target_pos), c(target_rot), c(dof_pos), c(dof_vel),
                                c(target_dof_pos), c(body_vel), c(body_ang_vel), c(motion_bodies), local_root_obs,
                                root_height_obs, obs, jpos=jpos)
        return obs

    def get_aux_losses(self, model_res_dict):
        """:694-722 - autograd-carrying, stays PyTorch."""
        from ..torch_ops import angle_axis_to_rot6d
        specs = self.cfg['env'].get('aux_loss_specs', dict())
        context = model_res_dict['extra']['context']
        aux, auxw = {}, {}
        w_dof = specs.get('w_dof', 0.0)
        if w_dof > 0:
            a = angle_axis_to_rot6d(context['dof_pos'].reshape(*context['dof_pos'].shape[:-1], -1, 3))
            b = angle_axis_to_rot6d(context['dof_pos_gt'].reshape(*context['dof_pos_gt'].shape[:-1], -1, 3))
            loss = ((a - b) ** 2).mean()
            aux['aux_dof_rot6d_loss'], auxw['aux_dof_rot6d_loss'] = loss, loss * w_dof
        w_pos = specs.get('w_pos', 0.0)
        if w_pos > 0:
            d = (context['body_pos_gt'] - context['body_pos']) * self.body_pos_weights[:, None]
            loss = (d ** 2).mean()
            aux['aux_body_pos_loss'], auxw['aux_body_pos_loss'] = loss, loss * w_pos
        return aux, auxw

    def render_vis(self, init=False):
        return
