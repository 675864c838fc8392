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


def resolve_test_motion_file(cfg):
    """humanoid_smpl_im.py:77-80: with args.test, cfg.env.test_motion_file replaces motion_file (and, with motion_assets, the test
    library's own cfg.env.test_motion_assets replace them).  Returns the test file, or None when the key is absent or args.test unset.
    A missing file, and motion_assets without test_motion_assets, are refused before anything is loaded."""
    env, args = cfg["env"], cfg.get("args", None)
    if args is None or not getattr(args, "test", False) or "test_motion_file" not in env:
        return None
    path = env["test_motion_file"]
    if not os.path.exists(path):
        raise FileNotFoundError(f"test_motion_file {path} does not exist")
    if "motion_assets" in env:
        if "test_motion_assets" not in env:
            raise ValueError(f"motion_assets names one asset per motion of motion_file; test_motion_file {path} needs its own "
                             "list in test_motion_assets")
        env["motion_assets"] = env["test_motion_assets"]
    env["motion_file"] = path
    return path


def motion_resample_share(cfg, test_task=False):
    """cfg.env.b200_resample_motions -> None when off, else the share h of the draws weighted by the motions' failure rates
    (cfg.env.b200_hard_motion_share, default 0).  Refuses the key in a test run (args.test, or test_task: HumanoidSMPLIMVis), with
    b200_motion_queue or motion_id, and h that is not a finite number in [0, 1] or is given without the key."""
    env = cfg["env"]
    if not env.get("b200_resample_motions", False):
        if "b200_hard_motion_share" in env:
            raise ValueError("b200_hard_motion_share weights the motions b200_resample_motions draws: set b200_resample_motions: True")
        return None
    args = cfg.get("args", None)
    if test_task or (args is not None and getattr(args, "test", False)):
        raise ValueError("b200_resample_motions draws training motions: a test run keeps each env's motion (or takes them from "
                         "b200_motion_queue)")
    if env.get("b200_motion_queue", False):
        raise ValueError("b200_resample_motions and b200_motion_queue both choose a finished env's next motion: set one of them")
    if "motion_id" in env:
        raise ValueError("b200_resample_motions draws from the whole library, motion_id pins every env to one motion: set one of them")
    h = env.get("b200_hard_motion_share", 0.0)
    if isinstance(h, bool) or not isinstance(h, (int, float, np.integer, np.floating)) or not 0.0 <= float(h) <= 1.0:
        raise ValueError(f"b200_hard_motion_share must be a finite number in [0, 1], got {h!r}")
    return float(h)


class HumanoidSMPLIM(BaseTask):
    _test_task = False      # HumanoidSMPLIMVis: the test run's task
    _rs = None              # the training resample's device state (cfg.env.b200_resample_motions), set by _bind
    _asset_error = None     # [1] int32 error word of b200env_set_env_assets when envs change body on the device

    def __init__(self, cfg, sim_params, physics_engine, device_type, device_id, headless):
        self.cfg = cfg
        self.args = cfg.get('args', None)
        env = cfg["env"]
        self._resample_share = motion_resample_share(cfg, self._test_task)
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
        self._test_motion_file = resolve_test_motion_file(cfg)
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
        env = self.cfg["env"]
        if self._test_motion_file is not None and "motion_assets" in env and len(env["motion_assets"]) != flat.num_motions():
            raise ValueError(f"test_motion_assets has {len(env['motion_assets'])} entries for the {flat.num_motions()} motions of "
                             f"test_motion_file {self._test_motion_file}")
        self._check_motion_lib(flat)
        self._motion_lib = flat
        dev = self.device
        self._ml_t = {k: torch.from_numpy(getattr(flat, k)).to(dev).contiguous() for k in FlatMotionLib.FIELDS}

    def _check_motion_lib(self, flat):
        """refusals that need the loaded library, before it goes to the device (none here)"""

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
        # cfg.env.b200_device_transforms (addition): the context window's transforms run in the window launches (include/b200env.h:
        # b200_motion_context_t), so reset_masked / reset_done and their graph serve transform_specs; the program is built here, once
        self._xf_program = None
        if self.cfg['env'].get('b200_device_transforms', False) and 'transform_specs' in self.cfg['env']:
            self._xf_program = abi.transform_program(self._transform_specs, self.body_names, nb)
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
        resolved = {}    # file name or id of a model dict -> asset index: a library of thousands of motions loads each file once
        for entry in entries:
            ref = os.path.splitext(os.path.basename(str(entry)))[0] if isinstance(entry, (str, os.PathLike)) else id(entry)
            if ref not in resolved:
                model = model_compiler.load_compiled(ref) if isinstance(ref, str) else entry
                ms, verts = self._pack(model)
                key = bytes(ms) + verts.tobytes()
                if key not in keys:
                    keys[key] = len(models)
                    models.append(model)
                resolved[ref] = keys[key]
            of_motion.append(resolved[ref])
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
            self._asset_models, self._motion_asset = models, of_motion
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
            if self._resample_share is not None and len(models) > 1:
                self._env.fix_mixed_plan()     # a resampled env takes its new motion's body
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
        # DOF force sensors (enable_actor_dof_force_sensors, :369; include/b200env.h b200_buffers_t::dof_force): with
        # cfg.env.dof_force_sensors the physics launch of every step writes the joints' drive + limit torques of its last substep here
        # (same storage for the task's lifetime); without it the tensor stays zero
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
        # reset_masked / reset_done: draw counter, work list of the context launch, mask of the finished envs, captured reset graph
        self._reset_rng = torch.zeros(1, device=dev, dtype=torch.long)
        self._reset_work = torch.zeros(N + 2, device=dev, dtype=torch.int32)
        self._reset_mask = torch.zeros(N, device=dev, dtype=torch.bool)
        self._reset_graph = None
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
        if self.cfg["env"].get("dof_force_sensors", False):
            t["dof_force"] = self.dof_force_tensor
        self._env.bind(t, actors_per_env=1, bodies_per_env=B, num_obs=self.num_obs)
        self._env.set_motion_lib(self._ml_t, nbl)
        if self._resample_share is not None:
            self._rs = self._resample_buffers()
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

    def _resample_buffers(self):
        """the training resample's device state: the CDF of the base distribution (b_m = motion_lengths[m] under
        motion_weights_from_length, else uniform, as _sample_motion_ids draws), the draw counter and its done ticket, the mask of an
        id-list reset; with b200_hard_motion_share > 0 the counts and the rates (r_m = 1 at the start); with several bodies each
        motion's and each env's asset"""
        N, M, dev = self.num_envs, self._motion_lib.num_motions(), self.device
        i64 = lambda n: torch.zeros(n, device=dev, dtype=torch.long)  # noqa: E731
        base = self._ml_t["motion_lengths"] if self.cfg["env"].get("motion_weights_from_length", False) else None
        rs = dict(base=base, cdf=torch.zeros(M, device=dev, dtype=torch.float64), counter=i64(1),
                  done=torch.zeros(1, device=dev, dtype=torch.int32), id_mask=torch.zeros(N, device=dev, dtype=torch.bool))
        if self._resample_share > 0:
            rs.update(tries=i64(M), fails=i64(M), rate=torch.ones(M, device=dev, dtype=torch.float64))
        native.motion_weights(dict(num_motions=M, h=0.0), dict(base=base, cdf=rs["cdf"]))
        if len(getattr(self, "_asset_models", ())) > 1:
            i32 = lambda a: torch.as_tensor(a, dtype=torch.int32, device=dev)  # noqa: E731
            rs.update(motion_asset=i32(self._motion_asset), env_asset=i32(self._env_asset))
            self._asset_error = torch.zeros(1, device=dev, dtype=torch.int32)
        return rs

    def _resample_motions(self, mask):
        """the masked envs that played a step draw their next motion (and body) on the device, before their reset"""
        rs = self._rs
        native.resample_motions(dict(n=self.num_envs, num_motions=self._motion_lib.num_motions(),
                                     shape_dim=self._reset_ref_motion_bodies.shape[1], seed=int(self.cfg.get("seed", 10))),
                                dict(rs, mask=mask, progress_buf=self.progress_buf, terminate_buf=self._terminate_buf,
                                     lib_motion_bodies=self._ml_t["motion_bodies"], motion_ids=self._reset_ref_motion_ids,
                                     motion_bodies=self._reset_ref_motion_bodies))
        if "env_asset" in rs:                  # the new bodies, read by the next physics launch
            self._env.set_env_assets(rs["env_asset"], self._asset_error)

    def _check_asset_error(self):
        """the host's check of b200env_set_env_assets' error word, at its sync points"""
        if self._asset_error is not None:
            e = int(self._asset_error)
            if e:
                raise ValueError(f"b200env_set_env_assets: env {e - 1} was given an asset index outside the handle's "
                                 f"{len(self._asset_models)} assets; its body was left unchanged")

    # ------------------------------------------------------------------ Task surface
    def register_model(self, model):
        self.model = model

    def pre_epoch(self, epoch):
        """with cfg.env.b200_resample_motions: reads the asset error word (the agent has just read its losses on the host, so this waits
        for no work), then, with b200_hard_motion_share > 0, rebuilds the resample's distribution from the last epoch's counts in one
        launch, in place, with no host synchronisation (include/b200env.h: b200env_motion_weights)"""
        if self._rs is None:
            return
        self._check_asset_error()
        if self._resample_share > 0:
            native.motion_weights(dict(num_motions=self._motion_lib.num_motions(), h=self._resample_share), self._rs)

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
            env_ids = env_ids.to(self.device, dtype=torch.long).contiguous()
            if self._rs is not None:
                mask = self._rs["id_mask"]
                mask.zero_()
                mask[env_ids] = True
                self._resample_motions(mask)
            self._reset_actors(env_ids)

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

    def reset_masked(self, mask, step=None):
        """Addition (not in the reference): `reset(mask.nonzero())` without the id list - the envs whose entry of `mask` ([num_envs]
        bool, device) is set are reset by two launches (include/b200env.h: b200env_reset_masked) that make no host synchronisation,
        so the call can be captured in a CUDA graph.  Same state init, rows and context window as `reset(env_ids)`; the motion
        times and the Hybrid choice are drawn on the device from a counter-based generator seeded by cfg["seed"], a different stream
        of the same distribution as the torch.rand / torch.bernoulli draws of `reset(env_ids)`.  With cfg.env.transform_specs only under
        cfg.env.b200_device_transforms (the window launch applies them, drawing at the same counter); otherwise the transforms are torch
        ops on the reset rows: use `reset(env_ids)` there.  step: a device step counter ([1] int64) the policy reads its context slot
        from; each window then starts step % context_length frames earlier, so the next slot read is the new game's first frame.
        With cfg.env.b200_resample_motions the masked envs that played a step first draw their next motion (and body) on the device,
        as `reset(env_ids)` does for its ids."""
        if self._transform_specs is not None and self._xf_program is None:
            raise ValueError("reset_masked: cfg.env.transform_specs transforms the context window in torch - use reset(env_ids), "
                             "or set cfg.env.b200_device_transforms")
        modes = {"Start": (False, 1.0), "Random": (True, 1.0), "Hybrid": (True, min(float(self._hybrid_init_prob), 1.0)),
                 "Default": (False, 0.0)}
        if self._state_init not in modes:
            raise ValueError(f"Unsupported state initialization strategy: {self._state_init}")
        sample_time, ref_prob = modes[self._state_init]
        truncate = self.context_length * self.dt if self.truncate_time else 0.0
        if self._rs is not None:
            self._resample_motions(mask)
        self._context_buffers()
        self._env.reset_masked(mask, sample_time, truncate, ref_prob, self.cfg.get("seed", 10), self._reset_rng,
                               self._initial_humanoid_root_states, self._initial_dof_pos, self._initial_dof_vel, self._reset_ref_motion_times,
                               self.context_length + self.context_padding * 2, -self.context_padding, self.dt, self.context_feat,
                               self.context_mask, self._reset_work, transforms=self._xf_program, step=step,
                               context_length=self.context_length if step is not None else None)
        self._forward_context()

    def reset_done(self):
        """Addition: reset the envs whose reset_buf is set, from the device flags: the mask is taken with torch.ne and the reset is
        one replay of the reset graph when one was captured (VecTaskPython.enable_cuda_graph(reset_graph=True)), else `reset_masked`.
        No host synchronisation.  With cfg.env.transform_specs and without cfg.env.b200_device_transforms: `reset(reset_buf.nonzero())`."""
        if self._transform_specs is not None and self._xf_program is None:
            self.reset(self.reset_buf.nonzero(as_tuple=False).flatten())
            return
        torch.ne(self.reset_buf, 0, out=self._reset_mask)
        if self._reset_graph is not None:
            self._reset_graph.replay()
        else:
            self.reset_masked(self._reset_mask)

    def _capture_reset_graph(self, tail=None):
        """capture `reset_masked(self._reset_mask)` and then `tail()` as the graph `reset_done` replays (warm-up: one eager call with an
        empty mask, which only advances the draw counter); nothing with cfg.env.transform_specs unless cfg.env.b200_device_transforms.
        Returns whether a graph was captured."""
        if self._transform_specs is not None and self._xf_program is None:
            return False
        self._reset_graph = None
        self._reset_mask.zero_()
        s = torch.cuda.Stream(device=self.device)
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            self.reset_masked(self._reset_mask)
            if tail is not None:
                tail()
        torch.cuda.current_stream().wait_stream(s)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            self.reset_masked(self._reset_mask)
            if tail is not None:
                tail()
        self._reset_graph = g
        return True

    def _context_buffers(self):
        P = self.context_length + self.context_padding * 2
        nbl, D = self._num_lib_bodies, self.num_dof
        W = 2 * (3 * nbl + D) + 4 * nbl
        with_conf = 'joint_conf' in self.context_names
        if not hasattr(self, "context_feat"):
            self.context_feat = torch.zeros(self.num_envs, P, W + (nbl if with_conf else 0), device=self.device)
            self.context_mask = torch.zeros(self.num_envs, P, device=self.device, dtype=torch.bool)
            torch_xf = with_conf and self._xf_program is None        # the torch transforms read the raw rows of a W-wide buffer
            self._context_raw = torch.zeros(self.num_envs, P, W, device=self.device) if torch_xf else self.context_feat
        return P, with_conf

    def _init_context(self, env_ids, motion_ids, motion_times):
        """:530-563: 48-frame MoCap window per env -> context_feat / context_mask (one launch).  Under cfg.env.b200_device_transforms
        the launch also applies transform_specs, drawing at the masked reset's counter, which it then advances (a torch add)."""
        P, with_conf = self._context_buffers()
        env_ids = env_ids.to(self.device, dtype=torch.long).contiguous()
        if self._xf_program is not None:
            self._env.motion_context(env_ids, motion_ids.contiguous(), motion_times.contiguous(), P, -self.context_padding, self.dt,
                                     self.context_feat, self.context_mask, transforms=self._xf_program, seed=self.cfg.get("seed", 10),
                                     counter=self._reset_rng)
            self._reset_rng.add_(1)
            self._forward_context()
            return
        self._env.motion_context(env_ids, motion_ids.contiguous(), motion_times.contiguous(),
                                 P, -self.context_padding, self.dt, self._context_raw, self.context_mask)
        if with_conf:
            self.context_feat[env_ids] = self._transform_target(self._context_raw[env_ids])
        self._forward_context()

    def _forward_context(self):
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
