"""PhysicsMVAEController mirror - the high-level vid2player env the PPO agent sees
(vid2player/env/tasks/physics_mvae_controller.py).  It owns a kinematic motion generator (the MVAE player in the
reference; PyTorch, stays PyTorch) and the physics player (low-level policy + HumanoidSMPLIMMVAE).  One `step`:

  pre_physics_step  (:247-269)  split the action, advance the motion generator, task.post_mvae_step()  [1 FK + 1 obs launch]
  physics_step      (:362-366)  low-level policy (PyTorch MLP) -> task.step                         [1 fused physics launch + 1]
  post_physics_step (:441-452)  bounce / estimator bookkeeping, reward, obs, reset FSM               [1 fused launch]

The MVAE checkpoints and the trained low-level policy are not released (README.md:13), so `SyntheticMotionPlayer` and a
zero-residual policy stand in for tests and benchmarks; any object with the MVAEPlayer attribute surface
(`_root_pos _joint_rotmat _phase_pred _swing_type _swing_type_cycle reset(ids) step(a, res)`) can be plugged in through
cfg['env']['motion_player'], and any callable obs->action through cfg['env']['low_level_policy'].
"""
import math
from types import SimpleNamespace

import numpy as np
import torch

from .. import ball as ball_data, native_v2p
from ..torch_ops import get_opponent_env_ids
from .humanoid_smpl_im_mvae import HumanoidSMPLIMMVAE, HumanoidSMPLIMMVAEDual

# SMPL shape coefficients of the three players (vid2player/env/tasks/physics_mvae_controller.py:119-125); they reach the
# low-level policy through the last 10 entries of the 734-d observation
SMPL_BETA = {
    'djokovic': [-0.9807, 1.4050, -0.4144, 1.4028, -1.3299, 2.0045, -1.3108, 0.7475, -0.0924, -0.3262],
    'federer': [-0.6303, 1.1747, -0.3463, 1.0915, -1.0501, 1.7888, -1.1762, 0.6059, 0.2589, -0.4568],
    'nadal': [-0.6278, 1.2620, -0.3143, 0.8561, -0.8136, 1.3917, -0.9902, 0.5112, 0.2334, -0.4266],
}

BASE_ROTMAT = [[0.0, 0.0, 1.0], [1.0, 0.0, 0.0], [0.0, 1.0, 0.0]]  # quaternion (.5,.5,.5,.5): SMPL y-up -> world z-up


_SKEW = None


def _aa_to_rotmat(aa):
    """rotation vectors [...,3] -> matrices, Rodrigues as I + s K + c K K with K from one matmul (10 launches instead of ~30)"""
    global _SKEW
    if _SKEW is None or _SKEW.device != aa.device:
        g = torch.zeros(3, 9, device=aa.device)
        g[0, 5], g[0, 7] = -1.0, 1.0      # x: K[1,2] = -x, K[2,1] = x
        g[1, 2], g[1, 6] = 1.0, -1.0      # y: K[0,2] = y,  K[2,0] = -y
        g[2, 1], g[2, 3] = -1.0, 1.0      # z: K[0,1] = -z, K[1,0] = z
        _SKEW = g
    K = (aa.reshape(-1, 3) @ _SKEW).view(-1, 3, 3)
    a2 = (aa * aa).sum(-1).reshape(-1, 1, 1).clamp_min(1e-12)
    a = a2.sqrt()
    R = torch.baddbmm(K * (torch.sin(a) / a), K, K * ((1 - torch.cos(a)) / a2))     # s K + c K K
    R.diagonal(dim1=-2, dim2=-1).add_(1.0)
    return R.view(*aa.shape[:-1], 3, 3)


class SyntheticMotionPlayer:
    """Stand-in for MVAEPlayer (vid2player/players/mvae_player.py:184-431): a mean-reverting random walk of the 24 SMPL joint
    rotations driven by the 32-d latent action, a slow planar root drift, a 2*pi/60 per step phase clock and a cycling swing type."""

    def __init__(self, num_envs, device, seed=10, court_min=(-5.0, -16.0), court_max=(5.0, -10.0)):
        self.N, self.device = num_envs, device
        self.gen = torch.Generator(device=device).manual_seed(seed)   # construction / reset only; step() uses the default generator
                                                                       # and updates its state IN PLACE so it can live inside a CUDA graph
        self._aa = torch.zeros(num_envs, 24, 3, device=device)
        self._root_pos = torch.zeros(num_envs, 3, device=device)
        self._joint_rotmat = torch.eye(3, device=device).repeat(num_envs, 24, 1, 1)
        self._phase_pred = torch.zeros(num_envs, device=device)
        self._swing_type = torch.zeros(num_envs, device=device, dtype=torch.long)
        self._swing_type_cycle = -torch.ones(num_envs, device=device, dtype=torch.long)
        self._heading = torch.zeros(num_envs, device=device)
        self._racket_pos = torch.zeros(num_envs, 3, device=device)        # kinematic racket position (serve toss point in dual mode)
        self._racket_off = torch.tensor([0.35, 0.25, 0.25], device=device)
        self._base = torch.tensor(BASE_ROTMAT, device=device)
        self._proj = torch.randn(32, 72, device=device, generator=self.gen) * 0.02
        self.court_min, self.court_max = court_min, court_max
        self._lo = torch.tensor([court_min[0] + 1, court_min[1] + 1, 0.95], device=device)
        self._span = torch.tensor([court_max[0] - court_min[0] - 2, court_max[1] - court_min[1] - 2, 0.0], device=device)

    def _update_rotmat(self, ids=None):
        aa, heading = (self._aa, self._heading) if ids is None else (self._aa[ids], self._heading[ids])
        R = _aa_to_rotmat(aa)
        c, s = torch.cos(heading), torch.sin(heading)
        z, o = torch.zeros_like(c), torch.ones_like(c)
        H = torch.stack([c, -s, z, s, c, z, z, z, o], -1).view(-1, 3, 3)
        R[:, 0] = H @ self._base @ R[:, 0]
        if ids is None:
            self._joint_rotmat.copy_(R)
        else:
            self._joint_rotmat[ids] = R

    def reset(self, env_ids):
        n = len(env_ids)
        r = torch.rand(n, 3, device=self.device, generator=self.gen)
        self._root_pos[env_ids] = self._lo + r * self._span
        self._aa[env_ids] = 0.05 * torch.randn(n, 24, 3, device=self.device, generator=self.gen)
        self._heading[env_ids] = math.pi / 2 + 0.2 * (r[:, 2] - 0.5)       # facing +y (the net)
        self._phase_pred.index_fill_(0, env_ids, 0.0)
        self._swing_type.index_fill_(0, env_ids, 0)
        self._swing_type_cycle.index_fill_(0, env_ids, -1)
        self._racket_pos[env_ids] = self._root_pos[env_ids] + self._racket_off
        self._update_rotmat(env_ids)

    def reset_masked(self, mask):
        """reset() for the envs whose mask is set, written as full-width in-place ops (no id list, default generator): it can be
        captured into a CUDA graph together with the rest of a mask-driven env reset"""
        N, m1, m3 = self.N, mask, mask[:, None]
        r = torch.rand(N, 3, device=self.device)
        self._root_pos.copy_(torch.where(m3, self._lo + r * self._span, self._root_pos))
        self._aa.copy_(torch.where(mask[:, None, None], 0.05 * torch.randn(N, 24, 3, device=self.device), self._aa))
        self._heading.copy_(torch.where(m1, math.pi / 2 + 0.2 * (r[:, 2] - 0.5), self._heading))
        self._phase_pred.masked_fill_(m1, 0.0)
        self._swing_type.masked_fill_(m1, 0)
        self._swing_type_cycle.masked_fill_(m1, -1)
        self._racket_pos.copy_(torch.where(m3, self._root_pos + self._racket_off, self._racket_pos))
        self._update_rotmat()          # all rows: the rotation matrices are a pure function of (_aa, _heading)

    def reset_dual(self, reset_reaction_env_ids, reset_recovery_env_ids):
        """players/mvae_player.py:167-182: both players of the listed pairs restart (ready pose / serve pose in the reference)"""
        self.reset(torch.cat([reset_reaction_env_ids, reset_recovery_env_ids]).sort().values)
        self._swing_type.index_fill_(0, reset_reaction_env_ids, -1)
        self._swing_type.index_fill_(0, reset_recovery_env_ids, -1)

    def step(self, mvae_actions, res_dof_actions=None):
        drive = (mvae_actions[:, :32] @ self._proj).view(self.N, 24, 3)
        noise = 0.02 * torch.randn(self.N, 24, 3, device=self.device)
        self._aa.mul_(0.97).add_(drive).add_(noise)
        self._aa[:, 0] *= 0.3
        if res_dof_actions is not None and res_dof_actions.numel():
            self._aa[:, 21] += res_dof_actions[:, :3] * 0.1          # residual on the racket wrist (add_residual_dof)
        self._root_pos[:, :2] += 0.01 * torch.randn(self.N, 2, device=self.device)
        self._racket_pos.copy_(self._root_pos + self._racket_off)
        self._phase_pred.copy_(torch.remainder(self._phase_pred + 2 * math.pi / 60, 2 * math.pi))
        wrap = self._phase_pred < 2 * math.pi / 60
        self._swing_type.copy_(torch.where(wrap, (self._swing_type + 1) % 4, self._swing_type))
        self._swing_type_cycle.copy_(torch.where(self._phase_pred > 2.0, self._swing_type, self._swing_type_cycle))
        self._update_rotmat()


class StreamMotionPlayer:
    """The "synthetic kinematic target stream" of SURVEY.md 8d (config 3): K frames of the SyntheticMotionPlayer's random walk are
    generated ONCE and kept in HBM (joint rotation matrices [K, N, 24, 3, 3] = 7 MB per frame at 8192 envs); a step gathers frame
    (t + offset[env]) % K of every env into the fixed buffers the FK kernel reads (one gather per field, no per-step math), a reset
    re-draws the env's offset.  Same fields and methods as SyntheticMotionPlayer; everything is in place and sync-free, so step and
    masked reset live in CUDA graphs.  The latent action does not steer the stream (throughput stand-in; the MVAE network is out of
    the kernel path, SURVEY.md 8d).  The stream is not periodic: an env's targets jump once every K steps."""

    FIELDS = ("_joint_rotmat", "_root_pos", "_racket_pos", "_phase_pred", "_swing_type", "_swing_type_cycle")

    def __init__(self, num_envs, device, seed=10, frames=48, court_min=(-5.0, -16.0), court_max=(5.0, -10.0)):
        src = SyntheticMotionPlayer(num_envs, device, seed=seed, court_min=court_min, court_max=court_max)
        self.N, self.K, self.device = num_envs, frames, device
        gen = torch.Generator(device=device).manual_seed(seed + 1)
        src.reset(torch.arange(num_envs, device=device))
        rings = {f: [] for f in self.FIELDS}
        for _ in range(frames):
            src.step(torch.clamp(torch.randn(num_envs, 32, device=device, generator=gen), -5, 5))
            for f in self.FIELDS:
                rings[f].append(getattr(src, f).clone())
        self._ring = {f: torch.stack(v, 0).reshape(frames * num_envs, *v[0].shape[1:]).contiguous() for f, v in rings.items()}
        for f in self.FIELDS:                                   # the live buffers the env reads (fixed addresses)
            setattr(self, f, rings[f][0].clone())
        self._t = torch.zeros(1, device=device, dtype=torch.long)
        self._seed = int(seed) * 104729 + 7
        self._done = torch.zeros(1, device=device, dtype=torch.int32)      # scratch of the launch (last-block counter)
        self._off = torch.randint(0, frames, (num_envs,), device=device, generator=gen)
        self._gt = dict(clock=self._t, done_counter=self._done, offset=self._off, ring_rotmat=self._ring["_joint_rotmat"], rotmat=self._joint_rotmat,
                        ring_root_pos=self._ring["_root_pos"], root_pos=self._root_pos, ring_racket_pos=self._ring["_racket_pos"],
                        racket_pos=self._racket_pos, ring_phase=self._ring["_phase_pred"], phase=self._phase_pred,
                        ring_swing_type=self._ring["_swing_type"], swing_type=self._swing_type,
                        ring_swing_type_cycle=self._ring["_swing_type_cycle"], swing_type_cycle=self._swing_type_cycle)
        self._gather()

    def _gather(self, advance=0, reseed_mask=None):
        """one launch (b200v2p_stream_gather): frame (t + advance + off[e]) % K of every field -> the live buffers; advance moves the
        clock; reseed_mask: those envs draw a new offset first (counter-based) and only they are re-read"""
        native_v2p.stream_gather(self.N, self.K, advance, self._gt, reseed_mask=reseed_mask, seed=self._seed)

    def step(self, mvae_actions, res_dof_actions=None):
        self._gather(advance=1)

    def reset(self, env_ids):
        self._off[env_ids] = torch.randint(0, self.K, (len(env_ids),), device=self.device)
        self._gather()

    def reset_masked(self, mask):
        self._gather(reseed_mask=mask)          # one launch: new offsets for the masked envs + their frames

    def reset_dual(self, reset_reaction_env_ids, reset_recovery_env_ids):
        self.reset(torch.cat([reset_reaction_env_ids, reset_recovery_env_ids]).sort().values)


class DecoderStreamPlayer(StreamMotionPlayer):
    """StreamMotionPlayer + the MVAE decoder forward of MVAEPlayer.step (vid2player/players/mvae_player.py:184-199) executed every
    step with parameters of the reference's shapes (random: the trained checkpoints are unreleased, README.md:13): the 32-d latent
    action and the 288-d condition go through `nn.MixedDecoder` (gate + three mixture-of-experts layers, wgmma GEMMs,
    include/b200nn.h), the predicted frame becomes the next condition like `_update_mvae_state` (:201-204, autoregressive, kept in
    the normalised range), the two extra outputs are the phase prediction (`_phase_decoded`).  The kinematic TARGETS still come from
    the resident stream - a random-weight decoder produces noise poses - so this measures the decoder where it runs (inside the
    step graph, on the live action) without letting it steer the humanoid."""

    def __init__(self, num_envs, device, seed=10, **kw):
        super().__init__(num_envs, device, seed=seed, **kw)
        from .. import nn
        self.decoder = nn.MixedDecoder.random(num_envs, device, seed=seed)
        g = torch.Generator(device=device).manual_seed(seed + 2)
        self._init_data = torch.randn(num_envs, self.decoder.cond, device=device, generator=g).clamp_(-3, 3)   # :160 `_init_data`
        self.decoder.set_condition(self._init_data)
        # the condition state lives in the decoder's bf16 operand buffer (columns latent .. latent + cond of its first layer input)
        self._cond_view = self.decoder.x0[:num_envs, self.decoder.L:self.decoder.L + self.decoder.cond]
        self._init_bf16 = self._init_data.to(torch.bfloat16)
        self._phase_decoded = torch.zeros(num_envs, device=device)

    def reset(self, env_ids):
        super().reset(env_ids)
        self._cond_view[env_ids] = self._init_bf16[env_ids]           # :162-166 condition of a reset env = its initial frame

    def reset_masked(self, mask):
        super().reset_masked(mask)
        self.decoder.set_condition(self._init_data, row_mask=mask)      # one launch, masked rows only

    def step(self, mvae_actions, res_dof_actions=None):
        super().step(mvae_actions, res_dof_actions)
        out = self.decoder(mvae_actions)           # condition = the previous prediction, already in the operand buffer
        self.decoder.feed_back(clamp=3.0)          # :201-204 the predicted frame is the next condition
        torch.atan2(out[:, -2], out[:, -1], out=self._phase_decoded)


class PhysicsMVAEController:
    def __init__(self, cfg, sim_params, physics_engine, device_type, device_id, headless):
        self.cfg = cfg
        env = cfg["env"]
        self.cfg_v2p = env["vid2player"]
        cfg["device_type"], cfg["device_id"], cfg["headless"] = device_type, device_id, headless
        if device_type not in ("cuda", "GPU"):
            raise RuntimeError("the environment runs on a CUDA device only (no CPU pipeline)")
        self._max_episode_length = env["episodeLength"]
        self._enable_early_termination = env.get("enableEarlyTermination", False)
        self._is_train = env.get("is_train", True)
        self.device_type, self.device_id = device_type, device_id
        self.device = "cuda:" + str(device_id)
        self.headless = headless
        self.num_envs = N = env["numEnvs"]
        self._sim_params, self._physics_engine = sim_params, physics_engine
        self._num_mvae_action = 32
        self._num_res_dof_action = 3 if self.cfg_v2p.get('add_residual_dof') else 0
        self._num_actions = self._num_mvae_action + self._num_res_dof_action + (3 if self.cfg_v2p.get('add_residual_root') else 0)
        self._obs_ball_traj_length = self.cfg_v2p.get('obs_ball_traj_length', 100)
        self._num_actor_obs = 3 + 3 + 24 * 3 + 24 * 6 + 3
        self._num_task_obs = 3 * self._obs_ball_traj_length + (2 if self.cfg_v2p.get('use_random_ball_target', False) else 0)
        self.num_obs = env["numObservations"] = self._num_actor_obs + self._num_task_obs
        self.num_actions = env["numActions"] = self._num_actions
        self.num_states = env.get("numStates", 0)
        if self.cfg_v2p.get('dual_mode') == 'different':          # :127-135
            self.cfg_v2p['smpl_beta'] = [SMPL_BETA[p] for p in self.cfg_v2p['player']]
        else:
            self.cfg_v2p['smpl_beta'] = SMPL_BETA.get(self.cfg_v2p.get('player'), [0.0] * 10)
        self.create_sim()
        dev = self.device
        f = lambda *s: torch.zeros(*s, device=dev, dtype=torch.float)  # noqa: E731
        b = lambda *s: torch.zeros(*s, device=dev, dtype=torch.bool)   # noqa: E731
        i64 = lambda *s: torch.zeros(*s, device=dev, dtype=torch.long)  # noqa: E731
        self.obs_buf, self.rew_buf = f(N, self.num_obs), f(N)
        self.states_buf = f(N, self.num_states)
        self.reset_buf = torch.ones(N, device=dev, dtype=torch.long)
        self.progress_buf = i64(N)
        self._terminate_buf = torch.ones(N, device=dev, dtype=torch.long)
        self.extras = {}
        self._sub_rewards = f(N, 2)
        self._has_init = False
        self._graph = None
        self._num_humanoid_bodies, self._racket_body_id, self._head_body_id = 24, 24, 13
        self._ball_traj = f(N, 100, 3)
        self._ball_obs = f(N, self._obs_ball_traj_length, 3)            # :65 history of ball positions (rolled at every observation)
        self._use_history = bool(self.cfg_v2p.get('use_history_ball_obs', False))
        self._bounce_in, self._est_bounce_in = b(N), b(N)
        self._est_bounce_pos, self._est_bounce_time, self._est_max_height = f(N, 3), f(N), f(N)
        self._court_min = torch.tensor(self.cfg_v2p.get('court_min', [-5, -16]), device=dev, dtype=torch.float)
        self._court_max = torch.tensor(self.cfg_v2p.get('court_max', [5, -10]), device=dev, dtype=torch.float)
        self._tar_time, self._tar_time_total, self._tar_action = i64(N), i64(N), i64(N)
        self._target_bounce_pos = f(N, 3)
        self._target_bounce_pos[:] = torch.tensor([0.0, 10.0, 0.0], device=dev)
        self._target_bounce_min = torch.tensor([-3.0, 9.0, 0.0], device=dev)
        self._target_bounce_max = torch.tensor([3.0, 11.0, 0.0], device=dev)
        self._reset_reaction_buf = torch.ones(N, device=dev, dtype=torch.bool)
        self._reset_recovery_buf = b(N)
        self._num_reset_reaction, self._num_reset = i64(N), i64(N)
        self._distance = f(N)
        self._res_root_actions = f(N, 3)
        self._mvae_actions_random = f(N, self._num_mvae_action)
        # outgoing-ball estimator tables on the device (the reference keeps them on the CPU and syncs every contact step)
        if not self.cfg_v2p.get('dual_mode'):
            tabs = self.cfg_v2p.get('ball_out_tables', None)
            if tabs is None:
                tabs = ball_data.synthetic_out_tables(spin_scale=self.cfg_v2p.get('spin_scale', 1.0))
            self._est_x = torch.tensor(tabs[0], device=dev).contiguous()
            self._est_y = torch.tensor(tabs[1], device=dev).contiguous()
            self._est_params = np.asarray(tabs[2], np.float64).reshape(-1)
        else:
            self._est_x = self._est_y = None
            self._est_params = np.zeros(15)
        scales = self.cfg_v2p.get('reward_scales', {})
        weights = self.cfg_v2p.get('reward_weights', {})
        rtype = self.cfg_v2p.get('reward_type', 'return')
        self._sub_rewards_names = 'pos_reward' if rtype == 'reach' else 'pos_reward,ball_pos_reward'
        self._post_cfg = dict(
            n=N, bodies_per_env=26, ball_stride=26, racket_body=24, num_obs=self.num_obs, obs_traj_len=self._obs_ball_traj_length,
            use_target=int(bool(self.cfg_v2p.get('use_random_ball_target', False))), reward_type=native_v2p.REWARD_TYPES[rtype],
            early_termination=int(bool(self._enable_early_termination)), max_episode_length=int(self._max_episode_length),
            est_nx=int(self._est_x.shape[1]) if self._est_x is not None else 0, est_ny=int(self._est_y.shape[1]) if self._est_y is not None else 0,
            scale_pos=float(scales.get('pos', 5.0)), scale_phase=float(scales.get('phase', 10.0)),
            scale_bounce_pos=float(scales.get('bounce_pos', 0.05)), scale_bounce_time=float(scales.get('bounce_time', 0.1)),
            w_pos=float(weights.get('pos', 1.0 if rtype == 'reach' else 0.0)), w_ball_pos=float(weights.get('ball_pos', 0.0)),
            court_min=self._court_min.tolist(), court_max=self._court_max.tolist(), est_params=self._est_params, dual=0,
            use_history=int(self._use_history))
        # fused step glue: action handling of pre_physics_step as one launch; trajectory roll + step counters inside the post launch
        self._fused_pre = bool(self.cfg.get("b200_fused_glue", True)) and not self.cfg_v2p.get('add_residual_root')
        self._fused_post = bool(self.cfg.get("b200_fused_glue", True))
        self._mvae_actions = f(N, self._num_mvae_action)
        self._res_dof_actions = f(N, max(self._num_res_dof_action, 1)) if self._num_res_dof_action else torch.empty(0, device=dev)
        self._rng_step = torch.zeros(1, device=dev, dtype=torch.long)
        self._rng_done = torch.zeros(1, device=dev, dtype=torch.int32)
        self._pre_cfg = dict(n=N, num_actions=self._num_actions, num_latent=self._num_mvae_action, num_res_dof=self._num_res_dof_action,
                             random_walk_in_recovery=int(bool(self.cfg_v2p.get('random_walk_in_recovery', False))),
                             vae_action_scale=float(self.cfg_v2p.get('vae_action_scale', 1.0)),
                             residual_dof_scale=float(self.cfg_v2p.get('residual_dof_scale', 0.1)), seed=int(self.cfg.get("seed", 10)) * 7919 + 13)

    # ------------------------------------------------------------------ construction (:118-158)
    def create_sim(self):
        env = self.cfg["env"]
        phys = env.get("physics", {})
        pcfg = {"env": dict(numEnvs=self.num_envs, episodeLength=self._max_episode_length, controlFrequencyInv=env.get("controlFrequencyInv", 2),
                            residual_force_scale=phys.get("residual_force_scale", 31.85), is_train=self._is_train,
                            asset=dict(assetFileName=phys.get("assetFileName", "smpl_mesh_humanoid_federer.xml")),
                            plane=dict(staticFriction=1.0, dynamicFriction=1.0, restitution=phys.get("plane_restitution", 0.0)),
                            vid2player=dict(self.cfg_v2p),
                            keyBodies=[], contactBodies=[]),
                "sim": {"substeps": phys.get("substeps", 2)}, "b200_physics": self.cfg.get("b200_physics", {})}
        cls = HumanoidSMPLIMMVAEDual if self.cfg_v2p.get('dual_mode') else HumanoidSMPLIMMVAE
        task = cls(pcfg, self._sim_params, self._physics_engine, "cuda", self.device_id, True)
        policy = env.get("low_level_policy", None)
        if policy is None:
            zeros = torch.zeros(self.num_envs, task.num_actions, device=self.device)
            policy = lambda obs: zeros  # noqa: E731  (zero residual: PD targets = kinematic targets)
        elif policy == "b200nn":     # the reference's actor shape (734 -> 1024 -> 1024 -> 512 -> 75, ReLU) with random weights, as
            from .. import nn        # wgmma layers; obs clamp and action clamp of run_one_step are folded into its first / last launch
            policy = nn.PolicyMLP.random(self.num_envs, self.device, in_dim=task.num_obs, out_dim=task.num_actions,
                                         seed=self.cfg.get("seed", 10), clamp_obs=5.0, clamp_actions=1.0,
                                         out_gain=float(env.get("low_level_policy_gain", 0.1)))
        self._low_level_policy = policy
        fused = getattr(policy, "clamp_obs", None) == 5.0 and getattr(policy, "clamp_actions", None) == 1.0 and hasattr(policy, "forward_prepared")
        if fused:     # the obs kernel writes the policy's normalised / clamped bf16 operand row itself: no cast launch
            task._obs_operand = (policy.x, policy.mean, policy.rstd, policy.clamp_obs)

        def run_one_step():   # ImitatorPlayer.run_one_step (players/im_player.py:187-202)
            # The reference clamps the raw observation to env.clip_obs, which player_builder.py:40 reads from `clip_observations`
            # (default inf; no imitation config sets it): the only observation clamp is the policy's own, after its running-mean-std
            # normalisation.  Both branches give the policy the raw observation.
            with torch.no_grad():
                if fused:
                    task.step(self._low_level_policy.forward_prepared())
                else:
                    action = self._low_level_policy(task.obs_buf)
                    task.step(torch.clamp(action, -1.0, 1.0))
        self._physics_player = SimpleNamespace(task=task, run_one_step=run_one_step)
        player = env.get("motion_player", None)
        pk = dict(seed=self.cfg.get("seed", 10), court_min=self.cfg_v2p.get('court_min', [-5, -16]), court_max=self.cfg_v2p.get('court_max', [5, -10]))
        if player == "stream":       # resident target stream (SURVEY.md 8d)
            player = StreamMotionPlayer(self.num_envs, self.device, **pk)
        elif player == "stream+decoder":   # + the MVAE mixture-of-experts decoder forward every step (the bench's choice)
            player = DecoderStreamPlayer(self.num_envs, self.device, **pk)
        if player is None:
            player = SyntheticMotionPlayer(self.num_envs, self.device, seed=self.cfg.get("seed", 10),
                                           court_min=self.cfg_v2p.get('court_min', [-5, -16]), court_max=self.cfg_v2p.get('court_max', [5, -10]))
        self._mvae_player = player
        task._mvae_player = player
        task._controller = self

    def get_action_size(self):
        return self._num_actions

    def get_actor_obs_size(self):
        return self._num_actor_obs

    def get_task_obs_size(self):
        return self._num_task_obs

    # ------------------------------------------------------------------ reset (:167-245)
    def reset(self, env_ids=None):
        if env_ids is None:
            if self._has_init and self.num_envs > 1:
                return
            env_ids = torch.arange(self.num_envs, device=self.device, dtype=torch.long)
        if not self._reset_via_graph(env_ids):
            self._reset_envs(env_ids)

    def _reset_via_graph(self, env_ids):
        """graph mode (enable_cuda_graph): the id list only fills a mask (2 launches), everything else is one replay of the reset graph"""
        if getattr(self, "_reset_graph", None) is None:
            return False
        self._reset_mask.zero_()
        if len(env_ids) > 0:
            self._reset_mask.index_fill_(0, env_ids.to(self.device, dtype=torch.long), True)
        self._reset_graph.replay()
        self._has_init = True
        return True

    def reset_done(self):
        """Addition: `reset(reset_buf.nonzero())` without the id list - the mask of the finished envs is taken from the device
        flags and the whole reset is one replay of the reset graph: no host synchronisation between steps.  Needs enable_cuda_graph()."""
        if getattr(self, "_reset_graph", None) is None:
            self.reset(self.reset_buf.nonzero(as_tuple=False).flatten())
            return
        torch.ne(self.reset_buf, 0, out=self._reset_mask)
        self._reset_graph.replay()
        self._has_init = True

    def _reset_tasks_fast(self, update_state=False, humanoid_mask=None):
        """_reset_envs (:173-201) when no humanoid needs a reset - the common per-step case: new balls for the envs whose reaction
        timer expired, recovery / reaction task bookkeeping, obs refresh.  Mask-driven: 4 RNG launches + 2 kernels, no host sync."""
        N, dev, t = self.num_envs, self.device, self._physics_player.task
        P = int(t._ball_pool.shape[0])
        mode = self.cfg_v2p.get('use_random_ball_target')
        tm = 1 if mode == 'continuous' else (2 if mode else 0)
        seed = torch.rand(3 if tm == 1 else (N if tm == 2 else 1), device=dev)
        cfg = dict(n=N, pool_size=P, ball_stride=26, bodies_per_env=26, reaction_nframes=int(self.cfg_v2p.get('reset_reaction_nframes', 70)),
                   obs_traj_len=self._obs_ball_traj_length, target_mode=tm, target_min=self._target_bounce_min.tolist() if not hasattr(self, "_tmin") else self._tmin,
                   target_max=self._target_bounce_max.tolist() if not hasattr(self, "_tmax") else self._tmax)
        self._tmin, self._tmax = cfg["target_min"], cfg["target_max"]
        native_v2p.task_reset(cfg, dict(
            reset_reaction=self._reset_reaction_buf, reset_recovery=self._reset_recovery_buf,
            pool_rand=torch.randint(0, P, (N,), device=dev), side_rand=torch.randint(-1000, 1000, (N,), device=dev),
            frame_rand=torch.randint(-5, 5, (N,), device=dev), target_seed=seed, pool=t._ball_pool, ball_states=t._root_states[1:],
            rigid_body_state=t._rigid_body_state, ball_pos=t._ball_pos, ball_vel=t._ball_vel, bounce_pos=t._bounce_pos,
            ball_traj=self._ball_traj, est_bounce_pos=self._est_bounce_pos, est_bounce_time=self._est_bounce_time,
            est_max_height=self._est_max_height, target_bounce_pos=self._target_bounce_pos, has_bounce=t._has_bounce,
            has_contact=t._has_racket_ball_contact, bounce_in=self._bounce_in, est_bounce_in=self._est_bounce_in, tar_time=self._tar_time,
            tar_time_total=self._tar_time_total, tar_action=self._tar_action, num_reset_reaction=self._num_reset_reaction,
            swing_type_cycle=self._mvae_player._swing_type_cycle, ball_obs=self._ball_obs if self._use_history else None))
        if update_state:
            self._physics_player.task._update_state_from_sim(only_mask=humanoid_mask)   # :186-187 "setting the right fields to compute obs"
        post = dict(self._post_cfg)
        post["obs_only"] = 1
        t = self._tensors()
        if humanoid_mask is not None:
            t["touch_mask"] = humanoid_mask
        native_v2p.controller_post(post, t)

    def _reset_envs(self, env_ids):
        """:173-201.  Humanoid part (id list from the agent): motion generator reset, FK pose -> sim state (2 launches), counters.
        Task part (device masks, sampled BEFORE they are cleared like the reference's id lists): balls, recovery / reaction
        bookkeeping, obs refresh.  No nonzero() / host sync inside."""
        task = self._physics_player.task
        n = len(env_ids)
        if n > 0:
            env_ids = env_ids.to(self.device, dtype=torch.long).contiguous()
            self._mvae_player.reset(env_ids)
            task._reset_actors(env_ids)
            for buf in (self.progress_buf, self.reset_buf, self._terminate_buf, self._num_reset_reaction):
                buf.index_fill_(0, env_ids, 0)
            self._distance.index_fill_(0, env_ids, 0.0)
            self._num_reset.index_add_(0, env_ids, torch.ones_like(env_ids))
        self._reset_tasks_fast(update_state=n > 0)
        if n > 0:
            self._reset_reaction_buf.index_fill_(0, env_ids, False)
            self._reset_recovery_buf.index_fill_(0, env_ids, False)
        self._has_init = True

    def _reset_envs_masked(self, mask):
        """_reset_envs (:173-201) driven by a device mask of the humanoids to reset instead of an id list: mask-aware kernels only, no
        host synchronisation - `enable_cuda_graph` captures it as the reset graph.  Kernels of the humanoid part skip the envs whose
        mask is clear, so a replay in which nobody finished costs little more than its launches."""
        task = self._physics_player.task
        self._mvae_player.reset_masked(mask)
        task._reset_actors_masked(mask)
        native_v2p.ctrl_reset(mask, self.progress_buf, self.reset_buf, self._terminate_buf, self._num_reset_reaction, self._distance, self._num_reset)
        self._reset_tasks_fast(update_state=True, humanoid_mask=mask)      # also clears the task flags of the reset humanoids at its end
        self._has_init = True

    def _reset_envs_idlist(self, env_ids):
        """The same reset written like the reference (nonzero() id lists + indexed torch ops, :173-201).  Kept as the
        executable specification the mask-driven kernels are tested against (tests/test_gpu_v2p.py); not used on the hot path."""
        task = self._physics_player.task
        reaction_ids = self._reset_reaction_buf.nonzero(as_tuple=False).flatten()
        recovery_ids = self._reset_recovery_buf.nonzero(as_tuple=False).flatten()
        all_ids = (self._reset_reaction_buf | self._reset_recovery_buf).nonzero(as_tuple=False).flatten()
        if len(env_ids) > 0:
            self.progress_buf[env_ids] = 0
            self.reset_buf[env_ids] = 0
            self._terminate_buf[env_ids] = 0
            self._reset_reaction_buf[env_ids] = False
            self._reset_recovery_buf[env_ids] = False
            self._num_reset_reaction[env_ids] = 0
            self._distance[env_ids] = 0
            self._mvae_player.reset(env_ids)
            self._num_reset[env_ids] += 1
        if len(env_ids) > 0 or len(reaction_ids) > 0:
            traj = task.reset(env_ids, reaction_ids)
            if traj is not None and not self._use_history:      # :187-188
                self._ball_traj[reaction_ids] = traj
        if len(env_ids) > 0:
            task._update_state_from_sim()
        if len(recovery_ids) > 0:
            self._tar_action[recovery_ids] = 0
            task._has_bounce[recovery_ids] = False
            task._bounce_pos[recovery_ids] = 0
        if len(reaction_ids) > 0:
            self._reset_reaction_tasks(reaction_ids)
        if len(all_ids) > 0:
            self._compute_observations()
        self._has_init = True

    def _reset_reaction_tasks(self, env_ids):
        """:203-240"""
        if self._use_history:                                   # :213-214
            self._ball_obs[env_ids] = self._physics_player.task._ball_pos[env_ids].view(-1, 1, 3).repeat(1, self._obs_ball_traj_length, 1)
        self._tar_time[env_ids] = 0
        self._tar_action[env_ids] = 1
        self._num_reset_reaction[env_ids] += 1
        self._bounce_in[env_ids] = False
        self._est_bounce_pos[env_ids] = 0
        self._est_bounce_time[env_ids] = 0
        self._est_bounce_in[env_ids] = False
        self._est_max_height[env_ids] = 0
        self._mvae_player._swing_type_cycle[env_ids] = -1
        self._tar_time_total[env_ids] = self.cfg_v2p.get('reset_reaction_nframes', 70) + torch.randint(-5, 5, (len(env_ids),), device=self.device)
        mode = self.cfg_v2p.get('use_random_ball_target')
        if mode == 'continuous':
            self._target_bounce_pos[env_ids] = torch.rand((3,), device=self.device) * (self._target_bounce_max - self._target_bounce_min) + self._target_bounce_min
        elif mode:
            seed = torch.rand(len(env_ids), device=self.device)
            x = torch.where(seed < 0.33, -3.0, torch.where(seed > 0.67, 3.0, 0.0))
            self._target_bounce_pos[env_ids, 0], self._target_bounce_pos[env_ids, 1], self._target_bounce_pos[env_ids, 2] = x, 10.0, 0.0

    # ------------------------------------------------------------------ step (:247-269, 362-366, 441-459)
    def pre_physics_step(self, actions):
        if self._fused_pre:
            # one launch: latent scaling, random walk in recovery (counter-based normals), residual-dof scaling (b200v2p_pre_step)
            self._actions = actions
            native_v2p.pre_step(self._pre_cfg, dict(actions=actions, tar_action=self._tar_action, step_counter=self._rng_step,
                                                    done_counter=self._rng_done, mvae_actions=self._mvae_actions,
                                                    res_dof_actions=self._res_dof_actions if self._num_res_dof_action else None))
            self._mvae_player.step(self._mvae_actions, self._res_dof_actions)
            self._physics_player.task.post_mvae_step()
            return
        self._actions = actions.clone()
        na = self._num_mvae_action
        self._mvae_actions = actions[:, :na].clone() * self.cfg_v2p.get('vae_action_scale', 1.0)
        if self.cfg_v2p.get('random_walk_in_recovery', False):
            in_rec = self._tar_action == 0
            rnd = torch.clamp(torch.randn_like(self._mvae_actions), -5, 5)
            self._mvae_actions = torch.where(in_rec[:, None], rnd, self._mvae_actions)
        self._res_dof_actions = torch.empty(0, device=self.device)
        if self.cfg_v2p.get('add_residual_dof'):
            self._res_dof_actions = actions[:, na:na + self._num_res_dof_action].clone() * self.cfg_v2p.get('residual_dof_scale', 0.1)
        self._mvae_player.step(self._mvae_actions, self._res_dof_actions)
        if self.cfg_v2p.get('add_residual_root'):
            o = na + self._num_res_dof_action
            self._res_root_actions = actions[:, o:o + 3].clone() * self.cfg_v2p.get('residual_root_scale', 0.02)
        self._physics_player.task.post_mvae_step()

    def physics_step(self):
        self._physics_player.run_one_step()
        if not self._fused_post:
            self._ball_traj.copy_(self._ball_traj.roll(-1, dims=1))   # in place: persistent state keeps its address (CUDA-graph safe)
            self._ball_traj[:, -1] = 0

    def post_physics_step(self):
        if not self._fused_post:
            self._tar_time += 1
            self.progress_buf += 1
        self._compute_post(advance=self._fused_post)
        self.extras["terminate"] = self._terminate_buf
        self.extras["sub_rewards"] = self._sub_rewards
        self.extras["sub_rewards_names"] = self._sub_rewards_names

    def _tensors(self):
        t, p = self._physics_player.task, self._mvae_player
        return dict(rigid_body_state=t._rigid_body_state, ball_states=t._root_states[1:], root_pos=t._root_pos, root_vel=t._root_vel,
                    racket_pos=t._racket_pos, racket_normal=t._racket_normal, ball_pos=t._ball_pos, has_contact=t._has_racket_ball_contact,
                    has_contact_now=t._has_racket_ball_contact_now, has_bounce=t._has_bounce, has_bounce_now=t._has_bounce_now,
                    bounce_pos=t._bounce_pos, ball_traj=self._ball_traj.contiguous(), target_bounce_pos=self._target_bounce_pos,
                    phase=p._phase_pred.contiguous(), swing_type=p._swing_type.contiguous(), swing_type_cycle=p._swing_type_cycle.contiguous(),
                    tar_action=self._tar_action, tar_time=self._tar_time, tar_time_total=self._tar_time_total, progress_buf=self.progress_buf,
                    est_x=self._est_x, est_y=self._est_y, bounce_in=self._bounce_in, est_bounce_in=self._est_bounce_in,
                    reset_reaction=self._reset_reaction_buf, reset_recovery=self._reset_recovery_buf, est_bounce_pos=self._est_bounce_pos,
                    est_bounce_time=self._est_bounce_time, est_max_height=self._est_max_height, distance=self._distance, obs_buf=self.obs_buf,
                    rew_buf=self.rew_buf, sub_rewards=self._sub_rewards, reset_buf=self.reset_buf, terminate_buf=self._terminate_buf,
                    ball_obs=self._ball_obs)

    def _compute_post(self, advance=False):
        """_update_state + _compute_reward + _compute_observations + _compute_reset as ONE launch (:271-436); advance: the launch first
        rolls the ball-trajectory window and counts tar_time / progress_buf (tail of physics_step + head of post_physics_step)"""
        self._ball_traj = self._ball_traj.contiguous()
        cfg = self._post_cfg
        if advance:
            cfg = dict(cfg)
            cfg["advance"] = 1
        native_v2p.controller_post(cfg, self._tensors())
        t = self._physics_player.task
        self._root_pos, self._root_vel, self._racket_pos, self._racket_vel, self._racket_normal = t._root_pos, t._root_vel, t._racket_pos, t._racket_vel, t._racket_normal
        self._ball_pos, self._ball_vel, self._ball_vspin = t._ball_pos, t._ball_vel, t._ball_vspin
        self._phase_pred = self._mvae_player._phase_pred
        if not self._is_train:
            self._joint_rot = t._joint_rot          # :274-275

    def _compute_observations(self, env_ids=None):
        """used on reset: the observation rows are refreshed by the same kernel (reward / reset flags of a reset env are rewritten
        by the next step before anyone reads them)"""
        keep = (self.rew_buf.clone(), self.reset_buf.clone(), self._terminate_buf.clone(), self._reset_reaction_buf.clone(),
                self._reset_recovery_buf.clone(), self._distance.clone(), self._sub_rewards.clone())
        self._compute_post()
        self.rew_buf.copy_(keep[0]); self.reset_buf.copy_(keep[1]); self._terminate_buf.copy_(keep[2])
        self._reset_reaction_buf.copy_(keep[3]); self._reset_recovery_buf.copy_(keep[4]); self._distance.copy_(keep[5])
        self._sub_rewards.copy_(keep[6])

    def step(self, actions):
        if self._graph is not None:
            self._graph_actions.copy_(actions)
            self._graph.replay()
            return
        self.pre_physics_step(actions.to(self.device, dtype=torch.float).contiguous())
        self.physics_step()
        self.post_physics_step()

    def enable_cuda_graph(self, warmup=3, count_nodes=False):
        """Capture one whole high-level step (motion generator + FK targets + obs + low-level policy + fused physics + fused
        post step: ~70 launches) into a CUDA graph; afterwards `step()` = one copy + one graph launch.  Requirements: the motion
        player and the low-level policy update their state in place and make no host synchronisation (true for the synthetic
        player and for plain nn.Module policies); `reset()` stays eager between replays (it edits the same buffers in place)."""
        assert self._graph is None
        self._graph_actions = torch.zeros(self.num_envs, self.num_actions, device=self.device)
        s = torch.cuda.Stream(device=self.device)
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            for _ in range(warmup):
                self.pre_physics_step(self._graph_actions)
                self.physics_step()
                self.post_physics_step()
        torch.cuda.current_stream().wait_stream(s)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            self.pre_physics_step(self._graph_actions)
            self.physics_step()
            self.post_physics_step()
        self._graph = g
        self.graph_kernel_nodes = self.reset_graph_kernel_nodes = None
        if hasattr(self._mvae_player, "reset_masked"):
            # second graph: the whole env reset, mask-driven (needs a graph-safe motion player)
            self._reset_mask = torch.zeros(self.num_envs, device=self.device, dtype=torch.bool)
            with torch.cuda.stream(s):
                self._reset_envs_masked(self._reset_mask)          # warm-up with an all-false humanoid mask: only the task masks act
            torch.cuda.current_stream().wait_stream(s)
            torch.cuda.synchronize()
            rg = torch.cuda.CUDAGraph()
            with torch.cuda.graph(rg):
                self._reset_envs_masked(self._reset_mask)
            self._reset_graph = rg
        if count_nodes:      # measurement aid (bench `gpu_launches`): the same launch sequences run eagerly once under the CUDA profiler
            def step_once():
                self.pre_physics_step(self._graph_actions)
                self.physics_step()
                self.post_physics_step()
            self.graph_kernel_nodes = self._count_kernels(step_once)
            if getattr(self, "_reset_graph", None) is not None:
                self._reset_mask.zero_()
                self.reset_graph_kernel_nodes = self._count_kernels(lambda: self._reset_envs_masked(self._reset_mask))

    @staticmethod
    def _count_kernels(fn):
        """number of kernels `fn` launches (CUPTI through torch.profiler; memcpy / memset activities are not counted)"""
        try:
            from torch.profiler import ProfilerActivity, profile
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                fn()
                torch.cuda.synchronize()
            n = 0
            for e in prof.events():
                if str(getattr(e, "device_type", "")).endswith("CUDA") and not any(t in e.name for t in ("Memcpy", "Memset", "memcpy", "memset")):
                    n += 1
            return n or None
        except Exception:
            return None

    def get_aux_losses(self, model_res_dict):
        """:461-472 (autograd-carrying, PyTorch)"""
        specs = self.cfg_v2p.get('aux_loss_specs', dict())
        dof_res = model_res_dict['mus'][:, self._num_mvae_action:self._num_mvae_action + self._num_res_dof_action]
        loss = (dof_res ** 2).sum(dim=-1).mean()
        return {'aux_dof_res_loss': loss}, {'aux_dof_res_loss': specs.get('dof_res', 0) * loss}

    def register_model(self, model):
        self.model = model

    def pre_epoch(self, epoch):
        self._epoch_num = epoch

    def render_vis(self):
        return


class PhysicsMVAEControllerDual(PhysicsMVAEController):
    """vid2player/env/tasks/physics_mvae_controller_dual.py: two players per rally in paired envs (2k, 2k+1).  The step is the
    base class's (motion generator, FK targets, obs, policy, physics launch per asset, fused post step) with the dual reset FSM
    selected in the post-step kernel; the reset below follows the reference's id lists (:27-64)."""

    def __init__(self, cfg, sim_params, physics_engine, device_type, device_id, headless):
        if cfg["env"]["numEnvs"] % 2:
            raise ValueError("dual mode needs an even number of envs")
        cfg["env"]["vid2player"].setdefault('dual_mode', True)
        super().__init__(cfg=cfg, sim_params=sim_params, physics_engine=physics_engine, device_type=device_type, device_id=device_id,
                         headless=headless)
        self._reset_reaction_buf[:] = False
        self._reset_recovery_buf[:] = False
        self._post_cfg["dual"] = 1

    def reset(self, env_ids=None):
        if env_ids is None:
            if self._has_init:
                return
            env_ids = torch.arange(self.num_envs, device=self.device, dtype=torch.long)
        if not self._reset_via_graph(env_ids):
            self._reset_envs(env_ids)

    def _reset_envs_masked(self, mask):
        """_reset_envs (:27-64) driven by a device mask of the humanoids to reset (both players of a pair set) instead of id lists:
        full-width in-place ops and mask-aware kernels, no host synchronisation (captured as the reset graph).  Same order of
        effects as the id-list form below: serve, then the ball hand-over through the incoming-ball table, then the task fields."""
        task, N, dev = self._physics_player.task, self.num_envs, self.device
        if not hasattr(self, "_near"):
            ar = torch.arange(N, device=dev)
            self._near = (ar % 2) == (0 if self.cfg_v2p.get('serve_from', 'near') == 'near' else 1)
            self._opp = (ar ^ 1).contiguous()
        reaction_actor, recovery_actor = mask & self._near, mask & ~self._near
        self._reset_reaction_buf.logical_or_(reaction_actor)
        self._reset_recovery_buf.logical_or_(recovery_actor)
        R, Cm = self._reset_reaction_buf.clone(), self._reset_recovery_buf.clone()     # the id lists of the reference, as masks
        self._mvae_player.reset_masked(mask)
        if hasattr(self._mvae_player, "_swing_type"):
            self._mvae_player._swing_type.masked_fill_(mask, -1)                       # reset_dual
        for buf in (self.progress_buf, self.reset_buf, self._terminate_buf, self._num_reset_reaction):      # _reset_env_tensors
            buf.masked_fill_(mask, 0)
        self._reset_reaction_buf.masked_fill_(mask, False)
        self._reset_recovery_buf.masked_fill_(mask, False)
        self._distance.masked_fill_(mask, 0.0)
        task._reset_actors_masked(mask)                                                # task.reset: the pairs' humanoids ...
        traj = task._reset_balls_masked(recovery_actor, R, self._opp)                  # ... serve + hand-over for the reaction envs
        if not self._use_history:
            self._ball_traj[:, :traj.shape[1]] = torch.where(R[:, None, None], traj, self._ball_traj[:, :traj.shape[1]])
        self._tar_action.masked_fill_(Cm, 0)                                           # _reset_recovery_tasks
        task._has_bounce.masked_fill_(Cm, False)
        task._bounce_pos.masked_fill_(Cm[:, None], 0.0)
        if self._use_history:                                                          # _reset_reaction_tasks
            self._ball_obs.copy_(torch.where(R[:, None, None], task._ball_pos[:, None, :].expand(-1, self._obs_ball_traj_length, -1), self._ball_obs))
        self._tar_time.masked_fill_(R, 0)
        self._tar_action.masked_fill_(R, 1)
        self._num_reset_reaction.add_(R.to(torch.long))
        self._bounce_in.masked_fill_(R, False)
        if self.cfg_v2p.get('use_random_ball_target'):
            seed = torch.rand(N, device=dev)
            x = torch.where(seed < 0.33, -3.0, torch.where(seed > 0.67, 3.0, 0.0))
            tgt = torch.stack([x, torch.full_like(x, 10.0), torch.zeros_like(x)], -1)
            self._target_bounce_pos.copy_(torch.where(R[:, None], tgt, self._target_bounce_pos))
        if self.cfg_v2p.get('reward_type') == 'return_w_estimate':
            self._est_bounce_pos.masked_fill_(R[:, None], 0.0)
            self._est_bounce_time.masked_fill_(R, 0.0)
            self._est_bounce_in.masked_fill_(R, False)
            self._est_max_height.masked_fill_(R, 0.0)
        post = dict(self._post_cfg)
        post["obs_only"] = 1
        native_v2p.controller_post(post, self._tensors())
        self._has_init = True

    def _reset_env_tensors(self, env_ids):
        """physics_mvae_controller.py:203-210"""
        for buf in (self.progress_buf, self.reset_buf, self._terminate_buf, self._num_reset_reaction):
            buf[env_ids] = 0
        self._reset_reaction_buf[env_ids] = False
        self._reset_recovery_buf[env_ids] = False
        self._distance[env_ids] = 0

    def _reset_envs(self, env_ids):
        """:27-64"""
        task = self._physics_player.task
        env_ids = env_ids.to(self.device, dtype=torch.long)
        empty = torch.zeros(0, device=self.device, dtype=torch.long)
        if len(env_ids) > 0:
            assert len(env_ids) % 2 == 0, len(env_ids)
            reaction_actor = env_ids[::2] if self.cfg_v2p.get('serve_from', 'near') == 'near' else env_ids[1::2]
            recovery_actor = get_opponent_env_ids(reaction_actor)
            self._reset_reaction_buf[reaction_actor] = True
            self._reset_recovery_buf[recovery_actor] = True
        else:
            reaction_actor = recovery_actor = empty
        reaction_ids = self._reset_reaction_buf.nonzero(as_tuple=False).flatten()
        recovery_ids = self._reset_recovery_buf.nonzero(as_tuple=False).flatten()
        if len(env_ids) > 0:
            self._mvae_player.reset_dual(reaction_actor, recovery_actor)
            self._reset_env_tensors(env_ids)
        if len(reaction_ids) > 0:
            new_traj = task.reset(reaction_actor, reaction_ids)
            if not self._use_history:
                self._ball_traj[reaction_ids, :new_traj.shape[1]] = new_traj
            # self._update_state() (:52) re-derives bounce_in from unchanged inputs: nothing to do on the device
        if len(recovery_ids) > 0:
            self._reset_recovery_tasks(recovery_ids)
        if len(reaction_ids) > 0:
            self._reset_reaction_tasks(reaction_ids)
            post = dict(self._post_cfg)
            post["obs_only"] = 1
            native_v2p.controller_post(post, self._tensors())
        self._has_init = True

    def _reset_reaction_tasks(self, env_ids):
        """:66-85"""
        if self._use_history:                                   # :69-70
            self._ball_obs[env_ids] = self._physics_player.task._ball_pos[env_ids].view(-1, 1, 3).repeat(1, self._obs_ball_traj_length, 1)
        self._tar_time[env_ids] = 0
        self._tar_action[env_ids] = 1
        self._num_reset_reaction[env_ids] += 1
        self._bounce_in[env_ids] = False
        if self.cfg_v2p.get('use_random_ball_target'):
            seed = torch.rand(len(env_ids), device=self.device)
            x = torch.where(seed < 0.33, -3.0, torch.where(seed > 0.67, 3.0, 0.0))
            self._target_bounce_pos[env_ids] = torch.stack([x, torch.full_like(x, 10.0), torch.zeros_like(x)], -1)
        if self.cfg_v2p.get('reward_type') == 'return_w_estimate':
            self._est_bounce_pos[env_ids] = 0
            self._est_bounce_time[env_ids] = 0
            self._est_bounce_in[env_ids] = False
            self._est_max_height[env_ids] = 0

    def _reset_recovery_tasks(self, env_ids):
        """:87-90"""
        self._tar_action[env_ids] = 0
        self._physics_player.task._has_bounce[env_ids] = False
        self._physics_player.task._bounce_pos[env_ids] = 0
