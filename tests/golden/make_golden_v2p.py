"""Golden fixtures for the vid2player rows (SURVEY.md 8a: a10-a17), produced by EXECUTING the reference's own
code (vid2player/env/tasks/humanoid_smpl_im_mvae.py, physics_mvae_controller.py, utils/tennis_ball*.py) on CPU
through fake `self` objects.  Run in the build container only:  python tests/golden/make_golden_v2p.py

  v2p_smpl_to_sim.npz   _smpl_to_sim / _forward_kinematics (:897-946) incl. finite-difference velocities   (a13)
  v2p_ball.npz          apply_external_force_to_ball (:711-739), _reset_balls (:503-524) + offline pool sampler (a10, a17)
  v2p_update_state.npz  _update_state_from_sim (:799-860)                                                   (a11, a12)
  v2p_dual.npz          dual mode: TennisBallInEstimator.estimate (utils/tennis_ball_in_estimator.py:22-81),
                        HumanoidSMPLIMMVAEDual._reset_balls (humanoid_smpl_im_mvae_dual.py:52-80),
                        PhysicsMVAEControllerDual._compute_reset (physics_mvae_controller_dual.py:92-120)
  v2p_controller.npz    actor/task obs (:333-360), rewards (:493-602), check_out_of_court, _update_state + estimator
                        (:271-314, tennis_ball_out_estimator.py:164-205), _compute_reset (:408-436)          (a14-a16)
  v2p_task_reset.npz    TennisBallGeneratorOffline.generate with start_pos (tennis_ball.py:436-444), the controller's
                        _reset_recovery_tasks / _reset_reaction_tasks (physics_mvae_controller.py:203-245), both target modes
"""
import os
import sys
from types import SimpleNamespace
from unittest.mock import MagicMock

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
import _refenv  # noqa: E402

_refenv.setup("vid2player")

from env.tasks import humanoid_smpl_im_mvae as M  # noqa: E402
from env.tasks import physics_mvae_controller as C  # noqa: E402
from utils import tennis_ball_out_estimator as E  # noqa: E402
from utils.tennis_ball import TennisBallGeneratorOffline  # noqa: E402
from utils.konia_transform import angle_axis_to_rotation_matrix  # noqa: E402

from vid2player3d_b200 import model_compiler  # noqa: E402

torch.set_num_threads(1)

SMPL_NAMES = ["Pelvis", "L_Hip", "R_Hip", "Torso", "L_Knee", "R_Knee", "Spine", "L_Ankle", "R_Ankle", "Chest", "L_Toe", "R_Toe",
              "Neck", "L_Thorax", "R_Thorax", "Head", "L_Shoulder", "R_Shoulder", "L_Elbow", "R_Elbow", "L_Wrist", "R_Wrist",
              "L_Hand", "R_Hand"]
SMPL_PARENTS = [-1, 0, 0, 0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 9, 9, 12, 13, 14, 16, 17, 18, 19, 20, 21]


def npz(name, **kw):
    out = {k: (v.detach().cpu().numpy() if isinstance(v, torch.Tensor) else np.asarray(v)) for k, v in kw.items()}
    np.savez_compressed(os.path.join(HERE, name), **out)
    print(name, {k: v.shape for k, v in out.items()})


def rq(g, *s):
    q = torch.randn(*s, 4, generator=g)
    return q / q.norm(dim=-1, keepdim=True)


class FakePlayer(M.HumanoidSMPLIMMVAE):
    def __init__(self):
        pass


class FakeController(C.PhysicsMVAEController):
    def __init__(self):
        pass


def rest_joints_smpl_order():
    """rest joint positions (SMPL joint order) of the shipped federer skeleton: cumulative MJCF offsets"""
    m = model_compiler.load_compiled("smpl_mesh_humanoid_federer")
    names = [str(x) for x in m["body_names"]][:24]
    pos = np.zeros((24, 3))
    for i in range(24):
        pos[i] = m["offset"][i] + (pos[m["parent"][i]] if m["parent"][i] >= 0 else 0)
    return torch.tensor(np.stack([pos[names.index(n)] for n in SMPL_NAMES]), dtype=torch.float32)


def smpl_to_sim():
    g = torch.Generator().manual_seed(21)
    N = 48
    t = FakePlayer()
    t.device = 'cpu'
    t.dt = 2 * (1.0 / 60.0)
    t._build_mujoco_smpl_transform()
    rest = rest_joints_smpl_order()
    t._smpl = SimpleNamespace(joint_pos_bind=rest.unsqueeze(0).repeat(N, 1, 1), parents=torch.tensor(SMPL_PARENTS))
    aa0 = 0.6 * torch.randn(N, 24, 3, generator=g)
    aa0[0] = 0                                  # identity rotations (trace = 3 branch, tiny angles)
    aa0[1, 5] = torch.tensor([3.1, 0.0, 0.0])   # near-pi rotation (negative-trace branches)
    aa0[2, 7] = torch.tensor([0.0, 3.0, 0.5])
    aa0[3, 9] = torch.tensor([0.1, 0.2, 3.05])
    aa1 = aa0 + 0.05 * torch.randn(N, 24, 3, generator=g)
    rm0 = angle_axis_to_rotation_matrix(aa0.view(-1, 3)).view(N, 24, 3, 3)
    rm1 = angle_axis_to_rotation_matrix(aa1.view(-1, 3)).view(N, 24, 3, 3)
    root0 = torch.randn(N, 3, generator=g)
    root1 = root0 + 0.02 * torch.randn(N, 3, generator=g)
    o0 = t._smpl_to_sim(root0.clone(), rm0)
    o1 = t._smpl_to_sim(root1.clone(), rm1, prev_root_pos=o0[0], prev_rb_rot=o0[7])
    names = ("root_pos", "root_rot", "dof_pos", "root_vel", "root_ang_vel", "dof_vel", "rb_pos", "rb_rot")
    npz("v2p_smpl_to_sim.npz", rest=rest, parents=np.array(SMPL_PARENTS), smpl_2_mujoco=np.array(t._smpl_2_mujoco),
        rotmat0=rm0, rotmat1=rm1, root0=root0, root1=root1, dt=np.array(t.dt),
        **{"a_" + k: v for k, v in zip(names, o0)}, **{"b_" + k: v for k, v in zip(names, o1)})


def ball():
    g = torch.Generator().manual_seed(22)
    N = 64
    out = {}
    for substeps in (2, 6):
        t = FakePlayer()
        t.device = 'cpu'
        t.num_envs = N
        t.cfg_v2p = {'spin_scale': 5.0}
        t.cfg = {'sim': {'substeps': substeps}}
        bs = torch.zeros(N, 13)
        bs[:, 0:3] = torch.randn(N, 3, generator=g) * torch.tensor([3.0, 8.0, 0.0]) + torch.tensor([0, 0, 0.0])
        bs[:, 2] = torch.rand(N, generator=g) * 0.5
        bs[:, 6] = 1
        bs[:, 7:10] = torch.randn(N, 3, generator=g) * torch.tensor([3.0, 20.0, 4.0])
        bs[:, 10:13] = torch.randn(N, 3, generator=g) * 40
        bs[0, 7:10] = 0          # zero velocity: divide-by-zero guard
        bs[1, 10:13] = 0         # zero spin: lift sign branch
        t._has_bounce = torch.zeros(N, dtype=torch.bool)
        t._has_bounce[::5] = True
        t._has_bounce_now = torch.zeros(N, dtype=torch.bool)
        t._bounce_pos = torch.zeros(N, 3)
        t.forces = torch.zeros(N, 26, 3)
        hb0 = t._has_bounce.clone()
        t.apply_external_force_to_ball(bs)
        out.update({f"s{substeps}_ball_states": bs, f"s{substeps}_has_bounce_in": hb0, f"s{substeps}_force": t.forces[:, -1].clone(),
                    f"s{substeps}_has_bounce": t._has_bounce.clone(), f"s{substeps}_has_bounce_now": t._has_bounce_now.clone(),
                    f"s{substeps}_bounce_pos": t._bounce_pos.clone()})
    # ball reset from the offline pool (sample_random=False path is deterministic: sample_idx per env)
    P = 50
    rng = np.random.default_rng(3)
    pool = np.zeros((P, 307), np.float32)
    pool[:, 0:3] = rng.uniform([-4, 12, 1], [4, 13, 1.5], (P, 3))
    pool[:, 3:6] = rng.normal(0, 1, (P, 3)) * [2, 3, 2] + [0, -25, 3]
    pool[:, 6] = rng.uniform(5, 10, P)
    pool[:, 7:] = rng.normal(0, 5, (P, 300))
    pool[3, 3:6] = [0, 0, -9.0]  # velocity parallel to -z: cross product is zero -> F.normalize eps branch
    path = os.path.join("/tmp", "v2p_pool.npy")
    np.save(path, pool)
    t = FakePlayer()
    t.device = 'cpu'
    t._ball_generator = TennisBallGeneratorOffline(traj_file=path, sample_random=False, num_envs=N)
    t._ball_generator.sample_idx[:] = torch.arange(N) % P
    t._ball_root_states = torch.zeros(N, 13)
    t._ball_pos, t._ball_vel = torch.zeros(N, 3), torch.zeros(N, 3)
    t._has_bounce = torch.ones(N, dtype=torch.bool)
    t._bounce_pos = torch.ones(N, 3)
    t._has_racket_ball_contact = torch.ones(N, dtype=torch.bool)
    ids = torch.tensor([0, 3, 5, 17, 40, 63])
    traj = t._reset_balls(ids)
    out.update(pool=pool, reset_ids=ids, reset_pool_index=(ids % P), reset_traj=traj, reset_ball_states=t._ball_root_states.clone(),
               reset_has_bounce=t._has_bounce.clone(), reset_contact=t._has_racket_ball_contact.clone(),
               reset_bounce_pos=t._bounce_pos.clone())
    npz("v2p_ball.npz", **out)


def update_state():
    g = torch.Generator().manual_seed(23)
    N = 40
    out = {}
    for grip in ("eastern", "semi_western"):
        t = FakePlayer()
        t.device = 'cpu'
        t.num_envs = N
        t.cfg = {'sim': {'substeps': 6}}
        t.cfg_v2p = {'grip': grip}
        t._is_train = True
        t._lefthand = None
        t._racket_body_id, t._racket_wrist_body_id = 24, 22
        rbs = torch.randn(N, 26, 13, generator=g)
        rbs[..., 3:7] = rq(g, N, 26)
        t._rigid_body_pos, t._rigid_body_rot = rbs[..., 0:3], rbs[..., 3:7]
        t._rigid_body_vel, t._rigid_body_ang_vel = rbs[..., 7:10], rbs[..., 10:13]
        t._humanoid_root_states = torch.randn(N, 13, generator=g)
        t._ball_root_states = torch.randn(N, 13, generator=g) * 8
        t._ball_vel = torch.randn(N, 3, generator=g) * 8   # velocity at the previous control step
        t._has_racket_ball_contact = torch.zeros(N, dtype=torch.bool)
        t._has_racket_ball_contact[::7] = True
        t._has_racket_ball_contact_now = torch.zeros(N, dtype=torch.bool)
        for k in ("_root_pos", "_root_vel", "_racket_pos", "_racket_vel", "_racket_normal", "_ball_pos"):
            setattr(t, k, torch.zeros(N, 3))
        t._ball_vspin = torch.zeros(N)
        inp = dict(rbs=rbs.clone(), root_states=t._humanoid_root_states.clone(), ball_states=t._ball_root_states.clone(),
                   prev_ball_vel=t._ball_vel.clone(), contact_in=t._has_racket_ball_contact.clone())
        t._update_state_from_sim()
        res = dict(root_pos=t._root_pos, root_vel=t._root_vel, racket_pos=t._racket_pos, racket_vel=t._racket_vel,
                   racket_normal=t._racket_normal, ball_pos=t._ball_pos, ball_vel=t._ball_vel, ball_vspin=t._ball_vspin,
                   contact=t._has_racket_ball_contact, contact_now=t._has_racket_ball_contact_now)
        out.update({f"{grip}_{k}": v for k, v in {**inp, **res}.items()})
    npz("v2p_update_state.npz", **out)


class SmallParams:  # same structure as traj_out_params, small grid
    VEL_X_RANGE = (10, 14, 1.0)
    VEL_Y_RANGE = (-5, -2, 1.0)
    VSPIN_RANGE = (-10, -6, 2.0)
    TRAJ_X_RANGE = (0, 30, 0.5)
    TRAJ_Y_RANGE = (0, 3, 0.1)


def controller():
    g = torch.Generator().manual_seed(24)
    N = 64
    player = SimpleNamespace()
    rbs = torch.randn(N, 25, 13, generator=g)   # humanoid 24 + Racket (the ball row is not part of these views)
    rbs[..., 3:7] = rq(g, N, 25)
    player._rigid_body_pos, player._rigid_body_rot = rbs[..., 0:3], rbs[..., 3:7]
    player._root_pos = rbs[:, 0, 0:3].clone()
    player._root_pos[:, :2] = torch.randn(N, 2, generator=g) * torch.tensor([6.0, 9.0])
    player._root_vel = torch.randn(N, 3, generator=g)
    player._racket_pos = rbs[:, 24, 0:3].clone()
    player._racket_vel = torch.randn(N, 3, generator=g)
    player._racket_normal = torch.nn.functional.normalize(torch.randn(N, 3, generator=g), dim=-1)
    player._ball_pos = player._racket_pos + 0.3 * torch.randn(N, 3, generator=g)
    player._ball_pos[:, 1] += torch.randn(N, generator=g) * 2
    player._ball_vel = torch.randn(N, 3, generator=g) * 10
    player._ball_vspin = torch.rand(N, generator=g) * 10
    player._has_racket_ball_contact = torch.rand(N, generator=g) < 0.4
    player._has_racket_ball_contact_now = player._has_racket_ball_contact & (torch.rand(N, generator=g) < 0.7)
    player._has_bounce = torch.rand(N, generator=g) < 0.5
    player._has_bounce_now = player._has_bounce & (torch.rand(N, generator=g) < 0.5)
    player._bounce_pos = torch.randn(N, 3, generator=g) * torch.tensor([4.0, 8.0, 0.0]) + torch.tensor([0.0, 6.0, 0.0])
    bstates = torch.zeros(N, 13)
    bstates[:, 0:3] = torch.randn(N, 3, generator=g) * torch.tensor([2.0, 3.0, 0.3]) + torch.tensor([0.0, -8.0, 1.0])
    bstates[:, 7] = torch.randn(N, generator=g) * 2
    bstates[:, 8] = torch.rand(N, generator=g) * 8 + 8      # some below the 10 m/s validity threshold
    bstates[:, 9] = torch.randn(N, generator=g) * 3 - 2
    bstates[:, 10:13] = torch.randn(N, 3, generator=g) * 20
    player._ball_root_states = bstates

    c = FakeController()
    c.device = 'cpu'
    c.num_envs = N
    c.cfg = {'env': {'enableEarlyTermination': True}}
    c.cfg_v2p = {'obs_ball_traj_length': 10, 'use_random_ball_target': True, 'reward_type': 'return_w_estimate',
                 'reward_weights': {'pos': 0.5, 'ball_pos': 0.5}}
    c._physics_player = SimpleNamespace(task=player)
    c._mvae_player = SimpleNamespace(_phase_pred=torch.rand(N, generator=g) * 6.28, _swing_type=torch.randint(-1, 4, (N,), generator=g),
                                     _swing_type_cycle=torch.randint(-1, 4, (N,), generator=g))
    c._num_humanoid_bodies, c._racket_body_id = 24, 24
    c._obs_ball_traj_length = 10
    c._is_train = True
    c._ball_traj = torch.randn(N, 100, 3, generator=g)
    c._ball_obs = torch.zeros(N, 10, 3)
    c._target_bounce_pos = torch.tensor([[0.0, 10.0, 0.0]]).repeat(N, 1)
    c._target_bounce_pos[::3, 0] = -3
    c._tar_action = torch.randint(0, 2, (N,), generator=g)
    c._tar_time = torch.randint(60, 80, (N,), generator=g)
    c._tar_time_total = torch.randint(65, 75, (N,), generator=g)
    c._bounce_in = torch.zeros(N, dtype=torch.bool)
    c._est_bounce_pos = torch.zeros(N, 3)
    c._est_bounce_time = torch.zeros(N)
    c._est_bounce_in = torch.zeros(N, dtype=torch.bool)
    c._est_max_height = torch.zeros(N)
    c._reward_scales = {'pos': 5.0, 'phase': 10.0, 'bounce_pos': 0.05, 'bounce_time': 0.1}
    c._court_min = torch.tensor([-8.0, -14.0])
    c._court_max = torch.tensor([8.0, 0.0])
    c._max_episode_length = 300
    c._distance = torch.zeros(N)
    c.obs_buf = torch.zeros(N, 225 + 30 + 2)
    c.rew_buf = torch.zeros(N)
    c.reset_buf = torch.zeros(N, dtype=torch.long)
    c.progress_buf = torch.randint(0, 310, (N,), generator=g)
    c._terminate_buf = torch.zeros(N, dtype=torch.long)
    c._reset_reaction_buf = torch.zeros(N, dtype=torch.bool)
    c._reset_recovery_buf = torch.zeros(N, dtype=torch.bool)

    # estimator with a small synthetic grid
    est = E.TennisBallOutEstimator.__new__(E.TennisBallOutEstimator)
    est.params = SmallParams
    rng = np.random.default_rng(4)
    nrow = 4 * 3 * 2
    est._ball_traj_out_x = torch.from_numpy(rng.normal(0.3, 0.6, (nrow, 60)).astype(np.float32))
    ty = np.zeros((nrow, 30, 2), np.float32)
    ty[..., 0] = rng.uniform(5, 25, (nrow, 30))
    ty[..., 1] = rng.uniform(0.3, 1.5, (nrow, 30))
    est._ball_traj_out_y = torch.from_numpy(ty)
    c._ball_out_estimator = est
    rec = dict(est_x=est._ball_traj_out_x, est_y=est._ball_traj_out_y,
               est_params=np.array([SmallParams.VEL_X_RANGE, SmallParams.VEL_Y_RANGE, SmallParams.VSPIN_RANGE,
                                    SmallParams.TRAJ_X_RANGE, SmallParams.TRAJ_Y_RANGE], np.float64),
               rbs=rbs, ball_states=bstates, ball_traj=c._ball_traj.clone(), target_bounce_pos=c._target_bounce_pos.clone(),
               tar_action=c._tar_action.clone(), tar_time=c._tar_time.clone(), tar_time_total=c._tar_time_total.clone(),
               phase=c._mvae_player._phase_pred, swing_type=c._mvae_player._swing_type, swing_type_cycle=c._mvae_player._swing_type_cycle,
               progress=c.progress_buf.clone(), court_min=c._court_min, court_max=c._court_max)
    for k in ("_root_pos", "_root_vel", "_racket_pos", "_racket_vel", "_racket_normal", "_ball_pos", "_ball_vel", "_ball_vspin",
              "_has_racket_ball_contact", "_has_racket_ball_contact_now", "_has_bounce", "_has_bounce_now", "_bounce_pos"):
        rec["p" + k] = getattr(player, k).clone()

    # the out-estimator calls .get_device() / .to(device) with CUDA tensors in mind; on CPU route them to 'cpu'
    orig = torch.Tensor.get_device
    torch.Tensor.get_device = lambda self: torch.device('cpu')
    try:
        c._update_state()
    finally:
        torch.Tensor.get_device = orig
    rec.update(bounce_in=c._bounce_in.clone(), est_bounce_pos=c._est_bounce_pos.clone(), est_bounce_time=c._est_bounce_time.clone(),
               est_bounce_in=c._est_bounce_in.clone(), est_max_height=c._est_max_height.clone())
    # rewards: all three types on the same state
    for rt in ("reach", "return", "return_w_estimate"):
        c.cfg_v2p['reward_type'] = rt
        c._compute_reward(None)
        rec[f"rew_{rt}"] = c.rew_buf.clone()
        rec[f"sub_{rt}"] = c._sub_rewards.clone()
        rec[f"names_{rt}"] = np.array(c._sub_rewards_names)
    c._compute_observations()
    rec.update(obs=c.obs_buf.clone(), ball_obs_after=c._ball_obs.clone())
    c.obs_buf[5, 7] = float('nan')   # NaN guard -> terminate
    rec["obs_for_reset"] = c.obs_buf.clone()
    c._compute_reset()
    rec.update(reset=c.reset_buf.clone(), terminate=c._terminate_buf.clone(), reset_reaction=c._reset_reaction_buf.clone(),
               reset_recovery=c._reset_recovery_buf.clone(), distance=c._distance.clone(),
               out_of_court=C.check_out_of_court(c._root_pos, c._court_min, c._court_max))
    # ---- use_history_ball_obs (:213-214, :345-351): a reaction reset fills the history with the ball position, every observation
    # rolls it by one and appends the current position; _compute_observations(ids) touches the listed rows only
    c.cfg_v2p['use_history_ball_obs'] = True
    c.cfg_v2p['reset_reaction_nframes'] = 70
    c._num_reset_reaction = torch.zeros(N, dtype=torch.long)
    c._mvae_player._swing_type_cycle = c._mvae_player._swing_type_cycle.clone()   # `rec` holds the recorded tensor itself
    hist = dict(hist_in=c._ball_obs.clone(), hist_ball_pos0=player._ball_pos.clone())
    ids = torch.tensor([1, 5, 9, 33])
    c._reset_reaction_tasks(ids)
    hist.update(hist_reset_ids=ids, hist_after_reset=c._ball_obs.clone(), hist_target_bounce_pos=c._target_bounce_pos.clone())
    part = torch.tensor([0, 1, 2, 40, 41])
    c._compute_observations(part)
    hist.update(hist_part_ids=part, hist_after_partial=c._ball_obs.clone(), hist_obs_partial=c.obs_buf.clone())
    for k in range(2):
        player._ball_pos += 0.1 * (k + 1) * torch.randn(N, 3, generator=g)     # in place: the controller's _ball_pos is this tensor
        c._compute_observations()
        hist[f"hist_ball_pos{k + 1}"] = player._ball_pos.clone()
        hist[f"hist_after_full{k + 1}"] = c._ball_obs.clone()
        hist[f"hist_obs_full{k + 1}"] = c.obs_buf.clone()
    rec.update(hist)
    npz("v2p_controller.npz", **rec)


def fix_head():
    """_set_target_motion_state with fix_head_orientation (:600-661): head / neck yaw correction towards the ball"""
    g = torch.Generator().manual_seed(25)
    N = 48
    t = FakePlayer()
    t.device = 'cpu'
    t.num_envs = N
    t.dt = 2 * (1.0 / 60.0)
    t.cfg_v2p = {'fix_head_orientation': True}
    t._head_body_id = 13
    t._build_mujoco_smpl_transform()
    rest = rest_joints_smpl_order()
    t._smpl = SimpleNamespace(joint_pos_bind=rest.unsqueeze(0).repeat(N, 1, 1), parents=torch.tensor(SMPL_PARENTS))
    aa = 0.4 * torch.randn(N, 24, 3, generator=g)
    aa[:, 0] = torch.tensor([1.2092, 1.2092, 1.2092]) + 0.1 * torch.randn(N, 3, generator=g)   # ~ the z-up base rotation
    aa[0, 15] = 0
    aa[0, 12] = 0
    rm = angle_axis_to_rotation_matrix(aa.view(-1, 3)).view(N, 24, 3, 3)
    t._mvae_player = SimpleNamespace(_root_pos=torch.randn(N, 3, generator=g) * torch.tensor([2.0, 2.0, 0.1]) + torch.tensor([0.0, -13.0, 0.95]),
                                     _joint_rotmat=rm.clone())
    t._ball_pos = torch.randn(N, 3, generator=g) * torch.tensor([3.0, 8.0, 0.5]) + torch.tensor([0.0, -2.0, 1.0])
    t._ball_pos[1, 0] = 4.5                       # |x| > 4: miss -> no correction
    t._ball_pos[2, 1] = -20.0                     # behind the player: miss
    t._root_pos = t._mvae_player._root_pos + 0.05 * torch.randn(N, 3, generator=g)
    t._prev_target_root_pos = t._mvae_player._root_pos - 0.02
    o = t._smpl_to_sim(t._mvae_player._root_pos.clone(), rm)
    t._prev_target_rb_rot = torch.nn.functional.normalize(o[7] + 0.02 * torch.randn(N, 24, 4, generator=g), dim=-1)
    t._set_target_motion_state()
    npz("v2p_fix_head.npz", rest=rest, parents=np.array(SMPL_PARENTS), smpl_2_mujoco=np.array(t._smpl_2_mujoco), dt=np.array(t.dt),
        rotmat_in=rm, player_root_pos=t._mvae_player._root_pos, ball_pos=t._ball_pos, root_pos=t._root_pos,
        prev_target_root_pos=t._prev_target_root_pos, prev_target_rb_rot=t._prev_target_rb_rot,
        rotmat_out=t._mvae_player._joint_rotmat, target_root_rot=t._target_root_rot, target_dof_pos=t._target_dof_pos,
        target_dof_vel=t._target_dof_vel, target_rb_pos=t._target_rb_pos, target_rb_rot=t._target_rb_rot,
        target_root_vel=t._target_root_vel)


class SmallInParams:
    VEL_X_RANGE = (25, 26, 0.25)
    VEL_Y_RANGE = (5, 6, 0.5)
    VSPIN_RANGE = (5, 7, 0.5)
    HEIGHT_RANGE = (0.5, 1.0, 0.1)


def dual():
    from env.tasks import humanoid_smpl_im_mvae_dual as MD
    from env.tasks import physics_mvae_controller_dual as CD
    from utils import tennis_ball_in_estimator as EI
    g = torch.Generator().manual_seed(26)
    rec = {}
    # ---- in-estimator on a small synthetic grid (one set on the full-size parameter grid's index math as well)
    est = EI.TennisBallInEstimator.__new__(EI.TennisBallInEstimator)
    est.params = SmallInParams
    rng = np.random.default_rng(5)
    nrow = 5 * 4 * 2 * 4
    tab = np.zeros((nrow, 50, 2), np.float32)
    tab[..., 0] = np.cumsum(rng.uniform(0.3, 0.5, (nrow, 50)), axis=1)
    tab[..., 1] = rng.uniform(0.05, 2.0, (nrow, 50))
    est._ball_traj = torch.from_numpy(tab)
    n = 96
    bs = torch.zeros(n, 13)
    bs[:, 0:3] = torch.randn(n, 3, generator=g) * torch.tensor([2.0, 2.0, 0.4]) + torch.tensor([0.0, -11.0, 0.8])
    bs[:, 3:7] = rq(g, n)
    bs[:, 7] = torch.randn(n, generator=g) * 4
    bs[:, 8] = torch.rand(n, generator=g) * 3 + 24
    bs[:, 9] = torch.rand(n, generator=g) * 2 + 4.5
    bs[:, 10:13] = torch.randn(n, 3, generator=g) * 25
    bs[0, 2], bs[1, 2] = 0.2, 3.0                       # clamped heights
    orig = torch.Tensor.get_device
    torch.Tensor.get_device = lambda self: torch.device('cpu')
    try:
        traj, s_in, s_out = est.estimate(bs.clone())
        idx, snapped = est.get_ball_traj_index(bs[:, 2], bs[:, 7:9].norm(dim=-1), bs[:, 9], bs[:, 10:13].norm(dim=1) / (np.pi * 2))
        # index math on the shipped (full-size) parameter grid
        est_full = EI.TennisBallInEstimator.__new__(EI.TennisBallInEstimator)
        est_full.params = EI.traj_in_params
        h = torch.rand(4096, generator=g) * 2.0 + 0.3
        vx = torch.rand(4096, generator=g) * 6 + 24.5
        vy = torch.rand(4096, generator=g) * 4 + 4.5
        vs = torch.rand(4096, generator=g) * 6 + 4.5
        idx_full, snapped_full = est_full.get_ball_traj_index(h, vx, vy, vs)
    finally:
        torch.Tensor.get_device = orig
    P = SmallInParams
    rec.update(in_table=tab, in_params=np.array([P.HEIGHT_RANGE, P.VEL_X_RANGE, P.VEL_Y_RANGE, P.VSPIN_RANGE], np.float64),
               in_params_full=np.array([EI.traj_in_params.HEIGHT_RANGE, EI.traj_in_params.VEL_X_RANGE, EI.traj_in_params.VEL_Y_RANGE,
                                        EI.traj_in_params.VSPIN_RANGE], np.float64),
               in_states=bs, in_traj=traj, in_states_in=s_in, in_states_out=s_out, in_index=idx,
               full_h=h, full_vx=vx, full_vy=vy, full_vs=vs, full_index=idx_full, full_snapped=torch.stack(snapped_full, dim=-1))

    # ---- HumanoidSMPLIMMVAEDual._reset_balls through the real method on a fake self
    class FakeDual(MD.HumanoidSMPLIMMVAEDual):
        def __init__(self):
            pass
    N = 32
    t = FakeDual()
    t.device = 'cpu'
    t.cfg_v2p = {}
    t._ball_in_estimator = est
    t._ball_root_states = torch.zeros(N, 13)
    t._ball_root_states[:, 0:3] = torch.randn(N, 3, generator=g) * torch.tensor([2.0, 2.0, 0.3]) + torch.tensor([0.0, -11.0, 0.8])
    t._ball_root_states[:, 6] = 1
    t._ball_root_states[:, 7] = torch.randn(N, generator=g) * 3
    t._ball_root_states[:, 8] = torch.rand(N, generator=g) * 2 + 24.5
    t._ball_root_states[:, 9] = torch.rand(N, generator=g) * 1.5 + 4.8
    t._ball_root_states[:, 10:13] = torch.randn(N, 3, generator=g) * 25
    t._mvae_player = SimpleNamespace(_racket_pos=torch.randn(N, 3, generator=g) * 0.5 + torch.tensor([0.3, -11.5, 1.0]))
    t._has_bounce = torch.ones(N, dtype=torch.bool)
    t._bounce_pos = torch.ones(N, 3)
    t._has_racket_ball_contact = torch.ones(N, dtype=torch.bool)
    t._ball_pos = torch.zeros(N, 3)
    t._ball_vel = torch.zeros(N, 3)
    rec["rb_states_before"] = t._ball_root_states.clone()
    rec["rb_racket_pos"] = t._mvae_player._racket_pos.clone()
    serve_recovery = torch.tensor([1, 5, 8])            # serving players (their opponents react): envs 0, 4, 9 receive
    ball_ids = torch.tensor([0, 4, 9, 12, 17, 30])       # reaction envs that get a new incoming ball
    torch.manual_seed(77)
    rec["rb_rand"] = torch.stack([torch.rand(3), torch.rand(3), torch.rand(3)])   # the three torch.rand(num_envs) draws, in order
    torch.manual_seed(77)
    torch.Tensor.get_device = lambda self: torch.device('cpu')
    try:
        traj2 = t._reset_balls(serve_recovery, ball_ids)
    finally:
        torch.Tensor.get_device = orig
    rec.update(rb_recovery_ids=serve_recovery, rb_ball_ids=ball_ids, rb_traj=traj2, rb_states_after=t._ball_root_states.clone(),
               rb_has_bounce=t._has_bounce, rb_bounce_pos=t._bounce_pos, rb_has_contact=t._has_racket_ball_contact, rb_ball_pos=t._ball_pos,
               rb_ball_vel=t._ball_vel)

    # ---- PhysicsMVAEControllerDual._compute_reset
    class FakeCtlDual(CD.PhysicsMVAEControllerDual):
        def __init__(self):
            pass
    N = 128
    c = FakeCtlDual()
    player = SimpleNamespace(_has_racket_ball_contact=torch.rand(N, generator=g) < 0.3, _has_bounce=torch.rand(N, generator=g) < 0.5)
    c._physics_player = SimpleNamespace(task=player)
    c._tar_action = torch.randint(0, 2, (N,), generator=g)
    c._ball_pos = torch.randn(N, 3, generator=g) * torch.tensor([3.0, 6.0, 0.1]) + torch.tensor([0.0, -9.0, 0.1])
    c._root_pos = torch.randn(N, 3, generator=g) * torch.tensor([2.0, 2.0, 0.05]) + torch.tensor([0.0, -12.0, 0.9])
    c._root_vel = torch.randn(N, 3, generator=g)
    c._bounce_in = torch.rand(N, generator=g) < 0.6
    c._distance = torch.rand(N, generator=g)
    c.reset_buf = (torch.rand(N, generator=g) < 0.05).long()
    c._reset_reaction_buf = torch.rand(N, generator=g) < 0.5
    c._reset_recovery_buf = torch.rand(N, generator=g) < 0.5
    for k in ("_tar_action", "_ball_pos", "_root_pos", "_root_vel", "_bounce_in", "_distance", "reset_buf"):
        rec["cr" + k] = getattr(c, k).clone()
    rec["cr_has_contact"], rec["cr_has_bounce"] = player._has_racket_ball_contact, player._has_bounce
    c._compute_reset()
    rec.update(cr_out_reset=c.reset_buf, cr_out_reaction=c._reset_reaction_buf, cr_out_recovery=c._reset_recovery_buf,
               cr_out_distance=c._distance)
    npz("v2p_dual.npz", **rec)


def task_reset():
    """the pool index rule with start_pos, the recovery / reaction task resets; the torch draws are recorded in call order"""
    P, N = 997, 96
    rng = np.random.default_rng(8)
    pool = rng.normal(0, 5, (P, 307)).astype(np.float32)
    path = os.path.join("/tmp", "v2p_pool_tr.npy")
    np.save(path, pool)
    gen = TennisBallGeneratorOffline(traj_file=path, sample_random=True, num_envs=N)
    start = np.stack([rng.uniform(-5, 5, N), rng.uniform(-3, 3, N), np.ones(N)], -1).astype(np.float32)
    start[:10, 0] = [-4, np.nextafter(np.float32(-4), np.float32(0)), 4, np.nextafter(np.float32(4), np.float32(0)), -4 - 8 / P, -5, 5, 0,
                     -4 + 8 / P, 4 - 8 / P]
    start[:10, 1] = 1.0
    start[10:13, 1] = [0.0, np.nextafter(np.float32(0), np.float32(1)), np.nextafter(np.float32(0), np.float32(-1))]
    draws, randint = [], torch.randint

    def rec_randint(*a, **k):
        draws.append(randint(*a, **k))
        return draws[-1]
    torch.manual_seed(4)
    torch.randint = rec_randint
    try:
        _, launch_pos, _, _ = gen.generate(N, need_init_state=True, start_pos=torch.from_numpy(start))
    finally:
        torch.randint = randint
    index = np.array([int(np.flatnonzero((pool[:, 0:3] == p).all(1))[0]) for p in launch_pos.numpy()])
    side = np.zeros(N, np.int64)
    side[start[:, 1] > 0] = draws[1].numpy()
    out = dict(tr_pool_size=P, tr_start=start, tr_pool_rand=draws[0].numpy(), tr_side_rand=side, tr_index=index)
    # _reset_recovery_tasks / _reset_reaction_tasks through a fake controller
    for mode in ("continuous", "discrete"):
        c = SimpleNamespace(device='cpu', cfg_v2p={'use_history_ball_obs': True, 'reset_reaction_nframes': 70, 'use_random_ball_target': mode},
                            _obs_ball_traj_length=10)
        c._ball_obs, c._ball_pos = torch.randn(N, 10, 3), torch.randn(N, 3)
        c._tar_time, c._tar_action, c._num_reset_reaction = torch.randint(0, 80, (N,)), torch.randint(0, 2, (N,)), torch.randint(0, 5, (N,))
        c._bounce_in, c._est_bounce_in = torch.rand(N) < 0.5, torch.rand(N) < 0.5
        c._est_bounce_pos, c._est_bounce_time, c._est_max_height = torch.randn(N, 3), torch.rand(N), torch.rand(N)
        c._mvae_player = SimpleNamespace(_swing_type_cycle=torch.randint(-1, 4, (N,)))
        c._tar_time_total, c._target_bounce_pos = torch.randint(60, 80, (N,)), torch.randn(N, 3)
        c._target_bounce_min, c._target_bounce_max = torch.tensor([-3.0, 9.0, 0.0]), torch.tensor([3.0, 11.0, 0.0])
        c._physics_player = SimpleNamespace(task=SimpleNamespace(_has_bounce=torch.rand(N) < 0.5, _bounce_pos=torch.randn(N, 3)))
        names = ("_ball_obs", "_ball_pos", "_tar_time", "_tar_action", "_num_reset_reaction", "_bounce_in", "_est_bounce_in", "_est_bounce_pos",
                 "_est_bounce_time", "_est_max_height", "_tar_time_total", "_target_bounce_pos")
        for k in names:
            out[f"{mode}_in{k}"] = getattr(c, k).clone()
        out[f"{mode}_in_cycle"] = c._mvae_player._swing_type_cycle.clone()
        out[f"{mode}_in_has_bounce"] = c._physics_player.task._has_bounce.clone()
        out[f"{mode}_in_bounce_pos"] = c._physics_player.task._bounce_pos.clone()
        rec_ids, rea_ids = torch.tensor([1, 4, 9, 33, 70]), torch.tensor([0, 4, 17, 33, 50, 51, 95])
        C.PhysicsMVAEController._reset_recovery_tasks(c, rec_ids)
        rd, rand = [], torch.rand
        torch.manual_seed(5)
        torch.randint = rec_randint
        torch.rand = lambda *a, **k: rd.append(rand(*a, **k)) or rd[-1]
        try:
            draws.clear()
            C.PhysicsMVAEController._reset_reaction_tasks(c, rea_ids)
        finally:
            torch.randint, torch.rand = randint, rand
        if mode == "discrete":
            rd[0][:3] = torch.tensor([0.33, 0.67, float(np.nextafter(np.float32(0.33), np.float32(1)))])
            torch.manual_seed(5)   # replay with the edge seeds written into the draw
            seeds = rd[0].clone()
            torch.randint = lambda *a, **k: draws[0]
            torch.rand = lambda *a, **k: seeds
            try:
                for k in names:
                    getattr(c, k).copy_(out[f"{mode}_in{k}"])
                c._mvae_player._swing_type_cycle.copy_(out[f"{mode}_in_cycle"])
                c._physics_player.task._has_bounce.copy_(out[f"{mode}_in_has_bounce"])
                c._physics_player.task._bounce_pos.copy_(out[f"{mode}_in_bounce_pos"])
                C.PhysicsMVAEController._reset_recovery_tasks(c, rec_ids)
                C.PhysicsMVAEController._reset_reaction_tasks(c, rea_ids)
            finally:
                torch.randint, torch.rand = randint, rand
        out.update({f"{mode}_rec_ids": rec_ids, f"{mode}_rea_ids": rea_ids, f"{mode}_frame_rand": draws[0], f"{mode}_seed": rd[0],
                    f"{mode}_out_cycle": c._mvae_player._swing_type_cycle, f"{mode}_out_has_bounce": c._physics_player.task._has_bounce,
                    f"{mode}_out_bounce_pos": c._physics_player.task._bounce_pos})
        for k in names:
            out[f"{mode}_out{k}"] = getattr(c, k).clone()
    npz("v2p_task_reset.npz", **out)


if __name__ == "__main__":
    if sys.argv[1:] == ["task_reset"]:
        task_reset()
        sys.exit(0)
    dual()
    fix_head()
    smpl_to_sim()
    ball()
    update_state()
    controller()
