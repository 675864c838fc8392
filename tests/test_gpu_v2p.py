"""GPU parity of the vid2player kernels (include/b200env_v2p.h) against the fixtures produced by executing the
reference's own vid2player code (tests/golden/v2p_*.npz)."""
import numpy as np
import pytest
import torch

from conftest import golden
from helpers import SIM_PARAMS, v2p_cfg

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def T(a, dtype=None):
    t = torch.tensor(a, device=DEV)
    return t.to(dtype).contiguous() if dtype is not None else t.contiguous()


def close(a, b, tol=1e-5, msg=""):
    np.testing.assert_allclose(a.detach().cpu().numpy() if isinstance(a, torch.Tensor) else a, b, rtol=0, atol=tol, err_msg=msg)


def test_smpl_to_sim_golden():
    from vid2player3d_b200 import native_v2p as V
    g = golden("v2p_smpl_to_sim.npz")
    n = g["root0"].shape[0]
    mk = lambda: dict(root_rot=torch.zeros(n, 4, device=DEV), dof_pos=torch.zeros(n, 69, device=DEV), root_vel=torch.zeros(n, 3, device=DEV),  # noqa: E731
                      root_ang_vel=torch.zeros(n, 3, device=DEV), dof_vel=torch.zeros(n, 69, device=DEV),
                      rb_pos=torch.zeros(n, 24, 3, device=DEV), rb_rot=torch.zeros(n, 24, 4, device=DEV))
    rest, par, s2m = T(g["rest"]), T(g["parents"], torch.int32), T(g["smpl_2_mujoco"], torch.int32)
    a = mk()
    V.smpl_to_sim(T(g["root0"]), T(g["rotmat0"]), rest, par, s2m, float(g["dt"]), a)
    for k in a:
        close(a[k], g["a_" + k], 2e-5, k)
    b = mk()
    V.smpl_to_sim(T(g["root1"]), T(g["rotmat1"]), rest, par, s2m, float(g["dt"]), b, prev_root_pos=T(g["a_root_pos"]), prev_rb_rot=T(g["a_rb_rot"]))
    for k in b:
        tol = {"dof_vel": 2e-3, "root_ang_vel": 6e-2}.get(k, 2e-5)   # finite differences: /dt and /dt^2 amplify 1e-7 rounding
        close(b[k], g["b_" + k], tol, k)


def test_ball_aero_and_reset_golden():
    from vid2player3d_b200 import native_v2p as V
    g = golden("v2p_ball.npz")
    for s in (2, 6):
        bs = T(g[f"s{s}_ball_states"])
        n = bs.shape[0]
        hb, now = T(g[f"s{s}_has_bounce_in"]), torch.zeros(n, dtype=torch.bool, device=DEV)
        bpos, force = torch.zeros(n, 3, device=DEV), torch.zeros(n, 3, device=DEV)
        V.ball_aero(bs, hb, now, bpos, force, s, 5.0)
        close(force, g[f"s{s}_force"], 1e-6)
        assert np.array_equal(hb.cpu().numpy(), g[f"s{s}_has_bounce"]) and np.array_equal(now.cpu().numpy(), g[f"s{s}_has_bounce_now"])
        close(bpos, g[f"s{s}_bounce_pos"], 0)
    N = 64
    ids, pidx = T(g["reset_ids"]), T(g["reset_pool_index"])
    bs = torch.zeros(N, 13, device=DEV)
    bpos, bvel, bounce = torch.zeros(N, 3, device=DEV), torch.zeros(N, 3, device=DEV), torch.ones(N, 3, device=DEV)
    hb, hc = torch.ones(N, dtype=torch.bool, device=DEV), torch.ones(N, dtype=torch.bool, device=DEV)
    traj = torch.zeros(N, 100, 3, device=DEV)
    V.ball_reset(ids, pidx, T(g["pool"]), bs, bpos, bvel, hb, bounce, hc, traj)
    V.ball_reset(ids[:0], pidx[:0], T(g["pool"]), bs, bpos, bvel, hb, bounce, hc, traj)  # empty id list: no-op
    close(bs, g["reset_ball_states"], 2e-5)
    close(traj[ids], g["reset_traj"], 0)
    assert np.array_equal(hb.cpu().numpy(), g["reset_has_bounce"]) and np.array_equal(hc.cpu().numpy(), g["reset_contact"])
    close(bounce, g["reset_bounce_pos"], 0)
    close(bpos[ids], g["reset_ball_states"][g["reset_ids"], 0:3], 0)


def test_update_state_golden():
    from vid2player3d_b200 import native_v2p as V
    g = golden("v2p_update_state.npz")
    for grip in ("eastern", "semi_western"):
        rbs, root, ball = T(g[f"{grip}_rbs"]), T(g[f"{grip}_root_states"]), T(g[f"{grip}_ball_states"])
        n = rbs.shape[0]
        t = dict(has_contact=T(g[f"{grip}_contact_in"]), has_contact_now=torch.zeros(n, dtype=torch.bool, device=DEV),
                 ball_vel=T(g[f"{grip}_prev_ball_vel"]), ball_vspin=torch.zeros(n, device=DEV))
        for k in ("root_pos", "root_vel", "racket_pos", "racket_vel", "racket_normal", "ball_pos"):
            t[k] = torch.zeros(n, 3, device=DEV)
        V.update_state(n, 26, rbs, root, 13, ball, 13, t, grip=grip)
        for k in ("root_pos", "root_vel", "racket_pos", "racket_vel", "racket_normal", "ball_pos", "ball_vel", "ball_vspin"):
            close(t[k], g[f"{grip}_{k}"], 2e-6, k)
        assert np.array_equal(t["has_contact"].cpu().numpy(), g[f"{grip}_contact"])
        assert np.array_equal(t["has_contact_now"].cpu().numpy(), g[f"{grip}_contact_now"])


@pytest.mark.parametrize("rtype", ["reach", "return", "return_w_estimate"])
def test_controller_post_golden(rtype):
    from vid2player3d_b200 import native_v2p as V
    g = golden("v2p_controller.npz")
    N = g["rbs"].shape[0]
    z = lambda *s, dt=torch.float32: torch.zeros(*s, device=DEV, dtype=dt)  # noqa: E731
    obs = z(N, 257)
    t = dict(rigid_body_state=T(g["rbs"]), ball_states=T(g["ball_states"]), root_pos=T(g["p_root_pos"]), root_vel=T(g["p_root_vel"]),
             racket_pos=T(g["p_racket_pos"]), racket_normal=T(g["p_racket_normal"]), ball_pos=T(g["p_ball_pos"]),
             has_contact=T(g["p_has_racket_ball_contact"]), has_contact_now=T(g["p_has_racket_ball_contact_now"]),
             has_bounce=T(g["p_has_bounce"]), has_bounce_now=T(g["p_has_bounce_now"]), bounce_pos=T(g["p_bounce_pos"]),
             ball_traj=T(g["ball_traj"]), target_bounce_pos=T(g["target_bounce_pos"]), phase=T(g["phase"]), swing_type=T(g["swing_type"]),
             swing_type_cycle=T(g["swing_type_cycle"]), tar_action=T(g["tar_action"]), tar_time=T(g["tar_time"]),
             tar_time_total=T(g["tar_time_total"]), progress_buf=T(g["progress"]), est_x=T(g["est_x"]), est_y=T(g["est_y"]),
             bounce_in=z(N, dt=torch.bool), est_bounce_in=z(N, dt=torch.bool), reset_reaction=z(N, dt=torch.bool),
             reset_recovery=z(N, dt=torch.bool), est_bounce_pos=z(N, 3), est_bounce_time=z(N), est_max_height=z(N), distance=z(N),
             obs_buf=obs, rew_buf=z(N), sub_rewards=z(N, 2), reset_buf=z(N, dt=torch.long), terminate_buf=z(N, dt=torch.long))
    cfg = dict(n=N, bodies_per_env=25, ball_stride=13, racket_body=24, num_obs=257, obs_traj_len=10, use_target=1,
               reward_type=V.REWARD_TYPES[rtype], early_termination=1, max_episode_length=300, est_nx=60, est_ny=30, scale_pos=5.0,
               scale_phase=10.0, scale_bounce_pos=0.05, scale_bounce_time=0.1, w_pos=0.5, w_ball_pos=0.5,
               court_min=g["court_min"], court_max=g["court_max"], est_params=g["est_params"].reshape(-1))
    V.controller_post(cfg, t)
    torch.cuda.synchronize()
    close(obs, g["obs"], 2e-6)
    assert np.array_equal(t["bounce_in"].cpu().numpy(), g["bounce_in"])
    close(t["est_bounce_pos"], g["est_bounce_pos"], 1e-5); close(t["est_bounce_time"], g["est_bounce_time"], 1e-6)
    close(t["est_max_height"], g["est_max_height"], 1e-5)
    assert np.array_equal(t["est_bounce_in"].cpu().numpy(), g["est_bounce_in"])
    close(t["rew_buf"], g[f"rew_{rtype}"], 1e-5)
    ns = g[f"sub_{rtype}"].shape[1]
    close(t["sub_rewards"][:, :ns], g[f"sub_{rtype}"], 1e-5)
    close(t["distance"], g["distance"], 1e-6)
    if rtype == "return_w_estimate":   # the golden _compute_reset ran with this reward type and a NaN row in obs
        t["root_pos"][5, 0] = float("nan")   # reproduces obs row 5 carrying a NaN (root_pos feeds obs[0])
        V.controller_post(cfg, t)
        torch.cuda.synchronize()
        for k, gk in (("reset_buf", "reset"), ("terminate_buf", "terminate"), ("reset_reaction", "reset_reaction"), ("reset_recovery", "reset_recovery")):
            got = t[k].cpu().numpy()
            want = g[gk]
            assert np.array_equal(got.astype(np.int64), want.astype(np.int64)), k


def test_controller_post_history_ball_obs():
    """use_history_ball_obs through the fused post kernel: obs_only refresh of the masked rows, then two full steps (golden)"""
    from vid2player3d_b200 import native_v2p as V
    g = golden("v2p_controller.npz")
    N = g["rbs"].shape[0]
    z = lambda *s, dt=torch.float32: torch.zeros(*s, device=DEV, dtype=dt)  # noqa: E731
    obs = T(g["hist_obs_partial"]).clone()
    obs[torch.isnan(obs)] = 0
    part = torch.tensor(g["hist_part_ids"], device=DEV)
    rea, rec = z(N, dt=torch.bool), z(N, dt=torch.bool)
    rea[part[:3]] = True
    rec[part[3:]] = True
    ball_pos = T(g["hist_ball_pos0"]).clone()
    hist = T(g["hist_after_reset"]).clone()
    t = dict(rigid_body_state=T(g["rbs"]), ball_states=T(g["ball_states"]), root_pos=T(g["p_root_pos"]), root_vel=T(g["p_root_vel"]),
             racket_pos=T(g["p_racket_pos"]), racket_normal=T(g["p_racket_normal"]), ball_pos=ball_pos,
             has_contact=T(g["p_has_racket_ball_contact"]), has_contact_now=T(g["p_has_racket_ball_contact_now"]),
             has_bounce=T(g["p_has_bounce"]), has_bounce_now=T(g["p_has_bounce_now"]), bounce_pos=T(g["p_bounce_pos"]),
             ball_traj=T(g["ball_traj"]), target_bounce_pos=T(g["hist_target_bounce_pos"]), phase=T(g["phase"]), swing_type=T(g["swing_type"]),
             swing_type_cycle=T(g["swing_type_cycle"]), tar_action=T(g["tar_action"]), tar_time=T(g["tar_time"]),
             tar_time_total=T(g["tar_time_total"]), progress_buf=T(g["progress"]), est_x=T(g["est_x"]), est_y=T(g["est_y"]),
             bounce_in=z(N, dt=torch.bool), est_bounce_in=z(N, dt=torch.bool), reset_reaction=rea, reset_recovery=rec,
             est_bounce_pos=z(N, 3), est_bounce_time=z(N), est_max_height=z(N), distance=z(N), obs_buf=obs, rew_buf=z(N), sub_rewards=z(N, 2),
             reset_buf=z(N, dt=torch.long), terminate_buf=z(N, dt=torch.long), ball_obs=hist)
    cfg = dict(n=N, bodies_per_env=25, ball_stride=13, racket_body=24, num_obs=257, obs_traj_len=10, use_target=1,
               reward_type=V.REWARD_TYPES["return_w_estimate"], early_termination=1, max_episode_length=300, est_nx=60, est_ny=30, scale_pos=5.0,
               scale_phase=10.0, scale_bounce_pos=0.05, scale_bounce_time=0.1, w_pos=0.5, w_ball_pos=0.5,
               court_min=g["court_min"], court_max=g["court_max"], est_params=g["est_params"].reshape(-1), use_history=1, obs_only=1)
    V.controller_post(cfg, t)          # the refresh of _reset_envs: only the rows whose reset masks are set
    torch.cuda.synchronize()
    assert np.array_equal(hist.cpu().numpy(), g["hist_after_partial"])
    close(obs[part], g["hist_obs_partial"][g["hist_part_ids"]], 2e-6)
    cfg["obs_only"] = 0
    for k in (1, 2):
        ball_pos.copy_(T(g[f"hist_ball_pos{k}"]))
        V.controller_post(cfg, t)
        torch.cuda.synchronize()
        assert np.array_equal(hist.cpu().numpy(), g[f"hist_after_full{k}"])
        close(obs, g[f"hist_obs_full{k}"], 2e-6)
    with pytest.raises(RuntimeError, match="use_history needs"):
        V.controller_post(cfg, dict(t, ball_obs=None))


def test_controller_history_mode_end_to_end():
    """PhysicsMVAEController with use_history_ball_obs: after the first reset the whole history is the launch position, afterwards its
    last row is the current ball position and the task observation is (history - racket position)"""
    from vid2player3d_b200.tasks import PhysicsMVAEController
    torch.manual_seed(3)
    env = PhysicsMVAEController(v2p_cfg(64, use_history_ball_obs=True), SIM_PARAMS, 1, "cuda", 0, True)
    env.reset()
    task = env._physics_player.task
    L = env._obs_ball_traj_length
    assert torch.equal(env._ball_obs, task._ball_pos[:, None, :].expand(-1, L, -1))
    prev = env._ball_obs.clone()
    for i in range(3):
        env.step(torch.clamp(torch.randn(64, env.num_actions, device=env.device), -5, 5))
        keep = ~(env._reset_reaction_buf | env._reset_recovery_buf)
        assert torch.equal(env._ball_obs[:, -1], task._ball_pos)
        assert torch.equal(env._ball_obs[:, :-1], prev[:, 1:])
        want = (env._ball_obs - task._rigid_body_state.view(64, 26, 13)[:, 24, 0:3][:, None]).reshape(64, -1)
        assert torch.allclose(env.obs_buf[:, 225:225 + 3 * L], want, atol=1e-6)
        env.reset(env.reset_buf.nonzero(as_tuple=False).flatten())
        prev = env._ball_obs.clone()
        assert keep.any()


def test_test_time_joint_rot_export():
    """is_train False (humanoid_smpl_im_mvae.py:814-820): _joint_rot = root angle-axis | dof_pos in SMPL joint order"""
    from scipy.spatial.transform import Rotation
    from vid2player3d_b200.tasks import PhysicsMVAEController
    cfg = v2p_cfg(16)
    cfg["env"]["is_train"] = False
    env = PhysicsMVAEController(cfg, SIM_PARAMS, 1, "cuda", 0, True)
    env.reset()
    env.step(torch.zeros(16, env.num_actions, device=env.device))
    task = env._physics_player.task
    jr = env._joint_rot.cpu().numpy()
    dof = task._dof_pos.cpu().numpy().reshape(16, 23, 3)
    root = Rotation.from_quat(task._rigid_body_rot[:, 0].cpu().numpy()).as_rotvec()
    mj_pose = np.concatenate([root[:, None], dof], 1)                     # mujoco body order (Pelvis first)
    assert np.abs(jr - mj_pose[:, task._mujoco_2_smpl]).max() < 1e-5
    assert np.abs(jr[:, 0] - root).max() < 1e-5                           # Pelvis is joint 0 in both orders


def test_masked_actor_reset_equals_id_list_reset_and_reset_graph_runs():
    """mask-driven humanoid reset (b200v2p_areset_t.mask, CUDA-graph safe) == the id-list one; the controller's reset graph keeps
    the reset contract: listed envs restart (progress 0, sim state = FK of the motion generator's pose), the others are untouched"""
    from vid2player3d_b200.tasks import PhysicsMVAEController
    envs = []
    for _ in range(2):
        torch.manual_seed(11)
        e = PhysicsMVAEController(v2p_cfg(48), SIM_PARAMS, 1, "cuda", 0, True)
        e.reset()
        for i in range(3):
            e.step(torch.zeros(48, e.num_actions, device=e.device))
        envs.append(e)
    a, b = envs
    ids = torch.tensor([0, 5, 6, 31, 47], device=DEV)
    mask = torch.zeros(48, dtype=torch.bool, device=DEV)
    mask[ids] = True
    ta, tb = a._physics_player.task, b._physics_player.task
    ta._reset_actors(ids)
    tb._reset_actors_masked(mask)
    torch.cuda.synchronize()
    for name in ("_root_states", "_dof_state", "_rigid_body_state", "_prev_target_root_pos", "_prev_target_rb_rot", "_root_pos", "_root_vel",
                 "_pd_target_dof_pos", "_target_root_pos", "progress_buf", "reset_buf", "_terminate_buf"):
        assert torch.equal(getattr(ta, name), getattr(tb, name)), name
    # the reset graph
    b.enable_cuda_graph()
    for i in range(4):
        b.step(torch.clamp(torch.randn(48, b.num_actions, device=DEV), -5, 5))
        done = b.reset_buf.nonzero(as_tuple=False).flatten()
        keep = torch.ones(48, dtype=torch.bool, device=DEV)
        keep[done] = False
        before = tb._dof_state.view(48, -1).clone()
        prog = b.progress_buf.clone()
        b.reset(done)
        torch.cuda.synchronize()
        assert torch.equal(tb._dof_state.view(48, -1)[keep], before[keep])                 # untouched envs
        assert bool((b.progress_buf[done] == 0).all()) and torch.equal(b.progress_buf[keep], prog[keep])
        assert bool((b.reset_buf[done] == 0).all()) and bool(torch.isfinite(b.obs_buf).all())
        if len(done):
            want = tb._tmp["dof_pos"][done]                                                # FK of the (re-drawn) generator pose
            assert torch.allclose(tb._dof_state.view(48, -1, 2)[done, :, 0], want) and bool((tb._dof_state.view(48, -1, 2)[done, :, 1] == 0).all())
    assert b._reset_graph is not None


def test_stream_motion_player_in_step_and_reset_graphs():
    """StreamMotionPlayer (resident target stream): a step is a gather of frame (t + offset) % K, a reset re-draws offsets; the
    controller's step graph and reset graph replay it"""
    from vid2player3d_b200.tasks import PhysicsMVAEController
    from vid2player3d_b200.tasks.physics_mvae_controller import StreamMotionPlayer
    cfg = v2p_cfg(40)
    cfg["env"]["motion_player"] = "stream"
    torch.manual_seed(2)
    env = PhysicsMVAEController(cfg, SIM_PARAMS, 1, "cuda", 0, True)
    p = env._mvae_player
    assert isinstance(p, StreamMotionPlayer)
    ring = p._ring["_joint_rotmat"].view(p.K, 40, 24, 3, 3)
    env.reset()
    env.enable_cuda_graph()
    for i in range(5):
        t0, off0 = int(p._t), p._off.clone()
        env.step(torch.zeros(40, env.num_actions, device=DEV))
        assert int(p._t) == t0 + 1
        want = ring[(t0 + 1 + off0) % p.K, torch.arange(40, device=DEV)]
        assert torch.equal(p._joint_rotmat, want)
        done = torch.tensor([1, 7, 20], device=DEV) if i == 2 else env.reset_buf.nonzero(as_tuple=False).flatten()
        env.reset(done)
        keep = torch.ones(40, dtype=torch.bool, device=DEV)
        keep[done] = False
        assert torch.equal(p._off[keep], off0[keep])
        assert bool(torch.isfinite(env.obs_buf).all())
    det = torch.linalg.det(p._joint_rotmat.reshape(-1, 3, 3))
    assert float((det - 1).abs().max()) < 1e-4


def test_dual_masked_reset_matches_id_list_reset_on_deterministic_fields():
    """PhysicsMVAEControllerDual: the mask-driven reset (reset graph) against the reference-shaped id-list reset from the same state -
    everything that does not depend on a random draw must agree"""
    from helpers import v2p_dual_cfg
    from vid2player3d_b200.tasks import PhysicsMVAEControllerDual
    envs = []
    for _ in range(2):
        torch.manual_seed(21)
        cfg = v2p_dual_cfg(32)
        cfg["env"]["motion_player"] = "stream"
        e = PhysicsMVAEControllerDual(cfg, SIM_PARAMS, 1, "cuda", 0, True)
        e.reset()
        for i in range(4):
            e.step(torch.zeros(32, e.num_actions, device=DEV))
        envs.append(e)
    a, b = envs
    ta, tb = a._physics_player.task, b._physics_player.task
    assert torch.equal(ta._root_states, tb._root_states) and torch.equal(a._reset_reaction_buf, b._reset_reaction_buf)
    ids = torch.tensor([4, 5, 18, 19], device=DEV)                      # two rallies restart; other envs may carry task resets
    mask = torch.zeros(32, dtype=torch.bool, device=DEV)
    mask[ids] = True
    b._mvae_player._off.copy_(a._mvae_player._off)
    a._reset_envs(ids)
    b._mvae_player._off.copy_(a._mvae_player._off)                       # the stream offsets are random draws: align them first ...
    b._mvae_player._gather()
    off = b._mvae_player._off.clone()
    b._reset_envs_masked(mask)
    b._mvae_player._off.copy_(off)                                       # ... and keep them aligned
    torch.cuda.synchronize()
    for name in ("progress_buf", "reset_buf", "_terminate_buf", "_reset_reaction_buf", "_reset_recovery_buf", "_tar_time", "_tar_action",
                 "_num_reset_reaction", "_bounce_in", "_distance"):
        assert torch.equal(getattr(a, name), getattr(b, name)), name
    for name in ("_has_bounce", "_bounce_pos", "_has_racket_ball_contact"):
        assert torch.equal(getattr(ta, name), getattr(tb, name)), name
    servers = ids[1::2]                                                  # serve_from near: the even env receives, the odd one serves
    sv = tb._ball_root_states[servers]                                   # the served ball: random velocity draw, then snapped to the
    assert bool(torch.isfinite(sv).all()) and bool((sv[:, 8] > 20).all())  # table grid (spin axis follows the velocity): towards the far side
    untouched = torch.ones(32, dtype=torch.bool, device=DEV)
    untouched[ids] = False
    untouched &= ~(a._num_reset_reaction > 0)
    assert torch.equal(ta._dof_state.view(32, -1)[untouched], tb._dof_state.view(32, -1)[untouched])
    assert bool(torch.isfinite(b.obs_buf).all()) and bool(torch.isfinite(tb._root_states).all())
    # and the graphs run
    b.enable_cuda_graph()
    for i in range(3):
        b.step(torch.clamp(torch.randn(32, b.num_actions, device=DEV), -5, 5))
        done = b.reset_buf.nonzero(as_tuple=False).flatten()
        b.reset(done)
        assert bool((b.reset_buf[done] == 0).all()) and bool(torch.isfinite(b.obs_buf).all())
    assert b._reset_graph is not None


def test_controller_end_to_end():
    """config-3 style rollout (synthetic motion generator, zero-residual low-level policy): 150 high-level steps"""
    from helpers import SIM_PARAMS, v2p_cfg
    from oracle import ref_port_v2p as V
    from vid2player3d_b200.tasks import PhysicsMVAEController
    torch.manual_seed(0)
    N = 256
    env = PhysicsMVAEController(v2p_cfg(N), SIM_PARAMS, 1, "cuda", 0, True)
    assert env.num_obs == 257 and env.num_actions == 35
    env.reset()
    task = env._physics_player.task
    torch.cuda.synchronize()
    assert torch.isfinite(env.obs_buf).all()
    y0 = task._ball_pos[:, 1].clone()
    assert (y0 > 11).all() and (task._ball_vel[:, 1] < -15).all()          # launched from the far side towards the player
    bounced, resets, hits = 0, 0, 0
    for step in range(150):
        a = torch.clamp(torch.randn(N, 35, device=DEV), -5, 5)
        env.step(a)
        done = env.reset_buf.nonzero(as_tuple=False).flatten()
        resets += len(done)
        env.reset(done)                                                      # agent loop: env_reset(done_indices)
        bounced = max(bounced, int(task._has_bounce.sum()))
        hits += int(task._has_racket_ball_contact_now.sum())
    torch.cuda.synchronize()
    assert torch.isfinite(env.obs_buf).all() and torch.isfinite(env.rew_buf).all()
    assert bounced > N // 4                       # balls reached the ground on the player's side
    assert (env.progress_buf > 0).any() and (env._num_reset_reaction > 1).any()   # reaction tasks were re-armed (tar_time FSM)
    close(env.obs_buf[:, 0:3], task._root_pos.cpu().numpy(), 0)
    # the fused post kernel agrees with the numpy oracle on the live GPU state
    g = lambda t: t.detach().cpu().numpy()  # noqa: E731
    rbs = g(task._rigid_body_state.view(N, 26, 13))
    obs = V.controller_obs(rbs[:, :25], g(task._root_pos), g(task._root_vel), g(task._racket_normal), g(env._ball_traj),
                           g(env._target_bounce_pos), 10)
    close(env.obs_buf, obs, 2e-6)
    qn = task._rigid_body_rot.norm(dim=-1)
    assert (qn - 1).abs().max() < 1e-4
    assert (task._ball_pos[:, 2] >= 0.0319).all()  # never below the ground


def test_racket_hit_is_detected():
    """aim the ball at the racket face: the swept impact fires, the velocity-jump detector (substeps > 2) or the exact flag sees it"""
    from helpers import SIM_PARAMS, v2p_cfg
    from vid2player3d_b200.tasks import PhysicsMVAEController
    torch.manual_seed(1)
    N = 64
    env = PhysicsMVAEController(v2p_cfg(N), SIM_PARAMS, 1, "cuda", 0, True)
    env.reset()
    task = env._physics_player.task
    env.step(torch.zeros(N, 35, device=DEV))      # one step so the racket row comes from the simulated FK
    n = task._racket_normal
    centre = task._racket_pos + 0.02125 * n
    ball = task._ball_root_states
    ball[:, 0:3] = centre + 0.25 * n
    ball[:, 7:10] = task._racket_vel - 25.0 * n
    ball[:, 10:13] = 0
    task._ball_vel.copy_(ball[:, 7:10])
    v_before = ball[:, 7:10].clone()
    env.step(torch.zeros(N, 35, device=DEV))
    torch.cuda.synchronize()
    assert task._racket_hit_now.float().mean() > 0.9
    dv = (task._ball_root_states[:, 7:10] - v_before).norm(dim=-1)
    assert (dv[task._racket_hit_now] > 20).all()   # restitution 0.9: the normal velocity is reversed


def test_controller_cuda_graph_matches_eager():
    """the captured high-level step replays EXACTLY the eager path: with the deterministic motion player (resident stream + MVAE decoder
    GEMMs), the wgmma policy and the counter-based random walk nothing in a step draws from torch's generator, so after 6 steps +
    resets every state tensor, observation, reward and flag must be bit-identical between eager launches and graph replays"""
    from helpers import SIM_PARAMS, v2p_cfg
    from vid2player3d_b200.tasks import PhysicsMVAEController

    def tensors(obj):
        return {k: v for k, v in vars(obj).items() if isinstance(v, torch.Tensor)}
    outs = []
    for use_graph in (False, True):
        torch.manual_seed(5)
        N = 128
        cfg = v2p_cfg(N, random_walk_in_recovery=True)
        cfg["env"]["motion_player"], cfg["env"]["low_level_policy"] = "stream+decoder", "b200nn"
        env = PhysicsMVAEController(cfg, SIM_PARAMS, 1, "cuda", 0, True)
        env.reset()
        task, player = env._physics_player.task, env._mvae_player
        objs = [env, task, player, player.decoder]
        if use_graph:
            snaps = [{k: v.clone() for k, v in tensors(o).items()} for o in objs]
            env.enable_cuda_graph()                      # warm-up + capture advance the state: restore it
            for snap, o in zip(snaps, objs):
                for k, v in snap.items():
                    getattr(o, k).copy_(v)
        g = torch.Generator(device=DEV).manual_seed(3)
        for i in range(6):
            env.step(torch.clamp(torch.randn(N, 35, device=DEV, generator=g), -5, 5))
            if use_graph and i % 2:
                env.reset_done()                         # device-flag reset (reset graph replay)
            else:
                torch.manual_seed(100 + i)               # the reset draws ball launches from torch's generator: same draws both ways
                env.reset(env.reset_buf.nonzero(as_tuple=False).flatten())
            if i % 2:
                torch.manual_seed(200 + i)
        torch.cuda.synchronize()
        outs.append({n: t.clone() for o in (env, task) for n, t in tensors(o).items()})
        outs[-1]["policy_out"] = env._low_level_policy.out.clone()
    # steps are deterministic; resets consume torch RNG differently between the id-list and the mask-driven path, so compare the
    # tensors no reset draw feeds: the humanoid state, the physics outputs and the low-level policy are functions of the steps alone
    # until a ball is relaunched - compare everything on the envs whose ball was never relaunched in either run
    same = (outs[0]["_num_reset_reaction"] == outs[1]["_num_reset_reaction"]) & (outs[0]["_num_reset_reaction"] <= 1)
    assert int(same.sum()) > 64
    for k in ("_dof_state", "_root_states", "_rigid_body_state", "obs_buf", "_target_dof_pos", "_pd_target_dof_pos"):
        a, b = outs[0][k], outs[1][k]
        n = same.shape[0]
        assert torch.equal(a.view(n, -1)[same], b.view(n, -1)[same]), k
    assert torch.equal(outs[0]["progress_buf"], outs[1]["progress_buf"]) and torch.equal(outs[0]["policy_out"][same], outs[1]["policy_out"][same])
    assert torch.equal(outs[0]["rew_buf"][same], outs[1]["rew_buf"][same]) and torch.equal(outs[0]["reset_buf"], outs[1]["reset_buf"])


def test_fast_task_reset_matches_slow_path():
    """mask-driven per-step task reset (b200v2p_task_reset) vs the id-list path of _reset_envs on the same masks"""
    from helpers import SIM_PARAMS, v2p_cfg
    from vid2player3d_b200.tasks import PhysicsMVAEController
    res = []
    for fast in (False, True):
        torch.manual_seed(11)
        N = 128
        env = PhysicsMVAEController(v2p_cfg(N, use_random_ball_target="discrete"), SIM_PARAMS, 1, "cuda", 0, True)
        env.reset()
        for _ in range(3):
            env.step(torch.zeros(N, 35, device=DEV))
            env.reset(torch.zeros(0, dtype=torch.long, device=DEV))
        env._reset_reaction_buf[:] = False
        env._reset_recovery_buf[:] = False
        env._reset_reaction_buf[::3] = True
        env._reset_recovery_buf[1::4] = True
        task = env._physics_player.task
        task._has_bounce[:] = True
        if fast:
            env._reset_tasks_fast()
        else:
            env._reset_envs_idlist(torch.zeros(0, dtype=torch.long, device=DEV))   # reference-shaped id-list path
        torch.cuda.synchronize()
        res.append(dict(tar_time=env._tar_time.clone(), tar_action=env._tar_action.clone(), nrr=env._num_reset_reaction.clone(),
                        has_bounce=task._has_bounce.clone(), contact=task._has_racket_ball_contact.clone(),
                        cycle=env._mvae_player._swing_type_cycle.clone(), ball=task._ball_root_states.clone(), traj=env._ball_traj.clone(),
                        tot=env._tar_time_total.clone(), tgt=env._target_bounce_pos.clone(), obs=env.obs_buf.clone()))
    a, b = res
    for k in ("tar_time", "tar_action", "nrr", "has_bounce", "contact", "cycle"):
        assert torch.equal(a[k], b[k]), k                          # deterministic bookkeeping is identical
    rea = torch.zeros(128, dtype=torch.bool, device=DEV); rea[::3] = True
    for r in res:                                                    # random draws differ, their ranges / structure must hold
        assert ((r["tot"][rea] >= 65) & (r["tot"][rea] < 75)).all()
        assert (r["ball"][rea, 1] > 11).all() and (r["ball"][rea, 8] < -15).all()
        assert torch.equal(r["traj"][rea][:, 0], r["ball"][rea, 0:3])   # trajectory row 0 = launch position of the chosen pool row
        assert (r["tgt"][rea, 1] == 10).all() and torch.isin(r["tgt"][rea, 0], torch.tensor([-3.0, 0.0, 3.0], device=DEV)).all()
        assert torch.isfinite(r["obs"]).all()
    assert torch.equal(a["ball"][~rea], b["ball"][~rea])


def test_humanoid_reset_kernel_matches_idlist_path():
    """b200v2p_actor_reset (+ counters) vs the reference-shaped indexed-assignment reset for a list of envs"""
    from helpers import SIM_PARAMS, v2p_cfg
    from vid2player3d_b200.tasks import PhysicsMVAEController
    N = 64
    torch.manual_seed(2)
    env = PhysicsMVAEController(v2p_cfg(N), SIM_PARAMS, 1, "cuda", 0, True)
    env.reset()
    for _ in range(4):
        env.step(torch.zeros(N, 35, device=DEV))
    task = env._physics_player.task
    ids = torch.tensor([1, 5, 17, 40], device=DEV)
    env._reset_reaction_buf[:] = False
    env._reset_recovery_buf[:] = False
    player = env._mvae_player
    gen_state = player.gen.get_state()
    before = {k: v.clone() for k, v in (("rs", task._root_states), ("ds", task._dof_state), ("rb", task._rigid_body_state))}
    env._reset_envs(ids)
    torch.cuda.synchronize()
    got = {k: v.clone() for k, v in (("rs", task._root_states), ("ds", task._dof_state), ("rb", task._rigid_body_state),
                                     ("prp", task._prev_target_root_pos), ("prr", task._prev_target_rb_rot), ("pd", task._pd_target_dof_pos))}
    # independent check: FK of the player's (now reset) pose written with plain torch indexing
    tmp = {k: torch.zeros_like(v) for k, v in task._tmp.items()}
    task._smpl_to_sim_into(player._root_pos.contiguous(), player._joint_rotmat, tmp)
    rs = task._humanoid_root_states
    assert torch.equal(rs[ids, 0:3], player._root_pos[ids]) and torch.equal(rs[ids, 3:7], tmp["root_rot"][ids]) and (rs[ids, 7:] == 0).all()
    rbs = task._rigid_body_state.view(N, 26, 13)
    assert torch.equal(rbs[ids, :24, 0:3], tmp["rb_pos"][ids]) and torch.equal(rbs[ids, :24, 3:7], tmp["rb_rot"][ids])
    assert (rbs[ids, :25, 7:] == 0).all()
    assert torch.equal(task._dof_pos[ids], tmp["dof_pos"][ids]) and (task._dof_vel[ids] == 0).all()
    assert torch.equal(got["prr"][ids], tmp["rb_rot"][ids]) and torch.equal(got["pd"][ids], tmp["dof_pos"][ids])
    assert (env.progress_buf[ids] == 0).all() and (env.reset_buf[ids] == 0).all() and (env._num_reset[ids] == 2).all()
    # racket row: wrist pose + rotated offset
    off = torch.tensor(task._model["offset"][24], device=DEV, dtype=torch.float)
    q = tmp["rb_rot"][ids, 22]
    t = 2.0 * torch.cross(q[:, :3], off.expand(len(ids), 3), dim=-1)
    want = tmp["rb_pos"][ids, 22] + off + q[:, 3:4] * t + torch.cross(q[:, :3], t, dim=-1)
    assert (rbs[ids, 24, 0:3] - want).abs().max() < 1e-6
    keep = torch.ones(N, dtype=torch.bool, device=DEV); keep[ids] = False
    assert torch.equal(got["ds"].view(N, -1)[keep], before["ds"].view(N, -1)[keep])      # other envs untouched
    assert torch.equal(got["rb"].view(N, 26, 13)[keep][:, :25], before["rb"].view(N, 26, 13)[keep][:, :25])


def test_fix_head_golden():
    from vid2player3d_b200 import native_v2p as V
    g = golden("v2p_fix_head.npz")
    n = g["rotmat_in"].shape[0]
    mk = lambda: dict(root_rot=torch.zeros(n, 4, device=DEV), dof_pos=torch.zeros(n, 69, device=DEV), root_vel=torch.zeros(n, 3, device=DEV),  # noqa: E731
                      root_ang_vel=torch.zeros(n, 3, device=DEV), dof_vel=torch.zeros(n, 69, device=DEV),
                      rb_pos=torch.zeros(n, 24, 3, device=DEV), rb_rot=torch.zeros(n, 24, 4, device=DEV))
    rest, par, s2m = T(g["rest"]), T(g["parents"], torch.int32), T(g["smpl_2_mujoco"], torch.int32)
    rm = T(g["rotmat_in"])
    a = mk()
    V.smpl_to_sim(T(g["player_root_pos"]), rm, rest, par, s2m, float(g["dt"]), a)
    V.fix_head(a["rb_pos"], a["rb_rot"], T(g["ball_pos"]), T(g["root_pos"]), rm)
    close(rm, g["rotmat_out"], 2e-6)
    b = mk()
    V.smpl_to_sim(T(g["player_root_pos"]), rm, rest, par, s2m, float(g["dt"]), b, prev_root_pos=T(g["prev_target_root_pos"]),
                  prev_rb_rot=T(g["prev_target_rb_rot"]))
    close(b["dof_pos"], g["target_dof_pos"], 2e-5); close(b["rb_pos"], g["target_rb_pos"], 2e-5); close(b["rb_rot"], g["target_rb_rot"], 2e-5)
    close(b["dof_vel"], g["target_dof_vel"], 2e-3)


# ------------------------------------------------------------------------------------------ dual mode (config 5)
def test_ball_in_estimate_golden():
    """b200v2p_ball_in_estimate vs TennisBallInEstimator.estimate run by the reference (tests/golden/v2p_dual.npz)"""
    from vid2player3d_b200 import native_v2p as V
    g = golden("v2p_dual.npz")
    bs = T(g["in_states"])
    n = bs.shape[0]
    ids = torch.arange(n, device=DEV)
    traj, s_in, s_out = torch.zeros(n, 50, 3, device=DEV), torch.zeros(n, 13, device=DEV), torch.zeros(n, 13, device=DEV)
    V.ball_in_estimate(ids, bs, 13, T(g["in_table"]), g["in_params"], traj, s_in, s_out)
    close(traj, g["in_traj"], 1e-5)
    close(s_in, g["in_states_in"], 2e-5)
    close(s_out, g["in_states_out"], 2e-5)
    # index math on the shipped 15 x 50 x 30 x 50 grid: query a table whose row r holds r (split in two float-exact halves)
    rows = 15 * 50 * 30 * 50
    tab = torch.zeros(rows, 50, 2, device=DEV)
    r = torch.arange(rows, device=DEV)
    tab[:, 0, 0], tab[:, 0, 1] = (r // 1024).float(), (r % 1024).float()
    m = g["full_h"].shape[0]
    q = torch.zeros(m, 13, device=DEV)
    q[:, 2], q[:, 8], q[:, 9], q[:, 10] = T(g["full_h"]), T(g["full_vx"]), T(g["full_vy"]), T(g["full_vs"]) * (2 * np.pi)
    traj, s_in, s_out = torch.zeros(m, 50, 3, device=DEV), torch.zeros(m, 13, device=DEV), torch.zeros(m, 13, device=DEV)
    V.ball_in_estimate(torch.arange(m, device=DEV), q, 13, tab, g["in_params_full"], traj, s_in, s_out)
    got = (-traj[:, 0, 1]).round().long() * 1024 + traj[:, 0, 2].round().long()      # o[1] = -(d * dy + y) with dy = 1, y = 0
    same = (got.cpu().numpy() == g["full_index"])
    assert same.mean() > 0.995, same.mean()          # vspin = |omega| / 2pi re-derived on the device: a rounding flip at a cell edge is legal
    snapped = np.stack([s_in[:, 2].cpu().numpy(), -s_in[:, 8].cpu().numpy(), s_in[:, 9].cpu().numpy()], -1)
    assert (np.abs(snapped - g["full_snapped"][:, :3]) < 1e-5).mean() > 0.995


def _dual_env(N, **over):
    from helpers import SIM_PARAMS, v2p_dual_cfg
    from vid2player3d_b200.tasks import PhysicsMVAEControllerDual
    return PhysicsMVAEControllerDual(v2p_dual_cfg(N, **over), SIM_PARAMS, 1, "cuda", 0, True)


def test_dual_reset_balls_golden(monkeypatch):
    """HumanoidSMPLIMMVAEDual._reset_balls vs the reference method (serve + hand-over through the table, mixed parities)"""
    g = golden("v2p_dual.npz")
    env = _dual_env(32, ball_in_table=(g["in_table"], g["in_params"]))
    task = env._physics_player.task
    task._ball_root_states[:] = T(g["rb_states_before"])
    env._mvae_player._racket_pos[:] = T(g["rb_racket_pos"])
    task._has_bounce[:], task._has_racket_ball_contact[:] = True, True
    task._bounce_pos[:] = 1.0
    task._ball_pos[:], task._ball_vel[:] = 0.0, 0.0
    draws = [T(x) for x in g["rb_rand"]]
    monkeypatch.setattr(torch, "rand", lambda *a, **k: draws.pop(0))
    traj = task._reset_balls(T(g["rb_recovery_ids"]), T(g["rb_ball_ids"]))
    monkeypatch.undo()
    close(traj, g["rb_traj"], 1e-5)
    close(task._ball_root_states, g["rb_states_after"], 2e-5)
    close(task._ball_pos, g["rb_ball_pos"], 2e-6)
    close(task._ball_vel, g["rb_ball_vel"], 2e-5)
    close(task._bounce_pos, g["rb_bounce_pos"], 0)
    assert np.array_equal(task._has_bounce.cpu().numpy(), g["rb_has_bounce"])
    assert np.array_equal(task._has_racket_ball_contact.cpu().numpy(), g["rb_has_contact"])
    rbs = task._rigid_body_state.view(32, 26, 13)
    touched = np.concatenate([g["rb_ball_ids"], g["rb_ball_ids"] ^ 1])
    close(rbs[touched, 25, 0:3], g["rb_states_after"][touched, 0:3], 2e-5)           # the simulator-side ball rows follow


def test_dual_compute_reset_golden():
    """the dual reset FSM of the fused post-step kernel vs PhysicsMVAEControllerDual._compute_reset run by the reference"""
    g = golden("v2p_dual.npz")
    N = 128
    env = _dual_env(N)
    env.reset()
    task = env._physics_player.task
    env._tar_action[:] = T(g["cr_tar_action"])
    task._ball_pos[:], task._root_pos[:], task._root_vel[:] = T(g["cr_ball_pos"]), T(g["cr_root_pos"]), T(g["cr_root_vel"])
    env._bounce_in[:], env._distance[:], env.reset_buf[:] = T(g["cr_bounce_in"]), T(g["cr_distance"]), T(g["crreset_buf"])
    task._has_racket_ball_contact[:], task._has_bounce[:] = T(g["cr_has_contact"]), T(g["cr_has_bounce"])
    task._has_bounce_now[:] = False
    term_before = env._terminate_buf.clone()
    env._compute_post()
    assert np.array_equal(env.reset_buf.cpu().numpy(), g["cr_out_reset"])
    assert np.array_equal(env._reset_reaction_buf.cpu().numpy(), g["cr_out_reaction"])
    assert np.array_equal(env._reset_recovery_buf.cpu().numpy(), g["cr_out_recovery"])
    close(env._distance, g["cr_out_distance"], 1e-6)
    assert torch.equal(env._terminate_buf, term_before)              # the dual FSM never writes _terminate_buf


def test_env_slices_match_single_asset():
    """two handles over the even / odd rows with the SAME asset must reproduce the single-handle step bit for bit"""
    from helpers import SIM_PARAMS, v2p_cfg
    from vid2player3d_b200.tasks import HumanoidSMPLIMMVAE
    N = 66                                             # 33 envs per slice: ragged last batch in both kernels
    outs = []
    for assets in ("smpl_mesh_humanoid_federer.xml", ["smpl_mesh_humanoid_federer.xml"] * 2):
        c = v2p_cfg(N)
        pcfg = {"env": dict(numEnvs=N, episodeLength=300, residual_force_scale=31.85, is_train=True, asset=dict(assetFileName=assets),
                            plane=dict(staticFriction=1.0, dynamicFriction=1.0, restitution=0.5), vid2player=c["env"]["vid2player"],
                            keyBodies=[], contactBodies=[]), "sim": {"substeps": 6}}
        t = HumanoidSMPLIMMVAE(pcfg, SIM_PARAMS, 1, "cuda", 0, True)
        gen = torch.Generator(device=DEV).manual_seed(5)
        t._dof_pos[:] = 0.2 * torch.randn(N, 69, device=DEV, generator=gen)
        t._humanoid_root_states[:, 2] = 0.95
        t._ball_root_states[:, 0:3] = torch.tensor([0.0, -8.0, 1.0], device=DEV) + torch.randn(N, 3, device=DEV, generator=gen) * 0.1
        t._ball_root_states[:, 7:10] = torch.tensor([0.0, -20.0, 1.0], device=DEV)
        t._target_dof_pos[:] = t._dof_pos
        t.reset_buf[:] = 0
        for _ in range(3):
            t.step(0.3 * torch.randn(N, t.num_actions, device=DEV, generator=gen))
        torch.cuda.synchronize()
        outs.append([x.clone() for x in (t._root_states, t._dof_state, t._rigid_body_state, t.obs_buf, t._racket_pos, t._ball_pos)])
        assert len(t._envs) == (1 if isinstance(assets, str) else 2)
    for a, b in zip(*outs):
        assert torch.equal(a, b)


def test_dual_end_to_end():
    """config-5 style rollout: federer vs djokovic in paired envs, agent loop with pair resets, ball hand-over through the table"""
    torch.manual_seed(0)
    N = 128
    env = _dual_env(N)
    assert env.num_obs == 257 and env.num_actions == 35
    task = env._physics_player.task
    assert len(task._envs) == 2 and task._rest_t.shape == (2, 24, 3) and not torch.equal(task._rest_t[0], task._rest_t[1])
    assert not torch.equal(task._reset_ref_motion_bodies[0], task._reset_ref_motion_bodies[1])
    env.reset()
    torch.cuda.synchronize()
    assert torch.isfinite(env.obs_buf).all()
    # serve from the near player: even envs react to a ball coming from y > 0, their partners serve and recover
    assert (env._tar_action[::2] == 1).all() and (env._tar_action[1::2] == 0).all()
    bs = task._ball_root_states
    close(bs[::2, 0:2], (-bs[1::2, 0:2]).cpu().numpy(), 1e-6)                 # one ball, seen from both courts
    close(bs[::2, 7:9], (-bs[1::2, 7:9]).cpu().numpy(), 1e-5)
    close(bs[::2, 2], bs[1::2, 2].cpu().numpy(), 0)
    handovers, resets = 0, 0
    for step in range(260):
        env.step(torch.clamp(torch.randn(N, 35, device=DEV), -5, 5))
        done = env.reset_buf.nonzero(as_tuple=False).flatten()
        assert len(done) % 2 == 0 and torch.equal(done[::2] + 1, done[1::2])   # opponents terminate together
        before = env._num_reset_reaction.clone()
        resets += len(done)
        env.reset(done)
        handovers += int(((env._num_reset_reaction - before) > 0).sum()) - len(done) // 2
    torch.cuda.synchronize()
    assert torch.isfinite(env.obs_buf).all() and torch.isfinite(env.rew_buf).all() and torch.isfinite(task._rigid_body_state).all()
    assert resets > 0                                                        # missed balls ended rallies (pairs reset together)
    assert (task._rigid_body_rot.norm(dim=-1) - 1).abs().max() < 1e-4
    assert (task._ball_pos[:, 2] >= 0.0319).all()
    # the two assets are really different bodies: federer and djokovic settle at different pelvis heights / masses
    assert abs(float(task._models[0]["mass"].sum()) - float(task._models[1]["mass"].sum())) > 0.1


def test_left_handed_dual_pair():
    """nadal (left-handed, semi-western) vs federer (right-handed, eastern): per-player wrist / grip / racket head (cfg nadal_federer.yaml)"""
    from helpers import SIM_PARAMS, v2p_dual_cfg
    from oracle import ref_port_v2p as V
    from vid2player3d_b200.tasks import PhysicsMVAEControllerDual
    torch.manual_seed(1)
    N = 32
    cfg = v2p_dual_cfg(N, assets=("smpl_mesh_humanoid_nadal.xml", "smpl_mesh_humanoid_federer.xml"), players=("nadal", "federer"))
    cfg["env"]["vid2player"].update(grip=["semi_western", "eastern"], righthand=[False, True])
    env = PhysicsMVAEControllerDual(cfg, SIM_PARAMS, 1, "cuda", 0, True)
    task = env._physics_player.task
    assert task._racket_wrist_body_id == [17, 22]
    env.reset()
    for _ in range(20):
        env.step(torch.clamp(torch.randn(N, 35, device=DEV), -5, 5))
        env.reset(env.reset_buf.nonzero(as_tuple=False).flatten())
    torch.cuda.synchronize()
    rbs = task._rigid_body_state.view(N, 26, 13).cpu().numpy()
    assert np.isfinite(rbs).all()
    for par, wrist, grip in ((0, 17, 'semi_western'), (1, 22, 'eastern')):
        o = V.update_state_from_sim(rbs[par::2, :25], task._humanoid_root_states[par::2].cpu().numpy(), task._ball_root_states[par::2].cpu().numpy(),
                                    task._ball_vel[par::2].cpu().numpy(), task._has_racket_ball_contact[par::2].cpu().numpy(), grip,
                                    racket_body=24, wrist_body=wrist)
        close(task._racket_normal[par::2], o["racket_normal"], 2e-6)
        close(task._racket_pos[par::2], o["racket_pos"], 0)
    # the welded racket hangs off the left wrist for nadal, off the right wrist for federer (0.5 m along -/+ x of the wrist frame)
    d_l = np.linalg.norm(rbs[0::2, 24, 0:3] - rbs[0::2, 17, 0:3], axis=1)
    d_r = np.linalg.norm(rbs[1::2, 24, 0:3] - rbs[1::2, 22, 0:3], axis=1)
    np.testing.assert_allclose(d_l, 0.5, atol=1e-4)
    np.testing.assert_allclose(d_r, 0.5, atol=1e-4)


def test_ball_body_contact_option_on_gpu():
    """b200_cfg_t::ball_body_contact through the product path (float32 kernels): balls thrown at the torso bounce off it when the
    option is on and fly through when it is off; double kernel == float64 restatement with the option on"""
    from oracle import physics_ref
    from vid2player3d_b200 import abi, model_compiler, native
    mod = model_compiler.canonical_racket_last(model_compiler.load_compiled("smpl_mesh_humanoid_federer"))
    ms, verts = abi.pack_model(mod, float(mod["mass"].sum()) / 90.0)
    names = [str(x) for x in mod["body_names"]]
    n = 32
    rng = np.random.default_rng(8)
    root = np.zeros((n, 13)); root[:, 2] = 2.0; root[:, 3:7] = [0.5, 0.5, 0.5, 0.5]
    q, qd = rng.normal(0, 0.2, (n, 69)), np.zeros((n, 69))
    tar, ext = q.copy(), np.zeros((n, 6))
    tiny = abi.Cfg.from_buffer_copy(abi.make_cfg(mod, substeps=6, ball={}, task_mode=1, pd_mode=1))
    tiny.sim_dt = 1e-12
    rb, _ = physics_ref.control_step(ms, verts, tiny, root.copy(), q.copy(), qd.copy(), tar.copy(), None)
    b = names.index("Chest")
    ball = np.zeros((n, 13))
    d = rng.normal(size=(n, 3)); d /= np.linalg.norm(d, axis=1, keepdims=True)
    ball[:, 0:3] = rb[:, b, 0:3] + 0.25 * d
    ball[:, 7:10] = -15.0 * d
    res = {}
    faces = abi.pack_faces(mod, verts)
    # 0: option off; 1: exact sphere / convex-hull query (hull faces installed, what the task does); 2: no faces - vertex spheres
    for on in (0, 1, 2):
        cfg = abi.make_cfg(mod, substeps=6, ball={"ball_body_contact": int(on > 0)}, task_mode=1, pd_mode=1)
        env = native.Env(ms, verts, cfg, 4, 0)
        if on == 1:
            env.set_hull_faces(*faces)
            physics_ref.set_hull_faces(*faces)
        else:
            physics_ref.clear_hull_faces()
        for dt, prec_tol in ((torch.float32, None), (torch.float64, 1e-8)):
            t = lambda a: torch.tensor(a, dtype=dt, device=DEV).contiguous()  # noqa: E731
            r, qq, vv, tt, ee, bb = t(root), t(q), t(qd), t(tar), t(ext), t(ball)
            rbo, cf = torch.zeros(n, 25, 13, dtype=dt, device=DEV), torch.zeros(n, 25, 3, dtype=dt, device=DEV)
            hits = torch.zeros(n, dtype=torch.int32, device=DEV)
            env.physics_only(r, qq, vv, tt, ee, rbo, cf, n_steps=2, ball=bb, ball_hits=hits)
            torch.cuda.synchronize()
            if prec_tol is not None:
                ro, qo, vo, bo = root.copy(), q.copy(), qd.copy(), ball.copy()
                physics_ref.control_step(ms, verts, cfg, ro, qo, vo, tar.copy(), ext.copy(), n_steps=2, ball=bo, hits=np.zeros(n, np.int32))
                np.testing.assert_allclose(bb.cpu().numpy(), bo, rtol=0, atol=prec_tol)
            else:
                res[on] = bb.cpu().numpy()
    physics_ref.clear_hull_faces()
    assert np.abs(res[1] - res[2]).max() > 1e-4              # the exact hull and the vertex-sphere stand-in are different surfaces
    along_on, along_off = (res[1][:, 7:10] * d).sum(1), (res[0][:, 7:10] * d).sum(1)     # velocity along the approach axis (-15 at launch)
    assert (along_off < -13).all()                          # option off: the ball flies through the body
    assert (along_on > -8).mean() >= 0.9                    # option on: stopped / thrown back by the chest (float64 oracle: -4 .. +6)


def test_stream_motion_player_gather():
    """StreamMotionPlayer (the bench's resident target stream, SURVEY.md 8d): step = gather of frame (t + offset[env]) % K,
    resets re-draw offsets of the listed / masked envs only; rotation matrices stay proper (b200v2p_stream_gather)"""
    from vid2player3d_b200.tasks.physics_mvae_controller import StreamMotionPlayer
    torch.manual_seed(0)
    p = StreamMotionPlayer(12, DEV, seed=4, frames=6)
    ring = p._ring["_joint_rotmat"].view(6, 12, 24, 3, 3)
    env = torch.arange(12, device=DEV)
    for k in range(8):                                   # runs past the end of the stream: wraps
        t0, off = int(p._t), p._off.clone()
        p.step(torch.zeros(12, 32, device=DEV))
        assert torch.equal(p._joint_rotmat, ring[(t0 + 1 + off) % 6, env])
        assert torch.equal(p._root_pos, p._ring["_root_pos"].view(6, 12, 3)[(t0 + 1 + off) % 6, env])
    off = p._off.clone()
    ids = torch.tensor([2, 9], device=DEV)
    p.reset(ids)
    keep = torch.ones(12, dtype=torch.bool, device=DEV)
    keep[ids] = False
    assert torch.equal(p._off[keep], off[keep]) and bool(((p._off >= 0) & (p._off < 6)).all())
    off = p._off.clone()
    mask = torch.zeros(12, dtype=torch.bool, device=DEV)
    mask[[0, 5]] = True
    p.reset_masked(mask)
    assert torch.equal(p._off[~mask], off[~mask])
    assert torch.equal(p._joint_rotmat, ring[(int(p._t) + p._off) % 6, env])
    det = torch.linalg.det(p._joint_rotmat.reshape(-1, 3, 3))
    assert float((det - 1).abs().max()) < 1e-4




def test_pre_step_kernel():
    """b200v2p_pre_step = the action handling of PhysicsMVAEController.pre_physics_step (:247-262): scaling is exact; the envs in
    recovery get fresh N(0,1) draws clamped to +-5 (statistics), different on every launch (device step counter)"""
    from vid2player3d_b200 import native_v2p
    N = 4096
    g = torch.Generator(device=DEV).manual_seed(2)
    actions = torch.randn(N, 35, device=DEV, generator=g)
    tar = (torch.arange(N, device=DEV) % 2).to(torch.long)         # even envs: recovery (tar_action 0)
    mv, rd = torch.zeros(N, 32, device=DEV), torch.zeros(N, 3, device=DEV)
    cnt, done = torch.zeros(1, device=DEV, dtype=torch.long), torch.zeros(1, device=DEV, dtype=torch.int32)
    cfg = dict(n=N, num_actions=35, num_latent=32, num_res_dof=3, random_walk_in_recovery=1, vae_action_scale=1.5, residual_dof_scale=0.4, seed=77)
    t = dict(actions=actions, tar_action=tar, step_counter=cnt, done_counter=done, mvae_actions=mv, res_dof_actions=rd)
    native_v2p.pre_step(cfg, t)
    first = mv.clone()
    assert int(cnt) == 1 and int(done) == 0
    assert torch.equal(mv[1::2], actions[1::2, :32] * 1.5) and torch.equal(rd, actions[:, 32:35] * 0.4)
    r = mv[0::2]
    assert abs(float(r.mean())) < 0.02 and abs(float(r.std()) - 1.0) < 0.02 and float(r.abs().max()) <= 5.0
    assert abs(float((r > 1.0).float().mean()) - 0.1587) < 0.01          # normal tail, not uniform
    native_v2p.pre_step(cfg, t)
    assert int(cnt) == 2 and not torch.equal(mv[0::2], first[0::2]) and torch.equal(mv[1::2], first[1::2])
    cfg["random_walk_in_recovery"] = 0
    native_v2p.pre_step(cfg, t)
    assert torch.equal(mv, actions[:, :32] * 1.5)


def test_obs_imitation_rows_matches_gathered_inputs():
    """b200env_obs_imitation_rows (state rows in place, + the bf16 operand row) == b200env_obs_imitation on contiguous gathers"""
    from vid2player3d_b200.tasks import PhysicsMVAEController
    torch.manual_seed(3)
    env = PhysicsMVAEController(v2p_cfg(96), SIM_PARAMS, 1, "cuda", 0, True)
    env.reset()
    for _ in range(3):
        env.step(torch.clamp(torch.randn(96, env.num_actions, device=DEV), -5, 5))
    task = env._physics_player.task
    rbs = task._rigid_body_state.view(96, 26, 13)
    c = lambda x: x.contiguous()  # noqa: E731
    ref = torch.zeros_like(task.obs_buf)
    task._env.obs_imitation(c(rbs[:, :24, 0:3]), c(rbs[:, :24, 3:7]), task._target_rb_pos, task._target_rb_rot, c(task._dof_pos), c(task._dof_vel),
                            task._target_dof_pos, c(rbs[:, :24, 7:10]), c(rbs[:, :24, 10:13]), task._reset_ref_motion_bodies, True, True, ref)
    out = torch.zeros_like(ref)
    op = torch.zeros(128, 768, device=DEV, dtype=torch.bfloat16)
    mean, rstd = torch.randn(734, device=DEV) * 0.1, torch.rand(734, device=DEV) + 0.5
    task._env.obs_imitation_rows(96, task._rigid_body_state, 26, task._dof_state, task._target_rb_pos, task._target_rb_rot, task._target_dof_pos,
                                 task._reset_ref_motion_bodies, True, True, out, obs_bf16=op, mean=mean, rstd=rstd, clamp=5.0)
    torch.cuda.synchronize()
    d = (out - ref).abs()
    assert torch.equal(out, ref), (float(d.max()), d.nonzero()[:8].tolist(), out[d > 0][:4].tolist(), ref[d > 0][:4].tolist())
    want = torch.clamp((ref - mean) * rstd, -5, 5).to(torch.bfloat16)
    assert torch.equal(op[:96, :734], want) and float(op[96:].abs().max()) == 0 and float(op[:, 734:].abs().max()) == 0

