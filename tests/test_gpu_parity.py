"""GPU parity tests (run on an H100): CUDA path through the C ABI vs the oracles.

Chain of trust: reference functions -> golden fixtures -> numpy oracle (tests/test_oracle_golden.py)
-> these tests.  The physics half compares against oracle/physics_ref.c (float64 restatement of OUR
model; parity with Isaac Gym / PhysX is unpinned, see DESIGN.md)."""
import numpy as np
import pytest
import torch

from conftest import golden
from helpers import SIM_PARAMS, im_cfg, lib_dict, rand_quat

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def model():
    from vid2player3d_b200 import model_compiler
    return model_compiler.load_compiled("smpl_mesh_humanoid_amass_v1")


@pytest.fixture(scope="module")
def small_lib(model):
    from vid2player3d_b200 import motion_lib
    flat = motion_lib.synthetic(model, num_motions=6, num_frames=60, seed=3, sigma=0.06, ragged=True)
    flat.min_verts_h = np.linspace(-0.02, 0.03, 6).astype(np.float32)
    flat.motion_bodies = np.random.default_rng(5).normal(size=(6, 11)).astype(np.float32)
    return flat


def make_task(n, lib, **kw):
    from vid2player3d_b200.tasks import HumanoidSMPLIM
    return HumanoidSMPLIM(im_cfg(n, lib, **kw), SIM_PARAMS, 1, "cuda", 0, True)


def phys_states(model, n, seed, contact=True):
    rng = np.random.default_rng(seed)
    root = np.zeros((n, 13))
    root[:, 0:2] = rng.uniform(-3, 3, (n, 2))
    root[:, 2] = rng.uniform(0.7, 1.1, n) if contact else rng.uniform(3, 5, n)
    root[:, 3:7] = rand_quat(rng, n)
    root[: n // 2, 3:7] = [0.5, 0.5, 0.5, 0.5]  # upright half
    root[:, 7:10] = rng.normal(0, 0.5, (n, 3))
    root[:, 10:13] = rng.normal(0, 1.0, (n, 3))
    q = rng.normal(0, 0.3, (n, 69))
    qd = rng.normal(0, 1.5, (n, 69))
    tar = q + rng.normal(0, 0.2, (n, 69))
    ext = rng.normal(0, 30, (n, 6))
    return root, q, qd, tar, ext


def run_kernel_physics(task, root, q, qd, tar, ext, dtype, n_steps=1):
    dev = task.device
    t = lambda a: torch.tensor(a, dtype=dtype, device=dev).contiguous()  # noqa: E731
    r, qq, vv, tt, ee = t(root), t(q), t(qd), t(tar), t(ext)
    n = root.shape[0]
    rb = torch.zeros(n, task.num_bodies, 13, dtype=dtype, device=dev)
    cf = torch.zeros(n, task.num_bodies, 3, dtype=dtype, device=dev)
    task._env.physics_only(r, qq, vv, tt, ee, rb, cf, n_steps=n_steps)
    torch.cuda.synchronize()
    return [x.double().cpu().numpy() for x in (r, qq, vv, rb, cf)]


def run_oracle_physics(task, root, q, qd, tar, ext, n_steps=1):
    from oracle import physics_ref
    r, qq, vv = root.copy(), q.copy(), qd.copy()
    rb, cf = physics_ref.control_step(task._model_struct, task._verts, task._cfg_struct, r, qq, vv, tar.copy(), ext.copy(),
                                      n_steps=n_steps)
    return r, qq, vv, rb, cf


@pytest.mark.parametrize("contact", [False, True])
def test_physics_f64_matches_oracle(model, small_lib, contact):
    """same algorithm, float64 on both sides: agreement to round-off over 1 and 8 control steps"""
    task = make_task(4, small_lib)
    st = phys_states(model, 32, 11, contact)
    for steps, tol in ((1, 1e-9), (8, 1e-7)):
        k = run_kernel_physics(task, *st, torch.float64, steps)
        o = run_oracle_physics(task, *st, steps)
        for a, b, name in zip(k, o, ("root", "dof_pos", "dof_vel", "rb", "contact")):
            scale = 1.0 if name != "contact" else 1e3
            np.testing.assert_allclose(a, b, rtol=0, atol=tol * scale, err_msg=f"{name} steps={steps}")
    if contact:
        assert np.abs(o[4]).max() > 10.0  # the contact branch was exercised


def test_physics_f32_config1_drop(model, small_lib):
    """BASELINE config 1: one humanoid, default pose (identity root at z=0.89), zero action, 60 control
    steps incl. ground impact; float32 kernel vs float64 restatement, tolerance 1e-4 on q and 1e-3 on qd
    (north_star: joint q/qd within 1e-4 - qd is held to 1e-3 through the impact, see DESIGN.md)."""
    task = make_task(4, small_lib)
    root = np.zeros((1, 13)); root[0, 2] = 0.89; root[0, 6] = 1.0
    q = np.zeros((1, 69)); qd = np.zeros((1, 69)); tar = np.zeros((1, 69)); ext = np.zeros((1, 6))
    worst_q = worst_qd = 0.0
    for steps in (10, 30, 60):
        k = run_kernel_physics(task, root, q, qd, tar, ext, torch.float32, steps)
        o = run_oracle_physics(task, root, q, qd, tar, ext, steps)
        worst_q = max(worst_q, np.abs(k[1] - o[1]).max(), np.abs(k[0][:, :7] - o[0][:, :7]).max())
        worst_qd = max(worst_qd, np.abs(k[2] - o[2]).max())
    print(f"config1 drop: max |dq| {worst_q:.3e}  max |dqd| {worst_qd:.3e}")
    assert o[0][0, 2] < 0.3 and np.abs(o[4]).max() > 100  # it did land
    assert worst_q < 1e-4
    assert worst_qd < 1e-3


def settled_contact_states(task, model, n, seed, settle_steps=25):
    """physically reachable contact states: drop random poses from ~1.4 m and let the float64 restatement run
    `settle_steps` control steps, so bodies rest on / slide over the ground with natural penetrations."""
    from oracle import physics_ref
    rng = np.random.default_rng(seed)
    root, q, qd, tar, ext = phys_states(model, n, seed, False)
    root[:, 2] = rng.uniform(1.1, 1.5, n)
    root[:, 7:13] *= 0.3
    qd *= 0.3
    physics_ref.control_step(task._model_struct, task._verts, task._cfg_struct, root, q, qd, tar, None, n_steps=settle_steps)
    return root, q, qd, tar, np.zeros_like(ext)


def test_physics_f32_random_one_step(model, small_lib):
    """float32 kernel vs float64 restatement, one control step from 256 random states:
    (a) free flight (smooth dynamics): every env within 1e-5 / 1e-3;
    (b) natural ground contact: the model is non-smooth (a hull vertex is in or out, friction regularisation),
        so a small fraction of envs may flip a vertex; the bulk must agree to 1e-4 on q."""
    task = make_task(4, small_lib)
    st = phys_states(model, 256, 6, False)
    k = run_kernel_physics(task, *st, torch.float32, 1)
    o = run_oracle_physics(task, *st, 1)
    assert np.abs(k[1] - o[1]).max() < 1e-5 and np.abs(k[0] - o[0]).max() < 1e-5
    assert np.abs(k[2] - o[2]).max() < 1e-3
    st = settled_contact_states(task, model, 256, 5)
    k = run_kernel_physics(task, *st, torch.float32, 1)
    o = run_oracle_physics(task, *st, 1)
    eq = np.maximum(np.abs(k[1] - o[1]).max(axis=1), np.abs(k[0] - o[0]).max(axis=1))
    ev = np.abs(k[2] - o[2]).max(axis=1)
    print(f"contact states: |dq| median {np.median(eq):.2e} p95 {np.quantile(eq, 0.95):.2e} max {eq.max():.2e}; "
          f"|dqd| median {np.median(ev):.2e} p95 {np.quantile(ev, 0.95):.2e} max {ev.max():.2e}; "
          f"contact force max {np.abs(o[4]).max():.0f} N")
    assert np.abs(o[4]).max() > 50.0
    assert eq.max() < 1e-4
    assert np.quantile(ev, 0.95) < 5e-4 and ev.max() < 2e-3


def test_motion_state_golden():
    """b200env_motion_state vs fixtures from the reference's MotionLib.get_motion_state"""
    from vid2player3d_b200 import motion_lib
    g = golden("motion_state.npz")
    flat = motion_lib.FlatMotionLib(**{k[4:]: g[k] for k in g if k.startswith("lib_")})
    task = make_task(4, flat)
    dev = task.device
    n = len(g["motion_ids"])
    ids = torch.tensor(g["motion_ids"], device=dev)
    times = torch.tensor(g["motion_times"], device=dev)
    shapes = dict(root_pos=(n, 3), root_rot=(n, 4), dof_pos=(n, 69), root_vel=(n, 3), root_ang_vel=(n, 3), dof_vel=(n, 69),
                  key_pos=(n, 4, 3), rb_pos=(n, 24, 3), rb_rot=(n, 24, 4))
    out = {k: torch.zeros(*s, device=dev) for k, s in shapes.items()}
    task._env.motion_state(ids, times, out)
    for k in shapes:
        np.testing.assert_allclose(out[k].cpu().numpy(), g[k], rtol=0, atol=1e-5, err_msg=k)


def test_obs_imitation_golden(small_lib):
    """b200env_obs_imitation vs fixtures from the reference's compute_humanoid_observations_imitation (1e-5)"""
    g = golden("obs_imitation.npz")
    task = make_task(4, small_lib)
    names = ("body_pos", "body_rot", "target_pos", "target_rot", "dof_pos", "dof_vel", "target_dof_pos", "body_vel",
             "body_ang_vel", "motion_bodies")
    args = [torch.tensor(g[k], device=task.device) for k in names]
    obs = task.compute_imitation_obs(*args, True, True)
    np.testing.assert_allclose(obs.cpu().numpy(), g["obs"], rtol=0, atol=1e-5)
    obs = task.compute_imitation_obs(*args, False, False)
    np.testing.assert_allclose(obs.cpu().numpy(), g["obs_nolocal_noheight"], rtol=0, atol=1e-5)
    jp = task.compute_imitation_obs(*args, True, True, obs_type='joint_pos')   # :853-915
    assert jp.shape[1] == 513
    np.testing.assert_allclose(jp.cpu().numpy(), g["obs_jpos"], rtol=0, atol=1e-5)


def snapshot(task):
    g = lambda t: t.detach().cpu().numpy().copy()  # noqa: E731
    return dict(root=g(task._root_states), dofs=g(task._dof_state.view(task.num_envs, -1, 2)),
                rbs=g(task._rigid_body_state.view(task.num_envs, -1, 13)), obs=g(task.obs_buf), rew=g(task.rew_buf),
                sub=g(task._sub_rewards), reset=g(task.reset_buf), term=g(task._terminate_buf), prog=g(task.progress_buf),
                times=g(task._cur_ref_motion_times), t_dof=g(task._target_dof_pos), t_dofv=g(task._target_dof_vel),
                t_rbp=g(task._target_rb_pos), t_rbr=g(task._target_rb_rot), t_key=g(task._target_key_pos),
                t_rootp=g(task._target_root_pos), t_rootr=g(task._target_root_rot), t_rootv=g(task._target_root_vel),
                pd=g(task._pd_target_dof_pos), acts=g(task.actions), cf=g(task._contact_forces))


def close_expmap(a, b, atol=1e-5):
    """exp-map joint coordinates from the reference's float32 quat_to_exp_map (torch_utils.py:82-120): for joint
    angles below ~1e-3 rad, sin_theta = sqrt(1 - w*w) is quantised to {0, 3.4e-4, ...} and the result jumps between
    0 and ~1e-3 on a 1-ulp change of w, so such entries (|value| < 2e-3) are only held to 2e-3; the rest to 1e-5."""
    tiny = (np.abs(a) < 2e-3) & (np.abs(b) < 2e-3)
    np.testing.assert_allclose(a[~tiny], b[~tiny], rtol=0, atol=atol)
    np.testing.assert_allclose(a[tiny], b[tiny], rtol=0, atol=2e-3)
    assert (np.abs(a - b) > atol).mean() < 0.01


def test_fused_step_vs_oracle(model, small_lib):
    """reset + 12 fused steps on 64 envs vs (numpy task oracle + float64 physics oracle), re-synchronised to
    the GPU state every step so that each step's arithmetic is checked in isolation."""
    from oracle import physics_ref, ref_port as R
    torch.manual_seed(0)
    N = 64
    task = make_task(N, small_lib, episodeLength=10)
    ml = lib_dict(small_lib, model)
    task.reset()
    torch.cuda.synchronize()
    s = snapshot(task)
    mids = task._reset_ref_motion_ids.cpu().numpy()
    t0 = task._reset_ref_motion_times.cpu().numpy()
    # reset state = MoCap state at t0 (humanoid_smpl_im.py:489-528)
    ms = R.get_motion_state(ml, mids, t0)
    np.testing.assert_allclose(s["root"][:, 0:3], ms[0], atol=1e-5)
    np.testing.assert_allclose(s["root"][:, 3:7], ms[1], atol=1e-5)
    close_expmap(s["dofs"][..., 0], ms[2])
    np.testing.assert_allclose(s["root"][:, 7:10], ms[3], atol=1e-5)
    np.testing.assert_allclose(s["dofs"][..., 1], ms[5], atol=1e-5)
    np.testing.assert_allclose(s["rbs"][..., 0:3], ms[7], atol=1e-5)
    np.testing.assert_allclose(s["rbs"][..., 3:7], ms[8], atol=1e-5)
    assert np.all(s["rbs"][..., 7:] == 0) and np.all(s["prog"] == 0) and np.all(s["reset"] == 0) and np.all(s["term"] == 0)
    np.testing.assert_allclose(s["obs"], R.compute_humanoid_obs_raw(s["rbs"][..., 0:3], s["rbs"][..., 3:7], s["dofs"][..., 0],
                                                                   s["dofs"][..., 1], s["rbs"][..., 7:10], s["rbs"][..., 10:13],
                                                                   ml["motion_bodies"][mids]), atol=1e-6)
    orc = R.ImTaskOracle(ml, mids, s["times"], s["prog"], s["reset"], s["term"], np.float32(2) * np.float32(1.0 / 60.0), 10,
                         task._termination_heights.cpu().numpy(), task._contact_body_ids.cpu().numpy(),
                         np.ones(24, np.float32), ml["motion_bodies"][mids])
    close_expmap(s["t_dof"], orc.t_dof_pos)
    np.testing.assert_allclose(s["t_rbp"], orc.t_rb_pos, atol=1e-5)
    n_reset_seen = 0
    for step in range(12):
        actions = torch.clamp(torch.randn(N, 75, device=task.device), -1, 1)
        if step == 3:
            actions[:, :69] *= 3
        before = s
        task.step(actions)
        torch.cuda.synchronize()
        s = snapshot(task)
        a_used, pd, f, tq = orc.pre_physics(actions.cpu().numpy(), before["dofs"][..., 0], before["rbs"][:, 0, 3:7])
        np.testing.assert_allclose(s["acts"], a_used, atol=0)
        np.testing.assert_allclose(s["pd"], pd, atol=1e-6)
        # physics: float64 oracle from the same pre-step state
        root = before["root"].astype(np.float64); q = before["dofs"][..., 0].astype(np.float64).copy()
        qd = before["dofs"][..., 1].astype(np.float64).copy()
        ext = np.concatenate([f, tq], -1).astype(np.float64)
        rb, cf = physics_ref.control_step(task._model_struct, task._verts, task._cfg_struct, root, q, qd, pd.astype(np.float64), ext)
        np.testing.assert_allclose(s["root"], root, atol=2e-4, err_msg=f"root step {step}")
        np.testing.assert_allclose(s["dofs"][..., 0], q, atol=2e-4, err_msg=f"q step {step}")
        np.testing.assert_allclose(s["dofs"][..., 1], qd, atol=5e-3, err_msg=f"qd step {step}")
        np.testing.assert_allclose(s["rbs"], rb, atol=5e-3, err_msg=f"rb step {step}")
        # task logic on the GPU's own post-physics state: obs / reward / reset / targets within 1e-5
        obs, rew, sub = orc.post_physics(s["rbs"], s["dofs"])
        np.testing.assert_allclose(s["obs"], obs, atol=1e-6)
        np.testing.assert_allclose(s["rew"], rew, atol=1e-5)
        np.testing.assert_allclose(s["sub"], sub, atol=1e-5)
        assert np.array_equal(s["reset"], orc.reset_buf) and np.array_equal(s["term"], orc.terminate_buf)
        assert np.array_equal(s["prog"], orc.progress)
        np.testing.assert_allclose(s["times"], orc.ref_times, atol=1e-6)
        close_expmap(s["t_dof"], orc.t_dof_pos)
        np.testing.assert_allclose(s["t_dofv"], orc.t_dof_vel, atol=1e-5)
        np.testing.assert_allclose(s["t_rbp"], orc.t_rb_pos, atol=1e-5)
        np.testing.assert_allclose(s["t_rbr"], orc.t_rb_rot, atol=1e-5)
        np.testing.assert_allclose(s["t_key"], orc.t_key_pos, atol=1e-5)
        np.testing.assert_allclose(s["t_rootp"], orc.t_root_pos, atol=1e-5)
        np.testing.assert_allclose(s["t_rootr"], orc.t_root_rot, atol=1e-5)
        np.testing.assert_allclose(s["t_rootv"], orc.t_root_vel, atol=1e-5)
        n_reset_seen = int(s["reset"].sum())
    assert n_reset_seen == N  # episodeLength 10: every env hit the sticky reset flag, rewards went to zero
    assert np.all(s["rew"] == 0)


def test_full_size_properties(model):
    """BASELINE size (8192 envs): determinism, finiteness, obs/state consistency, resets."""
    from vid2player3d_b200 import motion_lib
    flat = motion_lib.synthetic(model, num_motions=64, num_frames=300, seed=7)
    N = 8192
    outs = []
    for rep in range(2):
        torch.manual_seed(123)
        task = make_task(N, flat, episodeLength=300)
        task.reset()
        g = torch.Generator(device=task.device).manual_seed(9)
        for step in range(40):
            a = torch.rand(N, 75, device=task.device, generator=g) * 2 - 1
            task.step(a)
        torch.cuda.synchronize()
        outs.append((task.obs_buf.clone(), task.rew_buf.clone(), task.reset_buf.clone(), task._root_states.clone()))
    for a, b in zip(*outs):
        assert torch.equal(a, b)  # bit-identical across runs (no atomics, fixed reduction order)
    obs, rew, reset, root = outs[0]
    assert torch.isfinite(obs).all() and torch.isfinite(rew).all()
    assert (rew >= 0).all() and (rew <= 1.0 + 1e-6).all()
    assert torch.equal(obs[:, :72], task._rigid_body_pos.reshape(N, -1))
    assert torch.equal(obs[:, 72:168], task._rigid_body_rot.reshape(N, -1))
    assert torch.equal(obs[:, 168:237], task._dof_pos)
    assert torch.equal(obs[:, 237:306], task._dof_vel)
    qn = task._rigid_body_rot.norm(dim=-1)
    assert (qn - 1).abs().max() < 1e-4
    assert task._env.launch_count >= 41


def test_empty_and_partial_reset(model, small_lib):
    task = make_task(16, small_lib)
    task.reset()
    task.reset(torch.zeros(0, dtype=torch.long, device=task.device))  # empty id list is a no-op
    for _ in range(3):
        task.step(torch.zeros(16, 75, device=task.device))
    torch.cuda.synchronize()
    before = task.progress_buf.clone()
    ids = torch.tensor([3, 7], device=task.device)
    task.reset(ids)
    torch.cuda.synchronize()
    assert task.progress_buf[3] == 0 and task.progress_buf[7] == 0
    keep = torch.ones(16, dtype=torch.bool, device=task.device); keep[ids] = False
    assert torch.equal(task.progress_buf[keep], before[keep])
    assert task.context_feat.shape == (16, 48, 378) and task.context_mask.shape == (16, 48)


def test_missing_arguments_fail_loudly(small_lib):
    from vid2player3d_b200 import native
    task = make_task(4, small_lib)
    with pytest.raises(RuntimeError):
        native._check(native.lib().b200env_step(task._env._h, None, None))


# --------------------------------------------------------------------------------------- ball + racket (vid2player)
def make_ball_env(n=4, substeps=6, asset="federer"):
    """native env on a vid2player asset (24 bodies + welded Racket; nadal = left-handed, tilted head) with the tennis ball enabled"""
    from vid2player3d_b200 import abi, model_compiler, native
    mod = model_compiler.canonical_racket_last(model_compiler.load_compiled("smpl_mesh_humanoid_" + asset))
    ms, verts = abi.pack_model(mod, float(mod["mass"].sum()) / 90.0)
    cfg = abi.make_cfg(mod, substeps=substeps, ball={}, task_mode=1, pd_mode=1)
    return mod, ms, verts, cfg, native.Env(ms, verts, cfg, n, 0)


def ball_scene(mod, ms, verts, cfg, n, seed):
    """random flying humanoids; balls aimed at the racket head (half), at the ground with spin (quarter), free (rest)"""
    import ctypes
    from oracle import physics_ref
    from vid2player3d_b200 import abi
    root, q, qd, tar, ext = phys_states(mod, n, seed, False)
    root[:, 2] = np.random.default_rng(seed).uniform(1.5, 2.5, n)
    tiny = abi.Cfg.from_buffer_copy(cfg)
    tiny.sim_dt = 1e-12
    r0, q0, v0 = root.copy(), q.copy(), qd.copy()
    rb, _ = physics_ref.control_step(ms, verts, tiny, r0, q0, v0, tar.copy(), None)
    rng = np.random.default_rng(seed + 1)
    ball = np.zeros((n, 13)); ball[:, 6] = 1
    from scipy.spatial.transform import Rotation
    for e in range(n):
        Rr = Rotation.from_quat(rb[e, 24, 3:7]).as_matrix() @ Rotation.from_quat(list(cfg.racket_head_quat)).as_matrix()   # head frame
        pr, vr = rb[e, 24, 0:3], rb[e, 24, 7:10]
        kind = e % 4
        if kind in (0, 1):
            side = 1.0 if kind == 0 else -1.0
            off = np.array(list(cfg.racket_head_center)) + np.array([rng.uniform(-0.08, 0.08), side * rng.uniform(0.06, 0.10), rng.uniform(-0.08, 0.08)])
            ball[e, 0:3] = pr + Rr @ off
            ball[e, 7:10] = vr + Rr @ np.array([rng.normal(0, 3), -side * rng.uniform(15, 30), rng.normal(0, 3)])
            ball[e, 10:13] = rng.normal(0, 40, 3)
        elif kind == 2:
            ball[e, 0:3] = [rng.uniform(-3, 3), rng.uniform(-3, 3), rng.uniform(0.033, 0.08)]
            ball[e, 7:10] = [rng.normal(0, 8), rng.normal(0, 8), -rng.uniform(0.05, 12)]
            ball[e, 10:13] = rng.normal(0, 60, 3)
        else:
            ball[e, 0:3] = [rng.uniform(-3, 3), rng.uniform(5, 9), rng.uniform(1, 2)]
            ball[e, 7:10] = [rng.normal(0, 2), -rng.uniform(20, 30), rng.normal(2, 2)]
            ball[e, 10:13] = rng.normal(0, 40, 3)
    return root, q, qd, tar, ext, ball


@pytest.mark.parametrize("substeps,asset", [(2, "federer"), (6, "federer"), (6, "nadal")])
def test_ball_physics_f64_matches_oracle(substeps, asset):
    """humanoid + welded racket + ball (aero, swept racket impact with reaction on the wrist, ground bounce):
    double-precision kernel vs float64 restatement, 1 and 3 control steps"""
    from oracle import physics_ref
    mod, ms, verts, cfg, env = make_ball_env(4, substeps, asset)
    n = 64
    root, q, qd, tar, ext, ball = ball_scene(mod, ms, verts, cfg, n, 17)
    for steps, tol in ((1, 1e-9), (3, 1e-7)):
        t = lambda a: torch.tensor(a, dtype=torch.float64, device="cuda:0").contiguous()  # noqa: E731
        r, qq, vv, tt, ee, bb = t(root), t(q), t(qd), t(tar), t(ext), t(ball)
        rb = torch.zeros(n, 25, 13, dtype=torch.float64, device="cuda:0")
        cf = torch.zeros(n, 25, 3, dtype=torch.float64, device="cuda:0")
        hits = torch.zeros(n, dtype=torch.int32, device="cuda:0")
        env.physics_only(r, qq, vv, tt, ee, rb, cf, n_steps=steps, ball=bb, ball_hits=hits)
        torch.cuda.synchronize()
        ro, qo, vo, bo = root.copy(), q.copy(), qd.copy(), ball.copy()
        ho = np.zeros(n, np.int32)
        rbo, _ = physics_ref.control_step(ms, verts, cfg, ro, qo, vo, tar.copy(), ext.copy(), n_steps=steps, ball=bo, hits=ho)
        assert np.array_equal(hits.cpu().numpy(), ho)
        np.testing.assert_allclose(bb.cpu().numpy(), bo, rtol=0, atol=tol * 10)
        np.testing.assert_allclose(r.cpu().numpy(), ro, rtol=0, atol=tol)
        np.testing.assert_allclose(qq.cpu().numpy(), qo, rtol=0, atol=tol)
        np.testing.assert_allclose(vv.cpu().numpy(), vo, rtol=0, atol=tol * 100)
        np.testing.assert_allclose(rb.cpu().numpy(), rbo, rtol=0, atol=tol * 100)
    assert (ho > 0).sum() >= n // 4            # racket impacts happened ...
    hit = ho > 0
    assert np.all(np.linalg.norm(bo[hit, 7:10] - ball[hit, 7:10], axis=1) > 5.0)   # ... and turned the ball around
    ground = np.arange(n) % 4 == 2
    assert np.all(bo[ground, 2] >= cfg.ball_radius - 1e-9)


def test_ball_physics_f32_vs_oracle():
    from oracle import physics_ref
    mod, ms, verts, cfg, env = make_ball_env(4, 6)
    n = 64
    root, q, qd, tar, ext, ball = ball_scene(mod, ms, verts, cfg, n, 23)
    t = lambda a: torch.tensor(a, dtype=torch.float32, device="cuda:0").contiguous()  # noqa: E731
    r, qq, vv, tt, ee, bb = t(root), t(q), t(qd), t(tar), t(ext), t(ball)
    rb = torch.zeros(n, 25, 13, device="cuda:0"); cf = torch.zeros(n, 25, 3, device="cuda:0")
    hits = torch.zeros(n, dtype=torch.int32, device="cuda:0")
    env.physics_only(r, qq, vv, tt, ee, rb, cf, n_steps=1, ball=bb, ball_hits=hits)
    torch.cuda.synchronize()
    ro, qo, vo, bo = root.copy(), q.copy(), qd.copy(), ball.copy()
    ho = np.zeros(n, np.int32)
    physics_ref.control_step(ms, verts, cfg, ro, qo, vo, tar.copy(), ext.copy(), ball=bo, hits=ho)
    same = hits.cpu().numpy() == ho                      # a grazing impact may flip in float32
    assert same.mean() > 0.95
    np.testing.assert_allclose(bb.cpu().numpy()[same, 0:3], bo[same, 0:3], rtol=0, atol=1e-4)
    np.testing.assert_allclose(bb.cpu().numpy()[same, 7:10], bo[same, 7:10], rtol=0, atol=2e-3)
    np.testing.assert_allclose(qq.cpu().numpy()[same], qo[same], rtol=0, atol=1e-4)


def test_motion_context_matches_torch_composition(model, small_lib):
    """b200env_motion_context (one launch, writes context_feat / context_mask in place) vs the reference-shaped composition
    (b200env_motion_state over the 48-frame window + torch.cat + indexed assignment, humanoid_smpl_im.py:530-563): bit-identical"""
    task = make_task(64, small_lib)
    task.reset()
    for env_ids in (torch.arange(64, device=task.device), torch.tensor([3, 17, 18, 40, 63], device=task.device)):
        mids = task._reset_ref_motion_ids[env_ids]
        times = task.sample_time(mids).contiguous()
        task._init_context(env_ids, mids, times)
        feat, mask = task._init_context_torch(env_ids, mids, times)
        assert torch.equal(task.context_feat[env_ids], feat) and torch.equal(task.context_mask[env_ids], mask)
        assert feat.shape[1:] == (48, 378) and mask.any() and torch.isfinite(feat).all()
    assert not task.context_mask.all()        # windows reaching past the end of short motions are masked out


def test_vec_task_graph_step_equals_eager_step(model, small_lib):
    """VecTaskPython.enable_cuda_graph: the captured step (clamp -> 3 launches -> clamp) leaves the same buffers as the eager one"""
    from vid2player3d_b200.tasks import VecTaskPythonWrapper
    outs = []
    for use_graph in (False, True):
        torch.manual_seed(5)
        task = make_task(96, small_lib)
        vec = VecTaskPythonWrapper(task, task.device, 5.0, 1.0)
        g = torch.Generator(device=task.device).manual_seed(9)
        acts = [torch.rand(96, task.num_actions, device=task.device, generator=g) * 4 - 2 for _ in range(6)]   # beyond the clip range
        buf = torch.zeros_like(acts[0])
        if use_graph:
            assert vec.enable_cuda_graph(buf) is buf      # its warm-up steps the envs: enable before the reset that starts a rollout
        vec.reset()
        rec = []
        for i, a in enumerate(acts):
            buf.copy_(a)
            obs, rew, reset, extras = vec.step(buf if i % 2 == 0 else a)     # the static buffer and a foreign tensor
            rec.append((obs.clone(), rew.clone(), reset.clone(), extras["terminate"].clone()))
            if i == 3:
                vec.reset(torch.arange(0, 96, 3, device=task.device))
        outs.append(rec)
    for (o1, r1, d1, t1), (o2, r2, d2, t2) in zip(*outs):
        assert torch.equal(o1, o2) and torch.equal(r1, r2) and torch.equal(d1, d2) and torch.equal(t1, t2)
    assert float(outs[0][-1][0].abs().max()) <= 5.0


def test_no_residual_wrench_action_width(model, small_lib):
    """residual_force_scale = 0 (the code's own default, humanoid_smpl_im.py:39,111): the action rows are nd = 69 wide.  The step
    must use that stride (ADVICE r1: a hard-coded nd + 6 read misaligned rows and wrote past the tensors) and give exactly what the
    75-wide task gives with zero residual columns."""
    N = 96
    torch.manual_seed(11)
    ta = make_task(N, small_lib)
    torch.manual_seed(11)
    tb = make_task(N, small_lib, residual_force_scale=0.0)
    assert ta.num_actions == 75 and tb.num_actions == 69 and tuple(tb.actions.shape) == (N, 69)
    torch.manual_seed(12)
    ta.reset()
    torch.manual_seed(12)
    tb.reset()
    assert torch.equal(ta._dof_pos, tb._dof_pos)
    g = torch.Generator(device=ta.device).manual_seed(3)
    for _ in range(4):
        a = torch.rand(N, 69, device=ta.device, generator=g) * 2 - 1
        ta.step(torch.cat([a, torch.zeros(N, 6, device=ta.device)], 1))
        tb.step(a)
        torch.cuda.synchronize()
        assert torch.equal(tb.actions, ta.actions[:, :69])
        for name in ("_dof_pos", "_dof_vel", "obs_buf", "rew_buf", "reset_buf", "_pd_target_dof_pos"):
            assert torch.equal(getattr(ta, name), getattr(tb, name)), name
    with pytest.raises(ValueError):
        tb.step(torch.zeros(N, 75, device=tb.device))


def test_init_context_golden():
    """b200env_motion_context (+ the torch `_transform_target`) vs the fixture produced by the reference's own `_init_context` /
    `_transform_target` run on a fake self (tests/golden/make_golden_context.py; humanoid_smpl_im.py:530-592)."""
    from vid2player3d_b200 import motion_lib
    g = golden("init_context.npz")
    flat = motion_lib.FlatMotionLib(**{k[4:]: g[k] for k in g if k.startswith("lib_")})
    n = len(g["plain_ids"])
    for case, over in (("plain", {}), ("mask", {"transform_specs": {"mask_joints": {"joints": [str(j) for j in g["mask_joints"]]}}})):
        task = make_task(n, flat, **over)
        dev = task.device
        ids, times = torch.tensor(g[f"{case}_ids"], device=dev), torch.tensor(g[f"{case}_times"], device=dev)
        task._reset_ref_motion_ids[:] = ids
        task._init_context(torch.arange(n, device=dev), ids, times)
        torch.cuda.synchronize()
        assert tuple(task.context_feat.shape) == g[f"{case}_feat"].shape
        np.testing.assert_allclose(task.context_feat.cpu().numpy(), g[f"{case}_feat"], rtol=0, atol=1e-5, err_msg=case)
        assert np.array_equal(task.context_mask.cpu().numpy(), g[f"{case}_mask"]), case
        assert task.context_names[-1] == ("joint_conf" if over else "dof_pos_gt")
    # the two random transforms: invariants of :573-590 (confidence in [0, 1], dropped joints zeroed in body_pos only, root kept by
    # mask_random_joints, ground-truth columns untouched)
    specs = {"noisy_joints": {"noise_std": 0.05, "prob": 0.5, "conf_std": 0.05, "min_conf": 0.2}, "mask_random_joints": {"prob": 0.3}}
    task = make_task(n, flat, transform_specs=specs)
    ids, times = torch.tensor(g["plain_ids"], device=task.device), torch.tensor(g["plain_times"], device=task.device)
    torch.manual_seed(0)
    task._init_context(torch.arange(n, device=task.device), ids, times)
    f = task.context_feat.cpu().numpy()
    conf, bp, gt = f[..., 378:], f[..., :72].reshape(n, 48, 24, 3), g["plain_feat"]
    assert conf.min() >= 0.0 and conf.max() <= 1.0 and (conf == 0).mean() > 0.2 and (conf == 1).mean() > 0.1
    assert np.all(bp[conf == 0] == 0.0)
    np.testing.assert_allclose(f[..., 72:378], gt[..., 72:], rtol=0, atol=1e-5)
    clean = conf == 1.0
    np.testing.assert_allclose(bp[clean], gt[..., :72].reshape(n, 48, 24, 3)[clean], rtol=0, atol=1e-5)


def test_kernel_double_matches_jacobian_equations_of_motion(model):
    """GPU twin of tests/test_physics_anchor.py: the product kernel's device code instantiated for double, ONE contact-free substep,
    against the joint-space equations of motion assembled from body Jacobians (no articulated-body recursion in the reference):
    (M + diag(armature + h kd + h^2 kp)) du/dt = kp (target - q - h qd) - kd qd - c(q, u)."""
    from test_physics_anchor import Tree, implicit_reference, random_state
    from vid2player3d_b200 import abi, native
    m, verts = abi.pack_model(model, float(model["mass"].sum()) / 90.0)
    cfg = abi.make_cfg(model, sim_dt=1.0 / 120.0, substeps=1, control_freq_inv=1, ang_damping=0.0, max_ang_vel=1e6)
    h = float(cfg.sim_dt)
    n = 128
    env = native.Env(m, verts, cfg, n, 0)
    root, q, qd, tar = random_state(np.random.default_rng(3), n, 69)
    t = lambda a: torch.tensor(a, dtype=torch.float64, device="cuda:0").contiguous()  # noqa: E731
    r, qq, vv, tt = t(root), t(q), t(qd), t(tar)
    rb, cf = torch.zeros(n, 24, 13, dtype=torch.float64, device="cuda:0"), torch.zeros(n, 24, 3, dtype=torch.float64, device="cuda:0")
    env.physics_only(r, qq, vv, tt, torch.zeros(n, 6, dtype=torch.float64, device="cuda:0"), rb, cf, n_steps=1)
    torch.cuda.synchronize()
    r1, v1 = r.cpu().numpy(), vv.cpu().numpy()
    tree = Tree(m)
    worst = 0.0
    for i in range(n):
        u, ud, _ = implicit_reference(tree, root[i], q[i], qd[i], tar[i], h, cfg.gravity_z)
        u1 = np.concatenate([r1[i, 10:13], r1[i, 7:10], v1[i]])
        worst = max(worst, np.abs((u1 - u) / h - ud).max() / (1.0 + np.abs(ud).max()))
    assert worst < 1e-9, worst
