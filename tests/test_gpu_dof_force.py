"""DOF force sensor on the GPU (include/b200env.h b200_buffers_t::dof_force, b200env_physics_only's dof_force_out; csrc/packed.cuh
pk_dof_force): the double instantiation against the float64 restatement, the float step launch against the sensor's definition within
float32 bounds, the env slices of dual mode, no effect on the motion, CUDA-graph replay, the refusals of the A/B kernel forms and the
task-level tensor.  The restatement side and the definition are those of tests/test_dof_force.py."""
import numpy as np
import pytest
import torch

from test_dof_force import restatement_dof_force, sensor_from_state, start_of_last_substep, with_tight_limits, model_arrays
from test_emu_packed import states

U32 = 2.0 ** -24


def _amass_task(n, sensors=True, seed=0, **env_over):
    from helpers import SIM_PARAMS, im_cfg
    from test_gpu_launch import _flat
    from vid2player3d_b200.tasks import HumanoidSMPLIM
    cfg = im_cfg(n, _flat(), **env_over)
    if sensors:
        cfg["env"]["dof_force_sensors"] = True
    torch.manual_seed(seed)
    return HumanoidSMPLIM(cfg, SIM_PARAMS, 1, "cuda", 0, True)


def _ball_task(n, handles=1, sensors=True, seed=0):
    from helpers import SIM_PARAMS
    from test_gpu_launch import _ball_cfg
    from vid2player3d_b200.tasks import HumanoidSMPLIMMVAE
    cfg = _ball_cfg(n, handles)
    if sensors:
        cfg["env"]["dof_force_sensors"] = True
    torch.manual_seed(seed)
    return HumanoidSMPLIMMVAE(cfg, SIM_PARAMS, 1, "cuda", 0, True)


def _actions(t, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.rand(t.num_envs, t.get_action_size(), device="cuda", generator=g) * 2 - 1).contiguous()


def float_bound(ms, cfg, q, qdp, tar):
    """float32 bound of the sensor row the float kernel reports against the definition evaluated in float64 on the kernel's own end
    state: q at the start of the last substep is recovered from the float32 dof row (exp / log in float32 on the kernel side, each a
    few units of round-off of the angle, |q| <= pi + 1) and qd+ from the float32 velocity; each operand carries at most 16 u of
    relative error, and the sum of the magnitudes of the terms bounds the error of the result"""
    a = model_arrays(ms)
    h = float(cfg.sim_dt) / cfg.substeps
    k, c = float(cfg.limit_k), float(cfg.limit_c)
    mag = a["kp"] * (np.abs(tar) + np.abs(q) + 4.0 + h * np.abs(qdp)) + a["kd"] * np.abs(qdp)
    mag = mag + k * (np.maximum(np.abs(a["lim_lo"]), np.abs(a["lim_hi"])) + np.abs(q) + 4.0 + h * np.abs(qdp)) + c * np.abs(qdp)
    return 16 * U32 * mag


def _check_float_rows(t, tau, what):
    """tau [N, nd] float32 rows of the step against the definition on the task's own end state, within float_bound; DOFs within
    1e-4 of a limit (the branch may go either way in float32) are left out"""
    ms, cfg = t._model_struct, t._cfg_struct
    q = t._dof_pos.double().cpu().numpy()
    qd = t._dof_vel.double().cpu().numpy()
    pd = t._pd_target_dof_pos.double().cpu().numpy()
    qs, qdp = start_of_last_substep(ms, cfg, q, qd)
    ref = sensor_from_state(ms, cfg, qs, qdp, pd)
    bound = float_bound(ms, cfg, qs, qdp, pd)
    a = model_arrays(ms)
    edge = (np.abs(qs - a["lim_lo"]) < 1e-4) | (np.abs(qs - a["lim_hi"]) < 1e-4)
    err = np.abs(tau.astype(np.float64) - ref)
    ratio = np.where(edge, 0.0, err / bound)
    print(f"\n{what}: N = {len(tau)}, worst error / bound = {ratio.max():.3f}, max |tau| = {np.abs(ref).max():.1f}, "
          f"{int(edge.sum())} DOFs at a limit edge left out")
    assert ratio.max() <= 1.0, (what, np.unravel_index(ratio.argmax(), ratio.shape), err.max())


@pytest.mark.gpu
@pytest.mark.parametrize("wl", ["humanoid", "ball"])
def test_float_step_launch_within_bounds(wl):
    """the step's physics launch at N = 2 B G + 5 (two rounds and a ragged batch): every sensor row against the definition evaluated
    in float64 on the step's own end state, within the float32 bound; finite, and the drive does work"""
    probe = _amass_task(1) if wl == "humanoid" else _ball_task(1)
    B, G = probe._env.physics_launch_shape
    assert B == 32
    n = 2 * B * G + 5
    t = _amass_task(n) if wl == "humanoid" else _ball_task(n)
    if wl == "humanoid":
        t.reset()
    for s in range(3):
        t.step(_actions(t, s))
    torch.cuda.synchronize()
    tau = t.dof_force_tensor.cpu().numpy()
    assert np.isfinite(tau).all()
    assert float((t.dof_force_tensor * t._dof_vel).sum().abs()) > 0.0
    _check_float_rows(t, tau, wl)


def _phys_inputs(ms, n, seed, contact=True):
    root, q, qd, tar, ext = states(n, seed, contact)
    return root, q, qd, tar, ext


@pytest.mark.gpu
@pytest.mark.parametrize("wl", ["humanoid", "ball"])
def test_double_instantiation_matches_restatement(wl):
    """b200env_physics_only in float64 with dof_force_out, states in contact with active limits: the rows equal the restatement's to
    1e-9 of each env's torque scale"""
    from vid2player3d_b200 import abi, model_compiler, native
    if wl == "humanoid":
        mod = model_compiler.load_compiled("smpl_mesh_humanoid_amass_v1")
        cfg_kw = {}
    else:
        mod = model_compiler.canonical_racket_last(model_compiler.load_compiled("smpl_mesh_humanoid_federer"))
        cfg_kw = dict(substeps=6, ball={}, task_mode=1, pd_mode=1)
    ms, verts = abi.pack_model(mod, float(mod["mass"].sum()) / 90.0)
    ms = with_tight_limits(ms)
    cfg = abi.make_cfg(mod, **cfg_kw)
    n = 256
    root, q, qd, tar, ext = _phys_inputs(ms, n, 41)
    ball = hits = None
    if wl == "ball":
        rng = np.random.default_rng(3)
        ball = np.zeros((n, 13))
        ball[:, 0:3] = root[:, 0:3] + rng.normal(0, 0.6, (n, 3)) + [0, 0.5, 0.3]
        ball[:, 2] = np.abs(ball[:, 2]) + 0.04
        ball[:, 7:10] = rng.normal(0, 8, (n, 3))
        hits = np.zeros(n, np.int32)
    env = native.Env(ms, verts, cfg, n, 0)
    T = lambda a: torch.tensor(a, device="cuda:0").contiguous()  # noqa: E731
    r, qq, vv, tt, ee = T(root), T(q), T(qd), T(tar), T(ext)
    rb, cf = torch.zeros(n, ms.nb, 13, dtype=torch.float64, device="cuda:0"), torch.zeros(n, ms.nb, 3, dtype=torch.float64, device="cuda:0")
    tau = torch.full((n, ms.nd), float("nan"), dtype=torch.float64, device="cuda:0")
    bb = T(ball) if ball is not None else None
    hh = torch.zeros(n, dtype=torch.int32, device="cuda:0") if ball is not None else None
    env.physics_only(r, qq, vv, tt, ee, rb, cf, n_steps=1, ball=bb, ball_hits=hh, dof_force=tau)
    torch.cuda.synchronize()
    ref = restatement_dof_force(ms, verts, cfg, root.copy(), q.copy(), qd.copy(), tar.copy(), ext.copy(),
                                ball=ball.copy() if ball is not None else None, hits=hits)
    got = tau.cpu().numpy()
    scale = np.maximum(1.0, np.abs(ref).max(1, keepdims=True))
    worst = (np.abs(got - ref) / scale).max()
    print(f"\n{wl}: worst |tau - restatement| / row scale = {worst:.2e}")
    assert worst < 1e-9
    # the same launch without the sensor: identical state rows
    r2, q2, v2 = T(root), T(q), T(qd)
    rb2, cf2 = torch.zeros_like(rb), torch.zeros_like(cf)
    bb2 = T(ball) if ball is not None else None
    hh2 = torch.zeros_like(hh) if hh is not None else None
    env.physics_only(r2, q2, v2, tt, ee, rb2, cf2, n_steps=1, ball=bb2, ball_hits=hh2)
    for x, y in ((r, r2), (qq, q2), (vv, v2), (rb, rb2), (cf, cf2)) + (((bb, bb2),) if bb is not None else ()):
        assert torch.equal(x, y)


def _rows(t):
    out = [t._root_states, t._dof_state, t._rigid_body_state, t._contact_force_tensor, t.obs_buf, t.rew_buf, t.reset_buf, t.progress_buf,
           t._terminate_buf]
    return [x.clone() for x in out]


@pytest.mark.gpu
def test_sensor_does_not_change_the_step():
    """sensor on against off, 50 steps of the imitation task with the same actions: every state, observation, reward and flag row
    bit-identical"""
    n = 777
    on, off = _amass_task(n, True, seed=3), _amass_task(n, False, seed=3)
    for t in (on, off):
        torch.manual_seed(4)
        t.reset()
    assert not off.dof_force_tensor.any()
    for s in range(50):
        a = _actions(on, 100 + s)
        on.step(a)
        off.step(a)
    torch.cuda.synchronize()
    for x, y in zip(_rows(on), _rows(off)):
        assert torch.equal(x, y)
    assert not off.dof_force_tensor.any() and on.dof_force_tensor.abs().max() > 0


@pytest.mark.gpu
def test_graph_replay_and_storage():
    """the step captured in a CUDA graph replays to the rows of the eager step; dof_force_tensor keeps its storage through steps,
    replays and resets"""
    n = 300
    eager, graphed = _amass_task(n, seed=5), _amass_task(n, seed=5)
    for t in (eager, graphed):
        torch.manual_seed(6)
        t.reset()
    ptr = graphed.dof_force_tensor.data_ptr()
    a0 = _actions(eager, 1)
    eager.step(a0)
    graphed.step(a0)                        # warm-up outside the capture
    static = torch.zeros_like(a0)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        graphed.step(static)
    # the capture ran nothing: replay the steps 2..6 on the graphed task, eager on the other
    for s in range(2, 7):
        a = _actions(eager, s)
        eager.step(a)
        static.copy_(a)
        g.replay()
    torch.cuda.synchronize()
    assert torch.equal(eager.dof_force_tensor, graphed.dof_force_tensor)
    assert torch.equal(eager._dof_state, graphed._dof_state)
    assert graphed.dof_force_tensor.data_ptr() == ptr
    ids = torch.arange(0, n, 7, device="cuda")
    graphed.reset(ids)
    graphed.step(_actions(graphed, 9))
    torch.cuda.synchronize()
    assert graphed.dof_force_tensor.data_ptr() == ptr and torch.isfinite(graphed.dof_force_tensor).all()


@pytest.mark.gpu
def test_dual_mode_slices():
    """dual mode, one handle per player over the same tensors: stepping handle k fills rows k, k + 2, ... and leaves every bit of the
    other player's rows as it was"""
    n = 2 * 70
    t = _ball_task(n, handles=2)
    assert len(t._envs) == 2
    a = _actions(t, 2)
    t.dof_force_tensor.fill_(float("nan"))
    t._envs[0].step(a)
    torch.cuda.synchronize()
    df = t.dof_force_tensor
    assert torch.isfinite(df[0::2]).all() and torch.isnan(df[1::2]).all()
    even = df[0::2].clone()
    t._envs[1].step(a)
    torch.cuda.synchronize()
    assert torch.isfinite(df).all() and torch.equal(df[0::2], even)
    t.step(a)
    torch.cuda.synchronize()
    _check_float_rows(t, df.cpu().numpy(), "dual")


@pytest.mark.gpu
@pytest.mark.parametrize("form", [dict(B200ENV_KERNEL="tmem"), dict(B200ENV_KERNEL="lane"), dict(B200ENV_SPLIT="0")])
def test_ab_forms_refuse_the_sensor(form, monkeypatch):
    """the A/B kernel forms have no sensor: the task's bind and b200env_physics_only refuse it with the documented error; without the
    sensor the same task builds"""
    for k in ("B200ENV_KERNEL", "B200ENV_SPLIT", "B200ENV_SORT"):
        monkeypatch.delenv(k, raising=False)
    for k, v in form.items():
        monkeypatch.setenv(k, v)
    with pytest.raises(RuntimeError, match="DOF force sensor .* runs in the default kernel form only"):
        _amass_task(8)
    t = _amass_task(8, sensors=False)
    z = lambda *s: torch.zeros(*s, device="cuda:0")  # noqa: E731
    with pytest.raises(RuntimeError, match="DOF force sensor .* runs in the default kernel form only"):
        t._env.physics_only(z(2, 13), z(2, 69), z(2, 69), z(2, 69), z(2, 6), z(2, 24, 13), z(2, 24, 3), dof_force=z(2, 69))


@pytest.mark.gpu
def test_task_tensor_equals_physics_only():
    """task level: dof_force_tensor after a step equals b200env_physics_only's sensor on the same inputs (the step's PD targets and
    residual wrench, the state before the step), within the float32 bound and bit-identical where the two launches agree on the state"""
    n = 200
    t = _amass_task(n, seed=8, residual_force_scale=0.0)     # no residual wrench: physics_only gets the step's inputs exactly
    torch.manual_seed(9)
    t.reset()
    t.step(_actions(t, 3))
    torch.cuda.synchronize()
    root0, q0, qd0 = t._root_states.clone(), t._dof_pos.clone().contiguous(), t._dof_vel.clone().contiguous()
    a = _actions(t, 4)
    t.step(a)
    torch.cuda.synchronize()
    pd = t._pd_target_dof_pos.clone()
    ext = torch.zeros(n, 6, device="cuda:0")
    rb, cf = torch.zeros(n, 24, 13, device="cuda:0"), torch.zeros(n, 24, 3, device="cuda:0")
    tau = torch.zeros(n, 69, device="cuda:0")
    r, q, qd = root0.clone(), q0.clone(), qd0.clone()
    t._env.physics_only(r, q, qd, pd, ext, rb, cf, dof_force=tau)
    torch.cuda.synchronize()
    same_state = (q == t._dof_pos).all(1) & (qd == t._dof_vel).all(1)
    print(f"\n{int(same_state.sum())} of {n} envs with the same end state in both launches")
    assert same_state.sum() > n // 2
    assert torch.equal(tau[same_state], t.dof_force_tensor[same_state])
    _check_float_rows(t, t.dof_force_tensor.cpu().numpy(), "task")


def _assets_rows(monkeypatch, plan, assets, ea, envs, pool, single=None):
    """sensor rows after the steps of tests/test_gpu_assets.py::_run: a handle of several assets in the given plan, or (single = a) a
    one-asset handle of asset a running the envs of that asset"""
    import test_gpu_assets as TA
    from helpers import SIM_PARAMS
    if single is None:
        monkeypatch.setenv("B200ENV_ASSET_PLAN", plan)
        cfg = TA._cfg(TA.AMASS, assets, ea, True)
    else:
        monkeypatch.delenv("B200ENV_ASSET_PLAN", raising=False)
        cfg = TA._cfg(TA.AMASS, assets, ea, False, model=assets[single])
    cfg["env"]["dof_force_sensors"] = True
    torch.manual_seed(0)
    t = TA._task_class()(cfg, SIM_PARAMS, 1, "cuda", 0, True)
    if single is None:
        assert t._env.asset_plan_mixed == (plan == "mixed")
    TA._run(t, pool, envs)
    rows = t.dof_force_tensor.cpu().numpy().copy()
    del t
    return rows


@pytest.mark.gpu
def test_same_rows_across_asset_plans(monkeypatch):
    """several assets in one handle (64 scaled bodies at random over B G + 5 envs: two rounds): the grouped and the mixed plan give
    sensor rows bit-identical to each other and to one-asset handles of the envs' bodies"""
    import test_gpu_assets as TA
    from test_gpu_launch import _pool
    B, G = _amass_task(1)._env.physics_launch_shape
    n, S = B * G + 5, 64
    base = TA._model(TA.AMASS)
    assets = [base] + [TA.scaled(base, 0.88 + 0.24 * i / (S - 1)) for i in range(1, S)]
    ea = np.random.default_rng(S).integers(0, S, n)
    pool = _pool("humanoid")
    envs = np.arange(n) % len(pool["kind"])
    mixed = _assets_rows(monkeypatch, "mixed", assets, ea, envs, pool)
    grouped = _assets_rows(monkeypatch, "grouped", assets, ea, envs, pool)
    assert np.isfinite(mixed).all() and np.abs(mixed).max() > 0
    assert np.array_equal(mixed.view(np.uint32), grouped.view(np.uint32))
    for a in (0, 1, S - 1):
        mine = np.flatnonzero(ea == a)
        one = _assets_rows(monkeypatch, None, assets, ea[mine], envs[mine], pool, single=a)
        assert np.array_equal(mixed[mine].view(np.uint32), one.view(np.uint32)), f"asset {a}"
    print(f"\nN = {n}, S = {S}: mixed, grouped and one-asset sensor rows bit-identical")
