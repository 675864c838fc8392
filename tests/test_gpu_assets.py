"""Several assets of one topology in one physics launch (b200env_create_assets; HumanoidSMPLIM cfg.env.motion_assets), on the GPU.

Assets: federer + djokovic (25 bodies with the welded Racket), and amass_v1 with scaled variants (lengths, COMs, vertices and radii
times s, masses times s^3, inertias times s^5; the PD gains follow each variant's own mass).

1. Exactness: after several steps every env's rigid-body, root, dof, contact-force, obs, reward and reset rows are bit-identical to
   the same env stepped from the same state and actions by a single-asset handle of its own asset - per-asset counts 1, B-1, B, B+1,
   interleaved assignments (row order != env order), and N = 2 B G + 5 (more batches than CTAs: re-staged headers, a second round).
2. Parity at N = 2 B G + 5 with the float64 restatement (oracle/physics_ref.c) run with every env's own model.
3. End to end: HumanoidSMPLIM with motion_assets (6 motions, 3 distinct assets) through reset and 32 steps against oracle/ref_port.py.
4. Refusals of everything a handle of several assets does not support."""
import numpy as np
import pytest
import torch

from test_gpu_launch import EPW, SENTINEL, _load, _pool, _probe, _read, parity_failures

pytestmark = pytest.mark.gpu

AMASS, FEDERER, DJOKOVIC = "smpl_mesh_humanoid_amass_v1", "smpl_mesh_humanoid_federer", "smpl_mesh_humanoid_djokovic"
STEPS = 3


def scaled(model, s):
    """the asset scaled by s: lengths, COMs, vertices, radii (and so the hull faces' offsets) x s, mass x s^3, inertia x s^5"""
    m = dict(model)
    for k in ("offset", "com", "dyn_com", "verts", "radius"):
        m[k] = model[k] * s
    for k in ("mass", "dyn_mass"):
        m[k] = model[k] * s ** 3
    for k in ("inertia", "dyn_inertia"):
        m[k] = model[k] * s ** 5
    if len(model["prims"]):
        m["prims"] = model["prims"].copy()
        m["prims"][:, 1:8] *= s
    return m


_cache = {}


def _memo(key, fn):
    if key not in _cache:
        _cache[key] = fn()
    return _cache[key]


def _model(name):
    from vid2player3d_b200 import model_compiler
    return _memo(("model", name), lambda: model_compiler.load_compiled(name))


def _lib(num_motions):
    """a synthetic MoCap library on the 24 SMPL bodies (federer / djokovic carry the Racket as a 25th, welded body)"""
    from vid2player3d_b200 import motion_lib
    return _memo(("lib", num_motions), lambda: motion_lib.synthetic(_model(AMASS), num_motions=num_motions, num_frames=60, seed=1))


def _task_class():
    from vid2player3d_b200.tasks import HumanoidSMPLIM

    class FixedIds(HumanoidSMPLIM):
        """HumanoidSMPLIM whose motion ids are given (cfg.env.test_motion_ids) and whose one asset may be a compiled model dict
        (cfg.env.test_model): the tests choose which env runs which asset"""

        def _load_asset(self):
            super()._load_asset()
            m = self.cfg["env"].get("test_model")
            if m is not None:
                self._model = m
                self.humanoid_mass = float(m["mass"].sum())

        def _sample_motion_ids(self):
            return torch.as_tensor(np.asarray(self.cfg["env"]["test_motion_ids"], np.int64), device=self.device).contiguous()
    return FixedIds


def _cfg(base, assets, motion_ids, multi, model=None):
    from helpers import im_cfg
    cfg = im_cfg(len(motion_ids), _lib(len(assets)), asset=f"mjcf/{base}.xml")
    cfg["env"]["test_motion_ids"] = list(motion_ids)
    if multi:
        cfg["env"]["motion_assets"] = list(assets)
    if model is not None:
        cfg["env"]["test_model"] = model
    return cfg


def _multi(base, assets, env_asset):
    """a task of len(env_asset) envs, env e on assets[env_asset[e]] (motion m = asset m)"""
    from helpers import SIM_PARAMS
    torch.manual_seed(0)
    return _task_class()(_cfg(base, assets, env_asset, True), SIM_PARAMS, 1, "cuda", 0, True)


def _single(base, assets, a, motion_ids):
    from helpers import SIM_PARAMS
    torch.manual_seed(0)
    return _task_class()(_cfg(base, assets, motion_ids, False, model=assets[a]), SIM_PARAMS, 1, "cuda", 0, True)


def _run(t, pool, envs):
    """STEPS steps of task t with pool env envs[p] at position p (the same action rows every step); rows by position"""
    a = _load(t, "humanoid", pool, envs)
    for _ in range(STEPS):
        t.step(a)
    torch.cuda.synchronize()
    n = len(envs)
    rows = _read(t, "humanoid", n)
    g = lambda x: x.detach().cpu().numpy().reshape(n, -1).copy()  # noqa: E731
    rows.update(obs=g(t.obs_buf), rew=g(t.rew_buf), reset=g(t.reset_buf), term=g(t._terminate_buf), prog=g(t.progress_buf),
                pd=g(t._pd_target_dof_pos))
    nb = t.num_bodies
    assert not (rows["rb"].reshape(n, -1, 13)[:, :nb] == SENTINEL).any(), "a body row was not written"
    return rows


def _launch_shape(t):
    B, G = t._env.physics_launch_shape
    assert B == 32
    return B, G


def _check_exact(base, assets, env_asset, label):
    from vid2player3d_b200 import native
    env_asset = np.asarray(env_asset)
    pool = _pool("humanoid")
    n = len(env_asset)
    envs = np.arange(n) % len(pool["kind"])
    t = _multi(base, assets, env_asset)
    B, G = _launch_shape(t)
    na, rows_order, batches = t._env.asset_plan
    r2, b2 = native.plan_assets(env_asset, len(assets), B)
    assert na == len(assets) and np.array_equal(rows_order, r2) and np.array_equal(batches, b2)
    got = _run(t, pool, envs)
    del t
    for a in range(len(assets)):
        mine = np.flatnonzero(env_asset == a)
        if not len(mine):
            continue
        ref = _run(_single(base, assets, a, env_asset[mine]), pool, envs[mine])
        for k in ref:
            bad = np.flatnonzero((ref[k].view(np.uint8).reshape(len(mine), -1) != got[k][mine].view(np.uint8).reshape(len(mine), -1)).any(1))
            if len(bad):
                e = int(mine[bad[0]])
                p = int(np.flatnonzero(rows_order == e)[0])
                b = int(np.flatnonzero((batches[:, 1] <= p) & (p < batches[:, 1] + batches[:, 2]))[0])
                raise AssertionError(f"{label}: {len(bad)} of {len(mine)} envs of asset {a} differ in {k} from the single-asset handle; "
                                     f"first env {e}: row position {p}, batch {b} (round {b // G}), slot g {(p - batches[b, 1]) % EPW}")
    rounds = -(-len(batches) // G)
    print(f"\n{label}: N = {n}, {len(assets)} assets, {len(batches)} batches of <= {B}, G = {G}: {rounds} round(s); bit-identical")
    return len(batches), G


@pytest.mark.parametrize("case", ["amass counts around B", "federer + djokovic interleaved"])
def test_rows_match_single_asset_handles(case):
    B = 32
    rng = np.random.default_rng(3)
    if case == "amass counts around B":
        assets = [_model(AMASS), scaled(_model(AMASS), 0.9), scaled(_model(AMASS), 1.1), scaled(_model(AMASS), 1.05)]
        ea = rng.permutation(np.repeat(np.arange(4), [1, B - 1, B, B + 1]))
        base = AMASS
    else:
        assets = [_model(FEDERER), _model(DJOKOVIC)]
        ea = np.arange(2 * B + 3) % 2
        base = FEDERER
    _check_exact(base, assets, ea, case)


def test_rows_match_single_asset_handles_over_two_rounds():
    """N = 2 B G + 5 over three amass variants, assigned at random: more batches than CTAs, so CTAs move to batches of other
    assets (re-staging the header) and a second round runs"""
    t = _memo("probe", lambda: _multi(AMASS, [_model(AMASS)], [0]))
    B, G = _launch_shape(t)
    n = 2 * B * G + 5
    assets = [_model(AMASS), scaled(_model(AMASS), 0.95), scaled(_model(AMASS), 1.08)]
    ea = np.random.default_rng(5).integers(0, 3, n)
    nbat, G = _check_exact(AMASS, assets, ea, "three amass variants at random")
    assert nbat > G


def test_launch_matches_float64_restatement_per_asset():
    """one step at N = 2 B G + 5 over three amass variants against oracle/physics_ref.c run with each env's own model.  Free-flight
    envs are held to the free-flight bounds on every asset; the settled-contact states were settled on the unscaled body, so they are
    held to the settled bounds on that asset only (with the excuse rule of test_gpu_launch.py) and reported on the others; deep
    contact is reported."""
    from oracle import physics_ref, ref_port as R
    t0 = _memo("probe", lambda: _multi(AMASS, [_model(AMASS)], [0]))
    B, G = _launch_shape(t0)
    n = 2 * B * G + 5
    scales = (1.0, 0.95, 1.08)
    assets = [scaled(_model(AMASS), s) if s != 1.0 else _model(AMASS) for s in scales]
    ea = np.random.default_rng(9).integers(0, 3, n)
    pool = {k: v[:n] for k, v in _pool("humanoid").items()}
    t = _multi(AMASS, assets, ea)
    a = _load(t, "humanoid", pool, np.arange(n))
    t.step(a)
    torch.cuda.synchronize()
    rows = _read(t, "humanoid", n)
    pd = t._pd_target_dof_pos.cpu().numpy()
    cfg = t._cfg_struct
    f64 = lambda x: np.ascontiguousarray(x, np.float64)  # noqa: E731
    _, _, force, torque = R.pre_physics(f64(pool["act"]), np.zeros(n), f64(pool["q"]), f64(pool["root"][:, 3:7]), 69,
                                        float(cfg.pd_tar_lim), float(cfg.res_force_scale), float(cfg.res_torque_scale))
    o = dict(root=f64(pool["root"]), q=f64(pool["q"]), qd=f64(pool["qd"]))
    ext = f64(np.concatenate([force, torque], 1))
    for ai, m in enumerate(assets):
        idx = np.flatnonzero(ea == ai)
        ms, verts = t._pack(m)
        r, q, qd = o["root"][idx].copy(), o["q"][idx].copy(), o["qd"][idx].copy()
        physics_ref.control_step(ms, verts, cfg, r, q, qd, f64(pd[idx]), ext[idx].copy())
        o["root"][idx], o["q"][idx], o["qd"][idx] = r, q, qd
    dof = rows["dof"].reshape(n, 69, 2).astype(np.float64)
    k = dict(root=rows["root"].astype(np.float64), q=dof[..., 0], qd=dof[..., 1])
    cls = np.array(["free", "settled", "deep"])[pool["kind"]]
    cls[(pool["kind"] == 1) & (ea != 0)] = "contact"
    # settled envs outside the bound: excused when b200env_physics_only of a single-asset handle of their asset (the launch
    # test_gpu_parity.py validates) gives the same rows bit for bit, as test_gpu_launch.py does (their residual wrench is zero)
    out = (cls == "settled") & ~((np.maximum(np.abs(k["q"] - o["q"]).max(1), np.abs(k["root"] - o["root"]).max(1)) < 1e-4) &
                                  (np.abs(k["qd"] - o["qd"]).max(1) < 2e-3))
    excused = None
    idx = np.flatnonzero(out)
    if len(idx):
        assert not pool["act"][idx, 69:].any()
        T = lambda a: torch.tensor(np.ascontiguousarray(a), dtype=torch.float32, device="cuda:0")  # noqa: E731
        r, q, qd = T(pool["root"][idx]), T(pool["q"][idx]), T(pool["qd"][idx])
        single = _probe("humanoid", "default")
        single._env.physics_only(r, q, qd, T(pd[idx]), T(np.zeros((len(idx), 6))), torch.zeros(len(idx), 24, 13, device="cuda:0"),
                                 torch.zeros(len(idx), 24, 3, device="cuda:0"))
        torch.cuda.synchronize()
        same = (np.array_equal(r.cpu().numpy(), rows["root"][idx]) and
                np.array_equal(np.stack([q.cpu().numpy(), qd.cpu().numpy()], -1).reshape(len(idx), -1), rows["dof"][idx]))
        print(f"\n{len(idx)} settled envs outside the bound {idx.tolist()}: b200env_physics_only gives the same rows bit for bit: {same}")
        if same:
            excused = out
    fails, err = parity_failures(k, o, cls, excused)
    print(f"\nN = {n}, B = {B}, G = {G}; worst |error| against the float64 restatement by asset and kind")
    for ai, s in enumerate(scales):
        for kind in ("free", "settled", "contact", "deep"):
            m = (ea == ai) & (cls == kind)
            if m.any():
                print(f"  scale {s:4.2f} {kind:8s} ({int(m.sum()):4d} envs): " + " ".join(f"{c} {err[c][m].max():.1e}" for c in ("q", "root", "qd")))
    assert not fails, "\n".join(fails)
    # the scaled bodies really are other bodies: the restatement with asset 0's model misses the free-flight envs of the others
    free = np.flatnonzero((pool["kind"] == 0) & (ea == 1))[:64]
    ms, verts = t._pack(assets[0])
    r, q, qd = f64(pool["root"][free]).copy(), f64(pool["q"][free]).copy(), f64(pool["qd"][free]).copy()
    physics_ref.control_step(ms, verts, cfg, r, q, qd, f64(pd[free]), ext[free].copy())
    assert np.abs(q - k["q"][free]).max() > 1e-4


def test_motion_assets_task_end_to_end():
    """6 motions over 3 distinct assets (two entries of each: a file name and the dict it compiles to, two equal dicts, ...): reset
    and 32 steps, obs and reward against ImTaskOracle on the GPU's state rows, the per-env masses and the reference's leftovers"""
    from helpers import SIM_PARAMS, im_cfg, lib_dict
    from oracle import ref_port as R
    from vid2player3d_b200.tasks import HumanoidSMPLIM
    base = _model(AMASS)
    small, big = scaled(base, 0.92), scaled(base, 1.1)
    flat = _lib(6)
    N = 96
    cfg = im_cfg(N, flat)
    cfg["env"]["motion_assets"] = [f"mjcf/{AMASS}.xml", small, big, dict(base), dict(small), dict(big)]
    torch.manual_seed(0)
    task = HumanoidSMPLIM(cfg, SIM_PARAMS, 1, "cuda", 0, True)
    na, _, batches = task._env.asset_plan
    assert na == 3
    mids = task._reset_ref_motion_ids.cpu().numpy()
    assert np.array_equal(task._env_asset, mids % 3) and len(set(task._env_asset.tolist())) == 3
    mass = np.array([float(m["mass"].sum()) for m in (base, small, big)])
    assert np.allclose(task.humanoid_masses, mass[mids % 3])
    last = task._pack((base, small, big)[mids[-1] % 3])[0]
    assert np.array_equal(task.stiffness.cpu().numpy(), np.array(list(last.kp)[:69], np.float32))
    task.reset()
    g = lambda t: t.detach().cpu().numpy().copy()  # noqa: E731
    ml = lib_dict(flat, base)
    orc = R.ImTaskOracle(ml, mids, g(task._cur_ref_motion_times), g(task.progress_buf), g(task.reset_buf), g(task._terminate_buf),
                         np.float32(2) * np.float32(1 / 60), 300, g(task._termination_heights), g(task._contact_body_ids),
                         np.ones(24, np.float32), ml["motion_bodies"][mids])
    gen = torch.Generator(device=task.device).manual_seed(4)
    worst = 0.0
    for _ in range(32):
        a = torch.rand(N, 75, device=task.device, generator=gen) * 2 - 1
        dofs0, rbs0 = g(task._dof_state.view(N, -1, 2)), g(task._rigid_body_state.view(N, -1, 13))
        task.step(a)
        torch.cuda.synchronize()
        orc.pre_physics(g(a), dofs0[..., 0], rbs0[:, 0, 3:7])
        obs, rew, _ = orc.post_physics(g(task._rigid_body_state.view(N, -1, 13)), g(task._dof_state.view(N, -1, 2)))
        assert np.isfinite(g(task.obs_buf)).all()
        d = max(float(np.abs(g(task.obs_buf) - obs).max()), float(np.abs(g(task.rew_buf) - rew).max()))
        worst = max(worst, d)
        assert d < 1e-5, f"obs / reward differ from ImTaskOracle by {d:.3e}"
    print(f"\nmotion_assets: 3 assets, {len(batches)} batches, 32 steps, worst obs / reward |diff| {worst:.2e}")


def test_refusals_on_a_real_handle(monkeypatch):
    from vid2player3d_b200 import abi, native
    t = _multi(AMASS, [_model(AMASS), scaled(_model(AMASS), 0.9)], [0, 1, 1, 0])
    e = t._env
    with pytest.raises(RuntimeError, match="set_env_slice: not supported"):
        e.set_env_slice(0, 2)
    planes, tris, ntris, tmax = abi.pack_faces(t._model, t._verts)
    with pytest.raises(RuntimeError, match="set_hull_faces: not supported"):
        e.set_hull_faces(planes, tris, ntris, tmax)
    z = lambda *s: torch.zeros(*s, device="cuda:0")  # noqa: E731
    with pytest.raises(RuntimeError, match="physics_only: not supported"):
        e.physics_only(z(2, 13), z(2, 69), z(2, 69), z(2, 69), z(2, 6), z(2, 24, 13), z(2, 24, 3))
    models = [t._pack(m)[0] for m in (_model(AMASS), scaled(_model(AMASS), 0.9))]
    verts = [t._pack(m)[1] for m in (_model(AMASS), scaled(_model(AMASS), 0.9))]
    for var, val in (("B200ENV_KERNEL", "lane"), ("B200ENV_KERNEL", "tmem"), ("B200ENV_KERNEL", "packed3"), ("B200ENV_SPLIT", "0"),
                     ("B200ENV_SORT", "1")):
        with monkeypatch.context() as mp:
            mp.setenv(var, val)
            with pytest.raises(RuntimeError, match="default kernel form only"):
                native.Env(models, verts, t._cfg_struct, 4, 0, env_asset=[0, 1, 0, 1])
    fm = [t._pack(_model(n))[0] for n in (FEDERER, DJOKOVIC)]
    fv = [t._pack(_model(n))[1] for n in (FEDERER, DJOKOVIC)]
    with pytest.raises(RuntimeError, match="has_ball is not supported"):
        native.Env(fm, fv, abi.make_cfg(_model(FEDERER), ball={}), 4, 0, env_asset=[0, 1, 0, 1])
    ok = native.Env(models, verts, t._cfg_struct, 4, 0, env_asset=[0, 1, 0, 1])
    assert ok.kernel_form == "packed"
    ok.close()
