"""step_kernel_tmem (csrc/packed_t.cuh: 56 envs per SM, the lane-private fields of the bodies in thread-local memory) against
step_kernel_packed (32 envs per SM in the split form, everything in shared-memory records): the same arithmetic in the same order, so the two kernels
are held to EXACT equality - physics only (b200env_physics_only), the embodied_pose task step and the vid2player controller step.
The float64 parity of this form against oracle/physics_ref.c is checked on the CPU lane emulator (tests/test_emu_packed.py, variant
packedt); here the oracle comparison is repeated in float32 through the C ABI."""
import os

import numpy as np
import pytest
import torch

from helpers import SIM_PARAMS, im_cfg

pytestmark = pytest.mark.gpu


class kernel_form:
    """B200ENV_KERNEL for the handles created inside the block (read by b200env_create)"""

    def __init__(self, form):
        self.form = form

    def __enter__(self):
        self.old = os.environ.get("B200ENV_KERNEL")
        os.environ["B200ENV_KERNEL"] = self.form

    def __exit__(self, *a):
        if self.old is None:
            os.environ.pop("B200ENV_KERNEL", None)
        else:
            os.environ["B200ENV_KERNEL"] = self.old


EXACT = os.environ.get("B200_EXPECT_EXACT") == "1"   # builds with -fmad=false: no contraction freedom, the two kernels agree bit for bit


def _same(x, y, name, tol):
    """x == y exactly when EXACT, else within tol (absolute, scaled by max(1, |x|)): the two kernels run the same operations in the same
    order, but nvcc is free to contract a * b + c into FMA differently in differently shaped code"""
    assert torch.isfinite(x.float()).all() and torch.isfinite(y.float()).all(), f"{name}: not finite"
    if EXACT or not x.is_floating_point():
        assert torch.equal(x, y), f"{name} differ: max {float((x.double() - y.double()).abs().max())}"
    else:
        e = ((x - y).abs() / x.abs().clamp(min=1.0)).reshape(x.shape[0], -1).max(dim=1).values   # per env
        d, q99 = float(e.max()), float(torch.quantile(e, 0.99))
        print(f"  {name}: scaled diff max {d:.3e}, 99 % of the envs within {q99:.3e} (tol {tol:g})")
        assert q99 <= tol, f"{name} differ: 99 % quantile {q99:.3e} > {tol:g}"


def _t(a):
    return torch.tensor(a, dtype=torch.float32, device="cuda:0").contiguous()


def _physics(env, n, nb, root, q, qd, tar, ext, steps, ball=None):
    r, qq, vv, tt, ee = _t(root), _t(q), _t(qd), _t(tar), _t(ext)
    rb = torch.zeros(n, nb, 13, device="cuda:0")
    cf = torch.full((n, nb, 3), 7.0, device="cuda:0")
    bb = _t(ball) if ball is not None else None
    hits = torch.zeros(n, dtype=torch.int32, device="cuda:0") if ball is not None else None
    env.physics_only(r, qq, vv, tt, ee, rb, cf, n_steps=steps, ball=bb, ball_hits=hits)
    torch.cuda.synchronize()
    return [r, qq, vv, rb, cf] + ([bb, hits] if ball is not None else [])


@pytest.mark.parametrize("contact", [False, True])
def test_tmem_physics_bit_identical_to_packed(contact):
    from test_gpu_parity import phys_states
    from vid2player3d_b200 import abi, model_compiler, native
    mod = model_compiler.load_compiled("smpl_mesh_humanoid_amass_v1")
    ms, verts = abi.pack_model(mod, float(mod["mass"].sum()) / 90.0)
    cfg = abi.make_cfg(mod)
    n = 24 * 13 + 3                                   # several CTAs of the test kernel, a ragged last warp
    root, q, qd, tar, ext = phys_states(mod, n, 5, contact)
    with kernel_form("packed"):
        e0 = native.Env(ms, verts, cfg, 4, 0)
    with kernel_form("tmem"):
        e1 = native.Env(ms, verts, cfg, 4, 0)
    assert e0.kernel_form == "packed" and e1.kernel_form == "tmem"
    for steps in (1, 3):
        a = _physics(e0, n, ms.nb, root, q, qd, tar, ext, steps)
        b = _physics(e1, n, ms.nb, root, q, qd, tar, ext, steps)
        # random states in deep ground contact (stiff penalty contact) amplify the rounding-level differences of the product build
        tols = (2e-3, 2e-3, 0.2, 0.2, 0.2) if contact else (2e-5, 2e-5, 2e-3, 2e-3, 0.5)
        for x, y, name, tol in zip(a, b, ("root", "dof_pos", "dof_vel", "rigid bodies", "contact forces"), tols):
            _same(x, y, f"{name} after {steps} step(s)", tol * steps)
    if contact:
        assert float(a[4].abs().max()) > 10.0


@pytest.mark.parametrize("asset,ball_body", [("federer", 0), ("federer", 1), ("nadal", 1)])
def test_tmem_ball_physics_bit_identical_to_packed(asset, ball_body):
    from test_gpu_parity import ball_scene
    from vid2player3d_b200 import abi, model_compiler, native
    mod = model_compiler.canonical_racket_last(model_compiler.load_compiled("smpl_mesh_humanoid_" + asset))
    ms, verts = abi.pack_model(mod, float(mod["mass"].sum()) / 90.0)
    cfg = abi.make_cfg(mod, substeps=6, ball={}, task_mode=1, pd_mode=1)
    cfg.ball_body_contact = ball_body
    n = 100
    envs = []
    for form in ("packed", "tmem"):
        with kernel_form(form):
            e = native.Env(ms, verts, cfg, 4, 0)
        if ball_body:
            e.set_hull_faces(*abi.pack_faces(mod, verts))
        envs.append(e)
    assert envs[1].kernel_form == "tmem"
    root, q, qd, tar, ext, ball = ball_scene(mod, ms, verts, cfg, n, 31)
    if ball_body:                                     # a quarter of the balls onto the players' bodies
        rng = np.random.default_rng(3)
        for e in range(3, n, 4):
            ball[e, 0:3] = root[e, 0:3] + rng.normal(0, 0.15, 3) + np.array([0.0, 0.5, 0.0])
            ball[e, 7:10] = [rng.normal(0, 1), -rng.uniform(5, 15), rng.normal(0, 1)]
    for steps in (1, 2):
        a = _physics(envs[0], n, 25, root, q, qd, tar, ext, steps, ball)
        b = _physics(envs[1], n, 25, root, q, qd, tar, ext, steps, ball)
        same = a[6] == b[6]                            # a grazing impact may flip between two float32 evaluations
        assert float(same.float().mean()) > 0.97
        for x, y, name, tol in zip(a[:6], b[:6], ("root", "dof_pos", "dof_vel", "rigid bodies", "contact forces", "ball"), (2e-5, 2e-5, 2e-3, 2e-3, 0.5, 2e-3)):
            _same(x[same], y[same], f"{name} after {steps} step(s)", tol * steps)
    assert int(a[6].sum()) > n // 8                    # racket impacts happened


def test_tmem_physics_f32_vs_oracle():
    """the float32 kernel against the float64 restatement (same tolerances as test_gpu_parity.py::test_physics_f32_random_one_step)"""
    from oracle import physics_ref
    from test_gpu_parity import phys_states
    from vid2player3d_b200 import abi, model_compiler, native
    mod = model_compiler.load_compiled("smpl_mesh_humanoid_amass_v1")
    ms, verts = abi.pack_model(mod, float(mod["mass"].sum()) / 90.0)
    cfg = abi.make_cfg(mod)
    n = 256
    root, q, qd, tar, ext = phys_states(mod, n, 9, False)             # free flight: smooth dynamics, every env within 1e-5 / 1e-3
    with kernel_form("tmem"):
        env = native.Env(ms, verts, cfg, 4, 0)
    r, qq, vv, rb, cf = _physics(env, n, ms.nb, root, q, qd, tar, ext, 1)
    ro, qo, vo = root.copy(), q.copy(), qd.copy()
    physics_ref.control_step(ms, verts, cfg, ro, qo, vo, tar.copy(), ext.copy())
    dq, dr, dv = np.abs(qq.cpu().numpy() - qo).max(), np.abs(r.cpu().numpy()[:, :7] - ro[:, :7]).max(), np.abs(vv.cpu().numpy() - vo).max()
    print(f"  tmem kernel vs float64 restatement: |dq| {dq:.2e} |droot| {dr:.2e} |dqd| {dv:.2e}")
    assert dq < 1e-5 and dr < 1e-5 and dv < 1e-3


def test_tmem_task_step_bit_identical_to_packed():
    """the whole env step (pre_kernel -> physics -> post_kernel) of the embodied_pose task, 12 steps with resets in between"""
    from vid2player3d_b200 import model_compiler, motion_lib
    from vid2player3d_b200.tasks import HumanoidSMPLIM
    model = model_compiler.load_compiled("smpl_mesh_humanoid_amass_v1")
    flat = motion_lib.synthetic(model, num_motions=8, num_frames=90, seed=3)
    n = 56 * 3 + 17                                   # three full CTA batches of the one-wave kernel and a ragged one
    tasks = []
    for form in ("packed", "tmem"):
        with kernel_form(form):
            torch.manual_seed(11)
            tasks.append(HumanoidSMPLIM(im_cfg(n, flat), SIM_PARAMS, 1, "cuda", 0, True))
    assert tasks[0]._env.kernel_form == "packed" and tasks[1]._env.kernel_form == "tmem"
    g = torch.Generator(device="cuda:0").manual_seed(5)
    acts = [torch.rand(n, 75, device="cuda:0", generator=g) * 2 - 1 for _ in range(12)]
    for t in tasks:
        torch.manual_seed(13)
        t.reset()
    for i, a in enumerate(acts):
        for t in tasks:
            t.step(a)
        torch.cuda.synchronize()
        if EXACT:
            for name in ("obs_buf", "rew_buf", "reset_buf", "progress_buf", "_root_states", "_dof_state", "_rigid_body_state", "_contact_forces"):
                _same(getattr(tasks[0], name), getattr(tasks[1], name), f"{name} at step {i}", 0)
        else:   # rounding-level differences grow through contacts: compare the envs whose flags agree, loosely, and the flags mostly
            agree = tasks[0].reset_buf == tasks[1].reset_buf
            assert float(agree.float().mean()) > 0.97
            _same(tasks[0]._dof_state.view(n, -1)[agree], tasks[1]._dof_state.view(n, -1)[agree], f"_dof_state at step {i}", 5e-2)
            _same(tasks[0].rew_buf[agree], tasks[1].rew_buf[agree], f"rew_buf at step {i}", 1e-2)
            for t in tasks[1:]:                       # keep the two runs on the same trajectory: rounding noise must not accumulate over steps
                for name in ("_root_states", "_dof_state", "_rigid_body_state", "progress_buf", "reset_buf", "_terminate_buf"):
                    getattr(t, name).copy_(getattr(tasks[0], name))
        if i == 5:
            ids = torch.arange(0, n, 3, device="cuda:0")
            for t in tasks:
                torch.manual_seed(17)
                t.reset(ids)
    assert float(tasks[1]._contact_forces.abs().max()) > 10.0


def test_tmem_controller_step_bit_identical_to_packed():
    """the vid2player high-level step (humanoid + racket + ball, ball-body contact on): 6 steps"""
    from vid2player3d_b200.configs import v2p_cfg
    from vid2player3d_b200.tasks import PhysicsMVAEController
    n = 120
    envs = []
    for form in ("packed", "tmem"):
        with kernel_form(form):
            torch.manual_seed(21)
            envs.append(PhysicsMVAEController(v2p_cfg(n), SIM_PARAMS, 1, "cuda", 0, True))
    assert envs[1]._physics_player.task._env.kernel_form == "tmem"
    for e in envs:
        torch.manual_seed(23)
        e.reset()
    g = torch.Generator(device="cuda:0").manual_seed(7)
    for i in range(6):
        a = torch.clamp(torch.randn(n, envs[0].num_actions, device="cuda:0", generator=g), -5, 5)
        for e in envs:
            torch.manual_seed(100 + i)
            e.step(a)
        torch.cuda.synchronize()
        t0, t1 = envs[0]._physics_player.task, envs[1]._physics_player.task
        for name, tol in (("_root_states", 1e-3), ("_dof_state", 5e-2), ("_rigid_body_state", 5e-2)):
            _same(getattr(t0, name), getattr(t1, name), f"{name} at step {i}", 0 if EXACT else tol)
            if not EXACT:
                getattr(t1, name).copy_(getattr(t0, name))
        _same(envs[0].obs_buf, envs[1].obs_buf, f"obs_buf at step {i}", 0 if EXACT else 5e-2)
