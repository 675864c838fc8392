"""DOF force sensor (include/b200env.h b200_buffers_t::dof_force, csrc/packed.cuh::pk_dof_force) on the CPU lane emulator (tests/emu):
the device code of the sensor instantiation, compiled as host C++ in float64, against

- the float64 restatement oracle/physics_ref.c: its own articulated solve (full 6x6 matrices, Cholesky root solve) gives the state at
  the end of the control step; the joint state at the start of the last substep and the implicit drive's velocity follow from it
  exactly (q_start = q_end (x) exp(-h qd_end), qd+ = qd_end / damp: the integrator's last joint update run backwards), and the
  definition of the sensor is evaluated on them (`restatement_dof_force`);
- the joint-space equations of motion of tests/test_physics_anchor.py, which share nothing with ABA:
  tau = (M(q) + diag(armature)) qdd + c(q, u) over the joint rows, with and without active joint limits.

The sensor must also leave the motion alone: every state row with it is bit-identical to the step without it."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "emu"))

from oracle import physics_ref  # noqa: E402
from test_emu_packed import states  # noqa: E402
from test_physics_anchor import Tree, random_state, rodrigues  # noqa: E402
from vid2player3d_b200 import abi, model_compiler  # noqa: E402


def _p(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


def emu_lib():
    """tests/emu/emu_dof_force.cpp with the flags of tests/emu/build.py (the library also exports emu_packed_physics)"""
    import build as emu_build
    out = os.path.join(emu_build.HERE, "build", "libemu_dof_force.so")
    src = os.path.join(emu_build.HERE, "emu_dof_force.cpp")
    deps = [src, os.path.join(emu_build.HERE, "emu_packed.cpp"), os.path.join(emu_build.HERE, "cuda_compat.h")] + \
        [os.path.join(emu_build.CSRC, f) for f in os.listdir(emu_build.CSRC) if f.endswith(".cuh")]
    if not (os.path.exists(out) and all(os.path.getmtime(s) <= os.path.getmtime(out) for s in deps)):
        os.makedirs(os.path.dirname(out), exist_ok=True)
        cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
        subprocess.check_call([cxx, "-O1", "-std=c++17", "-pthread", "-shared", "-fPIC", "-x", "c++", "-Wno-unknown-pragmas",
                               "-ffp-contract=off", "-DEMU_PACKED=1", "-o", out, src])
    lib = C.CDLL(out)
    lib.emu_set_hull_faces(None, None, None, C.c_int(0))
    return lib


def emu_step(ms, verts, cfg, root, q, qd, tar, ext, n_steps=1, sensor=True, ball=None, hits=None):
    """in place on float64 root / q / qd (/ ball, hits); returns (rb, contact, dof_force or None)"""
    lib = emu_lib()
    n = root.shape[0]
    rb, cf = np.zeros((n, ms.nb, 13)), np.zeros((n, ms.nb, 3))
    args = [C.byref(ms), _p(np.ascontiguousarray(verts, np.float32)), C.byref(cfg), C.c_int(n), C.c_int(n_steps), _p(root), _p(q), _p(qd),
            _p(tar), _p(ext), _p(rb), _p(cf), _p(ball), _p(hits)]
    if not sensor:
        assert lib.emu_packed_physics(*args) == 0
        return rb, cf, None
    tau = np.full((n, ms.nd), np.nan)
    assert lib.emu_dof_force_physics(*args, _p(tau)) == 0
    return rb, cf, tau


def model_arrays(ms):
    nd = ms.nd
    return {k: np.array([getattr(ms, k)[d] for d in range(nd)], np.float64) for k in ("kp", "kd", "armature", "lim_lo", "lim_hi")}


def sensor_from_state(ms, cfg, q, qdp, tar):
    """the definition of the sensor (include/b200env.h) at joint coordinates q (start of the last substep) and implicit velocity qd+,
    in float64: kp (pd - q - h qd+) - kd qd+ [+ limk (lim - q - h qd+) - limc qd+ while a limit is active]"""
    a = model_arrays(ms)
    h = float(cfg.sim_dt) / cfg.substeps
    tau = a["kp"] * (tar - q - h * qdp) - a["kd"] * qdp
    lo, hi = q < a["lim_lo"], q > a["lim_hi"]
    k, c = float(cfg.limit_k), float(cfg.limit_c)
    tau = np.where(lo, tau + k * (a["lim_lo"] - q - h * qdp) - c * qdp, tau)
    tau = np.where(hi, tau + k * (a["lim_hi"] - q - h * qdp) - c * qdp, tau)
    return tau


def start_of_last_substep(ms, cfg, q_end, qd_end):
    """(q at the start of the last substep, qd+ = qd + h qdd) from the state at the end of the control step: the last joint update
    qj_end = qj (x) exp(h qd_end), qd_end = damp (qd + h qdd) run backwards (valid while |qd_end| stays below the clamp)"""
    from scipy.spatial.transform import Rotation
    h = float(cfg.sim_dt) / cfg.substeps
    damp = 1.0 - h * float(cfg.ang_damping)
    n, nd = q_end.shape
    assert np.linalg.norm(qd_end.reshape(n, -1, 3), axis=-1).max() < float(cfg.max_ang_vel)
    qs = (Rotation.from_rotvec(q_end.reshape(-1, 3)) * Rotation.from_rotvec(-h * qd_end.reshape(-1, 3))).as_rotvec().reshape(n, nd)
    return qs, qd_end / damp


def restatement_dof_force(ms, verts, cfg, root, q, qd, tar, ext=None, ball=None, hits=None):
    """one control step of oracle/physics_ref.c (in place) and the sensor of its last substep"""
    physics_ref.control_step(ms, verts, cfg, root, q, qd, tar, ext, ball=ball, hits=hits)
    qs, qdp = start_of_last_substep(ms, cfg, q, qd)
    return sensor_from_state(ms, cfg, qs, qdp, tar)


def with_tight_limits(ms, every=4, lim=0.2):
    """every `every`-th DOF gets the limits [-lim, lim], so that random poses (q ~ N(0, 0.3)) push some of them past a limit"""
    for d in range(0, ms.nd, every):
        ms.lim_lo[d], ms.lim_hi[d] = -lim, lim
    return ms


@pytest.fixture(scope="module")
def amass():
    mod = model_compiler.load_compiled("smpl_mesh_humanoid_amass_v1")
    ms, verts = abi.pack_model(mod, float(mod["mass"].sum()) / 90.0)
    return mod, with_tight_limits(ms), verts


def test_emulated_sensor_matches_restatement(amass):
    """256 random states in ground contact, active joint limits in some DOFs, one control step: the float64 sensor instantiation's
    rows equal the sensor evaluated on the restatement's trajectory to 1e-9 (relative to the torque scale)"""
    mod, ms, verts = amass
    cfg = abi.make_cfg(mod)
    n = 256
    root, q, qd, tar, _ = states(n, 23, True)
    r1, q1, v1 = root.copy(), q.copy(), qd.copy()
    _, cf1, tau = emu_step(ms, verts, cfg, r1, q1, v1, tar.copy(), None)
    r2, q2, v2 = root.copy(), q.copy(), qd.copy()
    ref = restatement_dof_force(ms, verts, cfg, r2, q2, v2, tar.copy())
    np.testing.assert_allclose(q1, q2, rtol=0, atol=1e-9)
    # the torque scale of each env's row: the two solves agree to ~1e-11 in qd+ in contact, which kp h + kd ~ 100 turns into ~1e-9 N m
    scale = np.maximum(1.0, np.abs(ref).max(1, keepdims=True))
    assert (np.abs(tau - ref) / scale).max() < 1e-9, (np.abs(tau - ref) / scale).max()
    qs, _ = start_of_last_substep(ms, cfg, q2, v2)
    a = model_arrays(ms)
    active = (qs < a["lim_lo"]) | (qs > a["lim_hi"])
    assert active.sum() > 100 and (~active).sum() > 100          # both branches exercised
    assert np.abs(cf1).max() > 10.0                             # in contact


def anchor_joint_force(tree, ms, cfg, root, q, qd, tar, limits):
    """(M + diag(armature)) qdd + c over the joint rows, with qdd from the joint-space equations of motion of one substep (the implicit
    PD / armature diagonal, plus the limit spring-damper on the DOFs past a limit when `limits`)"""
    h, gz = float(cfg.sim_dt) / cfg.substeps, float(cfg.gravity_z)
    u = np.concatenate([root[10:13], root[7:10], qd])
    M, c, _, _ = tree.mass_matrix_and_bias(root[0:3], root[3:7], q, u, gz)
    a = model_arrays(ms)
    e = h * tree.kd + h * h * tree.kp
    tau = tree.kp * (tar - q - h * qd) - tree.kd * qd
    if limits:
        k, cc = float(cfg.limit_k), float(cfg.limit_c)
        for lim, on in ((a["lim_lo"], q < a["lim_lo"]), (a["lim_hi"], q > a["lim_hi"])):
            tau = np.where(on, tau + k * (lim - q - h * qd) - cc * qd, tau)
            e = np.where(on, e + h * cc + h * h * k, e)
    n = 6 + tree.nd
    E, t = np.zeros(n), np.zeros(n)
    E[6:], t[6:] = tree.arm + e, tau
    ud = np.linalg.solve(M + np.diag(E), t - c)
    Ma = M + np.diag(np.concatenate([np.zeros(6), tree.arm]))
    return (Ma @ ud + c)[6:], M


@pytest.mark.parametrize("limits", [False, True])
def test_sensor_against_jacobian_equations_of_motion(amass, limits):
    """one contact-free substep (no damping, no clamp) of the emulated sensor instantiation: the reported force equals
    (M(q) + diag(armature)) qdd + c(q, u) of the Jacobian assembly to 1e-10 relative; with poses past the tight limits the reported
    force contains the limit term (the anchor with limk / limc added - and differs from the anchor without them)"""
    mod, ms, verts = amass
    tree = Tree(ms)
    cfg = abi.make_cfg(mod, sim_dt=1.0 / 120.0, substeps=1, control_freq_inv=1, ang_damping=0.0, max_ang_vel=1e6)
    rng = np.random.default_rng(5)
    n = 64
    root, q, qd, tar = random_state(rng, n, ms.nd)
    q = rng.normal(0, 0.3, q.shape) if limits else 0.7 * q      # inside every limit (the tight ones are +-0.2) or past some
    _, _, tau = emu_step(ms, verts, cfg, root.copy(), q.copy(), qd.copy(), tar.copy(), None)
    worst = worst_other = 0.0
    a = model_arrays(ms)
    for i in range(n):
        want, _ = anchor_joint_force(tree, ms, cfg, root[i], q[i], qd[i], tar[i], limits)
        worst = max(worst, np.abs(tau[i] - want).max() / (1.0 + np.abs(want).max()))
        if limits:
            other, _ = anchor_joint_force(tree, ms, cfg, root[i], q[i], qd[i], tar[i], False)
            on = (q[i] < a["lim_lo"]) | (q[i] > a["lim_hi"])
            worst_other = max(worst_other, np.abs(tau[i] - other)[on].max() / (1.0 + np.abs(other).max()))
    assert worst < 1e-10, worst
    if limits:
        assert worst_other > 1e-3, worst_other


def test_sensor_leaves_the_motion_alone(amass):
    """the step with the sensor on and off, 2 control steps in contact with the residual wrench: every state row bit-identical"""
    mod, ms, verts = amass
    cfg = abi.make_cfg(mod)
    root, q, qd, tar, ext = states(13, 31, True)
    out = []
    for sensor in (False, True):
        r, qq, vv = root.copy(), q.copy(), qd.copy()
        rb, cf, tau = emu_step(ms, verts, cfg, r, qq, vv, tar.copy(), ext.copy(), n_steps=2, sensor=sensor)
        out.append((r, qq, vv, rb, cf))
        if sensor:
            assert np.isfinite(tau).all() and np.abs(tau).max() > 1.0
    for a, b in zip(*out):
        assert np.array_equal(a, b)


def test_sensor_with_racket_and_ball():
    """the tennis player (welded racket, ball on lane 7 of each env group, 6 substeps): sensor rows against the restatement, the
    welded racket has no DOFs"""
    mod = model_compiler.canonical_racket_last(model_compiler.load_compiled("smpl_mesh_humanoid_federer"))
    ms, verts = abi.pack_model(mod, float(mod["mass"].sum()) / 90.0)
    ms = with_tight_limits(ms)
    cfg = abi.make_cfg(mod, substeps=6, ball={}, task_mode=1, pd_mode=1)
    n = 9
    root, q, qd, tar, ext = states(n, 7, True)
    rng = np.random.default_rng(3)
    ball = np.zeros((n, 13))
    ball[:, 0:3] = root[:, 0:3] + rng.normal(0, 0.6, (n, 3)) + [0, 0.5, 0.3]
    ball[:, 2] = np.abs(ball[:, 2]) + 0.04
    ball[:, 7:10] = rng.normal(0, 8, (n, 3))
    b1, b2, h1, h2 = ball.copy(), ball.copy(), np.zeros(n, np.int32), np.zeros(n, np.int32)
    r1, q1, v1 = root.copy(), q.copy(), qd.copy()
    _, _, tau = emu_step(ms, verts, cfg, r1, q1, v1, tar.copy(), ext.copy(), ball=b1, hits=h1)
    ref = restatement_dof_force(ms, verts, cfg, root.copy(), q.copy(), qd.copy(), tar.copy(), ext.copy(), ball=b2, hits=h2)
    assert (np.abs(tau - ref) / np.maximum(1.0, np.abs(ref))).max() < 1e-8
