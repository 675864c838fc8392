"""CPU checks of the imitation test run's pose metrics (cfg.env.b200_pose_metrics): the float64 restatement
oracle/ref_port_pose_metrics.py against an independent alignment and on hand-computed cases, the cfg refusals, the file keys and the
summary line of HumanoidSMPLIMVis, and the C ABI of the pose fields of b200_im_motion_stats_t."""
import ctypes as C
import io
import contextlib
import os
import subprocess
import types

import numpy as np
import pytest
import torch
from scipy.spatial.transform import Rotation

import test_host
from oracle import ref_port_pose_metrics as P
from vid2player3d_b200 import abi, model_compiler, motion_lib, native
from vid2player3d_b200.configs import im_cfg
from vid2player3d_b200.tasks import humanoid_smpl_im_vis as V


# ---------------------------------------------------------------------------------------------------------- the restatement
def pa_err(body, target):
    return np.linalg.norm(P.pa_aligned(body, target) - target, axis=-1).mean()


def pa_by_align_vectors(body, target):
    """the same optimum by another route: scipy's rotation of the centred body onto the centred target, then the least-squares scale"""
    x, y = body - body.mean(0), target - target.mean(0)
    rot, _ = Rotation.align_vectors(y, x)
    rx = rot.apply(x)
    s = (rx * y).sum() / (x * x).sum()
    return np.linalg.norm(s * rx - y, axis=-1).mean()


def test_pa_agrees_with_an_independent_alignment():
    g = np.random.default_rng(0)
    for B in (3, 5, 24, 32):
        for _ in range(20):
            body, target = g.normal(size=(B, 3)), g.normal(size=(B, 3))
            np.testing.assert_allclose(pa_err(body, target), pa_by_align_vectors(body, target), rtol=1e-10)


def frames(body, target):
    """one env's errors (g, l, pa) of one frame"""
    g, l, pa = P.frame_errors(body[None], target[None])
    return g[0], l[0], pa[0]


def pose(seed, B=24):
    return np.random.default_rng(seed).normal(size=(B, 3))


def test_identical_motion_is_all_zeros_and_a_success():
    m = run_games([[pose(k) for k in range(4)]], [[pose(k) for k in range(4)]])
    assert not m.pose_sums[0, [0, 2, 3]].any() and m.pose_sums[0, 4:6].tolist() == [3, 2] and m.pose_sums[0, 6] == 0.0
    assert m.pose_sums[0, 1] < 1e-13                              # the SVD's rounding
    assert m.success.tolist() == [1]


def test_constant_translation_is_global_error_only():
    d = np.array([0.3, -0.4, 0.0])
    r = pose(1)
    g, l, pa = frames(r + d, r)
    assert g == pytest.approx(0.5, rel=1e-14) and l == pytest.approx(0.0, abs=1e-15) and pa == pytest.approx(0.0, abs=1e-14)


def test_a_rotated_scaled_and_translated_copy_aligns_exactly():
    r = pose(2)
    p = 1.7 * r @ Rotation.from_euler("xyz", [0.3, -1.1, 2.0]).as_matrix().T + np.array([1.0, 2.0, -3.0])
    g, l, pa = frames(p, r)
    assert pa < 1e-12 and l > 0.1 and g > 0.1


def test_a_mirrored_pose_takes_the_best_proper_rotation():
    r = pose(3)
    p = r * np.array([-1.0, 1.0, 1.0])                            # a reflection aligns it exactly; no rotation does
    _, _, pa = frames(p, r)
    assert pa > 0.1
    assert pa == pytest.approx(pa_by_align_vectors(p, r), rel=1e-10)
    best = ((P.pa_aligned(p, r) - r) ** 2).sum()                   # the alignment minimises the squared distances:
    x, y = p - p.mean(0), r - r.mean(0)                            # no sampled rotation does better
    for R in Rotation.random(2000, random_state=4).as_matrix():
        rx = x @ R.T
        s = max((rx * y).sum() / (x * x).sum(), 0.0)
        assert ((s * rx - y) ** 2).sum() >= best * (1 - 1e-12)


def test_collinear_bodies_have_a_well_defined_alignment():
    t = np.linspace(-1.0, 1.0, 24)
    p = t[:, None] * np.array([1.0, 2.0, 2.0]) / 3.0 + 0.5        # bodies on a line: the rotation about it is free, the pose is not
    r = pose(5)
    _, _, pa = frames(p, r)
    alpha = t - t.mean()                                         # the best aligned pose is alpha_b v, v the least-squares direction
    y = r - r.mean(0)
    v = (alpha[:, None] * y).sum(0) / (alpha * alpha).sum()
    assert pa == pytest.approx(np.linalg.norm(alpha[:, None] * v - y, axis=-1).mean(), rel=1e-12)


def test_no_spread_puts_every_body_on_the_target_centroid():
    r = pose(6)
    p = np.tile([[0.2, 0.1, 0.9]], (24, 1))
    _, _, pa = frames(p, r)
    assert pa == np.linalg.norm(r - r.mean(0), axis=-1).mean()


def run_games(bodies, targets, ends=None, threshold=0.5, env_games=None):
    """one env of motion 0; each game a list of frames, ended at its last frame (reset_buf rises there), then a new game"""
    m = P.PoseMetrics([0], 1, threshold)
    for gi, (bs, ts) in enumerate(zip(bodies, targets)):
        m.new_game()
        for k, (b, t) in enumerate(zip(bs, ts)):
            done = np.array([int(k == len(bs) - 1)])
            m.step(np.zeros(1), np.zeros((1, 4)), done, np.zeros(1, np.int64), b[None], t[None])
    return m


def test_constant_velocity_drift_has_constant_velocity_error_and_no_acceleration_error():
    v = np.array([0.01, 0.0, -0.02])
    ts = [pose(7) + 0.1 * k for k in range(6)]
    bs = [t + v * k for k, t in enumerate(ts)]
    m = run_games([bs], [ts])
    assert m.pose_sums[0, 4:6].tolist() == [5, 4]
    assert m.pose_sums[0, 2] == pytest.approx(5 * np.linalg.norm(v), rel=1e-12)
    assert m.pose_sums[0, 3] == pytest.approx(0.0, abs=1e-13)


def test_velocity_and_acceleration_frames_of_short_games():
    """games of 1, 2 and 3 frames: velocity from a game's second frame, acceleration from its third; a game's end empties the
    history, so the next game starts afresh"""
    games = [[pose(10 + k) for k in range(n)] for n in (1, 2, 3)]
    m = run_games(games, [[g + 0.01 for g in game] for game in games])
    assert m.pose_sums[0, 4:6].tolist() == [0 + 1 + 2, 0 + 0 + 1]
    assert m.counts[0, 0] == 3 and m.pose_sums[0, 4] + m.counts[0, 0] == m.sums[0, 1]


def test_one_frame_above_the_threshold_is_not_a_success():
    ts = [pose(20) for _ in range(5)]
    bs = [t.copy() for t in ts]
    bs[2] = bs[2] + np.array([0.0, 0.0, 0.51])                   # g = 0.51 at one frame
    m = run_games([bs, ts], [ts, ts])
    assert m.success.tolist() == [1] and m.counts[0, 0] == 2
    assert m.pose_sums[0, 6] == pytest.approx(0.51, rel=1e-12)
    assert run_games([bs], [ts], threshold=0.52).success.tolist() == [1]


def test_a_nan_env_is_never_a_success_and_its_sums_are_nan():
    ts = [pose(30) for _ in range(4)]
    bs = [t + 0.01 for t in ts]
    bs[1] = bs[1].copy()
    bs[1][3, 0] = np.nan
    m = run_games([bs], [ts])
    assert m.success.tolist() == [0] and np.isnan(m.pose_sums[0, 6])
    assert np.isnan(m.sums[0, 6]) and np.isnan(m.pose_sums[0, :4]).all()


def test_stop_flag_and_other_motions():
    """while stopped nothing changes; a motion whose env never ends a game keeps zero buckets"""
    m = P.PoseMetrics([0, 1], 2)
    x = lambda k: np.stack([pose(40 + k), pose(50 + k)])  # noqa: E731
    m.step(np.zeros(2), np.zeros((2, 4)), np.array([0, 0]), np.zeros(2), x(0), x(0) + 0.1)
    before = (m.env_pose.copy(), m.fill.copy())
    m.step(np.zeros(2), np.zeros((2, 4)), np.array([1, 1]), np.zeros(2), x(1), x(1), stop=True)
    assert np.array_equal(m.env_pose, before[0]) and m.fill.tolist() == [1, 1]
    m.step(np.zeros(2), np.zeros((2, 4)), np.array([1, 0]), np.zeros(2), x(1), x(1) + 0.1)
    assert m.counts[:, 0].tolist() == [1, 0] and not m.pose_sums[1].any() and m.success.tolist() == [1, 0]
    assert m.pose_sums[0, 4] == 1 and m.fill.tolist() == [0, 2]


# ---------------------------------------------------------------------------------------------------------- the task's host side
@pytest.mark.parametrize("env, msg", [(dict(b200_pose_metrics=True), "set b200_motion_stats: True"),
                                      (dict(b200_pose_metrics=True, b200_motion_stats=True, b200_pose_success_threshold=0.0), "above 0"),
                                      (dict(b200_pose_metrics=True, b200_motion_stats=True, b200_pose_success_threshold=-1), "above 0"),
                                      (dict(b200_pose_metrics=True, b200_motion_stats=True, b200_pose_success_threshold=float("nan")),
                                       "finite"),
                                      (dict(b200_pose_metrics=True, b200_motion_stats=True, b200_pose_success_threshold=float("inf")),
                                       "finite"),
                                      (dict(b200_pose_metrics=True, b200_motion_stats=True, b200_pose_success_threshold="half"),
                                       "number of metres")])
def test_cfg_refusals(env, msg):
    with pytest.raises(ValueError, match=msg):
        V.pose_metrics_threshold(env)


def test_cfg_resolution():
    assert V.pose_metrics_threshold({}) is None and V.pose_metrics_threshold(dict(b200_motion_stats=True)) is None
    assert V.pose_metrics_threshold(dict(b200_pose_metrics=True, b200_motion_stats=True)) == 0.5
    assert V.pose_metrics_threshold(dict(b200_pose_metrics=True, b200_motion_stats=True, b200_pose_success_threshold="0.3")) == 0.3


def test_the_task_refuses_before_allocating(tmp_path):
    """the refusal comes from HumanoidSMPLIMVis' constructor before anything reaches the device (none is needed to see it)"""
    from vid2player3d_b200.tasks import HumanoidSMPLIMVis
    flat = motion_lib.synthetic(model_compiler.load_compiled("smpl_mesh_humanoid_amass_v1"), num_motions=2, num_frames=20, seed=1)
    path = str(tmp_path / "m.npz")
    flat.save(path)
    cfg = im_cfg(4, None, motion_file=path, b200_pose_metrics=True)
    cfg["args"] = types.SimpleNamespace(test=True)
    with pytest.raises(ValueError, match="b200_pose_metrics extends the per-motion meters"):
        HumanoidSMPLIMVis(cfg, None, 1, "cuda", 0, True)


def test_summary_line():
    counts = np.array([[2, 1], [0, 0], [2, 0]])
    sums = np.zeros((3, 7))
    sums[:, 1], sums[:, 6] = [10, 0, 6], [0.8, 0.0, 0.8]
    ps = np.zeros((3, 7))
    ps[:, 0], ps[:, 1], ps[:, 2], ps[:, 3], ps[:, 4], ps[:, 5] = [0.4, 0, 0.4], [0.16, 0, 0.16], [0.1, 0, 0.02], [0.01, 0, 0.01], \
        [8, 0, 4], [6, 0, 2]
    assert V.pose_metrics_summary(counts, sums, ps, np.array([1, 0, 2])) == (
        "success rate: 0.7500  MPJPE-g: 100.00 mm  MPJPE-l: 50.00 mm  PA-MPJPE: 20.00 mm  velocity error: 10.00 mm/frame"
        "  acceleration error: 2.50 mm/frame^2")
    assert "success rate: nan" in V.pose_metrics_summary(np.zeros((1, 2), np.int64), np.zeros((1, 7)), np.zeros((1, 7)), np.zeros(1))


def fake_task(tmp_path, pose_on):
    """a HumanoidSMPLIMVis without its constructor: the buckets on the host, for export_motion_stats"""
    t = object.__new__(V.HumanoidSMPLIMVis)
    M, N = 3, 4
    g = torch.Generator().manual_seed(0)
    t._ms = dict(counts=torch.tensor([[2, 1], [0, 0], [1, 0]]), sums=torch.rand(M, 7, generator=g, dtype=torch.float64))
    t._pose_threshold = 0.25 if pose_on else None
    if pose_on:
        ps = torch.rand(M, 7, generator=g, dtype=torch.float64)
        ps[:, 4:6] = torch.tensor([[5.0, 3.0], [0, 0], [7, 6]])
        t._ms.update(pose_sums=ps, success=torch.tensor([1, 0, 1]))
    t.cfg = dict(env=dict(b200_motion_stats_file=str(tmp_path / ("on.npz" if pose_on else "off.npz"))))
    t._reset_ref_motion_ids, t._test_motion_file, t.dt = torch.tensor([0, 2, 0, 0]), None, 1.0 / 30
    assert N == len(t._reset_ref_motion_ids)
    return t


PARENT_KEYS = {"games", "falls", "reward_sum", "steps", "sub_reward_sum", "body_pos_err_sum", "env_motion_ids", "test_motion_file"}
POSE_KEYS = {"mpjpe_l_sum", "mpjpe_pa_sum", "vel_err_sum", "acc_err_sum", "vel_frames", "acc_frames", "success", "max_body_pos_err",
             "success_threshold", "dt"}


def test_file_keys_and_lines(tmp_path):
    t = fake_task(tmp_path, True)
    with contextlib.redirect_stdout(io.StringIO()) as out:
        path = t.export_motion_stats()
    f = dict(np.load(path))
    assert set(f) == PARENT_KEYS | POSE_KEYS
    ps = t._ms["pose_sums"].numpy()
    for i, k in enumerate(("mpjpe_l_sum", "mpjpe_pa_sum", "vel_err_sum", "acc_err_sum")):
        assert f[k].dtype == np.float64 and np.array_equal(f[k], ps[:, i]), k
    assert f["vel_frames"].dtype == np.int64 and f["vel_frames"].tolist() == [5, 0, 7] and f["acc_frames"].tolist() == [3, 0, 6]
    assert f["success"].dtype == np.int64 and f["success"].tolist() == [1, 0, 1]
    assert np.array_equal(f["max_body_pos_err"], ps[:, 6]) and f["success_threshold"] == 0.25 and f["dt"] == 1.0 / 30
    lines = out.getvalue().splitlines()
    assert lines[0].startswith("motions evaluated: 2 of 3") and lines[1].startswith("success rate: 0.6667  MPJPE-g: ")
    assert "per-motion statistics written to" in lines[2]
    t = fake_task(tmp_path, False)
    with contextlib.redirect_stdout(io.StringIO()) as out:
        path = t.export_motion_stats()
    assert set(np.load(path)) == PARENT_KEYS and not any(x.startswith("success rate") for x in out.getvalue().splitlines())


# ---------------------------------------------------------------------------------------------------------- the C ABI
POSE_FIELDS = ["env_pose", "pose_hist", "pose_fill", "pose_sums", "success", "success_threshold"]


def test_pose_fields_follow_the_meters_fields_in_the_header(tmp_path):
    """b200_im_motion_meters_t, the meters' kernel parameter, is b200_im_motion_stats_t's first 120 bytes field by field"""
    S = abi.ImMotionStats
    assert [f for f, _ in S._fields_[-len(POSE_FIELDS):]] == POSE_FIELDS
    lines = ['printf("%zu %zu\\n", sizeof(b200_im_motion_meters_t), offsetof(b200_im_motion_stats_t, env_pose));']
    want = ["120 120"]
    for f, _ in S._fields_[:-len(POSE_FIELDS)]:
        lines.append(f'printf("{f} %zu\\n", offsetof(b200_im_motion_meters_t, {f}));')
        want.append(f"{f} {getattr(S, f).offset}")
    src, exe = tmp_path / "meters.c", tmp_path / "meters"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "b200env.h"\nint main(void) {\n' + "\n".join(lines) + "\nreturn 0;\n}\n")
    subprocess.check_call(["gcc", "-w", "-I", os.path.join(test_host.ROOT, "include"), str(src), "-o", str(exe)])
    assert subprocess.check_output([str(exe)], text=True).splitlines() == want
    assert C.sizeof(S) == 168 and S.success_threshold.offset == 160


def test_binding_refuses_a_library_without_the_pose_fields(monkeypatch):
    native.lib()
    old = type("ImMotionStats", (C.Structure,), {"_fields_": abi.ImMotionStats._fields_[:-len(POSE_FIELDS)]})
    assert C.sizeof(old) == 120
    monkeypatch.setattr(abi, "ImMotionStats", old)
    monkeypatch.setattr(native, "_lib", None)
    with pytest.raises(RuntimeError, match="takes a 168-byte ImMotionStats descriptor, the binding fills 120 - rebuild"):
        native.lib()


class _OnDevice:
    """a host tensor that reports device 0, so that native.fill's device rule lets it through on a machine without a GPU"""

    def __init__(self, t):
        self.t, self.dtype = t, t.dtype

    def is_contiguous(self):
        return self.t.is_contiguous()

    def get_device(self):
        return 0

    def data_ptr(self):
        return self.t.data_ptr()


DTYPES = {abi.F32P: torch.float32, abi.I64P: torch.int64, abi.I32P: torch.int32, abi.F64P: torch.float64}
SCALARS = dict(n=4, num_motions=3, num_bodies=24, num_lib_bodies=24)


def test_fill_fills_the_pose_fields():
    S = abi.ImMotionStats
    keep = {f: torch.zeros(2, dtype=DTYPES[ct]) for f, ct in S._fields_ if issubclass(ct, C.c_void_p)}
    d = native.fill(S, dict(SCALARS, success_threshold=0.4), {f: _OnDevice(t) for f, t in keep.items()})
    for f in POSE_FIELDS[:-1]:
        assert getattr(d, f).value == keep[f].data_ptr(), f
    assert d.success_threshold == 0.4
    d = native.fill(S, SCALARS, {f: _OnDevice(t) for f, t in keep.items() if f not in POSE_FIELDS})   # the meters alone
    assert all(getattr(d, f).value is None for f in POSE_FIELDS[:-1]) and d.success_threshold == 0.0
    with pytest.raises(ValueError, match=r"ImMotionStats\.pose_hist: torch\.float64, the header's pointee needs torch\.float32"):
        native.fill(S, SCALARS, dict({f: _OnDevice(t) for f, t in keep.items()}, pose_hist=_OnDevice(torch.zeros(2, dtype=torch.float64))))
    with pytest.raises(ValueError, match=r"ImMotionStats\.pose_fill: torch\.int64"):
        native.fill(S, SCALARS, dict({f: _OnDevice(t) for f, t in keep.items()}, pose_fill=_OnDevice(torch.zeros(2, dtype=torch.long))))


def refused(over, drop=()):
    """the launch's return code and message on fake device addresses: every case must be refused before a launch"""
    d = abi.ImMotionStats(**{**SCALARS, "success_threshold": 0.5, **over})
    for name, ct in abi.ImMotionStats._fields_:
        if issubclass(ct, C.c_void_p) and name not in drop:
            setattr(d, name, 0x10000)
    return native.lib().b200env_im_motion_stats(C.byref(d), None), native.lib().b200env_last_error().decode()


@pytest.mark.parametrize("over, code, msg", [
    (dict(num_bodies=40, num_lib_bodies=33), -2, "the pose metrics take at most 32 bodies"),
    (dict(success_threshold=0.0), -2, "success_threshold must be a finite positive number"),
    (dict(success_threshold=float("nan")), -2, "success_threshold must be"),
    (dict(success_threshold=float("inf")), -2, "success_threshold must be"),
    (dict(n=0, num_lib_bodies=33), -2, "n and num_motions must be positive"),          # the meters' refusals come first
    (dict(num_lib_bodies=25, success_threshold=0.0), -2, "num_lib_bodies must lie in [1, num_bodies]"),
])
def test_launch_refusals_before_any_launch(over, code, msg):
    rc, err = refused(over)
    assert rc == code and msg in err


@pytest.mark.parametrize("drop", [("env_pose",), ("pose_hist",), ("pose_fill",), ("pose_sums",), ("success",)])
def test_some_pose_pointers_null_is_refused(drop):
    rc, err = refused({}, drop)
    assert rc == -1 and "the pose pointers must be all set or all NULL" in err
