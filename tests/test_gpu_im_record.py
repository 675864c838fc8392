"""GPU checks of HumanoidSMPLIMVis' qpos recorder: the launch b200env_im_record against the float64 restatement
oracle/ref_port_record.py at several sizes and env lists, its frame counter, cap and stop flag, and run_test with recording (graphed
against eager, the printed lines against the restatement of render_vis' quit rule, the file), the eager render_vis API, a handle of
several assets and the task without the key.

Tolerances: the launch reads float32 state and computes the angles in double.  Root positions and quaternions: 1e-6 (copy 1's x + 1 rounds to
float32).  Euler angles: 2e-5 after wrapping the difference to (-pi, pi] while |2(wy - xz)| < 0.999; nearer the pole, where asin and
the two atan2 are ill-conditioned, the rotation Rz(yaw) Ry(pitch) Rx(roll) of the three angles within 1e-4."""
import io
import contextlib

import numpy as np
import pytest
import torch

from oracle import ref_port_record as R
from test_gpu_im_policy import make_task, network

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
NB, NBL, ND = 24, 24, 69
NQ = 7 + ND


def state(N, seed):
    g = torch.Generator().manual_seed(seed)
    rbs = torch.randn(N, NB, 13, generator=g) * 1.5
    rbs[..., 3:7] /= rbs[..., 3:7].norm(dim=-1, keepdim=True)
    dof = torch.rand(N, ND, generator=g) * 6 - 3
    pdof = torch.rand(N, ND, generator=g) * 6 - 3
    for k, a in enumerate([(0.0, 0.0, 0.0), (np.pi - 1e-6, 0, 0), (0, np.pi / 2, 0), (0, -np.pi / 2, 0), (0, np.pi / 2 - 1e-3, 0),
                           (np.pi, 0, 0), (-np.pi, 0, 0), (0, 0, np.pi), (0, 0, -np.pi), (1e-5, 0, 0)]):
        dof[:, 3 * k:3 * k + 3] = torch.tensor(a)
        pdof[:, 3 * (k + 5):3 * (k + 5) + 3] = torch.tensor(a)
    prb = torch.randn(N, NBL, 7, generator=g) * 1.5
    prb[..., 3:7] /= prb[..., 3:7].norm(dim=-1, keepdim=True)
    dof_state = torch.stack([dof, torch.randn(N, ND, generator=g)], -1)
    return dict(rigid_body_state=rbs.to(DEV).contiguous(), dof_state=dof_state.to(DEV).contiguous(), p_dof_pos=pdof.to(DEV),
                p_rb_pos=prb[..., :3].contiguous().to(DEV), p_rb_rot=prb[..., 3:].contiguous().to(DEV),
                reset_buf=torch.randint(0, 2, (N,), generator=g).to(DEV), motion_ids=torch.randint(0, 9, (N,), generator=g).to(DEV))


def buffers(E, cap):
    return dict(qpos=torch.full((E, cap, 2, NQ), -77.0, device=DEV), rec_motion_ids=torch.full((E, cap), -1, device=DEV, dtype=torch.long),
                rec_reset=torch.full((E, cap), -1, device=DEV, dtype=torch.long), frame=torch.zeros(1, device=DEV, dtype=torch.long),
                done=torch.zeros(1, device=DEV, dtype=torch.int32))


def launch(st, buf, ids, cap, init, games=None):
    from vid2player3d_b200 import native
    N = st["reset_buf"].shape[0]
    native.im_record(dict(n_rec=len(ids), num_envs=N, num_bodies=NB, num_lib_bodies=NBL, nd=ND, cap=cap, init=int(init)),
                     dict(st, **buf, env_ids=torch.tensor(ids, device=DEV, dtype=torch.long), games=games))


def expected(st, ids, init):
    g = lambda k: st[k].double().cpu().numpy()  # noqa: E731
    rbs = g("rigid_body_state")
    return R.sync_ref_motion(rbs[..., :3], rbs[..., 3:7], g("dof_state")[..., 0], g("p_rb_pos"), g("p_rb_rot"), g("p_dof_pos"), ids,
                             init)[:, :2 * NQ].reshape(len(ids), 2, NQ)


def rot(a):
    """Rz(yaw) Ry(pitch) Rx(roll) of angles [..., 3] = (yaw, pitch, roll)"""
    y, p, r = a[..., 0], a[..., 1], a[..., 2]
    cy, sy, cp, sp, cr, sr = np.cos(y), np.sin(y), np.cos(p), np.sin(p), np.cos(r), np.sin(r)
    return np.stack([np.stack([cy * cp, cy * sp * sr - sy * cr, cy * sp * cr + sy * sr], -1),
                     np.stack([sy * cp, sy * sp * sr + cy * cr, sy * sp * cr - cy * sr], -1),
                     np.stack([-sp, cp * sr, cp * cr], -1)], -2)


def assert_rows(got, want):
    """got / want [..., 2, nq]"""
    np.testing.assert_allclose(got[..., :7], want[..., :7], rtol=0, atol=1e-6)
    ga, wa = got[..., 7:].reshape(-1, 3), want[..., 7:].reshape(-1, 3)
    pole = np.abs(np.sin(wa[:, 1])) >= 0.999            # sin(pitch) = the clamped 2(wy - xz)
    d = np.abs(np.angle(np.exp(1j * (ga - wa))))
    assert d[~pole].max(initial=0) <= 2e-5, d[~pole].max()
    if pole.any():
        assert np.abs(rot(ga[pole]) - rot(wa[pole])).max() <= 1e-4


@pytest.mark.parametrize("N", [1, 127, 128, 129, 8192])
@pytest.mark.parametrize("which", ["all", "strided"])
def test_launch_is_the_restatement(N, which):
    st = state(N, N)
    ids = list(range(N)) if which == "all" else list(range(N - 1, -1, -3))
    cap = 3
    buf = buffers(len(ids), cap)
    for f, init in enumerate((True, False, False)):
        if f == 2:
            st = state(N, N + 7)
        launch(st, buf, ids, cap, init)
        torch.cuda.synchronize()
        assert int(buf["frame"]) == f + 1
        assert_rows(buf["qpos"][:, f].double().cpu().numpy(), expected(st, ids, init))
        idx = torch.tensor(ids, device=DEV)
        assert torch.equal(buf["rec_motion_ids"][:, f], st["motion_ids"][idx])
        assert torch.equal(buf["rec_reset"][:, f], torch.zeros_like(idx) if init else st["reset_buf"][idx])


def test_frames_cap_and_stop():
    N, cap, ids = 40, 4, [3, 39, 0]
    buf, games = buffers(len(ids), cap), torch.zeros(3, device=DEV, dtype=torch.long)
    sts = [state(N, 100 + k) for k in range(6)]
    launch(sts[0], buf, ids, cap, False, games)
    games[1] = 1                                           # stopped: nothing written, no advance
    launch(sts[1], buf, ids, cap, False, games)
    torch.cuda.synchronize()
    assert int(buf["frame"]) == 1 and bool((buf["qpos"][:, 1] == -77.0).all())
    games[1] = 0
    for k in (2, 3):
        launch(sts[k], buf, ids, cap, False, games)
    torch.cuda.synchronize()
    assert int(buf["frame"]) == 3 and int(games[1]) == 0
    launch(sts[4], buf, ids, cap, False, games)            # the last frame sets stop
    torch.cuda.synchronize()
    assert int(buf["frame"]) == 4 and int(games[1]) == 1
    snap = buf["qpos"].clone()
    games[1] = 0
    launch(sts[5], buf, ids, cap, False, games)            # full: nothing past cap, stop left alone
    launch(sts[5], buf, ids, cap, False, None)
    torch.cuda.synchronize()
    assert int(buf["frame"]) == 4 and int(games[1]) == 0 and torch.equal(buf["qpos"], snap)
    for f, k in enumerate((0, 2, 3, 4)):                   # rows in frame order
        assert_rows(buf["qpos"][:, f].double().cpu().numpy(), expected(sts[k], ids, False))


def rec_task(N=64, **over):
    torch.manual_seed(0)
    return make_task(N, b200_record_qpos=True, **over)


def run(task, tmp_path, name, graph, games_num=3, max_steps=40, **kw):
    task._rec_path = str(tmp_path / f"{name}.npz")
    out, exited = io.StringIO(), False
    with contextlib.redirect_stdout(out):
        try:
            task.run_test(network(5)[0], games_num, max_steps, graph=graph, clip_actions=1.0, **kw)
        except SystemExit:
            exited = True
    return dict(np.load(task._rec_path)), out.getvalue().splitlines(), exited


def stat_lines(lines):
    return [x for x in lines if x.startswith("reward:")]


def test_run_test_graphed_is_eager_and_quits_like_the_reference(tmp_path):
    full_task = rec_task(b200_record_envs="all", num_rec_frames=1000)
    hist = []
    full, full_lines, exited = run(full_task, tmp_path, "full", True, history=hist)
    assert not exited and any(x.startswith("av reward:") for x in full_lines)
    games = [[(r.cpu().numpy(), d.cpu().numpy()) for r, d in g] for g in hist]
    T = full["qpos"].shape[1]
    lines, frames, quit_ = R.run_with_record(games, 3, 40, 1000)
    assert not quit_ and len(frames) == T
    cap = T - 5
    want_lines, want_frames, quit_ = R.run_with_record(games, 3, 40, cap)
    assert quit_ and len(want_frames) == cap
    got = {}
    for graph in (True, False):
        got[graph], printed, exited = run(rec_task(b200_record_envs=[0, 63, 17], num_rec_frames=cap), tmp_path, f"g{graph}", graph)
        assert exited and not any(x.startswith("av reward:") for x in printed)
        assert stat_lines(printed) == [f"reward: {r / c} steps: {s / c}" for c, r, s in want_lines]
    for k in ("qpos", "env_ids", "motion_ids", "reset", "asset", "fps", "nq"):
        assert np.array_equal(got[True][k], got[False][k]), k
    g = got[True]
    assert g["qpos"].shape == (3, cap, 3 * NQ) and g["qpos"].dtype == np.float32 and g["motion_ids"].shape == (3, cap)
    assert g["reset"].shape == (3, cap) and list(g["env_ids"]) == [0, 63, 17] and int(g["nq"]) == NQ and len(g["asset"]) == 3
    assert float(g["fps"]) == pytest.approx(30.0)
    assert np.array_equal(g["qpos"], full["qpos"][[0, 63, 17], :cap])       # the same frames as the unbounded run's
    assert np.array_equal(g["reset"], full["reset"][[0, 63, 17], :cap])
    q = g["qpos"]
    assert np.array_equal(q[..., 2 * NQ + 2], (q[..., 2].astype(np.float32) + np.float32(1000.0)))


def test_one_frame_exits_after_the_init_frame(tmp_path):
    rec, printed, exited = run(rec_task(num_rec_frames=1), tmp_path, "one", True)
    assert exited and rec["qpos"].shape == (1, 1, 3 * NQ) and stat_lines(printed) == []


def test_eager_render_vis_records_what_run_test_records(tmp_path):
    task = rec_task(num_rec_frames=500)
    want, _, _ = run(task, tmp_path, "rt", True, games_num=1, max_steps=30)
    task = rec_task(num_rec_frames=500)
    task.set_policy(network(5)[0], clip_actions=1.0)
    task._rec_path = str(tmp_path / "eager.npz")
    task.reset()
    task.render_vis(init=True)
    g = lambda k: getattr(task, k).double().cpu().numpy()  # noqa: E731
    for n in range(30):
        if n > 0 and n % task.context_length == 0:
            task._init_context(torch.arange(task.num_envs, device=DEV), task._reset_ref_motion_ids, task._cur_ref_motion_times)
        with torch.no_grad():
            task._env.step(task.act())
        task._im_step += 1
        task.render_vis()
        rbs = g("_rigid_body_state").reshape(task.num_envs, -1, 13)
        ref = R.sync_ref_motion(rbs[..., :3], rbs[..., 3:7], g("_dof_pos"), g("_prev_target_rb_pos"), g("_prev_target_rb_rot"),
                                g("_prev_target_dof_pos"), [0], False)
        assert_rows(task._rec["qpos"][:, n + 1].double().cpu().numpy(), ref[:, :2 * NQ].reshape(1, 2, NQ))
        if bool(task.reset_buf.any()):
            break
    task.export_recording()
    got = dict(np.load(task._rec_path))
    for k in ("qpos", "motion_ids", "reset"):
        assert np.array_equal(got[k], want[k]), k


def test_motion_assets_record_each_envs_asset(tmp_path):
    from test_gpu_assets import scaled
    from vid2player3d_b200 import model_compiler
    big = dict(scaled(model_compiler.load_compiled("smpl_mesh_humanoid_amass_v1"), 1.1), name="smpl_big")
    entries = ["mjcf/smpl_mesh_humanoid_amass_v1.xml" if m % 2 == 0 else big for m in range(4)]
    task = rec_task(b200_record_envs="all", num_rec_frames=3, motion_assets=entries)
    rec, _, exited = run(task, tmp_path, "assets", True)
    mids = task._reset_ref_motion_ids.cpu().numpy()
    assert exited and list(rec["asset"]) == ["smpl_mesh_humanoid_amass_v1.xml" if m % 2 == 0 else "smpl_big" for m in mids]


def test_without_the_key_nothing_is_recorded():
    torch.manual_seed(0)
    task = make_task(64)
    task.reset()
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    assert task.render_vis(init=True) is None and task.render_vis() is None
    assert task._rec is None and torch.cuda.memory_allocated() == before
