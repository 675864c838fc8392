"""GPU checks of HumanoidSMPLIMVis' pose metrics (cfg.env.b200_pose_metrics): the launch b200env_im_motion_stats with the pose fields
against the float64 restatement oracle/ref_port_pose_metrics.py at several env and motion counts (random game ends, collinear bodies,
bodies without spread, a NaN env, the stop flag, a new game), the meters' columns unchanged by the pose fields, and run_test with the
key: the restatement on the device's own per-step inputs, graphed against eager, two runs of one seed, a task of several assets, the
recorder's quit, and the task without the key.  Counts are exact; the root-relative, velocity and acceleration sums within 1e-9
relative, PA-MPJPE within 1e-7 (a Jacobi eigen-solve against numpy's SVD)."""
import contextlib
import io

import numpy as np
import pytest
import torch

from oracle import ref_port_pose_metrics as P
from test_gpu_im_motion_stats import motion_map, run, train_lib, vis_task
from test_gpu_im_policy import network

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
NB, NBL = 24, 24


def inputs(N, seed, done, nan_env=None):
    """random poses (a unique alignment), every 7th env's bodies on a line, every 11th env's bodies on one point"""
    g = torch.Generator().manual_seed(seed)
    rbs = torch.randn(N, NB, 13, generator=g)
    tgt = torch.randn(N, NBL, 3, generator=g)
    rbs[:, :, :3] = tgt + 0.2 * torch.randn(N, NBL, 3, generator=g)
    line = torch.linspace(-1.0, 1.0, NB)[:, None] * torch.tensor([0.36, 0.48, 0.8])
    rbs[::7, :, :3] = line + torch.randn(len(range(0, N, 7)), 1, 3, generator=g)
    rbs[3::11, :, :3] = torch.randn(len(range(3, N, 11)), 1, 3, generator=g)
    if nan_env is not None and nan_env < N:
        rbs[nan_env, 5, 1] = float("nan")
    d = torch.from_numpy(done.astype(np.int64))
    return dict(rew=torch.rand(N, generator=g).to(DEV), sub_rewards=torch.rand(N, 4, generator=g).to(DEV), reset_buf=d.to(DEV),
                terminate_buf=(torch.randint(0, 2, (N,), generator=g) * d).to(DEV), rigid_body_state=rbs.to(DEV), target_rb_pos=tgt.to(DEV))


def buffers(N, M, mids, pose=True):
    from vid2player3d_b200.tasks.humanoid_smpl_im_vis import motion_env_lists
    start, envs = motion_env_lists(mids, M)
    b = dict(motion_start=torch.from_numpy(start).to(DEV), motion_envs=torch.from_numpy(envs).to(DEV),
             env_sums=torch.zeros(N, 7, device=DEV, dtype=torch.float64), env_flags=torch.zeros(N, 2, device=DEV, dtype=torch.int32),
             counts=torch.zeros(M, 2, device=DEV, dtype=torch.long), sums=torch.zeros(M, 7, device=DEV, dtype=torch.float64))
    if pose:
        b.update(env_pose=torch.zeros(N, 7, device=DEV, dtype=torch.float64), pose_hist=torch.zeros(N, 2, 2, NBL, 3, device=DEV),
                 pose_fill=torch.zeros(N, device=DEV, dtype=torch.int32), pose_sums=torch.zeros(M, 7, device=DEV, dtype=torch.float64),
                 success=torch.zeros(M, device=DEV, dtype=torch.long))
    return b


def launch(N, M, x, buf, games=None, threshold=0.5):
    from vid2player3d_b200 import native
    native.im_motion_stats(dict(n=N, num_motions=M, num_bodies=NB, num_lib_bodies=NBL, success_threshold=threshold),
                           dict(x, **buf, games=games))


def oracle_step(ms, x, stop=False):
    h = lambda k: x[k].double().cpu().numpy()  # noqa: E731
    ms.step(h("rew"), h("sub_rewards"), h("reset_buf"), h("terminate_buf"), h("rigid_body_state")[:, :NBL, :3], h("target_rb_pos"), stop)


def assert_pose(buf, ms):
    assert np.array_equal(buf["counts"].cpu().numpy(), ms.counts)
    np.testing.assert_allclose(buf["sums"].cpu().numpy(), ms.sums, rtol=1e-9, atol=0)
    ps = buf["pose_sums"].cpu().numpy()
    assert np.array_equal(ps[:, 4:6], ms.pose_sums[:, 4:6]) and np.array_equal(buf["success"].cpu().numpy(), ms.success)
    for c, rtol in ((0, 1e-9), (1, 1e-7), (2, 1e-9), (3, 1e-9), (6, 1e-12)):
        np.testing.assert_allclose(ps[:, c], ms.pose_sums[:, c], rtol=rtol, atol=1e-12, err_msg=f"column {c}")


@pytest.mark.parametrize("N", [1, 33, 8197])
@pytest.mark.parametrize("M", [1, 3, 1000])
def test_launch_is_the_restatement(N, M):
    """two games of up to 50 steps: envs finish at random steps and stay done (some drop back and finish again), the stop flag holds
    one step, env 2 has a NaN body at one step, then a new game starts from zero"""
    mids = motion_map(N, M, N + M)
    buf, ms = buffers(N, M, mids), P.PoseMetrics(mids, M, 0.9)
    games = torch.zeros(3, device=DEV, dtype=torch.long)
    g = np.random.default_rng(N * M)
    for game in range(2):
        if game:
            for k in ("env_sums", "env_flags", "env_pose", "pose_fill"):
                buf[k].zero_()
            ms.new_game()
        end = g.integers(1, 48, N)
        for k in range(50):
            done = k >= end
            done[g.random(N) < 0.05] = False
            stop = game == 0 and k == 6
            games[1] = int(stop)
            x = inputs(N, 1000 * game + k, done, nan_env=2 if (game, k) == (0, 3) else None)
            launch(N, M, x, buf, games, 0.9)
            oracle_step(ms, x, stop)
        torch.cuda.synchronize()
        assert_pose(buf, ms)
    assert ms.counts[:, 0].sum() > 0 and (N <= 2 or ms.success.sum() > 0)
    assert np.array_equal(ms.pose_sums[:, 4] + ms.counts[:, 0], ms.sums[:, 1])    # vel frames + games = steps


def test_the_meters_columns_do_not_change():
    """the same inputs with and without the pose fields: counts, sums and the per-env rows bit for bit"""
    N, M = 8197, 1000
    mids = motion_map(N, M, 3)
    on, off = buffers(N, M, mids), buffers(N, M, mids, pose=False)
    g = np.random.default_rng(1)
    end = g.integers(1, 20, N)
    for k in range(24):
        x = inputs(N, k, k >= end)
        launch(N, M, x, on)
        launch(N, M, x, off)
    torch.cuda.synchronize()
    for k in ("counts", "sums", "env_sums", "env_flags"):
        assert torch.equal(on[k], off[k]), k
    assert torch.equal(on["pose_sums"][:, 4].long() + on["counts"][:, 0], on["sums"][:, 1].long())


def test_replays_give_the_same_bits():
    N, M = 8197, 1000
    mids = motion_map(N, M, 5)
    xs = [inputs(N, k, np.random.default_rng(k).random(N) < 0.1 * k) for k in range(6)]
    eager = buffers(N, M, mids)
    for x in xs:
        launch(N, M, x, eager)
    graphed = buffers(N, M, mids)
    x = {k: v.clone() for k, v in xs[0].items()}
    launch(N, M, x, graphed)
    torch.cuda.synchronize()
    gr = torch.cuda.CUDAGraph()
    with torch.cuda.graph(gr):
        launch(N, M, x, graphed)
    for xk in xs[1:]:
        for k in x:
            x[k].copy_(xk[k])
        gr.replay()
    torch.cuda.synchronize()
    for k in eager:
        assert torch.equal(eager[k], graphed[k]), k


# ---------------------------------------------------------------------------------------------------------- run_test
POSE_KEYS = {"mpjpe_l_sum", "mpjpe_pa_sum", "vel_err_sum", "acc_err_sum", "vel_frames", "acc_frames", "success", "max_body_pos_err",
             "success_threshold", "dt"}


def pose_task(N=64, **over):
    return vis_task(N, train_lib(), b200_pose_metrics=True, **over)


def replay_oracle(task, record, threshold=0.5):
    ms = P.PoseMetrics(task._reset_ref_motion_ids.cpu().numpy(), task._motion_lib.num_motions(), threshold)
    for kind, stop, x in record:
        if kind == "game":
            ms.new_game()
        else:
            oracle_step(ms, x, stop)
    return ms


def assert_file(got, ms):
    assert np.array_equal(got["games"], ms.counts[:, 0]) and np.array_equal(got["success"], ms.success)
    assert np.array_equal(got["vel_frames"], ms.pose_sums[:, 4].astype(np.int64))
    assert np.array_equal(got["acc_frames"], ms.pose_sums[:, 5].astype(np.int64))
    for k, c, rtol in (("mpjpe_l_sum", 0, 1e-9), ("mpjpe_pa_sum", 1, 1e-7), ("vel_err_sum", 2, 1e-9), ("acc_err_sum", 3, 1e-9),
                       ("max_body_pos_err", 6, 1e-12)):
        np.testing.assert_allclose(got[k], ms.pose_sums[:, c], rtol=rtol, atol=1e-12, err_msg=k)
    np.testing.assert_allclose(got["body_pos_err_sum"], ms.sums[:, 6], rtol=1e-9)


def test_run_test_is_the_restatement(tmp_path):
    task = pose_task(sample_first_motions=True, b200_pose_success_threshold=0.3)
    record = []
    res, got, lines = run(task, tmp_path / "a.npz", record=record)
    assert_file(got, replay_oracle(task, record, 0.3))
    assert got["games"].sum() == res["games_played"] > 0 and got["success_threshold"] == 0.3 and got["dt"] == task.dt
    assert np.array_equal(got["vel_frames"] + got["games"], got["steps"])
    i = next(i for i, x in enumerate(lines) if x.startswith("motions evaluated"))
    assert lines[i + 1].startswith("success rate: ")


def test_run_test_graphed_is_eager_and_a_seed_repeats(tmp_path):
    files = {}
    for name, graph in (("g1", True), ("g2", True), ("eager", False)):
        _, files[name], _ = run(pose_task(), tmp_path / f"{name}.npz", graph=graph)
    assert files["g1"]["games"].sum() > 0 and POSE_KEYS <= set(files["g1"])
    for other in ("g2", "eager"):
        assert files[other].keys() == files["g1"].keys()
        for k, v in files["g1"].items():
            assert v.dtype == files[other][k].dtype and v.tobytes() == files[other][k].tobytes(), (other, k)


def test_a_task_of_several_assets(tmp_path):
    from test_gpu_assets import scaled
    from vid2player3d_b200 import model_compiler
    big = dict(scaled(model_compiler.load_compiled("smpl_mesh_humanoid_amass_v1"), 1.1), name="smpl_big")
    entries = ["mjcf/smpl_mesh_humanoid_amass_v1.xml" if m % 2 == 0 else big for m in range(4)]
    task = pose_task(sample_first_motions=True, motion_assets=entries)
    record = []
    _, got, _ = run(task, tmp_path / "assets.npz", record=record)
    assert got["games"].sum() > 0
    assert_file(got, replay_oracle(task, record))


def test_the_recorder_quit_writes_the_metrics_first(tmp_path):
    task = pose_task(b200_record_qpos=True, num_rec_frames=3)
    task._rec_path = str(tmp_path / "rec.npz")
    task.cfg["env"]["b200_motion_stats_file"] = str(tmp_path / "quit.npz")
    with contextlib.redirect_stdout(io.StringIO()) as out, pytest.raises(SystemExit):
        task.run_test(network(5)[0], 3, 80, clip_actions=1.0)
    got = dict(np.load(tmp_path / "quit.npz"))
    assert POSE_KEYS <= set(got) and any(x.startswith("success rate: ") for x in out.getvalue().splitlines())


def test_without_the_key_the_meters_launch_as_before(tmp_path, monkeypatch):
    """with b200_motion_stats alone the launch gets no pose pointer (the meters' own kernels) and the file holds the meters' keys"""
    from vid2player3d_b200 import abi, native
    seen = []
    fill = native.fill

    def spy(S, scalars, tensors):
        d = fill(S, scalars, tensors)
        if S is abi.ImMotionStats:
            seen.append((d.env_pose.value, d.pose_hist.value, d.pose_fill.value, d.pose_sums.value, d.success.value))
        return d
    monkeypatch.setattr(native, "fill", spy)
    task = vis_task(64, train_lib())
    _, got, lines = run(task, tmp_path / "off.npz")
    assert seen and all(s == (None,) * 5 for s in seen)
    assert set(got) == {"games", "falls", "reward_sum", "steps", "sub_reward_sum", "body_pos_err_sum", "env_motion_ids",
                        "test_motion_file"}
    assert not any(x.startswith("success rate") for x in lines) and "env_pose" not in task._ms
