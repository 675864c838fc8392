"""GPU checks of HumanoidSMPLIMVis' per-motion meters and held-out library: the launch b200env_im_motion_stats against the float64
restatement oracle/ref_port_motion_stats.py at several env and motion counts (uneven envs per motion, games ending, falls, new games,
the stop flag), and run_test with cfg.env.b200_motion_stats: the restatement on the device's own per-step inputs, the games, reward and
steps of the bookkeeping, graphed against eager, two runs of one seed, a test_motion_file of other motions, and the task without the
key.  Counts are exact; the float64 sums within 1e-9 relative (the launch sums the body distances in another order)."""
import io
import contextlib
import os
import types

import numpy as np
import pytest
import torch

from oracle import ref_port_motion_stats as R
from test_gpu_im_policy import network

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
NB, NBL = 24, 24


def motion_map(N, M, seed):
    """uneven envs per motion: motion m takes about a share proportional to m + 1, some motions none"""
    g = np.random.default_rng(seed)
    w = np.arange(1, M + 1, dtype=np.float64) ** 2
    return g.choice(M, size=N, p=w / w.sum()).astype(np.int64)


def inputs(N, seed, done):
    g = torch.Generator().manual_seed(seed)
    rbs = torch.randn(N, NB, 13, generator=g)
    return dict(rew=torch.rand(N, generator=g).to(DEV), sub_rewards=torch.rand(N, 4, generator=g).to(DEV),
                reset_buf=torch.from_numpy(done.astype(np.int64)).to(DEV),
                terminate_buf=torch.randint(0, 2, (N,), generator=g).to(DEV) * torch.from_numpy(done.astype(np.int64)).to(DEV),
                rigid_body_state=rbs.to(DEV), target_rb_pos=torch.randn(N, NBL, 3, generator=g).to(DEV))


def buffers(N, M, mids):
    from vid2player3d_b200.tasks.humanoid_smpl_im_vis import motion_env_lists
    start, envs = motion_env_lists(mids, M)
    return dict(motion_start=torch.from_numpy(start).to(DEV), motion_envs=torch.from_numpy(envs).to(DEV),
                env_sums=torch.zeros(N, 7, device=DEV, dtype=torch.float64), env_flags=torch.zeros(N, 2, device=DEV, dtype=torch.int32),
                counts=torch.zeros(M, 2, device=DEV, dtype=torch.long), sums=torch.zeros(M, 7, device=DEV, dtype=torch.float64))


def launch(N, M, x, buf, games=None):
    from vid2player3d_b200 import native
    native.im_motion_stats(dict(n=N, num_motions=M, num_bodies=NB, num_lib_bodies=NBL), dict(x, **buf, games=games))


def oracle_step(ms, x, stop=False):
    h = lambda k: x[k].double().cpu().numpy()  # noqa: E731
    ms.step(h("rew"), h("sub_rewards"), h("reset_buf"), h("terminate_buf"), h("rigid_body_state")[:, :NBL, :3], h("target_rb_pos"), stop)


def assert_buckets(buf, ms):
    assert np.array_equal(buf["counts"].cpu().numpy(), ms.counts)
    np.testing.assert_allclose(buf["sums"].cpu().numpy(), ms.sums, rtol=1e-9, atol=0)


@pytest.mark.parametrize("N", [1, 33, 8197])
@pytest.mark.parametrize("M", [1, 3, 1000])
def test_launch_is_the_restatement(N, M):
    """two games: envs finish at random steps and stay done (some drop back and finish again), the stop flag holds one step, then a
    new game starts from zero"""
    mids = motion_map(N, M, N + M)
    buf, ms = buffers(N, M, mids), R.MotionStats(mids, M)
    games = torch.zeros(3, device=DEV, dtype=torch.long)
    g = np.random.default_rng(N * M)
    for game in range(2):
        if game:
            buf["env_sums"].zero_()
            buf["env_flags"].zero_()
            ms.new_game()
        end = g.integers(1, 9, N)
        for k in range(10):
            done = k >= end
            done[g.random(N) < 0.05] = False                 # a few envs drop back: their next rise is a new game
            stop = game == 0 and k == 6
            games[1] = int(stop)
            x = inputs(N, 1000 * game + k, done)
            launch(N, M, x, buf, games)
            oracle_step(ms, x, stop)
        torch.cuda.synchronize()
        assert_buckets(buf, ms)
    assert ms.counts[:, 0].sum() > 0
    assert not ms.counts[np.setdiff1d(np.arange(M), mids)].any()    # motions without envs: no games


def test_replays_give_the_same_bits():
    N, M = 8197, 1000
    mids = motion_map(N, M, 5)
    xs = [inputs(N, k, np.random.default_rng(k).random(N) < 0.1 * k) for k in range(6)]
    eager = buffers(N, M, mids)
    for x in xs:
        launch(N, M, x, eager)
    graphed = buffers(N, M, mids)
    x = {k: torch.empty_like(v) for k, v in xs[0].items()}
    for k in x:
        x[k].copy_(xs[0][k])
    launch(N, M, x, graphed)                                 # the first step eagerly, then the captured launch
    torch.cuda.synchronize()
    gr = torch.cuda.CUDAGraph()
    with torch.cuda.graph(gr):                               # capturing does not run the launch
        launch(N, M, x, graphed)
    for xk in xs[1:]:
        for k in x:
            x[k].copy_(xk[k])
        gr.replay()
    torch.cuda.synchronize()
    for k in ("counts", "sums", "env_sums", "env_flags"):
        assert torch.equal(eager[k], graphed[k]), k


# ---------------------------------------------------------------------------------------------------------- run_test
def vis_task(N, flat, test=False, **over):
    from vid2player3d_b200.configs import SIM_PARAMS, im_cfg
    from vid2player3d_b200.tasks import HumanoidSMPLIMVis
    cfg = im_cfg(N, flat, stateInit="Start", b200_motion_stats=True, **over)
    cfg["args"] = types.SimpleNamespace(test=test)
    torch.manual_seed(0)
    return HumanoidSMPLIMVis(cfg, SIM_PARAMS, 1, "cuda", 0, True)


def train_lib():
    from vid2player3d_b200 import model_compiler, motion_lib
    return motion_lib.synthetic(model_compiler.load_compiled("smpl_mesh_humanoid_amass_v1"), num_motions=4, num_frames=60, seed=1)


def run(task, path, graph=True, games_num=3, max_steps=80, record=None):
    task.cfg["env"]["b200_motion_stats_file"] = str(path)
    if record is not None:                                   # the device's per-step inputs and the stop flag each step saw
        step, reset = task.test_step, task.reset

        def rec_step(n, graph=True):
            stop = bool(task._stats["games"][1])
            step(n, graph)
            record.append(("step", stop, dict(rew=task.rew_buf.clone(), sub_rewards=task._sub_rewards.clone(),
                                              reset_buf=task.reset_buf.clone(), terminate_buf=task._terminate_buf.clone(),
                                              rigid_body_state=task._rigid_body_state.view(task.num_envs, -1, 13).clone(),
                                              target_rb_pos=task._prev_target_rb_pos.clone())))

        def rec_reset(*a, **k):
            record.append(("game", None, None))
            return reset(*a, **k)
        task.test_step, task.reset = rec_step, rec_reset
    out = io.StringIO()
    with contextlib.redirect_stdout(out):
        res = task.run_test(network(5)[0], games_num, max_steps, graph=graph, clip_actions=1.0)
    return res, dict(np.load(path)), out.getvalue().splitlines()


def test_run_test_is_the_restatement_and_the_bookkeeping(tmp_path):
    task = vis_task(64, train_lib(), sample_first_motions=True)
    record = []
    res, got, lines = run(task, tmp_path / "a.npz", record=record)
    mids = task._reset_ref_motion_ids.cpu().numpy()
    ms = R.MotionStats(mids, 4)
    for kind, stop, x in record:
        if kind == "game":
            ms.new_game()
        else:
            oracle_step(ms, x, stop)
    assert np.array_equal(got["games"], ms.counts[:, 0]) and np.array_equal(got["falls"], ms.counts[:, 1])
    np.testing.assert_allclose(got["reward_sum"], ms.sums[:, 0], rtol=1e-9)
    assert np.array_equal(got["steps"], ms.sums[:, 1].astype(np.int64))
    np.testing.assert_allclose(got["sub_reward_sum"], ms.sums[:, 2:6], rtol=1e-9)
    np.testing.assert_allclose(got["body_pos_err_sum"], ms.sums[:, 6], rtol=1e-9)
    assert got["games"].sum() == res["games_played"] > 0
    np.testing.assert_allclose(got["reward_sum"].sum(), res["sum_rewards"], rtol=1e-5)
    np.testing.assert_allclose(got["steps"].sum(), res["sum_steps"], rtol=1e-6)
    assert np.array_equal(got["env_motion_ids"], mids) and str(got["test_motion_file"]) == ""
    assert any(x.startswith(f"motions evaluated: {int((got['games'] > 0).sum())} of 4") for x in lines)


def test_run_test_graphed_is_eager_and_a_seed_repeats(tmp_path):
    flat = train_lib()
    files = {}
    for name, graph in (("g1", True), ("g2", True), ("eager", False)):
        _, files[name], _ = run(vis_task(64, flat), tmp_path / f"{name}.npz", graph=graph)
    assert files["g1"]["games"].sum() > 0
    for other in ("g2", "eager"):
        assert files[other].keys() == files["g1"].keys()
        for k, v in files["g1"].items():
            assert v.dtype == files[other][k].dtype and v.tobytes() == files[other][k].tobytes(), (other, k)


def test_test_motion_file_serves_the_held_out_motions(tmp_path):
    from vid2player3d_b200 import model_compiler, motion_lib
    test = motion_lib.synthetic(model_compiler.load_compiled("smpl_mesh_humanoid_amass_v1"), num_motions=7, num_frames=45, seed=9)
    path = str(tmp_path / "held_out.npz")
    test.save(path)
    task = vis_task(64, train_lib(), test=True, test_motion_file=path, sample_first_motions=True)
    assert task._motion_lib.num_motions() == 7
    np.testing.assert_array_equal(task._motion_lib.motion_lengths, test.motion_lengths)
    mids = task._reset_ref_motion_ids.cpu().numpy()
    assert sorted(set(mids.tolist())) == list(range(7))
    res, got, _ = run(task, tmp_path / "held_out_stats.npz")
    assert got["games"].shape == (7,) and got["sub_reward_sum"].shape == (7, 4)
    assert got["games"].sum() == res["games_played"] and str(got["test_motion_file"]) == path
    assert np.array_equal(got["env_motion_ids"], mids)
    trained = vis_task(64, train_lib(), test=False, test_motion_file=path, sample_first_motions=True)
    assert trained._motion_lib.num_motions() == 4                 # without args.test the key is ignored


def test_without_the_key_nothing_is_allocated_or_written(tmp_path, monkeypatch):
    from vid2player3d_b200.configs import SIM_PARAMS, im_cfg
    from vid2player3d_b200.tasks import HumanoidSMPLIMVis
    torch.manual_seed(0)
    task = HumanoidSMPLIMVis(im_cfg(64, train_lib(), stateInit="Start"), SIM_PARAMS, 1, "cuda", 0, True)
    monkeypatch.chdir(tmp_path)
    with contextlib.redirect_stdout(io.StringIO()) as out:
        task.run_test(network(5)[0], 3, 80, clip_actions=1.0)
    assert task._ms is None and not os.path.exists(tmp_path / "out")
    assert not any(x.startswith("motions evaluated") for x in out.getvalue().splitlines())
