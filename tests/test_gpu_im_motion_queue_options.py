"""GPU checks of the imitation test run's motion queue (cfg.env.b200_motion_queue) with the test-run options it accepts, held to the
composed float64 restatements (oracle/ref_port_motion_queue.QueueRun with ref_port_pose_metrics.PoseMetrics, ref_port_transforms,
ref_port_record) rather than only graphed against eager:

1. the queue fold b200env_im_motion_queue_stats in both forms, driven with b200env_play_stats and b200env_im_motion_queue in the
   task's order over random done sequences: counts and successes exact, the root-relative, velocity and acceleration sums within
   1e-9 relative, PA-MPJPE within 1e-7, the largest error within 1e-12 and NaN where the restatement has NaN; the meters' columns
   bitwise those of the launches without the pose fields; graph replays bitwise eager; the stop flag freezing every row; every row
   written once;
2. non-finite games through the queue: a NaN or +-Inf body position of one env at one step poisons that game's entry only, the
   env's later entries are finite, every other row is bitwise that of the clean run; and a run_test whose env goes non-finite mid-game
   still plays every entry once, as the restatement on its own inputs;
3. the masked reset's window offset with device transforms (reset_context_ofs_xf_kernel) against the launch without transforms and
   the transforms restated from the counter draws at window slot j, and a queued run_test with transforms;
4. per-motion bodies with the pose metrics and the recorder: the metrics file and every recorded frame (motion id, reset flag, asset,
   qpos) against the restatements, the recorder's quit before the queue empties, graphed against eager and a seed against itself.

Not covered here: a poisoned dual tennis test run."""
import contextlib
import io

import numpy as np
import pytest
import torch

import test_gpu_im_motion_queue as GQ
import test_gpu_im_motion_queue_assets as GA
import test_gpu_im_pose_metrics as PM
from oracle import ref_port_motion_queue as Q
from oracle import ref_port_record as REC
from oracle import ref_port_transforms as X
from test_gpu_im_policy import network
from test_gpu_im_record import assert_rows
from test_gpu_im_transforms import ALL, CASES, SPECS, plain_task
from test_gpu_im_reset_masked import N as N_RAGGED, reset_mask_of

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
NB, NBL = PM.NB, PM.NBL
THRESHOLD = 0.5
TIE = slice(5, None, 13)        # envs whose every body sits exactly THRESHOLD from its target: a largest error equal to the threshold
GRID = {"N": lambda N: (N, 1), "N+1": lambda N: (N + 1, 1), "3N+5": lambda N: (3 * N + 5, 1), "3(N+2)": lambda N: (N + 2, 3)}


# ---------------------------------------------------------------------------------------------------------- 1. the queue fold
class Pipeline:
    """the queue's device state and the per-entry meters (pose=True: with the pose fields), stepped as the task steps them"""

    def __init__(self, N, M, R, pose):
        self.N, self.M, self.R = N, M, R
        self.q, self.st = GQ.queue_buffers(N, M, R, np.random.default_rng(7))
        self.ms = PM.buffers(N, M * R, np.zeros(N, np.int64), pose=pose)
        for k in ("motion_start", "motion_envs"):            # the queue fold reads the entries, not the env lists
            del self.ms[k]
        self.ms["env_entry"] = self.q["entry"]
        self.q["env_flags"] = self.ms["env_flags"]           # the assignment clears a restarted env's done memory

    def step(self, x):
        from vid2player3d_b200 import native
        N, Qn = self.N, self.M * self.R
        native.im_motion_queue_stats(dict(n=N, num_motions=Qn, num_bodies=NB, num_lib_bodies=NBL, success_threshold=THRESHOLD),
                                     dict(x, **self.ms, games=self.st["games"]))
        self.q["reset_buf"].copy_(x["reset_buf"])
        GQ.device_step(N, self.M, self.R, self.q, self.st)

    def state(self):
        return {k: v.clone() for d in (self.q, self.st, self.ms) for k, v in d.items()}


def step_inputs(N, rb, seed, poison=None):
    """one step's meters inputs on the done flags rb (PM.inputs, and the TIE envs' bodies THRESHOLD along x from targets on a grid of
    2^-8, so that the error is THRESHOLD exactly in float32 and double); poison (env, value): that value in body 5's y of env"""
    x = PM.inputs(N, seed, rb)
    t = torch.round(x["target_rb_pos"][TIE] * 256.0) / 256.0
    x["target_rb_pos"][TIE] = t
    x["rigid_body_state"][TIE, :NBL, :3] = t + torch.tensor([THRESHOLD, 0.0, 0.0], device=DEV)
    if poison is not None:
        x["rigid_body_state"][poison[0], 5, 1] = poison[1]
    return x


def oracle_step(ora, x):
    h = lambda k: x[k].double().cpu().numpy()  # noqa: E731
    return ora.step(h("rew"), h("sub_rewards"), h("reset_buf"), h("terminate_buf"), h("rigid_body_state")[:, :NBL, :3], h("target_rb_pos"))


def drive(N, M, R, seed, pipes, ora=None, steps=200, poison=None, stop_at=None, end=None):
    """random done sequences (sticky until the queue restarts the env) through every pipeline and the restatement; poison
    (step, env, value); end (step, env): that env's game ends at that step; stop_at: the stop flag set from that step on.
    Returns the number of steps run."""
    g = np.random.default_rng(seed)
    rb = np.zeros(N, np.int64)
    for k in range(steps):
        rb[g.random(N) < 0.3] = 1
        if end is not None and k == end[0]:
            rb[end[1]] = 1
        if stop_at is not None and k == stop_at:
            for p in pipes:
                p.st["games"][1] = 1
            if ora is not None:
                ora.queue.stop = True
        x = step_inputs(N, rb, 1000 * seed + k, poison[1:] if poison is not None and poison[0] == k else None)
        for p in pipes:
            p.step(x)
        if ora is not None:
            mask = oracle_step(ora, x)
            assert np.array_equal(pipes[0].q["mask"].cpu().numpy(), mask), k
        else:
            mask = pipes[0].q["mask"].cpu().numpy()
        rb[mask] = 0
        if ora is not None and ora.queue.stop and stop_at is None:
            return k + 1
    return steps


def assert_rows_are_the_restatement(p, ora, rows=slice(None)):
    ms, st = p.ms, ora.stats
    assert np.array_equal(ms["counts"].cpu().numpy()[rows], st.counts[rows])
    np.testing.assert_allclose(ms["sums"].cpu().numpy()[rows], st.sums[rows], rtol=1e-9, atol=0)
    ps = ms["pose_sums"].cpu().numpy()[rows]
    assert np.array_equal(ps[:, 4:6], st.pose_sums[rows, 4:6]) and np.array_equal(ms["success"].cpu().numpy()[rows], st.success[rows])
    for c, rtol in ((0, 1e-9), (1, 1e-7), (2, 1e-9), (3, 1e-9), (6, 1e-12)):
        np.testing.assert_allclose(ps[:, c], st.pose_sums[rows, c], rtol=rtol, atol=1e-12, err_msg=f"pose column {c}")
    assert np.array_equal(p.q["game_env"].cpu().numpy(), ora.queue.game_env)
    assert np.array_equal(p.q["game_start_step"].cpu().numpy(), ora.queue.game_start_step)


@pytest.mark.parametrize("N", [1, 33, 1024, 8197])
@pytest.mark.parametrize("MR", list(GRID))
def test_queue_fold_is_the_restatement_in_both_forms(N, MR):
    M, R = GRID[MR](N)
    pose, meters = Pipeline(N, M, R, True), Pipeline(N, M, R, False)
    ora = Q.QueueRun(N, M, R, pose_threshold=THRESHOLD)
    drive(N, M, R, N + M * R, [pose, meters], ora)
    torch.cuda.synchronize()
    assert ora.queue.stop and (ora.stats.counts[:, 0] == 1).all()
    assert_rows_are_the_restatement(pose, ora)
    if N > 5:
        assert 0 < ora.stats.success.sum() < M * R
        assert (ora.stats.pose_sums[:, 6] == THRESHOLD).any() and (ora.stats.pose_sums[:, 6] > THRESHOLD).any()
    for k in ("counts", "sums", "env_sums", "env_flags"):
        assert torch.equal(pose.ms[k], meters.ms[k]), k
    for k in pose.q:
        assert torch.equal(pose.q[k], meters.q[k]), k


def test_replays_are_bitwise_eager():
    N, M, R = 1024, 700, 3
    g = np.random.default_rng(5)
    rb = np.zeros(N, np.int64)
    eager, graphed = Pipeline(N, M, R, True), Pipeline(N, M, R, True)
    x = None
    gr = None
    for k in range(14):
        rb[g.random(N) < 0.2] = 1
        xk = step_inputs(N, rb, k)
        eager.step(xk)
        if gr is None:
            x = {n: v.clone() for n, v in xk.items()}
            graphed.step(x)
            torch.cuda.synchronize()
            gr = torch.cuda.CUDAGraph()
            with torch.cuda.graph(gr):
                graphed.step(x)
        else:
            for n in x:
                x[n].copy_(xk[n])
            gr.replay()
        mask = eager.q["mask"].cpu().numpy()
        assert np.array_equal(graphed.q["mask"].cpu().numpy(), mask), k
        rb[mask] = 0
    a, b = eager.state(), graphed.state()
    for k in a:
        assert a[k].cpu().numpy().tobytes() == b[k].cpu().numpy().tobytes(), k
    assert int(eager.q["cursor"][0]) > N


def test_the_stop_flag_freezes_every_row():
    N, M, R = 1024, 1500, 2
    p = Pipeline(N, M, R, True)
    ora = Q.QueueRun(N, M, R, pose_threshold=THRESHOLD)
    drive(N, M, R, 3, [p], ora, steps=6)
    torch.cuda.synchronize()
    assert not ora.queue.stop
    before = p.state()
    drive(N, M, R, 4, [p], ora, steps=6, stop_at=0)
    torch.cuda.synchronize()
    after = p.state()
    assert int(after["games"][0]) == int(before["games"][0])
    for k in before:
        if k not in ("reset_buf", "mask", "games"):            # the flags the test writes
            assert before[k].cpu().numpy().tobytes() == after[k].cpu().numpy().tobytes(), k
    assert_rows_are_the_restatement(p, ora)


def test_every_row_is_written_once():
    """a budget too short for the queue: the rows of entries that never finish stay zero; a second run of the same inputs with NaN in
    those rows, and -Inf (the largest error's identity) in the others' largest error, leaves them NaN and every other row as the first
    run wrote it"""
    N, M, R = 256, 300, 3
    runs = []
    for sentinel in (False, True):
        p = Pipeline(N, M, R, True)
        ora = Q.QueueRun(N, M, R, pose_threshold=THRESHOLD)
        if sentinel:
            for k in ("sums", "pose_sums"):
                p.ms[k][unfinished] = float("nan")
            p.ms["pose_sums"][~unfinished, 6] = float("-inf")
        drive(N, M, R, 9, [p], ora, steps=12)
        torch.cuda.synchronize()
        runs.append(p)
        if not sentinel:
            counts = p.ms["counts"][:, 0].cpu().numpy()
            unfinished = torch.from_numpy(counts == 0).to(DEV)
            assert 0 < (counts == 0).sum() < M * R and (counts <= 1).all()
            assert_rows_are_the_restatement(p, ora)
            for k in ("sums", "pose_sums", "counts", "success"):
                assert not p.ms[k][unfinished].any(), k
            played = ora.queue.game_env[counts > 0]
            assert np.bincount(played, minlength=N).max() >= 2         # some env wrote two rows
    a, b = runs
    for k in ("sums", "pose_sums"):
        assert torch.isnan(b.ms[k][unfinished]).all(), k
        assert a.ms[k][~unfinished].cpu().numpy().tobytes() == b.ms[k][~unfinished].cpu().numpy().tobytes(), k
    for k in ("counts", "success"):
        assert torch.equal(a.ms[k], b.ms[k]), k


# ---------------------------------------------------------------------------------------------------------- 2. non-finite games
@pytest.mark.parametrize("env", [0, 31, 32, "last"])
@pytest.mark.parametrize("value", [float("nan"), float("inf"), float("-inf")], ids=["nan", "+inf", "-inf"])
def test_a_non_finite_game_poisons_its_own_entry_only(env, value):
    N = 1024
    M, R = N + 2, 3
    e = N - 1 if env == "last" else env
    clean, poisoned = Pipeline(N, M, R, True), Pipeline(N, M, R, True)
    drive(N, M, R, 11, [clean], steps=60, end=(4, e))
    ora = Q.QueueRun(N, M, R, pose_threshold=THRESHOLD)
    drive(N, M, R, 11, [poisoned], ora, steps=60, poison=(0, e, value), end=(4, e))
    torch.cuda.synchronize()
    assert ora.queue.stop
    assert_rows_are_the_restatement(poisoned, ora)
    mine = np.flatnonzero(ora.queue.game_env == e)
    assert mine[0] == e and len(mine) >= 2                                   # entry e, then at least one more
    ps, sums = poisoned.ms["pose_sums"].cpu().numpy(), poisoned.ms["sums"].cpu().numpy()
    assert np.isnan(ps[e, 6]) and int(poisoned.ms["success"][e]) == 0
    assert np.isfinite(ps[mine[1:]]).all() and np.isfinite(sums[mine[1:]]).all()
    others = torch.ones(M * R, dtype=torch.bool, device=DEV)
    others[e] = False
    for k in ("counts", "sums", "pose_sums", "success"):
        assert clean.ms[k][others].cpu().numpy().tobytes() == poisoned.ms[k][others].cpu().numpy().tobytes(), k


def capture(task, record):
    """each step's meters inputs, as the meters launch reads them, and whether the stop flag was set when it ran"""
    launch = task._motion_stats_launch

    def rec(games=None):
        record.append(dict(rew=task.rew_buf.clone(), sub_rewards=task._sub_rewards.clone(), reset_buf=task.reset_buf.clone(),
                           terminate_buf=task._terminate_buf.clone(),
                           rigid_body_state=task._rigid_body_state.view(task.num_envs, -1, 13).clone(),
                           target_rb_pos=task._prev_target_rb_pos.clone(), stop=bool(games[1]) if games is not None else False))
        launch(games)
    task._motion_stats_launch = rec


def replay(N, M, R, record):
    ora = Q.QueueRun(N, M, R, pose_threshold=0.5)
    for x in record:
        if x["stop"]:
            ora.queue.stop = True
        oracle_step(ora, x)
    return ora


def assert_file(got, ora):
    counts, sums = ora.per_motion()
    ps, success = ora.per_motion_pose()
    assert np.array_equal(got["games"], counts[:, 0]) and np.array_equal(got["falls"], counts[:, 1])
    assert np.array_equal(got["steps"], sums[:, 1].astype(np.int64)) and np.array_equal(got["success"], success)
    np.testing.assert_allclose(got["reward_sum"], sums[:, 0], rtol=1e-9)
    np.testing.assert_allclose(got["sub_reward_sum"], sums[:, 2:6], rtol=1e-9)
    np.testing.assert_allclose(got["body_pos_err_sum"], sums[:, 6], rtol=1e-9)
    assert np.array_equal(got["vel_frames"], ps[:, 4].astype(np.int64)) and np.array_equal(got["acc_frames"], ps[:, 5].astype(np.int64))
    for k, c, rtol in (("mpjpe_l_sum", 0, 1e-9), ("mpjpe_pa_sum", 1, 1e-7), ("vel_err_sum", 2, 1e-9), ("acc_err_sum", 3, 1e-9),
                       ("max_body_pos_err", 6, 1e-12)):
        np.testing.assert_allclose(got[k], ps[:, c], rtol=rtol, atol=1e-12, err_msg=k)
    assert np.array_equal(got["game_env"].ravel(), ora.queue.game_env)
    assert np.array_equal(got["game_start_step"].ravel(), ora.queue.game_start_step)
    assert np.array_equal(np.sort(got["unfinished"]), np.flatnonzero(ora.stats.counts[:, 0] == 0))


def test_run_test_with_an_env_gone_non_finite_plays_every_entry_once(tmp_path):
    N, R = 32, 2
    M = 3 * N + 5
    task = GQ.vis_task(N, GQ.lib(M, 40, 6), b200_motion_queue=True, b200_motion_queue_repeats=R, b200_motion_stats=True,
                       b200_pose_metrics=True)
    record = []
    capture(task, record)
    e, at = 5, 10
    launches = task._test_launches

    def poisoned():
        if len(record) == at:                               # mid-game: env e's joints go non-finite before the step
            task._dof_state.view(N, -1, 2)[e, 3, 0] = float("nan")
        launches()
    task._test_launches = poisoned
    res, got, _ = GQ.run(task, tmp_path / "nan.npz", graph=False)
    assert got["games"].tolist() == [R] * M and got["unfinished"].size == 0 and res["games_played"] == M * R
    ora = replay(N, M, R, record)
    assert_file(got, ora)
    mine = np.flatnonzero(ora.queue.game_env == e)
    ps = task._ms["pose_sums"].cpu().numpy()
    assert np.isnan(ps[mine[0], 6]) and len(mine) >= 2
    assert np.isfinite(ps[mine[1:]]).all(), "a game restarted after a non-finite one is not finite"
    assert np.isfinite(np.delete(ps, mine[0], 0)).all()


# ---------------------------------------------------------------------------------------------------------- 3. device transforms
def masked_reset(t, mask, s, prog, feat, fmask, counter, seed=10):
    L, pad = t.context_length, t.context_padding
    t._reset_rng.fill_(counter)
    step = torch.full((1,), s, device=DEV, dtype=torch.long)
    t._env.reset_masked(mask, True, L * t.dt if t.truncate_time else 0.0, 1.0, seed, t._reset_rng, t._initial_humanoid_root_states,
                        t._initial_dof_pos, t._initial_dof_vel, t._reset_ref_motion_times, L + 2 * pad, -pad, t.dt, feat, fmask,
                        t._reset_work, transforms=prog, step=step, context_length=L)


@pytest.mark.parametrize("N", [1, N_RAGGED, 8192])
def test_offset_window_with_transforms_is_the_restatement(N):
    from vid2player3d_b200 import abi
    t = plain_task(N)
    nb, L, pad = t._num_lib_bodies, t.context_length, t.context_padding
    P, W = L + 2 * pad, 2 * (3 * nb + t.num_dof) + 4 * nb
    m = np.ones(1, bool) if N == 1 else reset_mask_of(N) if N == N_RAGGED else np.random.default_rng(2).random(N) < 0.5
    rows = np.flatnonzero(m)
    check = rows if N < 8192 else np.unique(np.r_[rows[0], rows[-1], np.random.default_rng(1).choice(rows, 200)])
    mask = torch.from_numpy(m).to(DEV)
    seed, counter = 10, 6
    plain, m0 = torch.full((N, P, W), 7.0, device=DEV), torch.zeros(N, P, dtype=torch.bool, device=DEV)
    feat, m1 = torch.full((N, P, W + nb), 7.0, device=DEV), torch.zeros(N, P, dtype=torch.bool, device=DEV)
    for s in (0, 1, L - 1, L + 1, 2 * L + 6):
        plain.fill_(7.0)
        m0.fill_(True)
        masked_reset(t, mask, s, None, plain, m0, counter, seed)
        assert int(t._reset_rng.item()) == counter + 1
        pos = plain[check, :, :3 * nb].reshape(len(check), P, nb, 3).double().cpu().numpy()
        for name in CASES:
            specs = SPECS[name]
            feat.fill_(7.0)
            m1.fill_(True)
            masked_reset(t, mask, s, abi.transform_program(specs, t.body_names, nb), feat, m1, counter, seed)
            assert int(t._reset_rng.item()) == counter + 1, (s, name)
            assert torch.equal(m0, m1), (s, name)
            assert torch.equal(feat[..., 3 * nb:W].view(torch.int32), plain[..., 3 * nb:].view(torch.int32)), (s, name)
            assert bool((feat[~mask] == 7.0).all()), (s, name)
            noisy, noise, drop = X.draws(seed, counter, N, check, P, nb, specs)
            want_pos, want_conf = X.transform_target(pos, specs, t.body_names, noisy=noisy, noise=noise, drop=drop)
            got_pos = feat[check, :, :3 * nb].reshape(len(check), P, nb, 3).double().cpu().numpy()
            got_conf = feat[check, :, W:].double().cpu().numpy()
            keep = np.ones(noisy.shape, bool)
            if "noisy_joints" in specs:
                keep = np.abs(X.pre_occlusion_conf(specs, noisy, noise) - specs["noisy_joints"]["min_conf"]) >= 1e-6
            assert np.abs(got_pos - want_pos)[keep].max() <= 1e-5, (s, name, "body_pos")
            assert np.abs(got_conf - want_conf)[keep].max() <= 1e-5, (s, name, "joint_conf")
            assert np.array_equal(got_conf[keep] == 0, want_conf[keep] == 0), (s, name, "occlusion decisions")
        assert bool((plain[~mask] == 7.0).all()) and bool(m0[~mask].all())


def test_run_test_with_transforms_plays_every_entry_once(tmp_path):
    N = 32
    M = 3 * N + 5
    flat = GQ.lib(M, 40, 6)
    files = {}
    for name, graph in (("g1", True), ("g2", True), ("eager", False)):
        task = GQ.vis_task(N, flat, b200_motion_queue=True, b200_motion_stats=True, transform_specs=ALL, b200_device_transforms=True)
        res, files[name], _ = GQ.run(task, tmp_path / f"{name}.npz", graph=graph)
        assert files[name]["games"].tolist() == [1] * M and files[name]["unfinished"].size == 0 and res["games_played"] == M
        assert int(task._reset_rng.item()) > 1
    for other in ("g2", "eager"):
        assert files[other].keys() == files["g1"].keys()
        for k, v in files["g1"].items():
            assert v.dtype == files[other][k].dtype and v.tobytes() == files[other][k].tobytes(), (other, k)


# ---------------------------------------------------------------------------------------------------------- 4. bodies and recorder
N_E, R_E = 16, 2
M_E = 3 * N_E + 5


def recorded_task(frames):
    """three bodies, named apart so that the recording's per-frame asset tells them apart"""
    import types
    from vid2player3d_b200.configs import SIM_PARAMS, im_cfg
    from vid2player3d_b200.tasks import HumanoidSMPLIMVis
    b = [dict(x, name=f"smpl_{k}") for k, x in enumerate(GA.bodies())]
    entries = [b[m % 3] for m in range(M_E)]
    cfg = im_cfg(N_E, GQ.lib(M_E, 40, 6), b200_motion_queue=True, motion_assets=entries, test_motion_assets=entries,
                 b200_motion_queue_repeats=R_E, b200_motion_stats=True, b200_pose_metrics=True, b200_record_qpos=True,
                 b200_record_envs="all", num_rec_frames=frames)
    cfg["args"] = types.SimpleNamespace(test=True)
    torch.manual_seed(0)
    return HumanoidSMPLIMVis(cfg, SIM_PARAMS, 1, "cuda", 0, True)


def recorded_run(task, tmp_path, name, graph, record=None, frames=None):
    """(metrics file, recording file, exited); record: the meters inputs per step; frames: the state each recorded frame reads"""
    task._rec_path = str(tmp_path / f"{name}_rec.npz")
    task.cfg["env"]["b200_motion_stats_file"] = str(tmp_path / f"{name}.npz")
    if record is not None:
        capture(task, record)
    if frames is not None:
        launch = task._record_launch

        def rec(init, games=None):
            n = task.num_envs
            frames.append(dict(rbs=task._rigid_body_state.view(n, -1, 13).double().cpu().numpy(),
                               dof=task._dof_pos.double().cpu().numpy(), p_rb_pos=task._prev_target_rb_pos.double().cpu().numpy(),
                               p_rb_rot=task._prev_target_rb_rot.double().cpu().numpy(),
                               p_dof=task._prev_target_dof_pos.double().cpu().numpy(), reset=task.reset_buf.cpu().numpy(), init=init))
            launch(init, games)
        task._record_launch = rec
    exited = False
    with contextlib.redirect_stdout(io.StringIO()):
        try:
            task.run_test(network(5)[0], 1, 3000, graph=graph, clip_actions=1.0)
        except SystemExit:
            exited = True
    return dict(np.load(tmp_path / f"{name}.npz")), dict(np.load(task._rec_path)), exited


def motion_at(queue, M, T):
    """[N, T] the motion each env plays at recorded frame f (frame 0 the reset, frame f >= 1 after step f)"""
    N = len(queue.entry)
    out = np.zeros((N, T), np.int64)
    for f in range(T):
        for e in range(N):
            q = np.flatnonzero((queue.game_env == e) & (queue.game_start_step < max(f, 1)))
            out[e, f] = q.max() % M
    return out


def test_bodies_pose_metrics_and_recorder_are_the_restatement(tmp_path):
    task = recorded_task(1000)
    record, frames = [], []
    got, rec, exited = recorded_run(task, tmp_path, "eager", False, record=record, frames=frames)
    assert not exited and got["games"].tolist() == [R_E] * M_E and got["unfinished"].size == 0
    ora = replay(N_E, M_E, R_E, record)
    assert_file(got, ora)
    T = rec["qpos"].shape[1]
    assert T < task._rec_cap and T == 1 + sum(not x["stop"] for x in record)     # the recorder stops with the queue
    frames = frames[:T]
    mids = motion_at(ora.queue, M_E, T)
    assert np.array_equal(rec["motion_ids"], mids)
    assert (mids != mids[:, :1]).any(axis=1).all()                       # every env restarted on another motion
    assert np.array_equal(rec["reset"][:, 0], np.zeros(N_E)) and np.array_equal(rec["reset"][:, 1:].T, [f["reset"] for f in frames[1:]])
    names = task._rec_motion_asset
    assert np.array_equal(rec["asset"], names[mids]) and names[:3].tolist() == ["smpl_0", "smpl_1", "smpl_2"]
    qpos = task._rec["qpos"][:, :T].double().cpu().numpy()
    ids = np.arange(N_E)
    for f, x in enumerate(frames):
        want = REC.sync_ref_motion(x["rbs"][..., :3], x["rbs"][..., 3:7], x["dof"], x["p_rb_pos"], x["p_rb_rot"], x["p_dof"], ids,
                                   x["init"])
        assert_rows(qpos[:, f], want[:, :2 * qpos.shape[-1]].reshape(N_E, 2, -1))
    # the recorder fills before the queue empties: the metrics of the games finished when it quit
    quit_task = recorded_task(T // 2)
    qrecord = []
    qgot, qrec, exited = recorded_run(quit_task, tmp_path, "quit", False, record=qrecord)
    assert exited and qrec["qpos"].shape[1] == T // 2 and not qrecord[0]["stop"] and qrecord[-1]["stop"]
    qora = replay(N_E, M_E, R_E, qrecord)
    assert_file(qgot, qora)
    assert 0 < qgot["unfinished"].size < M_E * R_E and np.array_equal(qrec["qpos"], rec["qpos"][:, :T // 2])
    # graphed against eager and a seed against itself, both files bit for bit
    for name in ("g1", "g2"):
        g, r, _ = recorded_run(recorded_task(1000), tmp_path, name, True)
        for want, have in ((got, g), (rec, r)):
            assert want.keys() == have.keys()
            for k, v in want.items():
                assert v.dtype == have[k].dtype and v.tobytes() == have[k].tobytes(), (name, k)
