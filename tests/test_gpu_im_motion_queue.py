"""GPU checks of the imitation test run's motion queue (cfg.env.b200_motion_queue): the assignment launch b200env_im_motion_queue with
the queue form of b200env_play_stats against oracle/ref_port_motion_queue.py over random done sequences; the masked reset's window
offset against the id-list b200env_motion_context; the operand row of a queued game's first step against step 0 of a game the full
reset started; and run_test over a library larger than the env count: every entry finished once, the per-motion sums against the
restatement on the run's own per-step inputs, graphed against eager and a seed against itself, bit for bit, and nothing launched
without the key."""
import contextlib
import io
import types

import numpy as np
import pytest
import torch

from oracle import ref_port_motion_queue as Q
from test_gpu_im_policy import network

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SHAPE = 11


def queue_buffers(N, M, R, g):
    i64 = lambda *s: torch.zeros(*s, device=DEV, dtype=torch.long)  # noqa: E731
    f32 = lambda *s: torch.zeros(*s, device=DEV)  # noqa: E731
    Qn = M * R
    e = torch.arange(N, device=DEV)
    q = dict(reset_buf=i64(N), lib_motion_bodies=torch.from_numpy(g.standard_normal((M, SHAPE)).astype(np.float32)).to(DEV),
             motion_ids=e % M, motion_bodies=f32(N, SHAPE), entry=e.clone(), mask=torch.zeros(N, device=DEV, dtype=torch.bool),
             idle=torch.zeros(N, device=DEV, dtype=torch.uint8), cursor=torch.full((1,), N, device=DEV, dtype=torch.long),
             game_env=torch.full((Qn,), -1, device=DEV, dtype=torch.long), game_start_step=torch.full((Qn,), -1, device=DEV, dtype=torch.long),
             env_flags=torch.zeros(N, 2, device=DEV, dtype=torch.int32))
    q["game_env"][:N] = e
    q["game_start_step"][:N] = 0
    st = dict(rew=f32(N), cr=f32(N), steps=f32(N), prev_dones=f32(N), totals=torch.zeros(2, device=DEV, dtype=torch.float64),
              log=torch.zeros(4, 3, device=DEV, dtype=torch.float64), games=i64(3), step=i64(1))
    return q, st


def device_step(N, M, R, q, st):
    from vid2player3d_b200 import native
    native.play_stats(dict(n=N, max_log=4, n_games=1 << 62, queue_games=M * R), dict(st, reset_buf=q["reset_buf"]))
    native.im_motion_queue(dict(n=N, num_motions=M, queue_len=M * R, shape_dim=SHAPE),
                           dict(q, step=st["step"], games=st["games"], prev_dones=st["prev_dones"]))


@pytest.mark.parametrize("N", [1, 33, 1024, 8197])
@pytest.mark.parametrize("MR", ["N", "N+1", "3N+5", "3(N+2)"])
def test_queue_launch_is_the_restatement(N, MR):
    M, R = {"N": (N, 1), "N+1": (N + 1, 1), "3N+5": (3 * N + 5, 1), "3(N+2)": (N + 2, 3)}[MR]
    g = np.random.default_rng(N + M * R)
    q, st = queue_buffers(N, M, R, g)
    ora = Q.MotionQueue(N, M, R)
    rb = np.zeros(N, np.int64)
    for k in range(200):
        rb[g.random(N) < 0.3] = 1                          # envs finish; idle envs stay done
        q["reset_buf"].copy_(torch.from_numpy(rb))
        device_step(N, M, R, q, st)
        ora.bookkeeping(rb)
        mask = ora.assign(rb)
        torch.cuda.synchronize()
        got = {k: v.cpu().numpy() for k, v in q.items()}
        assert np.array_equal(got["mask"], mask), k
        assert np.array_equal(got["motion_ids"], ora.motion_ids) and np.array_equal(got["entry"], ora.entry), k
        assert np.array_equal(got["idle"].astype(bool), ora.idle) and int(got["cursor"][0]) == ora.cursor, k
        assert np.array_equal(got["game_env"], ora.game_env) and np.array_equal(got["game_start_step"], ora.game_start_step), k
        assert bool(st["games"][1]) == ora.stop and int(st["games"][0]) == ora.games, k
        assert np.array_equal(st["prev_dones"].cpu().numpy() != 0, ora.prev_done), k
        assert not got["env_flags"][mask, 0].any()
        assert np.array_equal(got["motion_bodies"][mask], got["lib_motion_bodies"][ora.motion_ids[mask]])
        rb[mask] = 0                                       # the masked reset clears the flags
        if ora.stop:
            break
    assert ora.stop and ora.games == M * R and (ora.game_env >= 0).all()


def test_replays_give_the_same_assignment():
    N, M, R = 1024, 700, 3
    g = np.random.default_rng(3)
    flags = [(g.random(N) < 0.2).astype(np.int64) for _ in range(12)]
    out = []
    for graphed in (False, True):
        q, st = queue_buffers(N, M, R, np.random.default_rng(1))
        rb = np.zeros(N, np.int64)
        gr = None
        for f in flags:
            rb |= f
            q["reset_buf"].copy_(torch.from_numpy(rb))
            if not graphed:
                device_step(N, M, R, q, st)
            elif gr is None:
                device_step(N, M, R, q, st)
                torch.cuda.synchronize()
                gr = torch.cuda.CUDAGraph()
                with torch.cuda.graph(gr):
                    device_step(N, M, R, q, st)
            else:
                gr.replay()
            rb[q["mask"].cpu().numpy()] = 0
        torch.cuda.synchronize()
        out.append({k: v.cpu().numpy().copy() for k, v in q.items()})
    for k in out[0]:
        assert np.array_equal(out[0][k], out[1][k]), k


# ---------------------------------------------------------------------------------------------------------- window and operand row
def lib(M=5, frames=45, seed=4):
    from vid2player3d_b200 import model_compiler, motion_lib
    return motion_lib.synthetic(model_compiler.load_compiled("smpl_mesh_humanoid_amass_v1"), num_motions=M, num_frames=frames, seed=seed)


def vis_task(N, flat, **over):
    from vid2player3d_b200.configs import SIM_PARAMS, im_cfg
    from vid2player3d_b200.tasks import HumanoidSMPLIMVis
    cfg = im_cfg(N, flat, **over)
    cfg["args"] = types.SimpleNamespace(test=True)
    torch.manual_seed(0)
    return HumanoidSMPLIMVis(cfg, SIM_PARAMS, 1, "cuda", 0, True)


@pytest.mark.parametrize("s", [0, 1, 31, 33, 70])
def test_restarted_window_is_the_id_list_window_started_s_frames_earlier(s):
    N = 12
    task = vis_task(N, lib())
    L, pad = task.context_length, task.context_padding
    task.reset()
    envs = torch.tensor([1, 4, 11], device=DEV)
    mask = torch.zeros(N, device=DEV, dtype=torch.bool)
    mask[envs] = True
    step = torch.full((1,), s, device=DEV, dtype=torch.long)
    keep = task.context_feat.clone()
    task.reset_masked(mask, step=step)
    P = L + 2 * pad
    feat, fmask = torch.zeros(len(envs), P, task.context_feat.shape[2], device=DEV), torch.zeros(len(envs), P, device=DEV, dtype=torch.bool)
    task._env.motion_context(None, task._reset_ref_motion_ids[envs].contiguous(), torch.zeros(len(envs), device=DEV), P, -pad - s % L, task.dt,
                             feat, fmask)
    torch.cuda.synchronize()
    assert torch.equal(task.context_feat[envs], feat) and torch.equal(task.context_mask[envs], fmask)
    other = ~mask
    assert torch.equal(task.context_feat[other], keep[other])


@pytest.mark.parametrize("s", [1, 5, 31])
def test_a_queued_games_first_operand_row_is_a_fresh_games_step_0_row(s):
    N = 8
    task = vis_task(N, lib())
    task.set_policy(network(5)[0], clip_actions=1.0)
    task.reset()
    task._im_step.zero_()
    p = task._im_policy
    task.policy_rows()
    x0, r0 = p.x[:N].clone(), task._im_resid.clone()      # x: the layer operand, rows padded past N
    for _ in range(s):                                      # the envs move on, the step counter reaches s
        task.test_step(1, graph=False)
    task._im_step.fill_(s)
    mask = torch.zeros(N, device=DEV, dtype=torch.bool)
    mask[[2, 5]] = True
    task.reset_buf[mask] = 1
    task.reset_masked(mask, step=task._im_step)            # restart envs 2 and 5 on their own motions
    task.policy_rows()
    torch.cuda.synchronize()
    assert torch.equal(p.x[:N][mask], x0[mask]) and torch.equal(task._im_resid[mask], r0[mask])
    assert not torch.equal(p.x[:N][~mask], x0[~mask])     # the other envs moved on


# ---------------------------------------------------------------------------------------------------------- run_test
def run(task, path, graph=True, max_steps=3000, record=None):
    task.cfg["env"]["b200_motion_stats_file"] = str(path)
    if record is not None:                                  # what the meters and the bookkeeping saw, before the queue's reset
        launches = task._queue_launches

        def rec():
            record.append(dict(rew=task.rew_buf.clone(), sub_rewards=task._sub_rewards.clone(), reset_buf=task.reset_buf.clone(),
                               terminate_buf=task._terminate_buf.clone(),
                               rigid_body_state=task._rigid_body_state.view(task.num_envs, -1, 13).clone(),
                               target_rb_pos=task._prev_target_rb_pos.clone()))
            launches()
        task._queue_launches = rec
    out = io.StringIO()
    with contextlib.redirect_stdout(out):
        res = task.run_test(network(5)[0], 1, max_steps, graph=graph, clip_actions=1.0)
    return res, dict(np.load(path)), out.getvalue().splitlines()


@pytest.mark.parametrize("R", [1, 2])
def test_run_test_plays_every_entry_once_as_the_restatement(tmp_path, R):
    N = 32
    M = 3 * N + 5
    task = vis_task(N, lib(M, 40, 6), b200_motion_queue=True, b200_motion_queue_repeats=R, b200_motion_stats=True)
    record = []
    res, got, lines = run(task, tmp_path / "q.npz", graph=False, record=record)
    assert got["games"].tolist() == [R] * M and got["unfinished"].size == 0
    assert (got["game_env"] >= 0).all() and got["game_env"].shape == (R, M) and res["games_played"] == M * R
    ora = Q.QueueRun(N, M, R)
    h = lambda x, k: x[k].double().cpu().numpy()  # noqa: E731
    for x in record:
        ora.step(h(x, "rew"), h(x, "sub_rewards"), h(x, "reset_buf"), h(x, "terminate_buf"), h(x, "rigid_body_state")[:, :24, :3],
                 h(x, "target_rb_pos"))
    counts, sums = ora.per_motion()
    assert np.array_equal(got["games"], counts[:, 0]) and np.array_equal(got["falls"], counts[:, 1])
    np.testing.assert_allclose(got["reward_sum"], sums[:, 0], rtol=1e-9)
    assert np.array_equal(got["steps"], sums[:, 1].astype(np.int64))
    np.testing.assert_allclose(got["sub_reward_sum"], sums[:, 2:6], rtol=1e-9)
    np.testing.assert_allclose(got["body_pos_err_sum"], sums[:, 6], rtol=1e-9)
    assert np.array_equal(got["game_env"].ravel(), ora.queue.game_env)
    assert np.array_equal(got["game_start_step"].ravel(), ora.queue.game_start_step)
    assert np.array_equal(got["env_motion_ids"], np.arange(N) % M)
    np.testing.assert_allclose(got["reward_sum"].sum(), res["sum_rewards"], rtol=1e-5)
    assert any(x.startswith(f"motions evaluated: {M} of {M}") for x in lines)


def test_run_test_graphed_is_eager_and_a_seed_repeats(tmp_path):
    N, M = 32, 3 * 32 + 5
    flat = lib(M, 40, 6)
    files = {}
    for name, graph in (("g1", True), ("g2", True), ("eager", False)):
        task = vis_task(N, flat, b200_motion_queue=True, b200_motion_queue_repeats=2, b200_motion_stats=True, b200_pose_metrics=True)
        _, files[name], _ = run(task, tmp_path / f"{name}.npz", graph=graph)
    assert files["g1"]["games"].tolist() == [2] * M and "success" in files["g1"]
    for other in ("g2", "eager"):
        assert files[other].keys() == files["g1"].keys()
        for k, v in files["g1"].items():
            assert v.dtype == files[other][k].dtype and v.tobytes() == files[other][k].tobytes(), (other, k)


def test_a_short_budget_leaves_entries_unfinished(tmp_path):
    N, M = 16, 3 * 16 + 5
    task = vis_task(N, lib(M, 40, 6), b200_motion_queue=True, b200_motion_stats=True)
    res, got, _ = run(task, tmp_path / "short.npz", max_steps=40)
    fin = got["games"] > 0
    assert 0 < res["games_played"] < M and fin.sum() == res["games_played"]
    assert np.array_equal(np.sort(got["unfinished"]), np.flatnonzero(~fin)) and (got["reward_sum"][~fin] == 0).all()
    assert (got["game_env"][0][fin] >= 0).all()


def test_without_the_key_nothing_of_the_queue_runs(tmp_path, monkeypatch):
    from vid2player3d_b200 import native
    calls = []
    monkeypatch.setattr(native, "im_motion_queue", lambda *a: calls.append(a))
    task = vis_task(32, lib(8, 40, 6), sample_first_motions=True, b200_motion_stats=True)
    masked = []
    task.reset_masked = lambda *a, **k: masked.append(a)
    res, got, _ = run(task, tmp_path / "plain.npz", max_steps=200)
    assert not calls and not masked and task._q is None
    assert set(got) == {"games", "falls", "reward_sum", "steps", "sub_reward_sum", "body_pos_err_sum", "env_motion_ids", "test_motion_file"}
    assert got["games"].sum() == res["games_played"] > 0
