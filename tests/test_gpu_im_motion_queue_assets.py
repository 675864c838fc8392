"""GPU checks of the motion queue with a body per motion (cfg.env.b200_motion_queue with motion_assets):

1. the queue launch with motion_asset / env_asset against the restatement (tests/test_im_motion_queue_assets.py: AssetQueue) at
   N = 1, 33, 1024, 8197, with every other output bitwise that of the launch without them, and graph replays alike;
2. b200env_set_env_assets on a handle fixed to the mixed plan: envs moved at random among S = 2, 64, N bodies step bit for bit like
   single-asset handles of their new bodies; a bad index keeps the env's body and sets the error word; the refusals;
3. a game the queue restarts at step counter s on another body steps bit for bit like the same motion started at step 0 in a task
   created with that body;
4. run_test: every entry played once per round, the per-motion meters against the restatement, every env on its motion's body at
   every step, graphed against eager and a seed against itself, bit for bit; a bad asset index raises ValueError at the host check;
5. without motion_assets the queue's step launches one kernel less and never calls set_env_assets."""
import ctypes as C
import types

import numpy as np
import pytest
import torch

import test_gpu_assets as TA
import test_gpu_im_motion_queue as GQ
from oracle import ref_port_motion_queue as Q
from test_gpu_assets_mixed import _compare, _variants
from test_gpu_launch import _pool
from test_im_motion_queue_assets import AssetQueue

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
AMASS = TA.AMASS


# ---------------------------------------------------------------------------------------------------------- 1. the queue launch
def asset_buffers(N, M, g, S=5):
    motion_asset = torch.from_numpy(g.integers(0, S, M).astype(np.int32)).to(DEV)
    return motion_asset, motion_asset[torch.arange(N, device=DEV) % M].contiguous()


@pytest.mark.parametrize("N", [1, 33, 1024, 8197])
@pytest.mark.parametrize("MR", ["N", "N+1", "3N+5", "3(N+2)"])
def test_queue_launch_writes_the_restatements_assets_and_nothing_else_changes(N, MR):
    M, R = {"N": (N, 1), "N+1": (N + 1, 1), "3N+5": (3 * N + 5, 1), "3(N+2)": (N + 2, 3)}[MR]
    g = np.random.default_rng(N + M * R)
    plain, st_plain = GQ.queue_buffers(N, M, R, np.random.default_rng(7))
    q, st = GQ.queue_buffers(N, M, R, np.random.default_rng(7))
    q["motion_asset"], q["env_asset"] = asset_buffers(N, M, g)
    ora = AssetQueue(N, M, R, q["motion_asset"].cpu().numpy())
    rb = np.zeros(N, np.int64)
    for k in range(200):
        rb[g.random(N) < 0.3] = 1
        for b in (plain, q):
            b["reset_buf"].copy_(torch.from_numpy(rb))
        GQ.device_step(N, M, R, plain, st_plain)
        GQ.device_step(N, M, R, q, st)
        ora.bookkeeping(rb)
        mask = ora.assign(rb)
        torch.cuda.synchronize()
        assert np.array_equal(q["env_asset"].cpu().numpy(), ora.env_asset), k
        for name, v in plain.items():
            assert v.cpu().numpy().tobytes() == q[name].cpu().numpy().tobytes(), (k, name)
        for name, v in st_plain.items():
            assert v.cpu().numpy().tobytes() == st[name].cpu().numpy().tobytes(), (k, name)
        assert np.array_equal(q["mask"].cpu().numpy(), mask), k
        rb[mask] = 0
        if ora.stop:
            break
    assert ora.stop


def test_replays_give_the_same_assets():
    N, M, R = 1024, 700, 3
    g = np.random.default_rng(3)
    flags = [(g.random(N) < 0.2).astype(np.int64) for _ in range(12)]
    out = []
    for graphed in (False, True):
        q, st = GQ.queue_buffers(N, M, R, np.random.default_rng(1))
        q["motion_asset"], q["env_asset"] = asset_buffers(N, M, np.random.default_rng(2), S=64)
        rb = np.zeros(N, np.int64)
        gr = None
        for f in flags:
            rb |= f
            q["reset_buf"].copy_(torch.from_numpy(rb))
            if not graphed or gr is None:
                GQ.device_step(N, M, R, q, st)
                if graphed:
                    torch.cuda.synchronize()
                    gr = torch.cuda.CUDAGraph()
                    with torch.cuda.graph(gr):
                        GQ.device_step(N, M, R, q, st)
            else:
                gr.replay()
            rb[q["mask"].cpu().numpy()] = 0
        torch.cuda.synchronize()
        out.append({k: v.cpu().numpy().copy() for k, v in q.items()})
    for k in out[0]:
        assert np.array_equal(out[0][k], out[1][k]), k


# ---------------------------------------------------------------------------------------------------------- 2. set_env_assets
def _dynamic(monkeypatch, assets, ea0, plan):
    """a handle of the assets with env e on ea0[e], created under plan (None = the rule), then fixed to the mixed plan"""
    if plan is None:
        monkeypatch.delenv("B200ENV_ASSET_PLAN", raising=False)
    else:
        monkeypatch.setenv("B200ENV_ASSET_PLAN", plan)
    t = TA._multi(AMASS, assets, ea0)
    monkeypatch.delenv("B200ENV_ASSET_PLAN", raising=False)
    t._env.fix_mixed_plan()
    assert t._env.asset_plan_mixed
    return t


@pytest.mark.parametrize("S,n,plan", [(2, 70, "grouped"), (64, 96, None), ("N", 40, "mixed")])
def test_reassigned_envs_step_like_single_asset_handles_of_their_new_bodies(monkeypatch, S, n, plan):
    S = n if S == "N" else S
    assets = _variants(S)
    rng = np.random.default_rng(S * 31 + n)
    ea0 = np.arange(n) % S
    ea1 = rng.integers(0, S, n)
    assert (ea1 != ea0).sum() > n // 3
    t = _dynamic(monkeypatch, assets, ea0, plan)
    err = torch.zeros(1, device=DEV, dtype=torch.int32)
    t._env.set_env_assets(torch.from_numpy(ea1.astype(np.int32)).to(DEV), err)
    pool = _pool("humanoid")
    envs = np.arange(n) % len(pool["kind"])
    got = TA._run(t, pool, envs)
    assert int(err) == 0
    del t
    for a in np.unique(ea1):
        mine = np.flatnonzero(ea1 == a)                      # the motions stay those of the creation (motion m = asset ea0)
        ref = TA._run(TA._single(AMASS, assets, a, ea0[mine]), pool, envs[mine])
        _compare(got, ref, mine, f"S = {S}, N = {n}, new asset {a}")


def test_a_bad_index_keeps_the_body_and_sets_the_error_word(monkeypatch):
    n, S = 40, 3
    assets = [TA._model(AMASS), TA.scaled(TA._model(AMASS), 0.9), TA.scaled(TA._model(AMASS), 1.1)]   # distinct: the task merges equal ones
    ea0 = np.arange(n) % S
    ea1 = (ea0 + 1) % S
    ea1[17] = S                                             # out of range: env 17 keeps asset ea0[17]
    t = _dynamic(monkeypatch, assets, ea0, None)
    err = torch.zeros(1, device=DEV, dtype=torch.int32)
    t._env.set_env_assets(torch.from_numpy(ea1.astype(np.int32)).to(DEV), err)
    torch.cuda.synchronize()
    assert int(err) == 18
    pool = _pool("humanoid")
    envs = np.arange(n) % len(pool["kind"])
    got = TA._run(t, pool, envs)
    del t
    kept = ea1.copy()
    kept[17] = ea0[17]
    for a in range(S):
        mine = np.flatnonzero(kept == a)
        _compare(got, TA._run(TA._single(AMASS, assets, a, ea0[mine]), pool, envs[mine]), mine, f"asset {a}")
    ea1[3] = -1                                             # the word keeps the first error until the caller clears it
    t = _dynamic(monkeypatch, assets, ea0, None)
    t._env.set_env_assets(torch.from_numpy(ea1.astype(np.int32)).to(DEV), err)
    torch.cuda.synchronize()
    assert int(err) == 18


def test_refusals(monkeypatch):
    from vid2player3d_b200 import abi, native
    L = native.lib()
    one = TA._single(AMASS, _variants(2), 0, [0, 1])
    assert L.b200env_fix_mixed_plan(one._env._h) == -2 and "one asset" in L.b200env_last_error().decode()
    monkeypatch.setenv("B200ENV_ASSET_PLAN", "mixed")
    mixed = TA._multi(AMASS, _variants(2), [0, 1, 1, 0])
    monkeypatch.delenv("B200ENV_ASSET_PLAN")
    ea, err = torch.zeros(4, device=DEV, dtype=torch.int32), torch.zeros(1, device=DEV, dtype=torch.int32)
    for t in (one, mixed):                                  # a one-asset handle, and a mixed handle that was not fixed
        d = native.fill(abi.SetEnvAssets, dict(n=t.num_envs), dict(env_asset=ea[:t.num_envs], error=err))
        assert L.b200env_set_env_assets(t._env._h, C.byref(d), None) == -2
        assert "not fixed to the mixed plan" in L.b200env_last_error().decode()
    mixed._env.fix_mixed_plan()
    mixed._env.fix_mixed_plan()                             # twice is allowed
    d = native.fill(abi.SetEnvAssets, dict(n=3), dict(env_asset=ea, error=err))
    assert L.b200env_set_env_assets(mixed._env._h, C.byref(d), None) == -2 and "env count" in L.b200env_last_error().decode()
    with pytest.raises(RuntimeError, match="not fixed to the mixed plan"):
        one._env.set_env_assets(ea[:2], err)


# ---------------------------------------------------------------------------------------------------------- 3. a restarted game
def bodies():
    base = TA._model(AMASS)
    return [TA.scaled(base, 0.9), TA.scaled(base, 1.1), TA.scaled(base, 0.97)]


def asset_task(N, flat, motion_asset, **over):
    from vid2player3d_b200.configs import SIM_PARAMS, im_cfg
    from vid2player3d_b200.tasks import HumanoidSMPLIMVis
    b = bodies()
    entries = [b[a] for a in motion_asset]
    cfg = im_cfg(N, flat, **dict(dict(b200_motion_queue=True, motion_assets=entries, test_motion_assets=entries), **over))
    cfg["args"] = types.SimpleNamespace(test=True)
    torch.manual_seed(0)
    return HumanoidSMPLIMVis(cfg, SIM_PARAMS, 1, "cuda", 0, True)


def env_rows(t, e):
    n = t.num_envs
    return dict(rb=t._rigid_body_state.view(n, -1, 13)[e].cpu().numpy(), dof=t._dof_state.view(n, -1, 2)[e].cpu().numpy(),
                root=t._root_states[e].cpu().numpy())


@pytest.mark.parametrize("s", [1, 5, 31])
def test_a_restarted_game_steps_on_its_new_body(s):
    from helpers import SIM_PARAMS, im_cfg
    from test_gpu_im_policy import network
    N, M, K = 4, 8, 10
    flat = GQ.lib(M, 60, 5)
    motion_asset = [0, 0, 0, 0, 1, 1, 1, 1]                   # env 0 moves from motion 0 (body 0) to entry 4 (motion 4, body 1)
    task = asset_task(N, flat, motion_asset)
    task.set_policy(network(5)[0], clip_actions=1.0)
    task._start_queue()
    task.reset()
    for k in ("cr", "steps", "prev_dones", "step"):
        task._stats[k].zero_()
    g = torch.Generator(device=DEV).manual_seed(s)
    act = (torch.rand(N, task.num_actions, device=DEV, generator=g) * 2 - 1) * 0.3
    for _ in range(s):
        task.step(act)
    from vid2player3d_b200 import native
    task.reset_buf.zero_()
    task.reset_buf[0] = 1
    task._im_step.fill_(s - 1)                              # the bookkeeping below advances it to s, the restart's first step
    native.play_stats(dict(n=N, max_log=task._stats_cap, n_games=1 << 62, queue_games=M), dict(task._stats, rew=task.rew_buf,
                                                                                                reset_buf=task.reset_buf))
    task._queue_launches()
    torch.cuda.synchronize()
    assert int(task._reset_ref_motion_ids[0]) == 4 and task._q["env_asset"].tolist() == [1, 0, 0, 0]
    assert int(task._q["game_start_step"][4]) == s
    for _ in range(K):
        task.step(act)
    got = env_rows(task, 0)
    cfg = im_cfg(1, flat, stateInit="Start")
    cfg["env"]["test_motion_ids"], cfg["env"]["test_model"] = [4], bodies()[1]
    torch.manual_seed(0)
    ref = TA._task_class()(cfg, SIM_PARAMS, 1, "cuda", 0, True)
    ref.reset()
    for _ in range(K):
        ref.step(act[:1].contiguous())
    want = env_rows(ref, 0)
    for k in want:
        assert got[k].tobytes() == want[k].tobytes(), k


# ---------------------------------------------------------------------------------------------------------- 4. run_test
def run_assets(task, path, graph=True, record=None):
    if record is not None:                                  # the queue's assignment after each step, next to the meters' inputs
        launches = task._queue_launches

        def after():
            launches()
            record[-1].update(env_asset=task._q["env_asset"].cpu().numpy(), motion_ids=task._reset_ref_motion_ids.cpu().numpy())
        task._queue_launches = after
    return GQ.run(task, path, graph=graph, record=record)


@pytest.mark.parametrize("R", [1, 2])
def test_run_test_plays_every_entry_once_on_its_own_body(tmp_path, R):
    N = 32
    M = 3 * N + 5
    motion_asset = np.random.default_rng(R).integers(0, 3, M)
    task = asset_task(N, GQ.lib(M, 40, 6), motion_asset, b200_motion_queue_repeats=R, b200_motion_stats=True)
    assert task._env.asset_plan_mixed
    pairs = set(zip(motion_asset.tolist(), task._motion_asset.tolist()))   # the handle numbers the bodies in order of first use
    assert len(pairs) == 3 and len({p[1] for p in pairs}) == 3
    record = []
    res, got, lines = run_assets(task, tmp_path / "q.npz", graph=False, record=record)
    assert got["games"].tolist() == [R] * M and got["unfinished"].size == 0 and res["games_played"] == M * R
    ora = Q.QueueRun(N, M, R)
    h = lambda x, k: x[k].double().cpu().numpy()  # noqa: E731
    changed = 0
    for x in record:
        ora.step(h(x, "rew"), h(x, "sub_rewards"), h(x, "reset_buf"), h(x, "terminate_buf"), h(x, "rigid_body_state")[:, :24, :3],
                 h(x, "target_rb_pos"))
        assert np.array_equal(x["env_asset"], task._motion_asset[x["motion_ids"]])
        changed += int((x["env_asset"] != task._motion_asset[np.arange(N) % M]).sum())
    assert changed > 0
    counts, sums = ora.per_motion()
    assert np.array_equal(got["games"], counts[:, 0]) and np.array_equal(got["falls"], counts[:, 1])
    np.testing.assert_allclose(got["reward_sum"], sums[:, 0], rtol=1e-9)
    assert np.array_equal(got["steps"], sums[:, 1].astype(np.int64))
    np.testing.assert_allclose(got["sub_reward_sum"], sums[:, 2:6], rtol=1e-9)
    np.testing.assert_allclose(got["body_pos_err_sum"], sums[:, 6], rtol=1e-9)
    assert np.array_equal(got["game_env"].ravel(), ora.queue.game_env)
    assert np.array_equal(got["game_start_step"].ravel(), ora.queue.game_start_step)


def test_run_test_graphed_is_eager_and_a_seed_repeats(tmp_path):
    N, M = 32, 3 * 32 + 5
    flat = GQ.lib(M, 40, 6)
    motion_asset = np.arange(M) % 3
    files = {}
    for name, graph in (("g1", True), ("g2", True), ("eager", False)):
        task = asset_task(N, flat, motion_asset, b200_motion_queue_repeats=2, b200_motion_stats=True)
        _, files[name], _ = run_assets(task, tmp_path / f"{name}.npz", graph=graph)
    assert files["g1"]["games"].tolist() == [2] * M
    for other in ("g2", "eager"):
        assert files[other].keys() == files["g1"].keys()
        for k, v in files["g1"].items():
            assert v.dtype == files[other][k].dtype and v.tobytes() == files[other][k].tobytes(), (other, k)


def test_a_bad_asset_index_raises_at_the_host_check(tmp_path):
    N, M = 8, 20
    task = asset_task(N, GQ.lib(M, 40, 6), np.arange(M) % 2, b200_motion_stats=True)
    real = task._queue_assets

    def bad():
        q = real()
        q["motion_asset"][N + 1] = 7                        # entry N + 1 names an asset the handle does not have
        return q
    task._queue_assets = bad
    with pytest.raises(ValueError, match=r"env \d+ was given an asset index outside the handle's 2 assets"):
        GQ.run(task, tmp_path / "bad.npz", graph=True)


# ---------------------------------------------------------------------------------------------------------- 5. without motion_assets
def test_without_motion_assets_nothing_new_runs(monkeypatch):
    from test_gpu_im_policy import network
    from vid2player3d_b200 import native
    calls = []
    real = native.Env.set_env_assets
    monkeypatch.setattr(native.Env, "set_env_assets", lambda self, *a: calls.append(a) or real(self, *a))
    N, M = 32, 40
    per_step = {}
    for name in ("plain", "assets"):
        task = (GQ.vis_task(N, GQ.lib(M, 40, 6), b200_motion_queue=True) if name == "plain"
                else asset_task(N, GQ.lib(M, 40, 6), np.arange(M) % 2))
        task.set_policy(network(5)[0], clip_actions=1.0)
        task._start_queue()
        task.reset()
        c0 = task._env.launch_count
        task._test_launches()
        per_step[name] = task._env.launch_count - c0
        if name == "plain":
            assert not calls and "env_asset" not in task._q
    assert per_step["assets"] == per_step["plain"] + 1 and len(calls) == 2    # _start_queue and the step
