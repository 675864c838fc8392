"""GPU checks of the per-row results of the fixed test set (cfg.env.b200_ball_stats): both forms of b200v2p_eval_ball_stats against the
float64 restatement oracle/ref_port_ball_stats.py on random states, served through both reset paths against the cursor walk, and
MVAEControllerVis.run_test end to end: per step against the restatement, summed against the per-env meters, graphed against eager,
the file before the recorder's SystemExit, and nothing at all without the key."""
import os

import numpy as np
import pytest
import torch

from helpers import SIM_PARAMS, v2p_cfg
from oracle import ref_port_ball_stats as B
from test_gpu_ball_test_set import ordered_pool, rounds
from test_gpu_v2p_launch import ISENT, SENT, SLACK, _dev, _pad, f32
from test_gpu_v2p_policy import networks, policy

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
FIX = 2.0 ** 24
COUNTS = B.COUNTS


def event_state(rng, n):
    return dict(reset_recovery=rng.random(n) < 0.6, has_contact=rng.random(n) < 0.5, swing_type_cycle=rng.integers(-1, 4, n),
                est_bounce_in=rng.random(n) < 0.6, est_bounce_pos=(rng.normal(size=(n, 3)) * 3).astype(f32),
                target_bounce_pos=(rng.normal(size=(n, 3)) * 3).astype(f32))


def cursors(rng, n, P, layout):
    if layout == "one row":      # every env on the same row: full contention
        return np.full(n, rng.integers(0, P), np.int64)
    if layout == "own row":      # env e plays row e (P >= n), else neighbouring lanes on neighbouring rows
        return ((np.arange(n) + 1) % P).astype(np.int64)
    return rng.integers(0, P, n).astype(np.int64)


def launch(s, cursor, buckets, P):
    """the slack rows past n carry set flags and a valid cursor: a launch past n would count them"""
    from vid2player3d_b200 import native_v2p as NV
    n = len(cursor)
    t = dict(pool_cursor=_dev(_pad(cursor, 0)), buckets=buckets[:P],
             **{k: _dev(_pad(v, {"b": True, "i": 1}.get(v.dtype.kind, SENT))) for k, v in s.items()})
    NV.eval_ball_stats(dict(n=n, pool_size=P), t)


@pytest.mark.parametrize("layout", ["random", "one row", "own row"])
@pytest.mark.parametrize("P", [1, 3, 7, 2048])
@pytest.mark.parametrize("n", [1, 33, 8197])
def test_launch_matches_restatement(n, P, layout):
    """three launches into the same buckets: counts exactly, the error column exactly the fixed-point sum of the float32 values and
    within 1e-6 of the float64 restatement; slack bucket rows past P untouched"""
    rng = np.random.default_rng(n * 7 + P)
    start = np.zeros((P + SLACK, 5), np.int64)
    start[:P, :4] = rng.integers(0, 50, (P, 4))             # the launch adds to what is there
    start[P:] = ISENT
    buckets = _dev(start)
    st, fx = B.BallStats(P), np.zeros(P, np.int64)
    for k in range(3):
        s, cursor = event_state(rng, n), cursors(rng, n, P, layout)
        s["reset_recovery"][0] = True
        launch(s, cursor, buckets, P)
        st.events(s, s["reset_recovery"], cursor)
        ev = np.flatnonzero(s["reset_recovery"] & s["est_bounce_in"])
        v = B.bounce_err(s["est_bounce_pos"][ev], s["target_bounce_pos"][ev]).astype(np.float64)
        np.add.at(fx, B.playing_row(cursor[ev], P), np.rint(v * FIX).astype(np.int64))
    torch.cuda.synchronize()
    got = buckets.cpu().numpy()
    assert (got[P:] == ISENT).all(), "a bucket past the pool was written"
    for c, k in enumerate(COUNTS):
        np.testing.assert_array_equal(got[:P, c] - start[:P, c], getattr(st, k), f"n={n} P={P} {layout}: {k}")
    np.testing.assert_array_equal(got[:P, 4], fx)
    np.testing.assert_allclose(got[:P, 4] / FIX, st.bounce_err_sum, rtol=1e-6, atol=0)
    assert st.recoveries.sum() >= 3


@pytest.mark.parametrize("layout", ["random", "one row", "own row"])
@pytest.mark.parametrize("P", [1, 3, 7, 2048])
@pytest.mark.parametrize("n", [1, 33, 8197])
def test_draws_form_matches_the_cursor_walk(n, P, layout):
    """rounds of draws (the restatement's generate moves the cursors of the reaction envs), each followed by the draws form on the
    moved cursors: served counts every drawn row exactly; slack rows past P untouched"""
    from vid2player3d_b200 import native_v2p as NV
    rng = np.random.default_rng(n * 11 + P)
    served = _dev(np.concatenate([np.zeros(P, np.int64), np.full(SLACK, ISENT, np.int64)]))
    cursor, want, pool = cursors(rng, n, P, layout), B.BallStats(P), np.zeros((P, 307), f32)
    for k in range(4):
        rea = rng.random(n) < 0.5
        rea[0] = True
        want.generate(pool, cursor, np.flatnonzero(rea))
        NV.eval_ball_stats(dict(n=n, pool_size=P), dict(pool_cursor=_dev(_pad(cursor, 0)), reset_reaction=_dev(_pad(rea, True)),
                                                        row_served=served[:P]))
    got = served.cpu().numpy()
    assert (got[P:] == ISENT).all(), "a row past the pool was counted"
    np.testing.assert_array_equal(got[:P], want.served, f"n={n} P={P} {layout}")


def test_launch_of_no_event_writes_nothing():
    s = event_state(np.random.default_rng(0), 100)
    s["reset_recovery"][:] = False
    buckets = _dev(np.full((7 + SLACK, 5), ISENT, np.int64))
    launch(s, np.zeros(100, np.int64), buckets, 7)
    assert (buckets.cpu().numpy() == ISENT).all()


# ------------------------------------------------------------------------------------------------ served through both reset paths
def controller(N, pool):
    from vid2player3d_b200.tasks import PhysicsMVAEController
    torch.manual_seed(4)
    cfg = v2p_cfg(N, use_random_ball_target=False, test_mode="multiple_cycle", ball_pool_test=pool)
    cfg["env"].update(is_train=False)
    env = PhysicsMVAEController(cfg, SIM_PARAMS, 1, "cuda", 0, True)
    env._physics_player.task._ball_row_served = torch.zeros(len(pool), device=DEV, dtype=torch.long)
    return env


@pytest.mark.parametrize("P", [1, 7])
def test_served_counts_every_draw_of_both_reset_paths(P):
    """the first reset (every env draws row 0), then rounds of the id-list reset (_reset_envs_idlist -> _reset_balls) on one
    controller and the mask-driven one (b200v2p_task_reset) on the other: served is the cursor walk's count of drawn rows"""
    N, pool = 130, ordered_pool(P)
    envs = [controller(N, pool), controller(N, pool)]
    want = B.BallStats(P)
    cursor = np.zeros(N, np.int64)
    want.generate(pool, cursor, np.arange(N))
    for env in envs:
        env.reset()
    for r, (hm, rea, rec) in enumerate(rounds(N, 3, 6)):
        want.generate(pool, cursor, rea.nonzero(as_tuple=False).flatten().cpu().numpy())
        for i, env in enumerate(envs):
            env._reset_reaction_buf.copy_(rea)
            env._reset_recovery_buf.copy_(rec)
            if i == 0:
                env._reset_envs_idlist(hm.nonzero(as_tuple=False).flatten())
            else:
                env._reset_envs_masked(hm)
        torch.cuda.synchronize()
        for i, env in enumerate(envs):
            t = env._physics_player.task
            np.testing.assert_array_equal(t._ball_pool_cursor.cpu().numpy(), cursor, f"round {r} env {i}: cursor")
            np.testing.assert_array_equal(t._ball_row_served.cpu().numpy(), want.served, f"round {r} env {i}: served")
    assert want.served.sum() > N


# ------------------------------------------------------------------------------------------------ run_test end to end
def vis(tmp_path, N=64, P=7, stats=True, name="balls.npz", seed=0, **env_over):
    from vid2player3d_b200.tasks import MVAEControllerVis
    pool = ordered_pool(P)
    np.save(tmp_path / "balls_test.npy", pool)
    cfg = v2p_cfg(N)
    cfg["env"].update(ball_traj_file_test=str(tmp_path / "balls_test.npy"), **env_over)
    if stats:
        cfg["env"].update(b200_ball_stats=True, b200_ball_stats_file=str(tmp_path / name))
    torch.manual_seed(seed)
    return MVAEControllerVis(cfg, SIM_PARAMS, 1, "cuda", 0, True)


def post_state(env):
    t = env._physics_player.task
    g = lambda x: x.cpu().numpy()  # noqa: E731
    return dict(has_contact=g(t._has_racket_ball_contact), swing_type_cycle=g(env._mvae_player._swing_type_cycle),
                est_bounce_in=g(env._est_bounce_in), est_bounce_pos=g(env._est_bounce_pos), target_bounce_pos=g(env._target_bounce_pos))


def test_run_test_matches_restatement_and_the_meters(tmp_path):
    """a graphed test run stepped by hand: after each step (the post launch's flags and values still in place) the restatement takes
    the recovery events at the rows one behind the cursors, and the draws at the cursor moves; at the end the buckets equal it, and
    their sums over the rows equal the per-env meters' sums"""
    N, P, steps = 64, 7, 400
    env = vis(tmp_path, N, P)
    task = env._physics_player.task
    env.run_test(policy(networks(1, seed=9), N, clip_obs=5.0, clip_actions=1.0), 0, graph=True)   # reset, render_vis(init), export
    want, draws = B.BallStats(P), np.zeros(N, np.int64)
    want.served[0] = N
    cursor = task._ball_pool_cursor.cpu().numpy()
    assert (cursor == 1).all()
    for _ in range(steps):
        env.test_step(True)
        new = task._ball_pool_cursor.cpu().numpy()
        moved = np.flatnonzero(new != cursor)              # at most one draw per env and step; with P = 7 a draw moves the cursor
        np.add.at(want.served, cursor[moved], 1)
        draws[moved] += 1
        cursor = new
        want.events(post_state(env), env._reset_recovery_buf.cpu().numpy(), cursor)
    assert env._test_graphs is not None and env._test_steps == steps
    path = env.export_ball_stats()
    z = np.load(path)
    for k in ("served",) + COUNTS:
        np.testing.assert_array_equal(z[k], getattr(want, k), k)
    np.testing.assert_allclose(z["bounce_err_sum"], want.bounce_err_sum, rtol=1e-6, atol=0)
    assert int(z["num_envs"]) == N and int(z["test_steps"]) == steps and str(z["ball_traj_file_test"]) == str(tmp_path / "balls_test.npy")
    cnt, msum = env._meter_count.cpu().numpy(), env._meter_sum.cpu().numpy().astype(np.float64)
    assert z["recoveries"].sum() == cnt[0].sum() > N
    for k, m in (("hits", 0), ("forehands", 1), ("bounce_in", 2)):
        assert z[k].sum() == msum[m].sum(), k
    assert z["bounce_in"].sum() == cnt[3].sum()
    np.testing.assert_allclose(z["bounce_err_sum"].sum(), msum[3].sum(), rtol=1e-5)
    assert z["served"].sum() == N + draws.sum() and (draws > 0).all()


def run_file(tmp_path, graph, name):
    N = 64
    env = vis(tmp_path, N, 5, name=name, seed=3)
    env.run_test(policy(networks(1, seed=9), N, clip_obs=5.0, clip_actions=1.0), 150, graph=graph)
    return np.load(tmp_path / name), env


def test_graphed_equals_eager_and_a_seed_repeats_the_file(tmp_path, capsys):
    a, ea = run_file(tmp_path, False, "eager.npz")
    b, eb = run_file(tmp_path, True, "graphed.npz")
    c, _ = run_file(tmp_path, True, "graphed_again.npz")
    assert ea._test_graphs is None and eb._test_graphs is not None
    assert sorted(a.files) == sorted(b.files) == sorted(c.files)
    for k in a.files:
        np.testing.assert_array_equal(a[k], b[k], k)
        np.testing.assert_array_equal(b[k], c[k], k)
        assert a[k].dtype == b[k].dtype, k
    assert a["recoveries"].sum() > 0 and int(a["test_steps"]) == 150
    lines = [ln for ln in capsys.readouterr().out.splitlines() if ln.startswith("balls served:")]
    assert len(lines) == 3 and len(set(lines)) == 1


def test_file_is_written_before_the_recorders_exit(tmp_path):
    """with record, _render_host raises SystemExit at num_rec_frames: the ball statistics are written first"""
    N = 32
    env = vis(tmp_path, N, 3, record=True, num_rec_frames=20, rec_fname=str(tmp_path / "episode.npz"))
    with pytest.raises(SystemExit):
        env.run_test(policy(networks(1, seed=9), N, clip_obs=5.0, clip_actions=1.0), 100, graph=True)
    z = np.load(tmp_path / "balls.npz")
    assert int(z["test_steps"]) == 19 and z["served"].sum() >= N
    np.testing.assert_array_equal(z["recoveries"], env._bstats["buckets"][:, 0].cpu().numpy())


def test_without_the_key_nothing_is_allocated_or_launched(tmp_path, monkeypatch):
    from vid2player3d_b200 import native_v2p

    def refuse(*a, **k):
        raise AssertionError("eval_ball_stats launched without b200_ball_stats")
    monkeypatch.setattr(native_v2p, "eval_ball_stats", refuse)
    monkeypatch.chdir(tmp_path)
    N = 32
    env = vis(tmp_path, N, 3, stats=False)
    env.run_test(policy(networks(1, seed=9), N, clip_obs=5.0, clip_actions=1.0), 40, graph=True)
    assert env._test_graphs is not None and env._bstats is None and env._physics_player.task._ball_row_served is None
    assert not os.path.exists(tmp_path / "out")
