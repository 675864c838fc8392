"""GPU checks of the fixed test set of incoming balls: b200v2p_task_reset with pool_cursor against the restatement
oracle/ref_port_test_set.py bit for bit, the same launch without a cursor against the random branch's restatement, the id-list reset
(_reset_envs_idlist) and the graphed mask-driven reset against the eager one, and MVAEControllerVis.run_test on a three-row test set."""
import numpy as np
import pytest
import torch

from helpers import SIM_PARAMS, v2p_cfg
from oracle import ref_port_test_set as T
from oracle import ref_port_v2p as V
from test_gpu_v2p_launch import ISENT, SENT, SLACK, _dev, _pad, compare, f32
from test_gpu_v2p_policy import networks, policy

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
MODES = {None: 0, "continuous": 1, "discrete": 2}


def random_state(rng, n, L, hist):
    return dict(ball_pos=np.stack([rng.uniform(-5, 5, n), rng.uniform(-12, 12, n), rng.uniform(0, 3, n)], -1).astype(f32),
                ball_vel=rng.normal(size=(n, 3)).astype(f32), bounce_pos=rng.normal(size=(n, 3)).astype(f32),
                ball_traj=rng.normal(size=(n, 100, 3)).astype(f32), est_bounce_pos=rng.normal(size=(n, 3)).astype(f32),
                est_bounce_time=rng.random(n).astype(f32), est_max_height=rng.random(n).astype(f32),
                target_bounce_pos=rng.normal(size=(n, 3)).astype(f32), ball_states=rng.normal(size=(n, 13)).astype(f32),
                rbs_ball=rng.normal(size=(n, 13)).astype(f32), has_bounce=rng.random(n) < 0.5, has_contact=rng.random(n) < 0.5,
                bounce_in=rng.random(n) < 0.5, est_bounce_in=rng.random(n) < 0.5, tar_time=rng.integers(0, 80, n),
                tar_time_total=rng.integers(60, 80, n), tar_action=rng.integers(0, 2, n), num_reset_reaction=rng.integers(0, 5, n),
                swing_type_cycle=rng.integers(-1, 4, n), reset_reaction=np.zeros(n, bool), reset_recovery=np.zeros(n, bool),
                ball_obs=rng.normal(size=(n, L, 3)).astype(f32) if hist else None)


class Launch:
    """one set of device buffers (SLACK sentinel rows past n) that successive b200v2p_task_reset launches update in place"""

    def __init__(self, s, pool, cursor):
        n = len(s["ball_pos"])
        self.n, self.P = n, len(pool)
        self.t = {k: _dev(_pad(v, {"b": True, "i": ISENT}.get(v.dtype.kind, SENT))) for k, v in s.items()
                  if v is not None and k not in ("rbs_ball",)}
        rbs = np.full((n + SLACK, 26, 13), SENT, f32)
        rbs[:n, 25] = s["rbs_ball"]
        self.t.update(rigid_body_state=_dev(rbs), pool=_dev(pool), ball_obs=self.t.get("ball_obs"))
        self.t["pool_cursor"] = _dev(_pad(cursor, ISENT)) if cursor is not None else None

    def __call__(self, rea, rec, draws, mode, L):
        from vid2player3d_b200 import native_v2p as NV
        self.t["reset_reaction"].copy_(_dev(_pad(rea, True)))   # the slack rows carry set flags: a launch past n would act on them
        self.t["reset_recovery"].copy_(_dev(_pad(rec, True)))
        t = dict(self.t, **{k: _dev(v) for k, v in draws.items()})
        NV.task_reset(dict(n=self.n, pool_size=self.P, ball_stride=13, bodies_per_env=26, reaction_nframes=70, target_mode=MODES[mode],
                           target_min=(-3, 9, 0), target_max=(3, 11, 0), obs_traj_len=L), t)

    def read(self):
        torch.cuda.synchronize()
        n = self.n
        got = {k: v.cpu().numpy() for k, v in self.t.items() if v is not None and k not in ("pool", "rigid_body_state")}
        rb = self.t["rigid_body_state"].cpu().numpy()
        assert (rb[:, :25] == SENT).all(), "a humanoid body row was written"
        got["rbs_ball"] = rb[:, 25]
        for k, v in got.items():
            if k not in ("reset_reaction", "reset_recovery"):
                fill = {"b": True, "i": ISENT}.get(v.dtype.kind, SENT)
                assert (v[n:] == fill).all(), f"n = {n}: {k} written past n"
            got[k] = v[:n]
        return got


SPEC_KEYS = ("ball_pos", "ball_vel", "bounce_pos", "ball_traj", "est_bounce_pos", "est_bounce_time", "est_max_height", "target_bounce_pos",
             "ball_states", "rbs_ball", "has_bounce", "has_contact", "bounce_in", "est_bounce_in", "tar_time", "tar_time_total", "tar_action",
             "num_reset_reaction", "swing_type_cycle", "ball_obs")


@pytest.mark.parametrize("n", [1, 33, 8197])
@pytest.mark.parametrize("P", [1, 3, 1000, 20000])
def test_task_reset_with_cursor_matches_restatement(n, P):
    """four rounds of random reaction / recovery masks on one set of buffers: ball state, rigid-body row, trajectory or history, flags
    and cursor bit for bit; envs whose ball is on the far side (y > 0) take their cursor's row all the same.  pool_rand holds another
    valid row, so a launch that read it would pick a wrong one.  The same launch without a cursor is the random branch's restatement."""
    rng = np.random.default_rng(n * 31 + P)
    mode, hist = ((None, False), ("discrete", False), ("continuous", True), (None, True))[(n + P) % 4]
    L = 10
    pool = rng.uniform(-20, 20, (P, 307)).astype(f32)
    pool[:, 6] = rng.uniform(-10, 10, P)
    s = random_state(rng, n, L, hist)
    cursor = rng.integers(0, P, n)
    cursor[: min(n, 3)] = P - 1                                 # wraps at the first reset
    seq, rnd = Launch(s, pool, cursor), Launch(s, pool, None)
    ref_seq, ref_rnd = s, s
    for rnd_i in range(4):
        rea, rec = rng.random(n) < 0.5, rng.random(n) < 0.4
        rea[: min(n, 2)] = True
        far = rea & (rng.random(n) < 0.5)
        far[0] = True
        ys = rng.uniform(0.5, 12, int(far.sum())).astype(f32)
        for st, dev in ((ref_seq, seq), (ref_rnd, rnd)):       # balls on the far side: the random branch remaps these
            st["ball_pos"] = st["ball_pos"].copy()
            st["ball_pos"][far, 1] = ys
            dev.t["ball_pos"][torch.from_numpy(np.flatnonzero(far)).to(DEV), 1] = _dev(ys)
        st_cursor = cursor
        draws = dict(pool_rand=(st_cursor + 1) % P if P > 1 else np.zeros(n, np.int64), side_rand=rng.integers(-1000, 1000, n),
                     frame_rand=rng.integers(-5, 5, n))
        seeds = rng.random(n if mode == "discrete" else 3).astype(f32)
        ref_seq, cursor = T.task_reset(dict(ref_seq, reset_reaction=rea, reset_recovery=rec),
                                       dict(pool=pool, reaction_nframes=70, target_mode=mode, target_min=(-3, 9, 0), target_max=(3, 11, 0)),
                                       dict(draws, target_seed=seeds), cursor)
        ref_rnd = V.task_reset(dict(ref_rnd, reset_reaction=rea, reset_recovery=rec),
                               dict(pool=pool, reaction_nframes=70, target_mode=mode, target_min=(-3, 9, 0), target_max=(3, 11, 0)),
                               dict(draws, target_seed=seeds))
        for dev in (seq, rnd):
            dev(rea, rec, dict(draws, target_seed=seeds), mode, L)
        got_seq, got_rnd = seq.read(), rnd.read()
        spec = {k: "exact" for k in SPEC_KEYS if ref_seq.get(k) is not None}
        fails = compare(ref_seq, got_seq, spec)
        assert not fails, f"n = {n} P = {P} round {rnd_i}: " + "; ".join(fails[:6])
        np.testing.assert_array_equal(got_seq["pool_cursor"], cursor, f"n = {n} P = {P} round {rnd_i}: cursor")
        rows = np.flatnonzero(rea)
        np.testing.assert_array_equal(got_seq["ball_states"][rows, :3], pool[st_cursor[rows], :3])
        fails = compare(ref_rnd, got_rnd, spec)
        assert not fails, f"n = {n} P = {P} round {rnd_i} without cursor: " + "; ".join(fails[:6])


# ------------------------------------------------------------------------------------------------ the controller's reset paths
def ordered_pool(P=3):
    """launches along -y with no x velocity from x = -3, 0, 3, ...: the launch x of a ball names its row"""
    from vid2player3d_b200 import ball as ball_data
    pos = np.stack([np.arange(P) * 3.0 - 3.0, np.full(P, 12.5), np.full(P, 1.2)], -1)
    vel = np.tile([0.0, -28.0, 5.0], (P, 1))
    spin = np.full(P, 7.0)
    traj = ball_data.integrate(pos, vel, spin, spin_scale=5.0)
    return np.concatenate([pos, vel, spin[:, None], traj.reshape(P, 300)], -1).astype(np.float32)


def controller(N, pool, **env_over):
    from vid2player3d_b200.tasks import PhysicsMVAEController
    torch.manual_seed(4)
    cfg = v2p_cfg(N, use_random_ball_target=False, test_mode="multiple_cycle", ball_pool_test=pool)
    cfg["env"].update(is_train=False, **env_over)
    env = PhysicsMVAEController(cfg, SIM_PARAMS, 1, "cuda", 0, True)
    env.reset()
    for _ in range(2):
        env.step(torch.zeros(N, env.num_actions, device=DEV))
    return env


def task_fields(env):
    """what a reset does with no random draw: the ball, its flags and cursor, the reaction bookkeeping"""
    t = env._physics_player.task
    rbs = t._rigid_body_state.view(env.num_envs, 26, 13)
    return dict(cursor=t._ball_pool_cursor, ball=t._ball_root_states, rbs_ball=rbs[:, 25], ball_pos=t._ball_pos, ball_vel=t._ball_vel,
                bounce_pos=t._bounce_pos, has_bounce=t._has_bounce, contact=t._has_racket_ball_contact, traj=env._ball_traj,
                tar_time=env._tar_time, tar_action=env._tar_action, nrr=env._num_reset_reaction, bounce_in=env._bounce_in,
                est_bounce_in=env._est_bounce_in, cycle=env._mvae_player._swing_type_cycle, target=env._target_bounce_pos,
                progress=env.progress_buf, num_reset=env._num_reset)


def rounds(N, seed, k):
    g = np.random.default_rng(seed)
    for r in range(k):
        hm = g.random(N) < 0.15
        rea, rec = g.random(N) < 0.5, g.random(N) < 0.3
        rea[r % N] = True
        yield (torch.from_numpy(x).to(DEV) for x in (hm, rea, rec))


def test_idlist_reset_matches_masked_reset():
    """_reset_envs_idlist (the reference-shaped specification) and _reset_envs_masked take the same rows from the same cursors, over
    rounds that reset humanoids too: a humanoid reset leaves the cursor alone"""
    N, pool = 130, ordered_pool(7)
    envs = [controller(N, pool), controller(N, pool)]
    for a, b in zip(task_fields(envs[0]).values(), task_fields(envs[1]).values()):
        assert torch.equal(a, b)
    for r, (hm, rea, rec) in enumerate(rounds(N, 3, 5)):
        before = envs[0]._physics_player.task._ball_pool_cursor.clone()
        for i, env in enumerate(envs):
            env._reset_reaction_buf.copy_(rea)
            env._reset_recovery_buf.copy_(rec)
            if i == 0:
                env._reset_envs_idlist(hm.nonzero(as_tuple=False).flatten())
            else:
                env._reset_envs_masked(hm)
        torch.cuda.synchronize()
        fa, fb = task_fields(envs[0]), task_fields(envs[1])
        for k in fa:
            assert torch.equal(fa[k], fb[k]), f"round {r}: {k}"
        assert torch.equal(fa["cursor"], torch.where(rea, (before + 1) % len(pool), before)), f"round {r}"
        assert torch.equal(fa["ball"][rea, :3], torch.from_numpy(pool).to(DEV)[before[rea], :3]), f"round {r}"


def test_graphed_reset_matches_eager_reset():
    """the mask-driven reset captured once and replayed against the same reset run eagerly, round after round: the replays move the
    cursor with no host work"""
    N, pool = 257, ordered_pool(3)
    eager, graphed = controller(N, pool), controller(N, pool)
    gm = torch.zeros(N, dtype=torch.bool, device=DEV)
    for env in (eager, graphed):                     # one eager pass with every flag clear: the launches' one-time set-up
        env._reset_reaction_buf.zero_()
        env._reset_recovery_buf.zero_()
        env._reset_envs_masked(gm)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        graphed._reset_envs_masked(gm)
    for r, (hm, rea, rec) in enumerate(rounds(N, 8, 6)):
        for env in (eager, graphed):
            env._reset_reaction_buf.copy_(rea)
            env._reset_recovery_buf.copy_(rec)
        gm.copy_(hm)
        eager._reset_envs_masked(hm)
        g.replay()
        torch.cuda.synchronize()
        fa, fb = task_fields(eager), task_fields(graphed)
        for k in fa:
            assert torch.equal(fa[k], fb[k]), f"replay {r}: {k}"
    assert int(task_fields(graphed)["nrr"].max()) >= 1


# ------------------------------------------------------------------------------------------------ end to end
def test_run_test_walks_the_test_set_in_order(tmp_path):
    """MVAEControllerVis.run_test, graphed, with env.ball_traj_file_test naming a three-row pool: for every env the k-th reaction reset
    since its start launches row k mod 3, read from the launch x after the step and num_reset_reaction; the cursor is
    num_reset_reaction mod 3"""
    from vid2player3d_b200.tasks import MVAEControllerVis
    N, P, steps = 64, 3, 720
    pool = ordered_pool(P)
    np.save(tmp_path / "balls_test.npy", pool)
    cfg = v2p_cfg(N)
    cfg["env"].update(ball_traj_file_test=str(tmp_path / "balls_test.npy"), episodeLength=100000)
    torch.manual_seed(0)
    env = MVAEControllerVis(cfg, SIM_PARAMS, 1, "cuda", 0, True)
    assert env.cfg_v2p["test_mode"] == "multiple_cycle"
    task = env._physics_player.task
    assert task._ball_pool_cursor is not None and torch.equal(task._ball_pool.cpu(), torch.from_numpy(pool))
    env.run_test(policy(networks(1, seed=9), N, clip_obs=5.0, clip_actions=1.0), 1, graph=True)
    assert env._test_graphs is not None
    launch_x = pool[:, 0]
    read = lambda: (env._num_reset_reaction.cpu().numpy(), env._num_reset.cpu().numpy(), task._ball_pos[:, 0].cpu().numpy())  # noqa: E731
    nrr, nres0, x = read()
    first = nrr == 1
    assert first.all() and (np.abs(x - launch_x[0]) < 0.25).all()
    checked = 0
    for _ in range(steps):
        prev = nrr
        env.test_step(True)
        nrr, nres, x = read()
        keep = nres == nres0                           # no humanoid reset since the start: num_reset_reaction counts every ball
        new = keep & (nrr == prev + 1)
        assert (keep & (nrr != prev) & ~new).sum() == 0
        row = (nrr[new] - 1) % P
        assert (np.abs(x[new] - launch_x[row]) < 0.25).all(), (np.flatnonzero(new), x[new], row)
        checked += int(new.sum())
    keep = nres == nres0
    cursor = task._ball_pool_cursor.cpu().numpy()
    np.testing.assert_array_equal(cursor[keep], nrr[keep] % P)
    assert keep.mean() > 0.5 and checked > N and nrr[keep].max() >= P + 1, (keep.mean(), checked, nrr.max())
