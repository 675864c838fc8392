"""GPU checks of the rally results of the dual test run (cfg.env.b200_rally_stats): b200v2p_eval_rally_stats against the integer
restatement oracle/ref_port_rally_stats.py on random sequences and on the scripted rallies of tests/test_rally_stats.py, its refusals,
and MVAEControllerVisDual.run_test end to end: the file against the restatement fed with the run's own per-step flags, graphed against
eager, a seed against itself, the rallies against the pairs whose reset_buf rose, and nothing at all without the key."""
import os

import numpy as np
import pytest
import torch

from helpers import SIM_PARAMS, v2p_dual_cfg
from oracle import ref_port_rally_stats as RS
from test_gpu_v2p_launch import ISENT, SLACK, _dev, _pad
from test_gpu_v2p_policy import networks, policy
from test_rally_stats import SCRIPTS, check_invariants, check_script_counts, random_run, run_scripts

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
STATE = ("pair_open", "pair_hits")
ACC = ("totals", "ends", "player", "shots_hist")


class Device:
    """the pair state and accumulators on the device, each with SLACK sentinel rows behind it, and one launch per step; the input rows
    past n meet the ball with contact at progress 1, so a launch that read past n would count them"""

    def __init__(self, n):
        self.n, K = n, n // 2
        self.full = dict(pair_open=_dev(np.ones(K + SLACK, bool)), pair_hits=_dev(np.full((K + SLACK, 2), ISENT, np.int64)),
                         totals=_dev(np.full(3 + SLACK, ISENT, np.int64)), ends=_dev(np.full((2 + SLACK, 3), ISENT, np.int64)),
                         player=_dev(np.full((2 + SLACK, 3), ISENT, np.int64)), shots_hist=_dev(np.full(RS.HIST + SLACK, ISENT, np.int64)))
        size = dict(pair_open=K, pair_hits=K, totals=3, ends=2, player=2, shots_hist=RS.HIST)
        self.t = {k: v[:size[k]] for k, v in self.full.items()}
        self.t["pair_open"].zero_()
        self.t["pair_hits"].zero_()
        for k in ACC:
            self.t[k].zero_()

    def launch(self, s):
        from vid2player3d_b200 import native_v2p
        fill = dict(tar_action=1, has_contact=True, has_bounce=False, bounce_in=False, swing_type_cycle=1, progress_buf=1)
        inp = {k: _dev(_pad(np.asarray(s[k]), fill.get(k, np.float32(0)))) for k in RS.INPUTS}
        native_v2p.eval_rally_stats(dict(n=self.n), dict(inp, **self.t))

    def arrays(self):
        torch.cuda.synchronize()
        return {k: v.cpu().numpy() for k, v in self.t.items()}

    def slack_untouched(self):
        full = {k: v.cpu().numpy() for k, v in self.full.items()}
        K = self.n // 2
        return (full["pair_open"][K:].all() and (full["pair_hits"][K:] == ISENT).all() and (full["totals"][3:] == ISENT).all()
                and (full["ends"][2:] == ISENT).all() and (full["player"][2:] == ISENT).all() and (full["shots_hist"][RS.HIST:] == ISENT).all())


def assert_same(got, want, what=""):
    for k in STATE + ACC:
        np.testing.assert_array_equal(got[k], want[k], f"{what}{k}")


@pytest.mark.parametrize("n", [2, 34, 8194])
def test_launch_matches_restatement_on_random_sequences(n):
    """220 steps of random flags with resets after endings: pairs across warp and block edges and a ragged tail, counts exact at every
    20th step and at the end"""
    rng = np.random.default_rng(n)
    dev, want, k = Device(n), RS.RallyStats(n), [0]

    def step(s):
        dev.launch(s)
        end = want.step(s)
        k[0] += 1
        if k[0] % 20 == 0:
            assert_same(dev.arrays(), want.arrays(), f"n={n} step {k[0]}: ")
        return end
    random_run(rng, n, 220, step)
    got = dev.arrays()
    assert_same(got, want.arrays(), f"n={n}: ")
    check_invariants(got)
    assert dev.slack_untouched(), "a launch wrote past its pairs"
    assert got["totals"][0] > n // 2 and (got["ends"] > 0).all() and got["player"][:, 2].sum() > 0


def test_scripted_rallies_on_the_device():
    names = list(SCRIPTS)
    dev = Device(2 * len(names))
    run_scripts(names, dev.launch)
    check_script_counts(names, dev.arrays())
    assert dev.slack_untouched()


def test_refusals_with_the_reason():
    from vid2player3d_b200 import native_v2p
    n = 6
    dev = Device(n)
    s = {k: _dev(np.asarray(v)) for k, v in random_inputs(n).items()}
    with pytest.raises(RuntimeError, match="b200v2p_eval_rally_stats: n must be even"):
        native_v2p.eval_rally_stats(dict(n=5), dict(s, **dev.t))
    with pytest.raises(ValueError, match=r"V2PRallyStats\.shots_hist: None"):
        native_v2p.eval_rally_stats(dict(n=n), dict(s, **dict(dev.t, shots_hist=None)))
    got = dev.arrays()
    assert not got["pair_open"].any() and all((got[k] == 0).all() for k in ACC)


def random_inputs(n):
    out = {}
    random_run(np.random.default_rng(0), n, 1, lambda s: out.update(s) or np.zeros(n // 2, bool))
    return out


# ------------------------------------------------------------------------------------------------ run_test end to end
def vis(tmp_path, N=64, stats=True, name="rallies.npz", seed=0, **env_over):
    from vid2player3d_b200.tasks import MVAEControllerVisDual
    cfg = v2p_dual_cfg(N)
    cfg["env"]["physics"]["assetFileName"] = "smpl_mesh_humanoid_federer.xml"       # one asset; the players still differ
    cfg["env"].update(env_over)
    if stats:
        cfg["env"].update(b200_rally_stats=True, b200_rally_stats_file=str(tmp_path / name))
    torch.manual_seed(seed)
    np.random.seed(seed)
    return MVAEControllerVisDual(cfg, SIM_PARAMS, 1, "cuda", 0, True)


def flags(env):
    t = env._physics_player.task
    g = lambda x: x.cpu().numpy()  # noqa: E731
    return dict(tar_action=g(env._tar_action), has_contact=g(t._has_racket_ball_contact), has_bounce=g(t._has_bounce),
                bounce_in=g(env._bounce_in), ball_pos=g(t._ball_pos), root_pos=g(t._root_pos),
                swing_type_cycle=g(env._mvae_player._swing_type_cycle), progress_buf=g(env.progress_buf))


def expected_file(st, env, steps):
    a = st.arrays()
    return dict(rallies=a["totals"][0], shots_sum=a["totals"][1], frames_sum=a["totals"][2], shots_hist=a["shots_hist"], ends=a["ends"],
                end_causes=np.array(RS.CAUSES), faced=a["player"][:, 0], hits=a["player"][:, 1], forehands=a["player"][:, 2],
                open_rallies=np.int64(a["pair_open"].sum()), open_hits=a["pair_hits"][a["pair_open"]], players=np.array(["federer", "djokovic"]),
                num_envs=np.int64(env.num_envs), test_steps=np.int64(steps))


def test_eager_run_matches_restatement_on_its_own_flags(tmp_path):
    """an eager test loop stepped by hand: after each step the flags the post launch left are copied to the host and fed to the
    restatement; the written file equals it bit for bit, and its rallies are the pairs whose reset_buf rose"""
    N, steps = 64, 200
    env = vis(tmp_path, N, name="start.npz")
    env.run_test(policy(networks(2, seed=9), N, clip_obs=5.0, clip_actions=1.0), 0, graph=False)   # reset, render_vis(init), export
    want, rose = RS.RallyStats(N), 0
    for _ in range(steps):
        env.test_step(False)                 # the reset at its start clears reset_buf of the pairs it resets
        want.step(flags(env))
        rose += int((env.reset_buf[0::2] != 0).sum())
    env.cfg["env"]["b200_rally_stats_file"] = str(tmp_path / "end.npz")
    z = np.load(env.export_rally_stats())
    exp = expected_file(want, env, steps)
    assert sorted(z.files) == sorted(exp)
    for k, v in exp.items():
        assert z[k].dtype == np.asarray(v).dtype, k
        np.testing.assert_array_equal(z[k], v, k)
    assert int(z["rallies"]) == rose > N // 2
    assert int(z["hits"].sum()) > 0 and int(z["shots_sum"]) > 0
    check_invariants(want.arrays())


def run_file(tmp_path, graph, name, steps=150):
    N = 64
    env = vis(tmp_path, N, name=name, seed=3)
    env.run_test(policy(networks(2, seed=9), N, clip_obs=5.0, clip_actions=1.0), steps, graph=graph)
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
    assert int(a["rallies"]) > 0 and int(a["test_steps"]) == 150
    lines = [ln for ln in capsys.readouterr().out.splitlines() if ln.startswith("rallies:")]
    assert len(lines) == 3 and len(set(lines)) == 1


def test_file_is_written_before_the_recorders_exit(tmp_path, monkeypatch):
    monkeypatch.chdir(tmp_path)
    N = 32
    env = vis(tmp_path, N, record=True, num_rec_frames=20, num_eg=1, rec_fname=None)
    with pytest.raises(SystemExit):
        env.run_test(policy(networks(2, seed=9), N, clip_obs=5.0, clip_actions=1.0), 100, graph=True)
    z = np.load(tmp_path / "rallies.npz")
    assert int(z["test_steps"]) == 19
    np.testing.assert_array_equal(z["shots_hist"], env._rstats["shots_hist"].cpu().numpy())


def test_without_the_key_nothing_is_allocated_or_launched(tmp_path, monkeypatch):
    """the step graph of the test task without the key has the kernels of the training task's step; the key adds exactly one"""
    from vid2player3d_b200 import native_v2p
    from vid2player3d_b200.tasks import PhysicsMVAEControllerDual
    N = 32
    counts = {}
    for key in (False, True):
        env = vis(tmp_path, N, stats=key)
        env.reset()
        env.enable_cuda_graph(count_nodes=True)
        counts[key] = env.graph_kernel_nodes
    cfg = v2p_dual_cfg(N)
    cfg["env"]["physics"]["assetFileName"] = "smpl_mesh_humanoid_federer.xml"
    cfg["env"]["is_train"] = False                     # as the test task sets it
    train = PhysicsMVAEControllerDual(cfg, SIM_PARAMS, 1, "cuda", 0, True)
    train.reset()
    train.enable_cuda_graph(count_nodes=True)
    assert counts[False] is not None and counts[False] == train.graph_kernel_nodes and counts[True] == counts[False] + 1

    def refuse(*a, **k):
        raise AssertionError("eval_rally_stats launched without b200_rally_stats")
    monkeypatch.setattr(native_v2p, "eval_rally_stats", refuse)
    monkeypatch.chdir(tmp_path)
    env = vis(tmp_path, N, stats=False)
    env.run_test(policy(networks(2, seed=9), N, clip_obs=5.0, clip_actions=1.0), 40, graph=True)
    assert env._test_graphs is not None and env._rstats is None
    assert not os.path.exists(tmp_path / "out")
