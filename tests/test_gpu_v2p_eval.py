"""GPU checks of the test-time tasks' launches (include/b200env_v2p.h: the eval rule of b200v2p_controller_post, b200v2p_eval_record,
b200v2p_eval_best) against the fixture made by executing the reference (tests/golden/v2p_eval.npz) and against the float
restatement oracle/ref_port_eval.py, and the MVAEControllerVis / MVAEControllerVisDual loop the way V2PPlayer.run drives it."""
import numpy as np
import pytest
import torch

from conftest import golden
from helpers import SIM_PARAMS, v2p_cfg, v2p_dual_cfg
from oracle import ref_port_eval as R

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
RESET_IN = ("progress", "tar_time", "tar_time_total", "tar_action", "swing_type_cycle", "has_contact", "has_bounce", "est_bounce_in",
            "ball_pos", "root_pos", "ball_vel", "est_bounce_pos", "target_bounce_pos")
REC_FIELDS = ("joint_rot", "root_pos", "ball_pos", "phase", "swing_type", "tar_action")


def D(a):
    return torch.as_tensor(np.ascontiguousarray(a), device=DEV).contiguous()


class PostEval:
    """the post launch with the eval rule on a standalone state: no estimator, no new contact / bounce this step, no advance, so the
    reset rule sees exactly the given inputs"""

    def __init__(self, n):
        from vid2player3d_b200 import native_v2p as V
        self.V, self.n = V, n
        z = lambda *s, dt=torch.float32: torch.zeros(*s, device=DEV, dtype=dt)  # noqa: E731
        self.m = dict(meter_sum=z(4, n), meter_count=z(4, n, dt=torch.long), meter_avg=torch.ones(4, n, device=DEV), meter_max=z(4, n))
        self.t = dict(rigid_body_state=z(n, 26, 13), ball_states=z(n, 26), root_vel=z(n, 3), racket_pos=z(n, 3), racket_normal=z(n, 3),
                      has_contact_now=z(n, dt=torch.bool), has_bounce_now=z(n, dt=torch.bool), bounce_pos=z(n, 3), ball_traj=z(n, 100, 3),
                      phase=z(n), swing_type=z(n, dt=torch.long), bounce_in=z(n, dt=torch.bool), reset_reaction=z(n, dt=torch.bool),
                      reset_recovery=z(n, dt=torch.bool), est_bounce_time=z(n), est_max_height=z(n), distance=z(n), obs_buf=z(n, 255),
                      rew_buf=z(n), sub_rewards=z(n, 2), reset_buf=z(n, dt=torch.long), terminate_buf=z(n, dt=torch.long), est_x=None,
                      est_y=None, **self.m)

    def __call__(self, s, L):
        t = dict(self.t)
        for k in RESET_IN:
            t[{"progress": "progress_buf", "est_bounce_in": "est_bounce_in"}.get(k, k)] = D(s[k])
        cfg = dict(n=self.n, bodies_per_env=26, ball_stride=26, racket_body=24, num_obs=255, obs_traj_len=10, use_target=0, reward_type=2,
                   early_termination=0, max_episode_length=300, est_nx=0, est_ny=0, scale_pos=5.0, scale_phase=10.0, scale_bounce_pos=1.0,
                   scale_bounce_time=0.5, w_pos=0.1, w_ball_pos=0.9, court_min=(-5, -16), court_max=(5, -10), est_params=np.zeros(15),
                   eval=1, eval_episode_length=L)
        self.V.controller_post(cfg, t)
        return [t[k].cpu().numpy().astype(bool) for k in ("terminate_buf", "reset_reaction", "reset_recovery")]

    def meters(self):
        return {k[6:]: v.cpu().numpy() for k, v in self.m.items()}


def check_meters(got, want, what):
    np.testing.assert_array_equal(got["count"], want["count"], what)
    np.testing.assert_array_equal(got["sum"][:3], want["sum"][:3], what)
    for k in ("sum", "max", "avg"):   # the norm of the position error may round differently: 2 ulp
        np.testing.assert_array_max_ulp(got[k], want[k], maxulp=2)


def test_eval_rule_matches_reference_fixture():
    z = golden("v2p_eval.npz")
    T, N = z["reset_progress"].shape
    p = PostEval(N)
    for t in range(T):
        flags = p({k: z["reset_" + k][t] for k in RESET_IN}, int(z["reset_episode_length"]))
        for f, k in zip(flags, ("terminate", "reaction", "recovery")):
            np.testing.assert_array_equal(f, z["reset_out_" + k][t], f"step {t} {k}")
        check_meters(p.meters(), {k: z["reset_out_meter_" + k][t] for k in ("sum", "count", "avg", "max")}, f"step {t}")


def random_state(g, n, L):
    r = lambda *s: g.random(s)  # noqa: E731
    rp = g.standard_normal((n, 3)).astype(np.float32)
    return dict(progress=g.integers(L - 2, L + 2, n), tar_time=g.integers(60, 80, n), tar_time_total=g.integers(65, 75, n),
                tar_action=g.integers(0, 2, n), swing_type_cycle=g.integers(-1, 4, n), has_contact=r(n) < 0.5, has_bounce=r(n) < 0.5,
                est_bounce_in=r(n) < 0.6, root_pos=rp, ball_pos=(rp + g.standard_normal((n, 3)) * 1.5).astype(np.float32),
                ball_vel=(g.standard_normal((n, 3)) * 4).astype(np.float32), est_bounce_pos=(g.standard_normal((n, 3)) * 3).astype(np.float32),
                target_bounce_pos=(g.standard_normal((n, 3)) * 3).astype(np.float32))


@pytest.mark.parametrize("n", [1, 2, 4, 5, 8, 9, 8193])
def test_eval_rule_matches_restatement(n):
    g = np.random.default_rng(n)
    p, M = PostEval(n), R.new_meters(n)
    for step in range(6):
        s = random_state(g, n, 20)
        got = p(s, 20)
        want = R.eval_reset(s, 20, M)
        for a, b, k in zip(got, want, ("terminate", "reaction", "recovery")):
            np.testing.assert_array_equal(a, b, f"n={n} step {step} {k}")
    check_meters(p.meters(), M, f"n={n}")


def frame(g, n):
    return dict(joint_rot=g.standard_normal((n, 24, 3)).astype(np.float32), root_pos=g.standard_normal((n, 3)).astype(np.float32),
                ball_pos=g.standard_normal((n, 3)).astype(np.float32), target_pos=g.standard_normal((n, 3)).astype(np.float32),
                phase=g.random(n).astype(np.float32), swing_type=g.integers(-1, 4, n), tar_action=g.integers(0, 2, n))


def rec_buffers(n, cap, fields):
    shp = dict(joint_rot=(24, 3), root_pos=(3,), ball_pos=(3,), target_pos=(3,), phase=(), swing_type=(), tar_action=())
    return {k: np.zeros((n, cap) + shp[k], np.int64 if k in ("swing_type", "tar_action") else np.float32) for k in fields}


@pytest.mark.parametrize("n", [1, 5, 9, 8193])
def test_single_recorder_counter_and_capacity(n):
    from vid2player3d_b200 import native_v2p as V
    cap, g = 4, np.random.default_rng(n)
    fields = ("joint_rot", "root_pos", "ball_pos", "target_pos", "phase", "swing_type")
    want = rec_buffers(n, cap, fields)
    dev = {k: D(v) for k, v in want.items()}
    row, done = torch.zeros(1, device=DEV, dtype=torch.long), torch.zeros(1, device=DEV, dtype=torch.int32)
    for call in range(cap + 2):            # the last two calls are past the capacity: nothing is written
        f = frame(g, n)
        V.eval_record(n, cap, dict(row_counter=row, done_counter=done, **{k: D(f[k]) for k in fields},
                                   **{"rec_" + k: v for k, v in dev.items()}))
        R.record(want, np.full(n, call), f)
    assert int(row.item()) == cap + 2 and int(done.item()) == 0
    for k in fields:
        np.testing.assert_array_equal(dev[k].cpu().numpy(), want[k], k)


@pytest.mark.parametrize("n", [2, 8, 10, 8194])
def test_dual_recorder_rows_from_progress(n):
    """rows from progress_buf: row 0 written only while progress is 0 (the init call), rows at or past the capacity dropped"""
    from vid2player3d_b200 import native_v2p as V
    cap, g = 6, np.random.default_rng(n)
    want = rec_buffers(n, cap, REC_FIELDS)
    dev = {k: D(v) for k, v in want.items()}
    progress = np.zeros(n, np.int64)
    for call in range(10):
        if call:
            progress = np.where(g.random(n) < 0.15, 1, progress + 1)      # a reset pair restarts at row 1
        f = frame(g, n)
        V.eval_record(n, cap, dict(progress_buf=D(progress), **{k: D(f[k]) for k in REC_FIELDS}, **{"rec_" + k: v for k, v in dev.items()}))
        R.record(want, progress, f)
    for k in REC_FIELDS:
        np.testing.assert_array_equal(dev[k].cpu().numpy(), want[k], k)


class DeviceBest:
    def __init__(self, n, cap, eg):
        self.n, self.cap, self.eg = n, cap, eg
        i64 = lambda *s: torch.zeros(*s, device=DEV, dtype=torch.long)  # noqa: E731
        self.lst = dict(list_len=i64(1), order=i64(eg), best_distance=torch.zeros(eg, device=DEV), best_env=i64(eg), best_nframes=i64(eg),
                        copy_slot=i64(1))
        self.rec = {k: D(v) for k, v in rec_buffers(n, cap, REC_FIELDS).items()}
        self.best = {k: D(v.reshape((eg, 2) + v.shape[1:])) for k, v in rec_buffers(2 * eg, cap, REC_FIELDS).items()}

    def step(self, f, progress, reset, distance):
        from vid2player3d_b200 import native_v2p as V
        rec = {"rec_" + k: v for k, v in self.rec.items()}
        V.eval_record(self.n, self.cap, dict(progress_buf=D(progress), **{k: D(f[k]) for k in REC_FIELDS}, **rec))
        V.eval_best(self.n, self.cap, self.eg, dict(reset_buf=D(reset), progress_buf=D(progress), distance=D(distance), **self.lst, **rec,
                                                    **{"best_" + k: v for k, v in self.best.items()}))

    def entries(self):
        L = int(self.lst["list_len"].item())
        out = []
        for s in self.lst["order"][:L].tolist():
            nf = int(self.lst["best_nframes"][s])
            out.append(dict(distance=np.float32(self.lst["best_distance"][s].item()), env=int(self.lst["best_env"][s]), nframes=nf,
                            arrays={k: v[s, :, :nf].cpu().numpy() for k, v in self.best.items()}))
        return out


def same_list(got, want):
    assert [(e["distance"], e["env"], e["nframes"]) for e in got] == [(e["distance"], e["env"], e["nframes"]) for e in want]
    for a, b in zip(got, want):
        for k in REC_FIELDS:
            np.testing.assert_array_equal(a["arrays"][k], b["arrays"][k], k)


def test_best_list_matches_reference_fixture():
    z = golden("v2p_eval.npz")
    S, N = z["dual_progress"].shape
    b = DeviceBest(N, int(z["dual_capacity"]), int(z["dual_num_eg"]))
    for s in range(S):
        b.step({k: z["dual_" + k][s] for k in REC_FIELDS}, z["dual_progress"][s], z["dual_reset"][s], z["dual_distance"][s])
    got = b.entries()
    np.testing.assert_array_equal([e["distance"] for e in got], z["dual_best_distance"])
    np.testing.assert_array_equal([e["nframes"] for e in got], z["dual_best_nframes"])
    for k in REC_FIELDS:
        np.testing.assert_array_equal(np.concatenate([e["arrays"][k] for e in got], 1), z["dual_best_" + k])


@pytest.mark.parametrize("n,eg", [(2, 1), (8, 3), (10, 4), (8194, 5)])
def test_best_list_matches_restatement(n, eg):
    """random pair flags (both players, like the dual FSM), distances on a coarse grid so that equal sums occur, rallies past the
    capacity"""
    cap, g = 7, np.random.default_rng(n + eg)
    b, want = DeviceBest(n, cap, eg), []
    rec = rec_buffers(n, cap, REC_FIELDS)
    progress, flagged = np.zeros(n, np.int64), np.zeros(n, bool)
    for step in range(25):
        if step:
            progress = np.where(flagged, 0, progress) + 1
        pair = g.random(n // 2) < min(0.3, 6.0 / n)
        reset = np.repeat(pair, 2).astype(np.int64)
        distance = (g.integers(0, 8, n) * 0.5).astype(np.float32)
        f = frame(g, n)
        b.step(f, progress, reset, distance)
        R.record(rec, progress, f)
        R.best_update(want, reset, distance, progress, rec, eg)
        flagged = reset.astype(bool)
    same_list(b.entries(), want)
    idle = DeviceBest(n, cap, eg)            # no flag set: nothing happens
    idle.step(frame(g, n), progress, np.zeros(n, np.int64), np.ones(n, np.float32))
    assert int(idle.lst["list_len"].item()) == 0 and int(idle.lst["copy_slot"].item()) == -1


def run_player_loop(env, frames):
    """V2PPlayer.run (players/v2p_player.py:137-150): reset, render_vis(init=True), then reset of the finished envs + step +
    render_vis, with random high-level actions.  Every call before the last runs under sync-debug "error"; the last one writes the
    episodes (one host read-back per run) and raises SystemExit."""
    env.reset()
    env.render_vis(init=True)
    torch.cuda.synchronize()

    def one():
        env.reset_done()
        env.step(torch.randn(env.num_envs, env.num_actions, device=DEV))
        env.render_vis()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for _ in range(frames - 2):
            one()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    with pytest.raises(SystemExit):
        one()


@pytest.mark.parametrize("select_best", [True, False])
def test_single_player_loop_writes_the_selected_episodes(tmp_path, monkeypatch, select_best):
    """with select_best the candidates follow the restatement (a random policy may leave none); without it envs 0, 1, 2"""
    from vid2player3d_b200.tasks import MVAEControllerVis
    monkeypatch.chdir(tmp_path)
    cfg = v2p_cfg(512)
    cfg["env"].update(record=True, num_rec_frames=90, num_eg=3, select_best=select_best)
    cfg["args"] = type("Args", (), {"cfg": "federer"})
    env = MVAEControllerVis(cfg, SIM_PARAMS, 1, "cuda", 0, True)
    env.enable_cuda_graph()
    run_player_loop(env, cfg["env"]["num_rec_frames"])
    rec = {k: v.cpu().numpy() for k, v in env._rec.items()}
    want = R.select_best(rec["root_pos"], env.bounce_in_rate.avg.cpu().numpy(), env.fh_ratio.avg.cpu().numpy())[:3] if select_best else [0, 1, 2]
    assert int(env._meter_count.sum()) > 0
    assert [int(np.load(p)["env_id"]) for p in env.exported] == list(want)
    for i, p in enumerate(env.exported):
        assert p.endswith(f"out/episodes/federer_{i + 1:03d}.npz")
        z = np.load(p)
        for k, v in rec.items():
            np.testing.assert_array_equal(z[k], v[int(z["env_id"])], k)


def test_dual_loop_writes_the_best_rallies(tmp_path, monkeypatch):
    from vid2player3d_b200.tasks import MVAEControllerVisDual
    monkeypatch.chdir(tmp_path)
    cfg = v2p_dual_cfg(512)
    cfg["env"].update(record=True, num_rec_frames=60, num_eg=4, rec_fname=None)
    env = MVAEControllerVisDual(cfg, SIM_PARAMS, 1, "cuda", 0, True)
    env.enable_cuda_graph()
    run_player_loop(env, cfg["env"]["num_rec_frames"])
    entries = env.best_list()
    assert len(entries) == len(env.exported) and len(entries) > 0
    assert all(a[2] >= b[2] for a, b in zip(entries, entries[1:]))
    for (s, e, dist, nf), p in zip(entries, env.exported):
        z = np.load(p)
        assert list(z["env_ids"]) == [e, e + 1] and z["distance"] == np.float32(dist) and e % 2 == 0
        for k, v in env._best.items():
            np.testing.assert_array_equal(z[k], v[s, :, :nf].cpu().numpy(), k)
