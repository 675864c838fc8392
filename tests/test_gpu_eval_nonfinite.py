"""GPU checks of the test-time evaluation launches on the inputs of a failing policy: NaN, +Inf and -Inf in one float input field of
one env (env 0, envs 31 and 32 across a warp edge, the last env of a ragged final CTA), at the sizes of each launch's own test.  Every
case runs twice, once poisoned and once with the finite value in its place.  What the poisoned env does not feed (other envs' rows,
other motions' buckets, other pairs' state) is bit-identical between the two runs; what it feeds equals the restatement under the
NaN-aware comparator of test_eval_nonfinite (NaN and infinities where the restatement has them, the finite values within the launch's
own tolerance).

- b200env_im_record: a NaN or infinite component of a joint's rotation vector records three NaN angles, the pitch included (torch.clamp
  keeps a NaN); a non-finite root is copied.
- b200env_im_motion_stats, meters and pose forms: the poisoned game's sums and largest error are NaN or infinite in its motion's bucket,
  a NaN game is never a success, and the next game starts clean.
- the eval rule of b200v2p_controller_post: flags and meters as ref_port_eval.eval_reset (a NaN comparison is false; a NaN error does
  not move the meter's max).
- b200v2p_eval_rally_stats: counts as ref_port_rally_stats, whose comparisons are false for a NaN.
- b200v2p_eval_record: any payload copied bit for bit.
- b200env_play_stats, both forms: a non-finite reward of a finishing env makes its log row and the totals NaN or infinite as
  ref_port_im_policy.run_stats; cr stays NaN after the reset (NaN or Inf times 0); the stop flag and the counts do not change.
- b200v2p_eval_ball_stats in a graphed test run with a NaN or infinite ball or root: no recovery event with est_bounce_in set carries
  a non-finite estimate, so the fixed-point error sum never meets one.
- HumanoidSMPLIMVis.run_test with the pose metrics and the recorder on and one env's joint made NaN before a step: the metrics file is
  the restatement replayed on the recorded inputs, and graphed equals eager byte for byte.
- b200v2p_eval_best: the pair taken is torch.argmax's (a NaN above every number, the first NaN of several); a NaN pair enters only an
  empty list and then nothing passes it.  With several NaN pairs torch.argmax returns the first NaN on the CPU, where the fixture was
  made, and on an H100 (torch 2.11, CUDA 12.8: test_torch_argmax_on_the_device_takes_the_first_nan).

Not covered here: the queue fold b200env_im_motion_queue_stats on a poisoned env, and a dual tennis test run with the rally stats and
the best list on and one env poisoned mid-run (each of its launches is covered above on its own)."""
import numpy as np
import pytest
import torch

from oracle import ref_port_ball_stats as B
from oracle import ref_port_eval as E
from oracle import ref_port_im_policy as IP
from oracle import ref_port_pose_metrics as P
from oracle import ref_port_rally_stats as RS
from oracle.ref_port_motion_stats import MotionStats
from test_eval_nonfinite import assert_nonfinite_close
from test_gpu_ball_stats import COUNTS, post_state
from test_gpu_ball_stats import vis as ball_vis
from test_gpu_im_motion_stats import motion_map
from test_gpu_im_pose_metrics import buffers as ms_buffers
from test_gpu_im_pose_metrics import inputs as ms_inputs
from test_gpu_im_pose_metrics import launch as ms_launch
from test_gpu_im_pose_metrics import assert_file, pose_task, replay_oracle
from test_gpu_im_pose_metrics import oracle_step as ms_oracle_step
from test_gpu_im_motion_stats import run as im_run
from test_gpu_im_record import assert_rows
from test_gpu_im_record import buffers as rec_buffers
from test_gpu_im_record import expected as rec_expected
from test_gpu_im_record import launch as rec_launch
from test_gpu_im_record import state as rec_state
from test_gpu_rally_stats import STATE, Device
from test_gpu_v2p_eval import REC_FIELDS, D, DeviceBest, PostEval, frame, random_state
from test_gpu_v2p_eval import rec_buffers as v2p_rec_buffers
from test_gpu_v2p_policy import networks, policy
from test_rally_stats import random_run

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
BAD = {"nan": float("nan"), "+inf": float("inf"), "-inf": float("-inf")}


def placements(n):
    """env 0, envs 31 and 32 (a warp edge), the last env (of a ragged final CTA at the sizes used)"""
    return sorted({e for e in (0, 31, 32, n - 1) if 0 <= e < n})


def same_bits(a, b, what):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    assert a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes(), what


# ------------------------------------------------------------------------------------------------------------- im_record
# field -> (the state key, the element of env e's rows poisoned)
REC_POISON = {"dof_state": ("dof_state", (3 * 20 + 1, 0)), "p_dof_pos": ("p_dof_pos", (3 * 17 + 2,)), "root_pos": ("rigid_body_state", (0, 1)),
              "root_rot": ("rigid_body_state", (0, 4)), "target_root_pos": ("p_rb_pos", (0, 2)), "target_root_rot": ("p_rb_rot", (0, 3))}


@pytest.mark.parametrize("N", [33, 129])
@pytest.mark.parametrize("field", list(REC_POISON))
@pytest.mark.parametrize("bad", list(BAD))
def test_im_record_keeps_the_nan_pitch(N, field, bad):
    """4 envs per CTA: 129 leaves env 128 alone in the last one.  init False, so both copies of the frame read the poisoned rows"""
    key, idx = REC_POISON[field]
    clean = rec_state(N, N)
    ids = list(range(N))
    buf = rec_buffers(N, 1)
    rec_launch(clean, buf, ids, 1, False)
    want_clean = buf["qpos"][:, 0].cpu().numpy()
    for e in placements(N):
        st = {k: v.clone() for k, v in clean.items()}
        st[key][(e,) + idx] = BAD[bad]
        buf = rec_buffers(N, 1)
        rec_launch(st, buf, ids, 1, False)
        got = buf["qpos"][:, 0].cpu().numpy()
        others = np.arange(N) != e
        same_bits(got[others], want_clean[others], f"{field} {bad} env {e}: another env's row changed")
        want = rec_expected(st, [e], False)
        row = got[e:e + 1].astype(np.float64)
        assert_nonfinite_close(row, want, atol=np.inf, what=f"{field} {bad} env {e}")     # where NaN and Inf are
        assert not np.isfinite(want).all()
        fin = np.isfinite(want)
        assert_rows(np.where(fin, row, 0.0), np.where(fin, want, 0.0))                     # the finite values as the launch's own test
        if field in ("dof_state", "p_dof_pos"):
            j = idx[0] // 3
            cp = 0 if field == "dof_state" else 1
            assert np.isnan(row[0, cp, 7 + 3 * j:10 + 3 * j]).all(), "the joint's angles are not all NaN"
        assert_rows(want_clean[e:e + 1].astype(np.float64), rec_expected(clean, [e], False))


# ------------------------------------------------------------------------------------------------------------- eval_best
def nan_list(got, want, what):
    assert [(e["env"], e["nframes"]) for e in got] == [(e["env"], e["nframes"]) for e in want], what
    assert_nonfinite_close([e["distance"] for e in got], [e["distance"] for e in want], what=what)
    for a, b in zip(got, want):
        for k in REC_FIELDS:
            same_bits(a["arrays"][k], b["arrays"][k], f"{what} {k}")


def best_case(n, eg, prefill, flagged, cap=5, seed=0):
    """prefill: finite distances of the pairs flagged on the steps before, one pair a step; flagged {pair: (d0, d1)} of the last step.
    Returns the device list and the restatement's."""
    g = np.random.default_rng(seed)
    b, want = DeviceBest(n, cap, eg), []
    rec = v2p_rec_buffers(n, cap, REC_FIELDS)
    progress = np.zeros(n, np.int64)
    steps = [{p: (x, 1.0)} for p, x in prefill] + [flagged]
    for k, fl in enumerate(steps):
        progress = progress + 1
        reset = np.zeros(n, np.int64)
        distance = g.random(n).astype(np.float32)
        for p, (d0, d1) in fl.items():
            reset[2 * p] = reset[2 * p + 1] = 1
            distance[2 * p], distance[2 * p + 1] = d0, d1
        f = frame(g, n)
        b.step(f, progress, reset, distance)
        E.record(rec, progress, f)
        E.best_update(want, reset, distance, progress, rec, eg)
    return b.entries(), want


LISTS = {"empty": [], "short": [(0, 3.0)], "full": [(0, 1.0), (0, 2.0), (0, 3.0)]}     # pair 0 flagged on the steps before


@pytest.mark.parametrize("n", [2, 2048, 2052])
@pytest.mark.parametrize("lst", list(LISTS))
@pytest.mark.parametrize("bad", list(BAD) + ["inf-inf"])
def test_eval_best_takes_the_first_nan_pair(n, lst, bad):
    """the poisoned pair is the first, 1023 (the last thread's first), 1024 and 1025 (threads 0 and 1, second round) or the last, alone
    or with a larger finite pair before and after it; with the finite value in its place the list is the restatement's too"""
    K, eg = n // 2, 3
    pairs = sorted({p for p in (0, 1023, 1024, 1025, K - 1) if p < K})
    val = (float("inf"), float("-inf")) if bad == "inf-inf" else (BAD[bad], 0.5)
    for p in pairs:
        for company in ({}, {q: (6.0, 6.0) for q in (p - 1, p + 1) if 0 <= q < K}):
            for poisoned in (True, False):
                fl = {**company, p: val if poisoned else (2.5, 0.5)}
                got, want = best_case(n, eg, LISTS[lst], fl, seed=p)
                nan_list(got, want, f"n={n} {lst} {bad} pair {p} {'poisoned' if poisoned else 'finite'} company {sorted(company)}")


@pytest.mark.parametrize("n", [8, 2052])
def test_eval_best_several_nan_pairs_take_the_lowest(n):
    """NaN pairs in several threads, warps and rounds on one step: the lowest NaN pair enters the empty list; after it no pair enters"""
    K = n // 2
    for nans in ([K - 1, 1, 2], [1025, 1024, 1023, 3], [1024, 0], [1023, 1025]):
        nans = [p for p in nans if p < K]
        if len(nans) < 2:
            continue
        fl = {p: (float("nan"), 1.0) for p in nans}
        fl.update({q: (9.0, 9.0) for q in range(K) if q not in nans and q % 97 == 5})
        got, want = best_case(n, 3, [], fl, seed=len(nans))
        nan_list(got, want, f"n={n} NaN pairs {nans}")
        assert len(got) == 1 and got[0]["env"] == 2 * min(nans)
    b = DeviceBest(n, 5, 3)                                            # a NaN in the list: no later pair enters
    g = np.random.default_rng(1)
    for k, fl in enumerate(({1: (float("nan"), 0.0)}, {0: (50.0, 50.0)}, {K - 1: (float("inf"), 1.0)}, {0: (float("nan"), 1.0)})):
        reset = np.zeros(n, np.int64)
        distance = np.ones(n, np.float32)
        for p, (d0, d1) in fl.items():
            reset[2 * p] = reset[2 * p + 1] = 1
            distance[2 * p], distance[2 * p + 1] = d0, d1
        b.step(frame(g, n), np.full(n, k + 1, np.int64), reset, distance)
        e = b.entries()
        assert len(e) == 1 and np.isnan(e[0]["distance"]) and e[0]["env"] == 2 and e[0]["nframes"] == 1


@pytest.mark.parametrize("nan", ["nan", "inf-inf"])
def test_eval_best_a_thread_meets_a_nan_after_a_finite_pair(nan):
    """1026 pairs: threads 0 and 1 scan pairs 0 and 1024, 1 and 1025.  A larger finite pair first and a NaN pair after it in the same
    thread: the thread's own scan must keep the NaN"""
    val = (float("inf"), float("-inf")) if nan == "inf-inf" else (float("nan"), 1.0)
    for fl, env in (({0: (12.0, 0.0), 1024: val}, 2048), ({1: (12.0, 0.0), 1025: val}, 2050),
                    ({0: (12.0, 0.0), 1: (13.0, 0.0), 1024: val, 1025: val}, 2048), ({1: (12.0, 0.0), 1025: val, 7: (20.0, 0.0)}, 2050)):
        got, want = best_case(2052, 3, [], fl, seed=env)
        nan_list(got, want, f"{nan} {sorted(fl)}")
        assert len(got) == 1 and got[0]["env"] == env and np.isnan(got[0]["distance"])


def test_torch_argmax_on_the_device_takes_the_first_nan():
    """the reference runs torch.argmax on the device's distances; the fixture's rule (first NaN) holds there as on the CPU"""
    for n, nans in ((8, [5, 2, 7]), (4096, [3000, 17, 1025]), (1 << 20, [999_999, 70_000, 65_537])):
        x = torch.rand(n, device=DEV)
        x[nans] = float("nan")
        assert int(torch.argmax(x)) == min(nans)
        assert int(torch.argmax(x.cpu())) == min(nans)


# ------------------------------------------------------------------------------------------------------------- motion meters
MS_POISON = {"rew": ("rew", ()), "sub_rewards": ("sub_rewards", (2,)), "body": ("rigid_body_state", (5, 1)),
             "target": ("target_rb_pos", (7, 2))}


def ms_run(N, M, mids, xs, pose):
    buf = ms_buffers(N, M, mids, pose)
    games = torch.zeros(3, device=DEV, dtype=torch.long)
    snap = None
    for k, x in enumerate(xs):
        if x is None:                                             # a new game
            snap = {a: v.clone() for a, v in buf.items()}
            for a in ("env_sums", "env_flags") + (("env_pose", "pose_fill") if pose else ()):
                buf[a].zero_()
            continue
        ms_launch(N, M, x, buf, games, 0.9)
    torch.cuda.synchronize()
    return {a: v.cpu().numpy() for a, v in snap.items()}, {a: v.cpu().numpy() for a, v in buf.items()}


@pytest.mark.parametrize("N,M", [(1, 1), (33, 3), (8197, 1000)])
@pytest.mark.parametrize("pose", [False, True])
@pytest.mark.parametrize("field", list(MS_POISON))
def test_motion_meters_carry_the_poisoned_game(N, M, pose, field):
    """game 0: the poisoned value at step 2, the env's game ends at step 5 (vel at step 3 and acc at step 4 read the poisoned pose
    through pose_hist); game 1 after new_game: the env's next game ends at step 2 and is clean.  The poisoned motion's bucket against the
    restatement over that motion's envs; every other bucket and env row bit-identical to the run with the finite value."""
    mids = motion_map(N, M, N + M)
    g = np.random.default_rng(N)
    ends = [g.integers(1, 7, N), g.integers(1, 4, N)]
    key, idx = MS_POISON[field]
    for e in placements(N):
        ends[0][e], ends[1][e] = 5, 2
        xs = []
        for game, T in ((0, 7), (1, 4)):
            if game:
                xs.append(None)
            xs += [ms_inputs(N, 100 * game + k + 7 * N, k >= ends[game]) for k in range(T)]
        clean = ms_run(N, M, mids, xs, pose)
        m = mids[e]
        sel = np.flatnonzero(mids == m)
        for bad in BAD:
            ps = [None if x is None else {k: v.clone() for k, v in x.items()} for x in xs]
            ps[2][key][(e,) + idx] = BAD[bad]
            got = ms_run(N, M, mids, ps, pose)
            what = f"{field} {bad} env {e}"
            for s in range(2):
                for a in got[s]:
                    if a in ("motion_start", "motion_envs"):
                        continue
                    rows = np.arange(len(got[s][a])) != (m if a in ("counts", "sums", "pose_sums", "success") else e)
                    if a == "pose_hist":
                        continue                                  # a ring of frames: compared through the sums it feeds
                    same_bits(got[s][a][rows], clean[s][a][rows], f"{what}: {a} of another row changed (game {s})")
            for a in ("env_sums", "env_flags", "env_pose"):             # the next game starts clean: nothing carried by pose_hist
                if a in got[1]:
                    same_bits(got[1][a][e], clean[1][a][e], f"{what}: {a} of the poisoned env after new_game")
            ora = P.PoseMetrics(mids[sel], M, 0.9) if pose else MotionStats(mids[sel], M)
            for s, x in enumerate(ps):
                if x is None:
                    ora.new_game()
                else:
                    ms_oracle_step(ora, {k: v[torch.as_tensor(sel, device=v.device)] for k, v in x.items()})
            b = got[1]
            assert np.array_equal(b["counts"][m], ora.counts[m]), what
            assert_nonfinite_close(b["sums"][m], ora.sums[m], rtol=1e-9, atol=1e-12, what=what + " sums")
            assert not np.isfinite(ora.sums[m]).all(), what
            if pose:
                assert np.array_equal(b["success"][m], ora.success[m]) and np.array_equal(b["pose_sums"][m, 4:6], ora.pose_sums[m, 4:6]), what
                assert_nonfinite_close(b["pose_sums"][m], ora.pose_sums[m], rtol=1e-7, atol=1e-12, what=what + " pose sums")
                if field in ("body", "target"):                           # the game's largest error is not finite: no success
                    assert not np.isfinite(ora.pose_sums[m, 6]) and b["success"][m] <= clean[1]["success"][m], what


# ------------------------------------------------------------------------------------------------------------- eval rule
POST_POISON = ("ball_vel", "ball_pos", "root_pos", "est_bounce_pos", "target_bounce_pos")


@pytest.mark.parametrize("n", [1, 33, 8193])
@pytest.mark.parametrize("field", POST_POISON)
def test_eval_rule_on_non_finite_ball_and_root(n, field):
    """four steps of random states, the poisoned env a recovery candidate (to hit, bounce in) whose value is poisoned at steps 1 and 2,
    once without and once with contact; flags exact, meters within 2 ulp and NaN where the restatement's are"""
    L = 20
    g = np.random.default_rng(n)
    base = [random_state(g, n, L) for _ in range(4)]
    for s in base:
        s["progress"][:] = np.minimum(s["progress"], L - 1)
    for e in placements(n):
        for s, hc in zip(base, (False, False, True, False)):
            s["tar_action"][e], s["has_contact"][e], s["est_bounce_in"][e], s["progress"][e] = 1, hc, True, 3
            s["ball_vel"][e, 1] = 0.5                                  # slow: a recovery unless the poison says otherwise
        runs = {}
        for bad in ("finite",) + tuple(BAD):
            p, M, flags = PostEval(n), E.new_meters(n), []
            for k, s in enumerate(base):
                s = {a: v.copy() for a, v in s.items()}
                if bad != "finite" and k in (1, 2):
                    s[field][e, 1 if k == 1 else 0] = BAD[bad]
                got, want = p(s, L), E.eval_reset(s, L, M)
                for a, b, name in zip(got, want, ("terminate", "reaction", "recovery")):
                    np.testing.assert_array_equal(a, b, f"{field} {bad} env {e} step {k} {name}")
                flags.append(got)
            meters = p.meters()
            for k in ("sum", "max", "avg"):
                assert_nonfinite_close(meters[k], M[k], rtol=2.5e-7, what=f"{field} {bad} env {e} meter {k}")
            np.testing.assert_array_equal(meters["count"], M["count"])
            runs[bad] = meters, flags
        others = np.arange(n) != e
        for bad in BAD:
            for k in ("sum", "count", "avg", "max"):
                same_bits(runs[bad][0][k][:, others], runs["finite"][0][k][:, others], f"{field} {bad} env {e}: meter {k} of another env")
            for a, b in zip(runs[bad][1], runs["finite"][1]):
                for x, y in zip(a, b):
                    same_bits(x[others], y[others], f"{field} {bad} env {e}: flags of another env")


# ------------------------------------------------------------------------------------------------------------- rally stats
@pytest.mark.parametrize("n", [2, 34, 8194])
@pytest.mark.parametrize("field", ["ball_pos", "root_pos"])
def test_rally_stats_on_non_finite_ball_and_root(n, field):
    """60 steps of random flags; at step 7 the env's ball or root is poisoned in y (behind) or z (twice).  Counts and pair state exact"""
    for e in placements(n):
        for bad in BAD:
            for c in (1, 2):
                dev, want, k = Device(n), RS.RallyStats(n), [0]

                def step(s):
                    if k[0] == 7:
                        s[field] = s[field].copy()
                        s[field][e, c] = BAD[bad]
                    dev.launch(s)
                    k[0] += 1
                    return want.step(s)
                random_run(np.random.default_rng(n + c), n, 60, step)
                got, w = dev.arrays(), want.arrays()
                for a in STATE + ("totals", "ends", "player", "shots_hist"):
                    np.testing.assert_array_equal(got[a], w[a], f"{field}[{c}] {bad} env {e}: {a}")
                assert dev.slack_untouched()


# ------------------------------------------------------------------------------------------------------------- recorder
@pytest.mark.parametrize("n", [2, 34, 8194])
def test_eval_record_copies_non_finite_payloads(n):
    """the dual recorder: one field of one env poisoned (NaN with a payload, +-Inf) each call; every row as the restatement's, bit for
    bit"""
    from vid2player3d_b200 import native_v2p as V
    cap, g = 4, np.random.default_rng(n)
    want = v2p_rec_buffers(n, cap, REC_FIELDS)
    dev = {k: D(v) for k, v in want.items()}
    nan_payload = np.array([0x7FC01234], np.uint32).view(np.float32)[0]
    progress, call = np.zeros(n, np.int64), 0
    for e in placements(n):
        for field in ("joint_rot", "root_pos", "ball_pos", "phase"):
            for bad in (nan_payload, np.float32(np.inf), np.float32(-np.inf)):
                f = frame(g, n)
                row = f[field].reshape(n, -1)[e]
                row[call % row.size] = bad
                progress = (progress + 1) % cap
                V.eval_record(n, cap, dict(progress_buf=D(progress), **{k: D(f[k]) for k in REC_FIELDS},
                                           **{"rec_" + k: v for k, v in dev.items()}))
                E.record(want, progress, f)
                call += 1
    for k in REC_FIELDS:
        same_bits(dev[k].cpu().numpy(), want[k], k)


# ------------------------------------------------------------------------------------------------------------- play stats
def play_run(N, queue, rews, dones):
    """b200env_play_stats over the steps; returns the final state and the games row after each step"""
    from vid2player3d_b200 import native
    f32 = lambda *sh: torch.zeros(*sh, device=DEV)  # noqa: E731
    st = dict(rew=f32(N), cr=f32(N), steps=f32(N), prev_dones=f32(N), totals=torch.zeros(2, device=DEV, dtype=torch.float64),
              log=torch.zeros(8, 3, device=DEV, dtype=torch.float64), games=torch.zeros(3, device=DEV, dtype=torch.long),
              step=torch.zeros(1, device=DEV, dtype=torch.long))
    rb, games = torch.zeros(N, device=DEV, dtype=torch.long), []
    for r, d in zip(rews, dones):
        st["rew"].copy_(torch.from_numpy(r))
        rb.copy_(torch.from_numpy(d.astype(np.int64)))
        native.play_stats(dict(n=N, max_log=8, n_games=1 << 62, queue_games=(1 << 62) if queue else 0), dict(st, reset_buf=rb))
        games.append(st["games"].cpu().numpy())
    return {k: v.cpu().numpy() for k, v in st.items()}, np.stack(games)


@pytest.mark.parametrize("N", [1, 33, 1025])
@pytest.mark.parametrize("queue", [False, True])
def test_play_stats_with_a_non_finite_reward(N, queue):
    """1024 threads: env 1024 is thread 0's second.  The poisoned env's reward at step 2; it finishes at step 4 (env 0 at the last
    step, where the reference's loop ends).  Totals and log rows as ref_port_im_policy.run_stats; cr stays NaN after the reset (NaN or
    Inf times 0); the stop flag, the game counts and every other env's row as in the finite run"""
    T = 8
    g = np.random.default_rng(N)
    rews = [g.random(N).astype(np.float32) for _ in range(T)]
    for e in placements(N):
        end = g.integers(1, T - 1, N)
        end[0], end[e] = T - 1, (T - 1 if e == 0 else 4)
        keep = (np.arange(N) != e) & (np.arange(N) != 0)
        dones = [(k >= end) & ~((g.random(N) < 0.1) & keep) for k in range(T)]     # a few envs drop back
        for d in dones[:-1]:
            d[0] = False
        fin, fin_games = play_run(N, queue, rews, dones)
        for bad in BAD:
            rp = [r.copy() for r in rews]
            rp[2][e] = BAD[bad]
            got, games = play_run(N, queue, rp, dones)
            what = f"{'queue' if queue else 'run'} {bad} env {e}"
            same_bits(games, fin_games, what + ": games and stop flag")
            others = np.arange(N) != e
            for k in ("cr", "steps", "prev_dones"):
                same_bits(got[k][others], fin[k][others], f"{what}: {k} of another env")
            assert np.isnan(got["cr"][e]), what
            lines, sr, ss, gp = IP.run_stats([[(r, d) for r, d in zip(rp, dones)]], 1 << 40, T)
            rows = int(games[-1][2])
            assert rows == len(lines) and int(games[-1][0]) == gp, what
            np.testing.assert_array_equal(got["log"][:rows, 0], [c for c, _, _ in lines], what)
            assert_nonfinite_close(got["log"][:rows, 1:], [[r, st] for _, r, st in lines], rtol=1e-5, what=what + " log")
            assert_nonfinite_close(got["totals"], [sr, ss], rtol=1e-5, what=what + " totals")
            assert not np.isfinite(got["totals"][0])


# ------------------------------------------------------------------------------------------------------------- ball stats
@pytest.mark.parametrize("field", ["ball_pos", "ball_vel", "root_pos"])
def test_ball_stats_never_see_a_non_finite_estimate(tmp_path, field):
    """a graphed test run of 64 envs; before steps 20, 40, 60 and 80 the ball's (or the humanoid root's) state of env 0, 31, 32 and 63 is
    made NaN, +Inf, -Inf and NaN.  The estimator writes est_bounce_pos and est_bounce_in together, and in_court is false for a NaN, so
    every recovery event with est_bounce_in set carries a finite estimate and the fixed-point error sum never meets a NaN (which
    __double2ll_rn would turn into INT64_MIN).  The buckets equal the restatement fed the post launch's values."""
    N, P, steps = 64, 7, 160
    env = ball_vis(tmp_path, N, P)
    task = env._physics_player.task
    env.run_test(policy(networks(1, seed=9), N, clip_obs=5.0, clip_actions=1.0), 0, graph=True)
    want = B.BallStats(P)
    want.served[0] = N
    cursor = task._ball_pool_cursor.cpu().numpy()
    rbs = task._rigid_body_state.view(N, 26, 13)
    row, cols = {"ball_pos": (1, slice(0, 3)), "ball_vel": (1, slice(7, 10)), "root_pos": (0, slice(0, 3))}[field]
    poison = {20: (0, float("nan")), 40: (31, float("inf")), 60: (32, float("-inf")), 80: (63, float("nan"))}
    saw = 0
    for k in range(steps):
        if k in poison:
            e, v = poison[k]
            task._root_states.view(N, 2, 13)[e, row, cols] = v
            rbs[e, 25 if row else 0, cols] = v
        env.test_step(True)
        new = task._ball_pool_cursor.cpu().numpy()
        moved = np.flatnonzero(new != cursor)
        np.add.at(want.served, cursor[moved], 1)
        cursor = new
        ps, rec = post_state(env), env._reset_recovery_buf.cpu().numpy().astype(bool)
        ev = rec & ps["est_bounce_in"].astype(bool)
        assert np.isfinite(ps["est_bounce_pos"][ev]).all() and np.isfinite(ps["target_bounce_pos"][ev]).all(), f"step {k}"
        saw += int((~np.isfinite(task._ball_pos.cpu().numpy()).all(1) | ~np.isfinite(task._root_pos.cpu().numpy()).all(1)).any())
        want.events(ps, rec, cursor)
    assert saw > 0, "the poison never reached the post launch"
    z = np.load(env.export_ball_stats())
    for k in ("served",) + COUNTS:
        np.testing.assert_array_equal(z[k], getattr(want, k), k)
    assert np.isfinite(want.bounce_err_sum).all() and (z["bounce_err_sum"] >= 0).all()
    np.testing.assert_allclose(z["bounce_err_sum"], want.bounce_err_sum, rtol=1e-6, atol=0)


# ------------------------------------------------------------------------------------------------------------- imitation run_test
def poisoned_im_run(tmp_path, name, graph, record=None, env=5, before=2):
    """run_test with the pose metrics and the recorder on; env's joint position made NaN before step `before`"""
    task = pose_task(sample_first_motions=True, b200_record_qpos=True, b200_record_envs="all", num_rec_frames=1000)
    task._rec_path = str(tmp_path / f"{name}_rec.npz")
    step, calls = task.test_step, [0]

    def poisoned_step(*a, **k):
        if calls[0] == before:
            task._dof_state.view(task.num_envs, -1, 2)[env, 61, 0] = float("nan")
        calls[0] += 1
        return step(*a, **k)
    task.test_step = poisoned_step
    _, got, _ = im_run(task, tmp_path / f"{name}.npz", graph=graph, record=record)
    return task, got, dict(np.load(task._rec_path))


def test_im_run_test_with_a_nan_env(tmp_path):
    """the metrics file equals the restatement replayed on the recorded device inputs, NaN where it has NaN; graphed equals eager byte
    for byte, the recorded qpos included, where the poisoned env's rows carry the NaN and no other env's do"""
    record = []
    task, got, rec = poisoned_im_run(tmp_path, "g", True, record)
    assert_file(got, replay_oracle(task, record))                       # assert_allclose: NaN positions must match
    assert np.isnan(rec["qpos"][5]).any() and not np.isnan(rec["qpos"][np.arange(len(rec["qpos"])) != 5]).any()
    _, got_e, rec_e = poisoned_im_run(tmp_path, "e", False)
    for a, b in ((got, got_e), (rec, rec_e)):
        assert a.keys() == b.keys()
        for k, v in a.items():
            assert v.dtype == b[k].dtype and v.tobytes() == b[k].tobytes(), k
