"""Golden fixture of the test-time tasks (v2p_eval.npz), produced by EXECUTING the reference's own code on CPU through fake `self`
objects: MVAEControllerVis._compute_reset / _compute_stats / render_vis (vid2player/env/tasks/mvae_controller_vis.py:64-170) and
MVAEControllerVisDual.render_vis (mvae_controller_vis_dual.py:87-202), smpl_visualizer mocked, render_one_result replaced by a
capture of what it is given, exit() caught.  Run where the reference is present:  python tests/golden/make_golden_eval.py

A seeded, scripted sequence makes every branch occur: contact or none, bounce, in-time, ball behind, slow ball, progress past the
episode length, recovery with est_bounce_in on and off; in dual mode pairs flagged on the same step, equal distances, an insertion
refused while the list is short and a rally that fills the (small) recording buffer.
"""
import os
import sys
from types import SimpleNamespace

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import _refenv  # noqa: E402

_refenv.setup("vid2player")

from env.tasks import mvae_controller_vis as V  # noqa: E402
from env.tasks import mvae_controller_vis_dual as VD  # noqa: E402
from utils.common import AverageMeterUnSync  # noqa: E402

torch.set_num_threads(1)
OUT = {}

# ------------------------------------------------------------------ single: reset rule + statistics over a scripted sequence
N, T, L = 16, 12, 8


class FakeVis(V.MVAEControllerVis):
    def __init__(self):
        pass


g = torch.Generator().manual_seed(7)
s = FakeVis()
s.cfg = {"env": {"episodeLength": L}}
s.num_envs = N
s._terminate_buf = torch.zeros(N, dtype=torch.long)
s.reset_buf = torch.zeros(N, dtype=torch.long)
s.hit_rate, s.bounce_in_pos_error, s.bounce_in_rate, s.fh_ratio = (AverageMeterUnSync(dim=N) for _ in range(4))
task = SimpleNamespace()
s._physics_player = SimpleNamespace(task=task)
s._mvae_player = SimpleNamespace()
inputs = {k: [] for k in ("progress", "tar_time", "tar_time_total", "tar_action", "swing_type_cycle", "has_contact", "has_bounce",
                          "est_bounce_in", "ball_pos", "root_pos", "ball_vel", "est_bounce_pos", "target_bounce_pos")}
outputs = {k: [] for k in ("terminate", "reaction", "recovery", "meter_sum", "meter_count", "meter_avg", "meter_max")}
for t in range(T):
    r = lambda *sh: torch.rand(*sh, generator=g)  # noqa: E731
    st = dict(progress=torch.randint(L - 3, L + 3, (N,), generator=g), tar_time=torch.randint(60, 80, (N,), generator=g),
              tar_time_total=torch.randint(65, 75, (N,), generator=g), tar_action=torch.randint(0, 2, (N,), generator=g),
              swing_type_cycle=torch.randint(-1, 4, (N,), generator=g), has_contact=r(N) < 0.5, has_bounce=r(N) < 0.5,
              est_bounce_in=r(N) < 0.6, root_pos=torch.randn(N, 3, generator=g))
    st["ball_pos"] = st["root_pos"] + torch.randn(N, 3, generator=g) * torch.tensor([1.0, 1.5, 1.0])    # ball behind for some
    st["ball_vel"] = torch.randn(N, 3, generator=g) * 4.0                                                 # |vy| < 2 for some
    st["est_bounce_pos"] = torch.randn(N, 3, generator=g) * 3.0
    st["target_bounce_pos"] = torch.randn(N, 3, generator=g) * 3.0
    s.progress_buf, s._tar_time, s._tar_time_total, s._tar_action = st["progress"], st["tar_time"], st["tar_time_total"], st["tar_action"]
    task._has_racket_ball_contact, task._has_bounce = st["has_contact"], st["has_bounce"]
    s._ball_pos, s._root_pos, s._ball_vel = st["ball_pos"], st["root_pos"], st["ball_vel"]
    s._mvae_player._swing_type_cycle = st["swing_type_cycle"]
    s._est_bounce_in, s._est_bounce_pos, s._target_bounce_pos = st["est_bounce_in"], st["est_bounce_pos"], st["target_bounce_pos"]
    s._compute_reset()
    for k in inputs:
        inputs[k].append(st[k].numpy().copy())
    outputs["terminate"].append(s._terminate_buf.numpy().astype(bool))
    outputs["reaction"].append(s._reset_reaction_buf.numpy().copy())
    outputs["recovery"].append(s._reset_recovery_buf.numpy().copy())
    for f in ("sum", "count", "avg", "max"):
        outputs["meter_" + f].append(np.stack([getattr(getattr(s, m), f).numpy() for m in
                                               ("hit_rate", "fh_ratio", "bounce_in_rate", "bounce_in_pos_error")]).copy())
for k, v in inputs.items():
    OUT["reset_" + k] = np.stack(v)
for k, v in outputs.items():
    OUT["reset_out_" + k] = np.stack(v)
OUT["reset_episode_length"] = np.int64(L)
rec = OUT["reset_out_recovery"]
assert rec.any() and (rec & OUT["reset_est_bounce_in"]).any() and (rec & ~OUT["reset_est_bounce_in"]).any()
assert OUT["reset_out_terminate"].any() and (~OUT["reset_out_terminate"]).any() and OUT["reset_out_reaction"].any()

# ------------------------------------------------------------------ single: recording + select_best
NR, F, EG = 8, 5, 3


def render_single(select_best):
    v = FakeVis()
    v.cfg = {"env": {"record": True, "num_rec_frames": F, "select_best": select_best, "num_eg": EG, "start_eg_id": 1}}
    v.cfg_v2p = {}
    v.headless, v.num_envs, v.frame_index = True, NR, 0
    v.joint_rot_all = v.root_pos_all = v.ball_pos_all = v.target_pos_all = v.phase_all = v.swing_type_all = None
    v.bounce_in_rate, v.fh_ratio = AverageMeterUnSync(dim=NR), AverageMeterUnSync(dim=NR)
    v.bounce_in_rate.avg[:] = torch.tensor([1.0, 0.9, 0.96, 1.0, 1.0, 0.5, 1.0, 0.99])
    v.fh_ratio.avg[:] = torch.tensor([0.5, 0.1, 0.2, 1.0, 0.0, 0.1, 0.59, 0.3])
    v._mvae_player = SimpleNamespace()
    got = []
    v.render_one_result = lambda env_id, eg_id: got.append((int(env_id), int(eg_id)))
    gs = torch.Generator().manual_seed(11)
    frames = {k: [] for k in ("joint_rot", "root_pos", "ball_pos", "target_pos", "phase", "swing_type")}
    done = False
    for i in range(F):
        fr = dict(joint_rot=torch.randn(NR, 24, 3, generator=gs), root_pos=torch.randn(NR, 3, generator=gs),
                  ball_pos=torch.randn(NR, 3, generator=gs), target_pos=torch.randn(NR, 3, generator=gs),
                  phase=torch.rand(NR, generator=gs) * 6.0, swing_type=torch.randint(-1, 4, (NR,), generator=gs))
        v._joint_rot, v._root_pos, v._ball_pos, v._target_bounce_pos = fr["joint_rot"], fr["root_pos"], fr["ball_pos"], fr["target_pos"]
        v._mvae_player._phase_pred, v._mvae_player._swing_type_cycle = fr["phase"], fr["swing_type"]
        for k in frames:
            frames[k].append(fr[k].numpy())
        try:
            v.render_vis(init=(i == 0))
        except SystemExit:
            done = True
    assert done and len(got) == EG
    return frames, got, v


frames, got, v = render_single(True)
for k, x in frames.items():
    OUT["single_" + k] = np.stack(x, 1)          # [NR, F, ...] as recorded
OUT["single_bounce_in_avg"] = v.bounce_in_rate.avg.numpy()
OUT["single_fh_avg"] = v.fh_ratio.avg.numpy()
OUT["single_best_env_ids"] = np.array([e for e, _ in got])
OUT["single_best_eg_ids"] = np.array([e for _, e in got])
OUT["single_num_eg"] = np.int64(EG)
_, got_all, _ = render_single(False)
OUT["single_all_env_ids"] = np.array([e for e, _ in got_all])

# ------------------------------------------------------------------ dual: recording at progress_buf + best-episode list
ND, CAP, TD, EGD = 8, 12, 14, 3


class FakeVisDual(VD.MVAEControllerVisDual):
    def __init__(self):
        pass


def render_dual(schedule, seed, steps):
    """MVAEControllerVisDual.render_vis over steps + 1 scripted steps: schedule {step: {pair: (distance of player 0, of player 1)}}
    flags those pairs; other distances are random.  Returns the per-step inputs, the final list and the render_one_result indices."""
    d = FakeVisDual()
    d.cfg = {"env": {"record": True, "num_rec_frames": steps + 1, "num_eg": EGD, "start_eg_id": 1}}
    d.headless, d.num_envs, d.frame_index, d.num_best = True, ND, 0, EGD
    d.joint_rot_all = torch.zeros((ND, CAP, 24, 3))
    d.root_pos_all = torch.zeros((ND, CAP, 3))
    d.ball_pos_all = torch.zeros((ND, CAP, 3))
    d.target_pos_all = torch.zeros((ND, CAP, 3))
    d.phase_all = torch.zeros((ND, CAP))
    d.swing_type_all = torch.zeros((ND, CAP), dtype=torch.int64)
    d.tar_action_all = torch.zeros((ND, CAP), dtype=torch.int64)
    d.distance_best_all, d.joint_rot_best_all, d.root_pos_best_all, d.ball_pos_best_all = [], [], [], []
    d.phase_best_all, d.swing_type_best_all, d.tar_action_best_all = [], [], []
    d._mvae_player = SimpleNamespace()
    captured = []
    d.render_one_result = lambda best_idx, eg_id: captured.append((best_idx, eg_id))
    gd = torch.Generator().manual_seed(seed)
    progress = torch.zeros(ND, dtype=torch.long)
    keys = ("joint_rot", "root_pos", "ball_pos", "phase", "swing_type", "tar_action", "progress", "reset", "distance")
    dual_in = {k: [] for k in keys}
    flagged_prev = torch.zeros(ND, dtype=torch.bool)
    done = False
    for step in range(steps + 1):
        if step > 0:
            progress[flagged_prev] = 0                # env_reset of the previous step's finished pairs, then the step counts one
            progress += 1
        reset = torch.zeros(ND, dtype=torch.long)
        distance = (torch.rand(ND, generator=gd) * 4.0).float()
        for p, (d0, d1) in schedule.get(step, {}).items():
            reset[2 * p] = reset[2 * p + 1] = 1
            distance[2 * p], distance[2 * p + 1] = d0, d1
        fr = dict(joint_rot=torch.randn(ND, 24, 3, generator=gd), root_pos=torch.randn(ND, 3, generator=gd),
                  ball_pos=torch.randn(ND, 3, generator=gd), phase=torch.rand(ND, generator=gd) * 6.0,
                  swing_type=torch.randint(-1, 4, (ND,), generator=gd), tar_action=torch.randint(0, 2, (ND,), generator=gd))
        d._joint_rot, d._root_pos, d._ball_pos, d._tar_action = fr["joint_rot"], fr["root_pos"], fr["ball_pos"], fr["tar_action"]
        d._mvae_player._phase_pred, d._mvae_player._swing_type_cycle = fr["phase"], fr["swing_type"]
        d.progress_buf, d.reset_buf, d._distance = progress.clone(), reset, distance
        for k, x in dict(fr, progress=progress, reset=reset, distance=distance).items():
            dual_in[k].append(x.numpy().copy())
        try:
            d.render_vis(init=(step == 0))
        except SystemExit:
            done = True
        flagged_prev = reset.bool()
    assert done
    out = {"dual_" + k: np.stack(x) for k, x in dual_in.items()}
    out["dual_best_distance"] = np.array([float(x) for x in d.distance_best_all], np.float32)
    out["dual_best_nframes"] = np.array([x.shape[1] for x in d.root_pos_best_all])
    for k in ("joint_rot", "root_pos", "ball_pos", "phase", "swing_type", "tar_action"):
        lst = getattr(d, k + "_best_all")
        out["dual_best_" + k] = np.concatenate([x.numpy() for x in lst], 1)    # entries concatenated along the frame axis
    return out, captured


# pair -> pair distance by step: same-step pairs, equal distances, a refused insertion while short, the capacity rally
SCHEDULE = {3: {0: 5.0, 1: 7.0}, 5: {0: 3.0}, 7: {1: 9.0, 2: 9.0}, 9: {0: 8.0}, 11: {3: 10.0}, 13: {0: 8.5, 2: 2.0}}
dual, captured = render_dual({s: {p: (0.25 * x, 0.75 * x) for p, x in sch.items()} for s, sch in SCHEDULE.items()}, 13, TD)
OUT.update(dual)
assert int(np.max(OUT["dual_progress"])) == CAP - 1     # one rally fills the buffer
OUT["dual_capacity"] = np.int64(CAP)
OUT["dual_num_eg"] = np.int64(EGD)
assert [i for i, _ in captured] == list(range(EGD))

np.savez_compressed(os.path.join(HERE, "v2p_eval.npz"), **OUT)
print("v2p_eval.npz", {k: v.shape for k, v in OUT.items()})

# ------------------------------------------------------------------ dual: NaN pair distances (v2p_eval_nonfinite.npz)
# A pair's distance is NaN once its root velocity is.  distance.max() is then NaN and torch.argmax (CPU) returns the first NaN; the
# insertion's max_dist > last is false for a NaN, so a NaN pair enters only an empty list, and a NaN in the list stops it growing.
# Scenario i is stored under "s{i}_" with the keys of the dual_ fixture above.
NAN, INF = float("nan"), float("inf")
NONFINITE = [
    # into the empty list: three NaN pairs (one player NaN, both, Inf - Inf) and a larger finite pair on one step -> the first NaN,
    # then a larger finite pair and another NaN pair are refused
    {2: {0: (1.0, 2.0), 1: (NAN, 1.0), 2: (INF, -INF), 3: (0.5, NAN)}, 5: {0: (50.0, 50.0)}, 8: {2: (NAN, NAN), 3: (9.0, 9.0)}},
    # into a short list: a NaN pair with a larger finite pair is refused, a larger finite pair alone enters
    {2: {0: (2.0, 3.0)}, 5: {1: (NAN, 0.0), 2: (40.0, 1.0)}, 8: {3: (6.0, 1.0)}, 10: {2: (0.0, NAN)}},
    # into the full list: a NaN pair beside a larger finite pair is refused, +Inf enters at the head, a NaN pair beside a +Inf pair is
    # refused, a larger finite pair enters behind the +Inf
    {1: {0: (1.0, 1.0)}, 2: {1: (2.0, 2.0)}, 3: {2: (3.0, 3.0)}, 5: {3: (NAN, 9.0), 0: (10.0, 10.0)}, 7: {1: (INF, 1.0)},
     9: {2: (NAN, NAN), 3: (INF, 0.0)}, 11: {0: (20.0, 20.0)}},
    # the first flag of the run is a lone NaN pair: the list holds it and refuses everything after
    {1: {3: (NAN, 2.0)}, 4: {0: (1.0, 1.0)}, 6: {1: (INF, INF)}, 9: {2: (NAN, 0.0)}},
]
NF = {}
for i, sch in enumerate(NONFINITE):
    out, captured = render_dual(sch, 17 + i, CAP - 1)
    assert [j for j, _ in captured] == list(range(EGD))
    NF.update({f"s{i}_" + k[5:]: v for k, v in out.items()})
NF["capacity"], NF["num_eg"], NF["scenarios"] = np.int64(CAP), np.int64(EGD), np.int64(len(NONFINITE))
assert np.isnan(NF["s0_best_distance"]).all() and len(NF["s0_best_distance"]) == 1 and len(NF["s2_best_distance"]) == EGD
np.savez_compressed(os.path.join(HERE, "v2p_eval_nonfinite.npz"), **NF)
print("v2p_eval_nonfinite.npz", {k: v.shape for k, v in NF.items()})
