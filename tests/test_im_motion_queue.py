"""CPU checks of the imitation test run's motion queue (cfg.env.b200_motion_queue): the restatement oracle/ref_port_motion_queue.py on
scripted done sequences with hand-computed assignments, the cfg refusals, the export's keys and per-motion fold from fake buffers,
and the C ABI of b200_im_motion_queue_t and the fields appended to b200_play_stats_t, b200_reset_masked_t and b200_im_motion_stats_t."""
import ctypes as C
import os
import subprocess
import types

import numpy as np
import pytest
import torch

import test_host
from oracle import ref_port_motion_queue as Q
from vid2player3d_b200 import abi, model_compiler, motion_lib, native
from vid2player3d_b200.configs import im_cfg
from vid2player3d_b200.tasks import humanoid_smpl_im_vis as V

ASSET = "mjcf/smpl_mesh_humanoid_amass_v1.xml"


def done(n, *envs):
    d = np.zeros(n, np.int64)
    d[list(envs)] = 1
    return d


def step(q, reset_buf):
    """one device step of the queue on sticky flags: the bookkeeping, the assignment, then the masked reset clears the flags"""
    q.bookkeeping(reset_buf)
    mask = q.assign(reset_buf)
    reset_buf[mask] = 0
    return mask


# ---------------------------------------------------------------------------------------------------------- the restatement
def test_envs_start_on_their_own_entries():
    q = Q.MotionQueue(4, 3, 2)
    assert q.entry.tolist() == [0, 1, 2, 3] and q.motion_ids.tolist() == [0, 1, 2, 0] and q.cursor == 4
    assert q.game_env.tolist() == [0, 1, 2, 3, -1, -1] and q.game_start_step.tolist() == [0, 0, 0, 0, -1, -1]


def test_ties_in_one_step_take_entries_in_env_order():
    q = Q.MotionQueue(4, 5, 2)                  # entries 0..9, envs on 0..3
    rb = done(4, 3, 1)
    assert step(q, rb).tolist() == [False, True, False, True]
    assert q.entry.tolist() == [0, 4, 2, 5] and q.motion_ids.tolist() == [0, 4, 2, 0] and q.cursor == 6
    assert q.game_env[4] == 1 and q.game_env[5] == 3 and q.game_start_step[4] == q.game_start_step[5] == 1
    assert q.games == 2 and not q.stop
    rb[[0, 2]] = 1
    step(q, rb)
    assert q.entry.tolist() == [6, 4, 7, 5] and q.cursor == 8 and q.game_start_step[6] == 2


def test_the_queue_runs_dry_mid_step():
    q = Q.MotionQueue(4, 3, 2)                  # entries 0..5: two left after the start
    rb = done(4, 0, 1, 2)
    mask = step(q, rb)
    assert mask.tolist() == [True, True, False, False]
    assert q.entry.tolist() == [4, 5, 2, 3] and q.motion_ids.tolist() == [1, 2, 2, 0] and q.cursor == 6
    assert q.idle.tolist() == [False, False, True, False] and rb.tolist() == [0, 0, 1, 0]   # the idle env stays done
    for _ in range(3):                          # counted once, never assigned again
        step(q, rb)
    assert q.games == 3 and q.cursor == 6 and q.idle.tolist() == [False, False, True, False]
    rb[[0, 1, 3]] = 1
    mask = step(q, rb)
    assert not mask.any() and q.games == 6 and q.stop


def test_more_rounds_repeat_every_motion_in_library_order():
    q = Q.MotionQueue(2, 3, 3)                  # entries 0..8 = motions 0 1 2 0 1 2 0 1 2
    rb = np.zeros(2, np.int64)
    order = []
    while not q.stop:
        rb[:] = 1                               # both envs finish every step
        m = step(q, rb)
        order += q.motion_ids[m].tolist()
    assert order == [2, 0, 1, 2, 0, 1, 2] and q.games == 9
    assert sorted(q.game_env.tolist()) == [0, 0, 0, 0, 0, 1, 1, 1, 1]
    assert q.game_env.tolist() == [0, 1, 0, 1, 0, 1, 0, 1, 0]


def test_a_game_that_ends_on_its_first_step_is_counted():
    q = Q.MotionQueue(1, 3, 1)
    rb = done(1, 0)
    for k in range(3):                          # the env finishes every step; each new game starts with a cleared done memory
        rb[0] = 1
        step(q, rb)
    assert q.games == 3 and q.stop and q.game_env.tolist() == [0, 0, 0] and q.game_start_step.tolist() == [0, 1, 2]


def test_nothing_changes_while_stopped():
    q = Q.MotionQueue(2, 2, 2)
    q.stop = True
    rb = done(2, 0, 1)
    before = (q.entry.copy(), q.cursor, q.games, q.step_count)
    assert not step(q, rb).any()
    assert (q.entry.tolist(), q.cursor, q.games, q.step_count) == (before[0].tolist(), *before[1:]) and not q.idle.any()


def test_the_meters_fold_each_game_into_its_entry():
    run = Q.QueueRun(2, 2, 2)                   # entries 0..3, envs on 0, 1
    B = 1
    z = lambda: (np.zeros((2, 4)), np.zeros((2, B, 3)), np.zeros((2, B, 3)))  # noqa: E731
    sub, bp, tp = z()
    rb, tb = np.zeros(2, np.int64), np.zeros(2, np.int64)
    seq = [(0.5, 0.25, ()), (1.0, 2.0, (1,)), (4.0, 8.0, (0,)), (16.0, 32.0, (0, 1))]
    masks = []
    for r0, r1, fin in seq:
        rb[list(fin)] = 1
        tb[0] = int(0 in fin and r0 == 4.0)      # env 0's first game ends in a fall
        masks.append(run.step(np.array([r0, r1]), sub, rb, tb, bp, tp).tolist())
        rb[masks[-1]] = 0
    assert masks == [[False, False], [False, True], [True, False], [False, False]]
    assert run.stats.counts.tolist() == [[1, 1], [1, 0], [1, 0], [1, 0]]
    assert run.stats.sums[:, 0].tolist() == [0.5 + 1.0 + 4.0, 0.25 + 2.0, 8.0 + 32.0, 16.0]
    assert run.stats.sums[:, 1].tolist() == [3, 2, 2, 1]
    assert run.queue.game_env.tolist() == [0, 1, 1, 0] and run.queue.game_start_step.tolist() == [0, 0, 2, 3]
    assert run.queue.stop and run.queue.games == 4
    counts, sums = run.per_motion()
    assert counts.tolist() == [[2, 1], [2, 0]] and sums[:, 0].tolist() == [5.5 + 40.0, 2.25 + 16.0]


def pose_game(run, frames):
    """one env (N = 1) with two bodies, both at (a, 0, 0) against targets at the origin, for each a of frames; the game ends on the
    last frame and the queue restarts the env on its next entry.  Per frame: body-position error |a|, root-relative and PA errors 0
    (no spread), velocity error |a - a'|, acceleration error |a - 2 a' + a''| over the game's own earlier frames"""
    rb, z = np.zeros(1, np.int64), np.zeros((1, 4))
    for k, a in enumerate(frames):
        rb[0] = int(k == len(frames) - 1)
        bp = np.zeros((1, 2, 3))
        bp[0, :, 0] = a
        mask = run.step(np.zeros(1), z, rb, np.zeros(1, np.int64), bp, np.zeros((1, 2, 3)))
        rb[mask] = 0
    return mask


def test_a_restarted_envs_first_frame_adds_no_velocity_or_acceleration_frame():
    run = Q.QueueRun(1, 2, 1, pose_threshold=5.0)       # env 0 plays entry 0, then entry 1
    assert pose_game(run, [1.0, 2.0, 4.0]).tolist() == [True]
    pose_game(run, [10.0, 11.0])
    ps = run.stats.pose_sums
    assert ps[:, 0].tolist() == [0.0, 0.0] and ps[:, 1].tolist() == [0.0, 0.0]
    assert ps[0, 2:].tolist() == [1.0 + 2.0, 1.0, 2, 1, 4.0]               # vel, acc, vel frames, acc frames, largest error
    assert ps[1, 2:].tolist() == [1.0, 0.0, 1, 0, 11.0]                    # no frame against entry 0's last two
    assert run.stats.success.tolist() == [1, 0] and run.stats.counts[:, 0].tolist() == [1, 1]
    assert run.stats.sums[:, 1].tolist() == [3, 2] and run.queue.stop


def test_a_nan_game_poisons_its_own_entry_only():
    run = Q.QueueRun(1, 2, 1, pose_threshold=0.5)
    pose_game(run, [0.1, 0.2, np.nan])                   # the NaN frame is the last: the history the restart empties holds it
    pose_game(run, [0.3, 0.4])
    ps = run.stats.pose_sums
    assert np.isnan(ps[0, [0, 1, 2, 3, 6]]).all() and ps[0, 4:6].tolist() == [2, 1]
    assert np.isfinite(ps[1]).all() and ps[1, 4:].tolist() == [1, 0, 0.4]
    np.testing.assert_allclose(ps[1, 2], 0.1, rtol=1e-12)
    assert run.stats.success.tolist() == [0, 1] and run.stats.counts[:, 0].tolist() == [1, 1]
    assert np.isnan(run.stats.sums[0, 6]) and np.isfinite(run.stats.sums[1]).all()


@pytest.mark.parametrize("nan_round", [0, 1])
def test_a_nan_in_either_round_makes_the_motions_largest_error_nan(nan_round):
    run = Q.QueueRun(1, 2, 2, pose_threshold=0.5)       # entries 0..3: motions 0 1 0 1, all on env 0
    for q in range(4):
        pose_game(run, [0.1 * (q + 1), np.nan if q == 2 * nan_round else 0.05])
    ps, success = run.per_motion_pose()
    assert np.isnan(ps[0, 6]) and ps[1, 6] == 0.4 and success.tolist() == [1, 2]
    assert ps[:, 4].tolist() == [2, 2] and np.isnan(ps[0, 2]) and np.isfinite(ps[1]).all()
    counts, _ = run.per_motion()
    assert counts[:, 0].tolist() == [2, 2]


def test_queue_fold_of_the_largest_error_with_nan_inf_and_ties():
    run = Q.QueueRun(1, 3, 3, pose_threshold=0.5)       # only the fold is used: R = 3, M = 3
    col = np.array([np.inf, -np.inf, -np.inf,            # round 0
                    1.0, 2.0, -np.inf,                   # round 1
                    np.nan, 2.0, -np.inf])               # round 2
    rows = np.zeros((9, 7))
    rows[:, 0], rows[:, 6] = np.arange(9.0), col
    for f in (V.queue_fold(rows, 3, 3, max_col=6), run.fold(rows, max_col=6)):
        assert np.isnan(f[0, 6]) and f[1, 6] == 2.0 and f[2, 6] == -np.inf
        assert f[:, 0].tolist() == [0.0 + 3.0 + 6.0, 1.0 + 4.0 + 7.0, 2.0 + 5.0 + 8.0]
    rows[6, 6] = 0.5                                     # no NaN: +Inf wins
    assert V.queue_fold(rows, 3, 3, max_col=6)[0, 6] == run.fold(rows, max_col=6)[0, 6] == np.inf
    rows[0, 6] = np.nan                                  # a NaN in the first round survives the later ones
    assert np.isnan(V.queue_fold(rows, 3, 3, max_col=6)[0, 6]) and np.isnan(run.fold(rows, max_col=6)[0, 6])


# ---------------------------------------------------------------------------------------------------------- cfg refusals
def qcfg(N=4, flat=None, test=True, **over):
    cfg = im_cfg(N, flat, **dict(dict(b200_motion_queue=True), **over))
    cfg["args"] = types.SimpleNamespace(test=test)
    return cfg


@pytest.mark.parametrize("R", [0, -1, 1.5, "2", True, None])
def test_rounds_must_be_an_int_of_at_least_one(R):
    with pytest.raises(ValueError, match="b200_motion_queue_repeats must be an int >= 1"):
        V.motion_queue_rounds(qcfg(b200_motion_queue_repeats=R))


def test_rounds_default_and_off():
    assert V.motion_queue_rounds(qcfg()) == 1 and V.motion_queue_rounds(qcfg(b200_motion_queue_repeats=np.int64(3))) == 3
    assert V.motion_queue_rounds(qcfg(b200_motion_queue=False, b200_motion_queue_repeats=0)) is None


def test_several_assets_and_torch_transforms_and_other_state_inits_are_refused():
    with pytest.raises(ValueError, match="motion_assets"):
        V.motion_queue_rounds(qcfg(motion_assets=[ASSET] * 2))
    xf = dict(mask_joints=dict(joints=["L_Knee"]))
    with pytest.raises(ValueError, match="set b200_device_transforms"):
        V.motion_queue_rounds(qcfg(transform_specs=xf))
    assert V.motion_queue_rounds(qcfg(transform_specs=xf, b200_device_transforms=True)) == 1
    with pytest.raises(ValueError, match="needs args.test or stateInit: Start, got 'Random'"):
        V.motion_queue_rounds(qcfg(test=False, stateInit="Random"))
    assert V.motion_queue_rounds(qcfg(test=False, stateInit="Start")) == 1


@pytest.fixture(scope="module")
def lib3(tmp_path_factory):
    model = model_compiler.load_compiled("smpl_mesh_humanoid_amass_v1")
    path = str(tmp_path_factory.mktemp("queue") / "three.npz")
    motion_lib.synthetic(model, num_motions=3, num_frames=20, seed=2).save(path)
    return path


def test_the_task_refuses_before_allocating(lib3):
    """more envs than queued games, and the cfg refusals, before anything reaches the device (none is needed to see them)"""
    from vid2player3d_b200.tasks import HumanoidSMPLIMVis
    with pytest.raises(ValueError, match="7 envs for a queue of 3 motions x 2 rounds"):
        HumanoidSMPLIMVis(qcfg(7, None, motion_file=lib3, b200_motion_queue_repeats=2), None, 1, "cuda", 0, True)
    with pytest.raises(ValueError, match="b200_motion_queue_repeats"):
        HumanoidSMPLIMVis(qcfg(4, None, motion_file=lib3, b200_motion_queue_repeats=0), None, 1, "cuda", 0, True)
    with pytest.raises(ValueError, match="motion_assets"):
        HumanoidSMPLIMVis(qcfg(4, None, motion_file=lib3, motion_assets=[ASSET] * 3), None, 1, "cuda", 0, True)


# ---------------------------------------------------------------------------------------------------------- the export
def test_queue_fold_adds_rounds_in_order_and_takes_the_largest_error():
    rows = np.arange(12, dtype=np.float64).reshape(6, 2)      # R = 3, M = 2
    assert V.queue_fold(rows, 3, 2).tolist() == [[0 + 4 + 8, 1 + 5 + 9], [2 + 6 + 10, 3 + 7 + 11]]
    ps = np.zeros((4, 7))
    ps[:, 0], ps[:, 6] = [1.0, 2.0, 3.0, 4.0], [0.5, np.nan, 0.25, 0.75]
    f = V.queue_fold(ps, 2, 2, max_col=6)
    assert f[:, 0].tolist() == [4.0, 6.0] and f[0, 6] == 0.5 and np.isnan(f[1, 6])
    assert V.queue_fold(np.array([1, 0, 1, 1]), 2, 2).tolist() == [2, 1]


def fake_task(tmp_path, N=2, M=3, R=2, pose=False):
    """a HumanoidSMPLIMVis with host buffers in place of the device ones: what export_motion_stats reads"""
    t = V.HumanoidSMPLIMVis.__new__(V.HumanoidSMPLIMVis)
    Qn = M * R
    t.cfg = dict(env=dict(b200_motion_stats_file=str(tmp_path / "q.npz")))
    t.num_envs, t.device, t.dt, t._test_motion_file = N, "cpu", 1 / 30, None
    t._queue_rounds, t._pose_threshold = R, (0.5 if pose else None)
    t._motion_lib = types.SimpleNamespace(num_motions=lambda: M)
    t._reset_ref_motion_ids = torch.tensor([2, 1][:N])           # moved on by the queue
    counts = torch.tensor([[1, 0], [1, 1], [1, 0], [1, 0], [0, 0], [1, 0]])
    sums = torch.arange(Qn * 7, dtype=torch.float64).view(Qn, 7)
    sums[4] = 0.0
    t._ms = dict(counts=counts, sums=sums)
    if pose:
        t._ms.update(pose_sums=torch.ones(Qn, 7, dtype=torch.float64), success=torch.tensor([1, 0, 1, 1, 0, 1]))
    t._q = dict(game_env=torch.tensor([0, 1, 1, 0, 1, 0]), game_start_step=torch.tensor([0, 0, 5, 9, 12, 14]))
    return t


def test_export_keeps_the_keys_and_shapes_and_adds_the_queue(tmp_path, capsys):
    t = fake_task(tmp_path)
    got = dict(np.load(t.export_motion_stats()))
    assert set(got) == {"games", "falls", "reward_sum", "steps", "sub_reward_sum", "body_pos_err_sum", "env_motion_ids", "test_motion_file",
                        "game_env", "game_start_step", "unfinished"}
    assert got["games"].tolist() == [2, 1, 2] and got["falls"].tolist() == [0, 1, 0]
    sums = np.arange(42, dtype=np.float64).reshape(6, 7)
    sums[4] = 0.0
    assert got["reward_sum"].tolist() == (sums[:3, 0] + sums[3:, 0]).tolist() and got["sub_reward_sum"].shape == (3, 4)
    assert got["steps"].dtype == np.int64 and got["env_motion_ids"].tolist() == [0, 1]    # the initial assignment
    assert got["game_env"].tolist() == [[0, 1, 1], [0, 1, 0]] and got["game_start_step"].shape == (2, 3)
    assert got["unfinished"].tolist() == [4]
    assert "motions evaluated: 3 of 3" in capsys.readouterr().out


def test_export_folds_the_pose_metrics(tmp_path, capsys):
    got = dict(np.load(fake_task(tmp_path, pose=True).export_motion_stats()))
    assert got["success"].tolist() == [2, 0, 2] and got["mpjpe_l_sum"].tolist() == [2.0, 2.0, 2.0]
    assert got["max_body_pos_err"].tolist() == [1.0, 1.0, 1.0] and got["vel_frames"].dtype == np.int64
    assert "success rate:" in capsys.readouterr().out


# ---------------------------------------------------------------------------------------------------------- the C ABI
LAYOUTS = [("b200_im_motion_queue_t", "ImMotionQueue"), ("b200_play_stats_t", "PlayStats"), ("b200_reset_masked_t", "ResetMasked")]


def test_descriptor_layouts_match_the_header(tmp_path):
    names = {C.c_float: "float", C.c_int64: "int64_t", C.c_int32: "int32_t", C.c_double: "double", C.c_uint8: "uint8_t"}
    lines, want = [], []
    for ctype, cls in LAYOUTS:
        S = getattr(abi, cls)
        lines.append(f'printf("{ctype} %zu\\n", sizeof({ctype}));')
        want.append(f"{ctype} {C.sizeof(S)}")
        for f, ct in S._fields_:
            lines.append(f'printf("{ctype}.{f} %zu %zu\\n", offsetof({ctype}, {f}), sizeof((({ctype}*)0)->{f}));')
            want.append(f"{ctype}.{f} {getattr(S, f).offset} {getattr(S, f).size}")
            if issubclass(ct, C.c_void_p) and ct is not C.c_void_p:
                lines.append(f'printf("{ctype}.{f} %d\\n", __builtin_types_compatible_p(__typeof__(*(({ctype}*)0)->{f}), '
                             f'{names[ct.pointee]}));')
                want.append(f"{ctype}.{f} 1")
    S, ctype = abi.ImMotionQueueStats, "b200_im_motion_queue_stats_t"     # the meters' descriptor as its first member, then env_entry
    lines.append(f'printf("{ctype} %zu %zu\\n", sizeof({ctype}), offsetof({ctype}, env_entry));')
    want.append(f"{ctype} {C.sizeof(S)} {S.env_entry.offset}")
    for f, _ in abi.ImMotionStats._fields_:
        lines.append(f'printf("{ctype}.{f} %zu\\n", offsetof({ctype}, meters.{f}));')
        want.append(f"{ctype}.{f} {getattr(S, f).offset}")
    src, exe = tmp_path / "layout.c", tmp_path / "layout"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "b200env.h"\nint main(void) {\n' + "\n".join(lines) + "\nreturn 0;\n}\n")
    subprocess.check_call(["gcc", "-w", "-I", os.path.join(test_host.ROOT, "include"), str(src), "-o", str(exe)])
    assert subprocess.check_output([str(exe)], text=True).splitlines() == want
    assert S.env_entry.offset == C.sizeof(abi.ImMotionStats) == 168
    assert "#define B200_ABI_VERSION 11" in open(os.path.join(test_host.ROOT, "include", "b200env.h")).read()


def test_signatures_and_descriptor_sizes():
    assert test_host.signature_mismatches(abi.SIGNATURES, test_host.ENV_HEADERS) == []
    L = native.lib()
    assert L.b200env_im_motion_queue_desc_size() == C.sizeof(abi.ImMotionQueue)
    assert L.b200env_play_stats_desc_size() == C.sizeof(abi.PlayStats)
    assert L.b200env_reset_masked_desc_size() == C.sizeof(abi.ResetMasked)
    assert L.b200env_im_motion_queue_stats_desc_size() == C.sizeof(abi.ImMotionQueueStats)


@pytest.mark.parametrize("cls", ["ImMotionQueue", "PlayStats", "ImMotionQueueStats"])
def test_binding_refuses_a_library_of_another_descriptor_size(monkeypatch, cls):
    native.lib()
    S = getattr(abi, cls)
    monkeypatch.setattr(abi, cls, type(cls, (C.Structure,), {"_fields_": S._fields_[:-1]}))
    monkeypatch.setattr(native, "_lib", None)
    with pytest.raises(RuntimeError, match=f"{cls} descriptor.*rebuild"):
        native.lib()


SCALARS = dict(n=4, num_motions=3, queue_len=6, shape_dim=11)


def fake_queue(**over):
    d = abi.ImMotionQueue(**dict(SCALARS, **{k: v for k, v in over.items() if k in SCALARS}))
    for name, ct in abi.ImMotionQueue._fields_:
        if issubclass(ct, C.c_void_p):
            setattr(d, name, over.get(name, 0x10000))
    return d


@pytest.mark.parametrize("over, rc, msg", [
    (dict(n=0), -2, "n, num_motions and queue_len must be positive"), (dict(num_motions=0), -2, "n, num_motions and queue_len"),
    (dict(queue_len=0), -2, "n, num_motions and queue_len"), (dict(shape_dim=33), -2, "shape_dim must lie in [0, 32]"),
    (dict(shape_dim=-1), -2, "shape_dim"), (dict(cursor=None), -1, "null argument"), (dict(step=None), -1, "null argument"),
    (dict(mask=None), -1, "null argument")])
def test_queue_launch_refusals_before_any_launch(over, rc, msg):
    """refused on fake device addresses: the checks come before the launch"""
    assert native.lib().b200env_im_motion_queue(C.byref(fake_queue(**over)), None) == rc
    assert msg in native.lib().b200env_last_error().decode()


def test_play_stats_refuses_a_negative_queue():
    d = abi.PlayStats(n=4, max_log=2, n_games=1, queue_games=-1)
    for name, ct in abi.PlayStats._fields_:
        if issubclass(ct, C.c_void_p):
            setattr(d, name, 0x10000)
    assert native.lib().b200env_play_stats(C.byref(d), None) == -2
    assert "queue_games must not be negative" in native.lib().b200env_last_error().decode()


def test_queue_meters_need_the_entries_and_not_the_env_lists():
    S = abi.ImMotionQueueStats
    d = S(n=4, num_motions=3, num_bodies=24, num_lib_bodies=24)
    for name, ct in S._fields_:
        if issubclass(ct, C.c_void_p) and name not in S._nullable_:
            setattr(d, name, 0x10000)
    d.env_entry = None
    assert native.lib().b200env_im_motion_queue_stats(C.byref(d), None) == -1
    d.env_entry, d.num_motions = 0x10000, 0
    assert native.lib().b200env_im_motion_queue_stats(C.byref(d), None) == -2        # checked past the NULL env lists
    assert "b200env_im_motion_queue_stats: n and num_motions must be positive" in native.lib().b200env_last_error().decode()


def test_fill_takes_the_queue_fields():
    S = abi.ImMotionQueue
    ptrs = {f: torch.zeros(2, dtype={abi.F32P: torch.float32, abi.I64P: torch.int64, abi.U8P: torch.uint8,
                                     abi.I32P: torch.int32}[ct])
            for f, ct in S._fields_ if issubclass(ct, C.c_void_p)}

    class OnDevice:
        def __init__(self, t):
            self.t, self.dtype = t, t.dtype

        def is_contiguous(self):
            return True

        def get_device(self):
            return 0

        def data_ptr(self):
            return self.t.data_ptr()
    d = native.fill(S, SCALARS, {f: OnDevice(t) for f, t in ptrs.items()})
    assert all(getattr(d, f).value == t.data_ptr() for f, t in ptrs.items()) and (d.n, d.queue_len, d.shape_dim) == (4, 6, 11)
    with pytest.raises(ValueError, match=r"ImMotionQueue\.idle: torch\.int64"):
        native.fill(S, SCALARS, dict({f: OnDevice(t) for f, t in ptrs.items()}, idle=OnDevice(torch.zeros(2, dtype=torch.long))))
    r = native.fill(abi.ResetMasked, dict(sample_time=0, truncate=0.0, ref_prob=1.0, num_frames=48, first_frame=-8, dt=0.1, seed=1), {
        k: OnDevice(torch.zeros(2, dtype=dt)) for k, dt in (("mask", torch.bool), ("counter", torch.long), ("reset_times", torch.float),
                                                         ("context_feat", torch.float), ("context_mask", torch.bool), ("work", torch.int32))})
    assert r.step.value is None and r.context_length == 0                       # the parent's window
