"""CPU checks of the rally results of the dual test run (cfg.env.b200_rally_stats): the integer restatement oracle/ref_port_rally_stats.py
against the reference's dual reset rule it is composed from (the cr_* arrays of tests/golden/v2p_dual.npz), scripted rallies with
hand-computed counts, its invariants on random sequences, the cfg refusal, the file and its summary line, and the C ABI of
b200v2p_rstats_t."""
import ctypes as C
import datetime
import os
import subprocess

import numpy as np
import pytest
import torch

import test_host
from conftest import golden
from helpers import v2p_cfg, v2p_dual_cfg
from oracle import ref_port_rally_stats as RS
from oracle import ref_port_v2p as V
from vid2player3d_b200 import abi, native
from vid2player3d_b200.tasks import mvae_controller_vis as MV

CAUSE = {c: j for j, c in enumerate(RS.CAUSES)}


# ------------------------------------------------------------------------------------------------ the reference's rule
def test_events_rebuild_the_reference_reset_rule():
    """reset, reaction and recovery of dual_controller_reset on the golden inputs, rebuilt from the per-player events"""
    g = golden("v2p_dual.npz")
    args = [g["cr_" + k] for k in ("tar_action", "has_contact", "has_bounce", "ball_pos", "root_pos", "root_vel", "bounce_in", "distance")]
    ref = V.dual_controller_reset(*args, g["crreset_buf"])
    ev = RS.events(g["cr_tar_action"], g["cr_has_contact"], g["cr_has_bounce"], g["cr_ball_pos"], g["cr_root_pos"], g["cr_bounce_in"])
    got = RS.reset_flags(ev, g["crreset_buf"])
    for a, b, w in zip(got, ref[:3], ("reset", "reaction", "recovery")):
        np.testing.assert_array_equal(a, b, w)
    np.testing.assert_array_equal(got[0], g["cr_out_reset"])
    np.testing.assert_array_equal(got[1], g["cr_out_reaction"])
    np.testing.assert_array_equal(got[2], g["cr_out_recovery"])
    # the golden inputs reach every kind of event
    for k in ("hit", "behind", "out"):
        assert ev[k].any(), k
    assert (ev["rec"] == (ev["hit"] | ev["behind"] | ev["double_bounce"])).all()


# ------------------------------------------------------------------------------------------------ scripted rallies
# one player's situation at a step: (tar_action, has_contact, has_bounce, bounce_in, ball ahead / behind, ball height, swing_type_cycle)
TOKENS = {
    "wait": (1, 0, 0, 0, 5.0, 1.0, 0),      # to hit, the ball still coming
    "hit": (1, 1, 0, 0, 5.0, 1.0, 2),       # to hit, contact (a backhand)
    "fh": (1, 1, 0, 0, 5.0, 1.0, 1),        # to hit, contact, a forehand
    "behind": (1, 0, 0, 0, -1.5, 1.0, 0),   # to hit, the ball passed it
    "double": (1, 0, 1, 0, 5.0, 0.01, 0),   # to hit, the ball bounced and is at the ground again
    "rec": (0, 0, 0, 0, 5.0, 1.0, 0),       # recovering, its ball in the air
    "in": (0, 0, 1, 1, 5.0, 1.0, 0),        # recovering, its ball bounced in
    "out": (0, 0, 1, 0, 5.0, 1.0, 0),       # recovering, its ball bounced out
}
IDLE = ("rec", "rec")


def state(pairs, progress):
    """the launch inputs of pairs [(token of player 0, token of player 1), ...] with progress_buf [pairs]"""
    rows = np.array([TOKENS[t] for p in pairs for t in p], np.float64)
    n = len(rows)
    root = np.zeros((n, 3), np.float32)
    root[:, 1] = -12.0
    ball = np.stack([np.zeros(n), root[:, 1] + rows[:, 4], rows[:, 5]], -1).astype(np.float32)
    return dict(tar_action=rows[:, 0].astype(np.int64), has_contact=rows[:, 1] > 0, has_bounce=rows[:, 2] > 0, bounce_in=rows[:, 3] > 0,
                ball_pos=ball, root_pos=root, swing_type_cycle=rows[:, 6].astype(np.int64),
                progress_buf=np.repeat(np.asarray(progress, np.int64), 2))


def rally(shots, last):
    """`shots` alternate hits (player 0 first, the serve from player 1), then `last` (the pair's last step)"""
    steps = [("wait", "rec")]
    for s in range(shots):
        steps += [("hit", "rec") if s % 2 == 0 else ("rec", "hit"), ("rec", "wait") if s % 2 == 0 else ("wait", "rec")]
    return steps + [last]


SCRIPTS = {   # name -> (steps of one pair, reset before step k (progress back to 1) for k in resets)
    "served out": ([("wait", "rec"), ("wait", "out")], ()),
    "three shots, lost behind": ([("wait", "rec"), ("hit", "rec"), ("rec", "wait"), ("rec", "fh"), ("wait", "rec"), ("hit", "rec"),
                                  ("rec", "behind")], ()),
    "double bounce": ([("wait", "rec"), ("double", "rec")], ()),
    "both end one step": ([("wait", "rec"), ("hit", "rec"), ("rec", "wait"), ("out", "behind")], ()),
    "63 shots": (rally(63, ("behind", "rec") if 63 % 2 == 0 else ("rec", "behind")), ()),
    "64 shots": (rally(64, ("behind", "rec")), ()),
    "65 shots": (rally(65, ("rec", "behind")), ()),
    "open at export": ([("wait", "rec"), ("hit", "rec"), ("rec", "wait"), ("rec", "hit"), ("wait", "in")], ()),
    "stepped on unreset": ([("wait", "rec"), ("behind", "rec"), ("behind", "rec"), ("hit", "out"), ("double", "rec")], ()),
    "reset and a second rally": ([("wait", "rec"), ("wait", "out"), ("wait", "rec"), ("hit", "rec"), ("rec", "behind")], (2,)),
}


def z():
    return dict(rallies=0, shots_sum=0, frames_sum=0, hist={}, ends=np.zeros((2, 3), np.int64), player=np.zeros((2, 3), np.int64),
                open=False, pair_hits=[0, 0])


def expected(name):
    """the hand-computed counts of each script"""
    w = z()
    E = lambda p, c: w["ends"].__setitem__((p, CAUSE[c]), 1)  # noqa: E731
    if name == "served out":                            # the server's ball out: 0 shots, ended by the server (player 1)
        w.update(rallies=1, frames_sum=2, hist={0: 1})
        E(1, "out")
    elif name == "three shots, lost behind":
        w.update(rallies=1, shots_sum=3, frames_sum=7, hist={3: 1}, pair_hits=[2, 1])
        w["player"][:] = [[2, 2, 0], [2, 1, 1]]
        E(1, "behind")
    elif name == "double bounce":
        w.update(rallies=1, frames_sum=2, hist={0: 1})
        w["player"][0] = [1, 0, 0]
        E(0, "double_bounce")
    elif name == "both end one step":                   # player 0's return lands out as player 1 lets the ball pass
        w.update(rallies=1, shots_sum=1, frames_sum=4, hist={1: 1}, pair_hits=[1, 0])
        w["player"][:] = [[1, 1, 0], [1, 0, 0]]
        E(0, "out")
        E(1, "behind")
    elif name.endswith(" shots"):
        s = int(name.split()[0])
        h0, h1 = (s + 1) // 2, s // 2
        loser = 0 if s % 2 == 0 else 1
        w.update(rallies=1, shots_sum=s, frames_sum=2 * s + 2, hist={min(s, 64): 1}, pair_hits=[h0, h1])
        w["player"][:] = [[h0, h0, 0], [h1, h1, 0]]
        w["player"][loser, 0] += 1
        E(loser, "behind")
    elif name == "open at export":
        w.update(open=True, pair_hits=[1, 1])
        w["player"][:] = [[1, 1, 0], [1, 1, 0]]
    elif name == "stepped on unreset":                  # the ending counts once; later steps of the finished pair count nothing
        w.update(rallies=1, frames_sum=2, hist={0: 1})
        w["player"][0] = [1, 0, 0]
        E(0, "behind")
    elif name == "reset and a second rally":
        w.update(rallies=2, shots_sum=1, frames_sum=2 + 3, hist={0: 1, 1: 1}, pair_hits=[1, 0])
        w["player"][:] = [[1, 1, 0], [1, 0, 0]]
        E(1, "out")
        E(1, "behind")
    return w


def progress_of(steps, resets):
    p, out = 0, []
    for k in range(len(steps)):
        p = 1 if k in resets else p + 1
        out.append(p)
    return out


def run_scripts(names, launch):
    """all scripts side by side, one pair each (shorter ones padded with steps that carry no event), through `launch(state)`"""
    T = max(len(SCRIPTS[s][0]) for s in names)
    cols = []
    for s in names:
        steps, resets = SCRIPTS[s]
        prog = progress_of(steps, resets)
        cols.append([(steps[k], prog[k]) if k < len(steps) else (IDLE, prog[-1] + k - len(steps) + 1) for k in range(T)])
    for k in range(T):
        launch(state([c[k][0] for c in cols], [c[k][1] for c in cols]))


def check_script_counts(names, a):
    """a: the arrays of one run of run_scripts (pair_open, pair_hits, totals, ends, player, shots_hist); one pair per script"""
    tot = dict(rallies=0, shots_sum=0, frames_sum=0)
    hist, ends, player = np.zeros(RS.HIST, np.int64), np.zeros((2, 3), np.int64), np.zeros((2, 3), np.int64)
    for k, s in enumerate(names):
        w = expected(s)
        assert bool(a["pair_open"][k]) == w["open"], s
        assert a["pair_hits"][k].tolist() == w["pair_hits"], s
        for key in tot:
            tot[key] += w[key]
        for b, c in w["hist"].items():
            hist[b] += c
        ends += w["ends"]
        player += w["player"]
    assert a["totals"].tolist() == [tot["rallies"], tot["shots_sum"], tot["frames_sum"]]
    np.testing.assert_array_equal(a["shots_hist"], hist)
    np.testing.assert_array_equal(a["ends"], ends)
    np.testing.assert_array_equal(a["player"], player)


@pytest.mark.parametrize("name", list(SCRIPTS))
def test_scripted_rally_counts(name):
    st = RS.RallyStats(2)
    run_scripts([name], st.step)
    check_script_counts([name], st.arrays())


def test_all_scripts_side_by_side():
    names = list(SCRIPTS)
    st = RS.RallyStats(2 * len(names))
    run_scripts(names, st.step)
    check_script_counts(names, st.arrays())


# ------------------------------------------------------------------------------------------------ invariants
def random_state(rng, n, progress):
    return dict(tar_action=rng.integers(0, 2, n), has_contact=rng.random(n) < 0.3, has_bounce=rng.random(n) < 0.3,
                bounce_in=rng.random(n) < 0.9, ball_pos=np.stack([np.zeros(n), rng.normal(0, 1, n), rng.uniform(0, 0.4, n)], -1).astype(np.float32),
                root_pos=np.stack([np.zeros(n), rng.normal(-1.5, 1, n), np.ones(n)], -1).astype(np.float32),
                swing_type_cycle=rng.integers(-1, 4, n), progress_buf=np.repeat(progress, 2))


def random_run(rng, n, steps, on_step):
    """a test loop on random flags: pairs whose rally ended are reset (progress 1) at the next step with probability 1/2, as the
    mask-driven reset does from reset_buf; the rest step on"""
    progress = np.zeros(n // 2, np.int64)      # the first step opens every pair, as after the first reset
    ended = np.zeros(n // 2, bool)
    for _ in range(steps):
        reset = ended & (rng.random(n // 2) < 0.5)
        progress = np.where(reset, 0, progress) + 1
        ended &= ~reset
        s = random_state(rng, n, progress)
        ended |= on_step(s)


def check_invariants(a):
    pl, ends = a["player"], a["ends"]
    for w in range(2):
        assert pl[w, 0] == pl[w, 1] + ends[w, CAUSE["behind"]] + ends[w, CAUSE["double_bounce"]]
    assert pl[:, 1].sum() == a["totals"][1] + a["pair_hits"][a["pair_open"]].sum()
    assert a["shots_hist"].sum() == a["totals"][0]
    assert (pl[:, 2] <= pl[:, 1]).all()


@pytest.mark.parametrize("n", [2, 34, 200])
def test_invariants_on_random_sequences(n):
    rng = np.random.default_rng(n)
    st = RS.RallyStats(n)

    def step(s):
        end = st.step(s)
        check_invariants(st.arrays())
        return end
    random_run(rng, n, 300, step)
    assert st.totals[0] > n // 2 and st.player[:, 1].sum() > 0 and (st.ends > 0).all()


# ------------------------------------------------------------------------------------------------ cfg, file, export
def test_key_is_refused_on_the_single_player_task_before_anything_is_allocated(monkeypatch):
    from vid2player3d_b200.tasks import MVAEControllerVis
    cfg = v2p_cfg(4)
    cfg["env"]["b200_rally_stats"] = True
    monkeypatch.setattr(torch, "zeros", None)           # an allocation would fail with another error
    with pytest.raises(ValueError, match="rallies of MVAEControllerVisDual.*b200_ball_stats"):
        MVAEControllerVis(cfg, None, 1, "cuda", 0, True)


def test_key_is_accepted_in_dual_mode_and_opt_in():
    cfg = v2p_dual_cfg(4)
    cfg["env"]["b200_rally_stats"] = True
    MV._check_rally_stats_cfg(cfg, dual=True)
    MV._check_rally_stats_cfg(v2p_cfg(4), dual=False)


def test_file_path_rule():
    assert MV.rally_stats_path({"b200_rally_stats_file": "runs/rallies.npz"}) == "runs/rallies.npz"
    now = datetime.datetime(2026, 1, 2, 3, 4, 5)
    assert MV.rally_stats_path({}, now) == os.path.join("out", "rally_stats", "rally_stats_2026-01-02-03:04:05.npz")
    assert MV.rally_stats_path({"b200_rally_stats_file": ""}, now) == MV.rally_stats_path({}, now)
    assert MV.ball_stats_path({}, now) == os.path.join("out", "ball_stats", "ball_stats_2026-01-02-03:04:05.npz")


def _fake_task(tmp_path, r, v2p, path="rallies.npz"):
    t = MV.MVAEControllerVisDual.__new__(MV.MVAEControllerVisDual)
    t.cfg = dict(env=dict(b200_rally_stats_file=str(tmp_path / path)))
    t.cfg_v2p = v2p
    t.num_envs, t._test_steps = 2 * len(r["pair_open"]), 77
    t._rstats = {k: torch.tensor(v) for k, v in r.items()}
    return t


def fixed_arrays():
    hist = np.zeros(RS.HIST, np.int64)
    hist[[0, 3, 64]] = [1, 2, 1]
    return dict(pair_open=np.array([True, False, True]), pair_hits=np.array([[2, 1], [5, 5], [0, 1]], np.int64),
                totals=np.array([4, 76, 900], np.int64), ends=np.array([[1, 0, 1], [2, 1, 0]], np.int64),
                player=np.array([[40, 38, 20], [41, 39, 9]], np.int64), shots_hist=hist)


def test_export_arrays_dtypes_and_summary_line(tmp_path, capsys):
    r = fixed_arrays()
    t = _fake_task(tmp_path, r, dict(dual_mode="different", player=["federer", "djokovic"]), path="sub/dir/rallies.npz")
    path = t.export_rally_stats()
    assert path == str(tmp_path / "sub/dir/rallies.npz")
    a = np.load(path)
    assert sorted(a.files) == sorted(["rallies", "shots_sum", "frames_sum", "shots_hist", "ends", "end_causes", "faced", "hits",
                                      "forehands", "open_rallies", "open_hits", "players", "num_envs", "test_steps"])
    for k in a.files:
        if k not in ("end_causes", "players"):
            assert a[k].dtype == np.int64, k
    assert (int(a["rallies"]), int(a["shots_sum"]), int(a["frames_sum"])) == (4, 76, 900)
    np.testing.assert_array_equal(a["shots_hist"], r["shots_hist"])
    np.testing.assert_array_equal(a["ends"], r["ends"])
    assert a["end_causes"].tolist() == ["behind", "double_bounce", "out"]
    assert a["faced"].tolist() == [40, 41] and a["hits"].tolist() == [38, 39] and a["forehands"].tolist() == [20, 9]
    assert int(a["open_rallies"]) == 2 and a["open_hits"].tolist() == [[2, 1], [0, 1]]
    assert a["players"].tolist() == ["federer", "djokovic"] and int(a["num_envs"]) == 6 and int(a["test_steps"]) == 77
    out = capsys.readouterr().out.splitlines()
    assert out[0] == ("rallies: 4  shots per rally: 19.00  player 0 (federer): hit rate 0.9500, ended behind 0.2500 double_bounce "
                      "0.0000 out 0.2500  player 1 (djokovic): hit rate 0.9512, ended behind 0.5000 double_bounce 0.2500 out 0.0000")
    assert out[1] == f"============ rally statistics written to {path} ============"


def test_summary_without_rallies_and_one_player_twice(tmp_path, capsys):
    r = dict(pair_open=np.zeros(1, bool), pair_hits=np.zeros((1, 2), np.int64), totals=np.zeros(3, np.int64),
             ends=np.zeros((2, 3), np.int64), player=np.zeros((2, 3), np.int64), shots_hist=np.zeros(RS.HIST, np.int64))
    a = np.load(_fake_task(tmp_path, r, dict(dual_mode=True, player="nadal")).export_rally_stats())
    assert a["players"].tolist() == ["nadal", "nadal"] and int(a["open_rallies"]) == 0 and a["open_hits"].shape == (0, 2)
    assert capsys.readouterr().out.splitlines()[0] == ("rallies: 0  shots per rally: nan  player 0 (nadal): hit rate nan, ended "
                                                      "behind nan double_bounce nan out nan  player 1 (nadal): hit rate nan, ended "
                                                      "behind nan double_bounce nan out nan")


# ------------------------------------------------------------------------------------------------ the C ABI
def test_descriptor_layout_matches_the_header(tmp_path):
    """b200v2p_rstats_t field by field with its pointee types, and the histogram width and cause count of the header"""
    from test_ball_stats import _layout
    lines, want = _layout("b200v2p_rstats_t", abi.V2PRallyStats)
    lines.append('printf("%d %d\\n", B200V2P_RSTATS_HIST, B200V2P_RSTATS_CAUSES);')
    want.append(f"{abi.RSTATS_HIST} {len(abi.RSTATS_CAUSES)}")
    src, exe = tmp_path / "layout.c", tmp_path / "layout"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "b200env_v2p.h"\nint main(void) {\n' + "\n".join(lines) +
                   "\nreturn 0;\n}\n")
    subprocess.check_call(["gcc", "-w", "-I", os.path.join(test_host.ROOT, "include"), str(src), "-o", str(exe)])
    assert subprocess.check_output([str(exe)], text=True).splitlines() == want
    assert abi.RSTATS_HIST == RS.HIST and abi.RSTATS_CAUSES == RS.CAUSES and abi.RSTATS_PLAYER == RS.PLAYER
    assert abi.V2PRallyStats._nullable_ == ()


def test_signatures_export_and_descriptor_size():
    from vid2player3d_b200 import build
    assert test_host.signature_mismatches(abi.SIGNATURES, test_host.ENV_HEADERS) == []
    assert abi.SIGNATURES["b200v2p_eval_rally_stats"] == (C.c_int, [C.c_void_p, C.c_void_p])
    assert abi.SIGNATURES["b200v2p_eval_rally_stats_desc_size"] == (C.c_int32, [])
    L = C.CDLL(build.build())
    assert hasattr(L, "b200v2p_eval_rally_stats") and hasattr(L, "b200v2p_eval_rally_stats_desc_size")
    assert native.lib().b200v2p_eval_rally_stats_desc_size() == C.sizeof(abi.V2PRallyStats)


def test_binding_refuses_a_library_of_another_descriptor_size(monkeypatch):
    native.lib()
    S = abi.V2PRallyStats
    monkeypatch.setattr(abi, "V2PRallyStats", type("V2PRallyStats", (C.Structure,), {"_fields_": S._fields_[:-1]}))
    monkeypatch.setattr(native, "_lib", None)
    with pytest.raises(RuntimeError, match="V2PRallyStats descriptor.*rebuild"):
        native.lib()


def test_fill_fills_every_field_and_refuses_wrong_dtypes_and_nulls():
    from test_ball_stats import DTYPES, _OnDevice
    S = abi.V2PRallyStats
    keep = {f: torch.zeros(2, dtype=DTYPES[ct]) for f, ct in S._fields_ if issubclass(ct, C.c_void_p)}
    d = native.fill(S, dict(n=4), {f: _OnDevice(t) for f, t in keep.items()})
    for f, t in keep.items():
        assert getattr(d, f).value == t.data_ptr(), f
    assert d.n == 4 and d.pad_ == 0
    for f, ct in S._fields_:
        if not issubclass(ct, C.c_void_p):
            continue
        with pytest.raises(ValueError, match=rf"^V2PRallyStats\.{f}: None, but the header allows no NULL here"):
            native.fill(S, dict(n=4), dict({g: _OnDevice(t) for g, t in keep.items()}, **{f: None}))
        wrong = torch.float64 if ct is not abi.F32P else torch.int64
        with pytest.raises(ValueError, match=rf"^V2PRallyStats\.{f}: {wrong}, the header's pointee needs"):
            native.fill(S, dict(n=4), dict({g: _OnDevice(t) for g, t in keep.items()}, **{f: _OnDevice(torch.zeros(2, dtype=wrong))}))
    with pytest.raises(ValueError, match=r"^V2PRallyStats\.n: missing"):
        native.fill(S, {}, {f: _OnDevice(t) for f, t in keep.items()})


POINTERS = [f for f, ct in abi.V2PRallyStats._fields_ if issubclass(ct, C.c_void_p)]


@pytest.mark.parametrize("n, missing, msg", [(3, None, "n must be even"), (-2, None, "n must be even"), (0, "shots_hist", "shots_hist is NULL")]
                         + [(4, f, f"{f} is NULL") for f in POINTERS])
def test_launch_refusals_before_any_launch(n, missing, msg):
    """refused on fake device addresses with the reason, before anything is launched"""
    L = native.lib()
    d = abi.V2PRallyStats(n=n)
    for f in POINTERS:
        if f != missing:
            setattr(d, f, 0x10000)
    assert L.b200v2p_eval_rally_stats(C.byref(d), None) == -1
    assert L.b200v2p_last_error().decode() == f"b200v2p_eval_rally_stats: {msg}" + (" and >= 0 (the pairs 2k, 2k+1)" if "even" in msg else "")
