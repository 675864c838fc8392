"""CPU checks of the per-row results of the tennis controllers' fixed test set (cfg.env.b200_ball_stats): the float64 restatement
oracle/ref_port_ball_stats.py against the two fixtures it is composed from (tests/golden/v2p_eval.npz for the recovery events and
their values, tests/golden/v2p_ball_test_set.npz for the draws and the cursor walk), the cfg refusals, the file path, the export and
its summary line, and the C ABI of b200v2p_bstats_t."""
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
from oracle import ref_port_ball_stats as B
from oracle import ref_port_eval as R
from vid2player3d_b200 import abi, native
from vid2player3d_b200.tasks import mvae_controller_vis as V

RESET_IN = ("progress", "tar_time", "tar_time_total", "tar_action", "swing_type_cycle", "has_contact", "has_bounce", "est_bounce_in",
            "ball_pos", "root_pos", "ball_vel", "est_bounce_pos", "target_bounce_pos")


# ------------------------------------------------------------------------------------------------ the restatement
@pytest.mark.parametrize("P, layout", [(1, "one row"), (3, "wrap"), (16, "own row"), (21, "pool larger")])
def test_events_fold_the_reference_meters_by_row(P, layout):
    """the reference's reset rule and meters (v2p_eval.npz) over its 16 envs, each env fixed on one row: a row's counts are the meter
    counts and (integer-valued) sums of its envs, its error sum their meter-3 sums"""
    z = golden("v2p_eval.npz")
    T, N = z["reset_progress"].shape
    cursor = {"one row": np.zeros(N, np.int64), "wrap": np.arange(N) % P, "own row": (np.arange(N) + 1) % P,
              "pool larger": np.random.default_rng(1).permutation(P)[:N]}[layout].astype(np.int64)
    st, M = B.BallStats(P), R.new_meters(N)
    for t in range(T):
        out = st.eval_reset({k: z["reset_" + k][t] for k in RESET_IN}, int(z["reset_episode_length"]), M, cursor)
        np.testing.assert_array_equal(out[2], z["reset_out_recovery"][t])
    row = B.playing_row(cursor, P)
    fold = lambda v: np.bincount(row, weights=v.astype(np.float64), minlength=P)  # noqa: E731
    count, msum = z["reset_out_meter_count"][-1], z["reset_out_meter_sum"][-1]
    np.testing.assert_array_equal(st.recoveries, fold(count[0]))
    for k, m in (("hits", 0), ("forehands", 1), ("bounce_in", 2)):
        np.testing.assert_array_equal(getattr(st, k), fold(msum[m]), k)
        assert getattr(st, k).dtype == np.int64
    np.testing.assert_array_equal(st.bounce_in, fold(count[3]))          # meter 3 updates at the bounce-in events
    np.testing.assert_allclose(st.bounce_err_sum, fold(msum[3]), rtol=1e-6, atol=1e-6)
    assert st.recoveries.sum() == z["reset_out_recovery"].sum() > 0 and (st.served == 0).all()
    if layout == "own row":
        np.testing.assert_array_equal(st.recoveries, count[0])


@pytest.mark.parametrize("case", ["wrap", "one_row", "pool_larger"])
def test_draws_are_the_reference_generators(case):
    """every draw of the fixture's calls (repeated envs, a wrap past P, P = 1, P > N) is counted at its row, the cursor walks as the
    reference's, and after each call the row an env plays is the row it was just given"""
    z = golden("v2p_ball_test_set.npz")
    g = lambda k: z[f"{case}_{k}"]  # noqa: E731
    pool, lens, ids = g("pool"), g("lens"), g("env_ids")
    P = len(pool)
    st, cursor = B.BallStats(P), np.zeros(int(g("num_envs")), np.int64)
    start = np.concatenate([[0], np.cumsum(lens)])
    for a, b in zip(start[:-1], start[1:]):
        idx = st.generate(pool, cursor, ids[a:b])[0]
        np.testing.assert_array_equal(idx, g("index")[a:b])
        np.testing.assert_array_equal(B.playing_row(cursor[ids[a:b]], P), g("index")[a:b])
    np.testing.assert_array_equal(st.served, np.bincount(g("index"), minlength=P))
    np.testing.assert_array_equal(cursor, g("cursor"))
    assert st.served.sum() == len(ids) and st.recoveries.sum() == 0


def test_bounce_error_is_meter_threes_value():
    est = np.array([[3.0, 4.0, 0.0], [0.1, 0.2, 0.0]], np.float32)
    tgt = np.array([[0.0, 0.0, 0.0], [0.1, 0.2, 0.0]], np.float32)
    np.testing.assert_array_equal(B.bounce_err(est, tgt), np.array([5.0, 0.0], np.float32))
    assert B.playing_row(np.array([0, 1, 2]), 3).tolist() == [2, 0, 1] and B.playing_row(np.array([0]), 1).tolist() == [0]


# ------------------------------------------------------------------------------------------------ cfg, file, export
def _single(tmp_path, **v2p):
    cfg = v2p_cfg(4, **v2p)
    cfg["env"]["b200_ball_stats"] = True
    return cfg


@pytest.mark.parametrize("how", ["no test set", "test_mode random", "dual task", "dual cfg"])
def test_refusals_come_before_anything_is_allocated(tmp_path, how, monkeypatch):
    """random draws (no ball_traj_file_test, or test_mode random) and dual mode are refused in the constructor, before the physics
    task is built (no device is needed to see them)"""
    from vid2player3d_b200.tasks import MVAEControllerVis, MVAEControllerVisDual
    monkeypatch.setattr(torch, "zeros", None)           # an allocation would fail with another error
    cls, msg = MVAEControllerVis, "needs a fixed test set"
    if how == "no test set":
        cfg = _single(tmp_path)
    elif how == "test_mode random":
        cfg = _single(tmp_path, test_mode="random", ball_pool_test=np.zeros((3, 307), np.float32))
    else:
        cfg = v2p_dual_cfg(4)
        cfg["env"]["b200_ball_stats"] = True
        cls = MVAEControllerVisDual if how == "dual task" else MVAEControllerVis
        msg = "dual mode builds no ball pool"
    with pytest.raises(ValueError, match=msg):
        cls(cfg, None, 1, "cuda", 0, True)


def test_a_fixed_test_set_is_accepted_and_the_key_is_opt_in(tmp_path):
    cfg = _single(tmp_path)
    cfg["env"]["ball_traj_file_test"] = str(tmp_path / "balls_test.npy")
    V._check_ball_stats_cfg(cfg, dual=False)
    assert "test_mode" not in cfg["env"]["vid2player"]          # the check resolves on a copy
    V._check_ball_stats_cfg(_single(tmp_path, test_mode="single_cycle", ball_pool_test=np.zeros((2, 307), np.float32)), dual=False)
    for cfg in (v2p_cfg(4), v2p_dual_cfg(4)):                    # without the key nothing is checked
        V._check_ball_stats_cfg(cfg, dual=True)


def test_file_path_rule():
    assert V.ball_stats_path({"b200_ball_stats_file": "runs/balls.npz"}) == "runs/balls.npz"
    now = datetime.datetime(2026, 1, 2, 3, 4, 5)
    assert V.ball_stats_path({}, now) == os.path.join("out", "ball_stats", "ball_stats_2026-01-02-03:04:05.npz")
    assert V.ball_stats_path({"b200_ball_stats_file": ""}, now) == V.ball_stats_path({}, now)


def _fake_task(tmp_path, served, buckets, path="balls.npz", test_file="sets/balls_test_single.npy"):
    t = V.MVAEControllerVis.__new__(V.MVAEControllerVis)
    t.cfg = dict(env=dict(b200_ball_stats_file=str(tmp_path / path)))
    t.cfg_v2p = dict(ball_traj_file_test=test_file) if test_file else {}
    t.num_envs, t._test_steps = 6, 41
    t._bstats = dict(served=torch.tensor(served, dtype=torch.long), buckets=torch.tensor(buckets, dtype=torch.long))
    return t


def test_export_arrays_dtypes_and_summary_line(tmp_path, capsys):
    buckets = [[4, 3, 1, 2, 3 << 24], [2, 0, 0, 0, 0], [0, 0, 0, 0, 0], [6, 5, 2, 4, (1 << 23) + 5]]
    t = _fake_task(tmp_path, [5, 3, 1, 7], buckets, path="sub/dir/balls.npz")
    path = t.export_ball_stats()
    assert path == str(tmp_path / "sub/dir/balls.npz")
    z = np.load(path)
    assert sorted(z.files) == sorted(["served", "recoveries", "hits", "forehands", "bounce_in", "bounce_err_sum", "ball_traj_file_test",
                                      "num_envs", "test_steps"])
    b = np.array(buckets, np.int64)
    for k, col in (("recoveries", 0), ("hits", 1), ("forehands", 2), ("bounce_in", 3)):
        assert z[k].dtype == np.int64 and z[k].tolist() == b[:, col].tolist(), k
    assert z["served"].dtype == np.int64 and z["served"].tolist() == [5, 3, 1, 7]
    assert z["bounce_err_sum"].dtype == np.float64 and z["bounce_err_sum"].tolist() == [3.0, 0.0, 0.0, 0.5 + 5 * 2.0 ** -24]
    assert str(z["ball_traj_file_test"]) == "sets/balls_test_single.npy" and int(z["num_envs"]) == 6 and int(z["test_steps"]) == 41
    out = capsys.readouterr().out.splitlines()
    assert out[0] == "balls served: 16  recoveries: 12  hit rate: 0.6667  bounce-in rate: 0.5000  rows never hit: 2 of 4"
    assert out[1] == f"============ per-ball statistics written to {path} ============"


def test_summary_without_recoveries_and_in_memory_test_set(tmp_path, capsys):
    t = _fake_task(tmp_path, [2], [[0] * 5], test_file=None)
    z = np.load(t.export_ball_stats())
    assert str(z["ball_traj_file_test"]) == ""
    assert capsys.readouterr().out.splitlines()[0] == ("balls served: 2  recoveries: 0  hit rate: nan  bounce-in rate: nan  "
                                                      "rows never hit: 1 of 1")


# ------------------------------------------------------------------------------------------------ the C ABI
NAMES = {C.c_float: "float", C.c_int64: "int64_t", C.c_int32: "int32_t", C.c_uint8: "uint8_t"}


def _layout(ctype, S):
    lines, want = [f'printf("{ctype} %zu\\n", sizeof({ctype}));'], [f"{ctype} {C.sizeof(S)}"]
    for f, ct in S._fields_:
        lines.append(f'printf("{ctype}.{f} %zu %zu\\n", offsetof({ctype}, {f}), sizeof((({ctype}*)0)->{f}));')
        want.append(f"{ctype}.{f} {getattr(S, f).offset} {getattr(S, f).size}")
        if issubclass(ct, C.c_void_p) and ct is not C.c_void_p:
            lines.append(f'printf("{ctype}.{f} %d\\n", __builtin_types_compatible_p(__typeof__(*(({ctype}*)0)->{f}), {NAMES[ct.pointee]}));')
            want.append(f"{ctype}.{f} 1")
    return lines, want


def test_descriptor_layout_matches_the_header(tmp_path):
    """b200v2p_bstats_t field by field with its pointee types, and the bucket width and fixed-point scale of the header"""
    lines, want = _layout("b200v2p_bstats_t", abi.V2PBallStats)
    lines.append('printf("%d %.1f\\n", B200V2P_BSTATS_COLS, B200V2P_BSTATS_FIX_SCALE);')
    want.append(f"{abi.BSTATS_COLS} {abi.BSTATS_FIX_SCALE:.1f}")
    src, exe = tmp_path / "layout.c", tmp_path / "layout"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "b200env_v2p.h"\nint main(void) {\n' + "\n".join(lines) +
                   "\nreturn 0;\n}\n")
    subprocess.check_call(["gcc", "-w", "-I", os.path.join(test_host.ROOT, "include"), str(src), "-o", str(exe)])
    assert subprocess.check_output([str(exe)], text=True).splitlines() == want
    assert abi.BSTATS_COLS == 5 and abi.BSTATS_FIX_SCALE == 2.0 ** 24
    assert set(abi.V2PBallStats._nullable_) == {f for f, ct in abi.V2PBallStats._fields_ if issubclass(ct, C.c_void_p)} - {"pool_cursor"}
    assert "#define B200_ABI_VERSION 11" in open(os.path.join(test_host.ROOT, "include", "b200env.h")).read()


def test_signatures_and_descriptor_sizes():
    assert test_host.signature_mismatches(abi.SIGNATURES, test_host.ENV_HEADERS) == []
    assert abi.SIGNATURES["b200v2p_eval_ball_stats"] == (C.c_int, [C.c_void_p, C.c_void_p])
    assert abi.SIGNATURES["b200v2p_eval_ball_stats_desc_size"] == (C.c_int32, [])
    assert native.lib().b200v2p_eval_ball_stats_desc_size() == C.sizeof(abi.V2PBallStats)


def test_binding_refuses_a_library_of_another_descriptor_size(monkeypatch):
    """a library whose descriptor differs in size: native.lib() refuses it rather than pass a descriptor it would misread"""
    native.lib()
    S = abi.V2PBallStats
    monkeypatch.setattr(abi, "V2PBallStats", type("V2PBallStats", (C.Structure,), {"_fields_": S._fields_[:-1]}))
    monkeypatch.setattr(native, "_lib", None)
    with pytest.raises(RuntimeError, match="V2PBallStats descriptor.*rebuild"):
        native.lib()


class _OnDevice:
    """a host tensor that reports device 0, so that native.fill's device rule lets it through on a machine without a GPU"""

    def __init__(self, t):
        self.t, self.dtype = t, t.dtype

    def is_contiguous(self):
        return self.t.is_contiguous()

    def get_device(self):
        return 0

    def data_ptr(self):
        return self.t.data_ptr()


DTYPES = {abi.F32P: torch.float32, abi.I64P: torch.int64, abi.U8P: torch.bool}


def test_fill_fills_every_field_and_refuses_wrong_ones():
    S = abi.V2PBallStats
    keep = {f: torch.zeros(2, dtype=DTYPES[ct]) for f, ct in S._fields_ if issubclass(ct, C.c_void_p)}
    d = native.fill(S, dict(n=2, pool_size=3), {f: _OnDevice(t) for f, t in keep.items()})
    for f, t in keep.items():
        assert getattr(d, f).value == t.data_ptr(), f
    assert (d.n, d.pool_size) == (2, 3)
    with pytest.raises(ValueError, match=r"^V2PBallStats\.buckets: torch\.float64, the header's pointee needs torch\.int64"):
        native.fill(S, dict(n=2, pool_size=3), dict({f: _OnDevice(t) for f, t in keep.items()},
                                                    buckets=_OnDevice(torch.zeros(2, dtype=torch.float64))))
    with pytest.raises(ValueError, match=r"^V2PBallStats\.pool_cursor: None"):
        native.fill(S, dict(n=2, pool_size=3), dict({f: _OnDevice(t) for f, t in keep.items()}, pool_cursor=None))
    d = native.fill(S, dict(n=2, pool_size=3), {f: _OnDevice(keep[f]) for f in ("pool_cursor", "reset_reaction", "row_served")})
    assert d.row_served.value == keep["row_served"].data_ptr() and d.reset_recovery.value is None and d.buckets.value is None
    with pytest.raises(ValueError, match=r"^V2PBallStats\.pool_size: missing"):
        native.fill(S, dict(n=2), {f: _OnDevice(t) for f, t in keep.items()})


EVENTS = ("reset_recovery", "has_contact", "swing_type_cycle", "est_bounce_in", "est_bounce_pos", "target_bounce_pos", "buckets")


@pytest.mark.parametrize("given, P, msg", [
    (("pool_cursor", "reset_reaction", "row_served"), 0, "bad arguments"),
    (("reset_reaction", "row_served"), 3, "bad arguments"),
    (("pool_cursor",), 3, "not both or neither"),
    (("pool_cursor", "reset_reaction", "row_served") + EVENTS, 3, "not both or neither"),
    (("pool_cursor", "reset_reaction"), 3, "bad arguments"),
    (("pool_cursor",) + EVENTS[:-1], 3, "bad arguments"),
    (("pool_cursor", "row_served") + EVENTS[1:], 3, "not both or neither"),
])
def test_launch_refusals_before_any_launch(given, P, msg):
    """refused on fake device addresses: one complete form or nothing is launched"""
    L = native.lib()
    d = abi.V2PBallStats(n=4, pool_size=P)
    for name in given:
        setattr(d, name, 0x10000)
    assert L.b200v2p_eval_ball_stats(C.byref(d), None) == -1
    err = L.b200v2p_last_error().decode()
    assert err.startswith("b200v2p_eval_ball_stats: ") and msg in err
