"""CPU checks of the imitation test run's held-out library and per-motion meters: cfg.env.test_motion_file resolved as the reference
resolves it (humanoid_smpl_im.py:77-80) with its refusals, the float64 restatement oracle/ref_port_motion_stats.py on hand-built
histories, the env lists and the summary line of HumanoidSMPLIMVis, and the C ABI of b200_im_motion_stats_t."""
import ctypes as C
import datetime
import os
import subprocess
import types

import numpy as np
import pytest
import torch

import test_host
from oracle import ref_port_motion_stats as R
from vid2player3d_b200 import abi, model_compiler, motion_lib, native
from vid2player3d_b200.configs import im_cfg
from vid2player3d_b200.tasks import humanoid_smpl_im_vis as V
from vid2player3d_b200.tasks.humanoid_smpl_im import resolve_test_motion_file

ASSET = "mjcf/smpl_mesh_humanoid_amass_v1.xml"


@pytest.fixture(scope="module")
def libs(tmp_path_factory):
    """a 2-motion training library and a 3-motion test library on disk"""
    model = model_compiler.load_compiled("smpl_mesh_humanoid_amass_v1")
    d = tmp_path_factory.mktemp("motions")
    train, test = motion_lib.synthetic(model, num_motions=2, num_frames=20, seed=1), motion_lib.synthetic(model, num_motions=3,
                                                                                                           num_frames=20, seed=2)
    train.save(str(d / "train.npz"))
    test.save(str(d / "test.npz"))
    return str(d / "train.npz"), str(d / "test.npz")


def cfg_of(libs, test, **over):
    cfg = im_cfg(4, None, **dict(dict(motion_file=libs[0], test_motion_file=libs[1]), **over))
    cfg["args"] = types.SimpleNamespace(test=test)
    return cfg


def test_test_motion_file_is_read_only_under_args_test(libs):
    cfg = cfg_of(libs, True)
    assert resolve_test_motion_file(cfg) == libs[1] and cfg["env"]["motion_file"] == libs[1]
    for args in (types.SimpleNamespace(test=False), types.SimpleNamespace(), None):
        cfg = cfg_of(libs, False)
        cfg["args"] = args
        assert resolve_test_motion_file(cfg) is None and cfg["env"]["motion_file"] == libs[0]
    cfg = cfg_of(libs, True)
    del cfg["env"]["test_motion_file"]
    assert resolve_test_motion_file(cfg) is None and cfg["env"]["motion_file"] == libs[0]


def test_test_motion_assets_replace_motion_assets(libs):
    cfg = cfg_of(libs, True, motion_assets=[ASSET] * 2, test_motion_assets=[ASSET] * 3)
    resolve_test_motion_file(cfg)
    assert cfg["env"]["motion_assets"] == [ASSET] * 3
    cfg = cfg_of(libs, False, motion_assets=[ASSET] * 2, test_motion_assets=[ASSET] * 3)
    resolve_test_motion_file(cfg)
    assert cfg["env"]["motion_assets"] == [ASSET] * 2


def test_missing_file_is_refused_with_its_path(libs, tmp_path):
    missing = str(tmp_path / "held_out.npz")
    with pytest.raises(FileNotFoundError, match=f"test_motion_file {missing} does not exist"):
        resolve_test_motion_file(dict(cfg_of(libs, True), env=dict(cfg_of(libs, True)["env"], test_motion_file=missing)))


def test_motion_assets_without_test_motion_assets_are_refused(libs):
    with pytest.raises(ValueError, match="needs its own list in test_motion_assets"):
        resolve_test_motion_file(cfg_of(libs, True, motion_assets=[ASSET] * 2))


def test_the_task_refuses_before_allocating(libs):
    """the refusals of HumanoidSMPLIMVis' constructor come before anything reaches the device (none is needed to see them)"""
    from vid2player3d_b200.tasks import HumanoidSMPLIMVis
    with pytest.raises(ValueError, match=r"test_motion_assets has 2 entries for the 3 motions of test_motion_file .*test\.npz"):
        HumanoidSMPLIMVis(cfg_of(libs, True, motion_assets=[ASSET] * 2, test_motion_assets=[ASSET] * 2), None, 1, "cuda", 0, True)
    with pytest.raises(ValueError, match="needs its own list"):
        HumanoidSMPLIMVis(cfg_of(libs, True, motion_assets=[ASSET] * 2), None, 1, "cuda", 0, True)
    with pytest.raises(FileNotFoundError, match="nothing.npz does not exist"):
        HumanoidSMPLIMVis(cfg_of(libs, True, test_motion_file="nothing.npz"), None, 1, "cuda", 0, True)


# ---------------------------------------------------------------------------------------------------------- the restatement
def history(n, steps, B=2, seed=0):
    g = np.random.default_rng(seed)
    return [dict(rew=g.random(n), sub_rewards=g.random((n, 4)), reset_buf=np.zeros(n, np.int64), terminate_buf=np.zeros(n, np.int64),
                 body_pos=g.normal(size=(n, B, 3)), target_pos=g.normal(size=(n, B, 3))) for _ in range(steps)]


def run(ms, hist, stops=None):
    for k, h in enumerate(hist):
        ms.step(**h, stop=bool(stops and stops[k]))
    return ms


def test_body_position_error_is_the_mean_distance():
    body = np.zeros((1, 2, 3))
    target = np.array([[[3.0, 4.0, 0.0], [0.0, 0.0, 1.0]]])
    assert R.body_pos_err(body, target)[0] == 3.0


def test_a_game_is_counted_once_where_done_rises():
    """env 0 ends at step 1 and stays done (counted once); env 1 ends at step 3; a fall counts as a fall, a motion end does not"""
    h = history(2, 5)
    for k in range(1, 5):
        h[k]["reset_buf"][0] = 1
    h[1]["terminate_buf"][0] = 1
    h[3]["reset_buf"][1] = 1
    h[4]["reset_buf"][1] = 1
    ms = run(R.MotionStats([0, 1], 3), h)
    assert ms.counts.tolist() == [[1, 1], [1, 0], [0, 0]]          # motion 2 has no env: no games
    want0 = sum(np.concatenate([[h[k]["rew"][0], 1.0], h[k]["sub_rewards"][0], [R.body_pos_err(h[k]["body_pos"], h[k]["target_pos"])[0]]])
                for k in range(2))
    want1 = sum(np.concatenate([[h[k]["rew"][1], 1.0], h[k]["sub_rewards"][1], [R.body_pos_err(h[k]["body_pos"], h[k]["target_pos"])[1]]])
                for k in range(4))
    np.testing.assert_allclose(ms.sums[0], want0, rtol=1e-15)
    np.testing.assert_allclose(ms.sums[1], want1, rtol=1e-15)
    assert not ms.sums[2].any()
    # env 0 went on summing after its game: a step with done falling and rising again is a second game from zero
    ms.step(**dict(history(2, 1, seed=3)[0], reset_buf=np.array([0, 1])))
    last = history(2, 1, seed=4)[0]
    ms.step(**dict(last, reset_buf=np.array([1, 1])))
    assert ms.counts.tolist() == [[2, 1], [1, 0], [0, 0]]
    assert ms.sums[0, 1] == 2 + 5   # the first game's 2 steps, then steps 2-4 of the first run and the two new ones


def test_envs_of_one_motion_share_its_bucket_and_a_fall_is_the_end_step_flag():
    h = history(4, 3)
    h[0]["terminate_buf"][:] = 1                # a fall flag before the end step is not a fall
    h[2]["reset_buf"][:] = 1
    h[2]["terminate_buf"][[1, 3]] = 1
    ms = run(R.MotionStats([1, 1, 1, 0], 2), h)
    assert ms.counts.tolist() == [[1, 1], [3, 1]]
    assert ms.sums[:, 1].tolist() == [3.0, 9.0]


def test_nothing_changes_while_stopped_and_a_new_game_starts_from_zero():
    h = history(2, 4)
    h[1]["reset_buf"][:] = 1
    h[2]["reset_buf"][:] = [1, 0]
    h[3]["reset_buf"][:] = 1
    ms = run(R.MotionStats([0, 0], 1), h, stops=[0, 0, 1, 1])
    assert ms.counts.tolist() == [[2, 0]] and ms.sums[0, 1] == 4.0
    ms.new_game()
    assert not ms.env_sums.any() and not ms.prev_done.any()
    ms.step(**h[3])
    assert ms.counts.tolist() == [[4, 0]] and ms.sums[0, 1] == 6.0
    np.testing.assert_allclose(ms.sums[0, 0], h[0]["rew"].sum() + h[1]["rew"].sum() + h[3]["rew"].sum(), rtol=1e-15)


# ---------------------------------------------------------------------------------------------------------- the task's host side
def test_env_lists_group_the_envs_by_motion_in_env_order():
    start, envs = V.motion_env_lists(torch.tensor([2, 0, 2, 2, 0, 4]), 6)
    assert start.tolist() == [0, 2, 2, 5, 5, 6, 6] and envs.tolist() == [1, 4, 0, 2, 3, 5]


def test_summary_line_and_file_rules():
    counts = np.array([[2, 1], [0, 0], [2, 0]])
    sums = np.zeros((3, 7))
    sums[:, 0], sums[:, 1], sums[:, 6] = [3.0, 0.0, 5.0], [10, 0, 6], [0.8, 0.0, 0.8]
    assert V.motion_stats_summary(counts, sums) == ("motions evaluated: 2 of 3  games without a fall: 0.7500  reward per step: 0.500000"
                                                    "  body position error: 0.100000 m")
    assert V.motion_stats_path({"b200_motion_stats_file": "runs/eval.npz"}) == "runs/eval.npz"
    now = datetime.datetime(2026, 1, 2, 3, 4, 5)
    assert V.motion_stats_path({}, now) == os.path.join("out", "motion_stats", "motion_stats_2026-01-02-03:04:05.npz")


# ---------------------------------------------------------------------------------------------------------- the C ABI
def test_descriptor_layout_matches_the_header(tmp_path):
    ctype, S = "b200_im_motion_stats_t", abi.ImMotionStats
    lines, want = [f'printf("{ctype} %zu\\n", sizeof({ctype}));'], [f"{ctype} {C.sizeof(S)}"]
    names = {C.c_float: "float", C.c_int64: "int64_t", C.c_int32: "int32_t", C.c_double: "double"}
    for f, ct in S._fields_:
        lines.append(f'printf("{ctype}.{f} %zu %zu\\n", offsetof({ctype}, {f}), sizeof((({ctype}*)0)->{f}));')
        want.append(f"{ctype}.{f} {getattr(S, f).offset} {getattr(S, f).size}")
        if issubclass(ct, C.c_void_p) and ct is not C.c_void_p:
            lines.append(f'printf("{ctype}.{f} %d\\n", __builtin_types_compatible_p(__typeof__(*(({ctype}*)0)->{f}), {names[ct.pointee]}));')
            want.append(f"{ctype}.{f} 1")
    src, exe = tmp_path / "layout.c", tmp_path / "layout"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "b200env.h"\nint main(void) {\n' + "\n".join(lines) + "\nreturn 0;\n}\n")
    subprocess.check_call(["gcc", "-w", "-I", os.path.join(test_host.ROOT, "include"), str(src), "-o", str(exe)])
    assert subprocess.check_output([str(exe)], text=True).splitlines() == want
    assert "#define B200_ABI_VERSION 11" in open(os.path.join(test_host.ROOT, "include", "b200env.h")).read()


def test_signatures_and_descriptor_size():
    assert test_host.signature_mismatches(abi.SIGNATURES, test_host.ENV_HEADERS) == []
    assert "b200env_im_motion_stats" in abi.SIGNATURES and "b200env_im_motion_stats_desc_size" in abi.SIGNATURES
    assert native.lib().b200env_im_motion_stats_desc_size() == C.sizeof(abi.ImMotionStats)


def test_binding_refuses_a_library_of_another_descriptor_size(monkeypatch):
    native.lib()
    old = type("ImMotionStats", (C.Structure,), {"_fields_": abi.ImMotionStats._fields_[:-1]})
    monkeypatch.setattr(abi, "ImMotionStats", old)
    monkeypatch.setattr(native, "_lib", None)
    with pytest.raises(RuntimeError, match="ImMotionStats descriptor.*rebuild"):
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


DTYPES = {abi.F32P: torch.float32, abi.I64P: torch.int64, abi.I32P: torch.int32, abi.F64P: torch.float64}
SCALARS = dict(n=4, num_motions=3, num_bodies=24, num_lib_bodies=24)


def test_fill_fills_every_field():
    S = abi.ImMotionStats
    keep = {f: torch.zeros(2, dtype=DTYPES[ct]) for f, ct in S._fields_ if issubclass(ct, C.c_void_p)}
    d = native.fill(S, SCALARS, {f: _OnDevice(t) for f, t in keep.items()})
    for f, t in keep.items():
        assert getattr(d, f).value == t.data_ptr(), f
    assert (d.n, d.num_motions, d.num_bodies, d.num_lib_bodies) == (4, 3, 24, 24)
    d = native.fill(S, SCALARS, dict({f: _OnDevice(t) for f, t in keep.items()}, games=None))
    assert d.games.value is None
    with pytest.raises(ValueError, match=r"ImMotionStats\.env_flags: torch\.int64, the header's pointee needs torch\.int32"):
        native.fill(S, SCALARS, dict({f: _OnDevice(t) for f, t in keep.items()}, env_flags=_OnDevice(torch.zeros(2, dtype=torch.long))))
    with pytest.raises(ValueError, match=r"ImMotionStats\.sums: None"):
        native.fill(S, SCALARS, dict({f: _OnDevice(t) for f, t in keep.items()}, sums=None))


@pytest.mark.parametrize("over, msg", [(dict(n=0), "n and num_motions must be positive"), (dict(num_motions=0), "n and num_motions"),
                                       (dict(num_lib_bodies=0), "num_lib_bodies must lie in [1, num_bodies]"),
                                       (dict(num_lib_bodies=25), "num_lib_bodies must lie")])
def test_launch_refusals_before_any_launch(over, msg):
    """refused on fake device addresses: the checks come before the launch"""
    d = abi.ImMotionStats(**dict(SCALARS, **over))
    for name, ct in abi.ImMotionStats._fields_:
        if issubclass(ct, C.c_void_p):
            setattr(d, name, 0x10000)
    assert native.lib().b200env_im_motion_stats(C.byref(d), None) == -2
    assert msg in native.lib().b200env_last_error().decode()
