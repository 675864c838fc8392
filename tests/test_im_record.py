"""CPU checks of HumanoidSMPLIMVis' qpos recorder: the float64 restatement oracle/ref_port_record.py against tests/golden/im_record.npz
(made by executing the reference's own _sync_ref_motion, tests/golden/make_golden_record.py), the export assembly of the device rows,
the C ABI mirror of b200_im_record_t, native.fill's refusals, the cfg refusals and the file name and frame count rules."""
import ctypes as C
import datetime
import os
import subprocess
import types

import numpy as np
import pytest
import torch

import test_host
from conftest import golden
from oracle import ref_port_record as R
from vid2player3d_b200 import abi, native
from vid2player3d_b200.tasks import humanoid_smpl_im_vis as V

Z = golden("im_record.npz")
N, ND = 8, 69
NQ = 7 + ND


def oracle(init, ids=range(N)):
    return R.sync_ref_motion(Z["rb_pos"], Z["rb_rot"], Z["dof_pos"], Z["p_rb_pos"], Z["p_rb_rot"], Z["p_dof_pos"], list(ids), init)


@pytest.mark.parametrize("init", [0, 1])
def test_oracle_is_the_reference_sync(init):
    np.testing.assert_allclose(oracle(init), Z[f"qpos_init{init}"], rtol=0, atol=1e-12)


def test_oracle_serves_any_env_list():
    ids = [5, 0, 7, 2]
    np.testing.assert_allclose(oracle(0, ids), Z["qpos_init0"][ids], rtol=0, atol=1e-12)


@pytest.mark.parametrize("init", [0, 1])
def test_export_assembles_the_viewer_qpos(init):
    """device rows [E, T, 2, nq] (copy 1 with its x += 1, copy 2 left out) -> [E, T, 3 nq] equals the reference's qpos"""
    want = Z[f"qpos_init{init}"]
    rows = torch.from_numpy(np.stack([want[:, :NQ], want[:, NQ:2 * NQ]], 1))[:, None]        # [E, 1, 2, nq], T = 1
    got = V.assemble_qpos(rows)
    assert got.shape == (N, 1, 3 * NQ)
    np.testing.assert_allclose(got[:, 0].numpy(), want, rtol=0, atol=1e-12)
    got32 = V.assemble_qpos(rows.float())
    assert got32.dtype == torch.float32
    np.testing.assert_allclose(got32[:, 0].numpy(), want, rtol=1e-6, atol=1e-6)


def test_descriptor_layout_matches_the_header(tmp_path):
    ctype, S = "b200_im_record_t", abi.ImRecord
    lines, want = [f'printf("{ctype} %zu\\n", sizeof({ctype}));'], [f"{ctype} {C.sizeof(S)}"]
    names = {C.c_float: "float", C.c_int64: "int64_t", C.c_uint32: "uint32_t"}
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
    assert "b200env_im_record" in abi.SIGNATURES and "b200env_im_record_desc_size" in abi.SIGNATURES
    assert native.lib().b200env_im_record_desc_size() == C.sizeof(abi.ImRecord)


def _fill_args():
    f, i = (lambda *s: torch.zeros(*s)), (lambda *s: torch.zeros(*s, dtype=torch.long))   # noqa: E731
    s = dict(n_rec=2, num_envs=4, num_bodies=24, num_lib_bodies=24, nd=69, cap=3, init=0)
    t = dict(env_ids=i(2), rigid_body_state=f(4), dof_state=f(4), p_dof_pos=f(4), p_rb_pos=f(4), p_rb_rot=f(4), reset_buf=i(4),
             motion_ids=i(4), qpos=f(4), rec_motion_ids=i(4), rec_reset=i(4), frame=i(1), done=torch.zeros(1, dtype=torch.int32),
             games=None)
    return s, t


def test_fill_refusals():
    s, t = _fill_args()
    with pytest.raises(ValueError, match="ImRecord.env_ids: not on the CUDA device"):
        native.fill(abi.ImRecord, s, t)
    with pytest.raises(ValueError, match="ImRecord.env_ids: torch.int32"):
        native.fill(abi.ImRecord, s, dict(t, env_ids=torch.zeros(2, dtype=torch.int32)))
    with pytest.raises(ValueError, match="ImRecord.done: torch.int64"):
        native.fill(abi.ImRecord, s, dict(t, done=torch.zeros(1, dtype=torch.long)))
    with pytest.raises(ValueError, match="ImRecord.qpos: None"):
        native.fill(abi.ImRecord, s, dict(t, qpos=None))
    with pytest.raises(ValueError, match="ImRecord.init: missing"):
        native.fill(abi.ImRecord, dict(s, init=None), t)
    with pytest.raises(ValueError, match="ImRecord.qpos: not contiguous"):
        native.fill(abi.ImRecord, s, dict(t, qpos=torch.zeros(4, 2).t()))


@pytest.mark.parametrize("over, msg", [(dict(n_rec=0), "n_rec, cap and num_envs must be positive"),
                                       (dict(cap=0), "n_rec, cap and num_envs must be positive"),
                                       (dict(nd=68), "multiple of 3"), (dict(num_lib_bodies=0), "num_lib_bodies")])
def test_launch_refusals_before_any_launch(over, msg):
    """refused on fake device addresses: the checks come before the launch"""
    s, _ = _fill_args()
    d = abi.ImRecord(**dict(s, **over))
    for name, _ in abi.ImRecord._fields_[8:-1]:
        setattr(d, name, 0x10000)
    assert native.lib().b200env_im_record(C.byref(d), None) == -2
    assert msg in native.lib().b200env_last_error().decode()


@pytest.mark.parametrize("spec, msg", [([], "empty"), ([0, 4], r"\[4\] lie outside \[0, 4\)"), ([-1], "outside"),
                                       ([1, 2, 1], r"duplicate env ids \[1\]"), ("some", "list of env ids")])
def test_env_list_refusals(spec, msg):
    with pytest.raises(ValueError, match=msg):
        V.record_env_ids(spec, 4)


def test_env_list_rules():
    assert V.record_env_ids("all", 3) == [0, 1, 2]
    assert V.record_env_ids([2, 0], 3) == [2, 0]


def test_frames_rules():
    args = types.SimpleNamespace(rec_once=True)
    assert V.record_frames({}, None, [5, 9]) == 300
    assert V.record_frames({"num_rec_frames": 7}, types.SimpleNamespace(), [5, 9]) == 7     # embodied_pose's parser has no rec_once
    assert V.record_frames({"num_rec_frames": 7}, args, np.array([5, 91, 9])) == 91
    with pytest.raises(ValueError, match="at least 1, got 0"):
        V.record_frames({"num_rec_frames": 0}, None, [5])


def test_file_rules():
    assert V.record_path({"rec_fname": "out/clip.mp4"}) == "out/clip.npz"
    assert V.record_path({"rec_fname": "clip"}) == "clip.npz"
    now = datetime.datetime(2026, 1, 2, 3, 4, 5)
    assert V.record_path({}, now) == os.path.join("out", "recording", "qpos_2026-01-02-03:04:05.npz")


def test_memory_bound():
    assert V.record_bytes(8192, 300, 76) == 8192 * 300 * 2 * 76 * 4


@pytest.mark.parametrize("over, msg", [(dict(b200_record_envs=[0, 0]), "duplicate"), (dict(b200_record_envs=[9]), "outside"),
                                       (dict(num_rec_frames=0), "at least 1")])
def test_task_refuses_the_cfg_before_building(over, msg):
    """the refusals come before the task allocates anything (no device is needed to see them)"""
    from vid2player3d_b200.tasks import HumanoidSMPLIMVis
    cfg = {"env": dict(numEnvs=4, b200_record_qpos=True, **over)}
    with pytest.raises(ValueError, match=msg):
        HumanoidSMPLIMVis(cfg, None, 1, "cuda", 0, True)
