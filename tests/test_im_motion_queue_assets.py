"""CPU checks of the motion queue with a body per motion (cfg.env.b200_motion_queue with motion_assets): the restatement of the queue's
asset assignment (AssetQueue below, on oracle/ref_port_motion_queue.py's MotionQueue) on hand-built done sequences, the cfg checks, the
recording's per-frame `asset`, and the C ABI of b200_set_env_assets_t and the fields appended to b200_im_motion_queue_t."""
import ctypes as C
import os
import subprocess
import types

import numpy as np
import pytest
import torch

import test_host
from oracle import ref_port_motion_queue as Q
from test_im_motion_queue import ASSET, done, qcfg, step
from vid2player3d_b200 import abi, native
from vid2player3d_b200.tasks import humanoid_smpl_im_vis as V


class AssetQueue(Q.MotionQueue):
    """MotionQueue with each env's asset: env e starts on motion_asset[e % M]; an env that takes entry q gets motion_asset[q % M], an
    idle env and a stopped run keep theirs (b200env_im_motion_queue with motion_asset / env_asset).  Integers only."""

    def __init__(self, num_envs, num_motions, rounds, motion_asset):
        super().__init__(num_envs, num_motions, rounds)
        self.motion_asset = np.asarray(motion_asset, np.int32)
        assert self.motion_asset.shape == (num_motions,)
        self.env_asset = self.motion_asset[self.motion_ids]

    def assign(self, reset_buf):
        mask = super().assign(reset_buf)
        self.env_asset[mask] = self.motion_asset[self.motion_ids[mask]]
        return mask


# ---------------------------------------------------------------------------------------------------------- the restatement
def test_envs_start_on_their_motions_assets():
    q = AssetQueue(4, 3, 2, [2, 0, 1])
    assert q.env_asset.tolist() == [2, 0, 1, 2] and q.env_asset.dtype == np.int32


def test_ties_in_one_step_take_their_entries_assets():
    q = AssetQueue(4, 5, 2, [0, 1, 2, 3, 4])     # entries 0..9, envs on 0..3
    rb = done(4, 3, 1)
    step(q, rb)
    assert q.entry.tolist() == [0, 4, 2, 5] and q.env_asset.tolist() == [0, 4, 2, 0]   # entry 5 = motion 0
    rb[[0, 2]] = 1
    step(q, rb)
    assert q.entry.tolist() == [6, 4, 7, 5] and q.env_asset.tolist() == [1, 4, 2, 0]


def test_the_queue_running_dry_keeps_the_idle_envs_body():
    q = AssetQueue(4, 3, 2, [5, 6, 7])           # entries 0..5: two left after the start
    rb = done(4, 0, 1, 2)
    step(q, rb)
    assert q.entry.tolist() == [4, 5, 2, 3] and q.env_asset.tolist() == [6, 7, 7, 5] and q.idle.tolist() == [False, False, True, False]
    rb[[0, 1, 3]] = 1
    step(q, rb)                                  # every env finishes with the queue empty: nobody changes body
    assert q.env_asset.tolist() == [6, 7, 7, 5] and q.stop


def test_two_rounds_repeat_each_motions_asset():
    q = AssetQueue(2, 3, 2, [1, 0, 1])
    rb = np.zeros(2, np.int64)
    seen = []
    while not q.stop:
        rb[:] = 1
        m = step(q, rb)
        seen += list(zip(q.entry[m].tolist(), q.env_asset[m].tolist()))
    assert seen == [(2, 1), (3, 1), (4, 0), (5, 1)]


def test_nothing_changes_while_stopped():
    q = AssetQueue(2, 2, 2, [3, 4])
    q.stop = True
    rb = done(2, 0, 1)
    assert not step(q, rb).any() and q.env_asset.tolist() == [3, 4]


# ---------------------------------------------------------------------------------------------------------- cfg checks
def test_motion_assets_with_test_motion_assets_are_accepted():
    assert V.motion_queue_rounds(qcfg(motion_assets=[ASSET] * 2, test_motion_assets=[ASSET] * 3)) == 1
    assert V.motion_queue_rounds(qcfg(motion_assets=[ASSET] * 2, test_motion_assets=[ASSET] * 3, b200_motion_queue_repeats=2)) == 2
    with pytest.raises(ValueError, match="motion_assets alone is not supported"):
        V.motion_queue_rounds(qcfg(motion_assets=[ASSET] * 2))


def test_the_other_refusals_still_fire_with_assets():
    a = dict(motion_assets=[ASSET] * 2, test_motion_assets=[ASSET] * 3)
    with pytest.raises(ValueError, match="b200_motion_queue_repeats must be an int >= 1"):
        V.motion_queue_rounds(qcfg(b200_motion_queue_repeats=0, **a))
    with pytest.raises(ValueError, match="set b200_device_transforms"):
        V.motion_queue_rounds(qcfg(transform_specs=dict(mask_joints=dict(joints=["L_Knee"])), **a))
    with pytest.raises(ValueError, match="needs args.test or stateInit: Start, got 'Random'"):
        V.motion_queue_rounds(qcfg(test=False, stateInit="Random", **a))


def test_the_task_refuses_before_allocating(tmp_path):
    """the refusals come from the cfg, before a library is loaded or anything reaches the device"""
    from vid2player3d_b200.tasks import HumanoidSMPLIMVis
    a = dict(motion_assets=[ASSET] * 2, test_motion_assets=[ASSET] * 3, test_motion_file=str(tmp_path / "none.npz"))
    with pytest.raises(ValueError, match="b200_motion_queue_repeats"):
        HumanoidSMPLIMVis(qcfg(4, None, b200_motion_queue_repeats=0, **a), None, 1, "cuda", 0, True)
    with pytest.raises(ValueError, match="needs args.test or stateInit: Start"):
        HumanoidSMPLIMVis(qcfg(4, None, test=False, stateInit="Hybrid", **a), None, 1, "cuda", 0, True)


def test_each_distinct_asset_file_is_loaded_once(monkeypatch):
    """a 2000-entry list of three files: three loads, three packs of a distinct file"""
    from vid2player3d_b200 import model_compiler
    from vid2player3d_b200.tasks.humanoid_smpl_im import HumanoidSMPLIM
    loads, packs = [], []
    real_load = model_compiler.load_compiled
    monkeypatch.setattr(model_compiler, "load_compiled", lambda name: loads.append(name) or real_load(name))
    t = HumanoidSMPLIM.__new__(HumanoidSMPLIM)
    files = [ASSET, "mjcf/smpl_mesh_humanoid_federer.xml", "mjcf/smpl_mesh_humanoid_djokovic.xml"]
    entries = [files[i % 3] for i in range(2000)]
    t.cfg = dict(env=dict(motion_assets=entries))
    t.kp_scale = t.kd_scale = 1.0
    t._motion_lib = types.SimpleNamespace(num_motions=lambda: len(entries))
    real_pack = HumanoidSMPLIM._pack
    t._pack = lambda m: packs.append(1) or real_pack(t, m)
    models, of_motion = t._motion_asset_models()
    assert sorted(loads) == sorted(os.path.splitext(os.path.basename(f))[0] for f in files) and len(packs) == 3
    assert len(models) == 3 and of_motion.tolist() == [i % 3 for i in range(2000)]


# ---------------------------------------------------------------------------------------------------------- the recording
def fake_recorder(tmp_path, queue):
    t = V.HumanoidSMPLIMVis.__new__(V.HumanoidSMPLIMVis)
    E, T, nq = 2, 4, 7 + 69
    t.dt, t.num_dof = 1 / 30, 69
    t._rec = dict(qpos=torch.zeros(E, T + 2, 2, nq), env_ids=torch.tensor([0, 3]), rec_motion_ids=torch.tensor([[0, 0, 2, 2, 1, 1], [1, 3, 3, 0, 0, 0]]),
                  rec_reset=torch.zeros(E, T + 2, dtype=torch.long), frame=torch.tensor([T]))
    t._rec_cap, t._rec_assets, t._rec_path = T + 2, ["a.xml", "b.xml"], str(tmp_path / "rec.npz")
    if queue:
        t._rec_motion_asset = np.array(["a.xml", "b.xml", "c.xml", "a.xml"])
    return t


def test_the_recording_names_each_frames_body_with_the_queue(tmp_path, capsys):
    got = np.load(fake_recorder(tmp_path, True).export_recording())
    assert got["asset"].shape == (2, 4) and got["asset"].tolist() == [["a.xml", "a.xml", "c.xml", "c.xml"], ["b.xml", "a.xml", "a.xml", "a.xml"]]
    got = np.load(fake_recorder(tmp_path, False).export_recording())
    assert got["asset"].tolist() == ["a.xml", "b.xml"]                          # without the queue: one body per env, as before


# ---------------------------------------------------------------------------------------------------------- the C ABI
def test_descriptor_layouts_match_the_header(tmp_path):
    lines, want = [], []
    for ctype, S in (("b200_set_env_assets_t", abi.SetEnvAssets), ("b200_im_motion_queue_t", abi.ImMotionQueue)):
        lines.append(f'printf("{ctype} %zu\\n", sizeof({ctype}));')
        want.append(f"{ctype} {C.sizeof(S)}")
        for f, ct in S._fields_:
            lines.append(f'printf("{ctype}.{f} %zu %zu\\n", offsetof({ctype}, {f}), sizeof((({ctype}*)0)->{f}));')
            want.append(f"{ctype}.{f} {getattr(S, f).offset} {getattr(S, f).size}")
            if ct is abi.I32P:
                lines.append(f'printf("{ctype}.{f} %d\\n", __builtin_types_compatible_p(__typeof__(*(({ctype}*)0)->{f}), int32_t));')
                want.append(f"{ctype}.{f} 1")
    src, exe = tmp_path / "layout.c", tmp_path / "layout"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "b200env.h"\nint main(void) {\n' + "\n".join(lines) + "\nreturn 0;\n}\n")
    subprocess.check_call(["gcc", "-w", "-I", os.path.join(test_host.ROOT, "include"), str(src), "-o", str(exe)])
    assert subprocess.check_output([str(exe)], text=True).splitlines() == want
    assert abi.ImMotionQueue.motion_asset.offset == 136 and C.sizeof(abi.ImMotionQueue) == 152 and C.sizeof(abi.SetEnvAssets) == 24


def test_signatures_exports_and_descriptor_sizes():
    assert test_host.signature_mismatches(abi.SIGNATURES, test_host.ENV_HEADERS) == []
    for name in ("b200env_fix_mixed_plan", "b200env_set_env_assets", "b200env_set_env_assets_desc_size"):
        assert name in abi.SIGNATURES
    L = native.lib()
    for name in ("b200env_fix_mixed_plan", "b200env_set_env_assets", "b200env_set_env_assets_desc_size"):
        assert hasattr(L, name)
    assert L.b200env_set_env_assets_desc_size() == C.sizeof(abi.SetEnvAssets)
    assert L.b200env_im_motion_queue_desc_size() == C.sizeof(abi.ImMotionQueue)


@pytest.mark.parametrize("cls", ["SetEnvAssets", "ImMotionQueue"])
def test_binding_refuses_a_library_of_another_descriptor_size(monkeypatch, cls):
    native.lib()
    S = getattr(abi, cls)
    monkeypatch.setattr(abi, cls, type(cls, (C.Structure,), {"_fields_": S._fields_[:-1]}))
    monkeypatch.setattr(native, "_lib", None)
    with pytest.raises(RuntimeError, match=f"{cls} descriptor.*rebuild"):
        native.lib()


def test_null_handle_and_descriptor_are_refused():
    L = native.lib()
    assert L.b200env_fix_mixed_plan(None) == -1
    d = abi.SetEnvAssets(n=4, env_asset=0x10000, error=0x10000)
    assert L.b200env_set_env_assets(None, C.byref(d), None) == -1
    assert "b200env_set_env_assets: null argument" in L.b200env_last_error().decode()


def fake_queue(**over):
    d = abi.ImMotionQueue(n=4, num_motions=3, queue_len=6, shape_dim=11)
    for name, ct in abi.ImMotionQueue._fields_:
        if issubclass(ct, C.c_void_p):
            setattr(d, name, over.get(name, 0x10000))
    return d


@pytest.mark.parametrize("null", ["motion_asset", "env_asset"])
def test_the_queue_launch_needs_both_asset_pointers(null):
    """refused on fake device addresses, before the launch"""
    assert native.lib().b200env_im_motion_queue(C.byref(fake_queue(**{null: None})), None) == -1
    assert "motion_asset and env_asset must be both set or both NULL" in native.lib().b200env_last_error().decode()


class OnDevice:
    def __init__(self, t):
        self.t, self.dtype = t, t.dtype

    def is_contiguous(self):
        return True

    def get_device(self):
        return 0

    def data_ptr(self):
        return self.t.data_ptr()


@pytest.mark.parametrize("field", ["motion_asset", "env_asset"])
@pytest.mark.parametrize("dtype", [torch.int64, torch.float32, torch.uint8])
def test_fill_refuses_a_wrong_dtype_for_the_asset_arrays(field, dtype):
    S = abi.ImMotionQueue
    ptrs = {f: OnDevice(torch.zeros(2, dtype={abi.F32P: torch.float32, abi.I64P: torch.int64, abi.U8P: torch.uint8,
                                              abi.I32P: torch.int32}[ct]))
            for f, ct in S._fields_ if issubclass(ct, C.c_void_p)}
    d = native.fill(S, dict(n=4, num_motions=3, queue_len=6, shape_dim=11), ptrs)
    assert d.motion_asset.value == ptrs["motion_asset"].data_ptr() and d.env_asset.value == ptrs["env_asset"].data_ptr()
    with pytest.raises(ValueError, match=rf"ImMotionQueue\.{field}: {dtype}, the header's pointee needs torch\.int32"):
        native.fill(S, dict(n=4, num_motions=3, queue_len=6, shape_dim=11), dict(ptrs, **{field: OnDevice(torch.zeros(2, dtype=dtype))}))
    with pytest.raises(ValueError, match=rf"SetEnvAssets\.env_asset: {dtype}"):
        native.fill(abi.SetEnvAssets, dict(n=2), dict(env_asset=OnDevice(torch.zeros(2, dtype=dtype)), error=ptrs["env_flags"]))
    e = native.fill(S, dict(n=4, num_motions=3, queue_len=6, shape_dim=11), {k: v for k, v in ptrs.items() if k not in ("motion_asset", "env_asset")})
    assert e.motion_asset.value is None and e.env_asset.value is None       # the parent's launch
