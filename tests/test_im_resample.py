"""CPU checks of the training resample of HumanoidSMPLIM (cfg.env.b200_resample_motions, b200_hard_motion_share): the restatement
(oracle/ref_port_motion_resample.py) on hand-built sequences, the cfg refusals, and the C ABI of b200_resample_motions_t and
b200_motion_weights_t."""
import ctypes as C
import os
import subprocess
import types

import numpy as np
import pytest
import torch

import test_host
from helpers import im_cfg
from oracle import ref_port_motion_resample as R
from oracle.ref_port_v2p import counter_hash
from test_im_motion_queue_assets import OnDevice
from vid2player3d_b200 import abi, native
from vid2player3d_b200.tasks.humanoid_smpl_im import motion_resample_share


# ---------------------------------------------------------------------------------------------------------- the restatement
def test_h0_gives_the_base_cdf_and_counts_nothing():
    r = R.Resampler(np.ones(4), 0.0, seed=10)
    assert np.array_equal(r.cdf, [0.25, 0.5, 0.75, 1.0])
    ids, drew = r.resample([0, 1, 2], np.ones(3, bool), [3, 3, 3], [1, 0, 1])
    assert drew.all() and not r.tries.any() and not r.fails.any() and r.counter == 1
    r.rebuild()
    assert np.array_equal(r.cdf, [0.25, 0.5, 0.75, 1.0])


def test_length_weights():
    lengths = np.array([1.0, 3.0, 0.0, 4.0], np.float32)
    b = R.base_weights(lengths, True)
    assert np.array_equal(b, [1.0, 3.0, 0.0, 4.0]) and np.array_equal(R.base_weights(lengths, False), np.ones(4))
    cdf = R.Resampler(b, 0.0, 1).cdf
    assert np.array_equal(cdf, [0.125, 0.5, 0.5, 1.0])
    assert R.draw(cdf, [0.0, 0.124, 0.125, 0.4999, 0.5, 0.99]).tolist() == [0, 0, 1, 1, 3, 3]     # motion 2 has no weight


def test_the_draw_follows_the_counter_based_bits():
    """u_e from the 53 high bits of counter_bits(seed', c, e); seed' is the re-keyed seed, so the keys differ from the masked reset's"""
    seed, c, n = 10, 7, 50
    u = R.uniforms(seed, c, n)
    sp = R.resample_seed(seed)
    assert np.array_equal(u, (counter_hash(sp, c, np.arange(n)) >> np.uint64(11)).astype(np.float64) * 2.0 ** -53)
    assert (u >= 0).all() and (u < 1).all()
    reset_keys = set(counter_hash(seed, c, np.arange(2 * n)).tolist())
    assert not reset_keys & set(R.counter_bits(sp, c, np.arange(n)).tolist())
    assert not np.array_equal(R.uniforms(seed, c + 1, n), u) and not np.array_equal(R.uniforms(seed + 1, c, n), u)


def test_envs_that_played_no_step_are_not_drawn_or_counted():
    r = R.Resampler(np.ones(3), 0.5, seed=4)
    ids = np.array([0, 1, 2, 1])
    new, drew = r.resample(ids, np.array([1, 1, 0, 1], bool), [0, 2, 5, 1], [1, 1, 1, 0])
    assert drew.tolist() == [False, True, False, True]
    assert new[0] == 0 and new[2] == 2
    assert r.tries.tolist() == [0, 2, 0] and r.fails.tolist() == [0, 1, 0]


def test_the_rebuild_keeps_the_rate_of_an_unseen_motion():
    r = R.Resampler(np.ones(3), 0.5, seed=4)
    r.tries[:] = [4, 0, 2]
    r.fails[:] = [1, 0, 2]
    r.rebuild()
    assert r.rate.tolist() == [0.25, 1.0, 1.0] and not r.tries.any() and not r.fails.any()
    p = 0.5 / 3 + 0.5 * np.array([0.25, 1.0, 1.0]) / 2.25
    assert np.allclose(r.cdf, np.cumsum(p), rtol=0, atol=1e-15)
    r.tries[:] = [0, 5, 0]
    r.fails[:] = [0, 0, 0]
    r.rebuild()
    assert r.rate.tolist() == [0.25, 0.0, 1.0]           # motion 1 tried 5 times without a fall; 0 and 2 keep theirs


def test_no_failures_at_all_falls_back_to_the_base():
    r = R.Resampler(np.array([1.0, 2.0, 1.0]), 0.7, seed=4)
    r.tries[:] = [3, 1, 2]
    r.rebuild()
    assert r.rate.tolist() == [0.0, 0.0, 0.0] and np.array_equal(r.cdf, np.cumsum([0.25, 0.5, 0.25]))


def test_h1_draws_only_motions_that_failed():
    r = R.Resampler(np.ones(6), 1.0, seed=9)
    r.tries[:] = [1, 1, 1, 1, 1, 1]
    r.fails[:] = [0, 1, 0, 0, 1, 0]
    r.rebuild()
    new, _ = r.resample(np.zeros(4000, np.int64), np.ones(4000, bool), np.ones(4000), np.zeros(4000))
    assert set(new.tolist()) == {1, 4}


def test_one_motion_always_draws_it():
    r = R.Resampler(np.ones(1), 0.3, seed=1)
    new, _ = r.resample(np.zeros(9, np.int64), np.ones(9, bool), np.ones(9), np.ones(9))
    assert not new.any() and r.tries.tolist() == [9] and r.fails.tolist() == [9]


# ---------------------------------------------------------------------------------------------------------- cfg refusals
def rcfg(test=False, **over):
    cfg = im_cfg(4, None, **dict(dict(b200_resample_motions=True), **over))
    cfg["args"] = types.SimpleNamespace(test=test)
    return cfg


def test_the_key_is_off_by_default_and_h_defaults_to_zero():
    assert motion_resample_share(im_cfg(4, None)) is None
    assert motion_resample_share(rcfg()) == 0.0
    assert motion_resample_share(rcfg(b200_hard_motion_share=0.5)) == 0.5
    assert motion_resample_share(rcfg(b200_hard_motion_share=1)) == 1.0
    assert motion_resample_share(rcfg(sample_first_motions=True)) == 0.0


@pytest.mark.parametrize("over,match", [
    (dict(test=True), "a test run keeps each env's motion"),
    (dict(b200_motion_queue=True), "set one of them"),
    (dict(motion_id=3), "motion_id pins every env"),
    (dict(b200_hard_motion_share=-0.1), r"finite number in \[0, 1\]"),
    (dict(b200_hard_motion_share=1.5), r"finite number in \[0, 1\]"),
    (dict(b200_hard_motion_share=float("nan")), r"finite number in \[0, 1\]"),
    (dict(b200_hard_motion_share=float("inf")), r"finite number in \[0, 1\]"),
    (dict(b200_hard_motion_share="0.5"), r"finite number in \[0, 1\]"),
    (dict(b200_hard_motion_share=True), r"finite number in \[0, 1\]"),
    (dict(b200_hard_motion_share=None), r"finite number in \[0, 1\]"),
])
def test_refusals(over, match):
    with pytest.raises(ValueError, match=match):
        motion_resample_share(rcfg(**over))


def test_the_share_without_the_key_is_refused():
    cfg = im_cfg(4, None, b200_hard_motion_share=0.3)
    with pytest.raises(ValueError, match="set b200_resample_motions: True"):
        motion_resample_share(cfg)


def test_the_tasks_refuse_before_anything_reaches_the_device():
    """the refusals come first in the constructors: no library is loaded and no tensor is made"""
    from vid2player3d_b200.tasks import HumanoidSMPLIM, HumanoidSMPLIMVis
    with pytest.raises(ValueError, match="a test run keeps each env's motion"):
        HumanoidSMPLIMVis(rcfg(), None, 1, "cuda", 0, True)
    with pytest.raises(ValueError, match="a test run keeps each env's motion"):
        HumanoidSMPLIM(rcfg(test=True), None, 1, "cuda", 0, True)
    with pytest.raises(ValueError, match="set one of them"):
        HumanoidSMPLIM(rcfg(b200_motion_queue=True), None, 1, "cuda", 0, True)
    with pytest.raises(ValueError, match=r"finite number in \[0, 1\]"):
        HumanoidSMPLIM(rcfg(b200_hard_motion_share=2.0), None, 1, "cuda", 0, True)
    with pytest.raises(ValueError, match="set b200_resample_motions: True"):
        HumanoidSMPLIM(im_cfg(4, None, b200_hard_motion_share=0.3), None, 1, "cuda", 0, True)


# ---------------------------------------------------------------------------------------------------------- the C ABI
STRUCTS = (("b200_resample_motions_t", abi.ResampleMotions), ("b200_motion_weights_t", abi.MotionWeights))


def test_descriptor_layouts_match_the_header(tmp_path):
    lines, want = [], []
    pointee = {abi.I32P: "int32_t", abi.I64P: "int64_t", abi.F64P: "double", abi.F32P: "float", abi.U8P: "uint8_t", abi.U32P: "uint32_t"}
    for ctype, S in STRUCTS:
        lines.append(f'printf("{ctype} %zu\\n", sizeof({ctype}));')
        want.append(f"{ctype} {C.sizeof(S)}")
        for f, ct in S._fields_:
            lines.append(f'printf("{ctype}.{f} %zu %zu\\n", offsetof({ctype}, {f}), sizeof((({ctype}*)0)->{f}));')
            want.append(f"{ctype}.{f} {getattr(S, f).offset} {getattr(S, f).size}")
            if ct in pointee:
                lines.append(f'printf("{ctype}.{f} %d\\n", __builtin_types_compatible_p(__typeof__(*(({ctype}*)0)->{f}), {pointee[ct]}));')
                want.append(f"{ctype}.{f} 1")
    src, exe = tmp_path / "layout.c", tmp_path / "layout"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "b200env.h"\nint main(void) {\n' + "\n".join(lines) + "\nreturn 0;\n}\n")
    subprocess.check_call(["gcc", "-w", "-I", os.path.join(test_host.ROOT, "include"), str(src), "-o", str(exe)])
    assert subprocess.check_output([str(exe)], text=True).splitlines() == want
    assert C.sizeof(abi.ResampleMotions) == 128 and C.sizeof(abi.MotionWeights) == 56


def test_signatures_exports_and_descriptor_sizes():
    assert test_host.signature_mismatches(abi.SIGNATURES, test_host.ENV_HEADERS) == []
    L = native.lib()
    for name in ("b200env_resample_motions", "b200env_resample_motions_desc_size", "b200env_motion_weights",
                 "b200env_motion_weights_desc_size"):
        assert name in abi.SIGNATURES and hasattr(L, name)
    assert L.b200env_resample_motions_desc_size() == C.sizeof(abi.ResampleMotions)
    assert L.b200env_motion_weights_desc_size() == C.sizeof(abi.MotionWeights)


@pytest.mark.parametrize("cls", ["ResampleMotions", "MotionWeights"])
def test_binding_refuses_a_library_of_another_descriptor_size(monkeypatch, cls):
    native.lib()
    S = getattr(abi, cls)
    monkeypatch.setattr(abi, cls, type(cls, (C.Structure,), {"_fields_": S._fields_[:-1]}))
    monkeypatch.setattr(native, "_lib", None)
    with pytest.raises(RuntimeError, match=f"{cls} descriptor.*rebuild"):
        native.lib()


def fake(S, scalars, **over):
    d = S(**scalars)
    for name, ct in S._fields_:
        if issubclass(ct, C.c_void_p):
            setattr(d, name, over.get(name, 0x10000))
    return d


RS = dict(n=4, num_motions=3, shape_dim=11, seed=10)


@pytest.mark.parametrize("null", ["mask", "progress_buf", "terminate_buf", "cdf", "lib_motion_bodies", "motion_ids", "motion_bodies",
                                  "counter", "done", "tries", "fails", "motion_asset", "env_asset"])
def test_the_sampler_refuses_a_null_or_half_a_pair(null):
    """refused on fake device addresses, before any launch; tries / fails and motion_asset / env_asset are pairs"""
    L = native.lib()
    assert L.b200env_resample_motions(C.byref(fake(abi.ResampleMotions, RS, **{null: None})), None) == -1
    assert L.b200env_resample_motions(None, None) == -1


@pytest.mark.parametrize("over", [dict(n=0), dict(n=-3), dict(num_motions=0), dict(shape_dim=-1), dict(shape_dim=33)])
def test_the_sampler_refuses_sizes_before_launching(over):
    L = native.lib()
    assert L.b200env_resample_motions(C.byref(fake(abi.ResampleMotions, dict(RS, **over))), None) == -2


def test_the_weights_launch_refusals():
    L = native.lib()
    W = abi.MotionWeights
    for h in (-0.5, 1.5, float("nan"), float("inf")):
        assert L.b200env_motion_weights(C.byref(fake(W, dict(num_motions=3, h=h))), None) == -2
    assert "h must be a finite number in [0, 1]" in L.b200env_last_error().decode()
    assert L.b200env_motion_weights(C.byref(fake(W, dict(num_motions=0, h=0.0))), None) == -2
    assert L.b200env_motion_weights(C.byref(fake(W, dict(num_motions=3, h=0.0), cdf=None)), None) == -1
    for null in ("tries", "fails", "rate"):
        assert L.b200env_motion_weights(C.byref(fake(W, dict(num_motions=3, h=0.5), **{null: None})), None) == -1


def _on_device(S):
    dt = {abi.F32P: torch.float32, abi.I64P: torch.int64, abi.U8P: torch.uint8, abi.I32P: torch.int32, abi.F64P: torch.float64,
          abi.U32P: torch.int32}
    return {f: OnDevice(torch.zeros(2, dtype=dt[ct])) for f, ct in S._fields_ if issubclass(ct, C.c_void_p)}


@pytest.mark.parametrize("field,dtype", [("cdf", torch.float32), ("progress_buf", torch.int32), ("terminate_buf", torch.float32),
                                         ("motion_ids", torch.int32), ("motion_bodies", torch.float64), ("tries", torch.int32),
                                         ("motion_asset", torch.int64), ("env_asset", torch.int64), ("counter", torch.int32),
                                         ("mask", torch.int64)])
def test_fill_refuses_a_wrong_dtype_for_the_sampler(field, dtype):
    S, ptrs = abi.ResampleMotions, _on_device(abi.ResampleMotions)
    d = native.fill(S, RS, ptrs)
    assert d.cdf.value == ptrs["cdf"].data_ptr()
    with pytest.raises(ValueError, match=rf"ResampleMotions\.{field}: {dtype}"):
        native.fill(S, RS, dict(ptrs, **{field: OnDevice(torch.zeros(2, dtype=dtype))}))
    e = native.fill(S, RS, {k: v for k, v in ptrs.items() if k not in ("tries", "fails", "motion_asset", "env_asset")})
    assert e.tries.value is None and e.env_asset.value is None


@pytest.mark.parametrize("field,dtype", [("base", torch.float64), ("rate", torch.float32), ("cdf", torch.float32), ("fails", torch.int32)])
def test_fill_refuses_a_wrong_dtype_for_the_weights(field, dtype):
    S, ptrs = abi.MotionWeights, _on_device(abi.MotionWeights)
    native.fill(S, dict(num_motions=3, h=0.5), ptrs)
    with pytest.raises(ValueError, match=rf"MotionWeights\.{field}: {dtype}"):
        native.fill(S, dict(num_motions=3, h=0.5), dict(ptrs, **{field: OnDevice(torch.zeros(2, dtype=dtype))}))
    with pytest.raises(ValueError, match=r"MotionWeights\.cdf: None"):
        native.fill(S, dict(num_motions=3, h=0.0), dict(base=None))
