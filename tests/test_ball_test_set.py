"""CPU checks of the fixed test set of incoming balls (cfg.env.ball_traj_file_test): the restatement oracle/ref_port_test_set.py against
tests/golden/v2p_ball_test_set.npz (made by executing the reference's TennisBallGeneratorOffline and player_builder rule,
tests/golden/make_golden_test_set.py), the cfg resolution of PhysicsMVAEController and HumanoidSMPLIMMVAE with its refusals, and the
C ABI of b200v2p_treset_t's pool_cursor."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
import torch

import test_host
from conftest import golden
from oracle import ref_port_test_set as T
from vid2player3d_b200 import abi, native
from vid2player3d_b200.tasks.humanoid_smpl_im_mvae import resolve_ball_pool
from vid2player3d_b200.tasks.physics_mvae_controller import resolve_test_set

Z = golden("v2p_ball_test_set.npz")


@pytest.mark.parametrize("case", [str(c) for c in Z["cases"]])
def test_oracle_is_the_reference_generator(case):
    """indices, trajectories and launch states of every call, and the cursors after the last one, exactly"""
    g = lambda k: Z[f"{case}_{k}"]  # noqa: E731
    pool, lens = g("pool"), g("lens")
    cursor = np.zeros(int(g("num_envs")), np.int64)
    got = {k: [] for k in ("index", "traj", "launch_pos", "launch_vel", "launch_vspin")}
    start = np.concatenate([[0], np.cumsum(lens)])
    for a, b in zip(start[:-1], start[1:]):
        for k, v in zip(got, T.generate(pool, cursor, g("env_ids")[a:b])):
            got[k].append(v)
    for k, v in got.items():
        np.testing.assert_array_equal(np.concatenate(v), g(k), f"{case}: {k}")
    np.testing.assert_array_equal(cursor, g("cursor"), f"{case}: cursor")


def test_fixture_covers_its_edges():
    """repeated envs across calls, a wrap at P, P = 1, P > N, and start positions on the far side (which the random branch remaps)"""
    assert int(Z["one_row_pool"].shape[0]) == 1 and Z["pool_larger_pool"].shape[0] > int(Z["pool_larger_num_envs"])
    for case in Z["cases"]:
        ids, idx = Z[f"{case}_env_ids"], Z[f"{case}_index"]
        assert len(np.unique(ids)) < len(ids) and (Z[f"{case}_start_pos"][:, 1] > 0).any()
        P = Z[f"{case}_pool"].shape[0]
        if P > 1:       # some env comes back to row 0 after row P - 1
            assert any((idx[ids == e][1:] < idx[ids == e][:-1]).any() for e in np.unique(ids)), case


def test_mode_rule_is_player_builders():
    for name, mode in zip(Z["file_names"], Z["test_modes"]):
        assert T.mode_of(str(name)) == str(mode)
        env, v2p = dict(ball_traj_file_test=str(name)), dict(player="federer")
        resolve_test_set(env, v2p)
        assert v2p == dict(player="federer", ball_traj_file_test=str(name), test_mode=str(mode))


@pytest.mark.parametrize("value", [None, ""])
def test_mode_rule_leaves_the_cfg_alone_without_the_key(value):
    env, v2p = dict(ball_traj_file_test=value) if value is not None else {}, dict(player="federer", test_mode="random")
    resolve_test_set(env, v2p)
    assert v2p == dict(player="federer", test_mode="random")


# ------------------------------------------------------------------------------------------------ pool resolution
def _pool(P, seed):
    return np.random.default_rng(seed).uniform(-20, 20, (P, 307)).astype(np.float32)


@pytest.mark.parametrize("dual", [False, True])
@pytest.mark.parametrize("source", ["file", "array", "missing_file", "none"])
@pytest.mark.parametrize("mode", [None, "random", "single_cycle", "multiple_cycle"])
@pytest.mark.parametrize("is_train", [True, False])
def test_pool_resolution(tmp_path, is_train, mode, source, dual):
    """:121-130: training or test_mode random -> the training pool, drawn at random; test time with a cycle mode -> the test set, in
    order; a test set that is not there is refused with the reason; dual mode builds no pool and ignores the keys"""
    train, test = _pool(5, 1), _pool(3, 2)
    v2p = dict(ball_pool=train)
    if mode is not None:
        v2p["test_mode"] = mode
    if dual:
        v2p["dual_mode"] = "different"
    if source == "file":
        np.save(tmp_path / "test_single.npy", test)
        v2p["ball_traj_file_test"] = str(tmp_path / "test_single.npy")
    elif source == "array":
        v2p["ball_pool_test"] = test
    elif source == "missing_file":
        v2p["ball_traj_file_test"] = str(tmp_path / "absent.npy")
    sequential = not is_train and mode in ("single_cycle", "multiple_cycle") and not dual
    if sequential and source == "missing_file":
        with pytest.raises(ValueError, match=r"ball_traj_file_test '.*absent\.npy' does not exist"):
            resolve_ball_pool(v2p, is_train)
        return
    if sequential and source == "none":
        with pytest.raises(ValueError, match="neither ball_traj_file_test nor ball_pool_test is given"):
            resolve_ball_pool(v2p, is_train)
        return
    pool, seq = resolve_ball_pool(v2p, is_train)
    assert seq == sequential
    if dual:
        assert pool is None
    else:
        np.testing.assert_array_equal(pool, test if sequential else train)
        assert pool.dtype == np.float32


def test_training_pool_file_and_fallback_are_unchanged(tmp_path):
    train = _pool(4, 3)
    np.save(tmp_path / "train.npy", train)
    pool, seq = resolve_ball_pool(dict(ball_traj_file=str(tmp_path / "train.npy")), False)
    np.testing.assert_array_equal(pool, train)
    assert not seq
    pool, seq = resolve_ball_pool(dict(ball_traj_file=str(tmp_path / "absent.npy")), True)   # the synthetic pool, as before
    assert pool.shape == (2048, 307) and not seq


@pytest.mark.parametrize("v2p, msg", [
    (dict(test_mode="single"), r"test_mode 'single': must be one of random, single_cycle, multiple_cycle"),
    (dict(test_mode="multiple_cycle", ball_pool_test=np.zeros((0, 307), np.float32)), r"must be \[P >= 1, 307\].*got \[0, 307\]"),
    (dict(test_mode="single_cycle", ball_pool_test=np.zeros((3, 306), np.float32)), r"must be \[P >= 1, 307\].*got \[3, 306\]"),
    (dict(test_mode="single_cycle", ball_pool_test=np.zeros(307, np.float32)), r"must be \[P >= 1, 307\].*got \[307\]"),
])
def test_refusals(v2p, msg):
    with pytest.raises(ValueError, match=msg):
        resolve_ball_pool(v2p, False)


# ------------------------------------------------------------------------------------------------ C ABI
def test_descriptor_layout_matches_the_header(tmp_path):
    """pool_cursor is appended behind obs_traj_len / pad_: the fields before it keep their offsets"""
    ctype, S = "b200v2p_treset_t", abi.V2PTaskReset
    lines = [f'printf("%zu %zu %zu %d\\n", sizeof({ctype}), offsetof({ctype}, pool_cursor), offsetof({ctype}, pad_), '
             f'__builtin_types_compatible_p(__typeof__(*(({ctype}*)0)->pool_cursor), int64_t));']
    src, exe = tmp_path / "layout.c", tmp_path / "layout"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "b200env_v2p.h"\nint main(void) {\n' + "\n".join(lines) +
                   "\nreturn 0;\n}\n")
    subprocess.check_call(["gcc", "-w", "-I", os.path.join(test_host.ROOT, "include"), str(src), "-o", str(exe)])
    size, off, pad, typed = map(int, subprocess.check_output([str(exe)], text=True).split())
    assert (size, off, pad, typed) == (C.sizeof(S), S.pool_cursor.offset, S.pad_.offset, 1)
    assert off == pad + 4 and size == off + 8
    assert dict(S._fields_)["pool_cursor"] is abi.I64P and "pool_cursor" in S._nullable_


def test_signatures_and_descriptor_size():
    assert test_host.signature_mismatches(abi.SIGNATURES, test_host.ENV_HEADERS) == []
    assert abi.SIGNATURES["b200v2p_task_reset_desc_size"] == (C.c_int32, [])
    assert native.lib().b200v2p_task_reset_desc_size() == C.sizeof(abi.V2PTaskReset)


def test_binding_refuses_a_library_of_another_descriptor_size(monkeypatch):
    """a library built before pool_cursor would launch the random draw on a test set: native.lib() refuses it"""
    native.lib()
    old = type("V2PTaskReset", (C.Structure,), {"_fields_": abi.V2PTaskReset._fields_[:-1]})    # the layout before the field
    monkeypatch.setattr(abi, "V2PTaskReset", old)
    monkeypatch.setattr(native, "_lib", None)
    with pytest.raises(RuntimeError, match="V2PTaskReset descriptor.*rebuild"):
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


@pytest.mark.parametrize("with_cursor", [False, True])
def test_fill_writes_pool_cursor(with_cursor):
    S = abi.V2PTaskReset
    scalars = {f: ([1] * ct._length_ if issubclass(ct, C.Array) else 1) for f, ct in S._fields_
               if not issubclass(ct, C.c_void_p) and f not in S._defaults_}
    keep = {f: torch.zeros(2, dtype={abi.F32P: torch.float32, abi.I64P: torch.int64, abi.U8P: torch.bool}[ct]) for f, ct in S._fields_
            if issubclass(ct, C.c_void_p) and (f != "pool_cursor" or with_cursor)}
    d = native.fill(S, scalars, {f: _OnDevice(t) for f, t in keep.items()})
    assert d.pool_cursor.value == (keep["pool_cursor"].data_ptr() if with_cursor else None)
    assert d.pool.value == keep["pool"].data_ptr() and d.obs_traj_len == 0
    with pytest.raises(ValueError, match=r"^V2PTaskReset\.pool_cursor: torch\.int32, the header's pointee needs torch\.int64"):
        native.fill(S, scalars, dict({f: _OnDevice(t) for f, t in keep.items()}, pool_cursor=_OnDevice(torch.zeros(2, dtype=torch.int32))))
