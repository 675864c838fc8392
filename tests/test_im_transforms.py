"""The context window's transforms on the device (cfg.env.b200_device_transforms), CPU side: the float64 restatement against the
reference's own `_transform_target` (tests/golden/im_transforms.npz), the transform program's fields in the C ABI, and the cfg
refusals of abi.transform_program."""
import ctypes as C
import json
import os

import numpy as np
import pytest

import test_host
from conftest import golden
from oracle import ref_port_transforms as X
from vid2player3d_b200 import abi

G = golden("im_transforms.npz")
CASES = [str(c) for c in G["case_names"]]
NAMES = [str(x) for x in G["body_names"]]


def case(name):
    return dict(specs=json.loads(str(G[f"{name}_specs"])), pos=G[f"{name}_pos"], u0=G[f"{name}_u0"], u4=G[f"{name}_u4"], z=G[f"{name}_z"],
                body_pos=G[f"{name}_body_pos"], conf=G[f"{name}_conf"])


def near_threshold(specs, noisy, noise, tol=1e-6):
    """joints whose noise confidence lies within tol of min_conf: float32 and float64 may decide them either way"""
    if "noisy_joints" not in specs:
        return np.zeros(noisy.shape, bool)
    return np.abs(X.pre_occlusion_conf(specs, noisy, noise) - specs["noisy_joints"]["min_conf"]) < tol


def test_golden_covers_the_cases():
    orders = {tuple(case(c)["specs"]) for c in CASES if len(case(c)["specs"]) == 3}
    assert len(orders) == 6
    probs = {(k, s["prob"]) for c in CASES for k, s in case(c)["specs"].items() if "prob" in s}
    assert {("noisy_joints", 0.0), ("noisy_joints", 1.0), ("mask_random_joints", 0.0), ("mask_random_joints", 1.0)} <= probs
    conf = {s["min_conf"] for c in CASES for k, s in case(c)["specs"].items() if k == "noisy_joints"}
    assert {0.0, 1.0} <= conf
    ex = case("noisy_exact_threshold")
    m = np.float32(ex["specs"]["noisy_joints"]["min_conf"])
    assert (ex["conf"] == m).any(), "no joint's confidence equals min_conf: the threshold is not met exactly"


@pytest.mark.parametrize("name", CASES)
def test_oracle_equals_the_reference(name):
    c = case(name)
    specs = c["specs"]
    noisy = c["u0"] < np.float32(specs.get("noisy_joints", {}).get("prob", 0.0))
    drop = c["u4"] < np.float32(specs.get("mask_random_joints", {}).get("prob", 0.0))
    bp, conf = X.transform_target(c["pos"], specs, NAMES, noisy=noisy, noise=c["z"], drop=drop)
    keep = ~near_threshold(specs, noisy, c["z"])
    if name == "noisy_exact_threshold":
        assert (~keep).any(), "the exact threshold case has no joint at the threshold"
    np.testing.assert_allclose(bp[keep], c["body_pos"][keep], rtol=0, atol=1e-6)
    np.testing.assert_allclose(conf[keep], c["conf"][keep], rtol=0, atol=1e-6)


def test_noisy_before_mask_keeps_the_noise_confidence():
    """the reference's aliasing: after noisy_joints, mask_joints zeroes its joints' positions, keeps their noise confidence and
    scales no other joint"""
    c = case("noisy_then_mask_prob1")
    idx = [NAMES.index(j) for j in c["specs"]["mask_joints"]["joints"]]
    others = np.setdiff1d(np.arange(len(NAMES)), idx)
    assert (c["body_pos"][..., idx, :] == 0).all()
    assert (c["conf"][..., idx] > 0).any()
    moved = c["body_pos"][..., others, :] - c["pos"][..., others, :]
    kept = c["conf"][..., others] > 0
    assert np.abs(moved[kept]).max() < 0.5 and (np.abs(moved[kept]) > 0).any()


def test_restated_draw_keys():
    """draw k of (row e, frame j, body b) is 2 num_envs + ((e P + j) nb + b) 5 + k: consecutive, disjoint from the reset's 2e + k"""
    N, P, nb = 6, 4, 24
    base = X.draw_index(N, np.arange(N), P, nb)
    assert base.min() == 2 * N and np.array_equal(np.diff(base.reshape(-1)), np.full(N * P * nb - 1, 5))
    noisy, noise, drop = X.draws(10, 3, N, np.arange(N), P, nb, {"noisy_joints": {"prob": 0.5}, "mask_random_joints": {"prob": 0.5}})
    assert noisy.shape == drop.shape == (N, P, nb) and noise.shape == (N, P, nb, 3)
    n2, z2, d2 = X.draws(10, 3, N, np.arange(2, 4), P, nb, {"noisy_joints": {"prob": 0.5}, "mask_random_joints": {"prob": 0.5}})
    assert np.array_equal(n2, noisy[2:4]) and np.array_equal(z2, noise[2:4]) and np.array_equal(d2, drop[2:4])
    assert 0.4 < noisy.mean() < 0.6 and abs(noise.mean()) < 0.1 and not np.array_equal(noisy, drop)


def test_program_fields_are_32_bit_and_default_to_zero():
    for S in (abi.ResetMasked, abi.MotionContext):
        f = dict(S._fields_)
        assert f["xf_ops"]._type_ is C.c_int32 and f["xf_ops"]._length_ == 3 and f["xf_joint_mask"] is C.c_uint32
        for k in ("xf_noisy_prob", "xf_noise_std", "xf_conf_std", "xf_min_conf", "xf_random_prob"):
            assert f[k] is C.c_float, k
        assert f["feat_width"] is C.c_int32
        assert {n for n, _ in abi._XF_FIELDS} <= set(S._defaults_)
    f = dict(abi.MotionContext._fields_)
    assert f["seed"] is C.c_uint64 and f["counter"] is abi.I64P and "counter" in abi.MotionContext._nullable_
    text = open(os.path.join(test_host.ROOT, "include", "b200env.h")).read()
    for k, v in (("B200_XF_MASK_JOINTS", abi.XF_MASK_JOINTS), ("B200_XF_NOISY_JOINTS", abi.XF_NOISY_JOINTS),
                 ("B200_XF_MASK_RANDOM_JOINTS", abi.XF_MASK_RANDOM_JOINTS)):
        assert f"#define {k} {v}" in text


def test_library_reports_the_descriptor_sizes():
    """the descriptors grew within ABI version 11: the library's sizes equal the binding's (native.lib() refuses a mismatch)"""
    from vid2player3d_b200 import build, native
    L = C.CDLL(build.build())
    assert L.b200env_reset_masked_desc_size() == C.sizeof(abi.ResetMasked)
    assert L.b200env_motion_context_desc_size() == C.sizeof(abi.MotionContext)
    assert native.lib() is not None


def test_program_of_the_specs():
    specs = {"noisy_joints": {"prob": 0.25, "noise_std": 0.05, "conf_std": 0.04, "min_conf": 0.3},
             "mask_joints": {"joints": ["L_Knee", "Head"]}, "mask_random_joints": {"prob": 0.125}}
    p = abi.transform_program(specs, NAMES, 24)
    assert p["xf_ops"] == [abi.XF_NOISY_JOINTS, abi.XF_MASK_JOINTS, abi.XF_MASK_RANDOM_JOINTS]
    assert p["xf_joint_mask"] == (1 << NAMES.index("L_Knee")) | (1 << NAMES.index("Head"))
    assert (p["xf_noisy_prob"], p["xf_noise_std"], p["xf_conf_std"], p["xf_min_conf"], p["xf_random_prob"]) == (0.25, 0.05, 0.04, 0.3, 0.125)
    assert abi.transform_program({}, NAMES, 24)["xf_ops"] == [0, 0, 0]
    assert abi.transform_program({"mask_random_joints": {"prob": 1.0}}, NAMES, 24)["xf_ops"] == [abi.XF_MASK_RANDOM_JOINTS, 0, 0]


NOISY = {"prob": 0.5, "noise_std": 0.05, "conf_std": 0.04, "min_conf": 0.3}
REFUSED = [
    ({"blur_joints": {}}, "unknown transform 'blur_joints'"),
    ({"mask_joints": {"joints": ["L_Knee", "Tail"]}}, "'Tail' is not a body"),
    ({"mask_joints": {"joints": ["Racket"]}}, "'Racket' is not a body"),
    ({"noisy_joints": dict(NOISY, prob=1.5)}, r"prob 1.5 outside \[0, 1\]"),
    ({"noisy_joints": dict(NOISY, prob=-0.1)}, r"prob -0.1 outside \[0, 1\]"),
    ({"mask_random_joints": {"prob": float("nan")}}, r"prob nan outside \[0, 1\]"),
    ({"noisy_joints": dict(NOISY, conf_std=0.0)}, "conf_std 0.0 must be > 0"),
    ({"noisy_joints": dict(NOISY, noise_std=-0.01)}, "noise_std -0.01 < 0"),
    ({"noisy_joints": {"prob": 0.5}}, "missing 'noise_std'"),
    ({"mask_random_joints": {}}, "missing 'prob'"),
]


@pytest.mark.parametrize("specs,match", REFUSED, ids=[m.split(" ")[0].strip("'\\") + f"-{i}" for i, (_, m) in enumerate(REFUSED)])
def test_program_refuses(specs, match):
    with pytest.raises(ValueError, match=match):
        abi.transform_program(specs, NAMES + ["Racket"], 24)
