"""Golden fixture for the context window's transforms: the reference's own `HumanoidSMPLIM._transform_target`
(embodied_pose/env/tasks/humanoid_smpl_im.py:565-592) EXECUTED on a fake `self`, on CPU, with `torch.bernoulli` and `torch.randn_like`
patched to return recorded draws (Bernoulli = recorded uniform < prob) and scipy's `norm.cdf` as the reference ships it.

Run in the build container only (needs /root/reference):  python tests/golden/make_golden_transforms.py
Output: tests/golden/im_transforms.npz (committed): per case the specs (JSON), the uniforms of noisy_joints (u0) and
mask_random_joints (u4), the normals, and the reference's body_pos and joint_conf.  Cases: each transform alone, all six orders of the
three, prob 0 and 1 of both random transforms, min_conf 0 and 1, and a min_conf equal to one joint's float32 confidence (the
occlusion threshold met exactly: that joint is kept).
"""
import itertools
import json
import os
import sys
from unittest import mock

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
import make_golden as G  # noqa: E402  (sets up the reference import harness)

SHAPE = (3, 4, 24)      # envs, frames, bodies
MASK = {'joints': ['L_Knee', 'R_Wrist', 'Head', 'Pelvis']}
NOISY = {'prob': 0.5, 'noise_std': 0.05, 'conf_std': 0.04, 'min_conf': 0.3}
RANDOM = {'prob': 0.3}
PARTS = {'mask_joints': MASK, 'noisy_joints': NOISY, 'mask_random_joints': RANDOM}


def cases():
    out = [(k, {k: v}) for k, v in PARTS.items()]
    short = {'mask_joints': 'mask', 'noisy_joints': 'noisy', 'mask_random_joints': 'random'}
    out += [("order_" + "_".join(short[k] for k in perm), {k: PARTS[k] for k in perm})
            for perm in itertools.permutations(PARTS)]
    out += [("noisy_prob0", {'noisy_joints': dict(NOISY, prob=0.0)}), ("noisy_prob1", {'noisy_joints': dict(NOISY, prob=1.0)}),
            ("random_prob0", {'mask_random_joints': {'prob': 0.0}}), ("random_prob1", {'mask_random_joints': {'prob': 1.0}}),
            ("noisy_minconf0", {'noisy_joints': dict(NOISY, min_conf=0.0)}), ("noisy_minconf1", {'noisy_joints': dict(NOISY, min_conf=1.0)}),
            ("noisy_then_mask_prob1", {'noisy_joints': dict(NOISY, prob=1.0), 'mask_joints': MASK})]
    return out


def run(specs, body_names, pos, u0, u4, z):
    t = G.FakeTask()
    t.cfg = {'env': {'transform_specs': specs}}
    t.body_names = body_names
    queue = [{'noisy_joints': u0, 'mask_random_joints': u4}[k] for k in specs if k != 'mask_joints']   # bernoulli's calls in order

    def bernoulli(p, *a, **kw):
        return torch.from_numpy((queue.pop(0) < p.numpy()).astype(np.float32))

    def randn_like(x, *a, **kw):
        return torch.from_numpy(z.astype(np.float32))

    ctx = {'body_pos': torch.from_numpy(pos.copy()), 'body_rot': None}
    with mock.patch.object(torch, "bernoulli", bernoulli), mock.patch.object(torch, "randn_like", randn_like):
        G.H.HumanoidSMPLIM._transform_target(t, ctx)
    assert not queue
    return ctx['body_pos'].numpy(), ctx['joint_conf'].numpy()


def main():
    model = G.model_compiler.load_compiled("smpl_mesh_humanoid_amass_v1")
    body_names = [str(x) for x in model["body_names"]]
    rng = np.random.default_rng(31)
    rec = {"body_names": np.array(body_names), "case_names": []}
    for name, specs in cases():
        pos = rng.normal(0, 0.5, SHAPE + (3,)).astype(np.float32)
        u0 = rng.random(SHAPE, np.float32)
        u4 = rng.random(SHAPE, np.float32)
        z = rng.normal(0, 1, SHAPE + (3,)).astype(np.float32)
        bp, conf = run(specs, body_names, pos, u0, u4, z)
        rec["case_names"].append(name)
        rec.update({f"{name}_specs": np.array(json.dumps(specs)), f"{name}_pos": pos, f"{name}_u0": u0, f"{name}_u4": u4, f"{name}_z": z,
                    f"{name}_body_pos": bp, f"{name}_conf": conf})
    # the occlusion threshold met exactly: min_conf = the float32 confidence of one noised joint, which the reference keeps
    name, specs = "noisy_exact_threshold", {'noisy_joints': dict(NOISY, prob=1.0, min_conf=0.0)}
    pos = rng.normal(0, 0.5, SHAPE + (3,)).astype(np.float32)
    u0, u4, z = rng.random(SHAPE, np.float32), rng.random(SHAPE, np.float32), rng.normal(0, 1, SHAPE + (3,)).astype(np.float32)
    _, conf = run(specs, body_names, pos, u0, u4, z)
    specs = {'noisy_joints': dict(NOISY, prob=1.0, min_conf=float(np.sort(conf.ravel())[conf.size // 2]))}
    bp, conf2 = run(specs, body_names, pos, u0, u4, z)
    assert (conf2 == np.float32(specs['noisy_joints']['min_conf'])).any()
    rec["case_names"].append(name)
    rec.update({f"{name}_specs": np.array(json.dumps(specs)), f"{name}_pos": pos, f"{name}_u0": u0, f"{name}_u4": u4, f"{name}_z": z,
                f"{name}_body_pos": bp, f"{name}_conf": conf2})
    rec["case_names"] = np.array(rec["case_names"])
    G.npz("im_transforms.npz", **rec)


if __name__ == "__main__":
    main()
