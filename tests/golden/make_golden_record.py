"""Golden fixture for the recorded viewer frame: the reference's own `HumanoidSMPLIMVis._sync_ref_motion`,
`convert_dof_pos_to_dof_euler` and `set_mj_actor_qpos` (embodied_pose/env/tasks/humanoid_smpl_im_vis.py:117-152) EXECUTED in float64
on a fake `self` whose `mj_data.qpos` is a numpy array, with mujoco_py, glfw, imageio, utils.mjviewer and utils.tools stubbed.

Run in the build container only (needs /root/reference):  python tests/golden/make_golden_record.py
Output: tests/golden/im_record.npz (committed): the state of N envs (rb_pos, rb_rot, dof_pos and the previous target's p_rb_pos,
p_rb_rot, p_dof_pos; the target root is the root row of p_rb_*) and, per env, the qpos [N, 3 nq] the reference leaves with init False
(qpos_init0) and True (qpos_init1).  The reference syncs env 0, so env e is synced as env 0 of its own slice.  Joints of the random
state are overwritten with the edge cases: a zero rotation vector, |theta| near pi, pitch at and near +-pi/2 (where the yaw and roll
arguments both fall below eps), and rotations of pi about x and z (the +-pi branch cut of atan2).

Also tests/golden/im_record_nonfinite.npz, the same keys for the joints and roots of a failing policy: rotation vectors with NaN in one,
two or three components, +-Inf and +-1e30 (finite, but its square overflows float32), a NaN root position and an Inf root quaternion.
The reference's torch.clamp keeps a NaN pitch.
"""
import os
import sys
import types
from unittest.mock import MagicMock

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
import _refenv  # noqa: E402

_refenv.setup("embodied_pose")
for name in ("mujoco_py", "glfw", "imageio", "utils.mjviewer", "utils.tools"):
    m = types.ModuleType(name)
    m.load_model_from_path = m.MjSim = m.MjViewer = m.create_vis_model_xml = MagicMock()
    sys.modules[name] = m

from env.tasks import humanoid_smpl_im_vis as V  # noqa: E402

N, NB, ND = 8, 24, 69
NQ = 7 + ND
PI = np.pi
EDGES = [(0.0, 0.0, 0.0), (PI - 1e-7, 0.0, 0.0), (0.0, 0.0, -(PI - 1e-6)), tuple(np.array([1.0, -2.0, 0.5]) / np.sqrt(5.25) * (PI - 1e-7)),
         (0.0, PI / 2, 0.0), (0.0, -PI / 2, 0.0), (0.0, PI / 2 - 1e-4, 0.0), (0.0, -PI / 2 + 3e-4, 0.0), (PI, 0.0, 0.0), (-PI, 0.0, 0.0),
         (0.0, 0.0, PI), (0.0, 0.0, -PI), (1e-5, 0.0, 0.0), (3e-4, -2e-4, 1e-4)]


NAN, INF = float("nan"), float("inf")
NONFINITE = [(NAN, 0.3, -0.2), (0.1, NAN, 0.0), (NAN, NAN, 0.5), (NAN, NAN, NAN), (INF, 0.0, 0.0), (0.0, -INF, 0.0), (INF, -INF, 1.0),
             (0.0, 0.0, NAN), (1e30, 0.0, 0.0), (0.0, -1e30, 0.0), (1e30, 1e30, -1e30)]


def state(seed):
    g = np.random.default_rng(seed)
    rb_pos = g.normal(0, 1.5, (N, NB, 3))
    rb_rot = g.normal(size=(N, NB, 4))
    rb_rot /= np.linalg.norm(rb_rot, axis=-1, keepdims=True)
    dof = g.uniform(-2.5, 2.5, (N, ND))
    return rb_pos, rb_rot, dof


def with_edges(dof, shift, edges=EDGES):
    dof = dof.copy().reshape(N, ND // 3, 3)
    for k, a in enumerate(edges):
        dof[(k + shift) % N, (3 * k + shift) % (ND // 3)] = a
    return dof.reshape(N, ND)


def sync(st, e, init):
    rb_pos, rb_rot, dof, p_rb_pos, p_rb_rot, p_dof = (torch.from_numpy(x[e:e + 1]) for x in st)
    t = V.HumanoidSMPLIMVis.__new__(V.HumanoidSMPLIMVis)
    t.nq = NQ
    t.mj_data = types.SimpleNamespace(qpos=np.zeros(3 * NQ))
    t.mj_sim = types.SimpleNamespace(forward=lambda: None)
    t._rigid_body_pos, t._rigid_body_rot, t._dof_pos = rb_pos, rb_rot, dof
    t._prev_target_dof_pos, t._prev_target_root_pos, t._prev_target_root_rot = p_dof, p_rb_pos[:, 0], p_rb_rot[:, 0]
    V.HumanoidSMPLIMVis._sync_ref_motion(t, init)
    return t.mj_data.qpos.copy()


def main():
    rb_pos, rb_rot, dof = state(1)
    p_rb_pos, p_rb_rot, p_dof = state(2)
    st = (rb_pos, rb_rot, with_edges(dof, 0), p_rb_pos, p_rb_rot, with_edges(p_dof, 3))
    out = {k: v for k, v in zip(("rb_pos", "rb_rot", "dof_pos", "p_rb_pos", "p_rb_rot", "p_dof_pos"), st)}
    for init in (False, True):
        out[f"qpos_init{int(init)}"] = np.stack([sync(st, e, init) for e in range(N)])
    np.savez_compressed(os.path.join(HERE, "im_record.npz"), **out)
    print("im_record.npz", {k: v.shape for k, v in out.items()})

    rb_pos, rb_rot, dof = state(3)
    p_rb_pos, p_rb_rot, p_dof = state(4)
    rb_pos[1, 0, 2], rb_rot[2, 0, 0], p_rb_pos[5, 0, 0], p_rb_rot[6, 0, 3] = NAN, INF, NAN, -INF
    st = (rb_pos, rb_rot, with_edges(dof, 0, NONFINITE), p_rb_pos, p_rb_rot, with_edges(p_dof, 5, NONFINITE))
    out = {k: v for k, v in zip(("rb_pos", "rb_rot", "dof_pos", "p_rb_pos", "p_rb_rot", "p_dof_pos"), st)}
    for init in (False, True):
        out[f"qpos_init{int(init)}"] = np.stack([sync(st, e, init) for e in range(N)])
    assert np.isnan(out["qpos_init0"]).any() and np.isfinite(out["qpos_init0"]).any()
    np.savez_compressed(os.path.join(HERE, "im_record_nonfinite.npz"), **out)
    print("im_record_nonfinite.npz", {k: v.shape for k, v in out.items()})


if __name__ == "__main__":
    main()
