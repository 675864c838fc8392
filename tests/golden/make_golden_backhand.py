"""Golden fixture of the two-hand backhand fix (v2p_backhand.npz), produced by EXECUTING the reference's own
HumanoidSMPLIMMVAE.optimize_two_hand_backhand (vid2player/env/tasks/humanoid_smpl_im_mvae.py:948-1031), unchanged, on CPU through a
fake `self`, inside the selection and write-back of its caller (mvae_controller_vis.py:181-191).  Only its boundary is patched:
  - _smpl_to_sim returns the reference's eight outputs plus a placeholder (the method unpacks nine);
  - _smpl.joint_pos_bind is the player's rest joints repeated (the shipped djokovic / nadal skeletons);
  - torch.device('cuda:0') in the module gives the CPU;
  - the module's tqdm stops after k iterations, so the states after 1, 10 and 500 steps are pinned; the loss terms the method prints
    are captured.
Run where the reference is present:  python tests/golden/make_golden_backhand.py
"""
import itertools
import os
import sys
from types import SimpleNamespace

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
import _refenv  # noqa: E402

_refenv.setup("vid2player")

from env.tasks import humanoid_smpl_im_mvae as M  # noqa: E402
from utils.konia_transform import angle_axis_to_rotation_matrix, rotation_matrix_to_angle_axis  # noqa: E402

from vid2player3d_b200 import model_compiler  # noqa: E402

torch.set_num_threads(1)
SMPL_NAMES = ["Pelvis", "L_Hip", "R_Hip", "Torso", "L_Knee", "R_Knee", "Spine", "L_Ankle", "R_Ankle", "Chest", "L_Toe", "R_Toe",
              "Neck", "L_Thorax", "R_Thorax", "Head", "L_Shoulder", "R_Shoulder", "L_Elbow", "R_Elbow", "L_Wrist", "R_Wrist",
              "L_Hand", "R_Hand"]
SMPL_PARENTS = [-1, 0, 0, 0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 9, 9, 12, 13, 14, 16, 17, 18, 19, 20, 21]
STEPS = (1, 10, 500)


class _CpuTorch:
    """the module's `torch` with torch.device('cuda:0') mapped to the CPU"""

    def __getattr__(self, k):
        return getattr(torch, k)

    @staticmethod
    def device(*a, **k):
        return torch.device("cpu")


PRINTED = []
M.torch = _CpuTorch()
M.print = lambda *a, **k: PRINTED.append(a)


class FakePlayer(M.HumanoidSMPLIMMVAE):
    def __init__(self, rest, n):
        self.device = "cpu"
        self._build_mujoco_smpl_transform()
        self._smpl = SimpleNamespace(joint_pos_bind=rest.unsqueeze(0).repeat(max(n, 1), 1, 1), parents=torch.tensor(SMPL_PARENTS))

    def _smpl_to_sim(self, root_pos, joint_rotmat, *a, **k):
        return (*M.HumanoidSMPLIMMVAE._smpl_to_sim(self, root_pos, joint_rotmat, *a, **k), None)


def rest_joints(player):
    m = model_compiler.load_compiled("smpl_mesh_humanoid_" + player)
    names = [str(x) for x in m["body_names"]]
    pos = np.zeros((len(names), 3))
    for i in range(len(names)):
        pos[i] = m["offset"][i] + (pos[m["parent"][i]] if m["parent"][i] >= 0 else 0)
    return torch.tensor(np.stack([pos[names.index(n)] for n in SMPL_NAMES]), dtype=torch.float32)


def fix(joint_rot, phase, swing_type, rest, righthand, k):
    """mvae_controller_vis.py:181-191 with the reference's optimizer stopped after k steps"""
    joint_rot = joint_rot.clone()
    need_fix = (swing_type == 2) & (phase > 2.0) & (phase < 5.0)
    joint_rotmat = angle_axis_to_rotation_matrix(joint_rot[need_fix])
    M.tqdm = lambda it: itertools.islice(it, k)
    PRINTED.clear()
    joint_rotmat = FakePlayer(rest, int(need_fix.sum())).optimize_two_hand_backhand(joint_rotmat, single=True, righthand=righthand)
    joint_rot[need_fix] = rotation_matrix_to_angle_axis(joint_rotmat)
    return joint_rot, np.array(PRINTED[-1], np.float64)


def episode(g, T, segments):
    """a smooth random rally: a base pose plus a random walk; swing_type 2 with 2 < phase < 5 exactly on `segments` (frame ranges),
    boundary phases and other swing types around them"""
    jr = 0.35 * torch.randn(1, 24, 3, generator=g) + 0.03 * torch.randn(T, 24, 3, generator=g).cumsum(0)
    phase = torch.rand(T, generator=g) * 2.0                      # outside (2, 5)
    swing = torch.randint(0, 2, (T,), generator=g)
    for a, b in segments:
        phase[a:b] = torch.linspace(2.05, 4.95, b - a)
        swing[a:b] = 2
    edges = [a - 1 for a, _ in segments if a > 0] + [b for _, b in segments if b < T]
    for i, e in enumerate(edges):                                  # next to a segment: phase 2 or 5 exactly, or the wrong swing type
        phase[e], swing[e] = (2.0, 2) if i % 3 == 0 else ((5.0, 2) if i % 3 == 1 else (3.0, 1))
    return jr, phase, swing


g = torch.Generator().manual_seed(31)
cases = []
jr, ph, sw = episode(g, 12, [(5, 6)])                              # M = 1: no smoothness term
cases.append(("djokovic", True, jr, ph, sw))
jr, ph, sw = episode(g, 10, [(3, 5)])                              # M = 2
cases.append(("djokovic", True, jr, ph, sw))
jr, ph, sw = episode(g, 90, [(10, 40), (55, 85)])                 # M = 60 in two segments
jr[21] = jr[20]                                                    # identical consecutive frames
jr[30, 16] = torch.tensor([0.05, 3.1, 0.2])                        # fitted shoulder near theta = pi
jr[60, 9] = torch.tensor([3.08, 0.1, -0.05])                       # Spine3 near pi (the fixed part of the chain)
jr[70, 20] = 0.0                                                   # fitted wrist at rest: the Taylor branch at the first step
cases.append(("djokovic", True, jr, ph, sw))
jr, ph, sw = episode(g, 80, [(5, 35), (50, 80)])                  # left-handed, M = 60
jr[12, 17] = torch.tensor([-3.1, 0.1, 0.1])                        # fitted (right) shoulder near pi
jr[40] = jr[41]
cases.append(("nadal", False, jr, ph, sw))

OUT = dict(num_cases=np.int64(len(cases)), steps=np.array(STEPS))
for c, (player, rh, jr, ph, sw) in enumerate(cases):
    rest = rest_joints(player)
    OUT.update({f"c{c}_joint_rot": jr.numpy(), f"c{c}_phase": ph.numpy(), f"c{c}_swing_type": sw.numpy(), f"c{c}_rest": rest.numpy(),
                f"c{c}_righthand": np.bool_(rh)})
    for k in STEPS:
        out, losses = fix(jr, ph, sw, rest, rh, k)
        OUT[f"c{c}_out_{k}"] = out.numpy()
        OUT[f"c{c}_loss_{k}"] = losses
    print(player, "M =", int(((sw == 2) & (ph > 2) & (ph < 5)).sum()), "losses after", STEPS[-1], OUT[f"c{c}_loss_{STEPS[-1]}"])
np.savez_compressed(os.path.join(HERE, "v2p_backhand.npz"), **OUT)
print("v2p_backhand.npz", len(OUT), "arrays")
