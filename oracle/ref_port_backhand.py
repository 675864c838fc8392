"""Torch restatement of the two-hand backhand fix of the test-time export, what b200v2p_backhand_fix (csrc/b200env_v2p.cu) is tested
against: HumanoidSMPLIMMVAE.optimize_two_hand_backhand with single=True (vid2player/env/tasks/humanoid_smpl_im_mvae.py:948-1031) and
the frame selection and write-back of its callers (mvae_controller_vis.py:181-191, mvae_controller_vis_dual.py:213-231).  It runs in
float32 or float64 with autograd and torch.optim.Adam like the reference, and makes the three decisions the released reference
needs to run at all:
  1. rb_pos is the 7th output of _smpl_to_sim (the reference unpacks nine values of eight and raises ValueError);
  2. the FK uses the fixed player's own rest joints for every frame (the reference reads joint_pos_bind[:M], the rest joints of envs
     0..M-1: the two players alternate there in dual_mode 'different', and M > num_envs does not fit);
  3. the device is the caller's (the reference hard-codes cuda:0).
Pinned against tests/golden/v2p_backhand.npz, made by executing the reference's own optimize_two_hand_backhand
(tests/golden/make_golden_backhand.py)."""
import numpy as np
import torch

from . import ref_port_v2p as V

SMPL_PARENTS = [-1, 0, 0, 0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 9, 9, 12, 13, 14, 16, 17, 18, 19, 20, 21]
LR, ITERS, W_TARGET, W_REG, W_SMOOTH = 0.005, 500, 1.0, 0.2, 0.5


def arm_joints(righthand):
    """(fitted joints Wrist, Elbow, Shoulder, Collar; free hand; racket hand; racket wrist) in SMPL order"""
    return ([20, 18, 16, 13], 22, 23, 21) if righthand else ([21, 19, 17, 14], 23, 22, 20)


def select(swing_type, phase):
    """need_fix of the callers"""
    return (swing_type == 2) & (phase > 2.0) & (phase < 5.0)


def angle_axis_to_rotation_matrix(aa, eps=1e-6):
    """utils/konia_transform.py:250-334 as written, masked sum included, so that autograd sees what it sees in the reference"""
    aa = aa.reshape(-1, 3)
    theta2 = (aa * aa).sum(-1, keepdim=True)
    theta = torch.sqrt(theta2.clamp_min(eps))
    w = aa / (theta + eps)
    wx, wy, wz = w.unbind(-1)
    c, s = torch.cos(theta[:, 0]), torch.sin(theta[:, 0])
    k = 1.0 - c
    normal = torch.stack([c + wx * wx * k, wx * wy * k - wz * s, wy * s + wx * wz * k,
                          wz * s + wx * wy * k, c + wy * wy * k, -wx * s + wy * wz * k,
                          -wy * s + wx * wz * k, wx * s + wy * wz * k, c + wz * wz * k], -1)
    rx, ry, rz = aa.unbind(-1)
    one = torch.ones_like(rx)
    taylor = torch.stack([one, -rz, ry, rz, one, -rx, -ry, rx, one], -1)
    mask = (theta2 > eps).type_as(aa)
    return (mask * normal + (1.0 - mask) * taylor).view(-1, 3, 3)


def rotation_matrix_to_angle_axis(m):
    """konia's rotation_matrix_to_angle_axis (no gradient is needed through it): the numpy restatement of ref_port_v2p"""
    return torch.as_tensor(V.rotation_matrix_to_angle_axis(m.detach().cpu().numpy()), device=m.device)


def forward_kinematics(rotmat, rest):
    """utils/hybrik.py:597-652 batch_rigid_transform of [M,24,3,3] local rotations on one [24,3] rest pose: the 4x4 chain; posed
    joint positions [M,24,3]"""
    M = rotmat.shape[0]
    rel = rest.clone()
    rel[1:] = rest[1:] - rest[SMPL_PARENTS[1:]]
    tf = torch.zeros(M, 24, 4, 4, dtype=rotmat.dtype, device=rotmat.device)
    tf[:, :, :3, :3] = rotmat
    tf[:, :, :3, 3] = rel
    tf[:, :, 3, 3] = 1.0
    chain = [tf[:, 0]]
    for i in range(1, 24):
        chain.append(torch.matmul(chain[SMPL_PARENTS[i]], tf[:, i]))
    return torch.stack(chain, 1)[:, :, :3, 3]


def optimize(joint_rotmat, rest, righthand, iters=ITERS):
    """optimize_two_hand_backhand(single=True) on [M,24,3,3] rotations of one player with its rest joints [24,3]: the rotations after
    `iters` Adam steps and the (target, reg, smooth) terms of the last evaluated step (NaN where none was, like the mean of an
    empty L1)"""
    ik, free, hand, wrist = arm_joints(righthand)
    rest = rest.to(joint_rotmat.dtype)
    joint_rotmat = joint_rotmat.clone()
    root_diff = rest[0] - 0.0                                        # joint_pos_bind[:, :1] - root_pos, root_pos = 0
    rb = forward_kinematics(joint_rotmat, rest) - root_diff
    target = 2 * rb[:, hand] - rb[:, wrist] - rb[:, 0]
    base = rotation_matrix_to_angle_axis(joint_rotmat[:, ik])
    rot_delta = torch.zeros_like(base, requires_grad=True)
    opt = torch.optim.Adam([rot_delta], lr=LR, betas=(0.9, 0.999))
    l1 = torch.nn.L1Loss()
    terms = {}

    def closure():
        # the reference writes into joint_rotmat itself, so every step's graph hangs on to all earlier ones; those paths carry exact
        # zeros (the four slots are overwritten), so a fresh copy per step gives the same gradient in linear time
        opt.zero_grad()
        rm = joint_rotmat.clone()
        rm[:, ik] = angle_axis_to_rotation_matrix(base + rot_delta).view(-1, 4, 3, 3)
        cur = (forward_kinematics(rm, rest) - root_diff)[:, free]
        terms["target"] = l1(cur, target.detach()) * W_TARGET
        terms["reg"] = l1(rot_delta, torch.zeros_like(rot_delta)) * W_REG
        terms["smooth"] = l1(rot_delta[1:], rot_delta[:-1].detach()) * W_SMOOTH
        loss = sum(terms.values())
        loss.backward(retain_graph=True)
        return loss

    for _ in range(iters):
        opt.step(closure)
    with torch.no_grad():
        joint_rotmat[:, ik] = angle_axis_to_rotation_matrix(base + rot_delta).view(-1, 4, 3, 3)
    nan = float("nan")
    losses = [float(terms[k].detach()) if terms else nan for k in ("target", "reg", "smooth")]
    return joint_rotmat.detach(), np.array(losses)


def fix_episode(joint_rot, phase, swing_type, rest, righthand, iters=ITERS):
    """the callers' selection and write-back around optimize: joint_rot [T,24,3] -> (fixed copy, loss terms)"""
    joint_rot = joint_rot.clone()
    need = select(swing_type, phase)
    rm = angle_axis_to_rotation_matrix(joint_rot[need]).view(-1, 24, 3, 3)
    rm, losses = optimize(rm, rest, righthand, iters)
    joint_rot[need] = rotation_matrix_to_angle_axis(rm).to(joint_rot.dtype)
    return joint_rot, losses


def free_hand_distance(joint_rot, rest, righthand):
    """|free hand - target| per frame of [T,24,3] rows (the quantity the fix reduces)"""
    _, free, hand, wrist = arm_joints(righthand)
    rest = rest.to(joint_rot.dtype)
    rb = forward_kinematics(angle_axis_to_rotation_matrix(joint_rot).view(-1, 24, 3, 3), rest) - rest[0]
    return (rb[:, free] - (2 * rb[:, hand] - rb[:, wrist] - rb[:, 0])).norm(dim=-1)
