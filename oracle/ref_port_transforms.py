"""Float64 restatement of the context window's transforms (HumanoidSMPLIM._transform_target, embodied_pose/env/tasks/
humanoid_smpl_im.py:565-592) from given draws, and the draws restated from the counter keys of the device launch (include/b200env.h:
b200_motion_context_t).

The restatement keeps the reference's aliasing: `joint_conf` is the local tensor of :567, which `mask_joints` zeroes and multiplies
body_pos by; `noisy_joints` rebinds context_dict['joint_conf'] to a new tensor, so a later `mask_joints` zeroes its joints' positions
but keeps their noise confidence and scales no other joint."""
import numpy as np
from scipy.special import erfc

from oracle.ref_port_sampled_policy import counter_normal
from oracle.ref_port_v2p import counter_hash


def transform_target(body_pos, transform_specs, body_names, noisy=None, noise=None, drop=None):
    """body_pos [..., nb, 3] -> (body_pos, joint_conf [..., nb]) in float64.  Draws: noisy [..., nb] bool (the noisy_joints Bernoulli),
    noise [..., nb, 3] N(0, 1) (torch.randn_like), drop [..., nb] bool (the mask_random_joints Bernoulli, root included: the transform
    exempts it)."""
    ctx = {'body_pos': np.array(body_pos, np.float64)}
    ctx['joint_conf'] = joint_conf = np.ones(ctx['body_pos'].shape[:-1])
    for transform, specs in (transform_specs or {}).items():
        if transform == 'mask_joints':
            joint_conf[..., [body_names.index(j) for j in specs['joints']]] = 0.0
            ctx['body_pos'] = ctx['body_pos'] * joint_conf[..., None]
        elif transform == 'noisy_joints':
            std = np.where(np.asarray(noisy, bool), float(specs['noise_std']), 0.0)
            nz = np.asarray(noise, np.float64) * std[..., None]
            conf = erfc(np.linalg.norm(nz, axis=-1) / (np.sqrt(3) * specs['conf_std']) / np.sqrt(2.0))
            ctx['body_pos'] = ctx['body_pos'] + nz
            ctx['joint_conf'] = conf
            occluded = conf < specs['min_conf']
            conf[occluded] = 0.0
            ctx['body_pos'][occluded] = 0.0
        elif transform == 'mask_random_joints':
            d = np.array(drop, bool)
            d[..., 0] = False
            ctx['joint_conf'][d] = 0.0
            ctx['body_pos'][d] = 0.0
        else:
            raise ValueError(f"unknown transform {transform!r}")
    return ctx['body_pos'], ctx['joint_conf']


def pre_occlusion_conf(transform_specs, noisy, noise):
    """the noise confidence before the min_conf test (float64), for telling apart decisions within rounding of the threshold"""
    s = transform_specs['noisy_joints']
    nz = np.asarray(noise, np.float64) * np.where(np.asarray(noisy, bool), float(s['noise_std']), 0.0)[..., None]
    return erfc(np.linalg.norm(nz, axis=-1) / (np.sqrt(3) * s['conf_std']) / np.sqrt(2.0))


def draw_index(num_envs, rows, P, nb):
    """[len(rows), P, nb] index of draw k = 0 of (row e, frame j, body b): 2 num_envs + ((e P + j) nb + b) 5"""
    e = np.asarray(rows, np.uint64)[:, None, None]
    j = np.arange(P, dtype=np.uint64)[None, :, None]
    b = np.arange(nb, dtype=np.uint64)[None, None, :]
    return np.uint64(2 * num_envs) + ((e * np.uint64(P) + j) * np.uint64(nb) + b) * np.uint64(5)


def draws(seed, counter, num_envs, rows, P, nb, transform_specs):
    """(noisy [n, P, nb] bool, noise [n, P, nb, 3] float64, drop [n, P, nb] bool) of the device launch at this seed and counter value
    for the windows of env rows `rows`: u_k = (bits >> 40) 2^-24 in float32, noisy = u_0 < prob, drop = u_4 < prob, noise = the
    Box-Muller normals of k = 1..3 (oracle.ref_port_sampled_policy.counter_normal, row = ((e P + j) nb + b), ldo 5)."""
    seed = int(seed) & 0xFFFFFFFFFFFFFFFF
    base = draw_index(num_envs, rows, P, nb)
    u = lambda k: (counter_hash(seed, counter, base + np.uint64(k)) >> np.uint64(40)).astype(np.float32) * np.float32(2.0 ** -24)  # noqa: E731
    specs = transform_specs or {}
    noisy = u(0) < np.float32(specs['noisy_joints']['prob']) if 'noisy_joints' in specs else np.zeros(base.shape, bool)
    drop = u(4) < np.float32(specs['mask_random_joints']['prob']) if 'mask_random_joints' in specs else np.zeros(base.shape, bool)
    flat = ((np.asarray(rows, np.uint64)[:, None, None] * np.uint64(P) + np.arange(P, dtype=np.uint64)[None, :, None]) * np.uint64(nb)
            + np.arange(nb, dtype=np.uint64)[None, None, :]).reshape(-1)
    noise = counter_normal(seed, counter, flat, np.arange(1, 4), 5, 2 * num_envs).reshape(base.shape + (3,))
    return noisy, noise, drop
