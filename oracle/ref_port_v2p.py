"""ORACLE (test infrastructure, not product code) - numpy restatement of the vid2player rows of the hot path
(SURVEY.md 8a a10-a17).  Paths are relative to /root/reference/vid2player.  Pinned against fixtures produced by
executing the reference's own code (tests/golden/make_golden_v2p.py -> tests/golden/v2p_*.npz).
Only tests/, smoke() and bench.py's CPU-baseline legs may import this module."""
import math

import numpy as np

from . import ref_port as R

BALL_R = 0.032      # utils/tennis_ball.py:15-27
BALL_M = 0.057
RHO = 1.21
KF = (RHO * math.pi * BALL_R * BALL_R) / 2
BASE_CD = 0.55
NET_HEIGHT = 1.07


# --------------------------------------------------------------------------- konia conversions
def safe_zero_division(num, den, eps=1e-6):
    """utils/konia_transform.py:337-345"""
    den = np.where(np.abs(den) < eps, den + eps, den)
    return num / den


def rotation_matrix_to_quaternion_wxyz(m, eps=1e-6):
    """utils/konia_transform.py:348-438 (order WXYZ)"""
    f = m.dtype.type
    m00, m01, m02 = m[..., 0, 0], m[..., 0, 1], m[..., 0, 2]
    m10, m11, m12 = m[..., 1, 0], m[..., 1, 1], m[..., 1, 2]
    m20, m21, m22 = m[..., 2, 0], m[..., 2, 1], m[..., 2, 2]
    trace = m00 + m11 + m22
    sq = np.sqrt(np.maximum(trace + f(1.0), f(eps))) * f(2.0)
    c0 = np.stack((f(0.25) * sq, safe_zero_division(m21 - m12, sq), safe_zero_division(m02 - m20, sq),
                   safe_zero_division(m10 - m01, sq)), -1)
    sq = np.sqrt(np.maximum(f(1.0) + m00 - m11 - m22, f(eps))) * f(2.0)
    c1 = np.stack((safe_zero_division(m21 - m12, sq), f(0.25) * sq, safe_zero_division(m01 + m10, sq),
                   safe_zero_division(m02 + m20, sq)), -1)
    sq = np.sqrt(np.maximum(f(1.0) + m11 - m00 - m22, f(eps))) * f(2.0)
    c2 = np.stack((safe_zero_division(m02 - m20, sq), safe_zero_division(m01 + m10, sq), f(0.25) * sq,
                   safe_zero_division(m12 + m21, sq)), -1)
    sq = np.sqrt(np.maximum(f(1.0) + m22 - m00 - m11, f(eps))) * f(2.0)
    c3 = np.stack((safe_zero_division(m10 - m01, sq), safe_zero_division(m02 + m20, sq), safe_zero_division(m12 + m21, sq),
                   f(0.25) * sq), -1)
    w2 = np.where((m11 > m22)[..., None], c2, c3)
    w1 = np.where(((m00 > m11) & (m00 > m22))[..., None], c1, w2)
    return np.where((trace > 0.0)[..., None], c0, w1)


def torch_safe_atan2(y, x, eps=1e-6):
    """utils/konia_transform.py:41-49"""
    y = np.where((np.abs(y) < eps) & (np.abs(x) < eps), y + eps, y)
    return np.arctan2(y, x)


def quaternion_to_angle_axis_wxyz(q, eps=1e-6):
    """utils/konia_transform.py:558-628"""
    f = q.dtype.type
    cos_theta, q1, q2, q3 = q[..., 0], q[..., 1], q[..., 2], q[..., 3]
    s2 = q1 * q1 + q2 * q2 + q3 * q3
    sin_theta = np.sqrt(np.maximum(s2, f(eps)))
    two_theta = f(2.0) * np.where(cos_theta < 0.0, torch_safe_atan2(-sin_theta, -cos_theta), torch_safe_atan2(sin_theta, cos_theta))
    k = np.where(s2 > 0.0, safe_zero_division(two_theta, sin_theta, eps), f(2.0))
    return np.stack((q1 * k, q2 * k, q3 * k), -1)


def rotation_matrix_to_angle_axis(m):
    """utils/konia_transform.py:632-655"""
    return quaternion_to_angle_axis_wxyz(rotation_matrix_to_quaternion_wxyz(m))


def quaternion_to_rotation_matrix_wxyz(q):
    """utils/konia_transform.py:474-555 (normalises first, eps 1e-12)"""
    f = q.dtype.type
    q = q / np.maximum(np.linalg.norm(q, axis=-1, keepdims=True), f(1e-12))
    w, x, y, z = q[..., 0], q[..., 1], q[..., 2], q[..., 3]
    tx, ty, tz = f(2.0) * x, f(2.0) * y, f(2.0) * z
    twx, twy, twz = tx * w, ty * w, tz * w
    txx, txy, txz = tx * x, ty * x, tz * x
    tyy, tyz, tzz = ty * y, tz * y, tz * z
    one = f(1.0)
    return np.stack((one - (tyy + tzz), txy - twz, txz + twy, txy + twz, one - (txx + tzz), tyz - twx, txz - twy, tyz + twx,
                     one - (txx + tyy)), -1).reshape(q.shape[:-1] + (3, 3))


def quat_to_rot6d(q_xyzw_as_wxyz):
    """utils/torch_transform.py:248-250 + rotmat_to_rot6d :216-218.  NOTE the reference passes the xyzw body
    quaternion straight into the WXYZ-order converter (physics_mvae_controller.py:339) - reproduced as is."""
    m = quaternion_to_rotation_matrix_wxyz(q_xyzw_as_wxyz)
    return np.concatenate([m[..., 0], m[..., 1]], -1)


# --------------------------------------------------------------------------- a13: SMPL FK targets
def batch_rigid_transform(rot_mats, joints, parents):
    """utils/hybrik.py:597-652"""
    N, J = rot_mats.shape[:2]
    rel = joints.copy()
    rel[:, 1:] -= joints[:, parents[1:]]
    G = np.zeros((N, J, 3, 3), rot_mats.dtype)
    P = np.zeros((N, J, 3), rot_mats.dtype)
    G[:, 0], P[:, 0] = rot_mats[:, 0], rel[:, 0]
    for i in range(1, J):
        p = parents[i]
        G[:, i] = G[:, p] @ rot_mats[:, i]
        P[:, i] = (G[:, p] @ rel[:, i, :, None])[..., 0] + P[:, p]
    return P, G


def smpl_to_sim(root_pos, joint_rotmat, rest, parents, smpl_2_mujoco, dt, prev_root_pos=None, prev_rb_rot=None):
    """env/tasks/humanoid_smpl_im_mvae.py:897-946.  Quirk kept: root_ang_vel = dof_vel[:,0] / dt (a second
    division by dt, :917-919)."""
    N = root_pos.shape[0]
    f = root_pos.dtype.type
    dof_pos = rotation_matrix_to_angle_axis(joint_rotmat)[:, smpl_2_mujoco][:, 1:].reshape(N, 69)
    joints = np.broadcast_to(rest, (N, 24, 3)).astype(root_pos.dtype)
    P, G = batch_rigid_transform(joint_rotmat, joints, parents)
    q = rotation_matrix_to_quaternion_wxyz(G)[..., [1, 2, 3, 0]]
    rb_pos, rb_rot = P[:, smpl_2_mujoco], q[:, smpl_2_mujoco]
    root_rot = rb_rot[:, 0]
    rb_pos = rb_pos - (joints[:, :1] - root_pos[:, None])
    if prev_root_pos is not None:
        root_vel = (root_pos - prev_root_pos) / f(dt)
        diff = quat_mul_norm(R.quat_conjugate(prev_rb_rot), rb_rot)
        ang, axis = R.quat_to_angle_axis(diff)
        dv = axis * ang[..., None] / f(dt)
        root_ang_vel = dv[:, 0] / f(dt)
        dof_vel = dv[:, 1:].reshape(N, 69)
    else:
        root_vel, root_ang_vel, dof_vel = np.zeros_like(root_pos), np.zeros_like(root_pos), np.zeros_like(dof_pos)
    return root_pos, root_rot, dof_pos, root_vel, root_ang_vel, dof_vel, rb_pos, rb_rot


def quat_mul_norm(x, y):
    """utils/torch_utils.py quat_mul_norm: quat_unit(quat_mul(x, y)) then w >= 0 (quat_pos)"""
    q = R.normalize(R.quat_mul(x, y))
    return np.where(q[..., 3:] < 0, -q, q)


# --------------------------------------------------------------------------- a10 / a17: ball
def ball_aero(ball_states, has_bounce, substeps, spin_scale):
    """apply_external_force_to_ball (humanoid_smpl_im_mvae.py:711-739): returns (force, has_bounce, has_bounce_now, bounce_pos_new_mask)"""
    f = ball_states.dtype.type
    pos, vel = ball_states[:, 0:3], ball_states[:, 7:10]
    vs = np.linalg.norm(vel, axis=1, keepdims=True)
    vs = np.where(vs == 0, vs + 1, vs)
    vn = vel / vs
    g = np.broadcast_to(np.array([0, 0, -1], ball_states.dtype), vel.shape)
    vel_tan = np.cross(vn, g)
    vspin = np.linalg.norm(ball_states[:, 10:13], axis=1, keepdims=True) / f(math.pi * 2)
    cl = 1 / (2 + np.abs(vs / (vspin * f(spin_scale) + f(1e-6))))     # get_cl, tennis_ball.py:30-32
    cl = cl * np.where(vspin > 0, f(-1), f(1))
    force = -f(KF) * f(BASE_CD) * vs * vel - f(KF) * cl * vs ** 2 * np.cross(vel_tan, vn)
    thr = BALL_R * 6 if substeps > 2 else BALL_R * 4
    now = ~has_bounce & (pos[:, 2] <= thr)
    return force.astype(ball_states.dtype), has_bounce | now, now


def ball_reset(pool, pool_index):
    """_reset_balls (:503-524) with TennisBallGeneratorOffline.generate (tennis_ball.py:435-456): returns
    (traj[n,100,3], launch_pos, launch_vel, launch_ang_vel)"""
    f = pool.dtype.type
    row = pool[pool_index]
    pos, vel, spin = row[:, 0:3], row[:, 3:6], row[:, 6]
    c = np.cross(vel, np.broadcast_to(np.array([0, 0, -1], pool.dtype), vel.shape))
    c = c / np.maximum(np.linalg.norm(c, axis=1, keepdims=True), f(1e-12))   # F.normalize
    return row[:, 7:].reshape(-1, 100, 3), pos, vel, spin[:, None] * f(math.pi) * f(2) * c


# --------------------------------------------------------------------------- a11 / a12: state from sim
GRIP_NORMAL = {'eastern': [0, 1, 0], 'semi_western': [0, 1. / math.sqrt(2), 1. / math.sqrt(2)]}


def update_state_from_sim(rbs, root_states, ball_states, prev_ball_vel, contact, grip, racket_body=24, wrist_body=22):
    """_update_state_from_sim (:799-860), substeps > 2 branch (velocity-jump contact detector :800-808)"""
    f = rbs.dtype.type
    now = ~contact & (ball_states[:, 8] > 0) & ((ball_states[:, 8] - prev_ball_vel[:, 1]) > 10)
    m = quaternion_to_rotation_matrix_wxyz(rbs[:, wrist_body, 3:7][:, [3, 0, 1, 2]])
    normal = m @ np.array(GRIP_NORMAL[grip], rbs.dtype)
    return dict(root_pos=rbs[:, 0, 0:3], root_vel=root_states[:, 7:10], racket_pos=rbs[:, racket_body, 0:3],
                racket_vel=rbs[:, racket_body, 7:10], racket_normal=normal, ball_pos=ball_states[:, 0:3], ball_vel=ball_states[:, 7:10],
                ball_vspin=np.linalg.norm(ball_states[:, 10:13], axis=1) / f(math.pi * 2), contact=contact | now, contact_now=now)


# --------------------------------------------------------------------------- a14: high-level observation
def roll_ball_obs(ball_obs, ball_pos, ids=None):
    """_compute_task_obs :345-346 on the rows `ids` (None = all): the history shifts by one, the current ball position is appended"""
    ids = np.arange(len(ball_obs)) if ids is None else np.asarray(ids)
    out = ball_obs.copy()
    out[ids] = np.roll(ball_obs[ids], -1, axis=1)
    out[ids, -1] = ball_pos[ids]
    return out


def reset_ball_obs(ball_obs, ball_pos, ids):
    """_reset_reaction_tasks :213-214 (use_history_ball_obs): the rows of the reaction envs <- the ball position repeated"""
    out = ball_obs.copy()
    out[np.asarray(ids)] = ball_pos[np.asarray(ids)][:, None, :]
    return out


def controller_obs(rbs25, root_pos, root_vel, racket_normal, ball_traj, target_bounce_pos, obs_len, use_target=True, ball_obs=None):
    """_compute_actor_obs (physics_mvae_controller.py:333-342) + _compute_task_obs (:344-360); ball_obs (already rolled) selects the
    use_history_ball_obs variant (:348-349), else the future-trajectory window"""
    N = rbs25.shape[0]
    actor = np.concatenate([root_pos, root_vel, (rbs25[:, 1:, 0:3] - root_pos[:, None]).reshape(N, 72),
                            quat_to_rot6d(rbs25[:, :24, 3:7].reshape(-1, 4)).reshape(N, 144), racket_normal], -1)
    src = ball_traj[:, :obs_len] if ball_obs is None else ball_obs
    task = (src - rbs25[:, 24, 0:3][:, None]).reshape(N, -1)
    if use_target:
        task = np.concatenate([task, target_bounce_pos[:, :2] - root_pos[:, :2]], -1)
    return np.concatenate([actor, task], -1)


# --------------------------------------------------------------------------- a15: rewards
def _contact_phase(swing_type, phase, mode):
    if mode == "reach":
        return np.where(swing_type == -1, np.ones_like(phase) * 3, np.ones_like(phase) * phase.dtype.type(math.pi))
    return np.where(swing_type >= 2, np.ones_like(phase) * 3, np.ones_like(phase) * phase.dtype.type(math.pi))


def reward_reach(phase, tar_action, racket_pos, ball_pos, swing_type, scales, weights):
    """compute_reward_reach (:493-520)"""
    pos_err = np.sum((ball_pos - racket_pos) ** 2, -1)
    pe = (phase - _contact_phase(swing_type, phase, "reach")) ** 2
    r = (tar_action == 1) * np.exp(-scales.get('pos', 5.) * pos_err) * np.exp(-scales.get('phase', 10.) * pe)
    return (r * weights.get('pos', 1.0)).astype(phase.dtype), r[:, None].astype(phase.dtype)


def reward_return(phase, racket_pos, ball_pos, has_contact, has_bounce, bounce_pos, target_pos, swing_type, scales, weights):
    """compute_reward_return (:522-561)"""
    pos_err = np.sum((ball_pos - racket_pos) ** 2, -1)
    pe = (phase - _contact_phase(swing_type, phase, "return")) ** 2
    pos_r = ~has_contact * np.exp(-scales.get('pos', 5.) * pos_err) * np.exp(-scales.get('phase', 10.) * pe) + has_contact * np.ones_like(pos_err)
    err = np.where(has_bounce, np.sum((bounce_pos - target_pos) ** 2, -1), np.sum((ball_pos - target_pos) ** 2, -1))
    ball_r = has_contact * np.clip((400 - err) / 400, 0.0, 1.0)
    rew = weights.get('pos', 0.0) * pos_r + weights.get('ball_pos', 0.0) * ball_r
    return rew.astype(phase.dtype), np.stack([pos_r, ball_r], -1).astype(phase.dtype)


def reward_return_w_estimate(racket_pos, phase, swing_type, ball_pos, has_contact, bounce_pos, bounce_time, bounce_in, target_pos,
                             scales, weights):
    """compute_reward_return_w_estimate (:563-602)"""
    pos_err = np.sum((ball_pos - racket_pos) ** 2, -1)
    pe = (phase - _contact_phase(swing_type, phase, "return")) ** 2
    pos_r = ~has_contact * np.exp(-scales.get('pos', 5.) * pos_err) * np.exp(-scales.get('phase', 10.) * pe) + has_contact * np.ones_like(pos_err)
    err = np.sum((bounce_pos - target_pos) ** 2, -1)
    ball_r = bounce_in * np.exp(-scales.get('bounce_pos', 0.05) * err) * np.exp(-scales.get('bounce_time', 0.1) * bounce_time)
    rew = weights.get('pos', 0.0) * pos_r + weights.get('ball_pos', 0.0) * ball_r
    return rew.astype(phase.dtype), np.stack([pos_r, ball_r], -1).astype(phase.dtype)


# --------------------------------------------------------------------------- a16: estimator, bounce-in, reset FSM
COURT_MIN, COURT_MAX = (-4.11, 0.0), (4.11, 11.89)   # physics_mvae_controller.py:285-286


def in_court(p):
    return (p[:, 0] > COURT_MIN[0]) & (p[:, 0] < COURT_MAX[0]) & (p[:, 1] > COURT_MIN[1]) & (p[:, 1] < COURT_MAX[1])


def est_round(v):
    """torch.round: half to even"""
    return np.round(v)


def net_crossing_x(b):
    """x where the outgoing ball crosses the net (utils/tennis_ball_out_estimator.py:172): tensor ops, every product rounded"""
    with np.errstate(divide="ignore", invalid="ignore"):
        return b[:, 0] + b[:, 7] * np.abs(b[:, 1] / b[:, 8])


def estimator_estimate(ball_states, est_x, est_y, params):
    """TennisBallOutEstimator.estimate (utils/tennis_ball_out_estimator.py:164-205) with index math :126-162.
    params rows: VEL_X, VEL_Y, VSPIN, TRAJ_X, TRAJ_Y ranges (lo, hi, step).  Returns per-row
    (valid, bounce_pos[n,2], bounce_time, max_height) for ALL rows (invalid rows zero)."""
    f = ball_states.dtype.type
    VX, VY, VS, TX, TY = [tuple(float(v) for v in r) for r in params]
    b = ball_states
    valid = (b[:, 8] > VX[0]) & (b[:, 9] > VY[0]) & (b[:, 9] < VY[1]) & (b[:, 2] < TY[1])
    x_net = net_crossing_x(b)
    valid &= (x_net > -4) & (x_net < 4)
    n = len(b)
    bounce_pos, bounce_time, max_h = np.zeros((n, 2), b.dtype), np.zeros(n, b.dtype), np.zeros(n, b.dtype)
    if valid.any():
        s = b[valid]
        vel_x = np.linalg.norm(s[:, 7:9], axis=-1)
        vel_y = s[:, 9]
        vspin = np.linalg.norm(s[:, 10:13], axis=1) / f(math.pi * 2)

        def idx(v, rng):
            v = np.clip(v, f(rng[0]), f(rng[1] - rng[2]))
            return est_round((v - f(rng[0])) / f(rng[2]))
        dim = ((VX[1] - VX[0]) / VX[2], (VY[1] - VY[0]) / VY[2], (VS[1] - VS[0]) / VS[2])
        ti = (idx(vel_x, VX) * f(dim[1]) * f(dim[2]) + idx(vel_y, VY) * f(dim[2]) + idx(vspin, VS)).astype(np.int64)
        tx, ty = est_x[ti], est_y[ti]
        hi = idx(s[:, 2], TY).astype(np.int64)
        ar = np.arange(len(s))
        bp = s[:, :2] + ty[ar, hi, :1] * s[:, 7:9] / vel_x[:, None]
        bt = ty[ar, hi, 1].copy()
        net_dist = -s[:, 1] / s[:, 8] * vel_x
        ni = idx(net_dist, TX).astype(np.int64)
        miss = tx[ar, ni] + s[:, 2] < NET_HEIGHT
        bp[miss] = 0
        bt[miss] = 0
        bounce_pos[valid], bounce_time[valid], max_h[valid] = bp, bt, s[:, 2] + tx.max(axis=1)
    return valid, bounce_pos, bounce_time, max_h


def check_out_of_court(root_pos, court_min, court_max):
    """physics_mvae_controller.py:481-491"""
    return ((root_pos[:, 0] < court_min[0]) | (root_pos[:, 1] < court_min[1]) | (root_pos[:, 0] > court_max[0]) |
            (root_pos[:, 1] > court_max[1])).astype(np.int64)


def controller_reset(root_pos, court_min, court_max, obs_has_nan, progress, max_len, tar_time, tar_time_total, tar_action, has_contact,
                     ball_pos, est_bounce_in, early_termination=True, reward_w_estimate=True):
    """_compute_reset (physics_mvae_controller.py:408-436).  Returns (reset, terminate, reset_reaction, reset_recovery)."""
    terminated = check_out_of_court(root_pos, court_min, court_max).astype(bool) | obs_has_nan
    terminate_buf = terminated.astype(np.int64)
    reset = np.where(progress >= max_len - 1, 1, terminate_buf)
    reaction = tar_time == tar_time_total
    behind = ball_pos[:, 1] < root_pos[:, 1] - 1
    recovery = (tar_action == 1) & (has_contact | behind)
    terminate = terminate_buf.astype(bool)
    if early_termination:
        terminate = terminate | (recovery & ~has_contact) | behind
        if reward_w_estimate:
            terminate = terminate | (has_contact & ~est_bounce_in)
    terminate_buf = np.where(terminate, 1, terminate_buf)
    reset = np.where(terminate, 1, reset)
    recovery = recovery & ~terminate
    reaction = reaction | reset.astype(bool)
    return reset, terminate_buf, reaction, recovery


# --------------------------------------------------------------------------- a14-a16 as one step (b200v2p_controller_post)
REWARD_NAMES = ("reach", "return", "return_w_estimate")


def advance_counters(s):
    """tail of physics_step (:364-366) + head of post_physics_step (:441-442): the trajectory window rolls by one frame with a zero
    last frame, the reaction timer and the episode progress count one step"""
    tr = s["ball_traj"]
    s["ball_traj"] = np.concatenate([tr[:, 1:], np.zeros_like(tr[:, :1])], 1)
    s["tar_time"] = s["tar_time"] + 1
    s["progress"] = s["progress"] + 1


def history_rows(s, cfg):
    """rows whose ball history _compute_task_obs rolls (:345-346): every row in a step; in an observation refresh (_reset_envs
    :200-201, dual :64-66) the rows being reset"""
    if not cfg.get("obs_only"):
        return np.ones(len(s["root_pos"]), bool)
    return s["reset_reaction"] | (s["reset_recovery"] & (not cfg.get("dual")))


def controller_post(s, cfg):
    """One b200v2p_controller_post launch on the numpy state `s` (dict of per-env arrays, returned updated in a copy):
    post_physics_step (:440-452) = [advance] -> _update_state (:271-314) -> _compute_reward (:368-406) -> _compute_observations
    (:316-360, ball history rolled) -> _compute_reset (:408-436), or the dual FSM (physics_mvae_controller_dual.py:92-120).
    cfg keys: obs_traj_len, use_target, reward_type (REWARD_NAMES), early_termination, max_len, court_min, court_max, scales, weights,
    est (est_x, est_y, params) or None, and the launch flags advance / obs_only / dual / use_history.  obs_only: the observation refresh
    of _reset_envs; with s["touch_mask"] (the humanoids just reset) the rows neither in it nor flagged for a task reset are not
    touched and the task flags of the rows in it are cleared afterwards (:176-177)."""
    s = {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in s.items()}
    n = len(s["root_pos"])
    f = np.float32
    obs_only, dual, L = bool(cfg.get("obs_only")), bool(cfg.get("dual")), int(cfg["obs_traj_len"])
    touch = s.get("touch_mask")
    rows = np.ones(n, bool)
    if obs_only and touch is not None:
        rows = touch | s["reset_reaction"] | s["reset_recovery"]
    if cfg.get("advance") and not obs_only:
        advance_counters(s)
    if not obs_only:
        upd = (s["tar_action"] == 0) & s["has_bounce_now"]
        s["bounce_in"] = np.where(upd, in_court(s["bounce_pos"]), s["bounce_in"])
        est = cfg.get("est")
        if est is not None and s["has_contact_now"].any():
            ids = np.flatnonzero(s["has_contact_now"])
            valid, bp, bt, mh = estimator_estimate(s["ball_states"][ids, :13], est[0], est[1], est[2])
            ids = ids[valid]
            s["est_bounce_pos"][ids, :2] = bp[valid]
            s["est_bounce_time"][ids] = bt[valid]
            s["est_max_height"][ids] = mh[valid]
            s["est_bounce_in"][ids] = in_court(s["est_bounce_pos"][ids])
        rt, sc, w = cfg["reward_type"], cfg["scales"], cfg["weights"]
        if rt == "reach":
            rew, sub = reward_reach(s["phase"], s["tar_action"], s["racket_pos"], s["ball_pos"], s["swing_type"], sc, w)
            sub = np.concatenate([sub, np.zeros_like(sub)], 1)
        elif rt == "return":
            rew, sub = reward_return(s["phase"], s["racket_pos"], s["ball_pos"], s["has_contact"], s["has_bounce"], s["bounce_pos"],
                                     s["target_bounce_pos"], s["swing_type"], sc, w)
        else:
            rew, sub = reward_return_w_estimate(s["racket_pos"], s["phase"], s["swing_type_cycle"], s["ball_pos"], s["has_contact"],
                                                s["est_bounce_pos"], s["est_bounce_time"], s["est_bounce_in"], s["target_bounce_pos"], sc, w)
        s["rew"], s["sub"] = rew.astype(f), sub.astype(f)
    roll = history_rows(s, cfg) & rows
    if s.get("ball_obs") is not None and L > 0:
        s["ball_obs"] = roll_ball_obs(s["ball_obs"], s["ball_pos"], np.flatnonzero(roll))
    r = np.flatnonzero(rows)
    if len(r):
        hist = s["ball_obs"][r] if cfg.get("use_history") else None
        s["obs"][r] = controller_obs(s["rbs"][r, :25], s["root_pos"][r], s["root_vel"][r], s["racket_normal"][r], s["ball_traj"][r],
                                     s["target_bounce_pos"][r], L, bool(cfg["use_target"]), hist)
    if not obs_only:
        has_nan = np.isnan(s["obs"]).any(1)
        if dual:
            s["reset"], rea, rec, s["distance"] = dual_controller_reset(s["tar_action"], s["has_contact"], s["has_bounce"], s["ball_pos"],
                                                                        s["root_pos"], s["root_vel"], s["bounce_in"], s["distance"],
                                                                        s["reset"])
        else:
            s["distance"] = (s["distance"] + np.sqrt((s["root_vel"][:, :2] ** 2).sum(-1))).astype(f)
            s["reset"], s["terminate"], rea, rec = controller_reset(
                s["root_pos"], np.asarray(cfg["court_min"], f), np.asarray(cfg["court_max"], f), has_nan, s["progress"], cfg["max_len"],
                s["tar_time"], s["tar_time_total"], s["tar_action"], s["has_contact"], s["ball_pos"], s["est_bounce_in"],
                bool(cfg["early_termination"]), rt == "return_w_estimate")
        s["reset_reaction"], s["reset_recovery"] = rea.astype(bool), rec.astype(bool)
    elif touch is not None:
        s["reset_reaction"] = s["reset_reaction"] & ~touch
        s["reset_recovery"] = s["reset_recovery"] & ~touch
    return s


# --------------------------------------------------------------------------- task resets (b200v2p_task_reset)
def pool_index(ball_pos, pool_rand, side_rand, pool_size):
    """TennisBallGeneratorOffline.generate with start_pos (utils/tennis_ball.py:436-444): a ball coming back from the other side
    (y > 0) is drawn near its x: ((x + 4) / 8 * P) truncated, + side_rand, clamped to the pool; otherwise pool_rand"""
    f = np.float32
    x = ball_pos[:, 0].astype(f)
    near = (((x + f(4)) / f(8) * f(pool_size)).astype(np.int64) + side_rand).clip(0, pool_size - 1)
    return np.where(ball_pos[:, 1] > 0, near, pool_rand)


def task_reset(s, cfg, draws):
    """_reset_envs (:173-201) task part for the reset masks in s: _reset_balls (:503-524) of the reaction envs, _reset_recovery_tasks
    (:242-245), _reset_reaction_tasks (:203-240).  draws: pool_rand, side_rand, frame_rand, target_seed (3 floats: continuous, n: discrete).
    s["rbs"] ball row = the last body of each env.  Returns an updated copy."""
    s = {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in s.items()}
    f = np.float32
    rea, rec = np.flatnonzero(s["reset_reaction"]), np.flatnonzero(s["reset_recovery"])
    if len(rea):
        pool = cfg["pool"]
        idx = pool_index(s["ball_pos"][rea], draws["pool_rand"][rea], draws["side_rand"][rea], len(pool))
        traj, pos, vel, w = ball_reset(pool, idx)
        if s.get("ball_obs") is not None:
            s["ball_obs"][rea] = pos[:, None, :]
        else:
            s["ball_traj"][rea] = traj
        for key in ("ball_states", "rbs_ball"):
            s[key][rea, 0:3], s[key][rea, 7:10], s[key][rea, 10:13] = pos, vel, w
        s["ball_pos"][rea], s["ball_vel"][rea], s["bounce_pos"][rea] = pos, vel, 0
        s["has_bounce"][rea], s["has_contact"][rea] = False, False
    s["tar_action"][rec] = 0
    s["has_bounce"][rec] = False
    s["bounce_pos"][rec] = 0
    if len(rea):
        s["tar_time"][rea] = 0
        s["tar_action"][rea] = 1
        s["num_reset_reaction"][rea] += 1
        s["bounce_in"][rea], s["est_bounce_in"][rea] = False, False
        s["est_bounce_pos"][rea], s["est_bounce_time"][rea], s["est_max_height"][rea] = 0, 0, 0
        s["swing_type_cycle"][rea] = -1
        s["tar_time_total"][rea] = cfg["reaction_nframes"] + draws["frame_rand"][rea]
        seed = np.asarray(draws["target_seed"], f)
        tmin, tmax = np.asarray(cfg["target_min"], f), np.asarray(cfg["target_max"], f)
        if cfg["target_mode"] == "continuous":
            s["target_bounce_pos"][rea] = seed * (tmax - tmin) + tmin
        elif cfg["target_mode"] == "discrete":
            sd = seed[rea]
            s["target_bounce_pos"][rea, 0] = np.where(sd < f(0.33), f(-3), np.where(sd > f(0.67), f(3), f(0)))
            s["target_bounce_pos"][rea, 1:] = (10, 0)
    return s


def quat_rotate(q, v):
    """isaacgym.torch_utils.quat_rotate (xyzw): v (2w^2 - 1) + 2 w (q x v) + 2 q (q . v)"""
    f = q.dtype.type
    w, u = q[..., 3:4], q[..., :3]
    return v * (f(2) * w * w - f(1)) + np.cross(u, v) * w * f(2) + u * (u * v).sum(-1, keepdims=True) * f(2)


def actor_reset(s, src, ids, cfg):
    """HumanoidSMPLIMMVAE._reset_actors + _set_env_state (humanoid_smpl_im_mvae.py:463-501) + the humanoid part of _reset_env_tensors
    (:562-581) for the env ids: the FK pose src (root_pos, root_rot, dof_pos, rb_pos [N,24,3], rb_rot [N,24,4], velocities zero) is
    written into the sim state.  The welded racket row (cfg racket_body >= 0) is not in the reference, which gets it from the simulator's
    forward kinematics: here it is the parent body's pose with the racket offset rotated by the parent (quat_rotate); in dual mode odd
    envs use the second player's parent and offset."""
    s = {k: v.copy() for k, v in s.items()}
    ids = np.asarray(ids)
    rbs, nd = s["rbs"], s["dof_state"].shape[1]
    rbs[ids, :24, 0:3], rbs[ids, :24, 3:7], rbs[ids, :24, 7:13] = src["rb_pos"][ids], src["rb_rot"][ids], 0
    s["prev_target_rb_rot"][ids] = src["rb_rot"][ids]
    if cfg["racket_body"] >= 0:
        second = (ids % 2 == 1) & bool(cfg.get("dual"))
        par = np.where(second, cfg.get("racket_parent2", cfg["racket_parent"]), cfg["racket_parent"])
        off = np.where(second[:, None], np.asarray(cfg.get("racket_offset2", cfg["racket_offset"]), np.float32),
                       np.asarray(cfg["racket_offset"], np.float32)).astype(np.float32)
        q = src["rb_rot"][ids, par]
        rbs[ids, cfg["racket_body"], 0:3] = src["rb_pos"][ids, par] + quat_rotate(q, off)
        rbs[ids, cfg["racket_body"], 3:7], rbs[ids, cfg["racket_body"], 7:13] = q, 0
    s["dof_state"][ids, :, 0], s["dof_state"][ids, :, 1] = src["dof_pos"][ids, :nd], 0
    s["pd_target_dof_pos"][ids] = src["dof_pos"][ids, :nd]
    rs = s["root_states"]
    rs[ids, 0:3], rs[ids, 3:7], rs[ids, 7:13] = src["root_pos"][ids], src["root_rot"][ids], 0
    for k in ("prev_target_root_pos", "root_pos", "target_root_pos"):
        s[k][ids] = src["root_pos"][ids]
    s["root_vel"][ids] = 0
    for k in ("progress", "reset", "terminate"):
        s[k][ids] = 0
    return s


def ctrl_reset(s, mask):
    """PhysicsMVAEController._reset_env_tensors (:200-208) + num_reset += 1 for the envs in mask"""
    s = {k: v.copy() for k, v in s.items()}
    for k in ("progress", "reset", "terminate", "num_reset_reaction"):
        s[k][mask] = 0
    s["distance"][mask] = 0
    s["num_reset"][mask] += 1
    return s


# --------------------------------------------------------------------------- counter-based normals and the target stream
# Project contracts, not reference behaviour: their specification is the comment of include/b200env_v2p.h and b200env_v2p.cu.
M64 = (1 << 64) - 1


def splitmix64(x):
    x = np.asarray(x, np.uint64) + np.uint64(0x9E3779B97F4A7C15)
    x = (x ^ (x >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
    x = (x ^ (x >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return x ^ (x >> np.uint64(31))


def counter_hash(seed, step, idx):
    """splitmix64(splitmix64(seed ^ step * 0xD1B54A32D192ED03) + idx), all mod 2^64"""
    with np.errstate(over="ignore"):
        h0 = splitmix64(np.uint64(seed) ^ np.uint64((int(step) * 0xD1B54A32D192ED03) & M64))
        return splitmix64(h0 + np.asarray(idx, np.uint64))


def counter_normal(seed, step, idx):
    """Box-Muller from the 24-bit halves of the hash: u1 in (0, 1], u2 in [0, 1); float32 like the kernel"""
    f = np.float32
    h = counter_hash(seed, step, idx)
    u1 = ((h >> np.uint64(40)).astype(np.uint32) + np.uint32(1)).astype(f) * f(1.0 / 16777217.0)
    u2 = ((h >> np.uint64(8)) & np.uint64(0xFFFFFF)).astype(f) * f(1.0 / 16777216.0)
    return (np.sqrt(f(-2) * np.log(u1)) * np.cos(f(6.283185307179586) * u2)).astype(f)


def pre_step(actions, tar_action, step, cfg):
    """b200v2p_pre_step: (mvae_actions, res_dof_actions); element i = e * (latent + res) + k draws counter_normal(seed, step, i)"""
    f = np.float32
    n, nl, nr = len(actions), cfg["num_latent"], cfg["num_res_dof"]
    lat = (actions[:, :nl] * f(cfg["vae_action_scale"])).astype(f)
    if cfg["random_walk_in_recovery"]:
        i = np.arange(n)[:, None] * (nl + nr) + np.arange(nl)[None]
        rnd = np.clip(counter_normal(cfg["seed"], step, i), f(-5), f(5))
        lat = np.where((tar_action == 0)[:, None], rnd, lat)
    return lat, (actions[:, nl:nl + nr] * f(cfg["residual_dof_scale"])).astype(f)


def stream_frames(clock, advance, offset, frames, n, seed=0, reseed_mask=None):
    """b200v2p_stream_gather: (frame per env, new offsets).  t = clock + advance; a reseeded env draws offset = hash(seed, t, e) % frames;
    env e reads frame (t + offset[e]) mod frames (non-negative)"""
    t = int(clock) + int(advance)
    off = np.asarray(offset, np.int64).copy()
    if reseed_mask is not None:
        e = np.flatnonzero(reseed_mask)
        off[e] = (counter_hash(seed, t, e) % np.uint64(frames)).astype(np.int64)
    return np.mod(t + off, frames), off


# --------------------------------------------------------------------------- a13b: head look-at correction
def angle_axis_to_rotation_matrix(aa, eps=1e-6):
    """utils/konia_transform.py:250-334"""
    f = aa.dtype.type
    theta2 = np.sum(aa * aa, -1, keepdims=True)
    theta = np.sqrt(np.maximum(theta2, f(eps)))
    w = aa / (theta + f(eps))
    wx, wy, wz = w[..., 0:1], w[..., 1:2], w[..., 2:3]
    c, s_ = np.cos(theta), np.sin(theta)
    one = f(1.0)
    normal = np.concatenate([c + wx * wx * (one - c), wx * wy * (one - c) - wz * s_, wy * s_ + wx * wz * (one - c),
                             wz * s_ + wx * wy * (one - c), c + wy * wy * (one - c), -wx * s_ + wy * wz * (one - c),
                             -wy * s_ + wx * wz * (one - c), wx * s_ + wy * wz * (one - c), c + wz * wz * (one - c)], -1)
    rx, ry, rz = aa[..., 0:1], aa[..., 1:2], aa[..., 2:3]
    k1 = np.ones_like(rx)
    taylor = np.concatenate([k1, -rz, ry, rz, k1, -rx, -ry, rx, k1], -1)
    return np.where(theta2 > eps, normal, taylor).reshape(aa.shape[:-1] + (3, 3))


def fix_head_orientation(joint_rotmat, head_rot_xyzw, head_pos, ball_pos, root_pos, head=15, neck=12):
    """env/tasks/humanoid_smpl_im_mvae.py:605-634: returns the joint rotations with Head / Neck yawed half-way each towards
    the ball (no correction when the ball is behind the player or wider than 4 m)."""
    f = joint_rotmat.dtype.type
    m = quaternion_to_rotation_matrix_wxyz(head_rot_xyzw[:, [3, 0, 1, 2]])
    look = m @ np.array([0, 0, 1], joint_rotmat.dtype)
    look = look[:, :2] / np.maximum(np.linalg.norm(look[:, :2], axis=-1, keepdims=True), f(1e-12))
    hb = ball_pos[:, :2] - head_pos[:, :2]
    hb = hb / np.maximum(np.linalg.norm(hb, axis=-1, keepdims=True), f(1e-12))
    d = np.arctan2(hb[:, 1], hb[:, 0]) - np.arctan2(look[:, 1], look[:, 0])
    d = np.where(d > math.pi, d - f(math.pi * 2), d)
    d = np.where(d < -math.pi, d + f(math.pi * 2), d)
    miss = (ball_pos[:, 1] < root_pos[:, 1] - 0.5) | (np.abs(ball_pos[:, 0]) > 4)
    d = np.where(miss, f(0), d).astype(joint_rotmat.dtype)
    jr = rotation_matrix_to_angle_axis(joint_rotmat[:, [head, neck]])
    jr[:, 0, 1] += d / 2
    jr[:, 1, 1] += d / 2
    out = joint_rotmat.copy()
    out[:, [head, neck]] = angle_axis_to_rotation_matrix(jr)
    return out


# --------------------------------------------------------------------------- dual mode
def get_opponent_env_ids(env_ids):
    """utils/common.py:111-115: partner ids, SORTED (so aligned with a sorted id list unless both envs of a pair are in it)"""
    env_ids = np.asarray(env_ids)
    if len(env_ids) == 0:
        return env_ids
    even = env_ids % 2 == 0
    return np.sort(np.concatenate([env_ids[even] + 1, env_ids[~even] - 1]))


def in_estimator_index(height, vel_x, vel_y, vspin, params):
    """utils/tennis_ball_in_estimator.py:22-49: params rows = HEIGHT, VEL_X, VEL_Y, VSPIN ranges (lo, hi, step).
    float32 tensor arithmetic with python scalars folded in one at a time, torch.round = half-to-even; the row index is the
    float32 sum truncated by .long()."""
    f = np.float32
    H, VX, VY, VS = [tuple(float(x) for x in r) for r in np.asarray(params, np.float64)]
    cl = lambda v, r: np.clip(v.astype(f), f(r[0]), f(r[1] - r[2]))  # noqa: E731
    height, vel_x, vel_y, vspin = cl(height, H), cl(vel_x, VX), cl(vel_y, VY), cl(vspin, VS)
    dim = [(r[1] - r[0]) / r[2] for r in (H, VX, VY, VS)]
    rnd = lambda v, r: np.rint((v - f(r[0])) / f(r[2])).astype(f)  # noqa: E731
    rh, rx, ry, rs = rnd(height, H), rnd(vel_x, VX), rnd(vel_y, VY), rnd(vspin, VS)
    index = rh * f(dim[1]) * f(dim[2]) * f(dim[3]) + rx * f(dim[2]) * f(dim[3]) + ry * f(dim[3]) + rs
    snap = lambda r_, r: r_ * f(r[2]) + f(r[0])  # noqa: E731
    return index.astype(np.int64), (snap(rh, H), snap(rx, VX), snap(ry, VY), snap(rs, VS))


def in_estimator_estimate(ball_states, table, params):
    """TennisBallInEstimator.estimate (utils/tennis_ball_in_estimator.py:51-81): snap the outgoing ball to the table grid,
    return the incoming trajectory in the receiver's frame (xy mirrored) and the snapped in / out ball states."""
    f = np.float32
    bs = ball_states.astype(f)
    vel_x = np.sqrt((bs[:, 7:9] ** 2).sum(-1, dtype=f)).astype(f)
    d = bs[:, 7:9] / vel_x[:, None]
    vspin = (np.sqrt((bs[:, 10:13] ** 2).sum(-1, dtype=f)).astype(f) / f(math.pi * 2)).astype(f)
    idx, (height, vx, vy, vs) = in_estimator_index(bs[:, 2], vel_x, bs[:, 9], vspin, params)
    traj = table[idx].astype(f)
    tt = np.concatenate([traj[:, :, :1] * d[:, None, :] + bs[:, None, :2], traj[:, :, 1:]], axis=-1)
    tt[:, :, :2] *= f(-1)

    def omega(v):
        c = np.cross(v, np.array([0, 0, -1], f)).astype(f)
        nn = np.maximum(np.sqrt((c * c).sum(-1, keepdims=True, dtype=f)), f(1e-12))
        return (vs[:, None] * f(math.pi) * f(2)) * (c / nn)      # vspin * pi * 2 * normalize(.)
    s_in = bs.copy()
    s_in[:, :2] *= f(-1)
    s_in[:, 2] = height
    s_in[:, 7:9] = -vx[:, None] * d
    s_in[:, 9] = vy
    s_in[:, 10:13] = omega(s_in[:, 7:10])
    s_out = s_in.copy()
    s_out[:, :2] *= f(-1)
    s_out[:, 7:9] *= f(-1)
    s_out[:, 10:13] = omega(s_out[:, 7:10])
    return tt, s_in, s_out


def dual_reset_balls(ball_states, racket_pos, recovery_ids, ball_ids, rand3, table, params):
    """HumanoidSMPLIMMVAEDual._reset_balls (env/tasks/humanoid_smpl_im_mvae_dual.py:52-80).  rand3 [3,len(recovery_ids)] = the three
    torch.rand draws (vx, vy, vz of the serve) in call order.  Returns traj and the updated copy of ball_states; the flag / view
    updates (:74-78) are listed in the returned dict."""
    f = np.float32
    bs = ball_states.astype(f).copy()
    if len(recovery_ids) > 0:
        bs[recovery_ids, :3] = racket_pos[recovery_ids]
        bs[recovery_ids, 10:13] = np.array([-40, 0, 0], f)
        bs[recovery_ids, 7] = rand3[0].astype(f) * f(4) + f(-2)
        bs[recovery_ids, 8] = rand3[1].astype(f) * f(4) + f(28)
        bs[recovery_ids, 9] = rand3[2].astype(f) * f(3) + f(5)
    contact = get_opponent_env_ids(ball_ids)
    traj, s_in, s_out = in_estimator_estimate(bs[contact], table, params)
    bs[ball_ids] = s_in
    bs[contact] = s_out
    return traj, bs, dict(ball_pos=bs[ball_ids, 0:3], ball_vel=bs[ball_ids, 7:10])


def dual_controller_reset(tar_action, has_contact, has_bounce, ball_pos, root_pos, root_vel, bounce_in, distance, reset_buf):
    """PhysicsMVAEControllerDual._compute_reset (env/tasks/physics_mvae_controller_dual.py:92-120) + _compute_stats"""
    in_recovery = tar_action == 0
    miss_ball = ball_pos[:, 1] < root_pos[:, 1] - np.float32(1)
    twice = has_bounce & (ball_pos[:, 2] < np.float32(0.05))
    recovery = (tar_action == 1) & (has_contact | miss_ball | twice)
    distance = distance + np.sqrt((root_vel[:, :2] ** 2).sum(-1))
    reaction = np.zeros_like(recovery)
    reaction[::2] = recovery[1::2]
    reaction[1::2] = recovery[::2]
    terminate = (recovery & ~has_contact) | (in_recovery & has_bounce & ~bounce_in)
    reset = reset_buf.copy()
    if terminate.sum() > 0:
        terminate[::2] |= terminate[1::2]
        terminate[1::2] |= terminate[::2]
        reset[terminate] = 1
        reaction[terminate] = False
        recovery[terminate] = False
    return reset, reaction, recovery, distance
