"""Float64 restatement of HumanoidSMPLIMVis' viewer frame (embodied_pose/env/tasks/humanoid_smpl_im_vis.py: _sync_ref_motion,
convert_dof_pos_to_dof_euler, set_mj_actor_qpos) for any list of envs, and of render_vis' quit rule composed with ImitatorPlayer.run
(oracle/ref_port_im_policy.run_stats).  Test infrastructure: the device launch b200env_im_record and the task's export are held to it."""
import numpy as np

from .ref_port_im_policy import run_stats  # noqa: F401  (the same loop without the recorder)

EPS = 1e-6


def angle_axis_to_quaternion(a):
    """konia angle_axis_to_quaternion (eps 1e-6), wxyz: theta = sqrt(max(|a|^2, eps)); safe_zero_division never adds its eps, since
    theta >= 1e-3"""
    a = np.asarray(a, np.float64)
    th2 = (a * a).sum(-1, keepdims=True)
    th = np.sqrt(np.maximum(th2, EPS))
    k = np.where(th2 > 0, np.sin(th * 0.5) / th, 0.5)
    w = np.where(th2 > 0, np.cos(th * 0.5), 1.0)
    return np.concatenate([w, a * k], -1)


def _safe_atan2(y, x):
    """torch_safe_atan2 with eps 1e-6"""
    y = np.where((np.abs(y) < EPS) & (np.abs(x) < EPS), y + EPS, y)
    return np.arctan2(y, x)


def ypr_euler_from_quat(q):
    """(roll, pitch, yaw) of a wxyz quaternion, handle_singularity False"""
    w, x, y, z = q[..., 0], q[..., 1], q[..., 2], q[..., 3]
    yaw = _safe_atan2(2 * (w * z + x * y), 1 - 2 * (y * y + z * z))
    pitch = np.arcsin(np.clip(2 * (w * y - x * z), -1 + EPS, 1 - EPS))
    roll = _safe_atan2(2 * (w * x + y * z), 1 - 2 * (x * x + y * y))
    return np.stack([roll, pitch, yaw], -1)


def dof_euler(dof_pos):
    """convert_dof_pos_to_dof_euler of one env's dof_pos [nd]: [nd] = per joint (yaw, pitch, roll)"""
    q = angle_axis_to_quaternion(np.asarray(dof_pos, np.float64).reshape(-1, 3))
    return ypr_euler_from_quat(q)[..., [2, 1, 0]].reshape(-1)


def actor_qpos(root_pos, root_rot, dof_pos):
    """set_mj_actor_qpos: pos, the xyzw quaternion as wxyz, the joints' euler angles"""
    return np.concatenate([np.asarray(root_pos, np.float64), np.asarray(root_rot, np.float64)[[3, 0, 1, 2]], dof_euler(dof_pos)])


def sync_ref_motion(rb_pos, rb_rot, dof_pos, p_rb_pos, p_rb_rot, p_dof_pos, env_ids, init):
    """mj_data.qpos as _sync_ref_motion leaves it for each env of env_ids: [E, 3 nq].  rb_pos / rb_rot [N, nb, 3 / 4] (xyzw),
    dof_pos [N, nd], p_rb_pos / p_rb_rot [N, nbl, 3 / 4], p_dof_pos [N, nd]: the task's _rigid_body_*, _dof_pos and _prev_target_*
    (the root row of _prev_target_rb_* is _prev_target_root_*)"""
    out = []
    for e in env_ids:
        c0 = actor_qpos(rb_pos[e, 0], rb_rot[e, 0], dof_pos[e])
        c1 = c0.copy() if init else actor_qpos(p_rb_pos[e, 0], p_rb_rot[e, 0], p_dof_pos[e])
        c2 = c0.copy()
        c2[2] += 1000.0
        c1[0] += 1.0
        out.append(np.concatenate([c0, c1, c2]))
    return np.stack(out)


def run_with_record(games, games_num, max_steps, num_rec_frames, n_game_life=1):
    """ImitatorPlayer.run with render_vis recording: a frame at each game's start (init) and after every step the env ran, the quit
    (SystemExit) when frame num_rec_frames - 1 is written, before that step's done handling.  games as in run_stats.  Returns (lines
    printed before the quit, frames as (game, step) with step -1 for the init frame, quit)."""
    n_games = games_num * n_game_life
    games_played, lines, frames = 0, [], []
    for g, hist in enumerate(games):
        if games_played >= n_games:
            break
        frames.append((g, -1))
        if len(frames) >= num_rec_frames:
            return lines, frames, True
        N = len(hist[0][0])
        cr, steps, prev = np.zeros(N, np.float32), np.zeros(N, np.float32), np.zeros(N, np.float32)
        for n in range(min(max_steps, len(hist))):
            r, done = hist[n]
            done = (np.asarray(done) != 0).astype(np.float32)
            cr = cr + np.asarray(r, np.float32)
            steps = steps + np.float32(1)
            frames.append((g, n))
            if len(frames) >= num_rec_frames:
                return lines, frames, True
            sd = done * (1 - prev)
            idx = np.nonzero(sd)[0]
            games_played += len(idx)
            if len(idx) > 0:
                cur_r, cur_s = float(cr[idx].sum(dtype=np.float32)), float(steps[idx].sum(dtype=np.float32))
                cr = cr * (1 - done)
                steps = steps * (1 - done)
                lines.append((len(idx), cur_r, cur_s))
                if N == 1 or games_played >= n_games:
                    break
            prev = done.copy()
            if done[0]:
                break
    return lines, frames, False
