"""ORACLE (test infrastructure, not product code) - float64 restatement of the pose metrics of HumanoidSMPLIMVis' per-motion meters
(cfg.env.b200_pose_metrics; include/b200env.h: b200env_im_motion_stats with the pose fields): per frame the root-relative MPJPE, the
Procrustes-aligned MPJPE (HMR/SPIN's compute_similarity_transform, numpy's SVD), the velocity and acceleration errors over the game's
own frames, and per game the largest body-position error and success.  The games are ref_port_motion_stats.MotionStats' own: this
class extends it, so a game ends, folds and stops exactly where the meters do.  Only tests/ may import this module."""
import numpy as np

from . import ref_port_motion_stats as MS

POSE_COLS = 7   # root-relative, PA, velocity, acceleration sums, velocity frames, acceleration frames, largest body-position error


def pa_aligned(body_pos, target_pos):
    """body_pos [B, 3] aligned to target_pos [B, 3] by the best similarity transform (scale, proper rotation, translation), as
    compute_similarity_transform does it: R from the SVD of K = X1 X2^T with the sign of the last singular direction fixed so that
    det R = 1, scale = tr(R K) / var1.  With no spread in body_pos (var1 = 0) every body lands on the target's centroid."""
    s1, s2 = np.asarray(body_pos, np.float64).T, np.asarray(target_pos, np.float64).T
    mu1, mu2 = s1.mean(1, keepdims=True), s2.mean(1, keepdims=True)
    x1, x2 = s1 - mu1, s2 - mu2
    var1 = np.sum(x1 ** 2)
    if var1 == 0.0:
        return np.repeat(mu2.T, s1.shape[1], 0)
    k = x1 @ x2.T
    u, _, vh = np.linalg.svd(k)
    z = np.eye(3)
    z[-1, -1] *= np.sign(np.linalg.det(u @ vh))
    r = vh.T @ z @ u.T
    scale = np.trace(r @ k) / var1
    return (scale * r @ s1 + (mu2 - scale * r @ mu1)).T


def frame_errors(body_pos, target_pos):
    """one frame's (g, l, pa) [N] each: global, root-relative (body 0 the root) and Procrustes-aligned mean body distances; pa is NaN
    for an env with a non-finite position"""
    p, r = np.asarray(body_pos, np.float64), np.asarray(target_pos, np.float64)
    g = MS.body_pos_err(p, r)
    l = np.linalg.norm((p - p[:, :1]) - (r - r[:, :1]), axis=-1).mean(-1)
    pa = np.full(len(p), np.nan)
    ok = np.isfinite(p).all((1, 2)) & np.isfinite(r).all((1, 2))
    if ok.any():                        # pa_aligned, batched over the envs
        s1, s2 = p[ok], r[ok]
        mu1, mu2 = s1.mean(1, keepdims=True), s2.mean(1, keepdims=True)
        x1, x2 = s1 - mu1, s2 - mu2
        var1 = (x1 ** 2).sum((1, 2))
        k = np.einsum("nbi,nbj->nij", x1, x2)
        u, _, vh = np.linalg.svd(k)
        z = np.tile(np.eye(3), (len(k), 1, 1))
        z[:, -1, -1] = np.sign(np.linalg.det(u @ vh))
        rot = np.swapaxes(vh, 1, 2) @ z @ np.swapaxes(u, 1, 2)
        scale = np.where(var1 > 0, np.trace(rot @ k, axis1=1, axis2=2) / np.where(var1 > 0, var1, 1.0), 0.0)
        aligned = scale[:, None, None] * np.einsum("nij,nbj->nbi", rot, x1) + mu2
        pa[ok] = np.linalg.norm(aligned - s2, axis=-1).mean(-1)
    return g, l, pa


class PoseMetrics(MS.MotionStats):
    """MotionStats with the pose columns: per env the sums of the game so far (env_pose [N, 7], column 6 the largest g, NaN once a
    frame has a non-finite error), its last two frames (prev1 / prev2 [N, B, 3] of body and target positions, fill of them valid;
    a game's end empties them) and per motion pose_sums [M, 7] and success [M] (finished games whose largest g is <= threshold)"""

    def __init__(self, motion_ids, num_motions, threshold=0.5):
        super().__init__(motion_ids, num_motions)
        self.threshold = float(threshold)
        n = len(self.motion_ids)
        self.env_pose, self.pose_sums = np.zeros((n, POSE_COLS)), np.zeros((num_motions, POSE_COLS))
        self.success = np.zeros(num_motions, np.int64)
        self.fill, self.prev1, self.prev2 = np.zeros(n, np.int64), None, None

    def new_game(self):
        super().new_game()
        self.env_pose[:] = 0.0
        self.fill[:] = 0

    def step(self, rew, sub_rewards, reset_buf, terminate_buf, body_pos, target_pos, stop=False):
        if stop:
            return
        p, r = np.asarray(body_pos, np.float64), np.asarray(target_pos, np.float64)
        if self.prev1 is None:
            self.prev1, self.prev2 = (np.zeros((2,) + p.shape), np.zeros((2,) + p.shape))
        g, l, pa = frame_errors(p, r)
        (p1, r1), (p2, r2) = self.prev1, self.prev2
        with np.errstate(invalid="ignore"):
            vel = np.where(self.fill >= 1, np.linalg.norm((p - p1) - (r - r1), axis=-1).mean(-1), 0.0)
            acc = np.where(self.fill >= 2, np.linalg.norm((p - 2 * p1 + p2) - (r - 2 * r1 + r2), axis=-1).mean(-1), 0.0)
        ep = self.env_pose
        ep[:, 0] += l
        ep[:, 1] += pa
        ep[:, 2] += vel
        ep[:, 3] += acc
        ep[:, 4] += self.fill >= 1
        ep[:, 5] += self.fill >= 2
        v = np.where(np.isfinite(np.stack([l, pa, vel, acc])).all(0), g, np.nan)
        ep[:, 6] = nan_max(ep[:, 6], v)
        done = np.asarray(reset_buf) != 0
        ended = done & ~self.prev_done
        self.prev2, self.prev1 = self.prev1, np.stack([p, r])
        self.fill = np.where(ended, 0, np.minimum(self.fill + 1, 2))
        for e in np.flatnonzero(ended):
            m = self.motion_ids[e]
            self.pose_sums[m, :6] += ep[e, :6]
            self.pose_sums[m, 6] = nan_max(self.pose_sums[m, 6], ep[e, 6])
            self.success[m] += int(ep[e, 6] <= self.threshold)
            ep[e] = 0.0
        super().step(rew, sub_rewards, reset_buf, terminate_buf, body_pos, target_pos)


def nan_max(a, b):
    """the larger of a and b, NaN where either is NaN"""
    return np.where(np.isnan(a) | np.isnan(b), np.nan, np.maximum(a, b))
