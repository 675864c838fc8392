"""Integer / float64 restatement of the motion queue of HumanoidSMPLIMVis (include/b200env.h: b200env_im_motion_queue and the queue
form of b200env_play_stats): the queue holds the entries q = r M + m of R rounds of an M-motion library; env e starts on entry e.  Per
step, after the env step:
  - the bookkeeping counts the games that ended (done = reset_buf != 0, a game ends where done rises, ImitatorPlayer.run's rule),
    advances the step counter, and stops the run once R M games have finished;
  - the assignment walks the envs in env order: the k-th finished env that is not idle takes entry cursor + k while the queue lasts
    (its motion id, entry and reset mask are set, its done memory is cleared, and the entry records the env and the step
    counter), and becomes idle otherwise;
    the cursor moves by the entries taken.  While stopped it sets no mask and changes nothing.
QueueRun composes it with ref_port_motion_stats.MotionStats, or with ref_port_pose_metrics.PoseMetrics for the pose metrics, whose
buckets are then the entries: a game is folded into the row of the entry it played.  Test infrastructure: the device launches and the
task's export are held to it."""
import numpy as np

from .ref_port_motion_stats import MotionStats
from .ref_port_pose_metrics import PoseMetrics, nan_max


class MotionQueue:
    def __init__(self, num_envs, num_motions, rounds):
        if not 1 <= num_envs <= num_motions * rounds:
            raise ValueError(f"{num_envs} envs for a queue of {num_motions} x {rounds}")
        self.N, self.M, self.Q = num_envs, num_motions, num_motions * rounds
        self.entry = np.arange(num_envs, dtype=np.int64)
        self.motion_ids = self.entry % num_motions
        self.idle = np.zeros(num_envs, bool)
        self.cursor = num_envs
        self.game_env = np.full(self.Q, -1, np.int64)
        self.game_env[:num_envs] = self.entry
        self.game_start_step = np.full(self.Q, -1, np.int64)
        self.game_start_step[:num_envs] = 0
        self.prev_done = np.zeros(num_envs, bool)
        self.games, self.step_count, self.stop = 0, 0, False

    def bookkeeping(self, reset_buf):
        """b200env_play_stats' queue form: the games that ended, the step counter and the stop flag"""
        if self.stop:
            return
        done = np.asarray(reset_buf) != 0
        self.games += int((done & ~self.prev_done).sum())
        self.prev_done = done
        self.step_count += 1
        self.stop = self.games >= self.Q

    def assign(self, reset_buf):
        """b200env_im_motion_queue: the reset mask [N] bool of the envs that took an entry"""
        mask = np.zeros(self.N, bool)
        if self.stop:
            return mask
        fin = np.flatnonzero((np.asarray(reset_buf) != 0) & ~self.idle)
        q = self.cursor + np.arange(len(fin))
        take = q < self.Q
        e, q = fin[take], q[take]
        self.motion_ids[e], self.entry[e], mask[e] = q % self.M, q, True
        self.game_env[q], self.game_start_step[q] = e, self.step_count
        self.prev_done[e] = False
        self.idle[fin[~take]] = True
        self.cursor += len(e)
        return mask


class QueueRun:
    """the queue with the per-entry meters: step() takes one step's inputs as the device sees them before the queue's reset.
    pose_threshold: with a success threshold the stats are PoseMetrics (pose_sums and success per entry as well)"""

    def __init__(self, num_envs, num_motions, rounds, pose_threshold=None):
        self.queue = MotionQueue(num_envs, num_motions, rounds)
        ids = np.zeros(num_envs, np.int64)
        self.stats = MotionStats(ids, self.queue.Q) if pose_threshold is None else PoseMetrics(ids, self.queue.Q, pose_threshold)
        self.stats.motion_ids = self.queue.entry                    # the rows are the entries, read at the fold

    def step(self, rew, sub_rewards, reset_buf, terminate_buf, body_pos, target_pos):
        """the meters (which fold before the assignment moves an env to its next entry), the bookkeeping, then the assignment;
        returns the reset mask"""
        self.stats.step(rew, sub_rewards, reset_buf, terminate_buf, body_pos, target_pos, stop=self.queue.stop)
        self.queue.bookkeeping(reset_buf)
        mask = self.queue.assign(reset_buf)
        self.stats.prev_done[mask] = False
        return mask

    def fold(self, rows, max_col=None):
        """rows [R M, ...] -> [M, ...]: the R rows of each motion added in round order; column max_col by the NaN-propagating max"""
        R, M = self.queue.Q // self.queue.M, self.queue.M
        r = rows.reshape((R, M) + rows.shape[1:])
        out = r[0].copy()
        for k in range(1, R):
            top = out[:, max_col].copy() if max_col is not None else None
            out += r[k]
            if max_col is not None:
                out[:, max_col] = nan_max(top, r[k][:, max_col])
        return out

    def per_motion(self):
        """(counts [M, 2], sums [M, 7]) per motion"""
        return self.fold(self.stats.counts), self.fold(self.stats.sums)

    def per_motion_pose(self):
        """(pose_sums [M, 7], success [M]) per motion, the largest error (column 6) by the NaN-propagating max"""
        return self.fold(self.stats.pose_sums, max_col=6), self.fold(self.stats.success)
