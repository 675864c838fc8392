"""Float64 restatement of HumanoidSMPLIMVis' per-motion meters (include/b200env.h: b200env_im_motion_stats): per env, the sums of a
game (reward, steps, the four sub-rewards of compute_humanoid_reward, the mean body-position error against the targets the reward
used), folded into the bucket of the env's motion when the game ends on ImitatorPlayer.run's rule (done = reset_buf != 0, a game ends
where done (1 - prev_done)), with the falls (terminate_buf = 1) counted.  Test infrastructure: the device launch and the task's export
are held to it."""
import numpy as np

COLS = 7        # reward, steps, dof, vel, body_pos, body_rot sub-rewards, body-position error


def body_pos_err(body_pos, target_pos):
    """mean over the bodies of |body_pos - target_pos| [N, B, 3] -> [N], in float64"""
    d = np.asarray(body_pos, np.float64) - np.asarray(target_pos, np.float64)
    return np.sqrt((d * d).sum(-1)).mean(-1)


class MotionStats:
    def __init__(self, motion_ids, num_motions):
        self.motion_ids = np.asarray(motion_ids, np.int64)
        n = len(self.motion_ids)
        self.counts = np.zeros((num_motions, 2), np.int64)     # games, falls
        self.sums = np.zeros((num_motions, COLS))
        self.env_sums, self.prev_done = np.zeros((n, COLS)), np.zeros(n, bool)

    def new_game(self):
        """a full reset: the running sums and the done memory start again, the buckets run on"""
        self.env_sums[:] = 0.0
        self.prev_done[:] = False

    def step(self, rew, sub_rewards, reset_buf, terminate_buf, body_pos, target_pos, stop=False):
        """one step's inputs ([N], [N, 4], [N], [N], [N, B, 3], [N, B, 3]); stop: the bookkeeping's stop flag, set by an earlier step"""
        if stop:
            return
        self.env_sums += np.concatenate([np.asarray(rew, np.float64)[:, None], np.ones((len(self.motion_ids), 1)),
                                         np.asarray(sub_rewards, np.float64), body_pos_err(body_pos, target_pos)[:, None]], 1)
        done = np.asarray(reset_buf) != 0
        ended = done & ~self.prev_done
        self.prev_done = done
        for e in np.flatnonzero(ended):
            m = self.motion_ids[e]
            self.counts[m] += (1, int(terminate_buf[e] != 0))
            self.sums[m] += self.env_sums[e]
            self.env_sums[e] = 0.0
