"""ORACLE (test infrastructure, not product code) - float64 restatement of MVAEControllerVis' per-row results of the fixed test set
(cfg.env.b200_ball_stats; include/b200env_v2p.h: b200v2p_eval_ball_stats and b200v2p_treset_t.row_served).  It is composed from what
is already pinned: the draws and the cursor walk of ref_port_test_set (tests/golden/v2p_ball_test_set.npz) and the recovery events
and meter values of ref_port_eval.eval_reset (tests/golden/v2p_eval.npz).  The reference keeps per-env meters only
(env/tasks/mvae_controller_vis.py:80-93), so the per-row folding has no counterpart there: an event goes to the row its env plays,
the row of its last draw.  Only tests/ may import this module."""
import numpy as np

from . import ref_port_eval as E
from . import ref_port_test_set as T

F32 = np.float32
COUNTS = ("recoveries", "hits", "forehands", "bounce_in")


def bounce_err(est_bounce_pos, target_bounce_pos):
    """the value meter 3 takes for a bounce-in event (ref_port_eval.eval_reset): the distance, in float32"""
    d = (np.asarray(est_bounce_pos, F32) - np.asarray(target_bounce_pos, F32)).astype(F32)
    return np.sqrt((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]).astype(F32)


def playing_row(cursor, pool_size):
    """the row an env plays: its last draw's, one behind the cursor, which moves by one (mod P) at each draw only"""
    return (np.asarray(cursor, np.int64) + pool_size - 1) % pool_size


class BallStats:
    def __init__(self, pool_size):
        self.P = int(pool_size)
        self.served = np.zeros(self.P, np.int64)
        for k in COUNTS:
            setattr(self, k, np.zeros(self.P, np.int64))
        self.bounce_err_sum = np.zeros(self.P)

    def arrays(self):
        return dict(served=self.served, **{k: getattr(self, k) for k in COUNTS}, bounce_err_sum=self.bounce_err_sum)

    def generate(self, pool, cursor, env_ids):
        """ref_port_test_set.generate (the id-list draw), each drawn row counted as served"""
        out = T.generate(pool, cursor, env_ids)
        np.add.at(self.served, out[0], 1)
        return out

    def task_reset(self, s, cfg, draws, cursor):
        """ref_port_test_set.task_reset (the mask-driven draw), the rows of its reaction envs counted as served"""
        rea = np.flatnonzero(s["reset_reaction"])
        np.add.at(self.served, np.asarray(cursor, np.int64)[rea], 1)
        return T.task_reset(s, cfg, draws, cursor)

    def events(self, s, recovery, cursor):
        """the recovery events of one eval_reset (flags `recovery` on its input state s) into the rows their envs play"""
        ids = np.flatnonzero(recovery)
        rows = playing_row(np.asarray(cursor)[ids], self.P)
        np.add.at(self.recoveries, rows, 1)
        np.add.at(self.hits, rows, s["has_contact"][ids].astype(bool))
        np.add.at(self.forehands, rows, np.asarray(s["swing_type_cycle"])[ids] == 1)
        bin_ = s["est_bounce_in"][ids].astype(bool)
        np.add.at(self.bounce_in, rows, bin_)
        ins = ids[bin_]
        np.add.at(self.bounce_err_sum, rows[bin_], bounce_err(s["est_bounce_pos"][ins], s["target_bounce_pos"][ins]).astype(np.float64))

    def eval_reset(self, s, episode_length, M, cursor):
        """ref_port_eval.eval_reset (flags and per-env meters M), then its recovery events into the rows"""
        out = E.eval_reset(s, episode_length, M)
        self.events(s, out[2], cursor)
        return out
