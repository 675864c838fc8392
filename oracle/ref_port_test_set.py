"""ORACLE (test infrastructure, not product code) - numpy restatement of the fixed test set of incoming balls: the sequential branch of
TennisBallGeneratorOffline.generate (utils/tennis_ball.py:444-447, sample_random False) and the test_mode rule of
env/utils/player_builder.py:154-156.  Paths are relative to /root/reference/vid2player.  Pinned against
tests/golden/v2p_ball_test_set.npz, made by executing the reference's own generator (tests/golden/make_golden_test_set.py).
Only tests/ may import this module."""
import numpy as np

from . import ref_port_v2p as V


def mode_of(path):
    """the test_mode a ball_traj_file_test sets (player_builder.py:156)"""
    return 'single_cycle' if 'single' in path else 'multiple_cycle'


def generate(pool, cursor, env_ids):
    """generate(n, need_init_state=True, start_pos=..., env_ids) of the sequential branch (:445-447): the rows of env_ids are their
    cursors, each cursor then moves on by one modulo the pool size; start_pos is not looked at.  Returns (indices, traj [n,100,3],
    launch_pos, launch_vel, launch_vspin) and moves cursor [N] int64 in place"""
    env_ids = np.asarray(env_ids, np.int64)
    idx = cursor[env_ids].copy()
    cursor[env_ids] = (idx + 1) % len(pool)
    row = pool[idx]
    return idx, row[:, 7:].reshape(-1, 100, 3), row[:, 0:3], row[:, 3:6], row[:, 6]


def task_reset(s, cfg, draws, cursor):
    """ref_port_v2p.task_reset on the test set: each reaction env takes pool row cursor[e] (its ball's side is not looked at, pool_rand
    and side_rand are not used) and moves its cursor on; everything after the choice of the row is the random branch's.  Returns
    (updated copy of s, updated copy of cursor)."""
    rea = np.flatnonzero(s["reset_reaction"])
    s2 = dict(s, ball_pos=s["ball_pos"].copy())
    s2["ball_pos"][rea, 1] = -1            # near side: pool_index takes pool_rand, here the cursor; task_reset overwrites these rows
    out = V.task_reset(s2, cfg, dict(draws, pool_rand=np.asarray(cursor, np.int64)))
    cursor = np.array(cursor, np.int64)
    cursor[rea] = (cursor[rea] + 1) % len(cfg["pool"])
    return out, cursor
