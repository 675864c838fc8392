"""Float32 numpy restatement of the test-time tasks' device work (vid2player/env/tasks/mvae_controller_vis.py,
mvae_controller_vis_dual.py), what the eval launches of csrc/b200env_v2p.cu are tested against:

  eval_reset   MVAEControllerVis._compute_reset + _compute_stats (:64-93) with AverageMeterUnSync.update (utils/common.py:52-63)
  record       the per-frame append of render_vis (:140-146; dual :156-162), rows past the capacity dropped
  best_update  the best-episode list of MVAEControllerVisDual.render_vis (:164-195), as a rank-ordered Python list
  select_best  the candidate order of MVAEControllerVis.render_vis (:152-159)
"""
import numpy as np

F32 = np.float32
METERS = ("hit_rate", "fh_ratio", "bounce_in_rate", "bounce_in_pos_error")


def new_meters(n):
    return dict(sum=np.zeros((4, n), F32), count=np.zeros((4, n), np.int64), avg=np.ones((4, n), F32), max=np.zeros((4, n), F32))


def meter_update(M, m, val, ids):
    val = np.asarray(val, F32)
    M["sum"][m, ids] = M["sum"][m, ids] + val
    M["count"][m, ids] += 1
    nz = M["count"][m] > 0
    M["avg"][m, nz] = M["sum"][m, nz] / M["count"][m, nz].astype(F32)
    M["max"][m, ids] = np.where(val > M["max"][m, ids], val, M["max"][m, ids])


def eval_reset(s, episode_length, M):
    """s: progress, tar_time, tar_time_total, tar_action, swing_type_cycle [n] int64; has_contact, has_bounce, est_bounce_in [n] bool;
    ball_pos, root_pos, ball_vel, est_bounce_pos, target_bounce_pos [n,3] float32.  Updates the meters M in place; returns
    (terminate, reaction, recovery)."""
    hc, ta = s["has_contact"].astype(bool), s["tar_action"]
    terminate = s["progress"] > episode_length
    in_time = s["tar_time"] >= s["tar_time_total"]
    reaction = (hc & (ta == 0) & s["has_bounce"].astype(bool) & in_time) | (~hc & in_time)
    recovery = (ta == 1) & (hc | (s["ball_pos"][:, 1] < s["root_pos"][:, 1] - F32(1)) | (np.abs(s["ball_vel"][:, 1]) < F32(2)))
    reaction = reaction | terminate
    recovery = recovery & ~terminate
    ids = np.nonzero(recovery)[0]
    if len(ids):
        meter_update(M, 0, hc[ids], ids)
        meter_update(M, 1, s["swing_type_cycle"][ids] == 1, ids)
        bin_ = s["est_bounce_in"].astype(bool)
        meter_update(M, 2, bin_[ids], ids)
        ins = ids[bin_[ids]]
        if len(ins):
            d = (s["est_bounce_pos"][ins] - s["target_bounce_pos"][ins]).astype(F32)
            meter_update(M, 3, np.sqrt((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]).astype(F32), ins)
    return terminate, reaction, recovery


def record(rec, rows, frame):
    """rec: field -> [n, cap, ...]; rows [n] (the single recorder's frame counter broadcast, or progress_buf); frame: field -> [n, ...]"""
    n = len(rows)
    for k, buf in rec.items():
        ok = (rows >= 0) & (rows < buf.shape[1])
        buf[np.arange(n)[ok], rows[ok]] = frame[k][ok]


def best_update(best, reset_buf, distance, progress, rec, num_eg):
    """best: list of dict(distance, env, nframes, arrays) in rank order, updated in place like the reference's parallel lists"""
    pairs = np.nonzero(reset_buf[0::2] != 0)[0]
    if len(pairs) == 0:
        return None
    d = (distance[2 * pairs] + distance[2 * pairs + 1]).astype(F32)
    i = int(np.argmax(d))
    mx, k = d[i], int(pairs[i])
    if best and not mx > best[-1]["distance"]:
        return None
    ins = 0
    while ins < len(best) and not mx > best[ins]["distance"]:
        ins += 1
    cap = next(iter(rec.values())).shape[1]
    nf = int(min(progress[2 * k], cap))
    best.insert(ins, dict(distance=mx, env=2 * k, nframes=nf, arrays={f: v[2 * k:2 * k + 2, :nf].copy() for f, v in rec.items()}))
    del best[num_eg:]
    return ins


def select_best(root_pos_rec, bounce_in_avg, fh_avg):
    """candidate env ids, longest distance travelled over the recording first (ties by env id)"""
    rp = root_pos_rec.astype(F32)
    dist = np.sqrt(((rp[:, 1:] - rp[:, :-1]) ** 2).sum(-1)).sum(-1)
    cand = np.nonzero((bounce_in_avg > 0.95) & (fh_avg < 0.6))[0]
    return cand[np.argsort(-dist[cand], kind="stable")]
