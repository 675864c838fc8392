"""ORACLE (test infrastructure, not product code) - integer restatement of MVAEControllerVisDual's rally results
(cfg.env.b200_rally_stats; include/b200env_v2p.h: b200v2p_eval_rally_stats).  It is composed from ref_port_v2p.dual_controller_reset,
the reference's PhysicsMVAEControllerDual._compute_reset pinned by the cr_* arrays of tests/golden/v2p_dual.npz: `events` splits that
rule's terms into per-player events, `reset_flags` puts them back together into its reset / reaction / recovery (the tests compare
the two on the golden inputs), and every step takes the rally endings from dual_controller_reset itself.  The reference keeps no
meters in dual mode, so the counting has no counterpart there.  Only tests/ may import this module."""
import numpy as np

from . import ref_port_v2p as V

CAUSES = ("behind", "double_bounce", "out")
PLAYER = ("faced", "hits", "forehands")
HIST = 65               # shots per rally 0..63, then 64 = 64 or more
INPUTS = ("tar_action", "has_contact", "has_bounce", "bounce_in", "ball_pos", "root_pos", "swing_type_cycle", "progress_buf")


def events(tar_action, has_contact, has_bounce, ball_pos, root_pos, bounce_in):
    """per env, the terms of dual_controller_reset as events: rec (the player meets the ball), hit, the miss causes and out"""
    ta1, ta0 = np.asarray(tar_action) == 1, np.asarray(tar_action) == 0
    hc, hb, bin_ = (np.asarray(x).astype(bool) for x in (has_contact, has_bounce, bounce_in))
    ball_pos, root_pos = np.asarray(ball_pos, np.float32), np.asarray(root_pos, np.float32)
    behind = ball_pos[:, 1] < root_pos[:, 1] - np.float32(1)
    twice = hb & (ball_pos[:, 2] < np.float32(0.05))
    rec = ta1 & (hc | behind | twice)
    return dict(rec=rec, hit=rec & hc, behind=rec & ~hc & ~twice, double_bounce=rec & ~hc & twice, out=ta0 & hb & ~bin_)


def pair_end(ev):
    """[n/2]: a player of the pair missed or had out"""
    e = ev["behind"] | ev["double_bounce"] | ev["out"]
    return e[0::2] | e[1::2]


def reset_flags(ev, reset_buf):
    """dual_controller_reset's (reset, reaction, recovery) rebuilt from the events: an ending sets reset on both players and clears
    their flags; otherwise a player's rec is its own recovery and its opponent's reaction"""
    end = np.repeat(pair_end(ev), 2)
    reset = np.asarray(reset_buf).copy()
    reset[end] = 1
    opp = np.empty_like(ev["rec"])
    opp[0::2], opp[1::2] = ev["rec"][1::2], ev["rec"][0::2]
    return reset, opp & ~end, ev["rec"] & ~end


class RallyStats:
    """the accumulators and per-pair state of b200v2p_eval_rally_stats for n envs (n / 2 pairs); step() is one launch"""

    def __init__(self, n):
        K = n // 2
        self.n = n
        self.pair_open = np.zeros(K, bool)
        self.pair_hits = np.zeros((K, 2), np.int64)
        self.totals = np.zeros(3, np.int64)          # rallies, shots_sum, frames_sum
        self.ends = np.zeros((2, len(CAUSES)), np.int64)
        self.player = np.zeros((2, len(PLAYER)), np.int64)
        self.shots_hist = np.zeros(HIST, np.int64)

    def arrays(self):
        return dict(pair_open=self.pair_open, pair_hits=self.pair_hits, totals=self.totals, ends=self.ends, player=self.player,
                    shots_hist=self.shots_hist)

    def step(self, s):
        """s: the INPUTS of one launch, as the dual post launch leaves them; returns the [n/2] endings counted"""
        n = self.n
        ev = events(s["tar_action"], s["has_contact"], s["has_bounce"], s["ball_pos"], s["root_pos"], s["bounce_in"])
        b = lambda k: np.asarray(s[k]).astype(bool)  # noqa: E731
        reset = V.dual_controller_reset(np.asarray(s["tar_action"]), b("has_contact"), b("has_bounce"), np.asarray(s["ball_pos"], np.float32),
                                        np.asarray(s["root_pos"], np.float32), np.zeros((n, 3), np.float32), b("bounce_in"),
                                        np.zeros(n, np.float32), np.zeros(n, np.int64))[0]
        assert np.array_equal(reset[0::2] != 0, pair_end(ev)), "the events do not restate the reference's reset rule"
        progress = np.asarray(s["progress_buf"], np.int64)[0::2]
        opening = progress == 1
        act = opening | self.pair_open
        pair = lambda x: x.reshape(-1, 2) & act[:, None]  # noqa: E731
        rec, hit = pair(ev["rec"]), pair(ev["hit"])
        fh = hit & (np.asarray(s["swing_type_cycle"]).reshape(-1, 2) == 1)
        cause = np.stack([pair(ev[c]) for c in CAUSES], -1)                 # [K, 2, 3]
        end = (reset[0::2] != 0) & act
        self.pair_hits[opening] = 0
        self.pair_hits += hit
        shots = self.pair_hits.sum(1)
        self.totals += [end.sum(), shots[end].sum(), progress[end].sum()]
        self.ends += cause.sum(0)
        self.player += np.stack([rec.sum(0), hit.sum(0), fh.sum(0)], -1)
        np.add.at(self.shots_hist, np.minimum(shots[end], HIST - 1), 1)
        self.pair_open = act & ~end
        return end
