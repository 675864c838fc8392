"""Test-time tasks of the tennis controller (vid2player/env/tasks/mvae_controller_vis.py, mvae_controller_vis_dual.py): what
`run.py --test` builds from a controller cfg's `test_name`.  The rollout step is the training task's; what differs:

  MVAEControllerVis      the evaluation reset rule and the four per-env statistics (:64-93), inside the post launch
  both                   render_vis: every call records all envs' frame into device buffers (one launch, no host sync); after
                         num_rec_frames calls the chosen episodes are written as .npz files and SystemExit is raised like the
                         reference's exit()
  MVAEControllerVisDual  the best-episode list of finished rallies (:164-195), kept on the device (two launches per call)
  MVAEControllerVis      with cfg.env.b200_ball_stats on a fixed test set (an addition): per pool row, the balls served and the
                         recovery events with their hits, forehands, bounces in and bounce-in error, counted on the device inside
                         the test loop's reset and step graphs and written by export_ball_stats when run_test ends or the
                         recorder quits
  MVAEControllerVisDual  with cfg.env.b200_rally_stats (an addition): the rallies of the pairs - shots per rally, how each rally
                         ends and which player ended it, each player's balls faced, hits and forehands - counted on the device right
                         after every post launch (inside the step graph) and written by export_rally_stats when run_test ends or
                         the recorder quits

The renderer (SMPL meshes, video, HTML) is not part of this package: the .npz files hold exactly the arrays the reference's
render_one_result is given, so they can be rendered with its visualizer.  Deliberate departures from the reference:
  - a rally longer than the recording capacity keeps its first `capacity` rows (the reference raises IndexError);
  - fewer candidates (single) or list entries (dual) than num_eg: the ones that exist are written (`self.exported` lists them);
  - select_best orders candidates of equal distance by env id (stable sort).
With fix_two_hand_backhand_post (cfgs djokovic, nadal, federer_djokovic, nadal_federer) the written episode also holds
joint_rot_fixed ([T,24,3] single, [2,T,24,3] dual): the rows of the two-hand backhand fix the reference's render_one_result applies
before rendering (optimize_two_hand_backhand, env/tasks/humanoid_smpl_im_mvae.py:948-1031), made for all exported episodes and players
by one device launch (native_v2p.backhand_fix); joint_rot stays as recorded, since render_one_result applies the fix itself.  Dual
mode fixes each player of the pair whose name does not start with 'federer'.  The released optimiser does not run as it stands; the
launch keeps its evident intent: rb_pos is the 7th output of _smpl_to_sim (the reference unpacks nine of eight values), the FK uses
the fixed player's own rest joints for every frame (the reference reads the rest joints of envs 0..M-1), and the device is the
task's (the reference hard-codes cuda:0).  The loss terms the reference prints are kept in `backhand_losses` (episode id -> [3], or
[2,3] in dual mode with NaN for a player left alone).
Reference quirks kept: the meters' avg of an env that never recovered stays 1; the dual recording row 0 of an env is written by the
init call only, and an exported rally is rows [0, progress) - it starts with that row and leaves out the last frame; the dual list
grows only when a candidate beats its current last entry, even while it holds fewer than num_eg.
"""
import math
import os
import warnings
from datetime import datetime

import numpy as np
import torch

from .. import abi, native_v2p
from .physics_mvae_controller import PhysicsMVAEController, PhysicsMVAEControllerDual, resolve_test_set

METERS = ("hit_rate", "fh_ratio", "bounce_in_rate", "bounce_in_pos_error")   # rows of the meter arrays the post launch updates
DUAL_CAPACITY = 1800                                                            # mvae_controller_vis_dual.py:51 "hardcode maximum length"


class AverageMeterUnSync:
    """utils/common.py:40-63 with its tensors on the device: views of row `m` of the [4, N] meter arrays that the post launch
    updates in place for the envs in recovery"""

    def __init__(self, sums, counts, avgs, maxs, m):
        self.sum, self.count, self.avg, self.max = sums[m], counts[m], avgs[m], maxs[m]

    def reset(self):
        self.sum.zero_()
        self.count.zero_()
        self.avg.fill_(1.0)
        self.max.zero_()


def _check_eval_cfg(cfg, headless):
    """refuse what the test-time tasks cannot do, before anything is allocated"""
    env = cfg["env"]
    if int(env.get("num_eg", 1)) < 1:
        raise ValueError("num_eg must be at least 1")
    if int(env.get("num_rec_frames", 300)) < 1:
        raise ValueError("num_rec_frames must be at least 1")
    if not headless and not (env.get("record") or env.get("record_scenepic")):
        raise ValueError("there is no online viewer: run headless, with record to write the episodes")
    env["is_train"] = False          # utils/config.py:159 (--test); also makes the physics task export _joint_rot


def _check_ball_stats_cfg(cfg, dual):
    """b200_ball_stats counts results per row of a fixed test set, which only the single-player task walks in order: refuse it in
    dual mode (no pool is built) and on random draws (test_mode random, the default without ball_traj_file_test: a drawn row keeps no
    identity), before anything is allocated.  The test-time tasks never train (_check_eval_cfg), so the pool is the test set exactly
    when resolve_ball_pool would take it."""
    env = cfg["env"]
    if not env.get("b200_ball_stats", False):
        return
    v2p = dict(env.get("vid2player", {}))
    if dual or v2p.get("dual_mode"):
        raise ValueError("b200_ball_stats: dual mode builds no ball pool, so there are no test-set rows to count results by")
    resolve_test_set(env, v2p)          # on a copy: create_sim applies it to the task's own block
    if v2p.get("test_mode", "random") == "random":
        raise ValueError("b200_ball_stats needs a fixed test set (env.ball_traj_file_test, or vid2player.test_mode single_cycle / "
                         "multiple_cycle with ball_pool_test): random draws keep no row identity")


def _stats_path(env, kind, now):
    """cfg.env.b200_<kind>_file, or out/<kind>/<kind>_<date>.npz"""
    if env.get(f"b200_{kind}_file"):
        return str(env[f"b200_{kind}_file"])
    now = now or datetime.now()
    return os.path.join("out", kind, "%s_%s.npz" % (kind, now.strftime('%Y-%m-%d-%H:%M:%S')))


def ball_stats_path(env, now=None):
    """cfg.env.b200_ball_stats_file, or out/ball_stats/ball_stats_<date>.npz"""
    return _stats_path(env, "ball_stats", now)


def rally_stats_path(env, now=None):
    """cfg.env.b200_rally_stats_file, or out/rally_stats/rally_stats_<date>.npz"""
    return _stats_path(env, "rally_stats", now)


def ball_stats_summary(a):
    """the printed line of the per-row arrays of export_ball_stats: totals, the hit and bounce-in rates over the recovery events (as
    the hit_rate and bounce_in_rate meters take them) and the rows no env ever hit"""
    rec = int(a["recoveries"].sum())
    rate = lambda k: int(a[k].sum()) / rec if rec else float("nan")  # noqa: E731
    return (f"balls served: {int(a['served'].sum())}  recoveries: {rec}  hit rate: {rate('hits'):.4f}  "
            f"bounce-in rate: {rate('bounce_in'):.4f}  rows never hit: {int((a['hits'] == 0).sum())} of {len(a['hits'])}")


def _check_rally_stats_cfg(cfg, dual):
    """b200_rally_stats counts the rallies of the two-player task: refuse it on the single-player one, before anything is allocated"""
    if cfg["env"].get("b200_rally_stats", False) and not dual:
        raise ValueError("b200_rally_stats counts the rallies of MVAEControllerVisDual; the single-player task's per-ball results are "
                         "b200_ball_stats")


def rally_stats_summary(a):
    """the printed line of export_rally_stats: rallies, mean shots per rally, and per player the hit rate hits / faced and the share
    of all rallies it ended by each cause (both players can end the same rally)"""
    R = int(a["rallies"])
    nan = float("nan")
    line = f"rallies: {R}  shots per rally: {int(a['shots_sum']) / R if R else nan:.2f}"
    for w in range(2):
        faced = int(a["faced"][w])
        ends = " ".join(f"{c} {int(a['ends'][w, j]) / R if R else nan:.4f}" for j, c in enumerate(abi.RSTATS_CAUSES))
        line += f"  player {w} ({a['players'][w]}): hit rate {int(a['hits'][w]) / faced if faced else nan:.4f}, ended {ends}"
    return line


class _EvalRecorder:
    """host side shared by both tasks: frame counting, episode paths and the .npz export"""

    def _init_eval(self, cfg):
        env = cfg["env"]
        self.frame_index = 0
        self._record = bool(env.get("record") or env.get("record_scenepic"))
        self._num_rec_frames = int(env.get("num_rec_frames", 300))
        self._num_eg = int(env.get("num_eg", 1))
        self._start_eg_id = int(env.get("start_eg_id", 1))
        self._rec_fname = env.get("rec_fname")
        self._cfg_name = getattr(cfg.get("args"), "cfg", None) or cfg.get("name", "eval")
        self.exported = []
        self._fix_backhand = bool(self.cfg_v2p.get("fix_two_hand_backhand_post"))
        self.backhand_losses = {}
        self._bstats = None              # per-row buckets of b200_ball_stats (MVAEControllerVis)
        self._rstats = None              # pair state and counts of b200_rally_stats (MVAEControllerVisDual)
        self._test_steps = 0

    def _episode_path(self, eg_id):
        return self._rec_fname or os.path.join("out", "episodes", f"{self._cfg_name}_{eg_id:03d}.npz")

    def _write(self, eg_id, arrays):
        path = self._episode_path(eg_id)
        os.makedirs(os.path.dirname(path) or ".", exist_ok=True)
        with open(path, "wb") as f:
            np.savez(f, **{k: v.cpu().numpy() if torch.is_tensor(v) else np.asarray(v) for k, v in arrays.items()})
        self.exported.append(path)

    def _players(self):
        """(skip, righthand) of player j of a pair: mvae_controller_vis_dual.py:216-223"""
        v = self.cfg_v2p
        for j in range(2):
            if v.get("dual_mode") == "different":
                player, rh = v["player"][j], v["righthand"][j]
            else:
                player, rh = v.get("player"), v.get("righthand", True)
            yield str(player).startswith("federer"), bool(rh)

    def _tensors(self):
        t = super()._tensors()
        t.update(getattr(self, "_policy_t", {}))
        return t

    def render_vis(self, init=False):
        """the reference's render_vis without the renderer: record the frame of every env (device launches); after num_rec_frames
        calls write the chosen episodes and raise SystemExit"""
        self._record_frame()
        self._render_host()

    def _render_host(self):
        self.frame_index += 1
        if self._record and self.frame_index >= self._num_rec_frames:
            self.export_episodes()
            self._export_stats()
            raise SystemExit(0)

    def _export_stats(self):
        if self._bstats is not None:
            self.export_ball_stats()
        if self._rstats is not None:
            self.export_rally_stats()

    # ------------------------------------------------------------------ test loop of V2PPlayer.run (players/v2p_player.py:133-156)
    def set_policy(self, policy):
        """the high-level policy of the test loop (nn.V2PPolicy).  From now on every post launch, the reset's observation refresh
        included, also writes the policy's operand rows, so the policy needs no launch of its own before its layers.  Set it before
        reset(), which writes the first rows."""
        if policy.rows != self.num_envs or policy.in_dim != self.num_obs or policy.dual != bool(self._post_cfg.get("dual")):
            raise ValueError("the policy's env count, observation width or dual mode differs from the task's")
        cfg, t = policy.operand()
        self._post_cfg.update(cfg)
        self._policy_t, self._policy = t, policy
        self._test_mask = torch.zeros(self.num_envs, device=self.device, dtype=torch.bool)
        self._test_graphs = None

    def run_test(self, policy, max_steps, graph=True):
        """V2PPlayer.run with the policy's action (deterministic mu, or sampled for an nn.V2PPolicy built with deterministic=False: the
        noise is drawn inside the policy's last layer, so the graphs replay it afresh): reset, render_vis(init=True), then `max_steps`
        test_step() calls.  Ends like
        the reference, with SystemExit once num_rec_frames frames are recorded (with record).  With b200_ball_stats the per-row
        buckets are written when the run returns, or before that SystemExit; they count from the task's construction, so the first
        reset's draws are in them whether it ran here or before.  b200_rally_stats' counts are written at the same points; they count
        every post launch since the task's construction, step() included."""
        self.set_policy(policy)
        self.reset()
        self.render_vis(init=True)
        for _ in range(max_steps):
            self.test_step(graph)
        self._export_stats()

    def test_step(self, graph=True):
        """one iteration of V2PPlayer.run's loop: reset of the finished envs (mask-driven, from reset_buf), policy, env step,
        render_vis.  graph=True: the first iteration runs eagerly (one-time set-up of the launches), then the reset and the rest are
        captured as two CUDA graphs and every later iteration is two replays; the host only counts frames."""
        if self._test_graphs is not None:
            for g in self._test_graphs:
                g.replay()
        else:
            self._test_reset()
            self._test_launches()
            if graph:
                torch.cuda.synchronize()
                rg, sg = torch.cuda.CUDAGraph(), torch.cuda.CUDAGraph()
                with torch.cuda.graph(rg):
                    self._test_reset()
                with torch.cuda.graph(sg, pool=rg.pool()):
                    self._test_launches()
                self._test_graphs = (rg, sg)
        self._test_steps += 1
        self._render_host()

    def _test_reset(self):
        torch.ne(self.reset_buf, 0, out=self._test_mask)
        self._reset_envs_masked(self._test_mask)

    def _test_launches(self):
        with torch.no_grad():
            actions = self._policy.forward_prepared()
        self.pre_physics_step(actions)
        self.physics_step()
        self.post_physics_step()
        if self._bstats is not None:
            self._ball_stats_launch()
        self._record_frame()

    def _rec_buffers(self, n, cap, fields):
        dev = self.device
        shapes = dict(joint_rot=((24, 3), torch.float), root_pos=((3,), torch.float), ball_pos=((3,), torch.float),
                      target_pos=((3,), torch.float), phase=((), torch.float), swing_type=((), torch.long), tar_action=((), torch.long))
        return {k: torch.zeros((*n, cap, *shapes[k][0]), device=dev, dtype=shapes[k][1]) for k in fields}


class MVAEControllerVis(_EvalRecorder, PhysicsMVAEController):
    def __init__(self, cfg, sim_params, physics_engine, device_type, device_id, headless):
        _check_eval_cfg(cfg, headless)
        _check_ball_stats_cfg(cfg, dual=False)
        _check_rally_stats_cfg(cfg, dual=False)
        super().__init__(cfg=cfg, sim_params=sim_params, physics_engine=physics_engine, device_type=device_type, device_id=device_id,
                         headless=headless)
        self._init_eval(cfg)
        N, dev = self.num_envs, self.device
        self._meter_sum = torch.zeros(4, N, device=dev)
        self._meter_count = torch.zeros(4, N, device=dev, dtype=torch.long)
        self._meter_avg = torch.ones(4, N, device=dev)
        self._meter_max = torch.zeros(4, N, device=dev)
        for m, name in enumerate(METERS):
            setattr(self, name, AverageMeterUnSync(self._meter_sum, self._meter_count, self._meter_avg, self._meter_max, m))
        # :64-79 compares progress with cfg.env.episodeLength (default 600) itself, strictly
        self._post_cfg.update(eval=1, eval_episode_length=int(cfg["env"].get("episodeLength", 600)))
        if self._record:
            self._rec = self._rec_buffers((N,), self._num_rec_frames,
                                          ("joint_rot", "root_pos", "ball_pos", "target_pos", "phase", "swing_type"))
            self._rec_row = torch.zeros(1, device=dev, dtype=torch.long)
            self._rec_done = torch.zeros(1, device=dev, dtype=torch.int32)
        if cfg["env"].get("b200_ball_stats", False):
            task = self._physics_player.task
            P = int(task._ball_pool.shape[0])
            self._bstats = dict(served=torch.zeros(P, device=dev, dtype=torch.long),
                                buckets=torch.zeros(P, abi.BSTATS_COLS, device=dev, dtype=torch.long))
            task._ball_row_served = self._bstats["served"]      # both reset paths count their draws into it

    def _tensors(self):
        t = super()._tensors()
        t.update(ball_vel=self._physics_player.task._ball_vel, meter_sum=self._meter_sum, meter_count=self._meter_count,
                 meter_avg=self._meter_avg, meter_max=self._meter_max)
        return t

    def _record_frame(self):
        """:95-170's per-call device work: every env's frame into the recording (one launch)"""
        if not self._record:
            return
        t, p = self._physics_player.task, self._mvae_player
        native_v2p.eval_record(self.num_envs, self._num_rec_frames, dict(
            row_counter=self._rec_row, done_counter=self._rec_done, joint_rot=t._joint_rot, root_pos=t._root_pos, ball_pos=t._ball_pos,
            target_pos=self._target_bounce_pos, phase=p._phase_pred, swing_type=p._swing_type_cycle,
            **{"rec_" + k: v for k, v in self._rec.items()}))

    def _ball_stats_launch(self):
        """right after the post launch: every recovery event into the bucket of the row its env plays (b200v2p_eval_ball_stats)"""
        t = self._physics_player.task
        native_v2p.eval_ball_stats(dict(n=self.num_envs, pool_size=int(t._ball_pool.shape[0])), dict(
            pool_cursor=t._ball_pool_cursor, reset_recovery=self._reset_recovery_buf, has_contact=t._has_racket_ball_contact,
            swing_type_cycle=self._mvae_player._swing_type_cycle.contiguous(), est_bounce_in=self._est_bounce_in,
            est_bounce_pos=self._est_bounce_pos, target_bounce_pos=self._target_bounce_pos, buckets=self._bstats["buckets"]))

    def export_ball_stats(self):
        """writes the per-row results of the test set to b200_ball_stats_file and prints the summary line; returns the file's path.
        served, recoveries, hits, forehands, bounce_in: int64 [P]; bounce_err_sum: float64 [P], metres (the fixed-point sums over
        2^24); ball_traj_file_test ('' for an in-memory ball_pool_test), num_envs, test_steps."""
        b = self._bstats["buckets"].cpu().numpy()
        a = dict(served=self._bstats["served"].cpu().numpy(), recoveries=b[:, 0].copy(), hits=b[:, 1].copy(), forehands=b[:, 2].copy(),
                 bounce_in=b[:, 3].copy(), bounce_err_sum=b[:, 4] / abi.BSTATS_FIX_SCALE)
        path = ball_stats_path(self.cfg["env"])
        if os.path.dirname(path):
            os.makedirs(os.path.dirname(path), exist_ok=True)
        np.savez(path, **a, ball_traj_file_test=np.array(str(self.cfg_v2p.get("ball_traj_file_test") or "")),
                 num_envs=np.int64(self.num_envs), test_steps=np.int64(self._test_steps))
        print(ball_stats_summary(a))
        print(f"============ per-ball statistics written to {path} ============")
        return path

    def select_candidates(self):
        """:152-159: with select_best the envs with bounce_in_rate.avg > 0.95 and fh_ratio.avg < 0.6, by distance travelled over the
        recording, longest first; otherwise every env in order"""
        if not self.cfg["env"].get("select_best"):
            return torch.arange(self.num_envs, device=self.device)
        rp = self._rec["root_pos"]
        dist = (rp[:, 1:] - rp[:, :-1]).norm(dim=-1).sum(dim=-1)
        cand = (self.bounce_in_rate.avg > 0.95) & (self.fh_ratio.avg < 0.6)
        ids = cand.nonzero(as_tuple=False).flatten()
        return ids[torch.argsort(dist[cand], descending=True, stable=True)]

    def export_episodes(self):
        ids = self.select_candidates()[:self._num_eg].tolist()
        if len(ids) < self._num_eg:
            warnings.warn(f"{len(ids)} of the {self._num_eg} requested episodes qualify; writing those", stacklevel=2)
        fixed = {}
        if self._fix_backhand and ids:
            rest, rh = self._physics_player.task._rest_t[0], bool(self.cfg_v2p.get("righthand", True))
            outs, losses = native_v2p.backhand_fix([dict(joint_rot=self._rec["joint_rot"][e], phase=self._rec["phase"][e],
                                                    swing_type=self._rec["swing_type"][e], rest=rest, righthand=rh) for e in ids],
                                                   iters=native_v2p.BACKHAND_ITERS)
            for i, e in enumerate(ids):
                fixed[e] = dict(joint_rot_fixed=outs[i])
                self.backhand_losses[self._start_eg_id + i] = losses[i].cpu().numpy()
        for i, e in enumerate(ids):
            self._write(self._start_eg_id + i, dict(env_id=e, **{k: v[e] for k, v in self._rec.items()}, **fixed.get(e, {})))
        return self.exported


class MVAEControllerVisDual(_EvalRecorder, PhysicsMVAEControllerDual):
    def __init__(self, cfg, sim_params, physics_engine, device_type, device_id, headless, capacity=DUAL_CAPACITY):
        _check_eval_cfg(cfg, headless)
        _check_ball_stats_cfg(cfg, dual=True)
        _check_rally_stats_cfg(cfg, dual=True)
        super().__init__(cfg=cfg, sim_params=sim_params, physics_engine=physics_engine, device_type=device_type, device_id=device_id,
                         headless=headless)
        self._init_eval(cfg)
        self._cap = int(capacity)
        if cfg["env"].get("b200_rally_stats", False):
            i64 = lambda *s: torch.zeros(*s, device=self.device, dtype=torch.long)  # noqa: E731
            K = self.num_envs // 2
            self._rstats = dict(pair_open=torch.zeros(K, device=self.device, dtype=torch.bool), pair_hits=i64(K, 2), totals=i64(3),
                                ends=i64(2, len(abi.RSTATS_CAUSES)), player=i64(2, len(abi.RSTATS_PLAYER)), shots_hist=i64(abi.RSTATS_HIST))
        if self._record:
            N, E, dev = self.num_envs, self._num_eg, self.device
            fields = ("joint_rot", "root_pos", "ball_pos", "phase", "swing_type", "tar_action")
            self._rec = self._rec_buffers((N,), self._cap, fields)
            self._best = self._rec_buffers((E, 2), self._cap, fields)
            i64 = lambda *s: torch.zeros(*s, device=dev, dtype=torch.long)  # noqa: E731
            self._list = dict(list_len=i64(1), order=i64(E), best_distance=torch.zeros(E, device=dev), best_env=i64(E),
                              best_nframes=i64(E), copy_slot=i64(1))

    def _record_frame(self):
        """:87-202's per-call device work: record the frame of every env at row progress_buf, update the best-episode list with the
        rallies that ended on this step (two launches; the list's decisions are made on the device)"""
        if not self._record:
            return
        t, p = self._physics_player.task, self._mvae_player
        rec = {"rec_" + k: v for k, v in self._rec.items()}
        native_v2p.eval_record(self.num_envs, self._cap, dict(
            progress_buf=self.progress_buf, joint_rot=t._joint_rot, root_pos=t._root_pos, ball_pos=t._ball_pos, phase=p._phase_pred,
            swing_type=p._swing_type_cycle, tar_action=self._tar_action, **rec))
        native_v2p.eval_best(self.num_envs, self._cap, self._num_eg, dict(
            reset_buf=self.reset_buf, progress_buf=self.progress_buf, distance=self._distance, **self._list, **rec,
            **{"best_" + k: v for k, v in self._best.items()}))

    def post_physics_step(self):
        """the step's post launch, then with b200_rally_stats the pairs' rally results from its flags (b200v2p_eval_rally_stats), so that
        step(), its graph and run_test's step graph all count"""
        super().post_physics_step()
        if self._rstats is not None:
            t = self._physics_player.task
            native_v2p.eval_rally_stats(dict(n=self.num_envs), dict(
                tar_action=self._tar_action, has_contact=t._has_racket_ball_contact, has_bounce=t._has_bounce, bounce_in=self._bounce_in,
                ball_pos=t._ball_pos, root_pos=t._root_pos, swing_type_cycle=self._mvae_player._swing_type_cycle.contiguous(),
                progress_buf=self.progress_buf, **self._rstats))

    def rally_players(self):
        """the cfg's players of a pair: the `player` pair in dual_mode different, else the one player twice"""
        v = self.cfg_v2p
        return [str(p) for p in v["player"]] if v.get("dual_mode") == "different" else [str(v.get("player"))] * 2

    def export_rally_stats(self):
        """writes the rally results to b200_rally_stats_file and prints the summary line; returns the file's path.  int64: rallies,
        shots_sum, frames_sum, shots_hist [65] (shots per rally 0..63, then 64 or more), ends [2, 3] by end_causes, faced, hits,
        forehands [2], open_rallies and open_hits [open, 2] (the pairs still in a rally), num_envs, test_steps; players [2]."""
        r = {k: v.cpu().numpy() for k, v in self._rstats.items()}
        pl = r["player"]
        a = dict(rallies=r["totals"][0], shots_sum=r["totals"][1], frames_sum=r["totals"][2], shots_hist=r["shots_hist"], ends=r["ends"],
                 end_causes=np.array(abi.RSTATS_CAUSES), **{k: pl[:, j].copy() for j, k in enumerate(abi.RSTATS_PLAYER)},
                 open_rallies=np.int64(r["pair_open"].sum()), open_hits=r["pair_hits"][r["pair_open"]],
                 players=np.array(self.rally_players()), num_envs=np.int64(self.num_envs), test_steps=np.int64(self._test_steps))
        path = rally_stats_path(self.cfg["env"])
        if os.path.dirname(path):
            os.makedirs(os.path.dirname(path), exist_ok=True)
        np.savez(path, **a)
        print(rally_stats_summary(a))
        print(f"============ rally statistics written to {path} ============")
        return path

    def best_list(self):
        """the list in rank order: (slot, even env of the pair, distance, frames) per entry"""
        L = int(self._list["list_len"].item())
        slots = self._list["order"][:L].tolist()
        return [(s, int(self._list["best_env"][s]), float(self._list["best_distance"][s]), int(self._list["best_nframes"][s])) for s in slots]

    def export_episodes(self):
        entries = self.best_list()
        if len(entries) < self._num_eg:
            warnings.warn(f"{len(entries)} of the {self._num_eg} requested episodes were kept; writing those", stacklevel=2)
        fixed = {}
        if self._fix_backhand and entries:
            rest_t = self._physics_player.task._rest_t          # [K,24,3]: player j of a pair has shape j % K
            problems, slots = [], []
            for i, (s, e, d, nf) in enumerate(entries):
                fixed[i] = self._best["joint_rot"][s, :, :nf].clone()
                for j, (skip, rh) in enumerate(self._players()):
                    if not skip:
                        problems.append(dict(joint_rot=self._best["joint_rot"][s, j, :nf], phase=self._best["phase"][s, j, :nf],
                                             swing_type=self._best["swing_type"][s, j], rest=rest_t[j % rest_t.shape[0]], righthand=rh,
                                             out=fixed[i][j]))
                        slots.append((i, j))
            losses = native_v2p.backhand_fix(problems, iters=native_v2p.BACKHAND_ITERS)[1].cpu().numpy() if problems else np.zeros((0, 3))
            for i in range(len(entries)):
                self.backhand_losses[self._start_eg_id + i] = np.full((2, 3), math.nan)
            for (i, j), row in zip(slots, losses):
                self.backhand_losses[self._start_eg_id + i][j] = row
        for i, (s, e, d, nf) in enumerate(entries):
            extra = dict(joint_rot_fixed=fixed[i]) if i in fixed else {}
            self._write(self._start_eg_id + i, dict(env_ids=np.array([e, e + 1]), distance=np.float32(d),
                                                    **{k: v[s, :, :nf] for k, v in self._best.items()}, **extra))
        return self.exported
