"""HumanoidSMPLIMVis mirror (embodied_pose/env/tasks/humanoid_smpl_im_vis.py): the task `run.py --test` builds from the imitation cfgs'
`test_name`, and the test loop of ImitatorPlayer.run (embodied_pose/players/im_player.py:193-312) with the deterministic action, or the
sampled one of a stochastic player (a network dict with `sigma`, nn.im_networks_from_checkpoint(..., deterministic=False)).

The loop runs on the device.  Per step, one CUDA graph replays four pieces:
  - the policy's operand launch (include/b200env.h: b200env_im_policy_rows): the network's 734-wide observation from obs_buf and the
    context slot of the device step counter, normalised and cast to bf16, and that slot's target dof_pos;
  - the four wgmma layers of nn.PolicyMLP; the last one adds the target dof_pos (the residual action), for a stochastic player then
    sigma * N(0, 1) (counter-based, seeded by cfg["seed"], its step counter advanced by the launch itself), and applies the wrapper's
    action clamp in its epilogue;
  - the env step;
  - the player's bookkeeping (b200env_play_stats): cumulative rewards and steps, finished games and the per-step statistics lines.
The host only rebuilds the context window every context_length steps (it knows the step count) and reads the stop flag and the
statistics log every `sync_every` steps.  The steps run after the stop flag was set and before the host saw it change no statistic; the
next game's full reset discards their state, as the reference's `break` leaves it.

Not served: the MuJoCo viewer (headless=False is refused) and the video (`record` is ignored: the reference opens a video file when
headless but never writes a frame to it, since render_vis returns before rendering).

Recording (cfg.env.b200_record_qpos, an addition): render_vis records, for the envs of cfg.env.b200_record_envs ([0] or "all"), the
qpos the reference's viewer would show (_sync_ref_motion: the simulated humanoid, the target it tracked and the simulated one 1000 m
up), one frame per call, on the device (include/b200env.h: b200env_im_record).  After num_rec_frames frames (the longest motion's
frame count with args.rec_once) the frames go to an .npz (rec_fname with its extension replaced, or out/recording/qpos_<date>.npz)
and SystemExit is raised, as the reference's render_vis quits.  run_test puts the record launch in the step graph, between the env
step and the bookkeeping; a record launch that writes the last frame sets the bookkeeping's stop flag.

Per-motion meters (cfg.env.b200_motion_stats, an addition): run_test also sums, per finished game, the reward, the steps, the four
sub-rewards and the mean body-position error into the bucket of the env's motion, and counts games and falls per motion
(include/b200env.h: b200env_im_motion_stats, in the step graph after the record launch and before the bookkeeping, so it stops with
it).  When run_test ends (or the recorder quits) the buckets go to cfg.env.b200_motion_stats_file (default
out/motion_stats/motion_stats_<date>.npz) and one summary line is printed.

Pose metrics (cfg.env.b200_pose_metrics, an addition; needs b200_motion_stats): the same launch also sums, per finished game, the
metrics motion-imitation work compares policies on - root-relative and Procrustes-aligned MPJPE, velocity and acceleration error - and
counts the games whose largest body-position error (global MPJPE) stays within cfg.env.b200_pose_success_threshold (default 0.5 m).
The file then also holds those sums, their frame counts, the successes and each motion's largest error, and a second line is printed.

Motion queue (cfg.env.b200_motion_queue, an addition; the reference never resets an env mid-game): a library larger than the env count
is scored in one run.  The queue holds every motion once per round, R = cfg.env.b200_motion_queue_repeats rounds (default 1), entry
q = r M + m; env e starts on entry e, and when its game ends it takes the next unplayed entry inside the step graph (include/b200env.h:
b200env_im_motion_queue, then the masked reset with the window aligned to the policy's slot), with no host synchronisation.  An env
that finishes once the queue is empty stays done.  run_test then runs one full reset and steps until every queued game has finished
or max_steps steps have run; the per-motion meters fold each game into the row of its entry, and the file sums a motion's R rows.

Motion queue with a body per motion (cfg.env.motion_assets with test_motion_assets, the reference's per-motion actors): the handle holds
every distinct asset of the library, runs the mixed plan for its lifetime (include/b200env.h: b200env_fix_mixed_plan), and env e
starts on the asset of motion e % M.  When an env takes its next entry, the queue launch also writes that motion's asset, and
b200env_set_env_assets re-points the env's asset before the masked reset, so the restarted game is stepped with its own body.  The
recording's `asset` is then [E, T], each recorded env's body per frame.  humanoid_masses (host, informational) keeps the
creation-time assignment."""
import os
from datetime import datetime

import numpy as np
import torch

from .. import native, nn
from .humanoid_smpl_im import HumanoidSMPLIM


def record_env_ids(spec, num_envs):
    """cfg.env.b200_record_envs: a list of env ids or "all" -> the list of recorded envs"""
    if isinstance(spec, str):
        if spec != "all":
            raise ValueError(f'b200_record_envs: {spec!r}; give a list of env ids or "all"')
        return list(range(num_envs))
    ids = [int(i) for i in spec]
    if not ids:
        raise ValueError("b200_record_envs is empty")
    bad = [i for i in ids if not 0 <= i < num_envs]
    if bad:
        raise ValueError(f"b200_record_envs: env ids {bad} lie outside [0, {num_envs})")
    if len(set(ids)) != len(ids):
        raise ValueError(f"b200_record_envs: duplicate env ids {sorted({i for i in ids if ids.count(i) > 1})}")
    return ids


def record_frames(env, args, motion_num_frames):
    """the frames to record: num_rec_frames (default 300), or the longest motion's frame count with args.rec_once"""
    n = int(env.get("num_rec_frames", 300))
    if getattr(args, "rec_once", False):
        n = int(np.max(motion_num_frames))
        print(f"Recording only {n} frames")
    if n < 1:
        raise ValueError(f"num_rec_frames must be at least 1, got {n}")
    return n


def record_path(env, now=None):
    """rec_fname with its extension replaced by .npz, or out/recording/qpos_<date>.npz (next to the reference's video_<date>.mp4)"""
    if env.get("rec_fname"):
        return os.path.splitext(env["rec_fname"])[0] + ".npz"
    now = now or datetime.now()
    return os.path.join("out", "recording", "qpos_%s.npz" % now.strftime('%Y-%m-%d-%H:%M:%S'))


def record_bytes(n_rec, cap, nq):
    """device bytes of the qpos rows [n_rec, cap, 2, nq] float32"""
    return n_rec * cap * 2 * nq * 4


def assemble_qpos(rows):
    """device rows [E, T, 2, nq] -> the viewer's qpos [E, T, 3 nq]: copy 0, copy 1, copy 0 with z += 1000"""
    c2 = rows[:, :, 0].clone()
    c2[..., 2] += 1000.0
    return torch.cat([rows[:, :, 0], rows[:, :, 1], c2], -1)


def motion_stats_path(env, now=None):
    """cfg.env.b200_motion_stats_file, or out/motion_stats/motion_stats_<date>.npz"""
    if env.get("b200_motion_stats_file"):
        return str(env["b200_motion_stats_file"])
    now = now or datetime.now()
    return os.path.join("out", "motion_stats", "motion_stats_%s.npz" % now.strftime('%Y-%m-%d-%H:%M:%S'))


def motion_env_lists(motion_ids, num_motions):
    """env -> motion map [N] -> (motion_start [M + 1], motion_envs [N]): the envs of motion m, in env order, are
    motion_envs[motion_start[m]:motion_start[m + 1]]"""
    ids = np.asarray(motion_ids.cpu() if torch.is_tensor(motion_ids) else motion_ids, np.int64)
    start = np.zeros(num_motions + 1, np.int64)
    start[1:] = np.cumsum(np.bincount(ids, minlength=num_motions))
    return start, np.argsort(ids, kind="stable").astype(np.int64)


def pose_metrics_threshold(env):
    """cfg.env.b200_pose_metrics -> None when off, else the success threshold in metres (b200_pose_success_threshold, default 0.5);
    refuses the key without b200_motion_stats and a threshold that is not a finite number above 0"""
    if not env.get("b200_pose_metrics", False):
        return None
    if not env.get("b200_motion_stats", False):
        raise ValueError("b200_pose_metrics extends the per-motion meters: set b200_motion_stats: True as well")
    t = env.get("b200_pose_success_threshold", 0.5)
    try:
        t = float(t)
    except (TypeError, ValueError):
        raise ValueError(f"b200_pose_success_threshold must be a number of metres, got {t!r}") from None
    if not (np.isfinite(t) and t > 0):
        raise ValueError(f"b200_pose_success_threshold must be a finite number of metres above 0, got {t!r}")
    return t


def pose_metrics_summary(counts, sums, pose_sums, success):
    """the printed line of the pose metrics (counts [M, 2], sums [M, 7], pose_sums [M, 7], success [M]): success rate, the MPJPEs in
    mm and the velocity and acceleration errors in mm/frame and mm/frame^2 over the finished games"""
    games, steps = counts[:, 0].sum(), sums[:, 1].sum()
    vf, af = pose_sums[:, 4].sum(), pose_sums[:, 5].sum()
    mm = lambda x, n: 1000.0 * x / n if n else float("nan")  # noqa: E731
    rate = success.sum() / games if games else float("nan")
    return (f"success rate: {rate:.4f}  MPJPE-g: {mm(sums[:, 6].sum(), steps):.2f} mm  MPJPE-l: {mm(pose_sums[:, 0].sum(), steps):.2f} mm"
            f"  PA-MPJPE: {mm(pose_sums[:, 1].sum(), steps):.2f} mm  velocity error: {mm(pose_sums[:, 2].sum(), vf):.2f} mm/frame"
            f"  acceleration error: {mm(pose_sums[:, 3].sum(), af):.2f} mm/frame^2")


def motion_stats_summary(counts, sums):
    """the printed line of the per-motion buckets (counts [M, 2] games, falls; sums [M, 7] float64)"""
    games, falls = counts[:, 0], counts[:, 1]
    steps = sums[:, 1].sum()
    ok = 1.0 - falls.sum() / games.sum() if games.sum() else float("nan")
    per_step = (sums[:, 0].sum() / steps, sums[:, 6].sum() / steps) if steps else (float("nan"), float("nan"))
    return (f"motions evaluated: {int((games > 0).sum())} of {len(games)}  games without a fall: {ok:.4f}  "
            f"reward per step: {per_step[0]:.6f}  body position error: {per_step[1]:.6f} m")


def motion_queue_rounds(cfg):
    """cfg.env.b200_motion_queue -> None when off, else the rounds R of the queue (b200_motion_queue_repeats, default 1); refuses R
    that is not an int >= 1, motion_assets without test_motion_assets (several assets are served for the held-out library of a test
    run), transform_specs without b200_device_transforms (the queue restarts games through the masked reset) and a state init other
    than Start (every queued game starts at its motion's first frame)"""
    env = cfg["env"]
    if not env.get("b200_motion_queue", False):
        return None
    R = env.get("b200_motion_queue_repeats", 1)
    if isinstance(R, bool) or not isinstance(R, (int, np.integer)) or R < 1:
        raise ValueError(f"b200_motion_queue_repeats must be an int >= 1, got {R!r}")
    if "motion_assets" in env and "test_motion_assets" not in env:
        raise ValueError("b200_motion_queue with several assets scores a held-out library: give its bodies in test_motion_assets "
                         "(with test_motion_file); motion_assets alone is not supported")
    if "transform_specs" in env and not env.get("b200_device_transforms", False):
        raise ValueError("b200_motion_queue restarts games through the masked reset: with transform_specs set b200_device_transforms")
    args = cfg.get("args", None)
    state_init = "Start" if args is not None and getattr(args, "test", False) else env.get("stateInit", "Hybrid")
    if state_init != "Start":
        raise ValueError(f"b200_motion_queue starts every game at its motion's first frame: needs args.test or stateInit: Start, "
                         f"got {state_init!r}")
    return int(R)


def queue_fold(rows, R, M, max_col=None):
    """the queue's per-entry rows [R M, ...] -> per motion [M, ...]: the R rows of motion m (entries r M + m) added in r order; column
    max_col (the largest error) takes the largest instead, NaN if one is NaN"""
    rows = np.asarray(rows).reshape(R, M, *np.shape(rows)[1:])
    out = rows[0].copy()
    for r in range(1, R):
        if max_col is None:
            out += rows[r]
        else:
            keep = out[..., max_col].copy()
            out += rows[r]
            out[..., max_col] = np.maximum(keep, rows[r][..., max_col])
    return out


class HumanoidSMPLIMVis(HumanoidSMPLIM):
    _q = None               # the motion queue's device state (cfg.env.b200_motion_queue), set by set_policy
    _test_task = True       # refuses cfg.env.b200_resample_motions

    def __init__(self, cfg, sim_params, physics_engine, device_type, device_id, headless):
        if not headless:
            raise ValueError("HumanoidSMPLIMVis: there is no MuJoCo viewer; run headless")
        env = cfg["env"]
        self._rec = None
        rec_ids = None
        self._pose_threshold = pose_metrics_threshold(env)
        self._queue_rounds = motion_queue_rounds(cfg)
        if env.get("b200_record_qpos", False):
            rec_ids = record_env_ids(env.get("b200_record_envs", [0]), int(env["numEnvs"]))
            if not getattr(cfg.get("args", None), "rec_once", False) and int(env.get("num_rec_frames", 300)) < 1:
                raise ValueError(f"num_rec_frames must be at least 1, got {env['num_rec_frames']}")
        super().__init__(cfg=cfg, sim_params=sim_params, physics_engine=physics_engine, device_type=device_type, device_id=device_id,
                         headless=headless)
        self.headless = headless
        self.cam_inited = False
        self.vis_mode = getattr(self.args, "vis_mode", None)
        self._im_policy = None
        self._ms = None
        if rec_ids is not None:
            self._setup_record(rec_ids)

    def _check_motion_lib(self, flat):
        N = int(self.cfg["env"]["numEnvs"])
        if self._queue_rounds is not None and N > flat.num_motions() * self._queue_rounds:
            raise ValueError(f"b200_motion_queue: {N} envs for a queue of {flat.num_motions()} motions x {self._queue_rounds} rounds; every "
                             "env starts on its own entry, so give at most as many envs as queued games")

    def _sample_motion_ids(self):
        """with the queue env e starts on entry e, motion e % M; else humanoid_smpl_im.py:247-254"""
        if self._queue_rounds is None:
            return super()._sample_motion_ids()
        return torch.arange(self.num_envs, device=self.device) % self._motion_lib.num_motions()

    def _setup_queue(self):
        """the queue's device state: each env's entry, the idle flags, the cursor and, per entry, its env and first step"""
        N, Q, dev = self.num_envs, self._motion_lib.num_motions() * self._queue_rounds, self.device
        i64 = lambda n: torch.zeros(n, device=dev, dtype=torch.long)  # noqa: E731
        self._q = dict(entry=i64(N), idle=torch.zeros(N, device=dev, dtype=torch.uint8), cursor=i64(1), game_env=i64(Q),
                       game_start_step=i64(Q), **self._queue_assets())

    def _start_queue(self):
        """before the run's full reset: env e on entry e, the rest of the queue unplayed"""
        q, N = self._q, self.num_envs
        e = torch.arange(N, device=self.device)
        self._reset_ref_motion_ids.copy_(self._sample_motion_ids())
        self._reset_ref_motion_bodies.copy_(self._ml_t["motion_bodies"][self._reset_ref_motion_ids])
        q["entry"].copy_(e)
        q["idle"].zero_()
        q["cursor"].fill_(N)
        q["game_env"].fill_(-1)
        q["game_env"][:N] = e
        q["game_start_step"].fill_(-1)
        q["game_start_step"][:N] = 0
        if "env_asset" in q:                   # every env back on its start body
            q["env_asset"].copy_(q["start_env_asset"])
            q["asset_error"].zero_()
            self._env.set_env_assets(q["env_asset"], q["asset_error"])

    def _queue_launches(self):
        """the assignment of the finished envs' next entries, then their masked reset with the window aligned to the step counter"""
        M = self._motion_lib.num_motions()
        native.im_motion_queue(dict(n=self.num_envs, num_motions=M, queue_len=M * self._queue_rounds,
                                    shape_dim=self._reset_ref_motion_bodies.shape[1]),
                               dict(self._q, reset_buf=self.reset_buf, lib_motion_bodies=self._ml_t["motion_bodies"],
                                    motion_ids=self._reset_ref_motion_ids, motion_bodies=self._reset_ref_motion_bodies, mask=self._reset_mask,
                                    step=self._im_step, games=self._stats["games"], prev_dones=self._stats["prev_dones"],
                                    env_flags=self._ms["env_flags"] if self._ms is not None else None))
        if "env_asset" in self._q:             # the restarted envs' new bodies, read by the next physics launch
            self._env.set_env_assets(self._q["env_asset"], self._q["asset_error"])
        self.reset_masked(self._reset_mask, step=self._im_step)

    def _setup_record(self, ids):
        """the recorder's device buffers, after the cfg checks and the free-memory check"""
        env, dev = self.cfg["env"], self.device
        cap, nq, E = record_frames(env, self.args, self._motion_lib.num_frames), 7 + self.num_dof, len(ids)
        need, free = record_bytes(E, cap, nq), torch.cuda.mem_get_info(dev)[0]
        if need > free:
            raise ValueError(f"recording {E} envs x {cap} frames needs {need} bytes of device memory, {free} are free")
        if "motion_assets" in env:
            entries = env["motion_assets"]
            name = lambda a: os.path.basename(str(a)) if isinstance(a, (str, os.PathLike)) else str(a["name"])  # noqa: E731
            mids = self._reset_ref_motion_ids.cpu().numpy()
            assets = [name(entries[mids[e]]) for e in ids]
            if self._queue_rounds is not None:     # bodies change with the motion: the export names them per frame
                self._rec_motion_asset = np.array([name(x) for x in entries])
        else:
            assets = [os.path.basename(env["asset"]["assetFileName"])] * E
        i64 = lambda *s: torch.zeros(*s, device=dev, dtype=torch.long)  # noqa: E731
        self._rec = dict(env_ids=torch.tensor(ids, device=dev, dtype=torch.long), qpos=torch.zeros(E, cap, 2, nq, device=dev),
                         rec_motion_ids=i64(E, cap), rec_reset=i64(E, cap), frame=i64(1),
                         done=torch.zeros(1, device=dev, dtype=torch.int32))
        self._rec_cap, self._rec_assets, self._rec_path = cap, assets, record_path(env)
        self.frame_index = 0

    def _record_launch(self, init, games=None):
        nb, nbl = self.num_bodies, self._num_lib_bodies
        native.im_record(dict(n_rec=len(self._rec_assets), num_envs=self.num_envs, num_bodies=nb, num_lib_bodies=nbl, nd=self.num_dof,
                              cap=self._rec_cap, init=int(init)),
                         dict(self._rec, rigid_body_state=self._rigid_body_state, dof_state=self._dof_state,
                              p_dof_pos=self._prev_target_dof_pos, p_rb_pos=self._prev_target_rb_pos, p_rb_rot=self._prev_target_rb_rot,
                              reset_buf=self.reset_buf, motion_ids=self._reset_ref_motion_ids, games=games))

    def export_recording(self):
        """writes the frames recorded so far to the .npz; returns its path"""
        T = min(int(self._rec["frame"]), self._rec_cap)
        r = self._rec
        path = self._rec_path
        if os.path.dirname(path):
            os.makedirs(os.path.dirname(path), exist_ok=True)
        np.savez(path, qpos=assemble_qpos(r["qpos"][:, :T]).cpu().numpy(), env_ids=r["env_ids"].cpu().numpy(),
                 motion_ids=r["rec_motion_ids"][:, :T].cpu().numpy(), reset=r["rec_reset"][:, :T].cpu().numpy(),
                 asset=self._recorded_assets(T), fps=np.float64(1.0 / self.dt), nq=np.int64(7 + self.num_dof))
        print(f"============ qpos of {T} frames written to {path} ============")
        return path

    def _recorded_assets(self, T):
        """the recording's `asset`: each recorded env's body name [E], or per frame [E, T] from the recorded motion ids when the queue
        changes bodies"""
        if getattr(self, "_rec_motion_asset", None) is None:
            return np.array(self._rec_assets)
        return self._rec_motion_asset[self._rec["rec_motion_ids"][:, :T].cpu().numpy()]

    def create_sim(self):
        # humanoid_smpl_im_vis.py:35 sets max_episode_length = 3000; the step's reset rule reads it from the cfg struct made here
        self.max_episode_length = 3000
        super().create_sim()
        if self._queue_rounds is not None and "motion_assets" in self.cfg["env"]:
            self._env.fix_mixed_plan()         # envs change body as their games end

    def _queue_assets(self):
        """with motion_assets: the asset of each motion [M], each env's asset [N] (started as at create) and the error word of
        b200env_set_env_assets, all int32 on the device; else {}"""
        if "motion_assets" not in self.cfg["env"]:
            return {}
        dev, i32 = self.device, torch.int32
        start = torch.as_tensor(self._env_asset, dtype=i32, device=dev)
        self._asset_error = torch.zeros(1, device=dev, dtype=i32)     # read by _check_asset_error at the run's sync points
        return dict(motion_asset=torch.as_tensor(self._motion_asset, dtype=i32, device=dev), env_asset=start.clone(), start_env_asset=start,
                    asset_error=self._asset_error)

    def render_vis(self, init=False):
        """without b200_record_qpos the reference's headless branch: nothing.  With it: one frame of the recorded envs (init: after a
        reset, the target copy is the simulated one); after num_rec_frames calls the .npz is written and SystemExit raised"""
        if self._rec is None:
            return
        self._record_launch(init)
        self.frame_index += 1
        if self.frame_index >= self._rec_cap:
            self.export_recording()
            raise SystemExit

    # ------------------------------------------------------------------ test loop of ImitatorPlayer.run
    def set_policy(self, network, clip_obs=float("inf"), clip_actions=None, sync_every=None):
        """network: a dict of nn.im_networks_from_checkpoint (layers, mean, rstd, clip; with `sigma`: the sampled action, seeded by
        cfg["seed"]); clip_obs / clip_actions: the wrapper's clamps (VecTaskPython.clip_obs / clip_actions).  Allocates the operand, residual and statistics buffers; sync_every (default
        context_length) sizes the statistics log the host drains."""
        N, dev, nd = self.num_envs, self.device, self.num_dof
        w = self._env.obs_row_width()
        if network["layers"][0][0].shape[1] != w or network["layers"][-1][0].shape[0] != self.num_actions:
            raise ValueError(f"the network takes {network['layers'][0][0].shape[1]} inputs and gives {network['layers'][-1][0].shape[0]} "
                             f"actions; the task's observation is {w} wide and its action {self.num_actions}")
        self._context_buffers()
        self._im_step = torch.zeros(1, device=dev, dtype=torch.long)
        self._im_resid = torch.zeros(N, nd, device=dev)
        self._im_policy = nn.PolicyMLP(network["layers"], N, dev, obs_mean=network["mean"], obs_rstd=network["rstd"],
                                       clamp_obs=network["clip"], clamp_actions=clip_actions, residual=(self._im_resid, nd),
                                       noise_sigma=network.get("sigma"), seed=int(self.cfg.get("seed", 10)))
        self._im_clip_obs, self._im_clip = float(clip_obs), float(network["clip"])
        cap = int(sync_every or self.context_length) + 1
        f = lambda *s: torch.zeros(*s, device=dev)  # noqa: E731
        self._stats = dict(cr=f(N), steps=f(N), prev_dones=f(N), totals=torch.zeros(2, device=dev, dtype=torch.float64),
                           log=torch.zeros(cap, 3, device=dev, dtype=torch.float64), games=torch.zeros(3, device=dev, dtype=torch.long),
                           step=self._im_step)
        self._stats_cap = cap
        self._n_games = 1 << 62            # run_test sets games_num * n_game_life
        self._im_graph = None
        if self._queue_rounds is not None:
            self._setup_queue()
        if self.cfg["env"].get("b200_motion_stats", False):
            self._setup_motion_stats()

    def _setup_motion_stats(self):
        """the per-motion buckets and, from the env -> motion map the test run keeps, each motion's env list; with the queue one row
        per queued game, folded by its entry"""
        N, M, dev = self.num_envs, self._motion_lib.num_motions(), self.device
        if self._q is None:
            start, envs = motion_env_lists(self._reset_ref_motion_ids, M)
            self._ms = dict(motion_start=torch.from_numpy(start).to(dev), motion_envs=torch.from_numpy(envs).to(dev))
        else:
            M *= self._queue_rounds
            self._ms = dict(env_entry=self._q["entry"])
        self._ms.update(env_sums=torch.zeros(N, 7, device=dev, dtype=torch.float64),
                        env_flags=torch.zeros(N, 2, device=dev, dtype=torch.int32),
                        counts=torch.zeros(M, 2, device=dev, dtype=torch.long), sums=torch.zeros(M, 7, device=dev, dtype=torch.float64))
        if self._pose_threshold is not None:    # one warp per env, a lane per body
            nbl = self._num_lib_bodies
            if nbl > 32:
                raise ValueError(f"b200_pose_metrics compares at most 32 bodies, the motion library has {nbl}")
            self._ms.update(env_pose=torch.zeros(N, 7, device=dev, dtype=torch.float64), pose_hist=torch.zeros(N, 2, 2, nbl, 3, device=dev),
                            pose_fill=torch.zeros(N, device=dev, dtype=torch.int32),
                            pose_sums=torch.zeros(M, 7, device=dev, dtype=torch.float64), success=torch.zeros(M, device=dev, dtype=torch.long))

    def _motion_stats_launch(self, games=None):
        rows = self._motion_lib.num_motions() * (self._queue_rounds or 1)
        launch = native.im_motion_stats if self._q is None else native.im_motion_queue_stats
        launch(dict(n=self.num_envs, num_motions=rows, num_bodies=self.num_bodies, num_lib_bodies=self._num_lib_bodies,
                    success_threshold=self._pose_threshold),
               dict(self._ms, rew=self.rew_buf, sub_rewards=self._sub_rewards, reset_buf=self.reset_buf, terminate_buf=self._terminate_buf,
                    rigid_body_state=self._rigid_body_state, target_rb_pos=self._prev_target_rb_pos, games=games))

    def export_motion_stats(self):
        """writes the per-motion buckets to b200_motion_stats_file and prints the summary line; returns the file's path"""
        counts, sums = self._ms["counts"].cpu().numpy(), self._ms["sums"].cpu().numpy()
        pose = (self._ms["pose_sums"].cpu().numpy(), self._ms["success"].cpu().numpy()) if self._pose_threshold is not None else None
        env_motion_ids, queue = self._reset_ref_motion_ids.cpu().numpy(), {}
        if self._q is not None:
            R, M = self._queue_rounds, self._motion_lib.num_motions()
            queue = dict(game_env=self._q["game_env"].cpu().numpy().reshape(R, M),
                         game_start_step=self._q["game_start_step"].cpu().numpy().reshape(R, M),
                         unfinished=np.flatnonzero(counts[:, 0] == 0).astype(np.int64))
            counts, sums = queue_fold(counts, R, M), queue_fold(sums, R, M)
            if pose is not None:
                pose = queue_fold(pose[0], R, M, max_col=6), queue_fold(pose[1], R, M)
            env_motion_ids = self._sample_motion_ids().cpu().numpy()
        path = motion_stats_path(self.cfg["env"])
        if os.path.dirname(path):
            os.makedirs(os.path.dirname(path), exist_ok=True)
        np.savez(path, games=counts[:, 0], falls=counts[:, 1], reward_sum=sums[:, 0], steps=sums[:, 1].astype(np.int64),
                 sub_reward_sum=sums[:, 2:6], body_pos_err_sum=sums[:, 6], env_motion_ids=env_motion_ids,
                 test_motion_file=np.array(self._test_motion_file or ""), **self._pose_metrics_keys(pose), **queue)
        print(motion_stats_summary(counts, sums))
        if pose is not None:
            print(pose_metrics_summary(counts, sums, *pose))
        print(f"============ per-motion statistics written to {path} ============")
        return path

    def _pose_metrics_keys(self, pose):
        """the pose metrics' keys of the file from (pose_sums [M, 7], success [M]) (none without b200_pose_metrics)"""
        if pose is None:
            return {}
        ps, success = pose
        return dict(mpjpe_l_sum=ps[:, 0], mpjpe_pa_sum=ps[:, 1], vel_err_sum=ps[:, 2], acc_err_sum=ps[:, 3],
                    vel_frames=ps[:, 4].astype(np.int64), acc_frames=ps[:, 5].astype(np.int64), success=success,
                    max_body_pos_err=ps[:, 6], success_threshold=np.float64(self._pose_threshold), dt=np.float64(self.dt))

    def clear_motion_stats_games(self):
        """a game starts: the per-env sums, flags and pose history start again; the per-motion buckets run on"""
        for k in ("env_sums", "env_flags", "env_pose", "pose_fill"):
            if k in self._ms:
                self._ms[k].zero_()

    def policy_rows(self):
        """the operand launch: policy.x and the residual from obs_buf and the context slot context_padding + step % context_length"""
        p = self._im_policy
        self._env.im_policy_rows(
            dict(n=self.num_envs, num_obs=self.num_obs, num_frames=self.context_feat.shape[1], feat_width=self.context_feat.shape[2],
                 context_padding=self.context_padding, context_length=self.context_length, ld=p.x.shape[1], clip_obs=self._im_clip_obs,
                 clip=self._im_clip if p.mean is not None else None),
            dict(obs_buf=self.obs_buf, context_feat=self.context_feat, step=self._im_step, mean=p.mean, rstd=p.rstd, x=p.x,
                 resid=self._im_resid))

    def act(self):
        """operand launch + the four layers: the action, deterministic or sampled (float [N, num_actions], a static buffer)"""
        self.policy_rows()
        return self._im_policy.forward_prepared()

    def _test_launches(self):
        with torch.no_grad():
            actions = self.act()
        self._env.step(actions)
        if self._rec is not None:
            self._record_launch(False, games=self._stats["games"])
        if self._ms is not None:
            self._motion_stats_launch(games=self._stats["games"])
        queue_games = self._motion_lib.num_motions() * self._queue_rounds if self._q is not None else 0
        native.play_stats(dict(n=self.num_envs, max_log=self._stats_cap, n_games=self._n_games, queue_games=queue_games),
                          dict(self._stats, rew=self.rew_buf, reset_buf=self.reset_buf))
        if self._q is not None:
            self._queue_launches()

    def test_step(self, n, graph=True):
        """step n (0-based) of a game: the context rebuild of all envs when n > 0 and n % context_length == 0, then the operand launch,
        the layers, the env step and the bookkeeping.  graph=True: the first call runs them eagerly, later calls replay one CUDA graph."""
        if n > 0 and n % self.context_length == 0:
            ids = torch.arange(self.num_envs, device=self.device)
            self._init_context(ids, self._reset_ref_motion_ids, self._cur_ref_motion_times)
        if self._im_graph is not None:
            self._im_graph.replay()
            return
        self._test_launches()
        if graph:
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                self._test_launches()
            self._im_graph = g

    def _quit_recording(self):
        """render_vis' quit() inside run_test: the frames, the per-motion statistics of the games finished so far, SystemExit"""
        self.export_recording()
        if self._ms is not None:
            self.export_motion_stats()
        raise SystemExit

    def run_test(self, policy, games_num, max_steps, n_game_life=1, print_stats=True, sync_every=None, clip_obs=float("inf"),
                 clip_actions=None, graph=True, history=None):
        """ImitatorPlayer.run (im_player.py:193-312) with the deterministic mu, or the sampled action when `policy` has a sigma: per game a full reset(), then up to max_steps
        test_step() calls; the host reads the stop flag and the statistics log every sync_every (default context_length) steps and at
        max_steps, and prints the reference's lines in order.  With cfg.env.b200_motion_queue: one full reset, then up to max_steps
        steps in all, until every queued game has finished; games_played counts the finished queued games.  policy: a dict of
        nn.im_networks_from_checkpoint.  history: a list that receives, per game, the list of device copies (rew_buf, reset_buf) of
        every step run (for tests).  Returns dict(sum_rewards, sum_steps, games_played)."""
        sync_every = int(sync_every or self.context_length)
        self.set_policy(policy, clip_obs=clip_obs, clip_actions=clip_actions, sync_every=sync_every)
        n_games = games_num * n_game_life
        self._n_games = n_games
        st = self._stats
        for _ in range(n_games if self._q is None else 1):
            if int(st["games"][0]) >= n_games:
                break
            if self._q is not None:
                self._start_queue()
            self.reset()
            for k in ("cr", "steps", "prev_dones", "step"):
                st[k].zero_()
            st["games"][1:].zero_()            # stop flag and log rows; games_played and the totals run on
            if self._ms is not None:           # the games of the last run are folded; the buckets run on
                self.clear_motion_stats_games()
            if self._rec is not None:          # render_vis(init=True): the host reads the frame counter once per game
                self._record_launch(True, games=st["games"])
                if int(self._rec["frame"]) >= self._rec_cap:
                    self._quit_recording()
            game = [] if history is not None else None
            for n in range(max_steps):
                self.test_step(n, graph)
                if game is not None:
                    game.append((self.rew_buf.clone(), self.reset_buf.clone()))
                if (n + 1) % sync_every == 0 or n + 1 == max_steps:
                    games = st["games"].tolist()
                    self._check_asset_error()
                    rows = st["log"][:games[2]].tolist()    # at most sync_every rows since the last read
                    st["games"][2].zero_()
                    if print_stats:
                        for count, r, s in rows:
                            print('reward:', r / count, 'steps:', s / count)
                    if self._rec is not None and int(self._rec["frame"]) >= self._rec_cap:    # render_vis' quit()
                        self._quit_recording()
                    if games[1]:
                        break
            if history is not None:
                history.append(game)
        sum_rewards, sum_steps = st["totals"].tolist()
        games_played = int(st["games"][0])
        print(sum_rewards)
        print('av reward:', sum_rewards / games_played * n_game_life, 'av steps:', sum_steps / games_played * n_game_life)
        if self._rec is not None:              # the games ended before the recorder filled: the frames so far
            self.export_recording()
        if self._ms is not None:
            self.export_motion_stats()
        return dict(sum_rewards=sum_rewards, sum_steps=sum_steps, games_played=games_played)
