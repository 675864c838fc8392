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
headless but never writes a frame to it, since render_vis returns before rendering)."""
import torch

from .. import native, nn
from .humanoid_smpl_im import HumanoidSMPLIM


class HumanoidSMPLIMVis(HumanoidSMPLIM):
    def __init__(self, cfg, sim_params, physics_engine, device_type, device_id, headless):
        if not headless:
            raise ValueError("HumanoidSMPLIMVis: there is no MuJoCo viewer; run headless")
        super().__init__(cfg=cfg, sim_params=sim_params, physics_engine=physics_engine, device_type=device_type, device_id=device_id,
                         headless=headless)
        self.headless = headless
        self.cam_inited = False
        self.vis_mode = getattr(self.args, "vis_mode", None)
        self._im_policy = None

    def create_sim(self):
        # humanoid_smpl_im_vis.py:35 sets max_episode_length = 3000; the step's reset rule reads it from the cfg struct made here
        self.max_episode_length = 3000
        super().create_sim()

    def render_vis(self, init=False):
        """the reference's headless branch: nothing"""
        return

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
        native.play_stats(dict(n=self.num_envs, max_log=self._stats_cap, n_games=self._n_games),
                          dict(self._stats, rew=self.rew_buf, reset_buf=self.reset_buf))

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

    def run_test(self, policy, games_num, max_steps, n_game_life=1, print_stats=True, sync_every=None, clip_obs=float("inf"),
                 clip_actions=None, graph=True, history=None):
        """ImitatorPlayer.run (im_player.py:193-312) with the deterministic mu, or the sampled action when `policy` has a sigma: per game a full reset(), then up to max_steps
        test_step() calls; the host reads the stop flag and the statistics log every sync_every (default context_length) steps and at
        max_steps, and prints the reference's lines in order.  policy: a dict of nn.im_networks_from_checkpoint.  history: a list that
        receives, per game, the list of device copies (rew_buf, reset_buf) of every step run (for tests).  Returns dict(sum_rewards,
        sum_steps, games_played)."""
        sync_every = int(sync_every or self.context_length)
        self.set_policy(policy, clip_obs=clip_obs, clip_actions=clip_actions, sync_every=sync_every)
        n_games = games_num * n_game_life
        self._n_games = n_games
        st = self._stats
        for _ in range(n_games):
            if int(st["games"][0]) >= n_games:
                break
            self.reset()
            for k in ("cr", "steps", "prev_dones", "step"):
                st[k].zero_()
            st["games"][1:].zero_()            # stop flag and log rows; games_played and the totals run on
            game = [] if history is not None else None
            for n in range(max_steps):
                self.test_step(n, graph)
                if game is not None:
                    game.append((self.rew_buf.clone(), self.reset_buf.clone()))
                if (n + 1) % sync_every == 0 or n + 1 == max_steps:
                    games = st["games"].tolist()
                    rows = st["log"][:games[2]].tolist()    # at most sync_every rows since the last read
                    st["games"][2].zero_()
                    if print_stats:
                        for count, r, s in rows:
                            print('reward:', r / count, 'steps:', s / count)
                    if games[1]:
                        break
            if history is not None:
                history.append(game)
        sum_rewards, sum_steps = st["totals"].tolist()
        games_played = int(st["games"][0])
        print(sum_rewards)
        print('av reward:', sum_rewards / games_played * n_game_life, 'av steps:', sum_steps / games_played * n_game_life)
        return dict(sum_rewards=sum_rewards, sum_steps=sum_steps, games_played=games_played)
