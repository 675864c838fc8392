"""float64 restatement of the embodied_pose imitation policy at test time (paths relative to the embodied_pose tree):
  - ImitatorBuilder.Network.eval_actor with preprocess_input's non-training branch (models/im_network_builder.py:117-231): the raw
    observation split by obs_names / obs_dims, the target body_pos | body_rot | dof_pos of context slot context_padding + t
    (forward_context(flatten=False) + obtain_cur_context(t)), compute_humanoid_observations_imitation with local_root_obs =
    root_height_obs = True (oracle/ref_port.py), running_obs, actor_mlp Linear / ReLU x 3, linear mu, `mu[:, :nd] += target_dof_pos`;
  - both normalisers: RunningNorm (models/running_norm.py, eval: identity at n == 0, else clamp((x - mean) / (std + 1e-8), -5, 5)) and
    rl_games RunningMeanStd (clamp((x - mean) / sqrt(var + 1e-5), -5, 5)), with the statistics ImitatorPlayer.restore /
    load_pretrained load (players/im_player.py:43-94);
  - ImitatorPlayer.run's bookkeeping (:193-312, num_agents = 1) over a given history of (rew, done) per game.
tests/golden/im_policy.npz (made by executing the reference's own code, tests/golden/make_golden_im_policy.py) pins it."""
import numpy as np

from oracle import ref_port as R

ACTOR_KEYS = ("actor_mlp.0", "actor_mlp.2", "actor_mlp.4", "mu")
OBS_NAMES = ("body_pos", "body_rot", "dof_pos", "dof_vel", "body_vel", "body_ang_vel", "motion_bodies")


def split_obs(obs, nb, nd):
    """obs [N, 13 nb + 2 nd + S] -> the named blocks (humanoid_smpl_im.py:198-211)"""
    N = obs.shape[0]
    dims = (nb * 3, nb * 4, nd, nd, nb * 3, nb * 3, obs.shape[1] - 13 * nb - 2 * nd)
    shapes = ((nb, 3), (nb, 4), (nd,), (nd,), (nb, 3), (nb, 3), (dims[-1],))
    out, o = {}, 0
    for name, d, s in zip(OBS_NAMES, dims, shapes):
        out[name] = obs[:, o:o + d].reshape((N,) + s)
        o += d
    return out


def context_slot(context_feat, nb, nd, padding, t):
    """(body_pos [N, nb, 3], body_rot [N, nb, 4], dof_pos [N, nd]) of frame padding + t of the window [N, P, W]"""
    f = context_feat[:, padding + t]
    N = f.shape[0]
    return f[:, :3 * nb].reshape(N, nb, 3), f[:, 3 * nb:7 * nb].reshape(N, nb, 4), f[:, 7 * nb:7 * nb + nd]


def human_obs(obs, context_feat, nb, nd, padding, t, clip_obs=np.inf):
    """compute_humanoid_obs on the wrapper-clamped raw observation and the context slot, float64 [N, 734]"""
    o = split_obs(np.clip(np.asarray(obs, np.float64), -clip_obs, clip_obs), nb, nd)
    tp, tr, td = context_slot(np.asarray(context_feat, np.float64), nb, nd, padding, t)
    return R.compute_humanoid_observations_imitation(o["body_pos"], o["body_rot"], tp, tr, o["dof_pos"], o["dof_vel"], td, o["body_vel"],
                                                     o["body_ang_vel"], o["motion_bodies"], True, True), td


def normalize(x, net):
    if net["norm"] == "running":
        if net["n"] <= 0:
            return x
        return np.clip((x - net["mean"]) / (net["std"] + 1e-8), -5.0, 5.0)
    if net["norm"] == "rms":
        return np.clip((x - net["mean"]) / np.sqrt(net["var"] + 1e-5), -5.0, 5.0)
    return x


def eval_actor(x, layers):
    for i, (w, b) in enumerate(layers):
        x = x @ np.asarray(w, np.float64).T + np.asarray(b, np.float64)
        if i < len(layers) - 1:
            x = np.maximum(x, 0.0)
    return x


def act(obs, context_feat, net, nb, nd, padding, t, clip_obs=np.inf, clip_actions=None):
    """the action ImitatorPlayer.run steps with (deterministic mu, residual, then the wrapper's action clamp)"""
    h, td = human_obs(obs, context_feat, nb, nd, padding, t, clip_obs)
    mu = eval_actor(normalize(h, net), net["layers"])
    mu[:, :nd] += td
    return np.clip(mu, -clip_actions, clip_actions) if clip_actions else mu


def load(ck, running_obs_type="ours", use_running_obs=True, obs_dim=734):
    """the network ImitatorPlayer.restore / load_pretrained leave: actor layers and the normaliser (float64)"""
    lightning = "pytorch-lightning_version" in ck
    m = dict(ck["state_dict"]) if lightning else {k[len("a2c_network."):]: v for k, v in ck["model"].items() if k.startswith("a2c_network.")}
    f = lambda v: np.asarray(v, np.float64)  # noqa: E731
    layers = [(f(m[k + ".weight"]), f(m[k + ".bias"])) for k in ACTOR_KEYS]
    if not use_running_obs:
        return dict(layers=layers, norm=None)
    if running_obs_type == "rl_game":
        mean = f(m["running_obs.running_mean"]) if "running_obs.running_mean" in m else np.zeros(obs_dim)
        var = f(m["running_obs.running_var"]) if "running_obs.running_var" in m else np.ones(obs_dim)
        return dict(layers=layers, norm="rms", mean=mean, var=var)
    mean, std, n = np.zeros(obs_dim), np.zeros(obs_dim), 0
    if "running_obs.n" in m:
        n = int(m["running_obs.n"])
        mean[:len(m["running_obs.mean"])] = f(m["running_obs.mean"])
        std[:len(m["running_obs.std"])] = f(m["running_obs.std"])
    elif not lightning:
        rms = ck.get("running_mean_std")
        if rms is None and "running_obs.running_mean" in m:
            rms = {k: m["running_obs." + k] for k in ("running_mean", "running_var", "count")}
        if rms is not None:
            L = len(rms["running_mean"])
            n = int(rms["count"])
            mean[:L] = np.asarray(rms["running_mean"], np.float32)
            std[:L] = np.sqrt(np.asarray(rms["running_var"], np.float32))
    return dict(layers=layers, norm="running", n=n, mean=mean, std=std)


def run_stats(games, games_num, max_steps, n_game_life=1):
    """ImitatorPlayer.run's bookkeeping: games = per game the list of (rew [N], done [N]) of the steps the env ran (steps past the
    loop's break are ignored).  cr / steps are float32 as in the reference.  Returns (lines, sum_rewards, sum_steps, games_played)
    with lines = the printed (count, sum cr, sum steps) per step that finished games."""
    n_games = games_num * n_game_life
    sum_rewards, sum_steps, games_played, lines = 0.0, 0.0, 0, []
    for hist in games:
        if games_played >= n_games:
            break
        N = len(hist[0][0])
        cr, steps, prev = np.zeros(N, np.float32), np.zeros(N, np.float32), np.zeros(N, np.float32)
        for n in range(min(max_steps, len(hist))):
            r, done = hist[n]
            done = (np.asarray(done) != 0).astype(np.float32)
            cr = cr + np.asarray(r, np.float32)
            steps = steps + np.float32(1)
            sd = done * (1 - prev)
            idx = np.nonzero(sd)[0]
            games_played += len(idx)
            if len(idx) > 0:
                cur_r, cur_s = float(cr[idx].sum(dtype=np.float32)), float(steps[idx].sum(dtype=np.float32))
                cr = cr * (1 - done)
                steps = steps * (1 - done)
                sum_rewards += cur_r
                sum_steps += cur_s
                lines.append((len(idx), cur_r, cur_s))
                if N == 1 or games_played >= n_games:
                    break
            prev = done.copy()
            if done[0]:
                break
    return lines, sum_rewards, sum_steps, games_played
