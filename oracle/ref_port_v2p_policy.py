"""float64 torch restatement of the tennis controller's high-level policy at test time (the reference's V2PPlayer with the deterministic
action; paths relative to the vid2player tree):
  - rl_games RunningMeanStd in eval mode (single-player cfgs, normalize_input): clamp((x - mean) / sqrt(var + 1e-5), -5, 5);
  - RunningNorm.forward in eval mode (models/running_norm.py:32-43; dual cfgs, use_running_obs with running_obs_type 'ours'):
    identity while n == 0, else clamp((x - mean) / (std + 1e-8), -5, 5);
  - V2PBuilder.Network.eval_actor (models/v2p_network_builder.py:52-81): actor_mlp Linear / ReLU x 3, linear mu (mu_activation None);
  - V2PBuilderDual.Network.eval_actor (models/v2p_network_builder_dual.py:39-47): network1 on rows 0::2, network2 on rows 1::2, the
    outputs interleaved back into env order;
  - the weights and statistics V2PPlayer.restore (players/v2p_player.py:71-111) and load_dual_cp (:21-69) load, with the zero-padded
    first layer and the normaliser prefix when the network's obs dim is larger than the checkpoint's.
tests/golden/v2p_policy.npz (made by executing the reference's own code, tests/golden/make_golden_v2p_policy.py) pins it."""
import torch

ACTOR_KEYS = ("actor_mlp.0", "actor_mlp.2", "actor_mlp.4", "mu")
D64 = torch.float64


def rms_normalize(x, mean, var, eps=1e-5, clip=5.0):
    return torch.clamp((x - mean) / torch.sqrt(var + eps), -clip, clip)


def running_norm(x, n, mean, std, clip=5.0):
    if n <= 0:
        return x
    return torch.clamp((x - mean) / (std + 1e-8), -clip, clip)


def eval_actor(x, layers):
    for i, (w, b) in enumerate(layers):
        x = x @ w.T + b
        if i < len(layers) - 1:
            x = torch.relu(x)
    return x


def normalize(x, net):
    if net["norm"] == "rms":
        return rms_normalize(x, net["mean"], net["var"])
    if net["norm"] == "running":
        return running_norm(x, net["n"], net["mean"], net["std"])
    return x


def act(obs, nets, clip_obs=float("inf"), clip_actions=None):
    """the action V2PPlayer.run steps with: the wrapper's observation clamp, normaliser, eval_actor (dual: interleaved), the wrapper's
    action clamp; obs [N, D] float64"""
    obs = torch.clamp(obs, -clip_obs, clip_obs)
    if len(nets) == 1:
        mu = eval_actor(normalize(obs, nets[0]), nets[0]["layers"])
    else:
        a = eval_actor(normalize(obs[0::2], nets[0]), nets[0]["layers"])
        b = eval_actor(normalize(obs[1::2], nets[1]), nets[1]["layers"])
        mu = torch.stack([a, b], 1).reshape(-1, a.shape[1])
    return torch.clamp(mu, -clip_actions, clip_actions) if clip_actions else mu


def _padded(w, obs_dim):
    if w.shape[1] == obs_dim:
        return w
    assert obs_dim > w.shape[1]
    out = torch.zeros(w.shape[0], obs_dim, dtype=w.dtype)
    out[:, :w.shape[1]] = w
    return out


def load_single(ck, obs_dim, normalize_input=True):
    """V2PPlayer.restore: a2c_network.actor_mlp / mu, running_mean_std (prefix of a fresh mean 0 / var 1 when padded)"""
    m = ck["model"]
    layers = [(m["a2c_network." + k + ".weight"].to(D64), m["a2c_network." + k + ".bias"].to(D64)) for k in ACTOR_KEYS]
    layers[0] = (_padded(layers[0][0], obs_dim), layers[0][1])
    if not normalize_input:
        return dict(layers=layers, norm=None)
    rms = ck["running_mean_std"]
    mean, var = torch.zeros(obs_dim, dtype=D64), torch.ones(obs_dim, dtype=D64)
    L = rms["running_mean"].shape[0]
    mean[:L], var[:L] = rms["running_mean"].to(D64), rms["running_var"].to(D64)
    return dict(layers=layers, norm="rms", mean=mean, var=var)


def load_dual(cks, obs_dim):
    """load_dual_cp for network1 / network2: actor weights (padded first layer), the RunningNorm of the model or, when the checkpoint
    has none, the rl_games statistics (std = sqrt(var)) over a prefix of a fresh RunningNorm (mean 0, std 0, n 0)"""
    nets = []
    for ck in cks:
        m = {k[len("a2c_network."):]: v for k, v in ck["model"].items()}
        layers = [(m[k + ".weight"].to(D64), m[k + ".bias"].to(D64)) for k in ACTOR_KEYS]
        layers[0] = (_padded(layers[0][0], obs_dim), layers[0][1])
        mean, std, n = torch.zeros(obs_dim, dtype=D64), torch.zeros(obs_dim, dtype=D64), 0
        if "running_obs.n" in m:
            n = int(m["running_obs.n"])
            mean[:m["running_obs.mean"].shape[0]] = m["running_obs.mean"].to(D64)
            std[:m["running_obs.std"].shape[0]] = m["running_obs.std"].to(D64)
        else:
            rms = ck.get("running_mean_std")
            if rms is None and "running_obs.running_mean" in m:
                rms = {k: m["running_obs." + k] for k in ("running_mean", "running_var", "count")}
            if rms is not None:
                L = rms["running_mean"].shape[0]
                n = int(rms["count"])
                mean[:L] = rms["running_mean"].float().to(D64)
                std[:L] = torch.sqrt(rms["running_var"].float()).to(D64)
        nets.append(dict(layers=layers, norm="running", n=n, mean=mean, std=std))
    return nets
