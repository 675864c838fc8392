"""float64 restatement of the checkpoint loaders of the tennis controller's trained low-level imitation policy (vid2player's
ImitatorPlayer, players/im_player.py, paths relative to the vid2player tree).  The forward is oracle/ref_port_v2p_policy.act (RunningNorm,
eval_actor, the dual interleave); the single loader is oracle/ref_port_im_policy.load (load_pretrained, line for line the embodied_pose
one).  What is new here is load_dual_cp (:54-90), which differs from V2PPlayer.load_dual_cp (ref_port_v2p_policy.load_dual): the first
layer is loaded as it is (a narrower one makes load_state_dict fail), and rl_games statistics fill the whole RunningNorm row.
tests/golden/v2p_low_level_policy.npz (made by executing the reference's own code, tests/golden/make_golden_low_level_policy.py)
pins it."""
import torch

from oracle import ref_port_im_policy as IM
from oracle.ref_port_v2p_policy import ACTOR_KEYS

D64 = torch.float64


def load_single(ck, obs_dim=734):
    """load_pretrained (tennis_im.yaml: use_running_obs, running_obs_type ours) as ref_port_v2p_policy.act's network dict"""
    net = IM.load(ck, obs_dim=obs_dim)
    t = lambda a: torch.as_tensor(a, dtype=D64)  # noqa: E731
    return dict(layers=[(t(w), t(b)) for w, b in net["layers"]], norm="running", n=net["n"], mean=t(net["mean"]), std=t(net["std"]))


def load_dual(cks, obs_dim=734):
    """load_dual_cp for network1 / network2: the actor weights as they are, the model's RunningNorm or, when the checkpoint has none,
    the rl_games statistics (std = sqrt(var)) over the whole row; a fresh RunningNorm (n 0: identity) when there is neither"""
    nets = []
    for ck in cks:
        m = {k[len("a2c_network."):]: v for k, v in ck["model"].items()}
        layers = [(m[k + ".weight"].to(D64), m[k + ".bias"].to(D64)) for k in ACTOR_KEYS]
        assert layers[0][0].shape[1] == obs_dim, "load_state_dict refuses a first layer of another width"
        mean, std, n = torch.zeros(obs_dim, dtype=D64), torch.zeros(obs_dim, dtype=D64), 0
        if "running_obs.n" in m:
            n, mean, std = int(m["running_obs.n"]), m["running_obs.mean"].to(D64), m["running_obs.std"].to(D64)
        else:
            rms = ck.get("running_mean_std")
            if rms is None and "running_obs.running_mean" in m:
                rms = {k: m["running_obs." + k] for k in ("running_mean", "running_var", "count")}
            if rms is not None:
                n = int(rms["count"])
                mean = rms["running_mean"].float().to(D64)
                std = torch.sqrt(rms["running_var"].float()).to(D64)
        assert mean.shape[0] == obs_dim and std.shape[0] == obs_dim, "the statistics fill the whole row"
        nets.append(dict(layers=layers, norm="running", n=n, mean=mean, std=std))
    return nets
