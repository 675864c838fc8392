"""Golden fixture of the tennis controller's high-level policy at test time (v2p_policy.npz), produced by EXECUTING the reference's own
code on CPU: RunningNorm.forward (vid2player/models/running_norm.py), V2PBuilder.Network.eval_actor and V2PBuilderDual.Network.eval_actor
(models/v2p_network_builder.py, v2p_network_builder_dual.py) on fake networks, and V2PPlayer.restore / load_dual_cp
(players/v2p_player.py:21-111) on a fake player reading checkpoints written here.  rl_games is absent, so its base classes are stand-ins
and the single-player normaliser (RunningMeanStd, an rl_games class) is restated: clamp((x - mean) / sqrt(var + 1e-5), -5, 5).  The
actor MLP is restated as rl_games builds it (Linear / ReLU x 3, linear mu, mu_activation None), narrower than the shipped one to keep
the fixture small.
Run where the reference is present:  python tests/golden/make_golden_v2p_policy.py

Cases: single, checkpoint at the network's width and with a padded first layer (checkpoint 250 observations, network 257); dual with
(a) both networks' RunningNorm in the checkpoints, (b) one network at n == 0 (identity) and (c) a padded first layer with the rl_games
statistics loaded as RunningNorm's prefix.  Every observation batch mixes ordinary rows with "reset" rows at odd and even envs whose
values lie far outside the clamps.
"""
import os
import sys
import tempfile
import types

import numpy as np
import torch
import torch.nn as tnn

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import _refenv  # noqa: E402

REF_V2P = os.path.join(_refenv.REF, "vid2player")
sys.path.insert(0, REF_V2P)


# ---- stand-ins for the absent rl_games pieces the reference modules import
class _A2CNetwork(tnn.Module):
    def __init__(self, params, **kwargs):
        super().__init__()


class _A2CBuilder:
    Network = _A2CNetwork

    def __init__(self, **kwargs):
        pass


class _RunningMeanStd(tnn.Module):
    def __init__(self, shape, epsilon=1e-5):
        super().__init__()
        self.epsilon = epsilon
        self.register_buffer("running_mean", torch.zeros(shape, dtype=torch.float64))
        self.register_buffer("running_var", torch.ones(shape, dtype=torch.float64))
        self.register_buffer("count", torch.ones((), dtype=torch.float64))

    def forward(self, x):   # rl_games running_mean_std.py, eval mode, norm_only False
        y = (x - self.running_mean.float()) / torch.sqrt(self.running_var.float() + self.epsilon)
        return torch.clamp(y, min=-5.0, max=5.0)


def _module(name, **attrs):
    m = types.ModuleType(name)
    m.__dict__.update(attrs)
    sys.modules[name] = m
    return m


_module("rl_games")
_module("rl_games.algos_torch")
_module("rl_games.algos_torch.network_builder", A2CBuilder=_A2CBuilder)
_module("rl_games.algos_torch.running_mean_std", RunningMeanStd=_RunningMeanStd)
_module("rl_games.algos_torch.torch_ext", load_checkpoint=lambda p: torch.load(p, map_location="cpu", weights_only=False))
_module("learning")
_module("learning.common_player", CommonPlayer=object)
_module("tqdm", tqdm=lambda x: x)

from models.running_norm import RunningNorm  # noqa: E402
from models.v2p_network_builder import V2PBuilder  # noqa: E402
from models.v2p_network_builder_dual import V2PBuilderDual  # noqa: E402
from players.v2p_player import V2PPlayer  # noqa: E402

torch.set_num_threads(1)
OUT = {}
D, A, UNITS = 257, 35, (16, 16, 16)         # the shipped actor is 1024, 1024, 512 wide: the restatement is width-agnostic
D_CK = 250                                   # the narrower checkpoint of the padded cases
g = torch.Generator().manual_seed(11)


def mlp(dims):
    layers = []
    for i in range(len(dims) - 1):
        layers += [tnn.Linear(dims[i], dims[i + 1]), tnn.ReLU()]
    return tnn.Sequential(*layers)


class FakeNet(tnn.Module):
    """the attributes V2PBuilder.Network.eval_actor reads, with rl_games's actor layout"""
    eval_actor = V2PBuilder.Network.eval_actor

    def __init__(self, use_running_obs):
        super().__init__()
        self.use_running_obs = use_running_obs
        if use_running_obs:
            self.running_obs = RunningNorm(D)
        self.actor_cnn = tnn.Sequential()
        self.actor_mlp = mlp((D,) + UNITS)
        self.critic_mlp = mlp((D,) + UNITS)
        self.mu = tnn.Linear(UNITS[-1], A)
        self.value = tnn.Linear(UNITS[-1], 1)
        self.mu_act = self.sigma_act = tnn.Identity()
        self.sigma = tnn.Parameter(torch.zeros(A))
        self.is_discrete = self.is_multi_discrete = False
        self.is_continuous = True
        self.space_config = {"fixed_sigma": True}


def q(x, step):
    """x on a grid of `step` (a power of two): exact in float32 with short mantissas, so the fixture compresses to a few hundred KB"""
    return torch.round(x / step) * step


def randomize(net):
    with torch.no_grad():
        for p in net.parameters():
            p.copy_(q((torch.rand(p.shape, generator=g) * 2 - 1) * (2.0 / max(p.shape[-1], 1)) ** 0.5, 2.0 ** -10))


def trained_ckpt(obs_dim, use_running_obs, rl_stats, n=None):
    """a checkpoint as training writes it: a2c_network.* weights (+ running_obs buffers) and optionally rl_games running_mean_std"""
    src = FakeNet(False)
    if obs_dim != D:
        src.actor_mlp[0] = tnn.Linear(obs_dim, UNITS[0])
        src.critic_mlp[0] = tnn.Linear(obs_dim, UNITS[0])
    randomize(src)
    model = {"a2c_network." + k: v.clone() for k, v in src.state_dict().items()}
    mean = q(torch.randn(obs_dim, generator=g) * 2, 2.0 ** -6)
    var = q(torch.rand(obs_dim, generator=g) * 3, 2.0 ** -6) + 2.0 ** -6
    if use_running_obs:
        model["a2c_network.running_obs.n"] = torch.tensor(n, dtype=torch.long)
        model["a2c_network.running_obs.mean"] = mean.float()
        model["a2c_network.running_obs.var"] = var.float()
        model["a2c_network.running_obs.std"] = torch.sqrt(var).float()
    ck = {"model": model}
    if rl_stats:
        ck["running_mean_std"] = {"running_mean": mean.double(), "running_var": var.double(), "count": torch.tensor(4096.0, dtype=torch.float64)}
    return ck


def obs_batch(N):
    x = q(torch.randn(N, D, generator=g) * 3, 2.0 ** -4)
    reset = torch.zeros(N, dtype=torch.bool)
    reset[torch.tensor([1, 2, 5, 6, N - 1])] = True          # odd and even rows
    x[reset] = q((torch.rand(int(reset.sum()), D, generator=g) * 2 - 1) * 60, 2.0 ** -2)
    return x, reset


def save(tmp, name, ck):
    p = os.path.join(tmp, name)
    torch.save(ck, p)
    return p


def flat_ck(prefix, ck):
    for k, v in ck["model"].items():
        if "critic" not in k and "value" not in k:
            OUT[f"{prefix}_model:{k}"] = v.numpy()
    for k, v in ck.get("running_mean_std", {}).items():
        OUT[f"{prefix}_rms:{k}"] = v.numpy()


with tempfile.TemporaryDirectory() as tmp:
    # ---------------------------------------------------------------- single: restore + rl_games normaliser + eval_actor
    for case, obs_dim in (("single_full", D), ("single_padded", D_CK)):
        ck = trained_ckpt(obs_dim, False, True)
        net = FakeNet(False)
        randomize(net)                                    # overwritten by restore (the padded layer is zeroed first)
        player = types.SimpleNamespace(config={"name": "ctrl"}, network_path=tmp, normalize_input=True,
                                       model=types.SimpleNamespace(a2c_network=net, load_state_dict=lambda sd, strict=True, n=net:
                                                                   n.load_state_dict({k[len("a2c_network."):]: v for k, v in sd.items()}, strict=False)),
                                       running_mean_std=_RunningMeanStd(D))
        save(tmp, "ctrl_best.pth", ck)
        V2PPlayer.restore(player, "best")
        x, reset = obs_batch(16)
        with torch.no_grad():
            mu, _ = net.eval_actor({"obs": player.running_mean_std(x)})
        flat_ck(case, ck)
        OUT[f"{case}_obs"], OUT[f"{case}_reset_rows"], OUT[f"{case}_mu"] = x.numpy(), reset.numpy(), mu.numpy()
        OUT[f"{case}_rms_mean"] = player.running_mean_std.running_mean.numpy()
        OUT[f"{case}_rms_var"] = player.running_mean_std.running_var.numpy()
        if obs_dim != D:                                  # the zero-padded first layer restore leaves (else: the checkpoint's own)
            OUT[f"{case}_w0"] = net.actor_mlp[0].weight.detach().numpy()

    # ---------------------------------------------------------------- dual: load_dual_cp + RunningNorm + V2PBuilderDual.eval_actor
    cases = {
        "dual_running": (trained_ckpt(D, True, False, n=1000), trained_ckpt(D, True, False, n=7)),
        "dual_n0": (trained_ckpt(D, True, False, n=500), trained_ckpt(D, True, False, n=0)),
        "dual_padded": (trained_ckpt(D_CK, False, True), trained_ckpt(D_CK, False, True)),
    }
    for case, cks in cases.items():
        dual = types.SimpleNamespace(network1=FakeNet(True), network2=FakeNet(True))
        for n in (dual.network1, dual.network2):
            randomize(n)
            n.eval()
        player = types.SimpleNamespace(config={}, device="cpu", model=types.SimpleNamespace(a2c_network=dual))
        paths = [save(tmp, f"{case}_{i}.pth", ck) for i, ck in enumerate(cks)]
        V2PPlayer.load_dual_cp(player, paths)
        x, reset = obs_batch(16)
        with torch.no_grad():
            mu, _ = V2PBuilderDual.Network.eval_actor(dual, {"obs": x})
            norm = [n.running_obs(x[i::2]) for i, n in enumerate((dual.network1, dual.network2))]   # RunningNorm.forward alone
        for i, ck in enumerate(cks):
            flat_ck(f"{case}{i}", ck)
            n = (dual.network1, dual.network2)[i]
            OUT[f"{case}{i}_ro_n"] = np.array(int(n.running_obs.n))
            OUT[f"{case}{i}_ro_mean"] = n.running_obs.mean.numpy()
            OUT[f"{case}{i}_ro_std"] = n.running_obs.std.numpy()
            OUT[f"{case}{i}_norm"] = norm[i].numpy()
            if case == "dual_padded":
                OUT[f"{case}{i}_w0"] = n.actor_mlp[0].weight.detach().numpy()
        OUT[f"{case}_obs"], OUT[f"{case}_reset_rows"], OUT[f"{case}_mu"] = x.numpy(), reset.numpy(), mu.numpy()

np.savez_compressed(os.path.join(HERE, "v2p_policy.npz"), **OUT)
print(f"wrote v2p_policy.npz: {len(OUT)} arrays")
