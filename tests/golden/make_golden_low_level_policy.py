"""Golden fixture of the tennis controller's trained low-level imitation policy (v2p_low_level_policy.npz), produced by EXECUTING the
reference's own code on CPU: ImitatorPlayer.load_pretrained and load_dual_cp (vid2player/players/im_player.py:54-133) on fake players
reading checkpoints written here, RunningNorm.forward (models/running_norm.py), ImitatorBuilder.Network.eval_actor
(models/im_network_builder.py) and ImitatorBuilderDual.Network.eval_actor (models/im_network_builder_dual.py:37-45) on fake networks.
rl_games is absent, so its base classes are stand-ins; the actor MLP is built as rl_games builds it (Linear / ReLU x 3, linear mu,
mu_activation None), narrower than the shipped one to keep the fixture small (the observation keeps its 734 columns, the action its 75).
The networks run in float64 (the reference's code is dtype-agnostic), so that the fixture pins the float64 restatement closely.
Run where the reference is present:  python tests/golden/make_golden_low_level_policy.py

Cases, single (load_pretrained): RunningNorm keys, RunningNorm at n == 0, rl_games `running_mean_std` of the checkpoint, rl_games
`running_obs.running_*` of the model, a checkpoint with both RunningNorm and rl_games keys, and a Lightning checkpoint.  Dual
(load_dual_cp, one checkpoint per player): RunningNorm keys with the second network at n == 0; `running_mean_std` and the in-model
rl_games keys; both kinds of keys and RunningNorm keys.  Every observation batch mixes ordinary rows with rows far outside the clamps at
odd and even envs.
"""
import contextlib
import io
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

sys.path.insert(0, os.path.join(_refenv.REF, "vid2player"))


# ---- stand-ins for the absent rl_games pieces the reference modules import
class _A2CNetwork(tnn.Module):
    def __init__(self, params, **kwargs):
        super().__init__()


class _A2CBuilder:
    Network = _A2CNetwork

    def __init__(self, **kwargs):
        pass


def _module(name, **attrs):
    m = types.ModuleType(name)
    m.__dict__.update(attrs)
    sys.modules[name] = m
    return m


_module("rl_games")
_module("rl_games.algos_torch")
_module("rl_games.algos_torch.network_builder", A2CBuilder=_A2CBuilder)
_module("rl_games.algos_torch.running_mean_std", RunningMeanStd=object)
_module("rl_games.algos_torch.torch_ext", shape_whc_to_cwh=lambda s: s)
_module("rl_games.common")
_module("rl_games.common.player", BasePlayer=object)
_module("learning")
_module("learning.common_player", CommonPlayer=object)

from models.im_network_builder import ImitatorBuilder  # noqa: E402
from models.im_network_builder_dual import ImitatorBuilderDual  # noqa: E402
from models.running_norm import RunningNorm  # noqa: E402
from players.im_player import ImitatorPlayer  # noqa: E402

torch.set_num_threads(1)
OUT = {}
D, A, UNITS = 734, 75, (8, 8, 8)              # the shipped actor is 1024, 1024, 512 wide: the restatement is width-agnostic
g = torch.Generator().manual_seed(17)


def q(x, step):
    """x on a grid of `step` (a power of two): exact in float32 with short mantissas, so the fixture compresses well"""
    return torch.round(x / step) * step


def mlp(dims):
    layers = []
    for i in range(len(dims) - 1):
        layers += [tnn.Linear(dims[i], dims[i + 1]), tnn.ReLU()]
    return tnn.Sequential(*layers)


class FakeNet(tnn.Module):
    """the attributes ImitatorBuilder.Network.eval_actor reads, with rl_games's actor / critic layout and a RunningNorm"""
    eval_actor = ImitatorBuilder.Network.eval_actor

    def __init__(self):
        super().__init__()
        self.use_running_obs = True
        self.running_obs = RunningNorm(D)
        self.actor_cnn = tnn.Sequential()
        self.actor_mlp = mlp((D,) + UNITS)
        self.critic_mlp = mlp((D,) + UNITS)
        self.mu = tnn.Linear(UNITS[-1], A)
        self.value = tnn.Linear(UNITS[-1], 1)
        self.mu_act = self.sigma_act = tnn.Identity()
        self.sigma = tnn.Parameter(torch.zeros(A), requires_grad=False)
        self.is_discrete = self.is_multi_discrete = False
        self.is_continuous = True
        self.space_config = {"fixed_sigma": True}


class Model(tnn.Module):
    def __init__(self, net):
        super().__init__()
        self.a2c_network = net


def randomize(mod):
    with torch.no_grad():
        for name, p in mod.named_parameters():
            p.copy_(q((torch.rand(p.shape, generator=g) * 2 - 1) * (2.0 / max(p.shape[-1], 1)) ** 0.5, 2.0 ** -10))


def stats():
    mean = q(torch.randn(D, generator=g) * 2, 2.0 ** -6)
    var = q(torch.rand(D, generator=g) * 3, 2.0 ** -6) + 2.0 ** -6
    return mean, var


def checkpoint(kind):
    """a checkpoint as training writes it: a2c_network.* weights, plus
    running: RunningNorm buffers (n 4096); n0: RunningNorm at n == 0; rms: rl_games running_mean_std of the checkpoint; inmodel: the
    rl_games buffers running_obs.{running_mean,running_var,count} of the model; both: RunningNorm buffers (n 100) and a running_mean_std
    of other statistics; lightning: a Lightning checkpoint, state_dict without the a2c_network prefix, RunningNorm buffers (n 512)"""
    src = FakeNet()
    randomize(src)
    sd = {k: v.clone() for k, v in Model(src).state_dict().items() if "running_obs" not in k}
    ck = {"model": sd}
    mean, var = stats()
    if kind in ("running", "n0", "both", "lightning"):
        sd["a2c_network.running_obs.n"] = torch.tensor({"running": 4096, "n0": 0, "both": 100, "lightning": 512}[kind], dtype=torch.long)
        sd["a2c_network.running_obs.mean"], sd["a2c_network.running_obs.var"] = mean, var
        sd["a2c_network.running_obs.std"] = torch.sqrt(var)
    if kind in ("rms", "both"):
        m2, v2 = stats() if kind == "both" else (mean, var)
        ck["running_mean_std"] = {"running_mean": m2.double(), "running_var": v2.double(), "count": torch.tensor(2048.0, dtype=torch.float64)}
    if kind == "inmodel":
        sd["a2c_network.running_obs.running_mean"], sd["a2c_network.running_obs.running_var"] = mean.double(), var.double()
        sd["a2c_network.running_obs.count"] = torch.tensor(1024.0, dtype=torch.float64)
    if kind == "lightning":
        return {"pytorch-lightning_version": "1.5.0", "state_dict": {k[len("a2c_network."):]: v for k, v in sd.items()}}
    return ck


def obs_batch(N):
    x = q(torch.randn(N, D, generator=g) * 3, 2.0 ** -4)
    reset = torch.zeros(N, dtype=torch.bool)
    reset[torch.tensor([1, 2, 5, 6, N - 1])] = True          # odd and even rows
    x[reset] = q((torch.rand(int(reset.sum()), D, generator=g) * 2 - 1) * 60, 2.0 ** -2)
    return x.double(), reset


def fresh():
    net = FakeNet()
    randomize(net)                                           # overwritten by the loader
    return net.double().eval()


def record(prefix, ck, net, x=None):
    if "state_dict" in ck:
        OUT[f"{prefix}_lightning"] = np.array(1)
        items = {"a2c_network." + k: v for k, v in ck["state_dict"].items()}.items()
    else:
        items = ck["model"].items()
    for k, v in items:
        if "critic" not in k and "value" not in k and "sigma" not in k:
            OUT[f"{prefix}_model:{k}"] = v.numpy()
    for k, v in ck.get("running_mean_std", {}).items():
        OUT[f"{prefix}_rms:{k}"] = v.numpy()
    OUT[f"{prefix}_ro_n"] = np.array(int(net.running_obs.n))
    OUT[f"{prefix}_ro_mean"], OUT[f"{prefix}_ro_std"] = net.running_obs.mean.numpy(), net.running_obs.std.numpy()
    if x is not None:
        with torch.no_grad():
            OUT[f"{prefix}_norm"] = net.running_obs(x[:3]).float().numpy()   # RunningNorm.forward alone (3 rows in float32: a small file)


def save(tmp, name, ck):
    p = os.path.join(tmp, name)
    torch.save(ck, p)
    return p


SINGLE = ("running", "n0", "rms", "inmodel", "both", "lightning")
DUAL = {"running_n0": ("running", "n0"), "rms_inmodel": ("rms", "inmodel"), "both_running": ("both", "running")}
with tempfile.TemporaryDirectory() as tmp, contextlib.redirect_stdout(io.StringIO()):
    # ---------------------------------------------------------------- single: load_pretrained + RunningNorm + eval_actor
    for kind in SINGLE:
        ck = checkpoint(kind)
        net = fresh()
        player = types.SimpleNamespace(model=Model(net), config={}, normalize_input=False, device="cpu")
        player.set_weights = lambda w, p=player: ImitatorPlayer.set_weights(p, w)
        ImitatorPlayer.load_pretrained(player, save(tmp, f"{kind}.pth", ck))
        x, reset = obs_batch(8)
        with torch.no_grad():
            mu, _ = net.eval_actor({"obs": x})
        case = "single_" + kind
        record(case, ck, net, x)
        OUT[f"{case}_obs"], OUT[f"{case}_reset_rows"], OUT[f"{case}_mu"] = x.float().numpy(), reset.numpy(), mu.numpy()   # obs: exact in float32

    # ---------------------------------------------------------------- dual: load_dual_cp + ImitatorBuilderDual.eval_actor
    for name, kinds in DUAL.items():
        cks = [checkpoint(k) for k in kinds]
        dual = types.SimpleNamespace(network1=fresh(), network2=fresh())
        player = types.SimpleNamespace(config={}, device="cpu", model=types.SimpleNamespace(a2c_network=dual))
        ImitatorPlayer.load_dual_cp(player, [save(tmp, f"{name}_{i}.pth", ck) for i, ck in enumerate(cks)])
        x, reset = obs_batch(8)
        with torch.no_grad():
            mu, _ = ImitatorBuilderDual.Network.eval_actor(dual, {"obs": x})
        case = "dual_" + name
        for i, (ck, net) in enumerate(zip(cks, (dual.network1, dual.network2))):
            record(f"{case}{i}", ck, net, x[i::2])
        OUT[f"{case}_obs"], OUT[f"{case}_reset_rows"], OUT[f"{case}_mu"] = x.float().numpy(), reset.numpy(), mu.numpy()   # obs: exact in float32

np.savez_compressed(os.path.join(HERE, "v2p_low_level_policy.npz"), **OUT)
print(f"wrote v2p_low_level_policy.npz: {len(OUT)} arrays, {os.path.getsize(os.path.join(HERE, 'v2p_low_level_policy.npz'))} bytes")
