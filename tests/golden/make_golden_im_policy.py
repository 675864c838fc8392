"""Golden fixture of the embodied_pose imitation policy at test time (im_policy.npz), produced by EXECUTING the reference's own code on
CPU: ImitatorBuilder.Network.forward_context / preprocess_input / eval_actor (embodied_pose/models/im_network_builder.py) with
RunningNorm.forward (models/running_norm.py) on fake networks, ImitatorPlayer.load_pretrained (players/im_player.py:53-94) on a fake
player reading checkpoints written here, and ImitatorPlayer.run (:193-312) on a fake player and env with scripted rewards and
dones, its printed lines captured.  rl_games is absent, so its base classes are stand-ins; the actor MLP is built as rl_games builds it
(Linear / ReLU x 3, linear mu, mu_activation None), narrower than the shipped one to keep the fixture small (the observation keeps the
24-body shape, 734 wide).
Run where the reference is present:  python tests/golden/make_golden_im_policy.py

Cases of the actor: RunningNorm at n == 0 (identity), RunningNorm statistics of the checkpoint, rl_games statistics filled into the
RunningNorm by load_pretrained's load_rlgame_norm branch; every observation batch holds rows far outside the clamps; context slots
t = 0, 1 and L - 1.  Cases of the loop: an env that stays done for several steps, done[0] ending a game, and games_num reached in the
middle of a step."""
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
_module("rl_games.algos_torch.players", rescale_actions=None, unsqueeze_obs=None)
_module("rl_games.common")
_module("rl_games.common.player", BasePlayer=object)
_module("learning")
_module("learning.common_player", CommonPlayer=object)
_refenv.setup("embodied_pose")

from models.im_network_builder import ImitatorBuilder  # noqa: E402
from models.running_norm import RunningNorm  # noqa: E402
from players.im_player import ImitatorPlayer  # noqa: E402

torch.set_num_threads(1)
OUT = {}
NB, ND, SD = 24, 69, 11
D, A, UNITS = 734, 75, (16, 16, 16)
L, PAD = 4, 2                                 # the shipped window is 32 + 2 x 8 frames: the restatement is length-agnostic
P = L + 2 * PAD
g = torch.Generator().manual_seed(13)
Net = ImitatorBuilder.Network


def q(x, step):
    return torch.round(x / step) * step


def mlp(dims):
    layers = []
    for i in range(len(dims) - 1):
        layers += [tnn.Linear(dims[i], dims[i + 1]), tnn.ReLU()]
    return tnn.Sequential(*layers)


class FakeNet(tnn.Module):
    """the attributes ImitatorBuilder.Network's non-training forward reads, with rl_games's actor layout"""
    forward_context, obtain_cur_context, compute_humanoid_obs = Net.forward_context, Net.obtain_cur_context, Net.compute_humanoid_obs
    preprocess_input, eval_actor, setup_env_named_dims = Net.preprocess_input, Net.eval_actor, Net.setup_env_named_dims

    def __init__(self):
        super().__init__()
        self.context_padding, self.use_running_obs, self.use_ik, self.residual_action = PAD, True, False, True
        self.running_obs = RunningNorm(D)
        self.actor_cnn = tnn.Sequential()
        self.actor_mlp = mlp((D,) + UNITS)
        self.mu = tnn.Linear(UNITS[-1], A)
        self.mu_act = self.sigma_act = tnn.Identity()
        self.sigma = tnn.Parameter(torch.zeros(A), requires_grad=False)
        self.is_discrete = self.is_multi_discrete = False
        self.is_continuous = True
        self.space_config = {"fixed_sigma": True}
        shapes = {'body_pos': (NB, 3), 'body_pos_gt': (NB, 3), 'body_rot': (NB, 4), 'dof_pos': (ND,), 'dof_pos_gt': (ND,),
                  'dof_vel': (ND,), 'body_vel': (NB, 3), 'body_ang_vel': (NB, 3), 'motion_bodies': (SD,)}
        on = ['body_pos', 'body_rot', 'dof_pos', 'dof_vel', 'body_vel', 'body_ang_vel', 'motion_bodies']
        cn = ['body_pos', 'body_rot', 'dof_pos', 'body_pos_gt', 'dof_pos_gt']
        self.setup_env_named_dims(on, [shapes[x] for x in on], [int(np.prod(shapes[x])) for x in on], cn, [shapes[x] for x in cn],
                                  [int(np.prod(shapes[x])) for x in cn])


class Model(tnn.Module):
    def __init__(self, net):
        super().__init__()
        self.a2c_network = net


def randomize(mod):
    with torch.no_grad():
        for name, p in mod.named_parameters():
            if "running_obs" not in name:
                p.copy_(q((torch.rand(p.shape, generator=g) * 2 - 1) * (2.0 / max(p.shape[-1], 1)) ** 0.5, 2.0 ** -10))


def checkpoint(kind):
    """a checkpoint as training writes it: a2c_network.* weights and RunningNorm buffers (kind running / n0), or no running_obs keys
    and rl_games running_mean_std (kind rlgame)"""
    src = FakeNet()
    randomize(src)
    mean = q(torch.randn(D, generator=g), 2.0 ** -6)
    var = q(torch.rand(D, generator=g) * 3, 2.0 ** -6) + 2.0 ** -6
    sd = {k: v.clone() for k, v in Model(src).state_dict().items() if "running_obs" not in k}
    ck = {"model": sd}
    if kind in ("running", "n0"):
        sd["a2c_network.running_obs.n"] = torch.tensor(0 if kind == "n0" else 4096, dtype=torch.long)
        sd["a2c_network.running_obs.mean"], sd["a2c_network.running_obs.var"] = mean, var
        sd["a2c_network.running_obs.std"] = torch.sqrt(var)
    else:
        ck["running_mean_std"] = {"running_mean": mean.double(), "running_var": var.double(), "count": torch.tensor(2048.0, dtype=torch.float64)}
    return ck


def inputs(N):
    """raw observations (with rows far outside the clamps) and a context window"""
    obs = q(torch.randn(N, 13 * NB + 2 * ND + SD, generator=g), 2.0 ** -6)
    rot = torch.nn.functional.normalize(torch.randn(N, NB, 4, generator=g), dim=-1)
    obs[:, 3 * NB:7 * NB] = q(rot.reshape(N, -1), 2.0 ** -10)
    obs[1, ::5] = 40.0
    obs[N - 1, 2::5] = -40.0
    feat = q(torch.randn(N, P, 2 * (3 * NB + ND) + 4 * NB, generator=g), 2.0 ** -6)
    frot = torch.nn.functional.normalize(torch.randn(N, P, NB, 4, generator=g), dim=-1)
    feat[:, :, 3 * NB:7 * NB] = q(frot.reshape(N, P, -1), 2.0 ** -10)
    return obs, feat


obs, feat = inputs(6)
OUT["obs"], OUT["feat"] = obs.numpy(), feat.numpy()
with tempfile.TemporaryDirectory() as tmp:
    for case in ("n0", "running", "rlgame"):
        ck = checkpoint(case)
        path = os.path.join(tmp, f"{case}.pth")
        torch.save(ck, path)
        net = FakeNet()
        randomize(net)
        net.eval()
        player = types.SimpleNamespace(model=Model(net), config={}, normalize_input=False, device="cpu")
        player.set_weights = lambda w, p=player: ImitatorPlayer.set_weights(p, w)
        with contextlib.redirect_stdout(io.StringIO()):
            ImitatorPlayer.load_pretrained(player, path)
        with torch.no_grad():
            net.forward_context(feat, None)
            for t in (0, 1, L - 1):
                d = {"obs": obs.clone(), "t": t}
                mu, _ = net.eval_actor(d)
                OUT[f"{case}_mu_t{t}"] = mu.numpy()
                OUT[f"human_obs_t{t}"] = d["human_obs"].numpy()
                if t == 0:
                    OUT[f"{case}_norm"] = net.running_obs(d["human_obs"]).numpy()       # RunningNorm.forward alone
        for k, v in ck["model"].items():
            if "actor_mlp" in k or k.startswith("a2c_network.mu.") or "running_obs" in k:
                OUT[f"{case}_model:{k}"] = v.numpy()
        for k, v in ck.get("running_mean_std", {}).items():
            OUT[f"{case}_rms:{k}"] = v.numpy()
        OUT[f"{case}_ro_n"] = np.array(int(net.running_obs.n))
        OUT[f"{case}_ro_mean"], OUT[f"{case}_ro_std"] = net.running_obs.mean.numpy(), net.running_obs.std.numpy()

# ---------------------------------------------------------------- ImitatorPlayer.run on scripted rewards / dones
N, GAMES_NUM, MAX_STEPS = 6, 8, 12
hist = []


def script(game, n):
    """rewards on a 1/8 grid (sums exact in float32); dones: env 3 stays done from step 2 to 5 and again from 8, env 5 done at step 1
    and from 6; game 0 ends when env 0 is done at step 9; game 1 reaches games_num when three envs finish at step 4"""
    r = q(torch.rand(N, generator=g) * 2, 0.125)
    d = torch.zeros(N, dtype=torch.long)
    if game == 0:
        d[3] = int(2 <= n <= 5 or n >= 8)
        d[5] = int(n == 1 or n >= 6)
        d[0] = int(n >= 9)
        d[2] = int(n >= 7)
    else:
        d[[1, 2, 4]] = int(n >= 4)
        d[3] = int(n >= 2)
    return r, d


def env_reset():
    hist.append([])
    return {"obs": torch.zeros(N, 4)}


def env_step(env, action):
    r, d = script(len(hist) - 1, len(hist[-1]))
    hist[-1].append((r.numpy(), d.numpy()))
    return {"obs": torch.zeros(N, 4)}, r, d, {}


task = types.SimpleNamespace(context_length=L, _reset_ref_motion_ids=None, _cur_ref_motion_times=None,
                             _init_context=lambda *a: None, render_vis=lambda init=False: None)
player = types.SimpleNamespace(games_num=GAMES_NUM, render_env=False, n_game_life=1, is_determenistic=True, env=types.SimpleNamespace(),
                               env_reset=env_reset, get_batch_size=lambda obs, bs: obs.shape[0], is_rnn=False, task=task, max_steps=MAX_STEPS,
                               get_action=lambda obs, det: torch.zeros(N, A), env_step=env_step, _post_step=lambda info: None,
                               num_agents=1, print_stats=True, device="cpu")
buf = io.StringIO()
with contextlib.redirect_stdout(buf):
    ImitatorPlayer.run(player)
lines = buf.getvalue().splitlines()
OUT["run_printed"] = np.array(lines)
OUT["run_args"] = np.array([N, GAMES_NUM, MAX_STEPS, 1])
for i, game in enumerate(hist):
    OUT[f"run_game{i}_rew"] = np.stack([r for r, _ in game])
    OUT[f"run_game{i}_done"] = np.stack([d for _, d in game])

np.savez_compressed(os.path.join(HERE, "im_policy.npz"), **OUT)
print(f"wrote im_policy.npz: {len(OUT)} arrays; run printed:\n" + "\n".join(lines))
