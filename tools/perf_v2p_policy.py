"""Cost of the tennis controller's high-level policy in the test loop (V2PPlayer.run), single player at 8192 envs and dual at 2 x 8192
(16384 envs, two networks of 8192 rows each), in one run, alternating:

  policy alone   torch   the reference's fp32 path: normalise + clamp, four fp32 GEMMs with ReLU, the action clamp
                 wgmma   nn.V2PPolicy.forward_prepared: the four bf16 wgmma layers per network (the operand row comes from the post launch)
  test step      eager   reset_done + the torch policy on the clamped obs + the task's step graph + render_vis (the loop as the
                         reference runs it, with the step graph of enable_cuda_graph)
                 graph   MVAEControllerVis(Dual).test_step: the reset graph and one graph of policy + step + render_vis

Prints one JSON line: medians and spread (min, max) over the rounds in ms, with the card name and power limit read in the same run.
   python tools/perf_v2p_policy.py [--envs 8192] [--steps 30] [--rounds 5]
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from perf_eval import card  # noqa: E402
from vid2player3d_b200 import nn  # noqa: E402
from vid2player3d_b200.configs import SIM_PARAMS, v2p_cfg, v2p_dual_cfg  # noqa: E402
from vid2player3d_b200.tasks import MVAEControllerVis, MVAEControllerVisDual  # noqa: E402


def random_networks(P, obs, act, seed=0):
    g = torch.Generator().manual_seed(seed)
    dims = (obs, 1024, 1024, 512, act)
    nets = []
    for _ in range(P):
        layers = [((torch.rand(dims[i + 1], dims[i], generator=g) * 2 - 1) / dims[i] ** 0.5,
                   (torch.rand(dims[i + 1], generator=g) * 2 - 1) / dims[i] ** 0.5) for i in range(4)]
        nets.append(dict(layers=layers, mean=torch.randn(obs, generator=g) * 0.1, rstd=torch.rand(obs, generator=g) + 0.5, clip=5.0))
    return nets


class TorchPolicy:
    """the reference's fp32 policy forward on the device (per network: normaliser, actor MLP, mu), dual on rows 0::2 / 1::2"""

    def __init__(self, nets, clip_actions, dev):
        self.nets = [dict(layers=[(w.to(dev), b.to(dev)) for w, b in n["layers"]], mean=n["mean"].to(dev), rstd=n["rstd"].to(dev)) for n in nets]
        self.clip_actions = clip_actions

    @torch.no_grad()
    def __call__(self, obs):
        outs = []
        P = len(self.nets)
        for p, n in enumerate(self.nets):
            x = torch.clamp((obs[p::P] - n["mean"]) * n["rstd"], -5, 5)
            for i, (w, b) in enumerate(n["layers"]):
                x = torch.addmm(b, x, w.T)
                if i < 3:
                    x = torch.relu(x)
            outs.append(x)
        mu = torch.stack(outs, 1).reshape(obs.shape[0], -1) if P == 2 else outs[0]
        return torch.clamp(mu, -self.clip_actions, self.clip_actions)


def timed(fn, k):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    start.record()
    for _ in range(k):
        fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / k


def measure(mode, N, K, rounds):
    frames = (rounds + 2) * K * 2 + 10

    def make():
        cfg = v2p_dual_cfg(N) if mode == "dual" else v2p_cfg(N)
        cfg["env"].update(record=True, num_rec_frames=frames, num_eg=1)
        return (MVAEControllerVisDual if mode == "dual" else MVAEControllerVis)(cfg, SIM_PARAMS, 1, "cuda", 0, True)
    envs = dict(eager=make(), graph=make())
    P = 2 if mode == "dual" else 1
    e0 = envs["eager"]
    nets = random_networks(P, e0.num_obs, e0.num_actions)
    clip_obs, clip_act = 5.0, 1.0
    tp = TorchPolicy(nets, clip_act, e0.device)
    wp = nn.V2PPolicy(nets, N, e0.device, clip_obs=clip_obs, clip_actions=clip_act)
    envs["graph"].set_policy(wp)
    for env in envs.values():
        if env is e0:
            env.enable_cuda_graph()
        env.reset()
        env.render_vis(init=True)
    obs = torch.clamp(e0.obs_buf, -clip_obs, clip_obs)

    def eager_step():
        e0.reset_done()
        torch.clamp(e0.obs_buf, -clip_obs, clip_obs, out=obs)
        e0.step(tp(obs))
        e0.render_vis()

    fns = dict(policy_torch=lambda: tp(obs), policy_wgmma=wp.forward_prepared, step_eager=eager_step,
               step_graph=lambda: envs["graph"].test_step(True))
    for f in fns.values():                  # warm-up round (the graphed loop captures its graphs on its first call)
        timed(f, K)
    times = {k: [] for k in fns}
    for _ in range(rounds):
        for k, f in fns.items():
            times[k].append(timed(f, K))
    med = lambda v: sorted(v)[len(v) // 2]  # noqa: E731
    return dict(envs=N, networks=P, policy_gflop=round(wp.flops / 1e9, 3),
                ms={k: dict(median=round(med(v), 4), min=round(min(v), 4), max=round(max(v), 4)) for k, v in times.items()})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=8192)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--rounds", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("perf_v2p_policy needs a CUDA device")
    res = dict(single=measure("single", a.envs, a.steps, a.rounds), dual=measure("dual", 2 * a.envs, a.steps, a.rounds))
    name, plim, smax = card()
    print(json.dumps(dict(gpu=name, power_limit=plim, sm_clock_max=smax, steps_per_round=a.steps, rounds=a.rounds, **res)))


if __name__ == "__main__":
    main()
