"""Cost of the sampled action (a stochastic player) in the tennis controller's test loop, single player at 8192 envs and dual at 2 x 8192,
in one run, alternating deterministic and sampled in every round:

  policy   det       nn.V2PPolicy.forward_prepared: the four bf16 wgmma layers per network, mu
           sampled   the same with deterministic=False: the last layer adds sigma * N(0, 1) in its epilogue and advances its step counter
  step     det       MVAEControllerVis(Dual).test_step(graph=True) with the deterministic policy: reset graph + policy/step graph
           sampled   the same with the sampling policy

Prints one JSON line: medians and spread (min, max) over the rounds in ms, with the card name and power limit read in the same run.
   python tools/perf_sampled_policy.py [--envs 8192] [--steps 30] [--rounds 7]
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
from perf_v2p_policy import random_networks, timed  # noqa: E402
from vid2player3d_b200 import nn  # noqa: E402
from vid2player3d_b200.configs import SIM_PARAMS, v2p_cfg, v2p_dual_cfg  # noqa: E402
from vid2player3d_b200.tasks import MVAEControllerVis, MVAEControllerVisDual  # noqa: E402


def measure(mode, N, K, rounds):
    frames = (rounds + 2) * K * 2 + 10

    def make():
        cfg = v2p_dual_cfg(N) if mode == "dual" else v2p_cfg(N)
        cfg["env"].update(record=True, num_rec_frames=frames, num_eg=1)
        return (MVAEControllerVisDual if mode == "dual" else MVAEControllerVis)(cfg, SIM_PARAMS, 1, "cuda", 0, True)
    P = 2 if mode == "dual" else 1
    envs = dict(det=make(), sampled=make())
    e0 = envs["det"]
    g = torch.Generator().manual_seed(1)
    nets = [dict(n, sigma=torch.exp(torch.rand(e0.num_actions, generator=g) - 2.0)) for n in random_networks(P, e0.num_obs, e0.num_actions)]
    pols = {k: nn.V2PPolicy(nets, N, e0.device, clip_obs=5.0, clip_actions=1.0, deterministic=(k == "det"), seed=7) for k in envs}
    for k, env in envs.items():
        env.set_policy(pols[k])
        env.reset()
        env.render_vis(init=True)
    fns = dict(policy_det=pols["det"].forward_prepared, policy_sampled=pols["sampled"].forward_prepared,
               step_det=lambda: envs["det"].test_step(True), step_sampled=lambda: envs["sampled"].test_step(True))
    for f in fns.values():                  # warm-up round (the graphed loops capture their graphs on their first call)
        timed(f, K)
    times = {k: [] for k in fns}
    for _ in range(rounds):
        for k, f in fns.items():
            times[k].append(timed(f, K))
    med = lambda v: sorted(v)[len(v) // 2]  # noqa: E731
    return dict(envs=N, networks=P, ms={k: dict(median=round(med(v), 4), min=round(min(v), 4), max=round(max(v), 4)) for k, v in times.items()})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=8192)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--rounds", type=int, default=7)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("perf_sampled_policy needs a CUDA device")
    res = dict(single=measure("single", a.envs, a.steps, a.rounds), dual=measure("dual", 2 * a.envs, a.steps, a.rounds))
    name, plim, smax = card()
    print(json.dumps(dict(gpu=name, power_limit=plim, sm_clock_max=smax, steps_per_round=a.steps, rounds=a.rounds, **res)))


if __name__ == "__main__":
    main()
