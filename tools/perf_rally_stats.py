"""Cost of the rally results of the dual test run (cfg.env.b200_rally_stats) in MVAEControllerVisDual's graphed test loop, 2 x 8192
envs (8192 pairs), alternating the two in every round:

  off   test_step(graph=True) without the key
  on    the same with b200_rally_stats: b200v2p_eval_rally_stats right after the post launch, in the step graph

Both tasks run the same high-level policies (random weights of the shipped shape, one per player).  Prints the median (min - max) ms
per test step of each, with the card's name and power limit read in the same run, and one JSON line.  Writes no file.
   python tools/perf_rally_stats.py [--envs 16384] [--steps 30] [--rounds 7]
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
from vid2player3d_b200.configs import SIM_PARAMS, v2p_dual_cfg  # noqa: E402
from vid2player3d_b200.tasks import MVAEControllerVisDual  # noqa: E402


def measure(N, K, rounds):
    def make(stats):
        cfg = v2p_dual_cfg(N)
        cfg["env"]["b200_rally_stats"] = stats
        return MVAEControllerVisDual(cfg, SIM_PARAMS, 1, "cuda", 0, True)
    envs = dict(off=make(False), on=make(True))
    assert envs["on"]._rstats is not None and envs["off"]._rstats is None
    e0 = envs["off"]
    nets = random_networks(2, e0.num_obs, e0.num_actions)
    for env in envs.values():
        env.set_policy(nn.V2PPolicy(nets, N, env.device, clip_obs=5.0, clip_actions=1.0))
        env.reset()
        env.render_vis(init=True)
    fns = {k: (lambda env=env: env.test_step(True)) for k, env in envs.items()}
    for f in fns.values():                  # warm-up round (the first call captures the graphs)
        timed(f, K)
    times = {k: [] for k in fns}
    for _ in range(rounds):
        for k, f in fns.items():
            times[k].append(timed(f, K))
    r = envs["on"]._rstats
    counted = dict(rallies=int(r["totals"][0]), hits=int(r["player"][:, 1].sum()))
    med = lambda v: sorted(v)[len(v) // 2]  # noqa: E731
    return dict(envs=N, counted=counted,
                ms={k: dict(median=round(med(v), 4), min=round(min(v), 4), max=round(max(v), 4)) for k, v in times.items()})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=16384)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--rounds", type=int, default=7)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("perf_rally_stats needs a CUDA device")
    res = measure(a.envs, a.steps, a.rounds)
    name, plim, smax = card()
    print(f"{name}, power limit {plim}, SM clock max {smax}; {a.envs} envs ({a.envs // 2} pairs), {a.rounds} alternating rounds of "
          f"{a.steps} graphed test steps ({res['counted']['rallies']} rallies, {res['counted']['hits']} hits counted)")
    for k, v in res["ms"].items():
        print(f"  {k:3s}: {v['median']:.3f} ms per step (min {v['min']:.3f}, max {v['max']:.3f})")
    print(json.dumps(dict(gpu=name, power_limit=plim, sm_clock_max=smax, steps_per_round=a.steps, rounds=a.rounds, **res)))


if __name__ == "__main__":
    main()
