"""Cost of evaluating the tennis controller on a fixed test set of incoming balls (env.ball_traj_file_test) instead of random pool rows,
in MVAEControllerVis' graphed test loop, single player at 8192 envs, alternating the two in every round:

  random     test_step(graph=True) with the training pool drawn at random (b200v2p_task_reset, random branch)
  test_set   the same with the same rows as a test set walked in order (the launch's pool_cursor branch)

Both tasks run the same high-level policy (random weights of the shipped shape) on the same pool.  Prints one JSON line: median and
spread (min, max) over the rounds in ms per test step, with the card name and power limit read in the same run.
   python tools/perf_test_set.py [--envs 8192] [--steps 30] [--rounds 5]
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
from vid2player3d_b200 import ball as ball_data, nn  # noqa: E402
from vid2player3d_b200.configs import SIM_PARAMS, v2p_cfg  # noqa: E402
from vid2player3d_b200.tasks import MVAEControllerVis  # noqa: E402


def measure(N, K, rounds):
    pool = ball_data.synthetic_pool(2048, seed=10, spin_scale=5.0)

    def make(test_set):
        over = dict(test_mode="multiple_cycle", ball_pool_test=pool) if test_set else dict(ball_pool=pool)
        return MVAEControllerVis(v2p_cfg(N, **over), SIM_PARAMS, 1, "cuda", 0, True)
    envs = dict(random=make(False), test_set=make(True))
    assert envs["test_set"]._physics_player.task._ball_pool_cursor is not None
    assert envs["random"]._physics_player.task._ball_pool_cursor is None
    e0 = envs["random"]
    nets = random_networks(1, e0.num_obs, e0.num_actions)
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
    resets = {k: int(env._num_reset_reaction.sum()) for k, env in envs.items()}
    med = lambda v: sorted(v)[len(v) // 2]  # noqa: E731
    return dict(envs=N, reaction_resets=resets,
                ms={k: dict(median=round(med(v), 4), min=round(min(v), 4), max=round(max(v), 4)) for k, v in times.items()})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=8192)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--rounds", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("perf_test_set needs a CUDA device")
    res = measure(a.envs, a.steps, a.rounds)
    name, plim, smax = card()
    print(json.dumps(dict(gpu=name, power_limit=plim, sm_clock_max=smax, steps_per_round=a.steps, rounds=a.rounds, **res)))


if __name__ == "__main__":
    main()
