"""Cost of HumanoidSMPLIMVis' pose metrics in the graphed test step (HumanoidSMPLIMVis.test_step) at 8192 envs and 1000 motions, two
loops:

  meters: the graphed step with b200_motion_stats;
  pose:   with b200_motion_stats and b200_pose_metrics (the same launch with the pose fields: a Jacobi eigen-solve per env per step).
The meters take no stop flag here, so they accumulate and fold every step whatever env 0's episode does.  Alternating rounds of
--steps steps each; prints the median (min - max) ms per step of each loop with the card's name and power limit read in the same run,
and one JSON line.

    python tools/perf_im_pose_metrics.py [--envs 8192] [--motions 1000] [--steps 64] [--rounds 7]"""
import argparse
import json
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from perf_im_record import card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=8192)
    ap.add_argument("--motions", type=int, default=1000)
    ap.add_argument("--steps", type=int, default=64)
    ap.add_argument("--rounds", type=int, default=7)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("perf_im_pose_metrics needs a CUDA device")
    from vid2player3d_b200 import model_compiler, motion_lib
    from vid2player3d_b200.configs import SIM_PARAMS, im_cfg
    from vid2player3d_b200.tasks import HumanoidSMPLIMVis
    N = a.envs
    model = model_compiler.load_compiled("smpl_mesh_humanoid_amass_v1")
    flat = motion_lib.synthetic(model, num_motions=a.motions, num_frames=90, seed=1)
    g = torch.Generator().manual_seed(0)
    dims = (734, 1024, 1024, 512, 75)
    layers = [((torch.rand(dims[i + 1], dims[i], generator=g) * 2 - 1) / dims[i] ** 0.5 * (0.1 if i == 3 else 1.0),
               torch.zeros(dims[i + 1])) for i in range(4)]
    net = dict(layers=layers, mean=torch.zeros(734), rstd=torch.ones(734), clip=5.0)
    tasks = {}
    for name, over in (("meters", dict(b200_motion_stats=True)), ("pose", dict(b200_motion_stats=True, b200_pose_metrics=True))):
        torch.manual_seed(0)
        t = HumanoidSMPLIMVis(im_cfg(N, flat, stateInit="Start", sample_first_motions=True, **over), SIM_PARAMS, 1, "cuda", 0, True)
        t.set_policy(net, clip_obs=5.0, clip_actions=1.0)
        # no stop flag: the meters run every step
        t._motion_stats_launch = (lambda f: lambda games=None: f(None))(t._motion_stats_launch)
        tasks[name] = t

    def round_(name, steps):
        t = tasks[name]
        t.reset()
        for k in ("cr", "steps", "prev_dones", "step", "games"):
            t._stats[k].zero_()
        t.clear_motion_stats_games()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for n in range(steps):
            t.test_step(n)
            if (n + 1) % t.context_length == 0:
                t._stats["games"].tolist()
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) / steps * 1e3

    names = ("meters", "pose")
    for k in names:
        round_(k, 40)
    res = {k: [] for k in names}
    for _ in range(a.rounds):
        for k in names:
            res[k].append(round_(k, a.steps))
    c = card()
    med = {k: sorted(v)[len(v) // 2] for k, v in res.items()}
    games = int(tasks["pose"]._ms["counts"][:, 0].sum())
    print(f"{c}; {N} envs, {a.motions} motions, {a.rounds} alternating rounds of {a.steps} steps ({games} games folded)")
    for k in names:
        print(f"  {k:6s}: {med[k]:.3f} ms per step (min {min(res[k]):.3f}, max {max(res[k]):.3f})")
    print(json.dumps({"card": c, "envs": N, "motions": a.motions, "steps": a.steps, "rounds": a.rounds, "ms_per_step": res,
                      "median": med, "games_folded": games}))


if __name__ == "__main__":
    main()
