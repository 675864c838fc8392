"""Cost of the training resample of HumanoidSMPLIM (cfg.env.b200_resample_motions, b200_hard_motion_share) at 8192 envs:

  step:     ms per rollout step (the step graph + reset_done, the reset graph) on a synthetic library of 11 000 45-frame motions, so
            games end often, under uniform random actions, in four arms:
              off:        without the key;
              h0:         the resample from the base distribution;
              h0.5:       half of the draws weighted by the failure rates (pre_epoch rebuilds every 32 steps of the warm-up; the
                          rebuild is timed on its own below);
              h0.5-1024:  h0.5 with motion m on one of 1024 distinct scaled bodies (b200env_set_env_assets in the reset graph);
  rebuild:  b200env_motion_weights alone at M = 11 000 and 100 000 (CUDA events around 200 launches);
  coverage: the distinct motions played in 1000 steps, off and h0.5.
Alternating rounds; prints the median (min - max) of each with the card's name, power limit and max SM clock read in the same run, and
one JSON line.

    python tools/perf_im_resample.py [--envs 8192] [--rounds 3] [--steps 64] [--motions 11000]"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from perf_im_motion_queue_assets import scaled  # noqa: E402
from perf_im_record import card  # noqa: E402


def med(v):
    return float(np.median(v))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=8192)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=64)
    ap.add_argument("--motions", type=int, default=11000)
    ap.add_argument("--coverage-steps", type=int, default=1000)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("perf_im_resample needs a CUDA device")
    from vid2player3d_b200 import model_compiler, motion_lib, native
    from vid2player3d_b200.configs import SIM_PARAMS, im_cfg
    from vid2player3d_b200.tasks import HumanoidSMPLIM
    from vid2player3d_b200.tasks.vec_task import VecTaskPythonWrapper
    N, M, dev = a.envs, a.motions, "cuda:0"
    base = model_compiler.load_compiled("smpl_mesh_humanoid_amass_v1")
    flat = motion_lib.synthetic(base, num_motions=M, num_frames=45, seed=3)
    bodies = [scaled(base, 0.85 + 0.3 * k / 1023) for k in range(1024)]
    arms = {"off": {}, "h0": dict(b200_resample_motions=True), "h0.5": dict(b200_resample_motions=True, b200_hard_motion_share=0.5),
            "h0.5-1024": dict(b200_resample_motions=True, b200_hard_motion_share=0.5, motion_assets=[bodies[m % 1024] for m in range(M)])}
    g = torch.Generator(device=dev).manual_seed(5)
    acts = [torch.rand(N, 75, device=dev, generator=g) * 2 - 1 for _ in range(16)]

    def make(over):
        cfg = im_cfg(N, flat, stateInit="Random", terminationBodyHeight=0.3, contactBodies=["R_Ankle", "L_Ankle", "R_Toe", "L_Toe"],
                     **over)
        cfg["seed"] = 10
        torch.manual_seed(0)
        t = HumanoidSMPLIM(cfg, SIM_PARAMS, 1, "cuda", 0, True)
        w = VecTaskPythonWrapper(t, t.device)
        w.enable_cuda_graph(reset_graph=True)
        w.reset()
        return t, w

    def run(t, w, steps, i0=0, played=None, epochs=True):
        resets = torch.zeros((), dtype=torch.long, device=dev)
        for i in range(i0, i0 + steps):
            w.step(acts[i % len(acts)])
            resets += t.reset_buf.sum()
            if played is not None:
                played[t._reset_ref_motion_ids] = True
            w.reset_done()
            if epochs and i % 32 == 31:
                t.pre_epoch(i // 32)
        return resets

    tasks = {k: make(v) for k, v in arms.items()}
    for t, w in tasks.values():                              # warm-up: games under way in every arm
        run(t, w, 64)
    torch.cuda.synchronize()
    step_ms, games = {k: [] for k in arms}, {k: 0 for k in arms}
    for r in range(a.rounds):
        for k, (t, w) in tasks.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            res = run(t, w, a.steps, i0=64 + r * a.steps, epochs=False)
            e1.record()
            torch.cuda.synchronize()
            step_ms[k].append(e0.elapsed_time(e1) / a.steps)
            games[k] += int(res)
    rebuild_us = {}
    for m in (M, 100000):
        rng = np.random.default_rng(m)
        f = lambda x, dt: torch.from_numpy(np.ascontiguousarray(x)).to(dev, dt)  # noqa: E731
        tries = f(rng.integers(0, 3, m), torch.int64)
        t = dict(base=f(rng.uniform(0.5, 3.0, m), torch.float32), tries=tries, fails=torch.zeros_like(tries), rate=torch.ones(m, device=dev,
                 dtype=torch.float64), cdf=torch.zeros(m, device=dev, dtype=torch.float64))
        for _ in range(5):
            native.motion_weights(dict(num_motions=m, h=0.5), t)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(200):
            native.motion_weights(dict(num_motions=m, h=0.5), t)
        e1.record()
        torch.cuda.synchronize()
        rebuild_us[m] = e0.elapsed_time(e1) / 200 * 1000.0
    coverage = {}
    for k in ("off", "h0.5"):
        t, w = tasks[k]
        played = torch.zeros(M, dtype=torch.bool, device=dev)
        run(t, w, a.coverage_steps, played=played)
        coverage[k] = int(played.sum())
    c = card()
    print(f"card: {c}")
    print(f"{N} envs, {M} 45-frame motions, {a.rounds} alternating rounds of {a.steps} steps, ms per step (step graph + reset_done), "
          f"median (min - max):")
    for k, v in step_ms.items():
        print(f"  {k:10s} {med(v):.3f} ({min(v):.3f} - {max(v):.3f})  games ended in the windows: {games[k]}")
    for m, us in rebuild_us.items():
        print(f"pre_epoch rebuild (b200env_motion_weights) at M = {m}: {us:.1f} us")
    print(f"distinct motions played in {a.coverage_steps} steps: off {coverage['off']}, h0.5 {coverage['h0.5']} of {M}")
    print(json.dumps({"card": c, "envs": N, "motions": M, "rounds": a.rounds, "step_ms": step_ms,
                      "step_median": {k: med(v) for k, v in step_ms.items()}, "games": games, "rebuild_us": rebuild_us,
                      "coverage": coverage}))


if __name__ == "__main__":
    main()
