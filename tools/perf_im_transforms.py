"""Per-step cost of an embodied_pose rollout that resets its finished envs with the context window's transforms (cfg.env.
transform_specs: noisy_joints + mask_random_joints), config-4 style as tools/perf_im_reset.py (HumanoidSMPLIM on the djokovic asset,
synthetic MoCap 64 x 300 frames, 8192 envs, random policy U(-1, 1), so envs fall and reset every step), three ways:

    graph+ids          the step graph; nonzero + task.reset(ids), the transforms in torch on the reset rows (without the opt-in)
    graph+reset_done   the step graph; reset_done() replaying the masked-reset graph, the transforms in the window launch
                       (cfg.env.b200_device_transforms)
    graph+reset_done, no transforms   the same without transform_specs (the masked reset as tools/perf_im_reset.py times it)

    python tools/perf_im_transforms.py [--envs 8192] [--steps 64] [--warmup 16] [--reps 5]

Every step sits between two CUDA events with the L2 flushed by a 256 MiB memset before it, outside the pair; the variants alternate
over the repetitions in one process.  Prints one JSON line per measurement, then the median (min-max) of each variant."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from perf_im_reset import card, measure  # noqa: E402

SPECS = {"noisy_joints": {"prob": 0.5, "noise_std": 0.05, "conf_std": 0.04, "min_conf": 0.3}, "mask_random_joints": {"prob": 0.1}}
VARIANTS = ("graph+ids", "graph+reset_done", "graph+reset_done, no transforms")


def make(envs, variant):
    import torch
    from vid2player3d_b200 import model_compiler, motion_lib
    from vid2player3d_b200.configs import SIM_PARAMS, im_cfg
    from vid2player3d_b200.tasks import HumanoidSMPLIM
    from vid2player3d_b200.tasks.vec_task import VecTaskPythonWrapper
    flat = motion_lib.synthetic(model_compiler.load_compiled("smpl_mesh_humanoid_amass_v1"), num_motions=64, num_frames=300, seed=7, sigma=0.05)
    over = {} if variant.endswith("no transforms") else dict(transform_specs=SPECS)
    if variant.startswith("graph+reset_done") and over:
        over["b200_device_transforms"] = True
    torch.manual_seed(7)
    task = HumanoidSMPLIM(im_cfg(envs, flat, episodeLength=300, asset="mjcf/smpl_mesh_humanoid_djokovic.xml", **over), SIM_PARAMS, 1,
                          "cuda", 0, True)
    w = VecTaskPythonWrapper(task, task.device)
    w.enable_cuda_graph(reset_graph=variant.startswith("graph+reset_done"))
    assert (task._reset_graph is not None) == variant.startswith("graph+reset_done")
    task.reset()
    resets = torch.zeros((), dtype=torch.long, device=task.device)

    def step(a):
        w.step(a)
        resets.add_(task.reset_buf.sum())
        if variant.startswith("graph+reset_done"):
            w.reset_done()
        else:
            task.reset(task.reset_buf.nonzero(as_tuple=False).flatten())
    return step, resets


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--envs", type=int, default=8192)
    p.add_argument("--steps", type=int, default=64)
    p.add_argument("--warmup", type=int, default=16)
    p.add_argument("--reps", type=int, default=5, help="alternating repetitions of the variants")
    args = p.parse_args()
    import numpy as np
    import torch
    assert torch.cuda.is_available(), "perf_im_transforms.py needs a CUDA device"
    name, clocks = card()
    print(f"# {name}; power limit, SM clock, max SM clock: {clocks}", flush=True)
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device="cuda:0")
    gen = torch.Generator(device="cuda:0").manual_seed(100)
    fns = {v: make(args.envs, v) for v in VARIANTS}
    pool = [torch.rand(args.envs, 75, device="cuda:0", generator=gen) * 2 - 1 for _ in range(16)]
    res = {v: [] for v in VARIANTS}
    for rep in range(args.reps):
        for v in (VARIANTS if rep % 2 == 0 else VARIANTS[::-1]):
            ms, rps = measure(*fns[v], pool, args.steps, args.warmup, flush)
            res[v].append((ms, rps))
            print(json.dumps({"variant": v, "rep": rep, "ms_per_step": ms, "resets_per_step": rps, "envs": args.envs, "device": name,
                              "clocks": clocks}), flush=True)
    print(f"\n{name}, power limit / SM clock / max SM clock {clocks}; {args.envs} envs, median (min-max) of {args.reps} alternating "
          f"runs of {args.steps} steps")
    print(f"{'variant':>32} {'ms/step':>24} {'resets/step':>12}")
    for v in VARIANTS:
        a = np.array(res[v])
        print(f"{v:>32} {np.median(a[:, 0]):>8.4f} ({a[:, 0].min():.4f}-{a[:, 0].max():.4f}) {np.median(a[:, 1]):>12.1f}")


if __name__ == "__main__":
    main()
