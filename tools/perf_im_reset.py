"""Per-step cost of resetting the finished envs of an embodied_pose rollout (config-4 style: HumanoidSMPLIM on the djokovic asset,
synthetic MoCap 64 x 300 frames, 8192 envs, random policy U(-1, 1), so envs fall and reset every step), three ways:

    eager+ids         task.step(a); ids = reset_buf.nonzero(); task.reset(ids)      (the rl_games loop; bench.py's PPO leg)
    graph+ids         the step graph (VecTaskPython.enable_cuda_graph); nonzero + task.reset(ids)
    graph+reset_done  the step graph; VecTaskPythonWrapper.reset_done() replaying the masked-reset graph

    python tools/perf_im_reset.py [--envs 8192] [--steps 64] [--warmup 16] [--reps 3]

Every step sits between two CUDA events with the L2 flushed by a 256 MiB memset before it, outside the pair (as bench.py's
timed_steps); the variants alternate over the repetitions in one process.  Prints one JSON line per measurement, then the medians."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

VARIANTS = ("eager+ids", "graph+ids", "graph+reset_done")


def make(envs, variant):
    import torch
    from vid2player3d_b200 import model_compiler, motion_lib
    from vid2player3d_b200.configs import SIM_PARAMS, im_cfg
    from vid2player3d_b200.tasks import HumanoidSMPLIM
    from vid2player3d_b200.tasks.vec_task import VecTaskPythonWrapper
    flat = motion_lib.synthetic(model_compiler.load_compiled("smpl_mesh_humanoid_amass_v1"), num_motions=64, num_frames=300, seed=7, sigma=0.05)
    torch.manual_seed(7)
    task = HumanoidSMPLIM(im_cfg(envs, flat, episodeLength=300, asset="mjcf/smpl_mesh_humanoid_djokovic.xml"), SIM_PARAMS, 1, "cuda", 0, True)
    w = VecTaskPythonWrapper(task, task.device)
    if variant != "eager+ids":
        w.enable_cuda_graph(reset_graph=variant == "graph+reset_done")
    task.reset()
    resets = torch.zeros((), dtype=torch.long, device=task.device)

    def step(a):
        if variant == "eager+ids":
            task.step(torch.clamp(a, -1.0, 1.0))
        else:
            w.step(a)
        resets.add_(task.reset_buf.sum())
        if variant == "graph+reset_done":
            w.reset_done()
        else:
            task.reset(task.reset_buf.nonzero(as_tuple=False).flatten())
    return step, resets


def measure(step, resets, pool, steps, warmup, flush):
    import torch
    for i in range(warmup):
        step(pool[i % len(pool)])
    torch.cuda.synchronize()
    resets.zero_()
    evs = []
    for i in range(steps):
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        step(pool[(warmup + i) % len(pool)])
        e1.record()
        evs.append((e0, e1))
    torch.cuda.synchronize()
    return sum(a.elapsed_time(b) for a, b in evs) / steps, int(resets) / steps


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        return name, r.stdout.strip() or "unknown"
    except Exception as ex:
        return name, f"unknown ({ex!r:.60})"


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--envs", type=int, default=8192)
    p.add_argument("--steps", type=int, default=64)
    p.add_argument("--warmup", type=int, default=16)
    p.add_argument("--reps", type=int, default=3, help="alternating repetitions of the three variants")
    args = p.parse_args()
    import numpy as np
    import torch
    assert torch.cuda.is_available(), "perf_im_reset.py needs a CUDA device"
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
    print(f"\n{name}, power limit / SM clock / max SM clock {clocks}; {args.envs} envs, medians of {args.reps} alternating runs of "
          f"{args.steps} steps")
    print(f"{'variant':>18} {'ms/step':>8} {'spread':>7} {'resets/step':>12}")
    for v in VARIANTS:
        a = np.array(res[v])
        print(f"{v:>18} {np.median(a[:, 0]):>8.4f} {a[:, 0].max() - a[:, 0].min():>7.4f} {np.median(a[:, 1]):>12.1f}")


if __name__ == "__main__":
    main()
