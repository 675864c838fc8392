"""Cost of several assets in one physics launch (b200env_create_assets) at 8192 amass_im envs (config 2: HumanoidSMPLIM on amass_v1):
S scaled variants of amass_v1, assigned to the envs uniformly at random through cfg.env.motion_assets (one variant per motion of an
S-motion library), each measured next to the single-asset handle on the same library, alternating, in one process.

    python tools/perf_assets.py [--envs 8192] [--assets 1,2,8,64,256] [--steps 30] [--warmup 8] [--reps 3]

Physics launch: an event pair around it (set_kernel_timing / kernel_ms), the L2 flushed by a 256 MiB memset before every step, as
tools/perf_rounds.py.  Full step: host clock over `steps` steps (step + reset of the flagged envs) ending in a device synchronise.
One JSON line per measurement, then a table of medians over the repetitions."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def variant(model, s):
    """amass_v1 scaled by s: lengths, COMs, vertices, radii x s, mass x s^3, inertia x s^5"""
    m = dict(model)
    for k in ("offset", "com", "dyn_com", "verts", "radius"):
        m[k] = model[k] * s
    for k in ("mass", "dyn_mass"):
        m[k] = model[k] * s ** 3
    for k in ("inertia", "dyn_inertia"):
        m[k] = model[k] * s ** 5
    return m


def make_task(envs, S, multi):
    import torch
    from vid2player3d_b200 import model_compiler, motion_lib
    from vid2player3d_b200.configs import SIM_PARAMS, im_cfg
    from vid2player3d_b200.tasks import HumanoidSMPLIM
    base = model_compiler.load_compiled("smpl_mesh_humanoid_amass_v1")
    flat = motion_lib.synthetic(base, num_motions=S, num_frames=120, seed=1)
    cfg = im_cfg(envs, flat)
    if multi:
        cfg["env"]["motion_assets"] = [variant(base, 0.9 + 0.2 * i / max(S - 1, 1)) if S > 1 else base for i in range(S)]
    torch.manual_seed(0)
    t = HumanoidSMPLIM(cfg, SIM_PARAMS, 1, "cuda", 0, True)
    t.reset()
    return t


def measure(t, steps, warmup, flush, pool):
    import torch

    def step(i):
        t.step(pool[i % len(pool)])
        t.reset(t.reset_buf.nonzero(as_tuple=False).flatten())
    for i in range(warmup):
        step(i)
    torch.cuda.synchronize()
    t._env.set_kernel_timing(True)
    t._env.kernel_ms()
    for i in range(steps):
        flush.zero_()
        step(warmup + i)
    ms, n = t._env.kernel_ms()
    t._env.set_kernel_timing(False)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for i in range(steps):
        step(warmup + steps + i)
    torch.cuda.synchronize()
    return ms, n, (time.perf_counter() - t0) * 1e3 / steps


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"], capture_output=True,
                           text=True, timeout=30)
        return name, r.stdout.strip() or "unknown"
    except Exception as ex:
        return name, f"unknown ({ex!r:.60})"


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--envs", type=int, default=8192)
    p.add_argument("--assets", default="1,2,8,64,256", help="comma list of variant counts S")
    p.add_argument("--steps", type=int, default=30)
    p.add_argument("--warmup", type=int, default=8)
    p.add_argument("--reps", type=int, default=3, help="alternating repetitions of (several assets, one asset)")
    args = p.parse_args()
    import numpy as np
    import torch
    assert torch.cuda.is_available(), "perf_assets.py needs a CUDA device"
    name, power = card()
    print(f"# {name}; power limit, max SM clock: {power}", flush=True)
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device="cuda:0")
    gen = torch.Generator(device="cuda:0").manual_seed(100)
    pool = [torch.rand(args.envs, 75, device="cuda:0", generator=gen) * 2 - 1 for _ in range(16)]
    table = []
    for S in [int(x) for x in args.assets.split(",")]:
        tasks = {"assets": make_task(args.envs, S, True), "single": make_task(args.envs, S, False)}
        B, G = tasks["single"]._env.physics_launch_shape
        na, _, batches = tasks["assets"]._env.asset_plan
        shape = {"assets": (len(batches), -(-len(batches) // G)), "single": (-(-args.envs // B), -(-(-(-args.envs // B)) // G))}
        res = {k: [] for k in tasks}
        for rep in range(args.reps):
            for k in (("assets", "single") if rep % 2 == 0 else ("single", "assets")):
                ms, n, step_ms = measure(tasks[k], args.steps, args.warmup, flush, pool)
                res[k].append((ms, step_ms))
                print(json.dumps({"S": S, "handle": k, "distinct_assets": na if k == "assets" else 1, "batches": shape[k][0],
                                  "rounds": shape[k][1], "grid": G, "physics_launch_ms": ms, "launches_timed": n, "step_ms": step_ms,
                                  "env_steps_per_s": args.envs / step_ms * 1e3, "device": name, "power_limit": power}), flush=True)
        for k in tasks:
            a = np.array(res[k])
            table.append((S, k, shape[k][0], shape[k][1], float(np.median(a[:, 0])), float(np.median(a[:, 1])),
                          float(a[:, 0].max() - a[:, 0].min())))
        del tasks
        torch.cuda.empty_cache()
    print(f"\n{name}, power limit / max SM clock {power}; {args.envs} envs, medians of {args.reps} alternating runs")
    print(f"{'S':>4} {'handle':>7} {'batches':>8} {'rounds':>7} {'launch ms':>10} {'spread':>7} {'step ms':>8} {'M env-steps/s':>14}")
    for S, k, nb, r, ms, st, spread in table:
        print(f"{S:>4} {k:>7} {nb:>8} {r:>7} {ms:>10.4f} {spread:>7.4f} {st:>8.4f} {args.envs / st / 1e3:>14.3f}")


if __name__ == "__main__":
    main()
