"""Cost of several assets in one physics launch (b200env_create_assets) at 8192 amass_im envs (config 2: HumanoidSMPLIM on amass_v1):
S scaled variants of amass_v1, assigned to the envs uniformly at random through cfg.env.motion_assets (one variant per motion of an
S-motion library).  For each S three handles are measured, alternating, in one process: the grouped plan and the mixed plan of the
several-asset handle (B200ENV_ASSET_PLAN at create) and the single-asset handle on the same library.  "rule" says which of the two
plans b200env_create_assets picks for that S by itself.

    python tools/perf_assets.py [--envs 8192] [--assets 1,64,256,1024,8192] [--steps 30] [--warmup 8] [--reps 3]

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


def make_task(envs, S, multi, plan=None):
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
    if plan:
        os.environ["B200ENV_ASSET_PLAN"] = plan
    try:
        t = HumanoidSMPLIM(cfg, SIM_PARAMS, 1, "cuda", 0, True)
    finally:
        os.environ.pop("B200ENV_ASSET_PLAN", None)
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
    p.add_argument("--assets", default="1,64,256,1024,8192", help="comma list of variant counts S")
    p.add_argument("--steps", type=int, default=30)
    p.add_argument("--warmup", type=int, default=8)
    p.add_argument("--reps", type=int, default=3, help="alternating repetitions of (grouped, mixed, one asset)")
    args = p.parse_args()
    import numpy as np
    import torch
    from vid2player3d_b200 import native
    assert torch.cuda.is_available(), "perf_assets.py needs a CUDA device"
    name, power = card()
    print(f"# {name}; power limit, max SM clock: {power}", flush=True)
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device="cuda:0")
    gen = torch.Generator(device="cuda:0").manual_seed(100)
    pool = [torch.rand(args.envs, 75, device="cuda:0", generator=gen) * 2 - 1 for _ in range(16)]
    table = []
    for S in [int(x) for x in args.assets.split(",")]:
        tasks = {"grouped": make_task(args.envs, S, True, "grouped"), "mixed": make_task(args.envs, S, True, "mixed"),
                 "single": make_task(args.envs, S, False)}
        B, G = tasks["single"]._env.physics_launch_shape
        assert tasks["mixed"]._env.asset_plan_mixed and not tasks["grouped"]._env.asset_plan_mixed
        shape, na = {}, {"single": 1}
        for k in ("grouped", "mixed"):
            na[k], _, batches = tasks[k]._env.asset_plan
            shape[k] = (len(batches), -(-len(batches) // G))
        shape["single"] = (-(-args.envs // B), -(-(-(-args.envs // B)) // G))
        rule = "mixed" if native.choose_asset_plan(tasks["grouped"]._env_asset, na["grouped"], G) else "grouped"
        res = {k: [] for k in tasks}
        order = list(tasks)
        for rep in range(args.reps):
            for k in order[rep % 3:] + order[:rep % 3]:
                ms, n, step_ms = measure(tasks[k], args.steps, args.warmup, flush, pool)
                res[k].append((ms, step_ms))
                print(json.dumps({"S": S, "handle": k, "distinct_assets": na[k], "batches": shape[k][0], "rounds": shape[k][1], "grid": G,
                                  "rule": rule, "physics_launch_ms": ms, "launches_timed": n, "step_ms": step_ms,
                                  "env_steps_per_s": args.envs / step_ms * 1e3, "device": name, "power_limit": power}), flush=True)
        for k in tasks:
            a = np.array(res[k])
            table.append((S, k, rule, shape[k][0], shape[k][1], float(np.median(a[:, 0])), float(np.median(a[:, 1])),
                          float(a[:, 0].max() - a[:, 0].min())))
        del tasks
        torch.cuda.empty_cache()
    print(f"\n{name}, power limit / max SM clock {power}; {args.envs} envs, medians of {args.reps} alternating runs")
    print(f"{'S':>5} {'handle':>7} {'rule':>7} {'batches':>8} {'rounds':>7} {'launch ms':>10} {'spread':>7} {'ms/round':>9} {'step ms':>8} "
          f"{'M env-steps/s':>14}")
    for S, k, rule, nb, r, ms, st, spread in table:
        print(f"{S:>5} {k:>7} {rule:>7} {nb:>8} {r:>7} {ms:>10.4f} {spread:>7.4f} {ms / r:>9.4f} {st:>8.4f} {args.envs / st / 1e3:>14.3f}")


if __name__ == "__main__":
    main()
