"""Cost of the DOF force sensor: the physics launch alone at 8192 envs with cfg.env.dof_force_sensors off and on, alternating in one
process, for the imitation task (HumanoidSMPLIM, amass_v1 body) and the tennis player (HumanoidSMPLIMMVAE, federer + racket + ball).

    python tools/perf_dof_force.py [--envs 8192] [--steps 30] [--warmup 8] [--reps 3] [--out perf_dof_force.json]

Timing as tools/perf_rounds.py: eager steps with a CUDA event pair around the physics launch (set_kernel_timing / kernel_ms), the L2
flushed by a 256 MiB memset before every step.  Prints one JSON line per (workload, sensor, rep), then the medians, the card's name and
its power limit; --out also writes them to a file."""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(ROOT))
sys.path.insert(0, os.path.join(os.path.dirname(ROOT), "tests"))


def make_task(wl, n, sensors):
    import torch
    from vid2player3d_b200 import ball as ball_data, model_compiler, motion_lib
    from vid2player3d_b200.configs import SIM_PARAMS, im_cfg, v2p_cfg
    from vid2player3d_b200.tasks import HumanoidSMPLIM, HumanoidSMPLIMMVAE
    torch.manual_seed(0)
    if wl == "humanoid":
        flat = motion_lib.synthetic(model_compiler.load_compiled("smpl_mesh_humanoid_amass_v1"), num_motions=4, num_frames=60, seed=1)
        cfg = im_cfg(n, flat)
        cfg["env"]["dof_force_sensors"] = sensors
        t = HumanoidSMPLIM(cfg, SIM_PARAMS, 1, "cuda", 0, True)
        t.reset()
        return t
    v2p = dict(v2p_cfg(n)["env"]["vid2player"], ball_pool=ball_data.synthetic_pool(2048, seed=10, spin_scale=5))
    cfg = {"env": dict(numEnvs=n, episodeLength=300, residual_force_scale=31.85, is_train=True,
                       asset=dict(assetFileName="smpl_mesh_humanoid_federer.xml"),
                       plane=dict(staticFriction=1.0, dynamicFriction=1.0, restitution=0.5), vid2player=v2p, keyBodies=[], contactBodies=[],
                       dof_force_sensors=sensors),
           "sim": {"substeps": 6}}
    return HumanoidSMPLIMMVAE(cfg, SIM_PARAMS, 1, "cuda", 0, True)


def measure(task, steps, warmup, flush, seed):
    import torch
    n = task.num_envs
    gen = torch.Generator(device="cuda").manual_seed(seed)
    pool = [(torch.rand(n, task.get_action_size(), device="cuda", generator=gen) * 2 - 1).contiguous() for _ in range(8)]
    for i in range(warmup):
        task.step(pool[i % len(pool)])
    torch.cuda.synchronize()
    task._env.set_kernel_timing(True)
    task._env.kernel_ms()
    for i in range(steps):
        flush.zero_()
        task.step(pool[i % len(pool)])
    ms, k = task._env.kernel_ms()
    task._env.set_kernel_timing(False)
    torch.cuda.synchronize()
    assert k == steps
    return ms


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--envs", type=int, default=8192)
    p.add_argument("--steps", type=int, default=30)
    p.add_argument("--warmup", type=int, default=8)
    p.add_argument("--reps", type=int, default=3)
    p.add_argument("--workloads", default="humanoid,ball")
    p.add_argument("--out", default=None)
    a = p.parse_args()
    import torch
    assert torch.cuda.is_available(), "perf_dof_force.py needs a CUDA device"
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device="cuda")
    result = {"card": card(), "envs": a.envs, "steps": a.steps, "reps": a.reps, "workloads": {}}
    for wl in a.workloads.split(","):
        tasks = {s: make_task(wl, a.envs, s) for s in (False, True)}
        times = {False: [], True: []}
        for rep in range(a.reps):
            for s in ((False, True) if rep % 2 == 0 else (True, False)):
                ms = measure(tasks[s], a.steps, a.warmup, flush, seed=100 + rep)
                times[s].append(ms)
                print(json.dumps({"workload": wl, "sensor": s, "rep": rep, "physics_launch_ms": round(ms, 4)}), flush=True)
        off, on = statistics.median(times[False]), statistics.median(times[True])
        result["workloads"][wl] = {"off_ms": times[False], "on_ms": times[True], "median_off_ms": off, "median_on_ms": on,
                                   "ratio": on / off}
        del tasks
        torch.cuda.empty_cache()
    print(json.dumps(result))
    for wl, r in result["workloads"].items():
        print(f"{wl}: physics launch {r['median_off_ms']:.4f} ms sensor off, {r['median_on_ms']:.4f} ms on ({100 * (r['ratio'] - 1):+.1f} %), "
              f"spread off {max(r['off_ms']) - min(r['off_ms']):.4f} / on {max(r['on_ms']) - min(r['on_ms']):.4f} ms; {result['card']}")
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
