"""The physics launch alone over a list of env counts of the primary workload (config 3: federer humanoid + racket + ball, decoder +
policy MLP inside the step), to show the staircase of a persistent launch: with one CTA of B envs per SM on S SMs, the launch
takes ceil(envs / (B * S)) rounds of batches and costs about one round's time per round.

    python tools/perf_rounds.py [--envs 3696,4224,7392,8192,8448] [--steps 20] [--warmup 8]

Timing as bench.py's dominant_kernel: the step runs eagerly with an event pair around the physics launch (set_kernel_timing /
kernel_ms), the L2 flushed by a 256 MiB memset before every step.  One JSON line per env count, then a table."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def measure(envs, steps, warmup):
    import torch
    from bench import federer_env
    env = federer_env(envs, 0, seed=10)
    task = env._physics_player.task
    gen = torch.Generator(device=env.device).manual_seed(100)
    pool = [torch.clamp(torch.randn(envs, env.num_actions, device=env.device, generator=gen), -5, 5) for _ in range(16)]
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=env.device)

    def step(i):
        env.step(pool[i % len(pool)])
        env.reset(env.reset_buf.nonzero(as_tuple=False).flatten())
    for i in range(warmup):
        step(i)
    torch.cuda.synchronize()
    task._env.set_kernel_timing(True)
    task._env.kernel_ms()   # drop anything recorded so far
    for i in range(steps):
        flush.zero_()
        step(warmup + i)
    ms, n = task._env.kernel_ms()
    task._env.set_kernel_timing(False)
    torch.cuda.synchronize()
    del env, task, pool, flush
    torch.cuda.empty_cache()
    return ms, n


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--envs", default="3696,4224,7392,8192,8448", help="comma list of env counts")
    p.add_argument("--steps", type=int, default=20, help="timed steps per env count")
    p.add_argument("--warmup", type=int, default=8)
    args = p.parse_args()
    import torch
    assert torch.cuda.is_available(), "perf_rounds.py needs a CUDA device"
    prop = torch.cuda.get_device_properties(0)
    lib = os.environ.get("B200ENV_LIB", "default")
    rows = []
    for n in [int(x) for x in args.envs.split(",")]:
        ms, k = measure(n, args.steps, args.warmup)
        rows.append((n, ms))
        print(json.dumps({"envs": n, "physics_launch_ms": ms, "launches_timed": k, "us_per_env": ms * 1e3 / n, "lib": lib,
                          "device": prop.name, "sms": prop.multi_processor_count}), flush=True)
    print(f"{prop.name}, {prop.multi_processor_count} SMs, lib {lib}")
    print(f"{'envs':>7} {'launch ms':>10} {'us/env':>8} {'x first':>8}")
    for n, ms in rows:
        print(f"{n:>7} {ms:>10.4f} {ms * 1e3 / n:>8.4f} {ms / rows[0][1]:>8.2f}")


if __name__ == "__main__":
    main()
