"""Cost of the motion queue with a body per motion (HumanoidSMPLIMVis, cfg.env.b200_motion_queue with motion_assets) at 8192 envs:

  step:    the graphed test step on 45-frame motions, so games end and envs restart all through the timed window, in three forms:
             queue-1:      the queue on one body;
             queue-S:      the queue with S distinct scaled bodies (motion m on body m % S), envs changing body as their games end
                           (b200env_set_env_assets every step);
             fixed-S:      the same S bodies on a handle whose assignment is fixed at creation (mixed plan), without the queue.
  library: a 32768-motion library, motion m on one of 1024 distinct scaled bodies: the host time to resolve the per-motion asset list,
           the task's create time, the device memory of a handle of 1024 bodies and of one body, the wall time of
           run_test until every motion has been scored (against the same library on one body), and the launch b200env_set_env_assets
           alone (CUDA events around replays of a graph of 200 launches).
Alternating rounds; prints the median (min - max) of each with the card's name, power limit and max SM clock read in the same run, and
one JSON line.

    python tools/perf_im_motion_queue_assets.py [--envs 8192] [--rounds 3] [--steps 64] [--bodies 64,256,1024]"""
import argparse
import contextlib
import io
import json
import os
import sys
import tempfile
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from perf_im_record import card  # noqa: E402


def scaled(model, s):
    """the asset scaled by s (lengths, COMs, vertices x s, mass x s^3, inertia x s^5), as tests/test_gpu_assets.py builds them"""
    m = dict(model)
    for k in ("offset", "com", "dyn_com", "verts", "radius"):
        m[k] = model[k] * s
    for k in ("mass", "dyn_mass"):
        m[k] = model[k] * s ** 3
    for k in ("inertia", "dyn_inertia"):
        m[k] = model[k] * s ** 5
    if len(model["prims"]):
        m["prims"] = model["prims"].copy()
        m["prims"][:, 1:8] *= s
    return m


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=8192)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=64)
    ap.add_argument("--bodies", default="64,256,1024")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("perf_im_motion_queue_assets needs a CUDA device")
    import numpy as np
    from vid2player3d_b200 import model_compiler, motion_lib
    from vid2player3d_b200.configs import SIM_PARAMS, im_cfg
    from vid2player3d_b200.tasks import HumanoidSMPLIMVis
    N, S_list = a.envs, [int(s) for s in a.bodies.split(",")]
    model = model_compiler.load_compiled("smpl_mesh_humanoid_amass_v1")
    base = motion_lib.synthetic(model, num_motions=1024, num_frames=45, seed=1)
    lib4k = motion_lib.FlatMotionLib.merge([base] * 4)
    lib32k = motion_lib.FlatMotionLib.merge([lib4k] * 8)
    bodies = [scaled(model, 0.85 + 0.3 * i / (max(S_list) - 1)) for i in range(max(S_list))]
    g = torch.Generator().manual_seed(0)
    dims = (734, 1024, 1024, 512, 75)
    layers = [((torch.rand(dims[i + 1], dims[i], generator=g) * 2 - 1) / dims[i] ** 0.5 * (0.1 if i == 3 else 1.0),
               torch.zeros(dims[i + 1])) for i in range(4)]
    net = dict(layers=layers, mean=torch.zeros(734), rstd=torch.ones(734), clip=5.0)
    tmp = tempfile.mkdtemp()

    def task(flat, S=None, **over):
        """S: motion m on body m % S (None: one body)"""
        if S is not None:
            entries = [bodies[m % S] for m in range(flat.num_motions())]
            over = dict(over, motion_assets=entries, test_motion_assets=entries)
        torch.manual_seed(0)
        cfg = im_cfg(N, flat, stateInit="Start", b200_motion_stats=True, b200_motion_stats_file=os.path.join(tmp, "ms.npz"), **over)
        return HumanoidSMPLIMVis(cfg, SIM_PARAMS, 1, "cuda", 0, True)

    # ---- the step, with games ending and restarting in the window
    qover = dict(b200_motion_queue=True, b200_motion_queue_repeats=16)
    steps = {"queue-1": task(lib4k, **qover)}
    for S in S_list:
        steps[f"queue-{S}"] = task(lib4k, S, **qover)
        steps[f"fixed-{S}"] = task(lib4k, S, sample_first_motions=True)
        steps[f"fixed-{S}"]._env.fix_mixed_plan()
    for t in steps.values():
        t.set_policy(net, clip_obs=5.0, clip_actions=1.0)

    def round_(name, n_steps):
        t = steps[name]
        if t._q is not None:
            t._start_queue()
        t.reset()
        for k in ("cr", "steps", "prev_dones", "step", "games"):
            t._stats[k].zero_()
        t.clear_motion_stats_games()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for n in range(n_steps):
            t.test_step(n)
            if (n + 1) % t.context_length == 0:
                t._stats["games"].tolist()
        torch.cuda.synchronize()
        ms = (time.perf_counter() - t0) / n_steps * 1e3
        if t._q is not None:
            assert int(t._q["cursor"]) < t._q["game_env"].numel(), "the queue ran dry in the timed window"
            t._check_asset_error()
        return ms, int(t._stats["games"][0])

    for k in steps:
        round_(k, 40)
    step_res, step_games = {k: [] for k in steps}, {}
    for _ in range(a.rounds):
        for k in steps:
            ms, games = round_(k, a.steps)
            step_res[k].append(ms)
            step_games[k] = games
    changed = {k: int((t._q["env_asset"] != t._q["start_env_asset"]).sum()) for k, t in steps.items() if t._q is not None and "env_asset" in t._q}
    del steps
    torch.cuda.synchronize()

    # ---- the library of 32768 motions on 1024 bodies
    S = max(S_list)
    from vid2player3d_b200.tasks.humanoid_smpl_im import HumanoidSMPLIM
    probe = HumanoidSMPLIM.__new__(HumanoidSMPLIM)
    probe.cfg = dict(env=dict(motion_assets=[bodies[m % S] for m in range(lib32k.num_motions())]))
    probe.kp_scale = probe.kd_scale = 1.0
    probe._motion_lib = lib32k
    t0 = time.perf_counter()
    models, _ = probe._motion_asset_models()
    resolve_s = time.perf_counter() - t0
    assert len(models) == S

    def score(S_):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        t = task(lib32k, S_, b200_motion_queue=True)
        torch.cuda.synchronize()
        create = time.perf_counter() - t0
        t1 = time.perf_counter()
        with contextlib.redirect_stdout(io.StringIO()):
            res = t.run_test(net, 1, 100000, print_stats=False, clip_actions=1.0)
        torch.cuda.synchronize()
        run = time.perf_counter() - t1
        got = np.load(os.path.join(tmp, "ms.npz"))
        out = dict(create_s=create, run_s=run, scored=int((got["games"] > 0).sum()), games=res["games_played"])
        extra = None
        if S_ is not None:      # the launch alone on this handle, 200 of them in a CUDA graph as the step graph runs it
            ea, err = t._q["env_asset"], t._q["asset_error"]
            s = torch.cuda.Stream()
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                t._env.set_env_assets(ea, err)
            torch.cuda.current_stream().wait_stream(s)
            gr = torch.cuda.CUDAGraph()
            with torch.cuda.graph(gr):
                for _ in range(200):
                    t._env.set_env_assets(ea, err)
            gr.replay()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(20):
                gr.replay()
            e1.record()
            torch.cuda.synchronize()
            extra = e0.elapsed_time(e1) / 4000 * 1e3
        del t
        torch.cuda.synchronize()
        return out, extra

    def handle_bytes(t, k):
        """device memory a handle of the first k bodies of the library takes (cudaMemGetInfo difference, 2 MiB granularity)"""
        from vid2player3d_b200 import native
        packed = [t._pack(m) for m in models[:k]]
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        free0 = torch.cuda.mem_get_info()[0]
        e = native.Env([p[0] for p in packed], [p[1] for p in packed], t._cfg_struct, N, 0, env_asset=np.arange(N) % k)
        e.fix_mixed_plan()
        torch.cuda.synchronize()
        used = free0 - torch.cuda.mem_get_info()[0]
        e.close()
        return used

    t = task(lib32k, S, b200_motion_queue=True)
    table = {1: handle_bytes(t, 1), S: handle_bytes(t, S)}
    del t
    lib_res = {"queue-1": [], f"queue-{S}": []}
    launch_us = []
    for _ in range(a.rounds):
        for k, S_ in (("queue-1", None), (f"queue-{S}", S)):
            out, extra = score(S_)
            lib_res[k].append(out)
            if extra is not None:
                launch_us.append(extra)
    c = card()
    med = lambda v: sorted(v)[len(v) // 2]  # noqa: E731
    print(f"{c}; {N} envs; {a.rounds} alternating rounds")
    print(f"  graphed test step, 45-frame motions (games end and restart), {a.steps} steps per round:")
    for k in step_res:
        print(f"    {k:10s}: {med(step_res[k]):.3f} ms per step (min {min(step_res[k]):.3f}, max {max(step_res[k]):.3f}); "
              f"{step_games[k]} games finished in the last window" + (f"; {changed[k]} envs off their start body" if k in changed else ""))
    print(f"  library of {lib32k.num_motions()} motions over {S} bodies: asset list resolved in {resolve_s:.2f} s (host)")
    for k, v in lib_res.items():
        f = lambda key: [x[key] for x in v]  # noqa: E731
        print(f"    {k:10s}: create {med(f('create_s')):.2f} s (min {min(f('create_s')):.2f}, max {max(f('create_s')):.2f}), "
              f"run_test {med(f('run_s')):.2f} s (min {min(f('run_s')):.2f}, max {max(f('run_s')):.2f}), "
              f"{v[-1]['scored']} motions scored, {v[-1]['games']} games")
    print(f"    device memory of a handle at {N} envs: {table[1] / 2**20:.1f} MiB with 1 body, {table[S] / 2**20:.1f} MiB with {S} bodies")
    print(f"    b200env_set_env_assets alone at {N} envs: {med(launch_us):.2f} us (min {min(launch_us):.2f}, max {max(launch_us):.2f})")
    print(json.dumps({"card": c, "envs": N, "rounds": a.rounds, "step_ms": step_res, "step_median": {k: med(v) for k, v in step_res.items()},
                      "step_games": step_games, "changed": changed, "resolve_s": resolve_s, "library": lib_res, "set_env_assets_us": launch_us,
                      "handle_bytes": table}))


if __name__ == "__main__":
    main()
