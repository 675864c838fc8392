"""Cost and benefit of HumanoidSMPLIMVis' motion queue (cfg.env.b200_motion_queue) at 8192 envs, two measurements:

  library: the wall time to score a 4 x 8192-motion library - one task with the queue, against four tasks over 8192-motion slices with
           sample_first_motions (the way without the queue), each built, run and exported in the round (task construction, motion
           library upload, graph capture and run_test).  The library repeats 1024 distinct synthetic motions of 45 frames, so its
           generation stays short; each motion is scored on its own all the same.
  step:    the graphed test step with the queue (its assignment launch and the masked reset's two launches, every step) against the
           step without it, on 300-frame motions without early termination, so that no game finishes in the timed window.
Alternating rounds; prints the median (min - max) of each with the card's name and power limit read in the same run, and one JSON line.

    python tools/perf_im_motion_queue.py [--envs 8192] [--rounds 5] [--steps 64]"""
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=8192)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=64)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("perf_im_motion_queue needs a CUDA device")
    import numpy as np
    from vid2player3d_b200 import model_compiler, motion_lib
    from vid2player3d_b200.configs import SIM_PARAMS, im_cfg
    from vid2player3d_b200.tasks import HumanoidSMPLIMVis
    N = a.envs
    model = model_compiler.load_compiled("smpl_mesh_humanoid_amass_v1")
    base = motion_lib.synthetic(model, num_motions=1024, num_frames=45, seed=1)
    slice_lib = motion_lib.FlatMotionLib.merge([base] * (N // 1024))
    full = motion_lib.FlatMotionLib.merge([slice_lib] * 4)
    g = torch.Generator().manual_seed(0)
    dims = (734, 1024, 1024, 512, 75)
    layers = [((torch.rand(dims[i + 1], dims[i], generator=g) * 2 - 1) / dims[i] ** 0.5 * (0.1 if i == 3 else 1.0),
               torch.zeros(dims[i + 1])) for i in range(4)]
    net = dict(layers=layers, mean=torch.zeros(734), rstd=torch.ones(734), clip=5.0)
    tmp = tempfile.mkdtemp()

    def task(flat, **over):
        torch.manual_seed(0)
        cfg = im_cfg(N, flat, stateInit="Start", b200_motion_stats=True, b200_motion_stats_file=os.path.join(tmp, "ms.npz"), **over)
        return HumanoidSMPLIMVis(cfg, SIM_PARAMS, 1, "cuda", 0, True)

    def score(tasks_over):
        """(seconds, motions with a finished game, games) of building, running and exporting each (library, cfg) in turn"""
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        scored = games = 0
        for flat, over in tasks_over:
            t = task(flat, **over)
            with contextlib.redirect_stdout(io.StringIO()):
                t.run_test(net, 1, 3000, print_stats=False, clip_actions=1.0)
            got = np.load(os.path.join(tmp, "ms.npz"))
            scored += int((got["games"] > 0).sum())
            games += int(got["games"].sum())
            del t
        torch.cuda.synchronize()
        return time.perf_counter() - t0, scored, games

    lib_runs = {"queue": [(full, dict(b200_motion_queue=True))], "slices": [(slice_lib, dict(sample_first_motions=True))] * 4}
    lib_res = {k: [] for k in lib_runs}
    lib_scored = {}
    for _ in range(a.rounds):
        for k, runs in lib_runs.items():
            s, scored, games = score(runs)
            lib_res[k].append(s)
            lib_scored[k] = (scored, games)

    # the step: no game finishes in the window (300-frame motions, no early termination)
    long_lib = motion_lib.synthetic(model, num_motions=512, num_frames=300, seed=2)
    steps = {"without": task(long_lib, sample_first_motions=True, enableEarlyTermination=False),
             "queue": task(long_lib, b200_motion_queue=True, b200_motion_queue_repeats=N // 512 + 1, enableEarlyTermination=False)}
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
        assert int(t._stats["games"][0]) == 0, "a game finished in the timed window"
        return (time.perf_counter() - t0) / n_steps * 1e3

    for k in steps:
        round_(k, 40)
    step_res = {k: [] for k in steps}
    for _ in range(a.rounds):
        for k in steps:
            step_res[k].append(round_(k, a.steps))
    c = card()
    med = lambda v: sorted(v)[len(v) // 2]  # noqa: E731
    print(f"{c}; {N} envs; {a.rounds} alternating rounds")
    print(f"  library of {full.num_motions()} motions, build + run + export:")
    for k in lib_res:
        print(f"    {k:7s}: {med(lib_res[k]):.2f} s (min {min(lib_res[k]):.2f}, max {max(lib_res[k]):.2f}); "
              f"{lib_scored[k][0]} motions scored, {lib_scored[k][1]} games")
    print(f"  graphed test step, no game finishing, {a.steps} steps per round:")
    for k in step_res:
        print(f"    {k:7s}: {med(step_res[k]):.3f} ms per step (min {min(step_res[k]):.3f}, max {max(step_res[k]):.3f})")
    print(json.dumps({"card": c, "envs": N, "rounds": a.rounds, "library_s": lib_res, "library_scored": lib_scored,
                      "step_ms": step_res, "step_median": {k: med(v) for k, v in step_res.items()}}))


if __name__ == "__main__":
    main()
