"""Per-step time of the test-time task against the training task and a host path shaped like the reference's test-time loop, at the
size of the README's evaluation command (8192 envs), in one run, alternating:

  eval      MVAEControllerVis: step graph (the eval reset rule in the post launch) + render_vis (one recorder launch)
  train     PhysicsMVAEController: step graph
  host      PhysicsMVAEController (is_train False): step graph + the reference's render_vis / _compute_stats on the host - .cpu() copies
            of the six recorded fields appended every step, nonzero() of the recovery flags and .cpu() meter updates
            (mvae_controller_vis.py:81-93, 140-146; utils/common.py:52-63)

Prints one JSON line: the medians and the spread (min, max) over the rounds in ms per step, with the card name and power limit read in
the same run.   python tools/perf_eval.py [--envs 8192] [--steps 50] [--rounds 5]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from vid2player3d_b200.configs import SIM_PARAMS, v2p_cfg  # noqa: E402
from vid2player3d_b200.tasks import MVAEControllerVis, PhysicsMVAEController  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                             text=True, check=True).stdout.strip().splitlines()[0]
        return [x.strip() for x in out.split(",")]
    except Exception as e:   # the timing does not depend on it; say that it could not be read
        return [torch.cuda.get_device_name(0), f"unread ({e.__class__.__name__})", ""]


class HostRecorder:
    """the reference's per-step host work of the test-time task"""

    def __init__(self, env):
        self.env, N = env, env.num_envs
        self.frames = []
        self.meters = {k: (torch.zeros(N), torch.zeros(N, dtype=torch.long), torch.ones(N), torch.zeros(N)) for k in
                       ("hit", "fh", "bin", "err")}

    def _update(self, k, val, ids):
        s, c, a, m = self.meters[k]
        val, ids = val.cpu(), ids.cpu()
        s[ids] += val
        c[ids] += 1
        nz = c > 0
        a[nz] = s[nz] / c[nz]
        m[ids] = torch.where(val > m[ids], val.float(), m[ids])

    def __call__(self):
        e, t = self.env, self.env._physics_player.task
        ids = e._reset_recovery_buf.nonzero(as_tuple=False).flatten()
        if len(ids) > 0:
            self._update("hit", t._has_racket_ball_contact[ids].float(), ids)
            self._update("fh", (e._mvae_player._swing_type_cycle[ids] == 1).float(), ids)
            self._update("bin", e._est_bounce_in[ids].float(), ids)
            ins = ids[e._est_bounce_in[ids]]
            if len(ins) > 0:
                self._update("err", (e._est_bounce_pos[ins] - e._target_bounce_pos[ins]).norm(dim=1), ins)
        self.frames.append([x.cpu() for x in (t._joint_rot, t._root_pos, t._ball_pos, e._target_bounce_pos, e._mvae_player._phase_pred,
                                              e._mvae_player._swing_type_cycle)])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=8192)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("perf_eval needs a CUDA device")
    N, K = a.envs, a.steps
    frames = (a.rounds + 1) * K + 2
    ev_cfg = v2p_cfg(N)
    ev_cfg["env"].update(record=True, num_rec_frames=frames, num_eg=1)
    host_cfg = v2p_cfg(N)
    host_cfg["env"]["is_train"] = False
    envs = dict(eval=MVAEControllerVis(ev_cfg, SIM_PARAMS, 1, "cuda", 0, True), train=PhysicsMVAEController(v2p_cfg(N), SIM_PARAMS, 1, "cuda", 0, True),
                host=PhysicsMVAEController(host_cfg, SIM_PARAMS, 1, "cuda", 0, True))
    host_rec = HostRecorder(envs["host"])
    after = dict(eval=envs["eval"].render_vis, train=lambda: None, host=host_rec)
    for env in envs.values():
        env.enable_cuda_graph()
        env.reset()
    envs["eval"].render_vis(init=True)
    acts = torch.zeros(N, envs["eval"].num_actions, device="cuda")

    def run(name, k):
        env, post = envs[name], after[name]
        start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        start.record()
        for _ in range(k):
            env.reset_done()
            env.step(acts.normal_())
            post()
        end.record()
        torch.cuda.synchronize()
        return start.elapsed_time(end) / k

    for name in envs:                       # warm-up round
        run(name, K)
    times = {name: [] for name in envs}
    for _ in range(a.rounds):
        for name in envs:
            times[name].append(run(name, K))
    name, plim, smax = card()
    med = lambda v: sorted(v)[len(v) // 2]  # noqa: E731
    print(json.dumps(dict(gpu=name, power_limit=plim, sm_clock_max=smax, envs=N, steps_per_round=K, rounds=a.rounds,
                          ms_per_step={k: dict(median=round(med(v), 4), min=round(min(v), 4), max=round(max(v), 4)) for k, v in times.items()},
                          eval_over_train=round(med(times["eval"]) / med(times["train"]), 4))))


if __name__ == "__main__":
    main()
