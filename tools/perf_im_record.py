"""Cost of HumanoidSMPLIMVis' qpos recorder in the graphed test step (HumanoidSMPLIMVis.test_step) at 8192 envs, four loops:

  none:  the graphed step without b200_record_qpos;
  env0:  with the recorder for env 0 (b200env_im_record in the step graph);
  all:   with the recorder for every env;
  host:  the graphed step without the key, plus a host recorder shaped like the reference's _sync_ref_motion: env 0's joint euler
         angles of the state and of the previous target computed by torch on the device, then the root rows and the angles copied
         to the host with .cpu() every frame.
The recorders take no stop flag here, so they write every step whatever env 0's episode does.  Alternating rounds of --steps steps
each (the recorders' frame counters are rewound every round); prints the median (min - max) ms per
step of each loop with the card's name and power limit read in the same run, and one JSON line.

    python tools/perf_im_record.py [--envs 8192] [--steps 64] [--rounds 5]"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                              text=True, check=True).stdout.strip().splitlines()[0]
    except Exception:
        return torch.cuda.get_device_name(0) + ", power limit not readable"


def euler(dof):
    """torch restatement of convert_dof_pos_to_dof_euler (angle_axis_to_quaternion, ypr_euler_from_quat, [2, 1, 0])"""
    a = dof.view(-1, 3)
    th2 = (a * a).sum(-1, keepdim=True)
    th = torch.sqrt(th2.clamp_min(1e-6))
    k = torch.where(th2 > 0, torch.sin(th * 0.5) / th, torch.full_like(th, 0.5))
    w = torch.where(th2 > 0, torch.cos(th * 0.5), torch.ones_like(th))[:, 0]
    x, y, z = (a * k).unbind(-1)

    def atan2(yy, xx):
        yy = yy.clone()
        yy[(yy.abs() < 1e-6) & (xx.abs() < 1e-6)] += 1e-6
        return torch.atan2(yy, xx)
    yaw = atan2(2 * (w * z + x * y), 1 - 2 * (y * y + z * z))
    pitch = torch.asin(torch.clamp(2 * (w * y - x * z), -1 + 1e-6, 1 - 1e-6))
    roll = atan2(2 * (w * x + y * z), 1 - 2 * (x * x + y * y))
    return torch.stack([yaw, pitch, roll], -1).reshape(-1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=8192)
    ap.add_argument("--steps", type=int, default=64)
    ap.add_argument("--rounds", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("perf_im_record needs a CUDA device")
    from vid2player3d_b200 import model_compiler, motion_lib
    from vid2player3d_b200.configs import SIM_PARAMS, im_cfg
    from vid2player3d_b200.tasks import HumanoidSMPLIMVis
    N = a.envs
    model = model_compiler.load_compiled("smpl_mesh_humanoid_amass_v1")
    flat = motion_lib.synthetic(model, num_motions=16, num_frames=600, seed=1)
    g = torch.Generator().manual_seed(0)
    dims = (734, 1024, 1024, 512, 75)
    layers = [((torch.rand(dims[i + 1], dims[i], generator=g) * 2 - 1) / dims[i] ** 0.5 * (0.1 if i == 3 else 1.0),
               torch.zeros(dims[i + 1])) for i in range(4)]
    net = dict(layers=layers, mean=torch.zeros(734), rstd=torch.ones(734), clip=5.0)
    cap = a.steps + 8
    tasks = {}
    for name, over in (("none", {}), ("env0", dict(b200_record_qpos=True)),
                       ("all", dict(b200_record_qpos=True, b200_record_envs="all"))):
        torch.manual_seed(0)
        t = HumanoidSMPLIMVis(im_cfg(N, flat, stateInit="Start", num_rec_frames=cap, **over), SIM_PARAMS, 1, "cuda", 0, True)
        if t._rec is not None:     # the recorder writes every step: no stop flag, so env 0's episode end does not pause it
            t._record_launch = (lambda rec: lambda init, games=None: rec(init))(t._record_launch)
        t.set_policy(net, clip_obs=5.0, clip_actions=1.0)
        tasks[name] = t
    tasks["host"] = tasks["none"]
    frames = []

    def host_frame(t):
        rb = t._rigid_body_state.view(N, -1, 13)
        frames.append((rb[0, 0, :3].cpu().numpy(), rb[0, 0, 3:7].cpu().numpy(), euler(t._dof_pos[0]).cpu().numpy(),
                       t._prev_target_rb_pos[0, 0].cpu().numpy(), t._prev_target_rb_rot[0, 0].cpu().numpy(),
                       euler(t._prev_target_dof_pos[0]).cpu().numpy()))

    def round_(name, steps):
        t = tasks[name]
        t.reset()
        for k in ("cr", "steps", "prev_dones", "step", "games"):
            t._stats[k].zero_()
        if t._rec is not None:
            t._rec["frame"].zero_()
        frames.clear()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for n in range(steps):
            t.test_step(n)
            if name == "host":
                host_frame(t)
            if (n + 1) % t.context_length == 0:
                t._stats["games"].tolist()
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) / steps * 1e3

    names = ("none", "env0", "all", "host")
    for k in names:
        round_(k, 40)
    res = {k: [] for k in names}
    for _ in range(a.rounds):
        for k in names:
            res[k].append(round_(k, a.steps))
    c = card()
    med = {k: sorted(v)[len(v) // 2] for k, v in res.items()}
    print(f"{c}; {N} envs, {a.rounds} alternating rounds of {a.steps} steps")
    for k in names:
        print(f"  {k:5s}: {med[k]:.3f} ms per step (min {min(res[k]):.3f}, max {max(res[k]):.3f})")
    print(json.dumps({"card": c, "envs": N, "steps": a.steps, "rounds": a.rounds, "ms_per_step": res, "median": med}))


if __name__ == "__main__":
    main()
