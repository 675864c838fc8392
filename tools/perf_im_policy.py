"""Test-time step of the embodied_pose imitation policy (HumanoidSMPLIMVis) at 8192 envs, two loops on the same task:

  host:  shaped like the reference's ImitatorPlayer.run (embodied_pose/players/im_player.py:237-304): the network in fp32 torch on the
         device (compute_humanoid_obs on the clamped obs_buf chunks and the context slot, RunningNorm, 734 -> 1024 -> 1024 -> 512 -> 75,
         the residual, the action clamp), the env step, then the statistics with nonzero() / .item() (a host sync every step);
  graph: HumanoidSMPLIMVis.test_step: one CUDA graph replay per step (operand launch, four wgmma layers, step, device bookkeeping).
Both rebuild every env's context window every context_length steps.  Alternating rounds of --steps steps each; prints the median
(min - max) ms per step of each loop with the card's name and power limit read in the same run, and one JSON line.

    python tools/perf_im_policy.py [--envs 8192] [--steps 64] [--rounds 5]"""
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
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, check=True).stdout.strip().splitlines()[0]
        return q
    except Exception:
        return torch.cuda.get_device_name(0) + ", power limit not readable"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=8192)
    ap.add_argument("--steps", type=int, default=64)
    ap.add_argument("--rounds", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("perf_im_policy needs a CUDA device")
    from vid2player3d_b200 import model_compiler, motion_lib
    from vid2player3d_b200.configs import SIM_PARAMS, im_cfg
    from vid2player3d_b200.tasks import HumanoidSMPLIMVis
    N, dev = a.envs, "cuda:0"
    model = model_compiler.load_compiled("smpl_mesh_humanoid_amass_v1")
    flat = motion_lib.synthetic(model, num_motions=16, num_frames=600, seed=1)
    task = HumanoidSMPLIMVis(im_cfg(N, flat, stateInit="Start"), SIM_PARAMS, 1, "cuda", 0, True)
    g = torch.Generator().manual_seed(0)
    dims = (734, 1024, 1024, 512, task.num_actions)
    layers = [((torch.rand(dims[i + 1], dims[i], generator=g) * 2 - 1) / dims[i] ** 0.5 * (0.1 if i == 3 else 1.0),
               torch.zeros(dims[i + 1])) for i in range(4)]
    std = torch.rand(734, generator=g) + 0.5
    net = dict(layers=layers, mean=torch.zeros(734), rstd=1.0 / (std + 1e-8), clip=5.0)
    clip_obs, clip_act = 5.0, 1.0
    task.set_policy(net, clip_obs=clip_obs, clip_actions=clip_act)
    L, nb, nd = task.context_length, task._num_lib_bodies, task.num_dof
    W = [(w.to(dev), b.to(dev)) for w, b in layers]
    mean, sd = net["mean"].to(dev), std.to(dev)

    def torch_act(t):
        obs = torch.clamp(task.obs_buf, -clip_obs, clip_obs)
        ch, o = {}, 0
        for name, d, s in zip(task.obs_names, task.obs_dims, task.obs_shapes):
            ch[name] = obs[:, o:o + d].reshape((N,) + tuple(s))
            o += d
        f = task.context_feat[:, task.context_padding + t]
        tp, tr, td = f[:, :3 * nb].reshape(N, nb, 3), f[:, 3 * nb:7 * nb].reshape(N, nb, 4), f[:, 7 * nb:7 * nb + nd]
        x = task.compute_imitation_obs(ch["body_pos"], ch["body_rot"], tp, tr, ch["dof_pos"], ch["dof_vel"], td, ch["body_vel"],
                                       ch["body_ang_vel"], ch["motion_bodies"], True, True)
        x = torch.clamp((x - mean) / (sd + 1e-8), -5, 5)
        for i, (w, b) in enumerate(W):
            x = torch.nn.functional.linear(x, w, b)
            if i < 3:
                x = torch.relu(x)
        x[:, :nd] += td
        return torch.clamp(x, -clip_act, clip_act)

    def host_round(steps):
        task.reset()
        cr = torch.zeros(N, device=dev)
        st = torch.zeros(N, device=dev)
        prev = torch.zeros(N, device=dev)
        played = 0
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for n in range(steps):
            t = n % L
            if n > 0 and t == 0:
                task._init_context(torch.arange(N, device=dev), task._reset_ref_motion_ids, task._cur_ref_motion_times)
            with torch.no_grad():
                task.step(torch_act(t))
            done = task.reset_buf.float()
            cr += task.rew_buf
            st += 1
            idx = (done * (1 - prev)).nonzero(as_tuple=False)
            if len(idx) > 0:
                played += len(idx)
                cr[idx].sum().item()
                st[idx].sum().item()
                cr = cr * (1.0 - done)
                st = st * (1.0 - done)
            prev = done.clone()
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) / steps * 1e3

    def graph_round(steps):
        task.reset()
        for k in ("cr", "steps", "prev_dones", "step", "games"):
            task._stats[k].zero_()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for n in range(steps):
            task.test_step(n)
            if (n + 1) % L == 0:
                task._stats["games"].tolist()     # the host's read of the stop flag every sync_every = context_length steps
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) / steps * 1e3

    host_round(L + 2)
    graph_round(L + 2)
    res = {"host": [], "graph": []}
    for _ in range(a.rounds):
        res["host"].append(host_round(a.steps))
        res["graph"].append(graph_round(a.steps))
    c = card()
    med = {k: sorted(v)[len(v) // 2] for k, v in res.items()}
    print(f"{c}; {N} envs, {a.rounds} alternating rounds of {a.steps} steps")
    for k in ("host", "graph"):
        print(f"  {k:5s}: {med[k]:.3f} ms per step (min {min(res[k]):.3f}, max {max(res[k]):.3f})")
    print(json.dumps({"card": c, "envs": N, "steps": a.steps, "rounds": a.rounds, "ms_per_step": res, "median": med,
                      "speedup": med["host"] / med["graph"]}))


if __name__ == "__main__":
    main()
