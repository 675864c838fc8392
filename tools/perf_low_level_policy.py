"""Cost of the tennis controller's trained low-level imitation policy inside the high-level step (PhysicsMVAEController(Dual).step, with
the mask-driven reset_done), single player at 8192 envs and dual at 2 x 8192 (16384 envs), in one run, alternating:

  policy alone   trained  nn.V2PPolicy.forward_prepared: single one chain of four wgmma layers over N rows, dual two chains of N/2 rows
                 b200nn   nn.PolicyMLP.forward_prepared of the random `low_level_policy: b200nn` policy of the same shape: one chain of N
                 torch    the reference's fp32 eval_actor (RunningNorm, actor MLP, mu); dual on obs[0::2] / obs[1::2], cat + reshape back
  step           trained  the graphed step (enable_cuda_graph) driven by physics.pretrained_model_cp / dual_model_cp
                 b200nn   the graphed step with the random b200nn policy
                 torch    the step run eagerly from the host with the torch policy above (the loop as the reference runs it)

The trained networks are random checkpoints of the shipped shape (734 -> 1024 -> 1024 -> 512 -> 75) written to a temporary directory.
Prints one JSON line: medians and spread (min, max) over the rounds in ms, with the card name, power limit and max SM clock read in
the same run.
   python tools/perf_low_level_policy.py [--envs 8192] [--steps 20] [--rounds 5]
"""
import argparse
import json
import os
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from perf_eval import card  # noqa: E402
from vid2player3d_b200 import nn  # noqa: E402
from vid2player3d_b200.configs import SIM_PARAMS, v2p_cfg, v2p_dual_cfg  # noqa: E402
from vid2player3d_b200.tasks import PhysicsMVAEController, PhysicsMVAEControllerDual  # noqa: E402

OBS, ACT = 734, 75


def write_checkpoints(tmp, P, seed=0):
    """embodied_pose-style checkpoints of the shipped actor shape with RunningNorm statistics"""
    g = torch.Generator().manual_seed(seed)
    dims = (OBS, 1024, 1024, 512, ACT)
    paths = []
    for p in range(P):
        model = {}
        for i, k in enumerate(("actor_mlp.0", "actor_mlp.2", "actor_mlp.4", "mu")):
            model[f"a2c_network.{k}.weight"] = (torch.rand(dims[i + 1], dims[i], generator=g) * 2 - 1) / dims[i] ** 0.5
            model[f"a2c_network.{k}.bias"] = (torch.rand(dims[i + 1], generator=g) * 2 - 1) / dims[i] ** 0.5
        std = torch.rand(OBS, generator=g) + 0.5
        model.update({"a2c_network.running_obs.n": torch.tensor(1000), "a2c_network.running_obs.mean": torch.randn(OBS, generator=g) * 0.1,
                      "a2c_network.running_obs.std": std, "a2c_network.running_obs.var": std ** 2})
        paths.append(os.path.join(tmp, f"im_{p}.pth"))
        torch.save({"model": model}, paths[-1])
    return paths


class TorchPolicy:
    """the reference's fp32 eval_actor per network (RunningNorm: clamp((x - mean) / (std + 1e-8), -5, 5)); ImitatorBuilderDual splits
    the rows 0::2 / 1::2 and interleaves the outputs back with cat + reshape (im_network_builder_dual.py:37-45)"""

    def __init__(self, nets, dev):
        self.nets = [dict(layers=[(w.to(dev), b.to(dev)) for w, b in n["layers"]], mean=n["mean"].to(dev), rstd=n["rstd"].to(dev)) for n in nets]

    @torch.no_grad()
    def __call__(self, obs):
        outs = []
        P = len(self.nets)
        for p, n in enumerate(self.nets):
            x = torch.clamp((obs[p::P] - n["mean"]) * n["rstd"], -5, 5)
            for i, (w, b) in enumerate(n["layers"]):
                x = torch.addmm(b, x, w.T)
                if i < 3:
                    x = torch.relu(x)
            outs.append(x)
        if P == 1:
            return outs[0]
        return torch.cat([outs[0].unsqueeze(1), outs[1].unsqueeze(1)], dim=1).reshape(-1, outs[0].shape[1])


def timed(fn, k):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    start.record()
    for _ in range(k):
        fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / k


def measure(mode, N, K, rounds, tmp):
    P = 2 if mode == "dual" else 1
    paths = write_checkpoints(tmp, P)
    nets = nn.low_level_networks_from_cfg(dict(dual_model_cp=paths) if P == 2 else dict(pretrained_model_cp=paths[0]), OBS, ACT, P == 2)

    def make(policy=None, trained=False):
        cfg = v2p_dual_cfg(N) if mode == "dual" else v2p_cfg(N)
        if trained:
            cfg["env"]["physics"].update(dual_model_cp=paths) if P == 2 else cfg["env"]["physics"].update(pretrained_model_cp=paths[0])
        if policy is not None:
            cfg["env"]["low_level_policy"] = policy
        env = (PhysicsMVAEControllerDual if mode == "dual" else PhysicsMVAEController)(cfg, SIM_PARAMS, 1, "cuda", 0, True)
        env.reset()
        return env
    torch_policy = TorchPolicy(nets, "cuda:0")
    envs = dict(trained=make(trained=True), b200nn=make("b200nn"), torch=make(torch_policy))
    assert isinstance(envs["trained"]._low_level_policy, nn.V2PPolicy) and isinstance(envs["b200nn"]._low_level_policy, nn.PolicyMLP)
    for k in ("trained", "b200nn"):
        envs[k].enable_cuda_graph()
    actions = torch.clamp(torch.randn(N, envs["trained"].num_actions, device="cuda:0", generator=torch.Generator("cuda:0").manual_seed(1)), -5, 5)

    def stepper(env):
        def f():
            env.step(actions)
            env.reset_done()
        return f
    obs = envs["torch"]._physics_player.task.obs_buf
    fns = dict(policy_trained=envs["trained"]._low_level_policy.forward_prepared, policy_b200nn=envs["b200nn"]._low_level_policy.forward_prepared,
               policy_torch=lambda: torch_policy(obs), step_trained=stepper(envs["trained"]), step_b200nn=stepper(envs["b200nn"]),
               step_torch=stepper(envs["torch"]))
    for f in fns.values():                  # warm-up round: module loads, cuBLAS algorithm choice, first replays
        timed(f, K)
    times = {k: [] for k in fns}
    for _ in range(rounds):
        for k, f in fns.items():
            times[k].append(timed(f, K))
    med = lambda v: sorted(v)[len(v) // 2]  # noqa: E731
    return dict(envs=N, networks=P, policy_gflop=round(envs["trained"]._low_level_policy.flops / 1e9, 3),
                ms={k: dict(median=round(med(v), 4), min=round(min(v), 4), max=round(max(v), 4)) for k, v in times.items()})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=8192)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("perf_low_level_policy needs a CUDA device")
    with tempfile.TemporaryDirectory() as tmp:
        res = dict(single=measure("single", a.envs, a.steps, a.rounds, tmp), dual=measure("dual", 2 * a.envs, a.steps, a.rounds, tmp))
    name, plim, smax = card()
    print(json.dumps(dict(gpu=name, power_limit=plim, sm_clock_max=smax, steps_per_round=a.steps, rounds=a.rounds, **res)))


if __name__ == "__main__":
    main()
