"""Small workload for compute-sanitizer (memcheck / racecheck): a few env steps of every kernel form + the ball generators.
   compute-sanitizer --tool memcheck  python tools/sanitize_smoke.py
   compute-sanitizer --tool racecheck python tools/sanitize_smoke.py"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np
import torch
from helpers import SIM_PARAMS, im_cfg, v2p_cfg
from vid2player3d_b200 import ball_gen, model_compiler, motion_lib
from vid2player3d_b200.tasks import HumanoidSMPLIM, PhysicsMVAEController

model = model_compiler.load_compiled("smpl_mesh_humanoid_amass_v1")
flat = motion_lib.synthetic(model, num_motions=4, num_frames=60, seed=1)
torch.manual_seed(0)
task = HumanoidSMPLIM(im_cfg(70, flat), SIM_PARAMS, 1, "cuda", 0, True)      # 70: a ragged last batch / warp
task.reset()
for _ in range(3):
    task.step(torch.rand(70, 75, device=task.device) * 2 - 1)
task.reset(torch.arange(0, 70, 3, device=task.device))
env = PhysicsMVAEController(v2p_cfg(34, use_history_ball_obs=True), SIM_PARAMS, 1, "cuda", 0, True)
env.reset()
for _ in range(2):
    env.step(torch.clamp(torch.randn(34, env.num_actions, device=env.device), -5, 5))
    env.reset(env.reset_buf.nonzero(as_tuple=False).flatten())
rng = np.random.default_rng(0)
n = 300
pos = np.stack([rng.uniform(-4, 4, n), rng.uniform(12, 13, n), rng.uniform(1, 1.5, n)], 1).astype(np.float32)
vel = np.stack([rng.normal(0, 1, n), -rng.uniform(20, 28, n), rng.uniform(2, 6, n)], 1).astype(np.float32)
ball_gen.simulate(pos, vel, rng.uniform(-8, 8, n).astype(np.float32), num_frames=21)
ball_gen.simulate(pos, vel, rng.uniform(5, 8, n).astype(np.float32), num_frames=50, first_comp=1)
ball_gen.simulate_without_bounce(rng.uniform(10, 65, n).astype(np.float32), rng.uniform(-5, 10, n).astype(np.float32),
                                 rng.uniform(-10, 10, n).astype(np.float32))
torch.cuda.synchronize()
print("sanitize smoke done", float(task.rew_buf.mean()), float(env.rew_buf.mean()))
# dual mode: mask-driven reset incl. the incoming-ball table lookup for every env
from helpers import v2p_dual_cfg
from vid2player3d_b200.tasks import PhysicsMVAEControllerDual
cfg = v2p_dual_cfg(20)
cfg["env"]["motion_player"] = "stream"
dual = PhysicsMVAEControllerDual(cfg, SIM_PARAMS, 1, "cuda", 0, True)
dual.reset()
for _ in range(2):
    dual.step(torch.clamp(torch.randn(20, dual.num_actions, device=dual.device), -5, 5))
    m = torch.zeros(20, dtype=torch.bool, device=dual.device)
    m[4:6] = True
    dual._reset_envs_masked(m)
torch.cuda.synchronize()
print("dual masked reset done", bool(torch.isfinite(dual.obs_buf).all()))
# the wgmma layers and the fused step glue (policy + decoder in the step, masked reset through reset_done)
cfg = v2p_cfg(40)
cfg["env"]["motion_player"], cfg["env"]["low_level_policy"] = "stream+decoder", "b200nn"
env2 = PhysicsMVAEController(cfg, SIM_PARAMS, 1, "cuda", 0, True)
env2.reset()
for i in range(3):
    env2.step(torch.clamp(torch.randn(40, env2.num_actions, device=env2.device), -5, 5))
    m = torch.zeros(40, dtype=torch.bool, device=env2.device)
    m[i::7] = True
    env2._reset_envs_masked(m)
torch.cuda.synchronize()
print("fused step + b200nn done", bool(torch.isfinite(env2.obs_buf).all()), bool(torch.isfinite(env2._low_level_policy.out).all()))
