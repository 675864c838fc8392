"""Caller-side proof of the boundary (SURVEY.md 8b): the REFERENCE's own rl_games-facing code - `VecTaskPythonWrapper`
(embodied_pose/env/tasks/vec_task.py:16-63,120-138, vec_task_wrappers.py:22-28) and `RLGPUEnv.step/reset` (embodied_pose/run.py:93-137).

  * CPU part: tests/golden/reference_callers.json records what those reference classes touch on a task object when they drive it
    (tests/golden/make_golden_callers.py runs them unchanged over a recording stand-in); every attribute / method they touch must be
    provided by the task classes.
  * GPU part: the same call sequence (reset, steps with the wrapper's action / observation clamps, resets of the finished envs) drives
    `vid2player3d_b200.tasks.HumanoidSMPLIM` for 32 steps, and the imitation observation computed on the live GPU buffers matches
    oracle/ref_port.py's restatement of the reference's `compute_humanoid_observations_imitation` (pinned by test_oracle_golden.py)."""
import json
import os
import re

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _provided_names():
    """attributes the task classes define: class members + every `self.<name> =` of their sources (no CUDA needed)"""
    from vid2player3d_b200.tasks import base_task, humanoid_smpl_im
    names = set(dir(humanoid_smpl_im.HumanoidSMPLIM))
    for mod in (base_task, humanoid_smpl_im):
        names |= set(re.findall(r"self\.([A-Za-z_][A-Za-z_0-9]*)\s*(?:,\s*self\.[A-Za-z_0-9]+\s*)*=", open(mod.__file__).read()))
        names |= set(re.findall(r"self\.([A-Za-z_][A-Za-z_0-9]*)", open(mod.__file__).read()))
    return names


def test_reference_vec_task_and_rlgpu_env_touch_only_what_the_b200_task_provides():
    with open(os.path.join(ROOT, "tests", "golden", "reference_callers.json")) as f:
        out = json.load(f)
    provided = _provided_names()
    missing = [n for n in out["touched"] if n not in provided]
    assert not missing, f"the reference's callers touch task attributes the task does not define: {missing}"
    assert out["obs_max"] <= 5.0 and out["n_agents"] == 1 and out["info_keys"] == ["action_space", "observation_space"]
    assert out["steps"][0] == ["reset", None] and out["steps"][-1] == ["reset", 2] and out["steps"].count([6, 75]) == 3


@pytest.mark.gpu
def test_reference_callers_drive_the_b200_task_on_the_gpu():
    from oracle import ref_port as R
    from vid2player3d_b200 import model_compiler, motion_lib
    from vid2player3d_b200.configs import SIM_PARAMS, im_cfg
    from vid2player3d_b200.tasks import HumanoidSMPLIM
    model = model_compiler.load_compiled("smpl_mesh_humanoid_amass_v1")
    flat = motion_lib.synthetic(model, num_motions=6, num_frames=60, seed=3)
    torch.manual_seed(0)
    task = HumanoidSMPLIM(im_cfg(64, flat), SIM_PARAMS, 1, "cuda", 0, True)
    task.reset()
    finite, worst = True, 0.0
    c = lambda x: x.contiguous()  # noqa: E731
    g = lambda x: x.detach().cpu().numpy()  # noqa: E731   float32, as the reference evaluates it
    for i in range(32):
        task.step(torch.clamp(torch.rand(64, 75, device="cuda:0") * 2 - 1, -1.0, 1.0))     # VecTaskPythonWrapper: clip_actions = 1
        obs = torch.clamp(task.obs_buf, -5.0, 5.0)                                         # clip_obs = 5
        finite &= bool(torch.isfinite(obs).all() and torch.isfinite(task.rew_buf).all())
        rbs = task._rigid_body_state.view(64, -1, 13)
        args = (c(rbs[..., 0:3]), c(rbs[..., 3:7]), task._target_rb_pos, task._target_rb_rot, c(task._dof_pos), c(task._dof_vel),
                task._target_dof_pos, c(rbs[..., 7:10]), c(rbs[..., 10:13]), task._reset_ref_motion_bodies)
        ours = task.compute_imitation_obs(*args, True, True)
        ref = R.compute_humanoid_observations_imitation(*[g(a) for a in args], True, True)
        worst = max(worst, float(np.abs(ref - g(ours)).max()))
        ids = task.reset_buf.nonzero(as_tuple=False).flatten()
        if len(ids):
            task.reset(ids)
    assert finite and list(obs.shape) == [64, 461] and "terminate" in task.extras
    assert worst < 1e-5, worst
