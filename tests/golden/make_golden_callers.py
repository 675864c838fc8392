"""Generates tests/golden/reference_callers.json: what the reference's rl_games-facing code - `VecTaskPythonWrapper`
(embodied_pose/env/tasks/vec_task.py:16-63,120-138, vec_task_wrappers.py:22-28) and `RLGPUEnv.step/reset` (embodied_pose/run.py:93-137) -
touches on a task object when it drives one: reset, three steps, a reset of two envs, get_env_info.  The reference classes run unchanged
(through the isaacgym shim) over a recording stand-in with CPU buffers.  Needs the reference checkout (V2P_REFERENCE); run it from the
repository root: python tests/golden/make_golden_callers.py"""
import json
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))

CODE = r'''
import json, os, sys
sys.path.insert(0, os.path.join(%(root)r, "tests", "golden")); sys.path.insert(0, %(root)r)
import _refenv
_refenv.setup("embodied_pose")
import torch, types
import numpy as _np
if not hasattr(_np, 'Inf'):
    _np.Inf = _np.inf          # the reference targets numpy < 2 (vec_task.py:28-30)
for _pkg in ("agents", "players", "models", "learning"):          # the reference's top-level packages (no __init__.py): make sure they
    _m = types.ModuleType(_pkg)                                  # are not shadowed by same-named site-packages
    _m.__path__ = [os.path.join(_refenv.REF, "embodied_pose", _pkg)]
    sys.modules[_pkg] = _m
import rl_games.common                                             # mocked (rl_games is not installed); RLGPUEnv needs a real base class
_ve = types.ModuleType("rl_games.common.vecenv")
class _IVecEnv: pass
_ve.IVecEnv, _ve.register = _IVecEnv, (lambda *a, **k: None)
rl_games.common.vecenv = sys.modules["rl_games.common.vecenv"] = _ve
from env.tasks.vec_task_wrappers import VecTaskPythonWrapper      # the reference's classes, unchanged
import run as ref_run

class Recorder:
    """stand-in with the buffer contract of BaseTask (base_task.py:62-74); records what the reference code touches"""
    def __init__(self):
        object.__setattr__(self, "touched", set())
        d = dict(num_envs=6, num_obs=461, num_states=0, num_actions=75, obs_buf=torch.randn(6, 461) * 9, states_buf=torch.zeros(6, 0),
                 rew_buf=torch.rand(6), reset_buf=torch.zeros(6, dtype=torch.long), progress_buf=torch.zeros(6, dtype=torch.long),
                 extras={"terminate": torch.zeros(6, dtype=torch.long)}, steps=[])
        object.__setattr__(self, "d", d)
    def __getattr__(self, k):
        self.touched.add(k)
        if k == "step":
            return lambda a: self.d["steps"].append(tuple(a.shape))
        if k == "reset":
            return lambda ids=None: self.d["steps"].append(("reset", None if ids is None else len(ids)))
        return self.d[k]

torch.manual_seed(0)
t = Recorder()
vec = VecTaskPythonWrapper(t, "cpu", 5.0, 1.0)
env = ref_run.RLGPUEnv.__new__(ref_run.RLGPUEnv)     # __init__ only looks the env creator up in rl_games' registry
env.env, env.use_global_obs, env.full_state = vec, vec.num_states > 0, {}
env.full_state["obs"] = env.reset()
obs = env.reset()
for _ in range(3):
    obs, rew, done, info = env.step(torch.randn(6, 75) * 3)
env.reset(torch.tensor([1, 4]))
info_d = env.get_env_info()
print(json.dumps({"touched": sorted(t.touched), "steps": t.d["steps"], "obs_max": float(obs.abs().max()),
                  "n_agents": env.get_number_of_agents(), "info_keys": sorted(info_d)}))
'''

if __name__ == "__main__":
    r = subprocess.run([sys.executable, "-c", CODE % {"root": ROOT}], capture_output=True, text=True, timeout=600)
    if r.returncode != 0:
        sys.exit(r.stdout[-2000:] + r.stderr[-3000:])
    out = json.loads(r.stdout.strip().splitlines()[-1])
    with open(os.path.join(HERE, "reference_callers.json"), "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")
    print(out)
